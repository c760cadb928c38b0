// torch_ext.cpp -- thin PyTorch shim over the fdgs C-ABI (include/fdgs.h).
//
// Exposes the same three functions, with the same positional arguments and return tuples, as
// the reference's extension module (reference: diff-gaussian-rasterization/ext.cpp:15-19,
// rasterize_points.h:18-93, rasterize_points.cu:36-291), so that the reference's own
// gaussian_renderer/diff_gaussian_rasterization.py could be pointed at this module unchanged:
//
//   rasterize_gaussians(30 args)          -> (num_rendered, color, flow, depth, T, radii,
//                                             geomBuffer, binningBuffer, imgBuffer, covs3D_com, out_means3D)
//   rasterize_gaussians_backward(37 args) -> 12 gradient tensors
//   mark_visible(means3D, viewmatrix, projmatrix) -> bool[P]
//
// and one extended entry per direction, which the autograd Function of this package calls:
//
//   rasterize_gaussians_ext(30 args, sh_rest, raw_params, bg_image[, dL_dsh, dL_dsh_rest])  -> the same 11-tuple
//   rasterize_gaussians_backward_ext(37 args, sh_rest, raw_params, bg_image, sh_factor_mode, want_dbg[, dL_dsh,
//                                    dL_dsh_rest])  -> [12 gradients, sh_factors, dL_dsh_rest, dL_dbg_image]
//
// and a batched pair over B cameras of the same Gaussians (include/fdgs.h: fdgs_forward_batch):
//
//   rasterize_gaussians_batch / rasterize_gaussians_backward_batch
//
// and the backward with the camera gradients (include/fdgs.h: fdgs_backward_camera), single-view and batched:
//
//   rasterize_gaussians_backward_camera / rasterize_gaussians_backward_batch_camera
//
// and the batched forward sized by an instance capacity, which never synchronises (include/fdgs.h:
// fdgs_forward_batch_capacity): rasterize_gaussians_batch_capacity
//
// PyTorch is plumbing only: it owns the memory (tensors, the three growable byte buffers handed
// to the library through the allocation callback) and supplies the current CUDA stream.  No
// arithmetic happens here.  Differences from the reference shim, all performance-motivated and
// invisible to callers: outputs are torch::empty (the kernels write every element; the
// reference zero-fills 7 image planes in forward and 716 B/Gaussian in backward), out_means3D is
// written by the preprocess kernel instead of cloned, covs3D_com is an owning view into
// geomBuffer instead of a dangling from_blob alias (reference: rasterize_points.cu:147), and
// launches go to the current stream instead of the legacy default stream.
#include <torch/extension.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <memory>
#include <string>
#include <tuple>
#include <vector>
#include "../../include/fdgs.h"

namespace {

char* resize_cb(void* ctx, size_t bytes) {
    auto* t = reinterpret_cast<torch::Tensor*>(ctx);
    t->resize_({(long long)bytes});
    return reinterpret_cast<char*>(t->data_ptr());
}

void check(int rc, const char* where) {
    if (rc != FDGS_OK) throw std::runtime_error(std::string("fdgs ") + where + " failed: " + fdgs_last_error());
}

// The device guard and current stream every launch of a binding runs under.
struct DeviceStream {
    c10::cuda::CUDAGuard guard;
    cudaStream_t stream;
    explicit DeviceStream(const torch::Tensor& t) : guard(t.device()), stream(c10::cuda::getCurrentCUDAStream().stream()) {}
};

// ---- the rasterizer's contract (the reference's): any layout is accepted and copied contiguous; an empty tensor is
// "not provided", a null pointer in C (reference: diff_gaussian_rasterization.py:282-300) ----------------------------
const float* fptr(const torch::Tensor& t) {
    if (!t.defined() || t.numel() == 0) return nullptr;
    TORCH_CHECK(t.is_cuda(), "fdgs: expected a CUDA tensor");
    TORCH_CHECK(t.scalar_type() == torch::kFloat32, "fdgs: expected a float32 tensor");
    return t.data_ptr<float>();
}

torch::Tensor contig(const torch::Tensor& t) { return (t.defined() && t.numel() > 0) ? t.contiguous() : t; }

bool provided(const torch::Tensor& t) { return t.defined() && t.numel() != 0; }

// The contiguous copies of a call's input tensors, kept alive until the call returns
struct Inputs {
    std::vector<torch::Tensor> held;
    const float* operator()(const torch::Tensor& t) {
        held.push_back(contig(t));
        return fptr(held.back());
    }
    const char* bytes(const torch::Tensor& t) {
        held.push_back(contig(t));
        return provided(held.back()) ? reinterpret_cast<const char*>(held.back().data_ptr()) : nullptr;
    }
};

// SH coefficients per Gaussian: sh [P,M,3], or the raw-parameter entry's split rows sh [P,1,3] + sh_rest [P,M-1,3]
int sh_coefficients(const torch::Tensor& sh, const torch::Tensor& sh_rest) {
    return (provided(sh) ? (int)sh.size(1) : 0) + (provided(sh_rest) ? (int)sh_rest.size(1) : 0);
}

// The fields of fdgs_forward_args that the single-view and the batched binding fill alike: the Gaussians, the
// background colour, the image size and the flags.  The camera, the outputs and the precomputed colours / covariances
// are the caller's.
void forward_gaussians(fdgs_forward_args& a, Inputs& in, const torch::Tensor& background, const torch::Tensor& means3D,
                       const torch::Tensor& flows, const torch::Tensor& opacity, const torch::Tensor& ts,
                       const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                       const torch::Tensor& rotations_r, float scale_modifier, float prefilter_var, const torch::Tensor& sh,
                       const torch::Tensor& sh_rest, int degree, int degree_t, float time_duration, bool rot_4d,
                       int gaussian_dim, bool force_sh_3d, bool prefiltered, bool debug, bool raw_params, int H, int W) {
    a.P = means3D.size(0); a.D = degree; a.D_t = degree_t; a.M = sh_coefficients(sh, sh_rest);
    if (provided(sh_rest))
        TORCH_CHECK(provided(sh) && sh.size(1) == 1 && sh_rest.dim() == 3 && sh_rest.size(0) == a.P,
                    "fdgs: split SH rows are [P,1,3] + [P,M-1,3]");
    a.shs_rest = in(sh_rest); a.raw_params = raw_params;
    a.background = in(background); a.width = W; a.height = H;
    a.means3D = in(means3D); a.shs = in(sh); a.flows_precomp = in(flows);
    a.opacities = in(opacity); a.ts = in(ts); a.scales = in(scales); a.scales_t = in(scales_t);
    a.scale_modifier = scale_modifier; a.rotations = in(rotations); a.rotations_r = in(rotations_r);
    a.prefilter_var = prefilter_var; a.time_duration = time_duration; a.rot_4d = rot_4d; a.gaussian_dim = gaussian_dim;
    a.force_sh_3d = force_sh_3d; a.prefiltered = prefiltered; a.debug = debug;
}

// The same for fdgs_backward_args, with the forward's scratch buffers and the image gradients
void backward_gaussians(fdgs_backward_args& a, Inputs& in, const torch::Tensor& background, const torch::Tensor& means3D,
                        const torch::Tensor& flows, const torch::Tensor& opacities, const torch::Tensor& ts,
                        const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                        const torch::Tensor& rotations_r, float scale_modifier, float prefilter_var, const torch::Tensor& sh,
                        const torch::Tensor& sh_rest, int degree, int degree_t, float time_duration, bool rot_4d,
                        int gaussian_dim, bool force_sh_3d, bool debug, bool raw_params, int H, int W,
                        const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_depth,
                        const torch::Tensor& dL_dout_mask, const torch::Tensor& dL_dout_flow,
                        const torch::Tensor& geomBuffer, int R, const torch::Tensor& binningBuffer,
                        const torch::Tensor& imageBuffer) {
    a.P = means3D.size(0); a.D = degree; a.D_t = degree_t; a.M = sh_coefficients(sh, sh_rest); a.R = R;
    a.shs_rest = in(sh_rest); a.raw_params = raw_params;
    a.background = in(background); a.width = W; a.height = H;
    a.shs = in(sh); a.flows_2d = in(flows);
    a.opacities = in(opacities); a.ts = in(ts); a.scales = in(scales); a.scales_t = in(scales_t);
    a.scale_modifier = scale_modifier; a.rotations = in(rotations); a.rotations_r = in(rotations_r);
    a.prefilter_var = prefilter_var; a.time_duration = time_duration; a.rot_4d = rot_4d; a.gaussian_dim = gaussian_dim;
    a.force_sh_3d = force_sh_3d; a.debug = debug;
    a.geom_buffer = in.bytes(geomBuffer); a.binning_buffer = in.bytes(binningBuffer); a.image_buffer = in.bytes(imageBuffer);
    a.dL_dpix = in(dL_dout_color); a.dL_depths = in(dL_dout_depth); a.dL_masks = in(dL_dout_mask);
    a.dL_dpix_flow = in(dL_dout_flow);
}

// the per-pixel background image of a call, checked against the image size (undefined / empty = none)
torch::Tensor background_image(const torch::Tensor& bg_image, const torch::Tensor& like, int H, int W) {
    if (!bg_image.defined() || bg_image.numel() == 0) return torch::Tensor();
    TORCH_CHECK(bg_image.is_cuda() && bg_image.device() == like.device(), "fdgs: bg_image must be on the device of means3D");
    TORCH_CHECK(bg_image.scalar_type() == torch::kFloat32, "fdgs: bg_image must be float32");
    TORCH_CHECK(bg_image.dim() == 3 && bg_image.size(0) == 3 && bg_image.size(1) == H && bg_image.size(2) == W,
                "fdgs: bg_image must be [3, image_height, image_width]");
    return bg_image.contiguous();
}

// an SH gradient tensor handed in by the caller to be written in place: float32, contiguous, [P,m,3], on the device of
// means3D (undefined / empty = none)
float* sh_grad_rows(const torch::Tensor& t, const char* name, const torch::Tensor& like, int64_t P, int64_t m) {
    if (!provided(t)) return nullptr;
    TORCH_CHECK(t.is_cuda() && t.device() == like.device(), "fdgs: ", name, " must be on the device of means3D");
    TORCH_CHECK(t.scalar_type() == torch::kFloat32 && t.is_contiguous(), "fdgs: ", name, " must be contiguous float32");
    TORCH_CHECK(t.dim() == 3 && t.size(0) == P && t.size(1) == m && t.size(2) == 3, "fdgs: ", name, " has the wrong shape");
    return t.data_ptr<float>();
}

// ---- the training-step bindings' strict contract: no copies, so a tensor of the wrong dtype, layout or shape is an
// error.  dtype, layout and shape of every argument are checked first (arg), then the device (same_cuda_device), and
// only then is anything allocated or launched: a malformed call fails before any GPU work. ---------------------------

// "Float (float32)": ATen's name of a dtype and torch's
std::string dtype_name(torch::ScalarType t) {
    return std::string(c10::toString(t)) + " (" + c10::getDtypeNames(t).first + ")";
}

constexpr bool REQUIRED = true;

// The data pointer of tensor argument `name`: dtype T, contiguous, `rows` rows (size(0); < 0: any) and `numel`
// elements (< 0: any).  An undefined or empty optional tensor is "not provided" (nullptr; the C-ABI rejects a null it
// needs); a required one is checked like any other.
template <typename T>
T* arg(const torch::Tensor& t, const char* name, int64_t rows = -1, int64_t numel = -1, bool required = false) {
    TORCH_CHECK(!required || t.defined(), "fdgs: ", name, " is required");
    if (!t.defined() || (!required && t.numel() == 0)) return nullptr;
    const torch::ScalarType dtype = c10::CppTypeToScalarType<T>::value;
    TORCH_CHECK(t.scalar_type() == dtype, "fdgs: ", name, " must be ", dtype_name(dtype));
    TORCH_CHECK(t.is_contiguous(), "fdgs: ", name, " must be contiguous");
    TORCH_CHECK((rows < 0 || (t.dim() >= 1 && t.size(0) == rows)) && (numel < 0 || t.numel() == numel), "fdgs: ", name,
                " has the wrong shape");
    return t.data_ptr<T>();
}

// every provided (defined, non-empty) tensor of a call on one CUDA device, that of the first
void same_cuda_device(const char* what, const std::vector<torch::Tensor>& ts) {
    const torch::Tensor* first = nullptr;
    for (const torch::Tensor& t : ts) {
        if (!t.defined() || t.numel() == 0) continue;
        TORCH_CHECK(t.is_cuda(), "fdgs: ", what, " tensors must be CUDA tensors");
        if (!first) first = &t;
        TORCH_CHECK(t.device() == first->device(), "fdgs: ", what, " tensors on different devices");
    }
}

}  // namespace

using ForwardOut = std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
                              torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>;

// The reference's 30 arguments (rasterize_points.h:18-49) + the extensions of include/fdgs.h, each empty / false when
// unused: sh_rest and raw_params, the raw-parameter entry (fdgs_forward_args.raw_params: scales = log-scales, rotations
// un-normalised, opacity = logits; sh = features_dc [P,1,3], sh_rest = features_rest [P,M-1,3]), and bg_image, a
// per-pixel background [3,H,W] (fdgs_forward_bg).  Returns the reference's 11-tuple.
// dL_dsh / dL_dsh_rest: the SH gradient tensors the backward will return (shaped as it returns them); the forward then
// zeroes the rows of the Gaussians it does not render (fdgs_forward_zero_sh).  Empty: not provided.
ForwardOut RasterizeGaussiansExtZeroSh(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors,
                                 const torch::Tensor& flows, const torch::Tensor& opacity, const torch::Tensor& ts,
                                 const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                                 const torch::Tensor& rotations_r, const float scale_modifier,
                                 const torch::Tensor& cov3D_precomp, const float prefilter_var,
                                 const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
                                 const float tan_fovy, const int image_height, const int image_width,
                                 const torch::Tensor& sh, const int degree, const int degree_t, const torch::Tensor& campos,
                                 const float timestamp, const float time_duration, const bool rot_4d,
                                 const int gaussian_dim, const bool force_sh_3d, const bool prefiltered, const bool debug,
                                 const torch::Tensor& sh_rest, const bool raw_params, const torch::Tensor& bg_image,
                                 const torch::Tensor& dL_dsh, const torch::Tensor& dL_dsh_rest) {
    if (means3D.ndimension() != 2 || means3D.size(1) != 3) {
        AT_ERROR("means3D must have dimensions (num_points, 3)");   // reference: rasterize_points.cu:69-71
    }
    TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor");
    const DeviceStream on(means3D);

    const int P = means3D.size(0);
    const int H = image_height, W = image_width;
    auto fopts = means3D.options().dtype(torch::kFloat32);
    auto iopts = means3D.options().dtype(torch::kInt32);
    auto bopts = means3D.options().dtype(torch::kByte);

    torch::Tensor out_color = torch::empty({3, H, W}, fopts);
    torch::Tensor out_flow = torch::empty({2, H, W}, fopts);
    torch::Tensor out_depth = torch::empty({1, H, W}, fopts);
    torch::Tensor out_T = torch::empty({1, H, W}, fopts);
    torch::Tensor radii = torch::empty({P}, iopts);
    torch::Tensor out_means3D = torch::empty({P, 3}, fopts);
    torch::Tensor geomBuffer = torch::empty({0}, bopts);
    torch::Tensor binningBuffer = torch::empty({0}, bopts);
    torch::Tensor imgBuffer = torch::empty({0}, bopts);

    fdgs_forward_args a;
    memset(&a, 0, sizeof(a));
    Inputs in;
    forward_gaussians(a, in, background, means3D, flows, opacity, ts, scales, scales_t, rotations, rotations_r, scale_modifier,
                      prefilter_var, sh, sh_rest, degree, degree_t, time_duration, rot_4d, gaussian_dim, force_sh_3d,
                      prefiltered, debug, raw_params, H, W);
    a.colors_precomp = in(colors); a.cov3D_precomp = in(cov3D_precomp);
    a.viewmatrix = in(viewmatrix); a.projmatrix = in(projmatrix); a.cam_pos = in(campos);
    a.timestamp = timestamp; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
    a.out_means3D = out_means3D.data_ptr<float>(); a.out_color = out_color.data_ptr<float>();
    a.out_flow = out_flow.data_ptr<float>(); a.out_depth = out_depth.data_ptr<float>();
    a.out_T = out_T.data_ptr<float>(); a.radii = radii.data_ptr<int>();

    const auto bgi_c = background_image(bg_image, means3D, H, W);
    float* zero_sh = sh_grad_rows(dL_dsh, "dL_dsh", means3D, P, provided(sh_rest) ? 1 : a.M);
    float* zero_sh_rest = sh_grad_rows(dL_dsh_rest, "dL_dsh_rest", means3D, P, a.M - 1);
    fdgs_forward_result r;
    check(fdgs_forward_zero_sh(&a, fptr(bgi_c), zero_sh, zero_sh_rest, resize_cb, &geomBuffer, resize_cb, &binningBuffer,
                               resize_cb, &imgBuffer, (void*)on.stream, &r),
          "forward");

    torch::Tensor covs3D_com;
    if (P > 0) {
        const int64_t off = reinterpret_cast<const char*>(r.cov3D) - reinterpret_cast<const char*>(geomBuffer.data_ptr());
        covs3D_com = geomBuffer.narrow(0, off, (int64_t)P * 24).view(torch::kFloat32).view({P, 6});
    } else {
        covs3D_com = torch::empty({0, 6}, fopts);
    }
    return std::make_tuple(r.num_rendered, out_color, out_flow, out_depth, out_T, radii, geomBuffer, binningBuffer,
                           imgBuffer, covs3D_com, out_means3D);
}

ForwardOut RasterizeGaussiansExt(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors,
                                 const torch::Tensor& flows, const torch::Tensor& opacity, const torch::Tensor& ts,
                                 const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                                 const torch::Tensor& rotations_r, const float scale_modifier,
                                 const torch::Tensor& cov3D_precomp, const float prefilter_var,
                                 const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
                                 const float tan_fovy, const int image_height, const int image_width,
                                 const torch::Tensor& sh, const int degree, const int degree_t, const torch::Tensor& campos,
                                 const float timestamp, const float time_duration, const bool rot_4d,
                                 const int gaussian_dim, const bool force_sh_3d, const bool prefiltered, const bool debug,
                                 const torch::Tensor& sh_rest, const bool raw_params, const torch::Tensor& bg_image) {
    return RasterizeGaussiansExtZeroSh(background, means3D, colors, flows, opacity, ts, scales, scales_t, rotations,
                                       rotations_r, scale_modifier, cov3D_precomp, prefilter_var, viewmatrix, projmatrix,
                                       tan_fovx, tan_fovy, image_height, image_width, sh, degree, degree_t, campos, timestamp,
                                       time_duration, rot_4d, gaussian_dim, force_sh_3d, prefiltered, debug, sh_rest,
                                       raw_params, bg_image, torch::Tensor(), torch::Tensor());
}

// the reference's entry point: 30 positional arguments, 11-tuple (rasterize_points.h:18-49)
ForwardOut RasterizeGaussiansCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors,
                                  const torch::Tensor& flows, const torch::Tensor& opacity, const torch::Tensor& ts,
                                  const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                                  const torch::Tensor& rotations_r, const float scale_modifier,
                                  const torch::Tensor& cov3D_precomp, const float prefilter_var,
                                  const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
                                  const float tan_fovy, const int image_height, const int image_width,
                                  const torch::Tensor& sh, const int degree, const int degree_t, const torch::Tensor& campos,
                                  const float timestamp, const float time_duration, const bool rot_4d,
                                  const int gaussian_dim, const bool force_sh_3d, const bool prefiltered, const bool debug) {
    return RasterizeGaussiansExt(background, means3D, colors, flows, opacity, ts, scales, scales_t, rotations, rotations_r,
                                 scale_modifier, cov3D_precomp, prefilter_var, viewmatrix, projmatrix, tan_fovx, tan_fovy,
                                 image_height, image_width, sh, degree, degree_t, campos, timestamp, time_duration, rot_4d,
                                 gaussian_dim, force_sh_3d, prefiltered, debug, torch::Tensor(), false, torch::Tensor());
}

// The reference's 37 arguments (rasterize_points.h:51-89) + the forward's sh_rest, raw_params and bg_image, and:
//   sh_factor_mode: the view-parallel mode -- no dL_dsh rows, the [P,3] colour factors instead (include/fdgs.h: sh_factors)
//   want_dbg:       whether dL/dbg_image is wanted (fdgs_backward_bg)
//   sh_grad / sh_rest_grad: the tensors the forward zeroed (rasterize_gaussians_ext's dL_dsh / dL_dsh_rest), returned
//                   as the SH gradient with their rendered rows written (fdgs_backward_zero_sh); empty: allocated here
// Returns 15 tensors: the 12 gradients (w.r.t. the raw parameters under raw_params; dL_dsh is [P,1,3] when sh_rest is
// given), sh_factors [P,3], dL_dsh_rest [P,M-1,3] and dL_dbg_image [3,H,W]; a tensor not asked for comes back empty.
namespace {
// The camera gradients of a backward (include/fdgs.h: fdgs_backward_camera): viewmatrix-, projmatrix- and campos-shaped
// float32 tensors, and the scratch of the reduction
struct CameraGrads {
    torch::Tensor view, proj, campos, scratch;
    fdgs_camera_grad_out out;
    CameraGrads(const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const torch::Tensor& cam_pos,
                const torch::Tensor& like, int P, int B) {
        auto opts = like.options().dtype(torch::kFloat32);
        TORCH_CHECK(viewmatrix.numel() == 16ll * B && projmatrix.numel() == 16ll * B && cam_pos.numel() == 3ll * B,
                    "fdgs: the camera gradient needs viewmatrix / projmatrix of 16 and campos of 3 elements per view");
        view = torch::empty(viewmatrix.sizes(), opts);
        proj = torch::empty(projmatrix.sizes(), opts);
        campos = torch::empty(cam_pos.sizes(), opts);
        scratch = torch::empty({(int64_t)fdgs_camera_grad_scratch_bytes(P, B)}, like.options().dtype(torch::kByte));
        out.dL_dviewmatrix = view.data_ptr<float>();
        out.dL_dprojmatrix = proj.data_ptr<float>();
        out.dL_dcampos = campos.data_ptr<float>();
        out.scratch = reinterpret_cast<char*>(scratch.data_ptr());
    }
};

// rasterize_gaussians_backward_ext, and with `camera` rasterize_gaussians_backward_camera
std::vector<torch::Tensor>
backward_ext(const torch::Tensor& background, const torch::Tensor& means3D,
                              const torch::Tensor& out_means3D, const torch::Tensor& radii, const torch::Tensor& colors,
                              const torch::Tensor& flows_2d, const torch::Tensor& opacities, const torch::Tensor& ts,
                              const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                              const torch::Tensor& rotations_r, const float scale_modifier,
                              const torch::Tensor& cov3D_precomp, const float prefilter_var,
                              const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
                              const float tan_fovy, const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_depth,
                              const torch::Tensor& dL_dout_mask, const torch::Tensor& dL_dout_flow, const torch::Tensor& sh,
                              const int degree, const int degree_t, const torch::Tensor& campos, const float timestamp,
                              const float time_duration, const bool rot_4d, const int gaussian_dim,
                              const bool force_sh_3d, const torch::Tensor& geomBuffer, const int R,
                              const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const bool debug,
                              const torch::Tensor& sh_rest, const bool raw_params, const torch::Tensor& bg_image,
                              const bool sh_factor_mode, const bool want_dbg, const torch::Tensor& sh_grad,
                              const torch::Tensor& sh_rest_grad, const bool camera) {
    TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor");
    const DeviceStream on(means3D);
    const int P = means3D.size(0);
    const int H = dL_dout_color.size(1), W = dL_dout_color.size(2);
    const bool split = provided(sh_rest);
    const int M = sh_coefficients(sh, sh_rest);
    auto opts = means3D.options().dtype(torch::kFloat32);

    // accumulated by the blend kernel -> one zero-filled slab, sliced into the five API tensors
    torch::Tensor slab = torch::zeros({(int64_t)P * 13}, opts);
    torch::Tensor dL_dmeans2D = slab.narrow(0, 0, (int64_t)P * 3).view({P, 3});
    torch::Tensor dL_dconic = slab.narrow(0, (int64_t)P * 3, (int64_t)P * 4).view({P, 2, 2});
    torch::Tensor dL_dcolors = slab.narrow(0, (int64_t)P * 7, (int64_t)P * 3).view({P, 3});
    torch::Tensor dL_dflows = slab.narrow(0, (int64_t)P * 10, (int64_t)P * 2).view({P, 2});
    torch::Tensor dL_dopacity = slab.narrow(0, (int64_t)P * 12, (int64_t)P).view({P, 1});
    // fully overwritten by the backward-preprocess kernel
    torch::Tensor dL_dmeans3D = torch::empty({P, 3}, opts);
    torch::Tensor dL_dts = torch::empty({P, 1}, opts);
    torch::Tensor dL_dcov3D = torch::empty({P, 6}, opts);
    const bool factors = sh_factor_mode && M > 0;
    const bool zeroed = !factors && provided(sh_grad);
    if (zeroed) {
        sh_grad_rows(sh_grad, "dL_dsh", means3D, P, split ? 1 : M);
        TORCH_CHECK(split == provided(sh_rest_grad), "fdgs: split SH rows need both zeroed gradient tensors");
        if (split) sh_grad_rows(sh_rest_grad, "dL_dsh_rest", means3D, P, M - 1);
    }
    torch::Tensor dL_dsh = factors ? torch::empty({0}, opts) : zeroed ? sh_grad : torch::empty({P, split ? 1 : M, 3}, opts);
    torch::Tensor dL_dsh_rest = (split && !factors) ? (zeroed ? sh_rest_grad : torch::empty({P, M - 1, 3}, opts))
                                                    : torch::empty({0}, opts);
    torch::Tensor sh_factors = factors ? torch::empty({P, 3}, opts) : torch::empty({0}, opts);
    torch::Tensor dL_dscales = torch::empty({P, 3}, opts);
    torch::Tensor dL_dscales_t = torch::empty({P, 1}, opts);
    torch::Tensor dL_drotations = torch::empty({P, 4}, opts);
    torch::Tensor dL_drotations_r = torch::empty({P, 4}, opts);
    // overwritten for every pixel by the blend backward
    torch::Tensor dL_dbg_image = want_dbg ? torch::empty({3, H, W}, opts) : torch::empty({0}, opts);
    const auto bgi_c = background_image(bg_image, means3D, H, W);
    std::unique_ptr<CameraGrads> cam;
    if (camera) cam.reset(new CameraGrads(viewmatrix, projmatrix, campos, means3D, P, 1));

    if (P != 0 || want_dbg || camera) {
        fdgs_backward_args a;
        memset(&a, 0, sizeof(a));
        Inputs in;
        backward_gaussians(a, in, background, means3D, flows_2d, opacities, ts, scales, scales_t, rotations, rotations_r,
                           scale_modifier, prefilter_var, sh, sh_rest, degree, degree_t, time_duration, rot_4d, gaussian_dim,
                           force_sh_3d, debug, raw_params, H, W, dL_dout_color, dL_dout_depth, dL_dout_mask, dL_dout_flow,
                           geomBuffer, R, binningBuffer, imageBuffer);
        a.out_means3D = in(out_means3D); a.colors_precomp = in(colors); a.cov3D_precomp = in(cov3D_precomp);
        a.viewmatrix = in(viewmatrix); a.projmatrix = in(projmatrix); a.campos = in(campos);
        a.timestamp = timestamp; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
        const auto rad_c = contig(radii);
        a.radii = rad_c.numel() ? rad_c.data_ptr<int>() : nullptr;
        a.dL_dmean2D = dL_dmeans2D.data_ptr<float>(); a.dL_dconic = dL_dconic.data_ptr<float>();
        a.dL_dopacity = dL_dopacity.data_ptr<float>(); a.dL_dcolor = dL_dcolors.data_ptr<float>();
        a.dL_dflows = dL_dflows.data_ptr<float>(); a.dL_dmean3D = dL_dmeans3D.data_ptr<float>();
        a.dL_dcov3D = dL_dcov3D.data_ptr<float>(); a.dL_dsh = (M > 0 && !factors) ? dL_dsh.data_ptr<float>() : nullptr;
        a.sh_factors = factors ? sh_factors.data_ptr<float>() : nullptr;
        a.dL_dsh_rest = (split && !factors) ? dL_dsh_rest.data_ptr<float>() : nullptr;
        a.dL_dts = dL_dts.data_ptr<float>(); a.dL_dscale = dL_dscales.data_ptr<float>();
        a.dL_dscale_t = dL_dscales_t.data_ptr<float>(); a.dL_drot = dL_drotations.data_ptr<float>();
        a.dL_drot_r = dL_drotations_r.data_ptr<float>();
        float* dbg = want_dbg ? dL_dbg_image.data_ptr<float>() : nullptr;
        if (cam)
            check(fdgs_backward_camera(&a, fptr(bgi_c), dbg, zeroed ? 1 : 0, &cam->out, (void*)on.stream), "backward_camera");
        else
            check(fdgs_backward_zero_sh(&a, fptr(bgi_c), dbg, zeroed ? 1 : 0, (void*)on.stream), "backward");
    }
    std::vector<torch::Tensor> out = {dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dflows,
                                      dL_dts, dL_dscales, dL_dscales_t, dL_drotations, dL_drotations_r, sh_factors,
                                      dL_dsh_rest, dL_dbg_image};
    if (cam) out.insert(out.end(), {cam->view, cam->proj, cam->campos});
    return out;
}
}  // namespace

std::vector<torch::Tensor>
RasterizeGaussiansBackwardExtZeroSh(const torch::Tensor& background, const torch::Tensor& means3D,
                              const torch::Tensor& out_means3D, const torch::Tensor& radii, const torch::Tensor& colors,
                              const torch::Tensor& flows_2d, const torch::Tensor& opacities, const torch::Tensor& ts,
                              const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                              const torch::Tensor& rotations_r, const float scale_modifier,
                              const torch::Tensor& cov3D_precomp, const float prefilter_var,
                              const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
                              const float tan_fovy, const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_depth,
                              const torch::Tensor& dL_dout_mask, const torch::Tensor& dL_dout_flow, const torch::Tensor& sh,
                              const int degree, const int degree_t, const torch::Tensor& campos, const float timestamp,
                              const float time_duration, const bool rot_4d, const int gaussian_dim,
                              const bool force_sh_3d, const torch::Tensor& geomBuffer, const int R,
                              const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const bool debug,
                              const torch::Tensor& sh_rest, const bool raw_params, const torch::Tensor& bg_image,
                              const bool sh_factor_mode, const bool want_dbg, const torch::Tensor& sh_grad,
                              const torch::Tensor& sh_rest_grad) {
    return backward_ext(background, means3D, out_means3D, radii, colors, flows_2d, opacities, ts, scales, scales_t,
                        rotations, rotations_r, scale_modifier, cov3D_precomp, prefilter_var, viewmatrix, projmatrix,
                        tan_fovx, tan_fovy, dL_dout_color, dL_dout_depth, dL_dout_mask, dL_dout_flow, sh, degree, degree_t,
                        campos, timestamp, time_duration, rot_4d, gaussian_dim, force_sh_3d, geomBuffer, R, binningBuffer,
                        imageBuffer, debug, sh_rest, raw_params, bg_image, sh_factor_mode, want_dbg, sh_grad, sh_rest_grad,
                        false);
}

// rasterize_gaussians_backward_ext's arguments (with the zeroed SH gradient tensors, empty when none); returns its 15
// tensors and then dL_dviewmatrix, dL_dprojmatrix and dL_dcampos, shaped like viewmatrix, projmatrix and campos
// (include/fdgs.h: fdgs_backward_camera)
std::vector<torch::Tensor>
RasterizeGaussiansBackwardCamera(const torch::Tensor& background, const torch::Tensor& means3D,
                              const torch::Tensor& out_means3D, const torch::Tensor& radii, const torch::Tensor& colors,
                              const torch::Tensor& flows_2d, const torch::Tensor& opacities, const torch::Tensor& ts,
                              const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                              const torch::Tensor& rotations_r, const float scale_modifier,
                              const torch::Tensor& cov3D_precomp, const float prefilter_var,
                              const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
                              const float tan_fovy, const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_depth,
                              const torch::Tensor& dL_dout_mask, const torch::Tensor& dL_dout_flow, const torch::Tensor& sh,
                              const int degree, const int degree_t, const torch::Tensor& campos, const float timestamp,
                              const float time_duration, const bool rot_4d, const int gaussian_dim,
                              const bool force_sh_3d, const torch::Tensor& geomBuffer, const int R,
                              const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const bool debug,
                              const torch::Tensor& sh_rest, const bool raw_params, const torch::Tensor& bg_image,
                              const bool sh_factor_mode, const bool want_dbg, const torch::Tensor& sh_grad,
                              const torch::Tensor& sh_rest_grad) {
    return backward_ext(background, means3D, out_means3D, radii, colors, flows_2d, opacities, ts, scales, scales_t,
                        rotations, rotations_r, scale_modifier, cov3D_precomp, prefilter_var, viewmatrix, projmatrix,
                        tan_fovx, tan_fovy, dL_dout_color, dL_dout_depth, dL_dout_mask, dL_dout_flow, sh, degree, degree_t,
                        campos, timestamp, time_duration, rot_4d, gaussian_dim, force_sh_3d, geomBuffer, R, binningBuffer,
                        imageBuffer, debug, sh_rest, raw_params, bg_image, sh_factor_mode, want_dbg, sh_grad, sh_rest_grad,
                        true);
}

std::vector<torch::Tensor>
RasterizeGaussiansBackwardExt(const torch::Tensor& background, const torch::Tensor& means3D,
                              const torch::Tensor& out_means3D, const torch::Tensor& radii, const torch::Tensor& colors,
                              const torch::Tensor& flows_2d, const torch::Tensor& opacities, const torch::Tensor& ts,
                              const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                              const torch::Tensor& rotations_r, const float scale_modifier,
                              const torch::Tensor& cov3D_precomp, const float prefilter_var,
                              const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
                              const float tan_fovy, const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_depth,
                              const torch::Tensor& dL_dout_mask, const torch::Tensor& dL_dout_flow, const torch::Tensor& sh,
                              const int degree, const int degree_t, const torch::Tensor& campos, const float timestamp,
                              const float time_duration, const bool rot_4d, const int gaussian_dim,
                              const bool force_sh_3d, const torch::Tensor& geomBuffer, const int R,
                              const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const bool debug,
                              const torch::Tensor& sh_rest, const bool raw_params, const torch::Tensor& bg_image,
                              const bool sh_factor_mode, const bool want_dbg) {
    return RasterizeGaussiansBackwardExtZeroSh(
        background, means3D, out_means3D, radii, colors, flows_2d, opacities, ts, scales, scales_t, rotations, rotations_r,
        scale_modifier, cov3D_precomp, prefilter_var, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color,
        dL_dout_depth, dL_dout_mask, dL_dout_flow, sh, degree, degree_t, campos, timestamp, time_duration, rot_4d,
        gaussian_dim, force_sh_3d, geomBuffer, R, binningBuffer, imageBuffer, debug, sh_rest, raw_params, bg_image,
        sh_factor_mode, want_dbg, torch::Tensor(), torch::Tensor());
}

// the reference's entry point: 37 positional arguments, 12 gradients (rasterize_points.h:51-89)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
           torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansBackwardCUDA(const torch::Tensor& background, const torch::Tensor& means3D,
                               const torch::Tensor& out_means3D, const torch::Tensor& radii, const torch::Tensor& colors,
                               const torch::Tensor& flows_2d, const torch::Tensor& opacities, const torch::Tensor& ts,
                               const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                               const torch::Tensor& rotations_r, const float scale_modifier,
                               const torch::Tensor& cov3D_precomp, const float prefilter_var,
                               const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
                               const float tan_fovy, const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_depth,
                               const torch::Tensor& dL_dout_mask, const torch::Tensor& dL_dout_flow, const torch::Tensor& sh,
                               const int degree, const int degree_t, const torch::Tensor& campos, const float timestamp,
                               const float time_duration, const bool rot_4d, const int gaussian_dim,
                               const bool force_sh_3d, const torch::Tensor& geomBuffer, const int R,
                               const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const bool debug) {
    const std::vector<torch::Tensor> o = RasterizeGaussiansBackwardExt(
        background, means3D, out_means3D, radii, colors, flows_2d, opacities, ts, scales, scales_t, rotations, rotations_r,
        scale_modifier, cov3D_precomp, prefilter_var, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color,
        dL_dout_depth, dL_dout_mask, dL_dout_flow, sh, degree, degree_t, campos, timestamp, time_duration, rot_4d,
        gaussian_dim, force_sh_3d, geomBuffer, R, binningBuffer, imageBuffer, debug, torch::Tensor(), false,
        torch::Tensor(), false, false);
    return std::make_tuple(o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7], o[8], o[9], o[10], o[11]);
}

// ---- batched views (include/fdgs.h: fdgs_forward_batch / fdgs_backward_batch) ---------------------------------------
// The cameras are strict: viewmatrix / projmatrix [B,16] (or [B,4,4]) and campos [B,3] float32 CUDA tensors on the
// Gaussians' device, timestamps / tanfovx / tanfovy [B] float32 CPU tensors (CUDA tensors on that device for the capacity
// entry: device_scalars); bg_image empty or [B,3,H,W].  Checked before anything is allocated or launched.
namespace {
struct BatchCams {
    int B;
    const float *view, *proj, *campos, *timestamps, *tanfovx, *tanfovy;
};

BatchCams batch_cameras(const torch::Tensor& means3D, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
                        const torch::Tensor& campos, const torch::Tensor& timestamps, const torch::Tensor& tanfovx,
                        const torch::Tensor& tanfovy, bool device_scalars = false) {
    TORCH_CHECK(viewmatrix.defined() && viewmatrix.dim() >= 1, "fdgs: viewmatrix must be [B,16]");
    BatchCams c;
    const int64_t B = viewmatrix.size(0);
    TORCH_CHECK(B >= 1 && B <= 65535, "fdgs: the view count B must be in [1, 65535]");
    c.B = (int)B;
    c.view = arg<float>(viewmatrix, "viewmatrix", B, 16 * B, REQUIRED);
    c.proj = arg<float>(projmatrix, "projmatrix", B, 16 * B, REQUIRED);
    c.campos = arg<float>(campos, "campos", B, 3 * B, REQUIRED);
    c.timestamps = arg<float>(timestamps, "timestamps", B, B, REQUIRED);
    c.tanfovx = arg<float>(tanfovx, "tanfovx", B, B, REQUIRED);
    c.tanfovy = arg<float>(tanfovy, "tanfovy", B, B, REQUIRED);
    if (device_scalars) {
        TORCH_CHECK(timestamps.is_cuda() && tanfovx.is_cuda() && tanfovy.is_cuda(),
                    "fdgs: timestamps / tanfovx / tanfovy must be CUDA tensors");
    } else {
        TORCH_CHECK(!timestamps.is_cuda() && !tanfovx.is_cuda() && !tanfovy.is_cuda(),
                    "fdgs: timestamps / tanfovx / tanfovy must be CPU tensors");
    }
    TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor");
    if (device_scalars)
        same_cuda_device("batched camera", {means3D, viewmatrix, projmatrix, campos, timestamps, tanfovx, tanfovy});
    else
        same_cuda_device("batched camera", {means3D, viewmatrix, projmatrix, campos});
    return c;
}

const float* batch_bg_image(const torch::Tensor& bg_image, const torch::Tensor& means3D, int B, int H, int W) {
    if (!bg_image.defined() || bg_image.numel() == 0) return nullptr;
    TORCH_CHECK(bg_image.dim() == 4 && bg_image.size(0) == B && bg_image.size(1) == 3 && bg_image.size(2) == H &&
                    bg_image.size(3) == W,
                "fdgs: bg_image must be [B, 3, image_height, image_width]");
    const float* p = arg<float>(bg_image, "bg_image");
    same_cuda_device("bg_image", {means3D, bg_image});
    return p;
}
}  // namespace

// B views of the same Gaussians: (num_rendered, color [B,3,H,W], flow [B,2,H,W], depth [B,1,H,W], T [B,1,H,W],
// radii [B,P], geomBuffer, binningBuffer, imgBuffer, out_means3D [B,P,3]).  Gaussian inputs as in rasterize_gaussians_ext
// (SH and scales / rotations only: no precomputed colours or covariances).
namespace {
using BatchForwardOut = std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
                                   torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>;

// capacity < 0: fdgs_forward_batch; else fdgs_forward_batch_capacity, which writes `status` (int32 [4] on the device)
BatchForwardOut batch_forward(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& flows,
                              const torch::Tensor& opacity, const torch::Tensor& ts, const torch::Tensor& scales,
                              const torch::Tensor& scales_t, const torch::Tensor& rotations, const torch::Tensor& rotations_r,
                              const float scale_modifier, const float prefilter_var, const torch::Tensor& viewmatrix,
                              const torch::Tensor& projmatrix, const torch::Tensor& campos, const torch::Tensor& timestamps,
                              const torch::Tensor& tanfovx, const torch::Tensor& tanfovy, const int image_height,
                              const int image_width, const torch::Tensor& sh, const torch::Tensor& sh_rest, const int degree,
                              const int degree_t, const float time_duration, const bool rot_4d, const int gaussian_dim,
                              const bool force_sh_3d, const bool prefiltered, const bool debug, const bool raw_params,
                              const torch::Tensor& bg_image, int64_t capacity, torch::Tensor* status) {
    TORCH_CHECK(means3D.dim() == 2 && means3D.size(1) == 3, "means3D must have dimensions (num_points, 3)");
    const bool cap = capacity >= 0;
    const BatchCams cams = batch_cameras(means3D, viewmatrix, projmatrix, campos, timestamps, tanfovx, tanfovy, cap);
    const int B = cams.B, P = means3D.size(0), H = image_height, W = image_width;
    TORCH_CHECK(H > 0 && W > 0, "fdgs: bad image size");
    const float* bgi = batch_bg_image(bg_image, means3D, B, H, W);
    const DeviceStream on(means3D);
    auto fopts = means3D.options().dtype(torch::kFloat32);
    auto bopts = means3D.options().dtype(torch::kByte);
    torch::Tensor out_color = torch::empty({B, 3, H, W}, fopts);
    torch::Tensor out_flow = torch::empty({B, 2, H, W}, fopts);
    torch::Tensor out_depth = torch::empty({B, 1, H, W}, fopts);
    torch::Tensor out_T = torch::empty({B, 1, H, W}, fopts);
    torch::Tensor radii = torch::empty({B, P}, means3D.options().dtype(torch::kInt32));
    torch::Tensor out_means3D = torch::empty({B, P, 3}, fopts);
    torch::Tensor geomBuffer = torch::empty({0}, bopts), binningBuffer = torch::empty({0}, bopts),
                  imgBuffer = torch::empty({0}, bopts);
    fdgs_forward_batch_args b;
    memset(&b, 0, sizeof(b));
    fdgs_forward_args& a = b.view;
    Inputs in;
    forward_gaussians(a, in, background, means3D, flows, opacity, ts, scales, scales_t, rotations, rotations_r, scale_modifier,
                      prefilter_var, sh, sh_rest, degree, degree_t, time_duration, rot_4d, gaussian_dim, force_sh_3d,
                      prefiltered, debug, raw_params, H, W);
    a.viewmatrix = cams.view; a.projmatrix = cams.proj; a.cam_pos = cams.campos;
    a.out_means3D = out_means3D.data_ptr<float>(); a.out_color = out_color.data_ptr<float>();
    a.out_flow = out_flow.data_ptr<float>(); a.out_depth = out_depth.data_ptr<float>();
    a.out_T = out_T.data_ptr<float>(); a.radii = radii.data_ptr<int>();
    b.B = B; b.bg_image = bgi; b.bg_views = bgi ? B : 0;
    fdgs_forward_result r;
    if (cap) {
        *status = torch::empty({4}, means3D.options().dtype(torch::kInt32));
        fdgs_forward_capacity_args c;
        memset(&c, 0, sizeof(c));
        c.batch = b;
        c.timestamps = cams.timestamps; c.tan_fovx = cams.tanfovx; c.tan_fovy = cams.tanfovy;
        c.capacity = (int)capacity; c.status = status->data_ptr<int>();
        check(fdgs_forward_batch_capacity(&c, resize_cb, &geomBuffer, resize_cb, &binningBuffer, resize_cb, &imgBuffer,
                                          (void*)on.stream, &r),
              "forward_batch_capacity");
    } else {
        b.timestamps = cams.timestamps; b.tan_fovx = cams.tanfovx; b.tan_fovy = cams.tanfovy;
        check(fdgs_forward_batch(&b, resize_cb, &geomBuffer, resize_cb, &binningBuffer, resize_cb, &imgBuffer, (void*)on.stream,
                                 &r),
              "forward_batch");
    }
    return std::make_tuple(r.num_rendered, out_color, out_flow, out_depth, out_T, radii, geomBuffer, binningBuffer, imgBuffer,
                           out_means3D);
}
}  // namespace

BatchForwardOut RasterizeGaussiansBatch(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& flows,
                                        const torch::Tensor& opacity, const torch::Tensor& ts, const torch::Tensor& scales,
                                        const torch::Tensor& scales_t, const torch::Tensor& rotations,
                                        const torch::Tensor& rotations_r, const float scale_modifier, const float prefilter_var,
                                        const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
                                        const torch::Tensor& campos, const torch::Tensor& timestamps,
                                        const torch::Tensor& tanfovx, const torch::Tensor& tanfovy, const int image_height,
                                        const int image_width, const torch::Tensor& sh, const torch::Tensor& sh_rest,
                                        const int degree, const int degree_t, const float time_duration, const bool rot_4d,
                                        const int gaussian_dim, const bool force_sh_3d, const bool prefiltered, const bool debug,
                                        const bool raw_params, const torch::Tensor& bg_image) {
    return batch_forward(background, means3D, flows, opacity, ts, scales, scales_t, rotations, rotations_r, scale_modifier,
                         prefilter_var, viewmatrix, projmatrix, campos, timestamps, tanfovx, tanfovy, image_height, image_width,
                         sh, sh_rest, degree, degree_t, time_duration, rot_4d, gaussian_dim, force_sh_3d, prefiltered, debug,
                         raw_params, bg_image, -1, nullptr);
}

// rasterize_gaussians_batch sized by `capacity` instances (include/fdgs.h: fdgs_forward_batch_capacity): the same
// arguments, except that timestamps / tanfovx / tanfovy are float32 CUDA tensors [B] on the Gaussians' device, and the
// same tuple with status (int32 [4] on the device: R, largest tile, overflow, wrap) in place of num_rendered.  The
// backward is rasterize_gaussians_backward_batch with R = capacity.  No host synchronisation.
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
           torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansBatchCapacity(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& flows,
                                const torch::Tensor& opacity, const torch::Tensor& ts, const torch::Tensor& scales,
                                const torch::Tensor& scales_t, const torch::Tensor& rotations, const torch::Tensor& rotations_r,
                                const float scale_modifier, const float prefilter_var, const torch::Tensor& viewmatrix,
                                const torch::Tensor& projmatrix, const torch::Tensor& campos, const torch::Tensor& timestamps,
                                const torch::Tensor& tanfovx, const torch::Tensor& tanfovy, const int image_height,
                                const int image_width, const torch::Tensor& sh, const torch::Tensor& sh_rest, const int degree,
                                const int degree_t, const float time_duration, const bool rot_4d, const int gaussian_dim,
                                const bool force_sh_3d, const bool prefiltered, const bool debug, const bool raw_params,
                                const torch::Tensor& bg_image, const int64_t capacity) {
    TORCH_CHECK(capacity >= 0 && capacity <= 0x7fffffffLL, "fdgs: capacity must be in [0, 2^31 - 1]");
    torch::Tensor status;
    const BatchForwardOut o = batch_forward(background, means3D, flows, opacity, ts, scales, scales_t, rotations, rotations_r,
                                            scale_modifier, prefilter_var, viewmatrix, projmatrix, campos, timestamps, tanfovx,
                                            tanfovy, image_height, image_width, sh, sh_rest, degree, degree_t, time_duration,
                                            rot_4d, gaussian_dim, force_sh_3d, prefiltered, debug, raw_params, bg_image,
                                            capacity, &status);
    return std::make_tuple(status, std::get<1>(o), std::get<2>(o), std::get<3>(o), std::get<4>(o), std::get<5>(o),
                           std::get<6>(o), std::get<7>(o), std::get<8>(o), std::get<9>(o));
}

// Backward of rasterize_gaussians_batch.  Returns 11 tensors: dL_dmeans2D [B,P,3] per view, then the view sums
// dL_dopacity [P,1], dL_dmeans3D [P,3], dL_dsh ([P,M,3], or [P,1,3] with sh_rest), dL_dsh_rest, dL_dts [P,1],
// dL_dscales [P,3], dL_dscales_t [P,1], dL_drotations [P,4], dL_drotations_r [P,4], and dL_dbg_image [B,3,H,W] (empty
// unless want_dbg).
namespace {
// rasterize_gaussians_backward_batch, and with `camera` rasterize_gaussians_backward_batch_camera
std::vector<torch::Tensor>
backward_batch(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& out_means3D,
                                const torch::Tensor& radii, const torch::Tensor& flows, const torch::Tensor& opacities,
                                const torch::Tensor& ts, const torch::Tensor& scales, const torch::Tensor& scales_t,
                                const torch::Tensor& rotations, const torch::Tensor& rotations_r, const float scale_modifier,
                                const float prefilter_var, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
                                const torch::Tensor& campos, const torch::Tensor& timestamps, const torch::Tensor& tanfovx,
                                const torch::Tensor& tanfovy, const torch::Tensor& dL_dout_color,
                                const torch::Tensor& dL_dout_depth, const torch::Tensor& dL_dout_mask,
                                const torch::Tensor& dL_dout_flow, const torch::Tensor& sh, const torch::Tensor& sh_rest,
                                const int degree, const int degree_t, const float time_duration, const bool rot_4d,
                                const int gaussian_dim, const bool force_sh_3d, const torch::Tensor& geomBuffer, const int R,
                                const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const bool debug,
                                const bool raw_params, const torch::Tensor& bg_image, const bool want_dbg, const bool camera) {
    TORCH_CHECK(means3D.dim() == 2 && means3D.size(1) == 3, "means3D must have dimensions (num_points, 3)");
    const BatchCams cams = batch_cameras(means3D, viewmatrix, projmatrix, campos, timestamps, tanfovx, tanfovy);
    const int B = cams.B, P = means3D.size(0);
    TORCH_CHECK(dL_dout_color.dim() == 4 && dL_dout_color.size(0) == B && dL_dout_color.size(1) == 3,
                "fdgs: the colour gradient must be [B,3,H,W]");
    const int H = dL_dout_color.size(2), W = dL_dout_color.size(3);
    const float* bgi = batch_bg_image(bg_image, means3D, B, H, W);
    const float* om = arg<float>(out_means3D, "out_means3D", B, 3ll * B * P, REQUIRED);
    const int* rad = arg<int>(radii, "radii", B, (int64_t)B * P, REQUIRED);
    TORCH_CHECK(!provided(dL_dout_depth) || dL_dout_depth.numel() == (int64_t)B * H * W,
                "fdgs: the depth gradient must be [B,1,H,W]");
    TORCH_CHECK(!provided(dL_dout_mask) || dL_dout_mask.numel() == (int64_t)B * H * W,
                "fdgs: the alpha gradient must be [B,1,H,W]");
    TORCH_CHECK(!provided(dL_dout_flow) || dL_dout_flow.numel() == 2ll * B * H * W, "fdgs: the flow gradient must be [B,2,H,W]");
    const DeviceStream on(means3D);
    const bool split = provided(sh_rest);
    const int M = sh_coefficients(sh, sh_rest);
    auto opts = means3D.options().dtype(torch::kFloat32);
    torch::Tensor dL_dmeans2D = torch::zeros({B, P, 3}, opts);
    torch::Tensor dL_dopacity = torch::empty({P, 1}, opts), dL_dmeans3D = torch::empty({P, 3}, opts);
    torch::Tensor dL_dsh = torch::empty({P, split ? 1 : M, 3}, opts);
    torch::Tensor dL_dsh_rest = split ? torch::empty({P, M - 1, 3}, opts) : torch::empty({0}, opts);
    torch::Tensor dL_dts = torch::empty({P, 1}, opts), dL_dscales = torch::empty({P, 3}, opts),
                  dL_dscales_t = torch::empty({P, 1}, opts), dL_drot = torch::empty({P, 4}, opts),
                  dL_drot_r = torch::empty({P, 4}, opts);
    torch::Tensor dL_dbg_image = want_dbg ? torch::empty({B, 3, H, W}, opts) : torch::empty({0}, opts);
    torch::Tensor scratch = torch::empty({(int64_t)fdgs_backward_batch_scratch_bytes(P, B)}, means3D.options().dtype(torch::kByte));
    fdgs_backward_batch_args b;
    memset(&b, 0, sizeof(b));
    fdgs_backward_args& a = b.view;
    Inputs in;
    backward_gaussians(a, in, background, means3D, flows, opacities, ts, scales, scales_t, rotations, rotations_r,
                       scale_modifier, prefilter_var, sh, sh_rest, degree, degree_t, time_duration, rot_4d, gaussian_dim,
                       force_sh_3d, debug, raw_params, H, W, dL_dout_color, dL_dout_depth, dL_dout_mask, dL_dout_flow,
                       geomBuffer, R, binningBuffer, imageBuffer);
    a.out_means3D = om; a.radii = rad;
    a.viewmatrix = cams.view; a.projmatrix = cams.proj; a.campos = cams.campos;
    a.dL_dmean2D = dL_dmeans2D.data_ptr<float>(); a.dL_dopacity = dL_dopacity.data_ptr<float>();
    a.dL_dmean3D = dL_dmeans3D.data_ptr<float>(); a.dL_dsh = dL_dsh.data_ptr<float>();
    a.dL_dsh_rest = split ? dL_dsh_rest.data_ptr<float>() : nullptr;
    a.dL_dts = dL_dts.data_ptr<float>(); a.dL_dscale = dL_dscales.data_ptr<float>();
    a.dL_dscale_t = dL_dscales_t.data_ptr<float>(); a.dL_drot = dL_drot.data_ptr<float>(); a.dL_drot_r = dL_drot_r.data_ptr<float>();
    b.B = B; b.bg_image = bgi; b.bg_views = bgi ? B : 0;
    b.dL_dbg_image = want_dbg ? dL_dbg_image.data_ptr<float>() : nullptr;
    b.scratch = reinterpret_cast<char*>(scratch.data_ptr());
    if (!camera) {
        check(fdgs_backward_batch(&b, (void*)on.stream), "backward_batch");
        return {dL_dmeans2D, dL_dopacity, dL_dmeans3D, dL_dsh, dL_dsh_rest, dL_dts, dL_dscales, dL_dscales_t, dL_drot,
                dL_drot_r, dL_dbg_image};
    }
    CameraGrads cam(viewmatrix, projmatrix, campos, means3D, P, B);
    check(fdgs_backward_batch_camera(&b, &cam.out, (void*)on.stream), "backward_batch_camera");
    return {dL_dmeans2D, dL_dopacity, dL_dmeans3D, dL_dsh, dL_dsh_rest, dL_dts, dL_dscales, dL_dscales_t, dL_drot,
            dL_drot_r, dL_dbg_image, cam.view, cam.proj, cam.campos};
}
}  // namespace

std::vector<torch::Tensor>
RasterizeGaussiansBackwardBatch(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& out_means3D,
                                const torch::Tensor& radii, const torch::Tensor& flows, const torch::Tensor& opacities,
                                const torch::Tensor& ts, const torch::Tensor& scales, const torch::Tensor& scales_t,
                                const torch::Tensor& rotations, const torch::Tensor& rotations_r, const float scale_modifier,
                                const float prefilter_var, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
                                const torch::Tensor& campos, const torch::Tensor& timestamps, const torch::Tensor& tanfovx,
                                const torch::Tensor& tanfovy, const torch::Tensor& dL_dout_color,
                                const torch::Tensor& dL_dout_depth, const torch::Tensor& dL_dout_mask,
                                const torch::Tensor& dL_dout_flow, const torch::Tensor& sh, const torch::Tensor& sh_rest,
                                const int degree, const int degree_t, const float time_duration, const bool rot_4d,
                                const int gaussian_dim, const bool force_sh_3d, const torch::Tensor& geomBuffer, const int R,
                                const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const bool debug,
                                const bool raw_params, const torch::Tensor& bg_image, const bool want_dbg) {
    return backward_batch(background, means3D, out_means3D, radii, flows, opacities, ts, scales, scales_t, rotations,
                          rotations_r, scale_modifier, prefilter_var, viewmatrix, projmatrix, campos, timestamps, tanfovx,
                          tanfovy, dL_dout_color, dL_dout_depth, dL_dout_mask, dL_dout_flow, sh, sh_rest, degree, degree_t,
                          time_duration, rot_4d, gaussian_dim, force_sh_3d, geomBuffer, R, binningBuffer, imageBuffer, debug,
                          raw_params, bg_image, want_dbg, false);
}

// rasterize_gaussians_backward_batch's arguments; returns its 11 tensors and then each view's dL_dviewmatrix,
// dL_dprojmatrix and dL_dcampos, shaped like viewmatrix [B,4,4] | [B,16], projmatrix and campos [B,3]
// (include/fdgs.h: fdgs_backward_batch_camera)
std::vector<torch::Tensor>
RasterizeGaussiansBackwardBatchCamera(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& out_means3D,
                                const torch::Tensor& radii, const torch::Tensor& flows, const torch::Tensor& opacities,
                                const torch::Tensor& ts, const torch::Tensor& scales, const torch::Tensor& scales_t,
                                const torch::Tensor& rotations, const torch::Tensor& rotations_r, const float scale_modifier,
                                const float prefilter_var, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
                                const torch::Tensor& campos, const torch::Tensor& timestamps, const torch::Tensor& tanfovx,
                                const torch::Tensor& tanfovy, const torch::Tensor& dL_dout_color,
                                const torch::Tensor& dL_dout_depth, const torch::Tensor& dL_dout_mask,
                                const torch::Tensor& dL_dout_flow, const torch::Tensor& sh, const torch::Tensor& sh_rest,
                                const int degree, const int degree_t, const float time_duration, const bool rot_4d,
                                const int gaussian_dim, const bool force_sh_3d, const torch::Tensor& geomBuffer, const int R,
                                const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const bool debug,
                                const bool raw_params, const torch::Tensor& bg_image, const bool want_dbg) {
    return backward_batch(background, means3D, out_means3D, radii, flows, opacities, ts, scales, scales_t, rotations,
                          rotations_r, scale_modifier, prefilter_var, viewmatrix, projmatrix, campos, timestamps, tanfovx,
                          tanfovy, dL_dout_color, dL_dout_depth, dL_dout_mask, dL_dout_flow, sh, sh_rest, degree, degree_t,
                          time_duration, rot_4d, gaussian_dim, force_sh_3d, geomBuffer, R, binningBuffer, imageBuffer, debug,
                          raw_params, bg_image, want_dbg, true);
}

// Test hook: view `view` of a batch's tile ranges [tiles,2] and n_contrib [H,W]
std::tuple<torch::Tensor, torch::Tensor> DebugExportBinningView(const torch::Tensor& imgBuffer, const int W, const int H,
                                                                const int B, const int view) {
    const DeviceStream on(imgBuffer);
    auto i32 = imgBuffer.options().dtype(torch::kInt32);
    const int tiles = ((W + 15) / 16) * ((H + 15) / 16);
    torch::Tensor ranges = torch::zeros({tiles, 2}, i32), n_contrib = torch::zeros({H, W}, i32);
    check(fdgs_debug_export_binning_view(reinterpret_cast<const char*>(imgBuffer.data_ptr()), W, H, B, view,
                                         reinterpret_cast<unsigned int*>(ranges.data_ptr<int>()),
                                         reinterpret_cast<unsigned int*>(n_contrib.data_ptr<int>()), (void*)on.stream),
          "debug_export_binning_view");
    return std::make_tuple(ranges, n_contrib);
}

// ---- environment-map sky (include/fdgs.h: fdgs_sky_forward / fdgs_sky_backward) -----------------------------------
static fdgs_sky_args sky_args(const torch::Tensor& env_map, const torch::Tensor& c2w, const torch::Tensor& campos,
                              const double fl_x, const double fl_y, const double cx, const double cy, const double radius,
                              const int64_t H, const int64_t W) {
    fdgs_sky_args a;
    memset(&a, 0, sizeof(a));
    a.env_map = arg<float>(env_map, "env_map", 3, -1, REQUIRED);
    TORCH_CHECK(env_map.dim() == 3, "fdgs: env_map must be [3,Hm,Wm]");
    a.c2w = arg<float>(c2w, "c2w", -1, 16, REQUIRED);
    a.campos = arg<float>(campos, "campos", -1, 3, REQUIRED);
    same_cuda_device("sky", {env_map, c2w, campos});
    a.env_height = (int)env_map.size(1); a.env_width = (int)env_map.size(2);
    a.fl_x = (float)fl_x; a.fl_y = (float)fl_y; a.cx = (float)cx; a.cy = (float)cy; a.radius = (float)radius;
    a.width = (int)W; a.height = (int)H;
    return a;
}

// (sky [3,H,W], miss flag int32 [1]: 1 if a ray missed the sphere)
std::tuple<torch::Tensor, torch::Tensor> SkyForward(const torch::Tensor& env_map, const torch::Tensor& c2w, const torch::Tensor& campos,
                                                    const double fl_x, const double fl_y, const double cx, const double cy,
                                                    const double radius, const int64_t H, const int64_t W) {
    const fdgs_sky_args a = sky_args(env_map, c2w, campos, fl_x, fl_y, cx, cy, radius, H, W);
    const DeviceStream on(env_map);
    torch::Tensor sky = torch::empty({3, H, W}, env_map.options());
    torch::Tensor miss = torch::zeros({1}, env_map.options().dtype(torch::kInt32));
    check(fdgs_sky_forward(&a, sky.data_ptr<float>(), miss.data_ptr<int>(), (void*)on.stream), "sky_forward");
    return std::make_tuple(sky, miss);
}

// dL/d env_map [3,Hm,Wm] of dL_dsky [3,H,W]
torch::Tensor SkyBackward(const torch::Tensor& env_map, const torch::Tensor& c2w, const torch::Tensor& campos, const double fl_x,
                          const double fl_y, const double cx, const double cy, const double radius,
                          const torch::Tensor& dL_dsky) {
    TORCH_CHECK(dL_dsky.is_cuda() && dL_dsky.scalar_type() == torch::kFloat32 && dL_dsky.dim() == 3 && dL_dsky.size(0) == 3,
                "fdgs: dL_dsky must be a float32 CUDA tensor [3,H,W]");
    const fdgs_sky_args a = sky_args(env_map, c2w, campos, fl_x, fl_y, cx, cy, radius, dL_dsky.size(1), dL_dsky.size(2));
    const DeviceStream on(env_map);
    const auto g = dL_dsky.contiguous();
    torch::Tensor denv = torch::zeros_like(env_map);
    check(fdgs_sky_backward(&a, g.data_ptr<float>(), denv.data_ptr<float>(), (void*)on.stream), "sky_backward");
    return denv;
}

// ---- the sky of B views, cameras from device tables (include/fdgs.h: fdgs_sky_forward_batch / _backward_batch) -------
static fdgs_sky_batch_args sky_batch_args(const torch::Tensor& env_map, const torch::Tensor& c2w, const torch::Tensor& campos,
                                          const torch::Tensor& intrinsics, const double radius, const int64_t H,
                                          const int64_t W) {
    fdgs_sky_batch_args a;
    memset(&a, 0, sizeof(a));
    a.env_map = arg<float>(env_map, "env_map", 3, -1, REQUIRED);
    TORCH_CHECK(env_map.dim() == 3, "fdgs: env_map must be [3,Hm,Wm]");
    TORCH_CHECK(c2w.dim() == 3 && c2w.size(1) == 4 && c2w.size(2) == 4, "fdgs: c2w must be [B,4,4]");
    const int64_t B = c2w.size(0);
    a.c2w = arg<float>(c2w, "c2w", B, 16 * B, REQUIRED);
    a.campos = arg<float>(campos, "campos", B, 3 * B, REQUIRED);
    a.intrinsics = arg<float>(intrinsics, "intrinsics", B, 4 * B, REQUIRED);
    same_cuda_device("sky", {env_map, c2w, campos, intrinsics});
    a.env_height = (int)env_map.size(1); a.env_width = (int)env_map.size(2);
    a.radius = (float)radius;
    a.width = (int)W; a.height = (int)H; a.B = (int)B;
    return a;
}

// (sky [B,3,H,W], miss flag int32 [1]: 1 if a ray of any view missed the sphere)
std::tuple<torch::Tensor, torch::Tensor> SkyForwardBatch(const torch::Tensor& env_map, const torch::Tensor& c2w,
                                                         const torch::Tensor& campos, const torch::Tensor& intrinsics,
                                                         const double radius, const int64_t H, const int64_t W) {
    const fdgs_sky_batch_args a = sky_batch_args(env_map, c2w, campos, intrinsics, radius, H, W);
    const DeviceStream on(env_map);
    torch::Tensor sky = torch::empty({(int64_t)a.B, 3, H, W}, env_map.options());
    torch::Tensor miss = torch::zeros({1}, env_map.options().dtype(torch::kInt32));
    check(fdgs_sky_forward_batch(&a, sky.data_ptr<float>(), miss.data_ptr<int>(), (void*)on.stream), "sky_forward_batch");
    return std::make_tuple(sky, miss);
}

// dL/d env_map [3,Hm,Wm] of dL_dsky [B,3,H,W], summed over the views
torch::Tensor SkyBackwardBatch(const torch::Tensor& env_map, const torch::Tensor& c2w, const torch::Tensor& campos,
                               const torch::Tensor& intrinsics, const double radius, const torch::Tensor& dL_dsky) {
    TORCH_CHECK(dL_dsky.is_cuda() && dL_dsky.scalar_type() == torch::kFloat32 && dL_dsky.dim() == 4 && dL_dsky.size(1) == 3 &&
                    dL_dsky.size(0) == c2w.size(0),
                "fdgs: dL_dsky must be a float32 CUDA tensor [B,3,H,W]");
    const fdgs_sky_batch_args a = sky_batch_args(env_map, c2w, campos, intrinsics, radius, dL_dsky.size(2), dL_dsky.size(3));
    const DeviceStream on(env_map);
    const auto g = dL_dsky.contiguous();
    torch::Tensor denv = torch::zeros_like(env_map);
    check(fdgs_sky_backward_batch(&a, g.data_ptr<float>(), denv.data_ptr<float>(), (void*)on.stream), "sky_backward_batch");
    return denv;
}

// rebuild + sum the dL_dsh rows of all views from the gathered colour factors (include/fdgs.h: fdgs_sh_outer_sum)
void ShOuterSum(const torch::Tensor& table, const int64_t view_stride, const int64_t meta_off, const int64_t V,
                const int64_t K, const torch::Tensor& slot_of, const torch::Tensor& union_idx, const torch::Tensor& means3D,
                const torch::Tensor& ts,
                const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                const torch::Tensor& rotations_r, const double scale_modifier, const double time_duration,
                const bool rot_4d, const int64_t gaussian_dim, const bool force_sh_3d, const int64_t D, const int64_t D_t,
                std::vector<torch::Tensor> outs, const bool accumulate) {
    TORCH_CHECK(outs.size() == 1 || outs.size() == 2, "fdgs: one or two output tensors");
    const int P = means3D.size(0);
    fdgs_sh_sum_args a;
    memset(&a, 0, sizeof(a));
    a.slot_of = arg<int>(slot_of, "slot_of", -1, -1, REQUIRED);
    for (auto& o : outs) {
        arg<float>(o, "outputs", P, -1, REQUIRED);
        TORCH_CHECK(o.dim() == 3 && o.size(2) == 3, "fdgs: outputs must be [P, m, 3]");
    }
    a.union_idx = reinterpret_cast<const long long*>(arg<int64_t>(union_idx, "union_idx", -1, K, REQUIRED));
    std::vector<torch::Tensor> dev(outs);
    dev.push_back(slot_of);
    dev.push_back(union_idx);
    same_cuda_device("sh_outer_sum", dev);
    const DeviceStream on(means3D);
    const auto m_c = contig(means3D), ts_c = contig(ts), sc_c = contig(scales), sct_c = contig(scales_t),
               rot_c = contig(rotations), rotr_c = contig(rotations_r), tb_c = contig(table);
    a.P = P; a.V = (int)V; a.K = (int)K; a.table = fptr(tb_c); a.view_stride = view_stride; a.meta_off = meta_off;
    torch::Tensor dirs = torch::empty({std::max<int64_t>(V * K * 8, 1)}, means3D.options().dtype(torch::kFloat32));
    a.dir_scratch = dirs.data_ptr<float>();
    a.means3D = fptr(m_c); a.ts = fptr(ts_c); a.scales = fptr(sc_c);
    a.scales_t = fptr(sct_c); a.rotations = fptr(rot_c); a.rotations_r = fptr(rotr_c);
    a.scale_modifier = (float)scale_modifier; a.time_duration = (float)time_duration; a.rot_4d = rot_4d;
    a.gaussian_dim = (int)gaussian_dim; a.force_sh_3d = force_sh_3d; a.D = (int)D; a.D_t = (int)D_t;
    a.m0 = (int)outs[0].size(1);
    a.M = a.m0 + (outs.size() == 2 ? (int)outs[1].size(1) : 0);
    a.out0 = outs[0].data_ptr<float>();
    a.out1 = outs.size() == 2 ? outs[1].data_ptr<float>() : nullptr;
    a.accumulate = accumulate;
    if (V > 0) TORCH_CHECK(tb_c.numel() >= V * view_stride, "fdgs: factor table too small");
    check(fdgs_sh_outer_sum(&a, (void*)on.stream), "sh_outer_sum");
}

// (slot_of int32 [P], idx int64 [K]) from the radii, their inclusive prefix sum cs and K = cs[-1] (known to the host)
std::tuple<torch::Tensor, torch::Tensor> UnionMaps(const torch::Tensor& radii, const torch::Tensor& cs, const int64_t K) {
    const int* r = arg<int>(radii, "radii", -1, -1, REQUIRED);
    const int* c = arg<int>(cs, "cs", -1, radii.numel(), REQUIRED);
    same_cuda_device("union_maps", {radii, cs});
    const DeviceStream on(radii);
    torch::Tensor slot_of = torch::empty_like(radii);
    torch::Tensor idx = torch::empty({K}, radii.options().dtype(torch::kInt64));
    check(fdgs_union_maps(radii.numel(), r, c, slot_of.data_ptr<int>(), reinterpret_cast<long long*>(idx.data_ptr<int64_t>()),
                          (void*)on.stream),
          "union_maps");
    return std::make_tuple(slot_of, idx);
}

// per-view densification statistics, one pass (include/fdgs.h: fdgs_view_stats)
void ViewStats(const torch::Tensor& viewspace_grad, const torch::Tensor& radii, torch::Tensor& grad_norm_sum,
               torch::Tensor& visibility_count, torch::Tensor& max_radii) {
    const long long P = radii.numel();
    const float* vg = arg<float>(viewspace_grad, "viewspace_grad", P, -1, REQUIRED);
    TORCH_CHECK(viewspace_grad.dim() == 2 && viewspace_grad.size(1) >= 2, "fdgs: viewspace_grad must be [P, >= 2]");
    const int* r = arg<int>(radii, "radii", -1, -1, REQUIRED);
    float* gn = arg<float>(grad_norm_sum, "grad_norm_sum", -1, P, REQUIRED);
    float* vc = arg<float>(visibility_count, "visibility_count", -1, P, REQUIRED);
    int* mr = arg<int>(max_radii, "max_radii", -1, P, REQUIRED);
    same_cuda_device("view_stats", {viewspace_grad, radii});
    const DeviceStream on(radii);
    check(fdgs_view_stats(P, vg, (int)viewspace_grad.size(1), r, gn, vc, mr, (void*)on.stream), "view_stats");
}

// 1-element int32 tensor, non-zero if a row of `tensors` outside radii > 0 is not all-zero (sparse-exchange guard)
torch::Tensor CheckRowsZero(std::vector<torch::Tensor> tensors, const torch::Tensor& radii) {
    TORCH_CHECK((int)tensors.size() <= FDGS_MAX_PACK, "fdgs: too many tensors");
    const int* r = arg<int>(radii, "radii", -1, -1, REQUIRED);
    same_cuda_device("check_rows_zero", {radii});
    torch::Tensor flag = torch::zeros({1}, radii.options());
    const long long P = radii.numel();
    if (tensors.empty() || P == 0) return flag;
    std::vector<const float*> ptr;
    std::vector<int> widths;
    for (const auto& t : tensors) {
        ptr.push_back(arg<float>(t, "gradient tensor", P, -1, REQUIRED));
        widths.push_back((int)(t.numel() / P));
    }
    same_cuda_device("check_rows_zero", tensors);
    const DeviceStream on(radii);
    check(fdgs_check_rows_zero((int)ptr.size(), ptr.data(), widths.data(), P, r, flag.data_ptr<int>(), (void*)on.stream),
          "check_rows_zero");
    return flag;
}

torch::Tensor markVisible(torch::Tensor& means3D, torch::Tensor& viewmatrix, torch::Tensor& projmatrix) {
    const int P = means3D.size(0);
    torch::Tensor present = torch::full({P}, false, means3D.options().dtype(at::kBool));
    if (P != 0) {
        const DeviceStream on(means3D);
        const auto m = means3D.contiguous(), v = viewmatrix.contiguous(), pr = projmatrix.contiguous();
        check(fdgs_mark_visible(P, m.data_ptr<float>(), v.data_ptr<float>(), pr.data_ptr<float>(),
                                reinterpret_cast<unsigned char*>(present.data_ptr<bool>()), (void*)on.stream),
              "mark_visible");
    }
    return present;
}

// Test hooks: private forward state as plain tensors (parity tests compare them with the oracle).
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
DebugExportGeom(const torch::Tensor& geomBuffer, const int P) {
    const DeviceStream on(geomBuffer);
    auto f = geomBuffer.options().dtype(torch::kFloat32);
    torch::Tensor depths = torch::zeros({P}, f), means2D = torch::zeros({P, 2}, f), conic = torch::zeros({P, 4}, f),
                  rgb = torch::zeros({P, 3}, f);
    torch::Tensor clamped = torch::zeros({P}, geomBuffer.options().dtype(torch::kByte));
    torch::Tensor tiles = torch::zeros({P}, geomBuffer.options().dtype(torch::kInt32));
    if (P > 0)
        check(fdgs_debug_export_geom(reinterpret_cast<const char*>(geomBuffer.data_ptr()), P, depths.data_ptr<float>(),
                                     means2D.data_ptr<float>(), conic.data_ptr<float>(), rgb.data_ptr<float>(),
                                     clamped.data_ptr<uint8_t>(), reinterpret_cast<unsigned int*>(tiles.data_ptr<int>()),
                                     (void*)on.stream),
              "debug_export_geom");
    return std::make_tuple(depths, means2D, conic, rgb, clamped, tiles);
}

std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> DebugExportBinning(const torch::Tensor& binningBuffer,
                                                                           const torch::Tensor& imgBuffer, const int R,
                                                                           const int W, const int H) {
    const DeviceStream on(imgBuffer);
    auto i32 = imgBuffer.options().dtype(torch::kInt32);
    const int tiles = ((W + 15) / 16) * ((H + 15) / 16);
    torch::Tensor point_list = torch::zeros({R}, i32), ranges = torch::zeros({tiles, 2}, i32),
                  n_contrib = torch::zeros({H, W}, i32);
    check(fdgs_debug_export_binning(R > 0 ? reinterpret_cast<const char*>(binningBuffer.data_ptr()) : nullptr,
                                    reinterpret_cast<const char*>(imgBuffer.data_ptr()), R, W, H,
                                    reinterpret_cast<unsigned int*>(point_list.data_ptr<int>()),
                                    reinterpret_cast<unsigned int*>(ranges.data_ptr<int>()),
                                    reinterpret_cast<unsigned int*>(n_contrib.data_ptr<int>()), (void*)on.stream),
          "debug_export_binning");
    return std::make_tuple(point_list, ranges, n_contrib);
}

// Multi-GPU exchange: gather the rows `idx` of every gradient tensor into one flat buffer (one block of K rows
// per tensor, 16-byte aligned block starts) / scatter the reduced rows back.  See fdgs/dist.py.
static std::vector<long long> block_offsets(const std::vector<torch::Tensor>& ts, long long K, std::vector<int>& widths,
                                            long long& total) {
    std::vector<long long> off;
    total = 0;
    for (const auto& t : ts) {
        arg<float>(t, "gradient tensor", -1, -1, REQUIRED);
        TORCH_CHECK(t.dim() >= 1, "fdgs: gradient tensor has the wrong shape");
        const long long w = t.size(0) > 0 ? t.numel() / t.size(0) : 0;
        TORCH_CHECK(w > 0, "fdgs: empty gradient tensor");
        widths.push_back((int)w);
        off.push_back(total);
        total += (K * w + 3) / 4 * 4;
    }
    return off;
}

torch::Tensor PackRows(std::vector<torch::Tensor> tensors, const torch::Tensor& idx) {
    TORCH_CHECK((int)tensors.size() <= FDGS_MAX_PACK, "fdgs: too many tensors");
    const long long* ip = reinterpret_cast<const long long*>(arg<int64_t>(idx, "idx", -1, -1, REQUIRED));
    const long long K = idx.numel();
    std::vector<int> widths;
    long long total = 0;
    std::vector<long long> off = block_offsets(tensors, K, widths, total);
    std::vector<torch::Tensor> dev(tensors);
    dev.push_back(idx);
    same_cuda_device("pack_rows", dev);
    torch::Tensor flat = torch::empty({total}, idx.options().dtype(torch::kFloat32));
    if (K == 0 || tensors.empty()) return flat;
    const DeviceStream on(idx);
    std::vector<const float*> ptr;
    for (const auto& t : tensors) ptr.push_back(t.data_ptr<float>());
    check(fdgs_pack_rows((int)tensors.size(), ptr.data(), widths.data(), off.data(), ip, K, flat.data_ptr<float>(),
                         (void*)on.stream),
          "pack_rows");
    return flat;
}

void UnpackRows(const torch::Tensor& flat, std::vector<torch::Tensor> tensors, const torch::Tensor& idx) {
    TORCH_CHECK((int)tensors.size() <= FDGS_MAX_PACK, "fdgs: too many tensors");
    const long long K = idx.numel();
    std::vector<int> widths;
    long long total = 0;
    std::vector<long long> off = block_offsets(tensors, K, widths, total);
    float* fp = arg<float>(flat, "flat buffer", -1, total, REQUIRED);
    same_cuda_device("unpack_rows", tensors);
    if (K == 0 || tensors.empty()) return;
    const DeviceStream on(idx);
    std::vector<float*> ptr;
    for (auto& t : tensors) ptr.push_back(t.data_ptr<float>());
    check(fdgs_unpack_rows((int)tensors.size(), ptr.data(), widths.data(), off.data(),
                           reinterpret_cast<const long long*>(idx.data_ptr<int64_t>()), K, fp, (void*)on.stream),
          "unpack_rows");
}

// ---- fused L1 + SSIM (include/fdgs.h: fdgs_l1_ssim_forward / _backward) ------------------------------------------
// returns (sums double[2] = {sum |x - y|, sum SSIM}, maps float[3,C,H,W])
std::tuple<torch::Tensor, torch::Tensor> L1SsimForward(const torch::Tensor& x, const torch::Tensor& y) {
    TORCH_CHECK(x.scalar_type() == torch::kFloat32 && y.scalar_type() == torch::kFloat32,
                "fdgs: images must be ", dtype_name(torch::kFloat32));
    TORCH_CHECK(x.dim() == 3 && x.sizes() == y.sizes(), "fdgs: images must be [C,H,W] of equal shape");
    same_cuda_device("l1_ssim", {x, y});
    const DeviceStream on(x);
    const auto xc = x.contiguous(), yc = y.contiguous();
    const int C = x.size(0), H = x.size(1), W = x.size(2);
    torch::Tensor sums = torch::empty({2}, x.options().dtype(torch::kFloat64));
    torch::Tensor maps = torch::empty({3, C, H, W}, x.options());
    check(fdgs_l1_ssim_forward(xc.data_ptr<float>(), yc.data_ptr<float>(), C, H, W, maps.data_ptr<float>(),
                               sums.data_ptr<double>(), (void*)on.stream),
          "l1_ssim_forward");
    return std::make_tuple(sums, maps);
}

torch::Tensor L1SsimBackward(const torch::Tensor& x, const torch::Tensor& y, const torch::Tensor& maps,
                             const torch::Tensor& grad_scale, const double lambda_dssim) {
    const DeviceStream on(x);
    const auto xc = x.contiguous(), yc = y.contiguous(), gs = grad_scale.to(torch::kFloat32).contiguous();
    const int C = x.size(0), H = x.size(1), W = x.size(2);
    torch::Tensor dx = torch::empty({C, H, W}, x.options());
    check(fdgs_l1_ssim_backward(xc.data_ptr<float>(), yc.data_ptr<float>(), C, H, W, maps.data_ptr<float>(),
                                gs.numel() ? gs.data_ptr<float>() : nullptr, (float)lambda_dssim, dx.data_ptr<float>(),
                                (void*)on.stream),
          "l1_ssim_backward");
    return dx;
}

// ---- fused Adam (include/fdgs.h: fdgs_adam_step) -------------------------------------------------------------------
void AdamStep(std::vector<torch::Tensor> params, std::vector<torch::Tensor> grads, std::vector<torch::Tensor> exp_avg,
              std::vector<torch::Tensor> exp_avg_sq, std::vector<double> lrs, const torch::Tensor& rows, const bool sparse,
              const int64_t step, const double beta1, const double beta2, const double eps, const bool zero_grad) {
    const size_t n = params.size();
    TORCH_CHECK(n <= FDGS_MAX_PACK && grads.size() == n && exp_avg.size() == n && exp_avg_sq.size() == n && lrs.size() == n,
                "fdgs: adam_step table mismatch");
    if (n == 0) return;
    const long long P = params[0].size(0);
    std::vector<float*> p, g, m, v;
    std::vector<int> widths;
    std::vector<float> lr;
    for (size_t i = 0; i < n; ++i) {
        const int64_t numel = params[i].numel();
        p.push_back(arg<float>(params[i], "adam tensor", P, numel, REQUIRED));
        g.push_back(arg<float>(grads[i], "adam tensor", P, numel, REQUIRED));
        m.push_back(arg<float>(exp_avg[i], "adam tensor", P, numel, REQUIRED));
        v.push_back(arg<float>(exp_avg_sq[i], "adam tensor", P, numel, REQUIRED));
        widths.push_back(P > 0 ? (int)(numel / P) : 1);
        lr.push_back((float)lrs[i]);
    }
    const long long* rp = sparse ? reinterpret_cast<const long long*>(arg<int64_t>(rows, "rows", -1, -1, REQUIRED)) : nullptr;
    std::vector<torch::Tensor> dev;
    for (size_t i = 0; i < n; ++i) dev.insert(dev.end(), {params[i], grads[i], exp_avg[i], exp_avg_sq[i]});
    if (sparse) dev.push_back(rows);
    same_cuda_device("adam", dev);
    if (sparse && rows.numel() == 0) return;
    const DeviceStream on(params[0]);
    check(fdgs_adam_step((int)n, p.data(), g.data(), m.data(), v.data(), widths.data(), lr.data(), P, rp,
                         sparse ? rows.numel() : 0, step, beta1, beta2, eps, zero_grad, (void*)on.stream),
          "adam_step");
}

// Adam's per-tensor scalars for a staged step (include/fdgs.h: fdgs_adam_scalars), written into `table`, a CPU float32
// tensor of 3 n elements (a pinned staging buffer): lr / bc1, sqrt(bc2), enable.
void AdamScalars(std::vector<double> lrs, std::vector<int64_t> steps, std::vector<int64_t> enable, const double beta1,
                 const double beta2, torch::Tensor& table) {
    const size_t n = lrs.size();
    TORCH_CHECK(n <= FDGS_MAX_PACK && steps.size() == n && enable.size() == n, "fdgs: adam_scalars table mismatch");
    TORCH_CHECK(table.defined() && !table.is_cuda(), "fdgs: adam_scalars writes a host table");
    float* out = arg<float>(table, "adam scalar table", -1, 3 * (int64_t)n, REQUIRED);
    std::vector<float> lr(n);
    std::vector<long long> st(n);
    std::vector<int> en(n);
    for (size_t i = 0; i < n; ++i) { lr[i] = (float)lrs[i]; st[i] = steps[i]; en[i] = enable[i] != 0; }
    check(fdgs_adam_scalars((int)n, lr.data(), st.data(), en.data(), beta1, beta2, out), "adam_scalars");
}

// Dense Adam with the scalars read on the device (include/fdgs.h: fdgs_adam_step_staged): scalars = CUDA float32 [3 n]
// as adam_scalars fills it, status = the rasterizer's int32 [4] or empty.  Capturable in a CUDA graph.
void AdamStepStaged(std::vector<torch::Tensor> params, std::vector<torch::Tensor> grads, std::vector<torch::Tensor> exp_avg,
                    std::vector<torch::Tensor> exp_avg_sq, const torch::Tensor& scalars, const torch::Tensor& status,
                    const double beta1, const double beta2, const double eps) {
    const size_t n = params.size();
    TORCH_CHECK(n <= FDGS_MAX_PACK && grads.size() == n && exp_avg.size() == n && exp_avg_sq.size() == n,
                "fdgs: adam_step_staged table mismatch");
    if (n == 0) return;
    const long long P = params[0].size(0);
    std::vector<float*> p, g, m, v;
    std::vector<int> widths;
    for (size_t i = 0; i < n; ++i) {
        const int64_t numel = params[i].numel();
        p.push_back(arg<float>(params[i], "adam tensor", P, numel, REQUIRED));
        g.push_back(arg<float>(grads[i], "adam tensor", P, numel, REQUIRED));
        m.push_back(arg<float>(exp_avg[i], "adam tensor", P, numel, REQUIRED));
        v.push_back(arg<float>(exp_avg_sq[i], "adam tensor", P, numel, REQUIRED));
        widths.push_back(P > 0 ? (int)(numel / P) : 1);
    }
    const float* sc = arg<float>(scalars, "adam scalar table", -1, 3 * (int64_t)n, REQUIRED);
    const int* st = arg<int>(status, "status", -1, 4);
    std::vector<torch::Tensor> dev;
    for (size_t i = 0; i < n; ++i) dev.insert(dev.end(), {params[i], grads[i], exp_avg[i], exp_avg_sq[i]});
    dev.insert(dev.end(), {scalars, status});
    same_cuda_device("adam", dev);
    const DeviceStream on(params[0]);
    check(fdgs_adam_step_staged((int)n, p.data(), g.data(), m.data(), v.data(), widths.data(), P, sc, st, beta1, beta2, eps,
                                (void*)on.stream),
          "adam_step_staged");
}

// ---- densification (include/fdgs.h: fdgs_densify_*, fdgs_reset_opacity) --------------------------------------------
// geo = [xyz, t, scaling, scaling_t, rotation, rotation_r, opacity]; stats = [xyz_gradient_accum, denom, max_radii2D];
// thresholds = [max_grad, min_opacity, percent_dense * extent, 0.1 * extent, max_screen_size] (rounded to fp32 here,
// as ATen rounds a Python scalar it compares an fp32 tensor with); flags = [N, gaussian_dim, rot_4d, prune_only,
// use_max_screen_size]
static fdgs_densify_args densify_args(const std::vector<torch::Tensor>& geo, const std::vector<torch::Tensor>& stats,
                                      const std::vector<double>& thr, const std::vector<int64_t>& flags) {
    TORCH_CHECK(geo.size() == 7 && stats.size() == 3 && thr.size() == 5 && flags.size() == 5, "fdgs: densify argument lists");
    fdgs_densify_args a;
    memset(&a, 0, sizeof(a));
    const long long P = geo[2].defined() ? geo[2].size(0) : 0;
    a.P = P;
    a.N = (int)flags[0]; a.gaussian_dim = (int)flags[1]; a.rot_4d = (int)flags[2]; a.prune_only = (int)flags[3];
    a.use_max_screen_size = (int)flags[4];
    a.max_grad = (float)thr[0]; a.min_opacity = (float)thr[1]; a.dense_extent = (float)thr[2]; a.big_extent = (float)thr[3];
    a.max_screen_size = (float)thr[4];
    a.xyz = arg<float>(geo[0], "xyz", P, 3 * P);
    a.t = arg<float>(geo[1], "t", P, P);
    a.scaling = arg<float>(geo[2], "scaling", P, 3 * P);
    a.scaling_t = arg<float>(geo[3], "scaling_t", P, P);
    a.rotation = arg<float>(geo[4], "rotation", P, 4 * P);
    a.rotation_r = arg<float>(geo[5], "rotation_r", P, 4 * P);
    a.opacity = arg<float>(geo[6], "opacity", P, P);
    a.xyz_gradient_accum = arg<float>(stats[0], "xyz_gradient_accum", P, P);
    a.denom = arg<float>(stats[1], "denom", P, P);
    a.max_radii2D = arg<float>(stats[2], "max_radii2D", P, P);
    same_cuda_device("densification", {geo[0], geo[1], geo[2], geo[3], geo[4], geo[5], geo[6], stats[0], stats[1], stats[2]});
    return a;
}

std::tuple<torch::Tensor, torch::Tensor> DensifyPlan(const std::vector<torch::Tensor>& geo, const std::vector<torch::Tensor>& stats,
                                                     const std::vector<double>& thr, const std::vector<int64_t>& flags) {
    fdgs_densify_args a = densify_args(geo, stats, thr, flags);
    TORCH_CHECK(geo[2].defined() && geo[2].is_cuda(), "fdgs: scaling must be a CUDA tensor");
    const DeviceStream on(geo[2]);
    auto opts = geo[2].options();
    torch::Tensor scratch = torch::empty({(int64_t)fdgs_densify_scratch_bytes(a.P) + 16}, opts.dtype(torch::kByte));
    torch::Tensor totals = torch::empty({4}, opts.dtype(torch::kInt32));
    check(fdgs_densify_plan(&a, reinterpret_cast<char*>(scratch.data_ptr()), totals.data_ptr<int>(), (void*)on.stream),
          "densify_plan");
    return std::make_tuple(scratch, totals);
}

// srcs / dsts / kinds: the compaction table (include/fdgs.h FDGS_DENSIFY_*); totals: the plan's totals on the host
void DensifyApply(const std::vector<torch::Tensor>& geo, const std::vector<torch::Tensor>& stats, const std::vector<double>& thr,
                  const std::vector<int64_t>& flags, const std::vector<torch::Tensor>& srcs, const std::vector<torch::Tensor>& dsts,
                  const std::vector<int64_t>& kinds, const torch::Tensor& scratch, const std::vector<int64_t>& totals,
                  const torch::Tensor& samples, const torch::Tensor& samples_t) {
    fdgs_densify_args a = densify_args(geo, stats, thr, flags);
    const size_t n = srcs.size();
    TORCH_CHECK(n <= FDGS_DENSIFY_MAX_TENSORS && dsts.size() == n && kinds.size() == n && totals.size() == 4,
                "fdgs: densify tensor table mismatch");
    const long long P_new = totals[0] + totals[1] + (long long)a.N * totals[3];
    a.num_tensors = (int)n;
    for (size_t i = 0; i < n; ++i) {
        const long long w = a.P > 0 ? srcs[i].numel() / a.P : 1;
        a.src[i] = arg<float>(srcs[i], "source row tensor", a.P, a.P * w);
        a.dst[i] = arg<float>(dsts[i], "destination row tensor", P_new, P_new * w);
        if (a.P == 0 || P_new == 0) { a.num_tensors = 0; break; }     // nothing to copy from or to
        TORCH_CHECK(a.src[i] && a.dst[i], "fdgs: densify tensor table entry missing");
        a.kind[i] = (int)kinds[i];
        a.width[i] = (int)w;
    }
    const long long SN = totals[2] * (long long)a.N;
    a.samples = arg<float>(samples, "samples", SN, SN * (a.rot_4d ? 4 : 3));
    a.samples_t = arg<float>(samples_t, "samples_t", SN, SN);
    for (size_t i = 0; i < n; ++i) same_cuda_device("densification", {geo[2], srcs[i], dsts[i]});
    same_cuda_device("densification", {geo[2], samples, samples_t});
    TORCH_CHECK(scratch.is_cuda() && scratch.scalar_type() == torch::kByte &&
                scratch.numel() >= (int64_t)fdgs_densify_scratch_bytes(a.P), "fdgs: densify scratch of the plan required");
    int tot[4];
    for (int i = 0; i < 4; ++i) tot[i] = (int)totals[i];
    const DeviceStream on(scratch);
    check(fdgs_densify_apply(&a, reinterpret_cast<const char*>(scratch.data_ptr()), tot, (void*)on.stream), "densify_apply");
}

void ResetOpacity(torch::Tensor& opacity, torch::Tensor& exp_avg, torch::Tensor& exp_avg_sq) {
    const long long P = opacity.size(0);
    float* o = arg<float>(opacity, "opacity", P, P);
    float* m = arg<float>(exp_avg, "exp_avg", P, P);
    float* v = arg<float>(exp_avg_sq, "exp_avg_sq", P, P);
    same_cuda_device("densification", {opacity, exp_avg, exp_avg_sq});
    if (P == 0) return;
    const DeviceStream on(opacity);
    check(fdgs_reset_opacity(P, o, m, v, (void*)on.stream), "reset_opacity");
}

// batch_size 1: point_grad = viewspace_points.grad [P, >= 2], visibility_count empty; batch_size > 1: point_grad =
// the summed norms [P] and visibility_count [P] (fdgs.dist.ViewBatchStats).  t_grad / t_gradient_accum empty for 3D.
// status: the rasterizer's int32 [4] (render_batch's pkg["status"]) or empty: nothing is written on overflow or wrap.
void DensifyStatsStatus(int64_t batch_size, const torch::Tensor& point_grad, const torch::Tensor& visibility_count,
                        const torch::Tensor& radii, const torch::Tensor& t_grad, torch::Tensor& xyz_gradient_accum,
                        torch::Tensor& denom, torch::Tensor& t_gradient_accum, torch::Tensor& max_radii2D,
                        const torch::Tensor& status) {
    const long long P = xyz_gradient_accum.size(0);
    float* acc = arg<float>(xyz_gradient_accum, "xyz_gradient_accum", P, P);
    float* den = arg<float>(denom, "denom", P, P);
    float* tacc = arg<float>(t_gradient_accum, "t_gradient_accum", P, P);
    float* mr = arg<float>(max_radii2D, "max_radii2D", P, P);
    const float* tg = arg<float>(t_grad, "t_grad", P, P);
    const float* vis = arg<float>(visibility_count, "visibility_count", P, P);
    const float* pg = arg<float>(point_grad, "point_grad", P, batch_size == 1 ? -1 : P);
    TORCH_CHECK(point_grad.defined() && (batch_size > 1 || point_grad.dim() == 2), "fdgs: point_grad must be [P, >= 2] for one view");
    const int* r = arg<int>(radii, "radii", -1, P, REQUIRED);
    const int* st = arg<int>(status, "status", -1, 4);
    same_cuda_device("densification",
                     {xyz_gradient_accum, denom, t_gradient_accum, max_radii2D, t_grad, visibility_count, point_grad, radii,
                      status});
    const int stride = batch_size == 1 ? (int)(point_grad.dim() == 2 ? point_grad.size(1) : 0) : 1;
    if (P == 0) return;
    const DeviceStream on(xyz_gradient_accum);
    check(fdgs_densify_stats_status(P, (int)batch_size, pg, stride, vis, r, tg, acc, den, tacc, mr, st, (void*)on.stream),
          "densify_stats");
}

void DensifyStats(int64_t batch_size, const torch::Tensor& point_grad, const torch::Tensor& visibility_count,
                  const torch::Tensor& radii, const torch::Tensor& t_grad, torch::Tensor& xyz_gradient_accum, torch::Tensor& denom,
                  torch::Tensor& t_gradient_accum, torch::Tensor& max_radii2D) {
    DensifyStatsStatus(batch_size, point_grad, visibility_count, radii, t_grad, xyz_gradient_accum, denom, t_gradient_accum,
                       max_radii2D, torch::Tensor());
}

// ---- k nearest neighbours (include/fdgs.h: fdgs_knn) ---------------------------------------------------------------
std::tuple<torch::Tensor, torch::Tensor> Knn(const torch::Tensor& xyz, const int64_t k, const bool brute_force) {
    TORCH_CHECK(xyz.scalar_type() == torch::kFloat32, "fdgs: xyz must be ", dtype_name(torch::kFloat32));
    TORCH_CHECK(xyz.dim() == 2 && xyz.size(1) == 3, "fdgs: xyz must be [n,3]");
    TORCH_CHECK(xyz.is_cuda(), "fdgs: xyz must be a CUDA tensor");
    const DeviceStream on(xyz);
    const auto x = xyz.contiguous();
    const int n = x.size(0);
    torch::Tensor idx = torch::empty({n, k}, x.options().dtype(torch::kInt32));
    torch::Tensor d2 = torch::empty({n, k}, x.options());
    torch::Tensor scratch = torch::empty({(int64_t)(brute_force ? 16 : fdgs_knn_scratch_bytes(n))}, x.options().dtype(torch::kByte));
    check(fdgs_knn(n, (int)k, x.data_ptr<float>(), reinterpret_cast<char*>(scratch.data_ptr()), idx.data_ptr<int>(),
                   d2.data_ptr<float>(), brute_force, (void*)on.stream),
          "knn");
    return std::make_tuple(idx, d2);
}

// ---- rigidity and motion regularisers (include/fdgs.h: fdgs_rigid_*) -----------------------------------------------
// params = [t [n,1], scaling [n,3], scaling_t [n,1], rotation [n,4], rotation_r [n,4]] (the raw parameters)
static fdgs_rigid_args rigid_args(const std::vector<torch::Tensor>& params, int64_t k) {
    TORCH_CHECK(params.size() == 5, "fdgs: five parameter tensors (t, scaling, scaling_t, rotation, rotation_r)");
    TORCH_CHECK(params[1].defined() && params[1].dim() == 2, "fdgs: scaling must be [n,3]");
    const int64_t n = params[1].size(0);
    fdgs_rigid_args a;
    memset(&a, 0, sizeof(a));
    a.n = (int)n;
    a.k = (int)k;
    a.t = arg<float>(params[0], "t", n, n, REQUIRED);
    a.scaling = arg<float>(params[1], "scaling", n, 3 * n, REQUIRED);
    a.scaling_t = arg<float>(params[2], "scaling_t", n, n, REQUIRED);
    a.rotation = arg<float>(params[3], "rotation", n, 4 * n, REQUIRED);
    a.rotation_r = arg<float>(params[4], "rotation_r", n, 4 * n, REQUIRED);
    return a;
}

static void rigid_list(fdgs_rigid_args& a, const torch::Tensor& idx, const torch::Tensor& weight) {
    const int64_t n = a.n, k = a.k;
    a.idx = arg<int>(idx, "idx", n, n * k, REQUIRED);
    a.weight = arg<float>(weight, "weight", n, n * k, REQUIRED);
}

// (weight, in_offsets, in_edges) of fdgs_knn's (idx, dist2)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> RigidNeighbours(const torch::Tensor& idx, const torch::Tensor& dist2) {
    TORCH_CHECK(idx.defined() && idx.dim() == 2, "fdgs: idx must be [n,k]");
    const int64_t n = idx.size(0), k = idx.size(1);
    TORCH_CHECK(n > 0 && k >= 1 && k <= 32, "fdgs: bad n / k (n > 0, 1 <= k <= 32)");
    const int* ip = arg<int>(idx, "idx", n, n * k, REQUIRED);
    const float* dp = arg<float>(dist2, "dist2", n, n * k, REQUIRED);
    same_cuda_device("regulariser", {idx, dist2});
    const DeviceStream on(idx);
    auto opts = dist2.options();
    torch::Tensor weight = torch::empty({n, k}, opts);
    torch::Tensor in_offsets = torch::empty({n + 1}, opts.dtype(torch::kInt32));
    torch::Tensor in_edges = torch::empty({n * k}, opts.dtype(torch::kInt32));
    torch::Tensor scratch = torch::empty({(int64_t)fdgs_rigid_scratch_bytes((int)n, (int)k) + 256}, opts.dtype(torch::kByte));
    check(fdgs_rigid_neighbours((int)n, (int)k, ip, dp, reinterpret_cast<char*>(scratch.data_ptr()), weight.data_ptr<float>(),
                                in_offsets.data_ptr<int>(), in_edges.data_ptr<int>(), (void*)on.stream),
          "rigid_neighbours");
    return std::make_tuple(weight, in_offsets, in_edges);
}

// (velocity [n,3], loss_rigid, loss_motion); an unwanted loss comes back as 0
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> RigidForward(const std::vector<torch::Tensor>& params, const int64_t k,
                                                                     const torch::Tensor& idx, const torch::Tensor& weight,
                                                                     const bool want_rigid, const bool want_motion) {
    fdgs_rigid_args a = rigid_args(params, k);
    if (want_rigid) rigid_list(a, idx, weight);
    same_cuda_device("regulariser", {params[0], params[1], params[2], params[3], params[4], idx, weight});
    TORCH_CHECK(params[1].is_cuda(), "fdgs: regulariser tensors must be CUDA tensors");
    const DeviceStream on(params[1]);
    auto opts = params[1].options();
    torch::Tensor velocity = torch::empty({params[1].size(0), 3}, opts);
    torch::Tensor lr = want_rigid ? torch::empty({}, opts) : torch::zeros({}, opts);
    torch::Tensor lm = want_motion ? torch::empty({}, opts) : torch::zeros({}, opts);
    const size_t sb = fdgs_rigid_scratch_bytes(a.n, a.k);
    torch::Tensor scratch = torch::empty({(int64_t)sb + 256}, opts.dtype(torch::kByte));
    a.velocity = velocity.data_ptr<float>();
    check(fdgs_rigid_forward(&a, reinterpret_cast<char*>(scratch.data_ptr()), want_rigid ? lr.data_ptr<float>() : nullptr,
                             want_motion ? lm.data_ptr<float>() : nullptr, (void*)on.stream),
          "rigid_forward");
    return std::make_tuple(velocity, lr, lm);
}

// gradients (scaling, scaling_t, rotation, rotation_r) shaped like the parameters; grad_rigid / grad_motion: the upstream
// gradients (0-dim device tensors, empty = no such term)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor> RigidBackward(
    const std::vector<torch::Tensor>& params, const int64_t k, const torch::Tensor& velocity, const torch::Tensor& idx,
    const torch::Tensor& weight, const torch::Tensor& in_offsets, const torch::Tensor& in_edges, const torch::Tensor& grad_rigid,
    const torch::Tensor& grad_motion) {
    fdgs_rigid_args a = rigid_args(params, k);
    const int64_t n = a.n;
    a.velocity = arg<float>(velocity, "velocity", n, 3 * n, REQUIRED);
    const float* gr = arg<float>(grad_rigid, "grad_rigid", -1, 1);
    const float* gm = arg<float>(grad_motion, "grad_motion", -1, 1);
    if (gr) {
        rigid_list(a, idx, weight);
        a.in_offsets = arg<int>(in_offsets, "in_offsets", n + 1, n + 1, REQUIRED);
        a.in_edges = arg<int>(in_edges, "in_edges", n * k, n * k, REQUIRED);
    }
    same_cuda_device("regulariser", {params[0], params[1], params[2], params[3], params[4], velocity, idx, weight, in_offsets,
                                     in_edges, grad_rigid, grad_motion});
    TORCH_CHECK(params[1].is_cuda(), "fdgs: regulariser tensors must be CUDA tensors");
    const DeviceStream on(params[1]);
    torch::Tensor ds = torch::empty_like(params[1]), dst = torch::empty_like(params[2]);
    torch::Tensor dr = torch::empty_like(params[3]), drr = torch::empty_like(params[4]);
    check(fdgs_rigid_backward(&a, gr, gm, ds.data_ptr<float>(), dst.data_ptr<float>(), dr.data_ptr<float>(), drr.data_ptr<float>(),
                              (void*)on.stream),
          "rigid_backward");
    return std::make_tuple(ds, dst, dr, drr);
}

// ---- evaluation metrics (include/fdgs.h: fdgs_image_metrics) ---------------------------------------------------------
// x, y: [B,C,H,W] float32 contiguous CUDA tensors; accum: float64 [5] on the same device, or empty = none.
// Returns out [B,4] float64 (l1, psnr, ssim, msssim per view).  Checks dtype, layout and shape before the device.
torch::Tensor ImageMetrics(const torch::Tensor& x, const torch::Tensor& y, const bool clamp, const torch::Tensor& accum) {
    fdgs_metrics_args a;
    memset(&a, 0, sizeof(a));
    a.x = arg<float>(x, "images", -1, -1, REQUIRED);
    a.y = arg<float>(y, "images", -1, -1, REQUIRED);
    TORCH_CHECK(x.dim() == 4 && x.sizes() == y.sizes(), "fdgs: images must be [B,C,H,W] of equal shape");
    a.accum = arg<double>(accum, "accum", -1, 5);
    same_cuda_device("image_metrics", {x, y, accum});
    a.B = (int)x.size(0); a.C = (int)x.size(1); a.H = (int)x.size(2); a.W = (int)x.size(3);
    TORCH_CHECK(x.size(0) == a.B && x.size(1) == a.C && x.size(2) == a.H && x.size(3) == a.W, "fdgs: image size overflow");
    const size_t sb = fdgs_metrics_scratch_bytes(a.B, a.C, a.H, a.W);
    const DeviceStream on(x);
    torch::Tensor out = torch::empty({x.size(0), 4}, x.options().dtype(torch::kFloat64));
    torch::Tensor scratch = torch::empty({(int64_t)sb}, x.options().dtype(torch::kByte));
    a.clamp = clamp ? 1 : 0;
    a.out = out.data_ptr<double>();
    check(fdgs_image_metrics(&a, reinterpret_cast<char*>(scratch.data_ptr()), (void*)on.stream), "image_metrics");
    return out;
}

std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> DebugActivate(const torch::Tensor& log_s, const torch::Tensor& logit,
                                                                      const torch::Tensor& quat, const int64_t mode) {
    const DeviceStream on(log_s);
    const auto a = log_s.contiguous(), b = logit.contiguous(), q = quat.contiguous();
    const int n = (int)a.numel();
    TORCH_CHECK(b.numel() == n && q.numel() == 4 * (int64_t)n, "fdgs: debug_activate shapes");
    torch::Tensor s = torch::empty_like(a), o = torch::empty_like(b), qo = torch::empty_like(q);
    check(fdgs_debug_activate(n, a.data_ptr<float>(), b.data_ptr<float>(), q.data_ptr<float>(), (int)mode, s.data_ptr<float>(),
                              o.data_ptr<float>(), qo.data_ptr<float>(), (void*)on.stream),
          "debug_activate");
    return std::make_tuple(s, o, qo);
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.def("debug_activate", &DebugActivate);
    m.def("l1_ssim_forward", &L1SsimForward);
    m.def("l1_ssim_backward", &L1SsimBackward);
    m.def("adam_step", &AdamStep);
    m.def("adam_scalars", &AdamScalars);
    m.def("adam_step_staged", &AdamStepStaged);
    m.def("knn", &Knn);
    m.def("rigid_neighbours", &RigidNeighbours);
    m.def("rigid_forward", &RigidForward);
    m.def("rigid_backward", &RigidBackward);
    m.def("image_metrics", &ImageMetrics);
    m.def("densify_plan", &DensifyPlan);
    m.def("densify_apply", &DensifyApply);
    m.def("reset_opacity", &ResetOpacity);
    m.def("densify_stats", &DensifyStats);
    m.def("densify_stats", &DensifyStatsStatus);
    m.def("pack_rows", &PackRows);
    m.def("unpack_rows", &UnpackRows);
    m.def("rasterize_gaussians", &RasterizeGaussiansCUDA);
    m.def("rasterize_gaussians_backward", &RasterizeGaussiansBackwardCUDA);
    m.def("rasterize_gaussians_ext", &RasterizeGaussiansExt);
    m.def("rasterize_gaussians_ext", &RasterizeGaussiansExtZeroSh);
    m.def("rasterize_gaussians_backward_ext", &RasterizeGaussiansBackwardExt);
    m.def("rasterize_gaussians_backward_ext", &RasterizeGaussiansBackwardExtZeroSh);
    m.def("rasterize_gaussians_batch", &RasterizeGaussiansBatch);
    m.def("rasterize_gaussians_backward_batch", &RasterizeGaussiansBackwardBatch);
    m.def("rasterize_gaussians_backward_camera", &RasterizeGaussiansBackwardCamera);
    m.def("rasterize_gaussians_backward_batch_camera", &RasterizeGaussiansBackwardBatchCamera);
    m.def("rasterize_gaussians_batch_capacity", &RasterizeGaussiansBatchCapacity);
    m.def("debug_export_binning_view", &DebugExportBinningView);
    m.def("sky_forward", &SkyForward);
    m.def("sky_backward", &SkyBackward);
    m.def("sky_forward_batch", &SkyForwardBatch);
    m.def("sky_backward_batch", &SkyBackwardBatch);
    m.def("sh_outer_sum", &ShOuterSum);
    m.def("check_rows_zero", &CheckRowsZero);
    m.def("union_maps", &UnionMaps);
    m.def("view_stats", &ViewStats);
    m.def("mark_visible", &markVisible);
    m.def("debug_export_geom", &DebugExportGeom);
    m.def("debug_export_binning", &DebugExportBinning);
    m.def("fdgs_version", []() { return fdgs_version(); });
}
