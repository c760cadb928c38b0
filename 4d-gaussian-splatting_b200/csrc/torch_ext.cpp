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
#include <tuple>
#include <vector>
#include "../../include/fdgs.h"

namespace {

char* resize_cb(void* ctx, size_t bytes) {
    auto* t = reinterpret_cast<torch::Tensor*>(ctx);
    t->resize_({(long long)bytes});
    return reinterpret_cast<char*>(t->data_ptr());
}

const float* fptr(const torch::Tensor& t) {
    // empty tensor == "not provided" (reference: diff_gaussian_rasterization.py:282-300)
    if (!t.defined() || t.numel() == 0) return nullptr;
    TORCH_CHECK(t.is_cuda(), "fdgs: expected a CUDA tensor");
    TORCH_CHECK(t.scalar_type() == torch::kFloat32, "fdgs: expected a float32 tensor");
    return t.data_ptr<float>();
}

torch::Tensor contig(const torch::Tensor& t) { return (t.defined() && t.numel() > 0) ? t.contiguous() : t; }

// the per-pixel background image of a call, checked against the image size (undefined / empty = none)
torch::Tensor background_image(const torch::Tensor& bg_image, const torch::Tensor& like, int H, int W) {
    if (!bg_image.defined() || bg_image.numel() == 0) return torch::Tensor();
    TORCH_CHECK(bg_image.is_cuda() && bg_image.device() == like.device(), "fdgs: bg_image must be on the device of means3D");
    TORCH_CHECK(bg_image.scalar_type() == torch::kFloat32, "fdgs: bg_image must be float32");
    TORCH_CHECK(bg_image.dim() == 3 && bg_image.size(0) == 3 && bg_image.size(1) == H && bg_image.size(2) == W,
                "fdgs: bg_image must be [3, image_height, image_width]");
    return bg_image.contiguous();
}

void check(int rc, const char* where) {
    if (rc != FDGS_OK) throw std::runtime_error(std::string("fdgs ") + where + " failed: " + fdgs_last_error());
}

}  // namespace

#define FDGS_FWD_PARAMS                                                                                                \
    const torch::Tensor &background, const torch::Tensor &means3D, const torch::Tensor &colors,                        \
        const torch::Tensor &flows, const torch::Tensor &opacity, const torch::Tensor &ts, const torch::Tensor &scales, \
        const torch::Tensor &scales_t, const torch::Tensor &rotations, const torch::Tensor &rotations_r,               \
        const float scale_modifier, const torch::Tensor &cov3D_precomp, const float prefilter_var,                     \
        const torch::Tensor &viewmatrix, const torch::Tensor &projmatrix, const float tan_fovx, const float tan_fovy,  \
        const int image_height, const int image_width, const torch::Tensor &sh, const int degree, const int degree_t,  \
        const torch::Tensor &campos, const float timestamp, const float time_duration, const bool rot_4d,              \
        const int gaussian_dim, const bool force_sh_3d, const bool prefiltered, const bool debug
#define FDGS_FWD_ARGS                                                                                                  \
    background, means3D, colors, flows, opacity, ts, scales, scales_t, rotations, rotations_r, scale_modifier,         \
        cov3D_precomp, prefilter_var, viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh,       \
        degree, degree_t, campos, timestamp, time_duration, rot_4d, gaussian_dim, force_sh_3d, prefiltered, debug

using ForwardOut = std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
                              torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>;

// sh_rest (possibly empty) / raw_params: the raw-parameter entry of include/fdgs.h (fdgs_forward_args.raw_params)
static ForwardOut
forward_impl(const torch::Tensor& bg_image, const torch::Tensor& sh_rest, const bool raw_params,
                       const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors,
                       const torch::Tensor& flows, const torch::Tensor& opacity, const torch::Tensor& ts,
                       const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                       const torch::Tensor& rotations_r, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                       const float prefilter_var, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
                       const float tan_fovx, const float tan_fovy, const int image_height, const int image_width,
                       const torch::Tensor& sh, const int degree, const int degree_t, const torch::Tensor& campos,
                       const float timestamp, const float time_duration, const bool rot_4d, const int gaussian_dim,
                       const bool force_sh_3d, const bool prefiltered, const bool debug) {
    if (means3D.ndimension() != 2 || means3D.size(1) != 3) {
        AT_ERROR("means3D must have dimensions (num_points, 3)");   // reference: rasterize_points.cu:69-71
    }
    TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor");
    const c10::cuda::CUDAGuard guard(means3D.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();

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

    // keep contiguous copies alive for the duration of the call
    const auto bg_c = contig(background), means_c = contig(means3D), col_c = contig(colors), flow_c = contig(flows),
               op_c = contig(opacity), ts_c = contig(ts), sc_c = contig(scales), sct_c = contig(scales_t),
               rot_c = contig(rotations), rotr_c = contig(rotations_r), cov_c = contig(cov3D_precomp),
               view_c = contig(viewmatrix), proj_c = contig(projmatrix), sh_c = contig(sh), cam_c = contig(campos);

    fdgs_forward_args a;
    memset(&a, 0, sizeof(a));
    a.P = P; a.D = degree; a.D_t = degree_t;
    const auto shr_c = contig(sh_rest);
    a.M = (sh.defined() && sh.numel() != 0) ? (int)sh.size(1) : 0;
    if (shr_c.defined() && shr_c.numel() != 0) {
        TORCH_CHECK(a.M == 1 && shr_c.dim() == 3 && shr_c.size(0) == P, "fdgs: split SH rows are [P,1,3] + [P,M-1,3]");
        a.M += (int)shr_c.size(1);
        a.shs_rest = fptr(shr_c);
    }
    a.raw_params = raw_params;
    a.background = fptr(bg_c); a.width = W; a.height = H;
    a.means3D = fptr(means_c); a.shs = fptr(sh_c); a.colors_precomp = fptr(col_c); a.flows_precomp = fptr(flow_c);
    a.opacities = fptr(op_c); a.ts = fptr(ts_c); a.scales = fptr(sc_c); a.scales_t = fptr(sct_c);
    a.scale_modifier = scale_modifier; a.rotations = fptr(rot_c); a.rotations_r = fptr(rotr_c);
    a.cov3D_precomp = fptr(cov_c); a.prefilter_var = prefilter_var;
    a.viewmatrix = fptr(view_c); a.projmatrix = fptr(proj_c); a.cam_pos = fptr(cam_c);
    a.timestamp = timestamp; a.time_duration = time_duration; a.rot_4d = rot_4d; a.gaussian_dim = gaussian_dim;
    a.force_sh_3d = force_sh_3d; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy; a.prefiltered = prefiltered;
    a.debug = debug;
    a.out_means3D = out_means3D.data_ptr<float>(); a.out_color = out_color.data_ptr<float>();
    a.out_flow = out_flow.data_ptr<float>(); a.out_depth = out_depth.data_ptr<float>();
    a.out_T = out_T.data_ptr<float>(); a.radii = radii.data_ptr<int>();

    const auto bgi_c = background_image(bg_image, means3D, H, W);
    fdgs_forward_result r;
    check(fdgs_forward_bg(&a, fptr(bgi_c), resize_cb, &geomBuffer, resize_cb, &binningBuffer, resize_cb, &imgBuffer,
                          (void*)stream, &r),
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

// the reference's entry point: 30 positional arguments, 11-tuple (rasterize_points.h:18-49)
ForwardOut RasterizeGaussiansCUDA(FDGS_FWD_PARAMS) { return forward_impl(torch::Tensor(), torch::Tensor(), false, FDGS_FWD_ARGS); }

// the same + a per-pixel background image bg_image [3,H,W] (include/fdgs.h: fdgs_forward_bg; empty = none)
ForwardOut RasterizeGaussiansBg(FDGS_FWD_PARAMS, const torch::Tensor& bg_image) {
    return forward_impl(bg_image, torch::Tensor(), false, FDGS_FWD_ARGS);
}

// raw-parameter entry: the same 30 arguments (scales = log-scales, rotations un-normalised, opacity = logits when
// raw_params) + the second SH tensor (sh = features_dc [P,1,3], sh_rest = features_rest [P,M-1,3]; may be empty)
ForwardOut RasterizeGaussiansRaw(FDGS_FWD_PARAMS, const torch::Tensor& sh_rest, const bool raw_params) {
    return forward_impl(torch::Tensor(), sh_rest, raw_params, FDGS_FWD_ARGS);
}

ForwardOut RasterizeGaussiansRawBg(FDGS_FWD_PARAMS, const torch::Tensor& sh_rest, const bool raw_params,
                                   const torch::Tensor& bg_image) {
    return forward_impl(bg_image, sh_rest, raw_params, FDGS_FWD_ARGS);
}

namespace {
struct BackwardOut {
    torch::Tensor dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dflows, dL_dts, dL_dscales,
        dL_dscales_t, dL_drotations, dL_drotations_r, sh_factors, dL_dsh_rest, dL_dbg_image;
};
}  // namespace

// sh_factor_mode: view-parallel mode -- no dL_dsh rows, the [P,3] colour factors instead (include/fdgs.h: sh_factors)
static BackwardOut
backward_impl(const torch::Tensor& bg_image, const bool want_dbg, const bool sh_factor_mode, const torch::Tensor& sh_rest,
                               const bool raw_params,
                               const torch::Tensor& background, const torch::Tensor& means3D,
                               const torch::Tensor& out_means3D, const torch::Tensor& radii, const torch::Tensor& colors,
                               const torch::Tensor& flows_2d, const torch::Tensor& opacities, const torch::Tensor& ts,
                               const torch::Tensor& scales, const torch::Tensor& scales_t, const torch::Tensor& rotations,
                               const torch::Tensor& rotations_r, const float scale_modifier,
                               const torch::Tensor& cov3D_precomp, const float prefilter_var,
                               const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx,
                               const float tan_fovy, const torch::Tensor& dL_dout_color,
                               const torch::Tensor& dL_dout_depth, const torch::Tensor& dL_dout_mask,
                               const torch::Tensor& dL_dout_flow, const torch::Tensor& sh, const int degree,
                               const int degree_t, const torch::Tensor& campos, const float timestamp,
                               const float time_duration, const bool rot_4d, const int gaussian_dim,
                               const bool force_sh_3d, const torch::Tensor& geomBuffer, const int R,
                               const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const bool debug) {
    TORCH_CHECK(means3D.is_cuda(), "means3D must be a CUDA tensor");
    const c10::cuda::CUDAGuard guard(means3D.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    const int P = means3D.size(0);
    const int H = dL_dout_color.size(1), W = dL_dout_color.size(2);
    const bool split = sh_rest.defined() && sh_rest.numel() != 0;
    const int M = ((sh.defined() && sh.numel() != 0) ? (int)sh.size(1) : 0) + (split ? (int)sh_rest.size(1) : 0);
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
    torch::Tensor dL_dsh = factors ? torch::empty({0}, opts) : torch::empty({P, split ? 1 : M, 3}, opts);
    torch::Tensor dL_dsh_rest = (split && !factors) ? torch::empty({P, M - 1, 3}, opts) : torch::empty({0}, opts);
    torch::Tensor sh_factors = factors ? torch::empty({P, 3}, opts) : torch::empty({0}, opts);
    torch::Tensor dL_dscales = torch::empty({P, 3}, opts);
    torch::Tensor dL_dscales_t = torch::empty({P, 1}, opts);
    torch::Tensor dL_drotations = torch::empty({P, 4}, opts);
    torch::Tensor dL_drotations_r = torch::empty({P, 4}, opts);
    // overwritten for every pixel by the blend backward
    torch::Tensor dL_dbg_image = want_dbg ? torch::empty({3, H, W}, opts) : torch::empty({0}, opts);
    const auto bgi_c = background_image(bg_image, means3D, H, W);

    if (P != 0 || want_dbg) {
        const auto bg_c = contig(background), om_c = contig(out_means3D), rad_c = contig(radii), col_c = contig(colors),
                   flow_c = contig(flows_2d), op_c = contig(opacities), ts_c = contig(ts), sc_c = contig(scales),
                   sct_c = contig(scales_t), rot_c = contig(rotations), rotr_c = contig(rotations_r),
                   cov_c = contig(cov3D_precomp), view_c = contig(viewmatrix), proj_c = contig(projmatrix),
                   gc_c = contig(dL_dout_color), gd_c = contig(dL_dout_depth), gm_c = contig(dL_dout_mask),
                   gf_c = contig(dL_dout_flow), sh_c = contig(sh), cam_c = contig(campos), geo_c = contig(geomBuffer),
                   bin_c = contig(binningBuffer), img_c = contig(imageBuffer);
        fdgs_backward_args a;
        memset(&a, 0, sizeof(a));
        a.P = P; a.D = degree; a.D_t = degree_t; a.M = M; a.R = R;
        a.background = fptr(bg_c); a.width = W; a.height = H;
        a.out_means3D = fptr(om_c); a.shs = fptr(sh_c); a.colors_precomp = fptr(col_c); a.flows_2d = fptr(flow_c);
        a.opacities = fptr(op_c); a.ts = fptr(ts_c); a.scales = fptr(sc_c); a.scales_t = fptr(sct_c);
        a.scale_modifier = scale_modifier; a.rotations = fptr(rot_c); a.rotations_r = fptr(rotr_c);
        a.cov3D_precomp = fptr(cov_c); a.prefilter_var = prefilter_var;
        a.viewmatrix = fptr(view_c); a.projmatrix = fptr(proj_c); a.campos = fptr(cam_c);
        a.timestamp = timestamp; a.time_duration = time_duration; a.rot_4d = rot_4d; a.gaussian_dim = gaussian_dim;
        a.force_sh_3d = force_sh_3d; a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy;
        a.radii = rad_c.numel() ? rad_c.data_ptr<int>() : nullptr;
        a.geom_buffer = geo_c.numel() ? reinterpret_cast<const char*>(geo_c.data_ptr()) : nullptr;
        a.binning_buffer = bin_c.numel() ? reinterpret_cast<const char*>(bin_c.data_ptr()) : nullptr;
        a.image_buffer = reinterpret_cast<const char*>(img_c.data_ptr());
        a.dL_dpix = fptr(gc_c); a.dL_depths = fptr(gd_c); a.dL_masks = fptr(gm_c); a.dL_dpix_flow = fptr(gf_c);
        a.debug = debug;
        a.dL_dmean2D = dL_dmeans2D.data_ptr<float>(); a.dL_dconic = dL_dconic.data_ptr<float>();
        a.dL_dopacity = dL_dopacity.data_ptr<float>(); a.dL_dcolor = dL_dcolors.data_ptr<float>();
        a.dL_dflows = dL_dflows.data_ptr<float>(); a.dL_dmean3D = dL_dmeans3D.data_ptr<float>();
        a.dL_dcov3D = dL_dcov3D.data_ptr<float>(); a.dL_dsh = (M > 0 && !factors) ? dL_dsh.data_ptr<float>() : nullptr;
        a.sh_factors = factors ? sh_factors.data_ptr<float>() : nullptr;
        const auto shr_c = contig(sh_rest);
        a.shs_rest = split ? fptr(shr_c) : nullptr;
        a.dL_dsh_rest = (split && !factors) ? dL_dsh_rest.data_ptr<float>() : nullptr;
        a.raw_params = raw_params;
        a.dL_dts = dL_dts.data_ptr<float>(); a.dL_dscale = dL_dscales.data_ptr<float>();
        a.dL_dscale_t = dL_dscales_t.data_ptr<float>(); a.dL_drot = dL_drotations.data_ptr<float>();
        a.dL_drot_r = dL_drotations_r.data_ptr<float>();
        check(fdgs_backward_bg(&a, fptr(bgi_c), want_dbg ? dL_dbg_image.data_ptr<float>() : nullptr, (void*)stream),
              "backward");
    }
    return BackwardOut{dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dflows, dL_dts,
                       dL_dscales, dL_dscales_t, dL_drotations, dL_drotations_r, sh_factors, dL_dsh_rest, dL_dbg_image};
}

#define FDGS_BWD_PARAMS                                                                                                \
    const torch::Tensor &background, const torch::Tensor &means3D, const torch::Tensor &out_means3D,                  \
        const torch::Tensor &radii, const torch::Tensor &colors, const torch::Tensor &flows_2d,                        \
        const torch::Tensor &opacities, const torch::Tensor &ts, const torch::Tensor &scales,                          \
        const torch::Tensor &scales_t, const torch::Tensor &rotations, const torch::Tensor &rotations_r,               \
        const float scale_modifier, const torch::Tensor &cov3D_precomp, const float prefilter_var,                     \
        const torch::Tensor &viewmatrix, const torch::Tensor &projmatrix, const float tan_fovx, const float tan_fovy,  \
        const torch::Tensor &dL_dout_color, const torch::Tensor &dL_dout_depth, const torch::Tensor &dL_dout_mask,     \
        const torch::Tensor &dL_dout_flow, const torch::Tensor &sh, const int degree, const int degree_t,              \
        const torch::Tensor &campos, const float timestamp, const float time_duration, const bool rot_4d,              \
        const int gaussian_dim, const bool force_sh_3d, const torch::Tensor &geomBuffer, const int R,                  \
        const torch::Tensor &binningBuffer, const torch::Tensor &imageBuffer, const bool debug
#define FDGS_BWD_ARGS                                                                                                  \
    background, means3D, out_means3D, radii, colors, flows_2d, opacities, ts, scales, scales_t, rotations, rotations_r, \
        scale_modifier, cov3D_precomp, prefilter_var, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color,       \
        dL_dout_depth, dL_dout_mask, dL_dout_flow, sh, degree, degree_t, campos, timestamp, time_duration, rot_4d,     \
        gaussian_dim, force_sh_3d, geomBuffer, R, binningBuffer, imageBuffer, debug

// the reference's entry point: 37 positional arguments, 12 gradients (rasterize_points.h:51-89)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor,
           torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansBackwardCUDA(FDGS_BWD_PARAMS) {
    BackwardOut o = backward_impl(torch::Tensor(), false, false, torch::Tensor(), false, FDGS_BWD_ARGS);
    return std::make_tuple(o.dL_dmeans2D, o.dL_dcolors, o.dL_dopacity, o.dL_dmeans3D, o.dL_dcov3D, o.dL_dsh, o.dL_dflows,
                           o.dL_dts, o.dL_dscales, o.dL_dscales_t, o.dL_drotations, o.dL_drotations_r);
}

// view-parallel variant: same arguments; dL_dsh comes back EMPTY and a 13th tensor holds the [P,3] colour factors
std::vector<torch::Tensor> RasterizeGaussiansBackwardFactors(FDGS_BWD_PARAMS) {
    BackwardOut o = backward_impl(torch::Tensor(), false, true, torch::Tensor(), false, FDGS_BWD_ARGS);
    return {o.dL_dmeans2D, o.dL_dcolors, o.dL_dopacity, o.dL_dmeans3D, o.dL_dcov3D, o.dL_dsh, o.dL_dflows,
            o.dL_dts, o.dL_dscales, o.dL_dscales_t, o.dL_drotations, o.dL_drotations_r, o.sh_factors};
}

// per-pixel background image (include/fdgs.h: fdgs_backward_bg): the 37 arguments + the forward's bg_image (empty =
// none), the view-parallel switch of rasterize_gaussians_backward_factors and whether dL/dbg_image is wanted.  Returns
// the 12 gradients, the [P,3] colour factors (sh_factor_mode, else empty) and dL_dbg_image [3,H,W] (else empty).
std::vector<torch::Tensor> RasterizeGaussiansBackwardBg(FDGS_BWD_PARAMS, const torch::Tensor& bg_image, const bool sh_factor_mode,
                                                        const bool want_dbg) {
    BackwardOut o = backward_impl(bg_image, want_dbg, sh_factor_mode, torch::Tensor(), false, FDGS_BWD_ARGS);
    return {o.dL_dmeans2D, o.dL_dcolors, o.dL_dopacity, o.dL_dmeans3D, o.dL_dcov3D, o.dL_dsh, o.dL_dflows, o.dL_dts,
            o.dL_dscales, o.dL_dscales_t, o.dL_drotations, o.dL_drotations_r, o.sh_factors, o.dL_dbg_image};
}

// raw-parameter entry (see RasterizeGaussiansRaw): 14 tensors -- the 12 gradients (w.r.t. the RAW parameters when
// raw_params; dL_dsh is [P,1,3] when sh_rest is given), the [P,3] colour factors (sh_factor_mode, else empty) and
// dL_dsh_rest [P,M-1,3] (split rows, else empty)
std::vector<torch::Tensor> RasterizeGaussiansBackwardRaw(FDGS_BWD_PARAMS, const torch::Tensor& sh_rest, const bool raw_params,
                                                         const bool sh_factor_mode) {
    BackwardOut o = backward_impl(torch::Tensor(), false, sh_factor_mode, sh_rest, raw_params, FDGS_BWD_ARGS);
    return {o.dL_dmeans2D, o.dL_dcolors, o.dL_dopacity, o.dL_dmeans3D, o.dL_dcov3D, o.dL_dsh, o.dL_dflows,
            o.dL_dts, o.dL_dscales, o.dL_dscales_t, o.dL_drotations, o.dL_drotations_r, o.sh_factors, o.dL_dsh_rest};
}

// the raw entry's 40 arguments + bg_image and want_dbg: its 14 tensors, then dL_dbg_image [3,H,W] (else empty)
std::vector<torch::Tensor> RasterizeGaussiansBackwardRawBg(FDGS_BWD_PARAMS, const torch::Tensor& sh_rest, const bool raw_params,
                                                           const bool sh_factor_mode, const torch::Tensor& bg_image,
                                                           const bool want_dbg) {
    BackwardOut o = backward_impl(bg_image, want_dbg, sh_factor_mode, sh_rest, raw_params, FDGS_BWD_ARGS);
    return {o.dL_dmeans2D, o.dL_dcolors, o.dL_dopacity, o.dL_dmeans3D, o.dL_dcov3D, o.dL_dsh, o.dL_dflows, o.dL_dts,
            o.dL_dscales, o.dL_dscales_t, o.dL_drotations, o.dL_drotations_r, o.sh_factors, o.dL_dsh_rest, o.dL_dbg_image};
}

// ---- environment-map sky (include/fdgs.h: fdgs_sky_forward / fdgs_sky_backward) -----------------------------------
static fdgs_sky_args sky_args(const torch::Tensor& env_map, const torch::Tensor& c2w, const torch::Tensor& campos,
                              const double fl_x, const double fl_y, const double cx, const double cy, const double radius,
                              const int64_t H, const int64_t W) {
    TORCH_CHECK(env_map.is_cuda() && env_map.scalar_type() == torch::kFloat32 && env_map.is_contiguous() && env_map.dim() == 3 &&
                env_map.size(0) == 3, "fdgs: env_map must be a contiguous float32 CUDA tensor [3,Hm,Wm]");
    TORCH_CHECK(c2w.is_cuda() && c2w.scalar_type() == torch::kFloat32 && c2w.is_contiguous() && c2w.numel() == 16 &&
                campos.is_cuda() && campos.scalar_type() == torch::kFloat32 && campos.is_contiguous() && campos.numel() == 3,
                "fdgs: c2w [4,4] / campos [3] must be contiguous float32 CUDA tensors");
    TORCH_CHECK(c2w.device() == env_map.device() && campos.device() == env_map.device(), "fdgs: sky inputs on different devices");
    fdgs_sky_args a;
    memset(&a, 0, sizeof(a));
    a.env_map = env_map.data_ptr<float>(); a.env_height = (int)env_map.size(1); a.env_width = (int)env_map.size(2);
    a.c2w = c2w.data_ptr<float>(); a.campos = campos.data_ptr<float>();
    a.fl_x = (float)fl_x; a.fl_y = (float)fl_y; a.cx = (float)cx; a.cy = (float)cy; a.radius = (float)radius;
    a.width = (int)W; a.height = (int)H;
    return a;
}

// (sky [3,H,W], miss flag int32 [1]: 1 if a ray missed the sphere)
std::tuple<torch::Tensor, torch::Tensor> SkyForward(const torch::Tensor& env_map, const torch::Tensor& c2w, const torch::Tensor& campos,
                                                    const double fl_x, const double fl_y, const double cx, const double cy,
                                                    const double radius, const int64_t H, const int64_t W) {
    const fdgs_sky_args a = sky_args(env_map, c2w, campos, fl_x, fl_y, cx, cy, radius, H, W);
    const c10::cuda::CUDAGuard guard(env_map.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    torch::Tensor sky = torch::empty({3, H, W}, env_map.options());
    torch::Tensor miss = torch::zeros({1}, env_map.options().dtype(torch::kInt32));
    check(fdgs_sky_forward(&a, sky.data_ptr<float>(), miss.data_ptr<int>(), (void*)stream), "sky_forward");
    return std::make_tuple(sky, miss);
}

// dL/d env_map [3,Hm,Wm] of dL_dsky [3,H,W]
torch::Tensor SkyBackward(const torch::Tensor& env_map, const torch::Tensor& c2w, const torch::Tensor& campos, const double fl_x,
                          const double fl_y, const double cx, const double cy, const double radius,
                          const torch::Tensor& dL_dsky) {
    TORCH_CHECK(dL_dsky.is_cuda() && dL_dsky.scalar_type() == torch::kFloat32 && dL_dsky.dim() == 3 && dL_dsky.size(0) == 3,
                "fdgs: dL_dsky must be a float32 CUDA tensor [3,H,W]");
    const fdgs_sky_args a = sky_args(env_map, c2w, campos, fl_x, fl_y, cx, cy, radius, dL_dsky.size(1), dL_dsky.size(2));
    const c10::cuda::CUDAGuard guard(env_map.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    const auto g = dL_dsky.contiguous();
    torch::Tensor denv = torch::zeros_like(env_map);
    check(fdgs_sky_backward(&a, g.data_ptr<float>(), denv.data_ptr<float>(), (void*)stream), "sky_backward");
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
    TORCH_CHECK(slot_of.is_cuda() && slot_of.scalar_type() == torch::kInt32 && slot_of.is_contiguous(), "fdgs: slot_of must be int32 CUDA");
    const int P = means3D.size(0);
    for (auto& o : outs)
        TORCH_CHECK(o.is_cuda() && o.scalar_type() == torch::kFloat32 && o.is_contiguous() && o.dim() == 3 && o.size(0) == P &&
                    o.size(2) == 3, "fdgs: outputs must be contiguous float32 [P, m, 3] CUDA tensors");
    const c10::cuda::CUDAGuard guard(means3D.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    const auto m_c = contig(means3D), ts_c = contig(ts), sc_c = contig(scales), sct_c = contig(scales_t),
               rot_c = contig(rotations), rotr_c = contig(rotations_r), tb_c = contig(table);
    fdgs_sh_sum_args a;
    memset(&a, 0, sizeof(a));
    a.P = P; a.V = (int)V; a.K = (int)K; a.table = fptr(tb_c); a.view_stride = view_stride; a.meta_off = meta_off;
    TORCH_CHECK(union_idx.is_cuda() && union_idx.scalar_type() == torch::kInt64 && union_idx.is_contiguous() &&
                union_idx.numel() == K, "fdgs: union_idx must be int64 CUDA [K]");
    torch::Tensor dirs = torch::empty({std::max<int64_t>(V * K * 8, 1)}, means3D.options().dtype(torch::kFloat32));
    a.union_idx = reinterpret_cast<const long long*>(union_idx.data_ptr<int64_t>());
    a.dir_scratch = dirs.data_ptr<float>();
    a.slot_of = slot_of.data_ptr<int>(); a.means3D = fptr(m_c); a.ts = fptr(ts_c); a.scales = fptr(sc_c);
    a.scales_t = fptr(sct_c); a.rotations = fptr(rot_c); a.rotations_r = fptr(rotr_c);
    a.scale_modifier = (float)scale_modifier; a.time_duration = (float)time_duration; a.rot_4d = rot_4d;
    a.gaussian_dim = (int)gaussian_dim; a.force_sh_3d = force_sh_3d; a.D = (int)D; a.D_t = (int)D_t;
    a.m0 = (int)outs[0].size(1);
    a.M = a.m0 + (outs.size() == 2 ? (int)outs[1].size(1) : 0);
    a.out0 = outs[0].data_ptr<float>();
    a.out1 = outs.size() == 2 ? outs[1].data_ptr<float>() : nullptr;
    a.accumulate = accumulate;
    if (V > 0) TORCH_CHECK(tb_c.numel() >= V * view_stride, "fdgs: factor table too small");
    check(fdgs_sh_outer_sum(&a, (void*)stream), "sh_outer_sum");
}

// (slot_of int32 [P], idx int64 [K]) from the radii, their inclusive prefix sum cs and K = cs[-1] (known to the host)
std::tuple<torch::Tensor, torch::Tensor> UnionMaps(const torch::Tensor& radii, const torch::Tensor& cs, const int64_t K) {
    TORCH_CHECK(radii.is_cuda() && radii.scalar_type() == torch::kInt32 && radii.is_contiguous() && cs.is_cuda() &&
                cs.scalar_type() == torch::kInt32 && cs.is_contiguous() && cs.numel() == radii.numel(),
                "fdgs: radii / cs must be contiguous int32 CUDA tensors of equal length");
    const c10::cuda::CUDAGuard guard(radii.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    torch::Tensor slot_of = torch::empty_like(radii);
    torch::Tensor idx = torch::empty({K}, radii.options().dtype(torch::kInt64));
    check(fdgs_union_maps(radii.numel(), radii.data_ptr<int>(), cs.data_ptr<int>(), slot_of.data_ptr<int>(),
                          reinterpret_cast<long long*>(idx.data_ptr<int64_t>()), (void*)stream),
          "union_maps");
    return std::make_tuple(slot_of, idx);
}

// per-view densification statistics, one pass (include/fdgs.h: fdgs_view_stats)
void ViewStats(const torch::Tensor& viewspace_grad, const torch::Tensor& radii, torch::Tensor& grad_norm_sum,
               torch::Tensor& visibility_count, torch::Tensor& max_radii) {
    const long long P = radii.numel();
    TORCH_CHECK(viewspace_grad.is_cuda() && viewspace_grad.scalar_type() == torch::kFloat32 && viewspace_grad.is_contiguous() &&
                viewspace_grad.dim() == 2 && viewspace_grad.size(0) == P && viewspace_grad.size(1) >= 2, "fdgs: viewspace_grad must be [P,>=2] float32 CUDA");
    TORCH_CHECK(radii.is_cuda() && radii.scalar_type() == torch::kInt32 && radii.is_contiguous(), "fdgs: radii must be int32 CUDA");
    TORCH_CHECK(grad_norm_sum.is_contiguous() && grad_norm_sum.numel() == P && grad_norm_sum.scalar_type() == torch::kFloat32 &&
                visibility_count.is_contiguous() && visibility_count.numel() == P && visibility_count.scalar_type() == torch::kFloat32 &&
                max_radii.is_contiguous() && max_radii.numel() == P && max_radii.scalar_type() == torch::kInt32, "fdgs: statistics tensors");
    const c10::cuda::CUDAGuard guard(radii.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check(fdgs_view_stats(P, viewspace_grad.data_ptr<float>(), (int)viewspace_grad.size(1), radii.data_ptr<int>(),
                          grad_norm_sum.data_ptr<float>(), visibility_count.data_ptr<float>(), max_radii.data_ptr<int>(), (void*)stream),
          "view_stats");
}

// 1-element int32 tensor, non-zero if a row of `tensors` outside radii > 0 is not all-zero (sparse-exchange guard)
torch::Tensor CheckRowsZero(std::vector<torch::Tensor> tensors, const torch::Tensor& radii) {
    TORCH_CHECK((int)tensors.size() <= FDGS_MAX_PACK, "fdgs: too many tensors");
    TORCH_CHECK(radii.is_cuda() && radii.scalar_type() == torch::kInt32 && radii.is_contiguous(), "fdgs: radii must be int32 CUDA");
    torch::Tensor flag = torch::zeros({1}, radii.options());
    const long long P = radii.numel();
    if (tensors.empty() || P == 0) return flag;
    std::vector<const float*> ptr;
    std::vector<int> widths;
    for (const auto& t : tensors) {
        TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kFloat32 && t.is_contiguous() && t.size(0) == P,
                    "fdgs: gradient tensors must be contiguous float32 CUDA tensors with P rows");
        ptr.push_back(t.data_ptr<float>());
        widths.push_back((int)(t.numel() / P));
    }
    const c10::cuda::CUDAGuard guard(radii.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check(fdgs_check_rows_zero((int)ptr.size(), ptr.data(), widths.data(), P, radii.data_ptr<int>(), flag.data_ptr<int>(),
                               (void*)stream),
          "check_rows_zero");
    return flag;
}

torch::Tensor markVisible(torch::Tensor& means3D, torch::Tensor& viewmatrix, torch::Tensor& projmatrix) {
    const int P = means3D.size(0);
    torch::Tensor present = torch::full({P}, false, means3D.options().dtype(at::kBool));
    if (P != 0) {
        const c10::cuda::CUDAGuard guard(means3D.device());
        cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
        const auto m = means3D.contiguous(), v = viewmatrix.contiguous(), pr = projmatrix.contiguous();
        check(fdgs_mark_visible(P, m.data_ptr<float>(), v.data_ptr<float>(), pr.data_ptr<float>(),
                                reinterpret_cast<unsigned char*>(present.data_ptr<bool>()), (void*)stream),
              "mark_visible");
    }
    return present;
}

// Test hooks: private forward state as plain tensors (parity tests compare them with the oracle).
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
DebugExportGeom(const torch::Tensor& geomBuffer, const int P) {
    const c10::cuda::CUDAGuard guard(geomBuffer.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    auto f = geomBuffer.options().dtype(torch::kFloat32);
    torch::Tensor depths = torch::zeros({P}, f), means2D = torch::zeros({P, 2}, f), conic = torch::zeros({P, 4}, f),
                  rgb = torch::zeros({P, 3}, f);
    torch::Tensor clamped = torch::zeros({P}, geomBuffer.options().dtype(torch::kByte));
    torch::Tensor tiles = torch::zeros({P}, geomBuffer.options().dtype(torch::kInt32));
    if (P > 0)
        check(fdgs_debug_export_geom(reinterpret_cast<const char*>(geomBuffer.data_ptr()), P, depths.data_ptr<float>(),
                                     means2D.data_ptr<float>(), conic.data_ptr<float>(), rgb.data_ptr<float>(),
                                     clamped.data_ptr<uint8_t>(), reinterpret_cast<unsigned int*>(tiles.data_ptr<int>()),
                                     (void*)stream),
              "debug_export_geom");
    return std::make_tuple(depths, means2D, conic, rgb, clamped, tiles);
}

std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> DebugExportBinning(const torch::Tensor& binningBuffer,
                                                                           const torch::Tensor& imgBuffer, const int R,
                                                                           const int W, const int H) {
    const c10::cuda::CUDAGuard guard(imgBuffer.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    auto i32 = imgBuffer.options().dtype(torch::kInt32);
    const int tiles = ((W + 15) / 16) * ((H + 15) / 16);
    torch::Tensor point_list = torch::zeros({R}, i32), ranges = torch::zeros({tiles, 2}, i32),
                  n_contrib = torch::zeros({H, W}, i32);
    check(fdgs_debug_export_binning(R > 0 ? reinterpret_cast<const char*>(binningBuffer.data_ptr()) : nullptr,
                                    reinterpret_cast<const char*>(imgBuffer.data_ptr()), R, W, H,
                                    reinterpret_cast<unsigned int*>(point_list.data_ptr<int>()),
                                    reinterpret_cast<unsigned int*>(ranges.data_ptr<int>()),
                                    reinterpret_cast<unsigned int*>(n_contrib.data_ptr<int>()), (void*)stream),
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
        TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kFloat32 && t.is_contiguous() && t.dim() >= 1,
                    "fdgs: gradient tensors must be contiguous float32 CUDA tensors");
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
    TORCH_CHECK(idx.is_cuda() && idx.scalar_type() == torch::kInt64 && idx.is_contiguous(), "fdgs: idx must be int64 CUDA");
    const long long K = idx.numel();
    std::vector<int> widths;
    long long total = 0;
    std::vector<long long> off = block_offsets(tensors, K, widths, total);
    torch::Tensor flat = torch::empty({total}, idx.options().dtype(torch::kFloat32));
    if (K == 0 || tensors.empty()) return flat;
    const c10::cuda::CUDAGuard guard(idx.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    std::vector<const float*> ptr;
    for (const auto& t : tensors) ptr.push_back(t.data_ptr<float>());
    check(fdgs_pack_rows((int)tensors.size(), ptr.data(), widths.data(), off.data(), reinterpret_cast<const long long*>(idx.data_ptr<int64_t>()), K,
                         flat.data_ptr<float>(), (void*)stream),
          "pack_rows");
    return flat;
}

void UnpackRows(const torch::Tensor& flat, std::vector<torch::Tensor> tensors, const torch::Tensor& idx) {
    TORCH_CHECK((int)tensors.size() <= FDGS_MAX_PACK, "fdgs: too many tensors");
    const long long K = idx.numel();
    std::vector<int> widths;
    long long total = 0;
    std::vector<long long> off = block_offsets(tensors, K, widths, total);
    TORCH_CHECK(flat.numel() == total && flat.is_contiguous() && flat.scalar_type() == torch::kFloat32, "fdgs: flat buffer mismatch");
    if (K == 0 || tensors.empty()) return;
    const c10::cuda::CUDAGuard guard(idx.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    std::vector<float*> ptr;
    for (auto& t : tensors) ptr.push_back(t.data_ptr<float>());
    check(fdgs_unpack_rows((int)tensors.size(), ptr.data(), widths.data(), off.data(), reinterpret_cast<const long long*>(idx.data_ptr<int64_t>()), K,
                           flat.data_ptr<float>(), (void*)stream),
          "unpack_rows");
}

// ---- fused L1 + SSIM (include/fdgs.h: fdgs_l1_ssim_forward / _backward) ------------------------------------------
// returns (sums double[2] = {sum |x - y|, sum SSIM}, maps float[3,C,H,W])
std::tuple<torch::Tensor, torch::Tensor> L1SsimForward(const torch::Tensor& x, const torch::Tensor& y) {
    TORCH_CHECK(x.is_cuda() && y.is_cuda() && x.scalar_type() == torch::kFloat32 && y.scalar_type() == torch::kFloat32,
                "fdgs: images must be float32 CUDA tensors");
    TORCH_CHECK(x.dim() == 3 && x.sizes() == y.sizes(), "fdgs: images must be [C,H,W] of equal shape");
    const c10::cuda::CUDAGuard guard(x.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    const auto xc = x.contiguous(), yc = y.contiguous();
    const int C = x.size(0), H = x.size(1), W = x.size(2);
    torch::Tensor sums = torch::empty({2}, x.options().dtype(torch::kFloat64));
    torch::Tensor maps = torch::empty({3, C, H, W}, x.options());
    check(fdgs_l1_ssim_forward(xc.data_ptr<float>(), yc.data_ptr<float>(), C, H, W, maps.data_ptr<float>(),
                               sums.data_ptr<double>(), (void*)stream),
          "l1_ssim_forward");
    return std::make_tuple(sums, maps);
}

torch::Tensor L1SsimBackward(const torch::Tensor& x, const torch::Tensor& y, const torch::Tensor& maps,
                             const torch::Tensor& grad_scale, const double lambda_dssim) {
    const c10::cuda::CUDAGuard guard(x.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    const auto xc = x.contiguous(), yc = y.contiguous(), gs = grad_scale.to(torch::kFloat32).contiguous();
    const int C = x.size(0), H = x.size(1), W = x.size(2);
    torch::Tensor dx = torch::empty({C, H, W}, x.options());
    check(fdgs_l1_ssim_backward(xc.data_ptr<float>(), yc.data_ptr<float>(), C, H, W, maps.data_ptr<float>(),
                                gs.numel() ? gs.data_ptr<float>() : nullptr, (float)lambda_dssim, dx.data_ptr<float>(),
                                (void*)stream),
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
        for (const torch::Tensor* t : {&params[i], &grads[i], &exp_avg[i], &exp_avg_sq[i]})
            TORCH_CHECK(t->is_cuda() && t->scalar_type() == torch::kFloat32 && t->is_contiguous() && t->size(0) == P &&
                        t->numel() == params[i].numel(), "fdgs: adam tensors must be contiguous float32 CUDA [P, ...]");
        p.push_back(params[i].data_ptr<float>()); g.push_back(grads[i].data_ptr<float>());
        m.push_back(exp_avg[i].data_ptr<float>()); v.push_back(exp_avg_sq[i].data_ptr<float>());
        widths.push_back(P > 0 ? (int)(params[i].numel() / P) : 1);
        lr.push_back((float)lrs[i]);
    }
    if (sparse) {
        TORCH_CHECK(rows.is_cuda() && rows.scalar_type() == torch::kInt64 && rows.is_contiguous(), "fdgs: rows must be int64 CUDA");
        if (rows.numel() == 0) return;
    }
    const c10::cuda::CUDAGuard guard(params[0].device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check(fdgs_adam_step((int)n, p.data(), g.data(), m.data(), v.data(), widths.data(), lr.data(), P,
                         sparse ? reinterpret_cast<const long long*>(rows.data_ptr<int64_t>()) : nullptr, sparse ? rows.numel() : 0,
                         step, beta1, beta2, eps, zero_grad, (void*)stream),
          "adam_step");
}

// ---- densification (include/fdgs.h: fdgs_densify_*, fdgs_reset_opacity) --------------------------------------------
// An undefined or empty tensor is "not provided" (NULL; the C-ABI rejects a NULL it needs).  dtype, layout and shape are checked before the device, so a
// malformed argument is rejected before any GPU work.
static float* rows_ptr(const torch::Tensor& t, long long P, long long width, const char* name) {
    if (!t.defined() || t.numel() == 0) return nullptr;
    TORCH_CHECK(t.scalar_type() == torch::kFloat32, "fdgs: ", name, " must be float32");
    TORCH_CHECK(t.is_contiguous(), "fdgs: ", name, " must be contiguous");
    TORCH_CHECK(t.dim() >= 1 && t.size(0) == P && (width < 0 || t.numel() == P * width), "fdgs: ", name, " has the wrong shape");
    return t.data_ptr<float>();
}

// after every tensor of a call passed rows_ptr: all of them on the CUDA device of the first
static void same_cuda_device(std::initializer_list<const torch::Tensor*> ts) {
    const torch::Tensor* first = nullptr;
    for (const torch::Tensor* t : ts) {
        if (!t->defined() || t->numel() == 0) continue;
        TORCH_CHECK(t->is_cuda(), "fdgs: densification tensors must be CUDA tensors");
        if (!first) first = t;
        TORCH_CHECK(t->device() == first->device(), "fdgs: densification tensors on different devices");
    }
}

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
    a.xyz = rows_ptr(geo[0], P, 3, "xyz");
    a.t = rows_ptr(geo[1], P, 1, "t");
    a.scaling = rows_ptr(geo[2], P, 3, "scaling");
    a.scaling_t = rows_ptr(geo[3], P, 1, "scaling_t");
    a.rotation = rows_ptr(geo[4], P, 4, "rotation");
    a.rotation_r = rows_ptr(geo[5], P, 4, "rotation_r");
    a.opacity = rows_ptr(geo[6], P, 1, "opacity");
    a.xyz_gradient_accum = rows_ptr(stats[0], P, 1, "xyz_gradient_accum");
    a.denom = rows_ptr(stats[1], P, 1, "denom");
    a.max_radii2D = rows_ptr(stats[2], P, 1, "max_radii2D");
    same_cuda_device({&geo[0], &geo[1], &geo[2], &geo[3], &geo[4], &geo[5], &geo[6], &stats[0], &stats[1], &stats[2]});
    return a;
}

std::tuple<torch::Tensor, torch::Tensor> DensifyPlan(const std::vector<torch::Tensor>& geo, const std::vector<torch::Tensor>& stats,
                                                     const std::vector<double>& thr, const std::vector<int64_t>& flags) {
    fdgs_densify_args a = densify_args(geo, stats, thr, flags);
    TORCH_CHECK(geo[2].defined() && geo[2].is_cuda(), "fdgs: scaling must be a CUDA tensor");
    const c10::cuda::CUDAGuard guard(geo[2].device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    auto opts = geo[2].options();
    torch::Tensor scratch = torch::empty({(int64_t)fdgs_densify_scratch_bytes(a.P) + 16}, opts.dtype(torch::kByte));
    torch::Tensor totals = torch::empty({4}, opts.dtype(torch::kInt32));
    check(fdgs_densify_plan(&a, reinterpret_cast<char*>(scratch.data_ptr()), totals.data_ptr<int>(), (void*)stream), "densify_plan");
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
        a.src[i] = rows_ptr(srcs[i], a.P, w, "source row tensor");
        a.dst[i] = rows_ptr(dsts[i], P_new, w, "destination row tensor");
        if (a.P == 0 || P_new == 0) { a.num_tensors = 0; break; }     // nothing to copy from or to
        TORCH_CHECK(a.src[i] && a.dst[i], "fdgs: densify tensor table entry missing");
        a.kind[i] = (int)kinds[i];
        a.width[i] = (int)w;
    }
    const long long SN = totals[2] * (long long)a.N;
    a.samples = rows_ptr(samples, SN, a.rot_4d ? 4 : 3, "samples");
    a.samples_t = rows_ptr(samples_t, SN, 1, "samples_t");
    for (size_t i = 0; i < n; ++i) same_cuda_device({&geo[2], &srcs[i], &dsts[i]});
    same_cuda_device({&geo[2], &samples, &samples_t});
    TORCH_CHECK(scratch.is_cuda() && scratch.scalar_type() == torch::kByte &&
                scratch.numel() >= (int64_t)fdgs_densify_scratch_bytes(a.P), "fdgs: densify scratch of the plan required");
    int tot[4];
    for (int i = 0; i < 4; ++i) tot[i] = (int)totals[i];
    const c10::cuda::CUDAGuard guard(scratch.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check(fdgs_densify_apply(&a, reinterpret_cast<const char*>(scratch.data_ptr()), tot, (void*)stream), "densify_apply");
}

void ResetOpacity(torch::Tensor& opacity, torch::Tensor& exp_avg, torch::Tensor& exp_avg_sq) {
    const long long P = opacity.size(0);
    float* o = rows_ptr(opacity, P, 1, "opacity");
    float* m = rows_ptr(exp_avg, P, 1, "exp_avg");
    float* v = rows_ptr(exp_avg_sq, P, 1, "exp_avg_sq");
    same_cuda_device({&opacity, &exp_avg, &exp_avg_sq});
    if (P == 0) return;
    const c10::cuda::CUDAGuard guard(opacity.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check(fdgs_reset_opacity(P, o, m, v, (void*)stream), "reset_opacity");
}

// batch_size 1: point_grad = viewspace_points.grad [P, >= 2], visibility_count empty; batch_size > 1: point_grad =
// the summed norms [P] and visibility_count [P] (fdgs.dist.ViewBatchStats).  t_grad / t_gradient_accum empty for 3D.
void DensifyStats(int64_t batch_size, const torch::Tensor& point_grad, const torch::Tensor& visibility_count,
                  const torch::Tensor& radii, const torch::Tensor& t_grad, torch::Tensor& xyz_gradient_accum, torch::Tensor& denom,
                  torch::Tensor& t_gradient_accum, torch::Tensor& max_radii2D) {
    const long long P = xyz_gradient_accum.size(0);
    float* acc = rows_ptr(xyz_gradient_accum, P, 1, "xyz_gradient_accum");
    float* den = rows_ptr(denom, P, 1, "denom");
    float* tacc = rows_ptr(t_gradient_accum, P, 1, "t_gradient_accum");
    float* mr = rows_ptr(max_radii2D, P, 1, "max_radii2D");
    const float* tg = rows_ptr(t_grad, P, 1, "t_grad");
    const float* vis = rows_ptr(visibility_count, P, 1, "visibility_count");
    const float* pg = rows_ptr(point_grad, P, batch_size == 1 ? -1 : 1, "point_grad");
    TORCH_CHECK(point_grad.defined() && (batch_size > 1 || point_grad.dim() == 2), "fdgs: point_grad must be [P, >= 2] for one view");
    TORCH_CHECK(radii.defined() && radii.scalar_type() == torch::kInt32 && radii.is_contiguous() && radii.numel() == P,
                "fdgs: radii must be contiguous int32 [P]");
    same_cuda_device({&xyz_gradient_accum, &denom, &t_gradient_accum, &max_radii2D, &t_grad, &visibility_count, &point_grad, &radii});
    const int stride = batch_size == 1 ? (int)(point_grad.dim() == 2 ? point_grad.size(1) : 0) : 1;
    if (P == 0) return;
    const c10::cuda::CUDAGuard guard(xyz_gradient_accum.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    check(fdgs_densify_stats(P, (int)batch_size, pg, stride, vis, radii.data_ptr<int>(), tg, acc, den, tacc, mr, (void*)stream),
          "densify_stats");
}

// ---- k nearest neighbours (include/fdgs.h: fdgs_knn) ---------------------------------------------------------------
std::tuple<torch::Tensor, torch::Tensor> Knn(const torch::Tensor& xyz, const int64_t k, const bool brute_force) {
    TORCH_CHECK(xyz.is_cuda() && xyz.scalar_type() == torch::kFloat32 && xyz.dim() == 2 && xyz.size(1) == 3,
                "fdgs: xyz must be a float32 CUDA tensor [n,3]");
    const c10::cuda::CUDAGuard guard(xyz.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    const auto x = xyz.contiguous();
    const int n = x.size(0);
    torch::Tensor idx = torch::empty({n, k}, x.options().dtype(torch::kInt32));
    torch::Tensor d2 = torch::empty({n, k}, x.options());
    torch::Tensor scratch = torch::empty({(int64_t)(brute_force ? 16 : fdgs_knn_scratch_bytes(n))}, x.options().dtype(torch::kByte));
    check(fdgs_knn(n, (int)k, x.data_ptr<float>(), reinterpret_cast<char*>(scratch.data_ptr()), idx.data_ptr<int>(),
                   d2.data_ptr<float>(), brute_force, (void*)stream),
          "knn");
    return std::make_tuple(idx, d2);
}

// ---- rigidity and motion regularisers (include/fdgs.h: fdgs_rigid_*) -----------------------------------------------
// Every tensor is checked for dtype, layout, shape and device before the device is touched.  An undefined or empty
// optional tensor is "not provided".
static const void* rigid_ptr(const torch::Tensor& t, torch::ScalarType dtype, int64_t rows, int64_t numel, const char* name) {
    TORCH_CHECK(t.defined(), "fdgs: ", name, " is required");
    TORCH_CHECK(t.scalar_type() == dtype, "fdgs: ", name, " must be ", c10::toString(dtype));
    TORCH_CHECK(t.is_contiguous(), "fdgs: ", name, " must be contiguous");
    TORCH_CHECK(t.dim() >= 1 && t.size(0) == rows && t.numel() == numel, "fdgs: ", name, " has the wrong shape");
    return t.data_ptr();
}

static void rigid_same_device(std::initializer_list<const torch::Tensor*> ts) {
    const torch::Tensor* first = nullptr;
    for (const torch::Tensor* t : ts) {
        if (!t->defined() || t->numel() == 0) continue;
        TORCH_CHECK(t->is_cuda(), "fdgs: regulariser tensors must be CUDA tensors");
        if (!first) first = t;
        TORCH_CHECK(t->device() == first->device(), "fdgs: regulariser tensors on different devices");
    }
}

// params = [t [n,1], scaling [n,3], scaling_t [n,1], rotation [n,4], rotation_r [n,4]] (the raw parameters)
static fdgs_rigid_args rigid_args(const std::vector<torch::Tensor>& params, int64_t k) {
    TORCH_CHECK(params.size() == 5, "fdgs: five parameter tensors (t, scaling, scaling_t, rotation, rotation_r)");
    TORCH_CHECK(params[1].defined() && params[1].dim() == 2, "fdgs: scaling must be [n,3]");
    const int64_t n = params[1].size(0);
    fdgs_rigid_args a;
    memset(&a, 0, sizeof(a));
    a.n = (int)n;
    a.k = (int)k;
    a.t = static_cast<const float*>(rigid_ptr(params[0], torch::kFloat32, n, n, "t"));
    a.scaling = static_cast<const float*>(rigid_ptr(params[1], torch::kFloat32, n, 3 * n, "scaling"));
    a.scaling_t = static_cast<const float*>(rigid_ptr(params[2], torch::kFloat32, n, n, "scaling_t"));
    a.rotation = static_cast<const float*>(rigid_ptr(params[3], torch::kFloat32, n, 4 * n, "rotation"));
    a.rotation_r = static_cast<const float*>(rigid_ptr(params[4], torch::kFloat32, n, 4 * n, "rotation_r"));
    return a;
}

static void rigid_list(fdgs_rigid_args& a, const torch::Tensor& idx, const torch::Tensor& weight) {
    const int64_t n = a.n, k = a.k;
    a.idx = static_cast<const int*>(rigid_ptr(idx, torch::kInt32, n, n * k, "idx"));
    a.weight = static_cast<const float*>(rigid_ptr(weight, torch::kFloat32, n, n * k, "weight"));
}

static const float* rigid_scalar(const torch::Tensor& g, const char* name) {
    if (!g.defined() || g.numel() == 0) return nullptr;
    TORCH_CHECK(g.scalar_type() == torch::kFloat32 && g.numel() == 1, "fdgs: ", name, " must be one float32 element");
    return g.data_ptr<float>();
}

// (weight, in_offsets, in_edges) of fdgs_knn's (idx, dist2)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> RigidNeighbours(const torch::Tensor& idx, const torch::Tensor& dist2) {
    TORCH_CHECK(idx.defined() && idx.dim() == 2, "fdgs: idx must be [n,k]");
    const int64_t n = idx.size(0), k = idx.size(1);
    TORCH_CHECK(n > 0 && k >= 1 && k <= 32, "fdgs: bad n / k (n > 0, 1 <= k <= 32)");
    const int* ip = static_cast<const int*>(rigid_ptr(idx, torch::kInt32, n, n * k, "idx"));
    const float* dp = static_cast<const float*>(rigid_ptr(dist2, torch::kFloat32, n, n * k, "dist2"));
    rigid_same_device({&idx, &dist2});
    const c10::cuda::CUDAGuard guard(idx.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    auto opts = dist2.options();
    torch::Tensor weight = torch::empty({n, k}, opts);
    torch::Tensor in_offsets = torch::empty({n + 1}, opts.dtype(torch::kInt32));
    torch::Tensor in_edges = torch::empty({n * k}, opts.dtype(torch::kInt32));
    torch::Tensor scratch = torch::empty({(int64_t)fdgs_rigid_scratch_bytes((int)n, (int)k) + 256}, opts.dtype(torch::kByte));
    check(fdgs_rigid_neighbours((int)n, (int)k, ip, dp, reinterpret_cast<char*>(scratch.data_ptr()), weight.data_ptr<float>(),
                                in_offsets.data_ptr<int>(), in_edges.data_ptr<int>(), (void*)stream),
          "rigid_neighbours");
    return std::make_tuple(weight, in_offsets, in_edges);
}

// (velocity [n,3], loss_rigid, loss_motion); an unwanted loss comes back as 0
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> RigidForward(const std::vector<torch::Tensor>& params, const int64_t k,
                                                                     const torch::Tensor& idx, const torch::Tensor& weight,
                                                                     const bool want_rigid, const bool want_motion) {
    fdgs_rigid_args a = rigid_args(params, k);
    if (want_rigid) rigid_list(a, idx, weight);
    rigid_same_device({&params[0], &params[1], &params[2], &params[3], &params[4], &idx, &weight});
    TORCH_CHECK(params[1].is_cuda(), "fdgs: regulariser tensors must be CUDA tensors");
    const c10::cuda::CUDAGuard guard(params[1].device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    auto opts = params[1].options();
    torch::Tensor velocity = torch::empty({params[1].size(0), 3}, opts);
    torch::Tensor lr = want_rigid ? torch::empty({}, opts) : torch::zeros({}, opts);
    torch::Tensor lm = want_motion ? torch::empty({}, opts) : torch::zeros({}, opts);
    const size_t sb = fdgs_rigid_scratch_bytes(a.n, a.k);
    torch::Tensor scratch = torch::empty({(int64_t)sb + 256}, opts.dtype(torch::kByte));
    a.velocity = velocity.data_ptr<float>();
    check(fdgs_rigid_forward(&a, reinterpret_cast<char*>(scratch.data_ptr()), want_rigid ? lr.data_ptr<float>() : nullptr,
                             want_motion ? lm.data_ptr<float>() : nullptr, (void*)stream),
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
    a.velocity = static_cast<float*>(const_cast<void*>(rigid_ptr(velocity, torch::kFloat32, n, 3 * n, "velocity")));
    const float* gr = rigid_scalar(grad_rigid, "grad_rigid");
    const float* gm = rigid_scalar(grad_motion, "grad_motion");
    if (gr) {
        rigid_list(a, idx, weight);
        a.in_offsets = static_cast<const int*>(rigid_ptr(in_offsets, torch::kInt32, n + 1, n + 1, "in_offsets"));
        a.in_edges = static_cast<const int*>(rigid_ptr(in_edges, torch::kInt32, n * k, n * k, "in_edges"));
    }
    rigid_same_device({&params[0], &params[1], &params[2], &params[3], &params[4], &velocity, &idx, &weight, &in_offsets, &in_edges,
                       &grad_rigid, &grad_motion});
    TORCH_CHECK(params[1].is_cuda(), "fdgs: regulariser tensors must be CUDA tensors");
    const c10::cuda::CUDAGuard guard(params[1].device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    torch::Tensor ds = torch::empty_like(params[1]), dst = torch::empty_like(params[2]);
    torch::Tensor dr = torch::empty_like(params[3]), drr = torch::empty_like(params[4]);
    check(fdgs_rigid_backward(&a, gr, gm, ds.data_ptr<float>(), dst.data_ptr<float>(), dr.data_ptr<float>(), drr.data_ptr<float>(),
                              (void*)stream),
          "rigid_backward");
    return std::make_tuple(ds, dst, dr, drr);
}

// ---- evaluation metrics (include/fdgs.h: fdgs_image_metrics) ---------------------------------------------------------
// x, y: [B,C,H,W] float32 contiguous CUDA tensors; accum: float64 [5] on the same device, or empty = none.
// Returns out [B,4] float64 (l1, psnr, ssim, msssim per view).  Checks dtype, layout and shape before the device.
torch::Tensor ImageMetrics(const torch::Tensor& x, const torch::Tensor& y, const bool clamp, const torch::Tensor& accum) {
    TORCH_CHECK(x.defined() && y.defined(), "fdgs: image_metrics needs two images");
    TORCH_CHECK(x.scalar_type() == torch::kFloat32 && y.scalar_type() == torch::kFloat32, "fdgs: images must be Float (float32)");
    TORCH_CHECK(x.is_contiguous() && y.is_contiguous(), "fdgs: images must be contiguous");
    TORCH_CHECK(x.dim() == 4 && x.sizes() == y.sizes(), "fdgs: images must be [B,C,H,W] of equal shape");
    const bool has_accum = accum.defined() && accum.numel() > 0;
    if (has_accum) {
        TORCH_CHECK(accum.scalar_type() == torch::kFloat64 && accum.is_contiguous() && accum.numel() == 5,
                    "fdgs: accum must be a contiguous Double (float64) tensor of 5 elements");
    }
    TORCH_CHECK(x.is_cuda() && y.is_cuda() && x.device() == y.device() && (!has_accum || accum.device() == x.device()),
                "fdgs: image_metrics tensors must be CUDA tensors on one device");
    fdgs_metrics_args a;
    memset(&a, 0, sizeof(a));
    a.B = (int)x.size(0); a.C = (int)x.size(1); a.H = (int)x.size(2); a.W = (int)x.size(3);
    TORCH_CHECK(x.size(0) == a.B && x.size(1) == a.C && x.size(2) == a.H && x.size(3) == a.W, "fdgs: image size overflow");
    const size_t sb = fdgs_metrics_scratch_bytes(a.B, a.C, a.H, a.W);
    const c10::cuda::CUDAGuard guard(x.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    torch::Tensor out = torch::empty({x.size(0), 4}, x.options().dtype(torch::kFloat64));
    torch::Tensor scratch = torch::empty({(int64_t)sb}, x.options().dtype(torch::kByte));
    a.x = x.data_ptr<float>();
    a.y = y.data_ptr<float>();
    a.clamp = clamp ? 1 : 0;
    a.out = out.data_ptr<double>();
    a.accum = has_accum ? accum.data_ptr<double>() : nullptr;
    check(fdgs_image_metrics(&a, reinterpret_cast<char*>(scratch.data_ptr()), (void*)stream), "image_metrics");
    return out;
}

std::tuple<torch::Tensor, torch::Tensor, torch::Tensor> DebugActivate(const torch::Tensor& log_s, const torch::Tensor& logit,
                                                                      const torch::Tensor& quat, const int64_t mode) {
    const c10::cuda::CUDAGuard guard(log_s.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream().stream();
    const auto a = log_s.contiguous(), b = logit.contiguous(), q = quat.contiguous();
    const int n = (int)a.numel();
    TORCH_CHECK(b.numel() == n && q.numel() == 4 * (int64_t)n, "fdgs: debug_activate shapes");
    torch::Tensor s = torch::empty_like(a), o = torch::empty_like(b), qo = torch::empty_like(q);
    check(fdgs_debug_activate(n, a.data_ptr<float>(), b.data_ptr<float>(), q.data_ptr<float>(), (int)mode, s.data_ptr<float>(),
                              o.data_ptr<float>(), qo.data_ptr<float>(), (void*)stream),
          "debug_activate");
    return std::make_tuple(s, o, qo);
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.def("debug_activate", &DebugActivate);
    m.def("l1_ssim_forward", &L1SsimForward);
    m.def("l1_ssim_backward", &L1SsimBackward);
    m.def("adam_step", &AdamStep);
    m.def("knn", &Knn);
    m.def("rigid_neighbours", &RigidNeighbours);
    m.def("rigid_forward", &RigidForward);
    m.def("rigid_backward", &RigidBackward);
    m.def("image_metrics", &ImageMetrics);
    m.def("densify_plan", &DensifyPlan);
    m.def("densify_apply", &DensifyApply);
    m.def("reset_opacity", &ResetOpacity);
    m.def("densify_stats", &DensifyStats);
    m.def("pack_rows", &PackRows);
    m.def("unpack_rows", &UnpackRows);
    m.def("rasterize_gaussians", &RasterizeGaussiansCUDA);
    m.def("rasterize_gaussians_backward", &RasterizeGaussiansBackwardCUDA);
    m.def("rasterize_gaussians_backward_factors", &RasterizeGaussiansBackwardFactors);
    m.def("rasterize_gaussians_raw", &RasterizeGaussiansRaw);
    m.def("rasterize_gaussians_backward_raw", &RasterizeGaussiansBackwardRaw);
    m.def("rasterize_gaussians_bg", &RasterizeGaussiansBg);
    m.def("rasterize_gaussians_backward_bg", &RasterizeGaussiansBackwardBg);
    m.def("rasterize_gaussians_raw_bg", &RasterizeGaussiansRawBg);
    m.def("rasterize_gaussians_backward_raw_bg", &RasterizeGaussiansBackwardRawBg);
    m.def("sky_forward", &SkyForward);
    m.def("sky_backward", &SkyBackward);
    m.def("sh_outer_sum", &ShOuterSum);
    m.def("check_rows_zero", &CheckRowsZero);
    m.def("union_maps", &UnionMaps);
    m.def("view_stats", &ViewStats);
    m.def("mark_visible", &markVisible);
    m.def("debug_export_geom", &DebugExportGeom);
    m.def("debug_export_binning", &DebugExportBinning);
    m.def("fdgs_version", []() { return fdgs_version(); });
}
