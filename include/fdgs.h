/*
 * fdgs.h -- C-ABI of the H100-native differentiable 4D Gaussian rasterizer ("fdgs").
 *
 * This is the drop-in boundary of the hot path.  Every entry point replaces one
 * method of the reference's L0 C++ API `CudaRasterizer::Rasterizer`
 * (reference: diff-gaussian-rasterization/cuda_rasterizer/rasterizer.h:20-113):
 *
 *   fdgs_forward       <- Rasterizer::forward      (rasterizer.h:31-65,  rasterizer_impl.cu:199-364)
 *   fdgs_backward      <- Rasterizer::backward     (rasterizer.h:67-112, rasterizer_impl.cu:368-496)
 *   fdgs_mark_visible  <- Rasterizer::markVisible  (rasterizer.h:24-29,  rasterizer_impl.cu:142-154)
 *
 * Differences from the reference interface, all forced by "plain C, no C++ types":
 *   - the three `std::function<char*(size_t)>` scratch allocators become a C
 *     function pointer + opaque context (fdgs_alloc_fn);
 *   - the ~40 positional arguments become two POD structs of raw device
 *     pointers and scalars (field names = the reference's argument names);
 *   - every call takes the CUDA stream to launch on (the reference uses the
 *     legacy default stream implicitly) and returns an int status instead of
 *     throwing; fdgs_last_error() gives the message for the calling thread.
 *
 * All pointers are DEVICE pointers unless stated otherwise.  Nullable inputs
 * (colors_precomp, cov3D_precomp, shs, scales ...) follow the reference: NULL
 * means "not provided" (reference: rasterize_points.cu:110-141 passes the
 * data pointer of an empty tensor, i.e. NULL).
 *
 * The library never allocates or frees device memory itself; the three scratch
 * buffers are obtained through the callbacks and are opaque to the caller
 * (their layout is private and differs from the reference's GeometryState /
 * BinningState / ImageState; they only have to be handed back unchanged to
 * fdgs_backward, like the reference's geomBuffer/binningBuffer/imgBuffer).
 */
#ifndef FDGS_H_INCLUDED
#define FDGS_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FDGS_VERSION 2

/* status codes */
#define FDGS_OK 0
#define FDGS_ERR_INVALID_ARG 1
#define FDGS_ERR_CUDA 2
#define FDGS_ERR_ALLOC 3
#define FDGS_ERR_UNSUPPORTED 4

/* Scratch allocator callback: must return a device pointer to at least
 * `bytes` bytes (128-byte aligned or better), or NULL on failure.
 * Replaces std::function<char*(size_t)> (reference: rasterizer.h:32-34,
 * rasterize_points.cu:28-34 `resizeFunctional`). */
typedef char* (*fdgs_alloc_fn)(void* ctx, size_t bytes);

/* Inputs/outputs of one forward pass.  Field names follow
 * Rasterizer::forward (reference: rasterizer.h:31-65). */
typedef struct fdgs_forward_args {
    int P;                 /* number of Gaussians                              */
    int D;                 /* active spatial SH degree (0..3)                  */
    int D_t;               /* active temporal SH degree (0..2)                 */
    int M;                 /* SH coefficients per Gaussian (row length / 3)    */
    const float* background;      /* [3]                                       */
    int width, height;
    const float* means3D;         /* [P,3]                                     */
    const float* shs;             /* [P,M,3] or NULL                           */
    const float* colors_precomp;  /* [P,3] or NULL                             */
    const float* flows_precomp;   /* [P,2]                                     */
    const float* opacities;       /* [P]                                       */
    const float* ts;              /* [P] or NULL                               */
    const float* scales;          /* [P,3] or NULL                             */
    const float* scales_t;        /* [P] or NULL                               */
    float scale_modifier;
    const float* rotations;       /* [P,4] or NULL                             */
    const float* rotations_r;     /* [P,4] or NULL                             */
    const float* cov3D_precomp;   /* [P,6] or NULL                             */
    float prefilter_var;
    const float* viewmatrix;      /* [16], column-major (transposed torch)     */
    const float* projmatrix;      /* [16], column-major                        */
    const float* cam_pos;         /* [3]                                       */
    float timestamp;
    float time_duration;
    int rot_4d;
    int gaussian_dim;
    int force_sh_3d;
    float tan_fovx, tan_fovy;
    int prefiltered;
    int debug;             /* !=0: synchronise + check after every stage       */
    /* outputs */
    float* out_means3D;    /* [P,3]  written for every Gaussian (shifted mean) */
    float* out_color;      /* [3,H,W]                                          */
    float* out_flow;       /* [2,H,W]                                          */
    float* out_depth;      /* [1,H,W]                                          */
    float* out_T;          /* [1,H,W] final transmittance                      */
    int* radii;            /* [P]                                              */
    /* Raw-parameter entry (version 2; SURVEY.md section 8(f) row 1).  The reference activates the optimiser's raw
     * parameters in PyTorch before every render (scene/gaussian_model.py:179-219: exp, sigmoid, F.normalize, and a
     * torch.cat of features_dc / features_rest); with raw_params != 0 the kernels do it themselves:
     *   scales, scales_t   are LOG-scales            (exp applied)
     *   rotations(_r)      are un-normalised         (q / max(||q||, 1e-12))
     *   opacities          are logits                (sigmoid)
     * and, independently, a non-NULL shs_rest splits the SH row like the reference model's two tensors:
     *   shs = features_dc [P,1,3], shs_rest = features_rest [P,M-1,3]  (no 1.15 GB concatenation per frame). */
    int raw_params;
    const float* shs_rest;
} fdgs_forward_args;

/* Scratch handles returned by fdgs_forward (device pointers obtained through
 * the callbacks) plus what the torch shim needs to build `covs3D_com`. */
typedef struct fdgs_forward_result {
    int num_rendered;      /* R = number of (tile, Gaussian) instances         */
    char* geom_buffer;
    char* binning_buffer;
    char* image_buffer;
    size_t geom_bytes, binning_bytes, image_bytes;
    const float* cov3D;    /* [P,6] inside geom_buffer (reference: rasterize_points.cu:144-147) */
} fdgs_forward_result;

/* Inputs/outputs of one backward pass.  Field names follow
 * Rasterizer::backward (reference: rasterizer.h:67-112). */
typedef struct fdgs_backward_args {
    int P, D, D_t, M, R;
    const float* background;
    int width, height;
    const float* out_means3D;     /* shifted means written by the forward      */
    const float* shs;
    const float* colors_precomp;
    const float* flows_2d;
    const float* opacities;
    const float* ts;
    const float* scales;
    const float* scales_t;
    float scale_modifier;
    const float* rotations;
    const float* rotations_r;
    const float* cov3D_precomp;
    float prefilter_var;
    const float* viewmatrix;
    const float* projmatrix;
    const float* campos;
    float timestamp;
    float time_duration;
    int rot_4d;
    int gaussian_dim;
    int force_sh_3d;
    float tan_fovx, tan_fovy;
    const int* radii;
    const char* geom_buffer;
    const char* binning_buffer;
    const char* image_buffer;
    const float* dL_dpix;         /* [3,H,W]                                   */
    const float* dL_depths;       /* [1,H,W]  or NULL = no gradient (all zero) */
    const float* dL_masks;        /* [1,H,W]  grad of alpha = 1 - T, or NULL   */
    const float* dL_dpix_flow;    /* [2,H,W]  or NULL                          */
    int debug;
    /* Outputs.  The five "blend" gradients must be ZERO on entry (they are
     * accumulated into, like the reference: rasterize_points.cu:201-213); the
     * others are fully overwritten for every Gaussian (zeros where a Gaussian
     * was not rendered), so they may be uninitialised on entry. */
    float* dL_dmean2D;     /* [P,3]   accumulated                              */
    float* dL_dconic;      /* [P,2,2] accumulated (x, y, -, w)                 */
    float* dL_dopacity;    /* [P]     accumulated, then scaled by marginal_t   */
    float* dL_dcolor;      /* [P,3]   accumulated                              */
    float* dL_dflows;      /* [P,2]   accumulated                              */
    float* dL_dmean3D;     /* [P,3]   overwritten                              */
    float* dL_dcov3D;      /* [P,6]   overwritten                              */
    float* dL_dsh;         /* [P,M,3] overwritten                              */
    float* dL_dts;         /* [P]     overwritten                              */
    float* dL_dscale;      /* [P,3]   overwritten                              */
    float* dL_dscale_t;    /* [P]     overwritten                              */
    float* dL_drot;        /* [P,4]   overwritten                              */
    float* dL_drot_r;      /* [P,4]   overwritten                              */
    /* View-parallel mode (version 2; multi-GPU, see fdgs_sh_outer_sum below): when `sh_factors` is non-NULL and
     * dL_dsh is NULL the 12*M-byte dL_dsh rows are NOT written; instead sh_factors[P,3] receives the clamp-masked
     * colour gradient of every Gaussian (zeros where this view did not render it) -- the only view-dependent factor
     * of the rank-one dL_dsh row.  The direction / time terms of the SH backward still go to dL_dmean3D / dL_dts. */
    float* sh_factors;     /* [P,3]   overwritten, or NULL                     */
    /* Raw-parameter entry, as in fdgs_forward_args: the SAME values as in the forward.  With raw_params != 0 the
     * gradients dL_dscale, dL_dscale_t, dL_drot, dL_drot_r and dL_dopacity come out w.r.t. the RAW parameters (chain
     * rule through exp / normalize / sigmoid applied in the kernel).  With shs_rest the SH gradient is split the same
     * way: dL_dsh = [P,1,3], dL_dsh_rest = [P,M-1,3]. */
    int raw_params;
    const float* shs_rest;
    float* dL_dsh_rest;
} fdgs_backward_args;

/* Library / build identification. */
int fdgs_version(void);
/* Message of the last error on the calling thread ("" if none). */
const char* fdgs_last_error(void);

/* Sizes of the private scratch buffers (bytes), for callers that want to
 * pre-allocate (reference: required<GeometryState>(P) etc.,
 * rasterizer_impl.h:67-73). */
size_t fdgs_geom_bytes(int P);
size_t fdgs_image_bytes(int width, int height);
size_t fdgs_binning_bytes(int num_rendered, int width, int height);

/* Forward.  `stream` is a cudaStream_t passed as void*.  Performs exactly one
 * host synchronisation on `stream` (to learn num_rendered and size the binning
 * buffer), like the reference (rasterizer_impl.cu:302). */
int fdgs_forward(const fdgs_forward_args* args,
                 fdgs_alloc_fn geom_alloc, void* geom_ctx,
                 fdgs_alloc_fn binning_alloc, void* binning_ctx,
                 fdgs_alloc_fn image_alloc, void* image_ctx,
                 void* stream,
                 fdgs_forward_result* result);

/* Backward.  Fully asynchronous on `stream`. */
int fdgs_backward(const fdgs_backward_args* args, void* stream);

/* Per-pixel background image [3,H,W] (device, fp32) behind the Gaussians, e.g. an environment-map sky
 * (fdgs_sky_forward).  The colour image becomes
 *     out_color = (C + T * background) + (1 - (1 - T)) * bg_image
 * rounded step by step, i.e. bit-identical to `rendered + (1 - alpha) * bg_image` evaluated in fp32 on the images
 * fdgs_forward returns (alpha = 1 - T).  Every other output is unchanged.  bg_image == NULL: identical to
 * fdgs_forward / fdgs_backward.  The backward takes the SAME bg_image as the forward; dL_dbg_image [3,H,W] (or
 * NULL) is overwritten for every pixel with (1 - (1 - T)) * dL_dpix. */
int fdgs_forward_bg(const fdgs_forward_args* args, const float* bg_image,
                    fdgs_alloc_fn geom_alloc, void* geom_ctx,
                    fdgs_alloc_fn binning_alloc, void* binning_ctx,
                    fdgs_alloc_fn image_alloc, void* image_ctx,
                    void* stream,
                    fdgs_forward_result* result);
int fdgs_backward_bg(const fdgs_backward_args* args, const float* bg_image, float* dL_dbg_image, void* stream);

/* The SH gradient's zero rows written by the forward.  In training most Gaussians are not rendered by a view, and their
 * dL_dsh rows are zero: about 800 MB of a 2M-Gaussian model's 1.15 GB [P,48,3] gradient.  fdgs_forward_zero_sh is
 * fdgs_forward_bg that, with dL_dsh non-NULL, also writes those rows -- every row of a Gaussian with radii == 0 or no
 * tile touched -- from the blend kernel, whose DRAM is otherwise nearly idle.  dL_dsh is [P,M,3], or with shs_rest the
 * split pair dL_dsh [P,1,3] + dL_dsh_rest [P,M-1,3]; the other rows are left as they are.  Both NULL: fdgs_forward_bg.
 * fdgs_backward_zero_sh is fdgs_backward_bg; with sh_rows_zeroed != 0 it takes the SAME dL_dsh (| dL_dsh_rest) that its
 * forward zeroed and writes only the rendered rows (the view-parallel sh_factors mode ignores the flag), computed as
 * fdgs_backward_bg computes them: together the two calls leave the dense gradient fdgs_backward_bg writes. */
int fdgs_forward_zero_sh(const fdgs_forward_args* args, const float* bg_image, float* dL_dsh, float* dL_dsh_rest,
                         fdgs_alloc_fn geom_alloc, void* geom_ctx,
                         fdgs_alloc_fn binning_alloc, void* binning_ctx,
                         fdgs_alloc_fn image_alloc, void* image_ctx,
                         void* stream,
                         fdgs_forward_result* result);
int fdgs_backward_zero_sh(const fdgs_backward_args* args, const float* bg_image, float* dL_dbg_image, int sh_rows_zeroed,
                          void* stream);

/* Batched views: B >= 1 cameras of the same Gaussians in one call per direction, one launch per stage and ONE host
 * synchronisation for the whole batch.  Every view's outputs are bit-identical to fdgs_forward_bg on that camera.
 * `view` holds what the views share, as in fdgs_forward_args, except:
 *   viewmatrix / projmatrix / cam_pos   [B,16] / [B,16] / [B,3] device tables, one row per view
 *   timestamp / tan_fovx / tan_fovy     ignored: the per-view host arrays below
 *   out_means3D [B,P,3], radii [B,P], out_color [B,3,H,W], out_flow [B,2,H,W], out_depth / out_T [B,1,H,W]
 *   colors_precomp / cov3D_precomp      must be NULL (SH and scales / rotations only)
 * bg_image: [B,3,H,W] per-view background images (fdgs_forward_bg), or NULL; bg_views must then equal B. */
typedef struct fdgs_forward_batch_args {
    fdgs_forward_args view;
    int B;
    const float* timestamps;   /* host [B] */
    const float* tan_fovx;     /* host [B] */
    const float* tan_fovy;     /* host [B] */
    const float* bg_image;     /* [B,3,H,W] device, or NULL */
    int bg_views;              /* leading dimension of bg_image */
} fdgs_forward_batch_args;

/* Backward of fdgs_forward_batch, fully asynchronous.  `view` as in fdgs_backward_args, except:
 *   viewmatrix / projmatrix / campos, out_means3D, radii: the forward's per-view tables and outputs
 *   timestamp / tan_fovx / tan_fovy   ignored (the forward keeps the per-view values in geom_buffer)
 *   dL_dpix [B,3,H,W], dL_depths / dL_masks [B,1,H,W], dL_dpix_flow [B,2,H,W] (each optional but dL_dpix)
 *   dL_dmean2D [B,P,3]                per view, accumulated (ZERO on entry)
 *   dL_dopacity, dL_dmean3D, dL_dts, dL_dscale, dL_dscale_t, dL_drot, dL_drot_r: [P,...] sums over the views in
 *                                     view order, ((g_0 + g_1) + g_2) + ... in fp32, overwritten
 *   dL_dsh (+ dL_dsh_rest)            the SH rows summed over the views, overwritten
 *   dL_dconic, dL_dcolor, dL_dflows, dL_dcov3D, sh_factors: ignored (per-view scratch lives in `scratch`)
 * scratch: fdgs_backward_batch_scratch_bytes(P, B) bytes of device memory.  dL_dbg_image: [B,3,H,W] or NULL. */
typedef struct fdgs_backward_batch_args {
    fdgs_backward_args view;
    int B;
    const float* bg_image;     /* the forward's bg_image, or NULL */
    int bg_views;
    float* dL_dbg_image;       /* [B,3,H,W] overwritten, or NULL */
    char* scratch;
} fdgs_backward_batch_args;

size_t fdgs_geom_batch_bytes(int P, int B);
size_t fdgs_image_batch_bytes(int width, int height, int B);
size_t fdgs_backward_batch_scratch_bytes(int P, int B);
int fdgs_forward_batch(const fdgs_forward_batch_args* args,
                       fdgs_alloc_fn geom_alloc, void* geom_ctx,
                       fdgs_alloc_fn binning_alloc, void* binning_ctx,
                       fdgs_alloc_fn image_alloc, void* image_ctx,
                       void* stream,
                       fdgs_forward_result* result);
int fdgs_backward_batch(const fdgs_backward_batch_args* args, void* stream);

/* Camera gradients: the backward also returns dL/dviewmatrix, dL/dprojmatrix and dL/dcampos, for pose refinement,
 * rig calibration or tracking through the rasterizer.  fdgs_backward_camera is fdgs_backward_zero_sh and
 * fdgs_backward_batch_camera is fdgs_backward_batch, with every other output the same, plus:
 *   dL_dviewmatrix / dL_dprojmatrix   [16] ([B,16] batched), in the layout of viewmatrix / projmatrix: element 4c + r
 *                                     is the gradient of the caller's element 4c + r.  Entries the forward does not
 *                                     read are exactly 0: 3, 7, 11, 15 of the view matrix (view-space w) and 2, 6, 10,
 *                                     14 of the projection matrix (clip z).
 *   dL_dcampos                        [3] ([B,3]); the camera centre enters only the SH view direction, so it is 0 with
 *                                     colors_precomp.
 * Each is the sum over the Gaussians the view renders (radii > 0, a tile touched) of the reference backward's own
 * per-Gaussian terms (backward.cu: the view-space mean's gradient, the W part of the EWA Jacobian product T = J W,
 * the homogeneous projection and the SH direction), applied to the camera instead of the mean, so that
 *     sum_i dL/dmeans3D[i] + dL/dcampos = V[0:12] (3x4, row-major) @ dL/dV[12:16] + Pm[0:12] @ dL/dPm[12:16]
 * (moving world and camera together leaves the image unchanged).  The sums are reduced without floating-point
 * atomics, per block and then over the blocks in a fixed order in fp64: the camera gradient of a call is deterministic.
 * scratch: fdgs_camera_grad_scratch_bytes(P, B) bytes of device memory (B = 1 for fdgs_backward_camera).  A NULL output
 * or scratch, or a bad B, is rejected before any launch. */
typedef struct fdgs_camera_grad_out {
    float* dL_dviewmatrix;     /* [B,16] overwritten */
    float* dL_dprojmatrix;     /* [B,16] overwritten */
    float* dL_dcampos;         /* [B,3]  overwritten */
    char* scratch;
} fdgs_camera_grad_out;
size_t fdgs_camera_grad_scratch_bytes(int P, int B);
int fdgs_backward_camera(const fdgs_backward_args* args, const float* bg_image, float* dL_dbg_image, int sh_rows_zeroed,
                         const fdgs_camera_grad_out* cam, void* stream);
int fdgs_backward_batch_camera(const fdgs_backward_batch_args* args, const fdgs_camera_grad_out* cam, void* stream);

/* The batched forward sized by an instance capacity instead of the exact count: no host synchronisation, no read of
 * device memory on the host and no upload of host data, so the call can be captured in a CUDA graph and replayed with
 * new cameras.  `batch` as in fdgs_forward_batch, except that its host timestamps / tan_fovx / tan_fovy are ignored: the
 * per-view scalars come from the device arrays below.  The binning buffer is requested once, before the first launch,
 * at fdgs_binning_bytes(capacity, W, H) bytes, and result->num_rendered is set to `capacity`.
 *
 * status (device int[4]) receives {R, largest tile, overflow = R > capacity, wrap = R > 2^31 - 1}; R saturates at
 * 2^31 - 1.  Without overflow or wrap every output is bit-identical to fdgs_forward_batch's.  With either, the views
 * render as if no Gaussian were listed: the colour is the background (with bg_image: background + bg_image, as for an
 * empty tile), depth, flow, alpha and n_contrib are 0, radii and out_means3D are still the preprocess's; no write falls
 * outside the binning buffer.  The backward is fdgs_backward_batch with R = capacity; after an overflow it returns zero
 * per-Gaussian gradients.  debug != 0 is rejected while `stream` is capturing (debug synchronises after every stage). */
typedef struct fdgs_forward_capacity_args {
    fdgs_forward_batch_args batch;
    const float* timestamps;   /* device [B] */
    const float* tan_fovx;     /* device [B] */
    const float* tan_fovy;     /* device [B] */
    int capacity;              /* instances the binning buffer holds, summed over the B views */
    int* status;               /* device int[4] */
} fdgs_forward_capacity_args;
int fdgs_forward_batch_capacity(const fdgs_forward_capacity_args* args,
                                fdgs_alloc_fn geom_alloc, void* geom_ctx,
                                fdgs_alloc_fn binning_alloc, void* binning_ctx,
                                fdgs_alloc_fn image_alloc, void* image_ctx,
                                void* stream,
                                fdgs_forward_result* result);

/* Environment-map sky sphere (the reference's sky for scenes with an environment map: gaussian_renderer/__init__.py
 * and Camera.get_rays).  Each pixel's ray -- the pixel centre ((x + 0.5 - cx) / fl_x, (y + 0.5 - cy) / fl_y, 1, 1)
 * through c2w, minus campos, normalised -- is intersected with the sphere |X| = radius; the hit point gives
 * u = atan2(y, x) / 2pi + 0.5, v = acos(z / radius) / pi, and env_map is sampled bilinearly at (2u - 1, 2v - 1) like
 * F.grid_sample with its defaults (align_corners = False, zero padding, u along the width). */
typedef struct fdgs_sky_args {
    const float* env_map;         /* [3,Hm,Wm]                                 */
    int env_height, env_width;    /* Hm, Wm                                    */
    const float* c2w;             /* [16] row-major camera-to-world, torch.linalg.inv(world_view_transform.T) */
    const float* campos;          /* [3]  ray origin (camera centre)           */
    float fl_x, fl_y, cx, cy;     /* pinhole intrinsics in pixels              */
    float radius;                 /* sky sphere radius (60 in the reference)   */
    int width, height;            /* image size W, H                           */
} fdgs_sky_args;
/* (The colatitude is evaluated as atan2(sqrt(x^2 + y^2), z), equal to acos(z / radius) on the sphere and accurate at
 * the poles.)  out_sky [3,H,W] overwritten.  miss_flag (device int, or NULL) is set to 1 if any ray does not cross the sphere (the
 * reference asserts on this); it is never cleared, so zero it before the call. */
int fdgs_sky_forward(const fdgs_sky_args* args, float* out_sky, int* miss_flag, void* stream);
/* dL_denv [3,Hm,Wm] += the share of dL_dsky [3,H,W] of every texel (accumulated: zero it for a fresh gradient). */
int fdgs_sky_backward(const fdgs_sky_args* args, const float* dL_dsky, float* dL_denv, void* stream);
/* The sky of B views of one image size in one launch each way, every camera read from device tables, so that neither
 * entry synchronises or reads device memory on the host (a CUDA graph can capture both).  View b's sky is
 * fdgs_sky_forward's with c2w = c2w[b], campos = campos[b] and (fl_x, fl_y, cx, cy) = intrinsics[b], bit for bit. */
typedef struct fdgs_sky_batch_args {
    const float* env_map;         /* [3,Hm,Wm]                                 */
    int env_height, env_width;    /* Hm, Wm                                    */
    const float* c2w;             /* device [B,16] row-major camera-to-world, as fdgs_sky_args.c2w */
    const float* campos;          /* device [B,3] ray origins (camera centres) */
    const float* intrinsics;      /* device [B,4] fl_x, fl_y, cx, cy in pixels */
    float radius;                 /* sky sphere radius (60 in the reference)   */
    int width, height;            /* image size W, H                           */
    int B;                        /* views, >= 1                               */
} fdgs_sky_batch_args;
/* out_sky [B,3,H,W] overwritten; miss_flag (device int, or NULL) is set to 1 if any ray of any view does not cross the
 * sphere, and never cleared. */
int fdgs_sky_forward_batch(const fdgs_sky_batch_args* args, float* out_sky, int* miss_flag, void* stream);
/* dL_denv [3,Hm,Wm] += the share of every view's dL_dsky [B,3,H,W] of every texel (accumulated: zero it first). */
int fdgs_sky_backward_batch(const fdgs_sky_batch_args* args, const float* dL_dsky, float* dL_denv, void* stream);

/* present[i] = (view-space z of means3D[i] > 0.2)
 * (reference: rasterizer_impl.cu:54-67, auxiliary.h:140-163). */
int fdgs_mark_visible(int P, const float* means3D, const float* viewmatrix,
                      const float* projmatrix, unsigned char* present, void* stream);

/* Multi-GPU gradient exchange helpers (new: the reference has no multi-GPU path; it sums the gradients of
 * sequential views, train.py:104-166).  pack: flat[block_off[t] + r*width[t] + c] = tensors[t][idx[r]*width[t] + c]
 * for r < K; unpack: the inverse scatter.  `tensors` / `widths` / `block_off` are HOST arrays of n <=
 * FDGS_MAX_PACK entries, `idx` (sorted row indices, int64) and `flat` are device pointers. */
#define FDGS_MAX_PACK 16
int fdgs_pack_rows(int n, const float* const* tensors, const int* widths, const long long* block_off,
                   const long long* idx, long long K, float* flat, void* stream);
int fdgs_unpack_rows(int n, float* const* tensors, const int* widths, const long long* block_off,
                     const long long* idx, long long K, const float* flat, void* stream);

/* View-parallel SH gradient (multi-GPU; new -- the reference sums the dL_dsh of sequential views in autograd,
 * train.py:104-166).  After the colour factors of all V views of a step have been all-gathered for the K Gaussians
 * of the union (table = V blocks of `view_stride` floats: K rows of 3 floats, then at `meta_off` the view's
 * timestamp and camera position), rebuilds every view's rank-one dL_dsh row from the replicated Gaussian
 * parameters and sums them in view order: out[i] = sum_v w(dir_v(i), t_v) x factors_v[slot_of[i]], zeros for
 * slot_of[i] < 0.  Bit-identical to accumulating the views' dL_dsh tensors one after the other.  The row may be
 * split over two tensors (out0 = first m0 coefficients, out1 = the rest; out1 NULL and m0 = M for one tensor). */
typedef struct fdgs_sh_sum_args {
    int P, V, K;
    const float* table;
    long long view_stride;
    long long meta_off;
    const int* slot_of;           /* [P]                                       */
    const long long* union_idx;   /* [K] Gaussian index of every union row (ascending): the inverse of slot_of */
    float* dir_scratch;           /* [V*K*8] floats of scratch                 */
    const float* means3D;         /* [P,3] the rasterizer's inputs (replicated) */
    const float* ts;              /* [P] or NULL                               */
    const float* scales;          /* [P,3] (needed when rot_4d)                */
    const float* scales_t;        /* [P]                                       */
    const float* rotations;       /* [P,4]                                     */
    const float* rotations_r;     /* [P,4]                                     */
    float scale_modifier;
    float time_duration;
    int rot_4d, gaussian_dim, force_sh_3d;
    int D, D_t, M;
    float* out0;
    int m0;
    float* out1;
    int accumulate;
} fdgs_sh_sum_args;
int fdgs_sh_outer_sum(const fdgs_sh_sum_args* args, void* stream);

/* flag[0] |= 1 if a row r with radii[r] <= 0 of any of the n tensors ([P, widths[i]], device) holds a non-zero
 * element: the guard of the sparse (union-rows-only) gradient exchange.  `tensors` / `widths` are HOST arrays. */
int fdgs_check_rows_zero(int n, const float* const* tensors, const int* widths, long long P, const int* radii,
                         int* flag, void* stream);

/* Densification statistics of ONE view, accumulated in one pass (reference: train.py:164-183 -- viewspace gradient norm,
 * visibility, max radius per Gaussian): grad_norm_sum[i] += ||viewspace_grad[i, 0:2]||, visibility_count[i] += radii[i] > 0,
 * max_radii[i] = max(max_radii[i], radii[i]).  grad_stride = floats per row of viewspace_grad (3 for means2D.grad). */
int fdgs_view_stats(long long P, const float* viewspace_grad, int grad_stride, const int* radii, float* grad_norm_sum,
                    float* visibility_count, int* max_radii, void* stream);

/* Densification statistics of one optimisation step (reference: train.py:168-183 and :233-237,
 * scene/gaussian_model.py:579-589 add_densification_stats / _grad), one pass over the P Gaussians.
 *   batch_size == 1: point_grad = the view's viewspace_points.grad [P, point_grad_stride >= 2], visibility_count NULL,
 *                    radii = the view's radii; visible = radii > 0, g = ||point_grad[i, 0:2]||, tg = t_grad[i].
 *   batch_size  > 1: point_grad = the views' summed gradient norms [P] (stride 1), visibility_count [P] and radii (the
 *                    MAX over the views) as ViewBatchStats holds them; visible = visibility_count > 0,
 *                    g = point_grad[i] * batch_size / visibility_count[i], tg = t_grad[i] * batch_size / visibility_count[i].
 * For visible rows: xyz_gradient_accum += g, denom += 1, t_gradient_accum += tg, max_radii2D = max(max_radii2D, radii).
 * t_grad / t_gradient_accum: [P] (the _t.grad column), both NULL for 3D Gaussians. */
int fdgs_densify_stats(long long P, int batch_size, const float* point_grad, int point_grad_stride,
                       const float* visibility_count, const int* radii, const float* t_grad, float* xyz_gradient_accum,
                       float* denom, float* t_gradient_accum, float* max_radii2D, void* stream);
/* The same, predicated on the rasterizer's status (device int[4] {R, largest tile, overflow, wrap}, as
 * fdgs_forward_batch_capacity writes it; NULL = fdgs_densify_stats): with overflow or wrap set nothing is written, so a
 * CUDA graph whose forward overflowed can be replayed again without counting the step twice. */
int fdgs_densify_stats_status(long long P, int batch_size, const float* point_grad, int point_grad_stride,
                              const float* visibility_count, const int* radii, const float* t_grad, float* xyz_gradient_accum,
                              float* denom, float* t_gradient_accum, float* max_radii2D, const int* status, void* stream);

/* Densify and prune (reference: scene/gaussian_model.py:486-577 densify_and_prune with densify_and_clone,
 * densify_and_split and prune_points) as one compaction of every parameter row and Adam-moment row into new tensors.
 * The result rows are, in this order and each part in source order without its pruned rows: the original rows that
 * were neither split nor pruned; the clones; copy 1 of every split row; copy 2; ... copy N.
 *   grads = xyz_gradient_accum / denom (NaN -> 0); smax = max(exp(scaling[i, :]))
 *   clone : |grads| >= max_grad and smax <= dense_extent            (dense_extent = fp32(percent_dense * extent))
 *   split : grads >= max_grad and smax > dense_extent
 *   prune : sigmoid(opacity) < min_opacity, or with use_max_screen_size
 *           max_radii2D > max_screen_size or smax > big_extent   (big_extent = fp32(0.1 * extent)), tested on every
 *           output row with its own values; a densifying call has already zeroed max_radii2D, so only prune_only
 *           calls read it.
 * Split children: scaling(_t) = log(exp(scaling(_t)) * fp32(1 / fp32(0.8 N))), position = R sample + mean where
 * sample = samples row * exp(scaling) (rot_4d: 4-vector over [scaling, scaling_t] rotated by the 4D rotation of
 * (rotation, rotation_r), giving xyz and t; otherwise R = rotation matrix of `rotation` and t = t + samples_t row *
 * exp(scaling_t)).  Sample rows are [k * S + j] for copy k of the j-th selected row (S = split rows selected), as
 * torch.normal over the reference's repeat(N, 1) tiles draws them; positions are evaluated in double and rounded once.
 * The tensor table lists every row tensor to compact: src [P, width], dst [P_new, width] (caller-allocated):
 *   COPY       every output row copies its source row (features, opacity, rotations)
 *   MOMENT     original rows copy, clones and split children are zero (Adam moments; statistics of prune_only)
 *   XYZ/T/SCALING/SCALING_T  the parameters split children compute (widths 3 / 1 / 3 / 1). */
#define FDGS_DENSIFY_MAX_TENSORS 32
#define FDGS_DENSIFY_COPY 0
#define FDGS_DENSIFY_MOMENT 1
#define FDGS_DENSIFY_XYZ 2
#define FDGS_DENSIFY_T 3
#define FDGS_DENSIFY_SCALING 4
#define FDGS_DENSIFY_SCALING_T 5
typedef struct fdgs_densify_args {
    long long P;                  /* rows before the call                      */
    int N;                        /* children per split row (reference: 2)     */
    int gaussian_dim;             /* 3 or 4                                    */
    int rot_4d;
    int prune_only;
    int use_max_screen_size;      /* max_screen_size given (truthy)            */
    float max_grad;
    float min_opacity;
    float dense_extent;
    float big_extent;
    float max_screen_size;
    const float* xyz_gradient_accum;  /* [P]  (densifying calls)               */
    const float* denom;               /* [P]  (densifying calls)               */
    const float* max_radii2D;         /* [P]  (prune_only with use_max_screen_size) */
    const float* xyz;                 /* [P,3]                                 */
    const float* t;                   /* [P]   gaussian_dim 4                  */
    const float* scaling;             /* [P,3] log-scales                      */
    const float* scaling_t;           /* [P]   gaussian_dim 4                  */
    const float* rotation;            /* [P,4]                                 */
    const float* rotation_r;          /* [P,4] rot_4d                          */
    const float* opacity;             /* [P]   logits                          */
    const float* samples;             /* [S*N, 3] (rot_4d: [S*N, 4]) standard normal draws */
    const float* samples_t;           /* [S*N]  gaussian_dim 4 without rot_4d  */
    int num_tensors;
    int kind[FDGS_DENSIFY_MAX_TENSORS];
    int width[FDGS_DENSIFY_MAX_TENSORS];
    const float* src[FDGS_DENSIFY_MAX_TENSORS];
    float* dst[FDGS_DENSIFY_MAX_TENSORS];
} fdgs_densify_args;
/* Bytes of device scratch fdgs_densify_plan needs for P rows; hand the same buffer to fdgs_densify_apply. */
size_t fdgs_densify_scratch_bytes(long long P);
/* Decides every row's fate and each output row's index.  totals (device int[4]) receives: original rows kept, clones
 * kept, rows selected for splitting (S), children kept per copy; P_new = totals[0] + totals[1] + N * totals[3].
 * Asynchronous: the caller copies totals to the host once to size the outputs and the samples. */
int fdgs_densify_plan(const fdgs_densify_args* args, char* scratch, int* totals, void* stream);
/* Writes every dst tensor; totals = the HOST copy of fdgs_densify_plan's totals.  Fully asynchronous. */
int fdgs_densify_apply(const fdgs_densify_args* args, const char* scratch, const int* totals, void* stream);
/* Reset opacity in place (reference: scene/gaussian_model.py:371-374): opacity = log(x / (1 - x)) with
 * x = min(sigmoid(opacity), 0.01); exp_avg and exp_avg_sq (or NULL) of those rows are zeroed. */
int fdgs_reset_opacity(long long P, float* opacity, float* exp_avg, float* exp_avg_sq, void* stream);

/* ---- the callers either side of the rasterizer in a training step (SURVEY.md section 8(f)) ---------------------- */

/* Fused photometric loss (reference: utils/loss_utils.py:18-64 l1_loss + ssim, combined as train.py:115-117):
 *   loss = (1 - lambda) * mean|x - y| + lambda * (1 - mean(SSIM(x, y))),  11x11 Gaussian window, sigma 1.5, zero padding.
 * forward : sums[0] = sum|x - y|, sums[1] = sum SSIM map (device doubles; loss = combine on the device or host),
 *           maps[3,C,H,W] = per-pixel partial derivatives kept for the backward.
 * backward: dL_dx[C,H,W] = grad_scale[0] * d loss / d x   (grad_scale: device scalar, NULL = 1). */
int fdgs_l1_ssim_forward(const float* x, const float* y, int C, int H, int W, float* maps, double* sums, void* stream);
int fdgs_l1_ssim_backward(const float* x, const float* y, int C, int H, int W, const float* maps, const float* grad_scale,
                          float lambda_dssim, float* dL_dx, void* stream);

/* Fused multi-tensor Adam step (reference: torch.optim.Adam(eps=1e-15) over the parameter groups of
 * scene/gaussian_model.py:331-357, stepped at train.py:248-249).  n <= FDGS_MAX_PACK tensors [P, widths[i]] (device),
 * one learning rate each; `step` is the 1-based step count (bias correction).  beta1 / beta2 / eps are DOUBLES like the
 * Python floats torch receives: the weights 1 - beta are formed in double and then rounded to fp32 (1 - 0.999 in fp32
 * arithmetic is 1.3e-5 off 0.001f).  rows = NULL: every row (torch's dense
 * semantics); otherwise only the `num_rows` listed rows are touched (sparse Adam over the rendered Gaussians).
 * zero_grad != 0 clears the gradient elements it consumed. */
int fdgs_adam_step(int n, float* const* params, float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                   const int* widths, const float* lrs, long long P, const long long* rows, long long num_rows,
                   long long step, double beta1, double beta2, double eps, int zero_grad, void* stream);

/* Adam's per-tensor scalars, on the host, in the double arithmetic fdgs_adam_step uses (it calls this function):
 * for each of n <= FDGS_MAX_PACK tensors with enable[i] != 0 and its 1-based step count steps[i] (already advanced),
 *   table[3i] = (float)((double)lrs[i] / (1 - beta1^steps[i])),  table[3i+1] = (float)sqrt(1 - beta2^steps[i]),
 *   table[3i+2] = 1;
 * a tensor with enable[i] == 0 gets {0, 1, 0} (its step count is not read).  All pointers are host arrays. */
int fdgs_adam_scalars(int n, const float* lrs, const long long* steps, const int* enable, double beta1, double beta2,
                      float* table);

/* Dense fused Adam with the per-tensor scalars read on the device, for a step captured in a CUDA graph: the tensor
 * table of fdgs_adam_step; scalars = device float[3n], a table as fdgs_adam_scalars fills it (a tensor whose enable
 * entry is 0 keeps its parameter and both moments); status = NULL or the rasterizer's device int[4] {R, largest tile,
 * overflow, wrap}: with overflow or wrap set nothing is written.  Tensors of different step counts share the launch. */
int fdgs_adam_step_staged(int n, float* const* params, float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                          const int* widths, long long P, const float* scalars, const int* status, double beta1, double beta2,
                          double eps, void* stream);

/* k nearest neighbours (k <= 32) of every point among the same n points, squared distances ascending, the point
 * itself first (reference: pointops2 knnquery, pointops2/src/knnquery/knnquery_cuda_kernel.cu:65-107, as called by
 * utils/general_utils.py:170-184 for the rigidity loss, train.py:132-152).  Uniform-grid search; `scratch` must hold
 * fdgs_knn_scratch_bytes(n) bytes.  brute_force != 0 runs the reference's O(n^2) scan instead (validation). */
size_t fdgs_knn_scratch_bytes(int n);
int fdgs_knn(int n, int k, const float* xyz, char* scratch, int* idx, float* dist2, int brute_force, void* stream);

/* Rigidity and motion regularisers (reference: train.py:132-159, with the velocity of scene/gaussian_model.py:34-47,
 * 247-251 get_current_covariance_and_mean_offset(1.0, t + 0.1) for rot_4d models):
 *   dt = (t + 0.1f) - t;  v_i = Sigma[0:3,3] / Sigma[3,3] * dt   (Sigma = the 4D covariance of the raw parameters:
 *        scales exp(scaling), exp(scaling_t); quaternions q / ||q||; scaling modifier 1)
 *   w_ij = exp(-100 * dist2_ij)  over the k neighbours of fdgs_knn (the point itself first)
 *   loss_rigid  = (sum_i sum_j w_ij ||v_j - v_i||) / k / n        loss_motion = mean_i ||v_i||
 * v is evaluated in double from the fp32 parameters and rounded once; the sums are accumulated in double in a fixed
 * order and rounded once: results are bit-identical run to run.
 * Gradients go to scaling, scaling_t, rotation and rotation_r only (the reference's t gradient is exactly 0 and its
 * kNN input is detached); an edge with ||v_j - v_i|| = 0 contributes no gradient, like torch's norm backward.
 * Nothing synchronises the host. */
typedef struct fdgs_rigid_args {
    int n;                        /* Gaussians                                 */
    int k;                        /* neighbours per row, 1..32                 */
    const float* t;               /* [n]                                       */
    const float* scaling;         /* [n,3] log-scales                          */
    const float* scaling_t;       /* [n]   log-scale                           */
    const float* rotation;        /* [n,4] un-normalised                       */
    const float* rotation_r;      /* [n,4] un-normalised                       */
    const int* idx;               /* [n,k] neighbour list (rigidity only)      */
    const float* weight;          /* [n,k]                                     */
    const int* in_offsets;        /* [n+1] incoming edges (rigidity backward)  */
    const int* in_edges;          /* [n*k]                                     */
    float* velocity;              /* [n,3] written by the forward, read by the backward */
} fdgs_rigid_args;
/* Bytes of device scratch fdgs_rigid_neighbours and fdgs_rigid_forward need. */
size_t fdgs_rigid_scratch_bytes(int n, int k);
/* The neighbour list of one set of positions, reusable by every call until the positions change: weight [n,k] =
 * exp(-100 * dist2) (bit-identical to torch.exp(-100 * dist)) and the transpose -- the incoming edges of row j are
 * in_edges[in_offsets[j] .. in_offsets[j+1]), edge id = i * k + slot, ascending.  idx / dist2 = fdgs_knn's output. */
int fdgs_rigid_neighbours(int n, int k, const int* idx, const float* dist2, char* scratch, float* weight, int* in_offsets,
                          int* in_edges, void* stream);
/* Writes velocity and the requested losses (device floats; NULL = not wanted; the rigidity loss needs idx / weight). */
int fdgs_rigid_forward(const fdgs_rigid_args* args, char* scratch, float* loss_rigid, float* loss_motion, void* stream);
/* Gradients w.r.t. the raw parameters, overwritten for every row, given the upstream gradients of the two losses
 * (device scalars; NULL = no such term; the rigidity term needs the whole neighbour list).  args->velocity must hold
 * the forward's velocity. */
int fdgs_rigid_backward(const fdgs_rigid_args* args, const float* grad_rigid, const float* grad_motion, float* dL_dscaling,
                        float* dL_dscaling_t, float* dL_drotation, float* dL_drotation_r, void* stream);

/* Evaluation metrics of B image pairs (reference: train.py:312-334 training_report), per view b, in float64:
 *   out[4b + 0] = mean |x - y|                                            (utils/loss_utils.py:18-19)
 *   out[4b + 1] = mean over channels of 20 log10(1 / sqrt(mse_c))         (utils/image_utils.py:17-19; mse_c = 0: +inf)
 *   out[4b + 2] = mean of the SSIM map: 11x11 Gaussian, sigma 1.5, zero padding (utils/loss_utils.py:34-64)
 *   out[4b + 3] = MS-SSIM of torchmetrics 0.11.4 MultiScaleStructuralSimilarityIndexMeasure(data_range=1.0):
 *                 five scales, 2x2 average pooling between them, valid windows, betas (0.0448, 0.2856, 0.3001,
 *                 0.2363, 0.1333), relu of the per-scale means.
 * clamp != 0 clamps x (never y) to [0, 1] first.  accum (NULL = none): accum[0..3] += the four numbers and
 * accum[4] += 1 per view, in view order.  Per-tile partials are reduced in a fixed order, so results are bit-identical
 * run to run and a batch gives what B single-view calls give.  H and W must be at least 176 (MS-SSIM's five scales),
 * B * C at most 65535.  `scratch` holds fdgs_metrics_scratch_bytes bytes.  Nothing synchronises the host. */
typedef struct fdgs_metrics_args {
    int B, C, H, W;
    const float* x;               /* [B,C,H,W] render                          */
    const float* y;               /* [B,C,H,W] ground truth                    */
    int clamp;                    /* != 0: x is clamped to [0, 1]              */
    double* out;                  /* [B,4] l1, psnr, ssim, msssim              */
    double* accum;                /* [5] four sums and a view count, or NULL   */
} fdgs_metrics_args;
/* Bytes of device scratch fdgs_image_metrics needs (0 for sizes it rejects). */
size_t fdgs_metrics_scratch_bytes(int B, int C, int H, int W);
int fdgs_image_metrics(const fdgs_metrics_args* args, char* scratch, void* stream);

/* Union bookkeeping of the exchange: cs = inclusive prefix sum of (radii > 0) over the P Gaussians (device, int32).
 * Writes slot_of[i] = cs[i] - 1 for union Gaussians, -1 otherwise, and the inverse map idx[slot] = i (idx: K =
 * cs[P-1] entries, int64). */
int fdgs_union_maps(long long P, const int* radii, const int* cs, int* slot_of, long long* idx, void* stream);

/* Test/diagnostic hooks (used by tests/ and bench.py only): copy private
 * per-Gaussian / per-instance state out of the scratch buffers into plain
 * caller-provided device arrays so that parity tests can compare them with the
 * oracle bit for bit.  Any output pointer may be NULL. */
int fdgs_debug_export_geom(const char* geom_buffer, int P,
                           float* depths, float* means2D /*[P,2]*/,
                           float* conic_opacity /*[P,4]*/, float* rgb /*[P,3]*/,
                           unsigned char* clamped /*[P,3]*/, unsigned int* tiles_touched,
                           void* stream);
int fdgs_debug_export_binning(const char* binning_buffer, const char* image_buffer,
                              int num_rendered, int width, int height,
                              unsigned int* point_list /*[R]*/,
                              unsigned int* ranges /*[tiles,2]*/,
                              unsigned int* n_contrib /*[H*W]*/,
                              void* stream);
/* One view of a batch (fdgs_forward_batch): its tile ranges [tiles,2] (offsets into the batch's point_list, which
 * fdgs_debug_export_binning copies) and its n_contrib [H*W]. */
int fdgs_debug_export_binning_view(const char* image_buffer, int width, int height, int B, int view,
                                   unsigned int* ranges, unsigned int* n_contrib, void* stream);

/* Test hook of the raw-parameter entry: applies the in-kernel activations to plain arrays of n elements (log_s, logit:
 * [n]; quat: [n,4]).  mode must be 0, ATen's summation order of the quaternion norm, the only one the library has;
 * any other value returns FDGS_ERR_INVALID_ARG. */
int fdgs_debug_activate(int n, const float* log_s, const float* logit, const float* quat, int mode, float* s_out,
                        float* o_out, float* q_out, void* stream);

/* Tile lists.  The reference lists a Gaussian in every tile of the square of half-width ceil(3 sigma_max) around its
 * centre (auxiliary.h:46-59 getRect, rasterizer_impl.cu:71-112), although only the pixels where
 * alpha = min(0.99, opacity * exp(power)) reaches 1/255 ever blend it (forward.cu:590).
 *   mode 1 (default): a Gaussian is listed only in the tiles that ellipse can reach (exact conservative test per tile).
 *                     The instances dropped are instances no pixel would have blended: the images, radii, every other
 *                     output and every gradient are unchanged; the PRIVATE scratch state differs from the
 *                     reference's (shorter tile lists, smaller num_rendered, n_contrib counted in the shorter lists).
 *   mode 0:           the reference's tile lists exactly (point_list, ranges, num_rendered, n_contrib bit-identical).
 * Process-wide; returns the previous mode.  The environment variable FDGS_TILE_CULL sets the initial mode. */
int fdgs_set_tile_cull(int mode);

/* Measurement hooks (bench.py): per-stage device time with CUDA events recorded on the launch
 * stream, and a count of the kernels this library launched.  The reference has no equivalent
 * (it times whole iterations from Python, train.py:57-58,89,185). */
#define FDGS_NUM_STAGES 8
/* stage ids: 0 preprocess_fwd, 1 scan, 2 emit_keys, 3 sort, 4 pack_instances, 5 blend_fwd,
 *            6 blend_bwd, 7 preprocess_bwd
 * Stages launched on a stream that is capturing a CUDA graph record no events. */
int fdgs_profile_enable(int on);
/* Synchronises the recorded events, adds up the milliseconds and call counts per stage since the
 * last read, then resets the accumulators. */
int fdgs_profile_read(double ms[FDGS_NUM_STAGES], long long calls[FDGS_NUM_STAGES]);
/* number of CUDA kernels launched by this library since it was loaded */
long long fdgs_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* FDGS_H_INCLUDED */
