// fdgs_internal.h -- kernel parameter blocks and launch prototypes (library-private).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include "../../include/fdgs.h"
#include "fdgs_common.cuh"

namespace fdgs {

// ---- per-device launch configuration -------------------------------------------------------------
// Function attributes (the > 48 KB dynamic shared-memory opt-in) belong to the (function, device) pair, so a
// process that renders on several GPUs has to set them once on EACH device; the flag word is per call site, one
// bit per device ordinal, updated atomically (two racing threads both set the idempotent attribute -- harmless).
struct PerDeviceOnce {
    std::atomic<unsigned long long> done{0ull};
};
template <class Kernel>
inline cudaError_t ensure_dynamic_smem(Kernel kernel, int bytes, PerDeviceOnce& once) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const unsigned long long bit = 1ull << (dev & 63);
    if (dev < 64 && (once.done.load(std::memory_order_acquire) & bit)) return cudaSuccess;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess && dev < 64) once.done.fetch_or(bit, std::memory_order_release);
    return e;
}
// SM count of the current device (132 on an H100), cached per device ordinal
int device_sm_count();

// ---- batched views (fdgs_forward_batch / fdgs_backward_batch) --------------------------------------------------
// The per-view scalars of a batch, one 32-byte row per view in device memory (uploaded by the forward into the geometry
// buffer, or filled there by launch_view_table for the capacity entry).  focal_x / focal_y are computed exactly as the
// single-view entry computes them.
struct ViewScalars {
    float timestamp, tan_fovx, tan_fovy, focal_x, focal_y, pad[3];
};
// Batched kernels run one view per blockIdx.y (per-Gaussian kernels) or blockIdx.z (tile kernels); every per-view
// array is a [B][...] stack with the stride of one view's array.  One view is {1, NULL}: the single-view instantiations
// never read these.
struct ViewBatch {
    int B;                      // views
    const ViewScalars* scalars; // [B] device
};

// ---- forward preprocess ---------------------------------------------------------------------
struct PreprocessFwdParams {
    int P, D, D_t, M;
    const float* means3D;
    const float* ts;
    const float* scales;
    const float* scales_t;
    float scale_modifier;
    const float* rotations;
    const float* rotations_r;
    const float* opacities;
    const float* shs;
    const float* cov3D_precomp;
    float prefilter_var;
    const float* colors_precomp;
    const float* viewmatrix;
    const float* projmatrix;
    const float* cam_pos;
    float timestamp, time_duration;
    int rot_4d, gaussian_dim, force_sh_3d;
    int W, H;
    float tan_fovx, tan_fovy, focal_x, focal_y;
    int grid_x, grid_y;
    int prefiltered;
    int sh_bulk_ok;             // SH rows can be streamed with cp.async.bulk (16-byte aligned rows)
    int sh_row_stride_floats;   // padded shared-memory row stride (multiple of 4 floats)
    int raw_params;             // scales / scales_t are log-scales, rotations un-normalised, opacities logits
    const float* shs_rest;      // non-NULL: SH row split as shs = [P,1,3] (dc) | shs_rest = [P,M-1,3]
    // outputs
    const float* flows;     // [P,2] or NULL
    float* out_means3D;
    int* radii;
    float* cov3D;           // [P,6]
    InstRec* grec;          // [P] the 64-byte record every tile instance of the Gaussian copies
    uint8_t* clamped;       // bit ch set = channel ch was clamped at 0
    uint32_t* tiles_touched;
    uint4* binrec;          // [P] compact bin record of EVERY Gaussian (see launch_bin_count)
    int tile_cull;          // != 0: list a Gaussian only in the tiles its alpha >= 1/255 footprint reaches (fdgs_set_tile_cull)
    // batched entry (vb.scalars != NULL): viewmatrix / projmatrix / cam_pos are [B,16] / [B,16] / [B,3] tables, the
    // camera scalars come from vb.scalars, and every output above is a [B][P] stack
    ViewBatch vb;
};
cudaError_t launch_preprocess_fwd(const PreprocessFwdParams& p, cudaStream_t stream);
cudaError_t launch_debug_activate(int n, const float* log_s, const float* logit, const float* quat, float* s_out, float* o_out,
                                  float* q_out, cudaStream_t stream);

// ---- binning -----------------------------------------------------------------------------------
// counting sort of the (Gaussian, tile) instances by tile, BIN_CTAS persistent CTAs (binning.cu)
int bin_ctas();                                 // rows of the [bin_ctas()][num_tiles] count matrix
// binrec[i] = { x0 | y0 << 16, x1 | y1 << 16, depth bits, tile mask }: tile rectangle (empty = not listed anywhere) of
// Gaussian i; for rectangles of up to 32 tiles bit j of the mask = tile j (row-major) takes an instance
// a batch (vb.scalars != NULL): binrec is a [vb.B][P] stack, the matrix has vb.B * grid_x * grid_y columns and view v's
// tiles are the columns v * tiles .. v * tiles + tiles - 1
cudaError_t launch_bin_count(int P, const uint4* binrec, int grid_x, int grid_y, uint32_t* matrix, const ViewBatch& vb,
                             cudaStream_t stream);
// matrix -> per-CTA column prefixes; tile_offset / ranges; info[0] = total instances R, info[1] = largest tile.
// status != NULL (the capacity entry): also status[4] = {R, largest tile, R > capacity, wrap} and info[3] = overflow or
// wrap, in which case every tile's range is left empty
cudaError_t launch_tile_scan(int num_tiles, uint32_t* matrix, uint32_t* tile_total, uint32_t* tile_offset, uint2* ranges,
                             uint32_t* info, cudaStream_t stream, int capacity = 0, int* status = nullptr);
// info != NULL (the capacity entry, a batch): the tile_scan's info; the pass writes no key when info[3] != 0
cudaError_t launch_bin_scatter(int P, const uint4* binrec, int grid_x, int grid_y, uint32_t* matrix,
                               const uint32_t* tile_offset, uint64_t* keys, const ViewBatch& vb, cudaStream_t stream,
                               const uint32_t* info = nullptr);
// the capacity entry's view table from device [B] arrays, focal lengths as the host computes them
cudaError_t launch_view_table(int B, int W, int H, const float* timestamps, const float* tan_fovx, const float* tan_fovy,
                              ViewScalars* out, cudaStream_t stream);
// sorts every tile's keys and writes the 64-byte instance records + the sorted index list.  A batch: num_tiles =
// vb.B * tiles per view, and every tile gathers from the slice of its view in grec, a [vb.B][P] stack
int tile_sort_pack_kernel_count(int max_count);
cudaError_t launch_tile_sort_pack(int num_tiles, int max_count, int R, const uint2* ranges, uint64_t* keys,
                                  const InstRec* grec, int P, StageRec* recs, uint32_t* point_list, const ViewBatch& vb,
                                  cudaStream_t stream);
cudaError_t launch_unpack_grec(int P, const InstRec* grec, const int* radii, float* depths, float* means2D,
                               float* conic_opacity, float* rgb, cudaStream_t stream);

// ---- blend ---------------------------------------------------------------------------------------
struct BlendFwdParams {
    int W, H, grid_x, grid_y;
    const uint2* ranges;
    const StageRec* recs;
    const float* background;
    float* final_T;        // [H*W]  (scratch copy used by the backward)
    uint32_t* n_contrib;   // [H*W]
    float* out_color;      // [3,H,W]
    float* out_flow;       // [2,H,W]
    float* out_depth;      // [H,W]
    float* out_T;          // [H,W]
    const float* bg_image; // [3,H,W] per-pixel background behind the Gaussians, or NULL
    int views;             // > 0: batched entry, blockIdx.z = view; ranges and every image are [views] stacks
    // single view only: the SH gradient's rows of the Gaussians the view does not render (radii == 0 or no tile, the
    // test of sh_bwd_kernel), zeroed here so that the backward writes only the rendered rows.  zero_rows[0] is
    // [P, zero_row_floats[0]] (dL_dsh, or dL_dsh [P,1,3] of split rows), zero_rows[1] NULL or [P, zero_row_floats[1]]
    // (dL_dsh_rest).  Each CTA owns a stripe of zero_stripe consecutive rows.
    float* zero_rows[2];
    int zero_row_floats[2];
    int zero_stripe;
    int P;
    const int* radii;
    const uint32_t* tiles_touched;
};
cudaError_t launch_blend_fwd(const BlendFwdParams& p, cudaStream_t stream);

struct BlendBwdParams {
    int W, H, grid_x, grid_y;
    const uint2* ranges;
    const StageRec* recs;
    const float* background;
    const float* final_T;
    const uint32_t* n_contrib;
    const float* dL_dpix;
    const float* dL_depths;
    const float* dL_masks;
    const float* dL_dpix_flow;
    float* dL_dmean2D;    // [P,3]
    float* dL_dconic;     // [P,4]
    float* dL_dopacity;   // [P]
    float* dL_dcolor;     // [P,3]
    float* dL_dflows;     // [P,2]
    const float* bg_image;   // [3,H,W] or NULL (BlendFwdParams::bg_image)
    float* dL_dbg_image;     // [3,H,W] overwritten for every pixel, or NULL
    int views;               // > 0: batched entry, blockIdx.z = view; images and the five gradients are [views] stacks
    int P;                   // Gaussians per view (the batched entry's gradient stride)
};
// leaves RAW moment sums (W10, W01 | W20, W11, W02 | W00 of w = G dL/dalpha about each Gaussian's mean) in
// dL_dmean2D.xy / dL_dconic / dL_dopacity instead of the final gradients; launch_preprocess_bwd finishes them
cudaError_t launch_blend_bwd(const BlendBwdParams& p, cudaStream_t stream);

// ---- backward preprocess ------------------------------------------------------------------------
struct PreprocessBwdParams {
    int P, D, D_t, M;
    const float* means3D;   // shifted means (out_means3D of the forward)
    const int* radii;
    const float* shs;
    const float* ts;
    const float* opacities;
    const uint8_t* clamped;
    const uint32_t* tiles_touched;
    const float* scales;
    const float* scales_t;
    const float* rotations;
    const float* rotations_r;
    float scale_modifier;
    const float* cov3D;     // precomputed or the forward's
    float prefilter_var;
    const float* viewmatrix;
    const float* projmatrix;
    float focal_x, focal_y, tan_fovx, tan_fovy;
    const float* campos;
    float timestamp, time_duration;
    int rot_4d, gaussian_dim, force_sh_3d;
    int has_scales;         // scales != NULL in the reference's sense (backward.cu:908)
    int sh_bulk_ok;         // SH rows are 16-byte aligned and 16-byte multiples: stream with cp.async.bulk
    int sh_row_stride_floats;
    int raw_params;         // as in the forward: gradients then come out w.r.t. the RAW parameters
    const float* shs_rest;  // split SH input (see PreprocessFwdParams)
    float* dL_dsh_rest;     // [P,M-1,3] when shs_rest is given (dL_dsh is then [P,1,3])
    float* dL_dmean2D;      // in/out: .xy raw moment sums of the blend backward in, final gradients out
    float* dL_dconic;       // in/out: raw moment sums in, final gradients out
    float* dL_dopacity;     // in/out
    const float* dL_dcolor;
    const InstRec* grec;    // per-Gaussian records of the forward (conic, blended opacity)
    int W, H;
    float* dL_dmean3D;
    float* dL_dcov3D;
    float* dL_dsh;          // [P,M,3], or NULL when sh_factors is set
    float* sh_factors;      // [P,3] clamp-masked colour gradient (view-parallel mode) instead of the dL_dsh rows
    int sh_rows_zeroed;     // the forward's blend zeroed the non-rendered dL_dsh (| dL_dsh_rest) rows: write rendered rows only
    float* dL_dts;
    float* dL_dscale;
    float* dL_dscale_t;
    float* dL_drot;
    float* dL_drot_r;
    // batched entry (vb.scalars != NULL): cameras as in PreprocessFwdParams, every per-Gaussian input of the forward and
    // every output above is a [B][P] stack, sh_factors a [B][factor_stride] stack whose view block ends with the
    // view's timestamp and camera position at offset 3 P (the ShSumParams table)
    ViewBatch vb;
    long long factor_stride;
};
// The camera gradient (fdgs_backward_camera): geom_bwd reduces each rendered row's CAM_TERMS terms per block into
// `partials`, a [views][CAM_TERMS][camera_grad_blocks(P)] scratch, and one small kernel sums the blocks.  Term slots, in
// the torch tensors' [4,4] layout (element [c][r] = V[4c + r]):
//   0..11   dL/dviewmatrix[c][r], c = 0..3, r = 0..2   (column 3, the view-space w, is not used: 0)
//   12..23  dL/dprojmatrix[c][r], c = 0..3, r = 0, 1, 3 (column 2, clip z, is not used: 0)
//   24..26  dL/dcampos
constexpr int CAM_TERMS = 27;
struct CameraGradParams {
    float* partials;
    float* dL_dviewmatrix;   // [views,16] overwritten
    float* dL_dprojmatrix;   // [views,16] overwritten
    float* dL_dcampos;       // [views,3]  overwritten
};
int camera_grad_blocks(int P);
// the views' outputs from `blocks` partials per term (blocks == 0: zeros)
cudaError_t launch_camera_grad_finish(const CameraGradParams& c, int blocks, int views, cudaStream_t stream);
// cam != NULL: geom_bwd also reduces the camera gradient (one more launch)
cudaError_t launch_preprocess_bwd(const PreprocessBwdParams& p, cudaStream_t stream, const CameraGradParams* cam = nullptr);
int preprocess_bwd_kernel_count(const PreprocessBwdParams& p);
// dst_i[e] = ((src_i[0][e] + src_i[1][e]) + src_i[2][e]) + ... in fp32, view order: the order in which autograd's
// AccumulateGrad builds .grad over a sequential loop of views.  src_i is a [B][n_i] stack.
constexpr int VIEW_SUM_MAX = 8;
struct ViewSumParams {
    int n, B;
    const float* src[VIEW_SUM_MAX];
    float* dst[VIEW_SUM_MAX];
    long long count[VIEW_SUM_MAX];   // elements per view
};
cudaError_t launch_view_sum(const ViewSumParams& p, cudaStream_t stream);

// ---- view-parallel SH gradient (preprocess_bwd.cu: sh_outer_sum_kernel) -----------------------------------------
struct ShSumParams {
    int P, V, K;
    const float* table;       // [V][view_stride] floats: K rows of 3 (clamp-masked colour gradient), then metadata
    long long view_stride;    // floats per view block
    long long meta_off;       // offset of the view's metadata inside its block: timestamp, campos x, y, z
    const int* slot_of;       // [P] row of the Gaussian inside a view block, -1 = rendered by no view
    const long long* union_idx;   // [K] the inverse map: Gaussian of every row (sorted)
    float* dirs;              // [V][K][8] scratch: direction, temporal weights and colour factor per (view, row)
    const float* means3D;     // replicated Gaussian parameters, as handed to the rasterizer
    const float* ts;
    const float* scales;
    const float* scales_t;
    const float* rotations;
    const float* rotations_r;
    float scale_modifier, time_duration;
    int rot_4d, gaussian_dim, force_sh_3d, D, D_t, M;
    float* out0;              // [P, m0, 3]
    int m0;                   // coefficients 0 .. m0-1 of a row live in out0 ...
    float* out1;              // ... the rest in out1 [P, M - m0, 3] (NULL when m0 == M)
    int accumulate;           // add to the tensors' contents instead of overwriting them
    // batched entry: view_means != NULL takes view v's direction from the shifted means the forward wrote,
    // view_means[v][3 P]; union_idx / slot_of may then be NULL, meaning every row (K = P, the identity map)
    const float* view_means;
};
cudaError_t launch_sh_outer_sum(const ShSumParams& p, cudaStream_t stream);
// flag[0] |= 1 if any row r with mask[r] == 0 of any of the n tensors has a non-zero element
cudaError_t launch_rows_zero_check(int n, const float* const* tensors, const int* widths, long long P, const int* mask_radii,
                                   int* flag, cudaStream_t stream);

cudaError_t launch_union_maps(long long P, const int* radii, const int* cs, int* slot_of, long long* idx, cudaStream_t stream);
cudaError_t launch_view_stats(long long P, const float* vgrad, int vstride, const int* radii, float* grad_norm_sum,
                              float* visibility_count, int* max_radii, cudaStream_t stream);
cudaError_t launch_pack_rows(bool unpack, int n, float* const* tensors, const int* widths, const long long* block_off,
                             const long long* idx, long long K, float* flat, cudaStream_t stream);

// ---- training-step neighbours of the rasterizer (SURVEY.md section 8(f)) -----------------------------------------
// fused (1 - lambda) L1 + lambda (1 - SSIM): loss.cu
cudaError_t launch_l1_ssim_fwd(const float* x, const float* y, int C, int H, int W, float* maps, double* sums, cudaStream_t stream);
cudaError_t launch_l1_ssim_bwd(const float* x, const float* y, int C, int H, int W, const float* maps, const float* grad_scale,
                               float lambda_dssim, float* dL_dx, cudaStream_t stream);
// fused multi-tensor Adam, dense or over listed rows: optim.cu
cudaError_t launch_adam(int n, float* const* params, float* const* grads, float* const* m, float* const* v, const int* widths,
                        const float* step_sizes, long long rows, const long long* row_idx, float w1, float beta2, float w2,
                        float eps, float sqrt_bc2, int zero_grad, cudaStream_t stream);
// dense, per-tensor lr / bc1, sqrt(bc2) and enable flag from the device table `scalars`; nothing on a status overflow
cudaError_t launch_adam_staged(int n, float* const* params, float* const* grads, float* const* m, float* const* v,
                               const int* widths, long long rows, const float* scalars, const int* status, float w1,
                               float beta2, float w2, float eps, cudaStream_t stream);
// uniform-grid k nearest neighbours: knn.cu
size_t knn_scratch_bytes(int n);
cudaError_t launch_knn(int n, int k, const float* xyz, char* scratch, int* idx, float* dist2, cudaStream_t stream);
cudaError_t launch_knn_bruteforce(int n, int k, const float* xyz, int* idx, float* dist2, cudaStream_t stream);

// rigidity and motion regularisers (regularize.cu; the arguments are validated by fdgs_api.cu)
struct RigidParams {
    int n, k;
    const float* t;           // [n]
    const float* scaling;     // [n,3] log-scales
    const float* scaling_t;   // [n]   log-scale
    const float* rotation;    // [n,4] raw quaternions
    const float* rotation_r;  // [n,4]
    const int* idx;           // [n,k] neighbour list (fdgs_rigid_neighbours)
    const float* weight;      // [n,k]
    const int* in_offsets;    // [n+1]
    const int* in_edges;      // [n*k]
    float* velocity;          // [n,3] written by the forward, read by the backward
};
size_t rigid_scratch_bytes(int n, int k);
cudaError_t launch_rigid_neighbours(int n, int k, const int* idx, const float* dist2, char* scratch, float* weight,
                                    int* in_offsets, int* in_edges, cudaStream_t stream);
cudaError_t launch_rigid_forward(const RigidParams& p, char* scratch, float* loss_rigid, float* loss_motion, cudaStream_t stream);
cudaError_t launch_rigid_backward(const RigidParams& p, const float* grad_rigid, const float* grad_motion, float* dL_dscaling,
                                  float* dL_dscaling_t, float* dL_drotation, float* dL_drotation_r, cudaStream_t stream);

// evaluation metrics: L1, PSNR, SSIM, MS-SSIM (metrics.cu; the arguments are validated by fdgs_api.cu)
size_t metrics_scratch_bytes(int B, int C, int H, int W);
cudaError_t launch_image_metrics(const fdgs_metrics_args& a, char* scratch, cudaStream_t stream);

cudaError_t launch_mark_visible(int P, const float* means3D, const float* viewmatrix, unsigned char* present,
                                cudaStream_t stream);

// ---- densification surgery and statistics (densify.cu; the arguments are validated by fdgs_api.cu) ---------------
size_t densify_scratch_bytes(long long P);
cudaError_t launch_densify_plan(const fdgs_densify_args& a, char* scratch, int* totals, cudaStream_t stream);
// S = rows selected for splitting, child_kept = children kept per copy (the host copy of the plan's totals)
cudaError_t launch_densify_apply(const fdgs_densify_args& a, const char* scratch, long long S, long long child_kept,
                                 cudaStream_t stream);
cudaError_t launch_reset_opacity(long long P, float* opacity, float* m, float* v, cudaStream_t stream);
cudaError_t launch_densify_stats(long long P, int B, const float* pgrad, int stride, const float* vis, const int* radii,
                                 const float* tgrad, float* accum, float* denom, float* taccum, float* max_radii2D,
                                 const int* status, cudaStream_t stream);

// ---- environment-map sky (sky.cu) ------------------------------------------------------------------
struct SkyParams {
    const float* env_map;   // [3,Hm,Wm]
    int env_height, env_width;
    const float* c2w;       // [16] row-major camera-to-world
    const float* campos;    // [3]
    float fl_x, fl_y, cx, cy, radius;
    int W, H;
};
// out_sky [3,H,W]; miss_flag[0] = 1 if a ray misses the sphere (may be NULL)
cudaError_t launch_sky_fwd(const SkyParams& p, float* out_sky, int* miss_flag, cudaStream_t stream);
// dL_denv [3,Hm,Wm] += the bilinear taps' share of dL_dsky [3,H,W]
cudaError_t launch_sky_bwd(const SkyParams& p, const float* dL_dsky, float* dL_denv, cudaStream_t stream);
// B views of one image size, each camera from device tables (include/fdgs.h: fdgs_sky_batch_args)
struct SkyBatchParams {
    const float* env_map;     // [3,Hm,Wm]
    int env_height, env_width;
    const float* c2w;         // [B,16] row-major camera-to-world
    const float* campos;      // [B,3]
    const float* intrinsics;  // [B,4] fl_x, fl_y, cx, cy
    float radius;
    int W, H, B;
};
// out_sky [B,3,H,W]; miss_flag[0] = 1 if a ray of any view misses the sphere (may be NULL)
cudaError_t launch_sky_fwd_batch(const SkyBatchParams& b, float* out_sky, int* miss_flag, cudaStream_t stream);
// dL_denv [3,Hm,Wm] += every view's bilinear taps' share of dL_dsky [B,3,H,W]
cudaError_t launch_sky_bwd_batch(const SkyBatchParams& b, const float* dL_dsky, float* dL_denv, cudaStream_t stream);

}  // namespace fdgs
