// blend_fwd.cu -- per-tile front-to-back alpha blending (forward).
//
// Replaces the reference's renderCUDA<3> forward kernel (forward.cu:501-626).  Same tile
// decomposition (16x16 pixels per CTA, one thread per pixel), same per-pixel arithmetic in the
// same order (results are bit-identical to the reference kernel as compiled by nvcc), but a
// different execution structure:
//
//   * the tile's work list is a contiguous array of 64-byte instance records (binning.cu), so it
//     is streamed into shared memory with cp.async.bulk (TMA 1-D) through a 3-stage
//     full/empty mbarrier ring -- no __syncthreads in the loop, no index chasing, and the colour
//     / depth / flow payload arrives with the geometry instead of being re-read from global
//     memory per contributing pixel (reference: forward.cu:600-604);
//   * each warp owns an 8x4 pixel footprint and first culls every batch of 32 instances against
//     that footprint (one instance per lane, one ballot), then walks only the surviving
//     instances.  The cull box is the exact alpha >= 1/255 extent of the Gaussian, so skipped
//     (pixel, Gaussian) pairs are pairs the reference would have rejected anyway;
//   * pairs whose power is below log(1/(255*opacity)) skip expf() (same argument).
//
// In training (single view) the kernel also writes the zero rows of the dense SH gradient -- the rows of the Gaussians
// the view does not render, about 2/3 of the 1.15 GB tensor at 2M Gaussians.  The blend is bound by instruction issue
// and leaves DRAM nearly idle, so these rows go out as bulk (TMA) stores from a zeroed shared block, each CTA a stripe
// of rows, issued before the CTA blends and drained when it retires; the SH backward then streams only rendered rows.
#include "fdgs_internal.h"

namespace fdgs {
namespace {

constexpr int BF_THREADS = 256;
constexpr int BF_WARPS = BF_THREADS / 32;
constexpr int BF_BATCH = 128;
constexpr int BF_STAGES = 3;
constexpr int BF_ZERO_BYTES = 576;   // zero source of the bulk stores: one dL_dsh row of 48 coefficients

struct __align__(128) BlendFwdSmem {
    StageRec recs[BF_STAGES][BF_BATCH];
    float4 zero[BF_ZERO_BYTES / 16];
    uint64_t full[BF_STAGES];
    uint64_t empty[BF_STAGES];
    int done_warps;
};

// floats [0, n) at dst set to zero: the 16-byte-aligned interior as bulk stores from the zeroed shared block (row
// sizes and offsets of split rows are not multiples of 16 bytes), the few floats around it as plain stores
__device__ __forceinline__ void zero_row(float* dst, int n, const float4* zsrc) {
    float* end = dst + n;
    float* a = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(dst) + 15) & ~uintptr_t(15));
    float* b = reinterpret_cast<float*>(reinterpret_cast<uintptr_t>(end) & ~uintptr_t(15));
    if (a >= b) a = b = end;
    for (float* q = dst; q < a; ++q) *q = 0.f;
    for (float* q = b; q < end; ++q) *q = 0.f;
    for (char* q = reinterpret_cast<char*>(a); q < reinterpret_cast<char*>(b); q += BF_ZERO_BYTES)
        bulk_s2g(q, zsrc, (uint32_t)min(BF_ZERO_BYTES, (int)(reinterpret_cast<char*>(b) - q)));
}

// this CTA's stripe of SH gradient rows: every row of a Gaussian the view does not render (sh_bwd_kernel's test)
__device__ __forceinline__ void zero_unrendered_rows(const BlendFwdParams& p, int tile, const float4* zsrc) {
    const long long r0 = (long long)tile * p.zero_stripe;
    const long long r1 = min((long long)p.P, r0 + p.zero_stripe);
    bool issued = false;
    for (long long g = r0 + threadIdx.x; g < r1; g += BF_THREADS) {
        if (p.radii[g] > 0 && p.tiles_touched[g] != 0u) continue;
        zero_row(p.zero_rows[0] + g * p.zero_row_floats[0], p.zero_row_floats[0], zsrc);
        if (p.zero_rows[1]) zero_row(p.zero_rows[1] + g * p.zero_row_floats[1], p.zero_row_floats[1], zsrc);
        issued = true;
    }
    if (issued) bulk_commit();
}

// view v of a batch (blockIdx.z): the same kernel on the view's slices of ranges and of every image
__device__ __forceinline__ BlendFwdParams blend_fwd_view(BlendFwdParams p, int v) {
    const size_t HW = (size_t)p.W * p.H;
    p.ranges += (size_t)v * p.grid_x * p.grid_y;
    p.final_T += v * HW;
    p.n_contrib += v * HW;
    p.out_color += 3 * v * HW;
    p.out_flow += 2 * v * HW;
    p.out_depth += v * HW;
    p.out_T += v * HW;
    if (p.bg_image) p.bg_image += 3 * v * HW;
    return p;
}

template <bool BATCH>
__device__ __forceinline__ void blend_fwd_body(const BlendFwdParams& p_) {
    __shared__ BlendFwdSmem sm;
    // an lvalue on both sides: the single-view instantiation reads its parameters in place, no copy
    BlendFwdParams view_;
    if (BATCH) view_ = blend_fwd_view(p_, blockIdx.z);
    const BlendFwdParams& p = BATCH ? view_ : p_;
    const int tile = blockIdx.y * p.grid_x + blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // 8x4 footprint per warp: warps tile the 16x16 block as 2 (x) by 4 (y)
    const int wx0 = blockIdx.x * TILE_X + (warp & 1) * 8;
    const int wy0 = blockIdx.y * TILE_Y + (warp >> 1) * 4;
    const int pix_x = wx0 + (lane & 7), pix_y = wy0 + (lane >> 3);
    const bool inside = pix_x < p.W && pix_y < p.H;
    const float pxf = (float)pix_x, pyf = (float)pix_y;
    const float bx0 = (float)wx0, bx1 = (float)(wx0 + 7), by0 = (float)wy0, by1 = (float)(wy0 + 3);

    const uint2 range = p.ranges[tile];
    const int n = (int)(range.y - range.x);
    const int nb = (n + BF_BATCH - 1) / BF_BATCH;
    const StageRec* src = p.recs + range.x;
    const bool zero_rows = !BATCH && p.zero_rows[0] != nullptr;

    if (threadIdx.x == 0) {
        for (int s = 0; s < BF_STAGES; ++s) {
            mbar_init(&sm.full[s], 1);
            mbar_init(&sm.empty[s], BF_WARPS);
        }
        sm.done_warps = 0;
        mbar_fence_init();
    }
    if (zero_rows && threadIdx.x < BF_ZERO_BYTES / 16) {
        sm.zero[threadIdx.x] = make_float4(0.f, 0.f, 0.f, 0.f);
        fence_async_smem();
    }
    __syncthreads();

    int issued = 0;
    if (threadIdx.x == 0) {
        for (; issued < nb && issued < BF_STAGES; ++issued) {
            const int cnt = min(BF_BATCH, n - issued * BF_BATCH);
            mbar_expect_tx(&sm.full[issued], (uint32_t)cnt * kStageRecBytes);
            bulk_g2s(&sm.recs[issued][0], src + (size_t)issued * BF_BATCH, (uint32_t)cnt * kStageRecBytes, &sm.full[issued]);
        }
    }
    if (zero_rows) zero_unrendered_rows(p, tile, sm.zero);

    float T = 1.0f;
    float C0 = 0.f, C1 = 0.f, C2 = 0.f, F0 = 0.f, F1 = 0.f, Dp = 0.f;
    uint32_t last_contributor = 0;
    bool done = !inside;
    bool warp_done = false;
    volatile int* done_warps = &sm.done_warps;

    int b = 0;
    for (; b < nb; ++b) {
        const int s = b % BF_STAGES;
        const uint32_t ph = (uint32_t)(b / BF_STAGES) & 1u;
        // Wait for batch b -- or for the whole tile to finish.  Once every warp is done the producer
        // stops refilling (below), so a warp that ran ahead must not wait for a batch that will never
        // come; lane 0 polls both conditions and the warp leaves together.
        bool stop = false;
        if (lane == 0) {
            while (!mbar_try_wait(&sm.full[s], ph)) {
                if (*done_warps == BF_WARPS) { stop = true; break; }
            }
            if (!stop && *done_warps == BF_WARPS) stop = true;
        }
        if (__any_sync(0xffffffffu, stop)) break;
        mbar_wait(&sm.full[s], ph);   // already complete: gives every lane the acquire on the batch
        if (!warp_done) {
            const int cnt = min(BF_BATCH, n - b * BF_BATCH);
            const StageRec* st = sm.recs[s];
            for (int r0 = 0; r0 < cnt; r0 += 32) {
                const int j = r0 + lane;
                bool rel = false;
                if (j < cnt) {
                    const float4 a = st[j].q0;
                    const float4 c = st[j].q1;
                    const float4 e = st[j].q3;
                    rel = rect_may_contribute(a.x, a.y, c.x, c.y, c.z, a.z, e.z, e.w, bx0, bx1, by0, by1);
                }
                uint32_t m = __ballot_sync(0xffffffffu, rel);
                while (m) {
                    const int k = __ffs(m) - 1;
                    m &= m - 1;
                    const StageRec* g = st + (r0 + k);
                    const float4 q0 = g->q0;   // x, y, pmin, -
                    const float4 q1 = g->q1;   // A, B, C, opacity
                    // reference: forward.cu:578-581 (contraction as compiled)
                    const float dx = fsub(q0.x, pxf);
                    const float dy = fsub(q0.y, pyf);
                    const float power =
                        ffma(ffma(dx, fmul(dx, q1.x), fmul(dy, fmul(dy, q1.z))), -0.5f, -fmul(dy, fmul(dx, q1.y)));
                    if (done || power > 0.0f || power < q0.z) continue;
                    const float alpha = fminf(fmul(q1.w, expf(power)), 0.99f);
                    if (alpha < 1.0f / 255.0f) continue;
                    const float test_T = fmul(T, fsub(1.0f, alpha));
                    if (test_T < 0.0001f) {
                        done = true;
                        continue;
                    }
                    const float4 q2 = g->q2;   // r, g, b, depth
                    const float4 q3 = g->q3;   // flow x, flow y, ex, ey
                    C0 = ffma(T, fmul(alpha, q2.x), C0);
                    C1 = ffma(T, fmul(alpha, q2.y), C1);
                    C2 = ffma(T, fmul(alpha, q2.z), C2);
                    F0 = ffma(T, fmul(alpha, q3.x), F0);
                    F1 = ffma(T, fmul(alpha, q3.y), F1);
                    Dp = ffma(T, fmul(alpha, q2.w), Dp);
                    T = test_T;
                    last_contributor = (uint32_t)(b * BF_BATCH + r0 + k + 1);
                }
                if (__all_sync(0xffffffffu, done)) {
                    warp_done = true;
                    if (lane == 0) atomicAdd(&sm.done_warps, 1);
                    break;
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.empty[s]);
        if (threadIdx.x == 0 && issued < nb) {
            // refill this stage with batch `issued` once every warp has released it
            bool go = true;
            while (!mbar_try_wait(&sm.empty[s], ph)) {
                if (*done_warps == BF_WARPS) { go = false; break; }
            }
            if (go) {
                const int cnt = min(BF_BATCH, n - issued * BF_BATCH);
                mbar_expect_tx(&sm.full[s], (uint32_t)cnt * kStageRecBytes);
                bulk_g2s(&sm.recs[s][0], src + (size_t)issued * BF_BATCH, (uint32_t)cnt * kStageRecBytes, &sm.full[s]);
                ++issued;
            }
        }
    }
    // drain bulk copies that were issued but never consumed (early exit) before the CTA retires
    if (threadIdx.x == 0) {
        for (int j = b; j < issued; ++j) mbar_wait(&sm.full[j % BF_STAGES], (uint32_t)(j / BF_STAGES) & 1u);
    }

    if (inside) {
        const int pix_id = pix_y * p.W + pix_x;
        const int HW = p.H * p.W;
        p.final_T[pix_id] = T;
        p.out_T[pix_id] = T;
        p.n_contrib[pix_id] = last_contributor;
        float o0 = ffma(T, p.background[0], C0), o1 = ffma(T, p.background[1], C1), o2 = ffma(T, p.background[2], C2);
        if (p.bg_image) {
            // out + (1 - alpha) * bg_image with alpha = 1 - T, rounded step by step exactly as PyTorch evaluates that
            // expression on the returned images (no contraction into an FMA)
            const float w = __fsub_rn(1.0f, __fsub_rn(1.0f, T));
            o0 = __fadd_rn(o0, __fmul_rn(w, p.bg_image[0 * HW + pix_id]));
            o1 = __fadd_rn(o1, __fmul_rn(w, p.bg_image[1 * HW + pix_id]));
            o2 = __fadd_rn(o2, __fmul_rn(w, p.bg_image[2 * HW + pix_id]));
        }
        p.out_color[0 * HW + pix_id] = o0;
        p.out_color[1 * HW + pix_id] = o1;
        p.out_color[2 * HW + pix_id] = o2;
        p.out_flow[0 * HW + pix_id] = F0;
        p.out_flow[1 * HW + pix_id] = F1;
        p.out_depth[pix_id] = Dp;
    }
    // the zero block must outlive the bulk stores that read it
    if (zero_rows) bulk_wait_all();
}

__global__ void __launch_bounds__(BF_THREADS) blend_fwd_kernel(const BlendFwdParams p_) {
    blend_fwd_body<false>(p_);
}

// the batched entry (fdgs_forward_batch / fdgs_backward_batch): one view per blockIdx.z
__global__ void __launch_bounds__(BF_THREADS) blend_fwd_batch_kernel(const BlendFwdParams p_) {
    blend_fwd_body<true>(p_);
}

}  // namespace

cudaError_t launch_blend_fwd(const BlendFwdParams& p, cudaStream_t stream) {
    if (p.zero_rows[0] != nullptr && (p.views > 0 || p.zero_stripe <= 0 || !p.radii || !p.tiles_touched))
        return cudaErrorInvalidValue;
    if (p.views > 0) blend_fwd_batch_kernel<<<dim3(p.grid_x, p.grid_y, p.views), BF_THREADS, 0, stream>>>(p);
    else blend_fwd_kernel<<<dim3(p.grid_x, p.grid_y, 1), BF_THREADS, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace fdgs
