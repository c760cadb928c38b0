// blend_bwd.cu -- per-tile back-to-front alpha blending (backward).
//
// Replaces the reference's renderCUDA<3> backward kernel (backward.cu:926-1137): same per-pixel
// back-to-front recurrences, same threshold decisions as the forward (power > 0, alpha < 1/255,
// the per-pixel n_contrib cut), but
//
//   * the 12 fp32 atomicAdd per contributing (pixel, Gaussian) PAIR of the reference
//     (backward.cu:1076,1091,1124-1134) become one tensor-core reduction over the warp's 32 pixels
//     per 8 Gaussians followed by one RED per per-Gaussian sum, and none at all for Gaussians whose
//     alpha >= 1/255 footprint misses the warp's 8x4 pixel rectangle (culled before any math);
//   * the work list is streamed with cp.async.bulk through the same mbarrier ring as the
//     forward, walking the tile's contiguous record range from the back, starting at the deepest
//     position any pixel of the tile actually reached (max n_contrib) instead of the list end;
//   * when the caller has no gradient for the flow / depth / alpha images (the reference's default
//     training loss only touches the colour image) the AUX = false instantiation drops their
//     recurrences;
//   * the mean / conic / opacity gradients leave as raw moment sums of w = G dL/dalpha about each
//     Gaussian's mean; geom_bwd_kernel (preprocess_bwd.cu) applies their linear map once per Gaussian.
#include "fdgs_internal.h"

namespace fdgs {
namespace {

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Per-pixel background image (BlendBwdParams::bg_image): the colour behind the last Gaussian becomes bg + bg_image[pix],
// which only changes the background term of dL/dalpha.  dL/dbg_image = (1 - alpha) dL/dpix with alpha = 1 - T_final,
// rounded as PyTorch rounds that expression; it is written here, before the tile loop, so that the pixels of tiles
// with an empty list get theirs too.
__device__ __forceinline__ void background_image_terms(const BlendBwdParams& p, int pix_id, int HW, float T_final, float gp0,
                                                       float gp1, float gp2, float& bg0, float& bg1, float& bg2) {
    if (p.bg_image) {
        bg0 += p.bg_image[0 * HW + pix_id];
        bg1 += p.bg_image[1 * HW + pix_id];
        bg2 += p.bg_image[2 * HW + pix_id];
    }
    if (p.dL_dbg_image) {
        const float w = __fsub_rn(1.0f, __fsub_rn(1.0f, T_final));
        p.dL_dbg_image[0 * HW + pix_id] = __fmul_rn(w, gp0);
        p.dL_dbg_image[1 * HW + pix_id] = __fmul_rn(w, gp1);
        p.dL_dbg_image[2 * HW + pix_id] = __fmul_rn(w, gp2);
    }
}

// view v of a batch (blockIdx.z): the same kernel on the view's slices of ranges, of every image and of the five
// per-Gaussian gradients (their rows keep the Gaussian indices [0, P) of the instance records)
__device__ __forceinline__ BlendBwdParams blend_bwd_view(BlendBwdParams p, int v) {
    const size_t HW = (size_t)p.W * p.H, P = (size_t)p.P;
    p.ranges += (size_t)v * p.grid_x * p.grid_y;
    p.final_T += v * HW;
    p.n_contrib += v * HW;
    p.dL_dpix += 3 * v * HW;
    if (p.dL_depths) p.dL_depths += v * HW;
    if (p.dL_masks) p.dL_masks += v * HW;
    if (p.dL_dpix_flow) p.dL_dpix_flow += 2 * v * HW;
    p.dL_dmean2D += 3 * v * P;
    p.dL_dconic += 4 * v * P;
    p.dL_dopacity += v * P;
    p.dL_dcolor += 3 * v * P;
    p.dL_dflows += 2 * v * P;
    if (p.bg_image) p.bg_image += 3 * v * HW;
    if (p.dL_dbg_image) p.dL_dbg_image += 3 * v * HW;
    return p;
}

// =====================================================================================================
// The kernel.  The blend is bound by instruction issue, so two things set its speed: how a (warp, Gaussian)
// step is evaluated and how the 32 per-pixel partial sums of a Gaussian are reduced.
//
//   * power(pixel) is a quadratic in the pixel offset, so the lane that culls an instance against the
//     warp's 8x4 rectangle also expands it about the rectangle centre (6 coefficients, pre-scaled by
//     log2 e) and parks them in a per-warp shared-memory slot; a step is then 2 LDS.128 + 5 FFMA +
//     1 MUFU.EX2 instead of the forward's per-pixel expression.  The polynomial
//     differs from the forward's exact power by a few 1e-6 (absolute); pairs whose alpha lands within
//     6e-7 of the 1/255 cut, or whose power is within 1e-4 of 0, and every pair of an instance whose
//     quadratic has large cancelling terms (thin rotated Gaussians far from their centre), are re-decided
//     with the forward's exact arithmetic from the staged record, so both passes agree on the contributors.
//   * every per-Gaussian gradient is a weighted sum over the warp's 32 pixels with weights that do not
//     depend on the Gaussian: the pixel's colour gradient (3) for  a1 = alpha*T, and the monomials
//     1, u, v, u^2, uv, v^2 of the pixel offset for  w = G * dL/dalpha.  So the reduction is a matrix
//     product  [weights 16 x 32] x [values 32 x 8 Gaussians]  and runs on the tensor cores
//     (mma.sync m16n8k8 tf32, fp32 accumulate; values split hi+lo so the result is fp32-accurate; the
//     monomials are exact in tf32, the colour gradients are split as well): 2 STS per step and one
//     flush per 8 Gaussians (16 LDS + 16 splits + 16 HMMA + moment re-centring).  AUX adds the depth and
//     flow gradients as rows of the a1-weighted tile.  The raw moments are re-centred on the
//     Gaussian's own mean per (warp, Gaussian) -- small numbers, no cancellation -- and accumulated with
//     RED; their constant linear map to dL/dmean2D, dL/dconic (conic and opacity factors) is applied
//     once per Gaussian by geom_bwd_kernel.
constexpr int B2_THREADS = 256;
constexpr int B2_WARPS = B2_THREADS / 32;
constexpr int B2_BATCH = 64;
constexpr int B2_COLS = 8;        // Gaussians per tensor-core flush (the n of m16n8k8)
constexpr int B2_LD = 36;         // padded row length of the value tiles (conflict-free fragment loads)

// Per-warp scratch.  Slots (one per surviving instance of the current 32-instance chunk, compacted,
// back-to-front) are plane-major so that the culling lanes' STS.128 are conflict-free:
//   s0 = c0, c1, c2, opacity          power = c0 + c1 u + c2 v + c3 u^2 + c4 uv + c5 v^2 (log2 units)
//   s1 = c3, c4, c5, list position | exact << 31
// a1 / w: the value tiles of the tensor-core reduction, [column][pixel], rows padded to 36 floats; the
// 4 padding floats of an a1 row hold that column's record plane q0 = x, y, -, gaussian id (for the flush).
struct __align__(16) B2Warp {
    float4 s0[32], s1[32];
    float a1[B2_COLS][B2_LD];
    float w[B2_COLS][B2_LD];
    float mom[B2_COLS][8];
};
template <int STAGES, bool ACOL_SMEM, bool AUX>
struct __align__(128) B2Smem {
    StageRec recs[STAGES][B2_BATCH];
    B2Warp warp[B2_WARPS];
    float amom[8][32];      // A fragments of the moment tile (identical for every warp): [2 s + h][lane]
    // A fragments of the a1-weighted tile (per warp) when not kept in registers.  !AUX: [2 s + h][lane], rows 0..2 =
    // hi parts of the colour gradient, rows 4..6 = lo parts (rows 8..15 of the m16 tile are zero).  AUX: [4 s + 2 h + part][lane],
    // rows 0..5 = hi parts of { colour r, g, b, depth, flow x, flow y } gradients (part 0), rows 8..13 = their lo parts (part 1).
    float acol[ACOL_SMEM ? B2_WARPS : 1][AUX ? 16 : 8][32];
    uint64_t full[STAGES];
    uint64_t empty[STAGES];
    unsigned int nmax;
};

// The forward's exact evaluation of one (pixel, Gaussian) pair (forward.cu:578-590 as compiled; see
// blend_fwd.cu): decides the pairs the polynomial cannot (rare, kept out of line).
__device__ __noinline__ float2 exact_pair(const StageRec* g, float pxf, float pyf) {
    const float4 q0 = g->q0, q1 = g->q1;
    const float dx = fsub(q0.x, pxf), dy = fsub(q0.y, pyf);
    const float power = ffma(ffma(dx, fmul(dx, q1.x), fmul(dy, fmul(dy, q1.z))), -0.5f, -fmul(dy, fmul(dx, q1.y)));
    const float G = expf(power);
    // .x = G, .y = opacity * G, or -1 when the forward skipped the pair (power > 0, or below the cull bound)
    return make_float2(G, (power > 0.0f || power < q0.z) ? -1.0f : fmul(q1.w, G));
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {
    // rows 8..15 of A are zero (a1 = a3 = 0)
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a0), "r"(0u), "r"(a2), "r"(0u), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_tf32_full(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t tf32_hi(float x) { return __float_as_uint(x) & 0xffffe000u; }
// the tensor core reads only the upper 19 bits of a tf32 operand, so the remainder needs no masking
__device__ __forceinline__ uint32_t tf32_lo(float x, uint32_t hi) { return __float_as_uint(x - __uint_as_float(hi)); }

template <int STAGES, bool ACOL_SMEM, bool AUX, bool BATCH>
__device__ __forceinline__ void blend_bwd2_body(const BlendBwdParams& p_) {
    // an lvalue on both sides: the single-view instantiation reads its parameters in place, no copy
    BlendBwdParams view_;
    if (BATCH) view_ = blend_bwd_view(p_, blockIdx.z);
    const BlendBwdParams& p = BATCH ? view_ : p_;
    static_assert(!AUX || ACOL_SMEM, "the AUX instantiation keeps its A fragments in shared memory");
    constexpr int B2_STAGES = STAGES;
    extern __shared__ __align__(128) unsigned char b2_smem_raw[];
    B2Smem<STAGES, ACOL_SMEM, AUX>& sm = *reinterpret_cast<B2Smem<STAGES, ACOL_SMEM, AUX>*>(b2_smem_raw);
    const int tile = blockIdx.y * p.grid_x + blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wx0 = blockIdx.x * TILE_X + (warp & 1) * 8;
    const int wy0 = blockIdx.y * TILE_Y + (warp >> 1) * 4;
    const int pix_x = wx0 + (lane & 7), pix_y = wy0 + (lane >> 3);
    const bool inside = pix_x < p.W && pix_y < p.H;
    const float pxf = (float)pix_x, pyf = (float)pix_y;
    const float bx0 = (float)wx0, bx1 = (float)(wx0 + 7), by0 = (float)wy0, by1 = (float)(wy0 + 3);
    const float rcx = (float)wx0 + 3.5f, rcy = (float)wy0 + 1.5f;            // rectangle centre
    const float u = (float)(lane & 7) - 3.5f, v = (float)(lane >> 3) - 1.5f;   // this pixel's offset from it
    const int HW = p.H * p.W;
    const int pix_id = pix_y * p.W + pix_x;
    B2Warp& ws = sm.warp[warp];

    const uint2 range = p.ranges[tile];
    const int n_list = (int)(range.y - range.x);
    const unsigned int my_last = inside ? p.n_contrib[pix_id] : 0u;
    const unsigned int wmax = __reduce_max_sync(0xffffffffu, my_last);

    if (threadIdx.x == 0) {
        for (int s = 0; s < B2_STAGES; ++s) {
            mbar_init(&sm.full[s], 1);
            mbar_init(&sm.empty[s], B2_WARPS);
        }
        sm.nmax = 0;
        mbar_fence_init();
    }
    __syncthreads();
    if (lane == 0 && wmax) atomicMax(&sm.nmax, wmax);
    __syncthreads();
    const int n = min(n_list, (int)sm.nmax);
    const int nb = (n + B2_BATCH - 1) / B2_BATCH;
    const StageRec* src = p.recs + range.x;

    int issued = 0;
    if (threadIdx.x == 0) {
        for (; issued < nb && issued < B2_STAGES; ++issued) {
            const int hi = n - issued * B2_BATCH, lo = max(0, hi - B2_BATCH);
            mbar_expect_tx(&sm.full[issued], (uint32_t)(hi - lo) * kStageRecBytes);
            bulk_g2s(&sm.recs[issued][0], src + lo, (uint32_t)(hi - lo) * kStageRecBytes, &sm.full[issued]);
        }
    }

    const float T_final = inside ? p.final_T[pix_id] : 0.f;
    float T = T_final;
    float acc_c0 = 0.f, acc_c1 = 0.f, acc_c2 = 0.f;
    float acc_f0 = 0.f, acc_f1 = 0.f, acc_d = 0.f, acc_m = 0.f;   // AUX only
    float gp0 = 0.f, gp1 = 0.f, gp2 = 0.f;
    float gf0 = 0.f, gf1 = 0.f, gd = 0.f, gm = 0.f;               // AUX only
    if (inside) {
        gp0 = p.dL_dpix[0 * HW + pix_id];
        gp1 = p.dL_dpix[1 * HW + pix_id];
        gp2 = p.dL_dpix[2 * HW + pix_id];
        if (AUX) {
            if (p.dL_dpix_flow) { gf0 = p.dL_dpix_flow[0 * HW + pix_id]; gf1 = p.dL_dpix_flow[1 * HW + pix_id]; }
            if (p.dL_depths) gd = p.dL_depths[pix_id];
            if (p.dL_masks) gm = p.dL_masks[pix_id];
        }
    }
    float bg0 = p.background[0], bg1 = p.background[1], bg2 = p.background[2];
    if (inside) background_image_terms(p, pix_id, HW, T_final, gp0, gp1, gp2, bg0, bg1, bg2);
    const float tb = -T_final * (bg0 * gp0 + bg1 * gp1 + bg2 * gp2);

    // ---- constant A fragments (m16n8k8: a0 = A[g][t], a2 = A[g][t + 4], g = lane / 4, t = lane % 4; k = pixel) ----
    // colour tile: rows 0..2 = hi part of the colour gradient of pixel k, rows 4..6 = its lo part
    // moment tile: rows 0..5 = 1, u, v, u^2, uv, v^2 of pixel k (half-integers: exact in tf32)
    const int fg = lane >> 2, ft = lane & 3;
    uint32_t acol[4][2];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int srcl = 8 * s + ft + 4 * h;
            const float v0 = __shfl_sync(0xffffffffu, gp0, srcl);
            const float v1 = __shfl_sync(0xffffffffu, gp1, srcl);
            const float v2 = __shfl_sync(0xffffffffu, gp2, srcl);
            if (AUX) {
                // row fg of the 6 weights; hi part -> rows 0..7 (a0 / a2), lo part -> rows 8..15 (a1 / a3)
                const float v3 = __shfl_sync(0xffffffffu, gd, srcl);
                const float v4 = __shfl_sync(0xffffffffu, gf0, srcl);
                const float v5 = __shfl_sync(0xffffffffu, gf1, srcl);
                const float val = (fg == 0) ? v0 : (fg == 1) ? v1 : (fg == 2) ? v2 : (fg == 3) ? v3 : (fg == 4) ? v4 : (fg == 5) ? v5 : 0.f;
                const uint32_t hi = tf32_hi(val);
                sm.acol[warp][(AUX ? 4 : 0) * s + 2 * h + 0][lane] = __uint_as_float(hi);
                sm.acol[warp][(AUX ? 4 : 0) * s + 2 * h + 1][lane] = __uint_as_float(tf32_lo(val, hi));
                acol[s][h] = 0u;
            } else {
                const int ch = fg & 3;
                const float val = (ch == 0) ? v0 : (ch == 1) ? v1 : (ch == 2) ? v2 : 0.f;
                const uint32_t hi = tf32_hi(val);
                acol[s][h] = (fg < 4) ? hi : tf32_lo(val, hi);
                if (ACOL_SMEM) sm.acol[warp][2 * s + h][lane] = __uint_as_float(acol[s][h]);
            }
            const float ku = (float)(ft + 4 * h) - 3.5f, kv = (float)s - 1.5f;
            const float mono = (fg == 0) ? 1.f : (fg == 1) ? ku : (fg == 2) ? kv : (fg == 3) ? ku * ku
                             : (fg == 4) ? ku * kv : (fg == 5) ? kv * kv : 0.f;
            if (warp == 0) sm.amom[2 * s + h][lane] = mono;
        }
    }
    __syncthreads();

    int ncol = 0;   // filled columns of the value tiles (warp-uniform)
    float* const a1_lane = &ws.a1[0][lane];
    float* const w_lane = &ws.w[0][lane];

    // One flush: reduce the columns of ws.a1 / ws.w over the 32 pixels on the tensor cores, re-centre the
    // moments on each Gaussian's mean, accumulate with RED.
    auto flush = [&](int cols) {
        __syncwarp();
        float c1[4] = {0.f, 0.f, 0.f, 0.f}, c2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            const float x0 = ws.a1[fg][8 * s + ft], x1 = ws.a1[fg][8 * s + ft + 4];
            const float y0 = ws.w[fg][8 * s + ft], y1 = ws.w[fg][8 * s + ft + 4];
            const uint32_t x0h = tf32_hi(x0), x1h = tf32_hi(x1), y0h = tf32_hi(y0), y1h = tf32_hi(y1);
            if (AUX) {
                const uint32_t f0 = __float_as_uint(sm.acol[warp][(AUX ? 4 : 0) * s + 0][lane]);   // a0: hi, pixels ft
                const uint32_t f1 = __float_as_uint(sm.acol[warp][(AUX ? 4 : 0) * s + 1][lane]);   // a1: lo, pixels ft
                const uint32_t f2 = __float_as_uint(sm.acol[warp][(AUX ? 4 : 0) * s + 2][lane]);   // a2: hi, pixels ft + 4
                const uint32_t f3 = __float_as_uint(sm.acol[warp][(AUX ? 4 : 0) * s + 3][lane]);   // a3: lo, pixels ft + 4
                mma_tf32_full(c1, f0, f1, f2, f3, x0h, x1h);
                mma_tf32_full(c1, f0, f1, f2, f3, tf32_lo(x0, x0h), tf32_lo(x1, x1h));
            } else {
                const uint32_t ac0 = ACOL_SMEM ? __float_as_uint(sm.acol[warp][2 * s][lane]) : acol[s][0];
                const uint32_t ac1 = ACOL_SMEM ? __float_as_uint(sm.acol[warp][2 * s + 1][lane]) : acol[s][1];
                mma_tf32(c1, ac0, ac1, x0h, x1h);
                mma_tf32(c1, ac0, ac1, tf32_lo(x0, x0h), tf32_lo(x1, x1h));
            }
            const uint32_t am0 = __float_as_uint(sm.amom[2 * s][lane]), am1 = __float_as_uint(sm.amom[2 * s + 1][lane]);
            mma_tf32(c2, am0, am1, y0h, y1h);
            mma_tf32(c2, am0, am1, tf32_lo(y0, y0h), tf32_lo(y1, y1h));
        }
        // c1[0], c1[1]: row fg of the colour tile for columns 2 ft, 2 ft + 1; add the lo rows (fg + 4) to the hi rows
        if (AUX) {
            // rows fg (hi) and fg + 8 (lo) of the a1-weighted tile sit in the same lane
            c1[0] += c1[2];
            c1[1] += c1[3];
        } else {
            c1[0] += __shfl_xor_sync(0xffffffffu, c1[0], 16);
            c1[1] += __shfl_xor_sync(0xffffffffu, c1[1], 16);
        }
        if (fg < 6) {
            ws.mom[2 * ft][fg] = c2[0];
            ws.mom[2 * ft + 1][fg] = c2[1];
        }
        if (AUX) {
            if (fg < 6) {
                // rows: colour r, g, b -> dL_dcolor; depth -> dL_dmean2D.z (backward.cu:1091); flow x, y -> dL_dflows
                float* const base = (fg < 3) ? p.dL_dcolor + fg : (fg == 3) ? p.dL_dmean2D + 2 : p.dL_dflows + (fg - 4);
                const size_t mul = (fg < 4) ? 3 : 2;
                if (2 * ft < cols) atomicAdd(base + (size_t)__float_as_uint(ws.a1[2 * ft][35]) * mul, c1[0]);
                if (2 * ft + 1 < cols) atomicAdd(base + (size_t)__float_as_uint(ws.a1[2 * ft + 1][35]) * mul, c1[1]);
            }
        } else if (fg < 3) {
            if (2 * ft < cols) atomicAdd(p.dL_dcolor + (size_t)__float_as_uint(ws.a1[2 * ft][35]) * 3 + fg, c1[0]);
            if (2 * ft + 1 < cols) atomicAdd(p.dL_dcolor + (size_t)__float_as_uint(ws.a1[2 * ft + 1][35]) * 3 + fg, c1[1]);
        }
        __syncwarp();
        // lane = 4 * column + j: j = 0 -> W00, W10; j = 1 -> W01, W20; j = 2 -> W11, W02   (W_ab = sum w dx^a dy^b, d = mean - pixel)
        const int col = lane >> 2, j = lane & 3;
        if (col < cols && j < 3) {
            const float4 m03 = *reinterpret_cast<const float4*>(&ws.mom[col][0]);   // m00 m10 m01 m20
            const float2 m45 = *reinterpret_cast<const float2*>(&ws.mom[col][4]);   // m11 m02
            const float4 meta = *reinterpret_cast<const float4*>(&ws.a1[col][32]);
            const float X = meta.x - rcx, Y = meta.y - rcy;   // mean - rectangle centre
            const size_t gid = __float_as_uint(meta.w);
            const float W10 = fmaf(X, m03.x, -m03.y), W01 = fmaf(Y, m03.x, -m03.z);
            if (j == 0) {
                atomicAdd(p.dL_dopacity + gid, m03.x);
                atomicAdd(p.dL_dmean2D + gid * 3 + 0, W10);
            } else if (j == 1) {
                // sum w (X - u)^2 = X (X m00 - m10) - (X m10 - m20)
                atomicAdd(p.dL_dmean2D + gid * 3 + 1, W01);
                atomicAdd(p.dL_dconic + gid * 4 + 0, fmaf(X, W10, -fmaf(X, m03.y, -m03.w)));
            } else {
                // sum w (X - u)(Y - v) = Y (X m00 - m10) - (X m01 - m11);  sum w (Y - v)^2 likewise
                atomicAdd(p.dL_dconic + gid * 4 + 1, fmaf(Y, W10, -fmaf(X, m03.z, -m45.x)));
                atomicAdd(p.dL_dconic + gid * 4 + 3, fmaf(Y, W01, -fmaf(Y, m03.z, -m45.y)));
            }
        }
        __syncwarp();
    };

    constexpr float kLog2e = 1.4426950408889634f;
    for (int b = 0; b < nb; ++b) {
        const int s = b % B2_STAGES;
        const uint32_t ph = (uint32_t)(b / B2_STAGES) & 1u;
        const int hi = n - b * B2_BATCH, lo = max(0, hi - B2_BATCH), cnt = hi - lo;
        mbar_wait_backoff(&sm.full[s], ph);
        if ((unsigned)lo < wmax) {
            const StageRec* st = sm.recs[s];
            for (int r0 = ((cnt - 1) >> 5) << 5; r0 >= 0; r0 -= 32) {
                const int j = r0 + lane;
                bool rel = false;
                float4 a, c, e;
                if (j < cnt && (unsigned)(lo + j) < wmax) {
                    a = st[j].q0;
                    c = st[j].q1;
                    e = st[j].q3;
                    rel = rect_may_contribute(a.x, a.y, c.x, c.y, c.z, a.z, e.z, e.w, bx0, bx1, by0, by1);
                }
                const uint32_t m = __ballot_sync(0xffffffffu, rel);
                if (m == 0u) continue;
                if (rel) {
                    // back-to-front: the survivor with the highest list position goes to slot 0
                    const int rank = __popc(m >> lane) - 1;
                    const float X = a.x - rcx, Y = a.y - rcy;
                    const float AX = c.x * X, BY = c.y * Y, CY = c.z * Y, BX = c.y * X;
                    const float t0 = AX * X, t1 = CY * Y, t2 = BX * Y;
                    // pmin = -inf marks NaN / non-PD inputs; a large cancellation between the three terms of
                    // the quadratic (a thin, rotated Gaussian far from its centre) makes the expansion's rounding
                    // differ from the forward's by more than the threshold band: both are evaluated exactly
                    const bool exact = !(a.z > -3.0e38f) || !(fabsf(t0) + fabsf(t1) + 2.f * fabsf(t2) < 128.f);
                    ws.s0[rank] = make_float4(-(0.5f * (t0 + t1) + t2) * kLog2e, (AX + BY) * kLog2e, (CY + BX) * kLog2e, c.w);
                    ws.s1[rank] = make_float4(-0.5f * c.x * kLog2e, -c.y * kLog2e, -0.5f * c.z * kLog2e,
                                              __uint_as_float((unsigned)(lo + j) | (exact ? 0x80000000u : 0u)));
                }
                __syncwarp();
                const int nsurv = __popc(m);
                for (int i = 0; i < nsurv; ++i) {
                    const float4 s0 = ws.s0[i];
                    const float4 s1 = ws.s1[i];
                    const float pw = fmaf(u, fmaf(s1.x, u, fmaf(s1.y, v, s0.y)), fmaf(v, fmaf(s1.z, v, s0.z), s0.x));
                    const unsigned int posbits = __float_as_uint(s1.w);
                    const StageRec* rec = st + ((posbits & 0x7fffffffu) - (unsigned)lo);   // staged record of this slot
                    bool contrib = (posbits & 0x7fffffffu) < my_last;
                    float G_c = ex2_approx(pw);
                    float og = s0.w * G_c;
                    if (contrib && (fabsf(og - 0.00392156886f) < 6.0e-7f || pw > -1.0e-4f || (int)posbits < 0)) {
                        // too close to a threshold for the polynomial (the alpha cut, or power > 0 which the
                        // forward skips), or an instance flagged for exact evaluation: the forward's arithmetic decides
                        const float2 ex = exact_pair(rec, pxf, pyf);
                        G_c = ex.x;
                        og = ex.y;
                    }
                    const float alpha = fminf(og, 0.99f);
                    contrib = contrib && !(alpha < 1.0f / 255.0f);
                    if (!__any_sync(0xffffffffu, contrib)) continue;
                    float a1v = 0.f, wv = 0.f;
                    if (contrib) {
                        const float4 s2 = rec->q2;   // r, g, b, depth
                        const float om = 1.f - alpha;
                        float rom;
                        asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rom) : "f"(om));
                        T = T * rom;
                        a1v = alpha * T;
                        const float d0 = s2.x - acc_c0, d1 = s2.y - acc_c1, d2 = s2.z - acc_c2;
                        float dL_dalpha = d0 * gp0;
                        dL_dalpha = fmaf(d1, gp1, dL_dalpha);
                        dL_dalpha = fmaf(d2, gp2, dL_dalpha);
                        acc_c0 = fmaf(alpha, d0, acc_c0);
                        acc_c1 = fmaf(alpha, d1, acc_c1);
                        acc_c2 = fmaf(alpha, d2, acc_c2);
                        if (AUX) {
                            // flow / depth / alpha-image recurrences, backward.cu:1078-1102
                            const float2 fl = *reinterpret_cast<const float2*>(&rec->q3);
                            const float e0 = fl.x - acc_f0, e1 = fl.y - acc_f1, dd = s2.w - acc_d, dm = 1.0f - acc_m;
                            dL_dalpha = fmaf(e0, gf0, dL_dalpha);
                            dL_dalpha = fmaf(e1, gf1, dL_dalpha);
                            dL_dalpha = fmaf(dd, gd, dL_dalpha);
                            dL_dalpha = fmaf(dm, gm, dL_dalpha);
                            acc_f0 = fmaf(alpha, e0, acc_f0);
                            acc_f1 = fmaf(alpha, e1, acc_f1);
                            acc_d = fmaf(alpha, dd, acc_d);
                            acc_m = fmaf(alpha, dm, acc_m);
                        }
                        dL_dalpha = fmaf(tb, rom, dL_dalpha * T);
                        wv = G_c * dL_dalpha;
                    }
                    a1_lane[ncol * B2_LD] = a1v;
                    w_lane[ncol * B2_LD] = wv;
                    if (lane == 0) *reinterpret_cast<float4*>(&ws.a1[ncol][32]) = rec->q0;   // x, y, -, gaussian id
                    if (++ncol == B2_COLS) {
                        flush(B2_COLS);
                        ncol = 0;
                    }
                }
                __syncwarp();   // every lane is done with the slots before the next chunk overwrites them
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.empty[s]);
        if (threadIdx.x == 0 && issued < nb) {
            mbar_wait(&sm.empty[s], ph);
            const int nhi = n - issued * B2_BATCH, nlo = max(0, nhi - B2_BATCH);
            mbar_expect_tx(&sm.full[s], (uint32_t)(nhi - nlo) * kStageRecBytes);
            bulk_g2s(&sm.recs[s][0], src + nlo, (uint32_t)(nhi - nlo) * kStageRecBytes, &sm.full[s]);
            ++issued;
        }
    }
    if (ncol > 0) flush(ncol);
}

template <int STAGES, bool ACOL_SMEM, bool AUX>
__global__ void __launch_bounds__(B2_THREADS, (ACOL_SMEM && !AUX) ? 4 : 3) blend_bwd2_kernel(const BlendBwdParams p_) {
    blend_bwd2_body<STAGES, ACOL_SMEM, AUX, false>(p_);
}

// the batched entry (fdgs_forward_batch / fdgs_backward_batch): one view per blockIdx.z
template <int STAGES, bool ACOL_SMEM, bool AUX>
__global__ void __launch_bounds__(B2_THREADS, (ACOL_SMEM && !AUX) ? 4 : 3) blend_bwd2_batch_kernel(const BlendBwdParams p_) {
    blend_bwd2_body<STAGES, ACOL_SMEM, AUX, true>(p_);
}

}  // namespace

template <bool BATCH>
static cudaError_t blend_bwd(const BlendBwdParams& p, cudaStream_t stream) {
    const dim3 grid(p.grid_x, p.grid_y, BATCH ? p.views : 1);
    const bool aux = p.dL_depths || p.dL_masks || p.dL_dpix_flow;
    if (!aux) {
        // colour fragments in shared memory + 3 stages: 64 registers, 53 KB -> 4 CTAs / SM.  (Keeping them in
        // registers costs 80 registers -> 3 CTAs / SM and measured 8 % slower.)
        const auto k = BATCH ? blend_bwd2_batch_kernel<3, true, false> : blend_bwd2_kernel<3, true, false>;
        static PerDeviceOnce once;
        cudaError_t e = ensure_dynamic_smem(k, (int)sizeof(B2Smem<3, true, false>), once);
        if (e != cudaSuccess) return e;
        k<<<grid, B2_THREADS, sizeof(B2Smem<3, true, false>), stream>>>(p);
    } else {
        // upstream gradients for the depth / alpha / flow images too: 6 a1-weighted rows (16-row A tile), 3 CTAs / SM
        const auto k = BATCH ? blend_bwd2_batch_kernel<3, true, true> : blend_bwd2_kernel<3, true, true>;
        static PerDeviceOnce once_aux;
        cudaError_t e = ensure_dynamic_smem(k, (int)sizeof(B2Smem<3, true, true>), once_aux);
        if (e != cudaSuccess) return e;
        k<<<grid, B2_THREADS, sizeof(B2Smem<3, true, true>), stream>>>(p);
    }
    return cudaGetLastError();
}

cudaError_t launch_blend_bwd(const BlendBwdParams& p, cudaStream_t stream) {
    return p.views > 0 ? blend_bwd<true>(p, stream) : blend_bwd<false>(p, stream);
}

}  // namespace fdgs
