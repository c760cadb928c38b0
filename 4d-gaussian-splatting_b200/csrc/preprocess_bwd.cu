// preprocess_bwd.cu -- per-Gaussian backward preprocessing.
//
// Replaces the reference's two backward preprocessing kernels -- computeCov2DCUDA
// (backward.cu:486-617) and preprocessCUDA<3> (backward.cu:839-923) with its helpers
// computeColorFromSH (:20-139), computeColorFromSH_4D (:144-481), computeCov3D (:621-684),
// computeCov3D_conditional (:689-834).  Two kernels here, split by what bounds them:
//
//   sh_bwd_kernel    HBM-bound.  Reads the 12*M-byte SH row of every rendered Gaussian and writes
//                    the 12*M-byte dL_dsh row of EVERY Gaussian (zeros where not rendered, so the
//                    host never memsets the 1.15 GB tensor; reference: rasterize_points.cu:209) --
//                    or, when the forward's blend already zeroed the non-rendered rows
//                    (sh_rows_zeroed, blend_fwd.cu), the rendered rows only.
//                    Rows move with cp.async.bulk in both directions (global->shared on an
//                    mbarrier, shared->global as a bulk group); in shared memory a row is read and
//                    overwritten in place with conflict-free 128-bit accesses; only rendered rows
//                    occupy shared memory (block-level compaction), which keeps 5 CTAs per SM
//                    resident; zero rows are written with coalesced 16-byte stores.
//   geom_bwd_kernel  latency/ALU-bound.  Fuses computeCov2DCUDA with the projection and the
//                    3D / conditional-4D covariance chains, so dL_dcov3D and dL_dmeans never make
//                    a round trip through HBM; writes every row of the seven parameter-gradient
//                    tensors (zeros where not rendered; reference memsets them first,
//                    rasterize_points.cu:201-213).
//
// Bug-compatible with the reference where the bugs are observable (SURVEY.md section 8a quirks):
// dL_dsh[1] uses l0m0 in the 4D variant (backward.cu:190), the temporal derivative has no minus
// sign (:303,:384) and is overwritten, not accumulated, for deg_t > 1 (:403); the SH view
// direction is taken from the SHIFTED mean here (rasterizer_impl.cu:463) although the forward
// used the unshifted one.
#include "fdgs_internal.h"

namespace fdgs {
namespace {

constexpr int SB_THREADS = 128;   // SH kernel: Gaussians per CTA
constexpr int SB_CAP = 48;        // shared-memory row slots per CTA (rendered rows per round)
constexpr int GB_THREADS = 128;   // geometry kernel

__device__ __forceinline__ float3 dnormvdv3(float3 v, float3 dv) {   // auxiliary.h:108-118
    const float sum2 = v.x * v.x + v.y * v.y + v.z * v.z;
    const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
    float3 o;
    o.x = ((+sum2 - v.x * v.x) * dv.x - v.y * v.x * dv.y - v.z * v.x * dv.z) * invsum32;
    o.y = (-v.x * v.y * dv.x + (sum2 - v.y * v.y) * dv.y - v.z * v.y * dv.z) * invsum32;
    o.z = (-v.x * v.z * dv.x - v.y * v.z * dv.y + (sum2 - v.z * v.z) * dv.z) * invsum32;
    return o;
}

struct ShDeriv {
    float l[16], dx[16], dy[16], dz[16];
};

// basis values and their derivatives w.r.t. the normalised direction (backward.cu:172-263)
__device__ __forceinline__ void sh_basis_deriv(float x, float y, float z, int deg, ShDeriv& S) {
#pragma unroll
    for (int i = 0; i < 16; ++i) S.l[i] = S.dx[i] = S.dy[i] = S.dz[i] = 0.f;
    S.l[0] = kSH_C0;
    if (deg > 0) {
        S.l[1] = -kSH_C1 * y; S.dy[1] = -kSH_C1;
        S.l[2] = kSH_C1 * z;  S.dz[2] = kSH_C1;
        S.l[3] = -kSH_C1 * x; S.dx[3] = -kSH_C1;
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            S.l[4] = kSH_C2[0] * xy; S.dx[4] = kSH_C2[0] * y; S.dy[4] = kSH_C2[0] * x;
            S.l[5] = kSH_C2[1] * yz; S.dy[5] = kSH_C2[1] * z; S.dz[5] = kSH_C2[1] * y;
            S.l[6] = kSH_C2[2] * (2.0f * zz - xx - yy);
            S.dx[6] = -2.f * kSH_C2[2] * x; S.dy[6] = -2.f * kSH_C2[2] * y; S.dz[6] = 4.f * kSH_C2[2] * z;
            S.l[7] = kSH_C2[3] * xz; S.dx[7] = kSH_C2[3] * z; S.dz[7] = kSH_C2[3] * x;
            S.l[8] = kSH_C2[4] * (xx - yy); S.dx[8] = 2.f * kSH_C2[4] * x; S.dy[8] = -2.f * kSH_C2[4] * y;
            if (deg > 2) {
                S.l[9] = kSH_C3[0] * y * (3.f * xx - yy);
                S.dx[9] = kSH_C3[0] * y * 6.f * x; S.dy[9] = kSH_C3[0] * (3.f * xx - 3.f * yy);
                S.l[10] = kSH_C3[1] * xy * z;
                S.dx[10] = kSH_C3[1] * yz; S.dy[10] = kSH_C3[1] * xz; S.dz[10] = kSH_C3[1] * xy;
                S.l[11] = kSH_C3[2] * y * (4.f * zz - xx - yy);
                S.dx[11] = -kSH_C3[2] * y * 2.f * x; S.dy[11] = kSH_C3[2] * (4.f * zz - xx - 3.f * yy);
                S.dz[11] = kSH_C3[2] * y * 8.f * z;
                S.l[12] = kSH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy);
                S.dx[12] = -kSH_C3[3] * z * 6.f * x; S.dy[12] = -kSH_C3[3] * z * 6.f * y;
                S.dz[12] = kSH_C3[3] * (6.f * zz - 3.f * xx - 3.f * yy);
                S.l[13] = kSH_C3[4] * x * (4.f * zz - xx - yy);
                S.dx[13] = kSH_C3[4] * (4.f * zz - 3.f * xx - yy); S.dy[13] = -kSH_C3[4] * x * 2.f * y;
                S.dz[13] = kSH_C3[4] * x * 8.f * z;
                S.l[14] = kSH_C3[5] * z * (xx - yy);
                S.dx[14] = kSH_C3[5] * z * 2.f * x; S.dy[14] = -kSH_C3[5] * z * 2.f * y;
                S.dz[14] = kSH_C3[5] * (xx - yy);
                S.l[15] = kSH_C3[6] * x * (xx - 3.f * yy);
                S.dx[15] = kSH_C3[6] * (3.f * xx - 3.f * yy); S.dy[15] = -kSH_C3[6] * x * 6.f * y;
            }
        }
    }
}

// per-Gaussian constants of the SH backward
struct ShCtx {
    float3 dirn;           // unit view direction; the basis / derivative table is rebuilt from it where needed
    int deg;
    float dRGB[3];
    float3 dir_orig;
    float tw[3], dtw[3];   // temporal weight / its (reference-style) derivative per 16-coefficient block
    int nblk;              // active blocks: 1 (spatial) .. 3
    int ncoef;             // active coefficients per block: (D+1)^2
    bool sh4d;
};

__device__ __forceinline__ void sh_ctx_init(const PreprocessBwdParams& a, int idx, ShCtx& c) {
    c.sh4d = !((a.gaussian_dim == 3) || a.force_sh_3d);
    const unsigned cl = a.clamped[idx];
    c.dRGB[0] = (cl & 1u) ? 0.f : a.dL_dcolor[3 * idx + 0];
    c.dRGB[1] = (cl & 2u) ? 0.f : a.dL_dcolor[3 * idx + 1];
    c.dRGB[2] = (cl & 4u) ? 0.f : a.dL_dcolor[3 * idx + 2];
    const float mx = a.means3D[3 * idx + 0], my = a.means3D[3 * idx + 1], mz = a.means3D[3 * idx + 2];
    c.dir_orig = make_float3(mx - a.campos[0], my - a.campos[1], mz - a.campos[2]);
    const float len = sqrtf(c.dir_orig.x * c.dir_orig.x + c.dir_orig.y * c.dir_orig.y + c.dir_orig.z * c.dir_orig.z);
    c.dirn = make_float3(c.dir_orig.x / len, c.dir_orig.y / len, c.dir_orig.z / len);
    c.deg = a.D;
    c.ncoef = (a.D + 1) * (a.D + 1);
    c.tw[0] = 1.f; c.tw[1] = c.tw[2] = 0.f;
    c.dtw[0] = c.dtw[1] = c.dtw[2] = 0.f;
    c.nblk = 1;
    if (c.sh4d && a.D > 2 && a.D_t > 0) {
        const float dir_t = a.ts[idx] - a.timestamp;
        const double w = 2 * FDGS_MY_PI * (double)dir_t / (double)a.time_duration;
        c.tw[1] = (float)cos(w);
        c.dtw[1] = (float)(sin(w) * 2 * FDGS_MY_PI / (double)a.time_duration);
        c.nblk = 2;
        if (a.D_t > 1) {
            const double w2 = 2 * FDGS_MY_PI * (double)dir_t * 2 / (double)a.time_duration;
            c.tw[2] = (float)cos(w2);
            c.dtw[2] = (float)(sin(w2) * 2 * FDGS_MY_PI * 2 / (double)a.time_duration);
            c.nblk = 3;
        }
    }
}

// Consumes the SH row held in `rowq` (float4, in place) and replaces it by the dL_dsh row.
// Returns the direction sums and the temporal term.  NQ = number of float4 in the row (3*M/4).
template <bool WRITE = true>
__device__ __forceinline__ void sh_row_inplace(float4* rowq, int nq, const ShCtx& c, float& ddx, float& ddy,
                                               float& ddz, float& dtt) {
    const int ngroups = nq / 3;   // groups of 4 coefficients
    // Coefficient group (4 k .. 4 k + 3) outermost, the (up to) three 16-coefficient blocks inside: the basis
    // values / derivatives are evaluated per group (sh_basis_deriv is fully inlined and everything but the four
    // entries of the group is dead code), so the 64-entry table never occupies registers -- the kernel goes from
    // 127 to ~80 registers and from 4 to 6 CTAs per SM.  Per block the sums still run over k in ascending order.
    float sx[3] = {0.f, 0.f, 0.f}, sy[3] = {0.f, 0.f, 0.f}, sz[3] = {0.f, 0.f, 0.f}, sl[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int kg = 0; kg < 4; ++kg) {
        // opaque copies: keep the compiler from hoisting one shared 64-entry table out of the group loop
        float gx = c.dirn.x, gy = c.dirn.y, gz = c.dirn.z;
        asm volatile("" : "+f"(gx), "+f"(gy), "+f"(gz));
        ShDeriv S;
        sh_basis_deriv(gx, gy, gz, c.deg, S);
        const float l0 = S.l[0];
#pragma unroll
        for (int blk = 0; blk < 3; ++blk) {
            const int G = blk * 4 + kg;
            if (G >= ngroups) continue;
            const bool grp_on = (blk < c.nblk) && (kg * 4 < c.ncoef);
            float f[12];
            if (grp_on) {
                const float4 q0 = rowq[3 * G + 0], q1 = rowq[3 * G + 1], q2 = rowq[3 * G + 2];
                f[0] = q0.x; f[1] = q0.y; f[2] = q0.z; f[3] = q0.w;
                f[4] = q1.x; f[5] = q1.y; f[6] = q1.z; f[7] = q1.w;
                f[8] = q2.x; f[9] = q2.y; f[10] = q2.z; f[11] = q2.w;
            }
            float o[12];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int k = kg * 4 + j;
                float w = 0.f;
                if (grp_on && k < c.ncoef) {
                    const float sk = f[3 * j] * c.dRGB[0] + f[3 * j + 1] * c.dRGB[1] + f[3 * j + 2] * c.dRGB[2];
                    sx[blk] += S.dx[k] * sk;
                    sy[blk] += S.dy[k] * sk;
                    sz[blk] += S.dz[k] * sk;
                    sl[blk] += S.l[k] * sk;
                    // dL_dsh[1] = l0m0 * dL_dRGB in the 4D variant (quirk, backward.cu:190)
                    w = (blk == 0) ? ((c.sh4d && k == 1) ? l0 : S.l[k]) : c.tw[blk] * S.l[k];
                }
                o[3 * j + 0] = w * c.dRGB[0];
                o[3 * j + 1] = w * c.dRGB[1];
                o[3 * j + 2] = w * c.dRGB[2];
            }
            if (WRITE) {
                rowq[3 * G + 0] = make_float4(o[0], o[1], o[2], o[3]);
                rowq[3 * G + 1] = make_float4(o[4], o[5], o[6], o[7]);
                rowq[3 * G + 2] = make_float4(o[8], o[9], o[10], o[11]);
            }
        }
    }
    ddx = ddy = ddz = dtt = 0.f;
#pragma unroll
    for (int blk = 0; blk < 3; ++blk) {
        if (blk * 4 < ngroups && blk < c.nblk) {
            ddx += c.tw[blk] * sx[blk];
            ddy += c.tw[blk] * sy[blk];
            ddz += c.tw[blk] * sz[blk];
            if (blk > 0) dtt = c.dtw[blk] * sl[blk];   // overwrites: backward.cu:403
        }
    }
    // coefficients beyond the three 16-blocks (M > 48) are never used: zero gradient
    if (WRITE)
        for (int qi = 36; qi < nq; ++qi) rowq[qi] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// ---- SH backward ----------------------------------------------------------------------------------
// FACTORS (multi-GPU view parallelism, fdgs/dist.py): the dL_dsh row of a view is the outer product
// (basis weights of the view direction and time) x (clamp-masked colour gradient), so instead of the 12*M-byte row
// only the 3-float colour factor is written (sh_factors[P,3], zeros for Gaussians this view did not render); the rows
// of all views are rebuilt and summed after the exchange by sh_outer_sum_kernel (exchange.cu).  The SH row is still
// read: the direction / time gradients need sum_k dbasis_k (sh_k . dRGB).
// STAGE as in preprocess_fwd_kernel: 0 = global memory coefficient by coefficient, 1 = cp.async.bulk rows in and out,
// 2 = cooperative coalesced copies of split rows (features_dc | features_rest in, their two gradient tensors out).
// view v of a batch (blockIdx.y): the view's camera and its slices of the forward's per-Gaussian state and of every
// gradient (see PreprocessBwdParams::vb)
__device__ __forceinline__ PreprocessBwdParams preprocess_bwd_view(PreprocessBwdParams a, int v) {
    const size_t P = (size_t)a.P;
    const ViewScalars vs = a.vb.scalars[v];
    a.viewmatrix += 16 * v;
    a.projmatrix += 16 * v;
    a.campos += 3 * v;
    a.timestamp = vs.timestamp;
    a.tan_fovx = vs.tan_fovx;
    a.tan_fovy = vs.tan_fovy;
    a.focal_x = vs.focal_x;
    a.focal_y = vs.focal_y;
    a.means3D += 3 * v * P;
    a.radii += v * P;
    a.clamped += v * P;
    a.tiles_touched += v * P;
    a.cov3D += 6 * v * P;
    a.grec += v * P;
    a.dL_dmean2D += 3 * v * P;
    a.dL_dconic += 4 * v * P;
    a.dL_dopacity += v * P;
    a.dL_dcolor += 3 * v * P;
    a.dL_dmean3D += 3 * v * P;
    a.dL_dcov3D += 6 * v * P;
    if (a.sh_factors) a.sh_factors += v * a.factor_stride;
    a.dL_dts += v * P;
    a.dL_dscale += 3 * v * P;
    a.dL_dscale_t += v * P;
    a.dL_drot += 4 * v * P;
    a.dL_drot_r += 4 * v * P;
    return a;
}

// BATCH: one view per blockIdx.y (FACTORS only: the SH rows of a batch are summed over its views by sh_outer_sum)
template <int STAGE, bool FACTORS, bool BATCH>
__device__ __forceinline__ void sh_bwd_body(const PreprocessBwdParams& a_) {
    static_assert(!BATCH || FACTORS, "a batch emits colour factors");
    // an lvalue on both sides: the single-view instantiation reads its parameters in place, no copy
    PreprocessBwdParams view_;
    if (BATCH) view_ = preprocess_bwd_view(a_, blockIdx.y);
    const PreprocessBwdParams& a = BATCH ? view_ : a_;
    constexpr bool BULK = STAGE == 1;
    constexpr bool SPLIT = STAGE == 2;
    __shared__ int slot_idx[SB_CAP];   // STAGE 2: Gaussian whose row occupies each slot
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t bar;
    __shared__ short slot_of[SB_THREADS];   // rank among the rendered rows of this CTA, -1 = not rendered
    __shared__ int warp_cnt[SB_THREADS / 32];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int idx = blockIdx.x * SB_THREADS + tid;
    const bool in_range = idx < a.P;
    const bool vis = in_range && (a.radii[idx] > 0) && (a.tiles_touched[idx] != 0u);
    const int row_floats = 3 * a.M;
    const int nq = row_floats / 4;

    // block-level compaction of the rendered rows
    const unsigned bal = __ballot_sync(0xffffffffu, vis);
    if (lane == 0) warp_cnt[warp] = __popc(bal);
    if (BULK && tid == 0) {
        mbar_init(&bar, 1);
        mbar_fence_init();
    }
    __syncthreads();
    int base = 0, nvis = 0;
#pragma unroll
    for (int w = 0; w < SB_THREADS / 32; ++w) {
        if (w < warp) base += warp_cnt[w];
        nvis += warp_cnt[w];
    }
    const int my_rank = vis ? base + __popc(bal & ((1u << lane) - 1u)) : -1;
    slot_of[tid] = (short)my_rank;
    __syncthreads();

    if (BATCH && blockIdx.x == 0 && tid == 0) {
        // the view's metadata row of the sh_outer_sum table, after its P colour factors
        float* meta = a.sh_factors + 3 * (size_t)a.P;
        meta[0] = a.timestamp;
        meta[1] = a.campos[0];
        meta[2] = a.campos[1];
        meta[3] = a.campos[2];
    }
    // zero rows: every float4 of every non-rendered row of this CTA, coalesced (unless the forward's blend wrote them)
    if (FACTORS) {
        if (in_range && !vis) {
            a.sh_factors[3 * idx + 0] = 0.f;
            a.sh_factors[3 * idx + 1] = 0.f;
            a.sh_factors[3 * idx + 2] = 0.f;
        }
    } else if (a.sh_rows_zeroed) {
        // the non-rendered rows are already zero (blend_fwd.cu)
    } else if (a.dL_dsh_rest != nullptr) {
        // split gradient tensors: [P,1,3] and [P,M-1,3]; a warp per non-rendered row
        const int rows_here = min(SB_THREADS, a.P - blockIdx.x * SB_THREADS);
        const size_t r0 = (size_t)blockIdx.x * SB_THREADS;
        const int rest_floats = row_floats - 3;
        for (int r = warp; r < rows_here; r += SB_THREADS / 32) {
            if (slot_of[r] >= 0) continue;
            if (lane < 3) a.dL_dsh[(r0 + r) * 3 + lane] = 0.f;
            float* rest = a.dL_dsh_rest + (r0 + r) * rest_floats;
            for (int f = lane; f < rest_floats; f += 32) rest[f] = 0.f;
        }
    } else {
        const int rows_here = min(SB_THREADS, a.P - blockIdx.x * SB_THREADS);
        float4* dst = reinterpret_cast<float4*>(a.dL_dsh + (size_t)blockIdx.x * SB_THREADS * row_floats);
        const int total = rows_here * nq;
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        if (BULK) {
            for (int f = tid; f < total; f += SB_THREADS) {
                const int r = f / nq;
                if (slot_of[r] < 0) dst[f] = z;
            }
        } else {
            // generic path (row not a multiple of 16 bytes): scalar stores
            float* d1 = a.dL_dsh + (size_t)blockIdx.x * SB_THREADS * row_floats;
            for (int f = tid; f < rows_here * row_floats; f += SB_THREADS)
                if (slot_of[f / row_floats] < 0) d1[f] = 0.f;
        }
    }

    ShCtx c;
    if (vis) {
        sh_ctx_init(a, idx, c);
        if (FACTORS) {
            a.sh_factors[3 * idx + 0] = c.dRGB[0];
            a.sh_factors[3 * idx + 1] = c.dRGB[1];
            a.sh_factors[3 * idx + 2] = c.dRGB[2];
        }
    }

    if (STAGE != 0) {
        float* rows = reinterpret_cast<float*>(smem_raw);
        const int rest_floats = row_floats - 3;
        for (int round = 0, lo = 0; lo < nvis; ++round, lo += SB_CAP) {
            const int cnt = min(SB_CAP, nvis - lo);
            const bool mine = vis && my_rank >= lo && my_rank < lo + cnt;
            float4* rowq = reinterpret_cast<float4*>(rows + (size_t)(my_rank - lo) * a.sh_row_stride_floats);
            if (round > 0) {
                // the previous round's bulk stores must have finished reading the slots
                if (BULK && !FACTORS && vis) bulk_wait_read_all();
                __syncthreads();
            }
            if (BULK) {
                if (tid == 0) mbar_expect_tx(&bar, (uint32_t)cnt * (uint32_t)row_floats * 4u);
                if (mine) bulk_g2s(rowq, a.shs + (size_t)idx * row_floats, (uint32_t)row_floats * 4u, &bar);
            } else {
                if (mine) slot_idx[my_rank - lo] = idx;
                __syncthreads();
                for (int sidx = warp; sidx < cnt; sidx += SB_THREADS / 32) {
                    const size_t g = (size_t)slot_idx[sidx];
                    split_row_to_smem(rows + (size_t)sidx * a.sh_row_stride_floats, a.shs + g * 3, a.shs_rest + g * rest_floats,
                                      row_floats, lane);
                }
                cp_async_wait_all();
                __syncthreads();
            }
            if (mine) {
                if (BULK) mbar_wait(&bar, (uint32_t)round & 1u);
                float ddx, ddy, ddz, dtt;
                sh_row_inplace<!FACTORS>(rowq, nq, c, ddx, ddy, ddz, dtt);
                if (BULK && !FACTORS) {
                    fence_async_smem();
                    bulk_s2g(a.dL_dsh + (size_t)idx * row_floats, rowq, (uint32_t)row_floats * 4u);
                    bulk_commit();
                }
                const float3 dm = dnormvdv3(c.dir_orig, make_float3(ddx, ddy, ddz));
                a.dL_dmean3D[3 * idx + 0] = dm.x;
                a.dL_dmean3D[3 * idx + 1] = dm.y;
                a.dL_dmean3D[3 * idx + 2] = dm.z;
                a.dL_dts[idx] = c.sh4d ? dtt : 0.f;
            }
            if (SPLIT && !FACTORS) {
                // the gradient rows, now in the slots, go out the way the rows came in: coalesced, split over the two tensors
                __syncthreads();
                for (int sidx = warp; sidx < cnt; sidx += SB_THREADS / 32) {
                    const size_t g = (size_t)slot_idx[sidx];
                    const float* src = rows + (size_t)sidx * a.sh_row_stride_floats;
                    if (lane < 3) a.dL_dsh[g * 3 + lane] = src[lane];
                    float* rest = a.dL_dsh_rest + g * rest_floats;
                    for (int f = lane; f < rest_floats; f += 32) rest[f] = src[f + 3];
                }
            }
        }
        if (BULK && !FACTORS && vis) bulk_wait_all();
    } else if (vis) {
        // generic path: global loads / stores, one coefficient at a time
        // generic path; with split rows coefficient 0 lives in shs / dL_dsh [P,1,3], the others in *_rest [P,M-1,3]
        const bool split = a.shs_rest != nullptr;
        const float* grow = split ? a.shs_rest + (size_t)idx * (row_floats - 3) - 3 : a.shs + (size_t)idx * row_floats;
        const float* grow0 = split ? a.shs + (size_t)idx * 3 : grow;
        float* drow = FACTORS ? nullptr : (split ? a.dL_dsh_rest + (size_t)idx * (row_floats - 3) - 3 : a.dL_dsh + (size_t)idx * row_floats);
        float* drow0 = FACTORS ? nullptr : (split ? a.dL_dsh + (size_t)idx * 3 : drow);
        float ddx = 0.f, ddy = 0.f, ddz = 0.f, dtt = 0.f;
        ShDeriv SDg;
        sh_basis_deriv(c.dirn.x, c.dirn.y, c.dirn.z, c.deg, SDg);
        for (int blk = 0; blk * 16 < a.M; ++blk) {
            float sx = 0.f, sy = 0.f, sz = 0.f, sl = 0.f;
            const bool blk_on = blk < c.nblk;
            for (int k = 0; k < 16 && blk * 16 + k < a.M; ++k) {
                const int cidx = blk * 16 + k;
                float w = 0.f;
                if (blk_on && k < c.ncoef) {
                    const float* gsrc = (cidx == 0) ? grow0 : grow + 3 * cidx;
                    const float sk = __ldg(gsrc) * c.dRGB[0] + __ldg(gsrc + 1) * c.dRGB[1] + __ldg(gsrc + 2) * c.dRGB[2];
                    sx += SDg.dx[k] * sk; sy += SDg.dy[k] * sk; sz += SDg.dz[k] * sk; sl += SDg.l[k] * sk;
                    w = (blk == 0) ? ((c.sh4d && k == 1) ? SDg.l[0] : SDg.l[k]) : c.tw[blk < 3 ? blk : 0] * SDg.l[k];
                }
                if (!FACTORS) {
                    float* dd = (cidx == 0) ? drow0 : drow + 3 * cidx;
                    dd[0] = w * c.dRGB[0];
                    dd[1] = w * c.dRGB[1];
                    dd[2] = w * c.dRGB[2];
                }
            }
            if (blk_on) {
                ddx += c.tw[blk] * sx; ddy += c.tw[blk] * sy; ddz += c.tw[blk] * sz;
                if (blk > 0) dtt = c.dtw[blk] * sl;
            }
        }
        const float3 dm = dnormvdv3(c.dir_orig, make_float3(ddx, ddy, ddz));
        a.dL_dmean3D[3 * idx + 0] = dm.x;
        a.dL_dmean3D[3 * idx + 1] = dm.y;
        a.dL_dmean3D[3 * idx + 2] = dm.z;
        a.dL_dts[idx] = c.sh4d ? dtt : 0.f;
    }
}

template <int STAGE, bool FACTORS>
__global__ void __launch_bounds__(SB_THREADS, 6) sh_bwd_kernel(const PreprocessBwdParams a_) {
    sh_bwd_body<STAGE, FACTORS, false>(a_);
}

// the batched entry (fdgs_forward_batch / fdgs_backward_batch): one view per blockIdx.y
template <int STAGE>
__global__ void __launch_bounds__(SB_THREADS, 6) sh_bwd_batch_kernel(const PreprocessBwdParams a_) {
    sh_bwd_body<STAGE, true, true>(a_);
}

// ---- view-parallel SH gradient: rebuild and sum the rows of all views -------------------------------------------
// dL_dsh of ONE view is rank one per Gaussian: row[k][ch] = w_k(view direction, time) * dRGB[ch]  (sh_row_inplace
// above).  With the views of a step spread over ranks (fdgs/dist.py) only dRGB travels (3 floats per Gaussian and
// view, all-gathered for the union of rendered Gaussians); every rank then rebuilds w_k for every view from the
// REPLICATED Gaussian parameters and the view's (timestamp, camera position) and sums the outer products in global
// view order -- 12 bytes per (Gaussian, view) on NVLink instead of a 576-byte row in an all-reduce, and the sum is
// bit-identical to accumulating the views' dL_dsh one after the other (what the reference's sequential loop does,
// train.py:104-166): explicit round-to-nearest multiply then add, no fused rounding.
// The direction is the one sh_ctx_init() sees: the time-shifted mean the forward wrote to out_means3D
// (preprocess_fwd.cu: mean + dt * Sigma_xyz,t / Sigma_tt, same intrinsics, same order) minus the camera position.
// Two kernels: directions / temporal weights per (union Gaussian, view), then the row sums (dense warps over the
// union list) + zero rows for everything else.
// Phase A: one thread per (union Gaussian k, view v): the view's unit direction to the (time-shifted) mean and its two
// temporal weights, stored with the colour factor as dirs[(v K + k)] = { gx, gy, gz, tw1 | r, g, b, tw2 }.
__global__ void __launch_bounds__(256) sh_outer_dir_kernel(const ShSumParams a) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)a.K * a.V) return;
    const int k = (int)(t / a.V), v = (int)(t - (long long)k * a.V);
    const long long idx = a.union_idx ? a.union_idx[k] : k;
    const float* blk = a.table + (size_t)v * a.view_stride;
    const float r = blk[3 * (size_t)k + 0], g = blk[3 * (size_t)k + 1], b = blk[3 * (size_t)k + 2];
    float4 o0 = make_float4(0.f, 0.f, 1.f, 0.f), o1 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!(r == 0.f && g == 0.f && b == 0.f)) {   // rendered by view v
        const bool sh4d = !((a.gaussian_dim == 3) || a.force_sh_3d);
        const float* meta = blk + a.meta_off;   // timestamp, camera position
        const float timestamp = meta[0];
        const float t_g = (a.ts != nullptr) ? a.ts[idx] : 0.f;
        float mx = a.means3D[3 * idx + 0], my = a.means3D[3 * idx + 1], mz = a.means3D[3 * idx + 2];
        if (a.view_means) {
            // the shifted mean this view's forward wrote: exactly what sh_ctx_init() read
            const float* vm = a.view_means + (size_t)v * 3 * a.P + 3 * idx;
            mx = vm[0]; my = vm[1]; mz = vm[2];
        } else if (a.rot_4d) {
            // the forward's mean shift (preprocess_fwd.cu), same intrinsics, same order
            const float mod = a.scale_modifier;
            Sigma4 S;
            build_M4(fmul(mod, a.scales[3 * idx + 0]), fmul(mod, a.scales[3 * idx + 1]), fmul(mod, a.scales[3 * idx + 2]),
                     fmul(mod, a.scales_t[idx]), reinterpret_cast<const float4*>(a.rotations)[idx],
                     reinterpret_cast<const float4*>(a.rotations_r)[idx], S.M);
            sigma_from_M(S);
            const float dt = fsub(timestamp, t_g);
            mx = ffma(dt, fdiv(S.s03, S.s33), mx);
            my = ffma(dt, fdiv(S.s13, S.s33), my);
            mz = ffma(dt, fdiv(S.s23, S.s33), mz);
        }
        // exactly sh_ctx_init()
        const float dx = mx - meta[1], dy = my - meta[2], dz = mz - meta[3];
        const float len = sqrtf(dx * dx + dy * dy + dz * dz);
        float tw1 = 0.f, tw2 = 0.f;
        if (sh4d && a.D > 2 && a.D_t > 0) {
            const float dir_t = t_g - timestamp;
            tw1 = (float)cos(2 * FDGS_MY_PI * (double)dir_t / (double)a.time_duration);
            if (a.D_t > 1) tw2 = (float)cos(2 * FDGS_MY_PI * (double)dir_t * 2 / (double)a.time_duration);
        }
        o0 = make_float4(dx / len, dy / len, dz / len, tw1);
        o1 = make_float4(r, g, b, tw2);
    }
    float4* dst = reinterpret_cast<float4*>(a.dirs) + 2 * ((size_t)v * a.K + k);
    dst[0] = o0;
    dst[1] = o1;
}

// Coalesced store of one gradient row (row_floats = 3 M values; `src` = its first min(row_floats, 144) values in shared
// memory or NULL for a zero row) by the 32 lanes of a warp.  One tensor [P,M,3] with 16-byte rows: float4 stores, 512
// contiguous bytes per instruction; split tensors (features_dc [P,1,3] | features_rest [P,M-1,3]): 4-byte stores.
__device__ __forceinline__ void store_sh_row(const ShSumParams& a, size_t idx, const float* src, int lane) {
    const int row_floats = 3 * a.M;
    if (a.out1 == nullptr && (a.M % 4) == 0 && !a.accumulate) {
        float4* row = reinterpret_cast<float4*>(a.out0 + idx * row_floats);
        const int nq = row_floats / 4;
        for (int q = lane; q < nq; q += 32) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (src != nullptr && q < 36) v = *reinterpret_cast<const float4*>(src + 4 * q);
            row[q] = v;
        }
    } else {
        const int m0 = a.m0;
        for (int f = lane; f < row_floats; f += 32) {
            const float v = (src != nullptr && f < 144) ? src[f] : 0.f;
            const int c = f / 3, ch = f - 3 * c;
            float* dst = (c < m0) ? a.out0 + (idx * m0 + c) * 3 + ch : a.out1 + (idx * (a.M - m0) + (c - m0)) * 3 + ch;
            *dst = a.accumulate ? *dst + v : v;
        }
    }
}

// Phase B.  Blocks [0, union_blocks): 32 UNION Gaussians per block (dense: the list a.union_idx), one per lane; warp kg
// owns the coefficients 4 kg .. 4 kg + 3 of each of the three 16-blocks (warp-uniform, so only those four basis
// functions are evaluated) and sums the V rank-one rows into registers; the 32 rows of a block are staged in shared
// memory and stored warp-per-row, fully coalesced.
// Blocks beyond: the rows of all other Gaussians are zero-filled, warp per row.
constexpr int SO_ROWS = 32;          // union Gaussians per block (128 threads)
constexpr int SO_STRIDE = 148;       // floats per staged row (144 + padding: conflict-free float4 stores)

template <int KG>
__device__ __forceinline__ void sh_outer_accumulate(const ShSumParams& a, int k, float (&acc)[3][12]) {
    const bool sh4d = !((a.gaussian_dim == 3) || a.force_sh_3d);
    const int ncoef = (a.D + 1) * (a.D + 1);
    const int nblk = (sh4d && a.D > 2 && a.D_t > 0) ? ((a.D_t > 1) ? 3 : 2) : 1;
    for (int v = 0; v < a.V; ++v) {
        const float4* src = reinterpret_cast<const float4*>(a.dirs) + 2 * ((size_t)v * a.K + k);
        const float4 d0 = src[0], d1 = src[1];
        if (d1.x == 0.f && d1.y == 0.f && d1.z == 0.f) continue;   // not rendered by view v
        const float tw1 = d0.w, tw2 = d1.w;
        ShDeriv S;
        sh_basis_deriv(d0.x, d0.y, d0.z, a.D, S);   // only l[4 KG .. 4 KG + 3] (and l[0]) survive dead-code elimination
        const float drgb[3] = {d1.x, d1.y, d1.z};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k2 = 4 * KG + j;
            if (k2 >= ncoef) continue;
            const float lk = S.l[k2];
            const float w0 = (sh4d && k2 == 1) ? S.l[0] : lk;
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                acc[0][3 * j + ch] = __fadd_rn(acc[0][3 * j + ch], __fmul_rn(w0, drgb[ch]));
                if (nblk > 1) acc[1][3 * j + ch] = __fadd_rn(acc[1][3 * j + ch], __fmul_rn(__fmul_rn(tw1, lk), drgb[ch]));
                if (nblk > 2) acc[2][3 * j + ch] = __fadd_rn(acc[2][3 * j + ch], __fmul_rn(__fmul_rn(tw2, lk), drgb[ch]));
            }
        }
    }
}

__global__ void __launch_bounds__(128) sh_outer_sum_kernel(const ShSumParams a, const int union_blocks) {
    __shared__ __align__(16) float rowbuf[SO_ROWS][SO_STRIDE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if ((int)blockIdx.x >= union_blocks) {
        // zero rows: this block covers 128 consecutive Gaussians, 32 per warp; the warp reads their 32 union slots with
        // one coalesced load, then zero-fills the rows that are not in the union (no dependent load per row)
        if (a.accumulate) return;
        const long long base = (long long)(blockIdx.x - union_blocks) * 128 + 32 * warp;
        const long long mine = base + lane;
        unsigned todo = __ballot_sync(0xffffffffu, mine < a.P && a.slot_of[mine] < 0);
        while (todo) {
            const int r = __ffs(todo) - 1;
            todo &= todo - 1;
            store_sh_row(a, (size_t)(base + r), nullptr, lane);
        }
        return;
    }
    const int k = blockIdx.x * SO_ROWS + lane;
    const int kg = warp;
    float acc[3][12];
#pragma unroll
    for (int b = 0; b < 3; ++b)
#pragma unroll
        for (int i = 0; i < 12; ++i) acc[b][i] = 0.f;
    long long my_idx = -1;
    if (k < a.K) {
        if (kg == 0) sh_outer_accumulate<0>(a, k, acc);
        else if (kg == 1) sh_outer_accumulate<1>(a, k, acc);
        else if (kg == 2) sh_outer_accumulate<2>(a, k, acc);
        else sh_outer_accumulate<3>(a, k, acc);
        my_idx = a.union_idx ? a.union_idx[k] : k;     // the destination row of lane `lane`'s Gaussian (shuffled to the storing warp below)
    }
    // stage: coefficients 16 b + 4 kg + j of the row -> floats 48 b + 12 kg + 3 j + ch
    {
        float* dst = &rowbuf[lane][0];
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            float4* q = reinterpret_cast<float4*>(dst + 48 * b + 12 * kg);
            q[0] = make_float4(acc[b][0], acc[b][1], acc[b][2], acc[b][3]);
            q[1] = make_float4(acc[b][4], acc[b][5], acc[b][6], acc[b][7]);
            q[2] = make_float4(acc[b][8], acc[b][9], acc[b][10], acc[b][11]);
        }
    }
    __syncthreads();
    for (int r = warp; r < SO_ROWS; r += 4) {
        const long long dst_row = __shfl_sync(0xffffffffu, my_idx, r);
        if (dst_row < 0) break;     // rows beyond K (only in the last block; warp-uniform)
        store_sh_row(a, (size_t)dst_row, &rowbuf[r][0], lane);
    }
}

// 3x3 helper, glm convention as mat4_mul (fdgs_common.cuh): A[c][r], (A*B)[c][r] = sum_k A[k][r] * B[c][k]
__device__ __forceinline__ void mat3_mul(const float A[3][3], const float B[3][3], float C[3][3]) {
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int r = 0; r < 3; ++r) C[c][r] = A[0][r] * B[c][0] + A[1][r] * B[c][1] + A[2][r] * B[c][2];
}

// ---- geometry backward ---------------------------------------------------------------------------
// CAM: also write the rendered row's CAM_TERMS camera terms to cam[s * GB_THREADS] (s = the slot, see
// CameraGradParams); the caller zeroes the slots, so rows that are not rendered contribute 0
template <bool BATCH, bool CAM = false>
__device__ __forceinline__ void geom_bwd_body(const PreprocessBwdParams& a_, const int has_sh_part, float* cam = nullptr) {
    // an lvalue on both sides: the single-view instantiation reads its parameters in place, no copy
    PreprocessBwdParams view_;
    if (BATCH) view_ = preprocess_bwd_view(a_, blockIdx.y);
    const PreprocessBwdParams& a = BATCH ? view_ : a_;
    const int idx = blockIdx.x * GB_THREADS + threadIdx.x;
    if (idx >= a.P) return;
    const bool vis = (a.radii[idx] > 0) && (a.tiles_touched[idx] != 0u);

    float g_mean[3] = {0.f, 0.f, 0.f};
    float g_cov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float g_ts = 0.f, g_scale[3] = {0.f, 0.f, 0.f}, g_scale_t = 0.f;
    float g_rot[4] = {0.f, 0.f, 0.f, 0.f}, g_rotr[4] = {0.f, 0.f, 0.f, 0.f};

    if (vis) {
        const float* V = a.viewmatrix;
        const float mx = a.means3D[3 * idx + 0], my = a.means3D[3 * idx + 1], mz = a.means3D[3 * idx + 2];
        float c3[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) c3[i] = a.cov3D[6 * idx + i];

        // The blend backward leaves moment sums of w = G dL/dalpha about the mean: W10, W01 in dL_dmean2D.xy,
        // W20, W11, W02 in dL_dconic.  Their per-Gaussian linear map to the reference's gradients
        // (backward.cu:1119-1134: dG/ddel = -G (A dx + B dy), ddelx/dx = W/2, dL/dconic = -0.5 G d d^T dL/dG,
        // dL/dG = opacity dL/dalpha) is applied here, once, instead of per (pixel, Gaussian) pair.
        float d2x = a.dL_dmean2D[3 * idx + 0], d2y = a.dL_dmean2D[3 * idx + 1];
        float dcx = a.dL_dconic[4 * idx + 0], dcy = a.dL_dconic[4 * idx + 1], dcz = a.dL_dconic[4 * idx + 3];
        const float4 con = a.grec[idx].q1;   // A, B, C, blended opacity
        const float W10 = d2x, W01 = d2y;
        d2x = -0.5f * (float)a.W * con.w * (con.x * W10 + con.y * W01);
        d2y = -0.5f * (float)a.H * con.w * (con.z * W01 + con.y * W10);
        const float hs = -0.5f * con.w;
        dcx *= hs; dcy *= hs; dcz *= hs;
        a.dL_dmean2D[3 * idx + 0] = d2x;
        a.dL_dmean2D[3 * idx + 1] = d2y;
        a.dL_dconic[4 * idx + 0] = dcx;
        a.dL_dconic[4 * idx + 1] = dcy;
        a.dL_dconic[4 * idx + 3] = dcz;

        // ---------------- computeCov2DCUDA, backward.cu:486-617 ----------------
        {
            Proj2D Pj;
            build_T(V, mx, my, mz, a.focal_x, a.focal_y, a.tan_fovx, a.tan_fovy, Pj);
            const float limx = fmul(1.3f, a.tan_fovx), limy = fmul(1.3f, a.tan_fovy);
            const float x_grad_mul = (Pj.txtz < -limx || Pj.txtz > limx) ? 0.f : 1.f;
            const float y_grad_mul = (Pj.tytz < -limy || Pj.tytz > limy) ? 0.f : 1.f;
            float ca, cb, cc;
            cov2d_from_T(Pj, c3, ca, cb, cc);
            const float A = ca + 0.3f, B = cb, C = cc + 0.3f;
            const float denom = A * C - B * B;
            float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
            const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
            const float T00 = Pj.T00, T01 = Pj.T01, T02 = Pj.T02, T10 = Pj.T10, T11 = Pj.T11, T12 = Pj.T12;
            if (denom2inv != 0) {
                dL_da = denom2inv * (-C * C * dcx + 2 * B * C * dcy + (denom - A * C) * dcz);
                dL_dc = denom2inv * (-A * A * dcz + 2 * A * B * dcy + (denom - A * C) * dcx);
                dL_db = denom2inv * 2 * (B * C * dcx - (denom + 2 * B * B) * dcy + A * B * dcz);
                g_cov[0] = (T00 * T00 * dL_da + T00 * T10 * dL_db + T10 * T10 * dL_dc);
                g_cov[3] = (T01 * T01 * dL_da + T01 * T11 * dL_db + T11 * T11 * dL_dc);
                g_cov[5] = (T02 * T02 * dL_da + T02 * T12 * dL_db + T12 * T12 * dL_dc);
                g_cov[1] = 2 * T00 * T01 * dL_da + (T00 * T11 + T01 * T10) * dL_db + 2 * T10 * T11 * dL_dc;
                g_cov[2] = 2 * T00 * T02 * dL_da + (T00 * T12 + T02 * T10) * dL_db + 2 * T10 * T12 * dL_dc;
                g_cov[4] = 2 * T02 * T01 * dL_da + (T01 * T12 + T02 * T11) * dL_db + 2 * T11 * T12 * dL_dc;
            }
            // Vrk (symmetric): V0 = (c0,c1,c2), V1 = (c1,c3,c4), V2 = (c2,c4,c5)
            const float r0a = T00 * c3[0] + T01 * c3[1] + T02 * c3[2];
            const float r0b = T00 * c3[1] + T01 * c3[3] + T02 * c3[4];
            const float r0c = T00 * c3[2] + T01 * c3[4] + T02 * c3[5];
            const float r1a = T10 * c3[0] + T11 * c3[1] + T12 * c3[2];
            const float r1b = T10 * c3[1] + T11 * c3[3] + T12 * c3[4];
            const float r1c = T10 * c3[2] + T11 * c3[4] + T12 * c3[5];
            const float dL_dT00 = 2 * r0a * dL_da + r1a * dL_db;
            const float dL_dT01 = 2 * r0b * dL_da + r1b * dL_db;
            const float dL_dT02 = 2 * r0c * dL_da + r1c * dL_db;
            const float dL_dT10 = 2 * r1a * dL_dc + r0a * dL_db;
            const float dL_dT11 = 2 * r1b * dL_dc + r0b * dL_db;
            const float dL_dT12 = 2 * r1c * dL_dc + r0c * dL_db;
            // W[c][r] = view[4*r + c]   (backward.cu:525-528)
            const float dL_dJ00 = V[0] * dL_dT00 + V[4] * dL_dT01 + V[8] * dL_dT02;
            const float dL_dJ02 = V[2] * dL_dT00 + V[6] * dL_dT01 + V[10] * dL_dT02;
            const float dL_dJ11 = V[1] * dL_dT10 + V[5] * dL_dT11 + V[9] * dL_dT12;
            const float dL_dJ12 = V[2] * dL_dT10 + V[6] * dL_dT11 + V[10] * dL_dT12;
            const float tz = 1.f / Pj.tz, tz2 = tz * tz, tz3 = tz2 * tz;
            const float h_x = a.focal_x, h_y = a.focal_y;
            const float dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
            const float dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
            const float dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * Pj.tx) * tz3 * dL_dJ02 +
                                 (2 * h_y * Pj.ty) * tz3 * dL_dJ12;
            // transformVec4x3Transpose, plus the depth gradient riding in dL_dmean2D.z (:611)
            const float vx = dL_dtx, vy = dL_dty, vz = dL_dtz + a.dL_dmean2D[3 * idx + 2];
            g_mean[0] = V[0] * vx + V[1] * vy + V[2] * vz;
            g_mean[1] = V[4] * vx + V[5] * vy + V[6] * vz;
            g_mean[2] = V[8] * vx + V[9] * vy + V[10] * vz;
            if (CAM) {
                // view-space point t = W m + V[12..14]: dL/dV[4c + r] = m_c g_r with m_3 = 1, g = (vx, vy, vz); plus,
                // on c < 3, the W part of T = J W (build_T): dL/dW[r][c] = sum_i J[i][r] dL/dT[i][c], W[r][c] = V[4c + r]
                const float j00 = fdiv(h_x, Pj.tz), j11 = fdiv(h_y, Pj.tz);
                const float j02 = fdiv(fmul(h_x, -Pj.tx), fmul(Pj.tz, Pj.tz));
                const float j12 = fdiv(fmul(h_y, -Pj.ty), fmul(Pj.tz, Pj.tz));
                const float m[3] = {mx, my, mz};
                const float dT0[3] = {dL_dT00, dL_dT01, dL_dT02}, dT1[3] = {dL_dT10, dL_dT11, dL_dT12};
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    cam[(3 * c + 0) * GB_THREADS] = m[c] * vx + j00 * dT0[c];
                    cam[(3 * c + 1) * GB_THREADS] = m[c] * vy + j11 * dT1[c];
                    cam[(3 * c + 2) * GB_THREADS] = m[c] * vz + (j02 * dT0[c] + j12 * dT1[c]);
                }
                cam[9 * GB_THREADS] = vx;
                cam[10 * GB_THREADS] = vy;
                cam[11 * GB_THREADS] = vz;
            }
        }

        // ---------------- preprocessCUDA (backward), backward.cu:877-894 ----------------
        {
            const float* Pm = a.projmatrix;
            const float m_hw = Pm[3] * mx + Pm[7] * my + Pm[11] * mz + Pm[15];
            const float m_w = 1.0f / (m_hw + 0.0000001f);
            const float mul1 = (Pm[0] * mx + Pm[4] * my + Pm[8] * mz + Pm[12]) * m_w * m_w;
            const float mul2 = (Pm[1] * mx + Pm[5] * my + Pm[9] * mz + Pm[13]) * m_w * m_w;
            g_mean[0] += (Pm[0] * m_w - Pm[3] * mul1) * d2x + (Pm[1] * m_w - Pm[3] * mul2) * d2y;
            g_mean[1] += (Pm[4] * m_w - Pm[7] * mul1) * d2x + (Pm[5] * m_w - Pm[7] * mul2) * d2y;
            g_mean[2] += (Pm[8] * m_w - Pm[11] * mul1) * d2x + (Pm[9] * m_w - Pm[11] * mul2) * d2y;
            if (CAM) {
                // homogeneous projection p = P [m, 1]: dL/dPm[4c + r] = m_c gp_r, gp = (d2x m_w, d2y m_w, 0 (clip z is
                // not used), -(mul1 d2x + mul2 d2y)); the zero column is not reduced
                const float gp[3] = {d2x * m_w, d2y * m_w, -(mul1 * d2x + mul2 * d2y)};
                const float m[4] = {mx, my, mz, 1.f};
#pragma unroll
                for (int c = 0; c < 4; ++c)
#pragma unroll
                    for (int j = 0; j < 3; ++j) cam[(12 + 3 * c + j) * GB_THREADS] = m[c] * gp[j];
            }
        }

        // SH view-direction / time terms left by sh_bwd_kernel (backward.cu:896-906)
        if (has_sh_part) {
            g_mean[0] += a.dL_dmean3D[3 * idx + 0];
            g_mean[1] += a.dL_dmean3D[3 * idx + 1];
            g_mean[2] += a.dL_dmean3D[3 * idx + 2];
            g_ts += a.dL_dts[idx];
            if (CAM) {
                // the view direction is m - campos: its gradient w.r.t. campos is minus the term w.r.t. the mean
#pragma unroll
                for (int k = 0; k < 3; ++k) cam[(24 + k) * GB_THREADS] = -a.dL_dmean3D[3 * idx + k];
            }
        }

        // ---------------- covariance backward ----------------
        if (a.has_scales) {
            const float mod = a.scale_modifier;
            const bool raw = a.raw_params != 0;
            auto scale_in = [&](const float* sp, int i) { const float v = sp[i]; return raw ? act_exp(v) : v; };
            auto quat_in = [&](const float* qp) {
                const float4 q = reinterpret_cast<const float4*>(qp)[idx];
                return raw ? act_normalize(q) : q;
            };
            if (a.rot_4d) {
                // backward.cu:689-834
                const float t = a.ts[idx];
                const float dt = fsub(a.timestamp, t);
                const float4 rot = quat_in(a.rotations);
                const float4 rotr = quat_in(a.rotations_r);
                const float sc[4] = {fmul(mod, scale_in(a.scales, 3 * idx + 0)), fmul(mod, scale_in(a.scales, 3 * idx + 1)),
                                     fmul(mod, scale_in(a.scales, 3 * idx + 2)), fmul(mod, scale_in(a.scales_t, idx))};
                Sigma4 S;
                float R4[4][4];
                build_M4<true>(sc[0], sc[1], sc[2], sc[3], rot, rotr, S.M, R4);
                sigma_from_M(S);
                const float cov_t = S.s33;
                const float ctp = (a.prefilter_var > 0.0f) ? fadd(a.prefilter_var, cov_t) : cov_t;
                const float marginal = marginal_from(dt, cov_t, a.prefilter_var);
                if ((double)marginal > 0.05) {
                    const float c12[3] = {S.s03, S.s13, S.s23};
                    const float* d = g_cov;
                    float dc12[3];
                    dc12[0] = -(d[0] * c12[0] + d[1] * c12[1] * 0.5f + d[2] * c12[2] * 0.5f) * 2.0f / cov_t;
                    dc12[1] = -(d[1] * c12[0] * 0.5f + d[3] * c12[1] + d[4] * c12[2] * 0.5f) * 2.0f / cov_t;
                    dc12[2] = -(d[2] * c12[0] * 0.5f + d[4] * c12[1] * 0.5f + d[5] * c12[2]) * 2.0f / cov_t;
                    float dcovt = (c12[0] * c12[0] * d[0] + c12[0] * c12[1] * d[1] + c12[0] * c12[2] * d[2] +
                                   c12[1] * c12[1] * d[3] + c12[1] * c12[2] * d[4] + c12[2] * c12[2] * d[5]) /
                                  (cov_t * cov_t);
                    // opacity -> marginal chain (:769-774)
                    const float dop = a.dL_dopacity[idx];
                    const float dmarg = dop * (raw ? act_sigmoid(a.opacities[idx]) : a.opacities[idx]);
                    a.dL_dopacity[idx] = dop * marginal;
                    const float dmarg_dcovt = marginal * dt * dt / 2 / (ctp * ctp);
                    const float dmarg_dt = marginal * dt / ctp;
                    dcovt += dmarg_dcovt * dmarg;
                    float dL_dt = dmarg * dmarg_dt;
                    // mean-shift chain (:777-782)
                    dc12[0] += g_mean[0] / cov_t * dt;
                    dc12[1] += g_mean[1] / cov_t * dt;
                    dc12[2] += g_mean[2] / cov_t * dt;
                    const float ddot = g_mean[0] * c12[0] + g_mean[1] * c12[1] + g_mean[2] * c12[2];
                    dcovt += -ddot / (cov_t * cov_t) * dt;
                    dL_dt += -ddot / cov_t;
                    g_ts += dL_dt;

                    float gs[4];
                    cov4_bwd(d, dc12, dcovt, S.M, R4, sc, rot, rotr, gs, g_rot, g_rotr);
                    g_scale[0] = gs[0]; g_scale[1] = gs[1]; g_scale[2] = gs[2]; g_scale_t = gs[3];
                }
            } else {
                // backward.cu:621-684 (and no marginal-opacity gradient for non-rot 4D, :917-919)
                const float4 q = quat_in(a.rotations);
                const float sc[3] = {mod * scale_in(a.scales, 3 * idx + 0), mod * scale_in(a.scales, 3 * idx + 1),
                                     mod * scale_in(a.scales, 3 * idx + 2)};
                const float r = q.x, x = q.y, y = q.z, z = q.w;
                float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                                 {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                                 {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
                float M2[3][3];
#pragma unroll
                for (int c = 0; c < 3; ++c)
#pragma unroll
                    for (int rr = 0; rr < 3; ++rr) M2[c][rr] = 2.0f * sc[rr] * R[c][rr];
                const float* d = g_cov;
                const float dS[3][3] = {{d[0], 0.5f * d[1], 0.5f * d[2]}, {0.5f * d[1], d[3], 0.5f * d[4]},
                                        {0.5f * d[2], 0.5f * d[4], d[5]}};
                float dM[3][3];
                mat3_mul(M2, dS, dM);
                float Nt[3][3];   // dL_dMt after scaling: Nt[i][j] = s_i * dL_dM[j][i]
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                    float acc = 0.f;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        acc += R[c][i] * dM[c][i];
                        Nt[i][c] = sc[i] * dM[c][i];
                    }
                    g_scale[i] = acc;
                }
                g_rot[0] = 2 * z * (Nt[0][1] - Nt[1][0]) + 2 * y * (Nt[2][0] - Nt[0][2]) + 2 * x * (Nt[1][2] - Nt[2][1]);
                g_rot[1] = 2 * y * (Nt[1][0] + Nt[0][1]) + 2 * z * (Nt[2][0] + Nt[0][2]) + 2 * r * (Nt[1][2] - Nt[2][1]) -
                           4 * x * (Nt[2][2] + Nt[1][1]);
                g_rot[2] = 2 * x * (Nt[1][0] + Nt[0][1]) + 2 * r * (Nt[2][0] - Nt[0][2]) + 2 * z * (Nt[1][2] + Nt[2][1]) -
                           4 * y * (Nt[2][2] + Nt[0][0]);
                g_rot[3] = 2 * r * (Nt[0][1] - Nt[1][0]) + 2 * x * (Nt[2][0] + Nt[0][2]) + 2 * y * (Nt[1][2] + Nt[2][1]) -
                           4 * z * (Nt[1][1] + Nt[0][0]);
            }
            if (raw) {
                // chain through the activations the forward applied (autograd of exp / F.normalize in the reference's
                // getters, scene/gaussian_model.py:179-219): gradients now refer to the RAW parameters
#pragma unroll
                for (int i = 0; i < 3; ++i) g_scale[i] *= act_exp(a.scales[3 * idx + i]);
                if (a.scales_t) g_scale_t *= act_exp(a.scales_t[idx]);
                const float4 gq = act_normalize_bwd(reinterpret_cast<const float4*>(a.rotations)[idx],
                                                    make_float4(g_rot[0], g_rot[1], g_rot[2], g_rot[3]));
                g_rot[0] = gq.x; g_rot[1] = gq.y; g_rot[2] = gq.z; g_rot[3] = gq.w;
                if (a.rot_4d) {
                    const float4 gr = act_normalize_bwd(reinterpret_cast<const float4*>(a.rotations_r)[idx],
                                                        make_float4(g_rotr[0], g_rotr[1], g_rotr[2], g_rotr[3]));
                    g_rotr[0] = gr.x; g_rotr[1] = gr.y; g_rotr[2] = gr.z; g_rotr[3] = gr.w;
                }
            }
        }
        if (a.raw_params) {
            // d sigmoid: dL/dlogit = dL/dopacity * (1 - o) * o   (torch's sigmoid_backward)
            const float o = act_sigmoid(a.opacities[idx]);
            a.dL_dopacity[idx] = a.dL_dopacity[idx] * (1.f - o) * o;
        }
    }

    // every row of every overwritten tensor
#pragma unroll
    for (int i = 0; i < 3; ++i) a.dL_dmean3D[3 * idx + i] = g_mean[i];
#pragma unroll
    for (int i = 0; i < 6; ++i) a.dL_dcov3D[6 * idx + i] = g_cov[i];
    a.dL_dts[idx] = g_ts;
#pragma unroll
    for (int i = 0; i < 3; ++i) a.dL_dscale[3 * idx + i] = g_scale[i];
    a.dL_dscale_t[idx] = g_scale_t;
    reinterpret_cast<float4*>(a.dL_drot)[idx] = make_float4(g_rot[0], g_rot[1], g_rot[2], g_rot[3]);
    reinterpret_cast<float4*>(a.dL_drot_r)[idx] = make_float4(g_rotr[0], g_rotr[1], g_rotr[2], g_rotr[3]);
}

__global__ void __launch_bounds__(GB_THREADS, 8) geom_bwd_kernel(const PreprocessBwdParams a_, const int has_sh_part) {
    geom_bwd_body<false>(a_, has_sh_part);
}

// the batched entry (fdgs_forward_batch / fdgs_backward_batch): one view per blockIdx.y
__global__ void __launch_bounds__(GB_THREADS, 8) geom_bwd_batch_kernel(const PreprocessBwdParams a_, const int has_sh_part) {
    geom_bwd_body<true>(a_, has_sh_part);
}

// geom_bwd with the camera gradient: each block sums its rows' CAM_TERMS camera terms and writes one partial per term,
// partials[(view * CAM_TERMS + term) * gridDim.x + blockIdx.x].  The terms wait in shared memory, not registers, while
// the covariance chain runs (the kernel keeps geom_bwd's 8 CTAs per SM); then per term a butterfly over each warp and
// the four warps in order.  No floating-point atomics: the result does not depend on scheduling.
template <bool BATCH>
__global__ void __launch_bounds__(GB_THREADS, 8) geom_bwd_cam_kernel(const PreprocessBwdParams a_, const int has_sh_part,
                                                                     float* __restrict__ partials) {
    __shared__ float terms[CAM_TERMS][GB_THREADS];
    __shared__ float warp_sum[GB_THREADS / 32][CAM_TERMS];
#pragma unroll
    for (int s = 0; s < CAM_TERMS; ++s) terms[s][threadIdx.x] = 0.f;
    geom_bwd_body<BATCH, true>(a_, has_sh_part, &terms[0][threadIdx.x]);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int s = 0; s < CAM_TERMS; ++s) {   // every slot is read back by the thread that wrote it
        float v = terms[s][threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) warp_sum[warp][s] = v;
    }
    __syncthreads();
    if (threadIdx.x < CAM_TERMS) {
        float v = warp_sum[0][threadIdx.x];
#pragma unroll
        for (int w = 1; w < GB_THREADS / 32; ++w) v += warp_sum[w][threadIdx.x];
        partials[((size_t)blockIdx.y * CAM_TERMS + threadIdx.x) * gridDim.x + blockIdx.x] = v;
    }
}

// one block per view, one warp per term: the view's block partials summed in fp64 in a fixed order (lane l takes blocks
// l, l + 32, ...; then a butterfly), rounded once, and scattered to the [16] / [16] / [3] outputs in the tensors'
// layout, with exact zeros in the entries the forward does not use (see CameraGradParams)
__global__ void __launch_bounds__(CAM_TERMS * 32) camera_grad_finish_kernel(const CameraGradParams c, const int blocks) {
    const int view = blockIdx.x, s = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* src = c.partials + ((size_t)view * CAM_TERMS + s) * (size_t)blocks;
    double acc = 0.0;
    for (int b = lane; b < blocks; b += 32) acc += (double)src[b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
        const float v = (float)acc;
        if (s < 12) c.dL_dviewmatrix[16 * view + 4 * (s / 3) + s % 3] = v;
        else if (s < 24) c.dL_dprojmatrix[16 * view + 4 * ((s - 12) / 3) + ((s - 12) % 3 == 2 ? 3 : (s - 12) % 3)] = v;
        else c.dL_dcampos[3 * view + s - 24] = v;
    }
    if (threadIdx.x < 4) {
        c.dL_dviewmatrix[16 * view + 4 * threadIdx.x + 3] = 0.f;
        c.dL_dprojmatrix[16 * view + 4 * threadIdx.x + 2] = 0.f;
    }
}

// one thread per element of a tensor (blockIdx.y), its B view rows added in view order with round-to-nearest adds
__global__ void __launch_bounds__(256) view_sum_kernel(const ViewSumParams p) {
    const int i = blockIdx.y;
    const long long n = p.count[i];
    const float* __restrict__ src = p.src[i];
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        float s = src[e];
        for (int v = 1; v < p.B; ++v) s = __fadd_rn(s, src[(size_t)v * n + e]);
        p.dst[i][e] = s;
    }
}

// reference: rasterizer_impl.cu:54-67 checkFrustum + auxiliary.h:140-163
__global__ void mark_visible_kernel(int P, const float* __restrict__ means, const float* __restrict__ V,
                                    unsigned char* __restrict__ present) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const float z = xform_row(V[2], V[6], V[10], V[14], means[3 * idx], means[3 * idx + 1], means[3 * idx + 2]);
    present[idx] = (z <= 0.2f) ? 0 : 1;
}

}  // namespace

int preprocess_bwd_kernel_count(const PreprocessBwdParams& p) {
    return (p.shs != nullptr && p.M > 0 && (p.dL_dsh != nullptr || p.sh_factors != nullptr)) ? 2 : 1;
}

using PreprocessBwdKernel = void (*)(const PreprocessBwdParams);
using PreprocessBwdKernelG = void (*)(const PreprocessBwdParams, const int);

// the SH backward of one staging mode: dense rows or colour factors, or the batched entry's per-view factors
template <int STAGE, bool BATCH>
static PreprocessBwdKernel sh_bwd_for(bool factors) {
    if (BATCH) return sh_bwd_batch_kernel<STAGE>;
    return factors ? sh_bwd_kernel<STAGE, true> : sh_bwd_kernel<STAGE, false>;
}

template <bool BATCH>
static cudaError_t preprocess_bwd(const PreprocessBwdParams& p, cudaStream_t stream, const CameraGradParams* cam) {
    const bool factors = p.sh_factors != nullptr;
    const bool has_sh = p.shs != nullptr && p.M > 0 && (p.dL_dsh != nullptr || factors);
    const unsigned views = BATCH ? (unsigned)p.vb.B : 1u;
    if (has_sh) {
        const dim3 blocks((p.P + SB_THREADS - 1) / SB_THREADS, views);
        const bool split = p.shs_rest != nullptr;
        if (p.sh_bulk_ok && (!split || p.M % 16 == 0)) {
            const size_t smem = (size_t)SB_CAP * p.sh_row_stride_floats * sizeof(float);
            static PerDeviceOnce once[4];
            const PreprocessBwdKernel k = split ? sh_bwd_for<2, BATCH>(factors) : sh_bwd_for<1, BATCH>(factors);
            cudaError_t e0 = ensure_dynamic_smem(k, 200 * 1024, once[2 * split + factors]);
            if (e0 != cudaSuccess) return e0;
            k<<<blocks, SB_THREADS, smem, stream>>>(p);
        } else {
            sh_bwd_for<0, BATCH>(factors)<<<blocks, SB_THREADS, 0, stream>>>(p);
        }
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    const unsigned blocks = (unsigned)camera_grad_blocks(p.P);
    if (cam) {
        geom_bwd_cam_kernel<BATCH><<<dim3(blocks, views), GB_THREADS, 0, stream>>>(p, has_sh ? 1 : 0, cam->partials);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        return launch_camera_grad_finish(*cam, (int)blocks, (int)views, stream);
    }
    const PreprocessBwdKernelG g = BATCH ? geom_bwd_batch_kernel : geom_bwd_kernel;
    g<<<dim3(blocks, views), GB_THREADS, 0, stream>>>(p, has_sh ? 1 : 0);
    return cudaGetLastError();
}

cudaError_t launch_preprocess_bwd(const PreprocessBwdParams& p, cudaStream_t stream, const CameraGradParams* cam) {
    if (p.P <= 0) return cudaSuccess;
    return p.vb.scalars ? preprocess_bwd<true>(p, stream, cam) : preprocess_bwd<false>(p, stream, cam);
}

int camera_grad_blocks(int P) { return P > 0 ? (P + GB_THREADS - 1) / GB_THREADS : 0; }

cudaError_t launch_camera_grad_finish(const CameraGradParams& c, int blocks, int views, cudaStream_t stream) {
    camera_grad_finish_kernel<<<(unsigned)views, CAM_TERMS * 32, 0, stream>>>(c, blocks);
    return cudaGetLastError();
}

cudaError_t launch_view_sum(const ViewSumParams& p, cudaStream_t stream) {
    if (p.n <= 0) return cudaSuccess;
    long long most = 0;
    for (int i = 0; i < p.n; ++i) most = p.count[i] > most ? p.count[i] : most;
    if (most <= 0) return cudaSuccess;
    const long long blocks = (most + 255) / 256;
    view_sum_kernel<<<dim3((unsigned)(blocks < 65535 * 16 ? blocks : 65535 * 16), p.n), 256, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_sh_outer_sum(const ShSumParams& p, cudaStream_t stream) {
    if (p.P <= 0) return cudaSuccess;
    if ((long long)p.K * p.V > 0)
        sh_outer_dir_kernel<<<(unsigned)(((long long)p.K * p.V + 255) / 256), 256, 0, stream>>>(p);
    const int union_blocks = (int)(((long long)p.K + SO_ROWS - 1) / SO_ROWS);
    // without slot_of every row is in the union (K = P): no zero rows
    const int zero_blocks = p.slot_of ? (int)(((long long)p.P + 127) / 128) : 0;
    sh_outer_sum_kernel<<<(unsigned)(union_blocks + zero_blocks), 128, 0, stream>>>(p, union_blocks);
    return cudaGetLastError();
}

cudaError_t launch_mark_visible(int P, const float* means3D, const float* viewmatrix, unsigned char* present,
                                cudaStream_t stream) {
    if (P <= 0) return cudaSuccess;
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, viewmatrix, present);
    return cudaGetLastError();
}

}  // namespace fdgs
