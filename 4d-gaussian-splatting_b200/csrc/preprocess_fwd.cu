// preprocess_fwd.cu -- per-Gaussian forward preprocessing (one thread per Gaussian).
//
// Replaces the reference's preprocessCUDA<3> (forward.cu:355-496) together with its helpers
// computeCov3D_conditional (:279-352), computeCov3D (:242-276), computeCov2D (:198-237),
// computeColorFromSH (:20-71) / computeColorFromSH_4D (:73-195), in_frustum
// (auxiliary.h:140-163), ndc2Pix (:42-45) and getRect (:47-57).
//
// Design:
//   * geometry inputs (68 B/Gaussian) are read with coalesced 32/128-bit loads;
//   * the 12*M-byte SH row of every *visible* Gaussian is streamed global->shared with one
//     cp.async.bulk (TMA 1-D, SASS UBLKCP) per row into a compacted slot, all rows of a round
//     completing on one mbarrier; slots sit at a padded 16-byte-aligned stride so that the
//     per-thread LDS.128 reads are bank-conflict free; no register staging, no 12-byte strided LDG;
//   * out_means3D is written for every Gaussian here (the reference clones means3D first,
//     rasterize_points.cu:85, and overwrites the time-visible rows).
// All arithmetic that feeds radii / tiles / depth / conic / rgb follows the reference bit for
// bit (see fdgs_common.cuh).
#include "fdgs_internal.h"

namespace fdgs {

namespace {

constexpr int PRE_THREADS = 128;
constexpr int PRE_CAP = 48;       // shared-memory SH row slots per CTA (rendered rows per round)

__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float sqrt_approx(float x) {
    float y;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

struct ShBasis {
    float l[16];   // l0m0, l1m1, l1m0, l1p1, l2m2 .. l3p3
};

// degree-3 basis, shared by the 3D and 4D variants (reference: forward.cu:53-59 / :125-131); the
// polynomial factors are fused as in the reference kernel's SASS (3*xx - yy -> fma(xx,3,-yy) ...)
__device__ __forceinline__ void sh_basis_l3(float x, float y, float z, float xx, float yy, float zz, float xy,
                                            float l[16]) {
    const float four_zz_xx_yy = fadd(-yy, ffma(zz, 4.f, -xx));   // 4zz - xx - yy
    l[9] = fmul(fmul(y, kSH_C3[0]), ffma(xx, 3.f, -yy));
    l[10] = fmul(fmul(xy, kSH_C3[1]), z);
    l[11] = fmul(fmul(y, kSH_C3[2]), four_zz_xx_yy);
    l[12] = fmul(fmul(z, kSH_C3[3]), ffma(yy, -3.f, ffma(xx, -3.f, fadd(zz, zz))));
    l[13] = fmul(four_zz_xx_yy, fmul(x, kSH_C3[4]));
    l[14] = fmul(fsub(xx, yy), fmul(z, kSH_C3[5]));
    l[15] = fmul(fmul(x, kSH_C3[6]), ffma(yy, -3.f, xx));
}

// reference: forward.cu:79-131 (4D variant; the double-promoted l2m0 and integer literals)
__device__ __forceinline__ void sh_basis_4d(float x, float y, float z, int deg, ShBasis& B) {
    B.l[0] = kSH_C0;
    if (deg > 0) {
        B.l[1] = fmul(y, -kSH_C1);
        B.l[2] = fmul(z, kSH_C1);
        B.l[3] = fmul(x, -kSH_C1);
        if (deg > 1) {
            const float xx = fmul(x, x), yy = fmul(y, y), zz = fmul(z, z);
            const float xy = fmul(x, y), yz = fmul(y, z), xz = fmul(x, z);
            B.l[4] = fmul(xy, kSH_C2[0]);
            B.l[5] = fmul(yz, kSH_C2[1]);
            // SH_C2[2] * (2.0 * zz - xx - yy): double (forward.cu:112)
            B.l[6] = (float)(((((double)zz + (double)zz) - (double)xx) - (double)yy) * (double)kSH_C2[2]);
            B.l[7] = fmul(xz, kSH_C2[3]);
            B.l[8] = fmul(fsub(xx, yy), kSH_C2[4]);
            if (deg > 2) sh_basis_l3(x, y, z, xx, yy, zz, xy, B.l);
        }
    }
}

// Row access: v[3*i + ch] = coefficient (16*blk + i), channel ch.
struct RowSmem {
    const float4* q;   // padded shared-memory row, 16-byte aligned
    __device__ __forceinline__ void load_block(int blk, int /*M*/, float v[48]) const {
#pragma unroll
        for (int i = 0; i < 12; ++i) {
            const float4 t = q[blk * 12 + i];
            v[4 * i + 0] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
        }
    }
};
struct RowGmem {
    const float* p;    // global row (any alignment, any M); with a split row: its first 3 floats (features_dc)
    const float* p1;   // NULL, or the remaining 3 (M - 1) floats of a split row (features_rest)
    __device__ __forceinline__ void load_block(int blk, int M, float v[48]) const {
#pragma unroll
        for (int i = 0; i < 48; ++i) {
            const int k = blk * 48 + i;
            if (p1 == nullptr) v[i] = (k < 3 * M) ? __ldg(p + k) : 0.f;
            else v[i] = (k < 3) ? __ldg(p + k) : ((k < 3 * M) ? __ldg(p1 + (k - 3)) : 0.f);
        }
    }
};

// reference: forward.cu:73-195 computeColorFromSH_4D.  Returns result BEFORE the +0.5/clamp.
template <class Row>
__device__ __forceinline__ void sh_color_4d(const Row& row, int M, int deg, int deg_t, float x, float y, float z,
                                            float dir_t, float time_duration, float rgb[3]) {
    ShBasis B;
    sh_basis_4d(x, y, z, deg, B);
    float v[48];
    row.load_block(0, M, v);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        float r = fmul(v[ch], kSH_C0);
        if (deg > 0) {
            r = fadd(r, ffma(B.l[3], v[9 + ch], ffma(B.l[1], v[3 + ch], fmul(B.l[2], v[6 + ch]))));
            if (deg > 1) {
                float b = ffma(B.l[4], v[12 + ch], fmul(B.l[5], v[15 + ch]));
                b = ffma(v[18 + ch], B.l[6], b);
                b = ffma(B.l[8], v[24 + ch], ffma(B.l[7], v[21 + ch], b));
                r = fadd(r, b);
                if (deg > 2) {
                    float c = ffma(B.l[11], v[33 + ch], ffma(B.l[9], v[27 + ch], fmul(B.l[10], v[30 + ch])));
                    c = ffma(B.l[13], v[39 + ch], ffma(B.l[12], v[36 + ch], c));
                    c = ffma(B.l[15], v[45 + ch], ffma(B.l[14], v[42 + ch], c));
                    r = fadd(r, c);
                }
            }
        }
        rgb[ch] = r;
    }
    // temporal Fourier terms only exist under deg > 2 (forward.cu:142 nested in :123)
    if (deg > 2 && deg_t > 0) {
        const double ang = ((double)dir_t * (2 * FDGS_MY_PI)) / (double)time_duration;
        const float t1 = (float)cos(ang);
        row.load_block(1, M, v);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            float s = ffma(v[ch], B.l[0], fmul(B.l[1], v[3 + ch]));
#pragma unroll
            for (int k = 2; k < 16; ++k) s = ffma(B.l[k], v[3 * k + ch], s);
            rgb[ch] = ffma(s, t1, rgb[ch]);
        }
        if (deg_t > 1) {
            const double ang2 = (((double)dir_t * (2 * FDGS_MY_PI)) * 2.0) / (double)time_duration;
            const float t2 = (float)cos(ang2);
            row.load_block(2, M, v);
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                float s = ffma(v[ch], B.l[0], fmul(B.l[1], v[3 + ch]));
#pragma unroll
                for (int k = 2; k < 16; ++k) s = ffma(B.l[k], v[3 * k + ch], s);
                rgb[ch] = ffma(s, t2, rgb[ch]);
            }
        }
    }
}

// reference: forward.cu:20-71 computeColorFromSH (3D).  Returns result BEFORE the +0.5/clamp.
template <class Row>
__device__ __forceinline__ void sh_color_3d(const Row& row, int M, int deg, float x, float y, float z,
                                            float rgb[3]) {
    float v[48];
    row.load_block(0, M, v);
    const float xx = fmul(x, x), yy = fmul(y, y), zz = fmul(z, z);
    const float xy = fmul(x, y), yz = fmul(y, z), xz = fmul(x, z);
    float l3[16];
    if (deg > 2) sh_basis_l3(x, y, z, xx, yy, zz, xy, l3);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        float r = fmul(v[ch], kSH_C0);
        if (deg > 0) {
            // result - C1*y*sh1 + C1*z*sh2 - C1*x*sh3 ... : one FFMA chain in the reference's SASS
            r = ffma(-fmul(y, kSH_C1), v[3 + ch], r);
            r = ffma(fmul(z, kSH_C1), v[6 + ch], r);
            r = ffma(-fmul(x, kSH_C1), v[9 + ch], r);
            if (deg > 1) {
                r = ffma(fmul(xy, kSH_C2[0]), v[12 + ch], r);
                r = ffma(fmul(yz, kSH_C2[1]), v[15 + ch], r);
                r = ffma(fmul(fsub(fsub(fadd(zz, zz), xx), yy), kSH_C2[2]), v[18 + ch], r);
                r = ffma(fmul(xz, kSH_C2[3]), v[21 + ch], r);
                r = ffma(fmul(fsub(xx, yy), kSH_C2[4]), v[24 + ch], r);
                if (deg > 2) {
#pragma unroll
                    for (int k = 9; k < 16; ++k) r = ffma(l3[k], v[3 * k + ch], r);
                }
            }
        }
        rgb[ch] = r;
    }
}

// STAGE: how the SH rows of the rendered Gaussians reach shared memory -- 0: not at all (read from global memory
// coefficient by coefficient: odd row sizes), 1: one cp.async.bulk per row (TMA 1-D; contiguous 16-byte-aligned rows),
// 2: cooperative coalesced copy by the whole CTA (split rows features_dc | features_rest of the raw-parameter entry:
// 12-byte and 564-byte pieces, which the bulk-copy engine cannot address).
// view v of a batch (blockIdx.y): the view's camera and its slices of every per-Gaussian output
__device__ __forceinline__ PreprocessFwdParams preprocess_fwd_view(PreprocessFwdParams a, int v) {
    const size_t P = (size_t)a.P;
    const ViewScalars vs = a.vb.scalars[v];
    a.viewmatrix += 16 * v;
    a.projmatrix += 16 * v;
    a.cam_pos += 3 * v;
    a.timestamp = vs.timestamp;
    a.tan_fovx = vs.tan_fovx;
    a.tan_fovy = vs.tan_fovy;
    a.focal_x = vs.focal_x;
    a.focal_y = vs.focal_y;
    a.out_means3D += 3 * v * P;
    a.radii += v * P;
    a.cov3D += 6 * v * P;
    a.grec += v * P;
    a.clamped += v * P;
    a.tiles_touched += v * P;
    a.binrec += v * P;
    return a;
}

template <int STAGE, bool BATCH>
__device__ __forceinline__ void preprocess_fwd_body(const PreprocessFwdParams& a_) {
    // an lvalue on both sides: the single-view instantiation reads its parameters in place, no copy
    PreprocessFwdParams view_;
    if (BATCH) view_ = preprocess_fwd_view(a_, blockIdx.y);
    const PreprocessFwdParams& a = BATCH ? view_ : a_;
    constexpr bool BULK = STAGE == 1;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t bar;
    __shared__ int warp_cnt[PRE_THREADS / 32];
    __shared__ int slot_idx[PRE_CAP];   // STAGE 2: Gaussian whose row occupies each slot

    const int idx = blockIdx.x * PRE_THREADS + threadIdx.x;
    const bool in_range = idx < a.P;
    if (BULK) {
        if (threadIdx.x == 0) {
            mbar_init(&bar, 1);
            mbar_fence_init();
        }
        __syncthreads();
    }

    bool visible = false;
    float depth = 0.f, px = 0.f, py = 0.f, opacity = 0.f;
    float conx = 0.f, cony = 0.f, conz = 0.f;
    int radius = 0;
    uint32_t tiles = 0;
    int rx0 = 0, ry0 = 0, rx1 = 0, ry1 = 0;   // tile rectangle
    float mx = 0.f, my = 0.f, mz = 0.f;   // (shifted) mean
    float ox = 0.f, oy = 0.f, oz = 0.f;   // original mean (SH view direction, quirk: forward.cu:480,482)

    if (in_range) {
        ox = mx = a.means3D[3 * idx + 0];
        oy = my = a.means3D[3 * idx + 1];
        oz = mz = a.means3D[3 * idx + 2];
        opacity = a.opacities[idx];
        const bool raw = a.raw_params != 0;
        if (raw) opacity = act_sigmoid(opacity);
        // scales / rotations as the covariance code below sees them: activated here when the caller passed raw parameters
        auto scale_in = [&](const float* sp, int i) { const float v = sp[i]; return raw ? act_exp(v) : v; };
        auto quat_in = [&](const float* qp) {
            const float4 q = reinterpret_cast<const float4*>(qp)[idx];
            return raw ? act_normalize(q) : q;
        };
        bool alive = true;
        float c3[6];
        if (a.cov3D_precomp != nullptr) {
#pragma unroll
            for (int i = 0; i < 6; ++i) c3[i] = a.cov3D_precomp[6 * idx + i];
        } else if (a.rot_4d) {
            // forward.cu:279-352
            const float dt = fsub(a.timestamp, a.ts[idx]);
            const float4 rot = quat_in(a.rotations);
            const float4 rotr = quat_in(a.rotations_r);
            Sigma4 S;
            build_M4(fmul(a.scale_modifier, scale_in(a.scales, 3 * idx + 0)), fmul(a.scale_modifier, scale_in(a.scales, 3 * idx + 1)),
                     fmul(a.scale_modifier, scale_in(a.scales, 3 * idx + 2)), fmul(a.scale_modifier, scale_in(a.scales_t, idx)), rot,
                     rotr, S.M);
            sigma_from_M(S);
            const float cov_t = S.s33;
            const float marginal = marginal_from(dt, cov_t, a.prefilter_var);
            if (!((double)marginal > 0.05)) {
                alive = false;
            } else {
                opacity = fmul(opacity, marginal);
                c3[0] = fsub(S.s00, fdiv(fmul(S.s03, S.s03), cov_t));
                c3[1] = fsub(S.s01, fdiv(fmul(S.s13, S.s03), cov_t));
                c3[2] = fsub(S.s02, fdiv(fmul(S.s23, S.s03), cov_t));
                c3[3] = fsub(S.s11, fdiv(fmul(S.s13, S.s13), cov_t));
                c3[4] = fsub(S.s12, fdiv(fmul(S.s23, S.s13), cov_t));
                c3[5] = fsub(S.s22, fdiv(fmul(S.s23, S.s23), cov_t));
                mx = ffma(dt, fdiv(S.s03, cov_t), mx);
                my = ffma(dt, fdiv(S.s13, cov_t), my);
                mz = ffma(dt, fdiv(S.s23, cov_t), mz);
#pragma unroll
                for (int i = 0; i < 6; ++i) a.cov3D[6 * idx + i] = c3[i];
            }
        } else {
            // forward.cu:242-276 and :431-437
            float M3[3][3];
            build_M3(fmul(a.scale_modifier, scale_in(a.scales, 3 * idx + 0)), fmul(a.scale_modifier, scale_in(a.scales, 3 * idx + 1)),
                     fmul(a.scale_modifier, scale_in(a.scales, 3 * idx + 2)), quat_in(a.rotations), M3);
            cov3_from_M3(M3, c3);
#pragma unroll
            for (int i = 0; i < 6; ++i) a.cov3D[6 * idx + i] = c3[i];
            if (a.gaussian_dim == 4) {
                const float dt = fsub(a.ts[idx], a.timestamp);
                const float sigma = fmul(a.scale_modifier, scale_in(a.scales_t, idx));
                const float marginal = marginal_from(dt, sigma, a.prefilter_var);
                if ((double)marginal <= 0.05) alive = false;
                else opacity = fmul(opacity, marginal);
            }
        }
        // out_means3D: every row (shifted where the time slice applied)
        a.out_means3D[3 * idx + 0] = mx;
        a.out_means3D[3 * idx + 1] = my;
        a.out_means3D[3 * idx + 2] = mz;

        if (alive) {
            const float* V = a.viewmatrix;
            const float* Pm = a.projmatrix;
            // in_frustum: auxiliary.h:140-163 (only the view-z test is live)
            const float vz = xform_row(V[2], V[6], V[10], V[14], mx, my, mz);
            if (vz <= 0.2f) {
                alive = false;
                if (a.prefiltered) {
                    printf("Point is filtered although prefiltered is set. This shouldn't happen!");
                    __trap();
                }
            } else {
                depth = vz;
                const float hx = xform_row(Pm[0], Pm[4], Pm[8], Pm[12], mx, my, mz);
                const float hy = xform_row(Pm[1], Pm[5], Pm[9], Pm[13], mx, my, mz);
                const float hw = xform_row(Pm[3], Pm[7], Pm[11], Pm[15], mx, my, mz);
                const float p_w = frcp(fadd(hw, 0.0000001f));
                const float projx = fmul(hx, p_w), projy = fmul(hy, p_w);

                Proj2D Pj;
                build_T(V, mx, my, mz, a.focal_x, a.focal_y, a.tan_fovx, a.tan_fovy, Pj);
                float ca, cb, cc;
                cov2d_from_T(Pj, c3, ca, cb, cc);
                ca = fadd(ca, 0.3f);
                cc = fadd(cc, 0.3f);
                // cov.x*cov.z - cov.y*cov.y: ptxas fuses the first product (SASS of the reference)
                const float det = ffma(ca, cc, -fmul(cb, cb));
                if (det == 0.0f) {
                    alive = false;
                } else {
                    const float det_inv = frcp(det);
                    conx = fmul(cc, det_inv);
                    cony = fmul(det_inv, -cb);
                    conz = fmul(ca, det_inv);
                    const float mid = fmul(fadd(ca, cc), 0.5f);
                    const float sq = fsqrt(fmaxf(ffma(mid, mid, -det), 0.1f));
                    const float lam = fmaxf(fadd(mid, sq), fsub(mid, sq));
                    const float my_radius = ceilf(fmul(fsqrt(lam), 3.f));
                    px = ndc2pix(projx, a.W);
                    py = ndc2pix(projy, a.H);
                    radius = (int)my_radius;
                    get_rect(px, py, radius, a.grid_x, a.grid_y, rx0, ry0, rx1, ry1);
                    tiles = (uint32_t)((rx1 - rx0) * (ry1 - ry0));
                    if (tiles == 0 || radius < 1) alive = false;
                }
            }
        }
        visible = alive;
    }

    // ---- colour ------------------------------------------------------------------------------
    const bool need_sh = (a.colors_precomp == nullptr);
    float rgb[3] = {0.f, 0.f, 0.f};
    uint8_t clamp_bits = 0;
    if (need_sh) {
        const int row_floats = 3 * a.M;
        auto eval = [&](auto row) {
            const float dx = fsub(ox, a.cam_pos[0]), dy = fsub(oy, a.cam_pos[1]), dz = fsub(oz, a.cam_pos[2]);
            const float len = fsqrt(ffma(dz, dz, ffma(dx, dx, fmul(dy, dy))));
            const float x = fdiv(dx, len), y = fdiv(dy, len), z = fdiv(dz, len);
            const bool sh3d = (a.gaussian_dim == 3) || a.force_sh_3d;
            if (sh3d) sh_color_3d(row, a.M, a.D, x, y, z, rgb);
            else sh_color_4d(row, a.M, a.D, a.D_t, x, y, z, fsub(a.ts[idx], a.timestamp), a.time_duration, rgb);
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const float r = fadd(rgb[ch], 0.5f);
                if (r < 0.f) { clamp_bits |= (1u << ch); rgb[ch] = 0.f; }
                else rgb[ch] = r;
            }
        };
        if (STAGE != 0) {
            // Only the rows of RENDERED Gaussians are fetched, into PRE_CAP shared-memory slots handed out by a
            // block-level compaction (typically a third of a CTA's Gaussians are rendered): a third of the
            // shared memory of a slot-per-thread layout, so twice the CTAs per SM stay resident to hide the
            // latency of the fp32/fp64 chain above.  More rendered rows than slots -> another round.
            const unsigned bal = __ballot_sync(0xffffffffu, visible);
            const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
            if (lane == 0) warp_cnt[warp] = __popc(bal);
            __syncthreads();
            int base = 0, nvis = 0;
#pragma unroll
            for (int w = 0; w < PRE_THREADS / 32; ++w) {
                if (w < warp) base += warp_cnt[w];
                nvis += warp_cnt[w];
            }
            const int my_rank = base + __popc(bal & ((1u << lane) - 1u));
            float* rows = reinterpret_cast<float*>(smem_raw);
            const int stride = a.sh_row_stride_floats;   // padded, multiple of 4
            for (int round = 0, lo = 0; lo < nvis; ++round, lo += PRE_CAP) {
                const int cnt = min(PRE_CAP, nvis - lo);
                const bool mine = visible && my_rank >= lo && my_rank < lo + cnt;
                if (round > 0) __syncthreads();   // the previous round's readers are done with the slots
                float* slot = rows + (size_t)(my_rank - lo) * stride;
                if (BULK) {
                    if (threadIdx.x == 0) mbar_expect_tx(&bar, (uint32_t)cnt * (uint32_t)row_floats * 4u);
                    if (mine) {
                        bulk_g2s(slot, a.shs + (size_t)idx * row_floats, (uint32_t)row_floats * 4u, &bar);
                        mbar_wait(&bar, (uint32_t)round & 1u);
                    }
                } else {
                    // split rows: a warp per row, asynchronous 4-byte copies (LDGSTS) -- all rows of the round in flight at once
                    if (mine) slot_idx[my_rank - lo] = idx;
                    __syncthreads();
                    const int rest_floats = row_floats - 3;
                    for (int sidx = threadIdx.x >> 5; sidx < cnt; sidx += PRE_THREADS / 32) {
                        const size_t g = (size_t)slot_idx[sidx];
                        split_row_to_smem(rows + (size_t)sidx * stride, a.shs + g * 3, a.shs_rest + g * rest_floats, row_floats,
                                          threadIdx.x & 31);
                    }
                    cp_async_wait_all();
                    __syncthreads();
                }
                if (mine) eval(RowSmem{reinterpret_cast<const float4*>(slot)});
            }
        } else if (visible) {
            if (a.shs_rest) eval(RowGmem{a.shs + (size_t)idx * 3, a.shs_rest + (size_t)idx * (row_floats - 3)});
            else eval(RowGmem{a.shs + (size_t)idx * row_floats, nullptr});
        }
    } else if (visible) {
        rgb[0] = a.colors_precomp[3 * idx + 0];
        rgb[1] = a.colors_precomp[3 * idx + 1];
        rgb[2] = a.colors_precomp[3 * idx + 2];
    }

    if (in_range) {
        a.radii[idx] = visible ? radius : 0;
        a.tiles_touched[idx] = visible ? tiles : 0u;
        uint4 brec = make_uint4(0u, 0u, 0u, 0u);
        if (visible) {
            a.clamped[idx] = clamp_bits;
            // The 64-byte record every (tile, Gaussian) instance copies (binning.cu).  Besides the
            // reference's means2D / conic_opacity / rgb / depth it carries the culling data of the
            // blend kernels: the Gaussian can only contribute where alpha = min(0.99, o*exp(power))
            // reaches 1/255 (forward.cu:590), i.e. where q(d) = -power <= log(255*o).  pmin =
            // -(log(255*o) + slack) and the slopes -B/C, -B/A let a warp minimise the convex
            // quadratic q over its pixel rectangle exactly (fdgs_common.cuh: rect_may_contribute).
            // Conservative: used only to SKIP work, never to change a result.
            float pmin, sbc = 0.f, sba = 0.f;
            const float cdet = conx * conz - cony * cony;
            if (opacity < 0.00392156886f) {   // alpha <= o < 1/255 everywhere: never contributes
                pmin = INFINITY;
            } else if (!(opacity <= 3.0e38f) || !(conx > 0.f) || !(conz > 0.f) || !(cdet > 0.f) || !(cdet <= 3.0e38f)) {
                pmin = -INFINITY;             // irregular inputs (NaN/inf opacity, non-PD conic): no culling
            } else {
                pmin = -(logf(255.0f * opacity) + 0.02f);
                sbc = -cony / conz;
                sba = -cony / conx;
                if (!(fabsf(sbc) <= 3.0e38f) || !(fabsf(sba) <= 3.0e38f)) { pmin = -INFINITY; sbc = sba = 0.f; }
            }
            // Compact record for the binning passes: tile rectangle + depth bits + tile mask.  The reference lists the
            // Gaussian in every tile of the square of half-width ceil(3 sigma_max) around its centre
            // (auxiliary.h:46-59 getRect) although only the pixels of the alpha >= 1/255 ellipse can ever blend it;
            // with tile_cull the rectangle is shrunk to the tiles the ellipse's bounding box touches and, for
            // rectangles of up to 32 tiles, bit i of the mask says whether tile i (row-major inside the shrunk
            // rectangle) can contain such a pixel at all -- the same exact, conservative test the blend kernels apply
            // per 8x4 warp rectangle.  Instances dropped here are instances no pixel would have blended: the image,
            // every other output and every gradient are unchanged; only the private tile lists get shorter.
            int tx0 = rx0, ty0 = ry0, tx1 = rx1, ty1 = ry1;
            uint32_t tmask = 0xffffffffu;
            if (a.tile_cull) {
                if (pmin == INFINITY) {
                    tx1 = tx0; ty1 = ty0;
                } else if (pmin > -3.0e38f && cdet > 2.0e-3f * conx * conz) {
                    // (Very thin Gaussians -- axis ratio above ~2000, det < 2e-3 A C -- keep the reference's rectangle: far
                    // from their centre the terms of q are thousands of times larger than q itself, and the blend loop's
                    // own fp32 rounding of `power` can then exceed the 0.02 slack of the cut.)
                    // bounding box of { d : 0.5 d^T Q d <= -pmin }: half extents sqrt(2 q C / det), sqrt(2 q A / det)
                    // (approximate reciprocal / square root, 1-2 ulp: far inside the margins below)
                    const float q2 = -2.f * pmin;
                    const float q2_det = q2 * rcp_approx(cdet);
                    const float ex = sqrt_approx(q2_det * conz) * 1.0001f + 0.01f;
                    const float ey = sqrt_approx(q2_det * conx) * 1.0001f + 0.01f;
                    if (ex <= 1.0e6f && ey <= 1.0e6f && fabsf(px) <= 1.0e6f && fabsf(py) <= 1.0e6f) {
                        // pixel centres are the integers: pixel p lies in tile floor(p / 16)
                        tx0 = max(rx0, (int)floorf((px - ex) * (1.0f / TILE_X)));
                        tx1 = min(rx1, (int)floorf((px + ex) * (1.0f / TILE_X)) + 1);
                        ty0 = max(ry0, (int)floorf((py - ey) * (1.0f / TILE_Y)));
                        ty1 = min(ry1, (int)floorf((py + ey) * (1.0f / TILE_Y)) + 1);
                        if (tx1 <= tx0 || ty1 <= ty0) { tx1 = tx0; ty1 = ty0; }
                        const int tw = tx1 - tx0, tn = tw * (ty1 - ty0);
                        // Per tile row, the x-interval [L, U] of the ellipse inside the row's y-band (the ellipse cut by
                        // a band is convex: its x-extent peaks at dy* = -(B/C) dx, so when dy* lies outside the band the
                        // extent is reached on the band edge nearest to it: a root of A dx^2 + 2 B dy dx + C dy^2 = 2 q).
                        // A tile takes an instance iff its columns meet [L, U] -- in exact arithmetic the same decision as
                        // minimising q over the tile; margins of 1e-3 |x| + 0.01 px cover the rounding.
                        if (tn > 0 && tn <= 32 && (tx1 - tx0) > 1 && (ty1 - ty0) > 1) {
                            tmask = 0u;
                            const float inv_a = rcp_approx(conx);
                            const float dy_hi = sbc * ex, dy_lo = -dy_hi;     // dy of the right-most / left-most ellipse point
                            int bit0 = 0;
                            for (int cy = ty0; cy < ty1; ++cy, bit0 += tw) {
                                const float a0 = (float)(cy * TILE_Y) - py, b0 = a0 + (float)(TILE_Y - 1);
                                float U = ex, L = -ex;
                                bool hit = true;
                                if (!(dy_hi >= a0 && dy_hi <= b0)) {
                                    const float dyc = fminf(fmaxf(dy_hi, a0), b0);
                                    const float disc = q2 * conx - cdet * dyc * dyc;
                                    hit = disc >= -1.0e-3f * q2 * conx;
                                    U = (-cony * dyc + sqrt_approx(fmaxf(disc, 0.f))) * inv_a;
                                }
                                if (hit && !(dy_lo >= a0 && dy_lo <= b0)) {
                                    const float dyc = fminf(fmaxf(dy_lo, a0), b0);
                                    const float disc = q2 * conx - cdet * dyc * dyc;
                                    hit = disc >= -1.0e-3f * q2 * conx;
                                    L = (-cony * dyc - sqrt_approx(fmaxf(disc, 0.f))) * inv_a;
                                }
                                if (!hit) continue;
                                U += 1.0e-3f * fabsf(U) + 0.01f;
                                L -= 1.0e-3f * fabsf(L) + 0.01f;
                                const int c0 = max(tx0, (int)floorf((px + L) * (1.0f / TILE_X)));
                                const int c1 = min(tx1 - 1, (int)floorf((px + U) * (1.0f / TILE_X)));
                                if (c1 >= c0)
                                    tmask |= (uint32_t)(((1ull << (c1 - c0 + 1)) - 1ull) << (bit0 + c0 - tx0));
                            }
                            if (tmask == 0u) { tx1 = tx0; ty1 = ty0; }
                        }
                    }
                }
            }
            if (tx1 > tx0 && ty1 > ty0)
                brec = make_uint4((uint32_t)tx0 | ((uint32_t)ty0 << 16), (uint32_t)tx1 | ((uint32_t)ty1 << 16), __float_as_uint(depth), tmask);
            const float fx = a.flows ? a.flows[2 * idx + 0] : 0.f, fy = a.flows ? a.flows[2 * idx + 1] : 0.f;
            float4* dst = reinterpret_cast<float4*>(a.grec + idx);
            dst[0] = make_float4(px, py, pmin, __uint_as_float((uint32_t)idx));
            dst[1] = make_float4(conx, cony, conz, opacity);
            dst[2] = make_float4(rgb[0], rgb[1], rgb[2], depth);
            dst[3] = make_float4(fx, fy, sbc, sba);
        }
        a.binrec[idx] = brec;   // written for EVERY Gaussian; all zero = no tile
    }
}

template <int STAGE>
__global__ void __launch_bounds__(PRE_THREADS, 5) preprocess_fwd_kernel(const PreprocessFwdParams a_) {
    preprocess_fwd_body<STAGE, false>(a_);
}

// the batched entry (fdgs_forward_batch / fdgs_backward_batch): one view per blockIdx.y
template <int STAGE>
__global__ void __launch_bounds__(PRE_THREADS, 5) preprocess_fwd_batch_kernel(const PreprocessFwdParams a_) {
    preprocess_fwd_body<STAGE, true>(a_);
}

}  // namespace

// test hook: the in-kernel activations of the raw-parameter entry, applied to plain arrays (tests compare them with
// torch.exp / torch.sigmoid / F.normalize bit for bit)
__global__ void debug_activate_kernel(int n, const float* __restrict__ log_s, const float* __restrict__ logit,
                                      const float* __restrict__ quat, float* __restrict__ s_out,
                                      float* __restrict__ o_out, float* __restrict__ q_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    s_out[i] = act_exp(log_s[i]);
    o_out[i] = act_sigmoid(logit[i]);
    reinterpret_cast<float4*>(q_out)[i] = act_normalize(reinterpret_cast<const float4*>(quat)[i]);
}

cudaError_t launch_debug_activate(int n, const float* log_s, const float* logit, const float* quat, float* s_out, float* o_out,
                                  float* q_out, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    debug_activate_kernel<<<(n + 255) / 256, 256, 0, stream>>>(n, log_s, logit, quat, s_out, o_out, q_out);
    return cudaGetLastError();
}

template <int STAGE, bool BATCH>
static cudaError_t preprocess_fwd_stage(const PreprocessFwdParams& p, dim3 blocks, size_t smem, PerDeviceOnce* once,
                                        cudaStream_t stream) {
    const auto k = BATCH ? preprocess_fwd_batch_kernel<STAGE> : preprocess_fwd_kernel<STAGE>;
    if (once) {
        cudaError_t e = ensure_dynamic_smem(k, 200 * 1024, *once);
        if (e != cudaSuccess) return e;
    }
    k<<<blocks, PRE_THREADS, smem, stream>>>(p);
    return cudaGetLastError();
}

template <bool BATCH>
static cudaError_t preprocess_fwd(const PreprocessFwdParams& p, cudaStream_t stream) {
    const dim3 blocks((p.P + PRE_THREADS - 1) / PRE_THREADS, BATCH ? p.vb.B : 1);
    const bool staged = p.sh_bulk_ok && p.colors_precomp == nullptr;   // shared-memory staging possible (see sh_staging)
    if (!staged) return preprocess_fwd_stage<0, BATCH>(p, blocks, 0, nullptr, stream);
    const size_t smem = (size_t)PRE_CAP * p.sh_row_stride_floats * sizeof(float);
    static PerDeviceOnce once1, once2;
    return p.shs_rest ? preprocess_fwd_stage<2, BATCH>(p, blocks, smem, &once2, stream)
                      : preprocess_fwd_stage<1, BATCH>(p, blocks, smem, &once1, stream);
}

cudaError_t launch_preprocess_fwd(const PreprocessFwdParams& p, cudaStream_t stream) {
    if (p.P <= 0) return cudaSuccess;
    return p.vb.scalars ? preprocess_fwd<true>(p, stream) : preprocess_fwd<false>(p, stream);
}

}  // namespace fdgs
