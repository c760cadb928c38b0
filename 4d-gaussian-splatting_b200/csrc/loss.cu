// loss.cu -- fused photometric loss of the training step: (1 - lambda) * L1 + lambda * (1 - SSIM), forward and backward.
//
// Replaces, in the reference, the step right after the rasterizer (SURVEY.md section 8(f) row 3):
//   l1_loss (utils/loss_utils.py:18-19), ssim / _ssim (:39-64: five grouped 11x11 Gaussian conv2d's over the image,
//   the ground truth and their products, ~10 elementwise kernels) and their autograd backward (five more
//   convolutions), combined as train.py:115-117.
// Here: two kernels.
//   ssim_fwd_kernel   one CTA per 32x32 pixel tile and channel: stages the tile + 5-pixel halo of both images in shared
//                     memory once, runs the separable 11-tap Gaussian (sigma 1.5, zero padding like conv2d's
//                     padding = 5) over x, y, x^2, y^2 and d^2 (d = x - y), evaluates the SSIM map as
//                     S = (1 - mu_d^2 / B1)(1 - sigma_dd / B2) (ssim_common.cuh: ssim_diff_terms) and its three partial
//                     derivatives dS/dmu_x, dS/dE[x^2], dS/dE[d^2] per pixel (ground-truth moments fixed), writes those
//                     three planes and accumulates the two loss sums (sum |x - y|, sum SSIM) with one double atomicAdd
//                     per CTA each.
//   ssim_bwd_kernel   dL/dx = -lambda/N * (G*a + 2 x (G*b) + 2 (x - y) (G*c)) + (1 - lambda)/N * sign(x - y): the
//                     adjoint of the windowed means is the same symmetric separable filter applied to the derivative
//                     planes.
// x and y are filtered about a per-tile shift s (the render's value at the tile centre), which the variances do not
// depend on: the fp32 window's weights sum to 1 only to ~1e-7, which biases sigma = E[x^2] - mu^2 by ~1e-7 x^2; about
// the shift it is ~1e-7 (x - s)^2, negligible against C2 in the flat regions where B2 ~ C2.  The derivative with
// respect to E[(x - s)^2] is folded into the a plane (a - 2 s b), so the backward needs no shift.
// Filtering d^2 instead of xy is the reference's S in exact arithmetic.  In fp32 it keeps near-identical renders (late
// training) accurate: sigma_dd comes from the small d instead of from differences of terms of order E[x^2], and a, b
// and 2d c are each of the order of the gradient, where the xy form's 2x (G*b) and y (G*c) are of order 1/B2 ~ 10^3 and
// cancel to it.
// HBM traffic: forward reads 2 and writes 3 planes per channel, backward reads 5 and writes 1 -- 11 plane passes
// (181 MB at 3 x 1352 x 1014) against ~60 for the reference's op-by-op path; the kernels are bound by the shared-memory
// filter passes, not by HBM.  dL/dx is the dL_dpix the blend backward consumes (fdgs_backward_args.dL_dpix).
#include "fdgs_internal.h"
#include "ssim_common.cuh"

namespace fdgs {
namespace {

constexpr int LT = 32;            // tile edge (pixels)
constexpr int LR = SSIM_R;        // filter radius (ssim_common.cuh)
constexpr int LW = LT + 2 * LR;   // staged edge
constexpr int LTHREADS = 256;

// x, y: [C,H,W]; maps: [3,C,H,W] (a = dS/dmu_x, b = dS/dE[xx], c = dS/dE[dd]); sums[0] += sum|x-y|, sums[1] += sum SSIM
__global__ void __launch_bounds__(LTHREADS) ssim_fwd_kernel(const float* __restrict__ x, const float* __restrict__ y, int H, int W,
                                                           const GaussWin win, float* __restrict__ maps, size_t plane_stride,
                                                           double* __restrict__ sums) {
    __shared__ float sx[LW][LW + 1], sy[LW][LW + 1];
    __shared__ float hz[5][LW][LT + 1];          // horizontal pass of x, y, xx, yy, dd
    __shared__ double red[2][LTHREADS / 32];
    const int ch = blockIdx.z;
    const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT;
    const size_t HW = (size_t)H * W;
    const float* px = x + ch * HW;
    const float* py = y + ch * HW;
    const float sh = px[(size_t)min(y0 + LT / 2, H - 1) * W + min(x0 + LT / 2, W - 1)];   // the tile's shift
    for (int i = threadIdx.x; i < LW * LW; i += LTHREADS) {
        const int r = i / LW, c = i - r * LW;
        const int gy = y0 + r - LR, gx = x0 + c - LR;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;   // zero padding (F.conv2d padding = 5)
        sx[r][c] = in ? px[(size_t)gy * W + gx] : 0.f;
        sy[r][c] = in ? py[(size_t)gy * W + gx] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < LW * LT; i += LTHREADS) {
        const int r = i / LT, c = i - r * LT;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f;
#pragma unroll
        for (int k = 0; k <= 2 * LR; ++k) {
            const float u = sx[r][c + k], v = sy[r][c + k], w = win.g[k];
            const float us = u - sh, vs = v - sh, d = u - v;
            a0 = fmaf(w, us, a0);
            a1 = fmaf(w, vs, a1);
            a2 = fmaf(w, us * us, a2);
            a3 = fmaf(w, vs * vs, a3);
            a4 = fmaf(w, d * d, a4);
        }
        hz[0][r][c] = a0; hz[1][r][c] = a1; hz[2][r][c] = a2; hz[3][r][c] = a3; hz[4][r][c] = a4;
    }
    __syncthreads();
    float wsum = 0.f;
#pragma unroll
    for (int k = 0; k <= 2 * LR; ++k) wsum += win.g[k];
    const float shm = sh * (wsum * wsum);        // the window's mean of the constant s
    double l1 = 0.0, ss = 0.0;
    for (int i = threadIdx.x; i < LT * LT; i += LTHREADS) {
        const int r = i / LT, c = i - r * LT;
        const int gy = y0 + r, gx = x0 + c;
        if (gy >= H || gx >= W) continue;
        float m1 = 0.f, m2 = 0.f, e11 = 0.f, e22 = 0.f, edd = 0.f;
#pragma unroll
        for (int k = 0; k <= 2 * LR; ++k) {
            const float w = win.g[k];
            m1 = fmaf(w, hz[0][r + k][c], m1);
            m2 = fmaf(w, hz[1][r + k][c], m2);
            e11 = fmaf(w, hz[2][r + k][c], e11);
            e22 = fmaf(w, hz[3][r + k][c], e22);
            edd = fmaf(w, hz[4][r + k][c], edd);
        }
        // m1, m2, e11, e22: moments of x - s and y - s
        const float md = m1 - m2;
        const float mx = m1 + shm, my = m2 + shm;
        const SsimDiffTerms<float> t = ssim_diff_terms(mx, my, md, e11 - m1 * m1, e22 - m2 * m2, edd);
        const float sdd = t.sdd, B1 = t.B1, B2 = t.B2, P = t.P, Q = t.Q, S = t.S;
        // S = P Q as a function of (mu_{x-s}, E[(x-s)^2], E[dd]) with the ground-truth moments fixed:
        //   dP/dmu = -2 mu_d (mu_y (mu_x + mu_y) + C1) / B1^2,  dQ/dmu = 2 (mu_d B2 - mu_{x-s} sigma_dd) / B2^2,
        //   dQ/dE[(x-s)^2] = sigma_dd / B2^2,  dQ/dE[dd] = -1 / B2;  d E[(x-s)^2] / dx = 2x - 2s: a - 2 s b
        const float iB1 = 1.f / B1, iB2 = 1.f / B2;
        const float dP = -2.f * md * fmaf(my, mx + my, 0.01f * 0.01f) * iB1 * iB1;
        const float dQ = 2.f * (md * B2 - m1 * sdd) * iB2 * iB2;
        const float db = P * sdd * iB2 * iB2;
        const float da = fmaf(-2.f * sh, db, Q * dP + P * dQ);
        const float dc = -P * iB2;
        const size_t o = ch * HW + (size_t)gy * W + gx;
        maps[o] = da;
        maps[plane_stride + o] = db;
        maps[2 * plane_stride + o] = dc;
        l1 += (double)fabsf(sx[r + LR][c + LR] - sy[r + LR][c + LR]);
        ss += (double)S;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        l1 += __shfl_xor_sync(0xffffffffu, l1, d);
        ss += __shfl_xor_sync(0xffffffffu, ss, d);
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = l1; red[1][threadIdx.x >> 5] = ss; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double t0 = 0.0, t1 = 0.0;
        for (int w = 0; w < LTHREADS / 32; ++w) { t0 += red[0][w]; t1 += red[1][w]; }
        atomicAdd(&sums[0], t0);
        atomicAdd(&sums[1], t1);
    }
}

// dL_dx[C,H,W] = k_ssim * (G*a + 2 x (G*b) + 2 (x - y) (G*c)) + k_l1 * sign(x - y)
__global__ void __launch_bounds__(LTHREADS) ssim_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y, int H, int W,
                                                           const GaussWin win, const float* __restrict__ maps, size_t plane_stride,
                                                           const float* __restrict__ grad_scale, float k_l1, float k_ssim,
                                                           float* __restrict__ dL_dx) {
    __shared__ float sm[3][LW][LW + 1];
    __shared__ float hz[3][LW][LT + 1];
    const int ch = blockIdx.z;
    const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT;
    const size_t HW = (size_t)H * W;
    for (int i = threadIdx.x; i < LW * LW; i += LTHREADS) {
        const int r = i / LW, c = i - r * LW;
        const int gy = y0 + r - LR, gx = x0 + c - LR;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
        const size_t o = ch * HW + (size_t)(in ? gy : 0) * W + (in ? gx : 0);
#pragma unroll
        for (int m = 0; m < 3; ++m) sm[m][r][c] = in ? maps[m * plane_stride + o] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < LW * LT; i += LTHREADS) {
        const int r = i / LT, c = i - r * LT;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
        for (int k = 0; k <= 2 * LR; ++k) {
            const float w = win.g[k];
            a0 = fmaf(w, sm[0][r][c + k], a0);
            a1 = fmaf(w, sm[1][r][c + k], a1);
            a2 = fmaf(w, sm[2][r][c + k], a2);
        }
        hz[0][r][c] = a0; hz[1][r][c] = a1; hz[2][r][c] = a2;
    }
    __syncthreads();
    const float gs = grad_scale ? grad_scale[0] : 1.f;   // upstream d(total)/d(loss), a device scalar (no host sync)
    for (int i = threadIdx.x; i < LT * LT; i += LTHREADS) {
        const int r = i / LT, c = i - r * LT;
        const int gy = y0 + r, gx = x0 + c;
        if (gy >= H || gx >= W) continue;
        float ca = 0.f, cb = 0.f, cc = 0.f;
#pragma unroll
        for (int k = 0; k <= 2 * LR; ++k) {
            const float w = win.g[k];
            ca = fmaf(w, hz[0][r + k][c], ca);
            cb = fmaf(w, hz[1][r + k][c], cb);
            cc = fmaf(w, hz[2][r + k][c], cc);
        }
        const size_t o = ch * HW + (size_t)gy * W + gx;
        const float xv = x[o], yv = y[o];
        const float d = xv - yv;
        const float sgn = (d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f);   // torch.abs backward: sign, 0 at 0
        dL_dx[o] = gs * (k_ssim * (ca + 2.f * (xv * cb + d * cc)) + k_l1 * sgn);
    }
}

}  // namespace

cudaError_t launch_l1_ssim_fwd(const float* x, const float* y, int C, int H, int W, float* maps, double* sums, cudaStream_t stream) {
    if (C <= 0 || H <= 0 || W <= 0) return cudaSuccess;
    cudaError_t e = cudaMemsetAsync(sums, 0, 2 * sizeof(double), stream);
    if (e != cudaSuccess) return e;
    dim3 grid((W + LT - 1) / LT, (H + LT - 1) / LT, C);
    ssim_fwd_kernel<<<grid, LTHREADS, 0, stream>>>(x, y, H, W, make_window(), maps, (size_t)C * H * W, sums);
    return cudaGetLastError();
}

cudaError_t launch_l1_ssim_bwd(const float* x, const float* y, int C, int H, int W, const float* maps, const float* grad_scale,
                               float lambda_dssim, float* dL_dx, cudaStream_t stream) {
    if (C <= 0 || H <= 0 || W <= 0) return cudaSuccess;
    const float n = (float)((double)C * H * W);
    dim3 grid((W + LT - 1) / LT, (H + LT - 1) / LT, C);
    ssim_bwd_kernel<<<grid, LTHREADS, 0, stream>>>(x, y, H, W, make_window(), maps, (size_t)C * H * W, grad_scale,
                                                   (1.f - lambda_dssim) / n, -lambda_dssim / n, dL_dx);
    return cudaGetLastError();
}

}  // namespace fdgs
