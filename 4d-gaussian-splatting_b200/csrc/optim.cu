// optim.cu -- fused multi-tensor Adam over the per-Gaussian parameter groups, dense or sparse (rendered rows only).
//
// Replaces, in the reference, torch.optim.Adam(l, lr=0.0, eps=1e-15) over nine parameter groups
// (scene/gaussian_model.py:331-357) stepped once per iteration (train.py:248-249): per group a chain of foreach
// kernels -- ~7 array passes over 161 floats per Gaussian, 9 GB of traffic at 2M Gaussians (SURVEY.md 8(f) row 4).
// Here ONE launch updates every group (blockIdx.y = tensor): each element reads gradient, parameter and both moments
// once, writes parameter and moments once and (optionally) clears the gradient in the same pass.
//   dense : every row -- the same update as torch.optim.Adam (amsgrad off, weight decay 0, maximize off);
//   sparse: only the rows listed in `rows` (the Gaussians some view of the step rendered -- the rasterizer's gradient
//           rows of all others are exactly zero).  Rows not listed keep parameters AND moments untouched: this is the
//           "sparse Adam" of later 3DGS code bases, not torch's dense semantics (a dense step also moves unrendered
//           Gaussians along their decaying momentum); it is opt-in.
// Arithmetic follows torch's multi-tensor (foreach) Adam -- the default on CUDA -- op for op in fp32:
//   m = m + (g - m) * (1 - b1)          (_foreach_lerp_)
//   v = v * b2 + (g * g) * (1 - b2)     (_foreach_mul_ + _foreach_addcmul_: the product of the tensors first)
//   p = p - (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)
// with bc1 = 1 - b1^t, bc2 = 1 - b2^t computed on the host in double like torch does (fdgs_adam_scalars).  The staged
// kernel reads lr / bc1 and sqrt(bc2) per tensor from a device table instead of its arguments, so that a captured step
// runs with the learning rates and step counts of the replay, and skips its work when the rasterizer overflowed.
#include "../../include/fdgs.h"
#include "fdgs_internal.h"

namespace fdgs {
namespace {

struct AdamTable {
    float* param[FDGS_MAX_PACK];
    float* grad[FDGS_MAX_PACK];
    float* m[FDGS_MAX_PACK];
    float* v[FDGS_MAX_PACK];
    float step_size[FDGS_MAX_PACK];   // lr / bias_correction1
    int width[FDGS_MAX_PACK];
};

// The update of tensor t's rows (grid-stride over rows x width), shared by the eager and the staged kernels
template <bool SPARSE>
__device__ __forceinline__ void adam_rows(const AdamTable& tb, int t, long long rows, const long long* __restrict__ row_idx,
                                          float w1, float beta2, float w2, float eps, float ss, float sqrt_bc2, int zero_grad) {
    const int w = tb.width[t];
    float* __restrict__ P = tb.param[t];
    float* __restrict__ G = tb.grad[t];
    float* __restrict__ M = tb.m[t];
    float* __restrict__ V = tb.v[t];
    // w1 = (float)(1 - beta1), w2 = (float)(1 - beta2) formed in DOUBLE on the host, like the Python scalars torch passes
    const long long total = rows * w;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        long long e = i;
        if (SPARSE) {
            const long long r = i / w;
            e = row_idx[r] * w + (i - r * w);
        }
        const float g = G[e];
        float m = M[e], v = V[e];
        m = __fmaf_rn(__fsub_rn(g, m), w1, m);                          // lerp_: m + w1 * (g - m)
        v = __fmaf_rn(__fmul_rn(g, g), w2, __fmul_rn(v, beta2));        // _foreach_mul_ + _foreach_addcmul_: v*b2 + (g*g)*w2
        const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), sqrt_bc2), eps);     // sqrt(v) / sqrt(bc2) + eps
        P[e] = __fmaf_rn(-ss, __fdiv_rn(m, denom), P[e]);               // addcdiv_: p + (-step_size) * (m / denom)
        M[e] = m;
        V[e] = v;
        if (zero_grad) G[e] = 0.f;
    }
}

template <bool SPARSE>
__global__ void __launch_bounds__(256) adam_kernel(const AdamTable tb, long long rows, const long long* __restrict__ row_idx,
                                                   float w1, float beta2, float w2, float eps, float sqrt_bc2, int zero_grad) {
    const int t = blockIdx.y;
    adam_rows<SPARSE>(tb, t, rows, row_idx, w1, beta2, w2, eps, tb.step_size[t], sqrt_bc2, zero_grad);
}

// Dense, with the per-tensor scalars read from the device (a CUDA graph replays it with the values staged before the
// replay): scalars[3 t] = lr / bc1, scalars[3 t + 1] = sqrt(bc2), scalars[3 t + 2] = 0 holds tensor t.  status = the
// rasterizer's {R, largest tile, overflow, wrap} or NULL: an overflowed or wrapped step writes nothing.
__global__ void __launch_bounds__(256) adam_staged_kernel(const AdamTable tb, long long rows, const float* __restrict__ scalars,
                                                          const int* __restrict__ status, float w1, float beta2, float w2,
                                                          float eps) {
    if (status && (status[2] | status[3])) return;
    const int t = blockIdx.y;
    if (scalars[3 * t + 2] == 0.f) return;
    adam_rows<false>(tb, t, rows, nullptr, w1, beta2, w2, eps, scalars[3 * t], scalars[3 * t + 1], 0);
}

}  // namespace

namespace {

// The tensor table and grid of a launch over n tensors of `rows` rows
dim3 adam_table(int n, float* const* params, float* const* grads, float* const* m, float* const* v, const int* widths,
                const float* step_sizes, long long rows, AdamTable& tb) {
    long long widest = 1;
    for (int i = 0; i < n; ++i) {
        tb.param[i] = params[i]; tb.grad[i] = grads[i]; tb.m[i] = m[i]; tb.v[i] = v[i];
        tb.step_size[i] = step_sizes ? step_sizes[i] : 0.f; tb.width[i] = widths[i];
        if ((long long)widths[i] * rows > widest) widest = (long long)widths[i] * rows;
    }
    long long blocks = (widest + 255) / 256;
    if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
    return dim3((unsigned)blocks, (unsigned)n, 1);
}

}  // namespace

cudaError_t launch_adam(int n, float* const* params, float* const* grads, float* const* m, float* const* v, const int* widths,
                        const float* step_sizes, long long rows, const long long* row_idx, float w1, float beta2, float w2,
                        float eps, float sqrt_bc2, int zero_grad, cudaStream_t stream) {
    if (n <= 0 || rows <= 0) return cudaSuccess;
    AdamTable tb;
    const dim3 grid = adam_table(n, params, grads, m, v, widths, step_sizes, rows, tb);
    if (row_idx) adam_kernel<true><<<grid, 256, 0, stream>>>(tb, rows, row_idx, w1, beta2, w2, eps, sqrt_bc2, zero_grad);
    else adam_kernel<false><<<grid, 256, 0, stream>>>(tb, rows, nullptr, w1, beta2, w2, eps, sqrt_bc2, zero_grad);
    return cudaGetLastError();
}

cudaError_t launch_adam_staged(int n, float* const* params, float* const* grads, float* const* m, float* const* v,
                               const int* widths, long long rows, const float* scalars, const int* status, float w1,
                               float beta2, float w2, float eps, cudaStream_t stream) {
    if (n <= 0 || rows <= 0) return cudaSuccess;
    AdamTable tb;
    const dim3 grid = adam_table(n, params, grads, m, v, widths, nullptr, rows, tb);
    adam_staged_kernel<<<grid, 256, 0, stream>>>(tb, rows, scalars, status, w1, beta2, w2, eps);
    return cudaGetLastError();
}

}  // namespace fdgs
