// metrics.cu -- the evaluation metrics of a test view: L1, PSNR, SSIM and MS-SSIM of a batch of image pairs, in float64.
//
// Replaces, in the reference, the per-view evaluation of train.py:312-334 (training_report): l1_loss
// (utils/loss_utils.py:18-19), psnr (utils/image_utils.py:17-19), ssim (utils/loss_utils.py:34-64) on the GPU and
// torchmetrics' MultiScaleStructuralSimilarityIndexMeasure(data_range=1.0) (utils/loss_utils.py:66-71) on a host copy.
//   ms_scale_kernel     one CTA per 32x32 tile x (view, channel) of one pyramid level: stages the tile + 5-pixel halo
//                       once, runs the separable 11-tap Gaussian over x, y, x^2, y^2, xy in float64 and writes the
//                       tile's partial sums, plus the 2x2 average-pooled tile of x and y (float64) for the next level.
//                       Level 1 (FIRST) also sums |x - y|, (x - y)^2 and the SSIM map over every pixel (zero padding,
//                       ssim_common.cuh's expression, the one loss.cu evaluates in fp32).  Every level sums sim and cs
//                       over the pixels whose window lies inside the level: torchmetrics reflect-pads by 5 and crops 5
//                       again, a valid convolution, where the zero-padded moments are the valid ones.
//                       The moments are float64 and so is the window (WinD): with fp32 moments (loss.cu's arithmetic)
//                       the SSIM of near-identical 176x176 renders was 2.2x further from float64 than torch's fp32
//                       convolutions, and with the window rounded to fp32 MS-SSIM of uncorrelated images moved by
//                       ~4e-5 relative, about 2x torch's own distance.
//   ms_finalize_kernel  one CTA per view: reduces the partials in a fixed order and forms the four numbers in float64.
//   ms_accumulate_kernel  adds them to a test-set accumulator in view order.
// No floating-point atomics: results are bit-identical run to run, and a batch gives what single-view calls give.
#include "fdgs_internal.h"
#include "ssim_common.cuh"

namespace fdgs {
namespace {

constexpr int MT = 32;               // tile edge (pixels)
constexpr int MR = SSIM_R;           // filter radius
constexpr int MW = MT + 2 * MR;      // staged edge
constexpr int MTHREADS = 256;
constexpr int NQ = 5;                // partials per tile: sum |d|, sum d^2, sum S, sum sim, sum cs
constexpr int SCALES = 5;
__constant__ double BETAS[SCALES] = {0.0448, 0.2856, 0.3001, 0.2363, 0.1333};   // torchmetrics' defaults

// the window of ssim_common.cuh's make_window (11 taps, sigma 1.5), evaluated and normalised in float64
struct WinD {
    double g[2 * MR + 1];
};

WinD make_window_f64() {
    WinD w;
    double s = 0.0;
    for (int i = 0; i <= 2 * MR; ++i) s += (w.g[i] = exp(-(double)((i - MR) * (i - MR)) / (2.0 * 1.5 * 1.5)));
    for (int i = 0; i <= 2 * MR; ++i) w.g[i] /= s;
    return w;
}

struct MetricsSmem {
    double sx[MW][MW + 1], sy[MW][MW + 1];
    double hz[5][MW][MT + 1];                    // horizontal pass of x, y, xx, yy, xy
    double red[NQ][MTHREADS / 32];
};

struct Level {
    int H, W, tiles_x, tiles;
    size_t part_off;                             // doubles from the start of the partials
};
struct MetricsPlan {
    int B, C;
    Level lv[SCALES];
};

__device__ __forceinline__ float clamp01(float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); }   // NaN stays NaN

// x, y: one level [B*C, H, W] (fp32 input at level 1, float64 pyramid after); px, py: the next level [B*C, H/2, W/2]
// (NULL at the last level); part: [B*C][tiles][NQ]
template <bool FIRST, typename T>
__global__ void __launch_bounds__(MTHREADS) ms_scale_kernel(const T* __restrict__ x, const T* __restrict__ y, int H, int W,
                                                            int clamp, const WinD wd,
                                                            double* __restrict__ px,
                                                            double* __restrict__ py, double* __restrict__ part) {
    extern __shared__ __align__(16) unsigned char ms_smem_raw[];
    MetricsSmem& sm = *reinterpret_cast<MetricsSmem*>(ms_smem_raw);
    const int plane = blockIdx.z;
    const int x0 = blockIdx.x * MT, y0 = blockIdx.y * MT;
    const size_t HW = (size_t)H * W;
    const T* ix = x + plane * HW;
    const T* iy = y + plane * HW;
    for (int i = threadIdx.x; i < MW * MW; i += MTHREADS) {
        const int r = i / MW, c = i - r * MW;
        const int gy = y0 + r - MR, gx = x0 + c - MR;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;   // zero padding (the SSIM of loss.cu)
        double u = 0.0, v = 0.0;
        if (in) {
            const size_t o = (size_t)gy * W + gx;
            if (FIRST) {
                const float a = (float)ix[o];
                u = clamp ? clamp01(a) : a;
            } else {
                u = ix[o];
            }
            v = iy[o];
        }
        sm.sx[r][c] = u;
        sm.sy[r][c] = v;
    }
    __syncthreads();
    // float64 moments over the staged tile (zero padding), one pass for every number of the level
    for (int i = threadIdx.x; i < MW * MT; i += MTHREADS) {
        const int r = i / MT, c = i - r * MT;
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0, a4 = 0.0;
#pragma unroll
        for (int k = 0; k <= 2 * MR; ++k) {
            const double u = sm.sx[r][c + k], v = sm.sy[r][c + k], w = wd.g[k];
            a0 = fma(w, u, a0);
            a1 = fma(w, v, a1);
            a2 = fma(w, u * u, a2);
            a3 = fma(w, v * v, a3);
            a4 = fma(w, u * v, a4);
        }
        sm.hz[0][r][c] = a0; sm.hz[1][r][c] = a1; sm.hz[2][r][c] = a2; sm.hz[3][r][c] = a3; sm.hz[4][r][c] = a4;
    }
    __syncthreads();
    double q[NQ] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < MT * MT; i += MTHREADS) {
        const int r = i / MT, c = i - r * MT;
        const int gy = y0 + r, gx = x0 + c;
        const bool interior = gy >= MR && gy < H - MR && gx >= MR && gx < W - MR;   // the window lies inside the level
        if (gy >= H || gx >= W || (!FIRST && !interior)) continue;
        double m1 = 0.0, m2 = 0.0, e11 = 0.0, e22 = 0.0, e12 = 0.0;
#pragma unroll
        for (int k = 0; k <= 2 * MR; ++k) {
            const double w = wd.g[k];
            m1 = fma(w, sm.hz[0][r + k][c], m1);
            m2 = fma(w, sm.hz[1][r + k][c], m2);
            e11 = fma(w, sm.hz[2][r + k][c], e11);
            e22 = fma(w, sm.hz[3][r + k][c], e22);
            e12 = fma(w, sm.hz[4][r + k][c], e12);
        }
        const SsimTerms<double> t = ssim_terms(m1, m2, e11, e22, e12);
        if (FIRST) {
            const double d = sm.sx[r + MR][c + MR] - sm.sy[r + MR][c + MR];   // exact: two fp32 values
            q[0] += fabs(d);
            q[1] += d * d;
            q[2] += t.S;                               // the SSIM map of utils/loss_utils.py, zero padding
        }
        if (interior) {                                // torchmetrics' sim and cs: A2 / B2 = upper / lower
            q[3] += t.S;
            q[4] += t.A2 / t.B2;
        }
    }
    if (px) {   // avg_pool2d(2x2), floor: the tile origin is even, so every pooled pixel lies in one tile
        const int Hn = H >> 1, Wn = W >> 1;
        const size_t o = (size_t)plane * Hn * Wn;
        for (int i = threadIdx.x; i < (MT / 2) * (MT / 2); i += MTHREADS) {
            const int r = i / (MT / 2), c = i - r * (MT / 2);
            const int gy = (y0 >> 1) + r, gx = (x0 >> 1) + c;
            if (gy >= Hn || gx >= Wn) continue;
            const int sr = 2 * r + MR, sc = 2 * c + MR;
            px[o + (size_t)gy * Wn + gx] = (((sm.sx[sr][sc] + sm.sx[sr][sc + 1]) + sm.sx[sr + 1][sc]) + sm.sx[sr + 1][sc + 1]) * 0.25;
            py[o + (size_t)gy * Wn + gx] = (((sm.sy[sr][sc] + sm.sy[sr][sc + 1]) + sm.sy[sr + 1][sc]) + sm.sy[sr + 1][sc + 1]) * 0.25;
        }
    }
#pragma unroll
    for (int j = 0; j < NQ; ++j)
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) q[j] += __shfl_xor_sync(0xffffffffu, q[j], d);
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int j = 0; j < NQ; ++j) sm.red[j][threadIdx.x >> 5] = q[j];
    __syncthreads();
    if (threadIdx.x < NQ) {
        double t = 0.0;
        for (int w = 0; w < MTHREADS / 32; ++w) t += sm.red[threadIdx.x][w];
        const size_t tile = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
        part[((size_t)plane * gridDim.x * gridDim.y + tile) * NQ + threadIdx.x] = t;
    }
}

// sum of one value per thread over the CTA in a fixed order, returned to every thread
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    __syncthreads();                               // red may still be read by the previous call
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < MTHREADS / 32; ++w) t += red[w];
    return t;
}

// out[b*4 + 0..3] = l1, psnr, ssim, msssim of view b
__global__ void __launch_bounds__(MTHREADS) ms_finalize_kernel(const MetricsPlan p, const double* __restrict__ part,
                                                               double* __restrict__ out) {
    __shared__ double red[MTHREADS / 32];
    const int b = blockIdx.x, C = p.C;
    const Level l0 = p.lv[0];
    double l1 = 0.0, psnr = 0.0, ssim = 0.0;
    for (int c = 0; c < C; ++c) {
        const double* q = part + l0.part_off + (size_t)(b * C + c) * l0.tiles * NQ;
        double a = 0.0, d2 = 0.0, s = 0.0;
        for (int t = threadIdx.x; t < l0.tiles; t += MTHREADS) {
            a += q[(size_t)t * NQ + 0];
            d2 += q[(size_t)t * NQ + 1];
            s += q[(size_t)t * NQ + 2];
        }
        l1 += block_sum(a, red);
        ssim += block_sum(s, red);
        const double mse = block_sum(d2, red) / ((double)l0.H * l0.W);
        psnr += 20.0 * log10(1.0 / sqrt(mse));       // utils/image_utils.py:17-19, one value per channel
    }
    const double n = (double)C * l0.H * l0.W;
    double ms = 1.0;
#pragma unroll
    for (int s = 0; s < SCALES; ++s) {
        const Level l = p.lv[s];
        double sim = 0.0, cs = 0.0;
        for (int c = 0; c < C; ++c) {
            const double* q = part + l.part_off + (size_t)(b * C + c) * l.tiles * NQ;
            for (int t = threadIdx.x; t < l.tiles; t += MTHREADS) {
                sim += q[(size_t)t * NQ + 3];
                cs += q[(size_t)t * NQ + 4];
            }
        }
        const double kept = (double)C * (l.H - 2 * MR) * (l.W - 2 * MR);
        const double v = block_sum(s == SCALES - 1 ? sim : cs, red) / kept;
        const double r = fmax(v, 0.0);                 // normalize="relu"
        ms *= r > 0.0 ? exp(BETAS[s] * log(r)) : 0.0;  // r^beta (pow's general path would spill)
    }
    if (threadIdx.x == 0) {
        out[b * 4 + 0] = l1 / n;
        out[b * 4 + 1] = psnr / C;
        out[b * 4 + 2] = ssim / n;
        out[b * 4 + 3] = ms;
    }
}

// accum[0..3] += the four numbers of every view, in view order; accum[4] += 1 per view
__global__ void ms_accumulate_kernel(int B, const double* __restrict__ out, double* __restrict__ accum) {
    for (int b = 0; b < B; ++b) {
        for (int k = 0; k < 4; ++k) accum[k] += out[b * 4 + k];
        accum[4] += 1.0;
    }
}

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// level sizes, partial offsets and the scratch layout: [pyramid levels 2..5 of x and y (double)] [partials]
MetricsPlan plan_of(int B, int C, int H, int W, size_t* pyramid_bytes, size_t* total_bytes) {
    MetricsPlan p;
    p.B = B;
    p.C = C;
    const size_t planes = (size_t)B * C;
    size_t pyr = 0, part = 0;
    int h = H, w = W;
    for (int s = 0; s < SCALES; ++s) {
        Level& l = p.lv[s];
        l.H = h; l.W = w;
        l.tiles_x = (w + MT - 1) / MT;
        l.tiles = l.tiles_x * ((h + MT - 1) / MT);
        l.part_off = part;
        part += planes * l.tiles * NQ;
        if (s > 0) pyr += 2 * align256(planes * (size_t)h * w * sizeof(double));
        h >>= 1;
        w >>= 1;
    }
    *pyramid_bytes = pyr;
    *total_bytes = 256 + pyr + align256(part * sizeof(double));
    return p;
}

}  // namespace

size_t metrics_scratch_bytes(int B, int C, int H, int W) {
    size_t pyr, total;
    plan_of(B, C, H, W, &pyr, &total);
    return total;
}

cudaError_t launch_image_metrics(const fdgs_metrics_args& a, char* scratch, cudaStream_t stream) {
    static PerDeviceOnce once_first, once_next;
    const int smem = (int)sizeof(MetricsSmem);
    cudaError_t e = ensure_dynamic_smem(ms_scale_kernel<true, float>, smem, once_first);
    if (e == cudaSuccess) e = ensure_dynamic_smem(ms_scale_kernel<false, double>, smem, once_next);
    if (e != cudaSuccess) return e;
    size_t pyr, total;
    const MetricsPlan p = plan_of(a.B, a.C, a.H, a.W, &pyr, &total);
    char* base = reinterpret_cast<char*>(align256(reinterpret_cast<size_t>(scratch)));
    double* part = reinterpret_cast<double*>(base + pyr);
    double* lx[SCALES] = {nullptr};
    double* ly[SCALES] = {nullptr};
    const size_t planes = (size_t)a.B * a.C;
    char* cur = base;
    for (int s = 1; s < SCALES; ++s) {
        const size_t bytes = align256(planes * (size_t)p.lv[s].H * p.lv[s].W * sizeof(double));
        lx[s] = reinterpret_cast<double*>(cur);
        ly[s] = reinterpret_cast<double*>(cur + bytes);
        cur += 2 * bytes;
    }
    const WinD wd = make_window_f64();
    for (int s = 0; s < SCALES; ++s) {
        const Level& l = p.lv[s];
        const dim3 grid(l.tiles_x, l.tiles / l.tiles_x, (unsigned)planes);
        double* nx = s + 1 < SCALES ? lx[s + 1] : nullptr;
        double* ny = s + 1 < SCALES ? ly[s + 1] : nullptr;
        if (s == 0)
            ms_scale_kernel<true, float><<<grid, MTHREADS, smem, stream>>>(a.x, a.y, l.H, l.W, a.clamp, wd, nx, ny,
                                                                          part + l.part_off);
        else
            ms_scale_kernel<false, double><<<grid, MTHREADS, smem, stream>>>(lx[s], ly[s], l.H, l.W, 0, wd, nx, ny,
                                                                            part + l.part_off);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    ms_finalize_kernel<<<a.B, MTHREADS, 0, stream>>>(p, part, a.out);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if (a.accum) {
        ms_accumulate_kernel<<<1, 1, 0, stream>>>(a.B, a.out, a.accum);
        e = cudaGetLastError();
    }
    return e;
}

}  // namespace fdgs
