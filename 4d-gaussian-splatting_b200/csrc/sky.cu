// sky.cu -- environment-map sky sphere behind the Gaussians (forward and backward).
//
// Restates the PyTorch sky of the reference's render() for scenes with an environment map: every pixel's ray (the
// camera's get_rays: pixel centre through the pinhole, camera-to-world, normalised) is intersected with a sphere of
// radius R about the origin, the hit point is mapped to longitude / colatitude texture coordinates and the map is
// sampled bilinearly with F.grid_sample's defaults (align_corners = False, zero padding, x along the width).  One
// thread per pixel, IEEE division and square root and libdevice atan2f: no fast-math intrinsics.
//
// The backward scatters dL/dsky to the four texels of every pixel.  Neighbouring pixels share texels (at 1352x1014
// against a 500x500 map about a hundred pixels land on each), so the lanes of a warp that read the same 2x2 texel
// block add their contributions first (__match_any_sync) and one lane issues the RED per texel and channel.
#include "fdgs_internal.h"

namespace fdgs {
namespace {

constexpr int SKY_THREADS = 256;
constexpr float kPi = 3.14159265358979323846f;

struct SkyTap {
    int x0, y0;     // top-left texel of the 2x2 block (may lie outside the map: zero padding)
    float w[4];     // nw, ne, sw, se bilinear weights (F.grid_sample order)
    bool miss;      // the ray does not cross the sphere (the reference asserts on this)
};

__device__ __forceinline__ SkyTap sky_tap(const SkyParams& p, int x, int y) {
    const float* M = p.c2w;
    // view-space point of the pixel centre at depth 1 (homogeneous w = 1), then camera-to-world: pts_view @ c2w.T
    const float vx = __fdiv_rn(__fsub_rn((float)x + 0.5f, p.cx), p.fl_x);
    const float vy = __fdiv_rn(__fsub_rn((float)y + 0.5f, p.cy), p.fl_y);
    const float ox = p.campos[0], oy = p.campos[1], oz = p.campos[2];
    float dx = M[0] * vx + M[1] * vy + M[2] + M[3] - ox;
    float dy = M[4] * vx + M[5] * vy + M[6] + M[7] - oy;
    float dz = M[8] * vx + M[9] * vy + M[10] + M[11] - oz;
    const float n = __fsqrt_rn(dx * dx + dy * dy + dz * dz);
    dx = __fdiv_rn(dx, n);
    dy = __fdiv_rn(dy, n);
    dz = __fdiv_rn(dz, n);
    // ray o + t d against |X| = R; the reference's precedence: t = -(o.d) + sqrt(delta) / (d.d)
    const float od = ox * dx + oy * dy + oz * dz;
    const float dd = dx * dx + dy * dy + dz * dz;
    const float delta = od * od - dd * (ox * ox + oy * oy + oz * oz - p.radius * p.radius);
    SkyTap t;
    t.miss = !(delta > 0.0f);
    const float th = -od + __fdiv_rn(__fsqrt_rn(delta), dd);
    const float hx = ox + dx * th, hy = oy + dy * th, hz = oz + dz * th;
    // longitude / colatitude.  On the sphere acos(hz / R) = atan2(sqrt(hx^2 + hy^2), hz); the atan2 form stays
    // well-conditioned at the poles, where acos of the rounded hz / R loses half its digits (or is NaN an ulp past 1)
    const float tu = __fdiv_rn(atan2f(hy, hx), 2.0f * kPi) + 0.5f;
    const float tv = __fdiv_rn(atan2f(__fsqrt_rn(hx * hx + hy * hy), hz), kPi);
    // grid_sample: grid = 2 tc - 1, unnormalised with align_corners = False: ((g + 1) size - 1) / 2
    const float gx = tu * 2.0f - 1.0f, gy = tv * 2.0f - 1.0f;
    const float ix = __fdiv_rn((gx + 1.0f) * (float)p.env_width - 1.0f, 2.0f);
    const float iy = __fdiv_rn((gy + 1.0f) * (float)p.env_height - 1.0f, 2.0f);
    const float fx = floorf(ix), fy = floorf(iy);
    // NaN coordinates (a missed ray) sample nothing
    const bool ok = fx == fx && fy == fy && fabsf(fx) < 1.0e8f && fabsf(fy) < 1.0e8f;
    t.x0 = ok ? (int)fx : -2;
    t.y0 = ok ? (int)fy : -2;
    const float ex = ix - fx, ey = iy - fy, wx = (fx + 1.0f) - ix, wy = (fy + 1.0f) - iy;
    t.w[0] = wx * wy;
    t.w[1] = ex * wy;
    t.w[2] = wx * ey;
    t.w[3] = ex * ey;
    return t;
}

__device__ __forceinline__ bool texel_in(const SkyParams& p, int x, int y) {
    return x >= 0 && x < p.env_width && y >= 0 && y < p.env_height;
}

// one pixel of the forward: the sky colour of pixel `pix` of the camera in p into out [3,H,W]
__device__ __forceinline__ void sky_fwd_pixel(const SkyParams& p, int pix, float* __restrict__ out, int* miss_flag) {
    const int HW = p.W * p.H;
    const SkyTap t = sky_tap(p, pix % p.W, pix / p.W);
    if (t.miss && miss_flag) atomicOr(miss_flag, 1);
    const int HWm = p.env_width * p.env_height;
    float c0 = 0.f, c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int x = t.x0 + (k & 1), y = t.y0 + (k >> 1);
        if (!texel_in(p, x, y)) continue;
        const float* e = p.env_map + (size_t)y * p.env_width + x;
        c0 += __ldg(e) * t.w[k];
        c1 += __ldg(e + HWm) * t.w[k];
        c2 += __ldg(e + 2 * (size_t)HWm) * t.w[k];
    }
    out[pix] = c0;
    out[HW + pix] = c1;
    out[2 * (size_t)HW + pix] = c2;
}

// the backward of the block's pixels (blockIdx.x) of the camera in p, called by every thread of the block; the lanes
// sharing a 2x2 texel block sum their contributions before the RED (see the file comment)
__device__ __forceinline__ void sky_bwd_pixels(const SkyParams& p, const float* __restrict__ g, float* __restrict__ denv) {
    const int pix = blockIdx.x * SKY_THREADS + threadIdx.x;
    const int HW = p.W * p.H;
    const bool live = pix < HW;
    SkyTap t;
    float g0 = 0.f, g1 = 0.f, g2 = 0.f;
    if (live) {
        t = sky_tap(p, pix % p.W, pix / p.W);
        g0 = g[pix];
        g1 = g[HW + pix];
        g2 = g[2 * (size_t)HW + pix];
    } else {
        t.x0 = t.y0 = -2;
        t.w[0] = t.w[1] = t.w[2] = t.w[3] = 0.f;
    }
    const int HWm = p.env_width * p.env_height;
    // every lane of the warp takes part (dead lanes carry zero weights on a block no live lane can have)
    __shared__ float part[SKY_THREADS / 32][12][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned int key = ((unsigned)(t.y0 + 2) << 16) ^ (unsigned)(t.x0 + 2);
    const unsigned int peers = __match_any_sync(0xffffffffu, key);
    const int leader = __ffs(peers) - 1;
    float v[12];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        v[3 * k + 0] = t.w[k] * g0;
        v[3 * k + 1] = t.w[k] * g1;
        v[3 * k + 2] = t.w[k] * g2;
    }
#pragma unroll
    for (int i = 0; i < 12; ++i) part[warp][i][lane] = v[i];
    __syncwarp();
    if (lane != leader || !live) return;
    // the leader adds its peers' contributions in lane order
    for (unsigned int rest = peers & (peers - 1u); rest; rest &= rest - 1u) {
        const int src = __ffs(rest) - 1;
#pragma unroll
        for (int i = 0; i < 12; ++i) v[i] += part[warp][i][src];
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int x = t.x0 + (k & 1), y = t.y0 + (k >> 1);
        if (!texel_in(p, x, y)) continue;
        float* e = denv + (size_t)y * p.env_width + x;
        atomicAdd(e, v[3 * k + 0]);
        atomicAdd(e + HWm, v[3 * k + 1]);
        atomicAdd(e + 2 * (size_t)HWm, v[3 * k + 2]);
    }
}

__global__ void __launch_bounds__(SKY_THREADS) sky_fwd_kernel(const SkyParams p, float* __restrict__ out, int* miss_flag) {
    const int pix = blockIdx.x * SKY_THREADS + threadIdx.x;
    if (pix >= p.W * p.H) return;
    sky_fwd_pixel(p, pix, out, miss_flag);
}

__global__ void __launch_bounds__(SKY_THREADS) sky_bwd_kernel(const SkyParams p, const float* __restrict__ g,
                                                              float* __restrict__ denv) {
    sky_bwd_pixels(p, g, denv);
}

// view v's camera from the device tables: the single-view kernels' SkyParams, so the per-pixel arithmetic is theirs
__device__ __forceinline__ SkyParams batch_view(const SkyBatchParams& b, int v) {
    SkyParams p;
    p.env_map = b.env_map; p.env_height = b.env_height; p.env_width = b.env_width;
    p.c2w = b.c2w + 16 * (size_t)v;
    p.campos = b.campos + 3 * (size_t)v;
    const float* k = b.intrinsics + 4 * (size_t)v;
    p.fl_x = k[0]; p.fl_y = k[1]; p.cx = k[2]; p.cy = k[3];
    p.radius = b.radius;
    p.W = b.W; p.H = b.H;
    return p;
}

// blockIdx.y = view: sky [B,3,H,W], every view's misses ORed into one flag
__global__ void __launch_bounds__(SKY_THREADS) sky_fwd_batch_kernel(const SkyBatchParams b, float* __restrict__ out,
                                                                    int* miss_flag) {
    const int pix = blockIdx.x * SKY_THREADS + threadIdx.x;
    if (pix >= b.W * b.H) return;
    const int v = blockIdx.y;
    sky_fwd_pixel(batch_view(b, v), pix, out + (size_t)v * 3 * b.W * b.H, miss_flag);
}

// blockIdx.y = view: every view's dL_dsky [B,3,H,W] accumulated into the one dL_denv [3,Hm,Wm]
__global__ void __launch_bounds__(SKY_THREADS) sky_bwd_batch_kernel(const SkyBatchParams b, const float* __restrict__ g,
                                                                    float* __restrict__ denv) {
    const int v = blockIdx.y;
    sky_bwd_pixels(batch_view(b, v), g + (size_t)v * 3 * b.W * b.H, denv);
}

}  // namespace

cudaError_t launch_sky_fwd(const SkyParams& p, float* out_sky, int* miss_flag, cudaStream_t stream) {
    const long long n = (long long)p.W * p.H;
    const unsigned int blocks = (unsigned int)((n + SKY_THREADS - 1) / SKY_THREADS);
    sky_fwd_kernel<<<blocks, SKY_THREADS, 0, stream>>>(p, out_sky, miss_flag);
    return cudaGetLastError();
}

cudaError_t launch_sky_bwd(const SkyParams& p, const float* dL_dsky, float* dL_denv, cudaStream_t stream) {
    const long long n = (long long)p.W * p.H;
    const unsigned int blocks = (unsigned int)((n + SKY_THREADS - 1) / SKY_THREADS);
    sky_bwd_kernel<<<blocks, SKY_THREADS, 0, stream>>>(p, dL_dsky, dL_denv);
    return cudaGetLastError();
}

cudaError_t launch_sky_fwd_batch(const SkyBatchParams& b, float* out_sky, int* miss_flag, cudaStream_t stream) {
    const long long n = (long long)b.W * b.H;
    const dim3 grid((unsigned int)((n + SKY_THREADS - 1) / SKY_THREADS), (unsigned int)b.B);
    sky_fwd_batch_kernel<<<grid, SKY_THREADS, 0, stream>>>(b, out_sky, miss_flag);
    return cudaGetLastError();
}

cudaError_t launch_sky_bwd_batch(const SkyBatchParams& b, const float* dL_dsky, float* dL_denv, cudaStream_t stream) {
    const long long n = (long long)b.W * b.H;
    const dim3 grid((unsigned int)((n + SKY_THREADS - 1) / SKY_THREADS), (unsigned int)b.B);
    sky_bwd_batch_kernel<<<grid, SKY_THREADS, 0, stream>>>(b, dL_dsky, dL_denv);
    return cudaGetLastError();
}

}  // namespace fdgs
