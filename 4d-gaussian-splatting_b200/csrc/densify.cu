// densify.cu -- densify and prune as one compaction pass, reset opacity, densification statistics.
//
// Replaces, in the reference, GaussianModel.densify_and_prune (scene/gaussian_model.py:557-577: densify_and_clone,
// densify_and_split, two prune_points), reset_opacity (:371-374) and add_densification_stats(_grad) (:579-589) with
// the batch rescale and max-radius update of train.py:168-183, 233-237.  The reference's surgery concatenates every
// parameter and moment tensor twice and gathers it twice (four full passes over 161 floats x 3 per Gaussian, ~80 host
// synchronisations on boolean-mask indexing).  Here:
//   plan : classify_kernel decides every original row's fate and writes a packed count vector
//          (original kept, clone kept, split selected, children kept); one inclusive scan over it; map_kernel turns
//          counts and scan into each row's destination rows and sample row, and the four totals;
//   apply: ONE multi-tensor launch (blockIdx.y = tensor) reads every source row once and writes it to all its
//          destinations (zeros for the new rows' moments, the split children's log-scales computed on the way); one
//          thread-per-row launch writes the split children's positions and times.
// The only host synchronisation is the caller's read of the four totals between the two.
//
// Decisions are bit-identical to the reference's fp32 PyTorch ops: exp / sigmoid as the raw-parameter entry spells
// them (fdgs_common.cuh), thresholds compared in fp32 (ATen rounds a Python scalar to the tensor's dtype before a
// comparison), tensor / Python-scalar as a multiply by the fp32 reciprocal of the fp32 scalar (ATen's div_true with a
// CPU scalar), torch.norm of one element as sqrt(g * g), torch.max over a row propagating NaN.
#include <cub/cub.cuh>
#include "../../include/fdgs.h"
#include "fdgs_internal.h"

namespace fdgs {
namespace {

constexpr int THREADS = 256;

__device__ __forceinline__ float nan_max(float a, float b) { return (a > b || a != a) ? a : b; }   // torch.max: NaN wins

// max(exp(log_s)) over the three spatial log-scales (torch.max(get_scaling, dim=1).values)
__device__ __forceinline__ float scale_max(const float* s) {
    return nan_max(nan_max(act_exp(s[0]), act_exp(s[1])), act_exp(s[2]));
}

// log(exp(log_s) * mul): a split child's log-scale (scaling_inverse_activation(get_scaling / (0.8 N)))
__device__ __forceinline__ float child_log_scale(float log_s, float mul) { return logf(fmul(act_exp(log_s), mul)); }

struct PlanArgs {
    long long P;
    int densify, use_screen;
    float max_grad, min_opacity, dense_extent, big_extent, max_screen_size, split_mul;
    const float *accum, *denom, *radii, *scaling, *opacity;
};

__device__ __forceinline__ bool pruned(const PlanArgs& a, float opacity, float smax, float radius) {
    return act_sigmoid(opacity) < a.min_opacity ||
           (a.use_screen && (radius > a.max_screen_size || smax > a.big_extent));
}

__global__ void __launch_bounds__(THREADS) densify_classify_kernel(const PlanArgs a, int4* __restrict__ counts) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    const float* s = a.scaling + 3 * i;
    const float smax = scale_max(s);
    const float op = a.opacity[i];
    bool clone = false, split = false;
    float radius = 0.f;                       // a densifying call has zeroed max_radii2D before its prune
    if (a.densify) {
        float g = fdiv(a.accum[i], a.denom[i]);
        if (g != g) g = 0.f;
        clone = fsqrt(fmul(g, g)) >= a.max_grad && smax <= a.dense_extent;
        split = g >= a.max_grad && smax > a.dense_extent;
    } else if (a.use_screen) {
        radius = a.radii[i];
    }
    int4 c;
    c.x = !split && !pruned(a, op, smax, radius);
    c.y = clone && !pruned(a, op, smax, 0.f);
    c.z = split;
    c.w = 0;
    if (split) {
        const float cmax = nan_max(nan_max(act_exp(child_log_scale(s[0], a.split_mul)), act_exp(child_log_scale(s[1], a.split_mul))),
                                   act_exp(child_log_scale(s[2], a.split_mul)));
        c.w = !pruned(a, op, cmax, 0.f);
    }
    counts[i] = c;
}

struct Int4Sum {
    __device__ __forceinline__ int4 operator()(const int4& a, const int4& b) const {
        return make_int4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
};

// map[i] = (destination of the original row, of its clone, of its copy-1 child; its sample row) or -1 each;
// copy k of the child lives at map.z + k * totals[3].
__global__ void __launch_bounds__(THREADS) densify_map_kernel(long long P, const int4* __restrict__ counts,
                                                             const int4* __restrict__ incl, int4* __restrict__ map,
                                                             int* __restrict__ totals) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int4 T = incl[P - 1];
    const int4 c = counts[i], s = incl[i];
    int4 m;
    m.x = c.x ? s.x - 1 : -1;
    m.y = c.y ? T.x + s.y - 1 : -1;
    m.z = c.w ? T.x + T.y + s.w - 1 : -1;
    m.w = c.z ? s.z - 1 : -1;
    map[i] = m;
    if (i == P - 1) { totals[0] = T.x; totals[1] = T.y; totals[2] = T.z; totals[3] = T.w; }
}

struct ApplyTable {
    const float* src[FDGS_DENSIFY_MAX_TENSORS];
    float* dst[FDGS_DENSIFY_MAX_TENSORS];
    int width[FDGS_DENSIFY_MAX_TENSORS];
    int kind[FDGS_DENSIFY_MAX_TENSORS];
};

struct SplitGeo {
    const float *xyz, *t, *scaling, *scaling_t, *rotation, *rotation_r, *samples, *samples_t;
    int rot_4d;
};

// The split children's positions and times, one thread per source row, in double and rounded once:
//   rot_4d : [xyz, t] + build_rotation_4d(rotation, rotation_r) @ (sample4 * exp([scaling, scaling_t]))
//   3D rot : xyz + build_rotation(rotation) @ (sample3 * exp(scaling));  t + sample_t * exp(scaling_t)
// Kept out of densify_apply_kernel so that the copy loop keeps its low register count.
__global__ void __launch_bounds__(THREADS) densify_positions_kernel(const SplitGeo g, long long P, const int4* __restrict__ map,
                                                                   int N, long long S, long long child_kept,
                                                                   float* __restrict__ dst_xyz, float* __restrict__ dst_t) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= P) return;
    const int4 m = map[r];
    if (m.z < 0) return;
    double A[4][4];                       // rotation: rows 0..2 -> xyz, row 3 -> t (rot_4d)
    double sc[4];
    for (int j = 0; j < 3; ++j) sc[j] = act_exp(g.scaling[3 * r + j]);
    sc[3] = g.scaling_t ? (double)act_exp(g.scaling_t[r]) : 0.0;
    const float* l = g.rotation + 4 * r;
    const double nl = sqrt((double)l[0] * l[0] + (double)l[1] * l[1] + (double)l[2] * l[2] + (double)l[3] * l[3]);
    const double a = l[0] / nl, b = l[1] / nl, c = l[2] / nl, d = l[3] / nl;
    if (g.rot_4d) {
        const float* rr = g.rotation_r + 4 * r;
        const double nr = sqrt((double)rr[0] * rr[0] + (double)rr[1] * rr[1] + (double)rr[2] * rr[2] + (double)rr[3] * rr[3]);
        const double p = rr[0] / nr, q = rr[1] / nr, u = rr[2] / nr, s = rr[3] / nr;
        const double Ml[4][4] = {{a, -b, -c, -d}, {b, a, -d, c}, {c, d, a, -b}, {d, -c, b, a}};
        const double Mr[4][4] = {{p, q, u, s}, {-q, p, -s, u}, {-u, s, p, -q}, {-s, -u, q, p}};
        for (int i = 0; i < 4; ++i)          // (Ml @ Mr).flip(1, 2)[i][j] = (Ml @ Mr)[3 - i][3 - j]
            for (int j = 0; j < 4; ++j) {
                double v = 0.0;
                for (int k = 0; k < 4; ++k) v += Ml[3 - i][k] * Mr[k][3 - j];
                A[i][j] = v;
            }
    } else {                              // build_rotation with (r, x, y, z) = (a, b, c, d)
        A[0][0] = 1 - 2 * (c * c + d * d); A[0][1] = 2 * (b * c - a * d); A[0][2] = 2 * (b * d + a * c);
        A[1][0] = 2 * (b * c + a * d); A[1][1] = 1 - 2 * (b * b + d * d); A[1][2] = 2 * (c * d - a * b);
        A[2][0] = 2 * (b * d - a * c); A[2][1] = 2 * (c * d + a * b); A[2][2] = 1 - 2 * (b * b + c * c);
    }
    const int ns = g.rot_4d ? 4 : 3;
    for (int k = 0; k < N; ++k) {
        const long long q = k * S + m.w;
        const long long o = m.z + k * child_kept;
        double smp[4];
        for (int j = 0; j < ns; ++j) smp[j] = (double)g.samples[ns * q + j] * sc[j];
        for (int i = 0; i < 3; ++i) {
            double v = g.xyz[3 * r + i];
            for (int j = 0; j < ns; ++j) v += A[i][j] * smp[j];
            if (dst_xyz) dst_xyz[3 * o + i] = (float)v;
        }
        if (dst_t) {
            double v = g.t[r];
            if (g.rot_4d) for (int j = 0; j < 4; ++j) v += A[3][j] * smp[j];
            else v += (double)g.samples_t[q] * sc[3];
            dst_t[o] = (float)v;
        }
    }
}

// Thread per element of the flattened [P, width] source: a row's elements are contiguous in the source and in every
// destination, and kept rows are packed, so both the reads and the writes of a warp are coalesced for any width.
// The children's xyz / t are left to densify_positions_kernel.
__global__ void __launch_bounds__(THREADS) densify_apply_kernel(const ApplyTable tb, long long P, const int4* __restrict__ map,
                                                               int N, long long child_kept, float split_mul) {
    const int t = blockIdx.y;
    const int w = tb.width[t], kind = tb.kind[t];
    const float* __restrict__ src = tb.src[t];
    float* __restrict__ dst = tb.dst[t];
    const long long total = P * w;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long r = e / w;
        const int c = (int)(e - r * w);
        const int4 m = map[r];
        if ((m.x & m.y & m.z) < 0) continue;          // pruned everywhere
        const float v = src[e];
        if (m.x >= 0) dst[(long long)m.x * w + c] = v;
        if (m.y >= 0) dst[(long long)m.y * w + c] = kind == FDGS_DENSIFY_MOMENT ? 0.f : v;
        if (m.z < 0 || kind == FDGS_DENSIFY_XYZ || kind == FDGS_DENSIFY_T) continue;
        const float o = kind == FDGS_DENSIFY_MOMENT ? 0.f
                      : (kind == FDGS_DENSIFY_SCALING || kind == FDGS_DENSIFY_SCALING_T) ? child_log_scale(v, split_mul) : v;
        for (int k = 0; k < N; ++k) dst[(m.z + k * child_kept) * w + c] = o;
    }
}

__global__ void __launch_bounds__(THREADS) reset_opacity_kernel(long long P, float* __restrict__ opacity,
                                                               float* __restrict__ m, float* __restrict__ v) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float o = act_sigmoid(opacity[i]);
    const float x = (o < 0.01f || o != o) ? o : 0.01f;       // torch.min(get_opacity, 0.01): NaN wins
    opacity[i] = logf(fdiv(x, fsub(1.0f, x)));               // inverse_sigmoid: log(x / (1 - x))
    if (m) m[i] = 0.f;
    if (v) v[i] = 0.f;
}

// One thread per Gaussian.  With a status {R, largest tile, overflow, wrap} from the rasterizer, nothing is accumulated
// when it reports an overflow or a wrap: a captured step whose forward overflowed is replayed after a re-capture
__global__ void __launch_bounds__(THREADS) densify_stats_kernel(long long P, int B, const float* __restrict__ pgrad, int stride,
                                                               const float* __restrict__ vis, const int* __restrict__ radii,
                                                               const float* __restrict__ tgrad, float* __restrict__ accum,
                                                               float* __restrict__ denom, float* __restrict__ taccum,
                                                               float* __restrict__ max_radii2D,
                                                               const int* __restrict__ status) {
    if (status && (status[2] | status[3])) return;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int r = radii[i];
    float g, tg = 0.f;
    if (B == 1) {
        if (r <= 0) return;
        const float gx = pgrad[i * stride], gy = pgrad[i * stride + 1];
        g = fsqrt(fadd(fmul(gx, gx), fmul(gy, gy)));           // torch.norm of two elements: x^2 + y^2 rounded apart
        if (tgrad) tg = tgrad[i];
    } else {
        const float cnt = vis[i];
        if (!(cnt > 0.f)) return;
        g = fdiv(fmul(pgrad[i], (float)B), cnt);                // grad * batch_size / visibility_count
        if (tgrad) tg = fdiv(fmul(tgrad[i], (float)B), cnt);
    }
    const float rf = (float)r, mr = max_radii2D[i];
    max_radii2D[i] = (rf > mr || rf != rf) ? rf : mr;
    accum[i] = fadd(accum[i], g);
    denom[i] = fadd(denom[i], 1.0f);
    if (taccum) taccum[i] = fadd(taccum[i], tg);
}

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

size_t cub_scan_bytes(long long P) {
    size_t bytes = 0;
    cub::DeviceScan::InclusiveScan(nullptr, bytes, (const int4*)nullptr, (int4*)nullptr, Int4Sum(), (int)P);
    return bytes;
}

unsigned grid_for(long long n) { return (unsigned)((n + THREADS - 1) / THREADS); }

}  // namespace

// scratch layout: counts int4[P] | inclusive scan int4[P] | map int4[P] | cub temporary storage
size_t densify_scratch_bytes(long long P) { return 3 * align256(16 * (size_t)P) + align256(cub_scan_bytes(P)); }

float densify_split_mul(int N) { return 1.0f / (float)(0.8 * N); }

cudaError_t launch_densify_plan(const fdgs_densify_args& a, char* scratch, int* totals, cudaStream_t stream) {
    const long long P = a.P;
    if (P == 0) return cudaMemsetAsync(totals, 0, 4 * sizeof(int), stream);
    const size_t row = align256(16 * (size_t)P);
    int4* counts = reinterpret_cast<int4*>(scratch);
    int4* incl = reinterpret_cast<int4*>(scratch + row);
    int4* map = reinterpret_cast<int4*>(scratch + 2 * row);
    void* temp = scratch + 3 * row;
    PlanArgs pa;
    pa.P = P;
    pa.densify = !a.prune_only;
    pa.use_screen = a.use_max_screen_size;
    pa.max_grad = a.max_grad; pa.min_opacity = a.min_opacity; pa.dense_extent = a.dense_extent;
    pa.big_extent = a.big_extent; pa.max_screen_size = a.max_screen_size; pa.split_mul = densify_split_mul(a.N);
    pa.accum = a.xyz_gradient_accum; pa.denom = a.denom; pa.radii = a.max_radii2D;
    pa.scaling = a.scaling; pa.opacity = a.opacity;
    densify_classify_kernel<<<grid_for(P), THREADS, 0, stream>>>(pa, counts);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    size_t bytes = cub_scan_bytes(P);
    e = cub::DeviceScan::InclusiveScan(temp, bytes, counts, incl, Int4Sum(), (int)P, stream);
    if (e != cudaSuccess) return e;
    densify_map_kernel<<<grid_for(P), THREADS, 0, stream>>>(P, counts, incl, map, totals);
    return cudaGetLastError();
}

cudaError_t launch_densify_apply(const fdgs_densify_args& a, const char* scratch, long long S, long long child_kept,
                                 cudaStream_t stream) {
    const long long P = a.P;
    if (P == 0 || a.num_tensors == 0) return cudaSuccess;
    const int4* map = reinterpret_cast<const int4*>(scratch + 2 * align256(16 * (size_t)P));
    ApplyTable tb;
    int widest = 1;
    float *dst_xyz = nullptr, *dst_t = nullptr;
    for (int i = 0; i < a.num_tensors; ++i) {
        tb.src[i] = a.src[i]; tb.dst[i] = a.dst[i]; tb.width[i] = a.width[i]; tb.kind[i] = a.kind[i];
        if (a.width[i] > widest) widest = a.width[i];
        if (a.kind[i] == FDGS_DENSIFY_XYZ) dst_xyz = a.dst[i];
        if (a.kind[i] == FDGS_DENSIFY_T) dst_t = a.dst[i];
    }
    const float split_mul = densify_split_mul(a.N);
    long long blocks = (P * widest + THREADS - 1) / THREADS;
    if (blocks > device_sm_count() * 16) blocks = device_sm_count() * 16;
    dim3 grid((unsigned)blocks, (unsigned)a.num_tensors, 1);
    densify_apply_kernel<<<grid, THREADS, 0, stream>>>(tb, P, map, a.N, child_kept, split_mul);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess || child_kept == 0 || (!dst_xyz && !dst_t)) return e;
    SplitGeo g;
    g.xyz = a.xyz; g.t = a.t; g.scaling = a.scaling; g.scaling_t = a.gaussian_dim == 4 ? a.scaling_t : nullptr;
    g.rotation = a.rotation; g.rotation_r = a.rotation_r; g.samples = a.samples; g.samples_t = a.samples_t;
    g.rot_4d = a.rot_4d;
    densify_positions_kernel<<<grid_for(P), THREADS, 0, stream>>>(g, P, map, a.N, S, child_kept, dst_xyz, dst_t);
    return cudaGetLastError();
}

cudaError_t launch_reset_opacity(long long P, float* opacity, float* m, float* v, cudaStream_t stream) {
    if (P == 0) return cudaSuccess;
    reset_opacity_kernel<<<grid_for(P), THREADS, 0, stream>>>(P, opacity, m, v);
    return cudaGetLastError();
}

cudaError_t launch_densify_stats(long long P, int B, const float* pgrad, int stride, const float* vis, const int* radii,
                                 const float* tgrad, float* accum, float* denom, float* taccum, float* max_radii2D,
                                 const int* status, cudaStream_t stream) {
    if (P == 0) return cudaSuccess;
    densify_stats_kernel<<<grid_for(P), THREADS, 0, stream>>>(P, B, pgrad, stride, vis, radii, tgrad, accum, denom, taccum,
                                                             max_radii2D, status);
    return cudaGetLastError();
}

}  // namespace fdgs
