// regularize.cu -- the rigidity and motion regularisers of the training step: velocity, loss and backward.
//
// Replaces, in the reference, the PyTorch expressions of train.py:132-159 (configs/dnerf/lego.yaml:58 lambda_rigid):
//   dt       = (t + 0.1) - t                                              (fp32, per row)
//   v_i      = Sigma[0:3,3] / Sigma[3,3] * dt                             (scene/gaussian_model.py:34-47, 247-251:
//                                                                          get_current_covariance_and_mean_offset)
//   w_ij     = exp(-100 d2_ij)                                            (d2 = the kNN's squared distances)
//   L_rigid  = (sum_i sum_{j in N(i)} w_ij ||v_j - v_i||) / k / n
//   L_motion = mean_i ||v_i||
// and their autograd.  Gradients go to the raw log-scales and quaternions only: xyz feeds a detached kNN, and the
// reference's t gradient is +g - g = 0 exactly.
//
// Kernels:
//   rigid_weight_kernel   w = expf(-100 * d2) (bit-identical to torch.exp(-100 * dist)) and the edge ids to sort
//   (cub radix sort)      stable sort of the edges by destination row: the incoming edges of every row as a CSR, each
//                         segment in ascending edge id -- deterministic for any in-degree
//   rigid_offsets_kernel  CSR row starts from the sorted destinations (no atomics)
//   rigid_velocity_kernel one thread per Gaussian: v [n,3] (evaluated in double, rounded once), kept for the backward
//   rigid_loss_kernel     one thread per row walks its k outgoing edges; fp64 row sums, per-block fixed-tree partials
//   rigid_total_kernel    one block sums the partials in a fixed order and rounds once; the losses stay on the device
//   rigid_bwd_kernel      one thread per row: outgoing edges in slot order, then incoming edges in CSR order (edge terms
//                         recomputed from v and w), the motion term, then the chain to the raw parameters
//                         (in double)
// Every sum has a fixed order, so forward and backward are bit-identical run to run.  No host synchronisation.
#include <cub/cub.cuh>
#include "../../include/fdgs.h"
#include "fdgs_internal.h"

namespace fdgs {
namespace {

constexpr int RG_THREADS = 256;
constexpr int RG_BWD_THREADS = 128;
constexpr int RG_TOTAL_THREADS = 1024;

__global__ void __launch_bounds__(RG_THREADS) rigid_weight_kernel(long long nk, const float* __restrict__ d2,
                                                                  float* __restrict__ w, unsigned int* __restrict__ edge) {
    const long long e = (long long)blockIdx.x * RG_THREADS + threadIdx.x;
    if (e >= nk) return;
    w[e] = expf(__fmul_rn(-100.f, d2[e]));     // torch: mul by the fp32 scalar, then ATen's exp (expf)
    edge[e] = (unsigned int)e;
}

// dst = destinations sorted ascending: in_offsets[j] = first position with dst >= j, in_offsets[n] = nk
__global__ void __launch_bounds__(RG_THREADS) rigid_offsets_kernel(int n, long long nk, const unsigned int* __restrict__ dst,
                                                                   int* __restrict__ in_offsets) {
    const long long p = (long long)blockIdx.x * RG_THREADS + threadIdx.x;
    if (p > nk) return;
    const long long prev = p > 0 ? (long long)dst[p - 1] : -1;
    const long long cur = p < nk ? (long long)dst[p] : (long long)n;
    for (long long j = prev + 1; j <= cur; ++j) in_offsets[j] = (int)p;
}

__device__ __forceinline__ float4 load_quat(const float* q, int i) { return reinterpret_cast<const float4*>(q)[i]; }

// The 4D covariance of row i from its raw parameters at scaling modifier 1, in double: sc = exp(log-scales),
// rot / rotr = q / ||q||, R = M_r M_l, M[c][r] = sc[r] R[c][r] (build_M4's matrices, glm convention), and the entries of
// Sigma = M^T M the velocity needs.  Double, not the rasterizer's fp32 rounding pattern: v = Sigma[0:3,3] / Sigma[3,3]
// is a ratio of sums that cancel, and the quaternion gradients difference the velocities of neighbours; evaluated in
// fp32 with build_M4's roundings, their worst rows were measured at 2-5 x torch's own fp32 distance from float64.
struct RigidGeom {
    double sc[4];
    double4 rot, rotr;
    double R[4][4], M[4][4];
    double c12[3], cov_t;
};

__device__ __forceinline__ double4 normalize_f64(const float4 q) {
    const double n = sqrt((double)q.x * q.x + (double)q.y * q.y + (double)q.z * q.z + (double)q.w * q.w);
    return make_double4(q.x / n, q.y / n, q.z / n, q.w / n);
}

__device__ __forceinline__ void rigid_geometry(const RigidParams& p, int i, RigidGeom& G) {
    G.sc[0] = exp((double)p.scaling[3 * i + 0]);
    G.sc[1] = exp((double)p.scaling[3 * i + 1]);
    G.sc[2] = exp((double)p.scaling[3 * i + 2]);
    G.sc[3] = exp((double)p.scaling_t[i]);
    G.rot = normalize_f64(load_quat(p.rotation, i));
    G.rotr = normalize_f64(load_quat(p.rotation_r, i));
    const double a = G.rot.x, b = G.rot.y, c = G.rot.z, d = G.rot.w;
    const double pp = G.rotr.x, q = G.rotr.y, r = G.rotr.z, s = G.rotr.w;
    const double Ml[4][4] = {{a, b, -c, d}, {-b, a, d, c}, {c, -d, a, b}, {-d, -c, -b, a}};
    const double Mr[4][4] = {{pp, q, -r, -s}, {-q, pp, s, -r}, {r, -s, pp, -q}, {s, r, q, pp}};
    mat4_mul(Mr, Ml, G.R);
#pragma unroll
    for (int col = 0; col < 4; ++col)
#pragma unroll
        for (int row = 0; row < 4; ++row) G.M[col][row] = G.sc[row] * G.R[col][row];
    double acc[4] = {0.0, 0.0, 0.0, 0.0};     // Sigma[j][3] = sum_k M[3][k] M[j][k]
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[j] += G.M[3][k] * G.M[j][k];
    G.c12[0] = acc[0]; G.c12[1] = acc[1]; G.c12[2] = acc[2]; G.cov_t = acc[3];
}

// dt = (t + 0.1f) - t: the reference's timestamp t + 0.1 (Python scalar rounded to fp32) minus t
__device__ __forceinline__ float rigid_dt(float t) { return fsub(fadd(t, 0.1f), t); }

__device__ __forceinline__ float norm3(float x, float y, float z) { return fsqrt(fadd(fadd(fmul(x, x), fmul(y, y)), fmul(z, z))); }

__global__ void __launch_bounds__(RG_THREADS) rigid_velocity_kernel(const RigidParams p) {
    const int i = blockIdx.x * RG_THREADS + threadIdx.x;
    if (i >= p.n) return;
    RigidGeom G;
    rigid_geometry(p, i, G);
    const double dt = rigid_dt(p.t[i]);
    p.velocity[3 * i + 0] = (float)(G.c12[0] / G.cov_t * dt);
    p.velocity[3 * i + 1] = (float)(G.c12[1] / G.cov_t * dt);
    p.velocity[3 * i + 2] = (float)(G.c12[2] / G.cov_t * dt);
}

// per-block partial sums (fp64) of the rigidity edge terms w * ||v_j - v_i|| and the motion terms ||v_i||
__global__ void __launch_bounds__(RG_THREADS) rigid_loss_kernel(const RigidParams p, int want_rigid, int want_motion,
                                                                double* __restrict__ partials) {
    __shared__ double sr[RG_THREADS], sm[RG_THREADS];
    const int i = blockIdx.x * RG_THREADS + threadIdx.x;
    double r = 0.0, m = 0.0;
    if (i < p.n) {
        const float vx = p.velocity[3 * i], vy = p.velocity[3 * i + 1], vz = p.velocity[3 * i + 2];
        if (want_rigid) {
            const size_t base = (size_t)i * p.k;
            for (int s = 0; s < p.k; ++s) {
                const int j = p.idx[base + s];
                const float nrm = norm3(fsub(p.velocity[3 * j], vx), fsub(p.velocity[3 * j + 1], vy), fsub(p.velocity[3 * j + 2], vz));
                r += (double)fmul(p.weight[base + s], nrm);
            }
        }
        if (want_motion) m = (double)norm3(vx, vy, vz);
    }
    sr[threadIdx.x] = r;
    sm[threadIdx.x] = m;
    __syncthreads();
#pragma unroll
    for (int s = RG_THREADS / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            sr[threadIdx.x] += sr[threadIdx.x + s];
            sm[threadIdx.x] += sm[threadIdx.x + s];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        partials[2 * blockIdx.x] = sr[0];
        partials[2 * blockIdx.x + 1] = sm[0];
    }
}

// one block: the partials in a fixed order, rounded once to fp32, then the reference's divisions
__global__ void __launch_bounds__(RG_TOTAL_THREADS) rigid_total_kernel(int n, int k, int nblocks, const double* __restrict__ partials,
                                                                       float* loss_rigid, float* loss_motion) {
    __shared__ double sr[RG_TOTAL_THREADS], sm[RG_TOTAL_THREADS];
    double r = 0.0, m = 0.0;
    for (int b = threadIdx.x; b < nblocks; b += RG_TOTAL_THREADS) {
        r += partials[2 * b];
        m += partials[2 * b + 1];
    }
    sr[threadIdx.x] = r;
    sm[threadIdx.x] = m;
    __syncthreads();
#pragma unroll
    for (int s = RG_TOTAL_THREADS / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            sr[threadIdx.x] += sr[threadIdx.x + s];
            sm[threadIdx.x] += sm[threadIdx.x + s];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        // (weight * vel_dist).sum() / k / n                     (train.py:150)
        if (loss_rigid) *loss_rigid = fdiv(fdiv((float)sr[0], (float)k), (float)n);
        // velocity.norm(dim=1).mean(): ATen's mean multiplies the sum by the fp32 factor 1/n
        if (loss_motion) *loss_motion = fmul((float)sm[0], fdiv(1.0f, (float)n));
    }
}

// w * (v_b - v_a) / ||v_b - v_a|| added to (ax, ay, az); nothing where the norm is 0 (torch's norm backward mask)
__device__ __forceinline__ void add_edge(float w, float dx, float dy, float dz, double& ax, double& ay, double& az) {
    const float nrm = norm3(dx, dy, dz);
    if (nrm > 0.f) {
        ax += (double)fdiv(fmul(w, dx), nrm);
        ay += (double)fdiv(fmul(w, dy), nrm);
        az += (double)fdiv(fmul(w, dz), nrm);
    }
}

// gradient w.r.t. the raw quaternion q of q / ||q||, given g w.r.t. the normalised one: (g - (g . u) u) / ||q||, u = q / ||q||,
// in double (act_normalize_bwd in fdgs_common.cuh is its fp32 counterpart of the rasterizer's backward)
__device__ __forceinline__ float4 normalize_bwd_f64(const float4 qf, const double g[4]) {
    const double q[4] = {qf.x, qf.y, qf.z, qf.w};
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    if (!(n > 0.0)) return make_float4(0.f, 0.f, 0.f, 0.f);
    const double dot = (g[0] * q[0] + g[1] * q[1] + g[2] * q[2] + g[3] * q[3]) / (n * n);
    return make_float4((float)((g[0] - dot * q[0]) / n), (float)((g[1] - dot * q[1]) / n), (float)((g[2] - dot * q[2]) / n),
                       (float)((g[3] - dot * q[3]) / n));
}

__global__ void __launch_bounds__(RG_BWD_THREADS) rigid_bwd_kernel(const RigidParams p, const float* __restrict__ grad_rigid,
                                                                   const float* __restrict__ grad_motion, float* __restrict__ dL_dscaling,
                                                                   float* __restrict__ dL_dscaling_t, float* __restrict__ dL_drotation,
                                                                   float* __restrict__ dL_drotation_r) {
    const int i = blockIdx.x * RG_BWD_THREADS + threadIdx.x;
    if (i >= p.n) return;
    const float vx = p.velocity[3 * i], vy = p.velocity[3 * i + 1], vz = p.velocity[3 * i + 2];
    // dL/dv_i, accumulated in double
    double dv[3] = {0.0, 0.0, 0.0};
    if (grad_rigid) {
        // dv_i = s * (-sum_out w_ij (v_j - v_i)/||.|| + sum_in w_mi (v_i - v_m)/||.||), s = g / n / k (autograd's order)
        double ax = 0.0, ay = 0.0, az = 0.0;
        const size_t base = (size_t)i * p.k;
        for (int s = 0; s < p.k; ++s) {
            const int j = p.idx[base + s];
            add_edge(p.weight[base + s], fsub(vx, p.velocity[3 * j]), fsub(vy, p.velocity[3 * j + 1]), fsub(vz, p.velocity[3 * j + 2]),
                     ax, ay, az);
        }
        const int q0 = p.in_offsets[i], q1 = p.in_offsets[i + 1];
        for (int q = q0; q < q1; ++q) {
            const int e = p.in_edges[q];
            const int m = e / p.k;
            add_edge(p.weight[e], fsub(vx, p.velocity[3 * m]), fsub(vy, p.velocity[3 * m + 1]), fsub(vz, p.velocity[3 * m + 2]),
                     ax, ay, az);
        }
        const double s = (double)fdiv(fdiv(*grad_rigid, (float)p.n), (float)p.k);
        dv[0] = s * ax;
        dv[1] = s * ay;
        dv[2] = s * az;
    }
    if (grad_motion) {
        const float nrm = norm3(vx, vy, vz);
        if (nrm > 0.f) {
            const double s = (double)fdiv(*grad_motion, (float)p.n) / (double)nrm;
            dv[0] += s * vx;
            dv[1] += s * vy;
            dv[2] += s * vz;
        }
    }
    // the chain to the raw parameters, in double like the forward
    // v = c12 / cov_t * dt  ->  dL/dc12 = dv * dt / cov_t,  dL/dcov_t = -(dv . c12) * dt / cov_t^2
    RigidGeom G;
    rigid_geometry(p, i, G);
    const double dt = rigid_dt(p.t[i]);
    const double cov_t = G.cov_t;
    const double* c12 = G.c12;
    const double dc12[3] = {dv[0] * dt / cov_t, dv[1] * dt / cov_t, dv[2] * dt / cov_t};
    const double dcovt = -(dv[0] * c12[0] + dv[1] * c12[1] + dv[2] * c12[2]) * dt / (cov_t * cov_t);
    const double d0[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};     // no gradient reaches the 3x3 block
    double gs[4], g_rot[4], g_rotr[4];
    cov4_bwd(d0, dc12, dcovt, G.M, G.R, G.sc, G.rot, G.rotr, gs, g_rot, g_rotr);
    const double* sc = G.sc;
    // through exp and q / ||q|| to the raw parameters
#pragma unroll
    for (int a = 0; a < 3; ++a) dL_dscaling[3 * i + a] = (float)(gs[a] * sc[a]);
    dL_dscaling_t[i] = (float)(gs[3] * sc[3]);
    reinterpret_cast<float4*>(dL_drotation)[i] = normalize_bwd_f64(load_quat(p.rotation, i), g_rot);
    reinterpret_cast<float4*>(dL_drotation_r)[i] = normalize_bwd_f64(load_quat(p.rotation_r, i), g_rotr);
}

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

int key_bits(int n) {
    int b = 1;
    while (b < 31 && (1ll << b) < (long long)n) ++b;
    return b;
}

size_t cub_sort_bytes(long long nk, int n) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const unsigned int*)nullptr, (unsigned int*)nullptr,
                                    (const unsigned int*)nullptr, (unsigned int*)nullptr, (int)nk, 0, key_bits(n));
    return bytes;
}

unsigned grid_of(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace

// neighbours: sorted destinations u32[nk] | edge ids u32[nk] | cub temporary storage;  forward: 2 doubles per block
size_t rigid_scratch_bytes(int n, int k) {
    const long long nk = (long long)n * k;
    const size_t nb = align256(2 * align256(4 * (size_t)nk) + align256(cub_sort_bytes(nk, n)));
    const size_t fw = align256(16 * (size_t)grid_of(n, RG_THREADS));
    return nb > fw ? nb : fw;
}

cudaError_t launch_rigid_neighbours(int n, int k, const int* idx, const float* dist2, char* scratch, float* weight,
                                    int* in_offsets, int* in_edges, cudaStream_t stream) {
    const long long nk = (long long)n * k;
    const size_t row = align256(4 * (size_t)nk);
    unsigned int* sorted_dst = reinterpret_cast<unsigned int*>(scratch);
    unsigned int* edge = reinterpret_cast<unsigned int*>(scratch + row);
    void* temp = scratch + 2 * row;
    rigid_weight_kernel<<<grid_of(nk, RG_THREADS), RG_THREADS, 0, stream>>>(nk, dist2, weight, edge);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    size_t bytes = cub_sort_bytes(nk, n);
    // the neighbour index is the key: 0 <= idx < n, so its low key_bits(n) bits order it
    e = cub::DeviceRadixSort::SortPairs(temp, bytes, reinterpret_cast<const unsigned int*>(idx), sorted_dst, edge,
                                        reinterpret_cast<unsigned int*>(in_edges), (int)nk, 0, key_bits(n), stream);
    if (e != cudaSuccess) return e;
    rigid_offsets_kernel<<<grid_of(nk + 1, RG_THREADS), RG_THREADS, 0, stream>>>(n, nk, sorted_dst, in_offsets);
    return cudaGetLastError();
}

cudaError_t launch_rigid_forward(const RigidParams& p, char* scratch, float* loss_rigid, float* loss_motion, cudaStream_t stream) {
    const unsigned nb = grid_of(p.n, RG_THREADS);
    rigid_velocity_kernel<<<nb, RG_THREADS, 0, stream>>>(p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess || (!loss_rigid && !loss_motion)) return e;
    double* partials = reinterpret_cast<double*>(scratch);
    rigid_loss_kernel<<<nb, RG_THREADS, 0, stream>>>(p, loss_rigid != nullptr, loss_motion != nullptr, partials);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    rigid_total_kernel<<<1, RG_TOTAL_THREADS, 0, stream>>>(p.n, p.k, (int)nb, partials, loss_rigid, loss_motion);
    return cudaGetLastError();
}

cudaError_t launch_rigid_backward(const RigidParams& p, const float* grad_rigid, const float* grad_motion, float* dL_dscaling,
                                  float* dL_dscaling_t, float* dL_drotation, float* dL_drotation_r, cudaStream_t stream) {
    rigid_bwd_kernel<<<grid_of(p.n, RG_BWD_THREADS), RG_BWD_THREADS, 0, stream>>>(p, grad_rigid, grad_motion, dL_dscaling, dL_dscaling_t,
                                                                                 dL_drotation, dL_drotation_r);
    return cudaGetLastError();
}

}  // namespace fdgs
