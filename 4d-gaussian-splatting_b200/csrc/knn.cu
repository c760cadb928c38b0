// knn.cu -- k nearest neighbours of every Gaussian centre among all centres (k <= 32), uniform-grid search.
//
// Replaces, in the reference, pointops2's knnquery (pointops2/src/knnquery/knnquery_cuda_kernel.cu:65-107) as used by
// the rigidity loss (utils/general_utils.py:170-184 knn(), train.py:132-152: k = 20 neighbours of xyz among xyz, once
// per view).  The reference kernel is brute force -- every query scans all n points, O(n^2) per call: 10^10 distance
// evaluations at the 100k points of configs/dnerf/lego.yaml.  Here the points are binned into a uniform grid
// (counting sort by cell: histogram, one-block scan, scatter of a compact float4 copy) and every query walks cubic
// shells of cells outwards from its own cell, stopping as soon as its current k-th best distance cannot be beaten by
// anything outside the shells visited: O(n k) for reasonably uniform clouds.
// Same results as the reference: squared distances evaluated with its expression
// (dx*dx + dy*dy + dz*dz, :92), neighbours ordered by (distance, index) ascending -- the brute-force heap's strict `<`
// keeps the lower index among equal distances -- the query point itself first (distance 0).
// Scratch memory comes from the caller (fdgs_knn_scratch_bytes); nothing is allocated here.
#include "../../include/fdgs.h"
#include "fdgs_internal.h"

namespace fdgs {
namespace {

constexpr int KNN_MAX_K = 32;
constexpr int KNN_MAX_RES = 160;     // cells per axis (4.1 M cells)

struct KnnGrid {
    float lo[3];
    float inv_h, h;
    int res;
};

__device__ __forceinline__ unsigned int f2ord(float f) {      // order-preserving float -> uint
    const unsigned int u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned int u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// bbox[0..2] = min, bbox[3..5] = max (ordered-uint encoding), initialised by knn_init_kernel
__global__ void knn_init_kernel(unsigned int* bbox, unsigned int* cell_count, int ncell_plus1) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 3) bbox[i] = 0xffffffffu;
    else if (i < 6) bbox[i] = 0u;
    for (int c = i; c < ncell_plus1; c += gridDim.x * blockDim.x) cell_count[c] = 0u;
}

__global__ void __launch_bounds__(256) knn_bbox_kernel(int n, const float* __restrict__ xyz, unsigned int* bbox) {
    float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = xyz[3 * i + a];
            lo[a] = fminf(lo[a], v);
            hi[a] = fmaxf(hi[a], v);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], d));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], d));
        }
        if ((threadIdx.x & 31) == 0) {
            atomicMin(&bbox[a], f2ord(lo[a]));
            atomicMax(&bbox[3 + a], f2ord(hi[a]));
        }
    }
}

__device__ __forceinline__ KnnGrid load_grid(const unsigned int* bbox, int res) {
    KnnGrid g;
    float ext = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        g.lo[a] = ord2f(bbox[a]);
        ext = fmaxf(ext, ord2f(bbox[3 + a]) - g.lo[a]);
    }
    g.res = res;
    g.h = fmaxf(ext, 1e-20f) / (float)res * 1.0001f;     // the max corner stays inside the last cell
    g.inv_h = 1.f / g.h;
    return g;
}
__device__ __forceinline__ void cell_of(const KnnGrid& g, float x, float y, float z, int& cx, int& cy, int& cz) {
    cx = min(g.res - 1, max(0, (int)((x - g.lo[0]) * g.inv_h)));
    cy = min(g.res - 1, max(0, (int)((y - g.lo[1]) * g.inv_h)));
    cz = min(g.res - 1, max(0, (int)((z - g.lo[2]) * g.inv_h)));
}

__global__ void __launch_bounds__(256) knn_count_kernel(int n, const float* __restrict__ xyz, const unsigned int* __restrict__ bbox,
                                                        int res, unsigned int* __restrict__ cell_count, unsigned int* __restrict__ cell_of_pt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const KnnGrid g = load_grid(bbox, res);
    int cx, cy, cz;
    cell_of(g, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], cx, cy, cz);
    const unsigned int c = ((unsigned)cz * res + cy) * res + cx;
    cell_of_pt[i] = c;
    atomicAdd(&cell_count[c], 1u);
}

// exclusive scan of cell_count[0..ncell) in place; cell_count[ncell] = n.  One CTA (ncell <= 4.1 M: ~4000 passes of 1024).
__global__ void __launch_bounds__(1024) knn_scan_kernel(int ncell, unsigned int* __restrict__ cnt) {
    __shared__ unsigned int wsum[32];
    __shared__ unsigned int carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < ncell; base += 4096) {
        // 4 consecutive cells per thread
        unsigned int v[4], s = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = base + 4 * tid + j;
            v[j] = (c < ncell) ? cnt[c] : 0u;
            s += v[j];
        }
        unsigned int incl = s;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            unsigned int w = wsum[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned int t = __shfl_up_sync(0xffffffffu, w, d);
                if (lane >= d) w += t;
            }
            wsum[lane] = w;
        }
        __syncthreads();
        unsigned int run = carry + (warp > 0 ? wsum[warp - 1] : 0u) + (incl - s);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = base + 4 * tid + j;
            if (c < ncell) cnt[c] = run;
            run += v[j];
        }
        __syncthreads();
        if (tid == 1023) carry = run;
        __syncthreads();
    }
    if (tid == 0) cnt[ncell] = carry;
}

// cursor = copy of the cell starts; sorted[slot] = (x, y, z, index)
__global__ void __launch_bounds__(256) knn_scatter_kernel(int n, const float* __restrict__ xyz, const unsigned int* __restrict__ cell_of_pt,
                                                          unsigned int* __restrict__ cursor, float4* __restrict__ sorted) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned int slot = atomicAdd(&cursor[cell_of_pt[i]], 1u);
    sorted[slot] = make_float4(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], __int_as_float(i));
}

__global__ void __launch_bounds__(128) knn_search_kernel(int n, int k, const float* __restrict__ xyz, const unsigned int* __restrict__ bbox,
                                                         int res, const unsigned int* __restrict__ cell_start,
                                                         const float4* __restrict__ sorted, int* __restrict__ out_idx,
                                                         float* __restrict__ out_d2) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    const KnnGrid g = load_grid(bbox, res);
    const float qx = xyz[3 * q], qy = xyz[3 * q + 1], qz = xyz[3 * q + 2];
    int cx, cy, cz;
    cell_of(g, qx, qy, qz, cx, cy, cz);
    float bd[KNN_MAX_K];
    int bi[KNN_MAX_K];
    int cnt = 0;
    // distance from the query to the nearest face of its own cell: everything beyond shell r is at least r*h + margin away.
    // The faces the binning uses are where fl(fl(x - lo) * inv_h) crosses an integer, not the c*h measured here: the two
    // differ by the rounding of x - lo, of the product and of inv_h = fl(1/h), up to ~3 * 2^-24 * (c + 1) * h.  A query
    // within that of a face could otherwise stop at shell 0 before a closer point the rounding put in the next cell, so
    // the margin gives up 1e-6 * (res + 1) * h (>= 16x the bound; at most 1.6e-4 h at 160 cells per axis).
    float margin = g.h;
    {
        const float fx = (qx - g.lo[0]) - cx * g.h, fy = (qy - g.lo[1]) - cy * g.h, fz = (qz - g.lo[2]) - cz * g.h;
        margin = fminf(margin, fminf(fminf(fx, g.h - fx), fminf(fminf(fy, g.h - fy), fminf(fz, g.h - fz))));
        margin = fmaxf(margin - 1e-6f * (float)(res + 1) * g.h, 0.f);
    }
    for (int r = 0; r < res; ++r) {
        const int z0 = cz - r, z1 = cz + r, y0 = cy - r, y1 = cy + r, x0 = cx - r, x1 = cx + r;
        for (int z = max(z0, 0); z <= min(z1, res - 1); ++z) {
            for (int y = max(y0, 0); y <= min(y1, res - 1); ++y) {
                const bool face = (z == z0) || (z == z1) || (y == y0) || (y == y1);
                // on a face of the shell the whole x-row belongs to it; otherwise only its two end cells
                const int xs = face ? 1 : max(2 * r, 1);
                for (int x = x0; x <= x1; x += xs) {
                    if (x < 0 || x >= res) continue;
                    const unsigned int c = ((unsigned)z * res + y) * res + x;
                    const unsigned int s = cell_start[c], e = cell_start[c + 1];
                    for (unsigned int p = s; p < e; ++p) {
                        const float4 pt = sorted[p];
                        const float dx = qx - pt.x, dy = qy - pt.y, dz = qz - pt.z;
                        const float d2 = dx * dx + dy * dy + dz * dz;     // reference: knnquery_cuda_kernel.cu:92
                        const int id = __float_as_int(pt.w);
                        if (cnt == k && !(d2 < bd[k - 1] || (d2 == bd[k - 1] && id < bi[k - 1]))) continue;
                        // insertion into the list sorted by (d2, index)
                        int j = (cnt < k) ? cnt : k - 1;
                        while (j > 0 && (bd[j - 1] > d2 || (bd[j - 1] == d2 && bi[j - 1] > id))) {
                            bd[j] = bd[j - 1];
                            bi[j] = bi[j - 1];
                            --j;
                        }
                        bd[j] = d2;
                        bi[j] = id;
                        if (cnt < k) ++cnt;
                    }
                }
            }
        }
        if (cnt == k) {
            const float reach = (float)r * g.h + margin;
            if (bd[k - 1] <= reach * reach * 0.9999f) break;    // nothing outside the visited shells can be closer
        }
    }
    for (int j = 0; j < k; ++j) {
        // fewer than k points in total: pad like the reference's initial heap (index 0, distance 1e10, :82-85)
        out_idx[(size_t)q * k + j] = (j < cnt) ? bi[j] : 0;
        out_d2[(size_t)q * k + j] = (j < cnt) ? bd[j] : 1e10f;
    }
}

// brute force, the reference's algorithm (one thread per query scans all points): the checker of the grid search
__global__ void __launch_bounds__(128) knn_bruteforce_kernel(int n, int k, const float* __restrict__ xyz, int* __restrict__ out_idx,
                                                             float* __restrict__ out_d2) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    const float qx = xyz[3 * q], qy = xyz[3 * q + 1], qz = xyz[3 * q + 2];
    float bd[KNN_MAX_K];
    int bi[KNN_MAX_K];
    int cnt = 0;
    for (int i = 0; i < n; ++i) {
        const float dx = qx - xyz[3 * i], dy = qy - xyz[3 * i + 1], dz = qz - xyz[3 * i + 2];
        const float d2 = dx * dx + dy * dy + dz * dz;
        if (cnt == k && !(d2 < bd[k - 1])) continue;      // strict <: the lower index wins among equals (:93)
        int j = (cnt < k) ? cnt : k - 1;
        while (j > 0 && bd[j - 1] > d2) {
            bd[j] = bd[j - 1];
            bi[j] = bi[j - 1];
            --j;
        }
        bd[j] = d2;
        bi[j] = i;
        if (cnt < k) ++cnt;
    }
    for (int j = 0; j < k; ++j) {
        out_idx[(size_t)q * k + j] = (j < cnt) ? bi[j] : 0;
        out_d2[(size_t)q * k + j] = (j < cnt) ? bd[j] : 1e10f;
    }
}

int grid_res(int n) {
    // ~4 points per cell on average for a uniform cloud
    int res = (int)ceil(cbrt((double)n / 4.0));
    if (res < 1) res = 1;
    if (res > KNN_MAX_RES) res = KNN_MAX_RES;
    return res;
}

}  // namespace

size_t knn_scratch_bytes(int n) {
    const size_t res = (size_t)grid_res(n);
    const size_t ncell = res * res * res;
    // bbox (8 words) | cell starts (ncell + 1) | cursor (ncell + 1) | cell of point (n) | sorted float4 (n)
    return 128 + 4 * (8 + 2 * (ncell + 1) + (size_t)n) + 16 * ((size_t)n + 1) + 256;
}

cudaError_t launch_knn(int n, int k, const float* xyz, char* scratch, int* idx, float* dist2, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    const int res = grid_res(n);
    const int ncell = res * res * res;
    unsigned int* bbox = reinterpret_cast<unsigned int*>(scratch);
    unsigned int* cell_start = bbox + 8;
    unsigned int* cursor = cell_start + ncell + 1;
    unsigned int* cell_of_pt = cursor + ncell + 1;
    uintptr_t sp = reinterpret_cast<uintptr_t>(cell_of_pt + n);
    sp = (sp + 15) & ~(uintptr_t)15;
    float4* sorted = reinterpret_cast<float4*>(sp);
    const int nb = (n + 255) / 256;
    knn_init_kernel<<<min(1024, (ncell + 1 + 255) / 256), 256, 0, stream>>>(bbox, cell_start, ncell + 1);
    knn_bbox_kernel<<<min(nb, device_sm_count() * 8), 256, 0, stream>>>(n, xyz, bbox);
    knn_count_kernel<<<nb, 256, 0, stream>>>(n, xyz, bbox, res, cell_start, cell_of_pt);
    knn_scan_kernel<<<1, 1024, 0, stream>>>(ncell, cell_start);
    cudaError_t e = cudaMemcpyAsync(cursor, cell_start, (size_t)(ncell + 1) * 4, cudaMemcpyDeviceToDevice, stream);
    if (e != cudaSuccess) return e;
    knn_scatter_kernel<<<nb, 256, 0, stream>>>(n, xyz, cell_of_pt, cursor, sorted);
    knn_search_kernel<<<(n + 127) / 128, 128, 0, stream>>>(n, k, xyz, bbox, res, cell_start, sorted, idx, dist2);
    return cudaGetLastError();
}

cudaError_t launch_knn_bruteforce(int n, int k, const float* xyz, int* idx, float* dist2, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    knn_bruteforce_kernel<<<(n + 127) / 128, 128, 0, stream>>>(n, k, xyz, idx, dist2);
    return cudaGetLastError();
}

}  // namespace fdgs
