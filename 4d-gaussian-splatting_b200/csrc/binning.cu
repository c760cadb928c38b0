// binning.cu -- tile binning: per-tile counting, offsets, scatter, per-tile sort + instance packing.
//
// Replaces, in the reference: cub::DeviceScan::InclusiveSum over P Gaussians
// (rasterizer_impl.cu:298), duplicateWithKeys (:71-112), the 64-bit cub::DeviceRadixSort::SortPairs
// over all R instances (:325-330), the ranges memset + identifyTileRanges (:117-139, :332-339).
//
// The contract is the ORDER of every tile's work list ("tile assignment bit-exact"): instances of
// a tile sorted by depth bits, ties broken by Gaussian index -- exactly what the reference's
// stable LSD sort of (tile<<32 | depth_bits) with values emitted in Gaussian-index order produces.
// (depth, index) is a total order with unique keys, so ANY sorting algorithm gives the same list.
// That freedom is what this file exploits; no global sort exists here:
//
//   1. count      bin_pass_kernel<false>: BIN_CTAS persistent CTAs, each owning one contiguous chunk of
//                 Gaussians (read as compact 16-byte bin records: tile rectangle + depth bits, written by
//                 the preprocess), histogram the tiles their rendered Gaussians touch in SHARED memory
//                 (a warp walks one Gaussian's tile rectangle with 32 lanes) and store the
//                 histogram as one row of a [BIN_CTAS][tiles] matrix.  No global atomics.
//   2. offsets    column_scan_kernel: one thread per tile, exclusive prefix down the matrix column
//                 (= where each CTA's instances of that tile start inside the tile's list) and the
//                 tile's total.  tile_scan_kernel: one CTA, exclusive scan of the tile totals ->
//                 tile offsets; writes the per-tile [start,end) ranges directly (no
//                 identifyTileRanges pass, no memset), the total R and the largest tile, which the
//                 host reads back -- the one synchronisation of the forward, as in the reference
//                 (rasterizer_impl.cu:302).
//   3. scatter    bin_pass_kernel<true>: same chunks, same walk; the shared-memory histogram now
//                 starts at tile_offset + column prefix, so a shared-memory atomicAdd hands out the
//                 final slot of the 64-bit key depth_bits<<32 | index.  Order inside a CTA's
//                 segment is arbitrary; step 4 makes it canonical.
//   4. sort+pack  tile_sort_kernel: one CTA per tile merge-sorts the tile's keys in shared memory (a
//                 second, large-shared-memory instantiation takes the tiles above 2048 instances;
//                 tiles above 16384 fall back to a bitonic network in place in global memory), writes
//                 the sorted index list (the reference's point_list) and, from the ids still in shared
//                 memory, gathers the 64-byte per-Gaussian records into tile-sorted order -- the
//                 contiguous stream the blend kernels read with cp.async.bulk.  Gather latency of one
//                 CTA overlaps the shared-memory sort of its SM neighbours.
//
// Traffic per instance: 8 B key write + 8 B read + 64 B record write (+ 64 B L2-resident record
// read), versus ~200 B for the reference's 8-pass radix sort (SURVEY.md section 8a, row a10).
#include "fdgs_internal.h"

namespace fdgs {
namespace {

constexpr int BIN_CTAS_MAX = 192;  // upper bound of the row count of the count matrix (register array in column_scan)
// one persistent CTA per SM of the current device (132 on an H100); also the row count of the count matrix
inline int bin_cta_count() { return min(device_sm_count(), BIN_CTAS_MAX); }
constexpr int BIN_THREADS = 1024;
constexpr int BIN_SMALL = 8;       // rectangles of up to this many tiles are binned by their own lane
constexpr int SCAN_THREADS = 1024;
constexpr size_t BIN_SMEM_LIMIT = 200 * 1024;

// ---- 1 + 3. count / scatter ----------------------------------------------------------------------------
// SCATTER = false: row[t] = number of (Gaussian, tile) instances of this CTA's chunk in tile t.
// SCATTER = true : row[t] holds the column prefix on entry; keys are written to
//                  tile_offset[t] + row[t] + (arrival order inside the CTA).
// SMEM: histogram lives in shared memory; otherwise (very large tile grids) the CTA-private global row is used in place.
// BATCH: blockIdx.y = view; binrec is a [views][P] stack and view v owns the columns v * num_tiles .. of matrix rows of
// views * num_tiles columns (the shared-memory histogram stays one image's tiles)
template <bool SCATTER, bool SMEM, bool BATCH>
__device__ __forceinline__ void bin_pass_body(int P, int chunk, const uint4* __restrict__ binrec, int grid_x,
                                                               int num_tiles, uint32_t* __restrict__ matrix,
                                                               const uint32_t* __restrict__ tile_offset,
                                                               uint64_t* __restrict__ keys) {
    extern __shared__ uint32_t hist_smem[];
    uint32_t* row = matrix + (size_t)blockIdx.x * num_tiles;
    if (BATCH) {
        const size_t v = blockIdx.y;
        row = matrix + ((size_t)blockIdx.x * gridDim.y + v) * num_tiles;
        binrec += v * (size_t)P;
        if (SCATTER) tile_offset += v * (size_t)num_tiles;
    }
    uint32_t* hist = SMEM ? hist_smem : row;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int t = tid; t < num_tiles; t += BIN_THREADS) {
        if (SCATTER) hist[t] = row[t] + tile_offset[t];
        else hist[t] = 0u;
    }
    __syncthreads();
    const int begin = blockIdx.x * chunk;
    const int end = min(P, begin + chunk);
    // one coalesced 16-byte record per Gaussian (written by the preprocess for EVERY Gaussian; an empty
    // rectangle = not rendered); the next iteration's record is in flight while this one is binned
    const uint4 none = make_uint4(0u, 0u, 0u, 0u);
    int g0 = begin + warp * 32;
    uint4 nxt = (g0 + lane < end) ? binrec[g0 + lane] : none;
    for (; g0 < end; g0 += BIN_THREADS) {
        const uint4 br = nxt;
        const int gn = g0 + BIN_THREADS + lane;
        nxt = (gn < end) ? binrec[gn] : none;
        // x = x0 | y0 << 16, y = x1 | y1 << 16 (tile coordinates), z = depth bits
        const int x0 = (int)(br.x & 0xffffu), y0 = (int)(br.x >> 16), x1 = (int)(br.y & 0xffffu), y1 = (int)(br.y >> 16);
        const int w = x1 - x0;
        const int n = ((x1 > x0) && (y1 > y0)) ? w * (y1 - y0) : 0;
        // Small rectangles (the common case: a ~1.5-pixel-sigma Gaussian touches 1-4 tiles) are walked by their own
        // lane -- no shuffles, no division, the warp runs for max(n) <= BIN_SMALL iterations; only the large ones
        // are spread over the 32 lanes.  The order inside a tile's segment is arbitrary either way (sorted later).
        // br.w: tile mask of rectangles of up to 32 tiles (bit i = tile i, row-major, takes an instance; all ones when
        // the preprocess did not cull by tile)
        if (n > 0 && n <= BIN_SMALL) {
            const uint64_t key = SCATTER ? (((uint64_t)br.z << 32) | (uint32_t)(g0 + lane)) : 0ull;
            uint32_t m = br.w;
            for (int ty = y0; ty < y1; ++ty) {
                for (int tx = x0; tx < x1; ++tx, m >>= 1) {
                    if (!(m & 1u)) continue;
                    const uint32_t slot = atomicAdd(&hist[ty * grid_x + tx], 1u);
                    if (SCATTER) keys[slot] = key;
                }
            }
        }
        uint32_t mask = __ballot_sync(0xffffffffu, n > BIN_SMALL);
        while (mask) {
            const int src = __ffs(mask) - 1;
            mask &= mask - 1;
            const int bx0 = __shfl_sync(0xffffffffu, x0, src), by0 = __shfl_sync(0xffffffffu, y0, src);
            const int bw = __shfl_sync(0xffffffffu, w, src), bn = __shfl_sync(0xffffffffu, n, src);
            const uint32_t bmask = __shfl_sync(0xffffffffu, br.w, src);
            uint64_t key = 0;
            // key: depth bits (positive floats: integer order == float order) then Gaussian index
            if (SCATTER) key = ((uint64_t)__shfl_sync(0xffffffffu, br.z, src) << 32) | (uint32_t)(g0 + src);
            for (int i = lane; i < bn; i += 32) {
                if (bn <= 32 && !((bmask >> i) & 1u)) continue;
                const int ry = i / bw, rx = i - ry * bw;
                const int t = (by0 + ry) * grid_x + bx0 + rx;
                const uint32_t slot = atomicAdd(&hist[t], 1u);
                if (SCATTER) keys[slot] = key;
            }
        }
    }
    if (!SCATTER && SMEM) {
        __syncthreads();
        for (int t = tid; t < num_tiles; t += BIN_THREADS) row[t] = hist[t];
    }
}

template <bool SCATTER, bool SMEM>
__global__ void __launch_bounds__(BIN_THREADS) bin_pass_kernel(int P, int chunk, const uint4* __restrict__ binrec, int grid_x,
                                                               int num_tiles, uint32_t* __restrict__ matrix,
                                                               const uint32_t* __restrict__ tile_offset,
                                                               uint64_t* __restrict__ keys) {
    bin_pass_body<SCATTER, SMEM, false>(P, chunk, binrec, grid_x, num_tiles, matrix, tile_offset, keys);
}

// the batched entry (fdgs_forward_batch / fdgs_backward_batch): one view per blockIdx.y
template <bool SCATTER, bool SMEM>
__global__ void __launch_bounds__(BIN_THREADS) bin_pass_batch_kernel(int P, int chunk, const uint4* __restrict__ binrec, int grid_x,
                                                               int num_tiles, uint32_t* __restrict__ matrix,
                                                               const uint32_t* __restrict__ tile_offset,
                                                               uint64_t* __restrict__ keys) {
    bin_pass_body<SCATTER, SMEM, true>(P, chunk, binrec, grid_x, num_tiles, matrix, tile_offset, keys);
}

// the capacity entry (fdgs_forward_batch_capacity): info[3] != 0 -- the instances do not fit the binning buffer, or their
// total wraps the 32-bit offsets -- and no key is written (tile_scan_body<true> has emptied every tile's range)
template <bool SMEM>
__global__ void __launch_bounds__(BIN_THREADS) bin_scatter_cap_kernel(int P, int chunk, const uint4* __restrict__ binrec, int grid_x,
                                                                      int num_tiles, uint32_t* __restrict__ matrix,
                                                                      const uint32_t* __restrict__ tile_offset,
                                                                      uint64_t* __restrict__ keys, const uint32_t* __restrict__ info) {
    if (info[3] != 0u) return;
    bin_pass_body<true, SMEM, true>(P, chunk, binrec, grid_x, num_tiles, matrix, tile_offset, keys);
}

// ---- 2. offsets ------------------------------------------------------------------------------------
// 32 tiles x 8 row groups per CTA: every thread owns <= ceil(rows / 8) consecutive rows of one tile column
// (kept in registers), the groups' partial sums are combined through shared memory.  Coalesced along tiles.
constexpr int CS_GROUPS = 8;
constexpr int CS_MAXROWS = (BIN_CTAS_MAX + CS_GROUPS - 1) / CS_GROUPS;
__global__ void __launch_bounds__(256) column_scan_kernel(int num_tiles, int rows, uint32_t* __restrict__ matrix,
                                                          uint32_t* __restrict__ tile_total) {
    __shared__ uint32_t part[CS_GROUPS][32];
    const int tx = threadIdx.x & 31, grp = threadIdx.x >> 5;
    const int t = blockIdx.x * 32 + tx;
    const int per = (rows + CS_GROUPS - 1) / CS_GROUPS;
    const int r0 = grp * per, r1 = min(rows, r0 + per);
    uint32_t v[CS_MAXROWS];
    uint32_t sum = 0;
#pragma unroll
    for (int i = 0; i < CS_MAXROWS; ++i) {
        const int r = r0 + i;
        v[i] = (t < num_tiles && r < r1) ? matrix[(size_t)r * num_tiles + t] : 0u;
        sum += v[i];
    }
    part[grp][tx] = sum;
    __syncthreads();
    uint32_t run = 0, total = 0;
#pragma unroll
    for (int g = 0; g < CS_GROUPS; ++g) {
        const uint32_t pg = part[g][tx];
        if (g < grp) run += pg;
        total += pg;
    }
    if (t >= num_tiles) return;
#pragma unroll
    for (int i = 0; i < CS_MAXROWS; ++i) {
        const int r = r0 + i;
        if (r < r1) matrix[(size_t)r * num_tiles + t] = run;
        run += v[i];
    }
    if (grp == 0) tile_total[t] = total;
}

// CAP (the capacity entry): also status = {R, largest tile, R > capacity, wrap} and info[3] = overflow or wrap; on either,
// every tile's range is emptied afterwards, so the views render as if no Gaussian were listed
template <bool CAP>
__device__ __forceinline__ void tile_scan_body(int num_tiles, const uint32_t* __restrict__ tile_total,
                                               uint32_t* __restrict__ tile_offset, uint2* __restrict__ ranges,
                                               uint32_t* __restrict__ info, int capacity, int* __restrict__ status) {
    __shared__ uint32_t warp_sums[SCAN_THREADS / 32];
    __shared__ uint32_t carry;
    __shared__ uint32_t max_count;
    __shared__ unsigned long long total64;   // the true instance total: detects a wrap of the 32-bit offsets
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { carry = 0; max_count = 0; total64 = 0ull; }
    __syncthreads();
    uint32_t my_max = 0;
    for (int base = 0; base < num_tiles; base += SCAN_THREADS) {
        const int t = base + tid;
        const uint32_t c = (t < num_tiles) ? tile_total[t] : 0u;
        my_max = max(my_max, c);
        uint32_t incl = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t n = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += n;
        }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = warp_sums[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t n = __shfl_up_sync(0xffffffffu, w, d);
                if (lane >= d) w += n;
            }
            warp_sums[lane] = w;   // inclusive over warps
        }
        __syncthreads();
        const uint32_t before = carry + (warp > 0 ? warp_sums[warp - 1] : 0u) + (incl - c);
        if (t < num_tiles) {
            tile_offset[t] = before;
            // empty tiles get (0,0) like the reference's memset (rasterizer_impl.cu:332)
            ranges[t] = c ? make_uint2(before, before + c) : make_uint2(0u, 0u);
        }
        __syncthreads();
        if (tid == SCAN_THREADS - 1) {
            total64 += (unsigned long long)warp_sums[SCAN_THREADS / 32 - 1];
            carry = before + c;
        }
        __syncthreads();
    }
    atomicMax(&max_count, my_max);
    __syncthreads();
    // info[2] != 0: more than 2^31 - 1 instances -- the 32-bit offsets / the int num_rendered of the API cannot hold it
    if (tid == 0) { info[0] = carry; info[1] = max_count; info[2] = (total64 > 0x7fffffffull) ? 1u : 0u; info[3] = 0u; }
    if (CAP) {
        if (tid == 0) {
            const bool wrap = total64 > 0x7fffffffull, over = total64 > (unsigned long long)capacity;
            status[0] = (int)min(total64, 0x7fffffffull);
            status[1] = (int)max_count;
            status[2] = over ? 1 : 0;
            status[3] = wrap ? 1 : 0;
            info[3] = (over || wrap) ? 1u : 0u;
            warp_sums[0] = (over || wrap) ? 1u : 0u;   // the scan is done with it
        }
        __syncthreads();
        if (warp_sums[0] != 0u)
            for (int t = tid; t < num_tiles; t += SCAN_THREADS) ranges[t] = make_uint2(0u, 0u);
    }
}

__global__ void __launch_bounds__(SCAN_THREADS) tile_scan_kernel(int num_tiles, const uint32_t* __restrict__ tile_total,
                                                                 uint32_t* __restrict__ tile_offset,
                                                                 uint2* __restrict__ ranges, uint32_t* __restrict__ info) {
    tile_scan_body<false>(num_tiles, tile_total, tile_offset, ranges, info, 0, nullptr);
}

__global__ void __launch_bounds__(SCAN_THREADS) tile_scan_cap_kernel(int num_tiles, const uint32_t* __restrict__ tile_total,
                                                                     uint32_t* __restrict__ tile_offset,
                                                                     uint2* __restrict__ ranges, uint32_t* __restrict__ info,
                                                                     int capacity, int* __restrict__ status) {
    tile_scan_body<true>(num_tiles, tile_total, tile_offset, ranges, info, capacity, status);
}

// ---- 4. per-tile sort ------------------------------------------------------------------------------------
// Block merge sort of one tile's 64-bit keys: every thread sorts KPT keys in registers (bitonic
// network, static indices), then log2(runs) merge passes through shared memory -- each thread finds
// its KPT-element slice of the merged pair of runs with a merge-path binary search and merges it
// serially.  O(n log n) compare work and one shared-memory round trip per pass, against the
// O(n log^2 n) exchanges of a bitonic network.  Shared-memory slots are padded by one key per KPT
// (odd 8-byte stride per thread -> conflict-free stores).
constexpr uint64_t KEY_SENTINEL = ~0ull;   // > every real key (depth bits of a positive float are < 0x7f800000)

__device__ __forceinline__ void key_cswap(uint64_t& a, uint64_t& b) {
    if (a > b) { const uint64_t t = a; a = b; b = t; }
}

template <int KPT>
__device__ __forceinline__ void register_sort(uint64_t (&k)[KPT]) {
    static_assert((KPT & (KPT - 1)) == 0, "power of two");
#pragma unroll
    for (int size = 2; size <= KPT; size <<= 1) {
#pragma unroll
        for (int i = 0; i < KPT; ++i) {
            const int j = i ^ (size - 1);
            if (j > i) key_cswap(k[i], k[j]);
        }
#pragma unroll
        for (int stride = size >> 2; stride > 0; stride >>= 1) {
#pragma unroll
            for (int i = 0; i < KPT; ++i)
                if ((i & stride) == 0) key_cswap(k[i], k[i + stride]);
        }
    }
}

template <int KPT>
__device__ __forceinline__ int slot(int p) {   // padded shared-memory position of logical key p
    return p + p / KPT;
}

// Sorts gk[0..n) (n <= THREADS * KPT) and writes the sorted Gaussian indices to ids[0..n).
template <int THREADS, int KPT>
__device__ __forceinline__ void block_merge_sort(uint64_t* sm, const uint64_t* __restrict__ gk, int n,
                                                 uint32_t* __restrict__ ids) {
    const int tid = threadIdx.x;
    const int nthr = (n + KPT - 1) / KPT;   // threads that own at least one real key
    const int N = nthr * KPT;
    const int start = tid * KPT;
    uint64_t k[KPT];
#pragma unroll
    for (int i = 0; i < KPT; ++i) k[i] = (start + i < n) ? gk[start + i] : KEY_SENTINEL;
    if (tid < nthr) register_sort<KPT>(k);
    for (int len = KPT; len < N; len <<= 1) {
        __syncthreads();   // the previous pass has finished reading
        if (tid < nthr) {
#pragma unroll
            for (int i = 0; i < KPT; ++i) sm[slot<KPT>(start + i)] = k[i];
        }
        __syncthreads();
        if (tid < nthr) {
            const int pair = start & ~(2 * len - 1);
            const int a0 = pair, a1 = min(pair + len, N), b0 = a1, b1 = min(pair + 2 * len, N);
            const int diag = start - pair;
            // merge path: how many of the first `diag` outputs come from run A
            int lo = max(0, diag - (b1 - b0)), hi = min(diag, a1 - a0);
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                const uint64_t ka = sm[slot<KPT>(a0 + mid)], kb = sm[slot<KPT>(b0 + diag - 1 - mid)];
                if (ka <= kb) lo = mid + 1;
                else hi = mid;
            }
            int ia = a0 + lo, ib = b0 + diag - lo;
            uint64_t ka = (ia < a1) ? sm[slot<KPT>(ia)] : KEY_SENTINEL;
            uint64_t kb = (ib < b1) ? sm[slot<KPT>(ib)] : KEY_SENTINEL;
#pragma unroll
            for (int i = 0; i < KPT; ++i) {
                const bool take_a = ka <= kb;
                k[i] = take_a ? ka : kb;
                if (take_a) { ++ia; ka = (ia < a1) ? sm[slot<KPT>(ia)] : KEY_SENTINEL; }
                else { ++ib; kb = (ib < b1) ? sm[slot<KPT>(ib)] : KEY_SENTINEL; }
            }
        }
    }
    __syncthreads();   // the last merge pass has finished reading the key array: reuse it for the sorted ids
    uint32_t* sid = reinterpret_cast<uint32_t*>(sm);
    if (tid < nthr) {
#pragma unroll
        for (int i = 0; i < KPT; ++i)
            if (start + i < n) {
                const uint32_t id = (uint32_t)(k[i] & 0xffffffffu);
                ids[start + i] = id;
                sid[start + i] = id;
            }
    }
    __syncthreads();
}

// recs[i] = grec[ids[i]] for one tile: the 64-byte records in tile-sorted order, the contiguous stream the
// blend kernels read with cp.async.bulk.  4 lanes copy one record (coalesced 64-byte stores, gathered loads);
// 4 independent gathers per thread in flight.
template <int THREADS>
__device__ __forceinline__ void gather_records(const uint32_t* ids /* shared or global */, int n,
                                               const InstRec* __restrict__ grec, StageRec* __restrict__ recs) {
    const float4* src = reinterpret_cast<const float4*>(grec);
    float4* dst = reinterpret_cast<float4*>(recs);   // 5 float4 per staged record, the fifth is padding
    // thread q writes the q-th float4 of the tile's output stream: fully coalesced stores; 4 of every 5
    // consecutive threads read the 4 planes of one gathered record (one 64-byte line)
    const int total = 5 * n;
    for (int q0 = threadIdx.x; q0 < total; q0 += 4 * THREADS) {
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int q = q0 + u * THREADS;
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (q < total) {
                const int i = q / 5, part = q - 5 * i;
                if (part < 4) v[u] = __ldg(src + (size_t)ids[i] * 4 + part);
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int q = q0 + u * THREADS;
            if (q < total) dst[q] = v[u];
        }
    }
}

// Bitonic sorting network in its "flip" form (every sub-sequence ascending), for an arbitrary n:
// positions >= n behave as +infinity and never move, so comparisons that would touch them are
// simply skipped.  Only used in place in global memory, for tiles too large for shared memory.
__device__ __forceinline__ void bitonic_sort(uint64_t* k, int n, int tid, int nthreads) {
    int np = 1;
    while (np < n) np <<= 1;
    const int half = np >> 1;
    for (int size = 2; size <= np; size <<= 1) {
        __syncthreads();
        const int hs = size >> 1, lg = __ffs(hs) - 1;
        for (int i = tid; i < half; i += nthreads) {
            const int blk = i >> lg, j = i & (hs - 1);
            const int lo = blk * size + j, hi = blk * size + size - 1 - j;
            if (hi < n) {
                const uint64_t a = k[lo], b = k[hi];
                if (a > b) { k[lo] = b; k[hi] = a; }
            }
        }
        for (int stride = size >> 2; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int i = tid; i < half; i += nthreads) {
                const int lo = 2 * i - (i & (stride - 1));
                const int hi = lo + stride;
                if (hi < n) {
                    const uint64_t a = k[lo], b = k[hi];
                    if (a > b) { k[lo] = b; k[hi] = a; }
                }
            }
        }
    }
    __syncthreads();
}

constexpr int SORT_SMALL_THREADS = 256, SORT_SMALL_KEYS = 2048;      // 18 KB of shared memory, 8 keys per thread
constexpr int SORT_LARGE_THREADS = 1024, SORT_LARGE_KEYS = 16384;    // 139 KB of shared memory, 16 keys per thread

// One CTA per tile.  LARGE = false handles the tiles with n <= 2048, LARGE = true those above (launched
// only if the largest tile needs it); tiles above 16384 instances sort in place in global memory.
// BATCH: one CTA per (view, tile); the keys hold Gaussian indices in [0, P) and the records are gathered from the view's
// slice of grec, a [views][P] stack
template <bool LARGE, bool BATCH>
__device__ __forceinline__ void tile_sort_body(const uint2* __restrict__ ranges, uint64_t* __restrict__ keys, uint32_t* __restrict__ point_list,
                 const InstRec* __restrict__ grec, StageRec* __restrict__ recs, int tiles_per_view, int P) {
    extern __shared__ uint64_t skeys[];
    const uint2 range = ranges[blockIdx.x];
    const int n = (int)(range.y - range.x);
    if (n <= 0) return;
    if (BATCH) grec += (size_t)(blockIdx.x / tiles_per_view) * (size_t)P;
    uint64_t* gk = keys + range.x;
    uint32_t* ids = point_list + range.x;
    if (!LARGE) {
        if (n > SORT_SMALL_KEYS) return;
        block_merge_sort<SORT_SMALL_THREADS, 8>(skeys, gk, n, ids);
        gather_records<SORT_SMALL_THREADS>(reinterpret_cast<const uint32_t*>(skeys), n, grec, recs + range.x);
    } else {
        if (n <= SORT_SMALL_KEYS) return;
        if (n <= SORT_LARGE_KEYS) {
            block_merge_sort<SORT_LARGE_THREADS, 16>(skeys, gk, n, ids);
            gather_records<SORT_LARGE_THREADS>(reinterpret_cast<const uint32_t*>(skeys), n, grec, recs + range.x);
        } else {
            bitonic_sort(gk, n, threadIdx.x, SORT_LARGE_THREADS);
            for (int i = threadIdx.x; i < n; i += SORT_LARGE_THREADS) ids[i] = (uint32_t)(gk[i] & 0xffffffffu);
            __syncthreads();
            gather_records<SORT_LARGE_THREADS>(ids, n, grec, recs + range.x);
        }
    }
}

template <bool LARGE>
__global__ void __launch_bounds__(LARGE ? SORT_LARGE_THREADS : SORT_SMALL_THREADS) tile_sort_kernel(const uint2* __restrict__ ranges, uint64_t* __restrict__ keys, uint32_t* __restrict__ point_list,
                 const InstRec* __restrict__ grec, StageRec* __restrict__ recs, int tiles_per_view, int P) {
    tile_sort_body<LARGE, false>(ranges, keys, point_list, grec, recs, tiles_per_view, P);
}

// the batched entry (fdgs_forward_batch / fdgs_backward_batch): one view per (view, tile) CTA
template <bool LARGE>
__global__ void __launch_bounds__(LARGE ? SORT_LARGE_THREADS : SORT_SMALL_THREADS) tile_sort_batch_kernel(const uint2* __restrict__ ranges, uint64_t* __restrict__ keys, uint32_t* __restrict__ point_list,
                 const InstRec* __restrict__ grec, StageRec* __restrict__ recs, int tiles_per_view, int P) {
    tile_sort_body<LARGE, true>(ranges, keys, point_list, grec, recs, tiles_per_view, P);
}

// The capacity entry's per-view table from device arrays; the focal lengths are rounded as the host computes them for
// fdgs_forward_batch (W / (2 tan), IEEE division), so both entries see bit-identical tables
__global__ void view_table_kernel(int B, int W, int H, const float* __restrict__ timestamps, const float* __restrict__ tan_fovx,
                                  const float* __restrict__ tan_fovy, ViewScalars* __restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= B) return;
    ViewScalars s;
    s.timestamp = timestamps[v];
    s.tan_fovx = tan_fovx[v];
    s.tan_fovy = tan_fovy[v];
    s.focal_y = __fdiv_rn((float)H, __fmul_rn(2.0f, s.tan_fovy));
    s.focal_x = __fdiv_rn((float)W, __fmul_rn(2.0f, s.tan_fovx));
    s.pad[0] = s.pad[1] = s.pad[2] = 0.f;
    out[v] = s;
}

// test hook: unpack the per-Gaussian records into the reference's plain arrays; `radii` is any
// per-Gaussian int array that is > 0 exactly for the rendered Gaussians (radii or tiles_touched)
__global__ void unpack_grec_kernel(int P, const InstRec* __restrict__ grec, const int* __restrict__ radii,
                                   float* depths, float* means2D, float* conic_opacity, float* rgb) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const bool vis = radii[idx] > 0;
    const InstRec r = grec[idx];
    if (depths) depths[idx] = vis ? r.q2.w : 0.f;
    if (means2D) { means2D[2 * idx] = vis ? r.q0.x : 0.f; means2D[2 * idx + 1] = vis ? r.q0.y : 0.f; }
    if (conic_opacity) {
        conic_opacity[4 * idx + 0] = vis ? r.q1.x : 0.f; conic_opacity[4 * idx + 1] = vis ? r.q1.y : 0.f;
        conic_opacity[4 * idx + 2] = vis ? r.q1.z : 0.f; conic_opacity[4 * idx + 3] = vis ? r.q1.w : 0.f;
    }
    if (rgb) { rgb[3 * idx] = vis ? r.q2.x : 0.f; rgb[3 * idx + 1] = vis ? r.q2.y : 0.f; rgb[3 * idx + 2] = vis ? r.q2.z : 0.f; }
}

}  // namespace

int device_sm_count() {
    static std::atomic<int> cache[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev >= 0 && dev < 64) {
        const int c = cache[dev].load(std::memory_order_relaxed);
        if (c > 0) return c;
    }
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    if (dev >= 0 && dev < 64) cache[dev].store(n, std::memory_order_relaxed);
    return n;
}

int bin_ctas() { return bin_cta_count(); }

template <bool SCATTER, bool BATCH>
static cudaError_t launch_bin_pass(int P, int views, const uint4* binrec, int grid_x, int grid_y,
                                   uint32_t* matrix, const uint32_t* tile_offset, uint64_t* keys, cudaStream_t stream) {
    if (P <= 0) return cudaSuccess;
    const int num_tiles = grid_x * grid_y;
    const int ctas = bin_cta_count();
    int chunk = (P + ctas - 1) / ctas;
    chunk = (chunk + 31) & ~31;
    const size_t smem = (size_t)num_tiles * sizeof(uint32_t);
    const dim3 grid(ctas, BATCH ? views : 1);
    if (smem <= BIN_SMEM_LIMIT) {
        const auto k = BATCH ? bin_pass_batch_kernel<SCATTER, true> : bin_pass_kernel<SCATTER, true>;
        static PerDeviceOnce once;
        cudaError_t e = ensure_dynamic_smem(k, (int)BIN_SMEM_LIMIT, once);
        if (e != cudaSuccess) return e;
        k<<<grid, BIN_THREADS, smem, stream>>>(P, chunk, binrec, grid_x, num_tiles, matrix, tile_offset, keys);
    } else {
        const auto k = BATCH ? bin_pass_batch_kernel<SCATTER, false> : bin_pass_kernel<SCATTER, false>;
        k<<<grid, BIN_THREADS, 0, stream>>>(P, chunk, binrec, grid_x, num_tiles, matrix, tile_offset, keys);
    }
    return cudaGetLastError();
}

cudaError_t launch_bin_count(int P, const uint4* binrec, int grid_x, int grid_y, uint32_t* matrix, const ViewBatch& vb,
                             cudaStream_t stream) {
    if (P <= 0)
        return cudaMemsetAsync(matrix, 0, (size_t)bin_cta_count() * vb.B * grid_x * grid_y * sizeof(uint32_t), stream);
    if (vb.scalars) return launch_bin_pass<false, true>(P, vb.B, binrec, grid_x, grid_y, matrix, nullptr, nullptr, stream);
    return launch_bin_pass<false, false>(P, 1, binrec, grid_x, grid_y, matrix, nullptr, nullptr, stream);
}

cudaError_t launch_tile_scan(int num_tiles, uint32_t* matrix, uint32_t* tile_total, uint32_t* tile_offset, uint2* ranges,
                             uint32_t* info, cudaStream_t stream, int capacity, int* status) {
    column_scan_kernel<<<(num_tiles + 31) / 32, 256, 0, stream>>>(num_tiles, bin_cta_count(), matrix, tile_total);
    if (status) tile_scan_cap_kernel<<<1, SCAN_THREADS, 0, stream>>>(num_tiles, tile_total, tile_offset, ranges, info, capacity, status);
    else tile_scan_kernel<<<1, SCAN_THREADS, 0, stream>>>(num_tiles, tile_total, tile_offset, ranges, info);
    return cudaGetLastError();
}

cudaError_t launch_bin_scatter(int P, const uint4* binrec, int grid_x, int grid_y, uint32_t* matrix,
                               const uint32_t* tile_offset, uint64_t* keys, const ViewBatch& vb, cudaStream_t stream,
                               const uint32_t* info) {
    if (info) {
        if (P <= 0) return cudaSuccess;
        const int num_tiles = grid_x * grid_y, ctas = bin_cta_count();
        const int chunk = (((P + ctas - 1) / ctas) + 31) & ~31;
        const size_t smem = (size_t)num_tiles * sizeof(uint32_t);
        const dim3 grid(ctas, vb.B);
        if (smem <= BIN_SMEM_LIMIT) {
            static PerDeviceOnce once;
            cudaError_t e = ensure_dynamic_smem(bin_scatter_cap_kernel<true>, (int)BIN_SMEM_LIMIT, once);
            if (e != cudaSuccess) return e;
            bin_scatter_cap_kernel<true><<<grid, BIN_THREADS, smem, stream>>>(P, chunk, binrec, grid_x, num_tiles, matrix,
                                                                             tile_offset, keys, info);
        } else {
            bin_scatter_cap_kernel<false><<<grid, BIN_THREADS, 0, stream>>>(P, chunk, binrec, grid_x, num_tiles, matrix,
                                                                           tile_offset, keys, info);
        }
        return cudaGetLastError();
    }
    if (vb.scalars) return launch_bin_pass<true, true>(P, vb.B, binrec, grid_x, grid_y, matrix, tile_offset, keys, stream);
    return launch_bin_pass<true, false>(P, 1, binrec, grid_x, grid_y, matrix, tile_offset, keys, stream);
}

int tile_sort_pack_kernel_count(int max_count) { return max_count > SORT_SMALL_KEYS ? 2 : 1; }

template <bool BATCH>
static cudaError_t tile_sort_pack(int num_tiles, int max_count, const uint2* ranges, uint64_t* keys, const InstRec* grec,
                                  StageRec* recs, uint32_t* point_list, int tiles_per_view, int P, cudaStream_t stream) {
    constexpr size_t small_smem = (size_t)(SORT_SMALL_KEYS + SORT_SMALL_KEYS / 8) * sizeof(uint64_t);
    constexpr size_t large_smem = (size_t)(SORT_LARGE_KEYS + SORT_LARGE_KEYS / 16) * sizeof(uint64_t);
    const auto small = BATCH ? tile_sort_batch_kernel<false> : tile_sort_kernel<false>;
    small<<<num_tiles, SORT_SMALL_THREADS, small_smem, stream>>>(ranges, keys, point_list, grec, recs, tiles_per_view, P);
    if (max_count > SORT_SMALL_KEYS) {
        const auto large = BATCH ? tile_sort_batch_kernel<true> : tile_sort_kernel<true>;
        static PerDeviceOnce once;
        cudaError_t e = ensure_dynamic_smem(large, (int)large_smem, once);
        if (e != cudaSuccess) return e;
        large<<<num_tiles, SORT_LARGE_THREADS, large_smem, stream>>>(ranges, keys, point_list, grec, recs, tiles_per_view, P);
    }
    return cudaGetLastError();
}

cudaError_t launch_tile_sort_pack(int num_tiles, int max_count, int R, const uint2* ranges, uint64_t* keys,
                                  const InstRec* grec, int P, StageRec* recs, uint32_t* point_list, const ViewBatch& vb,
                                  cudaStream_t stream) {
    if (num_tiles <= 0 || R <= 0) return cudaSuccess;
    if (vb.scalars)
        return tile_sort_pack<true>(num_tiles, max_count, ranges, keys, grec, recs, point_list, num_tiles / vb.B, P, stream);
    return tile_sort_pack<false>(num_tiles, max_count, ranges, keys, grec, recs, point_list, 0, 0, stream);
}

cudaError_t launch_view_table(int B, int W, int H, const float* timestamps, const float* tan_fovx, const float* tan_fovy,
                              ViewScalars* out, cudaStream_t stream) {
    view_table_kernel<<<(B + 127) / 128, 128, 0, stream>>>(B, W, H, timestamps, tan_fovx, tan_fovy, out);
    return cudaGetLastError();
}

cudaError_t launch_unpack_grec(int P, const InstRec* grec, const int* radii, float* depths, float* means2D,
                               float* conic_opacity, float* rgb, cudaStream_t stream) {
    if (P <= 0) return cudaSuccess;
    unpack_grec_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, grec, radii, depths, means2D, conic_opacity, rgb);
    return cudaGetLastError();
}

}  // namespace fdgs
