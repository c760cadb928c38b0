// fdgs_api.cu -- C-ABI entry points (include/fdgs.h) and scratch-buffer carving.
//
// Host-side orchestration of one forward / backward pass; replaces
// CudaRasterizer::Rasterizer::forward / backward / markVisible
// (reference: rasterizer_impl.cu:199-364, :368-496, :142-154) and the GeometryState /
// ImageState / BinningState chunk carving (rasterizer_impl.cu:156-195, rasterizer_impl.h:21-73).
#include <limits.h>
#include <math.h>
#include <string.h>
#include <atomic>
#include <cstdlib>
#include <mutex>
#include <string>
#include <vector>
#include <nvtx3/nvToolsExt.h>   // header-only NVTX v3: ranges cost nothing unless a profiler is attached
#include "../../include/fdgs.h"
#include "fdgs_internal.h"

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string& msg) {
    g_last_error = msg;
    return code;
}

#define FDGS_CUDA(expr, what)                                                                         \
    do {                                                                                              \
        cudaError_t _e = (expr);                                                                      \
        if (_e != cudaSuccess)                                                                        \
            return fail(FDGS_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(_e));            \
    } while (0)

// ---- measurement hooks (include/fdgs.h: fdgs_profile_*, fdgs_launch_count) -----------------------
struct ProfEvent {
    int stage;
    cudaEvent_t a, b;
};
std::mutex g_prof_mu;
bool g_prof_on = false;
std::vector<ProfEvent> g_prof_events;
constexpr size_t kMaxProfEvents = 4096;
std::atomic<long long> g_kernel_launches{0};
// FDGS_TRACE=1 + debug=true: print every stage to stderr before and after its synchronisation
const bool g_trace = getenv("FDGS_TRACE") != nullptr;

// tile lists: 1 = only the tiles a Gaussian's alpha >= 1/255 footprint reaches, 0 = the reference's 3-sigma square
// (include/fdgs.h: fdgs_set_tile_cull)
std::atomic<int> g_tile_cull{getenv("FDGS_TILE_CULL") ? atoi(getenv("FDGS_TILE_CULL")) : 1};

bool stream_capturing(cudaStream_t s) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    return cudaStreamIsCapturing(s, &st) == cudaSuccess && st != cudaStreamCaptureStatusNone;
}

struct StageTimer {
    cudaEvent_t a = nullptr, b = nullptr;
    int stage;
    cudaStream_t stream;
    StageTimer(int stage_, cudaStream_t s, const char* name) : stage(stage_), stream(s) {
        nvtxRangePushA(name);   // one NVTX range per pipeline stage (nsys / ncu --nvtx)
        // a captured stage would record its events into the graph, not time this call
        if (g_prof_on && !stream_capturing(stream)) {
            cudaEventCreate(&a);
            cudaEventCreate(&b);
            cudaEventRecord(a, stream);
        }
    }
    bool open = true;
    ~StageTimer() {
        if (open) nvtxRangePop();   // error return between start and stop
    }
    void stop(int kernels) {
        nvtxRangePop();
        open = false;
        g_kernel_launches += kernels;
        if (a) {
            cudaEventRecord(b, stream);
            std::lock_guard<std::mutex> lk(g_prof_mu);
            if (g_prof_events.size() < kMaxProfEvents) {
                g_prof_events.push_back({stage, a, b});
            } else {   // nobody is reading (fdgs_profile_read): do not grow without bound
                cudaEventDestroy(a);
                cudaEventDestroy(b);
            }
        }
    }
};

// FDGS_STAGE(stage id, kernels launched, launch expression, name)
#define FDGS_STAGE(sid, nk, expr, what)                                                               \
    do {                                                                                              \
        StageTimer _t(sid, stream, what);                                                                \
        FDGS_CUDA(expr, what);                                                                        \
        _t.stop(nk);                                                                                  \
        if (debug) {                                                                                  \
            if (g_trace) fprintf(stderr, "[fdgs] %s launched, synchronising\n", what);               \
            cudaError_t _s = cudaStreamSynchronize(stream);                                           \
            if (g_trace) fprintf(stderr, "[fdgs] %s done: %s\n", what, cudaGetErrorString(_s));      \
            if (_s != cudaSuccess)                                                                    \
                return fail(FDGS_ERR_CUDA, std::string(what) + " (debug sync): " + cudaGetErrorString(_s)); \
        }                                                                                             \
    } while (0)

// bump allocator over one chunk; every sub-array 128-byte aligned (like the reference's obtain())
struct Carver {
    char* base;
    size_t off;
    explicit Carver(char* b) : base(b), off(0) {}
    template <typename T>
    T* take(size_t count) {
        off = (off + 127) & ~(size_t)127;
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += count * sizeof(T);
        return p;
    }
    size_t total() const { return off + 128; }
};

// batch: the batched entry's layout, [B][P] stacks of every array, then the [B] per-view scalars
struct GeomState {
    float* cov3D;            // [P,6]  (first: exposed as covs3D_com)
    fdgs::InstRec* grec;     // [P]    per-Gaussian 64-byte record
    uint8_t* clamped;        // [P]
    uint32_t* tiles_touched; // [P]
    uint4* binrec;           // [P] tile rectangle + depth bits of every Gaussian, for the binning passes
    fdgs::ViewScalars* scalars;   // [B] (batch only, else NULL)
    size_t bytes;
    static GeomState carve(char* base, int P, bool batch = false, int B = 0) {
        GeomState g;
        Carver c(base);
        const size_t p = (size_t)(P > 0 ? P : 0) * (batch ? (size_t)(B > 0 ? B : 0) : 1);
        g.cov3D = c.take<float>(6 * p);   // first: 128-byte aligned [P,6] view for covs3D_com
        g.grec = c.take<fdgs::InstRec>(p);
        g.clamped = c.take<uint8_t>(p);
        g.tiles_touched = c.take<uint32_t>(p);
        g.binrec = c.take<uint4>(p);
        g.scalars = nullptr;
        if (batch) {
            c.off += 128;   // the view table starts one 128-byte block past the stacks (fdgs_geom_batch_bytes' layout)
            g.scalars = c.take<fdgs::ViewScalars>((size_t)(B > 0 ? B : 0));
        }
        g.bytes = c.total();
        return g;
    }
};

struct ImageState {
    float* final_T;
    uint32_t* n_contrib;
    uint2* ranges;           // [tiles] start/end of every tile's instance list
    uint32_t* bin_matrix;    // [bin_ctas][tiles] per-CTA tile histograms -> column prefixes
    uint32_t* tile_total;    // [tiles]
    uint32_t* tile_offset;   // [tiles]
    uint32_t* bin_info;      // [4] total instances, largest tile, overflow flag, spare
    size_t tiles;
    size_t bytes;
    // views > 1: the batched entry's [views] stacks of every per-pixel and per-tile array (tiles = all views' tiles)
    static ImageState carve(char* base, int W, int H, int views = 1) {
        ImageState s;
        Carver c(base);
        const size_t N = (size_t)W * H * (size_t)views;
        s.tiles = (size_t)((W + fdgs::TILE_X - 1) / fdgs::TILE_X) * ((H + fdgs::TILE_Y - 1) / fdgs::TILE_Y) * (size_t)views;
        s.final_T = c.take<float>(N);
        s.n_contrib = c.take<uint32_t>(N);
        s.ranges = c.take<uint2>(s.tiles);
        s.bin_matrix = c.take<uint32_t>(s.tiles * (size_t)fdgs::bin_ctas());
        s.tile_total = c.take<uint32_t>(s.tiles);
        s.tile_offset = c.take<uint32_t>(s.tiles);
        s.bin_info = c.take<uint32_t>(4);
        s.bytes = c.total();
        return s;
    }
};

struct BinningState {
    fdgs::StageRec* recs;    // [R] instance records in tile-sorted order (80-byte stride, see fdgs_common.cuh)
    uint32_t* point_list;    // [R] sorted Gaussian indices (the reference's point_list)
    uint64_t* keys;          // [R] depth_bits<<32 | index, grouped by tile
    size_t bytes;
    static BinningState carve(char* base, int R) {
        BinningState b;
        Carver c(base);
        const size_t r = (size_t)(R > 0 ? R : 0);
        b.recs = c.take<fdgs::StageRec>(r);
        b.point_list = c.take<uint32_t>(r);
        b.keys = c.take<uint64_t>(r);
        b.bytes = c.total();
        return b;
    }
};

// The batched backward's scratch: per-view gradients before their view sums, and the sh_outer_sum table
struct BatchBwdScratch {
    float* dL_dconic;     // [B,P,4] accumulated by the blend (zeroed by the backward)
    float* dL_dcolor;     // [B,P,3] accumulated
    float* dL_dflows;     // [B,P,2] accumulated
    float* dL_dopacity;   // [B,P]   accumulated
    float* dL_dmean3D;    // [B,P,3]
    float* dL_dcov3D;     // [B,P,6]
    float* dL_dts;        // [B,P]
    float* dL_dscale;     // [B,P,3]
    float* dL_dscale_t;   // [B,P]
    float* dL_drot;       // [B,P,4]
    float* dL_drot_r;     // [B,P,4]
    float* table;         // [B][3P + 4] colour factors + view metadata
    float* dirs;          // [B][P][8]
    size_t zero_bytes;    // the accumulated arrays lead the buffer
    size_t bytes;
    static long long factor_stride(int P) { return 3ll * P + 4; }
    static BatchBwdScratch carve(char* base, int P, int B) {
        BatchBwdScratch s;
        Carver c(base);
        const size_t n = (size_t)(P > 0 ? P : 0) * (size_t)(B > 0 ? B : 0);
        s.dL_dconic = c.take<float>(4 * n);
        s.dL_dcolor = c.take<float>(3 * n);
        s.dL_dflows = c.take<float>(2 * n);
        s.dL_dopacity = c.take<float>(n);
        s.zero_bytes = c.off;
        s.dL_dmean3D = c.take<float>(3 * n);
        s.dL_dcov3D = c.take<float>(6 * n);
        s.dL_dts = c.take<float>(n);
        s.dL_dscale = c.take<float>(3 * n);
        s.dL_dscale_t = c.take<float>(n);
        s.dL_drot = c.take<float>(4 * n);
        s.dL_drot_r = c.take<float>(4 * n);
        s.table = c.take<float>((size_t)factor_stride(P > 0 ? P : 0) * (size_t)(B > 0 ? B : 0));
        s.dirs = c.take<float>(8 * n);
        s.bytes = c.total();
        return s;
    }
};

char* align128(char* p) {
    return reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(p) + 127) & ~(uintptr_t)127);
}

// `whole_blocks`: the forward reads a row in whole 16-coefficient blocks (RowSmem::load_block, 12 float4 each), so
// its staged path needs M % 16 == 0; the backward bounds its accesses by the row length and only needs M % 4 == 0.
void sh_staging(const float* shs, int M, bool whole_blocks, int* bulk_ok, int* stride_floats) {
    *bulk_ok = 0;
    *stride_floats = 0;
    if (!shs || M <= 0) return;
    if ((M % (whole_blocks ? 16 : 4)) != 0 || (reinterpret_cast<uintptr_t>(shs) % 16) != 0) return;
    int q = (3 * M) / 4 + 1;   // 16-byte units incl. padding
    if ((q & 1) == 0) ++q;     // odd stride in 16-byte units -> conflict-free LDS.128 / STS.128
    if ((size_t)q * 16 * 128 > 200 * 1024) return;
    *bulk_ok = 1;
    *stride_floats = q * 4;
}

}  // namespace

extern "C" {

int fdgs_version(void) { return FDGS_VERSION; }

const char* fdgs_last_error(void) { return g_last_error.c_str(); }

size_t fdgs_geom_bytes(int P) { return GeomState::carve(nullptr, P).bytes + 128; }
size_t fdgs_image_bytes(int width, int height) { return ImageState::carve(nullptr, width, height).bytes + 128; }
size_t fdgs_binning_bytes(int num_rendered, int, int) { return BinningState::carve(nullptr, num_rendered).bytes + 128; }
size_t fdgs_geom_batch_bytes(int P, int B) { return GeomState::carve(nullptr, P, true, B).bytes + 128; }
size_t fdgs_image_batch_bytes(int width, int height, int B) {
    return ImageState::carve(nullptr, width, height, B > 0 ? B : 0).bytes + 128;
}
size_t fdgs_backward_batch_scratch_bytes(int P, int B) { return BatchBwdScratch::carve(nullptr, P, B).bytes + 128; }
size_t fdgs_camera_grad_scratch_bytes(int P, int B) {
    return (size_t)fdgs::CAM_TERMS * fdgs::camera_grad_blocks(P) * (size_t)(B > 0 ? B : 0) * sizeof(float) + 128;
}

}  // extern "C"

namespace {

int check_forward_args(const fdgs_forward_args* a) {
    const int P = a->P, W = a->width, H = a->height;
    if (P < 0 || W <= 0 || H <= 0) return fail(FDGS_ERR_INVALID_ARG, "bad P / width / height");
    // the blend kernel writes every pixel of every image even when nothing is rendered (P == 0: background only)
    if (!a->out_color || !a->out_flow || !a->out_depth || !a->out_T || !a->background)
        return fail(FDGS_ERR_INVALID_ARG, "background and the output images must be set");
    if (P > 0) {
        if (!a->means3D || !a->opacities || !a->viewmatrix || !a->projmatrix || !a->cam_pos)
            return fail(FDGS_ERR_INVALID_ARG, "means3D/opacities/viewmatrix/projmatrix/cam_pos must be set");
        if (!a->out_means3D || !a->out_color || !a->out_flow || !a->out_depth || !a->out_T || !a->radii)
            return fail(FDGS_ERR_INVALID_ARG, "output pointers must be set");
        if (!a->cov3D_precomp) {
            if (!a->scales || !a->rotations) return fail(FDGS_ERR_INVALID_ARG, "scales/rotations or cov3D_precomp required");
            if (a->rot_4d && (!a->rotations_r || !a->scales_t || !a->ts))
                return fail(FDGS_ERR_INVALID_ARG, "rot_4d needs rotations_r, scales_t and ts");
            if (!a->rot_4d && a->gaussian_dim == 4 && (!a->scales_t || !a->ts))
                return fail(FDGS_ERR_INVALID_ARG, "gaussian_dim 4 needs scales_t and ts");
        }
        if (!a->colors_precomp) {
            // reference: rasterizer_impl.cu:255-258 (NUM_CHANNELS is 3 here, so SHs are required)
            if (!a->shs) return fail(FDGS_ERR_INVALID_ARG, "either shs or colors_precomp required");
            const bool sh3d = a->gaussian_dim == 3 || a->force_sh_3d;
            int need = (a->D + 1) * (a->D + 1);
            if (!sh3d && a->D > 2 && a->D_t > 0) need = 16 * (a->D_t + 1);
            if (a->D < 0 || a->D > 3 || a->D_t < 0 || a->D_t > 2 || a->M < need)
                return fail(FDGS_ERR_INVALID_ARG, "SH degree / coefficient count mismatch");
            if (!sh3d && !a->ts) return fail(FDGS_ERR_INVALID_ARG, "4D SH needs ts");
        }
    }
    const int grid_x = (W + fdgs::TILE_X - 1) / fdgs::TILE_X, grid_y = (H + fdgs::TILE_Y - 1) / fdgs::TILE_Y;
    // tile coordinates travel as 16-bit fields of the per-Gaussian bin record (preprocess_fwd.cu / binning.cu)
    if (grid_x > 65535 || grid_y > 65535) return fail(FDGS_ERR_UNSUPPORTED, "image larger than 1048560 pixels on a side");
    if (P > 0 && a->shs_rest && !a->colors_precomp && a->M < 2) return fail(FDGS_ERR_INVALID_ARG, "split SH rows need M >= 2");
    if (P > 0 && a->raw_params && a->cov3D_precomp)
        return fail(FDGS_ERR_INVALID_ARG, "raw_params needs scales / rotations, not cov3D_precomp");
    return FDGS_OK;
}

// The capacity entry's sizing (fdgs_forward_batch_capacity): the binning buffer holds `capacity` instances and the
// device status word reports the true count
struct CapacityMode {
    int capacity;
    int* status;
};

// The forward's stages on the carved geometry and image buffers, for one view (vb = {1, NULL}) or for the batched
// entry's B views (vb = {B, the view table}: every per-view array is then a [B] stack, and the camera tables and
// scalars are the views').  Allocates the binning buffer after the one host synchronisation, or, with cap (a batch), at
// cap->capacity instances before the first launch, and then does not synchronise.
// zero_sh / zero_sh_rest (single view): the SH gradient rows the blend zeroes (fdgs_forward_zero_sh), or NULL.
int forward_stages(const fdgs_forward_args* a, const float* bg_image, float* zero_sh, float* zero_sh_rest,
                   const fdgs::ViewBatch& vb, const GeomState& geom, const ImageState& img, fdgs_alloc_fn binning_alloc,
                   void* binning_ctx, cudaStream_t stream, fdgs_forward_result* res, const CapacityMode* cap = nullptr) {
    const bool debug = a->debug != 0, batch = vb.scalars != nullptr;
    const int P = a->P, W = a->width, H = a->height;
    const int grid_x = (W + fdgs::TILE_X - 1) / fdgs::TILE_X, grid_y = (H + fdgs::TILE_Y - 1) / fdgs::TILE_Y;
    BinningState bin;
    auto alloc_binning = [&](int R) {
        const size_t bin_bytes = fdgs_binning_bytes(R, W, H);
        char* bin_raw = binning_alloc(binning_ctx, bin_bytes);
        if (!bin_raw) return fail(FDGS_ERR_ALLOC, "binning buffer allocation failed");
        bin = BinningState::carve(align128(bin_raw), R);
        res->binning_buffer = bin_raw;
        res->binning_bytes = bin_bytes;
        res->num_rendered = R;
        return (int)FDGS_OK;
    };
    if (cap)
        if (int rc = alloc_binning(cap->capacity)) return rc;
    if (P > 0) {
        fdgs::PreprocessFwdParams pp;
        memset(&pp, 0, sizeof(pp));
        pp.P = P; pp.D = a->D; pp.D_t = a->D_t; pp.M = a->M;
        pp.means3D = a->means3D; pp.ts = a->ts; pp.scales = a->scales; pp.scales_t = a->scales_t;
        pp.scale_modifier = a->scale_modifier; pp.rotations = a->rotations; pp.rotations_r = a->rotations_r;
        pp.opacities = a->opacities; pp.shs = a->shs; pp.cov3D_precomp = a->cov3D_precomp;
        pp.prefilter_var = a->prefilter_var; pp.colors_precomp = a->colors_precomp;
        pp.viewmatrix = a->viewmatrix; pp.projmatrix = a->projmatrix; pp.cam_pos = a->cam_pos;
        pp.timestamp = a->timestamp; pp.time_duration = a->time_duration;
        pp.rot_4d = a->rot_4d; pp.gaussian_dim = a->gaussian_dim; pp.force_sh_3d = a->force_sh_3d;
        pp.W = W; pp.H = H; pp.tan_fovx = a->tan_fovx; pp.tan_fovy = a->tan_fovy;
        // reference: rasterizer_impl.cu:235-236
        pp.focal_y = H / (2.0f * a->tan_fovy);
        pp.focal_x = W / (2.0f * a->tan_fovx);
        pp.grid_x = grid_x; pp.grid_y = grid_y; pp.prefiltered = a->prefiltered;
        sh_staging(a->colors_precomp ? nullptr : a->shs, a->M, true, &pp.sh_bulk_ok, &pp.sh_row_stride_floats);
        pp.raw_params = a->raw_params;
        pp.shs_rest = a->colors_precomp ? nullptr : a->shs_rest;
        pp.flows = a->flows_precomp;
        pp.out_means3D = a->out_means3D; pp.radii = a->radii; pp.cov3D = geom.cov3D; pp.grec = geom.grec;
        pp.clamped = geom.clamped; pp.tiles_touched = geom.tiles_touched; pp.binrec = geom.binrec;
        pp.tile_cull = g_tile_cull.load();
        pp.vb = vb;
        FDGS_STAGE(0, 1, fdgs::launch_preprocess_fwd(pp, stream), batch ? "preprocess_fwd (batch)" : "preprocess_fwd");
    }
    // binning: per-tile counts, offsets, ranges and the total instance count R
    FDGS_STAGE(1, (P > 0 ? 1 : 0) + 2,
               [&]() {
                   cudaError_t e = fdgs::launch_bin_count(P, geom.binrec, grid_x, grid_y, img.bin_matrix, vb, stream);
                   if (e != cudaSuccess) return e;
                   return fdgs::launch_tile_scan((int)img.tiles, img.bin_matrix, img.tile_total, img.tile_offset, img.ranges,
                                                 img.bin_info, stream, cap ? cap->capacity : 0, cap ? cap->status : nullptr);
               }(),
               batch ? "bin_count + tile_scan (batch)" : "bin_count + tile_scan");
    int num_rendered = 0, max_count = 0;
    if (cap) {
        // sized by the capacity: an overflow is handled on the device (no key written, every range empty), and only
        // the device knows the largest tile, so both size classes of the tile sort run
        num_rendered = cap->capacity;
        max_count = INT_MAX;
    } else {
        // the one host synchronisation of the forward (reference: rasterizer_impl.cu:302): R over all views, the largest
        // tile of any view, the overflow flag
        int bin_info[4] = {0, 0, 0, 0};
        FDGS_CUDA(cudaMemcpyAsync(bin_info, img.bin_info, sizeof(bin_info), cudaMemcpyDeviceToHost, stream), "num_rendered copy");
        FDGS_CUDA(cudaStreamSynchronize(stream), "num_rendered sync");
        num_rendered = bin_info[0];
        max_count = bin_info[1];
        // bin_info[2]: the 64-bit total computed on the device exceeded 2^31 - 1 (a wrapped 32-bit total would look valid)
        if (num_rendered < 0 || bin_info[2] != 0) return fail(FDGS_ERR_UNSUPPORTED, "more than 2^31 - 1 tile instances");
        if (int rc = alloc_binning(num_rendered)) return rc;
    }

    if (num_rendered > 0) {
        FDGS_STAGE(2, 1,
                   fdgs::launch_bin_scatter(P, geom.binrec, grid_x, grid_y, img.bin_matrix, img.tile_offset, bin.keys, vb,
                                            stream, cap ? img.bin_info : nullptr),
                   batch ? "bin_scatter (batch)" : "bin_scatter");
        FDGS_STAGE(3, fdgs::tile_sort_pack_kernel_count(max_count),
                   fdgs::launch_tile_sort_pack((int)img.tiles, max_count, num_rendered, img.ranges, bin.keys, geom.grec, P,
                                               bin.recs, bin.point_list, vb, stream),
                   batch ? "tile_sort_pack (batch)" : "tile_sort_pack");
    }
    fdgs::BlendFwdParams bp;
    bp.W = W; bp.H = H; bp.grid_x = grid_x; bp.grid_y = grid_y;
    bp.ranges = img.ranges; bp.recs = bin.recs; bp.background = a->background;
    bp.final_T = img.final_T; bp.n_contrib = img.n_contrib;
    bp.out_color = a->out_color; bp.out_flow = a->out_flow; bp.out_depth = a->out_depth; bp.out_T = a->out_T;
    bp.bg_image = bg_image;
    bp.views = batch ? vb.B : 0;
    bp.zero_rows[0] = bp.zero_rows[1] = nullptr;
    bp.zero_row_floats[0] = bp.zero_row_floats[1] = 0;
    bp.zero_stripe = 0; bp.P = P; bp.radii = a->radii; bp.tiles_touched = geom.tiles_touched;
    if (zero_sh && P > 0) {
        const bool split = zero_sh_rest != nullptr;
        bp.zero_rows[0] = zero_sh; bp.zero_row_floats[0] = split ? 3 : 3 * a->M;
        bp.zero_rows[1] = zero_sh_rest; bp.zero_row_floats[1] = split ? 3 * (a->M - 1) : 0;
        const long long tiles = (long long)grid_x * grid_y;
        bp.zero_stripe = (int)((P + tiles - 1) / tiles);
    }
    FDGS_STAGE(5, 1, fdgs::launch_blend_fwd(bp, stream), batch ? "blend_fwd (batch)" : "blend_fwd");
    return FDGS_OK;
}

int forward_impl(const fdgs_forward_args* a, const float* bg_image, float* zero_sh, float* zero_sh_rest,
                 fdgs_alloc_fn geom_alloc, void* geom_ctx, fdgs_alloc_fn binning_alloc, void* binning_ctx,
                 fdgs_alloc_fn image_alloc, void* image_ctx, void* stream_v, fdgs_forward_result* res) {
    g_last_error.clear();
    if (!a || !res || !geom_alloc || !binning_alloc || !image_alloc) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    memset(res, 0, sizeof(*res));
    const int P = a->P, W = a->width, H = a->height;
    if (int rc = check_forward_args(a)) return rc;
    if (zero_sh_rest && !zero_sh) return fail(FDGS_ERR_INVALID_ARG, "dL_dsh_rest without dL_dsh");
    if (zero_sh && P > 0) {
        if (!a->shs || a->colors_precomp || a->M <= 0) return fail(FDGS_ERR_INVALID_ARG, "dL_dsh rows need shs, not colors_precomp");
        if (a->shs_rest && !zero_sh_rest) return fail(FDGS_ERR_INVALID_ARG, "split SH rows need dL_dsh_rest");
        if (!a->shs_rest && zero_sh_rest) return fail(FDGS_ERR_INVALID_ARG, "dL_dsh_rest without shs_rest");
    }

    // scratch: geometry + image
    const size_t geom_bytes = fdgs_geom_bytes(P);
    char* geom_raw = geom_alloc(geom_ctx, geom_bytes);
    if (!geom_raw) return fail(FDGS_ERR_ALLOC, "geometry buffer allocation failed");
    GeomState geom = GeomState::carve(align128(geom_raw), P);
    const size_t img_bytes = fdgs_image_bytes(W, H);
    char* img_raw = image_alloc(image_ctx, img_bytes);
    if (!img_raw) return fail(FDGS_ERR_ALLOC, "image buffer allocation failed");
    ImageState img = ImageState::carve(align128(img_raw), W, H);
    res->geom_buffer = geom_raw;
    res->geom_bytes = geom_bytes;
    res->image_buffer = img_raw;
    res->image_bytes = img_bytes;
    res->cov3D = geom.cov3D;
    return forward_stages(a, bg_image, zero_sh, zero_sh_rest, {1, nullptr}, geom, img, binning_alloc, binning_ctx,
                          reinterpret_cast<cudaStream_t>(stream_v), res);
}

// The camera gradient of `views` views with no Gaussian: zeros (fdgs_backward_camera)
int camera_grad_zero(const fdgs::CameraGradParams& cam, int views, bool debug, cudaStream_t stream) {
    FDGS_STAGE(7, 1, fdgs::launch_camera_grad_finish(cam, 0, views, stream), "camera_grad (no Gaussian)");
    return FDGS_OK;
}

// The camera outputs of fdgs_backward_camera / fdgs_backward_batch_camera, checked before anything is launched
int camera_grad_params(const fdgs_camera_grad_out* c, fdgs::CameraGradParams* p) {
    if (!c || !c->dL_dviewmatrix || !c->dL_dprojmatrix || !c->dL_dcampos || !c->scratch)
        return fail(FDGS_ERR_INVALID_ARG, "camera gradient outputs (dL_dviewmatrix / dL_dprojmatrix / dL_dcampos) and scratch required");
    p->partials = reinterpret_cast<float*>(align128(c->scratch));
    p->dL_dviewmatrix = c->dL_dviewmatrix; p->dL_dprojmatrix = c->dL_dprojmatrix; p->dL_dcampos = c->dL_dcampos;
    return FDGS_OK;
}

// The backward's stages on the forward's buffers: the blend backward (when there is an instance or dL_dbg_image to
// write), then the per-Gaussian backward (when there is a Gaussian).  vb as in forward_stages; for a batch, a's
// gradient outputs are the per-view stacks of BatchBwdScratch.  sh_rows_zeroed: the forward zeroed the non-rendered
// dL_dsh rows (fdgs_backward_zero_sh).  cam: also the camera gradient (fdgs_backward_camera), or NULL.  The arguments
// have been checked by the entry.
int backward_stages(const fdgs_backward_args* a, const float* bg_image, float* dL_dbg_image, int sh_rows_zeroed,
                    const fdgs::ViewBatch& vb, const GeomState& geom, const ImageState& img, cudaStream_t stream,
                    const fdgs::CameraGradParams* cam = nullptr) {
    const bool debug = a->debug != 0, batch = vb.scalars != nullptr;
    const int P = a->P, W = a->width, H = a->height, R = a->R;
    BinningState bin = BinningState::carve(a->binning_buffer ? align128(const_cast<char*>(a->binning_buffer)) : nullptr, R);

    // with no instance at all the blend only has dL_dbg_image to write (P == 0: the background image takes the whole
    // colour gradient, from empty tile lists)
    if ((P > 0 && R > 0) || dL_dbg_image) {
        fdgs::BlendBwdParams bp;
        bp.W = W; bp.H = H; bp.grid_x = (W + fdgs::TILE_X - 1) / fdgs::TILE_X; bp.grid_y = (H + fdgs::TILE_Y - 1) / fdgs::TILE_Y;
        bp.ranges = img.ranges; bp.recs = bin.recs; bp.background = a->background;
        bp.final_T = img.final_T; bp.n_contrib = img.n_contrib;
        bp.dL_dpix = a->dL_dpix; bp.dL_depths = a->dL_depths; bp.dL_masks = a->dL_masks; bp.dL_dpix_flow = a->dL_dpix_flow;
        bp.dL_dmean2D = a->dL_dmean2D; bp.dL_dconic = a->dL_dconic; bp.dL_dopacity = a->dL_dopacity;
        bp.dL_dcolor = a->dL_dcolor; bp.dL_dflows = a->dL_dflows;
        bp.bg_image = bg_image; bp.dL_dbg_image = dL_dbg_image;
        bp.views = batch ? vb.B : 0; bp.P = P;
        FDGS_STAGE(6, 1, fdgs::launch_blend_bwd(bp, stream), batch ? "blend_bwd (batch)" : "blend_bwd");
    }
    if (P <= 0) return cam ? camera_grad_zero(*cam, batch ? vb.B : 1, debug, stream) : FDGS_OK;
    fdgs::PreprocessBwdParams pb;
    memset(&pb, 0, sizeof(pb));
    pb.P = P; pb.D = a->D; pb.D_t = a->D_t; pb.M = a->M;
    pb.means3D = a->out_means3D; pb.radii = a->radii; pb.shs = a->shs; pb.ts = a->ts; pb.opacities = a->opacities;
    pb.clamped = geom.clamped; pb.tiles_touched = geom.tiles_touched;
    pb.scales = a->scales; pb.scales_t = a->scales_t; pb.rotations = a->rotations; pb.rotations_r = a->rotations_r;
    pb.scale_modifier = a->scale_modifier;
    pb.cov3D = a->cov3D_precomp ? a->cov3D_precomp : geom.cov3D;
    pb.prefilter_var = a->prefilter_var; pb.viewmatrix = a->viewmatrix; pb.projmatrix = a->projmatrix;
    pb.focal_y = H / (2.0f * a->tan_fovy);
    pb.focal_x = W / (2.0f * a->tan_fovx);
    pb.tan_fovx = a->tan_fovx; pb.tan_fovy = a->tan_fovy; pb.campos = a->campos;
    pb.timestamp = a->timestamp; pb.time_duration = a->time_duration;
    pb.rot_4d = a->rot_4d; pb.gaussian_dim = a->gaussian_dim; pb.force_sh_3d = a->force_sh_3d;
    pb.has_scales = (a->scales != nullptr) ? 1 : 0;
    pb.grec = geom.grec; pb.W = W; pb.H = H;
    sh_staging(a->shs, a->M, false, &pb.sh_bulk_ok, &pb.sh_row_stride_floats);
    if (a->dL_dsh && (reinterpret_cast<uintptr_t>(a->dL_dsh) % 16) != 0) pb.sh_bulk_ok = 0;
    pb.raw_params = a->raw_params;
    pb.shs_rest = a->shs ? a->shs_rest : nullptr; pb.dL_dsh_rest = a->dL_dsh_rest;
    pb.dL_dmean2D = a->dL_dmean2D; pb.dL_dconic = a->dL_dconic; pb.dL_dopacity = a->dL_dopacity; pb.dL_dcolor = a->dL_dcolor;
    pb.dL_dmean3D = a->dL_dmean3D; pb.dL_dcov3D = a->dL_dcov3D; pb.dL_dsh = a->dL_dsh; pb.sh_factors = a->sh_factors;
    pb.sh_rows_zeroed = (sh_rows_zeroed && a->dL_dsh && !batch) ? 1 : 0;
    pb.dL_dts = a->dL_dts;
    pb.dL_dscale = a->dL_dscale; pb.dL_dscale_t = a->dL_dscale_t; pb.dL_drot = a->dL_drot; pb.dL_drot_r = a->dL_drot_r;
    pb.vb = vb; pb.factor_stride = BatchBwdScratch::factor_stride(P);
    FDGS_STAGE(7, fdgs::preprocess_bwd_kernel_count(pb) + (cam ? 1 : 0), fdgs::launch_preprocess_bwd(pb, stream, cam),
               batch ? "preprocess_bwd (batch)" : "preprocess_bwd");
    return FDGS_OK;
}

int backward_impl(const fdgs_backward_args* a, const float* bg_image, float* dL_dbg_image, int sh_rows_zeroed,
                  void* stream_v, const fdgs::CameraGradParams* cam = nullptr) {
    g_last_error.clear();
    if (!a) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    const int P = a->P, W = a->width, H = a->height, R = a->R;
    if (P <= 0 && !dL_dbg_image)
        return cam ? camera_grad_zero(*cam, 1, a->debug != 0, reinterpret_cast<cudaStream_t>(stream_v)) : FDGS_OK;
    if (W <= 0 || H <= 0 || R < 0) return fail(FDGS_ERR_INVALID_ARG, "bad width / height / R");
    if (P <= 0) {
        if (!a->image_buffer || !a->dL_dpix || !a->background)
            return fail(FDGS_ERR_INVALID_ARG, "image buffer / colour image gradient / background required");
    } else {
        if (!a->geom_buffer || !a->image_buffer || (R > 0 && !a->binning_buffer))
            return fail(FDGS_ERR_INVALID_ARG, "scratch buffers of the forward pass required");
        // dL_depths / dL_masks / dL_dpix_flow may be NULL: no upstream gradient for that image
        if (!a->dL_dpix) return fail(FDGS_ERR_INVALID_ARG, "colour image gradient required");
        if (!a->background || !a->radii || !a->out_means3D || !a->viewmatrix || !a->projmatrix || !a->campos)
            return fail(FDGS_ERR_INVALID_ARG, "background / radii / out_means3D / viewmatrix / projmatrix / campos required");
        if (a->sh_factors && a->dL_dsh) return fail(FDGS_ERR_INVALID_ARG, "sh_factors and dL_dsh are mutually exclusive");
        if (!a->dL_dmean2D || !a->dL_dconic || !a->dL_dopacity || !a->dL_dcolor || !a->dL_dflows || !a->dL_dmean3D ||
            !a->dL_dcov3D || !a->dL_dts || !a->dL_dscale || !a->dL_dscale_t || !a->dL_drot || !a->dL_drot_r)
            return fail(FDGS_ERR_INVALID_ARG, "gradient outputs required");
        const bool split = a->shs && a->shs_rest;   // split SH rows are read only with shs
        if (split && a->dL_dsh && !a->dL_dsh_rest) return fail(FDGS_ERR_INVALID_ARG, "split SH rows need dL_dsh_rest");
        if (!split && a->dL_dsh_rest) return fail(FDGS_ERR_INVALID_ARG, "dL_dsh_rest without shs_rest");
        if (a->scales && a->rot_4d && (!a->rotations_r || !a->scales_t || !a->ts || !a->opacities))
            return fail(FDGS_ERR_INVALID_ARG, "rot_4d backward needs rotations_r, scales_t, ts, opacities");
    }
    GeomState geom = GeomState::carve(align128(const_cast<char*>(a->geom_buffer)), P);
    ImageState img = ImageState::carve(align128(const_cast<char*>(a->image_buffer)), W, H);
    return backward_stages(a, bg_image, dL_dbg_image, sh_rows_zeroed, {1, nullptr}, geom, img,
                           reinterpret_cast<cudaStream_t>(stream_v), cam);
}

// ---- batched views: B cameras of the same Gaussians in one pass per stage (include/fdgs.h: fdgs_forward_batch) -------
constexpr int kMaxViews = 65535;   // views run along gridDim.y / gridDim.z

int check_batch_views(int B, const float* bg_image, int bg_views) {
    if (B < 1 || B > kMaxViews) return fail(FDGS_ERR_INVALID_ARG, "bad view count B (1 <= B <= 65535)");
    if (bg_image && bg_views != B) return fail(FDGS_ERR_INVALID_ARG, "bg_image view count does not match B");
    return FDGS_OK;
}

// cap: the capacity entry's arguments (b is then &cap->batch), or NULL for fdgs_forward_batch
int forward_batch_impl(const fdgs_forward_batch_args* b, const fdgs_forward_capacity_args* cap, fdgs_alloc_fn geom_alloc,
                       void* geom_ctx, fdgs_alloc_fn binning_alloc, void* binning_ctx, fdgs_alloc_fn image_alloc, void* image_ctx,
                       void* stream_v, fdgs_forward_result* res) {
    g_last_error.clear();
    if (!b || !res || !geom_alloc || !binning_alloc || !image_alloc) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    memset(res, 0, sizeof(*res));
    const fdgs_forward_args* a = &b->view;
    const int B = b->B;
    if (cap) {
        if (!cap->status) return fail(FDGS_ERR_INVALID_ARG, "the device status word must be set");
        if (cap->capacity < 0) return fail(FDGS_ERR_INVALID_ARG, "capacity must be >= 0");
    }
    if (int rc = check_batch_views(B, b->bg_image, b->bg_views)) return rc;
    // the capacity entry takes the per-view scalars from device arrays, fdgs_forward_batch from host arrays
    const bool have_scalars = cap ? (cap->timestamps && cap->tan_fovx && cap->tan_fovy)
                                  : (b->timestamps && b->tan_fovx && b->tan_fovy);
    if (!a->viewmatrix || !a->projmatrix || !a->cam_pos || !have_scalars)
        return fail(FDGS_ERR_INVALID_ARG, "the per-view camera table (viewmatrix / projmatrix / cam_pos / timestamps / tan_fovx / "
                                          "tan_fovy) must be set");
    if (int rc = check_forward_args(a)) return rc;
    if (a->P > 0 && (a->colors_precomp || a->cov3D_precomp))
        return fail(FDGS_ERR_INVALID_ARG, "the batched entry takes SH and scales / rotations, not precomputed colours or covariances");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    const int P = a->P, W = a->width, H = a->height;
    const int grid_x = (W + fdgs::TILE_X - 1) / fdgs::TILE_X, grid_y = (H + fdgs::TILE_Y - 1) / fdgs::TILE_Y;
    if ((long long)grid_x * grid_y * B > 0x7fffffffLL || (long long)P * B > 0x7fffffffLL)
        return fail(FDGS_ERR_UNSUPPORTED, "B * tiles or B * P exceeds 2^31 - 1");
    if (cap && a->debug) {
        cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
        FDGS_CUDA(cudaStreamIsCapturing(stream, &st), "capture status query");
        if (st != cudaStreamCaptureStatusNone)
            return fail(FDGS_ERR_INVALID_ARG, "debug synchronises after every stage: not allowed while the stream is capturing");
    }

    const size_t geom_bytes = fdgs_geom_batch_bytes(P, B);
    char* geom_raw = geom_alloc(geom_ctx, geom_bytes);
    if (!geom_raw) return fail(FDGS_ERR_ALLOC, "geometry buffer allocation failed");
    GeomState geom = GeomState::carve(align128(geom_raw), P, true, B);
    const size_t img_bytes = fdgs_image_batch_bytes(W, H, B);
    char* img_raw = image_alloc(image_ctx, img_bytes);
    if (!img_raw) return fail(FDGS_ERR_ALLOC, "image buffer allocation failed");
    ImageState img = ImageState::carve(align128(img_raw), W, H, B);
    res->geom_buffer = geom_raw;
    res->geom_bytes = geom_bytes;
    res->image_buffer = img_raw;
    res->image_bytes = img_bytes;
    res->cov3D = geom.cov3D;

    if (cap) {
        const CapacityMode mode = {cap->capacity, cap->status};
        FDGS_CUDA(fdgs::launch_view_table(B, W, H, cap->timestamps, cap->tan_fovx, cap->tan_fovy, geom.scalars, stream),
                  "view table");
        g_kernel_launches += 1;
        return forward_stages(a, b->bg_image, nullptr, nullptr, {B, geom.scalars}, geom, img, binning_alloc, binning_ctx, stream,
                              res, &mode);
    }
    // the per-view scalars, focal lengths computed as the single-view entry computes them (reference: rasterizer_impl.cu:235-236);
    // a pageable host-to-device copy is staged before the call returns and does not synchronise
    std::vector<fdgs::ViewScalars> vs((size_t)B);
    for (int v = 0; v < B; ++v) {
        memset(&vs[v], 0, sizeof(vs[v]));
        vs[v].timestamp = b->timestamps[v];
        vs[v].tan_fovx = b->tan_fovx[v];
        vs[v].tan_fovy = b->tan_fovy[v];
        vs[v].focal_y = H / (2.0f * b->tan_fovy[v]);
        vs[v].focal_x = W / (2.0f * b->tan_fovx[v]);
    }
    FDGS_CUDA(cudaMemcpyAsync(geom.scalars, vs.data(), vs.size() * sizeof(vs[0]), cudaMemcpyHostToDevice, stream), "view table copy");
    return forward_stages(a, b->bg_image, nullptr, nullptr, {B, geom.scalars}, geom, img, binning_alloc, binning_ctx, stream,
                          res);
}

int backward_batch_impl(const fdgs_backward_batch_args* b, void* stream_v, const fdgs::CameraGradParams* cam = nullptr) {
    g_last_error.clear();
    if (!b) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    const fdgs_backward_args* a = &b->view;
    const int B = b->B;
    if (int rc = check_batch_views(B, b->bg_image, b->bg_views)) return rc;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    const bool debug = a->debug != 0;
    const int P = a->P, W = a->width, H = a->height, R = a->R;
    if (P < 0 || W <= 0 || H <= 0 || R < 0) return fail(FDGS_ERR_INVALID_ARG, "bad P / width / height / R");
    if (!a->image_buffer || !a->geom_buffer || !a->dL_dpix || !a->background)
        return fail(FDGS_ERR_INVALID_ARG, "scratch buffers of the forward pass / colour image gradient / background required");
    const int grid_x = (W + fdgs::TILE_X - 1) / fdgs::TILE_X, grid_y = (H + fdgs::TILE_Y - 1) / fdgs::TILE_Y;
    if ((long long)grid_x * grid_y * B > 0x7fffffffLL || (long long)P * B > 0x7fffffffLL)
        return fail(FDGS_ERR_UNSUPPORTED, "B * tiles or B * P exceeds 2^31 - 1");
    GeomState geom = GeomState::carve(align128(const_cast<char*>(a->geom_buffer)), P, true, B);
    ImageState img = ImageState::carve(align128(const_cast<char*>(a->image_buffer)), W, H, B);
    const fdgs::ViewBatch vb = {B, geom.scalars};
    if (P == 0) return backward_stages(a, b->bg_image, b->dL_dbg_image, 0, vb, geom, img, stream, cam);
    if (R > 0 && !a->binning_buffer) return fail(FDGS_ERR_INVALID_ARG, "scratch buffers of the forward pass required");
    if (!a->radii || !a->out_means3D || !a->viewmatrix || !a->projmatrix || !a->campos)
        return fail(FDGS_ERR_INVALID_ARG, "radii / out_means3D / viewmatrix / projmatrix / campos required");
    if (!a->shs || a->M <= 0 || a->colors_precomp || a->cov3D_precomp || !a->scales || !a->rotations)
        return fail(FDGS_ERR_INVALID_ARG, "the batched entry takes SH and scales / rotations, not precomputed colours or covariances");
    if (a->rot_4d && (!a->rotations_r || !a->scales_t || !a->ts || !a->opacities))
        return fail(FDGS_ERR_INVALID_ARG, "rot_4d backward needs rotations_r, scales_t, ts, opacities");
    if (!a->dL_dmean2D || !a->dL_dopacity || !a->dL_dmean3D || !a->dL_dsh || !a->dL_dts || !a->dL_dscale || !a->dL_dscale_t ||
        !a->dL_drot || !a->dL_drot_r || !b->scratch)
        return fail(FDGS_ERR_INVALID_ARG, "gradient outputs and scratch required");
    if (a->shs_rest && !a->dL_dsh_rest) return fail(FDGS_ERR_INVALID_ARG, "split SH rows need dL_dsh_rest");
    if (!a->shs_rest && a->dL_dsh_rest) return fail(FDGS_ERR_INVALID_ARG, "dL_dsh_rest without shs_rest");

    BatchBwdScratch sc = BatchBwdScratch::carve(align128(b->scratch), P, B);
    FDGS_CUDA(cudaMemsetAsync(sc.dL_dconic, 0, sc.zero_bytes, stream), "zero the accumulated gradients");
    // the stages write every view's gradients into the scratch stacks and its colour factors into the sh_outer_sum table;
    // dL_dmean2D stays the caller's [B,P,3]
    fdgs_backward_args views = *a;
    views.dL_dconic = sc.dL_dconic; views.dL_dopacity = sc.dL_dopacity; views.dL_dcolor = sc.dL_dcolor;
    views.dL_dflows = sc.dL_dflows; views.dL_dmean3D = sc.dL_dmean3D; views.dL_dcov3D = sc.dL_dcov3D;
    views.dL_dsh = nullptr; views.sh_factors = sc.table; views.dL_dsh_rest = nullptr; views.dL_dts = sc.dL_dts;
    views.dL_dscale = sc.dL_dscale; views.dL_dscale_t = sc.dL_dscale_t; views.dL_drot = sc.dL_drot;
    views.dL_drot_r = sc.dL_drot_r;
    if (int rc = backward_stages(&views, b->bg_image, b->dL_dbg_image, 0, vb, geom, img, stream, cam)) return rc;

    // every per-Gaussian gradient but the SH rows: summed over the views in view order
    fdgs::ViewSumParams vsum;
    memset(&vsum, 0, sizeof(vsum));
    vsum.B = B;
    const struct { const float* src; float* dst; int width; } sums[] = {
        {sc.dL_dmean3D, a->dL_dmean3D, 3}, {sc.dL_dopacity, a->dL_dopacity, 1}, {sc.dL_dts, a->dL_dts, 1},
        {sc.dL_dscale, a->dL_dscale, 3},   {sc.dL_dscale_t, a->dL_dscale_t, 1}, {sc.dL_drot, a->dL_drot, 4},
        {sc.dL_drot_r, a->dL_drot_r, 4}};
    for (const auto& t : sums) {
        vsum.src[vsum.n] = t.src;
        vsum.dst[vsum.n] = t.dst;
        vsum.count[vsum.n] = (long long)t.width * P;
        ++vsum.n;
    }
    FDGS_STAGE(7, 1, fdgs::launch_view_sum(vsum, stream), "view_sum (batch)");

    // the SH rows: the views' rank-one rows summed straight into dL_dsh (| dL_dsh_rest), every row (K = P)
    fdgs::ShSumParams sp;
    memset(&sp, 0, sizeof(sp));
    sp.P = P; sp.V = B; sp.K = P; sp.table = sc.table; sp.view_stride = BatchBwdScratch::factor_stride(P); sp.meta_off = 3ll * P;
    sp.slot_of = nullptr; sp.union_idx = nullptr; sp.dirs = sc.dirs; sp.means3D = a->out_means3D; sp.ts = a->ts;
    sp.scales = a->scales; sp.scales_t = a->scales_t; sp.rotations = a->rotations; sp.rotations_r = a->rotations_r;
    sp.scale_modifier = a->scale_modifier; sp.time_duration = a->time_duration; sp.rot_4d = a->rot_4d;
    sp.gaussian_dim = a->gaussian_dim; sp.force_sh_3d = a->force_sh_3d; sp.D = a->D; sp.D_t = a->D_t; sp.M = a->M;
    sp.out0 = a->dL_dsh; sp.m0 = a->shs_rest ? 1 : a->M; sp.out1 = a->shs_rest ? a->dL_dsh_rest : nullptr; sp.accumulate = 0;
    sp.view_means = a->out_means3D;
    FDGS_STAGE(7, 2, fdgs::launch_sh_outer_sum(sp, stream), "sh_outer_sum (batch)");
    return FDGS_OK;
}

int check_sky_args(const fdgs_sky_args* a) {
    if (!a) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    if (!a->env_map || !a->c2w || !a->campos) return fail(FDGS_ERR_INVALID_ARG, "env_map / c2w / campos required");
    if (a->env_height <= 0 || a->env_width <= 0 || a->env_width > 65000 || a->width <= 0 || a->height <= 0)
        return fail(FDGS_ERR_INVALID_ARG, "bad environment map / image size");
    if (!(a->radius > 0.0f)) return fail(FDGS_ERR_INVALID_ARG, "sky radius must be positive");
    return FDGS_OK;
}

fdgs::SkyParams sky_params(const fdgs_sky_args* a) {
    fdgs::SkyParams p;
    p.env_map = a->env_map; p.env_height = a->env_height; p.env_width = a->env_width;
    p.c2w = a->c2w; p.campos = a->campos;
    p.fl_x = a->fl_x; p.fl_y = a->fl_y; p.cx = a->cx; p.cy = a->cy; p.radius = a->radius;
    p.W = a->width; p.H = a->height;
    return p;
}

int check_sky_batch_args(const fdgs_sky_batch_args* a) {
    if (!a) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    if (!a->env_map || !a->c2w || !a->campos || !a->intrinsics)
        return fail(FDGS_ERR_INVALID_ARG, "env_map / c2w / campos / intrinsics required");
    if (a->B < 1 || a->B > 65535) return fail(FDGS_ERR_INVALID_ARG, "view count B must be in 1..65535");
    if (a->env_height <= 0 || a->env_width <= 0 || a->env_width > 65000 || a->width <= 0 || a->height <= 0)
        return fail(FDGS_ERR_INVALID_ARG, "bad environment map / image size");
    if ((long long)a->width * a->height * 3 * a->B > INT_MAX)
        return fail(FDGS_ERR_INVALID_ARG, "bad environment map / image size: B x 3 x H x W exceeds 2^31 - 1");
    if (!(a->radius > 0.0f)) return fail(FDGS_ERR_INVALID_ARG, "sky radius must be positive");
    return FDGS_OK;
}

fdgs::SkyBatchParams sky_batch_params(const fdgs_sky_batch_args* a) {
    fdgs::SkyBatchParams p;
    p.env_map = a->env_map; p.env_height = a->env_height; p.env_width = a->env_width;
    p.c2w = a->c2w; p.campos = a->campos; p.intrinsics = a->intrinsics; p.radius = a->radius;
    p.W = a->width; p.H = a->height; p.B = a->B;
    return p;
}

}  // namespace

extern "C" {

int fdgs_forward(const fdgs_forward_args* a, fdgs_alloc_fn geom_alloc, void* geom_ctx, fdgs_alloc_fn binning_alloc,
                 void* binning_ctx, fdgs_alloc_fn image_alloc, void* image_ctx, void* stream, fdgs_forward_result* res) {
    return forward_impl(a, nullptr, nullptr, nullptr, geom_alloc, geom_ctx, binning_alloc, binning_ctx, image_alloc, image_ctx,
                        stream, res);
}

int fdgs_forward_bg(const fdgs_forward_args* a, const float* bg_image, fdgs_alloc_fn geom_alloc, void* geom_ctx,
                    fdgs_alloc_fn binning_alloc, void* binning_ctx, fdgs_alloc_fn image_alloc, void* image_ctx, void* stream,
                    fdgs_forward_result* res) {
    return forward_impl(a, bg_image, nullptr, nullptr, geom_alloc, geom_ctx, binning_alloc, binning_ctx, image_alloc, image_ctx,
                        stream, res);
}

int fdgs_forward_zero_sh(const fdgs_forward_args* a, const float* bg_image, float* dL_dsh, float* dL_dsh_rest,
                         fdgs_alloc_fn geom_alloc, void* geom_ctx, fdgs_alloc_fn binning_alloc, void* binning_ctx,
                         fdgs_alloc_fn image_alloc, void* image_ctx, void* stream, fdgs_forward_result* res) {
    return forward_impl(a, bg_image, dL_dsh, dL_dsh_rest, geom_alloc, geom_ctx, binning_alloc, binning_ctx, image_alloc,
                        image_ctx, stream, res);
}

int fdgs_backward(const fdgs_backward_args* a, void* stream) { return backward_impl(a, nullptr, nullptr, 0, stream); }

int fdgs_backward_bg(const fdgs_backward_args* a, const float* bg_image, float* dL_dbg_image, void* stream) {
    return backward_impl(a, bg_image, dL_dbg_image, 0, stream);
}

int fdgs_backward_zero_sh(const fdgs_backward_args* a, const float* bg_image, float* dL_dbg_image, int sh_rows_zeroed,
                          void* stream) {
    return backward_impl(a, bg_image, dL_dbg_image, sh_rows_zeroed, stream);
}

int fdgs_forward_batch(const fdgs_forward_batch_args* args, fdgs_alloc_fn geom_alloc, void* geom_ctx,
                       fdgs_alloc_fn binning_alloc, void* binning_ctx, fdgs_alloc_fn image_alloc, void* image_ctx, void* stream,
                       fdgs_forward_result* res) {
    return forward_batch_impl(args, nullptr, geom_alloc, geom_ctx, binning_alloc, binning_ctx, image_alloc, image_ctx, stream, res);
}

int fdgs_forward_batch_capacity(const fdgs_forward_capacity_args* args, fdgs_alloc_fn geom_alloc, void* geom_ctx,
                                fdgs_alloc_fn binning_alloc, void* binning_ctx, fdgs_alloc_fn image_alloc, void* image_ctx,
                                void* stream, fdgs_forward_result* res) {
    return forward_batch_impl(args ? &args->batch : nullptr, args, geom_alloc, geom_ctx, binning_alloc, binning_ctx, image_alloc,
                              image_ctx, stream, res);
}

int fdgs_backward_batch(const fdgs_backward_batch_args* args, void* stream) { return backward_batch_impl(args, stream); }

int fdgs_backward_camera(const fdgs_backward_args* a, const float* bg_image, float* dL_dbg_image, int sh_rows_zeroed,
                         const fdgs_camera_grad_out* cam, void* stream) {
    g_last_error.clear();
    fdgs::CameraGradParams c;
    if (int rc = camera_grad_params(cam, &c)) return rc;
    return backward_impl(a, bg_image, dL_dbg_image, sh_rows_zeroed, stream, &c);
}

int fdgs_backward_batch_camera(const fdgs_backward_batch_args* args, const fdgs_camera_grad_out* cam, void* stream) {
    g_last_error.clear();
    fdgs::CameraGradParams c;
    if (int rc = camera_grad_params(cam, &c)) return rc;
    return backward_batch_impl(args, stream, &c);
}

int fdgs_sky_forward(const fdgs_sky_args* a, float* out_sky, int* miss_flag, void* stream_v) {
    g_last_error.clear();
    if (int rc = check_sky_args(a)) return rc;
    if (!out_sky) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    FDGS_CUDA(fdgs::launch_sky_fwd(sky_params(a), out_sky, miss_flag, reinterpret_cast<cudaStream_t>(stream_v)), "sky_forward");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_sky_backward(const fdgs_sky_args* a, const float* dL_dsky, float* dL_denv, void* stream_v) {
    g_last_error.clear();
    if (int rc = check_sky_args(a)) return rc;
    if (!dL_dsky || !dL_denv) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    FDGS_CUDA(fdgs::launch_sky_bwd(sky_params(a), dL_dsky, dL_denv, reinterpret_cast<cudaStream_t>(stream_v)), "sky_backward");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_sky_forward_batch(const fdgs_sky_batch_args* a, float* out_sky, int* miss_flag, void* stream_v) {
    g_last_error.clear();
    if (int rc = check_sky_batch_args(a)) return rc;
    if (!out_sky) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    FDGS_CUDA(fdgs::launch_sky_fwd_batch(sky_batch_params(a), out_sky, miss_flag, reinterpret_cast<cudaStream_t>(stream_v)),
              "sky_forward_batch");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_sky_backward_batch(const fdgs_sky_batch_args* a, const float* dL_dsky, float* dL_denv, void* stream_v) {
    g_last_error.clear();
    if (int rc = check_sky_batch_args(a)) return rc;
    if (!dL_dsky || !dL_denv) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    FDGS_CUDA(fdgs::launch_sky_bwd_batch(sky_batch_params(a), dL_dsky, dL_denv, reinterpret_cast<cudaStream_t>(stream_v)),
              "sky_backward_batch");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_mark_visible(int P, const float* means3D, const float* viewmatrix, const float*, unsigned char* present,
                      void* stream_v) {
    g_last_error.clear();
    if (P < 0 || (P > 0 && (!means3D || !viewmatrix || !present))) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    FDGS_CUDA(fdgs::launch_mark_visible(P, means3D, viewmatrix, present, reinterpret_cast<cudaStream_t>(stream_v)),
              "mark_visible");
    return FDGS_OK;
}

static int pack_common(bool unpack, int n, float* const* tensors, const int* widths, const long long* block_off,
                       const long long* idx, long long K, float* flat, void* stream_v) {
    g_last_error.clear();
    if (n < 0 || n > FDGS_MAX_PACK || K < 0) return fail(FDGS_ERR_INVALID_ARG, "bad tensor count / row count");
    if (n == 0 || K == 0) return FDGS_OK;
    if (!tensors || !widths || !block_off || !idx || !flat) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < n; ++i)
        if (!tensors[i] || widths[i] <= 0 || block_off[i] < 0) return fail(FDGS_ERR_INVALID_ARG, "bad tensor table entry");
    FDGS_CUDA(fdgs::launch_pack_rows(unpack, n, tensors, widths, block_off, idx, K, flat, reinterpret_cast<cudaStream_t>(stream_v)),
              unpack ? "unpack_rows" : "pack_rows");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_pack_rows(int n, const float* const* tensors, const int* widths, const long long* block_off, const long long* idx,
                   long long K, float* flat, void* stream) {
    return pack_common(false, n, const_cast<float* const*>(tensors), widths, block_off, idx, K, flat, stream);
}

int fdgs_unpack_rows(int n, float* const* tensors, const int* widths, const long long* block_off, const long long* idx,
                     long long K, const float* flat, void* stream) {
    return pack_common(true, n, tensors, widths, block_off, idx, K, const_cast<float*>(flat), stream);
}

int fdgs_sh_outer_sum(const fdgs_sh_sum_args* a, void* stream_v) {
    g_last_error.clear();
    if (!a) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    if (a->P <= 0) return FDGS_OK;
    if (a->V < 0 || a->K < 0 || a->M <= 0 || a->m0 <= 0 || a->m0 > a->M || a->D < 0 || a->D > 3 || a->D_t < 0 || a->D_t > 2)
        return fail(FDGS_ERR_INVALID_ARG, "bad V / K / M / m0 / degrees");
    if (!a->slot_of || !a->means3D || !a->out0 || (a->m0 < a->M && !a->out1) ||
        (a->V > 0 && a->K > 0 && (!a->table || !a->union_idx || !a->dir_scratch)))
        return fail(FDGS_ERR_INVALID_ARG, "slot_of / union_idx / dir_scratch / means3D / table / outputs required");
    if (a->rot_4d && (!a->scales || !a->scales_t || !a->rotations || !a->rotations_r || !a->ts))
        return fail(FDGS_ERR_INVALID_ARG, "rot_4d needs scales, scales_t, rotations, rotations_r, ts");
    const bool sh4d = !(a->gaussian_dim == 3 || a->force_sh_3d);
    if (sh4d && !a->ts) return fail(FDGS_ERR_INVALID_ARG, "4D SH needs ts");
    if (a->V > 0 && (a->meta_off < 3ll * a->K || a->view_stride < a->meta_off + 4))
        return fail(FDGS_ERR_INVALID_ARG, "view block too small for K rows + metadata");
    fdgs::ShSumParams p;
    p.P = a->P; p.V = a->V; p.K = a->K; p.table = a->table; p.view_stride = a->view_stride; p.meta_off = a->meta_off;
    p.slot_of = a->slot_of; p.union_idx = a->union_idx; p.dirs = a->dir_scratch; p.means3D = a->means3D; p.ts = a->ts; p.scales = a->scales; p.scales_t = a->scales_t;
    p.rotations = a->rotations; p.rotations_r = a->rotations_r; p.scale_modifier = a->scale_modifier;
    p.time_duration = a->time_duration; p.rot_4d = a->rot_4d; p.gaussian_dim = a->gaussian_dim;
    p.force_sh_3d = a->force_sh_3d; p.D = a->D; p.D_t = a->D_t; p.M = a->M;
    p.out0 = a->out0; p.m0 = a->m0; p.out1 = (a->m0 < a->M) ? a->out1 : nullptr; p.accumulate = a->accumulate;
    p.view_means = nullptr;
    FDGS_CUDA(fdgs::launch_sh_outer_sum(p, reinterpret_cast<cudaStream_t>(stream_v)), "sh_outer_sum");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_union_maps(long long P, const int* radii, const int* cs, int* slot_of, long long* idx, void* stream_v) {
    g_last_error.clear();
    if (P < 0) return fail(FDGS_ERR_INVALID_ARG, "bad P");
    if (P == 0) return FDGS_OK;
    if (!radii || !cs || !slot_of || !idx) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    FDGS_CUDA(fdgs::launch_union_maps(P, radii, cs, slot_of, idx, reinterpret_cast<cudaStream_t>(stream_v)), "union_maps");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_view_stats(long long P, const float* viewspace_grad, int grad_stride, const int* radii, float* grad_norm_sum,
                    float* visibility_count, int* max_radii, void* stream_v) {
    g_last_error.clear();
    if (P < 0 || grad_stride < 2) return fail(FDGS_ERR_INVALID_ARG, "bad P / gradient row stride");
    if (P == 0) return FDGS_OK;
    if (!viewspace_grad || !radii || !grad_norm_sum || !visibility_count || !max_radii) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    FDGS_CUDA(fdgs::launch_view_stats(P, viewspace_grad, grad_stride, radii, grad_norm_sum, visibility_count, max_radii,
                                      reinterpret_cast<cudaStream_t>(stream_v)), "view_stats");
    g_kernel_launches += 1;
    return FDGS_OK;
}

// ---- densification (densify.cu) -----------------------------------------------------------------------------------
static int check_densify_args(const fdgs_densify_args* a) {
    if (!a) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    if (a->P < 0 || a->P > 0x7fffffffLL || a->N < 1) return fail(FDGS_ERR_INVALID_ARG, "bad P / N");
    if ((a->gaussian_dim != 3 && a->gaussian_dim != 4) || (a->rot_4d && a->gaussian_dim != 4))
        return fail(FDGS_ERR_INVALID_ARG, "gaussian_dim must be 3 or 4 (4 with rot_4d)");
    if (a->num_tensors < 0 || a->num_tensors > FDGS_DENSIFY_MAX_TENSORS) return fail(FDGS_ERR_INVALID_ARG, "bad tensor count");
    if (a->P == 0) return FDGS_OK;
    if (!a->scaling || !a->opacity) return fail(FDGS_ERR_INVALID_ARG, "null argument: scaling / opacity required");
    if (!a->prune_only) {
        if (!a->xyz_gradient_accum || !a->denom || !a->xyz || !a->rotation)
            return fail(FDGS_ERR_INVALID_ARG, "null argument: densifying needs xyz_gradient_accum / denom / xyz / rotation");
        if (a->gaussian_dim == 4 && (!a->t || !a->scaling_t))
            return fail(FDGS_ERR_INVALID_ARG, "null argument: gaussian_dim 4 needs t / scaling_t");
        if (a->rot_4d && !a->rotation_r) return fail(FDGS_ERR_INVALID_ARG, "null argument: rot_4d needs rotation_r");
    } else if (a->use_max_screen_size && !a->max_radii2D) {
        return fail(FDGS_ERR_INVALID_ARG, "null argument: max_screen_size needs max_radii2D");
    }
    for (int i = 0; i < a->num_tensors; ++i) {
        const int k = a->kind[i], w = a->width[i];
        if (!a->src[i] || !a->dst[i]) return fail(FDGS_ERR_INVALID_ARG, "null argument: tensor table entry");
        if (k < FDGS_DENSIFY_COPY || k > FDGS_DENSIFY_SCALING_T) return fail(FDGS_ERR_INVALID_ARG, "bad tensor kind");
        const int need = (k == FDGS_DENSIFY_XYZ || k == FDGS_DENSIFY_SCALING) ? 3 : (k == FDGS_DENSIFY_T || k == FDGS_DENSIFY_SCALING_T) ? 1 : 0;
        if (w <= 0 || (need && w != need)) return fail(FDGS_ERR_INVALID_ARG, "tensor width does not match its kind");
        if ((k == FDGS_DENSIFY_T || k == FDGS_DENSIFY_SCALING_T) && a->gaussian_dim != 4)
            return fail(FDGS_ERR_INVALID_ARG, "t / scaling_t rows need gaussian_dim 4");
    }
    return FDGS_OK;
}

size_t fdgs_densify_scratch_bytes(long long P) { return fdgs::densify_scratch_bytes(P > 0 ? P : 0); }

int fdgs_densify_plan(const fdgs_densify_args* a, char* scratch, int* totals, void* stream_v) {
    g_last_error.clear();
    const int rc = check_densify_args(a);
    if (rc != FDGS_OK) return rc;
    if (!totals || (a->P > 0 && !scratch)) return fail(FDGS_ERR_INVALID_ARG, "null argument: scratch / totals");
    FDGS_CUDA(fdgs::launch_densify_plan(*a, scratch, totals, reinterpret_cast<cudaStream_t>(stream_v)), "densify_plan");
    g_kernel_launches += a->P > 0 ? 4 : 0;
    return FDGS_OK;
}

int fdgs_densify_apply(const fdgs_densify_args* a, const char* scratch, const int* totals, void* stream_v) {
    g_last_error.clear();
    const int rc = check_densify_args(a);
    if (rc != FDGS_OK) return rc;
    if (!totals || (a->P > 0 && !scratch)) return fail(FDGS_ERR_INVALID_ARG, "null argument: scratch / totals");
    for (int i = 0; i < 4; ++i)
        if (totals[i] < 0 || totals[i] > a->P) return fail(FDGS_ERR_INVALID_ARG, "totals inconsistent with P");
    const long long S = totals[2], kept = totals[3];
    if (kept > S || (a->prune_only && (totals[1] || S))) return fail(FDGS_ERR_INVALID_ARG, "totals inconsistent with the call");
    if (S > 0 && (!a->samples || (a->gaussian_dim == 4 && !a->rot_4d && !a->samples_t)))
        return fail(FDGS_ERR_INVALID_ARG, "null argument: split rows need samples (and samples_t)");
    FDGS_CUDA(fdgs::launch_densify_apply(*a, scratch, S, kept, reinterpret_cast<cudaStream_t>(stream_v)), "densify_apply");
    // the compaction, and the split-position kernel when children survive and xyz / t rows are in the table
    bool positions = false;
    for (int i = 0; i < a->num_tensors; ++i)
        positions |= a->kind[i] == FDGS_DENSIFY_XYZ || a->kind[i] == FDGS_DENSIFY_T;
    g_kernel_launches += (a->P > 0 && a->num_tensors > 0) ? 1 + (positions && kept > 0) : 0;
    return FDGS_OK;
}

int fdgs_reset_opacity(long long P, float* opacity, float* exp_avg, float* exp_avg_sq, void* stream_v) {
    g_last_error.clear();
    if (P < 0) return fail(FDGS_ERR_INVALID_ARG, "bad P");
    if (P == 0) return FDGS_OK;
    if (!opacity) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    FDGS_CUDA(fdgs::launch_reset_opacity(P, opacity, exp_avg, exp_avg_sq, reinterpret_cast<cudaStream_t>(stream_v)), "reset_opacity");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_densify_stats(long long P, int batch_size, const float* point_grad, int point_grad_stride, const float* visibility_count,
                       const int* radii, const float* t_grad, float* xyz_gradient_accum, float* denom, float* t_gradient_accum,
                       float* max_radii2D, void* stream_v) {
    return fdgs_densify_stats_status(P, batch_size, point_grad, point_grad_stride, visibility_count, radii, t_grad,
                                     xyz_gradient_accum, denom, t_gradient_accum, max_radii2D, nullptr, stream_v);
}

int fdgs_densify_stats_status(long long P, int batch_size, const float* point_grad, int point_grad_stride,
                              const float* visibility_count, const int* radii, const float* t_grad, float* xyz_gradient_accum,
                              float* denom, float* t_gradient_accum, float* max_radii2D, const int* status, void* stream_v) {
    g_last_error.clear();
    if (P < 0 || batch_size < 1) return fail(FDGS_ERR_INVALID_ARG, "bad P / batch size");
    if (batch_size == 1 ? point_grad_stride < 2 : point_grad_stride != 1) return fail(FDGS_ERR_INVALID_ARG, "bad gradient row stride");
    if (P == 0) return FDGS_OK;
    if (!point_grad || !radii || !xyz_gradient_accum || !denom || !max_radii2D || (batch_size > 1 && !visibility_count))
        return fail(FDGS_ERR_INVALID_ARG, "null argument");
    if (!t_grad != !t_gradient_accum) return fail(FDGS_ERR_INVALID_ARG, "t_grad and t_gradient_accum go together");
    FDGS_CUDA(fdgs::launch_densify_stats(P, batch_size, point_grad, point_grad_stride, visibility_count, radii, t_grad,
                                         xyz_gradient_accum, denom, t_gradient_accum, max_radii2D, status,
                                         reinterpret_cast<cudaStream_t>(stream_v)), "densify_stats");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_check_rows_zero(int n, const float* const* tensors, const int* widths, long long P, const int* radii, int* flag,
                         void* stream_v) {
    g_last_error.clear();
    if (n < 0 || n > FDGS_MAX_PACK || P < 0) return fail(FDGS_ERR_INVALID_ARG, "bad tensor count / row count");
    if (n == 0 || P == 0) return FDGS_OK;
    if (!tensors || !widths || !radii || !flag) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < n; ++i)
        if (!tensors[i] || widths[i] <= 0) return fail(FDGS_ERR_INVALID_ARG, "bad tensor table entry");
    FDGS_CUDA(fdgs::launch_rows_zero_check(n, tensors, widths, P, radii, flag, reinterpret_cast<cudaStream_t>(stream_v)),
              "rows_zero_check");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_l1_ssim_forward(const float* x, const float* y, int C, int H, int W, float* maps, double* sums, void* stream_v) {
    g_last_error.clear();
    if (C <= 0 || H <= 0 || W <= 0) return fail(FDGS_ERR_INVALID_ARG, "bad C / H / W");
    if (!x || !y || !maps || !sums) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    FDGS_CUDA(fdgs::launch_l1_ssim_fwd(x, y, C, H, W, maps, sums, reinterpret_cast<cudaStream_t>(stream_v)), "l1_ssim_forward");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_l1_ssim_backward(const float* x, const float* y, int C, int H, int W, const float* maps, const float* grad_scale,
                          float lambda_dssim, float* dL_dx, void* stream_v) {
    g_last_error.clear();
    if (C <= 0 || H <= 0 || W <= 0) return fail(FDGS_ERR_INVALID_ARG, "bad C / H / W");
    if (!x || !y || !maps || !dL_dx) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    FDGS_CUDA(fdgs::launch_l1_ssim_bwd(x, y, C, H, W, maps, grad_scale, lambda_dssim, dL_dx, reinterpret_cast<cudaStream_t>(stream_v)),
              "l1_ssim_backward");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_adam_scalars(int n, const float* lrs, const long long* steps, const int* enable, double beta1, double beta2,
                      float* table) {
    g_last_error.clear();
    if (n < 0 || n > FDGS_MAX_PACK) return fail(FDGS_ERR_INVALID_ARG, "bad tensor count");
    if (n == 0) return FDGS_OK;
    if (!lrs || !steps || !enable || !table) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < n; ++i)
        if (enable[i] && steps[i] < 1) return fail(FDGS_ERR_INVALID_ARG, "bad step count");
    for (int i = 0; i < n; ++i) {
        table[3 * i] = 0.f; table[3 * i + 1] = 1.f; table[3 * i + 2] = 0.f;
        if (!enable[i]) continue;
        // bias corrections in double on the host, like torch.optim.Adam's single-tensor path
        const double bc1 = 1.0 - pow(beta1, (double)steps[i]), bc2 = 1.0 - pow(beta2, (double)steps[i]);
        table[3 * i] = (float)((double)lrs[i] / bc1);
        table[3 * i + 1] = (float)sqrt(bc2);
        table[3 * i + 2] = 1.f;
    }
    return FDGS_OK;
}

int fdgs_adam_step(int n, float* const* params, float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                   const int* widths, const float* lrs, long long P, const long long* rows, long long num_rows, long long step,
                   double beta1, double beta2, double eps, int zero_grad, void* stream_v) {
    g_last_error.clear();
    if (n < 0 || n > FDGS_MAX_PACK || P < 0 || step < 1 || (rows && num_rows < 0))
        return fail(FDGS_ERR_INVALID_ARG, "bad tensor count / row count / step");
    if (n == 0 || P == 0 || (rows && num_rows == 0)) return FDGS_OK;
    if (!params || !grads || !exp_avg || !exp_avg_sq || !widths || !lrs) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < n; ++i)
        if (!params[i] || !grads[i] || !exp_avg[i] || !exp_avg_sq[i] || widths[i] <= 0)
            return fail(FDGS_ERR_INVALID_ARG, "bad tensor table entry");
    long long steps[FDGS_MAX_PACK];
    int enable[FDGS_MAX_PACK];
    float table[3 * FDGS_MAX_PACK], step_sizes[FDGS_MAX_PACK];
    for (int i = 0; i < n; ++i) { steps[i] = step; enable[i] = 1; }
    fdgs_adam_scalars(n, lrs, steps, enable, beta1, beta2, table);
    for (int i = 0; i < n; ++i) step_sizes[i] = table[3 * i];
    FDGS_CUDA(fdgs::launch_adam(n, params, grads, exp_avg, exp_avg_sq, widths, step_sizes, rows ? num_rows : P, rows, (float)(1.0 - beta1),
                                (float)beta2, (float)(1.0 - beta2), (float)eps, table[1], zero_grad, reinterpret_cast<cudaStream_t>(stream_v)),
              "adam_step");
    g_kernel_launches += 1;
    return FDGS_OK;
}

int fdgs_adam_step_staged(int n, float* const* params, float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                          const int* widths, long long P, const float* scalars, const int* status, double beta1, double beta2,
                          double eps, void* stream_v) {
    g_last_error.clear();
    if (n < 0 || n > FDGS_MAX_PACK || P < 0) return fail(FDGS_ERR_INVALID_ARG, "bad tensor count / row count");
    if (n == 0 || P == 0) return FDGS_OK;
    if (!params || !grads || !exp_avg || !exp_avg_sq || !widths || !scalars) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    for (int i = 0; i < n; ++i)
        if (!params[i] || !grads[i] || !exp_avg[i] || !exp_avg_sq[i] || widths[i] <= 0)
            return fail(FDGS_ERR_INVALID_ARG, "bad tensor table entry");
    FDGS_CUDA(fdgs::launch_adam_staged(n, params, grads, exp_avg, exp_avg_sq, widths, P, scalars, status, (float)(1.0 - beta1),
                                       (float)beta2, (float)(1.0 - beta2), (float)eps, reinterpret_cast<cudaStream_t>(stream_v)),
              "adam_step_staged");
    g_kernel_launches += 1;
    return FDGS_OK;
}

size_t fdgs_knn_scratch_bytes(int n) { return fdgs::knn_scratch_bytes(n > 0 ? n : 0); }

int fdgs_knn(int n, int k, const float* xyz, char* scratch, int* idx, float* dist2, int brute_force, void* stream_v) {
    g_last_error.clear();
    if (n < 0 || k < 1 || k > 32) return fail(FDGS_ERR_INVALID_ARG, "bad n / k (1 <= k <= 32)");
    if (n == 0) return FDGS_OK;
    if (!xyz || !idx || !dist2 || (!brute_force && !scratch)) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    if (brute_force) FDGS_CUDA(fdgs::launch_knn_bruteforce(n, k, xyz, idx, dist2, stream), "knn (brute force)");
    else FDGS_CUDA(fdgs::launch_knn(n, k, xyz, scratch, idx, dist2, stream), "knn");
    g_kernel_launches += brute_force ? 1 : 7;
    return FDGS_OK;
}

// ---- rigidity and motion regularisers (regularize.cu) ----------------------------------------------------------------
static int check_rigid_size(int n, int k) {
    if (n <= 0 || k < 1 || k > 32) return fail(FDGS_ERR_INVALID_ARG, "bad n / k (n > 0, 1 <= k <= 32)");
    if ((long long)n * k > 0x7fffffffLL) return fail(FDGS_ERR_INVALID_ARG, "n * k exceeds 2^31 - 1 edges");
    return FDGS_OK;
}

static int check_rigid_args(const fdgs_rigid_args* a, bool rigid, bool transpose) {
    if (!a) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    if (int rc = check_rigid_size(a->n, a->k)) return rc;
    if (!a->t || !a->scaling || !a->scaling_t || !a->rotation || !a->rotation_r)
        return fail(FDGS_ERR_INVALID_ARG, "null argument: t / scaling / scaling_t / rotation / rotation_r required");
    if (rigid && (!a->idx || !a->weight)) return fail(FDGS_ERR_INVALID_ARG, "null argument: the rigidity loss needs idx / weight");
    if (transpose && (!a->in_offsets || !a->in_edges))
        return fail(FDGS_ERR_INVALID_ARG, "null argument: the rigidity backward needs in_offsets / in_edges");
    return FDGS_OK;
}

static fdgs::RigidParams rigid_params(const fdgs_rigid_args* a) {
    fdgs::RigidParams p;
    p.n = a->n; p.k = a->k; p.t = a->t; p.scaling = a->scaling; p.scaling_t = a->scaling_t;
    p.rotation = a->rotation; p.rotation_r = a->rotation_r; p.idx = a->idx; p.weight = a->weight;
    p.in_offsets = a->in_offsets; p.in_edges = a->in_edges; p.velocity = a->velocity;
    return p;
}

size_t fdgs_rigid_scratch_bytes(int n, int k) {
    return (n > 0 && k >= 1 && k <= 32 && (long long)n * k <= 0x7fffffffLL) ? fdgs::rigid_scratch_bytes(n, k) : 0;
}

int fdgs_rigid_neighbours(int n, int k, const int* idx, const float* dist2, char* scratch, float* weight, int* in_offsets,
                          int* in_edges, void* stream_v) {
    g_last_error.clear();
    if (int rc = check_rigid_size(n, k)) return rc;
    if (!idx || !dist2 || !scratch || !weight || !in_offsets || !in_edges) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    FDGS_CUDA(fdgs::launch_rigid_neighbours(n, k, idx, dist2, scratch, weight, in_offsets, in_edges,
                                            reinterpret_cast<cudaStream_t>(stream_v)), "rigid_neighbours");
    g_kernel_launches += 2;     // + the radix sort's own kernels
    return FDGS_OK;
}

int fdgs_rigid_forward(const fdgs_rigid_args* a, char* scratch, float* loss_rigid, float* loss_motion, void* stream_v) {
    g_last_error.clear();
    if (int rc = check_rigid_args(a, loss_rigid != nullptr, false)) return rc;
    if (!a->velocity) return fail(FDGS_ERR_INVALID_ARG, "null argument: velocity");
    if ((loss_rigid || loss_motion) && !scratch) return fail(FDGS_ERR_INVALID_ARG, "null argument: scratch");
    FDGS_CUDA(fdgs::launch_rigid_forward(rigid_params(a), scratch, loss_rigid, loss_motion, reinterpret_cast<cudaStream_t>(stream_v)),
              "rigid_forward");
    g_kernel_launches += (loss_rigid || loss_motion) ? 3 : 1;
    return FDGS_OK;
}

int fdgs_rigid_backward(const fdgs_rigid_args* a, const float* grad_rigid, const float* grad_motion, float* dL_dscaling,
                        float* dL_dscaling_t, float* dL_drotation, float* dL_drotation_r, void* stream_v) {
    g_last_error.clear();
    if (int rc = check_rigid_args(a, grad_rigid != nullptr, grad_rigid != nullptr)) return rc;
    if (!a->velocity) return fail(FDGS_ERR_INVALID_ARG, "null argument: the forward's velocity is required");
    if (!dL_dscaling || !dL_dscaling_t || !dL_drotation || !dL_drotation_r) return fail(FDGS_ERR_INVALID_ARG, "null argument: gradient outputs");
    FDGS_CUDA(fdgs::launch_rigid_backward(rigid_params(a), grad_rigid, grad_motion, dL_dscaling, dL_dscaling_t, dL_drotation,
                                          dL_drotation_r, reinterpret_cast<cudaStream_t>(stream_v)),
              "rigid_backward");
    g_kernel_launches += 1;
    return FDGS_OK;
}

// ---- evaluation metrics (metrics.cu) --------------------------------------------------------------------------------
static int check_metrics_size(int B, int C, int H, int W) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0) return fail(FDGS_ERR_INVALID_ARG, "bad B / C / H / W");
    if (H < 176 || W < 176) return fail(FDGS_ERR_INVALID_ARG, "H and W must be at least 176 (MS-SSIM's five scales)");
    if ((long long)B * C > 65535) return fail(FDGS_ERR_INVALID_ARG, "B * C exceeds 65535 image planes");
    // the float64 pyramid is about 2/3 of 16 bytes per input pixel; tile rows must fit the grid's y extent
    if ((double)B * C * H * W * 16.0 > 9.0e18 || (H + 31) / 32 > 65535)
        return fail(FDGS_ERR_INVALID_ARG, "image size overflow");
    return FDGS_OK;
}

size_t fdgs_metrics_scratch_bytes(int B, int C, int H, int W) {
    if (check_metrics_size(B, C, H, W) != FDGS_OK) {
        g_last_error.clear();
        return 0;
    }
    return fdgs::metrics_scratch_bytes(B, C, H, W);
}

int fdgs_image_metrics(const fdgs_metrics_args* a, char* scratch, void* stream_v) {
    g_last_error.clear();
    if (!a) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    if (int rc = check_metrics_size(a->B, a->C, a->H, a->W)) return rc;
    if (!a->x || !a->y || !a->out || !scratch) return fail(FDGS_ERR_INVALID_ARG, "null argument: x / y / out / scratch");
    FDGS_CUDA(fdgs::launch_image_metrics(*a, scratch, reinterpret_cast<cudaStream_t>(stream_v)), "image_metrics");
    g_kernel_launches += a->accum ? 7 : 6;
    return FDGS_OK;
}

int fdgs_debug_activate(int n, const float* log_s, const float* logit, const float* quat, int mode, float* s_out, float* o_out,
                        float* q_out, void* stream_v) {
    g_last_error.clear();
    if (n < 0 || (n > 0 && (!log_s || !logit || !quat || !s_out || !o_out || !q_out))) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    if (mode != 0) return fail(FDGS_ERR_INVALID_ARG, "mode must be 0 (ATen's summation order of the quaternion norm)");
    FDGS_CUDA(fdgs::launch_debug_activate(n, log_s, logit, quat, s_out, o_out, q_out, reinterpret_cast<cudaStream_t>(stream_v)),
              "debug_activate");
    return FDGS_OK;
}

int fdgs_profile_enable(int on) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof_on = on != 0;
    return FDGS_OK;
}

int fdgs_profile_read(double ms[FDGS_NUM_STAGES], long long calls[FDGS_NUM_STAGES]) {
    std::vector<ProfEvent> ev;
    {
        std::lock_guard<std::mutex> lk(g_prof_mu);
        ev.swap(g_prof_events);
    }
    for (int i = 0; i < FDGS_NUM_STAGES; ++i) {
        if (ms) ms[i] = 0.0;
        if (calls) calls[i] = 0;
    }
    for (auto& e : ev) {
        cudaEventSynchronize(e.b);
        float t = 0.f;
        cudaEventElapsedTime(&t, e.a, e.b);
        if (e.stage >= 0 && e.stage < FDGS_NUM_STAGES) {
            if (ms) ms[e.stage] += t;
            if (calls) calls[e.stage] += 1;
        }
        cudaEventDestroy(e.a);
        cudaEventDestroy(e.b);
    }
    return FDGS_OK;
}

long long fdgs_launch_count(void) { return g_kernel_launches.load(); }

int fdgs_set_tile_cull(int mode) { return g_tile_cull.exchange(mode ? 1 : 0); }

int fdgs_debug_export_geom(const char* geom_buffer, int P, float* depths, float* means2D, float* conic_opacity,
                           float* rgb, unsigned char* clamped, unsigned int* tiles_touched, void* stream_v) {
    g_last_error.clear();
    if (!geom_buffer || P <= 0) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    GeomState g = GeomState::carve(align128(const_cast<char*>(geom_buffer)), P);
    const size_t p = (size_t)P;
    // rows the forward did not render read as zeros (their records are never written)
    FDGS_CUDA(fdgs::launch_unpack_grec(P, g.grec, reinterpret_cast<const int*>(g.tiles_touched), depths, means2D,
                                       conic_opacity, rgb, stream),
              "export records");
    if (clamped) FDGS_CUDA(cudaMemcpyAsync(clamped, g.clamped, p, cudaMemcpyDeviceToDevice, stream), "export clamped");
    if (tiles_touched)
        FDGS_CUDA(cudaMemcpyAsync(tiles_touched, g.tiles_touched, p * 4, cudaMemcpyDeviceToDevice, stream), "export tiles");
    return FDGS_OK;
}

int fdgs_debug_export_binning(const char* binning_buffer, const char* image_buffer, int R, int W, int H,
                              unsigned int* point_list, unsigned int* ranges, unsigned int* n_contrib, void* stream_v) {
    g_last_error.clear();
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    if (!image_buffer) return fail(FDGS_ERR_INVALID_ARG, "null argument");
    ImageState img = ImageState::carve(align128(const_cast<char*>(image_buffer)), W, H);
    const size_t tiles = (size_t)((W + fdgs::TILE_X - 1) / fdgs::TILE_X) * ((H + fdgs::TILE_Y - 1) / fdgs::TILE_Y);
    if (point_list && R > 0) {
        if (!binning_buffer) return fail(FDGS_ERR_INVALID_ARG, "null binning buffer");
        BinningState b = BinningState::carve(align128(const_cast<char*>(binning_buffer)), R);
        FDGS_CUDA(cudaMemcpyAsync(point_list, b.point_list, (size_t)R * 4, cudaMemcpyDeviceToDevice, stream),
                  "export point_list");
    }
    if (ranges) FDGS_CUDA(cudaMemcpyAsync(ranges, img.ranges, tiles * 8, cudaMemcpyDeviceToDevice, stream), "export ranges");
    if (n_contrib)
        FDGS_CUDA(cudaMemcpyAsync(n_contrib, img.n_contrib, (size_t)W * H * 4, cudaMemcpyDeviceToDevice, stream),
                  "export n_contrib");
    return FDGS_OK;
}

int fdgs_debug_export_binning_view(const char* image_buffer, int width, int height, int B, int view, unsigned int* ranges,
                                   unsigned int* n_contrib, void* stream_v) {
    g_last_error.clear();
    if (!image_buffer || width <= 0 || height <= 0 || B < 1 || view < 0 || view >= B)
        return fail(FDGS_ERR_INVALID_ARG, "bad image buffer / size / view");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
    ImageState img = ImageState::carve(align128(const_cast<char*>(image_buffer)), width, height, B);
    const size_t tiles = img.tiles / (size_t)B, N = (size_t)width * height;
    if (ranges)
        FDGS_CUDA(cudaMemcpyAsync(ranges, img.ranges + (size_t)view * tiles, tiles * 8, cudaMemcpyDeviceToDevice, stream),
                  "export ranges");
    if (n_contrib)
        FDGS_CUDA(cudaMemcpyAsync(n_contrib, img.n_contrib + (size_t)view * N, N * 4, cudaMemcpyDeviceToDevice, stream),
                  "export n_contrib");
    return FDGS_OK;
}

}  // extern "C"
