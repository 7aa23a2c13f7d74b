// api.cu -- the extern "C" boundary of libgsrast.so (declared in include/gsrast.h) and the
// forward / backward orchestration.  Replaces CudaRasterizer::Rasterizer::{forward,backward,
// markVisible} (rasterizer_impl.cu:141-153,198-444) and the buffer carving of
// rasterizer_impl.h:21-73.  All work is enqueued on the caller's stream; the only host
// synchronisation is the read-back of the instance count R (the reference blocks on the same
// value, rasterizer_impl.cu:283-284).
#include <atomic>
#include "common.cuh"

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <nvtx3/nvToolsExt.h>   // header-only NVTX v3: ranges are no-ops unless a profiler is attached

namespace gsr {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
    set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
    return (int)e;
}


// ---- optional per-stage device timing (bench.py's roofline numbers come from here) -------------
// Off by default.  When on, every stage is bracketed by two events on the caller's stream;
// gsr_profile_read() synchronises nothing itself: the caller synchronises the stream first.
static const char* const k_stage_names[ST_COUNT] = {"preprocess_fwd", "depth_sort", "offset_scan", "emit_cells",
                                                    "cell_sort", "cell_count", "tile_offsets", "tile_scatter",
                                                    "render_fwd", "render_bwd", "preprocess_bwd"};
static bool g_prof_on = false;
static cudaEvent_t g_prof_ev[ST_COUNT][2];
static bool g_prof_ev_ok = false;
static bool g_prof_used[ST_COUNT];
static std::atomic<unsigned long long> g_launches{0};

void count_launches(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

void prof_begin(int st, cudaStream_t s) {
    nvtxRangePushA(k_stage_names[st]);      // one NVTX range per stage (SURVEY section 5 "tracing"): visible in nsys / ncu --nvtx
    if (!g_prof_on) return;
    if (!g_prof_ev_ok) {
        for (int i = 0; i < ST_COUNT; ++i) { cudaEventCreate(&g_prof_ev[i][0]); cudaEventCreate(&g_prof_ev[i][1]); }
        g_prof_ev_ok = true;
    }
    cudaEventRecord(g_prof_ev[st][0], s);
}
void prof_end(int st, cudaStream_t s) {
    nvtxRangePop();
    if (!g_prof_on) return;
    cudaEventRecord(g_prof_ev[st][1], s);
    g_prof_used[st] = true;
}

// ---- carving -------------------------------------------------------------------------------
template <typename T>
static void take(char*& cur, T*& ptr, size_t count, size_t align = 256) {
    const uintptr_t a = (reinterpret_cast<uintptr_t>(cur) + align - 1) & ~(uintptr_t)(align - 1);
    ptr = reinterpret_cast<T*>(a);
    cur = reinterpret_cast<char*>(ptr + count);
}

size_t carve_geom(char* base, int P, int M, GeomState* out) {
    GeomState g;
    char* cur = base;
    const size_t n = (size_t)P;
    take(cur, g.rec, 2 * n);
    take(cur, g.rgb, M > 0 ? 3 * n : 0);
    take(cur, g.clamped, M > 0 ? n : 0);
    take(cur, g.depths, n);
    take(cur, g.tiles_touched, n);
    take(cur, g.cells_touched, n);
    take(cur, g.rect, n);
    take(cur, g.counters, 8);
    take(cur, g.key_a, n);
    take(cur, g.key_b, n);
    take(cur, g.val_a, n);
    take(cur, g.val_b, n);
    g.order = g.val_a;   // 32 key bits = 4 passes (even): the sorted pairs end up in (key_a, val_a)
    take(cur, g.cells_sorted, n);
    take(cur, g.rect_sorted, n);
    take(cur, g.offsets, n + 1);
    take(cur, g.radix_tmp, radix_tmp_elems(n) + scan_tmp_elems(n));
    if (out) *out = g;
    return (size_t)(cur - base) + 256;
}

size_t carve_img(char* base, int W, int H, ImgState* out) {
    ImgState im;
    char* cur = base;
    const size_t N = (size_t)W * H;
    const size_t T = (size_t)tiles_x(W) * tiles_y(H);
    take(cur, im.final_T, N, 128);   // first 128-B aligned field, like the reference ImageState
    take(cur, im.n_contrib, N);
    take(cur, im.ranges, T);
    take(cur, im.blend_mask, T * MASK_BLOCKS * MASK_WORDS);
    if (out) *out = im;
    return (size_t)(cur - base) + 256;
}

size_t carve_bin(char* base, size_t R, BinState* out) {
    BinState b;
    char* cur = base;
    take(cur, b.point_list, R);
    if (out) *out = b;
    return (size_t)(cur - base) + 256;
}

size_t carve_bin_scratch(char* base, size_t N1, int W, int H, BinScratch* out) {
    BinScratch b;
    char* cur = base;
    const int gx = tiles_x(W), gy = tiles_y(H);
    const size_t num_tiles = (size_t)gx * gy;
    const size_t num_cells = (size_t)((gx + CELL - 1) / CELL) * ((gy + CELL - 1) / CELL);
    take(cur, b.key_a, N1);
    take(cur, b.val_a, N1);
    take(cur, b.key_b, N1);
    take(cur, b.val_b, N1);
    take(cur, b.radix_tmp, radix_tmp_elems(N1));
    take(cur, b.cell_range, num_cells);
    take(cur, b.unit_base, num_cells + 1);
    b.units_cap = ((N1 / UNIT + num_cells + 7) / 8) * 8;
    take(cur, b.M, (size_t)CELL_TILES * b.units_cap);
    take(cur, b.row_total, CELL_TILES);
    take(cur, b.tile_start, num_tiles + 1);
    take(cur, b.block_sums, (num_tiles + 1023) / 1024);
    if (out) *out = b;
    return (size_t)(cur - base) + 256;
}

size_t carve_det(char* base, int P, size_t R, DetSlots* out, uint32_t** scan_tmp) {
    DetSlots d{};
    char* cur = base;
    const size_t n = (size_t)(P > 0 ? P : 0);
    uint32_t* b;
    uint32_t* tmp;
    take(cur, b, n + 1);
    take(cur, tmp, scan_tmp_elems(n));
    take(cur, d.rec, 3 * R);
    d.base = b;
    if (out) *out = d;
    if (scan_tmp) *scan_tmp = tmp;
    return (size_t)(cur - base) + 256;
}

size_t det_mark_bytes(size_t R) { return ((R * DetSlots::KB + 31) / 32) * sizeof(uint32_t); }

static int check_fwd_args(const GsrForwardArgs* a) {
    if (!a) { set_error("args is NULL"); return GSR_E_INVALID; }
    if (a->P < 0 || a->W <= 0 || a->H <= 0) { set_error("bad sizes P=%d W=%d H=%d", a->P, a->W, a->H); return GSR_E_INVALID; }
    if (a->P > 0) {
        if (!a->means3D || !a->opacities || !a->viewmatrix || !a->projmatrix || !a->background || !a->subpixel_offset ||
            (!a->out_color && !a->peer_images) || !a->radii) { set_error("a required pointer is NULL"); return GSR_E_INVALID; }
        if ((a->peer_images != nullptr) != (a->n_peer_images > 0)) { set_error("peer_images / n_peer_images mismatch"); return GSR_E_INVALID; }
        if ((a->shs == nullptr) == (a->colors_precomp == nullptr)) { set_error("provide exactly one of shs / colors_precomp"); return GSR_E_INVALID; }
        const bool have_sr = a->scales != nullptr && a->rotations != nullptr;
        if (have_sr == (a->cov3D_precomp != nullptr) || ((a->scales != nullptr) != (a->rotations != nullptr))) {
            set_error("provide exactly one of (scales, rotations) / cov3D_precomp");
            return GSR_E_INVALID;
        }
        if (a->shs && (a->M <= 0 || !a->campos)) { set_error("shs given but M<=0 or campos NULL"); return GSR_E_INVALID; }
        if (a->shs && (a->D < 0 || a->D > 3 || (a->D + 1) * (a->D + 1) > a->M)) { set_error("SH degree %d does not fit M=%d", a->D, a->M); return GSR_E_INVALID; }
    }
    if (tiles_x(a->W) > 65535 || tiles_y(a->H) > 65535 ||
        (size_t)((tiles_x(a->W) + CELL - 1) / CELL) * ((tiles_y(a->H) + CELL - 1) / CELL) > 65536) {
        set_error("image too large");
        return GSR_E_INVALID;
    }
    return 0;
}

static void shard_rows(int H, int ty0_in, int ty1_in, int* ty0, int* ty1) {
    const int gy = tiles_y(H);
    if (ty0_in == 0 && ty1_in == 0) { *ty0 = 0; *ty1 = gy; return; }
    *ty0 = ty0_in < 0 ? 0 : (ty0_in > gy ? gy : ty0_in);
    *ty1 = ty1_in < *ty0 ? *ty0 : (ty1_in > gy ? gy : ty1_in);
}

}  // namespace gsr

using namespace gsr;

extern "C" {

int gsr_abi_version(void) { return GSR_ABI_VERSION; }

void gsr_profile_enable(int on) {
    g_prof_on = on != 0;
    for (int i = 0; i < ST_COUNT; ++i) g_prof_used[i] = false;
}
int gsr_profile_stage_count(void) { return ST_COUNT; }
const char* gsr_profile_stage_name(int i) { return (i >= 0 && i < ST_COUNT) ? k_stage_names[i] : ""; }
int gsr_profile_read(float* ms, int n) {
    // elapsed device time of each stage of the most recent forward/backward; -1 for stages not run.
    // The caller must have synchronised the stream.
    for (int i = 0; i < n && i < ST_COUNT; ++i) {
        ms[i] = -1.f;
        if (g_prof_on && g_prof_ev_ok && g_prof_used[i]) {
            float t = 0.f;
            if (cudaEventElapsedTime(&t, g_prof_ev[i][0], g_prof_ev[i][1]) == cudaSuccess) ms[i] = t;
        }
    }
    return 0;
}
unsigned long long gsr_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
const char* gsr_last_error(void) { return g_err; }

int gsr_forward_sizes(int P, int M, int W, int H, size_t* geom_bytes, size_t* img_bytes) {
    if (P < 0 || W <= 0 || H <= 0 || M < 0) { set_error("bad sizes"); return GSR_E_INVALID; }
    if (geom_bytes) *geom_bytes = carve_geom(nullptr, P, M, nullptr);
    if (img_bytes) *img_bytes = carve_img(nullptr, W, H, nullptr);
    return 0;
}

int gsr_binning_sizes(int P, int W, int H, int num_rendered, int num_coarse, size_t* binning_bytes, size_t* scratch_bytes) {
    (void)P;
    if (num_rendered < 0 || num_coarse < 0 || W <= 0 || H <= 0) { set_error("bad sizes"); return GSR_E_INVALID; }
    if (binning_bytes) *binning_bytes = carve_bin(nullptr, (size_t)num_rendered, nullptr);
    if (scratch_bytes) *scratch_bytes = carve_bin_scratch(nullptr, (size_t)num_coarse, W, H, nullptr);
    return 0;
}

// projection, depth ordering (compacting away everything that is culled or outside the band) and coarse-item offsets;
// leaves R (exact), N1 and the number of sorted Gaussians in g.counters.  No host synchronisation.
static int geometry_stage(const GsrForwardArgs* a, const GeomState& g, int ty0, int ty1, cudaStream_t s) {
    const bool dbg = a->debug != 0;
    GSR_CUDA(cudaMemsetAsync(g.counters, 0, 8 * sizeof(int32_t), s));
    prof_begin(ST_PREPROCESS_FWD, s);
    int rc = launch_preprocess_fwd(*a, g, ty0, ty1, s);
    if (rc) return rc;
    GSR_STAGE(s, dbg, "preprocess_fwd_kernel");
    prof_end(ST_PREPROCESS_FWD, s);

    // front-to-back order of the Gaussians: stable sort on the depth bits (all 32, u32 compare like the reference's
    // key, rasterizer_impl.cu:104).  The first pass drops the Gaussians that are culled or do not meet this rank's
    // tile-row band (key = RADIX_DROP_KEY): the later passes, the scan and the emission only see the survivors, whose
    // number stays on the device (counters[5]).
    prof_begin(ST_DEPTH_SORT, s);
    // the last pass also gathers cells_touched and the tile rectangles into depth order (own arrays: the pass
    // reads key_b / val_b and writes key_a / val_a, nothing may alias those while it runs)
    RadixAux aux;
    aux.in32 = g.cells_touched;
    aux.out32 = g.cells_sorted;
    aux.in64 = reinterpret_cast<const uint2*>(g.rect);
    aux.out64 = reinterpret_cast<uint2*>(g.rect_sorted);
    uint32_t* n_sorted = reinterpret_cast<uint32_t*>(g.counters + 5);
    rc = radix_sort_pairs(g.key_a, g.val_a, g.key_b, g.val_b, (size_t)a->P, 0, 32, g.radix_tmp, s, dbg, &aux, nullptr, n_sorted);
    if (rc) return rc;
    prof_end(ST_DEPTH_SORT, s);

    // coarse-item offsets in depth order; the total (number of coarse items) goes to counters[4]
    prof_begin(ST_OFFSET_SCAN, s);
    rc = exclusive_scan_u32(g.cells_sorted, g.offsets, (size_t)a->P, g.radix_tmp + radix_tmp_elems((size_t)a->P), s,
                            n_sorted, reinterpret_cast<uint32_t*>(g.counters + 4));
    if (rc) return rc;
    GSR_STAGE(s, dbg, "exclusive_scan_u32");
    prof_end(ST_OFFSET_SCAN, s);
    return 0;
}

// synchronising read-back of the counters.  NOT a cudaMemcpy: a device-to-host copy would queue on the D2H copy engine behind
// whatever another stream is reading back at that moment (a host-buffer pipeline reads 229 MB of gradients per step: the
// 32-byte copy then waits ~4 ms and the forward with it).  A one-warp kernel stores the eight counters straight into mapped
// pinned host memory instead (SM stores over PCIe, no copy engine); one buffer per host thread, never freed.
__global__ void counters_to_host_kernel(const int32_t* __restrict__ counters, volatile int32_t* __restrict__ host) {
    if (threadIdx.x < 8) host[threadIdx.x] = counters[threadIdx.x];
    __threadfence_system();
}

static int read_counters(const GeomState& g, cudaStream_t s, int32_t out[8]) {
    static thread_local int32_t* h_counts = nullptr;
    static thread_local int32_t* d_alias = nullptr;
    if (!h_counts) {
        GSR_CUDA(cudaHostAlloc((void**)&h_counts, 8 * sizeof(int32_t), cudaHostAllocMapped | cudaHostAllocPortable));
        GSR_CUDA(cudaHostGetDevicePointer((void**)&d_alias, h_counts, 0));
    }
    counters_to_host_kernel<<<1, 32, 0, s>>>(g.counters, d_alias);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    GSR_CUDA(cudaStreamSynchronize(s));
    memcpy(out, h_counts, 8 * sizeof(int32_t));
    return 0;
}

static int counts_of(const int32_t c[8], int* num_rendered, int* num_coarse) {
    if (c[0] != 0) {
        set_error("Point is filtered although prefiltered is set. This shouldn't happen!");
        return GSR_E_PREFILTERED;
    }
    unsigned long long R = 0;
    memcpy(&R, &c[2], sizeof(R));
    const uint32_t N1 = (uint32_t)c[4];
    if (R > 0x7FFFFFFFull || N1 > 0x7FFFFFFFu) { set_error("instance count %llu overflows int", R); return GSR_E_OVERFLOW; }
    *num_rendered = (int)R;
    *num_coarse = (int)N1;
    return 0;
}

static int binning_and_render(const GsrForwardArgs* a, const GeomState& g, const ImgState& im, const BinState& b,
                              const BinScratch& bs, size_t R_cap, size_t N1_cap, int ty0, int ty1, cudaStream_t s) {
    const bool dbg = a->debug != 0;
    int rc = run_tile_binning(g, a->P, a->W, a->H, R_cap, N1_cap, bs, b.point_list, im.ranges, s, dbg);
    if (rc) return rc;
    const float* colors = a->colors_precomp ? a->colors_precomp : g.rgb;
    prof_begin(ST_RENDER_FWD, s);
    rc = launch_render_fwd(*a, g, b, im, colors, ty0, ty1, s);
    if (rc) return rc;
    GSR_STAGE(s, dbg, "render_fwd_packed_kernel");
    prof_end(ST_RENDER_FWD, s);
    return 0;
}

int gsr_forward_geometry(const GsrForwardArgs* a, void* geom_buffer, void* img_buffer, void* stream, int* num_rendered,
                         int* num_coarse) {
    (void)img_buffer;
    int rc = check_fwd_args(a);
    if (rc) return rc;
    if (!num_rendered || !num_coarse) { set_error("num_rendered / num_coarse is NULL"); return GSR_E_INVALID; }
    *num_rendered = 0;
    *num_coarse = 0;
    if (a->P == 0) return 0;
    if (!geom_buffer) { set_error("geom_buffer is NULL"); return GSR_E_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    GeomState g;
    carve_geom((char*)geom_buffer, a->P, a->M, &g);
    int ty0, ty1;
    shard_rows(a->H, a->tile_y0, a->tile_y1, &ty0, &ty1);
    rc = geometry_stage(a, g, ty0, ty1, s);
    if (rc) return rc;
    int32_t c[8];
    rc = read_counters(g, s, c);
    if (rc) return rc;
    return counts_of(c, num_rendered, num_coarse);
}

int gsr_forward_render(const GsrForwardArgs* a, void* geom_buffer, void* img_buffer, void* binning_buffer, void* scratch,
                       int num_rendered, int num_coarse, void* stream) {
    int rc = check_fwd_args(a);
    if (rc) return rc;
    if (a->P == 0) return 0;
    if (!geom_buffer || !img_buffer || (num_rendered > 0 && (!binning_buffer || !scratch))) {
        set_error("a buffer is NULL");
        return GSR_E_INVALID;
    }
    GeomState g;
    ImgState im;
    BinState b;
    BinScratch bs;
    carve_geom((char*)geom_buffer, a->P, a->M, &g);
    carve_img((char*)img_buffer, a->W, a->H, &im);
    carve_bin((char*)binning_buffer, (size_t)num_rendered, &b);
    carve_bin_scratch((char*)scratch, (size_t)num_coarse, a->W, a->H, &bs);
    int ty0, ty1;
    shard_rows(a->H, a->tile_y0, a->tile_y1, &ty0, &ty1);
    return binning_and_render(a, g, im, b, bs, (size_t)num_rendered, (size_t)num_coarse, ty0, ty1, (cudaStream_t)stream);
}

int gsr_forward(const GsrForwardArgs* a, gsr_alloc_fn alloc, void* ctx, void* stream, int* num_rendered) {
    int rc = check_fwd_args(a);
    if (rc) return rc;
    if (!alloc || !num_rendered) { set_error("alloc / num_rendered is NULL"); return GSR_E_INVALID; }
    size_t gb = 0, ib = 0, bb = 0, sb = 0;
    rc = gsr_forward_sizes(a->P, a->M, a->W, a->H, &gb, &ib);
    if (rc) return rc;
    void* geom = alloc(ctx, GSR_BUF_GEOM, gb);
    void* img = alloc(ctx, GSR_BUF_IMG, ib);
    if (!geom || !img) { set_error("allocation callback returned NULL"); return GSR_E_INVALID; }
    int num_coarse = 0;
    rc = gsr_forward_geometry(a, geom, img, stream, num_rendered, &num_coarse);
    if (rc) return rc;
    rc = gsr_binning_sizes(a->P, a->W, a->H, *num_rendered, num_coarse, &bb, &sb);
    if (rc) return rc;
    void* bin = alloc(ctx, GSR_BUF_BINNING, bb);
    void* scr = alloc(ctx, GSR_BUF_SCRATCH, sb);
    if (!bin || !scr) { set_error("allocation callback returned NULL"); return GSR_E_INVALID; }
    return gsr_forward_render(a, geom, img, bin, scr, *num_rendered, num_coarse, stream);
}

int gsr_forward_recolor(const GsrForwardArgs* a, const void* geom_buffer, const void* binning_buffer,
                        const void* img_buffer, void* img_buffer2, void* stream) {
    int rc = check_fwd_args(a);
    if (rc) return rc;
    if (a->P == 0) return 0;
    if (!a->colors_precomp) { set_error("gsr_forward_recolor needs colors_precomp"); return GSR_E_INVALID; }
    if (!geom_buffer || !binning_buffer || !img_buffer || !img_buffer2) { set_error("a buffer is NULL"); return GSR_E_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    GeomState g;
    ImgState im, im2;
    BinState b;
    carve_geom((char*)geom_buffer, a->P, a->M, &g);
    carve_img((char*)img_buffer, a->W, a->H, &im);
    carve_img((char*)img_buffer2, a->W, a->H, &im2);
    // R is only needed for carving offsets inside the binning buffer: point_list is first
    carve_bin((char*)binning_buffer, 0, &b);
    int ty0, ty1;
    shard_rows(a->H, a->tile_y0, a->tile_y1, &ty0, &ty1);
    const size_t T = (size_t)tiles_x(a->W) * tiles_y(a->H);
    if (im2.ranges != im.ranges)
        GSR_CUDA(cudaMemcpyAsync(im2.ranges, im.ranges, T * sizeof(uint2), cudaMemcpyDeviceToDevice, s));
    prof_begin(ST_RENDER_FWD, s);
    rc = launch_render_fwd(*a, g, b, im2, a->colors_precomp, ty0, ty1, s);
    if (rc) return rc;
    GSR_STAGE(s, a->debug != 0, "render_fwd_packed_kernel(recolor)");
    prof_end(ST_RENDER_FWD, s);
    return 0;
}

int gsr_forward_display(const GsrForwardArgs* a, const GsrDisplayArgs* d, void* geom_buffer, void* img_buffer,
                        void* binning_buffer, void* scratch, int num_rendered, int num_coarse, void* stream) {
    if (!a || !d) { set_error("args / display is NULL"); return GSR_E_INVALID; }
    GsrForwardArgs c = *a;
    c.out_color = d->out_color;             // the display image stands in for out_color in the common checks
    int rc = check_fwd_args(&c);
    if (rc) return rc;
    if (a->tile_y0 != 0 || a->tile_y1 != 0) { set_error("the display composite renders the whole image: tile-row shard set"); return GSR_E_INVALID; }
    if (a->peer_images || a->n_peer_images) { set_error("the display composite takes no peer images"); return GSR_E_INVALID; }
    if (num_rendered < 0 || num_coarse < 0) { set_error("bad counts"); return GSR_E_INVALID; }
    if (a->P == 0) return 0;
    if (!d->out_color || !d->out_accum) { set_error("out_color / out_accum is NULL"); return GSR_E_INVALID; }
    if (d->depth && !d->out_depth) { set_error("depth requested but out_depth is NULL"); return GSR_E_INVALID; }
    if (d->depth && !d->depth_values && (!d->depth_scratch || !a->campos)) {
        set_error("camera distances need depth_scratch and campos");
        return GSR_E_INVALID;
    }
    if (!geom_buffer || !img_buffer || (num_rendered > 0 && (!binning_buffer || !scratch))) {
        set_error("a buffer is NULL");
        return GSR_E_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const bool dbg = a->debug != 0;
    GeomState g;
    ImgState im;
    BinState b;
    BinScratch bs;
    carve_geom((char*)geom_buffer, a->P, a->M, &g);
    carve_img((char*)img_buffer, a->W, a->H, &im);
    carve_bin((char*)binning_buffer, (size_t)num_rendered, &b);
    carve_bin_scratch((char*)scratch, (size_t)num_coarse, a->W, a->H, &bs);
    const float* depth_values = d->depth_values;
    if (d->depth && !depth_values) {
        rc = launch_camera_distance(a->P, a->means3D, a->campos, d->depth_scratch, s);
        if (rc) return rc;
        GSR_STAGE(s, dbg, "camera_distance_kernel");
        depth_values = d->depth_scratch;
    }
    rc = run_tile_binning(g, a->P, a->W, a->H, (size_t)num_rendered, (size_t)num_coarse, bs, b.point_list, im.ranges, s, dbg);
    if (rc) return rc;
    prof_begin(ST_RENDER_FWD, s);
    rc = launch_render_display(*a, *d, g, b, im, a->colors_precomp ? a->colors_precomp : g.rgb, depth_values, s);
    if (rc) return rc;
    GSR_STAGE(s, dbg, "render_fwd_packed_kernel(display)");
    prof_end(ST_RENDER_FWD, s);
    return 0;
}

size_t gsr_backward_scratch_bytes(int P) { return (size_t)(P > 0 ? P : 0) * sizeof(BwdAccum) + 256; }

int gsr_backward_deterministic_sizes(int P, int R, size_t* scratch_bytes, size_t* mark_bytes) {
    if (P < 0 || R < 0) { set_error("bad sizes"); return GSR_E_INVALID; }
    if (scratch_bytes) *scratch_bytes = carve_det(nullptr, P, (size_t)R, nullptr, nullptr);
    if (mark_bytes) *mark_bytes = det_mark_bytes((size_t)R);
    return 0;
}

static int check_bwd_args(const GsrBackwardArgs* a, bool need_pix, bool need_outputs) {
    if (!a) { set_error("args is NULL"); return GSR_E_INVALID; }
    if (a->P < 0 || a->W <= 0 || a->H <= 0 || a->R < 0) { set_error("bad sizes"); return GSR_E_INVALID; }
    if (a->P == 0) return 0;
    if (!a->means3D || !a->radii || !a->viewmatrix || !a->projmatrix || !a->geom_buffer || !a->accum_scratch) {
        set_error("a required pointer is NULL");
        return GSR_E_INVALID;
    }
    if (need_pix) {
        if (!a->background || !a->subpixel_offset || !a->img_buffer || !a->dL_dpix) { set_error("a required pointer is NULL"); return GSR_E_INVALID; }
        if (a->R > 0 && !a->binning_buffer) { set_error("binning_buffer is NULL"); return GSR_E_INVALID; }
    }
    if (need_outputs) {
        if (!a->dL_dmean2D || !a->dL_dopacity || !a->dL_dcolor || !a->dL_dmean3D) { set_error("a required output pointer is NULL"); return GSR_E_INVALID; }
        if (a->shs && (!a->dL_dsh || !a->campos || a->M <= 0)) { set_error("shs given but dL_dsh / campos missing"); return GSR_E_INVALID; }
        if (a->scales && (!a->rotations || !a->dL_dscale || !a->dL_drot)) { set_error("scales given but rotations / dL_dscale / dL_drot missing"); return GSR_E_INVALID; }
        if (!a->scales && !a->cov3D_precomp) { set_error("neither scales nor cov3D_precomp"); return GSR_E_INVALID; }
    }
    return 0;
}

// slots of the deterministic reductions, with base = exclusive scan of tiles_touched enqueued on s
static int det_slots_of(const GsrBackwardArgs* a, const GeomState& g, cudaStream_t s, DetSlots* det) {
    if (!a->det_scratch || !a->det_marks) { set_error("deterministic: det_scratch / det_marks is NULL"); return GSR_E_INVALID; }
    uint32_t* tmp;
    carve_det((char*)a->det_scratch, a->P, (size_t)a->R, det, &tmp);
    det->rect = g.rect;
    det->marks = reinterpret_cast<uint32_t*>(a->det_marks);
    return exclusive_scan_u32(g.tiles_touched, const_cast<uint32_t*>(det->base), (size_t)a->P, tmp, s);
}

static BwdAccum* accum_of(const GsrBackwardArgs* a) {
    char* cur = (char*)a->accum_scratch;
    BwdAccum* accum;
    take(cur, accum, (size_t)a->P);
    return accum;
}

static int backward_partials_impl(const GsrBackwardArgs* a, void* stream, const PeerAccum* peer, unsigned char* touched = nullptr) {
    int rc = check_bwd_args(a, true, false);
    if (rc || a->P == 0) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const bool dbg = a->debug != 0;
    GeomState g;
    ImgState im;
    BinState b;
    carve_geom((char*)a->geom_buffer, a->P, a->M, &g);
    carve_img((char*)a->img_buffer, a->W, a->H, &im);
    carve_bin((char*)a->binning_buffer, (size_t)a->R, &b);
    int ty0, ty1;
    shard_rows(a->H, a->tile_y0, a->tile_y1, &ty0, &ty1);
    BwdAccum* accum = accum_of(a);
    const bool det = a->deterministic != 0;
    if (det && (peer || touched)) {
        set_error("the multi-GPU backward reductions have no deterministic form");
        return GSR_E_INVALID;
    }
    // with peer accumulators the caller zeroes them (all ranks, then a barrier) before any rank adds into them
    if (!peer && !a->accum_is_zero) GSR_CUDA(cudaMemsetAsync(accum, 0, (size_t)a->P * sizeof(BwdAccum), s));
    const float* colors = a->colors_precomp ? a->colors_precomp : g.rgb;
    if (a->R > 0) {
        DetSlots slots;
        if (det) {
            rc = det_slots_of(a, g, s, &slots);
            if (rc) return rc;
        }
        prof_begin(ST_RENDER_BWD, s);
        rc = launch_render_bwd(*a, g, b, im, colors, accum, ty0, ty1, s, peer, touched, det ? &slots : nullptr);
        if (rc) return rc;
        GSR_STAGE(s, dbg, "render_bwd_packed_kernel");
        if (det) {
            rc = launch_det_gather_accum(a->P, g, slots, accum, s);
            if (rc) return rc;
            GSR_STAGE(s, dbg, "det_gather_accum_kernel");
        }
        prof_end(ST_RENDER_BWD, s);
    }
    return 0;
}

int gsr_backward_partials(const GsrBackwardArgs* a, void* stream) { return backward_partials_impl(a, stream, nullptr); }

int gsr_backward_partials_peers(const GsrBackwardArgs* a, const void* const* peer_accum_dev, int n_peers,
                                void* multicast_accum, void* stream) {
    if ((!peer_accum_dev || n_peers <= 0) && !multicast_accum) {
        set_error("gsr_backward_partials_peers needs peer pointers or a multicast address");
        return GSR_E_INVALID;
    }
    PeerAccum peer;
    peer.peers = multicast_accum ? nullptr : peer_accum_dev;
    peer.n_peers = multicast_accum ? 0 : n_peers;
    peer.multicast = multicast_accum;
    return backward_partials_impl(a, stream, &peer);
}

int gsr_backward_partials_marked(const GsrBackwardArgs* a, unsigned char* touched, void* stream) {
    if (!touched) { set_error("touched is NULL"); return GSR_E_INVALID; }
    if (a && !a->accum_is_zero) { set_error("gsr_backward_partials_marked needs accum_is_zero (the pull-mode buffers are kept zero)"); return GSR_E_INVALID; }
    return backward_partials_impl(a, stream, nullptr, touched);
}

int gsr_backward_finalize_pull(const GsrBackwardArgs* a, const void* const* peer_accum_dev, const void* const* peer_touched_dev,
                               int n_peers, int self, void* clear_accum, unsigned char* clear_touched, void* stream) {
    int rc = check_bwd_args(a, false, true);
    if (rc || a->P == 0) return rc;
    if (!peer_accum_dev || !peer_touched_dev || n_peers <= 0 || n_peers > GSR_MAX_PULL_PEERS || self < 0 || self >= n_peers ||
        ((clear_accum == nullptr) != (clear_touched == nullptr))) {
        set_error("gsr_backward_finalize_pull: bad peer arguments");
        return GSR_E_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    GeomState g;
    carve_geom((char*)a->geom_buffer, a->P, a->M, &g);
    PullPeers pull;
    pull.accums = reinterpret_cast<const float* const*>(peer_accum_dev);
    pull.touched = reinterpret_cast<const unsigned char* const*>(peer_touched_dev);
    pull.n_peers = n_peers; pull.self = self;
    pull.clear_accum = reinterpret_cast<float*>(clear_accum); pull.clear_touched = clear_touched;
    prof_begin(ST_PREPROCESS_BWD, s);
    rc = launch_preprocess_bwd(*a, g, accum_of(a), s, &pull);
    if (rc) return rc;
    GSR_STAGE(s, a->debug != 0, "preprocess_bwd_kernel");
    prof_end(ST_PREPROCESS_BWD, s);
    return 0;     // nothing is cleared here: this pass's buffers are zeroed by the NEXT pass's call (see gsrast.h)
}

int gsr_backward_finalize(const GsrBackwardArgs* a, void* stream) {
    int rc = check_bwd_args(a, false, true);
    if (rc || a->P == 0) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    GeomState g;
    carve_geom((char*)a->geom_buffer, a->P, a->M, &g);
    prof_begin(ST_PREPROCESS_BWD, s);
    rc = launch_preprocess_bwd(*a, g, accum_of(a), s);
    if (rc) return rc;
    GSR_STAGE(s, a->debug != 0, "preprocess_bwd_kernel");
    prof_end(ST_PREPROCESS_BWD, s);
    // the kernel left the accumulator zeroed for the next backward pass: a caller that keeps the buffer passes
    // accum_is_zero = 1 next time, and the tile-row sharded path needs no fill + barrier in front of its peer reductions.
    // It clears only the rows it found non-zero (the Gaussians some pixel blended: 10-20 % of a dense scene; clearing ALL
    // rows in the kernel was measured 3.5x slower than the kernel + a memset).
    return 0;
}

int gsr_backward(const GsrBackwardArgs* a, void* stream) {
    int rc = check_bwd_args(a, true, true);
    if (rc || a->P == 0) return rc;
    rc = gsr_backward_partials(a, stream);
    if (rc) return rc;
    return gsr_backward_finalize(a, stream);
}

int gsr_backward_colors(const GsrBackwardArgs* a, void* stream) {
    if (!a) { set_error("args is NULL"); return GSR_E_INVALID; }
    if (a->P < 0 || a->M < 0 || a->W <= 0 || a->H <= 0 || a->R < 0) { set_error("bad sizes"); return GSR_E_INVALID; }
    if (a->P == 0) return 0;
    if (!a->geom_buffer || !a->img_buffer || !a->subpixel_offset || !a->dL_dpix || !a->dL_dcolor ||
        (a->R > 0 && !a->binning_buffer)) {
        set_error("a required pointer is NULL");
        return GSR_E_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const bool det = a->deterministic != 0 && a->R > 0;     // the gather writes every row of dL_dcolor
    if (!det) GSR_CUDA(cudaMemsetAsync(a->dL_dcolor, 0, (size_t)a->P * 3 * sizeof(float), s));
    if (a->R == 0) return 0;
    GeomState g;
    ImgState im;
    BinState b;
    carve_geom((char*)a->geom_buffer, a->P, a->M, &g);
    carve_img((char*)a->img_buffer, a->W, a->H, &im);
    carve_bin((char*)a->binning_buffer, (size_t)a->R, &b);
    int ty0, ty1;
    shard_rows(a->H, a->tile_y0, a->tile_y1, &ty0, &ty1);
    DetSlots slots;
    int rc = 0;
    if (det) {
        rc = det_slots_of(a, g, s, &slots);
        if (rc) return rc;
    }
    rc = launch_render_color_grad(*a, g, b, im, ty0, ty1, s, det ? &slots : nullptr);
    if (rc) return rc;
    GSR_STAGE(s, a->debug != 0, "render_color_grad_kernel");
    if (det) {
        rc = launch_det_gather_color(a->P, g, slots, a->dL_dcolor, s);
        if (rc) return rc;
        GSR_STAGE(s, a->debug != 0, "det_gather_color_kernel");
    }
    return 0;
}

int gsr_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix, uint8_t* present,
                     void* stream) {
    (void)projmatrix;
    if (P < 0) { set_error("bad P"); return GSR_E_INVALID; }
    if (P == 0) return 0;
    if (!means3D || !viewmatrix || !present) { set_error("a required pointer is NULL"); return GSR_E_INVALID; }
    int rc = launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)stream);
    if (rc) return rc;
    GSR_CUDA(cudaGetLastError());
    return 0;
}

int gsr_img_views(const void* img_buffer, int W, int H, const float** final_T, const uint32_t** n_contrib,
                  const uint32_t** ranges) {
    if (!img_buffer) { set_error("img_buffer is NULL"); return GSR_E_INVALID; }
    ImgState im;
    carve_img((char*)img_buffer, W, H, &im);
    if (final_T) *final_T = im.final_T;
    if (n_contrib) *n_contrib = im.n_contrib;
    if (ranges) *ranges = reinterpret_cast<const uint32_t*>(im.ranges);
    return 0;
}

int gsr_binning_views(const void* binning_buffer, int num_rendered, const uint32_t** point_list) {
    if (!binning_buffer) { set_error("binning_buffer is NULL"); return GSR_E_INVALID; }
    BinState b;
    carve_bin((char*)binning_buffer, (size_t)num_rendered, &b);
    if (point_list) *point_list = b.point_list;
    return 0;
}

int gsr_geom_views(const void* geom_buffer, int P, int M, const float** depths, const float** records,
                   const uint32_t** tiles_touched, const float** rgb) {
    if (!geom_buffer) { set_error("geom_buffer is NULL"); return GSR_E_INVALID; }
    GeomState g;
    carve_geom((char*)geom_buffer, P, M, &g);
    if (depths) *depths = g.depths;
    if (records) *records = reinterpret_cast<const float*>(g.rec);
    if (tiles_touched) *tiles_touched = g.tiles_touched;
    if (rgb) *rgb = g.rgb;
    return 0;
}

int gsr_get_stats(const void* geom_buffer, int P, int M, void* stream, GsrStats* out) {
    if (!geom_buffer || !out) { set_error("NULL argument"); return GSR_E_INVALID; }
    GeomState g;
    carve_geom((char*)geom_buffer, P, M, &g);
    int32_t c[8];
    int rc = read_counters(g, (cudaStream_t)stream, c);
    if (rc) return rc;
    out->num_visible = c[1];
    out->num_rendered = c[2];   // low word of the 64-bit instance counter
    out->num_tiles = 0;
    out->num_coarse = c[4];
    return 0;
}

}  // extern "C"

namespace gsr {

__global__ void __launch_bounds__(256) mark_visible_kernel(int P, const float* __restrict__ means3D,
                                                           const float* __restrict__ view, uint8_t* __restrict__ present) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const float x = means3D[3 * idx], y = means3D[3 * idx + 1], z = means3D[3 * idx + 2];
    const float vz = view[2] * x + view[6] * y + view[10] * z + view[14];
    present[idx] = vz <= NEAR_Z ? 0 : 1;
}

int launch_mark_visible(int P, const float* means3D, const float* view, uint8_t* present, cudaStream_t s) {
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, means3D, view, present);
    count_launches(1);
    return 0;
}

}  // namespace gsr
