// common.cuh -- shared declarations of libgsrast (sm_90a Gaussian-splat rasterizer).
// Internal header: the public boundary is include/gsrast.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include "gsrast.h"

namespace gsr {

constexpr int TILE = 16;              // tile edge in pixels (reference config.h:16-17)
constexpr int TILE_PIX = TILE * TILE;
constexpr int CELL = 8;               // binning cell edge in tiles (binning.cu)
constexpr int CELL_TILES = CELL * CELL;
constexpr int UNIT = 256;             // coarse items per binning unit (one warp)
constexpr float NEAR_Z = 0.2f;        // near cull (reference auxiliary.h:154)

// ----------------------------------------------------------------------------------------
// error plumbing
// ----------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
void count_launches(int n);   // kernels launched by this library (bench.py's gpu_launches)

// optional per-stage device timing (api.cu); no-ops unless gsr_profile_enable(1)
enum Stage { ST_PREPROCESS_FWD = 0, ST_DEPTH_SORT, ST_OFFSET_SCAN, ST_EMIT_CELLS, ST_CELL_SORT, ST_CELL_COUNT,
             ST_TILE_OFFSETS, ST_TILE_SCATTER, ST_RENDER_FWD, ST_RENDER_BWD, ST_PREPROCESS_BWD, ST_COUNT };
void prof_begin(int stage, cudaStream_t s);
void prof_end(int stage, cudaStream_t s);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define GSR_CUDA(expr)                                                        \
    do {                                                                      \
        cudaError_t _e = (expr);                                              \
        if (_e != cudaSuccess) return gsr::cuda_fail(_e, #expr, __FILE__, __LINE__); \
    } while (0)

// launch check; with debug also synchronises the stream (reference CHECK_CUDA, auxiliary.h:166-173)
#define GSR_STAGE(stream, debug, name)                                        \
    do {                                                                      \
        cudaError_t _e = cudaGetLastError();                                  \
        if (_e == cudaSuccess && (debug)) _e = cudaStreamSynchronize(stream); \
        if (_e != cudaSuccess) return gsr::cuda_fail(_e, name, __FILE__, __LINE__); \
    } while (0)

// ----------------------------------------------------------------------------------------
// buffer layouts (carved out of the caller's opaque byte buffers)
// ----------------------------------------------------------------------------------------
struct TileRect { uint16_t x0, y0, x1, y1; };   // half-open tile rectangle of one Gaussian

struct GeomState {
    // persistent (read by the backward pass)
    float4*   rec;            // [2P] {x, y, hx, hy | conic.x, conic.y, conic.z, opacity*coef}
    float*    rgb;            // [3P] SH-evaluated colours (SH path only)
    uint8_t*  clamped;        // [P]  bit c set: channel c was clamped to 0 (SH path only)
    float*    depths;         // [P]  view-space z (exported for parity tests)
    uint32_t* tiles_touched;  // [P]
    uint32_t* cells_touched;  // [P]  binning cells (8x8 tiles) overlapped by the tile rectangle
    TileRect* rect;           // [P]
    int32_t*  counters;       // [8]  0: prefiltered violation, 1: visible count, 2-3: R (u64), 4: coarse items
    // transient (depth ordering + instance offsets)
    uint32_t* key_a;          // [P]
    uint32_t* key_b;          // [P]
    uint32_t* val_a;          // [P]
    uint32_t* val_b;          // [P]
    uint32_t* order;          // alias of val_a: after the 4-pass depth sort, Gaussian ids front to back
    uint32_t* cells_sorted;   // [P]  cells_touched in depth order (written by the last sort pass)
    TileRect* rect_sorted;    // [P]  tile rectangles in depth order (written by the last sort pass)
    uint32_t* offsets;        // [P+1] exclusive scan of cells_touched in depth order
    uint32_t* radix_tmp;      // histogram / scan temporaries
};

// Blend masks: the forward records, for each tile, each 8x8 pixel block of the tile (in the packed kernels' warp
// order: block k covers pixels [8 (k % 2), +8) x [8 (k / 2), +8)) and each of the first MASK_K positions of the
// tile's list, whether some pixel of the block blended that position.  Bit b of word w is position 32 w + b.  The
// backward walks only the set bits; positions at or above MASK_K are culled by the footprint box instead.
constexpr int MASK_K = 1024;
constexpr int MASK_WORDS = MASK_K / 32;   // words per (tile, block)
constexpr int MASK_BLOCKS = 4;            // 8x8 blocks per tile

struct ImgState {
    float*    final_T;        // [N]  first, 128-B aligned (reference ImageState order)
    uint32_t* n_contrib;      // [N]
    uint2*    ranges;         // [T]
    uint32_t* blend_mask;     // [T][MASK_BLOCKS][MASK_WORDS]; only the words below the block's largest n_contrib are
                              // defined (the forward walked those batches with some pixel of the block compositing)
};

struct BinState {
    uint32_t* point_list;     // [R] sorted Gaussian ids (tile-major, depth-minor)
};

struct BinScratch {           // transient state of the two-level tile binning (binning.cu)
    uint32_t* key_a;          // [N1] coarse items: cell id | local rect
    uint32_t* val_a;          // [N1] Gaussian ids
    uint32_t* key_b;          // [N1]
    uint32_t* val_b;          // [N1]
    uint32_t* radix_tmp;
    uint2*    cell_range;     // [NC]
    uint32_t* unit_base;      // [NC+1]
    size_t    units_cap;      // upper bound of the number of units: N1 / UNIT + NC, rounded up to 8
    uint32_t* M;              // [64][units_cap] per-(local tile, unit) counts, then their row-wise prefix
    uint32_t* row_total;      // [64]
    uint32_t* tile_start;     // [T+1]
    unsigned long long* block_sums;   // [ceil(T / 1024)] per-CTA tile totals of tile_offsets_lookback_kernel
};

size_t carve_geom(char* base, int P, int M, GeomState* out);       // returns bytes used
size_t carve_img(char* base, int W, int H, ImgState* out);
size_t carve_bin(char* base, size_t R, BinState* out);
size_t carve_bin_scratch(char* base, size_t N1, int W, int H, BinScratch* out);

inline int tiles_x(int W) { return (W + TILE - 1) / TILE; }
inline int tiles_y(int H) { return (H + TILE - 1) / TILE; }

// ----------------------------------------------------------------------------------------
// stage launchers (each enqueues on `stream`, returns 0 or a status code)
// ----------------------------------------------------------------------------------------
int launch_preprocess_fwd(const GsrForwardArgs& a, const GeomState& g, int ty0, int ty1, cudaStream_t s);

// stable LSD radix partition of (key,val) pairs on key bits [shift, shift+bits)
size_t radix_tmp_elems(size_t n);
int radix_num_passes(int begin_bit, int end_bit);
// input in (key_a,val_a); result in A if radix_num_passes() is even, else in B; both clobbered
// optional side data delivered in sorted order by the LAST pass: out32[pos] = in32[val], out64[pos] = in64[val]
struct RadixAux {
    const uint32_t* in32;
    uint32_t* out32;
    const uint2* in64;
    uint2* out64;
};
// n_cap sizes the grids; with n_dev the item count is min(*n_dev, n_cap) (device side).  With n_compact the first pass
// drops the items whose key is RADIX_DROP_KEY and stores the number of remaining items in *n_compact.
constexpr uint32_t RADIX_DROP_KEY = 0xFFFFFFFFu;
int radix_sort_pairs(uint32_t* key_a, uint32_t* val_a, uint32_t* key_b, uint32_t* val_b, size_t n_cap,
                     int begin_bit, int end_bit, uint32_t* tmp, cudaStream_t s, bool debug, const RadixAux* aux = nullptr,
                     const uint32_t* n_dev = nullptr, uint32_t* n_compact = nullptr);
// digit totals (RADIX entries) left in `tmp` by the most recent pass of radix_sort_pairs over n items
const uint32_t* radix_pass_totals(const uint32_t* tmp, size_t n);
// exclusive scan of counts: out[i] = sum_{j<i} counts[j], out[n] = total
int exclusive_scan_u32(const uint32_t* counts, uint32_t* out, size_t n_cap, uint32_t* tmp, cudaStream_t s,
                       const uint32_t* n_dev = nullptr, uint32_t* total_out = nullptr);
size_t scan_tmp_elems(size_t n);

// in-place exclusive scan along each row of a [rows][cols] u32 matrix; row sums -> total[rows]
int row_scan_u32(uint32_t* m, int rows, size_t cols, uint32_t* total, cudaStream_t s);

// inclusive prefix sum over the 32 lanes of a warp; every lane of the warp must call it
__device__ __forceinline__ uint32_t warp_inclusive_scan(uint32_t x) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
        if (lane >= o) x += y;
    }
    return x;
}

// Deterministic block sum of N doubles per thread over a THREADS-thread block: warp shuffles, then the warps in order.
// Result in thread 0.  sh: [THREADS / 32][N] shared doubles.
template <int THREADS, int N>
__device__ __forceinline__ void block_sum_f64(double (&v)[N], double (*sh)[N]) {
#pragma unroll
    for (int k = 0; k < N; ++k)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < N; ++k) sh[warp][k] = v[k];
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < THREADS / 32; ++w)
#pragma unroll
            for (int k = 0; k < N; ++k) v[k] += sh[w][k];
}

// per-tile instance lists + ranges from the depth-ordered Gaussians (binning.cu)
int run_tile_binning(const GeomState& g, int P, int W, int H, size_t R, size_t N1, const BinScratch& bs,
                     uint32_t* point_list, uint2* ranges, cudaStream_t s, bool debug);

int launch_render_fwd(const GsrForwardArgs& a, const GeomState& g, const BinState& b, const ImgState& im,
                      const float* colors, int ty0, int ty1, cudaStream_t s);
// colour-only backward composite (render_fwd.cu): adds sum T alpha dL/dpixel into a.dL_dcolor
int launch_render_color_grad(const GsrBackwardArgs& a, const GeomState& g, const BinState& b, const ImgState& im, int ty0,
                             int ty1, cudaStream_t s);
// display composite of an inference render (render_fwd.cu): the whole image, no backward state, the epilogue of
// GsrDisplayArgs; depth_values [P] is composited as a fourth channel when d.depth != 0
int launch_render_display(const GsrForwardArgs& a, const GsrDisplayArgs& d, const GeomState& g, const BinState& b,
                          const ImgState& im, const float* colors, const float* depth_values, cudaStream_t s);
// dist[i] = |means3D[i] - campos| with torch.norm's operation order (render_fwd.cu)
int launch_camera_distance(int P, const float* means3D, const float* campos, float* dist, cudaStream_t s);

struct BwdAccum { float4 a, b, c; };  // per-Gaussian packed partial gradients (48 B)
// a = {dmean2D.x, dmean2D.y, |dmean2D|, dconic.x}  b = {dconic.y, dconic.w, dopacity, dcolor.r}
// c = {dcolor.g, dcolor.b, -, -}
// accumulators of all ranks (symmetric memory) for the reduction-fused sharded backward; see render_bwd.cu
struct PeerAccum {
    const void* const* peers;   // device array of n_peers device pointers, or NULL
    int n_peers;
    void* multicast;            // multicast address, or NULL
};
int launch_render_bwd(const GsrBackwardArgs& a, const GeomState& g, const BinState& b, const ImgState& im,
                      const float* colors, BwdAccum* accum, int ty0, int ty1, cudaStream_t s,
                      const PeerAccum* peer = nullptr, unsigned char* touched = nullptr);
// pull-mode reduction (render_bwd marks, preprocess_bwd gathers the marked rows of the other ranks): see gsrast.h
struct PullPeers {
    const float* const* accums;          // HOST array [n_peers] of accumulator pointers (peer-mapped device addresses)
    const unsigned char* const* touched; // HOST array [n_peers] of mark arrays
    int n_peers, self;
    float* clear_accum;                  // previous pass's own accumulator / marks to zero, or NULL
    unsigned char* clear_touched;
};
int launch_preprocess_bwd(const GsrBackwardArgs& a, const GeomState& g, BwdAccum* accum, cudaStream_t s,
                          const PullPeers* pull = nullptr);

int launch_mark_visible(int P, const float* means3D, const float* view, uint8_t* present, cudaStream_t s);

}  // namespace gsr
