// binning.cu -- two-level stable tile binning: from the depth-ordered Gaussians to the per-tile,
// front-to-back instance lists (point_list) and tile ranges.  Replaces duplicateWithKeys
// (rasterizer_impl.cu:70-111), the 64-bit radix sort (:303-311) and identifyTileRanges (:116-138,313-320).
//
// The reference materialises R = sum(tiles touched) 96-bit (key, value) pairs and radix-sorts them over
// 41-48 key bits: about 150 bytes of HBM traffic per instance.  The result it needs is much smaller:
// for every tile, the ids of the Gaussians overlapping it, front to back.  Because the Gaussians are
// already in depth order (4 radix passes over P pairs, radix.cu), that list is a *stable partition* of
// the depth-ordered instance stream by tile id, and a stable partition can be built hierarchically
// without ever writing a key per instance:
//
//   level 1  the screen is cut into cells of 8x8 tiles.  Each Gaussian emits one 8-byte coarse item per
//            cell its tile rectangle overlaps (about 2 per Gaussian instead of about 13 tile instances),
//            carrying the cell id and the rectangle clipped to the cell; a stable radix sort on the
//            cell id groups them by cell, depth order preserved inside each cell.
//   level 2  every cell's list is cut into units of 256 coarse items, one warp per unit.  A counting
//            kernel histograms each unit over the cell's 64 tiles; a row scan turns the counts into the
//            exact output position (and run length) of every (unit, tile); the scatter kernel then walks each unit
//            in order: lane l owns the cell's tiles l and l + 32 and appends the ids of the items covering them to
//            its slices of a shared-memory staging buffer, which is finally copied to the tile lists run by run.
//
// The order inside a tile is the order of the coarse items in the cell = depth order, ties by Gaussian
// index (the depth sort is stable) -- exactly the reference's (tile | depth) stable sort (SURVEY.md note
// N4).  Traffic is about 4 bytes per instance (the list itself) plus a few tens of bytes per Gaussian.
// No spin-waits anywhere: every kernel is a plain data-parallel launch.
#include "common.cuh"

namespace gsr {

// ---- level 1: coarse items ------------------------------------------------------------------------
// key = cell id (low 16 bits) | x0 << 16 | y0 << 20 | x1 << 24 | y1 << 28, rectangle local to the cell
// counters (GeomState::counters): [2..3] R = exact instance count of the band (u64, preprocess), [4] N1 = coarse
// items (scan total), [5] number of depth-sorted Gaussians, [7] N1 if the scene fits the counts the binning buffers
// were sized for, else 0 -- the item count every later binning kernel works with.  gsr_forward_render and
// gsr_forward_display take those counts from the caller: counts smaller than the scene's turn the rest of the forward
// into a harmless no-op (empty tile ranges) instead of writing out of bounds.
__global__ void __launch_bounds__(256) emit_cells_kernel(int cells_x, const uint32_t* __restrict__ order,
                                                         const uint32_t* __restrict__ offsets,
                                                         const TileRect* __restrict__ rect,
                                                         uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                         int32_t* __restrict__ counters, uint32_t n1_cap,
                                                         unsigned long long r_cap) {
    const uint32_t n1 = (uint32_t)counters[4];
    const unsigned long long R = *reinterpret_cast<const unsigned long long*>(counters + 2);
    const bool fits = n1 <= n1_cap && R <= r_cap;
    if (blockIdx.x == 0 && threadIdx.x == 0) counters[7] = fits ? (int32_t)n1 : 0;
    if (!fits) return;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;   // position in depth order
    if (i >= (uint32_t)counters[5]) return;
    const uint32_t g = order[i];
    const TileRect r = rect[i];      // rectangles arrive in depth order (gathered by the last sort pass)
    if (r.x1 <= r.x0 || r.y1 <= r.y0) return;
    uint32_t off = offsets[i];
    const int cx0 = r.x0 / CELL, cx1 = (r.x1 - 1) / CELL + 1;
    const int cy0 = r.y0 / CELL, cy1 = (r.y1 - 1) / CELL + 1;
    for (int cy = cy0; cy < cy1; ++cy) {
        const uint32_t ly0 = (uint32_t)max((int)r.y0 - cy * CELL, 0), ly1 = (uint32_t)min((int)r.y1 - cy * CELL, CELL);
        for (int cx = cx0; cx < cx1; ++cx) {
            const uint32_t lx0 = (uint32_t)max((int)r.x0 - cx * CELL, 0), lx1 = (uint32_t)min((int)r.x1 - cx * CELL, CELL);
            keys[off] = (uint32_t)(cy * cells_x + cx) | (lx0 << 16) | (ly0 << 20) | (lx1 << 24) | (ly1 << 28);
            vals[off] = g;
            ++off;
        }
    }
}

// cell_range[c] = [first, end) of cell c in the sorted coarse list; empty cells keep (0, 0)
__global__ void __launch_bounds__(256) cell_bounds_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ n1_dev,
                                                          uint2* __restrict__ cell_range) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n1 = (uint32_t)*n1_dev;
    if (i >= n1) return;
    const uint32_t c = keys[i] & 0xFFFFu;
    if (i == 0) {
        cell_range[c].x = 0;
    } else {
        const uint32_t prev = keys[i - 1] & 0xFFFFu;
        if (prev != c) {
            cell_range[prev].y = i;
            cell_range[c].x = i;
        }
    }
    if (i == n1 - 1) cell_range[c].y = n1;
}

// exclusive scan over the CTA's 1024 threads of two values at once; carries live in shared memory across calls
__device__ __forceinline__ void block_scan2_1024(uint32_t& a, uint32_t& b, uint32_t* s_warp_a, uint32_t* s_warp_b,
                                                 uint32_t* s_carry, uint32_t& excl_a, uint32_t& excl_b) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t xa = warp_inclusive_scan(a), xb = warp_inclusive_scan(b);
    if (lane == 31) { s_warp_a[warp] = xa; s_warp_b[warp] = xb; }
    __syncthreads();
    if (warp == 0) {
        const uint32_t wa = warp_inclusive_scan(s_warp_a[lane]), wb = warp_inclusive_scan(s_warp_b[lane]);
        s_warp_a[lane] = wa; s_warp_b[lane] = wb;
    }
    __syncthreads();
    excl_a = s_carry[0] + (warp == 0 ? 0u : s_warp_a[warp - 1]) + xa - a;
    excl_b = s_carry[1] + (warp == 0 ? 0u : s_warp_b[warp - 1]) + xb - b;
    __syncthreads();
    if (threadIdx.x == 1023) { s_carry[0] += s_warp_a[31]; s_carry[1] += s_warp_b[31]; }
    __syncthreads();
}

// One CTA: units per cell (ceil(len / UNIT)) and their exclusive scan unit_base[0..NC]; unit_base[NC] = number of
// units.  With cell_count != NULL (the digit totals of a single-pass cell sort = items per cell) the cell ranges
// are derived here too, instead of by cell_bounds_kernel.
__global__ void __launch_bounds__(1024) build_units_kernel(uint2* __restrict__ cell_range, uint32_t num_cells,
                                                           uint32_t* __restrict__ unit_base,
                                                           const uint32_t* __restrict__ cell_count) {
    __shared__ uint32_t s_wa[32], s_wb[32], s_carry[2];
    if (threadIdx.x < 2) s_carry[threadIdx.x] = 0;
    __syncthreads();
    for (uint32_t base = 0; base < num_cells; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        uint32_t len = 0;
        if (i < num_cells) {
            if (cell_count) len = cell_count[i];
            else { const uint2 cr = cell_range[i]; len = cr.y - cr.x; }
        }
        uint32_t units = (len + UNIT - 1) / UNIT, ex_units, ex_len;
        block_scan2_1024(units, len, s_wa, s_wb, s_carry, ex_units, ex_len);
        if (i < num_cells) {
            unit_base[i] = ex_units;
            // empty cells keep (0, 0) like cell_bounds_kernel leaves them
            if (cell_count) cell_range[i] = len ? make_uint2(ex_len, ex_len + len) : make_uint2(0u, 0u);
        }
    }
    if (threadIdx.x == 0) unit_base[num_cells] = s_carry[0];
}

// unit u belongs to the cell c with unit_base[c] <= u < unit_base[c+1]
__device__ __forceinline__ uint32_t cell_of_unit(const uint32_t* __restrict__ unit_base, uint32_t num_cells, uint32_t u) {
    uint32_t lo = 0, hi = num_cells;   // invariant: unit_base[lo] <= u < unit_base[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (unit_base[mid] <= u) lo = mid; else hi = mid;
    }
    return lo;
}

struct UnitInfo {
    uint32_t cell, first, count, first_unit_of_cell;
};
__device__ __forceinline__ UnitInfo unit_info(const uint32_t* __restrict__ unit_base, const uint2* __restrict__ cell_range,
                                              uint32_t num_cells, uint32_t u) {
    UnitInfo ui;
    ui.cell = cell_of_unit(unit_base, num_cells, u);
    ui.first_unit_of_cell = unit_base[ui.cell];
    const uint2 cr = cell_range[ui.cell];
    ui.first = cr.x + (u - ui.first_unit_of_cell) * UNIT;
    ui.count = min((uint32_t)UNIT, cr.y - ui.first);
    return ui;
}

// ---- level 2a: per-(unit, local tile) counts, tile-major: M[t][u] -----------------------------------
__global__ void __launch_bounds__(256) cell_count_kernel(const uint32_t* __restrict__ keys,
                                                         const uint32_t* __restrict__ unit_base,
                                                         const uint2* __restrict__ cell_range, uint32_t num_cells,
                                                         uint32_t cap, uint32_t* __restrict__ M) {
    __shared__ uint32_t s_cnt[8][CELL_TILES];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t u = blockIdx.x * 8 + warp;
    if (u >= cap) return;
    const uint32_t num_units = unit_base[num_cells];
    s_cnt[warp][lane] = 0;
    s_cnt[warp][lane + 32] = 0;
    __syncwarp();
    if (u < num_units) {
        const UnitInfo ui = unit_info(unit_base, cell_range, num_cells, u);
        for (uint32_t k = lane; k < ui.count; k += 32) {
            const uint32_t key = keys[ui.first + k];
            const uint32_t x0 = (key >> 16) & 15u, y0 = (key >> 20) & 15u, x1 = (key >> 24) & 15u, y1 = (key >> 28) & 15u;
            for (uint32_t y = y0; y < y1; ++y)
                for (uint32_t x = x0; x < x1; ++x) atomicAdd(&s_cnt[warp][y * CELL + x], 1u);
        }
        __syncwarp();
    }
    // units beyond num_units (capacity padding) get zero rows so the row scan is well defined
    M[(size_t)lane * cap + u] = s_cnt[warp][lane];
    M[(size_t)(lane + 32) * cap + u] = s_cnt[warp][lane + 32];
}

// ---- level 2b: per-tile totals in global tile order --------------------------------------------------
// After the row scan, Pm[t][u] = sum of M[t][u'] for u' < u (over all cells), row_total[t] = Pm[t][cap].
__device__ __forceinline__ uint32_t prefix_at(const uint32_t* __restrict__ Pm, const uint32_t* __restrict__ row_total,
                                              uint32_t cap, uint32_t t, uint32_t u) {
    return u >= cap ? row_total[t] : Pm[(size_t)t * cap + u];
}

// One CTA: per-tile instance counts (differences of the row-scanned count matrix at the cell's unit boundaries),
// their exclusive scan in global tile order and the tile ranges -- replaces a memset and five small launches.
// ranges[t] = [start, start + count); empty tiles are (0, 0) like the reference (rasterizer_impl.cu:313).
__global__ void __launch_bounds__(1024) tile_offsets_kernel(const uint32_t* __restrict__ Pm, const uint32_t* __restrict__ row_total,
                                                            const uint32_t* __restrict__ unit_base, uint32_t cap, int cells_x,
                                                            int grid_x, int num_tiles, uint32_t* __restrict__ tile_start,
                                                            uint2* __restrict__ ranges) {
    __shared__ uint32_t s_wa[32], s_wb[32], s_carry[2];
    if (threadIdx.x < 2) s_carry[threadIdx.x] = 0;
    __syncthreads();
    for (int base = 0; base < num_tiles; base += 1024) {
        const int t = base + (int)threadIdx.x;
        uint32_t cnt = 0, dummy = 0, start, ex_dummy;
        if (t < num_tiles) {
            const int tx = t % grid_x, ty = t / grid_x;
            const uint32_t c = (uint32_t)((ty / CELL) * cells_x + tx / CELL), lt = (uint32_t)((ty % CELL) * CELL + tx % CELL);
            cnt = prefix_at(Pm, row_total, cap, lt, unit_base[c + 1]) - prefix_at(Pm, row_total, cap, lt, unit_base[c]);
        }
        const uint32_t mine = cnt;
        block_scan2_1024(cnt, dummy, s_wa, s_wb, s_carry, start, ex_dummy);
        if (t < num_tiles) {
            tile_start[t] = start;
            ranges[t] = mine ? make_uint2(start, start + mine) : make_uint2(0u, 0u);
        }
    }
    if (threadIdx.x == 0) tile_start[num_tiles] = s_carry[0];
}

// Multi-CTA form: CTA b owns tiles [1024 b, 1024 (b + 1)); it publishes its block total (flag | sum in one 64-bit word) and
// adds up the totals of the CTAs before it (at most a few dozen, all resident: <= 120 CTAs are launched, lower indices are
// dispatched first), so the dependent global-load chain of the counts is paid once, in parallel, instead of once per 1024
// tiles.  `block_sums` must be zero on entry.
__global__ void __launch_bounds__(1024) tile_offsets_lookback_kernel(const uint32_t* __restrict__ Pm, const uint32_t* __restrict__ row_total,
                                                                     const uint32_t* __restrict__ unit_base, uint32_t cap, int cells_x,
                                                                     int grid_x, int num_tiles, uint32_t* __restrict__ tile_start,
                                                                     uint2* __restrict__ ranges, unsigned long long* block_sums) {
    __shared__ uint32_t s_wa[32], s_wb[32], s_carry[2];
    __shared__ uint32_t s_prev;
    if (threadIdx.x < 2) s_carry[threadIdx.x] = 0;
    if (threadIdx.x == 0) s_prev = 0;
    __syncthreads();
    const int t = (int)blockIdx.x * 1024 + (int)threadIdx.x;
    uint32_t cnt = 0, dummy = 0, local, ex_dummy;
    if (t < num_tiles) {
        const int tx = t % grid_x, ty = t / grid_x;
        const uint32_t c = (uint32_t)((ty / CELL) * cells_x + tx / CELL), lt = (uint32_t)((ty % CELL) * CELL + tx % CELL);
        cnt = prefix_at(Pm, row_total, cap, lt, unit_base[c + 1]) - prefix_at(Pm, row_total, cap, lt, unit_base[c]);
    }
    const uint32_t mine = cnt;
    block_scan2_1024(cnt, dummy, s_wa, s_wb, s_carry, local, ex_dummy);      // s_carry[0] = this CTA's total afterwards
    if (threadIdx.x == 0) {
        __threadfence();
        atomicExch(&block_sums[blockIdx.x], (1ull << 32) | (unsigned long long)s_carry[0]);
    }
    // totals of the CTAs in front: thread j < blockIdx.x waits for CTA j's word
    if (threadIdx.x < blockIdx.x) {
        unsigned long long w;
        unsigned spins = 0;       // bounded: a scheduling surprise must not hang the GPU (the ranges would be wrong instead)
        do { w = atomicAdd(&block_sums[threadIdx.x], 0ull); } while ((w >> 32) == 0ull && ++spins < (1u << 26));
        atomicAdd(&s_prev, (uint32_t)w);
    }
    __syncthreads();
    const uint32_t start = s_prev + local;
    if (t < num_tiles) {
        tile_start[t] = start;
        ranges[t] = mine ? make_uint2(start, start + mine) : make_uint2(0u, 0u);
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) tile_start[num_tiles] = s_prev + s_carry[0];
}

// ---- level 2c: scatter ------------------------------------------------------------------------------
// One warp per unit.  Lane l owns local tiles l and l + 32 of the cell.  The unit's coarse items are walked IN
// ORDER, 32 at a time, and each lane appends the ids of the items covering its tiles -- no ballots, no ranks: the
// order inside a tile list is the walk order = depth order.  The unit's output is first assembled in shared memory,
// tile run after tile run, and then copied to the tile lists with coalesced stores.  The run lengths of the unit
// are known exactly -- they are the differences of the row-scanned count matrix -- so every tile gets a fixed slice
// of the staging buffer (exclusive scan over the cell's 64 tiles) and an append is one predicated STS through a
// lane-private pointer.  Per coarse item the warp reads one 16-byte record {coverage bits of tiles 0-31, of tiles
// 32-63, id} and each lane tests "its" bit of the two words.
// Why staging: direct per-lane global stores (one 4-byte store per (lane, entry) into 64 different lists) gave 37.5 M
// single-sector L2 write requests at C3 (37.6 M entries), 227 MB DRAM written + 159 MB read back for partial
// sectors; staging turns them into ~3 M requests.
// A unit whose output does not fit the staging buffer (very large splats) is staged in several walks.
constexpr int SQ_ENTRIES = 2048;           // staging capacity per warp (a unit of 256 items averages ~1800 at C3)
constexpr int SQ_WARPS = 8;
constexpr int SQ_WARP_WORDS = SQ_ENTRIES + 32 * 4;           // staging + 32 item records (uint4)
constexpr size_t SQ_SMEM = (size_t)SQ_WARPS * SQ_WARP_WORDS * sizeof(uint32_t);

// if (hit) { shared[addr] = v; addr += 4; } as two predicated instructions
__device__ __forceinline__ void sts_append(uint32_t& addr, uint32_t v, uint32_t hit) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p st.shared.u32 [%0], %1;\n\t@p add.u32 %0, %0, 4;\n\t}"
                 : "+r"(addr) : "r"(v), "r"(hit) : "memory");
}

// 16-byte record of one coarse item: coverage bits of local tiles 0-31 and 32-63 (bit 8 y + x), Gaussian id
__device__ __forceinline__ uint4 item_record(uint32_t key, uint32_t id) {
    const uint32_t x0 = (key >> 16) & 15u, y0 = (key >> 20) & 15u, x1 = (key >> 24) & 15u, y1 = (key >> 28) & 15u;
    const uint32_t cm = ((1u << x1) - 1u) & ~((1u << x0) - 1u);      // columns, 8 bits
    const uint32_t rm = ((1u << y1) - 1u) & ~((1u << y0) - 1u);      // rows, 8 bits
    // the row bits are spread to the byte LSBs, times the column mask
    const uint32_t lo = cm * (((rm & 15u) * 0x00204081u) & 0x01010101u);
    const uint32_t hi = cm * (((rm >> 4) * 0x00204081u) & 0x01010101u);
    return make_uint4(lo, hi, id, 0u);
}

// One walk over the unit's coarse items: every lane appends the ids of the items covering "its" tiles (bit0 /
// bit1 select them in the two coverage words; 0 = this lane's tile is not part of the walk) to its slices of the
// staging buffer through the cursors a0 / a1.
template <bool S0, bool S1>
__device__ __forceinline__ void scatter_walk(const UnitInfo& ui, const uint32_t* __restrict__ keys,
                                             const uint32_t* __restrict__ vals, uint4* s_item, int lane, uint32_t bit0,
                                             uint32_t bit1, uint32_t a0, uint32_t a1) {
    uint32_t key = 0, id = 0;
    if ((uint32_t)lane < ui.count) { key = keys[ui.first + lane]; id = vals[ui.first + lane]; }
    for (uint32_t base = 0; base < ui.count; base += 32) {
        const int nitems = (int)min(32u, ui.count - base);
        __syncwarp();
        s_item[lane] = item_record(key, id);
        __syncwarp();
        // next batch's loads fly while this batch is appended
        const uint32_t nxt = base + 32 + lane;
        if (nxt < ui.count) { key = keys[ui.first + nxt]; id = vals[ui.first + nxt]; }
#pragma unroll 4
        for (int i = 0; i < nitems; ++i) {
            const uint4 it = s_item[i];
            if (S0) sts_append(a0, it.z, it.x & bit0);
            if (S1) sts_append(a1, it.z, it.y & bit1);
        }
    }
    __syncwarp();
}

// copy the staged runs of one tile half to the tile lists: two tiles per iteration, one per half warp
__device__ __forceinline__ void scatter_copy_out(const uint32_t* q, uint32_t len, uint32_t off, uint32_t pos, int lane,
                                                 uint32_t* __restrict__ point_list) {
    unsigned live = __ballot_sync(0xFFFFFFFFu, len != 0);
    const int sub = lane & 15;
    while (live) {
        const int ta = __ffs(live) - 1;
        live &= live - 1;
        const int tb = live ? __ffs(live) - 1 : -1;
        live &= live - 1;
        const int mine = lane < 16 ? ta : tb;
        const int src_lane = mine < 0 ? 0 : mine;
        uint32_t c = __shfl_sync(0xFFFFFFFFu, len, src_lane);
        const uint32_t o = __shfl_sync(0xFFFFFFFFu, off, src_lane);
        const uint32_t p = __shfl_sync(0xFFFFFFFFu, pos, src_lane);
        if (mine < 0) c = 0;
        for (uint32_t e = sub; e < c; e += 16) point_list[p + e] = q[o + e];
    }
}

__global__ void __launch_bounds__(SQ_WARPS * 32) cell_scatter_staged_kernel(
    const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, const uint32_t* __restrict__ unit_base,
    const uint2* __restrict__ cell_range, uint32_t num_cells, const uint32_t* __restrict__ Pm,
    const uint32_t* __restrict__ row_total, uint32_t cap, const uint32_t* __restrict__ tile_start, int cells_x, int grid_x,
    int grid_y, uint32_t* __restrict__ point_list) {
    extern __shared__ __align__(16) uint32_t sq_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t u = blockIdx.x * SQ_WARPS + warp;
    const uint32_t num_units = unit_base[num_cells];
    if (u >= num_units) return;
    uint32_t* q = sq_smem + (size_t)warp * SQ_WARP_WORDS;
    uint4* s_item = reinterpret_cast<uint4*>(q + SQ_ENTRIES);
    const UnitInfo ui = unit_info(unit_base, cell_range, num_cells, u);
    // global output position and run length of this unit in local tiles lane (h = 0) and lane + 32 (h = 1)
    uint32_t pos[2], len[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint32_t t = lane + 32 * h;
        const int tx = (int)(ui.cell % cells_x) * CELL + (int)(t % CELL), ty = (int)(ui.cell / cells_x) * CELL + (int)(t / CELL);
        uint32_t p = 0, l = 0;
        if (tx < grid_x && ty < grid_y) {
            const uint32_t before = prefix_at(Pm, row_total, cap, t, u);
            p = tile_start[ty * grid_x + tx] + before - prefix_at(Pm, row_total, cap, t, ui.first_unit_of_cell);
            l = prefix_at(Pm, row_total, cap, t, u + 1) - before;
        }
        pos[h] = p;
        len[h] = l;
    }
    // exclusive prefix of the run lengths in tile order (0..63): the staging slice of every tile
    uint32_t pre[2];
    {
        const uint32_t x0 = warp_inclusive_scan(len[0]), x1 = warp_inclusive_scan(len[1]);
        const uint32_t tot0 = __shfl_sync(0xFFFFFFFFu, x0, 31);
        pre[0] = x0 - len[0];
        pre[1] = tot0 + x1 - len[1];
    }
    // The unit's output is staged in as few walks as possible: the cell's 8 tile rows are cut greedily into
    // groups of consecutive rows whose runs fit the staging buffer together.  One row always fits (at most
    // UNIT items x 8 tiles = SQ_ENTRIES entries), typical units need a single walk over all rows.
    static_assert(UNIT * CELL <= SQ_ENTRIES, "one tile row of a unit must fit the staging buffer");
    // pre_row(r) = entries in rows < r = prefix at tile 8 r  (r = 0..8)
    auto pre_row = [&](int r) -> uint32_t {
        if (r >= 8) return __shfl_sync(0xFFFFFFFFu, pre[1] + len[1], 31);
        return r < 4 ? __shfl_sync(0xFFFFFFFFu, pre[0], 8 * r) : __shfl_sync(0xFFFFFFFFu, pre[1], 8 * (r - 4));
    };
    const uint32_t q_addr = (uint32_t)__cvta_generic_to_shared(q);
    const uint32_t bit = 1u << lane;
    const int my_row0 = lane >> 3, my_row1 = 4 + (lane >> 3);
    const uint32_t total = pre_row(8), half = pre_row(4);
    int r0 = 0;
    while (r0 < 8) {                                    // warp-uniform
        const uint32_t start = pre_row(r0);
        int r1;
        if (r0 == 0 && total <= (uint32_t)SQ_ENTRIES) r1 = 8;                                    // everything at once
        else if ((r0 == 0 || r0 == 4) && half <= (uint32_t)SQ_ENTRIES && total - half <= (uint32_t)SQ_ENTRIES)
            r1 = r0 + 4;                                                                         // tile halves
        else {
            r1 = r0 + 1;
            while (r1 < 8 && pre_row(r1 + 1) - start <= (uint32_t)SQ_ENTRIES) ++r1;
        }
        if (pre_row(r1) != start) {                     // the group has output
            const bool in0 = my_row0 >= r0 && my_row0 < r1, in1 = my_row1 >= r0 && my_row1 < r1;
            const uint32_t off0 = pre[0] - start, off1 = pre[1] - start;
            const uint32_t b0 = in0 ? bit : 0u, b1 = in1 ? bit : 0u;
            const uint32_t a0 = q_addr + 4u * off0, a1 = q_addr + 4u * off1;
            if (r1 <= 4) scatter_walk<true, false>(ui, keys, vals, s_item, lane, b0, b1, a0, a1);
            else if (r0 >= 4) scatter_walk<false, true>(ui, keys, vals, s_item, lane, b0, b1, a0, a1);
            else scatter_walk<true, true>(ui, keys, vals, s_item, lane, b0, b1, a0, a1);
            scatter_copy_out(q, in0 ? len[0] : 0u, off0, pos[0], lane, point_list);
            scatter_copy_out(q, in1 ? len[1] : 0u, off1, pos[1], lane, point_list);
            __syncwarp();
        }
        r0 = r1;
    }
}

// ---- orchestration -----------------------------------------------------------------------------------
int run_tile_binning(const GeomState& g, int P, int W, int H, size_t R_cap, size_t N1_cap, const BinScratch& bs,
                     uint32_t* point_list, uint2* ranges, cudaStream_t s, bool debug) {
    const int gx = tiles_x(W), gy = tiles_y(H);
    const int cells_x = (gx + CELL - 1) / CELL, cells_y = (gy + CELL - 1) / CELL;
    const uint32_t num_cells = (uint32_t)(cells_x * cells_y);
    const int num_tiles = gx * gy;
    if (N1_cap == 0 || R_cap == 0) {
        // nothing can be binned: empty ranges
        GSR_CUDA(cudaMemsetAsync(ranges, 0, (size_t)num_tiles * sizeof(uint2), s));
        return 0;
    }
    // level 1: emit + stable sort by cell id; the sorted result must land in (key_b, val_b)
    prof_begin(ST_EMIT_CELLS, s);
    int cell_bits = 0;
    while ((1u << cell_bits) < num_cells) ++cell_bits;
    const bool even = (radix_num_passes(0, cell_bits) % 2) == 0;
    uint32_t* ka = even ? bs.key_b : bs.key_a;
    uint32_t* va = even ? bs.val_b : bs.val_a;
    uint32_t* kb = even ? bs.key_a : bs.key_b;
    uint32_t* vb = even ? bs.val_a : bs.val_b;
    emit_cells_kernel<<<(P + 255) / 256, 256, 0, s>>>(cells_x, g.order, g.offsets, g.rect_sorted, ka, va, g.counters,
                                                      (uint32_t)N1_cap, (unsigned long long)R_cap);
    count_launches(1);
    GSR_STAGE(s, debug, "emit_cells_kernel");
    prof_end(ST_EMIT_CELLS, s);
    prof_begin(ST_CELL_SORT, s);
    const uint32_t* n1_dev = reinterpret_cast<const uint32_t*>(g.counters + 7);
    const size_t N1 = N1_cap;
    int rc = radix_sort_pairs(ka, va, kb, vb, N1, 0, cell_bits, bs.radix_tmp, s, debug, nullptr, n1_dev);
    if (rc) return rc;
    const uint32_t* keys = bs.key_b;
    const uint32_t* vals = bs.val_b;
    prof_end(ST_CELL_SORT, s);
    prof_begin(ST_CELL_COUNT, s);

    // units + per-unit tile counts
    const uint32_t cap = (uint32_t)bs.units_cap;
    if (radix_num_passes(0, cell_bits) == 1) {
        // one pass sorted by the whole cell id: its digit totals ARE the items per cell
        build_units_kernel<<<1, 1024, 0, s>>>(bs.cell_range, num_cells, bs.unit_base, radix_pass_totals(bs.radix_tmp, N1));
        count_launches(1);
    } else {
        GSR_CUDA(cudaMemsetAsync(bs.cell_range, 0, (size_t)num_cells * sizeof(uint2), s));
        cell_bounds_kernel<<<(unsigned)((N1 + 255) / 256), 256, 0, s>>>(keys, g.counters + 7, bs.cell_range);
        count_launches(1);
        build_units_kernel<<<1, 1024, 0, s>>>(bs.cell_range, num_cells, bs.unit_base, nullptr);
        count_launches(1);
    }
    GSR_STAGE(s, debug, "build_units_kernel");
    cell_count_kernel<<<(cap + 7) / 8, 256, 0, s>>>(keys, bs.unit_base, bs.cell_range, num_cells, cap, bs.M);
    count_launches(1);
    GSR_STAGE(s, debug, "cell_count_kernel");
    prof_end(ST_CELL_COUNT, s);
    prof_begin(ST_TILE_OFFSETS, s);

    // exact output positions
    rc = row_scan_u32(bs.M, CELL_TILES, cap, bs.row_total, s);
    if (rc) return rc;
    const int off_ctas = (num_tiles + 1023) / 1024;
    if (off_ctas > 1 && off_ctas <= 120) {
        GSR_CUDA(cudaMemsetAsync(bs.block_sums, 0, (size_t)off_ctas * sizeof(unsigned long long), s));
        tile_offsets_lookback_kernel<<<off_ctas, 1024, 0, s>>>(bs.M, bs.row_total, bs.unit_base, cap, cells_x, gx, num_tiles,
                                                               bs.tile_start, ranges, bs.block_sums);
    } else {
        tile_offsets_kernel<<<1, 1024, 0, s>>>(bs.M, bs.row_total, bs.unit_base, cap, cells_x, gx, num_tiles, bs.tile_start, ranges);
    }
    count_launches(1);
    GSR_STAGE(s, debug, "tile_offsets_kernel");
    prof_end(ST_TILE_OFFSETS, s);
    prof_begin(ST_TILE_SCATTER, s);

    // function attributes are per device / context: set it for the current device on every call (a process may
    // rasterize on several GPUs), it is a cheap driver call
    GSR_CUDA(cudaFuncSetAttribute(cell_scatter_staged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SQ_SMEM));
    cell_scatter_staged_kernel<<<(cap + SQ_WARPS - 1) / SQ_WARPS, SQ_WARPS * 32, SQ_SMEM, s>>>(
        keys, vals, bs.unit_base, bs.cell_range, num_cells, bs.M, bs.row_total, cap, bs.tile_start, cells_x, gx, gy,
        point_list);
    count_launches(1);
    GSR_STAGE(s, debug, "cell_scatter_staged_kernel");
    prof_end(ST_TILE_SCATTER, s);
    return 0;
}

}  // namespace gsr
