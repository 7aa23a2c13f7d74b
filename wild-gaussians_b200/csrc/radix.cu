// radix.cu -- stable LSD radix partition of (u32 key, u32 value) pairs and an exclusive scan
// of counts.  Hand-written replacement for the two CUB calls on the reference's
// path (cub::DeviceRadixSort::SortPairs, rasterizer_impl.cu:303-311, and
// cub::DeviceScan::InclusiveSum, :280).
//
// Why the result equals the reference's: both are stable sorts of the same multiset, and a
// stable sort has exactly one result.  The reference sorts R 64-bit keys (tile | depth) in
// one go; here the P Gaussians are ordered by depth bits once (4 passes over P pairs) and
// the R instances, emitted in that depth order, are then stably partitioned by their tile
// id only (2 passes over R pairs) -- see binning.cu.
//
// One pass = three launches, no spin-waiting between CTAs (so nothing can dead-lock):
//   radix_hist_kernel    per-CTA digit histogram of a CHUNK of the input (plain shared atomics) -> hist[digit][cta]
//   rowscan_wide_kernel  one CTA per digit: exclusive scan along the row    -> hist (in place), total[digit]
//   radix_scatter_kernel re-reads the chunk, ranks every item among equal digits in (warp, round, lane) = input
//                        order -- the lanes holding the same digit are found with 8 ballots, one per digit bit;
//                        __match_any_sync was measured 2-4x slower here because its cost grows with the number of
//                        distinct digits in the warp -- then sorts the chunk in shared memory and writes it out so
//                        that consecutive threads write consecutive addresses inside every digit run.
// The last pass of a sort can also deliver side data in sorted order (RadixAux).
#include "common.cuh"

namespace gsr {

constexpr int RADIX_BITS = 8;
constexpr int RADIX = 1 << RADIX_BITS;
constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_ITEMS = 8;                        // items per thread (16 needs 99 registers: 2 CTAs/SM, latency-bound)
constexpr int RS_CHUNK = RS_THREADS * RS_ITEMS;    // items per CTA
constexpr int RS_WARP_ITEMS = 32 * RS_ITEMS;       // items per warp (contiguous in the input)

static inline size_t radix_ctas(size_t n) { return (n + RS_CHUNK - 1) / RS_CHUNK; }

// hist[RADIX][ctas] + total[RADIX]
size_t radix_tmp_elems(size_t n) { return (size_t)RADIX * (radix_ctas(n) + 1); }

// The item count is min(*n_dev, n_cap) when n_dev != NULL (the grid is sized for n_cap; CTAs beyond the count publish
// zero histogram columns).  DROP: keys equal to RADIX_DROP_KEY are not part of the sort at all (neither counted nor
// scattered): the first pass of the depth sort compacts away the Gaussians that are culled / outside the tile-row band.
__device__ __forceinline__ size_t radix_count(size_t n_cap, const uint32_t* __restrict__ n_dev) {
    if (n_dev == nullptr) return n_cap;
    const size_t n = *n_dev;
    return n < n_cap ? n : n_cap;
}

template <bool DROP>
__global__ void __launch_bounds__(RS_THREADS) radix_hist_kernel(const uint32_t* __restrict__ keys, size_t n_cap,
                                                                const uint32_t* __restrict__ n_dev, int shift,
                                                                uint32_t mask, uint32_t* __restrict__ hist, uint32_t ctas) {
    __shared__ uint32_t s_hist[RADIX];
    const size_t n = radix_count(n_cap, n_dev);
    const size_t base = (size_t)blockIdx.x * RS_CHUNK;
    if (base >= n) {
        for (int i = threadIdx.x; i < RADIX; i += RS_THREADS) hist[(size_t)i * ctas + blockIdx.x] = 0;
        return;
    }
    for (int i = threadIdx.x; i < RADIX; i += RS_THREADS) s_hist[i] = 0;
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // plain shared-memory atomics: with 256 bins the lanes of a warp rarely collide on random digits, and a
    // warp whose lanes all hit one bin (constant high digits) is serialised by the hardware in ~32 cycles.
    // (__match_any_sync-based aggregation costs time proportional to the number of DISTINCT digits in the warp:
    // measured 24 us per 3M-key pass on random digits vs 15 us on constant ones.)
    uint32_t k[RS_ITEMS];
#pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        const size_t i = base + (size_t)warp * RS_WARP_ITEMS + r * 32 + lane;
        k[r] = i < n ? keys[i] : 0u;
    }
#pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        const size_t i = base + (size_t)warp * RS_WARP_ITEMS + r * 32 + lane;
        if (i < n && !(DROP && k[r] == RADIX_DROP_KEY)) atomicAdd(&s_hist[(k[r] >> shift) & mask], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < RADIX; i += RS_THREADS) hist[(size_t)i * ctas + blockIdx.x] = s_hist[i];
}

// One CTA per row of a [rows][cols] matrix: exclusive scan of the row in place, row total -> total[row].  K chunks of 1024
// columns per round share the two barriers of a round (warp w combines the warp totals of chunk w), so a LONG row (the
// count matrix of the tile binning: 64 rows of ~20 k columns) costs cols / (K * 1024) dependent rounds instead of
// cols / 1024; loads and stores stay coalesced.  K = 1 for short rows (radix histograms, scan partials).
template <int K>
__global__ void __launch_bounds__(1024) rowscan_wide_kernel(uint32_t* __restrict__ hist, uint32_t cols, uint32_t* __restrict__ total) {
    __shared__ uint32_t s_warp[K][32];
    __shared__ uint32_t s_carry;
    uint32_t* row = hist + (size_t)blockIdx.x * cols;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < cols; base += K * 1024) {
        uint32_t v[K], x[K];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const uint32_t i = base + k * 1024 + threadIdx.x;
            v[k] = i < cols ? row[i] : 0u;
        }
#pragma unroll
        for (int k = 0; k < K; ++k) {
            x[k] = warp_inclusive_scan(v[k]);
            if (lane == 31) s_warp[k][warp] = x[k];
        }
        __syncthreads();
        if (warp < K) s_warp[warp][lane] = warp_inclusive_scan(s_warp[warp][lane]);   // inclusive over the warps of chunk `warp`
        __syncthreads();
        uint32_t off = s_carry;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const uint32_t i = base + k * 1024 + threadIdx.x;
            if (i < cols) row[i] = off + (warp == 0 ? 0u : s_warp[k][warp - 1]) + x[k] - v[k];
            off += s_warp[k][31];
        }
        __syncthreads();
        if (threadIdx.x == 0) s_carry = off;
        __syncthreads();
    }
    if (threadIdx.x == 0) total[blockIdx.x] = s_carry;
}

template <bool DROP, bool AUX>
__global__ void __launch_bounds__(RS_THREADS) radix_scatter_kernel(const uint32_t* __restrict__ keys_in,
                                                                   const uint32_t* __restrict__ vals_in,
                                                                   uint32_t* __restrict__ keys_out,
                                                                   uint32_t* __restrict__ vals_out, size_t n_cap,
                                                                   const uint32_t* __restrict__ n_dev, int shift,
                                                                   uint32_t mask, const uint32_t* __restrict__ hist,
                                                                   const uint32_t* __restrict__ total, uint32_t ctas,
                                                                   const RadixAux aux, uint32_t* __restrict__ n_out) {
    __shared__ uint32_t s_cnt[RS_WARPS][RADIX];   // per-warp digit counters, later global bases
    __shared__ uint32_t s_digit_base[RADIX];
    __shared__ uint32_t s_key[RS_CHUNK];
    __shared__ uint32_t s_val[RS_CHUNK];
    __shared__ uint32_t s_kept;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t n = radix_count(n_cap, n_dev);
    // number of items that take part in the sort (all digit totals): the next passes' item count
    if (n_out != nullptr && blockIdx.x == 0) {
        __shared__ uint32_t s_t[RS_WARPS];
        const uint32_t v = __reduce_add_sync(0xFFFFFFFFu, total[threadIdx.x]);
        if (lane == 0) s_t[warp] = v;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t sum = 0;
            for (int w = 0; w < RS_WARPS; ++w) sum += s_t[w];
            *n_out = sum;
        }
    }
    if ((size_t)blockIdx.x * RS_CHUNK >= n) return;
    for (int i = threadIdx.x; i < RS_WARPS * RADIX; i += RS_THREADS) (&s_cnt[0][0])[i] = 0;

    // exclusive scan of the digit totals (256 values, one per thread)
    {
        __shared__ uint32_t s_w[RS_WARPS];
        const uint32_t v = total[threadIdx.x];
        const uint32_t x = warp_inclusive_scan(v);
        if (lane == 31) s_w[warp] = x;
        __syncthreads();
        uint32_t off = 0;
        for (int w = 0; w < warp; ++w) off += s_w[w];
        s_digit_base[threadIdx.x] = off + x - v + hist[(size_t)threadIdx.x * ctas + blockIdx.x];
    }
    __syncthreads();

    const size_t base = (size_t)blockIdx.x * RS_CHUNK + (size_t)warp * RS_WARP_ITEMS;
    uint32_t key[RS_ITEMS], val[RS_ITEMS];
    uint16_t rank[RS_ITEMS];
    const unsigned lt_mask = (1u << lane) - 1u;
#pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        const size_t i = base + r * 32 + lane;
        const bool valid = i < n;
        key[r] = valid ? keys_in[i] : RADIX_DROP_KEY;
        val[r] = valid ? vals_in[i] : 0u;
    }
#pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        const size_t i = base + r * 32 + lane;
        const bool valid = i < n && !(DROP && key[r] == RADIX_DROP_KEY);
        const uint32_t d = valid ? ((key[r] >> shift) & mask) : 0u;
        // lanes holding the same digit: 8 ballots (one per digit bit) instead of __match_any_sync, whose cost
        // grows with the number of distinct digits in the warp
        unsigned peers = __ballot_sync(0xFFFFFFFFu, valid);
#pragma unroll
        for (int b = 0; b < RADIX_BITS; ++b) {
            const bool bit = (d >> b) & 1u;
            const unsigned m = __ballot_sync(0xFFFFFFFFu, bit);
            peers &= bit ? m : ~m;
        }
        uint32_t old = 0;
        if (valid) old = s_cnt[warp][d];
        __syncwarp();
        if (valid && lane == (__ffs(peers) - 1)) s_cnt[warp][d] = old + __popc(peers);
        __syncwarp();
        rank[r] = (uint16_t)(old + __popc(peers & lt_mask));
    }
    __syncthreads();
    // Local (CTA-wide) stable order: per digit, running offset over the warps, then an exclusive scan over
    // the digits; s_cnt[w][d] becomes the position of the first item of (warp, digit) in the CTA's sorted
    // chunk and s_digit_base[d] the difference between that chunk position and the global output position.
    {
        __shared__ uint32_t s_w2[RS_WARPS];
        const int d = threadIdx.x;
        uint32_t run = 0;
        uint32_t c[RS_WARPS];
#pragma unroll
        for (int w = 0; w < RS_WARPS; ++w) { c[w] = s_cnt[w][d]; run += c[w]; }
        const uint32_t x = warp_inclusive_scan(run);     // inclusive scan of the digit totals of this CTA
        if (lane == 31) s_w2[warp] = x;
        __syncthreads();
        uint32_t off = 0;
        for (int w = 0; w < warp; ++w) off += s_w2[w];
        uint32_t loc = off + x - run;   // first chunk position of digit d
        if (d == RADIX - 1) s_kept = off + x;   // items of this chunk that take part in the sort
        s_digit_base[d] -= loc;         // global position = chunk position + s_digit_base[d]  (mod 2^32)
#pragma unroll
        for (int w = 0; w < RS_WARPS; ++w) { s_cnt[w][d] = loc; loc += c[w]; }
    }
    __syncthreads();
    // stage the chunk in sorted order, then write it out: consecutive threads write consecutive addresses
    // inside every digit run (the unstaged version issued one scattered 4-byte store per item and array)
#pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        const size_t i = base + r * 32 + lane;
        if (i < n && !(DROP && key[r] == RADIX_DROP_KEY)) {
            const uint32_t d = (key[r] >> shift) & mask;
            const uint32_t li = s_cnt[warp][d] + rank[r];
            s_key[li] = key[r];
            s_val[li] = val[r];
        }
    }
    __syncthreads();
    const uint32_t cta_n = s_kept;
#pragma unroll 4
    for (uint32_t i = threadIdx.x; i < cta_n; i += RS_THREADS) {
        const uint32_t k = s_key[i];
        const uint32_t pos = i + s_digit_base[(k >> shift) & mask];
        keys_out[pos] = k;
        const uint32_t v = s_val[i];
        vals_out[pos] = v;
        if (AUX) {
            // final pass: also deliver the per-item side data in sorted order (one gather here instead of one in
            // every later kernel that walks the sorted sequence)
            aux.out32[pos] = aux.in32[v];
            aux.out64[pos] = aux.in64[v];
        }
    }
}

// digit totals (RADIX entries) of the LAST pass of the most recent radix_sort_pairs over n items
const uint32_t* radix_pass_totals(const uint32_t* tmp, size_t n) { return tmp + (size_t)RADIX * radix_ctas(n); }

int row_scan_u32(uint32_t* m, int rows, size_t cols, uint32_t* total, cudaStream_t s) {
    if (rows <= 0 || cols == 0) return 0;
    if (cols > 4096) rowscan_wide_kernel<8><<<rows, 1024, 0, s>>>(m, (uint32_t)cols, total);
    else rowscan_wide_kernel<1><<<rows, 1024, 0, s>>>(m, (uint32_t)cols, total);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

int radix_num_passes(int begin_bit, int end_bit) {
    const int nbits = end_bit - begin_bit;
    return nbits <= 0 ? 0 : (nbits + RADIX_BITS - 1) / RADIX_BITS;
}

int radix_sort_pairs(uint32_t* key_a, uint32_t* val_a, uint32_t* key_b, uint32_t* val_b, size_t n_cap, int begin_bit,
                     int end_bit, uint32_t* tmp, cudaStream_t s, bool debug, const RadixAux* aux, const uint32_t* n_dev,
                     uint32_t* n_compact) {
    // Stable sort on key bits [begin_bit, end_bit).  The input is (key_a, val_a); passes
    // ping-pong A -> B -> A ..., clobbering both.  With an even number of passes
    // (radix_num_passes) the result is in A, with an odd number in B; callers place their
    // buffers accordingly.
    // n_cap sizes the grids; the item count is min(*n_dev, n_cap) when n_dev is given.  With n_compact != NULL the
    // first pass drops the items whose key is RADIX_DROP_KEY and stores the number of remaining items in *n_compact,
    // which is the item count of the following passes.
    if (n_cap == 0) return 0;
    const int passes = radix_num_passes(begin_bit, end_bit);
    const uint32_t ctas = (uint32_t)radix_ctas(n_cap);
    uint32_t* hist = tmp;
    uint32_t* total = tmp + (size_t)RADIX * ctas;
    for (int pass = 0; pass < passes; ++pass) {
        const int shift = begin_bit + pass * RADIX_BITS;
        const int bits = min(RADIX_BITS, end_bit - shift);
        const uint32_t mask = (1u << bits) - 1u;
        const bool a_to_b = (pass % 2) == 0;
        const uint32_t* kin = a_to_b ? key_a : key_b;
        const uint32_t* vin = a_to_b ? val_a : val_b;
        uint32_t* kout = a_to_b ? key_b : key_a;
        uint32_t* vout = a_to_b ? val_b : val_a;
        const bool drop = n_compact != nullptr && pass == 0;
        const uint32_t* nd = (n_compact != nullptr && pass > 0) ? n_compact : n_dev;
        if (drop) radix_hist_kernel<true><<<ctas, RS_THREADS, 0, s>>>(kin, n_cap, nd, shift, mask, hist, ctas);
        else radix_hist_kernel<false><<<ctas, RS_THREADS, 0, s>>>(kin, n_cap, nd, shift, mask, hist, ctas);
        count_launches(1);
        GSR_STAGE(s, debug, "radix_hist_kernel");
        rowscan_wide_kernel<1><<<RADIX, 1024, 0, s>>>(hist, ctas, total);
        count_launches(1);
        GSR_STAGE(s, debug, "rowscan_wide_kernel");
        const bool with_aux = aux && pass == passes - 1;
        const RadixAux ax = with_aux ? *aux : RadixAux{};
        if (drop && with_aux) radix_scatter_kernel<true, true><<<ctas, RS_THREADS, 0, s>>>(kin, vin, kout, vout, n_cap, nd, shift, mask, hist, total, ctas, ax, n_compact);
        else if (drop) radix_scatter_kernel<true, false><<<ctas, RS_THREADS, 0, s>>>(kin, vin, kout, vout, n_cap, nd, shift, mask, hist, total, ctas, ax, n_compact);
        else if (with_aux) radix_scatter_kernel<false, true><<<ctas, RS_THREADS, 0, s>>>(kin, vin, kout, vout, n_cap, nd, shift, mask, hist, total, ctas, ax, nullptr);
        else radix_scatter_kernel<false, false><<<ctas, RS_THREADS, 0, s>>>(kin, vin, kout, vout, n_cap, nd, shift, mask, hist, total, ctas, ax, nullptr);
        count_launches(1);
        GSR_STAGE(s, debug, "radix_scatter_kernel");
    }
    return 0;
}

// ----------------------------------------------------------------------------------------
// exclusive scan of the depth-ordered cell counts (coarse-item offsets)
// ----------------------------------------------------------------------------------------
constexpr int SC_THREADS = 256;
constexpr int SC_ITEMS = 8;
constexpr int SC_CHUNK = SC_THREADS * SC_ITEMS;

size_t scan_tmp_elems(size_t n) { return (n + SC_CHUNK - 1) / SC_CHUNK + 64; }

__device__ __forceinline__ uint32_t block_exclusive_scan_256(uint32_t v, uint32_t* s_warp, uint32_t* block_total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t x = warp_inclusive_scan(v);
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    uint32_t off = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < SC_THREADS / 32; ++w) {
        const uint32_t c = s_warp[w];
        if (w < warp) off += c;
        tot += c;
    }
    *block_total = tot;
    __syncthreads();
    return off + x - v;
}

__global__ void __launch_bounds__(SC_THREADS) scan_reduce_kernel(const uint32_t* __restrict__ counts, size_t n_cap,
                                                                 const uint32_t* __restrict__ n_dev,
                                                                 uint32_t* __restrict__ partial) {
    __shared__ uint32_t s_warp[SC_THREADS / 32];
    const size_t n = radix_count(n_cap, n_dev);
    const size_t base = (size_t)blockIdx.x * SC_CHUNK;
    if (base >= n) {
        if (threadIdx.x == 0) partial[blockIdx.x] = 0;
        return;
    }
    uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < SC_ITEMS; ++k) {
        const size_t i = base + (size_t)k * SC_THREADS + threadIdx.x;
        if (i < n) sum += counts[i];
    }
    uint32_t tot;
    block_exclusive_scan_256(sum, s_warp, &tot);
    if (threadIdx.x == 0) partial[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(SC_THREADS) scan_apply_kernel(const uint32_t* __restrict__ counts, size_t n_cap,
                                                                const uint32_t* __restrict__ n_dev,
                                                                const uint32_t* __restrict__ partial, uint32_t m,
                                                                uint32_t* __restrict__ out, uint32_t* __restrict__ total_out) {
    __shared__ uint32_t s_warp[SC_THREADS / 32];
    const size_t n = radix_count(n_cap, n_dev);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        out[n] = partial[m];
        if (total_out) *total_out = partial[m];
    }
    if ((size_t)blockIdx.x * SC_CHUNK >= n) return;
    // blocked arrangement: thread t owns items [t*SC_ITEMS, (t+1)*SC_ITEMS) of the chunk
    const size_t base = (size_t)blockIdx.x * SC_CHUNK + (size_t)threadIdx.x * SC_ITEMS;
    uint32_t v[SC_ITEMS];
    uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < SC_ITEMS; ++k) {
        const size_t i = base + k;
        v[k] = i < n ? counts[i] : 0u;
        sum += v[k];
    }
    uint32_t tot;
    uint32_t off = block_exclusive_scan_256(sum, s_warp, &tot) + partial[blockIdx.x];
#pragma unroll
    for (int k = 0; k < SC_ITEMS; ++k) {
        const size_t i = base + k;
        if (i < n) out[i] = off;
        off += v[k];
    }
}

// out[i] = sum_{j<i} counts[j] for i < n, out[n] = total (also stored in *total_out); n = min(*n_dev, n_cap)
int exclusive_scan_u32(const uint32_t* counts, uint32_t* out, size_t n_cap, uint32_t* tmp, cudaStream_t s,
                       const uint32_t* n_dev, uint32_t* total_out) {
    if (n_cap == 0) {
        GSR_CUDA(cudaMemsetAsync(out, 0, 4, s));
        if (total_out) GSR_CUDA(cudaMemsetAsync(total_out, 0, 4, s));
        return 0;
    }
    const uint32_t m = (uint32_t)((n_cap + SC_CHUNK - 1) / SC_CHUNK);
    scan_reduce_kernel<<<m, SC_THREADS, 0, s>>>(counts, n_cap, n_dev, tmp);
    count_launches(1);
    rowscan_wide_kernel<1><<<1, 1024, 0, s>>>(tmp, m, tmp + m);     // the partials in place, grand total -> tmp[m]
    count_launches(1);
    scan_apply_kernel<<<m, SC_THREADS, 0, s>>>(counts, n_cap, n_dev, tmp, m, out, total_out);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace gsr
