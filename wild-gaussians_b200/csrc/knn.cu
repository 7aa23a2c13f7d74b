// knn.cu -- mean squared distance of every point to its 3 nearest neighbours (SURVEY.md 8f-4).
//
// Replaces `distCUDA2` of the reference's simple-knn submodule (spatial.cu:15-26 -> SimpleKNN::knn,
// simple_knn.cu:185-220), which initialises the Gaussian scales from the SfM point cloud (method.py:1001).
// Same result: for every point the three smallest values of fma(dz, dz, fma(dx, dx, dy * dy)) over all OTHER points
// (identity, not coordinates, excludes the point itself: duplicates count with distance 0), summed smallest first
// and divided by 3.0f -- the multiset of three smallest distances does not depend on the search order, so an exact
// search with another acceleration structure yields the same bits.
//
// Design (not the reference's: it sorts by Morton code with CUB, builds ONE level of 1024-point boxes and lets every
// point test all P/1024 boxes and then scan whole 1024-point boxes, ~10^4 distance tests per point):
//   * 63-bit Morton codes (21 bits per axis: SfM clouds mix very dense clusters with far outliers, 10 bits per axis as in
//     the reference would leave thousands of points per cell), sorted by two stable passes of this library's 32-bit radix
//     sort (radix.cu; low word, then high word); points are copied into Morton order ({x, y, z, original index} as one
//     float4) so every later access is coalesced;
//   * a 32-ary hierarchy of axis-aligned boxes over the sorted points: leaves of 32 points (one warp, shuffles),
//     then boxes of 32 children, up to a top level of <= 1024 boxes;
//   * one thread per point walks the hierarchy top-down with the reference's pruning rule (skip a box whose distance
//     exceeds the current third-best / the bound from the 3 + 3 Morton neighbours).  Neighbouring threads are neighbouring
//     points, so a warp tests (almost) the same boxes: the box loads are broadcasts and divergence stays small.
//     About 300-600 tests per point instead of ~10^4.
// The box distance is evaluated with round-down arithmetic, which makes it a rigorous lower bound of the fp32 distance
// of every point inside the box: no true neighbour is ever pruned by a rounding coincidence.
#include "common.cuh"
#include <cfloat>

namespace gsr {

constexpr int KNN_THREADS = 256;
constexpr int KNN_FAN = 32;
constexpr int KNN_MAX_LEVELS = 6;          // 32^6 points

struct KnnBox { float4 lo, hi; };          // {min.x, min.y, min.z, -}, {max.x, max.y, max.z, -}

// order-preserving float <-> int map for atomicMin / atomicMax
__device__ __forceinline__ int f2ord(float f) { const int i = __float_as_int(f); return i ^ ((i >> 31) & 0x7FFFFFFF); }
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i ^ ((i >> 31) & 0x7FFFFFFF)); }

__global__ void __launch_bounds__(KNN_THREADS) knn_bbox_kernel(int P, const float* __restrict__ pts, int* __restrict__ bbox /*[6]*/) {
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int i = blockIdx.x * KNN_THREADS + threadIdx.x; i < P; i += gridDim.x * KNN_THREADS) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { const float v = pts[3 * (size_t)i + c]; lo[c] = fminf(lo[c], v); hi[c] = fmaxf(hi[c], v); }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[c] = fminf(lo[c], __shfl_xor_sync(0xFFFFFFFFu, lo[c], o));
            hi[c] = fmaxf(hi[c], __shfl_xor_sync(0xFFFFFFFFu, hi[c], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { atomicMin(&bbox[c], f2ord(lo[c])); atomicMax(&bbox[3 + c], f2ord(hi[c])); }
    }
}

__device__ __forceinline__ unsigned long long spread21(unsigned long long x) {     // 21 bits -> every third bit
    x = (x | (x << 32)) & 0x001F00000000FFFFull;
    x = (x | (x << 16)) & 0x001F0000FF0000FFull;
    x = (x | (x << 8)) & 0x100F00F00F00F00Full;
    x = (x | (x << 4)) & 0x10C30C30C30C30C3ull;
    x = (x | (x << 2)) & 0x1249249249249249ull;
    return x;
}

__global__ void __launch_bounds__(KNN_THREADS) knn_morton_kernel(int P, const float* __restrict__ pts, const int* __restrict__ bbox,
                                                                 uint32_t* __restrict__ key_lo, uint32_t* __restrict__ key_hi,
                                                                 uint32_t* __restrict__ val) {
    const int i = blockIdx.x * KNN_THREADS + threadIdx.x;
    if (i >= P) return;
    unsigned long long code = 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float lo = ord2f(bbox[c]), hi = ord2f(bbox[3 + c]);
        const float ext = hi - lo;
        float t = ext > 0.f ? (pts[3 * (size_t)i + c] - lo) / ext : 0.f;
        t = fminf(fmaxf(t, 0.f), 1.f);          // NaN coordinates land in cell 0; they only affect the ORDER, never the result
        code |= spread21((unsigned long long)(t * 2097151.0f)) << c;
    }
    key_lo[i] = (uint32_t)code;
    key_hi[i] = (uint32_t)(code >> 32);
    val[i] = (uint32_t)i;
}

// keys of the second (high word) sort in the order the first sort produced
__global__ void __launch_bounds__(KNN_THREADS) knn_regather_kernel(int P, const uint32_t* __restrict__ key_hi, const uint32_t* __restrict__ order,
                                                                   uint32_t* __restrict__ key) {
    const int i = blockIdx.x * KNN_THREADS + threadIdx.x;
    if (i < P) key[i] = key_hi[order[i]];
}

// points into Morton order + the leaf boxes (one warp = one leaf of 32 consecutive sorted points)
__global__ void __launch_bounds__(KNN_THREADS) knn_gather_kernel(int P, const float* __restrict__ pts, const uint32_t* __restrict__ order,
                                                                 float4* __restrict__ sorted, KnnBox* __restrict__ leaf) {
    const int i = blockIdx.x * KNN_THREADS + threadIdx.x;
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    if (i < P) {
        const uint32_t id = order[i];
        const float x = pts[3 * (size_t)id], y = pts[3 * (size_t)id + 1], z = pts[3 * (size_t)id + 2];
        sorted[i] = make_float4(x, y, z, __uint_as_float(id));
        lo[0] = hi[0] = x; lo[1] = hi[1] = y; lo[2] = hi[2] = z;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[c] = fminf(lo[c], __shfl_xor_sync(0xFFFFFFFFu, lo[c], o));
            hi[c] = fmaxf(hi[c], __shfl_xor_sync(0xFFFFFFFFu, hi[c], o));
        }
    }
    if ((threadIdx.x & 31) == 0 && i < P) leaf[i >> 5] = {make_float4(lo[0], lo[1], lo[2], 0.f), make_float4(hi[0], hi[1], hi[2], 0.f)};
}

// parent boxes: one warp per parent, lane = child
__global__ void __launch_bounds__(KNN_THREADS) knn_level_kernel(int n_child, const KnnBox* __restrict__ child, KnnBox* __restrict__ parent) {
    const int i = blockIdx.x * KNN_THREADS + threadIdx.x;
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    if (i < n_child) {
        const KnnBox b = child[i];
        lo[0] = b.lo.x; lo[1] = b.lo.y; lo[2] = b.lo.z; hi[0] = b.hi.x; hi[1] = b.hi.y; hi[2] = b.hi.z;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[c] = fminf(lo[c], __shfl_xor_sync(0xFFFFFFFFu, lo[c], o));
            hi[c] = fmaxf(hi[c], __shfl_xor_sync(0xFFFFFFFFu, hi[c], o));
        }
    }
    if ((threadIdx.x & 31) == 0 && i < n_child) parent[i >> 5] = {make_float4(lo[0], lo[1], lo[2], 0.f), make_float4(hi[0], hi[1], hi[2], 0.f)};
}

// rigorous lower bound (round-down arithmetic) of the squared distance from p to any point inside the box
__device__ __forceinline__ float box_dist_lb(const KnnBox& b, const float3 p) {
    const float dx = fmaxf(fmaxf(b.lo.x - p.x, p.x - b.hi.x), 0.f);       // exact differences are rounded monotonically
    const float dy = fmaxf(fmaxf(b.lo.y - p.y, p.y - b.hi.y), 0.f);
    const float dz = fmaxf(fmaxf(b.lo.z - p.z, p.z - b.hi.z), 0.f);
    return __fmaf_rd(dz, dz, __fmaf_rd(dx, dx, __fmul_rd(dy, dy)));      // same nesting as point_dist: bound holds step by step
}

// the reference's distance expression d.x*d.x + d.y*d.y + d.z*d.z (simple_knn.cu:134-135) as nvcc contracts it in the
// reference build: FMUL on the y term, then FFMA x, FFMA z (read off its SASS; pinned by the golden outputs: with any
// other nesting ~10 % of the results differ in the last bit)
__device__ __forceinline__ float point_dist(const float3 p, const float4 q) {
    const float dx = q.x - p.x, dy = q.y - p.y, dz = q.z - p.z;
    return fmaf(dz, dz, fmaf(dx, dx, __fmul_rn(dy, dy)));
}

__device__ __forceinline__ void keep3(float (&best)[3], float d) {       // simple_knn.cu:136-144
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        if (best[j] > d) { const float t = best[j]; best[j] = d; d = t; }
    }
}

struct KnnLevels {
    const KnnBox* box[KNN_MAX_LEVELS];     // box[0] = leaves (32 points each), box[l + 1] = parents of box[l]
    int count[KNN_MAX_LEVELS];
    int top;                               // index of the top level
};

template <int LEVEL>
__device__ __forceinline__ void knn_descend(const KnnLevels& L, int node, const float4* __restrict__ sorted, int P, int self,
                                            const float3 p, const float reject, float (&best)[3]) {
    // children of `node` at level LEVEL - 1 (points for LEVEL == 0)
    if constexpr (LEVEL == 0) {
        const int j0 = node * KNN_FAN, j1 = min(P, j0 + KNN_FAN);
        for (int j = j0; j < j1; ++j) {
            if (j == self) continue;
            keep3(best, point_dist(p, sorted[j]));
        }
    } else {
        const int c0 = node * KNN_FAN, c1 = min(L.count[LEVEL - 1], c0 + KNN_FAN);
        for (int c = c0; c < c1; ++c) {
            const float d = box_dist_lb(L.box[LEVEL - 1][c], p);
            if (d > reject || d > best[2]) continue;                     // simple_knn.cu:169-171
            knn_descend<LEVEL - 1>(L, c, sorted, P, self, p, reject, best);
        }
    }
}

__global__ void __launch_bounds__(KNN_THREADS) knn_query_kernel(int P, const float4* __restrict__ sorted, const __grid_constant__ KnnLevels L,
                                                                float* __restrict__ out) {
    const int i = blockIdx.x * KNN_THREADS + threadIdx.x;
    if (i >= P) return;
    const float4 me = sorted[i];
    const float3 p = {me.x, me.y, me.z};
    float best[3] = {FLT_MAX, FLT_MAX, FLT_MAX};
    // a first bound from the 3 + 3 neighbours in Morton order (simple_knn.cu:155-160)
    for (int j = max(0, i - 3); j <= min(P - 1, i + 3); ++j) {
        if (j == i) continue;
        keep3(best, point_dist(p, sorted[j]));
    }
    const float reject = best[2];
    best[0] = best[1] = best[2] = FLT_MAX;
    for (int t = 0; t < L.count[L.top]; ++t) {
        const float d = box_dist_lb(L.box[L.top][t], p);
        if (d > reject || d > best[2]) continue;
        switch (L.top) {
            case 0: knn_descend<0>(L, t, sorted, P, i, p, reject, best); break;
            case 1: knn_descend<1>(L, t, sorted, P, i, p, reject, best); break;
            case 2: knn_descend<2>(L, t, sorted, P, i, p, reject, best); break;
            case 3: knn_descend<3>(L, t, sorted, P, i, p, reject, best); break;
            case 4: knn_descend<4>(L, t, sorted, P, i, p, reject, best); break;
            default: knn_descend<5>(L, t, sorted, P, i, p, reject, best); break;
        }
    }
    out[__float_as_uint(me.w)] = __fdiv_rn(__fadd_rn(__fadd_rn(best[0], best[1]), best[2]), 3.0f);   // simple_knn.cu:182
}

static size_t knn_align(size_t x) { return (x + 255) & ~(size_t)255; }

struct KnnScratch {
    int* bbox;
    uint32_t *key_a, *val_a, *key_b, *val_b, *key_hi, *radix_tmp;
    float4* sorted;
    KnnBox* boxes;          // all levels, leaves first
    size_t bytes;
};

static KnnScratch knn_carve(char* base, int P) {
    KnnScratch s{};
    size_t off = 0;
    auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += knn_align(bytes); return p; };
    s.bbox = reinterpret_cast<int*>(take(256));
    s.key_a = reinterpret_cast<uint32_t*>(take((size_t)P * 4));
    s.val_a = reinterpret_cast<uint32_t*>(take((size_t)P * 4));
    s.key_b = reinterpret_cast<uint32_t*>(take((size_t)P * 4));
    s.val_b = reinterpret_cast<uint32_t*>(take((size_t)P * 4));
    s.key_hi = reinterpret_cast<uint32_t*>(take((size_t)P * 4));
    s.radix_tmp = reinterpret_cast<uint32_t*>(take(radix_tmp_elems((size_t)P) * 4));
    s.sorted = reinterpret_cast<float4*>(take((size_t)P * 16));
    size_t nboxes = 0;
    for (size_t n = ((size_t)P + KNN_FAN - 1) / KNN_FAN;; n = (n + KNN_FAN - 1) / KNN_FAN) { nboxes += n; if (n <= 1) break; }
    s.boxes = reinterpret_cast<KnnBox*>(take(nboxes * sizeof(KnnBox)));
    s.bytes = off;
    return s;
}

}  // namespace gsr

extern "C" size_t gsr_knn_scratch_bytes(int P) { return P > 0 ? gsr::knn_carve(nullptr, P).bytes : 0; }

extern "C" int gsr_knn_mean_dist2(int P, const float* points, float* mean_dist2, void* scratch, void* stream) {
    using namespace gsr;
    if (P < 0) { set_error("bad P"); return GSR_E_INVALID; }
    if (P == 0) return 0;
    if (!points || !mean_dist2 || !scratch) { set_error("a required pointer is NULL"); return GSR_E_INVALID; }
    if (reinterpret_cast<uintptr_t>(scratch) & 255u) { set_error("scratch must be 256-byte aligned"); return GSR_E_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    const KnnScratch k = knn_carve(reinterpret_cast<char*>(scratch), P);
    const int grid = (P + KNN_THREADS - 1) / KNN_THREADS;
    // bounding box (ordered-int encoding: min slots start at +max, max slots at -max)
    const int init[6] = {0x7F7FFFFF, 0x7F7FFFFF, 0x7F7FFFFF, (int)0x80800000, (int)0x80800000, (int)0x80800000};
    GSR_CUDA(cudaMemcpyAsync(k.bbox, init, sizeof(init), cudaMemcpyHostToDevice, s));
    knn_bbox_kernel<<<min(grid, 132 * 8), KNN_THREADS, 0, s>>>(P, points, k.bbox);
    knn_morton_kernel<<<grid, KNN_THREADS, 0, s>>>(P, points, k.bbox, k.key_a, k.key_hi, k.val_a);
    count_launches(2);
    GSR_CUDA(cudaGetLastError());
    // stable LSD sort of the 63-bit codes: low word (4 passes, result back in A), then high word (31 bits, 4 passes)
    int rc = radix_sort_pairs(k.key_a, k.val_a, k.key_b, k.val_b, (size_t)P, 0, 32, k.radix_tmp, s, false);
    if (rc) return rc;
    if (radix_num_passes(0, 32) % 2 != 0) { set_error("internal: odd number of radix passes"); return GSR_E_INVALID; }
    knn_regather_kernel<<<grid, KNN_THREADS, 0, s>>>(P, k.key_hi, k.val_a, k.key_a);
    count_launches(1);
    rc = radix_sort_pairs(k.key_a, k.val_a, k.key_b, k.val_b, (size_t)P, 0, 32, k.radix_tmp, s, false);
    if (rc) return rc;
    const uint32_t* order = k.val_a;
    KnnLevels L{};
    int n = (P + KNN_FAN - 1) / KNN_FAN;
    KnnBox* level = k.boxes;
    knn_gather_kernel<<<grid, KNN_THREADS, 0, s>>>(P, points, order, k.sorted, level);
    count_launches(1);
    L.box[0] = level; L.count[0] = n; L.top = 0;
    // further levels until the top one is small enough to be scanned linearly by every thread
    while (n > 1024 && L.top + 1 < KNN_MAX_LEVELS) {
        const int np = (n + KNN_FAN - 1) / KNN_FAN;
        KnnBox* parent = level + n;
        knn_level_kernel<<<(n + KNN_THREADS - 1) / KNN_THREADS, KNN_THREADS, 0, s>>>(n, level, parent);
        count_launches(1);
        ++L.top;
        L.box[L.top] = parent; L.count[L.top] = np;
        level = parent; n = np;
    }
    knn_query_kernel<<<grid, KNN_THREADS, 0, s>>>(P, k.sorted, L, mean_dist2);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}
