// densify.cu -- densification statistics of one training view in ONE pass over the Gaussians (SURVEY.md 8f-4).
//
// Replaces the PyTorch statements that consume the rasterizer's outputs right after the backward pass
// (wildgaussians/method.py:1997-1998 and GaussianModel.add_densification_stats, :1470-1477):
//     max_radii2D[vis]                = max(max_radii2D[vis], radii[vis])
//     xyz_grad[vis]                  += |viewspace_grad[vis, :2]|
//     xyz_gradient_accum_abs[vis]    += |viewspace_grad[vis, 2:]|            (use_gof_abs_gradient)
//     xyz_gradient_accum_abs_max[vis] = max(., |viewspace_grad[vis, 2:]|)
//     denom[vis]                     += 1
// with vis = radii > 0: five boolean-indexed gathers / scatters (each a nonzero() + index kernels + a host sync for
// the index count) become one bandwidth-bound kernel reading 16 B and touching 20 B per Gaussian.
#include "common.cuh"

namespace gsr {

__global__ void __launch_bounds__(256) densify_stats_kernel(int P, const int* __restrict__ radii,
                                                            const float* __restrict__ viewspace_grad,   // [P,3]
                                                            float* __restrict__ max_radii2D, float* __restrict__ xyz_grad,
                                                            float* __restrict__ accum_abs, float* __restrict__ accum_abs_max,
                                                            float* __restrict__ denom) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int r = radii[i];
    if (r <= 0) return;
    const float gx = viewspace_grad[3 * (size_t)i], gy = viewspace_grad[3 * (size_t)i + 1], gz = viewspace_grad[3 * (size_t)i + 2];
    max_radii2D[i] = fmaxf(max_radii2D[i], (float)r);
    xyz_grad[i] += sqrtf(gx * gx + gy * gy);               // torch.norm(grad[:, :2], dim=-1)
    if (accum_abs) {
        const float a = fabsf(gz);                          // torch.norm over the single column grad[:, 2:]
        accum_abs[i] += a;
        accum_abs_max[i] = fmaxf(accum_abs_max[i], a);
    }
    denom[i] += 1.0f;
}

}  // namespace gsr

extern "C" int gsr_densification_stats(int P, const int* radii, const float* viewspace_grad, float* max_radii2D, float* xyz_grad,
                                       float* xyz_gradient_accum_abs, float* xyz_gradient_accum_abs_max, float* denom, void* stream) {
    using namespace gsr;
    if (P < 0) { set_error("bad P"); return GSR_E_INVALID; }
    if (P == 0) return 0;
    if (!radii || !viewspace_grad || !max_radii2D || !xyz_grad || !denom || ((xyz_gradient_accum_abs == nullptr) != (xyz_gradient_accum_abs_max == nullptr))) {
        set_error("a required pointer is NULL");
        return GSR_E_INVALID;
    }
    densify_stats_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(P, radii, viewspace_grad, max_radii2D, xyz_grad,
                                                                            xyz_gradient_accum_abs, xyz_gradient_accum_abs_max, denom);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

// ================================================================================================================
// densify_and_prune (wildgaussians/method.py:1420-1468 with _densify_and_clone / _densify_and_split / _prune_points /
// _densification_postfix, :1280-1418) and reset_opacity (:1249-1278).
//
// Plan (gsr_densify_plan), all on the device, one read-back of the counts by the caller:
//   1. stats pass over P: grads_abs keys -> 2048-bin histogram of the top 11 key bits, and the count of |grad| >= max_grad
//      (the `ratio` of method.py:1433);
//   2. quantile select: ranks below / above of torch.quantile's linear interpolation, then two more short passes over
//      the 32-bit keys (11 + 11 + 10 bits of an MSD radix select, both ranks at once) -> Q;
//   3. fate pass over P: clone / split / final-prune decisions -> four 0/1 flags per row, laid out as four blocks of P;
//   4. ONE exclusive_scan_u32 over the 4P flags.  Because the blocks are scanned back to back, the scan of block b
//      already starts at the total of the blocks before it, so out[i] (survivors), out[P + i] (clones), out[2P + i]
//      (split copy 1; copy 2 adds the kept split count) are the rows' final positions in the reference's order, and
//      out[3P + i] - out[3P] is the rank of a split row among ALL split rows (its sample row in the normal draw);
//   5. one thread gathers the counts.
// Apply (gsr_densify_apply): one launch over row blocks; each CTA reads its rows' positions once and then walks every
// segment (parameter / moment / buffer), reading each source row once and writing it to its surviving, clone and split
// positions.  The split children's xyz and scales are computed on the fly.
//
// Arithmetic follows the reference's PyTorch statements operation by operation (separate roundings, no contraction):
// grads = xyz_grad / denom with NaN -> 0; the clone test uses torch.norm over the size-1 last dim (|g| on torch's CUDA
// build), the split test the padded vector itself; exp / sigmoid / log as torch's CUDA kernels evaluate them; a product
// over the 3 scales is reduced as (s0 s2) s1, as torch's reduction kernel splits a 3-element row over two threads.
// ================================================================================================================

namespace gsr {

#define PROD3(a, b, c) __fmul_rn(__fmul_rn((a), (c)), (b))

constexpr int DN_THREADS = 256;
constexpr int DN_ROWS = 256;              // rows per CTA of the apply kernel
constexpr int SEL_BINS = 2048;

struct SelState {                         // device words at the start of the scratch
    uint32_t n_ge;                        // rows with |grad| >= max_grad
    uint32_t clones;                      // rows selected for cloning (before the final prune)
    uint32_t big;                         // rows of the post-split set with max scale > prune_max_scale
    uint32_t k[2];                        // remaining rank of the lower / upper order statistic inside its prefix
    uint32_t prefix[2];                   // key bits fixed so far
    float weight;
    float Q;
    uint32_t pad[55];
};
static_assert(sizeof(SelState) == 64 * 4, "SelState is 64 words");

struct DensifyScratch {
    SelState* st;
    uint32_t* hist;                       // [5][SEL_BINS]: pass 1, pass 2 (x2 ranks), pass 3 (x2 ranks)
    uint32_t* flags;                      // [4P]
    uint32_t* out;                        // [4P + 1]
    uint32_t* scan_tmp;
};

static size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

static size_t carve_densify(char* base, int P, DensifyScratch* d) {
    const size_t n = 4 * (size_t)P;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* p = base + off; off += align16(bytes); return p; };
    char* st = take(sizeof(SelState));
    char* hist = take(5 * SEL_BINS * 4);
    char* flags = take(n * 4);
    char* out = take((n + 1) * 4);
    char* tmp = take(scan_tmp_elems(n) * 4);
    if (d) {
        d->st = reinterpret_cast<SelState*>(st);
        d->hist = reinterpret_cast<uint32_t*>(hist);
        d->flags = reinterpret_cast<uint32_t*>(flags);
        d->out = reinterpret_cast<uint32_t*>(out);
        d->scan_tmp = reinterpret_cast<uint32_t*>(tmp);
    }
    return off;
}

__device__ __forceinline__ float safe_ratio(float a, float b) {       // grads[grads.isnan()] = 0.0
    const float g = __fdiv_rn(a, b);
    return g != g ? 0.f : g;
}

// order-preserving key of a float (-0 is +0: torch's sort orders them as equal and every later use compares with >=)
__device__ __forceinline__ uint32_t float_key(float f) {
    uint32_t u = __float_as_uint(f);
    if (f == 0.f) u = 0u;
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float key_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

__device__ __forceinline__ float nanmax3(float a, float b, float c) {  // torch.max(dim=1): NaN propagates
    float m = a;
    if (!(m != m) && (b != b || b > m)) m = b;
    if (!(m != m) && (c != c || c > m)) m = c;
    return m;
}

__device__ __forceinline__ float sigmoid_ref(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

// pass 1: |grad| >= max_grad count and the histogram of the keys' top 11 bits
__global__ void __launch_bounds__(DN_THREADS) densify_stats_select_kernel(int P, const float* __restrict__ xyz_grad,
                                                                          const float* __restrict__ denom,
                                                                          const float* __restrict__ accum_abs, float max_grad,
                                                                          SelState* st, uint32_t* __restrict__ hist) {
    __shared__ uint32_t h[SEL_BINS];
    __shared__ uint32_t cnt;
    for (int b = threadIdx.x; b < SEL_BINS; b += DN_THREADS) h[b] = 0;
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    uint32_t ge = 0;
    for (size_t i = (size_t)blockIdx.x * DN_THREADS + threadIdx.x; i < (size_t)P; i += (size_t)gridDim.x * DN_THREADS) {
        const float d = denom[i];
        const float g = safe_ratio(xyz_grad[i], d);
        ge += fabsf(g) >= max_grad;                                   // torch.norm(grads, dim=-1) over one element: |g|
        atomicAdd(&h[float_key(safe_ratio(accum_abs[i], d)) >> 21], 1u);
    }
    atomicAdd(&cnt, ge);
    __syncthreads();
    for (int b = threadIdx.x; b < SEL_BINS; b += DN_THREADS)
        if (h[b]) atomicAdd(&hist[b], h[b]);
    if (threadIdx.x == 0) atomicAdd(&st->n_ge, cnt);
}

// passes 2 and 3: histogram of the next digit of the keys under each rank's prefix
template <int SHIFT_PREFIX, int SHIFT_DIGIT, int DIGIT_BITS>
__global__ void __launch_bounds__(DN_THREADS) densify_select_hist_kernel(int P, const float* __restrict__ denom,
                                                                         const float* __restrict__ accum_abs,
                                                                         const SelState* st, uint32_t* __restrict__ hist) {
    __shared__ uint32_t h[2][1 << DIGIT_BITS];
    for (int b = threadIdx.x; b < 2 << DIGIT_BITS; b += DN_THREADS) (&h[0][0])[b] = 0;
    __syncthreads();
    const uint32_t p0 = st->prefix[0], p1 = st->prefix[1];
    const uint32_t mask = (1u << DIGIT_BITS) - 1u;
    for (size_t i = (size_t)blockIdx.x * DN_THREADS + threadIdx.x; i < (size_t)P; i += (size_t)gridDim.x * DN_THREADS) {
        const uint32_t k = float_key(safe_ratio(accum_abs[i], denom[i]));
        const uint32_t pre = k >> SHIFT_PREFIX, dig = (k >> SHIFT_DIGIT) & mask;
        if (pre == p0) atomicAdd(&h[0][dig], 1u);
        if (pre == p1) atomicAdd(&h[1][dig], 1u);
    }
    __syncthreads();
    for (int b = threadIdx.x; b < 2 << DIGIT_BITS; b += DN_THREADS) {
        const uint32_t v = (&h[0][0])[b];
        if (v) atomicAdd(&hist[(b >> DIGIT_BITS) * SEL_BINS + (b & mask)], v);
    }
}

// one warp per rank: the digit whose cumulative count brackets the remaining rank; `stage` 0 first derives the ranks
// from the ratio exactly as torch.quantile(input, 1 - ratio) does (aten quantile: ranks = q * (n - 1), floor / ceil,
// weight = ranks - below), stage 2 finishes with torch.lerp
__global__ void __launch_bounds__(64) densify_select_step_kernel(int P, int stage, SelState* st, const uint32_t* __restrict__ hist,
                                                                 int bins, int digit_bits) {
    const int t = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __shared__ uint32_t k_s[2];
    if (stage == 0 && threadIdx.x == 0) {
        const float ratio = __fmul_rn((float)st->n_ge, __fdiv_rn(1.0f, (float)P));   // .float().mean(): sum * (1 / n)
        const float q = __fsub_rn(1.0f, ratio);
        float rank = __fmul_rn(q, (float)(P - 1));
        long long below = (long long)rank;
        const float w = __fsub_rn(rank, (float)below);
        long long above = (long long)ceilf(rank);
        // above 2^24 elements (where torch refuses) float(n - 1) may round up to n: clamp to the last index
        below = below > P - 1 ? P - 1 : below;
        above = above > P - 1 ? P - 1 : above;
        st->weight = w;
        k_s[0] = (uint32_t)below;
        k_s[1] = (uint32_t)above;
    } else if (stage != 0 && threadIdx.x < 2) {
        k_s[threadIdx.x] = st->k[threadIdx.x];
    }
    __syncthreads();
    const uint32_t* h = hist + (stage == 0 ? 0 : t * bins);
    const int per = bins / 32;
    uint32_t sum = 0;
    for (int j = 0; j < per; ++j) sum += h[lane * per + j];
    const uint32_t incl = warp_inclusive_scan(sum);
    const uint32_t k = k_s[t];
    const unsigned m = __ballot_sync(0xFFFFFFFFu, incl > k);
    const int L = __ffs(m) - 1;                                     // the lane holding the rank (m != 0: k < n)
    if (lane == L) {
        uint32_t c = incl - sum;
        int d = lane * per;
        for (; d < lane * per + per - 1; ++d) {
            if (c + h[d] > k) break;
            c += h[d];
        }
        const uint32_t prefix = (stage == 0 ? 0u : st->prefix[t]) << digit_bits | (uint32_t)d;
        st->prefix[t] = prefix;
        st->k[t] = k - c;
    }
    __syncthreads();
    if (stage == 2 && threadIdx.x == 0) {
        const float vb = key_float(st->prefix[0]), va = key_float(st->prefix[1]), w = st->weight;
        const float diff = __fsub_rn(va, vb);
        // at::lerp (ATen/native/Lerp.h): the weight < 0.5 form from below, the other from above
        // (torch's CUDA build contracts both forms into one fma each)
        st->Q = fabsf(w) < 0.5f ? fmaf(w, diff, vb) : fmaf(-diff, __fsub_rn(1.0f, w), va);
    }
}

// fate of every row: flags block 0 survivor, 1 kept clone, 2 kept split (both copies), 3 split (kept or not)
__global__ void __launch_bounds__(DN_THREADS) densify_fate_kernel(GsrDensifyArgs a, SelState* st, uint32_t* __restrict__ flags) {
    __shared__ uint32_t s_clone, s_big;
    if (threadIdx.x == 0) s_clone = s_big = 0;
    __syncthreads();
    const size_t P = (size_t)a.P;
    const bool use_abs = a.accum_abs != nullptr;
    const float Q = use_abs ? st->Q : 0.f;
    uint32_t n_clone = 0, n_big = 0;
    for (size_t i = (size_t)blockIdx.x * DN_THREADS + threadIdx.x; i < P; i += (size_t)gridDim.x * DN_THREADS) {
        const float d = a.denom[i];
        const float g = safe_ratio(a.xyz_grad[i], d);
        bool sel_clone = fabsf(g) >= a.max_grad;
        bool sel_split = g >= a.max_grad;
        if (use_abs) {
            const float ga = safe_ratio(a.accum_abs[i], d);
            sel_clone |= fabsf(ga) >= Q;
            sel_split |= ga >= Q;
        }
        const float s0 = expf(a.scales[3 * i]), s1 = expf(a.scales[3 * i + 1]), s2 = expf(a.scales[3 * i + 2]);
        const float m = nanmax3(s0, s1, s2);
        const bool clone = sel_clone && m <= a.clone_max_scale;
        const bool split = sel_split && m > a.clone_max_scale;
        const bool transparent = sigmoid_ref(a.opacities[i]) < a.min_opacity;
        bool keep;
        if (split) {
            const float c0 = expf(logf(__fmul_rn(s0, a.split_scale_mul))), c1 = expf(logf(__fmul_rn(s1, a.split_scale_mul))),
                        c2 = expf(logf(__fmul_rn(s2, a.split_scale_mul)));
            const bool big = nanmax3(c0, c1, c2) > a.prune_max_scale;
            keep = !(transparent || (a.size_pruning && big));
            n_big += big ? 2u : 0u;
        } else {
            const bool big = m > a.prune_max_scale;
            keep = !(transparent || (a.size_pruning && big));
            n_big += big ? (clone ? 2u : 1u) : 0u;
        }
        n_clone += clone;
        flags[i] = !split && keep;
        flags[P + i] = clone && keep;
        flags[2 * P + i] = split && keep;
        flags[3 * P + i] = split;
    }
    atomicAdd(&s_clone, n_clone);
    atomicAdd(&s_big, n_big);
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicAdd(&st->clones, s_clone);
        atomicAdd(&st->big, s_big);
    }
}

__global__ void densify_counts_kernel(int P, const SelState* st, const uint32_t* __restrict__ out, unsigned int* counts) {
    const size_t p = (size_t)P;
    const uint32_t kept_split = out[3 * p] - out[2 * p];
    counts[0] = st->clones;
    counts[1] = out[4 * p] - out[3 * p];                              // split rows
    counts[2] = out[3 * p] + kept_split;                              // rows after the final prune
    counts[3] = st->big;
    counts[4] = kept_split;
    counts[5] = st->n_ge;
    counts[6] = __float_as_uint(st->Q);
    counts[7] = 0;
}

struct DensifyApplyParams {
    GsrDensifySegment seg[GSR_DENSIFY_MAX_SEGMENTS];
    int num_segments;
};

__global__ void __launch_bounds__(DN_THREADS) densify_apply_kernel(const GsrDensifyArgs a, const uint32_t* __restrict__ out,
                                                                   const __grid_constant__ DensifyApplyParams sp) {
    __shared__ long long pos_keep[DN_ROWS], pos_clone[DN_ROWS], pos_child[DN_ROWS];
    __shared__ int rank_split[DN_ROWS];
    const size_t P = (size_t)a.P;
    const size_t r0 = (size_t)blockIdx.x * DN_ROWS;
    const int nr = (int)min((size_t)DN_ROWS, P - r0);
    const long long kept_split = (long long)out[3 * P] - (long long)out[2 * P];
    const int S = (int)(out[4 * P] - out[3 * P]);
    for (int r = threadIdx.x; r < nr; r += DN_THREADS) {
        const size_t i = r0 + r;
        pos_keep[r] = out[i + 1] != out[i] ? (long long)out[i] : -1;
        pos_clone[r] = out[P + i + 1] != out[P + i] ? (long long)out[P + i] : -1;
        pos_child[r] = out[2 * P + i + 1] != out[2 * P + i] ? (long long)out[2 * P + i] : -1;
        rank_split[r] = (int)(out[3 * P + i] - out[3 * P]);
    }
    __syncthreads();
    for (int s = 0; s < sp.num_segments; ++s) {
        const GsrDensifySegment g = sp.seg[s];
        const int w = g.width;
        const int n_el = nr * w;                                       // <= DN_ROWS * 4096
        const float* src = g.src + (long long)r0 * w;
        for (int e = threadIdx.x; e < n_el; e += DN_THREADS) {
            const int r = e / w, c = e - r * w;
            const float v = src[e];
            if (pos_keep[r] >= 0) g.dst[pos_keep[r] * w + c] = v;
            if (pos_clone[r] >= 0) g.dst[pos_clone[r] * w + c] = g.kind == GSR_DENSIFY_ZERO_NEW ? 0.f : v;
            if (pos_child[r] < 0) continue;
            const size_t i = r0 + r;
            float c1 = v, c2 = v;
            if (g.kind == GSR_DENSIFY_ZERO_NEW) {
                c1 = c2 = 0.f;
            } else if (g.kind == GSR_DENSIFY_SCALES) {                  // log(exp(s) / (0.8 N)), the division as a * (1 / b)
                c1 = c2 = logf(__fmul_rn(expf(v), a.split_scale_mul));
            } else if (g.kind == GSR_DENSIFY_XYZ) {
                // rots = build_rotation(normalize(rotations)); sample = normal(0, 1) * exp(s) + 0; xyz + rots @ sample
                float q[4] = {a.rotations[4 * i], a.rotations[4 * i + 1], a.rotations[4 * i + 2], a.rotations[4 * i + 3]};
                float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
                n = fmaxf(n, 1e-12f);                                   // F.normalize
#pragma unroll
                for (int k = 0; k < 4; ++k) q[k] /= n;
                const float n2 = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
                const float rr = q[0] / n2, x = q[1] / n2, y = q[2] / n2, z = q[3] / n2;
                float R[3];
                if (c == 0) { R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - rr * z); R[2] = 2.f * (x * z + rr * y); }
                else if (c == 1) { R[0] = 2.f * (x * y + rr * z); R[1] = 1.f - 2.f * (x * x + z * z); R[2] = 2.f * (y * z - rr * x); }
                else { R[0] = 2.f * (x * z - rr * y); R[1] = 2.f * (y * z + rr * x); R[2] = 1.f - 2.f * (x * x + y * y); }
                const float st0 = expf(a.scales[3 * i]), st1 = expf(a.scales[3 * i + 1]), st2 = expf(a.scales[3 * i + 2]);
                const float* z1 = a.normals + 3 * (size_t)rank_split[r];
                const float* z2 = a.normals + 3 * ((size_t)S + rank_split[r]);
                const float p0 = __fadd_rn(__fmul_rn(z1[0], st0), 0.f), p1 = __fadd_rn(__fmul_rn(z1[1], st1), 0.f),
                            p2 = __fadd_rn(__fmul_rn(z1[2], st2), 0.f);
                const float u0 = __fadd_rn(__fmul_rn(z2[0], st0), 0.f), u1 = __fadd_rn(__fmul_rn(z2[1], st1), 0.f),
                            u2 = __fadd_rn(__fmul_rn(z2[2], st2), 0.f);
                c1 = (R[0] * p0 + R[1] * p1 + R[2] * p2) + v;
                c2 = (R[0] * u0 + R[1] * u1 + R[2] * u2) + v;
            }
            g.dst[pos_child[r] * w + c] = c1;
            g.dst[(pos_child[r] + kept_split) * w + c] = c2;
        }
    }
}

// reset_opacity: logit(min(opacity_with_filter, 0.01) / coef) with the filtered scales' coef (method.py:1249-1266)
__global__ void __launch_bounds__(DN_THREADS) reset_opacity_kernel(int P, const float* __restrict__ opac,
                                                                   const float* __restrict__ scales,
                                                                   const float* __restrict__ filter_3D, float* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * DN_THREADS + threadIdx.x;
    if (i >= (size_t)P) return;
    const float f = filter_3D[i], f2 = __fmul_rn(f, f);
    float sq[3], sf2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float s = expf(scales[3 * i + k]);
        sq[k] = __fmul_rn(s, s);
        const float sf = __fsqrt_rn(__fadd_rn(sq[k], f2));            // get_gaussians: (s^2 + f^2).sqrt_()
        sf2[k] = __fmul_rn(sf, sf);
    }
    // get_gaussians' coefficient on the raw scales, then reset_opacity's own on the filtered ones
    const float det1 = PROD3(sq[0], sq[1], sq[2]);
    const float det2 = PROD3(__fadd_rn(sq[0], f2), __fadd_rn(sq[1], f2), __fadd_rn(sq[2], f2));
    const float op = __fmul_rn(sigmoid_ref(opac[i]), __fsqrt_rn(__fdiv_rn(det1, det2)));
    const float e1 = PROD3(sf2[0], sf2[1], sf2[2]);
    const float e2 = PROD3(__fadd_rn(sf2[0], f2), __fadd_rn(sf2[1], f2), __fadd_rn(sf2[2], f2));
    const float coef = __fsqrt_rn(__fdiv_rn(e1, e2));
    const float x = __fdiv_rn(fminf(op, 0.01f), coef);
    out[i] = logf(__fdiv_rn(x, __fsub_rn(1.0f, x)));                    // torch.special.logit without eps
}

}  // namespace gsr

extern "C" size_t gsr_densify_scratch_bytes(int P) {
    if (P < 0 || P > GSR_DENSIFY_MAX_P) return 0;
    return gsr::carve_densify(nullptr, P, nullptr);
}

static int densify_check(const GsrDensifyArgs* a) {
    using namespace gsr;
    if (!a) { set_error("args is NULL"); return GSR_E_INVALID; }
    if (a->P < 1 || a->P > GSR_DENSIFY_MAX_P) { set_error("P must be in [1, %d]", GSR_DENSIFY_MAX_P); return GSR_E_INVALID; }
    if (!a->xyz_grad || !a->denom || !a->xyz || !a->scales || !a->rotations || !a->opacities || !a->scratch || !a->counts) {
        set_error("a required pointer is NULL");
        return GSR_E_INVALID;
    }
    if (((uintptr_t)a->scratch & 15u) != 0) { set_error("scratch must be 16-byte aligned"); return GSR_E_INVALID; }
    return 0;
}

extern "C" int gsr_densify_plan(const GsrDensifyArgs* a, void* stream) {
    using namespace gsr;
    if (int rc = densify_check(a)) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    DensifyScratch d;
    carve_densify((char*)a->scratch, a->P, &d);
    GSR_CUDA(cudaMemsetAsync(d.st, 0, sizeof(SelState) + 5 * SEL_BINS * 4, s));
    const int ctas = (int)min((a->P + DN_THREADS - 1) / DN_THREADS, 132 * 8);
    if (a->accum_abs) {
        densify_stats_select_kernel<<<ctas, DN_THREADS, 0, s>>>(a->P, a->xyz_grad, a->denom, a->accum_abs, a->max_grad, d.st, d.hist);
        densify_select_step_kernel<<<1, 64, 0, s>>>(a->P, 0, d.st, d.hist, SEL_BINS, 11);
        densify_select_hist_kernel<21, 10, 11><<<ctas, DN_THREADS, 0, s>>>(a->P, a->denom, a->accum_abs, d.st, d.hist + SEL_BINS);
        densify_select_step_kernel<<<1, 64, 0, s>>>(a->P, 1, d.st, d.hist + SEL_BINS, SEL_BINS, 11);
        densify_select_hist_kernel<10, 0, 10><<<ctas, DN_THREADS, 0, s>>>(a->P, a->denom, a->accum_abs, d.st, d.hist + 3 * SEL_BINS);
        densify_select_step_kernel<<<1, 64, 0, s>>>(a->P, 2, d.st, d.hist + 3 * SEL_BINS, SEL_BINS, 10);
        count_launches(6);
    }
    densify_fate_kernel<<<ctas, DN_THREADS, 0, s>>>(*a, d.st, d.flags);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    if (int rc = exclusive_scan_u32(d.flags, d.out, 4 * (size_t)a->P, d.scan_tmp, s)) return rc;
    densify_counts_kernel<<<1, 1, 0, s>>>(a->P, d.st, d.out, a->counts);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int gsr_densify_apply(const GsrDensifyArgs* a, const GsrDensifySegment* segments, int num_segments, void* stream) {
    using namespace gsr;
    if (int rc = densify_check(a)) return rc;
    if (num_segments < 0 || num_segments > GSR_DENSIFY_MAX_SEGMENTS || (num_segments && !segments)) {
        set_error("num_segments must be in [0, %d]", GSR_DENSIFY_MAX_SEGMENTS);
        return GSR_E_INVALID;
    }
    DensifyApplyParams sp{};
    for (int i = 0; i < num_segments; ++i) {
        const GsrDensifySegment& g = segments[i];
        if (!g.src || !g.dst || g.width < 1 || g.width > 4096 || g.kind < GSR_DENSIFY_COPY || g.kind > GSR_DENSIFY_SCALES ||
            ((g.kind == GSR_DENSIFY_XYZ || g.kind == GSR_DENSIFY_SCALES) && g.width != 3)) {
            set_error("segment %d: bad pointer, width or kind", i);
            return GSR_E_INVALID;
        }
        sp.seg[i] = g;
    }
    sp.num_segments = num_segments;
    if (num_segments == 0) return 0;
    DensifyScratch d;
    carve_densify((char*)a->scratch, a->P, &d);
    const unsigned ctas = (unsigned)((a->P + DN_ROWS - 1) / DN_ROWS);
    densify_apply_kernel<<<ctas, DN_THREADS, 0, (cudaStream_t)stream>>>(*a, d.out, sp);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int gsr_reset_opacity(int P, const float* opacities, const float* scales, const float* filter_3D, float* out,
                                 void* stream) {
    using namespace gsr;
    if (P < 0) { set_error("bad P"); return GSR_E_INVALID; }
    if (P == 0) return 0;
    if (!opacities || !scales || !filter_3D || !out) { set_error("a required pointer is NULL"); return GSR_E_INVALID; }
    reset_opacity_kernel<<<(unsigned)((P + DN_THREADS - 1) / DN_THREADS), DN_THREADS, 0, (cudaStream_t)stream>>>(
        P, opacities, scales, filter_3D, out);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}
