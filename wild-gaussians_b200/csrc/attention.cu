// attention.cu -- exact softmax attention, forward only, for the DINOv2 backbone of wild-gaussians' uncertainty model.
//
// What it replaces: the core of `Attention.forward` (wildgaussians/dinov2.py:224-233) from the `qkv` Linear's output to
// the input of `proj`:  q = qkv[0] * 1/8,  softmax(q k^T) v,  heads concatenated.  Every DINOv2 variant has 64-wide
// heads; the head count H is free.  Input [B, N, 3, H, 64] fp32 as the Linear wrote it, output [B, N, H * 64] fp32.
//
// Two launches:
//   1. attention_split_kernel: per (batch, head, 64-key tile), one 80 KB image of the tile's K, split into tf32
//      hi + lo, and V, split exactly into tf32 hi + mid + lo, in the shared-memory layout the tensor cores read
//      (wgmma.cuh, K-major rows16).  K [key][dim] is K-major for S = Q K^T as it is; V is transposed to [dim][key] so
//      that it is K-major for O = P V.  Keys at or beyond N are zeros.
//   2. attention_fwd_kernel: one CTA per (128 query rows, head, batch): two consumer warpgroups of 64 rows each and one
//      producer warp that streams the tile images through a 2-stage ring with 1-D bulk copies (mbarriers for full and
//      empty).  Q (scaled by 1/8, which is exact) is split once into hi / lo images in shared memory.  Per key tile each
//      warpgroup runs S = Qlo Khi + Qhi Klo + Qhi Khi (24 wgmma m64n64k8), masks keys >= N, updates the running row
//      maximum and sum (online softmax, O and the sum rescaled by exp(m_old - m_new)), splits P = exp(S - m) into
//      tf32 hi + lo in registers, runs Plo Vhi + Phi (Vlo + Vmid + Vhi) (32 more) into a per-tile accumulator and adds
//      that to O in fp32.  O / sum is stored once.
// Split scheme: each 3xTF32 product drops lo * lo and rounds the lo parts, O(2^-22) relative, the size of the fp32
// reference's own rounding in q k^T and exp.  V is split exactly (11 + 11 + 11 bits cover fp32's 24) because one
// dominant key passes its V row through unchanged in the reference (N = 1 is exact there, and here).
// Nothing of size N^2 reaches memory; the scratch is B * H * ceil(N / 64) * 80 KB.  No atomics: bitwise reproducible.
//
// P as an A operand without a shuffle: the accumulator fragment gives lane (g, t) keys 8j + 2t and 8j + 2t + 1 of
// chunk j, the tf32 A fragment wants k-slots t and t + 4.  Slot t is therefore key 8j + 2t and slot t + 4 key
// 8j + 2t + 1; the split kernel stores V^T's keys in that slot order (even keys of each group of 8 first, then odd),
// so the contraction pairs every P column with its own V row.
#include "common.cuh"
#include "wgmma.cuh"

namespace gsr {
namespace {

constexpr int ATT_D = 64;                         // head dimension
constexpr int ATT_BN = 64;                        // keys per tile
constexpr int ATT_WG = 2;                         // consumer warpgroups per CTA, 64 query rows each
constexpr int ATT_BM = 64 * ATT_WG;               // query rows per CTA
constexpr int ATT_STAGES = 2;
constexpr int ATT_THREADS = 128 * ATT_WG + 32;    // + the producer warp
constexpr int ATT_PART = ATT_BN * ATT_D;          // floats of one operand image (16 KB)
constexpr int ATT_TILE = 5 * ATT_PART;            // K hi, K lo, V^T hi, V^T mid, V^T lo
constexpr int ATT_TILE_BYTES = ATT_TILE * 4;
constexpr size_t ATT_SMEM = (size_t)ATT_STAGES * ATT_TILE_BYTES + (size_t)ATT_WG * 2 * ATT_PART * 4 +   // K/V ring, Q hi / lo
                            2 * ATT_STAGES * sizeof(uint64_t);
constexpr int SPLIT_THREADS = 256;

// grid (T, H, B): one 80 KB image per (key tile, head, batch) at img + ((b * H + h) * T + tile) * ATT_TILE
__global__ void __launch_bounds__(SPLIT_THREADS) attention_split_kernel(int N, int H, int T, const float* __restrict__ qkv,
                                                                        float* __restrict__ img) {
    const int tile = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const size_t row_stride = (size_t)3 * H * ATT_D;
    const float* kb = qkv + (size_t)b * N * row_stride + (size_t)H * ATT_D + (size_t)h * ATT_D;   // K of (b, 0, h)
    const float* vb = kb + (size_t)H * ATT_D;
    float* dst = img + (((size_t)b * H + h) * T + tile) * ATT_TILE;
    const int key0 = tile * ATT_BN;
    // K: 16-byte unit (key, dims 4u..4u+3) at float offset (u * 64 + key) * 4
    for (int i = threadIdx.x; i < ATT_BN * ATT_D / 4; i += SPLIT_THREADS) {
        const int key = i % ATT_BN, u = i / ATT_BN, n = key0 + key;
        const float4 v = n < N ? *reinterpret_cast<const float4*>(kb + (size_t)n * row_stride + 4 * u) : make_float4(0, 0, 0, 0);
        float4 lo;
        const float4 hi = wg::split_tf32x4(v, lo);
        *reinterpret_cast<float4*>(dst + (u * ATT_BN + key) * 4) = hi;
        *reinterpret_cast<float4*>(dst + ATT_PART + (u * ATT_BN + key) * 4) = lo;
    }
    // V^T: 16-byte unit (dim, slots 4q..4q+3) at float offset (q * 64 + dim) * 4; slot 4q + i of key chunk c = q / 2 is
    // key 8c + 2i + (q % 2)
    for (int i = threadIdx.x; i < ATT_D * ATT_BN / 4; i += SPLIT_THREADS) {
        const int dim = i % ATT_D, q = i / ATT_D;
        float e[4];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            const int n = key0 + 8 * (q / 2) + 2 * s + (q % 2);
            e[s] = n < N ? vb[(size_t)n * row_stride + dim] : 0.f;
        }
        float4 rest, lo;
        const float4 hi = wg::split_tf32x4(make_float4(e[0], e[1], e[2], e[3]), rest);
        const float4 mid = wg::split_tf32x4(make_float4(e[0] - hi.x, e[1] - hi.y, e[2] - hi.z, e[3] - hi.w), lo);   // exact
        *reinterpret_cast<float4*>(dst + 2 * ATT_PART + (q * ATT_D + dim) * 4) = hi;
        *reinterpret_cast<float4*>(dst + 3 * ATT_PART + (q * ATT_D + dim) * 4) = mid;
        *reinterpret_cast<float4*>(dst + 4 * ATT_PART + (q * ATT_D + dim) * 4) = lo;
    }
}

template <int N>
__device__ __forceinline__ void keep_regs(uint32_t (&r)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}

// grid (ceil(N / 128), H, B)
__global__ void __launch_bounds__(ATT_THREADS, 1) attention_fwd_kernel(int N, int H, int T, const float* __restrict__ qkv,
                                                                       const float* __restrict__ img, float* __restrict__ out) {
    using namespace wg;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* tiles = reinterpret_cast<float*>(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + ATT_SMEM - 2 * ATT_STAGES * sizeof(uint64_t));
    uint64_t* empty = full + ATT_STAGES;
    const int h = blockIdx.y, b = blockIdx.z;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    if (threadIdx.x == 0) {
        for (int s = 0; s < ATT_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 4 * ATT_WG);          // one arrive per consumer warp
        }
        mbar_init_fence();
    }
    __syncthreads();

    if (warp == 4 * ATT_WG) {                          // producer
        if (lane == 0) {
            const float* src = img + ((size_t)b * H + h) * T * ATT_TILE;
            for (int i = 0; i < T; ++i) {
                const int s = i % ATT_STAGES;
                if (i >= ATT_STAGES && !mbar_wait(&empty[s], ((i / ATT_STAGES) - 1) & 1)) return;
                mbar_expect_tx(&full[s], ATT_TILE_BYTES);
                bulk_g2s(tiles + (size_t)s * ATT_TILE, src + (size_t)i * ATT_TILE, ATT_TILE_BYTES, &full[s]);
            }
        }
        return;
    }

    const int wgi = warp / 4, g = lane / 4, t = lane % 4;
    const int row0 = blockIdx.x * ATT_BM + wgi * 64 + 16 * (warp % 4) + g;     // this thread's rows: row0, row0 + 8
    // this warpgroup's 64 query rows, scaled by 1/8 and split, K-major like K: unit (row, dims 4u..4u+3) at (u * 64 + row) * 4
    float* qs = tiles + (size_t)ATT_STAGES * ATT_TILE + (size_t)wgi * 2 * ATT_PART;
    {
        const size_t row_stride = (size_t)3 * H * ATT_D;
        const float* qb = qkv + (size_t)b * N * row_stride + (size_t)h * ATT_D;
        const int wrow0 = blockIdx.x * ATT_BM + wgi * 64;
        for (int i = threadIdx.x % 128; i < 64 * ATT_D / 4; i += 128) {
            const int r = i % 64, u = i / 64, row = wrow0 + r;
            float4 v = row < N ? *reinterpret_cast<const float4*>(qb + (size_t)row * row_stride + 4 * u) : make_float4(0, 0, 0, 0);
            v = make_float4(v.x * 0.125f, v.y * 0.125f, v.z * 0.125f, v.w * 0.125f);
            float4 lo;
            const float4 hi = wg::split_tf32x4(v, lo);
            *reinterpret_cast<float4*>(qs + (u * 64 + r) * 4) = hi;
            *reinterpret_cast<float4*>(qs + ATT_PART + (u * 64 + r) * 4) = lo;
        }
        fence_async_smem();
        warpgroup_sync(wgi);
    }
    const uint32_t qbase = smem_u32(qs);

    float o[32], ot[32], sa[32], sb[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = ot[i] = sa[i] = sb[i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows row0 and row0 + 8; l: this thread's columns only
    bool ok = true;
    for (int i = 0; i < T; ++i) {
        const int s = i % ATT_STAGES;
        if (!mbar_wait(&full[s], (i / ATT_STAGES) & 1)) { ok = false; break; }
        const uint32_t base = smem_u32(tiles + (size_t)s * ATT_TILE);
        // Hopper's tensor cores add each k-step's products to the accumulator with truncation at the accumulator's
        // precision, so every k-step costs up to one ulp of the running sum.  The small split terms therefore go first,
        // while the sum is small, and the hi * hi steps are spread over two accumulators added in fp32.
        fence();
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            mma_tf32_n64(sa, smem_desc(qbase + ATT_PART * 4 + c * 2048, 64 * 16, 128), smem_desc(base + c * 2048, ATT_BN * 16, 128), c > 0);
            mma_tf32_n64(sa, smem_desc(qbase + c * 2048, 64 * 16, 128), smem_desc(base + ATT_PART * 4 + c * 2048, ATT_BN * 16, 128), true);
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const uint64_t qhi = smem_desc(qbase + c * 2048, 64 * 16, 128), khi = smem_desc(base + c * 2048, ATT_BN * 16, 128);
            if (c < 4) mma_tf32_n64(sa, qhi, khi, true);
            else mma_tf32_n64(sb, qhi, khi, c > 4);
        }
        commit_group();
        wait_all();
        fence_regs(sa);
        fence_regs(sb);
        float sc[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) sc[k] = sa[k] + sb[k];

        const int key0 = i * ATT_BN;
        if (key0 + ATT_BN > N) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (key0 + 8 * j + 2 * t + e >= N) sc[4 * j + e] = sc[4 * j + 2 + e] = -INFINITY;
        }
        float mx0 = m0, mx1 = m1;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            mx0 = fmaxf(mx0, fmaxf(sc[4 * j], sc[4 * j + 1]));
            mx1 = fmaxf(mx1, fmaxf(sc[4 * j + 2], sc[4 * j + 3]));
        }
#pragma unroll
        for (int x = 1; x <= 2; x *= 2) {
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, x));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, x));
        }
        // every tile holds at least one key < N, so mx is finite; exp(-inf - mx) = 0 on the first tile
        const float a0 = expf(m0 - mx0), a1 = expf(m1 - mx1);
        m0 = mx0;
        m1 = mx1;
        uint32_t ph[32], pl[32];
        float ls0 = 0.f, ls1 = 0.f;
#pragma unroll
        for (int k = 0; k < 32; ++k) {
            const float p = expf(sc[k] - ((k & 2) ? m1 : m0));
            if (k & 2) ls1 += p; else ls0 += p;
            split_tf32(p, ph[k], pl[k]);
        }
        l0 = fmaf(l0, a0, ls0);
        l1 = fmaf(l1, a1, ls1);
        // this tile's P V in a fresh accumulator (small terms first, as above), merged into O in fp32
        fence();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            // A fragment of key chunk j in slot order (t, t + 4) = (key 8j + 2t, key 8j + 2t + 1)
            const uint32_t ah[4] = {ph[4 * j], ph[4 * j + 2], ph[4 * j + 1], ph[4 * j + 3]};
            const uint32_t al[4] = {pl[4 * j], pl[4 * j + 2], pl[4 * j + 1], pl[4 * j + 3]};
            mma_tf32_n64(ot, al, smem_desc(base + 2 * ATT_PART * 4 + j * 2048, ATT_D * 16, 128), j > 0);
            mma_tf32_n64(ot, ah, smem_desc(base + 4 * ATT_PART * 4 + j * 2048, ATT_D * 16, 128), true);
            mma_tf32_n64(ot, ah, smem_desc(base + 3 * ATT_PART * 4 + j * 2048, ATT_D * 16, 128), true);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t ah[4] = {ph[4 * j], ph[4 * j + 2], ph[4 * j + 1], ph[4 * j + 3]};
            mma_tf32_n64(ot, ah, smem_desc(base + 2 * ATT_PART * 4 + j * 2048, ATT_D * 16, 128), true);
        }
        commit_group();
        wait_all();
        fence_regs(ot);
        keep_regs(ph);
        keep_regs(pl);
#pragma unroll
        for (int k = 0; k < 32; ++k) o[k] = fmaf(o[k], (k & 2) ? a1 : a0, ot[k]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);        // this warp is done reading stage s
    }

#pragma unroll
    for (int x = 1; x <= 2; x *= 2) {
        l0 += __shfl_xor_sync(0xffffffffu, l0, x);
        l1 += __shfl_xor_sync(0xffffffffu, l1, x);
    }
    // a timed-out barrier wait leaves NaN rows rather than a silently wrong result
    const float nan = __int_as_float(0x7fc00000);
    float* ob = out + (size_t)b * N * H * ATT_D + (size_t)h * ATT_D;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = row0 + 8 * r;
        if (row >= N) continue;
        const float l = r ? l1 : l0;
        float* orow = ob + (size_t)row * H * ATT_D;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float2 v = ok ? make_float2(o[4 * j + 2 * r] / l, o[4 * j + 2 * r + 1] / l) : make_float2(nan, nan);
            *reinterpret_cast<float2*>(orow + 8 * j + 2 * t) = v;
        }
    }
}

int attention_check(int B, int N, int H) {
    if (B <= 0 || N <= 0 || H <= 0) { set_error("bad sizes B=%d N=%d H=%d", B, N, H); return GSR_E_INVALID; }
    if (B > 65535 || H > 65535) { set_error("batch or head count too large (B=%d H=%d)", B, H); return GSR_E_INVALID; }
    // qkv holds B * N * 3 * H * 64 floats; every index is 64-bit, and the byte count must fit in one
    if ((uint64_t)B * (uint64_t)N > (1ull << 62) / ((uint64_t)H * 3 * ATT_D * sizeof(float))) {
        set_error("B * N * H too large (B=%d N=%d H=%d)", B, N, H);
        return GSR_E_INVALID;
    }
    return 0;
}

size_t attention_tiles(int N) { return ((size_t)N + ATT_BN - 1) / ATT_BN; }

}  // namespace
}  // namespace gsr

extern "C" size_t gsr_attention_scratch_bytes(int B, int N, int H) {
    using namespace gsr;
    if (attention_check(B, N, H)) return 0;
    return (size_t)B * H * attention_tiles(N) * ATT_TILE_BYTES;
}

extern "C" int gsr_attention_forward(int B, int N, int H, const float* qkv, float* out, void* scratch, void* stream) {
    using namespace gsr;
    if (int rc = attention_check(B, N, H)) return rc;
    if (!qkv || !out || !scratch) { set_error("qkv, out or scratch is NULL"); return GSR_E_INVALID; }
    const cudaStream_t st = (cudaStream_t)stream;
    const int T = (int)attention_tiles(N);
    attention_split_kernel<<<dim3(T, H, B), SPLIT_THREADS, 0, st>>>(N, H, T, qkv, (float*)scratch);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    GSR_CUDA(cudaFuncSetAttribute(attention_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ATT_SMEM));
    attention_fwd_kernel<<<dim3((N + ATT_BM - 1) / ATT_BM, H, B), ATT_THREADS, ATT_SMEM, st>>>(N, H, T, qkv,
                                                                                                (const float*)scratch, out);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}
