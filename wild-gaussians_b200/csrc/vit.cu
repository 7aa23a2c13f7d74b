// vit.cu -- the token-wise layers of the DINOv2 backbone, forward only, for wild-gaussians' uncertainty model.
//
// What it replaces (wildgaussians/dinov2.py): `prepare_tokens_with_masks` (:704-723, the 14x14 stride-14 patch
// convolution, the class token, the position embedding and the register tokens), the token-wise statements of
// `Block.forward` (:328-353: norm1, qkv, proj, ls1, the residual adds, norm2, fc1, GELU, fc2, ls2) and the final
// `norm` of `get_intermediate_layers` (:789-813).  The attention core between `qkv` and `proj` is attention.cu's.
//
// One GEMM kernel, Y[M][N] = epilogue(prologue(X)[M][K] W[N][K]^T), with the operand loader and the epilogue chosen
// by template:
//   A_ROWS   X is [M][K] fp32 rows;
//   A_LN     X is [M][K], LayerNorm-ed on the fly: the CTA first computes its 64 rows' mean and variance in double
//            (one pass over the row), then normalises each element as it stages it;
//   A_PATCH  X is the image [B][3][H][W]: row m = (b, patch), column k = (channel, ky, kx) gathered on the fly
//            (im2col), K = 3 p^2, zero past K;
//   E_BIAS   out = acc + b                                      (qkv)
//   E_GELU   out = gelu_erf(acc + b)                            (fc1)
//   E_RESID  out = resid + (acc + b) * gamma (gamma NULL: + 1)  (proj with ls1, fc2 with ls2; out may be resid)
//   E_TOKENS out = acc + b + pos[1 + p] at token 1 + R + p; CTAs of the first row tile also write the class token
//            (cls + pos[0]) and the R register tokens (no position embedding) of every image: token assembly in one launch.
// A CTA is one warpgroup and owns a 64 x 64 output tile.  Per 32-wide K chunk it stages both operands, split into
// tf32 hi + lo, in the K-major rows16 layout of wgmma.cuh, double-buffered: while the tensor cores run chunk i from
// one buffer, the threads split chunk i + 1 (loaded into registers one chunk earlier) into the other and load chunk
// i + 2.  The weights are split as they are staged, so there is no pre-split weight image to keep in step with the
// module's parameters.
//
// Numerics: 3xTF32, hi*hi + hi*lo + lo*hi.  Hopper's tensor cores add each k-step's products to the accumulator with
// truncation at the accumulator's precision (attention.cu).  So each chunk's hi*hi products (4 k-steps) and its two
// correction terms (8 k-steps) go into two fresh accumulators, which are added to the running fp32 sum in registers
// with round-to-nearest: the truncation never sees more than one chunk.  No atomics, no split-K: every output is one
// thread's fixed-order sum, bitwise reproducible.
//
// vit_output_kernel: the final LayerNorm (or a copy with norm=False) of one taken block's tokens, statistics in
// double, writing the patch tokens as [B][P][C] or, for reshape=True, as [B][C][P] (= [B][C][h][w]) through a shared
// memory transpose, and the class token as [B][C] when asked.
#include "common.cuh"
#include "wgmma.cuh"

namespace gsr {
namespace {

constexpr int VB = 64;                        // rows and output features per CTA
constexpr int VK = 32;                        // contraction per stage
constexpr int V_THREADS = 128;                // one warpgroup
constexpr int V_PART = VB * VK;               // floats of one operand image (8 KB)
constexpr int V_STAGE = 4 * V_PART;           // A hi, A lo, B hi, B lo
constexpr int V_UNITS = V_PART / 4 / V_THREADS;   // 16-byte units of one operand per thread and chunk (4)
constexpr size_t V_SMEM = (size_t)2 * V_STAGE * 4 + 2 * VB * sizeof(float);   // two stages + row statistics
constexpr int MAX_C = 1024;                   // widest embedding (ViT-L)

enum { A_ROWS = 0, A_LN = 1, A_PATCH = 2 };
enum { E_BIAS = 0, E_GELU = 1, E_RESID = 2, E_TOKENS = 3 };

struct Gemm {
    int M, K, N;                      // rows, contraction, output features
    const float* a;                   // [M][K] (A_ROWS, A_LN) or the image [B][3][H][W] (A_PATCH)
    const float* ln_w;                // [K] LayerNorm weight and bias (A_LN)
    const float* ln_b;
    float eps;
    const float* w;                   // [N][K]
    const float* bias;                // [N]
    const float* gamma;               // [N] or NULL (E_RESID)
    const float* resid;               // [M][N] (E_RESID; may equal out)
    float* out;                       // [M][N], or the tokens [B][T][N] (E_TOKENS)
    int H, W, p, gw, P, R, T;         // A_PATCH / E_TOKENS: image size, patch edge, grid width, patches, registers, tokens
    const float* cls;                 // [N]
    const float* reg;                 // [R][N]
    const float* pos;                 // [1 + P][N]
};

// unit u of a 64 x 32 operand chunk: row (u % 8) + 8 (u / 64), columns 4 ((u / 8) % 8) .. + 3.  Eight consecutive lanes
// take eight rows of one column group, which are eight consecutive 16-byte units of the rows16 image: the stores are
// free of bank conflicts, and each row's 128 bytes are read by four whole sectors per warp.
__device__ __forceinline__ int unit_row(int u) { return (u & 7) + 8 * (u >> 6); }
__device__ __forceinline__ int unit_cg(int u) { return (u >> 3) & 7; }

template <int AM>
__device__ __forceinline__ void load_a(const Gemm& g, int m0, int k0, float4 (&r)[V_UNITS]) {
#pragma unroll
    for (int j = 0; j < V_UNITS; ++j) {
        const int u = threadIdx.x + V_THREADS * j;
        const int m = m0 + unit_row(u), k = k0 + 4 * unit_cg(u);
        if (AM != A_PATCH) {
            r[j] = (m < g.M && k < g.K) ? __ldg(reinterpret_cast<const float4*>(g.a + (size_t)m * g.K + k)) : make_float4(0, 0, 0, 0);
        } else {
            float e[4];
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                const int kk = k + s;
                e[s] = 0.f;
                if (m < g.M && kk < g.K) {
                    const int b = m / g.P, pi = m - b * g.P, py = pi / g.gw, px = pi - py * g.gw;
                    const int c = kk / (g.p * g.p), rem = kk - c * g.p * g.p, ky = rem / g.p, kx = rem - ky * g.p;
                    e[s] = __ldg(g.a + (((size_t)b * 3 + c) * g.H + (size_t)py * g.p + ky) * g.W + (size_t)px * g.p + kx);
                }
            }
            r[j] = make_float4(e[0], e[1], e[2], e[3]);
        }
    }
}

__device__ __forceinline__ void load_w(const Gemm& g, int n0, int k0, float4 (&r)[V_UNITS]) {
#pragma unroll
    for (int j = 0; j < V_UNITS; ++j) {
        const int u = threadIdx.x + V_THREADS * j;
        const int n = n0 + unit_row(u), k = k0 + 4 * unit_cg(u);
        r[j] = k < g.K ? __ldg(reinterpret_cast<const float4*>(g.w + (size_t)n * g.K + k)) : make_float4(0, 0, 0, 0);
    }
}

__device__ __forceinline__ void store_split(float* img, int u, float4 v) {
    float4 lo;
    const float4 hi = wg::split_tf32x4(v, lo);
    const int off = (unit_cg(u) * VB + unit_row(u)) * 4;
    *reinterpret_cast<float4*>(img + off) = hi;
    *reinterpret_cast<float4*>(img + V_PART + off) = lo;
}

template <int AM>
__device__ __forceinline__ void stage(const Gemm& g, float* st, int k0, const float4 (&ra)[V_UNITS],
                                      const float4 (&rw)[V_UNITS], const float* mean, const float* rstd) {
#pragma unroll
    for (int j = 0; j < V_UNITS; ++j) {
        const int u = threadIdx.x + V_THREADS * j;
        float4 v = ra[j];
        if (AM == A_LN) {
            const int k = k0 + 4 * unit_cg(u), row = unit_row(u);
            if (k < g.K) {
                const float mu = mean[row], rs = rstd[row];
                const float4 w = __ldg(reinterpret_cast<const float4*>(g.ln_w + k));
                const float4 b = __ldg(reinterpret_cast<const float4*>(g.ln_b + k));
                v = make_float4((v.x - mu) * rs * w.x + b.x, (v.y - mu) * rs * w.y + b.y, (v.z - mu) * rs * w.z + b.z,
                                (v.w - mu) * rs * w.w + b.w);
            }
        }
        store_split(st, u, v);
        store_split(st + 2 * V_PART, u, rw[j]);
    }
}

// grid (ceil(M / 64), N / 64)
template <int AM, int EP>
__global__ void __launch_bounds__(V_THREADS) vit_gemm_kernel(const Gemm g) {
    using namespace wg;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* stages = reinterpret_cast<float*>(smem_raw);
    float* mean = stages + 2 * V_STAGE;
    float* rstd = mean + VB;
    const int m0 = blockIdx.x * VB, n0 = blockIdx.y * VB;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;

    if (AM == A_LN) {
        // row statistics in double, one pass: warp w takes rows 16 w .. 16 w + 15, eight lanes per row
        const int sub = lane / 8, l8 = lane % 8;
#pragma unroll 1
        for (int i = 0; i < 4; ++i) {
            const int row = 16 * warp + 4 * i + sub, m = m0 + row;
            double s = 0.0, q = 0.0;
            if (m < g.M) {
                const float* xr = g.a + (size_t)m * g.K;
#pragma unroll 4
                for (int k = 4 * l8; k < g.K; k += 32) {
                    const float4 v = __ldg(reinterpret_cast<const float4*>(xr + k));
                    s += (double)v.x + (double)v.y + (double)v.z + (double)v.w;
                    q += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
                }
            }
#pragma unroll
            for (int x = 1; x < 8; x *= 2) {
                s += __shfl_xor_sync(0xffffffffu, s, x);
                q += __shfl_xor_sync(0xffffffffu, q, x);
            }
            if (l8 == 0) {
                const double mu = s / g.K, var = fmax(q / g.K - mu * mu, 0.0);
                mean[row] = (float)mu;
                rstd[row] = (float)(1.0 / sqrt(var + (double)g.eps));
            }
        }
        __syncthreads();
    }

    float4 ra[V_UNITS], rw[V_UNITS];
    const int chunks = (g.K + VK - 1) / VK;
    load_a<AM>(g, m0, 0, ra);
    load_w(g, n0, 0, rw);
    stage<AM>(g, stages, 0, ra, rw, mean, rstd);
    if (chunks > 1) {
        load_a<AM>(g, m0, VK, ra);
        load_w(g, n0, VK, rw);
    }
    fence_async_smem();
    __syncthreads();

    float acc[32], hh[32], corr[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = hh[i] = corr[i] = 0.f;
    for (int i = 0; i < chunks; ++i) {
        float* st = stages + (i & 1) * V_STAGE;
        const uint32_t abase = smem_u32(st), bbase = smem_u32(st + 2 * V_PART);
        fence();
#pragma unroll
        for (int c = 0; c < VK / 8; ++c) {
            const uint32_t off = c * 2 * VB * 16;
            mma_tf32_n64(corr, smem_desc(abase + V_PART * 4 + off, VB * 16, 128), smem_desc(bbase + off, VB * 16, 128), c > 0);
            mma_tf32_n64(corr, smem_desc(abase + off, VB * 16, 128), smem_desc(bbase + V_PART * 4 + off, VB * 16, 128), true);
        }
#pragma unroll
        for (int c = 0; c < VK / 8; ++c) {
            const uint32_t off = c * 2 * VB * 16;
            mma_tf32_n64(hh, smem_desc(abase + off, VB * 16, 128), smem_desc(bbase + off, VB * 16, 128), c > 0);
        }
        commit_group();
        if (i + 1 < chunks) stage<AM>(g, stages + ((i + 1) & 1) * V_STAGE, (i + 1) * VK, ra, rw, mean, rstd);
        if (i + 2 < chunks) {
            load_a<AM>(g, m0, (i + 2) * VK, ra);
            load_w(g, n0, (i + 2) * VK, rw);
        }
        wait_all();
        fence_regs(hh);
        fence_regs(corr);
#pragma unroll
        for (int k = 0; k < 32; ++k) acc[k] += hh[k] + corr[k];
        fence_async_smem();
        __syncthreads();
    }

    // accumulator fragment: rows 16 warp + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) + {0, 1}
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int m = m0 + 16 * warp + lane / 4 + 8 * r;
        if (m >= g.M) continue;
        size_t orow = (size_t)m * g.N;
        const float* prow = nullptr;
        if (EP == E_TOKENS) {
            const int b = m / g.P, pi = m - b * g.P;
            orow = ((size_t)b * g.T + 1 + g.R + pi) * g.N;
            prow = g.pos + (size_t)(1 + pi) * g.N;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = n0 + 8 * j + 2 * (lane % 4);
            const float2 bb = *reinterpret_cast<const float2*>(g.bias + n);
            float v0 = acc[4 * j + 2 * r] + bb.x, v1 = acc[4 * j + 2 * r + 1] + bb.y;
            if (EP == E_GELU) {
                v0 = 0.5f * v0 * (1.f + erff(v0 * (float)M_SQRT1_2));
                v1 = 0.5f * v1 * (1.f + erff(v1 * (float)M_SQRT1_2));
            } else if (EP == E_RESID) {
                const float2 x = *reinterpret_cast<const float2*>(g.resid + orow + n);
                if (g.gamma) {
                    const float2 ga = *reinterpret_cast<const float2*>(g.gamma + n);
                    v0 *= ga.x;
                    v1 *= ga.y;
                }
                v0 = x.x + v0;
                v1 = x.y + v1;
            } else if (EP == E_TOKENS) {
                const float2 pe = *reinterpret_cast<const float2*>(prow + n);
                v0 += pe.x;
                v1 += pe.y;
            }
            *reinterpret_cast<float2*>(g.out + orow + n) = make_float2(v0, v1);
        }
    }
    if (EP == E_TOKENS && blockIdx.x == 0) {
        const int B = g.M / g.P;
        for (int i = threadIdx.x; i < B * (1 + g.R) * VB; i += V_THREADS) {
            const int n = n0 + i % VB, t = (i / VB) % (1 + g.R), b = i / (VB * (1 + g.R));
            g.out[((size_t)b * g.T + t) * g.N + n] = t == 0 ? g.cls[n] + g.pos[n] : g.reg[(size_t)(t - 1) * g.N + n];
        }
    }
}

constexpr int O_ROWS = 32;                    // patch tokens per CTA
constexpr int O_THREADS = 256;                // 8 warps, 4 tokens each

// grid (ceil(P / 32), B).  Tokens [B][T][C]; patch tokens are 1 + R .. T - 1; w == NULL: no norm (a copy).
__global__ void __launch_bounds__(O_THREADS) vit_output_kernel(int T, int C, int R, int layout, const float* __restrict__ x,
                                                               const float* __restrict__ w, const float* __restrict__ bn,
                                                               float eps, float* __restrict__ patches, float* __restrict__ cls) {
    __shared__ float tile[32][33];
    __shared__ float s_mean[O_ROWS + 1], s_rstd[O_ROWS + 1];
    const int P = T - 1 - R, p0 = blockIdx.x * O_ROWS, b = blockIdx.y;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const float* xb = x + (size_t)b * T * C;
    // statistics of this CTA's patch tokens (slots 0..31) and, in the first CTA with cls wanted, of the class token (slot 32)
    const int nslots = (blockIdx.x == 0 && cls) ? O_ROWS + 1 : O_ROWS;
    for (int slot = warp; slot < nslots; slot += O_THREADS / 32) {
        const int tok = slot == O_ROWS ? 0 : 1 + R + p0 + slot;
        double s = 0.0, q = 0.0;
        if (w && (slot == O_ROWS || p0 + slot < P)) {
            for (int c = lane; c < C; c += 32) {
                const double v = xb[(size_t)tok * C + c];
                s += v;
                q += v * v;
            }
#pragma unroll
            for (int k = 16; k >= 1; k /= 2) {
                s += __shfl_xor_sync(0xffffffffu, s, k);
                q += __shfl_xor_sync(0xffffffffu, q, k);
            }
        }
        if (lane == 0) {
            const double mu = s / C, var = fmax(q / C - mu * mu, 0.0);
            s_mean[slot] = (float)mu;
            s_rstd[slot] = (float)(1.0 / sqrt(var + (double)eps));
        }
    }
    __syncthreads();
    auto value = [&](int slot, int c) {
        const int tok = slot == O_ROWS ? 0 : 1 + R + p0 + slot;
        const float v = xb[(size_t)tok * C + c];
        return w ? (v - s_mean[slot]) * s_rstd[slot] * w[c] + bn[c] : v;
    };
    if (nslots > O_ROWS)
        for (int c = threadIdx.x; c < C; c += O_THREADS) cls[(size_t)b * C + c] = value(O_ROWS, c);
    if (layout == GSR_VIT_LAYOUT_TOKENS) {
        for (int slot = warp; slot < O_ROWS; slot += O_THREADS / 32) {
            if (p0 + slot >= P) break;
            for (int c = lane; c < C; c += 32) patches[((size_t)b * P + p0 + slot) * C + c] = value(slot, c);
        }
        return;
    }
    // [B][C][P]: 32 tokens x 32 channels per step through shared memory, both global sides coalesced
    for (int c0 = 0; c0 < C; c0 += 32) {
        for (int slot = warp; slot < O_ROWS; slot += O_THREADS / 32)
            if (p0 + slot < P) tile[lane][slot] = value(slot, c0 + lane);
        __syncthreads();
        for (int ch = warp; ch < 32; ch += O_THREADS / 32)
            if (p0 + lane < P) patches[((size_t)b * C + c0 + ch) * P + p0 + lane] = tile[ch][lane];
        __syncthreads();
    }
}

bool misaligned(const void* p) { return ((uintptr_t)p & 15) != 0; }

int launch_gemm(int am, int ep, const Gemm& g, cudaStream_t st) {
    const dim3 grid((unsigned)((g.M + VB - 1) / VB), (unsigned)(g.N / VB));
    auto go = [&](auto kernel) -> int {
        GSR_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)V_SMEM));
        kernel<<<grid, V_THREADS, V_SMEM, st>>>(g);
        count_launches(1);
        GSR_CUDA(cudaGetLastError());
        return 0;
    };
    if (am == A_LN && ep == E_BIAS) return go(vit_gemm_kernel<A_LN, E_BIAS>);
    if (am == A_LN && ep == E_GELU) return go(vit_gemm_kernel<A_LN, E_GELU>);
    if (am == A_ROWS && ep == E_RESID) return go(vit_gemm_kernel<A_ROWS, E_RESID>);
    return go(vit_gemm_kernel<A_PATCH, E_TOKENS>);
}

}  // namespace
}  // namespace gsr

extern "C" int gsr_vit_tokens(int B, int H, int W, int C, int patch, int R, const float* x, const float* weight,
                              const float* bias, const float* cls, const float* reg, const float* pos, float* tokens,
                              void* stream) {
    using namespace gsr;
    if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || patch <= 0 || R < 0) {
        set_error("bad sizes B=%d H=%d W=%d C=%d patch=%d R=%d", B, H, W, C, patch, R);
        return GSR_E_INVALID;
    }
    if (H % patch || W % patch || patch % 2 || C % VB || C > MAX_C) {
        set_error("bad sizes: H=%d and W=%d must be multiples of the patch size %d, which must be even; C=%d a multiple of "
                  "64 up to 1024", H, W, patch, C);
        return GSR_E_INVALID;
    }
    const uint64_t P = (uint64_t)(H / patch) * (uint64_t)(W / patch), T = 1 + (uint64_t)R + P;
    if (B > 65535 || (uint64_t)B * T > (uint64_t)INT32_MAX || (uint64_t)B * 3 * H > (uint64_t)INT32_MAX / (uint64_t)W) {
        set_error("B, image or token count too large (B=%d H=%d W=%d R=%d)", B, H, W, R);
        return GSR_E_INVALID;
    }
    if (!x || !weight || !bias || !cls || !pos || !tokens || (R > 0 && !reg)) {
        set_error("x, weight, bias, cls, reg, pos or tokens is NULL");
        return GSR_E_INVALID;
    }
    if (misaligned(weight) || misaligned(bias) || misaligned(pos) || misaligned(tokens)) {
        set_error("weight, bias, pos and tokens must be 16-byte aligned");
        return GSR_E_INVALID;
    }
    Gemm g{};
    g.M = (int)((uint64_t)B * P);
    g.K = 3 * patch * patch;
    g.N = C;
    g.a = x;
    g.w = weight;
    g.bias = bias;
    g.out = tokens;
    g.H = H;
    g.W = W;
    g.p = patch;
    g.gw = W / patch;
    g.P = (int)P;
    g.R = R;
    g.T = (int)T;
    g.cls = cls;
    g.reg = reg;
    g.pos = pos;
    return launch_gemm(A_PATCH, E_TOKENS, g, (cudaStream_t)stream);
}

extern "C" int gsr_vit_linear(int op, int M, int K, int N, const float* x, const float* ln_w, const float* ln_b, float eps,
                              const float* weight, const float* bias, const float* gamma, const float* resid, float* out,
                              void* stream) {
    using namespace gsr;
    if (op != GSR_VIT_LN_BIAS && op != GSR_VIT_LN_GELU && op != GSR_VIT_RESIDUAL) {
        set_error("unknown op %d", op);
        return GSR_E_INVALID;
    }
    if (M <= 0 || K <= 0 || N <= 0 || K % 4 || N % VB) {
        set_error("bad sizes M=%d K=%d N=%d (K a multiple of 4, N of 64)", M, K, N);
        return GSR_E_INVALID;
    }
    if (K > 4 * MAX_C || N > 4 * MAX_C) {
        set_error("K or N too large (K=%d N=%d, at most %d)", K, N, 4 * MAX_C);
        return GSR_E_INVALID;
    }
    const bool ln = op != GSR_VIT_RESIDUAL;
    if (!x || !weight || !bias || !out || (ln && (!ln_w || !ln_b)) || (!ln && !resid)) {
        set_error("x, ln_w, ln_b, weight, bias, resid or out is NULL");
        return GSR_E_INVALID;
    }
    if (misaligned(x) || misaligned(weight) || misaligned(bias) || misaligned(out) || (ln && (misaligned(ln_w) || misaligned(ln_b))) ||
        (!ln && (misaligned(resid) || misaligned(gamma)))) {
        set_error("every array must be 16-byte aligned");
        return GSR_E_INVALID;
    }
    if (ln && !(eps > 0.f)) {
        set_error("eps must be positive (eps=%g)", (double)eps);
        return GSR_E_INVALID;
    }
    Gemm g{};
    g.M = M;
    g.K = K;
    g.N = N;
    g.a = x;
    g.ln_w = ln_w;
    g.ln_b = ln_b;
    g.eps = eps;
    g.w = weight;
    g.bias = bias;
    g.gamma = gamma;
    g.resid = resid;
    g.out = out;
    return launch_gemm(ln ? A_LN : A_ROWS, op == GSR_VIT_LN_BIAS ? E_BIAS : op == GSR_VIT_LN_GELU ? E_GELU : E_RESID, g,
                       (cudaStream_t)stream);
}

extern "C" int gsr_vit_output(int B, int T, int C, int R, int layout, const float* tokens, const float* norm_w,
                              const float* norm_b, float eps, float* patches, float* cls, void* stream) {
    using namespace gsr;
    if (B <= 0 || C <= 0 || R < 0 || T < R + 2 || C % 32 || C > MAX_C) {
        set_error("bad sizes B=%d T=%d C=%d R=%d (T >= R + 2, C a multiple of 32 up to 1024)", B, T, C, R);
        return GSR_E_INVALID;
    }
    if (layout != GSR_VIT_LAYOUT_TOKENS && layout != GSR_VIT_LAYOUT_CHANNELS) {
        set_error("unknown layout %d", layout);
        return GSR_E_INVALID;
    }
    if (B > 65535 || (uint64_t)B * (uint64_t)T > (uint64_t)INT32_MAX) {
        set_error("batch or token count too large (B=%d T=%d)", B, T);
        return GSR_E_INVALID;
    }
    if (!tokens || !patches || (!norm_w) != (!norm_b)) {
        set_error("tokens or patches is NULL, or only one of norm_w and norm_b is");
        return GSR_E_INVALID;
    }
    if (norm_w && !(eps > 0.f)) {
        set_error("eps must be positive (eps=%g)", (double)eps);
        return GSR_E_INVALID;
    }
    const int P = T - 1 - R;
    vit_output_kernel<<<dim3((unsigned)((P + O_ROWS - 1) / O_ROWS), (unsigned)B), O_THREADS, 0, (cudaStream_t)stream>>>(
        T, C, R, layout, tokens, norm_w, norm_b, eps, patches, cls);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}
