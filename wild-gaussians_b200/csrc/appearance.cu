// appearance.cu -- fused per-Gaussian colour op of wild-gaussians on Hopper tensor cores (SURVEY.md 8f-2).
//
// What it replaces (PyTorch, wildgaussians/method.py): per Gaussian and per step
//   features = cat(features_dc, features_rest).clamp_max(1)                          method.py:1063-1066,1570
//   raw      = clamp_min(eval_sh(deg, features, dir) + 0.5, 0)                       method.py:1571-1579, eval_sh :493-548
//   x        = cat(features[:, :3], embeddings, appearance_embedding)     (59)       EmbeddingModel.forward :889-895
//   o        = 0.01 * MLP(x)   (59 -> 128 -> ReLU -> 128 -> ReLU -> 6)               method.py:882-888,896
//   t        = clamp_max(features * repeat(o[3:6]) + pad(o[0:3] / C0), 1)            method.py:897-900,1589-1593
//   toned    = clamp_min(eval_sh(deg, t, dir) + 0.5, 0)                              method.py:1594-1595
// with dir = normalize(means3D - campos) (:1572): about 60 elementwise / GEMM launches and several P x 128 and
// P x 48 fp32 intermediates per direction (measured: ~55 ms of a 61 ms train step at P = 3 M).
//
// Design: ONE kernel per direction.  A CTA owns tiles of 128 Gaussians and runs as two warpgroups, each issuing the
// warpgroup MMAs (wgmma, bf16 operands from shared memory, fp32 accumulation in registers, M = 64) for its 64 rows.  The
// activations never leave the SM: an epilogue takes the accumulator fragment, applies ReLU, converts to bf16 and writes
// the next layer's A operand straight into shared memory ("rows16" storage, wgmma.cuh).  The packed
// weights (49 KB) are fetched once per CTA by one bulk asynchronous copy (TMA engine) and stay resident; each
// tile's 23 KB of SH coefficients arrive by a bulk copy issued at the start of the tile and consumed in its last
// epilogue.  Biases ride inside the GEMMs: every A operand carries two constant-one columns and the weight images
// carry bias_hi / bias_lo (a bf16 pair, error 2^-17) in the matching rows; the image-wide appearance embedding is the
// same for every Gaussian, so W1[:, 27:59] . embedding is folded into the layer-1 bias (K shrinks from 59 to 32).
// The last epilogue evaluates the affine tone map, both SH colour sums (shared basis) and the clamps.
//
// Backward: recomputes the three layers per tile (cheaper than storing 2 x 128 activations per Gaussian), then runs
// the data-gradient chain dO -> dZ2 -> dZ1 -> dX and the three weight-gradient GEMMs on the same shared-memory
// tiles: an activation tile stored once serves as K-major operand (forward, dgrad) and as MN-major operand (wgrad)
// without a transposed copy.  Weight gradients accumulate in registers across all tiles of the CTA and are reduced to
// HBM once per CTA with vector reductions.
//
// Numerics: MLP operands are bf16 (fp32 accumulate); everything else fp32.  Colours agree with the fp32 PyTorch
// path to ~2e-3 absolute (bf16 rounding of a 128-term dot product scaled by 0.01), gradients to ~1e-2 of their
// largest magnitude; tests/test_appearance.py states the bars.
#include "common.cuh"
#include "wgmma.cuh"
#include "sh_math.cuh"

namespace gsr {

using namespace wg;

constexpr int AP_TILE = 128;
constexpr int AP_NDC = 3, AP_NREST = 45, AP_NGEMB = 24, AP_NAEMB = 32, AP_H = 128, AP_NOUT = 6;
constexpr int AP_K1 = 32;                 // layer-1 contraction: dc 3 + gemb 24 + {1, 1} + 3 pad
constexpr int AP_K2 = 144;                // hidden 128 + {1, 1} + 14 pad
constexpr int AP_N3 = 16;                 // layer-3 outputs padded to the smallest MMA N
constexpr int AP_ONE1 = 27;               // column of the first constant one in X
constexpr int AP_ONE2 = 128;              // column of the first constant one in H1 / H2
constexpr uint32_t CHUNK = AP_TILE * 16;  // bytes of one 8-column chunk of a 128-row rows16 matrix
// packed weight blob (bf16 rows16 images): W1p [128][32], W2p [128][144], W3p [16][144]
constexpr uint32_t W1P_BYTES = AP_H * AP_K1 * 2, W2P_BYTES = AP_H * AP_K2 * 2, W3P_BYTES = AP_N3 * AP_K2 * 2;
constexpr uint32_t BLOB_BYTES = W1P_BYTES + W2P_BYTES + W3P_BYTES;      // 49664
constexpr uint32_t ACT_BYTES = (AP_K2 / 8) * CHUNK;                      // 36864: 18 chunks incl. the constant ones
constexpr uint32_t REST_BYTES = AP_TILE * AP_NREST * 4;                  // 23040
// packed gradient image (fp32): gW1p [128][32], gW2p [128][144], gW3pT [128][16], gb3 [16]
constexpr size_t GW1P = 0, GW2P = GW1P + AP_H * AP_K1, GW3P = GW2P + AP_H * AP_K2, GB3 = GW3P + AP_H * AP_N3,
                 GPACK_FLOATS = GB3 + 16;

constexpr float SH_C0 = SHK0;

struct ApParams {
    int P, deg, num_tiles;
    const float* dc;        // [P,3]
    const float* rest;      // [P,45]
    const float* gemb;      // [P,24]
    const float* means;     // [P,3]
    const float* campos;    // [3]
    const uint8_t* blob;    // packed weights
    float* raw;             // [P,3] or NULL
    float* toned;           // [P,3]
    // backward
    const float* dL_raw;    // [P,3] or NULL
    const float* dL_toned;  // [P,3]
    float* g_dc;            // [P,3]
    float* g_rest;          // [P,45]
    float* g_gemb;          // [P,24]
    float* g_means;         // [P,3]
    float* g_pack;          // [GPACK_FLOATS] zero-initialised
    int* status;            // device flag: != 0 if a barrier wait timed out
};

// ---- rows16 helpers ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_chunk(uint8_t* base, int chunk, int row, uint4 v) {
    *reinterpret_cast<uint4*>(base + (uint32_t)chunk * CHUNK + (uint32_t)row * 16) = v;
}
__device__ __forceinline__ uint4 ld_chunk(const uint8_t* base, int chunk, int row) {
    return *reinterpret_cast<const uint4*>(base + (uint32_t)chunk * CHUNK + (uint32_t)row * 16);
}
// K-major operand of a 128-row activation / weight image: k-th K = 16 step
__device__ __forceinline__ uint64_t desc_k(const uint8_t* base, int kstep, uint32_t rows) {
    return smem_desc(smem_u32(base) + (uint32_t)kstep * 2u * rows * 16u, rows * 16u, 128u);
}
// MN-major operand (contraction over the rows of the image): k-th group of 16 rows
__device__ __forceinline__ uint64_t desc_mn(const uint8_t* base, int kstep, uint32_t rows) {
    return smem_desc(smem_u32(base) + (uint32_t)kstep * 256u, 128u, rows * 16u);
}

// ---- weight packing ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void put_bf16(uint8_t* img, uint32_t rows, int row, int col, float v) {
    *reinterpret_cast<__nv_bfloat16*>(img + (uint32_t)(col / 8) * rows * 16u + (uint32_t)row * 16u + (uint32_t)(col % 8) * 2u) =
        __float2bfloat16(v);
}
__device__ __forceinline__ void put_hi_lo(uint8_t* img, uint32_t rows, int row, int col, float v) {
    const float hi = __bfloat162float(__float2bfloat16(v));
    put_bf16(img, rows, row, col, hi);
    put_bf16(img, rows, row, col + 1, v - hi);
}
// one CTA of 128 threads; thread n = output neuron n
__global__ void __launch_bounds__(128) appearance_pack_kernel(const float* __restrict__ W1, const float* __restrict__ b1,
                                                              const float* __restrict__ W2, const float* __restrict__ b2,
                                                              const float* __restrict__ W3, const float* __restrict__ b3,
                                                              const float* __restrict__ aemb, uint8_t* __restrict__ blob) {
    const int n = threadIdx.x;
    uint8_t* w1p = blob;
    uint8_t* w2p = blob + W1P_BYTES;
    uint8_t* w3p = w2p + W2P_BYTES;
    constexpr int IN1 = AP_NDC + AP_NGEMB + AP_NAEMB;   // 59
    for (int k = 0; k < AP_K1; ++k) put_bf16(w1p, AP_H, n, k, k < AP_NDC + AP_NGEMB ? W1[n * IN1 + k] : 0.f);
    float bias = b1[n];
    for (int j = 0; j < AP_NAEMB; ++j) bias = fmaf(W1[n * IN1 + AP_NDC + AP_NGEMB + j], aemb[j], bias);
    put_hi_lo(w1p, AP_H, n, AP_ONE1, bias);
    for (int k = 0; k < AP_K2; ++k) put_bf16(w2p, AP_H, n, k, k < AP_H ? W2[n * AP_H + k] : 0.f);
    put_hi_lo(w2p, AP_H, n, AP_ONE2, b2[n]);
    if (n < AP_N3) {
        for (int k = 0; k < AP_K2; ++k) put_bf16(w3p, AP_N3, n, k, (n < AP_NOUT && k < AP_H) ? W3[n * AP_H + k] : 0.f);
        if (n < AP_NOUT) put_hi_lo(w3p, AP_N3, n, AP_ONE2, b3[n]);
    }
}

// packed gradient image -> parameter gradients (one CTA of 128 threads, thread n = hidden neuron n)
__global__ void __launch_bounds__(128) appearance_unpack_kernel(const float* __restrict__ g, const float* __restrict__ W1,
                                                                const float* __restrict__ aemb, float* __restrict__ gW1,
                                                                float* __restrict__ gb1, float* __restrict__ gW2,
                                                                float* __restrict__ gb2, float* __restrict__ gW3,
                                                                float* __restrict__ gb3, float* __restrict__ gaemb) {
    __shared__ float s_db1[AP_H];
    const int n = threadIdx.x;
    constexpr int IN1 = AP_NDC + AP_NGEMB + AP_NAEMB;
    const float db1 = g[GW1P + n * AP_K1 + AP_ONE1];
    s_db1[n] = db1;
    gb1[n] = db1;
    for (int k = 0; k < AP_NDC + AP_NGEMB; ++k) gW1[n * IN1 + k] = g[GW1P + n * AP_K1 + k];
    // the appearance embedding entered through the folded bias: dW1[n][27 + j] = db1'[n] * aemb[j]
    for (int j = 0; j < AP_NAEMB; ++j) gW1[n * IN1 + AP_NDC + AP_NGEMB + j] = db1 * aemb[j];
    for (int k = 0; k < AP_H; ++k) gW2[n * AP_H + k] = g[GW2P + n * AP_K2 + k];
    gb2[n] = g[GW2P + n * AP_K2 + AP_ONE2];
    for (int o = 0; o < AP_NOUT; ++o) gW3[o * AP_H + n] = g[GW3P + n * AP_N3 + o];
    if (n < AP_NOUT) gb3[n] = g[GB3 + n];
    __syncthreads();
    if (n < AP_NAEMB) {
        float s = 0.f;
        for (int m = 0; m < AP_H; ++m) s = fmaf(s_db1[m], W1[m * IN1 + AP_NDC + AP_NGEMB + n], s);
        gaemb[n] = s;
    }
}

// ---- shared pieces of the two kernels -----------------------------------------------------------------------------
struct RowIn {
    float dc[3];        // unclamped features_dc
    float3 dir;         // normalised view direction
    float inv_norm;     // 1 / max(|mean - campos|, 1e-12)
};

// thread `t` builds its row of X = [min(dc, 1) (3), gemb (24), 1, 1, 0, 0, 0] as bf16 in `xbuf` (4 chunks)
__device__ __forceinline__ void build_x_row(const ApParams& p, int row, bool valid, int t, uint8_t* xbuf, RowIn& in) {
    float x[AP_K1];
#pragma unroll
    for (int i = 0; i < AP_K1; ++i) x[i] = 0.f;
    in.dc[0] = in.dc[1] = in.dc[2] = 0.f;
    in.dir = {0.f, 0.f, 1.f};
    in.inv_norm = 0.f;
    if (valid) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { in.dc[c] = p.dc[(size_t)row * 3 + c]; x[c] = fminf(in.dc[c], 1.0f); }
        const float4* g4 = reinterpret_cast<const float4*>(p.gemb + (size_t)row * AP_NGEMB);
#pragma unroll
        for (int i = 0; i < AP_NGEMB / 4; ++i) {
            const float4 v = __ldg(g4 + i);
            x[3 + 4 * i + 0] = v.x; x[3 + 4 * i + 1] = v.y; x[3 + 4 * i + 2] = v.z; x[3 + 4 * i + 3] = v.w;
        }
        x[AP_ONE1] = 1.f; x[AP_ONE1 + 1] = 1.f;
        const float vx = p.means[(size_t)row * 3 + 0] - p.campos[0], vy = p.means[(size_t)row * 3 + 1] - p.campos[1],
                    vz = p.means[(size_t)row * 3 + 2] - p.campos[2];
        const float nrm = fmaxf(sqrtf(vx * vx + vy * vy + vz * vz), 1e-12f);      // F.normalize (method.py:1572)
        in.inv_norm = 1.0f / nrm;
        in.dir = {vx * in.inv_norm, vy * in.inv_norm, vz * in.inv_norm};
    }
#pragma unroll
    for (int c = 0; c < AP_K1 / 8; ++c)
        st_chunk(xbuf, c, t, make_uint4(pack_bf16(x[8 * c], x[8 * c + 1]), pack_bf16(x[8 * c + 2], x[8 * c + 3]),
                                        pack_bf16(x[8 * c + 4], x[8 * c + 5]), pack_bf16(x[8 * c + 6], x[8 * c + 7])));
}

// ---- accumulator fragments (wgmma.cuh) ------------------------------------------------------------------------------
// This thread's accumulator rows within the 128-row tile: r0 and r0 + 8 (warpgroup w owns rows 64 w .. 64 w + 63), and
// its column pair 2c of every 8-column group.
struct Frag {
    int r0, c;
};
__device__ __forceinline__ Frag frag_of(int tid) { return {64 * (tid >> 7) + 16 * ((tid >> 5) & 3) + ((tid & 31) >> 2), tid & 3}; }
__device__ __forceinline__ void st_pair(uint8_t* base, int chunk, int row, int c, uint32_t v) {
    *reinterpret_cast<uint32_t*>(base + (uint32_t)chunk * CHUNK + (uint32_t)row * 16 + (uint32_t)c * 4) = v;
}
__device__ __forceinline__ uint32_t ld_pair(const uint8_t* base, int chunk, int row, int c) {
    return *reinterpret_cast<const uint32_t*>(base + (uint32_t)chunk * CHUNK + (uint32_t)row * 16 + (uint32_t)c * 4);
}

// 64 x 128 accumulator -> ReLU -> bf16 -> chunks 0..15 of `hbuf` (this thread's rows only)
__device__ __forceinline__ void relu_epilogue(const float (&d)[64], uint8_t* hbuf, Frag f) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        st_pair(hbuf, j, f.r0, f.c, pack_bf16(fmaxf(d[4 * j], 0.f), fmaxf(d[4 * j + 1], 0.f)));
        st_pair(hbuf, j, f.r0 + 8, f.c, pack_bf16(fmaxf(d[4 * j + 2], 0.f), fmaxf(d[4 * j + 3], 0.f)));
    }
}

// a bf16 activation is positive iff its 15 magnitude bits are non-zero and the sign is clear (ReLU output: never negative)
__device__ __forceinline__ uint32_t relu_mask(uint32_t h, float lo, float hi) {
    return pack_bf16((h & 0x7FFFu) ? lo : 0.f, (h & 0x7FFF0000u) ? hi : 0.f);
}
// 64 x 128 accumulator * (activation > 0) -> bf16 -> chunks 0..15 of `dzbuf` (ReLU backward; `hbuf` holds the activation)
__device__ __forceinline__ void relu_bwd_epilogue(const float (&d)[64], const uint8_t* hbuf, uint8_t* dzbuf, Frag f) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        st_pair(dzbuf, j, f.r0, f.c, relu_mask(ld_pair(hbuf, j, f.r0, f.c), d[4 * j], d[4 * j + 1]));
        st_pair(dzbuf, j, f.r0 + 8, f.c, relu_mask(ld_pair(hbuf, j, f.r0 + 8, f.c), d[4 * j + 2], d[4 * j + 3]));
    }
}

// columns 0..7 of the layer-3 accumulator -> fp32 rows of `out` ([128][8]), read back per row by the colour stage
constexpr uint32_t OUT_BYTES = AP_TILE * 8 * 4;
__device__ __forceinline__ void store_out(const float (&d)[8], float* out, Frag f) {
    *reinterpret_cast<float2*>(out + f.r0 * 8 + 2 * f.c) = make_float2(d[0], d[1]);
    *reinterpret_cast<float2*>(out + (f.r0 + 8) * 8 + 2 * f.c) = make_float2(d[2], d[3]);
}

// the two constant-one columns (+ zero padding) of an H buffer: chunks 16 and 17
__device__ __forceinline__ void write_const_chunks(uint8_t* hbuf, int t) {
    st_chunk(hbuf, 16, t, make_uint4(0x3F803F80u, 0u, 0u, 0u));     // {1.0bf16, 1.0bf16, 0 ...}
    st_chunk(hbuf, 17, t, make_uint4(0u, 0u, 0u, 0u));
}

// forward GEMMs of warpgroup `w` (its 64 rows of the K-major activation image `act`, all of the weight image `wimg`);
// each returns with the accumulator complete
template <int KSTEPS>
__device__ __forceinline__ void gemm_n128(float (&d)[64], const uint8_t* act, const uint8_t* wimg, int w) {
    fence_regs(d);
    fence();
#pragma unroll
    for (int k = 0; k < KSTEPS; ++k) mma_n128<0, 0>(d, desc_k(act + w * 1024, k, AP_TILE), desc_k(wimg, k, AP_H), k > 0);
    commit_group();
    wait_all();
    fence_regs(d);
}
__device__ __forceinline__ void gemm_n16(float (&d)[8], const uint8_t* act, const uint8_t* w3p, int w) {
    fence_regs(d);
    fence();
#pragma unroll
    for (int k = 0; k < AP_K2 / 16; ++k) mma_n16<0, 0>(d, desc_k(act + w * 1024, k, AP_TILE), desc_k(w3p, k, AP_N3), k > 0);
    commit_group();
    wait_all();
    fence_regs(d);
}

#define AP_FAIL()                                  \
    do {                                           \
        if (p.status) atomicExch(p.status, 1);     \
        dead = true;                               \
    } while (0)

// =====================================================================================================================
// forward
// =====================================================================================================================
constexpr uint32_t FWD_SMEM = BLOB_BYTES + ACT_BYTES + REST_BYTES + OUT_BYTES + 64;

// 256 threads = two warpgroups: warpgroup w runs the three GEMMs and their epilogues for rows 64 w .. 64 w + 63 of the tile
// (wgmma M = 64) and only synchronises with itself between layers; the input row and the colour epilogue of row t are done
// by thread t < 128.  Two resident CTAs per SM (111 KB of shared memory each) keep 16 warps per SM.
constexpr int FWD_THREADS = 2 * AP_TILE;
__global__ void __launch_bounds__(FWD_THREADS, 2) appearance_fwd_kernel(const __grid_constant__ ApParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* s_blob = smem;
    uint8_t* s_act = smem + BLOB_BYTES;
    float* s_rest = reinterpret_cast<float*>(smem + BLOB_BYTES + ACT_BYTES);
    float* s_out = reinterpret_cast<float*>(smem + BLOB_BYTES + ACT_BYTES + REST_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + BLOB_BYTES + ACT_BYTES + REST_BYTES + OUT_BYTES);   // 0: loads, 1: weights
    const int tid = threadIdx.x, t = tid & (AP_TILE - 1), w = tid >> 7;
    const bool h0 = w == 0;
    const Frag f = frag_of(tid);

    if (tid == 0) {
        mbar_init(&bars[0], 1); mbar_init(&bars[1], 1);
        mbar_init_fence();
    }
    if (h0) write_const_chunks(s_act, t);
    fence_async_smem();
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(&bars[1], BLOB_BYTES);
        bulk_g2s(s_blob, p.blob, BLOB_BYTES, &bars[1]);
    }
    const uint8_t* w1p = s_blob;
    const uint8_t* w2p = s_blob + W1P_BYTES;
    const uint8_t* w3p = w2p + W2P_BYTES;
    float acc[64], acc3[8];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc3[i] = 0.f;
    uint32_t ph_ld = 0;
    bool dead = false;
    if (!mbar_wait(&bars[1], 0)) AP_FAIL();

    for (int tile = blockIdx.x; tile < p.num_tiles && !dead; tile += gridDim.x) {
        const int row0 = tile * AP_TILE, row = row0 + t;
        const int rows = min(AP_TILE, p.P - row0);
        const bool valid = h0 && t < rows;
        const bool bulk = rows == AP_TILE;           // whole tiles: one 23 KB bulk copy; the ragged last tile: plain loads
        if (bulk) {
            if (tid == 0) {
                mbar_expect_tx(&bars[0], REST_BYTES);
                bulk_g2s(s_rest, p.rest + (size_t)row0 * AP_NREST, REST_BYTES, &bars[0]);
            }
        } else {
            for (int i = tid; i < rows * AP_NREST; i += FWD_THREADS) s_rest[i] = p.rest[(size_t)row0 * AP_NREST + i];
        }
        RowIn in;
        in.dc[0] = in.dc[1] = in.dc[2] = 0.f; in.dir = {0.f, 0.f, 1.f}; in.inv_norm = 0.f;
        if (h0) build_x_row(p, row, valid, t, s_act, in);
        fence_async_smem();
        __syncthreads();
        // a warpgroup's GEMM reads only its own 64 rows of the activation image, which only its own threads overwrite
        gemm_n128<AP_K1 / 16>(acc, s_act, w1p, w);
        relu_epilogue(acc, s_act, f);
        fence_async_smem();
        warpgroup_sync(w);
        gemm_n128<AP_K2 / 16>(acc, s_act, w2p, w);
        relu_epilogue(acc, s_act, f);
        fence_async_smem();
        warpgroup_sync(w);
        gemm_n16(acc3, s_act, w3p, w);
        store_out(acc3, s_out, f);
        __syncthreads();
        if (bulk) {
            if (!mbar_wait(&bars[0], ph_ld)) AP_FAIL();
            ph_ld ^= 1u;
        }
        if (valid) {
            const float* o = s_out + t * 8;
            float b[16];
            sh_basis(p.deg, in.dir.x, in.dir.y, in.dir.z, b);
            const float* fr = s_rest + t * AP_NREST;
            float sr[3], st[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float mul = 0.01f * o[3 + c], off = 0.01f * o[c] / SH_C0;
                const float f0 = fminf(in.dc[c], 1.0f);
                float r = b[0] * f0, s = b[0] * fminf(fmaf(f0, mul, off), 1.0f);
#pragma unroll
                for (int k = 1; k < 16; ++k) {
                    const float fv = fminf(fr[3 * (k - 1) + c], 1.0f);
                    r = fmaf(b[k], fv, r);
                    s = fmaf(b[k], fminf(fv * mul, 1.0f), s);
                }
                sr[c] = fmaxf(r + 0.5f, 0.f);
                st[c] = fmaxf(s + 0.5f, 0.f);
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                if (p.raw) p.raw[(size_t)row * 3 + c] = sr[c];
                p.toned[(size_t)row * 3 + c] = st[c];
            }
        }
        fence_async_smem();       // generic reads of s_rest / s_act are ordered before the next tile's bulk copy into them
        __syncthreads();          // s_rest, s_act and s_out are free for the next tile
    }
}

// =====================================================================================================================
// backward
// =====================================================================================================================
constexpr uint32_t BX_BYTES = (AP_K1 / 8) * CHUNK;        //  8192
constexpr uint32_t BDZ_BYTES = (AP_H / 8) * CHUNK;        // 32768
constexpr uint32_t BDO_BYTES = (AP_N3 / 8) * CHUNK;       //  4096
constexpr int DX_LD = 36;                                 // fp32 row stride of the dX tile: conflict-free pair stores
constexpr uint32_t BDX_BYTES = AP_TILE * DX_LD * 4;       // 18432
constexpr uint32_t BWD_SMEM = BLOB_BYTES + BX_BYTES + 2 * ACT_BYTES + BDZ_BYTES + BDO_BYTES + REST_BYTES + OUT_BYTES + BDX_BYTES + 128;

// red.global.add.v2 of a weight-gradient accumulator fragment into the fp32 image `g` (row stride ld)
template <int R>
__device__ __forceinline__ void flush_frag(const float (&d)[R], float* g, int ld, Frag f) {
#pragma unroll
    for (int j = 0; j < R / 4; ++j) {
        float* a = g + (size_t)f.r0 * ld + 8 * j + 2 * f.c;
        float* b = a + (size_t)8 * ld;
        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(a), "f"(d[4 * j]), "f"(d[4 * j + 1]) : "memory");
        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(b), "f"(d[4 * j + 2]), "f"(d[4 * j + 3]) : "memory");
    }
}

// 256 threads = two warpgroups.  Data-gradient GEMMs (M = Gaussians): warpgroup w takes rows 64 w .. 64 w + 63 of the tile.
// Weight-gradient GEMMs (K = the 128 Gaussians of the tile): warpgroup w takes rows 64 w .. 64 w + 63 of each gradient
// image, whose accumulators stay in registers across all tiles of the CTA (dW2p 72 + dW1p 16 + dW3pT 8 per thread) and
// are reduced to HBM once per CTA.  Per-row work that cannot be split (input row, colour stage, dX) is done by thread
// t < 128.  One CTA per SM (209 KB of shared memory).
constexpr int BWD_THREADS = 2 * AP_TILE;
__global__ void __launch_bounds__(BWD_THREADS, 1) appearance_bwd_kernel(const __grid_constant__ ApParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* s_blob = smem;
    uint8_t* s_x = s_blob + BLOB_BYTES;
    uint8_t* s_h1 = s_x + BX_BYTES;
    uint8_t* s_h2 = s_h1 + ACT_BYTES;
    uint8_t* s_dz = s_h2 + ACT_BYTES;
    uint8_t* s_do = s_dz + BDZ_BYTES;
    float* s_rest = reinterpret_cast<float*>(s_do + BDO_BYTES);
    float* s_out = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(s_rest) + REST_BYTES);
    float* s_dx = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(s_out) + OUT_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(s_dx) + BDX_BYTES);
    float* s_db3 = reinterpret_cast<float*>(bars + 4);       // [8]
    const int tid = threadIdx.x, t = tid & (AP_TILE - 1), w = tid >> 7, lane = tid & 31;
    const bool h0 = w == 0;
    const Frag f = frag_of(tid);
    constexpr uint32_t MN_HALF = 8 * CHUNK;                   // warpgroup w's 64 M rows of an MN-major operand

    if (tid == 0) {
        mbar_init(&bars[0], 1); mbar_init(&bars[1], 1);
        mbar_init_fence();
    }
    if (tid < 8) s_db3[tid] = 0.f;
    if (h0) {
        write_const_chunks(s_h1, t);
        write_const_chunks(s_h2, t);
        st_chunk(s_do, 1, t, make_uint4(0u, 0u, 0u, 0u));
    }
    fence_async_smem();
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(&bars[1], BLOB_BYTES);
        bulk_g2s(s_blob, p.blob, BLOB_BYTES, &bars[1]);
    }
    const uint8_t* w1p = s_blob;
    const uint8_t* w2p = s_blob + W1P_BYTES;
    const uint8_t* w3p = w2p + W2P_BYTES;
    float gw2[72], gw1[16], gw3[8];           // weight-gradient accumulators: start at zero, always accumulate
    float acc[64], acc3[8], accx[16];
#pragma unroll
    for (int i = 0; i < 72; ++i) gw2[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) { gw1[i] = 0.f; accx[i] = 0.f; }
#pragma unroll
    for (int i = 0; i < 8; ++i) { gw3[i] = 0.f; acc3[i] = 0.f; }
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    uint32_t ph_ld = 0;
    bool dead = false;
    if (!mbar_wait(&bars[1], 0)) AP_FAIL();
    int iter = 0;

    for (int tile = blockIdx.x; tile < p.num_tiles && !dead; tile += gridDim.x, ++iter) {
        const int row0 = tile * AP_TILE, row = row0 + t;
        const int rows = min(AP_TILE, p.P - row0);
        const bool valid = h0 && t < rows;
        const bool bulk = rows == AP_TILE;
        if (bulk) {
            if (tid == 0) {
                mbar_expect_tx(&bars[0], REST_BYTES);
                bulk_g2s(s_rest, p.rest + (size_t)row0 * AP_NREST, REST_BYTES, &bars[0]);
            }
        } else {
            for (int i = tid; i < rows * AP_NREST; i += BWD_THREADS) s_rest[i] = p.rest[(size_t)row0 * AP_NREST + i];
        }
        RowIn in;
        in.dc[0] = in.dc[1] = in.dc[2] = 0.f; in.dir = {0.f, 0.f, 1.f}; in.inv_norm = 0.f;
        if (h0) build_x_row(p, row, valid, t, s_x, in);
        fence_async_smem();
        __syncthreads();
        // ---- forward recompute (per warpgroup, as in the forward kernel) ----------------------------------------------
        gemm_n128<AP_K1 / 16>(acc, s_x, w1p, w);
        relu_epilogue(acc, s_h1, f);
        fence_async_smem();
        warpgroup_sync(w);
        gemm_n128<AP_K2 / 16>(acc, s_h1, w2p, w);
        relu_epilogue(acc, s_h2, f);
        fence_async_smem();
        warpgroup_sync(w);
        gemm_n16(acc3, s_h2, w3p, w);
        store_out(acc3, s_out, f);
        __syncthreads();
        if (bulk) {
            if (!mbar_wait(&bars[0], ph_ld)) AP_FAIL();
            ph_ld ^= 1u;
        }

        // ---- colour stage backward: dL/d{raw, toned} -> dL/d features, dL/d(offset, mul), dL/d mean ----------------
        float dOut[AP_NOUT] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        float g_dc[3] = {0.f, 0.f, 0.f};          // gradient w.r.t. min(dc, 1) from the colour sums (the MLP path is added later)
        if (valid) {
            const float* o = s_out + t * 8;
            float b[16], gk[16];
            sh_basis(p.deg, in.dir.x, in.dir.y, in.dir.z, b);
#pragma unroll
            for (int k = 0; k < 16; ++k) gk[k] = 0.f;
            float* fr = s_rest + t * AP_NREST;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float mul = 0.01f * o[3 + c], off = 0.01f * o[c] / SH_C0;
                const float f0 = fminf(in.dc[c], 1.0f);
                const float t0p = fmaf(f0, mul, off);
                float r = b[0] * f0, s = b[0] * fminf(t0p, 1.0f);
#pragma unroll
                for (int k = 1; k < 16; ++k) {
                    const float fv = fminf(fr[3 * (k - 1) + c], 1.0f);
                    r = fmaf(b[k], fv, r);
                    s = fmaf(b[k], fminf(fv * mul, 1.0f), s);
                }
                // clamp_min(x + 0.5, 0) passes the gradient where x + 0.5 >= 0
                const float dLr = (p.dL_raw != nullptr && r + 0.5f >= 0.f) ? p.dL_raw[(size_t)row * 3 + c] : 0.f;
                const float dLt = (s + 0.5f >= 0.f) ? p.dL_toned[(size_t)row * 3 + c] : 0.f;
                float dmul = 0.f;
                {   // k = 0
                    const float dt = (t0p <= 1.0f) ? b[0] * dLt : 0.f;
                    dmul = dt * f0;
                    dOut[c] = 0.01f * dt / SH_C0;
                    g_dc[c] = fmaf(dt, mul, b[0] * dLr);
                    gk[0] += dLr * f0 + dLt * fminf(t0p, 1.0f);
                }
#pragma unroll
                for (int k = 1; k < 16; ++k) {
                    const float fu = fr[3 * (k - 1) + c];
                    const float fv = fminf(fu, 1.0f);
                    const float tp = fv * mul;
                    const float dt = (tp <= 1.0f) ? b[k] * dLt : 0.f;
                    dmul = fmaf(dt, fv, dmul);
                    gk[k] += dLr * fv + dLt * fminf(tp, 1.0f);
                    // gradient of features_rest (clamp_max(1) passes it where the raw value <= 1), written in place
                    fr[3 * (k - 1) + c] = (fu <= 1.0f) ? fmaf(dt, mul, b[k] * dLr) : 0.f;
                }
                dOut[3 + c] = 0.01f * dmul;
            }
            // view direction -> mean (eval_sh is differentiated through `dir`, method.py:1572)
            const float3 dd = sh_basis_grad_dot(p.deg, in.dir.x, in.dir.y, in.dir.z, gk);
            const float3 dm = through_normalize(in.dir, in.inv_norm, dd);
            p.g_means[(size_t)row * 3 + 0] = dm.x;
            p.g_means[(size_t)row * 3 + 1] = dm.y;
            p.g_means[(size_t)row * 3 + 2] = dm.z;
        }
        // dO (bf16) -> shared memory; bias gradient of the last layer = column sums of dO (fp32, warp shuffles)
        if (h0) {
            st_chunk(s_do, 0, t, make_uint4(pack_bf16(dOut[0], dOut[1]), pack_bf16(dOut[2], dOut[3]), pack_bf16(dOut[4], dOut[5]), 0u));
#pragma unroll
            for (int j = 0; j < AP_NOUT; ++j) {
                float v = dOut[j];
#pragma unroll
                for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, s);
                if (lane == 0) atomicAdd(&s_db3[j], v);
            }
        }
        fence_async_smem();
        __syncthreads();
        // coalesced copy-out of the tile's features_rest gradients (they replaced the features in s_rest)
        for (int i = tid; i < rows * AP_NREST; i += BWD_THREADS) p.g_rest[(size_t)row0 * AP_NREST + i] = s_rest[i];
        // ---- layer 3 backward --------------------------------------------------------------------------------------
        fence_regs(acc); fence_regs(gw3);
        fence();
        // dH2 = dO . W3           A: dO K-major (K = 16 outputs), B: W3p as MN-major (N = 128 inputs)
        mma_n128<0, 1>(acc, desc_k(s_do + w * 1024, 0, AP_TILE), desc_mn(w3p, 0, AP_N3), false);
        // dW3p^T[128 in][16 out] += H2^T . dO      both MN-major, K = the 128 Gaussians of the tile
#pragma unroll
        for (int k = 0; k < AP_TILE / 16; ++k) mma_n16<1, 1>(gw3, desc_mn(s_h2 + w * MN_HALF, k, AP_TILE), desc_mn(s_do, k, AP_TILE), true);
        commit_group();
        wait_all();
        fence_regs(acc); fence_regs(gw3);
        relu_bwd_epilogue(acc, s_h2, s_dz, f);
        fence_async_smem();
        __syncthreads();
        // ---- layer 2 backward --------------------------------------------------------------------------------------
        fence_regs(acc); fence_regs(gw2);
        fence();
        // dW2p[128 out][144 in] += dZ2^T . H1p   (column 128 of H1p is the constant one: bias gradient)
#pragma unroll
        for (int k = 0; k < AP_TILE / 16; ++k) mma_n144<1, 1>(gw2, desc_mn(s_dz + w * MN_HALF, k, AP_TILE), desc_mn(s_h1, k, AP_TILE), true);
        // dH1 = dZ2 . W2          A: dZ2 K-major (K = 128 outputs), B: W2p MN-major (N = 128 inputs)
#pragma unroll
        for (int k = 0; k < AP_H / 16; ++k) mma_n128<0, 1>(acc, desc_k(s_dz + w * 1024, k, AP_TILE), desc_mn(w2p, k, AP_H), k > 0);
        commit_group();
        wait_all();
        fence_regs(acc); fence_regs(gw2);
        __syncthreads();          // the other warpgroup's weight-gradient GEMM reads every row of s_dz
        relu_bwd_epilogue(acc, s_h1, s_dz, f);
        fence_async_smem();
        __syncthreads();
        // ---- layer 1 backward --------------------------------------------------------------------------------------
        fence_regs(accx); fence_regs(gw1);
        fence();
#pragma unroll
        for (int k = 0; k < AP_TILE / 16; ++k) mma_n32<1, 1>(gw1, desc_mn(s_dz + w * MN_HALF, k, AP_TILE), desc_mn(s_x, k, AP_TILE), true);
#pragma unroll
        for (int k = 0; k < AP_H / 16; ++k) mma_n32<0, 1>(accx, desc_k(s_dz + w * 1024, k, AP_TILE), desc_mn(w1p, k, AP_H), k > 0);
        commit_group();
        wait_all();
        fence_regs(accx); fence_regs(gw1);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            *reinterpret_cast<float2*>(s_dx + f.r0 * DX_LD + 8 * j + 2 * f.c) = make_float2(accx[4 * j], accx[4 * j + 1]);
            *reinterpret_cast<float2*>(s_dx + (f.r0 + 8) * DX_LD + 8 * j + 2 * f.c) = make_float2(accx[4 * j + 2], accx[4 * j + 3]);
        }
        __syncthreads();
        if (valid) {
            const float* dx = s_dx + t * DX_LD;
#pragma unroll
            for (int c = 0; c < 3; ++c)      // x[c] = min(dc, 1): both paths pass where dc <= 1
                p.g_dc[(size_t)row * 3 + c] = (in.dc[c] <= 1.0f) ? g_dc[c] + dx[c] : 0.f;
            float4* gg = reinterpret_cast<float4*>(p.g_gemb + (size_t)row * AP_NGEMB);
#pragma unroll
            for (int i = 0; i < AP_NGEMB / 4; ++i) gg[i] = make_float4(dx[3 + 4 * i], dx[4 + 4 * i], dx[5 + 4 * i], dx[6 + 4 * i]);
        }
        fence_async_smem();
        __syncthreads();
    }

    // ---- reduce the CTA's weight-gradient accumulators to HBM ---------------------------------------------------------
    if (iter > 0 && !dead) {
        float* g = p.g_pack;
        flush_frag(gw2, g + GW2P, AP_K2, f);
        flush_frag(gw1, g + GW1P, AP_K1, f);
        flush_frag(gw3, g + GW3P, AP_N3, f);
        if (tid < AP_NOUT) atomicAdd(g + GB3 + tid, s_db3[tid]);
    }
}

// =====================================================================================================================
// embedding-only backward (test-time appearance optimisation)
// =====================================================================================================================
// When only the image embedding is optimised, its gradient is W1[:, 27:59]^T . sum_rows dZ1 (the embedding is folded
// into the layer-1 bias), and the unpack kernel forms that product from the db1 slot of the gradient image.  This kernel
// therefore recomputes the three layers per tile as appearance_bwd_kernel does, runs dO -> dZ2 -> dZ1 and accumulates
// only sum_rows dZ1: no weight-gradient GEMM, no dX, no per-Gaussian input gradient.  The ReLU masks of H1 and H2 stay
// in registers (the dH accumulators have the layout of the forward accumulators), so one activation image serves all
// layers, dO reuses the layer-3 output rows and the per-warp column sums reuse the SH staging area: the shared memory
// is the forward kernel's and two CTAs fit an SM.

// relu_epilogue, also returning which of this thread's 64 accumulator entries are positive after the bf16 rounding
// (bit i of pos[i / 32] for d[i]), the mask relu_bwd_epilogue reads back from the activation image
__device__ __forceinline__ void relu_epilogue_mask(const float (&d)[64], uint8_t* hbuf, Frag f, uint32_t (&pos)[2]) {
    pos[0] = pos[1] = 0u;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const uint32_t a = pack_bf16(fmaxf(d[4 * j], 0.f), fmaxf(d[4 * j + 1], 0.f));
        const uint32_t b = pack_bf16(fmaxf(d[4 * j + 2], 0.f), fmaxf(d[4 * j + 3], 0.f));
        st_pair(hbuf, j, f.r0, f.c, a);
        st_pair(hbuf, j, f.r0 + 8, f.c, b);
        const uint32_t m = ((a & 0x7FFFu) ? 1u : 0u) | ((a & 0x7FFF0000u) ? 2u : 0u) | ((b & 0x7FFFu) ? 4u : 0u) |
                           ((b & 0x7FFF0000u) ? 8u : 0u);
        pos[j >> 3] |= m << (4 * (j & 7));
    }
}
__device__ __forceinline__ float masked_bf16(const uint32_t (&pos)[2], int i, float v) {
    return ((pos[i >> 5] >> (i & 31)) & 1u) ? __bfloat162float(__float2bfloat16(v)) : 0.f;
}

// the RowIn that build_x_row returns for a valid row (same expressions, so the same bits)
__device__ __forceinline__ void row_in(const ApParams& p, int row, RowIn& in) {
#pragma unroll
    for (int c = 0; c < 3; ++c) in.dc[c] = p.dc[(size_t)row * 3 + c];
    const float vx = p.means[(size_t)row * 3 + 0] - p.campos[0], vy = p.means[(size_t)row * 3 + 1] - p.campos[1],
                vz = p.means[(size_t)row * 3 + 2] - p.campos[2];
    const float nrm = fmaxf(sqrtf(vx * vx + vy * vy + vz * vz), 1e-12f);
    in.inv_norm = 1.0f / nrm;
    in.dir = {vx * in.inv_norm, vy * in.inv_norm, vz * in.inv_norm};
}

// dL/d(o) of the toned colour of one row (o = the six MLP outputs before the x 0.01): the colour-stage backward of
// appearance_bwd_kernel restricted to the toned path
__device__ __forceinline__ void toned_dout(int deg, const RowIn& in, const float* o, const float* fr, const float* dL_toned,
                                           float (&dOut)[AP_NOUT]) {
    float b[16];
    sh_basis(deg, in.dir.x, in.dir.y, in.dir.z, b);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float mul = 0.01f * o[3 + c], off = 0.01f * o[c] / SH_C0;
        const float f0 = fminf(in.dc[c], 1.0f);
        const float t0p = fmaf(f0, mul, off);
        float s = b[0] * fminf(t0p, 1.0f);
#pragma unroll
        for (int k = 1; k < 16; ++k) s = fmaf(b[k], fminf(fminf(fr[3 * (k - 1) + c], 1.0f) * mul, 1.0f), s);
        const float dLt = (s + 0.5f >= 0.f) ? dL_toned[c] : 0.f;
        const float dt0 = (t0p <= 1.0f) ? b[0] * dLt : 0.f;
        float dmul = dt0 * f0;
        dOut[c] = 0.01f * dt0 / SH_C0;
#pragma unroll
        for (int k = 1; k < 16; ++k) {
            const float fv = fminf(fr[3 * (k - 1) + c], 1.0f);
            const float dt = (fv * mul <= 1.0f) ? b[k] * dLt : 0.f;
            dmul = fmaf(dt, fv, dmul);
        }
        dOut[3 + c] = 0.01f * dmul;
    }
}

__global__ void __launch_bounds__(FWD_THREADS, 2) appearance_emb_bwd_kernel(const __grid_constant__ ApParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* s_blob = smem;
    uint8_t* s_act = smem + BLOB_BYTES;
    float* s_rest = reinterpret_cast<float*>(smem + BLOB_BYTES + ACT_BYTES);
    float* s_out = reinterpret_cast<float*>(smem + BLOB_BYTES + ACT_BYTES + REST_BYTES);
    uint8_t* s_do = reinterpret_cast<uint8_t*>(s_out);        // dO image (2 chunks) over the consumed layer-3 output rows
    float* s_colsum = s_rest;                                 // [8 warps][128] dZ1 column sums over the consumed SH rows
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + BLOB_BYTES + ACT_BYTES + REST_BYTES + OUT_BYTES);
    const int tid = threadIdx.x, t = tid & (AP_TILE - 1), w = tid >> 7, lane = tid & 31, warp = tid >> 5;
    const bool h0 = w == 0;
    const Frag f = frag_of(tid);

    if (tid == 0) {
        mbar_init(&bars[0], 1); mbar_init(&bars[1], 1);
        mbar_init_fence();
    }
    if (h0) write_const_chunks(s_act, t);
    fence_async_smem();
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(&bars[1], BLOB_BYTES);
        bulk_g2s(s_blob, p.blob, BLOB_BYTES, &bars[1]);
    }
    const uint8_t* w1p = s_blob;
    const uint8_t* w2p = s_blob + W1P_BYTES;
    const uint8_t* w3p = w2p + W2P_BYTES;
    float acc[64], acc3[8];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc3[i] = 0.f;
    float colsum = 0.f;                                       // thread n < 128: sum of dZ1[:, n] over this CTA's tiles
    uint32_t ph_ld = 0;
    bool dead = false;
    if (!mbar_wait(&bars[1], 0)) AP_FAIL();

    for (int tile = blockIdx.x; tile < p.num_tiles && !dead; tile += gridDim.x) {
        const int row0 = tile * AP_TILE, row = row0 + t;
        const int rows = min(AP_TILE, p.P - row0);
        const bool valid = h0 && t < rows;
        const bool bulk = rows == AP_TILE;
        if (bulk) {
            if (tid == 0) {
                mbar_expect_tx(&bars[0], REST_BYTES);
                bulk_g2s(s_rest, p.rest + (size_t)row0 * AP_NREST, REST_BYTES, &bars[0]);
            }
        } else {
            for (int i = tid; i < rows * AP_NREST; i += FWD_THREADS) s_rest[i] = p.rest[(size_t)row0 * AP_NREST + i];
        }
        {   // the row input is read again for the colour stage rather than held across the GEMMs (register budget)
            RowIn in;
            if (h0) build_x_row(p, row, valid, t, s_act, in);
        }
        fence_async_smem();
        __syncthreads();
        // ---- forward recompute (a warpgroup reads and overwrites only its own 64 rows) -----------------------------------
        uint32_t pos1[2], pos2[2];
        gemm_n128<AP_K1 / 16>(acc, s_act, w1p, w);
        relu_epilogue_mask(acc, s_act, f, pos1);
        fence_async_smem();
        warpgroup_sync(w);
        gemm_n128<AP_K2 / 16>(acc, s_act, w2p, w);
        relu_epilogue_mask(acc, s_act, f, pos2);
        fence_async_smem();
        warpgroup_sync(w);
        gemm_n16(acc3, s_act, w3p, w);
        store_out(acc3, s_out, f);
        __syncthreads();
        if (bulk) {
            if (!mbar_wait(&bars[0], ph_ld)) AP_FAIL();
            ph_ld ^= 1u;
        }
        // ---- colour stage: dL/d(toned) -> dO ------------------------------------------------------------------------
        float dOut[AP_NOUT] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (valid) {
            RowIn in;
            row_in(p, row, in);
            toned_dout(p.deg, in, s_out + t * 8, s_rest + t * AP_NREST, p.dL_toned + (size_t)row * 3, dOut);
        }
        __syncthreads();          // every row of s_out and s_rest has been read: both are rewritten below
        if (h0) {
            st_chunk(s_do, 0, t, make_uint4(pack_bf16(dOut[0], dOut[1]), pack_bf16(dOut[2], dOut[3]), pack_bf16(dOut[4], dOut[5]), 0u));
            st_chunk(s_do, 1, t, make_uint4(0u, 0u, 0u, 0u));
        }
        fence_async_smem();
        __syncthreads();
        // ---- dH2 = dO . W3 -> dZ2 (bf16, over H2 in the activation image) -------------------------------------------------
        // (the GEMM does not accumulate: clearing acc ends the previous GEMM's live range before the colour stage)
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        fence_regs(acc);
        fence();
        mma_n128<0, 1>(acc, desc_k(s_do + w * 1024, 0, AP_TILE), desc_mn(w3p, 0, AP_N3), false);
        commit_group();
        wait_all();
        fence_regs(acc);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            st_pair(s_act, j, f.r0, f.c, pack_bf16(masked_bf16(pos2, 4 * j, acc[4 * j]), masked_bf16(pos2, 4 * j + 1, acc[4 * j + 1])));
            st_pair(s_act, j, f.r0 + 8, f.c,
                    pack_bf16(masked_bf16(pos2, 4 * j + 2, acc[4 * j + 2]), masked_bf16(pos2, 4 * j + 3, acc[4 * j + 3])));
        }
        fence_async_smem();
        warpgroup_sync(w);
        // ---- dH1 = dZ2 . W2 -> dZ1 (bf16, as the weight-gradient GEMM of appearance_bwd_kernel reads it) -------------------
        fence_regs(acc);
        fence();
#pragma unroll
        for (int k = 0; k < AP_H / 16; ++k) mma_n128<0, 1>(acc, desc_k(s_act + w * 1024, k, AP_TILE), desc_mn(w2p, k, AP_H), k > 0);
        commit_group();
        wait_all();
        fence_regs(acc);
        // column sums of dZ1: this thread's two rows, then the 8 row groups of the warp (lanes differing in bits 2..4)
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            float s0 = masked_bf16(pos1, 4 * j, acc[4 * j]) + masked_bf16(pos1, 4 * j + 2, acc[4 * j + 2]);
            float s1 = masked_bf16(pos1, 4 * j + 1, acc[4 * j + 1]) + masked_bf16(pos1, 4 * j + 3, acc[4 * j + 3]);
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
                s0 += __shfl_xor_sync(0xFFFFFFFFu, s0, o);
                s1 += __shfl_xor_sync(0xFFFFFFFFu, s1, o);
            }
            if (lane < 4) *reinterpret_cast<float2*>(s_colsum + warp * AP_H + 8 * j + 2 * f.c) = make_float2(s0, s1);
        }
        __syncthreads();
        if (tid < AP_H) {
#pragma unroll
            for (int k = 0; k < FWD_THREADS / 32; ++k) colsum += s_colsum[k * AP_H + tid];
        }
        fence_async_smem();       // generic accesses of s_rest / s_act are ordered before the next tile's bulk copy into them
        __syncthreads();
    }
    // db1 slot of the gradient image: dW1p[n][AP_ONE1] = sum over the Gaussians of dZ1[:, n] (X[:, AP_ONE1] = 1)
    if (tid < AP_H && !dead && blockIdx.x < p.num_tiles) atomicAdd(p.g_pack + GW1P + (size_t)tid * AP_K1 + AP_ONE1, colsum);
}

// ---- host side ----------------------------------------------------------------------------------------------------
static int ap_num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
}

static int ap_check(const GsrAppearanceArgs* a, bool bwd) {
    if (!a) { set_error("args is NULL"); return GSR_E_INVALID; }
    if (a->P < 0 || a->sh_degree < 0 || a->sh_degree > 3) { set_error("bad P / sh_degree"); return GSR_E_INVALID; }
    if (a->P == 0) return 0;
    if (!a->features_dc || !a->features_rest || !a->embeddings || !a->means3D || !a->campos || !a->packed_weights ||
        (!bwd && !a->colors_toned)) {
        set_error("a required pointer is NULL");
        return GSR_E_INVALID;
    }
    if ((reinterpret_cast<uintptr_t>(a->features_rest) | reinterpret_cast<uintptr_t>(a->embeddings) |
         reinterpret_cast<uintptr_t>(a->packed_weights)) & 15u) {
        set_error("features_rest / embeddings / packed_weights must be 16-byte aligned");
        return GSR_E_INVALID;
    }
    if (bwd) {
        if (!a->dL_dcolors_toned || !a->dL_dfeatures_dc || !a->dL_dfeatures_rest || !a->dL_dembeddings || !a->dL_dmeans3D || !a->grad_pack) {
            set_error("a required gradient pointer is NULL");
            return GSR_E_INVALID;
        }
        if (reinterpret_cast<uintptr_t>(a->dL_dembeddings) & 15u) { set_error("dL_dembeddings must be 16-byte aligned"); return GSR_E_INVALID; }
    }
    return 0;
}

static ApParams ap_params(const GsrAppearanceArgs* a) {
    ApParams p{};
    p.P = a->P; p.deg = a->sh_degree; p.num_tiles = (a->P + AP_TILE - 1) / AP_TILE;
    p.dc = a->features_dc; p.rest = a->features_rest; p.gemb = a->embeddings; p.means = a->means3D; p.campos = a->campos;
    p.blob = reinterpret_cast<const uint8_t*>(a->packed_weights);
    p.raw = a->colors_raw; p.toned = a->colors_toned;
    p.dL_raw = a->dL_dcolors_raw; p.dL_toned = a->dL_dcolors_toned;
    p.g_dc = a->dL_dfeatures_dc; p.g_rest = a->dL_dfeatures_rest; p.g_gemb = a->dL_dembeddings; p.g_means = a->dL_dmeans3D;
    p.g_pack = a->grad_pack; p.status = a->status;
    return p;
}

}  // namespace gsr

using namespace gsr;

extern "C" {

size_t gsr_appearance_packed_weight_bytes(void) { return BLOB_BYTES; }
size_t gsr_appearance_grad_pack_bytes(void) { return GPACK_FLOATS * sizeof(float); }

int gsr_appearance_pack_weights(const float* W1, const float* b1, const float* W2, const float* b2, const float* W3,
                                const float* b3, const float* appearance_embedding, void* packed_weights, void* stream) {
    if (!W1 || !b1 || !W2 || !b2 || !W3 || !b3 || !appearance_embedding || !packed_weights) { set_error("NULL argument"); return GSR_E_INVALID; }
    appearance_pack_kernel<<<1, 128, 0, (cudaStream_t)stream>>>(W1, b1, W2, b2, W3, b3, appearance_embedding,
                                                                reinterpret_cast<uint8_t*>(packed_weights));
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

int gsr_appearance_colors_forward(const GsrAppearanceArgs* a, void* stream) {
    int rc = ap_check(a, false);
    if (rc || a->P == 0) return rc;
    const ApParams p = ap_params(a);
    GSR_CUDA(cudaFuncSetAttribute(appearance_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FWD_SMEM));
    const int grid = min(p.num_tiles, 2 * ap_num_sms());      // persistent: two resident CTAs per SM
    appearance_fwd_kernel<<<grid, FWD_THREADS, FWD_SMEM, (cudaStream_t)stream>>>(p);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

int gsr_appearance_colors_backward(const GsrAppearanceArgs* a, void* stream) {
    int rc = ap_check(a, true);
    if (rc || a->P == 0) return rc;
    const ApParams p = ap_params(a);
    cudaStream_t s = (cudaStream_t)stream;
    GSR_CUDA(cudaMemsetAsync(a->grad_pack, 0, GPACK_FLOATS * sizeof(float), s));
    GSR_CUDA(cudaFuncSetAttribute(appearance_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_SMEM));
    const int grid = min(p.num_tiles, ap_num_sms());          // persistent: one CTA per SM (187 KB of shared memory)
    appearance_bwd_kernel<<<grid, BWD_THREADS, BWD_SMEM, s>>>(p);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

int gsr_appearance_embedding_backward(const GsrAppearanceArgs* a, void* stream) {
    if (!a) { set_error("args is NULL"); return GSR_E_INVALID; }
    if (a->P < 0 || a->sh_degree < 0 || a->sh_degree > 3) { set_error("bad P / sh_degree"); return GSR_E_INVALID; }
    if (!a->grad_pack) { set_error("grad_pack is NULL"); return GSR_E_INVALID; }
    if (a->P > 0) {
        if (!a->features_dc || !a->features_rest || !a->embeddings || !a->means3D || !a->campos || !a->packed_weights ||
            !a->dL_dcolors_toned) {
            set_error("a required pointer is NULL");
            return GSR_E_INVALID;
        }
        if ((reinterpret_cast<uintptr_t>(a->features_rest) | reinterpret_cast<uintptr_t>(a->embeddings) |
             reinterpret_cast<uintptr_t>(a->packed_weights)) & 15u) {
            set_error("features_rest / embeddings / packed_weights must be 16-byte aligned");
            return GSR_E_INVALID;
        }
    }
    cudaStream_t s = (cudaStream_t)stream;
    GSR_CUDA(cudaMemsetAsync(a->grad_pack, 0, GPACK_FLOATS * sizeof(float), s));
    if (a->P == 0) return 0;
    const ApParams p = ap_params(a);
    GSR_CUDA(cudaFuncSetAttribute(appearance_emb_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FWD_SMEM));
    const int grid = min(p.num_tiles, 2 * ap_num_sms());      // persistent: two resident CTAs per SM, as the forward
    appearance_emb_bwd_kernel<<<grid, FWD_THREADS, FWD_SMEM, s>>>(p);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

int gsr_appearance_unpack_grads(const float* grad_pack, const float* W1, const float* appearance_embedding, float* dW1,
                                float* db1, float* dW2, float* db2, float* dW3, float* db3, float* dappearance_embedding,
                                void* stream) {
    if (!grad_pack || !W1 || !appearance_embedding || !dW1 || !db1 || !dW2 || !db2 || !dW3 || !db3 || !dappearance_embedding) {
        set_error("NULL argument");
        return GSR_E_INVALID;
    }
    appearance_unpack_kernel<<<1, 128, 0, (cudaStream_t)stream>>>(grad_pack, W1, appearance_embedding, dW1, db1, dW2, db2, dW3, db3,
                                                                  dappearance_embedding);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"
