// metrics.cu -- the evaluation metrics of wild-gaussians (wildgaussians/evaluation.py `compute_metrics`): per image the
// sums of the squared and absolute differences (MSE, MAE) and of the dm_pix SSIM map, plus, optionally, the LPIPS input
// x * 2 - 1 of both images.
//
//   metrics_tile_kernel   one CTA per (32 x 16 tile of the SSIM's valid map, image, channel); per-CTA partial sums
//   metrics_reduce_kernel one CTA per image; sums that image's partials in a fixed order
//
// Input: each image is [B][H][W][C], uint8 or fp32 (a flag per image), contiguous.  uint8 becomes v / 255.0f (IEEE
// division: numpy 2's `astype(float32) / 255.0`), then every value is clipped to [0, 1] as np.clip does it (NaN passes
// through, -0.0 stays -0.0).
//
// MSE / MAE: d = a - b, d * d and |d| in fp32 with explicitly rounded operations (the terms numpy forms; no contraction),
// accumulated in fp64.  Every input pixel is counted by exactly one CTA: the tile's own 32 x 16 block, and the tiles of the
// last tile row / column also take the 10 rows / columns past the SSIM's valid map.
//
// SSIM (dm_pix defaults: 11 taps, sigma 1.5, k1 0.01, k2 0.03, max_val 1): the maps a, b, a^2, b^2, ab in fp32, filtered
// in fp64 along x, then along y, valid mode ((H - 10) x (W - 10) outputs).  Per output in fp64: mu, sigma; sigma00 and
// sigma11 clamped below at eps_f32^2 = 2^-46, sigma01 clipped to sign(sigma01) min(sqrt(sigma00 sigma11), |sigma01|),
// then the map.  NaN propagates as numpy's maximum / minimum / sign propagate it.  The taps, c1 and c2 come from the host.
//
// No float atomics: the partials go to scratch by CTA index and are summed in a fixed order, so the result is bitwise
// reproducible run to run.
#include "common.cuh"

namespace gsr {

constexpr int MT_TX = 32, MT_TY = 16;                    // valid-map outputs per CTA
constexpr int MT_K = 11, MT_HALO = MT_K - 1;
constexpr int MT_IX = MT_TX + MT_HALO, MT_IY = MT_TY + MT_HALO;
constexpr int MT_THREADS = 256;
constexpr int MT_SUMS = 3;                               // squared differences, absolute differences, SSIM map
constexpr double MT_EPS2 = 1.4210854715202004e-14;       // np.finfo(np.float32).eps ** 2 = 2^-46

__device__ __forceinline__ float mt_load(const void* p, int u8, size_t i) {
    const float v = u8 ? __fdiv_rn((float)static_cast<const unsigned char*>(p)[i], 255.f) : static_cast<const float*>(p)[i];
    return v < 0.f ? 0.f : (v > 1.f ? 1.f : v);
}

// np.maximum / np.minimum: NaN from either side wins
__device__ __forceinline__ double np_max(double x, double y) { return isnan(x) || isnan(y) ? x + y : (x > y ? x : y); }
__device__ __forceinline__ double np_min(double x, double y) { return isnan(x) || isnan(y) ? x + y : (x < y ? x : y); }

__global__ void __launch_bounds__(MT_THREADS) metrics_tile_kernel(GsrMetricsArgs a, double* __restrict__ partials) {
    __shared__ float sa[MT_IY][MT_IX], sb[MT_IY][MT_IX];
    __shared__ double sh[5][MT_IY][MT_TX];
    __shared__ double red[MT_THREADS / 32][MT_SUMS];
    const int H = a.H, W = a.W, C = a.C, Ho = H - MT_HALO, Wo = W - MT_HALO;
    const int x0 = blockIdx.x * MT_TX, y0 = blockIdx.y * MT_TY;
    const int img = blockIdx.z / C, ch = blockIdx.z - img * C;
    // the input pixels this CTA counts: its own block, to the image's edge for the last tile row / column
    const int xe = blockIdx.x == gridDim.x - 1 ? W : x0 + MT_TX;
    const int ye = blockIdx.y == gridDim.y - 1 ? H : y0 + MT_TY;
    const size_t base = (size_t)img * H * W;
    double acc[MT_SUMS] = {0.0, 0.0, 0.0};

    for (int i = threadIdx.x; i < MT_IY * MT_IX; i += MT_THREADS) {
        const int ly = i / MT_IX, lx = i - ly * MT_IX, y = y0 + ly, x = x0 + lx;
        float va = 0.f, vb = 0.f;
        if (y < H && x < W) {
            const size_t e = (base + (size_t)y * W + x) * C + ch;
            va = mt_load(a.a, a.a_u8, e);
            vb = mt_load(a.b, a.b_u8, e);
            if (y < ye && x < xe) {
                const float d = __fsub_rn(va, vb);
                acc[0] += (double)__fmul_rn(d, d);
                acc[1] += (double)fabsf(d);
                if (a.lpips_a) {
                    a.lpips_a[e] = __fsub_rn(__fmul_rn(va, 2.f), 1.f);
                    a.lpips_b[e] = __fsub_rn(__fmul_rn(vb, 2.f), 1.f);
                }
            }
        }
        sa[ly][lx] = va;
        sb[ly][lx] = vb;
    }
    __syncthreads();

    // along x: out[x] = sum_k z[x + k] taps[10 - k] (np.convolve, valid mode)
    for (int i = threadIdx.x; i < MT_IY * MT_TX; i += MT_THREADS) {
        const int ly = i / MT_TX, lx = i - ly * MT_TX;
        double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
        for (int k = 0; k < MT_K; ++k) {
            const float va = sa[ly][lx + k], vb = sb[ly][lx + k];
            const double w = a.taps[MT_K - 1 - k];
            s[0] = fma((double)va, w, s[0]);
            s[1] = fma((double)vb, w, s[1]);
            s[2] = fma((double)__fmul_rn(va, va), w, s[2]);
            s[3] = fma((double)__fmul_rn(vb, vb), w, s[3]);
            s[4] = fma((double)__fmul_rn(va, vb), w, s[4]);
        }
#pragma unroll
        for (int m = 0; m < 5; ++m) sh[m][ly][lx] = s[m];
    }
    __syncthreads();

    // along y, then the SSIM map per output
    for (int i = threadIdx.x; i < MT_TY * MT_TX; i += MT_THREADS) {
        const int ly = i / MT_TX, lx = i - ly * MT_TX;
        if (y0 + ly >= Ho || x0 + lx >= Wo) continue;
        double f[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
        for (int k = 0; k < MT_K; ++k) {
            const double w = a.taps[MT_K - 1 - k];
#pragma unroll
            for (int m = 0; m < 5; ++m) f[m] = fma(sh[m][ly + k][lx], w, f[m]);
        }
        const double mu0 = f[0], mu1 = f[1];
        const double mu00 = __dmul_rn(mu0, mu0), mu11 = __dmul_rn(mu1, mu1), mu01 = __dmul_rn(mu0, mu1);
        const double s00 = np_max(MT_EPS2, __dsub_rn(f[2], mu00));
        const double s11 = np_max(MT_EPS2, __dsub_rn(f[3], mu11));
        double s01 = __dsub_rn(f[4], mu01);
        const double sgn = s01 > 0.0 ? 1.0 : (s01 < 0.0 ? -1.0 : s01);       // np.sign: 0 -> 0, NaN -> NaN
        s01 = __dmul_rn(sgn, np_min(__dsqrt_rn(__dmul_rn(s00, s11)), fabs(s01)));
        const double numer = __dmul_rn(__dadd_rn(__dmul_rn(2.0, mu01), a.c1), __dadd_rn(__dmul_rn(2.0, s01), a.c2));
        const double denom = __dmul_rn(__dadd_rn(__dadd_rn(mu00, mu11), a.c1), __dadd_rn(__dadd_rn(s00, s11), a.c2));
        acc[2] += __ddiv_rn(numer, denom);
    }

    block_sum_f64<MT_THREADS>(acc, red);
    if (threadIdx.x == 0) {
        const size_t cta = ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
#pragma unroll
        for (int k = 0; k < MT_SUMS; ++k) partials[cta * MT_SUMS + k] = acc[k];
    }
}

// image b's partials are the contiguous CTA range [b * per_image, (b + 1) * per_image) (blockIdx.z = b * C + c)
__global__ void __launch_bounds__(MT_THREADS) metrics_reduce_kernel(const double* __restrict__ partials, int per_image,
                                                                     double* __restrict__ sums) {
    __shared__ double red[MT_THREADS / 32][MT_SUMS];
    const double* p = partials + (size_t)blockIdx.x * per_image * MT_SUMS;
    double acc[MT_SUMS] = {0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < per_image; i += MT_THREADS)
#pragma unroll
        for (int k = 0; k < MT_SUMS; ++k) acc[k] += p[(size_t)i * MT_SUMS + k];
    block_sum_f64<MT_THREADS>(acc, red);
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < MT_SUMS; ++k) sums[(size_t)blockIdx.x * MT_SUMS + k] = acc[k];
}

static size_t mt_ctas(int B, int H, int W, int C) {
    return (size_t)((W - MT_HALO + MT_TX - 1) / MT_TX) * ((H - MT_HALO + MT_TY - 1) / MT_TY) * B * C;
}

static bool mt_sizes_ok(int B, int H, int W, int C) {
    if (B <= 0 || H < MT_K || W < MT_K || C <= 0) return false;
    if ((long long)B * C > 65535 || (H - MT_HALO + MT_TY - 1) / MT_TY > 65535) return false;
    return mt_ctas(1, H, W, C) <= 0x7fffffffu;           // one image's partials are counted in an int
}

}  // namespace gsr

extern "C" size_t gsr_metrics_scratch_bytes(int B, int H, int W, int C) {
    using namespace gsr;
    if (!mt_sizes_ok(B, H, W, C)) return 0;
    return mt_ctas(B, H, W, C) * MT_SUMS * sizeof(double);
}

extern "C" int gsr_metrics_forward(const GsrMetricsArgs* args, void* stream) {
    using namespace gsr;
    if (!args) { set_error("args is NULL"); return GSR_E_INVALID; }
    const GsrMetricsArgs& a = *args;
    if (!mt_sizes_ok(a.B, a.H, a.W, a.C)) {
        set_error("bad metric sizes B=%d H=%d W=%d C=%d (H, W >= 11, B * C <= 65535)", a.B, a.H, a.W, a.C);
        return GSR_E_INVALID;
    }
    if (!a.a || !a.b || !a.sums || !a.scratch) { set_error("a, b, sums or scratch is NULL"); return GSR_E_INVALID; }
    if (!a.lpips_a != !a.lpips_b) { set_error("lpips_a and lpips_b must both be given or both be NULL"); return GSR_E_INVALID; }
    for (int k = 0; k < MT_K; ++k)
        if (!isfinite(a.taps[k])) { set_error("taps[%d] is not finite", k); return GSR_E_INVALID; }
    if (!isfinite(a.c1) || !isfinite(a.c2)) { set_error("c1 or c2 is not finite"); return GSR_E_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    const dim3 grid((a.W - MT_HALO + MT_TX - 1) / MT_TX, (a.H - MT_HALO + MT_TY - 1) / MT_TY, a.B * a.C);
    double* partials = static_cast<double*>(a.scratch);
    metrics_tile_kernel<<<grid, MT_THREADS, 0, s>>>(a, partials);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    metrics_reduce_kernel<<<a.B, MT_THREADS, 0, s>>>(partials, (int)(grid.x * grid.y * a.C), a.sums);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}
