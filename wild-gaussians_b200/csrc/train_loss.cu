// train_loss.cu -- the photometric loss block of wild-gaussians' training step and its metric sums, plus the unpacking
// of byte-staged training images.
//
// What it replaces: wildgaussians/method.py:1920-1992 around the fused SSIM -- scale_grads by the mask and by loss_mult,
// l1_loss, the two weighted means of the loss, mse / psnr and the masked metric reductions -- about a dozen PyTorch
// launches forward, their autograd graph backward, and five (ten with a mask) `.item()` read-backs.
//
//   forward  (3 launches): train_loss_pixels_kernel -> gsr_ssim_forward -> train_loss_ssim_kernel
//   backward (2 launches): train_loss_bwd_kernel    -> the SSIM backward (ssim.cu), scaled per pixel
//
// Definitions (per pixel p, channel c; sg(v, s) = v s + v (1 - s) is the forward value of scale_grads, method.py:120-123):
//   T2 = sg(sg(toned, m), s),  R2 = sg(sg(raw, m), s)         m: mask (absent = no scaling), s: grad_scale (absent = 1)
//   L1 = |T2 - gt|,  MSE = (T2 - gt)^2,  S = ssim_map(R2, gt)
//   loss = c_l1 * mean(L1 * w) + c_ssim * mean((1 - S) * w)                 w: weight (absent = 1)
// with c_l1 = fp32(1 - lambda_dssim) and c_ssim = fp32(lambda_dssim) as the caller rounds them (method.py:1961-1964).
// sg is evaluated with explicitly rounded operations, so its value is the reference's bit for bit (no contraction).
// Every reduction goes through per-CTA partials in double and one final pass in a fixed order by the last CTA (an
// integer ticket picks it): no float atomics, results are bitwise reproducible run to run.  The outputs are computed
// from the double sums and rounded to fp32 once.  This deliberately differs from the reference's rounding: it evaluates
// the loss and psnr as chains of fp32 operations (fp32 means, fp32 products and sum, log10 of the fp32 mean), each step
// rounding; one rounding of the double value is at least as close to the exact result (tests/test_fused_train.py holds
// both to the float64 oracle).
//
// Backward (autograd's chain for :1920-1966, upstream g = dL/dloss):
//   dL/dT2 = (fl(fl(g c_l1) / 3HW) * w) * sign(T2 - gt),      dL/dtoned = (dL/dT2 * s) * m        (sign(0) = 0)
//   dL/dmap = -(fl(fl(g c_ssim) / HW) * w),                    dL/draw   = (ssim_backward(dL/dmap) * s) * m
#include "ssim_common.cuh"

namespace gsr {

constexpr int TL_THREADS = 256;
constexpr int TL_MAX_CTAS = 1024;
constexpr int TL_PIX_SUMS = 6;    // L1 * w, L1, MSE, L1 * m, MSE * m, m
constexpr int TL_MAP_SUMS = 3;    // (1 - S) * w, S, S * m

__device__ __forceinline__ float scale_grads_value(float v, float s) {
    return __fadd_rn(__fmul_rn(v, s), __fmul_rn(v, __fsub_rn(1.f, s)));
}

static int tl_ctas(long long HW) {
    const long long n = (HW + TL_THREADS - 1) / TL_THREADS;
    return (int)(n < TL_MAX_CTAS ? n : TL_MAX_CTAS);
}

struct TlScratch {
    double* pix;          // [TL_MAX_CTAS][TL_PIX_SUMS]
    double* map;          // [TL_MAX_CTAS][TL_MAP_SUMS]
    unsigned int* ticket;
};

static TlScratch tl_scratch(void* base) {
    TlScratch s;
    s.pix = (double*)base;
    s.map = s.pix + (size_t)TL_MAX_CTAS * TL_PIX_SUMS;
    s.ticket = (unsigned int*)(s.map + (size_t)TL_MAX_CTAS * TL_MAP_SUMS);
    return s;
}

__global__ void __launch_bounds__(TL_THREADS) train_loss_pixels_kernel(GsrTrainLossArgs a, TlScratch s) {
    __shared__ double sh[TL_THREADS / 32][TL_PIX_SUMS];
    const size_t HW = (size_t)a.H * a.W;
    if (blockIdx.x == 0 && threadIdx.x == 0) *s.ticket = 0u;     // read by train_loss_ssim_kernel, later in the stream
    double acc[TL_PIX_SUMS] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    const bool scale_raw = a.mask || a.grad_scale;
    for (size_t p = (size_t)blockIdx.x * TL_THREADS + threadIdx.x; p < HW; p += (size_t)gridDim.x * TL_THREADS) {
        const float m = a.mask ? a.mask[p] : 1.f;
        const float sc = a.grad_scale ? a.grad_scale[p] : 1.f;
        const float w = a.weight ? a.weight[p] : 1.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const size_t i = (size_t)c * HW + p;
            float t = a.toned[i];
            if (a.mask) t = scale_grads_value(t, m);
            if (a.grad_scale) t = scale_grads_value(t, sc);
            if (scale_raw) {
                float r = a.raw[i];
                if (a.mask) r = scale_grads_value(r, m);
                if (a.grad_scale) r = scale_grads_value(r, sc);
                a.raw_scaled[i] = r;
            }
            const float d = __fsub_rn(t, a.gt[i]);
            const float l1 = fabsf(d), e = __fmul_rn(d, d);
            acc[0] += a.weight ? (double)__fmul_rn(l1, w) : (double)l1;
            acc[1] += l1;
            acc[2] += e;
            if (a.mask) {
                acc[3] += __fmul_rn(l1, m);
                acc[4] += __fmul_rn(e, m);
            }
        }
        if (a.mask) acc[5] += m;
    }
    block_sum_f64<TL_THREADS>(acc, sh);
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < TL_PIX_SUMS; ++k) s.pix[(size_t)blockIdx.x * TL_PIX_SUMS + k] = acc[k];
}

__global__ void __launch_bounds__(TL_THREADS) train_loss_ssim_kernel(GsrTrainLossArgs a, TlScratch s, int n_pix_ctas) {
    __shared__ double sh[TL_THREADS / 32][TL_PIX_SUMS + TL_MAP_SUMS];
    __shared__ double shm[TL_THREADS / 32][TL_MAP_SUMS];
    __shared__ bool last;
    const size_t HW = (size_t)a.H * a.W;
    double acc[TL_MAP_SUMS] = {0.0, 0.0, 0.0};
    for (size_t p = (size_t)blockIdx.x * TL_THREADS + threadIdx.x; p < HW; p += (size_t)gridDim.x * TL_THREADS) {
        const float S = a.ssim_map[p];
        const float d = __fsub_rn(1.f, S);
        acc[0] += a.weight ? (double)__fmul_rn(d, a.weight[p]) : (double)d;
        acc[1] += S;
        if (a.mask) acc[2] += __fmul_rn(S, a.mask[p]);
    }
    block_sum_f64<TL_THREADS>(acc, shm);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < TL_MAP_SUMS; ++k) s.map[(size_t)blockIdx.x * TL_MAP_SUMS + k] = acc[k];
        __threadfence();
        last = atomicAdd(s.ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    // final pass: every thread sums a fixed, strided subset of the partials in order, then the fixed block tree
    double tot[TL_PIX_SUMS + TL_MAP_SUMS];
#pragma unroll
    for (int k = 0; k < TL_PIX_SUMS + TL_MAP_SUMS; ++k) tot[k] = 0.0;
    for (int b = threadIdx.x; b < n_pix_ctas; b += TL_THREADS)
#pragma unroll
        for (int k = 0; k < TL_PIX_SUMS; ++k) tot[k] += __ldcg(s.pix + (size_t)b * TL_PIX_SUMS + k);
    for (int b = threadIdx.x; b < (int)gridDim.x; b += TL_THREADS)
#pragma unroll
        for (int k = 0; k < TL_MAP_SUMS; ++k) tot[TL_PIX_SUMS + k] += __ldcg(s.map + (size_t)b * TL_MAP_SUMS + k);
    block_sum_f64<TL_THREADS>(tot, sh);
    if (threadIdx.x != 0) return;
    *s.ticket = 0u;
    // means, the loss and psnr from the double sums, each rounded to fp32 once
    const double n3 = 3.0 * (double)HW, n1 = (double)HW;
    const double mse = tot[2] / n3;
    *a.loss = (float)((double)a.c_l1 * (tot[0] / n3) + (double)a.c_ssim * (tot[TL_PIX_SUMS] / n1));
    float* o = a.metrics;
    o[0] = (float)(tot[1] / n3);                                  // l1_loss
    o[1] = (float)(tot[TL_PIX_SUMS + 1] / n1);                    // ssim
    o[2] = (float)mse;                                            // mse
    o[3] = (float)(-10.0 * log10(mse));                           // psnr (method.py:1970)
    if (a.mask) {
        o[4] = (float)(tot[5] / n1);                              // mask_percentage
        o[5] = (float)(tot[TL_PIX_SUMS + 2] / tot[5]);            // ssim_masked  (_reduce_masked, :1980-1983)
        o[6] = (float)(tot[4] / tot[5]);                          // mse_masked   (3-channel sum / 1-channel sum)
        o[7] = (float)(tot[3] / tot[5]);                          // l1_loss_masked
    } else {
        o[4] = o[5] = o[6] = o[7] = 0.f;
    }
}

__global__ void __launch_bounds__(TL_THREADS) train_loss_bwd_kernel(GsrTrainLossArgs a) {
    const size_t HW = (size_t)a.H * a.W;
    const float g = *a.dL_dloss;
    const float c1 = a.c_l1, c2 = a.c_ssim;
    const float gl = __fdiv_rn(__fmul_rn(g, c1), (float)(3 * HW));
    const float gs = __fdiv_rn(__fmul_rn(g, c2), (float)HW);
    for (size_t p = (size_t)blockIdx.x * TL_THREADS + threadIdx.x; p < HW; p += (size_t)gridDim.x * TL_THREADS) {
        const float m = a.mask ? a.mask[p] : 1.f;
        const float sc = a.grad_scale ? a.grad_scale[p] : 1.f;
        const float w = a.weight ? a.weight[p] : 1.f;
        const float gL = a.weight ? __fmul_rn(gl, w) : gl;
        a.dL_dmap[p] = -(a.weight ? __fmul_rn(gs, w) : gs);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const size_t i = (size_t)c * HW + p;
            float t = a.toned[i];
            if (a.mask) t = scale_grads_value(t, m);
            if (a.grad_scale) t = scale_grads_value(t, sc);
            const float d = __fsub_rn(t, a.gt[i]);
            const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
            float v = __fmul_rn(gL, sgn);
            if (a.grad_scale) v = __fmul_rn(v, sc);
            if (a.mask) v = __fmul_rn(v, m);
            a.d_toned[i] = v;
        }
    }
}

__global__ void __launch_bounds__(TL_THREADS) unpack_u8_kernel(int HW, const unsigned char* __restrict__ img_hwc,
                                                               const unsigned char* __restrict__ mask_hw,
                                                               float* __restrict__ img_chw, float* __restrict__ mask_out) {
    const int p = blockIdx.x * TL_THREADS + threadIdx.x;
    if (p >= HW) return;
    // IEEE division (no fast-math): the bits of numpy's `image.astype(np.float32) / 255.0` (method.py:44-54)
    if (img_hwc) {
#pragma unroll
        for (int c = 0; c < 3; ++c) img_chw[(size_t)c * HW + p] = (float)img_hwc[(size_t)p * 3 + c] / 255.0f;
    }
    if (mask_hw) mask_out[p] = (float)mask_hw[p] / 255.0f;
}

static int tl_check(const GsrTrainLossArgs* a, bool backward) {
    if (!a) { set_error("args is NULL"); return GSR_E_INVALID; }
    if (a->H <= 0 || a->W <= 0 || (long long)a->H * a->W > (1ll << 31) / 3) {
        set_error("bad image size H=%d W=%d", a->H, a->W);
        return GSR_E_INVALID;
    }
    if ((a->H + SSIM_TH - 1) / SSIM_TH > 65535) { set_error("image height too large (H=%d)", a->H); return GSR_E_INVALID; }
    if (!isfinite(a->c_l1) || !isfinite(a->c_ssim)) { set_error("c_l1 or c_ssim is not finite"); return GSR_E_INVALID; }
    if (!a->toned || !a->raw || !a->gt || !a->ssim_map) { set_error("toned, raw, gt or ssim_map is NULL"); return GSR_E_INVALID; }
    if ((a->mask || a->grad_scale) && !a->raw_scaled) {
        set_error("raw_scaled is NULL although a mask or grad_scale is given");
        return GSR_E_INVALID;
    }
    if (!backward && (!a->loss || !a->metrics || !a->scratch)) { set_error("loss, metrics or scratch is NULL"); return GSR_E_INVALID; }
    if (backward && (!a->ssim_partials || !a->dL_dloss || !a->dL_dmap || !a->d_toned || !a->d_raw)) {
        set_error("ssim_partials, dL_dloss, dL_dmap, d_toned or d_raw is NULL");
        return GSR_E_INVALID;
    }
    return 0;
}

}  // namespace gsr

extern "C" size_t gsr_train_loss_scratch_bytes(void) {
    using namespace gsr;
    return (size_t)TL_MAX_CTAS * (TL_PIX_SUMS + TL_MAP_SUMS) * sizeof(double) + 16;
}

extern "C" int gsr_train_loss_forward(const GsrTrainLossArgs* args, void* stream) {
    using namespace gsr;
    if (int rc = tl_check(args, false)) return rc;
    const GsrTrainLossArgs& a = *args;
    cudaStream_t s = (cudaStream_t)stream;
    const long long HW = (long long)a.H * a.W;
    const int n = tl_ctas(HW);
    TlScratch sc = tl_scratch(a.scratch);
    train_loss_pixels_kernel<<<n, TL_THREADS, 0, s>>>(a, sc);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    const float* raw = (a.mask || a.grad_scale) ? a.raw_scaled : a.raw;
    if (int rc = gsr_ssim_forward(1, a.H, a.W, raw, a.gt, a.ssim_map, a.ssim_partials, stream)) return rc;
    train_loss_ssim_kernel<<<n, TL_THREADS, 0, s>>>(a, sc, n);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int gsr_train_loss_backward(const GsrTrainLossArgs* args, void* stream) {
    using namespace gsr;
    if (int rc = tl_check(args, true)) return rc;
    const GsrTrainLossArgs& a = *args;
    cudaStream_t s = (cudaStream_t)stream;
    train_loss_bwd_kernel<<<tl_ctas((long long)a.H * a.W), TL_THREADS, 0, s>>>(a);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    const float* raw = (a.mask || a.grad_scale) ? a.raw_scaled : a.raw;
    return ssim_backward_launch(1, a.H, a.W, raw, a.gt, a.ssim_partials, a.dL_dmap, a.d_raw, a.grad_scale, a.mask, s);
}

extern "C" int gsr_unpack_u8(int H, int W, const unsigned char* img_hwc, const unsigned char* mask_hw, float* img_chw,
                             float* mask_out, void* stream) {
    using namespace gsr;
    if (H <= 0 || W <= 0 || (long long)H * W > (1ll << 31) / 3) { set_error("bad image size H=%d W=%d", H, W); return GSR_E_INVALID; }
    if (!img_hwc && !mask_hw) { set_error("img_hwc and mask_hw are both NULL"); return GSR_E_INVALID; }
    if ((img_hwc && !img_chw) || (mask_hw && !mask_out)) { set_error("an output for a given input is NULL"); return GSR_E_INVALID; }
    const int HW = H * W;
    unpack_u8_kernel<<<(HW + TL_THREADS - 1) / TL_THREADS, TL_THREADS, 0, (cudaStream_t)stream>>>(HW, img_hwc, mask_hw,
                                                                                                  img_chw, mask_out);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}
