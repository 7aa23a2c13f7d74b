// uncertainty.cu -- the head and the `dino`-mode loss of wild-gaussians' uncertainty model, forward and backward.
//
// What it replaces: after the frozen DINOv2 backbone, `UncertaintyModel._forward_uncertainty_features`
// (wildgaussians/method.py:300-323: dropout2d, BatchNorm in training mode, the 1x1 `conv_seg`, softplus, the bilinear
// upsample to the padded image and the crop) and the `dino` branch of `_compute_losses` (:363-433: loss_mult, the
// bilinear downsample to the 350-px map, the cosine map of the two 350-px feature maps, the loss and the seven metric
// scalars).  PyTorch runs that as ~80 launches and seven `.item()` synchronisations per step.
//
// Forward, six launches:
//   1. unc_bn_stats_kernel   (one CTA per channel): batch mean and biased variance of the dropout-scaled features (two
//      passes over the token row), invstd, and the running-statistics update of F.batch_norm in training mode.
//   2. unc_head_kernel       (one thread per token): logits = conv_seg(bn(x)) + log(e - 1), softplus.
//   3. unc_cosine_kernel     (one warp per 350-px token): F.cosine_similarity of the two 350-px feature maps.
//   4. unc_full_kernel       (full resolution): u = max(crop(upsample(softplus)), clip_min), loss_mult = min(1/(2u^2), 3)
//      written out, per-CTA partial sums of log u, loss_mult, ssim * loss_mult, mse * loss_mult, ssim, msssim.
//   5. unc_down_kernel       (350-px map): the downsample of the unclamped 1/(2u^2) (u evaluated at the four taps from the
//      logits), dino_part from the upsampled, cropped cosine map, per-CTA partial sums of dino_part * down(1/(2u^2)).
//   6. unc_finalize_kernel   (one CTA): fixed-order fp64 reduction of all partial sums into the loss and the metrics.
// Backward, three launches:
//   7. unc_bwd_pixel_kernel  (full resolution): dL/du from beta and, through the adjoint of the downsample (a gather over
//      the 350-px rows and columns whose taps include the pixel), from the 350-px term; times the clamp mask.
//   8. unc_bwd_token_kernel  (one thread per token): the adjoint of the crop and the upsample (a gather), times softplus'.
//   9. unc_bwd_param_kernel  (one CTA per channel): sum_t g_t xhat_ct and sum_t g_t, giving dW, db, dgamma, dbeta.
// Every reduction has a fixed order (no floating-point atomics): two runs are bitwise identical.
//
// Resampling restates PyTorch's upsample_bilinear2d with align_corners=False from sizes: scale = in / out in fp32,
// source = max(scale (dst + 0.5) - 0.5, 0), i0 = (int)source, i1 = i0 + (i0 < in - 1), l1 = source - i0, l0 = 1 - l1,
// out = l0y (l0x a + l1x b) + l1y (l0x c + l1x d).  Softplus has beta 1 and threshold 20; the cosine similarity divides
// each vector by max(|v|, 1e-8) before the product, as ATen's cosine_similarity does.
#include "common.cuh"
#include <math.h>

namespace gsr {
namespace {

constexpr int UNC_THREADS = 256;
constexpr int UNC_MAX_C = 2048;                  // 5 C floats of shared memory in the head kernel
constexpr int UNC_MAX_BLOCKS = 2048;             // partial-sum CTAs per map (fixed by the sizes alone)
constexpr int UNC_NFULL = 6;                     // full-resolution partial sums
constexpr float LOG_E_M1 = 0.541324854612918f;   // log(e - 1), method.py:314

struct Lerp { int i0, i1; float l0, l1; };

__device__ __forceinline__ Lerp lerp_at(int in, int out, int dst) {
    const float scale = (float)in / (float)out;
    const float src = fmaxf(scale * ((float)dst + 0.5f) - 0.5f, 0.f);
    Lerp t;
    t.i0 = (int)src;
    t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
    t.l1 = src - (float)t.i0;
    t.l0 = 1.f - t.l1;
    return t;
}

__device__ __forceinline__ float lerp2(const float* __restrict__ p, int w, const Lerp& ty, const Lerp& tx) {
    return ty.l0 * (tx.l0 * p[(size_t)ty.i0 * w + tx.i0] + tx.l1 * p[(size_t)ty.i0 * w + tx.i1]) +
           ty.l1 * (tx.l0 * p[(size_t)ty.i1 * w + tx.i0] + tx.l1 * p[(size_t)ty.i1 * w + tx.i1]);
}

// The weight with which output index `dst` of a resize in -> out reads input index `src` (0 when it does not).
__device__ __forceinline__ float tap_weight(int in, int out, int dst, int src) {
    const Lerp t = lerp_at(in, out, dst);
    return (t.i0 == src ? t.l0 : 0.f) + (t.i1 == src ? t.l1 : 0.f);
}

// Output indices of a resize in -> out whose taps may include input index `src` (a superset; tap_weight decides).
__device__ __forceinline__ void taps_of(int in, int out, int src, int& lo, int& hi) {
    const float inv = (float)out / (float)in;
    lo = max(0, (int)floorf(((float)src - 0.5f) * inv - 0.5f) - 1);
    hi = min(out - 1, (int)ceilf(((float)src + 1.5f) * inv - 0.5f) + 1);
}

__device__ __forceinline__ float softplus20(float x) { return x > 20.f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float clamp_min_nan(float v, float lo) { return v < lo ? lo : v; }   // NaN propagates
__device__ __forceinline__ float clamp_max_nan(float v, float hi) { return v > hi ? hi : v; }

// Deterministic CTA sum (fixed tree); every thread gets the result.
template <typename T>
__device__ T block_sum(T v, T* sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int s = UNC_THREADS / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
        __syncthreads();
    }
    const T r = sh[0];
    __syncthreads();
    return r;
}

struct Scratch {
    float *mean, *invstd, *logit, *sp, *cosine, *dpart, *pfull, *pdown, *dv, *dlogit;
};

int full_blocks(const GsrUncertaintyArgs& a) {
    const long long n = (long long)a.H * a.W, b = (n + UNC_THREADS - 1) / UNC_THREADS;
    return (int)(b < UNC_MAX_BLOCKS ? b : UNC_MAX_BLOCKS);
}
int down_blocks(const GsrUncertaintyArgs& a) {
    const long long n = (long long)a.nh * a.nw, b = (n + UNC_THREADS - 1) / UNC_THREADS;
    return (int)(b < UNC_MAX_BLOCKS ? b : UNC_MAX_BLOCKS);
}
size_t pad64(size_t floats) { return (floats + 63) / 64 * 64; }

size_t layout(const GsrUncertaintyArgs& a, Scratch* s) {
    const size_t T = (size_t)a.th * a.tw;
    const size_t sizes[10] = {(size_t)a.C, (size_t)a.C, T, T, (size_t)a.ch * a.cw, (size_t)a.nh * a.nw,
                              (size_t)UNC_NFULL * full_blocks(a), (size_t)down_blocks(a), (size_t)a.H * a.W, T};
    size_t off = 0;
    float** dst[10] = {&s->mean, &s->invstd, &s->logit, &s->sp, &s->cosine, &s->dpart, &s->pfull, &s->pdown, &s->dv,
                       &s->dlogit};
    for (int i = 0; i < 10; ++i) {
        *dst[i] = a.scratch ? (float*)a.scratch + off : nullptr;
        off += pad64(sizes[i]);
    }
    return off * sizeof(float);
}

// ---------------------------------------------------------------------------------------------------------- forward

__global__ void __launch_bounds__(UNC_THREADS) unc_bn_stats_kernel(int T, const float* __restrict__ feat,
                                                                   const float* __restrict__ mask, float eps, float momentum,
                                                                   float* __restrict__ mean_out, float* __restrict__ invstd_out,
                                                                   float* __restrict__ running_mean,
                                                                   float* __restrict__ running_var,
                                                                   long long* __restrict__ num_batches_tracked) {
    __shared__ float sh[UNC_THREADS];
    const int c = blockIdx.x;
    const float* x = feat + (size_t)c * T;
    const float m = mask[c];
    float s = 0.f;
    for (int t = threadIdx.x; t < T; t += UNC_THREADS) s += x[t] * m;
    const float mean = block_sum(s, sh) / (float)T;
    float q = 0.f;
    for (int t = threadIdx.x; t < T; t += UNC_THREADS) {
        const float d = x[t] * m - mean;
        q += d * d;
    }
    const float m2 = block_sum(q, sh);
    if (threadIdx.x == 0) {
        mean_out[c] = mean;
        invstd_out[c] = 1.f / sqrtf(m2 / (float)T + eps);
        if (running_mean) running_mean[c] = momentum * mean + (1.f - momentum) * running_mean[c];
        if (running_var) running_var[c] = momentum * (m2 / (float)(T - 1)) + (1.f - momentum) * running_var[c];
        if (num_batches_tracked && c == 0) *num_batches_tracked += 1;
    }
}

// Per token: sum_c W_c ((x_ct m_c - mean_c) invstd_c gamma_c + beta_c) + b + log(e - 1), then softplus.
__global__ void __launch_bounds__(UNC_THREADS) unc_head_kernel(int C, int T, const float* __restrict__ feat,
                                                               const float* __restrict__ mask, const float* __restrict__ mean,
                                                               const float* __restrict__ invstd, const float* __restrict__ w,
                                                               const float* __restrict__ b, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, float* __restrict__ logit,
                                                               float* __restrict__ sp) {
    extern __shared__ float prm[];                 // [5][C]: mask, mean, invstd * gamma, beta, W
    for (int c = threadIdx.x; c < C; c += UNC_THREADS) {
        prm[c] = mask[c];
        prm[C + c] = mean[c];
        prm[2 * C + c] = invstd[c] * gamma[c];
        prm[3 * C + c] = beta[c];
        prm[4 * C + c] = w[c];
    }
    __syncthreads();
    const int t = blockIdx.x * UNC_THREADS + threadIdx.x;
    if (t >= T) return;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};           // four interleaved chains: a shorter rounding path than one
    int c = 0;
    for (; c + 4 <= C; c += 4) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int j = c + k;
            const float y = (feat[(size_t)j * T + t] * prm[j] - prm[C + j]) * prm[2 * C + j] + prm[3 * C + j];
            acc[k] += prm[4 * C + j] * y;
        }
    }
    for (; c < C; ++c) {
        const float y = (feat[(size_t)c * T + t] * prm[c] - prm[C + c]) * prm[2 * C + c] + prm[3 * C + c];
        acc[0] += prm[4 * C + c] * y;
    }
    const float l = ((acc[0] + acc[1]) + (acc[2] + acc[3]) + b[0]) + LOG_E_M1;
    logit[t] = l;
    sp[t] = softplus20(l);
}

// One warp per token of the 350-px grid: sum_c (x_c / max(|x|, eps)) (y_c / max(|y|, eps)).
__global__ void __launch_bounds__(UNC_THREADS) unc_cosine_kernel(int C, int T, const float* __restrict__ fx,
                                                                 const float* __restrict__ fy, float* __restrict__ cosine) {
    const int t = blockIdx.x * (UNC_THREADS / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (t >= T) return;
    float xx = 0.f, yy = 0.f;
    for (int c = lane; c < C; c += 32) {
        const float x = fx[(size_t)c * T + t], y = fy[(size_t)c * T + t];
        xx += x * x;
        yy += y * y;
    }
    for (int o = 16; o > 0; o >>= 1) {
        xx += __shfl_xor_sync(0xffffffffu, xx, o);
        yy += __shfl_xor_sync(0xffffffffu, yy, o);
    }
    const float nx = fmaxf(sqrtf(xx), 1e-8f), ny = fmaxf(sqrtf(yy), 1e-8f);
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += (fx[(size_t)c * T + t] / nx) * (fy[(size_t)c * T + t] / ny);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) cosine[t] = s;
}

// u at image pixel (y, x): the softplus map upsampled to the padded size, cropped, clamped below.  `v` is the unclamped value.
__device__ __forceinline__ float u_at(const GsrUncertaintyArgs& a, const float* __restrict__ sp, int y, int x, float& v) {
    v = lerp2(sp, a.tw, lerp_at(a.th, a.Hp, y + a.pad_top), lerp_at(a.tw, a.Wp, x + a.pad_left));
    return clamp_min_nan(v, a.clip_min);
}

__device__ __forceinline__ float inv2sq(float u) { return 1.f / (2.f * (u * u)); }

__global__ void __launch_bounds__(UNC_THREADS) unc_full_kernel(const GsrUncertaintyArgs a, const float* __restrict__ sp,
                                                               float* __restrict__ partials) {
    __shared__ float sh[UNC_THREADS];
    const size_t HW = (size_t)a.H * a.W;
    float acc[UNC_NFULL] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (size_t p = blockIdx.x * (size_t)UNC_THREADS + threadIdx.x; p < HW; p += (size_t)gridDim.x * UNC_THREADS) {
        const int y = (int)(p / a.W), x = (int)(p - (size_t)y * a.W);
        float v;
        const float u = u_at(a, sp, y, x, v);
        const float lm = clamp_max_nan(inv2sq(u), 3.f);
        a.loss_mult[p] = lm;
        const float d0 = a.gt[p] - a.pred[p], d1 = a.gt[HW + p] - a.pred[HW + p], d2 = a.gt[2 * HW + p] - a.pred[2 * HW + p];
        const float s = a.ssim[p];
        acc[0] += logf(u);
        acc[1] += lm;
        acc[2] += s * lm;
        acc[3] += ((d0 * d0) * lm + (d1 * d1) * lm) + (d2 * d2) * lm;
        acc[4] += s;
        acc[5] += a.msssim[p];
    }
#pragma unroll
    for (int k = 0; k < UNC_NFULL; ++k) {
        const float r = block_sum(acc[k], sh);
        if (threadIdx.x == 0) partials[(size_t)k * gridDim.x + blockIdx.x] = r;
    }
}

__global__ void __launch_bounds__(UNC_THREADS) unc_down_kernel(const GsrUncertaintyArgs a, const float* __restrict__ sp,
                                                               const float* __restrict__ cosine, float* __restrict__ dpart,
                                                               float* __restrict__ partials) {
    __shared__ float sh[UNC_THREADS];
    const size_t n = (size_t)a.nh * a.nw;
    float acc = 0.f;
    for (size_t q = blockIdx.x * (size_t)UNC_THREADS + threadIdx.x; q < n; q += (size_t)gridDim.x * UNC_THREADS) {
        const int qy = (int)(q / a.nw), qx = (int)(q - (size_t)qy * a.nw);
        const Lerp ty = lerp_at(a.H, a.nh, qy), tx = lerp_at(a.W, a.nw, qx);
        float v;
        const float m00 = inv2sq(u_at(a, sp, ty.i0, tx.i0, v)), m01 = inv2sq(u_at(a, sp, ty.i0, tx.i1, v));
        const float m10 = inv2sq(u_at(a, sp, ty.i1, tx.i0, v)), m11 = inv2sq(u_at(a, sp, ty.i1, tx.i1, v));
        const float down = ty.l0 * (tx.l0 * m00 + tx.l1 * m01) + ty.l1 * (tx.l0 * m10 + tx.l1 * m11);
        const float cs = lerp2(cosine, a.cw, lerp_at(a.ch, a.nHp, qy + a.npad_top), lerp_at(a.cw, a.nWp, qx + a.npad_left));
        float part = 1.f - (cs - 0.5f) / 0.5f;
        part = part < 0.f ? 0.f : (part > 1.f ? 1.f : part);
        dpart[q] = part;
        acc += part * down;
    }
    const float r = block_sum(acc, sh);
    if (threadIdx.x == 0) partials[blockIdx.x] = r;
}

// metrics: loss, ssim, msssim, ssim_discounted, mse_discounted, psnr_discounted, beta (method.py:424-432)
__global__ void __launch_bounds__(UNC_THREADS) unc_finalize_kernel(const GsrUncertaintyArgs a, int nbf, int nbd,
                                                                   const float* __restrict__ pfull,
                                                                   const float* __restrict__ pdown) {
    __shared__ double sh[UNC_THREADS];
    double tot[UNC_NFULL + 1];
#pragma unroll
    for (int k = 0; k <= UNC_NFULL; ++k) {
        const int nb = k < UNC_NFULL ? nbf : nbd;
        const float* p = k < UNC_NFULL ? pfull + (size_t)k * nbf : pdown;
        double s = 0.0;
        for (int i = threadIdx.x; i < nb; i += UNC_THREADS) s += (double)p[i];
        tot[k] = block_sum(s, sh);
    }
    if (threadIdx.x == 0) {
        const double HW = (double)a.H * a.W;
        const float beta = (float)(tot[0] / HW);
        const float loss = (float)(tot[UNC_NFULL] / ((double)a.nh * a.nw) + (double)a.reg_weight * (double)beta);
        const double mse = (double)(float)(tot[3] / tot[1]);
        a.loss[0] = loss;
        a.metrics[0] = loss;
        a.metrics[1] = (float)(tot[4] / HW);
        a.metrics[2] = (float)(tot[5] / HW);
        a.metrics[3] = (float)(tot[2] / tot[1]);
        a.metrics[4] = (float)mse;
        a.metrics[5] = (float)(10.0 * log10(1.0 / mse));
        a.metrics[6] = beta;
    }
}

// --------------------------------------------------------------------------------------------------------- backward

__global__ void __launch_bounds__(UNC_THREADS) unc_bwd_pixel_kernel(const GsrUncertaintyArgs a, const float* __restrict__ sp,
                                                                    const float* __restrict__ dpart, float* __restrict__ dv) {
    const size_t HW = (size_t)a.H * a.W;
    const float g = a.dL_dloss[0];
    const float g_beta = g * a.reg_weight / (float)HW;
    const float g_down = g / (float)((size_t)a.nh * a.nw);
    for (size_t p = blockIdx.x * (size_t)UNC_THREADS + threadIdx.x; p < HW; p += (size_t)gridDim.x * UNC_THREADS) {
        const int y = (int)(p / a.W), x = (int)(p - (size_t)y * a.W);
        float v;
        const float u = u_at(a, sp, y, x, v);
        int ylo, yhi, xlo, xhi;
        taps_of(a.H, a.nh, y, ylo, yhi);
        taps_of(a.W, a.nw, x, xlo, xhi);
        float dlm = 0.f;
        for (int qy = ylo; qy <= yhi; ++qy) {
            const float wy = tap_weight(a.H, a.nh, qy, y);
            if (wy == 0.f) continue;
            float row = 0.f;
            for (int qx = xlo; qx <= xhi; ++qx) {
                const float wx = tap_weight(a.W, a.nw, qx, x);
                if (wx != 0.f) row += wx * dpart[(size_t)qy * a.nw + qx];
            }
            dlm += wy * row;
        }
        const float du = g_beta / u - (g_down * dlm) / (u * (u * u));
        dv[p] = v >= a.clip_min ? du : 0.f;
    }
}

__global__ void __launch_bounds__(UNC_THREADS) unc_bwd_token_kernel(const GsrUncertaintyArgs a, const float* __restrict__ logit,
                                                                    const float* __restrict__ dv, float* __restrict__ dlogit) {
    const int T = a.th * a.tw;
    const int t = blockIdx.x * UNC_THREADS + threadIdx.x;
    if (t >= T) return;
    const int ty = t / a.tw, tx = t - ty * a.tw;
    int rlo, rhi, clo, chi;
    taps_of(a.th, a.Hp, ty, rlo, rhi);
    taps_of(a.tw, a.Wp, tx, clo, chi);
    rlo = max(rlo, a.pad_top); rhi = min(rhi, a.pad_top + a.H - 1);        // the crop: only image pixels carry gradient
    clo = max(clo, a.pad_left); chi = min(chi, a.pad_left + a.W - 1);
    float acc = 0.f;
    for (int r = rlo; r <= rhi; ++r) {
        const float wy = tap_weight(a.th, a.Hp, r, ty);
        if (wy == 0.f) continue;
        const float* row = dv + (size_t)(r - a.pad_top) * a.W - a.pad_left;
        float s = 0.f;
        for (int c = clo; c <= chi; ++c) {
            const float wx = tap_weight(a.tw, a.Wp, c, tx);
            if (wx != 0.f) s += wx * row[c];
        }
        acc += wy * s;
    }
    const float l = logit[t];
    const float z = expf(l);
    dlogit[t] = l > 20.f ? acc : acc * z / (z + 1.f);
}

__global__ void __launch_bounds__(UNC_THREADS) unc_bwd_param_kernel(const GsrUncertaintyArgs a, const float* __restrict__ mean,
                                                                    const float* __restrict__ invstd,
                                                                    const float* __restrict__ dlogit) {
    __shared__ float sh[UNC_THREADS];
    const int c = blockIdx.x, T = a.th * a.tw;
    const float* x = a.feat + (size_t)c * T;
    const float m = a.mask[c], mu = mean[c], is = invstd[c];
    float sx = 0.f, sg = 0.f;
    for (int t = threadIdx.x; t < T; t += UNC_THREADS) {
        const float g = dlogit[t];
        sx += g * ((x[t] * m - mu) * is);
        sg += g;
    }
    const float Sx = block_sum(sx, sh), G = block_sum(sg, sh);
    if (threadIdx.x == 0) {
        const float w = a.conv_w[c];
        a.d_conv_w[c] = a.bn_w[c] * Sx + a.bn_b[c] * G;
        a.d_bn_w[c] = w * Sx;
        a.d_bn_b[c] = w * G;
        if (c == 0) a.d_conv_b[0] = G;
    }
}

int check_args(const GsrUncertaintyArgs* a, bool backward) {
    if (!a) { set_error("args is NULL"); return GSR_E_INVALID; }
    if (a->C <= 0 || a->C > UNC_MAX_C) { set_error("bad channel count C=%d (1..%d)", a->C, UNC_MAX_C); return GSR_E_INVALID; }
    const int dims[14] = {a->th, a->tw, a->Hp, a->Wp, a->H, a->W, a->nh, a->nw, a->ch, a->cw, a->nHp, a->nWp, 1, 1};
    for (int d : dims)
        if (d <= 0) { set_error("bad sizes: every size must be positive"); return GSR_E_INVALID; }
    if ((long long)a->th * a->tw < 2) { set_error("bad sizes: batch statistics need more than one token"); return GSR_E_INVALID; }
    if (a->th > a->Hp || a->tw > a->Wp || a->ch > a->nHp || a->cw > a->nWp) {
        set_error("bad sizes: a token grid is larger than its padded image");
        return GSR_E_INVALID;
    }
    if (a->pad_top < 0 || a->pad_left < 0 || a->pad_top + a->H > a->Hp || a->pad_left + a->W > a->Wp ||
        a->npad_top < 0 || a->npad_left < 0 || a->npad_top + a->nh > a->nHp || a->npad_left + a->nw > a->nWp) {
        set_error("bad sizes: the crop does not fit in the padded image");
        return GSR_E_INVALID;
    }
    if ((long long)a->Hp * a->Wp >= (1ll << 31) || (long long)a->nHp * a->nWp >= (1ll << 31)) {
        set_error("image too large");
        return GSR_E_INVALID;
    }
    if (!(a->clip_min > 0.f)) { set_error("clip_min must be positive"); return GSR_E_INVALID; }
    if (!a->feat || !a->feat_gt_down || !a->feat_pred_down || !a->mask || !a->conv_w || !a->conv_b || !a->bn_w || !a->bn_b ||
        !a->gt || !a->pred || !a->ssim || !a->msssim || !a->loss_mult || !a->loss || !a->metrics || !a->scratch) {
        set_error("a required pointer is NULL");
        return GSR_E_INVALID;
    }
    if (backward && (!a->dL_dloss || !a->d_conv_w || !a->d_conv_b || !a->d_bn_w || !a->d_bn_b)) {
        set_error("a gradient pointer is NULL");
        return GSR_E_INVALID;
    }
    return 0;
}

unsigned blocks_for(long long n) { return (unsigned)((n + UNC_THREADS - 1) / UNC_THREADS); }

// ------------------------------------------------------------------------- every mode, both BatchNorm modes, a cap
// gsr_uncertainty_mode_*: the head runs on the (possibly capped) head input of size uh x uw; H x W is the image.  The
// BatchNorm statistics, the cosine map and the backward's parameter kernel are the kernels above, the last called with
// a GsrUncertaintyArgs that views the head input as the image (head_view).
// Forward: unc_bn_stats_kernel (training) or unc_bn_eval_kernel (eval), unc_mode_head_kernel, [unc_cosine_kernel],
// unc_mode_full_kernel, [unc_mode_down_kernel], unc_mode_finalize_kernel; [..] for dino / dino+mssim only.
// Backward: [unc_mode_bwd_full_kernel] (l2reg / l1reg only), unc_mode_bwd_pixel_kernel, unc_mode_bwd_token_kernel,
// unc_bwd_param_kernel.

constexpr int UNC_NMODE = 7;                     // partial sums: log u (head input), then six at full resolution

__host__ __device__ __forceinline__ bool dino_mode(int mode) {
    return mode == GSR_UNC_MODE_DINO || mode == GSR_UNC_MODE_DINO_MSSIM;
}

struct ModeScratch {
    float *mean, *invstd, *ones, *logit, *sp, *cosine, *dpart, *pfull, *pdown, *dv, *dfull, *dlogit;
};

int mode_full_blocks(const GsrUncertaintyModeArgs& a) {
    const long long n = (long long)a.H * a.W, b = (n + UNC_THREADS - 1) / UNC_THREADS;
    return (int)(b < UNC_MAX_BLOCKS ? b : UNC_MAX_BLOCKS);
}
int mode_down_blocks(const GsrUncertaintyModeArgs& a) {
    if (!dino_mode(a.mode)) return 0;
    const long long n = (long long)a.nh * a.nw, b = (n + UNC_THREADS - 1) / UNC_THREADS;
    return (int)(b < UNC_MAX_BLOCKS ? b : UNC_MAX_BLOCKS);
}

size_t mode_layout(const GsrUncertaintyModeArgs& a, ModeScratch* s) {
    const size_t T = (size_t)a.th * a.tw, C = (size_t)a.C;
    const bool dino = dino_mode(a.mode);
    const size_t sizes[12] = {C, C, C, T, T, dino ? (size_t)a.ch * a.cw : 0, dino ? (size_t)a.nh * a.nw : 0,
                              (size_t)UNC_NMODE * mode_full_blocks(a), (size_t)mode_down_blocks(a), (size_t)a.uh * a.uw,
                              dino ? 0 : (size_t)a.H * a.W, T};
    float** dst[12] = {&s->mean, &s->invstd, &s->ones, &s->logit, &s->sp, &s->cosine, &s->dpart, &s->pfull, &s->pdown,
                       &s->dv, &s->dfull, &s->dlogit};
    size_t off = 0;
    for (int i = 0; i < 12; ++i) {
        *dst[i] = a.scratch ? (float*)a.scratch + off : nullptr;
        off += pad64(sizes[i]);
    }
    return off * sizeof(float);
}

// The head input seen as the image of GsrUncertaintyArgs: what unc_bwd_param_kernel reads.
GsrUncertaintyArgs head_view(const GsrUncertaintyModeArgs& a, const ModeScratch& s) {
    GsrUncertaintyArgs h = {};
    h.C = a.C; h.th = a.th; h.tw = a.tw; h.Hp = a.Hp; h.Wp = a.Wp; h.pad_top = a.pad_top; h.pad_left = a.pad_left;
    h.H = a.uh; h.W = a.uw;
    h.feat = a.feat; h.mask = a.training ? a.mask : s.ones;
    h.conv_w = a.conv_w; h.conv_b = a.conv_b; h.bn_w = a.bn_w; h.bn_b = a.bn_b;
    h.dL_dloss = a.dL_dloss; h.d_conv_w = a.d_conv_w; h.d_conv_b = a.d_conv_b; h.d_bn_w = a.d_bn_w; h.d_bn_b = a.d_bn_b;
    return h;
}

// F.batch_norm in evaluation mode: the running statistics, no update; the channel scales are all ones.
__global__ void __launch_bounds__(UNC_THREADS) unc_bn_eval_kernel(int C, const float* __restrict__ running_mean,
                                                                  const float* __restrict__ running_var, float eps,
                                                                  float* __restrict__ mean_out, float* __restrict__ invstd_out,
                                                                  float* __restrict__ ones) {
    const int c = blockIdx.x * UNC_THREADS + threadIdx.x;
    if (c >= C) return;
    mean_out[c] = running_mean[c];
    invstd_out[c] = 1.f / sqrtf(running_var[c] + eps);
    ones[c] = 1.f;
}

// unc_head_kernel with BatchNorm's output and the conv_seg sum over channels in double, rounded once to the logit.  In
// evaluation mode the running statistics need not match the features, so BatchNorm's outputs can be large and the
// channel sum cancel; the fp32 sum of unc_head_kernel then loses more than the reference's own fp32 statements do.
__global__ void __launch_bounds__(UNC_THREADS) unc_mode_head_kernel(int C, int T, const float* __restrict__ feat,
                                                                    const float* __restrict__ mask,
                                                                    const float* __restrict__ mean,
                                                                    const float* __restrict__ invstd,
                                                                    const float* __restrict__ w, const float* __restrict__ b,
                                                                    const float* __restrict__ gamma,
                                                                    const float* __restrict__ beta,
                                                                    float* __restrict__ logit, float* __restrict__ sp) {
    extern __shared__ float prm[];                 // [5][C]: mask, mean, invstd, gamma, beta; W read from global
    for (int c = threadIdx.x; c < C; c += UNC_THREADS) {
        prm[c] = mask[c];
        prm[C + c] = mean[c];
        prm[2 * C + c] = invstd[c];
        prm[3 * C + c] = gamma[c];
        prm[4 * C + c] = beta[c];
    }
    __syncthreads();
    const int t = blockIdx.x * UNC_THREADS + threadIdx.x;
    if (t >= T) return;
    double acc = 0.0;
    for (int c = 0; c < C; ++c) {
        const double y = ((double)feat[(size_t)c * T + t] * (double)prm[c] - (double)prm[C + c]) * (double)prm[2 * C + c] *
                         (double)prm[3 * C + c] + (double)prm[4 * C + c];
        acc += (double)__ldg(w + c) * y;
    }
    const float l = (float)(acc + (double)b[0] + 0.5413248546129181);      // log(e - 1)
    logit[t] = l;
    sp[t] = softplus20(l);
}

// u at head-input pixel (y, x) (clamped below; `v` unclamped).
__device__ __forceinline__ float u_head(const GsrUncertaintyModeArgs& a, const float* __restrict__ sp, int y, int x, float& v) {
    v = lerp2(sp, a.tw, lerp_at(a.th, a.Hp, y + a.pad_top), lerp_at(a.tw, a.Wp, x + a.pad_left));
    return clamp_min_nan(v, a.clip_min);
}

__device__ __forceinline__ float mult_of(int mode, float u) { return mode == GSR_UNC_MODE_L1REG ? 1.f / u : inv2sq(u); }

// The branch's full-resolution loss_mult at image pixel (y, x): l2reg / l1reg take it of the resized u (`uf`), the dino
// modes resize the head input's loss_mult and clamp it at 3 (uf is then not used).
__device__ __forceinline__ float full_mult(const GsrUncertaintyModeArgs& a, const float* __restrict__ sp, int y, int x,
                                           float& uf) {
    const bool dino = dino_mode(a.mode);
    float lm, v;
    if (a.uh == a.H && a.uw == a.W) {
        uf = u_head(a, sp, y, x, v);
        lm = mult_of(a.mode, uf);
    } else {
        const Lerp ty = lerp_at(a.uh, a.H, y), tx = lerp_at(a.uw, a.W, x);
        float q00 = u_head(a, sp, ty.i0, tx.i0, v), q01 = u_head(a, sp, ty.i0, tx.i1, v);
        float q10 = u_head(a, sp, ty.i1, tx.i0, v), q11 = u_head(a, sp, ty.i1, tx.i1, v);
        if (dino) { q00 = inv2sq(q00); q01 = inv2sq(q01); q10 = inv2sq(q10); q11 = inv2sq(q11); }
        const float r = ty.l0 * (tx.l0 * q00 + tx.l1 * q01) + ty.l1 * (tx.l0 * q10 + tx.l1 * q11);
        uf = r;
        lm = dino ? r : mult_of(a.mode, r);
    }
    return dino ? clamp_max_nan(lm, 3.f) : lm;
}

// Partials: [0] log u over the head input; over the image [1] loss_mult, [2] ssim loss_mult, [3] mse loss_mult,
// [4] ssim, [5] msssim, [6] (1 - msssim) loss_mult (the l2reg / l1reg loss).
__global__ void __launch_bounds__(UNC_THREADS) unc_mode_full_kernel(const GsrUncertaintyModeArgs a,
                                                                    const float* __restrict__ sp,
                                                                    float* __restrict__ partials) {
    __shared__ float sh[UNC_THREADS];
    const size_t stride = (size_t)gridDim.x * UNC_THREADS, first = blockIdx.x * (size_t)UNC_THREADS + threadIdx.x;
    float acc[UNC_NMODE] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const size_t UHW = (size_t)a.uh * a.uw;
    for (size_t p = first; p < UHW; p += stride) {
        const int y = (int)(p / a.uw), x = (int)(p - (size_t)y * a.uw);
        float v;
        acc[0] += logf(u_head(a, sp, y, x, v));
    }
    const size_t HW = (size_t)a.H * a.W;
    for (size_t p = first; p < HW; p += stride) {
        const int y = (int)(p / a.W), x = (int)(p - (size_t)y * a.W);
        float uf;
        const float lm = full_mult(a, sp, y, x, uf);
        a.loss_mult[p] = lm;
        const float d0 = a.gt[p] - a.pred[p], d1 = a.gt[HW + p] - a.pred[HW + p], d2 = a.gt[2 * HW + p] - a.pred[2 * HW + p];
        const float s = a.ssim[p], ms = a.msssim[p];
        acc[1] += lm;
        acc[2] += s * lm;
        acc[3] += ((d0 * d0) * lm + (d1 * d1) * lm) + (d2 * d2) * lm;
        acc[4] += s;
        acc[5] += ms;
        acc[6] += (1.f - ms) * lm;
    }
#pragma unroll
    for (int k = 0; k < UNC_NMODE; ++k) {
        const float r = block_sum(acc[k], sh);
        if (threadIdx.x == 0) partials[(size_t)k * gridDim.x + blockIdx.x] = r;
    }
}

__device__ __forceinline__ float min_nan(float x, float y) { return (x < y || x != x) ? x : y; }   // torch.min

// The 350-px map: the resize of the head input's 1 / (2 u^2) times the dino part (dino+mssim: the smaller of it and
// 1 - msssim_down).
__global__ void __launch_bounds__(UNC_THREADS) unc_mode_down_kernel(const GsrUncertaintyModeArgs a,
                                                                    const float* __restrict__ sp,
                                                                    const float* __restrict__ cosine,
                                                                    float* __restrict__ dpart, float* __restrict__ partials) {
    __shared__ float sh[UNC_THREADS];
    const size_t n = (size_t)a.nh * a.nw;
    float acc = 0.f;
    for (size_t q = blockIdx.x * (size_t)UNC_THREADS + threadIdx.x; q < n; q += (size_t)gridDim.x * UNC_THREADS) {
        const int qy = (int)(q / a.nw), qx = (int)(q - (size_t)qy * a.nw);
        const Lerp ty = lerp_at(a.uh, a.nh, qy), tx = lerp_at(a.uw, a.nw, qx);
        float v;
        const float m00 = inv2sq(u_head(a, sp, ty.i0, tx.i0, v)), m01 = inv2sq(u_head(a, sp, ty.i0, tx.i1, v));
        const float m10 = inv2sq(u_head(a, sp, ty.i1, tx.i0, v)), m11 = inv2sq(u_head(a, sp, ty.i1, tx.i1, v));
        const float down = ty.l0 * (tx.l0 * m00 + tx.l1 * m01) + ty.l1 * (tx.l0 * m10 + tx.l1 * m11);
        const float cs = lerp2(cosine, a.cw, lerp_at(a.ch, a.nHp, qy + a.npad_top), lerp_at(a.cw, a.nWp, qx + a.npad_left));
        float part = 1.f - (cs - 0.5f) / 0.5f;
        part = part < 0.f ? 0.f : (part > 1.f ? 1.f : part);
        if (a.mode == GSR_UNC_MODE_DINO_MSSIM) part = min_nan(part, 1.f - a.msssim_down[q]);
        dpart[q] = part;
        acc += part * down;
    }
    const float r = block_sum(acc, sh);
    if (threadIdx.x == 0) partials[blockIdx.x] = r;
}

__global__ void __launch_bounds__(UNC_THREADS) unc_mode_finalize_kernel(const GsrUncertaintyModeArgs a, int nbf, int nbd,
                                                                        const float* __restrict__ pfull,
                                                                        const float* __restrict__ pdown) {
    __shared__ double sh[UNC_THREADS];
    double tot[UNC_NMODE + 1];
#pragma unroll
    for (int k = 0; k <= UNC_NMODE; ++k) {
        const int nb = k < UNC_NMODE ? nbf : nbd;
        const float* p = k < UNC_NMODE ? pfull + (size_t)k * nbf : pdown;
        double s = 0.0;
        for (int i = threadIdx.x; i < nb; i += UNC_THREADS) s += (double)p[i];
        tot[k] = block_sum(s, sh);
    }
    if (threadIdx.x == 0) {
        const double HW = (double)a.H * a.W;
        const float beta = (float)(tot[0] / ((double)a.uh * a.uw));
        const double mean_loss = dino_mode(a.mode) ? tot[UNC_NMODE] / ((double)a.nh * a.nw) : tot[6] / HW;
        const float loss = (float)(mean_loss + (double)a.reg_weight * (double)beta);
        const double mse = (double)(float)(tot[3] / tot[1]);
        a.loss[0] = loss;
        a.metrics[0] = loss;
        a.metrics[1] = (float)(tot[4] / HW);
        a.metrics[2] = (float)(tot[5] / HW);
        a.metrics[3] = (float)(tot[2] / tot[1]);
        a.metrics[4] = (float)mse;
        a.metrics[5] = (float)(10.0 * log10(1.0 / mse));
        a.metrics[6] = beta;
    }
}

// l2reg / l1reg: dL/du of the resized u at every image pixel, g (1 - msssim) / (H W) dloss_mult/du.
__global__ void __launch_bounds__(UNC_THREADS) unc_mode_bwd_full_kernel(const GsrUncertaintyModeArgs a,
                                                                        const float* __restrict__ sp,
                                                                        float* __restrict__ dfull) {
    const size_t HW = (size_t)a.H * a.W;
    const float g = a.dL_dloss[0] / (float)HW;
    for (size_t p = blockIdx.x * (size_t)UNC_THREADS + threadIdx.x; p < HW; p += (size_t)gridDim.x * UNC_THREADS) {
        const int y = (int)(p / a.W), x = (int)(p - (size_t)y * a.W);
        float u;
        full_mult(a, sp, y, x, u);
        const float dm = a.mode == GSR_UNC_MODE_L1REG ? -1.f / (u * u) : -1.f / (u * (u * u));
        dfull[p] = (g * (1.f - a.msssim[p])) * dm;
    }
}

// sum over the outputs o of a resize in_h x in_w -> out_h x out_w of weight(o, (y, x)) src[o]: the resize's adjoint.
__device__ __forceinline__ float resize_adjoint(int in_h, int in_w, int out_h, int out_w, int y, int x,
                                                const float* __restrict__ src) {
    int ylo, yhi, xlo, xhi;
    taps_of(in_h, out_h, y, ylo, yhi);
    taps_of(in_w, out_w, x, xlo, xhi);
    float acc = 0.f;
    for (int qy = ylo; qy <= yhi; ++qy) {
        const float wy = tap_weight(in_h, out_h, qy, y);
        if (wy == 0.f) continue;
        float row = 0.f;
        for (int qx = xlo; qx <= xhi; ++qx) {
            const float wx = tap_weight(in_w, out_w, qx, x);
            if (wx != 0.f) row += wx * src[(size_t)qy * out_w + qx];
        }
        acc += wy * row;
    }
    return acc;
}

// dL/dv at every head-input pixel (v: u before the clamp): beta's term plus the loss term through its resize's adjoint.
__global__ void __launch_bounds__(UNC_THREADS) unc_mode_bwd_pixel_kernel(const GsrUncertaintyModeArgs a,
                                                                         const float* __restrict__ sp,
                                                                         const float* __restrict__ dpart,
                                                                         const float* __restrict__ dfull,
                                                                         float* __restrict__ dv) {
    const size_t UHW = (size_t)a.uh * a.uw;
    const float g = a.dL_dloss[0];
    const float g_beta = g * a.reg_weight / (float)UHW;
    const bool dino = dino_mode(a.mode), same = a.uh == a.H && a.uw == a.W;
    const float g_down = dino ? g / (float)((size_t)a.nh * a.nw) : 0.f;
    for (size_t p = blockIdx.x * (size_t)UNC_THREADS + threadIdx.x; p < UHW; p += (size_t)gridDim.x * UNC_THREADS) {
        const int y = (int)(p / a.uw), x = (int)(p - (size_t)y * a.uw);
        float v;
        const float u = u_head(a, sp, y, x, v);
        float du;
        if (dino) {
            const float dlm = resize_adjoint(a.uh, a.uw, a.nh, a.nw, y, x, dpart);
            du = g_beta / u - (g_down * dlm) / (u * (u * u));
        } else {
            du = g_beta / u + (same ? dfull[p] : resize_adjoint(a.uh, a.uw, a.H, a.W, y, x, dfull));
        }
        dv[p] = v >= a.clip_min ? du : 0.f;
    }
}

// unc_bwd_token_kernel on the head input with the gather summed in double: l2reg / l1reg give dL/dv two terms of
// opposite sign (beta's and the loss's), so the fp32 gather of unc_bwd_token_kernel loses more than the reference's
// own fp32 statements do.
__global__ void __launch_bounds__(UNC_THREADS) unc_mode_bwd_token_kernel(const GsrUncertaintyModeArgs a,
                                                                         const float* __restrict__ logit,
                                                                         const float* __restrict__ dv,
                                                                         float* __restrict__ dlogit) {
    const int T = a.th * a.tw;
    const int t = blockIdx.x * UNC_THREADS + threadIdx.x;
    if (t >= T) return;
    const int ty = t / a.tw, tx = t - ty * a.tw;
    int rlo, rhi, clo, chi;
    taps_of(a.th, a.Hp, ty, rlo, rhi);
    taps_of(a.tw, a.Wp, tx, clo, chi);
    rlo = max(rlo, a.pad_top); rhi = min(rhi, a.pad_top + a.uh - 1);       // the crop: only head-input pixels
    clo = max(clo, a.pad_left); chi = min(chi, a.pad_left + a.uw - 1);
    double acc = 0.0;
    for (int r = rlo; r <= rhi; ++r) {
        const float wy = tap_weight(a.th, a.Hp, r, ty);
        if (wy == 0.f) continue;
        const float* row = dv + (size_t)(r - a.pad_top) * a.uw - a.pad_left;
        double s = 0.0;
        for (int c = clo; c <= chi; ++c) {
            const float wx = tap_weight(a.tw, a.Wp, c, tx);
            if (wx != 0.f) s += (double)wx * (double)row[c];
        }
        acc += (double)wy * s;
    }
    const float l = logit[t];
    const double z = exp((double)l);
    dlogit[t] = (float)(l > 20.f ? acc : acc * z / (z + 1.0));
}

int check_mode_args(const GsrUncertaintyModeArgs* a, bool backward) {
    if (!a) { set_error("args is NULL"); return GSR_E_INVALID; }
    if (a->mode < GSR_UNC_MODE_L2REG || a->mode > GSR_UNC_MODE_DINO_MSSIM) {
        set_error("bad mode %d (0..3: l2reg, l1reg, dino, dino+mssim)", a->mode);
        return GSR_E_INVALID;
    }
    if (a->training != 0 && a->training != 1) { set_error("training must be 0 or 1"); return GSR_E_INVALID; }
    if (a->C <= 0 || a->C > UNC_MAX_C) { set_error("bad channel count C=%d (1..%d)", a->C, UNC_MAX_C); return GSR_E_INVALID; }
    const bool dino = dino_mode(a->mode);
    const int dims[14] = {a->th, a->tw, a->Hp, a->Wp, a->uh, a->uw, a->H, a->W,
                          dino ? a->nh : 1, dino ? a->nw : 1, dino ? a->ch : 1, dino ? a->cw : 1, dino ? a->nHp : 1,
                          dino ? a->nWp : 1};
    for (int d : dims)
        if (d <= 0) { set_error("bad sizes: every size must be positive"); return GSR_E_INVALID; }
    if (a->training && (long long)a->th * a->tw < 2) {
        set_error("bad sizes: batch statistics need more than one token");
        return GSR_E_INVALID;
    }
    if (a->th > a->Hp || a->tw > a->Wp || (dino && (a->ch > a->nHp || a->cw > a->nWp))) {
        set_error("bad sizes: a token grid is larger than its padded image");
        return GSR_E_INVALID;
    }
    if (a->pad_top < 0 || a->pad_left < 0 || a->pad_top + a->uh > a->Hp || a->pad_left + a->uw > a->Wp ||
        (dino && (a->npad_top < 0 || a->npad_left < 0 || a->npad_top + a->nh > a->nHp || a->npad_left + a->nw > a->nWp))) {
        set_error("bad sizes: the crop does not fit in the padded image");
        return GSR_E_INVALID;
    }
    if ((long long)a->Hp * a->Wp >= (1ll << 31) || (long long)a->H * a->W >= (1ll << 31) ||
        (dino && (long long)a->nHp * a->nWp >= (1ll << 31))) {
        set_error("image too large");
        return GSR_E_INVALID;
    }
    if (!(a->clip_min > 0.f)) { set_error("clip_min must be positive"); return GSR_E_INVALID; }
    if (!a->feat || !a->conv_w || !a->conv_b || !a->bn_w || !a->bn_b || !a->gt || !a->pred || !a->ssim || !a->msssim ||
        !a->loss_mult || !a->loss || !a->metrics || !a->scratch || (a->training && !a->mask) ||
        (!a->training && (!a->running_mean || !a->running_var)) || (dino && (!a->feat_gt_down || !a->feat_pred_down)) ||
        (a->mode == GSR_UNC_MODE_DINO_MSSIM && !a->msssim_down)) {
        set_error("a required pointer is NULL");
        return GSR_E_INVALID;
    }
    if (backward && (!a->dL_dloss || !a->d_conv_w || !a->d_conv_b || !a->d_bn_w || !a->d_bn_b)) {
        set_error("a gradient pointer is NULL");
        return GSR_E_INVALID;
    }
    return 0;
}

}  // namespace
}  // namespace gsr

extern "C" size_t gsr_uncertainty_scratch_bytes(const GsrUncertaintyArgs* a) {
    using namespace gsr;
    if (!a) return 0;
    GsrUncertaintyArgs c = *a;
    c.scratch = nullptr;
    if (c.C <= 0 || c.C > UNC_MAX_C || c.th <= 0 || c.tw <= 0 || c.H <= 0 || c.W <= 0 || c.nh <= 0 || c.nw <= 0 || c.ch <= 0 ||
        c.cw <= 0 || (long long)c.H * c.W >= (1ll << 31))
        return 0;
    Scratch s;
    return layout(c, &s);
}

extern "C" int gsr_uncertainty_forward(const GsrUncertaintyArgs* a, void* stream) {
    using namespace gsr;
    if (int rc = check_args(a, false)) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    Scratch s;
    layout(*a, &s);
    const int T = a->th * a->tw, CT = a->ch * a->cw, nbf = full_blocks(*a), nbd = down_blocks(*a);
    unc_bn_stats_kernel<<<a->C, UNC_THREADS, 0, st>>>(T, a->feat, a->mask, a->bn_eps, a->bn_momentum, s.mean, s.invstd,
                                                      a->running_mean, a->running_var, a->num_batches_tracked);
    unc_head_kernel<<<blocks_for(T), UNC_THREADS, 5 * a->C * sizeof(float), st>>>(
        a->C, T, a->feat, a->mask, s.mean, s.invstd, a->conv_w, a->conv_b, a->bn_w, a->bn_b, s.logit, s.sp);
    unc_cosine_kernel<<<(CT + UNC_THREADS / 32 - 1) / (UNC_THREADS / 32), UNC_THREADS, 0, st>>>(
        a->C, CT, a->feat_gt_down, a->feat_pred_down, s.cosine);
    unc_full_kernel<<<nbf, UNC_THREADS, 0, st>>>(*a, s.sp, s.pfull);
    unc_down_kernel<<<nbd, UNC_THREADS, 0, st>>>(*a, s.sp, s.cosine, s.dpart, s.pdown);
    unc_finalize_kernel<<<1, UNC_THREADS, 0, st>>>(*a, nbf, nbd, s.pfull, s.pdown);
    count_launches(6);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int gsr_uncertainty_backward(const GsrUncertaintyArgs* a, void* stream) {
    using namespace gsr;
    if (int rc = check_args(a, true)) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    Scratch s;
    layout(*a, &s);
    const int T = a->th * a->tw;
    unc_bwd_pixel_kernel<<<full_blocks(*a), UNC_THREADS, 0, st>>>(*a, s.sp, s.dpart, s.dv);
    unc_bwd_token_kernel<<<blocks_for(T), UNC_THREADS, 0, st>>>(*a, s.logit, s.dv, s.dlogit);
    unc_bwd_param_kernel<<<a->C, UNC_THREADS, 0, st>>>(*a, s.mean, s.invstd, s.dlogit);
    count_launches(3);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

extern "C" size_t gsr_uncertainty_mode_scratch_bytes(const GsrUncertaintyModeArgs* a) {
    using namespace gsr;
    if (!a) return 0;
    GsrUncertaintyModeArgs c = *a;
    c.scratch = nullptr;
    const bool dino = dino_mode(c.mode);
    if (c.mode < GSR_UNC_MODE_L2REG || c.mode > GSR_UNC_MODE_DINO_MSSIM || c.C <= 0 || c.C > UNC_MAX_C || c.th <= 0 ||
        c.tw <= 0 || c.uh <= 0 || c.uw <= 0 || c.H <= 0 || c.W <= 0 || (long long)c.H * c.W >= (1ll << 31) ||
        (dino && (c.nh <= 0 || c.nw <= 0 || c.ch <= 0 || c.cw <= 0)))
        return 0;
    ModeScratch s;
    return mode_layout(c, &s);
}

extern "C" int gsr_uncertainty_mode_forward(const GsrUncertaintyModeArgs* a, void* stream) {
    using namespace gsr;
    if (int rc = check_mode_args(a, false)) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    ModeScratch s;
    mode_layout(*a, &s);
    const bool dino = dino_mode(a->mode);
    const int T = a->th * a->tw, nbf = mode_full_blocks(*a), nbd = mode_down_blocks(*a);
    if (a->training)
        unc_bn_stats_kernel<<<a->C, UNC_THREADS, 0, st>>>(T, a->feat, a->mask, a->bn_eps, a->bn_momentum, s.mean, s.invstd,
                                                          a->running_mean, a->running_var, a->num_batches_tracked);
    else
        unc_bn_eval_kernel<<<blocks_for(a->C), UNC_THREADS, 0, st>>>(a->C, a->running_mean, a->running_var, a->bn_eps,
                                                                     s.mean, s.invstd, s.ones);
    unc_mode_head_kernel<<<blocks_for(T), UNC_THREADS, 5 * a->C * sizeof(float), st>>>(
        a->C, T, a->feat, a->training ? a->mask : s.ones, s.mean, s.invstd, a->conv_w, a->conv_b, a->bn_w, a->bn_b, s.logit,
        s.sp);
    if (dino) {
        const int CT = a->ch * a->cw;
        unc_cosine_kernel<<<(CT + UNC_THREADS / 32 - 1) / (UNC_THREADS / 32), UNC_THREADS, 0, st>>>(
            a->C, CT, a->feat_gt_down, a->feat_pred_down, s.cosine);
    }
    unc_mode_full_kernel<<<nbf, UNC_THREADS, 0, st>>>(*a, s.sp, s.pfull);
    if (dino) unc_mode_down_kernel<<<nbd, UNC_THREADS, 0, st>>>(*a, s.sp, s.cosine, s.dpart, s.pdown);
    unc_mode_finalize_kernel<<<1, UNC_THREADS, 0, st>>>(*a, nbf, nbd, s.pfull, s.pdown);
    count_launches(dino ? 6 : 4);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int gsr_uncertainty_mode_backward(const GsrUncertaintyModeArgs* a, void* stream) {
    using namespace gsr;
    if (int rc = check_mode_args(a, true)) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    ModeScratch s;
    mode_layout(*a, &s);
    const bool dino = dino_mode(a->mode);
    const int T = a->th * a->tw;
    const GsrUncertaintyArgs h = head_view(*a, s);
    if (!dino) unc_mode_bwd_full_kernel<<<mode_full_blocks(*a), UNC_THREADS, 0, st>>>(*a, s.sp, s.dfull);
    unc_mode_bwd_pixel_kernel<<<blocks_for((long long)a->uh * a->uw), UNC_THREADS, 0, st>>>(*a, s.sp, s.dpart, s.dfull,
                                                                                           s.dv);
    unc_mode_bwd_token_kernel<<<blocks_for(T), UNC_THREADS, 0, st>>>(*a, s.logit, s.dv, s.dlogit);
    unc_bwd_param_kernel<<<a->C, UNC_THREADS, 0, st>>>(h, s.mean, s.invstd, s.dlogit);
    count_launches(dino ? 3 : 4);
    GSR_CUDA(cudaGetLastError());
    return 0;
}
