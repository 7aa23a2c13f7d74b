// ssim.cu -- the SSIM term of wild-gaussians' photometric loss in ONE kernel per direction.
//
// What it replaces: `ssim(img1, img2, window_size=11, size_average=...)` (wildgaussians/method.py:644-673), called every
// training step at :1949 on the rendered image and the ground truth.  PyTorch runs it as 5 depthwise 11x11 convolutions
// forward (3 backward) and ~60 elementwise launches over full [3,H,W] fp32 tensors.  Here:
//   * forward: one CTA per 32x16 output tile, all three channels in that CTA.  Per channel the tile plus a 5-pixel halo
//     of both images is staged in shared memory (zeros outside the image: the reference's zero padding), the five
//     moments x, y, x^2, y^2, xy are blurred separably (11 horizontal taps, then 11 vertical taps), and the per-channel
//     SSIM is accumulated in registers, so the channel mean (method.py:673) never leaves the SM.  When a gradient is
//     wanted the three per-pixel factors of the backward are stored as well;
//   * backward: the three factor maps, scaled by the upstream dL/dmap / 3, are blurred the same way and combined with
//     x and y at the centre pixel.
// Traffic: forward reads 24 B and writes 4 B (+ 36 B of factors) per pixel, backward reads 24 + 36 + 4 B and writes
// 12 B per pixel; no atomics, so results are bitwise reproducible.
//
// Window, tile geometry and the separable blur: ssim_common.cuh.
//
// Backward, per channel, with window sums over pixels inside the image (the window is symmetric):
//     mu_x = w*x,  E_xx = w*x^2,  E_xy = w*xy,  sigma_x^2 = E_xx - mu_x^2,  sigma_xy = E_xy - mu_x mu_y
//     A1 = 2 mu_x mu_y + C1,  A2 = 2 sigma_xy + C2,  B1 = mu_x^2 + mu_y^2 + C1,  B2 = sigma_x^2 + sigma_y^2 + C2,
//     S = A1 A2 / (B1 B2)
//     dS/dmu_x = 2 mu_y (A2 - A1) / (B1 B2) - 2 mu_x S (B2 - B1) / (B1 B2)
//     dS/dE_xx = -S / B2
//     dS/dE_xy = 2 A1 / (B1 B2)
//     dL/dx_p  = w*(g dS/dmu_x)_p + 2 x_p w*(g dS/dE_xx)_p + y_p w*(g dS/dE_xy)_p,   g = dL/dmap / 3
// None of the factors divides by A1 or A2, so they stay finite where A2 <= 0.
#include "ssim_common.cuh"

namespace gsr {

__global__ void __launch_bounds__(SSIM_THREADS) ssim_fwd_kernel(int H, int W, const float* __restrict__ img1,
                                                                const float* __restrict__ img2, float* __restrict__ ssim_map,
                                                                float* __restrict__ partials, const SsimWindow win) {
    __shared__ float sx[SSIM_RH][SSIM_RW], sy[SSIM_RH][SSIM_RW];
    __shared__ float hb[5][SSIM_RH][SSIM_TW];
    const int x0 = blockIdx.x * SSIM_TW, y0 = blockIdx.y * SSIM_TH, b = blockIdx.z;
    const size_t HW = (size_t)H * W;
    float acc[SSIM_PPT];
#pragma unroll
    for (int j = 0; j < SSIM_PPT; ++j) acc[j] = 0.f;

    for (int c = 0; c < 3; ++c) {
        const size_t plane = ((size_t)b * 3 + c) * HW;
        if (c) __syncthreads();                      // the previous channel's vertical pass is done with hb
        ssim_stage(sx, img1 + plane, H, W, x0, y0);
        ssim_stage(sy, img2 + plane, H, W, x0, y0);
        __syncthreads();
        ssim_blur_rows(sx, sy, hb, win);
        __syncthreads();
        // vertical pass + the per-channel SSIM and its backward factors
#pragma unroll
        for (int j = 0; j < SSIM_PPT; ++j) {
            const int i = threadIdx.x + j * SSIM_THREADS;
            const int r = i / SSIM_TW, q = i - r * SSIM_TW;
            float mx, my, exx, eyy, exy;
            ssim_blur_column(hb, r, q, win, mx, my, exx, eyy, exy);
            const float mxx = mx * mx, myy = my * my, mxy = mx * my;
            const float A1 = 2.f * mxy + SSIM_C1, A2 = 2.f * (exy - mxy) + SSIM_C2;
            const float B1 = mxx + myy + SSIM_C1, B2 = (exx - mxx) + (eyy - myy) + SSIM_C2;
            const float D = B1 * B2;
            const float S = (A1 * A2) / D;
            acc[j] += S;
            const int gy = y0 + r, gx = x0 + q;
            if (partials && gy < H && gx < W) {
                const float invD = 1.f / D;
                const size_t p = (size_t)b * 9 * HW + (size_t)c * HW + (size_t)gy * W + gx;
                partials[p] = (2.f * my * (A2 - A1) - 2.f * mx * S * (B2 - B1)) * invD;   // dS/dmu_x
                partials[p + 3 * HW] = -S / B2;                                          // dS/dE_xx
                partials[p + 6 * HW] = 2.f * A1 * invD;                                  // dS/dE_xy
            }
        }
    }
#pragma unroll
    for (int j = 0; j < SSIM_PPT; ++j) {
        const int i = threadIdx.x + j * SSIM_THREADS;
        const int gy = y0 + i / SSIM_TW, gx = x0 + i % SSIM_TW;
        if (gy < H && gx < W) ssim_map[(size_t)b * HW + (size_t)gy * W + gx] = acc[j] / 3.f;
    }
}

// SCALED: the result is multiplied per pixel by s0 then s1 ([B,H,W] each, NULL = 1), the backward of scale_grads on img1
// (train_loss.cu); without it the kernel is the plain SSIM backward.
template <bool SCALED>
__global__ void __launch_bounds__(SSIM_THREADS) ssim_bwd_kernel(int H, int W, const float* __restrict__ img1,
                                                                const float* __restrict__ img2, const float* __restrict__ partials,
                                                                const float* __restrict__ dL_dmap, float* __restrict__ dL_dimg1,
                                                                const float* __restrict__ s0, const float* __restrict__ s1,
                                                                const SsimWindow win) {
    __shared__ float sf[3][SSIM_RH][SSIM_RW];
    __shared__ float hb[3][SSIM_RH][SSIM_TW];
    const int x0 = blockIdx.x * SSIM_TW, y0 = blockIdx.y * SSIM_TH, b = blockIdx.z;
    const size_t HW = (size_t)H * W;
    const float* G = dL_dmap + (size_t)b * HW;

    for (int c = 0; c < 3; ++c) {
        const float* P = partials + (size_t)b * 9 * HW + (size_t)c * HW;
        if (c) __syncthreads();                      // the previous channel's vertical pass is done with hb
        // g * factor, g = dL/dmap / 3 (the channel mean's backward), zero outside the image
        for (int i = threadIdx.x; i < SSIM_RH * SSIM_RW; i += SSIM_THREADS) {
            const int r = i / SSIM_RW, q = i - r * SSIM_RW;
            const int gy = y0 - SSIM_R + r, gx = x0 - SSIM_R + q;
            float f0 = 0.f, f1 = 0.f, f2 = 0.f;
            if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
                const size_t p = (size_t)gy * W + gx;
                const float g = G[p] / 3.f;
                f0 = g * P[p];
                f1 = g * P[p + 3 * HW];
                f2 = g * P[p + 6 * HW];
            }
            sf[0][r][q] = f0; sf[1][r][q] = f1; sf[2][r][q] = f2;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < SSIM_RH * SSIM_TW; i += SSIM_THREADS) {
            const int r = i / SSIM_TW, q = i - r * SSIM_TW;
            float m0 = 0.f, m1 = 0.f, m2 = 0.f;
#pragma unroll
            for (int k = 0; k < SSIM_K; ++k) {
                const float w = win.w[k];
                m0 = fmaf(w, sf[0][r][q + k], m0);
                m1 = fmaf(w, sf[1][r][q + k], m1);
                m2 = fmaf(w, sf[2][r][q + k], m2);
            }
            hb[0][r][q] = m0; hb[1][r][q] = m1; hb[2][r][q] = m2;
        }
        __syncthreads();
        const size_t plane = ((size_t)b * 3 + c) * HW;
#pragma unroll
        for (int j = 0; j < SSIM_PPT; ++j) {
            const int i = threadIdx.x + j * SSIM_THREADS;
            const int r = i / SSIM_TW, q = i - r * SSIM_TW;
            const int gy = y0 + r, gx = x0 + q;
            if (gy >= H || gx >= W) continue;
            float d0 = 0.f, d1 = 0.f, d2 = 0.f;
#pragma unroll
            for (int k = 0; k < SSIM_K; ++k) {
                const float w = win.w[k];
                d0 = fmaf(w, hb[0][r + k][q], d0);
                d1 = fmaf(w, hb[1][r + k][q], d1);
                d2 = fmaf(w, hb[2][r + k][q], d2);
            }
            const size_t p = plane + (size_t)gy * W + gx;
            float v = d0 + 2.f * img1[p] * d1 + img2[p] * d2;
            if (SCALED) {
                const size_t q = (size_t)b * HW + (size_t)gy * W + gx;
                if (s0) v = __fmul_rn(v, s0[q]);
                if (s1) v = __fmul_rn(v, s1[q]);
            }
            dL_dimg1[p] = v;
        }
    }
}

static int ssim_check_sizes(int B, int H, int W) {
    if (B <= 0 || H <= 0 || W <= 0) { set_error("bad sizes B=%d H=%d W=%d", B, H, W); return GSR_E_INVALID; }
    if (B > 65535 || (H + SSIM_TH - 1) / SSIM_TH > 65535) { set_error("image batch or height too large (B=%d H=%d)", B, H); return GSR_E_INVALID; }
    return 0;
}

int ssim_backward_launch(int B, int H, int W, const float* img1, const float* img2, const float* partials,
                         const float* dL_dmap, float* dL_dimg1, const float* s0, const float* s1, cudaStream_t stream) {
    static const SsimWindow win = ssim_window();
    if (s0 || s1)
        ssim_bwd_kernel<true><<<ssim_grid(B, H, W), SSIM_THREADS, 0, stream>>>(H, W, img1, img2, partials, dL_dmap, dL_dimg1,
                                                                              s0, s1, win);
    else
        ssim_bwd_kernel<false><<<ssim_grid(B, H, W), SSIM_THREADS, 0, stream>>>(H, W, img1, img2, partials, dL_dmap, dL_dimg1,
                                                                               nullptr, nullptr, win);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace gsr

extern "C" int gsr_ssim_forward(int B, int H, int W, const float* img1, const float* img2, float* ssim_map, float* partials,
                                void* stream) {
    using namespace gsr;
    if (int rc = ssim_check_sizes(B, H, W)) return rc;
    if (!img1 || !img2 || !ssim_map) { set_error("img1, img2 or ssim_map is NULL"); return GSR_E_INVALID; }
    static const SsimWindow win = ssim_window();
    ssim_fwd_kernel<<<ssim_grid(B, H, W), SSIM_THREADS, 0, (cudaStream_t)stream>>>(H, W, img1, img2, ssim_map, partials, win);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int gsr_ssim_backward(int B, int H, int W, const float* img1, const float* img2, const float* partials,
                                 const float* dL_dmap, float* dL_dimg1, void* stream) {
    using namespace gsr;
    if (int rc = ssim_check_sizes(B, H, W)) return rc;
    if (!img1 || !img2 || !partials || !dL_dmap || !dL_dimg1) {
        set_error("img1, img2, partials, dL_dmap or dL_dimg1 is NULL");
        return GSR_E_INVALID;
    }
    return ssim_backward_launch(B, H, W, img1, img2, partials, dL_dmap, dL_dimg1, nullptr, nullptr, (cudaStream_t)stream);
}
