// ssim_common.cuh -- the window, tile geometry and separable 5-moment blur shared by ssim.cu (the photometric loss's
// SSIM) and msssim.cu (the uncertainty loss's multi-scale SSIM and downsampled SSIM).
//
// Window: the reference's 1-D Gaussian (sigma 1.5, 11 taps) built in fp32 -- fp32(exp(.)) / fp32 sum -- applied
// separably; its 2-D window is the fp32 outer product of the same vector.  A CTA of SSIM_THREADS threads covers one
// SSIM_TW x SSIM_TH output tile; the tile plus a SSIM_R-pixel halo of both images is staged in shared memory with zeros
// outside the image (the reference's zero padding).
#pragma once

#include "common.cuh"

#include <math.h>

namespace gsr {

constexpr int SSIM_TW = 32;                       // output tile width (one warp per tile row)
constexpr int SSIM_TH = 16;                       // output tile height
constexpr int SSIM_R = 5;                         // window radius (window_size 11)
constexpr int SSIM_K = 2 * SSIM_R + 1;
constexpr int SSIM_RW = SSIM_TW + 2 * SSIM_R;     // staged region: tile plus halo
constexpr int SSIM_RH = SSIM_TH + 2 * SSIM_R;
constexpr int SSIM_THREADS = 256;
constexpr int SSIM_PPT = SSIM_TW * SSIM_TH / SSIM_THREADS;   // output pixels per thread
constexpr float SSIM_C1 = (float)(0.01 * 0.01);       // method.py:665-666, Python doubles rounded to fp32
constexpr float SSIM_C2 = (float)(0.03 * 0.03);
static_assert(SSIM_TW * SSIM_TH % SSIM_THREADS == 0, "whole pixels per thread");

struct SsimWindow {
    float w[SSIM_K];
};

// The reference's 1-D window (method.py:648-649): fp32(exp(-(x - 5)^2 / (2 sigma^2))), divided by the fp32 sum of those
// taps.  The sum is accumulated in double and rounded once, which reproduces PyTorch's `gauss.sum()` here; a plain fp32
// running sum lands one ulp away, and since sigma^2 = E[x^2] - mu^2 is sensitive to the window's total weight, that ulp
// shows up as a systematic ~1e-6 offset of the SSIM mean.
static SsimWindow ssim_window() {
    SsimWindow g;
    double sum = 0.0;
    for (int x = 0; x < SSIM_K; ++x) {
        g.w[x] = (float)exp(-(double)((x - SSIM_R) * (x - SSIM_R)) / (2.0 * 1.5 * 1.5));
        sum += g.w[x];
    }
    const float fsum = (float)sum;
    for (int x = 0; x < SSIM_K; ++x) g.w[x] = g.w[x] / fsum;
    return g;
}

// Stage the tile's region of one channel plane into `dst`, zeros outside the image.
__device__ __forceinline__ void ssim_stage(float (*dst)[SSIM_RW], const float* __restrict__ src, int H, int W, int x0, int y0) {
    for (int i = threadIdx.x; i < SSIM_RH * SSIM_RW; i += SSIM_THREADS) {
        const int r = i / SSIM_RW, q = i - r * SSIM_RW;
        const int gy = y0 - SSIM_R + r, gx = x0 - SSIM_R + q;
        dst[r][q] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? src[(size_t)gy * W + gx] : 0.f;
    }
}

// Horizontal pass over every staged row: the 5 moments x, y, x^2, y^2, xy per (row, output column) into hb.
__device__ __forceinline__ void ssim_blur_rows(const float (*sx)[SSIM_RW], const float (*sy)[SSIM_RW],
                                               float (*hb)[SSIM_RH][SSIM_TW], const SsimWindow& win) {
    for (int i = threadIdx.x; i < SSIM_RH * SSIM_TW; i += SSIM_THREADS) {
        const int r = i / SSIM_TW, q = i - r * SSIM_TW;
        float m0 = 0.f, m1 = 0.f, m2 = 0.f, m3 = 0.f, m4 = 0.f;
#pragma unroll
        for (int k = 0; k < SSIM_K; ++k) {
            const float x = sx[r][q + k], y = sy[r][q + k], w = win.w[k];
            m0 = fmaf(w, x, m0);
            m1 = fmaf(w, y, m1);
            m2 = fmaf(w, x * x, m2);
            m3 = fmaf(w, y * y, m3);
            m4 = fmaf(w, x * y, m4);
        }
        hb[0][r][q] = m0; hb[1][r][q] = m1; hb[2][r][q] = m2; hb[3][r][q] = m3; hb[4][r][q] = m4;
    }
}

// Vertical pass at output pixel (r, q) of the tile: mu_x, mu_y, E[x^2], E[y^2], E[xy].
__device__ __forceinline__ void ssim_blur_column(const float (*hb)[SSIM_RH][SSIM_TW], int r, int q, const SsimWindow& win,
                                                 float& mx, float& my, float& exx, float& eyy, float& exy) {
    mx = 0.f; my = 0.f; exx = 0.f; eyy = 0.f; exy = 0.f;
#pragma unroll
    for (int k = 0; k < SSIM_K; ++k) {
        const float w = win.w[k];
        mx = fmaf(w, hb[0][r + k][q], mx);
        my = fmaf(w, hb[1][r + k][q], my);
        exx = fmaf(w, hb[2][r + k][q], exx);
        eyy = fmaf(w, hb[3][r + k][q], eyy);
        exy = fmaf(w, hb[4][r + k][q], exy);
    }
}

static dim3 ssim_grid(int B, int H, int W) {
    return dim3((W + SSIM_TW - 1) / SSIM_TW, (H + SSIM_TH - 1) / SSIM_TH, B);
}

}  // namespace gsr
