// msssim.cu -- the image-quality statistics of wild-gaussians' uncertainty loss, forward only.
//
// What it replaces: `msssim(x, y, max_size, min_size)` (wildgaussians/method.py:171-187, with `_ssim_parts` :138-168) and
// `ssim_down(x, y, max_size)` (:126-135), which `UncertaintyModel._compute_losses` (:363-433) evaluates on every training
// step on the ground truth and the detached prediction.  PyTorch runs the pair as ~260 launches (25 depthwise 11x11
// convolutions) plus one pageable host-to-device copy of the window per SSIM evaluation.  No caller differentiates
// either statistic, so there is no backward.
//
// msssim, with (h, w) the host-computed area-resize size of the [B,3,H,W] inputs:
//   1. area_resize_kernel: adaptive average pooling of both images to [B,3,h,w] (skipped when (h, w) == (H, W));
//   2. level 0: msssim_parts_kernel writes l*c*s per channel;
//   3. per coarse level: avg_pool2_kernel (floor-sized 2x2 mean of both images), then msssim_parts_kernel writes the
//      contrast c and the structure s per channel as separate maps (their bilinear upsamplings are taken separately,
//      as the reference does: interp(c) * interp(s) != interp(c * s));
//   4. msssim_combine_kernel: per level-0 pixel and channel, l*c*s times the bilinear samples of every coarse c and s,
//      then the channel mean (bilinear interpolation is linear, so the mean may precede the final upsampling);
//   5. bilinear_up_kernel to [B,H,W] (skipped without a resize).
// At 1920x1080 with max_size 400, min_size 80 that is 10 launches (level 0 is 400x711 with 3 coarse levels).
// ssim_down: area_resize_kernel, the photometric loss's SSIM forward (ssim.cu, without backward factors), then
// bilinear_up_kernel: 3 launches.  No atomics, no host synchronisation; scratch is the caller's.
//
// Per level (method.py:148-168), with the 11-tap window of ssim_common.cuh and zero padding, C3 = C2 / 2:
//     sigma_x = sqrt(max(E[x^2] - mu_x^2, 0))
//     l = (2 mu_x mu_y + C1) / (mu_x^2 + mu_y^2 + C1)
//     c = (2 sigma_x sigma_y + C2) / (sigma_x^2 + sigma_y^2 + C2)      (the unclamped variances below the line)
//     s = (sigma_xy + C3) / (sigma_x sigma_y + C3)
// Resampling follows PyTorch's CUDA kernels: adaptive average pooling over [floor(i H/h), ceil((i+1) H/h)), and
// bilinear with align_corners=False from sizes (scale = in/out, source = max(scale (dst + 0.5) - 0.5, 0), the upper
// neighbour clamped at the edge).
#include "ssim_common.cuh"

namespace gsr {

constexpr int MSSSIM_MAX_LEVELS = 30;             // coarse levels; min_size >= 1 and h < 2^31 allow at most 30
constexpr int MS_THREADS = 256;
constexpr float SSIM_C3 = SSIM_C2 / 2.f;          // method.py:163 (C2 / 2 is exact in both precisions)

struct MsssimLevels {
    const float* cs[MSSSIM_MAX_LEVELS];          // [B][3][2 (c, s)][h][w] per coarse level
    int h[MSSSIM_MAX_LEVELS], w[MSSSIM_MAX_LEVELS];
    int n;
};

static unsigned ms_blocks(size_t n) {
    const size_t b = (n + MS_THREADS - 1) / MS_THREADS;
    return (unsigned)(b < 65536u * 16u ? b : 65536u * 16u);   // grid-stride loops cover the rest
}

// F.interpolate(mode='area') == adaptive_avg_pool2d to (h, w), both images; planes = B * 3.
__global__ void __launch_bounds__(MS_THREADS) area_resize_kernel(int planes, int H, int W, int h, int w,
                                                                 const float* __restrict__ x, const float* __restrict__ y,
                                                                 float* __restrict__ ox, float* __restrict__ oy) {
    const size_t hw = (size_t)h * w, n = (size_t)planes * hw, HW = (size_t)H * W;
    for (size_t i = blockIdx.x * (size_t)MS_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * MS_THREADS) {
        const size_t plane = i / hw;
        const int r = (int)((i - plane * hw) / w), q = (int)(i - plane * hw - (size_t)r * w);
        const int y0 = (int)((long long)r * H / h), y1 = (int)((((long long)r + 1) * H + h - 1) / h);
        const int x0 = (int)((long long)q * W / w), x1 = (int)((((long long)q + 1) * W + w - 1) / w);
        const float* px = x + plane * HW;
        const float* py = y + plane * HW;
        float sx = 0.f, sy = 0.f;
        for (int yy = y0; yy < y1; ++yy)
            for (int xx = x0; xx < x1; ++xx) {
                sx += px[(size_t)yy * W + xx];
                sy += py[(size_t)yy * W + xx];
            }
        const float kh = (float)(y1 - y0), kw = (float)(x1 - x0);
        ox[i] = sx / kh / kw;
        oy[i] = sy / kh / kw;
    }
}

// F.avg_pool2d(., 2) of both images: floor-sized 2x2 means.
__global__ void __launch_bounds__(MS_THREADS) avg_pool2_kernel(int planes, int hi, int wi, const float* __restrict__ x,
                                                               const float* __restrict__ y, float* __restrict__ ox,
                                                               float* __restrict__ oy) {
    const int ho = hi / 2, wo = wi / 2;
    const size_t hw = (size_t)ho * wo, n = (size_t)planes * hw, HW = (size_t)hi * wi;
    for (size_t i = blockIdx.x * (size_t)MS_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * MS_THREADS) {
        const size_t plane = i / hw;
        const int r = (int)((i - plane * hw) / wo), q = (int)(i - plane * hw - (size_t)r * wo);
        const size_t p = plane * HW + (size_t)(2 * r) * wi + 2 * q;
        ox[i] = (((x[p] + x[p + 1]) + x[p + wi]) + x[p + wi + 1]) / 4.f;
        oy[i] = (((y[p] + y[p + 1]) + y[p + wi]) + y[p + wi + 1]) / 4.f;
    }
}

// One pyramid level of _ssim_parts.  level0: out = [B][3][H][W] of l*c*s; otherwise out = [B][3][2][H][W] of (c, s).
__global__ void __launch_bounds__(SSIM_THREADS) msssim_parts_kernel(int H, int W, const float* __restrict__ img1,
                                                                    const float* __restrict__ img2, float* __restrict__ out,
                                                                    int level0, const SsimWindow win) {
    __shared__ float sx[SSIM_RH][SSIM_RW], sy[SSIM_RH][SSIM_RW];
    __shared__ float hb[5][SSIM_RH][SSIM_TW];
    const int x0 = blockIdx.x * SSIM_TW, y0 = blockIdx.y * SSIM_TH, b = blockIdx.z;
    const size_t HW = (size_t)H * W;

    for (int c = 0; c < 3; ++c) {
        const size_t plane = ((size_t)b * 3 + c) * HW;
        if (c) __syncthreads();                      // the previous channel's vertical pass is done with hb
        ssim_stage(sx, img1 + plane, H, W, x0, y0);
        ssim_stage(sy, img2 + plane, H, W, x0, y0);
        __syncthreads();
        ssim_blur_rows(sx, sy, hb, win);
        __syncthreads();
#pragma unroll
        for (int j = 0; j < SSIM_PPT; ++j) {
            const int i = threadIdx.x + j * SSIM_THREADS;
            const int r = i / SSIM_TW, q = i - r * SSIM_TW;
            const int gy = y0 + r, gx = x0 + q;
            if (gy >= H || gx >= W) continue;
            float mx, my, exx, eyy, exy;
            ssim_blur_column(hb, r, q, win, mx, my, exx, eyy, exy);
            const float mxx = mx * mx, myy = my * my, mxy = mx * my;
            const float vx = exx - mxx, vy = eyy - myy, cxy = exy - mxy;
            const float sdx = sqrtf(fmaxf(vx, 0.f)), sdy = sqrtf(fmaxf(vy, 0.f));
            const float cs = (2.f * sdx * sdy + SSIM_C2) / (vx + vy + SSIM_C2);
            const float st = (cxy + SSIM_C3) / (sdx * sdy + SSIM_C3);
            const size_t p = (size_t)gy * W + gx;
            if (level0) {
                const float lum = (2.f * mxy + SSIM_C1) / (mxx + myy + SSIM_C1);
                out[plane + p] = lum * cs * st;
            } else {
                const size_t q2 = ((size_t)b * 3 + c) * 2 * HW + p;
                out[q2] = cs;
                out[q2 + HW] = st;
            }
        }
    }
}

// Bilinear (align_corners=False, from sizes) source rows / columns and weights of output index `dst`.
struct Lerp {
    int i0, i1;
    float l0, l1;
};

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

// out[b][y][x] = mean over channels of lcs0 * prod over coarse levels of bilinear(c) * bilinear(s), at level-0 size.
__global__ void __launch_bounds__(MS_THREADS) msssim_combine_kernel(int B, int h, int w, const float* __restrict__ lcs0,
                                                                    const MsssimLevels lv, float* __restrict__ out) {
    const size_t hw = (size_t)h * w, n = (size_t)B * hw;
    for (size_t i = blockIdx.x * (size_t)MS_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * MS_THREADS) {
        const size_t b = i / hw, p = i - b * hw;
        const int r = (int)(p / w), q = (int)(p - (size_t)r * w);
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = lcs0[(b * 3 + c) * hw + p];
        for (int l = 0; l < lv.n; ++l) {
            const int hl = lv.h[l], wl = lv.w[l];
            const size_t hwl = (size_t)hl * wl;
            const Lerp ty = lerp_at(hl, h, r), tx = lerp_at(wl, w, q);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float* cs = lv.cs[l] + (b * 3 + c) * 2 * hwl;
                v[c] *= lerp2(cs, wl, ty, tx);
                v[c] *= lerp2(cs + hwl, wl, ty, tx);
            }
        }
        out[i] = ((v[0] + v[1]) + v[2]) / 3.f;
    }
}

// F.interpolate(mode='bilinear', align_corners=False) of [B][h][w] to [B][H][W].
__global__ void __launch_bounds__(MS_THREADS) bilinear_up_kernel(int B, int h, int w, int H, int W, const float* __restrict__ in,
                                                                 float* __restrict__ out) {
    const size_t HW = (size_t)H * W, n = (size_t)B * HW;
    for (size_t i = blockIdx.x * (size_t)MS_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * MS_THREADS) {
        const size_t b = i / HW, p = i - b * HW;
        const int r = (int)(p / W), q = (int)(p - (size_t)r * W);
        out[i] = lerp2(in + b * (size_t)h * w, w, lerp_at(h, H, r), lerp_at(w, W, q));
    }
}

// Number of coarse levels: the reference's `while h > min_size and w > min_size: pool` (method.py:180).
static int msssim_levels(int h, int w, int min_size) {
    int n = 0;
    while (h > min_size && w > min_size) {
        h /= 2; w /= 2; ++n;
    }
    return n;
}

static size_t pad64(size_t floats) { return (floats + 63) / 64 * 64; }   // 256-byte aligned regions

// Scratch layout in floats: resized x0, y0 | per coarse level: x, y, (c, s) | level-0 l*c*s | level-0 channel mean.
struct MsssimLayout {
    size_t x0, y0, lcs0, mean0, total;
    size_t x[MSSSIM_MAX_LEVELS], y[MSSSIM_MAX_LEVELS], cs[MSSSIM_MAX_LEVELS];
    int n, h[MSSSIM_MAX_LEVELS], w[MSSSIM_MAX_LEVELS];
};

static int msssim_check(int B, int h, int w, int min_size) {
    if (B <= 0 || h <= 0 || w <= 0) { set_error("bad sizes B=%d h=%d w=%d", B, h, w); return GSR_E_INVALID; }
    if (min_size < 1) { set_error("min_size must be >= 1, got %d", min_size); return GSR_E_INVALID; }
    if (B > 65535 || (h + SSIM_TH - 1) / SSIM_TH > 65535) { set_error("image batch or height too large (B=%d h=%d)", B, h); return GSR_E_INVALID; }
    if (msssim_levels(h, w, min_size) > MSSSIM_MAX_LEVELS) { set_error("more than %d pyramid levels", MSSSIM_MAX_LEVELS); return GSR_E_INVALID; }
    return 0;
}

static MsssimLayout msssim_layout(int B, int h, int w, int min_size) {
    MsssimLayout L;
    const size_t planes = (size_t)B * 3;
    size_t off = 0;
    L.x0 = off; off += pad64(planes * h * w);
    L.y0 = off; off += pad64(planes * h * w);
    L.n = msssim_levels(h, w, min_size);
    int hl = h, wl = w;
    for (int l = 0; l < L.n; ++l) {
        hl /= 2; wl /= 2;
        L.h[l] = hl; L.w[l] = wl;
        L.x[l] = off; off += pad64(planes * hl * wl);
        L.y[l] = off; off += pad64(planes * hl * wl);
        L.cs[l] = off; off += pad64(2 * planes * hl * wl);
    }
    L.lcs0 = off; off += pad64(planes * h * w);
    L.mean0 = off; off += pad64((size_t)B * h * w);
    L.total = off;
    return L;
}

}  // namespace gsr

extern "C" size_t gsr_msssim_scratch_bytes(int B, int h, int w, int min_size) {
    using namespace gsr;
    if (msssim_check(B, h, w, min_size)) return 0;
    return msssim_layout(B, h, w, min_size).total * sizeof(float);
}

extern "C" int gsr_msssim_forward(int B, int H, int W, int h, int w, int min_size, const float* img1, const float* img2,
                                  float* out, void* scratch, void* stream) {
    using namespace gsr;
    if (H <= 0 || W <= 0) { set_error("bad sizes H=%d W=%d", H, W); return GSR_E_INVALID; }
    if (int rc = msssim_check(B, h, w, min_size)) return rc;
    if (!img1 || !img2 || !out || !scratch) { set_error("img1, img2, out or scratch is NULL"); return GSR_E_INVALID; }
    static const SsimWindow win = ssim_window();
    const cudaStream_t st = (cudaStream_t)stream;
    const MsssimLayout L = msssim_layout(B, h, w, min_size);
    float* s = (float*)scratch;
    const bool resize = h != H || w != W;
    const float* x = img1;
    const float* y = img2;
    int launches = 0;
    if (resize) {
        area_resize_kernel<<<ms_blocks((size_t)B * 3 * h * w), MS_THREADS, 0, st>>>(B * 3, H, W, h, w, img1, img2, s + L.x0, s + L.y0);
        x = s + L.x0; y = s + L.y0; ++launches;
    }
    msssim_parts_kernel<<<ssim_grid(B, h, w), SSIM_THREADS, 0, st>>>(h, w, x, y, s + L.lcs0, 1, win);
    ++launches;
    MsssimLevels lv;
    lv.n = L.n;
    int hl = h, wl = w;
    for (int l = 0; l < L.n; ++l) {
        avg_pool2_kernel<<<ms_blocks((size_t)B * 3 * L.h[l] * L.w[l]), MS_THREADS, 0, st>>>(B * 3, hl, wl, x, y, s + L.x[l], s + L.y[l]);
        x = s + L.x[l]; y = s + L.y[l];
        hl = L.h[l]; wl = L.w[l];
        msssim_parts_kernel<<<ssim_grid(B, hl, wl), SSIM_THREADS, 0, st>>>(hl, wl, x, y, s + L.cs[l], 0, win);
        lv.cs[l] = s + L.cs[l]; lv.h[l] = hl; lv.w[l] = wl;
        launches += 2;
    }
    float* mean0 = resize ? s + L.mean0 : out;
    msssim_combine_kernel<<<ms_blocks((size_t)B * h * w), MS_THREADS, 0, st>>>(B, h, w, s + L.lcs0, lv, mean0);
    ++launches;
    if (resize) {
        bilinear_up_kernel<<<ms_blocks((size_t)B * H * W), MS_THREADS, 0, st>>>(B, h, w, H, W, mean0, out);
        ++launches;
    }
    count_launches(launches);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

extern "C" size_t gsr_ssim_down_scratch_bytes(int B, int h, int w) {
    using namespace gsr;
    if (B <= 0 || h <= 0 || w <= 0) return 0;
    const size_t planes = (size_t)B * 3;
    return (2 * pad64(planes * h * w) + pad64((size_t)B * h * w)) * sizeof(float);
}

extern "C" int gsr_ssim_down_forward(int B, int H, int W, int h, int w, const float* img1, const float* img2, float* out,
                                     void* scratch, void* stream) {
    using namespace gsr;
    if (B <= 0 || H <= 0 || W <= 0 || h <= 0 || w <= 0) {
        set_error("bad sizes B=%d H=%d W=%d h=%d w=%d", B, H, W, h, w);
        return GSR_E_INVALID;
    }
    if (B > 65535 || (h + SSIM_TH - 1) / SSIM_TH > 65535) { set_error("image batch or height too large (B=%d h=%d)", B, h); return GSR_E_INVALID; }
    const bool resize = h != H || w != W;
    if (!img1 || !img2 || !out || (resize && !scratch)) { set_error("img1, img2, out or scratch is NULL"); return GSR_E_INVALID; }
    if (!resize) return gsr_ssim_forward(B, H, W, img1, img2, out, nullptr, stream);
    const cudaStream_t st = (cudaStream_t)stream;
    const size_t planes = (size_t)B * 3;
    float* x = (float*)scratch;
    float* y = x + pad64(planes * h * w);
    float* map = y + pad64(planes * h * w);
    area_resize_kernel<<<ms_blocks(planes * h * w), MS_THREADS, 0, st>>>(B * 3, H, W, h, w, img1, img2, x, y);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    if (int rc = gsr_ssim_forward(B, h, w, x, y, map, nullptr, stream)) return rc;
    bilinear_up_kernel<<<ms_blocks((size_t)B * H * W), MS_THREADS, 0, st>>>(B, h, w, H, W, map, out);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}
