// render_common.cuh -- pieces shared by the forward and backward compositing kernels.
#pragma once
#include "common.cuh"

namespace gsr {

// Pair arithmetic of the packed composite kernels: each element is rounded exactly like the scalar instruction and
// never contracted, so a kernel that spells out the reference's expressions with these (fma2 exactly where nvcc fuses
// the reference's scalar expressions) gives the reference's bits.  sm_90 has no 2-wide fp32 instructions; the pairing
// keeps the packed kernels' staging (one LDS.128 = two ready-made broadcast pairs) and their fused epilogues.
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// Thread -> pixel mapping inside a 16x16 tile.  A thread owns 2 vertically adjacent pixels (k = 0, 1), a warp owns a
// compact 8x8 block, warp k being block k of the blend masks (the reference: one pixel per thread, a warp = a 16x2
// strip).  Per-pixel results do not depend on the mapping.  Two pixels per thread amortise the per-Gaussian
// shared-memory loads, loop control and (in the backward) the warp reduction over more (pixel, Gaussian) pairs; the
// compact block keeps the per-warp culling selective and every 32-byte output sector is written by one warp.
struct PixelMap {
    static constexpr int PPT = 2;                       // pixels per thread
    static constexpr int THREADS = TILE * TILE / PPT;
    static constexpr int WARPS = THREADS / 32;
    static constexpr int BW = 8, BH = 4 * PPT;          // warp block in pixels
    static constexpr int BLOCKS_X = TILE / BW;
    __device__ static __forceinline__ void pixel(int tid, int k, int& lx, int& ly) {
        const int warp = tid >> 5, lane = tid & 31;
        lx = (warp % BLOCKS_X) * BW + (lane & 7);
        ly = (warp / BLOCKS_X) * BH + (lane >> 3) * PPT + k;
    }
};

// Bounding box of the warp's (sub-pixel shifted) sample positions; lanes/pixels outside the image are ignored.
struct WarpBox {
    float x0, x1, y0, y1;
};
__device__ __forceinline__ WarpBox warp_box_reduce(float x0, float x1, float y0, float y1) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        x0 = fminf(x0, __shfl_xor_sync(0xFFFFFFFFu, x0, o));
        x1 = fmaxf(x1, __shfl_xor_sync(0xFFFFFFFFu, x1, o));
        y0 = fminf(y0, __shfl_xor_sync(0xFFFFFFFFu, y0, o));
        y1 = fmaxf(y1, __shfl_xor_sync(0xFFFFFFFFu, y1, o));
    }
    return {x0, x1, y0, y1};
}

// Can the Gaussian with centre/extents g = {x, y, hx, hy} reach alpha >= 1/255 anywhere in the box?
// Conservative (see preprocess_fwd.cu); every comparison is false for NaN, which keeps the Gaussian.
__device__ __forceinline__ bool box_may_touch(const float4 g, const WarpBox& b) {
    return !(g.z < 0.f || g.x + g.z < b.x0 || g.x - g.z > b.x1 || g.y + g.w < b.y0 || g.y - g.w > b.y1);
}

// Can the Gaussian with centre (x, y), conic (A, B, C) and opacity o reach alpha >= 1/255 at some sample of the box?
// With u = x - px, v = y - py the kernels' power is -q/2, q = A u^2 + 2 B u v + C v^2, and alpha >= 1/255 needs
// q <= 2 ln(255 o).  The minimum of q over the box is 0 if the centre is inside; otherwise it lies on the boundary
// (q is a convex 1-D quadratic along every edge since A, C > 0, and has no interior minimum off the centre), so it is
// the least of the four clamped 1-D edge minima.  Conservative like the extents (preprocess_fwd.cu): every q is
// lowered by 1e-3 of the magnitude of its terms and the bound raised by 2e-3, far above fp32 rounding and the error
// of __logf; a non-positive A or C, or a NaN, keeps the Gaussian.  Use after box_may_touch (negative extents).
__device__ __forceinline__ bool ellipse_may_touch(float x, float y, float A, float B, float C, float o, const WarpBox& b) {
    const float u0 = x - b.x1, u1 = x - b.x0, v0 = y - b.y1, v1 = y - b.y0;
    if (u0 <= 0.f && u1 >= 0.f && v0 <= 0.f && v1 >= 0.f) return true;
    if (!(A > 0.f && C > 0.f)) return true;
    const float rA = __frcp_rn(A), rC = __frcp_rn(C);
    auto q_lo = [&](float u, float v) {
        const float a = A * u * u, c = C * v * v, m = 2.f * B * u * v;
        return (a + c + m) - 1e-3f * (a + c + fabsf(m));
    };
    const float q = fminf(fminf(q_lo(u0, fminf(fmaxf(-B * u0 * rC, v0), v1)), q_lo(u1, fminf(fmaxf(-B * u1 * rC, v0), v1))),
                          fminf(q_lo(fminf(fmaxf(-B * v0 * rA, u0), u1), v0), q_lo(fminf(fmaxf(-B * v1 * rA, u0), u1), v1)));
    return !(q > 2.f * __logf(255.f * o) + 2e-3f);
}

}  // namespace gsr
