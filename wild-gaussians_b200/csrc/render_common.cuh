// render_common.cuh -- pieces shared by the forward and backward compositing kernels.
#pragma once
#include "common.cuh"

namespace gsr {

constexpr int RT_BATCH = 256;   // instances staged in shared memory per round

__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gmem_src) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_4(void* smem_dst, const void* gmem_src) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

// Pair arithmetic of the packed composite kernels: each element is rounded exactly like the scalar instruction and
// never contracted, so a pair gives the scalar kernel's bits.  sm_90 has no 2-wide fp32 instructions; the pairing
// keeps the packed kernels' staging (one LDS.128 = two ready-made broadcast pairs) and their fused epilogues.
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// Thread -> pixel mapping inside a 16x16 tile.  A thread owns PPT pixels (1, 2 or 4) arranged PX x PY,
// a warp owns a compact block of (8 PX) x (4 PY) pixels (the reference: one pixel per thread, a warp =
// a 16x2 strip).  Per-pixel results do not depend on the mapping.  More pixels per thread amortise the
// per-Gaussian shared-memory loads, loop control and (in the backward) the warp reduction over more
// (pixel, Gaussian) pairs; the compact block keeps the per-warp culling selective and every 32-byte
// output sector is written by one warp.
template <int PPT>
struct PixelMap {
    static_assert(PPT == 1 || PPT == 2 || PPT == 4, "PPT must be 1, 2 or 4");
    static constexpr int PX = PPT == 4 ? 2 : 1;
    static constexpr int PY = PPT >= 2 ? 2 : 1;
    static constexpr int THREADS = TILE * TILE / PPT;
    static constexpr int WARPS = THREADS / 32;
    static constexpr int BW = 8 * PX, BH = 4 * PY;          // warp block in pixels
    static constexpr int BLOCKS_X = TILE / BW;
    __device__ static __forceinline__ void pixel(int tid, int k, int& lx, int& ly) {
        const int warp = tid >> 5, lane = tid & 31;
        lx = (warp % BLOCKS_X) * BW + (lane & 7) * PX + (k % PX);
        ly = (warp / BLOCKS_X) * BH + (lane >> 3) * PY + (k / PX);
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

}  // namespace gsr
