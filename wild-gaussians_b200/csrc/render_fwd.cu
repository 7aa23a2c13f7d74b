// render_fwd.cu -- per-tile front-to-back alpha compositing.
// Replaces renderCUDA<3> of the reference (forward.cu:273-395).
//
// One CTA of 128 threads per 16x16 tile; a thread owns 2 vertically adjacent pixels, a warp an 8x8
// block (PixelMap, render_common.cuh).  The tile's slice of the sorted instance list is consumed in
// rounds of 128 instances, one per thread: each thread loads its instance's 32-byte projected record
// and colour into registers a round ahead and writes them to a double buffer in shared memory when
// the round starts, so the loads of round r+1 overlap the blending of round r.  Colours are staged
// too (the reference fetches them from global memory inside the blend loop, forward.cu:376).
//
// Per-warp culling: before blending 32 staged Gaussians, every lane tests one of them against the
// bounding box of the warp's sample positions using the conservative footprint extents computed in
// preprocess_fwd.cu, then against the footprint ellipse itself (ellipse_may_touch, render_common.cuh);
// a ballot gives the warp a 32-bit mask and only the set bits are blended.
// The skipped (pixel, Gaussian) pairs are pairs the reference rejects with alpha < 1/255
// (forward.cu:365), so the image, final_T and n_contrib are unchanged; `contributor` is derived from
// the position in the list, not counted, so it still counts every instance like forward.cu:349.
//
// Blend masks: for the first MASK_K positions of a tile's list, the training composite records per
// 8x8 pixel block whether some pixel of the block blended the position (common.cuh).  The backward
// walks only those positions.
//
// Numerics contract (SURVEY.md 8a note N3): power / alpha / test_T / the colour accumulation have
// the reference's expression shapes (forward.cu:353-378,393), fused exactly where nvcc fuses the
// reference's scalar expressions; every other operation is rounded as its scalar instruction and never
// contracted (add2 / mul2, render_common.cuh), and expf is the accurate one.  So the three
// discontinuous tests (power > 0, alpha < 1/255, T(1-alpha) < 1e-4) take the reference's branch and
// n_contrib / pixels match the reference bit for bit.
#include "render_common.cuh"

namespace gsr {

struct RenderFwdParams {
    int W, H, grid_x, ty0;
    const uint2* ranges;
    const uint32_t* point_list;
    const float2* subpixel_offset;
    const float4* rec;
    const float* colors;       // [P,3]
    const float* bg;
    float* final_T;
    uint32_t* n_contrib;
    float* out_color;
    uint32_t* blend_mask;      // [T][MASK_BLOCKS][MASK_WORDS] (common.cuh)
    // multi-GPU: the band is stored into the [4,H,W] images (colour + final transmittance) of ALL ranks through
    // peer-mapped pointers (image all-gather fused into the composite's epilogue); NULL / 0 = local out_color only
    float* const* peer_out;
    int n_peers;
    // display epilogue (render_fwd_packed_kernel<true, *>, gsr_forward_display): colour [H,W,3] as clamp(0, 1) then NaN -> 0,
    // accumulation 1 - T [H,W], and with DEPTH a fourth channel composited from depth_values [P] into out_depth [H,W]
    float* disp_color;
    float* disp_accum;
    float* disp_depth;
    const float* depth_values;
};

// word `word` of 8x8 block k of this CTA's tile
__device__ __forceinline__ uint32_t* blend_mask_word(const RenderFwdParams& p, int k, int word) {
    const int tile = (blockIdx.y + p.ty0) * p.grid_x + blockIdx.x;
    return p.blend_mask + ((size_t)tile * MASK_BLOCKS + k) * MASK_WORDS + word;
}

// ---- packed composite: 2 pixels per lane, their arithmetic written as pairs (add2 / mul2 / fma2) ----------------
// Both pixels of a lane share every per-Gaussian operand load and the loop control.  Each element of a pair goes through
// the reference's operations in the reference's order (forward.cu:353-378) -- power = fma(fma(dx, A dx, (C dy) dy),
// -0.5, -((B dx) dy)), alpha = min(0.99, o expf(power)), test_T = T (1 - alpha), C = fma(T, alpha c, C) -- so pixels,
// final_T and n_contrib are the reference's bits.  A pair that does not blend is carried as alpha = 0, which leaves C
// and T unchanged exactly.
// Staging: the raw records travel through registers and are written to shared memory already duplicated
// ({x, x, y, y}, ...), so one LDS.128 yields two ready-made broadcast pairs.
struct __align__(16) FwdPairRec {     // 80 bytes
    float4 xy;     // {x, x, y, y}
    float4 ac;     // {conic.x, conic.x, conic.z, conic.z}
    float4 bo;     // {-conic.y, -conic.y, opacity, opacity}
    float4 rg;     // {r, r, g, g}
    float4 bb;     // {b, b, hx, hy}: the footprint extents for the per-warp culling
};

// torch.clamp(x, 0, 1).nan_to_num_(0) of WildGaussians.render: clamp keeps a NaN, nan_to_num turns it into 0
__device__ __forceinline__ float display_value(float x) { return isnan(x) ? 0.f : fminf(fmaxf(x, 0.f), 1.f); }

// Two instantiations of one walk.  <false, false> is the training composite: colour planes, final_T, n_contrib and the
// blend masks the backward replays.  <true, DEPTH> is the display composite of an inference render: the same walk with
// the same pair arithmetic, culling and early-out, so its colour sums and T are the training kernel's bits, but it keeps
// no backward state and writes the display epilogue (RenderFwdParams::disp_*).  With DEPTH it carries a fourth channel,
// depth_values[id] composited with the colours' recurrence fma(T, alpha c, C); the values travel as {d, d} pairs in a
// shared array of their own (8 B per staged instance next to the 80 B record).
// (128, 9): at most 56 registers, so that 9 CTAs (36 warps) fit an SM, as the shared memory allows
template <bool DISPLAY, bool DEPTH>
__global__ void __launch_bounds__(128, 9) render_fwd_packed_kernel(const __grid_constant__ RenderFwdParams p) {
    static_assert(DISPLAY || !DEPTH, "the depth channel is a display output");
    using PM = PixelMap;
    constexpr int THREADS = 128;
    constexpr int PB = 128;               // instances per round
    __shared__ FwdPairRec s_rec[2][PB];
    __shared__ uint32_t s_blend[PixelMap::WARPS][MASK_WORDS];   // blend-mask words, written out at the end
    __shared__ float2 s_dep[2][DEPTH ? PB : 1];                 // {d, d} of the depth channel

    const int tid = threadIdx.x, lane = tid & 31;
    const int tile_x = blockIdx.x, tile_y = blockIdx.y + p.ty0;

    float2 npx, npy;
    unsigned pix_id[2];
    bool inside[2];
    bool live0 = false, live1 = false;
    float bx0 = 3.0e38f, bx1 = -3.0e38f, by0 = 3.0e38f, by1 = -3.0e38f;
    {
        float px[2], py[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            int lx, ly;
            PM::pixel(tid, k, lx, ly);
            const unsigned ux = tile_x * TILE + lx, uy = tile_y * TILE + ly;
            pix_id[k] = p.W * uy + ux;
            inside[k] = ux < (unsigned)p.W && uy < (unsigned)p.H;
            px[k] = (float)ux; py[k] = (float)uy;
            if (inside[k]) {
                const float2 so = p.subpixel_offset[pix_id[k]];
                px[k] += so.x; py[k] += so.y;
                bx0 = fminf(bx0, px[k]); bx1 = fmaxf(bx1, px[k]);
                by0 = fminf(by0, py[k]); by1 = fmaxf(by1, py[k]);
            }
        }
        live0 = inside[0]; live1 = inside[1];
        npx = make_float2(-px[0], -px[1]); npy = make_float2(-py[0], -py[1]);
    }
    const WarpBox box = warp_box_reduce(bx0, bx1, by0, by1);

    const uint2 range = p.ranges[tile_y * p.grid_x + tile_x];
    const int total = (int)(range.y - range.x);
    const int rounds = (total + PB - 1) / PB;

    float2 T = make_float2(1.f, 1.f), C0 = make_float2(0.f, 0.f), C1 = C0, C2 = C0;
    float2 Cd = C0;                       // depth channel (DEPTH only)
    uint32_t last0 = 0, last1 = 0;
    const float2 mhalf = make_float2(-0.5f, -0.5f), one = make_float2(1.f, 1.f);

    if (rounds > 0) {
        // raw record of the instance this thread stages next (register prefetch)
        float4 g = make_float4(0.f, 0.f, -1.f, -1.f), c = make_float4(0.f, 0.f, 0.f, 0.f);
        float cr = 0.f, cg = 0.f, cb = 0.f, cd = 0.f;
        auto fetch = [&](uint32_t id, bool valid) {
            if (valid) {
                const float4* src = p.rec + 2 * (size_t)id;
                g = src[0]; c = src[1];
                const float* col = p.colors + 3 * (size_t)id;
                cr = col[0]; cg = col[1]; cb = col[2];
                if constexpr (DEPTH) cd = p.depth_values[id];
            }
        };
        auto id_of = [&](int round) -> uint32_t {
            const int i = round * PB + tid;
            return (round < rounds && i < total) ? p.point_list[range.x + i] : 0u;
        };
        uint32_t id_next = id_of(0);
        fetch(id_next, tid < total);
        id_next = id_of(1);

        int toDo = total;
        for (int r = 0; r < rounds; ++r, toDo -= PB) {
            const int buf = r & 1;
            // write this round's (already loaded) record, duplicated, then start the next round's loads
            {
                FwdPairRec rec;
                rec.xy = make_float4(g.x, g.x, g.y, g.y);
                rec.ac = make_float4(c.x, c.x, c.z, c.z);
                rec.bo = make_float4(-c.y, -c.y, c.w, c.w);
                rec.rg = make_float4(cr, cr, cg, cg);
                rec.bb = make_float4(cb, cb, g.z, g.w);
                s_rec[buf][tid] = rec;
                if constexpr (DEPTH) s_dep[buf][tid] = make_float2(cd, cd);
            }
            if (r + 1 < rounds) {
                fetch(id_next, (r + 1) * PB + tid < total);
                id_next = id_of(r + 2);
            }
            // the round is visible to everyone; block-wide early-out vote (forward.cu:330-332).  One barrier per
            // round suffices: buffer `buf` is rewritten in round r+2, after the barrier of round r+1.
            const int num_done = __syncthreads_count(!(live0 || live1));
            if (num_done == THREADS) break;

            const int n = min(PB, toDo);
            const uint32_t round_base = (uint32_t)(r * PB);
            if (__any_sync(0xFFFFFFFFu, live0 || live1)) {
#pragma unroll 1
                for (int w = 0; w < PB / 32; ++w) {
                    const int jl = w * 32 + lane;
                    bool rel = false;
                    if (jl < n) {
                        const FwdPairRec& L = s_rec[buf][jl];
                        rel = box_may_touch(make_float4(L.xy.x, L.xy.z, L.bb.z, L.bb.w), box) &&
                              ellipse_may_touch(L.xy.x, L.xy.z, L.ac.x, -L.bo.x, L.ac.z, L.bo.z, box);
                    }
                    unsigned mm = __ballot_sync(0xFFFFFFFFu, rel);
                    uint32_t blended = 0;   // bit b: some pixel of the warp blended position round_base + 32 w + b
                    while (mm) {
                        const int j = w * 32 + __ffs(mm) - 1;
                        mm &= mm - 1;
                        const FwdPairRec& R = s_rec[buf][j];
                        const float4 xy = R.xy, ac = R.ac, bo = R.bo;
                        const float2 dx = add2(make_float2(xy.x, xy.y), npx), dy = add2(make_float2(xy.z, xy.w), npy);
                        const float2 t1 = mul2(make_float2(ac.x, ac.y), dx);
                        const float2 t3 = mul2(dy, mul2(make_float2(ac.z, ac.w), dy));
                        const float2 un = mul2(dy, mul2(make_float2(bo.x, bo.y), dx));     // -(B dx) dy
                        const float2 power = fma2(fma2(dx, t1, t3), mhalf, un);
                        const float2 oG = mul2(make_float2(bo.z, bo.w), make_float2(expf(power.x), expf(power.y)));
                        const float a0 = min(0.99f, oG.x), a1 = min(0.99f, oG.y);
                        const float2 test_T = mul2(T, add2(one, make_float2(-a0, -a1)));
                        const bool blend0 = live0 && !(power.x > 0.0f) && !(a0 < 1.0f / 255.0f);
                        const bool blend1 = live1 && !(power.y > 0.0f) && !(a1 < 1.0f / 255.0f);
                        const bool stop0 = blend0 && test_T.x < 0.0001f, stop1 = blend1 && test_T.y < 0.0001f;
                        live0 = live0 && !stop0;
                        live1 = live1 && !stop1;
                        const bool upd0 = blend0 && !stop0, upd1 = blend1 && !stop1;
                        if (!__any_sync(0xFFFFFFFFu, upd0 || upd1)) continue;
                        blended |= 1u << (j - w * 32);
                        const float2 alpha = make_float2(upd0 ? a0 : 0.f, upd1 ? a1 : 0.f);
                        const float4 rg = R.rg, bb = R.bb;
                        C0 = fma2(T, mul2(alpha, make_float2(rg.x, rg.y)), C0);
                        C1 = fma2(T, mul2(alpha, make_float2(rg.z, rg.w)), C1);
                        C2 = fma2(T, mul2(alpha, make_float2(bb.x, bb.y)), C2);
                        if constexpr (DEPTH) Cd = fma2(T, mul2(alpha, s_dep[buf][j]), Cd);
                        T = make_float2(upd0 ? test_T.x : T.x, upd1 ? test_T.y : T.y);
                        // 1-based position of this instance in the tile's list (forward.cu:349,382)
                        const uint32_t idx = round_base + (uint32_t)j + 1u;
                        last0 = upd0 ? idx : last0;
                        last1 = upd1 ? idx : last1;
                    }
                    if constexpr (!DISPLAY) {
                        const int word = (int)(round_base / 32) + w;
                        if (lane == 0 && word < MASK_WORDS) s_blend[tid >> 5][word] = blended;
                    }
                    if (!__any_sync(0xFFFFFFFFu, live0 || live1)) break;
                }
            }
        }
    }

    // PixelMap: warp k is 8x8 block k.  Words of batches no warp entered are copied too; they are never read.
    if constexpr (!DISPLAY) {
        __syncthreads();
        for (int i = tid; i < MASK_BLOCKS * MASK_WORDS; i += THREADS)
            *blend_mask_word(p, i / MASK_WORDS, i % MASK_WORDS) = s_blend[i / MASK_WORDS][i % MASK_WORDS];
    }

    const size_t plane = (size_t)p.H * p.W;
    const float bg0 = p.bg[0], bg1 = p.bg[1], bg2 = p.bg[2];
    const float r0 = C0.x + T.x * bg0, g0 = C1.x + T.x * bg1, b0 = C2.x + T.x * bg2;
    const float r1 = C0.y + T.y * bg0, g1 = C1.y + T.y * bg1, b1 = C2.y + T.y * bg2;
    if constexpr (DISPLAY) {
        // the depth channel's image is channel 0 of a composite of {d, d, d}, so its background term is T bg[0]
        const float rgb[2][3] = {{r0, g0, b0}, {r1, g1, b1}};
        const float tT[2] = {T.x, T.y}, dd[2] = {Cd.x + T.x * bg0, Cd.y + T.y * bg0};
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            if (!inside[k]) continue;
            float* col = p.disp_color + 3 * (size_t)pix_id[k];
            col[0] = display_value(rgb[k][0]); col[1] = display_value(rgb[k][1]); col[2] = display_value(rgb[k][2]);
            p.disp_accum[pix_id[k]] = 1.0f - tT[k];
            if constexpr (DEPTH) p.disp_depth[pix_id[k]] = dd[k];
        }
        return;
    }
    if (inside[0]) { p.final_T[pix_id[0]] = T.x; p.n_contrib[pix_id[0]] = last0; }
    if (inside[1]) { p.final_T[pix_id[1]] = T.y; p.n_contrib[pix_id[1]] = last1; }
    if (p.n_peers > 0) {
        for (int r = 0; r < p.n_peers; ++r) {
            float* img = p.peer_out[r];
            if (inside[0]) {
                img[0 * plane + pix_id[0]] = r0; img[1 * plane + pix_id[0]] = g0; img[2 * plane + pix_id[0]] = b0;
                img[3 * plane + pix_id[0]] = T.x;
            }
            if (inside[1]) {
                img[0 * plane + pix_id[1]] = r1; img[1 * plane + pix_id[1]] = g1; img[2 * plane + pix_id[1]] = b1;
                img[3 * plane + pix_id[1]] = T.y;
            }
        }
    } else {
        if (inside[0]) { p.out_color[0 * plane + pix_id[0]] = r0; p.out_color[1 * plane + pix_id[0]] = g0; p.out_color[2 * plane + pix_id[0]] = b0; }
        if (inside[1]) { p.out_color[0 * plane + pix_id[1]] = r1; p.out_color[1 * plane + pix_id[1]] = g1; p.out_color[2 * plane + pix_id[1]] = b1; }
    }
}

// ---- colour-only backward: dL/dcolour = sum over pixels of T alpha dL/dpixel -------------------------------------------
// When only the colours change (test-time appearance optimisation), the composite's gradient needs no conic, opacity or
// mean terms, and the weight of a Gaussian at a pixel is the T alpha of the forward walk.  This kernel repeats the
// packed forward's front-to-back walk with the same pair arithmetic, so T and alpha are the forward's bits, and
// replaces the colour accumulation by the accumulation of T alpha dL/dpixel per Gaussian.  A pixel blends position i
// iff i < n_contrib and the power / alpha tests pass (the position where a pixel saturates is never below n_contrib),
// so the walk needs no saturation test; below MASK_K a warp walks exactly the positions the forward's blend mask marks
// for its 8x8 block, above it the footprint culls as in the forward.  The three sums are reduced over the warp before
// the global atomics.
struct ColorGradParams {
    int W, H, grid_x, ty0;
    const uint2* ranges;
    const uint32_t* point_list;
    const float2* subpixel_offset;
    const float4* rec;
    const uint32_t* n_contrib;
    const uint32_t* blend_mask;
    const float* dL_dpix;      // [3,H,W]
    float* dL_dcolor;          // [P,3], zeroed before the launch
};

// sum of (v0, v1, v2) over the warp in 6 shuffles (a 4-value butterfly with one padding slot); lane l ends up holding the
// warp total of component 2 * bit4(l) + bit3(l) (3: padding)
__device__ __forceinline__ float butterfly3(float v0, float v1, float v2, int lane) {
    const bool h16 = lane & 16, h8 = lane & 8;
    const float w0 = (h16 ? v2 : v0) + __shfl_xor_sync(0xFFFFFFFFu, h16 ? v0 : v2, 16);
    const float w1 = (h16 ? 0.f : v1) + __shfl_xor_sync(0xFFFFFFFFu, h16 ? v1 : 0.f, 16);
    float x = (h8 ? w1 : w0) + __shfl_xor_sync(0xFFFFFFFFu, h8 ? w0 : w1, 8);
    x += __shfl_xor_sync(0xFFFFFFFFu, x, 4);
    x += __shfl_xor_sync(0xFFFFFFFFu, x, 2);
    x += __shfl_xor_sync(0xFFFFFFFFu, x, 1);
    return x;
}

__global__ void __launch_bounds__(128) render_color_grad_kernel(const __grid_constant__ ColorGradParams p) {
    using PM = PixelMap;
    constexpr int WARPS = PM::WARPS;
    constexpr int PB = 128;               // instances per round (one per thread)
    constexpr int NW = PB / 32;           // blend-mask words per round (rounds start at multiples of 32 positions)
    __shared__ __align__(16) float4 s_xy[PB];    // {x, x, y, y}
    __shared__ __align__(16) float4 s_ac[PB];    // {conic.x, conic.x, conic.z, conic.z}
    __shared__ __align__(16) float4 s_bo[PB];    // {-conic.y, -conic.y, opacity, opacity}
    __shared__ __align__(16) float4 s_geo[PB];   // {x, y, hx, hy} for the footprint culling
    __shared__ uint32_t s_id[PB];
    __shared__ uint32_t s_max[WARPS];
    __shared__ uint32_t s_mask[WARPS][NW];
    static_assert(WARPS == MASK_BLOCKS, "one warp per 8x8 blend-mask block");

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tile_x = blockIdx.x, tile_y = blockIdx.y + p.ty0;
    const int tile = tile_y * p.grid_x + tile_x;
    const size_t plane = (size_t)p.H * p.W;

    float2 npx, npy, dL0, dL1, dL2;
    uint32_t last0 = 0, last1 = 0;
    float bx0 = 3.0e38f, bx1 = -3.0e38f, by0 = 3.0e38f, by1 = -3.0e38f;
    {
        float px[2], py[2], d0[2] = {0.f, 0.f}, d1[2] = {0.f, 0.f}, d2[2] = {0.f, 0.f};
        uint32_t last[2] = {0u, 0u};
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            int lx, ly;
            PM::pixel(tid, k, lx, ly);
            const unsigned ux = tile_x * TILE + lx, uy = tile_y * TILE + ly;
            const unsigned pix_id = p.W * uy + ux;
            px[k] = (float)ux; py[k] = (float)uy;
            if (ux < (unsigned)p.W && uy < (unsigned)p.H) {
                const float2 so = p.subpixel_offset[pix_id];
                px[k] += so.x; py[k] += so.y;
                last[k] = p.n_contrib[pix_id];
                d0[k] = p.dL_dpix[pix_id]; d1[k] = p.dL_dpix[plane + pix_id]; d2[k] = p.dL_dpix[2 * plane + pix_id];
                bx0 = fminf(bx0, px[k]); bx1 = fmaxf(bx1, px[k]);
                by0 = fminf(by0, py[k]); by1 = fmaxf(by1, py[k]);
            }
        }
        npx = make_float2(-px[0], -px[1]); npy = make_float2(-py[0], -py[1]);
        dL0 = make_float2(d0[0], d0[1]); dL1 = make_float2(d1[0], d1[1]); dL2 = make_float2(d2[0], d2[1]);
        last0 = last[0]; last1 = last[1];
    }
    const WarpBox box = warp_box_reduce(bx0, bx1, by0, by1);
    const uint2 range = p.ranges[tile];
    const uint32_t warp_last = __reduce_max_sync(0xFFFFFFFFu, max(last0, last1));
    if (lane == 0) s_max[warp] = warp_last;
    __syncthreads();
    uint32_t tile_last = 0;
#pragma unroll
    for (int k = 0; k < WARPS; ++k) tile_last = max(tile_last, s_max[k]);
    const int total = (int)min(tile_last, range.y - range.x);   // nothing behind the tile's last contributor blends
    const int rounds = (total + PB - 1) / PB;
    const int comp = 2 * ((lane >> 4) & 1) + ((lane >> 3) & 1);   // component butterfly3 leaves in this lane
    const bool owner = (lane & 7) == 0 && comp < 3;

    float2 T = make_float2(1.f, 1.f);
    const float2 mhalf = make_float2(-0.5f, -0.5f), one = make_float2(1.f, 1.f);
    for (int r = 0; r < rounds; ++r) {
        const int n = min(PB, total - r * PB);
        __syncthreads();   // the previous round's staging is consumed
        if (tid < n) {
            const uint32_t id = p.point_list[range.x + r * PB + tid];
            const float4* src = p.rec + 2 * (size_t)id;
            const float4 g = src[0], c = src[1];
            s_id[tid] = id;
            s_geo[tid] = g;
            s_xy[tid] = make_float4(g.x, g.x, g.y, g.y);
            s_ac[tid] = make_float4(c.x, c.x, c.z, c.z);
            s_bo[tid] = make_float4(-c.y, -c.y, c.w, c.w);
        }
        if (tid < WARPS * NW) {            // words at or above the block's largest n_contrib may be stale: read as 0
            const int k = tid / NW, word = r * NW + tid % NW;
            uint32_t m = 0;
            if (word < MASK_WORDS && 32 * word < (int)s_max[k]) m = p.blend_mask[((size_t)tile * MASK_BLOCKS + k) * MASK_WORDS + word];
            s_mask[k][tid % NW] = m;
        }
        __syncthreads();

#pragma unroll 1
        for (int w = 0; w < PB / 32; ++w) {
            const int jl = w * 32 + lane;
            const uint32_t pos = (uint32_t)(r * PB + jl);
            bool rel = false;
            if (jl < n && pos < warp_last) {
                if (pos < (uint32_t)MASK_K) {
                    rel = (s_mask[warp][w] >> lane) & 1u;
                } else {
                    const float4 g = s_geo[jl], bo = s_bo[jl], ac = s_ac[jl];
                    rel = box_may_touch(g, box) && ellipse_may_touch(g.x, g.y, ac.x, -bo.x, ac.z, bo.z, box);
                }
            }
            unsigned mm = __ballot_sync(0xFFFFFFFFu, rel);
            while (mm) {
                const int j = w * 32 + __ffs(mm) - 1;
                mm &= mm - 1;
                const uint32_t jpos = (uint32_t)(r * PB + j);
                const float4 xy = s_xy[j], ac = s_ac[j], bo = s_bo[j];
                // the packed forward's expressions (render_fwd_packed_kernel), so that T and alpha are its bits
                const float2 dx = add2(make_float2(xy.x, xy.y), npx), dy = add2(make_float2(xy.z, xy.w), npy);
                const float2 t1 = mul2(make_float2(ac.x, ac.y), dx);
                const float2 t3 = mul2(dy, mul2(make_float2(ac.z, ac.w), dy));
                const float2 un = mul2(dy, mul2(make_float2(bo.x, bo.y), dx));
                const float2 power = fma2(fma2(dx, t1, t3), mhalf, un);
                const float2 oG = mul2(make_float2(bo.z, bo.w), make_float2(expf(power.x), expf(power.y)));
                const float a0 = min(0.99f, oG.x), a1 = min(0.99f, oG.y);
                const float2 test_T = mul2(T, add2(one, make_float2(-a0, -a1)));
                const bool upd0 = jpos < last0 && !(power.x > 0.0f) && !(a0 < 1.0f / 255.0f);
                const bool upd1 = jpos < last1 && !(power.y > 0.0f) && !(a1 < 1.0f / 255.0f);
                if (jpos >= (uint32_t)MASK_K && !__any_sync(0xFFFFFFFFu, upd0 || upd1)) continue;   // warp-uniform
                const float2 aT = mul2(make_float2(upd0 ? a0 : 0.f, upd1 ? a1 : 0.f), T);
                T = make_float2(upd0 ? test_T.x : T.x, upd1 ? test_T.y : T.y);
                const float2 c0 = mul2(aT, dL0), c1 = mul2(aT, dL1), c2 = mul2(aT, dL2);
                const float v = butterfly3(c0.x + c0.y, c1.x + c1.y, c2.x + c2.y, lane);
                if (owner) atomicAdd(p.dL_dcolor + 3 * (size_t)s_id[j] + comp, v);
            }
        }
    }
}

int launch_render_color_grad(const GsrBackwardArgs& a, const GeomState& g, const BinState& b, const ImgState& im, int ty0,
                             int ty1, cudaStream_t s) {
    ColorGradParams p;
    p.W = a.W; p.H = a.H; p.grid_x = tiles_x(a.W); p.ty0 = ty0;
    p.ranges = im.ranges; p.point_list = b.point_list;
    p.subpixel_offset = reinterpret_cast<const float2*>(a.subpixel_offset);
    p.rec = g.rec; p.n_contrib = im.n_contrib; p.blend_mask = im.blend_mask;
    p.dL_dpix = a.dL_dpix; p.dL_dcolor = a.dL_dcolor;
    if (ty1 <= ty0) return 0;
    dim3 grid(p.grid_x, ty1 - ty0, 1);
    render_color_grad_kernel<<<grid, 128, 0, s>>>(p);
    count_launches(1);
    return 0;
}

int launch_render_fwd(const GsrForwardArgs& a, const GeomState& g, const BinState& b, const ImgState& im,
                      const float* colors, int ty0, int ty1, cudaStream_t s) {
    RenderFwdParams p;
    p.W = a.W; p.H = a.H; p.grid_x = tiles_x(a.W); p.ty0 = ty0;
    p.ranges = im.ranges; p.point_list = b.point_list;
    p.subpixel_offset = reinterpret_cast<const float2*>(a.subpixel_offset);
    p.rec = g.rec; p.colors = colors; p.bg = a.background;
    p.final_T = im.final_T; p.n_contrib = im.n_contrib; p.out_color = a.out_color; p.blend_mask = im.blend_mask;
    p.peer_out = (float* const*)(a.peer_images); p.n_peers = a.n_peer_images;
    if (ty1 <= ty0) return 0;
    dim3 grid(p.grid_x, ty1 - ty0, 1);
    render_fwd_packed_kernel<false, false><<<grid, 128, 0, s>>>(p);
    count_launches(1);
    return 0;
}

// ---- display composite of an inference render ------------------------------------------------------------------------
// dist[i] = |means3D[i] - campos| in the operation order of torch.norm(means3D - campos, dim=-1) on the GPU: torch reduces
// the 3 elements with two threads (elements 0 and 2 in the first, 1 in the second) and adds the partial sums, all rounded
// products and sums (no fma), then a correctly rounded sqrt.
__global__ void __launch_bounds__(256) camera_distance_kernel(int P, const float* __restrict__ means3D,
                                                              const float* __restrict__ campos, float* __restrict__ dist) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float dx = means3D[3 * (size_t)i] - campos[0];
    const float dy = means3D[3 * (size_t)i + 1] - campos[1];
    const float dz = means3D[3 * (size_t)i + 2] - campos[2];
    dist[i] = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dz, dz)), __fmul_rn(dy, dy)));
}

int launch_camera_distance(int P, const float* means3D, const float* campos, float* dist, cudaStream_t s) {
    if (P <= 0) return 0;
    camera_distance_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, means3D, campos, dist);
    count_launches(1);
    return 0;
}

int launch_render_display(const GsrForwardArgs& a, const GsrDisplayArgs& d, const GeomState& g, const BinState& b,
                          const ImgState& im, const float* colors, const float* depth_values, cudaStream_t s) {
    RenderFwdParams p = {};
    p.W = a.W; p.H = a.H; p.grid_x = tiles_x(a.W); p.ty0 = 0;
    p.ranges = im.ranges; p.point_list = b.point_list;
    p.subpixel_offset = reinterpret_cast<const float2*>(a.subpixel_offset);
    p.rec = g.rec; p.colors = colors; p.bg = a.background;
    p.disp_color = d.out_color; p.disp_accum = d.out_accum; p.disp_depth = d.out_depth; p.depth_values = depth_values;
    dim3 grid(p.grid_x, tiles_y(a.H), 1);
    if (d.depth)
        render_fwd_packed_kernel<true, true><<<grid, 128, 0, s>>>(p);
    else
        render_fwd_packed_kernel<true, false><<<grid, 128, 0, s>>>(p);
    count_launches(1);
    return 0;
}

}  // namespace gsr
