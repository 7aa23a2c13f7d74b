// render_bwd.cu -- per-tile back-to-front re-composite producing per-Gaussian partial
// gradients dL/d{mean2D (+abs channel), conic, opacity*coef, colour}.
// Replaces renderCUDA<3> of the reference backward (backward.cu:435-606).
//
// Same per-pixel recurrence as the reference (T reconstructed by division, running
// accum_rec / last_alpha / last_color), but the accumulation is re-designed: the reference
// issues 10 global float atomics per blended (pixel, Gaussian) pair (backward.cu:568-603).
// Here all 32 lanes of a warp walk the same Gaussian in lock-step, so the 10 per-lane terms
// are summed across the warp with a multi-value shuffle butterfly (12 shuffles instead of
// 50), stored into the warp's private row of the staged Gaussian (PartRows), and a tile adds
// the rows in warp order and writes each visited Gaussian's 10 sums to HBM once, as three
// 128-bit vector reductions (red.global.add.v4.f32) into a packed 48-byte record.
// That is up to 256x fewer L2 atomics per Gaussian per tile.
//
// The walk starts at the tile's largest n_contrib instead of the end of the tile's range:
// instances behind every pixel's last contributor are skipped by the reference one by one
// (backward.cu:531-533); skipping them wholesale gives the same sums.  Below MASK_K a warp
// walks only the positions the forward's blend mask marks for its 8x8 block (common.cuh):
// for a pixel, "blends at position i in the backward" (i < n_contrib, power <= 0,
// alpha >= 1/255) is exactly "updated at position i in the forward", so no walked step is
// wasted.  Beyond MASK_K the footprint box culls as before.
//
// The |grad| channel (backward.cu:593-595) is the sum over pixels of |gx| + |gy|, so the
// absolute value is taken per lane BEFORE the warp reduction.
#include "render_common.cuh"

namespace gsr {

constexpr int RB_ACC = 12;   // floats per Gaussian in the shared / global accumulator

struct RenderBwdParams {
    int W, H, grid_x, ty0;
    const uint2* ranges;
    const uint32_t* point_list;
    const float2* subpixel_offset;
    const float* bg;
    const float4* rec;
    const float* colors;
    const float* final_T;
    const uint32_t* n_contrib;
    const float* dL_dpix;
    float* accum;   // [P][12]
    // Tile-row sharded (multi-GPU) backward fused with its reduction: instead of the local array, the per-(tile,
    // Gaussian) sums are added straight into the accumulators of ALL ranks -- one multimem.red per 16 bytes through
    // the NVSwitch multicast address `mc` (the switch applies the add to every replica), or one red per peer when
    // only peer pointers are available.  No all-reduce follows.
    float* const* peers;   // [n_peers] device array of the ranks' accumulators mapped into this process, or NULL
    int n_peers;
    float* mc;             // multicast address of the same symmetric buffer, or NULL
    unsigned char* touched;   // pull-mode reduction: touched[g] = 1 for every Gaussian this rank added to, or NULL
    const uint32_t* blend_mask;   // written by the forward (common.cuh)
};

// Stage the blend-mask words a round needs: for each warp (= 8x8 block k), the NW words from word w_lo on.  Words at or
// above the block's largest n_contrib were possibly never written by the forward, and words at or above MASK_WORDS do
// not exist: both read as 0 (their positions are culled by `pos < warp_last` or by the footprint box).
template <int WARPS, int NW>
__device__ __forceinline__ void stage_mask_words(const RenderBwdParams& p, int tile, int w_lo, const uint32_t* s_max,
                                                 uint32_t (*s_mask)[NW]) {
    const int tid = threadIdx.x;
    if (tid < WARPS * NW) {
        const int k = tid / NW, word = w_lo + tid % NW;
        uint32_t m = 0;
        if (word < MASK_WORDS && 32 * word < (int)s_max[k]) m = p.blend_mask[((size_t)tile * MASK_BLOCKS + k) * MASK_WORDS + word];
        s_mask[k][tid % NW] = m;
    }
}

// Does the warp walk staged entry jl of the round (list position pos = first_pos - jl)?  Below MASK_K: exactly when the
// forward blended that position in some pixel of the warp's block.  Above: when the footprint can reach alpha >= 1/255
// in the block (box, then ellipse; render_common.cuh).  con = {conic.x, conic.y, conic.z, opacity}.
__device__ __forceinline__ bool bwd_walks(int pos, uint32_t warp_last, int w_lo, const uint32_t* mask_words, const float4 geo,
                                          const float4 con, const WarpBox& box) {
    if ((uint32_t)pos >= warp_last) return false;
    if (pos < MASK_K) return (mask_words[(pos >> 5) - w_lo] >> (pos & 31)) & 1u;
    return box_may_touch(geo, box) && ellipse_may_touch(geo.x, geo.y, con.x, con.y, con.z, con.w, box);
}

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void multimem_red_add_v4(float* addr, float a, float b, float c, float d) {
    asm volatile("multimem.red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"l"(addr), "f"(a), "f"(b), "f"(c),
                 "f"(d) : "memory");
}
// add one Gaussian's 12-float row of sums to the accumulator(s)
template <bool PEER>
__device__ __forceinline__ void flush_row(const RenderBwdParams& p, size_t row, float4 A, float4 B, float4 C) {
    const size_t off = row * RB_ACC;
    if (PEER) {
        if (p.mc != nullptr) {
            multimem_red_add_v4(p.mc + off + 0, A.x, A.y, A.z, A.w);
            multimem_red_add_v4(p.mc + off + 4, B.x, B.y, B.z, B.w);
            multimem_red_add_v4(p.mc + off + 8, C.x, C.y, C.z, C.w);
        } else {
            for (int r = 0; r < p.n_peers; ++r) {
                float* dst = p.peers[r] + off;
                red_add_v4(dst + 0, A.x, A.y, A.z, A.w);
                red_add_v4(dst + 4, B.x, B.y, B.z, B.w);
                red_add_v4(dst + 8, C.x, C.y, C.z, C.w);
            }
        }
    } else {
        float* dst = p.accum + off;
        red_add_v4(dst + 0, A.x, A.y, A.z, A.w);
        red_add_v4(dst + 4, B.x, B.y, B.z, B.w);
        red_add_v4(dst + 8, C.x, C.y, C.z, C.w);
        if (p.touched != nullptr) p.touched[row] = 1;       // benign race: every writer stores the same value
    }
}

// Sum 10 per-lane values over the 32 lanes of the warp with a multi-value butterfly: at every step a
// lane keeps half of its values and ships the other half to its partner, so the exchange costs
// 5 + 3 + 2 + 1 + 1 = 12 shuffles instead of 10 x 5.  On return lane l holds in v[0] the warp total of
// component `slot` (returned); slots >= 10 are padding; every component is held by lanes l and l^1.
__device__ __forceinline__ int butterfly10(float (&v)[10], int lane) {
    float w[5], x[3], y[2];
    {   // xor 16: components (i, i+5)
        const bool hi = lane & 16;
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            const float send = hi ? v[i] : v[i + 5];
            const float keep = hi ? v[i + 5] : v[i];
            w[i] = keep + __shfl_xor_sync(0xFFFFFFFFu, send, 16);
        }
    }
    {   // xor 8: (0,3) (1,4) (2,-)
        const bool hi = lane & 8;
        x[0] = (hi ? w[3] : w[0]) + __shfl_xor_sync(0xFFFFFFFFu, hi ? w[0] : w[3], 8);
        x[1] = (hi ? w[4] : w[1]) + __shfl_xor_sync(0xFFFFFFFFu, hi ? w[1] : w[4], 8);
        x[2] = (hi ? 0.f : w[2]) + __shfl_xor_sync(0xFFFFFFFFu, hi ? w[2] : 0.f, 8);
    }
    {   // xor 4: (0,2) (1,-)
        const bool hi = lane & 4;
        y[0] = (hi ? x[2] : x[0]) + __shfl_xor_sync(0xFFFFFFFFu, hi ? x[0] : x[2], 4);
        y[1] = (hi ? 0.f : x[1]) + __shfl_xor_sync(0xFFFFFFFFu, hi ? x[1] : 0.f, 4);
    }
    {   // xor 2: (0,1)
        const bool hi = lane & 2;
        v[0] = (hi ? y[1] : y[0]) + __shfl_xor_sync(0xFFFFFFFFu, hi ? y[0] : y[1], 2);
    }
    v[0] += __shfl_xor_sync(0xFFFFFFFFu, v[0], 1);
    // which component did this lane end up with?
    //   bit4: +5; bit3: slots {0,1,2} -> {3,4,pad}; bit2: {0,1} -> {2,pad}; bit1: {0} -> {1}
    const int b4 = (lane >> 4) & 1, b3 = (lane >> 3) & 1, b2 = (lane >> 2) & 1, b1 = (lane >> 1) & 1;
    // index within w[0..4] after step 1, through steps 2-4
    int idx;            // position in the 5-vector w
    if (!b2) idx = b1 ? 1 : 0;       // y[0] (lo of xor 4) came from x[0]; y[1] from x[1]
    else idx = b1 ? -1 : 2;          // hi of xor 4: y[0] = x[2], y[1] = padding
    if (idx >= 0 && b3) idx = idx == 2 ? -1 : idx + 3;   // hi of xor 8: x[0] = w[3], x[1] = w[4], x[2] = padding
    return idx < 0 ? 15 : idx + 5 * b4;
}

// Per-warp private accumulator rows.  A warp visits a staged Gaussian at most once per round, so its butterfly sums go
// to its own row s_part[warp][slot] with plain stores (no shared-memory atomics, which sm_90 runs as a compare-and-swap
// loop), and bit slot of s_wrote[warp] records that the row holds this round's sums.  The flush adds the written rows
// of a slot in warp order, so the in-tile summation order is fixed.
template <int WARPS, int RB>
struct PartRows {
    float4 row[WARPS][RB][RB_ACC / 4];
    uint32_t wrote[WARPS][RB / 32];
    // sum of slot j's written rows into (a0, a1, a2); false if no warp wrote one.  One float4 column at a time, so that
    // few registers are live next to the per-pixel state.
    __device__ __forceinline__ bool sum(int j, float4& a0, float4& a1, float4& a2) const {
        unsigned writers = 0;
#pragma unroll
        for (int k = 0; k < WARPS; ++k) writers |= ((wrote[k][j >> 5] >> (j & 31)) & 1u) << k;
        a0 = column(j, 0, writers); a1 = column(j, 1, writers); a2 = column(j, 2, writers);
        return writers != 0;
    }
    __device__ __forceinline__ float4 column(int j, int c, unsigned writers) const {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
        for (; writers; writers &= writers - 1) {
            const float4 b = row[__ffs(writers) - 1][j][c];
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        return a;
    }
};

__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// ---- packed composite: 2 pixels per lane, their arithmetic written as pairs (add2 / mul2 / fma2, render_common.cuh) ----
// Both pixels of a lane share every per-Gaussian operand load and the loop control.  Every element is rounded as the
// scalar instruction, and the expressions that decide which pairs blend (power, alpha; forward.cu:353-368) are the
// forward's, fused exactly where nvcc fuses the reference's scalar expressions, so a pixel blends the positions it
// blended in the forward.
// Per-Gaussian operands are staged in shared memory already duplicated ({x, x, y, y} ...) so that one LDS.128 yields
// two ready-made broadcast pairs and no register moves are needed.
struct __align__(16) PairRec {      // 80 bytes per staged Gaussian
    float4 xy;     // {x, x, y, y}
    float4 ac;     // {conic.x, conic.x, conic.z, conic.z}
    float4 bo;     // {-conic.y, -conic.y, opacity, opacity}
    float4 rg;     // {r, r, g, g}
    float4 bk;     // {b, b, |opacity| W/2, |opacity| H/2}
};

__device__ __forceinline__ float2 lo2(const float4 v) { return make_float2(v.x, v.y); }
__device__ __forceinline__ float2 hi2(const float4 v) { return make_float2(v.z, v.w); }

// What one lane accumulates per Gaussian (summed over its pixels, then over the warp, then over the tile).
// With w = G * dL/dalpha of a blended (pixel, Gaussian) pair and d = mean2D - pixel:
//   0: sum w*dx   1: sum w*dy   2: sum |dL/dmean2D.x| + |dL/dmean2D.y|   3: sum w*dx*dx   4: sum w*dx*dy
//   5: sum w*dy*dy   6: sum w (= dL/d(opacity*coef))   7..9: sum alpha*T*dL/dpixel[ch] (= dL/dcolour)
// The reference's per-pair gradient terms (backward.cu:574-603) are linear in these moments:
//   dL/dmean2D.x = -o W/2 (A s0 + B s1)   dL/dmean2D.y = -o H/2 (C s1 + B s0)   dL/dconic = -o/2 (s3, s4, s5)
// (o = opacity*coef, (A, B, C) = conic), so the linear map is applied once per (tile, Gaussian) when the tile
// flushes its sums instead of once per pixel pair.
// (128, 9): at most 56 registers, so that 9 CTAs (36 warps) fit an SM, as the shared memory allows
template <bool PEER>
__global__ void __launch_bounds__(128, 9) render_bwd_packed_kernel(const __grid_constant__ RenderBwdParams p) {
    using PM = PixelMap;
    constexpr int THREADS = PM::THREADS;   // 128
    constexpr int WARPS = PM::WARPS;       // 4
    constexpr int PB = 64;                 // instances staged per round: four private rows of 64 slots keep 9 CTAs/SM
    __shared__ uint32_t s_id[PB];
    __shared__ __align__(16) float4 s_geo[PB];    // {x, y, hx, hy} for the per-warp culling
    __shared__ PairRec s_rec[PB];
    __shared__ PartRows<WARPS, PB> s_part;
    __shared__ uint32_t s_max[WARPS];
    constexpr int NW = PB / 32 + 1;
    __shared__ uint32_t s_mask[WARPS][NW];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tile_x = blockIdx.x, tile_y = blockIdx.y + p.ty0;
    const size_t plane = (size_t)p.H * p.W;
    const float bg0 = p.bg[0], bg1 = p.bg[1], bg2 = p.bg[2];

    // per-pixel state, pixel 0 in .x and pixel 1 in .y of every pair.  Tb = -T_final * (bg . dL/dpixel): the background
    // term of dL/dalpha is Tb / (1 - alpha) (backward.cu:576-579).  rdot / last_cd / last_alpha carry the reference's
    // accum_rec / last_color / last_alpha recurrence (backward.cu:560-572) projected on dL/dpixel: only
    // (colour - accum_rec) . dL/dpixel is ever used.
    float2 npx, npy, T, Tb, rdot, last_cd, last_alpha, dL0, dL1, dL2;
    uint32_t last_contributor[2];
    float bx0 = 3.0e38f, bx1 = -3.0e38f, by0 = 3.0e38f, by1 = -3.0e38f;
    {
        float px[2], py[2], t[2], tb[2], d0[2], d1[2], d2[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            int lx, ly;
            PM::pixel(tid, k, lx, ly);
            const unsigned ux = tile_x * TILE + lx, uy = tile_y * TILE + ly;
            const unsigned pix_id = p.W * uy + ux;
            const bool inside = ux < (unsigned)p.W && uy < (unsigned)p.H;
            px[k] = (float)ux; py[k] = (float)uy;
            t[k] = 0.f; d0[k] = d1[k] = d2[k] = 0.f;
            last_contributor[k] = 0;
            if (inside) {
                const float2 so = p.subpixel_offset[pix_id];
                px[k] += so.x; py[k] += so.y;
                t[k] = p.final_T[pix_id];
                last_contributor[k] = p.n_contrib[pix_id];
                d0[k] = p.dL_dpix[pix_id]; d1[k] = p.dL_dpix[plane + pix_id]; d2[k] = p.dL_dpix[2 * plane + pix_id];
                bx0 = fminf(bx0, px[k]); bx1 = fmaxf(bx1, px[k]);
                by0 = fminf(by0, py[k]); by1 = fmaxf(by1, py[k]);
            }
            tb[k] = -t[k] * (bg0 * d0[k] + bg1 * d1[k] + bg2 * d2[k]);
        }
        npx = make_float2(-px[0], -px[1]); npy = make_float2(-py[0], -py[1]);
        T = make_float2(t[0], t[1]); Tb = make_float2(tb[0], tb[1]);
        dL0 = make_float2(d0[0], d0[1]); dL1 = make_float2(d1[0], d1[1]); dL2 = make_float2(d2[0], d2[1]);
        rdot = last_cd = last_alpha = make_float2(0.f, 0.f);
    }
    const WarpBox box = warp_box_reduce(bx0, bx1, by0, by1);
    const uint2 range = p.ranges[tile_y * p.grid_x + tile_x];

    // warp-wide and tile-wide largest last_contributor: nothing behind it contributes
    const uint32_t warp_last = __reduce_max_sync(0xFFFFFFFFu, max(last_contributor[0], last_contributor[1]));
    if (lane == 0) s_max[warp] = warp_last;
    __syncthreads();
    uint32_t tile_last = 0;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) tile_last = max(tile_last, s_max[w]);
    const int total = (int)min(tile_last, range.y - range.x);
    const int rounds = (total + PB - 1) / PB;

    const float ddelx_dx = 0.5f * p.W, ddely_dy = 0.5f * p.H;
    const float2 mhalf = make_float2(-0.5f, -0.5f), one = make_float2(1.f, 1.f);

    // which butterfly slot this lane ends up holding is a function of the lane only
    int my_slot;
    {
        float dummy[10];
#pragma unroll
        for (int q = 0; q < 10; ++q) dummy[q] = 0.f;
        my_slot = butterfly10(dummy, lane);
    }
    const bool slot_owner = (lane & 1) == 0 && my_slot < 10;

    int toDo = total;
    for (int r = 0; r < rounds; ++r, toDo -= PB) {
        const int n = min(PB, toDo);
        // 0-based list position of staged entry j: pos(j) = first_pos - j  (walking back to front)
        const int first_pos = total - 1 - r * PB;
        const int w_lo = (first_pos - n + 1) >> 5;
        __syncthreads();
        stage_mask_words<WARPS, NW>(p, tile_y * p.grid_x + tile_x, w_lo, s_max, s_mask);
        {
            if (tid < n) {
                const uint32_t id = p.point_list[range.x + first_pos - tid];
                s_id[tid] = id;
                const float4* src = p.rec + 2 * (size_t)id;
                const float4 g = src[0], c = src[1];
                const float* col = p.colors + 3 * (size_t)id;
                const float cr = col[0], cg = col[1], cb = col[2];
                s_geo[tid] = g;
                PairRec rec;
                rec.xy = make_float4(g.x, g.x, g.y, g.y);
                rec.ac = make_float4(c.x, c.x, c.z, c.z);
                rec.bo = make_float4(-c.y, -c.y, c.w, c.w);
                rec.rg = make_float4(cr, cr, cg, cg);
                rec.bk = make_float4(cb, cb, fabsf(c.w) * ddelx_dx, fabsf(c.w) * ddely_dy);
                s_rec[tid] = rec;
            }
        }
        __syncthreads();

#pragma unroll 1
        for (int w = 0; w < PB / 32; ++w) {
            const int jl = w * 32 + lane;
            const bool rel = jl < n && bwd_walks(first_pos - jl, warp_last, w_lo, s_mask[warp], s_geo[jl],
                                                 make_float4(s_rec[jl].ac.x, -s_rec[jl].bo.x, s_rec[jl].ac.z, s_rec[jl].bo.z), box);
            unsigned mm = __ballot_sync(0xFFFFFFFFu, rel);
            uint32_t wrote = 0;
            while (mm) {
                const int j = w * 32 + __ffs(mm) - 1;
                mm &= mm - 1;
                const uint32_t pos = (uint32_t)(first_pos - j);
                const PairRec& R = s_rec[j];
                const float4 xy = R.xy, ac = R.ac, bo = R.bo;

                // power = -0.5 (A dx dx + C dy dy) - B dx dy, contracted as nvcc contracts the scalar expression:
                //   s = fma(dx, A dx, (C dy) dy);  power = fma(s, -0.5, -((B dx) dy))      (checked against the SASS)
                const float2 dx = add2(lo2(xy), npx), dy = add2(hi2(xy), npy);
                const float2 t1 = mul2(lo2(ac), dx);
                const float2 t3 = mul2(dy, mul2(hi2(ac), dy));
                const float2 un = mul2(dy, mul2(lo2(bo), dx));       // -(B dx) dy
                const float2 power = fma2(fma2(dx, t1, t3), mhalf, un);
                const float g0 = expf(power.x), g1 = expf(power.y);
                const float2 oG = mul2(hi2(bo), make_float2(g0, g1));
                const float a0 = min(0.99f, oG.x), a1 = min(0.99f, oG.y);
                // the reference visits an instance iff its position is below the pixel's n_contrib (backward.cu:529-533);
                // pixels outside the image have n_contrib = 0
                const bool act0 = pos < last_contributor[0] && !(power.x > 0.0f) && !(a0 < 1.0f / 255.0f);
                const bool act1 = pos < last_contributor[1] && !(power.y > 0.0f) && !(a1 < 1.0f / 255.0f);
                // below MASK_K some pixel of the warp blends by construction; above, the box test is only conservative
                if (pos >= (uint32_t)MASK_K && !__any_sync(0xFFFFFFFFu, act0 || act1)) continue;   // warp-uniform
                // a pair that does not blend is carried through the arithmetic below as G = alpha = 0: T, the sums and
                // the recurrence are then unchanged (the pending accum_rec update is merely applied one step early,
                // which commutes)
                const float2 G = make_float2(act0 ? g0 : 0.f, act1 ? g1 : 0.f);
                const float2 alpha = make_float2(act0 ? a0 : 0.f, act1 ? a1 : 0.f);

                const float4 rg = R.rg, bk = R.bk;
                const float2 oma = add2(one, make_float2(-alpha.x, -alpha.y));
                // T before this splat; 1 - alpha is in [0.01, 1], the approximate reciprocal is good to 1 ulp and gradients
                // are compared at 1e-3 (backward.cu:548,579 divide twice)
                const float2 inv = make_float2(rcp_approx(oma.x), rcp_approx(oma.y));
                T = mul2(T, inv);
                const float2 aT = mul2(alpha, T);
                rdot = fma2(last_alpha, add2(last_cd, make_float2(-rdot.x, -rdot.y)), rdot);
                const float2 cd = fma2(lo2(bk), dL2, fma2(hi2(rg), dL1, mul2(lo2(rg), dL0)));
                last_cd = cd;
                last_alpha = alpha;
                const float2 dL_dalpha = fma2(add2(cd, make_float2(-rdot.x, -rdot.y)), T, mul2(Tb, inv));
                const float2 wgt = mul2(G, dL_dalpha);
                const float2 wx = mul2(wgt, dx), wy = mul2(wgt, dy);
                // t1 = A wx + B wy, t2 = C wy + B wx  (lo2(bo) holds -B: the sign disappears under |.|)
                const float2 q1 = fma2(lo2(bo), wy, make_float2(-0.f, -0.f));   // -B wy
                const float2 u1 = fma2(lo2(ac), wx, make_float2(-q1.x, -q1.y));
                const float2 q2 = mul2(lo2(bo), wx);                             // -B wx
                const float2 u2 = fma2(hi2(ac), wy, make_float2(-q2.x, -q2.y));
                const float2 mxx = mul2(wx, dx), mxy = mul2(wx, dy), myy = mul2(wy, dy);
                const float2 c0 = mul2(aT, dL0), c1 = mul2(aT, dL1), c2 = mul2(aT, dL2);
                float v[10];
                v[0] = wx.x + wx.y;
                v[1] = wy.x + wy.y;
                v[2] = fmaf(fabsf(u2.x), bk.w, fabsf(u1.x) * bk.z) + fmaf(fabsf(u2.y), bk.w, fabsf(u1.y) * bk.z);
                v[3] = mxx.x + mxx.y;
                v[4] = mxy.x + mxy.y;
                v[5] = myy.x + myy.y;
                v[6] = wgt.x + wgt.y;
                v[7] = c0.x + c0.y;
                v[8] = c1.x + c1.y;
                v[9] = c2.x + c2.y;
                butterfly10(v, lane);
                if (slot_owner) reinterpret_cast<float*>(s_part.row[warp][j])[my_slot] = v[0];
                wrote |= 1u << (j - w * 32);
            }
            if (lane == 0) s_part.wrote[warp][w] = wrote;
        }
        __syncthreads();
        float4 a0, a1, a2;
        if (tid < n && s_part.sum(tid, a0, a1, a2)) {
            const bool any = (a0.x != 0.f) | (a0.y != 0.f) | (a0.z != 0.f) | (a0.w != 0.f) | (a1.x != 0.f) |
                             (a1.y != 0.f) | (a1.z != 0.f) | (a1.w != 0.f) | (a2.x != 0.f) | (a2.y != 0.f);
            if (any) {
                const PairRec& R = s_rec[tid];
                const float A = R.ac.x, C = R.ac.z, B = -R.bo.x, o = R.bo.z;
                const float gx = -o * ddelx_dx * (A * a0.x + B * a0.y);
                const float gy = -o * ddely_dy * (C * a0.y + B * a0.x);
                const float h = -0.5f * o;
                flush_row<PEER>(p, s_id[tid], make_float4(gx, gy, a0.z, h * a0.w), make_float4(h * a1.x, h * a1.y, a1.z, a1.w),
                          make_float4(a2.x, a2.y, 0.f, 0.f));
            }
        }
    }
}

int launch_render_bwd(const GsrBackwardArgs& a, const GeomState& g, const BinState& b, const ImgState& im,
                      const float* colors, BwdAccum* accum, int ty0, int ty1, cudaStream_t s, const PeerAccum* peer,
                      unsigned char* touched) {
    RenderBwdParams p;
    p.touched = touched;
    p.peers = peer ? (float* const*)(peer->peers) : nullptr;
    p.n_peers = peer ? peer->n_peers : 0;
    p.mc = peer ? reinterpret_cast<float*>(peer->multicast) : nullptr;
    p.W = a.W; p.H = a.H; p.grid_x = tiles_x(a.W); p.ty0 = ty0;
    p.ranges = im.ranges; p.point_list = b.point_list;
    p.subpixel_offset = reinterpret_cast<const float2*>(a.subpixel_offset);
    p.bg = a.background; p.rec = g.rec; p.colors = colors;
    p.final_T = im.final_T; p.n_contrib = im.n_contrib; p.dL_dpix = a.dL_dpix; p.blend_mask = im.blend_mask;
    p.accum = reinterpret_cast<float*>(accum);
    if (ty1 <= ty0) return 0;
    dim3 grid(p.grid_x, ty1 - ty0, 1);
    if (peer)   // the flush adds into every rank's accumulator
        render_bwd_packed_kernel<true><<<grid, 128, 0, s>>>(p);
    else
        render_bwd_packed_kernel<false><<<grid, 128, 0, s>>>(p);
    count_launches(1);
    return 0;
}

}  // namespace gsr
