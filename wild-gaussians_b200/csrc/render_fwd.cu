// render_fwd.cu -- per-tile front-to-back alpha compositing.
// Replaces renderCUDA<3> of the reference (forward.cu:273-395).
//
// One CTA per 16x16 tile; a thread owns PPT pixels, a warp a compact pixel block (render_common.cuh).
// The tile's slice of the sorted instance list is consumed in rounds of 256 instances; each round's
// 32-byte projected records and colours are gathered into shared memory with asynchronous copies
// (cp.async / LDGSTS, no register staging) into a double buffer, two rounds of Gaussian ids ahead, so
// the gather of round r+1 overlaps the blending of round r.  Colours are staged too (the reference
// fetches them from global memory inside the blend loop, forward.cu:376).
//
// Per-warp culling: before blending a round, every lane tests 8 of the 256 staged Gaussians against the
// bounding box of the warp's sample positions using the conservative footprint extents computed in
// preprocess_fwd.cu; eight ballots give the warp a 256-bit mask and only the set bits are blended.
// The skipped (pixel, Gaussian) pairs are pairs the reference rejects with alpha < 1/255
// (forward.cu:365), so the image, final_T and n_contrib are unchanged; `contributor` is derived from
// the position in the list, not counted, so it still counts every instance like forward.cu:349.
//
// Numerics contract (SURVEY.md 8a note N3): the expression shapes of power / alpha / test_T / the
// colour accumulation are exactly the reference's (forward.cu:353-378,393), and expf is the accurate
// one, so the three discontinuous tests (power > 0, alpha < 1/255, T(1-alpha) < 1e-4) take the same
// branch and n_contrib / pixels match bit for bit.
#include "render_common.cuh"
#include <cstdlib>

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
    // multi-GPU: the band is stored into the [4,H,W] images (colour + final transmittance) of ALL ranks through
    // peer-mapped pointers (image all-gather fused into the composite's epilogue); NULL / 0 = local out_color only
    float* const* peer_out;
    int n_peers;
};

template <int PPT>
__global__ void __launch_bounds__(PixelMap<PPT>::THREADS) render_fwd_kernel(const __grid_constant__ RenderFwdParams p) {
    using PM = PixelMap<PPT>;
    constexpr int THREADS = PM::THREADS;
    __shared__ __align__(16) float4 s_geo[2][RT_BATCH];   // {x, y, hx, hy}
    __shared__ __align__(16) float4 s_con[2][RT_BATCH];   // {conic.x, conic.y, conic.z, opacity}
    __shared__ __align__(16) float4 s_col[2][RT_BATCH];   // {r, g, b, -}

    const int tid = threadIdx.x, lane = tid & 31;
    const int tile_x = blockIdx.x, tile_y = blockIdx.y + p.ty0;

    float2 pixf[PPT];
    unsigned pix_id[PPT];
    bool inside[PPT];
    unsigned live = 0;          // bit k set: pixel k still compositing
    float bx0 = 3.0e38f, bx1 = -3.0e38f, by0 = 3.0e38f, by1 = -3.0e38f;
#pragma unroll
    for (int k = 0; k < PPT; ++k) {
        int lx, ly;
        PM::pixel(tid, k, lx, ly);
        const unsigned px = tile_x * TILE + lx, py = tile_y * TILE + ly;
        pix_id[k] = p.W * py + px;
        inside[k] = px < (unsigned)p.W && py < (unsigned)p.H;
        pixf[k] = {(float)px, (float)py};
        if (inside[k]) {
            const float2 so = p.subpixel_offset[pix_id[k]];
            pixf[k].x += so.x;
            pixf[k].y += so.y;
            live |= 1u << k;
            bx0 = fminf(bx0, pixf[k].x); bx1 = fmaxf(bx1, pixf[k].x);
            by0 = fminf(by0, pixf[k].y); by1 = fmaxf(by1, pixf[k].y);
        }
    }
    const WarpBox box = warp_box_reduce(bx0, bx1, by0, by1);

    const uint2 range = p.ranges[tile_y * p.grid_x + tile_x];
    const int total = (int)(range.y - range.x);
    const int rounds = (total + RT_BATCH - 1) / RT_BATCH;

    // gather of one round into buffer `buf`; ids were loaded one iteration earlier
    auto stage = [&](int buf, int round, const uint32_t (&ids)[PPT]) {
#pragma unroll
        for (int q = 0; q < PPT; ++q) {
            const int slot = q * THREADS + tid;
            if (round * RT_BATCH + slot < total) {
                const float4* src = p.rec + 2 * (size_t)ids[q];
                cp_async_16(&s_geo[buf][slot], src);
                cp_async_16(&s_con[buf][slot], src + 1);
                const float* c = p.colors + 3 * (size_t)ids[q];
                float* cdst = reinterpret_cast<float*>(&s_col[buf][slot]);
                cp_async_4(cdst, c);
                cp_async_4(cdst + 1, c + 1);
                cp_async_4(cdst + 2, c + 2);
            }
        }
    };
    auto load_ids = [&](int round, uint32_t (&ids)[PPT]) {
#pragma unroll
        for (int q = 0; q < PPT; ++q) {
            const int i = round * RT_BATCH + q * THREADS + tid;
            ids[q] = (round < rounds && i < total) ? p.point_list[range.x + i] : 0u;
        }
    };

    float T[PPT], C0[PPT], C1[PPT], C2[PPT];
    uint32_t last_contributor[PPT];
#pragma unroll
    for (int k = 0; k < PPT; ++k) { T[k] = 1.0f; C0[k] = C1[k] = C2[k] = 0.f; last_contributor[k] = 0; }

    if (rounds > 0) {
        uint32_t ids[PPT];
        load_ids(0, ids);
        stage(0, 0, ids);
        cp_async_commit();
        load_ids(1, ids);

        int toDo = total;
        for (int r = 0; r < rounds; ++r, toDo -= RT_BATCH) {
            const int buf = r & 1;
            // this round's data has landed (for this thread) ...
            cp_async_wait<0>();
            // ... and for everyone; also the block-wide early-out vote (forward.cu:330-332)
            const int num_done = __syncthreads_count(live == 0);
            if (num_done == THREADS) break;
            // next round's gather overlaps this round's blending
            if (r + 1 < rounds) {
                stage(buf ^ 1, r + 1, ids);
                cp_async_commit();
                load_ids(r + 2, ids);
            }

            const int n = min(RT_BATCH, toDo);
            const uint32_t round_base = (uint32_t)(r * RT_BATCH);
            if (__any_sync(0xFFFFFFFFu, live != 0)) {
                // which of the staged Gaussians can touch this warp's pixels?  32 at a time: one ballot, then only
                // the set bits are blended
#pragma unroll 1
                for (int w = 0; w < RT_BATCH / 32; ++w) {
                    const int jl = w * 32 + lane;
                    unsigned mm = __ballot_sync(0xFFFFFFFFu, jl < n && box_may_touch(s_geo[buf][jl], box));
                    while (mm) {
                        const int j = w * 32 + __ffs(mm) - 1;
                        mm &= mm - 1;
                        const float4 geo = s_geo[buf][j];
                        const float4 con_o = s_con[buf][j];
#pragma unroll
                        for (int k = 0; k < PPT; ++k) {
                            if (!(live & (1u << k))) continue;
                            const float2 xy = {geo.x, geo.y};
                            const float2 d = {xy.x - pixf[k].x, xy.y - pixf[k].y};
                            const float power = -0.5f * (con_o.x * d.x * d.x + con_o.z * d.y * d.y) - con_o.y * d.x * d.y;
                            if (power > 0.0f) continue;

                            const float alpha = min(0.99f, con_o.w * expf(power));
                            if (alpha < 1.0f / 255.0f) continue;
                            const float test_T = T[k] * (1 - alpha);
                            if (test_T < 0.0001f) {
                                live &= ~(1u << k);
                                continue;
                            }
                            const float4 col = s_col[buf][j];
                            C0[k] += col.x * alpha * T[k];
                            C1[k] += col.y * alpha * T[k];
                            C2[k] += col.z * alpha * T[k];
                            T[k] = test_T;
                            // 1-based position of this instance in the tile's list (forward.cu:349,382)
                            last_contributor[k] = round_base + (uint32_t)j + 1u;
                        }
                    }
                    if (!__any_sync(0xFFFFFFFFu, live != 0)) break;
                }
            }
            // everyone is finished with `buf` before round r+2 is staged into it
            __syncthreads();
        }
        cp_async_wait<0>();
    }

    const size_t plane = (size_t)p.H * p.W;
    const float bg0 = p.bg[0], bg1 = p.bg[1], bg2 = p.bg[2];
#pragma unroll
    for (int k = 0; k < PPT; ++k) {
        if (inside[k]) {
            p.final_T[pix_id[k]] = T[k];
            p.n_contrib[pix_id[k]] = last_contributor[k];
            p.out_color[0 * plane + pix_id[k]] = C0[k] + T[k] * bg0;
            p.out_color[1 * plane + pix_id[k]] = C1[k] + T[k] * bg1;
            p.out_color[2 * plane + pix_id[k]] = C2[k] + T[k] * bg2;
        }
    }
}

// ---- packed variant: 2 pixels per lane, their arithmetic written as pairs (add2 / mul2 / fma2) ----------------
// (see render_bwd.cu: both pixels of a lane share every per-Gaussian operand load and the loop control.)  Every element of a pair goes through the same
// IEEE operations, in the same order, as the scalar kernel above -- power = fma(fma(dx, A dx, (C dy) dy), -0.5,
// -((B dx) dy)), alpha = min(0.99, o expf(power)), test_T = T (1 - alpha), C = fma(T, alpha c, C) -- so pixels,
// final_T and n_contrib are bit-identical.  A pair that does not blend is carried as alpha = 0, which leaves C and T
// unchanged exactly.
// Staging: one instance per thread and round; the raw records travel through registers (loads of round r+1 are
// issued before round r is blended) and are written to shared memory already duplicated ({x, x, y, y}, ...), so one
// LDS.128 yields two ready-made broadcast pairs.
struct __align__(16) FwdPairRec {     // 80 bytes
    float4 xy;     // {x, x, y, y}
    float4 ac;     // {conic.x, conic.x, conic.z, conic.z}
    float4 bo;     // {-conic.y, -conic.y, opacity, opacity}
    float4 rg;     // {r, r, g, g}
    float4 bb;     // {b, b, -, -}
};

__global__ void __launch_bounds__(128) render_fwd_packed_kernel(const __grid_constant__ RenderFwdParams p) {
    using PM = PixelMap<2>;
    constexpr int THREADS = 128;
    constexpr int PB = 128;               // instances per round
    __shared__ __align__(16) float4 s_geo[2][PB];      // {x, y, hx, hy} for the per-warp culling
    __shared__ FwdPairRec s_rec[2][PB];

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
    uint32_t last0 = 0, last1 = 0;
    const float2 mhalf = make_float2(-0.5f, -0.5f), one = make_float2(1.f, 1.f);

    if (rounds > 0) {
        // raw record of the instance this thread stages next (register prefetch)
        float4 g = make_float4(0.f, 0.f, -1.f, -1.f), c = make_float4(0.f, 0.f, 0.f, 0.f);
        float cr = 0.f, cg = 0.f, cb = 0.f;
        auto fetch = [&](uint32_t id, bool valid) {
            if (valid) {
                const float4* src = p.rec + 2 * (size_t)id;
                g = src[0]; c = src[1];
                const float* col = p.colors + 3 * (size_t)id;
                cr = col[0]; cg = col[1]; cb = col[2];
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
            s_geo[buf][tid] = g;
            {
                FwdPairRec rec;
                rec.xy = make_float4(g.x, g.x, g.y, g.y);
                rec.ac = make_float4(c.x, c.x, c.z, c.z);
                rec.bo = make_float4(-c.y, -c.y, c.w, c.w);
                rec.rg = make_float4(cr, cr, cg, cg);
                rec.bb = make_float4(cb, cb, 0.f, 0.f);
                s_rec[buf][tid] = rec;
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
                    unsigned mm = __ballot_sync(0xFFFFFFFFu, jl < n && box_may_touch(s_geo[buf][jl], box));
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
                        const float2 alpha = make_float2(upd0 ? a0 : 0.f, upd1 ? a1 : 0.f);
                        const float4 rg = R.rg, bb = R.bb;
                        C0 = fma2(T, mul2(alpha, make_float2(rg.x, rg.y)), C0);
                        C1 = fma2(T, mul2(alpha, make_float2(rg.z, rg.w)), C1);
                        C2 = fma2(T, mul2(alpha, make_float2(bb.x, bb.y)), C2);
                        T = make_float2(upd0 ? test_T.x : T.x, upd1 ? test_T.y : T.y);
                        // 1-based position of this instance in the tile's list (forward.cu:349,382)
                        const uint32_t idx = round_base + (uint32_t)j + 1u;
                        last0 = upd0 ? idx : last0;
                        last1 = upd1 ? idx : last1;
                    }
                    if (!__any_sync(0xFFFFFFFFu, live0 || live1)) break;
                }
            }
        }
    }

    const size_t plane = (size_t)p.H * p.W;
    const float bg0 = p.bg[0], bg1 = p.bg[1], bg2 = p.bg[2];
    const float r0 = C0.x + T.x * bg0, g0 = C1.x + T.x * bg1, b0 = C2.x + T.x * bg2;
    const float r1 = C0.y + T.y * bg0, g1 = C1.y + T.y * bg1, b1 = C2.y + T.y * bg2;
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

#ifndef GSR_FWD_PPT
#define GSR_FWD_PPT 1     // default pixels per thread; GSR_FWD_PPT in the environment overrides (tuning aid)
#endif

static int fwd_ppt() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("GSR_FWD_PPT");
        v = e ? atoi(e) : GSR_FWD_PPT;
        if (v != 1 && v != 2 && v != 4) v = GSR_FWD_PPT;
    }
    return v;
}

int launch_render_fwd(const GsrForwardArgs& a, const GeomState& g, const BinState& b, const ImgState& im,
                      const float* colors, int ty0, int ty1, cudaStream_t s) {
    RenderFwdParams p;
    p.W = a.W; p.H = a.H; p.grid_x = tiles_x(a.W); p.ty0 = ty0;
    p.ranges = im.ranges; p.point_list = b.point_list;
    p.subpixel_offset = reinterpret_cast<const float2*>(a.subpixel_offset);
    p.rec = g.rec; p.colors = colors; p.bg = a.background;
    p.final_T = im.final_T; p.n_contrib = im.n_contrib; p.out_color = a.out_color;
    p.peer_out = (float* const*)(a.peer_images); p.n_peers = a.n_peer_images;
    if (ty1 <= ty0) return 0;
    dim3 grid(p.grid_x, ty1 - ty0, 1);
    static int packed = -1;
    if (packed < 0) {
        const char* e = getenv("GSR_FWD_PACKED");     // tuning aid: 1 = 2 pixels/lane in paired fp32 instructions
        packed = e ? atoi(e) : 1;
    }
    if (packed || p.n_peers > 0) {      // the fused all-gather epilogue exists in the packed kernel only
        render_fwd_packed_kernel<<<grid, 128, 0, s>>>(p);
        count_launches(1);
        return 0;
    }
    switch (fwd_ppt()) {
        case 1: render_fwd_kernel<1><<<grid, PixelMap<1>::THREADS, 0, s>>>(p); break;
        case 4: render_fwd_kernel<4><<<grid, PixelMap<4>::THREADS, 0, s>>>(p); break;
        default: render_fwd_kernel<2><<<grid, PixelMap<2>::THREADS, 0, s>>>(p); break;
    }
    count_launches(1);
    return 0;
}

}  // namespace gsr
