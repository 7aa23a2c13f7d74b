/*
 * fwd_bound.c -- TEST INFRASTRUCTURE, not product code.
 *
 * fp64 oracle of the training composite AS THE KERNEL COMPUTES IT (wild-gaussians_b200/csrc/render_fwd.cu,
 * render_fwd_packed_kernel<false, false>), with an a-priori bound on how far each of the kernel's fp32 outputs can be
 * from the exact value, pixel by pixel.  Front end: oracle/fwd_exact.py.
 *
 * Inputs are the kernel's own fp32 artefacts, taken as exact values: the projected records {x, y, hx, hy, A, B, C, o},
 * colours, the sorted instance list, the tile ranges, the sub-pixel offsets, bg, W, H and an optional tile-row band.
 * The oracle does NOT cull: it walks every list position of every pixel, so a pair that the kernel's per-warp culling
 * (box_may_touch / ellipse_may_touch, render_common.cuh) drops although it blends shows up as a pixel beyond its bound.
 * Outputs:
 *   S[4][H][W]   exact (fp64) value of the three colour channels and of final_T along the nominal decisions;
 *   B[4][H][W]   bound on |kernel - S| (+inf for a pixel with more than MAX_UND undetermined decisions on a path);
 *   nc_nom       n_contrib along the nominal decisions;
 *   nc_ok        (when a tested n_contrib nc_test is given) 1 if nc_test[pixel] is the n_contrib of one of the evaluated
 *                decision combinations (the single nominal value when determined; any value up to the list length for a
 *                pixel whose bound is infinite), else 0;
 *   und[H][W]    1 if a decision of the pixel is undetermined, 2 if its bound is infinite;
 *   mbits/msure  [T][4][MASK_WORDS] the blend-mask bit of every (tile, 8x8 block, position < MASK_K) and whether it is
 *                sure: 1 if some pixel of the block blends the position under every combination, 0 if no pixel of the
 *                block blends it under any combination, unsure otherwise.
 *
 * Arithmetic up to expf is IEEE and is reproduced here bit for bit in fp32 (render_fwd.cu line numbers):
 *   px = fl(ux + so.x) (:116-119), dx = fl(x + (-px)), dy likewise (:201), t1 = fl(A dx) (:202), t3 = fl(dy fl(C dy))
 *   (:203), un = fl(dy fl((-B) dx)) (:204), power = fma(fma(dx, t1, t3), -0.5, un) (:205), all __f*_rn; so the
 *   `power > 0` decision (:209) is exact.  (debug_f64 = 1 computes px and power in fp64 instead, in oracle.c's fp64
 *   expression order, so that S can be compared with its fp64 composite.)
 * From expf on, running error analysis: every value is a pair (v, e), v the exact value (fp64), e a bound on
 * |kernel's fp32 value - v|.  Each fp32 +, x or fma adds u (|v| + e) + 2^-126 (u = 2^-24, round to nearest; 2^-126
 * covers an underflowing result), except that an operation on exact operands whose exact result is an fp32 number
 * adds nothing (it is computed exactly).  Constants:
 *   expf            2 ulp (CUDA C Programming Guide, mathematical functions: expf, maximum ulp error 2; the library is
 *                   built without -use_fast_math), 1 ulp <= 2u |x|; expf(+-0) = 1 exactly (same table);
 *   oG = fl(o G)    (:206), alpha = min(0.99f, oG) (:207): 1-Lipschitz; both sides of the clamp give exactly 0.99f
 *                   when the whole interval of oG lies above it; fminf(0.99f, NaN) = 0.99f;
 *   test_T = fl(T fl(1 - alpha)) (:208); C = fma(T, fl(alpha c), C) (:219-221); T = test_T (:223);
 *   epilogue C + T bg (:248): bounded as the uncontracted fl(C + fl(T bg)), whose bound covers the contracted
 *   fma(T, bg, C) too.
 * Decisions: alpha < 1/255f (:209) and test_T < 1e-4f (:211) are UNDETERMINED when the interval [v - e, v + e] contains
 * values on both sides of the threshold.  A pixel is then evaluated under every combination of its undetermined
 * decisions along every path (a depth-first walk that forks at each; at most MAX_UND forks on a path), and
 * B = max over the leaves of |leaf value - nominal value| + leaf bound.  A path with more forks makes the pixel's
 * bound infinite and its mask contributions unsure; those pixels are counted.
 *
 * Build: make -C oracle  (gcc -O2 -ffp-contract=off -fopenmp; the fp32 steps are explicit float / fmaf, nothing is
 * contracted by gcc).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define TILE 16
#define MASK_K 1024
#define MASK_WORDS (MASK_K / 32)
#define MASK_BLOCKS 4
#define MAX_UND 4          /* forks per path evaluated exhaustively (at most 2^4 leaves) */
#define MAX_LEAVES (1 << MAX_UND)

static const double U = 0x1p-24;
static const double TINY = 0x1p-126;
static const double EXP_ERR = 2.0 * 0x1p-23;    /* 2 ulp, relative */

typedef struct {
    double v, e;
} ve;

static inline int f32_exact(double v) { return (double)(float)v == v && (v == 0.0 || fabs(v) >= 0x1p-126); }
/* error after one fp32 rounding of a result whose exact value is v and whose inputs carry e */
static inline double fin(double v, double e) { return (e == 0.0 && f32_exact(v)) ? 0.0 : e + U * (fabs(v) + e) + TINY; }
static inline ve X(double v) { ve r = {v, 0.0}; return r; }
static inline ve neg(ve a) { ve r = {-a.v, a.e}; return r; }
static inline ve add(ve a, ve b) {
    const double v = a.v + b.v;
    ve r = {v, fin(v, a.e + b.e)};
    return r;
}
static inline ve mul(ve a, ve b) {
    const double v = a.v * b.v;
    ve r = {v, fin(v, fabs(a.v) * b.e + fabs(b.v) * a.e + a.e * b.e)};
    return r;
}
static inline ve fma_(ve a, ve b, ve c) {
    const double v = a.v * b.v + c.v;
    ve r = {v, fin(v, fabs(a.v) * b.e + fabs(b.v) * a.e + a.e * b.e + c.e)};
    return r;
}

/* the kernel's fp32 sample position fl(ux + so.x) (render_fwd.cu:116-119) */
static inline float sample_f32(int u, double so) { return (float)u + (float)so; }

/* the kernel's fp32 power of record co at sample (pxf, pyf) (render_fwd.cu:201-205) */
static inline float power_f32(const double* co, float pxf, float pyf) {
    const float x = (float)co[0], y = (float)co[1];
    const float A = (float)co[4], Bc = (float)co[5], C = (float)co[6];
    const float dx = x + (-pxf), dy = y + (-pyf);
    const float t1 = A * dx;
    const float t3 = dy * (C * dy);
    const float un = dy * ((-Bc) * dx);
    return fmaf(fmaf(dx, t1, t3), -0.5f, un);
}

/* one list position of a pixel that may blend */
typedef struct {
    uint32_t pos, g;
    int und;          /* alpha within its error of 1/255 */
    int blend;        /* nominal alpha decision */
    ve a;
} Cand;

typedef struct {
    ve T, C[3];
    uint32_t last;
    int forks, nominal;
    uint32_t bits[MASK_WORDS];
} Path;

typedef struct {
    const Cand* cd;
    int nc;
    const double *colors, *bg;
    double t_min;
    int nofork;          /* take the nominal decision everywhere (the value of a pixel whose bound is infinite) */
    int overflow, nleaves;
    double out[MAX_LEAVES][4], err[MAX_LEAVES][4];
    uint32_t last[MAX_LEAVES];
    int nominal_leaf;
    uint32_t ever[MASK_WORDS], always[MASK_WORDS];
} Walk;

static void leaf(Walk* w, const Path* p) {
    if (w->nleaves >= MAX_LEAVES) { w->overflow = 1; return; }
    const int l = w->nleaves++;
    for (int c = 0; c < 3; ++c) {
        const ve o = add(p->C[c], mul(p->T, X(w->bg[c])));
        w->out[l][c] = o.v;
        w->err[l][c] = o.e;
    }
    w->out[l][3] = p->T.v;
    w->err[l][3] = p->T.e;
    w->last[l] = p->last;
    if (p->nominal) w->nominal_leaf = l;
    for (int i = 0; i < MASK_WORDS; ++i) {
        w->ever[i] |= p->bits[i];
        w->always[i] &= p->bits[i];
    }
}

static void walk(Walk* w, int k, Path p) {
    for (; k < w->nc; ++k) {
        if (w->overflow) return;
        const Cand* q = w->cd + k;
        if (q->und && !w->nofork) {
            if (p.forks >= MAX_UND) { w->overflow = 1; return; }
            ++p.forks;
            Path sk = p;                                 /* the pair does not blend: the rest of the list from here */
            sk.nominal = p.nominal && !q->blend;
            walk(w, k + 1, sk);
            if (w->overflow) return;
            p.nominal = p.nominal && q->blend;           /* the pair blends: continue below */
        } else if (!q->blend) {
            continue;
        }
        /* blend the pair unless the pixel stops here */
        const ve om = add(X(1.0), neg(q->a));
        const ve tT = mul(p.T, om);
        const int stop_nom = tT.v < w->t_min;
        const int und_s = (tT.v - tT.e < w->t_min) && !(tT.v + tT.e < w->t_min) && !w->nofork;
        if (und_s) {
            if (p.forks >= MAX_UND) { w->overflow = 1; return; }
            ++p.forks;
            Path st = p;                                 /* the stopping branch ends the path */
            st.nominal = p.nominal && stop_nom;
            leaf(w, &st);
            if (w->overflow) return;
            p.nominal = p.nominal && !stop_nom;
        } else if (stop_nom) {
            leaf(w, &p);
            return;
        }
        const double* col = w->colors + 3 * (size_t)q->g;
        for (int c = 0; c < 3; ++c) p.C[c] = fma_(p.T, mul(q->a, X(col[c])), p.C[c]);
        p.T = tT;
        p.last = q->pos + 1;
        if (q->pos < MASK_K) p.bits[q->pos >> 5] |= 1u << (q->pos & 31);
    }
    leaf(w, &p);
}

/* returns the number of pixels with an infinite bound; stats[0] = undetermined pixels, stats[1] = blended pairs
 * (nominal), stats[2] = undetermined decisions over all candidates (alpha tests only). */
long long fwd_bound(int W, int H, int ty0, int ty1, const uint32_t* ranges, const uint32_t* point_list,
                    const double* subpixel_offset, const double* bg, const double* rec, const double* colors,
                    double alpha_max, double alpha_min, double t_min, int debug_f64, double* S, double* Bnd,
                    uint32_t* nc_nom, const uint32_t* nc_test, uint8_t* nc_ok, uint8_t* und, uint32_t* mbits, uint32_t* msure,
                    double* stats) {
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    if (ty0 == 0 && ty1 == 0) ty1 = gy;
    const size_t plane = (size_t)W * H;
    uint32_t maxlen = 0;
    for (int t = 0; t < gx * gy; ++t) {
        const uint32_t l = ranges[2 * t + 1] - ranges[2 * t];
        if (l > maxlen) maxlen = l;
    }
    long long overflow = 0, n_und = 0, n_blend = 0, n_und_a = 0;
#pragma omp parallel reduction(+ : overflow, n_und, n_blend, n_und_a)
    {
        Cand* cd = malloc(sizeof(Cand) * (maxlen > 0 ? maxlen : 1));
        Walk* w = malloc(sizeof(Walk));
#pragma omp for collapse(2) schedule(dynamic, 1)
        for (int ty = ty0; ty < ty1; ++ty)
            for (int tx = 0; tx < gx; ++tx) {
                const int t = ty * gx + tx;
                const uint32_t r0 = ranges[2 * t], r1 = ranges[2 * t + 1];
                const uint32_t len = r1 - r0;
                uint32_t blk_ever[MASK_BLOCKS][MASK_WORDS], blk_always[MASK_BLOCKS][MASK_WORDS];
                memset(blk_ever, 0, sizeof(blk_ever));
                memset(blk_always, 0, sizeof(blk_always));
                for (int ly = 0; ly < TILE; ++ly)
                    for (int lx = 0; lx < TILE; ++lx) {
                        const int ux = tx * TILE + lx, uy = ty * TILE + ly;
                        if (ux >= W || uy >= H) continue;
                        const size_t pid = (size_t)W * uy + ux;
                        const int blk = (lx >= 8) + 2 * (ly >= 8);
                        const float pxf = sample_f32(ux, subpixel_offset[2 * pid]);
                        const float pyf = sample_f32(uy, subpixel_offset[2 * pid + 1]);
                        const double pxd = ux + subpixel_offset[2 * pid], pyd = uy + subpixel_offset[2 * pid + 1];
                        int nc = 0;
                        for (uint32_t k = 0; k < len; ++k) {
                            const uint32_t g = point_list[r0 + k];
                            const double* co = rec + 8 * (size_t)g;
                            double pw;
                            if (debug_f64) {
                                /* oracle.c's pair_power in its fp64 build */
                                const double dx = co[0] - pxd, dy = co[1] - pyd;
                                const double s = (co[4] * dx) * dx + (co[6] * dy) * dy, u = (co[5] * dx) * dy;
                                pw = s * -0.5 - u;
                            } else {
                                pw = (double)power_f32(co, pxf, pyf);
                            }
                            if (pw > 0.0) continue;
                            Cand q;
                            q.pos = k;
                            q.g = g;
                            ve oG;
                            if (isnan(pw)) {
                                oG = X(NAN);
                            } else if (pw == 0.0 && !debug_f64) {
                                oG = mul(X(co[7]), X(1.0));
                            } else {
                                const double G = exp(pw);
                                const ve Gv = {G, debug_f64 ? 0.0 : EXP_ERR * G + TINY};
                                oG = mul(X(co[7]), Gv);
                            }
                            if (isnan(oG.v)) {
                                q.a = X(alpha_max);
                            } else if (oG.v - oG.e >= alpha_max) {
                                q.a = X(alpha_max);
                            } else {
                                q.a.v = fmin(alpha_max, oG.v);
                                q.a.e = oG.e;
                            }
                            q.blend = !(q.a.v < alpha_min);
                            q.und = (q.a.v - q.a.e < alpha_min) && !(q.a.v + q.a.e < alpha_min);
                            if (!q.blend && !q.und) continue;
                            n_und_a += q.und;
                            cd[nc++] = q;
                        }
                        memset(w, 0, sizeof(Walk));
                        w->cd = cd;
                        w->nc = nc;
                        w->colors = colors;
                        w->bg = bg;
                        w->t_min = t_min;
                        w->nominal_leaf = -1;
                        for (int i = 0; i < MASK_WORDS; ++i) w->always[i] = 0xFFFFFFFFu;
                        Path p;
                        memset(&p, 0, sizeof(p));
                        p.T = X(1.0);
                        for (int c = 0; c < 3; ++c) p.C[c] = X(0.0);
                        p.nominal = 1;
                        walk(w, 0, p);
                        const int nl = w->nleaves;
                        if (w->overflow || w->nominal_leaf < 0) {
                            ++overflow;
                            und[pid] = 2;
                            /* value: the walk along the nominal decisions, bound infinite, every mask bit unsure */
                            w->nofork = 1;
                            w->nleaves = 0;
                            w->overflow = 0;
                            walk(w, 0, p);
                            w->nofork = 0;
                            for (int c = 0; c < 4; ++c) {
                                S[c * plane + pid] = w->out[0][c];
                                Bnd[c * plane + pid] = INFINITY;
                            }
                            nc_nom[pid] = w->last[0];
                            if (nc_test) nc_ok[pid] = nc_test[pid] <= len;
                            for (int i = 0; i < MASK_WORDS; ++i) blk_ever[blk][i] = 0xFFFFFFFFu;
                            continue;
                        }
                        const int nm = w->nominal_leaf;
                        for (int c = 0; c < 4; ++c) {
                            double b = 0.0;
                            for (int l = 0; l < nl; ++l) {
                                const double d = fabs(w->out[l][c] - w->out[nm][c]) + w->err[l][c];
                                if (d > b) b = d;
                            }
                            S[c * plane + pid] = w->out[nm][c];
                            Bnd[c * plane + pid] = b;
                        }
                        nc_nom[pid] = w->last[nm];
                        if (nc_test) {
                            int ok = 0;
                            for (int l = 0; l < nl; ++l) ok |= w->last[l] == nc_test[pid];
                            nc_ok[pid] = (uint8_t)ok;
                        }
                        und[pid] = nl > 1;
                        n_und += nl > 1;
                        for (int k = 0; k < nc; ++k) n_blend += cd[k].blend && cd[k].pos < w->last[nm];
                        for (int i = 0; i < MASK_WORDS; ++i) {
                            blk_ever[blk][i] |= w->ever[i];
                            blk_always[blk][i] |= w->always[i];
                        }
                    }
                for (int b = 0; b < MASK_BLOCKS; ++b)
                    for (int i = 0; i < MASK_WORDS; ++i) {
                        const size_t o = ((size_t)t * MASK_BLOCKS + b) * MASK_WORDS + i;
                        mbits[o] = blk_always[b][i];
                        msure[o] = blk_always[b][i] | ~blk_ever[b][i];
                    }
            }
        free(cd);
        free(w);
    }
    stats[0] = (double)n_und;
    stats[1] = (double)n_blend;
    stats[2] = (double)n_und_a;
    return overflow;
}

/* The fp32 power the oracle evaluates (sample_f32, power_f32: the code fwd_bound walks with) for n (pixel, Gaussian)
 * pairs: record g[i] at pixel (ux[i], uy[i]) with sub-pixel offset so[2 i], so[2 i + 1].  For comparison with other
 * restatements of the kernel's expression (tests/test_forward_exact.py). */
void fwd_pair_power(long long n, const double* rec, const uint32_t* g, const int32_t* ux, const int32_t* uy,
                    const double* so, float* out) {
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; ++i)
        out[i] = power_f32(rec + 8 * (size_t)g[i], sample_f32(ux[i], so[2 * i]), sample_f32(uy[i], so[2 * i + 1]));
}
