/*
 * bwd_bound.c -- TEST INFRASTRUCTURE, not product code.
 *
 * fp64 oracle of the backward composite AS THE KERNEL COMPUTES IT (wild-gaussians_b200/csrc/render_bwd.cu,
 * render_bwd_packed_kernel), with an a-priori bound on how far the kernel's fp32 accumulator can be from the exact
 * value, entry by entry.  Front end: oracle/bwd_exact.py.
 *
 * Inputs are the kernel's own fp32 forward artefacts, taken as exact values: the projected records
 * {x, y, hx, hy, A, B, C, o}, colours, the sorted instance list, the tile ranges, n_contrib, the sub-pixel offsets,
 * bg and dL/dpix.  Outputs, per Gaussian, in the layout of the kernel's accumulator (slots 0..9 of its 12):
 *   S[P][10]   exact (fp64) value: 0 dmean2D.x, 1 dmean2D.y, 2 |.| channel, 3..5 dconic (x, y, w), 6 sum G dL/dalpha,
 *              7..9 dcolour;
 *   B[P][10]   bound on |kernel - S| (+inf for the Gaussians of a pixel with more than MAX_UND undetermined pairs);
 *   M[P][10]   magnitude scale: the per-pair terms' absolute values summed through the absolute flush conversion
 *              (>= sum of |per-pair gradient|), for relative comparisons;
 *   und[P]     1 if a pair of the Gaussian is undetermined (a blend decision within its error of the threshold),
 *              2 if the Gaussian's bound is +inf.
 *
 * Error model: running error analysis over the kernel's expression tree.  Every value is a pair (v, e): v is the
 * exact value (fp64), e bounds |kernel's fp32 value - v|.  Each fp32 +, x or fma adds u (|v| + e) + 2^-126
 * (u = 2^-24, round to nearest; 2^-126 covers an underflowing result); products carry the second-order term e_a e_b,
 * so the bound is not only first order.  Constants:
 *   expf            2 ulp (CUDA C Programming Guide, mathematical functions: expf, maximum ulp error 2; the library is
 *                   built without -use_fast_math), 1 ulp <= 2u |x|;
 *   rcp.approx.ftz  1 ulp (PTX ISA, rcp.approx.f32: "maximum ulp error is 1 across the full range"), used at
 *                   render_bwd.cu:363 on 1 - alpha in [0.01, 1] (no subnormals);
 *   min(0.99f, .)   1-Lipschitz: the kink moves alpha by no more than its argument's error, and nothing downstream
 *                   depends on which side was taken (the kernel uses G, not d alpha / dG), so it is no decision.
 * Structure (render_bwd.cu line numbers):
 *   * T: the forward's test_T = T (1 - alpha) (render_fwd.cu:208) and the backward's 1 - alpha (:360) are the same
 *     fp32 bits, so their roundings cancel between final_T and the divisions T = T rcp(1 - alpha) (:363-364).  The
 *     kernel's T before splat i is  prod_{j<i} (1 - alpha_j)  times  (1 + d) with
 *       |d| <= expm1( sum_{j<i} (e_alpha_j / (1 - alpha_j) + u)  +  n u  +  sum_{j>=i} (u + 2u) )
 *     over the pixel's n blended splats j: the earlier splats' 1 - alpha and its rounding, the forward's n multiplies,
 *     one multiply and one reciprocal per division.  Pairs that do not blend run through the arithmetic with alpha = 0
 *     and G = 0 (:356-357): T rcp(1) = T, and every term is an exact zero.
 *   * Tb rcp(1 - alpha_i) (:262, :370) = -T_final / (1 - alpha_i) (bg . dL): the i-th factor of final_T cancels, the
 *     others and their roundings remain, plus the multiplies at :262 and :370 and the reciprocal.
 *   * rdot / last_cd / last_alpha (:366-369) are carried as (v, e) pairs through the kernel's fma; dL/dalpha (:370),
 *     wgt (:371), wx, wy (:372), u1, u2 (:374-377), the |.| term (:383), the moments (:378) and alpha T dL (:365, :379)
 *     likewise.
 *   * Inside a tile each slot is a sum over pixels: a pair add (:381-390), the 5-level butterfly (:116-142) and the
 *     PartRows sum of at most 4 warp rows from zero in warp order (:171-178): a tree of depth 1 + 5 + 3 = 9, so the
 *     sum adds gamma_9 sum |term| (terms at their kernel values, i.e. |v| + e).  (The colour-only walk,
 *     render_fwd.cu:430-434, computes the same alpha T dL with T multiplied forward -- an error no larger than the
 *     division's -- and adds each warp's butterfly sum with an atomic: depth 6, 4 partial sums per tile.)
 *   * The flush (:403-409) turns the tile's moments into gradients: gx = -o W/2 (A s0 + B s1),
 *     gy = -o H/2 (C s1 + B s0), h = -o/2 times s3..s5.  Its bound comes from the tile's moments and their bounds,
 *     which is where the cancellation of a Gaussian's moments shows up.  Any contraction nvcc picks rounds no more
 *     often than the two products, the sum and the two multiplies bounded here.
 *   * Across tiles red.global.add.v4.f32 (:79-81, :104-107) adds the rows of the k tiles that flush the Gaussian onto
 *     a zeroed accumulator in some order: gamma_k sum |row| (rows at their kernel values).
 *   The fp64 evaluation of the exact value itself errs by about 2^-53 per operation, 2^-29 of each u term above.
 * Decisions: the kernel blends a pair iff pos < n_contrib (exact integers) and !(power > 0) and !(alpha < 1/255f)
 * (:349-350).  A pair is UNDETERMINED when power or alpha lies within its bound of the threshold; the pixel is then
 * evaluated under every combination of its undetermined pairs (up to MAX_UND of them), and the largest difference to
 * the nominal evaluation is added to the bound of every slot the pixel feeds -- the earlier splats' rdot and T terms
 * and the background term included, since each evaluation recomputes T_final and the recurrence.  A pixel with more
 * undetermined pairs gives every Gaussian it could blend an infinite bound; those are counted.
 * n_contrib is an input, not re-decided.
 *
 * Build: make -C oracle  (gcc -O2 -ffp-contract=off -fopenmp; fp64 only, no fused operations of gcc's own).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define TILE 16
#define NS 10            /* accumulator slots checked (the kernel's 12 minus 2 padding) */
#define MAX_UND 4        /* undetermined pairs per pixel evaluated exhaustively (2^4 evaluations) */

static const double U = 0x1p-24;
static const double TINY = 0x1p-126;
static const double EXP_ERR = 2.0 * 0x1p-23;    /* 2 ulp, relative */
static const double RCP_ERR = 1.0 * 0x1p-23;    /* 1 ulp, relative */

static double gam(double n) { return n * U / (1.0 - n * U); }

typedef struct {
    double v, e;
} ve;

static inline double rnd(double v, double e) { return U * (fabs(v) + e) + TINY; }
static inline ve X(double v) { ve r = {v, 0.0}; return r; }
static inline ve neg(ve a) { ve r = {-a.v, a.e}; return r; }
static inline ve absv(ve a) { ve r = {fabs(a.v), a.e}; return r; }
static inline ve add(ve a, ve b) {
    const double v = a.v + b.v, e = a.e + b.e;
    ve r = {v, e + rnd(v, e)};
    return r;
}
static inline ve mul(ve a, ve b) {
    const double v = a.v * b.v, e = fabs(a.v) * b.e + fabs(b.v) * a.e + a.e * b.e;
    ve r = {v, e + rnd(v, e)};
    return r;
}
static inline ve fma_(ve a, ve b, ve c) {
    const double v = a.v * b.v + c.v, e = fabs(a.v) * b.e + fabs(b.v) * a.e + a.e * b.e + c.e;
    ve r = {v, e + rnd(v, e)};
    return r;
}
/* sum of k exact products (any association, any contraction): <= k roundings of partial sums of the |products| */
static inline ve dot3x(double a0, double b0, double a1, double b1, double a2, double b2) {
    const double m = fabs(a0 * b0) + fabs(a1 * b1) + fabs(a2 * b2);
    ve r = {a0 * b0 + a1 * b1 + a2 * b2, gam(3) * m + 3 * TINY};
    return r;
}

/* one candidate pair of a pixel: what the decisions and the recurrence need */
typedef struct {
    uint32_t g;
    int und;          /* decision within its error of a threshold */
    int blend;        /* nominal decision */
    ve dx, dy, G, a;
} Cand;

typedef struct {
    const double *rec, *colors, *bg, *dpix;
    double W, H;
    size_t plane;
} Ctx;

/* Evaluate one pixel under the decisions blend[] (flip: candidates whose decision is inverted): per-candidate term values
 * and bounds in val / err ([nc][NS], zero for pairs that do not blend). */
static void eval_pixel(const Ctx* c, const Cand* cd, int nc, const int* dec, size_t pid, double (*val)[NS],
                       double (*err)[NS]) {
    const double d0 = c->dpix[pid], d1 = c->dpix[c->plane + pid], d2 = c->dpix[2 * c->plane + pid];
    int nb = 0;
    double rsum = 0.0, Tfin = 1.0;
    for (int k = 0; k < nc; ++k) {
        memset(val[k], 0, sizeof(double) * NS);
        memset(err[k], 0, sizeof(double) * NS);
        if (!dec[k]) continue;
        ++nb;
        rsum += cd[k].a.e / (1.0 - cd[k].a.v) + U;
        Tfin *= 1.0 - cd[k].a.v;
    }
    if (nb == 0) return;
    const ve bgdot = dot3x(c->bg[0], d0, c->bg[1], d1, c->bg[2], d2);
    /* walk back to front; `before` = sum over the blended j < k of (e_alpha_j / (1 - alpha_j) + u), T = prod_{j<k} */
    double before = rsum, after = 0.0, Tk = Tfin;
    ve rdot = X(0.0), lcd = X(0.0), la = X(0.0);
    for (int k = nc - 1; k >= 0; --k) {
        if (!dec[k]) continue;
        const Cand* q = cd + k;
        const double* co = c->rec + 8 * (size_t)q->g;
        const double A = co[4], Bc = co[5], C = co[6], o = co[7];
        const double oma = 1.0 - q->a.v;
        before -= q->a.e / oma + U;
        after += U + RCP_ERR;                               /* this division: multiply u + reciprocal 1 ulp */
        Tk /= oma;                                          /* T before this splat: prod_{j<k} (1 - alpha_j) */
        const double Tv = Tk;
        const double relT = fmax(before, 0.0) + nb * U + after;
        const ve T = {Tv, Tv * expm1(relT) + TINY};
        /* Tb rcp(1 - alpha_k) = -prod_{j != k} (1 - alpha_j) (bg . dL) */
        const double Tfi = Tfin / oma;
        const double relA = (rsum - (q->a.e / oma + U)) + nb * U + 2.0 * U + RCP_ERR;   /* multiplies at :262, :370 */
        const double epsA = expm1(fmax(relA, 0.0));
        ve TbI = {-Tfi * bgdot.v, Tfi * (1.0 + epsA) * bgdot.e + Tfi * fabs(bgdot.v) * epsA + TINY};
        TbI.e += rnd(TbI.v, TbI.e);
        /* recurrence */
        rdot = fma_(la, add(lcd, neg(rdot)), rdot);
        const double* col = c->colors + 3 * (size_t)q->g;
        const ve cdv = dot3x(col[0], d0, col[1], d1, col[2], d2);
        lcd = cdv;
        la = q->a;
        const ve dLda = fma_(add(cdv, neg(rdot)), T, TbI);
        const ve w = mul(q->G, dLda);
        const ve wx = mul(w, q->dx), wy = mul(w, q->dy);
        const ve q1 = mul(X(-Bc), wy);
        const ve u1 = fma_(X(A), wx, neg(q1));
        const ve q2 = mul(X(-Bc), wx);
        const ve u2 = fma_(X(C), wy, neg(q2));
        const ve bkz = mul(X(fabs(o)), X(0.5 * c->W)), bkw = mul(X(fabs(o)), X(0.5 * c->H));
        const ve v2 = fma_(absv(u2), bkw, mul(absv(u1), bkz));
        const ve mxx = mul(wx, q->dx), mxy = mul(wx, q->dy), myy = mul(wy, q->dy);
        const ve aT = mul(q->a, T);
        const ve c0 = mul(aT, X(d0)), c1 = mul(aT, X(d1)), c2 = mul(aT, X(d2));
        const ve t[NS] = {wx, wy, v2, mxx, mxy, myy, w, c0, c1, c2};
        for (int s = 0; s < NS; ++s) {
            val[k][s] = t[s].v;
            err[k][s] = t[s].e;
        }
    }
}

/* returns the number of pixels with more than MAX_UND undetermined pairs; stats[0] = undetermined pairs,
 * stats[1] = blended pairs (nominal).  tree_tile: depth of the in-tile summation tree (9 for render_bwd.cu: pair add 1 +
 * butterfly 5 + PartRows 3); groups_per_tile: partial sums a tile adds to the accumulator per Gaussian (1 for
 * render_bwd.cu's one flush; 4 for the colour-only walk, render_fwd.cu:433-434, one atomicAdd per warp after a pair add and
 * a 5-level butterfly, so its tree_tile is 6). */
long long bwd_bound(int P, int W, int H, int ty0, int ty1, const uint32_t* ranges, const uint32_t* point_list,
                    const double* subpixel_offset, const double* bg, const double* rec, const double* colors,
                    const uint32_t* n_contrib, const double* dL_dpix, double alpha_max, double alpha_min, int tree_tile,
                    int groups_per_tile, double* S, double* Bnd, double* Mg, uint8_t* und, double* stats) {
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    if (ty0 == 0 && ty1 == 0) ty1 = gy;
    memset(S, 0, sizeof(double) * NS * (size_t)P);
    memset(Mg, 0, sizeof(double) * NS * (size_t)P);
    double* Bs = (double*)calloc((size_t)P * NS, sizeof(double));      /* sum of the rows' bounds */
    double* Rm = (double*)calloc((size_t)P * NS, sizeof(double));      /* sum of |row| at kernel values */
    int* ntile = (int*)calloc((size_t)P, sizeof(int));
    uint8_t* inf = (uint8_t*)calloc((size_t)P, 1);
    memset(und, 0, (size_t)P);
    uint32_t maxlen = 0;
    for (int t = 0; t < gx * gy; ++t) {
        const uint32_t l = ranges[2 * t + 1] - ranges[2 * t];
        if (l > maxlen) maxlen = l;
    }
    Ctx cx = {rec, colors, bg, dL_dpix, (double)W, (double)H, (size_t)W * H};
    long long overflow = 0, n_und = 0, n_blend = 0;
#pragma omp parallel reduction(+ : overflow, n_und, n_blend)
    {
        const size_t L = maxlen > 0 ? maxlen : 1;
        double(*mom)[NS] = malloc(sizeof(double) * NS * L);
        double(*me)[NS] = malloc(sizeof(double) * NS * L);
        double(*mm)[NS] = malloc(sizeof(double) * NS * L);
        double(*mx)[NS] = malloc(sizeof(double) * NS * L);       /* exact |term| sums, for M */
        uint8_t* used = malloc(L);
        uint8_t* tinf = malloc(L);
        Cand* cd = malloc(sizeof(Cand) * L);
        int* pos = malloc(sizeof(int) * L);
        int* dec = malloc(sizeof(int) * L);
        int* dec0 = malloc(sizeof(int) * L);
        double(*v0)[NS] = malloc(sizeof(double) * NS * L);
        double(*e0)[NS] = malloc(sizeof(double) * NS * L);
        double(*v1)[NS] = malloc(sizeof(double) * NS * L);
        double(*e1)[NS] = malloc(sizeof(double) * NS * L);
        double(*xe)[NS] = malloc(sizeof(double) * NS * L);
        double(*xm)[NS] = malloc(sizeof(double) * NS * L);
#pragma omp for collapse(2) schedule(dynamic, 1)
        for (int ty = ty0; ty < ty1; ++ty)
            for (int tx = 0; tx < gx; ++tx) {
                const uint32_t r0 = ranges[2 * (ty * gx + tx)], r1 = ranges[2 * (ty * gx + tx) + 1];
                const uint32_t len = r1 - r0;
                if (len == 0) continue;
                memset(mom, 0, sizeof(double) * NS * len);
                memset(me, 0, sizeof(double) * NS * len);
                memset(mm, 0, sizeof(double) * NS * len);
                memset(mx, 0, sizeof(double) * NS * len);
                memset(used, 0, len);
                memset(tinf, 0, len);
                for (int ly = 0; ly < TILE; ++ly)
                    for (int lx = 0; lx < TILE; ++lx) {
                        const int ux = tx * TILE + lx, uy = ty * TILE + ly;
                        if (ux >= W || uy >= H) continue;
                        const size_t pid = (size_t)W * uy + ux;
                        uint32_t nl = n_contrib[pid];
                        if (nl > len) nl = len;
                        /* pixel position as the kernel rounds it: (float)ux + so.x (:250, :255) */
                        const double pxv = ux + subpixel_offset[2 * pid], pyv = uy + subpixel_offset[2 * pid + 1];
                        const ve px = {pxv, rnd(pxv, 0.0)}, py = {pyv, rnd(pyv, 0.0)};
                        int nc = 0, nu = 0;
                        for (uint32_t k = 0; k < nl; ++k) {
                            const uint32_t g = point_list[r0 + k];
                            const double* co = rec + 8 * (size_t)g;
                            Cand q;
                            q.g = g;
                            /* :339-346 */
                            q.dx = add(X(co[0]), neg(px));
                            q.dy = add(X(co[1]), neg(py));
                            const ve t1 = mul(X(co[4]), q.dx);
                            const ve t3 = mul(q.dy, mul(X(co[6]), q.dy));
                            const ve un = mul(q.dy, mul(X(-co[5]), q.dx));
                            const ve pw = fma_(fma_(q.dx, t1, t3), X(-0.5), un);
                            const double G = exp(pw.v), eg = expm1(pw.e);
                            q.G.v = G;
                            q.G.e = G * eg + EXP_ERR * G * (1.0 + eg) + TINY;
                            const ve oG = mul(X(co[7]), q.G);
                            q.a.v = fmin(alpha_max, oG.v);
                            q.a.e = oG.e;
                            const int may_p = !(pw.v - pw.e > 0.0), may_a = !(q.a.v + q.a.e < alpha_min);
                            q.blend = !(pw.v > 0.0) && !(q.a.v < alpha_min);
                            const int und_p = fabs(pw.v) <= pw.e && may_a;
                            const int und_a = fabs(q.a.v - alpha_min) <= q.a.e && may_p;
                            q.und = und_p || und_a;
                            if (!q.blend && !q.und) continue;
                            n_blend += q.blend;
                            n_und += q.und;
                            nu += q.und;
                            pos[nc] = (int)k;
                            cd[nc++] = q;
                        }
                        if (nc == 0) continue;
                        if (nu > MAX_UND) {
                            ++overflow;
                            for (int k = 0; k < nc; ++k) tinf[pos[k]] = 1;
                            continue;
                        }
                        for (int k = 0; k < nc; ++k) dec0[k] = cd[k].blend;
                        eval_pixel(&cx, cd, nc, dec0, pid, v0, e0);
                        memset(xe, 0, sizeof(double) * NS * (size_t)nc);
                        memset(xm, 0, sizeof(double) * NS * (size_t)nc);
                        if (nu > 0) {
                            int ui[MAX_UND], m = 0;
                            for (int k = 0; k < nc; ++k)
                                if (cd[k].und) ui[m++] = k;
                            for (int mask = 1; mask < (1 << m); ++mask) {
                                memcpy(dec, dec0, sizeof(int) * nc);
                                for (int b = 0; b < m; ++b)
                                    if (mask >> b & 1) dec[ui[b]] = !dec[ui[b]];
                                eval_pixel(&cx, cd, nc, dec, pid, v1, e1);
                                for (int k = 0; k < nc; ++k)
                                    for (int s = 0; s < NS; ++s) {
                                        const double de = fabs(v1[k][s] - v0[k][s]) + e1[k][s] - e0[k][s];
                                        const double dm = fabs(v1[k][s]) + e1[k][s] - fabs(v0[k][s]) - e0[k][s];
                                        if (de > xe[k][s]) xe[k][s] = de;
                                        if (dm > xm[k][s]) xm[k][s] = dm;
                                    }
                            }
                            for (int k = 0; k < nc; ++k)
                                if (cd[k].und) und[cd[k].g] = 1;      /* benign race: every writer stores 1 */
                        }
                        for (int k = 0; k < nc; ++k) {
                            const int p = pos[k];
                            used[p] = 1;
                            for (int s = 0; s < NS; ++s) {
                                mom[p][s] += v0[k][s];
                                me[p][s] += e0[k][s] + xe[k][s];
                                mm[p][s] += fabs(v0[k][s]) + e0[k][s] + xm[k][s];
                                mx[p][s] += fabs(v0[k][s]);
                            }
                        }
                    }
                /* flush: the tile's moments -> its row of sums, with their bounds (:403-409) */
                const double gt = gam(tree_tile);
                for (uint32_t p = 0; p < len; ++p) {
                    if (!used[p] && !tinf[p]) continue;
                    const uint32_t g = point_list[r0 + p];
                    if (tinf[p]) {
#pragma omp atomic write
                        inf[g] = 1;
                    }
                    if (!used[p]) continue;
                    const double* co = rec + 8 * (size_t)g;
                    const double A = co[4], Bc = co[5], C = co[6], o = co[7];
                    ve M[NS];
                    for (int s = 0; s < NS; ++s) {
                        M[s].v = mom[p][s];
                        M[s].e = me[p][s] + gt * mm[p][s];
                    }
                    const ve fx = mul(X(-o), X(0.5 * W)), fy = mul(X(-o), X(0.5 * H));
                    const ve h = X(-0.5 * o);
                    ve row[NS];
                    row[0] = mul(fx, add(mul(X(A), M[0]), mul(X(Bc), M[1])));
                    row[1] = mul(fy, add(mul(X(C), M[1]), mul(X(Bc), M[0])));
                    row[2] = M[2];
                    row[3] = mul(h, M[3]);
                    row[4] = mul(h, M[4]);
                    row[5] = mul(h, M[5]);
                    row[6] = M[6];
                    row[7] = M[7];
                    row[8] = M[8];
                    row[9] = M[9];
                    /* |exact per-pair terms| through the same linear map (for relative comparisons only) */
                    double mg[NS];
                    mg[0] = fabs(o) * 0.5 * W * (fabs(A) * mx[p][0] + fabs(Bc) * mx[p][1]);
                    mg[1] = fabs(o) * 0.5 * H * (fabs(C) * mx[p][1] + fabs(Bc) * mx[p][0]);
                    mg[2] = mx[p][2];
                    for (int s = 3; s < 6; ++s) mg[s] = 0.5 * fabs(o) * mx[p][s];
                    for (int s = 6; s < NS; ++s) mg[s] = mx[p][s];
                    double* Sg = S + NS * (size_t)g;
                    double* Bg = Bs + NS * (size_t)g;
                    double* Rg = Rm + NS * (size_t)g;
                    double* Mgg = Mg + NS * (size_t)g;
                    for (int s = 0; s < NS; ++s) {
#pragma omp atomic
                        Sg[s] += row[s].v;
#pragma omp atomic
                        Bg[s] += row[s].e;
#pragma omp atomic
                        Rg[s] += fabs(row[s].v) + row[s].e;
#pragma omp atomic
                        Mgg[s] += mg[s];
                    }
#pragma omp atomic
                    ntile[g] += groups_per_tile;
                }
            }
        free(mom); free(me); free(mm); free(mx); free(used); free(tinf); free(cd); free(pos); free(dec); free(dec0);
        free(v0); free(e0); free(v1); free(e1); free(xe); free(xm);
    }
    for (size_t g = 0; g < (size_t)P; ++g) {
        const double gk = gam(ntile[g]);
        for (int s = 0; s < NS; ++s) Bnd[NS * g + s] = inf[g] ? INFINITY : Bs[NS * g + s] + gk * Rm[NS * g + s];
        if (inf[g]) und[g] = 2;
    }
    stats[0] = (double)n_und;
    stats[1] = (double)n_blend;
    free(Bs); free(Rm); free(ntile); free(inf);
    return overflow;
}
