/*
 * oracle.c -- TEST INFRASTRUCTURE, not product code.
 *
 * CPU restatement (plain C, OpenMP) of the differentiable Gaussian-splat rasterizer path of
 * jkulhanek/wild-gaussians, i.e. of submodules/diff-gaussian-rasterization (DGR).  It is the
 * checker for the CUDA path in wild-gaussians_b200/ and the "pure CPU projection/composite
 * path" baseline that bench.py times on the host cores.  Only tests/, __graft_entry__.smoke()
 * and bench.py (cpu_baseline / --impl reference fallback) may load it.
 *
 * Every function cites the reference lines it follows (paths relative to
 * /root/reference/submodules/diff-gaussian-rasterization/).
 *
 * Numerics.  The reference is compiled by nvcc with -fmad=true: products feeding sums are
 * contracted into fused multiply-adds.  The contraction pattern was read off the reference's
 * PTX/SASS (nvcc 12.9):
 *     a*b + c*d            -> fma(a, b, rnd(c*d))        (first product fused, second rounded)
 *     (a*b + c*d) + e*f    -> fma(e, f, fma(a, b, rnd(c*d)))
 *     x + a*b, a*b + x     -> fma(a, b, x)
 *     a*b - c, c - a*b     -> fma(a, b, -c), fma(-a, b, c)
 * and is written out below with explicit fmaf() (this file is compiled with
 * -ffp-contract=off so gcc adds none of its own).  With that, every integer artefact
 * (radii, tile rectangles, depth keys, sorted instance list, tile ranges) is bit-identical
 * to the reference's; this is pinned by tests/golden/ (vectors produced by the reference
 * itself on a GPU, see tests/golden/make_golden.py).  expf() is glibc's, not CUDA's
 * (MUFU.EX2 based) one, so composited pixels agree to ~1e-6 and a handful of alpha-threshold
 * decisions per million may flip; tests state the tolerance.
 *
 * Build:  make -C oracle        (gcc -O2 -ffp-contract=off -fopenmp)
 *         -DORACLE_DOUBLE builds the same algorithm in fp64 (for finite-difference checks).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#ifdef ORACLE_DOUBLE
typedef double real;
#define FMA(a, b, c) ((a) * (b) + (c))
#define R_SQRT sqrt
#define R_EXP exp
#define R_CEIL ceil
#define R_FABS fabs
#define R_MAX fmax
#define R_MIN fmin
#else
typedef float real;
#define FMA(a, b, c) fmaf((a), (b), (c))
#define R_SQRT sqrtf
#define R_EXP expf
#define R_CEIL ceilf
#define R_FABS fabsf
#define R_MAX fmaxf
#define R_MIN fminf
#endif

#define TILE 16
#define RL(x) ((real)(x))

int oracle_real_bytes(void) { return (int)sizeof(real); }
int oracle_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
void oracle_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

/* SH constants (auxiliary.h:22-39) */
static const real SH_C0 = RL(0.28209479177387814);
static const real SH_C1 = RL(0.4886025119029199);
static const real SH_C2[5] = {RL(1.0925484305920792), RL(-1.0925484305920792), RL(0.31539156525252005),
                              RL(-1.0925484305920792), RL(0.5462742152960396)};
static const real SH_C3[7] = {RL(-0.5900435899266435), RL(2.890611442640554), RL(-0.4570457994644658),
                              RL(0.3731763325901154), RL(-0.4570457994644658), RL(1.445305721320277),
                              RL(-0.5900435899266435)};

/* a0*b0 + a1*b1 + a2*b2 as nvcc contracts it */
static inline real dot3c(real a0, real b0, real a1, real b1, real a2, real b2) {
    return FMA(a2, b2, FMA(a0, b0, a1 * b1));
}
/* m[o]*x + m[o+4]*y + m[o+8]*z + m[o+12]  (auxiliary.h:58-77) */
static inline real xform_row(const real* m, int o, real x, real y, real z) {
    return dot3c(m[o], x, m[o + 4], y, m[o + 8], z) + m[o + 12];
}

/* column-major 3x3 product, element (c,r) = a[0][r]*b[c][0] + a[1][r]*b[c][1] + a[2][r]*b[c][2]
 * (glm/detail/type_mat3x3.inl:486-519) */
static void mat3_mul(const real a[3][3], const real b[3][3], real out[3][3]) {
    real t[3][3];
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) t[c][r] = dot3c(a[0][r], b[c][0], a[1][r], b[c][1], a[2][r], b[c][2]);
    memcpy(out, t, sizeof(t));
}
static void mat3_transpose(const real a[3][3], real out[3][3]) {
    real t[3][3];
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) t[c][r] = a[r][c];
    memcpy(out, t, sizeof(t));
}

/* forward.cu:129-163 -- Sigma = (S R)^T (S R); quaternion used un-normalised */
static void quat_to_R(const real* q, real R[3][3]) {
    const real r = q[0], x = q[1], y = q[2], z = q[3];
    /* Contraction as in the reference SASS (ptxas fuses a product into the add/sub only when every
     * use of that product can be fused; products shared as plain addends stay rounded):
     *   xz, rx, rz, yy, zz are rounded products; r*y, y*z, x*y, x*x are fused. */
    const real xz = x * z, rx = r * x, rz = r * z, yy = y * y, zz = z * z;
    R[0][0] = RL(1.0) - RL(2.0) * (yy + zz);
    R[0][1] = RL(2.0) * FMA(x, y, -rz);
    R[0][2] = RL(2.0) * FMA(r, y, xz);
    R[1][0] = RL(2.0) * FMA(x, y, rz);
    R[1][1] = RL(1.0) - RL(2.0) * FMA(x, x, zz);
    R[1][2] = RL(2.0) * FMA(y, z, -rx);
    R[2][0] = RL(2.0) * FMA(-r, y, xz);
    R[2][1] = RL(2.0) * FMA(y, z, rx);
    R[2][2] = RL(1.0) - RL(2.0) * FMA(x, x, yy);
}
static void cov3d_from_scale_rot(const real* scale, real mod, const real* rot, real* cov) {
    real S[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, R[3][3], M[3][3], Mt[3][3], Sg[3][3];
    S[0][0] = mod * scale[0];
    S[1][1] = mod * scale[1];
    S[2][2] = mod * scale[2];
    quat_to_R(rot, R);
    mat3_mul(S, R, M);
    mat3_transpose(M, Mt);
    mat3_mul(Mt, M, Sg);
    cov[0] = Sg[0][0]; cov[1] = Sg[0][1]; cov[2] = Sg[0][2];
    cov[3] = Sg[1][1]; cov[4] = Sg[1][2]; cov[5] = Sg[2][2];
}

typedef struct {
    real t[3], txtz, tytz, limx, limy;
    real T[3][3], Vrk[3][3], cov[3][3];
} Ewa;

/* forward.cu:74-106 / backward.cu:165-197 */
static void ewa_project(const real* mean, real fx, real fy, real tan_fovx, real tan_fovy, const real* cov3D,
                        const real* view, Ewa* e) {
    real t[3];
    t[0] = xform_row(view, 0, mean[0], mean[1], mean[2]);
    t[1] = xform_row(view, 1, mean[0], mean[1], mean[2]);
    t[2] = xform_row(view, 2, mean[0], mean[1], mean[2]);
    e->limx = RL(1.3) * tan_fovx;
    e->limy = RL(1.3) * tan_fovy;
    e->txtz = t[0] / t[2];
    e->tytz = t[1] / t[2];
    t[0] = R_MIN(e->limx, R_MAX(-e->limx, e->txtz)) * t[2];
    t[1] = R_MIN(e->limy, R_MAX(-e->limy, e->tytz)) * t[2];
    e->t[0] = t[0]; e->t[1] = t[1]; e->t[2] = t[2];
    real J[3][3] = {{fx / t[2], 0, -(fx * t[0]) / (t[2] * t[2])},
                    {0, fy / t[2], -(fy * t[1]) / (t[2] * t[2])},
                    {0, 0, 0}};
    real Wm[3][3] = {{view[0], view[4], view[8]}, {view[1], view[5], view[9]}, {view[2], view[6], view[10]}};
    mat3_mul(Wm, J, e->T);
    real V[3][3] = {{cov3D[0], cov3D[1], cov3D[2]}, {cov3D[1], cov3D[3], cov3D[4]}, {cov3D[2], cov3D[4], cov3D[5]}};
    memcpy(e->Vrk, V, sizeof(V));
    real Tt[3][3], Vt[3][3], tmp[3][3];
    mat3_transpose(e->T, Tt);
    mat3_transpose(V, Vt);
    mat3_mul(Tt, Vt, tmp);
    mat3_mul(tmp, e->T, e->cov);
}

/* forward.cu:20-71 */
static void sh_to_rgb(int deg, const real* sh, const real* pos, const real* campos, real* rgb, uint8_t* clamped) {
    real dx = pos[0] - campos[0], dy = pos[1] - campos[1], dz = pos[2] - campos[2];
    const real len = R_SQRT(FMA(dz, dz, FMA(dx, dx, dy * dy)));
    const real x = dx / len, y = dy / len, z = dz / len;
    real res[3];
    for (int c = 0; c < 3; ++c) res[c] = SH_C0 * sh[c];
    if (deg > 0) {
        const real k1 = SH_C1 * y, k2 = SH_C1 * z, k3 = SH_C1 * x;
        for (int c = 0; c < 3; ++c) {
            real r = res[c];
            r = FMA(-k1, sh[3 + c], r);
            r = FMA(k2, sh[6 + c], r);
            r = FMA(-k3, sh[9 + c], r);
            res[c] = r;
        }
        if (deg > 1) {
            const real xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            const real w4 = SH_C2[0] * xy, w5 = SH_C2[1] * yz, w6 = SH_C2[2] * (FMA(RL(2.0), zz, -xx) - yy),
                       w7 = SH_C2[3] * xz, w8 = SH_C2[4] * (xx - yy);
            for (int c = 0; c < 3; ++c) {
                real r = res[c];
                r = FMA(w4, sh[12 + c], r);
                r = FMA(w5, sh[15 + c], r);
                r = FMA(w6, sh[18 + c], r);
                r = FMA(w7, sh[21 + c], r);
                r = FMA(w8, sh[24 + c], r);
                res[c] = r;
            }
            if (deg > 2) {
                const real w9 = SH_C3[0] * y * (FMA(RL(3.0), xx, -yy));
                const real w10 = SH_C3[1] * xy * z;
                const real w11 = SH_C3[2] * y * (FMA(RL(4.0), zz, -xx) - yy);
                const real w12 = SH_C3[3] * z * (FMA(RL(-3.0), yy, FMA(RL(-3.0), xx, RL(2.0) * zz)));
                const real w13 = SH_C3[4] * x * (FMA(RL(4.0), zz, -xx) - yy);
                const real w14 = SH_C3[5] * z * (xx - yy);
                const real w15 = SH_C3[6] * x * (FMA(RL(-3.0), yy, xx));
                for (int c = 0; c < 3; ++c) {
                    real r = res[c];
                    r = FMA(w9, sh[27 + c], r);
                    r = FMA(w10, sh[30 + c], r);
                    r = FMA(w11, sh[33 + c], r);
                    r = FMA(w12, sh[36 + c], r);
                    r = FMA(w13, sh[39 + c], r);
                    r = FMA(w14, sh[42 + c], r);
                    r = FMA(w15, sh[45 + c], r);
                    res[c] = r;
                }
            }
        }
    }
    for (int c = 0; c < 3; ++c) {
        res[c] += RL(0.5);
        clamped[c] = res[c] < 0;
        rgb[c] = R_MAX(res[c], RL(0.0));
    }
}

/*
 * Per-Gaussian forward (forward.cu:166-268 with auxiliary.h:41-56,139-164).
 * Outputs (caller-allocated): radii i32[P], depths[P], means2D[2P], cov3D[6P], conic_opacity[4P], rgb[3P],
 * clamped u8[3P], tiles_touched u32[P], rect i32[4P] (x0,y0,x1,y1 tiles).  Arrays of culled Gaussians keep
 * the caller's initial contents except radii / tiles_touched / rect (set to 0).
 * ty0/ty1: tile-row shard (0,0 = all rows); only tiles_touched / rect are clipped.
 * Returns R = sum(tiles_touched), or -1 if prefiltered is set and a point is culled.
 */
long long oracle_preprocess(int P, int D, int M, int W, int H, const real* means3D, const real* shs,
                            const real* colors_precomp, const real* opacities, const real* scales, real scale_modifier,
                            const real* rotations, const real* cov3D_precomp, const real* view, const real* proj,
                            const real* campos, real tan_fovx, real tan_fovy, real kernel_size, int prefiltered,
                            int ty0, int ty1, int32_t* radii, real* depths, real* means2D, real* cov3Ds,
                            real* conic_opacity, real* rgb, uint8_t* clamped, uint32_t* tiles_touched, int32_t* rect) {
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    if (ty0 == 0 && ty1 == 0) ty1 = gy;
    const real focal_y = H / (RL(2.0) * tan_fovy);
    const real focal_x = W / (RL(2.0) * tan_fovx);
    int bad = 0;
    long long total = 0;
#pragma omp parallel for schedule(static) reduction(+ : total) reduction(| : bad)
    for (int idx = 0; idx < P; ++idx) {
        radii[idx] = 0;
        tiles_touched[idx] = 0;
        rect[4 * idx + 0] = rect[4 * idx + 1] = rect[4 * idx + 2] = rect[4 * idx + 3] = 0;
        const real* p = means3D + 3 * (size_t)idx;
        /* in_frustum (auxiliary.h:139-164): only the near plane culls */
        const real hx = xform_row(proj, 0, p[0], p[1], p[2]);
        const real hy = xform_row(proj, 1, p[0], p[1], p[2]);
        const real hw = xform_row(proj, 3, p[0], p[1], p[2]);
        const real p_w = RL(1.0) / (hw + RL(0.0000001));
        const real proj_x = hx * p_w, proj_y = hy * p_w;
        const real view_z = xform_row(view, 2, p[0], p[1], p[2]);
        if (view_z <= RL(0.2)) {
            if (prefiltered) bad |= 1;
            continue;
        }
        real cov_local[6];
        const real* cov3D;
        if (cov3D_precomp) {
            cov3D = cov3D_precomp + 6 * (size_t)idx;
        } else {
            cov3d_from_scale_rot(scales + 3 * (size_t)idx, scale_modifier, rotations + 4 * (size_t)idx, cov_local);
            memcpy(cov3Ds + 6 * (size_t)idx, cov_local, sizeof(cov_local));
            cov3D = cov_local;
        }
        Ewa e;
        ewa_project(p, focal_x, focal_y, tan_fovx, tan_fovy, cov3D, view, &e);
        real c00 = e.cov[0][0], c01 = e.cov[0][1], c11 = e.cov[1][1];
        /* forward.cu:112-121 (mixed precision: max / division / sqrt in double) */
        const real bb = c01 * c01;
        const real det_0 = (real)fmax(1e-6, (double)FMA(c00, c11, -bb));
        const real a1 = c00 + kernel_size, c1 = c11 + kernel_size;
        const real det_raw = FMA(a1, c1, -bb);
        const real det_1 = (real)fmax(1e-6, (double)det_raw);
        real coef = (real)sqrt((double)det_0 / ((double)det_1 + 1e-6) + 1e-6);
        if ((double)det_0 <= 1e-6 || (double)det_1 <= 1e-6) coef = 0;
        c00 = a1;
        c11 = c1;
        const real det = det_raw; /* same expression as det_1's argument (forward.cu:231) */
        if (det == 0) continue;
        const real det_inv = RL(1.0) / det;
        const real conic[3] = {c11 * det_inv, -c01 * det_inv, c00 * det_inv};
        const real mid = RL(0.5) * (c00 + c11);
        const real disc = R_SQRT(R_MAX(RL(0.1), FMA(mid, mid, -det)));
        const real lambda1 = mid + disc, lambda2 = mid - disc;
        const real my_radius = R_CEIL(RL(3.0) * R_SQRT(R_MAX(lambda1, lambda2)));
        /* ndc2Pix in double (auxiliary.h:41-44): ((v + 1.0) * S - 1.0) * 0.5, (v+1)*S - 1 is a DFMA */
        const real px = (real)(fma((double)proj_x + 1.0, (double)W, -1.0) * 0.5);
        const real py = (real)(fma((double)proj_y + 1.0, (double)H, -1.0) * 0.5);
        /* getRect (auxiliary.h:46-56) */
        const int max_radius = (int)my_radius;
        const real rr = (real)max_radius;
        int rx0 = (int)((px - rr) / TILE), ry0 = (int)((py - rr) / TILE);
        int rx1 = (int)((px + rr + TILE - 1) / TILE), ry1 = (int)((py + rr + TILE - 1) / TILE);
        rx0 = rx0 < 0 ? 0 : (rx0 > gx ? gx : rx0);
        ry0 = ry0 < 0 ? 0 : (ry0 > gy ? gy : ry0);
        rx1 = rx1 < 0 ? 0 : (rx1 > gx ? gx : rx1);
        ry1 = ry1 < 0 ? 0 : (ry1 > gy ? gy : ry1);
        if ((rx1 - rx0) * (ry1 - ry0) == 0) continue;
        if (!colors_precomp) {
            sh_to_rgb(D, shs + (size_t)idx * M * 3, p, campos, rgb + 3 * (size_t)idx, clamped + 3 * (size_t)idx);
        }
        depths[idx] = view_z;
        radii[idx] = (int32_t)my_radius;
        means2D[2 * (size_t)idx + 0] = px;
        means2D[2 * (size_t)idx + 1] = py;
        conic_opacity[4 * (size_t)idx + 0] = conic[0];
        conic_opacity[4 * (size_t)idx + 1] = conic[1];
        conic_opacity[4 * (size_t)idx + 2] = conic[2];
        conic_opacity[4 * (size_t)idx + 3] = opacities[idx] * coef;
        int cy0 = ry0 > ty0 ? ry0 : ty0, cy1 = ry1 < ty1 ? ry1 : ty1;
        if (cy1 < cy0) cy1 = cy0;
        const int cnt = (cy1 - cy0) * (rx1 - rx0);
        tiles_touched[idx] = (uint32_t)cnt;
        if (cnt) {
            rect[4 * idx + 0] = rx0; rect[4 * idx + 1] = cy0; rect[4 * idx + 2] = rx1; rect[4 * idx + 3] = cy1;
        }
        total += cnt;
    }
    return bad ? -1 : total;
}

/* ---- binning (rasterizer_impl.cu:70-138,303-320) ------------------------------------------ */
typedef struct {
    uint64_t key;
    uint32_t val;
    uint32_t seq;
} Inst;

static void merge_sort_inst(Inst* a, Inst* tmp, size_t n) {
    /* bottom-up stable merge sort on key */
    for (size_t w = 1; w < n; w *= 2) {
#pragma omp parallel for schedule(dynamic, 64)
        for (long long lo = 0; lo < (long long)n; lo += 2 * (long long)w) {
            size_t l = (size_t)lo, m = l + w < n ? l + w : n, h = l + 2 * w < n ? l + 2 * w : n;
            size_t i = l, j = m, k = l;
            while (i < m && j < h) tmp[k++] = (a[j].key < a[i].key) ? a[j++] : a[i++];
            while (i < m) tmp[k++] = a[i++];
            while (j < h) tmp[k++] = a[j++];
        }
        Inst* t = a; a = tmp; tmp = t;
    }
    /* caller passes buffers such that it can find the result: see oracle_bin */
}

/*
 * Emits (tile << 32 | depth bits, idx) per (Gaussian, tile) in Gaussian-index order, tile rectangle
 * row-major (rasterizer_impl.cu:88-108), sorts stably by key (CUB radix sort is stable), writes the sorted
 * Gaussian ids to point_list[R], the sorted keys' tile ids to tile_of[R] (may be NULL) and per-tile
 * [start,end) to ranges[2*T] (zero for empty tiles, rasterizer_impl.cu:313-320).
 */
int oracle_bin(int P, int W, int H, long long R, const int32_t* radii, const real* depths, const int32_t* rect,
               uint32_t* point_list, uint32_t* tile_of, uint32_t* ranges) {
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    memset(ranges, 0, sizeof(uint32_t) * 2 * (size_t)gx * gy);
    if (R <= 0) return 0;
    Inst* a = (Inst*)malloc(sizeof(Inst) * (size_t)R);
    Inst* b = (Inst*)malloc(sizeof(Inst) * (size_t)R);
    if (!a || !b) { free(a); free(b); return -1; }
    size_t off = 0;
    for (int idx = 0; idx < P; ++idx) {
        if (radii[idx] <= 0) continue;
        const int32_t* r = rect + 4 * (size_t)idx;
        uint32_t dbits;
        float df = (float)depths[idx];
        memcpy(&dbits, &df, 4);
        for (int y = r[1]; y < r[3]; ++y)
            for (int x = r[0]; x < r[2]; ++x) {
                a[off].key = ((uint64_t)((uint32_t)(y * gx + x)) << 32) | dbits;
                a[off].val = (uint32_t)idx;
                a[off].seq = (uint32_t)off;
                ++off;
            }
    }
    if ((long long)off != R) { free(a); free(b); return -2; }
    /* number of merge levels decides where the result lands */
    int levels = 0;
    for (size_t w = 1; w < (size_t)R; w *= 2) ++levels;
    merge_sort_inst(a, b, (size_t)R);
    Inst* s = (levels % 2 == 0) ? a : b;
    for (size_t i = 0; i < (size_t)R; ++i) {
        point_list[i] = s[i].val;
        const uint32_t tile = (uint32_t)(s[i].key >> 32);
        if (tile_of) tile_of[i] = tile;
        if (i == 0) ranges[2 * tile] = 0;
        else {
            const uint32_t prev = (uint32_t)(s[i - 1].key >> 32);
            if (prev != tile) { ranges[2 * prev + 1] = (uint32_t)i; ranges[2 * tile] = (uint32_t)i; }
        }
        if (i == (size_t)R - 1) ranges[2 * tile + 1] = (uint32_t)R;
    }
    free(a);
    free(b);
    return 0;
}

/* ---- forward composite (forward.cu:273-395) ------------------------------------------------ */
static inline real pair_power(const real* con_o, real dx, real dy) {
    /* -0.5f*(A*dx*dx + C*dy*dy) - B*dx*dy, contracted as in the reference SASS (SURVEY N3):
     * s = fma(A*dx, dx, (C*dy)*dy); u = (B*dx)*dy; power = fma(s, -0.5, -u) */
    const real s = FMA(con_o[0] * dx, dx, (con_o[2] * dy) * dy);
    const real u = (con_o[1] * dx) * dy;
    return FMA(s, RL(-0.5), -u);
}

/* the reference's sample position and power of splat g at pixel (px, py) (forward.cu:340-357) */
static inline real splat_power(const real* means2D, const real* conic_opacity, uint32_t g, int px, int py, real so_x,
                               real so_y) {
    const real pfx = (real)px + so_x, pfy = (real)py + so_y;
    const real dx = means2D[2 * (size_t)g] - pfx, dy = means2D[2 * (size_t)g + 1] - pfy;
    return pair_power(conic_opacity + 4 * (size_t)g, dx, dy);
}

/* splat_power for n (pixel, splat) pairs: splat g[i] at pixel (px[i], py[i]) with sub-pixel offset so[2 i], so[2 i + 1]
 * (for comparison with other restatements of the composite's power, tests/test_forward_exact.py) */
void oracle_pair_power(long long n, const real* means2D, const real* conic_opacity, const uint32_t* g,
                       const int32_t* px, const int32_t* py, const real* so, real* out) {
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; ++i)
        out[i] = splat_power(means2D, conic_opacity, g[i], px[i], py[i], so[2 * i], so[2 * i + 1]);
}

void oracle_render(int W, int H, int ty0, int ty1, const uint32_t* ranges, const uint32_t* point_list,
                   const real* subpixel_offset, const real* means2D, const real* colors, const real* conic_opacity,
                   const real* bg, real* final_T, uint32_t* n_contrib, real* out_color) {
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    if (ty0 == 0 && ty1 == 0) ty1 = gy;
    const size_t plane = (size_t)W * H;
#pragma omp parallel for collapse(2) schedule(dynamic, 1)
    for (int ty = ty0; ty < ty1; ++ty)
        for (int tx = 0; tx < gx; ++tx) {
            const uint32_t r0 = ranges[2 * (ty * gx + tx)], r1 = ranges[2 * (ty * gx + tx) + 1];
            for (int ly = 0; ly < TILE; ++ly)
                for (int lx = 0; lx < TILE; ++lx) {
                    const int px = tx * TILE + lx, py = ty * TILE + ly;
                    if (px >= W || py >= H) continue;
                    const size_t pid = (size_t)W * py + px;
                    real T = 1, C[3] = {0, 0, 0};
                    uint32_t contributor = 0, last = 0;
                    for (uint32_t i = r0; i < r1; ++i) {
                        contributor++;
                        const uint32_t g = point_list[i];
                        const real* co = conic_opacity + 4 * (size_t)g;
                        const real power = splat_power(means2D, conic_opacity, g, px, py, subpixel_offset[2 * pid],
                                                       subpixel_offset[2 * pid + 1]);
                        if (power > 0) continue;
                        const real alpha = R_MIN(RL(0.99), co[3] * R_EXP(power));
                        if (alpha < RL(1.0) / RL(255.0)) continue;
                        const real test_T = T * (1 - alpha);
                        if (test_T < RL(0.0001)) break;
                        for (int ch = 0; ch < 3; ++ch) C[ch] = FMA(colors[3 * (size_t)g + ch] * alpha, T, C[ch]);
                        T = test_T;
                        last = contributor;
                    }
                    final_T[pid] = T;
                    n_contrib[pid] = last;
                    for (int ch = 0; ch < 3; ++ch) out_color[ch * plane + pid] = FMA(T, bg[ch], C[ch]);
                }
        }
}

/* ---- backward composite (backward.cu:435-606) ---------------------------------------------- *
 * Per-pixel recurrence exactly as the reference; the per-Gaussian sums (10 atomics per pair in the
 * reference) are accumulated in double, tile by tile in a fixed order, so the result is deterministic.
 * acc[P][10] = {dmean2D.x, dmean2D.y, |.|, dconic.x, dconic.y, dconic.w, dopacity, dcolor rgb}        */
void oracle_render_backward(int P, int W, int H, int ty0, int ty1, const uint32_t* ranges, const uint32_t* point_list,
                            const real* subpixel_offset, const real* bg, const real* means2D,
                            const real* conic_opacity, const real* colors, const real* final_T,
                            const uint32_t* n_contrib, const real* dL_dpix, double* acc) {
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    if (ty0 == 0 && ty1 == 0) ty1 = gy;
    const size_t plane = (size_t)W * H;
    memset(acc, 0, sizeof(double) * 10 * (size_t)P);
    const real ddelx_dx = (real)(0.5 * W), ddely_dy = (real)(0.5 * H);
    int nthreads = 1;
#ifdef _OPENMP
    nthreads = omp_get_max_threads();
#endif
    /* per-thread accumulators would need P*10 doubles each; instead parallelise over tiles and use
     * atomics on doubles (order-insensitive to ~1e-16, far below the fp32 tolerances tested) */
    (void)nthreads;
#pragma omp parallel for collapse(2) schedule(dynamic, 1)
    for (int ty = ty0; ty < ty1; ++ty)
        for (int tx = 0; tx < gx; ++tx) {
            const uint32_t r0 = ranges[2 * (ty * gx + tx)], r1 = ranges[2 * (ty * gx + tx) + 1];
            for (int ly = 0; ly < TILE; ++ly)
                for (int lx = 0; lx < TILE; ++lx) {
                    const int px = tx * TILE + lx, py = ty * TILE + ly;
                    if (px >= W || py >= H) continue;
                    const size_t pid = (size_t)W * py + px;
                    const real pfx = (real)px + subpixel_offset[2 * pid], pfy = (real)py + subpixel_offset[2 * pid + 1];
                    const real T_final = final_T[pid];
                    real T = T_final;
                    const uint32_t last_contributor = n_contrib[pid];
                    real accum_rec[3] = {0, 0, 0}, last_color[3] = {0, 0, 0}, last_alpha = 0;
                    real dpx[3];
                    for (int ch = 0; ch < 3; ++ch) dpx[ch] = dL_dpix[ch * plane + pid];
                    /* walk back to front over the instances this pixel blended or skipped */
                    uint32_t n = r1 - r0;
                    if (n > last_contributor) n = last_contributor;
                    for (uint32_t k = n; k-- > 0;) {
                        const uint32_t g = point_list[r0 + k];
                        const real dx = means2D[2 * (size_t)g] - pfx, dy = means2D[2 * (size_t)g + 1] - pfy;
                        const real* co = conic_opacity + 4 * (size_t)g;
                        const real power = pair_power(co, dx, dy);
                        if (power > 0) continue;
                        const real G = R_EXP(power);
                        const real alpha = R_MIN(RL(0.99), co[3] * G);
                        if (alpha < RL(1.0) / RL(255.0)) continue;
                        T = T / (RL(1.0) - alpha);
                        const real dchannel_dcolor = alpha * T;
                        real dL_dalpha = 0;
                        double* a = acc + 10 * (size_t)g;
                        for (int ch = 0; ch < 3; ++ch) {
                            const real c = colors[3 * (size_t)g + ch];
                            accum_rec[ch] = FMA(last_alpha, last_color[ch], (RL(1.0) - last_alpha) * accum_rec[ch]);
                            last_color[ch] = c;
                            dL_dalpha = FMA(c - accum_rec[ch], dpx[ch], dL_dalpha);
                            const double v = (double)(dchannel_dcolor * dpx[ch]);
#pragma omp atomic
                            a[7 + ch] += v;
                        }
                        dL_dalpha *= T;
                        last_alpha = alpha;
                        real bg_dot = 0;
                        for (int ch = 0; ch < 3; ++ch) bg_dot = FMA(bg[ch], dpx[ch], bg_dot);
                        dL_dalpha = FMA(-T_final / (RL(1.0) - alpha), bg_dot, dL_dalpha);
                        const real dL_dG = co[3] * dL_dalpha;
                        const real gdx = G * dx, gdy = G * dy;
                        const real dG_ddelx = FMA(-gdx, co[0], -(gdy * co[1]));
                        const real dG_ddely = FMA(-gdy, co[2], -(gdx * co[1]));
                        const double v0 = (double)(dL_dG * dG_ddelx * ddelx_dx);
                        const double v1 = (double)(dL_dG * dG_ddely * ddely_dy);
                        const double v2 = (double)(R_FABS(dL_dG * dG_ddelx * ddelx_dx) + R_FABS(dL_dG * dG_ddely * ddely_dy));
                        const double v3 = (double)(RL(-0.5) * gdx * dx * dL_dG);
                        const double v4 = (double)(RL(-0.5) * gdx * dy * dL_dG);
                        const double v5 = (double)(RL(-0.5) * gdy * dy * dL_dG);
                        const double v6 = (double)(G * dL_dalpha);
#pragma omp atomic
                        a[0] += v0;
#pragma omp atomic
                        a[1] += v1;
#pragma omp atomic
                        a[2] += v2;
#pragma omp atomic
                        a[3] += v3;
#pragma omp atomic
                        a[4] += v4;
#pragma omp atomic
                        a[5] += v5;
#pragma omp atomic
                        a[6] += v6;
                    }
                }
        }
}

/* auxiliary.h:107-117 */
static void dnormvdv3(const real* v, const real* dv, real* out) {
    const real sum2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    const real invsum32 = RL(1.0) / R_SQRT(sum2 * sum2 * sum2);
    out[0] = ((+sum2 - v[0] * v[0]) * dv[0] - v[1] * v[0] * dv[1] - v[2] * v[0] * dv[2]) * invsum32;
    out[1] = (-v[0] * v[1] * dv[0] + (sum2 - v[1] * v[1]) * dv[1] - v[2] * v[1] * dv[2]) * invsum32;
    out[2] = (-v[0] * v[2] * dv[0] - v[1] * v[2] * dv[1] + (sum2 - v[2] * v[2]) * dv[2]) * invsum32;
}

/*
 * Per-Gaussian backward: backward.cu:144-310 (cov2D / conic / opacity-compensation), :382-432 (projection),
 * :20-139 (SH), :314-377 (scale / rotation).  acc = output of oracle_render_backward.
 * Gradient arithmetic is plain (uncontracted) fp32 with the reference's fp64 steps; gradients are compared
 * with a 1e-3 tolerance, not bit-exactly.  All outputs must be zero-initialised by the caller.
 */
void oracle_preprocess_backward(int P, int D, int M, int W, int H, const real* means3D, const int32_t* radii,
                                const real* shs, const uint8_t* clamped, const real* scales, real scale_modifier,
                                const real* rotations, const real* cov3D_all, const real* view, const real* proj,
                                const real* campos, real tan_fovx, real tan_fovy, real kernel_size,
                                const real* conic_opacity, const double* acc, real* dL_dmean2D, real* dL_dconic,
                                real* dL_dopacity, real* dL_dcolor, real* dL_dmean3D, real* dL_dcov3D, real* dL_dsh,
                                real* dL_dscale, real* dL_drot) {
    const real h_y = H / (RL(2.0) * tan_fovy);
    const real h_x = W / (RL(2.0) * tan_fovx);
#pragma omp parallel for schedule(static)
    for (int idx = 0; idx < P; ++idx) {
        if (!(radii[idx] > 0)) continue;
        const double* a = acc + 10 * (size_t)idx;
        const real m2d[3] = {(real)a[0], (real)a[1], (real)a[2]};
        const real dcon[3] = {(real)a[3], (real)a[4], (real)a[5]};
        real dop = (real)a[6];
        const real dcol[3] = {(real)a[7], (real)a[8], (real)a[9]};
        for (int k = 0; k < 3; ++k) dL_dmean2D[3 * (size_t)idx + k] = m2d[k];
        dL_dconic[4 * (size_t)idx + 0] = dcon[0];
        dL_dconic[4 * (size_t)idx + 1] = dcon[1];
        dL_dconic[4 * (size_t)idx + 3] = dcon[2];
        for (int k = 0; k < 3; ++k) dL_dcolor[3 * (size_t)idx + k] = dcol[k];

        const real* mean = means3D + 3 * (size_t)idx;
        const real* cov3D = cov3D_all + 6 * (size_t)idx;
        Ewa e;
        ewa_project(mean, h_x, h_y, tan_fovx, tan_fovy, cov3D, view, &e);
        const real* t = e.t;
        const real x_grad_mul = (e.txtz < -e.limx || e.txtz > e.limx) ? 0 : 1;
        const real y_grad_mul = (e.tytz < -e.limy || e.tytz > e.limy) ? 0 : 1;
        real c00 = e.cov[0][0], c01 = e.cov[0][1], c11 = e.cov[1][1];
        const real det_0 = (real)fmax(1e-6, (double)(c00 * c11 - c01 * c01));
        const real det_1 = (real)fmax(1e-6, (double)((c00 + kernel_size) * (c11 + kernel_size) - c01 * c01));
        const real coef = (real)sqrt((double)det_0 / ((double)det_1 + 1e-6) + 1e-6);
        const real combined_opacity = conic_opacity[4 * (size_t)idx + 3];
        const real opacity = (real)((double)combined_opacity / ((double)coef + 1e-6));
        const real dL_dcoef = dop * opacity;
        const real dL_dsqrtcoef = (real)((double)dL_dcoef * 0.5 * 1. / ((double)coef + 1e-6));
        const real dL_ddet0 = (real)((double)dL_dsqrtcoef / ((double)det_1 + 1e-6));
        const real dL_ddet1 = (real)((double)(dL_dsqrtcoef * det_0) * (double)(RL(-1.0) / (real)((double)(det_1 * det_1) + 1e-6)));
        const real dcoef_da = dL_ddet0 * c11 + dL_ddet1 * (c11 + kernel_size);
        const real dcoef_db = (real)((double)dL_ddet0 * (-2. * (double)c01) + (double)dL_ddet1 * (-2. * (double)c01));
        const real dcoef_dc = dL_ddet0 * c00 + dL_ddet1 * (c00 + kernel_size);
        const real aa = c00 + kernel_size, b = c01, cc = c11 + kernel_size;
        const real denom = aa * cc - b * b;
        real dL_da = 0, dL_db = 0, dL_dc = 0;
        const real denom2inv = RL(1.0) / ((denom * denom) + RL(0.0000001));
        real* dcov = dL_dcov3D + 6 * (size_t)idx;
        const real(*T)[3] = e.T;
        const real(*V)[3] = e.Vrk;
        if (denom2inv != 0) {
            dL_da = denom2inv * (-cc * cc * dcon[0] + 2 * b * cc * dcon[1] + (denom - aa * cc) * dcon[2]);
            dL_dc = denom2inv * (-aa * aa * dcon[2] + 2 * aa * b * dcon[1] + (denom - aa * cc) * dcon[0]);
            dL_db = denom2inv * 2 * (b * cc * dcon[0] - (denom + 2 * b * b) * dcon[1] + aa * b * dcon[2]);
            if ((double)det_0 <= 1e-6 || (double)det_1 <= 1e-6) {
                dop = 0;
            } else {
                dL_da += dcoef_da;
                dL_dc += dcoef_dc;
                dL_db += dcoef_db;
                dop = dop * coef;
            }
            dcov[0] = (T[0][0] * T[0][0] * dL_da + T[0][0] * T[1][0] * dL_db + T[1][0] * T[1][0] * dL_dc);
            dcov[3] = (T[0][1] * T[0][1] * dL_da + T[0][1] * T[1][1] * dL_db + T[1][1] * T[1][1] * dL_dc);
            dcov[5] = (T[0][2] * T[0][2] * dL_da + T[0][2] * T[1][2] * dL_db + T[1][2] * T[1][2] * dL_dc);
            dcov[1] = 2 * T[0][0] * T[0][1] * dL_da + (T[0][0] * T[1][1] + T[0][1] * T[1][0]) * dL_db + 2 * T[1][0] * T[1][1] * dL_dc;
            dcov[2] = 2 * T[0][0] * T[0][2] * dL_da + (T[0][0] * T[1][2] + T[0][2] * T[1][0]) * dL_db + 2 * T[1][0] * T[1][2] * dL_dc;
            dcov[4] = 2 * T[0][2] * T[0][1] * dL_da + (T[0][1] * T[1][2] + T[0][2] * T[1][1]) * dL_db + 2 * T[1][1] * T[1][2] * dL_dc;
        }
        dL_dopacity[idx] = dop;
        real dT0[3], dT1[3];
        for (int k = 0; k < 3; ++k) {
            const real r0 = T[0][0] * V[k][0] + T[0][1] * V[k][1] + T[0][2] * V[k][2];
            const real r1 = T[1][0] * V[k][0] + T[1][1] * V[k][1] + T[1][2] * V[k][2];
            dT0[k] = 2 * r0 * dL_da + r1 * dL_db;
            dT1[k] = 2 * r1 * dL_dc + r0 * dL_db;
        }
        /* W[c][r] = view[4*r + c] */
        const real dL_dJ00 = view[0] * dT0[0] + view[4] * dT0[1] + view[8] * dT0[2];
        const real dL_dJ02 = view[2] * dT0[0] + view[6] * dT0[1] + view[10] * dT0[2];
        const real dL_dJ11 = view[1] * dT1[0] + view[5] * dT1[1] + view[9] * dT1[2];
        const real dL_dJ12 = view[2] * dT1[0] + view[6] * dT1[1] + view[10] * dT1[2];
        const real tz = RL(1.0) / t[2], tz2 = tz * tz, tz3 = tz2 * tz;
        const real dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
        const real dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
        const real dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * t[0]) * tz3 * dL_dJ02 + (2 * h_y * t[1]) * tz3 * dL_dJ12;
        real dmean[3] = {view[0] * dL_dtx + view[1] * dL_dty + view[2] * dL_dtz,
                         view[4] * dL_dtx + view[5] * dL_dty + view[6] * dL_dtz,
                         view[8] * dL_dtx + view[9] * dL_dty + view[10] * dL_dtz};
        /* backward.cu:402-423 */
        const real mw_raw = proj[3] * mean[0] + proj[7] * mean[1] + proj[11] * mean[2] + proj[15];
        const real m_w = RL(1.0) / (mw_raw + RL(0.0000001));
        const real mul1 = (proj[0] * mean[0] + proj[4] * mean[1] + proj[8] * mean[2] + proj[12]) * m_w * m_w;
        const real mul2 = (proj[1] * mean[0] + proj[5] * mean[1] + proj[9] * mean[2] + proj[13]) * m_w * m_w;
        dmean[0] += (proj[0] * m_w - proj[3] * mul1) * m2d[0] + (proj[1] * m_w - proj[3] * mul2) * m2d[1];
        dmean[1] += (proj[4] * m_w - proj[7] * mul1) * m2d[0] + (proj[5] * m_w - proj[7] * mul2) * m2d[1];
        dmean[2] += (proj[8] * m_w - proj[11] * mul1) * m2d[0] + (proj[9] * m_w - proj[11] * mul2) * m2d[1];

        if (shs) { /* backward.cu:20-139 */
            const real* sh = shs + (size_t)idx * M * 3;
            real* dsh = dL_dsh + (size_t)idx * M * 3;
            const real dir_orig[3] = {mean[0] - campos[0], mean[1] - campos[1], mean[2] - campos[2]};
            const real len = R_SQRT(dir_orig[0] * dir_orig[0] + dir_orig[1] * dir_orig[1] + dir_orig[2] * dir_orig[2]);
            const real x = dir_orig[0] / len, y = dir_orig[1] / len, z = dir_orig[2] / len;
            real g[3];
            for (int c = 0; c < 3; ++c) g[c] = clamped[3 * (size_t)idx + c] ? 0 : dcol[c];
            real dx_[3] = {0, 0, 0}, dy_[3] = {0, 0, 0}, dz_[3] = {0, 0, 0};
#define SHV(k, c) sh[3 * (k) + (c)]
#define PUT(k, w) do { for (int c = 0; c < 3; ++c) dsh[3 * (k) + c] = (w) * g[c]; } while (0)
            PUT(0, SH_C0);
            if (D > 0) {
                PUT(1, -SH_C1 * y); PUT(2, SH_C1 * z); PUT(3, -SH_C1 * x);
                for (int c = 0; c < 3; ++c) { dx_[c] = -SH_C1 * SHV(3, c); dy_[c] = -SH_C1 * SHV(1, c); dz_[c] = SH_C1 * SHV(2, c); }
                if (D > 1) {
                    const real xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                    PUT(4, SH_C2[0] * xy); PUT(5, SH_C2[1] * yz); PUT(6, SH_C2[2] * (RL(2.0) * zz - xx - yy));
                    PUT(7, SH_C2[3] * xz); PUT(8, SH_C2[4] * (xx - yy));
                    for (int c = 0; c < 3; ++c) {
                        dx_[c] += SH_C2[0] * y * SHV(4, c) + SH_C2[2] * RL(2.0) * -x * SHV(6, c) + SH_C2[3] * z * SHV(7, c) + SH_C2[4] * RL(2.0) * x * SHV(8, c);
                        dy_[c] += SH_C2[0] * x * SHV(4, c) + SH_C2[1] * z * SHV(5, c) + SH_C2[2] * RL(2.0) * -y * SHV(6, c) + SH_C2[4] * RL(2.0) * -y * SHV(8, c);
                        dz_[c] += SH_C2[1] * y * SHV(5, c) + SH_C2[2] * RL(2.0) * RL(2.0) * z * SHV(6, c) + SH_C2[3] * x * SHV(7, c);
                    }
                    if (D > 2) {
                        PUT(9, SH_C3[0] * y * (RL(3.0) * xx - yy));
                        PUT(10, SH_C3[1] * xy * z);
                        PUT(11, SH_C3[2] * y * (RL(4.0) * zz - xx - yy));
                        PUT(12, SH_C3[3] * z * (RL(2.0) * zz - RL(3.0) * xx - RL(3.0) * yy));
                        PUT(13, SH_C3[4] * x * (RL(4.0) * zz - xx - yy));
                        PUT(14, SH_C3[5] * z * (xx - yy));
                        PUT(15, SH_C3[6] * x * (xx - RL(3.0) * yy));
                        for (int c = 0; c < 3; ++c) {
                            dx_[c] += (SH_C3[0] * SHV(9, c) * RL(3.0) * RL(2.0) * xy + SH_C3[1] * SHV(10, c) * yz +
                                       SH_C3[2] * SHV(11, c) * RL(-2.0) * xy + SH_C3[3] * SHV(12, c) * RL(-3.0) * RL(2.0) * xz +
                                       SH_C3[4] * SHV(13, c) * (RL(-3.0) * xx + RL(4.0) * zz - yy) +
                                       SH_C3[5] * SHV(14, c) * RL(2.0) * xz + SH_C3[6] * SHV(15, c) * RL(3.0) * (xx - yy));
                            dy_[c] += (SH_C3[0] * SHV(9, c) * RL(3.0) * (xx - yy) + SH_C3[1] * SHV(10, c) * xz +
                                       SH_C3[2] * SHV(11, c) * (RL(-3.0) * yy + RL(4.0) * zz - xx) +
                                       SH_C3[3] * SHV(12, c) * RL(-3.0) * RL(2.0) * yz + SH_C3[4] * SHV(13, c) * RL(-2.0) * xy +
                                       SH_C3[5] * SHV(14, c) * RL(-2.0) * yz + SH_C3[6] * SHV(15, c) * RL(-3.0) * RL(2.0) * xy);
                            dz_[c] += (SH_C3[1] * SHV(10, c) * xy + SH_C3[2] * SHV(11, c) * RL(4.0) * RL(2.0) * yz +
                                       SH_C3[3] * SHV(12, c) * RL(3.0) * (RL(2.0) * zz - xx - yy) +
                                       SH_C3[4] * SHV(13, c) * RL(4.0) * RL(2.0) * xz + SH_C3[5] * SHV(14, c) * (xx - yy));
                        }
                    }
                }
            }
#undef SHV
#undef PUT
            const real ddir[3] = {dx_[0] * g[0] + dx_[1] * g[1] + dx_[2] * g[2],
                                  dy_[0] * g[0] + dy_[1] * g[1] + dy_[2] * g[2],
                                  dz_[0] * g[0] + dz_[1] * g[1] + dz_[2] * g[2]};
            real dm[3];
            dnormvdv3(dir_orig, ddir, dm);
            dmean[0] += dm[0]; dmean[1] += dm[1]; dmean[2] += dm[2];
        }
        for (int k = 0; k < 3; ++k) dL_dmean3D[3 * (size_t)idx + k] = dmean[k];

        if (scales) { /* backward.cu:314-377 */
            const real* q = rotations + 4 * (size_t)idx;
            const real r = q[0], x = q[1], y = q[2], z = q[3];
            real R[3][3], S[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, Mm[3][3], M2[3][3], dSig[3][3], dM[3][3], Rt[3][3], dMt[3][3];
            quat_to_R(q, R);
            const real s[3] = {scale_modifier * scales[3 * (size_t)idx], scale_modifier * scales[3 * (size_t)idx + 1],
                               scale_modifier * scales[3 * (size_t)idx + 2]};
            S[0][0] = s[0]; S[1][1] = s[1]; S[2][2] = s[2];
            mat3_mul(S, R, Mm);
            real ds[3][3] = {{dcov[0], RL(0.5) * dcov[1], RL(0.5) * dcov[2]},
                             {RL(0.5) * dcov[1], dcov[3], RL(0.5) * dcov[4]},
                             {RL(0.5) * dcov[2], RL(0.5) * dcov[4], dcov[5]}};
            memcpy(dSig, ds, sizeof(ds));
            for (int c = 0; c < 3; ++c) for (int rr = 0; rr < 3; ++rr) M2[c][rr] = RL(2.0) * Mm[c][rr];
            mat3_mul(M2, dSig, dM);
            mat3_transpose(R, Rt);
            mat3_transpose(dM, dMt);
            real* dsc = dL_dscale + 3 * (size_t)idx;
            for (int k = 0; k < 3; ++k) dsc[k] = Rt[k][0] * dMt[k][0] + Rt[k][1] * dMt[k][1] + Rt[k][2] * dMt[k][2];
            for (int k = 0; k < 3; ++k) { dMt[0][k] *= s[0]; dMt[1][k] *= s[1]; dMt[2][k] *= s[2]; }
            real* dq = dL_drot + 4 * (size_t)idx;
            dq[0] = 2 * z * (dMt[0][1] - dMt[1][0]) + 2 * y * (dMt[2][0] - dMt[0][2]) + 2 * x * (dMt[1][2] - dMt[2][1]);
            dq[1] = 2 * y * (dMt[1][0] + dMt[0][1]) + 2 * z * (dMt[2][0] + dMt[0][2]) + 2 * r * (dMt[1][2] - dMt[2][1]) - 4 * x * (dMt[2][2] + dMt[1][1]);
            dq[2] = 2 * x * (dMt[1][0] + dMt[0][1]) + 2 * r * (dMt[2][0] - dMt[0][2]) + 2 * z * (dMt[1][2] + dMt[2][1]) - 4 * y * (dMt[2][2] + dMt[0][0]);
            dq[3] = 2 * r * (dMt[0][1] - dMt[1][0]) + 2 * x * (dMt[2][0] + dMt[0][2]) + 2 * y * (dMt[1][2] + dMt[2][1]) - 4 * z * (dMt[1][1] + dMt[0][0]);
        }
    }
}

/* rasterizer_impl.cu:54-66 */
void oracle_mark_visible(int P, const real* means3D, const real* view, uint8_t* present) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; ++i) {
        const real* p = means3D + 3 * (size_t)i;
        present[i] = !(xform_row(view, 2, p[0], p[1], p[2]) <= RL(0.2));
    }
}
