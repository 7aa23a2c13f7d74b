// preprocess_bwd.cu -- per-Gaussian backward: from the compositing partials
// (dL/d{mean2D, conic, opacity*coef, colour}) to the gradients of the rasterizer inputs.
//
// One fused kernel replaces the reference's two per-Gaussian launches, computeCov2DCUDA
// (backward.cu:144-310) and preprocessCUDA<3> (backward.cu:382-432, with the SH backward
// :20-139 and the scale/rotation backward :314-377).  Fusing removes the dL_dcov3D and
// dL_dmeans round trips through HBM between the two, and cov3D is recomputed from
// scale/rotation instead of being read back from the forward's scratch.  Every output row
// is written here (zeros for Gaussians that were not rendered), so the host does not have
// to zero-fill nine gradient tensors first (rasterize_points.cu:157-165).
// The reference's opacity-compensation gradient (backward.cu:199-217) is mixed fp32/fp64; it is evaluated in
// fp32 here (gradients are compared at 1e-3; see the comment in the kernel).
#include "common.cuh"
#include "gaussian_math.cuh"
#include "sh_math.cuh"

namespace gsr {

struct PreBwdParams {
    int P, D, M;
    int sh_vec;             // SH rows are 16-byte aligned multiples of 16 bytes
    float focal_x, focal_y, tan_fovx, tan_fovy, kernel_size, scale_modifier;
    const float* means3D;
    const int* radii;
    const float* shs;
    const uint8_t* clamped;
    const float* scales;
    const float* rotations;
    const float* cov3D_precomp;
    const float* view;
    const float* proj;
    const float* campos;
    const float4* rec;
    const float* accum;     // [P][12]
    float* accum_clear;     // the same array, whose consumed rows the kernel zeroes; NULL in pull mode (the other ranks still read it)
    // pull-mode multi-GPU reduction (gsrast.h, gsr_backward_finalize_pull): complete sums = rows of all ranks in rank order
    const float* pull_accums[GSR_MAX_PULL_PEERS];            // the ranks' accumulators (peer-mapped), by value: no pointer-table load
    const unsigned char* pull_touched[GSR_MAX_PULL_PEERS];   // the ranks' mark arrays
    int pull_n, pull_self;                                   // pull_n == 0: single-accumulator mode
    float* pull_clear_accum;                  // previous pass's own accumulator: rows marked in pull_clear_touched are zeroed
    unsigned char* pull_clear_touched;
    float* dL_dmean2D;      // [P,3]
    float* dL_dconic;       // [P,4] or NULL
    float* dL_dopacity;     // [P]
    float* dL_dcolor;       // [P,3]
    float* dL_dmean3D;      // [P,3]
    float* dL_dcov3D;       // [P,6] or NULL
    float* dL_dsh;          // [P,M,3] or NULL
    float* dL_dscale;       // [P,3] or NULL
    float* dL_drot;         // [P,4] or NULL
};

// SH colour backward (what backward.cu:20-139 computes): colour_c = max(sum_k b_k(dir) sh[k][c] + 0.5, 0), so
//   dL/dsh[k][c] = b_k(dir) * dL/dcolour_c            (0 for clamped channels and for k above the active degree)
//   dL/ddir      = sum_k (sum_c dL/dcolour_c sh[k][c]) * grad b_k(dir),   then through dir = v / |v| to the mean.
// Writes the dL_dsh row, returns the mean gradient caused by the view direction.  `vec`: rows are aligned multiples of
// 16 bytes -- the coefficients are read and the gradient row is written with 128-bit accesses (a scalar access pattern
// makes every instruction of a warp touch 32 sectors, one per Gaussian: measured 8x slower per Gaussian).
__device__ __forceinline__ float3 sh_backward(int deg, int max_coeffs, const float* __restrict__ sh_base, bool vec, float3 mean,
                                              const float* __restrict__ campos, unsigned clamp_bits, V3 dL_dRGB,
                                              float* __restrict__ dL_dsh_base) {
    const float3 v = {mean.x - campos[0], mean.y - campos[1], mean.z - campos[2]};
    const float inv_len = 1.0f / sqrtf(v.x * v.x + v.y * v.y + v.z * v.z);
    const float3 dir = {v.x * inv_len, v.y * inv_len, v.z * inv_len};
    if (clamp_bits & 1u) dL_dRGB.x = 0.f;
    if (clamp_bits & 2u) dL_dRGB.y = 0.f;
    if (clamp_bits & 4u) dL_dRGB.z = 0.f;

    const int used = (deg + 1) * (deg + 1);
    float shl[48];
    if (vec) {
        const float4* p4 = reinterpret_cast<const float4*>(sh_base);
        const int n4 = (3 * used + 3) >> 2;
#pragma unroll
        for (int i = 0; i < 12; ++i) {
            if (i < n4) {
                const float4 q = __ldg(p4 + i);
                shl[4 * i + 0] = q.x; shl[4 * i + 1] = q.y; shl[4 * i + 2] = q.z; shl[4 * i + 3] = q.w;
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < 48; ++i)
            if (i < 3 * used) shl[i] = sh_base[i];
    }
    float w[16], g[16];
    sh_basis(deg, dir.x, dir.y, dir.z, w);
#pragma unroll
    for (int k = 0; k < 16; ++k)
        g[k] = k < used ? dL_dRGB.x * shl[3 * k] + dL_dRGB.y * shl[3 * k + 1] + dL_dRGB.z * shl[3 * k + 2] : 0.f;

    // dL_dsh[k][c] = w[k] * dL_dRGB[c]; coefficients above the active degree get 0 (w[k] = 0)
    if (vec) {
        float4* o4 = reinterpret_cast<float4*>(dL_dsh_base);
        const int groups = (max_coeffs * 3) >> 2;   // 4 coefficients (12 floats) = 3 float4 per group of four
#pragma unroll
        for (int g4 = 0; g4 < 4; ++g4) {
            if (3 * g4 < groups) {
                const float w0 = w[4 * g4], w1 = w[4 * g4 + 1], w2 = w[4 * g4 + 2], w3 = w[4 * g4 + 3];
                o4[3 * g4 + 0] = make_float4(w0 * dL_dRGB.x, w0 * dL_dRGB.y, w0 * dL_dRGB.z, w1 * dL_dRGB.x);
                o4[3 * g4 + 1] = make_float4(w1 * dL_dRGB.y, w1 * dL_dRGB.z, w2 * dL_dRGB.x, w2 * dL_dRGB.y);
                o4[3 * g4 + 2] = make_float4(w2 * dL_dRGB.z, w3 * dL_dRGB.x, w3 * dL_dRGB.y, w3 * dL_dRGB.z);
            }
        }
    } else {
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            if (k < max_coeffs) {
                dL_dsh_base[3 * k + 0] = w[k] * dL_dRGB.x;
                dL_dsh_base[3 * k + 1] = w[k] * dL_dRGB.y;
                dL_dsh_base[3 * k + 2] = w[k] * dL_dRGB.z;
            }
        }
        for (int k = 16; k < max_coeffs; ++k) {      // tensors holding more than degree-3 coefficients
            dL_dsh_base[3 * k + 0] = 0.f;
            dL_dsh_base[3 * k + 1] = 0.f;
            dL_dsh_base[3 * k + 2] = 0.f;
        }
    }
    return through_normalize(dir, inv_len, sh_basis_grad_dot(deg, dir.x, dir.y, dir.z, g));
}

template <int MIN_CTAS, bool HAS_SH>
__global__ void __launch_bounds__(256, MIN_CTAS) preprocess_bwd_kernel(const __grid_constant__ PreBwdParams p) {
    __shared__ float s_view[16];
    __shared__ float s_proj[16];
    if (threadIdx.x < 16) s_view[threadIdx.x] = p.view[threadIdx.x];
    else if (threadIdx.x < 32) s_proj[threadIdx.x - 16] = p.proj[threadIdx.x - 16];
    __syncthreads();

    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= p.P) return;

    const bool rendered = p.radii[idx] > 0;

    float o_mean2D[3] = {0.f, 0.f, 0.f};
    float o_conic[4] = {0.f, 0.f, 0.f, 0.f};
    float o_opacity = 0.f;
    float o_color[3] = {0.f, 0.f, 0.f};
    float o_mean3D[3] = {0.f, 0.f, 0.f};
    float o_cov3D[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float o_scale[3] = {0.f, 0.f, 0.f};
    float o_rot[4] = {0.f, 0.f, 0.f, 0.f};
    bool sh_written = false;

    // A visible Gaussian that no pixel blended (occluded, or alpha < 1/255 everywhere: most of a dense scene) has an
    // all-zero row of sums: every gradient of it is zero, so its inputs are not even read.
    float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0;
    if (p.pull_n > 0) {
        // rows of all ranks, added in rank order (identical on every rank -> bit-identical gradients everywhere); a rank that
        // did not mark the Gaussian contributes an all-zero row, which is skipped (x + 0 = x) without reading it.  All marks
        // are requested first (independent remote loads: one NVLink round trip, not one per rank).
        if (rendered) {
            unsigned char mark[GSR_MAX_PULL_PEERS];
#pragma unroll
            for (int r = 0; r < GSR_MAX_PULL_PEERS; ++r)
                mark[r] = (r < p.pull_n && r != p.pull_self) ? p.pull_touched[r][idx] : (unsigned char)(r == p.pull_self);
#pragma unroll
            for (int r = 0; r < GSR_MAX_PULL_PEERS; ++r) {
                if (r >= p.pull_n || mark[r] == 0) continue;
                const float4* acc = reinterpret_cast<const float4*>((r == p.pull_self ? p.accum : p.pull_accums[r]) + (size_t)idx * 12);
                const float4 b0 = acc[0], b1 = acc[1], b2 = acc[2];
                a0.x += b0.x; a0.y += b0.y; a0.z += b0.z; a0.w += b0.w;
                a1.x += b1.x; a1.y += b1.y; a1.z += b1.z; a1.w += b1.w;
                a2.x += b2.x; a2.y += b2.y;
            }
        }
        // the PREVIOUS pass's buffers are no longer read by anyone (every rank passed this pass's barrier after finishing that
        // pass's chain rule): zero the rows this rank marked then, and the marks
        if (p.pull_clear_touched != nullptr && p.pull_clear_touched[idx] != 0) {
            float4* w = reinterpret_cast<float4*>(p.pull_clear_accum + (size_t)idx * 12);
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            w[0] = z; w[1] = z; w[2] = z;
            p.pull_clear_touched[idx] = 0;
        }
    } else if (rendered) {
        const float4* acc = reinterpret_cast<const float4*>(p.accum + (size_t)idx * 12);
        a0 = acc[0]; a1 = acc[1]; a2 = acc[2];
    }
    const bool touched = (a0.x != 0.f) | (a0.y != 0.f) | (a0.z != 0.f) | (a0.w != 0.f) | (a1.x != 0.f) | (a1.y != 0.f) |
                         (a1.z != 0.f) | (a1.w != 0.f) | (a2.x != 0.f) | (a2.y != 0.f);
    // keep the accumulator all-zero between passes by clearing just the rows that were non-zero (typically 10-20 % of the
    // Gaussians) instead of a 48 B x P memset after the kernel
    if (touched && p.accum_clear != nullptr) {
        float4* w = reinterpret_cast<float4*>(p.accum_clear + (size_t)idx * 12);
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        w[0] = z; w[1] = z; w[2] = z;
    }

    if (rendered && touched) {
        o_mean2D[0] = a0.x; o_mean2D[1] = a0.y; o_mean2D[2] = a0.z;
        o_conic[0] = a0.w; o_conic[1] = a1.x; o_conic[3] = a1.y;
        float dL_dopacity = a1.z;
        o_color[0] = a1.w; o_color[1] = a2.x; o_color[2] = a2.y;

        const float3 mean = {p.means3D[3 * idx], p.means3D[3 * idx + 1], p.means3D[3 * idx + 2]};

        float cov3D_local[6];
        const float* cov3D;
        float3 sc = {0.f, 0.f, 0.f};
        float4 rot = {0.f, 0.f, 0.f, 0.f};
        if (p.cov3D_precomp != nullptr) {
            cov3D = p.cov3D_precomp + 6 * (size_t)idx;
        } else {
            sc = float3{p.scales[3 * idx], p.scales[3 * idx + 1], p.scales[3 * idx + 2]};
            rot = reinterpret_cast<const float4*>(p.rotations)[idx];
            cov3d_from_scale_rot(sc, p.scale_modifier, rot, cov3D_local);
            cov3D = cov3D_local;
        }

        // ---- screen-space covariance / conic / compensation backward (what backward.cu:144-310 computes) ----------
        // Own derivation.  With the two rows t0, t1 of the 2x3 projection A = J W (columns 0 / 1 of the GLM matrix T):
        //   cov2D = A Sigma A^T + k I = [[a, b], [b, c]],   conic = cov2D^-1,   opacity' = opacity * coef(cov2D).
        const float4 rb = p.rec[2 * (size_t)idx + 1];
        const float fx = p.focal_x, fy = p.focal_y, ks = p.kernel_size;
        const Ewa e = ewa_project(mean, fx, fy, p.tan_fovx, p.tan_fovy, cov3D, s_view);
        const V3 t0 = {e.T.m[0][0], e.T.m[0][1], e.T.m[0][2]};
        const V3 t1 = {e.T.m[1][0], e.T.m[1][1], e.T.m[1][2]};
        const float ca0 = e.cov.m[0][0], b = e.cov.m[0][1], cc0 = e.cov.m[1][1];      // before the low-pass
        const float a = ca0 + ks, c = cc0 + ks;

        // (1) conic -> cov2D.  For K = cov^-1 and the symmetric gradient Gk = [[gx, gy], [gy, gz]] (gy is the
        //     per-off-diagonal-entry gradient the composite accumulates), dL/dcov = -adj Gk adj / det^2 with
        //     adj = [[c, -b], [-b, a]]; the reference regularises det^2 by + 1e-7 (backward.cu:229) -- kept.
        const float gx = o_conic[0], gy = o_conic[1], gz = o_conic[3];
        const float det = a * c - b * b;
        const float N = 1.0f / (det * det + 0.0000001f);
        float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
        if (N != 0.f) {
            const float r0x = c * gx - b * gy, r0y = c * gy - b * gz;      // row 0 of adj Gk
            const float r1x = a * gy - b * gx, r1y = a * gz - b * gy;      // row 1 of adj Gk
            dL_da = -N * (r0x * c - r0y * b);
            dL_db = -2.0f * N * (r0y * a - r0x * b);
            dL_dc = -N * (r1y * a - r1x * b);

            // (2) opacity compensation coef = sqrt(det0 / (det1 + eps) + eps), det0 / det1 before / after the low-pass
            //     (forward.cu:112-118; evaluated in fp32 here, the reference's mixed fp32 / fp64 only matters for the
            //     forward's bit-exact opacity; its eps terms and its clamps at 1e-6 are kept)
            const float det0 = fmaxf(1e-6f, ca0 * cc0 - b * b);
            const float det1 = fmaxf(1e-6f, a * c - b * b);
            if (det0 <= 1e-6f || det1 <= 1e-6f) {
                dL_dopacity = 0.f;
            } else {
                const float inv1 = 1.0f / (det1 + 1e-6f);
                const float coef = sqrtf(det0 * inv1 + 1e-6f);
                const float inv_c = 1.0f / (coef + 1e-6f);
                const float half = 0.5f * dL_dopacity * (rb.w * inv_c) * inv_c;       // dL/d(det0 / (det1 + eps))
                const float d0 = half * inv1;                                          // dL/ddet0
                const float d1 = -half * det0 / (det1 * det1 + 1e-6f);                 // dL/ddet1
                dL_da += d0 * cc0 + d1 * c;
                dL_db -= 2.0f * b * (d0 + d1);
                dL_dc += d0 * ca0 + d1 * a;
                dL_dopacity *= coef;
            }
        }
        o_opacity = dL_dopacity;

        // (3) cov2D -> Sigma and -> the projection rows.  G = dL_da t0 t0^T + dL_db/2 (t0 t1^T + t1 t0^T) + dL_dc t1 t1^T
        //     is dL/dSigma (rank 2); dL/dt0 = 2 dL_da Sigma t0 + dL_db Sigma t1, dL/dt1 = 2 dL_dc Sigma t1 + dL_db Sigma t0.
        const Mat3& S3 = e.Vrk;                   // Sigma (symmetric), already in registers
        auto sym = [&](const V3& v) -> V3 {       // Sigma v
            return {S3.m[0][0] * v.x + S3.m[1][0] * v.y + S3.m[2][0] * v.z, S3.m[0][1] * v.x + S3.m[1][1] * v.y + S3.m[2][1] * v.z,
                    S3.m[0][2] * v.x + S3.m[1][2] * v.y + S3.m[2][2] * v.z};
        };
        const V3 u0 = sym(t0), u1 = sym(t1);
        const V3 g0 = (2.0f * dL_da) * u0 + dL_db * u1;
        const V3 g1 = (2.0f * dL_dc) * u1 + dL_db * u0;
        if (N != 0.f) {      // stored like the reference: diagonal entries, and off-diagonals carrying both symmetric halves
            o_cov3D[0] = dL_da * t0.x * t0.x + dL_db * t0.x * t1.x + dL_dc * t1.x * t1.x;
            o_cov3D[3] = dL_da * t0.y * t0.y + dL_db * t0.y * t1.y + dL_dc * t1.y * t1.y;
            o_cov3D[5] = dL_da * t0.z * t0.z + dL_db * t0.z * t1.z + dL_dc * t1.z * t1.z;
            o_cov3D[1] = 2.0f * (dL_da * t0.x * t0.y + dL_dc * t1.x * t1.y) + dL_db * (t0.x * t1.y + t0.y * t1.x);
            o_cov3D[2] = 2.0f * (dL_da * t0.x * t0.z + dL_dc * t1.x * t1.z) + dL_db * (t0.x * t1.z + t0.z * t1.x);
            o_cov3D[4] = 2.0f * (dL_da * t0.y * t0.z + dL_dc * t1.y * t1.z) + dL_db * (t0.y * t1.z + t0.z * t1.y);
        }

        // (4) projection rows -> view-space mean.  t0 = J00 w0 + J02 w2, t1 = J11 w1 + J12 w2 with w_r the view axes in world
        //     coordinates and J00 = fx / z, J02 = -fx x / z^2, J11 = fy / z, J12 = -fy y / z^2 (x, y clamped to the frustum
        //     guard band: no gradient to x / y where the clamp is active).
        const V3 w0 = {s_view[0], s_view[4], s_view[8]}, w1 = {s_view[1], s_view[5], s_view[9]}, w2 = {s_view[2], s_view[6], s_view[10]};
        const float dJ00 = dot3(w0, g0), dJ02 = dot3(w2, g0), dJ11 = dot3(w1, g1), dJ12 = dot3(w2, g1);
        const float iz = 1.0f / e.t.z, iz2 = iz * iz, iz3 = iz2 * iz;
        const bool x_free = !(e.txtz < -e.limx || e.txtz > e.limx), y_free = !(e.tytz < -e.limy || e.tytz > e.limy);
        const float gvx = x_free ? -fx * iz2 * dJ02 : 0.f;
        const float gvy = y_free ? -fy * iz2 * dJ12 : 0.f;
        const float gvz = -iz2 * (fx * dJ00 + fy * dJ11) + 2.0f * iz3 * (fx * e.t.x * dJ02 + fy * e.t.y * dJ12);
        const V3 dmean_cov = gvx * w0 + gvy * w1 + gvz * w2;

        // (5) screen position (NDC-scaled gradient from the composite) -> mean, through the projective divide
        //     ndc = (P m).xy / ((P m).w + 1e-7)   (forward.cu:210-212)
        const float* proj = s_proj;
        const float4 mh = xform_point_4x4(mean, proj);
        const float iw = 1.0f / (mh.w + 0.0000001f);
        const float nx = mh.x * iw, ny = mh.y * iw;                 // ndc.x, ndc.y
        const float qx = o_mean2D[0] * iw, qy = o_mean2D[1] * iw, qw = -(qx * nx + qy * ny);
        const V3 dmean_pos = {proj[0] * qx + proj[1] * qy + proj[3] * qw, proj[4] * qx + proj[5] * qy + proj[7] * qw,
                              proj[8] * qx + proj[9] * qy + proj[11] * qw};
        o_mean3D[0] = dmean_cov.x + dmean_pos.x;
        o_mean3D[1] = dmean_cov.y + dmean_pos.y;
        o_mean3D[2] = dmean_cov.z + dmean_pos.z;

        // ---- SH backward (backward.cu:20-139) ----
        if (HAS_SH) {
            const float3 g = sh_backward(p.D, p.M, p.shs + (size_t)idx * p.M * 3, p.sh_vec != 0, mean, p.campos, p.clamped[idx],
                                         V3{o_color[0], o_color[1], o_color[2]}, p.dL_dsh + (size_t)idx * p.M * 3);
            o_mean3D[0] += g.x;
            o_mean3D[1] += g.y;
            o_mean3D[2] += g.z;
            sh_written = true;
        }

        // ---- Sigma -> scale / rotation (what backward.cu:314-377 computes) ----------------------------------------
        // Sigma = sum_i s_i^2 r_i r_i^T with r_i the i-th local axis (row i of the GLM rotation matrix, raw quaternion,
        // note N5) and s_i = modifier * scale_i.  With G of rank 2:  G r_i = al_i t0 + be_i t1,
        //   al_i = dL_da (t0.r_i) + dL_db/2 (t1.r_i),  be_i = dL_db/2 (t0.r_i) + dL_dc (t1.r_i), so
        //   dL/ds_i = 2 s_i r_i^T G r_i      (the reference applies no modifier factor here either)
        //   h_i = dL/dr_i = 2 s_i^2 G r_i    and the quaternion gradient follows from the skew / symmetric parts of H = [h_i].
        if (p.scales != nullptr) {
            const float qr = rot.x, qx = rot.y, qy = rot.z, qz = rot.w;
            const Mat3 R = quat_to_mat(rot);
            const float sv[3] = {p.scale_modifier * sc.x, p.scale_modifier * sc.y, p.scale_modifier * sc.z};
            V3 h[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const V3 r = {R.m[0][i], R.m[1][i], R.m[2][i]};
                const float pi = dot3(t0, r), qi = dot3(t1, r);
                const float al = dL_da * pi + 0.5f * dL_db * qi, be = 0.5f * dL_db * pi + dL_dc * qi;
                o_scale[i] = 2.0f * sv[i] * (al * pi + be * qi);
                h[i] = (2.0f * sv[i] * sv[i]) * (al * t0 + be * t1);
            }
            const float ax = h[1].z - h[2].y, ay = h[2].x - h[0].z, az = h[0].y - h[1].x;      // skew part
            const float sxy = h[0].y + h[1].x, sxz = h[0].z + h[2].x, syz = h[1].z + h[2].y;   // symmetric part
            o_rot[0] = 2.0f * (qx * ax + qy * ay + qz * az);
            o_rot[1] = 2.0f * (qr * ax + qy * sxy + qz * sxz) - 4.0f * qx * (h[1].y + h[2].z);
            o_rot[2] = 2.0f * (qr * ay + qx * sxy + qz * syz) - 4.0f * qy * (h[0].x + h[2].z);
            o_rot[3] = 2.0f * (qr * az + qx * sxz + qy * syz) - 4.0f * qz * (h[0].x + h[1].y);
        }
    }

    // ---- write every output row ----
    const size_t i = (size_t)idx;
    p.dL_dmean2D[3 * i + 0] = o_mean2D[0];
    p.dL_dmean2D[3 * i + 1] = o_mean2D[1];
    p.dL_dmean2D[3 * i + 2] = o_mean2D[2];
    if (p.dL_dconic) reinterpret_cast<float4*>(p.dL_dconic)[i] = make_float4(o_conic[0], o_conic[1], 0.f, o_conic[3]);
    p.dL_dopacity[i] = o_opacity;
    p.dL_dcolor[3 * i + 0] = o_color[0];
    p.dL_dcolor[3 * i + 1] = o_color[1];
    p.dL_dcolor[3 * i + 2] = o_color[2];
    p.dL_dmean3D[3 * i + 0] = o_mean3D[0];
    p.dL_dmean3D[3 * i + 1] = o_mean3D[1];
    p.dL_dmean3D[3 * i + 2] = o_mean3D[2];
    if (p.dL_dcov3D) {
#pragma unroll
        for (int k = 0; k < 6; ++k) p.dL_dcov3D[6 * i + k] = o_cov3D[k];
    }
    if (HAS_SH && !sh_written) {
        float* row = p.dL_dsh + i * p.M * 3;
        if (p.sh_vec) {
            float4* r4 = reinterpret_cast<float4*>(row);
            for (int k = 0; k < (p.M * 3) >> 2; ++k) r4[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
            for (int k = 0; k < p.M * 3; ++k) row[k] = 0.f;
        }
    }
    if (p.dL_dscale) {
        p.dL_dscale[3 * i + 0] = o_scale[0];
        p.dL_dscale[3 * i + 1] = o_scale[1];
        p.dL_dscale[3 * i + 2] = o_scale[2];
    }
    if (p.dL_drot) reinterpret_cast<float4*>(p.dL_drot)[i] = make_float4(o_rot[0], o_rot[1], o_rot[2], o_rot[3]);
}

int launch_preprocess_bwd(const GsrBackwardArgs& a, const GeomState& g, BwdAccum* accum, cudaStream_t s, const PullPeers* pull) {
    PreBwdParams p;
    p.P = a.P; p.D = a.D; p.M = a.M;
    p.focal_y = a.H / (2.0f * a.tan_fovy);
    p.focal_x = a.W / (2.0f * a.tan_fovx);
    p.tan_fovx = a.tan_fovx; p.tan_fovy = a.tan_fovy;
    p.kernel_size = a.kernel_size; p.scale_modifier = a.scale_modifier;
    p.means3D = a.means3D; p.radii = a.radii; p.shs = a.shs; p.clamped = g.clamped;
    p.scales = a.scales; p.rotations = a.rotations; p.cov3D_precomp = a.cov3D_precomp;
    p.view = a.viewmatrix; p.proj = a.projmatrix; p.campos = a.campos;
    p.rec = g.rec; p.accum = reinterpret_cast<const float*>(accum);
    p.accum_clear = pull ? nullptr : reinterpret_cast<float*>(accum);
    for (int r = 0; r < GSR_MAX_PULL_PEERS; ++r) {
        p.pull_accums[r] = (pull && r < pull->n_peers) ? pull->accums[r] : nullptr;
        p.pull_touched[r] = (pull && r < pull->n_peers) ? pull->touched[r] : nullptr;
    }
    p.pull_n = pull ? pull->n_peers : 0;
    p.pull_self = pull ? pull->self : 0;
    p.pull_clear_accum = pull ? pull->clear_accum : nullptr;
    p.pull_clear_touched = pull ? pull->clear_touched : nullptr;
    p.dL_dmean2D = a.dL_dmean2D; p.dL_dconic = a.dL_dconic; p.dL_dopacity = a.dL_dopacity;
    p.dL_dcolor = a.dL_dcolor; p.dL_dmean3D = a.dL_dmean3D; p.dL_dcov3D = a.dL_dcov3D;
    p.dL_dsh = a.dL_dsh; p.dL_dscale = a.dL_dscale; p.dL_drot = a.dL_drot;
    p.sh_vec = a.shs != nullptr && (a.M == 4 || a.M == 16) &&
               (reinterpret_cast<uintptr_t>(a.shs) & 15u) == 0 && (reinterpret_cast<uintptr_t>(a.dL_dsh) & 15u) == 0;
    if (a.shs != nullptr) preprocess_bwd_kernel<2, true><<<(a.P + 255) / 256, 256, 0, s>>>(p);   // 48 + 16 extra live registers
    else preprocess_bwd_kernel<4, false><<<(a.P + 255) / 256, 256, 0, s>>>(p);
    count_launches(1);
    return 0;
}

}  // namespace gsr
