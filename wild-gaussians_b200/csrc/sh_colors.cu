// sh_colors.cu -- SH colours of wild-gaussians models WITHOUT appearance, one bandwidth-bound pass per direction.
//
// Replaces, for appearance_enabled = False and storage degree 3, the PyTorch statements of
// GaussianModel._render_internal (wildgaussians/method.py:1555-1565, features from get_gaussians :1061-1064):
//     features = cat(features_dc, features_rest).clamp_max(1)                    [P,48]
//     dir      = normalize(means3D - campos)                                     (F.normalize, eps 1e-12)
//     colors   = clamp_min(eval_sh(deg, features.view(-1,16,3).transpose(1,2), dir) + 0.5, 0)
// (cat, clamp, repeat, normalize, a P x 3 x 16 transpose copy, ~40 eval_sh statements and their autograd graph).
//
// The arithmetic is that of the raw-colour stage of the fused appearance op (appearance.cu): the same direction
// expressions, r = b[0] * f0 followed by fmaf(b[k], f_k, r), the same clamp masks, so the colours agree with
// fused_colors' raw output; the sum stops at the active degree (b[k] = 0 above it, so the bits are the same).
//
// One row per thread, SHC_ROWS rows per CTA.  A 45-float features_rest row is not 16-byte aligned, so per-thread
// row loads would be uncoalesced: each CTA stages its contiguous block of rows (SHC_ROWS x 180 B, a multiple of
// 16 B) through shared memory with 16-byte cp.async copies, and the backward stages the features_rest gradient the
// same way for coalesced 16-byte stores.  The row stride of 45 words is odd: per-thread shared-memory accesses are
// free of bank conflicts.  HBM bytes per row: forward reads 204 (dc 12 + rest 180 + mean 12), writes 12; backward
// reads 216 (+ dL/dcolour 12), writes 204.  The backward recomputes the forward, so the clamp masks are exact.
#include "common.cuh"
#include "sh_math.cuh"

namespace gsr {

constexpr int SHC_ROWS = 128;
constexpr int SHC_NREST = 45;

__device__ __forceinline__ void cp_async16(float* smem, const float* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem)
                 : "memory");
}

// issue the copy of rows [row0, row0 + rows) of features_rest into s_rest (completed by shc_stage_wait)
__device__ __forceinline__ void shc_stage_issue(const float* __restrict__ rest, int row0, int rows, float* s_rest) {
    const float* src = rest + (size_t)row0 * SHC_NREST;
    const int n = rows * SHC_NREST, n4 = n >> 2;
    for (int i = threadIdx.x; i < n4; i += SHC_ROWS) cp_async16(s_rest + 4 * i, src + 4 * i);
    for (int i = 4 * n4 + threadIdx.x; i < n; i += SHC_ROWS) s_rest[i] = src[i];
    asm volatile("cp.async.commit_group;" ::: "memory");
}
__device__ __forceinline__ void shc_stage_wait() {
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
}

struct ShcRow {
    float dc[3];        // unclamped features_dc
    float3 dir;         // normalised view direction
    float inv_norm;     // 1 / max(|mean - campos|, 1e-12)
};

__device__ __forceinline__ ShcRow shc_row(const float* __restrict__ dc, const float* __restrict__ means,
                                          const float* __restrict__ campos, int row) {
    ShcRow in;
#pragma unroll
    for (int c = 0; c < 3; ++c) in.dc[c] = dc[(size_t)row * 3 + c];
    const float vx = means[(size_t)row * 3 + 0] - campos[0], vy = means[(size_t)row * 3 + 1] - campos[1],
                vz = means[(size_t)row * 3 + 2] - campos[2];
    const float nrm = fmaxf(sqrtf(vx * vx + vy * vy + vz * vz), 1e-12f);      // F.normalize (method.py:1557)
    in.inv_norm = 1.0f / nrm;
    in.dir = {vx * in.inv_norm, vy * in.inv_norm, vz * in.inv_norm};
    return in;
}

// sum_k b_k min(f_k, 1) of channel c over the active coefficients (nk = (deg + 1)^2)
__device__ __forceinline__ float shc_sum(const float (&b)[16], int nk, float dc, const float* fr, int c) {
    float r = b[0] * fminf(dc, 1.0f);
#pragma unroll
    for (int k = 1; k < 16; ++k)
        if (k < nk) r = fmaf(b[k], fminf(fr[3 * (k - 1) + c], 1.0f), r);
    return r;
}

__global__ void __launch_bounds__(SHC_ROWS) sh_colors_fwd_kernel(int P, int deg, const float* __restrict__ dc,
                                                                 const float* __restrict__ rest,
                                                                 const float* __restrict__ means,
                                                                 const float* __restrict__ campos,
                                                                 float* __restrict__ colors) {
    __shared__ __align__(16) float s_rest[SHC_ROWS * SHC_NREST];
    const int row0 = blockIdx.x * SHC_ROWS, t = threadIdx.x, row = row0 + t;
    const int rows = min(SHC_ROWS, P - row0);
    shc_stage_issue(rest, row0, rows, s_rest);
    const bool valid = t < rows;
    ShcRow in{};
    float b[16];
    const int nk = (deg + 1) * (deg + 1);
    if (valid) {
        in = shc_row(dc, means, campos, row);
        sh_basis(deg, in.dir.x, in.dir.y, in.dir.z, b);
    }
    shc_stage_wait();
    if (!valid) return;
    const float* fr = s_rest + t * SHC_NREST;
#pragma unroll
    for (int c = 0; c < 3; ++c) colors[(size_t)row * 3 + c] = fmaxf(shc_sum(b, nk, in.dc[c], fr, c) + 0.5f, 0.f);
}

__global__ void __launch_bounds__(SHC_ROWS) sh_colors_bwd_kernel(int P, int deg, const float* __restrict__ dc,
                                                                 const float* __restrict__ rest,
                                                                 const float* __restrict__ means,
                                                                 const float* __restrict__ campos,
                                                                 const float* __restrict__ dL_dcolors,
                                                                 float* __restrict__ g_dc, float* __restrict__ g_rest,
                                                                 float* __restrict__ g_means) {
    __shared__ __align__(16) float s_rest[SHC_ROWS * SHC_NREST];
    const int row0 = blockIdx.x * SHC_ROWS, t = threadIdx.x, row = row0 + t;
    const int rows = min(SHC_ROWS, P - row0);
    shc_stage_issue(rest, row0, rows, s_rest);
    const bool valid = t < rows;
    ShcRow in{};
    float b[16], dL[3] = {0.f, 0.f, 0.f};
    const int nk = (deg + 1) * (deg + 1);
    if (valid) {
        in = shc_row(dc, means, campos, row);
        sh_basis(deg, in.dir.x, in.dir.y, in.dir.z, b);
        if (dL_dcolors) {
#pragma unroll
            for (int c = 0; c < 3; ++c) dL[c] = dL_dcolors[(size_t)row * 3 + c];
        }
    }
    shc_stage_wait();
    if (valid) {
        float* fr = s_rest + t * SHC_NREST;
        float gk[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) gk[k] = 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            // clamp_min(x + 0.5, 0) passes the gradient where x + 0.5 >= 0
            const float dLr = (shc_sum(b, nk, in.dc[c], fr, c) + 0.5f >= 0.f) ? dL[c] : 0.f;
            // clamp_max(1) passes it where the raw value <= 1
            g_dc[(size_t)row * 3 + c] = (in.dc[c] <= 1.0f) ? b[0] * dLr : 0.f;
#pragma unroll
            for (int k = 1; k < 16; ++k) {
                const float fu = fr[3 * (k - 1) + c];
                const bool active = k < nk;
                gk[k] += active ? dLr * fminf(fu, 1.0f) : 0.f;
                // gradient of features_rest, written in place of the row; exactly zero above the active degree
                fr[3 * (k - 1) + c] = (active && fu <= 1.0f) ? b[k] * dLr : 0.f;
            }
        }
        // view direction -> mean (eval_sh is differentiated through `dir`, method.py:1557)
        const float3 dd = sh_basis_grad_dot(deg, in.dir.x, in.dir.y, in.dir.z, gk);
        const float3 dm = through_normalize(in.dir, in.inv_norm, dd);
        g_means[(size_t)row * 3 + 0] = dm.x;
        g_means[(size_t)row * 3 + 1] = dm.y;
        g_means[(size_t)row * 3 + 2] = dm.z;
    }
    __syncthreads();
    // coalesced copy-out of the block's features_rest gradients (same 16-byte aligned layout as the input block)
    float* dst = g_rest + (size_t)row0 * SHC_NREST;
    const int n = rows * SHC_NREST, n4 = n >> 2;
    for (int i = t; i < n4; i += SHC_ROWS) reinterpret_cast<float4*>(dst)[i] = reinterpret_cast<const float4*>(s_rest)[i];
    for (int i = 4 * n4 + t; i < n; i += SHC_ROWS) dst[i] = s_rest[i];
}

static int shc_check(int P, int sh_degree) {
    if (P < 0 || sh_degree < 0 || sh_degree > 3) { set_error("bad P / sh_degree"); return GSR_E_INVALID; }
    return 0;
}

}  // namespace gsr

using namespace gsr;

extern "C" int gsr_sh_colors_forward(int P, int sh_degree, const float* features_dc, const float* features_rest,
                                     const float* means3D, const float* campos, float* colors, void* stream) {
    if (int rc = shc_check(P, sh_degree)) return rc;
    if (P == 0) return 0;
    if (!features_dc || !features_rest || !means3D || !campos || !colors) {
        set_error("a required pointer is NULL");
        return GSR_E_INVALID;
    }
    if (reinterpret_cast<uintptr_t>(features_rest) & 15u) { set_error("features_rest must be 16-byte aligned"); return GSR_E_INVALID; }
    sh_colors_fwd_kernel<<<(P + SHC_ROWS - 1) / SHC_ROWS, SHC_ROWS, 0, (cudaStream_t)stream>>>(P, sh_degree, features_dc,
                                                                                              features_rest, means3D, campos,
                                                                                              colors);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int gsr_sh_colors_backward(int P, int sh_degree, const float* features_dc, const float* features_rest,
                                      const float* means3D, const float* campos, const float* dL_dcolors,
                                      float* dL_dfeatures_dc, float* dL_dfeatures_rest, float* dL_dmeans3D, void* stream) {
    if (int rc = shc_check(P, sh_degree)) return rc;
    if (P == 0) return 0;
    if (!features_dc || !features_rest || !means3D || !campos || !dL_dfeatures_dc || !dL_dfeatures_rest || !dL_dmeans3D) {
        set_error("a required pointer is NULL");
        return GSR_E_INVALID;
    }
    if ((reinterpret_cast<uintptr_t>(features_rest) | reinterpret_cast<uintptr_t>(dL_dfeatures_rest)) & 15u) {
        set_error("features_rest / dL_dfeatures_rest must be 16-byte aligned");
        return GSR_E_INVALID;
    }
    sh_colors_bwd_kernel<<<(P + SHC_ROWS - 1) / SHC_ROWS, SHC_ROWS, 0, (cudaStream_t)stream>>>(
        P, sh_degree, features_dc, features_rest, means3D, campos, dL_dcolors, dL_dfeatures_dc, dL_dfeatures_rest, dL_dmeans3D);
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}
