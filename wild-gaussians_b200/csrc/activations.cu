// activations.cu -- parameter activations + 3D smoothing filter of wild-gaussians in one pass per direction
// (SURVEY.md 8f-2, "activations + 3D-filter").
//
// Replaces the PyTorch statements of GaussianModel.get_gaussians (wildgaussians/method.py:1060-1086):
//     rotations = normalize(rotations_raw)                         (F.normalize, eps 1e-12)
//     raw       = exp(scales_raw);  opac = sigmoid(opacities_raw)
//     scales    = sqrt(raw^2 + filter_3D^2)
//     coef      = sqrt(prod(raw^2) / prod(raw^2 + filter_3D^2));   opacities = opac * coef
// (about 15 elementwise launches forward and 25 backward over P x {1,3,4} tensors) by one bandwidth-bound kernel per
// direction: 36 B in + 32 B out per Gaussian forward; the backward recomputes the forward from the raw parameters.
#include "common.cuh"

namespace gsr {

struct ActRow {
    float raw2[3], a[3], s[3];      // raw^2, raw^2 + f^2, sqrt of it
    float sig, coef;
    float4 q;                       // raw quaternion
    float inv_n;                    // 1 / max(|q|, 1e-12)
    bool q_clamped;                 // |q| < 1e-12: F.normalize divides by the constant eps
};

__device__ __forceinline__ ActRow act_forward(const float* __restrict__ scales, const float* __restrict__ opac,
                                              const float4* __restrict__ rot, const float* __restrict__ filt, int i) {
    ActRow r;
    const float f = filt[i], f2 = f * f;
    float num = 1.f, den = 1.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float raw = expf(scales[3 * (size_t)i + k]);
        r.raw2[k] = raw * raw;
        r.a[k] = r.raw2[k] + f2;
        r.s[k] = sqrtf(r.a[k]);
        num *= r.raw2[k];
        den *= r.a[k];
    }
    r.coef = sqrtf(num / den);
    r.sig = 1.0f / (1.0f + expf(-opac[i]));
    r.q = rot[i];
    const float qn = sqrtf(r.q.x * r.q.x + r.q.y * r.q.y + r.q.z * r.q.z + r.q.w * r.q.w);
    r.q_clamped = qn < 1e-12f;
    r.inv_n = 1.0f / fmaxf(qn, 1e-12f);
    return r;
}

__global__ void __launch_bounds__(256) activations_fwd_kernel(int P, const float* __restrict__ scales, const float* __restrict__ opac,
                                                              const float4* __restrict__ rot, const float* __restrict__ filt,
                                                              float* __restrict__ o_scales, float* __restrict__ o_opac,
                                                              float4* __restrict__ o_rot) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const ActRow r = act_forward(scales, opac, rot, filt, i);
#pragma unroll
    for (int k = 0; k < 3; ++k) o_scales[3 * (size_t)i + k] = r.s[k];
    o_opac[i] = r.sig * r.coef;
    o_rot[i] = make_float4(r.q.x * r.inv_n, r.q.y * r.inv_n, r.q.z * r.inv_n, r.q.w * r.inv_n);
}

__global__ void __launch_bounds__(256) activations_bwd_kernel(int P, const float* __restrict__ scales, const float* __restrict__ opac,
                                                              const float4* __restrict__ rot, const float* __restrict__ filt,
                                                              const float* __restrict__ g_scales, const float* __restrict__ g_opac,
                                                              const float4* __restrict__ g_rot, float* __restrict__ d_scales,
                                                              float* __restrict__ d_opac, float4* __restrict__ d_rot) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const ActRow r = act_forward(scales, opac, rot, filt, i);
    const float f = filt[i], f2 = f * f;
    const float go = g_opac ? g_opac[i] : 0.f;
    // d s_k / d log-scale_k = raw^2 / s_k;   d coef / d log-scale_k = coef f^2 / (raw^2 + f^2)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float gs = g_scales ? g_scales[3 * (size_t)i + k] : 0.f;
        d_scales[3 * (size_t)i + k] = gs * r.raw2[k] / r.s[k] + go * r.sig * r.coef * f2 / r.a[k];
    }
    d_opac[i] = go * r.coef * r.sig * (1.0f - r.sig);
    float4 g = g_rot ? g_rot[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    if (r.q_clamped) {      // x / clamp_min(|x|, eps): below eps the clamp passes no gradient to the norm
        d_rot[i] = make_float4(g.x * r.inv_n, g.y * r.inv_n, g.z * r.inv_n, g.w * r.inv_n);
        return;
    }
    const float4 n = make_float4(r.q.x * r.inv_n, r.q.y * r.inv_n, r.q.z * r.inv_n, r.q.w * r.inv_n);
    const float d = g.x * n.x + g.y * n.y + g.z * n.z + g.w * n.w;
    d_rot[i] = make_float4((g.x - n.x * d) * r.inv_n, (g.y - n.y * d) * r.inv_n, (g.z - n.z * d) * r.inv_n, (g.w - n.w * d) * r.inv_n);
}

}  // namespace gsr

using namespace gsr;

extern "C" int gsr_gaussian_activations_forward(int P, const float* scales_raw, const float* opacities_raw, const float* rotations_raw,
                                                const float* filter_3D, float* scales, float* opacities, float* rotations, void* stream) {
    if (P < 0) { set_error("bad P"); return GSR_E_INVALID; }
    if (P == 0) return 0;
    if (!scales_raw || !opacities_raw || !rotations_raw || !filter_3D || !scales || !opacities || !rotations) {
        set_error("a required pointer is NULL");
        return GSR_E_INVALID;
    }
    activations_fwd_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(P, scales_raw, opacities_raw,
                                                                              reinterpret_cast<const float4*>(rotations_raw), filter_3D, scales,
                                                                              opacities, reinterpret_cast<float4*>(rotations));
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int gsr_gaussian_activations_backward(int P, const float* scales_raw, const float* opacities_raw, const float* rotations_raw,
                                                 const float* filter_3D, const float* dL_dscales, const float* dL_dopacities,
                                                 const float* dL_drotations, float* dL_dscales_raw, float* dL_dopacities_raw,
                                                 float* dL_drotations_raw, void* stream) {
    if (P < 0) { set_error("bad P"); return GSR_E_INVALID; }
    if (P == 0) return 0;
    if (!scales_raw || !opacities_raw || !rotations_raw || !filter_3D || !dL_dscales_raw || !dL_dopacities_raw || !dL_drotations_raw) {
        set_error("a required pointer is NULL");
        return GSR_E_INVALID;
    }
    activations_bwd_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
        P, scales_raw, opacities_raw, reinterpret_cast<const float4*>(rotations_raw), filter_3D, dL_dscales, dL_dopacities,
        reinterpret_cast<const float4*>(dL_drotations), dL_dscales_raw, dL_dopacities_raw, reinterpret_cast<float4*>(dL_drotations_raw));
    count_launches(1);
    GSR_CUDA(cudaGetLastError());
    return 0;
}
