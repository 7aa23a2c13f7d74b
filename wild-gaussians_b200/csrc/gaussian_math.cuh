// gaussian_math.cuh -- per-Gaussian projection math shared by the forward and backward
// per-Gaussian kernels.
//
// Numerics contract (SURVEY.md section 8a, notes N1/N2/N5): tile and sort indices must be
// bit-identical to the reference, so every expression below keeps the reference's
// evaluation order (GLM column-major 3x3 products evaluated as a0*b0 + a1*b1 + a2*b2,
// forward.cu:74-163, auxiliary.h:41-97) and the same mixed fp32/fp64 steps.  The file is
// compiled with nvcc's default -fmad=true like the reference, so the fused-multiply-add
// contraction of identical expression trees is identical.  Do not "simplify" products
// with literal zeros or re-associate sums here.
#pragma once
#include <cuda_runtime.h>

namespace gsr {

// 3x3 matrix, column-major: m[c][r] is column c, row r.
struct Mat3 {
    float m[3][3];
};

__device__ __forceinline__ Mat3 mat3_cols(float c00, float c01, float c02,
                                          float c10, float c11, float c12,
                                          float c20, float c21, float c22) {
    Mat3 r;
    r.m[0][0] = c00; r.m[0][1] = c01; r.m[0][2] = c02;
    r.m[1][0] = c10; r.m[1][1] = c11; r.m[1][2] = c12;
    r.m[2][0] = c20; r.m[2][1] = c21; r.m[2][2] = c22;
    return r;
}

// a * b with each element accumulated left to right over k = 0,1,2.
__device__ __forceinline__ Mat3 mat3_mul(const Mat3& a, const Mat3& b) {
    Mat3 r;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int row = 0; row < 3; ++row) {
            r.m[c][row] = a.m[0][row] * b.m[c][0] + a.m[1][row] * b.m[c][1] + a.m[2][row] * b.m[c][2];
        }
    }
    return r;
}

__device__ __forceinline__ Mat3 mat3_transpose(const Mat3& a) {
    Mat3 r;
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int row = 0; row < 3; ++row) r.m[c][row] = a.m[row][c];
    return r;
}

// row-vector convention: matrix[12..14] is the translation (auxiliary.h:58-77)
__device__ __forceinline__ float3 xform_point_4x3(const float3& p, const float* __restrict__ mat) {
    float3 t = {
        mat[0] * p.x + mat[4] * p.y + mat[8] * p.z + mat[12],
        mat[1] * p.x + mat[5] * p.y + mat[9] * p.z + mat[13],
        mat[2] * p.x + mat[6] * p.y + mat[10] * p.z + mat[14],
    };
    return t;
}

__device__ __forceinline__ float4 xform_point_4x4(const float3& p, const float* __restrict__ mat) {
    float4 t = {
        mat[0] * p.x + mat[4] * p.y + mat[8] * p.z + mat[12],
        mat[1] * p.x + mat[5] * p.y + mat[9] * p.z + mat[13],
        mat[2] * p.x + mat[6] * p.y + mat[10] * p.z + mat[14],
        mat[3] * p.x + mat[7] * p.y + mat[11] * p.z + mat[15]
    };
    return t;
}

// rotation (raw quaternion r,x,y,z -- NOT normalised, note N5) as column-major matrix.
// The reference's contraction is written out (oracle/oracle.c quat_to_R): xz, rx, rz, yy, zz are rounded products,
// r*y, y*z, x*y, x*x are fused into the add / sub.  Which products ptxas fuses here depends on the target
// architecture, so the pattern is not left to the compiler.
__device__ __forceinline__ Mat3 quat_to_mat(const float4 q) {
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    const float xz = __fmul_rn(x, z), rx = __fmul_rn(r, x), rz = __fmul_rn(r, z), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
    return mat3_cols(
        1.f - 2.f * __fadd_rn(yy, zz), 2.f * __fmaf_rn(x, y, -rz), 2.f * __fmaf_rn(r, y, xz),
        2.f * __fmaf_rn(x, y, rz), 1.f - 2.f * __fmaf_rn(x, x, zz), 2.f * __fmaf_rn(y, z, -rx),
        2.f * __fmaf_rn(-r, y, xz), 2.f * __fmaf_rn(y, z, rx), 1.f - 2.f * __fmaf_rn(x, x, yy));
}

// world-space covariance from scale and rotation; upper triangle in cov[6]
// (forward.cu:129-163): Sigma = (S R)^T (S R), S = diag(mod * scale).
__device__ __forceinline__ void cov3d_from_scale_rot(const float3 scale, float mod, const float4 rot, float* cov) {
    Mat3 S = mat3_cols(1.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f);
    S.m[0][0] = mod * scale.x;
    S.m[1][1] = mod * scale.y;
    S.m[2][2] = mod * scale.z;
    const Mat3 R = quat_to_mat(rot);
    const Mat3 M = mat3_mul(S, R);
    const Mat3 Sigma = mat3_mul(mat3_transpose(M), M);
    cov[0] = Sigma.m[0][0];
    cov[1] = Sigma.m[0][1];
    cov[2] = Sigma.m[0][2];
    cov[3] = Sigma.m[1][1];
    cov[4] = Sigma.m[1][2];
    cov[5] = Sigma.m[2][2];
}

// EWA projection pieces shared by forward and backward (forward.cu:74-106, backward.cu:165-197)
struct Ewa {
    float3 t;        // view-space mean with x,y clamped to +-1.3 tanfov * z
    float txtz, tytz;
    float limx, limy;
    Mat3 T;          // W * J
    Mat3 Vrk;        // symmetric 3D covariance
    Mat3 cov;        // T^T Vrk^T T  (only [0][0], [0][1], [1][1] are meaningful)
};

__device__ __forceinline__ Ewa ewa_project(const float3& mean, float focal_x, float focal_y,
                                           float tan_fovx, float tan_fovy,
                                           const float* cov3D, const float* __restrict__ view) {
    Ewa e;
    float3 t = xform_point_4x3(mean, view);
    e.limx = 1.3f * tan_fovx;
    e.limy = 1.3f * tan_fovy;
    e.txtz = t.x / t.z;
    e.tytz = t.y / t.z;
    t.x = min(e.limx, max(-e.limx, e.txtz)) * t.z;
    t.y = min(e.limy, max(-e.limy, e.tytz)) * t.z;
    e.t = t;

    const Mat3 J = mat3_cols(
        focal_x / t.z, 0.0f, -(focal_x * t.x) / (t.z * t.z),
        0.0f, focal_y / t.z, -(focal_y * t.y) / (t.z * t.z),
        0, 0, 0);
    const Mat3 Wm = mat3_cols(
        view[0], view[4], view[8],
        view[1], view[5], view[9],
        view[2], view[6], view[10]);
    e.T = mat3_mul(Wm, J);
    e.Vrk = mat3_cols(
        cov3D[0], cov3D[1], cov3D[2],
        cov3D[1], cov3D[3], cov3D[4],
        cov3D[2], cov3D[4], cov3D[5]);
    e.cov = mat3_mul(mat3_mul(mat3_transpose(e.T), mat3_transpose(e.Vrk)), e.T);
    return e;
}

// SH basis constants (auxiliary.h:22-39)
#define GSR_SH_C0 0.28209479177387814f
#define GSR_SH_C1 0.4886025119029199f
#define GSR_SH_C2_0 1.0925484305920792f
#define GSR_SH_C2_1 (-1.0925484305920792f)
#define GSR_SH_C2_2 0.31539156525252005f
#define GSR_SH_C2_3 (-1.0925484305920792f)
#define GSR_SH_C2_4 0.5462742152960396f
#define GSR_SH_C3_0 (-0.5900435899266435f)
#define GSR_SH_C3_1 2.890611442640554f
#define GSR_SH_C3_2 (-0.4570457994644658f)
#define GSR_SH_C3_3 0.3731763325901154f
#define GSR_SH_C3_4 (-0.4570457994644658f)
#define GSR_SH_C3_5 1.445305721320277f
#define GSR_SH_C3_6 (-0.5900435899266435f)

struct V3 {
    float x, y, z;
};
__device__ __forceinline__ V3 operator*(float s, const V3& v) { return {s * v.x, s * v.y, s * v.z}; }
__device__ __forceinline__ V3 operator*(const V3& v, float s) { return {v.x * s, v.y * s, v.z * s}; }
__device__ __forceinline__ V3 operator+(const V3& a, const V3& b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ V3 operator-(const V3& a, const V3& b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ V3& operator+=(V3& a, const V3& b) { a.x += b.x; a.y += b.y; a.z += b.z; return a; }
__device__ __forceinline__ float dot3(const V3& a, const V3& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 ldv3(const float* p) { return {p[0], p[1], p[2]}; }

}  // namespace gsr
