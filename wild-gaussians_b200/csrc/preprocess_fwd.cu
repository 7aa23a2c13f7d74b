// preprocess_fwd.cu -- per-Gaussian forward stage: near cull, 3D->2D covariance projection
// with the Mip-Splatting low-pass + opacity compensation, conic, screen radius, tile
// rectangle, optional SH->RGB.  One thread per Gaussian; HBM-bound (about 44 B in, 56 B out
// per Gaussian on the colors_precomp path).
//
// Replaces preprocessCUDA<3> of the reference (forward.cu:166-268) together with
// computeColorFromSH (forward.cu:20-71), computeCov2D (:74-124), computeCov3D (:129-163),
// in_frustum / ndc2Pix / getRect (auxiliary.h:41-56,139-164).  Differences in data layout,
// not in arithmetic: the projected state is written as one 32-byte record per Gaussian
// ({x, y, hx, hy | conic.x, conic.y, conic.z, opacity*coef}; hx, hy = conservative half extents of
// the alpha >= 1/255 footprint) so the compositing kernels gather one aligned sector per instance; cov3D is not stored (the backward recomputes it);
// the tile rectangle is stored (8 B) so instance emission does not redo getRect; the depth
// sort key is emitted here.
#include "common.cuh"
#include "gaussian_math.cuh"

namespace gsr {

struct PreFwdParams {
    int P, D, M, W, H;
    int grid_x, grid_y;
    int ty0, ty1;                 // tile-row shard
    float focal_x, focal_y, tan_fovx, tan_fovy, kernel_size, scale_modifier;
    int prefiltered;
    int sh_vec;                   // SH rows are 16-byte aligned multiples of 16 bytes: 128-bit loads
    const float* means3D;
    const float* shs;
    const float* colors_precomp;
    const float* opacities;
    const float* scales;
    const float* rotations;
    const float* cov3D_precomp;
    const float* campos;
    const float* view;            // [16] device
    const float* proj;            // [16] device
    // outputs
    int* radii;
    float4* rec;
    float* rgb;
    uint8_t* clamped;
    float* depths;
    uint32_t* tiles_touched;
    uint32_t* cells_touched;
    TileRect* rect;
    uint32_t* sort_key;
    uint32_t* sort_val;
    int32_t* counters;
};

__device__ __forceinline__ float ndc_to_pix(float v, int S) {
    // evaluated in double like the reference (auxiliary.h:41-44)
    return ((v + 1.0) * S - 1.0) * 0.5;
}

// SH -> RGB (forward.cu:20-71).  The rounding sequence is part of the numerics contract (the clamp flags
// and the colours must have the reference's bits), so every product / sum is spelled out with
// non-contractable intrinsics in exactly the order nvcc emits for the reference (read off its SASS and
// pinned by tests/golden): each term is accumulated with one fma, res = fma(w_k, sh_k, res).
// The coefficients of one Gaussian are (max_deg+1)^2 * 3 contiguous floats.  Reading them with scalar loads
// makes every load instruction of a warp touch 32 different sectors (stride = one Gaussian); with 48 such loads the
// kernel is bound by L1 sector look-ups (measured 6x slower per Gaussian than the precomputed-colour path).  When a
// row is a whole number of 16-byte words and aligned, it is fetched with 128-bit loads instead (12 instead of 48).
__device__ __forceinline__ void load_sh_row(float (&dst)[48], const float* __restrict__ sh, int n_floats, bool vec) {
    if (vec) {
        const float4* p4 = reinterpret_cast<const float4*>(sh);
        const int n4 = (n_floats + 3) >> 2;
#pragma unroll
        for (int i = 0; i < 12; ++i) {
            if (i < n4) {
                const float4 v = __ldg(p4 + i);
                dst[4 * i + 0] = v.x; dst[4 * i + 1] = v.y; dst[4 * i + 2] = v.z; dst[4 * i + 3] = v.w;
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < 48; ++i)
            if (i < n_floats) dst[i] = sh[i];
    }
}

__device__ __forceinline__ V3 sh_to_rgb(int deg, const float* __restrict__ sh_row, bool vec, float3 p,
                                        const float* __restrict__ campos, unsigned* clamp_bits) {
    float sh[48];
    load_sh_row(sh, sh_row, 3 * (deg + 1) * (deg + 1), vec);
    const float dx = __fsub_rn(p.x, campos[0]), dy = __fsub_rn(p.y, campos[1]), dz = __fsub_rn(p.z, campos[2]);
    const float len = __fsqrt_rn(__fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy))));
    const float x = __fdiv_rn(dx, len), y = __fdiv_rn(dy, len), z = __fdiv_rn(dz, len);

    float res[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) res[c] = __fmul_rn(GSR_SH_C0, sh[c]);
    auto acc = [&](float w, int k) {
#pragma unroll
        for (int c = 0; c < 3; ++c) res[c] = __fmaf_rn(w, sh[3 * k + c], res[c]);
    };
    if (deg > 0) {
        acc(-__fmul_rn(GSR_SH_C1, y), 1);
        acc(__fmul_rn(GSR_SH_C1, z), 2);
        acc(-__fmul_rn(GSR_SH_C1, x), 3);
        if (deg > 1) {
            const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
            const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
            acc(__fmul_rn(GSR_SH_C2_0, xy), 4);
            acc(__fmul_rn(GSR_SH_C2_1, yz), 5);
            acc(__fmul_rn(GSR_SH_C2_2, __fsub_rn(__fmaf_rn(2.0f, zz, -xx), yy)), 6);
            acc(__fmul_rn(GSR_SH_C2_3, xz), 7);
            acc(__fmul_rn(GSR_SH_C2_4, __fsub_rn(xx, yy)), 8);
            if (deg > 2) {
                acc(__fmul_rn(__fmul_rn(GSR_SH_C3_0, y), __fmaf_rn(3.0f, xx, -yy)), 9);
                acc(__fmul_rn(__fmul_rn(GSR_SH_C3_1, xy), z), 10);
                acc(__fmul_rn(__fmul_rn(GSR_SH_C3_2, y), __fsub_rn(__fmaf_rn(4.0f, zz, -xx), yy)), 11);
                acc(__fmul_rn(__fmul_rn(GSR_SH_C3_3, z), __fmaf_rn(-3.0f, yy, __fmaf_rn(-3.0f, xx, __fmul_rn(2.0f, zz)))), 12);
                acc(__fmul_rn(__fmul_rn(GSR_SH_C3_4, x), __fsub_rn(__fmaf_rn(4.0f, zz, -xx), yy)), 13);
                acc(__fmul_rn(__fmul_rn(GSR_SH_C3_5, z), __fsub_rn(xx, yy)), 14);
                acc(__fmul_rn(__fmul_rn(GSR_SH_C3_6, x), __fmaf_rn(-3.0f, yy, xx)), 15);
            }
        }
    }
    unsigned bits = 0;
    V3 out;
    float* o = &out.x;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float r = __fadd_rn(res[c], 0.5f);
        if (r < 0) bits |= 1u << c;
        o[c] = fmaxf(r, 0.0f);
    }
    *clamp_bits = bits;
    return out;
}

template <bool HAS_SH>
__global__ void __launch_bounds__(256) preprocess_fwd_kernel(const __grid_constant__ PreFwdParams p) {
    // camera matrices: one coalesced read per block into shared memory
    __shared__ float s_view[16];
    __shared__ float s_proj[16];
    if (threadIdx.x < 16) s_view[threadIdx.x] = p.view[threadIdx.x];
    else if (threadIdx.x < 32) s_proj[threadIdx.x - 16] = p.proj[threadIdx.x - 16];
    __syncthreads();

    __shared__ unsigned s_block_tiles, s_block_visible;
    if (threadIdx.x == 0) { s_block_tiles = 0; s_block_visible = 0; }
    __syncthreads();

    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in_range = idx < p.P;

    // defaults for Gaussians that are not rendered
    int out_radius = 0;
    uint32_t out_tiles = 0, out_cells = 0;
    uint32_t out_key = RADIX_DROP_KEY;   // culled Gaussians (and those outside the tile-row band) are dropped by the depth sort
    TileRect out_rect = {0, 0, 0, 0};
    bool visible = false;

    float3 p_orig = {0.f, 0.f, 0.f};
    if (in_range) p_orig = float3{p.means3D[3 * idx], p.means3D[3 * idx + 1], p.means3D[3 * idx + 2]};
    const float4 p_hom = xform_point_4x4(p_orig, s_proj);
    const float p_w = 1.0f / (p_hom.w + 0.0000001f);
    const float3 p_proj = {p_hom.x * p_w, p_hom.y * p_w, p_hom.z * p_w};
    const float3 p_view = xform_point_4x3(p_orig, s_view);

    do {
        if (!in_range) break;
        if (p_view.z <= NEAR_Z) {
            if (p.prefiltered) atomicExch(&p.counters[0], 1);
            break;
        }

        float cov3D_local[6];
        const float* cov3D;
        if (p.cov3D_precomp != nullptr) {
            cov3D = p.cov3D_precomp + 6 * (size_t)idx;
        } else {
            const float3 sc = {p.scales[3 * idx], p.scales[3 * idx + 1], p.scales[3 * idx + 2]};
            const float4 rot = reinterpret_cast<const float4*>(p.rotations)[idx];
            cov3d_from_scale_rot(sc, p.scale_modifier, rot, cov3D_local);
            cov3D = cov3D_local;
        }

        const Ewa e = ewa_project(p_orig, p.focal_x, p.focal_y, p.tan_fovx, p.tan_fovy, cov3D, s_view);
        float c00 = e.cov.m[0][0], c01 = e.cov.m[0][1], c11 = e.cov.m[1][1];

        // opacity compensation of the low-pass filter; mixed precision as in forward.cu:112-118
        const float det_0 = max(1e-6, (double)(c00 * c11 - c01 * c01));
        const float det_1 = max(1e-6, (double)((c00 + p.kernel_size) * (c11 + p.kernel_size) - c01 * c01));
        float coef = sqrt(det_0 / (det_1 + 1e-6) + 1e-6);
        if (det_0 <= 1e-6 || det_1 <= 1e-6) coef = 0.0f;
        c00 += p.kernel_size;
        c11 += p.kernel_size;
        const float4 cov = {float(c00), float(c01), float(c11), float(coef)};

        const float det = (cov.x * cov.z - cov.y * cov.y);
        if (det == 0.0f) break;
        const float det_inv = 1.f / det;
        const float3 conic = {cov.z * det_inv, -cov.y * det_inv, cov.x * det_inv};

        const float mid = 0.5f * (cov.x + cov.z);
        const float lambda1 = mid + sqrtf(max(0.1f, mid * mid - det));
        const float lambda2 = mid - sqrtf(max(0.1f, mid * mid - det));
        const float my_radius = ceilf(3.f * sqrtf(max(lambda1, lambda2)));
        const float2 point_image = {ndc_to_pix(p_proj.x, p.W), ndc_to_pix(p_proj.y, p.H)};

        // tile rectangle (auxiliary.h:46-56); max_radius is the radius converted to int
        const int max_radius = (int)my_radius;
        const unsigned gx = (unsigned)p.grid_x, gy = (unsigned)p.grid_y;
        unsigned rx0 = min(gx, (unsigned)max((int)0, (int)((point_image.x - max_radius) / TILE)));
        unsigned ry0 = min(gy, (unsigned)max((int)0, (int)((point_image.y - max_radius) / TILE)));
        unsigned rx1 = min(gx, (unsigned)max((int)0, (int)((point_image.x + max_radius + TILE - 1) / TILE)));
        unsigned ry1 = min(gy, (unsigned)max((int)0, (int)((point_image.y + max_radius + TILE - 1) / TILE)));
        if ((rx1 - rx0) * (ry1 - ry0) == 0) break;

        // colour from SH (the colors_precomp path reads colours only while compositing)
        if (HAS_SH) {
            unsigned bits;
            const V3 c = sh_to_rgb(p.D, p.shs + (size_t)idx * p.M * 3, p.sh_vec != 0, p_orig, p.campos, &bits);
            p.rgb[3 * idx + 0] = c.x;
            p.rgb[3 * idx + 1] = c.y;
            p.rgb[3 * idx + 2] = c.z;
            p.clamped[idx] = (uint8_t)bits;
        }

        visible = true;
        out_radius = (int)my_radius;
        // shard clip: radii stay those of the full image, only the binned rows shrink
        const unsigned cy0 = max(ry0, (unsigned)p.ty0), cy1 = min(ry1, (unsigned)p.ty1);
        const unsigned rows = cy1 > cy0 ? cy1 - cy0 : 0u;
        out_tiles = rows * (rx1 - rx0);
        out_rect = {(uint16_t)rx0, (uint16_t)(rows ? cy0 : 0u), (uint16_t)rx1, (uint16_t)(rows ? cy1 : 0u)};
        if (rows) out_cells = ((rx1 - 1) / CELL - rx0 / CELL + 1) * ((cy1 - 1) / CELL - cy0 / CELL + 1);
        if (rows) out_key = __float_as_uint(p_view.z);    // view-space z > 0.2: never equals the drop key

        // Screen-space half extents of the region where this Gaussian can reach alpha >= 1/255
        // (axis-aligned box of the ellipse d^T Sigma^-1 d <= 2 ln(255 o)), inflated by a safety margin
        // far above fp32 rounding.  The compositing kernels use it to skip, per warp, Gaussians that
        // cannot touch any of the warp's pixels; the skipped pairs are exactly pairs the reference
        // rejects with its alpha < 1/255 test (forward.cu:365), so results are unchanged.
        // Negative extents: opacity too low to ever pass the test.  NaNs fall through as "keep".
        const float op = p.opacities[idx] * cov.w;
        float hx = -1.f, hy = -1.f;
        if (!(op < (1.0f / 255.0f) * 0.9999f)) {
            const float tau = logf(255.0f * op) * 1.0001f + 1e-4f;
            hx = sqrtf(2.f * tau * cov.x) * 1.0001f + 0.05f;
            hy = sqrtf(2.f * tau * cov.z) * 1.0001f + 0.05f;
            // The composite evaluates the fp32 conic, not Sigma^-1.  For a nearly singular 2D covariance (a needle
            // without a low-pass filter) the conic's small eigenvalue carries no correct digits and its alpha >= 1/255
            // region reaches far beyond Sigma's box: no box then (the ellipse test on the conic still applies).
            const double cdet = (double)conic.x * conic.z - (double)conic.y * conic.y;
            if (!(cdet > 1e-3 * ((double)conic.x * conic.z))) { hx = 1e30f; hy = 1e30f; }
        }
        p.rec[2 * (size_t)idx + 0] = make_float4(point_image.x, point_image.y, hx, hy);
        p.rec[2 * (size_t)idx + 1] = make_float4(conic.x, conic.y, conic.z, op);
        p.depths[idx] = p_view.z;
    } while (false);

    if (in_range) {
        p.radii[idx] = out_radius;
        p.tiles_touched[idx] = out_tiles;
        p.cells_touched[idx] = out_cells;
        p.rect[idx] = out_rect;
        p.sort_key[idx] = out_key;
        p.sort_val[idx] = (uint32_t)idx;
    }

    // visible count and total instance count R: warp reduce -> shared -> one global atomic per CTA
    const unsigned ballot = __ballot_sync(0xFFFFFFFFu, visible);
    const unsigned warp_tiles = __reduce_add_sync(0xFFFFFFFFu, out_tiles);
    if ((threadIdx.x & 31) == 0 && ballot != 0) {
        atomicAdd(&s_block_visible, (unsigned)__popc(ballot));
        atomicAdd(&s_block_tiles, warp_tiles);
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_block_visible != 0) {
        atomicAdd(&p.counters[1], (int)s_block_visible);
        atomicAdd(reinterpret_cast<unsigned long long*>(&p.counters[2]), (unsigned long long)s_block_tiles);
    }
}

int launch_preprocess_fwd(const GsrForwardArgs& a, const GeomState& g, int ty0, int ty1, cudaStream_t s) {
    PreFwdParams p;
    p.P = a.P; p.D = a.D; p.M = a.M; p.W = a.W; p.H = a.H;
    p.grid_x = tiles_x(a.W); p.grid_y = tiles_y(a.H);
    p.ty0 = ty0; p.ty1 = ty1;
    p.focal_y = a.H / (2.0f * a.tan_fovy);
    p.focal_x = a.W / (2.0f * a.tan_fovx);
    p.tan_fovx = a.tan_fovx; p.tan_fovy = a.tan_fovy;
    p.kernel_size = a.kernel_size; p.scale_modifier = a.scale_modifier;
    p.prefiltered = a.prefiltered;
    p.sh_vec = a.shs != nullptr && (a.M * 3) % 4 == 0 && (reinterpret_cast<uintptr_t>(a.shs) & 15u) == 0;
    p.means3D = a.means3D; p.shs = a.shs; p.colors_precomp = a.colors_precomp;
    p.opacities = a.opacities; p.scales = a.scales; p.rotations = a.rotations;
    p.cov3D_precomp = a.cov3D_precomp; p.campos = a.campos;
    p.view = a.viewmatrix; p.proj = a.projmatrix;
    p.radii = a.radii; p.rec = g.rec; p.rgb = g.rgb; p.clamped = g.clamped; p.depths = g.depths;
    p.tiles_touched = g.tiles_touched; p.cells_touched = g.cells_touched; p.rect = g.rect;
    p.sort_key = g.key_a; p.sort_val = g.val_a; p.counters = g.counters;
    const int blocks = (a.P + 255) / 256;
    if (a.colors_precomp == nullptr) preprocess_fwd_kernel<true><<<blocks, 256, 0, s>>>(p);
    else preprocess_fwd_kernel<false><<<blocks, 256, 0, s>>>(p);
    count_launches(1);
    return 0;
}

}  // namespace gsr
