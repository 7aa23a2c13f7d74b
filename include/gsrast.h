/*
 * gsrast.h -- C ABI of libgsrast.so, the sm_90a Gaussian-splat rasterizer.
 *
 * This header is the drop-in boundary for the hot path of jkulhanek/wild-gaussians:
 * it replaces the C++ entry points the reference's pybind11 module binds
 *   CudaRasterizer::Rasterizer::forward      (DGR/cuda_rasterizer/rasterizer.h:31-57,  rasterizer_impl.cu:198-340)
 *   CudaRasterizer::Rasterizer::backward     (DGR/cuda_rasterizer/rasterizer.h:59-88,  rasterizer_impl.cu:344-444)
 *   CudaRasterizer::Rasterizer::markVisible  (DGR/cuda_rasterizer/rasterizer.h:24-29,  rasterizer_impl.cu:141-153)
 * (DGR = submodules/diff-gaussian-rasterization) and is what
 *   RasterizeGaussiansCUDA / RasterizeGaussiansBackwardCUDA / markVisible  (DGR/rasterize_points.cu:35-225)
 * would call instead.  Plain C: raw device pointers, ints and floats, an opaque stream
 * handle (a cudaStream_t passed as void*), no torch types, no exceptions, no allocation
 * inside the library.  Every function returns 0 on success, a positive cudaError_t or a
 * negative GSR_E_* code on failure; gsr_last_error() then holds a thread-local message.
 *
 * All tensors are contiguous fp32 (ints where stated) on the current CUDA device.
 * "absent" optional inputs are NULL (the reference's zero-element tensors,
 * DGR/diff_gaussian_rasterization/__init__.py:218-228).
 *
 * Buffer protocol (replaces the reference's three std::function<char*(size_t)> resize
 * callbacks, rasterize_points.cu:27-33,78-80):
 *   1. gsr_forward_sizes()     -> bytes for geom_buffer and img_buffer      (caller allocates)
 *   2. gsr_forward_geometry()  -> per-Gaussian projection, depth ordering, instance counts
 *                                  (one stream sync, like rasterizer_impl.cu:283-284)
 *   3. gsr_binning_sizes()     -> bytes for binning_buffer and the transient scratch
 *   4. gsr_forward_render()    -> tile binning + per-tile front-to-back composite
 * gsr_forward() does 1-4 in one call through a C allocation callback.
 * geom/binning/img buffers must be kept (unmodified) for gsr_backward(); scratch may be
 * released as soon as gsr_forward_render() has been enqueued (stream-ordered allocators) or
 * completed.
 */
#ifndef GSRAST_H_INCLUDED
#define GSRAST_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSR_ABI_VERSION 2

/* negative status codes (positive values are cudaError_t) */
#define GSR_E_INVALID      (-1)  /* bad argument (NULL where required, P<0, ...)            */
#define GSR_E_PREFILTERED  (-2)  /* a Gaussian was culled although prefiltered=1
                                    (reference: printf + __trap, auxiliary.h:156-160)        */
#define GSR_E_CHANNELS     (-3)  /* reserved: non-RGB without colors_precomp
                                    (rasterizer_impl.cu:244-247); this build is RGB only     */
#define GSR_E_OVERFLOW     (-4)  /* instance count does not fit the supplied buffers         */

/* which buffer an allocation callback is asked for */
#define GSR_BUF_GEOM     0
#define GSR_BUF_BINNING  1
#define GSR_BUF_IMG      2
#define GSR_BUF_SCRATCH  3

/* Allocation callback for gsr_forward(): must return a device pointer to at least `bytes`
 * bytes, 256-byte aligned, valid at least until gsr_backward() for GEOM/BINNING/IMG.     */
typedef void* (*gsr_alloc_fn)(void* ctx, int which, size_t bytes);

/* Inputs of one forward rasterization.  Field meaning follows
 * CudaRasterizer::Rasterizer::forward (rasterizer_impl.cu:198-225).                        */
typedef struct GsrForwardArgs {
    int P;                        /* number of Gaussians                                    */
    int D;                        /* active SH degree (0..3); ignored with colors_precomp   */
    int M;                        /* SH coefficients per Gaussian, (deg_max+1)^2; 0 if none */
    int W, H;                     /* image size in pixels                                   */
    const float* background;      /* [3]                                                    */
    const float* means3D;         /* [P,3]                                                  */
    const float* shs;             /* [P,M,3] or NULL                                        */
    const float* colors_precomp;  /* [P,3]   or NULL (exactly one of shs/colors_precomp)    */
    const float* opacities;       /* [P] (or [P,1])                                         */
    const float* scales;          /* [P,3]   or NULL                                        */
    float        scale_modifier;
    const float* rotations;       /* [P,4] (r,x,y,z), used un-normalised; or NULL           */
    const float* cov3D_precomp;   /* [P,6]   or NULL (exactly one of scales+rot / cov3D)    */
    const float* viewmatrix;      /* [16] row-vector convention (translation at 12..14)     */
    const float* projmatrix;      /* [16] view*proj, same convention                        */
    const float* campos;          /* [3]                                                    */
    float tan_fovx, tan_fovy;
    float kernel_size;            /* Mip-Splatting 2D low-pass (forward.cu:108-121)         */
    const float* subpixel_offset; /* [H,W,2]                                                */
    int prefiltered;
    int debug;                    /* !=0: synchronise + check after every stage             */
    /* Screen-space shard (multi-GPU tile-row partition): only tile rows
     * [tile_y0, tile_y1) are binned and composited; pixels of other rows are not written.
     * tile_y0 = tile_y1 = 0 means the whole image.                                         */
    int tile_y0, tile_y1;
    /* outputs */
    float* out_color;             /* [3,H,W]  (rows of the shard are written)               */
    int*   radii;                 /* [P]      screen radius in px, 0 = not rendered         */
    /* Multi-GPU image all-gather fused into the composite (optional): `peer_images` is a DEVICE array of
     * `n_peer_images` pointers, one per rank (this rank included), each to a [4,H,W] fp32 image (colour planes +
     * final transmittance) in peer-mapped memory (NVLink / NVSwitch symmetric memory).  The composite then stores
     * every pixel of its band into ALL of them instead of out_color (which may be NULL); after a barrier across the
     * ranks every rank holds the full image.  NULL / 0: single-GPU behaviour.                                   */
    const void* const* peer_images;
    int    n_peer_images;
} GsrForwardArgs;

/* Inputs/outputs of the backward pass.  Field meaning follows
 * CudaRasterizer::Rasterizer::backward (rasterizer_impl.cu:344-377).
 * Every output array is written completely by the call (zeros for Gaussians that were not
 * rendered): no pre-zeroing is required, unlike rasterize_points.cu:157-165.               */
typedef struct GsrBackwardArgs {
    int P, D, M;
    int R;                        /* num_rendered returned by the forward                   */
    int W, H;
    const float* background;
    const float* means3D;
    const float* shs;
    const float* colors_precomp;
    const float* scales;
    float        scale_modifier;
    const float* rotations;
    const float* cov3D_precomp;
    const float* viewmatrix;
    const float* projmatrix;
    const float* campos;
    float tan_fovx, tan_fovy;
    float kernel_size;
    const float* subpixel_offset;
    const int*   radii;           /* [P] from the forward                                   */
    const void*  geom_buffer;
    const void*  binning_buffer;
    const void*  img_buffer;
    const float* dL_dpix;         /* [3,H,W] upstream gradient of out_color                 */
    int debug;
    int tile_y0, tile_y1;         /* same shard as the forward                              */
    void*  accum_scratch;         /* gsr_backward_scratch_bytes(P) bytes.  gsr_backward / _partials zero it first unless
                                     accum_is_zero != 0; gsr_backward_finalize leaves it ZEROED again (a stream-
                                     ordered fill after its kernel), so a caller that keeps the buffer skips the fill. */
    int    accum_is_zero;
    /* outputs */
    float* dL_dmean2D;            /* [P,3]  x,y: NDC-scaled screen grad; z: sum |gx|+|gy|
                                     (backward.cu:590-595)                                  */
    float* dL_dconic;             /* [P,4]  (x,y,-,w) as backward.cu:598-600; may be NULL   */
    float* dL_dopacity;           /* [P]                                                    */
    float* dL_dcolor;             /* [P,3]                                                  */
    float* dL_dmean3D;            /* [P,3]                                                  */
    float* dL_dcov3D;             /* [P,6]; may be NULL when cov3D_precomp is NULL          */
    float* dL_dsh;                /* [P,M,3]; required iff shs != NULL                      */
    float* dL_dscale;             /* [P,3];  required iff scales != NULL                    */
    float* dL_drot;               /* [P,4];  required iff rotations != NULL                 */
    /* Fixed-order reductions: with deterministic != 0, gsr_backward / _partials and gsr_backward_colors give bitwise
     * identical results from run to run on the same device model.  Each (tile, Gaussian) pair's sums are stored to a slot
     * of its own, and each Gaussian adds its slots in the order of its tiles, instead of adding into the accumulator in
     * arrival order.  Needs det_scratch (contents arbitrary) and det_marks (ALL-ZERO on entry, left all-zero), sized by
     * gsr_backward_deterministic_sizes for this R.  The multi-GPU entry points (_peers, _marked) reject it.           */
    int    deterministic;
    void*  det_scratch;
    void*  det_marks;
} GsrBackwardArgs;

/* Counters of the last forward on this geom buffer (device->host copied on request).     */
typedef struct GsrStats {
    int      num_rendered;        /* R: (Gaussian, tile) instances                          */
    int      num_visible;         /* V: Gaussians with radii > 0                            */
    int      num_tiles;           /* tiles in the shard                                     */
    int      num_coarse;          /* N1: (Gaussian, 8x8-tile cell) items of the two-level binning */
} GsrStats;

int         gsr_abi_version(void);
const char* gsr_last_error(void);

/* -- forward ----------------------------------------------------------------------------- */
int gsr_forward_sizes(int P, int M, int W, int H, size_t* geom_bytes, size_t* img_bytes);
/* num_rendered = R, the number of (Gaussian, tile) instances (what the reference returns);
 * num_coarse   = number of (Gaussian, 8x8-tile cell) items of the two-level binning: it sizes the
 *                transient scratch and must be passed back to gsr_binning_sizes / gsr_forward_render. */
int gsr_forward_geometry(const GsrForwardArgs* args, void* geom_buffer, void* img_buffer,
                         void* stream, int* num_rendered, int* num_coarse);
int gsr_binning_sizes(int P, int W, int H, int num_rendered, int num_coarse,
                      size_t* binning_bytes, size_t* scratch_bytes);
int gsr_forward_render(const GsrForwardArgs* args, void* geom_buffer, void* img_buffer,
                       void* binning_buffer, void* scratch, int num_rendered, int num_coarse,
                       void* stream);
int gsr_forward(const GsrForwardArgs* args, gsr_alloc_fn alloc, void* alloc_ctx,
                void* stream, int* num_rendered);

/* Re-composite with different per-Gaussian colours on the SAME geometry/binning state
 * (wild-gaussians renders raw + appearance-toned colours per step, method.py:1573-1611).
 * Writes out_color (and final_T / n_contrib into img_buffer2, sized like img_buffer).     */
int gsr_forward_recolor(const GsrForwardArgs* args, const void* geom_buffer,
                        const void* binning_buffer, const void* img_buffer,
                        void* img_buffer2, void* stream);

/* Display composite of an inference render (WildGaussians.render): after gsr_forward_geometry, tile binning and one
 * composite over the whole image that walks the tile lists with the training composite's arithmetic (the colour sums and
 * T are its bits) but keeps no backward state (no final_T, n_contrib or blend masks in img_buffer; only the tile ranges)
 * and writes, instead of args->out_color (which is ignored and may be NULL):
 *   out_color [H,W,3]  clamp(C + T bg, 0, 1), then NaN -> 0 (the reference's clamp + nan_to_num_, permuted to HWC)
 *   out_accum [H,W]    1 - T
 *   out_depth [H,W]    with depth != 0: D + T bg[0], D composited from one value per Gaussian by the colours' recurrence
 *                      fma(T, alpha d, D).  The values are depth_values [P] when given, otherwise the camera distance
 *                      |means3D - campos| (in the reference's norm's operation order), computed into depth_scratch [P]
 *                      first.
 * Takes the arguments of gsr_forward_render otherwise.  A tile-row shard or peer images are rejected (GSR_E_INVALID).
 * P = 0 writes nothing.                                                                                                */
typedef struct GsrDisplayArgs {
    float* out_color;
    float* out_accum;
    int    depth;
    float* out_depth;
    const float* depth_values;
    float* depth_scratch;
} GsrDisplayArgs;
int gsr_forward_display(const GsrForwardArgs* args, const GsrDisplayArgs* display, void* geom_buffer, void* img_buffer,
                        void* binning_buffer, void* scratch, int num_rendered, int num_coarse, void* stream);

/* -- backward ---------------------------------------------------------------------------- */
size_t gsr_backward_scratch_bytes(int P);
/* scratch_bytes: 48 B per instance + 4 B per Gaussian + scan temporaries; mark_bytes: 4 bits per instance.          */
int    gsr_backward_deterministic_sizes(int P, int R, size_t* scratch_bytes, size_t* mark_bytes);
int    gsr_backward(const GsrBackwardArgs* args, void* stream);
/* The two halves of gsr_backward(), for the tile-row sharded (multi-GPU) path where the
 * per-Gaussian partial sums of all shards are added (NCCL all-reduce over accum_scratch, a dense
 * [P][12] fp32 array starting at the first 256-byte aligned address) between them:
 *   partials: zero accum_scratch, run the per-tile backward composite of this shard into it
 *             (needs dL_dpix, img/binning buffers; writes no output tensor)
 *   finalize: per-Gaussian chain rule from accum_scratch to every output tensor                     */
int    gsr_backward_partials(const GsrBackwardArgs* args, void* stream);
int    gsr_backward_finalize(const GsrBackwardArgs* args, void* stream);
/* Reduction-fused variant of gsr_backward_partials for ranks that share a symmetric accumulator (one [P][12] fp32
 * array per rank, each mapped into every process; NVLink/NVSwitch peer memory): the per-tile backward composite adds
 * its sums directly into the accumulators of ALL ranks -- through `multicast_accum` (NVSwitch multicast address: one
 * multimem.red per 16 bytes, the switch updates every replica) when it is non-NULL, else through the `n_peers` device
 * pointers stored in the DEVICE array `peer_accum_dev`.  The arrays must have been zeroed on every rank (and a
 * barrier passed) before any rank calls this; after a second barrier every rank holds the complete sums and calls
 * gsr_backward_finalize with accum_scratch = its own array.  Replaces partials + all-reduce.                       */
int    gsr_backward_partials_peers(const GsrBackwardArgs* args, const void* const* peer_accum_dev, int n_peers,
                                   void* multicast_accum, void* stream);

/* "Pull" form of the multi-GPU reduction (GSR_PEER_REDUCE=3): no remote atomics at all.  gsr_backward_partials_marked adds
 * this rank's band into ITS OWN accumulator (args->accum_scratch) and sets touched[i] = 1 for every Gaussian i it added to
 * (one byte per Gaussian, all-zero on entry).  After a barrier, gsr_backward_finalize_pull forms each Gaussian's complete
 * sums as own row + the rows the other ranks marked, read through their peer-mapped accumulators in rank order 0..n-1
 * (the same order on every rank: the resulting gradients are bit-identical across ranks), and runs the chain rule.
 * peer_accums / peer_touched: HOST arrays of n_peers (<= GSR_MAX_PULL_PEERS) device pointers -- the ranks' buffers as mapped
 * into this process (entry `self` = this rank's own buffers).
 * The buffers of THIS pass must stay untouched until every rank has finished reading them, i.e. until the barrier of the
 * next pass: keep two sets and pass the previous pass's set as clear_accum / clear_touched (may be NULL) -- its marked
 * rows and marks are zeroed by this call.                                                                             */
int    gsr_backward_partials_marked(const GsrBackwardArgs* args, unsigned char* touched, void* stream);
#define GSR_MAX_PULL_PEERS 8
int    gsr_backward_finalize_pull(const GsrBackwardArgs* args, const void* const* peer_accums,
                                  const void* const* peer_touched, int n_peers, int self, void* clear_accum,
                                  unsigned char* clear_touched, void* stream);

/* Colour gradient alone: dL_dcolor [P,3] = sum over the pixels of T alpha dL_dpix, the colour part of gsr_backward,
 * for callers that optimise nothing but the colours (test-time appearance optimisation).  Reads P, M, R, W, H,
 * subpixel_offset, geom_buffer, binning_buffer, img_buffer (that of the forward or of gsr_forward_recolor), dL_dpix,
 * tile_y0 / tile_y1 and debug; every other field is ignored.  dL_dcolor is written completely (zero for Gaussians no
 * pixel blends).                                                                                                        */
int gsr_backward_colors(const GsrBackwardArgs* args, void* stream);

/* -- markVisible (rasterizer_impl.cu:54-66,141-153): present[i] = (view*p).z > 0.2 ------- */
int gsr_mark_visible(int P, const float* means3D, const float* viewmatrix,
                     const float* projmatrix, uint8_t* present, void* stream);

/* -- introspection used by parity tests and the benchmark -------------------------------- */
/* accum_alpha (= final transmittance T per pixel, [H,W] f32) lives at the first
 * 128-byte-aligned address of img_buffer, as in the reference ImageState
 * (rasterizer_impl.cu:172-178; read by __init__.py:101-113).                               */
int gsr_img_views(const void* img_buffer, int W, int H,
                  const float** final_T, const uint32_t** n_contrib, const uint32_t** ranges /* uint2[T] */);
/* sorted (tile-major, depth-minor) Gaussian index list, R entries                          */
int gsr_binning_views(const void* binning_buffer, int num_rendered, const uint32_t** point_list);
/* per-Gaussian projected state: depths f32[P], packed records float4[2P]
 * {x, y, hx, hy | conic.x, conic.y, conic.z, opacity*coef} (hx, hy: conservative half extents of the
 * alpha >= 1/255 footprint, used for per-warp culling), tiles_touched u32[P], rgb f32[3P]            */
int gsr_geom_views(const void* geom_buffer, int P, int M, const float** depths,
                   const float** records, const uint32_t** tiles_touched, const float** rgb);
int gsr_get_stats(const void* geom_buffer, int P, int M, void* stream, GsrStats* out);

/* -- fused per-Gaussian colour op of wild-gaussians (SURVEY.md 8f-2; optional entry points) ---------------------------
 * Replaces, for sh_degree = 3 (48 SH features), 24 per-Gaussian embedding features and a 32-d image embedding, the
 * PyTorch statements of wildgaussians/method.py that turn the model's features into the two colour sets the rasterizer
 * composites: `features.clamp_max(1)` (:1570), eval_sh + 0.5 + clamp_min(0) for the raw colours (:1571-1579, :493-548),
 * EmbeddingModel.forward (59 -> 128 -> 128 -> 6 MLP, x 0.01, affine on the features; :874-900) and the toned colours
 * (:1586-1598).  The MLP runs on wgmma tensor cores (bf16 operands, fp32 accumulation).
 *   1. gsr_appearance_pack_weights(): fp32 nn.Linear parameters + the image embedding -> packed bf16 operand image
 *      (gsr_appearance_packed_weight_bytes() bytes, 16-byte aligned); once per step
 *   2. gsr_appearance_colors_forward():  colors_raw (optional) and colors_toned, [P,3] each
 *   3. gsr_appearance_colors_backward(): gradients of every per-Gaussian input; weight gradients are accumulated in
 *      `grad_pack` (gsr_appearance_grad_pack_bytes() bytes, zeroed by the call)
 *   4. gsr_appearance_unpack_grads():    grad_pack -> dW1 [128,59], db1 [128], dW2 [128,128], db2 [128], dW3 [6,128],
 *      db3 [6], d(image embedding) [32]
 * `status` (optional, device int, zero it first) becomes non-zero if an internal barrier wait timed out.              */
typedef struct GsrAppearanceArgs {
    int P;
    int sh_degree;                    /* ACTIVE degree 0..3 (method.py: active_sh_degree); storage is always degree 3 */
    const float* features_dc;         /* [P,3]   raw (unclamped) DC features                                          */
    const float* features_rest;       /* [P,45]  raw higher-order features, coefficient-major (k, channel)            */
    const float* embeddings;          /* [P,24]  per-Gaussian appearance features                                      */
    const float* means3D;             /* [P,3]                                                                         */
    const float* campos;              /* [3]                                                                           */
    const void*  packed_weights;      /* from gsr_appearance_pack_weights                                              */
    float* colors_raw;                /* [P,3] out, may be NULL                                                        */
    float* colors_toned;              /* [P,3] out                                                                     */
    /* backward only */
    const float* dL_dcolors_raw;      /* [P,3] or NULL                                                                 */
    const float* dL_dcolors_toned;    /* [P,3]                                                                         */
    float* dL_dfeatures_dc;           /* [P,3]                                                                         */
    float* dL_dfeatures_rest;         /* [P,45]                                                                        */
    float* dL_dembeddings;            /* [P,24]                                                                        */
    float* dL_dmeans3D;               /* [P,3]  through the view direction of the SH evaluation                        */
    float* grad_pack;                 /* packed weight-gradient image                                                  */
    int*   status;                    /* optional                                                                      */
    /* deterministic != 0: the backward entry points add the per-CTA weight-gradient partials in CTA order (one row
     * of det_scratch per CTA, gsr_appearance_deterministic_scratch_bytes() bytes) instead of with float atomics, so the
     * gradients are bitwise identical from run to run on the same device model.                                       */
    int    deterministic;
    float* det_scratch;
} GsrAppearanceArgs;

size_t gsr_appearance_packed_weight_bytes(void);
size_t gsr_appearance_grad_pack_bytes(void);
size_t gsr_appearance_deterministic_scratch_bytes(void);
int gsr_appearance_pack_weights(const float* W1, const float* b1, const float* W2, const float* b2, const float* W3,
                                const float* b3, const float* appearance_embedding, void* packed_weights, void* stream);
int gsr_appearance_colors_forward(const GsrAppearanceArgs* args, void* stream);
int gsr_appearance_colors_backward(const GsrAppearanceArgs* args, void* stream);
int gsr_appearance_unpack_grads(const float* grad_pack, const float* W1, const float* appearance_embedding, float* dW1,
                                float* db1, float* dW2, float* db2, float* dW3, float* db3,
                                float* dappearance_embedding, void* stream);
/* Gradient of the image embedding alone (test-time appearance optimisation, where nothing else is trained): recomputes
 * the MLP like gsr_appearance_colors_backward and writes sum over the P rows of dL/d(layer-1 pre-activation) into the
 * db1 slot of `grad_pack` (the rest of the image is zeroed); gsr_appearance_unpack_grads then gives d(image embedding)
 * (and db1; its other outputs are zero).  Reads features_dc / features_rest / embeddings / means3D / campos /
 * packed_weights / dL_dcolors_toned; every other pointer of `args` is ignored.  P = 0 is valid (a zero gradient).     */
int gsr_appearance_embedding_backward(const GsrAppearanceArgs* args, void* stream);

/* -- parameter activations + 3D filter (SURVEY.md 8f-2; optional entry points) --------------------------------------------
 * GaussianModel.get_gaussians (wildgaussians/method.py:1060-1086) in one kernel per direction: rotations = normalize(raw),
 * scales = sqrt(exp(raw)^2 + filter_3D^2), opacities = sigmoid(raw) * sqrt(prod(exp(raw)^2) / prod(exp(raw)^2 + filter_3D^2)).
 * All arrays fp32, [P,3] / [P] / [P,4] (16-byte aligned) / [P].  The backward recomputes the forward; upstream gradients may be
 * NULL (treated as zero).                                                                                                  */
int gsr_gaussian_activations_forward(int P, const float* scales_raw, const float* opacities_raw, const float* rotations_raw,
                                     const float* filter_3D, float* scales, float* opacities, float* rotations, void* stream);
int gsr_gaussian_activations_backward(int P, const float* scales_raw, const float* opacities_raw, const float* rotations_raw,
                                      const float* filter_3D, const float* dL_dscales, const float* dL_dopacities,
                                      const float* dL_drotations, float* dL_dscales_raw, float* dL_dopacities_raw,
                                      float* dL_drotations_raw, void* stream);

/* -- SH colours of models without appearance (optional entry points) ---------------------------------------------------
 * The colour statements of GaussianModel._render_internal for appearance_enabled = False (wildgaussians/method.py:1555-1565)
 * in one kernel per direction: colors = clamp_min(eval_sh(sh_degree, clamp_max(cat(features_dc, features_rest), 1),
 * normalize(means3D - campos)) + 0.5, 0).  Storage degree 3: features_dc [P,3] and features_rest [P,45] (coefficient-major
 * (k, channel), 16-byte aligned) raw and unclamped; sh_degree is the ACTIVE degree 0..3.  means3D [P,3], campos [3],
 * colors [P,3], all fp32.  The backward recomputes the forward; dL_dcolors may be NULL (treated as zero).  It writes every
 * entry of dL_dfeatures_dc [P,3], dL_dfeatures_rest [P,45] (16-byte aligned; zero above the active degree) and
 * dL_dmeans3D [P,3] (through the view direction).  P = 0 is valid.                                                      */
int gsr_sh_colors_forward(int P, int sh_degree, const float* features_dc, const float* features_rest, const float* means3D,
                          const float* campos, float* colors, void* stream);
int gsr_sh_colors_backward(int P, int sh_degree, const float* features_dc, const float* features_rest, const float* means3D,
                           const float* campos, const float* dL_dcolors, float* dL_dfeatures_dc, float* dL_dfeatures_rest,
                           float* dL_dmeans3D, void* stream);

/* -- densification statistics (SURVEY.md 8f-4; optional entry point) -----------------------------------------------------
 * One pass over the Gaussians replacing wildgaussians/method.py:1997-1998 + GaussianModel.add_densification_stats
 * (:1470-1477): for every Gaussian with radii > 0: max_radii2D = max(., radii); xyz_grad += |grad.xy|;
 * accum_abs += |grad.z|; accum_abs_max = max(., |grad.z|) (both NULL when use_gof_abs_gradient is off); denom += 1.
 * viewspace_grad is the [P,3] gradient the rasterizer leaves in means2D.grad (summed over the step's passes).          */
int gsr_densification_stats(int P, const int* radii, const float* viewspace_grad, float* max_radii2D, float* xyz_grad,
                            float* xyz_gradient_accum_abs, float* xyz_gradient_accum_abs_max, float* denom, void* stream);

/* -- densify_and_prune / reset_opacity (optional entry points) ---------------------------------------------------------------
 * GaussianModel.densify_and_prune (wildgaussians/method.py:1420-1468, with _densify_and_clone / _densify_and_split /
 * _densification_postfix / _prune_points) in two steps that share `scratch` (gsr_densify_scratch_bytes(P) bytes of device
 * memory, 16-byte aligned, kept alive from the plan to the apply):
 *   gsr_densify_plan  decides every row's fate -- clone, split and the final prune, on the reference's fp32 arithmetic,
 *                     with Q = the reference's quantile(grads_abs, 1 - ratio) (linear interpolation) found by a radix
 *                     select, for any P -- and writes GSR_DENSIFY_COUNTS words to the DEVICE array `counts`:
 *                     [0] rows cloned, [1] rows split (S), [2] rows after the final prune (P'), [3] rows of the post-split
 *                     set whose largest scale exceeds prune_max_scale, [4] split rows kept, [5] rows with |grad| >= max_grad,
 *                     [6] the bits of Q (float; 0 when accum_abs is NULL), [7] 0.
 *   gsr_densify_apply writes every dynamically sized tensor of P' rows in the reference's order -- survivors of the rows
 *                     that were not split, clones, split copy 1, split copy 2 -- from its old rows.  `normals` is the
 *                     [2S,3] standard-normal draw the reference makes for the split children (its normal
 *                     sample over a [2S,3] mean), split copy c of the r-th split row takes row c S + r.
 * Inputs: xyz_grad / denom / accum_abs [P] (accum_abs NULL when use_gof_abs_gradient is off), xyz [P,3], scales [P,3] (log),
 * rotations [P,4] (unnormalised), opacities [P] (logit), fp32.  The thresholds are the reference's Python floats rounded to
 * fp32 (as the reference's fp32 tensor comparisons round them): max_grad, clone_max_scale = percent_dense * extent,
 * min_opacity, prune_max_scale = 0.1 * extent (used only when size_pruning != 0).  split_scale_mul = fp32(1 / fp32(0.8 N)).
 * Segments: src [P, width] -> dst [P', width]; COPY: clones and split copies repeat the source row; ZERO_NEW: new rows are
 * zero (Adam moments, densification buffers); XYZ / SCALES (width 3): the split copies' positions (rotated samples) and
 * log(exp(s) / 1.6).  Element offsets are 64-bit.  1 <= P <= GSR_DENSIFY_MAX_P.                                          */
#define GSR_DENSIFY_COUNTS 8
#define GSR_DENSIFY_MAX_SEGMENTS 48
#define GSR_DENSIFY_MAX_P 0x3FFFFFFF
enum { GSR_DENSIFY_COPY = 0, GSR_DENSIFY_ZERO_NEW = 1, GSR_DENSIFY_XYZ = 2, GSR_DENSIFY_SCALES = 3 };
typedef struct GsrDensifyArgs {
    int P;
    const float *xyz_grad, *denom, *accum_abs;
    const float *xyz, *scales, *rotations, *opacities;
    float max_grad, clone_max_scale, min_opacity, prune_max_scale;
    int size_pruning;
    float split_scale_mul;
    void* scratch;
    unsigned int* counts;
    const float* normals;   /* apply only; may be NULL when S = 0 */
} GsrDensifyArgs;
typedef struct GsrDensifySegment {
    const float* src;
    float* dst;
    int width;
    int kind;
} GsrDensifySegment;
size_t gsr_densify_scratch_bytes(int P);   /* 0 for an invalid P */
int gsr_densify_plan(const GsrDensifyArgs* args, void* stream);
int gsr_densify_apply(const GsrDensifyArgs* args, const GsrDensifySegment* segments, int num_segments, void* stream);
/* GaussianModel.reset_opacity (method.py:1249-1266): out[i] = logit(min(opacity_with_filter, 0.01) / coef) on the 3D-filtered
 * scales, opacities [P] (logit), scales [P,3] (log), filter_3D [P]; out may not alias opacities.  P = 0 is valid.          */
int gsr_reset_opacity(int P, const float* opacities, const float* scales, const float* filter_3D, float* out, void* stream);

/* -- optimizer step (SURVEY.md 8f-4; optional entry point) ------------------------------------------------------------------
 * One launch replacing `self.model.optimizer.step()` (wildgaussians/method.py:2019) of the Adam optimizer built at
 * method.py:1033-1049 (lr per group, eps = 1e-15, weight_decay on the appearance-embedding table only; amsgrad /
 * maximize off).  The algorithm lives in the reference's third-party dependency PyTorch (optim/adam.py,
 * _multi_tensor_adam); this entry point performs the same fp32 operations per element, all tensors in one pass.
 * `step` is the 1-based step count of the tensor AFTER this update (PyTorch increments state["step"] first); lr / step
 * may differ per segment.  All pointers are device pointers to fp32 arrays of `n` elements; `grad` is only written when
 * zero_grads != 0 (it is then left all-zero, the in-place counterpart of zero_grad()).                                  */
#define GSR_ADAM_MAX_SEGMENTS 32
typedef struct GsrAdamSegment {
    float* param;
    float* grad;
    float* exp_avg;
    float* exp_avg_sq;
    long long n;
    long long step;
    double lr;
    double weight_decay;
} GsrAdamSegment;
int gsr_adam_step(const GsrAdamSegment* segments, int num_segments, double beta1, double beta2, double eps, int zero_grads,
                  void* stream);

/* -- 3D filter sizes over all training cameras (SURVEY.md 8f-4; optional entry point) -----------------------------------------
 * Replaces GaussianModel.compute_3D_filter (wildgaussians/method.py:1140-1190): per Gaussian the smallest camera-space depth
 * over the cameras that see it (depth > 0.2 and projection inside the image enlarged by 15 %), Gaussians no camera sees get
 * the largest such depth; filter_3D = distance / focal_length * sqrt(0.2).  `cameras` is a device array of num_cameras
 * records of 20 floats: R[9] (row-major, the matrix method.py:1165 multiplies with: xyz @ R + T), T[3], fx, fy, W/2, H/2,
 * -0.15 W, 1.15 W, -0.15 H, 1.15 H; `focal_length` = the largest fx (method.py:1178-1179).  `scratch`: device memory of
 * gsr_filter3d_scratch_bytes(P) bytes, 16-byte aligned.  filter_3D: [P] (the reference stores it as [P,1]).               */
size_t gsr_filter3d_scratch_bytes(int P);
int gsr_compute_3d_filter(int P, const float* xyz, int num_cameras, const float* cameras, float focal_length,
                          float* filter_3D, void* scratch, void* stream);

/* -- initial scales from the point cloud (SURVEY.md 8f-4; optional entry point) -------------------------------------------
 * Replaces distCUDA2 of the reference's simple-knn submodule (spatial.cu:15-26 -> SimpleKNN::knn, simple_knn.cu:185-220;
 * called once at method.py:1001): mean_dist2[i] = mean of the squared distances from point i to its 3 nearest OTHER points
 * (fp32, the reference's expression and summation order; exact search, so the values are the reference's).
 * points: [P,3] fp32 on the device; scratch: gsr_knn_scratch_bytes(P) bytes of device memory, 256-byte aligned.           */
size_t gsr_knn_scratch_bytes(int P);
int gsr_knn_mean_dist2(int P, const float* points, float* mean_dist2, void* scratch, void* stream);

/* -- SSIM of the photometric loss (optional entry points) ---------------------------------------------------------------
 * The `ssim` of wildgaussians/method.py:644-673 (11-tap Gaussian window, sigma 1.5, zero padding 5, C1 = 0.01^2,
 * C2 = 0.03^2; map = mean over the 3 channels of the per-channel SSIM), one kernel per direction.  img1, img2:
 * [B,3,H,W] fp32, contiguous, on the device; ssim_map: [B,H,W].  partials: NULL when no backward follows, otherwise
 * [B][3 factors][3 channels][H][W] fp32 (36 B per pixel: dS/dmu_x, dS/dE_xx, dS/dE_xy per channel), written by the
 * forward and read by the backward.  The backward takes the upstream dL_dmap [B,H,W] and writes dL_dimg1 [B,3,H,W]
 * (no gradient for img2).  B <= 65535.                                                                                    */
int gsr_ssim_forward(int B, int H, int W, const float* img1, const float* img2, float* ssim_map, float* partials /* NULL: no backward */,
                     void* stream);
int gsr_ssim_backward(int B, int H, int W, const float* img1, const float* img2, const float* partials, const float* dL_dmap,
                      float* dL_dimg1, void* stream);

/* -- loss block of the training step (optional entry points) -----------------------------------------------------------
 * wildgaussians/method.py:1920-1992 around the SSIM: scale_grads by the mask and loss_mult, l1_loss, the weighted loss
 * means and the metric sums.  toned, raw, gt: [3][H][W] fp32; mask, weight, grad_scale: [H][W] or NULL (mask NULL: no
 * mask; weight NULL: loss_mult 1 in the loss; grad_scale NULL: no scale_grads by loss_mult).  raw_scaled [3][H][W]:
 * raw after scale_grads, required when mask or grad_scale is given (it is the SSIM's input).  ssim_map [H][W],
 * ssim_partials [9][H][W] (NULL when no backward follows): the buffers of gsr_ssim_forward, which the forward calls.
 * c_l1 = fp32(1 - lambda_dssim), c_ssim = fp32(lambda_dssim).  Forward outputs: loss [1] (without the uncertainty
 * term); metrics [8]: means of L1, SSIM and MSE, psnr, then with a mask mean(mask), sum(ssim m) / sum(m),
 * sum(mse m) / sum(m), sum(L1 m) / sum(m) (zeros without a mask).  scratch: gsr_train_loss_scratch_bytes() bytes of
 * device memory, 16-byte aligned.  The backward takes dL_dloss [1] and writes dL_dmap [H][W] (a scratch map),
 * d_toned and d_raw [3][H][W].  Three launches forward, two backward; no float atomics, no host synchronisation.       */
typedef struct GsrTrainLossArgs {
    int H, W;
    float c_l1, c_ssim;
    const float *toned, *raw, *gt, *mask, *weight, *grad_scale;
    float *raw_scaled, *ssim_map, *ssim_partials, *loss, *metrics;
    void* scratch;
    const float* dL_dloss;
    float *dL_dmap, *d_toned, *d_raw;
} GsrTrainLossArgs;
size_t gsr_train_loss_scratch_bytes(void);
int gsr_train_loss_forward(const GsrTrainLossArgs* args, void* stream);
int gsr_train_loss_backward(const GsrTrainLossArgs* args, void* stream);
/* Byte-staged training images: img_hwc [H][W][3] uint8 -> img_chw [3][H][W] fp32 and mask_hw [H][W] uint8 -> mask_out
 * [H][W] fp32, each as x / 255.0f (IEEE division: the bits of numpy's astype(float32) / 255.0).  Either input may be
 * NULL (not both).  One launch.                                                                                          */
int gsr_unpack_u8(int H, int W, const unsigned char* img_hwc, const unsigned char* mask_hw, float* img_chw, float* mask_out,
                  void* stream);
/* The inverse of gsr_unpack_u8 for training data kept on the device, with its byte-exactness check.  Each item is one
 * fp32 image (C = 3, element (c, y, x) at src[c * stride_c + y * stride_y + x * stride_x], so the reference's [3,H,W]
 * views of HWC arrays and contiguous CHW tensors both qualify) or mask (C = 1, stride_c unused).  It writes dst
 * [H][W][C] uint8 with u = clip(rint(x * 255), 0, 255), rounding half to even, and ORs into *flags (device memory,
 * cleared by the caller): GSR_PACK_NOT_EXACT when some element's (float)u / 255.0f differs from it bit for bit (NaN,
 * +-inf, -0.0, out of range, off the k / 255 grid), GSR_PACK_NOT_BINARY when some element is neither 0 nor 1.  Up to
 * GSR_PACK_MAX_ITEMS items per call, one launch, no host synchronisation; `items` is host memory.                      */
#define GSR_PACK_MAX_ITEMS 32
#define GSR_PACK_NOT_EXACT 1u
#define GSR_PACK_NOT_BINARY 2u
typedef struct GsrPackItem {
    const float* src;
    unsigned char* dst;
    unsigned int* flags;
    long long stride_c, stride_y, stride_x;
    int H, W, C, reserved;
} GsrPackItem;
int gsr_pack_u8_exact(const GsrPackItem* items, int n, void* stream);

/* -- Image-quality statistics of the uncertainty loss (optional entry points, forward only) -----------------------------
 * `msssim(x, y, max_size, min_size)` and `ssim_down(x, y, max_size)` of wildgaussians/method.py:126-187.  img1, img2:
 * [B,3,H,W] fp32, contiguous, on the device; out: [B,H,W].  (h, w) is the area-resize size the caller computed with
 * the reference's own expression (F.interpolate(scale_factor=s, mode='area') gives int(H * s)); h == H && w == W means
 * no resize.  The images are area-resized to (h, w), evaluated there, and the result bilinearly upsampled back to (H, W).
 * msssim: level 0 contributes l*c*s, each 2x2-pooled level (while both sides exceed min_size) its c and s, upsampled to
 * level 0 separately; the product is averaged over the channels.  ssim_down: the SSIM map of gsr_ssim_forward.
 * scratch: device memory of gsr_*_scratch_bytes bytes (ssim_down needs none without a resize).  B <= 65535,
 * min_size >= 1.  No host synchronisation.                                                                                */
size_t gsr_msssim_scratch_bytes(int B, int h, int w, int min_size);   /* 0 for invalid sizes */
int gsr_msssim_forward(int B, int H, int W, int h, int w, int min_size, const float* img1, const float* img2, float* out,
                       void* scratch, void* stream);
size_t gsr_ssim_down_scratch_bytes(int B, int h, int w);              /* 0 for invalid sizes */
int gsr_ssim_down_forward(int B, int H, int W, int h, int w, const float* img1, const float* img2, float* out,
                          void* scratch, void* stream);

/* -- Attention of the DINOv2 backbone (optional entry points, forward only) ---------------------------------------------
 * The core of `Attention.forward` (wildgaussians/dinov2.py:224-233) for 64-wide heads: softmax((q / 8) k^T) v per head.
 * qkv: the `qkv` Linear's output [B][N][3][H][64] fp32, contiguous, 16-byte aligned, on the device; out: [B][N][H * 64]
 * fp32 (heads concatenated, the input of `proj`).  Exact softmax with 3xTF32 tensor-core products.  scratch: device
 * memory of gsr_attention_scratch_bytes bytes (B * H * ceil(N / 64) * 80 KB).  B <= 65535, H <= 65535, N >= 1.
 * Two launches, no atomics, no host synchronisation.                                                                     */
size_t gsr_attention_scratch_bytes(int B, int N, int H);            /* 0 for invalid sizes */
int gsr_attention_forward(int B, int N, int H, const float* qkv, float* out, void* scratch, void* stream);

/* -- Token-wise layers of the DINOv2 backbone (optional entry points, forward only) ------------------------------------
 * The rest of `get_intermediate_layers` (wildgaussians/dinov2.py:704-813) around gsr_attention_forward, fp32 in and
 * out with 3xTF32 tensor-core products (two accumulators per 32-wide K chunk, summed in fp32), LayerNorm statistics in
 * double, exact-erf GELU.  Every array is contiguous on the device; those marked (16) must be 16-byte aligned.  One
 * launch per call, no atomics (two calls are bitwise identical), no scratch, no host synchronisation.
 *
 * gsr_vit_tokens: `prepare_tokens_with_masks` without masks.  x: [B][3][H][W], H and W multiples of the (even) patch
 *   size p; weight (16): the patch convolution's [C][3][p][p]; bias (16): [C]; cls: [C]; reg: [R][C] (NULL when R = 0);
 *   pos (16): the interpolated position embedding [1 + P][C] (P = H / p * W / p); tokens (16): [B][T][C] out,
 *   T = 1 + R + P, in the reference's order: class token + pos[0], the R register tokens, patch p + pos[1 + p].
 *   C a multiple of 64 up to 1024, B <= 65535, B * T < 2^31.
 * gsr_vit_linear: out = epilogue(prologue(x) weight^T + bias) for x [M][K] (16), weight [N][K] (16) (an nn.Linear's
 *   weight as it is), bias [N] (16), out [M][N] (16); K a multiple of 4, N of 64, both up to 4096.
 *   GSR_VIT_LN_BIAS   LayerNorm(x; ln_w, ln_b, eps) first          (norm1 + qkv)
 *   GSR_VIT_LN_GELU   LayerNorm first, gelu_erf after the bias       (norm2 + fc1 + act)
 *   GSR_VIT_RESIDUAL  out = resid + (x weight^T + bias) * gamma      (proj + ls1, fc2 + ls2); gamma [N] (16) or NULL
 *                     (LayerScale is Identity), resid [M][N] (16); out may be resid (updated in place).
 * gsr_vit_output: the final `norm` of one taken block's tokens [B][T][C] (norm_w and norm_b [C], or both NULL for
 *   norm=False: a copy).  The patch tokens go to `patches` as [B][P][C] (GSR_VIT_LAYOUT_TOKENS) or [B][C][P], which is
 *   reshape=True's [B][C][H / p][W / p] (GSR_VIT_LAYOUT_CHANNELS); the class token to cls [B][C] unless it is NULL.
 *   C a multiple of 32 up to 1024, T >= R + 2, B <= 65535.                                                                 */
#define GSR_VIT_LN_BIAS 0
#define GSR_VIT_LN_GELU 1
#define GSR_VIT_RESIDUAL 2
#define GSR_VIT_LAYOUT_TOKENS 0
#define GSR_VIT_LAYOUT_CHANNELS 1
int gsr_vit_tokens(int B, int H, int W, int C, int patch, int R, const float* x, const float* weight, const float* bias,
                   const float* cls, const float* reg, const float* pos, float* tokens, void* stream);
int gsr_vit_linear(int op, int M, int K, int N, const float* x, const float* ln_w, const float* ln_b, float eps,
                   const float* weight, const float* bias, const float* gamma, const float* resid, float* out, void* stream);
int gsr_vit_output(int B, int T, int C, int R, int layout, const float* tokens, const float* norm_w, const float* norm_b,
                   float eps, float* patches, float* cls, void* stream);

/* -- Head and `dino`-mode loss of the uncertainty model (optional entry points) -----------------------------------------
 * After the frozen backbone: `_forward_uncertainty_features` (wildgaussians/method.py:300-323; dropout2d, BatchNorm in
 * training mode, the 1x1 conv_seg, + log(e - 1), softplus, bilinear upsample, clamp, crop) and the `dino` branch of
 * `_compute_losses` (:363-433) for batch 1, fp32, everything contiguous on the device.
 *   feat: [C][th][tw] backbone features of the normalised, padded ground truth (padded size Hp x Wp, image H x W at
 *   (pad_top, pad_left)); mask: [C] dropout2d channel scales (0 or 1 / (1 - p)); conv_w [C], conv_b [1], bn_w [C],
 *   bn_b [C]: the head's parameters; running_mean / running_var [C] and num_batches_tracked (int64) are updated as
 *   F.batch_norm in training mode does with exponential factor bn_momentum (any of the three may be NULL).
 *   gt, pred: [3][H][W]; ssim, msssim: [H][W] (the statistics of method.py:368-369).  (nh, nw): the 350-px map size
 *   (dino_downsample; == (H, W) without a resize); feat_gt_down, feat_pred_down: [C][ch][cw] features of the two 350-px
 *   images, padded to nHp x nWp with the map at (npad_top, npad_left).
 *   Outputs: loss_mult [H][W] (min(1 / (2 u^2), 3)); loss [1]; metrics [7]: loss, ssim, msssim, ssim_discounted,
 *   mse_discounted, psnr_discounted, beta.  scratch: gsr_uncertainty_scratch_bytes bytes of device memory, kept
 *   unchanged from a forward to its backward.  The backward takes dL_dloss [1] and writes d_conv_w, d_conv_b, d_bn_w,
 *   d_bn_b (the backbone features take no gradient).  Six launches forward, three backward; no atomics, no host
 *   synchronisation; 1 <= C <= 2048, th * tw >= 2.                                                                         */
typedef struct GsrUncertaintyArgs {
    int C, th, tw, Hp, Wp, pad_top, pad_left, H, W;
    int nh, nw, ch, cw, nHp, nWp, npad_top, npad_left;
    float clip_min, reg_weight, bn_eps, bn_momentum;
    const float *feat, *feat_gt_down, *feat_pred_down, *mask;
    const float *conv_w, *conv_b, *bn_w, *bn_b;
    float *running_mean, *running_var;
    long long* num_batches_tracked;
    const float *gt, *pred, *ssim, *msssim;
    float *loss_mult, *loss, *metrics;
    void* scratch;
    const float* dL_dloss;
    float *d_conv_w, *d_conv_b, *d_bn_w, *d_bn_b;
} GsrUncertaintyArgs;
size_t gsr_uncertainty_scratch_bytes(const GsrUncertaintyArgs* args);   /* 0 for invalid sizes */
int gsr_uncertainty_forward(const GsrUncertaintyArgs* args, void* stream);
int gsr_uncertainty_backward(const GsrUncertaintyArgs* args, void* stream);

/* -- Uncertainty loss of every mode, in training or evaluation mode, with a capped head input (optional entry points) --
 * The same head and `_compute_losses` (wildgaussians/method.py:339-433) for uncertainty_mode l2reg, l1reg, dino and
 * dino+mssim (mode: GSR_UNC_MODE_*), with training = 1 (dropout2d scales in mask, BatchNorm with batch statistics and
 * the running-statistics update, as GsrUncertaintyArgs) or 0 (BatchNorm from running_mean / running_var, which are
 * then required and left unchanged, as is num_batches_tracked; mask is ignored).  The head runs on the head input of
 * size uh x uw (`_scale_input`; (H, W) without a cap), padded to Hp x Wp with the input at (pad_top, pad_left); u,
 * log u and beta are at that size.  H x W: the images gt, pred [3][H][W], ssim and msssim [H][W].
 *   l2reg / l1reg: u is resized bilinearly to H x W when the sizes differ; loss_mult = 1 / (2 u^2) or 1 / u (not
 *   clamped); loss = mean((1 - msssim) loss_mult) + reg_weight beta.  The 350-px fields are not read.
 *   dino / dino+mssim: loss_mult = 1 / (2 u^2) at uh x uw, resized to the 350-px map nh x nw (the map of the image; the
 *   caller guarantees dino_downsample gives the same grid from uh x uw), times the dino part (for dino+mssim the
 *   smaller of it and 1 - msssim_down [nh][nw]); the loss_mult written is the resize to H x W clamped at 3.
 *   Metrics as GsrUncertaintyArgs, from the written loss_mult.  Forward: four launches (l2reg, l1reg) or six (dino,
 *   dino+mssim); backward four or three.  No atomics, no host synchronisation; training needs th * tw >= 2.           */
enum { GSR_UNC_MODE_L2REG = 0, GSR_UNC_MODE_L1REG = 1, GSR_UNC_MODE_DINO = 2, GSR_UNC_MODE_DINO_MSSIM = 3 };
typedef struct GsrUncertaintyModeArgs {
    int mode, training;
    int C, th, tw, Hp, Wp, pad_top, pad_left, uh, uw, H, W;
    int nh, nw, ch, cw, nHp, nWp, npad_top, npad_left;
    float clip_min, reg_weight, bn_eps, bn_momentum;
    const float *feat, *feat_gt_down, *feat_pred_down, *mask;
    const float *conv_w, *conv_b, *bn_w, *bn_b;
    float *running_mean, *running_var;
    long long* num_batches_tracked;
    const float *gt, *pred, *ssim, *msssim, *msssim_down;
    float *loss_mult, *loss, *metrics;
    void* scratch;
    const float* dL_dloss;
    float *d_conv_w, *d_conv_b, *d_bn_w, *d_bn_b;
} GsrUncertaintyModeArgs;
size_t gsr_uncertainty_mode_scratch_bytes(const GsrUncertaintyModeArgs* args);   /* 0 for invalid sizes */
int gsr_uncertainty_mode_forward(const GsrUncertaintyModeArgs* args, void* stream);
int gsr_uncertainty_mode_backward(const GsrUncertaintyModeArgs* args, void* stream);

/* -- Evaluation metrics (optional entry points) ------------------------------------------------------------------------
 * The per-image sums behind `compute_metrics` of wildgaussians/evaluation.py:331-352.  a, b: [B][H][W][C], each uint8
 * (a_u8 != 0, read as v / 255.0f) or fp32, contiguous, on the device; both are clipped to [0, 1] as np.clip does it.
 * taps: the 11 dm_pix Gaussian taps (sigma 1.5, as the host computes them); c1 = (k1 max_val)^2, c2 = (k2 max_val)^2.
 * Outputs: sums [B][3] fp64: sum of (a - b)^2 and of |a - b| over all H W C values (fp32 terms), and sum of the SSIM
 * map over its (H - 10) (W - 10) C valid outputs (filtered in fp64); lpips_a, lpips_b (both or neither): x * 2 - 1 of the
 * clipped a and b, fp32 [B][H][W][C].  scratch: gsr_metrics_scratch_bytes bytes of device memory, 8-byte aligned.
 * H >= 11, W >= 11, B * C <= 65535.  Two launches, no atomics, no host synchronisation.                               */
typedef struct GsrMetricsArgs {
    int B, H, W, C;
    int a_u8, b_u8;
    const void *a, *b;
    double taps[11];
    double c1, c2;
    float *lpips_a, *lpips_b;
    double* sums;
    void* scratch;
} GsrMetricsArgs;
size_t gsr_metrics_scratch_bytes(int B, int H, int W, int C);   /* 0 for invalid sizes */
int gsr_metrics_forward(const GsrMetricsArgs* args, void* stream);

/* Optional per-stage device timing (cudaEvents on the caller's stream around each stage of the
 * next forward / backward calls).  The caller synchronises the stream, then reads the stage times of
 * the most recent calls in milliseconds (-1 for stages that did not run).  Not thread-safe.        */
void        gsr_profile_enable(int on);
int         gsr_profile_stage_count(void);
const char* gsr_profile_stage_name(int i);
int         gsr_profile_read(float* ms, int n);
/* number of kernels this library has launched in this process                                     */
unsigned long long gsr_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* GSRAST_H_INCLUDED */
