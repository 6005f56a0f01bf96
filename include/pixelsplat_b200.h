/*
 * pixelsplat_b200.h -- C ABI of the native (H100, sm_90a) render hot path of pixelSplat.
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference binds its rasterizer through the
 * Python extension `diff_gaussian_rasterization` (imported at
 * /root/reference/src/model/decoder/cuda_splatting.py:5-8, called at :99-124 and :192-217);
 * that extension's own C++ entry points are `_C.rasterize_gaussians` /
 * `_C.rasterize_gaussians_backward` (un-vendored dependency, requirements.txt:17).  The two
 * functions below replace exactly those two, generalised to a batch of scenes x views so that
 * `render_cuda`'s per-view Python loop (cuda_splatting.py:91-126), its two `.item()` host syncs
 * (:102-103), the SH permute copy (:75), the covariance triu gather (:123) and
 * DecoderSplattingCUDA's `repeat` of every Gaussian tensor per view
 * (decoder_splatting_cuda.py:53-56) all disappear.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless it says "host"; nothing here is a torch type;
 *   - all work is enqueued on `stream`; no call synchronises the device;
 *   - every function returns PS_OK (0) or a PS_ERR_* code; ps_last_error() gives the text;
 *   - matrices are 16 floats, column-major (element [4*col+row]) -- the flattened row-major
 *     transpose that cuda_splatting.py:85-87 builds;
 *   - fp32 throughout; indices uint32; sort keys uint64.
 */
#ifndef PIXELSPLAT_B200_H
#define PIXELSPLAT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define PS_API __attribute__((visibility("default")))
#else
#define PS_API
#endif

#define PS_OK 0
#define PS_ERR_INVALID_ARGUMENT 1
#define PS_ERR_CUDA 2
#define PS_ERR_UNSUPPORTED 3

#define PS_TILE 16 /* upstream BLOCK_X = BLOCK_Y */

/* sh_layout */
#define PS_SH_M3 0 /* [P, M, 3]  what GaussianRasterizer.forward receives (cuda_splatting.py:75) */
#define PS_SH_3M 1 /* [P, 3, M]  pixelSplat's native Gaussians.harmonics (model/types.py:11)    */
/* SH convention (ps_raster_desc.sh_basis, ps_sh_rotation_matrices' `convention`):
 *   3DGS  z polar, Condon-Shortley sign (-1)^m, degree 1 = C1 (-y, z, -x): upstream 3DGS (SURVEY.md A.4);
 *   E3NN  y polar, no Condon-Shortley sign, degree 1 = C1 (x, y, z): the basis of e3nn's real harmonics,
 *         in which the reference rotates its coefficients (/root/reference/src/misc/sh_rotation.py:18-22,
 *         ply_export.py:75 "our axes are swizzled for the spherical harmonics").
 *   Y_e3nn,i(x, y, z) = (-1)^m Y_3dgs,i(z, x, y). */
#define PS_SH_BASIS_3DGS 0
#define PS_SH_BASIS_E3NN 1
/* cov_layout */
#define PS_COV_TRIU6 0 /* [P, 6]  xx,xy,xz,yy,yz,zz = cov3D_precomp (cuda_splatting.py:115,123) */
#define PS_COV_3X3 1   /* [P, 3, 3]  Gaussians.covariances; only the upper triangle is read, and
                          only the upper triangle receives gradient (autograd of the triu gather) */

typedef struct ps_raster_desc {
    int32_t n_scenes;        /* S: independent Gaussian sets                                   */
    int32_t views_per_scene; /* V: cameras that share one Gaussian set                         */
    int32_t n_gaussians;     /* P per scene                                                    */
    int32_t sh_coeffs;       /* M (1..25) when colours come from SH; 0 = colors_precomp [P,3]  */
    int32_t sh_degree;       /* active degree, 0..4, (sh_degree+1)^2 <= M                      */
    int32_t sh_layout;       /* PS_SH_*                                                        */
    int32_t cov_layout;      /* PS_COV_*                                                       */
    int32_t height, width;   /* image size in pixels                                           */
    int32_t sort_impl;       /* 0 = native per-tile radix sort; 1 = CUB segmented sort (debug)  */
    int32_t sort_segment_hint; /* longest (view,tile) list expected (from a previous call's
                                  n_instances_host[1]); 0 = unknown.  Only selects the shared-memory
                                  size of the sort; any value is correct                        */
    int64_t instance_capacity; /* room, in (tile,Gaussian) instances, summed over all S*V views */
    /* appended in round 2 (struct grows at the end only) */
    int32_t sh_basis;        /* PS_SH_BASIS_*: the convention the SH coefficients are evaluated in    */
    int32_t depth_mode;      /* PS_DEPTH_*: also composite a depth channel (0 = colour only)    */
} ps_raster_desc;

/* depth_mode: the per-(view, Gaussian) value d composited into the depth image sum_i w_i d_i (background 0, no
 * clamp) with the colour pass's alphas, from z = the camera-space depth in WORLD units (view-space z / scene_scale);
 * the "colour" render_depth_cuda composites (/root/reference/src/model/decoder/cuda_splatting.py:238-251).
 * near / far are ps_raster_inputs.near_far (world units), eps = 1e-10. */
#define PS_DEPTH_NONE 0
#define PS_DEPTH_Z 1                 /* d = z                                                                */
#define PS_DEPTH_DISPARITY 2         /* d = 1 / z                                                            */
#define PS_DEPTH_RELATIVE_DISPARITY 3 /* d = 1 - (1/(z+eps) - 1/(far+eps)) / (1/(near+eps) - 1/(far+eps) + eps) */
#define PS_DEPTH_LOG 4               /* d = log(max(min(z, near), far)), as the reference writes it         */

/* Per-call inputs. Camera arrays are indexed by flat view id  vid = scene * V + view. */
typedef struct ps_raster_inputs {
    const float *means;      /* [S, P, 3]                                                      */
    const float *cov;        /* [S, P, 6] or [S, P, 3, 3] (cov_layout)                         */
    const float *opacities;  /* [S, P]                                                         */
    const float *sh;         /* [S, P, M, 3] / [S, P, 3, M] (sh_layout), or colours [S, P, 3]  */
    const float *viewmatrix; /* [S*V, 16] world->camera, column-major                          */
    const float *projmatrix; /* [S*V, 16] world->clip (view @ proj), column-major              */
    const float *campos;     /* [S*V, 3]                                                       */
    const float *tanfov;     /* [S*V, 2] tan(fov_x/2), tan(fov_y/2)                            */
    const float *background; /* [S*V, 3]                                                       */
    const float *scene_scale; /* [S*V] or NULL: means*=s, cov*=s*s before use -- the
                                 scale_invariant rescale of cuda_splatting.py:64-71, fused     */
    /* appended with depth_mode */
    const float *near_far;    /* [S*V, 2] (near, far) in world units; required for PS_DEPTH_RELATIVE_DISPARITY
                                 and PS_DEPTH_LOG, unused otherwise (may be NULL)               */
} ps_raster_inputs;

/* Opaque state that lives from forward to backward (the analogue of upstream's geomBuffer /
 * binningBuffer / imgBuffer byte tensors).  The caller allocates; sizes from ps_raster_sizes. */
typedef struct ps_raster_state {
    void *geom;    size_t geom_bytes;
    void *binning; size_t binning_bytes;
    void *image;   size_t image_bytes;
} ps_raster_state;

typedef struct ps_raster_sizes {
    size_t geom_bytes, binning_bytes, image_bytes, backward_bytes;
} ps_raster_sizes;

/* Byte offsets of the intermediates inside the state buffers (parity tests read them;
 * "bit-exact tile/bin indices" is checked on keys / tile_start / tile_count). */
typedef struct ps_raster_layout {
    /* geom */
    size_t depth;         /* f32  [S*V*P]                                                      */
    size_t radii;         /* i32  [S*V*P]                                                      */
    size_t xy;            /* f32x2                                                             */
    size_t conic_opacity; /* f32x4                                                             */
    size_t rgb;           /* f32x4 (r,g,b,unused)                                              */
    size_t rect;          /* u16x4 (minx,miny,maxx,maxy) in tiles                              */
    size_t clamped;       /* u8   bit c set = channel c was clamped to 0                       */
    size_t tile_count;    /* u32  [S*V*tiles]                                                  */
    size_t tile_start;    /* u32  [S*V*tiles] exclusive scan, global instance offsets          */
    size_t tile_cursor;   /* u32  [S*V*tiles] after the sort: live entries per tile (keys_alt)  */
    size_t n_instances;   /* i64  [4] instances needed (may exceed capacity), longest segment,
                                     #visible (view,Gaussian) pairs, unused (0)                     */
    size_t vis_pairs;     /* u32  [S*V*P] compact list of on-screen (view,Gaussian) flat indices  */
    size_t vis_any;       /* u32  [S*P]   unused (no longer written; the offset is kept)            */
    /* binning */
    size_t keys;          /* u64  [capacity]  per tile sorted (float_bits(depth)<<32 | gaussian) */
    size_t keys_alt;      /* u64  [capacity]  sort scratch; after the sort, per tile at tile_start:
                             u32x2 (position << 8 | 8x4-block mask, gaussian) of the entries whose
                             cull box meets the tile, in list order (the compositor's live lists) */
    /* image */
    size_t final_T;       /* f32  [S*V*H*W]                                                    */
    size_t n_contrib;     /* u32  [S*V*H*W]                                                    */
    /* appended in round 2 (struct grows at the end only) */
    size_t cull;          /* geom: f32x4 [S*V*P] (x, y, half-extent x, half-extent y) of the
                             alpha >= 1/255 box -- the compositor's cull record                */
    size_t color;         /* image: f32 [S*V*3*H*W] copy of the rendered colour (the backward's
                             forward-order prefix form needs C . dL/dC per pixel)              */
    size_t block_hits;    /* binning: u32x2 [8 * capacity] per-(tile, 8x4 block, run) hit lists (position, Gaussian)
                             the composite forward leaves for its backward; 0 when not kept (large capacity)   */
    size_t run_hits;      /* binning: u32 [S*V*tiles*8*4] their lengths                                        */
    size_t run_state;     /* image: f32x4 [S*V*3*H*W] (T, Cr, Cg, Cb) in front of list runs 1..3 when the
                             compositor cuts a tile's list into runs (small batches)            */
    size_t sh_jacobian;   /* geom: f32x4 [S*V*P][3] per on-screen (view, Gaussian) pair, row c = the gradient of
                             colour channel c before the clamp with respect to the normalised view direction
                             (x, y, z, unused); written by the forward, read by the backward.  0 and not
                             allocated when sh_coeffs == 0.  (The depth fields stay last.)                     */
    /* appended with depth_mode (both 0 and not allocated when depth_mode == 0) */
    size_t depth_image;   /* image: f32 [S*V*H*W] the composited depth channel                                  */
    size_t run_depth;     /* image: f32 [S*V*3*H*W] depth in front of list runs 1..3 (next to run_state)        */
} ps_raster_layout;

/* Camera gradients of a rasterizer backward (ps_raster_grads.camera).  The function differentiated is the one whose
 * Gaussian gradients the backward returns, with viewmatrix, projmatrix, campos and tanfov as independent inputs:
 * upstream's straight-through min(0.99, .) and hard skip masks, no gradient through radii, tile rectangles or the
 * sort, and the +-1.3 tan(fov) clamp (it removes d/dt.x (d/dt.y) and passes nothing through its limit), so tanfov
 * receives a gradient only through the focal lengths W / (2 tanfov) of the projection Jacobian.  Entries the forward
 * never reads -- viewmatrix [3] [7] [11] [15], projmatrix [2] [6] [10] [14] -- get exactly 0, and so does campos with
 * colours instead of SH.  With a depth gradient the depth value's chain to the viewmatrix is included;
 * scene_scale and near_far are not differentiated.  After a binning overflow every entry is 0.
 * Each output may be NULL (not written); the others are written in full, so they need no initialisation.  No float
 * atomics: in deterministic mode the camera gradients are the same bits on every run.
 * `workspace` (16-byte aligned, no initialisation) has ps_raster_camera_workspace_bytes: the preprocess backward
 * stores one partial sum per (warp of 32 Gaussians, view) there and a finish kernel adds them in a fixed order.
 * Camera-only backward: with `camera` set, d_means, d_cov, d_opacities, d_sh and d_means2d may ALL be NULL.  The call
 * then writes the camera gradients and nothing else (no Gaussian gradient is formed; for the campos term the forward's
 * colour-direction Jacobian, ps_raster_layout.sh_jacobian, is read instead of the SH rows).  Its camera gradients are the full backward's (the same per-Gaussian terms
 * summed in the same order; the compiler may round the campos term differently), and it takes the same scratch and
 * workspace sizes and the same number of launches.  Some but not all of the four required Gaussian pointers NULL, or all five
 * NULL without `camera`, is PS_ERR_INVALID_ARGUMENT before anything is enqueued. */
typedef struct ps_raster_camera_grads {
    float *d_viewmatrix; /* [S*V, 16] column-major like viewmatrix                              */
    float *d_projmatrix; /* [S*V, 16]                                                           */
    float *d_campos;     /* [S*V, 3]                                                            */
    float *d_tanfov;     /* [S*V, 2]                                                            */
    void *workspace;
    size_t workspace_bytes;
} ps_raster_camera_grads;

typedef struct ps_raster_grads {   /* Gaussian outputs all NULL with `camera` set: camera-only backward (above) */
    float *d_means;     /* [S, P, 3]                                                           */
    float *d_cov;       /* same layout as cov                                                  */
    float *d_opacities; /* [S, P]                                                              */
    float *d_sh;        /* same layout as sh (or [S, P, 3] for colours)                        */
    float *d_means2d;   /* [S*V, P, 3] or NULL: upstream's screen-space gradient (x, y, 0)     */
    /* appended with camera gradients (struct grows at the end only) */
    const ps_raster_camera_grads *camera; /* NULL: no camera gradients (the backward is unchanged)  */
} ps_raster_grads;

/* Workspace of ps_raster_grads.camera for a descriptor, closed form (no device needed):
 *   S * V * ((P - 1) / 32 + 2) * 128 bytes  (one 32-float row per warp overlapping a scene, per view).
 * No other size query changes when camera gradients are requested. */
PS_API int ps_raster_camera_workspace_bytes(const ps_raster_desc *desc, size_t *out);

PS_API int ps_version(void);
PS_API const char *ps_last_error(void); /* thread-local, valid until the next failing call */

/* Instrumentation used by bench.py: number of kernels this library has launched so far, and
 * optional per-stage CUDA-event timing (on the launching stream) of the most recent
 * forward + backward pair: ms[7] = preprocess, count-scan + scatter, sort, composite forward,
 * clearing of the on-screen gradient scratch rows, composite backward, preprocess backward. */
PS_API unsigned long long ps_launch_count(void);
PS_API void ps_timing_enable(int on);
PS_API int ps_timing_read(float *ms);

/* Process-wide tunables of the compositor, for A/B measurements and tests (defaults are automatic):
 *   "composite_impl"      2 = warp-task compositor (default), 1 = round-1 CTA-per-tile compositor;
 *   "composite_segments"  0 = automatic (default), 1 | 2 | 4 = list runs per warp task;
 *   "composite_hit_lists" 2 = automatic (default: kept while 64 x instance_capacity <= 512 MB), 0 = never keep,
 *                         1 = always keep the forward's per-block hit lists for the backward (binning_bytes grows).
 * Takes effect for forwards issued afterwards (a backward uses the split and the hit lists its forward used only if
 * the options are unchanged in between).  Also read once from PIXELSPLAT_B200_COMPOSITE / PIXELSPLAT_B200_SEGMENTS /
 * PIXELSPLAT_B200_HIT_LISTS.
 *   "deterministic"       0 = off (default), 1 = fixed-order composite backward and loss epilogue: the same inputs, call
 *                         shape, options and GPU give the same bits on every run (no float atomics on the rasterizer
 *                         path).  Takes effect for calls issued afterwards (sizes queried, forwards and backwards).
 *                         The legacy compositor has no fixed-order form: with the option on its forward and backward
 *                         return PS_ERR_UNSUPPORTED before anything is enqueued.  Workspace with the option on, where
 *                         A(x) rounds x up to a multiple of 256, C = instance_capacity, T = S*V*tiles (16x16 tiles):
 *                           backward_bytes = A(8 S V P) + A(16 S V P) + A(16 S V P)           (as with the option off)
 *                                          + A(8 * 8C) + A(16 * 8C) + A(16 * 8C)  the composite's per-(tile block, list
 *                                                                                 position) gradient records;
 *                           image_bytes    = (the size with the option off) + A(8 * 8T)  per-warp-task loss partials.
 *                         geom_bytes, binning_bytes and the ps_raster_layout offsets do not change. */
PS_API int ps_set_option(const char *name, int value);
/* The value of an option above as it is in force (the environment included): composite_impl 1 | 2,
 * composite_segments 0 | 1 | 2 | 4, composite_hit_lists 0 | 1 | 2, deterministic 0 | 1. */
PS_API int ps_get_option(const char *name, int *value);

/* Workspace sizes / layout for a descriptor. */
PS_API int ps_raster_sizes_query(const ps_raster_desc *desc, ps_raster_sizes *out);
PS_API int ps_raster_layout_query(const ps_raster_desc *desc, ps_raster_layout *out);

/*
 * Camera set-up for n_views views in one launch: the device-side restatement of
 * cuda_splatting.py:64-87 (scale-invariant rescale of the extrinsics translation and near/far,
 * get_fov, get_projection_matrix, extrinsics.inverse(), view @ proj) without the per-view
 * `.item()` host syncs of :102-103.
 *   extrinsics [n,4,4] camera-to-world row-major, intrinsics [n,3,3] normalised, near/far [n]
 *   -> viewmatrix/projmatrix [n,16] (column-major), campos [n,3], tanfov [n,2],
 *      scene_scale [n] (= 1/near when scale_invariant, else 1; feed to ps_raster_inputs).
 */
PS_API int ps_camera_setup(int32_t n_views, const float *extrinsics, const float *intrinsics,
                           const float *near_plane, const float *far_plane, int32_t scale_invariant,
                           float *viewmatrix, float *projmatrix, float *campos, float *tanfov,
                           float *scene_scale, void *stream);

/*
 * Reverse mode of ps_camera_setup, one thread per view (float64 inside): the gradients of the four camera arrays
 * (each may be NULL = zero) are carried back through campos, view @ proj, the 4x4 inverse, the projection matrix,
 * tan / acos of the field of view and the 3x3 inverse of the intrinsics, and the scale-invariant rescale of the
 * translation, to d_extrinsics [n,4,4] and d_intrinsics [n,3,3] (both written in full).  near / far and
 * scene_scale are not differentiated.  Bad arguments return PS_ERR_INVALID_ARGUMENT before anything is enqueued;
 * the call does not synchronise the host (graph-capturable).
 */
PS_API int ps_camera_setup_backward(int32_t n_views, const float *extrinsics, const float *intrinsics,
                                    const float *near_plane, const float *far_plane, int32_t scale_invariant,
                                    const float *d_viewmatrix, const float *d_projmatrix, const float *d_campos,
                                    const float *d_tanfov, float *d_extrinsics, float *d_intrinsics, void *stream);

/*
 * Forward: preprocess -> per-tile count/scan -> scatter -> per-tile radix sort -> composite.
 * Replaces _C.rasterize_gaussians for S*V views at once.
 *   out_color      [S*V, 3, H, W]
 *   out_radii      [S*V, P] int32 or NULL
 *   n_instances_host  pinned HOST int64[2] or NULL: receives {instance count, longest (view,tile)
 *                  list} asynchronously (valid once `stream` reaches this point).  If the count exceeds
 *                  desc->instance_capacity the binning was truncated and out_color is INVALID:
 *                  the caller must re-run with a larger capacity (pixelsplat_b200.rasterizer does).
 */
PS_API int ps_raster_forward(const ps_raster_desc *desc, const ps_raster_inputs *in,
                      const ps_raster_state *state, float *out_color, int32_t *out_radii,
                      int64_t *n_instances_host, void *stream);

/*
 * Backward: composite backward (warp-reduced, one atomic per (tile, Gaussian)) ->
 * per-Gaussian cov2D / projection / SH backward summed over the V views of a scene.
 * Replaces _C.rasterize_gaussians_backward.  `scratch` has ps_raster_sizes.backward_bytes.
 * Every element of every gradient in `grads` is written (zeros where no gradient flows), so they need no
 * initialisation; `scratch` needs none either.
 */
PS_API int ps_raster_backward(const ps_raster_desc *desc, const ps_raster_inputs *in,
                       const ps_raster_state *state, const float *d_color /* [S*V,3,H,W] */,
                       void *scratch, size_t scratch_bytes, const ps_raster_grads *grads,
                       void *stream);

/* With desc->depth_mode != 0, ps_raster_forward / ps_raster_forward_loss also composite the depth channel into
 * the image state (ps_raster_layout.depth_image; the colour, radii and every other output are unchanged).  The
 * legacy compositor (composite_impl = 1) has no depth channel: PS_ERR_UNSUPPORTED before anything is enqueued.
 * ps_raster_backward / ps_raster_backward_loss after such a forward take dL/dD = 0. */

/* Backward of a depth forward with a depth gradient d_depth [S*V, H, W]: dL/dD reaches the Gaussians through the
 * alphas and through d (the means, summed over the V views).  d_color [S*V, 3, H, W], or NULL: then dL/dC comes
 * from the fused loss as in ps_raster_backward_loss (loss_target, grad_scale). */
PS_API int ps_raster_backward_depth(const ps_raster_desc *desc, const ps_raster_inputs *in,
                                    const ps_raster_state *state, const float *d_color /* or NULL */,
                                    const float *loss_target, const float *grad_scale, const float *d_depth,
                                    void *scratch, size_t scratch_bytes, const ps_raster_grads *grads,
                                    void *stream);

/* ---- fused loss epilogue (SURVEY.md 8 row f-4) --------------------------------------------------
 * The training loss the reference applies to the render, LossMse (/root/reference/src/loss/loss_mse.py:30-31,
 * weight * mean((prediction - target)^2)), and the PSNR it logs (src/evaluation/metrics.py:11-19) need, per view,
 * sum (C - t)^2 and sum (clip(C) - clip(t))^2.  ps_raster_forward_loss accumulates both in the compositor's
 * epilogue (the image is not re-read for the loss; out_color may be NULL when nobody needs the pixels), and
 * ps_raster_backward_loss forms dL/dC = grad_scale[view] * (C - target) inside the composite backward, so no
 * gradient image exists as a tensor either.  Host side: pixelsplat_b200/loss.py. */
#define PS_LOSS_SLOTS 64
typedef struct ps_raster_loss {
    const float *target; /* [S*V, 3, H, W] */
    float *sums;         /* [S*V, 2, PS_LOSS_SLOTS]: partial sums, [.,0,.] raw, [.,1,.] clipped to [0, 1];
                            zeroed by the call; sum over the last axis for the per-view totals          */
} ps_raster_loss;

PS_API int ps_raster_forward_loss(const ps_raster_desc *desc, const ps_raster_inputs *in,
                                  const ps_raster_state *state, const ps_raster_loss *loss,
                                  float *out_color /* or NULL */, int32_t *out_radii,
                                  int64_t *n_instances_host, void *stream);
PS_API int ps_raster_backward_loss(const ps_raster_desc *desc, const ps_raster_inputs *in,
                                   const ps_raster_state *state, const float *target /* [S*V,3,H,W] */,
                                   const float *grad_scale /* [S*V]: dL/d(sum of squares) * 2 */,
                                   void *scratch, size_t scratch_bytes, const ps_raster_grads *grads,
                                   void *stream);

/* ------------------------------------------------------------------------------------------
 * Epipolar sampled cross-attention (SURVEY.md 8 rows a8-a13).
 * Replaces, inside EpipolarTransformer.forward
 * (/root/reference/src/model/encoder/epipolar/epipolar_transformer.py:96-142):
 *   ps_epipolar_geometry            EpipolarSampler's ray generation + project_rays
 *                                   (epipolar_sampler.py:62-88, geometry/epipolar_lines.py:157-251),
 *                                   get_depth (epipolar_lines.py:264-292, projection.py:176-230),
 *                                   depth clip + depth_to_relative_disparity
 *                                   (epipolar_transformer.py:103-119, conversions.py:17-27);
 *   ps_epipolar_attention_forward / _backward
 *                                   F.grid_sample of the samples (epipolar_sampler.py:98-111), the
 *                                   depth positional encoding (epipolar_transformer.py:120-121,
 *                                   positional_encoding.py:28-33) and Attention.forward with z != None
 *                                   (transformer/attention.py:54-70) for one transformer layer.
 * Ray index r = row * grid_w + col over the (down-scaled) feature grid; "other view" ov of view v
 * is view ov if ov < v else ov + 1 (misc/heterogeneous_pairings.py:9-24).
 */
typedef struct ps_epipolar_desc {
    int32_t batch, views;     /* b, v (v >= 2)                                                  */
    int32_t grid_h, grid_w;   /* ray / feature grid                                             */
    int32_t samples;          /* S <= 32 samples per epipolar segment                           */
    int32_t channels;         /* feature channels, must be 128                                  */
    int32_t heads;            /* 1..4                                                           */
    int32_t pe_dim;           /* 2 * num_octaves of the depth encoding (<= 32, heads*pe_dim<=96) */
} ps_epipolar_desc;

typedef struct ps_epipolar_inputs {
    const float *features;      /* [b, v, grid_h, grid_w, 128] channels-last                    */
    const float *segments;      /* [b, v, v-1, R, 4] xy_min.xy, xy_max.xy (from ps_epipolar_geometry) */
    const uint8_t *valid;       /* [b, v, v-1, R]                                               */
    const float *rel_disparity; /* [b, v, v-1, R, S]                                            */
    const float *q_feat;        /* [b*v*R, heads, 128]  scale * W_k,h^T q_h                     */
    const float *q_pe;          /* [b*v*R, heads, pe_dim]  W_d^T of the above                   */
    const float *bias;          /* [b*v*R, heads, v-1] or NULL (view-embedding score term)      */
} ps_epipolar_inputs;

/* segments/valid/rel_disparity as above; t_range [b, v, v-1, R, 2] (t_min, t_max) or NULL.
 * PS_ERR_INVALID_ARGUMENT for a count below its minimum (b, grid, samples >= 1, v >= 2) or a NULL required pointer,
 * and PS_ERR_UNSUPPORTED when b * v * (v - 1) > 65535 or grid_h * grid_w >= 2^31, both before anything is
 * enqueued. */
PS_API int ps_epipolar_geometry(int32_t batch, int32_t views, int32_t grid_h, int32_t grid_w,
                                int32_t samples, const float *extrinsics /* [b,v,4,4] c2w */,
                                const float *intrinsics /* [b,v,3,3] */, const float *near_plane,
                                const float *far_plane /* [b,v] */, float *segments, uint8_t *valid,
                                float *rel_disparity, float *t_range, void *stream);

/* View overlap of one step of the evaluation-index walk (EvaluationIndexGenerator.test_step,
 * src/evaluation/evaluation_index_generator.py in the reference).  Over one scene's cameras (extrinsics [views,4,4]
 * c2w, normalised intrinsics [views,3,3]) and the grid_h x grid_w ray grid at pixel centres, for each candidate
 * frame k = first + i, i < count:
 *   counts[i, 0] = rays of frame k whose unbounded projection (project_rays with near = far = None) overlaps the
 *                  image of frame `context`;
 *   counts[i, 1] = rays of frame `context` that overlap the image of frame k.
 * counts [count, 2] int32 is overwritten (zeroed on the stream, then accumulated with one integer atomic per CTA,
 * so the result does not depend on scheduling).  The geometry is ps_epipolar_geometry's, in float64.  One launch,
 * graph-capturable, no host synchronisation.  PS_ERR_INVALID_ARGUMENT for a count below 1 (views, grid, count), a
 * NULL pointer, or a context / candidate range outside [0, views); PS_ERR_UNSUPPORTED when count > 65535 or
 * grid_h * grid_w >= 2^31; both before anything is enqueued. */
PS_API int ps_view_overlap(int32_t views, int32_t grid_h, int32_t grid_w, const float *extrinsics,
                           const float *intrinsics, int32_t context, int32_t first, int32_t count, int32_t *counts,
                           void *stream);

/* z [N,heads,128] = sum_s a_s f_s;  e [N,heads,pe_dim] = sum_s a_s PE(rd_s);
 * mass [N,heads,v-1] = per-other-view attention mass (or NULL);  lse [N,heads] log-sum-exp. */
PS_API int ps_epipolar_attention_forward(const ps_epipolar_desc *desc, const ps_epipolar_inputs *in,
                                         float *z, float *e, float *mass, float *lse, void *stream);

/* d_row [N,heads] = dz.z + de.e (+ dmass.mass).  dfeatures [b,v,grid_h,grid_w,128] must be
 * zero-initialised by the caller; the kernel accumulates into it atomically.  Like the forward, it returns
 * PS_ERR_INVALID_ARGUMENT for a NULL required pointer, in->q_pe included when pe_dim > 0, before anything is
 * enqueued. */
PS_API int ps_epipolar_attention_backward(const ps_epipolar_desc *desc, const ps_epipolar_inputs *in,
                                          const float *lse, const float *dz, const float *de,
                                          const float *dmass, const float *d_row, float *dq_feat,
                                          float *dq_pe, float *dbias, float *dfeatures, void *stream);

/* Fixed-order form of the backward above: dq_feat, dq_pe and dbias are computed by the same code, and dfeatures is
 * summed without float atomics, so the same inputs, desc and GPU give the same bits on every run.  dfeatures is
 * fully written (no zero-fill needed).  Each (query, other view, sample) slot t = (n (v-1) + ov) S + s stores its
 * sample gradient, bilinear weights and cell key; a stable radix sort of the slots by cell, a per-cell sum in
 * ascending slot id and a per-texel sum of its four cells in a fixed order then form dfeatures.  No host
 * synchronisation (graph-capturable).  Workspace, where A(x) rounds x up to a multiple of 256,
 * T = b v R (v-1) S slots and Cn = b v (grid_h+1) (grid_w+1) cells:
 *   A(512 T)                  per-slot sample gradients [T, 128] f32
 * + A(16 T)                   per-slot bilinear weights [T, 4] f32
 * + 4 A(4 T)                  cell keys and slot ids, two of each (radix ping-pong)
 * + A(1024 ceil(T / 4096))    radix histograms [256, chunks of 4096 slots] u32
 * + A(4 (Cn + 1))             cell_start u32
 * + A(2048 Cn)                per-cell tap sums [Cn, 4, 128] f32.
 * Both functions return what ps_epipolar_attention_forward's descriptor check returns, and PS_ERR_INVALID_ARGUMENT
 * for a NULL pointer or a short workspace, before anything is enqueued; PS_ERR_UNSUPPORTED when T or Cn does not
 * fit 31 bits. */
PS_API int ps_epipolar_attention_backward_workspace_bytes(const ps_epipolar_desc *desc, size_t *out);
PS_API int ps_epipolar_attention_backward_deterministic(const ps_epipolar_desc *desc, const ps_epipolar_inputs *in,
                                                        const float *lse, const float *dz, const float *de,
                                                        const float *dmass, const float *d_row, float *dq_feat,
                                                        float *dq_pe, float *dbias, float *dfeatures /* fully written */,
                                                        void *workspace, size_t workspace_bytes, void *stream);

/* ---- dense per-image self-attention (wgmma, TF32 operands, FP32 accumulate) -----------------------
 * Replaces the z = None branch of /root/reference/src/model/transformer/attention.py:54-70 as used by
 * ImageSelfAttention (/root/reference/src/model/encoder/epipolar/image_self_attention.py:57-79):
 *   qkv  [n_images, tokens, 3 * heads * dim_head]   output of to_qkv ("b n (qkv h d)")
 *   out  [n_images, tokens, heads * dim_head]       softmax(q k^T * scale) v, "b n (h d)"
 * Supported shape: tokens == 256, dim_head == 128 (pixelSplat's ViT stage at 256x256), heads <= 16,
 * n_images <= 65535; anything else returns PS_ERR_UNSUPPORTED before anything is enqueued.  scale must be finite
 * and >= 0 (the row max is taken on the unscaled logits), else PS_ERR_INVALID_ARGUMENT, as for a NULL or not
 * 16-byte aligned pointer; the backward checks the same.  debug_mode 1 writes the raw q k^T logits instead
 * (out is then [n_images, heads, 256, 256]); used by the tests only. */
PS_API int ps_self_attention_forward(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                     const float *qkv, float scale, float *out, int32_t debug_mode,
                                     void *stream);

/* The same forward, additionally saving what the backward needs to rebuild the forward's probabilities bit for
 * bit: stats [n_images, heads, 256, 2] = (row max * scale * log2 e, 1 / row sum of the TF32-rounded numerators). */
PS_API int ps_self_attention_forward_stats(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                           const float *qkv, float scale, float *out, float *stats, void *stream);

/* Backward (wgmma, TF32 operands, FP32 accumulate; csrc/self_attention_tc.cu): autograd of the forward
 * above.  out / d_out [n_images, 256, heads * 128]; d_qkv has qkv's layout and is fully written. */
PS_API int ps_self_attention_backward(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                      const float *qkv, const float *out, const float *d_out, const float *stats,
                                      float scale, float *d_qkv, void *stream);

/* ---- fused GaussianAdapter (SURVEY.md 8 row f-1) ----------------------------------------------
 * Replaces /root/reference/src/model/encoder/common/gaussian_adapter.py:48-95 (+ gaussians.py:8-44):
 * per-ray raw network outputs -> world-space Gaussians.  One camera = one (batch, view) pair; every
 * ray carries n_samples Gaussians that share its raw features and differ in depth.
 *   means [n_views, n_rays, n_samples, 3]      covariances [.., 3, 3]      harmonics [.., 3, sh_coeffs]
 *   scales [.., 3] (optional, may be NULL)      rotations [n_views, n_rays, 4] xyzw (optional)
 * Opacities pass through the reference's adapter unchanged and are not part of this call. */
typedef struct ps_adapter_desc {
    int32_t n_views;      /* b * v cameras */
    int32_t n_rays;       /* rays x surfaces per camera */
    int32_t n_samples;    /* Gaussians per ray (1..8) */
    int32_t sh_coeffs;    /* (degree + 1)^2, degree <= 4 */
    int32_t image_h, image_w;
    float scale_min, scale_max; /* GaussianAdapterCfg.gaussian_scale_min / max */
    float eps;            /* 1e-8 in the reference */
    int32_t reserved;
} ps_adapter_desc;

typedef struct ps_adapter_inputs {
    const float *extrinsics;   /* [n_views, 4, 4] camera-to-world */
    const float *intrinsics;   /* [n_views, 3, 3] normalised */
    const float *sh_rotation;  /* [n_views, sh_coeffs, sh_coeffs] block-diagonal D(c2w): c' = D c */
    const float *sh_mask;      /* [sh_coeffs] */
    const float *coordinates;  /* [n_views, n_rays, 2] */
    const float *depths;       /* [n_views, n_rays, n_samples] */
    const float *raw;          /* [n_views, n_rays, 7 + 3 sh_coeffs]: scale logits 3, quaternion xyzw 4, sh [3, sh_coeffs] */
} ps_adapter_inputs;

PS_API int ps_gaussian_adapter_forward(const ps_adapter_desc *desc, const ps_adapter_inputs *in, float *means,
                                       float *covariances, float *harmonics, float *scales, float *rotations,
                                       void *stream);

/* d_scales / d_rotations may be NULL (no gradient reached those outputs).  Outputs: d_coordinates
 * [n_views, n_rays, 2], d_depths [n_views, n_rays, n_samples], d_raw [n_views, n_rays, 7 + 3 sh_coeffs]
 * (all fully written, no zero-initialisation needed). */
PS_API int ps_gaussian_adapter_backward(const ps_adapter_desc *desc, const ps_adapter_inputs *in,
                                        const float *d_means, const float *d_covariances,
                                        const float *d_harmonics, const float *d_scales,
                                        const float *d_rotations, float *d_coordinates, float *d_depths,
                                        float *d_raw, void *stream);

/* Block-diagonal SH rotation matrices D(c2w) [n_views, sh_coeffs, sh_coeffs] for ps_adapter_inputs.sh_rotation
 * (replaces /root/reference/src/misc/sh_rotation.py:10-30, row f-3): c' = D c makes the rotated function at
 * d equal the original at R^T d, in the basis `convention` names.  PS_SH_BASIS_E3NN reproduces the reference's
 * wigner_D(l, *matrix_to_angles(R)) (degree-1 block == R); PS_SH_BASIS_3DGS is the rotation consistent with the
 * rasterizer's default basis.  fit_dirs [n_dirs, 3] are unit directions and fit_pinv [sh_coeffs, n_dirs] the
 * per-degree pseudo-inverse of the 3DGS basis sampled there (pixelsplat_b200/sh.py builds both once, in
 * float64).  extrinsics [n_views, 4, 4] camera-to-world. */
PS_API int ps_sh_rotation_matrices(int32_t n_views, int32_t sh_coeffs, int32_t n_dirs, int32_t convention,
                                   const float *extrinsics, const float *fit_dirs, const float *fit_pinv,
                                   float *out, void *stream);

/* ---- SSIM of image planes (csrc/ssim.cu) ------------------------------------------------------------------
 * Replaces the skimage call of /root/reference/src/evaluation/metrics.py:36-52, structural_similarity(win_size=11,
 * gaussian_weights=True, data_range=1.0) with skimage's defaults (K1 = 0.01, K2 = 0.03, sigma = 1.5, truncate =
 * 3.5, use_sample_covariance), one plane at a time.  For x (ground truth) and y (prediction) [n_planes, H, W] and
 * G the normalised 11 x 11 Gaussian window (sigma 1.5):
 *   mu_x = G*x, mu_y = G*y,  var_x = n (G*x^2 - mu_x^2),  var_y alike,  cov = n (G*xy - mu_x mu_y),  n = 121/120,
 *   S = (2 mu_x mu_y + C1)(2 cov + C2) / ((mu_x^2 + mu_y^2 + C1)(var_x + var_y + C2)),  C1 = 0.01^2, C2 = 0.03^2,
 * and the plane's score is the mean of S over the crop [5, H-5) x [5, W-5), where every window lies inside the
 * image (so no padding mode is involved).  Nothing is clipped.  The constants are fixed; H, W >= 11.
 * No call synchronises the host; the forward's sum is in a fixed order (the same bits every run).  Every entry point
 * rejects n_planes < 1, H < 11, W < 11, NULL pointers and a short workspace with PS_ERR_INVALID_ARGUMENT before
 * anything is enqueued. */
PS_API int ps_ssim_workspace_bytes(int32_t n_planes, int32_t H, int32_t W, size_t *out);

/* out_mean [n_planes] = the planes' scores.  The workspace (ps_ssim_workspace_bytes) holds per-tile partial sums. */
PS_API int ps_ssim_forward(int32_t n_planes, int32_t H, int32_t W, const float *x, const float *y, float *out_mean,
                           void *workspace, size_t workspace_bytes, void *stream);

/* Given d_mean [n_planes] = dL/d(score), writes d_y = dL/dy and, when d_x is not NULL, d_x = dL/dx ([n_planes, H, W],
 * fully written: no zero-fill needed).  The filtered moments are recomputed, not stored.  The workspace is the
 * forward's (same size check, so one buffer serves both); the backward does not write it. */
PS_API int ps_ssim_backward(int32_t n_planes, int32_t H, int32_t W, const float *x, const float *y,
                            const float *d_mean, float *d_x /* or NULL */, float *d_y, void *workspace,
                            size_t workspace_bytes, void *stream);

/* ---- 3DGS's L1 + D-SSIM loss (csrc/l1_dssim.cu) ------------------------------------------------------------
 * For prediction `pred` and ground truth `gt` [n, C, H, W], per image: loss = (1 - lambda) L1 + lambda (1 - SSIM),
 * L1 = mean |pred - gt|, SSIM = 3DGS's training SSIM: the 11x11 Gaussian window of sigma 1.5 correlated "same"-size
 * with zero padding, population (co)variances, C1 = 0.01^2, C2 = 0.03^2, the map averaged over every pixel and channel
 * (no crop; not the evaluation's ps_ssim_*).  Any H, W >= 1.  One launch over (plane, 16 x 32 tile) writes per-tile
 * partial sums and, when d_pred is not NULL, d_pred = d(sum_n loss_n)/d pred (fully written; L1 part
 * (1 - lambda) sign(pred - gt) / (C H W), sign(0) = 0); a second one adds the partials in a fixed order, so the
 * results are the same bits every run and do not depend on whether d_pred is asked for.  No call synchronises the
 * host.  Every entry point rejects a non-positive extent, a grid that does not fit one launch, lambda outside [0, 1]
 * or NaN, NULL required pointers and a short workspace with PS_ERR_INVALID_ARGUMENT before anything is enqueued. */
PS_API int ps_l1_dssim_workspace_bytes(int32_t n, int32_t C, int32_t H, int32_t W, size_t *out);

/* out_loss [n]; out_l1 [n] and out_ssim [n] (the two terms) when not NULL. */
PS_API int ps_l1_dssim(int32_t n, int32_t C, int32_t H, int32_t W, const float *pred, const float *gt, float lambda,
                       float *out_loss, float *out_l1 /* or NULL */, float *out_ssim /* or NULL */,
                       float *d_pred /* or NULL */, void *workspace, size_t workspace_bytes, void *stream);

/* ---- ViT self-attention, flash-style (csrc/vit_attention.cu; wgmma, TF32 operands, FP32 accumulate) --------
 * The attention of DINO's ViT blocks, softmax(q k^T * scale) v, without any L x L tensor:
 *   qkv  [n_images, tokens, 3 * heads * 64]   "(qkv h d)": DINO's qkv(x).reshape(B, N, 3, H, C // H)
 *   out  [n_images, tokens, heads * 64]       "(h d)": (attn @ v).transpose(1, 2).reshape(B, N, C)
 *   lse  [n_images, heads, tokens]            ln sum_j exp(q_i . k_j * scale), saved for the backward
 * Supported: dim_head == 64, 1 <= tokens <= 16384 (any count, no tile multiple), 1 <= heads <= 16,
 * n_images <= 65535; anything else returns PS_ERR_UNSUPPORTED (counts < 1: PS_ERR_INVALID_ARGUMENT).  qkv, out,
 * d_out and d_qkv must be 16-byte aligned.  No host synchronisation: both calls can be captured in a CUDA graph. */
PS_API int ps_vit_attention_forward(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                    const float *qkv, float scale, float *out, float *lse, void *stream);

/* Bytes of workspace ps_vit_attention_backward needs (D = rowsum(dO o O), n_images * heads * tokens floats). */
PS_API int ps_vit_attention_backward_workspace_bytes(int32_t n_images, int32_t tokens, int32_t heads,
                                                     int32_t dim_head, size_t *out);

/* Backward of the forward above, with P recomputed from lse.  d_qkv has qkv's layout and is fully written; there
 * are no float atomics, so the result is the same bits on every run. */
PS_API int ps_vit_attention_backward(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                     const float *qkv, const float *out, const float *d_out, const float *lse,
                                     float scale, float *d_qkv, void *workspace, size_t workspace_bytes,
                                     void *stream);

/* ---- LPIPS distance head (csrc/lpips.cu)---------------------------------------------------------------------
 * The head of the lpips package's LPIPS(net="vgg") (version 0.1) on up to five feature layers.  For layer l with
 * features x0, x1 [N, C, H, W] (contiguous NCHW) and the 1x1 `lin` weight w [C] (no bias), per image n and pixel p:
 *   f^ = f / (sqrt(sum_c f_c^2) + 1e-10)   (each side),   u = f^0 - f^1,
 *   d_l[n] = (1 / (H W)) sum_p sum_c w_c m_{l,n,c,p} u_c^2,        out[n] = sum_l d_l[n].
 * u is formed from the normalised features directly (never from expanded moment sums), so identical inputs give
 * exactly 0 and a zero gradient.
 * Dropout: m = 1 when dropout_seed is NULL (eval).  Otherwise m = 2 * keep with keep a fair bit, the top bit of
 *   h = mix(key_l + (i + 1) * G),  key_l = mix(seed + (l + 1) * G),  G = 0x9E3779B97F4A7C15,
 * where seed is *dropout_seed read as uint64, i = ((n * C + c) * H + y) * W + x the flat index in the layer, all
 * arithmetic mod 2^64, and mix the splitmix64 finaliser: z ^= z >> 30; z *= 0xBF58476D1CE4E5B9; z ^= z >> 27;
 * z *= 0x94D049BB133111EB; z ^= z >> 31.  The seed is read on the device, so a call can be captured in a graph with
 * the seed drawn inside the capture; the backward recomputes the mask from the same seed.
 * No float atomics: forward and backward give the same bits on every run.  No call synchronises the host.
 * Every entry point rejects n_layers outside [1, 5], N < 1, C outside [1, 8192], H or W < 1, a layer with more
 * than 2^31 - 1 elements, NULL required pointers and a short workspace with PS_ERR_INVALID_ARGUMENT before anything is
 * enqueued. */
#define PS_LPIPS_MAX_LAYERS 5

typedef struct {
    const float *x0, *x1;   /* [N, C, H, W] */
    const float *weight;    /* [C] */
    int32_t C, H, W;
} ps_lpips_layer;

typedef struct {
    int32_t n_layers, N;
    ps_lpips_layer layers[PS_LPIPS_MAX_LAYERS];
    const int64_t *dropout_seed;   /* device pointer to one int64, or NULL: eval mode (no dropout) */
} ps_lpips_desc;

/* Per layer, dL/dx0 and dL/dx1 ([N, C, H, W], fully written: no zero-fill needed).  Either may be NULL, not both. */
typedef struct {
    float *d_x0[PS_LPIPS_MAX_LAYERS];
    float *d_x1[PS_LPIPS_MAX_LAYERS];
} ps_lpips_grads;

PS_API int ps_lpips_workspace_bytes(const ps_lpips_desc *desc, size_t *out);

/* out [N] = sum over layers of d_l.  The workspace (ps_lpips_workspace_bytes) holds per-tile partial sums, which a
 * second kernel adds in a fixed order. */
PS_API int ps_lpips_forward(const ps_lpips_desc *desc, float *out, void *workspace, size_t workspace_bytes,
                            void *stream);

/* Given d_out [N] = dL/dout, writes the gradients of `grads`.  With z_c = 2 k_c u_c, k = w m d_out / (H W) and n the
 * norm of the side's column: d f_j = +-[z_j / (n + eps) - f_j (sum_c z_c f_c) / (n (n + eps)^2)] (+ for x0, - for
 * x1).  At an all-zero column (n = 0) this is the analytic limit +-z_j / eps (the second term is 0), where autograd
 * of the formula gives NaN (sqrt's derivative at 0).  No workspace. */
PS_API int ps_lpips_backward(const ps_lpips_desc *desc, const float *d_out, const ps_lpips_grads *grads,
                             void *stream);

/* ---- Crop shim of the data pipeline (csrc/image_resample.cu) --------------------------------------------------
 * Replaces the reference's per-view host route src/dataset/shims/crop_shim.py (rescale: float -> uint8 -> PIL
 * Image.resize(LANCZOS) -> / 255; center_crop) with the flip of augmentation_shim.py applied first, for a batch of
 * decoded views in one launch:
 *   images [n_images, in_h, in_w, 3] uint8 (HWC, as PIL decodes them)  ->  out [n_images, 3, out_h, out_w] float32.
 * Per image: flip horizontally when flip[i] != 0 (flip NULL: no image is flipped); resample exactly as Pillow's
 * ImagingResample does for 8-bit images (a horizontal pass, then a vertical one, each summing in int32 from 2^21
 * and clipping to uint8, coefficients with 22 fraction bits); keep only the crop; write u / 255.0f.
 * The coefficient tables cover the crop only.  Output column j reads input columns [bounds_h[2j], + bounds_h[2j+1])
 * with weights weights_h[j * taps_h + ...]; output row i reads intermediate rows [bounds_v[2i], + bounds_v[2i+1])
 * with weights_v[i * taps_v + ...].  A pass Pillow skips (its axis keeps its size) is an identity table: taps 1,
 * bounds (crop offset + j, 1), weight 1 << 22.  pixelsplat_b200/data/crop_shim.py builds the tables in float64 on
 * the host, as Pillow does; the kernel clamps each window to the image and never evaluates a filter.
 * All arithmetic after the tables is integer: the same bits as Pillow on every run.  No host synchronisation and
 * no host memory, so a call can be captured in a CUDA graph.  Rejects n_images outside [1, 65535], non-positive
 * sizes, an output larger than the input, taps_h outside [1, in_w] or taps_v outside [1, in_h], and NULL pointers
 * (flip excepted) with PS_ERR_INVALID_ARGUMENT before anything is enqueued. */
typedef struct {
    int32_t n_images, in_h, in_w;
    int32_t out_h, out_w;               /* the crop */
    int32_t taps_h, taps_v;             /* coefficients per output column / row */
    const uint8_t *images;              /* [n_images, in_h, in_w, 3] */
    const uint8_t *flip;                /* [n_images] or NULL */
    const int32_t *bounds_h;            /* [out_w, 2] first input column, count */
    const int32_t *weights_h;           /* [out_w, taps_h] */
    const int32_t *bounds_v;            /* [out_h, 2] first input row, count */
    const int32_t *weights_v;           /* [out_h, taps_v] */
} ps_resample_desc;

PS_API int ps_image_resample(const ps_resample_desc *desc, float *out, void *stream);

/* ---- 8-bit frame pass of an evaluation (csrc/eval_images.cu) ------------------------------------------------------
 * The reference scores 8-bit frames, not float renders: its test step writes each render as a PNG through
 * src/misc/image_io.py's prep_image, (clip(x, 0, 1) * 255).type(uint8), and its metric computer reads the PNGs back
 * through ToTensor (u / 255).  One launch per chunk of up to PS_EVAL_MAX_IMAGES images [n, 3, h, w]:
 *   PS_EVAL_RENDER  render float32 [n, 3, h, w] (CHW): u = the float32 product clip(x, 0, 1) * 255 truncated toward
 *                   zero (prep_image's cast); NaN, which has no defined value there, gives u = 0;
 *   PS_EVAL_FRAME   frame_in uint8 [n, h, w, 3] (HWC): u = the decoded bytes as they are.
 * Outputs, each NULL when not wanted (at least one is required):
 *   frame_out  uint8 [n, h, w, 3]: u, the byte layout PIL.Image.fromarray takes (render mode only);
 *   planes     float32 [n, 3, h, w]: u / 255.0f (what ToTensor gives for the PNG);
 *   sse        float64 [n]: sum over the image's 3 h w values of (u / 255.0f - clip(target, 0, 1))^2 formed in
 *              float64, with target float32 [n, 3, h, w] (torch's clip: NaN stays NaN).  target and sse go together.
 * The sum is formed in a fixed order (per-tile partials in `workspace`, then a finish launch), so the same inputs give
 * the same bits on every run; the workspace (ps_eval_images_workspace_bytes, no initialisation) is needed only with
 * sse.  No host synchronisation (graph-capturable).  Rejects a NULL desc, an unknown mode, n_images outside
 * [1, PS_EVAL_MAX_IMAGES], non-positive sizes, more than 2^31 - 1 values, a missing input or an input of the other
 * mode, no output, frame_out in frame mode, target without sse or sse without target, and a NULL or short workspace
 * with sse, with PS_ERR_INVALID_ARGUMENT before anything is enqueued. */
#define PS_EVAL_RENDER 0
#define PS_EVAL_FRAME 1
#define PS_EVAL_MAX_IMAGES 32

typedef struct {
    int32_t mode;                       /* PS_EVAL_* */
    int32_t n_images, height, width;
    const float *render;                /* [n, 3, h, w] (render mode) or NULL */
    const uint8_t *frame_in;            /* [n, h, w, 3] (frame mode) or NULL */
    const float *target;                /* [n, 3, h, w] or NULL */
    uint8_t *frame_out;                 /* [n, h, w, 3] or NULL */
    float *planes;                      /* [n, 3, h, w] or NULL */
    double *sse;                        /* [n] or NULL */
} ps_eval_desc;

PS_API int ps_eval_images_workspace_bytes(int32_t n_images, int32_t height, int32_t width, size_t *out);
PS_API int ps_eval_images(const ps_eval_desc *desc, void *workspace, size_t workspace_bytes, void *stream);

/* ---- Gradient clipping + Adam over a table of tensors (csrc/optimizer.cu) -----------------------------------------
 * One optimiser step of the reference's training (gradient_clip_val 0.5, optim.Adam without weight decay or amsgrad,
 * LinearLR(1 / W, 1, total_iters = W) stepped once per optimiser step) on float32 tensors, in two launches whatever
 * their number:
 *   norm    total = L2 norm of the tensors' L2 norms (torch's clip_grad_norm_), written to state->grad_norm;
 *   update  coef = min(1, max_norm / (total + 1e-6)), g' = coef g (never written back: the gradients are only read),
 *           t = *state->step + 1, lr_t = lr (1 / W + (1 - 1 / W) min(t - 1, W) / W)  (lr when W = 0),
 *           m += (1 - beta1) (g' - m),  v = beta2 v + (1 - beta2) g'^2,
 *           p -= lr_t / (1 - beta1^t) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps);  then *state->step = t.
 * Everything the step depends on lives on the device (the table, the int64 step counter, the norm), and nothing is
 * read back: the call can be captured in a CUDA graph, and each replay is one more step.  Every sum has a fixed order:
 * equal inputs give equal bits.  A NaN gradient makes the norm, the coefficient and so every parameter NaN, as torch
 * does with error_if_nonfinite=False.  A tensor whose gradient and moments are zero is left bit-unchanged.
 *
 * `segments` is a device array of desc->n_segments rows.  Row i's first_chunk is the sum of
 * ps_clip_adam_segment_chunks(grad, count) over the rows before it, and desc->n_chunks is the sum over all rows (a
 * tensor is cut into chunks of PS_CLIP_ADAM_CHUNK elements on a grid aligned to its gradient's 16-byte boundary).
 * count >= 1 in every row; tensors may start at any 4-byte aligned address.  The rows are trusted.
 * `workspace`: ps_clip_adam_workspace_bytes, 16-byte aligned, zero-filled before the first call and not touched by the
 * caller afterwards.  Rejects NULL pointers, n_segments < 1, n_chunks outside [n_segments, 2^31 - 1], scalars outside
 * lr >= 0, 0 <= beta < 1, eps >= 0, max_norm > 0, warm_up_steps >= 0, and a short or misaligned workspace with
 * PS_ERR_INVALID_ARGUMENT before anything is enqueued. */
#define PS_CLIP_ADAM_CHUNK 4096

typedef struct {
    float *param;
    const float *grad;
    float *exp_avg, *exp_avg_sq;
    int64_t count;                      /* elements, >= 1 */
    int64_t first_chunk;
} ps_clip_adam_segment;

typedef struct {
    int32_t n_segments, reserved;
    int64_t n_chunks;
    int64_t warm_up_steps;              /* W */
    double lr, beta1, beta2, eps, max_norm;
} ps_clip_adam_desc;

typedef struct {
    int64_t *step;                      /* device: optimiser steps taken so far */
    float *grad_norm;                   /* device: the last step's total gradient norm (before clipping) */
} ps_clip_adam_state;

PS_API int64_t ps_clip_adam_segment_chunks(const void *grad, int64_t count);
PS_API int ps_clip_adam_workspace_bytes(const ps_clip_adam_desc *desc, size_t *out);
PS_API int ps_clip_adam_step(const ps_clip_adam_desc *desc, const ps_clip_adam_segment *segments,
                             const ps_clip_adam_state *state, void *workspace, size_t workspace_bytes, void *stream);

/* ---- PLY export: one scene's Gaussians as 3D Gaussian splatting vertex records (csrc/ply_export.cu) ---------------
 * Writes desc->n_gaussians records of little-endian float32, one after the other, to `out` (the bytes that follow a
 * PLY file's ASCII header).  With c = center[0..2] and s = scale[0] (device memory: the median of the means and the
 * 0.95 quantile of the centred means' absolute values, so nothing is read back first) and M = desc->frame
 * (row-major), every record starts x y z = M (mean - c) / s, nx ny nz = 0.
 *   PS_PLY_REFERENCE  17 floats, the reference's export_ply: f_dc_0..2 = harmonics[g, :, 0], opacity = opacities[g]
 *                     raw, scale_0..2 = log(scales[g] / s), rot_0..3 = wxyz of M R(q), q = rotations[g] (xyzw,
 *                     normalised first).  `covariances` is not read; sh_degree must be 0.
 *   PS_PLY_VIEWER     17 + 3 ((sh_degree + 1)^2 - 1) floats: f_dc_c, f_rest_{c ((d+1)^2 - 1) + k - 1} = (T h_c)_k with
 *                     h_c = harmonics[g, c, :(d+1)^2] and T the block-diagonal sh_transform (blocks of degree 0..d,
 *                     row-major, at float offsets 0, 1, 10, 35), opacity = logit(clamp(o, 1e-7, 1 - 1e-7)) in float64,
 *                     and scale / rot from the eigendecomposition of M Sigma M^T / s^2 (cyclic Jacobi in float64 on
 *                     the upper triangle of covariances[g], as the rasterizer reads it): scale_i = log sqrt(max(l_i,
 *                     PS_PLY_MIN_EIGENVALUE)), rot = wxyz of the eigenvector matrix made proper (det +1), w >= 0.
 *                     `scales` and `rotations` are not read.
 * Both modes write rot with w >= 0.  Records are staged in shared memory and stored as 16-byte vectors; offsets are
 * 64-bit.  No host synchronisation.  `harmonics` is [n, 3, sh_coeffs] with sh_coeffs >= (sh_degree + 1)^2, every
 * other input is dense float32; `out` is 16-byte aligned.  Rejects a NULL desc, pointer or input the mode reads,
 * an unknown mode, n_gaussians < 1, sh_degree outside [0, 3] (0 in reference mode), sh_coeffs < (sh_degree + 1)^2
 * and a misaligned `out` with PS_ERR_INVALID_ARGUMENT before anything is enqueued. */
#define PS_PLY_REFERENCE 0
#define PS_PLY_VIEWER 1
#define PS_PLY_SH_TRANSFORM_FLOATS 84   /* 1 + 9 + 25 + 49: degrees 0..3, the most the format holds */
#define PS_PLY_MIN_EIGENVALUE 1e-20

typedef struct {
    int32_t mode;                       /* PS_PLY_* */
    int32_t sh_degree;                  /* of the written record: 0..3 (viewer), 0 (reference) */
    int32_t sh_coeffs;                  /* last dimension of harmonics */
    int32_t reserved;
    int64_t n_gaussians;
    double frame[9];                    /* M, row-major */
    float sh_transform[PS_PLY_SH_TRANSFORM_FLOATS];
    const float *means;                 /* [n, 3] */
    const float *covariances;           /* [n, 3, 3] (viewer) */
    const float *scales;                /* [n, 3] (reference) */
    const float *rotations;             /* [n, 4] xyzw (reference) */
    const float *harmonics;             /* [n, 3, sh_coeffs] */
    const float *opacities;             /* [n] */
    const float *center;                /* [3] */
    const float *scale;                 /* [1] */
} ps_ply_desc;

PS_API int ps_ply_pack(const ps_ply_desc *desc, float *out, void *stream);

/* ---- PLY import: 3D Gaussian splatting vertex records as one scene's Gaussians (csrc/ply_import.cu) --------------
 * Reads desc->n_gaussians records of n_props float32 each (a binary little-endian PLY body, uploaded unchanged) and
 * writes the Gaussians layout.  Every column is given by index, so properties may come in any order and extra
 * properties are ignored.  With the record's x, y, z = p, f_dc_c, f_rest_* (channel-major: f_rest_{c K + k - 1},
 * K = (sh_degree + 1)^2 - 1), opacity o, scale_0..2 = l, rot_0..3 = q (wxyz), and the inverse frame (M = frame,
 * row-major, s = scale, c = center):
 *   means        [n, 3]            M^T p s + c
 *   covariances  [n, 3, 3]         s^2 M^T R(q) diag(exp(2 l)) R(q)^T M, full and symmetric; q is normalised, and a
 *                                  zero quaternion is the identity rotation
 *   harmonics    [n, 3, sh_coeffs] per channel and degree l <= sh_degree, the block of sh_transform (degrees 0..3
 *                                  at float offsets 0, 1, 10, 35, row-major) times the file's coefficients; zero
 *                                  above sh_degree
 *   opacities    [n]               sigmoid(o)
 * All of it in float64, rounded once to float32.  Without a frame, pass M = I, s = 1, c = 0.  One thread per
 * Gaussian, 64 per CTA; each CTA's records are staged in shared memory with 16-byte loads and its outputs stored as
 * 16-byte vectors, every output entry once.  No host synchronisation.  Rejects a NULL desc or pointer,
 * n_gaussians < 1, sh_degree outside [0, 3], sh_coeffs outside [(sh_degree + 1)^2, 25], n_props outside
 * [1, PS_PLY_IMPORT_MAX_PROPERTIES], a column outside [0, n_props) and a pointer that is not 16-byte aligned with
 * PS_ERR_INVALID_ARGUMENT before anything is enqueued. */
#define PS_PLY_IMPORT_MAX_PROPERTIES 512
#define PS_PLY_IMPORT_MAX_COEFFS 25

typedef struct {
    int32_t sh_degree;                  /* of the file: 0..3 */
    int32_t sh_coeffs;                  /* last dimension of harmonics */
    int32_t n_props;                    /* floats per record */
    int32_t reserved;
    int64_t n_gaussians;
    int32_t col_xyz[3];                 /* column of each field in the record */
    int32_t col_dc[3];
    int32_t col_rest[45];               /* f_rest_0..; only the first 3 ((sh_degree + 1)^2 - 1) are read */
    int32_t col_opacity;
    int32_t col_scale[3];
    int32_t col_rot[4];
    int32_t reserved2;
    double frame[9];                    /* M, row-major */
    double center[3];                   /* c */
    double scale;                       /* s */
    float sh_transform[PS_PLY_SH_TRANSFORM_FLOATS];
    const float *records;               /* [n, n_props] */
    float *means;                       /* [n, 3] */
    float *covariances;                 /* [n, 3, 3] */
    float *harmonics;                   /* [n, 3, sh_coeffs] */
    float *opacities;                   /* [n] */
} ps_ply_import_desc;

PS_API int ps_ply_unpack(const ps_ply_import_desc *desc, void *stream);

/* ---- PLY refinement: one Adam step on a scene's vertex records (csrc/ply_import.cu) ---------------------------------
 * One launch per optimisation step over the n = unpack.n_gaussians records [n, n_props] that unpack.records points
 * at, given the gradients of a loss with respect to ps_ply_unpack's outputs for those records (d_means [n, 3],
 * d_covariances [n, 3, 3], d_harmonics [n, 3, sh_coeffs], d_opacities [n]).  Per Gaussian, in float64:
 *   backward   d_p = s M d_mean;  d_l_k = 2 var_k b_k^T dSigma b_k with var_k = s^2 exp(2 l_k) and b = R(q^)^T M (both
 *              halves of an off-diagonal pair count: the unpack writes each twice);  d_q^ = dR/dq^ . (M db^T) with
 *              db_k = 2 var_k (dSigma + dSigma^T)/2 b_k, then d_q = (d_q^ - q^ (q^ . d_q^)) / |q|, and 0 for a zero
 *              quaternion (the unpack's identity rotation does not depend on q);  d_o = d_opacity sigmoid(o)
 *              (1 - sigmoid(o));  f_dc / f_rest: T_l^T d_h per channel and degree l <= sh_degree (coefficients of
 *              d_harmonics above the file's degree are not read).  Rounded once to float32: g.
 *   Adam       torch.optim.Adam's float32 update (no weight decay, no amsgrad) of every column the unpack reads,
 *              with lr[column]: m += (1 - beta1) (g - m), v = beta2 v + (1 - beta2) g^2, p -= lr / (1 - beta1^t)
 *              * m / (sqrt(v) / sqrt(1 - beta2^t) + eps), t = step; the two corrections are formed on the host in
 *              float64 and rounded to float32, as torch rounds its scalars.  Columns the unpack does not read
 *              (normals, other pipelines' fields) have a gradient of exactly 0 and are not updated: the record and
 *              both moments keep their bits.
 *   unpack     the updated record through ps_ply_unpack's own per-record code into unpack.means, .covariances,
 *              .harmonics, .opacities: bit-identical to ps_ply_unpack of records_out.
 * records_out [n, n_props] receives the updated records and may be unpack.records itself (in place); exp_avg and
 * exp_avg_sq [n, n_props] are updated in place; d_records [n, n_props], when not NULL, receives g (0 in the columns
 * the unpack does not read).  Every output entry is written once, nothing past n is touched, there are no atomics
 * (a Gaussian's outputs have one writer: equal inputs give equal bits) and no host synchronisation.  Staging and
 * stores are ps_ply_unpack's.  Rejects what ps_ply_unpack rejects, n_props above PS_PLY_REFINE_MAX_PROPERTIES, a
 * NULL or misaligned records_out, exp_avg, exp_avg_sq or gradient, a misaligned d_records, step < 1, a learning rate
 * of a read column that is negative or not finite, and betas outside [0, 1) or eps < 0 with PS_ERR_INVALID_ARGUMENT
 * before anything is enqueued. */
#define PS_PLY_REFINE_MAX_PROPERTIES 256

typedef struct {
    ps_ply_import_desc unpack;          /* columns, frame, SH blocks, the records read and the Gaussians written */
    int64_t step;                       /* t >= 1: the number of this step (bias corrections) */
    double beta1, beta2, eps;
    double lr[PS_PLY_REFINE_MAX_PROPERTIES];   /* per column; only the columns the unpack reads are used */
    float *records_out;                 /* [n, n_props], may equal unpack.records */
    float *exp_avg, *exp_avg_sq;        /* [n, n_props], in place */
    const float *d_means;               /* [n, 3] */
    const float *d_covariances;         /* [n, 3, 3] */
    const float *d_harmonics;           /* [n, 3, sh_coeffs] */
    const float *d_opacities;           /* [n] */
    float *d_records;                   /* [n, n_props] or NULL */
} ps_ply_refine_desc;

PS_API int ps_ply_refine_step(const ps_ply_refine_desc *desc, void *stream);

/* ---- PLY densification: 3DGS's adaptive density control on a scene's vertex records (csrc/ply_densify.cu) --------
 * Three entry points over the n = n_gaussians records [n, n_props] of a refinement (ps_ply_refine_step's layout):
 *   ps_ply_densify_stats   per Gaussian i, in view order v = 0..n_views-1 where radii[v, i] > 0:
 *                          accum[i] += |d_means2d[v, i, 0:2]| (the norm in float64, rounded once; the sum in float32)
 *                          and count[i] += 1.  d_means2d [n_views, n, 3], radii [n_views, n] int32: the rasterizer's
 *                          screen-space gradient and radii of one call over the views.  One writer per entry.
 *   ps_ply_densify_count   per Gaussian: g = count > 0 ? accum / count : 0 (float32); big = max_k exp(l_k) >
 *                          percent_dense extent (float64); clone = g >= grad_threshold && !big, split = g >=
 *                          grad_threshold && big; prune(o, l) = sigmoid(o) < min_opacity || (prune_world && max_k
 *                          exp(l_k) > 0.1 extent), both in float64.  keep = !split && !prune(o, l); a clone is kept
 *                          when !prune(o, l); both copies of a split are kept when !prune(o, l') with l' the copies'
 *                          float32 log-scales.  Writes the flags and per-CTA segment offsets to the workspace, and
 *                          counts[0..3] = kept originals, kept clones, kept splits (each split gives two rows), n_new.
 *   ps_ply_densify_apply   records_out, exp_avg_out, exp_avg_sq_out [n_new, n_props] from the flags and offsets in
 *                          3DGS's order: kept originals (record and moments copied), clones (record copied, moments
 *                          0), first copies of the splits, second copies (moments 0).  Every segment keeps input order.
 *                          A split's copy k (0, 1) is the record with p' = p + R(q^) (exp(l) * eps[k, i, :]) and
 *                          l' = l - log(1.6), in float64 rounded once (a zero quaternion is the identity); every other
 *                          column is copied bit for bit.  eps [2, n, 3] float32: N(0, 1) draws.
 * count and apply read the same workspace (ps_ply_densify_workspace_bytes(n)); count's counts must be in place when
 * apply runs (stream order).  Nothing past n_new is written, there are no atomics (equal inputs give equal bits) and
 * no host synchronisation.  Rejects a NULL or misaligned pointer (16 bytes for the record arrays, 8 for counts, 4 for
 * the others), n < 1, n_views < 1, n_props outside [1, PS_PLY_REFINE_MAX_PROPERTIES], a column outside [0, n_props),
 * a threshold that is negative or not finite, extent <= 0 and a workspace smaller than the query with
 * PS_ERR_INVALID_ARGUMENT before anything is enqueued. */
typedef struct {
    int64_t n_gaussians;
    int32_t n_props;                    /* floats per record */
    int32_t prune_world;                /* 1: also prune max_k exp(l_k) > 0.1 extent */
    int32_t col_xyz[3];                 /* column of each field in the record */
    int32_t col_opacity;
    int32_t col_scale[3];
    int32_t col_rot[4];                 /* wxyz */
    int32_t reserved;
    double grad_threshold, percent_dense, min_opacity, extent;
} ps_ply_densify_desc;

PS_API int ps_ply_densify_workspace_bytes(int64_t n_gaussians, size_t *bytes);
PS_API int ps_ply_densify_stats(int64_t n_gaussians, int32_t n_views, const float *d_means2d, const int32_t *radii,
                                float *accum, int32_t *count, void *stream);
PS_API int ps_ply_densify_count(const ps_ply_densify_desc *desc, const float *records, const float *accum,
                                const int32_t *count, void *workspace, size_t workspace_bytes, int64_t *counts,
                                void *stream);
PS_API int ps_ply_densify_apply(const ps_ply_densify_desc *desc, const float *records, const float *exp_avg,
                                const float *exp_avg_sq, const float *eps, const void *workspace,
                                size_t workspace_bytes, const int64_t *counts, float *records_out,
                                float *exp_avg_out, float *exp_avg_sq_out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* PIXELSPLAT_B200_H */
