// Shared declarations of the rasterizer kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pixelsplat_b200.h"

namespace ps {

constexpr int kTile = PS_TILE;
constexpr int kTilePixels = kTile * kTile;

// Resolved device views of the workspace (host-built, passed by value to kernels).
struct Geom {
    float *depth;
    int32_t *radii;
    float2 *xy;
    float4 *conic_opacity;
    float4 *rgb;
    ushort4 *rect;
    uint8_t *clamped;
    uint32_t *tile_count;
    uint32_t *tile_start;
    uint32_t *tile_cursor;
    long long *n_instances;   // [0] instances, [1] longest segment, [2] #vis_pairs, [3] unused (0)
    uint32_t *vis_pairs;      // compact list of (view, Gaussian) flat indices that are on screen
    float4 *cull;             // xy + half-extents of the alpha >= 1/255 box (compositor's cull record)
    float4 *sh_jac;           // [S*V*P][3] (M > 0, else null): d(colour channel before the clamp) / d(direction)
};

// Per-view image-space state kept from forward to backward.
struct ImageState {
    float *final_T;           // [S*V*H*W]
    uint32_t *n_contrib;      // [S*V*H*W]
    float *color;             // [S*V*3*H*W] copy of the rendered colour (backward's forward-order prefix form)
    float4 *run_state;        // [S*V*(kMaxSegments-1)*H*W] (T, Cr, Cg, Cb) in front of list runs 1.. (segK > 1)
    float *depth_image;       // [S*V*H*W] composited depth channel (depth_mode != 0, else null)
    float *run_depth;         // [S*V*(kMaxSegments-1)*H*W] depth in front of list runs 1.. (depth_mode != 0)
};

// Fused loss epilogue of the compositor (SURVEY.md 8 row f-4): squared error against a target image summed per
// view in the forward, dL/dC = grad_scale[view] (C - target) formed inside the backward.  All null = off.
constexpr int kLossSlots = PS_LOSS_SLOTS;
struct LossEpilogue {
    const float *target;       // [S*V, 3, H, W]
    float *sums;               // forward: [S*V, 2, kLossSlots] partial sums (raw, clipped), zeroed by the caller
    const float *grad_scale;   // backward: [S*V]
};

constexpr int kMaxSegments = 4;   // list runs per warp task (raster_composite2.cu)

// The composite forward's per-(tile, block, run) hit lists, kept for the backward (binning state).  Run k of block
// `sub` of tile segment `seg` owns hits[(tile_start[seg] * 8 + sub * tile_count[seg]) + run_begin ...] (a run cannot
// have more hits than entries), its length is run_hits[(seg * 8 + sub) * kMaxSegments + k].
struct HitLists {
    uint2 *hits;              // (list position, Gaussian id)
    uint32_t *run_hits;
};

struct Dims {
    int S, V, P, M, deg, sh_layout, cov_layout, H, W, gx, gy, tiles, sh_basis, segK, hit_lists;
    int depth_mode;           // PS_DEPTH_*; in a backward, 0 unless a depth gradient is given
    long long capacity;
};

struct Inputs {
    const float *means, *cov, *opac, *sh, *view, *proj, *campos, *tanfov, *bg, *scale;
    const float *near_far;    // [S*V, 2] world units (depth modes 3, 4)
};

// The Gaussian-side outputs of ps_raster_grads, as the preprocess backward receives them.
struct GaussGrads {
    float *d_means, *d_cov, *d_opacities, *d_sh, *d_means2d;
};

// Camera gradients (ps_raster_camera_grads): 29 used entries per partial row, rows of 32 floats, at most
// (P - 1) / 32 + 2 warps of 32 consecutive (scene, Gaussian) indices overlap one scene's P Gaussians.
constexpr int kCamEntries = 29, kCamRowFloats = 32;
__host__ __device__ __forceinline__ int cam_rows_per_view(int P) { return (P - 1) / 32 + 2; }

// Per-(view,Gaussian) gradient scratch written by the composite backward.
struct ViewGrads {
    float2 *d_mean2d;  // NDC-scaled like upstream (x * 0.5 W, y * 0.5 H)
    float4 *d_conic;   // x, y (half-weighted B), z, w = d_opacity
    float4 *d_color;   // r, g, b, depth value d (the latter only with a depth gradient)
};

// Depth channel (PS_DEPTH_*): the value d composited for a Gaussian at view-space depth vz of a view whose
// scene_scale is `sc` (null scale = 1).  z = vz / sc is the depth in world units.  Compiled into the preprocess
// (--fmad=false, both producers of d give the same bits) and the preprocess backward (depth_value_grad).
constexpr float kDepthEps = 1e-10f;

__device__ __forceinline__ float depth_value(int mode, float vz, const float *scale, const float *near_far, int vid) {
    const float z = scale ? vz / scale[vid] : vz;
    if (mode == PS_DEPTH_DISPARITY) return 1.0f / z;
    if (mode == PS_DEPTH_RELATIVE_DISPARITY) {
        const float dn = 1.0f / (near_far[2 * vid] + kDepthEps), df = 1.0f / (near_far[2 * vid + 1] + kDepthEps);
        return 1.0f - (1.0f / (z + kDepthEps) - df) / (dn - df + kDepthEps);
    }
    if (mode == PS_DEPTH_LOG) return logf(fmaxf(fminf(z, near_far[2 * vid]), near_far[2 * vid + 1]));
    return z;
}

// dd/dz of depth_value.  The log mode follows torch's minimum / maximum backward (a tie splits the gradient in
// half): for near < far, max(min(z, near), far) = far and the derivative is 0, as in the reference.
__device__ __forceinline__ float depth_value_grad(int mode, float vz, const float *scale, const float *near_far, int vid) {
    const float z = scale ? vz / scale[vid] : vz;
    if (mode == PS_DEPTH_DISPARITY) return -1.0f / (z * z);
    if (mode == PS_DEPTH_RELATIVE_DISPARITY) {
        const float dn = 1.0f / (near_far[2 * vid] + kDepthEps), df = 1.0f / (near_far[2 * vid + 1] + kDepthEps);
        const float iz = 1.0f / (z + kDepthEps);
        return iz * iz / (dn - df + kDepthEps);
    }
    if (mode == PS_DEPTH_LOG) {
        const float nr = near_far[2 * vid], fr = near_far[2 * vid + 1];
        const float m = fminf(z, nr);
        const float gm = z < nr ? 1.0f : (z == nr ? 0.5f : 0.0f);
        const float gr = m > fr ? 1.0f : (m == fr ? 0.5f : 0.0f);
        return gm * gr / fmaxf(m, fr);
    }
    return 1.0f;
}

// Half-extents (pixels) of the axis-aligned box outside of which a splat's alpha is certainly
// < 1/255: alpha = o exp(-0.5 d^T Sigma^-1 d) >= 1/255  <=>  d^T Sigma^-1 d <= 2 ln(255 o), whose bounding
// box is sqrt(2 ln(255 o) Sigma_ii) -- taken from the 2D covariance itself (a, c = its diagonal), so no
// cancellation; the margins cover the compositor's approximate exp2 and the rounding of the conic.
// Large negative = never contributes; large positive = always evaluated (NaN inputs then propagate into
// the image exactly as they would upstream).
__device__ __forceinline__ float2 cull_extent(float a, float c, float o) {
    if (!(a > 0.0f) || !(c > 0.0f) || !(o <= 3.0e38f)) return make_float2(3.0e38f, 3.0e38f);
    if (!(o * 255.0f >= 1.0f - 1e-3f)) return make_float2(-3.0e38f, -3.0e38f);
    const float tau2 = 2.0f * (__logf(fmaxf(o * 255.0f, 1.0f)) + 0.01f);
    return make_float2(sqrtf(tau2 * a) * 1.001f + 0.01f, sqrtf(tau2 * c) * 1.001f + 0.01f);
}

// Per-tile LIVE LISTS (written by the tile sort, walked by the warp-task compositor).  After a (view, tile) segment
// is sorted, its entries whose cull box meets at least one of the tile's eight 8x4 pixel blocks are compacted, in
// list order, into uint2 records (position in the tile's list << 8 | block mask, Gaussian id) at the segment's
// tile_start offset of keys_alt; tile_cursor[segment] holds how many there are.  Block b of a tile covers pixels
// x0 + (b & 1) * 8 + 0..7, y0 + (b >> 1) * 4 + 0..3.  A segment longer than kLivePosLimit (positions no longer fit
// in 24 bits) keeps every entry, so that there the position of a record is its index in the live list.
constexpr uint32_t kLivePosLimit = 1u << 24;

// Bit b set = the cull record's box meets block b of the tile whose top-left pixel is (x0, y0).  The test (and its
// float arithmetic) is the one the compositor applied per block before the live lists: alpha >= 1/255 somewhere in
// the block's rectangle [rx0, rx0 + 7] x [ry0, ry0 + 3] is possible only if the box overlaps it.
__device__ __forceinline__ uint32_t tile_block_mask(const float4 &cr, int x0, int y0) {
    const float xl = cr.x - cr.z, xh = cr.x + cr.z, yl = cr.y - cr.w, yh = cr.y + cr.w;
    uint32_t xm = 0, m = 0;
#pragma unroll
    for (int bx = 0; bx < 2; ++bx)
        xm |= ((xh >= (float)(x0 + 8 * bx)) && (xl <= (float)(x0 + 8 * bx + 7))) ? 1u << bx : 0u;
#pragma unroll
    for (int by = 0; by < 4; ++by)
        m |= ((yh >= (float)(y0 + 4 * by)) && (yl <= (float)(y0 + 4 * by + 3))) ? xm << (2 * by) : 0u;
    return m;
}

void set_error(const char *fmt, ...);

// Optional per-stage device timing (bench.py's roofline leg): when enabled, the entry points
// record CUDA events on the launching stream between stages.
enum Mark { kMarkFwdStart = 0, kMarkPreprocess, kMarkScatter, kMarkSort, kMarkCompositeFwd,
            kMarkBwdStart, kMarkBwdZero, kMarkCompositeBwd, kMarkPreprocessBwd, kNumMarks };
void mark(int id, cudaStream_t st);
void count_launch();

// Once-per-DEVICE flags (a host process may drive several GPUs; kernel attributes and the library's
// side stream are per device).  `mask` is a caller-owned static, one bit per device ordinal.
// Thread-safe: the test-and-set happens under a process-wide mutex (the caller then sets a kernel attribute,
// which is idempotent, so a second thread racing past the flag at worst repeats it).
bool first_use_on_device(unsigned long long &mask);

#define PS_CUDA_CHECK(expr)                                                              \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            ps::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return PS_ERR_CUDA;                                                          \
        }                                                                                \
    } while (0)

#define PS_LAUNCH_CHECK(name)                                                            \
    do {                                                                                 \
        cudaError_t _e = cudaGetLastError();                                             \
        if (_e != cudaSuccess) {                                                         \
            ps::set_error("launch of %s failed: %s", name, cudaGetErrorString(_e));      \
            return PS_ERR_CUDA;                                                          \
        }                                                                                \
        ps::count_launch();                                                              \
    } while (0)

// stage launchers (each returns PS_OK / PS_ERR_*)
int launch_preprocess(const Dims &d, const Inputs &in, const Geom &g, cudaStream_t st);
int launch_sh_color(const Dims &d, const Inputs &in, const Geom &g, cudaStream_t st);
// `scanned` (may be null) is recorded on `st` once the scan has written the instance count and the longest segment.
int launch_binning(const Dims &d, const Geom &g, unsigned long long *keys,
                   unsigned long long *keys_alt, int sort_impl, int segment_hint, cudaEvent_t scanned,
                   cudaStream_t st);
// Deterministic mode (ps_set_option "deterministic"): the forward's loss epilogue goes through loss_partials
// ([S*V*tiles*8] float2 per-task (sse, sse_clipped), image state) and a fixed-order finish; the backward stores into
// `records` (the per-(tile block, list position) gradients, 8 x instance_capacity entries of each array, backward
// scratch) and gathers them into vg in a fixed order.  Null = the default float-atomic path.
// `live`: the tile sort's live lists (keys_alt, see kLivePosLimit); `keys`: the sorted segments.
int launch_composite_forward(const Dims &d, const Inputs &in, const Geom &g,
                             const unsigned long long *keys, const uint2 *live, const ImageState &img,
                             float *out_color, const LossEpilogue &loss, const HitLists &hl, float *loss_partials,
                             cudaStream_t st);
int launch_composite_backward(const Dims &d, const Inputs &in, const Geom &g,
                              const unsigned long long *keys, const uint2 *live, const ImageState &img,
                              const float *d_color, const float *d_depth, const ViewGrads &vg,
                              const ViewGrads *records, const LossEpilogue &loss, const HitLists &hl,
                              cudaStream_t st);
// legacy CTA-per-tile compositor (round 1), kept selectable for A/B measurements
int launch_composite_forward_v1(const Dims &d, const Inputs &in, const Geom &g,
                                const unsigned long long *keys, const ImageState &img,
                                float *out_color, cudaStream_t st);
int launch_composite_backward_v1(const Dims &d, const Inputs &in, const Geom &g,
                                 const unsigned long long *keys, const ImageState &img,
                                 const float *d_color, const ViewGrads &vg, cudaStream_t st);
int composite_impl();   // 1 = legacy, 2 = warp-task compositor (env PIXELSPLAT_B200_COMPOSITE, default 2)
int set_composite_option(int which, int value);   // 0: impl (1 | 2), 1: segments (0 = auto | 1 | 2 | 4),
                                                  // 2: hit lists (0 = never | 1 = always | 2 = auto)
int get_composite_option(int which);              // the value in force (environment included)
int composite_segments(long long tasks);
bool composite_hit_lists(long long capacity);      // keep the forward's hit lists for the backward?
// With grads.camera set, the camera-gradient instantiation runs and a finish kernel writes the camera gradients.
int launch_preprocess_backward(const Dims &d, const Inputs &in, const Geom &g, const ViewGrads &vg,
                               const ps_raster_grads &grads, cudaStream_t st);
// Clears the gradient scratch rows of the on-screen (view, Gaussian) pairs: the only rows the composite backward
// writes and the preprocess backward reads.
int launch_clear_pair_grads(const Dims &d, const Geom &g, const ViewGrads &vg, cudaStream_t st);

}  // namespace ps
