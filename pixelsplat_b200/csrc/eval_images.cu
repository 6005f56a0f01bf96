// The 8-bit frame pass of an evaluation (the reference's ModelWrapper.test_step writes every render as a PNG through
// src/misc/image_io.py's prep_image, (clip(x, 0, 1) * 255).type(uint8), and MetricComputer reads the PNGs back
// through ToTensor, u / 255): per chunk of up to PS_EVAL_MAX_IMAGES images, in one launch,
//   render mode  x float32 [n, 3, h, w] -> u = trunc(clip(x, 0, 1) * 255) (the float32 product; NaN -> 0),
//   frame mode   u uint8 [n, h, w, 3] (decoded PNG bytes),
// then the uint8 HWC frame (render mode), the float32 planes u / 255.0f and, per image, the double sum of
// (u / 255.0f - clip(target, 0, 1))^2 over its 3 h w values.
//
// One CTA per (image, tile of kEvTilePix pixels); each thread walks its pixels in a fixed order, the CTA reduces in a
// fixed tree and writes one partial to the workspace, and a finish kernel adds an image's partials in a fixed order.
// No float atomics: the same inputs give the same bits on every run.
#include "ps_common.cuh"

namespace ps {

constexpr int kEvThreads = 256;
constexpr int kEvTilePix = kEvThreads * 8;   // pixels per CTA

// prep_image's quantisation: clip to [0, 1] (NaN stays NaN in torch's clip), times 255 in float32, truncated toward
// zero by the cast.  NaN has no defined uint8 value there; it maps to 0 here.
__device__ __forceinline__ uint32_t quantise(float x) {
    if (!(x == x)) return 0u;
    const float c = x < 0.0f ? 0.0f : (x > 1.0f ? 1.0f : x);
    return (uint32_t)__fmul_rn(c, 255.0f);
}

// torch's clip(min=0, max=1): NaN propagates.
__device__ __forceinline__ float clip01(float t) { return t < 0.0f ? 0.0f : (t > 1.0f ? 1.0f : t); }

template <int MODE>
__global__ void __launch_bounds__(kEvThreads) k_eval_images(ps_eval_desc d, double *__restrict__ partial) {
    __shared__ double red[kEvThreads / 32];
    const int n = blockIdx.y;
    const long long hw = (long long)d.height * d.width;
    const long long p0 = (long long)blockIdx.x * kEvTilePix, p1 = min(hw, p0 + kEvTilePix);
    const size_t img = (size_t)n * 3 * hw;
    double acc = 0.0;
    for (long long p = p0 + threadIdx.x; p < p1; p += kEvThreads) {
        uint32_t u[3];
        if (MODE == PS_EVAL_RENDER) {
#pragma unroll
            for (int c = 0; c < 3; ++c) u[c] = quantise(__ldg(d.render + img + c * hw + p));
            if (d.frame_out) {
                uint8_t *o = d.frame_out + img + 3 * p;
                o[0] = (uint8_t)u[0];
                o[1] = (uint8_t)u[1];
                o[2] = (uint8_t)u[2];
            }
        } else {
            const uint8_t *f = d.frame_in + img + 3 * p;
#pragma unroll
            for (int c = 0; c < 3; ++c) u[c] = __ldg(f + c);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float v = (float)u[c] / 255.0f;
            if (d.planes) d.planes[img + c * hw + p] = v;
            if (d.target) {
                const double e = (double)v - (double)clip01(__ldg(d.target + img + c * hw + p));
                acc = fma(e, e, acc);
            }
        }
    }
    if (!d.target) return;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kEvThreads / 32; ++w) s += red[w];
        partial[(size_t)n * gridDim.x + blockIdx.x] = s;
    }
}

// One warp per image: its partials in a fixed order.
__global__ void k_eval_finish(int tiles, const double *__restrict__ partial, double *__restrict__ sse) {
    const double *p = partial + (size_t)blockIdx.x * tiles;
    double s = 0.0;
    for (int t = threadIdx.x; t < tiles; t += 32) s += p[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) sse[blockIdx.x] = s;
}

static int eval_tiles(int h, int w) { return (int)(((long long)h * w + kEvTilePix - 1) / kEvTilePix); }

static size_t eval_workspace(int n, int h, int w) {
    return ((size_t)n * eval_tiles(h, w) * sizeof(double) + 255) / 256 * 256;
}

static int check_eval_shape(const char *who, int n, int h, int w) {
    if (n < 1 || n > PS_EVAL_MAX_IMAGES || h < 1 || w < 1) {
        set_error("%s: bad shape (n_images %d, %d x %d): need 1 <= n_images <= %d and positive sizes", who, n, h, w,
                  PS_EVAL_MAX_IMAGES);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if ((long long)n * 3 * h * w > 0x7fffffffLL) {
        set_error("%s: %d images of %d x %d are too large for one call", who, n, h, w);
        return PS_ERR_INVALID_ARGUMENT;
    }
    return PS_OK;
}

static int check_eval(const ps_eval_desc *d, const void *workspace, size_t workspace_bytes) {
    if (!d) {
        set_error("ps_eval_images: desc is NULL");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->mode != PS_EVAL_RENDER && d->mode != PS_EVAL_FRAME) {
        set_error("ps_eval_images: unknown mode %d", d->mode);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const int rc = check_eval_shape("ps_eval_images", d->n_images, d->height, d->width);
    if (rc != PS_OK) return rc;
    if (d->mode == PS_EVAL_RENDER ? (!d->render || d->frame_in) : (!d->frame_in || d->render || d->frame_out)) {
        set_error("ps_eval_images: %s mode takes %s", d->mode == PS_EVAL_RENDER ? "render" : "frame",
                  d->mode == PS_EVAL_RENDER ? "`render` and no `frame_in`"
                                            : "`frame_in` and neither `render` nor `frame_out`");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (!d->frame_out && !d->planes && !d->sse) {
        set_error("ps_eval_images: no output requested");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (!d->target != !d->sse) {
        set_error("ps_eval_images: `target` and `sse` go together");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->sse) {
        const size_t need = eval_workspace(d->n_images, d->height, d->width);
        if (!workspace || workspace_bytes < need) {
            set_error("ps_eval_images: workspace of %zu bytes, %zu needed", workspace ? workspace_bytes : 0, need);
            return PS_ERR_INVALID_ARGUMENT;
        }
    }
    return PS_OK;
}

}  // namespace ps

extern "C" PS_API int ps_eval_images_workspace_bytes(int32_t n_images, int32_t height, int32_t width, size_t *out) {
    const int rc = ps::check_eval_shape("ps_eval_images_workspace_bytes", n_images, height, width);
    if (rc != PS_OK) return rc;
    if (!out) {
        ps::set_error("ps_eval_images_workspace_bytes: out is NULL");
        return PS_ERR_INVALID_ARGUMENT;
    }
    *out = ps::eval_workspace(n_images, height, width);
    return PS_OK;
}

extern "C" PS_API int ps_eval_images(const ps_eval_desc *desc, void *workspace, size_t workspace_bytes,
                                     void *stream) {
    const int rc = ps::check_eval(desc, workspace, workspace_bytes);
    if (rc != PS_OK) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int tiles = ps::eval_tiles(desc->height, desc->width);
    double *partial = static_cast<double *>(workspace);
    const dim3 grid(tiles, desc->n_images);
    if (desc->mode == PS_EVAL_RENDER)
        ps::k_eval_images<PS_EVAL_RENDER><<<grid, ps::kEvThreads, 0, st>>>(*desc, partial);
    else
        ps::k_eval_images<PS_EVAL_FRAME><<<grid, ps::kEvThreads, 0, st>>>(*desc, partial);
    PS_LAUNCH_CHECK("k_eval_images");
    if (desc->sse) {
        ps::k_eval_finish<<<desc->n_images, 32, 0, st>>>(tiles, partial, desc->sse);
        PS_LAUNCH_CHECK("k_eval_finish");
    }
    return PS_OK;
}
