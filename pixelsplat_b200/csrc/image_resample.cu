// The crop shim of the reference's data pipeline on the device (src/dataset/shims/crop_shim.py, with the flip of
// src/dataset/shims/augmentation_shim.py): per image, an optional horizontal flip, Pillow's 8-bit LANCZOS resample
// (Image.resize(..., Image.LANCZOS), libImaging/Resample.c), the centre crop and the conversion u / 255 to float32.
//
// Pillow's resample is two separable integer passes over uint8 images, horizontal then vertical:
//   h[y][c] = clip8(2^21 + sum_x in[y][xmin_c + x] * kh[c][x]),   out[r][c] = clip8(2^21 + sum_y h[ymin_r + y][c] * kv[r][y])
// with clip8(s) = s >> 22 clamped to [0, 255] and kh / kv Pillow's fixed-point coefficients (PRECISION_BITS = 22).
// The caller supplies both coefficient tables already restricted to the crop (pixelsplat_b200/data/crop_shim.py
// builds them on the host in float64, as Pillow does); a pass Pillow skips has an identity table (one tap, 2^22),
// which reproduces Pillow's copy.  Every step after the tables is integer arithmetic, so the output has the same
// bits as Pillow's on every run, and the order in which the sums are formed does not matter.
//
// One CTA per (image, 16 x 32 output tile).  The intermediate rows a tile needs are produced in chunks of kChunk
// rows into shared memory (horizontal pass), and each thread adds a chunk's rows into the int32 sums of its two
// output pixels (vertical pass).  Only input rows some output row of the tile reads are touched.
#include "ps_common.cuh"

namespace ps {

constexpr int kRsThreads = 256;
constexpr int kRsTH = 16, kRsTW = 32;              // output tile: rows x columns
constexpr int kRsPix = kRsTH * kRsTW / kRsThreads;  // output pixels per thread
constexpr int kChunk = 64;                          // intermediate rows per shared-memory chunk
constexpr int kPrecisionBits = 22;

// Pillow's clip8: s >> 22 clamped to [0, 255].
__device__ __forceinline__ uint32_t clip8(int32_t s) {
    return s <= 0 ? 0u : (s >= (1 << (kPrecisionBits + 8)) ? 255u : (uint32_t)s >> kPrecisionBits);
}

// A table row's window, clamped to the image so that no table can make the kernel read outside it.
__device__ __forceinline__ int2 window(const int32_t *__restrict__ bounds, int i, int taps, int size) {
    const int cnt = min(max(__ldg(bounds + 2 * i + 1), 0), taps);
    const int lo = min(max(__ldg(bounds + 2 * i), 0), size - cnt);
    return make_int2(lo, cnt);
}

__global__ void __launch_bounds__(kRsThreads) k_image_resample(ps_resample_desc d, float *__restrict__ out) {
    __shared__ uint8_t tmp[kChunk * kRsTW * 3];
    __shared__ int span[2];
    const int n = blockIdx.z, r0 = blockIdx.y * kRsTH, c0 = blockIdx.x * kRsTW;
    const int rows = min(kRsTH, d.out_h - r0);
    if (threadIdx.x == 0) {
        int lo = d.in_h, hi = 0;
        for (int r = 0; r < rows; ++r) {
            const int2 w = window(d.bounds_v, r0 + r, d.taps_v, d.in_h);
            lo = min(lo, w.x);
            hi = max(hi, w.x + w.y);
        }
        span[0] = lo;
        span[1] = hi;
    }
    const bool flip = d.flip && d.flip[n];
    const uint8_t *img = d.images + (size_t)n * d.in_h * d.in_w * 3;

    int32_t acc[kRsPix][3];
    int2 vw[kRsPix];
#pragma unroll
    for (int k = 0; k < kRsPix; ++k) {
        acc[k][0] = acc[k][1] = acc[k][2] = 1 << (kPrecisionBits - 1);
        const int r = (threadIdx.x + k * kRsThreads) / kRsTW;
        vw[k] = r < rows ? window(d.bounds_v, r0 + r, d.taps_v, d.in_h) : make_int2(0, 0);
    }
    __syncthreads();
    const int y_lo = span[0], y_hi = span[1];

    for (int y0 = y_lo; y0 < y_hi; y0 += kChunk) {
        const int ch = min(kChunk, y_hi - y0);
        // horizontal pass of intermediate rows [y0, y0 + ch) for the tile's columns
        for (int i = threadIdx.x; i < ch * kRsTW; i += kRsThreads) {
            const int yy = i / kRsTW, c = i % kRsTW;
            if (c0 + c >= d.out_w) continue;
            const int2 w = window(d.bounds_h, c0 + c, d.taps_h, d.in_w);
            const int32_t *kh = d.weights_h + (size_t)(c0 + c) * d.taps_h;
            const uint8_t *row = img + (size_t)(y0 + yy) * d.in_w * 3;
            int32_t s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
            for (int x = 0; x < w.y; ++x) {
                const int xi = flip ? d.in_w - 1 - (w.x + x) : w.x + x;
                const int32_t k = __ldg(kh + x);
                s0 += (int32_t)__ldg(row + 3 * xi) * k;
                s1 += (int32_t)__ldg(row + 3 * xi + 1) * k;
                s2 += (int32_t)__ldg(row + 3 * xi + 2) * k;
            }
            uint8_t *t = tmp + i * 3;
            t[0] = (uint8_t)clip8(s0);
            t[1] = (uint8_t)clip8(s1);
            t[2] = (uint8_t)clip8(s2);
        }
        __syncthreads();
        // vertical pass: the chunk's rows that fall in each of this thread's output windows
#pragma unroll
        for (int k = 0; k < kRsPix; ++k) {
            const int p = threadIdx.x + k * kRsThreads, r = p / kRsTW, c = p % kRsTW;
            const int lo = max(vw[k].x, y0), hi = min(vw[k].x + vw[k].y, y0 + ch);
            const int32_t *kv = d.weights_v + (size_t)(r0 + r) * d.taps_v - vw[k].x;
            for (int y = lo; y < hi; ++y) {
                const int32_t w = __ldg(kv + y);
                const uint8_t *t = tmp + ((y - y0) * kRsTW + c) * 3;
                acc[k][0] += (int32_t)t[0] * w;
                acc[k][1] += (int32_t)t[1] * w;
                acc[k][2] += (int32_t)t[2] * w;
            }
        }
        __syncthreads();
    }

    const size_t plane = (size_t)d.out_h * d.out_w;
    float *o = out + (size_t)n * 3 * plane;
#pragma unroll
    for (int k = 0; k < kRsPix; ++k) {
        const int p = threadIdx.x + k * kRsThreads, r = p / kRsTW, c = p % kRsTW;
        if (r >= rows || c0 + c >= d.out_w) continue;
        const size_t q = (size_t)(r0 + r) * d.out_w + c0 + c;
#pragma unroll
        for (int j = 0; j < 3; ++j) o[j * plane + q] = (float)clip8(acc[k][j]) / 255.0f;
    }
}

static int check_resample(const ps_resample_desc *d) {
    if (!d) {
        set_error("ps_image_resample: desc is NULL");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->n_images < 1 || d->n_images > 65535 || d->in_h < 1 || d->in_w < 1 || d->out_h < 1 || d->out_w < 1) {
        set_error("ps_image_resample: bad shape (n_images %d, in %d x %d, out %d x %d): need 1 <= n_images <= 65535 "
                  "and positive sizes", d->n_images, d->in_h, d->in_w, d->out_h, d->out_w);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->out_h > d->in_h || d->out_w > d->in_w) {
        set_error("ps_image_resample: output %d x %d is larger than the input %d x %d", d->out_h, d->out_w, d->in_h,
                  d->in_w);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if ((long long)d->in_h * d->in_w * 3 > 0x7fffffffLL) {
        set_error("ps_image_resample: input image of %d x %d is too large", d->in_h, d->in_w);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->taps_h < 1 || d->taps_h > d->in_w || d->taps_v < 1 || d->taps_v > d->in_h) {
        set_error("ps_image_resample: table sizes do not match the image: taps_h %d (need 1..%d), taps_v %d "
                  "(need 1..%d)", d->taps_h, d->in_w, d->taps_v, d->in_h);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (!d->images || !d->bounds_h || !d->weights_h || !d->bounds_v || !d->weights_v) {
        set_error("ps_image_resample: NULL pointer");
        return PS_ERR_INVALID_ARGUMENT;
    }
    return PS_OK;
}

}  // namespace ps

extern "C" PS_API int ps_image_resample(const ps_resample_desc *desc, float *out, void *stream) {
    const int rc = ps::check_resample(desc);
    if (rc != PS_OK) return rc;
    if (!out) {
        ps::set_error("ps_image_resample: out is NULL");
        return PS_ERR_INVALID_ARGUMENT;
    }
    const dim3 grid((desc->out_w + ps::kRsTW - 1) / ps::kRsTW, (desc->out_h + ps::kRsTH - 1) / ps::kRsTH,
                    desc->n_images);
    ps::k_image_resample<<<grid, ps::kRsThreads, 0, static_cast<cudaStream_t>(stream)>>>(*desc, out);
    PS_LAUNCH_CHECK("k_image_resample");
    return PS_OK;
}
