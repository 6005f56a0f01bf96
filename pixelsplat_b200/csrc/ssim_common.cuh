// The SSIM building blocks shared by csrc/ssim.cu (the evaluation's skimage SSIM) and csrc/l1_dssim.cu (3DGS's
// training SSIM): the 11x11 Gaussian window, the staging of a shifted plane region, the separable passes of the
// five moments and the per-pixel SSIM terms.
//
// Numerics: the second moments are formed of values shifted by one pixel of the tile (x - kx, y - ky).  Variance
// and covariance do not change under the shift and the means get it back, but G*x^2 - mu^2 no longer cancels two
// numbers near 1 on a bright, flat patch (0.95 +- 0.002 would lose ~4 % of the variance otherwise).
#pragma once

#include "ps_common.cuh"

namespace ps {

constexpr int kR = 5;                        // window radius: int(3.5 * 1.5 + 0.5)
constexpr int kWin = 2 * kR + 1;
constexpr float kC1 = 1e-4f;                 // (0.01 * data_range)^2
constexpr float kC2 = 9e-4f;                 // (0.03 * data_range)^2
constexpr int kThreads = 256;
constexpr int kTH = 16, kTW = 32;            // output tile: rows x columns

// exp(-k^2 / (2 1.5^2)) normalised to sum 1, k = -5..5 (scipy.ndimage's kernel for sigma 1.5, truncate 3.5; also
// 3DGS's create_window(11, C), whose taps are the same)
__constant__ float kSsimG[kWin] = {1.028380084e-03f, 7.598758135e-03f, 3.600077213e-02f, 1.093606895e-01f,
                                   2.130055377e-01f, 2.660117249e-01f, 2.130055377e-01f, 1.093606895e-01f,
                                   3.600077213e-02f, 7.598758135e-03f, 1.028380084e-03f};

// Filtered moments at one pixel, of the shifted values x' = x - kx, y' = y - ky.
struct Moments {
    float mx, my;   // G*x', G*y'
    float xx, yy, xy;
};

struct Ssim {
    float mux, muy, S, A1, A2, B1, B2;
};

// `cov` scales the (co)variances: 121/120 for a sample covariance, 1 for a population one.
__device__ __forceinline__ Ssim ssim_at(const Moments &m, float kx, float ky, float cov) {
    Ssim r;
    const float vx = cov * (m.xx - m.mx * m.mx);
    const float vy = cov * (m.yy - m.my * m.my);
    const float cxy = cov * (m.xy - m.mx * m.my);
    r.mux = m.mx + kx;
    r.muy = m.my + ky;
    r.A1 = 2.0f * r.mux * r.muy + kC1;
    r.A2 = 2.0f * cxy + kC2;
    r.B1 = __fadd_rn(__fmul_rn(r.mux, r.mux), __fmul_rn(r.muy, r.muy)) + kC1;   // no FMA: symmetric in x, y
    r.B2 = vx + vy + kC2;
    r.S = (r.A1 * r.A2) / (r.B1 * r.B2);
    return r;
}

// Loads rows [r0, r0 + rows) x columns [c0, c0 + cols) of a plane, shifted, into shared memory.  Outside the image
// the stored value is 0, or with ZERO_PAD the shifted zero (-kx, -ky): the plane padded with zeros.
template <bool ZERO_PAD = false>
__device__ __forceinline__ void stage(const float *__restrict__ x, const float *__restrict__ y, int H, int W,
                                      int r0, int c0, int rows, int cols, float kx, float ky, float *sx, float *sy) {
    for (int i = threadIdx.x; i < rows * cols; i += kThreads) {
        const int r = r0 + i / cols, c = c0 + i % cols;
        const bool in = r >= 0 && r < H && c >= 0 && c < W;
        sx[i] = in ? __ldg(x + (size_t)r * W + c) - kx : (ZERO_PAD ? -kx : 0.0f);
        sy[i] = in ? __ldg(y + (size_t)r * W + c) - ky : (ZERO_PAD ? -ky : 0.0f);
    }
}

// Horizontal 11-tap pass of the five products over a (rows x in_cols) staged region into h[5][rows][out_cols],
// out_cols = in_cols - 10.
__device__ __forceinline__ void moments_h(const float *sx, const float *sy, int rows, int in_cols, float *h) {
    const int out_cols = in_cols - 2 * kR, plane = rows * out_cols;
    for (int i = threadIdx.x; i < plane; i += kThreads) {
        const int r = i / out_cols, c = i % out_cols;
        const float *px = sx + r * in_cols + c, *py = sy + r * in_cols + c;
        float m0 = 0.0f, m1 = 0.0f, m2 = 0.0f, m3 = 0.0f, m4 = 0.0f;
#pragma unroll
        for (int k = 0; k < kWin; ++k) {
            const float a = px[k], b = py[k], g = kSsimG[k];
            m0 = fmaf(g, a, m0);
            m1 = fmaf(g, b, m1);
            m2 = fmaf(g, a * a, m2);
            m3 = fmaf(g, b * b, m3);
            m4 = fmaf(g, a * b, m4);
        }
        h[i] = m0; h[plane + i] = m1; h[2 * plane + i] = m2; h[3 * plane + i] = m3; h[4 * plane + i] = m4;
    }
}

// Vertical 11-tap pass at (r, c) of h[5][.][cols] (rows r..r+10).
__device__ __forceinline__ Moments moments_v(const float *h, int plane, int cols, int r, int c) {
    Moments m{0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    const float *p = h + r * cols + c;
#pragma unroll
    for (int k = 0; k < kWin; ++k) {
        const float g = kSsimG[k];
        const int o = k * cols;
        m.mx = fmaf(g, p[o], m.mx);
        m.my = fmaf(g, p[plane + o], m.my);
        m.xx = fmaf(g, p[2 * plane + o], m.xx);
        m.yy = fmaf(g, p[3 * plane + o], m.yy);
        m.xy = fmaf(g, p[4 * plane + o], m.xy);
    }
    return m;
}

// The shift of a tile: the plane's value at the pixel nearest the tile's centre (uniform over the CTA).
__device__ __forceinline__ float shift_of(const float *__restrict__ p, int H, int W, int r, int c) {
    return __ldg(p + (size_t)min(max(r, 0), H - 1) * W + min(max(c, 0), W - 1));
}

}  // namespace ps
