// 3DGS's photometric loss of N images of C channels, prediction p and ground truth g, with its gradient in one pass:
//   loss = (1 - lambda) L1 + lambda (1 - SSIM),   L1 = mean |p - g| over C H W,
// where SSIM is 3DGS's training SSIM, not the evaluation's (csrc/ssim.cu): the same 11x11 Gaussian window (sigma
// 1.5), correlated "same"-size with zero padding (conv2d(padding=5, groups=C)), population (co)variances, C1 = 0.01^2,
// C2 = 0.03^2, and the SSIM map averaged over every pixel and channel, with no crop.
//
// One CTA per (plane, 16 x 32 tile of the image), as ssim.cu's backward: the moments over a 10-pixel halo (out-of-image
// inputs are 0, i.e. -k after the tile's shift k), the SSIM terms on the tile and a 5-pixel halo, and, with the
// gradient, the chain rule's maps on that halo filtered back onto the tile:
//   d(sum S)/dp = G*a_p + 2 p (G*b) + g (G*c)    (p, g, a_p shifted as in ssim.cu; b, c zero outside the image)
// plus the L1 term (1 - lambda) sign(p - g) / (C H W), sign(0) = 0 as torch's abs backward.  Each CTA writes the sums
// of S and |p - g| over its tile; a one-warp-per-image kernel adds them in a fixed order.  No float atomics: the same
// inputs give the same bits every run.  The loss does not depend on whether the gradient is asked for: the tile's S
// values come from the same code path either way and are summed in the same order.
#include "ssim_common.cuh"

namespace ps {

constexpr int kInH = kTH + 4 * kR, kInW = kTW + 4 * kR;     // staged inputs: 36 x 52
constexpr int kMapH = kTH + 2 * kR, kMapW = kTW + 2 * kR;   // SSIM terms and maps: 26 x 42
constexpr int kMapPlane = kMapH * kMapW;
constexpr int kHPlane = kMapH * kTW;                        // maps after the horizontal pass: 26 x 32
constexpr int kSmemFloats = 2 * kInH * kInW + 5 * kInH * kMapW + 3 * kMapPlane + kTH * kTW;
constexpr size_t kSmemBytes = sizeof(float) * kSmemFloats;
static_assert(3 * kHPlane <= 5 * kInH * kMapW, "the filtered maps reuse the moments' buffer");

// grid: n_planes * tiles_per_plane CTAs.  partial[0 .. grid) = sum of S over the tile, partial[grid .. 2 grid) = sum
// of |p - g|.  With GRAD, d_p = d(sum over images of loss)/dp.  s_map = -lambda / (C H W),
// s_l1 = (1 - lambda) / (C H W).
template <bool GRAD>
__global__ void __launch_bounds__(kThreads) k_l1_dssim(int H, int W, int tiles_x, int tiles_per_plane,
                                                       const float *__restrict__ p, const float *__restrict__ g,
                                                       float s_map, float s_l1, float *__restrict__ partial,
                                                       float *__restrict__ d_p) {
    extern __shared__ float smem[];
    float *sg = smem, *sp = sg + kInH * kInW;
    float *h = sp + kInH * kInW;                     // moments after the horizontal pass, then the filtered maps
    float *maps = h + 5 * kInH * kMapW;              // a_p, b, c on the map region
    float *s_tile = maps + 3 * kMapPlane;            // S on the tile
    const int plane = blockIdx.x / tiles_per_plane, tile = blockIdx.x % tiles_per_plane;
    const int R0 = (tile / tiles_x) * kTH, C0 = (tile % tiles_x) * kTW;
    const size_t base = (size_t)plane * H * W;
    p += base;
    g += base;
    const float kg = shift_of(g, H, W, R0 + kTH / 2, C0 + kTW / 2);
    const float kp = shift_of(p, H, W, R0 + kTH / 2, C0 + kTW / 2);
    stage<true>(g, p, H, W, R0 - 2 * kR, C0 - 2 * kR, kInH, kInW, kg, kp, sg, sp);
    __syncthreads();
    moments_h(sg, sp, kInH, kInW, h);
    __syncthreads();
    for (int i = threadIdx.x; i < kMapPlane; i += kThreads) {
        const int r = i / kMapW, c = i % kMapW;
        const int qr = R0 - kR + r, qc = C0 - kR + c;
        const bool on_tile = r >= kR && r < kR + kTH && c >= kR && c < kR + kTW;
        if (!GRAD && !on_tile) continue;
        float ap = 0.0f, b = 0.0f, cc = 0.0f, S = 0.0f;
        if (qr >= 0 && qr < H && qc >= 0 && qc < W) {
            const Moments m = moments_v(h, kInH * kMapW, kMapW, r, c);
            const Ssim q = ssim_at(m, kg, kp, 1.0f);
            S = q.S;
            if (GRAD) {
                const float inv = 1.0f / (q.B1 * q.B2);
                const float dS_dv = -q.S / q.B2;                 // d/d var_g = d/d var_p
                const float dS_dc = 2.0f * q.A1 * inv;           // d/d cov
                const float dS_dmup = 2.0f * q.mux * q.A2 * inv - 2.0f * q.muy * q.S / q.B1;
                ap = s_map * (dS_dmup - 2.0f * m.my * dS_dv - m.mx * dS_dc);
                b = s_map * dS_dv;
                cc = s_map * dS_dc;
            }
        }
        if (on_tile) s_tile[(r - kR) * kTW + c - kR] = S;
        if (GRAD) { maps[i] = ap; maps[kMapPlane + i] = b; maps[2 * kMapPlane + i] = cc; }
    }
    __syncthreads();
    if (GRAD) {
        for (int i = threadIdx.x; i < kHPlane; i += kThreads) {
            const int r = i / kTW, c = i % kTW;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const float *q = maps + j * kMapPlane + r * kMapW + c;
                float acc = 0.0f;
#pragma unroll
                for (int k = 0; k < kWin; ++k) acc = fmaf(kSsimG[k], q[k], acc);
                h[j * kHPlane + i] = acc;
            }
        }
        __syncthreads();
    }
    float acc_s = 0.0f, acc_l1 = 0.0f;
    for (int i = threadIdx.x; i < kTH * kTW; i += kThreads) {
        const int r = i / kTW, c = i % kTW;
        const int pr = R0 + r, pc = C0 + c;
        if (pr >= H || pc >= W) continue;
        const size_t at = (size_t)pr * W + pc;
        const float diff = __ldg(p + at) - __ldg(g + at);
        acc_s += s_tile[i];
        acc_l1 += fabsf(diff);
        if (GRAD) {
            float f[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const float *q = h + j * kHPlane + r * kTW + c;
                float acc = 0.0f;
#pragma unroll
                for (int k = 0; k < kWin; ++k) acc = fmaf(kSsimG[k], q[k * kTW], acc);
                f[j] = acc;
            }
            const int o = (r + 2 * kR) * kInW + c + 2 * kR;
            const float gs = sg[o], ps = sp[o];                  // shifted, like the means in a_p
            const float sgn = diff > 0.0f ? 1.0f : (diff < 0.0f ? -1.0f : 0.0f);
            d_p[base + at] = f[0] + 2.0f * ps * f[1] + gs * f[2] + s_l1 * sgn;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        acc_s += __shfl_xor_sync(0xffffffffu, acc_s, o);
        acc_l1 += __shfl_xor_sync(0xffffffffu, acc_l1, o);
    }
    __shared__ float red[2][kThreads / 32];
    if ((threadIdx.x & 31) == 0) {
        red[0][threadIdx.x >> 5] = acc_s;
        red[1][threadIdx.x >> 5] = acc_l1;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.0f, l = 0.0f;
#pragma unroll
        for (int w = 0; w < kThreads / 32; ++w) {
            s += red[0][w];
            l += red[1][w];
        }
        partial[blockIdx.x] = s;
        partial[gridDim.x + blockIdx.x] = l;
    }
}

// One warp per image: its C * tiles_per_plane partials of each sum in a fixed order.
__global__ void k_l1_dssim_finish(int per_image, int n_partials, float inv_area, float lambda,
                                  const float *__restrict__ partial, float *__restrict__ out_loss,
                                  float *__restrict__ out_l1, float *__restrict__ out_ssim) {
    const float *ps = partial + (size_t)blockIdx.x * per_image, *pl = ps + n_partials;
    float s = 0.0f, l = 0.0f;
    for (int t = threadIdx.x; t < per_image; t += 32) {
        s += ps[t];
        l += pl[t];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        l += __shfl_xor_sync(0xffffffffu, l, o);
    }
    if (threadIdx.x == 0) {
        const float ssim = s * inv_area, l1 = l * inv_area;
        out_loss[blockIdx.x] = (1.0f - lambda) * l1 + lambda * (1.0f - ssim);
        if (out_l1) out_l1[blockIdx.x] = l1;
        if (out_ssim) out_ssim[blockIdx.x] = ssim;
    }
}

// Validates the shape; sets the tiling and the workspace size (two float partials per CTA).
static int check_shape(const char *who, int32_t n, int32_t C, int32_t H, int32_t W, int *tiles_x, int *tiles_per_plane,
                       size_t *workspace) {
    if (n < 1 || C < 1 || H < 1 || W < 1) {
        set_error("%s: bad shape (n %d, C %d, H %d, W %d): every extent must be >= 1", who, n, C, H, W);
        return PS_ERR_INVALID_ARGUMENT;
    }
    *tiles_x = (W + kTW - 1) / kTW;
    *tiles_per_plane = *tiles_x * ((H + kTH - 1) / kTH);
    if ((long long)n * C * *tiles_per_plane > 0x7fffffffLL) {
        set_error("%s: too many planes for one launch (%d x %d of %d x %d)", who, n, C, H, W);
        return PS_ERR_INVALID_ARGUMENT;
    }
    *workspace = (2 * (size_t)n * C * *tiles_per_plane * sizeof(float) + 255) / 256 * 256;
    return PS_OK;
}

}  // namespace ps

extern "C" PS_API int ps_l1_dssim_workspace_bytes(int32_t n, int32_t C, int32_t H, int32_t W, size_t *out) {
    int tx, tpp;
    size_t ws;
    const int rc = ps::check_shape("ps_l1_dssim_workspace_bytes", n, C, H, W, &tx, &tpp, &ws);
    if (rc != PS_OK) return rc;
    if (!out) { ps::set_error("ps_l1_dssim_workspace_bytes: out is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    *out = ws;
    return PS_OK;
}

extern "C" PS_API int ps_l1_dssim(int32_t n, int32_t C, int32_t H, int32_t W, const float *pred, const float *gt,
                                  float lambda, float *out_loss, float *out_l1, float *out_ssim, float *d_pred,
                                  void *workspace, size_t workspace_bytes, void *stream) {
    int tx, tpp;
    size_t ws;
    const int rc = ps::check_shape("ps_l1_dssim", n, C, H, W, &tx, &tpp, &ws);
    if (rc != PS_OK) return rc;
    if (!(lambda >= 0.0f && lambda <= 1.0f)) {   // also refuses NaN
        ps::set_error("ps_l1_dssim: lambda %g is not in [0, 1]", (double)lambda);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (!pred || !gt || !out_loss || !workspace) {
        ps::set_error("ps_l1_dssim: NULL pointer");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (workspace_bytes < ws) {
        ps::set_error("ps_l1_dssim: workspace of %zu bytes, %zu needed", workspace_bytes, ws);
        return PS_ERR_INVALID_ARGUMENT;
    }
    static unsigned long long attr_devices = 0;
    if (ps::first_use_on_device(attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(ps::k_l1_dssim<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)ps::kSmemBytes));
        PS_CUDA_CHECK(cudaFuncSetAttribute(ps::k_l1_dssim<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)ps::kSmemBytes));
    }
    const double area = (double)C * H * W;
    const float s_map = (float)(-(double)lambda / area), s_l1 = (float)((1.0 - (double)lambda) / area);
    const int grid = n * C * tpp;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    float *partial = static_cast<float *>(workspace);
    if (d_pred)
        ps::k_l1_dssim<true><<<grid, ps::kThreads, ps::kSmemBytes, st>>>(H, W, tx, tpp, pred, gt, s_map, s_l1, partial,
                                                                         d_pred);
    else
        ps::k_l1_dssim<false><<<grid, ps::kThreads, ps::kSmemBytes, st>>>(H, W, tx, tpp, pred, gt, s_map, s_l1,
                                                                          partial, nullptr);
    PS_LAUNCH_CHECK("k_l1_dssim");
    ps::k_l1_dssim_finish<<<n, 32, 0, st>>>(C * tpp, grid, (float)(1.0 / area), lambda, partial, out_loss, out_l1,
                                            out_ssim);
    PS_LAUNCH_CHECK("k_l1_dssim_finish");
    return PS_OK;
}
