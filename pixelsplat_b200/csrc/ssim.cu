// SSIM of image planes, forward and backward (/root/reference/src/evaluation/metrics.py:36-52: skimage's
// structural_similarity(win_size=11, gaussian_weights=True, data_range=1.0), sigma 1.5, truncate 3.5,
// use_sample_covariance=True).  Per plane x (ground truth), y (prediction), with G the 11x11 Gaussian window:
//   mu = G*x, G*y;  var = n (G*x^2 - mu^2), cov = n (G*xy - mu_x mu_y), n = 121/120;
//   S = (2 mu_x mu_y + C1)(2 cov + C2) / ((mu_x^2 + mu_y^2 + C1)(var_x + var_y + C2)),  C1 = 0.01^2, C2 = 0.03^2;
//   score = mean of S over the crop [5, H-5) x [5, W-5) (only windows that lie inside the image).
// The filter is separable: a horizontal 11-tap pass into shared memory, then a vertical one.  The window, the
// staging and the passes are in ssim_common.cuh, with the numerics of the shifted moments they form.
//
// Forward: one CTA per (plane, 16 x 32 tile of the crop) writes the sum of S over its tile to the workspace; a
// second kernel sums a plane's partials in a fixed order.  No float atomics: the result is the same bits every run.
// Backward: one CTA per (plane, 16 x 32 tile of the image) recomputes the moments over a 10-pixel halo, forms the
// per-pixel maps a_x, a_y, b, c of the chain rule on a 5-pixel halo and filters them:
//   dL/dy = G*a_y + 2 y (G*b) + x (G*c),   dL/dx = G*a_x + 2 x (G*b) + y (G*c)
// (G is symmetric, so the correlation is its own adjoint; b and c are shared by both inputs).
#include "ssim_common.cuh"

namespace ps {

constexpr float kCov = 121.0f / 120.0f;      // sample covariance over the 121-pixel window

constexpr int kFInH = kTH + 2 * kR, kFInW = kTW + 2 * kR;   // forward staged region: 26 x 42

// grid: n_planes * tiles_per_plane CTAs; tile t of a plane covers crop rows [ty*16, +16), columns [tx*32, +32),
// i.e. image rows 5 + ty*16 ..; its input rows are [ty*16, ty*16 + 26).
__global__ void __launch_bounds__(kThreads) k_ssim_fwd(int H, int W, int tiles_x, int tiles_per_plane,
                                                       const float *__restrict__ x, const float *__restrict__ y,
                                                       float *__restrict__ partial) {
    __shared__ float sx[kFInH * kFInW], sy[kFInH * kFInW];
    __shared__ float h[5 * kFInH * kTW];
    __shared__ float red[kThreads / 32];
    const int plane = blockIdx.x / tiles_per_plane, tile = blockIdx.x % tiles_per_plane;
    const int r0 = (tile / tiles_x) * kTH, c0 = (tile % tiles_x) * kTW;
    const size_t base = (size_t)plane * H * W;
    x += base;
    y += base;
    const float kx = shift_of(x, H, W, r0 + kR + kTH / 2, c0 + kR + kTW / 2);
    const float ky = shift_of(y, H, W, r0 + kR + kTH / 2, c0 + kR + kTW / 2);
    stage(x, y, H, W, r0, c0, kFInH, kFInW, kx, ky, sx, sy);
    __syncthreads();
    moments_h(sx, sy, kFInH, kFInW, h);
    __syncthreads();
    const int crop_h = H - 2 * kR, crop_w = W - 2 * kR;
    float acc = 0.0f;
    for (int i = threadIdx.x; i < kTH * kTW; i += kThreads) {
        const int r = i / kTW, c = i % kTW;
        if (r0 + r < crop_h && c0 + c < crop_w) acc += ssim_at(moments_v(h, kFInH * kTW, kTW, r, c), kx, ky, kCov).S;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.0f;
#pragma unroll
        for (int w = 0; w < kThreads / 32; ++w) s += red[w];
        partial[blockIdx.x] = s;
    }
}

// One warp per plane: the plane's partials in a fixed order, over the crop's area.
__global__ void k_ssim_finish(int tiles_per_plane, float area, const float *__restrict__ partial,
                              float *__restrict__ out) {
    const float *p = partial + (size_t)blockIdx.x * tiles_per_plane;
    float s = 0.0f;
    for (int t = threadIdx.x; t < tiles_per_plane; t += 32) s += p[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) out[blockIdx.x] = s / area;
}

// Backward regions of a 16 x 32 output tile at image (R0, C0): maps on rows [R0-5, R0+21), columns [C0-5, C0+37);
// their moments need inputs on rows [R0-10, R0+26), columns [C0-10, C0+42).
constexpr int kBInH = kTH + 4 * kR, kBInW = kTW + 4 * kR;   // 36 x 52
constexpr int kMapH = kTH + 2 * kR, kMapW = kTW + 2 * kR;   // 26 x 42
constexpr int kBwdSmemFloats = 2 * kBInH * kBInW + 5 * kBInH * kMapW + 4 * kMapH * kMapW;
constexpr size_t kBwdSmemBytes = sizeof(float) * kBwdSmemFloats;
static_assert(4 * kMapH * kTW <= 5 * kBInH * kMapW, "the filtered maps reuse the moments' buffer");

template <bool WANT_X>
__global__ void __launch_bounds__(kThreads) k_ssim_bwd(int H, int W, int tiles_x, int tiles_per_plane,
                                                       const float *__restrict__ x, const float *__restrict__ y,
                                                       const float *__restrict__ d_mean, float *__restrict__ d_x,
                                                       float *__restrict__ d_y) {
    extern __shared__ float smem[];
    float *sx = smem, *sy = sx + kBInH * kBInW;
    float *h = sy + kBInH * kBInW;                   // moments after the horizontal pass, then the filtered maps
    float *maps = h + 5 * kBInH * kMapW;             // a_y, b, c, a_x on the map region
    const int plane = blockIdx.x / tiles_per_plane, tile = blockIdx.x % tiles_per_plane;
    const int R0 = (tile / tiles_x) * kTH, C0 = (tile % tiles_x) * kTW;
    const size_t base = (size_t)plane * H * W;
    x += base;
    y += base;
    const float kx = shift_of(x, H, W, R0 + kTH / 2, C0 + kTW / 2);
    const float ky = shift_of(y, H, W, R0 + kTH / 2, C0 + kTW / 2);
    stage(x, y, H, W, R0 - 2 * kR, C0 - 2 * kR, kBInH, kBInW, kx, ky, sx, sy);
    __syncthreads();
    moments_h(sx, sy, kBInH, kBInW, h);
    __syncthreads();
    // the chain rule's per-pixel maps, zero outside the crop (s = dL/dscore / |crop| inside)
    const float s = d_mean[plane] / (float)((H - 2 * kR) * (W - 2 * kR));
    constexpr int kMapPlane = kMapH * kMapW;
    for (int i = threadIdx.x; i < kMapPlane; i += kThreads) {
        const int r = i / kMapW, c = i % kMapW;
        const int qr = R0 - kR + r, qc = C0 - kR + c;
        float ay = 0.0f, ax = 0.0f, b = 0.0f, cc = 0.0f;
        if (qr >= kR && qr < H - kR && qc >= kR && qc < W - kR) {
            const Moments m = moments_v(h, kBInH * kMapW, kMapW, r, c);
            const Ssim q = ssim_at(m, kx, ky, kCov);
            const float inv = 1.0f / (q.B1 * q.B2);
            const float dS_dv = -q.S / q.B2;                 // d/d var_x = d/d var_y
            const float dS_dc = 2.0f * q.A1 * inv;           // d/d cov
            const float dS_dmuy = 2.0f * q.mux * q.A2 * inv - 2.0f * q.muy * q.S / q.B1;
            ay = s * (dS_dmuy - 2.0f * kCov * m.my * dS_dv - kCov * m.mx * dS_dc);
            if (WANT_X) {
                const float dS_dmux = 2.0f * q.muy * q.A2 * inv - 2.0f * q.mux * q.S / q.B1;
                ax = s * (dS_dmux - 2.0f * kCov * m.mx * dS_dv - kCov * m.my * dS_dc);
            }
            b = s * kCov * dS_dv;
            cc = s * kCov * dS_dc;
        }
        maps[i] = ay; maps[kMapPlane + i] = b; maps[2 * kMapPlane + i] = cc;
        if (WANT_X) maps[3 * kMapPlane + i] = ax;
    }
    __syncthreads();
    constexpr int kNMaps = WANT_X ? 4 : 3;
    constexpr int kHPlane = kMapH * kTW;
    for (int i = threadIdx.x; i < kHPlane; i += kThreads) {
        const int r = i / kTW, c = i % kTW;
#pragma unroll
        for (int j = 0; j < kNMaps; ++j) {
            const float *p = maps + j * kMapPlane + r * kMapW + c;
            float acc = 0.0f;
#pragma unroll
            for (int k = 0; k < kWin; ++k) acc = fmaf(kSsimG[k], p[k], acc);
            h[j * kHPlane + i] = acc;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kTH * kTW; i += kThreads) {
        const int r = i / kTW, c = i % kTW;
        const int pr = R0 + r, pc = C0 + c;
        if (pr >= H || pc >= W) continue;
        float g[kNMaps];
#pragma unroll
        for (int j = 0; j < kNMaps; ++j) {
            const float *p = h + j * kHPlane + r * kTW + c;
            float acc = 0.0f;
#pragma unroll
            for (int k = 0; k < kWin; ++k) acc = fmaf(kSsimG[k], p[k * kTW], acc);
            g[j] = acc;
        }
        const int o = (r + 2 * kR) * kBInW + c + 2 * kR;
        const float xp = sx[o], yp = sy[o];                  // shifted, like the means in a_y / a_x
        const size_t out = base + (size_t)pr * W + pc;
        d_y[out] = g[0] + 2.0f * yp * g[1] + xp * g[2];
        if (WANT_X) d_x[out] = g[3] + 2.0f * xp * g[1] + yp * g[2];
    }
}

static int tiles_of(int rows, int cols, int *tiles_x) {
    *tiles_x = (cols + kTW - 1) / kTW;
    return *tiles_x * ((rows + kTH - 1) / kTH);
}

// Validates the shape; sets the forward's tiling (over the crop) and its workspace size.
static int check_shape(const char *who, int32_t n_planes, int32_t H, int32_t W, int *tiles_x, int *tiles_per_plane,
                size_t *workspace) {
    if (n_planes < 1 || H < kWin || W < kWin) {
        set_error("%s: bad shape (n_planes %d, H %d, W %d): need n_planes >= 1 and H, W >= 11", who, n_planes, H, W);
        return PS_ERR_INVALID_ARGUMENT;
    }
    *tiles_per_plane = tiles_of(H - 2 * kR, W - 2 * kR, tiles_x);
    int bx;
    if ((long long)n_planes * tiles_of(H, W, &bx) > 0x7fffffffLL) {
        set_error("%s: too many planes for one launch (%d of %d x %d)", who, n_planes, H, W);
        return PS_ERR_INVALID_ARGUMENT;
    }
    *workspace = ((size_t)n_planes * *tiles_per_plane * sizeof(float) + 255) / 256 * 256;
    return PS_OK;
}

}  // namespace ps

extern "C" PS_API int ps_ssim_workspace_bytes(int32_t n_planes, int32_t H, int32_t W, size_t *out) {
    int tx, tpp;
    size_t ws;
    const int rc = ps::check_shape("ps_ssim_workspace_bytes", n_planes, H, W, &tx, &tpp, &ws);
    if (rc != PS_OK) return rc;
    if (!out) { ps::set_error("ps_ssim_workspace_bytes: out is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    *out = ws;
    return PS_OK;
}

extern "C" PS_API int ps_ssim_forward(int32_t n_planes, int32_t H, int32_t W, const float *x, const float *y,
                                      float *out_mean, void *workspace, size_t workspace_bytes, void *stream) {
    int tx, tpp;
    size_t ws;
    const int rc = ps::check_shape("ps_ssim_forward", n_planes, H, W, &tx, &tpp, &ws);
    if (rc != PS_OK) return rc;
    if (!x || !y || !out_mean || !workspace) {
        ps::set_error("ps_ssim_forward: NULL pointer");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (workspace_bytes < ws) {
        ps::set_error("ps_ssim_forward: workspace of %zu bytes, %zu needed", workspace_bytes, ws);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    float *partial = static_cast<float *>(workspace);
    ps::k_ssim_fwd<<<n_planes * tpp, ps::kThreads, 0, st>>>(H, W, tx, tpp, x, y, partial);
    PS_LAUNCH_CHECK("k_ssim_fwd");
    ps::k_ssim_finish<<<n_planes, 32, 0, st>>>(tpp, (float)(H - 2 * ps::kR) * (float)(W - 2 * ps::kR), partial,
                                               out_mean);
    PS_LAUNCH_CHECK("k_ssim_finish");
    return PS_OK;
}

extern "C" PS_API int ps_ssim_backward(int32_t n_planes, int32_t H, int32_t W, const float *x, const float *y,
                                       const float *d_mean, float *d_x, float *d_y, void *workspace,
                                       size_t workspace_bytes, void *stream) {
    int tx, tpp;
    size_t ws;
    const int rc = ps::check_shape("ps_ssim_backward", n_planes, H, W, &tx, &tpp, &ws);
    if (rc != PS_OK) return rc;
    if (!x || !y || !d_mean || !d_y || !workspace) {
        ps::set_error("ps_ssim_backward: NULL pointer");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (workspace_bytes < ws) {
        ps::set_error("ps_ssim_backward: workspace of %zu bytes, %zu needed", workspace_bytes, ws);
        return PS_ERR_INVALID_ARGUMENT;
    }
    static unsigned long long attr_devices = 0;
    if (ps::first_use_on_device(attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(ps::k_ssim_bwd<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)ps::kBwdSmemBytes));
        PS_CUDA_CHECK(cudaFuncSetAttribute(ps::k_ssim_bwd<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)ps::kBwdSmemBytes));
    }
    int bx;
    const int tiles = ps::tiles_of(H, W, &bx);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (d_x)
        ps::k_ssim_bwd<true><<<n_planes * tiles, ps::kThreads, ps::kBwdSmemBytes, st>>>(H, W, bx, tiles, x, y, d_mean,
                                                                                         d_x, d_y);
    else
        ps::k_ssim_bwd<false><<<n_planes * tiles, ps::kThreads, ps::kBwdSmemBytes, st>>>(H, W, bx, tiles, x, y,
                                                                                          d_mean, nullptr, d_y);
    PS_LAUNCH_CHECK("k_ssim_bwd");
    return PS_OK;
}
