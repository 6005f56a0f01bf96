// Fused GaussianAdapter (SURVEY.md 8 row f-1): per-pixel network outputs -> rasterizer-ready
// Gaussians, forward and backward, one thread per ray (its n_samples Gaussians share the raw
// features).  Restates /root/reference/src/model/encoder/common/gaussian_adapter.py:48-95 and
// gaussians.py:8-44 (scale range map, depth * pixel-size multiplier, quaternion -> rotation,
// covariance R S S^T R^T moved to world space, world rays origin + direction * depth, SH mask and
// camera-to-world SH rotation), which in the reference is ~40 element-wise / tiny-matmul torch
// kernels with [b, v, r, srf, spp, ...] intermediates.
//
// The kernel is a streaming one (HBM-bound): per ray it reads 7 + 3 d_sh raw floats, 2
// coordinates and n_samples depths and writes n_samples x (3 + 9 + 3 d_sh) floats.  The raw rows
// and the harmonics go through shared memory so that every global access is a coalesced run
// (a per-lane walk over a 328-byte row would cost 32 sectors per load instruction).  The SH
// rotation is a block-diagonal matrix per camera (blocks 1, 3, 5, 7, 9; built on the host side by
// pixelsplat_b200/sh.py), pre-multiplied by the reference's sh_mask and kept in shared memory.
#include "ps_common.cuh"
#include "raster_math.cuh"

namespace ps {

constexpr int kAdThreads = 128;
constexpr int kAdWarps = kAdThreads / 32;
constexpr int kAdMaxSh = 25;
constexpr int kAdMaxSamples = 8;

struct AdapterView {
    float C[9];      // camera-to-world rotation, row-major
    float o[3];      // camera origin
    float Ki[9];     // inverse intrinsics
    float mult;      // 0.1 * sum(K[:2,:2]^-1 (1/w, 1/h))
};

__device__ __forceinline__ void adapter_view_setup(const float *E, const float *K, int w, int h, AdapterView &v) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) v.C[3 * r + c] = E[4 * r + c];
        v.o[r] = E[4 * r + 3];
    }
    const float a = K[0], b = K[1], c = K[2], d = K[3], e = K[4], f = K[5], g = K[6], hh = K[7], i = K[8];
    const float A = e * i - f * hh, B = -(d * i - f * g), Cc = d * hh - e * g;
    const float inv = 1.0f / (a * A + b * B + c * Cc);
    v.Ki[0] = A * inv; v.Ki[1] = (c * hh - b * i) * inv; v.Ki[2] = (b * f - c * e) * inv;
    v.Ki[3] = B * inv; v.Ki[4] = (a * i - c * g) * inv; v.Ki[5] = (c * d - a * f) * inv;
    v.Ki[6] = Cc * inv; v.Ki[7] = (b * g - a * hh) * inv; v.Ki[8] = (a * e - b * d) * inv;
    // get_scale_multiplier (gaussian_adapter.py:98-109): inverse of the 2x2 block only
    const float det2 = a * e - b * d, px = 1.0f / (float)w, py = 1.0f / (float)h;
    v.mult = 0.1f * ((e * px - b * py) + (-d * px + a * py)) / det2;
}

// Packed block-diagonal SH rotation: block l starts at kBlockOff[l], row-major (2l+1)^2.
__device__ __constant__ int kBlockOff[6] = {0, 1, 10, 35, 84, 165};

__device__ __forceinline__ void load_rotation(const float *D, const float *mask, int n, float *sD, int tid, int nthreads) {
    // sD[off_l + i * n_l + j] = D[l^2 + i][l^2 + j] * mask[l^2 + j]
    for (int e = tid; e < 165; e += nthreads) {
        int l = 0;
        while (e >= kBlockOff[l + 1]) ++l;
        const int nl = 2 * l + 1, rem = e - kBlockOff[l], i = rem / nl, j = rem - i * nl, base = l * l;
        sD[e] = (base + nl <= n) ? D[(size_t)(base + i) * n + base + j] * mask[base + j] : 0.0f;
    }
}

struct QuatFrame {
    float q[4], nq, ts, R[9];
};

__device__ __forceinline__ void quat_forward(const float *qr, float eps, QuatFrame &f) {
    f.nq = sqrtf(qr[0] * qr[0] + qr[1] * qr[1] + qr[2] * qr[2] + qr[3] * qr[3]);
    const float inv = 1.0f / (f.nq + eps);
#pragma unroll
    for (int a = 0; a < 4; ++a) f.q[a] = qr[a] * inv;
    const float i = f.q[0], j = f.q[1], k = f.q[2], r = f.q[3];
    f.ts = 2.0f / (i * i + j * j + k * k + r * r + eps);
    const float ts = f.ts;
    f.R[0] = 1.0f - ts * (j * j + k * k); f.R[1] = ts * (i * j - k * r); f.R[2] = ts * (i * k + j * r);
    f.R[3] = ts * (i * j + k * r); f.R[4] = 1.0f - ts * (i * i + k * k); f.R[5] = ts * (j * k - i * r);
    f.R[6] = ts * (i * k - j * r); f.R[7] = ts * (j * k + i * r); f.R[8] = 1.0f - ts * (i * i + j * j);
}

__device__ __forceinline__ float sigmoidf(float x) { return 1.0f / (1.0f + expf(-x)); }

// One degree-L block of the rotation applied to the three colour channels of a lane's row, in place:
// out[i] = sum_j M[i][j] in[j]  (kTranspose = false)  or  out[j] = sum_i M[i][j] in[i]  (true).
template <int L, bool kTranspose>
__device__ __forceinline__ void sh_rotate_block(float *row, const float *sD, int n_sh) {
    constexpr int nl = 2 * L + 1, base = L * L;
    constexpr int off = L == 0 ? 0 : L == 1 ? 1 : L == 2 ? 10 : L == 3 ? 35 : 84;
    const float *M = sD + off;
    float in[3][nl], out[3][nl];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int j = 0; j < nl; ++j) {
            in[c][j] = row[c * n_sh + base + j];
            out[c][j] = 0.0f;
        }
#pragma unroll
    for (int i = 0; i < nl; ++i)
#pragma unroll
        for (int j = 0; j < nl; ++j) {
            const float m = M[i * nl + j];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                if (kTranspose) out[c][j] += m * in[c][i];
                else out[c][i] += m * in[c][j];
            }
        }
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int j = 0; j < nl; ++j) row[c * n_sh + base + j] = out[c][j];
}

template <bool kTranspose>
__device__ __forceinline__ void sh_rotate_row(float *row, const float *sD, int n_sh) {
    sh_rotate_block<0, kTranspose>(row, sD, n_sh);
    if (n_sh >= 4) sh_rotate_block<1, kTranspose>(row, sD, n_sh);
    if (n_sh >= 9) sh_rotate_block<2, kTranspose>(row, sD, n_sh);
    if (n_sh >= 16) sh_rotate_block<3, kTranspose>(row, sD, n_sh);
    if (n_sh >= 25) sh_rotate_block<4, kTranspose>(row, sD, n_sh);
}

// Coalesced copy of `rows` consecutive n-float rows into padded shared rows, four independent 32-wide
// loads in flight per lane rather than one at a time (this kernel is latency-bound at ~20 warps per SM,
// so memory-level parallelism per warp is what moves it).
__device__ __forceinline__ void stage_rows_x4(const float *__restrict__ src, float *dst, int rows, int n,
                                              int row_stride, int lane) {
    const int total = rows * n;
    int r = lane / n, c = lane - r * n;
    const int step_r = 32 / n, step_c = 32 - step_r * n;
    for (int e = lane; e < total; e += 128) {
        float v[4];
        int off[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            off[q] = r * row_stride + c;
            v[q] = (e + 32 * q < total) ? __ldg(src + e + 32 * q) : 0.0f;
            r += step_r; c += step_c;
            if (c >= n) { c -= n; ++r; }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (e + 32 * q < total) dst[off[q]] = v[q];
    }
}

// Block prologue of both directions: the view's SH rotation and camera into shared memory, then the warp's 32
// rays: rows_valid of them exist, the first at flat (view, ray) index vr0, their staged rows at float row0 of the
// dynamic shared memory.  Returns false for a warp past n_rays, only after the barrier the whole block must reach.
__device__ __forceinline__ bool adapter_prologue(const ps_adapter_desc &d, const ps_adapter_inputs &in, float *sD,
                                                 AdapterView &sv, int row_stride, int &rows_valid, size_t &vr0,
                                                 size_t &row0) {
    const int view = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, n_sh = d.sh_coeffs;
    load_rotation(in.sh_rotation + (size_t)view * n_sh * n_sh, in.sh_mask, n_sh, sD, tid, kAdThreads);
    if (tid == 0) adapter_view_setup(in.extrinsics + 16 * view, in.intrinsics + 9 * view, d.image_w, d.image_h, sv);
    __syncthreads();
    const int ray0 = (blockIdx.x * kAdWarps + warp) * 32;
    if (ray0 >= d.n_rays) return false;
    rows_valid = min(32, d.n_rays - ray0);
    vr0 = (size_t)view * d.n_rays + ray0;
    row0 = (size_t)warp * 32 * row_stride;
    return true;
}

// Everything a ray's Gaussians share.  The backward differentiates the function the forward evaluates only
// because both build this frame here; it also keeps sg, qr, dh and inv_n, which the forward does not use.
struct RayFrame {
    float sg[3], sigma[3];   // sigmoid of the scale logits, the range-mapped scales
    float qr[4];             // the raw quaternion
    QuatFrame qf;
    float A[9];              // C * Rq
    float dh[3], inv_n;      // unit camera-space ray direction, 1 / |K^-1 (x, y, 1)|
    float dw[3];             // world-space ray direction
};

__device__ __forceinline__ void ray_frame(const float *raw7, const float *coordinates, size_t vr, const AdapterView &sv,
                                          const ps_adapter_desc &d, RayFrame &f) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        f.sg[k] = sigmoidf(raw7[k]);
        f.sigma[k] = d.scale_min + (d.scale_max - d.scale_min) * f.sg[k];
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) f.qr[a] = raw7[3 + a];
    quat_forward(f.qr, d.eps, f.qf);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            f.A[3 * r + c] = sv.C[3 * r] * f.qf.R[c] + sv.C[3 * r + 1] * f.qf.R[3 + c] + sv.C[3 * r + 2] * f.qf.R[6 + c];
    const float x = coordinates[2 * vr], y = coordinates[2 * vr + 1];
    float dc[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) dc[r] = sv.Ki[3 * r] * x + sv.Ki[3 * r + 1] * y + sv.Ki[3 * r + 2];
    f.inv_n = 1.0f / sqrtf(dc[0] * dc[0] + dc[1] * dc[1] + dc[2] * dc[2]);
#pragma unroll
    for (int r = 0; r < 3; ++r) f.dh[r] = dc[r] * f.inv_n;
#pragma unroll
    for (int r = 0; r < 3; ++r) f.dw[r] = sv.C[3 * r] * f.dh[0] + sv.C[3 * r + 1] * f.dh[1] + sv.C[3 * r + 2] * f.dh[2];
}

__global__ void __launch_bounds__(kAdThreads)
k_gaussian_adapter_fwd(ps_adapter_desc d, ps_adapter_inputs in, float *__restrict__ means, float *__restrict__ cov,
                       float *__restrict__ harmonics, float *__restrict__ scales, float *__restrict__ rotations,
                       int row_stride) {
    extern __shared__ float s_rows[];                 // [warps][32][row_stride]
    __shared__ float sD[165];
    __shared__ AdapterView sv;
    const int lane = threadIdx.x & 31, n_sh = d.sh_coeffs, raw_n = 7 + 3 * n_sh, ns = d.n_samples;
    int rows_valid;
    size_t vr0, row0;
    if (!adapter_prologue(d, in, sD, sv, row_stride, rows_valid, vr0, row0)) return;
    float *wrows = s_rows + row0;
    stage_rows_x4(in.raw + vr0 * raw_n, wrows, rows_valid, raw_n, row_stride, lane);
    __syncwarp();
    const bool live = lane < rows_valid;
    float *row = wrows + lane * row_stride;
    if (live) {
        const size_t vr = vr0 + lane;
        sh_rotate_row<false>(row + 7, sD, n_sh);
        RayFrame f;
        ray_frame(row, in.coordinates, vr, sv, d, f);
        if (rotations) {
#pragma unroll
            for (int a = 0; a < 4; ++a) rotations[4 * vr + a] = f.qf.q[a];
        }
        for (int j = 0; j < ns; ++j) {
            const size_t g = vr * ns + j;
            const float dep = in.depths[g];
            float sc2[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float sc = f.sigma[k] * dep * sv.mult;
                if (scales) scales[3 * g + k] = sc;
                sc2[k] = sc * sc;
            }
#pragma unroll
            for (int r = 0; r < 3; ++r) means[3 * g + r] = sv.o[r] + f.dw[r] * dep;
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    cov[9 * g + 3 * r + c] = sc2[0] * f.A[3 * r] * f.A[3 * c] + sc2[1] * f.A[3 * r + 1] * f.A[3 * c + 1] +
                                             sc2[2] * f.A[3 * r + 2] * f.A[3 * c + 2];
        }
    }
    __syncwarp();
    // ---- harmonics: the n_samples Gaussians of a ray carry the same rotated coefficients
    // (3 sh_coeffs <= 75 floats per Gaussian: at most three 32-wide coalesced runs, held in registers
    // and stored once per sample)
    const int sh_n = 3 * n_sh;
    const bool has1 = lane + 32 < sh_n, has2 = lane + 64 < sh_n, has0 = lane < sh_n;
    for (int r = 0; r < rows_valid; ++r) {
        const float *src = wrows + r * row_stride + 7;
        const float v0 = has0 ? src[lane] : 0.0f, v1 = has1 ? src[lane + 32] : 0.0f, v2 = has2 ? src[lane + 64] : 0.0f;
        float *dst = harmonics + (vr0 + r) * ns * sh_n + lane;
        for (int j = 0; j < ns; ++j, dst += sh_n) {
            if (has0) dst[0] = v0;
            if (has1) dst[32] = v1;
            if (has2) dst[64] = v2;
        }
    }
}

__global__ void __launch_bounds__(kAdThreads)
k_gaussian_adapter_bwd(ps_adapter_desc d, ps_adapter_inputs in, const float *__restrict__ d_means,
                       const float *__restrict__ d_cov, const float *__restrict__ d_harm,
                       const float *__restrict__ d_scales, const float *__restrict__ d_rot,
                       float *__restrict__ d_coord, float *__restrict__ d_depths, float *__restrict__ d_raw,
                       int row_stride) {
    extern __shared__ float s_rows[];                 // [warps][32][row_stride] gradient rows
    __shared__ float sD[165];
    __shared__ AdapterView sv;
    const int lane = threadIdx.x & 31, n_sh = d.sh_coeffs, raw_n = 7 + 3 * n_sh, ns = d.n_samples, sh_n = 3 * n_sh;
    int rows_valid;
    size_t vr0, row0;
    if (!adapter_prologue(d, in, sD, sv, row_stride, rows_valid, vr0, row0)) return;
    float *wrows = s_rows + row0;
    // ---- dL/d(harmonics), summed over the ray's samples, coalesced into the gradient rows
    {
        const bool has0 = lane < sh_n, has1 = lane + 32 < sh_n, has2 = lane + 64 < sh_n;
        for (int r = 0; r < rows_valid; ++r) {
            const float *src = d_harm + (vr0 + r) * ns * sh_n + lane;
            float t0 = 0.0f, t1 = 0.0f, t2 = 0.0f;
            for (int j = 0; j < ns; ++j, src += sh_n) {
                if (has0) t0 += src[0];
                if (has1) t1 += src[32];
                if (has2) t2 += src[64];
            }
            float *dst = wrows + r * row_stride + 7;
            if (has0) dst[lane] = t0;
            if (has1) dst[lane + 32] = t1;
            if (has2) dst[lane + 64] = t2;
        }
    }
    __syncwarp();
    const bool live = lane < rows_valid;
    float *row = wrows + lane * row_stride;
    if (live) {
        const size_t vr = vr0 + lane;
        sh_rotate_row<true>(row + 7, sD, n_sh);
        RayFrame f;
        ray_frame(in.raw + vr * raw_n, in.coordinates, vr, sv, d, f);
        // ---- accumulate over the ray's samples
        float g_dw[3] = {0.0f, 0.0f, 0.0f}, g_sigma[3] = {0.0f, 0.0f, 0.0f};
        float gA[9] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
        for (int j = 0; j < ns; ++j) {
            const size_t g = vr * ns + j;
            const float dep = in.depths[g];
            float gm[3], G[9];
#pragma unroll
            for (int r = 0; r < 3; ++r) gm[r] = d_means[3 * g + r];
#pragma unroll
            for (int e = 0; e < 9; ++e) G[e] = d_cov[9 * g + e];
            float g_dep = gm[0] * f.dw[0] + gm[1] * f.dw[1] + gm[2] * f.dw[2];
#pragma unroll
            for (int r = 0; r < 3; ++r) g_dw[r] += gm[r] * dep;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float a0 = f.A[k], a1 = f.A[3 + k], a2 = f.A[6 + k];    // column k of A
                // (G + G^T) a_k
                const float u0 = 2.0f * G[0] * a0 + (G[1] + G[3]) * a1 + (G[2] + G[6]) * a2;
                const float u1 = (G[3] + G[1]) * a0 + 2.0f * G[4] * a1 + (G[5] + G[7]) * a2;
                const float u2 = (G[6] + G[2]) * a0 + (G[7] + G[5]) * a1 + 2.0f * G[8] * a2;
                const float quad = 0.5f * (a0 * u0 + a1 * u1 + a2 * u2);      // a_k^T G a_k
                const float sc = f.sigma[k] * dep * sv.mult;
                const float g_sc = 2.0f * sc * quad + (d_scales ? d_scales[3 * g + k] : 0.0f);
                g_dep += g_sc * f.sigma[k] * sv.mult;
                g_sigma[k] += g_sc * dep * sv.mult;
                const float s2 = sc * sc;
                gA[k] += s2 * u0; gA[3 + k] += s2 * u1; gA[6 + k] += s2 * u2;
            }
            d_depths[g] = g_dep;
        }
        // ---- scale logits
#pragma unroll
        for (int k = 0; k < 3; ++k) row[k] = g_sigma[k] * (d.scale_max - d.scale_min) * f.sg[k] * (1.0f - f.sg[k]);
        // ---- rotation: dL/dRq = C^T dL/dA, then through quaternion_to_matrix and the normalisation
        float gR[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                gR[3 * r + c] = sv.C[r] * gA[c] + sv.C[3 + r] * gA[3 + c] + sv.C[6 + r] * gA[6 + c];
        const float i = f.qf.q[0], j = f.qf.q[1], k = f.qf.q[2], r = f.qf.q[3], ts = f.qf.ts;
        const float g_ts = -gR[0] * (j * j + k * k) + gR[1] * (i * j - k * r) + gR[2] * (i * k + j * r) +
                           gR[3] * (i * j + k * r) - gR[4] * (i * i + k * k) + gR[5] * (j * k - i * r) +
                           gR[6] * (i * k - j * r) + gR[7] * (j * k + i * r) - gR[8] * (i * i + j * j);
        float gq[4];
        gq[0] = ts * (gR[1] * j + gR[2] * k + gR[3] * j - 2.0f * gR[4] * i - gR[5] * r + gR[6] * k + gR[7] * r - 2.0f * gR[8] * i);
        gq[1] = ts * (-2.0f * gR[0] * j + gR[1] * i + gR[2] * r + gR[3] * i + gR[5] * k - gR[6] * r + gR[7] * k - 2.0f * gR[8] * j);
        gq[2] = ts * (-2.0f * gR[0] * k - gR[1] * r + gR[2] * i + gR[3] * r - 2.0f * gR[4] * k + gR[5] * j + gR[6] * i + gR[7] * j);
        gq[3] = ts * (-gR[1] * k + gR[2] * j + gR[3] * k - gR[5] * i - gR[6] * j + gR[7] * i);
        const float g_s2 = -0.5f * ts * ts * g_ts;                             // d ts / d (q.q)
#pragma unroll
        for (int a = 0; a < 4; ++a) gq[a] += 2.0f * g_s2 * f.qf.q[a] + (d_rot ? d_rot[4 * vr + a] : 0.0f);
        const float den = f.qf.nq + d.eps;
        const float dotq = f.qr[0] * gq[0] + f.qr[1] * gq[1] + f.qr[2] * gq[2] + f.qr[3] * gq[3];
        const float corr = f.qf.nq > 0.0f ? dotq / (f.qf.nq * den * den) : 0.0f;
#pragma unroll
        for (int a = 0; a < 4; ++a) row[3 + a] = gq[a] / den - f.qr[a] * corr;
        // ---- pixel coordinates: through C, the normalisation and K^-1
        float g_dh[3], g_dc[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) g_dh[c] = sv.C[c] * g_dw[0] + sv.C[3 + c] * g_dw[1] + sv.C[6 + c] * g_dw[2];
        const float proj = f.dh[0] * g_dh[0] + f.dh[1] * g_dh[1] + f.dh[2] * g_dh[2];
#pragma unroll
        for (int c = 0; c < 3; ++c) g_dc[c] = (g_dh[c] - f.dh[c] * proj) * f.inv_n;
        d_coord[2 * vr] = sv.Ki[0] * g_dc[0] + sv.Ki[3] * g_dc[1] + sv.Ki[6] * g_dc[2];
        d_coord[2 * vr + 1] = sv.Ki[1] * g_dc[0] + sv.Ki[4] * g_dc[1] + sv.Ki[7] * g_dc[2];
    }
    __syncwarp();
    unstage_sh_rows(wrows, d_raw + vr0 * raw_n, rows_valid, raw_n, row_stride, lane);
}

// D(R) for every camera: c' = D c  <=>  sum_i c'_i Y_i(d) = sum_i c_i Y_i(R^T d).  Y+ (the per-degree
// pseudo-inverse of the 3DGS basis sampled at `m` fixed directions, float64-fitted on the host once) turns
// the basis values at the rotated directions into the block-diagonal matrix: D_l = Y+_l Y_l(R^T d).
// One CTA per camera; the dot products accumulate in double (m = 192 terms).
// convention PS_SH_BASIS_E3NN (what the reference's rotate_sh computes, sh_rotation.py:18-22): e3nn's
// harmonics are Y_e,i(x, y, z) = s_i Y_3dgs,i(z, x, y), s_i = (-1)^m, hence
// D_e3nn(R) = S D_3dgs(Q R Q^T) S with Q the axis permutation (x, y, z) -> (z, x, y): the same fit on the
// permuted rotation, then a sign per entry.
__global__ void __launch_bounds__(256)
k_sh_rotation(int n_sh, int m, int convention, const float *__restrict__ extrinsics, const float *__restrict__ dirs,
              const float *__restrict__ pinv, float *__restrict__ out) {
    extern __shared__ float s_y[];                    // [m][n_sh] basis at R^T d, then [n_sh][m] pinv
    float *s_pinv = s_y + (size_t)m * n_sh;
    const int view = blockIdx.x, tid = threadIdx.x;
    const float *E = extrinsics + 16 * view;
    const int deg = n_sh >= 25 ? 4 : n_sh >= 16 ? 3 : n_sh >= 9 ? 2 : n_sh >= 4 ? 1 : 0;
    for (int e = tid; e < n_sh * m; e += blockDim.x) s_pinv[e] = pinv[e];
    for (int t = tid; t < m; t += blockDim.x) {
        const float dx = dirs[3 * t], dy = dirs[3 * t + 1], dz = dirs[3 * t + 2];
        float x, y, z;
        if (convention == PS_SH_BASIS_E3NN) {
            // R' = Q R Q^T, R'[a][b] = R[p(a)][p(b)], p = (2, 0, 1);  (R'^T d)_b = sum_a R[p(a)][p(b)] d_a
            x = E[4 * 2 + 2] * dx + E[4 * 0 + 2] * dy + E[4 * 1 + 2] * dz;
            y = E[4 * 2 + 0] * dx + E[4 * 0 + 0] * dy + E[4 * 1 + 0] * dz;
            z = E[4 * 2 + 1] * dx + E[4 * 0 + 1] * dy + E[4 * 1 + 1] * dz;
        } else {
            x = E[0] * dx + E[4] * dy + E[8] * dz;                   // R^T d  (R = E[:3,:3], row-major, stride 4)
            y = E[1] * dx + E[5] * dy + E[9] * dz;
            z = E[2] * dx + E[6] * dy + E[10] * dz;
        }
        float *row = s_y + (size_t)t * n_sh;
        sh_for_each(deg, x, y, z, [&](int i, float v, float, float, float) { row[i] = v; });
    }
    __syncthreads();
    for (int e = tid; e < n_sh * n_sh; e += blockDim.x) {
        const int i = e / n_sh, j = e - i * n_sh;
        int li = 0, lj = 0;
        while ((li + 1) * (li + 1) <= i) ++li;
        while ((lj + 1) * (lj + 1) <= j) ++lj;
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
        if (li == lj) {
            const float *pr = s_pinv + (size_t)i * m, *yc = s_y + j;
            int t = 0;
            for (; t + 3 < m; t += 4) {
                a0 += (double)pr[t] * (double)yc[(size_t)t * n_sh];
                a1 += (double)pr[t + 1] * (double)yc[(size_t)(t + 1) * n_sh];
                a2 += (double)pr[t + 2] * (double)yc[(size_t)(t + 2) * n_sh];
                a3 += (double)pr[t + 3] * (double)yc[(size_t)(t + 3) * n_sh];
            }
            for (; t < m; ++t) a0 += (double)pr[t] * (double)yc[(size_t)t * n_sh];
        }
        float v = (float)((a0 + a1) + (a2 + a3));
        // (-1)^(m_i + m_j), m = index - l^2 - l: same degree => parity of (i - j)
        if (convention == PS_SH_BASIS_E3NN && ((i - j) & 1)) v = -v;
        out[(size_t)view * n_sh * n_sh + e] = v;
    }
}

static int adapter_check(const ps_adapter_desc *d, const ps_adapter_inputs *in, const char *who) {
    if (!d || !in) { set_error("%s: null descriptor", who); return PS_ERR_INVALID_ARGUMENT; }
    if (d->n_views < 1 || d->n_rays < 1 || d->n_samples < 1 || d->n_samples > kAdMaxSamples || d->image_h < 1 || d->image_w < 1) {
        set_error("%s: bad sizes (views %d, rays %d, samples %d)", who, d->n_views, d->n_rays, d->n_samples);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->sh_coeffs != 1 && d->sh_coeffs != 4 && d->sh_coeffs != 9 && d->sh_coeffs != 16 && d->sh_coeffs != 25) {
        set_error("%s: sh_coeffs must be (degree + 1)^2 with degree <= 4 (got %d)", who, d->sh_coeffs);
        return PS_ERR_UNSUPPORTED;
    }
    if (!in->extrinsics || !in->intrinsics || !in->sh_rotation || !in->sh_mask || !in->coordinates || !in->depths || !in->raw) {
        set_error("%s: null input pointer", who);
        return PS_ERR_INVALID_ARGUMENT;
    }
    return PS_OK;
}

// Runs launch(grid, smem, row_stride) for either kernel: kAdThreads rays per block, rows at an odd shared stride.
template <class Launch>
static int launch_adapter(const ps_adapter_desc &d, const char *kernel, Launch launch) {
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_gaussian_adapter_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_gaussian_adapter_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    }
    const int row_stride = (7 + 3 * d.sh_coeffs) | 1;
    launch(dim3((d.n_rays + kAdThreads - 1) / kAdThreads, d.n_views), sizeof(float) * kAdThreads * row_stride, row_stride);
    PS_LAUNCH_CHECK(kernel);
    return PS_OK;
}

}  // namespace ps

extern "C" PS_API int ps_gaussian_adapter_forward(const ps_adapter_desc *desc, const ps_adapter_inputs *in,
                                                  float *means, float *covariances, float *harmonics,
                                                  float *scales, float *rotations, void *stream) {
    using namespace ps;
    const int rc = adapter_check(desc, in, "ps_gaussian_adapter_forward");
    if (rc != PS_OK) return rc;
    if (!means || !covariances || !harmonics) { set_error("ps_gaussian_adapter_forward: null output pointer"); return PS_ERR_INVALID_ARGUMENT; }
    return launch_adapter(*desc, "k_gaussian_adapter_fwd", [&](dim3 grid, size_t smem, int row_stride) {
        k_gaussian_adapter_fwd<<<grid, kAdThreads, smem, static_cast<cudaStream_t>(stream)>>>(
            *desc, *in, means, covariances, harmonics, scales, rotations, row_stride);
    });
}

extern "C" PS_API int ps_gaussian_adapter_backward(const ps_adapter_desc *desc, const ps_adapter_inputs *in,
                                                   const float *d_means, const float *d_covariances,
                                                   const float *d_harmonics, const float *d_scales,
                                                   const float *d_rotations, float *d_coordinates,
                                                   float *d_depths, float *d_raw, void *stream) {
    using namespace ps;
    const int rc = adapter_check(desc, in, "ps_gaussian_adapter_backward");
    if (rc != PS_OK) return rc;
    if (!d_means || !d_covariances || !d_harmonics || !d_coordinates || !d_depths || !d_raw) {
        set_error("ps_gaussian_adapter_backward: null gradient pointer");
        return PS_ERR_INVALID_ARGUMENT;
    }
    return launch_adapter(*desc, "k_gaussian_adapter_bwd", [&](dim3 grid, size_t smem, int row_stride) {
        k_gaussian_adapter_bwd<<<grid, kAdThreads, smem, static_cast<cudaStream_t>(stream)>>>(
            *desc, *in, d_means, d_covariances, d_harmonics, d_scales, d_rotations, d_coordinates, d_depths, d_raw,
            row_stride);
    });
}

extern "C" PS_API int ps_sh_rotation_matrices(int32_t n_views, int32_t sh_coeffs, int32_t n_dirs, int32_t convention,
                                              const float *extrinsics, const float *fit_dirs,
                                              const float *fit_pinv, float *out, void *stream) {
    using namespace ps;
    if (n_views < 1 || n_dirs < 1 || n_dirs > 512 || !extrinsics || !fit_dirs || !fit_pinv || !out) {
        set_error("ps_sh_rotation_matrices: bad argument");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (convention != PS_SH_BASIS_3DGS && convention != PS_SH_BASIS_E3NN) {
        set_error("ps_sh_rotation_matrices: convention must be PS_SH_BASIS_3DGS or PS_SH_BASIS_E3NN (got %d)", convention);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (sh_coeffs != 1 && sh_coeffs != 4 && sh_coeffs != 9 && sh_coeffs != 16 && sh_coeffs != 25) {
        set_error("ps_sh_rotation_matrices: sh_coeffs must be (degree + 1)^2 with degree <= 4 (got %d)", sh_coeffs);
        return PS_ERR_UNSUPPORTED;
    }
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_sh_rotation, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
    }
    k_sh_rotation<<<n_views, 256, 2 * sizeof(float) * n_dirs * sh_coeffs, static_cast<cudaStream_t>(stream)>>>(
        sh_coeffs, n_dirs, convention, extrinsics, fit_dirs, fit_pinv, out);
    PS_LAUNCH_CHECK("k_sh_rotation");
    return PS_OK;
}
