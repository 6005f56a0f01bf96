// Per-Gaussian projection math shared by the preprocess forward and backward kernels.
// Semantics: SURVEY.md Appendix A.1 / A.4 / A.5 (EWA splatting of a 3D covariance with a
// 0.3 px low-pass, 3-sigma radius, real SH up to degree 4 in the 3DGS sign convention).
//
// The expression shapes (operand order, no re-association) are deliberate: the forward kernel
// is compiled with --fmad=false so that depth bits, radii and tile rectangles are IEEE-exact
// and can be checked bit-for-bit ("bit-exact tile/bin indices").
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ps {

constexpr float kShC0 = 0.28209479177387814f;
constexpr float kShC1 = 0.4886025119029199f;

struct Cov2D {
    float tx, ty, tz;    // view-space mean
    float ctx, cty;      // after the +-1.3 tan(fov) clamp
    bool clamp_x, clamp_y;
    float m0[3], m1[3];  // rows of M = J * R  (2x3)
    float a, b, c;       // 2D covariance + 0.3 I
};

__device__ __forceinline__ void load_cov6(const float *cov, int layout, float scale2, float s[6]) {
    if (layout == PS_COV_TRIU6) {
#pragma unroll
        for (int i = 0; i < 6; ++i) s[i] = cov[i];
    } else {
        s[0] = cov[0]; s[1] = cov[1]; s[2] = cov[2]; s[3] = cov[4]; s[4] = cov[5]; s[5] = cov[8];
    }
    if (scale2 != 1.0f) {
#pragma unroll
        for (int i = 0; i < 6; ++i) s[i] = s[i] * scale2;
    }
}

__device__ __forceinline__ void compute_cov2d(float px, float py, float pz, const float s[6],
                                              const float *__restrict__ vm, float focal_x,
                                              float focal_y, float tanfovx, float tanfovy,
                                              Cov2D &o) {
    o.tx = vm[0] * px + vm[4] * py + vm[8] * pz + vm[12];
    o.ty = vm[1] * px + vm[5] * py + vm[9] * pz + vm[13];
    o.tz = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14];
    const float limx = 1.3f * tanfovx, limy = 1.3f * tanfovy;
    const float txtz = o.tx / o.tz, tytz = o.ty / o.tz;
    o.clamp_x = (txtz < -limx) || (txtz > limx);
    o.clamp_y = (tytz < -limy) || (tytz > limy);
    o.ctx = fminf(limx, fmaxf(-limx, txtz)) * o.tz;
    o.cty = fminf(limy, fmaxf(-limy, tytz)) * o.tz;
    const float tz = o.tz;
    const float j00 = focal_x / tz;
    const float j02 = -(focal_x * o.ctx) / (tz * tz);
    const float j11 = focal_y / tz;
    const float j12 = -(focal_y * o.cty) / (tz * tz);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        o.m0[j] = j00 * vm[4 * j + 0] + j02 * vm[4 * j + 2];
        o.m1[j] = j11 * vm[4 * j + 1] + j12 * vm[4 * j + 2];
    }
    const float sxx = s[0], sxy = s[1], sxz = s[2], syy = s[3], syz = s[4], szz = s[5];
    const float v0x = sxx * o.m0[0] + sxy * o.m0[1] + sxz * o.m0[2];
    const float v0y = sxy * o.m0[0] + syy * o.m0[1] + syz * o.m0[2];
    const float v0z = sxz * o.m0[0] + syz * o.m0[1] + szz * o.m0[2];
    const float v1x = sxx * o.m1[0] + sxy * o.m1[1] + sxz * o.m1[2];
    const float v1y = sxy * o.m1[0] + syy * o.m1[1] + syz * o.m1[2];
    const float v1z = sxz * o.m1[0] + syz * o.m1[1] + szz * o.m1[2];
    o.a = o.m0[0] * v0x + o.m0[1] * v0y + o.m0[2] * v0z + 0.3f;
    o.b = o.m0[0] * v1x + o.m0[1] * v1y + o.m0[2] * v1z;
    o.c = o.m1[0] * v1x + o.m1[1] * v1y + o.m1[2] * v1z + 0.3f;
}

// Real SH up to degree 4 (3DGS sign convention), visited term by term: f(k, Y_k, dY_k/dx,
// dY_k/dy, dY_k/dz) is called for k = 0 .. (deg+1)^2-1 in order, with x, y, z treated as
// independent variables in the derivatives.  Consuming the terms as they are produced keeps
// the 25 (or 100, with derivatives) values out of registers; callers that ignore the
// derivatives pay nothing for them.  The value expressions are written exactly as in the oracle
// (operand order matters: the forward kernel is compiled without FMA contraction).
template <class F>
__device__ __forceinline__ void sh_for_each(int deg, float x, float y, float z, F &&f) {
    f(0, kShC0, 0.0f, 0.0f, 0.0f);
    if (deg < 1) return;
    f(1, -kShC1 * y, 0.0f, -kShC1, 0.0f);
    f(2, kShC1 * z, 0.0f, 0.0f, kShC1);
    f(3, -kShC1 * x, -kShC1, 0.0f, 0.0f);
    if (deg < 2) return;
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    {
        const float c0 = 1.0925484305920792f, c2 = 0.31539156525252005f, c4 = 0.5462742152960396f;
        f(4, 1.0925484305920792f * xy, c0 * y, c0 * x, 0.0f);
        f(5, -1.0925484305920792f * yz, 0.0f, -c0 * z, -c0 * y);
        f(6, 0.31539156525252005f * (2.0f * zz - xx - yy), -2.0f * c2 * x, -2.0f * c2 * y, 4.0f * c2 * z);
        f(7, -1.0925484305920792f * xz, -c0 * z, 0.0f, -c0 * x);
        f(8, 0.5462742152960396f * (xx - yy), 2.0f * c4 * x, -2.0f * c4 * y, 0.0f);
    }
    if (deg < 3) return;
    {
        const float c0 = -0.5900435899266435f, c1 = 2.890611442640554f, c2 = -0.4570457994644658f,
                    c3 = 0.3731763325901154f, c5 = 1.445305721320277f;
        f(9, -0.5900435899266435f * y * (3.0f * xx - yy), c0 * 6.0f * xy, c0 * (3.0f * xx - 3.0f * yy), 0.0f);
        f(10, 2.890611442640554f * xy * z, c1 * yz, c1 * xz, c1 * xy);
        f(11, -0.4570457994644658f * y * (4.0f * zz - xx - yy), c2 * -2.0f * xy, c2 * (4.0f * zz - xx - 3.0f * yy), c2 * 8.0f * yz);
        f(12, 0.3731763325901154f * z * (2.0f * zz - 3.0f * xx - 3.0f * yy), c3 * -6.0f * xz, c3 * -6.0f * yz,
          c3 * (6.0f * zz - 3.0f * xx - 3.0f * yy));
        f(13, -0.4570457994644658f * x * (4.0f * zz - xx - yy), c2 * (4.0f * zz - 3.0f * xx - yy), c2 * -2.0f * xy, c2 * 8.0f * xz);
        f(14, 1.445305721320277f * z * (xx - yy), c5 * 2.0f * xz, c5 * -2.0f * yz, c5 * (xx - yy));
        f(15, -0.5900435899266435f * x * (xx - 3.0f * yy), c0 * (3.0f * xx - 3.0f * yy), c0 * -6.0f * xy, 0.0f);
    }
    if (deg < 4) return;
    {
        const float c0 = 2.5033429417967046f, c1 = -1.7701307697799304f, c2 = 0.9461746957575601f,
                    c3 = -0.6690465435572892f, c4 = 0.10578554691520431f, c6 = 0.47308734787878004f,
                    c8 = 0.6258357354491761f;
        f(16, 2.5033429417967046f * xy * (xx - yy), c0 * (3.0f * xx * y - yy * y), c0 * (xx * x - 3.0f * x * yy), 0.0f);
        f(17, -1.7701307697799304f * yz * (3.0f * xx - yy), c1 * 6.0f * xy * z, c1 * z * (3.0f * xx - 3.0f * yy), c1 * y * (3.0f * xx - yy));
        f(18, 0.9461746957575601f * xy * (7.0f * zz - 1.0f), c2 * y * (7.0f * zz - 1.0f), c2 * x * (7.0f * zz - 1.0f), c2 * 14.0f * xy * z);
        f(19, -0.6690465435572892f * yz * (7.0f * zz - 3.0f), 0.0f, c3 * z * (7.0f * zz - 3.0f), c3 * y * (21.0f * zz - 3.0f));
        f(20, 0.10578554691520431f * (zz * (35.0f * zz - 30.0f) + 3.0f), 0.0f, 0.0f, c4 * (140.0f * zz * z - 60.0f * z));
        f(21, -0.6690465435572892f * xz * (7.0f * zz - 3.0f), c3 * z * (7.0f * zz - 3.0f), 0.0f, c3 * x * (21.0f * zz - 3.0f));
        f(22, 0.47308734787878004f * (xx - yy) * (7.0f * zz - 1.0f), c6 * 2.0f * x * (7.0f * zz - 1.0f), c6 * -2.0f * y * (7.0f * zz - 1.0f),
          c6 * 14.0f * z * (xx - yy));
        f(23, -1.7701307697799304f * xz * (xx - 3.0f * yy), c1 * z * (3.0f * xx - 3.0f * yy), c1 * -6.0f * xy * z, c1 * x * (xx - 3.0f * yy));
        f(24, 0.6258357354491761f * (xx * (xx - 3.0f * yy) - yy * (3.0f * xx - yy)), c8 * (4.0f * xx * x - 12.0f * x * yy),
          c8 * (4.0f * yy * y - 12.0f * xx * y), 0.0f);
    }
}

// The e3nn convention (PS_SH_BASIS_E3NN) on top of the same polynomials:
//   Y_e3nn,k(x, y, z) = (-1)^m Y_k(z, x, y), and (-1)^m = (-1)^k because l^2 + l is even.
// Callers evaluate sh_for_each at sh_arg(basis, x, y, z), flip the sign of odd-k terms with sh_sign()
// (an exact operation: results stay bit-identical to the oracle's), and map the derivative triple back
// with sh_grad_unpermute().  k is a literal at every call site of the visitor, so `k & 1` folds away.
__device__ __forceinline__ float3 sh_arg(int basis, float x, float y, float z) {
    return basis == PS_SH_BASIS_E3NN ? make_float3(z, x, y) : make_float3(x, y, z);
}
__device__ __forceinline__ float sh_sign(uint32_t flip_mask, int k, float v) {
    return (k & 1) ? __uint_as_float(__float_as_uint(v) ^ flip_mask) : v;
}
__device__ __forceinline__ uint32_t sh_flip_mask(int basis) { return basis == PS_SH_BASIS_E3NN ? 0x80000000u : 0u; }
// f(x, y, z) = g(a, b, c) at (a, b, c) = (z, x, y):  df/dx = dg/db, df/dy = dg/dc, df/dz = dg/da
__device__ __forceinline__ float3 sh_grad_unpermute(int basis, float da, float db, float dc) {
    return basis == PS_SH_BASIS_E3NN ? make_float3(db, dc, da) : make_float3(da, db, dc);
}

// One warp's `rows` staged rows of sh_n floats (shared memory, row stride padded to an odd word count so that
// per-lane row accesses are bank-conflict free) back to global as one contiguous, coalesced run of rows*sh_n floats.
__device__ __forceinline__ void unstage_sh_rows(const float *src, float *__restrict__ dst, int rows, int sh_n,
                                                int row_stride, int lane) {
    const int total = rows * sh_n;
    if (row_stride == sh_n) {
        const bool vec_ok = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
        const int nvec = vec_ok ? total >> 2 : 0;
        for (int i = lane; i < nvec; i += 32)
            reinterpret_cast<float4 *>(dst)[i] = reinterpret_cast<const float4 *>(src)[i];
        for (int e = 4 * nvec + lane; e < total; e += 32) dst[e] = src[e];
        return;
    }
    int e = lane, r = e / sh_n, c = e - r * sh_n;
    const int step_r = 32 / sh_n, step_c = 32 - step_r * sh_n;
    for (; e < total; e += 32) {
        dst[e] = src[r * row_stride + c];
        r += step_r; c += step_c;
        if (c >= sh_n) { c -= sh_n; ++r; }
    }
}

// Gathers 32 scattered rows of sh_n floats (one per lane's Gaussian, `row_of_lane` = the flat row index held by
// each lane) into the warp's shared staging area, one padded row per lane.  Every element is one cp.async (LDGSTS,
// 4 bytes -- rows start on 4-byte boundaries only), so the whole warp's 32 x sh_n floats are in flight at once and
// the caller can do unrelated work before gather_rows_wait().  Only the rows of the lanes set in `rows` are fetched;
// the others are left as they are.
__device__ __forceinline__ void gather_rows_async(const float *__restrict__ base, unsigned long long row_of_lane,
                                                  unsigned rows, int sh_n, float *wrows, int row_stride, int lane) {
    for (unsigned m = rows; m != 0u; m &= m - 1u) {
        const int r = __ffs(m) - 1;
        const unsigned long long rs = __shfl_sync(0xffffffffu, row_of_lane, r);
        const float *src = base + rs * (unsigned long long)sh_n;
        float *dst = wrows + r * row_stride;
        for (int c = lane; c < sh_n; c += 32) {
            const uint32_t saddr = (uint32_t)__cvta_generic_to_shared(dst + c);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(saddr), "l"(src + c) : "memory");
        }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

__device__ __forceinline__ void gather_rows_wait() {
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncwarp();
}

// Zeros dst[0 .. n) with the warp: 16-byte stores where dst is 16-byte aligned.
__device__ __forceinline__ void zero_fill_warp(float *__restrict__ dst, int n, int lane) {
    const int nvec = (reinterpret_cast<uintptr_t>(dst) & 15) == 0 ? n >> 2 : 0;
    for (int i = lane; i < nvec; i += 32) reinterpret_cast<float4 *>(dst)[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    for (int e = 4 * nvec + lane; e < n; e += 32) dst[e] = 0.0f;
}

__device__ __forceinline__ int sh_index(int layout, int M, int k, int ch) {
    return layout == PS_SH_M3 ? k * 3 + ch : ch * M + k;
}

}  // namespace ps
