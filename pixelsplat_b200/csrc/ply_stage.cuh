// Staging shared by the kernels over PLY vertex records (ply_import.cu, ply_densify.cu): one thread per record, 64
// records per CTA; a CTA's records are one contiguous range of the input, loaded into shared memory with 16-byte
// loads, and its outputs stored from shared memory as 16-byte vectors.
#pragma once
#include "ps_common.cuh"

namespace ps {

constexpr int kPlyImportThreads = 64;

// Odd strides: a warp's threads read the same column of 32 staged rows (and write the same entry of 32 outputs), so
// an even stride would put several of them in one shared-memory bank.
__host__ __device__ constexpr int odd(int n) { return n | 1; }

// `count` floats to global `dst` (16-byte aligned): element e is src[(e / width) stride + e % width] in shared memory
__device__ __forceinline__ void store_range(float *__restrict__ dst, const float *__restrict__ src, int count,
                                            int width, int stride) {
    auto at = [&](int e) { const int row = e / width; return src[row * stride + e - row * width]; };
    float4 *d4 = reinterpret_cast<float4 *>(dst);
    for (int i = threadIdx.x; i < count / 4; i += kPlyImportThreads)
        d4[i] = make_float4(at(4 * i), at(4 * i + 1), at(4 * i + 2), at(4 * i + 3));
    for (int i = (count & ~3) + threadIdx.x; i < count; i += kPlyImportThreads) dst[i] = at(i);
}

// Staging: `total` floats of global `src` (16-byte aligned) into shared memory, element e to
// dst[(e / width) stride + e % width].  store_range reversed.
__device__ __forceinline__ void load_range(float *__restrict__ dst, const float *__restrict__ src, int count,
                                           int width, int stride) {
    auto put = [&](int e, float v) { const int row = e / width; dst[row * stride + e - row * width] = v; };
    const float4 *s4 = reinterpret_cast<const float4 *>(src);
    for (int i = threadIdx.x; i < count / 4; i += kPlyImportThreads) {
        const float4 v = __ldg(s4 + i);
        put(4 * i, v.x); put(4 * i + 1, v.y); put(4 * i + 2, v.z); put(4 * i + 3, v.w);
    }
    for (int i = (count & ~3) + threadIdx.x; i < count; i += kPlyImportThreads) put(i, __ldg(src + i));
}

// The quaternion (wxyz) normalised in place, a zero one made the identity; rot = R(q^), row-major.  Returns |q|^2.
__device__ __forceinline__ double unit_rotation(double &qw, double &qx, double &qy, double &qz, double rot[3][3]) {
    const double qn = qw * qw + qx * qx + qy * qy + qz * qz;
    if (qn > 0.0) {
        const double inv = 1.0 / sqrt(qn);
        qw *= inv; qx *= inv; qy *= inv; qz *= inv;
    } else {
        qw = 1.0;   // a zero quaternion is the identity rotation
    }
    rot[0][0] = 1.0 - 2.0 * (qy * qy + qz * qz); rot[0][1] = 2.0 * (qx * qy - qw * qz); rot[0][2] = 2.0 * (qx * qz + qw * qy);
    rot[1][0] = 2.0 * (qx * qy + qw * qz); rot[1][1] = 1.0 - 2.0 * (qx * qx + qz * qz); rot[1][2] = 2.0 * (qy * qz - qw * qx);
    rot[2][0] = 2.0 * (qx * qz - qw * qy); rot[2][1] = 2.0 * (qy * qz + qw * qx); rot[2][2] = 1.0 - 2.0 * (qx * qx + qy * qy);
    return qn;
}

}  // namespace ps
