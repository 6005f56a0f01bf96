// PLY import: the vertex records of a 3D Gaussian splatting PLY file unpacked into one scene's Gaussians (the
// contract is in include/pixelsplat_b200.h, ps_ply_unpack).  ps_ply_pack's store pattern, reversed: the CTA loads its
// records, which are one contiguous range of the input, with 16-byte loads into shared memory; every thread turns
// its record into its Gaussian's outputs in shared memory; the CTA stores each output array's contiguous range as
// 16-byte vectors.  The kernel is bound by HBM traffic: 248 B read and 244 B written per Gaussian at degree 3 with
// normals in and 16 coefficients out.
//
// The file's SH degree is a template parameter, so every index into the staged record's columns and the SH
// transform is a compile-time constant.
#include "ps_common.cuh"

namespace ps {

constexpr int kPlyImportThreads = 64;

// Odd strides: a warp's threads read the same column of 32 staged rows (and write the same entry of 32 outputs), so
// an even stride would put several of them in one shared-memory bank.
__host__ __device__ constexpr int odd(int n) { return n | 1; }

__host__ __device__ constexpr int ply_import_smem_floats(int n_props, int sh_coeffs) {
    return kPlyImportThreads * (odd(n_props) + 3 + 9 + 1 + odd(3 * sh_coeffs));
}

// `count` floats to global `dst` (16-byte aligned): element e is src[(e / width) stride + e % width] in shared memory
__device__ __forceinline__ void store_range(float *__restrict__ dst, const float *__restrict__ src, int count,
                                            int width, int stride) {
    auto at = [&](int e) { const int row = e / width; return src[row * stride + e - row * width]; };
    float4 *d4 = reinterpret_cast<float4 *>(dst);
    for (int i = threadIdx.x; i < count / 4; i += kPlyImportThreads)
        d4[i] = make_float4(at(4 * i), at(4 * i + 1), at(4 * i + 2), at(4 * i + 3));
    for (int i = (count & ~3) + threadIdx.x; i < count; i += kPlyImportThreads) dst[i] = at(i);
}

template <int DEG>
__global__ void __launch_bounds__(kPlyImportThreads) k_ply_unpack(const ps_ply_import_desc d) {
    constexpr int NC = (DEG + 1) * (DEG + 1);   // coefficients per channel in the file
    extern __shared__ float4 smem4[];
    const int P = d.n_props, C = d.sh_coeffs, PS = odd(P), HS = odd(3 * C);
    float *rows = reinterpret_cast<float *>(smem4);    // [64, PS]
    float *om = rows + kPlyImportThreads * PS;         // means [64, 3]
    float *oc = om + kPlyImportThreads * 3;            // covariances [64, 9]
    float *oo = oc + kPlyImportThreads * 9;            // opacities [64]
    float *oh = oo + kPlyImportThreads;                // harmonics [64, HS], [3, C] used

    const long long g0 = (long long)blockIdx.x * kPlyImportThreads;
    const int cnt = (int)min((long long)kPlyImportThreads, d.n_gaussians - g0);
    {
        // the CTA's records: cnt P floats from g0 P, 16-byte aligned (64 P floats per CTA), into rows of PS
        const float *src = d.records + g0 * P;
        const int total = cnt * P;
        auto put = [&](int e, float v) { const int row = e / P; rows[row * PS + e - row * P] = v; };
        const float4 *s4 = reinterpret_cast<const float4 *>(src);
        for (int i = threadIdx.x; i < total / 4; i += kPlyImportThreads) {
            const float4 v = __ldg(s4 + i);
            put(4 * i, v.x); put(4 * i + 1, v.y); put(4 * i + 2, v.z); put(4 * i + 3, v.w);
        }
        for (int i = (total & ~3) + threadIdx.x; i < total; i += kPlyImportThreads) put(i, __ldg(src + i));
    }
    __syncthreads();

    const int t = threadIdx.x;
    if (t < cnt) {
        const float *r = rows + t * PS;
        const double s = d.scale;
        // means: M^T p s + c
        const double p[3] = {r[d.col_xyz[0]], r[d.col_xyz[1]], r[d.col_xyz[2]]};
#pragma unroll
        for (int j = 0; j < 3; ++j)
            om[t * 3 + j] = (float)(fma(d.frame[j] * p[0] + d.frame[3 + j] * p[1] + d.frame[6 + j] * p[2], s,
                                        d.center[j]));

        // covariance: s^2 (R^T M)^T diag(exp(2 l)) (R^T M)
        double qw = r[d.col_rot[0]], qx = r[d.col_rot[1]], qy = r[d.col_rot[2]], qz = r[d.col_rot[3]];
        const double qn = qw * qw + qx * qx + qy * qy + qz * qz;
        if (qn > 0.0) {
            const double inv = 1.0 / sqrt(qn);
            qw *= inv; qx *= inv; qy *= inv; qz *= inv;
        } else {
            qw = 1.0;   // a zero quaternion is the identity rotation
        }
        const double rot[3][3] = {{1.0 - 2.0 * (qy * qy + qz * qz), 2.0 * (qx * qy - qw * qz), 2.0 * (qx * qz + qw * qy)},
                                  {2.0 * (qx * qy + qw * qz), 1.0 - 2.0 * (qx * qx + qz * qz), 2.0 * (qy * qz - qw * qx)},
                                  {2.0 * (qx * qz - qw * qy), 2.0 * (qy * qz + qw * qx), 1.0 - 2.0 * (qx * qx + qy * qy)}};
        double var[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) var[k] = exp(2.0 * (double)r[d.col_scale[k]]) * (s * s);
        double b[3][3];   // b = R^T M: row k is column k of R mapped back by M^T
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int j = 0; j < 3; ++j)
                b[k][j] = rot[0][k] * d.frame[j] + rot[1][k] * d.frame[3 + j] + rot[2][k] * d.frame[6 + j];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = i; j < 3; ++j) {
                const float v = (float)(var[0] * b[0][i] * b[0][j] + var[1] * b[1][i] * b[1][j] +
                                        var[2] * b[2][i] * b[2][j]);
                oc[t * 9 + 3 * i + j] = v;
                oc[t * 9 + 3 * j + i] = v;
            }

        oo[t] = (float)(1.0 / (1.0 + exp(-(double)r[d.col_opacity])));

        // harmonics: per channel and degree, the block of the transform times the file's coefficients
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float *h = oh + t * HS + c * C;
#pragma unroll
            for (int l = 0; l <= DEG; ++l) {
                const int b0 = l * l, n = 2 * l + 1, off = l * (4 * l * l - 1) / 3;   // sum of (2k+1)^2, k < l
#pragma unroll
                for (int i = 0; i < n; ++i) {
                    double acc = 0.0;
#pragma unroll
                    for (int j = 0; j < n; ++j) {
                        const int k = b0 + j;
                        const float f = k == 0 ? r[d.col_dc[c]] : r[d.col_rest[c * (NC - 1) + k - 1]];
                        acc = fma((double)d.sh_transform[off + i * n + j], (double)f, acc);
                    }
                    h[b0 + i] = (float)acc;
                }
            }
            for (int k = NC; k < C; ++k) h[k] = 0.0f;
        }
    }
    __syncthreads();

    store_range(d.means + g0 * 3, om, cnt * 3, 3, 3);
    store_range(d.covariances + g0 * 9, oc, cnt * 9, 9, 9);
    store_range(d.opacities + g0, oo, cnt, 1, 1);
    store_range(d.harmonics + g0 * 3 * C, oh, cnt * 3 * C, 3 * C, HS);
}

static int check_ply_import(const ps_ply_import_desc *d) {
    if (!d) {
        set_error("ps_ply_unpack: desc is NULL");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->n_gaussians < 1) {
        set_error("ps_ply_unpack: n_gaussians %lld < 1", (long long)d->n_gaussians);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->sh_degree < 0 || d->sh_degree > 3) {
        set_error("ps_ply_unpack: sh_degree %d outside [0, 3]", d->sh_degree);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const int nc = (d->sh_degree + 1) * (d->sh_degree + 1);
    if (d->sh_coeffs < nc || d->sh_coeffs > PS_PLY_IMPORT_MAX_COEFFS) {
        set_error("ps_ply_unpack: sh_coeffs %d outside [(sh_degree + 1)^2 = %d, %d]", d->sh_coeffs, nc,
                  PS_PLY_IMPORT_MAX_COEFFS);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->n_props < 1 || d->n_props > PS_PLY_IMPORT_MAX_PROPERTIES) {
        set_error("ps_ply_unpack: n_props %d outside [1, %d]", d->n_props, PS_PLY_IMPORT_MAX_PROPERTIES);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const int nrest = 3 * (nc - 1);
    const struct { const int32_t *cols; int n; const char *name; } cols[] = {
        {d->col_xyz, 3, "col_xyz"}, {d->col_dc, 3, "col_dc"}, {d->col_rest, nrest, "col_rest"},
        {&d->col_opacity, 1, "col_opacity"}, {d->col_scale, 3, "col_scale"}, {d->col_rot, 4, "col_rot"}};
    for (const auto &c : cols)
        for (int i = 0; i < c.n; ++i)
            if (c.cols[i] < 0 || c.cols[i] >= d->n_props) {
                set_error("ps_ply_unpack: %s[%d] = %d outside [0, n_props = %d)", c.name, i, c.cols[i], d->n_props);
                return PS_ERR_INVALID_ARGUMENT;
            }
    const struct { const void *p; const char *name; } ptrs[] = {
        {d->records, "records"}, {d->means, "means"}, {d->covariances, "covariances"}, {d->harmonics, "harmonics"},
        {d->opacities, "opacities"}};
    for (const auto &p : ptrs) {
        if (!p.p) {
            set_error("ps_ply_unpack: %s is NULL", p.name);
            return PS_ERR_INVALID_ARGUMENT;
        }
        if (reinterpret_cast<uintptr_t>(p.p) % 16 != 0) {
            set_error("ps_ply_unpack: %s is not 16-byte aligned", p.name);
            return PS_ERR_INVALID_ARGUMENT;
        }
    }
    return PS_OK;
}

template <int DEG>
static int launch_unpack(const ps_ply_import_desc &d, dim3 grid, cudaStream_t st) {
    const size_t smem = sizeof(float) * ply_import_smem_floats(d.n_props, d.sh_coeffs);
    if (smem > 48 * 1024)
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_ply_unpack<DEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_ply_unpack<DEG><<<grid, kPlyImportThreads, smem, st>>>(d);
    PS_LAUNCH_CHECK("k_ply_unpack");
    return PS_OK;
}

}  // namespace ps

extern "C" PS_API int ps_ply_unpack(const ps_ply_import_desc *desc, void *stream) {
    const int rc = ps::check_ply_import(desc);
    if (rc != PS_OK) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long blocks = (desc->n_gaussians + ps::kPlyImportThreads - 1) / ps::kPlyImportThreads;
    if (blocks > 0x7fffffffLL) {
        ps::set_error("ps_ply_unpack: %lld Gaussians are too many for one call", (long long)desc->n_gaussians);
        return PS_ERR_UNSUPPORTED;
    }
    const dim3 grid((unsigned)blocks);
    switch (desc->sh_degree) {
        case 0: return ps::launch_unpack<0>(*desc, grid, st);
        case 1: return ps::launch_unpack<1>(*desc, grid, st);
        case 2: return ps::launch_unpack<2>(*desc, grid, st);
        default: return ps::launch_unpack<3>(*desc, grid, st);
    }
}
