// PLY export: one scene's Gaussians packed into the vertex records of a 3D Gaussian splatting PLY file (the contract
// is in include/pixelsplat_b200.h, ps_ply_pack).  One thread per Gaussian, kPlyThreads Gaussians per CTA.  The CTA
// first stages the SH coefficients its records use (coalesced loads of each Gaussian's [3, sh_coeffs] rows), then
// every thread builds its record in shared memory, and the CTA stores its records, which are contiguous in the
// output, as 16-byte vectors.  The kernel is bound by HBM traffic: about 350 B read and 68 or 248 B written per
// Gaussian at SH degree 4 in and 3 out.
//
// The record layout is templated on the mode and the written SH degree, so every index into the record, the staged
// coefficients and the descriptor's SH transform is a compile-time constant: nothing is copied to local memory.
#include "ps_common.cuh"

namespace ps {

constexpr int kPlyThreads = 64;
constexpr double kPlyOpacityEps = 1e-7;

// One Jacobi rotation in the (P, Q) plane of the symmetric 3x3 matrix a, zeroing a[P][Q]; v accumulates the rotations
// (its columns become the eigenvectors).
template <int P, int Q>
__device__ __forceinline__ void jacobi_rotate(double (&a)[3][3], double (&v)[3][3]) {
    const double apq = a[P][Q];
    if (apq == 0.0) return;
    const double theta = (a[Q][Q] - a[P][P]) / (2.0 * apq);
    // |theta| so large that theta^2 overflows: t = 0, and a[P][Q] is negligible next to the diagonal
    const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(fma(theta, theta, 1.0)));
    const double c = 1.0 / sqrt(fma(t, t, 1.0)), s = t * c;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double akp = a[k][P], akq = a[k][Q];
        a[k][P] = c * akp - s * akq;
        a[k][Q] = s * akp + c * akq;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double apk = a[P][k], aqk = a[Q][k];
        a[P][k] = c * apk - s * aqk;
        a[Q][k] = s * apk + c * aqk;
    }
    a[P][Q] = a[Q][P] = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double vkp = v[k][P], vkq = v[k][Q];
        v[k][P] = c * vkp - s * vkq;
        v[k][Q] = s * vkp + c * vkq;
    }
}

// Cyclic Jacobi: a becomes diagonal (the eigenvalues), v holds the eigenvectors as columns.
__device__ __forceinline__ void jacobi_eigen(double (&a)[3][3], double (&v)[3][3]) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) v[i][j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 16; ++sweep) {
        const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
        const double diag = fabs(a[0][0]) + fabs(a[1][1]) + fabs(a[2][2]);
        if (!(off > 1e-300) || off <= 1e-18 * diag) break;
        jacobi_rotate<0, 1>(a, v);
        jacobi_rotate<0, 2>(a, v);
        jacobi_rotate<1, 2>(a, v);
    }
}

// Rotation matrix -> unit quaternion (x, y, z, w) by the branch on the largest of the diagonal and the trace (the
// method scipy's Rotation.from_matrix uses, which the reference's exporter calls), with w >= 0.
__device__ __forceinline__ double4 matrix_to_quat(const double (&m)[3][3]) {
    const double tr = m[0][0] + m[1][1] + m[2][2];
    int choice = 0;
    double best = m[0][0];
    if (m[1][1] > best) { choice = 1; best = m[1][1]; }
    if (m[2][2] > best) { choice = 2; best = m[2][2]; }
    if (tr > best) choice = 3;
    double x, y, z, w;
    if (choice == 0) {
        x = 1.0 - tr + 2.0 * m[0][0]; y = m[1][0] + m[0][1]; z = m[2][0] + m[0][2]; w = m[2][1] - m[1][2];
    } else if (choice == 1) {
        y = 1.0 - tr + 2.0 * m[1][1]; z = m[2][1] + m[1][2]; x = m[0][1] + m[1][0]; w = m[0][2] - m[2][0];
    } else if (choice == 2) {
        z = 1.0 - tr + 2.0 * m[2][2]; x = m[0][2] + m[2][0]; y = m[1][2] + m[2][1]; w = m[1][0] - m[0][1];
    } else {
        x = m[2][1] - m[1][2]; y = m[0][2] - m[2][0]; z = m[1][0] - m[0][1]; w = 1.0 + tr;
    }
    const double r = (w < 0.0 ? -1.0 : 1.0) / sqrt(x * x + y * y + z * z + w * w);
    return make_double4(x * r, y * r, z * r, w * r);
}

template <int MODE, int DEG>
__global__ void __launch_bounds__(kPlyThreads) k_ply_pack(const ps_ply_desc d, float *__restrict__ out) {
    constexpr int NC = MODE == PS_PLY_VIEWER ? (DEG + 1) * (DEG + 1) : 1;   // coefficients per channel written
    constexpr int NF = 17 + 3 * (NC - 1);                                    // floats per record
    constexpr int OPA = 9 + 3 * (NC - 1);                                    // opacity, then 3 scales, 4 rotations
    __shared__ float coef[kPlyThreads * 3 * NC];
    __shared__ __align__(16) float rec[kPlyThreads * NF];

    const long long g0 = (long long)blockIdx.x * kPlyThreads;
    const int cnt = (int)min((long long)kPlyThreads, d.n_gaussians - g0);
    const int sc = d.sh_coeffs;
    for (int i = threadIdx.x; i < cnt * 3 * NC; i += kPlyThreads) {
        const int row = i / NC;                                   // (Gaussian, channel) row of harmonics
        coef[i] = __ldg(d.harmonics + (g0 * 3 + row) * sc + (i - row * NC));
    }
    __syncthreads();

    const int t = threadIdx.x;
    if (t < cnt) {
        const long long g = g0 + t;
        float *r = rec + t * NF;
        const float s = __ldg(d.scale);
        // the reference centres, divides and rotates in float32, in that order
        float dm[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) dm[k] = __fdiv_rn(__fsub_rn(__ldg(d.means + 3 * g + k), __ldg(d.center + k)), s);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            r[i] = __fmaf_rn((float)d.frame[3 * i + 2], dm[2],
                             __fmaf_rn((float)d.frame[3 * i + 1], dm[1], __fmul_rn((float)d.frame[3 * i], dm[0])));
            r[3 + i] = 0.0f;
        }
        double rot[3][3];
        if (MODE == PS_PLY_REFERENCE) {
#pragma unroll
            for (int c = 0; c < 3; ++c) r[6 + c] = coef[t * 3 + c];
            r[OPA] = __ldg(d.opacities + g);
#pragma unroll
            for (int k = 0; k < 3; ++k) r[OPA + 1 + k] = logf(__fdiv_rn(__ldg(d.scales + 3 * g + k), s));
            double x = __ldg(d.rotations + 4 * g), y = __ldg(d.rotations + 4 * g + 1);
            double z = __ldg(d.rotations + 4 * g + 2), w = __ldg(d.rotations + 4 * g + 3);
            const double n = 1.0 / sqrt(x * x + y * y + z * z + w * w);
            x *= n; y *= n; z *= n; w *= n;
            const double q[3][3] = {{1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - z * w), 2.0 * (x * z + y * w)},
                                    {2.0 * (x * y + z * w), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - x * w)},
                                    {2.0 * (x * z - y * w), 2.0 * (y * z + x * w), 1.0 - 2.0 * (x * x + y * y)}};
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int j = 0; j < 3; ++j)
                    rot[i][j] = d.frame[3 * i] * q[0][j] + d.frame[3 * i + 1] * q[1][j] + d.frame[3 * i + 2] * q[2][j];
        } else {
            // SH: per channel and degree, the block of the transform times the staged coefficients
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float *h = coef + (t * 3 + c) * NC;
#pragma unroll
                for (int l = 0; l <= DEG; ++l) {
                    const int b0 = l * l, n = 2 * l + 1, off = l * (4 * l * l - 1) / 3;   // sum of (2k+1)^2, k < l
#pragma unroll
                    for (int i = 0; i < n; ++i) {
                        float acc = 0.0f;
#pragma unroll
                        for (int j = 0; j < n; ++j) acc = __fmaf_rn(d.sh_transform[off + i * n + j], h[b0 + j], acc);
                        const int k = b0 + i;
                        r[k == 0 ? 6 + c : 9 + c * (NC - 1) + k - 1] = acc;
                    }
                }
            }
            const double o = fmin(fmax((double)__ldg(d.opacities + g), kPlyOpacityEps), 1.0 - kPlyOpacityEps);
            r[OPA] = (float)log(o / (1.0 - o));
            // A = M Sigma M^T / s^2 on the upper triangle of Sigma
            const float *cv = d.covariances + 9 * g;
            const double c00 = __ldg(cv), c01 = __ldg(cv + 1), c02 = __ldg(cv + 2), c11 = __ldg(cv + 4),
                         c12 = __ldg(cv + 5), c22 = __ldg(cv + 8);
            const double sig[3][3] = {{c00, c01, c02}, {c01, c11, c12}, {c02, c12, c22}};
            const double is2 = 1.0 / ((double)s * (double)s);
            double ms[3][3], a[3][3];
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int j = 0; j < 3; ++j)
                    ms[i][j] = d.frame[3 * i] * sig[0][j] + d.frame[3 * i + 1] * sig[1][j] + d.frame[3 * i + 2] * sig[2][j];
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int j = 0; j < 3; ++j)
                    a[i][j] = (ms[i][0] * d.frame[3 * j] + ms[i][1] * d.frame[3 * j + 1] + ms[i][2] * d.frame[3 * j + 2]) * is2;
            jacobi_eigen(a, rot);
            const double det = rot[0][0] * (rot[1][1] * rot[2][2] - rot[1][2] * rot[2][1]) -
                               rot[0][1] * (rot[1][0] * rot[2][2] - rot[1][2] * rot[2][0]) +
                               rot[0][2] * (rot[1][0] * rot[2][1] - rot[1][1] * rot[2][0]);
            if (det < 0.0) {
#pragma unroll
                for (int k = 0; k < 3; ++k) rot[k][2] = -rot[k][2];
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) r[OPA + 1 + k] = (float)(0.5 * log(fmax(a[k][k], PS_PLY_MIN_EIGENVALUE)));
        }
        const double4 q = matrix_to_quat(rot);
        r[OPA + 4] = (float)q.w;
        r[OPA + 5] = (float)q.x;
        r[OPA + 6] = (float)q.y;
        r[OPA + 7] = (float)q.z;
    }
    __syncthreads();

    // the CTA's records are one contiguous, 16-byte aligned range of the output (g0 NF floats in)
    const int total = cnt * NF;
    float *o = out + g0 * NF;
    const float4 *src = reinterpret_cast<const float4 *>(rec);
    float4 *dst = reinterpret_cast<float4 *>(o);
    for (int i = threadIdx.x; i < total / 4; i += kPlyThreads) dst[i] = src[i];
    for (int i = (total & ~3) + threadIdx.x; i < total; i += kPlyThreads) o[i] = rec[i];
}

static int check_ply(const ps_ply_desc *d, const float *out) {
    if (!d || !out) {
        set_error("ps_ply_pack: %s is NULL", d ? "out" : "desc");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->mode != PS_PLY_REFERENCE && d->mode != PS_PLY_VIEWER) {
        set_error("ps_ply_pack: unknown mode %d", d->mode);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->n_gaussians < 1) {
        set_error("ps_ply_pack: n_gaussians %lld < 1", (long long)d->n_gaussians);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const int max_deg = d->mode == PS_PLY_VIEWER ? 3 : 0;
    if (d->sh_degree < 0 || d->sh_degree > max_deg) {
        set_error("ps_ply_pack: sh_degree %d outside [0, %d]", d->sh_degree, max_deg);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->sh_coeffs < (d->sh_degree + 1) * (d->sh_degree + 1)) {
        set_error("ps_ply_pack: sh_coeffs %d < (sh_degree + 1)^2 = %d", d->sh_coeffs,
                  (d->sh_degree + 1) * (d->sh_degree + 1));
        return PS_ERR_INVALID_ARGUMENT;
    }
    const bool ref = d->mode == PS_PLY_REFERENCE;
    const struct { const void *p; const char *name; } need[] = {
        {d->means, "means"}, {d->harmonics, "harmonics"}, {d->opacities, "opacities"}, {d->center, "center"},
        {d->scale, "scale"}, {ref ? (const void *)d->scales : d->covariances, ref ? "scales" : "covariances"},
        {ref ? (const void *)d->rotations : d->covariances, ref ? "rotations" : "covariances"}};
    for (const auto &n : need)
        if (!n.p) {
            set_error("ps_ply_pack: %s is NULL", n.name);
            return PS_ERR_INVALID_ARGUMENT;
        }
    if (reinterpret_cast<uintptr_t>(out) % 16 != 0) {
        set_error("ps_ply_pack: out is not 16-byte aligned");
        return PS_ERR_INVALID_ARGUMENT;
    }
    return PS_OK;
}

}  // namespace ps

extern "C" PS_API int ps_ply_pack(const ps_ply_desc *desc, float *out, void *stream) {
    const int rc = ps::check_ply(desc, out);
    if (rc != PS_OK) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long blocks = (desc->n_gaussians + ps::kPlyThreads - 1) / ps::kPlyThreads;
    if (blocks > 0x7fffffffLL) {
        ps::set_error("ps_ply_pack: %lld Gaussians are too many for one call", (long long)desc->n_gaussians);
        return PS_ERR_UNSUPPORTED;
    }
    const dim3 grid((unsigned)blocks);
    if (desc->mode == PS_PLY_REFERENCE) {
        ps::k_ply_pack<PS_PLY_REFERENCE, 0><<<grid, ps::kPlyThreads, 0, st>>>(*desc, out);
    } else {
        switch (desc->sh_degree) {
            case 0: ps::k_ply_pack<PS_PLY_VIEWER, 0><<<grid, ps::kPlyThreads, 0, st>>>(*desc, out); break;
            case 1: ps::k_ply_pack<PS_PLY_VIEWER, 1><<<grid, ps::kPlyThreads, 0, st>>>(*desc, out); break;
            case 2: ps::k_ply_pack<PS_PLY_VIEWER, 2><<<grid, ps::kPlyThreads, 0, st>>>(*desc, out); break;
            default: ps::k_ply_pack<PS_PLY_VIEWER, 3><<<grid, ps::kPlyThreads, 0, st>>>(*desc, out); break;
        }
    }
    PS_LAUNCH_CHECK("k_ply_pack");
    return PS_OK;
}
