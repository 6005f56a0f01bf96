// PLY import: the vertex records of a 3D Gaussian splatting PLY file unpacked into one scene's Gaussians (the
// contract is in include/pixelsplat_b200.h, ps_ply_unpack).  ps_ply_pack's store pattern, reversed: the CTA loads its
// records, which are one contiguous range of the input, with 16-byte loads into shared memory; every thread turns
// its record into its Gaussian's outputs in shared memory; the CTA stores each output array's contiguous range as
// 16-byte vectors.  The kernel is bound by HBM traffic: 248 B read and 244 B written per Gaussian at degree 3 with
// normals in and 16 coefficients out.
//
// The file's SH degree is a template parameter, so every index into the staged record's columns and the SH
// transform is a compile-time constant.
//
// ps_ply_refine_step (one Adam step of test-time refinement) has the same structure: it also stages the gradients
// of the unpack's outputs, forms each record's gradient (unpack_record_backward), updates the CTA's record entries
// and moments in file order, and unpacks the updated records through the same unpack_record.
#include "adam.cuh"
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

// What the covariance of a record is made of: the normalised quaternion (identity for a zero one), R(q^), the
// variances s^2 exp(2 l) and b = R^T M (row k is column k of R mapped back by M^T).
struct RecordShape {
    double qw, qx, qy, qz, qn;
    double rot[3][3], var[3], b[3][3];
};

__device__ __forceinline__ void record_shape(const ps_ply_import_desc &d, const float *r, RecordShape &o) {
    const double s = d.scale;
    double qw = r[d.col_rot[0]], qx = r[d.col_rot[1]], qy = r[d.col_rot[2]], qz = r[d.col_rot[3]];
    const double qn = qw * qw + qx * qx + qy * qy + qz * qz;
    if (qn > 0.0) {
        const double inv = 1.0 / sqrt(qn);
        qw *= inv; qx *= inv; qy *= inv; qz *= inv;
    } else {
        qw = 1.0;   // a zero quaternion is the identity rotation
    }
    o.qw = qw; o.qx = qx; o.qy = qy; o.qz = qz; o.qn = qn;
    const double rot[3][3] = {{1.0 - 2.0 * (qy * qy + qz * qz), 2.0 * (qx * qy - qw * qz), 2.0 * (qx * qz + qw * qy)},
                              {2.0 * (qx * qy + qw * qz), 1.0 - 2.0 * (qx * qx + qz * qz), 2.0 * (qy * qz - qw * qx)},
                              {2.0 * (qx * qz - qw * qy), 2.0 * (qy * qz + qw * qx), 1.0 - 2.0 * (qx * qx + qy * qy)}};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) o.rot[i][j] = rot[i][j];
#pragma unroll
    for (int k = 0; k < 3; ++k) o.var[k] = exp(2.0 * (double)r[d.col_scale[k]]) * (s * s);
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            o.b[k][j] = rot[0][k] * d.frame[j] + rot[1][k] * d.frame[3 + j] + rot[2][k] * d.frame[6 + j];
}

// One record `r` (staged) to its Gaussian: means om[3], covariances oc[9], opacity *oo, harmonics oh[3 C] (channel
// c at oh + c C).  The per-record code of both ps_ply_unpack and ps_ply_refine_step.
template <int DEG>
__device__ __forceinline__ void unpack_record(const ps_ply_import_desc &d, const float *r, int C, float *om,
                                              float *oc, float *oo, float *oh) {
    constexpr int NC = (DEG + 1) * (DEG + 1);   // coefficients per channel in the file
    const double s = d.scale;
    // means: M^T p s + c
    const double p[3] = {r[d.col_xyz[0]], r[d.col_xyz[1]], r[d.col_xyz[2]]};
#pragma unroll
    for (int j = 0; j < 3; ++j)
        om[j] = (float)(fma(d.frame[j] * p[0] + d.frame[3 + j] * p[1] + d.frame[6 + j] * p[2], s, d.center[j]));

    // covariance: s^2 (R^T M)^T diag(exp(2 l)) (R^T M)
    RecordShape q;
    record_shape(d, r, q);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = i; j < 3; ++j) {
            const float v = (float)(q.var[0] * q.b[0][i] * q.b[0][j] + q.var[1] * q.b[1][i] * q.b[1][j] +
                                    q.var[2] * q.b[2][i] * q.b[2][j]);
            oc[3 * i + j] = v;
            oc[3 * j + i] = v;
        }

    *oo = (float)(1.0 / (1.0 + exp(-(double)r[d.col_opacity])));

    // harmonics: per channel and degree, the block of the transform times the file's coefficients
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float *h = oh + c * C;
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

template <int DEG>
__global__ void __launch_bounds__(kPlyImportThreads) k_ply_unpack(const ps_ply_import_desc d) {
    extern __shared__ float4 smem4[];
    const int P = d.n_props, C = d.sh_coeffs, PS = odd(P), HS = odd(3 * C);
    float *rows = reinterpret_cast<float *>(smem4);    // [64, PS]
    float *om = rows + kPlyImportThreads * PS;         // means [64, 3]
    float *oc = om + kPlyImportThreads * 3;            // covariances [64, 9]
    float *oo = oc + kPlyImportThreads * 9;            // opacities [64]
    float *oh = oo + kPlyImportThreads;                // harmonics [64, HS], [3, C] used

    const long long g0 = (long long)blockIdx.x * kPlyImportThreads;
    const int cnt = (int)min((long long)kPlyImportThreads, d.n_gaussians - g0);
    // the CTA's records: cnt P floats from g0 P, 16-byte aligned (64 P floats per CTA), into rows of PS
    load_range(rows, d.records + g0 * P, cnt * P, P, PS);
    __syncthreads();

    const int t = threadIdx.x;
    if (t < cnt) unpack_record<DEG>(d, rows + t * PS, C, om + t * 3, oc + t * 9, oo + t, oh + t * HS);
    __syncthreads();

    store_range(d.means + g0 * 3, om, cnt * 3, 3, 3);
    store_range(d.covariances + g0 * 9, oc, cnt * 9, 9, 9);
    store_range(d.opacities + g0, oo, cnt, 1, 1);
    store_range(d.harmonics + g0 * 3 * C, oh, cnt * 3 * C, 3 * C, HS);
}

// ---- refinement step ----------------------------------------------------------------------------------------------

struct RefineParams {
    ps_ply_import_desc u;
    float *records_out, *m, *v;
    const float *dm, *dc, *dh, *dop;
    float *d_records;
    AdamConsts k;
    float bc2_sqrt;
    uint32_t read[PS_PLY_REFINE_MAX_PROPERTIES / 32];   // bit c: the unpack reads column c
    float step_size[PS_PLY_REFINE_MAX_PROPERTIES];      // lr[c] / (1 - beta1^t), rounded once
};

__host__ __device__ constexpr int ply_refine_smem_floats(int n_props, int sh_coeffs) {
    return ply_import_smem_floats(n_props, sh_coeffs) + kPlyImportThreads * odd(n_props) + n_props;
}

// The gradient of one record (staged `r`) from its Gaussian's gradients (staged: gm[3], gc[9], *go, gh[3 C]),
// formed in float64 and rounded once, into g[] at the record's columns.  Columns the unpack does not read are left.
template <int DEG>
__device__ __forceinline__ void unpack_record_backward(const ps_ply_import_desc &d, const float *r, int C,
                                                       const float *gm, const float *gc, const float *go,
                                                       const float *gh, float *g) {
    constexpr int NC = (DEG + 1) * (DEG + 1);
    const double s = d.scale;
    // means: d_p = s M d_mean
#pragma unroll
    for (int i = 0; i < 3; ++i)
        g[d.col_xyz[i]] = (float)(s * (d.frame[3 * i] * (double)gm[0] + d.frame[3 * i + 1] * (double)gm[1] +
                                       d.frame[3 * i + 2] * (double)gm[2]));

    // covariance = sum_k var_k b_k b_k^T, so with S = (dSigma + dSigma^T) / 2: d var_k = b_k^T S b_k,
    // d b_k = 2 var_k S b_k, d l_k = 2 var_k d var_k, dR = M db^T
    RecordShape q;
    record_shape(d, r, q);
    double S[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) S[i][j] = 0.5 * ((double)gc[3 * i + j] + (double)gc[3 * j + i]);
    double db[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        double sb[3], quad = 0.0;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            sb[i] = S[i][0] * q.b[k][0] + S[i][1] * q.b[k][1] + S[i][2] * q.b[k][2];
            quad += q.b[k][i] * sb[i];
        }
        g[d.col_scale[k]] = (float)(2.0 * q.var[k] * quad);
#pragma unroll
        for (int j = 0; j < 3; ++j) db[k][j] = 2.0 * q.var[k] * sb[j];
    }
    double dR[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int k = 0; k < 3; ++k)
            dR[i][k] = d.frame[3 * i] * db[k][0] + d.frame[3 * i + 1] * db[k][1] + d.frame[3 * i + 2] * db[k][2];
    const double w = q.qw, x = q.qx, y = q.qy, z = q.qz;
    const double dw = 2.0 * (-z * dR[0][1] + y * dR[0][2] + z * dR[1][0] - x * dR[1][2] - y * dR[2][0] + x * dR[2][1]);
    const double dx = 2.0 * (y * dR[0][1] + z * dR[0][2] + y * dR[1][0] - 2.0 * x * dR[1][1] - w * dR[1][2] +
                             z * dR[2][0] + w * dR[2][1] - 2.0 * x * dR[2][2]);
    const double dy = 2.0 * (-2.0 * y * dR[0][0] + x * dR[0][1] + w * dR[0][2] + x * dR[1][0] + z * dR[1][2] -
                             w * dR[2][0] + z * dR[2][1] - 2.0 * y * dR[2][2]);
    const double dz = 2.0 * (-2.0 * z * dR[0][0] - w * dR[0][1] + x * dR[0][2] + w * dR[1][0] - 2.0 * z * dR[1][1] +
                             y * dR[1][2] + x * dR[2][0] + y * dR[2][1]);
    double dq[4] = {0.0, 0.0, 0.0, 0.0};   // a zero quaternion: the identity, which does not depend on q
    if (q.qn > 0.0) {
        const double inv = 1.0 / sqrt(q.qn), dot = w * dw + x * dx + y * dy + z * dz;
        dq[0] = (dw - w * dot) * inv;
        dq[1] = (dx - x * dot) * inv;
        dq[2] = (dy - y * dot) * inv;
        dq[3] = (dz - z * dot) * inv;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) g[d.col_rot[i]] = (float)dq[i];

    const double o = 1.0 / (1.0 + exp(-(double)r[d.col_opacity]));
    g[d.col_opacity] = (float)((double)*go * o * (1.0 - o));

    // harmonics: T_l^T d_h per channel and degree (the channel loop kept rolled: unrolled, degree 3 spills)
#pragma unroll 1
    for (int c = 0; c < 3; ++c) {
        const float *h = gh + c * C;
#pragma unroll
        for (int l = 0; l <= DEG; ++l) {
            const int b0 = l * l, n = 2 * l + 1, off = l * (4 * l * l - 1) / 3;
#pragma unroll
            for (int j = 0; j < n; ++j) {
                double acc = 0.0;
#pragma unroll
                for (int i = 0; i < n; ++i) acc = fma((double)d.sh_transform[off + i * n + j], (double)h[b0 + i], acc);
                const int k = b0 + j;
                g[k == 0 ? d.col_dc[c] : d.col_rest[c * (NC - 1) + k - 1]] = (float)acc;
            }
        }
    }
}

template <int DEG>
__global__ void __launch_bounds__(kPlyImportThreads) k_ply_refine_step(const RefineParams prm) {
    const ps_ply_import_desc &d = prm.u;
    extern __shared__ float4 smem4[];
    const int P = d.n_props, C = d.sh_coeffs, PS = odd(P), HS = odd(3 * C);
    float *rows = reinterpret_cast<float *>(smem4);    // records [64, PS]
    float *om = rows + kPlyImportThreads * PS;         // d_means, then means [64, 3]
    float *oc = om + kPlyImportThreads * 3;            // d_covariances, then covariances [64, 9]
    float *oo = oc + kPlyImportThreads * 9;            // d_opacities, then opacities [64]
    float *oh = oo + kPlyImportThreads;                // d_harmonics, then harmonics [64, HS]
    float *grows = oh + kPlyImportThreads * HS;        // record gradients [64, PS]
    float *steps = grows + kPlyImportThreads * PS;     // step size per column, -1 for a column Adam leaves [P]

    const long long g0 = (long long)blockIdx.x * kPlyImportThreads;
    const int cnt = (int)min((long long)kPlyImportThreads, d.n_gaussians - g0);
    const int t = threadIdx.x;
    load_range(rows, d.records + g0 * P, cnt * P, P, PS);
    load_range(om, prm.dm + g0 * 3, cnt * 3, 3, 3);
    load_range(oc, prm.dc + g0 * 9, cnt * 9, 9, 9);
    load_range(oo, prm.dop + g0, cnt, 1, 1);
    load_range(oh, prm.dh + g0 * 3 * C, cnt * 3 * C, 3 * C, HS);
    for (int c = 0; c < P; ++c) grows[t * PS + c] = 0.0f;
    // per column in shared memory: lanes of a warp ask for different columns, which a kernel parameter serialises
    for (int c = t; c < P; c += kPlyImportThreads)
        steps[c] = (prm.read[c >> 5] >> (c & 31)) & 1u ? prm.step_size[c] : -1.0f;
    __syncthreads();

    if (t < cnt)
        unpack_record_backward<DEG>(d, rows + t * PS, C, om + t * 3, oc + t * 9, oo + t, oh + t * HS, grows + t * PS);
    __syncthreads();

    // Adam over the CTA's cnt P record entries, in file order: the moments go straight between global memory and
    // registers as 16-byte vectors; the updated record goes to global memory and back to its staged row.
    {
        const int total = cnt * P;
        const long long base = g0 * P;
        auto update = [&](int e, float &m, float &v) -> float {
            const int row = e / P, c = e - row * P;
            float &p = rows[row * PS + c];
            const float step = steps[c];
            if (step >= 0.0f) adam(p, grows[row * PS + c], m, v, prm.k, step, prm.bc2_sqrt);
            return p;
        };
        auto grad = [&](int e) { const int row = e / P; return grows[row * PS + e - row * P]; };
        float4 *m4 = reinterpret_cast<float4 *>(prm.m + base), *v4 = reinterpret_cast<float4 *>(prm.v + base);
        float4 *p4 = reinterpret_cast<float4 *>(prm.records_out + base);
        float4 *g4 = prm.d_records ? reinterpret_cast<float4 *>(prm.d_records + base) : nullptr;
        for (int i = t; i < total / 4; i += kPlyImportThreads) {
            float4 m = m4[i], v = v4[i], p;
            p.x = update(4 * i, m.x, v.x);
            p.y = update(4 * i + 1, m.y, v.y);
            p.z = update(4 * i + 2, m.z, v.z);
            p.w = update(4 * i + 3, m.w, v.w);
            m4[i] = m;
            v4[i] = v;
            p4[i] = p;
            if (g4) g4[i] = make_float4(grad(4 * i), grad(4 * i + 1), grad(4 * i + 2), grad(4 * i + 3));
        }
        for (int e = (total & ~3) + t; e < total; e += kPlyImportThreads) {
            float m = prm.m[base + e], v = prm.v[base + e];
            prm.records_out[base + e] = update(e, m, v);
            prm.m[base + e] = m;
            prm.v[base + e] = v;
            if (prm.d_records) prm.d_records[base + e] = grad(e);
        }
    }
    __syncthreads();

    if (t < cnt) unpack_record<DEG>(d, rows + t * PS, C, om + t * 3, oc + t * 9, oo + t, oh + t * HS);
    __syncthreads();

    store_range(d.means + g0 * 3, om, cnt * 3, 3, 3);
    store_range(d.covariances + g0 * 9, oc, cnt * 9, 9, 9);
    store_range(d.opacities + g0, oo, cnt, 1, 1);
    store_range(d.harmonics + g0 * 3 * C, oh, cnt * 3 * C, 3 * C, HS);
}

static int check_ply_import(const ps_ply_import_desc *d, const char *who = "ps_ply_unpack") {
    if (!d) {
        set_error("%s: desc is NULL", who);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->n_gaussians < 1) {
        set_error("%s: n_gaussians %lld < 1", who, (long long)d->n_gaussians);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->sh_degree < 0 || d->sh_degree > 3) {
        set_error("%s: sh_degree %d outside [0, 3]", who, d->sh_degree);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const int nc = (d->sh_degree + 1) * (d->sh_degree + 1);
    if (d->sh_coeffs < nc || d->sh_coeffs > PS_PLY_IMPORT_MAX_COEFFS) {
        set_error("%s: sh_coeffs %d outside [(sh_degree + 1)^2 = %d, %d]", who, d->sh_coeffs, nc,
                  PS_PLY_IMPORT_MAX_COEFFS);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->n_props < 1 || d->n_props > PS_PLY_IMPORT_MAX_PROPERTIES) {
        set_error("%s: n_props %d outside [1, %d]", who, d->n_props, PS_PLY_IMPORT_MAX_PROPERTIES);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const int nrest = 3 * (nc - 1);
    const struct { const int32_t *cols; int n; const char *name; } cols[] = {
        {d->col_xyz, 3, "col_xyz"}, {d->col_dc, 3, "col_dc"}, {d->col_rest, nrest, "col_rest"},
        {&d->col_opacity, 1, "col_opacity"}, {d->col_scale, 3, "col_scale"}, {d->col_rot, 4, "col_rot"}};
    for (const auto &c : cols)
        for (int i = 0; i < c.n; ++i)
            if (c.cols[i] < 0 || c.cols[i] >= d->n_props) {
                set_error("%s: %s[%d] = %d outside [0, n_props = %d)", who, c.name, i, c.cols[i], d->n_props);
                return PS_ERR_INVALID_ARGUMENT;
            }
    const struct { const void *p; const char *name; } ptrs[] = {
        {d->records, "records"}, {d->means, "means"}, {d->covariances, "covariances"}, {d->harmonics, "harmonics"},
        {d->opacities, "opacities"}};
    for (const auto &p : ptrs) {
        if (!p.p) {
            set_error("%s: %s is NULL", who, p.name);
            return PS_ERR_INVALID_ARGUMENT;
        }
        if (reinterpret_cast<uintptr_t>(p.p) % 16 != 0) {
            set_error("%s: %s is not 16-byte aligned", who, p.name);
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

// The columns the unpack reads, as a bit set; -1 when a column is read twice.
static int read_columns(const ps_ply_import_desc &d, uint32_t *bits) {
    const int nc = (d.sh_degree + 1) * (d.sh_degree + 1);
    for (int i = 0; i < PS_PLY_REFINE_MAX_PROPERTIES / 32; ++i) bits[i] = 0;
    auto mark = [&](int c) {
        if ((bits[c >> 5] >> (c & 31)) & 1u) return c;
        bits[c >> 5] |= 1u << (c & 31);
        return -1;
    };
    int twice = -1;
    for (int i = 0; i < 3; ++i) twice = max(twice, max(mark(d.col_xyz[i]), mark(d.col_dc[i])));
    for (int i = 0; i < 3 * (nc - 1); ++i) twice = max(twice, mark(d.col_rest[i]));
    twice = max(twice, mark(d.col_opacity));
    for (int i = 0; i < 3; ++i) twice = max(twice, mark(d.col_scale[i]));
    for (int i = 0; i < 4; ++i) twice = max(twice, mark(d.col_rot[i]));
    return twice;
}

static int check_ply_refine(const ps_ply_refine_desc *d, RefineParams &prm) {
    const char *who = "ps_ply_refine_step";
    if (!d) {
        set_error("%s: desc is NULL", who);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const int rc = check_ply_import(&d->unpack, who);
    if (rc != PS_OK) return rc;
    const ps_ply_import_desc &u = d->unpack;
    if (u.n_props > PS_PLY_REFINE_MAX_PROPERTIES) {
        set_error("%s: n_props %d above %d", who, u.n_props, PS_PLY_REFINE_MAX_PROPERTIES);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const struct { const void *p; const char *name; bool nullable; } ptrs[] = {
        {d->records_out, "records_out", false}, {d->exp_avg, "exp_avg", false}, {d->exp_avg_sq, "exp_avg_sq", false},
        {d->d_means, "d_means", false}, {d->d_covariances, "d_covariances", false},
        {d->d_harmonics, "d_harmonics", false}, {d->d_opacities, "d_opacities", false},
        {d->d_records, "d_records", true}};
    for (const auto &p : ptrs) {
        if (!p.p && !p.nullable) {
            set_error("%s: %s is NULL", who, p.name);
            return PS_ERR_INVALID_ARGUMENT;
        }
        if (reinterpret_cast<uintptr_t>(p.p) % 16 != 0) {
            set_error("%s: %s is not 16-byte aligned", who, p.name);
            return PS_ERR_INVALID_ARGUMENT;
        }
    }
    if (d->step < 1) {
        set_error("%s: step %lld < 1", who, (long long)d->step);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (!(d->beta1 >= 0.0 && d->beta1 < 1.0) || !(d->beta2 >= 0.0 && d->beta2 < 1.0) || !(d->eps >= 0.0) ||
        !isfinite(d->eps)) {
        set_error("%s: betas %g %g outside [0, 1) or eps %g not finite and >= 0", who, d->beta1, d->beta2, d->eps);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const int twice = read_columns(u, prm.read);
    if (twice >= 0) {
        set_error("%s: column %d is read as two fields", who, twice);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const double bc1 = 1.0 - pow(d->beta1, (double)d->step);
    for (int c = 0; c < u.n_props; ++c) {
        const bool read = (prm.read[c >> 5] >> (c & 31)) & 1u;
        if (read && !(d->lr[c] >= 0.0 && isfinite(d->lr[c]))) {
            set_error("%s: lr[%d] = %g is negative or not finite", who, c, d->lr[c]);
            return PS_ERR_INVALID_ARGUMENT;
        }
        prm.step_size[c] = read ? (float)(d->lr[c] / bc1) : 0.0f;
    }
    prm.u = u;
    prm.records_out = d->records_out;
    prm.m = d->exp_avg;
    prm.v = d->exp_avg_sq;
    prm.dm = d->d_means;
    prm.dc = d->d_covariances;
    prm.dh = d->d_harmonics;
    prm.dop = d->d_opacities;
    prm.d_records = d->d_records;
    prm.k = {(float)(1.0 - d->beta1), (float)d->beta2, (float)(1.0 - d->beta2), (float)d->eps};
    prm.bc2_sqrt = (float)sqrt(1.0 - pow(d->beta2, (double)d->step));
    return PS_OK;
}

template <int DEG>
static int launch_refine(const RefineParams &prm, dim3 grid, cudaStream_t st) {
    const size_t smem = sizeof(float) * ply_refine_smem_floats(prm.u.n_props, prm.u.sh_coeffs);
    if (smem > 48 * 1024)
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_ply_refine_step<DEG>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)smem));
    k_ply_refine_step<DEG><<<grid, kPlyImportThreads, smem, st>>>(prm);
    PS_LAUNCH_CHECK("k_ply_refine_step");
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

extern "C" PS_API int ps_ply_refine_step(const ps_ply_refine_desc *desc, void *stream) {
    ps::RefineParams prm;
    const int rc = ps::check_ply_refine(desc, prm);
    if (rc != PS_OK) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long blocks = (desc->unpack.n_gaussians + ps::kPlyImportThreads - 1) / ps::kPlyImportThreads;
    if (blocks > 0x7fffffffLL) {
        ps::set_error("ps_ply_refine_step: %lld Gaussians are too many for one call",
                      (long long)desc->unpack.n_gaussians);
        return PS_ERR_UNSUPPORTED;
    }
    const dim3 grid((unsigned)blocks);
    switch (desc->unpack.sh_degree) {
        case 0: return ps::launch_refine<0>(prm, grid, st);
        case 1: return ps::launch_refine<1>(prm, grid, st);
        case 2: return ps::launch_refine<2>(prm, grid, st);
        default: return ps::launch_refine<3>(prm, grid, st);
    }
}
