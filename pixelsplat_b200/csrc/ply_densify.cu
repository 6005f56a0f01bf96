// PLY densification: 3DGS's adaptive density control on the vertex records of a refinement (the contract is in
// include/pixelsplat_b200.h, ps_ply_densify_*).
//
//   stats   one thread per Gaussian folds its views' screen-space gradient norms into accum / count: V 16 B read
//           (d_means2d and radii), 8 B read and 8 B written per Gaussian.
//   count   one thread per Gaussian decides keep / clone / split from its opacity, log-scales, accum and count (20 B
//           read, 1 B of flags written); ballots give each 64-record CTA its three segment totals, and one CTA then
//           scans the totals in CTA order into per-CTA segment offsets and the four counts the host reads.
//   apply   the CTAs of count, again: a CTA stages its records with ps_ply_unpack's 16-byte loads, forms the split
//           copies' positions and log-scales, and writes each segment's rows, which are contiguous because every
//           segment keeps input order.  The moments follow through the same staging; new rows get zeros.
#include <cmath>

#include "ply_stage.cuh"

namespace ps {

constexpr int kStatsThreads = 256;
constexpr int kScanThreads = 1024;
enum : uint8_t { kKeep = 1, kClone = 2, kSplit = 4 };

// Workspace: the flags (n bytes, padded to 16) then the per-CTA segment totals, scanned into offsets in place
// ([ctas, 3] int64).
static long long densify_ctas(long long n) { return (n + kPlyImportThreads - 1) / kPlyImportThreads; }
static size_t densify_offsets_at(long long n) { return ((size_t)n + 15) & ~(size_t)15; }
static size_t densify_workspace(long long n) { return densify_offsets_at(n) + (size_t)densify_ctas(n) * 3 * 8; }

struct DensifyParams {
    ps_ply_densify_desc d;
    float grad_threshold;               // float32, as 3DGS compares its float32 gradient norms
    double log_split;                   // log(1.6): the copies' scale is the original's / (0.8 N), N = 2
    signed char slot[PS_PLY_REFINE_MAX_PROPERTIES];   // column -> 0..2 position, 3..5 log-scale, -1 copied
};

__global__ void __launch_bounds__(kStatsThreads) k_ply_densify_stats(long long n, int views, const float *dm2,
                                                                      const int *radii, float *accum, int *count) {
    const long long i = (long long)blockIdx.x * kStatsThreads + threadIdx.x;
    if (i >= n) return;
    float a = accum[i];
    int c = count[i];
    for (int v = 0; v < views; ++v) {
        const long long k = (long long)v * n + i;
        if (__ldg(radii + k) > 0) {   // an off-screen row of d_means2d is not written by the backward
            const double x = __ldg(dm2 + 3 * k), y = __ldg(dm2 + 3 * k + 1);
            a += (float)sqrt(x * x + y * y);
            ++c;
        }
    }
    accum[i] = a;
    count[i] = c;
}

__device__ __forceinline__ double max_scale(const float l[3]) {
    return fmax(fmax(exp((double)l[0]), exp((double)l[1])), exp((double)l[2]));
}

__global__ void __launch_bounds__(kPlyImportThreads) k_ply_densify_count(const DensifyParams p, const float *records,
                                                                          const float *accum, const int *count,
                                                                          uint8_t *flags, long long *totals) {
    const ps_ply_densify_desc &d = p.d;
    const long long i = (long long)blockIdx.x * kPlyImportThreads + threadIdx.x;
    uint8_t f = 0;
    if (i < d.n_gaussians) {
        const float *r = records + i * d.n_props;
        const float l[3] = {__ldg(r + d.col_scale[0]), __ldg(r + d.col_scale[1]), __ldg(r + d.col_scale[2])};
        const int c = count[i];
        const float g = c > 0 ? accum[i] / (float)c : 0.0f;
        const double s = max_scale(l);
        const bool selected = g >= p.grad_threshold, big = s > d.percent_dense * d.extent;
        const bool transparent = 1.0 / (1.0 + exp(-(double)__ldg(r + d.col_opacity))) < d.min_opacity;
        const double world = 0.1 * d.extent;
        if (selected && big) {
            const float l2[3] = {(float)((double)l[0] - p.log_split), (float)((double)l[1] - p.log_split),
                                 (float)((double)l[2] - p.log_split)};
            if (!(transparent || (d.prune_world && max_scale(l2) > world))) f = kSplit;
        } else if (!(transparent || (d.prune_world && s > world))) {
            f = selected ? kKeep | kClone : kKeep;
        }
        flags[i] = f;
    }
    const unsigned keep = __ballot_sync(~0u, f & kKeep), clone = __ballot_sync(~0u, f & kClone),
                   split = __ballot_sync(~0u, f & kSplit);
    __shared__ int warp_totals[kPlyImportThreads / 32][3];
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        warp_totals[warp][0] = __popc(keep);
        warp_totals[warp][1] = __popc(clone);
        warp_totals[warp][2] = __popc(split);
    }
    __syncthreads();
    if (threadIdx.x < 3) totals[(long long)blockIdx.x * 3 + threadIdx.x] = warp_totals[0][threadIdx.x] + warp_totals[1][threadIdx.x];
}

// One CTA: the [ctas, 3] totals scanned in CTA order into exclusive offsets within each segment, in place, and
// counts = {kept originals, clones, splits, n_new}.
__global__ void __launch_bounds__(kScanThreads) k_ply_densify_scan(long long ctas, long long *totals,
                                                                    long long *counts) {
    __shared__ long long warp_sums[kScanThreads / 32][3];
    __shared__ long long carry[3];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t < 3) carry[t] = 0;
    __syncthreads();
    for (long long base = 0; base < ctas; base += kScanThreads) {
        const long long i = base + t;
        long long v[3], x[3];
#pragma unroll
        for (int s = 0; s < 3; ++s) {
            v[s] = i < ctas ? totals[i * 3 + s] : 0;
            x[s] = v[s];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const long long y = __shfl_up_sync(~0u, x[s], o);
                if (lane >= o) x[s] += y;
            }
            if (lane == 31) warp_sums[warp][s] = x[s];
        }
        __syncthreads();
        if (warp == 0) {
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                long long w = warp_sums[lane][s];
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const long long y = __shfl_up_sync(~0u, w, o);
                    if (lane >= o) w += y;
                }
                warp_sums[lane][s] = w;   // inclusive over warps
            }
        }
        __syncthreads();
#pragma unroll
        for (int s = 0; s < 3; ++s) {
            const long long before = carry[s] + (warp ? warp_sums[warp - 1][s] : 0) + x[s] - v[s];
            if (i < ctas) totals[i * 3 + s] = before;
        }
        __syncthreads();
        if (t < 3) carry[t] += warp_sums[kScanThreads / 32 - 1][t];
        __syncthreads();
    }
    if (t == 0) {
        counts[0] = carry[0];
        counts[1] = carry[1];
        counts[2] = carry[2];
        counts[3] = carry[0] + carry[1] + 2 * carry[2];
    }
}

struct ApplyArgs {
    const float *records, *m, *v, *eps;
    const uint8_t *flags;
    const long long *offsets, *counts;
    float *records_out, *m_out, *v_out;
};

// `rows` [n_rows, P] of a segment to dst: row j is staged row src[j]; with `split`, the columns of slot[] >= 0 come
// from split[src[j] * 6 + slot].
__device__ __forceinline__ void write_rows(float *dst, const float *staged, const int *src, int n_rows, int P, int PS,
                                           const signed char *slot, const float *split) {
    for (int e = threadIdx.x; e < n_rows * P; e += kPlyImportThreads) {
        const int j = e / P, c = e - j * P, row = src[j];
        float x = staged[row * PS + c];
        if (split && slot[c] >= 0) x = split[row * 6 + slot[c]];
        dst[e] = x;
    }
}

__device__ __forceinline__ void zero_rows(float *dst, long long count) {
    for (long long e = threadIdx.x; e < count; e += kPlyImportThreads) dst[e] = 0.0f;
}

__global__ void __launch_bounds__(kPlyImportThreads) k_ply_densify_apply(const DensifyParams p, const ApplyArgs a) {
    const ps_ply_densify_desc &d = p.d;
    extern __shared__ float4 smem4[];
    const int P = d.n_props, PS = odd(P);
    float *rows = reinterpret_cast<float *>(smem4);     // [64, PS]
    __shared__ float split[2][kPlyImportThreads * 6];    // per copy and row: p'[3], l'[3]
    __shared__ int src[3][kPlyImportThreads];            // the staged rows of each segment, in order
    __shared__ unsigned warp_bits[kPlyImportThreads / 32][3];
    __shared__ signed char slot[PS_PLY_REFINE_MAX_PROPERTIES];

    const long long n = d.n_gaussians, g0 = (long long)blockIdx.x * kPlyImportThreads;
    const int cnt = (int)min((long long)kPlyImportThreads, n - g0);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint8_t f = t < cnt ? a.flags[g0 + t] : 0;
    const unsigned bits[3] = {__ballot_sync(~0u, f & kKeep), __ballot_sync(~0u, f & kClone),
                              __ballot_sync(~0u, f & kSplit)};
    if (lane == 0)
        for (int s = 0; s < 3; ++s) warp_bits[warp][s] = bits[s];
    for (int c = t; c < P; c += kPlyImportThreads) slot[c] = p.slot[c];
    load_range(rows, a.records + g0 * P, cnt * P, P, PS);
    __syncthreads();
    int seg_rows[3];
#pragma unroll
    for (int s = 0; s < 3; ++s) {
        const int below = warp ? __popc(warp_bits[0][s]) : 0;
        if ((bits[s] >> lane) & 1u) src[s][below + __popc(bits[s] & ((1u << lane) - 1u))] = t;
        seg_rows[s] = __popc(warp_bits[0][s]) + __popc(warp_bits[1][s]);
    }
    if (f & kSplit) {
        const float *r = rows + t * PS;
        double qw = r[d.col_rot[0]], qx = r[d.col_rot[1]], qy = r[d.col_rot[2]], qz = r[d.col_rot[3]], rot[3][3];
        unit_rotation(qw, qx, qy, qz, rot);
        double s[3], l2[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            s[k] = exp((double)r[d.col_scale[k]]);
            l2[k] = (double)r[d.col_scale[k]] - p.log_split;
        }
#pragma unroll
        for (int copy = 0; copy < 2; ++copy) {
            const float *e = a.eps + ((long long)copy * n + g0 + t) * 3;
            const double se[3] = {s[0] * (double)__ldg(e), s[1] * (double)__ldg(e + 1), s[2] * (double)__ldg(e + 2)};
            float *o = split[copy] + t * 6;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                o[j] = (float)((double)r[d.col_xyz[j]] + (rot[j][0] * se[0] + rot[j][1] * se[1] + rot[j][2] * se[2]));
                o[3 + j] = (float)l2[j];
            }
        }
    }
    __syncthreads();

    // segment starts: kept originals, clones, first copies, second copies
    const long long *off = a.offsets + (long long)blockIdx.x * 3;
    const long long keep0 = off[0], clone0 = a.counts[0] + off[1], split0 = a.counts[0] + a.counts[1] + off[2],
                    split1 = split0 + a.counts[2];
    write_rows(a.records_out + keep0 * P, rows, src[0], seg_rows[0], P, PS, slot, nullptr);
    write_rows(a.records_out + clone0 * P, rows, src[1], seg_rows[1], P, PS, slot, nullptr);
    write_rows(a.records_out + split0 * P, rows, src[2], seg_rows[2], P, PS, slot, split[0]);
    write_rows(a.records_out + split1 * P, rows, src[2], seg_rows[2], P, PS, slot, split[1]);
#pragma unroll 1
    for (int k = 0; k < 2; ++k) {
        const float *moment = k ? a.v : a.m;
        float *out = k ? a.v_out : a.m_out;
        zero_rows(out + clone0 * P, (long long)seg_rows[1] * P);
        zero_rows(out + split0 * P, (long long)seg_rows[2] * P);
        zero_rows(out + split1 * P, (long long)seg_rows[2] * P);
        if (!seg_rows[0]) continue;   // uniform across the CTA
        __syncthreads();              // the staged rows are still being read
        load_range(rows, moment + g0 * P, cnt * P, P, PS);
        __syncthreads();
        write_rows(out + keep0 * P, rows, src[0], seg_rows[0], P, PS, slot, nullptr);
    }
}

// ---- host --------------------------------------------------------------------------------------------------------

static bool aligned(const void *p, int bytes) { return p && reinterpret_cast<uintptr_t>(p) % bytes == 0; }

#define PS_DENSIFY_REQUIRE(cond, ...)   \
    do {                                \
        if (!(cond)) {                  \
            ps::set_error(__VA_ARGS__); \
            return PS_ERR_INVALID_ARGUMENT; \
        }                               \
    } while (0)

static int check_densify(const char *who, const ps_ply_densify_desc *d, const void *ws, size_t ws_bytes,
                         DensifyParams &p) {
    PS_DENSIFY_REQUIRE(d, "%s: desc is NULL", who);
    PS_DENSIFY_REQUIRE(d->n_gaussians >= 1, "%s: n_gaussians %lld < 1", who, (long long)d->n_gaussians);
    PS_DENSIFY_REQUIRE(densify_ctas(d->n_gaussians) <= 0x7fffffffLL, "%s: %lld Gaussians are too many for one call",
                       who, (long long)d->n_gaussians);
    PS_DENSIFY_REQUIRE(d->n_props >= 1 && d->n_props <= PS_PLY_REFINE_MAX_PROPERTIES,
                       "%s: n_props %d outside [1, %d]", who, d->n_props, PS_PLY_REFINE_MAX_PROPERTIES);
    const struct { const int32_t *cols; int n; const char *name; } cols[] = {
        {d->col_xyz, 3, "col_xyz"}, {&d->col_opacity, 1, "col_opacity"}, {d->col_scale, 3, "col_scale"},
        {d->col_rot, 4, "col_rot"}};
    for (const auto &c : cols)
        for (int i = 0; i < c.n; ++i)
            PS_DENSIFY_REQUIRE(c.cols[i] >= 0 && c.cols[i] < d->n_props, "%s: %s[%d] = %d outside [0, n_props = %d)",
                               who, c.name, i, c.cols[i], d->n_props);
    const struct { double v; const char *name; } thresholds[] = {
        {d->grad_threshold, "grad_threshold"}, {d->percent_dense, "percent_dense"},
        {d->min_opacity, "min_opacity"}, {d->extent, "extent"}};
    for (const auto &x : thresholds)
        PS_DENSIFY_REQUIRE(std::isfinite(x.v) && x.v >= 0.0, "%s: %s %g is negative or not finite", who, x.name, x.v);
    PS_DENSIFY_REQUIRE(d->extent > 0.0, "%s: extent %g is not positive", who, d->extent);
    PS_DENSIFY_REQUIRE(aligned(ws, 16), "%s: workspace is NULL or not 16-byte aligned", who);
    PS_DENSIFY_REQUIRE(ws_bytes >= densify_workspace(d->n_gaussians), "%s: workspace of %zu bytes, %zu needed", who,
                       ws_bytes, densify_workspace(d->n_gaussians));
    p.d = *d;
    p.grad_threshold = (float)d->grad_threshold;
    p.log_split = std::log(1.6);
    for (int c = 0; c < PS_PLY_REFINE_MAX_PROPERTIES; ++c) p.slot[c] = -1;
    for (int k = 0; k < 3; ++k) {
        p.slot[d->col_xyz[k]] = (signed char)k;
        p.slot[d->col_scale[k]] = (signed char)(3 + k);
    }
    return PS_OK;
}

}  // namespace ps

extern "C" PS_API int ps_ply_densify_workspace_bytes(int64_t n_gaussians, size_t *bytes) {
    if (!bytes || n_gaussians < 1) {
        ps::set_error("ps_ply_densify_workspace_bytes: bytes is NULL or n_gaussians %lld < 1", (long long)n_gaussians);
        return PS_ERR_INVALID_ARGUMENT;
    }
    *bytes = ps::densify_workspace(n_gaussians);
    return PS_OK;
}

extern "C" PS_API int ps_ply_densify_stats(int64_t n_gaussians, int32_t n_views, const float *d_means2d,
                                           const int32_t *radii, float *accum, int32_t *count, void *stream) {
    const char *who = "ps_ply_densify_stats";
    PS_DENSIFY_REQUIRE(n_gaussians >= 1 && n_views >= 1, "%s: n_gaussians %lld or n_views %d < 1", who,
                       (long long)n_gaussians, n_views);
    PS_DENSIFY_REQUIRE((n_gaussians + ps::kStatsThreads - 1) / ps::kStatsThreads <= 0x7fffffffLL,
                       "%s: %lld Gaussians are too many for one call", who, (long long)n_gaussians);
    const struct { const void *p; const char *name; } ptrs[] = {
        {d_means2d, "d_means2d"}, {radii, "radii"}, {accum, "accum"}, {count, "count"}};
    for (const auto &q : ptrs) PS_DENSIFY_REQUIRE(ps::aligned(q.p, 4), "%s: %s is NULL or misaligned", who, q.name);
    const unsigned blocks = (unsigned)((n_gaussians + ps::kStatsThreads - 1) / ps::kStatsThreads);
    ps::k_ply_densify_stats<<<blocks, ps::kStatsThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        n_gaussians, n_views, d_means2d, radii, accum, count);
    PS_LAUNCH_CHECK("k_ply_densify_stats");
    return PS_OK;
}

extern "C" PS_API int ps_ply_densify_count(const ps_ply_densify_desc *desc, const float *records, const float *accum,
                                           const int32_t *count, void *workspace, size_t workspace_bytes,
                                           int64_t *counts, void *stream) {
    const char *who = "ps_ply_densify_count";
    ps::DensifyParams p;
    const int rc = ps::check_densify(who, desc, workspace, workspace_bytes, p);
    if (rc != PS_OK) return rc;
    const struct { const void *p; int align; const char *name; } ptrs[] = {
        {records, 16, "records"}, {accum, 4, "accum"}, {count, 4, "count"}, {counts, 8, "counts"}};
    for (const auto &q : ptrs)
        PS_DENSIFY_REQUIRE(ps::aligned(q.p, q.align), "%s: %s is NULL or misaligned", who, q.name);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long ctas = ps::densify_ctas(desc->n_gaussians);
    uint8_t *flags = static_cast<uint8_t *>(workspace);
    long long *totals = reinterpret_cast<long long *>(flags + ps::densify_offsets_at(desc->n_gaussians));
    ps::k_ply_densify_count<<<(unsigned)ctas, ps::kPlyImportThreads, 0, st>>>(p, records, accum, count, flags, totals);
    PS_LAUNCH_CHECK("k_ply_densify_count");
    ps::k_ply_densify_scan<<<1, ps::kScanThreads, 0, st>>>(ctas, totals, reinterpret_cast<long long *>(counts));
    PS_LAUNCH_CHECK("k_ply_densify_scan");
    return PS_OK;
}

extern "C" PS_API int ps_ply_densify_apply(const ps_ply_densify_desc *desc, const float *records,
                                           const float *exp_avg, const float *exp_avg_sq, const float *eps,
                                           const void *workspace, size_t workspace_bytes, const int64_t *counts,
                                           float *records_out, float *exp_avg_out, float *exp_avg_sq_out,
                                           void *stream) {
    const char *who = "ps_ply_densify_apply";
    ps::DensifyParams p;
    const int rc = ps::check_densify(who, desc, workspace, workspace_bytes, p);
    if (rc != PS_OK) return rc;
    const struct { const void *p; int align; const char *name; } ptrs[] = {
        {records, 16, "records"}, {exp_avg, 16, "exp_avg"}, {exp_avg_sq, 16, "exp_avg_sq"}, {eps, 4, "eps"},
        {counts, 8, "counts"}, {records_out, 16, "records_out"}, {exp_avg_out, 16, "exp_avg_out"},
        {exp_avg_sq_out, 16, "exp_avg_sq_out"}};
    for (const auto &q : ptrs)
        PS_DENSIFY_REQUIRE(ps::aligned(q.p, q.align), "%s: %s is NULL or misaligned", who, q.name);
    const long long n = desc->n_gaussians, ctas = ps::densify_ctas(n);
    const uint8_t *flags = static_cast<const uint8_t *>(workspace);
    const ps::ApplyArgs a{records, exp_avg, exp_avg_sq, eps, flags,
                          reinterpret_cast<const long long *>(flags + ps::densify_offsets_at(n)),
                          reinterpret_cast<const long long *>(counts), records_out, exp_avg_out, exp_avg_sq_out};
    const size_t smem = sizeof(float) * ps::kPlyImportThreads * ps::odd(desc->n_props);
    if (smem > 48 * 1024)
        PS_CUDA_CHECK(cudaFuncSetAttribute(ps::k_ply_densify_apply, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)smem));
    ps::k_ply_densify_apply<<<(unsigned)ctas, ps::kPlyImportThreads, smem, static_cast<cudaStream_t>(stream)>>>(p, a);
    PS_LAUNCH_CHECK("k_ply_densify_apply");
    return PS_OK;
}
