// Epipolar sampling geometry, one launch for a whole batch: for every (batch, view, other view,
// ray) clip the ray to the other camera's frustum (near/far along the ray, image frame), and for
// each of the S samples on the projected segment compute the depth along the query ray and its
// relative disparity (the input of the depth positional encoding).
//
// Replaces, with identical semantics (SURVEY.md Appendix B steps 1-5):
//   EpipolarSampler.generate_image_rays / project_rays   epipolar_sampler.py:62-88,125-145,
//                                                         geometry/epipolar_lines.py:157-251
//   get_depth -> lift_to_3d -> intersect_rays (lstsq)     epipolar_lines.py:264-292, projection.py:176-230
//   depth clip + depth_to_relative_disparity              epipolar_transformer.py:103-119, conversions.py:17-27
// i.e. ~60 small elementwise torch kernels, 16 boolean-mask scatters (host syncs) and a batched
// lstsq over b*v*ov*r*s 3x3 systems.  The two-ray least-squares point has the closed form
// p = (o1 + t d1 + o2 + s d2)/2 (midpoint of the common perpendicular).
//
// Arithmetic is float64 on purpose: the result feeds a 10-octave positional encoding
// (phase = rd * 2 pi * 2^k, k <= 9), which amplifies fp32 noise of the near-parallel-ray depth
// by up to 3.2e3; the work is a few hundred flops per sample, invisible next to the attention.
#include "ps_common.cuh"

namespace ps {

struct EpiCam {      // per (batch, view), prepared by one thread per block
    double e[16];    // camera-to-world
    double w2c[16];  // inverse
    double k[9];
    double kinv[9];
};

__device__ void inv3d(const double *m, double *o) {
    const double a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
    const double A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
    const double r = 1.0 / (a * A + b * B + c * C);
    o[0] = A * r; o[1] = -(b * i - c * h) * r; o[2] = (b * f - c * e) * r;
    o[3] = B * r; o[4] = (a * i - c * g) * r;  o[5] = -(a * f - c * d) * r;
    o[6] = C * r; o[7] = -(a * h - b * g) * r; o[8] = (a * e - b * d) * r;
}

// Inverse of a 4x4 by Gauss-Jordan with partial pivoting (general, like torch.linalg.inv).
__device__ void inv4d(const double *m, double *out) {
    double a[4][8];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) { a[r][c] = m[4 * r + c]; a[r][4 + c] = r == c ? 1.0 : 0.0; }
    for (int col = 0; col < 4; ++col) {
        int piv = col;
        for (int r = col + 1; r < 4; ++r) if (fabs(a[r][col]) > fabs(a[piv][col])) piv = r;
        if (piv != col) for (int c = 0; c < 8; ++c) { const double t = a[col][c]; a[col][c] = a[piv][c]; a[piv][c] = t; }
        const double inv = 1.0 / a[col][col];
        for (int c = 0; c < 8; ++c) a[col][c] *= inv;
        for (int r = 0; r < 4; ++r) if (r != col) {
            const double f = a[r][col];
            if (f != 0.0) for (int c = 0; c < 8; ++c) a[r][c] -= f * a[col][c];
        }
    }
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) out[4 * r + c] = a[r][4 + c];
}

__device__ void load_cam(const float *extr, const float *intr, EpiCam &c) {
    for (int i = 0; i < 16; ++i) c.e[i] = (double)extr[i];
    for (int i = 0; i < 9; ++i) c.k[i] = (double)intr[i];
    inv4d(c.e, c.w2c);
    inv3d(c.k, c.kinv);
}

struct Proj { double t, x, y; bool valid; };

constexpr double kEps = 1e-6;

__device__ __forceinline__ bool in_bounds(double x, double y) {
    return x >= -kEps && y >= -kEps && x <= 1.0 + kEps && y <= 1.0 + kEps;
}

// Intersection of the projected camera-space ray with the image-frame line  coord[dim] = value.
__device__ Proj frame_hit(const double *k, const double *o, const double *d, int dim, double value) {
    const int od = 1 - dim;
    const double fs = k[4 * dim], fo = k[4 * od], cs = k[3 * dim + 2], co = k[3 * od + 2];
    const double os = o[dim], oo = o[od], ds = d[dim], dd = d[od], oz = o[2], dz = d[2];
    const double c = (value - cs) / fs;
    Proj p;
    p.t = (c * oz - os) / (ds - c * dz);
    const double other = co + fo * (oo * (c * dz - ds) + dd * (os - c * oz)) / (dz * os - ds * oz);
    p.x = dim == 0 ? value : other;
    p.y = dim == 0 ? other : value;
    const double z = oz + p.t * dz;
    p.valid = in_bounds(p.x, p.y) && (z > -kEps) && (p.t > -kEps);
    return p;
}

__device__ __forceinline__ double nan_to_num(double v, double pinf, double ninf) {
    if (v != v) return 0.0;
    if (isinf(v)) return v > 0 ? pinf : ninf;
    return v;
}

// Projection of the camera-space point p, with the ray parameter t it stands for, with the reference's guards
// (project_camera_space: p / (p_z + eps32), nan_to_num(+-1e8)).
__device__ Proj project_point(const double *k, double px, double py, double pz, double t) {
    const double eps32 = 1.1920928955078125e-07;
    const double den = pz + eps32;
    const double qx = nan_to_num(px / den, 1e8, -1e8), qy = nan_to_num(py / den, 1e8, -1e8),
                 qz = nan_to_num(pz / den, 1e8, -1e8);
    Proj p;
    p.t = t;
    p.x = k[0] * qx + k[1] * qy + k[2] * qz;
    p.y = k[3] * qx + k[4] * qy + k[5] * qz;
    p.valid = in_bounds(p.x, p.y) && (pz > -kEps) && (t > -kEps);
    return p;
}

// Projection of the point o + t d (camera space): project_rays' bounded near / far branch.
__device__ Proj point_proj(const double *k, const double *o, const double *d, double t) {
    return project_point(k, o[0] + t * d[0], o[1] + t * d[1], o[2] + t * d[2], t);
}

// project_rays' unbounded near branch, the projection at zero depth: an origin within kEps of the camera centre is
// replaced by the direction; any other origin with z < kEps projects as invalid.
__device__ Proj zero_depth_proj(const double *k, const double *o, const double *d) {
    const bool at_camera = sqrt(o[0] * o[0] + o[1] * o[1] + o[2] * o[2]) < kEps;
    const double *p = at_camera ? d : o;
    Proj r = project_point(k, p[0], p[1], p[2], 0.0);
    if (o[2] < kEps && !at_camera) r.valid = false;
    return r;
}

// project_rays' unbounded far branch, the projection of the direction at infinity.
__device__ Proj infinity_proj(const double *k, const double *d) {
    return project_point(k, d[0], d[1], d[2], INFINITY);
}

// World ray (origin ow, unit direction dw) through the centre of cell r of an h x w grid of camera `cam`
// (sample_image_grid + get_world_rays).
__device__ __forceinline__ void world_ray(const EpiCam &cam, int r, int h, int w, double *ow, double *dw) {
    const double x = ((r % w) + 0.5) / w, y = ((r / w) + 0.5) / h;
    double dc[3];
    for (int i = 0; i < 3; ++i) dc[i] = cam.kinv[3 * i] * x + cam.kinv[3 * i + 1] * y + cam.kinv[3 * i + 2];
    const double dn = sqrt(dc[0] * dc[0] + dc[1] * dc[1] + dc[2] * dc[2]);
    for (int i = 0; i < 3; ++i) dc[i] /= dn;
    for (int i = 0; i < 3; ++i) {
        dw[i] = cam.e[4 * i] * dc[0] + cam.e[4 * i + 1] * dc[1] + cam.e[4 * i + 2] * dc[2];
        ow[i] = cam.e[4 * i + 3];
    }
}

// A world ray in camera `cam`'s space.
__device__ __forceinline__ void to_camera(const EpiCam &cam, const double *ow, const double *dw, double *oc,
                                          double *dcam) {
    for (int i = 0; i < 3; ++i) {
        const double *m = cam.w2c + 4 * i;
        oc[i] = m[0] * ow[0] + m[1] * ow[1] + m[2] * ow[2] + m[3];
        dcam[i] = m[0] * dw[0] + m[1] * dw[1] + m[2] * dw[2];
    }
}

// The ray's intersections with the four lines of the image frame: the first minimum (lo) and first maximum (hi) of
// t over the valid ones, invalid ones ranked +inf / -inf (project_rays' _compare_projections); tmin / tmax are
// those ranked values.
__device__ __forceinline__ void frame_extremes(const double *k, const double *oc, const double *dcam, Proj &lo,
                                               Proj &hi, double &tmin, double &tmax) {
    Proj fr[4] = {frame_hit(k, oc, dcam, 0, 0.0), frame_hit(k, oc, dcam, 0, 1.0),
                  frame_hit(k, oc, dcam, 1, 0.0), frame_hit(k, oc, dcam, 1, 1.0)};
    lo = fr[0];
    hi = fr[0];
    tmin = fr[0].valid ? fr[0].t : INFINITY;
    tmax = fr[0].valid ? fr[0].t : -INFINITY;
#pragma unroll
    for (int i = 1; i < 4; ++i) {
        const double tlo = fr[i].valid ? fr[i].t : INFINITY, thi = fr[i].valid ? fr[i].t : -INFINITY;
        if (tlo < tmin) { tmin = tlo; lo = fr[i]; }
        if (thi > tmax) { tmax = thi; hi = fr[i]; }
    }
}

__global__ void __launch_bounds__(128)
k_epipolar_geometry(int B, int V, int h, int w, int S, const float *__restrict__ extr,
                    const float *__restrict__ intr, const float *__restrict__ near_,
                    const float *__restrict__ far_, float *__restrict__ seg, uint8_t *__restrict__ valid_out,
                    float *__restrict__ rel_disp, float *__restrict__ t_range) {
    __shared__ EpiCam cam_q, cam_o;
    const int OV = V - 1;
    const int bvo = blockIdx.y;                  // ((b * V) + v) * OV + ov
    const int ov = bvo % OV, v = (bvo / OV) % V, b = bvo / (OV * V);
    const int o_view = ov < v ? ov : ov + 1;     // "all other views" index (heterogeneous_pairings.py:9-24)
    if (threadIdx.x == 0) load_cam(extr + 16 * (b * V + v), intr + 9 * (b * V + v), cam_q);
    if (threadIdx.x == 32) load_cam(extr + 16 * (b * V + o_view), intr + 9 * (b * V + o_view), cam_o);
    __syncthreads();
    const int R = h * w;
    if ((int64_t)blockIdx.x * blockDim.x + threadIdx.x >= R) return;
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    const double nearv = (double)near_[b * V + v], farv = (double)far_[b * V + v];

    // --- world ray through the centre of ray-grid cell r of view v, into the other camera's space
    double dw[3], ow[3], oc[3], dcam[3];
    world_ray(cam_q, r, h, w, ow, dw);
    to_camera(cam_o, ow, dw, oc, dcam);
    Proj frame_lo, frame_hi;
    double tmin, tmax;
    frame_extremes(cam_o.k, oc, dcam, frame_lo, frame_hi, tmin, tmax);
    const Proj pn = point_proj(cam_o.k, oc, dcam, nearv), pf = point_proj(cam_o.k, oc, dcam, farv);
    Proj lo = pn.valid ? pn : frame_lo, hi = pf.valid ? pf : frame_hi;
    if (!pn.valid) lo.t = tmin;
    if (!pf.valid) hi.t = tmax;
    const bool overlaps = lo.valid && hi.valid;
    const double m = overlaps ? 1.0 : 0.0;
    const double x0 = nan_to_num(lo.x, 0.0, 0.0) * m, y0 = nan_to_num(lo.y, 0.0, 0.0) * m;
    const double x1 = nan_to_num(hi.x, 0.0, 0.0) * m, y1 = nan_to_num(hi.y, 0.0, 0.0) * m;
    const size_t idx = (size_t)bvo * R + r;
    seg[4 * idx + 0] = (float)x0; seg[4 * idx + 1] = (float)y0;
    seg[4 * idx + 2] = (float)x1; seg[4 * idx + 3] = (float)y1;
    valid_out[idx] = overlaps ? 1 : 0;
    if (t_range) { t_range[2 * idx] = (float)lo.t; t_range[2 * idx + 1] = (float)hi.t; }

    // --- per-sample depth along the query ray (closest point of two rays) -> relative disparity
    const double eps = 1e-10;
    const double disp_near = 1.0 / (nearv + eps), disp_far = 1.0 / (farv + eps);
    for (int s = 0; s < S; ++s) {
        const double u = (s + 0.5) / S;
        // the reference forms the sample in the tensors' dtype (fp32) as a multiply and an add, each rounded: keep
        // its rounding of xy (intrinsics, not operators, so FMA contraction cannot fuse the two)
        const float fx = __fadd_rn((float)x0, __fmul_rn((float)u, (float)x1 - (float)x0));
        const float fy = __fadd_rn((float)y0, __fmul_rn((float)u, (float)y1 - (float)y0));
        double d2c[3], d2[3], o2[3];
        for (int i = 0; i < 3; ++i)
            d2c[i] = cam_o.kinv[3 * i] * (double)fx + cam_o.kinv[3 * i + 1] * (double)fy + cam_o.kinv[3 * i + 2];
        const double n2 = sqrt(d2c[0] * d2c[0] + d2c[1] * d2c[1] + d2c[2] * d2c[2]);
        for (int i = 0; i < 3; ++i) d2c[i] /= n2;
        for (int i = 0; i < 3; ++i) {
            d2[i] = cam_o.e[4 * i] * d2c[0] + cam_o.e[4 * i + 1] * d2c[1] + cam_o.e[4 * i + 2] * d2c[2];
            o2[i] = cam_o.e[4 * i + 3];
        }
        const double c = dw[0] * d2[0] + dw[1] * d2[1] + dw[2] * d2[2];
        double depth;
        if (c > 1.0 - 1e-5) {
            // parallel: the reference sets the point to (1e10, 1e10, 1e10)
            const double ex = 1e10 - ow[0], ey = 1e10 - ow[1], ez = 1e10 - ow[2];
            depth = sqrt(ex * ex + ey * ey + ez * ez);
        } else {
            const double wx = o2[0] - ow[0], wy = o2[1] - ow[1], wz = o2[2] - ow[2];
            const double a = wx * dw[0] + wy * dw[1] + wz * dw[2];
            const double bb = wx * d2[0] + wy * d2[1] + wz * d2[2];
            const double den = 1.0 - c * c;
            const double t = (a - bb * c) / den, sp = (a * c - bb) / den;
            const double qx = 0.5 * (ow[0] + t * dw[0] + o2[0] + sp * d2[0]) - ow[0];
            const double qy = 0.5 * (ow[1] + t * dw[1] + o2[1] + sp * d2[1]) - ow[1];
            const double qz = 0.5 * (ow[2] + t * dw[2] + o2[2] + sp * d2[2]) - ow[2];
            depth = sqrt(qx * qx + qy * qy + qz * qz);
        }
        depth = fmin(fmax(depth, nearv), farv);
        const double disp = 1.0 / (depth + eps);
        rel_disp[idx * S + s] = (float)(1.0 - (disp - disp_far) / (disp_near - disp_far + eps));
    }
}

}  // namespace ps

extern "C" PS_API int ps_epipolar_geometry(int32_t batch, int32_t views, int32_t grid_h, int32_t grid_w,
                                           int32_t samples, const float *extrinsics, const float *intrinsics,
                                           const float *near_plane, const float *far_plane, float *segments,
                                           uint8_t *valid, float *rel_disparity, float *t_range, void *stream) {
    if (batch < 1 || views < 2 || grid_h < 1 || grid_w < 1 || samples < 1 || !extrinsics || !intrinsics ||
        !near_plane || !far_plane || !segments || !valid || !rel_disparity) {
        ps::set_error("ps_epipolar_geometry: bad argument (views must be >= 2, pointers non-NULL)");
        return PS_ERR_INVALID_ARGUMENT;
    }
    // one block row per (batch, view, other view) on the grid's y axis, and a 32-bit ray index
    const int64_t slices = (int64_t)batch * views * (views - 1), rays = (int64_t)grid_h * grid_w;
    if (slices > 65535 || rays > INT32_MAX) {
        ps::set_error("ps_epipolar_geometry: batch * views * (views - 1) must be <= 65535 and grid_h * grid_w < 2^31");
        return PS_ERR_UNSUPPORTED;
    }
    dim3 grid((unsigned)((rays + 127) / 128), (unsigned)slices);
    ps::k_epipolar_geometry<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(
        batch, views, grid_h, grid_w, samples, extrinsics, intrinsics, near_plane, far_plane, segments, valid,
        rel_disparity, t_range);
    PS_LAUNCH_CHECK("k_epipolar_geometry");
    return PS_OK;
}

namespace ps {

constexpr int kOverlapThreads = 128;
constexpr int kOverlapRaysPerThread = 8;

// View overlap of an evaluation-index walk (EvaluationIndexGenerator.test_step): for candidate frame k = first +
// blockIdx.y and direction blockIdx.z, the number of rays of the source camera's h x w grid whose unbounded
// projection (project_rays without near / far) overlaps the destination camera's image.  Direction 0 sends the
// rays of k into camera `context`, direction 1 the rays of `context` into camera k.  Each thread counts up to
// kOverlapRaysPerThread rays; the CTA's count is a warp reduction plus one integer atomic, so the result does not
// depend on the order the CTAs run in.
__global__ void __launch_bounds__(kOverlapThreads)
k_view_overlap(int h, int w, int context, int first, const float *__restrict__ extr, const float *__restrict__ intr,
               int *__restrict__ counts) {
    __shared__ EpiCam cam_src, cam_dst;
    __shared__ int warp_count[kOverlapThreads / 32];
    const int k = first + blockIdx.y, dir = blockIdx.z;
    const int src = dir == 0 ? k : context, dst = dir == 0 ? context : k;
    if (threadIdx.x == 0) load_cam(extr + 16 * src, intr + 9 * src, cam_src);
    if (threadIdx.x == 32) load_cam(extr + 16 * dst, intr + 9 * dst, cam_dst);
    __syncthreads();
    const int R = h * w;
    int n = 0;
    for (int r = blockIdx.x * kOverlapThreads + threadIdx.x; r < R; r += gridDim.x * kOverlapThreads) {
        double ow[3], dw[3], oc[3], dcam[3];
        world_ray(cam_src, r, h, w, ow, dw);
        to_camera(cam_dst, ow, dw, oc, dcam);
        Proj frame_lo, frame_hi;
        double tmin, tmax;
        frame_extremes(cam_dst.k, oc, dcam, frame_lo, frame_hi, tmin, tmax);
        const bool lo = zero_depth_proj(cam_dst.k, oc, dcam).valid || frame_lo.valid;
        const bool hi = infinity_proj(cam_dst.k, dcam).valid || frame_hi.valid;
        n += lo && hi;
    }
    n = __reduce_add_sync(0xffffffffu, n);
    if ((threadIdx.x & 31) == 0) warp_count[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        int total = 0;
        for (int i = 0; i < kOverlapThreads / 32; ++i) total += warp_count[i];
        atomicAdd(counts + 2 * blockIdx.y + dir, total);
    }
}

}  // namespace ps

extern "C" PS_API int ps_view_overlap(int32_t views, int32_t grid_h, int32_t grid_w, const float *extrinsics,
                                      const float *intrinsics, int32_t context, int32_t first, int32_t count,
                                      int32_t *counts, void *stream) {
    if (views < 1 || grid_h < 1 || grid_w < 1 || count < 1 || !extrinsics || !intrinsics || !counts) {
        ps::set_error("ps_view_overlap: bad argument (views, grid and count must be >= 1, pointers non-NULL)");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (context < 0 || context >= views || first < 0 || first > views - count) {
        ps::set_error("ps_view_overlap: the context frame and the candidate range must lie in [0, views)");
        return PS_ERR_INVALID_ARGUMENT;
    }
    // one block row per candidate on the grid's y axis, and a 32-bit ray index
    const int64_t rays = (int64_t)grid_h * grid_w;
    if (count > 65535 || rays > INT32_MAX) {
        ps::set_error("ps_view_overlap: count must be <= 65535 and grid_h * grid_w < 2^31");
        return PS_ERR_UNSUPPORTED;
    }
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    PS_CUDA_CHECK(cudaMemsetAsync(counts, 0, sizeof(int32_t) * 2 * (size_t)count, s));
    const int64_t per_block = (int64_t)ps::kOverlapThreads * ps::kOverlapRaysPerThread;
    dim3 grid((unsigned)((rays + per_block - 1) / per_block), (unsigned)count, 2);
    ps::k_view_overlap<<<grid, ps::kOverlapThreads, 0, s>>>(grid_h, grid_w, context, first, extrinsics, intrinsics,
                                                             counts);
    PS_LAUNCH_CHECK("k_view_overlap");
    return PS_OK;
}
