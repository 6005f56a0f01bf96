// Preprocess backward: one thread per (scene, Gaussian), summing over the scene's V views.
//   dL/dconic -> dL/dcov2D -> dL/dcov3D and dL/dmean (through the projection Jacobian),
//   dL/dmean2D -> dL/dmean (perspective divide), dL/drgb -> dL/dSH and dL/dmean (view direction).
// Semantics: SURVEY.md A.5 (upstream backward.cu computeCov2DCUDA + preprocessCUDA), including
// upstream's 1/(det^2 + 1e-7) and the clamp rule (x/y terms vanish when the +-1.3 tan(fov)
// clamp was active).  Because the thread owns the Gaussian, the per-view gradients are summed
// in registers and every output (300 B of dL/dSH at M = 25) is written exactly once per scene
// instead of once per view -- the reference writes them per view and then lets autograd sum
// the `repeat` (decoder_splatting_cuda.py:53-56).
#include "ps_common.cuh"
#include "raster_math.cuh"

namespace ps {

constexpr int kPreBwdThreads = 128;

// Camera-gradient partial row of (scene s, view v) stored by the warp that owns indices sg0.. of S*P: rows of one
// view are indexed by the warp's position among the warps overlapping the scene, kCamRowFloats floats each:
//   [0..11]  d viewmatrix [0 1 2 | 4 5 6 | 8 9 10 | 12 13 14]
//   [12..23] d projmatrix [0 1 3 | 4 5 7 | 8 9 11 | 12 13 15]
//   [24..26] d campos, [27..28] d tanfov, [29..31] unused
__device__ __forceinline__ float *cam_row(float *ws, const Dims &d, int s, int v, long long sg0) {
    const long long w = sg0 / 32 - ((long long)s * d.P) / 32;
    return ws + ((size_t)(s * d.V + v) * cam_rows_per_view(d.P) + (size_t)w) * kCamRowFloats;
}

// Word kCamEntries of a view's row 0 is k_camera_finish's arrival counter: every producer of a partial row stores all
// kCamRowFloats words, the unused ones as 0, so the counter starts at 0 on every call.
__device__ __forceinline__ unsigned *cam_counter(float *ws, const Dims &d, int vid) {
    return reinterpret_cast<unsigned *>(ws + (size_t)vid * cam_rows_per_view(d.P) * kCamRowFloats) + kCamEntries;
}

// The warp's partial rows of view v: per scene its lanes belong to, the kCamEntries entries summed over those lanes in
// a fixed xor-butterfly order, stored by lane 0 (with the unused words as 0).  A warp whose Gaussians span two scenes
// (P not a multiple of 32) stores one row for each.
__device__ __forceinline__ void store_cam_partials(const float (&cam)[kCamEntries], float *cam_ws, const Dims &d,
                                                   int v, long long sg0, int rows, uint32_t scene, int lane) {
    const int s_lo = (int)(sg0 / d.P), s_hi = (int)((sg0 + rows - 1) / d.P);
    for (int s = s_lo; s <= s_hi; ++s) {
        const bool mine = (int)scene == s;
        float sum[kCamEntries];
#pragma unroll
        for (int k = 0; k < kCamEntries; ++k) {
            float x = mine ? cam[k] : 0.0f;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
            sum[k] = x;
        }
        if (lane == 0) {
            float *r = cam_row(cam_ws, d, s, v, sg0);
#pragma unroll
            for (int k = 0; k < kCamEntries; ++k) r[k] = sum[k];
#pragma unroll
            for (int k = kCamEntries; k < kCamRowFloats; ++k) r[k] = 0.0f;
        }
    }
}

// The gradient math of one on-screen (view, Gaussian) pair, shared by k_preprocess_bwd and k_camera_bwd so that the
// camera gradients of both come out of the same expressions.  The statement order is the one the kernels were tuned
// with (the dcov sums inside the denom2inv branch, then dM, dJ, dL/dt, g, then the perspective terms): computing all
// of dM, dJ and dL/dt before the dcov sums makes k_preprocess_bwd<false, false> spill.  The SH walk that forms
// dL/d(direction) for the campos entries stays written out in each kernel: moved into a shared function or visitor,
// it changed the register allocation and instruction count of every k_preprocess_bwd instantiation.

// What the projection backward of a pair leaves for its callers: dL/dM (rows of M = J W), dL/dJ, the view-space
// gradient dL/dt, the perspective-divide terms, and the pair's gradient (gx, gy, gz) with respect to the scaled mean.
struct PairGrad {
    float dM0[3], dM1[3];
    float dJ00, dJ02, dJ11, dJ12;
    float tz, tz2;                 // 1 / t.z and its square
    float dL_dtx, dL_dty, dL_dtz;
    float m_w, mul1, mul2;         // 1 / (hw + 1e-7), hx m_w^2, hy m_w^2
    float gx, gy, gz;
};

// dL/dconic -> dL/dcov2D -> dL/dM, dL/dJ -> dL/dt -> dL/dmean, plus dL/dmean2D through the perspective divide.
// COV: also adds the pair's dL/dcov3D (upper triangle, unscaled covariance) to dcov.
template <bool COV>
__device__ __forceinline__ PairGrad projection_bwd(const Cov2D &cv, const float (&s6)[6], float sc,
                                                   const float *__restrict__ vm, const float *__restrict__ pm,
                                                   float focal_x, float focal_y, float px, float py, float pz,
                                                   float4 gc, float2 g2, float *dcov) {
    PairGrad q;
    const float a = cv.a, b = cv.b, c = cv.c;
    const float denom = a * c - b * b;
    const float denom2inv = 1.0f / (denom * denom + 0.0000001f);
    float dL_da = 0.0f, dL_db = 0.0f, dL_dc = 0.0f;
    const float *m0 = cv.m0, *m1 = cv.m1;
    if (denom2inv != 0.0f) {
        dL_da = denom2inv * (-c * c * gc.x + 2.0f * b * c * gc.y + (denom - a * c) * gc.z);
        dL_dc = denom2inv * (-a * a * gc.z + 2.0f * a * b * gc.y + (denom - a * c) * gc.x);
        dL_db = denom2inv * 2.0f * (b * c * gc.x - (denom + 2.0f * b * b) * gc.y + a * b * gc.z);
        if constexpr (COV) {
            const float s2 = sc * sc;
            dcov[0] += s2 * (m0[0] * m0[0] * dL_da + m0[0] * m1[0] * dL_db + m1[0] * m1[0] * dL_dc);
            dcov[3] += s2 * (m0[1] * m0[1] * dL_da + m0[1] * m1[1] * dL_db + m1[1] * m1[1] * dL_dc);
            dcov[5] += s2 * (m0[2] * m0[2] * dL_da + m0[2] * m1[2] * dL_db + m1[2] * m1[2] * dL_dc);
            dcov[1] += s2 * (2.0f * m0[0] * m0[1] * dL_da + (m0[0] * m1[1] + m0[1] * m1[0]) * dL_db + 2.0f * m1[0] * m1[1] * dL_dc);
            dcov[2] += s2 * (2.0f * m0[0] * m0[2] * dL_da + (m0[0] * m1[2] + m0[2] * m1[0]) * dL_db + 2.0f * m1[0] * m1[2] * dL_dc);
            dcov[4] += s2 * (2.0f * m0[2] * m0[1] * dL_da + (m0[1] * m1[2] + m0[2] * m1[1]) * dL_db + 2.0f * m1[1] * m1[2] * dL_dc);
        }
    }
    // dL/dM (rows) from a = m0 S m0, b = m0 S m1, c = m1 S m1
    const float S[3][3] = {{s6[0], s6[1], s6[2]}, {s6[1], s6[3], s6[4]}, {s6[2], s6[4], s6[5]}};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float sm0 = m0[0] * S[k][0] + m0[1] * S[k][1] + m0[2] * S[k][2];
        const float sm1 = m1[0] * S[k][0] + m1[1] * S[k][1] + m1[2] * S[k][2];
        q.dM0[k] = 2.0f * sm0 * dL_da + sm1 * dL_db;
        q.dM1[k] = 2.0f * sm1 * dL_dc + sm0 * dL_db;
    }
    q.dJ00 = vm[0] * q.dM0[0] + vm[4] * q.dM0[1] + vm[8] * q.dM0[2];
    q.dJ02 = vm[2] * q.dM0[0] + vm[6] * q.dM0[1] + vm[10] * q.dM0[2];
    q.dJ11 = vm[1] * q.dM1[0] + vm[5] * q.dM1[1] + vm[9] * q.dM1[2];
    q.dJ12 = vm[2] * q.dM1[0] + vm[6] * q.dM1[1] + vm[10] * q.dM1[2];
    q.tz = 1.0f / cv.tz; q.tz2 = q.tz * q.tz;
    const float tz3 = q.tz2 * q.tz;
    q.dL_dtx = cv.clamp_x ? 0.0f : -focal_x * q.tz2 * q.dJ02;
    q.dL_dty = cv.clamp_y ? 0.0f : -focal_y * q.tz2 * q.dJ12;
    q.dL_dtz = -focal_x * q.tz2 * q.dJ00 - focal_y * q.tz2 * q.dJ11 +
               (2.0f * focal_x * cv.ctx) * tz3 * q.dJ02 + (2.0f * focal_y * cv.cty) * tz3 * q.dJ12;
    q.gx = vm[0] * q.dL_dtx + vm[1] * q.dL_dty + vm[2] * q.dL_dtz;
    q.gy = vm[4] * q.dL_dtx + vm[5] * q.dL_dty + vm[6] * q.dL_dtz;
    q.gz = vm[8] * q.dL_dtx + vm[9] * q.dL_dty + vm[10] * q.dL_dtz;

    // screen-space mean through the perspective divide
    const float hx = pm[0] * px + pm[4] * py + pm[8] * pz + pm[12];
    const float hy = pm[1] * px + pm[5] * py + pm[9] * pz + pm[13];
    const float hw = pm[3] * px + pm[7] * py + pm[11] * pz + pm[15];
    q.m_w = 1.0f / (hw + 0.0000001f);
    q.mul1 = hx * q.m_w * q.m_w; q.mul2 = hy * q.m_w * q.m_w;
    q.gx += (pm[0] * q.m_w - pm[3] * q.mul1) * g2.x + (pm[1] * q.m_w - pm[3] * q.mul2) * g2.y;
    q.gy += (pm[4] * q.m_w - pm[7] * q.mul1) * g2.x + (pm[5] * q.m_w - pm[7] * q.mul2) * g2.y;
    q.gz += (pm[8] * q.m_w - pm[11] * q.mul1) * g2.x + (pm[9] * q.m_w - pm[11] * q.mul2) * g2.y;
    return q;
}

// The pair's share of the 26 geometric camera entries (cam_row order: [0..23] and [27..28]):
//   viewmatrix: t = W p + (vm[12], vm[13], vm[14]) and M = J W (W[i][j] = vm[4j+i]);
//   projmatrix: h = pm p (p.w = 1), screen xy from (hx, hy) / (hw + 1e-7);
//   tanfov: only through the focal lengths in J (f = size / (2 tanfov); the clamp limit passes nothing).
__device__ __forceinline__ void camera_geometry_grads(const PairGrad &q, const Cov2D &cv, float px, float py, float pz,
                                                      float2 g2, float focal_x, float focal_y, float tanfovx,
                                                      float tanfovy, float (&cam)[kCamEntries]) {
    const float j00 = focal_x * q.tz, j02 = -focal_x * cv.ctx * q.tz2;
    const float j11 = focal_y * q.tz, j12 = -focal_y * cv.cty * q.tz2;
    const float p[3] = {px, py, pz};
    const float dhx = g2.x * q.m_w, dhy = g2.y * q.m_w, dhw = -(q.mul1 * g2.x + q.mul2 * g2.y);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        cam[3 * j + 0] = q.dM0[j] * j00 + q.dL_dtx * p[j];
        cam[3 * j + 1] = q.dM1[j] * j11 + q.dL_dty * p[j];
        cam[3 * j + 2] = q.dM0[j] * j02 + q.dM1[j] * j12 + q.dL_dtz * p[j];
        cam[12 + 3 * j + 0] = dhx * p[j];
        cam[12 + 3 * j + 1] = dhy * p[j];
        cam[12 + 3 * j + 2] = dhw * p[j];
    }
    cam[9] = q.dL_dtx; cam[10] = q.dL_dty; cam[11] = q.dL_dtz;
    cam[21] = dhx; cam[22] = dhy; cam[23] = dhw;
    cam[27] = (q.dJ00 * q.tz - q.dJ02 * cv.ctx * q.tz2) * (-focal_x / tanfovx);
    cam[28] = (q.dJ11 * q.tz - q.dJ12 * cv.cty * q.tz2) * (-focal_y / tanfovy);
}

// campos entries [24..26]: minus the gradient of the view direction p - campos (dd = p - campos, len2 = |dd|^2,
// inv3 = 1 / |dd|^3, dLd = dL/d(normalised direction) from the SH walk).  Rounded intrinsics: plain products shared
// with the Gaussian's own direction chain in k_preprocess_bwd would change how that is contracted, and the Gaussian
// gradients must keep their bits.
__device__ __forceinline__ void camera_campos_grads(float ddx, float ddy, float ddz, float len2, float inv3,
                                                    float3 dLd, float (&cam)[kCamEntries]) {
    const float dLdx = dLd.x, dLdy = dLd.y, dLdz = dLd.z;
    const float xx = __fmul_rn(ddx, ddx), yy = __fmul_rn(ddy, ddy), zz = __fmul_rn(ddz, ddz);
    const float xy = __fmul_rn(ddx, ddy), xz = __fmul_rn(ddx, ddz), yz = __fmul_rn(ddy, ddz);
    const float ex = __fadd_rn(__fadd_rn(__fmul_rn(__fsub_rn(len2, xx), dLdx), -__fmul_rn(xy, dLdy)), -__fmul_rn(xz, dLdz));
    const float ey = __fadd_rn(__fadd_rn(-__fmul_rn(xy, dLdx), __fmul_rn(__fsub_rn(len2, yy), dLdy)), -__fmul_rn(yz, dLdz));
    const float ez = __fadd_rn(__fadd_rn(-__fmul_rn(xz, dLdx), -__fmul_rn(yz, dLdy)), __fmul_rn(__fsub_rn(len2, zz), dLdz));
    cam[24] = -__fmul_rn(ex, inv3); cam[25] = -__fmul_rn(ey, inv3); cam[26] = -__fmul_rn(ez, inv3);
}

// The depth chain's camera terms: z = (vm[2], vm[6], vm[10]) . mean + vm[14] / sc, dz = dL/dz.
__device__ __forceinline__ void camera_depth_grads(float dz, float mx0, float my0, float mz0, float sc,
                                                   float (&cam)[kCamEntries]) {
    cam[2] += dz * mx0; cam[5] += dz * my0; cam[8] += dz * mz0; cam[11] += dz / sc;
}

// Each warp owns 32 consecutive (scene, Gaussian) indices of S*P and writes every element of their rows of every
// output gradient, which the caller may hand over uninitialised: a Gaussian that is on screen in no view gets zeros,
// and so does every Gaussian when the binning overflowed its capacity (the composite backward then did not run).  A
// warp none of whose Gaussians is on screen only stores zeros.  On screen in view v means radii > 0, the rows
// k_clear_pair_grads cleared and the composite backward accumulated into.  SH rows are staged per warp in shared
// memory: the coefficients of the on-screen lanes come in with cp.async, dL/dSH of all 32 rows goes out as one
// contiguous block.
// DEPTH: the depth value's chain to the means is added (a depth gradient was given); built for 4 resident CTAs so
// that it does not spill.
// CAM: camera gradients are requested.  Each lane also forms its Gaussian's contribution to the kCamEntries camera
// entries of every view it is on screen in; the warp sums them per (scene, view) in a fixed shuffle order and
// stores one partial row per (warp, view) into `cam_ws` (layout: cam_row), zeros included, which k_camera_finish
// sums.  Built for 2 resident CTAs: the 29 partial sums are live beside the colour chain.
template <bool DEPTH, bool CAM>
__global__ void __launch_bounds__(kPreBwdThreads, CAM ? 2 : (DEPTH ? 4 : 5))
k_preprocess_bwd(Dims d, Inputs in, Geom geo, ViewGrads vgr, GaussGrads out, int row_stride, float *cam_ws) {
    extern __shared__ float s_dsh[];   // [warps][32][row_stride] coefficients (V == 1: reused for the gradient)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long sp = (long long)d.S * d.P;
    const long long sg0 = ((long long)blockIdx.x * kPreBwdThreads) + warp * 32;
    if (sg0 >= sp) return;
    const int rows = (int)min((long long)32, sp - sg0);
    const bool live = lane < rows;
    const uint32_t sgi = (uint32_t)(live ? sg0 + lane : sg0);
    const uint32_t scene = sgi / (uint32_t)d.P, g = sgi - scene * (uint32_t)d.P;
    const size_t sg = sgi;
    const int cov_n = d.cov_layout == PS_COV_TRIU6 ? 6 : 9;
    const int sh_n = d.M > 0 ? 3 * d.M : 3;
    const int M = d.M, layout = d.sh_layout;

    bool any = false;
    if (live && *geo.n_instances <= d.capacity)
        for (int v = 0; v < d.V; ++v) any |= geo.radii[(size_t)((int)scene * d.V + v) * d.P + g] > 0;
    const unsigned vis_lanes = __ballot_sync(0xffffffffu, any);
    if (vis_lanes == 0u) {
        for (int e = lane; e < rows * 3; e += 32) out.d_means[3 * sg0 + e] = 0.0f;
        for (int e = lane; e < rows * cov_n; e += 32) out.d_cov[cov_n * sg0 + e] = 0.0f;
        if (lane < rows) out.d_opacities[sg0 + lane] = 0.0f;
        for (int e = lane; e < rows * sh_n; e += 32) out.d_sh[sh_n * sg0 + e] = 0.0f;
        if (out.d_means2d && live)
            for (int v = 0; v < d.V; ++v) {
                float *m2 = out.d_means2d + 3 * ((size_t)((int)scene * d.V + v) * d.P + g);
                m2[0] = 0.0f; m2[1] = 0.0f; m2[2] = 0.0f;
            }
        if (CAM) {
            const int s_lo = (int)(sg0 / d.P), s_hi = (int)((sg0 + rows - 1) / d.P);
            for (int s = s_lo; s <= s_hi; ++s)
                for (int v = 0; v < d.V; ++v) cam_row(cam_ws, d, s, v, sg0)[lane] = 0.0f;
        }
        return;
    }

    float *wrows = s_dsh + (size_t)warp * 32 * row_stride;
    float *row = wrows + lane * row_stride;
    const bool in_place = M > 0 && d.V == 1;     // read each coefficient, then overwrite its slot with the gradient
    float *grow = in_place ? row : row + (size_t)kPreBwdThreads * row_stride;   // separate gradient rows when V > 1

    // the SH rows stream into shared memory while the geometry part below runs; waited for at first use
    if (M > 0) gather_rows_async(in.sh, (unsigned long long)sg, vis_lanes, sh_n, wrows, row_stride, lane);

    float mx0 = 0.0f, my0 = 0.0f, mz0 = 0.0f;
    if (any) { mx0 = in.means[3 * sg + 0]; my0 = in.means[3 * sg + 1]; mz0 = in.means[3 * sg + 2]; }
    const float *covp = in.cov + sg * cov_n;

    float dmx = 0.0f, dmy = 0.0f, dmz = 0.0f, dop = 0.0f;
    float dcov[6] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    float dcol[3] = {0.0f, 0.0f, 0.0f};
    bool sh_written = false, sh_ready = false;

    for (int v = 0; v < d.V; ++v) {
        const int vid = (int)scene * d.V + v;
        const size_t vg = (size_t)vid * d.P + g;
        const bool vis = any && geo.radii[vg] > 0;
        if (live && out.d_means2d) {
            float *m2 = out.d_means2d + 3 * vg;
            const float2 t = vis ? vgr.d_mean2d[vg] : make_float2(0.0f, 0.0f);
            m2[0] = t.x; m2[1] = t.y; m2[2] = 0.0f;
        }
        // (no `continue` for the views this Gaussian is not on screen in: the warp must stay convergent for the
        //  shared-memory hand-over of the SH rows below)
        float gx = 0.0f, gy = 0.0f, gz = 0.0f;
        float4 gcol = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        float cam[CAM ? kCamEntries : 1];   // this Gaussian's share of the view's camera gradient (cam_row order)
        if (CAM) {
#pragma unroll
            for (int k = 0; k < kCamEntries; ++k) cam[k] = 0.0f;
        }
        const float sc = in.scale ? in.scale[vid] : 1.0f;
        const float px = mx0 * sc, py = my0 * sc, pz = mz0 * sc;
        if (vis) {
        const float *__restrict__ vm = in.view + 16 * vid;
        const float *__restrict__ pm = in.proj + 16 * vid;
        const float tanfovx = in.tanfov[2 * vid], tanfovy = in.tanfov[2 * vid + 1];
        const float focal_x = (float)d.W / (2.0f * tanfovx), focal_y = (float)d.H / (2.0f * tanfovy);
        float s6[6];
        load_cov6(covp, d.cov_layout, sc * sc, s6);
        Cov2D cv;
        compute_cov2d(px, py, pz, s6, vm, focal_x, focal_y, tanfovx, tanfovy, cv);

        const float2 g2 = vgr.d_mean2d[vg];
        const float4 gc = vgr.d_conic[vg];
        gcol = vgr.d_color[vg];
        dop += gc.w;

        const PairGrad q = projection_bwd<true>(cv, s6, sc, vm, pm, focal_x, focal_y, px, py, pz, gc, g2, dcov);
        gx = q.gx; gy = q.gy; gz = q.gz;
        if constexpr (CAM) camera_geometry_grads(q, cv, px, py, pz, g2, focal_x, focal_y, tanfovx, tanfovy, cam);
        }   // vis (geometry part)

        if (M > 0 && !sh_ready) {          // warp-uniform; the rows have had the geometry math to arrive
            gather_rows_wait();
            sh_ready = true;
        }
        if (M > 0 && vis) {
            const float cx = in.campos[3 * vid], cy = in.campos[3 * vid + 1], cz = in.campos[3 * vid + 2];
            const float ddx = px - cx, ddy = py - cy, ddz = pz - cz;
            const float len2 = ddx * ddx + ddy * ddy + ddz * ddz;
            const float len = sqrtf(len2);
            const float x = ddx / len, y = ddy / len, z = ddz / len;
            const uint8_t cl = geo.clamped[vg];
            const float dl[3] = {(cl & 1) ? 0.0f : gcol.x, (cl & 2) ? 0.0f : gcol.y, (cl & 4) ? 0.0f : gcol.z};
            float dLda = 0.0f, dLdb = 0.0f, dLdc = 0.0f;
            const bool first = !sh_written;
            const float3 sa = sh_arg(d.sh_basis, x, y, z);
            const uint32_t flip = sh_flip_mask(d.sh_basis);
            sh_for_each(d.deg, sa.x, sa.y, sa.z, [&](int k, float Y, float Ya, float Yb, float Yc) {
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) {
                    const int idx = sh_index(layout, M, k, ch);
                    const float coef = row[idx];
                    const float sdl = sh_sign(flip, k, dl[ch]);      // the term's sign rides on dL/dcolour
                    const float val = Y * sdl;
                    grow[idx] = first ? val : grow[idx] + val;
                    const float cd = coef * sdl;
                    dLda += Ya * cd; dLdb += Yb * cd; dLdc += Yc * cd;
                }
            });
            const float3 dLd = sh_grad_unpermute(d.sh_basis, dLda, dLdb, dLdc);
            const float dLdx = dLd.x, dLdy = dLd.y, dLdz = dLd.z;
            if (first) {
                const int nb = (d.deg + 1) * (d.deg + 1);
                for (int k = nb; k < M; ++k)
                    for (int ch = 0; ch < 3; ++ch) grow[sh_index(layout, M, k, ch)] = 0.0f;
            }
            sh_written = true;
            const float inv3 = 1.0f / (len2 * len);
            gx += ((len2 - ddx * ddx) * dLdx - ddy * ddx * dLdy - ddz * ddx * dLdz) * inv3;
            gy += (-ddx * ddy * dLdx + (len2 - ddy * ddy) * dLdy - ddz * ddy * dLdz) * inv3;
            gz += (-ddx * ddz * dLdx - ddy * ddz * dLdy + (len2 - ddz * ddz) * dLdz) * inv3;
            if constexpr (CAM) camera_campos_grads(ddx, ddy, ddz, len2, inv3, dLd, cam);
        } else if (vis) {
            dcol[0] += gcol.x; dcol[1] += gcol.y; dcol[2] += gcol.z;
        }
        dmx += gx * sc; dmy += gy * sc; dmz += gz * sc;
        if (DEPTH && vis) {
            // depth channel: d = f(z), z = vz / sc = (vm[2], vm[6], vm[10]) . mean + vm[14] / sc, so the chain to the
            // (unscaled) mean carries no scale factor.  Re-read here, after the SH part, to keep registers free there.
            const float *__restrict__ vm = in.view + 16 * vid;
            const float dz = vgr.d_color[vg].w * depth_value_grad(d.depth_mode, geo.depth[vg], in.scale, in.near_far, vid);
            dmx += dz * vm[2]; dmy += dz * vm[6]; dmz += dz * vm[10];
            if constexpr (CAM) camera_depth_grads(dz, mx0, my0, mz0, sc, cam);
        }
        if constexpr (CAM) store_cam_partials(cam, cam_ws, d, v, sg0, rows, scene, lane);
    }

    if (live) {
        out.d_means[3 * sg + 0] = dmx; out.d_means[3 * sg + 1] = dmy; out.d_means[3 * sg + 2] = dmz;
        out.d_opacities[sg] = dop;
        float *dc = out.d_cov + sg * cov_n;
        if (d.cov_layout == PS_COV_TRIU6) {
#pragma unroll
            for (int i = 0; i < 6; ++i) dc[i] = dcov[i];
        } else {
            dc[0] = dcov[0]; dc[1] = dcov[1]; dc[2] = dcov[2];
            dc[3] = 0.0f; dc[4] = dcov[3]; dc[5] = dcov[4];
            dc[6] = 0.0f; dc[7] = 0.0f; dc[8] = dcov[5];      // the lower triangle receives no gradient
        }
        if (M == 0) {
            float *dsh = out.d_sh + sg * 3;
            dsh[0] = dcol[0]; dsh[1] = dcol[1]; dsh[2] = dcol[2];
        }
    }
    if (M > 0) {
        if (!sh_written)                   // on screen in no view: the row was neither fetched nor written
            for (int c = 0; c < sh_n; ++c) grow[c] = 0.0f;
        __syncwarp();
        const float *gsrc = in_place ? wrows : wrows + (size_t)kPreBwdThreads * row_stride;
        store_rows(out.d_sh + (size_t)sg0 * sh_n, rows, sh_n, gsrc, row_stride, lane);
    }
}

// Clears the per-(view, Gaussian) gradient scratch rows of the on-screen pairs (the compact list k_preprocess built):
// those, and only those, are accumulated into by the composite backward (its tile lists hold exactly the listed
// pairs), stored by the fixed-order gather, and read by k_preprocess_bwd (radii > 0 implies listed).  Every other row
// of the scratch is left as it is.  One thread per list entry; the count lives on the device, so the grid is sized
// for the worst case and surplus threads exit at once.
constexpr int kClearThreads = 256;

__global__ void __launch_bounds__(kClearThreads) k_clear_pair_grads(Geom geo, ViewGrads vg) {
    const long long i = (long long)blockIdx.x * kClearThreads + threadIdx.x;
    if (i >= geo.n_instances[2]) return;
    const uint32_t p = geo.vis_pairs[i];
    vg.d_mean2d[p] = make_float2(0.0f, 0.0f);
    vg.d_conic[p] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    vg.d_color[p] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

int launch_clear_pair_grads(const Dims &d, const Geom &g, const ViewGrads &vg, cudaStream_t st) {
    const long long pairs = (long long)d.S * d.V * d.P;
    k_clear_pair_grads<<<(unsigned)((pairs + kClearThreads - 1) / kClearThreads), kClearThreads, 0, st>>>(g, vg);
    PS_LAUNCH_CHECK("k_clear_pair_grads");
    return PS_OK;
}

// Camera-only backward (ps_raster_grads with every Gaussian gradient NULL): the 29 camera entries of k_preprocess_bwd's
// CAM path, formed by the same functions, and nothing else.  One thread per (view, Gaussian) pair; a CTA covers kCamBwdThreads consecutive (scene,
// Gaussian) indices of S*P for ONE view v (blockIdx.x = chunk * V + v: the V CTAs of a chunk run side by side and share
// its SH rows in L2), so each warp stores exactly the partial rows k_preprocess_bwd<·, true> stores for (its 32
// indices, v), summed in the same order, and the same k_camera_finish adds them.  It reads the scratch of the on-screen
// pairs and the means, covariances and (for campos) SH rows of the on-screen lanes only; no Gaussian gradient is formed
// or stored.  Walking the Gaussians, not the compact list of on-screen pairs (whose order changes from run to run),
// keeps every float sum in a fixed order.
constexpr int kCamBwdThreads = 128;

template <bool DEPTH>
__global__ void __launch_bounds__(kCamBwdThreads, 4)
k_camera_bwd(Dims d, Inputs in, Geom geo, ViewGrads vgr, int row_stride, float *cam_ws) {
    extern __shared__ float s_sh[];    // [warps][32][row_stride] SH coefficients of the on-screen lanes
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int v = (int)(blockIdx.x % (unsigned)d.V);
    const long long sp = (long long)d.S * d.P;
    const long long sg0 = (long long)(blockIdx.x / (unsigned)d.V) * kCamBwdThreads + warp * 32;
    if (sg0 >= sp) return;
    const int rows = (int)min((long long)32, sp - sg0);
    const bool live = lane < rows;
    const uint32_t sgi = (uint32_t)(live ? sg0 + lane : sg0);
    const uint32_t scene = sgi / (uint32_t)d.P, g = sgi - scene * (uint32_t)d.P;
    const size_t sg = sgi;
    const int vid = (int)scene * d.V + v;
    const size_t vg = (size_t)vid * d.P + g;
    const int M = d.M, sh_n = 3 * M;

    const bool vis = live && *geo.n_instances <= d.capacity && geo.radii[vg] > 0;
    const unsigned vis_lanes = __ballot_sync(0xffffffffu, vis);
    float cam[kCamEntries];
#pragma unroll
    for (int k = 0; k < kCamEntries; ++k) cam[k] = 0.0f;
    if (vis_lanes == 0u) {
        store_cam_partials(cam, cam_ws, d, v, sg0, rows, scene, lane);
        return;
    }
    float *wrows = s_sh + (size_t)warp * 32 * row_stride;
    const float *row = wrows + lane * row_stride;
    if (M > 0) gather_rows_async(in.sh, (unsigned long long)sg, vis_lanes, sh_n, wrows, row_stride, lane);

    float mx0 = 0.0f, my0 = 0.0f, mz0 = 0.0f;
    const float sc = in.scale ? in.scale[vid] : 1.0f;
    if (vis) {
        mx0 = in.means[3 * sg + 0]; my0 = in.means[3 * sg + 1]; mz0 = in.means[3 * sg + 2];
        const float px = mx0 * sc, py = my0 * sc, pz = mz0 * sc;
        const float *__restrict__ vm = in.view + 16 * vid;
        const float *__restrict__ pm = in.proj + 16 * vid;
        const float tanfovx = in.tanfov[2 * vid], tanfovy = in.tanfov[2 * vid + 1];
        const float focal_x = (float)d.W / (2.0f * tanfovx), focal_y = (float)d.H / (2.0f * tanfovy);
        float s6[6];
        load_cov6(in.cov + sg * (d.cov_layout == PS_COV_TRIU6 ? 6 : 9), d.cov_layout, sc * sc, s6);
        Cov2D cv;
        compute_cov2d(px, py, pz, s6, vm, focal_x, focal_y, tanfovx, tanfovy, cv);
        const float2 g2 = vgr.d_mean2d[vg];
        const float4 gc = vgr.d_conic[vg];
        const PairGrad q = projection_bwd<false>(cv, s6, sc, vm, pm, focal_x, focal_y, px, py, pz, gc, g2, nullptr);
        camera_geometry_grads(q, cv, px, py, pz, g2, focal_x, focal_y, tanfovx, tanfovy, cam);
    }
    if (M > 0) gather_rows_wait();         // warp-uniform
    if (M > 0 && vis) {
        // campos: minus the gradient of the view direction p - campos through the SH evaluation
        const float px = mx0 * sc, py = my0 * sc, pz = mz0 * sc;
        const float4 gcol = vgr.d_color[vg];
        const float cx = in.campos[3 * vid], cy = in.campos[3 * vid + 1], cz = in.campos[3 * vid + 2];
        const float ddx = px - cx, ddy = py - cy, ddz = pz - cz;
        const float len2 = ddx * ddx + ddy * ddy + ddz * ddz;
        const float len = sqrtf(len2);
        const float x = ddx / len, y = ddy / len, z = ddz / len;
        const uint8_t cl = geo.clamped[vg];
        const float dl[3] = {(cl & 1) ? 0.0f : gcol.x, (cl & 2) ? 0.0f : gcol.y, (cl & 4) ? 0.0f : gcol.z};
        float dLda = 0.0f, dLdb = 0.0f, dLdc = 0.0f;
        const float3 sa = sh_arg(d.sh_basis, x, y, z);
        const uint32_t flip = sh_flip_mask(d.sh_basis);
        const int layout = d.sh_layout;
        sh_for_each(d.deg, sa.x, sa.y, sa.z, [&](int k, float Y, float Ya, float Yb, float Yc) {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const float cd = row[sh_index(layout, M, k, ch)] * sh_sign(flip, k, dl[ch]);
                dLda += Ya * cd; dLdb += Yb * cd; dLdc += Yc * cd;
            }
        });
        const float3 dLd = sh_grad_unpermute(d.sh_basis, dLda, dLdb, dLdc);
        const float inv3 = 1.0f / (len2 * len);
        camera_campos_grads(ddx, ddy, ddz, len2, inv3, dLd, cam);
    }
    if (DEPTH && vis) {
        const float dz = vgr.d_color[vg].w * depth_value_grad(d.depth_mode, geo.depth[vg], in.scale, in.near_far, vid);
        camera_depth_grads(dz, mx0, my0, mz0, sc, cam);
    }
    store_cam_partials(cam, cam_ws, d, v, sg0, rows, scene, lane);
}

// Sums the partial rows of every flat view in a fixed order over many CTAs (grid: kCamFinishRows-row chunks x views).
// CTA c of a view adds rows [c R, (c + 1) R) -- 8 strided running sums, then a fixed tree over the 8 -- and, when the
// view has more than one chunk, stores its sum over row c R (which only it has read) and counts itself in on the
// view's counter (cam_counter).  The CTA that arrives last adds the chunk sums in chunk order, the same way.  Which
// CTA that is does not change the order of any float sum, so the same rows give the same bits.  Writes all 16 / 16 /
// 3 / 2 entries of the four camera gradients (the entries the forward never reads get 0).
constexpr int kCamFinishThreads = 8 * kCamRowFloats;
constexpr int kCamFinishRows = 256;

__device__ __forceinline__ void cam_finish_sum(const float *rows, size_t step, int n, int k, int grp,
                                               float (&part)[8][kCamRowFloats]) {
    float acc = 0.0f;
    for (int r = grp; r < n; r += 8) acc += __ldcg(rows + (size_t)r * step + k);
    part[grp][k] = acc;
    __syncthreads();
#pragma unroll
    for (int stride = 4; stride > 0; stride >>= 1) {
        if (grp < stride) part[grp][k] += part[grp + stride][k];
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kCamFinishThreads) k_camera_finish(Dims d, float *__restrict__ ws,
                                                                     ps_raster_camera_grads cg) {
    __shared__ float part[8][kCamRowFloats];
    __shared__ bool last;
    const int vid = blockIdx.y, s = vid / d.V, chunk = blockIdx.x, chunks = gridDim.x;
    const int k = threadIdx.x % kCamRowFloats, grp = threadIdx.x / kCamRowFloats;
    const long long w_lo = ((long long)s * d.P) / 32, w_hi = ((long long)(s + 1) * d.P - 1) / 32;
    const int nrows = (int)(w_hi - w_lo + 1);
    float *rows = ws + (size_t)vid * cam_rows_per_view(d.P) * kCamRowFloats;
    float *mine = rows + (size_t)chunk * kCamFinishRows * kCamRowFloats;
    cam_finish_sum(mine, kCamRowFloats, min(kCamFinishRows, nrows - chunk * kCamFinishRows), k, grp, part);
    if (chunks > 1) {
        if (threadIdx.x < kCamEntries) mine[threadIdx.x] = part[0][threadIdx.x];   // word kCamEntries: the counter
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) last = atomicAdd(cam_counter(ws, d, vid), 1u) == (unsigned)chunks - 1u;
        __syncthreads();
        if (!last) return;
        __threadfence();
        cam_finish_sum(rows, (size_t)kCamFinishRows * kCamRowFloats, chunks, k, grp, part);
    }
    const int t = threadIdx.x;
    if (t < 16) {
        const int j = t / 4, i = t % 4;
        if (cg.d_viewmatrix) cg.d_viewmatrix[16 * vid + t] = i == 3 ? 0.0f : part[0][3 * j + i];
        if (cg.d_projmatrix) cg.d_projmatrix[16 * vid + t] = i == 2 ? 0.0f : part[0][12 + 3 * j + (i == 3 ? 2 : i)];
    }
    if (t < 3 && cg.d_campos) cg.d_campos[3 * vid + t] = part[0][24 + t];
    if (t < 2 && cg.d_tanfov) cg.d_tanfov[2 * vid + t] = part[0][27 + t];
}

template <bool DEPTH, bool CAM>
static int launch_preprocess_bwd_kernel(unsigned blocks, size_t smem, const Dims &d, const Inputs &in, const Geom &g,
                                        const ViewGrads &vg, const GaussGrads &out, int row_stride, float *cam_ws,
                                        cudaStream_t st) {
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices))
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_preprocess_bwd<DEPTH, CAM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           96 * 1024));
    k_preprocess_bwd<DEPTH, CAM><<<blocks, kPreBwdThreads, smem, st>>>(d, in, g, vg, out, row_stride, cam_ws);
    PS_LAUNCH_CHECK("k_preprocess_bwd");
    return PS_OK;
}

int launch_preprocess_backward(const Dims &d, const Inputs &in, const Geom &g, const ViewGrads &vg,
                               const ps_raster_grads &grads, cudaStream_t st) {
    const int row_stride = d.M > 0 ? ((3 * d.M) | 1) : 1;   // odd word count: conflict-free per-lane rows
    const size_t smem = d.M > 0 ? sizeof(float) * kPreBwdThreads * row_stride * (d.V == 1 ? 1 : 2) : 0;
    const long long sp = (long long)d.S * d.P;
    const unsigned blocks = (unsigned)((sp + kPreBwdThreads - 1) / kPreBwdThreads);
    const GaussGrads out{grads.d_means, grads.d_cov, grads.d_opacities, grads.d_sh, grads.d_means2d};
    const ps_raster_camera_grads *cg = grads.camera;
    float *ws = cg ? static_cast<float *>(cg->workspace) : nullptr;
    int rc = PS_OK;
    if (!grads.d_means) {               // camera-only backward (the caller checked that cg is set)
        const unsigned cam_blocks = (unsigned)((sp + kCamBwdThreads - 1) / kCamBwdThreads) * (unsigned)d.V;
        const size_t cam_smem = d.M > 0 ? sizeof(float) * kCamBwdThreads * row_stride : 0;
        if (d.depth_mode)
            k_camera_bwd<true><<<cam_blocks, kCamBwdThreads, cam_smem, st>>>(d, in, g, vg, row_stride, ws);
        else
            k_camera_bwd<false><<<cam_blocks, kCamBwdThreads, cam_smem, st>>>(d, in, g, vg, row_stride, ws);
        PS_LAUNCH_CHECK("k_camera_bwd");
    } else if (d.depth_mode)
        rc = cg ? launch_preprocess_bwd_kernel<true, true>(blocks, smem, d, in, g, vg, out, row_stride, ws, st)
                : launch_preprocess_bwd_kernel<true, false>(blocks, smem, d, in, g, vg, out, row_stride, ws, st);
    else
        rc = cg ? launch_preprocess_bwd_kernel<false, true>(blocks, smem, d, in, g, vg, out, row_stride, ws, st)
                : launch_preprocess_bwd_kernel<false, false>(blocks, smem, d, in, g, vg, out, row_stride, ws, st);
    if (rc || !cg) return rc;
    const dim3 finish_grid((unsigned)((cam_rows_per_view(d.P) + kCamFinishRows - 1) / kCamFinishRows),
                           (unsigned)(d.S * d.V));
    k_camera_finish<<<finish_grid, kCamFinishThreads, 0, st>>>(d, ws, *cg);
    PS_LAUNCH_CHECK("k_camera_finish");
    return PS_OK;
}

}  // namespace ps
