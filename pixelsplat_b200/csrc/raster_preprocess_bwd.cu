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

        const float a = cv.a, b = cv.b, c = cv.c;
        const float denom = a * c - b * b;
        const float denom2inv = 1.0f / (denom * denom + 0.0000001f);
        float dL_da = 0.0f, dL_db = 0.0f, dL_dc = 0.0f;
        const float *m0 = cv.m0, *m1 = cv.m1;
        if (denom2inv != 0.0f) {
            dL_da = denom2inv * (-c * c * gc.x + 2.0f * b * c * gc.y + (denom - a * c) * gc.z);
            dL_dc = denom2inv * (-a * a * gc.z + 2.0f * a * b * gc.y + (denom - a * c) * gc.x);
            dL_db = denom2inv * 2.0f * (b * c * gc.x - (denom + 2.0f * b * b) * gc.y + a * b * gc.z);
            const float s2 = sc * sc;
            dcov[0] += s2 * (m0[0] * m0[0] * dL_da + m0[0] * m1[0] * dL_db + m1[0] * m1[0] * dL_dc);
            dcov[3] += s2 * (m0[1] * m0[1] * dL_da + m0[1] * m1[1] * dL_db + m1[1] * m1[1] * dL_dc);
            dcov[5] += s2 * (m0[2] * m0[2] * dL_da + m0[2] * m1[2] * dL_db + m1[2] * m1[2] * dL_dc);
            dcov[1] += s2 * (2.0f * m0[0] * m0[1] * dL_da + (m0[0] * m1[1] + m0[1] * m1[0]) * dL_db + 2.0f * m1[0] * m1[1] * dL_dc);
            dcov[2] += s2 * (2.0f * m0[0] * m0[2] * dL_da + (m0[0] * m1[2] + m0[2] * m1[0]) * dL_db + 2.0f * m1[0] * m1[2] * dL_dc);
            dcov[4] += s2 * (2.0f * m0[2] * m0[1] * dL_da + (m0[1] * m1[2] + m0[2] * m1[1]) * dL_db + 2.0f * m1[1] * m1[2] * dL_dc);
        }
        // dL/dM (rows) from a = m0 S m0, b = m0 S m1, c = m1 S m1
        const float S[3][3] = {{s6[0], s6[1], s6[2]}, {s6[1], s6[3], s6[4]}, {s6[2], s6[4], s6[5]}};
        float dM0[3], dM1[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float sm0 = m0[0] * S[k][0] + m0[1] * S[k][1] + m0[2] * S[k][2];
            const float sm1 = m1[0] * S[k][0] + m1[1] * S[k][1] + m1[2] * S[k][2];
            dM0[k] = 2.0f * sm0 * dL_da + sm1 * dL_db;
            dM1[k] = 2.0f * sm1 * dL_dc + sm0 * dL_db;
        }
        const float dJ00 = vm[0] * dM0[0] + vm[4] * dM0[1] + vm[8] * dM0[2];
        const float dJ02 = vm[2] * dM0[0] + vm[6] * dM0[1] + vm[10] * dM0[2];
        const float dJ11 = vm[1] * dM1[0] + vm[5] * dM1[1] + vm[9] * dM1[2];
        const float dJ12 = vm[2] * dM1[0] + vm[6] * dM1[1] + vm[10] * dM1[2];
        const float tz = 1.0f / cv.tz, tz2 = tz * tz, tz3 = tz2 * tz;
        const float dL_dtx = cv.clamp_x ? 0.0f : -focal_x * tz2 * dJ02;
        const float dL_dty = cv.clamp_y ? 0.0f : -focal_y * tz2 * dJ12;
        const float dL_dtz = -focal_x * tz2 * dJ00 - focal_y * tz2 * dJ11 +
                             (2.0f * focal_x * cv.ctx) * tz3 * dJ02 + (2.0f * focal_y * cv.cty) * tz3 * dJ12;
        gx = vm[0] * dL_dtx + vm[1] * dL_dty + vm[2] * dL_dtz;
        gy = vm[4] * dL_dtx + vm[5] * dL_dty + vm[6] * dL_dtz;
        gz = vm[8] * dL_dtx + vm[9] * dL_dty + vm[10] * dL_dtz;

        // screen-space mean through the perspective divide
        const float hx = pm[0] * px + pm[4] * py + pm[8] * pz + pm[12];
        const float hy = pm[1] * px + pm[5] * py + pm[9] * pz + pm[13];
        const float hw = pm[3] * px + pm[7] * py + pm[11] * pz + pm[15];
        const float m_w = 1.0f / (hw + 0.0000001f);
        const float mul1 = hx * m_w * m_w, mul2 = hy * m_w * m_w;
        gx += (pm[0] * m_w - pm[3] * mul1) * g2.x + (pm[1] * m_w - pm[3] * mul2) * g2.y;
        gy += (pm[4] * m_w - pm[7] * mul1) * g2.x + (pm[5] * m_w - pm[7] * mul2) * g2.y;
        gz += (pm[8] * m_w - pm[11] * mul1) * g2.x + (pm[9] * m_w - pm[11] * mul2) * g2.y;
        if (CAM) {
            // viewmatrix: t = W p + (vm[12], vm[13], vm[14]) and M = J W (W[i][j] = vm[4j+i]);
            // projmatrix: h = pm p (p.w = 1), screen xy from (hx, hy) / (hw + 1e-7);
            // tanfov: only through the focal lengths in J (f = size / (2 tanfov); the clamp limit passes nothing)
            const float j00 = focal_x * tz, j02 = -focal_x * cv.ctx * tz2;
            const float j11 = focal_y * tz, j12 = -focal_y * cv.cty * tz2;
            const float p[3] = {px, py, pz};
            const float dhx = g2.x * m_w, dhy = g2.y * m_w, dhw = -(mul1 * g2.x + mul2 * g2.y);
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                cam[3 * j + 0] = dM0[j] * j00 + dL_dtx * p[j];
                cam[3 * j + 1] = dM1[j] * j11 + dL_dty * p[j];
                cam[3 * j + 2] = dM0[j] * j02 + dM1[j] * j12 + dL_dtz * p[j];
                cam[12 + 3 * j + 0] = dhx * p[j];
                cam[12 + 3 * j + 1] = dhy * p[j];
                cam[12 + 3 * j + 2] = dhw * p[j];
            }
            cam[9] = dL_dtx; cam[10] = dL_dty; cam[11] = dL_dtz;
            cam[21] = dhx; cam[22] = dhy; cam[23] = dhw;
            cam[27] = (dJ00 * tz - dJ02 * cv.ctx * tz2) * (-focal_x / tanfovx);
            cam[28] = (dJ11 * tz - dJ12 * cv.cty * tz2) * (-focal_y / tanfovy);
        }
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
            if (CAM) {
                // the direction is p - campos.  Rounded intrinsics: plain products shared with the lines above
                // would change how those are contracted, and the Gaussian gradients must keep their bits.
                const float xx = __fmul_rn(ddx, ddx), yy = __fmul_rn(ddy, ddy), zz = __fmul_rn(ddz, ddz);
                const float xy = __fmul_rn(ddx, ddy), xz = __fmul_rn(ddx, ddz), yz = __fmul_rn(ddy, ddz);
                const float ex = __fadd_rn(__fadd_rn(__fmul_rn(__fsub_rn(len2, xx), dLdx), -__fmul_rn(xy, dLdy)), -__fmul_rn(xz, dLdz));
                const float ey = __fadd_rn(__fadd_rn(-__fmul_rn(xy, dLdx), __fmul_rn(__fsub_rn(len2, yy), dLdy)), -__fmul_rn(yz, dLdz));
                const float ez = __fadd_rn(__fadd_rn(-__fmul_rn(xz, dLdx), -__fmul_rn(yz, dLdy)), __fmul_rn(__fsub_rn(len2, zz), dLdz));
                cam[24] = -__fmul_rn(ex, inv3); cam[25] = -__fmul_rn(ey, inv3); cam[26] = -__fmul_rn(ez, inv3);
            }
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
            if (CAM) {   // z = (vm[2], vm[6], vm[10]) . mean + vm[14] / sc
                cam[2] += dz * mx0; cam[5] += dz * my0; cam[8] += dz * mz0; cam[11] += dz / sc;
            }
        }
        if (CAM) {
            // per (scene, view) sums over the warp's lanes in a fixed butterfly order; a warp whose Gaussians span
            // two scenes (P not a multiple of 32) stores one row for each
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
                }
            }
        }
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

// One CTA per flat view: sums the view's partial rows in ascending warp order -- 8 strided running sums, then a
// fixed tree over the 8 -- and writes all 16 / 16 / 3 / 2 entries of the four camera gradients (the entries the
// forward never reads get 0).  No atomics: the same rows give the same bits.
constexpr int kCamFinishThreads = 8 * kCamRowFloats;

__global__ void __launch_bounds__(kCamFinishThreads) k_camera_finish(Dims d, const float *__restrict__ ws,
                                                                     ps_raster_camera_grads cg) {
    __shared__ float part[8][kCamRowFloats];
    const int vid = blockIdx.x, s = vid / d.V;
    const int k = threadIdx.x % kCamRowFloats, grp = threadIdx.x / kCamRowFloats;
    const long long w_lo = ((long long)s * d.P) / 32, w_hi = ((long long)(s + 1) * d.P - 1) / 32;
    const int nrows = (int)(w_hi - w_lo + 1);
    const float *rows = ws + (size_t)vid * cam_rows_per_view(d.P) * kCamRowFloats;
    float acc = 0.0f;
    for (int r = grp; r < nrows; r += 8) acc += rows[(size_t)r * kCamRowFloats + k];
    part[grp][k] = acc;
    __syncthreads();
#pragma unroll
    for (int stride = 4; stride > 0; stride >>= 1) {
        if (grp < stride) part[grp][k] += part[grp + stride][k];
        __syncthreads();
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
    int rc;
    if (d.depth_mode)
        rc = cg ? launch_preprocess_bwd_kernel<true, true>(blocks, smem, d, in, g, vg, out, row_stride, ws, st)
                : launch_preprocess_bwd_kernel<true, false>(blocks, smem, d, in, g, vg, out, row_stride, ws, st);
    else
        rc = cg ? launch_preprocess_bwd_kernel<false, true>(blocks, smem, d, in, g, vg, out, row_stride, ws, st)
                : launch_preprocess_bwd_kernel<false, false>(blocks, smem, d, in, g, vg, out, row_stride, ws, st);
    if (rc || !cg) return rc;
    k_camera_finish<<<(unsigned)(d.S * d.V), kCamFinishThreads, 0, st>>>(d, ws, *cg);
    PS_LAUNCH_CHECK("k_camera_finish");
    return PS_OK;
}

}  // namespace ps
