// LEGACY (round-1) compositor, selectable with PIXELSPLAT_B200_COMPOSITE=1 for A/B measurements; the
// default is the warp-task compositor in raster_composite2.cu.
// Alpha compositing, forward (front-to-back) and backward (back-to-front).
// One CTA per (view, 16x16 tile); each warp owns an 8x4 pixel sub-rectangle, each lane a pixel.
// The tile's sorted instance list is staged 256 entries at a time in shared memory.
//
// Differences from upstream's renderCUDA (SURVEY.md A.3 / A.5), none of which
// change a per-pixel decision:
//   * warp-level culling: for every staged Gaussian one lane tests the axis-aligned bound of
//     the region where alpha >= 1/255 can hold (|d| <= sqrt(2 ln(255 o) Sigma_ii)) against the
//     warp's 8x4 rectangle; a ballot keeps only Gaussians that can touch the warp, so most
//     (pixel, Gaussian) pairs of the 3-sigma-square binning are never evaluated;
//   * backward: gradients are reduced across the warp with shuffles, combined across the
//     CTA's warps in shared memory, and flushed with ONE global atomic per value per
//     (tile, Gaussian) instead of one per (pixel, Gaussian).
#include "ps_common.cuh"

namespace ps {

constexpr int kCompThreads = 256;
constexpr int kStage = 256;
constexpr float kAlphaMin = 1.0f / 255.0f;

// Half-extents (in pixels) of the axis-aligned box outside of which this Gaussian's alpha is
// certainly < 1/255 (conservative).  Returns a negative x to mean "never contributes".
__device__ __forceinline__ float2 alpha_extent(const float4 co) {
    const float A = co.x, B = co.y, C = co.z, o = co.w;
    const float det = A * C - B * B;
    if (!(det > 0.0f) || !(A > 0.0f) || !(C > 0.0f) || !(o <= 3.0e38f)) return make_float2(3.0e38f, 3.0e38f);
    if (!(o * 255.0f >= 1.0f - 1e-3f)) return make_float2(-1.0f, -1.0f);  // also catches NaN/neg
    const float tau = __logf(fmaxf(o * 255.0f, 1.0f)) + 0.01f;                // q = -power <= tau
    const float inv = 2.0f * tau / det;
    return make_float2(sqrtf(inv * C) * 1.001f + 0.01f, sqrtf(inv * A) * 1.001f + 0.01f);
}

// Shared-memory staging is SoA so that both the lane-varying cull reads (8 B stride) and the
// broadcast reads of the evaluation loop are bank-conflict free.
struct StageBuf {
    float2 xy[kStage];
    float2 ext[kStage];
    float4 co[kStage];
    float4 rgb[kStage];
};

// The staged conic is pre-multiplied so that  power * log2(e) = qa dx^2 + qc dy^2 + qb dx dy
// (one MUFU.EX2, no extra multiply, per evaluation); the sign test `power > 0` is unchanged.
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// 2^x with the hardware approximation only (MUFU.EX2, flush-to-zero); exp2f() adds denormal
// range handling that the compositor does not need (alpha below 1/255 is discarded anyway).
__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Staging is software-pipelined: the gathers of round r+1 (key -> xy / conic / rgb, two dependent
// L2 round trips) are issued into registers before round r is processed and only parked in shared
// memory at the top of the next iteration, so their latency hides behind the composite math
// instead of stalling all 8 warps of the CTA once per 256 entries.
struct StagedRegs {
    float2 xy;
    float4 co, rgb;
    uint32_t g;
};

__device__ __forceinline__ StagedRegs stage_load(const Geom &geo, size_t base, uint32_t g) {
    StagedRegs r;
    r.g = g;
    r.xy = geo.xy[base + g];
    r.co = geo.conic_opacity[base + g];
    r.rgb = geo.rgb[base + g];
    return r;
}

__device__ __forceinline__ void stage_store(StageBuf &s, int slot, const StagedRegs &r) {
    s.xy[slot] = r.xy;
    s.co[slot] = make_float4(-0.5f * kLog2e * r.co.x, -kLog2e * r.co.y, -0.5f * kLog2e * r.co.z, r.co.w);
    s.rgb[slot] = r.rgb;
    s.ext[slot] = alpha_extent(r.co);
}

// Warp-uniform FIFO of up to three staged-slot indices carried from one 32-entry cull chunk to the
// next.  The backward evaluation loop consumes FOUR list entries per iteration (one transposed
// reduction serves all four); a chunk leaves 6.4 hits on average, so draining every chunk separately
// ran one iteration in five half empty.  With the carry
// only the last chunk of a 256-entry stage can end on a partial group.  Order is preserved (carried
// entries precede the new chunk's).
struct HitCarry {
    uint32_t c0, c1, c2;
    int n;
};

__device__ __forceinline__ void carry_push_all(HitCarry &c, uint32_t &mask, uint32_t jb) {
    while (mask) {
        const uint32_t j = jb + (uint32_t)(__ffs(mask) - 1);
        mask &= mask - 1;
        if (c.n == 0) c.c0 = j;
        else if (c.n == 1) c.c1 = j;
        else c.c2 = j;
        ++c.n;
    }
}

// Next four entries: carried ones first, then the lowest set bits of `mask`; unused slots point at
// the (valid) slot jb with has = false.
__device__ __forceinline__ void take4(HitCarry &c, uint32_t &mask, uint32_t jb, uint32_t (&jx)[4], bool (&has)[4]) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        if (q < c.n) {
            jx[q] = q == 0 ? c.c0 : q == 1 ? c.c1 : c.c2;
            has[q] = true;
        } else {
            has[q] = mask != 0;
            const int bq = has[q] ? __ffs(mask) - 1 : 0;
            mask &= mask - 1;
            jx[q] = jb + (uint32_t)bq;
        }
    }
    c.n = 0;
}

__global__ void __launch_bounds__(kCompThreads)
k_composite_fwd(Dims d, Geom geo, const float *__restrict__ bg_all,
                const unsigned long long *__restrict__ keys, float *__restrict__ final_T,
                uint32_t *__restrict__ n_contrib, float *__restrict__ state_color,
                float *__restrict__ out_color) {
    __shared__ StageBuf s;
    const int vid = blockIdx.y, tile = blockIdx.x;
    const int tx = tile % d.gx, ty = tile / d.gx;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wx0 = tx * kTile + (warp & 1) * 8, wy0 = ty * kTile + (warp >> 1) * 4;
    const int pxi = wx0 + (lane & 7), pyi = wy0 + (lane >> 3);
    const bool inside = pxi < d.W && pyi < d.H;
    const float px = (float)pxi, py = (float)pyi;
    const float rx0 = (float)wx0, rx1 = (float)(wx0 + 7), ry0 = (float)wy0, ry1 = (float)(wy0 + 3);
    const bool truncated = *geo.n_instances > d.capacity;
    const size_t seg = (size_t)vid * d.tiles + tile;
    const uint32_t start = geo.tile_start[seg];
    const uint32_t count = truncated ? 0u : geo.tile_count[seg];
    const size_t gbase = (size_t)vid * d.P;

    float T = 1.0f, Cr = 0.0f, Cg = 0.0f, Cb = 0.0f;
    uint32_t last = 0;
    bool done = !inside;
    bool warp_done = __all_sync(0xffffffffu, done);

    StagedRegs nxt;
    nxt.g = 0; nxt.xy = make_float2(0.0f, 0.0f); nxt.co = nxt.rgb = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if ((uint32_t)tid < count) nxt = stage_load(geo, gbase, (uint32_t)keys[start + tid]);
    for (uint32_t round0 = 0; round0 < count; round0 += kStage) {
        if (__syncthreads_count(warp_done ? 1 : 0) == kCompThreads) break;
        const uint32_t n_here = min((uint32_t)kStage, count - round0);
        if ((uint32_t)tid < n_here) stage_store(s, tid, nxt);
        __syncthreads();
        if (round0 + kStage + (uint32_t)tid < count)         // prefetch the next round
            nxt = stage_load(geo, gbase, (uint32_t)keys[start + round0 + kStage + tid]);
        if (!warp_done) {
            for (uint32_t jb = 0; jb < n_here; jb += 32) {
                const uint32_t j = jb + lane;
                bool hit = false;
                if (j < n_here) {
                    const float2 c = s.xy[j], e = s.ext[j];
                    hit = (c.x + e.x >= rx0) && (c.x - e.x <= rx1) && (c.y + e.y >= ry0) && (c.y - e.y <= ry1);
                }
                uint32_t mask = __ballot_sync(0xffffffffu, hit);
                // four entries per iteration: their power / exp evaluations are independent, only
                // the transmittance update chains (the warp has few peers to hide latency behind:
                // a 256x256 view is just 2048 warps on 132 SMs).  (Carrying partial groups across
                // chunks as the backward does costs the forward more in bookkeeping than it saves.)
                while (mask) {
                    uint32_t jx[4];
                    bool has[4];
                    float pw[4], al[4];
                    float4 col[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        has[q] = mask != 0;
                        const int bq = has[q] ? __ffs(mask) - 1 : 0;
                        mask &= mask - 1;
                        jx[q] = jb + (uint32_t)bq;
                        const float2 xy = s.xy[jx[q]];
                        const float4 co = s.co[jx[q]];
                        col[q] = s.rgb[jx[q]];
                        const float dx = xy.x - px, dy = xy.y - py;
                        pw[q] = co.x * dx * dx + co.z * dy * dy + co.y * dx * dy;
                        al[q] = fminf(0.99f, co.w * fast_exp2(pw[q]));
                    }
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const bool contrib = has[q] && !done && !(pw[q] > 0.0f) && !(al[q] < kAlphaMin);
                        const float test_T = T * (1.0f - al[q]);
                        const bool stop = contrib && (test_T < 0.0001f);
                        const bool blend = contrib && !stop;
                        const float w = blend ? al[q] * T : 0.0f;
                        Cr += col[q].x * w; Cg += col[q].y * w; Cb += col[q].z * w;
                        T = blend ? test_T : T;
                        last = blend ? round0 + jx[q] + 1u : last;
                        done = done || stop;
                    }
                }
                warp_done = __all_sync(0xffffffffu, done);
                if (warp_done) break;
            }
        }
        __syncthreads();
    }
    if (inside) {
        const size_t pix = (size_t)pyi * d.W + pxi;
        const size_t hw = (size_t)d.H * d.W;
        final_T[(size_t)vid * hw + pix] = T;
        n_contrib[(size_t)vid * hw + pix] = last;
        const float *bg = bg_all + 3 * vid;
        float *o = out_color + (size_t)vid * 3 * hw;
        float *sc = state_color + (size_t)vid * 3 * hw;
        sc[pix] = o[pix] = Cr + T * bg[0];
        sc[hw + pix] = o[hw + pix] = Cg + T * bg[1];
        sc[2 * hw + pix] = o[2 * hw + pix] = Cb + T * bg[2];
    }
}

// ---------------------------------------------------------------------------- backward

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Sum each of 32 per-lane values over the warp with 31 shuffles instead of 160: at every step a
// lane keeps half of its values and hands the other half to its partner.  On return lane i
// holds the warp total of v[i].
__device__ __forceinline__ float transpose_reduce32(float (&v)[32], int lane) {
#pragma unroll
    for (int half = 16; half >= 1; half >>= 1) {
        const bool up = (lane & half) != 0;
#pragma unroll
        for (int i = 0; i < half; ++i) {
            const float keep = up ? v[i + half] : v[i];
            const float send = up ? v[i] : v[i + half];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, half);
        }
    }
    return v[0];
}

// Same for 4 values: lane l ends with the total of v[(l >> 3) & 3].
__device__ __forceinline__ float transpose_reduce4(float (&v)[4], int lane) {
    {
        const bool up = (lane & 16) != 0;
        const float k0 = up ? v[2] : v[0], s0 = up ? v[0] : v[2];
        const float k1 = up ? v[3] : v[1], s1 = up ? v[1] : v[3];
        v[0] = k0 + __shfl_xor_sync(0xffffffffu, s0, 16);
        v[1] = k1 + __shfl_xor_sync(0xffffffffu, s1, 16);
    }
    {
        const bool up = (lane & 8) != 0;
        const float k0 = up ? v[1] : v[0], s0 = up ? v[0] : v[1];
        v[0] = k0 + __shfl_xor_sync(0xffffffffu, s0, 8);
    }
    float t = v[0];
    t += __shfl_xor_sync(0xffffffffu, t, 4);
    t += __shfl_xor_sync(0xffffffffu, t, 2);
    t += __shfl_xor_sync(0xffffffffu, t, 1);
    return t;
}

// Per-pixel backward of one list entry (SURVEY.md A.5).  Returns whether the entry contributed;
// g[0..7] = d_mean2d.xy, d_conic.xyz, d_color.rgb ; op = d_opacity.
struct PixelState {
    float T, acc_r, acc_g, acc_b, last_alpha, lc_r, lc_g, lc_b;
};

// Straight-line (predicated, no divergent branches): on average only ~10 of a warp's 32 pixels
// take a given entry, but the warp executes the whole body anyway, and the reconvergence
// bookkeeping of a branchy version costs issued instructions of its own.
__device__ __forceinline__ bool pixel_bwd(bool in_range, const float2 exy, const float4 eco, const float4 ergb,
                                          float px, float py, float dpr, float dpg, float dpb, float T_final,
                                          float bg_dot, float ddelx_dx, float ddely_dy, PixelState &st,
                                          float *g, float &op) {
    const float dx = exy.x - px, dy = exy.y - py;
    const float p2 = eco.x * dx * dx + eco.z * dy * dy + eco.y * dx * dy;   // power * log2(e)
    const float G = fast_exp2(p2);
    const float alpha = fminf(0.99f, eco.w * G);
    const bool active = in_range && !(p2 > 0.0f) && !(alpha < kAlphaMin);
    // An entry the pixel skips behaves exactly like one with alpha = 0 and G = 0: T is unchanged,
    // the colour-behind recurrence folds the previous entry and then carries a zero-weight one,
    // and every gradient term vanishes -- so no per-field predication is needed.
    const float a = active ? alpha : 0.0f;
    const float Gs = active ? G : 0.0f;             // also keeps an overflowed exp2 out of 0 * inf
    const float rcp = __fdividef(1.0f, 1.0f - a);
    st.T = st.T * rcp;
    const float la = st.last_alpha;
    st.acc_r = st.acc_r + la * (st.lc_r - st.acc_r);      // = la * lc + (1 - la) * acc
    st.acc_g = st.acc_g + la * (st.lc_g - st.acc_g);
    st.acc_b = st.acc_b + la * (st.lc_b - st.acc_b);
    st.lc_r = ergb.x; st.lc_g = ergb.y; st.lc_b = ergb.z;
    st.last_alpha = a;
    const float w_color = a * st.T;
    g[5] = w_color * dpr; g[6] = w_color * dpg; g[7] = w_color * dpb;
    float dL_dalpha = (ergb.x - st.acc_r) * dpr + (ergb.y - st.acc_g) * dpg + (ergb.z - st.acc_b) * dpb;
    dL_dalpha = dL_dalpha * st.T - T_final * rcp * bg_dot;
    const float wG = eco.w * dL_dalpha * Gs;        // dL/dG * G
    const float sx = wG * dx, sy = wG * dy;
    // dG/d(delta) = -G (A dx + B dy) with A = -2 qa / log2e, B = -qb / log2e
    g[0] = (kLn2 * ddelx_dx) * (2.0f * eco.x * sx + eco.y * sy);
    g[1] = (kLn2 * ddely_dy) * (2.0f * eco.z * sy + eco.y * sx);
    g[2] = -0.5f * sx * dx;
    g[3] = -0.5f * sx * dy;
    g[4] = -0.5f * sy * dy;
    op = Gs * dL_dalpha;
    return active;
}

// Two list entries at once.  Everything that is element-wise per entry -- the quadratic form,
// alpha, the gradient terms -- is evaluated on (entry a, entry b) register pairs; the short
// per-pixel recurrences (T, colour behind) stay scalar and run a then b, exactly as the list
// order demands.  sm_90 has no packed FP32x2 arithmetic, so each pair operation is two scalar
// round-to-nearest operations that the compiler may not contract (the same roundings as packed
// FADD2 / FMUL2 / FFMA2), and the pairing gives the scheduler two independent chains.
__device__ __forceinline__ float2 pk(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

__device__ __forceinline__ void pixel_bwd_pair(bool in_a, bool in_b, const float2 xya, const float2 xyb,
                                               const float4 coa, const float4 cob, const float4 ca,
                                               const float4 cb, float px, float py, float dpr, float dpg,
                                               float dpb, float T_final, float bg_dot, float kx, float ky,
                                               PixelState &st, float *ga, float *gb, float &opa, float &opb,
                                               bool &act_a, bool &act_b) {
    const float2 DX = add2(pk(xya.x, xyb.x), pk(-px, -px));
    const float2 DY = add2(pk(xya.y, xyb.y), pk(-py, -py));
    const float2 QA = pk(coa.x, cob.x), QB = pk(coa.y, cob.y), QC = pk(coa.z, cob.z), W = pk(coa.w, cob.w);
    float2 P = mul2(mul2(QA, DX), DX);
    P = fma2(mul2(QC, DY), DY, P);
    P = fma2(mul2(QB, DX), DY, P);                       // power * log2(e), both entries
    const float2 G = pk(fast_exp2(P.x), fast_exp2(P.y));
    const float2 AL = mul2(W, G);
    const float al_a = fminf(0.99f, AL.x), al_b = fminf(0.99f, AL.y);
    act_a = in_a && !(P.x > 0.0f) && !(al_a < kAlphaMin);
    act_b = in_b && !(P.y > 0.0f) && !(al_b < kAlphaMin);
    // skipped entries behave like alpha = 0, G = 0 (see pixel_bwd)
    const float2 A = pk(act_a ? al_a : 0.0f, act_b ? al_b : 0.0f);
    const float2 GS = pk(act_a ? G.x : 0.0f, act_b ? G.y : 0.0f);
    const float2 OM = add2(pk(1.0f, 1.0f), pk(-A.x, -A.y));
    const float rcp_a = __fdividef(1.0f, OM.x), rcp_b = __fdividef(1.0f, OM.y);
    // ---- entry a, then entry b: transmittance and colour-behind recurrences (scalar / channel-packed)
    const float Ta = st.T * rcp_a;
    float2 acc_rg = pk(st.acc_r, st.acc_g);
    float acc_b_ = st.acc_b;
    {
        const float la = st.last_alpha;
        acc_rg = fma2(pk(la, la), add2(pk(st.lc_r, st.lc_g), pk(-acc_rg.x, -acc_rg.y)), acc_rg);
        acc_b_ = acc_b_ + la * (st.lc_b - acc_b_);
    }
    const float2 da_rg = add2(pk(ca.x, ca.y), pk(-acc_rg.x, -acc_rg.y));
    const float2 ta_rg = mul2(da_rg, pk(dpr, dpg));
    float dLa = ta_rg.x + ta_rg.y + (ca.z - acc_b_) * dpb;
    dLa = dLa * Ta - T_final * rcp_a * bg_dot;
    const float Tb = Ta * rcp_b;
    {
        const float la = A.x;
        acc_rg = fma2(pk(la, la), add2(pk(ca.x, ca.y), pk(-acc_rg.x, -acc_rg.y)), acc_rg);
        acc_b_ = acc_b_ + la * (ca.z - acc_b_);
    }
    const float2 db_rg = add2(pk(cb.x, cb.y), pk(-acc_rg.x, -acc_rg.y));
    const float2 tb_rg = mul2(db_rg, pk(dpr, dpg));
    float dLb = tb_rg.x + tb_rg.y + (cb.z - acc_b_) * dpb;
    dLb = dLb * Tb - T_final * rcp_b * bg_dot;
    st.T = Tb;
    st.acc_r = acc_rg.x; st.acc_g = acc_rg.y; st.acc_b = acc_b_;
    st.lc_r = cb.x; st.lc_g = cb.y; st.lc_b = cb.z;
    st.last_alpha = A.y;
    // ---- gradient terms, packed across the two entries
    const float2 DL = pk(dLa, dLb);
    const float2 WC = mul2(A, pk(Ta, Tb));                     // alpha * T
    const float2 CR = mul2(WC, pk(dpr, dpr)), CG = mul2(WC, pk(dpg, dpg)), CB = mul2(WC, pk(dpb, dpb));
    const float2 WG = mul2(mul2(W, DL), GS);             // dL/dG * G
    const float2 SX = mul2(WG, DX), SY = mul2(WG, DY);
    const float2 two = pk(2.0f, 2.0f);
    const float2 MX = mul2(pk(kx, kx), fma2(mul2(two, QA), SX, mul2(QB, SY)));
    const float2 MY = mul2(pk(ky, ky), fma2(mul2(two, QC), SY, mul2(QB, SX)));
    const float2 mh = pk(-0.5f, -0.5f);
    const float2 HX = mul2(mh, SX), HY = mul2(mh, SY);
    const float2 CA = mul2(HX, DX), CBc = mul2(HX, DY), CC = mul2(HY, DY);
    const float2 OP = mul2(GS, DL);
    ga[0] = MX.x; ga[1] = MY.x; ga[2] = CA.x; ga[3] = CBc.x; ga[4] = CC.x; ga[5] = CR.x; ga[6] = CG.x; ga[7] = CB.x;
    gb[0] = MX.y; gb[1] = MY.y; gb[2] = CA.y; gb[3] = CBc.y; gb[4] = CC.y; gb[5] = CR.y; gb[6] = CG.y; gb[7] = CB.y;
    opa = OP.x; opb = OP.y;
}

__global__ void __launch_bounds__(kCompThreads)
k_composite_bwd(Dims d, Geom geo, const float *__restrict__ bg_all,
                const unsigned long long *__restrict__ keys, const float *__restrict__ final_T,
                const uint32_t *__restrict__ n_contrib, const float *__restrict__ d_color,
                ViewGrads vg) {
    __shared__ StageBuf s;
    __shared__ uint32_t s_g[kStage];
    // Per-warp private gradient accumulators [warp][entry][9 (+1 pad)] in dynamic shared memory:
    // shared-memory float atomics compile to CAS loops, and 8 warps hammering the same entry
    // serialised (they were 1/6 of this kernel's stall samples).
    extern __shared__ float s_acc_all[];
    float(*s_acc)[10] = reinterpret_cast<float(*)[10]>(s_acc_all) + (size_t)(threadIdx.x >> 5) * kStage;
    __shared__ uint32_t s_max_last;
    const int vid = blockIdx.y, tile = blockIdx.x;
    const int tx = tile % d.gx, ty = tile / d.gx;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wx0 = tx * kTile + (warp & 1) * 8, wy0 = ty * kTile + (warp >> 1) * 4;
    const int pxi = wx0 + (lane & 7), pyi = wy0 + (lane >> 3);
    const bool inside = pxi < d.W && pyi < d.H;
    const float px = (float)pxi, py = (float)pyi;
    const float rx0 = (float)wx0, rx1 = (float)(wx0 + 7), ry0 = (float)wy0, ry1 = (float)(wy0 + 3);
    if (*geo.n_instances > d.capacity) return;
    const size_t seg = (size_t)vid * d.tiles + tile;
    const uint32_t start = geo.tile_start[seg];
    const size_t gbase = (size_t)vid * d.P;
    const size_t hw = (size_t)d.H * d.W;
    const size_t pix = (size_t)pyi * d.W + pxi;

    const float T_final = inside ? final_T[(size_t)vid * hw + pix] : 0.0f;
    const uint32_t last = inside ? n_contrib[(size_t)vid * hw + pix] : 0u;
    float dpr = 0.0f, dpg = 0.0f, dpb = 0.0f;
    if (inside) {
        const float *dc = d_color + (size_t)vid * 3 * hw;
        dpr = dc[pix]; dpg = dc[hw + pix]; dpb = dc[2 * hw + pix];
    }
    const float *bg = bg_all + 3 * vid;
    const float bg_dot = bg[0] * dpr + bg[1] * dpg + bg[2] * dpb;
    const float ddelx_dx = 0.5f * (float)d.W, ddely_dy = 0.5f * (float)d.H;

    if (tid == 0) s_max_last = 0;
    __syncthreads();
    const uint32_t warp_last = __reduce_max_sync(0xffffffffu, last);
    if (lane == 0) atomicMax(&s_max_last, warp_last);
    __syncthreads();
    const uint32_t block_last = s_max_last;   // entries at list position >= block_last are unused

    PixelState st;
    st.T = T_final;
    st.acc_r = st.acc_g = st.acc_b = st.last_alpha = st.lc_r = st.lc_g = st.lc_b = 0.0f;

    // walk positions block_last-1 .. 0, staged in chunks of kStage (highest position first)
    StagedRegs nxt;
    nxt.g = 0; nxt.xy = make_float2(0.0f, 0.0f); nxt.co = nxt.rgb = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if ((uint32_t)tid < block_last) nxt = stage_load(geo, gbase, (uint32_t)keys[start + (block_last - 1u - (uint32_t)tid)]);
    for (uint32_t hi = block_last; hi > 0;) {
        const uint32_t n_here = min((uint32_t)kStage, hi);
        // staged index j <-> list position  pos = hi - 1 - j
        if ((uint32_t)tid < n_here) {
            stage_store(s, tid, nxt);
            s_g[tid] = nxt.g;
        }
        if (hi > n_here && (uint32_t)tid < hi - n_here)      // prefetch the next (lower) chunk
            nxt = stage_load(geo, gbase, (uint32_t)keys[start + (hi - n_here - 1u - (uint32_t)tid)]);
        for (int i = tid; i < (kCompThreads / 32) * kStage * 10; i += kCompThreads) s_acc_all[i] = 0.0f;
        __syncthreads();
        HitCarry carry = {0u, 0u, 0u, 0};
        for (uint32_t jb = 0; jb < n_here; jb += 32) {
            const uint32_t j = jb + lane;
            bool hit = false;
            if (j < n_here && (hi - 1u - j) < warp_last) {
                const float2 c = s.xy[j], e = s.ext[j];
                hit = (c.x + e.x >= rx0) && (c.x - e.x <= rx1) && (c.y + e.y >= ry0) && (c.y - e.y <= ry1);
            }
            uint32_t mask = __ballot_sync(0xffffffffu, hit);
            const bool last_chunk = jb + 32u >= n_here;
            // four list entries per iteration: their exp / gradient math is independent (only the
            // cheap T / colour-behind recurrences chain), which gives the scheduler something to
            // issue while shuffles are in flight (a 256x256 view is 14 warps per SM), and one
            // 32-wide transposed shuffle reduction serves all four
            while (carry.n + __popc(mask) >= 4 || (last_chunk && (carry.n != 0 || mask != 0u))) {
                uint32_t jx[4];
                bool has[4];
                take4(carry, mask, jb, jx, has);
                float v[32], op[4];
                unsigned any = 0;
#pragma unroll
                for (int q = 0; q < 4; q += 2) {
                    bool a0, a1;
                    pixel_bwd_pair(has[q] && (hi - 1u - jx[q]) < last, has[q + 1] && (hi - 1u - jx[q + 1]) < last,
                                   s.xy[jx[q]], s.xy[jx[q + 1]], s.co[jx[q]], s.co[jx[q + 1]], s.rgb[jx[q]],
                                   s.rgb[jx[q + 1]], px, py, dpr, dpg, dpb, T_final, bg_dot, kLn2 * ddelx_dx,
                                   kLn2 * ddely_dy, st, v + 8 * q, v + 8 * q + 8, op[q], op[q + 1], a0, a1);
                    any |= __ballot_sync(0xffffffffu, a0) ? (1u << q) : 0u;
                    any |= __ballot_sync(0xffffffffu, a1) ? (2u << q) : 0u;
                }
                if (any == 0u) continue;
                const float tot = transpose_reduce32(v, lane);      // lane 8q + k: value k of entry q
                const float opt = transpose_reduce4(op, lane);      // lanes 8q ..: opacity of entry q
                // this warp's private copy: plain read-modify-write, no other warp touches it
                const int q = lane >> 3, k = lane & 7;
                const uint32_t jq = q == 0 ? jx[0] : q == 1 ? jx[1] : q == 2 ? jx[2] : jx[3];
                const bool live_q = (any >> q) & 1u;
                if (live_q) s_acc[jq][k] += tot;
                __syncwarp();
                if (live_q && k == 0) s_acc[jq][8] += opt;
                __syncwarp();
            }
            carry_push_all(carry, mask, jb);              // fewer than four left: they join the next chunk
        }
        __syncthreads();
        if ((uint32_t)tid < n_here) {
            float a[9];
            bool any = false;
#pragma unroll
            for (int k = 0; k < 9; ++k) {
                float t = 0.0f;
#pragma unroll
                for (int w8 = 0; w8 < kCompThreads / 32; ++w8) t += s_acc_all[((size_t)w8 * kStage + tid) * 10 + k];
                a[k] = t;
                any |= (t != 0.0f);
            }
            if (any) {
                const size_t o = gbase + s_g[tid];
                float *m = reinterpret_cast<float *>(vg.d_mean2d + o);
                float *c = reinterpret_cast<float *>(vg.d_conic + o);
                float *col = reinterpret_cast<float *>(vg.d_color + o);
                atomicAdd(m + 0, a[0]); atomicAdd(m + 1, a[1]);
                atomicAdd(c + 0, a[2]); atomicAdd(c + 1, a[3]); atomicAdd(c + 2, a[4]); atomicAdd(c + 3, a[8]);
                atomicAdd(col + 0, a[5]); atomicAdd(col + 1, a[6]); atomicAdd(col + 2, a[7]);
            }
        }
        __syncthreads();
        hi -= n_here;
    }
}

int launch_composite_forward_v1(const Dims &d, const Inputs &in, const Geom &g,
                                const unsigned long long *keys, const ImageState &img,
                                float *out_color, cudaStream_t st) {
    dim3 grid(d.tiles, d.S * d.V);
    k_composite_fwd<<<grid, kCompThreads, 0, st>>>(d, g, in.bg, keys, img.final_T, img.n_contrib, img.color, out_color);
    PS_LAUNCH_CHECK("k_composite_fwd");
    return PS_OK;
}

int launch_composite_backward_v1(const Dims &d, const Inputs &in, const Geom &g,
                                 const unsigned long long *keys, const ImageState &img,
                                 const float *d_color, const ViewGrads &vg, cudaStream_t st) {
    const float *final_T = img.final_T;
    const uint32_t *n_contrib = img.n_contrib;
    dim3 grid(d.tiles, d.S * d.V);
    const size_t acc_bytes = sizeof(float) * (kCompThreads / 32) * kStage * 10;
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_composite_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)acc_bytes));
    }
    k_composite_bwd<<<grid, kCompThreads, acc_bytes, st>>>(d, g, in.bg, keys, final_T, n_contrib, d_color, vg);
    PS_LAUNCH_CHECK("k_composite_bwd");
    return PS_OK;
}

}  // namespace ps
