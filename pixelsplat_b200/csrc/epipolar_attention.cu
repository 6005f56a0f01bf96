// Sampled epipolar cross-attention, fused: for every query ray, gather the S bilinear feature
// samples on its epipolar segment in each other view straight from the (L2-resident) feature
// map, add the depth positional encoding analytically, soft-max the scores and form the
// attention-weighted sums -- without ever materialising the sampled features
// ([b,v,ov,r,s,128] = 0.94 GB at configs[2]) or K/V ([b*v*r, 32, 1024] = 7.5 GB per layer).
//
// Maths (SURVEY.md Appendix B step 7, /root/reference/src/model/transformer/attention.py:54-70,
// epipolar_transformer.py:115-137), restructured with the same result up to fp32 rounding:
//   kv_s   = f_s + W_d PE(rd_s) + b_d (+ emb_ov),        f_s = bilinear(feat_o, xy_s) * valid
//   score  = q_h . (W_k,h kv_s) * scale = qt_h . f_s + pq_h . PE(rd_s) + bias_h,ov + const
//            with qt_h = scale * W_k,h^T q_h (folded by a GEMM outside), pq_h = W_d^T qt_h,
//            bias = qt_h . emb, and const (the b_d term) dropping out of the soft-max;
//   out_h  = W_v,h sum_s a_s kv_s = W_v,h ( z_h + W_d e_h + b_d + sum_ov mass_h,ov emb_ov )
//            with z_h = sum a_s f_s, e_h = sum a_s PE(rd_s), mass_h,ov = sum_{s in ov} a_s.
// The kernel maps (qt, pq, bias) -> (z, e, mass, lse); the small dense projections around it
// stay GEMMs.  One warp per query; lane l owns channels 4l..4l+3 for the gather and sample l
// for the soft-max / PE.  C = 128, S <= 32.
#include <cstdlib>
#include <initializer_list>
#include <type_traits>

#include "ps_common.cuh"

namespace ps {

constexpr int kEpiC = 128;
constexpr int kEpiWarps = 4;
constexpr int kMaxPE = 32;

struct EpiParams {
    int B, V, OV, h, w, S, npe;        // npe = 2 * num_octaves
    const float *feat;                 // [B, V, h, w, C] channels-last
    const float *seg;                  // [B, V, OV, R, 4]
    const uint8_t *valid;              // [B, V, OV, R]
    const float *rd;                   // [B, V, OV, R, S]
    const float *qt;                   // [N, H, C]
    const float *pq;                   // [N, H, npe]
    const float *bias;                 // [N, H, OV] or NULL
};

__device__ __forceinline__ float4 ldg4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }

// Bilinear tap set of grid_sample(align_corners=False, padding_mode="zeros") at normalised (x, y).
struct Taps {
    int off[4];      // element offset of the tap's channel vector inside one view's map, -1 = outside
    float w[4];
};

// (x0, y0) receives the cell's top-left tap, which may lie outside the map.
__device__ __forceinline__ Taps make_taps(float x, float y, int h, int w, int &x0, int &y0) {
    const float ix = x * (float)w - 0.5f, iy = y * (float)h - 0.5f;
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    const float ax = ix - fx0, ay = iy - fy0;
    // clamp before the int cast so wild coordinates cannot overflow; they are outside anyway
    x0 = (int)fminf(fmaxf(fx0, -2.0f), (float)w + 1.0f);
    y0 = (int)fminf(fmaxf(fy0, -2.0f), (float)h + 1.0f);
    Taps t;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int xi = x0 + (k & 1), yi = y0 + (k >> 1);
        const bool in = xi >= 0 && xi < w && yi >= 0 && yi < h;
        t.off[k] = in ? (yi * w + xi) * kEpiC : -1;
        t.w[k] = ((k & 1) ? ax : 1.0f - ax) * ((k >> 1) ? ay : 1.0f - ay);
    }
    return t;
}

// PE(rd)[2k] = sin(f_k rd), [2k+1] = sin(f_k rd + pi/2), layout "(d f p)"
// (positional_encoding.py:14-33).  The reference's frequency buffer is float32(2 pi) * 2^k, i.e.
// 2 pi (1 + delta) 2^k with delta = 2.78e-8 -- a phase shift of up to 9e-5 rad at k = 9 that is
// part of its semantics (the buffer is non-persistent, so every checkpoint gets it), so it is
// reproduced: phase/pi = u (1 + delta), u = rd 2^(k+1) formed exactly, reduced exactly mod 2, and
// evaluated with sincospif.  (The reference's own fp32 `sin(rd * f_k + phi)` rounds the product,
// up to 2e-4 rad at k = 9; this evaluation is closer to its float64 result.)
__device__ __forceinline__ void positional_encoding(float rd, int npe, float (&pe)[kMaxPE]) {
    constexpr float kTwoPiF32Excess = 2.7827534e-8f;   // float32(2 pi) / (2 pi) - 1
    float scale = 2.0f;
#pragma unroll
    for (int k = 0; k < kMaxPE / 2; ++k) {
        if (2 * k < npe) {
            float s, c;
            const float u = rd * scale;
            const float ur = u - 2.0f * floorf(0.5f * u);
            sincospif(ur + u * kTwoPiF32Excess, &s, &c);
            pe[2 * k] = s;
            pe[2 * k + 1] = c;
            scale *= 2.0f;
        }
    }
}

// Sum over the 32 lanes of SUB per-lane values v[0..SUB-1] (SUB = 4 or 8); every lane receives the total of
// v[lane & (SUB - 1)].  Halving butterflies on the low lane bits, plain butterflies on the rest.
template <int SUB>
__device__ __forceinline__ float transpose_reduce_sub(float (&v)[SUB], int lane) {
#pragma unroll
    for (int half = SUB / 2; half >= 1; half >>= 1) {
        const bool up = (lane & half) != 0;
#pragma unroll
        for (int i = 0; i < half; ++i) {
            const float keep = up ? v[i + half] : v[i];
            const float send = up ? v[i] : v[i + half];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, half);
        }
    }
    float r = v[0];
#pragma unroll
    for (int o = SUB; o < 32; o <<= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    return r;
}

// max / sum over the SUB distinct values held by an aligned group of SUB lanes (replicated across groups)
template <int SUB>
__device__ __forceinline__ float group_max(float v) {
#pragma unroll
    for (int o = SUB / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
template <int SUB>
__device__ __forceinline__ float group_add(float v) {
#pragma unroll
    for (int o = SUB / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Round 2: the S samples of a segment are processed in SUB-CHUNKS of SUB samples (8 forward, 4 backward) instead
// of all 32 at once.  Holding f[32][4] pinned both kernels at 255 registers = 8 warps per SM (12 % occupancy),
// which is what bounded them: they are latency-bound on the bilinear gathers (ncu r01: 22-27 % issue-active).
// With SUB samples in registers the forward needs <= 128 registers (16 warps / SM) and the backward <= 128 too;
// the soft-max is already streaming (online max / sum), so sub-chunks only add rescales.  The positional-
// encoding half of every score (and of d score) is evaluated once per other view with lane = sample, as before,
// and parked in shared memory for the sub-chunks to pick up.
struct __align__(16) EpiWarpSmem {
    float p[8][4];           // soft-max numerators (forward) / probabilities (backward) of the sub-chunk
    float dsub[8][4];        // backward: d score of the sub-chunk
    float scpe[32][4];       // PE half of the scores (+ bias), [sample][head]; -inf beyond S
    float dape[32][4];       // backward: PE half of d a (+ dmass)
    float ds_all[32][4];     // backward: d score of all samples of this other view (for dpq)
    float pe[32][kMaxPE + 1];
    float pq[4][kMaxPE];
    float aux[4][kMaxPE];    // backward: d_e
};

// ---- Shared by both kernels.  The backward recomputes the forward's probabilities as exp(score - lse), so both
// must form the query, the samples and their scores with the same code.

// Query n = (b V + v) R + r of the warp.
struct EpiQuery {
    int r, bv, v, b;         // bv = b V + v
};

// Decodes query n and loads its qt (lane = channels 4 lane .. 4 lane + 3) and its pq (into sm.pq; the caller's
// __syncwarp publishes it).  The backward loads its own per-query rows in the same two loops: per_head(hd) after
// qt_hd, per_pe(i) after entry i of the [HEADS, npe] pq row.
template <int HEADS, class PerHead, class PerPe>
__device__ __forceinline__ EpiQuery epi_query(const EpiParams &P, int n, int lane, EpiWarpSmem &sm,
                                              float (&qt)[HEADS][4], PerHead &&per_head, PerPe &&per_pe) {
    const int R = P.h * P.w;
    EpiQuery q;
    q.r = n % R; q.bv = n / R;
    q.v = q.bv % P.V; q.b = q.bv / P.V;
#pragma unroll
    for (int hd = 0; hd < HEADS; ++hd) {
        const float4 t = ldg4(P.qt + ((size_t)n * HEADS + hd) * kEpiC + 4 * lane);
        qt[hd][0] = t.x; qt[hd][1] = t.y; qt[hd][2] = t.z; qt[hd][3] = t.w;
        per_head(hd);
    }
    for (int i = lane; i < HEADS * P.npe; i += 32) {
        sm.pq[i / P.npe][i % P.npe] = P.pq[(size_t)n * HEADS * P.npe + i];
        per_pe(i);
    }
    return q;
}

// The query's ray in other view ov, which is view ov < v ? ov : ov + 1.
struct EpiRay {
    size_t ray;              // (bv OV + ov) R + r: the row of seg, valid and rd
    float4 seg;
    bool ok;                 // valid[ray]
    int map;                 // b V + the other view: its feature map
    size_t map_base;         // element offset of the lane's channels in that map
};

__device__ __forceinline__ EpiRay epi_ray(const EpiParams &P, const EpiQuery &q, int ov, int lane) {
    const int R = P.h * P.w;
    EpiRay y;
    const int o_view = ov < q.v ? ov : ov + 1;
    y.ray = ((size_t)(q.bv * P.OV + ov)) * R + q.r;
    y.seg = ldg4(P.seg + 4 * y.ray);
    y.ok = P.valid[y.ray] != 0;
    y.map = q.b * P.V + o_view;
    y.map_base = (size_t)y.map * R * kEpiC + 4 * lane;
    return y;
}

// Lane = sample s = lane of the ray.  taps: its bilinear taps, none (offset -1, weight 0) past S or on an invalid
// ray.  (bx, by): the top-left tap of its bilinear cell, (-2, -2) -- a cell that touches no texel -- where there are
// no taps.  PE(rd_s) goes into pe and sm.pe[s] (zero past S), and the PE half of its scores plus the bias into
// sm.scpe[s] (-inf past S).
template <int HEADS>
__device__ __forceinline__ void epi_sample(const EpiParams &P, const EpiRay &ray, int n, int ov, int lane,
                                           EpiWarpSmem &sm, Taps &taps, int &bx, int &by, float (&pe)[kMaxPE]) {
    const bool has_sample = lane < P.S;
    if (has_sample && ray.ok) {
        const float u = ((float)lane + 0.5f) / (float)P.S;
        const float sx = ray.seg.x + u * (ray.seg.z - ray.seg.x), sy = ray.seg.y + u * (ray.seg.w - ray.seg.y);
        taps = make_taps(sx, sy, P.h, P.w, bx, by);
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) { taps.off[k] = -1; taps.w[k] = 0.0f; }
        bx = by = -2;
    }
    positional_encoding(has_sample ? P.rd[ray.ray * P.S + lane] : 0.0f, P.npe, pe);
#pragma unroll
    for (int j = 0; j < kMaxPE; ++j)
        if (j < P.npe) sm.pe[lane][j] = has_sample ? pe[j] : 0.0f;
#pragma unroll
    for (int hd = 0; hd < HEADS; ++hd) {
        float sc = 0.0f;
#pragma unroll
        for (int j = 0; j < kMaxPE; ++j)
            if (j < P.npe) sc += sm.pq[hd][j] * pe[j];
        if (P.bias) sc += P.bias[((size_t)n * HEADS + hd) * P.OV + ov];
        sm.scpe[lane][hd] = has_sample ? sc : -INFINITY;
    }
}

// f[i] = channels 4 lane .. 4 lane + 3 of sample sub SUB + i, gathered from the map at fmap.
template <int SUB>
__device__ __forceinline__ void epi_gather(const float *fmap, const Taps &my_taps, int sub, float (&f)[SUB][4]) {
#pragma unroll
    for (int i = 0; i < SUB; ++i) {
        const int s = sub * SUB + i;
        f[i][0] = f[i][1] = f[i][2] = f[i][3] = 0.0f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            // the taps of sample s were formed once, by lane s (every lane needs the same four)
            const int off = __shfl_sync(0xffffffffu, my_taps.off[k], s);
            const float wk = __shfl_sync(0xffffffffu, my_taps.w[k], s);
            if (off >= 0) {
                const float4 a = ldg4(fmap + off);
                f[i][0] += wk * a.x; f[i][1] += wk * a.y;
                f[i][2] += wk * a.z; f[i][3] += wk * a.w;
            }
        }
    }
}

// For the lane's sample s_mine = sub SUB + (lane & (SUB - 1)) of a sub-chunk: x . f over the 128 channels plus
// pe_half[s_mine][hd].  With qt_hd and sm.scpe this is the sample's score (-inf past S); the backward forms d a
// from dz_hd and sm.dape the same way.
template <int SUB>
__device__ __forceinline__ float epi_sub_dot(const float (&x)[4], const float (&f)[SUB][4],
                                             const float (&pe_half)[32][4], int s_mine, int hd, int lane) {
    float part[SUB];
#pragma unroll
    for (int i = 0; i < SUB; ++i) part[i] = x[0] * f[i][0] + x[1] * f[i][1] + x[2] * f[i][2] + x[3] * f[i][3];
    return transpose_reduce_sub<SUB>(part, lane) + pe_half[s_mine][hd];
}

// The lane's entries of a query's [HEADS, npe] row (e, dpq; HEADS npe <= 96): fn(i, o, head, pe index) for each
// o = lane + 32 i < HEADS npe.
template <int HEADS, class Fn>
__device__ __forceinline__ void for_lane_pe_entries(int npe, int lane, Fn &&fn) {
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const int o = lane + 32 * i;
        if (o < HEADS * npe) fn(i, o, o / npe, o % npe);
    }
}

template <int HEADS, int SUB>
__global__ void __launch_bounds__(kEpiWarps * 32, 4)
k_epi_attn_fwd(EpiParams P, int n_queries, float *__restrict__ z_out, float *__restrict__ e_out,
               float *__restrict__ mass_out, float *__restrict__ lse_out) {
    __shared__ EpiWarpSmem sm_all[kEpiWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    EpiWarpSmem &sm = sm_all[warp];
    const int n = blockIdx.x * kEpiWarps + warp;
    if (n >= n_queries) return;
    float qt[HEADS][4];
    const EpiQuery q = epi_query<HEADS>(P, n, lane, sm, qt, [](int) {}, [](int) {});
    __syncwarp();

    float m_run[HEADS], l_run[HEADS], z[HEADS][4], e_acc[3];   // e_acc: outputs lane, lane+32, lane+64
    float mass_acc[HEADS];                                     // lane ov (< OV) accumulates the mass of view ov
#pragma unroll
    for (int hd = 0; hd < HEADS; ++hd) {
        m_run[hd] = -INFINITY; l_run[hd] = 0.0f; mass_acc[hd] = 0.0f;
        z[hd][0] = z[hd][1] = z[hd][2] = z[hd][3] = 0.0f;
    }
    e_acc[0] = e_acc[1] = e_acc[2] = 0.0f;
    const int nsub = (P.S + SUB - 1) / SUB;

    for (int ov = 0; ov < P.OV; ++ov) {
        const EpiRay ray = epi_ray(P, q, ov, lane);
        Taps my_taps;
        int bx, by;
        float pe[kMaxPE];
        epi_sample<HEADS>(P, ray, n, ov, lane, sm, my_taps, bx, by, pe);
        __syncwarp();

        for (int sub = 0; sub < nsub; ++sub) {
            float f[SUB][4];
            epi_gather<SUB>(P.feat + ray.map_base, my_taps, sub, f);
            // ---- scores: every lane ends up with the score of sample sub*SUB + (lane & (SUB-1))
            const int s_mine = sub * SUB + (lane & (SUB - 1));
            float scale_old[HEADS];
#pragma unroll
            for (int hd = 0; hd < HEADS; ++hd) {
                const float sc = epi_sub_dot<SUB>(qt[hd], f, sm.scpe, s_mine, hd, lane);   // -inf beyond S
                const float m_new = fmaxf(m_run[hd], group_max<SUB>(sc));     // >= one finite score per sub-chunk
                scale_old[hd] = __expf(m_run[hd] - m_new);                     // exp(-inf) = 0 on the first one
                const float pnum = __expf(sc - m_new);                         // exp(-inf) = 0 beyond S
                const float psum = group_add<SUB>(pnum);
                l_run[hd] = l_run[hd] * scale_old[hd] + psum;
                m_run[hd] = m_new;
                if (lane < SUB) sm.p[lane][hd] = pnum;
                if (lane <= ov) mass_acc[hd] = mass_acc[hd] * scale_old[hd] + (lane == ov ? psum : 0.0f);
            }
            __syncwarp();
            // ---- weighted sums
#pragma unroll
            for (int hd = 0; hd < HEADS; ++hd) {
                z[hd][0] *= scale_old[hd]; z[hd][1] *= scale_old[hd];
                z[hd][2] *= scale_old[hd]; z[hd][3] *= scale_old[hd];
            }
#pragma unroll
            for (int i = 0; i < SUB; ++i) {
                float pw[4];
                *reinterpret_cast<float4 *>(pw) = *reinterpret_cast<const float4 *>(sm.p[i]);
#pragma unroll
                for (int hd = 0; hd < HEADS; ++hd) {
                    z[hd][0] += pw[hd] * f[i][0]; z[hd][1] += pw[hd] * f[i][1];
                    z[hd][2] += pw[hd] * f[i][2]; z[hd][3] += pw[hd] * f[i][3];
                }
            }
            // e[h][j] = sum_s p[s][h] * pe[s][j]
            for_lane_pe_entries<HEADS>(P.npe, lane, [&](int i3, int, int hd, int j) {
                float acc = 0.0f;
#pragma unroll
                for (int i = 0; i < SUB; ++i) acc += sm.p[i][hd] * sm.pe[sub * SUB + i][j];
                float so = 0.0f;
#pragma unroll
                for (int k = 0; k < HEADS; ++k) so = (k == hd) ? scale_old[k] : so;
                e_acc[i3] = e_acc[i3] * so + acc;
            });
            __syncwarp();
        }
    }

    // ---- normalise and store
#pragma unroll
    for (int hd = 0; hd < HEADS; ++hd) {
        const float inv = 1.0f / l_run[hd];
        float4 o = make_float4(z[hd][0] * inv, z[hd][1] * inv, z[hd][2] * inv, z[hd][3] * inv);
        *reinterpret_cast<float4 *>(z_out + ((size_t)n * HEADS + hd) * kEpiC + 4 * lane) = o;
        if (lane == 0) lse_out[(size_t)n * HEADS + hd] = m_run[hd] + __logf(l_run[hd]);
        if (mass_out && lane < P.OV) mass_out[((size_t)n * HEADS + hd) * P.OV + lane] = mass_acc[hd] * inv;
    }
    for_lane_pe_entries<HEADS>(P.npe, lane, [&](int i3, int o, int hd, int) {
        float lr = 1.0f;
#pragma unroll
        for (int k = 0; k < HEADS; ++k) lr = (k == hd) ? l_run[k] : lr;
        e_out[(size_t)n * (HEADS * P.npe) + o] = e_acc[i3] / lr;
    });
}

// Slot records of the fixed-order d(feature map) (ps_epipolar_attention_backward_deterministic).  Slot
// t = (n * OV + ov) * S + s is one (query, other view, sample); its record holds the sample's gradient vector
// d f_s [128], its four bilinear tap weights and its cell key
//   m (h+1)(w+1) + (by+1)(w+1) + (bx+1),   m = b V + o_view,  (by, bx) the cell's top-left tap (make_taps),
// for cells that touch an in-bounds texel (by in [-1, h-1], bx in [-1, w-1]); every other slot (invalid ray,
// cell off the map) gets the sentinel key n_cells and no record.
struct EpiDetRecords {
    float *df;            // [T, 128]
    float4 *w;            // [T]
    unsigned *key;        // [T]
    unsigned n_cells;     // B V (h+1) (w+1)
};

// Backward of k_epi_attn_fwd.  Inputs: the forward inputs, lse, the output cotangents (dz, de,
// dmass) and D_h = dz_h.z_h + de_h.e_h + dmass_h.mass_h (flash-attention's row term, formed
// outside by one elementwise pass).  Outputs: dqt, dpq, dbias, and d(feature map) accumulated with
// 16-byte vector atomics (the map gradient is L2-resident; consecutive samples that fall in the
// same bilinear cell are merged in registers first, which removes most of the atomics on short
// epipolar segments).  With lse known every sample is independent, so sub-chunks need no rescaling here.
// DET: instead of the atomics, every slot's record goes to `det` (dfeat is not touched); the sort, per-cell sums
// and per-texel finish below add them up in a fixed order.
template <int HEADS, int SUB, bool DET = false>
__global__ void __launch_bounds__(kEpiWarps * 32, DET ? 3 : 4)   // DET: 168 registers, no spills
k_epi_attn_bwd(EpiParams P, int n_queries, const float *__restrict__ lse, const float *__restrict__ dz,
               const float *__restrict__ de, const float *__restrict__ dmass, const float *__restrict__ Drow,
               float *__restrict__ dqt_out, float *__restrict__ dpq_out, float *__restrict__ dbias_out,
               float *__restrict__ dfeat, EpiDetRecords det) {
    __shared__ EpiWarpSmem sm_all[kEpiWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    EpiWarpSmem &sm = sm_all[warp];
    const int n = blockIdx.x * kEpiWarps + warp;
    if (n >= n_queries) return;
    float qt[HEADS][4], gz[HEADS][4], dq[HEADS][4], lse_h[HEADS], D_h[HEADS];
    const EpiQuery q = epi_query<HEADS>(P, n, lane, sm, qt, [&](int hd) {
        const float4 g = ldg4(dz + ((size_t)n * HEADS + hd) * kEpiC + 4 * lane);
        gz[hd][0] = g.x; gz[hd][1] = g.y; gz[hd][2] = g.z; gz[hd][3] = g.w;
        dq[hd][0] = dq[hd][1] = dq[hd][2] = dq[hd][3] = 0.0f;
        lse_h[hd] = lse[(size_t)n * HEADS + hd];
        D_h[hd] = Drow[(size_t)n * HEADS + hd];
    }, [&](int i) { sm.aux[i / P.npe][i % P.npe] = de[(size_t)n * HEADS * P.npe + i]; });
    __syncwarp();
    float dpq_acc[3] = {0.0f, 0.0f, 0.0f};
    const int nsub = (P.S + SUB - 1) / SUB;

    for (int ov = 0; ov < P.OV; ++ov) {
        const EpiRay ray = epi_ray(P, q, ov, lane);
        Taps my_taps;
        int bx, by;
        float pe[kMaxPE];
        epi_sample<HEADS>(P, ray, n, ov, lane, sm, my_taps, bx, by, pe);
        // ---- PE half of d a (+ dmass), beside the score's
#pragma unroll
        for (int hd = 0; hd < HEADS; ++hd) {
            float da = 0.0f;
#pragma unroll
            for (int j = 0; j < kMaxPE; ++j)
                if (j < P.npe) da += sm.aux[hd][j] * pe[j];
            if (dmass) da += dmass[((size_t)n * HEADS + hd) * P.OV + ov];
            sm.dape[lane][hd] = da;
            sm.ds_all[lane][hd] = 0.0f;
        }
        const int my_cell = by * (P.w + 4) + bx;          // the bilinear cell (samples that share it are merged)
        unsigned my_key = det.n_cells;                    // DET only: the sentinel unless the cell touches the map
        if constexpr (DET) {
            if (bx >= -1 && bx < P.w && by >= -1 && by < P.h)
                my_key = (unsigned)((ray.map * (P.h + 1) + by + 1) * (P.w + 1) + bx + 1);
            if (lane < P.S) {
                const size_t t = ((size_t)n * P.OV + ov) * P.S + lane;
                det.key[t] = my_key;
                if (my_key != det.n_cells) det.w[t] = make_float4(my_taps.w[0], my_taps.w[1], my_taps.w[2], my_taps.w[3]);
            }
        }
        __syncwarp();

        float dbias_acc[HEADS];
#pragma unroll
        for (int hd = 0; hd < HEADS; ++hd) dbias_acc[hd] = 0.0f;
        int cur_base = -0x7fffffff;
        float tap_acc[4][4];
        int tap_off[4] = {-1, -1, -1, -1};
#pragma unroll
        for (int k = 0; k < 4; ++k) tap_acc[k][0] = tap_acc[k][1] = tap_acc[k][2] = tap_acc[k][3] = 0.0f;
        auto flush = [&]() {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (tap_off[k] >= 0)
                    atomicAdd(reinterpret_cast<float4 *>(dfeat + ray.map_base + tap_off[k]),
                              make_float4(tap_acc[k][0], tap_acc[k][1], tap_acc[k][2], tap_acc[k][3]));
                tap_acc[k][0] = tap_acc[k][1] = tap_acc[k][2] = tap_acc[k][3] = 0.0f;
            }
        };

        for (int sub = 0; sub < nsub; ++sub) {
            float f[SUB][4];
            epi_gather<SUB>(P.feat + ray.map_base, my_taps, sub, f);
            const int s_mine = sub * SUB + (lane & (SUB - 1));
#pragma unroll
            for (int hd = 0; hd < HEADS; ++hd) {
                const float sc = epi_sub_dot<SUB>(qt[hd], f, sm.scpe, s_mine, hd, lane);
                const float da = epi_sub_dot<SUB>(gz[hd], f, sm.dape, s_mine, hd, lane);
                const float a = __expf(sc - lse_h[hd]);                 // 0 beyond S (score -inf)
                const float dsc = a * (da - D_h[hd]);
                if (lane < SUB) {
                    sm.p[lane][hd] = a;
                    sm.dsub[lane][hd] = dsc;
                    sm.ds_all[s_mine][hd] = dsc;
                }
                dbias_acc[hd] += group_add<SUB>(dsc);
            }
            __syncwarp();

            // dqt += sum_s ds[s] f[s];  d f[s] = sum_h a[s,h] dz_h + ds[s,h] qt_h  -> scatter to the taps
#pragma unroll
            for (int i = 0; i < SUB; ++i) {
                const int s = sub * SUB + i;
                float aw[4], dw[4];
                *reinterpret_cast<float4 *>(aw) = *reinterpret_cast<const float4 *>(sm.p[i]);
                *reinterpret_cast<float4 *>(dw) = *reinterpret_cast<const float4 *>(sm.dsub[i]);
                float df[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
                for (int hd = 0; hd < HEADS; ++hd) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        dq[hd][c] += dw[hd] * f[i][c];
                        df[c] += aw[hd] * gz[hd][c] + dw[hd] * qt[hd][c];
                    }
                }
                if constexpr (DET) {
                    if (s < P.S && ray.ok) {
                        if (__shfl_sync(0xffffffffu, my_key, s) != det.n_cells)
                            *reinterpret_cast<float4 *>(det.df + (((size_t)n * P.OV + ov) * P.S + s) * kEpiC + 4 * lane) =
                                make_float4(df[0], df[1], df[2], df[3]);
                    }
                } else if (s < P.S && ray.ok) {
                    Taps t;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        t.off[k] = __shfl_sync(0xffffffffu, my_taps.off[k], s);
                        t.w[k] = __shfl_sync(0xffffffffu, my_taps.w[k], s);
                    }
                    // identify the bilinear cell by its top-left tap position (may be outside)
                    const int base = __shfl_sync(0xffffffffu, my_cell, s);
                    if (base != cur_base) {
                        flush();
                        cur_base = base;
#pragma unroll
                        for (int k = 0; k < 4; ++k) tap_off[k] = t.off[k];
                    }
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        tap_acc[k][0] += t.w[k] * df[0]; tap_acc[k][1] += t.w[k] * df[1];
                        tap_acc[k][2] += t.w[k] * df[2]; tap_acc[k][3] += t.w[k] * df[3];
                    }
                }
            }
            __syncwarp();
        }
        if constexpr (!DET) flush();
        if (dbias_out && lane == 0) {
#pragma unroll
            for (int hd = 0; hd < HEADS; ++hd) dbias_out[((size_t)n * HEADS + hd) * P.OV + ov] = dbias_acc[hd];
        }
        // dpq[h][j] += sum_s ds[s][h] pe[s][j]
        for_lane_pe_entries<HEADS>(P.npe, lane, [&](int i, int, int hd, int j) {
            float acc = 0.0f;
            for (int s = 0; s < 32; ++s) acc += sm.ds_all[s][hd] * sm.pe[s][j];
            dpq_acc[i] += acc;
        });
        __syncwarp();
    }
#pragma unroll
    for (int hd = 0; hd < HEADS; ++hd)
        *reinterpret_cast<float4 *>(dqt_out + ((size_t)n * HEADS + hd) * kEpiC + 4 * lane) =
            make_float4(dq[hd][0], dq[hd][1], dq[hd][2], dq[hd][3]);
    for_lane_pe_entries<HEADS>(P.npe, lane,
                               [&](int i, int o, int, int) { dpq_out[(size_t)n * (HEADS * P.npe) + o] = dpq_acc[i]; });
}

constexpr int kEpiSubFwd = 8, kEpiSubBwd = 4;

// fn(std::integral_constant<int, heads>()) for heads in [1, 4] (epi_check has checked the range).
template <class Fn>
static void with_heads(int heads, Fn &&fn) {
    switch (heads) {
        case 1: fn(std::integral_constant<int, 1>()); break;
        case 2: fn(std::integral_constant<int, 2>()); break;
        case 3: fn(std::integral_constant<int, 3>()); break;
        default: fn(std::integral_constant<int, 4>()); break;
    }
}

static int launch_epi_fwd(const EpiParams &P, int heads, int n, float *z, float *e, float *mass, float *lse,
                          cudaStream_t st) {
    static int sub_fwd = 0;                           // PIXELSPLAT_B200_EPI_SUB_FWD = 4 | 8 (A/B runs)
    if (sub_fwd == 0) {
        const char *env = getenv("PIXELSPLAT_B200_EPI_SUB_FWD");
        sub_fwd = (env && env[0] == '4') ? 4 : kEpiSubFwd;
    }
    const int blocks = (n + kEpiWarps - 1) / kEpiWarps;
    with_heads(heads, [&](auto H) {
        constexpr int HEADS = decltype(H)::value;
        if (sub_fwd == 4) k_epi_attn_fwd<HEADS, 4><<<blocks, kEpiWarps * 32, 0, st>>>(P, n, z, e, mass, lse);
        else k_epi_attn_fwd<HEADS, kEpiSubFwd><<<blocks, kEpiWarps * 32, 0, st>>>(P, n, z, e, mass, lse);
    });
    PS_LAUNCH_CHECK("k_epi_attn_fwd");
    return PS_OK;
}

// The backward's cotangents and gradients, as its entry points take them.
struct EpiGrads {
    const float *lse, *dz, *de, *dmass, *d_row;
    float *dq_feat, *dq_pe, *dbias, *dfeatures;
};

// DET: the slot records go to `det`, and dfeatures is left to the fixed-order sum that follows.
template <bool DET>
static int launch_epi_bwd(const EpiParams &P, int heads, int n, const EpiGrads &g, const EpiDetRecords &det,
                          cudaStream_t st) {
    with_heads(heads, [&](auto H) {
        k_epi_attn_bwd<decltype(H)::value, kEpiSubBwd, DET><<<(n + kEpiWarps - 1) / kEpiWarps, kEpiWarps * 32, 0, st>>>(
            P, n, g.lse, g.dz, g.de, g.dmass, g.d_row, g.dq_feat, g.dq_pe, g.dbias, DET ? nullptr : g.dfeatures, det);
    });
    PS_LAUNCH_CHECK(DET ? "k_epi_attn_bwd<DET>" : "k_epi_attn_bwd");
    return PS_OK;
}

// ---- fixed-order d(feature map) -------------------------------------------------------------------------------
// A stable LSD radix sort of the slot ids by cell key (8-bit digits, reduce-then-scan), then one warp per cell sums
// its slots' weighted records in ascending slot id, then one warp per texel adds its four cells' tap sums in a fixed
// order.  Every sum runs in an order fixed by the inputs, so the result is the same bits on every run.
constexpr int kSortThreads = 256, kSortTiles = 16, kSortChunk = kSortThreads * kSortTiles;   // slots per chunk
constexpr int kScanThreads = 1024;

// hist[d * chunks + c] = number of slots of chunk c whose digit is d.
__global__ void __launch_bounds__(kSortThreads)
k_epi_radix_hist(const unsigned *__restrict__ keys, int T, int shift, int chunks, unsigned *__restrict__ hist) {
    __shared__ unsigned h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int base = blockIdx.x * kSortChunk;
    for (int i = threadIdx.x; i < kSortChunk; i += kSortThreads)
        if (base + i < T) atomicAdd(&h[(keys[base + i] >> shift) & 255u], 1u);   // integer counts: order-free
    __syncthreads();
    hist[(size_t)threadIdx.x * chunks + blockIdx.x] = h[threadIdx.x];
}

// Exclusive scan of the [256, chunks] histogram in place (digit-major: digit d of chunk c starts after every
// smaller digit and after digit d of every earlier chunk).  One block; each thread scans a contiguous run.
__global__ void __launch_bounds__(kScanThreads)
k_epi_radix_scan(unsigned *__restrict__ hist, int m) {
    __shared__ unsigned warp_tot[kScanThreads / 32];
    const int per = (m + kScanThreads - 1) / kScanThreads;
    const int beg = min(m, (int)threadIdx.x * per), end = min(m, beg + per);
    unsigned sum = 0;
    for (int i = beg; i < end; ++i) sum += hist[i];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        unsigned t = warp_tot[lane], ti = t;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(0xffffffffu, ti, o);
            if (lane >= o) ti += y;
        }
        warp_tot[lane] = ti - t;
    }
    __syncthreads();
    unsigned run = warp_tot[warp] + incl - sum;
    for (int i = beg; i < end; ++i) {
        const unsigned c = hist[i];
        hist[i] = run;
        run += c;
    }
}

// Stable scatter of one chunk: tiles of 256 slots in order; inside a tile, a slot's position among equal digits is
// (earlier chunks and tiles) + (earlier warps) + (earlier lanes, from match.any).  ids_in NULL = the identity.
__global__ void __launch_bounds__(kSortThreads)
k_epi_radix_scatter(const unsigned *__restrict__ keys_in, const unsigned *__restrict__ ids_in, int T, int shift,
                    int chunks, const unsigned *__restrict__ offsets, unsigned *__restrict__ keys_out,
                    unsigned *__restrict__ ids_out) {
    constexpr int kWarps = kSortThreads / 32;
    __shared__ unsigned wcnt[kWarps][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned run = offsets[(size_t)threadIdx.x * chunks + blockIdx.x];   // thread d keeps digit d's cursor
    const unsigned lt = (1u << lane) - 1u;
    for (int tile = 0; tile < kSortTiles; ++tile) {
        const int idx = blockIdx.x * kSortChunk + tile * kSortThreads + threadIdx.x;
#pragma unroll
        for (int j = 0; j < kWarps; ++j) wcnt[j][threadIdx.x] = 0;
        __syncthreads();
        const bool valid = idx < T;
        const unsigned key = valid ? keys_in[idx] : 0u;
        const unsigned id = valid ? (ids_in ? ids_in[idx] : (unsigned)idx) : 0u;
        const unsigned d = valid ? (key >> shift) & 255u : 256u;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const unsigned rank = __popc(peers & lt);
        if (valid && rank == 0) wcnt[warp][d] = __popc(peers);
        __syncthreads();
        {
            unsigned acc = run;
#pragma unroll
            for (int j = 0; j < kWarps; ++j) {
                const unsigned c = wcnt[j][threadIdx.x];
                wcnt[j][threadIdx.x] = acc;
                acc += c;
            }
            run = acc;
        }
        __syncthreads();
        if (valid) {
            const unsigned pos = wcnt[warp][d] + rank;
            keys_out[pos] = key;
            ids_out[pos] = id;
        }
        __syncthreads();
    }
}

// cell_start[c] = first sorted position whose key is >= c, for c in [0, n_cells]; cell_start[n_cells] = the number
// of slots with a record.  Position i fills the cells in (key[i-1], key[i]].
__global__ void k_epi_cell_bounds(const unsigned *__restrict__ keys, int T, unsigned n_cells,
                                  unsigned *__restrict__ cell_start) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > T) return;
    const long long hi = i < T ? (long long)keys[i] : (long long)n_cells;
    const long long lo = i > 0 ? (long long)keys[i - 1] : -1;
    for (long long c = lo + 1; c <= hi; ++c) cell_start[c] = (unsigned)i;
}

// One warp per cell, lane = 4 channels: cell_sum[c][k] = sum over the cell's slots, in ascending slot id, of
// w_k * d f.  An empty cell writes zeros.
constexpr int kCellWarps = 8;
__global__ void __launch_bounds__(kCellWarps * 32)
k_epi_cell_sums(const float *__restrict__ df, const float4 *__restrict__ w, const unsigned *__restrict__ ids,
                const unsigned *__restrict__ cell_start, unsigned n_cells, float *__restrict__ cell_sum) {
    const int lane = threadIdx.x & 31;
    const unsigned c = blockIdx.x * kCellWarps + (threadIdx.x >> 5);
    if (c >= n_cells) return;
    const unsigned beg = cell_start[c], end = cell_start[c + 1];
    float acc[4][4] = {};
#pragma unroll 4
    for (unsigned j = beg; j < end; ++j) {
        const unsigned t = ids[j];
        const float4 wk = w[t];
        const float4 g = ldg4(df + (size_t)t * kEpiC + 4 * lane);
        const float wv[4] = {wk.x, wk.y, wk.z, wk.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            acc[k][0] += wv[k] * g.x; acc[k][1] += wv[k] * g.y;
            acc[k][2] += wv[k] * g.z; acc[k][3] += wv[k] * g.w;
        }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
        *reinterpret_cast<float4 *>(cell_sum + ((size_t)c * 4 + k) * kEpiC + 4 * lane) =
            make_float4(acc[k][0], acc[k][1], acc[k][2], acc[k][3]);
}

// One warp per texel (y, x) of map m, lane = 4 channels: the four cells whose taps land on it, in a fixed order --
// (y-1, x-1) tap 3, (y-1, x) tap 2, (y, x-1) tap 1, (y, x) tap 0.  Writes every texel.
__global__ void __launch_bounds__(kCellWarps * 32)
k_epi_texel_finish(const float *__restrict__ cell_sum, int n_texels, int h, int w, float *__restrict__ dfeat) {
    const int lane = threadIdx.x & 31;
    const int q = blockIdx.x * kCellWarps + (threadIdx.x >> 5);
    if (q >= n_texels) return;
    const int x = q % w, y = (q / w) % h, m = q / (w * h);
    const size_t c0 = ((size_t)m * (h + 1) + y) * (w + 1) + x;          // cell (y-1, x-1)
    const float *base = cell_sum + 4 * lane;
    const float4 a = ldg4(base + (c0 * 4 + 3) * kEpiC);
    const float4 b = ldg4(base + ((c0 + 1) * 4 + 2) * kEpiC);
    const float4 c = ldg4(base + ((c0 + w + 1) * 4 + 1) * kEpiC);
    const float4 d = ldg4(base + ((c0 + w + 2) * 4 + 0) * kEpiC);
    *reinterpret_cast<float4 *>(dfeat + (size_t)q * kEpiC + 4 * lane) =
        make_float4(((a.x + b.x) + c.x) + d.x, ((a.y + b.y) + c.y) + d.y, ((a.z + b.z) + c.z) + d.z,
                    ((a.w + b.w) + c.w) + d.w);
}

// Workspace of the deterministic backward (A(x) = x rounded up to 256; the header states the same formula).
struct EpiDetLayout {
    long long T;                  // slots
    unsigned n_cells;
    int chunks, passes;
    size_t df, w, key[2], id[2], hist, cell_start, cell_sum, total;
};

static size_t align256(size_t x) { return (x + 255) / 256 * 256; }

static int epi_det_layout(const ps_epipolar_desc *d, EpiDetLayout *L) {
    const long long rays = (long long)d->batch * d->views * d->grid_h * d->grid_w;
    const long long T = rays * (d->views - 1) * d->samples;
    const long long cells = (long long)d->batch * d->views * (d->grid_h + 1) * (d->grid_w + 1);
    if (rays > 0x7fffffffLL || T > 0x7fffffffLL || cells >= 0x7fffffffLL) {
        set_error("ps_epipolar_attention_backward_deterministic: b*v*R*(v-1)*S slots and b*v*(h+1)*(w+1) cells must fit 31 bits");
        return PS_ERR_UNSUPPORTED;
    }
    L->T = T;
    L->n_cells = (unsigned)cells;
    L->chunks = (int)((T + kSortChunk - 1) / kSortChunk);
    const int bits = 32 - __builtin_clz(L->n_cells);          // the sentinel key n_cells needs this many bits
    L->passes = (bits + 7) / 8;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += align256(bytes); return o; };
    L->df = take(512 * (size_t)T);
    L->w = take(16 * (size_t)T);
    L->key[0] = take(4 * (size_t)T);
    L->key[1] = take(4 * (size_t)T);
    L->id[0] = take(4 * (size_t)T);
    L->id[1] = take(4 * (size_t)T);
    L->hist = take(4 * 256 * (size_t)L->chunks);
    L->cell_start = take(4 * ((size_t)cells + 1));
    L->cell_sum = take(2048 * (size_t)cells);
    L->total = off;
    return PS_OK;
}

static int launch_epi_bwd_det(const EpiParams &P, int heads, int n, const EpiDetLayout &L, char *ws,
                              const EpiGrads &g, cudaStream_t st) {
    EpiDetRecords rec;
    rec.df = reinterpret_cast<float *>(ws + L.df);
    rec.w = reinterpret_cast<float4 *>(ws + L.w);
    rec.key = reinterpret_cast<unsigned *>(ws + L.key[0]);
    rec.n_cells = L.n_cells;
    const int rc = launch_epi_bwd<true>(P, heads, n, g, rec, st);
    if (rc) return rc;

    const int T = (int)L.T;
    unsigned *hist = reinterpret_cast<unsigned *>(ws + L.hist);
    int cur = 0;                                                   // ping-pong buffer holding the current order
    for (int pass = 0; pass < L.passes; ++pass) {
        const unsigned *keys_in = reinterpret_cast<const unsigned *>(ws + L.key[cur]);
        const unsigned *ids_in = pass == 0 ? nullptr : reinterpret_cast<const unsigned *>(ws + L.id[cur]);
        k_epi_radix_hist<<<L.chunks, kSortThreads, 0, st>>>(keys_in, T, 8 * pass, L.chunks, hist);
        PS_LAUNCH_CHECK("k_epi_radix_hist");
        k_epi_radix_scan<<<1, kScanThreads, 0, st>>>(hist, 256 * L.chunks);
        PS_LAUNCH_CHECK("k_epi_radix_scan");
        k_epi_radix_scatter<<<L.chunks, kSortThreads, 0, st>>>(
            keys_in, ids_in, T, 8 * pass, L.chunks, hist, reinterpret_cast<unsigned *>(ws + L.key[cur ^ 1]),
            reinterpret_cast<unsigned *>(ws + L.id[cur ^ 1]));
        PS_LAUNCH_CHECK("k_epi_radix_scatter");
        cur ^= 1;
    }
    unsigned *cell_start = reinterpret_cast<unsigned *>(ws + L.cell_start);
    k_epi_cell_bounds<<<(T + 1 + 255) / 256, 256, 0, st>>>(reinterpret_cast<const unsigned *>(ws + L.key[cur]), T,
                                                          L.n_cells, cell_start);
    PS_LAUNCH_CHECK("k_epi_cell_bounds");
    float *cell_sum = reinterpret_cast<float *>(ws + L.cell_sum);
    k_epi_cell_sums<<<(L.n_cells + kCellWarps - 1) / kCellWarps, kCellWarps * 32, 0, st>>>(
        rec.df, rec.w, reinterpret_cast<const unsigned *>(ws + L.id[cur]), cell_start, L.n_cells, cell_sum);
    PS_LAUNCH_CHECK("k_epi_cell_sums");
    const int texels = P.B * P.V * P.h * P.w;
    k_epi_texel_finish<<<(texels + kCellWarps - 1) / kCellWarps, kCellWarps * 32, 0, st>>>(cell_sum, texels, P.h, P.w,
                                                                                            g.dfeatures);
    PS_LAUNCH_CHECK("k_epi_texel_finish");
    return PS_OK;
}

static int epi_check(const ps_epipolar_desc *d) {
    if (!d) { set_error("desc is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    if (d->batch < 1 || d->views < 2 || d->grid_h < 1 || d->grid_w < 1) {
        set_error("ps_epipolar: need batch >= 1, views >= 2, positive grid"); return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->channels != kEpiC) { set_error("ps_epipolar: channels must be %d, got %d", kEpiC, d->channels); return PS_ERR_UNSUPPORTED; }
    if (d->heads < 1 || d->heads > 4) { set_error("ps_epipolar: heads must be in [1, 4], got %d", d->heads); return PS_ERR_UNSUPPORTED; }
    if (d->samples < 1 || d->samples > 32) { set_error("ps_epipolar: samples must be in [1, 32], got %d", d->samples); return PS_ERR_UNSUPPORTED; }
    if (d->pe_dim < 0 || d->pe_dim > kMaxPE || (d->pe_dim & 1) || d->heads * d->pe_dim > 96) {
        set_error("ps_epipolar: pe_dim must be even, <= %d and heads*pe_dim <= 96 (got %d)", kMaxPE, d->pe_dim);
        return PS_ERR_UNSUPPORTED;
    }
    if (d->views - 1 > 32) { set_error("ps_epipolar: at most 33 views"); return PS_ERR_UNSUPPORTED; }
    return PS_OK;
}

// Argument check of the attention entry points, before anything is enqueued: the descriptor, `in` and the inputs
// every call reads, then the entry point's own pointers -- `always` must be non-NULL, `with_pe` too when pe_dim > 0.
static int epi_check_call(const char *who, const ps_epipolar_desc *d, const ps_epipolar_inputs *in,
                          std::initializer_list<const void *> always, std::initializer_list<const void *> with_pe) {
    const int rc = epi_check(d);
    if (rc) return rc;
    bool ok = in && in->features && in->segments && in->valid && in->rel_disparity && in->q_feat &&
              (d->pe_dim == 0 || in->q_pe);
    for (const void *p : always) ok = ok && p;
    if (d->pe_dim > 0)
        for (const void *p : with_pe) ok = ok && p;
    if (!ok) { set_error("%s: a required pointer is NULL", who); return PS_ERR_INVALID_ARGUMENT; }
    return PS_OK;
}

static EpiParams epi_params(const ps_epipolar_desc *d, const ps_epipolar_inputs *in) {
    EpiParams P;
    P.B = d->batch; P.V = d->views; P.OV = d->views - 1; P.h = d->grid_h; P.w = d->grid_w; P.S = d->samples;
    P.npe = d->pe_dim; P.feat = in->features; P.seg = in->segments; P.valid = in->valid;
    P.rd = in->rel_disparity; P.qt = in->q_feat; P.pq = in->q_pe; P.bias = in->bias;
    return P;
}

}  // namespace ps

using namespace ps;

extern "C" PS_API int ps_epipolar_attention_forward(const ps_epipolar_desc *d, const ps_epipolar_inputs *in,
                                                    float *z, float *e, float *mass, float *lse, void *stream) {
    const int rc = epi_check_call("ps_epipolar_attention_forward", d, in, {z, lse}, {e});
    if (rc) return rc;
    return launch_epi_fwd(epi_params(d, in), d->heads, d->batch * d->views * d->grid_h * d->grid_w, z, e, mass, lse,
                          static_cast<cudaStream_t>(stream));
}

extern "C" PS_API int ps_epipolar_attention_backward(const ps_epipolar_desc *d, const ps_epipolar_inputs *in,
                                                     const float *lse, const float *dz, const float *de,
                                                     const float *dmass, const float *d_row, float *dq_feat,
                                                     float *dq_pe, float *dbias, float *dfeatures, void *stream) {
    const int rc = epi_check_call("ps_epipolar_attention_backward", d, in, {lse, dz, d_row, dq_feat, dfeatures},
                                  {de, dq_pe});
    if (rc) return rc;
    const EpiGrads g{lse, dz, de, dmass, d_row, dq_feat, dq_pe, dbias, dfeatures};
    return launch_epi_bwd<false>(epi_params(d, in), d->heads, d->batch * d->views * d->grid_h * d->grid_w, g,
                                 EpiDetRecords{}, static_cast<cudaStream_t>(stream));
}

extern "C" PS_API int ps_epipolar_attention_backward_workspace_bytes(const ps_epipolar_desc *d, size_t *out) {
    int rc = epi_check(d);
    if (rc) return rc;
    if (!out) { set_error("ps_epipolar_attention_backward_workspace_bytes: out is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    EpiDetLayout L;
    if ((rc = epi_det_layout(d, &L))) return rc;
    *out = L.total;
    return PS_OK;
}

extern "C" PS_API int ps_epipolar_attention_backward_deterministic(
        const ps_epipolar_desc *d, const ps_epipolar_inputs *in, const float *lse, const float *dz, const float *de,
        const float *dmass, const float *d_row, float *dq_feat, float *dq_pe, float *dbias, float *dfeatures,
        void *workspace, size_t workspace_bytes, void *stream) {
    int rc = epi_check_call("ps_epipolar_attention_backward_deterministic", d, in,
                            {lse, dz, d_row, dq_feat, dfeatures, workspace}, {de, dq_pe});
    if (rc) return rc;
    EpiDetLayout L;
    if ((rc = epi_det_layout(d, &L))) return rc;
    if (workspace_bytes < L.total) {
        set_error("ps_epipolar_attention_backward_deterministic: workspace of %zu bytes, %zu needed", workspace_bytes,
                  L.total);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const EpiGrads g{lse, dz, de, dmass, d_row, dq_feat, dq_pe, dbias, dfeatures};
    return launch_epi_bwd_det(epi_params(d, in), d->heads, d->batch * d->views * d->grid_h * d->grid_w, L,
                              static_cast<char *>(workspace), g, static_cast<cudaStream_t>(stream));
}
