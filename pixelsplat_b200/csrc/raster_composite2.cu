// Alpha compositing, forward and backward, as independent WARP TASKS (round-2 compositor).
//
// A task is one 8x4 pixel block of one (view, 16x16 tile); a warp owns a task from start to end and
// never meets another warp at a barrier.  Replaces the per-pixel blend loop of upstream's renderCUDA
// (SURVEY.md A.3 / A.5; the call the reference makes at
// /root/reference/src/model/decoder/cuda_splatting.py:113-124) without changing a per-pixel decision.
//
// Front end (shared by both directions): the warp streams the tile's LIVE LIST 32 records at a time (written by
// the tile sort, ps_common.cuh: the entries whose alpha >= 1/255 box meets the tile, in list order, each with the
// mask of the 8x4 blocks the box meets), takes a ballot of its block's mask bit, and only for the hits gathers
// position/conic/opacity/colour into a per-warp shared-memory queue.  The box test happened once per entry in the
// sort, not once per block here.  The loads are software-pipelined across iterations (records one chunk ahead,
// hit records parked one iteration later), so nothing waits on L2.
//
// Both kernels are bound by instruction issue (ncu: 65-80 % issue-active forward), so the per-hit loop is
// built to be short:
//   * a queued hit carries its log2-power as a POLYNOMIAL in the block-local pixel offsets (i, j in 0..7 x
//     0..3, lane = 8 j + i):  p2(i, j) = A + i (B + i qa + j qb) + j (C + j qc), five FFMAs per (hit, pixel)
//     with the coefficients formed once per hit by the lane that queues it.  Offsets are measured from the
//     block origin, so |A|, |B i|, ... stay O(10) for every hit that can contribute and the rounding error
//     of the expansion is ~1e-6 absolute in the exponent (the MUFU.EX2 that follows is no better).  Upstream's
//     `power > 0` rejection (unreachable for a positive-definite conic except through rounding) becomes
//     `p2 > 1e-4` so that this rounding cannot drop a pixel that sits on a Gaussian's centre;
//   * the queue is a ring consumed in ALIGNED GROUPS OF FOUR (zero-opacity records pad the last group):
//     one address computation per group, no per-entry bounds logic.
//
// Backward: per batch of queued hits
//   phase 1 (lane = pixel): walk the batch FRONT TO BACK carrying (T, S) with
//            S_i = sum_{j<=i} w_j (c_j . dL/dC),  w_j = alpha_j T_j,  and, from the forward's stored
//            pixel colour C,  Q = C . dL/dC = S_last + T_final (bg . dL/dC):
//            dL/dalpha_i = T_i (c_i . dL/dC) - (Q - S_i) / (1 - alpha_i)
//            (algebraically upstream's back-to-front recurrence).  Writes the two scalars every
//            gradient is built from, u = G dL/dalpha and w, to shared memory [entry][pixel];
//   phase 2 (lane = entry): each lane sums its entry's RAW moments sum_p u (1, i, j, i^2, i j, j^2) and
//            sum_p w dL/dC over the block's pixels straight out of shared memory (i, j are literals in the
//            unrolled loop: ~4 FFMAs per pixel), shifts them to the Gaussian's centre once, and adds the nine
//            gradients to the per-(view, Gaussian) scratch with three vector RED instructions.
//
// List SEGMENTS (d.segK = 1, 2 or 4 warps per task).  One 256x256 view is only 2048 tasks -- 14 warps per
// SM, each a long serial chain -- so when the batch is small a tile's sorted list is cut into segK runs of
// whole 32-entry chunks and each run gets its own warp:
//   forward : every warp composites its run as if nothing lay in front of it (T = 1), giving (C_k, T_k);
//             front-to-back composition is associative, (C, T) o (C_k, T_k) = (C + T C_k, T T_k), so one warp
//             folds the runs in order.  Upstream's early exit (stop once T (1 - alpha) < 1e-4) depends on
//             the true T, so a run is accepted only when T T_k stays clear of the threshold (T T_k is a lower
//             bound of every intermediate test); otherwise -- rare: the pixel saturates inside this run --
//             the run is replayed for those pixels with the true T, i.e. exactly the sequential loop.
//             The state in front of each run, (T, C), is kept per pixel for the backward.
//   backward: the forward-order prefix form needs only (T, S = C . dL/dC) in front of a run, which the
//             forward stored, so the runs are independent warps with no combination step at all.
//
// Fixed-order (DET) instantiations, for the "deterministic" option (include/pixelsplat_b200.h): the same kernels
// with the two float-atomic sums replaced by stores and a fixed-order reduction afterwards.
//   backward: phase 2 STORES its ten numbers (d_mean2d x2, d_conic x3, d_opacity, d_color x3, depth lane) into the
//             record of (tile block, list position): index tile_start * 8 + block * count + position, the index space
//             of the forward's hit lists.  Each record has exactly one writer: a list position lies in exactly one run
//             (K = 1 / 2 / 4), each (tile, block) is exactly one warp task, and a task queues a position at most once.
//             k_gather_block_records then sums, per on-screen (view, Gaussian), its records in a fixed order (tiles
//             row-major within a block, then blocks 0..7) and stores the per-(view, Gaussian) gradients
//             k_preprocess_bwd reads.
//   forward : the loss epilogue stores each warp task's (sse, sse_clipped) pair; k_loss_finish sums each view's
//             tasks in a fixed order into the PS_LOSS_SLOTS slots.
// Everything else (K, hit lists, cull, the arithmetic that forms the numbers) is the default instantiations'.
#include <cstdlib>

#include "ps_common.cuh"

namespace ps {

namespace {

constexpr int kQ = 64;                  // hit-queue slots per warp (ring, consumed in aligned groups of 4)
constexpr float kAlphaMin = 1.0f / 255.0f;
constexpr float kPowerEps = 1.0e-4f;    // see the file header: rounding slack of the polynomial exponent
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ float fast_rcp(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ void red_add_v4(float4 *addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

__device__ __forceinline__ void red_add_v2(float2 *addr, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// Per-warp hit queue (see the file header for the polynomial form).
struct HitQueue {
    float4 r0[kQ];   // A, B, C, opacity
    float4 r1[kQ];   // qa, qb, qc, list position (bits)
    float4 r2[kQ];   // r, g, b, Gaussian id (bits) -- forward with a depth channel: r, g, b, depth value d
};

// log2 of the Gaussian falloff at block-local pixel (fi, fj)
__device__ __forceinline__ float hit_power2(const float4 &a0, const float4 &a1, float fi, float fj) {
    const float t1 = fmaf(fj, a1.y, fmaf(fi, a1.x, a0.y));     // B + i qa + j qb
    const float t2 = fmaf(fj, a1.z, a0.z);                     // C + j qc
    return fmaf(fj, t2, fmaf(fi, t1, a0.x));
}

// Registers of the live-list pipeline (see file header).
struct CullPipe {
    uint2 rec;                     // live record of chunk c (this lane's entry)
    // hit of chunk c - 1 waiting to be parked in the queue
    float4 h_co, h_rgb;
    float2 h_xy;
    uint32_t h_g, h_pos, h_slot;
    bool h_pending;
};

struct TaskGeom {
    int vid, pxi, pyi, sub;
    bool inside;
    float fi, fj;                 // block-local pixel offsets of this lane (0..7, 0..3)
    float rx0, ry0;               // the block's origin
    uint32_t start, count;        // the tile's list
    uint32_t run_begin, run_len;  // this warp's run of it, in list positions (whole list when segK == 1)
    const uint2 *live;            // the tile's live list (ps_common.cuh, kLivePosLimit)
    uint32_t n_live;              // its length
    uint32_t live_begin;          // index of the run's first live entry; the run takes the live entries from there
                                  // on whose position is < run_begin + run_len
    size_t gbase, pix, hw;
};

// Run k of segK over a list of `count` entries: whole 32-entry chunks of the FULL list, the same split in both
// directions (so the fold of the runs, and with it every pixel's bits, does not depend on the live lists).
__device__ __forceinline__ void run_bounds(uint32_t count, int segK, int k, uint32_t &begin, uint32_t &len) {
    const uint32_t chunks = (count + 31u) >> 5;
    const uint32_t per = (chunks + (uint32_t)segK - 1u) / (uint32_t)segK;
    begin = min(count, (uint32_t)k * per * 32u);
    len = min(count, (uint32_t)(k + 1) * per * 32u) - begin;
}

__device__ __forceinline__ bool task_setup(const Dims &d, const Geom &geo, const uint2 *live, long long task, int lane,
                                           TaskGeom &t) {
    t.sub = (int)(task & 7);
    const long long seg = task >> 3;
    if (seg >= (long long)d.S * d.V * d.tiles) return false;
    t.vid = (int)(seg / d.tiles);
    const int tile = (int)(seg - (long long)t.vid * d.tiles);
    const int tx = tile % d.gx, ty = tile / d.gx;
    const int wx0 = tx * kTile + (t.sub & 1) * 8, wy0 = ty * kTile + (t.sub >> 1) * 4;
    t.pxi = wx0 + (lane & 7);
    t.pyi = wy0 + (lane >> 3);
    t.inside = t.pxi < d.W && t.pyi < d.H;
    t.fi = (float)(lane & 7); t.fj = (float)(lane >> 3);
    t.rx0 = (float)wx0; t.ry0 = (float)wy0;
    t.start = geo.tile_start[seg];
    t.count = geo.tile_count[seg];
    t.run_begin = 0;
    t.run_len = t.count;
    t.live = live + t.start;
    t.n_live = 0;
    t.live_begin = 0;
    t.gbase = (size_t)t.vid * d.P;
    t.hw = (size_t)d.H * d.W;
    t.pix = (size_t)t.pyi * d.W + t.pxi;
    return true;
}

// Index of the first live entry at list position >= pos (n_live if none): a 32-way search, two or three rounds of
// coalescing-free but independent loads for the lists seen in practice.
__device__ __forceinline__ uint32_t live_lower_bound(const TaskGeom &t, uint32_t pos, int lane) {
    if (t.count > kLivePosLimit) return min(pos, t.n_live);     // every entry kept: index = position
    uint32_t lo = 0, hi = t.n_live;                             // the answer lies in [lo, hi]
    while (lo < hi) {
        const uint32_t step = (hi - lo + 31u) >> 5;
        const uint32_t i = lo + (uint32_t)lane * step;
        const bool below = i < hi && (t.live[i].x >> 8) < pos;
        const uint32_t c = (uint32_t)__popc(__ballot_sync(0xffffffffu, below));
        if (c == 0) break;
        lo += (c - 1u) * step + 1u;       // past the last probe below pos; the next probe (if any) is not
        hi = min(hi, lo - 1u + step);
    }
    return lo;
}

// Positions the run [run_begin, run_begin + run_len) of the task's list on its live list.
__device__ __forceinline__ void live_run(TaskGeom &t, const Geom &geo, long long task, int lane) {
    t.n_live = geo.tile_cursor[task >> 3];
    t.live_begin = t.run_len == 0 ? t.n_live : t.run_begin == 0 ? 0u : live_lower_bound(t, t.run_begin, lane);
}

// ---- live-list pipeline ---------------------------------------------------------------------------
__device__ __forceinline__ void cull_prologue(CullPipe &p, const TaskGeom &t, int lane) {
    p.h_pending = false;
    p.h_slot = 0; p.h_g = 0; p.h_pos = 0;
    p.h_xy = make_float2(0.0f, 0.0f);
    p.h_co = p.h_rgb = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    p.rec = make_uint2(0u, 0u);
    if (t.live_begin + (uint32_t)lane < t.n_live) p.rec = t.live[t.live_begin + lane];
}

// Parks the hit found in the previous iteration (its gathers have had a whole iteration to land): forms the
// polynomial coefficients of the hit about the block origin.  D0 = also keep (dx0, dy0) for the backward.
// DEPTH: the forward carries the depth value in r2.w instead of the id (it never reads the id); the backward keeps
// the id there and parks the depth value in dd[].
template <bool D0, bool DEPTH = false>
__device__ __forceinline__ void cull_park(CullPipe &p, HitQueue &q, float2 *d0, const TaskGeom &t,
                                          float *dd = nullptr) {
    if (p.h_pending) {
        const float qa = -0.5f * kLog2e * p.h_co.x, qb = -kLog2e * p.h_co.y, qc = -0.5f * kLog2e * p.h_co.z;
        const float dx0 = p.h_xy.x - t.rx0, dy0 = p.h_xy.y - t.ry0;
        const float ax = qa * dx0, cy = qc * dy0;
        const float A = fmaf(ax, dx0, fmaf(cy, dy0, qb * dx0 * dy0));
        const float B = -(2.0f * ax + qb * dy0);
        const float C = -(2.0f * cy + qb * dx0);
        q.r0[p.h_slot] = make_float4(A, B, C, p.h_co.w);
        q.r1[p.h_slot] = make_float4(qa, qb, qc, __uint_as_float(p.h_pos));
        q.r2[p.h_slot] = make_float4(p.h_rgb.x, p.h_rgb.y, p.h_rgb.z,
                                     (DEPTH && !D0) ? p.h_rgb.w : __uint_as_float(p.h_g));
        if (D0) d0[p.h_slot] = make_float2(dx0, dy0);
        if (D0 && DEPTH) dd[p.h_slot] = p.h_rgb.w;
    }
    p.h_pending = false;
    __syncwarp();
}

// Zero-opacity records up to the next multiple of four (they can never contribute: alpha = 0 < 1/255).  Their
// colour (and depth value, dd) is zero too, so that a weight of zero never meets an uninitialised value.
__device__ __forceinline__ uint32_t queue_pad(HitQueue &q, uint32_t tail, int lane, float *dd = nullptr) {
    const uint32_t padded = (tail + 3u) & ~3u;
    if ((uint32_t)lane < padded - tail) {
        const uint32_t slot = (tail + (uint32_t)lane) & (kQ - 1);
        q.r0[slot] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        q.r1[slot] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(0xffffffffu));   // position beyond any `last`
        q.r2[slot] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (dd) dd[slot] = 0.0f;
    }
    __syncwarp();
    return padded;
}

// Takes chunk c of the run's live entries (indices live_begin + 32c ...): the block's mask bit decides, nothing is
// box-tested here.  Returns the number of hits -- they become readable in the queue after the NEXT cull_park -- or
// -1 when the chunk lies past the run.
__device__ __forceinline__ int cull_step(CullPipe &p, const Geom &geo, const TaskGeom &t, uint32_t c, uint32_t tail,
                                         int lane, uint2 *__restrict__ hit_out = nullptr) {
    const uint32_t i = t.live_begin + c * 32u + (uint32_t)lane;
    const uint2 rec = p.rec;
    const uint32_t pos = t.count > kLivePosLimit ? i : rec.x >> 8;   // position in the TILE's list
    const bool in_run = i < t.n_live && pos < t.run_begin + t.run_len;
    if (!__any_sync(0xffffffffu, in_run)) return -1;
    const bool hit = in_run && ((rec.x >> t.sub) & 1u);
    const uint32_t mask = __ballot_sync(0xffffffffu, hit);
    if (hit) {
        p.h_pending = true;
        const uint32_t idx = tail + (uint32_t)__popc(mask & ((1u << lane) - 1u));
        p.h_slot = idx & (kQ - 1);
        p.h_g = rec.y;
        p.h_pos = pos;                        // (n_contrib semantics)
        if (hit_out) hit_out[idx] = make_uint2(pos, rec.y);     // the backward walks this list instead
        p.h_xy = *reinterpret_cast<const float2 *>(geo.cull + t.gbase + rec.y);
        p.h_co = geo.conic_opacity[t.gbase + rec.y];
        p.h_rgb = geo.rgb[t.gbase + rec.y];
    }
    // advance: the live record of chunk c + 1
    p.rec = make_uint2(0u, 0u);
    if (i + 32u < t.n_live) p.rec = t.live[i + 32u];
    return __popc(mask);
}

}  // namespace

// ================================================================================== forward
constexpr int kFwdWarps = 4;
#ifndef PS_FWD_MIN_CTAS
#define PS_FWD_MIN_CTAS 6              // <= 80 registers: 24 resident warps per SM
#endif
constexpr float kStopT = 0.0001f;          // upstream: stop once T (1 - alpha) < 1e-4
constexpr float kStopGuard = 1.01e-4f;     // a run is folded without replay only if T T_k stays above this

struct FwdPixel {
    float T, Cr, Cg, Cb;
    float D;            // depth channel (DEPTH instantiations only)
    uint32_t last;      // 1 + list position of the last blended entry (0 = none)
    bool done;          // no further blending for this lane (stopped, or outside the image / masked)
    bool stopped;       // the early-exit test fired
};

// Four queued hits (an aligned group) onto the lane's pixel, front to back.  DEPTH: D accumulates r2.w with the
// colour's weights (an independent chain; the colour arithmetic is unchanged).
template <bool DEPTH>
__device__ __forceinline__ void fwd_blend4(const HitQueue &q, uint32_t base, const TaskGeom &t, float &T, float &Cr,
                                           float &Cg, float &Cb, float &D, uint32_t &last, bool &done, bool &stopped) {
    float pw[4], al[4], dv[4];
    float3 col[4];
    uint32_t ps[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float4 a0 = q.r0[base + k], a1 = q.r1[base + k], a2 = q.r2[base + k];
        pw[k] = hit_power2(a0, a1, t.fi, t.fj);
        al[k] = fminf(0.99f, a0.w * fast_exp2(pw[k]));
        col[k] = make_float3(a2.x, a2.y, a2.z);
        dv[k] = a2.w;
        ps[k] = __float_as_uint(a1.w);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const bool contrib = !done && !(pw[k] > kPowerEps) && !(al[k] < kAlphaMin);
        const float test_T = T * (1.0f - al[k]);
        const bool stop = contrib && (test_T < kStopT);
        const bool blend = contrib && !stop;
        const float w = blend ? al[k] * T : 0.0f;
        Cr = fmaf(col[k].x, w, Cr); Cg = fmaf(col[k].y, w, Cg); Cb = fmaf(col[k].z, w, Cb);
        if (DEPTH) D = fmaf(dv[k], w, D);
        T = blend ? test_T : T;
        last = blend ? ps[k] + 1u : last;
        done = done || stop;
        stopped = stopped || stop;
    }
}

// Front-to-back blend of the warp's run [t.run_begin, t.run_begin + t.run_len) onto the per-lane state px.
template <bool DEPTH>
__device__ __forceinline__ uint32_t fwd_run(const Geom &geo, const TaskGeom &t, HitQueue &q, FwdPixel &px, int lane,
                                            uint2 *__restrict__ hit_out = nullptr) {
    float T = px.T, Cr = px.Cr, Cg = px.Cg, Cb = px.Cb, D = px.D;
    uint32_t last = px.last;
    bool done = px.done, stopped = px.stopped;
    CullPipe p;
    cull_prologue(p, t, lane);
    uint32_t head = 0, tail = 0;
    for (uint32_t c = 0;; ++c) {                       // the first chunk past the run drains the last parked hits
        cull_park<false, DEPTH>(p, q, nullptr, t);
        uint32_t avail = tail;                         // parked so far
        const int nh = cull_step(p, geo, t, c, tail, lane, hit_out);
        if (nh >= 0) tail += (uint32_t)nh;
        else avail = queue_pad(q, tail, lane);
        // whole groups of four (their power / exp evaluations are independent, only the transmittance chains)
        while (avail - head >= 4u) {
            fwd_blend4<DEPTH>(q, head & (kQ - 1), t, T, Cr, Cg, Cb, D, last, done, stopped);
            head += 4u;
        }
        // (hits beyond this point are behind every pixel's last contributor)
        if (nh < 0 || __all_sync(0xffffffffu, done)) break;
        __syncwarp();
    }
    __syncwarp();
    px.T = T; px.Cr = Cr; px.Cg = Cg; px.Cb = Cb; px.D = D; px.last = last; px.done = done; px.stopped = stopped;
    return tail;
}

// DEPTH instantiations carry one more accumulator through the same loop (and the fold of the K > 1 runs); they are
// built for fewer resident CTAs (5, or 4 with runs) so that it does not spill.
// DET: loss.sums is the per-task partials array [S*V*tiles*8] of (sse, sse_clipped) (see the file header); the colour-
// only DET instantiations are built for the DEPTH ones' CTA counts so that they do not spill.
template <int K, bool DEPTH, bool DET>
__global__ void __launch_bounds__(kFwdWarps * 32, (DEPTH || DET) ? (K > 1 ? 4 : 5) : PS_FWD_MIN_CTAS)
k_composite_fwd2(Dims d, Geom geo, const float *__restrict__ bg_all, const uint2 *__restrict__ live,
                 ImageState img, float *__restrict__ out_color, LossEpilogue loss, HitLists hl) {
    __shared__ HitQueue s_q[kFwdWarps];
    __shared__ float4 s_ct[K > 1 ? kFwdWarps : 1][32];      // a run's (Cr, Cg, Cb, T)
    __shared__ float s_d[K > 1 && DEPTH ? kFwdWarps : 1][32];   // its depth
    __shared__ uint32_t s_last[K > 1 ? kFwdWarps : 1][32];   // its last contributor | stopped << 31
    __shared__ uint32_t s_live_begin[K > 1 ? kFwdWarps : 1];   // where each run starts on the live list
    constexpr int kTasksPerCta = kFwdWarps / K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int run = warp % K;
    HitQueue &q = s_q[warp];
    TaskGeom t;
    const long long task = (long long)blockIdx.x * kTasksPerCta + warp / K;
    const bool valid = task_setup(d, geo, live, task, lane, t);
    const bool truncated = *geo.n_instances > d.capacity;
    const uint32_t count = (valid && !truncated) ? t.count : 0u;
    t.count = count;
    t.run_len = count;
    if (K > 1) run_bounds(count, K, run, t.run_begin, t.run_len);
    if (count) live_run(t, geo, task, lane);

    FwdPixel px;
    px.T = 1.0f; px.Cr = px.Cg = px.Cb = 0.0f; px.D = 0.0f;
    px.last = 0; px.stopped = false;
    px.done = !valid || !t.inside;
    if (valid) {
        uint2 *hit_out = nullptr;
        if (hl.hits)   // this run's slice of the block's region (a run has at most run_len hits)
            hit_out = hl.hits + ((size_t)t.start * 8 + (size_t)(task & 7) * t.count + t.run_begin);
        const uint32_t nh = fwd_run<DEPTH>(geo, t, q, px, lane, hit_out);
        if (hl.run_hits && lane == 0) hl.run_hits[task * kMaxSegments + run] = nh;
    }

    if (K > 1) {
        if (lane == 0) s_live_begin[warp] = t.live_begin;
        s_ct[warp][lane] = make_float4(px.Cr, px.Cg, px.Cb, px.T);
        if (DEPTH) s_d[warp][lane] = px.D;
        s_last[warp][lane] = px.last | (px.stopped ? 0x80000000u : 0u);
        __syncthreads();
        if (run != 0 || !valid) return;
        // fold the runs in list order; px is run 0's result, i.e. the exact sequential state after run 0
        for (int j = 1; j < K; ++j) {
            if (t.inside) {  // state in front of run j: what the backward's run j starts from
                const size_t o = ((size_t)t.vid * (kMaxSegments - 1) + (j - 1)) * t.hw + t.pix;
                img.run_state[o] = make_float4(px.T, px.Cr, px.Cg, px.Cb);
                if (DEPTH) img.run_depth[o] = px.D;
            }
            const float4 r = s_ct[warp + j][lane];
            const uint32_t rl = s_last[warp + j][lane];
            const bool replay = !px.done && ((rl >> 31) != 0u || px.T * r.w < kStopGuard);
            if (__any_sync(0xffffffffu, replay)) {
                // the pixel saturates inside (or near) run j: replay it with the true transmittance
                TaskGeom tj = t;
                run_bounds(count, K, j, tj.run_begin, tj.run_len);
                tj.live_begin = s_live_begin[warp + j];
                FwdPixel pj = px;
                pj.done = px.done || !replay;
                fwd_run<DEPTH>(geo, tj, q, pj, lane);
                if (replay) px = pj;
            }
            if (!replay && !px.done) {
                px.Cr = fmaf(px.T, r.x, px.Cr); px.Cg = fmaf(px.T, r.y, px.Cg); px.Cb = fmaf(px.T, r.z, px.Cb);
                if (DEPTH) px.D = fmaf(px.T, s_d[warp + j][lane], px.D);
                px.T *= r.w;
                const uint32_t r_last = rl & 0x7fffffffu;
                px.last = r_last ? r_last : px.last;
            }
        }
    } else if (!valid) {
        return;
    }
    float sse = 0.0f, sse_clip = 0.0f;
    if (t.inside) {
        const size_t o1 = (size_t)t.vid * t.hw + t.pix;
        img.final_T[o1] = px.T;
        img.n_contrib[o1] = px.last;
        if (DEPTH) img.depth_image[o1] = px.D;     // background 0: nothing behind the last contributor
        const float *bg = bg_all + 3 * t.vid;
        const float r = px.Cr + px.T * bg[0], g = px.Cg + px.T * bg[1], b = px.Cb + px.T * bg[2];
        const size_t o3 = (size_t)t.vid * 3 * t.hw + t.pix;
        if (out_color) { out_color[o3] = r; out_color[o3 + t.hw] = g; out_color[o3 + 2 * t.hw] = b; }
        img.color[o3] = r; img.color[o3 + t.hw] = g; img.color[o3 + 2 * t.hw] = b;
        if (loss.target) {
            // loss epilogue (loss_mse.py:30-31, metrics.py:11-19): squared error of this pixel, raw and clipped
            const float tr = loss.target[o3], tg = loss.target[o3 + t.hw], tb = loss.target[o3 + 2 * t.hw];
            const float er = r - tr, eg = g - tg, eb = b - tb;
            sse = er * er + eg * eg + eb * eb;
            const float cr = __saturatef(r) - __saturatef(tr), cg = __saturatef(g) - __saturatef(tg),
                        cb = __saturatef(b) - __saturatef(tb);
            sse_clip = cr * cr + cg * cg + cb * cb;
        }
    }
    if (loss.target) {
        // one pair of atomics per warp task, spread over kLossSlots addresses per view
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            sse += __shfl_xor_sync(0xffffffffu, sse, o);
            sse_clip += __shfl_xor_sync(0xffffffffu, sse_clip, o);
        }
        if (lane == 0) {
            if constexpr (DET) {
                // this task's own pair; k_loss_finish sums them per view in a fixed order
                reinterpret_cast<float2 *>(loss.sums)[(long long)blockIdx.x * kTasksPerCta + warp / K] =
                    make_float2(sse, sse_clip);
            } else {
                const int slot = (int)((blockIdx.x * kTasksPerCta + warp / K) & (kLossSlots - 1));
                float *dst = loss.sums + ((size_t)t.vid * 2) * kLossSlots + slot;
                atomicAdd(dst, sse);
                atomicAdd(dst + kLossSlots, sse_clip);
            }
        }
    }
}

// Fixed-order finish of the DET loss epilogue: block = view, thread s sums the view's tasks s, s + 64, ... in order.
__global__ void __launch_bounds__(kLossSlots)
k_loss_finish(const float2 *__restrict__ partials, int tasks_per_view, float *__restrict__ sums) {
    const int vid = blockIdx.x, s = threadIdx.x;
    const float2 *p = partials + (size_t)vid * tasks_per_view;
    float raw = 0.0f, clipped = 0.0f;
    for (int i = s; i < tasks_per_view; i += kLossSlots) {
        const float2 v = p[i];
        raw += v.x;
        clipped += v.y;
    }
    sums[(size_t)vid * 2 * kLossSlots + s] = raw;
    sums[((size_t)vid * 2 + 1) * kLossSlots + s] = clipped;
}

// ================================================================================== backward
constexpr int kBwdWarps = 4;
constexpr int kBatch = 16;              // queued hits per batch (phase 2: lanes = entry x pixel half)
static_assert(kBatch == 32 || kBatch == 16, "phase 2 maps lanes to (entry, pixel half)");
constexpr int kHalves = 32 / kBatch;    // lanes per entry in phase 2
constexpr int kRowsPerLane = 4 / kHalves;   // pixel rows (of 8) each phase-2 lane sums

template <bool DEPTH>
struct BwdSmem {
    HitQueue q;
    float2 d0[kQ];                      // (dx0, dy0): the hit's centre relative to the block origin
    float su[kBatch][33];               // u = G dL/dalpha   [entry][pixel], +1 pad: conflict-free both ways
    float sw[kBatch][33];               // w = alpha T
    float4 dp[32];                      // dL/dC of the block's pixels (r, g, b, dL/dD)
    float dd[DEPTH ? kQ : 1];           // depth value d of each queued hit (r2.w holds the id)
};

struct BwdPixel {
    float dpr, dpg, dpb, dpd, Q, T, S;  // dpd = dL/dD (DEPTH instantiations only)
    uint32_t last;
};

// Phase 1 + phase 2 for the queue entries [head, head + cnt), head a multiple of kBatch, cnt <= kBatch
// (warp-uniform; entries up to the next multiple of four exist as zero-opacity padding).
// DET: vg points at the block records and rbase = tile_start * 8 + block * count (see the file header).
template <bool FULL, bool DEPTH, bool DET>
__device__ __forceinline__ void bwd_batch(BwdSmem<DEPTH> &sm, BwdPixel &px, const TaskGeom &t, const ViewGrads &vg,
                                          uint32_t head, int cnt, float kx, float ky, int lane, size_t rbase) {
    // ---- phase 1: lane = pixel, entries front to back
    const uint32_t base = head & (kQ - 1);
#pragma unroll
    for (int j = 0; j < kBatch; ++j) {
        if (!FULL && (j & 3) == 0 && j >= cnt) break;
        const float4 a0 = sm.q.r0[base + j], a1 = sm.q.r1[base + j], a2 = sm.q.r2[base + j];
        const float p2 = hit_power2(a0, a1, t.fi, t.fj);
        const float G = fast_exp2(p2);
        const float al = fminf(0.99f, a0.w * G);
        const bool active = __float_as_uint(a1.w) < px.last && !(p2 > kPowerEps) && !(al < kAlphaMin);
        const float a = active ? al : 0.0f;
        const float Gs = active ? G : 0.0f;        // also keeps an overflowed exp2 out of 0 * inf
        float cdp = fmaf(a2.z, px.dpb, fmaf(a2.y, px.dpg, a2.x * px.dpr));
        if (DEPTH) cdp = fmaf(sm.dd[base + j], px.dpd, cdp);     // c . dL/dC + d dL/dD
        const float w = a * px.T;
        px.S = fmaf(w, cdp, px.S);
        const float om = 1.0f - a;
        const float dL = fmaf(px.T, cdp, -(px.Q - px.S) * fast_rcp(om));
        px.T *= om;
        sm.su[j][lane] = Gs * dL;
        sm.sw[j][lane] = w;
    }
    __syncwarp();
    // ---- phase 2: lane = (entry e, pixel half h); raw moments over the lane's rows, i / j literals
    const int e = lane & (kBatch - 1), h = lane / kBatch;
    float m00 = 0.0f, m10 = 0.0f, m01 = 0.0f, m20 = 0.0f, m11 = 0.0f, m02 = 0.0f, s_r = 0.0f, s_g = 0.0f, s_b = 0.0f;
    float s_d = 0.0f;
#pragma unroll
    for (int jr = 0; jr < kRowsPerLane; ++jr) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int p = (h * kRowsPerLane + jr) * 8 + i;
            const float u = sm.su[e][p], w = sm.sw[e][p];
            const float4 dpp = sm.dp[p];
            m00 += u;
            if (i) { m10 = fmaf(u, (float)i, m10); m20 = fmaf(u, (float)(i * i), m20); }
            if (jr) { m01 = fmaf(u, (float)jr, m01); m02 = fmaf(u, (float)(jr * jr), m02); }
            if (i && jr) m11 = fmaf(u, (float)(i * jr), m11);
            s_r = fmaf(w, dpp.x, s_r); s_g = fmaf(w, dpp.y, s_g); s_b = fmaf(w, dpp.z, s_b);
            if (DEPTH) s_d = fmaf(w, dpp.w, s_d);
        }
    }
    // shift to the Gaussian's centre: dx = ca - i, dy = cb - jr, (ca, cb) = centre relative to this lane's first row
    const uint32_t slot = base + (uint32_t)e;
    const float2 c0 = sm.d0[slot];
    const float ca = c0.x, cb = c0.y - (float)(h * kRowsPerLane);
    float s_u = m00;
    float s_x = fmaf(ca, m00, -m10);
    float s_y = fmaf(cb, m00, -m01);
    float s_xx = fmaf(ca, fmaf(ca, m00, -2.0f * m10), m20);
    float s_xy = fmaf(ca, fmaf(cb, m00, -m01), fmaf(-cb, m10, m11));
    float s_yy = fmaf(cb, fmaf(cb, m00, -2.0f * m01), m02);
    if (kHalves == 2) {
        s_u += __shfl_xor_sync(0xffffffffu, s_u, 16); s_x += __shfl_xor_sync(0xffffffffu, s_x, 16);
        s_y += __shfl_xor_sync(0xffffffffu, s_y, 16); s_xx += __shfl_xor_sync(0xffffffffu, s_xx, 16);
        s_xy += __shfl_xor_sync(0xffffffffu, s_xy, 16); s_yy += __shfl_xor_sync(0xffffffffu, s_yy, 16);
        s_r += __shfl_xor_sync(0xffffffffu, s_r, 16); s_g += __shfl_xor_sync(0xffffffffu, s_g, 16);
        s_b += __shfl_xor_sync(0xffffffffu, s_b, 16);
        if (DEPTH) s_d += __shfl_xor_sync(0xffffffffu, s_d, 16);
    }
    const bool any = (s_u != 0.0f) | (s_x != 0.0f) | (s_y != 0.0f) | (s_xx != 0.0f) | (s_xy != 0.0f) |
                     (s_yy != 0.0f) | (s_r != 0.0f) | (s_g != 0.0f) | (s_b != 0.0f) | (DEPTH && s_d != 0.0f);
    if (h == 0 && e < cnt && any) {
        const float4 b0 = sm.q.r0[slot], b1 = sm.q.r1[slot], b2 = sm.q.r2[slot];
        const float o = b0.w;
        const size_t rec = t.gbase + __float_as_uint(b2.w);
        // u excludes the opacity factor: position / conic terms pick it up here, dL/dopacity does not
        const float ox = o * s_x, oy = o * s_y;
        if constexpr (DET) {
            // the record of (this block, the hit's list position): its only writer, so a plain store
            const size_t r = rbase + __float_as_uint(b1.w);
            vg.d_mean2d[r] = make_float2(kx * (2.0f * b1.x * ox + b1.y * oy), ky * (2.0f * b1.z * oy + b1.y * ox));
            vg.d_conic[r] = make_float4(-0.5f * o * s_xx, -0.5f * o * s_xy, -0.5f * o * s_yy, s_u);
            vg.d_color[r] = make_float4(s_r, s_g, s_b, DEPTH ? s_d : 0.0f);
        } else {
            red_add_v2(vg.d_mean2d + rec, kx * (2.0f * b1.x * ox + b1.y * oy), ky * (2.0f * b1.z * oy + b1.y * ox));
            red_add_v4(vg.d_conic + rec, -0.5f * o * s_xx, -0.5f * o * s_xy, -0.5f * o * s_yy, s_u);
            red_add_v4(vg.d_color + rec, s_r, s_g, s_b, DEPTH ? s_d : 0.0f);
        }
    }
    __syncwarp();
}

// DEPTH: dL/dD = d_depth rides along (see bwd_batch); built for 5 resident CTAs so that it does not spill.
// DET: vg points at the block records (see the file header).
template <int K, bool DEPTH, bool DET>
__global__ void __launch_bounds__(kBwdWarps * 32, DEPTH ? 5 : 6)
k_composite_bwd2(Dims d, Geom geo, const float *__restrict__ bg_all, const uint2 *__restrict__ live,
                 ImageState img, const float *__restrict__ d_color, const float *__restrict__ d_depth, ViewGrads vg,
                 LossEpilogue loss, HitLists hl) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    constexpr int kTasksPerCta = kBwdWarps / K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int run = warp % K;
    BwdSmem<DEPTH> &sm = reinterpret_cast<BwdSmem<DEPTH> *>(s_raw)[warp];
    if (*geo.n_instances > d.capacity) return;
    TaskGeom t;
    const long long task = (long long)blockIdx.x * kTasksPerCta + warp / K;
    if (!task_setup(d, geo, live, task, lane, t)) return;

    BwdPixel px;
    px.T = 1.0f; px.S = 0.0f;
    px.last = 0; px.dpr = px.dpg = px.dpb = px.dpd = 0.0f; px.Q = 0.0f;
    if (t.inside) {
        const size_t o1 = (size_t)t.vid * t.hw + t.pix, o3 = (size_t)t.vid * 3 * t.hw + t.pix;
        px.last = img.n_contrib[o1];
        const float c_r = img.color[o3], c_g = img.color[o3 + t.hw], c_b = img.color[o3 + 2 * t.hw];
        if (d_color) {
            px.dpr = d_color[o3]; px.dpg = d_color[o3 + t.hw]; px.dpb = d_color[o3 + 2 * t.hw];
        } else {
            // fused loss: dL/dC = scale[view] * (C - target), never materialised as a tensor
            const float sc = loss.grad_scale[t.vid];
            px.dpr = sc * (c_r - loss.target[o3]); px.dpg = sc * (c_g - loss.target[o3 + t.hw]);
            px.dpb = sc * (c_b - loss.target[o3 + 2 * t.hw]);
        }
        px.Q = c_r * px.dpr + c_g * px.dpg + c_b * px.dpb;
        if (DEPTH) {   // Q = C . dL/dC + D dL/dD (the background adds nothing to the depth channel)
            px.dpd = d_depth[o1];
            px.Q = fmaf(img.depth_image[o1], px.dpd, px.Q);
        }
    }
    sm.dp[lane] = make_float4(px.dpr, px.dpg, px.dpb, px.dpd);
    // nothing beyond the block's last contributor; the run split is the forward's (on the full count)
    const uint32_t nmax = min(t.count, __reduce_max_sync(0xffffffffu, px.last));
    if (K > 1) {
        run_bounds(t.count, K, run, t.run_begin, t.run_len);
        if (run > 0 && t.inside && t.run_begin < nmax) {
            // (T, C) in front of this run, stored by the forward: S = sum_{j < run} w_j (c_j . dL/dC) = C . dL/dC
            const float4 st = img.run_state[((size_t)t.vid * (kMaxSegments - 1) + (run - 1)) * t.hw + t.pix];
            px.T = st.x;
            px.S = st.y * px.dpr + st.z * px.dpg + st.w * px.dpb;
            if (DEPTH)
                px.S = fmaf(img.run_depth[((size_t)t.vid * (kMaxSegments - 1) + (run - 1)) * t.hw + t.pix], px.dpd, px.S);
        }
    }
    const uint32_t run_end = min(t.run_begin + t.run_len, nmax);
    const uint32_t n = run_end > t.run_begin ? run_end - t.run_begin : 0u;
    t.run_len = n;
    const float kx = kLn2 * 0.5f * (float)d.W, ky = kLn2 * 0.5f * (float)d.H;
    (void)bg_all;
    // DET: this block's records of the tile's list (the hit lists' index space)
    const size_t rbase = DET ? (size_t)t.start * 8 + (size_t)(task & 7) * t.count : 0;

    uint32_t head = 0, tail = 0;
    if (hl.hits) {
        // ---- the forward left this run's hit list: no cull, every lane parks a hit
        const uint2 *__restrict__ hits = hl.hits + ((size_t)t.start * 8 + (size_t)(task & 7) * t.count + t.run_begin);
        const uint32_t nh = n ? hl.run_hits[task * kMaxSegments + run] : 0u;
        uint2 hnext = make_uint2(0u, 0u);
        if ((uint32_t)lane < nh) hnext = hits[lane];
        for (uint32_t h0 = 0; h0 < nh; h0 += 32u) {
            const uint2 hcur = hnext;
            const bool live = h0 + (uint32_t)lane < nh && hcur.x < nmax;     // nothing behind the last contributor
            if (h0 + 32u + (uint32_t)lane < nh) hnext = hits[h0 + 32u + lane];
            float4 cr = make_float4(0.0f, 0.0f, 0.0f, 0.0f), co = cr, rgb = cr;
            if (live) {
                cr = geo.cull[t.gbase + hcur.y];
                co = geo.conic_opacity[t.gbase + hcur.y];
                rgb = geo.rgb[t.gbase + hcur.y];
            }
            const uint32_t m = __ballot_sync(0xffffffffu, live);
            if (live) {
                const uint32_t slot = (tail + (uint32_t)__popc(m & ((1u << lane) - 1u))) & (kQ - 1);
                const float qa = -0.5f * kLog2e * co.x, qb = -kLog2e * co.y, qc = -0.5f * kLog2e * co.z;
                const float dx0 = cr.x - t.rx0, dy0 = cr.y - t.ry0;
                const float ax = qa * dx0, cy = qc * dy0;
                sm.q.r0[slot] = make_float4(fmaf(ax, dx0, fmaf(cy, dy0, qb * dx0 * dy0)), -(2.0f * ax + qb * dy0),
                                            -(2.0f * cy + qb * dx0), co.w);
                sm.q.r1[slot] = make_float4(qa, qb, qc, __uint_as_float(hcur.x));
                sm.q.r2[slot] = make_float4(rgb.x, rgb.y, rgb.z, __uint_as_float(hcur.y));
                sm.d0[slot] = make_float2(dx0, dy0);
                if (DEPTH) sm.dd[slot] = rgb.w;
            }
            tail += (uint32_t)__popc(m);
            __syncwarp();
            while (tail - head >= (uint32_t)kBatch) {
                bwd_batch<true, DEPTH, DET>(sm, px, t, vg, head, kBatch, kx, ky, lane, rbase);
                head += kBatch;
            }
            if (m != 0xffffffffu) break;                                      // the list is ordered by position
        }
    } else {
        // ---- walk the run's live entries in front of nmax
        live_run(t, geo, task, lane);
        CullPipe p;
        cull_prologue(p, t, lane);
        for (uint32_t c = 0;; ++c) {
            cull_park<true, DEPTH>(p, sm.q, sm.d0, t, sm.dd);
            const uint32_t avail = tail;
            const int nh = cull_step(p, geo, t, c, tail, lane);
            if (nh >= 0) tail += (uint32_t)nh;
            while (avail - head >= (uint32_t)kBatch) {
                bwd_batch<true, DEPTH, DET>(sm, px, t, vg, head, kBatch, kx, ky, lane, rbase);
                head += kBatch;
            }
            if (nh < 0) break;
        }
    }
    if (tail != head) {
        queue_pad(sm.q, tail, lane, DEPTH ? sm.dd : nullptr);
        bwd_batch<false, DEPTH, DET>(sm, px, t, vg, head, (int)(tail - head), kx, ky, lane, rbase);
    }
}

// ================================================================================== launchers
// Tunables (A/B measurements, tests): initialised from the environment once, changeable through ps_set_option.
static int g_impl = 0;        // 1 = legacy CTA-per-tile compositor, 2 = warp tasks
static int g_segments = -1;   // 0 = automatic, else 1 | 2 | 4 list runs per task
static int g_hit_lists = -1;  // 0 = never keep, 1 = always keep, 2 = automatic

int composite_impl() {
    if (g_impl == 0) {
        const char *e = getenv("PIXELSPLAT_B200_COMPOSITE");
        g_impl = (e && e[0] == '1') ? 1 : 2;
    }
    return g_impl;
}

int get_composite_option(int which) {
    if (which == 0) return composite_impl();
    composite_segments(0);           // reads the environment once
    composite_hit_lists(0);
    return which == 1 ? g_segments : g_hit_lists;
}

int set_composite_option(int which, int value) {
    if (which == 0 && (value == 1 || value == 2)) { g_impl = value; return PS_OK; }
    if (which == 1 && (value == 0 || value == 1 || value == 2 || value == 4)) { g_segments = value; return PS_OK; }
    if (which == 2 && (value == 0 || value == 1 || value == 2)) { g_hit_lists = value; return PS_OK; }
    return PS_ERR_INVALID_ARGUMENT;
}

template <int K, bool DEPTH, bool DET>
static int launch_fwd(const Dims &d, const Inputs &in, const Geom &g, const uint2 *live,
                      const ImageState &img, float *out_color, const LossEpilogue &loss, const HitLists &hl,
                      cudaStream_t st) {
    const long long tasks = (long long)d.S * d.V * d.tiles * 8;
    constexpr int per_cta = kFwdWarps / K;
    k_composite_fwd2<K, DEPTH, DET><<<(unsigned)((tasks + per_cta - 1) / per_cta), kFwdWarps * 32, 0, st>>>(d, g, in.bg, live, img, out_color, loss, hl);
    PS_LAUNCH_CHECK("k_composite_fwd2");
    return PS_OK;
}

template <int K, bool DET>
static int launch_fwd(const Dims &d, const Inputs &in, const Geom &g, const uint2 *live,
                      const ImageState &img, float *out_color, const LossEpilogue &loss, const HitLists &hl,
                      cudaStream_t st) {
    return d.depth_mode ? launch_fwd<K, true, DET>(d, in, g, live, img, out_color, loss, hl, st)
                        : launch_fwd<K, false, DET>(d, in, g, live, img, out_color, loss, hl, st);
}

template <bool DET>
static int launch_fwd(const Dims &d, const Inputs &in, const Geom &g, const uint2 *live,
                      const ImageState &img, float *out_color, const LossEpilogue &loss, const HitLists &hl,
                      cudaStream_t st) {
    switch (d.segK) {
        case 4: return launch_fwd<4, DET>(d, in, g, live, img, out_color, loss, hl, st);
        case 2: return launch_fwd<2, DET>(d, in, g, live, img, out_color, loss, hl, st);
        default: return launch_fwd<1, DET>(d, in, g, live, img, out_color, loss, hl, st);
    }
}

int launch_composite_forward(const Dims &d, const Inputs &in, const Geom &g, const unsigned long long *keys,
                             const uint2 *live, const ImageState &img, float *out_color, const LossEpilogue &loss, const HitLists &hl,
                             float *loss_partials, cudaStream_t st) {
    if (composite_impl() == 1) {
        if (loss.target || !out_color) { set_error("the legacy compositor has no loss epilogue"); return PS_ERR_UNSUPPORTED; }
        return launch_composite_forward_v1(d, in, g, keys, img, out_color, st);
    }
    if (!loss.target || !loss_partials) return launch_fwd<false>(d, in, g, live, img, out_color, loss, hl, st);
    // fixed-order loss epilogue: per-task partials, then k_loss_finish writes every slot of loss.sums
    LossEpilogue le = loss;
    le.sums = loss_partials;
    int rc = launch_fwd<true>(d, in, g, live, img, out_color, le, hl, st);
    if (rc) return rc;
    k_loss_finish<<<(unsigned)(d.S * d.V), kLossSlots, 0, st>>>(reinterpret_cast<const float2 *>(loss_partials),
                                                                d.tiles * 8, loss.sums);
    PS_LAUNCH_CHECK("k_loss_finish");
    return PS_OK;
}

template <int K, bool DEPTH, bool DET>
static int launch_bwd(const Dims &d, const Inputs &in, const Geom &g, const uint2 *live,
                      const ImageState &img, const float *d_color, const float *d_depth, const ViewGrads &vg,
                      const LossEpilogue &loss, const HitLists &hl, cudaStream_t st) {
    const long long tasks = (long long)d.S * d.V * d.tiles * 8;
    constexpr int per_cta = kBwdWarps / K;
    const size_t smem = sizeof(BwdSmem<DEPTH>) * kBwdWarps;
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_composite_bwd2<K, DEPTH, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    k_composite_bwd2<K, DEPTH, DET><<<(unsigned)((tasks + per_cta - 1) / per_cta), kBwdWarps * 32, smem, st>>>(
        d, g, in.bg, live, img, d_color, d_depth, vg, loss, hl);
    PS_LAUNCH_CHECK("k_composite_bwd2");
    return PS_OK;
}

template <int K, bool DET>
static int launch_bwd(const Dims &d, const Inputs &in, const Geom &g, const uint2 *live,
                      const ImageState &img, const float *d_color, const float *d_depth, const ViewGrads &vg,
                      const LossEpilogue &loss, const HitLists &hl, cudaStream_t st) {
    return d_depth ? launch_bwd<K, true, DET>(d, in, g, live, img, d_color, d_depth, vg, loss, hl, st)
                   : launch_bwd<K, false, DET>(d, in, g, live, img, d_color, nullptr, vg, loss, hl, st);
}

template <bool DET>
static int launch_bwd(const Dims &d, const Inputs &in, const Geom &g, const uint2 *live,
                      const ImageState &img, const float *d_color, const float *d_depth, const ViewGrads &vg,
                      const LossEpilogue &loss, const HitLists &hl, cudaStream_t st) {
    switch (d.segK) {
        case 4: return launch_bwd<4, DET>(d, in, g, live, img, d_color, d_depth, vg, loss, hl, st);
        case 2: return launch_bwd<2, DET>(d, in, g, live, img, d_color, d_depth, vg, loss, hl, st);
        default: return launch_bwd<1, DET>(d, in, g, live, img, d_color, d_depth, vg, loss, hl, st);
    }
}

// Fixed-order gather of the DET backward's block records: 8 lanes per on-screen (view, Gaussian) pair, lane b = block b.
// For each tile of the pair's rectangle, row-major, the pair's position in the tile's sorted segment is found by a
// binary search for the exact key the scatter wrote (float_bits(depth) << 32 | Gaussian; every tile of the rectangle
// holds exactly one instance of the pair), and lane b adds block b's record of that position.  The 8 lanes' sums are
// then added in block order 0..7 and STORED into the per-(view, Gaussian) scratch (every listed pair's row, the rows
// the preprocess backward reads).  Every sum has a fixed order: tiles row-major within a block, blocks 0..7.
constexpr int kGatherThreads = 128;

__global__ void __launch_bounds__(kGatherThreads)
k_gather_block_records(Dims d, Geom geo, const unsigned long long *__restrict__ keys, ViewGrads rec, ViewGrads vg) {
    if (*geo.n_instances > d.capacity) return;
    const long long i = ((long long)blockIdx.x * kGatherThreads + threadIdx.x) >> 3;
    const int lane = threadIdx.x & 31, b = lane & 7;
    if (((long long)blockIdx.x * kGatherThreads + (threadIdx.x & ~31)) >> 3 >= geo.n_instances[2]) return;   // warp
    const bool live = i < geo.n_instances[2];
    uint32_t vgi = 0;
    float2 m = make_float2(0.0f, 0.0f);
    float4 c = make_float4(0.0f, 0.0f, 0.0f, 0.0f), col = c;
    if (live) {
        vgi = geo.vis_pairs[i];
        const uint32_t vid = vgi / (uint32_t)d.P, gid = vgi - vid * (uint32_t)d.P;
        const ushort4 r = geo.rect[vgi];
        const unsigned long long key = ((unsigned long long)__float_as_uint(geo.depth[vgi]) << 32) | gid;
        const uint32_t *__restrict__ t_start = geo.tile_start + (size_t)vid * d.tiles;
        const uint32_t *__restrict__ t_count = geo.tile_count + (size_t)vid * d.tiles;
        for (uint32_t ty = r.y; ty < r.w; ++ty)
            for (uint32_t tx = r.x; tx < r.z; ++tx) {
                const uint32_t tile = ty * (uint32_t)d.gx + tx;
                const uint32_t start = t_start[tile], count = t_count[tile];
                const unsigned long long *__restrict__ seg = keys + start;
                uint32_t lo = 0, hi = count;       // lower bound of key in the tile's sorted segment
                while (lo < hi) {
                    const uint32_t mid = (lo + hi) >> 1;
                    if (seg[mid] < key) lo = mid + 1; else hi = mid;
                }
                if (lo == count || seg[lo] != key) continue;     // (not reached: the scatter wrote it)
                const size_t q = (size_t)start * 8 + (size_t)b * count + lo;
                const float2 a = rec.d_mean2d[q];
                const float4 e = rec.d_conic[q], f = rec.d_color[q];
                m.x += a.x; m.y += a.y;
                c.x += e.x; c.y += e.y; c.z += e.z; c.w += e.w;
                col.x += f.x; col.y += f.y; col.z += f.z; col.w += f.w;
            }
    }
    // blocks 0..7, in order, into lane 0 of the group
    const int g0 = lane & ~7;
    float2 sm = make_float2(0.0f, 0.0f);
    float4 sc = make_float4(0.0f, 0.0f, 0.0f, 0.0f), scol = sc;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int src = g0 + k;
        sm.x += __shfl_sync(0xffffffffu, m.x, src); sm.y += __shfl_sync(0xffffffffu, m.y, src);
        sc.x += __shfl_sync(0xffffffffu, c.x, src); sc.y += __shfl_sync(0xffffffffu, c.y, src);
        sc.z += __shfl_sync(0xffffffffu, c.z, src); sc.w += __shfl_sync(0xffffffffu, c.w, src);
        scol.x += __shfl_sync(0xffffffffu, col.x, src); scol.y += __shfl_sync(0xffffffffu, col.y, src);
        scol.z += __shfl_sync(0xffffffffu, col.z, src); scol.w += __shfl_sync(0xffffffffu, col.w, src);
    }
    if (live && b == 0) {
        vg.d_mean2d[vgi] = sm;
        vg.d_conic[vgi] = sc;
        vg.d_color[vgi] = scol;
    }
}

int launch_composite_backward(const Dims &d, const Inputs &in, const Geom &g, const unsigned long long *keys,
                              const uint2 *live, const ImageState &img, const float *d_color, const float *d_depth, const ViewGrads &vg,
                              const ViewGrads *records, const LossEpilogue &loss, const HitLists &hl,
                              cudaStream_t st) {
    if (composite_impl() == 1) {
        if (!d_color) { set_error("the legacy compositor has no loss epilogue"); return PS_ERR_UNSUPPORTED; }
        return launch_composite_backward_v1(d, in, g, keys, img, d_color, vg, st);
    }
    if (!records) return launch_bwd<false>(d, in, g, live, img, d_color, d_depth, vg, loss, hl, st);
    int rc = launch_bwd<true>(d, in, g, live, img, d_color, d_depth, *records, loss, hl, st);
    if (rc) return rc;
    // the pair count lives on the device: launch for the worst case, surplus threads exit at once
    const long long lanes = (long long)d.S * d.V * d.P * 8;
    k_gather_block_records<<<(unsigned)((lanes + kGatherThreads - 1) / kGatherThreads), kGatherThreads, 0, st>>>(
        d, g, keys, *records, vg);
    PS_LAUNCH_CHECK("k_gather_block_records");
    return PS_OK;
}

// Runs per task for a batch of `tasks` warp tasks: enough warps to fill the machine (132 SMs x ~24 resident
// warps), none when the batch already does.  PIXELSPLAT_B200_SEGMENTS = 1 | 2 | 4 overrides (A/B runs).
int composite_segments(long long tasks) {
    if (g_segments < 0) {
        const char *e = getenv("PIXELSPLAT_B200_SEGMENTS");
        g_segments = (e && (e[0] == '1' || e[0] == '2' || e[0] == '4') && e[1] == 0) ? e[0] - '0' : 0;
    }
    if (composite_impl() == 1) return 1;
    if (g_segments) return g_segments;
    return tasks <= 2048 ? 4 : tasks <= 4096 ? 2 : 1;
}

// The forward's hit lists cost 64 bytes of binning state per unit of instance capacity: kept while that is at most
// 512 MB (every configuration of BASELINE.json at batch 1-2), dropped beyond (the backward then culls for itself).
// PIXELSPLAT_B200_HIT_LISTS = 0 | 1 forces it (A/B runs); the legacy compositor never uses them.
bool composite_hit_lists(long long capacity) {
    if (g_hit_lists < 0) {
        const char *e = getenv("PIXELSPLAT_B200_HIT_LISTS");
        g_hit_lists = (e && (e[0] == '0' || e[0] == '1') && e[1] == 0) ? (e[0] - '0') : 2;
    }
    if (composite_impl() == 1) return false;
    if (g_hit_lists != 2) return g_hit_lists == 1;
    return capacity * 64 <= (512ll << 20);
}

}  // namespace ps
