// The optimiser end of a training step (the reference's gradient_clip_val 0.5, optim.Adam and LinearLR warm-up,
// src/model/model_wrapper.py configure_optimizers): gradient clipping by the global L2 norm and the Adam update of
// every parameter tensor, in two launches whatever the number of tensors.
//
// The tensors are rows of a device-resident segment table (parameter, gradient, exp_avg, exp_avg_sq, count).  Each
// segment is cut into chunks of kOptChunk elements on a grid aligned to the gradient pointer's 16-byte boundary, so
// a chunk's interior is whole float4 units; one CTA owns one chunk and finds its segment by binary search on the
// rows' first_chunk.
//
//   k_clip_adam_norm    each CTA: the sum of squares of its chunk, reduced in a fixed tree, to partial[chunk].  The
//                       CTA that finishes last then forms, in a fixed order, every tensor's norm from its partials,
//                       the norm of those norms (what torch's clip_grad_norm_ forms), and the step's scalars from
//                       the device step counter: clip coefficient, warmed-up lr over the first bias correction, the
//                       root of the second bias correction.
//   k_clip_adam_update  each CTA: Adam on its chunk with g' = coef * g; gradients are only read.  CTA 0 increments
//                       the step counter (nothing in this launch reads it).
//
// Only the question "which CTA is last" goes through an atomic; every sum has a fixed order, so a step gives the same
// bits on every run.  Nothing is read back by the host: the call can be captured in a CUDA graph.
#include "adam.cuh"
#include "ps_common.cuh"

namespace ps {

constexpr int kOptThreads = 256;
constexpr int kOptChunk = PS_CLIP_ADAM_CHUNK;
constexpr int kOptUnits = kOptChunk / 4 / kOptThreads;   // float4 units per thread per chunk
static_assert(kOptChunk == kOptThreads * 4 * kOptUnits, "a chunk is a whole number of float4 units per thread");

struct OptHeader {          // workspace[0..63]; zero before the first call, the ticket returns to zero in every call
    unsigned int ticket;
    float coef;             // min(1, max_norm / (norm + 1e-6)), NaN when the norm is
    float step_size;        // lr_t / (1 - beta1^t)
    float bc2_sqrt;         // sqrt(1 - beta2^t)
};
constexpr size_t kOptHeaderBytes = 64;

__host__ __device__ __forceinline__ long long grad_skew(const void *grad) {
    return (long long)(((uintptr_t)grad >> 2) & 3);   // elements past the 16-byte boundary below the pointer
}

__host__ __device__ __forceinline__ long long segment_chunks(const void *grad, long long count) {
    return (grad_skew(grad) + count + kOptChunk - 1) / kOptChunk;
}

__device__ __forceinline__ int find_segment(const ps_clip_adam_segment *__restrict__ segs, int n, long long chunk) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(&segs[mid].first_chunk) <= chunk) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// Sum over the CTA in a fixed tree; the result is valid in thread 0.
__device__ __forceinline__ double block_sum(double x, double *red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = x;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int w = 0; w < kOptThreads / 32; ++w) s += red[w];
    }
    __syncthreads();
    return s;
}

// The step's scalars, by one thread.  `t` steps have been taken: this is step t + 1.
__device__ void step_scalars(const ps_clip_adam_desc &d, long long t, float norm, OptHeader *hdr) {
    const float c = (float)d.max_norm / (norm + 1e-6f);
    hdr->coef = c > 1.0f ? 1.0f : c;                  // not fminf: a NaN norm gives a NaN coefficient, as torch's clamp
    double factor = 1.0;
    if (d.warm_up_steps > 0) {                        // LinearLR(1 / W, 1, total_iters = W) after t scheduler steps
        const double W = (double)d.warm_up_steps, start = 1.0 / W;
        factor = start + (1.0 - start) * (double)(t < d.warm_up_steps ? t : d.warm_up_steps) / W;
    }
    const double n = (double)(t + 1);
    hdr->step_size = (float)(d.lr * factor / (1.0 - pow(d.beta1, n)));
    hdr->bc2_sqrt = (float)sqrt(1.0 - pow(d.beta2, n));
}

__global__ void __launch_bounds__(kOptThreads)
k_clip_adam_norm(ps_clip_adam_desc d, const ps_clip_adam_segment *__restrict__ segs, ps_clip_adam_state st,
                 OptHeader *hdr, double *__restrict__ partial) {
    __shared__ double red[kOptThreads / 32];
    __shared__ bool last;
    const long long chunk = blockIdx.x;
    const ps_clip_adam_segment S = segs[find_segment(segs, d.n_segments, chunk)];
    const long long c = chunk - S.first_chunk, s = grad_skew(S.grad);
    const float *gv = S.grad - s;                     // 16-byte aligned; elements [s, s + count) are the tensor's
    const long long lo = c == 0 ? s : c * kOptChunk, hi = min(s + S.count, (c + 1) * kOptChunk);
    float acc = 0.0f;
#pragma unroll
    for (int k = 0; k < kOptUnits; ++k) {
        const long long j = c * kOptChunk + 4LL * (threadIdx.x + k * kOptThreads);
        if (j >= lo && j + 4 <= hi) {
            const float4 g = __ldg(reinterpret_cast<const float4 *>(gv + j));
            acc = fmaf(g.x, g.x, acc);
            acc = fmaf(g.y, g.y, acc);
            acc = fmaf(g.z, g.z, acc);
            acc = fmaf(g.w, g.w, acc);
        } else {
            for (long long e = max(j, lo); e < min(j + 4, hi); ++e) {
                const float g = __ldg(gv + e);
                acc = fmaf(g, g, acc);
            }
        }
    }
    const double sum = block_sum((double)acc, red);
    if (threadIdx.x == 0) {
        partial[chunk] = sum;
        __threadfence();
        last = atomicAdd(&hdr->ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();

    // Every partial is written.  A tensor's norm is the float32 root of its sum; the total is the root of the sum of
    // the squared norms.  Tensors of up to 4 chunks: one thread each; longer ones: one warp each, lanes striding the
    // chunks.  Which thread adds what, and in which order, depends only on the table.
    double acc2 = 0.0;
    for (int i = threadIdx.x; i < d.n_segments; i += kOptThreads) {
        const long long first = __ldg(&segs[i].first_chunk);
        const long long n = segment_chunks(segs[i].grad, __ldg(&segs[i].count));
        if (n > 4) continue;
        double q = 0.0;
        for (long long k = 0; k < n; ++k) q += __ldcg(partial + first + k);
        const float nrm = sqrtf((float)q);
        acc2 += (double)nrm * (double)nrm;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = warp; i < d.n_segments; i += kOptThreads / 32) {
        const long long first = __ldg(&segs[i].first_chunk);
        const long long n = segment_chunks(segs[i].grad, __ldg(&segs[i].count));
        if (n <= 4) continue;
        double q = 0.0;
        for (long long k = lane; k < n; k += 32) q += __ldcg(partial + first + k);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
        const float nrm = sqrtf((float)q);
        if (lane == 0) acc2 += (double)nrm * (double)nrm;
    }
    const double total = block_sum(acc2, red);
    if (threadIdx.x == 0) {
        const float norm = sqrtf((float)total);
        *st.grad_norm = norm;
        step_scalars(d, *st.step, norm, hdr);
        hdr->ticket = 0;
    }
}

// Adam (adam.cuh) on the clipped gradient coef * g, with the step's scalars.
__device__ __forceinline__ void adam(float &p, float g, float &m, float &v, const AdamConsts &k, const OptHeader &h) {
    adam(p, g * h.coef, m, v, k, h.step_size, h.bc2_sqrt);
}

__global__ void __launch_bounds__(kOptThreads)
k_clip_adam_update(ps_clip_adam_desc d, const ps_clip_adam_segment *__restrict__ segs, ps_clip_adam_state st,
                   const OptHeader *__restrict__ hdr) {
    const long long chunk = blockIdx.x;
    const ps_clip_adam_segment S = segs[find_segment(segs, d.n_segments, chunk)];
    const OptHeader h = *hdr;
    const AdamConsts k = {(float)(1.0 - d.beta1), (float)d.beta2, (float)(1.0 - d.beta2), (float)d.eps};
    const long long c = chunk - S.first_chunk, s = grad_skew(S.grad);
    const long long lo = c == 0 ? s : c * kOptChunk, hi = min(s + S.count, (c + 1) * kOptChunk);
    const float *gv = S.grad - s;
    float *pv = S.param - s, *mv = S.exp_avg - s, *vv = S.exp_avg_sq - s;
    // float4 units need all four tensors at the same offset from a 16-byte boundary (the moments always follow the
    // gradient; a parameter does when its storage happens to)
    const bool vec = ((((uintptr_t)S.param ^ (uintptr_t)S.grad) | ((uintptr_t)S.exp_avg ^ (uintptr_t)S.grad) |
                       ((uintptr_t)S.exp_avg_sq ^ (uintptr_t)S.grad)) & 15) == 0;
    if (vec) {
        float4 g[kOptUnits], p[kOptUnits], m[kOptUnits], v[kOptUnits];
        bool full[kOptUnits];
#pragma unroll
        for (int u = 0; u < kOptUnits; ++u) {
            const long long j = c * kOptChunk + 4LL * (threadIdx.x + u * kOptThreads);
            full[u] = j >= lo && j + 4 <= hi;
            if (full[u]) {
                g[u] = __ldg(reinterpret_cast<const float4 *>(gv + j));
                p[u] = *reinterpret_cast<const float4 *>(pv + j);
                m[u] = *reinterpret_cast<const float4 *>(mv + j);
                v[u] = *reinterpret_cast<const float4 *>(vv + j);
            }
        }
#pragma unroll
        for (int u = 0; u < kOptUnits; ++u) {
            const long long j = c * kOptChunk + 4LL * (threadIdx.x + u * kOptThreads);
            if (full[u]) {
                adam(p[u].x, g[u].x, m[u].x, v[u].x, k, h);
                adam(p[u].y, g[u].y, m[u].y, v[u].y, k, h);
                adam(p[u].z, g[u].z, m[u].z, v[u].z, k, h);
                adam(p[u].w, g[u].w, m[u].w, v[u].w, k, h);
                *reinterpret_cast<float4 *>(pv + j) = p[u];
                *reinterpret_cast<float4 *>(mv + j) = m[u];
                *reinterpret_cast<float4 *>(vv + j) = v[u];
            } else {
                for (long long e = max(j, lo); e < min(j + 4, hi); ++e) adam(pv[e], __ldg(gv + e), mv[e], vv[e], k, h);
            }
        }
    } else {                                          // coalesced scalar accesses, eight in flight per thread
        constexpr int kBatch = 8;
        for (long long j0 = lo + threadIdx.x; j0 < hi; j0 += (long long)kBatch * kOptThreads) {
            float g[kBatch], p[kBatch], m[kBatch], v[kBatch];
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {
                const long long e = j0 + (long long)u * kOptThreads;
                if (e < hi) {
                    g[u] = __ldg(gv + e);
                    p[u] = pv[e];
                    m[u] = mv[e];
                    v[u] = vv[e];
                }
            }
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {
                const long long e = j0 + (long long)u * kOptThreads;
                if (e < hi) {
                    adam(p[u], g[u], m[u], v[u], k, h);
                    pv[e] = p[u];
                    mv[e] = m[u];
                    vv[e] = v[u];
                }
            }
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *st.step += 1;
}

static size_t clip_adam_workspace(long long n_chunks) {
    return (kOptHeaderBytes + (size_t)n_chunks * sizeof(double) + 255) / 256 * 256;
}

static int check_clip_adam_desc(const char *who, const ps_clip_adam_desc *d) {
    if (!d) {
        set_error("%s: desc is NULL", who);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->n_segments < 1 || d->n_chunks < d->n_segments || d->n_chunks > 0x7fffffffLL) {
        set_error("%s: %d segments in %lld chunks: need at least one segment, at least one chunk per segment and at "
                  "most 2^31 - 1 chunks", who, d->n_segments, (long long)d->n_chunks);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (!(d->lr >= 0.0) || !(d->beta1 >= 0.0 && d->beta1 < 1.0) || !(d->beta2 >= 0.0 && d->beta2 < 1.0) ||
        !(d->eps >= 0.0) || !(d->max_norm > 0.0) || d->warm_up_steps < 0) {
        set_error("%s: bad scalars (lr %g, betas %g %g, eps %g, max_norm %g, warm_up_steps %lld)", who, d->lr,
                  d->beta1, d->beta2, d->eps, d->max_norm, (long long)d->warm_up_steps);
        return PS_ERR_INVALID_ARGUMENT;
    }
    return PS_OK;
}

}  // namespace ps

extern "C" PS_API int64_t ps_clip_adam_segment_chunks(const void *grad, int64_t count) {
    return count < 1 ? 0 : (int64_t)ps::segment_chunks(grad, count);
}

extern "C" PS_API int ps_clip_adam_workspace_bytes(const ps_clip_adam_desc *desc, size_t *out) {
    const int rc = ps::check_clip_adam_desc("ps_clip_adam_workspace_bytes", desc);
    if (rc != PS_OK) return rc;
    if (!out) {
        ps::set_error("ps_clip_adam_workspace_bytes: out is NULL");
        return PS_ERR_INVALID_ARGUMENT;
    }
    *out = ps::clip_adam_workspace(desc->n_chunks);
    return PS_OK;
}

extern "C" PS_API int ps_clip_adam_step(const ps_clip_adam_desc *desc, const ps_clip_adam_segment *segments,
                                        const ps_clip_adam_state *state, void *workspace, size_t workspace_bytes,
                                        void *stream) {
    const int rc = ps::check_clip_adam_desc("ps_clip_adam_step", desc);
    if (rc != PS_OK) return rc;
    if (!segments || !state || !state->step || !state->grad_norm) {
        ps::set_error("ps_clip_adam_step: segments, state, state->step and state->grad_norm must be given");
        return PS_ERR_INVALID_ARGUMENT;
    }
    const size_t need = ps::clip_adam_workspace(desc->n_chunks);
    if (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 15)) {
        ps::set_error("ps_clip_adam_step: workspace of %zu bytes, %zu needed, 16-byte aligned",
                      workspace ? workspace_bytes : 0, need);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    ps::OptHeader *hdr = static_cast<ps::OptHeader *>(workspace);
    double *partial = reinterpret_cast<double *>(static_cast<char *>(workspace) + ps::kOptHeaderBytes);
    const unsigned grid = (unsigned)desc->n_chunks;
    ps::k_clip_adam_norm<<<grid, ps::kOptThreads, 0, st>>>(*desc, segments, *state, hdr, partial);
    PS_LAUNCH_CHECK("k_clip_adam_norm");
    ps::k_clip_adam_update<<<grid, ps::kOptThreads, 0, st>>>(*desc, segments, *state, hdr);
    PS_LAUNCH_CHECK("k_clip_adam_update");
    return PS_OK;
}
