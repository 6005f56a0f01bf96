// LPIPS distance head (the lpips package's LPIPS(net="vgg"), version 0.1, on the VGG16 trunk's relu1_2 .. relu5_3),
// forward and backward over up to five layers in one launch.  Per layer l, image n and pixel p, with the features
// x0, x1 [N, C, H, W] and the 1x1 lin weight w [C]:
//   f^ = f / (sqrt(sum_c f_c^2) + eps), eps = 1e-10;   u = f^0 - f^1;
//   d_l[n] = (1 / (H W)) sum_p sum_c w_c m u_c^2;       out[n] = sum_l d_l[n].
// u is formed directly from the normalised features.  Expanding sum_c w (a/n0 - b/n1)^2 into moment sums would
// cancel catastrophically when the prediction is close to the target; the direct form gives exactly 0 (and a zero
// gradient) for identical inputs.
//
// Work items are (layer, image, tile of TP consecutive pixels), layer-major.  A CTA stages the tile's channel
// columns of both sides in shared memory with cp.async (every feature element is read from HBM once), takes each
// pixel's two norms, then its weighted sum over channels.  TP is the largest power of two <= min(256, 8192 / C), so
// a tile is at most 2 x 8192 floats (64 KB, three CTAs per SM) and each channel row of a tile is TP * 4 contiguous
// bytes.  Thread t of 256 owns pixel t % TP and channels t / TP, + 256 / TP, ...: the sums over channels are in a
// fixed order, the per-pixel and per-tile sums too, and the forward's per-tile partials are added by a finish kernel
// in a fixed order.  No float atomics: the same bits on every run.
//
// Backward (same tiling, no workspace): with z_c = 2 k_c u_c, k = w m d_out[n] / (H W) and, per side, n its norm
// and T = sum_c z_c f_c (a second per-pixel reduction over the staged column),
//   d x0_j = z_j / (n0 + eps) - x0_j T0 / (n0 (n0 + eps)^2),
//   d x1_j = -(z_j / (n1 + eps) - x1_j T1 / (n1 (n1 + eps)^2)).
// At an all-zero column (n = 0) the second term is taken as its limit 0, giving z_j / (n + eps) = z_j / eps; torch's
// autograd of the formula gives NaN there (sqrt's derivative at 0).
//
// Dropout (train mode, the package's Dropout(p = 0.5) in front of each lin layer): m = 2 * keep, keep the top bit of
// a splitmix64 hash of (seed, layer, flat element index) as the header states.  The seed is read on the device.
#include <cuda_pipeline.h>

#include <algorithm>

#include "ps_common.cuh"

namespace ps {

constexpr int kLpThreads = 256;
constexpr int kLpTileFloats = 8192;                   // per side: 2 x 32 KB of shared memory per CTA at most
constexpr float kLpEps = 1e-10f;
constexpr unsigned long long kGolden = 0x9E3779B97F4A7C15ull;

struct LpLayer {
    const float *x0, *x1, *w;
    float *d0, *d1;                                   // backward outputs (either may be null)
    int C, HW, tp_shift, tiles;                       // TP = 1 << tp_shift pixels per tile
    int item_begin;                                   // first work item (and partial) of the layer
};

struct LpParams {
    LpLayer L[PS_LPIPS_MAX_LAYERS];
    int n_layers, N;
    const long long *seed;                            // null: eval
};

__device__ __forceinline__ unsigned long long splitmix_mix(unsigned long long z) {
    z ^= z >> 30;
    z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27;
    z *= 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// The dropout factor of flat element i of a layer whose key is `key`: 2 (kept) or 0.
__device__ __forceinline__ float drop_factor(unsigned long long key, unsigned long long i) {
    return (splitmix_mix(key + (i + 1ull) * kGolden) >> 63) ? 2.0f : 0.0f;
}

// Which layer work item `item` belongs to (the layers' items are consecutive, layer-major).
__device__ __forceinline__ int layer_of(const LpParams &P, int item) {
    int l = 0;
#pragma unroll
    for (int k = 1; k < PS_LPIPS_MAX_LAYERS; ++k)
        if (k < P.n_layers && item >= P.L[k].item_begin) l = k;
    return l;
}

// Copies the tile's columns of both sides into s0 / s1 [C][TP] (zeros past the last pixel) and waits for them.
__device__ __forceinline__ void stage_tile(const LpLayer &L, int n, int p0, float *s0, float *s1) {
    const int TP = 1 << L.tp_shift, count = L.C * TP;
    const size_t base = (size_t)n * L.C * L.HW;
    for (int i = threadIdx.x; i < count; i += kLpThreads) {
        const int c = i >> L.tp_shift, pix = p0 + (i & (TP - 1));
        const bool in = pix < L.HW;
        const size_t off = in ? base + (size_t)c * L.HW + pix : 0;
        __pipeline_memcpy_async(s0 + i, L.x0 + off, sizeof(float), in ? 0 : sizeof(float));
        __pipeline_memcpy_async(s1 + i, L.x1 + off, sizeof(float), in ? 0 : sizeof(float));
    }
    __pipeline_commit();
    __pipeline_wait_prior(0);
    __syncthreads();
}

// Sum over the channel groups of red[g * TP + p] for this thread's pixel p, in group order.
__device__ __forceinline__ float group_sum(const float *red, int TP, int G, int p) {
    float s = 0.0f;
    for (int g = 0; g < G; ++g) s += red[g * TP + p];
    return s;
}

// Per-pixel norms of both sides, n = sqrt(sum_c f_c^2), reduced over the channel groups in a fixed order.
__device__ __forceinline__ void column_norms(const LpLayer &L, const float *s0, const float *s1, float *red0,
                                             float *red1, float &n0, float &n1) {
    const int TP = 1 << L.tp_shift, G = kLpThreads >> L.tp_shift;
    const int p = threadIdx.x & (TP - 1), g = threadIdx.x >> L.tp_shift;
    float q0 = 0.0f, q1 = 0.0f;
    for (int c = g; c < L.C; c += G) {
        const float a = s0[c * TP + p], b = s1[c * TP + p];
        q0 = fmaf(a, a, q0);
        q1 = fmaf(b, b, q1);
    }
    red0[threadIdx.x] = q0;
    red1[threadIdx.x] = q1;
    __syncthreads();
    n0 = sqrtf(group_sum(red0, TP, G, p));
    n1 = sqrtf(group_sum(red1, TP, G, p));
    __syncthreads();                                   // red0 / red1 are reused by the caller
}

// grid: one CTA per work item; partial[item] = sum over the tile's pixels of sum_c w m u^2.
__global__ void __launch_bounds__(kLpThreads) k_lpips_fwd(const __grid_constant__ LpParams P,
                                                         float *__restrict__ partial) {
    extern __shared__ float smem[];
    __shared__ float red0[kLpThreads], red1[kLpThreads], warp_sum[kLpThreads / 32];
    const int item = blockIdx.x, l = layer_of(P, item);
    const LpLayer &L = P.L[l];
    const int local = item - L.item_begin, n = local / L.tiles, tile = local % L.tiles;
    const int TP = 1 << L.tp_shift, G = kLpThreads >> L.tp_shift;
    const int p = threadIdx.x & (TP - 1), g = threadIdx.x >> L.tp_shift, p0 = tile * TP;
    float *s0 = smem, *s1 = smem + L.C * TP;
    stage_tile(L, n, p0, s0, s1);
    float n0, n1;
    column_norms(L, s0, s1, red0, red1, n0, n1);
    const float d0 = n0 + kLpEps, d1 = n1 + kLpEps;
    const bool drop = P.seed != nullptr;
    const unsigned long long key =
        drop ? splitmix_mix((unsigned long long)*P.seed + (unsigned long long)(l + 1) * kGolden) : 0ull;
    const unsigned long long row0 = (unsigned long long)n * L.C;
    float acc = 0.0f;
    for (int c = g; c < L.C; c += G) {
        const float u = s0[c * TP + p] / d0 - s1[c * TP + p] / d1;
        float k = __ldg(L.w + c);
        if (drop) k *= drop_factor(key, (row0 + c) * (unsigned long long)L.HW + (unsigned long long)(p0 + p));
        acc = fmaf(k * u, u, acc);
    }
    red0[threadIdx.x] = acc;
    __syncthreads();
    float v = 0.0f;
    if (threadIdx.x < TP && p0 + threadIdx.x < L.HW) v = group_sum(red0, TP, G, threadIdx.x);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.0f;
#pragma unroll
        for (int w = 0; w < kLpThreads / 32; ++w) s += warp_sum[w];
        partial[item] = s;
    }
}

// One warp per image: each layer's tile partials in a fixed order, over the layer's pixel count, summed over layers
// in layer order.
__global__ void k_lpips_finish(const __grid_constant__ LpParams P, const float *__restrict__ partial,
                               float *__restrict__ out) {
    const int n = blockIdx.x;
    float total = 0.0f;
    for (int l = 0; l < P.n_layers; ++l) {
        const LpLayer &L = P.L[l];
        const float *q = partial + L.item_begin + (size_t)n * L.tiles;
        float s = 0.0f;
        for (int t = threadIdx.x; t < L.tiles; t += 32) s += q[t];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        total += s / (float)L.HW;
    }
    if (threadIdx.x == 0) out[n] = total;
}

__global__ void __launch_bounds__(kLpThreads) k_lpips_bwd(const __grid_constant__ LpParams P,
                                                         const float *__restrict__ d_out) {
    extern __shared__ float smem[];
    __shared__ float red0[kLpThreads], red1[kLpThreads];
    const int item = blockIdx.x, l = layer_of(P, item);
    const LpLayer &L = P.L[l];
    const int local = item - L.item_begin, n = local / L.tiles, tile = local % L.tiles;
    const int TP = 1 << L.tp_shift, G = kLpThreads >> L.tp_shift;
    const int p = threadIdx.x & (TP - 1), g = threadIdx.x >> L.tp_shift, p0 = tile * TP;
    float *s0 = smem, *s1 = smem + L.C * TP;
    stage_tile(L, n, p0, s0, s1);
    float n0, n1;
    column_norms(L, s0, s1, red0, red1, n0, n1);
    const float d0 = n0 + kLpEps, d1 = n1 + kLpEps;
    const bool drop = P.seed != nullptr;
    const unsigned long long key =
        drop ? splitmix_mix((unsigned long long)*P.seed + (unsigned long long)(l + 1) * kGolden) : 0ull;
    const unsigned long long row0 = (unsigned long long)n * L.C;
    const float scale = 2.0f * (__ldg(d_out + n) / (float)L.HW);      // z = scale * w m u
    auto z_of = [&](int c, float a, float b) {
        const float u = a / d0 - b / d1;
        float k = __ldg(L.w + c);
        if (drop) k *= drop_factor(key, (row0 + c) * (unsigned long long)L.HW + (unsigned long long)(p0 + p));
        return scale * k * u;
    };
    float t0 = 0.0f, t1 = 0.0f;
    for (int c = g; c < L.C; c += G) {
        const float a = s0[c * TP + p], b = s1[c * TP + p], z = z_of(c, a, b);
        t0 = fmaf(z, a, t0);
        t1 = fmaf(z, b, t1);
    }
    red0[threadIdx.x] = t0;
    red1[threadIdx.x] = t1;
    __syncthreads();
    const float T0 = group_sum(red0, TP, G, p), T1 = group_sum(red1, TP, G, p);
    // second term's coefficient; 0 at an all-zero column (its limit), where f = 0 as well
    const float e0 = n0 > 0.0f ? T0 / (n0 * d0 * d0) : 0.0f;
    const float e1 = n1 > 0.0f ? T1 / (n1 * d1 * d1) : 0.0f;
    const int pix = p0 + p;
    if (pix >= L.HW) return;
    const size_t base = (size_t)n * L.C * L.HW + pix;
    for (int c = g; c < L.C; c += G) {
        const float a = s0[c * TP + p], b = s1[c * TP + p], z = z_of(c, a, b);
        const size_t o = base + (size_t)c * L.HW;
        if (L.d0) L.d0[o] = z / d0 - a * e0;
        if (L.d1) L.d1[o] = -(z / d1 - b * e1);
    }
}

// Validates the descriptor and fills the kernels' parameters, the work-item count and the dynamic shared memory.
static int lpips_setup(const char *who, const ps_lpips_desc *desc, LpParams *P, int *items, size_t *smem,
                       size_t *workspace) {
    if (!desc) {
        set_error("%s: desc is NULL", who);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (desc->n_layers < 1 || desc->n_layers > PS_LPIPS_MAX_LAYERS || desc->N < 1) {
        set_error("%s: bad shape (n_layers %d, N %d): need 1 <= n_layers <= %d and N >= 1", who, desc->n_layers,
                  desc->N, PS_LPIPS_MAX_LAYERS);
        return PS_ERR_INVALID_ARGUMENT;
    }
    *P = LpParams{};
    P->n_layers = desc->n_layers;
    P->N = desc->N;
    P->seed = reinterpret_cast<const long long *>(desc->dropout_seed);
    long long total = 0;
    *smem = 0;
    for (int l = 0; l < desc->n_layers; ++l) {
        const ps_lpips_layer &in = desc->layers[l];
        if (in.C < 1 || in.C > kLpTileFloats || in.H < 1 || in.W < 1 ||
            (long long)desc->N * in.C * in.H * in.W > 0x7fffffffLL) {
            set_error("%s: bad shape of layer %d (N %d, C %d, H %d, W %d): need 1 <= C <= %d, H, W >= 1 and at "
                      "most 2^31 - 1 elements", who, l, desc->N, in.C, in.H, in.W, kLpTileFloats);
            return PS_ERR_INVALID_ARGUMENT;
        }
        LpLayer &L = P->L[l];
        L.x0 = in.x0;
        L.x1 = in.x1;
        L.w = in.weight;
        L.C = in.C;
        L.HW = in.H * in.W;
        int shift = 0;
        while (shift < 8 && (in.C << (shift + 1)) <= kLpTileFloats) ++shift;
        L.tp_shift = shift;
        L.tiles = (L.HW + (1 << shift) - 1) >> shift;
        L.item_begin = (int)total;
        total += (long long)desc->N * L.tiles;
        if (total > 0x7fffffffLL) {
            set_error("%s: too many tiles for one launch", who);
            return PS_ERR_INVALID_ARGUMENT;
        }
        *smem = std::max(*smem, 2 * sizeof(float) * ((size_t)in.C << shift));
    }
    *items = (int)total;
    *workspace = ((size_t)total * sizeof(float) + 255) / 256 * 256;
    return PS_OK;
}

static int check_layer_pointers(const char *who, const ps_lpips_desc *desc) {
    for (int l = 0; l < desc->n_layers; ++l) {
        const ps_lpips_layer &in = desc->layers[l];
        if (!in.x0 || !in.x1 || !in.weight) {
            set_error("%s: NULL pointer in layer %d", who, l);
            return PS_ERR_INVALID_ARGUMENT;
        }
    }
    return PS_OK;
}

static int set_smem_attributes() {
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices)) {
        const int bytes = (int)(2 * sizeof(float) * kLpTileFloats);
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_lpips_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_lpips_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    }
    return PS_OK;
}

}  // namespace ps

extern "C" PS_API int ps_lpips_workspace_bytes(const ps_lpips_desc *desc, size_t *out) {
    ps::LpParams P;
    int items;
    size_t smem, ws;
    const int rc = ps::lpips_setup("ps_lpips_workspace_bytes", desc, &P, &items, &smem, &ws);
    if (rc != PS_OK) return rc;
    if (!out) { ps::set_error("ps_lpips_workspace_bytes: out is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    *out = ws;
    return PS_OK;
}

extern "C" PS_API int ps_lpips_forward(const ps_lpips_desc *desc, float *out, void *workspace,
                                       size_t workspace_bytes, void *stream) {
    ps::LpParams P;
    int items;
    size_t smem, ws;
    int rc = ps::lpips_setup("ps_lpips_forward", desc, &P, &items, &smem, &ws);
    if (rc != PS_OK) return rc;
    if ((rc = ps::check_layer_pointers("ps_lpips_forward", desc)) != PS_OK) return rc;
    if (!out || !workspace) {
        ps::set_error("ps_lpips_forward: NULL pointer");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (workspace_bytes < ws) {
        ps::set_error("ps_lpips_forward: workspace of %zu bytes, %zu needed", workspace_bytes, ws);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if ((rc = ps::set_smem_attributes()) != PS_OK) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    float *partial = static_cast<float *>(workspace);
    ps::k_lpips_fwd<<<items, ps::kLpThreads, smem, st>>>(P, partial);
    PS_LAUNCH_CHECK("k_lpips_fwd");
    ps::k_lpips_finish<<<P.N, 32, 0, st>>>(P, partial, out);
    PS_LAUNCH_CHECK("k_lpips_finish");
    return PS_OK;
}

extern "C" PS_API int ps_lpips_backward(const ps_lpips_desc *desc, const float *d_out, const ps_lpips_grads *grads,
                                        void *stream) {
    ps::LpParams P;
    int items;
    size_t smem, ws;
    int rc = ps::lpips_setup("ps_lpips_backward", desc, &P, &items, &smem, &ws);
    if (rc != PS_OK) return rc;
    if ((rc = ps::check_layer_pointers("ps_lpips_backward", desc)) != PS_OK) return rc;
    if (!d_out || !grads) {
        ps::set_error("ps_lpips_backward: NULL pointer");
        return PS_ERR_INVALID_ARGUMENT;
    }
    for (int l = 0; l < desc->n_layers; ++l) {
        if (!grads->d_x0[l] && !grads->d_x1[l]) {
            ps::set_error("ps_lpips_backward: NULL pointer: layer %d has neither d_x0 nor d_x1", l);
            return PS_ERR_INVALID_ARGUMENT;
        }
        P.L[l].d0 = grads->d_x0[l];
        P.L[l].d1 = grads->d_x1[l];
    }
    if ((rc = ps::set_smem_attributes()) != PS_OK) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    ps::k_lpips_bwd<<<items, ps::kLpThreads, smem, st>>>(P, d_out);
    PS_LAUNCH_CHECK("k_lpips_bwd");
    return PS_OK;
}
