// Binning: (view, tile) instance counts -> exclusive scan -> scatter of
// (float_bits(depth) << 32 | gaussian) keys into per-tile segments -> per-tile LSD radix sort -> per-tile live
// list (the entries whose cull box meets the tile, with their 8x4 block masks; see kLivePosLimit).
//
// The sorted order inside a tile (ascending depth bits, ties by ascending Gaussian index) is
// exactly what upstream obtains from its global stable radix sort of (tile << 32 | depth) keys
// over Gaussian-ordered emission (SURVEY.md A.2), so keys / tile ranges are bit-identical to
// the reference's binning buffers while the sort itself never leaves shared memory.
#include <cub/device/device_segmented_radix_sort.cuh>

#include "ps_common.cuh"

namespace ps {

// ---------------------------------------------------------------- scan of tile counts
constexpr int kScanThreads = 1024;

__global__ void __launch_bounds__(kScanThreads)
k_tile_scan(int n, const uint32_t *__restrict__ count, uint32_t *__restrict__ start,
            uint32_t *__restrict__ cursor, long long *__restrict__ n_instances) {
    __shared__ uint32_t warp_sums[32];
    __shared__ unsigned long long carry_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry_s = 0;
    __syncthreads();
    uint32_t cmax = 0;
    for (int base = 0; base < n; base += kScanThreads) {
        const int i = base + tid;
        const uint32_t c = i < n ? count[i] : 0u;
        cmax = max(cmax, c);
        uint32_t x = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_sums[warp] = x;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = warp_sums[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += y;
            }
            warp_sums[lane] = w;  // inclusive
        }
        __syncthreads();
        const unsigned long long carry = carry_s;
        const uint32_t warp_off = warp ? warp_sums[warp - 1] : 0u;
        const unsigned long long excl = carry + warp_off + (x - c);
        if (i < n) {
            // offsets beyond 2^32-1 cannot be represented; clamp (capacity check rejects the call)
            const uint32_t e = excl > 0xffffffffull ? 0xffffffffu : (uint32_t)excl;
            start[i] = e;
            cursor[i] = e;
        }
        __syncthreads();
        if (tid == kScanThreads - 1) carry_s = carry + warp_sums[31];
        __syncthreads();
    }
    if (tid == 0) *n_instances = (long long)carry_s;
    // longest (view, tile) segment -> n_instances[1]; lets the host pick the sort configuration
    cmax = __reduce_max_sync(0xffffffffu, cmax);
    if (lane == 0 && cmax) atomicMax(reinterpret_cast<unsigned long long *>(n_instances + 1), (unsigned long long)cmax);
}

// ---------------------------------------------------------------- scatter
constexpr int kScatterThreads = 256;
constexpr int kScatterMaxSmemTiles = 8192;

// One CTA = 256 consecutive Gaussians of one view.  Slots are reserved per (CTA, tile) with a
// single global atomic; ranks inside the CTA come from shared-memory atomics.  (Consecutive
// Gaussians are neighbouring context pixels and land on a handful of tiles, so per-instance
// global atomics serialise on ~tiles addresses: 68 us -> a few us at configs[1].)
__global__ void __launch_bounds__(kScatterThreads)
k_scatter(Dims d, Geom geo, unsigned long long *__restrict__ keys, int use_smem) {
    extern __shared__ uint32_t s_scatter[];          // cnt[tiles], base[tiles]
    if (*geo.n_instances > d.capacity) return;       // truncated call: caller re-runs with more room
    const int vid = blockIdx.y;
    const int g = blockIdx.x * kScatterThreads + threadIdx.x;
    uint32_t *cnt = s_scatter, *base = s_scatter + d.tiles;
    uint32_t *cur = geo.tile_cursor + (size_t)vid * d.tiles;
    const size_t vg = (size_t)vid * d.P + g;
    const bool vis = g < d.P && geo.radii[vg] > 0;
    ushort4 r = make_ushort4(0, 0, 0, 0);
    unsigned long long key = 0;
    if (vis) {
        r = geo.rect[vg];
        key = ((unsigned long long)__float_as_uint(geo.depth[vg]) << 32) | (uint32_t)g;
    }
    if (!use_smem) {
        for (int ty = r.y; ty < r.w; ++ty)
            for (int tx = r.x; tx < r.z; ++tx) keys[atomicAdd(&cur[ty * d.gx + tx], 1u)] = key;
        return;
    }
    for (int i = threadIdx.x; i < d.tiles; i += kScatterThreads) cnt[i] = 0;
    __syncthreads();
    for (int ty = r.y; ty < r.w; ++ty)
        for (int tx = r.x; tx < r.z; ++tx) atomicAdd(&cnt[ty * d.gx + tx], 1u);
    __syncthreads();
    for (int i = threadIdx.x; i < d.tiles; i += kScatterThreads) {
        const uint32_t c = cnt[i];
        if (c) { base[i] = atomicAdd(&cur[i], c); cnt[i] = 0; }
    }
    __syncthreads();
    for (int ty = r.y; ty < r.w; ++ty)
        for (int tx = r.x; tx < r.z; ++tx) {
            const int t = ty * d.gx + tx;
            keys[base[t] + atomicAdd(&cnt[t], 1u)] = key;
        }
}

// Bitonic network over s_keys[0, n_pad) (n_pad a power of two), executed by the whole CTA; only
// used as the fallback for segments with long runs of identical depth.  Each warp owns a
// contiguous chunk: compare-exchange steps whose stride stays inside the chunk need only
// __syncwarp; the CTA barrier is paid for the few long-stride steps.
template <int THREADS>
__device__ void bitonic_sort_smem(unsigned long long *s_keys, int n_pad) {
    constexpr int kWarps = THREADS / 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int chunk = max(n_pad / kWarps, 2);
    const int warps_used = n_pad / chunk;
    const int half = n_pad >> 1;
    for (int k = 2; k <= n_pad; k <<= 1) {
        int j = k >> 1;
        const bool had_global = j >= chunk;
        for (; j >= chunk; j >>= 1) {
            for (int t = threadIdx.x; t < half; t += THREADS) {
                const int i = 2 * t - (t & (j - 1));      // bit j of i is clear
                const int p = i + j;
                const unsigned long long a = s_keys[i], b = s_keys[p];
                const bool up = (i & k) == 0;
                if ((a > b) == up) { s_keys[i] = b; s_keys[p] = a; }
            }
            __syncthreads();
        }
        if (warp < warps_used) {
            const int base = warp * chunk;
            for (; j > 0; j >>= 1) {
                for (int t = lane; t < (chunk >> 1); t += 32) {
                    const int i = base + 2 * t - (t & (j - 1));
                    const int p = i + j;
                    const unsigned long long a = s_keys[i], b = s_keys[p];
                    const bool up = (i & k) == 0;
                    if ((a > b) == up) { s_keys[i] = b; s_keys[p] = a; }
                }
                __syncwarp();
            }
        }
        if (had_global || 2 * k > chunk) __syncthreads();
    }
}

// ---------------------------------------------------------------- per-tile radix sort
// One CTA of 512 threads per (view, tile) segment of `depth_bits << 32 | gaussian` keys.
//   * n <= cap: the segment lives in shared memory and is sorted on (depth - min depth of the tile)
//     with stable 8-bit LSD passes -- as many as the depth range of the tile needs (3-4) -- then the
//     Gaussian-index tie-break of the full 64-bit order is restored: runs of identical depth (exact
//     float collisions, rare) are insertion-sorted by their first thread; a segment with a run
//     longer than 64 falls back to a bitonic network on the full key.
//   * n > cap: the same passes over the full key (index bits, then depth bits), ping-ponging
//     through HBM.  Always correct, just slower.
// 16 warps each own a contiguous ~n/16-key slice, so a pass is two short warp loops (count with
// fire-and-forget shared atomics, stable rank with match.any) around one column scan: the sort is
// bound by shared-memory latency chains, and short slices are what keeps those chains short.
constexpr int kSortThreads = 512;   // 64 regs x 512 threads: two CTAs per SM
constexpr int kSortWarps = kSortThreads / 32;

constexpr int kLiveItems = 4;      // entries per thread per round of the live-list compaction
static_assert(kLiveItems * kSortWarps == 64, "write_live_list scans the (item, warp) counts two per lane");

struct SortSmem {
    uint32_t cnt[kSortWarps * 256];
    uint32_t misc[64];
    uint32_t live[kLiveItems * kSortWarps];   // per-(item, warp) live counts of a compaction round
};

// passes [0, num_passes): digit p = ((key >> key_shift) - sub) >> (8 p) & 255 (key_shift = 32 and
// sub = tile min depth for the depth-only mode; key_shift = 0 / 32, sub = 0 for raw key bytes).
// Returns the buffer holding the result.
__device__ unsigned long long *radix8_passes(unsigned long long *a, unsigned long long *b, int n, SortSmem &sm,
                                             int key_shift, uint32_t sub, int num_passes) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int lo = (int)(((long long)n * warp) / kSortWarps);
    const int hi = (int)(((long long)n * (warp + 1)) / kSortWarps);
    uint32_t *cnt = sm.cnt, *misc = sm.misc;
    for (int p = 0; p < num_passes; ++p) {
        const int shift = 8 * p;
        auto digit = [&](unsigned long long k) -> uint32_t {
            return ((((uint32_t)(k >> key_shift)) - sub) >> shift) & 255u;
        };
        for (int i = tid; i < kSortWarps * 256; i += kSortThreads) cnt[i] = 0;
        if (tid == 0) misc[0] = 0;
        __syncthreads();
        for (int i = lo + lane; i < hi; i += 32) atomicAdd(&cnt[warp * 256 + digit(a[i])], 1u);
        __syncthreads();
        uint32_t total = 0, incl = 0;
        if (tid < 256) {   // thread t owns digit t: column prefix over the 32 warp rows
            uint32_t c[kSortWarps];
#pragma unroll
            for (int w = 0; w < kSortWarps; ++w) c[w] = cnt[w * 256 + tid];
#pragma unroll
            for (int w = 0; w < kSortWarps; ++w) { const uint32_t t = c[w]; c[w] = total; total += t; }
            if (total == (uint32_t)n) misc[0] = 1;          // uniform digit: nothing to move
            incl = total;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += y;
            }
            if (lane == 31) misc[8 + warp] = incl;
#pragma unroll
            for (int w = 0; w < kSortWarps; ++w) cnt[w * 256 + tid] = c[w];
        }
        __syncthreads();
        if (misc[0]) { __syncthreads(); continue; }
        if (tid < 256) {
            uint32_t off = incl - total;
            for (int w = 0; w < warp; ++w) off += misc[8 + w];
#pragma unroll
            for (int w = 0; w < kSortWarps; ++w) cnt[w * 256 + tid] += off;
        }
        __syncthreads();
        for (int base = lo; base < hi; base += 32) {       // stable scatter of this warp's slice
            const int i = base + lane;
            const bool valid = i < hi;
            const unsigned long long key = valid ? a[i] : 0ull;
            const uint32_t dg = valid ? digit(key) : (256u + (uint32_t)lane);
            const uint32_t peers = __match_any_sync(0xffffffffu, dg);
            const int leader = __ffs(peers) - 1;
            const int rank = __popc(peers & ((1u << lane) - 1u));
            uint32_t off = 0;
            if (valid && lane == leader) {
                off = cnt[warp * 256 + dg];
                cnt[warp * 256 + dg] = off + (uint32_t)__popc(peers);
            }
            off = __shfl_sync(0xffffffffu, off, leader);
            if (valid) b[off + rank] = key;
            __syncwarp();
        }
        __syncthreads();
        unsigned long long *t = a; a = b; b = t;
    }
    return a;
}

static size_t sort_smem_bytes(int cap) { return sizeof(SortSmem) + sizeof(unsigned long long) * 2 * (size_t)cap; }

// The live list of segment `seg` (see kLivePosLimit) from its sorted keys `sorted[0, n)` (shared or global memory),
// written by the whole CTA: rounds of kSortThreads * kLiveItems entries, each thread gathering the cull records of
// kLiveItems entries at once (one L2 latency per round), then a stable CTA-wide compaction in list order.
__device__ void write_live_list(const Dims &d, const Geom &geo, const unsigned long long *sorted, int n, int seg,
                                uint2 *__restrict__ live, SortSmem &sm) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int vid = seg / d.tiles, tile = seg - vid * d.tiles;
    const int x0 = (tile % d.gx) * kTile, y0 = (tile / d.gx) * kTile;
    const float4 *__restrict__ cull = geo.cull + (size_t)vid * d.P;
    const bool keep_all = (uint32_t)n > kLivePosLimit;
    uint32_t carry = 0;
    for (int base = 0; base < n; base += kSortThreads * kLiveItems) {
        uint32_t g[kLiveItems];
        float4 cr[kLiveItems];
#pragma unroll
        for (int k = 0; k < kLiveItems; ++k) {
            const int i = base + k * kSortThreads + tid;
            g[k] = i < n ? (uint32_t)sorted[i] : 0u;
            cr[k] = i < n ? cull[g[k]] : make_float4(0.0f, 0.0f, -3.0e38f, -3.0e38f);
        }
        uint32_t mask[kLiveItems], ballot[kLiveItems];
#pragma unroll
        for (int k = 0; k < kLiveItems; ++k) {
            const int i = base + k * kSortThreads + tid;
            mask[k] = i < n ? tile_block_mask(cr[k], x0, y0) : 0u;
            ballot[k] = __ballot_sync(0xffffffffu, i < n && (mask[k] != 0u || keep_all));
            if (lane == 0) sm.live[k * kSortWarps + warp] = (uint32_t)__popc(ballot[k]);
        }
        __syncthreads();
        // exclusive prefix of the 64 (item, warp) counts in list order, two per lane, by every warp at once
        const uint32_t c0 = sm.live[lane], c1 = sm.live[32 + lane];
        uint32_t e0 = c0, e1 = c1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y0 = __shfl_up_sync(0xffffffffu, e0, o), y1 = __shfl_up_sync(0xffffffffu, e1, o);
            if (lane >= o) { e0 += y0; e1 += y1; }
        }
        const uint32_t half = __shfl_sync(0xffffffffu, e0, 31);
        const uint32_t total = half + __shfl_sync(0xffffffffu, e1, 31);
        e0 -= c0;
        e1 += half - c1;
        uint32_t off[kLiveItems];      // (item k, this warp) sits at index k * 16 + warp
        off[0] = carry + __shfl_sync(0xffffffffu, e0, warp);
        off[1] = carry + __shfl_sync(0xffffffffu, e0, 16 + warp);
        off[2] = carry + __shfl_sync(0xffffffffu, e1, warp);
        off[3] = carry + __shfl_sync(0xffffffffu, e1, 16 + warp);
        carry += total;
#pragma unroll
        for (int k = 0; k < kLiveItems; ++k) {
            const int i = base + k * kSortThreads + tid;
            if ((ballot[k] >> lane) & 1u)
                live[off[k] + (uint32_t)__popc(ballot[k] & ((1u << lane) - 1u))] =
                    make_uint2(((uint32_t)i << 8) | mask[k], g[k]);
        }
        __syncthreads();
    }
    if (tid == 0) geo.tile_cursor[seg] = carry;
}

__global__ void __launch_bounds__(kSortThreads)
k_tile_sort(Dims d, Geom geo, unsigned long long *__restrict__ keys, unsigned long long *__restrict__ keys_alt,
            int cap, int id_bits) {
    extern __shared__ __align__(16) unsigned char s_sort[];
    if (*geo.n_instances > d.capacity) return;
    const int seg = blockIdx.x;
    const int n = (int)geo.tile_count[seg];
    const uint32_t s0 = geo.tile_start[seg];
    SortSmem &sm = *reinterpret_cast<SortSmem *>(s_sort);
    uint2 *live = reinterpret_cast<uint2 *>(keys_alt + s0);   // keys_alt is dead once the segment is sorted
    if (n < 2) { write_live_list(d, geo, keys + s0, n, seg, live, sm); return; }
    const int tid = threadIdx.x, lane = tid & 31;
    if (n > cap) {   // too long for shared memory: full-key radix through HBM
        unsigned long long *r = radix8_passes(keys + s0, keys_alt + s0, n, sm, 0, 0u, (id_bits + 7) / 8);
        unsigned long long *o = (r == keys + s0) ? keys_alt + s0 : keys + s0;
        r = radix8_passes(r, o, n, sm, 32, 0u, 4);
        if (r != keys + s0)
            for (int i = tid; i < n; i += kSortThreads) keys[s0 + i] = r[i];
        __syncthreads();
        write_live_list(d, geo, keys + s0, n, seg, live, sm);
        return;
    }
    unsigned long long *A = reinterpret_cast<unsigned long long *>(s_sort + sizeof(SortSmem));
    unsigned long long *B = A + cap;
    if (tid == 0) { sm.misc[1] = 0xffffffffu; sm.misc[2] = 0u; sm.misc[3] = 0u; }
    __syncthreads();
    uint32_t dlo = 0xffffffffu, dhi = 0u;
    for (int i = tid; i < n; i += kSortThreads) {
        const unsigned long long k = keys[s0 + i];
        A[i] = k;
        const uint32_t dpt = (uint32_t)(k >> 32);
        dlo = min(dlo, dpt); dhi = max(dhi, dpt);
    }
    dlo = __reduce_min_sync(0xffffffffu, dlo);
    dhi = __reduce_max_sync(0xffffffffu, dhi);
    if (lane == 0) { atomicMin(&sm.misc[1], dlo); atomicMax(&sm.misc[2], dhi); }
    __syncthreads();
    const uint32_t dmin = sm.misc[1], range = sm.misc[2] - dmin;
    const int bits = range ? 32 - __clz(range) : 0;
    __syncthreads();
    A = radix8_passes(A, B, n, sm, 32, dmin, (bits + 7) / 8);
    // ---- restore the Gaussian-index order inside runs of identical depth
    for (int i = tid; i < n; i += kSortThreads) {
        const uint32_t dpt = (uint32_t)(A[i] >> 32);
        const bool starts = (i == 0 || (uint32_t)(A[i - 1] >> 32) != dpt) && (i + 1 < n) &&
                            (uint32_t)(A[i + 1] >> 32) == dpt;
        if (starts) {
            int e = i + 2;
            while (e < n && (uint32_t)(A[e] >> 32) == dpt) ++e;
            if (e - i > 64) {
                sm.misc[3] = 1u;
            } else {
                for (int x = i + 1; x < e; ++x) {          // insertion sort of [i, e) on the full key
                    const unsigned long long v = A[x];
                    int y = x - 1;
                    while (y >= i && A[y] > v) { A[y + 1] = A[y]; --y; }
                    A[y + 1] = v;
                }
            }
        }
    }
    __syncthreads();
    if (sm.misc[3]) {
        int n_pad = 2;
        while (n_pad < n) n_pad <<= 1;                      // <= cap (cap is a power of two)
        for (int i = n + tid; i < n_pad; i += kSortThreads) A[i] = ~0ull;
        __syncthreads();
        bitonic_sort_smem<kSortThreads>(A, n_pad);
    }
    for (int i = tid; i < n; i += kSortThreads) keys[s0 + i] = A[i];
    write_live_list(d, geo, A, n, seg, live, sm);
}

// The live lists after the CUB debug sort (one CTA per segment, as in k_tile_sort).
__global__ void __launch_bounds__(kSortThreads)
k_live_lists(Dims d, Geom geo, const unsigned long long *__restrict__ keys, unsigned long long *__restrict__ keys_alt) {
    __shared__ SortSmem sm;
    if (*geo.n_instances > d.capacity) return;
    const int seg = blockIdx.x;
    const uint32_t s0 = geo.tile_start[seg];
    write_live_list(d, geo, keys + s0, (int)geo.tile_count[seg], seg, reinterpret_cast<uint2 *>(keys_alt + s0), sm);
}

int launch_binning(const Dims &d, const Geom &g, unsigned long long *keys,
                   unsigned long long *keys_alt, int sort_impl, int segment_hint, cudaEvent_t scanned,
                   cudaStream_t st) {
    const int n_seg = d.S * d.V * d.tiles;
    k_tile_scan<<<1, kScanThreads, 0, st>>>(n_seg, g.tile_count, g.tile_start, g.tile_cursor, g.n_instances);
    PS_LAUNCH_CHECK("k_tile_scan");
    if (scanned) PS_CUDA_CHECK(cudaEventRecord(scanned, st));
    const int use_smem = d.tiles <= kScatterMaxSmemTiles;
    static unsigned long long scatter_attr_devices = 0;
    if (first_use_on_device(scatter_attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)(2 * sizeof(uint32_t) * kScatterMaxSmemTiles)));
    }
    dim3 sgrid((d.P + kScatterThreads - 1) / kScatterThreads, d.S * d.V);
    k_scatter<<<sgrid, kScatterThreads, use_smem ? 2 * sizeof(uint32_t) * d.tiles : 0, st>>>(d, g, keys, use_smem);
    PS_LAUNCH_CHECK("k_scatter");
    mark(kMarkScatter, st);

    int id_bits = 1;
    while ((1ll << id_bits) < d.P) ++id_bits;

    if (sort_impl == 1) {
        // Debug path: CUB segmented sort over the same segments (used only to cross-check
        // the native sort in tests; needs n_instances <= capacity, guaranteed by the caller).
        size_t temp = 0;
        cub::DoubleBuffer<unsigned long long> db(keys, keys_alt);
        PS_CUDA_CHECK(cub::DeviceSegmentedRadixSort::SortKeys(nullptr, temp, db, (int)d.capacity, n_seg,
                                                              g.tile_start, g.tile_cursor, 0, 64, st));
        void *tmp = nullptr;
        PS_CUDA_CHECK(cudaMallocAsync(&tmp, temp, st));
        PS_CUDA_CHECK(cub::DeviceSegmentedRadixSort::SortKeys(tmp, temp, db, (int)d.capacity, n_seg,
                                                              g.tile_start, g.tile_cursor, 0, 64, st));
        if (db.Current() != keys)
            PS_CUDA_CHECK(cudaMemcpyAsync(keys, db.Current(), sizeof(unsigned long long) * (size_t)d.capacity,
                                          cudaMemcpyDeviceToDevice, st));
        PS_CUDA_CHECK(cudaFreeAsync(tmp, st));
        k_live_lists<<<n_seg, kSortThreads, 0, st>>>(d, g, keys, keys_alt);
        PS_LAUNCH_CHECK("k_live_lists");
        return PS_OK;
    }

    // shared-memory capacity: a power of two picked from the previous call's longest segment
    // (+25 % head-room); longer segments are still sorted correctly, through HBM
    int cap = 2048;
    if (segment_hint > 0) {
        const long long want = (long long)segment_hint + segment_hint / 4;
        while (cap < want && cap < 8192) cap <<= 1;
    }
    static unsigned long long battr_devices = 0;
    if (first_use_on_device(battr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_tile_sort, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)sort_smem_bytes(8192)));
    }
    k_tile_sort<<<n_seg, kSortThreads, sort_smem_bytes(cap), st>>>(d, g, keys, keys_alt, cap, id_bits);
    PS_LAUNCH_CHECK("k_tile_sort");
    return PS_OK;
}

}  // namespace ps
