// Flash-style multi-head self-attention of DINO's ViT blocks on the Hopper tensor cores (wgmma, TF32 operands,
// FP32 accumulators), forward and backward, for any token count L (the CLS token makes it odd: 257, 1025, 4097):
//     out[img, i, head] = softmax(q k^T * scale) v       q, k, v: [L, 64] per (image, head)
// No L x L tensor exists anywhere: the forward keeps one 64 x 64 tile of logits per warpgroup in registers.
//
// Forward (k_vit_attn_fwd): one CTA per (128-query tile, head, image), warpgroup w owns queries 64 w .. 64 w + 63.
// The 64-key tiles of K and V stream through shared memory, double-buffered with cp.async (rows past L are
// zero-filled without being read).  Per tile: S = Q K^T (m64n64k8 x 8), keys past L -> -inf, online soft-max
// (running max, per-thread partial row sums rescaled by the same factor as O), O += P V with A = P straight from
// the S registers and B = V^T transposed in shared memory.  The epilogue divides by the row sum and saves the
// per-row log-sum-exp lse = ln sum_j exp(s_ij * scale).
//
// Backward (FA2, P recomputed from lse; every operand rounded to the nearest TF32 like the forward's):
//   k_vit_attn_bwd_d:    D_i = dO_i . O_i                              (workspace [n, H, L])
//   k_vit_attn_bwd_dkdv: one CTA per 128-key tile; for each 64-query tile C: S^T = K_J Q_C^T, dP^T = V_J dO_C^T,
//                        P^T = exp(S^T scale - lse), dS^T = P^T o (dP^T - D) scale, dV_J += P^T dO_C,
//                        dK_J += dS^T Q_C.
//   k_vit_attn_bwd_dq:   one CTA per 128-query tile; for each 64-key tile: the same P and dS, dQ_I += dS K_j.
// Each output row is owned by exactly one thread and summed in a fixed order: no atomics, the same bits every run.
#include <initializer_list>

#include "wgmma_tf32.cuh"

namespace ps {

namespace {

constexpr int kVaD = 64;              // head dimension
constexpr int kVaThreads = 256;       // two warpgroups
constexpr int kVaRows = 128;          // rows a CTA owns (64 per warpgroup)
constexpr int kVaTile = 64;           // rows of a streamed tile
constexpr int kVaMaxTokens = 16384;
constexpr int kVaMaxHeads = 16;
constexpr uint32_t kLbo64 = 64 * 16;  // bytes between 16-byte K chunks of a 64-row tile
constexpr uint32_t kLbo128 = 128 * 16;
constexpr int kTileBytes = kVaTile * kVaD * 4;   // 16 KB
constexpr int kRowsBytes = kVaRows * kVaD * 4;   // 32 KB

__device__ __forceinline__ void cp_async16(void *dst, const void *src, bool valid) {
    const int n = valid ? 16 : 0;                                  // 0: zero-fill, nothing is read
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ROWS x 64 fp32 rows `src` (row stride in floats) -> canonical K-major no-swizzle layout: 16-byte chunk c of row r
// at c * ROWS * 16 + r * 16.  Rows >= rows_valid are zero-filled without touching global memory.
template <int ROWS>
__device__ __forceinline__ void load_async(unsigned char *dst, const float *src, size_t row_stride, int rows_valid,
                                           int tid) {
#pragma unroll 4
    for (int i = tid; i < ROWS * 16; i += kVaThreads) {
        const int r = i % ROWS, c = i / ROWS;
        const bool ok = r < rows_valid;
        cp_async16(dst + (size_t)i * 16, src + (ok ? (size_t)r * row_stride : 0) + 4 * c, ok);
    }
}

// In place fp32 -> nearest TF32 of a landed tile (the tensor core would truncate).
template <int ROWS>
__device__ __forceinline__ void round_tile(unsigned char *buf, int tid) {
#pragma unroll 4
    for (int i = tid; i < ROWS * 16; i += kVaThreads) {
        float4 *p = reinterpret_cast<float4 *>(buf + (size_t)i * 16);
        *p = to_tf32(*p);
    }
}

// Rounds a landed 64-token natural tile in place and writes its transpose: MMA rows (N) = the 64 channels, K = the
// 64 tokens in acc_to_a's order (chunk 2 kk + h holds tokens 8 kk + h + {0, 2, 4, 6} of one channel).
__device__ __forceinline__ void round_and_transpose(unsigned char *nat, unsigned char *tr, int tid) {
#pragma unroll 4
    for (int i = tid; i < kVaTile * 16; i += kVaThreads) {
        const int r = i % kVaTile, c = i / kVaTile;                 // token r, channels 4 c .. 4 c + 3
        float4 *p = reinterpret_cast<float4 *>(nat + (size_t)i * 16);
        const float4 v = to_tf32(*p);
        *p = v;
        const int w = r & 7;
        float *d = reinterpret_cast<float *>(tr + ((2 * (r >> 3) + (w & 1)) * kVaD + 4 * c) * 16) + (w >> 1);
        d[0] = v.x;
        d[4] = v.y;
        d[8] = v.z;
        d[12] = v.w;
    }
}

// Double-buffered stream of the 64-row tiles of two [L, 64] operands a and b (row strides in floats), each through
// two kTileBytes buffers: tile j of a lands at tile_a(j).
struct TileStream {
    unsigned char *sa, *sb;
    const float *a, *b;
    size_t rs_a, rs_b;
    int L, n_tiles;
    __device__ __forceinline__ unsigned char *tile_a(int j) const { return sa + (j & 1) * kTileBytes; }
    __device__ __forceinline__ unsigned char *tile_b(int j) const { return sb + (j & 1) * kTileBytes; }
    // Rows r0 .. r0 + 63 of a and b into buffer pair `buf` (0 or 1).
    __device__ __forceinline__ void load(int buf, int r0, int tid) const {
        load_async<kVaTile>(sa + buf * kTileBytes, a + (size_t)r0 * rs_a, rs_a, L - r0, tid);
        load_async<kVaTile>(sb + buf * kTileBytes, b + (size_t)r0 * rs_b, rs_b, L - r0, tid);
    }
    // Prefetches tile j + 1, waits for tile j (tile 0 is loaded in the kernel's first commit group), syncs the CTA.
    __device__ __forceinline__ void wait(int j, int tid) const {
        if (j + 1 < n_tiles) {
            load((j + 1) & 1, j * kVaTile + kVaTile, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
    }
};

// This CTA's (image, head) slice: its q, k, v columns in qkv-shaped tensors (rows rs3 floats apart, k and v at
// + inner and + 2 inner), its columns in [n, L, H * 64] tensors (rows rs1 apart), its row of [n, H, L] tensors.
struct HeadSlice {
    int inner;
    size_t rs3, rs1, qkv, rows, hl;
    __device__ __forceinline__ HeadSlice(int L, int n_heads) {
        const int head = blockIdx.y, img = blockIdx.z;
        inner = n_heads * kVaD;
        rs3 = 3 * (size_t)inner;
        rs1 = (size_t)inner;
        qkv = (size_t)img * L * rs3 + (size_t)head * kVaD;
        rows = (size_t)img * L * rs1 + (size_t)head * kVaD;
        hl = ((size_t)img * n_heads + head) * L;
    }
};

// The backward's rebuild of the forward's probability P = exp(s scale - lse) of logit s, lse in log2 units, and
// of dS = P o (dP - D) scale, rounded as the next MMA sees it.
__device__ __forceinline__ float prob(float s, float scale_log2e, float lse2) { return exp2f(s * scale_log2e - lse2); }
__device__ __forceinline__ float dscore(float p, float dp, float D, float scale) { return to_tf32(p * (dp - D) * scale); }

}  // namespace

__global__ void __launch_bounds__(kVaThreads, 1)
k_vit_attn_fwd(const float *__restrict__ qkv, float *__restrict__ out, float *__restrict__ lse, int L, int n_heads,
               float scale_log2e) {
    extern __shared__ __align__(128) unsigned char s_va[];
    unsigned char *sQ = s_va;                                        // 128 x 64
    unsigned char *sK = sQ + kRowsBytes;                             // 2 x (64 x 64)
    unsigned char *sV = sK + 2 * kTileBytes;                         // 2 x (64 x 64), natural
    unsigned char *sVt = sV + 2 * kTileBytes;                        // V^T of the current tile
    const int tid = threadIdx.x;
    const Frag f;
    const int t = f.t, row = f.row;                                  // rows `row` and `row + 8`
    const int q0 = blockIdx.x * kVaRows, head = blockIdx.y, img = blockIdx.z;
    const HeadSlice hs(L, n_heads);
    const int inner = hs.inner;
    const float *q_img = qkv + hs.qkv;
    const TileStream kv{sK, sV, q_img + inner, q_img + 2 * inner, hs.rs3, hs.rs3, L, (L + kVaTile - 1) / kVaTile};

    load_async<kVaRows>(sQ, q_img + (size_t)q0 * hs.rs3, hs.rs3, L - q0, tid);
    kv.load(0, 0, tid);
    cp_async_commit();

    float o[32];
    zero(o);
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.0f, l1 = 0.0f;     // running max (log2 units), partial row sums
#pragma unroll 1
    for (int j = 0; j < kv.n_tiles; ++j) {
        const int k0 = j * kVaTile;
        unsigned char *bK = kv.tile_a(j), *bV = kv.tile_b(j);
        kv.wait(j, tid);
        if (j == 0) round_tile<kVaRows>(sQ, tid);
        round_tile<kVaTile>(bK, tid);
        round_and_transpose(bV, sVt, tid);
        sync_before_mma();

        float s[32];
        zero(s);
        mma_ss<kVaD / 8, kVaD / 8>(s, {smem_u32(sQ) + f.a_row(), kLbo128}, {smem_u32(bK), kLbo64});

        // online soft-max over this tile's keys of rows `row` (s[4 x + 0 / 1]) and `row + 8` (s[4 x + 2 / 3])
        float mx0 = m0, mx1 = m1;
#pragma unroll
        for (int x = 0; x < 32; ++x) {
            const bool valid = k0 + f.col(x) < L;
            s[x] = valid ? s[x] * scale_log2e : -INFINITY;
            if (x & 2) mx1 = fmaxf(mx1, s[x]);
            else mx0 = fmaxf(mx0, s[x]);
        }
#pragma unroll
        for (int sh = 1; sh < 4; sh <<= 1) {
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, sh));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, sh));
        }
        // every tile holds at least one valid key, so mx is finite and alpha = 0 on the first tile
        const float a0 = exp2f(m0 - mx0), a1 = exp2f(m1 - mx1);
        m0 = mx0;
        m1 = mx1;
        float sum0 = 0.0f, sum1 = 0.0f;
#pragma unroll
        for (int x = 0; x < 32; ++x) {
            s[x] = to_tf32(exp2f(s[x] - ((x & 2) ? mx1 : mx0)));    // the row sum is over what the MMA sees
            if (x & 2) sum1 += s[x];
            else sum0 += s[x];
            o[x] *= (x & 2) ? a1 : a0;
        }
        l0 = l0 * a0 + sum0;
        l1 = l1 * a1 + sum1;

        mma_rs<kVaTile / 8>(o, s, {smem_u32(sVt), kLbo64}, true);
        __syncthreads();                                             // buffers of tile j are free for tile j + 2
    }

#pragma unroll
    for (int sh = 1; sh < 4; sh <<= 1) {
        l0 += __shfl_xor_sync(0xffffffffu, l0, sh);
        l1 += __shfl_xor_sync(0xffffffffu, l1, sh);
    }
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    const int i0 = q0 + row, i1 = i0 + 8;
    float *dst = out + ((size_t)img * L + i0) * inner + (size_t)head * kVaD + 2 * t;
    if (i0 < L) {
#pragma unroll
        for (int x = 0; x < 8; ++x) store_cols(dst + 8 * x, o, x, 0, inv0);
        if (t == 0) lse[hs.hl + i0] = (m0 + log2f(l0)) * 0.6931471805599453f;
    }
    if (i1 < L) {
#pragma unroll
        for (int x = 0; x < 8; ++x) store_cols(dst + 8 * (size_t)inner + 8 * x, o, x, 1, inv1);
        if (t == 0) lse[hs.hl + i1] = (m1 + log2f(l1)) * 0.6931471805599453f;
    }
}

// D[img, head, i] = dO_i . O_i (dO rounded to TF32): 16 threads per (token, head) row of 64 channels, one float4 each.
__global__ void __launch_bounds__(256)
k_vit_attn_bwd_d(const float *__restrict__ out, const float *__restrict__ d_out, float *__restrict__ D, long long n_rows,
                 int L, int n_heads) {
    const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t r = g >> 4;                                         // (img * L + i) * H + head
    float acc = 0.0f;
    if (r < (size_t)n_rows) {
        const float4 a = __ldg(reinterpret_cast<const float4 *>(out + r * kVaD) + (g & 15));
        // dO rounded as the dP = dO V^T MMA sees it, so that the TF32 error of dO cancels in dP - D (it does not
        // when D takes the fp32 dO: under near-uniform attention dP - D is small and dQ, dK lose digits)
        const float4 b = to_tf32(__ldg(reinterpret_cast<const float4 *>(d_out + r * kVaD) + (g & 15)));
        acc = a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
    }
#pragma unroll
    for (int sh = 1; sh < 16; sh <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, sh);
    if (r < (size_t)n_rows && (g & 15) == 0) {
        const int head = (int)(r % n_heads);
        const size_t ti = r / n_heads, img = ti / L, i = ti % L;
        D[(img * n_heads + head) * L + i] = acc;
    }
}

__global__ void __launch_bounds__(kVaThreads, 1)
k_vit_attn_bwd_dkdv(const float *__restrict__ qkv, const float *__restrict__ d_out, const float *__restrict__ lse,
                    const float *__restrict__ Dws, float *__restrict__ d_qkv, int L, int n_heads, float scale,
                    float scale_log2e) {
    extern __shared__ __align__(128) unsigned char s_va[];
    unsigned char *sK = s_va;                                        // 128 x 64 (this CTA's keys)
    unsigned char *sV = sK + kRowsBytes;                             // 128 x 64
    unsigned char *sQ = sV + kRowsBytes;                             // 2 x (64 x 64), natural
    unsigned char *sO = sQ + 2 * kTileBytes;                         // 2 x (64 x 64) dO, natural
    unsigned char *sQt = sO + 2 * kTileBytes;                        // Q_C^T
    unsigned char *sOt = sQt + kTileBytes;                           // dO_C^T
    float *s_lse = reinterpret_cast<float *>(sOt + kTileBytes);      // [64] lse * log2 e of the chunk's queries
    float *s_D = s_lse + kVaTile;                                    // [64]
    const int tid = threadIdx.x;
    const Frag f;
    const int t = f.t, row = f.row;
    const int j0 = blockIdx.x * kVaRows, head = blockIdx.y, img = blockIdx.z;
    const HeadSlice hs(L, n_heads);
    const int inner = hs.inner;
    const size_t rs3 = hs.rs3, rs1 = hs.rs1;
    const float *q_img = qkv + hs.qkv;
    const float *k_img = q_img + inner, *v_img = q_img + 2 * inner;
    const float *do_img = d_out + hs.rows;
    const float *lse_h = lse + hs.hl, *D_h = Dws + hs.hl;
    const TileStream qo{sQ, sO, q_img, do_img, rs3, rs1, L, (L + kVaTile - 1) / kVaTile};
    const uint32_t a_row = f.a_row();

    load_async<kVaRows>(sK, k_img + (size_t)j0 * rs3, rs3, L - j0, tid);
    load_async<kVaRows>(sV, v_img + (size_t)j0 * rs3, rs3, L - j0, tid);
    qo.load(0, 0, tid);
    cp_async_commit();

    float dv[32], dk[32];
    zero(dv);
    zero(dk);
#pragma unroll 1
    for (int c = 0; c < qo.n_tiles; ++c) {
        const int i0 = c * kVaTile;
        unsigned char *bQ = qo.tile_a(c), *bO = qo.tile_b(c);
        qo.wait(c, tid);
        if (c == 0) {
            round_tile<kVaRows>(sK, tid);
            round_tile<kVaRows>(sV, tid);
        }
        round_and_transpose(bQ, sQt, tid);
        round_and_transpose(bO, sOt, tid);
        if (tid < kVaTile) {
            // a query past L gets lse = +inf, so that its P (and dS) is exactly 0
            const bool ok = i0 + tid < L;
            s_lse[tid] = ok ? lse_h[i0 + tid] * kLog2e : INFINITY;
            s_D[tid] = ok ? D_h[i0 + tid] : 0.0f;
        }
        sync_before_mma();

        float st[32], dpt[32];
        zero(st);
        zero(dpt);
        mma_ss<kVaD / 8, kVaD / 8>(st, {smem_u32(sK) + a_row, kLbo128}, {smem_u32(bQ), kLbo64},
                                   dpt, {smem_u32(sV) + a_row, kLbo128}, {smem_u32(bO), kLbo64});
        // thread = key row: S^T -> P^T, dP^T -> dS^T in place; query i0 + column
#pragma unroll
        for (int x = 0; x < 32; ++x) {
            const int q = f.col(x);
            const float p = prob(st[x], scale_log2e, s_lse[q]);
            st[x] = to_tf32(p);
            dpt[x] = dscore(p, dpt[x], s_D[q], scale);
        }
        mma_rs<kVaTile / 8>(dv, st, {smem_u32(sOt), kLbo64}, dk, dpt, {smem_u32(sQt), kLbo64});
        __syncthreads();
    }
    float *dk_img = d_qkv + (size_t)img * L * rs3 + inner + (size_t)head * kVaD;
    float *dv_img = dk_img + inner;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int j = j0 + row + 8 * h;
        if (j >= L) continue;
        float *dkp = dk_img + (size_t)j * rs3 + 2 * t, *dvp = dv_img + (size_t)j * rs3 + 2 * t;
#pragma unroll
        for (int x = 0; x < 8; ++x) {
            store_cols(dkp + 8 * x, dk, x, h);
            store_cols(dvp + 8 * x, dv, x, h);
        }
    }
}

__global__ void __launch_bounds__(kVaThreads, 1)
k_vit_attn_bwd_dq(const float *__restrict__ qkv, const float *__restrict__ d_out, const float *__restrict__ lse,
                  const float *__restrict__ Dws, float *__restrict__ d_qkv, int L, int n_heads, float scale,
                  float scale_log2e) {
    extern __shared__ __align__(128) unsigned char s_va[];
    unsigned char *sQ = s_va;                                        // 128 x 64 (this CTA's queries)
    unsigned char *sO = sQ + kRowsBytes;                             // 128 x 64 dO
    unsigned char *sK = sO + kRowsBytes;                             // 2 x (64 x 64), natural
    unsigned char *sV = sK + 2 * kTileBytes;                         // 2 x (64 x 64), natural
    unsigned char *sKt = sV + 2 * kTileBytes;                        // K_j^T
    const int tid = threadIdx.x;
    const Frag f;
    const int q0 = blockIdx.x * kVaRows;
    const HeadSlice hs(L, n_heads);
    const size_t rs3 = hs.rs3, rs1 = hs.rs1, hL = hs.hl;
    const float *q_img = qkv + hs.qkv;
    const float *do_img = d_out + hs.rows;
    const TileStream kv{sK, sV, q_img + hs.inner, q_img + 2 * hs.inner, rs3, rs3, L, (L + kVaTile - 1) / kVaTile};
    const uint32_t a_row = f.a_row();

    load_async<kVaRows>(sQ, q_img + (size_t)q0 * rs3, rs3, L - q0, tid);
    load_async<kVaRows>(sO, do_img + (size_t)q0 * rs1, rs1, L - q0, tid);
    kv.load(0, 0, tid);
    cp_async_commit();

    const int i0 = q0 + f.row, i1 = i0 + 8;
    const float lse0 = i0 < L ? lse[hL + i0] * kLog2e : 0.0f, D0 = i0 < L ? Dws[hL + i0] : 0.0f;
    const float lse1 = i1 < L ? lse[hL + i1] * kLog2e : 0.0f, D1 = i1 < L ? Dws[hL + i1] : 0.0f;
    float dq[32];
    zero(dq);
#pragma unroll 1
    for (int j = 0; j < kv.n_tiles; ++j) {
        const int k0 = j * kVaTile;
        unsigned char *bK = kv.tile_a(j), *bV = kv.tile_b(j);
        kv.wait(j, tid);
        if (j == 0) {
            round_tile<kVaRows>(sQ, tid);
            round_tile<kVaRows>(sO, tid);
        }
        round_and_transpose(bK, sKt, tid);
        round_tile<kVaTile>(bV, tid);
        sync_before_mma();

        float s[32], dp[32];
        zero(s);
        zero(dp);
        mma_ss<kVaD / 8, kVaD / 8>(s, {smem_u32(sQ) + a_row, kLbo128}, {smem_u32(bK), kLbo64},
                                   dp, {smem_u32(sO) + a_row, kLbo128}, {smem_u32(bV), kLbo64});
        // keys past L: P = dS = 0
#pragma unroll
        for (int x = 0; x < 32; ++x) {
            const bool valid = k0 + f.col(x) < L;
            const float p = valid ? prob(s[x], scale_log2e, (x & 2) ? lse1 : lse0) : 0.0f;
            s[x] = dscore(p, dp[x], (x & 2) ? D1 : D0, scale);
        }
        mma_rs<kVaTile / 8>(dq, s, {smem_u32(sKt), kLbo64}, true);
        __syncthreads();
    }
    float *dq_img = d_qkv + hs.qkv + 2 * f.t;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int i = i0 + 8 * h;
        if (i >= L) continue;
#pragma unroll
        for (int x = 0; x < 8; ++x) store_cols(dq_img + (size_t)i * rs3 + 8 * x, dq, x, h);
    }
}

namespace {

constexpr size_t kFwdSmem = kRowsBytes + 5 * kTileBytes;                            // 112 KB
constexpr size_t kDkdvSmem = 2 * kRowsBytes + 6 * kTileBytes + 2 * kVaTile * 4;   // 160.5 KB
constexpr size_t kDqSmem = 2 * kRowsBytes + 5 * kTileBytes;                         // 144 KB

int check_shape(const char *who, int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head) {
    if (n_images < 1 || tokens < 1 || heads < 1) {
        set_error("%s: n_images, tokens and heads must be >= 1 (got %d, %d, %d)", who, n_images, tokens, heads);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (dim_head != kVaD || tokens > kVaMaxTokens || heads > kVaMaxHeads || n_images > 65535) {
        set_error("%s: supported are dim_head == 64, tokens <= %d, heads <= %d, n_images <= 65535 "
                  "(got %d, %d, %d, %d)", who, kVaMaxTokens, kVaMaxHeads, dim_head, tokens, heads, n_images);
        return PS_ERR_UNSUPPORTED;
    }
    return PS_OK;
}

size_t workspace_bytes(int32_t n_images, int32_t tokens, int32_t heads) {
    return (size_t)n_images * heads * tokens * sizeof(float);                      // D = rowsum(dO o O)
}

bool misaligned(std::initializer_list<const void *> ps) {
    uintptr_t a = 0;
    for (const void *p : ps) a |= (uintptr_t)p;
    return (a & 15) != 0;
}

unsigned long long attr_devices = 0;

// Launches one of the three tiled kernels over (128-row tile, head, image).  The first launch on a device raises the
// dynamic shared-memory limit of all three.
template <typename Kernel, typename... Args>
int launch_tiled(Kernel kernel, size_t smem, const char *name, int32_t n_images, int32_t tokens, int32_t heads,
                 cudaStream_t st, Args... args) {
    if (first_use_on_device(attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_vit_attn_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFwdSmem));
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_vit_attn_bwd_dkdv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDkdvSmem));
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_vit_attn_bwd_dq, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDqSmem));
    }
    kernel<<<dim3((tokens + kVaRows - 1) / kVaRows, heads, n_images), kVaThreads, smem, st>>>(args...);
    PS_LAUNCH_CHECK(name);
    return PS_OK;
}

}  // namespace

}  // namespace ps

extern "C" PS_API int ps_vit_attention_forward(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                               const float *qkv, float scale, float *out, float *lse, void *stream) {
    using namespace ps;
    const int rc = check_shape("ps_vit_attention_forward", n_images, tokens, heads, dim_head);
    if (rc != PS_OK) return rc;
    if (!qkv || !out || !lse) { set_error("ps_vit_attention_forward: NULL pointer"); return PS_ERR_INVALID_ARGUMENT; }
    if (misaligned({qkv, out})) {
        set_error("ps_vit_attention_forward: qkv and out must be 16-byte aligned");
        return PS_ERR_INVALID_ARGUMENT;
    }
    return launch_tiled(k_vit_attn_fwd, kFwdSmem, "k_vit_attn_fwd", n_images, tokens, heads,
                        static_cast<cudaStream_t>(stream), qkv, out, lse, tokens, heads, scale * kLog2e);
}

extern "C" PS_API int ps_vit_attention_backward_workspace_bytes(int32_t n_images, int32_t tokens, int32_t heads,
                                                                int32_t dim_head, size_t *out) {
    using namespace ps;
    const int rc = check_shape("ps_vit_attention_backward_workspace_bytes", n_images, tokens, heads, dim_head);
    if (rc != PS_OK) return rc;
    if (!out) { set_error("ps_vit_attention_backward_workspace_bytes: out is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    *out = workspace_bytes(n_images, tokens, heads);
    return PS_OK;
}

extern "C" PS_API int ps_vit_attention_backward(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                                const float *qkv, const float *out, const float *d_out,
                                                const float *lse, float scale, float *d_qkv, void *workspace,
                                                size_t workspace_bytes_, void *stream) {
    using namespace ps;
    const int rc = check_shape("ps_vit_attention_backward", n_images, tokens, heads, dim_head);
    if (rc != PS_OK) return rc;
    if (!qkv || !out || !d_out || !lse || !d_qkv || !workspace) {
        set_error("ps_vit_attention_backward: NULL pointer");
        return PS_ERR_INVALID_ARGUMENT;
    }
    const size_t ws = workspace_bytes(n_images, tokens, heads);
    if (workspace_bytes_ < ws) {
        set_error("ps_vit_attention_backward: workspace of %zu bytes, %zu needed", workspace_bytes_, ws);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (misaligned({qkv, out, d_out, d_qkv})) {
        set_error("ps_vit_attention_backward: qkv, out, d_out and d_qkv must be 16-byte aligned");
        return PS_ERR_INVALID_ARGUMENT;
    }
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    float *D = static_cast<float *>(workspace);
    const long long n_rows = (long long)n_images * tokens * heads;
    k_vit_attn_bwd_d<<<(unsigned)(((size_t)n_rows * 16 + 255) / 256), 256, 0, st>>>(out, d_out, D, n_rows, tokens, heads);
    PS_LAUNCH_CHECK("k_vit_attn_bwd_d");
    const int rc2 = launch_tiled(k_vit_attn_bwd_dkdv, kDkdvSmem, "k_vit_attn_bwd_dkdv", n_images, tokens, heads, st,
                                 qkv, d_out, lse, D, d_qkv, tokens, heads, scale, scale * kLog2e);
    if (rc2 != PS_OK) return rc2;
    return launch_tiled(k_vit_attn_bwd_dq, kDqSmem, "k_vit_attn_bwd_dq", n_images, tokens, heads, st,
                        qkv, d_out, lse, D, d_qkv, tokens, heads, scale, scale * kLog2e);
}
