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
constexpr float kLog2e = 1.4426950408889634f;

__device__ __forceinline__ void cp_async16(void *dst, const void *src, bool valid) {
    const int n = valid ? 16 : 0;                                  // 0: zero-fill, nothing is read
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void sync_before_mma() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic -> async proxy (smem operands)
    __syncthreads();
}

template <int N>
__device__ __forceinline__ void zero(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) d[i] = 0.0f;
}

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

}  // namespace

__global__ void __launch_bounds__(kVaThreads, 1)
k_vit_attn_fwd(const float *__restrict__ qkv, float *__restrict__ out, float *__restrict__ lse, int L, int n_heads,
               float scale_log2e) {
    extern __shared__ __align__(128) unsigned char s_va[];
    unsigned char *sQ = s_va;                                        // 128 x 64
    unsigned char *sK = sQ + kRowsBytes;                             // 2 x (64 x 64)
    unsigned char *sV = sK + 2 * kTileBytes;                         // 2 x (64 x 64), natural
    unsigned char *sVt = sV + 2 * kTileBytes;                        // V^T of the current tile
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int t = lane & 3;
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);         // first of this thread's rows (+8)
    const int q0 = blockIdx.x * kVaRows, head = blockIdx.y, img = blockIdx.z;
    const int inner = n_heads * kVaD;
    const size_t rs3 = 3 * (size_t)inner;
    const float *q_img = qkv + (size_t)img * L * rs3 + (size_t)head * kVaD;
    const float *k_img = q_img + inner, *v_img = q_img + 2 * inner;
    const int n_tiles = (L + kVaTile - 1) / kVaTile;

    load_async<kVaRows>(sQ, q_img + (size_t)q0 * rs3, rs3, L - q0, tid);
    load_async<kVaTile>(sK, k_img, rs3, L, tid);
    load_async<kVaTile>(sV, v_img, rs3, L, tid);
    cp_async_commit();

    float o[32];
    zero(o);
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.0f, l1 = 0.0f;     // running max (log2 units), partial row sums
#pragma unroll 1
    for (int j = 0; j < n_tiles; ++j) {
        const int k0 = j * kVaTile;
        unsigned char *bK = sK + (j & 1) * kTileBytes, *bV = sV + (j & 1) * kTileBytes;
        if (j + 1 < n_tiles) {
            const int k1 = k0 + kVaTile;
            load_async<kVaTile>(sK + ((j + 1) & 1) * kTileBytes, k_img + (size_t)k1 * rs3, rs3, L - k1, tid);
            load_async<kVaTile>(sV + ((j + 1) & 1) * kTileBytes, v_img + (size_t)k1 * rs3, rs3, L - k1, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (j == 0) round_tile<kVaRows>(sQ, tid);
        round_tile<kVaTile>(bK, tid);
        round_and_transpose(bV, sVt, tid);
        sync_before_mma();

        float s[32];
        zero(s);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kVaD / 8; ++k)
            wgmma_ss_n64(s, gmma_desc(smem_u32(sQ) + k * 2 * kLbo128 + wg * 64 * 16, kLbo128, 128),
                         gmma_desc(smem_u32(bK) + k * 2 * kLbo64, kLbo64, 128), k > 0);
        wgmma_commit();
        wgmma_wait_all();
        fence_operands(s);

        // online soft-max over this tile's keys of rows `row` (s[4 x + 0 / 1]) and `row + 8` (s[4 x + 2 / 3])
        float mx0 = m0, mx1 = m1;
#pragma unroll
        for (int x = 0; x < 32; ++x) {
            const bool valid = k0 + 8 * (x >> 2) + 2 * t + (x & 1) < L;
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

        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kVaTile / 8; ++kk) {
            uint32_t a[4];
            acc_to_a(s, kk, a);
            wgmma_rs_n64(o, a, gmma_desc(smem_u32(sVt) + kk * 2 * kLbo64, kLbo64, 128), 1);
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_operands(o);
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
        for (int x = 0; x < 8; ++x)
            *reinterpret_cast<float2 *>(dst + 8 * x) = make_float2(o[4 * x] * inv0, o[4 * x + 1] * inv0);
        if (t == 0) lse[((size_t)img * n_heads + head) * L + i0] = (m0 + log2f(l0)) * 0.6931471805599453f;
    }
    if (i1 < L) {
#pragma unroll
        for (int x = 0; x < 8; ++x)
            *reinterpret_cast<float2 *>(dst + 8 * (size_t)inner + 8 * x) = make_float2(o[4 * x + 2] * inv1, o[4 * x + 3] * inv1);
        if (t == 0) lse[((size_t)img * n_heads + head) * L + i1] = (m1 + log2f(l1)) * 0.6931471805599453f;
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
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int t = lane & 3;
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int j0 = blockIdx.x * kVaRows, head = blockIdx.y, img = blockIdx.z;
    const int inner = n_heads * kVaD;
    const size_t rs3 = 3 * (size_t)inner, rs1 = (size_t)inner;
    const float *q_img = qkv + (size_t)img * L * rs3 + (size_t)head * kVaD;
    const float *k_img = q_img + inner, *v_img = q_img + 2 * inner;
    const float *do_img = d_out + (size_t)img * L * rs1 + (size_t)head * kVaD;
    const float *lse_h = lse + ((size_t)img * n_heads + head) * L;
    const float *D_h = Dws + ((size_t)img * n_heads + head) * L;
    const int n_tiles = (L + kVaTile - 1) / kVaTile;
    const uint32_t a_row = (uint32_t)wg * 64 * 16;

    load_async<kVaRows>(sK, k_img + (size_t)j0 * rs3, rs3, L - j0, tid);
    load_async<kVaRows>(sV, v_img + (size_t)j0 * rs3, rs3, L - j0, tid);
    load_async<kVaTile>(sQ, q_img, rs3, L, tid);
    load_async<kVaTile>(sO, do_img, rs1, L, tid);
    cp_async_commit();

    float dv[32], dk[32];
    zero(dv);
    zero(dk);
#pragma unroll 1
    for (int c = 0; c < n_tiles; ++c) {
        const int i0 = c * kVaTile;
        unsigned char *bQ = sQ + (c & 1) * kTileBytes, *bO = sO + (c & 1) * kTileBytes;
        if (c + 1 < n_tiles) {
            const int i1 = i0 + kVaTile;
            load_async<kVaTile>(sQ + ((c + 1) & 1) * kTileBytes, q_img + (size_t)i1 * rs3, rs3, L - i1, tid);
            load_async<kVaTile>(sO + ((c + 1) & 1) * kTileBytes, do_img + (size_t)i1 * rs1, rs1, L - i1, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
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
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kVaD / 8; ++k) {
            wgmma_ss_n64(st, gmma_desc(smem_u32(sK) + k * 2 * kLbo128 + a_row, kLbo128, 128),
                         gmma_desc(smem_u32(bQ) + k * 2 * kLbo64, kLbo64, 128), k > 0);
            wgmma_ss_n64(dpt, gmma_desc(smem_u32(sV) + k * 2 * kLbo128 + a_row, kLbo128, 128),
                         gmma_desc(smem_u32(bO) + k * 2 * kLbo64, kLbo64, 128), k > 0);
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_operands(st);
        fence_operands(dpt);
        // thread = key row: S^T -> P^T, dP^T -> dS^T in place; query i0 + q, q = column 8 (x >> 2) + 2 t + (x & 1)
#pragma unroll
        for (int x = 0; x < 32; ++x) {
            const int q = 8 * (x >> 2) + 2 * t + (x & 1);
            const float p = exp2f(st[x] * scale_log2e - s_lse[q]);
            st[x] = to_tf32(p);
            dpt[x] = to_tf32(p * (dpt[x] - s_D[q]) * scale);
        }
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kVaTile / 8; ++kk) {
            uint32_t a[4];
            acc_to_a(st, kk, a);
            wgmma_rs_n64(dv, a, gmma_desc(smem_u32(sOt) + kk * 2 * kLbo64, kLbo64, 128), 1);
        }
#pragma unroll
        for (int kk = 0; kk < kVaTile / 8; ++kk) {
            uint32_t a[4];
            acc_to_a(dpt, kk, a);
            wgmma_rs_n64(dk, a, gmma_desc(smem_u32(sQt) + kk * 2 * kLbo64, kLbo64, 128), 1);
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_operands(dv);
        fence_operands(dk);
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
            *reinterpret_cast<float2 *>(dkp + 8 * x) = make_float2(dk[4 * x + 2 * h], dk[4 * x + 2 * h + 1]);
            *reinterpret_cast<float2 *>(dvp + 8 * x) = make_float2(dv[4 * x + 2 * h], dv[4 * x + 2 * h + 1]);
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
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int t = lane & 3;
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int q0 = blockIdx.x * kVaRows, head = blockIdx.y, img = blockIdx.z;
    const int inner = n_heads * kVaD;
    const size_t rs3 = 3 * (size_t)inner, rs1 = (size_t)inner;
    const float *q_img = qkv + (size_t)img * L * rs3 + (size_t)head * kVaD;
    const float *k_img = q_img + inner, *v_img = q_img + 2 * inner;
    const float *do_img = d_out + (size_t)img * L * rs1 + (size_t)head * kVaD;
    const size_t hL = ((size_t)img * n_heads + head) * L;
    const int n_tiles = (L + kVaTile - 1) / kVaTile;
    const uint32_t a_row = (uint32_t)wg * 64 * 16;

    load_async<kVaRows>(sQ, q_img + (size_t)q0 * rs3, rs3, L - q0, tid);
    load_async<kVaRows>(sO, do_img + (size_t)q0 * rs1, rs1, L - q0, tid);
    load_async<kVaTile>(sK, k_img, rs3, L, tid);
    load_async<kVaTile>(sV, v_img, rs3, L, tid);
    cp_async_commit();

    const int i0 = q0 + row, i1 = i0 + 8;
    const float lse0 = i0 < L ? lse[hL + i0] * kLog2e : 0.0f, D0 = i0 < L ? Dws[hL + i0] : 0.0f;
    const float lse1 = i1 < L ? lse[hL + i1] * kLog2e : 0.0f, D1 = i1 < L ? Dws[hL + i1] : 0.0f;
    float dq[32];
    zero(dq);
#pragma unroll 1
    for (int j = 0; j < n_tiles; ++j) {
        const int k0 = j * kVaTile;
        unsigned char *bK = sK + (j & 1) * kTileBytes, *bV = sV + (j & 1) * kTileBytes;
        if (j + 1 < n_tiles) {
            const int k1 = k0 + kVaTile;
            load_async<kVaTile>(sK + ((j + 1) & 1) * kTileBytes, k_img + (size_t)k1 * rs3, rs3, L - k1, tid);
            load_async<kVaTile>(sV + ((j + 1) & 1) * kTileBytes, v_img + (size_t)k1 * rs3, rs3, L - k1, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
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
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kVaD / 8; ++k) {
            wgmma_ss_n64(s, gmma_desc(smem_u32(sQ) + k * 2 * kLbo128 + a_row, kLbo128, 128),
                         gmma_desc(smem_u32(bK) + k * 2 * kLbo64, kLbo64, 128), k > 0);
            wgmma_ss_n64(dp, gmma_desc(smem_u32(sO) + k * 2 * kLbo128 + a_row, kLbo128, 128),
                         gmma_desc(smem_u32(bV) + k * 2 * kLbo64, kLbo64, 128), k > 0);
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_operands(s);
        fence_operands(dp);
#pragma unroll
        for (int x = 0; x < 32; ++x) {
            const bool valid = k0 + 8 * (x >> 2) + 2 * t + (x & 1) < L;
            const float p = valid ? exp2f(s[x] * scale_log2e - ((x & 2) ? lse1 : lse0)) : 0.0f;
            s[x] = to_tf32(p * (dp[x] - ((x & 2) ? D1 : D0)) * scale);
        }
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kVaTile / 8; ++kk) {
            uint32_t a[4];
            acc_to_a(s, kk, a);
            wgmma_rs_n64(dq, a, gmma_desc(smem_u32(sKt) + kk * 2 * kLbo64, kLbo64, 128), 1);
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_operands(dq);
        __syncthreads();
    }
    float *dq_img = d_qkv + (size_t)img * L * rs3 + (size_t)head * kVaD + 2 * t;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int i = i0 + 8 * h;
        if (i >= L) continue;
#pragma unroll
        for (int x = 0; x < 8; ++x)
            *reinterpret_cast<float2 *>(dq_img + (size_t)i * rs3 + 8 * x) = make_float2(dq[4 * x + 2 * h], dq[4 * x + 2 * h + 1]);
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
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices))
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_vit_attn_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFwdSmem));
    const dim3 grid((tokens + kVaRows - 1) / kVaRows, heads, n_images);
    k_vit_attn_fwd<<<grid, kVaThreads, kFwdSmem, static_cast<cudaStream_t>(stream)>>>(qkv, out, lse, tokens, heads,
                                                                                      scale * kLog2e);
    PS_LAUNCH_CHECK("k_vit_attn_fwd");
    return PS_OK;
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
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_vit_attn_bwd_dkdv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDkdvSmem));
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_vit_attn_bwd_dq, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDqSmem));
    }
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    float *D = static_cast<float *>(workspace);
    const long long n_rows = (long long)n_images * tokens * heads;
    k_vit_attn_bwd_d<<<(unsigned)(((size_t)n_rows * 16 + 255) / 256), 256, 0, st>>>(out, d_out, D, n_rows, tokens, heads);
    PS_LAUNCH_CHECK("k_vit_attn_bwd_d");
    const dim3 grid((tokens + kVaRows - 1) / kVaRows, heads, n_images);
    k_vit_attn_bwd_dkdv<<<grid, kVaThreads, kDkdvSmem, st>>>(qkv, d_out, lse, D, d_qkv, tokens, heads, scale, scale * kLog2e);
    PS_LAUNCH_CHECK("k_vit_attn_bwd_dkdv");
    k_vit_attn_bwd_dq<<<grid, kVaThreads, kDqSmem, st>>>(qkv, d_out, lse, D, d_qkv, tokens, heads, scale, scale * kLog2e);
    PS_LAUNCH_CHECK("k_vit_attn_bwd_dq");
    return PS_OK;
}
