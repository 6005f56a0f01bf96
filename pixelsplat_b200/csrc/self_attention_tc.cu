// Dense per-image multi-head self-attention on the Hopper tensor cores (wgmma, TF32), forward and backward:
//     out[img, :, head] = softmax(Q K^T * scale) V      Q, K, V: [256 tokens, 128] per (image, head)
// for the ViT blocks of pixelSplat's ImageSelfAttention (reference: src/model/encoder/epipolar/
// image_self_attention.py:57-79 -> src/model/transformer/attention.py:54-70 with z = None): the only dense
// contractions of the hot path (SURVEY.md 8 row a14).
//
// Forward: one CTA (two warpgroups) per (image, head, 128-query half); warpgroup w owns queries 64 w .. 64 w + 63:
//   1. Q half [128 x 128] and K [256 x 128] are copied (fp32 rounded to the nearest TF32) into shared
//      memory in the canonical K-major no-swizzle layout (8-row x 16-byte core matrices);
//   2. each warpgroup issues 16 wgmma m64n256k8 accumulating its S = Q K^T rows in registers (128 per thread);
//   3. K's shared buffer is overwritten with V^T (d-major x tokens, same K-major layout); each thread turns
//      its two rows' S into un-normalised probabilities in place (row max and sum over the four threads that
//      share a row), rounded to TF32;
//   4. 32 wgmma m64n128k8 with A = P straight from those registers and B = V^T from shared memory accumulate O;
//   5. epilogue: scale by 1 / row sum, store.
// No TMA: the tiles are tiny and L2-resident; the copy is plain ld.global / st.shared followed by a proxy fence.
//
// Backward, per (image, head), with Pn the forward's probabilities -- rebuilt from the saved per-row (max, 1 / sum)
// by the forward's own `prob`, so the backward differentiates the forward that actually ran:
//     dPn = dO V^T      D_i = dO_i . O_i      dS = Pn o (dPn - D) * scale
//     dQ = dS K         dK = dS^T Q           dV = Pn^T dO
// Two CTA roles (grid.x = 4), two warpgroups of 64 rows each, every contraction a wgmma with FP32 accumulators
// in registers:
//   role 0/1 "query half I" -> dQ_I.  S = Q_I K^T (m64n256, 128 registers) becomes Pn in place; dPn = dO_I V^T
//            follows in two 128-key halves (64 registers each), each turned into dS over Pn's registers; then
//            dQ_I = dS K with A = dS straight from registers and B = K^T staged transposed.
//   role 2/3 "key half J"   -> dK_J, dV_J.  The transposed problem, so that the rows a CTA owns are the rows it
//            sums over: for the four 64-query chunks C in turn, S^T = K_J Q_C^T and dPn^T = V_J dO_C^T
//            (m64n64), thread = key row builds Pn^T and dS^T in place (the per-query constants max, 1 / sum
//            and D are per COLUMN here: 256-entry shared arrays), then dV_J += Pn^T dO_C and dK_J += dS^T Q_C
//            with A from registers and B = dO_C^T / Q_C^T staged transposed over the chunk's natural copies.
// Shared memory: 3 x 64 KB operand buffers (Q / dO + K / V in role 0/1; K_J, V_J + the chunk's two 32 KB
// operands in role 2/3); operands are rounded to the nearest TF32 on the way in, like the forward's.
#include <initializer_list>

#include "wgmma_tf32.cuh"

namespace ps {

namespace {

constexpr int kSaL = 256;        // tokens per image
constexpr int kSaD = 128;        // head dimension
constexpr int kSaThreads = 256;  // two warpgroups; warpgroup w owns MMA rows 64 w .. 64 w + 63 of the CTA's 128
constexpr uint32_t kLbo64 = 64 * 16;     // bytes between 16-byte K chunks of a 64-row tile
constexpr uint32_t kLbo128 = 128 * 16;
constexpr uint32_t kLbo256 = 256 * 16;
constexpr size_t kFwdSmem = 192 * 1024;
constexpr size_t kBwdSmem = 192 * 1024 + 3 * 256 * sizeof(float);

// Un-normalised probability of logit s in a row whose saved max is mb (max * scale * log2 e), rounded as the
// P V MMA sees it.
__device__ __forceinline__ float prob(float s, float scale_log2e, float mb) { return to_tf32(exp2f(s * scale_log2e - mb)); }

// dS = Pn o (dPn - D) * scale, rounded as the dQ / dK MMA sees it.
__device__ __forceinline__ float dscore(float pn, float dp, float D, float scale) { return to_tf32(pn * (dp - D) * scale); }

}  // namespace

// debug_mode: 0 = attention output; 1 = write the raw logits S = Q K^T instead (`out` is then
// [n_img, H, 256, 256]) -- used by the tests to isolate the first MMA stage.
__global__ void __launch_bounds__(kSaThreads, 1)
k_self_attention_tc(const float *__restrict__ qkv, float *__restrict__ out, float *__restrict__ stats, int n_heads,
                    float scale_log2e, int debug_mode) {
    extern __shared__ __align__(128) unsigned char s_sa[];
    unsigned char *sQ = s_sa;                                                      // 128 x 128 fp32 = 64 KB
    unsigned char *sK = s_sa + 64 * 1024;                                          // 256 x 128 fp32 = 128 KB (later V^T)
    const int tid = threadIdx.x;
    const Frag f;
    const int t = f.t, row = f.row;                                                // rows `row` and `row + 8`
    const int half = blockIdx.x, head = blockIdx.y, img = blockIdx.z;
    const int inner = n_heads * kSaD;
    const size_t row_stride = 3 * (size_t)inner;                                   // floats per token in qkv
    const float *q_base = qkv + ((size_t)img * kSaL + (size_t)half * 128) * row_stride + (size_t)head * kSaD;
    const float *k_base = qkv + (size_t)img * kSaL * row_stride + inner + (size_t)head * kSaD;
    const float *v_base = qkv + (size_t)img * kSaL * row_stride + 2 * inner + (size_t)head * kSaD;

    stage_natural<128>(sQ, q_base, row_stride, tid, kSaThreads);
    stage_natural<256>(sK, k_base, row_stride, tid, kSaThreads);
    sync_before_mma();

    // ---- S = Q K^T, this warpgroup's 64 rows
    float s[128];
    zero(s);
    mma_ss<kSaD / 8, 1>(s, {smem_u32(sQ) + f.a_row(), kLbo128}, {smem_u32(sK), kLbo256});
    if (debug_mode == 1) {
        store_row_pair<32>(out + ((((size_t)img * n_heads + head) * 2 + half) * 128 + row) * 256 + 2 * t, 256, s);
        return;
    }
    __syncthreads();                                   // both warpgroups' MMAs have completed: K is dead
    stage_transposed<256>(sK, v_base, row_stride, tid, kSaThreads);

    // ---- soft-max over the 256 keys of rows `row` (s[4 j], s[4 j + 1]) and `row + 8` (s[4 j + 2 / 3])
    float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        m0 = fmaxf(m0, fmaxf(s[4 * j], s[4 * j + 1]));
        m1 = fmaxf(m1, fmaxf(s[4 * j + 2], s[4 * j + 3]));
    }
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
        m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
        m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
    }
    const float mb0 = m0 * scale_log2e, mb1 = m1 * scale_log2e;
    float sum0 = 0.0f, sum1 = 0.0f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        s[4 * j] = prob(s[4 * j], scale_log2e, mb0);                      // the row sum is over what the MMA will see
        s[4 * j + 1] = prob(s[4 * j + 1], scale_log2e, mb0);
        s[4 * j + 2] = prob(s[4 * j + 2], scale_log2e, mb1);
        s[4 * j + 3] = prob(s[4 * j + 3], scale_log2e, mb1);
        sum0 += s[4 * j] + s[4 * j + 1];
        sum1 += s[4 * j + 2] + s[4 * j + 3];
    }
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
        sum0 += __shfl_xor_sync(0xffffffffu, sum0, o);
        sum1 += __shfl_xor_sync(0xffffffffu, sum1, o);
    }
    const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
    if (stats && t == 0) {   // what the backward needs to rebuild exactly these probabilities: (max * scale * log2 e, 1 / sum)
        float2 *st = reinterpret_cast<float2 *>(stats) + ((size_t)img * n_heads + head) * kSaL + half * 128 + row;
        st[0] = make_float2(mb0, inv0);
        st[8] = make_float2(mb1, inv1);
    }
    sync_before_mma();

    // ---- O = P V   (A = P from registers, B = V^T from shared memory)
    float o[64];
    zero(o);
    mma_rs<kSaL / 8>(o, s, {smem_u32(sK), kLbo128}, false);
    store_row_pair<16>(out + ((size_t)img * kSaL + (size_t)half * 128 + row) * inner + (size_t)head * kSaD + 2 * t,
                       inner, o, inv0, inv1);
}

__global__ void __launch_bounds__(kSaThreads, 1)
k_self_attention_tc_bwd(const float *__restrict__ qkv, const float *__restrict__ out, const float *__restrict__ d_out,
                        const float *__restrict__ stats, float *__restrict__ d_qkv, int n_heads, float scale,
                        float scale_log2e) {
    extern __shared__ __align__(128) unsigned char s_sa[];
    unsigned char *buf0 = s_sa, *buf1 = s_sa + 64 * 1024, *buf2 = s_sa + 128 * 1024;
    float *s_mb = reinterpret_cast<float *>(s_sa + 192 * 1024);          // [256] row max * scale * log2 e
    float *s_inv = s_mb + 256;                                            // [256] 1 / row sum
    float *s_D = s_inv + 256;                                             // [256] dO_i . O_i
    const int tid = threadIdx.x;
    const Frag f;
    const int row = f.row;                                                // first of this thread's rows (+8)
    const int role = blockIdx.x >> 1, half = blockIdx.x & 1, head = blockIdx.y, img = blockIdx.z;
    const int inner = n_heads * kSaD;
    const size_t rs3 = 3 * (size_t)inner, rs1 = (size_t)inner;            // floats per token in qkv / out
    const float *q_img = qkv + (size_t)img * kSaL * rs3 + (size_t)head * kSaD;
    const float *k_img = q_img + inner, *v_img = q_img + 2 * inner;
    const float *o_img = out + (size_t)img * kSaL * rs1 + (size_t)head * kSaD;
    const float *do_img = d_out + (size_t)img * kSaL * rs1 + (size_t)head * kSaD;
    float *dq_img = d_qkv + (size_t)img * kSaL * rs3 + (size_t)head * kSaD;
    float *dk_img = dq_img + inner, *dv_img = dq_img + 2 * inner;

    // per-query constants of all 256 queries: (max, 1 / sum) saved by the forward, D = dO . O
    {
        const int i = tid;                                                  // kSaThreads == kSaL
        const float2 st = reinterpret_cast<const float2 *>(stats)[((size_t)img * n_heads + head) * kSaL + i];
        s_mb[i] = st.x;
        s_inv[i] = st.y;
        const float4 *a = reinterpret_cast<const float4 *>(do_img + (size_t)i * rs1);
        const float4 *b = reinterpret_cast<const float4 *>(o_img + (size_t)i * rs1);
        float acc = 0.0f;
#pragma unroll 8
        for (int c = 0; c < kSaD / 4; ++c) {
            const float4 x = __ldg(a + c), y = __ldg(b + c);
            acc += x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
        }
        s_D[i] = acc;
    }

    if (role == 0) {
        // ================================================================= dQ for query half `half`
        unsigned char *sQ = buf0, *sK = buf1;                                 // 64 KB + 128 KB
        stage_natural<128>(sQ, q_img + (size_t)half * 128 * rs3, rs3, tid, kSaThreads);
        stage_natural<256>(sK, k_img, rs3, tid, kSaThreads);
        sync_before_mma();
        float s[128];
        zero(s);
        mma_ss<kSaD / 8, 1>(s, {smem_u32(sQ) + f.a_row(), kLbo128}, {smem_u32(sK), kLbo256});
        // S -> Pn in place (rows i0 = s[4 j + 0 / 1], i0 + 8 = s[4 j + 2 / 3])
        const int i0 = half * 128 + row;
        const float mb0 = s_mb[i0], inv0 = s_inv[i0], D0 = s_D[i0];
        const float mb1 = s_mb[i0 + 8], inv1 = s_inv[i0 + 8], D1 = s_D[i0 + 8];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            s[4 * j] = prob(s[4 * j], scale_log2e, mb0) * inv0;
            s[4 * j + 1] = prob(s[4 * j + 1], scale_log2e, mb0) * inv0;
            s[4 * j + 2] = prob(s[4 * j + 2], scale_log2e, mb1) * inv1;
            s[4 * j + 3] = prob(s[4 * j + 3], scale_log2e, mb1) * inv1;
        }
        __syncthreads();                                                      // Q and K are dead
        stage_natural<128>(sQ, do_img + (size_t)half * 128 * rs1, rs1, tid, kSaThreads);
        stage_natural<256>(sK, v_img, rs3, tid, kSaThreads);
        sync_before_mma();
        // dPn = dO_I V^T one 128-key half at a time; Pn -> dS (TF32) in place
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float dp[64];
            zero(dp);
            mma_ss<kSaD / 8, 1>(dp, {smem_u32(sQ) + f.a_row(), kLbo128}, {smem_u32(sK) + h * 128 * 16, kLbo256});
#pragma unroll
            for (int x = 0; x < 64; ++x) {
                float &p = s[64 * h + x];
                p = dscore(p, dp[x], (x & 2) ? D1 : D0, scale);
            }
        }
        __syncthreads();                                                      // dO and V are dead
        stage_transposed<256>(sK, k_img, rs3, tid, kSaThreads);              // K^T (B of dQ)
        sync_before_mma();
        float dq[64];
        zero(dq);
        mma_rs<kSaL / 8>(dq, s, {smem_u32(sK), kLbo128}, false);
        store_row_pair<16>(dq_img + (size_t)i0 * rs3 + 2 * f.t, rs3, dq);
    } else {
        // ================================================================= dK, dV for key half `half`
        unsigned char *sKj = buf0, *sVj = buf1, *sQc = buf2, *sOc = buf2 + 32 * 1024;
        stage_natural<128>(sKj, k_img + (size_t)half * 128 * rs3, rs3, tid, kSaThreads);
        stage_natural<128>(sVj, v_img + (size_t)half * 128 * rs3, rs3, tid, kSaThreads);
        float dv[64], dk[64];
        zero(dv);
        zero(dk);
#pragma unroll 1
        for (int q0 = 0; q0 < kSaL; q0 += 64) {
            const float *q_c = q_img + (size_t)q0 * rs3, *do_c = do_img + (size_t)q0 * rs1;
            stage_natural<64>(sQc, q_c, rs3, tid, kSaThreads);
            stage_natural<64>(sOc, do_c, rs1, tid, kSaThreads);
            sync_before_mma();
            // S^T = K_J Q_C^T, dPn^T = V_J dO_C^T
            float st[32], dpt[32];
            zero(st);
            zero(dpt);
            mma_ss<kSaD / 8, 1>(st, {smem_u32(sKj) + f.a_row(), kLbo128}, {smem_u32(sQc), kLbo64},
                                dpt, {smem_u32(sVj) + f.a_row(), kLbo128}, {smem_u32(sOc), kLbo64});
            // thread = key row: S^T -> Pn^T, dPn^T -> dS^T, in place; query i = q0 + column
#pragma unroll
            for (int x = 0; x < 32; ++x) {
                const int i = q0 + f.col(x);
                const float p = prob(st[x], scale_log2e, s_mb[i]) * s_inv[i];
                st[x] = to_tf32(p);
                dpt[x] = dscore(p, dpt[x], s_D[i], scale);
            }
            __syncthreads();                                                  // Q_C, dO_C natural copies are dead
            stage_transposed<64>(sOc, do_c, rs1, tid, kSaThreads);            // dO_C^T (B of dV)
            stage_transposed<64>(sQc, q_c, rs3, tid, kSaThreads);             // Q_C^T (B of dK)
            sync_before_mma();
            mma_rs<8>(dv, st, {smem_u32(sOc), kLbo128}, dk, dpt, {smem_u32(sQc), kLbo128});
            __syncthreads();                                                  // before the next chunk restages
        }
        const size_t j0 = (size_t)half * 128 + row;
        float *dkp = dk_img + j0 * rs3 + 2 * f.t, *dvp = dv_img + j0 * rs3 + 2 * f.t;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            store_cols(dkp + 8 * j, dk, j, 0);
            store_cols(dkp + 8 * rs3 + 8 * j, dk, j, 1);
            store_cols(dvp + 8 * j, dv, j, 0);
            store_cols(dvp + 8 * rs3 + 8 * j, dv, j, 1);
        }
    }
}

// Shape, pointer and alignment checks of the three entry points: `ptrs` must be non-NULL and 16-byte aligned.
static int sa_check(const char *who, int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                    std::initializer_list<const void *> ptrs) {
    bool null = false;
    uintptr_t bits = 0;
    for (const void *p : ptrs) {
        null |= !p;
        bits |= (uintptr_t)p;
    }
    if (n_images < 1 || heads < 1 || heads > 16 || null) {
        set_error("%s: bad argument", who);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (tokens != kSaL || dim_head != kSaD) {
        set_error("%s: only 256 tokens x 128-dim heads are supported (got %d x %d)", who, tokens, dim_head);
        return PS_ERR_UNSUPPORTED;
    }
    if (bits & 15) {
        set_error("%s: pointers must be 16-byte aligned", who);
        return PS_ERR_INVALID_ARGUMENT;
    }
    return PS_OK;
}

static int sa_forward(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head, const float *qkv, float scale,
                      float *out, float *stats, int32_t debug_mode, void *stream) {
    const int rc = sa_check("ps_self_attention_forward", n_images, tokens, heads, dim_head, {qkv, out});
    if (rc != PS_OK) return rc;
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices))
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_self_attention_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFwdSmem));
    k_self_attention_tc<<<dim3(2, heads, n_images), kSaThreads, kFwdSmem, static_cast<cudaStream_t>(stream)>>>(
        qkv, out, stats, heads, scale * kLog2e, debug_mode);
    PS_LAUNCH_CHECK("k_self_attention_tc");
    return PS_OK;
}

}  // namespace ps

extern "C" PS_API int ps_self_attention_forward(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                                const float *qkv, float scale, float *out, int32_t debug_mode,
                                                void *stream) {
    return ps::sa_forward(n_images, tokens, heads, dim_head, qkv, scale, out, nullptr, debug_mode, stream);
}

extern "C" PS_API int ps_self_attention_forward_stats(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                                      const float *qkv, float scale, float *out, float *stats,
                                                      void *stream) {
    if (!stats) { ps::set_error("ps_self_attention_forward_stats: stats is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    return ps::sa_forward(n_images, tokens, heads, dim_head, qkv, scale, out, stats, 0, stream);
}

extern "C" PS_API int ps_self_attention_backward(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                                 const float *qkv, const float *out, const float *d_out,
                                                 const float *stats, float scale, float *d_qkv, void *stream) {
    using namespace ps;
    const int rc = sa_check("ps_self_attention_backward", n_images, tokens, heads, dim_head,
                            {qkv, out, d_out, d_qkv, stats});
    if (rc != PS_OK) return rc;
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices))
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_self_attention_tc_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBwdSmem));
    k_self_attention_tc_bwd<<<dim3(4, heads, n_images), kSaThreads, kBwdSmem, static_cast<cudaStream_t>(stream)>>>(
        qkv, out, d_out, stats, d_qkv, heads, scale, scale * kLog2e);
    PS_LAUNCH_CHECK("k_self_attention_tc_bwd");
    return PS_OK;
}
