// Backward of the dense per-image self-attention (self_attention_tc.cu) on the same wgmma path: autograd of
// softmax(Q K^T * scale) V for the ViT blocks of ImageSelfAttention (reference: src/model/encoder/epipolar/
// image_self_attention.py:57-79 -> src/model/transformer/attention.py:54-70 with z = None; SURVEY.md 8 row a14).
//
// Per (image, head), with Pn the forward's probabilities -- rebuilt from the saved per-row (max, 1 / sum) with
// the same TF32 roundings, so the backward differentiates the forward that actually ran:
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
#include "wgmma_tf32.cuh"

namespace ps {

namespace {

constexpr uint32_t kLbo64 = 64 * 16;     // bytes between 16-byte K chunks of a 64-row tile
constexpr uint32_t kLbo128 = 128 * 16;
constexpr uint32_t kLbo256 = 256 * 16;

__device__ __forceinline__ void sync_before_mma() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic -> async proxy (smem operands)
    __syncthreads();
}

template <int N>
__device__ __forceinline__ void zero(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) d[i] = 0.0f;
}

}  // namespace

__global__ void __launch_bounds__(kSaThreads, 1)
k_self_attention_tc_bwd(const float *__restrict__ qkv, const float *__restrict__ out, const float *__restrict__ d_out,
                        const float *__restrict__ stats, float *__restrict__ d_qkv, int n_heads, float scale,
                        float scale_log2e) {
    extern __shared__ __align__(128) unsigned char s_sa[];
    unsigned char *buf0 = s_sa, *buf1 = s_sa + 64 * 1024, *buf2 = s_sa + 128 * 1024;
    float *s_mb = reinterpret_cast<float *>(s_sa + 192 * 1024);          // [256] row max * scale * log2 e
    float *s_inv = s_mb + 256;                                            // [256] 1 / row sum
    float *s_D = s_inv + 256;                                             // [256] dO_i . O_i
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int t = lane & 3;
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);              // first of this thread's rows (+8)
    const int role = blockIdx.x >> 1, half = blockIdx.x & 1, head = blockIdx.y, img = blockIdx.z;
    const int inner = n_heads * kSaD;
    const size_t rs3 = 3 * (size_t)inner, rs1 = (size_t)inner;            // floats per token in qkv / out
    const float *q_img = qkv + (size_t)img * kSaL * rs3 + (size_t)head * kSaD;
    const float *k_img = q_img + inner, *v_img = q_img + 2 * inner;
    const float *o_img = out + (size_t)img * kSaL * rs1 + (size_t)head * kSaD;
    const float *do_img = d_out + (size_t)img * kSaL * rs1 + (size_t)head * kSaD;
    float *dq_img = d_qkv + (size_t)img * kSaL * rs3 + (size_t)head * kSaD;
    float *dk_img = dq_img + inner, *dv_img = dq_img + 2 * inner;
    const uint32_t a_row = (uint32_t)wg * 64 * 16;                          // this warpgroup's rows in an A tile

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
        wgmma_fence();
#pragma unroll 1
        for (int k = 0; k < kSaD / 8; ++k)
            wgmma_ss_n256(s, gmma_desc(smem_u32(sQ) + k * 2 * kLbo128 + a_row, kLbo128, 128),
                          gmma_desc(smem_u32(sK) + k * 2 * kLbo256, kLbo256, 128), k > 0);
        wgmma_commit();
        wgmma_wait_all();
        fence_operands(s);
        // S -> Pn in place (rows i0 = s[4 j + 0 / 1], i0 + 8 = s[4 j + 2 / 3])
        const int i0 = half * 128 + row;
        const float mb0 = s_mb[i0], inv0 = s_inv[i0], D0 = s_D[i0];
        const float mb1 = s_mb[i0 + 8], inv1 = s_inv[i0 + 8], D1 = s_D[i0 + 8];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            s[4 * j] = to_tf32(exp2f(s[4 * j] * scale_log2e - mb0)) * inv0;
            s[4 * j + 1] = to_tf32(exp2f(s[4 * j + 1] * scale_log2e - mb0)) * inv0;
            s[4 * j + 2] = to_tf32(exp2f(s[4 * j + 2] * scale_log2e - mb1)) * inv1;
            s[4 * j + 3] = to_tf32(exp2f(s[4 * j + 3] * scale_log2e - mb1)) * inv1;
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
            wgmma_fence();
#pragma unroll 1
            for (int k = 0; k < kSaD / 8; ++k)
                wgmma_ss_n128(dp, gmma_desc(smem_u32(sQ) + k * 2 * kLbo128 + a_row, kLbo128, 128),
                              gmma_desc(smem_u32(sK) + k * 2 * kLbo256 + h * 128 * 16, kLbo256, 128), k > 0);
            wgmma_commit();
            wgmma_wait_all();
            fence_operands(dp);
#pragma unroll
            for (int x = 0; x < 64; ++x) {
                float &p = s[64 * h + x];
                p = to_tf32(p * (dp[x] - ((x & 2) ? D1 : D0)) * scale);
            }
        }
        __syncthreads();                                                      // dO and V are dead
        stage_transposed<256>(sK, k_img, rs3, tid, kSaThreads);              // K^T (B of dQ)
        sync_before_mma();
        float dq[64];
        zero(dq);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kSaL / 8; ++kk) {
            uint32_t a[4];
            acc_to_a(s, kk, a);
            wgmma_rs_n128(dq, a, gmma_desc(smem_u32(sK) + kk * 2 * kLbo128, kLbo128, 128), kk > 0);
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_operands(dq);
        float *dst = dq_img + (size_t)i0 * rs3 + 2 * t;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            *reinterpret_cast<float2 *>(dst + 8 * j) = make_float2(dq[4 * j], dq[4 * j + 1]);
            *reinterpret_cast<float2 *>(dst + 8 * rs3 + 8 * j) = make_float2(dq[4 * j + 2], dq[4 * j + 3]);
        }
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
            wgmma_fence();
#pragma unroll 1
            for (int k = 0; k < kSaD / 8; ++k) {
                wgmma_ss_n64(st, gmma_desc(smem_u32(sKj) + k * 2 * kLbo128 + a_row, kLbo128, 128),
                             gmma_desc(smem_u32(sQc) + k * 2 * kLbo64, kLbo64, 128), k > 0);
                wgmma_ss_n64(dpt, gmma_desc(smem_u32(sVj) + k * 2 * kLbo128 + a_row, kLbo128, 128),
                             gmma_desc(smem_u32(sOc) + k * 2 * kLbo64, kLbo64, 128), k > 0);
            }
            wgmma_commit();
            wgmma_wait_all();
            fence_operands(st);
            fence_operands(dpt);
            // thread = key row: S^T -> Pn^T, dPn^T -> dS^T, in place; query i = column 8 j + 2 t (+1)
#pragma unroll
            for (int x = 0; x < 32; ++x) {
                const int i = q0 + 8 * (x >> 2) + 2 * t + (x & 1);
                const float p = to_tf32(exp2f(st[x] * scale_log2e - s_mb[i])) * s_inv[i];
                st[x] = to_tf32(p);
                dpt[x] = to_tf32(p * (dpt[x] - s_D[i]) * scale);
            }
            __syncthreads();                                                  // Q_C, dO_C natural copies are dead
            stage_transposed<64>(sOc, do_c, rs1, tid, kSaThreads);            // dO_C^T (B of dV)
            stage_transposed<64>(sQc, q_c, rs3, tid, kSaThreads);             // Q_C^T (B of dK)
            sync_before_mma();
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                uint32_t a[4];
                acc_to_a(st, kk, a);
                wgmma_rs_n128(dv, a, gmma_desc(smem_u32(sOc) + kk * 2 * kLbo128, kLbo128, 128), 1);
            }
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                uint32_t a[4];
                acc_to_a(dpt, kk, a);
                wgmma_rs_n128(dk, a, gmma_desc(smem_u32(sQc) + kk * 2 * kLbo128, kLbo128, 128), 1);
            }
            wgmma_commit();
            wgmma_wait_all();
            fence_operands(dv);
            fence_operands(dk);
            __syncthreads();                                                  // before the next chunk restages
        }
        const size_t j0 = (size_t)half * 128 + row;
        float *dkp = dk_img + j0 * rs3 + 2 * t, *dvp = dv_img + j0 * rs3 + 2 * t;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            *reinterpret_cast<float2 *>(dkp + 8 * j) = make_float2(dk[4 * j], dk[4 * j + 1]);
            *reinterpret_cast<float2 *>(dkp + 8 * rs3 + 8 * j) = make_float2(dk[4 * j + 2], dk[4 * j + 3]);
            *reinterpret_cast<float2 *>(dvp + 8 * j) = make_float2(dv[4 * j], dv[4 * j + 1]);
            *reinterpret_cast<float2 *>(dvp + 8 * rs3 + 8 * j) = make_float2(dv[4 * j + 2], dv[4 * j + 3]);
        }
    }
}

}  // namespace ps

extern "C" PS_API int ps_self_attention_backward(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                                 const float *qkv, const float *out, const float *d_out,
                                                 const float *stats, float scale, float *d_qkv, void *stream) {
    using namespace ps;
    if (n_images < 1 || heads < 1 || heads > 16 || !qkv || !out || !d_out || !stats || !d_qkv) {
        set_error("ps_self_attention_backward: bad argument");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (tokens != kSaL || dim_head != kSaD) {
        set_error("ps_self_attention_backward: only 256 tokens x 128-dim heads are supported (got %d x %d)", tokens, dim_head);
        return PS_ERR_UNSUPPORTED;
    }
    if (((uintptr_t)qkv | (uintptr_t)out | (uintptr_t)d_out | (uintptr_t)d_qkv | (uintptr_t)stats) & 15) {
        set_error("ps_self_attention_backward: pointers must be 16-byte aligned");
        return PS_ERR_INVALID_ARGUMENT;
    }
    const size_t smem = 192 * 1024 + 3 * 256 * sizeof(float);
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_self_attention_tc_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    dim3 grid(4, heads, n_images);
    k_self_attention_tc_bwd<<<grid, kSaThreads, smem, static_cast<cudaStream_t>(stream)>>>(
        qkv, out, d_out, stats, d_qkv, heads, scale, scale * 1.4426950408889634f);
    PS_LAUNCH_CHECK("k_self_attention_tc_bwd");
    return PS_OK;
}
