// Dense per-image multi-head self-attention on the Hopper tensor cores (wgmma, TF32):
//     out[img, :, head] = softmax(Q K^T * scale) V      Q, K, V: [256 tokens, 128] per (image, head)
// for the ViT blocks of pixelSplat's ImageSelfAttention (reference: src/model/encoder/epipolar/
// image_self_attention.py:57-79 -> src/model/transformer/attention.py:54-70 with z = None): the only dense
// contractions of the hot path (SURVEY.md 8 row a14).
//
// One CTA (two warpgroups) per (image, head, 128-query half); warpgroup w owns queries 64 w .. 64 w + 63:
//   1. Q half [128 x 128] and K [256 x 128] are copied (fp32 rounded to the nearest TF32) into shared
//      memory in the canonical K-major no-swizzle layout (8-row x 16-byte core matrices);
//   2. each warpgroup issues 16 wgmma m64n256k8 accumulating its S = Q K^T rows in registers (128 per thread);
//   3. K's shared buffer is overwritten with V^T (d-major x tokens, same K-major layout); each thread turns
//      its two rows' S into un-normalised probabilities in place (row max and sum over the four threads that
//      share a row), rounded to TF32;
//   4. 32 wgmma m64n128k8 with A = P straight from those registers and B = V^T from shared memory accumulate O;
//   5. epilogue: scale by 1 / row sum, store.
// No TMA: the tiles are tiny and L2-resident; the copy is plain ld.global / st.shared followed by a proxy fence.
#include "wgmma_tf32.cuh"

namespace ps {

// debug_mode: 0 = attention output; 1 = write the raw logits S = Q K^T instead (`out` is then
// [n_img, H, 256, 256]) -- used by the tests to isolate the first MMA stage.
__global__ void __launch_bounds__(kSaThreads, 1)
k_self_attention_tc(const float *__restrict__ qkv, float *__restrict__ out, float *__restrict__ stats, int n_heads,
                    float scale_log2e, int debug_mode) {
    extern __shared__ __align__(128) unsigned char s_sa[];
    unsigned char *sQ = s_sa;                                                      // 128 x 128 fp32 = 64 KB
    unsigned char *sK = s_sa + 64 * 1024;                                          // 256 x 128 fp32 = 128 KB (later V^T)
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int t = lane & 3;
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);                       // first of this thread's rows (+8)
    const int half = blockIdx.x, head = blockIdx.y, img = blockIdx.z;
    const int inner = n_heads * kSaD;
    const size_t row_stride = 3 * (size_t)inner;                                   // floats per token in qkv
    const float *q_base = qkv + ((size_t)img * kSaL + (size_t)half * 128) * row_stride + (size_t)head * kSaD;
    const float *k_base = qkv + (size_t)img * kSaL * row_stride + inner + (size_t)head * kSaD;
    const float *v_base = qkv + (size_t)img * kSaL * row_stride + 2 * inner + (size_t)head * kSaD;
    constexpr uint32_t kLboQ = 128 * 16, kLboK = 256 * 16, kLboV = 128 * 16;       // bytes between K chunks

    stage_natural<128>(sQ, q_base, row_stride, tid, kSaThreads);
    stage_natural<256>(sK, k_base, row_stride, tid, kSaThreads);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");                  // generic -> async proxy
    __syncthreads();

    // ---- S = Q K^T, this warpgroup's 64 rows
    float s[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) s[i] = 0.0f;
    wgmma_fence();
#pragma unroll 1
    for (int k = 0; k < kSaD / 8; ++k)
        wgmma_ss_n256(s, gmma_desc(smem_u32(sQ) + k * 2 * kLboQ + wg * 64 * 16, kLboQ, 128),
                      gmma_desc(smem_u32(sK) + k * 2 * kLboK, kLboK, 128), k > 0);
    wgmma_commit();
    wgmma_wait_all();
    fence_operands(s);
    if (debug_mode == 1) {
        float *dst = out + ((((size_t)img * n_heads + head) * 2 + half) * 128 + row) * 256 + 2 * t;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            *reinterpret_cast<float2 *>(dst + 8 * j) = make_float2(s[4 * j], s[4 * j + 1]);
            *reinterpret_cast<float2 *>(dst + 8 * 256 + 8 * j) = make_float2(s[4 * j + 2], s[4 * j + 3]);
        }
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
        s[4 * j] = to_tf32(exp2f(s[4 * j] * scale_log2e - mb0));          // the row sum is over what the MMA will see
        s[4 * j + 1] = to_tf32(exp2f(s[4 * j + 1] * scale_log2e - mb0));
        s[4 * j + 2] = to_tf32(exp2f(s[4 * j + 2] * scale_log2e - mb1));
        s[4 * j + 3] = to_tf32(exp2f(s[4 * j + 3] * scale_log2e - mb1));
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
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    // ---- O = P V   (A = P from registers, B = V^T from shared memory)
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.0f;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kSaL / 8; ++kk) {
        uint32_t a[4];
        acc_to_a(s, kk, a);
        wgmma_rs_n128(o, a, gmma_desc(smem_u32(sK) + kk * 2 * kLboV, kLboV, 128), kk > 0);
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_operands(o);
    // ---- epilogue
    float *dst = out + ((size_t)img * kSaL + (size_t)half * 128 + row) * inner + (size_t)head * kSaD + 2 * t;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        *reinterpret_cast<float2 *>(dst + 8 * j) = make_float2(o[4 * j] * inv0, o[4 * j + 1] * inv0);
        *reinterpret_cast<float2 *>(dst + 8 * (size_t)inner + 8 * j) = make_float2(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1);
    }
}

}  // namespace ps

static int self_attention_forward_impl(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                       const float *qkv, float scale, float *out, float *stats, int32_t debug_mode,
                                       void *stream) {
    using namespace ps;
    if (n_images < 1 || heads < 1 || heads > 16 || !qkv || !out) {
        set_error("ps_self_attention_forward: bad argument");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (tokens != kSaL || dim_head != kSaD) {
        set_error("ps_self_attention_forward: only 256 tokens x 128-dim heads are supported (got %d x %d)", tokens, dim_head);
        return PS_ERR_UNSUPPORTED;
    }
    if (((uintptr_t)qkv | (uintptr_t)out) & 15) { set_error("ps_self_attention_forward: pointers must be 16-byte aligned"); return PS_ERR_INVALID_ARGUMENT; }
    const size_t smem = 192 * 1024;
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_self_attention_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    dim3 grid(2, heads, n_images);
    k_self_attention_tc<<<grid, kSaThreads, smem, static_cast<cudaStream_t>(stream)>>>(
        qkv, out, stats, heads, scale * 1.4426950408889634f, debug_mode);
    PS_LAUNCH_CHECK("k_self_attention_tc");
    return PS_OK;
}

extern "C" PS_API int ps_self_attention_forward(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                                const float *qkv, float scale, float *out, int32_t debug_mode,
                                                void *stream) {
    return self_attention_forward_impl(n_images, tokens, heads, dim_head, qkv, scale, out, nullptr, debug_mode, stream);
}

extern "C" PS_API int ps_self_attention_forward_stats(int32_t n_images, int32_t tokens, int32_t heads, int32_t dim_head,
                                                      const float *qkv, float scale, float *out, float *stats,
                                                      void *stream) {
    if (!stats) { ps::set_error("ps_self_attention_forward_stats: stats is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    return self_attention_forward_impl(n_images, tokens, heads, dim_head, qkv, scale, out, stats, 0, stream);
}
