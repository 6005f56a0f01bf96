// TF32 wgmma (Hopper warpgroup MMA) layer of the attention kernels (self_attention_tc.cu, vit_attention.cu):
// operands in the canonical K-major no-swizzle shared-memory layout, FP32 accumulators in registers, CTAs of two
// warpgroups.
#pragma once
#include "ps_common.cuh"

namespace ps {

constexpr float kLog2e = 1.4426950408889634f;

// fp32 -> nearest TF32 (ties away), kept in an fp32 container: the tensor core ignores the low 13
// mantissa bits, so rounding here instead of letting it truncate halves the operand error and removes its bias.
__device__ __forceinline__ float to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
__device__ __forceinline__ float4 to_tf32(float4 v) { return make_float4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w)); }

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Shared-memory matrix descriptor, K-major, no swizzle: core matrix = 8 rows x 16 bytes (contiguous 128 B);
// 8-row groups are adjacent (SBO = 128 B), 16-byte K chunks are `lbo` bytes apart.  One k8 step of TF32 reads
// two chunks, so step k starts 2 k lbo bytes further on.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3fffu);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32;
    return d;                                // base offset 0, layout type 0 (no swizzle)
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// After wgmma_wait_all: keeps the compiler from moving reads of the accumulators above the wait.
template <int N>
__device__ __forceinline__ void fence_operands(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}

// m64nNk8, D (+)= A B^T with D = F32, A = B = TF32 K-major.  Accumulator fragment of thread (warp w of the
// warpgroup, lane = 4 g + t): d[4 j + 0 / 1] = row 16 w + g, columns 8 j + 2 t / 8 j + 2 t + 1; d[4 j + 2 / 3] =
// the same columns of row 16 w + g + 8.  _ss: A and B from shared memory; _rs: A from registers.
__device__ __forceinline__ void wgmma_ss_n256(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127 "
        "}, %128, %129, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}

__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63 "
        "}, %64, %65, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}

__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31 "
        "}, %32, %33, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}

__device__ __forceinline__ void wgmma_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63 "
        "}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
        : "memory");
}

__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31 "
        "}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
        : "memory");
}

// A fragment (rows 16 w + g / + 8, k = t / t + 4) of an _rs MMA taken straight from accumulator columns
// 8 kk .. 8 kk + 7 of an earlier MMA: the thread holds columns 2 t and 2 t + 1 there, so k index t stands for
// column 8 kk + 2 t and k index t + 4 for column 8 kk + 2 t + 1.  B's K dimension must be staged in that same
// order, which stage_transposed does.
template <int N>
__device__ __forceinline__ void acc_to_a(const float (&d)[N], int kk, uint32_t (&a)[4]) {
    a[0] = __float_as_uint(d[4 * kk]);
    a[1] = __float_as_uint(d[4 * kk + 2]);
    a[2] = __float_as_uint(d[4 * kk + 1]);
    a[3] = __float_as_uint(d[4 * kk + 3]);
}

// Makes the CTA's generic-proxy shared-memory stores visible to the wgmma operand reads that follow.
__device__ __forceinline__ void sync_before_mma() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
}

template <int N>
__device__ __forceinline__ void zero(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) d[i] = 0.0f;
}

// This thread's place in the accumulator fragments of a 256-thread CTA: warpgroup wg owns MMA rows
// 64 wg .. 64 wg + 63, and the thread holds rows `row` and `row + 8`, element x of an accumulator at column col(x).
struct Frag {
    int wg, t, row;
    __device__ __forceinline__ Frag() {
        const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
        wg = warp >> 2;
        t = lane & 3;
        row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    }
    __device__ __forceinline__ int col(int x) const { return 8 * (x >> 2) + 2 * t + (x & 1); }
    __device__ __forceinline__ uint32_t a_row() const { return (uint32_t)wg * 64 * 16; }  // its rows in an A tile
};

// A K-major no-swizzle operand tile in shared memory: `lbo` bytes between its 16-byte K chunks.
struct SmemTile {
    uint32_t addr, lbo;
    __device__ __forceinline__ uint64_t desc(int k) const { return gmma_desc(addr + k * 2 * lbo, lbo, 128); }
};

// One k8 step, the instruction picked by the accumulator width (N registers = N / 2 columns).
template <int N>
__device__ __forceinline__ void wgmma_ss(float (&d)[N], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    static_assert(N == 32 || N == 64 || N == 128, "accumulator width");
    if constexpr (N == 32) wgmma_ss_n64(d, a_desc, b_desc, accumulate);
    else if constexpr (N == 64) wgmma_ss_n128(d, a_desc, b_desc, accumulate);
    else wgmma_ss_n256(d, a_desc, b_desc, accumulate);
}
template <int N>
__device__ __forceinline__ void wgmma_rs(float (&d)[N], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
    static_assert(N == 32 || N == 64, "accumulator width");
    if constexpr (N == 32) wgmma_rs_n64(d, a, b_desc, accumulate);
    else wgmma_rs_n128(d, a, b_desc, accumulate);
}

// D = A B^T over K k8 steps (the first step overwrites D), A and B from shared memory; returns once D is in
// registers; UNROLL unrolls the k loop.  The two-accumulator form issues both products step by step in one commit
// group.
template <int K, int UNROLL, int N>
__device__ __forceinline__ void mma_ss(float (&d)[N], SmemTile a, SmemTile b) {
    wgmma_fence();
#pragma unroll UNROLL
    for (int k = 0; k < K; ++k) wgmma_ss(d, a.desc(k), b.desc(k), k > 0);
    wgmma_commit();
    wgmma_wait_all();
    fence_operands(d);
}
template <int K, int UNROLL, int N>
__device__ __forceinline__ void mma_ss(float (&d0)[N], SmemTile a0, SmemTile b0, float (&d1)[N], SmemTile a1, SmemTile b1) {
    wgmma_fence();
#pragma unroll UNROLL
    for (int k = 0; k < K; ++k) {
        wgmma_ss(d0, a0.desc(k), b0.desc(k), k > 0);
        wgmma_ss(d1, a1.desc(k), b1.desc(k), k > 0);
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_operands(d0);
    fence_operands(d1);
}

// D (+)= P B^T over K k8 steps with A = P straight from an earlier accumulator (acc_to_a's order); the first step
// overwrites D unless `accumulate`.  The two-accumulator form accumulates into both, D0's steps then D1's, in one
// commit group.
template <int K, int N, int M>
__device__ __forceinline__ void mma_rs(float (&d)[N], const float (&p)[M], SmemTile b, bool accumulate) {
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < K; ++kk) {
        uint32_t a[4];
        acc_to_a(p, kk, a);
        wgmma_rs(d, a, b.desc(kk), accumulate || kk > 0);
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_operands(d);
}
template <int K, int N, int M>
__device__ __forceinline__ void mma_rs(float (&d0)[N], const float (&p0)[M], SmemTile b0, float (&d1)[N],
                                       const float (&p1)[M], SmemTile b1) {
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < K; ++kk) {
        uint32_t a[4];
        acc_to_a(p0, kk, a);
        wgmma_rs(d0, a, b0.desc(kk), 1);
    }
#pragma unroll
    for (int kk = 0; kk < K; ++kk) {
        uint32_t a[4];
        acc_to_a(p1, kk, a);
        wgmma_rs(d1, a, b1.desc(kk), 1);
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_operands(d0);
    fence_operands(d1);
}

// Epilogue: columns 8 j + 2 t and 8 j + 2 t + 1 of row `row + 8 h` of accumulator d, times f, as one float2 at dst.
template <int N>
__device__ __forceinline__ void store_cols(float *dst, const float (&d)[N], int j, int h, float f = 1.0f) {
    *reinterpret_cast<float2 *>(dst) = make_float2(d[4 * j + 2 * h] * f, d[4 * j + 2 * h + 1] * f);
}

// Columns [0, 8 J) of both rows: `row` times f0 at dst, `row + 8` times f1 at dst + 8 stride.
template <int J, int N>
__device__ __forceinline__ void store_row_pair(float *dst, size_t stride, const float (&d)[N], float f0 = 1.0f,
                                               float f1 = 1.0f) {
#pragma unroll
    for (int j = 0; j < J; ++j) {
        store_cols(dst + 8 * j, d, j, 0, f0);
        store_cols(dst + 8 * stride + 8 * j, d, j, 1, f1);
    }
}

// ---- staging of fp32 global tiles into the K-major no-swizzle layout (rounded to the nearest TF32) ---------
// natural: tile rows = MMA rows (M or N), the 128 channels are the K dimension.  Consecutive threads take
// consecutive rows of the same 16-byte chunk, so the shared stores are contiguous (chunk c of row r lives at
// c * LBO + r * 16, LBO = ROWS * 16); eight independent 16-byte loads are in flight per thread.
template <int ROWS>
__device__ __forceinline__ void stage_natural(unsigned char *dst, const float *__restrict__ src, size_t row_stride,
                                              int tid, int nthreads) {
    constexpr int kBatch = 8;
    constexpr int kShift = ROWS == 256 ? 8 : ROWS == 128 ? 7 : 6;
    static_assert(ROWS == 64 || ROWS == 128 || ROWS == 256, "tile rows");
#pragma unroll 1
    for (int i0 = tid; i0 < ROWS * 32; i0 += nthreads * kBatch) {
        float4 v[kBatch];
#pragma unroll
        for (int j = 0; j < kBatch; ++j) {
            const int i = i0 + j * nthreads;
            v[j] = (i < ROWS * 32) ? __ldg(reinterpret_cast<const float4 *>(src + (size_t)(i & (ROWS - 1)) * row_stride) + (i >> kShift))
                                   : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        }
#pragma unroll
        for (int j = 0; j < kBatch; ++j) {
            const int i = i0 + j * nthreads;
            if (i < ROWS * 32)
                *reinterpret_cast<float4 *>(dst + (size_t)(i >> kShift) * (ROWS * 16) + (i & (ROWS - 1)) * 16) = to_tf32(v[j]);
        }
    }
}

// transposed: MMA rows (N) = the 128 channels, K dimension = TOKENS tokens in acc_to_a's order: the two 16-byte
// chunks of k step kk hold tokens 8 kk + {0, 2, 4, 6} and 8 kk + {1, 3, 5, 7} of one channel (LBO = 128 * 16);
// 16 scalar loads in flight per thread.
template <int TOKENS>
__device__ __forceinline__ void stage_transposed(unsigned char *dst, const float *__restrict__ src, size_t row_stride,
                                                 int tid, int nthreads) {
#pragma unroll 1
    for (int i0 = tid; i0 < 128 * (TOKENS / 4); i0 += nthreads * 4) {
        float4 v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int i = i0 + j * nthreads;
            v[j] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            if (i < 128 * (TOKENS / 4)) {
                const int c = i >> 7;
                const float *p = src + (size_t)(8 * (c >> 1) + (c & 1)) * row_stride + (i & 127);
                v[j].x = __ldg(p);
                v[j].y = __ldg(p + 2 * row_stride);
                v[j].z = __ldg(p + 4 * row_stride);
                v[j].w = __ldg(p + 6 * row_stride);
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int i = i0 + j * nthreads;
            if (i < 128 * (TOKENS / 4))
                *reinterpret_cast<float4 *>(dst + (size_t)(i >> 7) * (128 * 16) + (i & 127) * 16) = to_tf32(v[j]);
        }
    }
}

}  // namespace ps
