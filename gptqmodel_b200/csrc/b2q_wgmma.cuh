// b2q_wgmma.cuh — Hopper warpgroup MMA (wgmma.mma_async, sm_90a) wrappers for the tensor-core tiers.
//
// Both operands come from shared memory as K-major SWIZZLE_128B tiles: rows of 64 fp16/bf16 k (128 bytes), 8-row atoms
// 1024 bytes apart — the layout TMA writes for x and the dequant warps write for the weights.  One call is
// m64 x nN x k16 with fp32 accumulators in the registers of the issuing warpgroup (128 threads): thread t = 32 w + l
// holds, for column block j (8 columns), d[4j + {0,1}] = rows 16 w + l/4, columns 8 j + 2 (l % 4) + {0,1} and
// d[4j + {2,3}] = the same columns of row 16 w + l/4 + 8.
#pragma once
#include "b2q_common.cuh"

namespace b2q {

// Shared-memory matrix descriptor (PTX ISA "Matrix Descriptor Format" for wgmma): [0,14) addr>>4, [16,30) LBO>>4 (unused
// for swizzled K-major), [32,46) SBO>>4 = 1024 B between 8-row atoms, [62,64) layout (1 = SWIZZLE_128B).  Advancing by
// 16 k (32 bytes) inside the atom is +2; by 64 rows (8 atoms) +512.
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator accesses across wgmma_wait
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Wgmma<FMT, N>::mma(d, a, b, accumulate): d (+)= A[64 x 16] * B[N x 16]^T, FMT 0 = fp16, 1 = bf16 operands
template <int FMT, int N>
struct Wgmma;
template <>
struct Wgmma<0, 16> {
  __device__ static __forceinline__ void mma(float (&d)[8], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %10, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma<0, 32> {
  __device__ static __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %18, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma<0, 64> {
  __device__ static __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %34, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma<0, 128> {
  __device__ static __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %66, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma<1, 16> {
  __device__ static __forceinline__ void mma(float (&d)[8], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %10, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma<1, 32> {
  __device__ static __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %18, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma<1, 64> {
  __device__ static __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %34, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma<1, 128> {
  __device__ static __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %66, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};

// Int8 (W4A8 / QQQ) tier: Wgmma8<N>::mma(d, a, b, accumulate): d (+)= A[64 x 32] * B[N x 32]^T with s8 operands and s32
// accumulators, both operands K-major SWIZZLE_128B (one 128-byte row = 128 k).  The accumulator fragment has the fp32
// layout described at the top of this file.  Integer wgmma takes no operand negation or transpose immediates.
template <int N>
struct Wgmma8;
template <>
struct Wgmma8<8> {
  __device__ static __forceinline__ void mma(int (&d)[4], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %6, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n8k32.s32.s8.s8 {%0,%1,%2,%3}, %4, %5, p; }"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma8<16> {
  __device__ static __forceinline__ void mma(int (&d)[8], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %10, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p; }"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma8<32> {
  __device__ static __forceinline__ void mma(int (&d)[16], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %18, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p; }"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma8<64> {
  __device__ static __forceinline__ void mma(int (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %34, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p; }"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma8<128> {
  __device__ static __forceinline__ void mma(int (&d)[64], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %66, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p; }"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
// Block-FP8 (W8A8) tier: Wgmma8F<N>::mma(d, a, b, accumulate): d (+)= A[64 x 32] * B[N x 32]^T with e4m3 operands and
// fp32 accumulators, both operands K-major SWIZZLE_128B (one 128-byte row = 128 k), the fp32 fragment layout described
// at the top of this file.  8-bit floating-point wgmma takes the negation immediates but no transpose immediates.
template <int N>
struct Wgmma8F;
template <>
struct Wgmma8F<8> {
  __device__ static __forceinline__ void mma(float (&d)[4], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %6, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n8k32.f32.e4m3.e4m3 {%0,%1,%2,%3}, %4, %5, p, 1, 1; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma8F<16> {
  __device__ static __forceinline__ void mma(float (&d)[8], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %10, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n16k32.f32.e4m3.e4m3 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma8F<32> {
  __device__ static __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %18, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e4m3 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma8F<64> {
  __device__ static __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %34, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n64k32.f32.e4m3.e4m3 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <>
struct Wgmma8F<128> {
  __device__ static __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %66, 0;\n"
        "  wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1; }"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(int (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// ------------------------------------------------------------------------------------------------
// shared epilogue of the swapped-operand tiers (b2q_midm.cu, b2q_qqq.cu, b2q_fp8blk.cu): the weights are the A operand,
// so D[feature][token] is parked transposed, part[token][128 features], for the split-K reduction (dsmem_sum4)
// ------------------------------------------------------------------------------------------------
// the m64 x NTOK fragment d (NTOK / 2 registers, layout above) of feature block mb of the tile, by warp (w & 3) of its
// warpgroup, into part at shared address `part`
__device__ __forceinline__ void st_shared_4b(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void st_shared_4b(uint32_t addr, int v) {
  asm volatile("st.shared.s32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
template <int R, typename V>
__device__ __forceinline__ void park_partial(uint32_t part, int mb, int w, const V (&d)[R]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int v = 0; v < R; ++v) {
    const int j = v >> 2, h = (v >> 1) & 1, c = v & 1;
    const int feat = 64 * mb + 16 * w + (lane >> 2) + 8 * h, tok = 8 * j + 2 * (lane & 3) + c;
    st_shared_4b(part + (uint32_t)(tok * 128 + feat) * 4, d[v]);
  }
}

// Grouped launches over the experts of a MoE block (MODE 1 = gate|up, 2 = down): z0 + blockIdx.z = (expert, token block)
// over the expert-sorted rows that b2q_moe_align ordered; the rows of an expert are contiguous.
struct MoeRoute {
  const int32_t* counts;        // [E] rows of expert e
  const int32_t* offsets;       // [E] first sorted row of expert e
  const int32_t* sorted_pairs;  // [rows] pair index (token * top_k + j) of sorted row i   (MODE 2)
  const float* pair_weights;    // [rows] routing weight, indexed by pair index           (MODE 2)
  float* ypair;                 // [rows, N] fp32, row = pair index                         (MODE 2)
  int tblocks;                  // token blocks (of NTOK rows) per expert
  int z0;                       // (expert, token block) of blockIdx.z == 0 (launch_split_z)
};
// Waits for the routing tables (the output of the preceding kernels: nothing may be read before they have finished) and
// returns false for a block past its expert's rows — the same decision in every CTA of a cluster, which differ in
// blockIdx.y only.  Else e = the expert, row0 = the block's first sorted row, rows = its row count (<= NTOK).
template <int NTOK>
__device__ __forceinline__ bool moe_block(const MoeRoute& R, int& e, int& row0, int& rows) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int z = R.z0 + (int)blockIdx.z;
  e = z / R.tblocks;
  const int tb = z - e * R.tblocks, cnt = R.counts[e];
  if (tb * NTOK >= cnt) return false;
  row0 = R.offsets[e] + tb * NTOK;
  rows = min(NTOK, cnt - tb * NTOK);
  return true;
}

// four consecutive outputs: T(acc), or T(T(acc) + bias) in the reference order (round the matmul to the output dtype,
// then add bias: torch.py:337-342) of features nc .. nc + 3; bias = [N] or nullptr
template <typename T>
__device__ __forceinline__ void store_out4(T* dst, const T* bias, int nc, float (&a)[4]) {
  using E = ET<T>;
  if (bias != nullptr) {
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = E::to_f(E::from_f(a[i])) + E::to_f(bias[nc + i]);
  }
  *reinterpret_cast<uint2*>(dst) = make_uint2(E::pack2(a[0], a[1]), E::pack2(a[2], a[3]));
}
// MODE 1: the per-expert module loop of the reference model rounds at every module boundary (act_fn(w1(x)) * w3(x) with
// 16-bit tensors): g = T(x W1), a = T(silu(g)), u = T(x W3), h = T(a * u)
template <typename T>
__device__ __forceinline__ void store_silu_mul4(T* dst, const float (&g)[4], const float (&u)[4]) {
  using E = ET<T>;
  float h[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float gq = E::to_f(E::from_f(g[i])), uq = E::to_f(E::from_f(u[i]));
    const float aq = E::to_f(E::from_f(gq / (1.f + __expf(-gq))));
    h[i] = aq * uq;
  }
  *reinterpret_cast<uint2*>(dst) = make_uint2(E::pack2(h[0], h[1]), E::pack2(h[2], h[3]));
}
// MODE 2: y = T(h W2) like the module, times the routing weight, kept in fp32 in the pair's row of ypair — the top_k rows
// of a token are summed (and rounded ONCE) by moe_combine_kernel: no atomics, deterministic
template <typename T>
__device__ __forceinline__ void store_ypair4(float* dst, float w, const float (&a)[4]) {
  using E = ET<T>;
  *reinterpret_cast<float4*>(dst) = make_float4(w * E::to_f(E::from_f(a[0])), w * E::to_f(E::from_f(a[1])),
                                                w * E::to_f(E::from_f(a[2])), w * E::to_f(E::from_f(a[3])));
}

}  // namespace b2q
