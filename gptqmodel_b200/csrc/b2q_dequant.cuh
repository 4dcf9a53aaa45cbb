// b2q_dequant.cuh — exact (q - z) * s dequantisation of packed B2Q words for the tensor-core tiers, and the exact
// e4m3 / scale division of FP8 layers.
#pragma once
#include <cuda_fp8.h>

#include "b2q_common.cuh"

namespace b2q {

struct SZRaw {
  uint32_t s;   // scale, 16-bit payload
  uint32_t zw;  // packed zero word (or unused)
};

template <typename T, int BITS, bool ASYM>
__device__ __forceinline__ SZRaw load_sz(const T* __restrict__ scales, const uint32_t* __restrict__ qzeros, int g,
                                         int n, int N) {
  SZRaw r;
  r.s = *reinterpret_cast<const uint16_t*>(scales + (size_t)g * N + n);
  r.zw = 0;
  if (ASYM) {
    constexpr int PF = 32 / BITS;
    r.zw = qzeros[(size_t)g * (N / PF) + n / PF];
  }
  return r;
}

// exact dequant of one packed uint4 (32 k of one feature for 4-bit, 16 k for 8-bit) into K-consecutive
// 16-byte groups; out[i] holds 8 consecutive k.
template <typename T, int BITS>
struct Dequant;

// 4-bit fragment-major uint4 (see b2q_common.cuh): features (g, g+8) x 16 consecutive k.
// lo[c] / hi[c] = 8 consecutive k (chunk c = 0,1 of the lane's 16) of feature g / g+8, exactly (q - z) * s.
template <>
struct Dequant<__half, 4> {
  __device__ static __forceinline__ void run(const uint4& pv, uint32_t slo16, int zlo_i, uint32_t shi16, int zhi_i,
                                             uint4 (&lo)[2], uint4 (&hi)[2]) {
    const uint32_t slu = slo16 | (slo16 << 16), shu = shi16 | (shi16 << 16);
    const __half2 sl = *reinterpret_cast<const __half2*>(&slu), sh = *reinterpret_cast<const __half2*>(&shu);
    const __half2 zlo = __float2half2_rn(1024.f + (float)zlo_i);  // exact
    const __half2 zhi = __float2half2_rn(-(64.f + (float)zhi_i));  // exact
    const __half2 sixteenth = __float2half2_rn(0.0625f);
    const uint32_t w[4] = {pv.x, pv.y, pv.z, pv.w};
    uint32_t l[8], u[8];
#pragma unroll
    for (int s4 = 0; s4 < 4; ++s4) {
      uint32_t h[4];
      ET<__half>::unpack_w4(w[s4], h);
      __half2 v0 = __hmul2(__hsub2(*reinterpret_cast<__half2*>(&h[0]), zlo), sl);
      __half2 v1 = __hmul2(__hfma2(*reinterpret_cast<__half2*>(&h[1]), sixteenth, zhi), sh);
      __half2 v2 = __hmul2(__hsub2(*reinterpret_cast<__half2*>(&h[2]), zlo), sl);
      __half2 v3 = __hmul2(__hfma2(*reinterpret_cast<__half2*>(&h[3]), sixteenth, zhi), sh);
      l[2 * s4] = *reinterpret_cast<uint32_t*>(&v0);
      l[2 * s4 + 1] = *reinterpret_cast<uint32_t*>(&v2);
      u[2 * s4] = *reinterpret_cast<uint32_t*>(&v1);
      u[2 * s4 + 1] = *reinterpret_cast<uint32_t*>(&v3);
    }
    lo[0] = make_uint4(l[0], l[1], l[2], l[3]);
    lo[1] = make_uint4(l[4], l[5], l[6], l[7]);
    hi[0] = make_uint4(u[0], u[1], u[2], u[3]);
    hi[1] = make_uint4(u[4], u[5], u[6], u[7]);
  }
};

template <>
struct Dequant<__nv_bfloat16, 4> {
  __device__ static __forceinline__ void run(const uint4& pv, uint32_t slo16, int zlo_i, uint32_t shi16, int zhi_i,
                                             uint4 (&lo)[2], uint4 (&hi)[2]) {
    const uint32_t slu = slo16 | (slo16 << 16), shu = shi16 | (shi16 << 16);
    const __nv_bfloat162 sl = *reinterpret_cast<const __nv_bfloat162*>(&slu);
    const __nv_bfloat162 sh = *reinterpret_cast<const __nv_bfloat162*>(&shu);
    const __nv_bfloat162 zl = __float2bfloat162_rn(128.f + (float)zlo_i);  // exact (<= 143)
    const __nv_bfloat162 zh = __float2bfloat162_rn(128.f + (float)zhi_i);
    const uint32_t w[4] = {pv.x, pv.y, pv.z, pv.w};
    uint32_t l[8], u[8];
#pragma unroll
    for (int s4 = 0; s4 < 4; ++s4) {
      uint32_t h[4];
      ET<__nv_bfloat16>::unpack_w4(w[s4], h);
      __nv_bfloat162 v0 = __hmul2(__hsub2(*reinterpret_cast<__nv_bfloat162*>(&h[0]), zl), sl);
      __nv_bfloat162 v1 = __hmul2(__hsub2(*reinterpret_cast<__nv_bfloat162*>(&h[1]), zh), sh);
      __nv_bfloat162 v2 = __hmul2(__hsub2(*reinterpret_cast<__nv_bfloat162*>(&h[2]), zl), sl);
      __nv_bfloat162 v3 = __hmul2(__hsub2(*reinterpret_cast<__nv_bfloat162*>(&h[3]), zh), sh);
      l[2 * s4] = *reinterpret_cast<uint32_t*>(&v0);
      l[2 * s4 + 1] = *reinterpret_cast<uint32_t*>(&v2);
      u[2 * s4] = *reinterpret_cast<uint32_t*>(&v1);
      u[2 * s4 + 1] = *reinterpret_cast<uint32_t*>(&v3);
    }
    lo[0] = make_uint4(l[0], l[1], l[2], l[3]);
    lo[1] = make_uint4(l[4], l[5], l[6], l[7]);
    hi[0] = make_uint4(u[0], u[1], u[2], u[3]);
    hi[1] = make_uint4(u[4], u[5], u[6], u[7]);
  }
};

template <>
struct Dequant<__half, 8> {
  // 16 k per uint4 -> 2 x uint4
  __device__ static __forceinline__ void run(const uint4& pv, uint32_t s16, int z, uint4 (&o)[2]) {
    const uint32_t s2u = s16 | (s16 << 16);
    const __half2 s2 = *reinterpret_cast<const __half2*>(&s2u);
    const __half2 zb = __float2half2_rn(1024.f + (float)z);  // exact (<= 1279)
    const uint32_t w[4] = {pv.x, pv.y, pv.z, pv.w};
    uint32_t r[8];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      uint32_t p0 = __byte_perm(w[t], 0x64006400u, 0x7150);
      uint32_t p1 = __byte_perm(w[t], 0x64006400u, 0x7352);
      __half2 v0 = __hmul2(__hsub2(*reinterpret_cast<__half2*>(&p0), zb), s2);
      __half2 v1 = __hmul2(__hsub2(*reinterpret_cast<__half2*>(&p1), zb), s2);
      r[2 * t] = *reinterpret_cast<uint32_t*>(&v0);
      r[2 * t + 1] = *reinterpret_cast<uint32_t*>(&v1);
    }
    o[0] = make_uint4(r[0], r[1], r[2], r[3]);
    o[1] = make_uint4(r[4], r[5], r[6], r[7]);
  }
};

template <>
struct Dequant<__nv_bfloat16, 8> {
  __device__ static __forceinline__ void run(const uint4& pv, uint32_t s16, int z, uint4 (&o)[2]) {
    const float s = __uint_as_float(s16 << 16);
    const uint32_t w[4] = {pv.x, pv.y, pv.z, pv.w};
    uint32_t r[8];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      // (q - z) exact in fp32, product with the bf16 scale exact in fp32, ONE rounding to bf16
      const float q0 = (float)((int)(w[t] & 0xFFu) - z), q1 = (float)((int)((w[t] >> 8) & 0xFFu) - z);
      const float q2 = (float)((int)((w[t] >> 16) & 0xFFu) - z), q3 = (float)((int)(w[t] >> 24) - z);
      r[2 * t] = ET<__nv_bfloat16>::pack2(q0 * s, q1 * s);
      r[2 * t + 1] = ET<__nv_bfloat16>::pack2(q2 * s, q3 * s);
    }
    o[0] = make_uint4(r[0], r[1], r[2], r[3]);
    o[1] = make_uint4(r[4], r[5], r[6], r[7]);
  }
};

// ---- FP8 (e4m3fn) weights: W = T(w) / T(scale_inv), one correctly rounded division per weight ------------------------
// Two e4m3 codes (low byte first) -> the exact half2 of their values: every e4m3fn value, NaN included, is an fp16 value.
__device__ __forceinline__ __half2 e4m3x2_to_h2(uint32_t two_bytes) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(two_bytes & 0xFFFFu), __NV_E4M3);
  return *reinterpret_cast<const __half2*>(&h);
}

// Divisor of one quantisation group: s = float(T scale), r = RN32(1 / s).  For |s| in [2^-100, 2^100] (every fp16 value,
// and every bf16 scale a real checkpoint carries) q0 = w r, e = w - q0 s (exact), q = q0 + e r is RN32(w / s) for every
// e4m3 w (Markstein: r correctly rounded, q0 faithful).  RN_T of it is RN_T(w / s): an fp32 quotient rounded to a 16-bit
// type is not a double rounding (24 >= 2 * 11 + 2), and it is what torch computes for T(w) / T(s).  Outside that range
// (bf16 scales, and an fp16 scale that overflowed to inf) the reciprocal over- or underflows and the IEEE division is
// used instead.
struct Fp8Div {
  float s, r;
  bool fast;
};

template <typename T>
__device__ __forceinline__ Fp8Div fp8_div_of(uint32_t s16) {
  Fp8Div d;
  d.s = ET<T>::to_f(*reinterpret_cast<const T*>(&s16));
  d.r = __frcp_rn(d.s);
  const uint32_t ex = (__float_as_uint(d.s) >> 23) & 0xFFu;
  d.fast = ex >= 127u - 100u && ex <= 127u + 100u;
  return d;
}

// The remainder is formed negated (q0 s - w) so that a zero weight keeps its sign: -0 / s = -0, as torch computes it.
__device__ __forceinline__ float fp8_div_fast(float w, const Fp8Div& d) {
  const float q0 = __fmul_rn(w, d.r);
  const float en = fmaf(q0, d.s, -w);
  return fmaf(-en, d.r, q0);
}

// 16 consecutive k of one feature (one T8 uint4, natural byte order) -> 2 x uint4 of T, the same layout Dequant<T, 8>
// produces.
template <typename T>
struct DequantFp8 {
  __device__ static __forceinline__ void run(const uint4& pv, const Fp8Div& d, uint4 (&o)[2]) {
    const uint32_t w[4] = {pv.x, pv.y, pv.z, pv.w};
    float f[16];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 a = __half22float2(e4m3x2_to_h2(w[t])), b = __half22float2(e4m3x2_to_h2(w[t] >> 16));
      f[4 * t] = a.x;
      f[4 * t + 1] = a.y;
      f[4 * t + 2] = b.x;
      f[4 * t + 3] = b.y;
    }
    if (d.fast) {
#pragma unroll
      for (int i = 0; i < 16; ++i) f[i] = fp8_div_fast(f[i], d);
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) f[i] = __fdiv_rn(f[i], d.s);
    }
    uint32_t r[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) r[i] = ET<T>::pack2(f[2 * i], f[2 * i + 1]);
    o[0] = make_uint4(r[0], r[1], r[2], r[3]);
    o[1] = make_uint4(r[4], r[5], r[6], r[7]);
  }
};

}  // namespace b2q
