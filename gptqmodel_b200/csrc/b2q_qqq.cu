// b2q_qqq.cu — QQQ (W4A8) tier: per-token int8 activations times 4-bit weights on the int8 tensor cores.
//
// out[M, N] = fp16( fp32(acc) * s_channel[n] * s_tok[m] ) (+ bias, rounded again), acc = sum_k q[m, k] * w[k, n] in int32
// (exact for K <= 65536), the serving arithmetic of the reference's QQQLinear.forward + qqq_gemm.  Two kernels:
//   * qqq_quant_kernel: one CTA per token row.  A = fp16(x); s_tok = fp32(fp16(max|A| / 127)); q = clamp(rint(A / s_tok))
//     with IEEE fp32 division, written as int8 [M, Kp] (Kp = K rounded up to 128, padding codes 0).
//   * qqq_gemm_kernel: the structure of b2q_midm.cu with int8 operands.  The WEIGHTS are the wgmma A operand (128 output
//     features = two m64 blocks), the TOKENS the B operand (n = NTOK in {8, 16, 32, 64, 128}).  A k-block is 128 k, one
//     SWIZZLE_128B row of int8.  Warp 8 loads the activation codes with TMA; warps 4..7 expand the packed codes of the
//     block (one feature row per thread) into int8 rows; warps 0..3 issue m64nNk32.s32.s8.s8 into int32 registers.  The
//     `ks` CTAs of a cluster split the k-blocks of a tile and reduce their integer partials over distributed shared
//     memory, so any split gives the same bits; token blocks of NTOK rows are spread over gridDim.z.  No atomics.
//   * qqq_moe_gemm_kernel: grouped modes of the same GEMM body for MoE experts (MODE 1 / 2) over the expert-sorted rows
//     of b2q_moe_align, the weights the stacks of all experts.  MODE 1 pairs 64 gate features (w1, m64 block 0) with
//     the same 64 up features (w3, m64 block 1) in one 128-row tile and stores h = T(T(silu(g)) * u); MODE 2 (down)
//     stores w[pair] * T(y) in fp32 to the pair's row of ypair.
//   * qqq_moe_gather_kernel: the quantiser over the sorted rows, row i quantising token sorted_pairs[i] / top_k.
//
// Packed weights (b2q_qqq_prepack): tile (nt, kb) of 128 features x 128 k is 8 KB at ((nt * KB + kb) * 8192), laid out
// uint4 [4 quads][128 features]: quad q of feature f holds k = 32 q .. 32 q + 31 as four 32-bit words of eight nibbles.
// Inside a word covering k0 .. k0 + 7 the nibble order depends on the layer kind, so that dequantisation needs no shuffle:
//   per-channel: nibbles 1, 3, 5, 7 = k0..3 and 0, 2, 4, 6 = k4..7: (w & 0xF0F0F0F0) and ((w << 4) & 0xF0F0F0F0) are the
//                int8 weights (signed code * 16) of k0..3 and k4..7;
//   group 128  : nibbles 0, 1, 4, 5 = k0..3 and 2, 3, 6, 7 = k4..7: half2 lanes (code - 8) * s + 1280 with ONE fp16
//                rounding (ulp 1 in [1024, 2048)) carry round_half_even((code - 8) * s) in their low byte, and one byte
//                permute per four weights gathers them in k order.
#include <cuda.h>

#include "b2q_common.cuh"
#include "b2q_internal.h"
#include "b2q_wgmma.cuh"

namespace b2q {

constexpr int Q_BF = 128;                // features per tile
constexpr int Q_BK = 128;                // k per block (one SWIZZLE_128B row of int8)
constexpr int Q_TILE_BYTES = Q_BF * Q_BK / 2;
constexpr int Q_MMA_THREADS = 128;       // warps 0..3
constexpr int Q_DQ_THREADS = 128;        // warps 4..7: thread t expands feature row t
constexpr int Q_THREADS = Q_MMA_THREADS + Q_DQ_THREADS + 32;  // + warp 8: activation producer
constexpr int Q_RED_WARPS = 8;
constexpr int Q_QUANT_THREADS = 512;  // one CTA per token row: a decode row of 14336 is one 16-byte load per thread

template <int NTOK>
struct QqqCfg {
  static constexpr int PST = 8;                       // packed stages (8 KB): the HBM stream in flight
  static constexpr int WST = 4;                       // expanded int8 stages (16 KB)
  static constexpr int XST = 4;                       // activation stages
  static constexpr int W_BYTES = Q_BF * Q_BK;
  static constexpr int X_BYTES = NTOK * Q_BK;
  static constexpr int BAR_BYTES = 256;
  static constexpr int RING_BYTES = WST * W_BYTES + XST * X_BYTES + PST * Q_TILE_BYTES;
  static constexpr int SMEM_BYTES = RING_BYTES + BAR_BYTES + 1024;
  static constexpr int ACC = NTOK / 2;
  static_assert(X_BYTES % 1024 == 0, "activation tiles must stay 1024-byte aligned (SWIZZLE_128B atoms)");
  static_assert(NTOK * Q_BF * 4 <= WST * W_BYTES, "the int32 partial tile reuses the expanded-weight stages");
  static_assert((PST + 2 * XST + 2 * WST) * 8 <= BAR_BYTES, "mbarrier area");
  static_assert(SMEM_BYTES <= 227 * 1024, "dynamic shared memory of one CTA");
};

// ------------------------------------------------------------------------------------------------
// activation quantiser
// ------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float to_half_f(T v);
template <>
__device__ __forceinline__ float to_half_f<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_half_f<__nv_bfloat16>(__nv_bfloat16 v) {
  return __half2float(__float2half_rn(__bfloat162float(v)));  // bf16 callers are converted to fp16 first
}

__device__ __forceinline__ int quant_code(float a, float s) {
  const float v = a / s;  // IEEE division (a reciprocal multiply gives different codes)
  if (v != v) return 0;   // 0 / 0: an all-zero row
  return (int)fminf(fmaxf(rintf(v), -128.f), 127.f);
}

// one CTA quantises one row: token `xrow` of x [*, K] -> codes row `row` of q [*, Kp] and s_tok[row]
template <typename T>
__device__ __forceinline__ void qqq_quant_row(const T* __restrict__ x, int8_t* __restrict__ q, float* __restrict__ s_tok,
                                              int K, int Kp, int xrow, int row) {
  __shared__ float red[Q_QUANT_THREADS / 32];
  const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)xrow * K);
  const int n8 = K >> 3;
  float amax = 0.f;
  for (int i = threadIdx.x; i < n8; i += Q_QUANT_THREADS) {
    union {
      uint4 u;
      T h[8];
    } in;
    in.u = xr[i];
#pragma unroll
    for (int e = 0; e < 8; ++e) amax = fmaxf(amax, fabsf(to_half_f<T>(in.h[e])));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
  __syncthreads();
  amax = red[0];
#pragma unroll
  for (int w = 1; w < Q_QUANT_THREADS / 32; ++w) amax = fmaxf(amax, red[w]);
  const float s = __half2float(__float2half_rn(amax / 127.f));
  if (threadIdx.x == 0) s_tok[row] = s;
  uint2* qr = reinterpret_cast<uint2*>(q + (size_t)row * Kp);
  for (int i = threadIdx.x; i < (Kp >> 3); i += Q_QUANT_THREADS) {
    uint32_t w[2] = {0u, 0u};
    if (i < n8) {
      union {
        uint4 u;
        T h[8];
      } in;
      in.u = xr[i];
#pragma unroll
      for (int e = 0; e < 8; ++e) w[e >> 2] |= ((uint32_t)quant_code(to_half_f<T>(in.h[e]), s) & 0xFFu) << (8 * (e & 3));
    }
    qr[i] = make_uint2(w[0], w[1]);
  }
}

template <typename T>
__global__ void __launch_bounds__(Q_QUANT_THREADS)
    qqq_quant_kernel(const T* __restrict__ x, int8_t* __restrict__ q, float* __restrict__ s_tok, int K, int Kp) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // x is the previous kernel's output
  const int row = blockIdx.x;
  qqq_quant_row<T>(x, q, s_tok, K, Kp, row, row);
}

// the quantiser over the expert-sorted rows of a MoE block: row i is token sorted_pairs[i] / top_k of x [T, K], so its
// codes and scale are those qqq_quant_kernel gives that token
template <typename T>
__global__ void __launch_bounds__(Q_QUANT_THREADS)
    qqq_moe_gather_kernel(const T* __restrict__ x, const int32_t* __restrict__ sorted_pairs, int8_t* __restrict__ q,
                          float* __restrict__ s_tok, int top_k, int K, int Kp) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // sorted_pairs (and x) are the previous kernels' output
  const int row = blockIdx.x;
  qqq_quant_row<T>(x, q, s_tok, K, Kp, sorted_pairs[row] / top_k, row);
}

// ------------------------------------------------------------------------------------------------
// one-time repack: canonical codes uint8 [K, N] (0..15) -> the tile layout above
// ------------------------------------------------------------------------------------------------
__global__ void qqq_prepack_kernel(const uint8_t* __restrict__ codes, uint32_t* __restrict__ out, int K, int N, int KB,
                                   int grouped) {
  const size_t words = (size_t)KB * Q_TILE_BYTES / 4 * ((N + Q_BF - 1) / Q_BF);
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < words; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t tile = idx / (Q_TILE_BYTES / 4);
    const int r = (int)(idx % (Q_TILE_BYTES / 4));  // [quad][feature][word]
    const int quad = r / (Q_BF * 4), f = (r / 4) % Q_BF, j = r % 4;
    const int nt = (int)(tile / KB), kb = (int)(tile % KB);
    const int n = nt * Q_BF + f;
    const int k0 = kb * Q_BK + 32 * quad + 8 * j;
    uint32_t w = 0;
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      const int kk = grouped ? ((p & 1) | ((p & 2) << 1) | ((p & 4) >> 1)) : ((p & 1) ? (p >> 1) : 4 + (p >> 1));
      const int k = k0 + kk;
      const uint32_t c = (k < K && n < N) ? (uint32_t)(codes[(size_t)k * N + n] & 15u) : 0u;
      w |= c << (4 * p);
    }
    out[idx] = w;
  }
}

// ------------------------------------------------------------------------------------------------
// GEMM
// ------------------------------------------------------------------------------------------------
// one packed word (8 k) -> int8 weights of k0..3 (lo) and k4..7 (hi)
__device__ __forceinline__ void expand_channel(uint32_t w, uint32_t& lo, uint32_t& hi) {
  lo = w & 0xF0F0F0F0u;
  hi = (w << 4) & 0xF0F0F0F0u;
}
__device__ __forceinline__ void expand_group(uint32_t w, uint32_t s2, uint32_t& lo, uint32_t& hi) {
  const uint32_t EX = 0x64006400u;   // half2(1024 + nibble)
  const uint32_t SUB = 0x64086408u;  // half2(1032): (1024 + c) - 1032 = c - 8, exact
  const uint32_t MAG = 0x65006500u;  // half2(1280): low byte of 1280 + n is n (two's complement) for |n| <= 128
  uint32_t h[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t t = lop3_and_or(w >> (4 * i), 0x000f000fu, EX);  // lanes: nibbles (i, i + 4)
    __half2 d = __hsub2(*reinterpret_cast<__half2*>(&t), *reinterpret_cast<const __half2*>(&SUB));
    __half2 r = __hfma2(d, *reinterpret_cast<const __half2*>(&s2), *reinterpret_cast<const __half2*>(&MAG));
    h[i] = *reinterpret_cast<uint32_t*>(&r);
  }
  // nibbles 0, 1, 4, 5 = k0..3: bytes 0 of h0, h1 and bytes 2 of h0, h1
  lo = __byte_perm(h[0], h[1], 0x6240);
  hi = __byte_perm(h[2], h[3], 0x6240);
}

// grouped launches (MODE 1 / 2) over the experts of a MoE block: the stacks hold E experts back to back, one expert's
// b2q_qqq_packed_bytes(K, N), N channel scales and K/128 x N group scales apart
struct QqqMoeArgs {
  MoeRoute route;
  const uint4* packed3;     // MODE 1: the w3 (up) stack, shaped like the w1 (gate) stack
  const float* s_channel3;
  const __half* s_group3;
};

// the GEMM of qqq_gemm_kernel (MODE 0) and qqq_moe_gemm_kernel (MODE 1 / 2, G their grouped arguments).  MODE 1 pairs 64
// gate features (w1, m64 block 0) with the same 64 up features (w3, m64 block 1) in one 128-row tile and stores
// h = T(T(silu(g)) * u); MODE 2 (down) stores w[pair] * T(y) in fp32 to the pair's row of ypair
template <int NTOK, bool GROUPED, int MODE>
__device__ __forceinline__ void qqq_gemm_body(const CUtensorMap& tmap_q, const uint4* __restrict__ packed,
                                              const float* __restrict__ s_channel, const __half* __restrict__ s_group,
                                              const float* __restrict__ s_tok, const __half* __restrict__ bias,
                                              void* __restrict__ out, int M, int KB, int N, int kpc, int out_bf16,
                                              const QqqMoeArgs* G) {
  using C = QqqCfg<NTOK>;
  constexpr int PST = C::PST, WST = C::WST, XST = C::XST;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t sW = smem_base;                 // [WST][128 features][128 k]   (also: int32 partial tile)
  const uint32_t sX = sW + WST * C::W_BYTES;     // [XST][NTOK][128 k]
  const uint32_t sP = sX + XST * C::X_BYTES;     // [PST] packed tile
  const uint32_t sBar = sP + PST * Q_TILE_BYTES;
  const uint32_t bar_pfull = sBar, bar_xfull = bar_pfull + 8 * PST, bar_xempty = bar_xfull + 8 * XST;
  const uint32_t bar_wready = bar_xempty + 8 * XST, bar_wempty = bar_wready + 8 * WST;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = blockIdx.x, n0 = nt * (MODE == 1 ? Q_BF / 2 : Q_BF);  // MODE 1: 64 gate + 64 up features
  int row0 = blockIdx.z * NTOK, rows = NTOK;  // first row and row bound of this CTA's token block
  const uint4* packed3 = nullptr;
  const float* s_channel3 = nullptr;
  const __half* s_group3 = nullptr;
  if (MODE != 0) {
    int e;
    if (!moe_block<NTOK>(G->route, e, row0, rows)) return;
    // one expert: KB x ceil(N/128) packed tiles, N channel scales, KB x N group scales
    const size_t pstride = (size_t)KB * ((N + Q_BF - 1) / Q_BF) * (Q_TILE_BYTES / 16);
    packed += (size_t)e * pstride;
    s_channel += (size_t)e * N;
    if (GROUPED) s_group += (size_t)e * KB * N;
    if (MODE == 1) {
      packed3 = G->packed3 + (size_t)e * pstride;
      s_channel3 = G->s_channel3 + (size_t)e * N;
      if (GROUPED) s_group3 = G->s_group3 + (size_t)e * KB * N;
    }
  }
  const uint32_t nrank = cluster_nctarank(), crank = cluster_ctarank();
  const int kb0 = (int)crank * kpc, kb1 = min(KB, kb0 + kpc);
  const int nkb = kb1 - kb0;

  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_q);
    for (int s = 0; s < PST; ++s) mbar_init(bar_pfull + 8 * s, 1);
    for (int s = 0; s < XST; ++s) {
      mbar_init(bar_xfull + 8 * s, 1);
      mbar_init(bar_xempty + 8 * s, 1);
    }
    for (int s = 0; s < WST; ++s) {
      mbar_init(bar_wready + 8 * s, Q_DQ_THREADS);
      mbar_init(bar_wempty + 8 * s, 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  // MODE 1: the tile's 64 gate and 64 up features are one half of packed tile n0 / 128 of each stack
  const uint4* ptile = packed + (size_t)(MODE == 1 ? n0 / Q_BF : nt) * KB * (Q_TILE_BYTES / 16);
  const uint4* ptile3 = MODE == 1 ? packed3 + (size_t)(n0 / Q_BF) * KB * (Q_TILE_BYTES / 16) : nullptr;
  auto load_weights = [&](int i, int s) {
    mbar_expect_tx(bar_pfull + 8 * s, Q_TILE_BYTES);
    if (MODE == 1) {
      // quad q of a packed tile is [128 features] x 16 bytes: the 64-feature half of each stack is one 1 KB run per
      // quad, staged as features 0..63 (gate) and 64..127 (up) of the stage's quad
      const int half = (n0 / (Q_BF / 2)) & 1;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const size_t src = (size_t)(kb0 + i) * (Q_TILE_BYTES / 16) + q * Q_BF + half * (Q_BF / 2);
        const uint32_t dst = sP + s * Q_TILE_BYTES + q * Q_BF * 16;
        bulk_load(dst, ptile + src, Q_TILE_BYTES / 8, bar_pfull + 8 * s);
        bulk_load(dst + Q_TILE_BYTES / 8, ptile3 + src, Q_TILE_BYTES / 8, bar_pfull + 8 * s);
      }
    } else {
      bulk_load(sP + s * Q_TILE_BYTES, ptile + (size_t)(kb0 + i) * (Q_TILE_BYTES / 16), Q_TILE_BYTES, bar_pfull + 8 * s);
    }
  };

  if (warp == 8) {
    // ================================ activation producer ================================
    if (lane == 0) {
      asm volatile("griddepcontrol.wait;" ::: "memory");  // the codes are the quantiser's output
      for (int i = 0; i < nkb; ++i) {
        const int xs = i % XST;
        if (i >= XST) mbar_wait(bar_xempty + 8 * xs, ((i / XST) & 1) ^ 1);
        mbar_expect_tx(bar_xfull + 8 * xs, C::X_BYTES);
        tma_load_2d(sX + xs * C::X_BYTES, &tmap_q, bar_xfull + 8 * xs, (kb0 + i) * Q_BK, row0);
      }
    }
  } else if (warp < 4) {
    // ================================ MMA warpgroup ================================
    int acc[2][C::ACC];
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
      for (int v = 0; v < C::ACC; ++v) acc[mb][v] = 0;
    for (int i = 0; i < nkb; ++i) {
      const int xs = i % XST, ws = i % WST;
      mbar_wait(bar_xfull + 8 * xs, (i / XST) & 1);
      mbar_wait(bar_wready + 8 * ws, (i / WST) & 1);
      const uint64_t wdesc = wgmma_desc_k_sw128(sW + ws * C::W_BYTES);
      const uint64_t xdesc = wgmma_desc_k_sw128(sX + xs * C::X_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < Q_BK / 32; ++k)
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)
          Wgmma8<NTOK>::mma(acc[mb], wdesc + 512 * mb + 2 * k, xdesc + 2 * k, (i == 0 && k == 0) ? 0u : 1u);
      wgmma_commit();
      wgmma_wait<1>();
      if (i > 0 && threadIdx.x == 0) {
        mbar_arrive(bar_wempty + 8 * ((i - 1) % WST));
        mbar_arrive(bar_xempty + 8 * ((i - 1) % XST));
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) wgmma_fence_regs(acc[mb]);
    // this rank's int32 partial -> part[token][feature] in its own shared memory (the stage buffers are idle: every
    // load was consumed by an MMA that has completed)
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) park_partial(sW, mb, warp, acc[mb]);
  } else {
    // ================================ dequant warps ================================
    const int f = threadIdx.x - Q_MMA_THREADS;  // feature row of the tile
    // MODE 1: rows 0..63 expand gate feature n0 + f of w1, rows 64..127 up feature n0 + f - 64 of w3
    const int n = MODE == 1 ? n0 + (f & (Q_BF / 2 - 1)) : n0 + f;
    const __half* sgr = (MODE == 1 && f >= Q_BF / 2) ? s_group3 : s_group;
    // the weight stream of the first PST blocks starts at once (under programmatic dependent launch: while the
    // quantiser still runs)
    if (f == 0)
      for (int i = 0; i < nkb && i < PST; ++i) load_weights(i, i);
    for (int i = 0; i < nkb; ++i) {
      const int s = i % PST, ws = i % WST;
      uint32_t s2 = 0;
      if (GROUPED) {
        const __half sg = n < N ? sgr[(size_t)(kb0 + i) * N + n] : __float2half_rn(0.f);
        const __half2 sg2 = __halves2half2(sg, sg);
        s2 = *reinterpret_cast<const uint32_t*>(&sg2);
      }
      mbar_wait(bar_pfull + 8 * s, (i / PST) & 1);
      uint4 pv[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) pv[q] = reinterpret_cast<const uint4*>(smem + (sP - smem_base) + s * Q_TILE_BYTES)[q * Q_BF + f];
      // every thread has read the stage: refill it with block i + PST
      asm volatile("bar.sync 1, %0;" ::"r"(Q_DQ_THREADS) : "memory");
      if (f == 0 && i + PST < nkb) load_weights(i + PST, s);
      if (i >= WST) mbar_wait(bar_wempty + 8 * ws, ((i / WST) & 1) ^ 1);
      const uint32_t row = sW + ws * C::W_BYTES + f * 128;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint32_t wv[4] = {pv[q].x, pv[q].y, pv[q].z, pv[q].w};
        uint32_t o[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (GROUPED) expand_group(wv[j], s2, o[2 * j], o[2 * j + 1]);
          else expand_channel(wv[j], o[2 * j], o[2 * j + 1]);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {  // 16-byte chunk 2q + h = k 32q + 16h .. +15
          const uint32_t addr = row + ((((uint32_t)(2 * q + h)) ^ (uint32_t)(f & 7)) << 4);
          asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(o[4 * h]), "r"(o[4 * h + 1]),
                       "r"(o[4 * h + 2]), "r"(o[4 * h + 3])
                       : "memory");
        }
      }
      fence_proxy_async_smem();
      mbar_arrive(bar_wready + 8 * ws);
    }
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");  // (already satisfied) orders the global stores below
  __syncwarp();
  cluster_sync_all();
  // the reference epilogue: fp32(acc) * s_channel * s_tok, rounded to fp16
  auto y16 = [](int a, float sc, float st) { return __float2half_rn(__fmul_rn(__fmul_rn(__int2float_rn(a), sc), st)); };
  if (MODE == 1 && warp < Q_RED_WARPS) {
    // rank z reduces token rows z, z + nrank, ... , a half-warp per row: lane l holds gate features 4 (l & 15) .. + 3 of
    // the tile (those columns of h) and their up features at + 64
    const int hw = 2 * warp + (lane >> 4), c = lane & 15;
    const int nc = n0 + 4 * c;
    const float4 sg4 = *reinterpret_cast<const float4*>(s_channel + nc);
    const float4 su4 = *reinterpret_cast<const float4*>(s_channel3 + nc);
    const float scg[4] = {sg4.x, sg4.y, sg4.z, sg4.w}, scu[4] = {su4.x, su4.y, su4.z, su4.w};
    for (int tok = (int)crank + (int)nrank * hw; tok < rows; tok += (int)nrank * (2 * Q_RED_WARPS)) {
      int a[2][4];
      dsmem_sum4<2, true>(sW + (uint32_t)tok * (Q_BF * 4) + (uint32_t)c * 16, (Q_BF / 2) * 4, nrank, a);
      const float st = s_tok[row0 + tok];
      float g[4], u[4];  // the fp16 values of the layers' outputs
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        g[e] = __half2float(y16(a[0][e], scg[e], st));
        u[e] = __half2float(y16(a[1][e], scu[e], st));
      }
      const size_t o = (size_t)(row0 + tok) * N + nc;
      if (out_bf16) store_silu_mul4(reinterpret_cast<__nv_bfloat16*>(out) + o, g, u);
      else store_silu_mul4(reinterpret_cast<__half*>(out) + o, g, u);
    }
  } else if (MODE != 1 && warp < Q_RED_WARPS) {
    // rank z reduces token rows z, z + nrank, ... over all ranks: integer sums, so the order does not matter
    const int chunk = threadIdx.x & 31;
    const int nc = n0 + chunk * 4;
    if (nc < N) {
      const float4 sc = *reinterpret_cast<const float4*>(s_channel + nc);
      for (int tok = (int)crank + (int)nrank * warp; tok < NTOK && tok < rows && row0 + tok < M;
           tok += (int)nrank * Q_RED_WARPS) {
        int a[1][4];
        dsmem_sum4<1, true>(sW + (uint32_t)tok * (Q_BF * 4) + (uint32_t)chunk * 16, 0, nrank, a);
        const int m = row0 + tok;
        const float st = s_tok[m];
        const float scs[4] = {sc.x, sc.y, sc.z, sc.w};
        __half y[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          // then D.add_(bias)
          y[e] = y16(a[0][e], scs[e], st);
          if (bias != nullptr) y[e] = __float2half_rn(__half2float(y[e]) + __half2float(bias[nc + e]));
        }
        if (MODE == 2) {
          const int pair = G->route.sorted_pairs[m];
          float* yp = G->route.ypair + (size_t)pair * N + nc;
          const float yf[4] = {__half2float(y[0]), __half2float(y[1]), __half2float(y[2]), __half2float(y[3])};
          if (out_bf16) store_ypair4<__nv_bfloat16>(yp, G->route.pair_weights[pair], yf);
          else store_ypair4<__half>(yp, G->route.pair_weights[pair], yf);
        } else if (out_bf16) {
          __nv_bfloat16 b[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) b[e] = __float2bfloat16_rn(__half2float(y[e]));
          *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + (size_t)m * N + nc) =
              *reinterpret_cast<const uint2*>(b);
        } else {
          *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(out) + (size_t)m * N + nc) =
              *reinterpret_cast<const uint2*>(y);
        }
      }
    }
  }
  __syncwarp();
  cluster_sync_all();  // keep every rank's shared memory alive until all peers have read it
}

template <int NTOK, bool GROUPED>
__global__ void __launch_bounds__(Q_THREADS, 1)
    qqq_gemm_kernel(const __grid_constant__ CUtensorMap tmap_q, const uint4* __restrict__ packed,
                    const float* __restrict__ s_channel, const __half* __restrict__ s_group,
                    const float* __restrict__ s_tok, const __half* __restrict__ bias, void* __restrict__ out, int M,
                    int KB, int N, int kpc, int out_bf16) {
  qqq_gemm_body<NTOK, GROUPED, 0>(tmap_q, packed, s_channel, s_group, s_tok, bias, out, M, KB, N, kpc, out_bf16,
                                  nullptr);
}

// grouped launches over the experts of a MoE block: M = rows, N / K of one expert, out = h (MODE 1); the stacks of w1
// (MODE 1) or w2 (MODE 2) in packed / s_channel / s_group
template <int NTOK, bool GROUPED, int MODE>
__global__ void __launch_bounds__(Q_THREADS, 1)
    qqq_moe_gemm_kernel(const __grid_constant__ CUtensorMap tmap_q, const uint4* __restrict__ packed,
                        const float* __restrict__ s_channel, const __half* __restrict__ s_group,
                        const float* __restrict__ s_tok, void* __restrict__ out, int M, int KB, int N, int kpc,
                        int out_bf16, const __grid_constant__ QqqMoeArgs G) {
  qqq_gemm_body<NTOK, GROUPED, MODE>(tmap_q, packed, s_channel, s_group, s_tok, nullptr, out, M, KB, N, kpc, out_bf16,
                                     &G);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int launch_qqq_quant(const void* x, void* q, float* s_tok, int M, int K, int dtype, cudaStream_t stream) {
  const int Kp = (K + Q_BK - 1) / Q_BK * Q_BK;
  if (dtype == 0)
    return launch_kernel(qqq_quant_kernel<__half>, dim3(M, 1, 1), dim3(Q_QUANT_THREADS, 1, 1), 0, stream, 0, true,
                         (const __half*)x, (int8_t*)q, s_tok, K, Kp);
  return launch_kernel(qqq_quant_kernel<__nv_bfloat16>, dim3(M, 1, 1), dim3(Q_QUANT_THREADS, 1, 1), 0, stream, 0, true,
                       (const __nv_bfloat16*)x, (int8_t*)q, s_tok, K, Kp);
}

int launch_qqq_prepack(const uint8_t* codes, void* packed, int K, int N, int grouped, cudaStream_t stream) {
  const int KB = (K + Q_BK - 1) / Q_BK;
  const size_t words = (size_t)KB * ((N + Q_BF - 1) / Q_BF) * (Q_TILE_BYTES / 4);
  const int blocks = (int)((words + 255) / 256 < 65535 ? (words + 255) / 256 : 65535);
  qqq_prepack_kernel<<<blocks, 256, 0, stream>>>(codes, (uint32_t*)packed, K, N, KB, grouped);
  return (int)cudaGetLastError();
}

// tokens per CTA: the narrowest wgmma n that holds M (decode wastes no MMA width), 128-token blocks beyond; split-K over
// (tiles x token blocks) CTAs, at least 2 k-blocks per rank
SwapPlan qqq_plan(int M, int K, int N) {
  const int KB = (K + Q_BK - 1) / Q_BK, tiles = (N + Q_BF - 1) / Q_BF;
  SwapPlan p;
  p.ntok = swap_ntok(M, 8, 128);
  p.tblocks = (M + p.ntok - 1) / p.ntok;
  p.ks = trim_ranks(split_k_ranks((long long)tiles * p.tblocks, KB, 2), KB);
  p.kpc = (KB + p.ks - 1) / p.ks;
  return p;
}

template <int NTOK, bool GROUPED>
static int launch_qqq_gemm_t(const QqqArgs& a, const SwapPlan& p) {
  using C = QqqCfg<NTOK>;
  const int KB = (a.K + Q_BK - 1) / Q_BK;
  CUtensorMap tmap;  // the codes [M, Kp] in boxes of 128 k x NTOK tokens; rows >= M are zero-filled
  if (make_tmap_2d(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.q, KB * Q_BK, a.M, (size_t)KB * Q_BK, Q_BK, NTOK,
                   CU_TENSOR_MAP_SWIZZLE_128B) != 0)
    return -1;
  auto kern = qqq_gemm_kernel<NTOK, GROUPED>;
  static int smem_opted[32] = {};
  if (int e = ensure_dyn_smem(kern, C::SMEM_BYTES, smem_opted, "b2q_qqq")) return e;
  return launch_kernel(kern, dim3((a.N + Q_BF - 1) / Q_BF, p.ks, p.tblocks), dim3(Q_THREADS, 1, 1), C::SMEM_BYTES,
                       a.stream, p.ks, true, tmap, (const uint4*)a.packed, a.s_channel, (const __half*)a.s_group,
                       a.s_tok, (const __half*)a.bias, a.out, a.M, KB, a.N, p.kpc, a.out_dtype);
}

int launch_qqq_gemm(const QqqArgs& a) {
  const bool g = a.s_group != nullptr;
  const SwapPlan p = qqq_plan(a.M, a.K, a.N);
  switch (p.ntok) {
    case 8: return g ? launch_qqq_gemm_t<8, true>(a, p) : launch_qqq_gemm_t<8, false>(a, p);
    case 16: return g ? launch_qqq_gemm_t<16, true>(a, p) : launch_qqq_gemm_t<16, false>(a, p);
    case 32: return g ? launch_qqq_gemm_t<32, true>(a, p) : launch_qqq_gemm_t<32, false>(a, p);
    case 64: return g ? launch_qqq_gemm_t<64, true>(a, p) : launch_qqq_gemm_t<64, false>(a, p);
    default: return g ? launch_qqq_gemm_t<128, true>(a, p) : launch_qqq_gemm_t<128, false>(a, p);
  }
}

int launch_qqq_moe_gather(const void* x, const int32_t* sorted_pairs, void* q, float* s_tok, int rows, int top_k, int K,
                          int dtype, cudaStream_t stream) {
  const int Kp = (K + Q_BK - 1) / Q_BK * Q_BK;
  if (dtype == 0)
    return launch_kernel(qqq_moe_gather_kernel<__half>, dim3(rows, 1, 1), dim3(Q_QUANT_THREADS, 1, 1), 0, stream, 0,
                         true, (const __half*)x, sorted_pairs, (int8_t*)q, s_tok, top_k, K, Kp);
  return launch_kernel(qqq_moe_gather_kernel<__nv_bfloat16>, dim3(rows, 1, 1), dim3(Q_QUANT_THREADS, 1, 1), 0, stream, 0,
                       true, (const __nv_bfloat16*)x, sorted_pairs, (int8_t*)q, s_tok, top_k, K, Kp);
}

// grouped launches: the token box of qqq_plan for all rows; split-K ranks fill the SMs with the CTAs of all rows' token
// blocks or of `active` experts' first blocks, whichever is more (the rule of fp8blk_plan)
static SwapPlan qqq_moe_plan(int mode, int M, int K, int N, int active) {
  const int KB = (K + Q_BK - 1) / Q_BK, fb = mode == 1 ? Q_BF / 2 : Q_BF, tiles = (N + fb - 1) / fb;
  SwapPlan p;
  p.ntok = swap_ntok(M, 8, 128);
  p.tblocks = (M + p.ntok - 1) / p.ntok;
  if (active < 1) active = 1;
  p.ks = trim_ranks(split_k_ranks((long long)tiles * (p.tblocks > active ? p.tblocks : active), KB, 2), KB);
  p.kpc = (KB + p.ks - 1) / p.ks;
  return p;
}

template <int NTOK, bool GROUPED, int MODE>
static int launch_qqq_moe_t(const QqqArgs& a, const QqqMoe& g, const SwapPlan& p) {
  using C = QqqCfg<NTOK>;
  const int KB = (a.K + Q_BK - 1) / Q_BK;
  CUtensorMap tmap;  // the sorted rows' codes [M, Kp]; a box may run into the next expert's rows, which are not stored
  if (make_tmap_2d(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.q, KB * Q_BK, a.M, (size_t)KB * Q_BK, Q_BK, NTOK,
                   CU_TENSOR_MAP_SWIZZLE_128B) != 0)
    return -1;
  QqqMoeArgs G = {};
  G.route = {g.counts, g.offsets, g.sorted_pairs, g.pair_weights, g.ypair, p.tblocks, 0};
  G.packed3 = (const uint4*)g.packed3;
  G.s_channel3 = g.s_channel3;
  G.s_group3 = (const __half*)g.s_group3;
  auto kern = qqq_moe_gemm_kernel<NTOK, GROUPED, MODE>;
  static int smem_opted[32] = {};
  if (int e = ensure_dyn_smem(kern, C::SMEM_BYTES, smem_opted, "b2q_qqq_moe")) return e;
  const int tiles = (a.N + (MODE == 1 ? Q_BF / 2 : Q_BF) - 1) / (MODE == 1 ? Q_BF / 2 : Q_BF);
  return launch_split_z((long long)g.E * p.tblocks, [&](int z0, int grid_z) {
    G.route.z0 = z0;
    return launch_kernel(kern, dim3(tiles, p.ks, grid_z), dim3(Q_THREADS, 1, 1), C::SMEM_BYTES, a.stream, p.ks, true,
                         tmap, (const uint4*)a.packed, a.s_channel, (const __half*)a.s_group, a.s_tok, a.out, a.M, KB,
                         a.N, p.kpc, a.out_dtype, G);
  });
}

int launch_qqq_moe(int mode, const QqqArgs& a, const QqqMoe& g) {
  const bool gr = a.s_group != nullptr;
  const SwapPlan p = qqq_moe_plan(mode, a.M, a.K, a.N, g.active);
#define B2Q_QQM(NTOK) \
  return mode == 1 ? (gr ? launch_qqq_moe_t<NTOK, true, 1>(a, g, p) : launch_qqq_moe_t<NTOK, false, 1>(a, g, p)) \
                   : (gr ? launch_qqq_moe_t<NTOK, true, 2>(a, g, p) : launch_qqq_moe_t<NTOK, false, 2>(a, g, p));
  switch (p.ntok) {
    case 8: B2Q_QQM(8)
    case 16: B2Q_QQM(16)
    case 32: B2Q_QQM(32)
    case 64: B2Q_QQM(64)
    default: B2Q_QQM(128)
  }
#undef B2Q_QQM
}

}  // namespace b2q
