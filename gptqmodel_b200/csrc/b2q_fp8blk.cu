// b2q_fp8blk.cu — block-FP8 (HF / DeepSeek-native, W8A8) tier: e4m3 weights with 128 x 128 block scales times
// per-token-group e4m3 activations on the e4m3 tensor cores.  include/b2q.h states the arithmetic.  Kernels:
//   * fp8blk_quant_kernel: one half-warp per (token, 128-k group): amax, s_x = max(amax, 1e-10) / 448 (IEEE division),
//     codes = e4m3_rn_satfinite(x / s_x) (IEEE division), written as uint8 [M, K] and fp32 s_x [K/128, Mp].
//   * fp8blk_gemm_kernel: the structure of qqq_gemm_kernel without dequant warps.  The checkpoint weight [N, K] e4m3 is
//     already the K-major wgmma A operand: warp 8 loads 128 features x 128 k per k-block straight from it with TMA
//     (SWIZZLE_128B, rows >= N zero-filled), and the activation codes (B operand, n = NTOK tokens) with their token
//     scales.  Warpgroup 0 multiplies features 0..63 of the tile, warpgroup 1 features 64..127, each on
//     m64nNk32.f32.e4m3.e4m3 into a per-block fp32 temporary P that is promoted once per k-block:
//     acc = fmaf(P, s_x[m] * s_w[tile], acc).  The `ks` CTAs of a cluster split the k-blocks of a tile in contiguous
//     runs and sum their fp32 partials over distributed shared memory in rank order; token blocks of NTOK rows are
//     spread over gridDim.z.  No atomics, deterministic for a given launch plan.
//     Decode (M <= 8, FUSED): there is no quantiser launch.  Warp 8 quantises each k-block of x it hands to the MMA
//     warps itself, with the same device functions as fp8blk_quant_kernel (1 x 128 groups are local to a k-block), writes
//     the swizzled B tile and the block's s_x, and fences them to the async proxy.
//   * fp8blk_moe_gemm_kernel: grouped modes of the same GEMM body for MoE experts (MODE 1 / 2): z0 + blockIdx.z =
//     (expert, token block) over the expert-sorted rows that b2q_moe_align ordered; the weights are the stacked
//     checkpoint tensors [E*N, K] and [E, ceil(N/128), K/128].  MODE 1
//     pairs 64 gate features (w1, warpgroup 0) with the same 64 up features (w3, warpgroup 1) in one 128-row tile and
//     stores h = T(T(silu(T(g))) * T(u)); MODE 2 (down) stores w[pair] * T(acc) in fp32 to the pair's row of ypair.
//   * fp8blk_moe_gather_kernel: the quantiser over the sorted rows, row i reading token sorted_pairs[i] / top_k.
#include <cuda.h>

#include <type_traits>

#include "b2q_common.cuh"
#include "b2q_internal.h"
#include "b2q_wgmma.cuh"

namespace b2q {

constexpr int F_BF = 128;                 // features per tile (= the checkpoint's scale block rows)
constexpr int F_BK = 128;                 // k per block (= the scale block columns; one SWIZZLE_128B row of e4m3)
constexpr int F_MMA_THREADS = 256;        // warps 0..7: two MMA warpgroups
constexpr int F_THREADS = F_MMA_THREADS + 32;  // + warp 8: producer
constexpr int F_MAX_KB = 512;             // K <= 65536: the tile's s_w row lives in shared memory
constexpr int F_QUANT_THREADS = 256;      // quantiser: 16 groups of 128 k per CTA

template <int NTOK, int MODE = 0>
struct FblkCfg {
  static constexpr int ST = NTOK == 128 ? 6 : 8;  // stages
  static constexpr int W_BYTES = F_BF * F_BK;
  static constexpr int X_BYTES = NTOK * F_BK;
  // grouped modes: a block's first row is any row, so its token scales are loaded from the 16-byte aligned row below it
  // (4 more scales) — the innermost TMA coordinate stays 16-byte aligned
  static constexpr int SX_BYTES = (NTOK + (MODE != 0 ? 4 : 0)) * 4;
  static constexpr int STAGE_BYTES = (W_BYTES + X_BYTES + SX_BYTES + 1023) / 1024 * 1024;
  static constexpr int SW_BYTES = (MODE == 1 ? 2 : 1) * F_MAX_KB * 4;  // MODE 1: the gate row, then the up row
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = ST * STAGE_BYTES + SW_BYTES + BAR_BYTES + 1024;
  static constexpr int ACC = NTOK / 2;  // fp32 accumulators per thread of one m64 x NTOK warpgroup tile
  static_assert(X_BYTES % 1024 == 0, "activation tiles must stay 1024-byte aligned (SWIZZLE_128B atoms)");
  static_assert(NTOK * F_BF * 4 <= ST * STAGE_BYTES, "the fp32 partial tile reuses the stages");
  static_assert(2 * ST * 8 <= BAR_BYTES, "mbarrier area");
  static_assert(SMEM_BYTES <= 227 * 1024, "dynamic shared memory of one CTA");
};

// ------------------------------------------------------------------------------------------------
// the quantiser's arithmetic: one device function per step, shared by both kernels so their codes are identical
// ------------------------------------------------------------------------------------------------
// A group of 128 k is held by a half-warp, lane j (= lane & 15) owning elements 8 j .. 8 j + 7 in `v`.  All 32 lanes
// call this (the shuffles span the warp; the halves do not mix): the group's scale max(amax, 1e-10) / 448.
template <typename T>
__device__ __forceinline__ float fblk_group_scale(const uint4& v) {
  const T* h = reinterpret_cast<const T*>(&v);
  float a = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) a = fmaxf(a, fabsf(ET<T>::to_f(h[e])));
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
  return fmaxf(a, 1e-10f) / 448.f;  // IEEE division
}

// one half-warp per (token m, k-block b); lane j of it owns elements 8 j .. 8 j + 7
template <typename T>
__global__ void __launch_bounds__(F_QUANT_THREADS)
    fp8blk_quant_kernel(const T* __restrict__ x, uint8_t* __restrict__ codes, float* __restrict__ s_x, int M, int K,
                        int Mp) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // x is the previous kernel's output
  const int KB = K / F_BK;
  const long long g = ((long long)blockIdx.x * F_QUANT_THREADS + threadIdx.x) >> 4;
  const int j = threadIdx.x & 15;
  const bool live = g < (long long)M * KB;  // the whole warp stays for the shuffles
  const int m = live ? (int)(g / KB) : 0, b = live ? (int)(g % KB) : 0;
  const size_t off = (size_t)m * K + (size_t)b * F_BK + 8 * j;
  const uint4 v = live ? *reinterpret_cast<const uint4*>(x + off) : make_uint4(0u, 0u, 0u, 0u);
  const float s = fblk_group_scale<T>(v);
  if (!live) return;
  *reinterpret_cast<uint2*>(codes + off) = fblk_code8<T>(v, s);
  if (j == 0) s_x[(size_t)b * Mp + m] = s;
}

// the quantiser over the expert-sorted rows of a MoE block: row i is token sorted_pairs[i] / top_k of x [T, K], so its
// codes and scale are those fp8blk_quant_kernel gives that token
template <typename T>
__global__ void __launch_bounds__(F_QUANT_THREADS)
    fp8blk_moe_gather_kernel(const T* __restrict__ x, const int32_t* __restrict__ sorted_pairs,
                             uint8_t* __restrict__ codes, float* __restrict__ s_x, int rows, int top_k, int K, int Mp) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // sorted_pairs (and x) are the previous kernels' output
  const int KB = K / F_BK;
  const long long g = ((long long)blockIdx.x * F_QUANT_THREADS + threadIdx.x) >> 4;
  const int j = threadIdx.x & 15;
  const bool live = g < (long long)rows * KB;  // the whole warp stays for the shuffles
  const int i = live ? (int)(g / KB) : 0, b = live ? (int)(g % KB) : 0;
  const int tok = live ? sorted_pairs[i] / top_k : 0;
  const uint4 v = live ? *reinterpret_cast<const uint4*>(x + (size_t)tok * K + (size_t)b * F_BK + 8 * j)
                       : make_uint4(0u, 0u, 0u, 0u);
  const float s = fblk_group_scale<T>(v);
  if (!live) return;
  *reinterpret_cast<uint2*>(codes + (size_t)i * K + (size_t)b * F_BK + 8 * j) = fblk_code8<T>(v, s);
  if (j == 0) s_x[(size_t)b * Mp + i] = s;
}

// ------------------------------------------------------------------------------------------------
// GEMM
// ------------------------------------------------------------------------------------------------
// grouped launches (MODE 1 / 2) over the experts of a MoE block
struct FblkMoeArgs {
  CUtensorMap tmap_w3;           // MODE 1: the w3 stack [E*N, K], 64-row boxes (tmap_w: the w1 stack, the same boxes)
  MoeRoute route;
  const float* s_w3;             // [E, ceil(N/128), K/128] scales of w3                     (MODE 1)
};

// the GEMM of fp8blk_gemm_kernel (MODE 0) and fp8blk_moe_gemm_kernel (MODE 1 / 2, G their grouped arguments).
// FUSED: 0 = codes and token scales come from fp8blk_quant_kernel (TMA); 1 / 2 = M <= 8, the producer quantises x
// (fp16 / bf16) itself.  MODE: 0 = one layer, 1 = grouped gate|up, 2 = grouped down (FUSED == 0)
template <int NTOK, int FUSED, int MODE>
__device__ __forceinline__ void fp8blk_gemm_body(const CUtensorMap& tmap_w, const CUtensorMap& tmap_q,
                                                 const CUtensorMap& tmap_s, const void* __restrict__ x,
                                                 const float* __restrict__ s_w, const void* __restrict__ bias,
                                                 void* __restrict__ out, int M, int K, int N, int kpc, int out_bf16,
                                                 const FblkMoeArgs* G) {
  using C = FblkCfg<NTOK, MODE>;
  constexpr int ST = C::ST;
  static_assert(!FUSED || NTOK == 8, "the fused quantiser serves 8-token tiles");
  static_assert(MODE == 0 || !FUSED, "the grouped modes read quantised codes");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
  // stage s: [W 128 x 128][X NTOK x 128][s_x NTOK]; then the tile's s_w row; then the barriers
  const uint32_t sSW = smem_base + ST * C::STAGE_BYTES;
  const uint32_t bar_full = sSW + C::SW_BYTES, bar_empty = bar_full + 8 * ST;
  const float* sw_s = reinterpret_cast<const float*>(smem + ST * C::STAGE_BYTES);
  auto sW = [&](int s) { return smem_base + (uint32_t)(s * C::STAGE_BYTES); };
  auto sX = [&](int s) { return sW(s) + C::W_BYTES; };
  auto sSX = [&](int s) { return sX(s) + C::X_BYTES; };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = blockIdx.x, n0 = nt * (MODE == 1 ? F_BF / 2 : F_BF);  // MODE 1: 64 gate + 64 up features
  int row0 = blockIdx.z * NTOK, rows = min(NTOK, M - row0);  // first row and row count of this CTA's token block
  int e = 0;                                                   // expert (grouped modes)
  if (MODE != 0 && !moe_block<NTOK>(G->route, e, row0, rows)) return;
  const int wrow = MODE == 0 ? n0 : e * N + n0;  // first row of the tile in the (stacked) weight tensor
  const int KB = K / F_BK;
  const uint32_t nrank = cluster_nctarank(), crank = cluster_ctarank();
  const int kb0 = min(KB, (int)crank * kpc), kb1 = min(KB, kb0 + kpc);
  const int nkb = kb1 - kb0;

  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_w);
    if (MODE == 1) prefetch_tmap(&G->tmap_w3);
    if (!FUSED) {
      prefetch_tmap(&tmap_q);
      prefetch_tmap(&tmap_s);
    }
    for (int s = 0; s < ST; ++s) {
      mbar_init(bar_full + 8 * s, FUSED ? 32 : 1);
      mbar_init(bar_empty + 8 * s, F_MMA_THREADS / 32);
    }
    fence_mbar_init();
  }
  // the tile's weight scales (a layer constant: no dependency on the previous kernel)
  if (MODE == 0) {
    for (int i = threadIdx.x; i < nkb; i += F_THREADS)
      reinterpret_cast<float*>(smem + ST * C::STAGE_BYTES)[i] = s_w[(size_t)nt * KB + kb0 + i];
  } else {
    // the scale row of the tile's features in expert e's [ceil(N/128), K/128] grid (MODE 1: of the gate and the up set)
    const size_t sr = ((size_t)e * ((N + F_BF - 1) / F_BF) + n0 / F_BF) * KB + kb0;
    for (int i = threadIdx.x; i < nkb; i += F_THREADS) {
      reinterpret_cast<float*>(smem + ST * C::STAGE_BYTES)[i] = s_w[sr + i];
      if (MODE == 1) reinterpret_cast<float*>(smem + ST * C::STAGE_BYTES)[F_MAX_KB + i] = G->s_w3[sr + i];
    }
  }
  __syncthreads();

  if (warp == 8) {
    // ================================ producer ================================
    auto load_weights = [&](int i, int s) {
      mbar_expect_tx_only(bar_full + 8 * s, C::W_BYTES);
      tma_load_2d(sW(s), &tmap_w, bar_full + 8 * s, (kb0 + i) * F_BK, wrow);
      // MODE 1: the up features' 64-row box fills the second m64 half of the tile
      if (MODE == 1) tma_load_2d(sW(s) + C::W_BYTES / 2, &G->tmap_w3, bar_full + 8 * s, (kb0 + i) * F_BK, wrow);
    };
    // the weight stream of the first ST blocks starts at once (under programmatic dependent launch: while the
    // previous kernel still runs)
    if (lane == 0)
      for (int i = 0; i < nkb && i < ST; ++i) load_weights(i, i);
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (FUSED) {
      using T = typename std::conditional<FUSED == 1, __half, __nv_bfloat16>::type;
      // the quantiser kernel's mapping: half-warp h of pass p holds token t = 2 p + h, lane j = lane & 15 its elements
      // 8 j .. 8 j + 7 of the k-block; rows t >= M keep the zero codes and scales written here once
      constexpr int PD = 4;  // k-blocks of activations in flight ahead of the one being quantised
      const int h = lane >> 4, j = lane & 15;
      for (int s = 0; s < ST; ++s) {
        for (int o = lane; o < C::X_BYTES / 16; o += 32)
          asm volatile("st.shared.v4.u32 [%0], {%1,%1,%1,%1};" ::"r"(sX(s) + 16u * o), "r"(0u) : "memory");
        if (lane < NTOK) asm volatile("st.shared.f32 [%0], %1;" ::"r"(sSX(s) + 4u * lane), "f"(0.f) : "memory");
      }
      const T* xr = reinterpret_cast<const T*>(x) + (size_t)kb0 * F_BK + 8 * j;
      uint4 buf[PD][4];  // [in-flight k-block][pass]
      auto fetch = [&](int i, uint4(&dst)[4]) {
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const int t = 2 * p + h;
          dst[p] = (t < M && i < nkb) ? *reinterpret_cast<const uint4*>(xr + (size_t)t * K + (size_t)i * F_BK)
                                      : make_uint4(0u, 0u, 0u, 0u);
        }
      };
#pragma unroll
      for (int u = 0; u < PD; ++u) fetch(u, buf[u]);
      for (int i0 = 0; i0 < nkb; i0 += PD) {
#pragma unroll
        for (int u = 0; u < PD; ++u) {
          const int i = i0 + u;
          if (i >= nkb) break;
          const int s = i % ST;
          uint4 cur[4];
#pragma unroll
          for (int p = 0; p < 4; ++p) cur[p] = buf[u][p];
          fetch(i + PD, buf[u]);
          if (i >= ST) {
            mbar_wait(bar_empty + 8 * s, ((i / ST) & 1) ^ 1);
            if (lane == 0) load_weights(i, s);
          }
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            if (2 * p >= M) break;  // warp-uniform: both halves take part in the shuffles
            const int t = 2 * p + h;
            const float sx = fblk_group_scale<T>(cur[p]);
            if (t < M) {
              const uint2 q = fblk_code8<T>(cur[p], sx);
              const uint32_t addr = sX(s) + (uint32_t)t * 128 + ((((uint32_t)(j >> 1)) ^ (uint32_t)t) << 4) + 8u * (j & 1);
              asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(addr), "r"(q.x), "r"(q.y) : "memory");
              if (j == 0) asm volatile("st.shared.f32 [%0], %1;" ::"r"(sSX(s) + 4u * t), "f"(sx) : "memory");
            }
          }
          fence_proxy_async_smem();
          mbar_arrive(bar_full + 8 * s);
        }
      }
    } else if (lane == 0) {
      for (int i = 0; i < nkb; ++i) {
        const int s = i % ST;
        if (i >= ST) {
          mbar_wait(bar_empty + 8 * s, ((i / ST) & 1) ^ 1);
          load_weights(i, s);
        }
        mbar_expect_tx(bar_full + 8 * s, C::X_BYTES + C::SX_BYTES);
        tma_load_2d(sX(s), &tmap_q, bar_full + 8 * s, (kb0 + i) * F_BK, row0);
        tma_load_2d(sSX(s), &tmap_s, bar_full + 8 * s, MODE == 0 ? row0 : row0 & ~3, kb0 + i);
      }
    }
  } else {
    // ================================ MMA warpgroups ================================
    const int wg = warp >> 2;  // features 64 wg .. 64 wg + 63 of the tile
    float acc[C::ACC], p[C::ACC];
#pragma unroll
    for (int v = 0; v < C::ACC; ++v) acc[v] = 0.f;
    for (int i = 0; i < nkb; ++i) {
      const int s = i % ST;
      mbar_wait(bar_full + 8 * s, (i / ST) & 1);
      const uint64_t wdesc = wgmma_desc_k_sw128(sW(s)) + 512 * wg;
      const uint64_t xdesc = wgmma_desc_k_sw128(sX(s));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < F_BK / 32; ++k) Wgmma8F<NTOK>::mma(p, wdesc + 2 * k, xdesc + 2 * k, k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(p);
      // promotion: one s_w per tile and k-block, one s_x per token
      const float sw = sw_s[(MODE == 1 ? wg * F_MAX_KB : 0) + i];
      const float* sxs = reinterpret_cast<const float*>(smem + (sSX(s) - smem_base)) + (MODE == 0 ? 0 : row0 & 3);
#pragma unroll
      for (int j = 0; j < NTOK / 8; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const float sc = sxs[8 * j + 2 * (lane & 3) + c] * sw;
          acc[4 * j + c] = fmaf(p[4 * j + c], sc, acc[4 * j + c]);
          acc[4 * j + 2 + c] = fmaf(p[4 * j + 2 + c], sc, acc[4 * j + 2 + c]);
        }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * s);
    }
    // both warpgroups are done with the stages before either overwrites them with its partial tile
    asm volatile("bar.sync 1, %0;" ::"r"(F_MMA_THREADS) : "memory");
    // this rank's fp32 partial -> part[token][feature] in its own shared memory
    park_partial(smem_base, wg, warp & 3, acc);
  }
  __syncwarp();
  cluster_sync_all();
  if (MODE == 1 && warp < F_MMA_THREADS / 32) {
    // rank z reduces token rows z, z + nrank, ... , a half-warp per row: lane l holds gate features 4 (l & 15) .. + 3 of
    // the tile (those columns of h) and their up features at + 64
    const int hw = 2 * warp + (lane >> 4), c = lane & 15;
    for (int tok = (int)crank + (int)nrank * hw; tok < rows; tok += (int)nrank * (2 * F_MMA_THREADS / 32)) {
      float gu[2][4];
      dsmem_sum4<2, false>(smem_base + (uint32_t)tok * (F_BF * 4) + (uint32_t)c * 16, (F_BF / 2) * 4, nrank, gu);
      const size_t o = (size_t)(row0 + tok) * N + n0 + 4 * c;
      if (out_bf16) store_silu_mul4(reinterpret_cast<__nv_bfloat16*>(out) + o, gu[0], gu[1]);
      else store_silu_mul4(reinterpret_cast<__half*>(out) + o, gu[0], gu[1]);
    }
  } else if (MODE != 1 && warp < F_MMA_THREADS / 32) {
    // rank z reduces token rows z, z + nrank, ... , a warp per row
    const int nc = n0 + lane * 4;
    if (nc < N) {
      for (int tok = (int)crank + (int)nrank * warp; tok < rows; tok += (int)nrank * (F_MMA_THREADS / 32)) {
        float a[1][4];
        dsmem_sum4<1, false>(smem_base + (uint32_t)tok * (F_BF * 4) + (uint32_t)lane * 16, 0, nrank, a);
        if (MODE == 2) {
          const int pair = G->route.sorted_pairs[row0 + tok];
          float* y = G->route.ypair + (size_t)pair * N + nc;
          if (out_bf16) store_ypair4<__nv_bfloat16>(y, G->route.pair_weights[pair], a[0]);
          else store_ypair4<__half>(y, G->route.pair_weights[pair], a[0]);
        } else {
          const size_t o = (size_t)(row0 + tok) * N + nc;
          if (out_bf16)
            store_out4(reinterpret_cast<__nv_bfloat16*>(out) + o, reinterpret_cast<const __nv_bfloat16*>(bias), nc, a[0]);
          else
            store_out4(reinterpret_cast<__half*>(out) + o, reinterpret_cast<const __half*>(bias), nc, a[0]);
        }
      }
    }
  }
  __syncwarp();
  cluster_sync_all();  // keep every rank's shared memory alive until all peers have read it
}

template <int NTOK, int FUSED>
__global__ void __launch_bounds__(F_THREADS, 1)
    fp8blk_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_q,
                       const __grid_constant__ CUtensorMap tmap_s, const void* __restrict__ x,
                       const float* __restrict__ s_w, const void* __restrict__ bias, void* __restrict__ out, int M,
                       int K, int N, int kpc, int out_bf16) {
  fp8blk_gemm_body<NTOK, FUSED, 0>(tmap_w, tmap_q, tmap_s, x, s_w, bias, out, M, K, N, kpc, out_bf16, nullptr);
}

// grouped launches over the experts of a MoE block: M = rows, N / K of one expert, out = h (MODE 1)
template <int NTOK, int MODE>
__global__ void __launch_bounds__(F_THREADS, 1)
    fp8blk_moe_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_q,
                           const __grid_constant__ CUtensorMap tmap_s, const float* __restrict__ s_w,
                           void* __restrict__ out, int M, int K, int N, int kpc, int out_bf16,
                           const __grid_constant__ FblkMoeArgs G) {
  fp8blk_gemm_body<NTOK, 0, MODE>(tmap_w, tmap_q, tmap_s, nullptr, s_w, nullptr, out, M, K, N, kpc, out_bf16, &G);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int fp8blk_mp(int M) { return (M + 3) / 4 * 4; }

int launch_fp8blk_quant(const void* x, void* codes, float* s_x, int M, int K, int dtype, cudaStream_t stream) {
  const long long threads = (long long)M * (K / F_BK) * 16;
  const dim3 grid((unsigned)((threads + F_QUANT_THREADS - 1) / F_QUANT_THREADS), 1, 1);
  if (dtype == 0)
    return launch_kernel(fp8blk_quant_kernel<__half>, grid, dim3(F_QUANT_THREADS, 1, 1), 0, stream, 0, true,
                         (const __half*)x, (uint8_t*)codes, s_x, M, K, fp8blk_mp(M));
  return launch_kernel(fp8blk_quant_kernel<__nv_bfloat16>, grid, dim3(F_QUANT_THREADS, 1, 1), 0, stream, 0, true,
                       (const __nv_bfloat16*)x, (uint8_t*)codes, s_x, M, K, fp8blk_mp(M));
}

// tokens per CTA: the narrowest wgmma n that holds M, 128-token blocks beyond.  Split-K ranks: fill the SMs with
// (tiles x token blocks x ranks) CTAs, at least 2 k-blocks per rank; a grouped launch counts the token blocks of all
// rows or `active` experts' first blocks, whichever is more.  A pinned ks (> 0) is taken as given, untrimmed.
SwapPlan fp8blk_plan(int mode, int M, int K, int N, int active, int ks) {
  const int KB = K / F_BK, fb = mode == 1 ? F_BF / 2 : F_BF, tiles = (N + fb - 1) / fb;
  SwapPlan p;
  p.ntok = swap_ntok(M, 8, 128);
  p.tblocks = (M + p.ntok - 1) / p.ntok;
  if (active < 1) active = 1;
  const long long blocks = (long long)tiles * (mode == 0 || p.tblocks > active ? p.tblocks : active);
  p.ks = ks > 0 ? ks : trim_ranks(split_k_ranks(blocks, KB, 2), KB);
  p.kpc = (KB + p.ks - 1) / p.ks;
  return p;
}

template <int NTOK, int FUSED>
static int launch_fp8blk_gemm_t(const Fp8BlkArgs& a, const SwapPlan& p) {
  using C = FblkCfg<NTOK>;
  const int KB = a.K / F_BK;
  CUtensorMap tw, tq, ts;
  if (make_tmap_2d(&tw, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.weight, a.K, a.N, (size_t)a.K, F_BK, F_BF,
                   CU_TENSOR_MAP_SWIZZLE_128B) != 0)
    return -1;
  if (FUSED) {
    tq = tw;  // unused
    ts = tw;
  } else {
    if (make_tmap_2d(&tq, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.codes, a.K, a.M, (size_t)a.K, F_BK, NTOK,
                     CU_TENSOR_MAP_SWIZZLE_128B) != 0)
      return -1;
    if (make_tmap_2d(&ts, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, a.s_x, a.M, KB, (size_t)fp8blk_mp(a.M) * 4, NTOK, 1,
                     CU_TENSOR_MAP_SWIZZLE_NONE) != 0)
      return -1;
  }
  auto kern = fp8blk_gemm_kernel<NTOK, FUSED>;
  static int smem_opted[32] = {};
  if (int e = ensure_dyn_smem(kern, C::SMEM_BYTES, smem_opted, "b2q_fp8blk")) return e;
  return launch_kernel(kern, dim3((a.N + F_BF - 1) / F_BF, p.ks, p.tblocks), dim3(F_THREADS, 1, 1), C::SMEM_BYTES,
                       a.stream, p.ks, true, tw, tq, ts, a.x, a.s_w, a.bias, a.out, a.M, a.K, a.N, p.kpc, a.dtype);
}

int launch_fp8blk_gemm(const Fp8BlkArgs& a) {
  const SwapPlan p = fp8blk_plan(0, a.M, a.K, a.N, 1, a.ks);
  if (a.x != nullptr) return a.dtype == 0 ? launch_fp8blk_gemm_t<8, 1>(a, p) : launch_fp8blk_gemm_t<8, 2>(a, p);
  switch (p.ntok) {
    case 8: return launch_fp8blk_gemm_t<8, 0>(a, p);
    case 16: return launch_fp8blk_gemm_t<16, 0>(a, p);
    case 32: return launch_fp8blk_gemm_t<32, 0>(a, p);
    case 64: return launch_fp8blk_gemm_t<64, 0>(a, p);
    default: return launch_fp8blk_gemm_t<128, 0>(a, p);
  }
}

int launch_fp8blk_moe_gather(const void* x, const int32_t* sorted_pairs, void* codes, float* s_x, int rows, int top_k,
                             int K, int dtype, cudaStream_t stream) {
  const long long threads = (long long)rows * (K / F_BK) * 16;
  const dim3 grid((unsigned)((threads + F_QUANT_THREADS - 1) / F_QUANT_THREADS), 1, 1);
  if (dtype == 0)
    return launch_kernel(fp8blk_moe_gather_kernel<__half>, grid, dim3(F_QUANT_THREADS, 1, 1), 0, stream, 0, true,
                         (const __half*)x, sorted_pairs, (uint8_t*)codes, s_x, rows, top_k, K, fp8blk_mp(rows));
  return launch_kernel(fp8blk_moe_gather_kernel<__nv_bfloat16>, grid, dim3(F_QUANT_THREADS, 1, 1), 0, stream, 0, true,
                       (const __nv_bfloat16*)x, sorted_pairs, (uint8_t*)codes, s_x, rows, top_k, K, fp8blk_mp(rows));
}

template <int NTOK, int MODE>
static int launch_fp8blk_moe_t(const Fp8BlkArgs& a, const Fp8BlkMoe& g, const SwapPlan& p) {
  using C = FblkCfg<NTOK, MODE>;
  const int KB = a.K / F_BK;
  const int wbox = MODE == 1 ? F_BF / 2 : F_BF;
  FblkMoeArgs G = {};
  CUtensorMap tw, tq, ts;
  if (make_tmap_2d(&tw, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.weight, a.K, g.E * a.N, (size_t)a.K, F_BK, wbox,
                   CU_TENSOR_MAP_SWIZZLE_128B) != 0)
    return -1;
  if (MODE == 1 && make_tmap_2d(&G.tmap_w3, CU_TENSOR_MAP_DATA_TYPE_UINT8, g.w3, a.K, g.E * a.N, (size_t)a.K, F_BK, wbox,
                                CU_TENSOR_MAP_SWIZZLE_128B) != 0)
    return -1;
  if (make_tmap_2d(&tq, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.codes, a.K, a.M, (size_t)a.K, F_BK, NTOK,
                   CU_TENSOR_MAP_SWIZZLE_128B) != 0)
    return -1;
  if (make_tmap_2d(&ts, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, a.s_x, a.M, KB, (size_t)fp8blk_mp(a.M) * 4, C::SX_BYTES / 4, 1,
                   CU_TENSOR_MAP_SWIZZLE_NONE) != 0)
    return -1;
  G.route = {g.counts, g.offsets, g.sorted_pairs, g.pair_weights, g.ypair, p.tblocks, 0};
  G.s_w3 = g.s_w3;
  auto kern = fp8blk_moe_gemm_kernel<NTOK, MODE>;
  static int smem_opted[32] = {};
  if (int e = ensure_dyn_smem(kern, C::SMEM_BYTES, smem_opted, "b2q_fp8blk_moe")) return e;
  const int tiles = (a.N + wbox - 1) / wbox;
  return launch_split_z((long long)g.E * p.tblocks, [&](int z0, int grid_z) {
    G.route.z0 = z0;
    return launch_kernel(kern, dim3(tiles, p.ks, grid_z), dim3(F_THREADS, 1, 1), C::SMEM_BYTES, a.stream, p.ks, true, tw,
                         tq, ts, a.s_w, a.out, a.M, a.K, a.N, p.kpc, a.dtype, G);
  });
}

int launch_fp8blk_moe(int mode, const Fp8BlkArgs& a, const Fp8BlkMoe& g) {
  // a pinned ks is taken as given, like b2q_fp8blk_mm's, so both run the same split
  const SwapPlan p = fp8blk_plan(mode, a.M, a.K, a.N, g.active, a.ks);
#define B2Q_FBM(MODE)                                                    \
  switch (p.ntok) {                                                       \
    case 8: return launch_fp8blk_moe_t<8, MODE>(a, g, p);                 \
    case 16: return launch_fp8blk_moe_t<16, MODE>(a, g, p);               \
    case 32: return launch_fp8blk_moe_t<32, MODE>(a, g, p);               \
    case 64: return launch_fp8blk_moe_t<64, MODE>(a, g, p);               \
    default: return launch_fp8blk_moe_t<128, MODE>(a, g, p);              \
  }
  if (mode == 1) B2Q_FBM(1)
  B2Q_FBM(2)
#undef B2Q_FBM
}

}  // namespace b2q
