// b2q_fp8ch.cu — per-channel / per-tensor 8-bit W8A8 tier: 8-bit weights with one fp32 scale per output feature times
// per-token (dynamic) or per-tensor (static) 8-bit activations on the 8-bit tensor cores.  Two formats share the GEMM:
// e4m3 (compressed-tensors FP8 / FP8_DYNAMIC, fbgemm_fp8) and int8 (compressed-tensors int-quantized W8A8).
// include/b2q.h states the arithmetic of both.  Kernels:
//   * fp8ch_quant_kernel: one CTA per token row: amax over the whole row, s_x = max(min(amax, ub), 1e-10) / 448 (IEEE
//     division), codes = e4m3_rn_satfinite(x / s_x) (fblk_code8, IEEE division), written as uint8 [M, K] and fp32 [M].
//   * fp8ch_static_quant_kernel: elementwise codes = e4m3_rn_satfinite(x / s_in), s_x[m] = s_in.
//   * int8ch_quant_kernel / int8ch_static_quant_kernel: the same two with s_x = max(amax, 1e-10) / 127 and int8 codes
//     clamp(rint(x / s_x), -128, 127) (int8_code8).
//   * fp8ch_gemm_kernel: the pipeline of fp8blk_gemm_kernel (b2q_fp8blk.cu) with the scales taken out of the k-loop:
//     warp 8 loads 128 features x 128 k of the checkpoint weight [N, K] and NTOK x 128 activation codes per k-block with
//     TMA, warpgroups 0 / 1 multiply features 0..63 / 64..127 on m64nNk32.f32.e4m3.e4m3 into a per-block fp32 P that is
//     added to the fp32 accumulator once per k-block (acc += P).  The `ks` CTAs of a cluster split the k-blocks in
//     contiguous runs and sum their partials over distributed shared memory in rank order; the epilogue then applies
//     y = T(acc * (s_x[m] * s_w[n]) + bias[n]), one rounding.
//     Static-scale decode (M <= 8, MODE 1 / 2): no quantiser launch.  Warp 8 quantises each k-block it hands to the MMA
//     warps with the layer's s_in and fblk_code8, so the codes equal fp8ch_static_quant_kernel's.  Per-token scales
//     depend on the whole row, which a split-K rank does not read: their decode runs fp8ch_quant_kernel and the GEMM under
//     programmatic dependent launch, which measured faster than finding the row amax inside the GEMM (DESIGN.md).
//   * int8ch_gemm_kernel: the same body (ch_gemm_body MODE 3) on m64nNk32.s32.s8.s8 into int32 registers that
//     accumulate across all of the rank's k-blocks (integer sums are exact, so there is no per-block promotion), an
//     integer DSMEM reduction, and float(acc) once in the same epilogue.  Both int8 activation kinds run a quantiser and
//     the GEMM under programmatic dependent launch at every M.
//   * fp8ch_moe_gemm_kernel / int8ch_moe_gemm_kernel: grouped modes of the same body for MoE experts (GM 1 / 2):
//     z0 + blockIdx.z = (expert, token block) over the expert-sorted rows that b2q_moe_align ordered; the weights are
//     the stacked checkpoint codes [E*N, K] and scales [E, N].  GM 1 pairs 64 gate features (w1, warpgroup 0) with the
//     same 64 up features (w3, warpgroup 1) in one 128-row tile and stores h = T(T(silu(T(g))) * T(u)); GM 2 (down)
//     stores w[pair] * T(yp) in fp32 to the pair's row of ypair.
//   * fp8ch_moe_gather_kernel / int8ch_moe_gather_kernel: the layer quantisers' row code over the sorted rows, row i
//     reading token sorted_pairs[i] / top_k (or row i of an already sorted x), with per-token scales or the static
//     input scale of the row's expert.
#include <cuda.h>

#include <type_traits>

#include "b2q_common.cuh"
#include "b2q_internal.h"
#include "b2q_wgmma.cuh"

namespace b2q {

constexpr int C_BF = 128;                 // features per tile
constexpr int C_BK = 128;                 // k per block (one SWIZZLE_128B row of e4m3)
constexpr int C_MMA_THREADS = 256;        // warps 0..7: two MMA warpgroups
constexpr int C_THREADS = C_MMA_THREADS + 32;  // + warp 8: producer
constexpr int C_QUANT_THREADS = 256;      // quantisers

template <int NTOK>
struct FchCfg {
  static constexpr int ST = NTOK == 128 ? 6 : 8;  // stages
  static constexpr int W_BYTES = C_BF * C_BK;
  static constexpr int X_BYTES = NTOK * C_BK;
  static constexpr int STAGE_BYTES = W_BYTES + X_BYTES;
  static constexpr int SX_BYTES = 128 * 4;  // the token scales of the CTA's rows (NTOK <= 128)
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = ST * STAGE_BYTES + SX_BYTES + BAR_BYTES + 1024;
  static constexpr int ACC = NTOK / 2;
  static_assert(STAGE_BYTES % 1024 == 0, "stages must stay 1024-byte aligned (SWIZZLE_128B atoms)");
  static_assert(NTOK * C_BF * 4 <= ST * STAGE_BYTES, "the fp32 partial tile reuses the stages");
  static_assert(2 * ST * 8 <= BAR_BYTES, "mbarrier area");
  static_assert(SMEM_BYTES <= 227 * 1024, "dynamic shared memory of one CTA");
};

// ------------------------------------------------------------------------------------------------
// quantisers
// ------------------------------------------------------------------------------------------------
// max |x| of eight elements
template <typename T>
__device__ __forceinline__ float amax8(const uint4& v) {
  const T* h = reinterpret_cast<const T*>(&v);
  float a = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) a = fmaxf(a, fabsf(ET<T>::to_f(h[e])));
  return a;
}
__device__ __forceinline__ float warp_max(float a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
  return a;
}

// eight int8 codes clamp(rint(x / s), -128, 127) (IEEE division, round half to even), packed in k order
template <typename T>
__device__ __forceinline__ uint2 int8_code8(const uint4& v, float s) {
  const T* h = reinterpret_cast<const T*>(&v);
  uint32_t w[2] = {0u, 0u};
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float q = fminf(fmaxf(rintf(__fdiv_rn(ET<T>::to_f(h[e]), s)), -128.f), 127.f);
    w[e >> 2] |= ((uint32_t)(int)q & 0xFFu) << (8 * (e & 3));
  }
  return make_uint2(w[0], w[1]);
}

// the codes of eight elements with the scale s: int8 (S8) or e4m3
template <typename T, bool S8>
__device__ __forceinline__ uint2 ch_code8(const uint4& v, float s) {
  if constexpr (S8) return int8_code8<T>(v, s);
  else return fblk_code8<T>(v, s);
}

// the row body of the per-token quantisers, shared by the layer kernels and the MoE gather so their codes are identical:
// a CTA of C_QUANT_THREADS reads row x + xrow (K elements), finds the amax, writes the codes to codes + crow and returns
// the row scale: int8 (S8) max(amax, 1e-10) / 127, e4m3 max(min(amax, ub), 1e-10) / 448 (IEEE divisions)
template <typename T, bool S8, typename C>
__device__ __forceinline__ float ch_quant_row(const T* __restrict__ x, size_t xrow, C* __restrict__ codes, size_t crow,
                                              int K, float ub) {
  __shared__ float red[C_QUANT_THREADS / 32];
  const uint4* xr = reinterpret_cast<const uint4*>(x + xrow);
  const int n8 = K / 8;
  float a = 0.f;
  for (int o = threadIdx.x; o < n8; o += C_QUANT_THREADS) a = fmaxf(a, amax8<T>(xr[o]));
  a = warp_max(a);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  a = 0.f;
#pragma unroll
  for (int w = 0; w < C_QUANT_THREADS / 32; ++w) a = fmaxf(a, red[w]);
  float s;
  if constexpr (S8) s = fmaxf(a, 1e-10f) / 127.f;  // IEEE division
  else s = fmaxf(fminf(a, ub), 1e-10f) / 448.f;     // IEEE division; ub = +inf: no bound
  uint2* cr = reinterpret_cast<uint2*>(codes + crow);
  for (int o = threadIdx.x; o < n8; o += C_QUANT_THREADS) cr[o] = ch_code8<T, S8>(xr[o], s);
  return s;
}

// one CTA per token row m
template <typename T>
__global__ void __launch_bounds__(C_QUANT_THREADS)
    fp8ch_quant_kernel(const T* __restrict__ x, uint8_t* __restrict__ codes, float* __restrict__ s_x, int K, float ub) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // x is the previous kernel's output
  const size_t row = (size_t)blockIdx.x * K;
  const float s = ch_quant_row<T, false>(x, row, codes, row, K, ub);
  if (threadIdx.x == 0) s_x[blockIdx.x] = s;
}

// elementwise over the M * K / 8 eight-element chunks; thread g < M also writes s_x[g] = s_in
template <typename T>
__global__ void __launch_bounds__(C_QUANT_THREADS)
    fp8ch_static_quant_kernel(const T* __restrict__ x, const float* __restrict__ s_in, uint8_t* __restrict__ codes,
                              float* __restrict__ s_x, int M, long long n8) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const long long g = (long long)blockIdx.x * C_QUANT_THREADS + threadIdx.x;
  const float s = *s_in;
  if (g < n8) reinterpret_cast<uint2*>(codes)[g] = ch_code8<T, false>(reinterpret_cast<const uint4*>(x)[g], s);
  if (g < M) s_x[g] = s;
}

// one CTA per token row m: s_x = max(amax, 1e-10) / 127; an all-zero row gets codes 0 and a finite scale
template <typename T>
__global__ void __launch_bounds__(C_QUANT_THREADS)
    int8ch_quant_kernel(const T* __restrict__ x, int8_t* __restrict__ codes, float* __restrict__ s_x, int K) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // x is the previous kernel's output
  const size_t row = (size_t)blockIdx.x * K;
  const float s = ch_quant_row<T, true>(x, row, codes, row, K, 0.f);
  if (threadIdx.x == 0) s_x[blockIdx.x] = s;
}

// elementwise over the M * K / 8 eight-element chunks; thread g < M also writes s_x[g] = s_in
template <typename T>
__global__ void __launch_bounds__(C_QUANT_THREADS)
    int8ch_static_quant_kernel(const T* __restrict__ x, const float* __restrict__ s_in, int8_t* __restrict__ codes,
                               float* __restrict__ s_x, int M, long long n8) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const long long g = (long long)blockIdx.x * C_QUANT_THREADS + threadIdx.x;
  const float s = *s_in;
  if (g < n8) reinterpret_cast<uint2*>(codes)[g] = ch_code8<T, true>(reinterpret_cast<const uint4*>(x)[g], s);
  if (g < M) s_x[g] = s;
}

// the quantiser over the expert-sorted rows of a MoE block, one CTA per row i: it reads token sorted_pairs[i] / top_k of
// x [T, K] (sorted_pairs == nullptr: row i of x [rows, K], already in sorted order, e.g. h).  Dynamic (s_in ==
// nullptr): the per-token row body; static: the scale s_in[e] of the expert e whose rows hold i.  So row i's codes and
// scale are those the layer quantiser gives its token (static: with that expert's input_scale).
template <typename T, bool S8>
__device__ __forceinline__ void ch_moe_gather_body(const T* __restrict__ x, const int32_t* __restrict__ sorted_pairs,
                                                   const int32_t* __restrict__ offsets, const float* __restrict__ s_in,
                                                   int E, uint8_t* __restrict__ codes, float* __restrict__ s_x, int top_k,
                                                   int K, float ub) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // the routing tables (and x) are the previous kernels' output
  const int i = blockIdx.x;
  const int r = sorted_pairs != nullptr ? sorted_pairs[i] / top_k : i;
  float s;
  if (s_in == nullptr) {
    s = ch_quant_row<T, S8>(x, (size_t)r * K, codes, (size_t)i * K, K, ub);
  } else {
    const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)r * K);
    uint2* cr = reinterpret_cast<uint2*>(codes + (size_t)i * K);
    // the last expert whose first row is <= i (an expert without rows has the offset of the next one)
    int lo = 0, hi = E;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (offsets[mid] <= i) lo = mid + 1;
      else hi = mid;
    }
    s = s_in[lo > 0 ? lo - 1 : 0];
    for (int o = threadIdx.x; o < K / 8; o += C_QUANT_THREADS) cr[o] = ch_code8<T, S8>(xr[o], s);
  }
  if (threadIdx.x == 0) s_x[i] = s;
}

template <typename T>
__global__ void __launch_bounds__(C_QUANT_THREADS)
    fp8ch_moe_gather_kernel(const T* __restrict__ x, const int32_t* __restrict__ sorted_pairs,
                            const int32_t* __restrict__ offsets, const float* __restrict__ s_in, int E,
                            uint8_t* __restrict__ codes, float* __restrict__ s_x, int top_k, int K, float ub) {
  ch_moe_gather_body<T, false>(x, sorted_pairs, offsets, s_in, E, codes, s_x, top_k, K, ub);
}

template <typename T>
__global__ void __launch_bounds__(C_QUANT_THREADS)
    int8ch_moe_gather_kernel(const T* __restrict__ x, const int32_t* __restrict__ sorted_pairs,
                             const int32_t* __restrict__ offsets, const float* __restrict__ s_in, int E,
                             uint8_t* __restrict__ codes, float* __restrict__ s_x, int top_k, int K) {
  ch_moe_gather_body<T, true>(x, sorted_pairs, offsets, s_in, E, codes, s_x, top_k, K, 0.f);
}

// ------------------------------------------------------------------------------------------------
// GEMM
// ------------------------------------------------------------------------------------------------
// four consecutive outputs of features nc .. nc + 3: T(acc * (sx * s_w[n]) + bias[n]), rounded once; bias [N] or nullptr
template <typename T>
__device__ __forceinline__ void store_scaled4(T* dst, const float* __restrict__ s_w, const T* bias, int nc, float sx,
                                              const float (&a)[4]) {
  using E = ET<T>;
  const float4 sw = *reinterpret_cast<const float4*>(s_w + nc);
  const float w4[4] = {sw.x, sw.y, sw.z, sw.w};
  float y[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    y[i] = __fmul_rn(a[i], __fmul_rn(sx, w4[i]));  // no contraction into an fma with the bias
    if (bias != nullptr) y[i] = __fadd_rn(y[i], E::to_f(bias[nc + i]));
  }
  *reinterpret_cast<uint2*>(dst) = make_uint2(E::pack2(y[0], y[1]), E::pack2(y[2], y[3]));
}

// four fp32 products acc * (sx * s_w[n]) of features nc .. nc + 3, not rounded: the grouped epilogues' g, u and yp
__device__ __forceinline__ void scale4(float (&y)[4], const float* __restrict__ s_w, int nc, float sx,
                                       const float (&a)[4]) {
  const float4 sw = *reinterpret_cast<const float4*>(s_w + nc);
  const float w4[4] = {sw.x, sw.y, sw.z, sw.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) y[i] = __fmul_rn(a[i], __fmul_rn(sx, w4[i]));
}

// grouped launches (GM 1 / 2) over the experts of a MoE block
struct ChMoeArgs {
  CUtensorMap tmap_w3;  // GM 1: the w3 stack [E*N, K], 64-row boxes (tmap_w: the w1 stack, the same boxes)
  MoeRoute route;
  const float* s_w3;    // GM 1: [E, N] scales of w3
};

// MODE: 0 = e4m3 codes and token scales come from a quantiser kernel (TMA for the codes); 1 / 2 = M <= 8, x fp16 / bf16
// is quantised to e4m3 by the producer with the static scale s_in; 3 = int8 codes and token scales from a quantiser.
// GM (orthogonal to the code type of MODE 0 / 3): 0 = one layer; 1 = grouped gate|up, 64 gate features of the w1 stack
// (warpgroup 0) and the same 64 up features of the w3 stack (warpgroup 1) per tile, h = T(T(silu(T(g))) * T(u)) into
// out; 2 = grouped down, w[pair] * T(yp) in fp32 to the pair's row of G->route.ypair.  Grouped: z0 + blockIdx.z =
// (expert e, token block) over the expert-sorted rows, weights [E*N, K] and s_w [E, N]; no bias.
template <int NTOK, int MODE, int GM = 0>
__device__ __forceinline__ void ch_gemm_body(const CUtensorMap& tmap_w, const CUtensorMap& tmap_q,
                                             const void* __restrict__ x, const float* __restrict__ s_x,
                                             const float* __restrict__ s_in, const float* __restrict__ s_w,
                                             const void* __restrict__ bias, void* __restrict__ out, int M, int K, int N,
                                             int kpc, int out_bf16, const ChMoeArgs* G = nullptr) {
  using C = FchCfg<NTOK>;
  constexpr int ST = C::ST;
  constexpr bool FUSED = MODE == 1 || MODE == 2, S8 = MODE == 3;
  static_assert(!FUSED || NTOK == 8, "the fused quantiser serves 8-token tiles");
  static_assert(GM == 0 || !FUSED, "the grouped modes read quantised codes");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
  // stage s: [W 128 x 128][X NTOK x 128]; then the token scales and the barriers
  float* sxr = reinterpret_cast<float*>(smem + ST * C::STAGE_BYTES);
  const uint32_t bar_full = smem_base + ST * C::STAGE_BYTES + C::SX_BYTES, bar_empty = bar_full + 8 * ST;
  auto sW = [&](int s) { return smem_base + (uint32_t)(s * C::STAGE_BYTES); };
  auto sX = [&](int s) { return sW(s) + C::W_BYTES; };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * (GM == 1 ? C_BF / 2 : C_BF);  // GM 1: 64 gate + 64 up features
  int row0 = blockIdx.z * NTOK, rows = min(NTOK, M - row0);
  int e = 0;  // expert (grouped modes)
  if constexpr (GM != 0) {
    if (!moe_block<NTOK>(G->route, e, row0, rows)) return;
  }
  const int wrow = GM == 0 ? n0 : e * N + n0;  // first row of the tile in the (stacked) weight tensor
  const int KB = K / C_BK;
  const uint32_t nrank = cluster_nctarank(), crank = cluster_ctarank();
  const int kb0 = min(KB, (int)crank * kpc), kb1 = min(KB, kb0 + kpc);
  const int nkb = kb1 - kb0;

  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_w);
    if constexpr (GM == 1) prefetch_tmap(&G->tmap_w3);
    if (!FUSED) prefetch_tmap(&tmap_q);
    for (int s = 0; s < ST; ++s) {
      mbar_init(bar_full + 8 * s, FUSED ? 32 : 1);
      mbar_init(bar_empty + 8 * s, C_MMA_THREADS / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  auto load_weights = [&](int i, int s) {
    mbar_expect_tx_only(bar_full + 8 * s, C::W_BYTES);
    tma_load_2d(sW(s), &tmap_w, bar_full + 8 * s, (kb0 + i) * C_BK, wrow);
    // GM 1: the up features' 64-row box fills the second m64 half of the tile
    if constexpr (GM == 1) tma_load_2d(sW(s) + C::W_BYTES / 2, &G->tmap_w3, bar_full + 8 * s, (kb0 + i) * C_BK, wrow);
  };
  // the weight stream of the first ST blocks starts at once (under programmatic dependent launch: while the previous
  // kernel still runs)
  if (warp == 8 && lane == 0)
    for (int i = 0; i < nkb && i < ST; ++i) load_weights(i, i);
  asm volatile("griddepcontrol.wait;" ::: "memory");  // x / codes / s_x are the previous kernels' output

  // the scales of the CTA's token rows -> sxr (rows past M: 0)
  if (!FUSED) {
    for (int t = threadIdx.x; t < NTOK; t += C_THREADS) sxr[t] = t < rows ? s_x[row0 + t] : 0.f;
  } else if (threadIdx.x < NTOK) {
    sxr[threadIdx.x] = (int)threadIdx.x < M ? *s_in : 0.f;
  }
  __syncthreads();

  if (warp == 8) {
    // ================================ producer ================================
    if constexpr (FUSED) {
      using T = typename std::conditional<MODE == 1, __half, __nv_bfloat16>::type;
      // half-warp h of pass p holds token t = 2 p + h, lane j = lane & 15 its elements 8 j .. 8 j + 7 of the k-block;
      // rows t >= M keep the zero codes written here once
      constexpr int PD = 4;  // k-blocks of activations in flight ahead of the one being quantised
      const int h = lane >> 4, j = lane & 15;
      for (int s = 0; s < ST; ++s)
        for (int o = lane; o < C::X_BYTES / 16; o += 32)
          asm volatile("st.shared.v4.u32 [%0], {%1,%1,%1,%1};" ::"r"(sX(s) + 16u * o), "r"(0u) : "memory");
      float sc[4];
#pragma unroll
      for (int p = 0; p < 4; ++p) sc[p] = sxr[2 * p + h];
      const T* xr = reinterpret_cast<const T*>(x) + (size_t)kb0 * C_BK + 8 * j;
      uint4 buf[PD][4];  // [in-flight k-block][pass]
      auto fetch = [&](int i, uint4(&dst)[4]) {
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const int t = 2 * p + h;
          dst[p] = (t < M && i < nkb) ? *reinterpret_cast<const uint4*>(xr + (size_t)t * K + (size_t)i * C_BK)
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
            const int t = 2 * p + h;
            if (t < M) {
              const uint2 q = fblk_code8<T>(cur[p], sc[p]);
              const uint32_t addr = sX(s) + (uint32_t)t * 128 + ((((uint32_t)(j >> 1)) ^ (uint32_t)t) << 4) + 8u * (j & 1);
              asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(addr), "r"(q.x), "r"(q.y) : "memory");
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
        mbar_expect_tx(bar_full + 8 * s, C::X_BYTES);
        tma_load_2d(sX(s), &tmap_q, bar_full + 8 * s, (kb0 + i) * C_BK, row0);
      }
    }
  } else if constexpr (S8) {
    // ================================ MMA warpgroups, int8 ================================
    // the int32 sums are exact (|acc| <= 2^30 for K <= 65536), so every k-block accumulates into the same registers
    const int wg = warp >> 2;
    int acc[C::ACC];
#pragma unroll
    for (int v = 0; v < C::ACC; ++v) acc[v] = 0;
    for (int i = 0; i < nkb; ++i) {
      const int s = i % ST;
      mbar_wait(bar_full + 8 * s, (i / ST) & 1);
      const uint64_t wdesc = wgmma_desc_k_sw128(sW(s)) + 512 * wg;
      const uint64_t xdesc = wgmma_desc_k_sw128(sX(s));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < C_BK / 32; ++k) Wgmma8<NTOK>::mma(acc, wdesc + 2 * k, xdesc + 2 * k, 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * s);
    }
    asm volatile("bar.sync 1, %0;" ::"r"(C_MMA_THREADS) : "memory");
    park_partial(smem_base, wg, warp & 3, acc);
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
      for (int k = 0; k < C_BK / 32; ++k) Wgmma8F<NTOK>::mma(p, wdesc + 2 * k, xdesc + 2 * k, k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(p);
      // promotion: the block's product joins the fp32 accumulator (no per-block scale)
#pragma unroll
      for (int v = 0; v < C::ACC; ++v) acc[v] += p[v];
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * s);
    }
    // both warpgroups are done with the stages before either overwrites them with its partial tile
    asm volatile("bar.sync 1, %0;" ::"r"(C_MMA_THREADS) : "memory");
    park_partial(smem_base, wg, warp & 3, acc);
  }
  __syncwarp();
  cluster_sync_all();
  if (GM == 1 && warp < C_MMA_THREADS / 32) {
    // rank z reduces token rows z, z + nrank, ... , a half-warp per row: lane l holds gate features 4 (l & 15) .. + 3 of
    // the tile (those columns of h) and their up features at + 64
    const int hw = 2 * warp + (lane >> 4), c = lane & 15, nc = e * N + n0 + 4 * c;
    for (int tok = (int)crank + (int)nrank * hw; tok < rows; tok += (int)nrank * (2 * C_MMA_THREADS / 32)) {
      float gu[2][4];
      if constexpr (S8) {
        int ia[2][4];
        dsmem_sum4<2, true>(smem_base + (uint32_t)tok * (C_BF * 4) + (uint32_t)c * 16, (C_BF / 2) * 4, nrank, ia);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < 4; ++i) gu[h][i] = __int2float_rn(ia[h][i]);  // one rounding of the exact sum
      } else {
        dsmem_sum4<2, false>(smem_base + (uint32_t)tok * (C_BF * 4) + (uint32_t)c * 16, (C_BF / 2) * 4, nrank, gu);
      }
      float g[4], u[4];
      scale4(g, s_w, nc, sxr[tok], gu[0]);
      scale4(u, G->s_w3, nc, sxr[tok], gu[1]);
      const size_t o = (size_t)(row0 + tok) * N + n0 + 4 * c;
      if (out_bf16) store_silu_mul4(reinterpret_cast<__nv_bfloat16*>(out) + o, g, u);
      else store_silu_mul4(reinterpret_cast<__half*>(out) + o, g, u);
    }
  } else if (GM == 2 && warp < C_MMA_THREADS / 32) {
    // rank z reduces token rows z, z + nrank, ... , a warp per row
    const int nc = n0 + lane * 4;
    if (nc < N) {
      for (int tok = (int)crank + (int)nrank * warp; tok < rows; tok += (int)nrank * (C_MMA_THREADS / 32)) {
        float a[1][4];
        if constexpr (S8) {
          int ia[1][4];
          dsmem_sum4<1, true>(smem_base + (uint32_t)tok * (C_BF * 4) + (uint32_t)lane * 16, 0, nrank, ia);
#pragma unroll
          for (int i = 0; i < 4; ++i) a[0][i] = __int2float_rn(ia[0][i]);
        } else {
          dsmem_sum4<1, false>(smem_base + (uint32_t)tok * (C_BF * 4) + (uint32_t)lane * 16, 0, nrank, a);
        }
        float yp[4];
        scale4(yp, s_w, e * N + nc, sxr[tok], a[0]);
        const int pair = G->route.sorted_pairs[row0 + tok];
        float* y = G->route.ypair + (size_t)pair * N + nc;
        if (out_bf16) store_ypair4<__nv_bfloat16>(y, G->route.pair_weights[pair], yp);
        else store_ypair4<__half>(y, G->route.pair_weights[pair], yp);
      }
    }
  } else if (GM == 0 && warp < C_MMA_THREADS / 32) {
    // rank z reduces token rows z, z + nrank, ... , a warp per row
    const int nc = n0 + lane * 4;
    if (nc < N) {
      for (int tok = (int)crank + (int)nrank * warp; tok < rows; tok += (int)nrank * (C_MMA_THREADS / 32)) {
        float a[1][4];
        if constexpr (S8) {
          int ia[1][4];
          dsmem_sum4<1, true>(smem_base + (uint32_t)tok * (C_BF * 4) + (uint32_t)lane * 16, 0, nrank, ia);
#pragma unroll
          for (int e = 0; e < 4; ++e) a[0][e] = __int2float_rn(ia[0][e]);  // one rounding of the exact sum
        } else {
          dsmem_sum4<1, false>(smem_base + (uint32_t)tok * (C_BF * 4) + (uint32_t)lane * 16, 0, nrank, a);
        }
        const size_t o = (size_t)(row0 + tok) * N + nc;
        if (out_bf16)
          store_scaled4(reinterpret_cast<__nv_bfloat16*>(out) + o, s_w, reinterpret_cast<const __nv_bfloat16*>(bias),
                        nc, sxr[tok], a[0]);
        else
          store_scaled4(reinterpret_cast<__half*>(out) + o, s_w, reinterpret_cast<const __half*>(bias), nc, sxr[tok],
                        a[0]);
      }
    }
  }
  __syncwarp();
  cluster_sync_all();  // keep every rank's shared memory alive until all peers have read it
}

// FUSED: 0 = e4m3 codes from a quantiser; 1 / 2 = static-scale decode of fp16 / bf16 x (MODE of ch_gemm_body)
template <int NTOK, int FUSED>
__global__ void __launch_bounds__(C_THREADS, 1)
    fp8ch_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_q,
                      const void* __restrict__ x, const float* __restrict__ s_x, const float* __restrict__ s_in,
                      const float* __restrict__ s_w, const void* __restrict__ bias, void* __restrict__ out, int M, int K,
                      int N, int kpc, int out_bf16) {
  ch_gemm_body<NTOK, FUSED>(tmap_w, tmap_q, x, s_x, s_in, s_w, bias, out, M, K, N, kpc, out_bf16);
}

// grouped launches over the experts of a MoE block (GM 1 = gate|up, 2 = down): M = rows, N / K of one expert,
// out = h (GM 1); e4m3 codes and weights
template <int NTOK, int GM>
__global__ void __launch_bounds__(C_THREADS, 1)
    fp8ch_moe_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_q,
                          const float* __restrict__ s_x, const float* __restrict__ s_w, void* __restrict__ out, int M,
                          int K, int N, int kpc, int out_bf16, const __grid_constant__ ChMoeArgs G) {
  ch_gemm_body<NTOK, 0, GM>(tmap_w, tmap_q, nullptr, s_x, nullptr, s_w, nullptr, out, M, K, N, kpc, out_bf16, &G);
}

// int8 codes from int8ch_quant_kernel / int8ch_static_quant_kernel and int8 weights
template <int NTOK>
__global__ void __launch_bounds__(C_THREADS, 1)
    int8ch_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_q,
                       const void* __restrict__ x, const float* __restrict__ s_x, const float* __restrict__ s_in,
                       const float* __restrict__ s_w, const void* __restrict__ bias, void* __restrict__ out, int M,
                       int K, int N, int kpc, int out_bf16) {
  ch_gemm_body<NTOK, 3>(tmap_w, tmap_q, x, s_x, s_in, s_w, bias, out, M, K, N, kpc, out_bf16);
}

// the grouped launches on int8 codes and weights
template <int NTOK, int GM>
__global__ void __launch_bounds__(C_THREADS, 1)
    int8ch_moe_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_q,
                           const float* __restrict__ s_x, const float* __restrict__ s_w, void* __restrict__ out, int M,
                           int K, int N, int kpc, int out_bf16, const __grid_constant__ ChMoeArgs G) {
  ch_gemm_body<NTOK, 3, GM>(tmap_w, tmap_q, nullptr, s_x, nullptr, s_w, nullptr, out, M, K, N, kpc, out_bf16, &G);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int launch_fp8ch_quant(const void* x, void* codes, float* s_x, int M, int K, float ub, int dtype, cudaStream_t stream) {
  const dim3 grid((unsigned)M, 1, 1), block(C_QUANT_THREADS, 1, 1);
  if (dtype == 0)
    return launch_kernel(fp8ch_quant_kernel<__half>, grid, block, 0, stream, 0, true, (const __half*)x, (uint8_t*)codes,
                         s_x, K, ub);
  return launch_kernel(fp8ch_quant_kernel<__nv_bfloat16>, grid, block, 0, stream, 0, true, (const __nv_bfloat16*)x,
                       (uint8_t*)codes, s_x, K, ub);
}

int launch_fp8ch_static_quant(const void* x, const float* s_in, void* codes, float* s_x, int M, int K, int dtype,
                              cudaStream_t stream) {
  const long long n8 = (long long)M * (K / 8), threads = n8 > M ? n8 : M;
  const dim3 grid((unsigned)((threads + C_QUANT_THREADS - 1) / C_QUANT_THREADS), 1, 1), block(C_QUANT_THREADS, 1, 1);
  if (dtype == 0)
    return launch_kernel(fp8ch_static_quant_kernel<__half>, grid, block, 0, stream, 0, true, (const __half*)x, s_in,
                         (uint8_t*)codes, s_x, M, n8);
  return launch_kernel(fp8ch_static_quant_kernel<__nv_bfloat16>, grid, block, 0, stream, 0, true,
                       (const __nv_bfloat16*)x, s_in, (uint8_t*)codes, s_x, M, n8);
}

template <int NTOK, int MODE>
static int launch_fp8ch_gemm_t(const Fp8ChArgs& a, const SwapPlan& p) {
  using C = FchCfg<NTOK>;
  CUtensorMap tw, tq;
  if (make_tmap_2d(&tw, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.weight, a.K, a.N, (size_t)a.K, C_BK, C_BF,
                   CU_TENSOR_MAP_SWIZZLE_128B) != 0)
    return -1;
  if (MODE == 1 || MODE == 2) {
    tq = tw;  // unused
  } else if (make_tmap_2d(&tq, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.codes, a.K, a.M, (size_t)a.K, C_BK, NTOK,
                          CU_TENSOR_MAP_SWIZZLE_128B) != 0) {
    return -1;
  }
  void (*kern)(const CUtensorMap, const CUtensorMap, const void*, const float*, const float*, const float*, const void*,
               void*, int, int, int, int, int);
  if constexpr (MODE == 3)
    kern = int8ch_gemm_kernel<NTOK>;
  else
    kern = fp8ch_gemm_kernel<NTOK, MODE>;
  static int smem_opted[32] = {};
  if (int e = ensure_dyn_smem(kern, C::SMEM_BYTES, smem_opted, "b2q_fp8ch")) return e;
  return launch_kernel(kern, dim3((a.N + C_BF - 1) / C_BF, p.ks, p.tblocks), dim3(C_THREADS, 1, 1), C::SMEM_BYTES,
                       a.stream, p.ks, true, tw, tq, a.x, a.s_x, a.s_in, a.s_w, a.bias, a.out, a.M, a.K, a.N, p.kpc,
                       a.dtype);
}

// the launch plan of the block-FP8 GEMM (same tiles, token blocks and split-K ranks)
int launch_fp8ch_gemm(const Fp8ChArgs& a) {
  const SwapPlan p = fp8blk_plan(0, a.M, a.K, a.N, 1, a.ks);
  if (a.x != nullptr) return a.dtype == 0 ? launch_fp8ch_gemm_t<8, 1>(a, p) : launch_fp8ch_gemm_t<8, 2>(a, p);
  switch (p.ntok) {
    case 8: return launch_fp8ch_gemm_t<8, 0>(a, p);
    case 16: return launch_fp8ch_gemm_t<16, 0>(a, p);
    case 32: return launch_fp8ch_gemm_t<32, 0>(a, p);
    case 64: return launch_fp8ch_gemm_t<64, 0>(a, p);
    default: return launch_fp8ch_gemm_t<128, 0>(a, p);
  }
}

int launch_int8ch_quant(const void* x, void* codes, float* s_x, int M, int K, int dtype, cudaStream_t stream) {
  const dim3 grid((unsigned)M, 1, 1), block(C_QUANT_THREADS, 1, 1);
  if (dtype == 0)
    return launch_kernel(int8ch_quant_kernel<__half>, grid, block, 0, stream, 0, true, (const __half*)x, (int8_t*)codes,
                         s_x, K);
  return launch_kernel(int8ch_quant_kernel<__nv_bfloat16>, grid, block, 0, stream, 0, true, (const __nv_bfloat16*)x,
                       (int8_t*)codes, s_x, K);
}

int launch_int8ch_static_quant(const void* x, const float* s_in, void* codes, float* s_x, int M, int K, int dtype,
                               cudaStream_t stream) {
  const long long n8 = (long long)M * (K / 8), threads = n8 > M ? n8 : M;
  const dim3 grid((unsigned)((threads + C_QUANT_THREADS - 1) / C_QUANT_THREADS), 1, 1), block(C_QUANT_THREADS, 1, 1);
  if (dtype == 0)
    return launch_kernel(int8ch_static_quant_kernel<__half>, grid, block, 0, stream, 0, true, (const __half*)x, s_in,
                         (int8_t*)codes, s_x, M, n8);
  return launch_kernel(int8ch_static_quant_kernel<__nv_bfloat16>, grid, block, 0, stream, 0, true,
                       (const __nv_bfloat16*)x, s_in, (int8_t*)codes, s_x, M, n8);
}

// int8 codes (a.x == nullptr): the plan and tiles of the e4m3 GEMM
int launch_int8ch_gemm(const Fp8ChArgs& a) {
  const SwapPlan p = fp8blk_plan(0, a.M, a.K, a.N, 1, a.ks);
  switch (p.ntok) {
    case 8: return launch_fp8ch_gemm_t<8, 3>(a, p);
    case 16: return launch_fp8ch_gemm_t<16, 3>(a, p);
    case 32: return launch_fp8ch_gemm_t<32, 3>(a, p);
    case 64: return launch_fp8ch_gemm_t<64, 3>(a, p);
    default: return launch_fp8ch_gemm_t<128, 3>(a, p);
  }
}

int launch_ch_moe_gather(int s8, const void* x, const int32_t* sorted_pairs, const int32_t* offsets, const float* s_in,
                         int E, void* codes, float* s_x, int rows, int top_k, int K, float ub, int dtype,
                         cudaStream_t stream) {
  const dim3 grid((unsigned)rows, 1, 1), block(C_QUANT_THREADS, 1, 1);
  uint8_t* c = (uint8_t*)codes;
  if (s8) {
    if (dtype == 0)
      return launch_kernel(int8ch_moe_gather_kernel<__half>, grid, block, 0, stream, 0, true, (const __half*)x,
                           sorted_pairs, offsets, s_in, E, c, s_x, top_k, K);
    return launch_kernel(int8ch_moe_gather_kernel<__nv_bfloat16>, grid, block, 0, stream, 0, true,
                         (const __nv_bfloat16*)x, sorted_pairs, offsets, s_in, E, c, s_x, top_k, K);
  }
  if (dtype == 0)
    return launch_kernel(fp8ch_moe_gather_kernel<__half>, grid, block, 0, stream, 0, true, (const __half*)x,
                         sorted_pairs, offsets, s_in, E, c, s_x, top_k, K, ub);
  return launch_kernel(fp8ch_moe_gather_kernel<__nv_bfloat16>, grid, block, 0, stream, 0, true, (const __nv_bfloat16*)x,
                       sorted_pairs, offsets, s_in, E, c, s_x, top_k, K, ub);
}

template <int NTOK, int S8, int GM>
static int launch_ch_moe_t(const Fp8ChArgs& a, const Fp8ChMoe& g, const SwapPlan& p) {
  using C = FchCfg<NTOK>;
  const int wbox = GM == 1 ? C_BF / 2 : C_BF;
  ChMoeArgs G = {};
  CUtensorMap tw, tq;
  if (make_tmap_2d(&tw, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.weight, a.K, g.E * a.N, (size_t)a.K, C_BK, wbox,
                   CU_TENSOR_MAP_SWIZZLE_128B) != 0)
    return -1;
  if (GM == 1 && make_tmap_2d(&G.tmap_w3, CU_TENSOR_MAP_DATA_TYPE_UINT8, g.w3, a.K, g.E * a.N, (size_t)a.K, C_BK, wbox,
                              CU_TENSOR_MAP_SWIZZLE_128B) != 0)
    return -1;
  if (make_tmap_2d(&tq, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.codes, a.K, a.M, (size_t)a.K, C_BK, NTOK,
                   CU_TENSOR_MAP_SWIZZLE_128B) != 0)
    return -1;
  G.route = {g.counts, g.offsets, g.sorted_pairs, g.pair_weights, g.ypair, p.tblocks, 0};
  G.s_w3 = g.s_w3;
  void (*kern)(const CUtensorMap, const CUtensorMap, const float*, const float*, void*, int, int, int, int, int,
               const ChMoeArgs);
  if constexpr (S8)
    kern = int8ch_moe_gemm_kernel<NTOK, GM>;
  else
    kern = fp8ch_moe_gemm_kernel<NTOK, GM>;
  static int smem_opted[32] = {};
  if (int e = ensure_dyn_smem(kern, C::SMEM_BYTES, smem_opted, "b2q_fp8ch_moe")) return e;
  const int tiles = (a.N + wbox - 1) / wbox;
  return launch_split_z((long long)g.E * p.tblocks, [&](int z0, int grid_z) {
    G.route.z0 = z0;
    return launch_kernel(kern, dim3(tiles, p.ks, grid_z), dim3(C_THREADS, 1, 1), C::SMEM_BYTES, a.stream, p.ks, true, tw,
                         tq, a.s_x, a.s_w, a.out, a.M, a.K, a.N, p.kpc, a.dtype, G);
  });
}

template <int S8, int GM>
static int launch_ch_moe_mode(const Fp8ChArgs& a, const Fp8ChMoe& g, const SwapPlan& p) {
  switch (p.ntok) {
    case 8: return launch_ch_moe_t<8, S8, GM>(a, g, p);
    case 16: return launch_ch_moe_t<16, S8, GM>(a, g, p);
    case 32: return launch_ch_moe_t<32, S8, GM>(a, g, p);
    case 64: return launch_ch_moe_t<64, S8, GM>(a, g, p);
    default: return launch_ch_moe_t<128, S8, GM>(a, g, p);
  }
}

// the plan of the grouped block-FP8 launches; a pinned ks is taken as given, like b2q_fp8ch_mm's, so each expert's rows
// run the dense kernel's split
int launch_ch_moe(int mode, int s8, const Fp8ChArgs& a, const Fp8ChMoe& g) {
  const SwapPlan p = fp8blk_plan(mode, a.M, a.K, a.N, g.active, a.ks);
  if (s8) return mode == 1 ? launch_ch_moe_mode<1, 1>(a, g, p) : launch_ch_moe_mode<1, 2>(a, g, p);
  return mode == 1 ? launch_ch_moe_mode<0, 1>(a, g, p) : launch_ch_moe_mode<0, 2>(a, g, p);
}

}  // namespace b2q
