// b2q_gemm.cuh — tile geometry of the wgmma prefill kernel (b2q_gemm.cu).
#pragma once
#include "b2q_common.cuh"

namespace b2q {

constexpr int G_BM = 128;  // tokens per CTA tile (two m64 wgmma blocks)
constexpr int G_BN = 128;  // features per CTA tile (wgmma N)
constexpr int G_BK = 64;
constexpr int G_MMA_THREADS = 128;  // warps 0..3: the wgmma warpgroup (+ epilogue)
constexpr int G_DQ_THREADS = 128;   // warps 4..7: dequant warpgroup
constexpr int G_THREADS = G_MMA_THREADS + G_DQ_THREADS + 32;  // + warp 8: TMA / bulk-copy producer

template <int BITS, int STAGES>
struct GemmCfg {
  static constexpr int SUB = BITS / 4;
  static constexpr int A_BYTES = G_BM * G_BK * 2;
  static constexpr int B_BYTES = G_BN * G_BK * 2;
  static constexpr int P_CHUNK_BYTES = 4 * SUB * 512;  // 8-bit: 4 feature tiles (of 32) x 32 k
  // 128 features x 64 k of packed codes (4-bit: one 4 KB T4 row block) + for 4-bit the scale / zero-point rows of
  // the (up to 2) groups of the block: 2 x (256 B scales + 64 B packed zeros), staged by the producer
  static constexpr int P_BYTES = 2 * P_CHUNK_BYTES + (BITS == 4 ? 1024 : 0);
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES + P_BYTES;
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + BAR_BYTES + 1024;
  static_assert(SMEM_BYTES <= 227 * 1024, "dynamic shared memory of one CTA");
};

// Sibling QuantLinears that consume the SAME activations (q|k|v, gate|up) share ONE launch: the 128-feature tile columns
// of all sets form one index space (tn_end = running totals).
constexpr int G_MAX_SETS = 3;
struct GemmSets {
  int nsets;
  int tn_end[G_MAX_SETS];
  int N[G_MAX_SETS];
  const uint4* packed[G_MAX_SETS];
  const void* scales[G_MAX_SETS];
  const uint32_t* qzeros[G_MAX_SETS];
  const void* bias[G_MAX_SETS];
  void* out[G_MAX_SETS];
};

}  // namespace b2q
