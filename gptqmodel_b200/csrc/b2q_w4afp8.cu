// b2q_w4afp8.cu — W4AFP8 tier (compressed-tensors `W4AFP8`): symmetric 4-bit weights with one scale per 128 k times
// dynamic per-token e4m3 activations on the e4m3 tensor cores.  include/b2q.h states the arithmetic.
//   * the activation codes and token scales come from fp8ch_quant_kernel (b2q_fp8ch.cu, ub = +inf), so they are
//     bit-identical to the per-channel FP8_DYNAMIC layer's;
//   * w4afp8_gemm_kernel: the structure of qqq_gemm_kernel (b2q_qqq.cu) with e4m3 operands.  The WEIGHTS are the wgmma A
//     operand (128 output features; warpgroup 0 multiplies features 0..63, warpgroup 1 features 64..127), the TOKENS the
//     B operand (n = NTOK in {8, 16, 32, 64, 128}); 128-token blocks beyond that are spread over gridDim.z.  A k-block is
//     128 k = one quantisation group = one SWIZZLE_128B row of e4m3.  Thread 0 loads the codes with TMA (a separate
//     producer warp would cap the CTA at 128 registers per thread, which the 128-token accumulators exceed); warps 8..11 form
//     two dequant groups that take alternate k-blocks (so the decode pace is not one group's serial latency chain):
//     each expands the packed 4-bit tile of its block into e4m3 A rows (exact: every integer in [-8, 7] is an e4m3
//     value) and copies the block's 128 group scales beside them.  The MMA warpgroups issue m64nNk32.f32.e4m3.e4m3 into
//     a per-block fp32 P and promote it once per block, acc = fma(P, s_w[n, b], acc).  The `ks` CTAs of a cluster split
//     the k-blocks in contiguous runs and sum their partials over distributed shared memory in rank order; the epilogue
//     applies y = T(acc * s_x[m] + bias[n]), one rounding.  No atomics: the output is deterministic for a given ks.
//
// Packed weights: the grouped tile layout of b2q_qqq_prepack (tile (nt, kb) of 128 features x 128 k is 8 KB at
// ((nt * KB + kb) * 8192), uint4 [4 quads][128 features], a word covering k0 .. k0 + 7 holds k0..3 in nibbles 0, 1, 4, 5
// and k4..7 in nibbles 2, 3, 6, 7), written in one pass from the checkpoint's `weight_packed` (w4afp8_prepack_kernel).
// A nibble is the stored code c = q + 8.
#include <cuda.h>

#include "b2q_common.cuh"
#include "b2q_internal.h"
#include "b2q_wgmma.cuh"

namespace b2q {

constexpr int A_BF = 128;                // features per tile
constexpr int A_BK = 128;                // k per block = one quantisation group
constexpr int A_TILE_BYTES = A_BF * A_BK / 2;
constexpr int A_SC_BYTES = A_BF * 4;     // the fp32 group scales of a tile's features for one block
constexpr int A_MMA_THREADS = 256;       // warps 0..7: two MMA warpgroups
constexpr int A_DQG = 2;                 // dequant groups (warps 8..9 and 10..11), on alternate k-blocks
constexpr int A_DQ_THREADS = 128;
constexpr int A_TG = A_DQ_THREADS / A_DQG;   // threads per dequant group: thread tl expands feature rows tl, tl + 64
constexpr int A_THREADS = A_MMA_THREADS + A_DQ_THREADS;

template <int NTOK>
struct W4fCfg {
  static constexpr int PST = 8;                       // packed stages (8.5 KB): the HBM stream in flight
  static constexpr int WST = 4;                       // expanded e4m3 stages (16 KB)
  static constexpr int XST = 4;                       // activation stages
  static constexpr int W_BYTES = A_BF * A_BK;
  static constexpr int X_BYTES = NTOK * A_BK;
  static constexpr int P_BYTES = A_TILE_BYTES + A_SC_BYTES;  // packed tile | its block's group scales
  static constexpr int BAR_BYTES = 256;
  static constexpr int RING_BYTES = WST * W_BYTES + XST * X_BYTES + PST * P_BYTES + WST * A_SC_BYTES;
  static constexpr int SMEM_BYTES = RING_BYTES + BAR_BYTES + 1024;
  static constexpr int ACC = NTOK / 2;
  static_assert(PST % A_DQG == 0 && WST % A_DQG == 0, "every use of a ring stage must belong to the same dequant group");
  static_assert(X_BYTES % 1024 == 0, "activation tiles must stay 1024-byte aligned (SWIZZLE_128B atoms)");
  static_assert(NTOK * A_BF * 4 <= WST * W_BYTES, "the fp32 partial tile reuses the expanded-weight stages");
  static_assert((PST + 2 * XST + 2 * WST) * 8 <= BAR_BYTES, "mbarrier area");
  static_assert(SMEM_BYTES <= 227 * 1024, "dynamic shared memory of one CTA");
};

// ------------------------------------------------------------------------------------------------
// one-time repack: weight_packed int32 [N, K/8] (code of k in bits 4 (k % 8) of word k / 8) -> the tile layout above
// ------------------------------------------------------------------------------------------------
__global__ void w4afp8_prepack_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ out, int K, int N) {
  const int KB = K / A_BK;
  const size_t words = (size_t)KB * (N / A_BF) * (A_TILE_BYTES / 4);
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < words; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t tile = idx / (A_TILE_BYTES / 4);
    const int r = (int)(idx % (A_TILE_BYTES / 4));  // [quad][feature][word]
    const int quad = r / (A_BF * 4), f = (r / 4) % A_BF, j = r % 4;
    const int nt = (int)(tile / KB), kb = (int)(tile % KB);
    const int n = nt * A_BF + f, k0 = kb * A_BK + 32 * quad + 8 * j;
    const uint32_t w = src[(size_t)n * (K / 8) + k0 / 8];
    uint32_t o = 0;
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      const int kk = (p & 1) | ((p & 2) << 1) | ((p & 4) >> 1);
      o |= ((w >> (4 * kk)) & 15u) << (4 * p);
    }
    out[idx] = o;
  }
}

// ------------------------------------------------------------------------------------------------
// GEMM
// ------------------------------------------------------------------------------------------------
// one packed word (8 k) -> the e4m3 weights q = c - 8 of k0..3 (lo) and k4..7 (hi), in k order
__device__ __forceinline__ void expand_e4m3(uint32_t w, uint32_t& lo, uint32_t& hi) {
  const uint32_t EX = 0x64006400u;   // half2(1024 + nibble)
  const uint32_t SUB = 0x64086408u;  // half2(1032): (1024 + c) - 1032 = c - 8, exact
  uint32_t e[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t t = lop3_and_or(w >> (4 * i), 0x000f000fu, EX);  // lanes: nibbles (i, i + 4)
    const __half2 d = __hsub2(*reinterpret_cast<__half2*>(&t), *reinterpret_cast<const __half2*>(&SUB));
    uint16_t r;
    asm("cvt.rn.satfinite.e4m3x2.f16x2 %0, %1;" : "=h"(r) : "r"(*reinterpret_cast<const uint32_t*>(&d)));
    e[i] = r;
  }
  // e0 = (k0, k2), e1 = (k1, k3), e2 = (k4, k6), e3 = (k5, k7) in bytes (0, 1)
  lo = __byte_perm(e[0], e[1], 0x5140);
  hi = __byte_perm(e[2], e[3], 0x5140);
}

template <int NTOK>
__global__ void __launch_bounds__(A_THREADS, 1)
    w4afp8_gemm_kernel(const __grid_constant__ CUtensorMap tmap_q, const uint4* __restrict__ packed,
                       const float* __restrict__ s_w, const float* __restrict__ s_x, const void* __restrict__ bias,
                       void* __restrict__ out, int M, int KB, int N, int kpc, int out_bf16) {
  using C = W4fCfg<NTOK>;
  constexpr int PST = C::PST, WST = C::WST, XST = C::XST;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t sW = smem_base;                 // [WST][128 features][128 k]   (also: fp32 partial tile)
  const uint32_t sX = sW + WST * C::W_BYTES;     // [XST][NTOK][128 k]
  const uint32_t sP = sX + XST * C::X_BYTES;     // [PST]{ packed tile | group scales }
  const uint32_t sS = sP + PST * C::P_BYTES;     // [WST][128] fp32 group scales of the expanded stage
  const uint32_t sBar = sS + WST * A_SC_BYTES;
  const uint32_t bar_pfull = sBar, bar_xfull = bar_pfull + 8 * PST, bar_xempty = bar_xfull + 8 * XST;
  const uint32_t bar_wready = bar_xempty + 8 * XST, bar_wempty = bar_wready + 8 * WST;
  const float* scs = reinterpret_cast<const float*>(smem + (sS - smem_base));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = blockIdx.x, n0 = nt * A_BF;
  const int row0 = blockIdx.z * NTOK, rows = min(NTOK, M - row0);
  const uint32_t nrank = cluster_nctarank(), crank = cluster_ctarank();
  const int kb0 = min(KB, (int)crank * kpc), kb1 = min(KB, kb0 + kpc);
  const int nkb = kb1 - kb0;

  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_q);
    for (int s = 0; s < PST; ++s) mbar_init(bar_pfull + 8 * s, 1);
    for (int s = 0; s < XST; ++s) {
      mbar_init(bar_xfull + 8 * s, 1);
      mbar_init(bar_xempty + 8 * s, A_MMA_THREADS / 32);
    }
    for (int s = 0; s < WST; ++s) {
      mbar_init(bar_wready + 8 * s, A_TG);
      mbar_init(bar_wempty + 8 * s, A_MMA_THREADS / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const uint4* ptile = packed + (size_t)nt * KB * (A_TILE_BYTES / 16);
  // block i of this rank into packed stage s: the tile and the 128 fp32 scales s_w[kb, n0 .. n0 + 127]
  auto load_weights = [&](int i, int s) {
    const int kb = kb0 + i;
    mbar_expect_tx(bar_pfull + 8 * s, C::P_BYTES);
    bulk_load(sP + s * C::P_BYTES, ptile + (size_t)kb * (A_TILE_BYTES / 16), A_TILE_BYTES, bar_pfull + 8 * s);
    bulk_load(sP + s * C::P_BYTES + A_TILE_BYTES, s_w + (size_t)kb * N + n0, A_SC_BYTES, bar_pfull + 8 * s);
  };

  auto load_codes = [&](int i, int xs) {
    mbar_expect_tx(bar_xfull + 8 * xs, C::X_BYTES);
    tma_load_2d(sX + xs * C::X_BYTES, &tmap_q, bar_xfull + 8 * xs, (kb0 + i) * A_BK, row0);
  };

  if (warp < 8) {
    // ================================ MMA warpgroups ================================
    const int wg = warp >> 2;  // features 64 wg .. 64 wg + 63 of the tile
    const int fr = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // this thread's accumulator rows fr, fr + 8
    if (threadIdx.x == 0) {
      asm volatile("griddepcontrol.wait;" ::: "memory");  // the codes are the quantiser's output
      for (int i = 0; i < nkb && i < XST; ++i) load_codes(i, i);
    }
    float acc[C::ACC], p[C::ACC];
#pragma unroll
    for (int v = 0; v < C::ACC; ++v) acc[v] = 0.f;
    for (int i = 0; i < nkb; ++i) {
      const int xs = i % XST, ws = i % WST;
      mbar_wait(bar_xfull + 8 * xs, (i / XST) & 1);
      mbar_wait(bar_wready + 8 * ws, (i / WST) & 1);
      const uint64_t wdesc = wgmma_desc_k_sw128(sW + ws * C::W_BYTES) + 512 * wg;
      const uint64_t xdesc = wgmma_desc_k_sw128(sX + xs * C::X_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < A_BK / 32; ++k) Wgmma8F<NTOK>::mma(p, wdesc + 2 * k, xdesc + 2 * k, k > 0 ? 1u : 0u);
      wgmma_commit();
      // while the block runs: once both warpgroups have read the codes of block i - 1, refill that stage
      if (threadIdx.x == 0 && i >= 1 && i - 1 + XST < nkb) {
        const int ps = (i - 1) % XST;
        mbar_wait(bar_xempty + 8 * ps, ((i - 1) / XST) & 1);
        load_codes(i - 1 + XST, ps);
      }
      wgmma_wait<0>();
      wgmma_fence_regs(p);
      const float sc[2] = {scs[ws * A_BF + fr], scs[ws * A_BF + fr + 8]};
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(bar_wempty + 8 * ws);
        mbar_arrive(bar_xempty + 8 * xs);
      }
      // promotion: the block's product times its group scale joins the fp32 accumulator
#pragma unroll
      for (int v = 0; v < C::ACC; ++v) acc[v] = fmaf(p[v], sc[(v >> 1) & 1], acc[v]);
    }
    // both warpgroups are done with the stages before either overwrites them with its partial tile
    asm volatile("bar.sync 3, %0;" ::"r"(A_MMA_THREADS) : "memory");
    park_partial(sW, wg, warp & 3, acc);
  } else {
    // ================================ dequant groups ================================
    const int t = threadIdx.x - A_MMA_THREADS, gq = t / A_TG, tl = t - gq * A_TG;
    // the group's leader starts the weight stream of its first blocks at once (under programmatic dependent launch:
    // while the quantiser still runs)
    if (tl == 0)
      for (int i = gq; i < nkb && i < PST; i += A_DQG) load_weights(i, i);
    for (int i = gq; i < nkb; i += A_DQG) {
      const int s = i % PST, ws = i % WST;
      mbar_wait(bar_pfull + 8 * s, (i / PST) & 1);
      const uint8_t* pst = smem + (sP - smem_base) + s * C::P_BYTES;
      uint4 pv[2][4];
      float sc[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
#pragma unroll
        for (int q = 0; q < 4; ++q) pv[r][q] = reinterpret_cast<const uint4*>(pst)[q * A_BF + tl + 64 * r];
        sc[r] = reinterpret_cast<const float*>(pst + A_TILE_BYTES)[tl + 64 * r];
      }
      // every thread of the group has read the stage: its leader refills it with block i + PST
      asm volatile("bar.sync %0, %1;" ::"r"(1 + gq), "r"(A_TG) : "memory");
      if (tl == 0 && i + PST < nkb) load_weights(i + PST, s);
      if (i >= WST) mbar_wait(bar_wempty + 8 * ws, ((i / WST) & 1) ^ 1);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int f = tl + 64 * r;
        const uint32_t row = sW + ws * C::W_BYTES + f * 128;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t wv[4] = {pv[r][q].x, pv[r][q].y, pv[r][q].z, pv[r][q].w};
          uint32_t o[8];
#pragma unroll
          for (int j = 0; j < 4; ++j) expand_e4m3(wv[j], o[2 * j], o[2 * j + 1]);
#pragma unroll
          for (int h = 0; h < 2; ++h) {  // 16-byte chunk 2q + h = k 32q + 16h .. +15
            const uint32_t addr = row + ((((uint32_t)(2 * q + h)) ^ (uint32_t)(f & 7)) << 4);
            asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(o[4 * h]), "r"(o[4 * h + 1]),
                         "r"(o[4 * h + 2]), "r"(o[4 * h + 3])
                         : "memory");
          }
        }
        asm volatile("st.shared.f32 [%0], %1;" ::"r"(sS + (uint32_t)(ws * A_BF + f) * 4), "f"(sc[r]) : "memory");
      }
      fence_proxy_async_smem();
      mbar_arrive(bar_wready + 8 * ws);
    }
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");  // s_x is the quantiser's output; orders the global stores below
  __syncwarp();
  cluster_sync_all();
  if (warp < A_MMA_THREADS / 32) {
    // rank z reduces token rows z, z + nrank, ... , a warp per row: y = T(acc * s_x[m] + bias[n]), one rounding
    const int nc = n0 + lane * 4;
    for (int tok = (int)crank + (int)nrank * warp; tok < rows; tok += (int)nrank * (A_MMA_THREADS / 32)) {
      float a[1][4];
      dsmem_sum4<1, false>(sW + (uint32_t)tok * (A_BF * 4) + (uint32_t)lane * 16, 0, nrank, a);
      const int m = row0 + tok;
      const float sx = s_x[m];
      float y[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) y[e] = __fmul_rn(a[0][e], sx);  // no contraction into an fma with the bias
      if (out_bf16) {
        using E = ET<__nv_bfloat16>;
        const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(bias);
        if (b != nullptr)
#pragma unroll
          for (int e = 0; e < 4; ++e) y[e] = __fadd_rn(y[e], E::to_f(b[nc + e]));
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + (size_t)m * N + nc) =
            make_uint2(E::pack2(y[0], y[1]), E::pack2(y[2], y[3]));
      } else {
        using E = ET<__half>;
        const __half* b = reinterpret_cast<const __half*>(bias);
        if (b != nullptr)
#pragma unroll
          for (int e = 0; e < 4; ++e) y[e] = __fadd_rn(y[e], E::to_f(b[nc + e]));
        *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(out) + (size_t)m * N + nc) =
            make_uint2(E::pack2(y[0], y[1]), E::pack2(y[2], y[3]));
      }
    }
  }
  __syncwarp();
  cluster_sync_all();  // keep every rank's shared memory alive until all peers have read it
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int launch_w4afp8_prepack(const int32_t* weight_packed, void* packed, int K, int N, cudaStream_t stream) {
  const size_t words = (size_t)(K / A_BK) * (N / A_BF) * (A_TILE_BYTES / 4);
  const int blocks = (int)((words + 255) / 256 < 65535 ? (words + 255) / 256 : 65535);
  w4afp8_prepack_kernel<<<blocks, 256, 0, stream>>>((const uint32_t*)weight_packed, (uint32_t*)packed, K, N);
  return (int)cudaGetLastError();
}

template <int NTOK>
static int launch_w4afp8_gemm_t(const W4Fp8Args& a, const SwapPlan& p) {
  using C = W4fCfg<NTOK>;
  CUtensorMap tq;  // the codes [M, K] in boxes of 128 k x NTOK tokens; rows >= M are zero-filled
  if (make_tmap_2d(&tq, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.codes, a.K, a.M, (size_t)a.K, A_BK, NTOK,
                   CU_TENSOR_MAP_SWIZZLE_128B) != 0)
    return -1;
  auto kern = w4afp8_gemm_kernel<NTOK>;
  static int smem_opted[32] = {};
  if (int e = ensure_dyn_smem(kern, C::SMEM_BYTES, smem_opted, "b2q_w4afp8")) return e;
  return launch_kernel(kern, dim3(a.N / A_BF, p.ks, p.tblocks), dim3(A_THREADS, 1, 1), C::SMEM_BYTES, a.stream, p.ks,
                       true, tq, (const uint4*)a.packed, a.s_w, a.s_x, a.bias, a.out, a.M, a.K / A_BK, a.N, p.kpc,
                       a.dtype);
}

// the plan of the per-channel FP8 GEMM (same 128-feature tiles, token blocks and split-K ranks); a pinned ks is taken
// as given
int launch_w4afp8_gemm(const W4Fp8Args& a) {
  const SwapPlan p = fp8blk_plan(0, a.M, a.K, a.N, 1, a.ks);
  switch (p.ntok) {
    case 8: return launch_w4afp8_gemm_t<8>(a, p);
    case 16: return launch_w4afp8_gemm_t<16>(a, p);
    case 32: return launch_w4afp8_gemm_t<32>(a, p);
    case 64: return launch_w4afp8_gemm_t<64>(a, p);
    default: return launch_w4afp8_gemm_t<128>(a, p);
  }
}

}  // namespace b2q
