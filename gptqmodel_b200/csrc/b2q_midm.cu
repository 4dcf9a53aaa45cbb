// b2q_midm.cu — small-batch tier (2 <= tokens <= 128; every 8-bit / group_size 32 shape the decode tier does not
// take): out[M, N] = x[M, K] @ dequant(W)[K, N] (+ bias) with SWAPPED wgmma operands and cluster split-K.
//
// Batched decode / speculative decoding is HBM-bound like batch-1 decode: the layer's packed weights must stream once,
// the token count only changes the width of the MMA.  The prefill tier pads tokens to its 128-token tile and launches
// N/128 CTAs (32 of 132 SMs for a 4096-wide layer).  Here
//   * the WEIGHTS are the wgmma A operand: 128 output features = two m64 blocks, the TOKENS are the B operand,
//     N = NTOK in {16, 32, 64, 128}: no padding of tokens to 128, the accumulator D[feature][token] is NTOK registers per
//     thread of the MMA warpgroup and the x tile is NTOK x 64 k (TMA, SWIZZLE_128B);
//   * `ks` CTAs of a thread-block cluster split the k-blocks of one 128-feature tile (4096 x 4096: 32 tiles x 4 = 128
//     CTAs), park their fp32 partials TRANSPOSED ([token][feature]) in their own shared memory and reduce an interleaved
//     share of the token rows over distributed shared memory: no atomics, no workspace, deterministic, and the global
//     stores are 256 contiguous bytes per warp (features are the fast axis of `out`);
//   * 4 dequant warps (fragment-major uint4 = 2 features x 16 k each) produce the exact (q - z) * s operand (integer
//     subtract first, ONE rounding: qlinear/__init__.py:1001-1003) as 16-byte swizzled K-major rows.  Each dequant warp
//     takes every 4th k-block and issues the bulk copies of its own packed stages, warp 8 only the x tile TMA: no single
//     thread issues every asynchronous copy of every k-block, and the weight stream + dequant of the first blocks run
//     BEFORE griddepcontrol.wait (programmatic dependent launch), i.e. under the previous kernel's tail.
// Reference counterparts: Swordfish's Stream-K / atomic split-K decode for 17 <= M < 128 (swordfish_mm.cu:113-154,
// 229-276), its swapped-problem-shape trick (swordfish_prefill_impl.cuh:219-227), Marlin's small-M tiles
// (marlin_template.h).
#include <cuda.h>

#include "b2q_common.cuh"
#include "b2q_dequant.cuh"
#include "b2q_internal.h"
#include "b2q_wgmma.cuh"

namespace b2q {

constexpr int MM_BF = 128;                  // features per tile (two wgmma m64 blocks)
constexpr int MM_BK = 64;                   // k per block (one SWIZZLE_128B row of fp16)
constexpr int MM_MMA_THREADS = 128;         // warps 0..3: the wgmma warpgroup
constexpr int MM_DQ_WARPS = 4;              // warps 4..7
constexpr int MM_DQ_THREADS = MM_DQ_WARPS * 32;
constexpr int MM_THREADS = MM_MMA_THREADS + MM_DQ_THREADS + 32;  // + warp 8: activation producer
constexpr int MM_RED_WARPS = 8;             // warps 0..7 reduce the split-K partials

// Two rings.  The PACKED ring (PST stages: x tile + packed codes + scale / zero rows, 7-21 KB each) is what hides the HBM
// latency: with 4 stages (the first version of this kernel) only 16 KB of weights per SM were in flight and every k-block
// cost one HBM round trip / 4; Little's law asks for tens of KB in flight per SM.  The DEQUANTISED ring (WST stages of 16 KB) only
// decouples the dequant warps from the tensor core.
// MODE 0: one QuantLinear.  MODE 1 / 2: GROUPED over the experts of a MoE block (b2q_moe.cu): blockIdx.z = (expert, token
// block); the rows of an expert are contiguous in the expert-sorted activation matrix; CTAs beyond an expert's row count
// exit at once.  MODE 1 runs TWO weight sets (w1 = gate, w3 = up) through the pipeline back to back into two register
// accumulators and stores silu(gate) * up; MODE 2 (w2 = down) scales each row by its routing weight and scatters it to the
// row's (token, k) slot of an fp32 buffer.
struct MoeArgs {
  const int32_t* counts;        // [E] rows of expert e
  const int32_t* offsets;       // [E] first row of expert e in the sorted order
  const int32_t* sorted_pairs;  // [rows] pair index (token * top_k + j) of sorted row i            (MODE 2)
  const float* pair_weights;    // [rows] routing weight, indexed by PAIR index                      (MODE 2)
  const uint4* packed3;         // second weight set, same shapes / strides as the first             (MODE 1)
  const void* scales3;
  const uint32_t* qzeros3;
  float* ypair;                 // [rows, N] fp32, row = pair index                                   (MODE 2)
  int tblocks;                  // token blocks (of NTOK rows) per expert in gridDim.z
};

template <int BITS, int NTOK, int PST, int WST, int MODE = 0>
struct MidCfg {
  static constexpr int NSETS = MODE == 1 ? 2 : 1;
  static constexpr int XST = NTOK >= 64 ? 4 : 8;         // activation-tile stages (own ring: one TMA per k-block)
  static constexpr int SUB = BITS / 4;
  static constexpr int W_BYTES = MM_BF * MM_BK * 2;      // dequantised weights, A operand: 16 KB
  static constexpr int X_BYTES = NTOK * MM_BK * 2;       // activations, B operand (first in its stage: 1024-B aligned)
  static constexpr int P_CHUNK_BYTES = 4 * SUB * 512;    // 8-bit: 4 feature tiles (of 32) x 32 k
  static constexpr int P_BYTES = 2 * P_CHUNK_BYTES + (BITS == 4 ? 1024 : 0);  // + scale / zero rows (4-bit)
  static constexpr int BAR_BYTES = 512;
  static constexpr int RING_BYTES = WST * W_BYTES + XST * X_BYTES + PST * P_BYTES;
  static constexpr int SMEM_BYTES = RING_BYTES + BAR_BYTES + 1024;
  static constexpr int ACC = NTOK / 2;                   // fp32 accumulator registers per thread, per set and m64 block
  static_assert(NSETS * NTOK <= 128, "accumulators of the MMA warpgroup: at most 128 registers per thread");
  static constexpr int PART_BYTES = NSETS * NTOK * MM_BF * 4;  // fp32 partial tile(s) [set][token][feature]
  static_assert(MODE == 0 || BITS == 4, "the grouped (MoE) modes are built for 4-bit experts");
  static_assert(X_BYTES % 1024 == 0, "x tiles must stay 1024-byte aligned (SWIZZLE_128B atoms)");
  static_assert(PART_BYTES <= RING_BYTES, "the fp32 partial tile reuses the idle stage buffers");
  static_assert((PST + 2 * XST + 2 * WST) * 8 <= BAR_BYTES, "mbarrier area");
  static_assert(SMEM_BYTES <= 227 * 1024, "dynamic shared memory of one CTA");
};

template <typename T, int BITS, bool ASYM, int NTOK, int PST, int WST, int MODE, int DQG>
__global__ void __launch_bounds__(MM_THREADS, 1)
    midm_kernel(const __grid_constant__ CUtensorMap tmap_x, const uint4* __restrict__ packed,
                const T* __restrict__ scales, const uint32_t* __restrict__ qzeros, const T* __restrict__ bias,
                T* __restrict__ out, int M, int K, int N, int gshc, int kpc, const __grid_constant__ MoeArgs G) {
  using C = MidCfg<BITS, NTOK, PST, WST, MODE>;
  using E = ET<T>;
  constexpr int NSETS = C::NSETS;
  int row0 = 0;  // first row of this CTA's token block in the activation matrix
  const uint4* packed_b = nullptr;
  const T* scales_b = nullptr;
  const uint32_t* qzeros_b = nullptr;
  if (MODE != 0) {
    // the routing tables are written by the preceding kernel of the stream: nothing may be read before it has finished
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int e = (int)blockIdx.z / G.tblocks, tb = (int)blockIdx.z - e * G.tblocks;
    const int cnt = G.counts[e];
    if (tb * NTOK >= cnt) return;  // same decision in every CTA of the cluster (they differ in blockIdx.y only)
    row0 = G.offsets[e] + tb * NTOK;
    M = min(NTOK, cnt - tb * NTOK);
    const size_t groups = (size_t)(K >> 5) >> gshc;  // quantisation groups along K (gshc = log2(32-k chunks per group))
    const size_t wstride = (size_t)K * N / 32, sstride = (gshc >= 31 ? 1 : groups) * (size_t)N;
    packed += (size_t)e * wstride;
    scales += (size_t)e * sstride;
    if (ASYM) qzeros += (size_t)e * (sstride >> 3);
    if (MODE == 1) {
      packed_b = G.packed3 + (size_t)e * wstride;
      scales_b = reinterpret_cast<const T*>(G.scales3) + (size_t)e * sstride;
      if (ASYM) qzeros_b = G.qzeros3 + (size_t)e * (sstride >> 3);
    }
  }
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));

  constexpr int XST = C::XST;
  constexpr bool ISSUER_REFILL = PST >= 3 * DQG;  // who refills the packed stages (see the dequant warps)
  const uint32_t sW = smem_base;                      // [WST][128 features][64 k]      (also: fp32 partial tile)
  const uint32_t sXr = sW + WST * C::W_BYTES;         // [XST] x tile [NTOK][64 k]
  const uint32_t sPr = sXr + XST * C::X_BYTES;        // [PST]{ packed codes | scale / zero rows }
  const uint32_t sBar = sPr + PST * C::P_BYTES;
  const uint32_t bar_pfull = sBar, bar_xfull = bar_pfull + 8 * PST, bar_xempty = bar_xfull + 8 * XST;
  const uint32_t bar_wready = bar_xempty + 8 * XST, bar_wempty = bar_wready + 8 * WST;
  auto sXs = [&](int s) { return sXr + (uint32_t)s * C::X_BYTES; };
  auto sPs = [&](int s) { return sPr + (uint32_t)s * C::P_BYTES; };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int NT = N >> 5;
  const int n0 = blockIdx.x * MM_BF;
  const int nt0 = n0 >> 5;
  const int ntiles = min(4, NT - nt0);
  // split-K: cluster rank owns k-blocks [kb0, kb1); i = kb - kb0 drives the stage / phase bookkeeping
  const uint32_t nrank = cluster_nctarank(), crank = cluster_ctarank();
  const int kb0 = (int)crank * kpc, kb1 = min(K / MM_BK, kb0 + kpc);
  const int nkb = kb1 - kb0;
  const int NI = NSETS * nkb;  // pipeline iterations: the k-blocks of set 0, then (MODE 1) of set 1

  // PDL: the next kernel in the stream may start its own prologue / weight prefetch now
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_x);
    for (int s = 0; s < PST; ++s) mbar_init(bar_pfull + 8 * s, 1);
    for (int s = 0; s < XST; ++s) {
      mbar_init(bar_xfull + 8 * s, 1);
      mbar_init(bar_xempty + 8 * s, 1);
    }
    for (int s = 0; s < WST; ++s) {
      mbar_init(bar_wready + 8 * s, MM_DQ_THREADS / DQG);
      mbar_init(bar_wempty + 8 * s, 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  // ---- weight loads of pipeline iteration i into packed stage s (issued by the LEADER of the dequant group that will
  // consume the stage, see below: one thread per SM issuing every asynchronous copy of every k-block serialises the
  // copy issue)
  const int FT = N >> 4, ft0 = n0 >> 4;
  const uint32_t pbytes4 = (uint32_t)min(8, FT - ft0) * 512u;
  const uint32_t pbytes8 = (uint32_t)ntiles * C::SUB * 512u;
  const uint32_t sbytes = (uint32_t)min(MM_BF, N - n0) * 2u, zbytes = ASYM ? sbytes / 4u : 0u;
  auto load_weights = [&](int i, int s) {
    const bool second = NSETS > 1 && i >= nkb;
    const int kb = kb0 + (second ? i - nkb : i);
    const uint4* pk = second ? packed_b : packed;
    const T* sc = second ? scales_b : scales;
    const uint32_t* zq = second ? qzeros_b : qzeros;
    if (BITS == 4) {
      // the scale / zero rows of the block's group(s) travel with the packed codes (no LDG in the dequant warps)
      const int g0 = (2 * kb) >> gshc, g1 = (2 * kb + 1) >> gshc;
      const int nrows = (g1 != g0) ? 2 : 1;
      mbar_expect_tx(bar_pfull + 8 * s, pbytes4 + nrows * (sbytes + zbytes));
      bulk_load(sPs(s), pk + ((size_t)kb * FT + ft0) * 32, pbytes4, bar_pfull + 8 * s);
      for (int r = 0; r < nrows; ++r) {
        const int gr = r ? g1 : g0;
        bulk_load(sPs(s) + 4096 + r * 320, sc + (size_t)gr * N + n0, sbytes, bar_pfull + 8 * s);
        if (ASYM)
          bulk_load(sPs(s) + 4096 + r * 320 + 256, zq + (size_t)gr * (N >> 3) + (n0 >> 3), zbytes, bar_pfull + 8 * s);
      }
    } else {
      mbar_expect_tx(bar_pfull + 8 * s, 2 * pbytes8);
#pragma unroll
      for (int j = 0; j < 2; ++j)
        bulk_load(sPs(s) + j * C::P_CHUNK_BYTES, pk + ((size_t)(kb * 2 + j) * NT + nt0) * C::SUB * 32, pbytes8,
                  bar_pfull + 8 * s);
    }
  };

  if (warp == 8) {
    // ================================ activation producer ================================
    // one TMA per pipeline iteration: the x tile of the k-block (the weights are loaded by the dequant group leaders)
    if (lane == 0) {
      asm volatile("griddepcontrol.wait;" ::: "memory");  // x is the previous kernel's output
      for (int i = 0; i < NI; ++i) {
        const int xs = i % XST;
        if (i >= XST) mbar_wait(bar_xempty + 8 * xs, ((i / XST) & 1) ^ 1);
        const int kb = kb0 + ((NSETS > 1 && i >= nkb) ? i - nkb : i);
        mbar_expect_tx(bar_xfull + 8 * xs, C::X_BYTES);
        tma_load_2d(sXs(xs), &tmap_x, bar_xfull + 8 * xs, kb * MM_BK, row0);
      }
    }
  } else if (warp < 4) {
    // ================================ MMA warpgroup ================================
    // One wgmma group (4 k16 steps x 2 m64 feature blocks) per pipeline iteration, one group kept in flight: the stages of
    // iteration i - 1 are released once the group of iteration i has been issued and i - 1 has completed.
    float acc[NSETS][2][C::ACC];
#pragma unroll
    for (int st = 0; st < NSETS; ++st)
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int v = 0; v < C::ACC; ++v) acc[st][mb][v] = 0.f;
    // one loop per weight set: the wgmma of a loop always targets the same accumulator registers (a set chosen at run time
    // inside the loop would put the wgmma on a divergent path, which ptxas serialises)
    auto step = [&](int i, float (&ac)[2][C::ACC], bool first) {
      const int xs = i % XST, ws = i % WST;
      mbar_wait(bar_xfull + 8 * xs, (i / XST) & 1);
      mbar_wait(bar_wready + 8 * ws, (i / WST) & 1);
      // wready(i) completed => the dequant group has read packed stage i % PST: stream block i + PST into it (one
      // thread per k-block, off the dequant groups' latency chain)
      if (ISSUER_REFILL && threadIdx.x == 0 && i + PST < NI) load_weights(i + PST, i % PST);
      const uint64_t wdesc = wgmma_desc_k_sw128(sW + ws * C::W_BYTES);
      const uint64_t xdesc = wgmma_desc_k_sw128(sXs(xs));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < MM_BK / 16; ++k) {
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)  // the first block of a set overwrites
          Wgmma<E::FMT, NTOK>::mma(ac[mb], wdesc + 512 * mb + 2 * k, xdesc + 2 * k, (first && k == 0) ? 0u : 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (i > 0 && threadIdx.x == 0) {
        mbar_arrive(bar_wempty + 8 * ((i - 1) % WST));  // the dequantised stage may be overwritten
        mbar_arrive(bar_xempty + 8 * ((i - 1) % XST));  // the x tile has been read
      }
    };
    for (int i = 0; i < nkb; ++i) step(i, acc[0], i == 0);
    if (NSETS > 1)
      for (int i = nkb; i < NI; ++i) step(i, acc[NSETS - 1], i == nkb);
    wgmma_wait<0>();
#pragma unroll
    for (int st = 0; st < NSETS; ++st)
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) wgmma_fence_regs(acc[st][mb]);

    // ---- this rank's fp32 accumulator D[feature][token] -> its own shared memory, transposed: part[set][token][feature]
    // (the stage buffers are idle now: every load was consumed by an MMA that has completed)
#pragma unroll
    for (int st = 0; st < NSETS; ++st)
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int v = 0; v < C::ACC; ++v) {
          const int j = v >> 2, h = (v >> 1) & 1, c = v & 1;
          const int feat = 64 * mb + 16 * warp + (lane >> 2) + 8 * h, tok = 8 * j + 2 * (lane & 3) + c;
          asm volatile("st.shared.f32 [%0], %1;" ::"r"(sW + (uint32_t)((st * NTOK + tok) * MM_BF + feat) * 4),
                       "f"(acc[st][mb][v])
                       : "memory");
        }
  } else {
    // ================================ dequant warps ================================
    // The dequant warps form DQG groups of TG threads; group gq takes the pipeline iterations i = gq, gq + DQG, ...  One
    // iteration is a serial chain of latencies for a warp (mbarrier wake-up, LDS, ~75 ALU instructions per uint4, STS,
    // fence.proxy.async, arrive: ~800 clk) — with all eight warps on the SAME k-block (first version) that chain WAS the
    // k-block time at any ring depth; with DQG blocks in flight the
    // chains overlap and the tier becomes issue-bound instead.
    const int t = threadIdx.x - MM_MMA_THREADS;  // 0..127
    constexpr int TG = MM_DQ_THREADS / DQG;
    static_assert(PST % DQG == 0 && WST % DQG == 0, "every use of a ring stage must belong to the same dequant group");
    const int gq = t / TG, tl = t - gq * TG;
    constexpr int PF = 32 / BITS;
    constexpr int ZSYM = 1 << (BITS - 1);
    // the group's leader starts the weight stream of the group's first PST / DQG blocks (never depends on the previous
    // kernel: under programmatic dependent launch this runs while the producer of x is still executing)
    if (tl == 0)
      for (int i = gq; i < NI && i < PST; i += DQG) load_weights(i, i);
    if (BITS == 4) {
      // U fragment-major uint4 per thread and iteration: q = tl + TG*u -> feature tile q>>5 (16 features), lane' = q&31
      constexpr int U = 256 / TG;
      const int lp = tl & 31, g = lp >> 2, tt = lp & 3;
      for (int i = gq; i < NI; i += DQG) {
        const int kb = kb0 + ((NSETS > 1 && i >= nkb) ? i - nkb : i), s = i % PST, ws = i % WST;
        mbar_wait(bar_pfull + 8 * s, (i / PST) & 1);
        const uint8_t* pst = smem + (sPs(s) - smem_base);
        // this lane's 16 k of block kb lie in 32-k chunk 2*kb + (tt>>1)
        const int grow = ((2 * kb + (tt >> 1)) >> gshc) - ((2 * kb) >> gshc);  // 0 or 1
        const uint8_t* srow = pst + 4096 + grow * 320;
        uint4 pv[U];
        uint32_t s_lo[U], s_hi[U];
        int zl[U], zh[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int q = tl + TG * u;
          const int f_lo = (q >> 5) * 16 + g, f_hi = f_lo + 8;
          pv[u] = reinterpret_cast<const uint4*>(pst)[q];
          s_lo[u] = *reinterpret_cast<const uint16_t*>(srow + f_lo * 2);
          s_hi[u] = *reinterpret_cast<const uint16_t*>(srow + f_hi * 2);
          zl[u] = zh[u] = ZSYM;
          if (ASYM) {
            const uint32_t zwl = *reinterpret_cast<const uint32_t*>(srow + 256 + (f_lo >> 3) * 4);
            const uint32_t zwh = *reinterpret_cast<const uint32_t*>(srow + 256 + (f_hi >> 3) * 4);
            zl[u] = (int)((zwl >> (4 * g)) & 15u);  // feature % 8 == g for both rows
            zh[u] = (int)((zwh >> (4 * g)) & 15u);
          }
        }
        // Refill of the packed stage for block i + PST.  With >= 3 packed stages per group the MMA issuer of block i does it
        // (it observes wready(i), which this group only signals after every thread has read the stage: no barrier or copy
        // issue inside this chain).  With 1-2 stages per group that is too late — the group would
        // wait a full HBM round trip per block — so the group's leader refills right
        // after the whole group has read.
        if (!ISSUER_REFILL) {
          asm volatile("bar.sync %0, %1;" ::"r"(1 + gq), "r"(TG) : "memory");
          if (tl == 0 && i + PST < NI) load_weights(i + PST, s);
        }
        if (i >= WST) mbar_wait(bar_wempty + 8 * ws, ((i / WST) & 1) ^ 1);  // the MMA of block i - WST has read the stage
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int q = tl + TG * u;
          const int f_lo = (q >> 5) * 16 + g;
          uint4 lo[2], hi[2];
          Dequant<T, 4>::run(pv[u], s_lo[u], zl[u], s_hi[u], zh[u], lo, hi);
          const uint32_t rlo = sW + ws * C::W_BYTES + f_lo * 128;
          const uint32_t rhi = rlo + 8 * 128;
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const uint32_t off = (((uint32_t)(2 * tt + c)) ^ (uint32_t)g) << 4;  // (row & 7) == g for rows f and f+8
            asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(rlo + off), "r"(lo[c].x), "r"(lo[c].y),
                         "r"(lo[c].z), "r"(lo[c].w)
                         : "memory");
            asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(rhi + off), "r"(hi[c].x), "r"(hi[c].y),
                         "r"(hi[c].z), "r"(hi[c].w)
                         : "memory");
          }
        }
        fence_proxy_async_smem();
        mbar_arrive(bar_wready + 8 * ws);
      }
    } else {
      // 8-bit: a group covers the 128 feature rows x two 32-k halves of a block: thread -> rows tl + TG*r, both halves,
      // two uint4 (16 k each) per (row, half)
      constexpr int R = (128 / TG) > 0 ? 128 / TG : 1;  // (TG = 256 only exists for the 4-bit debug variant)
      for (int i = gq; i < NI; i += DQG) {
        const int kb = kb0 + i, s = i % PST, ws = i % WST;
        SZRaw sz[R][2];
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int n = n0 + tl + TG * r;
#pragma unroll
          for (int j = 0; j < 2; ++j) sz[r][j] = load_sz<T, BITS, ASYM>(scales, qzeros, (2 * kb + j) >> gshc, n < N ? n : 0, N);
        }
        mbar_wait(bar_pfull + 8 * s, (i / PST) & 1);
        uint4 pvs[R][2][2];
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int fr = tl + TG * r;
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const uint4* pj = reinterpret_cast<const uint4*>(smem + (sPs(s) - smem_base) + j * C::P_CHUNK_BYTES);
#pragma unroll
            for (int h = 0; h < 2; ++h) pvs[r][j][h] = pj[((fr >> 5) * 2 + h) * 32 + (fr & 31)];
          }
        }
        if (!ISSUER_REFILL) {  // see the 4-bit path
          asm volatile("bar.sync %0, %1;" ::"r"(1 + gq), "r"(TG) : "memory");
          if (tl == 0 && i + PST < NI) load_weights(i + PST, s);
        }
        if (i >= WST) mbar_wait(bar_wempty + 8 * ws, ((i / WST) & 1) ^ 1);
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int fr = tl + TG * r;
          const int n = n0 + fr;
          const int nsafe = n < N ? n : 0;
          const uint32_t brow = sW + ws * C::W_BYTES + fr * 128;
          const uint32_t sw = (uint32_t)(fr & 7);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            int z = ZSYM;
            if (ASYM) z = (int)((sz[r][j].zw >> (BITS * (nsafe % PF))) & ((1u << BITS) - 1));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              uint4 o[2];
              Dequant<T, 8>::run(pvs[r][j][h], sz[r][j].s, z, o);
#pragma unroll
              for (int c = 0; c < 2; ++c) {
                const uint32_t addr = brow + (((uint32_t)(j * 4 + h * 2 + c) ^ sw) << 4);
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(o[c].x), "r"(o[c].y), "r"(o[c].z),
                             "r"(o[c].w)
                             : "memory");
              }
            }
          }
        }
        fence_proxy_async_smem();
        mbar_arrive(bar_wready + 8 * ws);
      }
    }
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");  // (already satisfied) orders the global stores below
  // all ranks' partials are in place (cluster barrier = CTA barrier + cross-CTA release / acquire)
  __syncwarp();
  cluster_sync_all();
  if (warp < MM_RED_WARPS) {
    // rank z reduces token rows z, z + nrank, ... over all ranks through distributed shared memory; a warp owns one
    // token row at a time: 32 lanes x 4 features = the 128 features of the tile = 256 contiguous output bytes
    const int t = threadIdx.x;
    const int chunk = t & 31;
    const int nc = n0 + chunk * 4;
    if (nc < N) {
      for (int tok = (int)crank + (int)nrank * (t >> 5); tok < M; tok += (int)nrank * MM_RED_WARPS) {
        const uint32_t local = sW + (uint32_t)tok * (MM_BF * 4) + (uint32_t)chunk * 16;
        float acc[4] = {0.f, 0.f, 0.f, 0.f}, acc2[4] = {0.f, 0.f, 0.f, 0.f};
        for (uint32_t r = 0; r < nrank; ++r) {
          uint32_t ra;
          float4 v;
          asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local), "r"(r));
          asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];"
                       : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                       : "r"(ra)
                       : "memory");
          acc[0] += v.x;
          acc[1] += v.y;
          acc[2] += v.z;
          acc[3] += v.w;
          if (MODE == 1) {
            asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];"
                         : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                         : "r"(ra + (uint32_t)NTOK * (MM_BF * 4))
                         : "memory");
            acc2[0] += v.x;
            acc2[1] += v.y;
            acc2[2] += v.z;
            acc2[3] += v.w;
          }
        }
        if (MODE == 0) {
          if (bias != nullptr) {
            // reference order: round the matmul to the output dtype, then add bias (torch.py:337-342)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[i] = E::to_f(E::from_f(acc[i])) + E::to_f(bias[nc + i]);
          }
          *reinterpret_cast<uint2*>(out + (size_t)tok * N + nc) =
              make_uint2(E::pack2(acc[0], acc[1]), E::pack2(acc[2], acc[3]));
        } else if (MODE == 1) {
          // the per-expert module loop of the reference model rounds at every module boundary
          // (act_fn(w1(x)) * w3(x) with 16-bit tensors): g = T(x W1), a = T(silu(g)), u = T(x W3), h = T(a * u)
          float hv[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float gq = E::to_f(E::from_f(acc[i])), uq = E::to_f(E::from_f(acc2[i]));
            const float aq = E::to_f(E::from_f(gq / (1.f + __expf(-gq))));
            hv[i] = aq * uq;
          }
          *reinterpret_cast<uint2*>(out + (size_t)(row0 + tok) * N + nc) =
              make_uint2(E::pack2(hv[0], hv[1]), E::pack2(hv[2], hv[3]));
        } else {
          // y = T(h W2) like the module, then the routing weight; kept in fp32 in the row's (token, k) slot — the k slots
          // of a token are summed (and rounded ONCE) by moe_combine_kernel: no atomics, deterministic
          const int pair = G.sorted_pairs[row0 + tok];
          const float w = G.pair_weights[pair];
          float4 o;
          o.x = w * E::to_f(E::from_f(acc[0]));
          o.y = w * E::to_f(E::from_f(acc[1]));
          o.z = w * E::to_f(E::from_f(acc[2]));
          o.w = w * E::to_f(E::from_f(acc[3]));
          *reinterpret_cast<float4*>(G.ypair + (size_t)pair * N + nc) = o;
        }
      }
    }
  }
  __syncwarp();
  cluster_sync_all();  // keep every rank's shared memory alive until all peers have read it
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int make_x_tmap_box(CUtensorMap* map, const void* x, int M, int K, int dtype, int box_rows);  // b2q_gemm.cu

// split-K ranks (cluster size) for one launch: fill the SMs, keep >= 4 k-blocks per rank, portable cluster size <= 8
int midm_ranks(int K, int N) {
  const int tiles = (N + MM_BF - 1) / MM_BF, nkb = K / MM_BK;
  int ks = 1;
  while (ks < 8 && tiles * ks * 2 <= num_sms() && nkb / (ks * 2) >= 4) ks *= 2;
  return ks;
}

constexpr int MM_DQG = 4;  // dequant groups = k-blocks dequantised concurrently

template <typename T, int BITS, bool ASYM, int NTOK, int PST, int WST, int MODE = 0, int DQG = MM_DQG>
static int launch_midm_t(const MmArgs& a, const void* x, int ks, const MoeArgs& G = MoeArgs{}, int x_rows = 0,
                         int grid_z = 1) {
  using C = MidCfg<BITS, NTOK, PST, WST, MODE>;
  if constexpr (BITS == 4 && MODE == 0 && DQG == MM_DQG) {
    if (env().midm_dqg1)  // debugging: all dequant warps on the same k-block
      return launch_midm_t<T, BITS, ASYM, NTOK, PST, WST, 0, 1>(a, x, ks, G, x_rows, grid_z);
  }
  CUtensorMap tmap;
  if (make_x_tmap_box(&tmap, x, MODE == 0 ? a.M : x_rows, a.K, a.dtype, NTOK) != 0) return -1;
  auto kern = midm_kernel<T, BITS, ASYM, NTOK, PST, WST, MODE, DQG>;
  static uint32_t smem_ok = 0;  // per-device bit mask (a process may drive several GPUs)
  if (int e = ensure_dyn_smem(kern, C::SMEM_BYTES, smem_ok, "b2q_midm")) return e;
  const int nkb = a.K / MM_BK;
  const int kpc = (nkb + ks - 1) / ks;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((a.N + MM_BF - 1) / MM_BF, ks, grid_z);
  cfg.blockDim = dim3(MM_THREADS, 1, 1);
  cfg.dynamicSmemBytes = C::SMEM_BYTES;
  cfg.stream = a.stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = ks;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = a.pdl ? 2 : 1;
  return (int)cudaLaunchKernelEx(&cfg, kern, tmap, (const uint4*)a.packed, (const T*)a.scales,
                                 (const uint32_t*)a.qzeros, (const T*)a.bias, (T*)a.out, a.M, a.K, a.N, gemm_gshc(a),
                                 kpc, G);
}

bool midm_supported(const MmArgs& a) { return a.M >= 1 && a.M <= 128 && a.K % MM_BK == 0 && a.N % 32 == 0; }

// x: activations with act-order already applied (launch_gemm permutes into the workspace first)
int launch_midm(const MmArgs& a, const void* x) {
  int ks = env().midm_ks > 0 ? env().midm_ks : midm_ranks(a.K, a.N);
  if (ks > 8) ks = 8;
  const int nkb = a.K / MM_BK;
  while (ks > 1 && (ks - 1) * ((nkb + ks - 1) / ks) >= nkb) ks >>= 1;  // every rank needs at least one k-block
  const bool asym = a.qzeros != nullptr;
  // ring depths: BOTH must be multiples of the number of dequant groups, so that every use of a stage is served by the
  // SAME group.  mbarrier waits only distinguish the parity of a phase: with 6-stage rings and 4 groups (first version)
  // consecutive uses of a stage belonged to different groups, a group that ran two uses ahead saw the phase of use u - 2 as
  // "its" completed phase, consumed a stage that had not been refilled and corrupted the arrival counts — every
  // single-launch parity test and all three sanitizer tools passed, back-to-back launches at full size faulted
  // .  8 dequantised stages = two per group; 4-8 packed stages (refilled by the group's own
  // leader); 4-8 activation stages in their own ring.
#define B2Q_MM_NTOK(T, BITS, AS)                                                                  \
  (a.M <= 16   ? launch_midm_t<T, BITS, AS, 16, (BITS == 4 ? 12 : 8), 8>(a, x, ks)                \
   : a.M <= 32 ? launch_midm_t<T, BITS, AS, 32, (BITS == 4 ? 12 : 8), 8>(a, x, ks)                \
   : a.M <= 64 ? launch_midm_t<T, BITS, AS, 64, (BITS == 4 ? 8 : 4), 8>(a, x, ks)                 \
               : launch_midm_t<T, BITS, AS, 128, 4, 8>(a, x, ks))
#define B2Q_MM_CASE(T)                                                          \
  (a.bits == 4 ? (asym ? B2Q_MM_NTOK(T, 4, true) : B2Q_MM_NTOK(T, 4, false))   \
               : (asym ? B2Q_MM_NTOK(T, 8, true) : B2Q_MM_NTOK(T, 8, false)))
  return a.dtype == 0 ? B2Q_MM_CASE(__half) : B2Q_MM_CASE(__nv_bfloat16);
#undef B2Q_MM_CASE
#undef B2Q_MM_NTOK
}

// ------------------------------------------------------------------------------------------------
// grouped launches for a MoE block (b2q_moe.cu): a = {x = expert-sorted activations [rows, K], packed / scales / qzeros =
// the STACKED tensors of all experts (expert stride = one expert's tensor), out = h [rows, N] (mode 1), M = token-box
// width hint (largest row count one expert is expected to get), N / K of ONE expert}
int midm_grouped_ranks(int K, int N, int active) {
  const int tiles = (N + MM_BF - 1) / MM_BF, nkb = K / MM_BK;
  int ks = 1;
  while (ks < 8 && tiles * active * ks * 2 <= num_sms() && nkb / (ks * 2) >= 4) ks *= 2;
  return ks;
}

int launch_midm_grouped(int mode, const MmArgs& a, const MoeGroupedArgs& g) {
  if (a.bits != 4 || a.K % MM_BK != 0 || a.N % 32 != 0 || (mode != 1 && mode != 2) || g.E < 1 || g.rows < 1) {
    set_error("b2q_moe: grouped launch needs bits=4, K %% 64 == 0, N %% 32 == 0 (bits=%d K=%d N=%d E=%d rows=%d)", a.bits,
              a.K, a.N, g.E, g.rows);
    return -1;
  }
  MoeArgs G = {};
  G.counts = g.counts;
  G.offsets = g.offsets;
  G.sorted_pairs = g.sorted_pairs;
  G.pair_weights = g.pair_weights;
  G.packed3 = (const uint4*)g.packed3;
  G.scales3 = g.scales3;
  G.qzeros3 = (const uint32_t*)g.qzeros3;
  G.ypair = g.ypair;
  // token-box width: every expert may receive up to `rows` rows; boxes of 16 serve decode-sized batches with one block
  // per expert, larger batches take 128-row blocks (CTAs of blocks beyond an expert's count exit immediately)
  // (mode 1 holds two accumulator sets in the registers of the MMA warpgroup: blocks of at most 64 tokens)
  const int ntok = g.rows <= 16 ? 16 : g.rows <= 32 ? 32 : (g.rows <= 64 || mode == 1) ? 64 : 128;
  G.tblocks = (g.rows + ntok - 1) / ntok;
  const int grid_z = g.E * G.tblocks;
  int ks = env().midm_ks > 0 ? env().midm_ks : midm_grouped_ranks(a.K, a.N, g.active > 0 ? g.active : 1);
  if (ks > 8) ks = 8;
  const int nkb = a.K / MM_BK;
  while (ks > 1 && (ks - 1) * ((nkb + ks - 1) / ks) >= nkb) ks >>= 1;
  const bool asym = a.qzeros != nullptr;
#define B2Q_MG_NTOK(T, AS, MODE)                                                             \
  (ntok == 16   ? launch_midm_t<T, 4, AS, 16, 12, 8, MODE>(a, a.x, ks, G, g.rows, grid_z)    \
   : ntok == 32 ? launch_midm_t<T, 4, AS, 32, 12, 8, MODE>(a, a.x, ks, G, g.rows, grid_z)    \
   : ntok == 64 ? launch_midm_t<T, 4, AS, 64, 8, 8, MODE>(a, a.x, ks, G, g.rows, grid_z)     \
                : launch_midm_t<T, 4, AS, (MODE == 1 ? 64 : 128), (MODE == 1 ? 8 : 4), 8, MODE>(a, a.x, ks, G, g.rows, grid_z))
#define B2Q_MG_CASE(T)                                                                       \
  (mode == 1 ? (asym ? B2Q_MG_NTOK(T, true, 1) : B2Q_MG_NTOK(T, false, 1))                   \
             : (asym ? B2Q_MG_NTOK(T, true, 2) : B2Q_MG_NTOK(T, false, 2)))
  return a.dtype == 0 ? B2Q_MG_CASE(__half) : B2Q_MG_CASE(__nv_bfloat16);
#undef B2Q_MG_CASE
#undef B2Q_MG_NTOK
}

}  // namespace b2q
