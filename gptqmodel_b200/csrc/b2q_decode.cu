// b2q_decode.cu — decode tier for 4-bit weights: out[M, N] = x[M, K] @ dequant(W) for M <= 8 (batch-1 decode and
// small speculative / multi-sequence batches), HBM-bound.
//
// 8,732,672 algorithmic bytes for 4096x4096 g128 at M=1 (BASELINE.md §2); the roofline is the HBM copy bandwidth.
// Multiplying on the CUDA cores (as b2q_gemv.cu does for 8-bit) is issue-bound: ~156 warp-instructions per 1024
// weights.  This tier needs ~27:
//  * the prepacked T4 layout stores every 32-bit word as the four A-operand registers of one
//    mma.sync.m16n8k16 (16 features x 16 k): 4 LOP3 + 1 SHF produce them as exact 1024+q / 1024+16q halves, with
//    NO per-weight scaling, zero-point subtraction or conversion;
//  * the tensor pipe accumulates sum_k (bias+q) * x in fp32 for all (<= 8) tokens at once; once per quantisation
//    group the accumulators are folded into the running output with ONE fp32 fix-up per (feature, token):
//        out += s * (acc * c - (bias + z) * sum_k x)     (c = 1 or 1/16; sum_k x pre-reduced in shared memory)
//    which is algebraically the reference's  s * (q - z)  applied inside the sum (qlinear/__init__.py:1001-1003);
//  * grid = (N/32 feature tiles) x (KS split-K CTAs in a thread-block cluster); partial sums are reduced through
//    distributed shared memory (no atomics, no workspace, no output zeroing, deterministic);
//  * each warp's first ring stages (weights + their scales, b2q_decode.cuh issue_quad) are requested BEFORE
//    griddepcontrol.wait (programmatic dependent launch): weights never depend on the previous kernel;
//  * act-order: rows sorted by group at prepack; the activation staging reads x and the INVERSE permutation coalesced
//    and scatters into shared memory (stage_x_act_order, b2q_decode.cuh).
// Replaces the decode tiers of swordfish_mm (swordfish_mm.cu:216-286, mma.sync + cp.async + atomics) and Marlin's
// small-M path (marlin_template.h) in the reference.
#include "b2q_common.cuh"
#include "b2q_decode.cuh"
#include "b2q_internal.h"

namespace b2q {

// MOE: a separate instantiation for the one-token MoE launches (DecSets::moe), so that the dense kernels carry none of it
template <typename T, bool ASYM, bool G64, bool MOE>
__global__ void __launch_bounds__(DEC_MAX_WARPS * 32)
    decode_kernel(const __grid_constant__ DecSets S, const int32_t* __restrict__ perm, const T* __restrict__ x, int M,
                  int K, int gsh, int qpc, int max_tiles, int stl, const __grid_constant__ DecodeAR ar) {
  using E = ET<T>;
  extern __shared__ __align__(128) uint8_t dsm[];
  // MoE decode (DecSets::moe): the experts are data of an earlier kernel, so nothing expert-dependent may be prefetched
  // ahead of the PDL wait — the wait moves to the top (the later one is then a no-op)
  if (MOE) asm volatile("griddepcontrol.wait;" ::: "memory");
  // dynamic smem: ring[nwarps][DEC_STAGES][2 KB] | sx[M][kspan] (T) | xsum[kblocks][8] | red[2][nwarps][8][32] |
  //               part[max_tiles][8][32] | mbarriers[nwarps][DEC_STAGES] | scale slots[nwarps][nst][SCB]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  // The CTA walks tiles tile0, tile0 + C, ...; all `gw` warps split the k-quads of every tile (wg = warp's index).
  const int gw = nwarps, wg = warp;
  const int C = gridDim.x;                      // tile stride of a CTA
  const int tile0 = (int)blockIdx.x;
  const int TT = S.tile_end[S.nsets - 1];       // tiles of all sets
  const int ntiles = (tile0 < TT) ? (TT - tile0 + C - 1) / C : 0;  // tiles of this CTA
  const int nquads = K >> 7;
  // moe == 2: every cluster rank owns a whole expert (k-range 0 .. K of ITS weights) and its own row of activations
  const int q0 = (MOE && S.moe >= 2) ? 0 : blockIdx.y * qpc;
  const int q1 = min(q0 + qpc, nquads);
  const int kspan = qpc * 128;
  if (MOE && S.moe >= 2) x += (size_t)blockIdx.y * K * (S.moe == 3 ? 2 : 1);  // row r (or rows 2r, 2r + 1) of the rank
  const int nst = 1 << stl;  // ring stages per warp (2 or 4)
  uint8_t* ring = dsm + (size_t)warp * nst * DEC_QUAD_BYTES;
  T* sx = reinterpret_cast<T*>(dsm + (size_t)nwarps * nst * DEC_QUAD_BYTES);
  float* xsum = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(sx) + (size_t)M * kspan * sizeof(T));
  float* red = xsum + qpc * 2 * 8;
  float* part = red + 2 * nwarps * 256;  // [max_tiles][256]
  const uint32_t bars = smem_u32(part + max_tiles * 256) + warp * DEC_STAGES * 8;
  constexpr int NG = G64 ? 2 : 1, SCB = dec_sc_bytes(ASYM, G64);
  const uint32_t sring_w = smem_u32(part + max_tiles * 256) + nwarps * DEC_STAGES * 8 + warp * nst * SCB;
  const bool PERM = perm != nullptr;

  // ---- 1. the first DEC_STAGES quads of this warp requested before anything else -----------------
  const int nq = (q0 + wg < q1) ? (q1 - q0 - wg + gw - 1) / gw : 0;  // quads per tile for this warp
  const int U = ntiles * nq;                                                     // units of this warp
  // issue cursor (lane 0): quads of a tile are 2*nwarps k-blocks apart; the tile -> (weight set, local tile) mapping is
  // resolved once per tile
  // quantisation groups between consecutive quads of this warp, and the group of its first quad in every tile
  const int gstep = (2 * gw) >> gsh;
  const int g_first = (2 * (q0 + wg)) >> gsh;
  const uint4* iss_src = nullptr;
  const T* iss_sc = nullptr;          // scale row of the next quad to issue (features of its tile)
  const uint32_t* iss_zq = nullptr;   // qzeros row of the same
  int iss_N = 0;
  size_t iss_kbs = 0;  // k-block stride (uint4) of the set being issued
  int iss_q = 0, iss_u = 0, iss_ti = 0;
  auto iss_begin_tile = [&]() {
    const TileRef<T> r = resolve_tile<T, MOE>(S, tile0 + iss_ti * C);
    iss_kbs = (size_t)(r.N >> 4) * 32;
    iss_src = r.w + (size_t)(2 * (q0 + wg)) * iss_kbs + (size_t)(2 * r.nt) * 32;
    iss_N = r.N;
    iss_sc = r.sc + (size_t)g_first * r.N + r.nt * 32;
    if (ASYM) iss_zq = r.zq + (size_t)g_first * (r.N >> 3) + r.nt * 4;
  };
  auto iss_one = [&](uint32_t dst, uint32_t sdst, uint32_t bar) {
    issue_quad<T, ASYM, G64>(dst, sdst, bar, iss_src, iss_kbs, iss_sc, iss_zq, iss_N);
    ++iss_u;
    if (++iss_q == nq) {
      iss_q = 0;
      ++iss_ti;
      if (iss_u < U) iss_begin_tile();
    } else {
      iss_src += (size_t)(2 * gw) * iss_kbs;
      iss_sc += (size_t)gstep * iss_N;
      if (ASYM) iss_zq += (size_t)gstep * (iss_N >> 3);
    }
  };
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < DEC_STAGES; ++i) mbar_init(bars + 8 * i, 1);
    fence_mbar_init();
    if (U > 0) iss_begin_tile();
#pragma unroll
    for (int i = 0; i < DEC_STAGES; ++i)
      if (i < nst && iss_u < U) iss_one(smem_u32(ring) + i * DEC_QUAD_BYTES, sring_w + i * SCB, bars + 8 * i);
  }
  // scale / zero prefetch cursor (all lanes): this lane's 4 feature rows are +0, +8, +16, +24 from sc_next

  if (PERM) prefetch_inverse_perm(perm + K, K);
  // zero the token columns >= M of the block sums once (read by the fix-up of lanes whose columns are padding): own shared
  // memory, nothing to wait for — everything between griddepcontrol.wait and the first main-loop iteration is on the critical
  // path of every launch.  Without act-order every warp stages its own quads (stage_x_own_quads): no CTA barrier before
  // the main loop.
  if (!PERM) {
    zero_own_xsum_padding(xsum, M, nq, wg, gw);
  } else {
    for (int i = threadIdx.x; i < (q1 - q0) * 2 * 8; i += blockDim.x)
      if ((i & 7) >= M) xsum[i] = 0.f;
  }
  // PDL: let the next kernel start its own weight prefetch; wait for the producer of x only now.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");

  // ---- 2. stage x[m, k-range] (act-order gather fused) + per-(64 k block, token) sums, ONCE ------
  if (MOE && S.moe == 3) {
    stage_x_own_quads<T, true>(x, sx, xsum, 1, K, q0, nq, wg, gw, kspan);
  } else if (!PERM) {
    stage_x_own_quads<T>(x, sx, xsum, M, K, q0, nq, wg, gw, kspan);
  } else {
    stage_x_act_order<T>(x, perm + K, sx, xsum, M, K, q0 * 128, (q1 - q0) * 128, kspan);
  }
  if (PERM) __syncthreads();

  // ---- 3. loop over this CTA's tiles; inside a tile the warps split the k-quads --------------------
  // All loop-carried addresses are 32-bit shared-window addresses / running global pointers computed ONCE here:
  // recomputing them per quad costs about a third of the loop's instructions.
  constexpr float ZSYM = 8.f;
  const uint32_t nrank = cluster_nctarank();
  const uint32_t ring_a = smem_u32(ring) + lane * 16;
  const uint32_t xf_a0 = smem_u32(sx) + (uint32_t)((g * kspan + t * 16 + wg * 128) * 2);
  const uint32_t xs_a0 = smem_u32(xsum) + (uint32_t)((2 * t + wg * 16) * 4);
  const uint32_t xf_qstep = (uint32_t)gw * 256u, xs_qstep = (uint32_t)gw * 64u;
  // fused all-reduce: the sequence number of this call (advanced by the previous launch's last CTA)
  uint32_t ar_seq = 0;
  if (ar.world > 1) ar_seq = *reinterpret_cast<const volatile uint32_t*>(ar.ctl);
  int u = 0;
  for (int ti = 0; ti < ntiles; ++ti) {
    const TileRef<T> tr = resolve_tile<T, MOE>(S, tile0 + ti * C);
    const int nt = tr.nt, N = tr.N;
    const T* bias = tr.bias;
    T* out = tr.out;
    float tot[2][4];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) tot[a][b] = 0.f;

    uint32_t xf_a = xf_a0, xs_a = xs_a0;
    for (int qi = 0; qi < nq; ++qi, ++u, xf_a += xf_qstep, xs_a += xs_qstep) {
      const int st = u & (nst - 1);
      mbar_wait(bars + 8 * st, (uint32_t)(u >> stl) & 1u);
      const uint32_t wq_a = ring_a + st * DEC_QUAD_BYTES;
      const uint32_t sc_a = sring_w + st * SCB;  // this quad's scales / zeros (complete with the stage's barrier)
      float dd[2][2][4];  // [kbl][ftl][c]: four independent mma accumulator chains
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
          for (int c = 0; c < 4; ++c) dd[a][b][c] = 0.f;
      float xs0 = 0.f, xs1 = 0.f;  // sum_k x for token columns 2t, 2t+1 over the current group
#pragma unroll
      for (int kbl = 0; kbl < 2; ++kbl) {
        // activation fragment: token (column) g, k = 64*kb + 16t .. +15  -> 8 registers, 2 per k-step
        uint32_t bx[8];
        if (g < M) {
          const uint4 x0 = lds128(xf_a + kbl * 128), x1 = lds128(xf_a + kbl * 128 + 16);
          bx[0] = x0.x; bx[1] = x0.y; bx[2] = x0.z; bx[3] = x0.w;
          bx[4] = x1.x; bx[5] = x1.y; bx[6] = x1.z; bx[7] = x1.w;
        } else {
#pragma unroll
          for (int r = 0; r < 8; ++r) bx[r] = 0u;
        }
#pragma unroll
        for (int ftl = 0; ftl < 2; ++ftl) {
          const uint4 wv = lds128(wq_a + (kbl * 2 + ftl) * 512);
          const uint32_t w[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
          for (int s = 0; s < 4; ++s) {
            uint32_t a[4];
            E::unpack_w4(w[s], a);
            mma_16816<T>(dd[kbl][ftl], a, bx[2 * s], bx[2 * s + 1]);
          }
        }
        const float2 xs = lds_f2(xs_a + kbl * 32);
        xs0 += xs.x;
        xs1 += xs.y;
        if (kbl == 1 || G64) {
          // group boundary: fold the raw accumulators into the output with the per-(group, feature) scale / zero
          const int gi = G64 ? kbl : 0;  // compile-time after unrolling
#pragma unroll
          for (int ftl = 0; ftl < 2; ++ftl) {
            const uint16_t slr = lds_u16(sc_a + gi * 64 + (ftl * 16 + g) * 2);
            const uint16_t shr = lds_u16(sc_a + gi * 64 + (ftl * 16 + g + 8) * 2);
            const float sl = E::to_f(*reinterpret_cast<const T*>(&slr));
            const float sh = E::to_f(*reinterpret_cast<const T*>(&shr));
            float zl = ZSYM, zh = ZSYM;
            if (ASYM) {
              zl = (float)((lds_u32(sc_a + NG * 64 + gi * 16 + ftl * 8) >> (4 * g)) & 15u);  // feature % 8 == g for all rows
              zh = (float)((lds_u32(sc_a + NG * 64 + gi * 16 + ftl * 8 + 4) >> (4 * g)) & 15u);
            }
            const float bl = E::LO_BASE + zl, bh = E::HI_BASE + zh;
            float d[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) d[c] = G64 ? dd[kbl][ftl][c] : dd[0][ftl][c] + dd[1][ftl][c];
            tot[ftl][0] = fmaf(sl, d[0] - bl * xs0, tot[ftl][0]);
            tot[ftl][1] = fmaf(sl, d[1] - bl * xs1, tot[ftl][1]);
            tot[ftl][2] = fmaf(sh, d[2] * E::HI_SCALE - bh * xs0, tot[ftl][2]);
            tot[ftl][3] = fmaf(sh, d[3] * E::HI_SCALE - bh * xs1, tot[ftl][3]);
          }
          xs0 = xs1 = 0.f;
        }
      }
      // recycle the stage for the next not-yet-issued unit (all lanes have finished reading it)
      __syncwarp();
      if (lane == 0 && iss_u < U) iss_one(ring_a + st * DEC_QUAD_BYTES, sring_w + st * SCB, bars + 8 * st);
    }

    // ---- tile epilogue: warps -> CTA through (double-buffered) smem, one barrier per tile ---------
    // (decoupled variants — "last warp to arrive reduces", "rotating reducer warp on a split arrive/sync named
    //  barrier" — add synchronisation without removing the barrier's latency)
    // tot[ftl][c]: feature nt*32 + ftl*16 + g (+8 if c >= 2), token 2t + (c & 1)
    float* rbuf = red + (ti & 1) * gw * 256;
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) rbuf[(wg * 8 + a * 4 + b) * 32 + lane] = tot[a][b];
    asm volatile("bar.sync 1, %0;" ::"r"(gw * 32) : "memory");
    for (int i = wg * 32 + lane; i < 256; i += gw * 32) {
      float v = 0.f;
      for (int w = 0; w < gw; ++w) v += rbuf[w * 256 + i];
      if (nrank > 1) {
        part[ti * 256 + i] = v;
      } else {
        const int acc = i >> 5, ln = i & 31;
        const int m = 2 * (ln & 3) + (acc & 1);
        if (m < M) {
          const int n = nt * 32 + (acc >> 2) * 16 + (ln >> 2) + ((acc & 2) ? 8 : 0);
          if (ar.world > 1) {
            // row-parallel shard + all-reduce in this launch (launch_decode_allreduce: one tile per CTA, no split-K): the
            // fp32 partial sum goes into slot (seq & 1), row `rank`, of EVERY rank's symmetric buffer; the bias of a
            // row-parallel layer lives on one rank only and joins that rank's partial
            if (bias != nullptr) v += E::to_f(bias[n]);
            const size_t o = ((size_t)(ar_seq & 1u) * ar.world + ar.rank) * (size_t)ar.max_elems + (size_t)m * N + n;
            for (int p = 0; p < ar.world; ++p) reinterpret_cast<float*>(ar.buf[p])[o] = v;
          } else {
            // reference order: round the matmul to the output dtype, then add bias (qlinear/torch.py:337-342)
            T o = E::from_f(v);
            if (bias != nullptr) o = E::from_f(E::to_f(o) + E::to_f(bias[n]));
            out[(size_t)m * N + n] = o;
          }
        }
      }
    }
  }

  // ---- 3b. fused all-reduce across GPUs (same protocol as decode2_kernel; one tile per CTA, nrank == 1) ------------
  if (ar.world > 1) {
    __threadfence_system();  // the pushed partial sums are visible system-wide before the flag
    __syncthreads();
    const int cta = (int)blockIdx.x;
    if ((int)threadIdx.x < ar.world) {
      const int p = threadIdx.x;
      uint32_t* peer_flags = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(ar.buf[p]) + ar.flag_offset);
      asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(peer_flags + ar.rank * 160 + cta), "r"(ar_seq + 1u)
                   : "memory");
      const uint32_t* my_flags =
          reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(ar.buf[ar.rank]) + ar.flag_offset);
      if (!spin_until_geq_sys(my_flags + p * 160 + cta, ar_seq + 1u)) ar.ctl[2] = 1u + (uint32_t)p;  // dead peer
    }
    __syncthreads();
    if (ntiles > 0) {
      const TileRef<T> tr = resolve_tile<T, MOE>(S, tile0);
      const float* mine = reinterpret_cast<const float*>(ar.buf[ar.rank]) + (size_t)(ar_seq & 1u) * ar.world * ar.max_elems;
      for (int i = wg * 32 + lane; i < 256; i += gw * 32) {
        const int acc = i >> 5, ln = i & 31;
        const int m = 2 * (ln & 3) + (acc & 1);
        if (m < M) {
          const int n = tr.nt * 32 + (acc >> 2) * 16 + (ln >> 2) + ((acc & 2) ? 8 : 0);
          float v = 0.f;
          for (int p = 0; p < ar.world; ++p) v += __ldcg(mine + (size_t)p * ar.max_elems + (size_t)m * tr.N + n);
          tr.out[(size_t)m * tr.N + n] = E::from_f(v);  // summed in rank order: identical on every rank
        }
      }
    }
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned total = gridDim.x * gridDim.y;
      if (atomicAdd(ar.ctl + 1, 1u) == total - 1u) {  // every CTA has read seq: the last one advances it
        ar.ctl[1] = 0u;
        __threadfence();
        *reinterpret_cast<volatile uint32_t*>(ar.ctl) = ar_seq + 1u;
      }
    }
  }

  // ---- 4. split-K: the cluster ranks share the tiles of the final DSMEM reduction -----------------
  if (nrank > 1) {
    __syncthreads();  // every tile's reducer has written its partials
    cluster_sync_all();
    const uint32_t rank = cluster_ctarank();
    for (int ti = (int)rank; ti < ntiles; ti += (int)nrank) {
      const TileRef<T> tr = resolve_tile<T, MOE>(S, tile0 + ti * C);
      const int nt = tr.nt, N = tr.N;
      const T* bias = tr.bias;
      T* out = tr.out;
      for (int i = wg * 32 + lane; i < 256; i += gw * 32) {
        const int acc = i >> 5, ln = i & 31;
        const int m = 2 * (ln & 3) + (acc & 1);
        if (m < M) {
          float v = 0.f;
          for (uint32_t r = 0; r < nrank; ++r) {
            float pr = ld_dsmem_f32(smem_u32(&part[ti * 256 + i]), r);
            // MoE down: rank r holds expert r's complete output: y_r = T(h_r W2) like the module, then the routing weight
            if (MOE && S.moe >= 2) pr = S.wts[r] * E::to_f(E::from_f(pr));
            v += pr;
          }
          const int n = nt * 32 + (acc >> 2) * 16 + (ln >> 2) + ((acc & 2) ? 8 : 0);
          T o = E::from_f(v);
          if (bias != nullptr) o = E::from_f(E::to_f(o) + E::to_f(bias[n]));
          out[(size_t)m * N + n] = o;
        }
      }
    }
    cluster_sync_all();  // keep every rank's smem alive until all peers have read it
  }
}

static size_t decode_smem(const MmArgs& a, int warps, int qpc, int max_tiles, int nst) {
  const int scb = dec_sc_bytes(a.qzeros != nullptr, a.group_size == 64);
  return (size_t)warps * nst * DEC_QUAD_BYTES + (size_t)a.M * qpc * 128 * 2 + (size_t)qpc * 2 * 8 * 4 +
         (size_t)2 * warps * 256 * 4 + (size_t)max_tiles * 256 * 4 + (size_t)warps * DEC_STAGES * 8 +
         (size_t)warps * nst * scb + 16;
}

// Pick (C tile-columns, ks split-K ranks, warps) minimising the critical path in "quads per warp" on one CTA per SM.
static bool decode_config(const MmArgs& a, int NT, DecodePlan& best) {
  const int quads = a.K / 128;
  const int SMS = num_sms();
  double best_cost = 1e30;
  bool found = false;
  for (int ks = 1; ks <= 8; ks *= 2) {
    if (a.tune_ks > 0 && ks != a.tune_ks) continue;
    if (ks > quads) break;
    const int qpc = (quads + ks - 1) / ks;
    for (int warps = 4; warps <= DEC_MAX_WARPS; warps *= 2) {  // 4, 8, 16
      if (a.tune_warps > 0 && warps != a.tune_warps) continue;
      int C = SMS / ks;
      if (C > NT) C = NT;
      if (C < 1) C = 1;
      const int max_tiles = (NT + C - 1) / C;
      DecodePlan p = {C, ks, warps, warps, qpc, ks > 1 ? max_tiles : 0, 0, 0};
      if (!fit_ring(p, [&](int nst) { return decode_smem(a, warps, qpc, p.max_tiles, nst); })) continue;
      const int qpw = (qpc + warps - 1) / warps;  // quads per warp per tile
      // relative cost in units of one quad per warp: per tile = quads/warp + barrier epilogue, split-K adds a cluster
      // barrier + DSMEM pass, fewer warps hide less latency (the weights are heuristic, not fitted to one GPU)
      const double cost =
          (double)max_tiles * (qpw + 0.35) + (ks > 1 ? 0.6 : 0.0) + (16 - warps) * 0.04 * max_tiles * qpw;
      if (cost < best_cost) {
        best_cost = cost;
        best = p;
        found = true;
      }
    }
  }
  return found;
}

// Host-side planner query (b2q_debug_decode_plan): {C, ks, warps, warps per group, quads per CTA, max tiles per group,
// ring stages, dynamic shared memory bytes}
bool decode_plan(int version, const MmArgs& a, int NT, int* out8) {
  DecodePlan c;
  if (!(version == 2 ? decode2_config(a, NT, c) : decode_config(a, NT, c))) return false;
  const int v[8] = {c.C, c.ks, c.warps, c.gw, c.qpc, c.max_tiles, 1 << c.stl, (int)c.smem};
  for (int i = 0; i < 8; ++i) out8[i] = v[i];
  return true;
}

int decode2_occupancy(const DecodePlan& c, int* blocks);  // b2q_decode2.cu

int decode_occupancy(int version, const MmArgs& a, int NT, int* blocks) {
  DecodePlan c;
  if (!(version == 2 ? decode2_config(a, NT, c) : decode_config(a, NT, c))) {
    set_error("b2q_debug_decode_occupancy: no configuration fits shared memory (version=%d M=%d K=%d N=%d)", version,
              a.M, a.K, a.N);
    return -1;
  }
  if (version == 2) return decode2_occupancy(c, blocks);
  return plan_occupancy(decode_kernel<__half, false, false, false>, c, blocks);
}

template <typename I>
static int launch_decode_t(const MmArgs& a, const DecSets& sets, const DecodePlan& c, const DecodeAR& ar) {
  using T = typename I::T;
  auto kern = decode_kernel<T, I::ASYM, I::G64, I::MOE>;
  static int smem_opted[32] = {};
  if (int e = ensure_dyn_smem(kern, (int)c.smem, smem_opted, "b2q_decode")) return e;
  return launch_kernel(kern, dim3(c.C, c.ks, 1), dim3(c.warps * 32, 1, 1), c.smem, a.stream, c.ks, true, sets, a.perm,
                       (const T*)a.x, a.M, a.K, decode_gsh(a.group_size), c.qpc, c.max_tiles, c.stl, ar);
}

static int launch_decode_plan(const MmArgs& a, const DecSets& sets, const DecodePlan& c, const DecodeAR& ar) {
  if (!sets_aligned(sets, "b2q_decode")) return -1;
  return dispatch_decode(a, sets, [&](auto inst) { return launch_decode_t<decltype(inst)>(a, sets, c, ar); });
}

bool decode_supported(const MmArgs& a) {
  return a.bits == 4 && a.M >= 1 && a.M <= DEC_MAXM && a.K % 128 == 0 && a.N % 32 == 0 &&
         (a.group_size == 64 || a.group_size == 128 || a.group_size == a.K);
}

int launch_decode2_sets(const MmArgs& a, const DecSets& sets);  // b2q_decode2.cu, -2 = no configuration

static int launch_decode_sets(const MmArgs& a, const DecSets& sets) {
  // Kernel choice per launch shape: launches whose CTAs walk SEVERAL 32-feature tiles (more tiles than SMs: fused q|k|v,
  // gate|up) run on decode2_kernel with one 16-warp group and no split-K — warps park their partial sums and the CTA meets
  // once; the others keep decode_kernel.  Measured on an H100 80GB HBM3 (700 W limit, power-capped; results/h100_bench.json):
  // Llama-3-8B decode 588 tok/s with this choice, 528 with decode_kernel everywhere, 604 with decode2_kernel everywhere —
  // but decode2_kernel everywhere dropped the Llama-3-70B TP-8 shard stack from 372 to 277 tok/s and Mixtral TP-4 from 647
  // to 607, so it is not the default.  B2Q_DECODE_V2=1 / 0 forces one kernel for A/B runs.
  {
    const int mode = env().decode_v2;  // -1 auto, 0 never, 1 always
    const int NT = sets.tile_end[sets.nsets - 1];
    if (mode == 1 || (mode < 0 && NT > num_sms() && a.tune_ks <= 0 && a.tune_warps <= 0)) {
      MmArgs a2 = a;
      if (mode < 0) {  // one 16-warp group, no split-K
        a2.tune_ks = 1;
        a2.tune_warps = 16;
      }
      const int rc = launch_decode2_sets(a2, sets);
      if (rc != -2) return rc;
    }
  }
  DecodePlan c;
  if (!decode_config(a, sets.tile_end[sets.nsets - 1], c)) {
    set_error("b2q_decode: no configuration fits shared memory for M=%d K=%d (ks=%d warps=%d)", a.M, a.K, a.tune_ks,
              a.tune_warps);
    return -1;
  }
  return launch_decode_plan(a, sets, c, DecodeAR{});
}

// Row-parallel shard + all-reduce on decode_kernel: only for launches in which every CTA owns at most ONE tile and K is not
// split (o_proj / down_proj of a 4096-wide model at any TP degree: 128 tiles) — where decode_kernel is the faster of the
// two decode kernels; everything else takes decode2_kernel's epilogue.  -2 = not applicable.
int launch_decode1_allreduce(const MmArgs& a, const DecSets& sets, const DecodeAR& ar) {
  const int NT = sets.tile_end[sets.nsets - 1];
  if (NT > num_sms() || a.perm != nullptr) return -2;
  MmArgs a1 = a;
  a1.tune_ks = 1;
  DecodePlan c;
  if (!decode_config(a1, NT, c) || c.ks != 1 || c.C < NT || c.C > 160) return -2;
  return launch_decode_plan(a1, sets, c, ar);
}

int launch_decode(const MmArgs& a) {
  if (!decode_supported(a)) {
    set_error("b2q_decode: unsupported (bits=%d M=%d K=%d N=%d group=%d)", a.bits, a.M, a.K, a.N, a.group_size);
    return -1;
  }
  return launch_decode_sets(a, layer_sets(a));
}

// Sibling QuantLinears (same x, same K / group size / symmetry, no act-order) in ONE launch.
int launch_decode_multi(const MmArgs& a, int nsets, const void* const* packed, const void* const* scales,
                        const int32_t* const* qzeros, const void* const* bias, void* const* out, const int* Ns) {
  if (nsets < 1 || nsets > DEC_MAX_SETS) {
    set_error("b2q_decode_multi: nsets=%d out of range (1..%d)", nsets, DEC_MAX_SETS);
    return -1;
  }
  DecSets sets = {};
  sets.nsets = nsets;
  int tiles = 0;
  for (int i = 0; i < nsets; ++i) {
    MmArgs ai = a;
    ai.N = Ns[i];
    if (!decode_supported(ai) || Ns[i] % 32 != 0 || packed[i] == nullptr || scales[i] == nullptr ||
        out[i] == nullptr || ((qzeros[i] != nullptr) != (qzeros[0] != nullptr))) {
      set_error("b2q_decode_multi: set %d unsupported (N=%d; all sets must share bits=4, K, group size and symmetry)", i,
                Ns[i]);
      return -1;
    }
    tiles += Ns[i] / 32;
    sets.tile_end[i] = tiles;
    sets.N[i] = Ns[i];
    sets.packed[i] = (const uint4*)packed[i];
    sets.scales[i] = scales[i];
    sets.qzeros[i] = (const uint32_t*)qzeros[i];
    sets.bias[i] = bias[i];
    sets.out[i] = out[i];
  }
  for (int i = nsets; i < DEC_MAX_SETS; ++i) sets.tile_end[i] = tiles;
  MmArgs a0 = a;
  a0.qzeros = qzeros[0];
  return launch_decode_sets(a0, sets);
}

// ---- MoE decode: one token, top_k experts chosen on the device (DecSets::moe; b2q_moe_decode_*) -------------------------
// The grouped small-batch kernels (b2q_midm.cu MODE 1 / 2) pad a single token to MMA tiles of >= 16 token columns; the
// decode tier streams the same bytes without that padding.  gate | up: the 2 * top_k (expert, w1 | w3)
// matrices are virtual sibling sets of ONE decode launch over the same activations.  down: a cluster of top_k CTAs per tile
// column, rank r multiplying pair r's activations with ITS expert's w2; the DSMEM reduction applies the routing weights.
static void moe_strides(DecSets& sets, int K, int N, int group_size) {
  const size_t G = (size_t)K / (size_t)group_size;
  sets.estride_w = (size_t)K * (size_t)N / 2 / 16;  // uint4
  sets.estride_s = G * (size_t)N;                   // elements
  sets.estride_z = G * (size_t)N / 8;               // uint32
}

int launch_moe_decode_gate_up(const MmArgs& a, const void* packed1, const void* scales1, const int32_t* qzeros1,
                              const void* packed3, const void* scales3, const int32_t* qzeros3, const int32_t* ids,
                              int top_k, int E, void* gu) {
  if (!decode_supported(a) || a.M != 1 || top_k < 1 || top_k > 8 || (qzeros1 != nullptr) != (qzeros3 != nullptr)) {
    set_error("b2q_moe_decode_gate_up: needs one token, bits=4, K %% 128 == 0, group_size 64|128|K, 1 <= top_k <= 8 "
              "(M=%d K=%d N=%d g=%d top_k=%d)", a.M, a.K, a.N, a.group_size, top_k);
    return -1;
  }
  DecSets sets = {};
  sets.nsets = 1;
  const int tiles = 2 * top_k * (a.N / 32);
  for (int i = 0; i < DEC_MAX_SETS; ++i) sets.tile_end[i] = tiles;
  sets.N[0] = a.N;
  sets.packed[0] = (const uint4*)packed1;
  sets.packed[1] = (const uint4*)packed3;
  sets.scales[0] = scales1;
  sets.scales[1] = scales3;
  sets.qzeros[0] = (const uint32_t*)qzeros1;
  sets.qzeros[1] = (const uint32_t*)qzeros3;
  sets.out[0] = gu;
  sets.moe = 1;
  sets.nexperts = E;
  sets.ids = ids;
  moe_strides(sets, a.K, a.N, a.group_size);
  MmArgs a0 = a;
  a0.qzeros = qzeros1;
  a0.perm = nullptr;
  a0.bias = nullptr;
  a0.out = gu;
  return launch_decode_sets(a0, sets);
}

int launch_moe_decode_down(const MmArgs& a, const int32_t* ids, const float* wts, int top_k, int E, int fused_act) {
  if (!decode_supported(a) || a.M != 1 || !(top_k == 2 || top_k == 4 || top_k == 8)) {
    set_error("b2q_moe_decode_down: needs one token, bits=4, K %% 128 == 0, group_size 64|128|K, top_k 2|4|8 (M=%d K=%d N=%d "
              "g=%d top_k=%d)", a.M, a.K, a.N, a.group_size, top_k);
    return -1;
  }
  MmArgs a0 = a;
  a0.perm = nullptr;
  a0.bias = nullptr;
  DecSets sets = layer_sets(a0);
  sets.moe = fused_act ? 3 : 2;
  sets.nexperts = E;
  sets.ids = ids;
  sets.wts = wts;
  moe_strides(sets, a.K, a.N, a.group_size);
  const int NT = a.N / 32;
  DecodePlan c = {};
  c.ks = top_k;
  c.warps = c.gw = DEC_MAX_WARPS;
  c.qpc = a.K / 128;  // a rank's k-range is its expert's whole K
  c.C = num_sms() / top_k;
  if (c.C > NT) c.C = NT;
  c.max_tiles = (NT + c.C - 1) / c.C;
  if (!fit_ring(c, [&](int nst) { return decode_smem(a, c.warps, c.qpc, c.max_tiles, nst); })) {
    set_error("b2q_moe_decode_down: K=%d does not fit shared memory", a.K);
    return -1;
  }
  return launch_decode_plan(a0, sets, c, DecodeAR{});
}

}  // namespace b2q
