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
//  * every lane issues its 4 x LDG.128 of weights (+ scales) BEFORE griddepcontrol.wait (programmatic dependent
//    launch): weights never depend on the previous kernel, so consecutive layers overlap their HBM streams;
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
                  int K, int gsh, int qpc, int max_tiles, int ngroups, int stl,
                  const __grid_constant__ DecodeAR ar, unsigned long long* __restrict__ trace) {
  using E = ET<T>;
  extern __shared__ __align__(128) uint8_t dsm[];
  // optional phase timestamps (debug): trace[blockIdx.x * 16 + slot] = %globaltimer (ns)
  auto stamp = [&](int slot) {
    if (trace != nullptr && threadIdx.x == 0 && blockIdx.y == 0) {
      unsigned long long tns;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tns));
      trace[blockIdx.x * 16 + slot] = tns;
    }
  };
  stamp(0);
  // MoE decode (DecSets::moe): the experts are data of an earlier kernel, so nothing expert-dependent may be prefetched
  // ahead of the PDL wait — the wait moves to the top (the later one is then a no-op)
  if (MOE) asm volatile("griddepcontrol.wait;" ::: "memory");
  // dynamic smem: ring[nwarps][DEC_STAGES][2 KB] | sx[M][kspan] (T) | xsum[kblocks][8] | red[2][nwarps][8][32] |
  //               part[max_tiles][8][32] | mbarriers[nwarps][DEC_STAGES]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  // The CTA's warps form `ngroups` independent groups (1 or 2); a group owns whole tiles (group-strided over the
  // launch) and its `gw` warps split the k-quads of a tile.  With 2 groups, one group's tile epilogue (barrier + cross-
  // warp reduction, mostly latency) overlaps the other group's main loop on the same SM.
  const int gw = nwarps / ngroups;              // warps per group
  const int grp = warp / gw, wg = warp - grp * gw;
  const int C = gridDim.x * ngroups;            // tile stride of a group
  const int tile0 = (int)blockIdx.x * ngroups + grp;
  const int TT = S.tile_end[S.nsets - 1];       // tiles of all sets
  const int ntiles = (tile0 < TT) ? (TT - tile0 + C - 1) / C : 0;  // tiles of this group
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
  float* part = red + 2 * nwarps * 256;  // [ngroups][max_tiles][256]
  const uint32_t bars = smem_u32(part + max_tiles * 256) + warp * DEC_STAGES * 8;
  const bool PERM = perm != nullptr;

  // ---- 1. the first DEC_STAGES quads of this warp requested before anything else -----------------
  const int nq = (q0 + wg < q1) ? (q1 - q0 - wg + gw - 1) / gw : 0;  // quads per tile for this warp
  const int U = ntiles * nq;                                                     // units of this warp
  // issue cursor (lane 0): quads of a tile are 2*nwarps k-blocks apart; the tile -> (weight set, local tile) mapping is
  // resolved once per tile
  const uint4* iss_src = nullptr;
  size_t iss_kbs = 0;  // k-block stride (uint4) of the set being issued
  int iss_q = 0, iss_u = 0, iss_ti = 0;
  auto iss_begin_tile = [&]() {
    const TileRef<T> r = resolve_tile<T, MOE>(S, tile0 + iss_ti * C);
    iss_kbs = (size_t)(r.N >> 4) * 32;
    iss_src = r.w + (size_t)(2 * (q0 + wg)) * iss_kbs + (size_t)(2 * r.nt) * 32;
  };
  auto iss_one = [&](uint32_t dst, uint32_t bar) {
    issue_quad(dst, bar, iss_src, iss_kbs);
    ++iss_u;
    if (++iss_q == nq) {
      iss_q = 0;
      ++iss_ti;
      if (iss_u < U) iss_begin_tile();
    } else {
      iss_src += (size_t)(2 * gw) * iss_kbs;
    }
  };
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < DEC_STAGES; ++i) mbar_init(bars + 8 * i, 1);
    fence_mbar_init();
    if (U > 0) iss_begin_tile();
#pragma unroll
    for (int i = 0; i < DEC_STAGES; ++i)
      if (i < nst && iss_u < U) iss_one(smem_u32(ring) + i * DEC_QUAD_BYTES, bars + 8 * i);
  }
  // scale / zero prefetch cursor (all lanes): this lane's 4 feature rows are +0, +8, +16, +24 from sc_next
  const int gstep = (2 * gw) >> gsh;           // quantisation groups between consecutive quads of this warp
  const int g_first = (2 * (q0 + wg)) >> gsh;  // quantisation group of this warp's first quad in every tile
  const T* sc_next = nullptr;
  const uint32_t* zq_next = nullptr;
  int pre_q = 0, pre_ti = 0, pre_N = 0;
  auto pre_begin_tile = [&]() {
    const TileRef<T> r = resolve_tile<T, MOE>(S, tile0 + pre_ti * C);
    pre_N = r.N;
    sc_next = r.sc + (size_t)g_first * r.N + r.nt * 32 + g;
    if (ASYM) zq_next = r.zq + (size_t)g_first * (r.N >> 3) + r.nt * 4;
  };
  auto fetch_scales = [&](DScale<ASYM, G64>& d) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      d.s[0][i] = *reinterpret_cast<const uint16_t*>(sc_next + i * 8);
      if (ASYM) d.zw[0][i] = zq_next[i];
    }
    if (G64) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        d.s[G64 ? 1 : 0][i] = *reinterpret_cast<const uint16_t*>(sc_next + (size_t)pre_N + i * 8);
        if (ASYM) d.zw[G64 ? 1 : 0][i] = zq_next[(pre_N >> 3) + i];
      }
    }
    // advance to the next unit
    if (++pre_q == nq) {
      pre_q = 0;
      ++pre_ti;
      if (pre_ti < ntiles) pre_begin_tile();
    } else {
      sc_next += (size_t)gstep * pre_N;
      if (ASYM) zq_next += (size_t)gstep * (pre_N >> 3);
    }
  };
  DScale<ASYM, G64> cur;
  if (U > 0) {
    pre_begin_tile();
    fetch_scales(cur);
  }

  if (PERM) prefetch_inverse_perm(perm + K, K);
  // zero the token columns >= M of the block sums once (read by the fix-up of lanes whose columns are padding): own shared
  // memory, nothing to wait for — everything between griddepcontrol.wait and the first main-loop iteration is on the critical
  // path of every launch
  const bool OWN = !PERM && ngroups == 1;  // per-warp staging (stage_x_own_quads): no CTA barrier before the main loop
  if (OWN) {
    zero_own_xsum_padding(xsum, M, nq, wg, gw);
  } else {
    for (int i = threadIdx.x; i < (q1 - q0) * 2 * 8; i += blockDim.x)
      if ((i & 7) >= M) xsum[i] = 0.f;
  }
  // PDL: let the next kernel start its own weight prefetch; wait for the producer of x only now.
  stamp(1);
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  stamp(2);

  // ---- 2. stage x[m, k-range] (act-order gather fused) + per-(64 k block, token) sums, ONCE ------
  // A thread's loads (up to SX_UNROLL x 16 bytes, K = 14336 needs 3.5 per thread) are all issued BEFORE the first is
  // consumed: a rolled loop pays one dependent L2 round trip per iteration.
  if (MOE && S.moe == 3) {
    stage_x_own_quads<T, true>(x, sx, xsum, 1, K, q0, nq, wg, gw, kspan);
  } else if (OWN) {
    stage_x_own_quads<T>(x, sx, xsum, M, K, q0, nq, wg, gw, kspan);
  } else if (PERM) {
    stage_x_act_order<T>(x, perm + K, sx, xsum, M, K, q0 * 128, (q1 - q0) * 128, kspan);
  } else {
    const int n8 = (q1 - q0) * 16;   // uint4 (8 halves) per token row in this CTA's k-range
    const int tot = M * n8;
    const int totr = (tot + 31) & ~31;
    constexpr int SX_UNROLL = 4;
    auto f2 = [](uint32_t u) {
      const T* h = reinterpret_cast<const T*>(&u);
      return E::to_f(h[0]) + E::to_f(h[1]);
    };
    for (int i0 = threadIdx.x; i0 < totr; i0 += blockDim.x * SX_UNROLL) {
      uint4 xv[SX_UNROLL];
      int mm[SX_UNROLL], jj[SX_UNROLL];
#pragma unroll
      for (int u = 0; u < SX_UNROLL; ++u) {
        const int i = i0 + u * blockDim.x;
        xv[u] = make_uint4(0, 0, 0, 0);
        mm[u] = 0;
        jj[u] = 0;
        if (i < tot) {
          const int m = (M == 1) ? 0 : i / n8, j = i - m * n8;  // batch-1 decode: no integer division ahead of the load
          mm[u] = m;
          jj[u] = j;
          const T* xr = x + (size_t)m * K;
          xv[u] = reinterpret_cast<const uint4*>(xr + (size_t)q0 * 128)[j];
        }
      }
#pragma unroll
      for (int u = 0; u < SX_UNROLL; ++u) {
        const int i = i0 + u * blockDim.x;
        if (i < totr) {  // warp-uniform (totr and the strides are multiples of 32)
          if (i < tot) reinterpret_cast<uint4*>(sx + (size_t)mm[u] * kspan)[jj[u]] = xv[u];
          float sm = (f2(xv[u].x) + f2(xv[u].y)) + (f2(xv[u].z) + f2(xv[u].w));
          sm += __shfl_xor_sync(0xffffffffu, sm, 1);
          sm += __shfl_xor_sync(0xffffffffu, sm, 2);
          sm += __shfl_xor_sync(0xffffffffu, sm, 4);
          if ((i & 7) == 0 && i < tot) xsum[(jj[u] >> 3) * 8 + mm[u]] = sm;  // 8 uint4 = one 64-k block
        }
      }
    }
  }
  if (!OWN) __syncthreads();
  stamp(3);

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
      DScale<ASYM, G64> nxt;
      if (u + 1 < U) fetch_scales(nxt);
      const int st = u & (nst - 1);
      mbar_wait(bars + 8 * st, (uint32_t)(u >> stl) & 1u);
      const uint32_t wq_a = ring_a + st * DEC_QUAD_BYTES;
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
            const uint16_t slr = cur.s[gi][ftl * 2], shr = cur.s[gi][ftl * 2 + 1];
            const float sl = E::to_f(*reinterpret_cast<const T*>(&slr));
            const float sh = E::to_f(*reinterpret_cast<const T*>(&shr));
            float zl = ZSYM, zh = ZSYM;
            if (ASYM) {
              zl = (float)((cur.zw[ASYM ? gi : 0][ftl * 2] >> (4 * g)) & 15u);  // feature % 8 == g for all rows
              zh = (float)((cur.zw[ASYM ? gi : 0][ftl * 2 + 1] >> (4 * g)) & 15u);
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
      if (lane == 0 && iss_u < U) iss_one(ring_a + st * DEC_QUAD_BYTES, bars + 8 * st);
      if (u + 1 < U) cur = nxt;
    }

    // ---- tile epilogue: warps -> CTA through (double-buffered) smem, one barrier per tile ---------
    // (decoupled variants — "last warp to arrive reduces", "rotating reducer warp on a split arrive/sync named
    //  barrier" — add synchronisation without removing the barrier's latency)
    // tot[ftl][c]: feature nt*32 + ftl*16 + g (+8 if c >= 2), token 2t + (c & 1)
    if (ti < 5) stamp(4 + 2 * ti);
    float* rbuf = red + (grp * 2 + (ti & 1)) * gw * 256;
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) rbuf[(wg * 8 + a * 4 + b) * 32 + lane] = tot[a][b];
    asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(gw * 32) : "memory");  // this group's warps only
    for (int i = wg * 32 + lane; i < 256; i += gw * 32) {
      float v = 0.f;
      for (int w = 0; w < gw; ++w) v += rbuf[w * 256 + i];
      if (nrank > 1) {
        part[(grp * max_tiles + ti) * 256 + i] = v;
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
    if (ti < 5) stamp(5 + 2 * ti);
  }
  stamp(15);

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
    // each group reduces its own tiles (same tile <-> group mapping in every rank of the cluster)
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
            float pr = ld_dsmem_f32(smem_u32(&part[(grp * max_tiles + ti) * 256 + i]), r);
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

void* g_trace_ptr = nullptr;

struct DecodeCfg {
  int C, ks, warps, qpc, max_tiles, ngroups, stl;
  size_t smem;
};

static size_t decode_smem(int M, int warps, int qpc, int max_tiles, int nst) {
  return (size_t)warps * nst * DEC_QUAD_BYTES + (size_t)M * qpc * 128 * 2 + (size_t)qpc * 2 * 8 * 4 +
         (size_t)2 * warps * 256 * 4 + (size_t)max_tiles * 256 * 4 + (size_t)warps * DEC_STAGES * 8 + 16;
}

// Pick (C tile-columns, ks split-K ranks, warps) minimising the critical path in "quads per warp" on one CTA per SM.
static bool decode_config(const MmArgs& a, int NT, DecodeCfg& best) {
  const int quads = a.K / 128;
  const int SMS = num_sms();
  double best_cost = 1e30;
  bool found = false;
  const bool two_groups = env().decode_groups2 != 0;
  for (int ks = 1; ks <= 8; ks *= 2) {
    if (a.tune_ks > 0 && ks != a.tune_ks) continue;
    if (ks > quads) break;
    const int qpc = (quads + ks - 1) / ks;
    for (int warps = 4; warps <= DEC_MAX_WARPS; warps *= 2) {  // 4, 8, 16
      if (a.tune_warps > 0 && warps != a.tune_warps) continue;
      // two independent 8-warp groups per CTA overlap one group's tile epilogue with the other's main loop (+5 % on the
      // Llama-3-8B step) but one full-size parity case failed with it in round 1: experimental, off by default
      int ngroups = 1;
      if (two_groups && warps == 16 && ks == 1) ngroups = 2;  // (the split-K + groups combination faults)
      const int gwarps = warps / ngroups;
      int C = SMS / ks;
      if (C * ngroups > NT) C = (NT + ngroups - 1) / ngroups;
      if (C < 1) C = 1;
      const int max_tiles = (NT + C * ngroups - 1) / (C * ngroups);  // per group
      // ring depth 4 when it fits, else 2
      int stl = 2;
      size_t smem = decode_smem(a.M, warps, qpc, ks > 1 ? max_tiles * ngroups : 0, 4);
      if (smem > 200 * 1024) {
        stl = 1;
        smem = decode_smem(a.M, warps, qpc, ks > 1 ? max_tiles * ngroups : 0, 2);
      }
      if (smem > 200 * 1024) continue;
      const int qpw = (qpc + gwarps - 1) / gwarps;  // quads per warp per tile
      // relative cost in units of one quad per warp: per tile = quads/warp + barrier epilogue, split-K adds a cluster
      // barrier + DSMEM pass, fewer warps hide less latency (the weights are heuristic, not fitted to one GPU)
      const double cost =
          (double)max_tiles * (qpw + 0.35) / ngroups + (ks > 1 ? 0.6 : 0.0) + (16 - warps) * 0.04 * max_tiles * qpw;
      if (cost < best_cost) {
        best_cost = cost;
        best = DecodeCfg{C, ks, warps, qpc, ks > 1 ? max_tiles : 0, ngroups, stl, smem};
        found = true;
      }
    }
  }
  return found;
}

bool decode2_plan(const MmArgs& a, int NT, int* out8);  // b2q_decode2.cu

// Host-side planner query (b2q_debug_decode_plan): {C, ks, warps, warps per group, quads per CTA, max tiles per group,
// ring stages, dynamic shared memory bytes}
bool decode_plan(int version, const MmArgs& a, int NT, int* out8) {
  if (version == 2) return decode2_plan(a, NT, out8);
  DecodeCfg c;
  if (!decode_config(a, NT, c)) return false;
  const int v[8] = {c.C, c.ks, c.warps, c.warps / c.ngroups, c.qpc, c.max_tiles, 1 << c.stl, (int)c.smem};
  for (int i = 0; i < 8; ++i) out8[i] = v[i];
  return true;
}

template <typename T, bool ASYM, bool G64, bool MOE = false>
static int launch_decode_t(const MmArgs& a, const DecSets& sets, const DecodeCfg& c, const DecodeAR& ar) {
  auto kern = decode_kernel<T, ASYM, G64, MOE>;
  if (c.smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem);
    if (e != cudaSuccess) return (int)e;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(c.C, c.ks, 1);
  cfg.blockDim = dim3(c.warps * 32, 1, 1);
  cfg.dynamicSmemBytes = c.smem;
  cfg.stream = a.stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = c.ks;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = a.pdl ? 2 : 1;
  int gsh = 31;  // per-channel: every k-block is group 0
  if (a.group_size == 64) gsh = 0;
  else if (a.group_size == 128) gsh = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, sets, a.perm, (const T*)a.x, a.M, a.K, gsh, c.qpc, c.max_tiles,
                                     c.ngroups, c.stl, ar, (unsigned long long*)g_trace_ptr);
  return (int)e;
}

bool decode_supported(const MmArgs& a) {
  return a.bits == 4 && a.M >= 1 && a.M <= DEC_MAXM && a.K % 128 == 0 && a.N % 32 == 0 &&
         (a.group_size == 64 || a.group_size == 128 || a.group_size == a.K);
}

int launch_decode2_sets(const MmArgs& a, const DecSets& sets);  // b2q_decode2.cu (experimental), -2 = no configuration

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
  DecodeCfg c;
  if (!decode_config(a, sets.tile_end[sets.nsets - 1], c)) {
    set_error("b2q_decode: no configuration fits shared memory for M=%d K=%d (ks=%d warps=%d)", a.M, a.K, a.tune_ks,
              a.tune_warps);
    return -1;
  }
  const bool asym = a.qzeros != nullptr, g64 = a.group_size == 64;
  const DecodeAR none = {};
#define B2Q_DEC_CASE(T, MOE)                                                     \
  (asym ? (g64 ? launch_decode_t<T, true, true, MOE>(a, sets, c, none)           \
               : launch_decode_t<T, true, false, MOE>(a, sets, c, none))         \
        : (g64 ? launch_decode_t<T, false, true, MOE>(a, sets, c, none)          \
               : launch_decode_t<T, false, false, MOE>(a, sets, c, none)))
  if (sets.moe != 0) return a.dtype == 0 ? B2Q_DEC_CASE(__half, true) : B2Q_DEC_CASE(__nv_bfloat16, true);
  return a.dtype == 0 ? B2Q_DEC_CASE(__half, false) : B2Q_DEC_CASE(__nv_bfloat16, false);
#undef B2Q_DEC_CASE
}

// Row-parallel shard + all-reduce on decode_kernel: only for launches in which every CTA owns at most ONE tile and K is not
// split (o_proj / down_proj of a 4096-wide model at any TP degree: 128 tiles) — where decode_kernel is the faster of the
// two decode kernels; everything else takes decode2_kernel's epilogue.  -2 = not applicable.
int launch_decode1_allreduce(const MmArgs& a, const DecSets& sets, const DecodeAR& ar) {
  const int NT = sets.tile_end[sets.nsets - 1];
  if (NT > num_sms() || a.perm != nullptr) return -2;
  MmArgs a1 = a;
  a1.tune_ks = 1;
  DecodeCfg c;
  if (!decode_config(a1, NT, c) || c.ks != 1 || c.ngroups != 1 || c.C < NT || c.C > 160) return -2;
  const bool asym = a.qzeros != nullptr, g64 = a.group_size == 64;
#define B2Q_DEC_CASE(T)                                                          \
  (asym ? (g64 ? launch_decode_t<T, true, true>(a1, sets, c, ar)                 \
               : launch_decode_t<T, true, false>(a1, sets, c, ar))               \
        : (g64 ? launch_decode_t<T, false, true>(a1, sets, c, ar)                \
               : launch_decode_t<T, false, false>(a1, sets, c, ar)))
  return a.dtype == 0 ? B2Q_DEC_CASE(__half) : B2Q_DEC_CASE(__nv_bfloat16);
#undef B2Q_DEC_CASE
}

int launch_decode(const MmArgs& a) {
  if (!decode_supported(a)) {
    set_error("b2q_decode: unsupported (bits=%d M=%d K=%d N=%d group=%d)", a.bits, a.M, a.K, a.N, a.group_size);
    return -1;
  }
  DecSets sets = {};
  sets.nsets = 1;
  sets.tile_end[0] = a.N / 32;
  sets.N[0] = a.N;
  sets.packed[0] = (const uint4*)a.packed;
  sets.scales[0] = a.scales;
  sets.qzeros[0] = (const uint32_t*)a.qzeros;
  sets.bias[0] = a.bias;
  sets.out[0] = a.out;
  return launch_decode_sets(a, sets);
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
  DecSets sets = {};
  sets.nsets = 1;
  const int NT = a.N / 32;
  for (int i = 0; i < DEC_MAX_SETS; ++i) sets.tile_end[i] = NT;
  sets.N[0] = a.N;
  sets.packed[0] = (const uint4*)a.packed;
  sets.scales[0] = a.scales;
  sets.qzeros[0] = (const uint32_t*)a.qzeros;
  sets.out[0] = a.out;
  sets.moe = fused_act ? 3 : 2;
  sets.nexperts = E;
  sets.ids = ids;
  sets.wts = wts;
  moe_strides(sets, a.K, a.N, a.group_size);
  DecodeCfg c = {};
  c.ks = top_k;
  c.warps = DEC_MAX_WARPS;
  c.ngroups = 1;
  c.qpc = a.K / 128;  // a rank's k-range is its expert's whole K
  c.C = num_sms() / top_k;
  if (c.C > NT) c.C = NT;
  c.max_tiles = (NT + c.C - 1) / c.C;
  c.stl = 2;
  c.smem = decode_smem(1, c.warps, c.qpc, c.max_tiles, 4);
  if (c.smem > 200 * 1024) {
    c.stl = 1;
    c.smem = decode_smem(1, c.warps, c.qpc, c.max_tiles, 2);
  }
  if (c.smem > 200 * 1024) {
    set_error("b2q_moe_decode_down: K=%d does not fit shared memory", a.K);
    return -1;
  }
  MmArgs a0 = a;
  a0.perm = nullptr;
  a0.bias = nullptr;
  const bool asym = a.qzeros != nullptr, g64 = a.group_size == 64;
  const DecodeAR none = {};
#define B2Q_DEC_CASE(T)                                                            \
  (asym ? (g64 ? launch_decode_t<T, true, true, true>(a0, sets, c, none)           \
               : launch_decode_t<T, true, false, true>(a0, sets, c, none))         \
        : (g64 ? launch_decode_t<T, false, true, true>(a0, sets, c, none)          \
               : launch_decode_t<T, false, false, true>(a0, sets, c, none)))
  return a.dtype == 0 ? B2Q_DEC_CASE(__half) : B2Q_DEC_CASE(__nv_bfloat16);
#undef B2Q_DEC_CASE
}

}  // namespace b2q
