// b2q_decode2.cu — second generation of the 4-bit decode tier (M <= 8).  The whole parity suite passes with it forced on
// (B2Q_DECODE_V2=1); it is selected per launch shape by launch_decode_sets
// (b2q_decode.cu): multi-tile launches run here, single-tile launches on decode_kernel.
//
// Same data path as b2q_decode.cu (fragment-major T4 tiles -> per-warp cp.async.bulk ring -> mma.sync on raw
// bias+q operands -> per-group fp32 fix-up, cluster split-K through distributed shared memory); what changes is
// everything AROUND the main loop:
//  * no per-tile epilogue: a warp parks its partial sums of a finished tile in its own slice of shared memory
//    (tokens < M only: 128 B per warp and tile at M = 1) and moves on; the CTA meets ONCE, after its last tile, and
//    reduces all tiles together.  v1 paid a CTA barrier + a 16-partial reduction (mostly latency) per tile,
//    3-7 times per launch;
//  * because nothing synchronises the warps between tiles any more, the warps of a CTA can form independent groups
//    of `gw` warps that walk different tiles (gw = 16, 8, 4 ...): the launch picks (split-K ranks, warps, gw)
//    minimising quads per warp, so small K-slices no longer leave warps idle.
// The activations are staged as in v1: with one warp group every warp stages and sums its OWN k-quads (the same quads in
// every tile), so no CTA barrier separates staging from the main loop; several groups read the same quads, so the CTA
// stages its k-range once; act-order layers gather through the inverse permutation.  B2Q_DECODE2_XTMA=1 (off by
// default) instead loads each token row with one cp.async.bulk and lets every warp sum its own quads.
// Arithmetic per output element is the same as v1 except for the summation order of the fp32 partials.
#include "b2q_common.cuh"
#include "b2q_decode.cuh"
#include "b2q_internal.h"

namespace b2q {

constexpr int DEC_AR_MAXCTA = 160;  // flag columns per source rank (>= CTAs of one launch: one per SM)
int launch_decode1_allreduce(const MmArgs& a, const DecSets& sets, const DecodeAR& ar);  // b2q_decode.cu

__device__ __forceinline__ void dec_st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t dec_ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Row-parallel QuantLinear + all-reduce in ONE kernel (ar.world > 1).  Every rank runs the same launch
// plan on its K-shard, so CTA c of every rank finishes the same output rows.  Instead of storing them, the CTA
//   1. pushes its fp32 partial sums into slot (seq & 1), row `rank`, of EVERY rank's symmetric buffer (P2P stores over
//      NVLink; 128 B per warp and row),
//   2. publishes seq + 1 in its flag column of every rank (st.release.sys after a system fence),
//   3. spins until the same column holds seq + 1 from every rank (ld.acquire.sys),
//   4. sums the `world` rows in rank order (same result on every rank), rounds once and stores the output.
// seq is a device counter advanced by the last CTA of the launch (CUDA-graph replay safe, nothing is ever reset);
// slots alternate with seq so a fast rank's next call never overwrites rows a slow rank is still summing.
// symmetric buffer: f32 data[2][world][max_elems] | (at flag_offset) u32 flags[world][DEC_AR_MAXCTA]
// dynamic smem: ring[nwarps][nst][2 KB] | sx[M][kspan] (T) | xsum[qpc * 2][8] f32 |
//               wpart[ngroups][max_tiles][M][gw][32] f32 | cpart[ngroups][max_tiles][M][32] f32 (split-K only) |
//               mbarriers[nwarps][DEC_STAGES] + 1 (activations) | 8 B pad | scale slots[nwarps][nst][SCB]
template <typename T, bool ASYM, bool G64, bool MOE>
__global__ void __launch_bounds__(DEC_MAX_WARPS * 32)
    decode2_kernel(const __grid_constant__ DecSets S, const int32_t* __restrict__ perm, const T* __restrict__ x, int M,
                   int K, int gsh, int qpc, int max_tiles, int gw, int stl, int xtma,
                   const __grid_constant__ DecodeAR ar) {
  using E = ET<T>;
  extern __shared__ __align__(128) uint8_t dsm2[];
  // MoE decode (DecSets::moe == 1): expert ids are data of an earlier kernel — wait before the first expert-dependent address
  if (MOE) asm volatile("griddepcontrol.wait;" ::: "memory");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int ngroups = nwarps / gw;               // independent warp groups; a group owns whole tiles
  const int grp = warp / gw, wg = warp - grp * gw;
  const int C = gridDim.x * ngroups;             // tile stride of a group
  const int tile0 = (int)blockIdx.x * ngroups + grp;
  const int TT = S.tile_end[S.nsets - 1];        // tiles of all sets
  const int ntiles = (tile0 < TT) ? (TT - tile0 + C - 1) / C : 0;
  const int nquads = K >> 7;
  const int q0 = blockIdx.y * qpc;
  const int q1 = min(q0 + qpc, nquads);
  const int kspan = qpc * 128;
  const int nst = 1 << stl;
  const uint32_t nrank = cluster_nctarank();
  uint8_t* ring = dsm2 + (size_t)warp * nst * DEC_QUAD_BYTES;
  T* sx = reinterpret_cast<T*>(dsm2 + (size_t)nwarps * nst * DEC_QUAD_BYTES);
  float* xsum = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(sx) + (size_t)M * kspan * sizeof(T));
  float* wpart = xsum + qpc * 2 * 8;
  const int rows = ngroups * max_tiles * M;      // (group, tile, token) rows of 32 features
  float* cpart = wpart + (size_t)rows * gw * 32;
  const uint32_t bars0 = smem_u32(cpart + (nrank > 1 ? (size_t)rows * 32 : 0));
  const uint32_t bars = bars0 + warp * DEC_STAGES * 8;
  const uint32_t xbar = bars0 + nwarps * DEC_STAGES * 8;
  constexpr int NG = G64 ? 2 : 1, SCB = dec_sc_bytes(ASYM, G64);
  const uint32_t sring_w = xbar + 16 + warp * nst * SCB;
  const bool PERM = perm != nullptr;
  const bool XTMA = (xtma & 1) != 0 && !PERM;  // bulk-copied activations (B2Q_DECODE2_XTMA=1)

  // ---- 1. the first ring stages of this warp requested before anything else -------------------------
  const int nq = (q0 + wg < q1) ? (q1 - q0 - wg + gw - 1) / gw : 0;  // quads per tile for this warp
  const int U = ntiles * nq;                                         // units (quads) of this warp
  // quantisation groups between consecutive quads of this warp, and the group of its first quad in every tile
  const int gstep = (2 * gw) >> gsh;
  const int g_first = (2 * (q0 + wg)) >> gsh;
  const uint4* iss_src = nullptr;
  const T* iss_sc = nullptr;          // scale row of the next quad to issue (features of its tile)
  const uint32_t* iss_zq = nullptr;   // qzeros row of the same
  int iss_N = 0;
  size_t iss_kbs = 0;
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
    if (warp == 0) mbar_init(xbar, 1);
    fence_mbar_init();
    if (U > 0) iss_begin_tile();
#pragma unroll
    for (int i = 0; i < DEC_STAGES; ++i)
      if (i < nst && iss_u < U) iss_one(smem_u32(ring) + i * DEC_QUAD_BYTES, sring_w + i * SCB, bars + 8 * i);
  }
  // every warp's mbarriers (and the activation barrier) are initialised before anybody polls them; this barrier sits
  // in the part of the kernel that overlaps the previous layer (PDL), so it is free
  __syncthreads();

  if (PERM) prefetch_inverse_perm(perm + K, K);
  // the block sums' padding columns (tokens >= M) are zeroed before the wait (LDG / act-order staging; the bulk-copy
  // variant writes every column itself)
  const bool OWN = !XTMA && !PERM && ngroups == 1;  // per-warp staging (stage_x_own_quads): no CTA barrier before the loop
  if (OWN) {
    zero_own_xsum_padding(xsum, M, nq, wg, gw);
  } else if (!XTMA) {
    for (int i = threadIdx.x; i < (q1 - q0) * 2 * 8; i += blockDim.x)
      if ((i & 7) >= M) xsum[i] = 0.f;
  }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");

  const uint32_t xf_a0 = smem_u32(sx) + (uint32_t)((g * kspan + t * 16 + wg * 128) * 2);
  const uint32_t xs_a0 = smem_u32(xsum) + (uint32_t)((2 * t + wg * 16) * 4);
  const uint32_t xf_qstep = (uint32_t)gw * 256u, xs_qstep = (uint32_t)gw * 64u;

  // ---- 2. activations --------------------------------------------------------------------------------
  if (XTMA) {
    // one bulk copy per token row; the sums over each 64-k block are made by the warp that consumes the block
    if (threadIdx.x == 0) {
      const uint32_t bytes = (uint32_t)(q1 - q0) * 256u;
      mbar_expect_tx(xbar, bytes * (uint32_t)M);
      for (int m = 0; m < M; ++m)
        bulk_load(smem_u32(sx) + (uint32_t)(m * kspan * 2), x + (size_t)m * K + (size_t)q0 * 128, bytes, xbar);
    }
    mbar_wait(xbar, 0);
    for (int qi = 0; qi < nq; ++qi) {
      const int ql = wg + qi * gw;  // quad inside this CTA's k-range
#pragma unroll
      for (int kbl = 0; kbl < 2; ++kbl) {
        float sm = 0.f;
        if (g < M) {
          const uint32_t a = xf_a0 + (uint32_t)qi * xf_qstep + kbl * 128;
          const uint4 x0 = lds128(a), x1 = lds128(a + 16);
          auto f2 = [](uint32_t u) {
            const T* h = reinterpret_cast<const T*>(&u);
            return E::to_f(h[0]) + E::to_f(h[1]);
          };
          sm = ((f2(x0.x) + f2(x0.y)) + (f2(x0.z) + f2(x0.w))) + ((f2(x1.x) + f2(x1.y)) + (f2(x1.z) + f2(x1.w)));
        }
        sm += __shfl_xor_sync(0xffffffffu, sm, 1);
        sm += __shfl_xor_sync(0xffffffffu, sm, 2);
        // token g (0 for the padding tokens >= M); groups > 0 would write the same values: group 0 writes, and the
        // CTA barrier below publishes them
        if (t == 0 && (ngroups == 1 || grp == 0)) xsum[(ql * 2 + kbl) * 8 + g] = sm;
      }
    }
    if (ngroups > 1) __syncthreads();
    else __syncwarp();
  } else if (OWN) {
    stage_x_own_quads<T>(x, sx, xsum, M, K, q0, nq, wg, gw, kspan);
  } else if (PERM) {
    stage_x_act_order<T>(x, perm + K, sx, xsum, M, K, q0 * 128, (q1 - q0) * 128, kspan);
    __syncthreads();
  } else {
    // several warp groups read the same quads: the CTA stages its k-range once
    const int n8 = (q1 - q0) * 16;  // uint4 (8 halves) per token row in this CTA's k-range
    const int tot = M * n8;
    const int totr = (tot + 31) & ~31;
    for (int i = threadIdx.x; i < totr; i += blockDim.x) {
      uint4 xv = make_uint4(0, 0, 0, 0);
      int m = 0, j = 0;
      if (i < tot) {
        m = (M == 1) ? 0 : i / n8;  // batch-1 decode: no integer division ahead of the load
        j = i - m * n8;
        const T* xr = x + (size_t)m * K;
        xv = reinterpret_cast<const uint4*>(xr + (size_t)q0 * 128)[j];
        reinterpret_cast<uint4*>(sx + (size_t)m * kspan)[j] = xv;
      }
      auto f2 = [](uint32_t u) {
        const T* h = reinterpret_cast<const T*>(&u);
        return E::to_f(h[0]) + E::to_f(h[1]);
      };
      float sm = (f2(xv.x) + f2(xv.y)) + (f2(xv.z) + f2(xv.w));
      sm += __shfl_xor_sync(0xffffffffu, sm, 1);
      sm += __shfl_xor_sync(0xffffffffu, sm, 2);
      sm += __shfl_xor_sync(0xffffffffu, sm, 4);
      if ((i & 7) == 0 && i < tot) xsum[(j >> 3) * 8 + m] = sm;
    }
    __syncthreads();
  }

  // ---- 3. main loop: the warp's quads of all its tiles, no CTA-level synchronisation ------------------
  constexpr float ZSYM = 8.f;
  const uint32_t ring_a = smem_u32(ring) + lane * 16;
  int u = 0;
  for (int ti = 0; ti < ntiles; ++ti) {
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
      float xs0 = 0.f, xs1 = 0.f;
#pragma unroll
      for (int kbl = 0; kbl < 2; ++kbl) {
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
          const int gi = G64 ? kbl : 0;
#pragma unroll
          for (int ftl = 0; ftl < 2; ++ftl) {
            const uint16_t slr = lds_u16(sc_a + gi * 64 + (ftl * 16 + g) * 2);
            const uint16_t shr = lds_u16(sc_a + gi * 64 + (ftl * 16 + g + 8) * 2);
            const float sl = E::to_f(*reinterpret_cast<const T*>(&slr));
            const float sh = E::to_f(*reinterpret_cast<const T*>(&shr));
            float zl = ZSYM, zh = ZSYM;
            if (ASYM) {
              zl = (float)((lds_u32(sc_a + NG * 64 + gi * 16 + ftl * 8) >> (4 * g)) & 15u);
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
      __syncwarp();
      if (lane == 0 && iss_u < U) iss_one(ring_a + st * DEC_QUAD_BYTES, sring_w + st * SCB, bars + 8 * st);
    }

    // park the warp's partial sums of this tile: wpart[(grp, ti, m)][wg][f], f rotated by 8 * (m / 2) so that the four
    // token pairs of a store instruction fall into different banks.
    // tot[ftl][c]: feature ftl*16 + g (+8 if c >= 2), token 2t + (c & 1)
    float* wp = wpart + ((size_t)(grp * max_tiles + ti) * M * gw + wg) * 32;
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int m = 2 * t + (b & 1);
        if (m < M) {
          const int f = a * 16 + g + ((b & 2) ? 8 : 0);
          wp[(size_t)m * gw * 32 + ((f + 8 * t) & 31)] = tot[a][b];
        }
      }
  }

  // ---- 4. ONE meeting per CTA: warps -> CTA for all tiles, then (split-K) CTA -> cluster -----------------
  __syncthreads();
  const bool AR = ar.world > 1;
  uint32_t seq = 0;
  if (AR) seq = *reinterpret_cast<const volatile uint32_t*>(ar.ctl);  // advanced by the previous launch's last CTA
  const size_t ar_slot = (size_t)(seq & 1u) * ar.world;
  struct RowRef {
    T* out;
    const T* bias;
    size_t idx;  // m * N + n
  };
  auto row_ref = [&](int row) {  // row = (group, tile, token); lane = feature inside the 32-feature tile
    const int m = row % M, r2 = row / M;
    const int ti = r2 % max_tiles, g2 = r2 / max_tiles;
    const TileRef<T> tr = resolve_tile<T, MOE>(S, (int)blockIdx.x * ngroups + g2 + ti * C);
    const int n = tr.nt * 32 + lane;
    RowRef r;
    r.out = tr.out;
    r.bias = tr.bias != nullptr ? tr.bias + n : nullptr;
    r.idx = (size_t)m * tr.N + n;
    return r;
  };
  bool pushed = false;  // this thread stored partial sums into peer memory
  auto emit = [&](int row, float v) {
    const RowRef r = row_ref(row);
    if (AR) {
      pushed = true;
      // the bias of a row-parallel layer lives on one rank only (tp.shard_rows): it joins that rank's partial sum
      if (r.bias != nullptr) v += E::to_f(*r.bias);
      const size_t o = (ar_slot + ar.rank) * (size_t)ar.max_elems + r.idx;
      for (int p = 0; p < ar.world; ++p) reinterpret_cast<float*>(ar.buf[p])[o] = v;
    } else {
      // reference order: round the matmul to the output dtype, then add bias (qlinear/torch.py:337-342)
      T o = E::from_f(v);
      if (r.bias != nullptr) o = E::from_f(E::to_f(o) + E::to_f(*r.bias));
      r.out[r.idx] = o;
    }
  };
  auto row_live = [&](int row) {
    const int r2 = row / M;
    const int ti = r2 % max_tiles, g2 = r2 / max_tiles;
    return (int)blockIdx.x * ngroups + g2 + ti * C < TT;
  };
  for (int row = warp; row < rows; row += nwarps) {
    if (!row_live(row)) continue;
    const int m = row % M;
    const float* src = wpart + (size_t)row * gw * 32 + ((lane + 8 * (m >> 1)) & 31);
    float v = 0.f;
    for (int w = 0; w < gw; ++w) v += src[w * 32];
    if (nrank > 1) cpart[row * 32 + lane] = v;
    else emit(row, v);
  }
  const int crank = nrank > 1 ? (int)cluster_ctarank() : 0;
  if (nrank > 1) {
    cluster_sync_all();  // every rank's cpart is complete (also a CTA barrier)
    for (int row = crank * nwarps + warp; row < rows; row += (int)nrank * nwarps) {
      if (!row_live(row)) continue;
      float v = 0.f;
      for (uint32_t r = 0; r < nrank; ++r) v += ld_dsmem_f32(smem_u32(&cpart[row * 32 + lane]), r);
      emit(row, v);
    }
    cluster_sync_all();  // keep every rank's smem alive until all peers have read it
  }
  if (AR) {
    // ---- 5. all-reduce across GPUs over peer memory (the rows this CTA emitted are the rows it sums) ----
    if (pushed) __threadfence_system();  // only the (few) warps that pushed rows pay the system-scope membar
    __syncthreads();
    const int cta = (int)(blockIdx.y * gridDim.x + blockIdx.x);
    if ((int)threadIdx.x < ar.world) {
      const int p = threadIdx.x;
      uint32_t* peer_flags = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(ar.buf[p]) + ar.flag_offset);
      dec_st_release_sys(peer_flags + ar.rank * DEC_AR_MAXCTA + cta, seq + 1u);
      const uint32_t* my_flags =
          reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(ar.buf[ar.rank]) + ar.flag_offset);
      if (!spin_until_geq_sys(my_flags + p * DEC_AR_MAXCTA + cta, seq + 1u)) ar.ctl[2] = 1u + (uint32_t)p;  // dead peer
    }
    __syncthreads();
    const float* mine = reinterpret_cast<const float*>(ar.buf[ar.rank]) + ar_slot * (size_t)ar.max_elems;
    for (int row = crank * nwarps + warp; row < rows; row += (int)nrank * nwarps) {
      if (!row_live(row)) continue;
      const RowRef r = row_ref(row);
      float v = 0.f;
      for (int p = 0; p < ar.world; ++p) v += __ldcg(mine + (size_t)p * ar.max_elems + r.idx);
      r.out[r.idx] = E::from_f(v);
    }
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned total = gridDim.x * gridDim.y;
      if (atomicAdd(ar.ctl + 1, 1u) == total - 1u) {  // every CTA has read seq: the last one advances it
        ar.ctl[1] = 0u;
        __threadfence();
        *reinterpret_cast<volatile uint32_t*>(ar.ctl) = seq + 1u;
      }
    }
  }
}

static size_t decode2_smem(const MmArgs& a, int warps, int gw, int qpc, int max_tiles, int ks, int nst) {
  const int M = a.M, scb = dec_sc_bytes(a.qzeros != nullptr, a.group_size == 64);
  const size_t rows = (size_t)(warps / gw) * max_tiles * M;
  return (size_t)warps * nst * DEC_QUAD_BYTES + (size_t)M * qpc * 128 * 2 + (size_t)qpc * 2 * 8 * 4 +
         rows * gw * 32 * 4 + (ks > 1 ? rows * 32 * 4 : 0) + (size_t)warps * DEC_STAGES * 8 + 8 + 16 +
         (size_t)warps * nst * scb;
}

// Pick (split-K ranks, warps per CTA, warps per group) minimising the critical path in quads per warp.
bool decode2_config(const MmArgs& a, int NT, DecodePlan& best) {
  const int quads = a.K / 128;
  const int SMS = num_sms();
  const int force_gw = env().decode2_gw;  // A/B switch (read once at load; b2q_debug_reload_env() re-reads it)
  double best_cost = 1e30;
  bool found = false;
  for (int ks = 1; ks <= 8; ks *= 2) {
    if (a.tune_ks > 0 && ks != a.tune_ks) continue;
    if (ks > quads) break;
    const int qpc = (quads + ks - 1) / ks;
    if ((ks - 1) * qpc >= quads) continue;  // the last rank would own no quads
    for (int warps = 8; warps <= DEC_MAX_WARPS; warps *= 2) {
      if (a.tune_warps > 0 && warps != a.tune_warps) continue;
      for (int gw = warps; gw >= 1; gw /= 2) {
        if (force_gw > 0 && gw != force_gw) continue;
        if (force_gw <= 0 && a.tune_warps > 0 && a.tune_ks > 0 && gw != warps) continue;  // pinned plan: one group
        const int ngroups = warps / gw;
        int C = SMS / ks;
        if (C * ngroups > NT) C = (NT + ngroups - 1) / ngroups;
        if (C < 1) C = 1;
        const int max_tiles = (NT + C * ngroups - 1) / (C * ngroups);  // per group
        DecodePlan p = {C, ks, warps, gw, qpc, max_tiles, 0, 0};
        if (!fit_ring(p, [&](int nst) { return decode2_smem(a, warps, gw, qpc, max_tiles, ks, nst); })) continue;
        const int qpw = (qpc + gw - 1) / gw;  // quads per warp per tile
        const double units = (double)max_tiles * qpw;
        // relative cost in units of one quad per warp at 16 warps / SM (heuristic weights); fewer warps hide less
        // latency; a tile switch costs a few dozen instructions; split-K adds a cluster barrier + DSMEM pass
        const double cost = units * (1.0 + (16 - warps) * 0.04) + 0.03 * max_tiles + (ks > 1 ? 0.5 : 0.0) +
                            0.02 * ngroups;
        if (cost < best_cost) {
          best_cost = cost;
          best = p;
          found = true;
        }
      }
    }
  }
  return found;
}

template <typename I>
static int launch_decode2_t(const MmArgs& a, const DecSets& sets, const DecodePlan& c, const DecodeAR& ar) {
  using T = typename I::T;
  auto kern = decode2_kernel<T, I::ASYM, I::G64, I::MOE>;
  static int smem_opted[32] = {};
  if (int e = ensure_dyn_smem(kern, (int)c.smem, smem_opted, "b2q_decode2")) return e;
  const int xtma = env().decode2_xtma ? 1 : 0;
  return launch_kernel(kern, dim3(c.C, c.ks, 1), dim3(c.warps * 32, 1, 1), c.smem, a.stream, c.ks, true, sets, a.perm,
                       (const T*)a.x, a.M, a.K, decode_gsh(a.group_size), c.qpc, c.max_tiles, c.gw, c.stl, xtma, ar);
}

int decode2_occupancy(const DecodePlan& c, int* blocks) {  // b2q_decode.cu: decode_occupancy
  return plan_occupancy(decode2_kernel<__half, false, false, false>, c, blocks);
}

// Returns -2 when no v2 configuration fits shared memory (the caller falls back to the v1 kernel).
static int launch_decode2_ar(const MmArgs& a, const DecSets& sets, const DecodeAR& ar) {
  DecodePlan c;
  if (!decode2_config(a, sets.tile_end[sets.nsets - 1], c)) return -2;
  if (ar.world > 1 && c.C * c.ks > DEC_AR_MAXCTA) return -2;
  if (!sets_aligned(sets, "b2q_decode2")) return -1;
  return dispatch_decode(a, sets, [&](auto inst) { return launch_decode2_t<decltype(inst)>(a, sets, c, ar); });
}

int launch_decode2_sets(const MmArgs& a, const DecSets& sets) {
  DecodeAR none = {};
  return launch_decode2_ar(a, sets, none);
}

size_t decode_allreduce_flag_bytes() { return (size_t)8 * DEC_AR_MAXCTA * sizeof(uint32_t); }

// Row-parallel QuantLinear shard + all-reduce(sum) across ranks in one launch (always the v2 kernel).
int launch_decode_allreduce(const MmArgs& a, const DecodeAR& ar) {
  const DecSets sets = layer_sets(a);
  // single-tile launches run faster on decode_kernel (b2q_decode.cu), which carries the same epilogue for that case
  if (env().decode_v2 != 1) {
    const int rc1 = launch_decode1_allreduce(a, sets, ar);
    if (rc1 != -2) return rc1;
  }
  const int rc = launch_decode2_ar(a, sets, ar);
  if (rc == -2) {
    set_error("b2q_decode_allreduce: no launch plan fits shared memory for M=%d K=%d N=%d", a.M, a.K, a.N);
    return -1;
  }
  return rc;
}

}  // namespace b2q
