// b2q_decode.cuh — definitions shared by the decode-tier kernels (b2q_decode.cu, b2q_decode2.cu): the per-warp
// cp.async.bulk ring geometry, the mma.sync wrapper, the per-unit scale / zero registers and the multi-set ("sibling"
// QuantLinears) tile index space.
#pragma once
#include "b2q_common.cuh"

namespace b2q {

constexpr int DEC_MAX_WARPS = 16;
constexpr int DEC_MAXM = 8;

template <typename T>
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <>
__device__ __forceinline__ void mma_16816<__half>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma_16816<__nv_bfloat16>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0,
                                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// One "quad" = 128 k x 32 features = two contiguous 1 KB pieces of T4 (k-blocks 2q and 2q+1, feature tiles 2nt and
// 2nt+1).  Each warp owns a private ring of DEC_STAGES quad buffers in shared memory, filled by cp.async.bulk
// (UBLKCP) and tracked by one mbarrier per stage: up to DEC_STAGES * 2 KB per warp are in flight with no register
// cost, which is what keeps > 100 KB per SM outstanding (a register-prefetch ring keeps only 2 KB per warp in flight,
// too little to cover HBM latency).
constexpr int DEC_STAGES = 4;  // maximum ring depth; the launch picks 4 or 2 stages (`stl` = log2) to fit shared memory
constexpr int DEC_QUAD_BYTES = 2048;

template <bool ASYM, bool G64>
struct DScale {
  uint16_t s[G64 ? 2 : 1][4];  // [group in quad][ftl * 2 + hi]
  uint32_t zw[(ASYM ? 1 : 0) * (G64 ? 2 : 1) + (ASYM ? 0 : 1)][4];
};

__device__ __forceinline__ uint4 lds128(uint32_t a) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a));
  return r;
}
__device__ __forceinline__ float2 lds_f2(uint32_t a) {
  float2 r;
  asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(r.x), "=f"(r.y) : "r"(a));
  return r;
}

__device__ __forceinline__ void issue_quad(uint32_t dst, uint32_t bar, const uint4* __restrict__ src,
                                           size_t kb_stride) {
  mbar_expect_tx(bar, DEC_QUAD_BYTES);
  bulk_load(dst, src, 1024, bar);                     // k-block 2q   : feature tiles 2nt, 2nt+1
  bulk_load(dst + 1024, src + kb_stride, 1024, bar);  // k-block 2q+1
}

// Persistent-style CTA: blockIdx.x strides over the 32-feature tiles (tile = blockIdx.x + i * gridDim.x), blockIdx.y is
// the split-K rank inside the cluster.  x is staged ONCE per CTA; the warps split the k-quads of every tile; each
// warp's bulk-copy ring runs ahead across tile boundaries.
// Up to DEC_MAX_SETS weight sets that consume the SAME activations (q/k/v, gate/up: "sibling" QuantLinears) are served
// by one launch: the 32-feature tiles of all sets form one index space (tile_end = running totals).
// ---- act-order activation staging -------------------------------------------------------------------------------------
// `perm` (ABI v3) is int32 [2K]: perm[0:K] the sorted-by-group order (x'[k'] = x[perm[k']]), perm[K:2K] its inverse.
// Gathering x[perm[k']] with one 2-byte global load per element costs 4096 .. 14336 uncoalesced requests per CTA and
// token.  Here every
// CTA reads x and the INVERSE permutation with coalesced 16-byte loads and scatters the halves into the shared staging
// buffer (sx[m][inv[k] - k0] = x[m][k] for the sorted positions this CTA owns): 8x fewer global requests, the scattered
// accesses hit shared memory banks instead.  The per-(64-k block, token) sums are taken from shared memory afterwards.
__device__ __forceinline__ void prefetch_inverse_perm(const int32_t* __restrict__ inv, int K) {
  // static data: requested into L2 BEFORE griddepcontrol.wait (a layer's 16 .. 56 KB are HBM-cold on every token)
  for (int i = threadIdx.x * 32; i < K; i += blockDim.x * 32)
    asm volatile("prefetch.global.L2 [%0];" ::"l"(inv + i));
}

template <typename T>
__device__ __forceinline__ void stage_x_act_order(const T* __restrict__ x, const int32_t* __restrict__ inv, T* sx,
                                                  float* xsum, int M, int K, int k0, int kvalid, int kspan) {
  using E = ET<T>;
  constexpr int U = 4;  // independent (x, inverse) loads in flight per thread
  const int n8 = K >> 3;
  const int tot = M * n8;
  for (int i0 = threadIdx.x; i0 < tot; i0 += blockDim.x * U) {
    uint4 xv[U];
    int4 p0[U], p1[U];
    int mm[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * blockDim.x;
      mm[u] = -1;
      if (i < tot) {
        const int m = i / n8, j = i - m * n8;
        mm[u] = m;
        xv[u] = reinterpret_cast<const uint4*>(x + (size_t)m * K)[j];
        p0[u] = reinterpret_cast<const int4*>(inv)[2 * j];
        p1[u] = reinterpret_cast<const int4*>(inv)[2 * j + 1];
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (mm[u] >= 0) {
        uint16_t* row = reinterpret_cast<uint16_t*>(sx + (size_t)mm[u] * kspan);
        auto put = [&](int idx, uint32_t h) {
          const unsigned d = (unsigned)(idx - k0);
          if (d < (unsigned)kvalid) row[d] = (uint16_t)h;
        };
        put(p0[u].x, xv[u].x & 0xffffu);
        put(p0[u].y, xv[u].x >> 16);
        put(p0[u].z, xv[u].y & 0xffffu);
        put(p0[u].w, xv[u].y >> 16);
        put(p1[u].x, xv[u].z & 0xffffu);
        put(p1[u].y, xv[u].z >> 16);
        put(p1[u].z, xv[u].w & 0xffffu);
        put(p1[u].w, xv[u].w >> 16);
      }
    }
  }
  __syncthreads();
  // xsum[(64-k block) * 8 + token] = sum of the block's 64 staged activations: 8 lanes x one 16-byte shared load each
  const int nblk = kvalid >> 6;
  const int units = M * nblk * 8;
  const int unitsr = (units + 31) & ~31;
  for (int i = threadIdx.x; i < unitsr; i += blockDim.x) {
    float sm = 0.f;
    int b = 0, m = 0;
    if (i < units) {
      const int l = i & 7, bm = i >> 3;
      m = bm / nblk;
      b = bm - m * nblk;
      const uint4 v = *reinterpret_cast<const uint4*>(sx + (size_t)m * kspan + b * 64 + l * 8);
      auto f2 = [](uint32_t w) {
        const T* h = reinterpret_cast<const T*>(&w);
        return E::to_f(h[0]) + E::to_f(h[1]);
      };
      sm = (f2(v.x) + f2(v.y)) + (f2(v.z) + f2(v.w));
    }
    sm += __shfl_xor_sync(0xffffffffu, sm, 1);
    sm += __shfl_xor_sync(0xffffffffu, sm, 2);
    sm += __shfl_xor_sync(0xffffffffu, sm, 4);
    if ((i & 7) == 0 && i < units) xsum[b * 8 + m] = sm;
  }
}

// ---- per-warp activation staging (no act-order, one warp group) ------------------------------------------------------------
// Warp `wg` of `gw` stages exactly the k-quads it reads in the main loop (quads wg, wg + gw, ... of the CTA's k-range: 16
// lanes x 16 bytes per quad and token) and their 64-k block sums, so only the WARP synchronises between the load of x and its
// first mma — the CTA-wide loop it replaces made every warp wait at a CTA barrier for the slowest L2 round trip of the CTA.
// Everything between griddepcontrol.wait and the first main-loop iteration is on the critical path of every launch
// (a few percent of the whole Llama-3-8B decode step).
__device__ __forceinline__ void zero_own_xsum_padding(float* xsum, int M, int nq, int wg, int gw) {
  // token columns >= M of this warp's block sums (read by the fix-up of lanes whose columns are padding); before the wait
  const int lane = threadIdx.x & 31;
  for (int idx = lane; idx < nq * 16; idx += 32) {
    const int qi = idx >> 4, b = (idx >> 3) & 1, m = idx & 7;
    if (m >= M) xsum[((wg + qi * gw) * 2 + b) * 8 + m] = 0.f;
  }
}

// SILU: the activations are h = T(T(silu(g)) * u) of two rows g = x, u = x + K computed while staging (MoE down launch with
// the SiLU-mul of the reference's module boundary folded in: midm_kernel<MODE 1>'s epilogue arithmetic); one token only.
template <typename T, bool SILU = false>
__device__ __forceinline__ void stage_x_own_quads(const T* __restrict__ x, T* sx, float* xsum, int M, int K, int q0, int nq,
                                                  int wg, int gw, int kspan) {
  using E = ET<T>;
  constexpr int U = 4;  // independent 16-byte loads in flight per lane
  const int lane = threadIdx.x & 31, half = lane >> 4, j = lane & 15;
  const int np = (nq + 1) >> 1;  // quad pairs: one warp-wide load covers two quads
  const int units = M * np;      // (token, quad pair)
  auto f2 = [](uint32_t w) {
    const T* h = reinterpret_cast<const T*>(&w);
    return E::to_f(h[0]) + E::to_f(h[1]);
  };
  for (int v0 = 0; v0 < units; v0 += U) {
    uint4 xv[U], uv[U];
    int mm[U], ql[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int v = v0 + u;
      xv[u] = make_uint4(0, 0, 0, 0);
      uv[u] = make_uint4(0, 0, 0, 0);
      mm[u] = 0;
      ql[u] = -1;
      if (v < units) {
        const int m = (M == 1) ? 0 : v / np;  // batch-1 decode: no integer division ahead of the load
        const int qi = 2 * (v - m * np) + half;
        if (qi < nq) {
          mm[u] = m;
          ql[u] = wg + qi * gw;
          xv[u] = reinterpret_cast<const uint4*>(x + (size_t)m * K + (size_t)q0 * 128)[ql[u] * 16 + j];
          if (SILU) uv[u] = reinterpret_cast<const uint4*>(x + (size_t)K + (size_t)q0 * 128)[ql[u] * 16 + j];
        }
      }
    }
    if (SILU) {
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (ql[u] >= 0) {
          uint32_t gw4[4] = {xv[u].x, xv[u].y, xv[u].z, xv[u].w};
          const uint32_t uw4[4] = {uv[u].x, uv[u].y, uv[u].z, uv[u].w};
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const T* gp = reinterpret_cast<const T*>(&gw4[c]);
            const T* up = reinterpret_cast<const T*>(&uw4[c]);
            float hv[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float gq = E::to_f(gp[i]), uq = E::to_f(up[i]);
              const float aq = E::to_f(E::from_f(gq / (1.f + __expf(-gq))));
              hv[i] = aq * uq;
            }
            gw4[c] = E::pack2(hv[0], hv[1]);
          }
          xv[u] = make_uint4(gw4[0], gw4[1], gw4[2], gw4[3]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (v0 + u < units) {  // warp-uniform
        if (ql[u] >= 0) reinterpret_cast<uint4*>(sx + (size_t)mm[u] * kspan)[ql[u] * 16 + j] = xv[u];
        float sm = (f2(xv[u].x) + f2(xv[u].y)) + (f2(xv[u].z) + f2(xv[u].w));
        sm += __shfl_xor_sync(0xffffffffu, sm, 1);
        sm += __shfl_xor_sync(0xffffffffu, sm, 2);
        sm += __shfl_xor_sync(0xffffffffu, sm, 4);
        if (ql[u] >= 0 && (j & 7) == 0) xsum[(ql[u] * 2 + (j >> 3)) * 8 + mm[u]] = sm;  // 8 lanes = one 64-k block
      }
    }
  }
  __syncwarp();
}

constexpr int DEC_MAX_SETS = 3;
struct DecSets {
  int nsets;
  int tile_end[DEC_MAX_SETS];
  int N[DEC_MAX_SETS];
  const uint4* packed[DEC_MAX_SETS];
  const void* scales[DEC_MAX_SETS];
  const uint32_t* qzeros[DEC_MAX_SETS];
  const void* bias[DEC_MAX_SETS];
  void* out[DEC_MAX_SETS];
  // MoE decode: ONE token, its top_k experts picked on the device (b2q_moe_decode_*; no host synchronisation).
  //   moe = 1 (gate | up)  tile gt -> virtual set s = gt / (N[0] / 32): expert ids[s >> 1], weights of stack packed[s & 1]
  //                        (0: w1, 1: w3), output row s of out[0] ([2 * top_k, N]); every set reads the same activations;
  //   moe = 2 (down)       cluster rank r = pair r of the token: expert ids[r], the rank's k-range is the expert's WHOLE K,
  //                        its activations are row r of x ([top_k, K]), and the DSMEM reduction sums wts[r] * T(rank r's
  //                        output) — y = sum_j w_j * w2_e(h_j) with the module's rounding, in one launch;
  //   moe = 3 (down + act) as 2, but x is the gate | up buffer [2 * top_k, K] of moe = 1 and rank r stages
  //                        h = T(T(silu(x[2r])) * x[2r + 1]) itself: the SiLU-mul launch disappears.
  // ids are data of an earlier kernel: a moe launch executes griddepcontrol.wait BEFORE its first expert-dependent address.
  int moe;
  int nexperts;
  const int32_t* ids;
  const float* wts;
  size_t estride_w, estride_s, estride_z;  // expert strides of the stacks in uint4 / elements / uint32
};

template <typename T>
struct TileRef {
  const uint4* w;
  const T* sc;
  const uint32_t* zq;
  const T* bias;
  T* out;
  int N, nt;
};

template <typename T, bool MOE = false>
__device__ __forceinline__ TileRef<T> resolve_tile(const DecSets& S, int gt) {
  TileRef<T> r;
  if (MOE) {
    int s = 0, nt = gt, slot;
    if (S.moe == 1) {
      const int nts = S.N[0] >> 5;
      s = gt / nts;
      nt = gt - s * nts;
      slot = s >> 1;
    } else {
      slot = (int)cluster_ctarank();
    }
    int e = S.ids[slot];
    e = e < 0 ? 0 : (e >= S.nexperts ? S.nexperts - 1 : e);  // a corrupt id must not become a wild pointer
    const int b = (S.moe == 1) ? (s & 1) : 0;
    r.w = S.packed[b] + (size_t)e * S.estride_w;
    r.sc = reinterpret_cast<const T*>(S.scales[b]) + (size_t)e * S.estride_s;
    r.zq = S.qzeros[b] != nullptr ? S.qzeros[b] + (size_t)e * S.estride_z : nullptr;
    r.bias = nullptr;
    r.out = reinterpret_cast<T*>(S.out[0]) + (S.moe == 1 ? (size_t)s * S.N[0] : 0);
    r.N = S.N[0];
    r.nt = nt;
    return r;
  }
  int s = 0, start = 0;
  if (S.nsets > 1 && gt >= S.tile_end[0]) {
    s = 1;
    start = S.tile_end[0];
    if (S.nsets > 2 && gt >= S.tile_end[1]) {
      s = 2;
      start = S.tile_end[1];
    }
  }
  r.w = S.packed[s];
  r.sc = reinterpret_cast<const T*>(S.scales[s]);
  r.zq = S.qzeros[s];
  r.bias = reinterpret_cast<const T*>(S.bias[s]);
  r.out = reinterpret_cast<T*>(S.out[s]);
  r.N = S.N[s];
  r.nt = gt - start;
  return r;
}

}  // namespace b2q
