// b2q_gemv.cu — 8-bit, batch-1 decode path: out[n] = sum_k x[k] * s[g(k), n] * (q[k, n] - z[g(k), n])  (+ bias).
//
// CUDA-core tier on the T8 layout (uint4 T8[K/32][N/32][2][32], natural byte order).  (The 4-bit decode path started
// as this kernel, is issue-bound and lives in b2q_decode.cu on mma.sync.)
//  * grid = (N/32 feature tiles) x (KS split-K CTAs); the KS CTAs of one feature tile form a thread-block cluster
//    and reduce their partial sums through distributed shared memory (no atomics, no workspace, deterministic);
//  * each lane owns ONE output feature; a warp reads 32 features x 16 k per coalesced 512-byte request, 8 requests in
//    flight per lane, issued BEFORE griddepcontrol.wait / the activation staging (weights do not depend on x);
//  * PRMT builds exact 1024+q half pairs; the multiply-accumulate is an fp32 FMA of the exactly widened halves:
//    exact fp16 x fp16 product, fp32 accumulate.  The zero-point and the 1024 bias
//    are removed once per group with pre-reduced activation sums: sum (q-z) x = sum (1024+q) x - (1024+z) sum x;
//  * act-order: rows sorted by group at prepack; the x[perm[k']] gather is fused into the smem staging.
// Replaces, for 8-bit M == 1, TorchLinear.forward (qlinear/torch.py:302-347) / Marlin's small-M path.
#include "b2q_common.cuh"
#include "b2q_internal.h"

namespace b2q {

constexpr int GEMV_MAX_WARPS = 8;
constexpr int GEMV_MAX_CPC = 128;  // chunks (of 32 k) per CTA  -> 8 KB of staged activations

template <typename T, int BITS, bool ASYM>
struct Quad {
  uint4 v[4 * (BITS / 4)];
  uint16_t s[4];   // raw scale of the group each chunk belongs to
  uint32_t zw[4];  // packed zero-point word (ASYM only)
};

// Issue every global load one quad (4 chunks = 128 k of one feature) needs: 4 (8) x LDG.128 of packed weights
// plus the per-group scale / zero words, so nothing on the critical path waits for a dependent load later.
template <typename T, int BITS, bool ASYM>
__device__ __forceinline__ void load_quad(Quad<T, BITS, ASYM>& q, const uint4* __restrict__ packed,
                                          const T* __restrict__ scales, const uint32_t* __restrict__ qzeros, int kc,
                                          int c1, int NT, int nt, int lane, int gchunks, int N) {
  constexpr int SUB = BITS / 4;
  constexpr int PF = 32 / BITS;
  const int n = nt * 32 + lane;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int h = 0; h < SUB; ++h) {
      if (kc + j < c1)
        q.v[j * SUB + h] = ldg_nc_v4(packed + (((size_t)(kc + j) * NT + nt) * SUB + h) * 32 + lane);
      else
        q.v[j * SUB + h] = make_uint4(0, 0, 0, 0);
    }
    if (kc + j < c1 && (j == 0 || (kc + j) % gchunks == 0)) {
      const int g = (kc + j) / gchunks;
      q.s[j] = *reinterpret_cast<const uint16_t*>(scales + (size_t)g * N + n);
      if (ASYM) q.zw[j] = qzeros[(size_t)g * (N / PF) + n / PF];
    } else if (j > 0) {
      q.s[j] = q.s[j - 1];
      if (ASYM) q.zw[j] = q.zw[j - 1];
    } else {
      q.s[j] = 0;
      if (ASYM) q.zw[j] = 0;
    }
  }
}

// dot of one 32-k chunk of one feature with the staged activations; returns sum (BASE+q)*x split in the two
// magic-number classes (lo: BASE = LO_BASE, hi: BASE = HI_BASE after HI_SCALE).
template <typename T, int BITS>
__device__ __forceinline__ void chunk_dot(const uint4* v, const uint4* __restrict__ xs, float& lo, float& hi) {
  using E = ET<T>;
  float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
  static_assert(BITS == 8, "this tier handles the 8-bit T8 layout only");
  {
    // 8-bit: natural byte order, 4 k per word; pair (k0,k1) = prmt(w, MAGIC8, 0x7150), (k2,k3) = 0x7352
    // fp16 only here (1024 + q, q < 256 fits the 10-bit mantissa); bf16 converts through fp32 instead.
#pragma unroll
    for (int hsub = 0; hsub < 2; ++hsub) {
      const uint32_t w[4] = {v[hsub].x, v[hsub].y, v[hsub].z, v[hsub].w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const uint2 xv = reinterpret_cast<const uint2*>(xs)[hsub * 4 + t];  // x[16h+4t .. +3]
        if (E::FMT == 0) {
          const uint32_t p0 = __byte_perm(w[t], 0x64006400u, 0x7150);
          const uint32_t p1 = __byte_perm(w[t], 0x64006400u, 0x7352);
          a0 = E::fma_lo(p0, xv.x, a0);
          a1 = E::fma_hi(p0, xv.x, a1);
          b0 = E::fma_lo(p1, xv.y, b0);
          b1 = E::fma_hi(p1, xv.y, b1);
        } else {
          // bf16 activations: q as fp32 integers (exact), x widened by a 16-bit shift
          const float q0 = (float)(w[t] & 0xFFu), q1 = (float)((w[t] >> 8) & 0xFFu);
          const float q2 = (float)((w[t] >> 16) & 0xFFu), q3 = (float)(w[t] >> 24);
          a0 = fmaf(q0, __uint_as_float(xv.x << 16), a0);
          a1 = fmaf(q1, __uint_as_float(xv.x & 0xFFFF0000u), a1);
          b0 = fmaf(q2, __uint_as_float(xv.y << 16), b0);
          b1 = fmaf(q3, __uint_as_float(xv.y & 0xFFFF0000u), b1);
        }
      }
    }
    lo += (a0 + a1) + (b0 + b1);
  }
}

template <typename T, int BITS, bool ASYM, bool PERM>
__global__ void __launch_bounds__(GEMV_MAX_WARPS * 32)
    gemv_kernel(const uint4* __restrict__ packed, const T* __restrict__ scales, const uint32_t* __restrict__ qzeros,
                const int32_t* __restrict__ perm, const T* __restrict__ x, const T* __restrict__ bias,
                T* __restrict__ out, int K, int N, int group_size, int cpc) {
  using E = ET<T>;
  __shared__ __align__(16) T sx[GEMV_MAX_CPC * 32];
  __shared__ float2 csum[GEMV_MAX_CPC];
  __shared__ float red[GEMV_MAX_WARPS][32];
  __shared__ float part[32];

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int NT = N >> 5, nt = blockIdx.x, n = nt * 32 + lane;
  const int nchunks = K >> 5;
  const int c0 = blockIdx.y * cpc;
  const int c1 = min(c0 + cpc, nchunks);
  constexpr float ZSYM = (float)(1 << (BITS - 1));
  // 8-bit codes carry no magic bias on the bf16 path (converted to fp32 directly)
  constexpr float LO_BASE = (BITS == 8 && E::FMT == 1) ? 0.f : (BITS == 8 ? 1024.f : E::LO_BASE);
  constexpr float HI_BASE = E::HI_BASE;

  // ---- 1. first weight quad (+ its scales) in flight before anything else ----------------------
  const int gchunks = group_size >> 5;  // chunks per group (>= 1)
  int q = c0 + warp * 4;
  Quad<T, BITS, ASYM> cur;
  load_quad<T, BITS, ASYM>(cur, packed, scales, qzeros, q, c1, NT, nt, lane, gchunks, N);

  // Programmatic dependent launch: the weights above never depend on the previous kernel in the stream,
  // the activations do.  Let the NEXT kernel start prefetching its weights now, and wait for the PREVIOUS
  // kernel's output (our x) only here.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");

  // ---- 2. stage activations (act-order gather fused) and reduce the per-chunk sums in one pass --
  //   thread i owns 8 consecutive k (one uint4); 4 neighbouring lanes own one 32-k chunk.
  {
    const int n4 = (c1 - c0) * 4;                 // uint4 slots of valid activations
    const int n4r = (n4 + 31) & ~31;              // whole warps take part in the shuffles
    uint4* xsm = reinterpret_cast<uint4*>(sx);
    for (int i = threadIdx.x; i < n4r; i += blockDim.x) {
      uint4 xv = make_uint4(0, 0, 0, 0);
      if (i < n4) {
        if (PERM) {
          const int4* pp = reinterpret_cast<const int4*>(perm + (size_t)c0 * 32) + 2 * i;
          const int4 p0 = pp[0], p1 = pp[1];
          const uint16_t* xu = reinterpret_cast<const uint16_t*>(x);
          xv.x = (uint32_t)xu[p0.x] | ((uint32_t)xu[p0.y] << 16);
          xv.y = (uint32_t)xu[p0.z] | ((uint32_t)xu[p0.w] << 16);
          xv.z = (uint32_t)xu[p1.x] | ((uint32_t)xu[p1.y] << 16);
          xv.w = (uint32_t)xu[p1.z] | ((uint32_t)xu[p1.w] << 16);
        } else {
          xv = reinterpret_cast<const uint4*>(x + (size_t)c0 * 32)[i];
        }
        xsm[i] = xv;
      }
      // pairs .x/.z are the "lo" magic class (k%8 in {0,1,4,5}), .y/.w the "hi" class (4-bit only)
      auto f2 = [](uint32_t u) {
        const T* h = reinterpret_cast<const T*>(&u);
        return E::to_f(h[0]) + E::to_f(h[1]);
      };
      float lo, hi;
      if (BITS == 4) {
        lo = f2(xv.x) + f2(xv.z);
        hi = f2(xv.y) + f2(xv.w);
      } else {
        lo = (f2(xv.x) + f2(xv.z)) + (f2(xv.y) + f2(xv.w));
        hi = 0.f;
      }
      lo += __shfl_xor_sync(0xffffffffu, lo, 1);
      hi += __shfl_xor_sync(0xffffffffu, hi, 1);
      lo += __shfl_xor_sync(0xffffffffu, lo, 2);
      hi += __shfl_xor_sync(0xffffffffu, hi, 2);
      if ((i & 3) == 0 && i < n4) csum[i >> 2] = make_float2(lo, hi);
    }
  }
  __syncthreads();

  // ---- 3. main loop: one quad (4 chunks = 128 k) per iteration, next quad prefetched -----------
  float total = 0.f;
  while (q < c1) {
    const int qn = q + nwarps * 4;
    Quad<T, BITS, ASYM> nxt;
    if (qn < c1) load_quad<T, BITS, ASYM>(nxt, packed, scales, qzeros, qn, c1, NT, nt, lane, gchunks, N);
    float lo = 0.f, hi = 0.f, cl = 0.f, ch = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int kc = q + j;
      if (kc < c1) {
        chunk_dot<T, BITS>(&cur.v[j * (BITS / 4)], reinterpret_cast<const uint4*>(sx + (kc - c0) * 32), lo, hi);
        const float2 cs = csum[kc - c0];
        cl += cs.x;
        ch += cs.y;
        const bool group_end = ((kc + 1) % gchunks == 0) || (kc + 1 == c1) || (j == 3);
        if (group_end) {
          const uint16_t sraw = cur.s[j];
          const float s = E::to_f(*reinterpret_cast<const T*>(&sraw));
          float z = ZSYM;
          if (ASYM) {
            constexpr int PF = 32 / BITS;
            z = (float)((cur.zw[j] >> (BITS * (n % PF))) & ((1u << BITS) - 1));
          }
          const float dot = lo + hi * E::HI_SCALE - ((LO_BASE + z) * cl + (HI_BASE + z) * ch);
          total = fmaf(s, dot, total);
          lo = hi = cl = ch = 0.f;
        }
      }
    }
    if (qn < c1) cur = nxt;
    q = qn;
  }

  // ---- 4. reduce: warps -> CTA (smem) -> cluster (DSMEM) ---------------------------------------
  red[warp][lane] = total;
  __syncthreads();
  const uint32_t nrank = cluster_nctarank();
  if (warp == 0) {
    float v = 0.f;
    for (int w = 0; w < nwarps; ++w) v += red[w][lane];
    part[lane] = v;
  }
  if (nrank > 1) cluster_sync_all();
  if (cluster_ctarank() == 0 && warp == 0) {
    float v = part[lane];
    for (uint32_t r = 1; r < nrank; ++r) v += ld_dsmem_f32(smem_u32(&part[lane]), r);
    // reference order: round the matmul to the output dtype, then add bias (qlinear/torch.py:337-342)
    T o = E::from_f(v);
    if (bias != nullptr) o = E::from_f(E::to_f(o) + E::to_f(bias[n]));
    out[n] = o;
  }
  if (nrank > 1) cluster_sync_all();  // keep peers' smem alive until rank 0 has read it
}

template <typename T, int BITS, bool ASYM, bool PERM>
static int launch_gemv_t(const MmArgs& a, int ks, int warps, int cpc) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(a.N / 32, ks, 1);
  cfg.blockDim = dim3(warps * 32, 1, 1);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = a.stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = ks;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;  // PDL, see the kernel prologue
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = a.pdl ? 2 : 1;
  auto kern = gemv_kernel<T, BITS, ASYM, PERM>;
  if (ks > 8) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e != cudaSuccess) return (int)e;
  }
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, (const uint4*)a.packed, (const T*)a.scales,
                                     (const uint32_t*)a.qzeros, a.perm, (const T*)a.x, (const T*)a.bias, (T*)a.out,
                                     a.K, a.N, a.group_size, cpc);
  return (int)e;
}

// split-K / CTA-shape heuristic: aim for >= ~4 CTAs per SM in a single wave, whole quads per warp.
static void gemv_config(const MmArgs& a, int& ks, int& warps, int& cpc) {
  const int nchunks = a.K / 32;
  const int quads = (nchunks + 3) / 4;
  const int NT = a.N / 32;
  warps = a.tune_warps > 0 ? a.tune_warps : 4;
  if (a.tune_ks > 0) {
    ks = a.tune_ks;
  } else {
    ks = 1;
    while (ks < 8 && NT * ks < num_sms() * 6 && quads / (ks * 2) >= 1) ks *= 2;
  }
  while (4 * ((quads + ks - 1) / ks) > GEMV_MAX_CPC && ks < 16) ks *= 2;
  cpc = 4 * ((quads + ks - 1) / ks);
}

int launch_gemv(const MmArgs& a) {
  if (a.bits != 8) {
    set_error("b2q_gemv(FHFMA): only the 8-bit T8 layout is handled here; 4-bit uses the decode tier");
    return -1;
  }
  int ks, warps, cpc;
  gemv_config(a, ks, warps, cpc);
  if (cpc > GEMV_MAX_CPC) {
    set_error("b2q_gemv: K=%d too large for the split-K configuration (cpc=%d)", a.K, cpc);
    return -1;
  }
  const bool asym = a.qzeros != nullptr, perm = a.perm != nullptr;
#define B2Q_GEMV_CASE(T, BITS)                                                        \
  (asym ? (perm ? launch_gemv_t<T, BITS, true, true>(a, ks, warps, cpc)               \
                : launch_gemv_t<T, BITS, true, false>(a, ks, warps, cpc))             \
        : (perm ? launch_gemv_t<T, BITS, false, true>(a, ks, warps, cpc)              \
                : launch_gemv_t<T, BITS, false, false>(a, ks, warps, cpc)))
  if (a.dtype == 0) return B2Q_GEMV_CASE(__half, 8);
  return B2Q_GEMV_CASE(__nv_bfloat16, 8);
#undef B2Q_GEMV_CASE
}

}  // namespace b2q
