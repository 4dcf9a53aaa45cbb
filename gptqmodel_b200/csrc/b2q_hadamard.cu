// b2q_hadamard.cu — online Hadamard transform of a rotated (QuaRot / SpinQuant) layer's input, in front of b2q_mm.
//
// For one row v of length n = K*P (P a power of two), viewed as V [K, P] row-major:
//   T(v) = vec(had_K . V . H_P) / sqrt(n),   H_P[i, j] = (-1)^popcount(i & j) (Sylvester, natural order)
// which is what the reference's matmul_hadU computes (gptqmodel/quantization/rotation/hadamard_utils.py:72-94).
//
// With P = P1 * P2, H_P = H_P1 (x) H_P2, so V viewed as [K, P1, P2] is transformed along its three axes in turn.  Each
// row is given a thread-block cluster of C CTAs (C = 1 when the rows alone fill the GPU):
//   phase 1: CTA c loads the contiguous slice [c*n/C, (c+1)*n/C) of the row (K*P1/C whole segments of length P2) and
//            applies H_P2 to every segment in fp32 shared memory;
//   phase 2: CTA c owns the column stripe [c*W, (c+1)*W) of the P2 columns (W = P2 / C).  It gathers that stripe of all
//            K*P1 segments from the cluster's shared memory (DSMEM), applies H_P1 along p1 and had_K along k, and stores.
// Everything stays in fp32 until the single rounding to the activation dtype; the summation order is fixed, so the
// result is deterministic.
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cmath>

#include "b2q_internal.h"

namespace cg = cooperative_groups;

namespace b2q {

constexpr int HAD_THREADS = 256;

struct HadPlan {
  int C;       // CTAs per row (cluster size)
  int logP1;   // outer power-of-two factor, transformed in phase 2
  int logP2;   // inner factor (contiguous segments), transformed in phase 1
  int logW;    // column stripe width per CTA = P2 / C
  size_t smem; // bytes: had_K as int8 (16-byte padded) + two fp32 buffers of n / C
  int grid_x;  // clusters in the grid; each walks rows blockIdx.x, blockIdx.x + grid_x, ...
};

static inline int ilog2(int v) {
  int r = 0;
  while ((1 << (r + 1)) <= v) ++r;
  return r;
}

// One radix-2^R pass of the Walsh-Hadamard transform along the L axis of s viewed as [A][L][S] (L = 2^logL, S = 2^logS),
// covering bits [b, b + R) of the L index.  Consecutive threads take consecutive S (then low L) positions.
template <int R>
__device__ __forceinline__ void wht_pass(float* s, int total, int logL, int logS, int b) {
  const int groups = total >> R;
  const int hib = logL - b - R;
  for (int g = threadIdx.x; g < groups; g += HAD_THREADS) {
    int t = g;
    const int si = t & ((1 << logS) - 1);
    t >>= logS;
    const int lo = t & ((1 << b) - 1);
    t >>= b;
    const int hi = t & ((1 << hib) - 1);
    const int a = t >> hib;
    const int base = ((((a << logL) + (hi << (b + R)) + lo)) << logS) + si;
    const int step = 1 << (b + logS);
    float v[1 << R];
#pragma unroll
    for (int i = 0; i < (1 << R); ++i) v[i] = s[base + i * step];
#pragma unroll
    for (int h = 1; h < (1 << R); h <<= 1)
#pragma unroll
      for (int i = 0; i < (1 << R); ++i)
        if (!(i & h)) {
          const float x = v[i], y = v[i + h];
          v[i] = x + y;
          v[i + h] = x - y;
        }
#pragma unroll
    for (int i = 0; i < (1 << R); ++i) s[base + i * step] = v[i];
  }
}

// bits [b0, logL) of the L axis, three at a time; ends with the block synchronised
__device__ __forceinline__ void wht_axis(float* s, int total, int logL, int logS, int b0) {
  for (int b = b0; b < logL; b += 3) {
    const int r = logL - b < 3 ? logL - b : 3;
    if (r == 3) wht_pass<3>(s, total, logL, logS, b);
    else if (r == 2) wht_pass<2>(s, total, logL, logS, b);
    else wht_pass<1>(s, total, logL, logS, b);
    __syncthreads();
  }
}

template <typename T>
__device__ __forceinline__ float to_f(T v);
template <>
__device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T>
__device__ __forceinline__ T from_f(float v);
template <>
__device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename T>
__device__ __forceinline__ void store4(T* dst, float a, float b, float c, float d) {
  union {
    T h[4];
    uint2 u;
  } o;
  o.h[0] = from_f<T>(a);
  o.h[1] = from_f<T>(b);
  o.h[2] = from_f<T>(c);
  o.h[3] = from_f<T>(d);
  *reinterpret_cast<uint2*>(dst) = o.u;
}

// had_K along k for every (p1, 4-column group) of the stripe B [K][P1][W], KT outputs per thread, the K-term sums split
// over NA interleaved accumulators (a shorter fp32 rounding chain for the large orders); stores the result
template <typename T, int KT, int NA>
__device__ __forceinline__ void had_store(const float* B, const int8_t* hs, T* orow, int K, int logP1, int logW,
                                          int P, int col0, float scale) {
  const int W4 = 1 << (logW - 2);
  const int P1 = 1 << logP1;
  const int cols = P1 * W4;
  const int items = (K / KT) * cols;
  const int P2 = P >> logP1;
  for (int it = threadIdx.x; it < items; it += HAD_THREADS) {
    const int c = it % cols;
    const int k0 = (it / cols) * KT;
    const int w4 = c & (W4 - 1);
    const int p1 = c >> (logW - 2);
    const float4* src = reinterpret_cast<const float4*>(B) + ((size_t)p1 << (logW - 2)) + w4;
    const int jstride = P1 * W4;  // float4 stride between consecutive j (k rows of B)
    float acc[NA][KT][4];
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
      for (int t = 0; t < KT; ++t) acc[a][t][0] = acc[a][t][1] = acc[a][t][2] = acc[a][t][3] = 0.f;
    for (int j = 0; j < K; j += NA) {  // K % NA == 0
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        const float4 x = src[(j + a) * jstride];
#pragma unroll
        for (int t = 0; t < KT; ++t) {
          const float h = (float)hs[(k0 + t) * K + j + a];
          acc[a][t][0] = fmaf(h, x.x, acc[a][t][0]);
          acc[a][t][1] = fmaf(h, x.y, acc[a][t][1]);
          acc[a][t][2] = fmaf(h, x.z, acc[a][t][2]);
          acc[a][t][3] = fmaf(h, x.w, acc[a][t][3]);
        }
      }
    }
#pragma unroll
    for (int a = NA / 2; a >= 1; a /= 2)  // pairwise combination of the partial sums
#pragma unroll
      for (int b = 0; b < a; ++b)
#pragma unroll
        for (int t = 0; t < KT; ++t)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[b][t][e] += acc[b + a][t][e];
#pragma unroll
    for (int t = 0; t < KT; ++t)
      store4<T>(orow + (size_t)(k0 + t) * P + p1 * P2 + col0 + w4 * 4, acc[0][t][0] * scale, acc[0][t][1] * scale,
                acc[0][t][2] * scale, acc[0][t][3] * scale);
  }
}

template <typename T>
__global__ void __launch_bounds__(HAD_THREADS)
    hadamard_kernel(const T* __restrict__ x, const int8_t* __restrict__ had, T* __restrict__ out, int rows, int K,
                    int logP1, int logP2, int logW, float scale) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  cg::cluster_group cluster = cg::this_cluster();
  const int C = (int)cluster.num_blocks();
  const int rank = (int)cluster.block_rank();
  const int P = 1 << (logP1 + logP2);
  const int n = K * P;
  const int nc = n / C;  // elements per CTA in both phases
  const int hbytes = (K * K + 15) & ~15;
  int8_t* hs = reinterpret_cast<int8_t*>(smem_raw);
  float* A = reinterpret_cast<float*>(smem_raw + hbytes);  // phase 1: this CTA's segments [K*P1/C][P2]
  float* B = A + nc;                                       // phase 2: the column stripe [K][P1][W]

  // had_K is static data: stage it before waiting for the producer of x
  if (had != nullptr) {
    const int full = (K * K) >> 4;  // had is 16-byte aligned; a tail of K*K % 16 bytes is copied bytewise
    for (int i = threadIdx.x; i < full; i += HAD_THREADS)
      reinterpret_cast<int4*>(hs)[i] = reinterpret_cast<const int4*>(had)[i];
    for (int i = (full << 4) + threadIdx.x; i < K * K; i += HAD_THREADS) hs[i] = had[i];
  }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  __syncthreads();

  const int P2 = 1 << logP2;
  const int W = 1 << logW;
  const int segs = nc >> logP2;  // segments held by this CTA in phase 1
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    // ---- phase 1: load 8 contiguous elements per thread, first three butterfly stages in registers ----
    const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)row * n + (size_t)rank * nc);
    for (int i = threadIdx.x; i < (nc >> 3); i += HAD_THREADS) {
      union {
        uint4 u;
        T h[8];
      } in;
      in.u = xr[i];
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = to_f<T>(in.h[e]);
#pragma unroll
      for (int h = 1; h < 8; h <<= 1)
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (!(e & h)) {
            const float a = v[e], b = v[e + h];
            v[e] = a + b;
            v[e + h] = a - b;
          }
      float4* dst = reinterpret_cast<float4*>(A + i * 8);
      dst[0] = make_float4(v[0], v[1], v[2], v[3]);
      dst[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
    __syncthreads();
    wht_axis(A, nc, logP2, 0, 3);
    cluster.sync();  // every CTA's segments are transformed

    // ---- phase 2: gather this CTA's column stripe of all K*P1 segments ----
    const int W4 = W >> 2;
    const int total4 = (K << logP1) * W4;
    for (int i = threadIdx.x; i < total4; i += HAD_THREADS) {
      const int seg = i / W4;  // k * P1 + p1
      const int w4 = i - seg * W4;
      const int owner = seg / segs;
      const float4* src =
          reinterpret_cast<const float4*>(cluster.map_shared_rank(A, owner) + (size_t)(seg - owner * segs) * P2 + rank * W);
      reinterpret_cast<float4*>(B)[i] = src[w4];
    }
    cluster.sync();  // the remote reads are done: A may be overwritten (next row) and the CTAs may exit
    wht_axis(B, nc, logP1, logW, 0);

    T* orow = out + (size_t)row * n;
    if (had == nullptr) {  // K == 1: the stripe is the result
      for (int i = threadIdx.x; i < (nc >> 2); i += HAD_THREADS) {
        const float4 v = reinterpret_cast<const float4*>(B)[i];
        const int p1 = i / W4, w4 = i - p1 * W4;
        store4<T>(orow + p1 * P2 + rank * W + w4 * 4, v.x * scale, v.y * scale, v.z * scale, v.w * scale);
      }
    } else if (K % 4 == 0) {
      had_store<T, 4, 4>(B, hs, orow, K, logP1, logW, P, rank * W, scale);
    } else {
      had_store<T, 1, 1>(B, hs, orow, K, logP1, logW, P, rank * W, scale);
    }
    __syncthreads();  // B is rewritten by the next row's gather
  }
}

// C, the P = P1 * P2 split and the grid for `rows` rows of n = K * P.  False if no split satisfies the kernel's layout
// conditions (P2 >= 8 for the in-register first stages, stripes of >= 4 columns, K * P1 segments divisible by C).
static bool hadamard_plan(int rows, int n, int K, HadPlan* pl) {
  const int P = n / K;
  const int logP = ilog2(P);
  // two fp32 buffers of n / C per CTA: at most 2 x 32 KB, so that two or more CTAs share an SM at prefill sizes
  int cmin = 1;
  while (n / cmin > 8192 && cmin < 8) cmin *= 2;
  int C = cmin;
  while (C < 8 && (long long)rows * C < num_sms()) C *= 2;  // decode: spread a row over up to 8 SMs
  for (; C >= 1; C >>= 1) {
    int kpow = 0;  // power-of-two factor of K
    while (kpow < 3 && ((K >> kpow) & 1) == 0) ++kpow;
    const int logC = ilog2(C);
    const int logP1 = logC > kpow ? logC - kpow : 0;
    const int logP2 = logP - logP1;
    const int logW = logP2 - logC;
    if (logP1 > logP || logP2 < 3 || logW < 2) continue;
    const size_t hbytes = ((size_t)K * K + 15) & ~(size_t)15;
    const size_t smem = hbytes + 2 * sizeof(float) * (size_t)(n / C);
    if (smem > 200 * 1024) return false;
    pl->C = C;
    pl->logP1 = logP1;
    pl->logP2 = logP2;
    pl->logW = logW;
    pl->smem = smem;
    const int per_sm = (int)((228 * 1024) / (smem + 1024));
    const int ctas = num_sms() * (per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm));
    const int g = ctas / C;
    pl->grid_x = rows < g ? rows : (g < 1 ? 1 : g);
    return true;
  }
  return false;
}

template <typename T>
static int launch_hadamard_t(const void* x, const int8_t* had, int K, void* out, int rows, int n, const HadPlan& pl,
                             cudaStream_t stream) {
  static int opted[32] = {};
  int e = ensure_dyn_smem(hadamard_kernel<T>, (int)pl.smem, opted, "b2q_hadamard");
  if (e != 0) return e;
  const float scale = (float)(1.0 / std::sqrt((double)n));
  return launch_kernel(hadamard_kernel<T>, dim3(pl.grid_x, pl.C, 1), dim3(HAD_THREADS, 1, 1), pl.smem, stream, pl.C,
                       true, (const T*)x, had, (T*)out, rows, K, pl.logP1, pl.logP2, pl.logW, scale);
}

int launch_hadamard(const void* x, const int8_t* had, int K, void* out, int rows, int n, int dtype,
                    cudaStream_t stream) {
  HadPlan pl;
  if (!hadamard_plan(rows, n, K, &pl)) {
    set_error("b2q_hadamard: no launch plan for n=%d K=%d", n, K);
    return -2;
  }
  return dtype == 0 ? launch_hadamard_t<__half>(x, had, K, out, rows, n, pl, stream)
                    : launch_hadamard_t<__nv_bfloat16>(x, had, K, out, rows, n, pl, stream);
}

}  // namespace b2q
