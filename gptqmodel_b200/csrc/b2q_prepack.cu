// b2q_prepack.cu — one-time repack of the GPTQ checkpoint layout into B2Q tiles (see b2q_common.cuh).
//
// Source layout (reference: gptqmodel/nn_modules/qlinear/__init__.py:827-865, packer :1536-1539):
//   qweight int32 [K*bits/32, N] row-major; word [i, n] holds rows i*pf..i*pf+pf-1 of column n, row i*pf+j at
//   bits [bits*j, bits*(j+1)).
// The role of this kernel is the one gptq_marlin_repack / swordfish_prepack_B play in the reference's
// post_init (qlinear/marlin.py:246-293, qlinear/swordfish.py:221-297): load-time only, not on the hot path.
#include "b2q_common.cuh"
#include "b2q_internal.h"

namespace b2q {

// 4-bit: T4[K/64][N/16][32] fragment-major (see b2q_common.cuh)
__global__ void prepack4_kernel(const uint32_t* __restrict__ qweight, const int32_t* __restrict__ perm,
                                uint4* __restrict__ out, int K, int N) {
  const int FT = N / 16;
  const long long total = (long long)(K / 64) * FT * 32;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int lane = (int)(idx & 31);
  const long long rest = idx >> 5;
  const int ft = (int)(rest % FT);
  const int kb = (int)(rest / FT);
  const int g = lane >> 2, t = lane & 3;
  uint32_t w[4];
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    uint32_t word = 0;
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      const int koff = ((p & 2) ? 2 : 0) + (p >> 2);
      const int n = ft * 16 + g + ((p & 1) ? 8 : 0);
      const int kp = kb * 64 + t * 16 + s * 4 + koff;
      const int k = perm ? perm[kp] : kp;
      const uint32_t q = (qweight[(size_t)(k >> 3) * N + n] >> (4 * (k & 7))) & 0xFu;
      word |= q << (4 * p);
    }
    w[s] = word;
  }
  out[idx] = make_uint4(w[0], w[1], w[2], w[3]);
}

// 8-bit: T8[K/32][N/32][2][32], natural byte order
__global__ void prepack8_kernel(const uint32_t* __restrict__ qweight, const int32_t* __restrict__ perm,
                                uint4* __restrict__ out, int K, int N) {
  const int NT = N / 32;
  const long long total = (long long)(K / 32) * NT * 2 * 32;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int lane = (int)(idx & 31);
  long long rest = idx >> 5;
  const int h = (int)(rest % 2);
  rest /= 2;
  const int nt = (int)(rest % NT);
  const int kc = (int)(rest / NT);
  const int n = nt * 32 + lane;
  uint32_t w[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint32_t word = 0;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int kp = kc * 32 + h * 16 + j * 4 + b;
      const int k = perm ? perm[kp] : kp;
      const uint32_t q = (qweight[(size_t)(k >> 2) * N + n] >> (8 * (k & 3))) & 0xFFu;
      word |= q << (8 * b);
    }
    w[j] = word;
  }
  out[idx] = make_uint4(w[0], w[1], w[2], w[3]);
}

int launch_prepack(const void* qweight, const int32_t* perm, void* out, int K, int N, int bits,
                   cudaStream_t stream) {
  const int threads = 256;
  if (bits == 4) {
    const long long total = (long long)(K / 64) * (N / 16) * 32;
    prepack4_kernel<<<(unsigned)((total + threads - 1) / threads), threads, 0, stream>>>(
        (const uint32_t*)qweight, perm, (uint4*)out, K, N);
  } else {
    const long long total = (long long)(K / 32) * (N / 32) * 2 * 32;
    prepack8_kernel<<<(unsigned)((total + threads - 1) / threads), threads, 0, stream>>>(
        (const uint32_t*)qweight, perm, (uint4*)out, K, N);
  }
  return (int)cudaGetLastError();
}

// x'[m, k'] = x[m, perm[k']]  (act-order activation gather for the tensor-core tiers; the decode tiers fuse it).
// Same job as permute_cols_kernel in the reference's Marlin (gptq_marlin.cu:86-164).
// One 2-byte global load per element would be M x K uncoalesced requests.  Here a CTA stages one row of x in shared memory with coalesced 16-byte loads, gathers from shared memory
// and writes 16-byte rows; the thread's slice of `perm` is read once and reused for every row the CTA walks.
template <int UNITS>
__global__ void __launch_bounds__(256)
    permute_rows_kernel(const uint16_t* __restrict__ x, const int32_t* __restrict__ perm, uint16_t* __restrict__ out, int M,
                        int K) {
  extern __shared__ __align__(16) uint4 srow[];
  const int n8 = K >> 3;
  int4 p0[UNITS], p1[UNITS];
#pragma unroll
  for (int u = 0; u < UNITS; ++u) {
    const int j = threadIdx.x + u * 256;
    if (j < n8) {
      p0[u] = reinterpret_cast<const int4*>(perm)[2 * j];
      p1[u] = reinterpret_cast<const int4*>(perm)[2 * j + 1];
    }
  }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");  // x is the previous kernel's output; `out` may still be read by it
  const uint16_t* s = reinterpret_cast<const uint16_t*>(srow);
  for (int m = blockIdx.x; m < M; m += gridDim.x) {
    const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)m * K);
#pragma unroll
    for (int u = 0; u < UNITS; ++u) {
      const int j = threadIdx.x + u * 256;
      if (j < n8) srow[j] = xr[j];
    }
    __syncthreads();
    uint4* orow = reinterpret_cast<uint4*>(out + (size_t)m * K);
#pragma unroll
    for (int u = 0; u < UNITS; ++u) {
      const int j = threadIdx.x + u * 256;
      if (j < n8) {
        uint4 o;
        o.x = (uint32_t)s[p0[u].x] | ((uint32_t)s[p0[u].y] << 16);
        o.y = (uint32_t)s[p0[u].z] | ((uint32_t)s[p0[u].w] << 16);
        o.z = (uint32_t)s[p1[u].x] | ((uint32_t)s[p1[u].y] << 16);
        o.w = (uint32_t)s[p1[u].z] | ((uint32_t)s[p1[u].w] << 16);
        orow[j] = o;
      }
    }
    __syncthreads();
  }
}

// any K (no shared-memory row): the element-wise form
__global__ void permute_cols_kernel(const uint16_t* __restrict__ x, const int32_t* __restrict__ perm,
                                    uint16_t* __restrict__ out, int M, int K) {
  for (int m = blockIdx.y; m < M; m += gridDim.y)
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < K; k += gridDim.x * blockDim.x)
      out[(size_t)m * K + k] = x[(size_t)m * K + perm[k]];
}

template <int UNITS>
static int launch_permute_rows(const void* x, const int32_t* perm, void* out, int M, int K, cudaStream_t stream) {
  auto kern = permute_rows_kernel<UNITS>;
  const size_t smem = (size_t)K * 2;  // <= 32 KB: inside the default dynamic shared memory limit
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(M < num_sms() * 8 ? M : num_sms() * 8, 1, 1);
  cfg.blockDim = dim3(256, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = env().disable_pdl ? 0 : 1;
  return (int)cudaLaunchKernelEx(&cfg, kern, (const uint16_t*)x, perm, (uint16_t*)out, M, K);
}

int launch_permute_cols(const void* x, const int32_t* perm, void* out, int M, int K, cudaStream_t stream) {
  if (K % 8 == 0 && K <= 16384) {
    if (K <= 4096) return launch_permute_rows<2>(x, perm, out, M, K, stream);
    if (K <= 8192) return launch_permute_rows<4>(x, perm, out, M, K, stream);
    return launch_permute_rows<8>(x, perm, out, M, K, stream);
  }
  dim3 grid((K + 255) / 256 > 64 ? 64 : (K + 255) / 256, M > 32768 ? 32768 : M);
  permute_cols_kernel<<<grid, 256, 0, stream>>>((const uint16_t*)x, perm, (uint16_t*)out, M, K);
  return (int)cudaGetLastError();
}

}  // namespace b2q
