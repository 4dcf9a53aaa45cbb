// b2q_moe.cu — routing helpers of the grouped MoE expert path (BASELINE configs[4]: Mixtral-8x7B int4 g64 asym).
//
// The reference ships a fused MoE op it never calls (swordfish_moe.cu:9-17,38-48: moe_align_block_size(16) ->
// sorted_token_ids / expert_ids -> one grouped launch); its models run every expert's w1 / w3 / w2 QuantLinear from a Python
// loop.  Here the whole block is five launches with NO host synchronisation (CUDA-graph capturable):
//   1. moe_align_kernel   topk_ids [T, k] -> counts[E], offsets[E], sorted_pairs[T*k]   (stable sort of the (token, j)
//                         pairs by expert: rows of one expert are contiguous, in token order)
//   2. moe_gather_kernel  xs[i, :] = x[sorted_pairs[i] / k, :]
//   3. midm_kernel<MODE 1> (b2q_midm.cu) over (feature tile, split-K rank, expert x token block):
//                         h[i, :] = silu(xs[i] W1_e) * (xs[i] W3_e)      both weight sets in ONE launch, SiLU-mul epilogue
//   4. midm_kernel<MODE 2>: ypair[pair(i), :] = w[pair(i)] * (h[i] W2_e)  routing weight + scatter to the pair's slot
//   5. moe_combine_kernel y[t, :] = sum_j ypair[t*k + j, :]               fp32 sum, ONE rounding, deterministic
// Expert weights are the prepacked B2Q tensors of the per-expert QuantLinears, stacked (expert stride = one tensor).
#include "b2q_common.cuh"
#include "b2q_internal.h"

namespace b2q {

constexpr int MOE_MAX_EXPERTS = 256;

__global__ void __launch_bounds__(256)
    moe_align_kernel(const int32_t* __restrict__ topk_ids, int npairs, int E, int32_t* __restrict__ counts,
                     int32_t* __restrict__ offsets, int32_t* __restrict__ sorted_pairs) {
  __shared__ int cnt[MOE_MAX_EXPERTS];
  __shared__ int off[MOE_MAX_EXPERTS];
  asm volatile("griddepcontrol.wait;" ::: "memory");  // topk_ids may come from a PDL-launched producer
  for (int e = threadIdx.x; e < E; e += blockDim.x) cnt[e] = 0;
  __syncthreads();
  for (int p = threadIdx.x; p < npairs; p += blockDim.x) {
    const int e = topk_ids[p];
    if (e >= 0 && e < E) atomicAdd(&cnt[e], 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int e = 0; e < E; ++e) {
      off[e] = run;
      run += cnt[e];
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    counts[e] = cnt[e];
    offsets[e] = off[e];
  }
  // stable placement: warp w scans all pairs in order for each of its experts (ballot prefix), so the rows of an expert
  // keep token order and the result does not depend on thread scheduling
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int e = warp; e < E; e += nwarps) {
    if (cnt[e] == 0) continue;
    int run = off[e];
    for (int base = 0; base < npairs; base += 32) {
      const int p = base + lane;
      const bool mine = p < npairs && topk_ids[p] == e;
      const unsigned mask = __ballot_sync(0xffffffffu, mine);
      if (mine) sorted_pairs[run + __popc(mask & ((1u << lane) - 1u))] = p;
      run += __popc(mask);
    }
  }
}

// one CTA per sorted row: 16-byte copies of the token's activations
__global__ void __launch_bounds__(128)
    moe_gather_kernel(const uint4* __restrict__ x, const int32_t* __restrict__ sorted_pairs, uint4* __restrict__ xs,
                      int top_k, int k16) {
  const int i = blockIdx.x;
  const int tok = sorted_pairs[i] / top_k;
  const uint4* src = x + (size_t)tok * k16;
  uint4* dst = xs + (size_t)i * k16;
  for (int j = threadIdx.x; j < k16; j += blockDim.x) dst[j] = src[j];
}

template <typename T>
__global__ void __launch_bounds__(256)
    moe_combine_kernel(const float* __restrict__ ypair, T* __restrict__ y, int top_k, int N) {
  using E = ET<T>;
  const int t = blockIdx.y;
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (n >= N) return;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j = 0; j < top_k; ++j) {
    const float4 v = *reinterpret_cast<const float4*>(ypair + ((size_t)t * top_k + j) * N + n);
    acc.x += v.x;
    acc.y += v.y;
    acc.z += v.z;
    acc.w += v.w;
  }
  *reinterpret_cast<uint2*>(y + (size_t)t * N + n) = make_uint2(E::pack2(acc.x, acc.y), E::pack2(acc.z, acc.w));
}

int launch_moe_align(const int32_t* topk_ids, int T, int top_k, int E, int32_t* counts, int32_t* offsets,
                     int32_t* sorted_pairs, cudaStream_t stream) {
  if (E > MOE_MAX_EXPERTS) {
    set_error("b2q_moe_align: at most %d experts (got %d)", MOE_MAX_EXPERTS, E);
    return -1;
  }
  moe_align_kernel<<<1, 256, 0, stream>>>(topk_ids, T * top_k, E, counts, offsets, sorted_pairs);
  return (int)cudaGetLastError();
}

int launch_moe_gather(const void* x, const int32_t* sorted_pairs, void* xs, int rows, int top_k, int K,
                      cudaStream_t stream) {
  moe_gather_kernel<<<rows, 128, 0, stream>>>((const uint4*)x, sorted_pairs, (uint4*)xs, top_k, K / 8);
  return (int)cudaGetLastError();
}

int launch_moe_combine(const float* ypair, void* y, int T, int top_k, int N, int dtype, cudaStream_t stream) {
  dim3 grid((N / 4 + 255) / 256, T, 1);
  if (dtype == 0) moe_combine_kernel<__half><<<grid, 256, 0, stream>>>(ypair, (__half*)y, top_k, N);
  else moe_combine_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(ypair, (__nv_bfloat16*)y, top_k, N);
  return (int)cudaGetLastError();
}

// MoE decode (one token): h[j, n] = T(T(silu(g)) * u) with g = gu[2j, n], u = gu[2j + 1, n] — the rounding points of the
// reference's per-expert module loop (act_fn(w1(x)) * w3(x) on 16-bit tensors), as in midm_kernel<MODE 1>'s epilogue.
template <typename T>
__global__ void __launch_bounds__(256)
    moe_decode_act_kernel(const T* __restrict__ gu, T* __restrict__ h, int top_k, int N) {
  using E = ET<T>;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int j = blockIdx.y;
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (n >= N) return;
  const uint32_t gw = *reinterpret_cast<const uint32_t*>(gu + (size_t)(2 * j) * N + n);
  const uint32_t uw = *reinterpret_cast<const uint32_t*>(gu + (size_t)(2 * j + 1) * N + n);
  const T* gp = reinterpret_cast<const T*>(&gw);
  const T* up = reinterpret_cast<const T*>(&uw);
  float hv[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float gq = E::to_f(gp[i]), uq = E::to_f(up[i]);
    const float aq = E::to_f(E::from_f(gq / (1.f + __expf(-gq))));
    hv[i] = aq * uq;
  }
  *reinterpret_cast<uint32_t*>(h + (size_t)j * N + n) = E::pack2(hv[0], hv[1]);
}

int launch_moe_decode_act(const void* gu, void* h, int top_k, int N, int dtype, cudaStream_t stream) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((N / 2 + 255) / 256, top_k, 1);
  cfg.blockDim = dim3(256, 1, 1);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = env().disable_pdl ? 0 : 1;
  if (dtype == 0)
    return (int)cudaLaunchKernelEx(&cfg, moe_decode_act_kernel<__half>, (const __half*)gu, (__half*)h, top_k, N);
  return (int)cudaLaunchKernelEx(&cfg, moe_decode_act_kernel<__nv_bfloat16>, (const __nv_bfloat16*)gu, (__nv_bfloat16*)h,
                                 top_k, N);
}

}  // namespace b2q
