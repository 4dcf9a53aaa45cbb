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
// Expert weights are the prepacked B2Q tensors of the per-expert QuantLinears, stacked (expert stride = one tensor), 4- or
// 8-bit.  Act-order experts were prepacked with their rows in group order, so each expert reads its activations in its
// own column order: moe_gather_perm_kernel replaces step 2 (xs[i, k'] = x[sorted_pairs[i] / k, P13_e[k']]) and, when w2
// has act-order, permutes h between steps 3 and 4 (h2[i, k'] = h[i, P2_e[k']]).
// Ahead of step 1, moe_route_kernel turns router logits [T, E] into the topk_ids / topk_weights those steps read (softmax
// top-k or DeepSeek-V3 grouped sigmoid; include/b2q.h states the arithmetic and the order of the slots).
#include "b2q_common.cuh"
#include "b2q_internal.h"

namespace b2q {

constexpr int MOE_MAX_EXPERTS = 256;
constexpr int ROUTE_WARPS = 4;  // tokens per CTA of moe_route_kernel

// router logits to fp32, exactly
__device__ __forceinline__ float route_f32(float v) { return v; }
__device__ __forceinline__ float route_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float route_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

// (v, i) ranks above (bv, bi): the larger value, ties to the lower index
__device__ __forceinline__ bool route_better(float v, int i, float bv, int bi) {
  return v > bv || (v == bv && i < bi);
}

// One round of a warp arg-max over N values per lane, entry (lane, j) standing for index lane + 32 j.  `ok` has bit j set
// where entry j may still be chosen.  Every lane returns the winner's index (INT_MAX if nothing was eligible) and value;
// the winning lane also gets its slot in `slot`.
template <int N>
__device__ __forceinline__ int route_argmax(const float (&v)[N], unsigned ok, int lane, float& best, int& slot) {
  float bv = -INFINITY;
  int bi = INT_MAX;
  slot = 0;
#pragma unroll
  for (int j = 0; j < N; ++j) {
    if (((ok >> j) & 1u) && route_better(v[j], lane + 32 * j, bv, bi)) {  // ascending j: ties keep the lower index
      bv = v[j];
      bi = lane + 32 * j;
      slot = j;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
    if (route_better(ov, oi, bv, bi)) {
      bv = ov;
      bi = oi;
    }
  }
  best = bv;
  return bi;
}

// One warp per token; lane l holds experts l, l + 32, ... (NPER = ceil(E / 32) of them) in registers.  Selection scores
// are the logits (softmax) or c = sigmoid(l) + bias (grouped sigmoid), NaN selected as -inf.  The grouped mode keeps the
// topk_group groups with the largest sum of their two largest c; experts of the other groups are never chosen.  The
// group scores need a group's experts side by side, so the warp stages c in its own 1 KB of shared memory (__syncwarp
// only).  k rounds of arg-max give the slots in descending score, ties to the lower index.
template <typename T, int NPER>
__global__ void __launch_bounds__(ROUTE_WARPS * 32)
    moe_route_kernel(const T* __restrict__ logits, const float* __restrict__ bias, int ntok, int E, int top_k,
                     int scoring, int n_group, int topk_group, int renormalize, float scale,
                     int32_t* __restrict__ topk_ids, float* __restrict__ topk_weights) {
  __shared__ float cs[ROUTE_WARPS][MOE_MAX_EXPERTS];
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int t = blockIdx.x * ROUTE_WARPS + warp;
  asm volatile("griddepcontrol.wait;" ::: "memory");  // the logits are the previous kernel's output
  if (t >= ntok) return;
  const T* row = logits + (size_t)t * E;
  float sel[NPER], wq[NPER];  // selection score; softmax: logit, sigmoid: s = sigmoid(l)
  unsigned ok = 0;
#pragma unroll
  for (int j = 0; j < NPER; ++j) {
    const int e = lane + 32 * j;
    sel[j] = -INFINITY;
    wq[j] = 0.f;
    if (e < E) {
      const float l = route_f32(row[e]);
      ok |= 1u << j;
      if (scoring == 0) {
        sel[j] = l;
      } else {
        const float s = 1.f / (1.f + expf(-l));
        wq[j] = s;
        sel[j] = s + bias[e];
      }
      if (sel[j] != sel[j]) sel[j] = -INFINITY;
    }
  }
  float mx = -INFINITY, denom = 1.f;
  if (scoring == 0) {  // softmax over all E logits: p_e = expf(l_e - max) / sum
#pragma unroll
    for (int j = 0; j < NPER; ++j) mx = fmaxf(mx, sel[j]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < NPER; ++j)
      if ((ok >> j) & 1u) sum += expf(sel[j] - mx);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    denom = sum;
  } else if (topk_group < n_group) {  // group-limited: keep topk_group groups (all kept: nothing to drop)
    float* c = cs[warp];
#pragma unroll
    for (int j = 0; j < NPER; ++j)
      if ((ok >> j) & 1u) c[lane + 32 * j] = sel[j];
    __syncwarp();
    const int gs = E / n_group;
    constexpr int GPER = MOE_MAX_EXPERTS / 2 / 32;  // n_group <= E / 2 <= 128 groups, lane l holds l, l + 32, ...
    float gsc[GPER];
    unsigned gok = 0;
#pragma unroll
    for (int j = 0; j < GPER; ++j) {
      const int g = lane + 32 * j;
      gsc[j] = -INFINITY;
      if (g < n_group) {
        float a = -INFINITY, b = -INFINITY;  // the two largest c of the group
        for (int i = g * gs; i < (g + 1) * gs; ++i) {
          const float v = c[i];
          if (v > a) {
            b = a;
            a = v;
          } else if (v > b) {
            b = v;
          }
        }
        gsc[j] = a + b;
        if (gsc[j] != gsc[j]) gsc[j] = -INFINITY;
        gok |= 1u << j;
      }
    }
    unsigned long long keep_lo = 0, keep_hi = 0;  // kept groups, bit g
    for (int r = 0; r < topk_group; ++r) {
      float bv;
      int slot;
      const int g = route_argmax<GPER>(gsc, gok, lane, bv, slot);
      if (lane == (g & 31)) gok &= ~(1u << slot);
      if (g < 64) keep_lo |= 1ull << g;
      else keep_hi |= 1ull << (g - 64);
    }
#pragma unroll
    for (int j = 0; j < NPER; ++j) {
      const int g = (lane + 32 * j) / gs;
      const bool kept = g < 64 ? (keep_lo >> g) & 1ull : (keep_hi >> (g - 64)) & 1ull;
      if (!kept) ok &= ~(1u << j);
    }
  }
  int my_id = 0;
  float my_w = 0.f, sel_sum = 0.f;
  for (int r = 0; r < top_k; ++r) {
    float bv;
    int slot;
    const int e = route_argmax<NPER>(sel, ok, lane, bv, slot);
    const int owner = e & 31;
    float w;
    if (scoring == 0) {
      w = expf(bv - mx) / denom;
    } else {
      float mine = 0.f;
#pragma unroll
      for (int j = 0; j < NPER; ++j)
        if (j == slot) mine = wq[j];
      w = __shfl_sync(0xffffffffu, mine, owner);
    }
    if (lane == owner) ok &= ~(1u << slot);
    sel_sum += w;  // slot order
    if (lane == r) {
      my_id = e;
      my_w = w;
    }
  }
  if (lane < top_k) {
    if (renormalize) my_w = scoring == 0 ? my_w / sel_sum : my_w / (sel_sum + 1e-20f);
    topk_ids[(size_t)t * top_k + lane] = my_id;
    topk_weights[(size_t)t * top_k + lane] = my_w * scale;
  }
}

template <typename T>
static int launch_moe_route_t(const void* logits, const float* bias, int T_, int E, int top_k, int scoring, int n_group,
                              int topk_group, int renormalize, float scale, int32_t* ids, float* wts,
                              cudaStream_t stream) {
  const dim3 grid((T_ + ROUTE_WARPS - 1) / ROUTE_WARPS, 1, 1), block(ROUTE_WARPS * 32, 1, 1);
  const T* x = (const T*)logits;
#define B2Q_ROUTE(NP)                                                                                                      \
  return launch_kernel(moe_route_kernel<T, NP>, grid, block, 0, stream, 0, true, x, bias, T_, E, top_k, scoring, n_group, \
                       topk_group, renormalize, scale, ids, wts)
  if (E <= 32) B2Q_ROUTE(1);
  if (E <= 64) B2Q_ROUTE(2);
  if (E <= 128) B2Q_ROUTE(4);
  B2Q_ROUTE(8);
#undef B2Q_ROUTE
}

int launch_moe_route(const void* logits, int dtype, const float* bias, int T, int E, int top_k, int scoring, int n_group,
                     int topk_group, int renormalize, float scale, int32_t* topk_ids, float* topk_weights,
                     cudaStream_t stream) {
  if (dtype == 0)
    return launch_moe_route_t<__half>(logits, bias, T, E, top_k, scoring, n_group, topk_group, renormalize, scale,
                                      topk_ids, topk_weights, stream);
  if (dtype == 1)
    return launch_moe_route_t<__nv_bfloat16>(logits, bias, T, E, top_k, scoring, n_group, topk_group, renormalize, scale,
                                             topk_ids, topk_weights, stream);
  return launch_moe_route_t<float>(logits, bias, T, E, top_k, scoring, n_group, topk_group, renormalize, scale, topk_ids,
                                   topk_weights, stream);
}

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

// act-order experts: one CTA per sorted row i, dst[i, k'] = src[r(i), perms[e(i) * K + k']] with r(i) = sorted_pairs[i] /
// top_k (or i when sorted_pairs is NULL) and e(i) the expert whose sorted rows hold i.  16-bit elements gathered from the
// source row (it stays in L1 / L2), stored as 16-byte vectors.
__global__ void __launch_bounds__(128)
    moe_gather_perm_kernel(const uint16_t* __restrict__ src, const int32_t* __restrict__ sorted_pairs,
                           const int32_t* __restrict__ perms, const int32_t* __restrict__ offsets, int E,
                           uint4* __restrict__ dst, int top_k, int K) {
  const int i = blockIdx.x;
  // upper bound of i over offsets, minus one: the last expert whose first row is <= i (an expert without rows has the
  // offset of the next one, so the search passes over it)
  int lo = 0, hi = E;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (offsets[mid] <= i) lo = mid + 1;
    else hi = mid;
  }
  const int e = lo > 0 ? lo - 1 : 0;
  const int r = sorted_pairs != nullptr ? sorted_pairs[i] / top_k : i;
  const uint16_t* s = src + (size_t)r * K;
  const int4* p = reinterpret_cast<const int4*>(perms + (size_t)e * K);
  uint4* d = dst + (size_t)i * (K / 8);
  for (int j = threadIdx.x; j < K / 8; j += blockDim.x) {
    const int4 a = p[2 * j], b = p[2 * j + 1];
    uint4 o;
    o.x = (uint32_t)__ldg(s + a.x) | ((uint32_t)__ldg(s + a.y) << 16);
    o.y = (uint32_t)__ldg(s + a.z) | ((uint32_t)__ldg(s + a.w) << 16);
    o.z = (uint32_t)__ldg(s + b.x) | ((uint32_t)__ldg(s + b.y) << 16);
    o.w = (uint32_t)__ldg(s + b.z) | ((uint32_t)__ldg(s + b.w) << 16);
    d[j] = o;
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
    moe_combine_kernel(const float* __restrict__ ypair, T* __restrict__ y, int ntokens, int top_k, int N) {
  using E = ET<T>;
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (n >= N) return;
  // tokens stride by gridDim.y (at most 65535): one pass for every T the grid covers, more for longer inputs
  for (int t = blockIdx.y; t < ntokens; t += gridDim.y) {
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

int launch_moe_gather_perm(const void* src, const int32_t* sorted_pairs, const int32_t* perms, const int32_t* offsets,
                           int E, void* dst, int rows, int top_k, int K, cudaStream_t stream) {
  if (E > MOE_MAX_EXPERTS) {
    set_error("b2q_moe_gather_perm: at most %d experts (got %d)", MOE_MAX_EXPERTS, E);
    return -1;
  }
  moe_gather_perm_kernel<<<rows, 128, 0, stream>>>((const uint16_t*)src, sorted_pairs, perms, offsets, E, (uint4*)dst,
                                                   top_k, K);
  return (int)cudaGetLastError();
}

int launch_moe_combine(const float* ypair, void* y, int T, int top_k, int N, int dtype, cudaStream_t stream) {
  dim3 grid((N / 4 + 255) / 256, T < 65535 ? T : 65535, 1);
  if (dtype == 0) moe_combine_kernel<__half><<<grid, 256, 0, stream>>>(ypair, (__half*)y, T, top_k, N);
  else moe_combine_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(ypair, (__nv_bfloat16*)y, T, top_k, N);
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
  const dim3 grid((N / 2 + 255) / 256, top_k, 1), block(256, 1, 1);
  if (dtype == 0)
    return launch_kernel(moe_decode_act_kernel<__half>, grid, block, 0, stream, 0, true, (const __half*)gu, (__half*)h,
                         top_k, N);
  return launch_kernel(moe_decode_act_kernel<__nv_bfloat16>, grid, block, 0, stream, 0, true, (const __nv_bfloat16*)gu,
                       (__nv_bfloat16*)h, top_k, N);
}

}  // namespace b2q
