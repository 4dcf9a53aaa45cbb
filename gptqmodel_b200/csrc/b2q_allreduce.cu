// b2q_allreduce.cu — latency-optimised one-shot all-reduce(sum) of a small vector over NVLink peer memory, for the
// row-parallel QuantLinear output at decode time (8-16 KB per call, 2 calls per decoder layer).
//
// Every rank owns one SYMMETRIC buffer (same layout on all GPUs, peers mapped through torch's symmetric-memory
// rendezvous): data[2 slots][world][max_elems] (16-bit) followed by flags[2 slots][world] (u32).
//   1. push : my vector is written into slot (seq & 1), row `rank`, of EVERY peer's buffer with 16-byte P2P stores
//   2. flag : __threadfence_system(), then one st.release.sys per peer publishes seq+1 in that peer's flag row
//   3. wait : one thread per peer spins (ld.acquire.sys) until its flag reaches seq+1
//   4. sum  : the `world` rows are summed in rank order in fp32 (identical result on every rank) and rounded once
// seq lives in device memory and only grows, so nothing is ever reset: CUDA-graph replay safe.  Slots alternate with
// seq, so a fast rank's call n+1 never overwrites data a slow rank is still reading for call n.
// The flag wait is bounded (2 s of %globaltimer): a dead peer leaves 1 + its rank in seq[1] instead of hanging the GPU.
// One CTA, no NCCL; the reference has no collective at all.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "b2q_common.cuh"
#include "b2q_internal.h"

namespace b2q {

struct ARPeers {
  void* buf[8];
};

__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

template <typename T>
__global__ void __launch_bounds__(256) allreduce_kernel(ARPeers peers, T* inout, int n, int rank, int world,
                                                        int max_elems, size_t flag_offset, uint32_t* seq_ptr) {
  // programmatic dependent launch on both sides: the NEXT kernel of the stream (a decode launch) may start its weight
  // prefetch now, and this kernel was itself launched while the matmul that produces `inout` was still running — a plainly
  // launched all-reduce between two PDL kernels serialised the whole chain (a TP-2 decode step slower than one GPU)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const uint32_t seq = *seq_ptr;
  const uint32_t slot = seq & 1u;
  const int n8 = n >> 3;  // uint4 = 8 elements
  const size_t row = ((size_t)slot * world + rank) * (size_t)max_elems;
  // 1. push
  for (int i = threadIdx.x; i < n8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(inout)[i];
    for (int r = 0; r < world; ++r)
      reinterpret_cast<uint4*>(reinterpret_cast<T*>(peers.buf[r]) + row)[i] = v;
  }
  __threadfence_system();
  __syncthreads();
  // 2. flag  + 3. wait
  if ((int)threadIdx.x < world) {
    const int r = threadIdx.x;
    uint32_t* peer_flags = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(peers.buf[r]) + flag_offset);
    st_release_sys_u32(peer_flags + slot * world + rank, seq + 1u);
    const uint32_t* my_flags =
        reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(peers.buf[rank]) + flag_offset);
    if (!spin_until_geq_sys(my_flags + slot * world + r, seq + 1u)) seq_ptr[1] = 1u + (uint32_t)r;  // peer r is dead
  }
  __syncthreads();
  // 4. sum in rank order
  const T* mine = reinterpret_cast<const T*>(peers.buf[rank]) + (size_t)slot * world * max_elems;
  for (int i = threadIdx.x; i < n8; i += blockDim.x) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int r = 0; r < world; ++r) {
      const uint4 v = reinterpret_cast<const uint4*>(mine + (size_t)r * max_elems)[i];
      const T* h = reinterpret_cast<const T*>(&v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += static_cast<float>(h[j]);
    }
    uint4 o;
    T* oh = reinterpret_cast<T*>(&o);
#pragma unroll
    for (int j = 0; j < 8; ++j) oh[j] = static_cast<T>(acc[j]);
    reinterpret_cast<uint4*>(inout)[i] = o;
  }
  if (threadIdx.x == 0) *seq_ptr = seq + 1u;
}

int launch_allreduce(void* inout, int n, int dtype, int rank, int world, const void* const* peer_bufs,
                     size_t flag_offset, int max_elems, void* seq, cudaStream_t stream) {
  ARPeers p = {};
  for (int i = 0; i < world; ++i) p.buf[i] = const_cast<void*>(peer_bufs[i]);
  if (dtype == 0)
    return launch_kernel(allreduce_kernel<__half>, dim3(1, 1, 1), dim3(256, 1, 1), 0, stream, 0, true, p,
                         (__half*)inout, n, rank, world, max_elems, flag_offset, (uint32_t*)seq);
  return launch_kernel(allreduce_kernel<__nv_bfloat16>, dim3(1, 1, 1), dim3(256, 1, 1), 0, stream, 0, true, p,
                       (__nv_bfloat16*)inout, n, rank, world, max_elems, flag_offset, (uint32_t*)seq);
}

}  // namespace b2q
