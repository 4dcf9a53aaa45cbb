/* b2q.h — C ABI of libb2q.so: the H100-native (sm_90a) GPTQ W4A16/W8A16 QuantLinear hot path.
 *
 * This is the boundary a host framework binds (ctypes / cffi / a torch.library shim); no torch or C++ types cross
 * it.  All pointers are DEVICE pointers unless noted, all calls are asynchronous on `stream` (a cudaStream_t passed
 * as void*), no call allocates, synchronises or throws; every call returns 0 on success or a non-zero code and
 * leaves a message for b2q_last_error().
 *
 * Reference interfaces replaced (paths relative to ModelCloud/GPTQModel):
 *   b2q_prepack  <- the post_init repack ops: gptq_marlin_repack (gptqmodel/nn_modules/qlinear/marlin.py:246-293,
 *                   gptqmodel_ext/marlin/gptq_marlin_repack.cu:254) and swordfish_prepack_B
 *                   (gptqmodel/nn_modules/qlinear/swordfish.py:221-297, gptqmodel/utils/swordfish.py:292-311)
 *   b2q_mm       <- the forward ops: torch.ops.gptqmodel_swordfish.swordfish_mm (gptqmodel_ext/swordfish/.../
 *                   swordfish_mm.cu:290-444), gptq_marlin_gemm (gptqmodel/utils/marlin.py:562-608), and the torch
 *                   oracle TorchLinear._forward_eager (gptqmodel/nn_modules/qlinear/torch.py:326-347)
 *   b2q_permute_cols <- Marlin's permute_cols_kernel (gptqmodel_ext/marlin/gptq_marlin.cu:86-164) / the
 *                   x[:, perm] gather in SwordfishLinear.forward (qlinear/swordfish.py:314-318)
 *
 * Checkpoint tensors consumed (gptqmodel/nn_modules/qlinear/__init__.py:827-865):
 *   qweight int32 [K*bits/32, N], qzeros int32 [G, N*bits/32] (v2 = true zero-point), scales [G, N],
 *   g_idx int32 [K].  The host derives perm = stable argsort(g_idx) for act-order layers and hands the forward entry points
 *   an int32 [2K] array: perm[0:K] that order (x'[k'] = x[perm[k']]), perm[K:2K] its INVERSE (the decode tiers read x
 *   coalesced and scatter through the inverse; ABI v3).  b2q_prepack and b2q_permute_cols read perm[0:K] only.
 */
#ifndef B2Q_H_
#define B2Q_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2Q_ABI_VERSION 3
#define B2Q_DTYPE_F16 0
#define B2Q_DTYPE_BF16 1

/* ABI version of the loaded library (B2Q_ABI_VERSION). */
int b2q_version(void);

/* Message of the last failing call on this thread ("" if none). Host pointer, valid until the next failure. */
const char* b2q_last_error(void);

/* Size in bytes of the prepacked weight buffer (== K*N*bits/8: the repack is a permutation). */
size_t b2q_packed_bytes(int K, int N, int bits);

/* Workspace b2q_mm / b2q_gemm need for M rows.  b2q_workspace_bytes is the tier-independent upper bound (M*K*2 for any
 * act-order layer, 0 otherwise); b2q_mm_workspace_bytes is exact for b2q_mm's own dispatch (0 when the decode / GEMV
 * tiers, which gather x[perm] while staging the activations, serve the call). */
size_t b2q_workspace_bytes(int M, int K, int N, int has_perm);
size_t b2q_mm_workspace_bytes(int M, int K, int N, int bits, int group_size, int has_perm);

/* Repack checkpoint-layout qweight into B2Q tiles.  perm (int32 [K], k' -> original row) may be NULL.
 * Requires K % 64 == 0, N % 32 == 0, bits in {4, 8}. */
int b2q_prepack(const int32_t* qweight, const int32_t* perm, void* packed, int K, int N, int bits, void* stream);

/* out[M, N] = x[M, K] @ dequant(W) (+ bias).  Dispatches on M inside the library so a CUDA graph sees the true M:
 *   M <= 8 (4-bit, group 64|128|K)  : decode tier (mma.sync, cluster split-K)           b2q_decode.cu
 *   M == 1 (8-bit)                  : CUDA-core GEMV                                     b2q_gemv.cu
 *   M <= 128 otherwise              : small-batch tier (swapped wgmma operands, cluster split-K)  b2q_midm.cu
 *   M  > 128                        : wgmma prefill tier                                         b2q_gemm.cu
 * The call runs on the device that owns `packed`, whatever the caller's current device is.
 *   x, scales, bias, out : fp16 (dtype 0) or bf16 (dtype 1), all the same type; x and out contiguous row-major
 *   qzeros               : NULL for symmetric layers (zero-point 2^(bits-1)), else int32 [G, N*bits/32]
 *   perm                 : NULL, or int32 [2K]: the act-order permutation used at prepack followed by its inverse
 *   group_size           : 32 | 64 | 128 | K (per-channel; the reference's -1)
 *   workspace            : >= b2q_workspace_bytes(M, K, N, perm != NULL) bytes, may be NULL when that is 0 */
int b2q_mm(const void* x, const void* packed, const void* scales, const int32_t* qzeros, const int32_t* perm,
           const void* bias, void* out, int M, int K, int N, int bits, int group_size, int dtype, void* workspace,
           size_t workspace_bytes, void* stream);

/* The tiers individually (tests, benchmarks, tuning); ks (split-K cluster size) / warps <= 0 = heuristic.
 *   b2q_decode : 4-bit, 1 <= M <= 8, K % 128 == 0, group_size 64|128|K: fragment-major weights -> mma.sync, per-group
 *                fix-up, cluster split-K reduced through distributed shared memory (the bs=1 decode path)
 *   b2q_gemv   : M == 1 (routes 4-bit to b2q_decode, 8-bit to the CUDA-core fma.rn.f32.f16 GEMV)
 *   b2q_gemm   : any M, the wgmma + TMA tensor-core tiers */
int b2q_decode(const void* x, const void* packed, const void* scales, const int32_t* qzeros, const int32_t* perm,
               const void* bias, void* out, int M, int K, int N, int bits, int group_size, int dtype, int ks,
               int warps, void* stream);
int b2q_gemv(const void* x, const void* packed, const void* scales, const int32_t* qzeros, const int32_t* perm,
             const void* bias, void* out, int K, int N, int bits, int group_size, int dtype, int ks, int warps,
             void* stream);
int b2q_gemm(const void* x, const void* packed, const void* scales, const int32_t* qzeros, const int32_t* perm,
             const void* bias, void* out, int M, int K, int N, int bits, int group_size, int dtype, void* workspace,
             size_t workspace_bytes, void* stream);

/* Sibling layers that consume the SAME activations (q/k/v, gate/up; module order in the reference:
 * gptqmodel/models/definitions/llama.py:17-27) in ONE decode launch: nsets <= 3 weight sets given as HOST arrays of
 * device pointers; all sets share M <= 8, K, bits = 4, group_size, dtype, symmetry (qzeros all NULL or all non-NULL) and
 * the act-order permutation `perm` (NULL, or int32 [2K], permutation + inverse — q/k/v and gate/up of a GPTQ checkpoint are quantised against the
 * same input Hessian and therefore carry the same g_idx).  out[i] is [M, N[i]].  Same arithmetic as nsets separate b2q_decode calls; results are bit-identical
 * whenever the fused launch cuts K like the single launches would (see b2q_debug_decode_plan), else they differ only
 * in the order the fp32 partial sums are added. */
int b2q_decode_multi(const void* x, int nsets, const void* const* packed, const void* const* scales,
                     const int32_t* const* qzeros, const int32_t* perm, const void* const* bias, void* const* out,
                     const int* N, int M, int K, int bits, int group_size, int dtype, void* stream);

/* The same for the prefill tier (bits = 4, M > 128): the 256-feature tile columns of all sets form one index space for the
 * persistent CTA pairs (q|k|v: 192 tiles instead of 128 + 32 + 32 at M = 2048), one launch instead of nsets, and act-order
 * siblings gather x[:, perm] ONCE into `workspace` (>= M*K*2 bytes when perm != NULL). */
int b2q_gemm_multi(const void* x, int nsets, const void* const* packed, const void* const* scales,
                   const int32_t* const* qzeros, const int32_t* perm, const void* const* bias, void* const* out,
                   const int* N, int M, int K, int bits, int group_size, int dtype, void* workspace,
                   size_t workspace_bytes, void* stream);

/* ---- Grouped MoE expert path (BASELINE configs[4]; the reference's unused analogue: swordfish_moe.cu:9-17,38-48) --------
 * y[t] = sum_j w[t, j] * W2_e( silu(W1_e x[t]) * W3_e x[t] ),  e = topk_ids[t, j], in FIVE launches without any host
 * synchronisation (CUDA-graph capturable).  Expert weights are the b2q_prepack'ed tensors of the per-expert QuantLinears
 * STACKED along a leading expert dimension (packed [E][K*N/2 bytes], scales [E][G][N], qzeros [E][G][N/8] or NULL when every
 * expert is symmetric); 4-bit, any supported group size, no act-order.  rows = T * top_k (token, j) pairs; pair p = t*top_k+j.
 *   b2q_moe_align   : topk_ids int32 [T, top_k] -> counts [E], offsets [E], sorted_pairs [rows] (stable by expert)
 *   b2q_moe_gather  : xs [rows, K]  <- x[sorted_pairs[i] / top_k]
 *   b2q_moe_gate_up : h [rows, N]   <- silu(xs W1_e) * (xs W3_e), both weight sets in one launch (rounded to the 16-bit
 *                     dtype at every module boundary of the reference's per-expert loop); `active` = experts expected to
 *                     receive rows (grid sizing only, e.g. min(E, rows))
 *   b2q_moe_down    : ypair [rows, N] fp32, row = PAIR index <- pair_weights[p] * T(h W2_e)   (K = intermediate size)
 *   b2q_moe_combine : y [T, N]      <- sum over the top_k slots of each token, one rounding */
int b2q_moe_align(const int32_t* topk_ids, int T, int top_k, int E, int32_t* counts, int32_t* offsets,
                  int32_t* sorted_pairs, void* stream);
int b2q_moe_gather(const void* x, const int32_t* sorted_pairs, void* xs, int rows, int top_k, int K, void* stream);
int b2q_moe_gate_up(const void* xs, const void* packed1, const void* scales1, const int32_t* qzeros1,
                    const void* packed3, const void* scales3, const int32_t* qzeros3, void* h, const int32_t* counts,
                    const int32_t* offsets, int E, int rows, int active, int K, int N, int bits, int group_size, int dtype,
                    void* stream);
int b2q_moe_down(const void* h, const void* packed2, const void* scales2, const int32_t* qzeros2, const int32_t* counts,
                 const int32_t* offsets, const int32_t* sorted_pairs, const float* pair_weights, float* ypair, int E,
                 int rows, int active, int K, int N, int bits, int group_size, int dtype, void* stream);
int b2q_moe_combine(const float* ypair, void* y, int T, int top_k, int N, int dtype, void* stream);

/* ---- MoE decode: ONE token through its top_k experts on the decode tier (same stacked expert tensors as above) -------------
 * The experts are read from topk_ids ON THE DEVICE (no host synchronisation, CUDA-graph capturable); three launches:
 *   b2q_moe_decode_gate_up : gu [2*top_k, N] <- rows 2j / 2j+1 = x W1_e / x W3_e for e = topk_ids[j]: the 2*top_k matrices are
 *                            sibling sets of one decode launch over the same activations x [1, K]      (1 <= top_k <= 8)
 *   b2q_moe_decode_act     : h [top_k, N]    <- T(T(silu(gu[2j])) * gu[2j+1])                      (module rounding points)
 *   b2q_moe_decode_down    : y [1, N]        <- sum_j topk_weights[j] * T(h[j] W2_e): a cluster of top_k CTAs per tile column,
 *                            rank j multiplies row j with ITS expert's w2 (K = intermediate size), the reduction through
 *                            distributed shared memory applies the routing weights; one rounding      (top_k in {2, 4, 8}).
 *                            fused_act = 1: `h` is the gu buffer itself and every rank computes its row of h while staging
 *                            the activations (same arithmetic as b2q_moe_decode_act) — two launches per block
 * 4-bit, K % 128 == 0, group_size 64 | 128 | K (the decode tier's envelope). */
int b2q_moe_decode_gate_up(const void* x, const void* packed1, const void* scales1, const int32_t* qzeros1,
                           const void* packed3, const void* scales3, const int32_t* qzeros3, const int32_t* topk_ids,
                           int top_k, int E, int K, int N, int bits, int group_size, int dtype, void* gu, void* stream);
int b2q_moe_decode_act(const void* gu, void* h, int top_k, int N, int dtype, void* stream);
int b2q_moe_decode_down(const void* h, const void* packed2, const void* scales2, const int32_t* qzeros2,
                        const int32_t* topk_ids, const float* topk_weights, int top_k, int E, int K, int N, int bits,
                        int group_size, int dtype, int fused_act, void* y, void* stream);

/* In-place all-reduce(sum) of a small 16-bit vector (n % 8 == 0, n <= max_elems) across `world` <= 8 GPUs of one
 * NVLink domain: the single collective of a row-parallel QuantLinear at decode time (the reference has
 * none).  peer_bufs is a HOST array of `world` device pointers to every rank's symmetric buffer (this rank's included),
 * each laid out as data[2][world][max_elems] (16-bit) followed at byte `flag_offset` by flags[2][world] (u32),
 * zero-initialised once; `seq` is a device u32[2] owned by this rank, zero-initialised once: {call counter, status}.  Every
 * rank must issue the same sequence of calls.  One CTA pushes, flags, waits and sums over peer memory; no NCCL.  The wait
 * for a peer's flag is bounded (2 s): a dead peer leaves status = 1 + its rank instead of hanging the GPU. */
int b2q_allreduce(void* inout, int n, int dtype, int rank, int world, const void* const* peer_bufs, size_t flag_offset,
                  int max_elems, void* seq, void* stream);

/* Row-parallel QuantLinear shard AND its all-reduce(sum) in ONE launch (decode tier: bits = 4, 1 <= M <= 8, no
 * act-order — the reference has no collective).  Every rank calls it with its K-shard (x [M, K/world],
 * weights of those rows) and the same M, N; the kernel pushes its fp32 partial sums into every rank's symmetric buffer
 * over NVLink peer memory, exchanges per-CTA flags, sums the `world` partials in rank order and stores
 * out[M, N] = round(sum_r x_r @ dequant(W_r) (+ bias)) on every rank.  Pass the bias on ONE rank only
 * (gptqmodel_b200.tp.shard_rows keeps it on rank 0).
 *   peer_bufs   : HOST array of `world` device pointers to every rank's symmetric buffer (this rank's included), laid
 *                 out as f32 data[2][world][max_elems], then at byte `flag_offset` (multiple of 16,
 *                 >= 2*world*max_elems*4) u32 flags of b2q_decode_allreduce_flag_bytes() bytes; zero-initialised once
 *   ctl         : this rank's device u32[4] {sequence, arrivals, status (1 + rank of a peer that timed out), -}, zeroed once
 * Every rank must issue the same sequence of calls with the same shapes.  CUDA-graph safe (nothing is reset).
 * EXPERIMENTAL: validated only by tools/tp_fused_smoke.py on several GPUs, not by the single-GPU suite. */
int b2q_decode_allreduce(const void* x, const void* packed, const void* scales, const int32_t* qzeros,
                         const void* bias, void* out, int M, int K, int N, int bits, int group_size, int dtype,
                         int rank, int world, const void* const* peer_bufs, size_t flag_offset, int max_elems,
                         void* ctl, void* stream);
size_t b2q_decode_allreduce_flag_bytes(void);

/* Debug / A-B tools: re-read the B2Q_* environment switches (they are read once when the library is loaded, never on the
 * call path). */
void b2q_debug_reload_env(void);

/* Debug: device buffer (>= 160*16 uint64) receiving %globaltimer phase stamps of the decode kernel; NULL = off. */
void b2q_debug_set_trace(void* device_buffer);

/* Debug / tests (host only, no GPU needed): the launch plan the decode tier would use for out[M, N] with N the total
 * width of the (fused sibling) weight sets.  version 1 = b2q_decode.cu, 2 = the experimental b2q_decode2.cu.
 * out8 = {CTA columns, split-K ranks (cluster size), warps per CTA, warps per tile group, k-quads (128 k) per CTA,
 * tiles (32 features) per group, ring stages, dynamic shared memory bytes}.  ks / warps <= 0 = heuristic. */
int b2q_debug_decode_plan(int version, int M, int K, int N, int ks, int warps, int* out8);

/* out[m, k'] = x[m, perm[k']] for 16-bit elements. */
int b2q_permute_cols(const void* x, const int32_t* perm, void* out, int M, int K, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2Q_H_ */
