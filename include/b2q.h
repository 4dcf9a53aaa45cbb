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

#define B2Q_ABI_VERSION 8
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
 *   group_size           : 32 | 64 | 128 | K (per-channel; the reference's -1); any other size returns -2, in every
 *                          entry point that takes a GPTQ group size
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

/* The same for the prefill tier (bits = 4, M > 128): the 128-feature tile columns of all sets form one grid (q|k|v of
 * Llama-3-8B: 48 tile columns instead of 32 + 8 + 8), one launch instead of nsets, and act-order
 * siblings gather x[:, perm] ONCE into `workspace` (>= M*K*2 bytes when perm != NULL). */
int b2q_gemm_multi(const void* x, int nsets, const void* const* packed, const void* const* scales,
                   const int32_t* const* qzeros, const int32_t* perm, const void* const* bias, void* const* out,
                   const int* N, int M, int K, int bits, int group_size, int dtype, void* workspace,
                   size_t workspace_bytes, void* stream);

/* ---- Grouped MoE expert path (BASELINE configs[4]; the reference's unused analogue: swordfish_moe.cu:9-17,38-48) --------
 * y[t] = sum_j w[t, j] * W2_e( silu(W1_e x[t]) * W3_e x[t] ),  e = topk_ids[t, j], in FIVE launches without any host
 * synchronisation (CUDA-graph capturable).  Expert weights are the b2q_prepack'ed tensors of the per-expert QuantLinears
 * STACKED along a leading expert dimension (packed [E][K*N*bits/8 bytes], scales [E][G][N], qzeros [E][G][N*bits/32] or NULL
 * when every expert is symmetric); bits 4 or 8 (one width per stack, gate_up and down may differ), any supported group
 * size.  rows = T * top_k (token, j) pairs; pair p = t*top_k+j.
 *   b2q_moe_align   : topk_ids int32 [T, top_k] -> counts [E], offsets [E], sorted_pairs [rows] (stable by expert)
 *   b2q_moe_gather  : xs [rows, K]  <- x[sorted_pairs[i] / top_k]
 *   b2q_moe_gather_perm : act-order experts (prepacked with their rows in group order) read their activations in their own
 *                     column order; this replaces b2q_moe_gather (perms = P13 [E, K], the order half of each expert's w1
 *                     permutation, w3 sharing it; the identity for an expert without act-order) and, when w2 has act-order,
 *                     permutes h before b2q_moe_down (sorted_pairs = NULL, perms = P2 [E, N of gate_up]):
 *                       dst[i, k'] = src[r(i), perms[e(i) * K + k']],  r(i) = sorted_pairs[i] / top_k (or i when
 *                       sorted_pairs == NULL),  e(i) = the last expert e with offsets[e] <= i (the expert whose sorted rows
 *                       hold i).  16-bit elements, E <= 256, K % 8 == 0; src, dst and perms 16-byte aligned, dst != src.
 *   b2q_moe_gate_up : h [rows, N]   <- silu(xs W1_e) * (xs W3_e), both weight sets in one launch (rounded to the 16-bit
 *                     dtype at every module boundary of the reference's per-expert loop); `active` = experts expected to
 *                     receive rows (grid sizing only, e.g. min(E, rows))
 *   b2q_moe_down    : ypair [rows, N] fp32, row = PAIR index <- pair_weights[p] * T(h W2_e)   (K = intermediate size)
 *   b2q_moe_combine : y [T, N]      <- sum over the top_k slots of each token, one rounding */
int b2q_moe_align(const int32_t* topk_ids, int T, int top_k, int E, int32_t* counts, int32_t* offsets,
                  int32_t* sorted_pairs, void* stream);
int b2q_moe_gather(const void* x, const int32_t* sorted_pairs, void* xs, int rows, int top_k, int K, void* stream);
int b2q_moe_gather_perm(const void* src, const int32_t* sorted_pairs, const int32_t* perms, const int32_t* offsets,
                        int E, void* dst, int rows, int top_k, int K, void* stream);
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

/* MoE routing (an addition to ABI v8): router logits [T, E] (contiguous; logits_dtype 0 fp16, 1 bf16, 2 fp32, converted to
 * fp32 exactly, all arithmetic in fp32) -> topk_ids int32 [T, top_k] and topk_weights fp32 [T, top_k], what b2q_moe_align,
 * b2q_moe_decode_* and the grouped expert launches read.  One launch (one warp per token, programmatic dependent launch:
 * it waits before the first logits load), no host synchronisation, CUDA-graph capturable.
 *   scoring 0, softmax (Mixtral, Qwen2/3-MoE, OLMoE, DBRX): experts are selected on the logits l (softmax is monotonic);
 *     p_e = expf(l_e - max l) / sum_e' expf(l_e' - max l);  w_j = p_j / sum_sel p  (renormalize) or p_j;  then w_j *= scale.
 *     n_group = topk_group = 1, bias = NULL.
 *   scoring 1, grouped sigmoid (DeepSeek-V3/R1: n_group 8, topk_group 4; GLM-4.5 / dots1: n_group 1):
 *     s_e = 1 / (1 + expf(-l_e)),  c_e = s_e + bias_e  (bias = e_score_correction_bias fp32 [E]);
 *     group score = the sum of the two largest c of the group's E / n_group consecutive experts; the topk_group best groups
 *     are kept and the top_k largest c are selected among their experts only: experts of the other groups count as -inf
 *     (vLLM's grouped_topk, DeepSeek's inference code).  transformers' DeepseekV3MoE fills them with 0.0 instead; the two
 *     agree unless a kept group holds an expert with c < 0.
 *     w_j = s_j / (sum_sel s + 1e-20) (renormalize) or s_j;  then w_j *= scale (routed_scaling_factor).
 * Order: ties break toward the lower index, for groups and experts alike; slot j holds the j-th selection, i.e. slots come
 * in descending selection score (l or c), ties by lower index.  NaN scores select as -inf.
 * Envelope (-2 otherwise): 1 <= E <= 256, 1 <= top_k <= min(E, 16); scoring 1: n_group divides E, E / n_group >= 2,
 * 1 <= topk_group <= n_group, top_k <= topk_group * E / n_group.  T = 0 is a no-op. */
int b2q_moe_route(const void* logits, int logits_dtype, const float* bias, int T, int E, int top_k, int scoring, int n_group,
                  int topk_group, int renormalize, float scale, int32_t* topk_ids, float* topk_weights, void* stream);

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

/* Debug / tests (host only, no GPU needed): the launch plan the decode tier would use for out[M, N] with N the total
 * width of the (fused sibling) weight sets.  version 1 = b2q_decode.cu, 2 = b2q_decode2.cu.
 * out8 = {CTA columns, split-K ranks (cluster size), warps per CTA, warps per tile group, k-quads (128 k) per CTA,
 * tiles (32 features) per group, ring stages, dynamic shared memory bytes}.  ks / warps <= 0 = heuristic. */
int b2q_debug_decode_plan(int version, int M, int K, int N, int ks, int warps, int* out8);

/* Debug / tests (host only, no GPU needed): the launch plan of a swapped-operand wgmma tier, computed by the code its
 * launcher runs.  tier 0 = the small-batch tier of b2q_mm / b2q_moe_gate_up / b2q_moe_down, 1 = QQQ (b2q_qqq_mm),
 * 2 = block-FP8 (b2q_fp8blk_mm / _forward / _moe_gate_up / _moe_down).  mode 0 = one layer of M tokens (tier 0: M <= 128);
 * 1 / 2 = grouped gate|up / down over M expert-sorted rows with `active` experts expected (tiers 0 and 2).  ks > 0: the
 * B2Q_MIDM_KS override (tier 0) or a pinned ks (tier 2); tier 1 takes none.  Shapes as the tier's entry points accept them.
 * out4 = {tokens per CTA, split-K ranks, k-blocks per rank, token blocks}.  Bad arguments return -2. */
int b2q_debug_wgmma_plan(int tier, int mode, int M, int K, int N, int active, int ks, int* out4);

/* Resident CTAs per SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor on the current device) of the fp16, symmetric,
 * group-128 instantiation of decode kernel `version`, at the block size and dynamic shared memory of the plan
 * b2q_debug_decode_plan returns for the same arguments. */
int b2q_debug_decode_occupancy(int version, int M, int K, int N, int ks, int warps, int* blocks);

/* out[m, k'] = x[m, perm[k']] for 16-bit elements. */
int b2q_permute_cols(const void* x, const int32_t* perm, void* out, int M, int K, void* stream);

/* Online Hadamard transform of a rotated (QuaRot / SpinQuant) layer's input (ABI v6): for each of `rows` rows v of
 * length n = K * P, P a power of two,
 *   out = vec(had . V . H_P) / sqrt(n),   V = v viewed as [K, P] row-major,  H_P[i, j] = (-1)^popcount(i & j)
 * the reference's matmul_hadU (gptqmodel/quantization/rotation/hadamard_utils.py), computed in fp32 and rounded once.
 *   had   : int8 +-1 [K, K] row-major, 16-byte aligned; NULL exactly when K == 1
 *   x, out: fp16 (dtype 0) or bf16 (dtype 1) [rows, n], 16-byte aligned, out must not overlap x
 * Requires 1 <= K <= 256, P >= 8, n <= 65536, rows >= 0 (0: no-op).  Deterministic.  Launched with programmatic dependent
 * launch, so a following b2q_mm / b2q_decode may start loading its weights while the transform runs. */
int b2q_hadamard(const void* x, const int8_t* had, int K, void* out, int rows, int n, int dtype, void* stream);

/* QQQ (W4A8) tier (ABI v7): 4-bit weights, per-token int8 activations, int8 tensor cores (b2q_qqq.cu).  The arithmetic
 * of the reference's QQQLinear.forward + qqq_gemm (gptqmodel/nn_modules/qlinear/qqq.py, gptqmodel_ext/qqq):
 *   A = fp16(x);  s_tok[m] = fp32(fp16(max_k |A[m,k]| / 127));  q[m,k] = clamp(rint(A[m,k] / s_tok[m]), -128, 127)
 *   (IEEE fp32 division; an all-zero row gets s_tok = 0 and codes 0);
 *   w[k,n] = signed code * 16 (group_size -1) or round_half_even((code - 8) * s_group[k/128, n]) (group_size 128);
 *   acc = sum_k q * w in int32 (exact);  y = fp16(fp32(acc) * s_channel[n] * s_tok[m]);  y = fp16(y + bias[n]);
 *   bf16 output (out_dtype 1) = bf16(y).
 * Shapes: K % 128 == 0 and N % 64 == 0, or K % 64 == 0 and N % 128 == 0; K <= 65536; group_size -1, or 128 dividing K.
 * Tensors: codes uint8 [K, N] (canonical 4-bit codes, one per byte), s_channel fp32 [N] (16-byte aligned),
 * s_group fp16 [K/128, N] (NULL exactly for group_size -1), bias fp16 [N] or NULL.  Deterministic for any launch split. */
size_t b2q_qqq_packed_bytes(int K, int N);
/* Workspace of b2q_qqq_forward: the token scales and int8 codes of M rows. */
size_t b2q_qqq_workspace_bytes(int M, int K);
/* One-time repack of canonical codes into the kernel's tile layout (zero-padded to 128 k and 128 features). */
int b2q_qqq_prepack(const uint8_t* codes, void* packed, int K, int N, int group_size, void* stream);
/* Activation quantiser: x fp16/bf16 [M, K] -> q int8 [M, K rounded up to 128] (padding codes 0), s_tok fp32 [M].
 * Launched with programmatic dependent launch, so a following b2q_qqq_mm starts streaming its weights meanwhile. */
int b2q_qqq_quantize(const void* x, int8_t* q, float* s_tok, int M, int K, int dtype, void* stream);
/* out[M, N] from codes and token scales (b2q_qqq_quantize's output). */
int b2q_qqq_mm(const int8_t* q, const float* s_tok, const void* packed, const float* s_channel, const void* s_group,
               const void* bias, void* out, int M, int K, int N, int group_size, int out_dtype, void* stream);
/* b2q_qqq_quantize + b2q_qqq_mm through a caller workspace of b2q_qqq_workspace_bytes(M, K) bytes (16-byte aligned);
 * dispatches on M inside the library, so a CUDA graph sees the true M. */
int b2q_qqq_forward(const void* x, const void* packed, const float* s_channel, const void* s_group, const void* bias,
                    void* out, int M, int K, int N, int group_size, int dtype, int out_dtype, void* workspace,
                    size_t workspace_bytes, void* stream);

/* QQQ MoE experts (an addition to ABI v8): each role's experts stacked back to back — packed [E, b2q_qqq_packed_bytes(K,
 * N)], s_channel fp32 [E, N], s_group fp16 [E, K/128, N] (NULL exactly for group_size -1) — and the routing tables of
 * b2q_moe_align.  One block is six launches with no host synchronisation: b2q_moe_align, b2q_qqq_moe_gather,
 * b2q_qqq_moe_gate_up, b2q_qqq_quantize of h, b2q_qqq_moe_down, b2q_moe_combine.  For every routed pair (token t, slot j,
 * expert e), with Q the quantiser and F the layer arithmetic of b2q_qqq_mm above (F rounds to fp16):
 *   (q, s)     = Q(x_t)                           (the codes b2q_qqq_quantize gives the token)
 *   g = T(F(q, s, W1_e)),  u = T(F(q, s, W3_e))   (for T = bf16: bf16 of the fp16 value, as QQQLinear returns it)
 *   h = T(T(silu(g)) * u)                         (silu(g) = g / (1 + __expf(-g)) in fp32)
 *   (q_h, s_h) = Q(h)                             (down_proj quantises its own input; bf16 h goes through fp16 first)
 *   yp_j = T(F(q_h, s_h, W2_e))
 *   y_t  = T(sum_j fp32(w_j * yp_j))              (fp32, slot order, one rounding: b2q_moe_combine)
 * These are the rounding points of the reference model's per-expert loop over QQQLinear modules.  The accumulation is
 * int32 and exact, so the gate / up values and the down output of each expert's rows equal b2q_qqq_mm on those rows for
 * any split.  Envelope: each matmul meets the shape envelope of b2q_qqq_mm, the intermediate size N of gate|up is a
 * multiple of 64, w1 and w3 share one group_size, E <= 256; the pointers as for b2q_qqq_mm. */
/* q int8 [T*top_k, Kp], s_tok fp32 [T*top_k]: sorted row i = Q(x[sorted_pairs[i] / top_k]) (Kp = K rounded up to 128). */
int b2q_qqq_moe_gather(const void* x, const int32_t* sorted_pairs, int8_t* q, float* s_tok, int T, int top_k, int K,
                       int dtype, void* stream);
/* h T [rows, N] (dtype = T of the block): w1 / w3 stacks of one group_size, N = the intermediate size; active = experts
 * expected to hold rows (grid sizing). */
int b2q_qqq_moe_gate_up(const int8_t* q, const float* s_tok, const void* packed1, const float* s_channel1,
                        const void* s_group1, const void* packed3, const float* s_channel3, const void* s_group3, void* h,
                        const int32_t* counts, const int32_t* offsets, int E, int rows, int active, int K, int N,
                        int group_size, int dtype, void* stream);
/* ypair fp32 [rows, N]: row pair = w[pair] * yp of sorted row i, pair = sorted_pairs[i]; K = the intermediate size. */
int b2q_qqq_moe_down(const int8_t* q_h, const float* s_h, const void* packed2, const float* s_channel2,
                     const void* s_group2, const int32_t* counts, const int32_t* offsets, const int32_t* sorted_pairs,
                     const float* pair_weights, float* ypair, int E, int rows, int active, int K, int N, int group_size,
                     int dtype, void* stream);

/* FP8 (e4m3fn, W8A16) layers on the 8-bit tiers (ABI v8).  The arithmetic of the reference's TorchFP8Linear
 * (gptqmodel/nn_modules/qlinear/fp8.py, its dequantise-then-matmul path), T = fp16 (dtype 0) or bf16 (dtype 1):
 *   W[k, n] = RN_T( float(T(w[n, k])) / float(scales[k / group_size, n]) )      (correctly rounded division)
 *   out     = T(x @ W) (fp32 accumulation), then T(out + bias)
 * The M > 1 tiers feed the tensor cores exactly that W; the M = 1 GEMV (K % 128 == 0) sums w * x of a group in fp32 and
 * divides the sum by the scale once.
 *   packed : b2q_prepack(bits = 8) of the codes packed like an 8-bit GPTQ qweight (int32 [K/4, N], code of row 4i+j in
 *            byte j of word [i, n]); the byte is the e4m3fn bit pattern
 *   scales : T [K / group_size, N], scale_inv rounded to T and expanded over the output rows of its block;
 *            group_size 64 | 128 (dividing K) or K (per-channel and per-tensor layers)
 *   x, out: T, [M, K] / [M, N] contiguous, 16-byte aligned; bias T [N] or NULL; workspace unused (may be NULL)
 * Dispatches on M inside the library, so a CUDA graph sees the true M.  K % 64 == 0, N % 32 == 0. */
int b2q_fp8_mm(const void* x, const void* packed, const void* scales, const void* bias, void* out, int M, int K, int N,
               int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream);
/* out[K, N] (T, row-major) = W of b2q_fp8_mm, exactly the operand the tensor-core tiers multiply. */
int b2q_fp8_dequant(const void* packed, const void* scales, void* out, int K, int N, int group_size, int dtype,
                    void* stream);
/* FP8 MoE experts (an addition to ABI v8): the grouped modes of b2q_moe_gate_up / b2q_moe_down with W = the operand of
 * b2q_fp8_dequant.  Stacks: packed [E, b2q_packed_bytes(K, N, 8)] and scales T [E, K / group_size, N], one group_size per
 * role.  One block is five launches with no host synchronisation: b2q_moe_align, b2q_moe_gather, b2q_fp8_moe_gate_up,
 * b2q_fp8_moe_down, b2q_moe_combine.  The arithmetic is that of the GPTQ grouped path: g = T(x W1_e), u = T(x W3_e),
 * h = T(T(silu(g)) * u), yp_j = T(h W2_e), y_t = T(sum_j fp32(w_j * yp_j)) (fp32 accumulation on the tensor cores).
 * An fp16 scale table that is not finite gives zero weights, as in b2q_fp8_mm; callers refuse fp16 input for it.
 * Envelope: that of b2q_fp8_mm, E <= 256, xs / h 16-byte aligned. */
int b2q_fp8_moe_gate_up(const void* xs, const void* packed1, const void* scales1, const void* packed3,
                        const void* scales3, void* h, const int32_t* counts, const int32_t* offsets, int E, int rows,
                        int active, int K, int N, int group_size, int dtype, void* stream);
int b2q_fp8_moe_down(const void* h, const void* packed2, const void* scales2, const int32_t* counts,
                     const int32_t* offsets, const int32_t* sorted_pairs, const float* pair_weights, float* ypair, int E,
                     int rows, int active, int K, int N, int group_size, int dtype, void* stream);

/* Block-FP8 (W8A8) layers of HF / DeepSeek-native checkpoints (an addition to ABI v8 that changes no earlier entry
 * point): `quant_method: fp8`, `fmt: e4m3`, `activation_scheme: dynamic`, `weight_block_size: [128, 128]` (transformers' FineGrainedFP8Config, DeepSeek-V3, the
 * Qwen3 *-FP8 releases).  Weights e4m3 w [N, K] (the checkpoint tensor, unchanged), s_w = weight_scale_inv fp32
 * [ceil(N/128), K/128], which MULTIPLIES the weights.  T = fp16 (dtype 0) or bf16 (dtype 1), KB = K / 128.  For every
 * token row m and k-block b:
 *   a[m,b]   = max_{k in b} |x[m,k]|                                (exact: x is T, widened to fp32)
 *   s_x[m,b] = fmaxf(a[m,b], 1e-10f) / 448.f                       (IEEE fp32 division)
 *   q[m,k]   = e4m3_rn_satfinite(float(x[m,k]) / s_x[m,b])           (IEEE fp32 division)
 *   P_b[m,n] = sum_{k in b} q[m,k] * w[n,k]                         (e4m3 wgmma, fp32 accumulation)
 *   acc[m,n] = fmaf(P_b[m,n], s_x[m,b] * s_w[n/128, b], acc[m,n])     for b in increasing order
 *   y        = T(acc);  y = T(y + bias[n])                          (bias optional, T [N])
 * The 1e-10 epsilon keeps an all-zero group finite (codes 0).  The fp8 tensor-core accumulator is not an exact fp32 sum,
 * so P_b is not exact in general; the scales are promoted once per 128-k block.  Split-K: each of the `ks` ranks of a
 * tile promotes its own contiguous run of k-blocks in order from acc = 0, and the ranks' fp32 partials are added in rank
 * order.  Results are deterministic for a launch plan; they may differ in the last bits between splits.
 * Envelope: K % 128 == 0, K <= 65536, N % 64 == 0; x, codes, s_x, weight, s_w, out and workspace 16-byte aligned.
 * Bad arguments return -2 before any CUDA work. */
/* Workspace of b2q_fp8blk_forward for M rows: the codes and token scales (0 for M <= 8, which quantise inside the GEMM). */
size_t b2q_fp8blk_workspace_bytes(int M, int K);
/* Activation quantiser: x T [M, K] -> codes e4m3 [M, K], s_x fp32 [K/128, Mp] (Mp = M rounded up to 4; s_x[b, m]).
 * Launched with programmatic dependent launch, so a following b2q_fp8blk_mm starts streaming its weights meanwhile. */
int b2q_fp8blk_quantize(const void* x, void* codes, float* s_x, int M, int K, int dtype, void* stream);
/* out T [M, N] from b2q_fp8blk_quantize's codes and scales; ks = split-K ranks (1..8), <= 0: the heuristic. */
int b2q_fp8blk_mm(const void* codes, const float* s_x, const void* weight, const float* s_w, const void* bias,
                  void* out, int M, int K, int N, int dtype, int ks, void* stream);
/* The layer: M <= 8 in ONE launch that quantises the activation blocks it consumes (the codes of b2q_fp8blk_quantize,
 * the plan of b2q_fp8blk_mm with ks <= 0, so the output is identical to theirs); M > 8 b2q_fp8blk_quantize +
 * b2q_fp8blk_mm through the workspace.  Dispatches on M inside the library, so a CUDA graph sees the true M. */
int b2q_fp8blk_forward(const void* x, const void* weight, const float* s_w, const void* bias, void* out, int M, int K,
                       int N, int dtype, void* workspace, size_t workspace_bytes, void* stream);

/* Per-channel FP8 (W8A8) layers (an addition to ABI v8 that changes no earlier entry point): compressed-tensors
 * `float-quantized` FP8_DYNAMIC (channel weights, dynamic per-token activations) and FP8 (tensor weights, a static
 * per-tensor input_scale), and transformers' fbgemm_fp8 (channel weights, per-token activations with amax bounded by
 * activation_scale_ub).  Weights e4m3 w [N, K] (the checkpoint tensor, unchanged), s_w fp32 [N], one scale per output
 * feature that MULTIPLIES the weights (a per-tensor scale is broadcast to [N] by the caller).  T = fp16 (dtype 0) or bf16
 * (dtype 1), KB = K / 128.  For every token row m:
 *   dynamic: s_x[m] = fmaxf(fminf(max_k |x[m,k]|, ub), 1e-10f) / 448.f     (ub = +inf: no bound; IEEE fp32 division)
 *   static:  s_x[m] = s_in                                                   (the layer's input_scale)
 *   q[m,k]   = e4m3_rn_satfinite(float(x[m,k]) / s_x[m])                    (IEEE fp32 division)
 *   P_b[m,n] = sum_{k in b} q[m,k] * w[n,k]                                 (e4m3 wgmma, fp32 accumulation)
 *   acc[m,n] = acc[m,n] + P_b[m,n]                                           for b in increasing order, from 0
 *   y        = T((acc * (s_x[m] * s_w[n])) + bias[n])                       (fp32 products and sum, NOT fused; one
 *                                                                             rounding to T; bias optional, T [N])
 * The bias is added before the one rounding (fbgemm rounds the product first and adds the bias in T).  The fp8
 * tensor-core accumulator is not an exact fp32 sum, so P_b is not exact in general; it joins the fp32 accumulator once
 * per 128-k block.  Split-K: each of the `ks` ranks of a tile sums its own contiguous run of k-blocks in order from 0,
 * and the ranks' fp32 partials are added in rank order before the epilogue.  Deterministic for a launch plan.
 * Envelope: that of block-FP8 (K % 128 == 0, K <= 65536, N % 64 == 0); x, codes, weight, s_w, out, workspace and the
 * quantisers' s_x 16-byte aligned.  Bad arguments return -2 before any CUDA work. */
/* Workspace of b2q_fp8ch_forward for M rows: the codes and token scales (unused by a static-scale layer at M <= 8). */
size_t b2q_fp8ch_workspace_bytes(int M, int K);
/* Dynamic per-token quantiser: x T [M, K] -> codes e4m3 [M, K], s_x fp32 [M]; ub > 0 (+inf: no bound).  Launched with
 * programmatic dependent launch, like b2q_fp8blk_quantize. */
int b2q_fp8ch_quantize(const void* x, void* codes, float* s_x, int M, int K, float ub, int dtype, void* stream);
/* Static quantiser: codes = e4m3_rn_satfinite(x / s_in) with s_in a device fp32 [1]; s_x[m] = s_in for every row. */
int b2q_fp8ch_quantize_static(const void* x, const float* s_in, void* codes, float* s_x, int M, int K, int dtype,
                              void* stream);
/* out T [M, N] from either quantiser's codes and scales; ks = split-K ranks (1..8), <= 0: the heuristic (the plan of
 * b2q_fp8blk_mm). */
int b2q_fp8ch_mm(const void* codes, const float* s_x, const void* weight, const float* s_w, const void* bias, void* out,
                 int M, int K, int N, int dtype, int ks, void* stream);
/* The layer: s_in != NULL selects static scales, else dynamic per-token scales bounded by ub.  Static scales at M <= 8
 * run in ONE launch that quantises the activation blocks it consumes (the codes of b2q_fp8ch_quantize_static, the plan
 * of b2q_fp8ch_mm with ks <= 0, so the output is identical to theirs); otherwise a quantiser + b2q_fp8ch_mm through the
 * workspace under programmatic dependent launch.  Dispatches on M inside the library, so a CUDA graph sees the true M. */
int b2q_fp8ch_forward(const void* x, const void* weight, const float* s_w, const float* s_in, float ub,
                      const void* bias, void* out, int M, int K, int N, int dtype, void* workspace,
                      size_t workspace_bytes, void* stream);

/* Per-channel INT8 (W8A8) layers (an addition to ABI v8 that changes no earlier entry point): compressed-tensors
 * `int-quantized` W8A8 (channel or tensor weights; dynamic per-token or static per-tensor activations).  Weights int8
 * w [N, K] (the checkpoint tensor, unchanged), s_w fp32 [N] as for per-channel FP8.  T = fp16 (dtype 0) or bf16
 * (dtype 1).  For every token row m:
 *   dynamic: s_x[m] = fmaxf(max_k |x[m,k]|, 1e-10f) / 127.f                   (IEEE fp32 division)
 *   static:  s_x[m] = s_in                                                    (the layer's input_scale)
 *   q[m,k]   = (int8) clamp(rint(float(x[m,k]) / s_x[m]), -128, 127)         (IEEE fp32 division, half to even)
 *   acc[m,n] = sum_k q[m,k] * w[n,k]                                          (int32, exact: |acc| <= 2^30)
 *   y        = T(__fmul_rn(float(acc), __fmul_rn(s_x[m], s_w[n])) + bias[n])  (float(acc) rounds to nearest; fp32
 *                                                                              products and sum, NOT fused; one
 *                                                                              rounding to T; bias optional, T [N])
 * An all-zero row gets codes 0 and a finite scale.  The sum is exact, so the output does not depend on the split-K
 * plan: ks = 1, 2, ... and the heuristic give the same bits.  The s8 wgmma accumulates every k-block into the same int32
 * registers and the ranks' partials are added as integers over distributed shared memory.  The envelope is that of
 * per-channel FP8 (K % 128 == 0, K <= 65536, N % 64 == 0; 16-byte aligned x, codes, weight, s_w, out, workspace and
 * the quantisers' s_x).  Bad arguments return -2 before any CUDA work. */
/* Workspace of b2q_int8ch_forward for M rows: the codes and token scales. */
size_t b2q_int8ch_workspace_bytes(int M, int K);
/* Dynamic per-token quantiser: x T [M, K] -> codes int8 [M, K], s_x fp32 [M]; programmatic dependent launch. */
int b2q_int8ch_quantize(const void* x, void* codes, float* s_x, int M, int K, int dtype, void* stream);
/* Static quantiser: codes of x / s_in with s_in a device fp32 [1]; s_x[m] = s_in for every row. */
int b2q_int8ch_quantize_static(const void* x, const float* s_in, void* codes, float* s_x, int M, int K, int dtype,
                               void* stream);
/* out T [M, N] from either quantiser's codes and scales; ks = split-K ranks (1..8), <= 0: the heuristic (the plan of
 * b2q_fp8ch_mm). */
int b2q_int8ch_mm(const void* codes, const float* s_x, const void* weight, const float* s_w, const void* bias, void* out,
                  int M, int K, int N, int dtype, int ks, void* stream);
/* The layer: s_in != NULL selects static scales, else dynamic per-token scales.  A quantiser + b2q_int8ch_mm (ks <= 0)
 * through the workspace under programmatic dependent launch at every M, so the output is identical to theirs.
 * Dispatches on M inside the library, so a CUDA graph sees the true M. */
int b2q_int8ch_forward(const void* x, const void* weight, const float* s_w, const float* s_in, const void* bias,
                       void* out, int M, int K, int N, int dtype, void* workspace, size_t workspace_bytes,
                       void* stream);

/* W4AFP8 layers (an addition to ABI v8 that changes no earlier entry point): compressed-tensors `W4AFP8` checkpoints
 * (`pack-quantized`): symmetric int4 weights q in [-8, 7] with one scale per 128 k, dynamic per-token e4m3 activations,
 * on the e4m3 tensor cores (b2q_w4afp8.cu).  The arithmetic:
 *   (c, s_x) = b2q_fp8ch_quantize(x, ub = +inf)   (the FP8_DYNAMIC quantiser, unchanged: the same codes and scales);
 *   P[m, n, b] = sum over k in block b (128 k = one group) of c[m, k] * q[n, k]  (e4m3 x e4m3 wgmma, fp32 accumulator);
 *   acc[m, n]  = sum over b of P[m, n, b] * s_w[b, n]: acc = fma(P, s_w, acc) once per k-block, in block order within a
 *                split-K rank; the ranks' partials are then summed in rank order (rank 0 first);
 *   y[m, n]    = T(acc[m, n] * s_x[m] + bias[n])  (__fmul_rn, __fadd_rn, one rounding to the output dtype T).
 * Every int4 value is exact in e4m3 and each group scale is applied exactly once, in fp32, to its k-block's partial.
 * Envelope: K % 128 == 0, K <= 65536, N % 128 == 0; bad arguments return an error (never a partial result).
 * Tensors: packed = b2q_w4afp8_packed_bytes(K, N) bytes (16-byte aligned), s_w fp32 [K/128, N] (the checkpoint's
 * weight_scale [N, K/128] widened and transposed), bias [N] in the output dtype or NULL, out [M, N] fp16 / bf16 (dtype
 * of x).  For a given ks the output is deterministic. */
size_t b2q_w4afp8_packed_bytes(int K, int N);
/* Workspace of b2q_w4afp8_forward for M rows: the e4m3 codes and token scales (= b2q_fp8ch_workspace_bytes). */
size_t b2q_w4afp8_workspace_bytes(int M, int K);
/* One-time repack of the checkpoint's weight_packed int32 [N, K/8] (code q + 8 of k in bits 4 (k % 8) of word k / 8)
 * into the kernel's tile layout, in one device pass. */
int b2q_w4afp8_prepack(const int32_t* weight_packed, void* packed, int K, int N, void* stream);
/* out[M, N] from e4m3 codes [M, K] and token scales [M] (b2q_fp8ch_quantize's output).  ks in 1..8 pins the split-K
 * ranks, ks <= 0 takes the heuristic of b2q_w4afp8_forward. */
int b2q_w4afp8_mm(const void* codes, const float* s_x, const void* packed, const float* s_w, const void* bias,
                  void* out, int M, int K, int N, int dtype, int ks, void* stream);
/* The layer: b2q_fp8ch_quantize (ub = +inf) + b2q_w4afp8_mm (ks <= 0) under programmatic dependent launch, through a
 * caller workspace of b2q_w4afp8_workspace_bytes(M, K) bytes (16-byte aligned).  M is dispatched inside the library; no
 * allocation and no host synchronisation, so it can be captured in a CUDA graph. */
int b2q_w4afp8_forward(const void* x, const void* packed, const float* s_w, const void* bias, void* out, int M, int K,
                       int N, int dtype, void* workspace, size_t workspace_bytes, void* stream);

/* Block-FP8 MoE experts (an addition to ABI v8): the experts' w1 / w3 [E*I, K], w2 [E*H, I] e4m3 stacks and their scale
 * stacks [E, ceil(N/128), K/128] (each expert's checkpoint tensors, back to back), the routing tables of b2q_moe_align.
 * One block is six launches with no host synchronisation: b2q_moe_align, b2q_fp8blk_moe_gather, b2q_fp8blk_moe_gate_up,
 * b2q_fp8blk_quantize of h, b2q_fp8blk_moe_down, b2q_moe_combine.  For every routed pair (token t, slot j, expert e),
 * with Q the quantiser and the promotion chain of b2q_fp8blk_mm above:
 *   (c, s_x)  = Q(x_t)                           (the codes b2q_fp8blk_quantize gives the token)
 *   g = T(chain(c, s_x, W1_e)),  u = T(chain(c, s_x, W3_e))
 *   a = T(silu(g)) (silu(g) = g / (1 + __expf(-g)) in fp32),  h = T(a * u)
 *   (c_h, s_h) = Q(h)                            (down_proj quantises its own input, as transformers' FP8Linear)
 *   yp_j = T(chain(c_h, s_h, W2_e))
 *   y_t  = T(sum_j fp32(w_j * yp_j))             (fp32, slot order, one rounding: b2q_moe_combine)
 * These are the rounding points of transformers' per-expert FP8Linear loop.  Each expert's rows run the dense kernel's
 * promotion chain and split-K rank order, so for a pinned ks the grouped results equal b2q_fp8blk_mm on that expert's
 * rows.  Envelope: K % 128 == 0, N % 64 == 0 (the h width I of gate|up also % 128 for its quantiser), E <= 256,
 * ks <= 8, pointers as for b2q_fp8blk_mm. */
/* codes e4m3 [T*top_k, K], s_x fp32 [K/128, Mp(T*top_k)]: sorted row i = Q(x[sorted_pairs[i] / top_k]). */
int b2q_fp8blk_moe_gather(const void* x, const int32_t* sorted_pairs, void* codes, float* s_x, int T, int top_k, int K,
                          int dtype, void* stream);
/* h T [rows, N]: w1 / w3 [E*N, K], N = the intermediate size; active = experts expected to hold rows (grid sizing). */
int b2q_fp8blk_moe_gate_up(const void* codes, const float* s_x, const void* w1, const float* s_w1, const void* w3,
                           const float* s_w3, void* h, const int32_t* counts, const int32_t* offsets, int E, int rows,
                           int active, int K, int N, int dtype, int ks, void* stream);
/* ypair fp32 [rows, N]: row pair = w[pair] * yp of sorted row i, pair = sorted_pairs[i]; w2 [E*N, K], K = the
 * intermediate size. */
int b2q_fp8blk_moe_down(const void* codes_h, const float* s_h, const void* w2, const float* s_w2, const int32_t* counts,
                        const int32_t* offsets, const int32_t* sorted_pairs, const float* pair_weights, float* ypair,
                        int E, int rows, int active, int K, int N, int dtype, int ks, void* stream);

/* Per-channel W8A8 MoE experts, FP8 (b2q_fp8ch_moe_*) and INT8 (b2q_int8ch_moe_*) (an addition to ABI v8): the
 * experts' w1 / w3 [E*I, K], w2 [E*H, I] code stacks (each expert's checkpoint weight [N, K], back to back) and their
 * scale stacks s_w fp32 [E, N] (per-tensor scales broadcast to N), the routing tables of b2q_moe_align.  One block is
 * six launches with no host synchronisation: b2q_moe_align, b2q_*ch_moe_gather, b2q_*ch_moe_gate_up, the quantiser on
 * h, b2q_*ch_moe_down, b2q_moe_combine.  The quantiser on h is b2q_*ch_quantize (dynamic) or b2q_*ch_moe_gather with
 * sorted_pairs = NULL and w2's input scales (static).  For every routed pair (token t, slot j, expert e), with Q the
 * layer quantiser above and s_in[e] the expert's input_scale (static activations):
 *   (c, s_x)  = Q(x_t)                            (dynamic: the token's codes; static: with s_in1[e] = s_in3[e])
 *   g = T(fp32(acc(c, W1_e)) * (s_x * s_w1[e]))   (the layer's y without bias: g and u are the values of the layers)
 *   u = T(fp32(acc(c, W3_e)) * (s_x * s_w3[e]))
 *   a = T(silu(g)) (silu(g) = g / (1 + __expf(-g)) in fp32),  h = T(a * u)
 *   (c_h, s_h) = Q(h)                             (down_proj quantises its own input; static: s_in2[e])
 *   yp_j = T(fp32(acc(c_h, W2_e)) * (s_h * s_w2[e]))
 *   y_t  = T(sum_j fp32(w_j * yp_j))              (fp32, slot order, one rounding: b2q_moe_combine)
 * acc is the k-sum of the dense kernels: exact int32 for INT8 (so every expert's g, u and yp equal b2q_int8ch_mm on its
 * rows at any split), the per-block fp32 chain for FP8 (each expert's rows run the dense kernel's split-K rank order, so
 * for a pinned ks its results equal b2q_fp8ch_mm on that expert's rows).  Envelope: K % 128 == 0, N % 64 == 0 (the h
 * width I also % 128, as the down launch's K), E <= 256, ks <= 8, pointers as for b2q_fp8ch_mm; bad arguments return
 * -2 before any CUDA work. */
/* codes [T*top_k, K], s_x fp32 [T*top_k]: sorted row i = Q(x[sorted_pairs[i] / top_k]), or Q(x[i]) of an x already
 * [T*top_k, K] in sorted order when sorted_pairs is NULL.  s_in NULL: dynamic per-token scales (FP8: amax bounded by
 * ub > 0, +inf: no bound); else fp32 [E], row i takes the scale of the expert whose rows hold it (offsets [E], E). */
int b2q_fp8ch_moe_gather(const void* x, const int32_t* sorted_pairs, const int32_t* offsets, const float* s_in, int E,
                         void* codes, float* s_x, int T, int top_k, int K, float ub, int dtype, void* stream);
/* h T [rows, N]: w1 / w3 [E*N, K], s_w1 / s_w3 [E, N], N = the intermediate size; active = experts expected to hold
 * rows (grid sizing); ks = split-K ranks (1..8), <= 0: the heuristic. */
int b2q_fp8ch_moe_gate_up(const void* codes, const float* s_x, const void* w1, const float* s_w1, const void* w3,
                          const float* s_w3, void* h, const int32_t* counts, const int32_t* offsets, int E, int rows,
                          int active, int K, int N, int dtype, int ks, void* stream);
/* ypair fp32 [rows, N]: row pair = w[pair] * yp of sorted row i, pair = sorted_pairs[i]; w2 [E*N, K], K = the
 * intermediate size. */
int b2q_fp8ch_moe_down(const void* codes_h, const float* s_h, const void* w2, const float* s_w2, const int32_t* counts,
                       const int32_t* offsets, const int32_t* sorted_pairs, const float* pair_weights, float* ypair,
                       int E, int rows, int active, int K, int N, int dtype, int ks, void* stream);
/* The INT8 twins: int8 codes and weights, no amax bound. */
int b2q_int8ch_moe_gather(const void* x, const int32_t* sorted_pairs, const int32_t* offsets, const float* s_in, int E,
                          void* codes, float* s_x, int T, int top_k, int K, int dtype, void* stream);
int b2q_int8ch_moe_gate_up(const void* codes, const float* s_x, const void* w1, const float* s_w1, const void* w3,
                           const float* s_w3, void* h, const int32_t* counts, const int32_t* offsets, int E, int rows,
                           int active, int K, int N, int dtype, int ks, void* stream);
int b2q_int8ch_moe_down(const void* codes_h, const float* s_h, const void* w2, const float* s_w2, const int32_t* counts,
                        const int32_t* offsets, const int32_t* sorted_pairs, const float* pair_weights, float* ypair,
                        int E, int rows, int active, int K, int N, int dtype, int ks, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2Q_H_ */
