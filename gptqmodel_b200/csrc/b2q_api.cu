// b2q_api.cu — the extern "C" boundary declared in include/b2q.h: argument validation + tier dispatch.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "../../include/b2q.h"
#include "b2q_gemm.cuh"
#include "b2q_internal.h"

namespace b2q {
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  return (e != nullptr && e[0] != 0) ? atoi(e) : dflt;
}

static EnvCfg read_env() {
  EnvCfg c;
  c.disable_pdl = env_int("B2Q_DISABLE_PDL", 0);
  c.midm = env_int("B2Q_MIDM", 1);
  c.decode_v2 = env_int("B2Q_DECODE_V2", -1);
  c.decode2_gw = env_int("B2Q_DECODE2_GW", 0);
  c.decode2_xtma = env_int("B2Q_DECODE2_XTMA", 0);
  c.midm_ks = env_int("B2Q_MIDM_KS", 0);
  return c;
}

int num_sms() {
  static int cache[32] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 32) {
    (void)cudaGetLastError();
    return 132;
  }
  if (cache[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      (void)cudaGetLastError();
      n = 132;
    }
    cache[dev] = n < 160 ? n : 160;  // the decode all-reduce keeps flag columns for at most 160 CTAs per launch
  }
  return cache[dev];
}

static EnvCfg g_env = read_env();  // once, at library load
const EnvCfg& env() { return g_env; }
void reload_env() { g_env = read_env(); }

// Every entry point runs on the device that owns its pointers, whatever the caller's current device is (a module on
// cuda:1 called while cuda:0 is current — ADVICE r01): switch for the duration of the call, restore afterwards.
struct DeviceGuard {
  int prev = -1, dev = -1;
  explicit DeviceGuard(const void* p) {
    cudaPointerAttributes at;
    if (p != nullptr && cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeDevice) {
      dev = at.device;
      if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) cudaSetDevice(dev);
      else prev = -1;
    }
    (void)cudaGetLastError();
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

static int check_cuda(int e, const char* what) {
  if (e > 0) set_error("%s: CUDA error %d (%s)", what, e, cudaGetErrorString((cudaError_t)e));
  return e;
}

static int validate(const char* fn, const void* x, const void* packed, const void* scales, const void* out, int M,
                    int K, int N, int bits, int group_size, int dtype) {
  if (x == nullptr || packed == nullptr || scales == nullptr || out == nullptr) {
    set_error("%s: null pointer argument", fn);
    return -2;
  }
  if (bits != 4 && bits != 8) {
    set_error("%s: bits=%d not supported (4 or 8)", fn, bits);
    return -2;
  }
  if (dtype != B2Q_DTYPE_F16 && dtype != B2Q_DTYPE_BF16) {
    set_error("%s: dtype=%d not supported (0 fp16, 1 bf16)", fn, dtype);
    return -2;
  }
  if (M < 0 || K <= 0 || N <= 0 || K % 64 != 0 || N % 32 != 0) {
    set_error("%s: shape M=%d K=%d N=%d not supported (K multiple of 64, N multiple of 32)", fn, M, K, N);
    return -2;
  }
  // the tensor-core tiers index scale rows by log2(32-k chunks per group) and treat any other size as per-channel
  // (gemm_gshc): a group of 96 or 256 would read group 0's scales for every k
  if (!((group_size == 32 || group_size == 64 || group_size == 128) && K % group_size == 0) && group_size != K) {
    set_error("%s: group_size=%d not supported for K=%d (32 | 64 | 128 dividing K, or K)", fn, group_size, K);
    return -2;
  }
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(out) & 15) ||
      (reinterpret_cast<uintptr_t>(packed) & 15)) {
    set_error("%s: x, out and packed must be 16-byte aligned", fn);
    return -2;
  }
  return 0;
}

static MmArgs make_args(const void* x, const void* packed, const void* scales, const int32_t* qzeros,
                        const int32_t* perm, const void* bias, void* out, int M, int K, int N, int bits,
                        int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  MmArgs a;
  a.x = x;
  a.packed = packed;
  a.scales = scales;
  a.qzeros = qzeros;
  a.perm = perm;
  a.bias = bias;
  a.out = out;
  a.M = M;
  a.K = K;
  a.N = N;
  a.bits = bits;
  a.group_size = group_size;
  a.dtype = dtype;
  a.workspace = workspace;
  a.workspace_bytes = workspace_bytes;
  a.stream = (cudaStream_t)stream;
  a.tune_ks = 0;
  a.tune_warps = 0;
  a.fp8 = 0;
  return a;
}

// forced split-K cluster size / warps per CTA of b2q_gemv and b2q_decode (0: the planner's choice)
static int check_tune(const char* fn, int ks, int warps) {
  if (ks > 16 || warps > 16 || (ks > 0 && (ks & (ks - 1)) != 0)) {
    set_error("%s: ks=%d (power of two <= 16) / warps=%d (<= 16) out of range", fn, ks, warps);
    return -2;
  }
  return 0;
}
}  // namespace b2q

using namespace b2q;

extern "C" {

int b2q_version(void) { return B2Q_ABI_VERSION; }

int b2q_debug_decode_plan(int version, int M, int K, int N, int ks, int warps, int* out8) {
  if (out8 == nullptr || (version != 1 && version != 2) || M < 1 || M > 8 || K < 128 || K % 128 != 0 || N < 32 ||
      N % 32 != 0) {
    set_error("b2q_debug_decode_plan: bad argument (version=%d M=%d K=%d N=%d)", version, M, K, N);
    return -2;
  }
  MmArgs a = {};
  a.M = M;
  a.K = K;
  a.N = N;
  a.bits = 4;
  a.group_size = 128;
  a.tune_ks = ks;
  a.tune_warps = warps;
  if (!decode_plan(version, a, N / 32, out8)) {
    set_error("b2q_debug_decode_plan: no configuration fits shared memory (version=%d M=%d K=%d N=%d)", version, M, K, N);
    return -1;
  }
  return 0;
}

int b2q_debug_wgmma_plan(int tier, int mode, int M, int K, int N, int active, int ks, int* out4) {
  bool ok = out4 != nullptr && M >= 1 && K > 0 && N > 0 && active >= 0 && ks >= 0 && ks <= 8;
  if (tier == 0) ok = ok && mode >= 0 && mode <= 2 && (mode != 0 || M <= 128) && K % 64 == 0 && N % 32 == 0;
  else if (tier == 1) ok = ok && mode == 0 && ks == 0 && K <= 65536 && K % 64 == 0 && N % 64 == 0 && (K % 128 == 0 || N % 128 == 0);
  else if (tier == 2) ok = ok && mode >= 0 && mode <= 2 && K <= 65536 && K % 128 == 0 && N % 64 == 0;
  else ok = false;
  if (!ok) {
    set_error("b2q_debug_wgmma_plan: bad argument (tier=%d mode=%d M=%d K=%d N=%d active=%d ks=%d)", tier, mode, M, K, N,
              active, ks);
    return -2;
  }
  const SwapPlan p = tier == 0 ? midm_plan(mode, M, K, N, active, ks)
                     : tier == 1 ? qqq_plan(M, K, N)
                                 : fp8blk_plan(mode, M, K, N, active, ks);
  out4[0] = p.ntok;
  out4[1] = p.ks;
  out4[2] = p.kpc;
  out4[3] = p.tblocks;
  return 0;
}

int b2q_debug_decode_occupancy(int version, int M, int K, int N, int ks, int warps, int* blocks) {
  if (blocks == nullptr || (version != 1 && version != 2) || M < 1 || M > 8 || K < 128 || K % 128 != 0 || N < 32 ||
      N % 32 != 0) {
    set_error("b2q_debug_decode_occupancy: bad argument (version=%d M=%d K=%d N=%d)", version, M, K, N);
    return -2;
  }
  MmArgs a = {};
  a.M = M;
  a.K = K;
  a.N = N;
  a.bits = 4;
  a.group_size = 128;
  a.tune_ks = ks;
  a.tune_warps = warps;
  return decode_occupancy(version, a, N / 32, blocks);
}

const char* b2q_last_error(void) { return g_err; }

size_t b2q_packed_bytes(int K, int N, int bits) { return (size_t)K * (size_t)N * (size_t)bits / 8; }

size_t b2q_workspace_bytes(int M, int K, int N, int has_perm) {
  // conservative (tier-independent) size: an act-order layer may need the permuted copy of x at ANY M >= 1 when no
  // decode-tier configuration applies (8-bit, group_size 32, K % 128 != 0).  b2q_mm_workspace_bytes() is exact.
  (void)N;
  return (has_perm && M >= 1) ? (size_t)M * (size_t)K * 2 : 0;
}

size_t b2q_mm_workspace_bytes(int M, int K, int N, int bits, int group_size, int has_perm) {
  if (!has_perm || M < 1) return 0;
  MmArgs a = {};
  a.M = M;
  a.K = K;
  a.N = N;
  a.bits = bits;
  a.group_size = group_size;
  // the decode tier gathers x[perm] while staging the activations, and so does the 8-bit GEMV
  if (decode_supported(a) || gemv_supported(a)) return 0;
  return (size_t)M * (size_t)K * 2;
}

void b2q_debug_reload_env(void) { reload_env(); }

int b2q_prepack(const int32_t* qweight, const int32_t* perm, void* packed, int K, int N, int bits, void* stream) {
  if (qweight == nullptr || packed == nullptr) {
    set_error("b2q_prepack: null pointer argument");
    return -2;
  }
  if ((bits != 4 && bits != 8) || K <= 0 || N <= 0 || K % 64 != 0 || N % 32 != 0) {
    set_error("b2q_prepack: bits=%d K=%d N=%d not supported (bits 4|8, K multiple of 64, N multiple of 32)", bits, K,
              N);
    return -2;
  }
  DeviceGuard dg(packed);
  return check_cuda(launch_prepack(qweight, perm, packed, K, N, bits, (cudaStream_t)stream), "b2q_prepack");
}

int b2q_allreduce(void* inout, int n, int dtype, int rank, int world, const void* const* peer_bufs, size_t flag_offset,
                  int max_elems, void* seq, void* stream) {
  if (inout == nullptr || peer_bufs == nullptr || seq == nullptr || world < 1 || world > 8 || rank < 0 ||
      rank >= world || n <= 0 || n % 8 != 0 || n > max_elems || (dtype != 0 && dtype != 1) ||
      (reinterpret_cast<uintptr_t>(inout) & 15) || flag_offset % 16 != 0) {
    set_error("b2q_allreduce: bad argument (n=%d max=%d rank=%d world=%d; n %% 8 == 0, 16-byte aligned, world <= 8)", n,
              max_elems, rank, world);
    return -2;
  }
  for (int i = 0; i < world; ++i)
    if (peer_bufs[i] == nullptr) {
      set_error("b2q_allreduce: peer buffer %d is NULL", i);
      return -2;
    }
  DeviceGuard dg(inout);
  return check_cuda(launch_allreduce(inout, n, dtype, rank, world, peer_bufs, flag_offset, max_elems, seq,
                                     (cudaStream_t)stream), "b2q_allreduce");
}

int b2q_decode_allreduce(const void* x, const void* packed, const void* scales, const int32_t* qzeros,
                         const void* bias, void* out, int M, int K, int N, int bits, int group_size, int dtype,
                         int rank, int world, const void* const* peer_bufs, size_t flag_offset, int max_elems,
                         void* ctl, void* stream) {
  int v = validate("b2q_decode_allreduce", x, packed, scales, out, M, K, N, bits, group_size, dtype);
  if (v != 0) return v;
  DeviceGuard dg(packed);
  if (peer_bufs == nullptr || ctl == nullptr || world < 2 || world > 8 || rank < 0 || rank >= world || max_elems <= 0 ||
      (size_t)M * (size_t)N > (size_t)max_elems || flag_offset % 16 != 0 ||
      flag_offset < (size_t)2 * world * (size_t)max_elems * sizeof(float)) {
    set_error("b2q_decode_allreduce: bad argument (rank=%d world=%d M*N=%lld max_elems=%d flag_offset=%zu; 2 <= world <= 8, "
              "M*N <= max_elems, flag_offset >= 2*world*max_elems*4 and a multiple of 16)",
              rank, world, (long long)M * N, max_elems, flag_offset);
    return -2;
  }
  DecodeAR ar = {};
  ar.world = world;
  ar.rank = rank;
  ar.max_elems = max_elems;
  ar.flag_offset = flag_offset;
  ar.ctl = (uint32_t*)ctl;
  for (int i = 0; i < world; ++i) {
    if (peer_bufs[i] == nullptr) {
      set_error("b2q_decode_allreduce: peer buffer %d is NULL", i);
      return -2;
    }
    ar.buf[i] = const_cast<void*>(peer_bufs[i]);
  }
  MmArgs a = make_args(x, packed, scales, qzeros, nullptr, bias, out, M, K, N, bits, group_size, dtype, nullptr, 0,
                       stream);
  if (!decode_supported(a)) {
    set_error("b2q_decode_allreduce: needs bits=4, 1 <= M <= 8, K %% 128 == 0, group_size 64|128|K (got bits=%d M=%d K=%d "
              "g=%d)", bits, M, K, group_size);
    return -2;
  }
  return check_cuda(launch_decode_allreduce(a, ar), "b2q_decode_allreduce");
}

size_t b2q_decode_allreduce_flag_bytes(void) { return decode_allreduce_flag_bytes(); }

int b2q_permute_cols(const void* x, const int32_t* perm, void* out, int M, int K, void* stream) {
  if (x == nullptr || perm == nullptr || out == nullptr || M < 0 || K <= 0) {
    set_error("b2q_permute_cols: bad argument");
    return -2;
  }
  if (M == 0) return 0;
  DeviceGuard dg(out);
  return check_cuda(launch_permute_cols(x, perm, out, M, K, (cudaStream_t)stream), "b2q_permute_cols");
}

int b2q_hadamard(const void* x, const int8_t* had, int K, void* out, int rows, int n, int dtype, void* stream) {
  if (x == nullptr || out == nullptr || rows < 0) {
    set_error("b2q_hadamard: bad argument (x, out non-NULL, rows=%d >= 0)", rows);
    return -2;
  }
  if (dtype != B2Q_DTYPE_F16 && dtype != B2Q_DTYPE_BF16) {
    set_error("b2q_hadamard: dtype=%d not supported (0 fp16, 1 bf16)", dtype);
    return -2;
  }
  if (K < 1 || K > 256 || n <= 0 || n > 65536 || n % K != 0) {
    set_error("b2q_hadamard: K=%d n=%d outside 1 <= K <= 256, n <= 65536, K dividing n", K, n);
    return -2;
  }
  const int P = n / K;
  if (P < 8 || (P & (P - 1)) != 0) {
    set_error("b2q_hadamard: P = n/K = %d must be a power of two >= 8 (n=%d K=%d)", P, n, K);
    return -2;
  }
  if ((had == nullptr) != (K == 1)) {
    set_error("b2q_hadamard: had must be NULL exactly when K == 1 (K=%d)", K);
    return -2;
  }
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(out) & 15) ||
      (reinterpret_cast<uintptr_t>(had) & 15)) {
    set_error("b2q_hadamard: x, out and had must be 16-byte aligned");
    return -2;
  }
  const uintptr_t xb = reinterpret_cast<uintptr_t>(x), ob = reinterpret_cast<uintptr_t>(out);
  const uintptr_t bytes = (uintptr_t)rows * (uintptr_t)n * 2;
  if (xb == ob || (rows > 0 && xb < ob + bytes && ob < xb + bytes)) {
    set_error("b2q_hadamard: out must not overlap x");
    return -2;
  }
  if (rows == 0) return 0;
  DeviceGuard dg(out);
  return check_cuda(launch_hadamard(x, had, K, out, rows, n, dtype, (cudaStream_t)stream), "b2q_hadamard");
}

// ---- QQQ (W4A8) tier ----
static size_t qqq_kp(int K) { return ((size_t)K + 127) / 128 * 128; }
static size_t qqq_scale_bytes(int M) { return ((size_t)M * 4 + 127) / 128 * 128; }
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// the reference's IN_OUTPUT_FEATURES_DIVISIBLE_BY, K <= 65536 (exact int32 sums), group size -1 or 128
static int qqq_check_shape(const char* fn, int M, int K, int N, int group_size) {
  const bool env_ok = (K % 128 == 0 && N % 64 == 0) || (K % 64 == 0 && N % 128 == 0);
  if (M < 0 || K <= 0 || N <= 0 || K > 65536 || !env_ok) {
    set_error("%s: shape M=%d K=%d N=%d outside the envelope (K %% 128 == 0 and N %% 64 == 0, or K %% 64 == 0 and "
              "N %% 128 == 0; K <= 65536)", fn, M, K, N);
    return -2;
  }
  if (group_size != -1 && !(group_size == 128 && K % 128 == 0)) {
    set_error("%s: group_size=%d not supported for K=%d (-1, or 128 dividing K)", fn, group_size, K);
    return -2;
  }
  return 0;
}

size_t b2q_qqq_packed_bytes(int K, int N) {
  if (K <= 0 || N <= 0) return 0;
  return qqq_kp(K) * (((size_t)N + 127) / 128 * 128) / 2;
}

size_t b2q_qqq_workspace_bytes(int M, int K) {
  if (M <= 0 || K <= 0) return 0;
  return qqq_scale_bytes(M) + (size_t)M * qqq_kp(K);
}

int b2q_qqq_prepack(const uint8_t* codes, void* packed, int K, int N, int group_size, void* stream) {
  if (codes == nullptr || packed == nullptr) {
    set_error("b2q_qqq_prepack: null pointer argument");
    return -2;
  }
  if (int e = qqq_check_shape("b2q_qqq_prepack", 0, K, N, group_size)) return e;
  if (!aligned16(packed)) {
    set_error("b2q_qqq_prepack: packed must be 16-byte aligned");
    return -2;
  }
  DeviceGuard dg(packed);
  return check_cuda(launch_qqq_prepack(codes, packed, K, N, group_size == 128 ? 1 : 0, (cudaStream_t)stream),
                    "b2q_qqq_prepack");
}

int b2q_qqq_quantize(const void* x, int8_t* q, float* s_tok, int M, int K, int dtype, void* stream) {
  if ((M > 0 && (x == nullptr || q == nullptr || s_tok == nullptr)) || M < 0 || K <= 0 || K % 64 != 0 || K > 65536) {
    set_error("b2q_qqq_quantize: bad argument (non-NULL pointers, M=%d >= 0, K=%d a multiple of 64 <= 65536)", M, K);
    return -2;
  }
  if (dtype != B2Q_DTYPE_F16 && dtype != B2Q_DTYPE_BF16) {
    set_error("b2q_qqq_quantize: dtype=%d not supported (0 fp16, 1 bf16)", dtype);
    return -2;
  }
  if (!aligned16(x) || !aligned16(q)) {
    set_error("b2q_qqq_quantize: x and q must be 16-byte aligned");
    return -2;
  }
  if (M == 0) return 0;
  DeviceGuard dg(q);
  return check_cuda(launch_qqq_quant(x, q, s_tok, M, K, dtype, (cudaStream_t)stream), "b2q_qqq_quantize");
}

static int qqq_mm(const char* fn, const int8_t* q, const float* s_tok, const void* packed, const float* s_channel,
                  const void* s_group, const void* bias, void* out, int M, int K, int N, int out_dtype,
                  cudaStream_t stream) {
  QqqArgs a = {q, s_tok, packed, s_channel, s_group, bias, out, M, K, N, out_dtype, stream};
  return check_cuda(launch_qqq_gemm(a), fn);
}

static int qqq_check_mm(const char* fn, const void* packed, const float* s_channel, const void* s_group, void* out,
                        int M, int K, int N, int group_size, int out_dtype) {
  if (packed == nullptr || s_channel == nullptr || out == nullptr) {
    set_error("%s: null pointer argument", fn);
    return -2;
  }
  if (int e = qqq_check_shape(fn, M, K, N, group_size)) return e;
  if ((group_size == 128) != (s_group != nullptr)) {
    set_error("%s: s_group must be given exactly for group_size 128 (group_size=%d)", fn, group_size);
    return -2;
  }
  if (out_dtype != B2Q_DTYPE_F16 && out_dtype != B2Q_DTYPE_BF16) {
    set_error("%s: dtype=%d not supported (0 fp16, 1 bf16)", fn, out_dtype);
    return -2;
  }
  if (!aligned16(packed) || !aligned16(out) || !aligned16(s_channel)) {
    set_error("%s: packed, out and s_channel must be 16-byte aligned", fn);
    return -2;
  }
  return 0;
}

int b2q_qqq_mm(const int8_t* q, const float* s_tok, const void* packed, const float* s_channel, const void* s_group,
               const void* bias, void* out, int M, int K, int N, int group_size, int out_dtype, void* stream) {
  if (int e = qqq_check_mm("b2q_qqq_mm", packed, s_channel, s_group, out, M, K, N, group_size, out_dtype)) return e;
  if (M > 0 && (q == nullptr || s_tok == nullptr || !aligned16(q))) {
    set_error("b2q_qqq_mm: q (16-byte aligned) and s_tok must be given");
    return -2;
  }
  if (M == 0) return 0;
  DeviceGuard dg(packed);
  return qqq_mm("b2q_qqq_mm", q, s_tok, packed, s_channel, s_group, bias, out, M, K, N, out_dtype,
                (cudaStream_t)stream);
}

int b2q_qqq_forward(const void* x, const void* packed, const float* s_channel, const void* s_group, const void* bias,
                    void* out, int M, int K, int N, int group_size, int dtype, int out_dtype, void* workspace,
                    size_t workspace_bytes, void* stream) {
  if (int e = qqq_check_mm("b2q_qqq_forward", packed, s_channel, s_group, out, M, K, N, group_size, out_dtype))
    return e;
  if (dtype != B2Q_DTYPE_F16 && dtype != B2Q_DTYPE_BF16) {
    set_error("b2q_qqq_forward: dtype=%d not supported (0 fp16, 1 bf16)", dtype);
    return -2;
  }
  if (M == 0) return 0;
  if (x == nullptr || !aligned16(x) || workspace == nullptr || !aligned16(workspace) ||
      workspace_bytes < b2q_qqq_workspace_bytes(M, K)) {
    set_error("b2q_qqq_forward: x and a workspace of b2q_qqq_workspace_bytes(M, K) = %zu bytes (16-byte aligned) "
              "must be given, got %zu", b2q_qqq_workspace_bytes(M, K), workspace_bytes);
    return -2;
  }
  DeviceGuard dg(packed);
  float* s_tok = reinterpret_cast<float*>(workspace);
  int8_t* q = reinterpret_cast<int8_t*>(workspace) + qqq_scale_bytes(M);
  int e = check_cuda(launch_qqq_quant(x, q, s_tok, M, K, dtype, (cudaStream_t)stream), "b2q_qqq_forward");
  if (e != 0) return e;
  return qqq_mm("b2q_qqq_forward", q, s_tok, packed, s_channel, s_group, bias, out, M, K, N, out_dtype,
                (cudaStream_t)stream);
}

// ---- QQQ MoE experts: the grouped modes of qqq_gemm_kernel over the routing tables of b2q_moe_align ----
int b2q_qqq_moe_gather(const void* x, const int32_t* sorted_pairs, int8_t* q, float* s_tok, int T, int top_k, int K,
                       int dtype, void* stream) {
  if (T < 1 || top_k < 1 || K <= 0 || K % 64 != 0 || K > 65536) {
    set_error("b2q_qqq_moe_gather: T=%d, top_k=%d must be >= 1 and K=%d a multiple of 64 <= 65536", T, top_k, K);
    return -2;
  }
  if (dtype != B2Q_DTYPE_F16 && dtype != B2Q_DTYPE_BF16) {
    set_error("b2q_qqq_moe_gather: dtype=%d not supported (0 fp16, 1 bf16)", dtype);
    return -2;
  }
  if (x == nullptr || sorted_pairs == nullptr || q == nullptr || s_tok == nullptr || !aligned16(x) || !aligned16(q)) {
    set_error("b2q_qqq_moe_gather: x, sorted_pairs, q and s_tok must be device pointers, x and q 16-byte aligned");
    return -2;
  }
  DeviceGuard dg(q);
  return check_cuda(launch_qqq_moe_gather(x, sorted_pairs, q, s_tok, T * top_k, top_k, K, dtype, (cudaStream_t)stream),
                    "b2q_qqq_moe_gather");
}

static int qqq_moe_check(const char* fn, const int8_t* q, const float* s_tok, const void* packed,
                         const float* s_channel, const void* s_group, void* out, const int32_t* counts,
                         const int32_t* offsets, int E, int rows, int K, int N, int group_size, int dtype) {
  if (int e = qqq_check_mm(fn, packed, s_channel, s_group, out, rows, K, N, group_size, dtype)) return e;
  if (q == nullptr || s_tok == nullptr || counts == nullptr || offsets == nullptr || !aligned16(q)) {
    set_error("%s: q, s_tok, counts and offsets must be device pointers, q 16-byte aligned", fn);
    return -2;
  }
  if (E < 1 || E > 256 || rows < 1) {
    set_error("%s: E=%d (1..256), rows=%d (>= 1) outside the envelope", fn, E, rows);
    return -2;
  }
  return 0;
}

int b2q_qqq_moe_gate_up(const int8_t* q, const float* s_tok, const void* packed1, const float* s_channel1,
                        const void* s_group1, const void* packed3, const float* s_channel3, const void* s_group3, void* h,
                        const int32_t* counts, const int32_t* offsets, int E, int rows, int active, int K, int N,
                        int group_size, int dtype, void* stream) {
  if (int e = qqq_moe_check("b2q_qqq_moe_gate_up", q, s_tok, packed1, s_channel1, s_group1, h, counts, offsets, E, rows,
                            K, N, group_size, dtype))
    return e;
  if (int e = qqq_check_mm("b2q_qqq_moe_gate_up", packed3, s_channel3, s_group3, h, rows, K, N, group_size, dtype))
    return e;
  if (N % 64 != 0) {
    set_error("b2q_qqq_moe_gate_up: N=%d must be a multiple of 64 (64 gate + 64 up features per tile)", N);
    return -2;
  }
  DeviceGuard dg(packed1);
  QqqArgs a = {q, s_tok, packed1, s_channel1, s_group1, nullptr, h, rows, K, N, dtype, (cudaStream_t)stream};
  QqqMoe g = {};
  g.counts = counts;
  g.offsets = offsets;
  g.packed3 = packed3;
  g.s_channel3 = s_channel3;
  g.s_group3 = s_group3;
  g.E = E;
  g.active = active;
  return check_cuda(launch_qqq_moe(1, a, g), "b2q_qqq_moe_gate_up");
}

int b2q_qqq_moe_down(const int8_t* q_h, const float* s_h, const void* packed2, const float* s_channel2,
                     const void* s_group2, const int32_t* counts, const int32_t* offsets, const int32_t* sorted_pairs,
                     const float* pair_weights, float* ypair, int E, int rows, int active, int K, int N, int group_size,
                     int dtype, void* stream) {
  if (int e = qqq_moe_check("b2q_qqq_moe_down", q_h, s_h, packed2, s_channel2, s_group2, ypair, counts, offsets, E, rows,
                            K, N, group_size, dtype))
    return e;
  if (sorted_pairs == nullptr || pair_weights == nullptr) {
    set_error("b2q_qqq_moe_down: sorted_pairs and pair_weights must be device pointers");
    return -2;
  }
  DeviceGuard dg(packed2);
  QqqArgs a = {q_h, s_h, packed2, s_channel2, s_group2, nullptr, ypair, rows, K, N, dtype, (cudaStream_t)stream};
  QqqMoe g = {};
  g.counts = counts;
  g.offsets = offsets;
  g.sorted_pairs = sorted_pairs;
  g.pair_weights = pair_weights;
  g.ypair = ypair;
  g.E = E;
  g.active = active;
  return check_cuda(launch_qqq_moe(2, a, g), "b2q_qqq_moe_down");
}

// ---- FP8 (e4m3fn, W8A16) layers on the 8-bit tiers ----
static int fp8_check(const char* fn, const void* packed, const void* scales, const void* out, int K, int N,
                     int group_size, int dtype) {
  if (packed == nullptr || scales == nullptr || out == nullptr) {
    set_error("%s: null pointer argument", fn);
    return -2;
  }
  if (dtype != B2Q_DTYPE_F16 && dtype != B2Q_DTYPE_BF16) {
    set_error("%s: dtype=%d not supported (0 fp16, 1 bf16)", fn, dtype);
    return -2;
  }
  if (K <= 0 || N <= 0 || K % 64 != 0 || N % 32 != 0) {
    set_error("%s: shape K=%d N=%d not supported (K multiple of 64, N multiple of 32)", fn, K, N);
    return -2;
  }
  if (!((group_size == 64 || group_size == 128 || group_size == K) && K % group_size == 0)) {
    set_error("%s: group_size=%d not supported for K=%d (64 | 128 dividing K, or K)", fn, group_size, K);
    return -2;
  }
  if (!aligned16(packed) || !aligned16(out)) {
    set_error("%s: packed and out must be 16-byte aligned", fn);
    return -2;
  }
  return 0;
}

int b2q_fp8_mm(const void* x, const void* packed, const void* scales, const void* bias, void* out, int M, int K, int N,
               int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  if (int e = fp8_check("b2q_fp8_mm", packed, scales, out, K, N, group_size, dtype)) return e;
  if (M < 0 || (M > 0 && (x == nullptr || !aligned16(x)))) {
    set_error("b2q_fp8_mm: M=%d must be >= 0 and x a 16-byte aligned pointer", M);
    return -2;
  }
  if (M == 0) return 0;
  DeviceGuard dg(packed);
  MmArgs a = make_args(x, packed, scales, nullptr, nullptr, bias, out, M, K, N, 8, group_size, dtype, workspace,
                       workspace_bytes, stream);
  a.fp8 = 1;
  if (gemv_supported(a)) return check_cuda(launch_gemv(a), "b2q_fp8_mm(gemv)");
  return check_cuda(launch_gemm(a), "b2q_fp8_mm(gemm)");
}

int b2q_fp8_dequant(const void* packed, const void* scales, void* out, int K, int N, int group_size, int dtype,
                    void* stream) {
  if (int e = fp8_check("b2q_fp8_dequant", packed, scales, out, K, N, group_size, dtype)) return e;
  DeviceGuard dg(packed);
  return check_cuda(launch_fp8_dequant(packed, scales, out, K, N, group_size, dtype, (cudaStream_t)stream),
                    "b2q_fp8_dequant");
}

// ---- FP8 MoE experts: the grouped modes of the small-batch tier with the FP8 dequantisation ----
static int fp8_moe_check(const char* fn, const void* x, const void* packed, const void* scales, const void* out,
                         const int32_t* counts, const int32_t* offsets, int E, int rows, int K, int N, int group_size,
                         int dtype) {
  if (int e = fp8_check(fn, packed, scales, out, K, N, group_size, dtype)) return e;
  if (x == nullptr || counts == nullptr || offsets == nullptr || !aligned16(x)) {
    set_error("%s: x, counts and offsets must be device pointers, x 16-byte aligned", fn);
    return -2;
  }
  if (E < 1 || E > 256 || rows < 1) {
    set_error("%s: E=%d (1..256), rows=%d (>= 1) outside the envelope", fn, E, rows);
    return -2;
  }
  return 0;
}

int b2q_fp8_moe_gate_up(const void* xs, const void* packed1, const void* scales1, const void* packed3,
                        const void* scales3, void* h, const int32_t* counts, const int32_t* offsets, int E, int rows,
                        int active, int K, int N, int group_size, int dtype, void* stream) {
  if (int e = fp8_moe_check("b2q_fp8_moe_gate_up", xs, packed1, scales1, h, counts, offsets, E, rows, K, N, group_size,
                            dtype))
    return e;
  if (int e = fp8_check("b2q_fp8_moe_gate_up", packed3, scales3, h, K, N, group_size, dtype)) return e;
  DeviceGuard dg(packed1);
  MmArgs a = make_args(xs, packed1, scales1, nullptr, nullptr, nullptr, h, rows, K, N, 8, group_size, dtype, nullptr, 0,
                       stream);
  a.fp8 = 1;
  MoeGroupedArgs g = {};
  g.counts = counts;
  g.offsets = offsets;
  g.packed3 = packed3;
  g.scales3 = scales3;
  g.E = E;
  g.rows = rows;
  g.active = active;
  return check_cuda(launch_midm_grouped(1, a, g), "b2q_fp8_moe_gate_up");
}

int b2q_fp8_moe_down(const void* h, const void* packed2, const void* scales2, const int32_t* counts,
                     const int32_t* offsets, const int32_t* sorted_pairs, const float* pair_weights, float* ypair, int E,
                     int rows, int active, int K, int N, int group_size, int dtype, void* stream) {
  if (int e = fp8_moe_check("b2q_fp8_moe_down", h, packed2, scales2, ypair, counts, offsets, E, rows, K, N, group_size,
                            dtype))
    return e;
  if (sorted_pairs == nullptr || pair_weights == nullptr) {
    set_error("b2q_fp8_moe_down: sorted_pairs and pair_weights must be device pointers");
    return -2;
  }
  DeviceGuard dg(packed2);
  MmArgs a = make_args(h, packed2, scales2, nullptr, nullptr, nullptr, ypair, rows, K, N, 8, group_size, dtype, nullptr, 0,
                       stream);
  a.fp8 = 1;
  MoeGroupedArgs g = {};
  g.counts = counts;
  g.offsets = offsets;
  g.sorted_pairs = sorted_pairs;
  g.pair_weights = pair_weights;
  g.ypair = ypair;
  g.E = E;
  g.rows = rows;
  g.active = active;
  return check_cuda(launch_midm_grouped(2, a, g), "b2q_fp8_moe_down");
}

// ---- block-FP8 (HF / DeepSeek-native, W8A8) tier ----
static size_t fp8blk_codes_bytes(int M, int K) { return ((size_t)M * K + 127) / 128 * 128; }

size_t b2q_fp8blk_workspace_bytes(int M, int K) {
  if (M <= 8 || K <= 0 || K % 128 != 0) return 0;  // decode quantises inside the GEMM
  return fp8blk_codes_bytes(M, K) + (size_t)(K / 128) * fp8blk_mp(M) * 4;
}

static int fp8blk_check_shape(const char* fn, int M, int K, int N, int dtype) {
  if (M < 0 || K <= 0 || K % 128 != 0 || K > 65536 || N <= 0 || N % 64 != 0) {
    set_error("%s: shape M=%d K=%d N=%d outside the envelope (M >= 0, K %% 128 == 0, K <= 65536, N %% 64 == 0)", fn, M,
              K, N);
    return -2;
  }
  if (dtype != B2Q_DTYPE_F16 && dtype != B2Q_DTYPE_BF16) {
    set_error("%s: dtype=%d not supported (0 fp16, 1 bf16)", fn, dtype);
    return -2;
  }
  return 0;
}

static int fp8blk_check_layer(const char* fn, const void* weight, const float* s_w, const void* out) {
  if (weight == nullptr || s_w == nullptr || out == nullptr) {
    set_error("%s: null pointer argument", fn);
    return -2;
  }
  if (!aligned16(weight) || !aligned16(s_w) || !aligned16(out)) {
    set_error("%s: weight, s_w and out must be 16-byte aligned", fn);
    return -2;
  }
  return 0;
}

int b2q_fp8blk_quantize(const void* x, void* codes, float* s_x, int M, int K, int dtype, void* stream) {
  if (int e = fp8blk_check_shape("b2q_fp8blk_quantize", M, K, 64, dtype)) return e;
  if (M == 0) return 0;
  if (x == nullptr || codes == nullptr || s_x == nullptr || !aligned16(x) || !aligned16(codes) || !aligned16(s_x)) {
    set_error("b2q_fp8blk_quantize: x, codes and s_x must be 16-byte aligned device pointers");
    return -2;
  }
  DeviceGuard dg(codes);
  return check_cuda(launch_fp8blk_quant(x, codes, s_x, M, K, dtype, (cudaStream_t)stream), "b2q_fp8blk_quantize");
}

int b2q_fp8blk_mm(const void* codes, const float* s_x, const void* weight, const float* s_w, const void* bias,
                  void* out, int M, int K, int N, int dtype, int ks, void* stream) {
  if (int e = fp8blk_check_shape("b2q_fp8blk_mm", M, K, N, dtype)) return e;
  if (int e = fp8blk_check_layer("b2q_fp8blk_mm", weight, s_w, out)) return e;
  if (ks > 8) {
    set_error("b2q_fp8blk_mm: ks=%d exceeds the cluster limit 8", ks);
    return -2;
  }
  if (M == 0) return 0;
  if (codes == nullptr || s_x == nullptr || !aligned16(codes) || !aligned16(s_x)) {
    set_error("b2q_fp8blk_mm: codes and s_x must be 16-byte aligned device pointers");
    return -2;
  }
  DeviceGuard dg(weight);
  Fp8BlkArgs a = {nullptr, codes, s_x, weight, s_w, bias, out, M, K, N, dtype, ks, (cudaStream_t)stream};
  return check_cuda(launch_fp8blk_gemm(a), "b2q_fp8blk_mm");
}

int b2q_fp8blk_forward(const void* x, const void* weight, const float* s_w, const void* bias, void* out, int M, int K,
                       int N, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  if (int e = fp8blk_check_shape("b2q_fp8blk_forward", M, K, N, dtype)) return e;
  if (int e = fp8blk_check_layer("b2q_fp8blk_forward", weight, s_w, out)) return e;
  if (M == 0) return 0;
  const size_t need = b2q_fp8blk_workspace_bytes(M, K);
  if (x == nullptr || !aligned16(x) || (need > 0 && (workspace == nullptr || !aligned16(workspace) ||
                                                     workspace_bytes < need))) {
    set_error("b2q_fp8blk_forward: x and a workspace of b2q_fp8blk_workspace_bytes(M, K) = %zu bytes (16-byte "
              "aligned) must be given, got %zu", need, workspace_bytes);
    return -2;
  }
  DeviceGuard dg(weight);
  Fp8BlkArgs a = {x, nullptr, nullptr, weight, s_w, bias, out, M, K, N, dtype, 0, (cudaStream_t)stream};
  if (M <= 8) return check_cuda(launch_fp8blk_gemm(a), "b2q_fp8blk_forward(fused)");
  uint8_t* codes = reinterpret_cast<uint8_t*>(workspace);
  float* s_x = reinterpret_cast<float*>(codes + fp8blk_codes_bytes(M, K));
  int e = check_cuda(launch_fp8blk_quant(x, codes, s_x, M, K, dtype, (cudaStream_t)stream), "b2q_fp8blk_forward");
  if (e != 0) return e;
  a.x = nullptr;
  a.codes = codes;
  a.s_x = s_x;
  return check_cuda(launch_fp8blk_gemm(a), "b2q_fp8blk_forward");
}

// ---- per-channel / per-tensor FP8 (compressed-tensors FP8 / FP8_DYNAMIC, fbgemm_fp8; W8A8) tier ----
size_t b2q_fp8ch_workspace_bytes(int M, int K) {
  if (M <= 0 || K <= 0 || K % 128 != 0) return 0;
  return fp8blk_codes_bytes(M, K) + ((size_t)M * 4 + 15) / 16 * 16;
}

static int fp8ch_check_ub(const char* fn, float ub) {
  if (!(ub > 0.f)) {  // NaN fails too; +inf: no bound
    set_error("%s: ub=%g must be positive (+inf: no bound)", fn, (double)ub);
    return -2;
  }
  return 0;
}

int b2q_fp8ch_quantize(const void* x, void* codes, float* s_x, int M, int K, float ub, int dtype, void* stream) {
  if (int e = fp8blk_check_shape("b2q_fp8ch_quantize", M, K, 64, dtype)) return e;
  if (int e = fp8ch_check_ub("b2q_fp8ch_quantize", ub)) return e;
  if (M == 0) return 0;
  if (x == nullptr || codes == nullptr || s_x == nullptr || !aligned16(x) || !aligned16(codes) || !aligned16(s_x)) {
    set_error("b2q_fp8ch_quantize: x, codes and s_x must be 16-byte aligned device pointers");
    return -2;
  }
  DeviceGuard dg(codes);
  return check_cuda(launch_fp8ch_quant(x, codes, s_x, M, K, ub, dtype, (cudaStream_t)stream), "b2q_fp8ch_quantize");
}

int b2q_fp8ch_quantize_static(const void* x, const float* s_in, void* codes, float* s_x, int M, int K, int dtype,
                              void* stream) {
  if (int e = fp8blk_check_shape("b2q_fp8ch_quantize_static", M, K, 64, dtype)) return e;
  if (M == 0) return 0;
  if (x == nullptr || s_in == nullptr || codes == nullptr || s_x == nullptr || !aligned16(x) || !aligned16(codes) ||
      !aligned16(s_x)) {
    set_error("b2q_fp8ch_quantize_static: x, s_in, codes and s_x must be device pointers, x, codes and s_x 16-byte "
              "aligned");
    return -2;
  }
  DeviceGuard dg(codes);
  return check_cuda(launch_fp8ch_static_quant(x, s_in, codes, s_x, M, K, dtype, (cudaStream_t)stream),
                    "b2q_fp8ch_quantize_static");
}

int b2q_fp8ch_mm(const void* codes, const float* s_x, const void* weight, const float* s_w, const void* bias, void* out,
                 int M, int K, int N, int dtype, int ks, void* stream) {
  if (int e = fp8blk_check_shape("b2q_fp8ch_mm", M, K, N, dtype)) return e;
  if (int e = fp8blk_check_layer("b2q_fp8ch_mm", weight, s_w, out)) return e;
  if (ks > 8) {
    set_error("b2q_fp8ch_mm: ks=%d exceeds the cluster limit 8", ks);
    return -2;
  }
  if (M == 0) return 0;
  if (codes == nullptr || s_x == nullptr || !aligned16(codes)) {
    set_error("b2q_fp8ch_mm: codes (16-byte aligned) and s_x must be device pointers");
    return -2;
  }
  DeviceGuard dg(weight);
  Fp8ChArgs a = {nullptr, codes, s_x, nullptr, weight, s_w, bias, out, M, K, N, dtype, ks, (cudaStream_t)stream};
  return check_cuda(launch_fp8ch_gemm(a), "b2q_fp8ch_mm");
}

int b2q_fp8ch_forward(const void* x, const void* weight, const float* s_w, const float* s_in, float ub,
                      const void* bias, void* out, int M, int K, int N, int dtype, void* workspace,
                      size_t workspace_bytes, void* stream) {
  if (int e = fp8blk_check_shape("b2q_fp8ch_forward", M, K, N, dtype)) return e;
  if (int e = fp8blk_check_layer("b2q_fp8ch_forward", weight, s_w, out)) return e;
  if (s_in == nullptr) {
    if (int e = fp8ch_check_ub("b2q_fp8ch_forward", ub)) return e;
  }
  if (M == 0) return 0;
  const bool fused = M <= 8 && s_in != nullptr;  // static-scale decode quantises inside the GEMM
  const size_t need = fused ? 0 : b2q_fp8ch_workspace_bytes(M, K);
  if (x == nullptr || !aligned16(x) || (need > 0 && (workspace == nullptr || !aligned16(workspace) ||
                                                     workspace_bytes < need))) {
    set_error("b2q_fp8ch_forward: x and a workspace of b2q_fp8ch_workspace_bytes(M, K) = %zu bytes (16-byte "
              "aligned) must be given, got %zu", need, workspace_bytes);
    return -2;
  }
  DeviceGuard dg(weight);
  Fp8ChArgs a = {x, nullptr, nullptr, s_in, weight, s_w, bias, out, M, K, N, dtype, 0, (cudaStream_t)stream};
  if (fused) return check_cuda(launch_fp8ch_gemm(a), "b2q_fp8ch_forward(fused)");
  uint8_t* codes = reinterpret_cast<uint8_t*>(workspace);
  float* s_x = reinterpret_cast<float*>(codes + fp8blk_codes_bytes(M, K));
  int e = s_in != nullptr ? launch_fp8ch_static_quant(x, s_in, codes, s_x, M, K, dtype, (cudaStream_t)stream)
                          : launch_fp8ch_quant(x, codes, s_x, M, K, ub, dtype, (cudaStream_t)stream);
  if ((e = check_cuda(e, "b2q_fp8ch_forward")) != 0) return e;
  a.x = nullptr;
  a.codes = codes;
  a.s_x = s_x;
  return check_cuda(launch_fp8ch_gemm(a), "b2q_fp8ch_forward");
}

// ---- per-channel / per-tensor INT8 (compressed-tensors int-quantized W8A8) tier: the GEMM of b2q_fp8ch on s8 ----
size_t b2q_int8ch_workspace_bytes(int M, int K) { return b2q_fp8ch_workspace_bytes(M, K); }

int b2q_int8ch_quantize(const void* x, void* codes, float* s_x, int M, int K, int dtype, void* stream) {
  if (int e = fp8blk_check_shape("b2q_int8ch_quantize", M, K, 64, dtype)) return e;
  if (M == 0) return 0;
  if (x == nullptr || codes == nullptr || s_x == nullptr || !aligned16(x) || !aligned16(codes) || !aligned16(s_x)) {
    set_error("b2q_int8ch_quantize: x, codes and s_x must be 16-byte aligned device pointers");
    return -2;
  }
  DeviceGuard dg(codes);
  return check_cuda(launch_int8ch_quant(x, codes, s_x, M, K, dtype, (cudaStream_t)stream), "b2q_int8ch_quantize");
}

int b2q_int8ch_quantize_static(const void* x, const float* s_in, void* codes, float* s_x, int M, int K, int dtype,
                               void* stream) {
  if (int e = fp8blk_check_shape("b2q_int8ch_quantize_static", M, K, 64, dtype)) return e;
  if (M == 0) return 0;
  if (x == nullptr || s_in == nullptr || codes == nullptr || s_x == nullptr || !aligned16(x) || !aligned16(codes) ||
      !aligned16(s_x)) {
    set_error("b2q_int8ch_quantize_static: x, s_in, codes and s_x must be device pointers, x, codes and s_x 16-byte "
              "aligned");
    return -2;
  }
  DeviceGuard dg(codes);
  return check_cuda(launch_int8ch_static_quant(x, s_in, codes, s_x, M, K, dtype, (cudaStream_t)stream),
                    "b2q_int8ch_quantize_static");
}

int b2q_int8ch_mm(const void* codes, const float* s_x, const void* weight, const float* s_w, const void* bias, void* out,
                  int M, int K, int N, int dtype, int ks, void* stream) {
  if (int e = fp8blk_check_shape("b2q_int8ch_mm", M, K, N, dtype)) return e;
  if (int e = fp8blk_check_layer("b2q_int8ch_mm", weight, s_w, out)) return e;
  if (ks > 8) {
    set_error("b2q_int8ch_mm: ks=%d exceeds the cluster limit 8", ks);
    return -2;
  }
  if (M == 0) return 0;
  if (codes == nullptr || s_x == nullptr || !aligned16(codes)) {
    set_error("b2q_int8ch_mm: codes (16-byte aligned) and s_x must be device pointers");
    return -2;
  }
  DeviceGuard dg(weight);
  Fp8ChArgs a = {nullptr, codes, s_x, nullptr, weight, s_w, bias, out, M, K, N, dtype, ks, (cudaStream_t)stream};
  return check_cuda(launch_int8ch_gemm(a), "b2q_int8ch_mm");
}

int b2q_int8ch_forward(const void* x, const void* weight, const float* s_w, const float* s_in, const void* bias,
                       void* out, int M, int K, int N, int dtype, void* workspace, size_t workspace_bytes,
                       void* stream) {
  if (int e = fp8blk_check_shape("b2q_int8ch_forward", M, K, N, dtype)) return e;
  if (int e = fp8blk_check_layer("b2q_int8ch_forward", weight, s_w, out)) return e;
  if (M == 0) return 0;
  const size_t need = b2q_int8ch_workspace_bytes(M, K);
  if (x == nullptr || !aligned16(x) || workspace == nullptr || !aligned16(workspace) || workspace_bytes < need) {
    set_error("b2q_int8ch_forward: x and a workspace of b2q_int8ch_workspace_bytes(M, K) = %zu bytes (16-byte "
              "aligned) must be given, got %zu", need, workspace_bytes);
    return -2;
  }
  DeviceGuard dg(weight);
  int8_t* codes = reinterpret_cast<int8_t*>(workspace);
  float* s_x = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + fp8blk_codes_bytes(M, K));
  int e = s_in != nullptr ? launch_int8ch_static_quant(x, s_in, codes, s_x, M, K, dtype, (cudaStream_t)stream)
                          : launch_int8ch_quant(x, codes, s_x, M, K, dtype, (cudaStream_t)stream);
  if ((e = check_cuda(e, "b2q_int8ch_forward")) != 0) return e;
  Fp8ChArgs a = {nullptr, codes, s_x, nullptr, weight, s_w, bias, out, M, K, N, dtype, 0, (cudaStream_t)stream};
  return check_cuda(launch_int8ch_gemm(a), "b2q_int8ch_forward");
}

// ---- W4AFP8 (compressed-tensors W4AFP8: 4-bit group-128 weights, dynamic per-token e4m3 activations) tier ----
static int w4afp8_check_shape(const char* fn, int M, int K, int N, int dtype) {
  if (M < 0 || K <= 0 || K % 128 != 0 || K > 65536 || N <= 0 || N % 128 != 0) {
    set_error("%s: shape M=%d K=%d N=%d outside the envelope (M >= 0, K %% 128 == 0, K <= 65536, N %% 128 == 0)", fn,
              M, K, N);
    return -2;
  }
  if (dtype != B2Q_DTYPE_F16 && dtype != B2Q_DTYPE_BF16) {
    set_error("%s: dtype=%d not supported (0 fp16, 1 bf16)", fn, dtype);
    return -2;
  }
  return 0;
}

static int w4afp8_check_layer(const char* fn, const void* packed, const float* s_w, const void* out) {
  if (packed == nullptr || s_w == nullptr || out == nullptr) {
    set_error("%s: null pointer argument", fn);
    return -2;
  }
  if (!aligned16(packed) || !aligned16(s_w) || !aligned16(out)) {
    set_error("%s: packed, s_w and out must be 16-byte aligned", fn);
    return -2;
  }
  return 0;
}

size_t b2q_w4afp8_packed_bytes(int K, int N) {
  if (K <= 0 || K % 128 != 0 || K > 65536 || N <= 0 || N % 128 != 0) return 0;
  return (size_t)K * N / 2;
}

size_t b2q_w4afp8_workspace_bytes(int M, int K) { return b2q_fp8ch_workspace_bytes(M, K); }

int b2q_w4afp8_prepack(const int32_t* weight_packed, void* packed, int K, int N, void* stream) {
  if (int e = w4afp8_check_shape("b2q_w4afp8_prepack", 0, K, N, B2Q_DTYPE_F16)) return e;
  if (weight_packed == nullptr || packed == nullptr || !aligned16(packed)) {
    set_error("b2q_w4afp8_prepack: weight_packed and packed (16-byte aligned) must be device pointers");
    return -2;
  }
  DeviceGuard dg(packed);
  return check_cuda(launch_w4afp8_prepack(weight_packed, packed, K, N, (cudaStream_t)stream), "b2q_w4afp8_prepack");
}

int b2q_w4afp8_mm(const void* codes, const float* s_x, const void* packed, const float* s_w, const void* bias,
                  void* out, int M, int K, int N, int dtype, int ks, void* stream) {
  if (int e = w4afp8_check_shape("b2q_w4afp8_mm", M, K, N, dtype)) return e;
  if (int e = w4afp8_check_layer("b2q_w4afp8_mm", packed, s_w, out)) return e;
  if (ks > 8) {
    set_error("b2q_w4afp8_mm: ks=%d exceeds the cluster limit 8", ks);
    return -2;
  }
  if (M == 0) return 0;
  if (codes == nullptr || s_x == nullptr || !aligned16(codes)) {
    set_error("b2q_w4afp8_mm: codes (16-byte aligned) and s_x must be device pointers");
    return -2;
  }
  DeviceGuard dg(packed);
  W4Fp8Args a = {codes, s_x, packed, s_w, bias, out, M, K, N, dtype, ks, (cudaStream_t)stream};
  return check_cuda(launch_w4afp8_gemm(a), "b2q_w4afp8_mm");
}

int b2q_w4afp8_forward(const void* x, const void* packed, const float* s_w, const void* bias, void* out, int M, int K,
                       int N, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  if (int e = w4afp8_check_shape("b2q_w4afp8_forward", M, K, N, dtype)) return e;
  if (int e = w4afp8_check_layer("b2q_w4afp8_forward", packed, s_w, out)) return e;
  if (M == 0) return 0;
  const size_t need = b2q_w4afp8_workspace_bytes(M, K);
  if (x == nullptr || !aligned16(x) || workspace == nullptr || !aligned16(workspace) || workspace_bytes < need) {
    set_error("b2q_w4afp8_forward: x and a workspace of b2q_w4afp8_workspace_bytes(M, K) = %zu bytes (16-byte "
              "aligned) must be given, got %zu", need, workspace_bytes);
    return -2;
  }
  DeviceGuard dg(packed);
  uint8_t* codes = reinterpret_cast<uint8_t*>(workspace);
  float* s_x = reinterpret_cast<float*>(codes + fp8blk_codes_bytes(M, K));
  int e = check_cuda(launch_fp8ch_quant(x, codes, s_x, M, K, INFINITY, dtype, (cudaStream_t)stream),
                     "b2q_w4afp8_forward");
  if (e != 0) return e;
  W4Fp8Args a = {codes, s_x, packed, s_w, bias, out, M, K, N, dtype, 0, (cudaStream_t)stream};
  return check_cuda(launch_w4afp8_gemm(a), "b2q_w4afp8_forward");
}

// ---- block-FP8 MoE experts: the grouped modes of fp8blk_gemm_kernel over the routing tables of b2q_moe_align ----
static int fp8blk_moe_check(const char* fn, const void* codes, const float* s_x, const void* w, const float* s_w,
                            const void* out, const int32_t* counts, const int32_t* offsets, int E, int rows, int K, int N,
                            int dtype, int ks) {
  if (int e = fp8blk_check_shape(fn, rows, K, N, dtype)) return e;
  if (int e = fp8blk_check_layer(fn, w, s_w, out)) return e;
  if (codes == nullptr || s_x == nullptr || counts == nullptr || offsets == nullptr || !aligned16(codes) ||
      !aligned16(s_x)) {
    set_error("%s: codes, s_x, counts and offsets must be device pointers, codes and s_x 16-byte aligned", fn);
    return -2;
  }
  if (E < 1 || E > 256 || rows < 1 || ks > 8) {
    set_error("%s: E=%d (1..256), rows=%d (>= 1), ks=%d (<= 8) outside the envelope", fn, E, rows, ks);
    return -2;
  }
  return 0;
}

int b2q_fp8blk_moe_gather(const void* x, const int32_t* sorted_pairs, void* codes, float* s_x, int T, int top_k, int K,
                          int dtype, void* stream) {
  if (T < 1 || top_k < 1) {
    set_error("b2q_fp8blk_moe_gather: T=%d, top_k=%d must be >= 1", T, top_k);
    return -2;
  }
  if (int e = fp8blk_check_shape("b2q_fp8blk_moe_gather", T * top_k, K, 64, dtype)) return e;
  if (x == nullptr || sorted_pairs == nullptr || codes == nullptr || s_x == nullptr || !aligned16(x) ||
      !aligned16(codes) || !aligned16(s_x)) {
    set_error("b2q_fp8blk_moe_gather: x, sorted_pairs, codes and s_x must be device pointers, x, codes and s_x 16-byte "
              "aligned");
    return -2;
  }
  DeviceGuard dg(codes);
  return check_cuda(launch_fp8blk_moe_gather(x, sorted_pairs, codes, s_x, T * top_k, top_k, K, dtype,
                                             (cudaStream_t)stream),
                    "b2q_fp8blk_moe_gather");
}

int b2q_fp8blk_moe_gate_up(const void* codes, const float* s_x, const void* w1, const float* s_w1, const void* w3,
                           const float* s_w3, void* h, const int32_t* counts, const int32_t* offsets, int E, int rows,
                           int active, int K, int N, int dtype, int ks, void* stream) {
  if (int e = fp8blk_moe_check("b2q_fp8blk_moe_gate_up", codes, s_x, w1, s_w1, h, counts, offsets, E, rows, K, N, dtype,
                               ks))
    return e;
  if (int e = fp8blk_check_layer("b2q_fp8blk_moe_gate_up", w3, s_w3, h)) return e;
  DeviceGuard dg(w1);
  Fp8BlkArgs a = {nullptr, codes, s_x, w1, s_w1, nullptr, h, rows, K, N, dtype, ks, (cudaStream_t)stream};
  Fp8BlkMoe g = {};
  g.counts = counts;
  g.offsets = offsets;
  g.w3 = w3;
  g.s_w3 = s_w3;
  g.E = E;
  g.active = active;
  return check_cuda(launch_fp8blk_moe(1, a, g), "b2q_fp8blk_moe_gate_up");
}

int b2q_fp8blk_moe_down(const void* codes_h, const float* s_h, const void* w2, const float* s_w2, const int32_t* counts,
                        const int32_t* offsets, const int32_t* sorted_pairs, const float* pair_weights, float* ypair,
                        int E, int rows, int active, int K, int N, int dtype, int ks, void* stream) {
  if (int e = fp8blk_moe_check("b2q_fp8blk_moe_down", codes_h, s_h, w2, s_w2, ypair, counts, offsets, E, rows, K, N,
                               dtype, ks))
    return e;
  if (sorted_pairs == nullptr || pair_weights == nullptr) {
    set_error("b2q_fp8blk_moe_down: sorted_pairs and pair_weights must be device pointers");
    return -2;
  }
  DeviceGuard dg(w2);
  Fp8BlkArgs a = {nullptr, codes_h, s_h, w2, s_w2, nullptr, ypair, rows, K, N, dtype, ks, (cudaStream_t)stream};
  Fp8BlkMoe g = {};
  g.counts = counts;
  g.offsets = offsets;
  g.sorted_pairs = sorted_pairs;
  g.pair_weights = pair_weights;
  g.ypair = ypair;
  g.E = E;
  g.active = active;
  return check_cuda(launch_fp8blk_moe(2, a, g), "b2q_fp8blk_moe_down");
}

// ---- per-channel W8A8 MoE experts (FP8 and INT8): the grouped modes of the b2q_fp8ch GEMM over b2q_moe_align's tables ----
static int ch_moe_gather(const char* fn, int s8, const void* x, const int32_t* sorted_pairs, const int32_t* offsets,
                         const float* s_in, int E, void* codes, float* s_x, int T, int top_k, int K, float ub, int dtype,
                         void* stream) {
  if (T < 1 || top_k < 1) {
    set_error("%s: T=%d, top_k=%d must be >= 1", fn, T, top_k);
    return -2;
  }
  if (int e = fp8blk_check_shape(fn, T * top_k, K, 64, dtype)) return e;
  if (!s8 && s_in == nullptr) {
    if (int e = fp8ch_check_ub(fn, ub)) return e;
  }
  if (x == nullptr || codes == nullptr || s_x == nullptr || !aligned16(x) || !aligned16(codes) || !aligned16(s_x)) {
    set_error("%s: x, codes and s_x must be 16-byte aligned device pointers", fn);
    return -2;
  }
  if (s_in != nullptr && (offsets == nullptr || E < 1 || E > 256)) {
    set_error("%s: static scales need the offsets of b2q_moe_align and E=%d in 1..256", fn, E);
    return -2;
  }
  DeviceGuard dg(codes);
  return check_cuda(launch_ch_moe_gather(s8, x, sorted_pairs, offsets, s_in, E, codes, s_x, T * top_k, top_k, K, ub,
                                         dtype, (cudaStream_t)stream),
                    fn);
}

static int ch_moe_gate_up(const char* fn, int s8, const void* codes, const float* s_x, const void* w1,
                          const float* s_w1, const void* w3, const float* s_w3, void* h, const int32_t* counts,
                          const int32_t* offsets, int E, int rows, int active, int K, int N, int dtype, int ks,
                          void* stream) {
  if (int e = fp8blk_moe_check(fn, codes, s_x, w1, s_w1, h, counts, offsets, E, rows, K, N, dtype, ks)) return e;
  if (int e = fp8blk_check_layer(fn, w3, s_w3, h)) return e;
  DeviceGuard dg(w1);
  Fp8ChArgs a = {nullptr, codes, s_x, nullptr, w1, s_w1, nullptr, h, rows, K, N, dtype, ks, (cudaStream_t)stream};
  Fp8ChMoe g = {};
  g.counts = counts;
  g.offsets = offsets;
  g.w3 = w3;
  g.s_w3 = s_w3;
  g.E = E;
  g.active = active;
  return check_cuda(launch_ch_moe(1, s8, a, g), fn);
}

static int ch_moe_down(const char* fn, int s8, const void* codes_h, const float* s_h, const void* w2, const float* s_w2,
                       const int32_t* counts, const int32_t* offsets, const int32_t* sorted_pairs,
                       const float* pair_weights, float* ypair, int E, int rows, int active, int K, int N, int dtype,
                       int ks, void* stream) {
  if (int e = fp8blk_moe_check(fn, codes_h, s_h, w2, s_w2, ypair, counts, offsets, E, rows, K, N, dtype, ks)) return e;
  if (sorted_pairs == nullptr || pair_weights == nullptr) {
    set_error("%s: sorted_pairs and pair_weights must be device pointers", fn);
    return -2;
  }
  DeviceGuard dg(w2);
  Fp8ChArgs a = {nullptr, codes_h, s_h, nullptr, w2, s_w2, nullptr, ypair, rows, K, N, dtype, ks, (cudaStream_t)stream};
  Fp8ChMoe g = {};
  g.counts = counts;
  g.offsets = offsets;
  g.sorted_pairs = sorted_pairs;
  g.pair_weights = pair_weights;
  g.ypair = ypair;
  g.E = E;
  g.active = active;
  return check_cuda(launch_ch_moe(2, s8, a, g), fn);
}

int b2q_fp8ch_moe_gather(const void* x, const int32_t* sorted_pairs, const int32_t* offsets, const float* s_in, int E,
                         void* codes, float* s_x, int T, int top_k, int K, float ub, int dtype, void* stream) {
  return ch_moe_gather("b2q_fp8ch_moe_gather", 0, x, sorted_pairs, offsets, s_in, E, codes, s_x, T, top_k, K, ub, dtype,
                       stream);
}

int b2q_fp8ch_moe_gate_up(const void* codes, const float* s_x, const void* w1, const float* s_w1, const void* w3,
                          const float* s_w3, void* h, const int32_t* counts, const int32_t* offsets, int E, int rows,
                          int active, int K, int N, int dtype, int ks, void* stream) {
  return ch_moe_gate_up("b2q_fp8ch_moe_gate_up", 0, codes, s_x, w1, s_w1, w3, s_w3, h, counts, offsets, E, rows, active,
                        K, N, dtype, ks, stream);
}

int b2q_fp8ch_moe_down(const void* codes_h, const float* s_h, const void* w2, const float* s_w2, const int32_t* counts,
                       const int32_t* offsets, const int32_t* sorted_pairs, const float* pair_weights, float* ypair,
                       int E, int rows, int active, int K, int N, int dtype, int ks, void* stream) {
  return ch_moe_down("b2q_fp8ch_moe_down", 0, codes_h, s_h, w2, s_w2, counts, offsets, sorted_pairs, pair_weights, ypair,
                     E, rows, active, K, N, dtype, ks, stream);
}

int b2q_int8ch_moe_gather(const void* x, const int32_t* sorted_pairs, const int32_t* offsets, const float* s_in, int E,
                          void* codes, float* s_x, int T, int top_k, int K, int dtype, void* stream) {
  return ch_moe_gather("b2q_int8ch_moe_gather", 1, x, sorted_pairs, offsets, s_in, E, codes, s_x, T, top_k, K, 0.f,
                       dtype, stream);
}

int b2q_int8ch_moe_gate_up(const void* codes, const float* s_x, const void* w1, const float* s_w1, const void* w3,
                           const float* s_w3, void* h, const int32_t* counts, const int32_t* offsets, int E, int rows,
                           int active, int K, int N, int dtype, int ks, void* stream) {
  return ch_moe_gate_up("b2q_int8ch_moe_gate_up", 1, codes, s_x, w1, s_w1, w3, s_w3, h, counts, offsets, E, rows,
                        active, K, N, dtype, ks, stream);
}

int b2q_int8ch_moe_down(const void* codes_h, const float* s_h, const void* w2, const float* s_w2, const int32_t* counts,
                        const int32_t* offsets, const int32_t* sorted_pairs, const float* pair_weights, float* ypair,
                        int E, int rows, int active, int K, int N, int dtype, int ks, void* stream) {
  return ch_moe_down("b2q_int8ch_moe_down", 1, codes_h, s_h, w2, s_w2, counts, offsets, sorted_pairs, pair_weights,
                     ypair, E, rows, active, K, N, dtype, ks, stream);
}

int b2q_gemv(const void* x, const void* packed, const void* scales, const int32_t* qzeros, const int32_t* perm,
             const void* bias, void* out, int K, int N, int bits, int group_size, int dtype, int ks, int warps,
             void* stream) {
  int v = validate("b2q_gemv", x, packed, scales, out, 1, K, N, bits, group_size, dtype);
  if (v != 0) return v;
  DeviceGuard dg(packed);
  v = check_tune("b2q_gemv", ks, warps);
  if (v != 0) return v;
  MmArgs a = make_args(x, packed, scales, qzeros, perm, bias, out, 1, K, N, bits, group_size, dtype, nullptr, 0,
                       stream);
  a.tune_ks = ks;
  a.tune_warps = warps;
  if (decode_supported(a)) return check_cuda(launch_decode(a), "b2q_gemv(decode)");
  if (gemv_supported(a)) return check_cuda(launch_gemv(a), "b2q_gemv");
  set_error("b2q_gemv: no M=1 tier for bits=%d K=%d group_size=%d (use b2q_mm)", bits, K, group_size);
  return -2;
}

int b2q_decode(const void* x, const void* packed, const void* scales, const int32_t* qzeros, const int32_t* perm,
               const void* bias, void* out, int M, int K, int N, int bits, int group_size, int dtype, int ks,
               int warps, void* stream) {
  int v = validate("b2q_decode", x, packed, scales, out, M, K, N, bits, group_size, dtype);
  if (v != 0) return v;
  DeviceGuard dg(packed);
  v = check_tune("b2q_decode", ks, warps);
  if (v != 0) return v;
  MmArgs a = make_args(x, packed, scales, qzeros, perm, bias, out, M, K, N, bits, group_size, dtype, nullptr, 0,
                       stream);
  a.tune_ks = ks;
  a.tune_warps = warps;
  if (!decode_supported(a)) {
    set_error("b2q_decode: needs bits=4, 1 <= M <= 8, K %% 128 == 0, group_size 64|128|K (got bits=%d M=%d K=%d g=%d)",
              bits, M, K, group_size);
    return -2;
  }
  return check_cuda(launch_decode(a), "b2q_decode");
}

int b2q_decode_multi(const void* x, int nsets, const void* const* packed, const void* const* scales,
                     const int32_t* const* qzeros, const int32_t* perm, const void* const* bias, void* const* out,
                     const int* N, int M, int K, int bits, int group_size, int dtype, void* stream) {
  if (x == nullptr || packed == nullptr || scales == nullptr || qzeros == nullptr || bias == nullptr ||
      out == nullptr || N == nullptr || nsets < 1) {
    set_error("b2q_decode_multi: null pointer argument");
    return -2;
  }
  int v = validate("b2q_decode_multi", x, packed[0], scales[0], out[0], M, K, N[0], bits, group_size, dtype);
  if (v != 0) return v;
  DeviceGuard dg(packed[0]);
  MmArgs a = make_args(x, packed[0], scales[0], qzeros[0], perm, bias[0], out[0], M, K, N[0], bits, group_size,
                       dtype, nullptr, 0, stream);
  return check_cuda(launch_decode_multi(a, nsets, packed, scales, qzeros, bias, out, N), "b2q_decode_multi");
}

int b2q_gemm_multi(const void* x, int nsets, const void* const* packed, const void* const* scales,
                   const int32_t* const* qzeros, const int32_t* perm, const void* const* bias, void* const* out,
                   const int* N, int M, int K, int bits, int group_size, int dtype, void* workspace,
                   size_t workspace_bytes, void* stream) {
  if (x == nullptr || packed == nullptr || scales == nullptr || qzeros == nullptr || bias == nullptr ||
      out == nullptr || N == nullptr) {
    set_error("b2q_gemm_multi: null pointer argument");
    return -2;
  }
  if (nsets < 1 || nsets > G_MAX_SETS) {
    set_error("b2q_gemm_multi: nsets=%d out of range (1..%d)", nsets, G_MAX_SETS);
    return -2;
  }
  int v = validate("b2q_gemm_multi", x, packed[0], scales[0], out[0], M, K, N[0], bits, group_size, dtype);
  if (v != 0) return v;
  if (bits != 4 || M <= 128) {
    set_error("b2q_gemm_multi: the fused prefill launch serves bits=4, M > 128 (got bits=%d M=%d)", bits, M);
    return -2;
  }
  for (int i = 1; i < nsets; ++i) {
    if (N[i] <= 0 || N[i] % 32 != 0 || packed[i] == nullptr || scales[i] == nullptr || out[i] == nullptr ||
        ((qzeros[i] != nullptr) != (qzeros[0] != nullptr)) || (reinterpret_cast<uintptr_t>(packed[i]) & 15) ||
        (reinterpret_cast<uintptr_t>(out[i]) & 15)) {
      set_error("b2q_gemm_multi: set %d unsupported (N=%d; all sets share K, group size and symmetry, packed and out "
                "16-byte aligned)", i, N[i]);
      return -2;
    }
  }
  DeviceGuard dg(packed[0]);
  MmArgs a = make_args(x, packed[0], scales[0], qzeros[0], perm, bias[0], out[0], M, K, N[0], bits, group_size, dtype,
                       workspace, workspace_bytes, stream);
  const void* xa = x;
  if (perm != nullptr) {  // act-order siblings share g_idx: ONE gather of x serves all sets
    const size_t need = (size_t)M * K * 2;
    if (workspace == nullptr || workspace_bytes < need) {
      set_error("b2q_gemm_multi: act-order needs a %zu-byte workspace (got %zu)", need, workspace_bytes);
      return -2;
    }
    int e = check_cuda(launch_permute_cols(x, perm, workspace, M, K, (cudaStream_t)stream), "b2q_gemm_multi(permute)");
    if (e != 0) return e;
    xa = workspace;
  }
  return check_cuda(launch_gemm_multi(a, xa, nsets, packed, scales, qzeros, bias, out, N), "b2q_gemm_multi");
}

int b2q_gemm(const void* x, const void* packed, const void* scales, const int32_t* qzeros, const int32_t* perm,
             const void* bias, void* out, int M, int K, int N, int bits, int group_size, int dtype, void* workspace,
             size_t workspace_bytes, void* stream) {
  int v = validate("b2q_gemm", x, packed, scales, out, M, K, N, bits, group_size, dtype);
  if (v != 0) return v;
  DeviceGuard dg(packed);
  if (M == 0) return 0;
  MmArgs a = make_args(x, packed, scales, qzeros, perm, bias, out, M, K, N, bits, group_size, dtype, workspace,
                       workspace_bytes, stream);
  return check_cuda(launch_gemm(a), "b2q_gemm");
}

int b2q_mm(const void* x, const void* packed, const void* scales, const int32_t* qzeros, const int32_t* perm,
           const void* bias, void* out, int M, int K, int N, int bits, int group_size, int dtype, void* workspace,
           size_t workspace_bytes, void* stream) {
  int v = validate("b2q_mm", x, packed, scales, out, M, K, N, bits, group_size, dtype);
  if (v != 0) return v;
  DeviceGuard dg(packed);
  if (M == 0) return 0;
  MmArgs a = make_args(x, packed, scales, qzeros, perm, bias, out, M, K, N, bits, group_size, dtype, workspace,
                       workspace_bytes, stream);
  if (decode_supported(a)) return check_cuda(launch_decode(a), "b2q_mm(decode)");
  if (gemv_supported(a)) return check_cuda(launch_gemv(a), "b2q_mm(gemv)");
  return check_cuda(launch_gemm(a), "b2q_mm(gemm)");
}

// ---- grouped MoE expert path (b2q_moe.cu + the grouped modes of b2q_midm.cu) -----------------------------------------
int b2q_moe_align(const int32_t* topk_ids, int T, int top_k, int E, int32_t* counts, int32_t* offsets,
                  int32_t* sorted_pairs, void* stream) {
  if (topk_ids == nullptr || counts == nullptr || offsets == nullptr || sorted_pairs == nullptr || T < 1 || top_k < 1 ||
      E < 1) {
    set_error("b2q_moe_align: bad argument (T=%d top_k=%d E=%d)", T, top_k, E);
    return -2;
  }
  DeviceGuard dg(counts);
  return check_cuda(launch_moe_align(topk_ids, T, top_k, E, counts, offsets, sorted_pairs, (cudaStream_t)stream),
                    "b2q_moe_align");
}

int b2q_moe_gather(const void* x, const int32_t* sorted_pairs, void* xs, int rows, int top_k, int K, void* stream) {
  if (x == nullptr || sorted_pairs == nullptr || xs == nullptr || rows < 1 || top_k < 1 || K < 8 || K % 8 != 0 ||
      (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(xs) & 15)) {
    set_error("b2q_moe_gather: bad argument (rows=%d top_k=%d K=%d; K %% 8 == 0, 16-byte aligned)", rows, top_k, K);
    return -2;
  }
  DeviceGuard dg(xs);
  return check_cuda(launch_moe_gather(x, sorted_pairs, xs, rows, top_k, K, (cudaStream_t)stream), "b2q_moe_gather");
}

int b2q_moe_gather_perm(const void* src, const int32_t* sorted_pairs, const int32_t* perms, const int32_t* offsets, int E,
                        void* dst, int rows, int top_k, int K, void* stream) {
  if (src == nullptr || perms == nullptr || offsets == nullptr || dst == nullptr || E < 1 || rows < 1 || top_k < 1 ||
      K < 8 || K % 8 != 0 || (reinterpret_cast<uintptr_t>(src) & 15) || (reinterpret_cast<uintptr_t>(dst) & 15) ||
      (reinterpret_cast<uintptr_t>(perms) & 15)) {
    set_error("b2q_moe_gather_perm: bad argument (E=%d rows=%d top_k=%d K=%d; K %% 8 == 0, 16-byte aligned)", E, rows,
              top_k, K);
    return -2;
  }
  DeviceGuard dg(dst);
  return check_cuda(launch_moe_gather_perm(src, sorted_pairs, perms, offsets, E, dst, rows, top_k, K, (cudaStream_t)stream),
                    "b2q_moe_gather_perm");
}

static int moe_check(const char* fn, const void* x, const void* packed, const void* scales, const int32_t* counts,
                     const int32_t* offsets, int E, int rows, int K, int N, int bits, int group_size, int dtype) {
  if (counts == nullptr || offsets == nullptr || E < 1 || rows < 1 || (bits != 4 && bits != 8)) {
    set_error("%s: bad argument (E=%d rows=%d bits=%d; the grouped path serves 4- and 8-bit experts)", fn, E, rows, bits);
    return -2;
  }
  return validate(fn, x, packed, scales, x, rows, K, N, bits, group_size, dtype);
}

int b2q_moe_gate_up(const void* xs, const void* packed1, const void* scales1, const int32_t* qzeros1,
                    const void* packed3, const void* scales3, const int32_t* qzeros3, void* h, const int32_t* counts,
                    const int32_t* offsets, int E, int rows, int active, int K, int N, int bits, int group_size, int dtype,
                    void* stream) {
  int v = moe_check("b2q_moe_gate_up", xs, packed1, scales1, counts, offsets, E, rows, K, N, bits, group_size, dtype);
  if (v != 0) return v;
  if (packed3 == nullptr || scales3 == nullptr || h == nullptr || ((qzeros1 != nullptr) != (qzeros3 != nullptr)) ||
      (reinterpret_cast<uintptr_t>(h) & 15) || (reinterpret_cast<uintptr_t>(packed3) & 15)) {
    set_error("b2q_moe_gate_up: w3 / h missing or misaligned, or w1 and w3 differ in symmetry");
    return -2;
  }
  DeviceGuard dg(packed1);
  MmArgs a = make_args(xs, packed1, scales1, qzeros1, nullptr, nullptr, h, rows, K, N, bits, group_size, dtype, nullptr,
                       0, stream);
  MoeGroupedArgs g = {};
  g.counts = counts;
  g.offsets = offsets;
  g.packed3 = packed3;
  g.scales3 = scales3;
  g.qzeros3 = qzeros3;
  g.E = E;
  g.rows = rows;
  g.active = active;
  return check_cuda(launch_midm_grouped(1, a, g), "b2q_moe_gate_up");
}

int b2q_moe_down(const void* h, const void* packed2, const void* scales2, const int32_t* qzeros2, const int32_t* counts,
                 const int32_t* offsets, const int32_t* sorted_pairs, const float* pair_weights, float* ypair, int E,
                 int rows, int active, int K, int N, int bits, int group_size, int dtype, void* stream) {
  int v = moe_check("b2q_moe_down", h, packed2, scales2, counts, offsets, E, rows, K, N, bits, group_size, dtype);
  if (v != 0) return v;
  if (sorted_pairs == nullptr || pair_weights == nullptr || ypair == nullptr ||
      (reinterpret_cast<uintptr_t>(ypair) & 15)) {
    set_error("b2q_moe_down: sorted_pairs / pair_weights / ypair missing or misaligned");
    return -2;
  }
  DeviceGuard dg(packed2);
  MmArgs a = make_args(h, packed2, scales2, qzeros2, nullptr, nullptr, ypair, rows, K, N, bits, group_size, dtype, nullptr,
                       0, stream);
  MoeGroupedArgs g = {};
  g.counts = counts;
  g.offsets = offsets;
  g.sorted_pairs = sorted_pairs;
  g.pair_weights = pair_weights;
  g.ypair = ypair;
  g.E = E;
  g.rows = rows;
  g.active = active;
  return check_cuda(launch_midm_grouped(2, a, g), "b2q_moe_down");
}

int b2q_moe_combine(const float* ypair, void* y, int T, int top_k, int N, int dtype, void* stream) {
  if (ypair == nullptr || y == nullptr || T < 1 || top_k < 1 || N < 4 || N % 4 != 0 || (dtype != 0 && dtype != 1) ||
      (reinterpret_cast<uintptr_t>(ypair) & 15) || (reinterpret_cast<uintptr_t>(y) & 7)) {
    set_error("b2q_moe_combine: bad argument (T=%d top_k=%d N=%d)", T, top_k, N);
    return -2;
  }
  DeviceGuard dg(y);
  return check_cuda(launch_moe_combine(ypair, y, T, top_k, N, dtype, (cudaStream_t)stream), "b2q_moe_combine");
}

int b2q_moe_route(const void* logits, int logits_dtype, const float* bias, int T, int E, int top_k, int scoring,
                  int n_group, int topk_group, int renormalize, float scale, int32_t* topk_ids, float* topk_weights,
                  void* stream) {
  const int max_k = E < 16 ? E : 16;
  if (T < 0 || E < 1 || E > 256 || top_k < 1 || top_k > max_k || logits_dtype < 0 || logits_dtype > 2 ||
      (scoring != 0 && scoring != 1)) {
    set_error("b2q_moe_route: bad argument (T=%d E=%d top_k=%d dtype=%d scoring=%d; 1 <= E <= 256, "
              "1 <= top_k <= min(E, 16))", T, E, top_k, logits_dtype, scoring);
    return -2;
  }
  if (scoring == 0 && (n_group != 1 || topk_group != 1 || bias != nullptr)) {
    set_error("b2q_moe_route: softmax routing takes n_group = topk_group = 1 and no bias (got %d, %d, %s)", n_group,
              topk_group, bias != nullptr ? "a bias" : "no bias");
    return -2;
  }
  if (scoring == 1 && (bias == nullptr || n_group < 1 || E % n_group != 0 || E / n_group < 2 || topk_group < 1 ||
                       topk_group > n_group || top_k > topk_group * (E / n_group))) {
    set_error("b2q_moe_route: grouped sigmoid routing needs a bias, n_group dividing E with >= 2 experts per group, "
              "1 <= topk_group <= n_group and top_k <= topk_group * E / n_group (E=%d n_group=%d topk_group=%d top_k=%d)",
              E, n_group, topk_group, top_k);
    return -2;
  }
  if (T == 0) return 0;
  if (logits == nullptr || topk_ids == nullptr || topk_weights == nullptr) {
    set_error("b2q_moe_route: logits / topk_ids / topk_weights missing");
    return -2;
  }
  DeviceGuard dg(topk_ids);
  return check_cuda(launch_moe_route(logits, logits_dtype, bias, T, E, top_k, scoring, n_group, topk_group, renormalize,
                                     scale, topk_ids, topk_weights, (cudaStream_t)stream),
                    "b2q_moe_route");
}

// ---- MoE decode: one token through its top_k experts on the decode tier (b2q_decode.cu, DecSets::moe) ---------------------
int b2q_moe_decode_gate_up(const void* x, const void* packed1, const void* scales1, const int32_t* qzeros1,
                           const void* packed3, const void* scales3, const int32_t* qzeros3, const int32_t* topk_ids,
                           int top_k, int E, int K, int N, int bits, int group_size, int dtype, void* gu, void* stream) {
  int v = validate("b2q_moe_decode_gate_up", x, packed1, scales1, gu, 1, K, N, bits, group_size, dtype);
  if (v != 0) return v;
  if (packed3 == nullptr || scales3 == nullptr || topk_ids == nullptr || E < 1 ||
      (reinterpret_cast<uintptr_t>(packed3) & 15)) {
    set_error("b2q_moe_decode_gate_up: w3 stack / topk_ids missing or misaligned (E=%d)", E);
    return -2;
  }
  DeviceGuard dg(packed1);
  MmArgs a = make_args(x, packed1, scales1, qzeros1, nullptr, nullptr, gu, 1, K, N, bits, group_size, dtype, nullptr, 0,
                       stream);
  return check_cuda(launch_moe_decode_gate_up(a, packed1, scales1, qzeros1, packed3, scales3, qzeros3, topk_ids, top_k, E,
                                              gu), "b2q_moe_decode_gate_up");
}

int b2q_moe_decode_act(const void* gu, void* h, int top_k, int N, int dtype, void* stream) {
  if (gu == nullptr || h == nullptr || top_k < 1 || N < 2 || N % 2 != 0 || (dtype != 0 && dtype != 1) ||
      (reinterpret_cast<uintptr_t>(gu) & 3) || (reinterpret_cast<uintptr_t>(h) & 3)) {
    set_error("b2q_moe_decode_act: bad argument (top_k=%d N=%d)", top_k, N);
    return -2;
  }
  DeviceGuard dg(h);
  return check_cuda(launch_moe_decode_act(gu, h, top_k, N, dtype, (cudaStream_t)stream), "b2q_moe_decode_act");
}

int b2q_moe_decode_down(const void* h, const void* packed2, const void* scales2, const int32_t* qzeros2,
                        const int32_t* topk_ids, const float* topk_weights, int top_k, int E, int K, int N, int bits,
                        int group_size, int dtype, int fused_act, void* y, void* stream) {
  int v = validate("b2q_moe_decode_down", h, packed2, scales2, y, 1, K, N, bits, group_size, dtype);
  if (v != 0) return v;
  if (topk_ids == nullptr || topk_weights == nullptr || E < 1) {
    set_error("b2q_moe_decode_down: topk_ids / topk_weights missing (E=%d)", E);
    return -2;
  }
  DeviceGuard dg(packed2);
  MmArgs a = make_args(h, packed2, scales2, qzeros2, nullptr, nullptr, y, 1, K, N, bits, group_size, dtype, nullptr, 0,
                       stream);
  return check_cuda(launch_moe_decode_down(a, topk_ids, topk_weights, top_k, E, fused_act), "b2q_moe_decode_down");
}

}  // extern "C"
