// b2q_api.cu — the extern "C" boundary declared in include/b2q.h: argument validation + tier dispatch.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "../../include/b2q.h"
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
  c.decode_blocks_m = env_int("B2Q_DECODE_BLOCKS_M", 0);
  c.decode_groups2 = env_int("B2Q_DECODE_GROUPS", 1) == 2;
  c.decode_v2 = env_int("B2Q_DECODE_V2", -1);
  c.decode2_gw = env_int("B2Q_DECODE2_GW", 0);
  c.decode2_ks = env_int("B2Q_DECODE2_KS", 0);
  c.decode2_xtma = env_int("B2Q_DECODE2_XTMA", 0);
  c.decode2_fastsync = env_int("B2Q_DECODE2_FASTSYNC", 0);
  c.midm_ks = env_int("B2Q_MIDM_KS", 0);
  c.midm_dqg1 = env_int("B2Q_MIDM_DQG1", 0);
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
  if (group_size < 32 || group_size % 32 != 0 || K % group_size != 0) {
    set_error("%s: group_size=%d not supported for K=%d (multiple of 32 dividing K)", fn, group_size, K);
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
  a.pdl = env().disable_pdl ? 0 : 1;
  return a;
}
}  // namespace b2q

using namespace b2q;

extern "C" {

int b2q_version(void) { return B2Q_ABI_VERSION; }

void b2q_debug_set_trace(void* device_buffer) { g_trace_ptr = device_buffer; }

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
  if (decode_supported(a)) return 0;                 // the decode tier gathers x[perm] while staging the activations
  if (M == 1 && bits == 8 && K % 128 == 0) return 0;  // so does the 8-bit GEMV
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

int b2q_gemv(const void* x, const void* packed, const void* scales, const int32_t* qzeros, const int32_t* perm,
             const void* bias, void* out, int K, int N, int bits, int group_size, int dtype, int ks, int warps,
             void* stream) {
  int v = validate("b2q_gemv", x, packed, scales, out, 1, K, N, bits, group_size, dtype);
  if (v != 0) return v;
  DeviceGuard dg(packed);
  if (ks > 16 || warps > 16 || (ks > 0 && (ks & (ks - 1)) != 0)) {
    set_error("b2q_gemv: ks=%d (power of two <= 16) / warps=%d (<= 16) out of range", ks, warps);
    return -2;
  }
  MmArgs a = make_args(x, packed, scales, qzeros, perm, bias, out, 1, K, N, bits, group_size, dtype, nullptr, 0,
                       stream);
  a.tune_ks = ks;
  a.tune_warps = warps;
  if (decode_supported(a)) return check_cuda(launch_decode(a), "b2q_gemv(decode)");
  if (bits == 8 && K % 128 == 0) return check_cuda(launch_gemv(a), "b2q_gemv");
  set_error("b2q_gemv: no M=1 tier for bits=%d K=%d group_size=%d (use b2q_mm)", bits, K, group_size);
  return -2;
}

int b2q_decode(const void* x, const void* packed, const void* scales, const int32_t* qzeros, const int32_t* perm,
               const void* bias, void* out, int M, int K, int N, int bits, int group_size, int dtype, int ks,
               int warps, void* stream) {
  int v = validate("b2q_decode", x, packed, scales, out, M, K, N, bits, group_size, dtype);
  if (v != 0) return v;
  DeviceGuard dg(packed);
  if (ks > 16 || warps > 16 || (ks > 0 && (ks & (ks - 1)) != 0)) {
    set_error("b2q_decode: ks=%d (power of two <= 16) / warps=%d (<= 16) out of range", ks, warps);
    return -2;
  }
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
      out == nullptr || N == nullptr || nsets < 1) {
    set_error("b2q_gemm_multi: null pointer argument");
    return -2;
  }
  int v = validate("b2q_gemm_multi", x, packed[0], scales[0], out[0], M, K, N[0], bits, group_size, dtype);
  if (v != 0) return v;
  if (bits != 4 || M <= 128) {
    set_error("b2q_gemm_multi: the fused prefill launch serves bits=4, M > 128 (got bits=%d M=%d)", bits, M);
    return -2;
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
  // 9 <= M <= B2Q_DECODE_BLOCKS_M (default off): passes of the decode tier over blocks of 8 rows, an earlier answer to
  // the padded 128-token tile's waste; superseded by the small-batch tier (b2q_midm.cu), kept for A/B measurements
  {
    MmArgs a8 = a;
    a8.M = 8;
    if (M > 8 && M <= env().decode_blocks_m && decode_supported(a8) && perm == nullptr) {
      for (int m0 = 0; m0 < M; m0 += 8) {
        MmArgs ab = a;
        ab.M = (M - m0 < 8) ? (M - m0) : 8;
        ab.x = static_cast<const char*>(x) + (size_t)m0 * K * 2;
        ab.out = static_cast<char*>(out) + (size_t)m0 * N * 2;
        int e = check_cuda(launch_decode(ab), "b2q_mm(decode x blocks)");
        if (e != 0) return e;
      }
      return 0;
    }
  }
  if (M == 1 && bits == 8 && K % 128 == 0) return check_cuda(launch_gemv(a), "b2q_mm(gemv)");
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

static int moe_check(const char* fn, const void* x, const void* packed, const void* scales, const int32_t* counts,
                     const int32_t* offsets, int E, int rows, int K, int N, int bits, int group_size, int dtype) {
  if (counts == nullptr || offsets == nullptr || E < 1 || rows < 1 || bits != 4) {
    set_error("%s: bad argument (E=%d rows=%d bits=%d; the grouped path serves 4-bit experts)", fn, E, rows, bits);
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
