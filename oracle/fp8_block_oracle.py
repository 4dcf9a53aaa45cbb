"""Numpy oracle of the block-FP8 (W8A8) layer (include/b2q.h, "Block-FP8"): HF / DeepSeek-native checkpoints with e4m3
weights [N, K], fp32 weight_scale_inv [ceil(N/128), K/128] that multiplies them, and per-token groups of 128 k quantised
to e4m3 at run time.

  * quantize(x)            : the activation quantiser, bit-exact in fp32 (codes and token scales);
  * promote(...)           : a float32 mirror of the kernel's promotion chain for a given split-K, with an exact fmaf;
  * reference(...)         : float64 sum_b s_x s_w sum_k q w (exact for e4m3 products) and the matching magnitude sum;
  * dequantize_weight(...) : W [K, N] = RN_T(T(w) * T(s_w)), the HF dequantiser's arithmetic.
Activations and 16-bit results travel as float32 arrays holding fp16 / bf16 values (numpy has no bf16).
"""
from __future__ import annotations

import numpy as np

BLOCK = 128
FP8_MAX = 448.0
F32, F64 = np.float32, np.float64


def _e4m3_table() -> np.ndarray:
    c = np.arange(256)
    e, m = (c >> 3) & 15, (c & 7).astype(F64)
    mag = np.where(e == 0, m * 2.0 ** -9, (1.0 + m / 8.0) * 2.0 ** (e - 7.0))
    val = np.where(c >= 128, -mag, mag)
    val[[0x7F, 0xFF]] = np.nan
    return val


E4M3 = _e4m3_table()


def e4m3_decode(codes: np.ndarray) -> np.ndarray:
    """uint8 e4m3fn bit patterns -> float64 values."""
    return E4M3[np.asarray(codes, np.uint8)]


def e4m3_encode_rn_satfinite(v: np.ndarray) -> np.ndarray:
    """float32 -> e4m3fn codes: round to nearest even, finite values beyond 448 saturate (cvt.rn.satfinite)."""
    v = np.asarray(v, F32).astype(F64)
    a = np.abs(v)
    _, ex = np.frexp(np.where(a > 0, a, 1.0))  # a = f * 2^ex, f in [0.5, 1)
    step = np.where(a < 2.0 ** -6, 2.0 ** -9, np.ldexp(1.0, ex - 4))  # ulp: 3 mantissa bits, subnormal ulp 2^-9
    q = np.minimum(np.rint(a / step) * step, FP8_MAX)  # power-of-two scaling is exact; rint ties to even
    _, qe = np.frexp(np.where(q > 0, q, 1.0))
    sub = q < 2.0 ** -6
    efield = np.where(sub, 0, qe + 6)  # q = (1 + m/8) 2^(qe - 1), bias 7
    mant = np.where(sub, q / 2.0 ** -9, (np.ldexp(q, -(qe - 1)) - 1.0) * 8.0)
    code = (efield.astype(np.int64) << 3) | np.rint(mant).astype(np.int64)
    code = np.where(np.signbit(v), code | 0x80, code)
    return code.astype(np.uint8)


def quantize(x: np.ndarray):
    """x [M, K] (fp16 / bf16 values as float32) -> (codes uint8 [M, K], s_x float32 [M, K/128])."""
    x = np.asarray(x, F32)
    M, K = x.shape
    g = x.reshape(M, K // BLOCK, BLOCK)
    amax = np.abs(g).max(axis=2)
    s = np.maximum(amax, F32(1e-10)) / F32(FP8_MAX)  # IEEE fp32 division
    v = g / s[:, :, None]  # IEEE fp32 division
    return e4m3_encode_rn_satfinite(v).reshape(M, K), s.astype(F32)


def fma32(a, b, c) -> np.ndarray:
    """Correctly rounded float32 a * b + c (fmaf).  a * b is exact in float64; the float64 sum's rounding error is
    recovered with TwoSum and decides the one case where rounding to float32 again would differ: a float64 sum that lies
    exactly halfway between two float32 values."""
    a, b, c = (np.asarray(t, F32) for t in (a, b, c))
    p = a.astype(F64) * b.astype(F64)
    c64 = c.astype(F64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)
    r = s.astype(F32)
    back = r.astype(F64)
    with np.errstate(over="ignore", invalid="ignore"):
        other = np.nextafter(r, np.where(s > back, np.inf, -np.inf).astype(F32))
        mid = (back + other.astype(F64)) * 0.5
    tie = (s != back) & (s == mid) & (err != 0)
    away = np.sign(err) == np.sign(s - back)
    return np.where(tie & away, other, r).astype(F32)


def block_sums(codes: np.ndarray, w: np.ndarray) -> np.ndarray:
    """P[b, m, n] = sum_{k in b} q[m, k] w[n, k] in float64 (exact: e4m3 products have 8 significant bits)."""
    M, K = codes.shape
    KB = K // BLOCK
    q = e4m3_decode(codes).reshape(M, KB, BLOCK).transpose(1, 0, 2)
    wv = e4m3_decode(w).reshape(w.shape[0], KB, BLOCK).transpose(1, 2, 0)
    return np.matmul(q, wv)


def expand_sw(s_w: np.ndarray, N: int) -> np.ndarray:
    """s_w [ceil(N/128), KB] -> [KB, N] (the scale of feature n is row n // 128)."""
    return np.repeat(np.asarray(s_w, F32), BLOCK, axis=0)[:N].T


def promote(codes, s_x, w, s_w, ks: int = 1) -> np.ndarray:
    """float32 acc [M, N] of the kernel's chain: per rank, acc = fmaf(float32(P_b), s_x[m, b] * s_w[n/128, b], acc) over
    the rank's k-blocks in order from acc = 0; rank r holds blocks [r kpc, (r + 1) kpc), kpc = ceil(KB / ks); the ranks'
    partials are added in rank order.  P_b is taken exact (what the tensor cores give when the block sums are exact)."""
    M, K = codes.shape
    N = w.shape[0]
    KB = K // BLOCK
    P = block_sums(codes, w).astype(F32)
    sw = expand_sw(s_w, N)
    kpc = -(-KB // ks)
    total = None
    for r in range(ks):
        acc = np.zeros((M, N), F32)
        for b in range(r * kpc, min(KB, (r + 1) * kpc)):
            sc = np.asarray(s_x, F32)[:, b][:, None] * sw[b][None, :]  # float32 product, rounded once
            acc = fma32(P[b], sc, acc)
        total = acc if total is None else (total + acc).astype(F32)
    return total


def reference(codes, s_x, w, s_w):
    """(float64 sum_b s_x s_w sum_k q w, float64 sum_b |s_x s_w| sum_k |q w|), both [M, N]."""
    M, K = codes.shape
    N = w.shape[0]
    P = block_sums(codes, w)
    A = np.matmul(np.abs(e4m3_decode(codes)).reshape(M, K // BLOCK, BLOCK).transpose(1, 0, 2),
                  np.abs(e4m3_decode(w)).reshape(N, K // BLOCK, BLOCK).transpose(1, 2, 0))
    sc = np.asarray(s_x, F64).T[:, :, None] * expand_sw(s_w, N).astype(F64)[:, None, :]
    return (P * sc).sum(axis=0), (A * np.abs(sc)).sum(axis=0)


def round_bf16(v: np.ndarray) -> np.ndarray:
    """float32 -> nearest bf16 (ties to even), returned as float32 (finite inputs)."""
    u = np.asarray(v, F32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(F32)


def unpack16(a: np.ndarray) -> np.ndarray:
    """A stored 16-bit array -> float32: float16 values, or bf16 bit patterns held as uint16."""
    a = np.asarray(a)
    if a.dtype == np.uint16:
        return (a.astype(np.uint32) << 16).view(F32)
    return a.astype(F32)


def round_t(v: np.ndarray, dtype: str) -> np.ndarray:
    """float32 -> T ("fp16" / "bf16"), returned as float32."""
    v = np.asarray(v, F32)
    return v.astype(np.float16).astype(F32) if dtype == "fp16" else round_bf16(v)


def dequantize_weight(w: np.ndarray, s_w: np.ndarray, dtype: str = "fp16") -> np.ndarray:
    """W [K, N] = RN_T(T(w[n, k]) * T(s_w[n / 128, k / 128])) as float32 (the T * T product is exact in float32)."""
    N, K = w.shape
    wt = round_t(e4m3_decode(w).astype(F32), dtype)
    st = round_t(np.repeat(np.repeat(np.asarray(s_w, F32), BLOCK, 0)[:N], BLOCK, 1), dtype)
    return round_t(wt * st, dtype).T.copy()
