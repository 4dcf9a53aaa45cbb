"""Numpy mirror of the per-channel FP8 (W8A8) layer (include/b2q.h, "Per-channel FP8"): e4m3 weights [N, K] with one
fp32 scale per output feature, activations quantised per token (dynamic, amax optionally bounded by ub) or with one
static per-tensor scale.

  * quantize_dynamic / quantize_static : the activation quantisers, bit-exact in fp32 (codes and token scales);
  * promote(...)   : a float32 mirror of the kernel's k-sum for a given split-K (acc += fp32(P_b), ranks in order);
  * epilogue(...)  : y = T(acc * (s_x[m] * s_w[n]) + bias[n]) in float32, one rounding;
  * reference(...) : float64 s_x s_w sum_k q w (exact for e4m3 products) and the matching magnitude sum.
Activations and 16-bit results travel as float32 arrays holding fp16 / bf16 values (numpy has no bf16).
"""
import numpy as np

from oracle.fp8_block_oracle import BLOCK, FP8_MAX, block_sums, e4m3_decode, e4m3_encode_rn_satfinite, round_t

F32, F64 = np.float32, np.float64


def quantize_dynamic(x: np.ndarray, ub: float = np.inf):
    """x [M, K] -> (codes uint8 [M, K], s_x float32 [M]): s_x = max(min(amax, ub), 1e-10) / 448, codes of x / s_x."""
    x = np.asarray(x, F32)
    amax = np.abs(x).max(axis=1)
    s = np.maximum(np.minimum(amax, F32(ub)), F32(1e-10)) / F32(FP8_MAX)  # IEEE fp32 division
    return e4m3_encode_rn_satfinite(x / s[:, None]), s.astype(F32)


def quantize_static(x: np.ndarray, s_in: float):
    """x [M, K] -> (codes of x / s_in, s_x = s_in for every row)."""
    x = np.asarray(x, F32)
    s = np.full(x.shape[0], F32(s_in), F32)
    return e4m3_encode_rn_satfinite(x / s[:, None]), s


def promote(codes, w, ks: int = 1) -> np.ndarray:
    """float32 acc [M, N]: per rank acc += float32(P_b) over the rank's k-blocks in order from 0 (rank r holds blocks
    [r kpc, (r + 1) kpc), kpc = ceil(KB / ks)); the ranks' partials are added in rank order.  P_b is taken exact."""
    KB = codes.shape[1] // BLOCK
    P = block_sums(codes, w).astype(F32)
    kpc = -(-KB // ks)
    total = None
    for r in range(ks):
        acc = np.zeros(P.shape[1:], F32)
        for b in range(r * kpc, min(KB, (r + 1) * kpc)):
            acc = (acc + P[b]).astype(F32)
        total = acc if total is None else (total + acc).astype(F32)
    return total


def epilogue(acc, s_x, s_w, bias, dtype: str) -> np.ndarray:
    """T(acc * (s_x[m] * s_w[n]) + bias[n]) with float32 products and sum, rounded once to T; bias may be None."""
    sc = (np.asarray(s_x, F32)[:, None] * np.asarray(s_w, F32)[None, :]).astype(F32)
    y = (np.asarray(acc, F32) * sc).astype(F32)
    if bias is not None:
        y = (y + np.asarray(bias, F32)[None, :]).astype(F32)
    return round_t(y, dtype)


def reference(codes, s_x, w, s_w):
    """(float64 s_x s_w sum_k q w, float64 |s_x s_w| sum_k |q w|), both [M, N]."""
    q, wv = e4m3_decode(codes), e4m3_decode(w)
    sc = np.asarray(s_x, F64)[:, None] * np.asarray(s_w, F64)[None, :]
    return (q @ wv.T) * sc, (np.abs(q) @ np.abs(wv).T) * np.abs(sc)
