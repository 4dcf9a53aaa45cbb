"""Numpy mirror of the per-channel INT8 (W8A8) layer (include/b2q.h, "Per-channel INT8"): int8 weights [N, K] with one
fp32 scale per output feature, activations quantised per token (dynamic) or with one static per-tensor scale.

  * quantize_dynamic / quantize_static : the activation quantisers, bit-exact in fp32 (codes and token scales);
  * int_sums(...)  : the exact k-sums sum_k q w in int64 (the kernel's int32 sums, which cannot overflow);
  * epilogue(...)  : y = T(float32(acc) * (s_x[m] * s_w[n]) + bias[n]) in float32, one rounding.
Activations and 16-bit results travel as float32 arrays holding fp16 / bf16 values (numpy has no bf16).
"""
import numpy as np

from oracle.fp8_block_oracle import round_t

F32 = np.float32


def codes_of(x: np.ndarray, s: np.ndarray) -> np.ndarray:
    """int8 clamp(rint(x / s), -128, 127): IEEE fp32 division, round half to even."""
    return np.clip(np.rint(np.asarray(x, F32) / s[:, None]), -128, 127).astype(np.int8)


def quantize_dynamic(x: np.ndarray):
    """x [M, K] -> (codes int8 [M, K], s_x float32 [M]): s_x = max(amax, 1e-10) / 127, codes of x / s_x."""
    x = np.asarray(x, F32)
    s = (np.maximum(np.abs(x).max(axis=1), F32(1e-10)) / F32(127)).astype(F32)  # IEEE fp32 division
    return codes_of(x, s), s


def quantize_static(x: np.ndarray, s_in: float):
    """x [M, K] -> (codes of x / s_in, s_x = s_in for every row)."""
    s = np.full(np.asarray(x).shape[0], F32(s_in), F32)
    return codes_of(x, s), s


def int_sums(codes, w) -> np.ndarray:
    """int64 acc [M, N] = sum_k q[m, k] w[n, k], exact."""
    return np.asarray(codes, np.int64) @ np.asarray(w, np.int64).T


def epilogue(acc, s_x, s_w, bias, dtype: str) -> np.ndarray:
    """T(float32(acc) * (s_x[m] * s_w[n]) + bias[n]) with float32 products and sum, rounded once to T; bias may be
    None.  float32(acc) rounds to nearest (exact for |acc| <= 2^24)."""
    sc = (np.asarray(s_x, F32)[:, None] * np.asarray(s_w, F32)[None, :]).astype(F32)
    y = (np.asarray(acc).astype(F32) * sc).astype(F32)
    if bias is not None:
        y = (y + np.asarray(bias, F32)[None, :]).astype(F32)
    return round_t(y, dtype)
