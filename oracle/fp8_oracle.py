"""Float64 oracle of FP8 (e4m3fn, W8A16) layers — the arithmetic of the reference's TorchFP8Linear
(gptqmodel/nn_modules/qlinear/fp8.py, the CUDA branch of dequantize_weight + _forward_dequant_matmul), in numpy:

    W[k, n] = RN_T( float(w[n, k]) / float(RN_T(scale_inv[blk(n, k)])) )      (correctly rounded division)
    out     = RN_T( RN_T(x @ W) + bias )                                         (x @ W exact in float64)

T is fp16 or bf16.  bf16 values are carried as float32 arrays holding bf16 values (numpy has no bf16).
"""
from __future__ import annotations

import numpy as np


def e4m3_table() -> np.ndarray:
    """float64 value of each of the 256 e4m3fn codes (NaN for 0x7F / 0xFF): sign, 4 exponent bits (bias 7), 3 mantissa
    bits, subnormals at exponent 0, no infinities."""
    v = np.empty(256, np.float64)
    for c in range(256):
        s, e, m = c >> 7, (c >> 3) & 15, c & 7
        if e == 15 and m == 7:
            x = np.nan
        elif e == 0:
            x = m / 8.0 * 2.0 ** -6
        else:
            x = (1 + m / 8.0) * 2.0 ** (e - 7)
        v[c] = -x if s else x
    return v


def round_bf16(a) -> np.ndarray:
    """float32 -> nearest bf16 value (ties to even), as float32; NaN stays NaN."""
    a = np.asarray(a, np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16 << 16).astype(np.uint32).view(np.float32)
    return np.where(np.isnan(a), np.float32(np.nan), r)


def round_to(a, dtype: str) -> np.ndarray:
    """float32 values -> dtype ('fp16' | 'bf16') values: fp16 as float16, bf16 as float32."""
    a = np.asarray(a, np.float32)
    return a.astype(np.float16) if dtype == "fp16" else round_bf16(a)


def div_t(w, s, dtype: str) -> np.ndarray:
    """RN_T(w / s) for T-valued w, s: the IEEE fp32 quotient rounded to T (no double rounding: 24 >= 2 p + 2)."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return round_to(np.asarray(w, np.float32) / np.asarray(s, np.float32), dtype)


def expand_scale_inv(scale_inv, N: int, K: int, method: str, block=None) -> np.ndarray:
    """fp32 scale_inv -> fp32 [N, K], each scale repeated over its block."""
    s = np.asarray(scale_inv, np.float32)
    if method == "tensor":
        return np.full((N, K), s.reshape(-1)[0], np.float32)
    if method == "row":
        return np.repeat(s.reshape(N, 1), K, axis=1)
    br, bc = block
    return np.repeat(np.repeat(s.reshape(N // br, K // bc), br, axis=0), bc, axis=1)


def dequantize(codes, scale_inv, method: str, block, dtype: str) -> np.ndarray:
    """codes uint8 [N, K] (e4m3fn bit patterns) -> W [K, N] of dtype (float16, or float32 holding bf16 values)."""
    codes = np.asarray(codes, np.uint8)
    N, K = codes.shape
    w = e4m3_table()[codes].astype(np.float32)  # exact in fp16 and bf16 as well
    s = round_to(expand_scale_inv(scale_inv, N, K, method, block), dtype)
    return np.ascontiguousarray(div_t(w, s, dtype).T)


def round64_to(a, dtype: str) -> np.ndarray:
    """float64 -> nearest dtype value in ONE rounding (ties to even; normal range)."""
    a = np.asarray(a, np.float64)
    if dtype == "fp16":
        return a.astype(np.float16)
    m, e = np.frexp(a)
    return np.ldexp(np.rint(m * 256.0) / 256.0, e).astype(np.float32)


def forward(x, W, bias=None, dtype: str = "fp16") -> np.ndarray:
    """x [M, K] (T values), W [K, N] (T values) -> out [M, N] of dtype: the float64 product rounded to T once, then the
    bias added and rounded again (the reference's order)."""
    y = round64_to(np.asarray(x, np.float64) @ np.asarray(W, np.float64), dtype)
    if bias is not None:
        y = round_to(y.astype(np.float32) + round_to(np.asarray(bias, np.float32), dtype).astype(np.float32), dtype)
    return y
