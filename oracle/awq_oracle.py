"""TEST INFRASTRUCTURE ONLY — CPU oracle for the AWQ (FORMAT.GEMM) checkpoint layout.

Restates (no code copied) what the reference computes for an AWQ GEMM-format layer:
  * layout: ``qweight int32 [K, N*bits/32]`` packed along the OUTPUT dimension, ``qzeros int32 [G, N*bits/32]`` packed the
    same way, ``scales fp16 [G, N]`` (gptqmodel/nn_modules/qlinear/__init__.py:1634-1668);
  * inside every 32-bit word the 8 nibbles are interleaved: nibble i (bits 4i..4i+3) holds logical column
    8c + AWQ_ORDER[i], AWQ_ORDER = [0, 2, 4, 6, 1, 3, 5, 7]; reading logical column j means nibble
    AWQ_REVERSE_ORDER[j] = [0, 4, 1, 5, 2, 6, 3, 7][j] (quantization/awq/utils/packing_utils.py:9-10, 43-58);
  * dequant: ``(q - z) * scale`` with the TRUE zero-point (no +1), one fp16 rounding (packing_utils.py:106-121);
  * forward: ``matmul(x, W)`` rounded to the activation dtype, then ``+ bias`` (qlinear/torch_awq.py:157-197).
Pinned against fixtures produced by running the unmodified reference (tests/golden/make_golden_awq.py ->
tests/golden/awq_cases.npz; tests/test_awq.py).  The product path never imports this module.
"""
from __future__ import annotations

import torch

AWQ_ORDER = [0, 2, 4, 6, 1, 3, 5, 7]
AWQ_REVERSE_ORDER = [0, 4, 1, 5, 2, 6, 3, 7]

__all__ = ["awq_unpack", "awq_dequantize", "awq_forward", "awq_forward_exact", "awq_pack", "AWQ_ORDER", "AWQ_REVERSE_ORDER"]


def awq_unpack(packed: torch.Tensor, bits: int = 4) -> torch.Tensor:
    """int32 [R, C*bits/32] -> codes int16 [R, C] in LOGICAL column order."""
    assert packed.dtype == torch.int32 and bits == 4
    R, W = packed.shape
    out = torch.empty(R, W * 8, dtype=torch.int16)
    for j in range(8):  # logical column 8c + j lives in nibble AWQ_REVERSE_ORDER[j]
        out[:, j::8] = ((packed >> (4 * AWQ_REVERSE_ORDER[j])) & 0xF).to(torch.int16)
    return out


def awq_dequantize(qweight, qzeros, scales, group_size: int) -> torch.Tensor:
    """-> W [K, N] in scales.dtype: (q - z) computed in integers, ONE rounding by the multiplication."""
    q = awq_unpack(qweight)
    z = awq_unpack(qzeros)
    K = q.shape[0]
    gs = group_size if group_size > 0 else K
    g = torch.arange(K) // gs
    return ((q - z[g]).to(scales.dtype) * scales[g])


def awq_forward(x, qweight, qzeros, scales, group_size: int, bias=None) -> torch.Tensor:
    W = awq_dequantize(qweight, qzeros, scales.to(x.dtype), group_size)
    y = (x.float() @ W.float()).to(x.dtype)  # fp32 accumulation, rounded once to the activation dtype
    if bias is not None:
        y = y + bias.to(x.dtype)
    return y


def awq_forward_exact(x, qweight, qzeros, scales, group_size: int, bias=None) -> torch.Tensor:
    """The same layer in EXACT arithmetic: W = (q - z) * s WITHOUT the reference's per-weight rounding to 16 bits, the dot
    product in float64, one rounding of the result to the activation dtype (then + bias like the reference).  Not what
    the reference computes — it is what a kernel that applies the scale once per group to an exact integer dot product
    (the decode / GEMV tiers) converges to; tests use it to separate kernel arithmetic errors from the reference's own
    weight-rounding noise (tests/helpers.py::ref_rounding_slack)."""
    q = awq_unpack(qweight).double()
    z = awq_unpack(qzeros).double()
    K = q.shape[0]
    gs = group_size if group_size > 0 else K
    g = torch.arange(K) // gs
    W = (q - z[g]) * scales.to(x.dtype).double()[g]
    y = (x.double() @ W).to(x.dtype)
    if bias is not None:
        y = y + bias.to(x.dtype)
    return y


def awq_pack(codes: torch.Tensor) -> torch.Tensor:
    """codes [R, C] (0..15, logical order) -> int32 [R, C/8] in the AWQ interleaved order (fixture helper)."""
    R, C = codes.shape
    acc = torch.zeros(R, C // 8, dtype=torch.int64)
    for i in range(8):  # nibble i holds logical column 8c + AWQ_ORDER[i]
        acc |= (codes[:, AWQ_ORDER[i]::8].to(torch.int64) & 0xF) << (4 * i)
    acc = torch.where(acc >= 2 ** 31, acc - 2 ** 32, acc)
    return acc.to(torch.int32)
