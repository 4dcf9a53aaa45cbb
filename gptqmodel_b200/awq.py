"""AWQ (FORMAT.GEMM) front-end onto the same B200 kernels.

An AWQ GEMM-format checkpoint stores ``qweight int32 [K, N/8]`` packed along the OUTPUT dimension with the nibbles of
every word interleaved (nibble i holds logical column 8c + [0, 2, 4, 6, 1, 3, 5, 7][i]), ``qzeros int32 [G, N/8]`` packed
the same way and ``scales fp16 [G, N]``; its dequantisation is ``(q - z) * scale`` with the true zero-point
(gptqmodel/nn_modules/qlinear/__init__.py:1634-1668,
gptqmodel/quantization/awq/utils/packing_utils.py:9-10, 106-121).  That is exactly the arithmetic of a
GPTQ v2 layer, so one exact integer re-packing at load time (``awq_gemm_to_gptq``) lets the fragment-major prepack and
every kernel of this package serve AWQ models unchanged — the route the reference's own AwqSwordfishLinear / AwqMarlin
take (qlinear/swordfish.py:358-394, 565-606).

``B200AwqQuantLinear`` mirrors the reference's AWQuantLinear contract: AWQ-shaped ``qweight / qzeros / scales`` buffers
for the loader to fill, ``post_init()`` converts on the weights' device, ``forward(x)`` is the shared hot path.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn as nn

from .qlinear import B200QuantLinear

AWQ_REVERSE_ORDER = (0, 4, 1, 5, 2, 6, 3, 7)  # logical column j of a word lives in nibble AWQ_REVERSE_ORDER[j]


def _wrap_i32(acc: torch.Tensor) -> torch.Tensor:
    """int64 bit pattern (0 .. 2^32-1) -> the int32 with the same 32 bits."""
    return torch.where(acc >= 2 ** 31, acc - 2 ** 32, acc).to(torch.int32)


@torch.no_grad()
def awq_gemm_to_gptq(qweight: torch.Tensor, qzeros: torch.Tensor, scales: torch.Tensor, group_size: int,
                     bits: int = 4) -> Dict[str, torch.Tensor]:
    """AWQ GEMM-layout tensors -> GPTQ v2 checkpoint-layout tensors (exact; runs on the tensors' device).

    Returns ``qweight int32 [K/8, N]`` (row 8i+j of column n in bits 4j.. of word [i, n]), ``qzeros int32 [G, N/8]``
    (column 8c+j in bits 4j.., true zero-points), ``scales`` (unchanged) and the trivial ``g_idx``.
    """
    if bits != 4:
        raise NotImplementedError("AWQ front-end: 4-bit GEMM format only")
    if qweight.dtype != torch.int32 or qzeros.dtype != torch.int32:
        raise ValueError("AWQ qweight / qzeros must be int32")
    K, W = qweight.shape
    N = W * 8
    gs = group_size if group_size > 0 else K
    if K % 8 != 0 or K % gs != 0 or qzeros.shape != (K // gs, W) or scales.shape != (K // gs, N):
        raise ValueError(f"AWQ tensor shapes do not match K={K} N={N} group_size={gs}: qzeros {tuple(qzeros.shape)}, "
                         f"scales {tuple(scales.shape)}")
    dev = qweight.device
    # zero-points stay packed along N: only the nibbles inside every word move (new nibble j = old nibble REV[j])
    z64 = qzeros.to(torch.int64) & 0xFFFFFFFF
    zacc = torch.zeros_like(z64)
    for j, src in enumerate(AWQ_REVERSE_ORDER):
        zacc |= ((z64 >> (4 * src)) & 0xF) << (4 * j)
    # weights change packing direction (along N -> along K): unpack to codes [K, N] in logical order, repack 8 rows/word
    q64 = qweight.to(torch.int64) & 0xFFFFFFFF
    codes = torch.empty((K, N), dtype=torch.uint8, device=dev)
    for j, src in enumerate(AWQ_REVERSE_ORDER):
        codes[:, j::8] = ((q64 >> (4 * src)) & 0xF).to(torch.uint8)
    del q64
    c3 = codes.view(K // 8, 8, N)
    wacc = torch.zeros((K // 8, N), dtype=torch.int64, device=dev)
    for j in range(8):
        wacc |= c3[:, j, :].to(torch.int64) << (4 * j)
    return {
        "qweight": _wrap_i32(wacc).contiguous(),
        "qzeros": _wrap_i32(zacc).contiguous(),
        "scales": scales.contiguous(),
        "g_idx": (torch.arange(K, dtype=torch.int32, device=dev) // gs).contiguous(),
    }


class B200AwqQuantLinear(B200QuantLinear):
    """AWQ GEMM-format QuantLinear on the B200 kernels (4-bit, group_size 32|64|128|-1, asymmetric by construction)."""

    SUPPORTS_BITS = [4]
    SUPPORTS_DESC_ACT = [False]
    SUPPORTS_FORMATS = {"gemm": 110}
    SUPPORTS_METHODS = ["awq"]
    REQUIRES_FORMAT_V2 = False  # AWQ zero-points are already true zero-points
    QUANT_TYPE = "b200_awq"

    def __init__(self, bits: int, group_size: int, sym: bool = False, desc_act: bool = False, in_features: int = None,
                 out_features: int = None, bias: bool = False, register_buffers: bool = True, **kwargs):
        if desc_act:
            raise NotImplementedError("B200AwqQuantLinear: AWQ has no act-order")
        super().__init__(bits=bits, group_size=group_size, desc_act=False, sym=sym, in_features=in_features,
                         out_features=out_features, bias=bias, register_buffers=False, **kwargs)
        K, N = in_features, out_features
        G = K // self.group_size
        if register_buffers:  # AWQ-shaped, what the reference's AWQuantLinear registers (qlinear/__init__.py:1646-1668)
            mk = lambda t: nn.Parameter(t, requires_grad=False)  # noqa: E731
            self.qweight = mk(torch.zeros((K, N // 8), dtype=torch.int32))
            self.qzeros = mk(torch.zeros((G, N // 8), dtype=torch.int32))
            self.scales = mk(torch.zeros((G, N), dtype=torch.float16))
            self.bias = mk(torch.zeros(N, dtype=torch.float16)) if bias else None

    @torch.no_grad()
    def post_init(self):
        if self._prepacked:
            return
        conv = awq_gemm_to_gptq(self.qweight.data, self.qzeros.data, self.scales.data, self.group_size, self.bits)
        mk = lambda t: nn.Parameter(t, requires_grad=False)  # noqa: E731
        self.qweight, self.qzeros, self.g_idx = mk(conv["qweight"]), mk(conv["qzeros"]), mk(conv["g_idx"])
        self.scales = mk(conv["scales"])
        self._qzeros_format = 2
        super().post_init()

    @classmethod
    def from_awq_tensors(cls, qweight, qzeros, scales, group_size: int, bias: Optional[torch.Tensor] = None,
                         device="cuda", dtype=None):
        """Build + post_init a module from AWQ GEMM-layout tensors."""
        K, N = qweight.shape[0], qweight.shape[1] * 8
        m = cls(bits=4, group_size=group_size, in_features=K, out_features=N, bias=bias is not None,
                register_buffers=False, dtype=dtype)
        mk = lambda t: nn.Parameter(t.detach().clone().contiguous().to(device), requires_grad=False)  # noqa: E731
        m.qweight, m.qzeros, m.scales = mk(qweight), mk(qzeros), mk(scales)
        m.bias = mk(bias) if bias is not None else None
        m.post_init()
        return m
