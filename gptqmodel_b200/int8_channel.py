"""Per-channel / per-tensor INT8 (W8A8) checkpoints on the s8 tensor cores: ``B200ChannelInt8Linear``.

These checkpoints (llm-compressor / compressed-tensors ``W8A8``, ``format: int-quantized``) store per module
  ``weight``        int8 [N, K],
  ``weight_scale``  [N, 1] / [N] (per channel) or [1] / [] (per tensor), fp32, bf16 or fp16, which MULTIPLIES the weight,
  ``input_scale``   [1] / [] (static activations only),
  ``bias``          optional.
``forward()`` quantises the activations to int8 (per token, ``max|x| / 127``, or with the static ``input_scale``) and
runs an s8 GEMM with exact int32 sums whose scales are applied once, after the k-sum (``b2q_int8ch_forward``;
include/b2q.h states the arithmetic).  The checkpoint weight is the kernel's operand: ``post_init()`` widens the scales
to fp32 (exactly) and broadcasts a per-tensor weight scale, it repacks nothing.  There is no torch fallback.
"""
from __future__ import annotations

from typing import Optional

import torch

from ._lib import check, lib
from .fp8_block import _DTYPE_CODE, _ptr
from .fp8_channel import ChannelW8A8Linear


class B200ChannelInt8Linear(ChannelW8A8Linear):
    """Per-channel / per-tensor INT8 linear (buffers ``weight``, ``weight_scale``, ``input_scale``, ``bias``) on the
    sm_90a s8 wgmma kernels.  ``activation``: "dynamic" (per-token scales) or "static" (the per-tensor
    ``input_scale``)."""

    CODE_DTYPE = torch.int8
    WEIGHT_DTYPES = (torch.int8,)
    SUPPORTS_METHODS = ["compressed-tensors"]
    QUANT_TYPE = "b200_int8_channel"

    def __init__(self, in_features: int, out_features: int, bias: bool = False, activation: str = "dynamic",
                 ub: Optional[float] = None, adapter=None, register_buffers: bool = True, **kwargs):
        if ub is not None:
            raise ValueError(f"ub={ub!r}: int8 activations take no amax bound")
        super().__init__(in_features, out_features, bias=bias, activation=activation, adapter=adapter,
                         register_buffers=register_buffers, **kwargs)

    def _launch(self, x2: torch.Tensor, out: torch.Tensor) -> None:
        (M, K), N = x2.shape, self.out_features
        nws = int(lib.b2q_int8ch_workspace_bytes(M, K))
        ws = torch.empty(nws, dtype=torch.uint8, device=x2.device)
        check(lib.b2q_int8ch_forward(_ptr(x2), _ptr(self.weight), _ptr(self.weight_scale), _ptr(self.input_scale),
                                     _ptr(self._bias.get(x2.dtype)), _ptr(out), M, K, N, _DTYPE_CODE[x2.dtype],
                                     _ptr(ws), nws, torch.cuda.current_stream(x2.device).cuda_stream),
              "b2q_int8ch_forward")

    def extra_repr(self) -> str:
        act = "static per-tensor" if self.activation == "static" else "dynamic per-token"
        return (f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, "
                f"int8 W8A8, per-channel weight scales, {act} activations")
