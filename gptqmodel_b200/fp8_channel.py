"""Per-channel / per-tensor FP8 (W8A8) checkpoints on the e4m3 tensor cores: ``B200ChannelFp8Linear``.

These checkpoints store per module
  ``weight``        float8_e4m3fn [N, K],
  ``weight_scale``  [N, 1] / [N] (per channel) or [1] / [] (per tensor), fp32, bf16 or fp16, which MULTIPLIES the weight,
  ``input_scale``   [1] / [] (static activations only),
  ``bias``          optional.
They come from llm-compressor / compressed-tensors (``FP8_DYNAMIC``: channel weights and dynamic per-token activations;
``FP8``: a tensor weight scale and a static ``input_scale``) and transformers' ``fbgemm_fp8`` (channel weights and
per-token activations whose amax is bounded by ``activation_scale_ub``).  ``forward()`` quantises the activations to
e4m3 and runs a W8A8 GEMM whose scales are applied once, after the k-sum (``b2q_fp8ch_forward``; include/b2q.h states
the arithmetic).  The checkpoint weight is the kernel's operand: ``post_init()`` widens the scales to fp32 (exactly) and
broadcasts a per-tensor weight scale to all features, it repacks nothing.  There is no torch fallback.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn

from ._lib import B2QError, check, lib
from .adapter import Lora
from .fp8_block import _DTYPE_CODE, _aligned, _ptr, check_envelope

SCALE_DTYPES = (torch.float32, torch.bfloat16, torch.float16)
KINDS = ("dynamic", "static")


def channel_scales(weight_scale: torch.Tensor, out_features: int) -> torch.Tensor:
    """The kernel's s_w: fp32 [N], one scale per output feature.  fp16 / bf16 -> fp32 is exact; a per-tensor scale
    ([1] or []) is broadcast to every feature."""
    return weight_scale.to(torch.float32).reshape(-1).expand(out_features).contiguous()


class ChannelW8A8Linear(nn.Module):
    """The module contract shared by the per-channel 8-bit W8A8 layers (buffers ``weight`` [N, K] of CODE_DTYPE codes,
    ``weight_scale``, ``input_scale``, ``bias``).  A subclass names its code dtype and runs its forward ABI call."""

    CODE_DTYPE: torch.dtype       # the weight codes the kernels read
    WEIGHT_DTYPES: tuple = ()     # checkpoint weight dtypes accepted (viewed as CODE_DTYPE)

    SUPPORTS_BACKENDS = ["b200"]
    SUPPORTS_BITS = [8]
    SUPPORTS_SHARDS = False
    SUPPORTS_TRAINING = False
    SUPPORTS_AUTO_PADDING = False
    SUPPORTS_IN_FEATURES_DIVISIBLE_BY = [128]
    SUPPORTS_OUT_FEATURES_DIVISIBLE_BY = [64]
    SUPPORTS_ADAPTERS = [Lora]
    SUPPORTS_DEVICES = ["cuda"]
    SUPPORTS_PLATFORM = ["linux"]
    SUPPORTS_DTYPES = [torch.float16, torch.bfloat16]

    def __init__(self, in_features: int, out_features: int, bias: bool = False, activation: str = "dynamic",
                 ub: Optional[float] = None, adapter=None, register_buffers: bool = True, **kwargs):
        nn.Module.__init__(self)
        check_envelope(in_features, out_features)
        dtype = kwargs.get("dtype")
        if dtype is not None and dtype not in self.SUPPORTS_DTYPES:
            raise NotImplementedError(f"{self.__class__.__name__}: dtype={dtype} unsupported")
        if activation not in KINDS:
            raise ValueError(f"activation must be one of {KINDS}, got {activation!r}")
        if ub is not None and (activation != "dynamic" or not (float(ub) > 0.0)):
            raise ValueError(f"ub={ub!r}: a positive amax bound of dynamic activations")
        self.in_features, self.out_features = in_features, out_features
        self.activation, self.ub = activation, None if ub is None else float(ub)
        self.name = kwargs.get("name") or f"{self.__class__.__module__}.{self.__class__.__qualname__}"
        self.adapter = adapter
        if register_buffers:
            self.register_buffer("weight", torch.zeros((out_features, in_features), dtype=self.CODE_DTYPE))
            self.register_buffer("weight_scale", torch.ones((out_features, 1), dtype=torch.float32))
            if activation == "static":
                self.register_buffer("input_scale", torch.ones(1, dtype=torch.float32))
            else:
                self.input_scale = None
            if bias:
                self.register_buffer("bias", torch.zeros(out_features, dtype=torch.float16))
            else:
                self.bias = None
        else:
            self.weight = self.weight_scale = self.input_scale = self.bias = None
        self.scale_dtype = torch.float32  # the checkpoint's scale dtype (dequantize_weight computes in it)
        self._ready = False
        self._bias = {}

    @classmethod
    def validate_device(cls, device) -> None:
        dev = torch.device(device) if not isinstance(device, torch.device) else device
        if dev.type != "cuda":
            raise NotImplementedError(f"{cls.__name__} supports CUDA devices only, got `{dev}`")

    def list_buffers(self) -> List[torch.Tensor]:
        out = [t for t in (self.weight, self.weight_scale, self.input_scale, self.bias) if isinstance(t, torch.Tensor)]
        return out + [t for t in self._bias.values() if isinstance(t, torch.Tensor)]

    def check_tensors(self) -> None:
        """dtype, shape and values of the checkpoint tensors; ValueError / NotImplementedError when they do not fit."""
        K, N = self.in_features, self.out_features
        if self.weight.dtype not in self.WEIGHT_DTYPES:
            raise NotImplementedError(f"{self.name}: weight dtype {self.weight.dtype} is not "
                                      f"{str(self.CODE_DTYPE).replace('torch.', '')}")
        if tuple(self.weight.shape) != (N, K):
            raise ValueError(f"{self.name}: weight {tuple(self.weight.shape)} is not [{N}, {K}]")
        ws = self.weight_scale
        if tuple(ws.shape) not in ((N, 1), (N,), (1,), ()):
            raise ValueError(f"{self.name}: weight_scale {tuple(ws.shape)} is not [{N}, 1], [{N}], [1] or []")
        if self.activation == "static":
            if self.input_scale is None:
                raise NotImplementedError(f"{self.name}: static activations need an `input_scale`")
            if tuple(self.input_scale.shape) not in ((1,), ()):
                raise ValueError(f"{self.name}: input_scale {tuple(self.input_scale.shape)} is not [1] or []")
        elif self.input_scale is not None:
            raise NotImplementedError(f"{self.name}: an `input_scale` on a layer with dynamic activations")
        for what, t in (("weight_scale", ws), ("input_scale", self.input_scale)):
            if t is None:
                continue
            if t.dtype not in SCALE_DTYPES:
                raise ValueError(f"{self.name}: {what} dtype {t.dtype} is not fp32, bf16 or fp16")
            v = t.float()
            if not bool(torch.isfinite(v).all()) or not bool((v > 0).all()):
                raise ValueError(f"{self.name}: {what} must be finite and positive")
        if self.bias is not None and tuple(self.bias.shape) != (N,):
            raise ValueError(f"{self.name}: bias {tuple(self.bias.shape)} is not [{N}]")

    # ---- one-time set-up ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def post_init(self):
        if self._ready:
            return
        dev = self.weight.device
        if dev.type != "cuda":
            raise B2QError(f"{self.name}: post_init(): weights must be on a CUDA device (no CPU path)")
        self.check_tensors()
        N = self.out_features
        self.scale_dtype = self.weight_scale.dtype
        self.weight = _aligned(self.weight.data.view(self.CODE_DTYPE))
        self.weight_scale = _aligned(channel_scales(self.weight_scale.data.to(dev), N))
        if self.input_scale is not None:
            self.input_scale = _aligned(self.input_scale.data.to(device=dev, dtype=torch.float32).reshape(1))
        if self.bias is not None:
            for dt in _DTYPE_CODE:
                self._bias[dt] = self.bias.data.to(device=dev, dtype=dt).contiguous()
        self._ready = True
        if self.adapter is not None and hasattr(self.adapter, "post_init"):
            self.adapter.post_init(weight_key=self.name, device=dev,
                                   lora_A=getattr(self, "lora_A", None), lora_B=getattr(self, "lora_B", None))

    # ---- hot path -------------------------------------------------------------------------------------------------
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not self._ready:
            raise B2QError(f"{self.name}: forward() before post_init()")
        K, N = self.in_features, self.out_features
        if x.shape[-1] != K:
            raise ValueError(f"expected last dim {K}, got {x.shape[-1]}")
        if x.dtype not in _DTYPE_CODE:
            raise B2QError(f"{self.__class__.__name__} supports fp16/bf16 activations, got {x.dtype}")
        if x.device != self.weight.device:
            raise B2QError(f"input on {x.device} but weights on {self.weight.device}")
        out_shape = x.shape[:-1] + (N,)
        x2 = _aligned(x.reshape(-1, K))
        M = x2.shape[0]
        out = torch.empty((M, N), dtype=x.dtype, device=x.device)
        if M > 0:
            self._launch(x2, out)
        if self.adapter:
            out = self.adapter.apply(x=x2, out=out)
        return out.reshape(out_shape)

    @torch.no_grad()
    def dequantize_weight(self, device=None, dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """W [K, N] = RN_dtype(S(w[n, k]) * s_w[n]) computed in the checkpoint's scale dtype S, transposed — the
        arithmetic of compressed-tensors' dequantiser; fp16 (default) or bf16.  Works on the CPU tensors of a module
        that was not post_init()'ed as well."""
        dtype = torch.float16 if dtype is None else dtype
        if dtype not in _DTYPE_CODE:
            raise NotImplementedError(f"{self.name}: dequantize_weight() computes fp16 or bf16 weights, not {dtype}")
        sd = self.scale_dtype if self._ready else self.weight_scale.dtype
        w = self.weight.view(self.CODE_DTYPE)
        s = self.weight_scale.to(device=w.device, dtype=sd).reshape(-1)
        s = s[:, None] if s.numel() > 1 else s.reshape(())
        out = (w.to(sd) * s).to(dtype).t().contiguous()
        return out if device is None else out.to(device)

    # ---- helpers --------------------------------------------------------------------------------------------------
    @classmethod
    def from_checkpoint_tensors(cls, weight, weight_scale, input_scale=None, bias=None, activation: Optional[str] = None,
                                ub: Optional[float] = None, device="cuda", dtype=None, adapter=None,
                                post_init: bool = True, name: Optional[str] = None):
        """Build (and post_init) a module from checkpoint tensors.  ``activation`` defaults to "static" when an
        ``input_scale`` is given, else "dynamic".  ValueError / NotImplementedError when the tensors do not fit."""
        N, K = weight.shape
        activation = activation or ("static" if input_scale is not None else "dynamic")
        m = cls(in_features=K, out_features=N, bias=bias is not None, activation=activation, ub=ub,
                register_buffers=False, dtype=dtype, adapter=adapter, name=name)
        m.weight = weight.detach().contiguous().to(device)
        m.weight_scale = weight_scale.detach().contiguous().to(device)
        m.input_scale = None if input_scale is None else input_scale.detach().contiguous().to(device)
        m.bias = None if bias is None else bias.detach().contiguous().to(device)
        m.check_tensors()
        m.scale_dtype = m.weight_scale.dtype
        if post_init:
            m.post_init()
        return m


class B200ChannelFp8Linear(ChannelW8A8Linear):
    """Per-channel / per-tensor FP8 linear (buffers ``weight``, ``weight_scale``, ``input_scale``, ``bias``) on the
    sm_90a e4m3 wgmma kernels.  ``activation``: "dynamic" (per-token scales, optionally bounded by ``ub``) or
    "static" (the per-tensor ``input_scale``)."""

    CODE_DTYPE = torch.float8_e4m3fn
    WEIGHT_DTYPES = (torch.float8_e4m3fn, torch.uint8)
    SUPPORTS_METHODS = ["compressed-tensors", "fbgemm_fp8"]
    QUANT_TYPE = "b200_fp8_channel"

    def _launch(self, x2: torch.Tensor, out: torch.Tensor) -> None:
        (M, K), N = x2.shape, self.out_features
        nws = int(lib.b2q_fp8ch_workspace_bytes(M, K))
        ws = torch.empty(nws, dtype=torch.uint8, device=x2.device) if nws else None
        ub = float("inf") if self.ub is None else self.ub
        check(lib.b2q_fp8ch_forward(_ptr(x2), _ptr(self.weight), _ptr(self.weight_scale), _ptr(self.input_scale),
                                    ub, _ptr(self._bias.get(x2.dtype)), _ptr(out), M, K, N, _DTYPE_CODE[x2.dtype],
                                    _ptr(ws), nws, torch.cuda.current_stream(x2.device).cuda_stream),
              "b2q_fp8ch_forward")

    def extra_repr(self) -> str:
        act = "static per-tensor" if self.activation == "static" else "dynamic per-token"
        ub = "" if self.ub is None else f" (amax <= {self.ub:g})"
        return (f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, "
                f"fp8 e4m3 W8A8, per-channel weight scales, {act} activations{ub}")
