"""Block-FP8 (W8A8) checkpoints of the HF / DeepSeek-native layout on the e4m3 tensor cores: ``B200BlockFp8Linear``.

These checkpoints (transformers' ``FineGrainedFP8Config``, DeepSeek-V3 / R1, the Qwen3 ``*-FP8`` releases) carry the
config ``{"quant_method": "fp8", "fmt": "e4m3", "activation_scheme": "dynamic", "weight_block_size": [128, 128]}`` and
store per module
  ``weight``            float8_e4m3fn [N, K],
  ``weight_scale_inv``  fp32 [ceil(N / 128), K / 128], which MULTIPLIES the weight despite its name,
  ``bias``              optional.
``forward()`` quantises the activations per token in groups of 128 k to e4m3 and runs a W8A8 GEMM with the scales
promoted once per 128-k block (``b2q_fp8blk_forward``; include/b2q.h states the arithmetic), the scheme of
transformers' ``FP8Linear``.  The checkpoint tensor is the kernel's operand: ``post_init()`` validates and moves the
tensors, it repacks nothing.  There is no torch fallback.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from ._lib import B2QError, check, lib
from .adapter import Lora

_DTYPE_CODE = {torch.float16: 0, torch.bfloat16: 1}
BLOCK = 128


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _aligned(t: torch.Tensor) -> torch.Tensor:
    t = t if t.is_contiguous() else t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def scale_shape(in_features: int, out_features: int) -> Tuple[int, int]:
    """Shape of a layer's ``weight_scale_inv``: one scale per 128 x 128 block, the last row block may be partial."""
    return (out_features + BLOCK - 1) // BLOCK, in_features // BLOCK


def check_envelope(K: int, N: int) -> None:
    """Shapes the block-FP8 kernels serve; NotImplementedError otherwise."""
    if K <= 0 or N <= 0 or K % BLOCK != 0 or K > 65536 or N % 64 != 0:
        raise NotImplementedError(f"block FP8: in_features={K} (multiple of 128, <= 65536), out_features={N} "
                                  "(multiple of 64) unsupported")


class B200BlockFp8Linear(nn.Module):
    """Block-FP8 linear (HF ``FP8Linear`` buffers: ``weight``, ``weight_scale_inv``, ``bias``) on the sm_90a e4m3
    wgmma kernels."""

    SUPPORTS_BACKENDS = ["b200"]
    SUPPORTS_METHODS = ["fp8"]
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
    QUANT_TYPE = "b200_fp8_block"

    def __init__(self, in_features: int, out_features: int, bias: bool = False, adapter=None,
                 register_buffers: bool = True, **kwargs):
        nn.Module.__init__(self)
        check_envelope(in_features, out_features)
        dtype = kwargs.get("dtype")
        if dtype is not None and dtype not in self.SUPPORTS_DTYPES:
            raise NotImplementedError(f"{self.__class__.__name__}: dtype={dtype} unsupported")
        self.in_features, self.out_features = in_features, out_features
        self.weight_block_size = (BLOCK, BLOCK)
        self.name = kwargs.get("name") or f"{self.__class__.__module__}.{self.__class__.__qualname__}"
        self.adapter = adapter
        if register_buffers:
            self.register_buffer("weight", torch.zeros((out_features, in_features), dtype=torch.float8_e4m3fn))
            self.register_buffer("weight_scale_inv", torch.ones(scale_shape(in_features, out_features),
                                                                dtype=torch.float32))
            if bias:
                self.register_buffer("bias", torch.zeros(out_features, dtype=torch.float16))
            else:
                self.bias = None
        else:
            self.weight = self.weight_scale_inv = self.bias = None
        self._ready = False
        self._bias = {}

    @classmethod
    def validate_device(cls, device) -> None:
        dev = torch.device(device) if not isinstance(device, torch.device) else device
        if dev.type != "cuda":
            raise NotImplementedError(f"{cls.__name__} supports CUDA devices only, got `{dev}`")

    def list_buffers(self) -> List[torch.Tensor]:
        out = [t for t in (self.weight, self.weight_scale_inv, self.bias) if isinstance(t, torch.Tensor)]
        return out + [t for t in self._bias.values() if isinstance(t, torch.Tensor)]

    def check_tensors(self) -> None:
        """dtype and shape of the checkpoint tensors; ValueError / NotImplementedError when they do not fit."""
        K, N = self.in_features, self.out_features
        if self.weight.dtype not in (torch.float8_e4m3fn, torch.uint8):
            raise NotImplementedError(f"{self.name}: weight dtype {self.weight.dtype} is not float8_e4m3fn")
        if tuple(self.weight.shape) != (N, K):
            raise ValueError(f"{self.name}: weight {tuple(self.weight.shape)} is not [{N}, {K}]")
        if tuple(self.weight_scale_inv.shape) != scale_shape(K, N):
            raise ValueError(f"{self.name}: weight_scale_inv {tuple(self.weight_scale_inv.shape)} is not the "
                             f"[ceil(N / 128), K / 128] = {list(scale_shape(K, N))} grid of a [{N}, {K}] weight")
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
        self.weight = _aligned(self.weight.data.view(torch.float8_e4m3fn))
        self.weight_scale_inv = _aligned(self.weight_scale_inv.data.to(device=dev, dtype=torch.float32))
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
            nws = int(lib.b2q_fp8blk_workspace_bytes(M, K))
            ws = torch.empty(nws, dtype=torch.uint8, device=x.device) if nws else None
            check(lib.b2q_fp8blk_forward(_ptr(x2), _ptr(self.weight), _ptr(self.weight_scale_inv),
                                         _ptr(self._bias.get(x.dtype)), _ptr(out), M, K, N, _DTYPE_CODE[x.dtype],
                                         _ptr(ws), nws, torch.cuda.current_stream(x.device).cuda_stream),
                  "b2q_fp8blk_forward")
        if self.adapter:
            out = self.adapter.apply(x=x2, out=out)
        return out.reshape(out_shape)

    @torch.no_grad()
    def dequantize_weight(self, device=None, dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """W [K, N] = RN_T(T(w[n, k]) * T(s_w[n / 128, k / 128])), transposed; fp16 (default) or bf16.  Works on the
        CPU tensors of a module that was not post_init()'ed as well."""
        dtype = torch.float16 if dtype is None else dtype
        if dtype not in _DTYPE_CODE:
            raise NotImplementedError(f"{self.name}: dequantize_weight() computes fp16 or bf16 weights, not {dtype}")
        K, N = self.in_features, self.out_features
        w = self.weight.view(torch.float8_e4m3fn).to(dtype)
        s = self.weight_scale_inv.to(dtype).repeat_interleave(BLOCK, 0)[:N].repeat_interleave(BLOCK, 1)
        out = (w * s.to(w.device)).t().contiguous()
        return out if device is None else out.to(device)

    # ---- helpers --------------------------------------------------------------------------------------------------
    @classmethod
    def from_checkpoint_tensors(cls, weight, weight_scale_inv, bias=None, device="cuda", dtype=None, adapter=None,
                                post_init: bool = True, name: Optional[str] = None):
        """Build (and post_init) a module from checkpoint tensors; ValueError when the scale grid does not fit."""
        N, K = weight.shape
        m = cls(in_features=K, out_features=N, bias=bias is not None, register_buffers=False, dtype=dtype,
                adapter=adapter, name=name)
        m.weight = weight.detach().contiguous().to(device)
        m.weight_scale_inv = weight_scale_inv.detach().to(device=device, dtype=torch.float32).contiguous()
        m.bias = None if bias is None else bias.detach().contiguous().to(device)
        m.check_tensors()
        if post_init:
            m.post_init()
        return m

    def extra_repr(self) -> str:
        return (f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, "
                "fp8 e4m3 W8A8, weight_block_size=(128, 128), dynamic per-token-group activations")
