"""W4AFP8 checkpoints on the e4m3 tensor cores: ``B200W4Fp8Linear``.

compressed-tensors ``W4AFP8`` checkpoints (llm-compressor, ``format: pack-quantized``) store per module
  ``weight_packed``  int32 [N, K/8]: the code q + 8 of weight q in [-8, 7] at bits 4 (k % 8) of word k / 8,
  ``weight_scale``   [N, K/128] in the model dtype, one scale per 128 k (symmetric: no zero point),
  ``weight_shape``   [2] = (N, K),
  ``bias``           optional,
and quantise the activations to e4m3 per token, dynamically.  ``forward()`` runs the per-token quantiser of the
per-channel FP8 layer and a GEMM that multiplies e4m3 codes by the 4-bit weights (exact in e4m3) on the tensor cores and
applies each group scale in fp32 to its 128-k block's partial sum (``b2q_w4afp8_forward``; include/b2q.h states the
arithmetic).  ``post_init()`` repacks ``weight_packed`` into the kernel's tile layout in one device pass and keeps the
scales as fp32 [K/128, N]; afterwards the module holds no other copy of the weights.  There is no torch fallback.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn

from ._lib import B2QError, check, lib
from .adapter import Lora
from .fp8_block import _DTYPE_CODE, _aligned, _ptr

GROUP = 128
SCALE_DTYPES = (torch.float32, torch.bfloat16, torch.float16)
# nibble p of a tile word holds k0 + NIBBLE_K[p] (b2q_w4afp8.cu); the map is its own inverse
NIBBLE_K = (0, 1, 4, 5, 2, 3, 6, 7)


def check_envelope(K: int, N: int) -> None:
    """Shapes the W4AFP8 kernels serve; NotImplementedError otherwise."""
    if K <= 0 or N <= 0 or K % GROUP != 0 or K > 65536 or N % 128 != 0:
        raise NotImplementedError(f"W4AFP8: in_features={K} (multiple of 128, <= 65536), out_features={N} "
                                  "(multiple of 128) unsupported")


def unpack_codes(weight_packed: torch.Tensor) -> torch.Tensor:
    """weight_packed int32 [N, K/8] -> the stored codes c = q + 8 as uint8 [N, K] (compressed-tensors' packing)."""
    w = weight_packed.to(torch.int32)
    shifts = torch.arange(0, 32, 4, dtype=torch.int32, device=w.device)
    return ((w[:, :, None] >> shifts) & 15).to(torch.uint8).reshape(w.shape[0], -1)


def tile_codes(packed: torch.Tensor, K: int, N: int) -> torch.Tensor:
    """The inverse of b2q_w4afp8_prepack: the kernel's tiles (uint8, K * N / 2 bytes) -> codes c uint8 [N, K]."""
    KB = K // GROUP
    words = packed.view(torch.int32).reshape(N // 128, KB, 4, 128, 4)  # [tile row][k-block][quad][feature][word]
    shifts = torch.arange(0, 32, 4, dtype=torch.int32, device=packed.device)
    nib = (words[..., None] >> shifts) & 15                             # [..., nibble p]
    nib = nib[..., list(NIBBLE_K)]                                      # [..., k offset]
    return nib.permute(0, 3, 1, 2, 4, 5).reshape(N, K).to(torch.uint8)


class B200W4Fp8Linear(nn.Module):
    """W4AFP8 linear (checkpoint tensors ``weight_packed``, ``weight_scale``, optional ``bias``) on the sm_90a e4m3
    wgmma kernels, with dynamic per-token e4m3 activations."""

    SUPPORTS_BACKENDS = ["b200"]
    SUPPORTS_METHODS = ["compressed-tensors"]
    SUPPORTS_BITS = [4]
    SUPPORTS_GROUP_SIZE = [GROUP]
    SUPPORTS_SHARDS = False
    SUPPORTS_TRAINING = False
    SUPPORTS_AUTO_PADDING = False
    SUPPORTS_IN_FEATURES_DIVISIBLE_BY = [128]
    SUPPORTS_OUT_FEATURES_DIVISIBLE_BY = [128]
    SUPPORTS_ADAPTERS = [Lora]
    SUPPORTS_DEVICES = ["cuda"]
    SUPPORTS_PLATFORM = ["linux"]
    SUPPORTS_DTYPES = [torch.float16, torch.bfloat16]
    QUANT_TYPE = "b200_w4afp8"

    def __init__(self, in_features: int, out_features: int, bias: bool = False, adapter=None,
                 register_buffers: bool = True, **kwargs):
        nn.Module.__init__(self)
        check_envelope(in_features, out_features)
        dtype = kwargs.get("dtype")
        if dtype is not None and dtype not in self.SUPPORTS_DTYPES:
            raise NotImplementedError(f"{self.__class__.__name__}: dtype={dtype} unsupported")
        self.in_features, self.out_features = in_features, out_features
        self.name = kwargs.get("name") or f"{self.__class__.__module__}.{self.__class__.__qualname__}"
        self.adapter = adapter
        K, N = in_features, out_features
        if register_buffers:
            self.register_buffer("weight_packed", torch.zeros((N, K // 8), dtype=torch.int32))
            self.register_buffer("weight_scale", torch.ones((N, K // GROUP), dtype=torch.float16))
            if bias:
                self.register_buffer("bias", torch.zeros(N, dtype=torch.float16))
            else:
                self.bias = None
        else:
            self.weight_packed = self.weight_scale = self.bias = None
        self.packed = None   # after post_init(): the kernel's tiles (uint8, K * N / 2 bytes)
        self.s_w = None      # after post_init(): fp32 [K/128, N]
        self.scale_dtype = torch.float16  # the checkpoint's scale dtype (dequantize_weight computes in it)
        self._ready = False
        self._bias = {}

    @classmethod
    def validate_device(cls, device) -> None:
        dev = torch.device(device) if not isinstance(device, torch.device) else device
        if dev.type != "cuda":
            raise NotImplementedError(f"{cls.__name__} supports CUDA devices only, got `{dev}`")

    def list_buffers(self) -> List[torch.Tensor]:
        out = [t for t in (self.weight_packed, self.weight_scale, self.packed, self.s_w, self.bias)
               if isinstance(t, torch.Tensor)]
        return out + [t for t in self._bias.values() if isinstance(t, torch.Tensor)]

    def check_tensors(self) -> None:
        """dtype, shape and values of the checkpoint tensors; ValueError when they do not fit."""
        K, N = self.in_features, self.out_features
        wp, ws = self.weight_packed, self.weight_scale
        if wp.dtype != torch.int32 or tuple(wp.shape) != (N, K // 8):
            raise ValueError(f"{self.name}: weight_packed {wp.dtype} {tuple(wp.shape)} is not int32 [{N}, {K // 8}]")
        if ws.dtype not in SCALE_DTYPES or tuple(ws.shape) != (N, K // GROUP):
            raise ValueError(f"{self.name}: weight_scale {ws.dtype} {tuple(ws.shape)} is not fp32 / bf16 / fp16 "
                             f"[{N}, {K // GROUP}]")
        v = ws.float()
        if not bool(torch.isfinite(v).all()) or bool((v < 0).any()):
            raise ValueError(f"{self.name}: weight_scale must be finite and non-negative")
        if self.bias is not None and tuple(self.bias.shape) != (N,):
            raise ValueError(f"{self.name}: bias {tuple(self.bias.shape)} is not [{N}]")

    # ---- one-time set-up ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def post_init(self):
        if self._ready:
            return
        dev = self.weight_packed.device
        if dev.type != "cuda":
            raise B2QError(f"{self.name}: post_init(): weights must be on a CUDA device (no CPU path)")
        self.check_tensors()
        K, N = self.in_features, self.out_features
        src = _aligned(self.weight_packed.data)
        packed = torch.empty(int(lib.b2q_w4afp8_packed_bytes(K, N)), dtype=torch.uint8, device=dev)
        check(lib.b2q_w4afp8_prepack(_ptr(src), _ptr(packed), K, N, torch.cuda.current_stream(dev).cuda_stream),
              "b2q_w4afp8_prepack")
        self.scale_dtype = self.weight_scale.dtype
        self.packed = packed
        self.s_w = _aligned(self.weight_scale.data.to(device=dev, dtype=torch.float32).t().contiguous())
        # the checkpoint tensors are not kept: the tiles and fp32 scales are the module's only copy of the weights
        self.weight_packed = self.weight_scale = None
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
        if x.device != self.packed.device:
            raise B2QError(f"input on {x.device} but weights on {self.packed.device}")
        out_shape = x.shape[:-1] + (N,)
        x2 = _aligned(x.reshape(-1, K))
        M = x2.shape[0]
        out = torch.empty((M, N), dtype=x.dtype, device=x.device)
        if M > 0:
            nws = int(lib.b2q_w4afp8_workspace_bytes(M, K))
            ws = torch.empty(nws, dtype=torch.uint8, device=x2.device)
            check(lib.b2q_w4afp8_forward(_ptr(x2), _ptr(self.packed), _ptr(self.s_w), _ptr(self._bias.get(x2.dtype)),
                                         _ptr(out), M, K, N, _DTYPE_CODE[x2.dtype], _ptr(ws), nws,
                                         torch.cuda.current_stream(x2.device).cuda_stream),
                  "b2q_w4afp8_forward")
        if self.adapter:
            out = self.adapter.apply(x=x2, out=out)
        return out.reshape(out_shape)

    @torch.no_grad()
    def dequantize_weight(self, device=None, dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """W [K, N] = RN_dtype(S(q[n, k]) * S(s[n, k / 128])) computed in the checkpoint's scale dtype S, transposed —
        compressed-tensors' dequantisation T(q * s); fp16 (default) or bf16.  Works before and after post_init()."""
        dtype = torch.float16 if dtype is None else dtype
        if dtype not in _DTYPE_CODE:
            raise NotImplementedError(f"{self.name}: dequantize_weight() computes fp16 or bf16 weights, not {dtype}")
        K, N = self.in_features, self.out_features
        if self._ready:
            codes, s = tile_codes(self.packed, K, N), self.s_w.t()
        else:
            codes, s = unpack_codes(self.weight_packed), self.weight_scale
        sd = self.scale_dtype if self._ready else self.weight_scale.dtype
        q = codes.to(torch.int16) - 8
        s = s.to(device=q.device, dtype=sd).repeat_interleave(GROUP, dim=1)
        out = (q.to(sd) * s).to(dtype).t().contiguous()
        return out if device is None else out.to(device)

    # ---- helpers --------------------------------------------------------------------------------------------------
    @classmethod
    def from_checkpoint_tensors(cls, weight_packed, weight_scale, weight_shape=None, bias=None, device="cuda",
                                dtype=None, adapter=None, post_init: bool = True, name: Optional[str] = None):
        """Build (and post_init) a module from checkpoint tensors.  ValueError / NotImplementedError when the tensors
        do not fit."""
        if weight_packed.dim() != 2 or weight_scale.dim() != 2:
            raise ValueError(f"W4AFP8: weight_packed {tuple(weight_packed.shape)} and weight_scale "
                             f"{tuple(weight_scale.shape)} must be 2-D")
        N, K = int(weight_packed.shape[0]), int(weight_packed.shape[1]) * 8
        if weight_shape is not None:
            shp = tuple(int(v) for v in torch.as_tensor(weight_shape).reshape(-1).tolist())
            if len(shp) != 2 or shp[0] != N or shp[1] > K or shp[1] <= K - 8:
                raise ValueError(f"W4AFP8: weight_shape {shp} does not match weight_packed {tuple(weight_packed.shape)}")
            K = shp[1]
        m = cls(in_features=K, out_features=N, bias=bias is not None, register_buffers=False, dtype=dtype,
                adapter=adapter, name=name)
        m.weight_packed = weight_packed.detach().contiguous().to(device)
        m.weight_scale = weight_scale.detach().contiguous().to(device)
        m.bias = None if bias is None else bias.detach().contiguous().to(device)
        m.check_tensors()
        m.scale_dtype = m.weight_scale.dtype
        if post_init:
            m.post_init()
        return m

    def extra_repr(self) -> str:
        return (f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, "
                "W4AFP8: int4 group-128 weights, dynamic per-token e4m3 activations")
