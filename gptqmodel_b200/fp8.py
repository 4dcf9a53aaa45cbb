"""FP8 (e4m3fn, W8A16) checkpoints on the 8-bit tiers: ``B200Fp8QuantLinear``.

An FP8 checkpoint (the reference's ``METHOD.FP8`` / ``FORMAT.FP8``, gptqmodel/nn_modules/qlinear/fp8.py) stores per
module
  ``weight``            float8_e4m3fn [N, K],
  ``weight_scale_inv``  fp32: [] (tensor), [N] (row) or [N / br, K / bc] (block [br, bc]),
  ``bias``              optional.
The layer computes ``out = T(x @ W) + bias`` with ``W[k, n] = T(w[n, k]) / T(scale_inv[blk(n, k)])`` (one correctly
rounded division per weight, T = the activations' fp16 / bf16): the reference's dequantise-then-matmul arithmetic.  The
reference sends tensor-scaled layers through ``torch._scaled_mm`` on CUDA instead (fp8 activations); this module keeps
the 16-bit activations for every scale layout.

``post_init()`` packs the e4m3 bytes like an 8-bit GPTQ ``qweight`` and repacks them once with ``b2q_prepack``; the
scales become ``[K / g, N]`` tables in fp16 and bf16 (g = bc, or K for row / tensor scales).  ``forward()`` is one
``b2q_fp8_mm`` call (include/b2q.h).  There is no torch fallback.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from ._lib import B2QError, check, lib
from .adapter import Lora

_DTYPE_CODE = {torch.float16: 0, torch.bfloat16: 1}

# the reference's format aliases (quantization/config.py), restated; only e4m3fn is served here
FP8_FORMAT_ALIASES = {
    "e4m3": "float8_e4m3fn", "float8_e4m3": "float8_e4m3fn", "float8_e4m3fn": "float8_e4m3fn",
    "e5m2": "float8_e5m2", "float8_e5m2": "float8_e5m2",
    "e4m3fnuz": "float8_e4m3fnuz", "float8_e4m3fnuz": "float8_e4m3fnuz",
    "e5m2fnuz": "float8_e5m2fnuz", "float8_e5m2fnuz": "float8_e5m2fnuz",
    "e8m0": "float8_e8m0fnu", "e8m0fnu": "float8_e8m0fnu", "float8_e8m0": "float8_e8m0fnu",
    "float8_e8m0fnu": "float8_e8m0fnu",
}
SCALE_METHODS = ("tensor", "row", "block")
BLOCK_COLS = (64, 128)  # group sizes along K the 8-bit tiers read (and K itself)


def normalize_fp8_format(value) -> str:
    """Canonical torch dtype name of an FP8 format alias ("fp8" / None: e4m3fn).  ValueError for an unknown name,
    NotImplementedError for the formats this package does not serve (e5m2, the fnuz formats, e8m0)."""
    name = "float8_e4m3fn" if value is None else str(value).strip().lower()
    if name in ("", "fp8"):
        name = "float8_e4m3fn"
    resolved = FP8_FORMAT_ALIASES.get(name)
    if resolved is None:
        raise ValueError(f"FP8: unsupported `format` `{value}` (one of {', '.join(sorted(FP8_FORMAT_ALIASES))})")
    if resolved != "float8_e4m3fn":
        raise NotImplementedError(f"FP8: format `{resolved}` is not served (float8_e4m3fn only)")
    return resolved


def normalize_block_size(value) -> Optional[Tuple[int, int]]:
    if value is None:
        return None
    if not isinstance(value, (list, tuple)) or len(value) != 2:
        raise ValueError("FP8: `weight_block_size` must be a 2-item list/tuple or None")
    br, bc = int(value[0]), int(value[1])
    if br <= 0 or bc <= 0:
        raise ValueError("FP8: `weight_block_size` entries must be positive integers")
    return br, bc


def normalize_scale_method(value, block_size) -> str:
    """The reference's rule: a block size without a method means "block"; no method means "row"."""
    method = "block" if block_size is not None and value is None else (value or "row")
    method = str(method).strip().lower()
    if method not in SCALE_METHODS:
        raise ValueError(f"FP8: `weight_scale_method` must be one of {SCALE_METHODS}, got `{value}`")
    if method == "block" and block_size is None:
        raise ValueError("FP8: `weight_scale_method='block'` requires `weight_block_size`")
    if method != "block" and block_size is not None:
        raise ValueError("FP8: `weight_block_size` is only valid when `weight_scale_method='block'`")
    return method


def normalize_scale_semantics(value) -> str:
    sem = "inverse" if value is None else str(value).strip().lower()
    if sem != "inverse":
        raise NotImplementedError(f"FP8: `weight_scale_semantics` `{value}` is not served (inverse only: W = w / scale_inv)")
    return sem


def infer_fp8_layout(weight_shape, scale_inv: torch.Tensor) -> Tuple[str, Optional[Tuple[int, int]]]:
    """Scale layout from the shapes of a checkpoint's tensors: one value -> tensor, [N] -> row, [N / br, K / bc] ->
    block [br, bc].  ValueError when the scale tensor fits none of them."""
    N, K = int(weight_shape[0]), int(weight_shape[1])
    if scale_inv.numel() == 1:
        return "tensor", None
    if scale_inv.ndim == 1 and scale_inv.shape[0] == N:
        return "row", None
    if scale_inv.ndim == 2:
        rb, cb = int(scale_inv.shape[0]), int(scale_inv.shape[1])
        if rb > 0 and cb > 0 and N % rb == 0 and K % cb == 0:
            return "block", (N // rb, K // cb)
    raise ValueError(f"FP8: weight_scale_inv of shape {tuple(scale_inv.shape)} fits no scale layout of a "
                     f"[{N}, {K}] weight")


def check_envelope(K: int, N: int, method: str, block_size) -> None:
    """Shapes and block sizes the 8-bit tiers serve; NotImplementedError otherwise."""
    if K <= 0 or N <= 0 or K % 64 != 0 or N % 32 != 0:
        raise NotImplementedError(f"FP8: in_features={K} (multiple of 64), out_features={N} (multiple of 32) unsupported")
    if method == "block":
        br, bc = block_size
        if N % br != 0:
            raise NotImplementedError(f"FP8: block rows {br} must divide out_features={N}")
        if not ((bc in BLOCK_COLS and K % bc == 0) or bc == K):
            raise NotImplementedError(f"FP8: block columns {bc} unsupported for in_features={K} (64 or 128 dividing K, "
                                      "or K)")


# ---- codes <-> the 8-bit qweight word layout ----------------------------------------------------------------------------
def pack_fp8_codes(weight: torch.Tensor) -> torch.Tensor:
    """float8 / uint8 [N, K] -> int32 [K / 4, N]: the byte of row 4i + j (e4m3 bit pattern) in byte j of word [i, n],
    the 8-bit GPTQ qweight layout b2q_prepack reads.  Runs on the tensor's device."""
    codes = weight.view(torch.uint8) if weight.dtype != torch.uint8 else weight
    N, K = codes.shape
    return codes.t().reshape(K // 4, 4, N).permute(0, 2, 1).contiguous().view(torch.int32).reshape(K // 4, N)


def unpack_fp8_codes(qweight: torch.Tensor) -> torch.Tensor:
    """Inverse of pack_fp8_codes: int32 [K / 4, N] -> uint8 [N, K]."""
    K4, N = qweight.shape
    return qweight.contiguous().view(torch.uint8).reshape(K4, N, 4).permute(1, 0, 2).reshape(N, K4 * 4).contiguous()


def expand_scales(scale_inv: torch.Tensor, N: int, K: int, method: str, block_size, dtype: torch.dtype):
    """scale_inv (fp32) -> (table [K / g, N] of dtype, g): each scale rounded to `dtype` first, then repeated over the
    output rows of its block (the reference's order)."""
    s = scale_inv.to(dtype)
    if method == "tensor":
        return s.reshape(1, 1).expand(1, N).contiguous(), K
    if method == "row":
        return s.reshape(1, N).contiguous(), K
    br, bc = block_size
    return s.reshape(N // br, K // bc).repeat_interleave(br, dim=0).t().contiguous(), bc


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _aligned(t: torch.Tensor) -> torch.Tensor:
    t = t if t.is_contiguous() else t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


class B200Fp8QuantLinear(nn.Module):
    """FP8 QuantLinear (the reference's ``TorchFP8Linear`` constructor and buffers) on the sm_90a 8-bit tiers."""

    SUPPORTS_BACKENDS = ["b200"]
    SUPPORTS_METHODS = ["fp8"]
    SUPPORTS_FORMATS = {"fp8": 20}  # > TorchFP8Linear 15
    SUPPORTS_BITS = [8]
    SUPPORTS_SHARDS = False
    SUPPORTS_TRAINING = False
    SUPPORTS_AUTO_PADDING = False
    SUPPORTS_IN_FEATURES_DIVISIBLE_BY = [64]
    SUPPORTS_OUT_FEATURES_DIVISIBLE_BY = [32]
    SUPPORTS_PACK_DTYPES = [torch.int8, torch.int16, torch.int32, torch.int64]
    SUPPORTS_ADAPTERS = [Lora]
    SUPPORTS_DEVICES = ["cuda"]
    SUPPORTS_PLATFORM = ["linux"]
    SUPPORTS_DTYPES = [torch.float16, torch.bfloat16]
    QUANT_TYPE = "b200_fp8"

    def __init__(self, bits: int, group_size: int, sym: bool, desc_act: bool, in_features: int, out_features: int,
                 bias: bool = False, pack_dtype: torch.dtype = torch.int32, adapter=None, register_buffers: bool = True,
                 format: str = "float8_e4m3fn", weight_scale_method: str = "row",
                 weight_block_size: Optional[Tuple[int, int]] = None, weight_scale_semantics: str = "inverse", **kwargs):
        nn.Module.__init__(self)
        self.fp8_format = normalize_fp8_format(format)
        block = normalize_block_size(weight_block_size)
        self.weight_scale_method = normalize_scale_method(weight_scale_method, block)
        self.weight_block_size = block
        self.weight_scale_semantics = normalize_scale_semantics(weight_scale_semantics)
        ok, err = self.validate(bits=bits, in_features=in_features, out_features=out_features, pack_dtype=pack_dtype,
                                dtype=kwargs.get("dtype"), weight_scale_method=self.weight_scale_method,
                                weight_block_size=block)
        if not ok:
            raise err
        self.bits, self.group_size, self.sym, self.desc_act, self.pack_dtype = 8, -1, True, False, pack_dtype
        self.in_features, self.out_features = in_features, out_features
        self.name = kwargs.get("name") or f"{self.__class__.__module__}.{self.__class__.__qualname__}"
        self.adapter = adapter
        if register_buffers:
            self.register_buffer("weight", torch.zeros((out_features, in_features), dtype=torch.float8_e4m3fn))
            self.register_buffer("weight_scale_inv", torch.ones(self._scale_shape(), dtype=torch.float32))
            if bias:
                self.register_buffer("bias", torch.zeros(out_features, dtype=torch.float16))
            else:
                self.bias = None
        else:
            self.weight = self.weight_scale_inv = self.bias = None
        self._prepacked = False
        self.packed: Optional[torch.Tensor] = None
        self._scales = {}
        self._bias = {}
        self._gs = in_features
        self._fp16_ok = True

    def _scale_shape(self) -> tuple:
        if self.weight_scale_method == "tensor":
            return ()
        if self.weight_scale_method == "row":
            return (self.out_features,)
        br, bc = self.weight_block_size
        return (self.out_features // br, self.in_features // bc)

    # ---- validation -----------------------------------------------------------------------------------------------
    @classmethod
    def validate_once(cls) -> Tuple[bool, Optional[Exception]]:
        if not torch.cuda.is_available():
            return False, NotImplementedError(f"{cls.__name__} needs a CUDA device")
        major, minor = torch.cuda.get_device_capability()
        if (major, minor) != (9, 0):
            return False, NotImplementedError(f"{cls.__name__} is built for sm_90a only, found sm_{major}{minor}")
        return True, None

    @classmethod
    def validate(cls, bits: int = 8, in_features: int = None, out_features: int = None, pack_dtype: torch.dtype = None,
                 dtype: Optional[torch.dtype] = None, weight_scale_method: str = "row", weight_block_size=None,
                 **_ignored) -> Tuple[bool, Optional[Exception]]:
        """Static parameter check; NotImplementedError means "unsupported here, try the next kernel"."""
        if bits not in cls.SUPPORTS_BITS:
            return False, NotImplementedError(f"{cls.__name__}: bits={bits} not in {cls.SUPPORTS_BITS}")
        if pack_dtype is not None and pack_dtype not in cls.SUPPORTS_PACK_DTYPES:
            return False, NotImplementedError(f"{cls.__name__}: pack_dtype={pack_dtype} unsupported")
        if dtype is not None and dtype not in cls.SUPPORTS_DTYPES:
            return False, NotImplementedError(f"{cls.__name__}: dtype={dtype} unsupported")
        if in_features is not None and out_features is not None:
            try:
                check_envelope(in_features, out_features, weight_scale_method, weight_block_size)
            except NotImplementedError as e:
                return False, NotImplementedError(f"{cls.__name__}: {e}")
        return True, None

    @classmethod
    def validate_device(cls, device) -> None:
        dev = torch.device(device) if not isinstance(device, torch.device) else device
        if dev.type != "cuda":
            raise NotImplementedError(f"{cls.__name__} supports CUDA devices only, got `{dev}`")

    def list_buffers(self) -> List[torch.Tensor]:
        out = [t for t in (self.weight, self.weight_scale_inv, self.bias) if isinstance(t, torch.Tensor)]
        out += [t for t in (self.packed, *self._scales.values(), *self._bias.values()) if isinstance(t, torch.Tensor)]
        return out

    # ---- one-time repack ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def post_init(self):
        if self._prepacked:
            return
        dev = self.weight.device
        if dev.type != "cuda":
            raise B2QError(f"{self.name}: post_init(): weights must be on a CUDA device (no CPU path)")
        if self.weight.dtype not in (torch.float8_e4m3fn, torch.uint8):
            raise NotImplementedError(f"{self.name}: weight dtype {self.weight.dtype} is not float8_e4m3fn")
        K, N = self.in_features, self.out_features
        if tuple(self.weight.shape) != (N, K) or tuple(self.weight_scale_inv.shape) != self._scale_shape():
            raise ValueError(f"{self.name}: weight {tuple(self.weight.shape)} / weight_scale_inv "
                             f"{tuple(self.weight_scale_inv.shape)} do not match [{N}, {K}] / {self._scale_shape()}")
        with torch.cuda.device(dev):
            qweight = pack_fp8_codes(self.weight.data)
            packed = torch.empty(int(lib.b2q_packed_bytes(K, N, 8)), dtype=torch.uint8, device=dev)
            check(lib.b2q_prepack(_ptr(qweight), None, _ptr(packed), K, N, 8, torch.cuda.current_stream(dev).cuda_stream),
                  "b2q_prepack")
            sinv = self.weight_scale_inv.data.to(device=dev, dtype=torch.float32)
            for dt in _DTYPE_CODE:
                self._scales[dt], self._gs = expand_scales(sinv, N, K, self.weight_scale_method, self.weight_block_size,
                                                           dt)
                if self.bias is not None:
                    self._bias[dt] = self.bias.data.to(device=dev, dtype=dt).contiguous()
            # a scale_inv above 65504 is inf in fp16: the reference then silently computes zero weights; fp16 inputs are
            # refused instead (checked here once, so forward() never synchronises)
            self._fp16_ok = bool(torch.isfinite(self._scales[torch.float16]).all())
        self.packed = packed
        self._prepacked = True
        if self.adapter is not None and hasattr(self.adapter, "post_init"):
            self.adapter.post_init(weight_key=self.name, device=dev,
                                   lora_A=getattr(self, "lora_A", None), lora_B=getattr(self, "lora_B", None))

    # ---- hot path -------------------------------------------------------------------------------------------------
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not self._prepacked:
            raise B2QError(f"{self.name}: forward() before post_init()")
        K, N = self.in_features, self.out_features
        if x.shape[-1] != K:
            raise ValueError(f"expected last dim {K}, got {x.shape[-1]}")
        if x.dtype not in _DTYPE_CODE:
            raise B2QError(f"{self.__class__.__name__} supports fp16/bf16 activations, got {x.dtype}")
        if x.dtype == torch.float16 and not self._fp16_ok:
            raise ValueError(f"{self.name}: a weight_scale_inv overflows fp16 (> 65504): fp16 activations would give "
                             "zero weights; run this layer in bf16")
        if x.device != self.packed.device:
            raise B2QError(f"input on {x.device} but weights on {self.packed.device}")
        out_shape = x.shape[:-1] + (N,)
        x2 = _aligned(x.reshape(-1, K))
        M = x2.shape[0]
        out = torch.empty((M, N), dtype=x.dtype, device=x.device)
        if M > 0:
            check(lib.b2q_fp8_mm(_ptr(x2), _ptr(self.packed), _ptr(self._scales[x.dtype]), _ptr(self._bias.get(x.dtype)),
                                 _ptr(out), M, K, N, self._gs, _DTYPE_CODE[x.dtype], None, 0,
                                 torch.cuda.current_stream(x.device).cuda_stream), "b2q_fp8_mm")
        if self.adapter:
            out = self.adapter.apply(x=x2, out=out)
        return out.reshape(out_shape)

    @torch.no_grad()
    def dequantize_weight(self, device=None, dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """W [K, N] in fp16 (default) or bf16: exactly the operand the tensor-core tiers multiply (b2q_fp8_dequant)."""
        if not self._prepacked:
            raise B2QError(f"{self.name}: dequantize_weight() before post_init()")
        dtype = torch.float16 if dtype is None else dtype
        if dtype not in _DTYPE_CODE:
            raise NotImplementedError(f"{self.name}: dequantize_weight() computes fp16 or bf16 weights, not {dtype}")
        K, N = self.in_features, self.out_features
        dev = self.packed.device
        out = torch.empty((K, N), dtype=dtype, device=dev)
        check(lib.b2q_fp8_dequant(_ptr(self.packed), _ptr(self._scales[dtype]), _ptr(out), K, N, self._gs,
                                  _DTYPE_CODE[dtype], torch.cuda.current_stream(dev).cuda_stream), "b2q_fp8_dequant")
        return out if device is None else out.to(device)

    # ---- helpers --------------------------------------------------------------------------------------------------
    @classmethod
    def from_checkpoint_tensors(cls, weight, weight_scale_inv, bias=None, weight_scale_method: Optional[str] = None,
                                weight_block_size=None, format: str = "float8_e4m3fn", device="cuda", dtype=None,
                                adapter=None, post_init: bool = True, name: Optional[str] = None):
        """Build (and post_init) a module from checkpoint tensors; the scale layout is inferred from the shapes when
        `weight_scale_method` is None, and must agree with it otherwise."""
        method, block = infer_fp8_layout(weight.shape, weight_scale_inv)
        if weight_scale_method is not None:
            want_block = normalize_block_size(weight_block_size)
            want = normalize_scale_method(weight_scale_method, want_block)
            if (want, want_block) != (method, block):
                raise ValueError(f"FP8: weight_scale_inv {tuple(weight_scale_inv.shape)} is a {method} layout "
                                 f"{block or ''}, the config says {want} {want_block or ''}")
        N, K = weight.shape
        m = cls(bits=8, group_size=-1, sym=True, desc_act=False, in_features=K, out_features=N, bias=bias is not None,
                register_buffers=False, format=format, weight_scale_method=method, weight_block_size=block, dtype=dtype,
                adapter=adapter, name=name)
        m.weight = weight.detach().contiguous().to(device)
        m.weight_scale_inv = weight_scale_inv.detach().to(device=device, dtype=torch.float32).reshape(m._scale_shape())
        m.bias = None if bias is None else bias.detach().to(device)
        if post_init:
            m.post_init()
        return m

    def extra_repr(self) -> str:
        return (f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, "
                f"format={self.fp8_format}, weight_scale_method={self.weight_scale_method}"
                + (f", weight_block_size={self.weight_block_size}" if self.weight_block_size else ""))
