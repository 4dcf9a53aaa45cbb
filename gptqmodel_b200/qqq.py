"""QQQ (W4A8) checkpoints on the int8 tensor cores: ``B200QqqQuantLinear``.

A QQQ checkpoint (the reference's ``METHOD.QQQ`` / ``FORMAT.QQQ``, gptqmodel/nn_modules/qlinear/qqq.py) stores per module
  ``B``         int32 [K/16, 2N]  4-bit codes in Marlin-QQQ tile order,
  ``s_channel`` fp32  [1, N]      per-output-channel scales (permuted; already divided by 16 for per-channel layers),
  ``s_group``   fp16  [K/128, N]  per-group scales (permuted), empty for per-channel layers,
  ``bias``      fp16  [N]         optional.
``post_init()`` undoes the permutations on the host side of the library (``unpermute_qqq``), checks that every int8 weight
of a group-128 layer is representable, and repacks the canonical codes once into the kernel's tile layout
(``b2q_qqq_prepack``).  ``forward()`` quantises the activations per token to int8 and multiplies on wgmma s8 in one
library call (``b2q_qqq_forward``, include/b2q.h states the arithmetic).  There is no fp16 fallback.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from ._lib import B2QError, check, lib
from .adapter import Lora

_DTYPE_CODE = {torch.float16: 0, torch.bfloat16: 1}
TILE = 16


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


# ---- the Marlin-QQQ permutations (restated from the format's definition) -----------------------------------------------
def qqq_perm(per_channel: bool) -> torch.Tensor:
    """Order of the 1024 nibbles of 8 consecutive [16 x 16] tiles inside the packed words: nibble slot j of a 1024-slot
    row chunk holds tile-major position perm[j].  Per 32-slot run i (a thread's fragment), tile column i // 4 of rows
    4 (i % 4) .. +3, then the same rows 8 columns on; the run repeats for the four 256-slot tiles; finally the 8 slots of
    every word are interleaved so that the kernel's dequantisation reads them in its fragment order."""
    base = []
    for i in range(32):
        rows = [4 * (i % 4) + r for r in range(4)]
        run = [16 * row + i // 4 + 8 * blk for blk in (0, 1) for row in rows]
        for j in range(4):
            base.extend(p + 256 * j for p in run)
    inter = (4, 0, 5, 1, 6, 2, 7, 3) if per_channel else (0, 2, 4, 6, 1, 3, 5, 7)
    t = torch.tensor(base, dtype=torch.int64).view(-1, 8)[:, list(inter)]
    return t.reshape(-1)


def qqq_scale_perm() -> torch.Tensor:
    """Order of the group scales inside each run of 64 columns: the transpose of an 8 x 8 block."""
    return torch.tensor([i + 8 * j for i in range(8) for j in range(8)], dtype=torch.int64)


def qqq_scale_perm_single() -> torch.Tensor:
    """Order of the channel scales inside each run of 32 columns."""
    return torch.tensor([2 * i + j for i in range(4) for j in (0, 1, 8, 9, 16, 17, 24, 25)], dtype=torch.int64)


@torch.no_grad()
def unpermute_qqq(B: torch.Tensor, s_channel: torch.Tensor, s_group: Optional[torch.Tensor], group_size: int):
    """Checkpoint ``B`` / ``s_channel`` / ``s_group`` -> canonical ``codes`` uint8 [K, N] (the 4-bit nibble of w[k, n]),
    ``s_channel`` fp32 [N] and ``s_group`` fp16 [K/128, N] (None for per-channel layers).  Exact; runs on B's device."""
    K, N = B.shape[0] * TILE, B.shape[1] * 8 // TILE
    per_channel = group_size == -1 or group_size == K
    dev = B.device
    words = B.to(torch.int64) & 0xFFFFFFFF
    nib = torch.stack([(words >> (4 * i)) & 0xF for i in range(8)], dim=-1).reshape(K // TILE, N * TILE)
    perm = qqq_perm(per_channel).to(dev)
    tiles = torch.empty_like(nib).view(-1, perm.numel())
    tiles[:, perm] = nib.view(-1, perm.numel())
    codes = tiles.view(K // TILE, N // TILE, TILE, TILE).permute(0, 2, 1, 3).reshape(K, N).to(torch.uint8)
    sp = qqq_scale_perm_single().to(s_channel.device)
    sc = torch.empty_like(s_channel.reshape(-1, sp.numel()))
    sc[:, sp] = s_channel.reshape(-1, sp.numel())
    sc = sc.reshape(N).to(torch.float32).contiguous()
    sg = None
    if not per_channel:
        gp = qqq_scale_perm().to(s_group.device)
        sg = torch.empty_like(s_group.reshape(-1, gp.numel()))
        sg[:, gp] = s_group.reshape(-1, gp.numel())
        sg = sg.reshape(K // 128, N).to(torch.float16).contiguous()
    return codes.contiguous(), sc, sg


class B200QqqQuantLinear(nn.Module):
    """QQQ QuantLinear (the reference's ``QQQLinear`` class contract) on the sm_90a int8 wgmma kernels."""

    SUPPORTS_BACKENDS = ["b200"]
    SUPPORTS_METHODS = ["qqq"]
    SUPPORTS_FORMATS = {"qqq": 110}  # > QQQLinear 100 / QQQTorchLinear 90
    SUPPORTS_BITS = [4]
    SUPPORTS_GROUP_SIZE = [-1, 128]
    SUPPORTS_DESC_ACT = [True, False]  # the format carries no g_idx: act-order is already folded into the weights
    SUPPORTS_SYM = [True]
    SUPPORTS_SHARDS = False
    SUPPORTS_TRAINING = False
    SUPPORTS_AUTO_PADDING = False
    SUPPORTS_IN_FEATURES_DIVISIBLE_BY = [64]
    SUPPORTS_OUT_FEATURES_DIVISIBLE_BY = [64]
    IN_OUTPUT_FEATURES_DIVISIBLE_BY = [(128, 64), (64, 128)]  # the reference's list, reduced
    SUPPORTS_PACK_DTYPES = [torch.int32]
    SUPPORTS_ADAPTERS = [Lora]
    SUPPORTS_DEVICES = ["cuda"]
    SUPPORTS_PLATFORM = ["linux"]
    SUPPORTS_DTYPES = [torch.float16, torch.bfloat16]
    REQUIRES_FORMAT_V2 = False
    QUANT_TYPE = "b200_qqq"

    def __init__(self, bits: int, group_size: int, desc_act: bool, sym: bool, in_features: int, out_features: int,
                 bias: bool = False, pack_dtype: torch.dtype = torch.int32, adapter=None, register_buffers: bool = True,
                 **kwargs):
        nn.Module.__init__(self)
        ok, err = self.validate(bits=bits, group_size=group_size, desc_act=desc_act, sym=sym, in_features=in_features,
                                out_features=out_features, pack_dtype=pack_dtype, dtype=kwargs.get("dtype"))
        if not ok:
            raise err
        K, N = in_features, out_features
        self.bits, self.sym, self.pack_dtype = bits, sym, pack_dtype
        self.desc_act = bool(desc_act) and group_size != -1
        self.in_features, self.out_features = K, N
        self.group_size = group_size if group_size != -1 else K
        self.requested_group_size = group_size
        self.name = kwargs.get("name") or f"{self.__class__.__module__}.{self.__class__.__qualname__}"
        self.adapter = adapter
        if register_buffers:
            self.register_buffer("B", torch.empty((K // TILE, N * TILE // 8), dtype=torch.int32))
            self.register_buffer("s_channel", torch.empty((1, N), dtype=torch.float32))
            G = K // self.group_size
            self.register_buffer("s_group", torch.empty((G, N) if group_size != -1 else (0,), dtype=torch.float16))
            if bias:
                self.register_buffer("bias", torch.zeros(N, dtype=torch.float16))
            else:
                self.bias = None
        else:
            self.B = self.s_channel = self.s_group = self.bias = None
        self._prepacked = False
        self.packed: Optional[torch.Tensor] = None
        self._sc: Optional[torch.Tensor] = None
        self._sg: Optional[torch.Tensor] = None

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
    def validate(cls, bits: int, group_size: int = -1, desc_act: bool = False, sym: bool = True,
                 in_features: int = None, out_features: int = None, pack_dtype: torch.dtype = None,
                 dtype: Optional[torch.dtype] = None, **_ignored) -> Tuple[bool, Optional[Exception]]:
        """Static parameter check; NotImplementedError means "unsupported here, try the next kernel"."""
        if bits not in cls.SUPPORTS_BITS:
            return False, NotImplementedError(f"{cls.__name__}: bits={bits} not in {cls.SUPPORTS_BITS}")
        if group_size not in cls.SUPPORTS_GROUP_SIZE:
            return False, NotImplementedError(f"{cls.__name__}: group_size={group_size} not in {cls.SUPPORTS_GROUP_SIZE}")
        if sym not in cls.SUPPORTS_SYM:
            return False, NotImplementedError(f"{cls.__name__}: sym={sym} unsupported (symmetric only)")
        if pack_dtype is not None and pack_dtype not in cls.SUPPORTS_PACK_DTYPES:
            return False, NotImplementedError(f"{cls.__name__}: pack_dtype={pack_dtype} unsupported")
        if dtype is not None and dtype not in cls.SUPPORTS_DTYPES:
            return False, NotImplementedError(f"{cls.__name__}: dtype={dtype} unsupported")
        if in_features is not None and out_features is not None:
            K, N = in_features, out_features
            if K <= 0 or N <= 0 or K > 65536 or not any(K % a == 0 and N % b == 0
                                                        for a, b in cls.IN_OUTPUT_FEATURES_DIVISIBLE_BY):
                return False, NotImplementedError(
                    f"{cls.__name__}: in_features={K}, out_features={N} outside the envelope (K % 128 == 0 and "
                    "N % 64 == 0, or K % 64 == 0 and N % 128 == 0; K <= 65536)")
            if group_size == 128 and K % 128 != 0:
                return False, NotImplementedError(f"{cls.__name__}: in_features={K} not a multiple of group_size 128")
        return True, None

    @classmethod
    def validate_device(cls, device) -> None:
        dev = torch.device(device) if not isinstance(device, torch.device) else device
        if dev.type != "cuda":
            raise NotImplementedError(f"{cls.__name__} supports CUDA devices only, got `{dev}`")

    def list_buffers(self) -> List[torch.Tensor]:
        out = [t for t in (self.B, self.s_channel, self.s_group, self.bias) if isinstance(t, torch.Tensor)]
        out += [t for t in (self.packed, self._sc, self._sg) if isinstance(t, torch.Tensor)]
        return out

    # ---- one-time repack ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def post_init(self):
        if self._prepacked:
            return
        dev = self.B.device
        if dev.type != "cuda":
            raise B2QError(f"{self.name}: post_init(): weights must be on a CUDA device (no CPU path)")
        K, N = self.in_features, self.out_features
        gs = self.requested_group_size
        with torch.cuda.device(dev):
            codes, sc, sg = unpermute_qqq(self.B.data, self.s_channel.data.to(dev), None if self.s_group is None
                                          else self.s_group.data.to(dev), gs)
            if sg is not None:
                check_group_range(codes, sg, self.name)
            # group_size == in_features is the per-channel format (the reference packs it that way)
            kgs = 128 if sg is not None else -1
            packed = torch.empty(lib.b2q_qqq_packed_bytes(K, N), dtype=torch.uint8, device=dev)
            check(lib.b2q_qqq_prepack(_ptr(codes), _ptr(packed), K, N, kgs,
                                      torch.cuda.current_stream(dev).cuda_stream), "b2q_qqq_prepack")
        self.packed, self._sc, self._sg, self._kgs = packed, sc, sg, kgs
        if self.bias is not None:
            self.bias = self.bias.to(device=dev, dtype=torch.float16).contiguous()
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
        if x.device != self.packed.device:
            raise B2QError(f"input on {x.device} but weights on {self.packed.device}")
        out_shape = x.shape[:-1] + (N,)
        x2 = x.reshape(-1, K)
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        M = x2.shape[0]
        # the adapter sees the fp16 output and the fp16 activations, before the cast back (QQQLinear.forward)
        out_dtype = torch.float16 if self.adapter else x.dtype
        out = torch.empty((M, N), dtype=out_dtype, device=x.device)
        if M == 0:
            return out.to(x.dtype).reshape(out_shape)
        ws = torch.empty(lib.b2q_qqq_workspace_bytes(M, K), dtype=torch.uint8, device=x.device)
        check(lib.b2q_qqq_forward(_ptr(x2), _ptr(self.packed), _ptr(self._sc), _ptr(self._sg), _ptr(self.bias),
                                  _ptr(out), M, K, N, self._kgs, _DTYPE_CODE[x.dtype],
                                  _DTYPE_CODE[out_dtype], _ptr(ws), ws.numel(),
                                  torch.cuda.current_stream(x.device).cuda_stream), "b2q_qqq_forward")
        out = out.reshape(out_shape)
        if self.adapter:
            a = x2 if x2.dtype == torch.float16 else x2.to(torch.float16)
            out = self.adapter.apply(x=a, out=out).to(x.dtype)
        return out

    # ---- helpers --------------------------------------------------------------------------------------------------
    @classmethod
    def from_checkpoint_tensors(cls, B, s_channel, s_group, group_size: int, bias=None, device="cuda", dtype=None,
                                post_init: bool = True):
        """Build (and post_init) a module from checkpoint-layout QQQ tensors."""
        K, N = B.shape[0] * TILE, B.shape[1] * 8 // TILE
        m = cls(bits=4, group_size=group_size, desc_act=False, sym=True, in_features=K, out_features=N,
                bias=bias is not None, register_buffers=False, dtype=dtype)
        cp = lambda t: t.detach().clone().contiguous().to(device)  # noqa: E731
        m.B, m.s_channel = cp(B), cp(s_channel).to(torch.float32)
        m.s_group = cp(s_group).to(torch.float16) if s_group is not None else torch.empty(0, dtype=torch.float16,
                                                                                          device=device)
        m.bias = cp(bias).to(torch.float16) if bias is not None else None
        if post_init:
            m.post_init()
        return m

    def extra_repr(self) -> str:
        return (f"in_features={self.in_features}, out_features={self.out_features}, bits=4, "
                f"group_size={self.requested_group_size}, qqq (W4A8)")


@torch.no_grad()
def check_group_range(codes: torch.Tensor, s_group: torch.Tensor, name: str = "qqq") -> None:
    """Every int8 weight round_half_even((code - 8) * s) of a group-128 layer must lie in [-128, 127]: outside it the
    reference's CUDA path wraps and its torch path clamps, so no answer would be the reference's.  Raises ValueError."""
    K, N = codes.shape
    c = codes.view(K // 128, 128, N)
    d_lo = c.amin(1).to(torch.float32) - 8.0
    d_hi = c.amax(1).to(torch.float32) - 8.0
    s = s_group.to(torch.float32)
    if not bool(torch.isfinite(s).all()):
        raise ValueError(f"{name}: s_group has non-finite entries")
    w = torch.stack([(d_lo * s).round(), (d_hi * s).round()])
    lo, hi = float(w.min()), float(w.max())
    if lo < -128 or hi > 127:
        raise ValueError(f"{name}: a group-128 weight (code - 8) * s_group rounds to {lo if lo < -128 else hi}, outside "
                         "int8 [-128, 127]")
