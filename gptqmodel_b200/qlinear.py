"""B200QuantLinear — drop-in GPTQ QuantLinear whose forward() runs hand-written sm_90a (H100) CUDA.

Mirrors the class contract of the reference's kernels:
  constructor / buffers : gptqmodel/nn_modules/qlinear/__init__.py:664-692, 827-865 (qweight, qzeros, scales, g_idx,
                          bias in CHECKPOINT layout so a loader can fill them), qlinear/swordfish.py:66-148
  capability attributes : qlinear/swordfish.py:40-62 / qlinear/marlin.py:59-75 (`SUPPORTS_*`, REQUIRES_FORMAT_V2)
  validate()/validate_once() -> (ok, err), NotImplementedError = "try the next kernel" (utils/model.py:703-707)
  post_init()           : one-time repack after the weights are on the device (qlinear/marlin.py:246-293)
  forward(x)            : x [..., K] fp16/bf16 -> [..., N] same dtype, bias added, adapter applied
                          (qlinear/swordfish.py:305-355, qlinear/torch.py:302-347)

The module is stand-alone (no import of the reference package); INTEGRATION.md shows the 20-line file a
maintainer drops into gptqmodel/nn_modules/qlinear/ to register it with the reference's kernel selection.
There is no CPU / PyTorch fallback: every forward goes through libb2q.so (include/b2q.h) or raises.
"""
from __future__ import annotations

import os

import math
from typing import Optional, Tuple

import torch
import torch.nn as nn

import ctypes

from . import layouts
from ._lib import B2QError, check, lib
from .adapter import Lora

_DTYPE_CODE = {torch.float16: 0, torch.bfloat16: 1}
DECODE_MAX_M = 8
PREFILL_MIN_M = 128  # M > 128: the CTA-pair prefill tier (b2q_gemm_multi serves sibling groups there)


class SiblingGroup:
    """QuantLinears that consume the SAME activations (q/k/v, gate/up) served by ONE launch: `b2q_decode_multi` for
    <= 8 tokens, `b2q_gemm_multi` (persistent prefill tier) for > 128 tokens; 9..128 tokens run per module.

    The first member called with a new `x` launches for all members and parks the siblings'
    outputs; each sibling's `forward(x)` then just picks its result up.  Every module keeps the reference's
    per-module `forward(x) -> y` contract (same arithmetic; bit-identical to separate calls whenever the fused launch
    splits K like the single launches would, see `b2q_debug_decode_plan`); only the launch count changes.

    Contract: parked outputs are keyed on (data_ptr, version, M, dtype) of the activations, are handed out once, and
    are dropped as soon as any member is called with different activations.  The group keeps a strong reference to the
    activations it launched on until the parked outputs are consumed or replaced: while it is held the caching allocator
    cannot hand that address to another tensor, so "same data_ptr" means "same tensor" even under
    `torch.inference_mode()` (where tensors carry no version counter and fresh activations often reuse addresses).  What
    remains undetectable there is an IN-PLACE overwrite of that very tensor between sibling calls; a member that finds
    its own parked output already consumed (called twice on one key) therefore always relaunches.
    """

    def __init__(self, members):
        self.members = list(members)
        self.key = None
        self.pending = {}
        self._x_ref = None  # pins the activations the parked outputs belong to

    @staticmethod
    def _version(t):
        try:
            return t._version
        except RuntimeError:  # inference tensors do not track a version counter (reference runs under inference_mode)
            return -1

    def run(self, who, x2, M):
        # parked outputs are only handed out for the very same activations, to siblings that have not consumed theirs yet
        key = (x2.data_ptr(), self._version(x2), M, x2.dtype)
        if self.key == key and id(who) in self.pending:
            out = self.pending.pop(id(who))
            if not self.pending:
                self.key = None
                self._x_ref = None
            return out
        mods = self.members
        n = len(mods)
        K = who.in_features
        outs = [torch.empty((M, m.out_features), dtype=x2.dtype, device=x2.device) for m in mods]
        vp = ctypes.c_void_p * n
        packed = vp(*[m.packed.data_ptr() for m in mods])
        scales = vp(*[m._scales_for(x2.dtype).data_ptr() for m in mods])
        zeros = vp(*[_ptr(m._zeros_dev) for m in mods])
        bias = vp(*[_ptr(m._bias_for(x2.dtype)) for m in mods])
        outp = vp(*[o.data_ptr() for o in outs])
        Ns = (ctypes.c_int * n)(*[m.out_features for m in mods])
        stream = torch.cuda.current_stream(x2.device).cuda_stream
        if M <= DECODE_MAX_M:
            check(lib.b2q_decode_multi(x2.data_ptr(), n, packed, scales, zeros, _ptr(who.perm), bias, outp, Ns, M, K,
                                       who.kbits, who._kgs, _DTYPE_CODE[x2.dtype], stream), "b2q_decode_multi")
        else:  # prefill tier: one persistent launch over the tile columns of all siblings, x[:, perm] gathered once
            ws, ws_bytes = None, 0
            if who.perm is not None:
                ws_bytes = M * K * 2
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x2.device)
            check(lib.b2q_gemm_multi(x2.data_ptr(), n, packed, scales, zeros, _ptr(who.perm), bias, outp, Ns, M, K,
                                     who.kbits, who._kgs, _DTYPE_CODE[x2.dtype], _ptr(ws), ws_bytes, stream),
                  "b2q_gemm_multi")
        self.key = key
        self._x_ref = x2
        self.pending = {id(m): o for m, o in zip(mods, outs) if m is not who}
        return outs[mods.index(who)]


def fuse_siblings(mods) -> bool:
    """Group post_init'ed B200QuantLinear modules that are always called with the same input (q/k/v or gate/up).
    Returns False (and changes nothing) if the set cannot share a launch."""
    mods = list(mods)
    if not (2 <= len(mods) <= 3):
        return False
    m0 = mods[0]
    for m in mods:
        if not isinstance(m, B200KernelMixin) or not m._prepacked or m.kbits != 4 or m._gather is not None:
            return False
        # act-order siblings share a launch only if they share the permutation (q/k/v and gate/up of a GPTQ checkpoint
        # are quantised against the same input Hessian, hence the same g_idx)
        if (m.perm is None) != (m0.perm is None) or (m.perm is not None and not torch.equal(m.perm, m0.perm)):
            return False
        if (m.in_features, m._kgs, m._is_sym, m.packed.device, m.scales.dtype) != (
                m0.in_features, m0._kgs, m0._is_sym, m0.packed.device, m0.scales.dtype):
            return False
        if m.in_features % 128 != 0 or m._kgs not in (64, 128, m.in_features) or m.adapter:
            return False
    grp = SiblingGroup(mods)
    for m in mods:
        m._siblings = grp
    return True


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


class B200KernelMixin:
    """State + behaviour of the B200 kernels behind the reference's QuantLinear contract, independent of the nn.Module
    base it is mixed into: `B200QuantLinear` (stand-alone, below) and the subclass of the reference's own
    `GPTQQuantLinear` that `gptqmodel_b200.reference_shim.make_reference_kernel` builds (INTEGRATION.md §2)."""

    def _b200_setup(
        self,
        bits: int,
        group_size: int,
        desc_act: bool,
        sym: bool,
        in_features: int,
        out_features: int,
        bias: bool = False,
        pack_dtype: torch.dtype = torch.int32,
        adapter=None,
        register_buffers: bool = True,
        **kwargs,
    ):
        """Everything the kernels need on `self`; called by the constructor of the concrete class AFTER its nn.Module
        base(s) are initialised (B200QuantLinear below, or the reference-side subclass of GPTQQuantLinear built by
        gptqmodel_b200.reference_shim — which is why this is not a cooperative __init__)."""
        self.bits = bits
        self.requested_group_size = group_size
        self.group_size = group_size if group_size != -1 else in_features
        self.desc_act = desc_act
        self.sym = sym
        self.in_features = in_features
        self.out_features = out_features
        self.pack_dtype = pack_dtype
        self.pack_dtype_bits = 32
        self.pack_factor = 32 // bits
        self.maxq = (1 << bits) - 1
        # checkpoint layout (2 / 3-bit continuous, planar 3 / 5 / 6 / 7-bit: qlinear/__init__.py:766-773) vs the container
        # the kernels stream: post_init() widens b-bit codes exactly into 4- or 8-bit fields (layouts.py)
        if not hasattr(self, "format") or getattr(self, "format", None) is None:
            self.format = kwargs.get("format")
        self.planar = layouts.is_planar(bits, self.format)
        self.kbits = layouts.container_bits(bits)
        self._kK = in_features         # reduction length / group size the kernels see: differ from in_features /
        self._kgs = self.group_size    # group_size only after regrouping an arbitrary g_idx (post_init)
        self._gather: Optional[torch.Tensor] = None
        if not hasattr(self, "name") or self.name is None:
            self.name = kwargs.get("name") or f"{self.__class__.__module__}.{self.__class__.__qualname__}"
        if not hasattr(self, "backend"):
            self.backend = kwargs.get("backend", "b200")
        self.compute_dtype = kwargs.get("dtype") or torch.float16
        if not hasattr(self, "adapter"):  # the reference's BaseQuantLinear keeps its own deep copy (qlinear/__init__.py:126)
            self.adapter = adapter
        # the reference's GPTQQuantLinear starts at format 1 and its loader flips it after converting the zero-points
        # (utils/model.py:750-846); stand-alone modules are handed v2 tensors
        if not hasattr(self, "_qzeros_format"):
            self._qzeros_format = 2
        self._prepacked = False
        self._scales_cache = {}
        self._siblings = None

        K, N, G = in_features, out_features, math.ceil(in_features / self.group_size)
        # checkpoint-shaped, non-trainable Parameters (what Marlin/Swordfish register: swordfish.py:108-148)
        mk = lambda t: nn.Parameter(t, requires_grad=False)  # noqa: E731
        if register_buffers:
            self.qweight = mk(torch.zeros((K * bits // 32, N), dtype=torch.int32))
            self.qzeros = mk(torch.zeros((G, N * bits // 32), dtype=torch.int32))
            self.scales = mk(torch.zeros((G, N), dtype=torch.float16))
            self.g_idx = mk(torch.tensor([i // self.group_size for i in range(K)], dtype=torch.int32))
            self.bias = mk(torch.zeros(N, dtype=torch.float16)) if bias else None
        else:
            self.qweight = self.qzeros = self.scales = self.g_idx = None
            self.bias = None
        # runtime tensors created by post_init()
        self.packed: Optional[torch.Tensor] = None
        self.perm: Optional[torch.Tensor] = None
        self._zeros_dev: Optional[torch.Tensor] = None

    def qzero_format(self, format: int = None) -> int:
        if format is None:
            return self._qzeros_format
        if format not in (1, 2):
            raise ValueError("Unsupported qzero format. Only 1 and 2 are supported.")
        self._qzeros_format = format
        return format

    def convert_gptq_v1_to_v2(self):
        """In-place v1 -> v2 zero-points (what utils/model.py:810-818 does when REQUIRES_FORMAT_V2)."""
        if self._qzeros_format == 1:
            if self.bits in (4, 8) and not self.planar:
                self.qzeros.data += {4: 0x11111111, 8: 0x01010101}[self.bits]
            else:  # fields that wrap or straddle words: shift the decoded zero-points (utils/model_dequant.py:900-907)
                self.qzeros.data.copy_(layouts.shift_zero_points(self.qzeros.data, self.bits, self.planar, +1))
            self._qzeros_format = 2

    @torch.no_grad()
    def pack_block(self, linear: nn.Module, scales: torch.Tensor, zeros: torch.Tensor, g_idx: torch.Tensor = None,
                   **_ignored):
        """Quantiser-side entry of the reference contract (`pack_block` / `pack_original` / `pack`,
        qlinear/__init__.py:1326-1583): fill the checkpoint-layout tensors (v2 zero-points) from a float nn.Linear and
        its [out_features, groups] scale / zero-point grids.  Runs on the weights' device (gptqmodel_b200/pack.py)."""
        from .pack import pack_gptq

        if self._prepacked:
            raise B2QError("pack_block() after post_init()")
        w = linear.weight.data
        if g_idx is None:
            g_idx = torch.arange(self.in_features, dtype=torch.int32, device=w.device) // self.group_size
        out = pack_gptq(w, scales, zeros, g_idx, self.bits, bias=getattr(linear, "bias", None), planar=self.planar)
        mk = lambda t: None if t is None else nn.Parameter(t, requires_grad=False)  # noqa: E731
        self.qweight, self.qzeros, self.scales, self.g_idx = (mk(out[k]) for k in ("qweight", "qzeros", "scales", "g_idx"))
        self.bias = mk(out["bias"])
        self._qzeros_format = 2

    pack = pack_block
    pack_original = pack_block

    def list_buffers(self):
        out, seen = [], set()
        for state in (self._parameters, self._buffers):
            for t in state.values():
                if isinstance(t, torch.Tensor) and id(t) not in seen:
                    seen.add(id(t))
                    out.append(t)
        for t in (self.packed, self.perm, self._zeros_dev):
            if isinstance(t, torch.Tensor) and id(t) not in seen:
                out.append(t)
        return out

    # ---- one-time repack ---------------------------------------------------------------------------
    @torch.no_grad()
    def post_init(self):
        if self._prepacked:
            return
        dev = self.qweight.device
        if dev.type != "cuda":
            raise B2QError("B200QuantLinear.post_init(): weights must be on a CUDA device (no CPU path)")
        if self._qzeros_format != 2:
            raise B2QError("B200QuantLinear needs v2 qzeros; call convert_gptq_v1_to_v2() after loading a v1 file")
        K, N = self.in_features, self.out_features
        gs = self.group_size
        kb = self.kbits
        with torch.cuda.device(dev):
            qw = self.qweight.data.contiguous()
            qz = self.qzeros.data.contiguous()
            G = qz.shape[0]
            g_idx = self.g_idx.data.to(torch.int64)
            trivial = G == K // gs and torch.equal(g_idx, torch.arange(K, device=dev) // gs)
            uniform = trivial
            if not trivial and G == K // gs:
                counts = torch.bincount(g_idx, minlength=G)
                uniform = counts.numel() == G and bool((counts == gs).all())
            perm = None
            if uniform:
                # act-order: sort rows by group so every group is contiguous; x is gathered with the same permutation
                if not trivial:
                    # int32 [2K]: the order followed by its inverse (include/b2q.h: the decode tiers scatter through the
                    # inverse, the tensor-core tiers gather through the order)
                    order = torch.argsort(g_idx, stable=True)
                    inv = torch.empty_like(order)
                    inv[order] = torch.arange(K, device=dev)
                    perm = torch.cat([order, inv]).to(torch.int32).contiguous()
                if kb != self.bits or self.planar:
                    qw, qz, _ = layouts.widen(qw, qz, self.bits, self.planar)
                kK, kgs = K, gs
            else:
                # arbitrary g_idx (unequal groups; a K-slice of an act-order layer with replicated scale tables): sort,
                # pad every group to a granule with zero-weight rows, re-index the tables per granule (layouts.regroup).
                # The activations' columns are gathered (and padded) by forward(); the kernels see a plain layer.
                r = layouts.regroup(layouts.unpack_rows(qw, self.bits, self.planar),
                                    layouts.unpack_cols(qz, self.bits, self.planar), self.scales.data, g_idx)
                qw, qz = layouts.pack_rows(r["q"], kb), layouts.pack_cols(r["z"], kb)
                self.scales.data = r["scales"]
                self._gather = r["gather"]
                kK, kgs = int(r["gather"].numel()), int(r["granule"])
            # symmetric layers (every zero-point == 2^(kbits-1)) never read qzeros
            zsym = {4: 0x88888888 - (1 << 32), 8: 0x80808080 - (1 << 32)}[kb]
            is_sym = bool((qz == zsym).all())
            packed = torch.empty(lib.b2q_packed_bytes(kK, N, kb), dtype=torch.uint8, device=dev)
            # (no stream synchronisation: the repack runs on the current stream and the caching allocator is stream-ordered,
            #  so releasing the checkpoint-layout weights below is safe — 224 syncs per model load otherwise)
            check(lib.b2q_prepack(_ptr(qw), _ptr(perm), _ptr(packed), kK, N, kb,
                                  torch.cuda.current_stream(dev).cuda_stream), "b2q_prepack")
        self._kK, self._kgs = kK, kgs
        self.packed = packed
        self.perm = perm
        self._zeros_dev = None if is_sym else qz.contiguous()
        self._is_sym = is_sym
        # the checkpoint-layout weights are no longer needed (Marlin/Swordfish free them as well)
        self.qweight = nn.Parameter(torch.empty(0, dtype=torch.int32, device=dev), requires_grad=False)
        self.g_idx = nn.Parameter(torch.empty(0, dtype=torch.int32, device=dev), requires_grad=False)
        self.scales.data = self.scales.data.contiguous()
        self._prepacked = True
        base_post_init = getattr(super(), "post_init", None)
        if base_post_init is not None:
            base_post_init()  # reference base: BaseQuantLinear.post_init() initialises the adapter (qlinear/__init__.py:224-234)
        elif self.adapter is not None and hasattr(self.adapter, "post_init"):
            self.adapter.post_init(weight_key=self.name, device=dev,
                                   lora_A=getattr(self, "lora_A", None), lora_B=getattr(self, "lora_B", None))

    def _scales_for(self, dtype: torch.dtype) -> torch.Tensor:
        s = self.scales.data
        if s.dtype == dtype:
            return s
        c = self._scales_cache.get(dtype)
        if c is None or c.device != s.device:
            c = s.to(dtype).contiguous()  # Marlin re-casts scales to x.dtype the same way (marlin.py:312-315)
            self._scales_cache[dtype] = c
        return c

    def _bias_for(self, dtype: torch.dtype) -> Optional[torch.Tensor]:
        if self.bias is None:
            return None
        b = self.bias.data
        if b.dtype == dtype:
            return b
        key = ("bias", dtype)
        c = self._scales_cache.get(key)
        if c is None or c.device != b.device:
            c = b.to(dtype).contiguous()
            self._scales_cache[key] = c
        return c

    # ---- hot path ------------------------------------------------------------------------------------
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not self._prepacked:
            raise B2QError("B200QuantLinear.forward() before post_init()")
        K, N = self.in_features, self.out_features
        out_shape = x.shape[:-1] + (N,)
        if x.shape[-1] != K:
            raise ValueError(f"expected last dim {K}, got {x.shape[-1]}")
        if x.dtype not in _DTYPE_CODE:
            raise B2QError(f"B200QuantLinear supports fp16/bf16 activations, got {x.dtype}")
        if x.device != self.packed.device:
            raise B2QError(f"input on {x.device} but weights on {self.packed.device}")
        x2 = x.reshape(-1, K)
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        M = x2.shape[0]
        if self._siblings is not None and (1 <= M <= DECODE_MAX_M or M > PREFILL_MIN_M):
            return self._siblings.run(self, x2, M).reshape(out_shape)
        out = torch.empty((M, N), dtype=x.dtype, device=x.device)
        if M == 0:
            return out.reshape(out_shape)
        if self._gather is not None:
            x2 = x2.index_select(1, self._gather)  # regrouped layer: columns in sorted-by-group order, padded per group
        kK = self._kK
        ws, ws_bytes = None, 0
        if self.perm is not None:
            # act-order: the tensor-core tiers read x[:, perm] from a workspace (the decode / GEMV tiers gather it while
            # staging the activations and need none; b2q_mm_workspace_bytes mirrors b2q_mm's dispatch exactly)
            ws_bytes = lib.b2q_mm_workspace_bytes(M, kK, N, self.kbits, self._kgs, 1)
            if ws_bytes:
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        check(
            lib.b2q_mm(_ptr(x2), _ptr(self.packed), _ptr(self._scales_for(x.dtype)), _ptr(self._zeros_dev),
                       _ptr(self.perm), _ptr(self._bias_for(x.dtype)), _ptr(out), M, kK, N, self.kbits,
                       self._kgs, _DTYPE_CODE[x.dtype], _ptr(ws), ws_bytes,
                       torch.cuda.current_stream(x.device).cuda_stream),
            "b2q_mm",
        )
        out = out.reshape(out_shape)
        if self.adapter:
            out = self.adapter.apply(x=x, out=out)
        return out

    def forward_allreduce(self, x: torch.Tensor, ar) -> torch.Tensor:
        """Row-parallel shard + all-reduce(sum) across the TP group in ONE launch (`b2q_decode_allreduce`).

        `ar` is a `gptqmodel_b200.tp.FusedDecodeAllReduce`; decode tier only (4-bit, <= 8 tokens, no act-order).
        EXPERIMENTAL in round 1 (compiled, not yet validated on GPUs)."""
        if not self._prepacked:
            raise B2QError("B200QuantLinear.forward_allreduce() before post_init()")
        K, N = self.in_features, self.out_features
        x2 = x.reshape(-1, K)
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        M = x2.shape[0]
        if not (1 <= M <= DECODE_MAX_M) or self.kbits != 4 or self.perm is not None or self._gather is not None \
                or x.dtype not in _DTYPE_CODE:
            raise B2QError("forward_allreduce: decode tier only (bits=4, 1 <= tokens <= 8, no act-order, fp16/bf16)")
        if self.adapter:
            # the adapter's low-rank update belongs to the FULL layer output; applying it to one rank's partial sum (or
            # dropping it silently, ADVICE r01) would change the result: callers use forward() + all-reduce instead
            raise B2QError("forward_allreduce: modules with an adapter must use forward() followed by the all-reduce")
        out = torch.empty((M, N), dtype=x.dtype, device=x.device)
        check(
            lib.b2q_decode_allreduce(_ptr(x2), _ptr(self.packed), _ptr(self._scales_for(x.dtype)),
                                     _ptr(self._zeros_dev), _ptr(self._bias_for(x.dtype)), _ptr(out), M, K, N,
                                     self.kbits, self._kgs, _DTYPE_CODE[x.dtype], ar.rank, ar.world, ar._peers,
                                     ar.flag_offset, ar.max_elems, ar.ctl.data_ptr(),
                                     torch.cuda.current_stream(x.device).cuda_stream),
            "b2q_decode_allreduce",
        )
        return out.reshape(x.shape[:-1] + (N,))

    # ---- helpers for tests / tools -------------------------------------------------------------------
    @classmethod
    def from_checkpoint_tensors(cls, qweight, qzeros, scales, g_idx, bits, group_size, bias=None, desc_act=None,
                                sym=None, device="cuda", dtype=None, format=None):
        """Build + post_init a module from checkpoint-layout tensors (v2 qzeros; `format="gptq_p"` for planar 3-bit)."""
        K = g_idx.shape[0]
        N = qweight.shape[1]
        m = cls(bits=bits, group_size=group_size, desc_act=bool(desc_act), sym=bool(sym) if sym is not None else True,
                in_features=K, out_features=N, bias=bias is not None, register_buffers=False, dtype=dtype, format=format)
        mk = lambda t: nn.Parameter(t.detach().clone().contiguous().to(device), requires_grad=False)  # noqa: E731
        m.qweight, m.qzeros, m.scales, m.g_idx = mk(qweight), mk(qzeros), mk(scales), mk(g_idx.to(torch.int32))
        m.bias = mk(bias) if bias is not None else None
        m.post_init()
        return m

    @torch.no_grad()
    def dequantize_weight(self, num_itr: int = 1, chunk: int = 2048) -> torch.Tensor:
        """Dense W [in_features, out_features] in the scales' dtype, identical to the reference's
        `dequantize_weight()` (qlinear/__init__.py:947-1021): rows of the identity are pushed through the tensor-core
        tier, whose operands are the exact `(q - z) * s` values (one rounding), so every output element is one weight
        times 1.0 plus zeros.  After post_init() only (the checkpoint-layout tensors are released there)."""
        if not self._prepacked:
            raise B2QError("dequantize_weight() before post_init()")
        K, N = self.in_features, self.out_features
        dt = self.scales.dtype
        dev = self.packed.device
        out = torch.empty((K, N), dtype=dt, device=dev)
        chunk = max(256, chunk)  # > 128 rows: always the exact-dequant tensor-core tiers, never the decode tier
        stream = torch.cuda.current_stream(dev).cuda_stream
        for k0 in range(0, K, chunk):
            rows = min(chunk, K - k0)
            if rows <= 128:  # short tail: widen the block backwards so the tier stays the same
                k0, rows = max(0, K - 256), min(256, K)
            x = torch.zeros((rows, K), dtype=dt, device=dev)
            x[torch.arange(rows, device=dev), torch.arange(k0, k0 + rows, device=dev)] = 1
            if self._gather is not None:
                x = x.index_select(1, self._gather)
            ws, ws_bytes = None, 0
            if self.perm is not None:
                ws_bytes = lib.b2q_workspace_bytes(rows, self._kK, N, 1)
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            y = out[k0:k0 + rows]
            check(lib.b2q_gemm(_ptr(x), _ptr(self.packed), _ptr(self._scales_for(dt)), _ptr(self._zeros_dev),
                               _ptr(self.perm), None, _ptr(y), rows, self._kK, N, self.kbits, self._kgs, _DTYPE_CODE[dt],
                               _ptr(ws), ws_bytes, stream), "b2q_gemm(dequantize_weight)")
        return out

    def extra_repr(self) -> str:
        return (f"in_features={self.in_features}, out_features={self.out_features}, bits={self.bits}, "
                f"group_size={self.group_size}, desc_act={self.desc_act}, sym={self.sym}")


class B200QuantLinear(B200KernelMixin, nn.Module):
    """Stand-alone module (no import of the reference package)."""

    # ---- capability declaration (names follow the reference's BaseQuantLinear) ----
    SUPPORTS_BACKENDS = ["b200"]
    SUPPORTS_METHODS = ["gptq"]
    SUPPORTS_FORMATS = {"gptq": 120, "gptq_v2": 120, "gptq_p": 120}  # > TorchAten 110 (CPU) / Swordfish 101 / Machete 100 / Marlin 90
    SUPPORTS_BITS = [2, 3, 4, 5, 6, 7, 8]  # 4 / 8 native; 2 / 3 widened to 4-bit, 5 / 6 / 7 (planar) to 8-bit fields at post_init
    SUPPORTS_GROUP_SIZE = [-1, 32, 64, 128]
    SUPPORTS_DESC_ACT = [True, False]
    SUPPORTS_SYM = [True, False]
    SUPPORTS_SHARDS = True
    SUPPORTS_TRAINING = False
    SUPPORTS_AUTO_PADDING = False
    SUPPORTS_IN_FEATURES_DIVISIBLE_BY = [64]
    SUPPORTS_OUT_FEATURES_DIVISIBLE_BY = [32]
    SUPPORTS_PACK_DTYPES = [torch.int32]
    SUPPORTS_ADAPTERS = [Lora]  # gptqmodel_b200/adapter.py; any object with .apply(x=, out=) works, see forward()
    SUPPORTS_DEVICES = ["cuda"]
    SUPPORTS_PLATFORM = ["linux"]
    SUPPORTS_DTYPES = [torch.float16, torch.bfloat16]
    REQUIRES_FORMAT_V2 = True  # qzeros hold the true zero-point (loader adds 0x11111111 to v1 files)
    QUANT_TYPE = "b200"

    def __init__(
        self,
        bits: int,
        group_size: int,
        desc_act: bool,
        sym: bool,
        in_features: int,
        out_features: int,
        bias: bool = False,
        pack_dtype: torch.dtype = torch.int32,
        adapter=None,
        register_buffers: bool = True,
        **kwargs,
    ):
        nn.Module.__init__(self)
        ok, err = self.validate(
            bits=bits, group_size=group_size, desc_act=desc_act, sym=sym, in_features=in_features,
            out_features=out_features, pack_dtype=pack_dtype, dtype=kwargs.get("dtype"),
        )
        if not ok:
            raise err
        self._b200_setup(bits, group_size, desc_act, sym, in_features, out_features, bias=bias, pack_dtype=pack_dtype,
                         adapter=adapter, register_buffers=register_buffers, **kwargs)

    # ---- validation -------------------------------------------------------------------------------
    @classmethod
    def validate_once(cls) -> Tuple[bool, Optional[Exception]]:
        if not torch.cuda.is_available():
            return False, NotImplementedError("B200QuantLinear needs a CUDA device")
        major, minor = torch.cuda.get_device_capability()
        if (major, minor) != (9, 0):
            return False, NotImplementedError(f"B200QuantLinear is built for sm_90a only, found sm_{major}{minor}")
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
        if pack_dtype is not None and pack_dtype not in cls.SUPPORTS_PACK_DTYPES:
            return False, NotImplementedError(f"{cls.__name__}: pack_dtype={pack_dtype} unsupported")
        if dtype is not None and dtype not in cls.SUPPORTS_DTYPES:
            return False, NotImplementedError(f"{cls.__name__}: dtype={dtype} unsupported")
        if in_features is not None:
            if in_features % 64 != 0:
                return False, NotImplementedError(f"{cls.__name__}: in_features={in_features} must be divisible by 64")
            if group_size != -1 and in_features % group_size != 0:
                return False, NotImplementedError(f"{cls.__name__}: in_features % group_size != 0")
        if out_features is not None and out_features % 32 != 0:
            return False, NotImplementedError(f"{cls.__name__}: out_features={out_features} must be divisible by 32")
        return True, None

    @classmethod
    def validate_device(cls, device) -> None:
        """Reference contract (qlinear/__init__.py validate_device): raise if the module cannot live on `device`."""
        dev = torch.device(device) if not isinstance(device, torch.device) else device
        if dev.type != "cuda":
            raise NotImplementedError(f"{cls.__name__} supports CUDA devices only, got `{dev}`")
