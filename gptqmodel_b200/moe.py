"""Mixture-of-experts block over QuantLinear experts (BASELINE configs[4]: Mixtral-8x7B int4 g64 asym).

In the reference every expert's ``w1 / w3 / w2`` is an independent QuantLinear module
(gptqmodel/models/definitions/mixtral.py:30-34) that the model's own Python loop calls per expert; the
fused MoE kernel it ships (``swordfish_moe.cu``) is exported but never called.  This module is that
per-expert loop, arranged for the B200 kernels and for tensor parallelism:

  * ONE TOKEN (batch-1 decode) through grouped-eligible 4-bit experts without act-order: three launches on the decode tier —
    the 2 * top_k gate / up matrices as sibling sets of one decode launch (experts read from `topk_ids` on the device),
    SiLU-mul, and a cluster of top_k CTAs per tile column for w2 whose DSMEM reduction applies the routing weights
    (`b2q_moe_decode_*`); other grouped-eligible stacks take the grouped path at one token as well;
  * GROUPED path (default whenever every expert is a B200 QuantLinear of one shape, see `_build_stack`): the (token, k)
    pairs are sorted by expert ON THE DEVICE (`b2q_moe_align`), and the whole block is five launches with no host
    synchronisation — align, gather, ONE grouped launch for w1 and w3 with the SiLU-mul epilogue, ONE grouped launch for w2
    with the routing weight + scatter epilogue, combine (gptqmodel_b200/csrc/b2q_moe.cu, grouped modes of b2q_midm.cu) —
    CUDA-graph capturable; the experts' prepacked tensors are stacked once (the per-expert modules keep views into the
    stack).  Experts are 4- or 8-bit in the kernels (2 / 3 / 5 / 6 / 7-bit checkpoints are widened exactly by post_init), one
    width for w1 / w3 and one for w2.  Act-order experts were prepacked with their rows in group order: the gather reads
    each expert's activations in that expert's column order (`b2q_moe_gather_perm`), and a w2 with act-order gets h
    permuted the same way before the down launch (six launches);
  * BLOCK-FP8 experts (every w1 / w3 / w2 a post_init'ed B200BlockFp8Linear, HF / DeepSeek-native checkpoints): the same
    routing with no host synchronisation, six launches on the e4m3 tensor cores — align, gather-and-quantise, ONE grouped
    gate|up launch, the quantiser on h, ONE grouped down launch, combine (grouped modes of b2q_fp8blk.cu; include/b2q.h
    states the rounding points, those of transformers' per-expert FP8Linear loop).  The checkpoint tensors are stacked
    once and the modules keep views into the stack;
  * QQQ experts (every w1 / w3 / w2 a post_init'ed B200QqqQuantLinear, W4A8): the same six launches on the int8 tensor
    cores — align, gather-and-quantise, ONE grouped gate|up launch, the quantiser on h, ONE grouped down launch, combine
    (grouped modes of b2q_qqq.cu; include/b2q.h states the rounding points, those of the per-expert QQQLinear loop);
  * FP8 W8A16 experts (every w1 / w3 / w2 a post_init'ed B200Fp8QuantLinear): the five launches of the GPTQ grouped path
    on the FP8 instantiations of the grouped small-batch kernels, W the exact b2q_fp8_dequant operand.  Both keep the
    modules working on views into the stacks;
  * per-channel W8A8 experts (B200ChannelFp8Linear / B200ChannelInt8Linear, dynamic or static activations): the same six
    launches on the e4m3 or s8 tensor cores (grouped modes of b2q_fp8ch.cu).  `MoEExperts` keeps the loop for them;
    the grouped path is the subclass `B200ChannelW8A8Experts`;
  * LOOP path (fallback: dense stand-ins in CPU tests, mixed experts, regrouped act-order shards): tokens are sorted by
    expert once, every expert sees one contiguous block of its routed tokens; one host sync per block for the per-expert
    counts, like the reference's loop;
  * tensor parallel: ``w1 / w3`` column-sharded, ``w2`` row-sharded (`tp.shard_moe_expert`), so every rank holds a slice
    of EVERY expert and the block ends in exactly one all-reduce of the combined output, as for a dense MLP.

Experts are any callables mapping ``[m, K] -> [m, N]`` (B200QuantLinear modules in production; dense stand-ins in the
CPU tests), so the routing / combination / sharding algebra is testable without a GPU.
"""
from __future__ import annotations

from typing import Callable, Sequence

import torch
import torch.nn.functional as F

from . import tp


def route_topk(router_logits: torch.Tensor, top_k: int):
    """Mixtral routing: softmax over experts, top-k, renormalise (HF MixtralSparseMoeBlock)."""
    probs = F.softmax(router_logits.float(), dim=-1)
    w, ids = torch.topk(probs, top_k, dim=-1)
    w = w / w.sum(dim=-1, keepdim=True)
    return ids, w


_ROUTE_DTYPES = {torch.float16: 0, torch.bfloat16: 1, torch.float32: 2}


def _route(logits, bias, top_k, scoring, n_group, topk_group, renormalize, scale, who):
    """Check the arguments of b2q_moe_route (include/b2q.h) and launch it on the logits' device and current stream."""
    if not isinstance(logits, torch.Tensor):
        raise ValueError(f"{who}: logits must be a CUDA tensor, got {type(logits).__name__}")
    if logits.dtype not in _ROUTE_DTYPES or logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError(f"{who}: logits must be a contiguous [T, E] fp16 / bf16 / fp32 tensor, got "
                         f"{logits.dtype} {tuple(logits.shape)}")
    T, E = logits.shape
    top_k, n_group, topk_group = int(top_k), int(n_group), int(topk_group)
    if not 1 <= E <= 256 or not 1 <= top_k <= min(E, 16):
        raise ValueError(f"{who}: need 1 <= E <= 256 and 1 <= top_k <= min(E, 16), got E={E} top_k={top_k}")
    if bias is not None:
        if (not isinstance(bias, torch.Tensor) or bias.dtype != torch.float32 or tuple(bias.shape) != (E,)
                or not bias.is_contiguous() or bias.device != logits.device):
            raise ValueError(f"{who}: correction_bias must be a contiguous fp32 [{E}] tensor on {logits.device}")
        if n_group < 1 or E % n_group != 0 or E // n_group < 2 or not 1 <= topk_group <= n_group \
                or top_k > topk_group * (E // n_group):
            raise ValueError(f"{who}: need n_group dividing E={E} with >= 2 experts per group, 1 <= topk_group <= "
                             f"n_group and top_k <= topk_group * E / n_group, got n_group={n_group} "
                             f"topk_group={topk_group} top_k={top_k}")
    if not logits.is_cuda:
        raise ValueError(f"{who}: logits must be a CUDA tensor (there is no CPU routing kernel), got {logits.device}")
    from ._lib import check, lib

    dev = logits.device
    ids = torch.empty((T, top_k), dtype=torch.int32, device=dev)
    w = torch.empty((T, top_k), dtype=torch.float32, device=dev)
    if T == 0:
        return ids, w
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream(dev).cuda_stream
        check(lib.b2q_moe_route(logits.data_ptr(), _ROUTE_DTYPES[logits.dtype], None if bias is None else bias.data_ptr(),
                                T, E, top_k, scoring, n_group, topk_group, int(bool(renormalize)), float(scale),
                                ids.data_ptr(), w.data_ptr(), st), "b2q_moe_route")
    return ids, w


def route_softmax_topk(logits: torch.Tensor, top_k: int, renormalize: bool = True, scale: float = 1.0):
    """Softmax top-k routing (Mixtral, Qwen2/3-MoE with ``norm_topk_prob`` on or off, OLMoE, DBRX) in one kernel.

    logits: CUDA [T, E] fp16 / bf16 / fp32, contiguous, E <= 256; 1 <= top_k <= min(E, 16).  Returns (ids int32 [T, top_k],
    weights fp32 [T, top_k]) on the logits' device and current stream, ready for ``MoEExperts.forward``:
    p = softmax(logits) in fp32, the top_k experts by logit, weights p (divided by their sum when ``renormalize``) times
    ``scale``.  Slots come in descending logit, ties to the lower expert index (include/b2q.h: b2q_moe_route)."""
    return _route(logits, None, top_k, 0, 1, 1, renormalize, scale, "route_softmax_topk")


def route_grouped_sigmoid(logits: torch.Tensor, correction_bias: torch.Tensor, top_k: int, n_group: int, topk_group: int,
                          renormalize: bool = True, scale: float = 1.0):
    """Grouped sigmoid routing (DeepSeek-V3/R1: n_group 8, topk_group 4; GLM-4.5 / dots1: n_group 1) in one kernel.

    s = sigmoid(logits), c = s + correction_bias (``e_score_correction_bias``, fp32 [E]); the topk_group groups of E / n_group
    consecutive experts with the largest sum of their two largest c are kept, and the top_k largest c among their experts
    are selected (experts of dropped groups are never chosen, as in vLLM's grouped_topk; transformers fills them with 0.0,
    which differs only when a kept group holds a negative c).  Weights are s (divided by sum + 1e-20 when ``renormalize``)
    times ``scale`` (``routed_scaling_factor``).  Returns (ids int32 [T, top_k], weights fp32 [T, top_k]); slots come in
    descending c, ties to the lower index (include/b2q.h: b2q_moe_route)."""
    if not isinstance(correction_bias, torch.Tensor):
        raise ValueError("route_grouped_sigmoid: correction_bias must be an fp32 tensor")
    return _route(logits, correction_bias, top_k, 1, n_group, topk_group, renormalize, scale, "route_grouped_sigmoid")


class MoEExperts(torch.nn.Module):
    """``y = sum_k w_k * w2_e( silu(w1_e x) * w3_e x )`` over the top-k experts e of every token."""

    def __init__(self, w1: Sequence[Callable], w3: Sequence[Callable], w2: Sequence[Callable], fuse: bool = True,
                 group=None, reduce=None, grouped=None):
        """grouped: None = use the grouped kernels when the experts qualify, True = require them, False = per-expert loop."""
        super().__init__()
        if not (len(w1) == len(w3) == len(w2)) or len(w1) == 0:
            raise ValueError("MoEExperts: need the same number (>= 1) of w1 / w3 / w2 experts")
        as_list = lambda xs: torch.nn.ModuleList(xs) if all(isinstance(x, torch.nn.Module) for x in xs) else list(xs)  # noqa: E731
        self.w1, self.w3, self.w2 = as_list(w1), as_list(w3), as_list(w2)
        self.group = group
        self.reduce = reduce  # optional tp.P2PAllReduce for decode-sized outputs
        self.decode_path = True  # one token: the decode-tier launches (False: always the grouped small-batch kernels; A/B)
        # SiLU-mul folded into the down launch's activation staging (two launches instead of three).  OFF by default: every
        # CTA of a rank recomputes the row's exp() on the critical path between the PDL wait and its first mma, while the
        # separate small kernel overlaps
        self.fuse_act = False
        self._stack = None
        self._refusal = None  # why the experts do not qualify, when the stack builder says so
        if grouped is None or grouped:
            self._stack = self._build_stack()
            if grouped and self._stack is None and self._refusal is not None:
                raise ValueError(f"{type(self).__name__}(grouped=True): {self._refusal}")
            if grouped and self._stack is None:
                raise ValueError("MoEExperts(grouped=True): experts must be post_init'ed B200 QuantLinears of one shape / "
                                 "group size, with one kernel bit width (4 or 8) for w1 / w3 and one for w2, the same "
                                 "act-order permutation in w1 and w3 of every expert, and no regrouped g_idx, bias or "
                                 "adapters; or post_init'ed B200BlockFp8Linears only, one shape per role on one device, "
                                 "an intermediate size that is a multiple of 128, and no bias or adapters; or post_init'ed "
                                 "B200QqqQuantLinears only (one shape and group kind per role, w1 and w3 alike, an "
                                 "intermediate size that is a multiple of 64, at most 256 experts on one device, no bias "
                                 "or adapters); or post_init'ed B200Fp8QuantLinears only (one shape and scale group per "
                                 "role, at most 256 experts on one device, no bias or adapters).  Per-channel W8A8 "
                                 "experts run grouped through B200ChannelW8A8Experts")
        if fuse and self._stack is None:
            from .qlinear import B200KernelMixin, fuse_siblings

            for a, b in zip(self.w1, self.w3):
                if isinstance(a, B200KernelMixin) and isinstance(b, B200KernelMixin):
                    fuse_siblings([a, b])

    def _build_stack(self):
        """Stack the experts' prepacked tensors for the grouped kernels; None if the experts do not qualify."""
        from .fp8_block import B200BlockFp8Linear
        from .qlinear import B200KernelMixin

        from .fp8 import B200Fp8QuantLinear
        from .qqq import B200QqqQuantLinear

        from .w4afp8 import B200W4Fp8Linear

        every = [m for mods in (self.w1, self.w3, self.w2) for m in mods]
        if any(isinstance(m, B200W4Fp8Linear) for m in every):
            self._refusal = "W4AFP8 experts (B200W4Fp8Linear) have no grouped kernels; they run the per-expert loop"
            return None
        if all(isinstance(m, B200BlockFp8Linear) for m in every):
            return self._build_fp8blk_stack()
        if all(isinstance(m, B200QqqQuantLinear) for m in every):
            return self._build_qqq_stack()
        if all(isinstance(m, B200Fp8QuantLinear) for m in every):
            return self._build_fp8_stack()
        sets = []
        for mods in (self.w1, self.w3, self.w2):
            m0 = mods[0]
            for m in mods:
                # kbits: the 4- or 8-bit container the kernels stream (post_init widens other widths exactly); a
                # regrouped g_idx (unequal groups) gathers and pads x per layer, which the stacked launches cannot do
                if not isinstance(m, B200KernelMixin) or not m._prepacked or m.kbits not in (4, 8) or m._gather is not None \
                        or m.bias is not None or m.adapter:
                    return None
                if (m.in_features, m.out_features, m.group_size, m.kbits, m.packed.device, m.scales.dtype) != (
                        m0.in_features, m0.out_features, m0.group_size, m0.kbits, m0.packed.device, m0.scales.dtype):
                    return None
            sets.append(list(mods))
        w1, w3, w2 = sets
        if (w1[0].in_features, w1[0].out_features, w1[0].group_size, w1[0].kbits) != (
                w3[0].in_features, w3[0].out_features, w3[0].group_size, w3[0].kbits):
            return None
        if w2[0].in_features != w1[0].out_features:
            return None
        # w1 and w3 of an expert read the same gathered activations: they must share the act-order permutation (true of
        # real checkpoints, where both are quantised against the same inputs)
        for a, b in zip(w1, w3):
            if (a.perm is None) != (b.perm is None) or (a.perm is not None and not torch.equal(a.perm, b.perm)):
                return None
        out = {}
        for name, mods in (("w1", w1), ("w3", w3), ("w2", w2)):
            asym = any(not m._is_sym for m in mods) if name == "w2" else any(not m._is_sym for m in w1 + w3)
            packed = torch.stack([m.packed for m in mods]).contiguous()
            scales = torch.stack([m.scales.data for m in mods]).contiguous()
            zeros = torch.stack([self._kernel_zeros(m) for m in mods]).contiguous() if asym else None
            for e, m in enumerate(mods):  # the modules keep working on their own; no second copy of the weights
                m.packed = packed[e]
                m.scales.data = scales[e]
                m._scales_cache.clear()
                if zeros is not None:
                    if m.kbits == m.bits:  # a widened module's qzeros keeps the checkpoint's narrower fields
                        m.qzeros.data = zeros[e]
                    if m._zeros_dev is not None:
                        m._zeros_dev = zeros[e]
            perm = None  # [E, K]: the order half of every expert's permutation, the identity where there is none
            if any(m.perm is not None for m in mods):
                K = mods[0].in_features
                ident = torch.arange(K, dtype=torch.int32, device=packed.device)
                perm = torch.stack([ident if m.perm is None else m.perm[:K] for m in mods]).contiguous()
            out[name] = dict(packed=packed, scales={scales.dtype: scales}, zeros=zeros, K=mods[0].in_features,
                             N=mods[0].out_features, group=mods[0].group_size, bits=mods[0].kbits, perm=perm)
        return out

    def _build_fp8blk_stack(self):
        """Stack the block-FP8 experts' checkpoint tensors (weight [E, N, K] e4m3, weight_scale_inv [E, ceil(N/128),
        K/128]) for the grouped kernels; None if the experts do not qualify."""
        w1, w3, w2 = list(self.w1), list(self.w3), list(self.w2)
        for mods in (w1, w3, w2):
            m0 = mods[0]
            for m in mods:
                if not m._ready or m.bias is not None or m.adapter:
                    return None
                if (m.in_features, m.out_features, m.weight.device) != (m0.in_features, m0.out_features, m0.weight.device):
                    return None
        K, inter = w1[0].in_features, w1[0].out_features
        # w2's envelope (in_features % 128) makes inter a multiple of 128: h is quantised in 128-k groups for the down launch
        if (w3[0].in_features, w3[0].out_features) != (K, inter) or w2[0].in_features != inter:
            return None
        out = {"fp8blk": True}
        for name, mods in (("w1", w1), ("w3", w3), ("w2", w2)):
            weight = torch.stack([m.weight.view(torch.uint8) for m in mods]).view(torch.float8_e4m3fn)
            scale = torch.stack([m.weight_scale_inv for m in mods]).contiguous()
            for e, m in enumerate(mods):  # the modules keep working on their own; no second copy of the weights
                m.weight = weight[e]
                if scale[e].data_ptr() % 16 == 0:  # the layer kernel wants 16-byte aligned scales (a few bytes each)
                    m.weight_scale_inv = scale[e]
            out[name] = dict(weight=weight, scale=scale, K=mods[0].in_features, N=mods[0].out_features)
        return out

    def _role_ok(self, attrs):
        """The checks every role of a QQQ / FP8 stack passes: post_init'ed, no bias or adapter, one value of `attrs` per
        role, w1 and w3 alike, w2 reading the intermediate size, at most 256 experts."""
        w1, w3, w2 = list(self.w1), list(self.w3), list(self.w2)
        if len(w1) > 256:
            return False
        for mods in (w1, w3, w2):
            for m in mods:
                if not m._prepacked or m.bias is not None or m.adapter or attrs(m) != attrs(mods[0]):
                    return False
        return attrs(w1[0]) == attrs(w3[0]) and w2[0].in_features == w1[0].out_features

    def _build_qqq_stack(self):
        """Stack the QQQ experts' prepacked tensors (packed [E, bytes], s_channel [E, N], s_group [E, K/128, N]) for the
        grouped int8 kernels; None if the experts do not qualify."""
        if not self._role_ok(lambda m: (m.in_features, m.out_features, m._kgs, m.packed.device)):
            return None
        if self.w1[0].out_features % 64 != 0:  # gate|up tiles pair 64 gate with 64 up features
            return None
        out = {"qqq": True}
        for name, mods in (("w1", self.w1), ("w3", self.w3), ("w2", self.w2)):
            packed = torch.stack([m.packed for m in mods]).contiguous()
            sc = torch.stack([m._sc for m in mods]).contiguous()
            sg = torch.stack([m._sg for m in mods]).contiguous() if mods[0]._kgs == 128 else None
            for e, m in enumerate(mods):  # the modules keep working on their own; no second copy of the weights
                m.packed, m._sc = packed[e], sc[e]
                if sg is not None:
                    m._sg = sg[e]
            out[name] = dict(packed=packed, sc=sc, sg=sg, K=mods[0].in_features, N=mods[0].out_features,
                             group=mods[0]._kgs)
        return out

    def _build_fp8_stack(self):
        """Stack the FP8 (W8A16) experts' prepacked codes and per-dtype scale tables [E, K/g, N] for the grouped
        small-batch kernels; None if the experts do not qualify."""
        if not self._role_ok(lambda m: (m.in_features, m.out_features, m._gs, m.packed.device)):
            return None
        out = {"fp8": True}
        for name, mods in (("w1", self.w1), ("w3", self.w3), ("w2", self.w2)):
            packed = torch.stack([m.packed for m in mods]).contiguous()
            scales = {dt: torch.stack([m._scales[dt] for m in mods]).contiguous() for dt in mods[0]._scales}
            for e, m in enumerate(mods):  # the modules keep working on their own; no second copy of the weights
                m.packed = packed[e]
                for dt, st in scales.items():
                    m._scales[dt] = st[e]
            out[name] = dict(packed=packed, scales=scales, K=mods[0].in_features, N=mods[0].out_features,
                             group=mods[0]._gs, fp16_ok=all(m._fp16_ok for m in mods))
        return out

    def _check_x(self, x, T, top_k, K, topk_weights, dev):
        # the gather kernels read x [T, K] by token index: a mismatched x would be read out of bounds
        if x.dtype not in (torch.float16, torch.bfloat16):
            raise ValueError(f"MoEExperts: quantised experts take fp16 / bf16 activations, got {x.dtype}")
        if tuple(x.shape) != (T, K) or x.device != dev or tuple(topk_weights.shape) != (T, top_k):
            raise ValueError(f"MoEExperts: x {tuple(x.shape)} on {x.device} does not fit [{T}, {K}] on {dev}, "
                             f"or topk_weights {tuple(topk_weights.shape)} is not [{T}, {top_k}]")

    def _forward_grouped_qqq(self, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor) -> torch.Tensor:
        """QQQ experts: align -> gather-and-quantise -> gate|up -> quantise h -> down -> combine (include/b2q.h)."""
        from ._lib import check, lib

        T, top_k = topk_ids.shape
        rows, E = T * top_k, self.num_experts
        s1, s3, s2 = self._stack["w1"], self._stack["w3"], self._stack["w2"]
        K, inter, Kout = s1["K"], s1["N"], s2["N"]
        self._check_x(x, T, top_k, K, topk_weights, s1["packed"].device)
        dev, dt = x.device, x.dtype
        code = 0 if dt == torch.float16 else 1
        st = torch.cuda.current_stream(dev).cuda_stream
        ids = topk_ids.to(torch.int32).contiguous()
        wts = topk_weights.to(torch.float32).contiguous()
        x2 = x.contiguous()
        if x2.data_ptr() % 16 != 0:
            x2 = x2.clone()
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        kp = lambda k: (k + 127) // 128 * 128  # noqa: E731  (codes rows are padded to 128 k)
        tables = torch.empty(2 * E + rows, dtype=torch.int32, device=dev)
        counts, offsets, sorted_pairs = tables[:E], tables[E:2 * E], tables[2 * E:]
        codes = torch.empty((rows, kp(K)), dtype=torch.int8, device=dev)
        s_x = torch.empty(rows, dtype=torch.float32, device=dev)
        h = torch.empty((rows, inter), dtype=dt, device=dev)
        codes_h = torch.empty((rows, kp(inter)), dtype=torch.int8, device=dev)
        s_h = torch.empty(rows, dtype=torch.float32, device=dev)
        ypair = torch.empty((rows, Kout), dtype=torch.float32, device=dev)
        y = torch.empty((T, Kout), dtype=dt, device=dev)
        active = min(E, rows)
        check(lib.b2q_moe_align(p(ids), T, top_k, E, p(counts), p(offsets), p(sorted_pairs), st), "b2q_moe_align")
        check(lib.b2q_qqq_moe_gather(p(x2), p(sorted_pairs), p(codes), p(s_x), T, top_k, K, code, st),
              "b2q_qqq_moe_gather")
        check(lib.b2q_qqq_moe_gate_up(p(codes), p(s_x), p(s1["packed"]), p(s1["sc"]), p(s1["sg"]), p(s3["packed"]),
                                      p(s3["sc"]), p(s3["sg"]), p(h), p(counts), p(offsets), E, rows, active, K, inter,
                                      s1["group"], code, st), "b2q_qqq_moe_gate_up")
        check(lib.b2q_qqq_quantize(p(h), p(codes_h), p(s_h), rows, inter, code, st), "b2q_qqq_quantize")
        check(lib.b2q_qqq_moe_down(p(codes_h), p(s_h), p(s2["packed"]), p(s2["sc"]), p(s2["sg"]), p(counts),
                                   p(offsets), p(sorted_pairs), p(wts), p(ypair), E, rows, active, inter, Kout,
                                   s2["group"], code, st), "b2q_qqq_moe_down")
        check(lib.b2q_moe_combine(p(ypair), p(y), T, top_k, Kout, code, st), "b2q_moe_combine")
        return y

    def _forward_grouped_fp8(self, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor) -> torch.Tensor:
        """FP8 (W8A16) experts: align -> gather -> gate|up -> down -> combine on the grouped small-batch kernels."""
        from ._lib import check, lib

        T, top_k = topk_ids.shape
        rows, E = T * top_k, self.num_experts
        s1, s3, s2 = self._stack["w1"], self._stack["w3"], self._stack["w2"]
        K, inter, Kout = s1["K"], s1["N"], s2["N"]
        self._check_x(x, T, top_k, K, topk_weights, s1["packed"].device)
        dev, dt = x.device, x.dtype
        if dt == torch.float16 and not all(s["fp16_ok"] for s in (s1, s3, s2)):
            raise ValueError("MoEExperts: a weight_scale_inv of the FP8 experts overflows fp16 (> 65504): fp16 "
                             "activations would give zero weights; run this block in bf16")
        code = 0 if dt == torch.float16 else 1
        st = torch.cuda.current_stream(dev).cuda_stream
        ids = topk_ids.to(torch.int32).contiguous()
        wts = topk_weights.to(torch.float32).contiguous()
        x2 = x.contiguous()
        if x2.data_ptr() % 16 != 0:
            x2 = x2.clone()
        p = lambda t: t.data_ptr()  # noqa: E731
        tables = torch.empty(2 * E + rows, dtype=torch.int32, device=dev)
        counts, offsets, sorted_pairs = tables[:E], tables[E:2 * E], tables[2 * E:]
        xs = torch.empty((rows, K), dtype=dt, device=dev)
        h = torch.empty((rows, inter), dtype=dt, device=dev)
        ypair = torch.empty((rows, Kout), dtype=torch.float32, device=dev)
        y = torch.empty((T, Kout), dtype=dt, device=dev)
        active = min(E, rows)
        check(lib.b2q_moe_align(p(ids), T, top_k, E, p(counts), p(offsets), p(sorted_pairs), st), "b2q_moe_align")
        check(lib.b2q_moe_gather(p(x2), p(sorted_pairs), p(xs), rows, top_k, K, st), "b2q_moe_gather")
        check(lib.b2q_fp8_moe_gate_up(p(xs), p(s1["packed"]), p(s1["scales"][dt]), p(s3["packed"]),
                                      p(s3["scales"][dt]), p(h), p(counts), p(offsets), E, rows, active, K, inter,
                                      s1["group"], code, st), "b2q_fp8_moe_gate_up")
        check(lib.b2q_fp8_moe_down(p(h), p(s2["packed"]), p(s2["scales"][dt]), p(counts), p(offsets), p(sorted_pairs),
                                   p(wts), p(ypair), E, rows, active, inter, Kout, s2["group"], code, st),
              "b2q_fp8_moe_down")
        check(lib.b2q_moe_combine(p(ypair), p(y), T, top_k, Kout, code, st), "b2q_moe_combine")
        return y

    def _forward_grouped_fp8blk(self, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor) -> torch.Tensor:
        """Block-FP8 experts: align -> gather-and-quantise -> gate|up -> quantise h -> down -> combine (include/b2q.h)."""
        from ._lib import check, lib

        if x.dtype not in (torch.float16, torch.bfloat16):
            raise ValueError(f"MoEExperts: block-FP8 experts take fp16 / bf16 activations, got {x.dtype}")
        T, top_k = topk_ids.shape
        rows, E = T * top_k, self.num_experts
        dev, dt = x.device, x.dtype
        code = 0 if dt == torch.float16 else 1
        s1, s3, s2 = self._stack["w1"], self._stack["w3"], self._stack["w2"]
        K, inter, Kout = s1["K"], s1["N"], s2["N"]
        # the gather kernel reads x [T, K] by token index: a mismatched x would be read out of bounds
        if tuple(x.shape) != (T, K) or dev != s1["weight"].device or tuple(topk_weights.shape) != (T, top_k):
            raise ValueError(f"MoEExperts: x {tuple(x.shape)} on {dev} does not fit [{T}, {K}] on {s1['weight'].device}, "
                             f"or topk_weights {tuple(topk_weights.shape)} is not [{T}, {top_k}]")
        st = torch.cuda.current_stream(dev).cuda_stream
        ids = topk_ids.to(torch.int32).contiguous()
        wts = topk_weights.to(torch.float32).contiguous()
        x2 = x.contiguous()
        if x2.data_ptr() % 16 != 0:
            x2 = x2.clone()
        p = lambda t: t.data_ptr()  # noqa: E731
        mp = (rows + 3) // 4 * 4  # token-scale row length of the quantiser's [K/128, Mp] layout
        tables = torch.empty(2 * E + rows, dtype=torch.int32, device=dev)
        counts, offsets, sorted_pairs = tables[:E], tables[E:2 * E], tables[2 * E:]
        codes = torch.empty((rows, K), dtype=torch.uint8, device=dev)
        s_x = torch.empty((K // 128, mp), dtype=torch.float32, device=dev)
        h = torch.empty((rows, inter), dtype=dt, device=dev)
        codes_h = torch.empty((rows, inter), dtype=torch.uint8, device=dev)
        s_h = torch.empty((inter // 128, mp), dtype=torch.float32, device=dev)
        ypair = torch.empty((rows, Kout), dtype=torch.float32, device=dev)
        y = torch.empty((T, Kout), dtype=dt, device=dev)
        active = min(E, rows)
        check(lib.b2q_moe_align(p(ids), T, top_k, E, p(counts), p(offsets), p(sorted_pairs), st), "b2q_moe_align")
        check(lib.b2q_fp8blk_moe_gather(p(x2), p(sorted_pairs), p(codes), p(s_x), T, top_k, K, code, st),
              "b2q_fp8blk_moe_gather")
        check(lib.b2q_fp8blk_moe_gate_up(p(codes), p(s_x), p(s1["weight"]), p(s1["scale"]), p(s3["weight"]),
                                         p(s3["scale"]), p(h), p(counts), p(offsets), E, rows, active, K, inter, code, 0,
                                         st), "b2q_fp8blk_moe_gate_up")
        check(lib.b2q_fp8blk_quantize(p(h), p(codes_h), p(s_h), rows, inter, code, st), "b2q_fp8blk_quantize")
        check(lib.b2q_fp8blk_moe_down(p(codes_h), p(s_h), p(s2["weight"]), p(s2["scale"]), p(counts), p(offsets),
                                      p(sorted_pairs), p(wts), p(ypair), E, rows, active, inter, Kout, code, 0, st),
              "b2q_fp8blk_moe_down")
        check(lib.b2q_moe_combine(p(ypair), p(y), T, top_k, Kout, code, st), "b2q_moe_combine")
        return y

    @staticmethod
    def _kernel_zeros(m):
        """The zero points of one expert in the layout the kernels read (int32 [G, N * kbits / 32]): the widened tensor of
        an asymmetric module, the kbits symmetric word for a symmetric one."""
        if m._zeros_dev is not None:
            return m._zeros_dev
        zsym = {4: 0x88888888 - (1 << 32), 8: 0x80808080 - (1 << 32)}[m.kbits]
        return torch.full((m.scales.shape[0], m.out_features * m.kbits // 32), zsym, dtype=torch.int32,
                          device=m.packed.device)

    def _scales(self, name, dtype):
        d = self._stack[name]["scales"]
        if dtype not in d:
            d[dtype] = next(iter(d.values())).to(dtype).contiguous()
        return d[dtype]

    def _forward_grouped(self, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor) -> torch.Tensor:
        from ._lib import check, lib

        T, top_k = topk_ids.shape
        rows, E = T * top_k, self.num_experts
        dev, dt = x.device, x.dtype
        code = 0 if dt == torch.float16 else 1
        st = torch.cuda.current_stream(dev).cuda_stream
        s1, s3, s2 = self._stack["w1"], self._stack["w3"], self._stack["w2"]
        K, inter, Kout = s1["K"], s1["N"], s2["N"]
        ids = topk_ids.to(torch.int32).contiguous()
        wts = topk_weights.to(torch.float32).contiguous()
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        if T == 1 and self.decode_path and self._decode_ok(top_k):
            # batch-1 decode: the token's top_k experts on the decode tier, three launches (include/b2q.h: b2q_moe_decode_*)
            x2 = x.contiguous()
            gu = torch.empty((2 * top_k, inter), dtype=dt, device=dev)
            h = torch.empty((top_k, inter), dtype=dt, device=dev)
            y = torch.empty((1, Kout), dtype=dt, device=dev)
            check(lib.b2q_moe_decode_gate_up(p(x2), p(s1["packed"]), p(self._scales("w1", dt)), p(s1["zeros"]),
                                             p(s3["packed"]), p(self._scales("w3", dt)), p(s3["zeros"]), p(ids), top_k, E, K,
                                             inter, 4, s1["group"], code, p(gu), st), "b2q_moe_decode_gate_up")
            if self.fuse_act:  # SiLU-mul computed by the down launch while it stages its activations: two launches
                check(lib.b2q_moe_decode_down(p(gu), p(s2["packed"]), p(self._scales("w2", dt)), p(s2["zeros"]), p(ids),
                                              p(wts), top_k, E, inter, Kout, 4, s2["group"], code, 1, p(y), st),
                      "b2q_moe_decode_down")
                return y
            check(lib.b2q_moe_decode_act(p(gu), p(h), top_k, inter, code, st), "b2q_moe_decode_act")
            check(lib.b2q_moe_decode_down(p(h), p(s2["packed"]), p(self._scales("w2", dt)), p(s2["zeros"]), p(ids), p(wts),
                                          top_k, E, inter, Kout, 4, s2["group"], code, 0, p(y), st), "b2q_moe_decode_down")
            return y
        tables = torch.empty(2 * E + rows, dtype=torch.int32, device=dev)
        counts, offsets, sorted_pairs = tables[:E], tables[E:2 * E], tables[2 * E:]
        x2 = x.contiguous()
        xs = torch.empty((rows, K), dtype=dt, device=dev)
        h = torch.empty((rows, inter), dtype=dt, device=dev)
        ypair = torch.empty((rows, Kout), dtype=torch.float32, device=dev)
        y = torch.empty((T, Kout), dtype=dt, device=dev)
        active = min(E, rows)
        check(lib.b2q_moe_align(p(ids), T, top_k, E, p(counts), p(offsets), p(sorted_pairs), st), "b2q_moe_align")
        if s1["perm"] is None:
            check(lib.b2q_moe_gather(p(x2), p(sorted_pairs), p(xs), rows, top_k, K, st), "b2q_moe_gather")
        else:  # act-order w1 / w3: every expert's rows gathered in its own column order
            check(lib.b2q_moe_gather_perm(p(x2), p(sorted_pairs), p(s1["perm"]), p(offsets), E, p(xs), rows, top_k, K, st),
                  "b2q_moe_gather_perm")
        check(lib.b2q_moe_gate_up(p(xs), p(s1["packed"]), p(self._scales("w1", dt)), p(s1["zeros"]), p(s3["packed"]),
                                  p(self._scales("w3", dt)), p(s3["zeros"]), p(h), p(counts), p(offsets), E, rows, active,
                                  K, inter, s1["bits"], s1["group"], code, st), "b2q_moe_gate_up")
        if s2["perm"] is not None:  # act-order w2: h permuted per expert (its rows are already in expert order)
            h2 = torch.empty_like(h)
            check(lib.b2q_moe_gather_perm(p(h), None, p(s2["perm"]), p(offsets), E, p(h2), rows, top_k, inter, st),
                  "b2q_moe_gather_perm")
            h = h2
        check(lib.b2q_moe_down(p(h), p(s2["packed"]), p(self._scales("w2", dt)), p(s2["zeros"]), p(counts), p(offsets),
                               p(sorted_pairs), p(wts), p(ypair), E, rows, active, inter, Kout, s2["bits"], s2["group"],
                               code, st), "b2q_moe_down")
        check(lib.b2q_moe_combine(p(ypair), p(y), T, top_k, Kout, code, st), "b2q_moe_combine")
        return y

    def _decode_ok(self, top_k: int) -> bool:
        """The decode tier's envelope for the one-token path: 4-bit experts without act-order, K % 128 == 0 on both
        matmuls, group_size 64 / 128 / K, top_k in {2, 4, 8} (cluster size of the down launch)."""
        s1, s2 = self._stack["w1"], self._stack["w2"]
        ok_g = lambda s: s["group"] in (64, 128, s["K"])  # noqa: E731
        return (top_k in (2, 4, 8) and s1["bits"] == 4 and s2["bits"] == 4 and s1["perm"] is None
                and s2["perm"] is None and s1["K"] % 128 == 0 and s2["K"] % 128 == 0 and s1["N"] % 32 == 0
                and s2["N"] % 32 == 0 and ok_g(s1) and ok_g(s2))

    @property
    def num_experts(self) -> int:
        return len(self.w1)

    def forward(self, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor) -> torch.Tensor:
        """x [T, K]; topk_ids / topk_weights [T, top_k] (weights already normalised) -> [T, K_out] (all-reduced)."""
        T, top_k = topk_ids.shape
        if self._stack is not None and x.is_cuda and x.dim() == 2:
            if "fp8blk" in self._stack:
                out = self._forward_grouped_fp8blk(x, topk_ids, topk_weights)
            elif "qqq" in self._stack:
                out = self._forward_grouped_qqq(x, topk_ids, topk_weights)
            elif "fp8" in self._stack:
                out = self._forward_grouped_fp8(x, topk_ids, topk_weights)
            else:
                out = self._forward_grouped(x, topk_ids, topk_weights)
            if self.reduce is not None and out.numel() <= self.reduce.max_elems and out.numel() % 8 == 0:
                return self.reduce(out.contiguous())
            return tp.all_reduce_sum_(out, self.group)
        flat_e = topk_ids.reshape(-1)
        order = torch.argsort(flat_e, stable=True)             # (token, k) pairs sorted by expert
        tok = order // top_k
        counts = torch.bincount(flat_e, minlength=self.num_experts).tolist()  # one host sync per block, like the
        xs = x.index_select(0, tok)                                            # reference's per-expert Python loop
        wts = topk_weights.reshape(-1).index_select(0, order).to(torch.float32)
        out = None
        start = 0
        for e, cnt in enumerate(counts):
            if cnt == 0:
                continue
            blk = xs[start:start + cnt]
            h = F.silu(self.w1[e](blk)) * self.w3[e](blk)
            y = self.w2[e](h)
            if out is None:
                out = torch.zeros((T, y.shape[-1]), dtype=torch.float32, device=x.device)
            out.index_add_(0, tok[start:start + cnt], y.float() * wts[start:start + cnt, None])
            start += cnt
        if out is None:
            raise ValueError("MoEExperts.forward: empty routing")
        out = out.to(x.dtype)
        if self.reduce is not None and out.numel() <= self.reduce.max_elems and out.numel() % 8 == 0:
            return self.reduce(out.contiguous())
        return tp.all_reduce_sum_(out, self.group)


class B200ChannelW8A8Experts(MoEExperts):
    """`MoEExperts` over per-channel / per-tensor W8A8 experts (B200ChannelFp8Linear or B200ChannelInt8Linear) that runs
    the block on the grouped kernels: align -> gather-and-quantise -> gate|up -> quantise h -> down -> combine, six
    launches with no host synchronisation (include/b2q.h states the rounding points, those of the per-expert loop).

    The stack qualifies when every w1 / w3 / w2 is a post_init'ed module of one of the two classes, with one activation
    kind and one ``ub`` across the block, no bias or adapter, one device, w1 / w3 [inter, K] and w2 [Kout, inter] with
    inter % 128 == 0, at most 256 experts, and (static activations) ``w1.input_scale == w3.input_scale`` for every expert,
    since both quantise the same gathered rows.  Otherwise ``grouped=None`` keeps the inherited loop and ``grouped=True``
    raises a ValueError naming the failed condition.  ``ks`` pins the split-K ranks of both grouped GEMMs (0: the
    heuristic)."""

    ks = 0

    def _w8a8_refusal(self):
        """None when the experts qualify for the grouped W8A8 kernels, else the reason they do not."""
        from .fp8_channel import B200ChannelFp8Linear
        from .int8_channel import B200ChannelInt8Linear

        w1, w3, w2 = list(self.w1), list(self.w3), list(self.w2)
        every = w1 + w3 + w2
        cls = type(every[0])
        if cls not in (B200ChannelFp8Linear, B200ChannelInt8Linear) or any(type(m) is not cls for m in every):
            return "experts must all be B200ChannelFp8Linear or all B200ChannelInt8Linear modules"
        if len(w1) > 256:
            return f"at most 256 experts, got {len(w1)}"
        if not all(m._ready for m in every):
            return "every expert module must be post_init'ed"
        if any(m.bias is not None for m in every):
            return "expert modules must have no bias"
        if any(m.adapter for m in every):
            return "expert modules must have no adapter"
        if len({m.weight.device for m in every}) != 1:
            return "expert modules must live on one device"
        if len({(m.activation, m.ub) for m in every}) != 1:
            return "every expert module must have the same activation kind and ub"
        K, inter = w1[0].in_features, w1[0].out_features
        Kout = w2[0].out_features
        if any((m.in_features, m.out_features) != (K, inter) for m in w1 + w3):
            return f"w1 and w3 must all be [{inter}, {K}]"
        if any((m.in_features, m.out_features) != (inter, Kout) for m in w2):
            return f"w2 must all be [{Kout}, {inter}]"
        if inter % 128 != 0:
            return f"the intermediate size {inter} must be a multiple of 128"
        if w1[0].activation == "static":
            for e, (a, b) in enumerate(zip(w1, w3)):
                if not torch.equal(a.input_scale, b.input_scale):
                    return f"expert {e}: w1 and w3 quantise the same rows, so their input_scale must be equal"
        return None

    def _build_stack(self):
        """Stack the experts' checkpoint tensors (weight [E, N, K], weight_scale [E, N] fp32, static input_scale [E]) once
        per role; the modules keep views into the stacks.  None (and the reason in `_refusal`) if they do not qualify."""
        self._refusal = self._w8a8_refusal()
        if self._refusal is not None:
            return None
        from .int8_channel import B200ChannelInt8Linear

        m0 = self.w1[0]
        out = {"w8a8": True, "int8": isinstance(m0, B200ChannelInt8Linear), "static": m0.activation == "static",
               "ub": float("inf") if m0.ub is None else m0.ub}
        for name, mods in (("w1", self.w1), ("w3", self.w3), ("w2", self.w2)):
            weight = torch.stack([m.weight.view(torch.uint8) for m in mods]).view(m0.CODE_DTYPE)
            scale = torch.stack([m.weight_scale for m in mods])
            s_in = torch.cat([m.input_scale.reshape(1) for m in mods]) if out["static"] else None
            for e, m in enumerate(mods):  # the modules keep working on their own; no second copy of the weights
                m.weight = weight[e]
                m.weight_scale = scale[e]
            out[name] = dict(weight=weight, scale=scale, s_in=s_in, K=mods[0].in_features, N=mods[0].out_features)
        return out

    def _forward_grouped(self, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor) -> torch.Tensor:
        """align -> gather-and-quantise -> gate|up -> quantise h -> down -> combine (include/b2q.h)."""
        from ._lib import check, lib

        T, top_k = topk_ids.shape
        rows, E = T * top_k, self.num_experts
        s1, s3, s2 = self._stack["w1"], self._stack["w3"], self._stack["w2"]
        K, inter, Kout = s1["K"], s1["N"], s2["N"]
        self._check_x(x, T, top_k, K, topk_weights, s1["weight"].device)
        dev, dt = x.device, x.dtype
        code = 0 if dt == torch.float16 else 1
        st = torch.cuda.current_stream(dev).cuda_stream
        int8, static, ks = self._stack["int8"], self._stack["static"], int(self.ks)
        pre = "b2q_int8ch" if int8 else "b2q_fp8ch"
        ub = () if int8 else (self._stack["ub"],)  # the FP8 quantisers' amax bound (+inf: none)
        ids = topk_ids.to(torch.int32).contiguous()
        wts = topk_weights.to(torch.float32).contiguous()
        x2 = x.contiguous()
        if x2.data_ptr() % 16 != 0:
            x2 = x2.clone()
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        tables = torch.empty(2 * E + rows, dtype=torch.int32, device=dev)
        counts, offsets, sorted_pairs = tables[:E], tables[E:2 * E], tables[2 * E:]
        codes = torch.empty((rows, K), dtype=torch.uint8, device=dev)
        s_x = torch.empty(rows, dtype=torch.float32, device=dev)
        h = torch.empty((rows, inter), dtype=dt, device=dev)
        codes_h = torch.empty((rows, inter), dtype=torch.uint8, device=dev)
        s_h = torch.empty(rows, dtype=torch.float32, device=dev)
        ypair = torch.empty((rows, Kout), dtype=torch.float32, device=dev)
        y = torch.empty((T, Kout), dtype=dt, device=dev)
        active = min(E, rows)
        gather, gate_up, down = (getattr(lib, f"{pre}_moe_{n}") for n in ("gather", "gate_up", "down"))
        check(lib.b2q_moe_align(p(ids), T, top_k, E, p(counts), p(offsets), p(sorted_pairs), st), "b2q_moe_align")
        check(gather(p(x2), p(sorted_pairs), p(offsets), p(s1["s_in"]), E, p(codes), p(s_x), T, top_k, K, *ub, code, st),
              f"{pre}_moe_gather")
        check(gate_up(p(codes), p(s_x), p(s1["weight"]), p(s1["scale"]), p(s3["weight"]), p(s3["scale"]), p(h), p(counts),
                      p(offsets), E, rows, active, K, inter, code, ks, st), f"{pre}_moe_gate_up")
        if static:  # h is already in sorted order: each row takes its expert's w2 input_scale
            check(gather(p(h), None, p(offsets), p(s2["s_in"]), E, p(codes_h), p(s_h), rows, 1, inter, *ub, code, st),
                  f"{pre}_moe_gather")
        else:
            check(getattr(lib, f"{pre}_quantize")(p(h), p(codes_h), p(s_h), rows, inter, *ub, code, st), f"{pre}_quantize")
        check(down(p(codes_h), p(s_h), p(s2["weight"]), p(s2["scale"]), p(counts), p(offsets), p(sorted_pairs), p(wts),
                   p(ypair), E, rows, active, inter, Kout, code, ks, st), f"{pre}_moe_down")
        check(lib.b2q_moe_combine(p(ypair), p(y), T, top_k, Kout, code, st), "b2q_moe_combine")
        return y
