"""Mixture-of-experts block over QuantLinear experts (BASELINE configs[4]: Mixtral-8x7B int4 g64 asym).

In the reference every expert's ``w1 / w3 / w2`` is an independent QuantLinear module
(gptqmodel/models/definitions/mixtral.py:30-34) that the model's own Python loop calls per expert; the
fused MoE kernel it ships (``swordfish_moe.cu``) is exported but never called.  This module is that
per-expert loop, arranged for the B200 kernels and for tensor parallelism:

  * ONE TOKEN (batch-1 decode) through grouped-eligible experts: three launches on the decode tier — the 2 * top_k gate / up
    matrices as sibling sets of one decode launch (experts read from `topk_ids` on the device), SiLU-mul, and a cluster of
    top_k CTAs per tile column for w2 whose DSMEM reduction applies the routing weights (`b2q_moe_decode_*`);
  * GROUPED path (default whenever every expert is a 4-bit B200 QuantLinear of one shape): the (token, k) pairs are sorted
    by expert ON THE DEVICE (`b2q_moe_align`), and the whole block is five launches with no host synchronisation —
    align, gather, ONE grouped launch for w1 and w3 with the SiLU-mul epilogue, ONE grouped launch for w2 with the routing
    weight + scatter epilogue, combine (gptqmodel_b200/csrc/b2q_moe.cu, grouped modes of b2q_midm.cu) — CUDA-graph
    capturable; the experts' prepacked tensors are stacked once (the per-expert modules keep views into the stack);
  * LOOP path (fallback: dense stand-ins in CPU tests, mixed experts): tokens are sorted by expert once, every expert sees one
    contiguous block of its routed tokens; one host sync per block for the per-expert counts, like the reference's loop;
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
        if grouped is None or grouped:
            self._stack = self._build_stack()
            if grouped and self._stack is None:
                raise ValueError("MoEExperts(grouped=True): experts must be post_init'ed 4-bit B200 QuantLinears of one "
                                 "shape / group size without act-order, bias or adapters")
        if fuse and self._stack is None:
            from .qlinear import B200KernelMixin, fuse_siblings

            for a, b in zip(self.w1, self.w3):
                if isinstance(a, B200KernelMixin) and isinstance(b, B200KernelMixin):
                    fuse_siblings([a, b])

    def _build_stack(self):
        """Stack the experts' prepacked tensors for the grouped kernels; None if the experts do not qualify."""
        from .qlinear import B200KernelMixin

        sets = []
        for mods in (self.w1, self.w3, self.w2):
            m0 = mods[0]
            for m in mods:
                if not isinstance(m, B200KernelMixin) or not m._prepacked or m.bits != 4 or m.perm is not None or m._gather is not None \
                        or m.bias is not None or m.adapter:
                    return None
                if (m.in_features, m.out_features, m.group_size, m.packed.device, m.scales.dtype) != (
                        m0.in_features, m0.out_features, m0.group_size, m0.packed.device, m0.scales.dtype):
                    return None
            sets.append(list(mods))
        w1, w3, w2 = sets
        if (w1[0].in_features, w1[0].out_features, w1[0].group_size) != (w3[0].in_features, w3[0].out_features,
                                                                         w3[0].group_size):
            return None
        if w2[0].in_features != w1[0].out_features:
            return None
        out = {}
        for name, mods in (("w1", w1), ("w3", w3), ("w2", w2)):
            asym = any(not m._is_sym for m in mods) if name == "w2" else any(not m._is_sym for m in w1 + w3)
            packed = torch.stack([m.packed for m in mods]).contiguous()
            scales = torch.stack([m.scales.data for m in mods]).contiguous()
            zeros = torch.stack([m.qzeros.data for m in mods]).contiguous() if asym else None
            for e, m in enumerate(mods):  # the modules keep working on their own; no second copy of the weights
                m.packed = packed[e]
                m.scales.data = scales[e]
                m._scales_cache.clear()
                if zeros is not None:
                    m.qzeros.data = zeros[e]
                    if m._zeros_dev is not None:
                        m._zeros_dev = zeros[e]
            out[name] = dict(packed=packed, scales={scales.dtype: scales}, zeros=zeros, K=mods[0].in_features,
                             N=mods[0].out_features, group=mods[0].group_size)
        return out

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
        check(lib.b2q_moe_gather(p(x2), p(sorted_pairs), p(xs), rows, top_k, K, st), "b2q_moe_gather")
        check(lib.b2q_moe_gate_up(p(xs), p(s1["packed"]), p(self._scales("w1", dt)), p(s1["zeros"]), p(s3["packed"]),
                                  p(self._scales("w3", dt)), p(s3["zeros"]), p(h), p(counts), p(offsets), E, rows, active,
                                  K, inter, 4, s1["group"], code, st), "b2q_moe_gate_up")
        check(lib.b2q_moe_down(p(h), p(s2["packed"]), p(self._scales("w2", dt)), p(s2["zeros"]), p(counts), p(offsets),
                               p(sorted_pairs), p(wts), p(ypair), E, rows, active, inter, Kout, 4, s2["group"], code, st),
              "b2q_moe_down")
        check(lib.b2q_moe_combine(p(ypair), p(y), T, top_k, Kout, code, st), "b2q_moe_combine")
        return y

    def _decode_ok(self, top_k: int) -> bool:
        """The decode tier's envelope for the one-token path: K % 128 == 0 on both matmuls, group_size 64 / 128 / K,
        top_k in {2, 4, 8} (cluster size of the down launch)."""
        s1, s2 = self._stack["w1"], self._stack["w2"]
        ok_g = lambda s: s["group"] in (64, 128, s["K"])  # noqa: E731
        return (top_k in (2, 4, 8) and s1["K"] % 128 == 0 and s2["K"] % 128 == 0 and s1["N"] % 32 == 0
                and s2["N"] % 32 == 0 and ok_g(s1) and ok_g(s2))

    @property
    def num_experts(self) -> int:
        return len(self.w1)

    def forward(self, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor) -> torch.Tensor:
        """x [T, K]; topk_ids / topk_weights [T, top_k] (weights already normalised) -> [T, K_out] (all-reduced)."""
        T, top_k = topk_ids.shape
        if self._stack is not None and x.is_cuda and x.dim() == 2:
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
