"""Fused neighbours of the GEMM: ``act_fn(gate_proj(x)) * up_proj(x)`` of a Llama-style MLP in ONE
launch with the SiLU-mul in the epilogue (module order in the reference's model definitions:
gptqmodel/models/definitions/llama.py:17-27 — gate_proj and up_proj are separate QuantLinear modules whose
outputs a Python expression combines: two matmul launches, one activation launch, one multiply launch).

The kernel is the two-weight-set mode of the small-batch tier (b2q_midm.cu MODE 1, the same launch the grouped MoE path uses
with one "expert"): both weight sets run through the pipeline back to back into two register accumulators, the epilogue rounds
at the module boundaries exactly like the separate modules would (g = T(x W_gate), a = T(silu(g)), u = T(x W_up),
h = T(a * u)) and stores h only — the two [M, intermediate] intermediates never reach HBM.  Serves 1 <= tokens <= 128 per
call (larger batches: `forward` falls back to the two modules' own tiers + torch ops).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from ._lib import check, lib
from .qlinear import B200KernelMixin


class FusedGateUpSilu(torch.nn.Module):
    def __init__(self, gate: B200KernelMixin, up: B200KernelMixin):
        super().__init__()
        for m in (gate, up):
            if not isinstance(m, B200KernelMixin) or not m._prepacked or m.bits != 4 or m.perm is not None or m._gather is not None \
                    or m.bias is not None or m.adapter:
                raise NotImplementedError("FusedGateUpSilu: post_init'ed 4-bit B200 QuantLinears without act-order, bias "
                                          "or adapter")
        if (gate.in_features, gate.out_features, gate.group_size, gate._is_sym) != (
                up.in_features, up.out_features, up.group_size, up._is_sym):
            raise NotImplementedError("FusedGateUpSilu: gate_proj and up_proj must share shape, group size and symmetry")
        self.gate, self.up = gate, up
        self._tables = {}  # tokens -> int32 [2] = {count, offset 0} on the device (created outside graph capture)

    def _table(self, M: int, device) -> torch.Tensor:
        t = self._tables.get((M, device))
        if t is None:
            t = torch.tensor([M, 0], dtype=torch.int32, device=device)
            self._tables[(M, device)] = t
        return t

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        g, u = self.gate, self.up
        K, N = g.in_features, g.out_features
        x2 = x.reshape(-1, K)
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        M = x2.shape[0]
        if M == 0 or M > 128:
            return F.silu(g(x)) * u(x)
        tab = self._table(M, x.device)
        h = torch.empty((M, N), dtype=x.dtype, device=x.device)
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        check(lib.b2q_moe_gate_up(p(x2), p(g.packed), p(g._scales_for(x.dtype)), p(g._zeros_dev), p(u.packed),
                                  p(u._scales_for(x.dtype)), p(u._zeros_dev), p(h), tab.data_ptr(), tab.data_ptr() + 4,
                                  1, M, 1, K, N, 4, g.group_size, 0 if x.dtype == torch.float16 else 1,
                                  torch.cuda.current_stream(x.device).cuda_stream), "b2q_moe_gate_up")
        return h.reshape(x.shape[:-1] + (N,))
