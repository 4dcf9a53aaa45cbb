"""Swap the nn.Linear modules of a model for B200 QuantLinears (the caller side of the hot path).

The reference does this in `make_quant` / `create_quant_module` (gptqmodel/utils/model.py:475-649): walk
the model, replace every targeted `nn.Linear` by the selected QuantLinear class, load the packed tensors, `post_init()`.
`replace_linears` is that walk.  `rtn_grid` + `quantize_linear` build the packed tensors from float weights with a plain
round-to-nearest grid (per-group min/max or abs-max) through the device-side packer — enough to turn any float model into
a GPTQ-layout model for tests and synthetic benchmarks; it is NOT a replacement for the reference's calibrated GPTQ / AWQ
quantisers (out of scope).
"""
from __future__ import annotations

from typing import Callable, Dict, Iterable, Optional

import torch
import torch.nn as nn

from .pack import pack_gptq


@torch.no_grad()
def rtn_grid(weight: torch.Tensor, bits: int, group_size: int, sym: bool):
    """weight [N, K] -> (scales [N, G], zeros [N, G]) of a round-to-nearest grid, groups of `group_size` along K."""
    N, K = weight.shape
    gs = group_size if group_size > 0 else K
    if K % gs != 0:
        raise ValueError(f"rtn_grid: K={K} is not a multiple of group_size={gs}")
    maxq = (1 << bits) - 1
    Wg = weight.float().reshape(N, K // gs, gs)
    if sym:
        half = (maxq + 1) // 2
        scales = Wg.abs().amax(dim=2).clamp(min=1e-8) / (half - 1)
        zeros = torch.full_like(scales, float(half))
    else:
        lo = Wg.amin(dim=2).clamp(max=0)
        hi = Wg.amax(dim=2).clamp(min=0)
        scales = ((hi - lo) / maxq).clamp(min=1e-8)
        zeros = torch.round(-lo / scales).clamp(0, maxq)
    return scales, zeros


@torch.no_grad()
def quantize_linear(linear: nn.Linear, bits: int = 4, group_size: int = 128, sym: bool = True, device=None,
                    dtype: Optional[torch.dtype] = None, name: Optional[str] = None) -> nn.Module:
    """nn.Linear -> B200QuantLinear holding its RTN-quantised weights (post_init() run when `device` is CUDA)."""
    from .qlinear import B200QuantLinear

    N, K = linear.weight.shape
    m = B200QuantLinear(bits=bits, group_size=group_size, desc_act=False, sym=sym, in_features=K, out_features=N,
                        bias=linear.bias is not None, register_buffers=False, dtype=dtype, name=name)
    scales, zeros = rtn_grid(linear.weight.data, bits, group_size, sym)
    m.pack_block(linear, scales, zeros)
    dev = torch.device(device) if device is not None else linear.weight.device
    for k in ("qweight", "qzeros", "scales", "g_idx", "bias"):
        t = getattr(m, k)
        if t is not None:
            setattr(m, k, nn.Parameter(t.data.to(dev), requires_grad=False))
    if dev.type == "cuda":
        m.post_init()
    return m


def replace_linears(model: nn.Module, factory: Callable[[str, nn.Linear], Optional[nn.Module]],
                    skip: Iterable[str] = ("lm_head",)) -> Dict[str, nn.Module]:
    """Replace every nn.Linear whose qualified name does not end with one of `skip` by `factory(name, linear)`
    (None = keep the dense layer).  Returns {name: new module}."""
    skip = tuple(skip)
    swapped: Dict[str, nn.Module] = {}
    for name, mod in list(model.named_modules()):
        if not isinstance(mod, nn.Linear) or any(name.endswith(s) for s in skip):
            continue
        new = factory(name, mod)
        if new is None:
            continue
        parent_name, _, child = name.rpartition(".")
        parent = model.get_submodule(parent_name) if parent_name else model
        setattr(parent, child, new)
        swapped[name] = new
    return swapped
