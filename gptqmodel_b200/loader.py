"""Checkpoint loader for real GPTQ / AWQ safetensors checkpoints.

What the reference does for this step, restated for this package (no model definitions, no accelerate):
  * the quantisation config is read from ``quantize_config.json``, ``quant_config.json`` or the ``quantization_config``
    entry of ``config.json``, in that order (gptqmodel/quantization/config.py:73-74), with the legacy
    aliases ``w_bit / wbits -> bits``, ``q_group_size -> group_size``, ``version / checkpoint_format -> format``,
    ``quant_method -> method`` and ``zero_point -> not sym`` (config.py:1504-1525);
  * ``dynamic`` maps module-name regexes to per-module overrides; the FIRST matching pattern wins, a ``-:`` prefix means
    "this module is not quantised", ``+:`` is an explicit positive match (config.py:1579-1652, 1822-1854);
  * a quantised linear ``<prefix>`` is stored as ``<prefix>.qweight / .qzeros / .scales / .g_idx [/ .bias]``
    (nn_modules/qlinear/__init__.py:827-865); AWQ GEMM checkpoints have no ``g_idx`` (:1634-1668);
  * ``format == "gptq"`` files hold v1 zero-points (stored as zero - 1): kernels that need the true zero-point get
    ``qzeros += 0x11111111`` (4-bit) / ``0x01010101`` (8-bit) at load (utils/model.py:800-846, models/loader.py:1657-1675);
    the reference refuses asymmetric v1 files that were not produced by its own >= 0.9.0 quantiser (loader.py:1659-1663).

`load_quantized_linears(path)` returns ``{prefix: module}`` with the tensors loaded (on `device`, post_init() run when
it is a CUDA device); wiring the modules into a model graph is the caller's business (the reference's
``make_quant`` / ``create_quant_module``, utils/model.py:475-649).
"""
from __future__ import annotations

import json
import os
import re
from dataclasses import dataclass, field
from typing import Dict, Iterable, Optional

import torch
import torch.nn as nn

QUANT_CONFIG_FILES = ("quantize_config.json", "quant_config.json", "config.json")
_ALIASES = {"w_bit": "bits", "wbits": "bits", "q_group_size": "group_size", "version": "format",
            "checkpoint_format": "format", "quant_method": "method"}
_TENSOR_SUFFIXES = ("qweight", "qzeros", "scales", "g_idx", "bias")


@dataclass
class QuantSpec:
    bits: int = 4
    group_size: int = 128
    desc_act: bool = False
    sym: bool = True
    format: str = "gptq"   # "gptq" (v1 zero-points) | "gptq_v2" | "gptq_p" (planar, v2 zero-points) | "gemm" (AWQ)
    method: str = "gptq"   # "gptq" | "awq"
    lm_head: bool = False
    dynamic: Optional[Dict[str, dict]] = None
    meta: dict = field(default_factory=dict)

    def for_module(self, name: str) -> Optional["QuantSpec"]:
        """Per-module view after `dynamic` overrides; None if a negative (`-:`) pattern excludes the module."""
        if not self.dynamic:
            return self
        for pattern, overrides in self.dynamic.items():  # first match wins, in file order
            negative = pattern.startswith("-:")
            raw = pattern[2:] if pattern.startswith(("-:", "+:")) else pattern
            if re.match(raw, name):
                if negative:
                    return None
                out = QuantSpec(**{**self.__dict__, "dynamic": None})
                for k, v in (overrides or {}).items():
                    k = _ALIASES.get(k, k)
                    if k in ("bits", "group_size"):
                        setattr(out, k, int(v))
                    elif k in ("desc_act", "sym"):
                        setattr(out, k, bool(v))
                return out
        return self


def parse_quant_config(raw: dict) -> QuantSpec:
    """Normalise a quantisation-config dict (any of the spellings the reference accepts) into a QuantSpec."""
    d = {}
    for k, v in raw.items():
        if k == "zero_point":  # AutoAWQ: zero_point=True means asymmetric
            d["sym"] = not bool(v)
        else:
            d.setdefault(_ALIASES.get(k, k), v)
    if "is_marlin_format" in raw:
        raise ValueError("`is_marlin_format` checkpoints are not supported (the reference rejects them as well)")
    spec = QuantSpec()
    spec.bits = int(d.get("bits", spec.bits))
    spec.group_size = int(d.get("group_size", spec.group_size))
    spec.desc_act = bool(d.get("desc_act", False))
    spec.sym = bool(d.get("sym", True))
    spec.method = str(d.get("method", "gptq")).lower()
    fmt = d.get("format")
    spec.format = str(fmt).lower() if fmt is not None else ("gemm" if spec.method == "awq" else "gptq")
    spec.lm_head = bool(d.get("lm_head", False))
    spec.dynamic = d.get("dynamic") or None
    spec.meta = dict(d.get("meta") or {})
    pack_dtype = str(d.get("pack_dtype", "int32")).replace("torch.", "")
    if pack_dtype != "int32":
        raise NotImplementedError(f"pack_dtype `{pack_dtype}` is not supported (int32 words only, like Marlin / Swordfish)")
    if spec.method not in ("gptq", "awq"):
        raise NotImplementedError(f"quantisation method `{spec.method}` is outside this package (gptq, awq)")
    if spec.method == "gptq" and spec.format not in ("gptq", "gptq_v2", "gptq_p"):
        raise NotImplementedError(f"GPTQ checkpoint format `{spec.format}` is not supported (gptq, gptq_v2, gptq_p)")
    if spec.method == "awq" and spec.format != "gemm":
        raise NotImplementedError(f"AWQ checkpoint format `{spec.format}` is not supported (gemm)")
    return spec


def read_quant_config(path: str) -> QuantSpec:
    for fn in QUANT_CONFIG_FILES:
        p = os.path.join(path, fn)
        if not os.path.exists(p):
            continue
        with open(p) as f:
            raw = json.load(f)
        if fn == "config.json":
            raw = raw.get("quantization_config")
            if raw is None:
                continue
        return parse_quant_config(raw)
    raise FileNotFoundError(f"no quantisation config ({', '.join(QUANT_CONFIG_FILES)}) under {path}")


def _weight_map(path: str) -> Dict[str, str]:
    """tensor name -> safetensors file (single file or sharded with model.safetensors.index.json)."""
    idx = os.path.join(path, "model.safetensors.index.json")
    if os.path.exists(idx):
        with open(idx) as f:
            return {k: os.path.join(path, v) for k, v in json.load(f)["weight_map"].items()}
    from safetensors import safe_open

    files = sorted(fn for fn in os.listdir(path) if fn.endswith(".safetensors"))
    if not files:
        raise FileNotFoundError(f"no .safetensors file under {path}")
    out = {}
    for fn in files:
        with safe_open(os.path.join(path, fn), framework="pt") as f:
            for k in f.keys():
                out[k] = os.path.join(path, fn)
    return out


def quantized_prefixes(names: Iterable[str]) -> list:
    """Module prefixes that carry a packed weight (`<prefix>.qweight`)."""
    return sorted(n[: -len(".qweight")] for n in names if n.endswith(".qweight"))


def _v1_sym_ok(spec: QuantSpec) -> bool:
    # asymmetric v1 files are only trustworthy when written by the reference's own >= 0.9.0 code path
    # (models/loader.py:1659-1663, quantization/config.py:2786-2792: meta.quantizer = "gptqmodel:<version>");
    # everybody else's `qzeros - 1` may have wrapped
    if spec.sym:
        return True
    q = spec.meta.get("quantizer", [])
    for entry in ([q] if isinstance(q, str) else list(q)):
        producer, _, ver = str(entry).partition(":")
        if producer.strip().lower() == "gptqmodel":
            nums = [int(x) for x in re.findall(r"\d+", ver)[:3]]
            return tuple(nums + [0] * (3 - len(nums))) >= (0, 9, 0)
    return False


@torch.no_grad()
def load_quantized_linears(path: str, device="cuda", dtype: Optional[torch.dtype] = None,
                           only: Optional[Iterable[str]] = None, post_init: Optional[bool] = None) -> Dict[str, nn.Module]:
    """Load every quantised linear of a checkpoint directory into B200 QuantLinear modules.

    only      : optional iterable of module prefixes to load (default: all `<prefix>.qweight` found)
    post_init : default True on CUDA devices (prepack for the kernels), False on CPU (tensors only; host tests)
    """
    from safetensors import safe_open

    from .awq import B200AwqQuantLinear
    from .qlinear import B200QuantLinear

    spec = read_quant_config(path)
    wmap = _weight_map(path)
    prefixes = quantized_prefixes(wmap) if only is None else list(only)
    dev = torch.device(device)
    do_post = (dev.type == "cuda") if post_init is None else post_init
    handles: Dict[str, object] = {}

    def tensor(name):
        fn = wmap.get(name)
        if fn is None:
            return None
        if fn not in handles:
            handles[fn] = safe_open(fn, framework="pt").__enter__()
        return handles[fn].get_tensor(name)

    mods: Dict[str, nn.Module] = {}
    try:
        for prefix in prefixes:
            ms = spec.for_module(prefix)
            if ms is None:
                continue  # excluded by a negative dynamic pattern: stays a dense layer in the model
            t = {s: tensor(f"{prefix}.{s}") for s in _TENSOR_SUFFIXES}
            if t["qweight"] is None or t["qzeros"] is None or t["scales"] is None:
                raise KeyError(f"{prefix}: checkpoint misses qweight / qzeros / scales")
            mk = lambda x: None if x is None else nn.Parameter(x.contiguous().to(dev), requires_grad=False)  # noqa: E731
            if ms.method == "awq":
                K, N = t["qweight"].shape[0], t["qweight"].shape[1] * 32 // ms.bits
                m = B200AwqQuantLinear(bits=ms.bits, group_size=ms.group_size, in_features=K, out_features=N,
                                       bias=t["bias"] is not None, register_buffers=False, dtype=dtype, name=prefix)
                m.qweight, m.qzeros, m.scales, m.bias = mk(t["qweight"]), mk(t["qzeros"]), mk(t["scales"]), mk(t["bias"])
            else:
                K, N = t["qweight"].shape[0] * 32 // ms.bits, t["qweight"].shape[1]
                g_idx = t["g_idx"]
                gs = ms.group_size if ms.group_size > 0 else K
                if g_idx is None:
                    g_idx = (torch.arange(K, dtype=torch.int32) // gs)
                m = B200QuantLinear(bits=ms.bits, group_size=ms.group_size, desc_act=ms.desc_act, sym=ms.sym, in_features=K,
                                    out_features=N, bias=t["bias"] is not None, register_buffers=False, dtype=dtype,
                                    name=prefix, format=ms.format)
                m.qweight, m.qzeros, m.scales = mk(t["qweight"]), mk(t["qzeros"]), mk(t["scales"])
                m.g_idx, m.bias = mk(g_idx.to(torch.int32)), mk(t["bias"])
                if ms.format == "gptq":
                    if not _v1_sym_ok(ms):
                        raise ValueError(f"{prefix}: asymmetric checkpoint in GPTQ v1 format not written by gptqmodel >= 0.9.0 "
                                         "(zero-points may have wrapped); the reference refuses it as well")
                    m.qzero_format(1)
                    m.convert_gptq_v1_to_v2()
            if do_post:
                m.post_init()
            mods[prefix] = m
    finally:
        for h in handles.values():  # safe_open keeps the file mapped until closed (ADVICE r01)
            close = getattr(h, "__exit__", None)
            if close is not None:
                close(None, None, None)
        handles.clear()
    return mods
