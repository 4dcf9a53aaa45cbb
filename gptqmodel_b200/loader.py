"""Checkpoint loader for real GPTQ / AWQ safetensors checkpoints.

What the reference does for this step, restated for this package (no model definitions, no accelerate):
  * the quantisation config is read from ``quantize_config.json``, ``quant_config.json`` or the ``quantization_config``
    entry of ``config.json``, in that order (gptqmodel/quantization/config.py:73-74), with the legacy
    aliases ``w_bit / wbits -> bits``, ``q_group_size -> group_size``, ``version / checkpoint_format -> format``,
    ``quant_method -> method`` and ``zero_point -> not sym`` (config.py:1504-1525);
  * ``dynamic`` maps module-name regexes to per-module overrides; the FIRST matching pattern wins, a ``-:`` prefix means
    "this module is not quantised", ``+:`` is an explicit positive match (config.py:1579-1652, 1822-1854);
  * a quantised linear ``<prefix>`` is stored as ``<prefix>.qweight / .qzeros / .scales / .g_idx [/ .bias]``
    (nn_modules/qlinear/__init__.py:827-865); AWQ GEMM checkpoints have no ``g_idx`` (:1634-1668); QQQ (W4A8)
    checkpoints store ``<prefix>.B / .s_channel / .s_group [/ .bias]`` (nn_modules/qlinear/qqq.py); FP8 checkpoints
    ``<prefix>.weight`` (float8_e4m3fn) ``/ .weight_scale_inv [/ .bias]`` (nn_modules/qlinear/fp8.py);
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
    method: str = "gptq"   # "gptq" | "awq" | "qqq" | "fp8"
    lm_head: bool = False
    dynamic: Optional[Dict[str, dict]] = None
    meta: dict = field(default_factory=dict)
    rotation: Optional[str] = None  # None | "hadamard" | "random": QuaRot / SpinQuant checkpoint, see load_quantized_linears
    # FP8 checkpoints (method "fp8"): the e4m3 format and the scale layout of the reference's FP8Config
    fp8_format: str = "float8_e4m3fn"
    weight_scale_method: Optional[str] = None
    weight_block_size: Optional[tuple] = None

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
                if self.method == "fp8":
                    _fp8_override(out, name, overrides or {})
                    return out
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
    spec.rotation = d.get("rotation") or None
    pack_dtype = str(d.get("pack_dtype", "int32")).replace("torch.", "")
    if pack_dtype != "int32":
        raise NotImplementedError(f"pack_dtype `{pack_dtype}` is not supported (int32 words only, like Marlin / Swordfish)")
    if spec.method not in ("gptq", "awq", "qqq", "fp8"):
        raise NotImplementedError(f"quantisation method `{spec.method}` is outside this package (gptq, awq, qqq, fp8)")
    if spec.method == "fp8":
        _parse_fp8(spec, raw)
        return spec
    if spec.method == "qqq":
        if fmt is None:
            spec.format = "qqq"
        _check_qqq(spec)
    if spec.method == "gptq" and spec.format not in ("gptq", "gptq_v2", "gptq_p"):
        raise NotImplementedError(f"GPTQ checkpoint format `{spec.format}` is not supported (gptq, gptq_v2, gptq_p)")
    if spec.method == "awq" and spec.format != "gemm":
        raise NotImplementedError(f"AWQ checkpoint format `{spec.format}` is not supported (gemm)")
    # the reference's checks for rotated checkpoints (models/loader.py:283-284, 1392-1396)
    if spec.rotation is not None:
        if spec.rotation not in ("hadamard", "random"):
            raise ValueError(f"Unsupported rotation mode: `{spec.rotation}`")
        if spec.method != "gptq" or spec.format not in ("gptq", "gptq_v2"):
            raise NotImplementedError(f"`rotation` is only supported for GPTQ/GPTQ_V2 checkpoints, got `{spec.format}`")
    return spec


def _check_qqq(spec: QuantSpec) -> None:
    """QQQ (W4A8) checkpoints: 4-bit, symmetric, group size -1 or 128 (the reference's QQQLinear), no rotation."""
    if spec.format != "qqq":
        raise NotImplementedError(f"QQQ checkpoint format `{spec.format}` is not supported (qqq)")
    if spec.bits != 4 or spec.group_size not in (-1, 128) or not spec.sym:
        raise NotImplementedError(f"QQQ: bits={spec.bits} group_size={spec.group_size} sym={spec.sym} unsupported "
                                  "(4-bit, group size -1 or 128, symmetric)")
    if spec.rotation is not None:
        raise NotImplementedError("`rotation` is not supported for QQQ checkpoints")


def _parse_fp8(spec: QuantSpec, raw: dict) -> None:
    """FP8 configs as the reference's FP8Config writes them: `format` (or the legacy `fmt`) names the e4m3 dtype,
    `weight_scale_method` / `weight_block_size` / `weight_scale_semantics` the scales, group size and act-order do not
    apply.  HF / DeepSeek-native FP8 configs (`activation_scheme`, or `fmt` without `format`) store a `weight_scale_inv`
    that MULTIPLIES the weights; serving them with this package's division would give wrong outputs, so they are refused."""
    from .fp8 import normalize_block_size, normalize_fp8_format, normalize_scale_method, normalize_scale_semantics

    if "activation_scheme" in raw or ("fmt" in raw and "format" not in raw):
        raise NotImplementedError("HF / DeepSeek-native FP8 checkpoints (weight_scale_inv as a multiplier) are not "
                                  "served here (this entry point reads the reference's FP8Config, weight = w / "
                                  "weight_scale_inv); load block-FP8 checkpoints with parse_block_fp8_config / "
                                  "load_block_fp8_linears")
    if raw.get("rotation"):
        raise NotImplementedError("`rotation` is not supported for FP8 checkpoints")
    if int(raw.get("bits", 8)) != 8:
        raise ValueError("FP8: `bits` must be 8")
    fmt = raw.get("format", raw.get("fmt"))
    spec.fp8_format = normalize_fp8_format(fmt)
    spec.format = "fp8"
    spec.bits, spec.group_size, spec.desc_act, spec.sym = 8, -1, False, True
    spec.weight_block_size = normalize_block_size(raw.get("weight_block_size"))
    spec.weight_scale_method = normalize_scale_method(raw.get("weight_scale_method"), spec.weight_block_size)
    normalize_scale_semantics(raw.get("weight_scale_semantics"))
    for layer, overrides in (spec.dynamic or {}).items():
        if not layer.startswith("-:"):
            _fp8_override(QuantSpec(**{**spec.__dict__, "dynamic": None}), layer, overrides or {})


def _fp8_override(out: QuantSpec, name: str, overrides: dict) -> None:
    """Apply one `dynamic` entry of an FP8 config (the reference's per-layer rules) to a module's spec."""
    from .fp8 import normalize_block_size, normalize_fp8_format, normalize_scale_method, normalize_scale_semantics

    if "bits" in overrides and int(overrides["bits"]) != 8:
        raise ValueError(f"FP8: layer `{name}` only supports 8-bit FP8 weights")
    if overrides.get("group_size") not in (-1, None):
        raise ValueError("FP8: `group_size` is not used; keep it at `-1`")
    fmt = overrides.get("format", overrides.get("fmt"))
    if fmt is not None:
        out.fp8_format = normalize_fp8_format(fmt)
    block = normalize_block_size(overrides.get("weight_block_size"))
    if "weight_scale_method" in overrides or block is not None:
        out.weight_scale_method = normalize_scale_method(overrides.get("weight_scale_method"), block)
        out.weight_block_size = block
    if "weight_scale_semantics" in overrides:
        normalize_scale_semantics(overrides["weight_scale_semantics"])


def fp8_prefixes(names: Iterable[str]) -> list:
    """Module prefixes of an FP8 checkpoint (`<prefix>.weight_scale_inv` together with `<prefix>.weight`)."""
    names = set(names)
    sfx = ".weight_scale_inv"
    return sorted(n[: -len(sfx)] for n in names if n.endswith(sfx) and n[: -len(sfx)] + ".weight" in names)


def _read_raw_config(path: str) -> dict:
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
        return raw
    raise FileNotFoundError(f"no quantisation config ({', '.join(QUANT_CONFIG_FILES)}) under {path}")


def read_quant_config(path: str) -> QuantSpec:
    return parse_quant_config(_read_raw_config(path))


@dataclass
class BlockFp8Spec:
    """An HF / DeepSeek-native block-FP8 config (transformers' FineGrainedFP8Config)."""
    weight_block_size: tuple = (128, 128)
    activation_scheme: str = "dynamic"
    modules_to_not_convert: Optional[list] = None


def parse_block_fp8_config(raw: dict) -> BlockFp8Spec:
    """`{"quant_method": "fp8", "fmt": "e4m3", "activation_scheme": "dynamic", "weight_block_size": [128, 128]}`:
    `fmt` may be absent or e4m3, `activation_scheme` absent or dynamic, the block size must be [128, 128].
    NotImplementedError for what the block-FP8 kernels do not serve (static activations, per-tensor HF FP8, other block
    sizes, e5m2 / fnuz / e8m0, the reference's own FP8Config), ValueError for malformed entries."""
    from .fp8 import FP8_FORMAT_ALIASES

    if not isinstance(raw, dict):
        raise ValueError(f"block FP8: the quantisation config must be a dict, got {type(raw).__name__}")
    method = raw.get("quant_method", raw.get("method"))
    if str(method).lower() != "fp8":
        raise NotImplementedError(f"block FP8: quant_method `{method}` is not fp8")
    if "format" in raw or "weight_scale_semantics" in raw or "weight_scale_method" in raw:
        raise NotImplementedError("block FP8: this is the reference's FP8Config (weight = w / weight_scale_inv); load it "
                                  "with load_quantized_linears")
    fmt = raw.get("fmt")
    if fmt is not None:
        if not isinstance(fmt, str):
            raise ValueError(f"block FP8: `fmt` must be a string, got {fmt!r}")
        resolved = FP8_FORMAT_ALIASES.get(fmt.strip().lower())
        if resolved is None:
            raise ValueError(f"block FP8: unknown `fmt` `{fmt}`")
        if resolved != "float8_e4m3fn":
            raise NotImplementedError(f"block FP8: `fmt` `{fmt}` is not served (e4m3 only)")
    scheme = raw.get("activation_scheme", "dynamic")
    if not isinstance(scheme, str):
        raise ValueError(f"block FP8: `activation_scheme` must be a string, got {scheme!r}")
    if scheme.strip().lower() == "static":
        raise NotImplementedError("block FP8: static activation scales (`input_scale`) are not served (dynamic only)")
    if scheme.strip().lower() != "dynamic":
        raise ValueError(f"block FP8: unknown `activation_scheme` `{scheme}`")
    block = raw.get("weight_block_size")
    if block is None:
        raise NotImplementedError("block FP8: per-tensor FP8 checkpoints (no `weight_block_size`) are not served")
    if not isinstance(block, (list, tuple)) or len(block) != 2 or not all(isinstance(b, int) and b > 0 for b in block):
        raise ValueError(f"block FP8: `weight_block_size` must be two positive integers, got {block!r}")
    if tuple(block) != (128, 128):
        raise NotImplementedError(f"block FP8: weight_block_size {list(block)} is not served ([128, 128] only)")
    skip = raw.get("modules_to_not_convert")
    if skip is not None and not (isinstance(skip, (list, tuple)) and all(isinstance(s, str) for s in skip)):
        raise ValueError(f"block FP8: `modules_to_not_convert` must be a list of names, got {skip!r}")
    return BlockFp8Spec((128, 128), "dynamic", list(skip) if skip is not None else None)


@torch.no_grad()
def load_block_fp8_linears(path: str, device="cuda", dtype: Optional[torch.dtype] = None,
                           only: Optional[Iterable[str]] = None,
                           post_init: Optional[bool] = None) -> Dict[str, nn.Module]:
    """Load every block-FP8 linear of an HF / DeepSeek-native checkpoint into B200BlockFp8Linear modules.

    Modules are the `<prefix>.weight` + `<prefix>.weight_scale_inv` pairs; modules without `weight_scale_inv` (an
    unquantised lm_head, norms, embeddings) stay dense and are not returned.  Raises ValueError when a scale grid does
    not fit its weight.
    only      : optional iterable of module prefixes to load (default: all found)
    post_init : default True on CUDA devices, False on CPU (tensors only; host tests)
    """
    from safetensors import safe_open

    from .fp8_block import B200BlockFp8Linear

    parse_block_fp8_config(_read_raw_config(path))
    wmap = _weight_map(path)
    prefixes = list(only) if only is not None else fp8_prefixes(wmap)
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
            t = {s: tensor(f"{prefix}.{s}") for s in ("weight", "weight_scale_inv", "input_scale", "bias")}
            if t["weight"] is None or t["weight_scale_inv"] is None:
                raise KeyError(f"{prefix}: checkpoint misses weight / weight_scale_inv")
            if t["input_scale"] is not None:
                raise NotImplementedError(f"{prefix}: static activation scales (`input_scale`) are not served")
            if t["weight"].dtype != torch.float8_e4m3fn:
                raise NotImplementedError(f"{prefix}: weight dtype {t['weight'].dtype} is not served "
                                          "(float8_e4m3fn only)")
            mods[prefix] = B200BlockFp8Linear.from_checkpoint_tensors(
                t["weight"], t["weight_scale_inv"], bias=t["bias"], device=dev, dtype=dtype, post_init=do_post,
                name=prefix)
    finally:
        for h in handles.values():
            close = getattr(h, "__exit__", None)
            if close is not None:
                close(None, None, None)
        handles.clear()
    return mods


@dataclass
class Fp8W8A8Spec:
    """A per-channel / per-tensor FP8 (W8A8) config: compressed-tensors `float-quantized` or transformers' fbgemm_fp8.
    kv_cache_scheme is the checkpoint's KV-cache quantisation, returned untouched: the attention that would apply it is
    the caller's, not this package's."""
    method: str                       # "compressed-tensors" | "fbgemm_fp8"
    weight_strategy: str = "channel"  # "channel" | "tensor"
    activation: str = "dynamic"       # "dynamic" (per token) | "static" (per tensor, input_scale)
    ub: Optional[float] = None        # fbgemm_fp8: activation_scale_ub
    ignore: tuple = ()                # compressed-tensors: names / "re:" patterns; fbgemm_fp8: name fragments
    kv_cache_scheme: Optional[dict] = None

    def ignores(self, name: str) -> bool:
        if self.method == "fbgemm_fp8":  # transformers' modules_to_not_convert: a fragment of the module's name
            return any(k in name for k in self.ignore)
        return _ct_ignores(self.ignore, name)


def _ct_ignores(ignore: tuple, name: str) -> bool:
    """compressed-tensors `ignore`: module names and `re:` patterns."""
    return any(re.match(k[3:], name) if k.startswith("re:") else k == name for k in ignore)


def _ct_args(where: str, a, kinds, want: str = "float", bits: int = 8) -> tuple:
    """(strategy, dynamic) of one compressed-tensors QuantizationArgs dict that this package serves."""
    if not isinstance(a, dict):
        raise ValueError(f"compressed-tensors: `{where}` must be a dict, got {a!r}")
    nb, typ, sym, strat, dyn = (a.get(k) for k in ("num_bits", "type", "symmetric", "strategy", "dynamic"))
    if not isinstance(nb, int) or isinstance(nb, bool) or nb <= 0:
        raise ValueError(f"compressed-tensors: `{where}.num_bits` must be a positive integer, got {nb!r}")
    if typ not in ("int", "float") or not isinstance(sym, bool) or not isinstance(strat, str):
        raise ValueError(f"compressed-tensors: `{where}` needs type int | float, a boolean `symmetric` and a `strategy`")
    if not (isinstance(dyn, bool) or dyn == "local"):
        raise ValueError(f"compressed-tensors: `{where}.dynamic` must be a boolean, got {dyn!r}")
    if typ != want or nb != bits:
        raise NotImplementedError(f"compressed-tensors: {where} of {nb}-bit {typ} are not served ({bits}-bit {want} only)")
    if not sym:
        raise NotImplementedError(f"compressed-tensors: asymmetric {where} are not served")
    if strat not in ("tensor", "channel", "group", "block", "token", "tensor_group", "attn_head"):
        raise ValueError(f"compressed-tensors: unknown `{where}.strategy` `{strat}`")
    if (strat, dyn) not in kinds:
        raise NotImplementedError(f"compressed-tensors: {where} with strategy `{strat}`, dynamic={dyn} are not served "
                                  f"(served: {', '.join(f'{s} / dynamic={d}' for s, d in kinds)})")
    return strat, dyn


def _ct_w8a8(raw: dict, fmt_name: str, want: str) -> tuple:
    """(weight strategy, activation kind, ignore, kv_cache_scheme) of a compressed-tensors W8A8 config whose groups all
    target ["Linear"] with 8-bit `want` (float | int) symmetric weights (channel | tensor, static) and input activations
    (token / dynamic or tensor / static), the same kind in every group."""
    def kind(gname: str, g: dict) -> tuple:
        ws, _ = _ct_args(f"{gname}.weights", g["weights"], {("channel", False), ("tensor", False)}, want)
        _, dyn = _ct_args(f"{gname}.input_activations", g["input_activations"], {("token", True), ("tensor", False)},
                           want)
        return ws, "dynamic" if dyn else "static"

    (ws, act), ignore, kv = _ct_groups(raw, fmt_name, "W8A8", kind)
    return ws, act, ignore, kv


def _ct_groups(raw: dict, fmt_name: str, scheme: str, kind) -> tuple:
    """(kind, ignore, kv_cache_scheme) of a compressed-tensors config of format `fmt_name` whose groups all target
    ["Linear"] with weights and input activations (`scheme`) and no output activations; kind(name, group) checks a
    group's arguments and returns what it is, which must be the same in every group."""
    fmt = raw.get("format")
    if fmt != fmt_name:
        raise NotImplementedError(f"compressed-tensors: format `{fmt}` is not served ({fmt_name} only)")
    groups = raw.get("config_groups")
    if not isinstance(groups, dict) or not groups:
        raise ValueError("compressed-tensors: `config_groups` must be a non-empty dict")
    kinds = set()
    for gname, g in groups.items():
        if not isinstance(g, dict):
            raise ValueError(f"compressed-tensors: config group `{gname}` must be a dict")
        targets = g.get("targets")
        if not (isinstance(targets, list) and all(isinstance(t, str) for t in targets)):
            raise ValueError(f"compressed-tensors: `{gname}.targets` must be a list of names")
        if targets != ["Linear"]:
            raise NotImplementedError(f"compressed-tensors: `{gname}` targets {targets} (only [\"Linear\"] is served)")
        if g.get("format") not in (None, fmt_name):
            raise NotImplementedError(f"compressed-tensors: `{gname}` has format `{g.get('format')}`")
        if g.get("output_activations") is not None:
            raise NotImplementedError(f"compressed-tensors: `{gname}` quantises output activations")
        if g.get("weights") is None or g.get("input_activations") is None:
            raise NotImplementedError(f"compressed-tensors: `{gname}` is not {scheme} (weights and input activations)")
        kinds.add(kind(gname, g))
    if len(kinds) != 1:
        raise NotImplementedError(f"compressed-tensors: mixed config groups {sorted(kinds)} are not served")
    ignore = raw.get("ignore") or []
    if not (isinstance(ignore, (list, tuple)) and all(isinstance(s, str) for s in ignore)):
        raise ValueError(f"compressed-tensors: `ignore` must be a list of names, got {ignore!r}")
    for k in ignore:
        if k.startswith("re:"):
            try:
                re.compile(k[3:])
            except re.error as e:
                raise ValueError(f"compressed-tensors: bad `ignore` pattern `{k}`: {e}") from None
    kv = raw.get("kv_cache_scheme")
    if kv is not None and not isinstance(kv, dict):
        raise ValueError(f"compressed-tensors: `kv_cache_scheme` must be a dict, got {kv!r}")
    (k,) = kinds
    return k, tuple(ignore), kv


def parse_fp8_w8a8_config(raw: dict) -> Fp8W8A8Spec:
    """Per-channel / per-tensor FP8 (W8A8) configs:
      * `quant_method: compressed-tensors`, `format: float-quantized`; every config group targets ["Linear"] with weights
        {num_bits: 8, type: float, symmetric: true, dynamic: false, strategy: channel | tensor} and input activations
        {num_bits: 8, type: float, symmetric: true} either {strategy: token, dynamic: true} or {strategy: tensor,
        dynamic: false}, the same in every group.  `ignore` holds module names and `re:` patterns;
      * `quant_method: fbgemm_fp8` with `activation_scale_ub` (default 1200.0) and `modules_to_not_convert`.
    NotImplementedError for what the kernels do not serve (group / block strategies, int types, asymmetric or dynamic
    weights, mixed groups, other targets or formats), ValueError for malformed entries."""
    if not isinstance(raw, dict):
        raise ValueError(f"FP8 W8A8: the quantisation config must be a dict, got {type(raw).__name__}")
    method = raw.get("quant_method")
    if method == "fbgemm_fp8":
        ub = raw.get("activation_scale_ub", 1200.0)
        if isinstance(ub, bool) or not isinstance(ub, (int, float)) or not (0.0 < float(ub) < float("inf")):
            raise ValueError(f"fbgemm_fp8: `activation_scale_ub` must be a positive number, got {ub!r}")
        skip = raw.get("modules_to_not_convert") or []
        if not (isinstance(skip, (list, tuple)) and all(isinstance(s, str) for s in skip)):
            raise ValueError(f"fbgemm_fp8: `modules_to_not_convert` must be a list of names, got {skip!r}")
        return Fp8W8A8Spec("fbgemm_fp8", "channel", "dynamic", float(ub), tuple(skip))
    if method != "compressed-tensors":
        raise NotImplementedError(f"FP8 W8A8: quant_method `{method}` is not compressed-tensors or fbgemm_fp8")
    ws, act, ignore, kv = _ct_w8a8(raw, "float-quantized", "float")
    return Fp8W8A8Spec("compressed-tensors", ws, act, None, ignore, kv)


@torch.no_grad()
def load_fp8_w8a8_linears(path: str, device="cuda", dtype: Optional[torch.dtype] = None,
                          only: Optional[Iterable[str]] = None,
                          post_init: Optional[bool] = None) -> Dict[str, nn.Module]:
    """Load every FP8 W8A8 linear of a compressed-tensors FP8 / FP8_DYNAMIC or fbgemm_fp8 checkpoint into
    B200ChannelFp8Linear modules.

    Modules are the `<prefix>.weight` + `<prefix>.weight_scale` pairs that the config does not ignore; the rest (an
    unquantised lm_head, norms, embeddings) stay dense and are not returned.  A static layer must carry its
    `input_scale` and a dynamic one must not (NotImplementedError); shapes are checked (ValueError).
    only      : optional iterable of module prefixes to load (default: all found)
    post_init : default True on CUDA devices, False on CPU (tensors only; host tests)
    """
    from .fp8_channel import B200ChannelFp8Linear

    spec = parse_fp8_w8a8_config(_read_raw_config(path))
    return _load_channel_w8a8(path, spec, B200ChannelFp8Linear, device, dtype, only, post_init)


def _load_channel_w8a8(path: str, spec, cls, device, dtype, only, post_init) -> Dict[str, nn.Module]:
    """The `<prefix>.weight` + `<prefix>.weight_scale` modules of a per-channel W8A8 checkpoint as `cls` modules (their
    weights of cls.CODE_DTYPE).  A `weight_zero_point` / `input_zero_point` tensor must be all zeros: the kernels are
    symmetric."""
    code = str(cls.CODE_DTYPE).replace("torch.", "")
    wmap = _weight_map(path)
    if only is not None:
        prefixes = list(only)
    else:
        sfx = ".weight_scale"
        prefixes = sorted(n[: -len(sfx)] for n in wmap if n.endswith(sfx) and n[: -len(sfx)] + ".weight" in wmap)
        prefixes = [p for p in prefixes if not spec.ignores(p)]
    dev = torch.device(device)
    do_post = (dev.type == "cuda") if post_init is None else post_init
    mods: Dict[str, nn.Module] = {}
    with _TensorReader(wmap) as tensor:
        for prefix in prefixes:
            t = {s: tensor(f"{prefix}.{s}") for s in ("weight", "weight_scale", "input_scale", "bias")}
            if t["weight"] is None or t["weight_scale"] is None:
                raise KeyError(f"{prefix}: checkpoint misses weight / weight_scale")
            if t["weight"].dtype != cls.CODE_DTYPE:
                raise NotImplementedError(f"{prefix}: weight dtype {t['weight'].dtype} is not served "
                                          f"({code} only)")
            for zp in ("weight_zero_point", "input_zero_point"):
                z = tensor(f"{prefix}.{zp}")
                if z is not None and bool((z.to(torch.float32) != 0).any()):
                    raise NotImplementedError(f"{prefix}: a non-zero `{zp}` (asymmetric quantisation) is not served")
            if spec.activation == "static" and t["input_scale"] is None:
                raise NotImplementedError(f"{prefix}: static activations need `input_scale`, the checkpoint has none")
            if spec.activation == "dynamic" and t["input_scale"] is not None:
                raise NotImplementedError(f"{prefix}: `input_scale` on a layer with dynamic activations")
            ws = t["weight_scale"]
            if spec.weight_strategy == "tensor" and ws.numel() != 1:
                raise ValueError(f"{prefix}: per-tensor weight_scale has shape {tuple(ws.shape)}")
            mods[prefix] = cls.from_checkpoint_tensors(
                t["weight"], ws, input_scale=t["input_scale"], bias=t["bias"], activation=spec.activation,
                ub=spec.ub, device=dev, dtype=dtype, post_init=do_post, name=prefix)
    return mods


class _TensorReader:
    """`with _TensorReader(weight_map) as tensor:` tensor(name) reads a checkpoint tensor (None when absent), opening
    each safetensors file once; the files are closed on exit."""

    def __init__(self, wmap: Dict[str, str]):
        self.wmap, self.handles = wmap, {}

    def __enter__(self):
        return self.tensor

    def tensor(self, name):
        from safetensors import safe_open

        fn = self.wmap.get(name)
        if fn is None:
            return None
        if fn not in self.handles:
            self.handles[fn] = safe_open(fn, framework="pt").__enter__()
        return self.handles[fn].get_tensor(name)

    def __exit__(self, *exc):
        for h in self.handles.values():
            close = getattr(h, "__exit__", None)
            if close is not None:
                close(None, None, None)
        self.handles.clear()
        return False


@dataclass
class Int8W8A8Spec:
    """A per-channel / per-tensor INT8 (W8A8) config: compressed-tensors `int-quantized`.  kv_cache_scheme is returned
    untouched, as for Fp8W8A8Spec."""
    weight_strategy: str = "channel"  # "channel" | "tensor"
    activation: str = "dynamic"       # "dynamic" (per token) | "static" (per tensor, input_scale)
    ignore: tuple = ()                # names / "re:" patterns
    kv_cache_scheme: Optional[dict] = None
    ub = None                         # int8 activations have no amax bound

    def ignores(self, name: str) -> bool:
        return _ct_ignores(self.ignore, name)


def parse_int8_w8a8_config(raw: dict) -> Int8W8A8Spec:
    """Per-channel / per-tensor INT8 (W8A8) configs: `quant_method: compressed-tensors`, `format: int-quantized`; every
    config group targets ["Linear"] with weights {num_bits: 8, type: int, symmetric: true, dynamic: false, strategy:
    channel | tensor} and input activations {num_bits: 8, type: int, symmetric: true} either {strategy: token, dynamic:
    true} or {strategy: tensor, dynamic: false}, the same in every group.  `ignore` holds module names and `re:`
    patterns.  NotImplementedError for what the kernels do not serve (asymmetric activations, group / block strategies,
    float or 4-bit types, pack-quantized, mixed groups, output activations, other targets), ValueError for malformed
    entries."""
    if not isinstance(raw, dict):
        raise ValueError(f"INT8 W8A8: the quantisation config must be a dict, got {type(raw).__name__}")
    method = raw.get("quant_method")
    if method != "compressed-tensors":
        raise NotImplementedError(f"INT8 W8A8: quant_method `{method}` is not compressed-tensors")
    ws, act, ignore, kv = _ct_w8a8(raw, "int-quantized", "int")
    return Int8W8A8Spec(ws, act, ignore, kv)


@torch.no_grad()
def load_int8_w8a8_linears(path: str, device="cuda", dtype: Optional[torch.dtype] = None,
                           only: Optional[Iterable[str]] = None,
                           post_init: Optional[bool] = None) -> Dict[str, nn.Module]:
    """Load every INT8 W8A8 linear of a compressed-tensors `int-quantized` checkpoint into B200ChannelInt8Linear
    modules, as load_fp8_w8a8_linears does for FP8: ignored modules stay dense and are not returned, a static layer must
    carry its `input_scale` and a dynamic one must not, and zero-point tensors must be all zeros (NotImplementedError).
    only      : optional iterable of module prefixes to load (default: all found)
    post_init : default True on CUDA devices, False on CPU (tensors only; host tests)
    """
    from .int8_channel import B200ChannelInt8Linear

    spec = parse_int8_w8a8_config(_read_raw_config(path))
    return _load_channel_w8a8(path, spec, B200ChannelInt8Linear, device, dtype, only, post_init)


@dataclass
class W4Fp8Spec:
    """A compressed-tensors `W4AFP8` config (`pack-quantized`): symmetric 4-bit int weights with group-128 scales and
    dynamic per-token e4m3 activations.  kv_cache_scheme is returned untouched, as for Fp8W8A8Spec."""
    ignore: tuple = ()                # names / "re:" patterns
    kv_cache_scheme: Optional[dict] = None

    def ignores(self, name: str) -> bool:
        return _ct_ignores(self.ignore, name)


def parse_w4afp8_config(raw: dict) -> W4Fp8Spec:
    """W4AFP8 configs: `quant_method: compressed-tensors`, `format: pack-quantized`; every config group targets
    ["Linear"] with weights {num_bits: 4, type: int, symmetric: true, dynamic: false, strategy: group, group_size: 128,
    actorder: null | "weight"} and input activations {num_bits: 8, type: float, symmetric: true, strategy: token,
    dynamic: true}.  `ignore` holds module names and `re:` patterns.  NotImplementedError for what the kernels do not
    serve (other group sizes, channel / tensor strategies, other bit widths, asymmetric weights, `actorder: group`,
    static, per-tensor or int activations, mixed groups, output activations, other targets), ValueError for malformed
    entries."""
    if not isinstance(raw, dict):
        raise ValueError(f"W4AFP8: the quantisation config must be a dict, got {type(raw).__name__}")
    method = raw.get("quant_method")
    if method != "compressed-tensors":
        raise NotImplementedError(f"W4AFP8: quant_method `{method}` is not compressed-tensors")

    def kind(gname: str, g: dict) -> tuple:
        w = g["weights"]
        _ct_args(f"{gname}.weights", w, {("group", False)}, "int", 4)
        gs = w.get("group_size")
        if not isinstance(gs, int) or isinstance(gs, bool):
            raise ValueError(f"compressed-tensors: `{gname}.weights.group_size` must be an integer, got {gs!r}")
        if gs != 128:
            raise NotImplementedError(f"compressed-tensors: {gname}.weights with group_size {gs} are not served "
                                      "(128 only)")
        ao = w.get("actorder")
        if ao is not None and not isinstance(ao, str):
            raise ValueError(f"compressed-tensors: `{gname}.weights.actorder` must be a string or null, got {ao!r}")
        if ao not in (None, "weight"):
            raise NotImplementedError(f"compressed-tensors: {gname}.weights with actorder `{ao}` are not served "
                                      "(null or `weight`: the groups stay contiguous)")
        _ct_args(f"{gname}.input_activations", g["input_activations"], {("token", True)}, "float", 8)
        return ("group", "dynamic")

    _, ignore, kv = _ct_groups(raw, "pack-quantized", "W4AFP8", kind)
    return W4Fp8Spec(ignore, kv)


@torch.no_grad()
def load_w4afp8_linears(path: str, device="cuda", dtype: Optional[torch.dtype] = None,
                        only: Optional[Iterable[str]] = None,
                        post_init: Optional[bool] = None) -> Dict[str, nn.Module]:
    """Load every linear of a compressed-tensors W4AFP8 checkpoint into B200W4Fp8Linear modules.

    Modules are the `<prefix>.weight_packed` + `<prefix>.weight_scale` pairs that the config does not ignore; the rest
    stay dense and are not returned.  A `weight_zero_point` must be all zeros and a `weight_g_idx` must be
    arange(K) // 128 (NotImplementedError); shapes outside the kernels' envelope raise NotImplementedError, malformed
    tensors ValueError.
    only      : optional iterable of module prefixes to load (default: all found)
    post_init : default True on CUDA devices, False on CPU (tensors only; host tests)
    """
    from .w4afp8 import GROUP, B200W4Fp8Linear

    spec = parse_w4afp8_config(_read_raw_config(path))
    wmap = _weight_map(path)
    if only is not None:
        prefixes = list(only)
    else:
        sfx = ".weight_packed"
        prefixes = sorted(n[: -len(sfx)] for n in wmap if n.endswith(sfx) and n[: -len(sfx)] + ".weight_scale" in wmap)
        prefixes = [p for p in prefixes if not spec.ignores(p)]
    dev = torch.device(device)
    do_post = (dev.type == "cuda") if post_init is None else post_init
    mods: Dict[str, nn.Module] = {}
    with _TensorReader(wmap) as tensor:
        for prefix in prefixes:
            t = {s: tensor(f"{prefix}.{s}") for s in ("weight_packed", "weight_scale", "weight_shape", "bias",
                                                      "weight_zero_point", "weight_g_idx")}
            if t["weight_packed"] is None or t["weight_scale"] is None:
                raise KeyError(f"{prefix}: checkpoint misses weight_packed / weight_scale")
            z = t["weight_zero_point"]
            if z is not None and bool((z.to(torch.float32) != 0).any()):
                raise NotImplementedError(f"{prefix}: a non-zero `weight_zero_point` (asymmetric weights) is not served")
            g = t["weight_g_idx"]
            if g is not None:
                K = int(t["weight_packed"].shape[-1]) * 8
                if g.dim() != 1 or g.numel() != K or not torch.equal(g.to(torch.int64), torch.arange(K) // GROUP):
                    raise NotImplementedError(f"{prefix}: a `weight_g_idx` other than arange(K) // 128 (activation "
                                              "order by group) is not served")
            mods[prefix] = B200W4Fp8Linear.from_checkpoint_tensors(
                t["weight_packed"], t["weight_scale"], weight_shape=t["weight_shape"], bias=t["bias"], device=dev,
                dtype=dtype, post_init=do_post, name=prefix)
    return mods


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


def qqq_prefixes(names: Iterable[str]) -> list:
    """Module prefixes of a QQQ checkpoint (`<prefix>.B` together with `<prefix>.s_channel`)."""
    names = set(names)
    return sorted(n[: -len(".s_channel")] for n in names if n.endswith(".s_channel") and n[: -len(".s_channel")] + ".B" in names)


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


# Orders of the non-power-of-two Hadamard factor, in the precedence the reference's get_hadK tests them
# (quantization/rotation/hadamard_utils.py:20-70): the first order dividing n is used, even where a later one would too.
HADAMARD_ORDERS = (172, 156, 140, 108, 60, 52, 36, 28, 40, 20, 12)
ROTATED_SUFFIX = "mlp.down_proj"  # the modules that transform their input online (models/loader.py:273-310)


def hadamard_order(n: int) -> int:
    """Order K of the rotation's +-1 factor for a transform of length n = K * 2^m (1: n is a power of two).
    Raises ValueError for a length the reference cannot rotate either."""
    def pow2(v):
        return v > 0 and v & (v - 1) == 0

    for k in HADAMARD_ORDERS:
        if n % k == 0:
            if not pow2(n // k):
                raise ValueError(f"no Hadamard transform of length {n}: {n} / {k} is not a power of two")
            return k
    if not pow2(n):
        raise ValueError(f"no Hadamard transform of length {n}: not a power of two times one of {HADAMARD_ORDERS}")
    return 1


def _hadamard_table(hadamard, order: int, n: int) -> torch.Tensor:
    """The caller's +-1 matrix of `order` for a transform of length n: `hadamard` maps order -> tensor, or is a callable
    like the reference's get_hadK(n) -> (tensor, K)."""
    t = None
    if callable(hadamard):
        t, k = hadamard(n)
        if k != order:
            t = None
    elif hadamard is not None:
        t = hadamard.get(order)
    if t is None:
        raise NotImplementedError(f"rotated checkpoint needs the Hadamard matrix of order {order}: pass it in "
                                  "load_quantized_linears(..., hadamard={order: tensor}) or hadamard=get_hadK")
    return torch.as_tensor(t)


@torch.no_grad()
def load_quantized_linears(path: str, device="cuda", dtype: Optional[torch.dtype] = None,
                           only: Optional[Iterable[str]] = None, post_init: Optional[bool] = None,
                           hadamard=None) -> Dict[str, nn.Module]:
    """Load every quantised linear of a checkpoint directory into B200 QuantLinear modules.

    only      : optional iterable of module prefixes to load (default: all `<prefix>.qweight` found)
    post_init : default True on CUDA devices (prepack for the kernels), False on CPU (tensors only; host tests)
    hadamard  : rotated checkpoints (`rotation` in the quantisation config) only: the +-1 matrices of the non-power-of-two
                Hadamard orders, as a mapping {order: tensor [order, order]} or a callable such as the reference's
                `get_hadK`.  Every `*mlp.down_proj` module gets the reference's online transform of its input; a size whose
                order has no matrix raises NotImplementedError (power-of-two sizes need none).
    """
    from safetensors import safe_open

    from .awq import B200AwqQuantLinear
    from .fp8 import B200Fp8QuantLinear
    from .qlinear import B200QuantLinear
    from .qqq import B200QqqQuantLinear

    spec = read_quant_config(path)
    wmap = _weight_map(path)
    if only is not None:
        prefixes = list(only)
    else:
        prefixes = {"qqq": qqq_prefixes, "fp8": fp8_prefixes}.get(spec.method, quantized_prefixes)(wmap)
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
            if ms.method == "fp8":
                t = {s: tensor(f"{prefix}.{s}") for s in ("weight", "weight_scale_inv", "weight_scale", "bias")}
                if t["weight"] is None or t["weight_scale_inv"] is None:
                    if t["weight_scale"] is not None:
                        raise NotImplementedError(f"{prefix}: ModelOpt-style FP8 tensors (`weight_scale` without "
                                                  "`weight_scale_inv`) are not supported")
                    raise KeyError(f"{prefix}: checkpoint misses weight / weight_scale_inv")
                if t["weight"].dtype != torch.float8_e4m3fn:
                    raise NotImplementedError(f"{prefix}: weight dtype {t['weight'].dtype} is not served "
                                              "(float8_e4m3fn only)")
                m = B200Fp8QuantLinear.from_checkpoint_tensors(
                    t["weight"], t["weight_scale_inv"], bias=t["bias"], weight_scale_method=ms.weight_scale_method,
                    weight_block_size=ms.weight_block_size, format=ms.fp8_format, device=dev, dtype=dtype,
                    post_init=do_post, name=prefix)
                mods[prefix] = m
                continue
            if ms.method == "qqq":
                _check_qqq(ms)  # a `dynamic` override may have changed bits / group size
                t = {s: tensor(f"{prefix}.{s}") for s in ("B", "s_channel", "s_group", "bias")}
                if t["B"] is None or t["s_channel"] is None:
                    raise KeyError(f"{prefix}: checkpoint misses B / s_channel")
                K, N = t["B"].shape[0] * 16, t["B"].shape[1] // 2
                m = B200QqqQuantLinear(bits=4, group_size=ms.group_size, desc_act=ms.desc_act, sym=True, in_features=K,
                                       out_features=N, bias=t["bias"] is not None, register_buffers=False, dtype=dtype,
                                       name=prefix)
                sg = t["s_group"] if t["s_group"] is not None else torch.empty(0, dtype=torch.float16)
                m.B, m.s_channel, m.s_group = t["B"].to(dev), t["s_channel"].to(dev, torch.float32), sg.to(dev)
                m.bias = None if t["bias"] is None else t["bias"].to(dev, torch.float16)
                if do_post:
                    m.post_init()
                mods[prefix] = m
                continue
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
                if spec.rotation and prefix.endswith(ROTATED_SUFFIX):
                    order = hadamard_order(K)
                    m.online_full_had = True
                    m.K = order
                    if order > 1:
                        m.set_had_K(_hadamard_table(hadamard, order, K))  # validated and copied by post_init()
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
