"""Per-channel / per-tensor FP8 (W8A8) host side: config parsing and refusals of both spellings (compressed-tensors and
fbgemm_fp8), the loader on a synthetic checkpoint, the module's scales and dequantiser, compressed-tensors' fixture, the
ABI's argument checks and the compiler's report on the new kernels.  No GPU needed."""
import json
import os
import re

import numpy as np
import pytest
import torch

import fp8_w8a8_mirror as fm
from gptqmodel_b200 import B200ChannelFp8Linear, lib
from gptqmodel_b200.fp8_channel import channel_scales
from gptqmodel_b200.loader import load_fp8_w8a8_linears, parse_fp8_w8a8_config
from oracle import fp8_block_oracle as fo

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = np.load(os.path.join(HERE, "golden", "fp8_w8a8_cases.npz"))


def ct_config(preset, **kw):
    """A compressed-tensors config as its own QuantizationConfig writes it."""
    from compressed_tensors.quantization import QuantizationConfig, preset_name_to_scheme

    cfg = QuantizationConfig(config_groups={"group_0": preset_name_to_scheme(preset, ["Linear"])},
                             format="float-quantized", **kw)
    return json.loads(json.dumps(cfg.model_dump(mode="json")))


def _set(raw, where, **kw):
    """A deep copy of raw with config_groups.group_0.<where> updated by kw (where = "" for the group itself)."""
    raw = json.loads(json.dumps(raw))
    g = raw["config_groups"]["group_0"]
    (g[where] if where else g).update(kw)
    return raw


DYN, STATIC = ct_config("FP8_DYNAMIC", ignore=["lm_head"]), ct_config("FP8", ignore=["lm_head"])


# ---- config parsing ---------------------------------------------------------------------------------------------------
def test_compressed_tensors_presets_accepted():
    s = parse_fp8_w8a8_config(DYN)
    assert (s.method, s.weight_strategy, s.activation, s.ub, s.ignore) == (
        "compressed-tensors", "channel", "dynamic", None, ("lm_head",))
    s = parse_fp8_w8a8_config(STATIC)
    assert (s.weight_strategy, s.activation) == ("tensor", "static")
    kv = {"num_bits": 8, "type": "float", "strategy": "tensor", "dynamic": False, "symmetric": True}
    assert parse_fp8_w8a8_config({**DYN, "kv_cache_scheme": kv}).kv_cache_scheme == kv  # left to the caller
    two = json.loads(json.dumps(DYN))
    two["config_groups"]["group_1"] = two["config_groups"]["group_0"]
    assert parse_fp8_w8a8_config(two).activation == "dynamic"
    # channel weights with static activations, and tensor weights with dynamic ones, are served too
    assert parse_fp8_w8a8_config(_set(DYN, "input_activations", strategy="tensor", dynamic=False)).activation == "static"
    assert parse_fp8_w8a8_config(_set(STATIC, "weights", strategy="channel")).weight_strategy == "channel"


def test_fbgemm_accepted():
    s = parse_fp8_w8a8_config({"quant_method": "fbgemm_fp8"})
    assert (s.method, s.weight_strategy, s.activation, s.ub, s.ignore) == ("fbgemm_fp8", "channel", "dynamic", 1200.0, ())
    s = parse_fp8_w8a8_config({"quant_method": "fbgemm_fp8", "activation_scale_ub": 800,
                               "modules_to_not_convert": ["lm_head", "mlp.gate"]})
    assert s.ub == 800.0 and s.ignores("lm_head") and s.ignores("model.layers.3.mlp.gate")
    assert s.ignores("model.layers.3.mlp.gate_proj")  # transformers matches name fragments
    assert not s.ignores("model.layers.3.self_attn.q_proj")


def test_ignore_names_and_patterns():
    s = parse_fp8_w8a8_config({**DYN, "ignore": ["lm_head", "re:.*mlp\\.gate$", "re:model\\.layers\\.0\\..*"]})
    assert s.ignores("lm_head") and not s.ignores("model.lm_head")
    assert s.ignores("model.layers.5.mlp.gate") and not s.ignores("model.layers.5.mlp.gate_proj")
    assert s.ignores("model.layers.0.self_attn.q_proj") and not s.ignores("model.layers.10.self_attn.q_proj")


@pytest.mark.parametrize("raw", [
    _set(DYN, "weights", strategy="group", group_size=128),
    _set(DYN, "weights", strategy="block", block_structure=[128, 128]),
    _set(DYN, "weights", type="int"),
    _set(DYN, "weights", num_bits=4),
    _set(DYN, "weights", symmetric=False),
    _set(DYN, "weights", dynamic=True),
    _set(DYN, "input_activations", strategy="group", group_size=128),
    _set(DYN, "input_activations", type="int"),
    _set(DYN, "input_activations", symmetric=False),
    _set(DYN, "input_activations", dynamic=False),  # static per-token
    _set(STATIC, "input_activations", dynamic=True),  # dynamic per-tensor
    _set(DYN, "", input_activations=None),  # weight-only (W8A16)
    _set(DYN, "", output_activations=dict(DYN["config_groups"]["group_0"]["weights"])),
    _set(DYN, "", targets=["Linear", "Embedding"]),
    _set(DYN, "", targets=["re:.*q_proj"]),
    _set(DYN, "", format="pack-quantized"),
    {**DYN, "format": "pack-quantized"},
    {**DYN, "format": "naive-quantized"},
    {"quant_method": "fp8", "activation_scheme": "dynamic"},
    {"quant_method": "gptq", "bits": 4},
])
def test_refusals(raw):
    with pytest.raises(NotImplementedError):
        parse_fp8_w8a8_config(raw)


def test_mixed_groups_refused():
    w4a16 = ct_config("W4A16")["config_groups"]["group_0"]
    mixed = json.loads(json.dumps(DYN))
    mixed["config_groups"]["group_1"] = w4a16
    with pytest.raises(NotImplementedError):
        parse_fp8_w8a8_config(mixed)
    mixed["config_groups"]["group_1"] = STATIC["config_groups"]["group_0"]  # FP8_DYNAMIC with FP8
    with pytest.raises(NotImplementedError, match="mixed"):
        parse_fp8_w8a8_config(mixed)


@pytest.mark.parametrize("raw", [
    [],
    {**DYN, "config_groups": {}},
    {**DYN, "config_groups": []},
    {**DYN, "config_groups": {"group_0": 3}},
    _set(DYN, "weights", num_bits="8"),
    _set(DYN, "weights", type="fp"),
    _set(DYN, "weights", strategy="rows"),
    _set(DYN, "weights", symmetric="yes"),
    _set(DYN, "weights", dynamic=None),
    _set(DYN, "", weights=7),
    _set(DYN, "", targets="Linear"),
    {**DYN, "ignore": "lm_head"},
    {**DYN, "ignore": ["re:("]},
    {**DYN, "kv_cache_scheme": "fp8"},
    {"quant_method": "fbgemm_fp8", "activation_scale_ub": -1.0},
    {"quant_method": "fbgemm_fp8", "activation_scale_ub": "1200"},
    {"quant_method": "fbgemm_fp8", "modules_to_not_convert": "lm_head"},
])
def test_malformed(raw):
    with pytest.raises(ValueError):
        parse_fp8_w8a8_config(raw)


# ---- loader -------------------------------------------------------------------------------------------------------------
def _write_ckpt(path, cfg, tensors):
    from safetensors.torch import save_file

    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump({"model_type": "llama", "quantization_config": cfg}, f)
    save_file(tensors, os.path.join(path, "model.safetensors"))


def _fp8(N, K, seed):
    return (torch.randn(N, K, generator=torch.Generator().manual_seed(seed)) * 30).to(torch.float8_e4m3fn)


def _scale(shape, dtype, seed):
    return (torch.rand(shape, generator=torch.Generator().manual_seed(seed)) * 1e-2 + 1e-4).to(dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", [(192, 1), (192,), (1,), ()])
def test_loader_scale_shapes_and_exact_widening(tmp_path, shape, dtype):
    ws = _scale(shape, dtype, 1)
    t = {"m.q.weight": _fp8(192, 256, 0), "m.q.weight_scale": ws, "m.q.bias": torch.zeros(192, dtype=torch.bfloat16),
         "lm_head.weight": torch.randn(64, 256, dtype=torch.bfloat16), "m.norm.weight": torch.ones(256)}
    _write_ckpt(str(tmp_path), DYN, t)
    mods = load_fp8_w8a8_linears(str(tmp_path), device="cpu", post_init=False)
    assert sorted(mods) == ["m.q"]
    m = mods["m.q"]
    assert (m.in_features, m.out_features, m.activation, m.ub, m.input_scale) == (256, 192, "dynamic", None, None)
    assert torch.equal(m.weight.view(torch.uint8), t["m.q.weight"].view(torch.uint8))
    assert m.weight_scale.dtype == dtype and m.bias is not None
    s = channel_scales(m.weight_scale, 192)
    assert s.dtype == torch.float32 and s.shape == (192,)
    assert torch.equal(s.to(dtype), ws.reshape(-1).expand(192))  # widening is exact: it narrows back bit for bit
    assert torch.equal(s.double(), ws.double().reshape(-1).expand(192))


def test_loader_static_and_fbgemm(tmp_path):
    t = {"m.q.weight": _fp8(128, 256, 0), "m.q.weight_scale": _scale((1,), torch.bfloat16, 2),
         "m.q.input_scale": _scale((1,), torch.bfloat16, 3),
         "m.k.weight": _fp8(64, 256, 1), "m.k.weight_scale": _scale((), torch.float32, 4),
         "m.k.input_scale": _scale((), torch.float16, 5)}
    _write_ckpt(str(tmp_path / "ct"), STATIC, t)
    mods = load_fp8_w8a8_linears(str(tmp_path / "ct"), device="cpu", post_init=False)
    assert sorted(mods) == ["m.k", "m.q"] and all(m.activation == "static" for m in mods.values())
    assert torch.equal(mods["m.k"].input_scale, t["m.k.input_scale"])
    assert set(load_fp8_w8a8_linears(str(tmp_path / "ct"), device="cpu", only=["m.q"], post_init=False)) == {"m.q"}
    f = {"model.layers.0.mlp.down_proj.weight": _fp8(128, 256, 0),
         "model.layers.0.mlp.down_proj.weight_scale": _scale((128, 1), torch.float32, 6),
         "model.layers.0.mlp.gate.weight": _fp8(64, 256, 1),
         "model.layers.0.mlp.gate.weight_scale": _scale((64, 1), torch.float32, 7)}
    _write_ckpt(str(tmp_path / "fb"), {"quant_method": "fbgemm_fp8", "activation_scale_ub": 1000.0,
                                       "modules_to_not_convert": ["mlp.gate"]}, f)
    mods = load_fp8_w8a8_linears(str(tmp_path / "fb"), device="cpu", post_init=False)
    assert sorted(mods) == ["model.layers.0.mlp.down_proj"]  # mlp.gate is not converted
    assert mods["model.layers.0.mlp.down_proj"].ub == 1000.0


def test_loader_ignore_patterns(tmp_path):
    t = {f"model.layers.{i}.{n}.{s}": (_fp8(64, 128, i) if s == "weight" else _scale((64, 1), torch.bfloat16, i))
         for i in range(2) for n in ("self_attn.q_proj", "mlp.gate") for s in ("weight", "weight_scale")}
    _write_ckpt(str(tmp_path), {**DYN, "ignore": ["re:.*mlp\\.gate$", "model.layers.1.self_attn.q_proj"]}, t)
    assert sorted(load_fp8_w8a8_linears(str(tmp_path), device="cpu", post_init=False)) == [
        "model.layers.0.self_attn.q_proj"]


def test_loader_refuses_missing_or_extra_input_scale(tmp_path):
    t = {"m.q.weight": _fp8(128, 256, 0), "m.q.weight_scale": _scale((1,), torch.float32, 1)}
    _write_ckpt(str(tmp_path / "a"), STATIC, t)
    with pytest.raises(NotImplementedError, match="input_scale"):
        load_fp8_w8a8_linears(str(tmp_path / "a"), device="cpu", post_init=False)
    t = {"m.q.weight": _fp8(128, 256, 0), "m.q.weight_scale": _scale((128, 1), torch.float32, 1),
         "m.q.input_scale": torch.ones(1)}
    _write_ckpt(str(tmp_path / "b"), DYN, t)
    with pytest.raises(NotImplementedError, match="input_scale"):
        load_fp8_w8a8_linears(str(tmp_path / "b"), device="cpu", post_init=False)


@pytest.mark.parametrize("ws,what", [(torch.rand(128, 2), "weight_scale"), (torch.rand(64, 1), "weight_scale"),
                                     (-torch.rand(128, 1), "weight_scale"), (torch.full((1,), float("inf")), "weight_scale"),
                                     (torch.zeros(()), "weight_scale")])
def test_loader_rejects_bad_scales(tmp_path, ws, what):
    _write_ckpt(str(tmp_path), DYN, {"m.q.weight": _fp8(128, 256, 0), "m.q.weight_scale": ws})
    with pytest.raises(ValueError, match=what):
        load_fp8_w8a8_linears(str(tmp_path), device="cpu", post_init=False)


def test_module_envelope_and_arguments():
    for K, N in ((192, 128), (256, 96), (0, 128), (65536 + 128, 128)):
        with pytest.raises(NotImplementedError):
            B200ChannelFp8Linear(in_features=K, out_features=N)
    with pytest.raises(ValueError):
        B200ChannelFp8Linear(256, 128, activation="sometimes")
    with pytest.raises(ValueError):
        B200ChannelFp8Linear(256, 128, activation="static", ub=100.0)
    with pytest.raises(ValueError):
        B200ChannelFp8Linear(256, 128, ub=0.0)
    with pytest.raises(ValueError):
        B200ChannelFp8Linear.from_checkpoint_tensors(_fp8(128, 256, 0), torch.ones(128), input_scale=torch.ones(2),
                                                     device="cpu", post_init=False)


# ---- dequantisation and compressed-tensors' fixture ----------------------------------------------------------------------
@pytest.mark.parametrize("sdt", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", [(128, 1), (1,)])
def test_dequantize_weight_is_w_times_s(shape, sdt):
    w, s = _fp8(128, 256, 3), _scale(shape, sdt, 4)
    m = B200ChannelFp8Linear.from_checkpoint_tensors(w, s, device="cpu", post_init=False)
    for dt in (torch.float16, torch.bfloat16):
        want = (w.to(sdt) * s.reshape(-1, 1) if s.numel() > 1 else w.to(sdt) * s.reshape(())).to(dt).t()
        assert torch.equal(m.dequantize_weight(dtype=dt), want)


NAMES = sorted({k.split(".")[0] for k in CASES.files})
_DT = {"bf": torch.bfloat16, "16": torch.float16}


def _t16(a, dtype):
    return torch.from_numpy(fo.unpack16(a)).to(dtype)


@pytest.mark.parametrize("name", NAMES)
def test_dequantize_matches_compressed_tensors(name):
    dt = _DT[name.rsplit("_", 1)[1]]
    c = lambda k: CASES[f"{name}.{k}"]  # noqa: E731
    m = B200ChannelFp8Linear.from_checkpoint_tensors(
        torch.from_numpy(c("weight")).view(torch.float8_e4m3fn), _t16(c("weight_scale"), dt),
        input_scale=_t16(c("input_scale"), dt) if f"{name}.input_scale" in CASES.files else None,
        device="cpu", post_init=False)
    assert torch.equal(m.dequantize_weight(dtype=dt), _t16(c("W"), dt))


@pytest.mark.parametrize("name", NAMES)
def test_quantiser_mirror_within_one_step_of_compressed_tensors(name):
    """compressed-tensors rounds the scale and the quotient to T before the e4m3 cast; the fp32 arithmetic of this
    package picks the same code or one e4m3 step (one code apart, same sign) away."""
    c = lambda k: CASES[f"{name}.{k}"]  # noqa: E731
    x = fo.unpack16(c("x"))
    if f"{name}.input_scale" in CASES.files:
        codes, _ = fm.quantize_static(x, fo.unpack16(c("input_scale"))[0])
    else:
        codes, s = fm.quantize_dynamic(x)
        live = np.abs(x).max(axis=1) > 0  # an all-zero row: compressed-tensors' scale is eps(T), this one 1e-10 / 448
        assert not live.all() and np.all(np.abs(s - fo.unpack16(c("s_x"))[:, 0])[live] <= 2.0 ** -7 * s[live])
    ct = c("codes")
    same = codes == ct
    a, b = codes.astype(np.int16), ct.astype(np.int16)
    one_step = (np.abs(a - b) == 1) & ((a & 0x80) == (b & 0x80))
    zero_pair = np.isin(a, (0, 0x80)) & np.isin(b, (0, 1, 0x80, 0x81)) | np.isin(b, (0, 0x80)) & np.isin(a, (0, 1, 0x80, 0x81))
    assert np.all(same | one_step | zero_pair)
    print(f"{name}: {100 * (1 - same.mean()):.2f} % of codes one step from compressed-tensors'")


# ---- ABI argument checks (return -2 before any CUDA work) ---------------------------------------------------------------
def test_abi_argument_checks_without_gpu():
    P = 1 << 20  # any 16-byte aligned non-NULL value: a refused call never dereferences it
    assert lib.b2q_fp8ch_workspace_bytes(0, 4096) == 0 and lib.b2q_fp8ch_workspace_bytes(8, 100) == 0
    assert lib.b2q_fp8ch_workspace_bytes(8, 4096) == 8 * 4096 + 32  # dynamic decode quantises in its own launch
    assert lib.b2q_fp8ch_workspace_bytes(9, 4096) == 9 * 4096 + 48
    assert lib.b2q_fp8ch_workspace_bytes(300, 256) == 300 * 256 + 1200
    good = dict(x=P, w=P, s=P, s_in=None, ub=float("inf"), bias=None, out=P, M=16, K=256, N=128, dt=0, ws=P, nws=1 << 30)

    def fwd(**kw):
        a = {**good, **kw}
        return lib.b2q_fp8ch_forward(a["x"], a["w"], a["s"], a["s_in"], a["ub"], a["bias"], a["out"], a["M"], a["K"],
                                     a["N"], a["dt"], a["ws"], a["nws"], None)

    bad = (dict(w=None), dict(s=None), dict(out=None), dict(x=None), dict(dt=2), dict(M=-1), dict(K=64), dict(K=0),
           dict(K=65536 + 128), dict(N=96), dict(N=0), dict(x=P + 8), dict(out=P + 2), dict(w=P + 4), dict(s=P + 4),
           dict(ws=None), dict(ws=P + 8), dict(nws=16 * 256), dict(ub=0.0), dict(ub=-1.0), dict(ub=float("nan")),
           dict(M=8, ws=None), dict(M=1, nws=256))
    for kw in bad:
        assert fwd(**kw) == -2, kw
        assert lib.b2q_last_error()
    assert fwd(M=0) == 0 and fwd(M=0, x=None, ws=None) == 0  # an empty batch is a no-op
    assert fwd(M=0, s_in=P, ub=float("nan")) == 0  # static scales take no bound
    assert fwd(M=9, s_in=P, ws=None) == -2  # static prefill needs the workspace, static decode does not (no GPU call here)

    def mm(**kw):
        a = {**good, "codes": P, "sx": P, "ks": 0, **kw}
        return lib.b2q_fp8ch_mm(a["codes"], a["sx"], a["w"], a["s"], a["bias"], a["out"], a["M"], a["K"], a["N"],
                                a["dt"], a["ks"], None)

    for kw in (dict(codes=None), dict(sx=None), dict(codes=P + 1), dict(ks=9), dict(w=None), dict(K=192), dict(N=32),
               dict(dt=-1)):
        assert mm(**kw) == -2, kw
    assert mm(M=0) == 0

    def quant(**kw):
        a = {"x": P, "codes": P, "sx": P, "M": 4, "K": 256, "ub": float("inf"), "dt": 1, **kw}
        return lib.b2q_fp8ch_quantize(a["x"], a["codes"], a["sx"], a["M"], a["K"], a["ub"], a["dt"], None)

    for kw in (dict(x=None), dict(codes=None), dict(sx=None), dict(x=P + 2), dict(sx=P + 4), dict(K=100), dict(M=-2),
               dict(dt=3), dict(ub=0.0)):
        assert quant(**kw) == -2, kw
    assert quant(M=0) == 0

    def squant(**kw):
        a = {"x": P, "s_in": P, "codes": P, "sx": P, "M": 4, "K": 256, "dt": 0, **kw}
        return lib.b2q_fp8ch_quantize_static(a["x"], a["s_in"], a["codes"], a["sx"], a["M"], a["K"], a["dt"], None)

    for kw in (dict(x=None), dict(s_in=None), dict(codes=None), dict(sx=None), dict(codes=P + 8), dict(K=64),
               dict(dt=2)):
        assert squant(**kw) == -2, kw
    assert squant(M=0) == 0


# ---- what the compiler made ---------------------------------------------------------------------------------------------
def test_new_kernels_do_not_spill():
    log = os.path.join(os.path.dirname(HERE), "gptqmodel_b200", "csrc", "b2q_fp8ch.o.log")
    if not os.path.exists(log):
        pytest.skip("b2q_fp8ch.o.log is written by the in-tree build")
    text = open(log).read()
    entries = re.findall(r"Compiling entry function '(\w+)'.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", text, flags=re.S)
    names = [e[0] for e in entries]
    assert sum("fp8ch_gemm_kernel" in n for n in names) == 7
    assert sum("fp8ch_quant_kernel" in n for n in names) == 2 and sum("fp8ch_static_quant_kernel" in n for n in names) == 2
    for name, stack, st, ld in entries:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), name
