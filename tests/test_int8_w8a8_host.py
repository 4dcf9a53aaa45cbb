"""Per-channel / per-tensor INT8 (W8A8) host side: compressed-tensors `int-quantized` config parsing and refusals, the
loader on a synthetic checkpoint, the module's scales and dequantiser, compressed-tensors' fixture, the ABI's argument
checks and the compiler's report on the new kernels.  No GPU needed."""
import json
import os
import re

import numpy as np
import pytest
import torch

import int8_w8a8_mirror as im
from gptqmodel_b200 import B200ChannelInt8Linear, lib
from gptqmodel_b200.fp8_channel import channel_scales
from gptqmodel_b200.loader import load_int8_w8a8_linears, parse_fp8_w8a8_config, parse_int8_w8a8_config
from oracle import fp8_block_oracle as fo

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = np.load(os.path.join(HERE, "golden", "int8_w8a8_cases.npz"))


def ct_config(preset, fmt="int-quantized", **kw):
    """A compressed-tensors config as its own QuantizationConfig writes it."""
    from compressed_tensors.quantization import QuantizationConfig, preset_name_to_scheme

    cfg = QuantizationConfig(config_groups={"group_0": preset_name_to_scheme(preset, ["Linear"])}, format=fmt, **kw)
    return json.loads(json.dumps(cfg.model_dump(mode="json")))


def _set(raw, where, **kw):
    """A deep copy of raw with config_groups.group_0.<where> updated by kw (where = "" for the group itself)."""
    raw = json.loads(json.dumps(raw))
    g = raw["config_groups"]["group_0"]
    (g[where] if where else g).update(kw)
    return raw


DYN = ct_config("W8A8", ignore=["lm_head"])
STATIC = _set(DYN, "input_activations", strategy="tensor", dynamic=False)
TENSOR_W = _set(STATIC, "weights", strategy="tensor")


# ---- config parsing ---------------------------------------------------------------------------------------------------
def test_presets_accepted():
    w = DYN["config_groups"]["group_0"]["weights"]
    assert (w["type"], w["num_bits"], w["symmetric"], w["strategy"]) == ("int", 8, True, "channel")
    s = parse_int8_w8a8_config(DYN)
    assert (s.weight_strategy, s.activation, s.ub, s.ignore) == ("channel", "dynamic", None, ("lm_head",))
    assert (parse_int8_w8a8_config(STATIC).weight_strategy, parse_int8_w8a8_config(STATIC).activation) == (
        "channel", "static")
    assert parse_int8_w8a8_config(TENSOR_W).weight_strategy == "tensor"
    assert parse_int8_w8a8_config(_set(TENSOR_W, "input_activations", strategy="token", dynamic=True)).activation == \
        "dynamic"
    kv = {"num_bits": 8, "type": "float", "strategy": "tensor", "dynamic": False, "symmetric": True}
    assert parse_int8_w8a8_config({**DYN, "kv_cache_scheme": kv}).kv_cache_scheme == kv  # left to the caller
    two = json.loads(json.dumps(DYN))
    two["config_groups"]["group_1"] = two["config_groups"]["group_0"]
    assert parse_int8_w8a8_config(two).activation == "dynamic"


def test_ignore_names_and_patterns():
    s = parse_int8_w8a8_config({**DYN, "ignore": ["lm_head", "re:.*mlp\\.gate$", "re:model\\.layers\\.0\\..*"]})
    assert s.ignores("lm_head") and not s.ignores("model.lm_head")
    assert s.ignores("model.layers.5.mlp.gate") and not s.ignores("model.layers.5.mlp.gate_proj")
    assert s.ignores("model.layers.0.self_attn.q_proj") and not s.ignores("model.layers.10.self_attn.q_proj")


@pytest.mark.parametrize("raw", [DYN, STATIC, TENSOR_W])
def test_fp8_parser_still_refuses_int(raw):
    with pytest.raises(NotImplementedError):
        parse_fp8_w8a8_config(raw)
    with pytest.raises(NotImplementedError, match="8-bit float only"):
        parse_fp8_w8a8_config({**raw, "format": "float-quantized"})


@pytest.mark.parametrize("raw", [
    _set(DYN, "input_activations", symmetric=False),  # asymmetric (azp) activations
    _set(DYN, "weights", symmetric=False),
    _set(DYN, "weights", strategy="group", group_size=128),
    _set(DYN, "weights", strategy="block", block_structure=[128, 128]),
    _set(DYN, "input_activations", strategy="group", group_size=128),
    _set(DYN, "weights", type="float"),
    _set(DYN, "input_activations", type="float"),
    _set(DYN, "weights", num_bits=4),
    _set(DYN, "input_activations", num_bits=4),
    _set(DYN, "weights", dynamic=True),
    _set(DYN, "input_activations", dynamic=False),  # static per-token
    _set(STATIC, "input_activations", dynamic=True),  # dynamic per-tensor
    _set(DYN, "", input_activations=None),  # weight-only (W8A16)
    _set(DYN, "", output_activations=dict(DYN["config_groups"]["group_0"]["weights"])),
    _set(DYN, "", targets=["Linear", "Embedding"]),
    _set(DYN, "", format="pack-quantized"),
    {**DYN, "format": "pack-quantized"},
    {**DYN, "format": "float-quantized"},
    ct_config("FP8_DYNAMIC", fmt="float-quantized"),
    ct_config("W4A16", fmt="pack-quantized"),
    {"quant_method": "fbgemm_fp8"},
    {"quant_method": "gptq", "bits": 4},
])
def test_refusals(raw):
    with pytest.raises(NotImplementedError):
        parse_int8_w8a8_config(raw)


def test_mixed_groups_refused():
    mixed = json.loads(json.dumps(DYN))
    mixed["config_groups"]["group_1"] = STATIC["config_groups"]["group_0"]  # dynamic with static
    with pytest.raises(NotImplementedError, match="mixed"):
        parse_int8_w8a8_config(mixed)
    mixed["config_groups"]["group_1"] = ct_config("W4A16")["config_groups"]["group_0"]
    with pytest.raises(NotImplementedError):
        parse_int8_w8a8_config(mixed)


@pytest.mark.parametrize("raw", [
    [],
    {**DYN, "config_groups": {}},
    {**DYN, "config_groups": {"group_0": 3}},
    _set(DYN, "weights", num_bits="8"),
    _set(DYN, "weights", type="integer"),
    _set(DYN, "weights", strategy="rows"),
    _set(DYN, "input_activations", symmetric="yes"),
    _set(DYN, "weights", dynamic=None),
    _set(DYN, "", weights=7),
    _set(DYN, "", targets="Linear"),
    {**DYN, "ignore": "lm_head"},
    {**DYN, "ignore": ["re:("]},
    {**DYN, "kv_cache_scheme": "int8"},
])
def test_malformed(raw):
    with pytest.raises(ValueError):
        parse_int8_w8a8_config(raw)


# ---- loader -------------------------------------------------------------------------------------------------------------
def _write_ckpt(path, cfg, tensors):
    from safetensors.torch import save_file

    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump({"model_type": "llama", "quantization_config": cfg}, f)
    save_file(tensors, os.path.join(path, "model.safetensors"))


def _i8(N, K, seed):
    return torch.randint(-128, 128, (N, K), generator=torch.Generator().manual_seed(seed), dtype=torch.int8)


def _scale(shape, dtype, seed):
    return (torch.rand(shape, generator=torch.Generator().manual_seed(seed)) * 1e-2 + 1e-4).to(dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", [(192, 1), (192,), (1,), ()])
def test_loader_scale_shapes_and_exact_widening(tmp_path, shape, dtype):
    ws = _scale(shape, dtype, 1)
    pre = "model.layers.0.self_attn.q_proj"
    t = {f"{pre}.weight": _i8(192, 256, 0), f"{pre}.weight_scale": ws, f"{pre}.bias": torch.zeros(192, dtype=dtype),
         f"{pre}.weight_zero_point": torch.zeros(ws.shape, dtype=torch.int8),
         "lm_head.weight": torch.randn(64, 256, dtype=torch.bfloat16), "model.norm.weight": torch.ones(256)}
    _write_ckpt(str(tmp_path), DYN if len(shape) and shape[0] > 1 else _set(DYN, "weights", strategy="tensor"), t)
    mods = load_int8_w8a8_linears(str(tmp_path), device="cpu", post_init=False)
    assert sorted(mods) == [pre]
    m = mods[pre]
    assert isinstance(m, B200ChannelInt8Linear)
    assert (m.in_features, m.out_features, m.activation, m.input_scale) == (256, 192, "dynamic", None)
    assert torch.equal(m.weight, t[f"{pre}.weight"]) and m.weight_scale.dtype == dtype and m.bias is not None
    s = channel_scales(m.weight_scale, 192)
    assert s.dtype == torch.float32 and s.shape == (192,)
    assert torch.equal(s.to(dtype), ws.reshape(-1).expand(192))  # widening is exact
    assert "int8 W8A8" in m.extra_repr() and "dynamic per-token" in m.extra_repr()


def test_loader_static_qwen_names_ignore_and_zero_points(tmp_path):
    t = {}
    for i in range(2):
        for n, N in (("self_attn.q_proj", 128), ("mlp.down_proj", 64), ("mlp.gate", 64)):
            p = f"model.layers.{i}.{n}"
            t[f"{p}.weight"] = _i8(N, 256, i)
            t[f"{p}.weight_scale"] = _scale((N, 1), torch.bfloat16, i)
            t[f"{p}.input_scale"] = _scale((1,), torch.bfloat16, i + 10)
            t[f"{p}.input_zero_point"] = torch.zeros(1, dtype=torch.int8)
    cfg = {**STATIC, "ignore": ["re:.*mlp\\.gate$", "model.layers.1.self_attn.q_proj"]}
    _write_ckpt(str(tmp_path / "a"), cfg, t)
    mods = load_int8_w8a8_linears(str(tmp_path / "a"), device="cpu", post_init=False)
    assert sorted(mods) == ["model.layers.0.mlp.down_proj", "model.layers.0.self_attn.q_proj",
                            "model.layers.1.mlp.down_proj"]
    assert all(m.activation == "static" for m in mods.values())
    m = mods["model.layers.0.self_attn.q_proj"]
    assert torch.equal(m.input_scale, t["model.layers.0.self_attn.q_proj.input_scale"])
    assert "static per-tensor" in m.extra_repr()
    assert set(load_int8_w8a8_linears(str(tmp_path / "a"), device="cpu", only=["model.layers.1.mlp.down_proj"],
                                      post_init=False)) == {"model.layers.1.mlp.down_proj"}
    for zp in ("input_zero_point", "weight_zero_point"):
        bad = dict(t)
        bad[f"model.layers.0.mlp.down_proj.{zp}"] = torch.ones(64 if zp == "weight_zero_point" else 1, dtype=torch.int8)
        _write_ckpt(str(tmp_path / zp), cfg, bad)
        with pytest.raises(NotImplementedError, match=zp):
            load_int8_w8a8_linears(str(tmp_path / zp), device="cpu", post_init=False)


def test_loader_refuses_missing_or_extra_input_scale_and_fp8_weights(tmp_path):
    _write_ckpt(str(tmp_path / "a"), STATIC, {"m.q.weight": _i8(128, 256, 0),
                                             "m.q.weight_scale": _scale((128, 1), torch.float32, 1)})
    with pytest.raises(NotImplementedError, match="input_scale"):
        load_int8_w8a8_linears(str(tmp_path / "a"), device="cpu", post_init=False)
    _write_ckpt(str(tmp_path / "b"), DYN, {"m.q.weight": _i8(128, 256, 0), "m.q.input_scale": torch.ones(1),
                                          "m.q.weight_scale": _scale((128, 1), torch.float32, 1)})
    with pytest.raises(NotImplementedError, match="input_scale"):
        load_int8_w8a8_linears(str(tmp_path / "b"), device="cpu", post_init=False)
    _write_ckpt(str(tmp_path / "c"), DYN, {"m.q.weight": torch.zeros(128, 256).to(torch.float8_e4m3fn),
                                          "m.q.weight_scale": _scale((128, 1), torch.float32, 1)})
    with pytest.raises(NotImplementedError, match="int8"):
        load_int8_w8a8_linears(str(tmp_path / "c"), device="cpu", post_init=False)


@pytest.mark.parametrize("ws", [torch.rand(128, 2), torch.rand(64, 1), -torch.rand(128, 1),
                                torch.full((1,), float("inf")), torch.zeros(()), torch.full((128,), float("nan"))])
def test_loader_rejects_bad_scales(tmp_path, ws):
    _write_ckpt(str(tmp_path), DYN, {"m.q.weight": _i8(128, 256, 0), "m.q.weight_scale": ws})
    with pytest.raises(ValueError, match="weight_scale"):
        load_int8_w8a8_linears(str(tmp_path), device="cpu", post_init=False)


def test_module_envelope_and_arguments():
    for K, N in ((192, 128), (256, 96), (0, 128), (65536 + 128, 128)):
        with pytest.raises(NotImplementedError):
            B200ChannelInt8Linear(in_features=K, out_features=N)
    with pytest.raises(ValueError):
        B200ChannelInt8Linear(256, 128, activation="sometimes")
    with pytest.raises(ValueError):
        B200ChannelInt8Linear(256, 128, ub=100.0)
    m = B200ChannelInt8Linear(256, 128, bias=True)
    assert m.weight.dtype == torch.int8 and m.weight.shape == (128, 256) and m.input_scale is None
    assert B200ChannelInt8Linear(256, 128, activation="static").input_scale.shape == (1,)
    mk = lambda w, **kw: B200ChannelInt8Linear.from_checkpoint_tensors(w, torch.ones(128), device="cpu",  # noqa: E731
                                                                       post_init=False, **kw)
    with pytest.raises(NotImplementedError, match="int8"):
        mk(_i8(128, 256, 0).to(torch.uint8))
    with pytest.raises(NotImplementedError, match="int8"):
        mk(torch.zeros(128, 256).to(torch.float8_e4m3fn))
    with pytest.raises(ValueError):
        mk(_i8(128, 256, 0), input_scale=torch.ones(2))
    with pytest.raises(ValueError):
        mk(_i8(128, 256, 0), input_scale=torch.zeros(1))
    with pytest.raises(NotImplementedError, match="input_scale"):
        mk(_i8(128, 256, 0), activation="static")
    with pytest.raises(NotImplementedError, match="input_scale"):
        mk(_i8(128, 256, 0), activation="dynamic", input_scale=torch.ones(1))


# ---- dequantisation and compressed-tensors' fixture ----------------------------------------------------------------------
@pytest.mark.parametrize("sdt", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", [(128, 1), (128,), (1,), ()])
def test_dequantize_weight_is_w_times_s(shape, sdt):
    w, s = _i8(128, 256, 3), _scale(shape, sdt, 4)
    m = B200ChannelInt8Linear.from_checkpoint_tensors(w, s, device="cpu", post_init=False)
    for dt in (torch.float16, torch.bfloat16):
        want = (w.to(sdt) * s.reshape(-1, 1) if s.numel() > 1 else w.to(sdt) * s.reshape(())).to(dt).t()
        assert torch.equal(m.dequantize_weight(dtype=dt), want)


NAMES = sorted({k.split(".")[0] for k in CASES.files})
_DT = {"bf": torch.bfloat16, "16": torch.float16}


def _t16(a, dtype):
    return torch.from_numpy(fo.unpack16(a)).to(dtype)


def test_fixture_cases():
    assert NAMES == ["dyn_16", "dyn_bf", "static_16", "static_bf"]


@pytest.mark.parametrize("name", NAMES)
def test_dequantize_matches_compressed_tensors(name):
    dt = _DT[name.rsplit("_", 1)[1]]
    c = lambda k: CASES[f"{name}.{k}"]  # noqa: E731
    m = B200ChannelInt8Linear.from_checkpoint_tensors(
        torch.from_numpy(c("weight")), _t16(c("weight_scale"), dt),
        input_scale=_t16(c("input_scale"), dt) if f"{name}.input_scale" in CASES.files else None,
        device="cpu", post_init=False)
    assert torch.equal(m.dequantize_weight(dtype=dt), _t16(c("W"), dt))


@pytest.mark.parametrize("name", NAMES)
def test_quantiser_mirror_against_compressed_tensors(name):
    """compressed-tensors' token scale is amax / 127.5 (this package's amax / 127, as vLLM's and SmoothQuant's) and it
    rounds the scale and the quotient to T: codes may differ by one step.  The share that differs is printed."""
    c = lambda k: CASES[f"{name}.{k}"]  # noqa: E731
    x = fo.unpack16(c("x"))
    if f"{name}.input_scale" in CASES.files:
        codes, _ = im.quantize_static(x, fo.unpack16(c("input_scale"))[0])
    else:
        codes, s = im.quantize_dynamic(x)
        live = np.abs(x).max(axis=1) > 0
        assert not live.all() and not codes[~live].any() and np.all(np.isfinite(s))
        ct_s = fo.unpack16(c("s_x"))[:, 0]
        assert np.all(np.abs(s * np.float32(127 / 127.5) - ct_s)[live] <= 2.0 ** -7 * s[live])
    ct = c("codes").astype(np.int16)
    diff = np.abs(codes.astype(np.int16) - ct)
    assert diff.max() <= 1
    print(f"{name}: {100 * (diff > 0).mean():.2f} % of codes one step from compressed-tensors'")


def test_mirror_rounds_half_to_even_and_saturates():
    x = np.array([[0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 1000.0, -1000.0]], np.float32)
    codes, s = im.quantize_static(x, 1.0)
    assert codes.tolist() == [[0, 2, 2, 0, -2, -2, 127, -128]] and s.tolist() == [1.0]
    codes, s = im.quantize_dynamic(np.zeros((2, 16), np.float32))
    assert not codes.any() and np.all(s == np.float32(1e-10) / np.float32(127))


# ---- ABI argument checks (return -2 before any CUDA work) ---------------------------------------------------------------
def test_abi_argument_checks_without_gpu():
    P = 1 << 20  # any 16-byte aligned non-NULL value: a refused call never dereferences it
    assert lib.b2q_int8ch_workspace_bytes(0, 4096) == 0 and lib.b2q_int8ch_workspace_bytes(8, 100) == 0
    assert lib.b2q_int8ch_workspace_bytes(1, 4096) == 4096 + 16  # every M quantises in its own launch
    assert lib.b2q_int8ch_workspace_bytes(9, 4096) == 9 * 4096 + 48
    assert lib.b2q_int8ch_workspace_bytes(300, 256) == 300 * 256 + 1200
    good = dict(x=P, w=P, s=P, s_in=None, bias=None, out=P, M=16, K=256, N=128, dt=0, ws=P, nws=1 << 30)

    def fwd(**kw):
        a = {**good, **kw}
        return lib.b2q_int8ch_forward(a["x"], a["w"], a["s"], a["s_in"], a["bias"], a["out"], a["M"], a["K"], a["N"],
                                      a["dt"], a["ws"], a["nws"], None)

    bad = (dict(w=None), dict(s=None), dict(out=None), dict(x=None), dict(dt=2), dict(M=-1), dict(K=64), dict(K=0),
           dict(K=65536 + 128), dict(N=96), dict(N=0), dict(x=P + 8), dict(out=P + 2), dict(w=P + 4), dict(s=P + 4),
           dict(ws=None), dict(ws=P + 8), dict(nws=16 * 256), dict(M=1, ws=None), dict(M=1, s_in=P, ws=None),
           dict(M=1, nws=256))
    for kw in bad:
        assert fwd(**kw) == -2, kw
        assert lib.b2q_last_error()
    assert fwd(M=0) == 0 and fwd(M=0, x=None, ws=None) == 0  # an empty batch is a no-op

    def mm(**kw):
        a = {**good, "codes": P, "sx": P, "ks": 0, **kw}
        return lib.b2q_int8ch_mm(a["codes"], a["sx"], a["w"], a["s"], a["bias"], a["out"], a["M"], a["K"], a["N"],
                                 a["dt"], a["ks"], None)

    for kw in (dict(codes=None), dict(sx=None), dict(codes=P + 1), dict(ks=9), dict(w=None), dict(s=None),
               dict(out=None), dict(K=192), dict(N=32), dict(dt=-1), dict(M=-1)):
        assert mm(**kw) == -2, kw
    assert mm(M=0) == 0

    def quant(**kw):
        a = {"x": P, "codes": P, "sx": P, "M": 4, "K": 256, "dt": 1, **kw}
        return lib.b2q_int8ch_quantize(a["x"], a["codes"], a["sx"], a["M"], a["K"], a["dt"], None)

    for kw in (dict(x=None), dict(codes=None), dict(sx=None), dict(x=P + 2), dict(sx=P + 4), dict(K=100), dict(M=-2),
               dict(dt=3)):
        assert quant(**kw) == -2, kw
    assert quant(M=0) == 0

    def squant(**kw):
        a = {"x": P, "s_in": P, "codes": P, "sx": P, "M": 4, "K": 256, "dt": 0, **kw}
        return lib.b2q_int8ch_quantize_static(a["x"], a["s_in"], a["codes"], a["sx"], a["M"], a["K"], a["dt"], None)

    for kw in (dict(x=None), dict(s_in=None), dict(codes=None), dict(sx=None), dict(codes=P + 8), dict(K=64),
               dict(dt=2)):
        assert squant(**kw) == -2, kw
    assert squant(M=0) == 0


# ---- what the compiler made ---------------------------------------------------------------------------------------------
def test_new_kernels_do_not_spill():
    log = os.path.join(os.path.dirname(HERE), "gptqmodel_b200", "csrc", "b2q_fp8ch.o.log")
    if not os.path.exists(log):
        pytest.skip("b2q_fp8ch.o.log is written by the in-tree build")
    entries = re.findall(r"Compiling entry function '(\w+)'.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", open(log).read(), flags=re.S)
    new = [e for e in entries if "int8ch_" in e[0]]
    assert sum("int8ch_gemm_kernel" in e[0] for e in new) == 5
    assert sum("int8ch_quant_kernel" in e[0] for e in new) == 2
    assert sum("int8ch_static_quant_kernel" in e[0] for e in new) == 2
    for name, stack, st, ld in new:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), name
