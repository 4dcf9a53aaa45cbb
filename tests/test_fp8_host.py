"""FP8 (e4m3fn, W8A16) host side: config parsing and refusals, layout inference, the oracle against the reference's
fixtures, the exhaustive check of the kernels' division sequence, code packing, the module envelope and the ABI's
argument checks.  No GPU needed."""
import json
import os

import numpy as np
import pytest
import torch

from gptqmodel_b200 import B200Fp8QuantLinear, lib
from gptqmodel_b200 import fp8 as F
from gptqmodel_b200.loader import load_quantized_linears, parse_quant_config
from oracle import fp8_oracle as fo

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = np.load(os.path.join(HERE, "golden", "fp8_cases.npz"))
NAMES = sorted({k.split(".")[0] for k in CASES.files})


# ---- config parsing ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [None, "fp8", "e4m3", "float8_e4m3", "float8_e4m3fn", " E4M3 "])
def test_config_format_aliases(fmt):
    raw = {"quant_method": "fp8", "bits": 8, "weight_scale_method": "row"}
    if fmt is not None:
        raw["format"] = fmt
    s = parse_quant_config(raw)
    assert (s.method, s.format, s.fp8_format, s.bits) == ("fp8", "fp8", "float8_e4m3fn", 8)
    assert (s.weight_scale_method, s.weight_block_size, s.group_size, s.desc_act) == ("row", None, -1, False)


def test_config_block_inferred_from_block_size():
    s = parse_quant_config({"method": "fp8", "format": "float8_e4m3fn", "weight_block_size": [128, 128]})
    assert (s.weight_scale_method, s.weight_block_size) == ("block", (128, 128))
    s = parse_quant_config({"method": "fp8", "weight_scale_method": "tensor"})
    assert (s.weight_scale_method, s.weight_block_size) == ("tensor", None)


@pytest.mark.parametrize("fmt", ["e5m2", "float8_e5m2", "e4m3fnuz", "e5m2fnuz", "e8m0", "float8_e8m0fnu"])
def test_config_refuses_other_fp8_formats(fmt):
    with pytest.raises(NotImplementedError):
        parse_quant_config({"method": "fp8", "format": fmt})


@pytest.mark.parametrize("raw", [
    {"quant_method": "fp8", "activation_scheme": "dynamic", "fmt": "e4m3", "weight_block_size": [128, 128]},
    {"quant_method": "fp8", "activation_scheme": "static"},
    {"quant_method": "fp8", "fmt": "e4m3"},
    {"method": "fp8", "weight_scale_semantics": "direct"},
    {"method": "fp8", "rotation": "hadamard"},
])
def test_config_refusals(raw):
    with pytest.raises(NotImplementedError):
        parse_quant_config(raw)


@pytest.mark.parametrize("raw", [
    {"method": "fp8", "format": "bogus"},
    {"method": "fp8", "bits": 4},
    {"method": "fp8", "weight_scale_method": "row", "weight_block_size": [128, 128]},
    {"method": "fp8", "weight_scale_method": "block"},
    {"method": "fp8", "weight_scale_method": "column"},
    {"method": "fp8", "weight_block_size": [128]},
    {"method": "fp8", "weight_block_size": [0, 128]},
])
def test_config_invalid(raw):
    with pytest.raises(ValueError):
        parse_quant_config(raw)


def test_config_dynamic_overrides():
    raw = {"method": "fp8", "format": "e4m3", "weight_block_size": [128, 128],
           "dynamic": {"-:.*lm_head": {}, r".*mlp\.down_proj": {"weight_scale_method": "row"},
                       r".*o_proj": {"weight_block_size": [64, 128], "fmt": "float8_e4m3fn"}}}
    s = parse_quant_config(raw)
    assert s.for_module("model.lm_head") is None
    d = s.for_module("model.layers.0.mlp.down_proj")
    assert (d.weight_scale_method, d.weight_block_size) == ("row", None)
    o = s.for_module("model.layers.0.self_attn.o_proj")
    assert (o.weight_scale_method, o.weight_block_size, o.fp8_format) == ("block", (64, 128), "float8_e4m3fn")
    q = s.for_module("model.layers.0.self_attn.q_proj")
    assert (q.weight_scale_method, q.weight_block_size) == ("block", (128, 128))
    for bad, exc in (({"bits": 4}, ValueError), ({"group_size": 128}, ValueError), ({"format": "e5m2"}, NotImplementedError),
                     ({"weight_scale_semantics": "direct"}, NotImplementedError)):
        with pytest.raises(exc):
            parse_quant_config({"method": "fp8", "dynamic": {".*x": bad}})


# ---- layout inference ---------------------------------------------------------------------------------------------------
def test_layout_inference():
    assert F.infer_fp8_layout((256, 512), torch.ones(())) == ("tensor", None)
    assert F.infer_fp8_layout((256, 512), torch.ones(1)) == ("tensor", None)
    assert F.infer_fp8_layout((256, 512), torch.ones(256)) == ("row", None)
    assert F.infer_fp8_layout((256, 512), torch.ones(2, 4)) == ("block", (128, 128))
    assert F.infer_fp8_layout((256, 512), torch.ones(4, 8)) == ("block", (64, 64))
    assert F.infer_fp8_layout((256, 512), torch.ones(256, 4)) == ("block", (1, 128))
    for bad in (torch.ones(100), torch.ones(3, 4), torch.ones(2, 2, 2)):
        with pytest.raises(ValueError):
            F.infer_fp8_layout((256, 512), bad)


def test_layout_disagreement_raises():
    w = torch.zeros(256, 512, dtype=torch.float8_e4m3fn)
    with pytest.raises(ValueError, match="layout"):
        B200Fp8QuantLinear.from_checkpoint_tensors(w, torch.ones(256), weight_scale_method="tensor", device="cpu",
                                                   post_init=False)
    with pytest.raises(ValueError, match="layout"):
        B200Fp8QuantLinear.from_checkpoint_tensors(w, torch.ones(2, 4), weight_scale_method="block",
                                                   weight_block_size=[64, 128], device="cpu", post_init=False)
    m = B200Fp8QuantLinear.from_checkpoint_tensors(w, torch.ones(2, 4), weight_scale_method="block",
                                                   weight_block_size=[128, 128], device="cpu", post_init=False)
    assert (m.weight_scale_method, m.weight_block_size) == ("block", (128, 128))


# ---- the loader on a tiny checkpoint -----------------------------------------------------------------------------------
def _write_ckpt(path, cfg, tensors):
    from safetensors.torch import save_file

    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "quantize_config.json"), "w") as f:
        json.dump(cfg, f)
    save_file(tensors, os.path.join(path, "model.safetensors"))


def test_loader_finds_fp8_modules(tmp_path):
    w = torch.randn(128, 256).to(torch.float8_e4m3fn)
    t = {"a.q.weight": w, "a.q.weight_scale_inv": torch.full((1, 2), 3.0), "a.q.bias": torch.zeros(128, dtype=torch.float16),
         "a.o.weight": w.clone(), "a.o.weight_scale_inv": torch.full((128,), 2.0), "a.norm.weight": torch.ones(256)}
    _write_ckpt(str(tmp_path), {"method": "fp8", "format": "float8_e4m3fn", "weight_block_size": [128, 128],
                                "dynamic": {r".*\.o": {"weight_scale_method": "row"}}}, t)
    mods = load_quantized_linears(str(tmp_path), device="cpu")
    assert sorted(mods) == ["a.o", "a.q"]
    assert (mods["a.q"].weight_scale_method, mods["a.q"].weight_block_size) == ("block", (128, 128))
    assert mods["a.q"].bias is not None and mods["a.o"].weight_scale_method == "row"
    assert torch.equal(mods["a.q"].weight.view(torch.uint8), w.view(torch.uint8))


def test_loader_refuses_disagreeing_and_modelopt_tensors(tmp_path):
    w = torch.randn(128, 256).to(torch.float8_e4m3fn)
    _write_ckpt(str(tmp_path / "a"), {"method": "fp8", "weight_scale_method": "row"},
                {"l.weight": w, "l.weight_scale_inv": torch.ones(1, 2)})
    with pytest.raises(ValueError, match="layout"):
        load_quantized_linears(str(tmp_path / "a"), device="cpu")
    _write_ckpt(str(tmp_path / "b"), {"method": "fp8"}, {"l.weight": w, "l.weight_scale": torch.ones(128)})
    with pytest.raises(NotImplementedError, match="ModelOpt"):
        load_quantized_linears(str(tmp_path / "b"), device="cpu", only=["l"])
    _write_ckpt(str(tmp_path / "c"), {"method": "fp8", "weight_scale_method": "row"},
                {"l.weight": torch.randn(128, 256).to(torch.float8_e5m2), "l.weight_scale_inv": torch.ones(128)})
    with pytest.raises(NotImplementedError, match="float8_e4m3fn"):
        load_quantized_linears(str(tmp_path / "c"), device="cpu")


# ---- oracle against the reference's fixtures -------------------------------------------------------------------------
def _case(name):
    p = name + "."
    method = str(CASES[p + "method"])
    block = tuple(int(v) for v in CASES[p + "block"]) if method == "block" else None
    bias = CASES[p + "bias"]
    return CASES[p + "weight"], CASES[p + "scale_inv"], method, block, (bias if bias.size else None)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("tag,dt", [("16", "fp16"), ("bf", "bf16")])
def test_oracle_dequant_equals_fixture_bit_for_bit(name, tag, dt):
    codes, sinv, method, block, _ = _case(name)
    W = fo.dequantize(codes, sinv, method, block, dt)
    ref = CASES[f"{name}.W{tag}"]
    assert W.dtype == ref.dtype and W.shape == ref.shape
    assert np.array_equal(W.view(np.uint16 if dt == "fp16" else np.uint32), ref.view(np.uint16 if dt == "fp16" else np.uint32))


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("tag,dt", [("16", "fp16"), ("bf", "bf16")])
def test_oracle_forward_matches_fixture(name, tag, dt):
    """The reference multiplies in T with fp32 accumulation; the oracle is exact: within a few ulp of T."""
    codes, sinv, method, block, bias = _case(name)
    W = fo.dequantize(codes, sinv, method, block, dt)
    y = fo.forward(CASES[f"{name}.x{tag}"], W, bias, dt).astype(np.float64)
    ref = CASES[f"{name}.y{tag}"].astype(np.float64)
    ulp = 2.0 ** -10 if dt == "fp16" else 2.0 ** -7
    assert np.all(np.abs(y - ref) <= 2 * ulp * np.abs(ref) + 1e-6 * np.abs(ref).max())


def test_module_scale_tables_match_oracle():
    for name in NAMES:
        codes, sinv, method, block, _ = _case(name)
        N, K = codes.shape
        for dt, t in ((torch.float16, "fp16"), (torch.bfloat16, "bf16")):
            table, g = F.expand_scales(torch.from_numpy(sinv), N, K, method, block, dt)
            assert g == (block[1] if block else K) and table.shape == (K // g, N)
            full = fo.round_to(fo.expand_scale_inv(sinv, N, K, method, block), t).astype(np.float32)  # [N, K]
            got = table.float().repeat_interleave(g, dim=0).t().numpy()
            assert np.array_equal(got, full)


# ---- the kernels' division sequence, exhaustively ---------------------------------------------------------------------
def _mirror(w, s):
    """numpy mirror of DequantFp8 (b2q_dequant.cuh) in fp32: r = RN(1/s); q0 = RN(w r); en = fma(q0, s, -w);
    q = fma(-en, r, q0) for |s| in [2^-100, 2^100], the IEEE quotient otherwise.  fp32 fma is emulated in float64: the product of two fp32
    values is exact in float64 and a float64 sum rounded to fp32 is the fp32-rounded sum (53 >= 2 * 24 + 2)."""
    f32 = np.float32
    with np.errstate(all="ignore"):
        r = (f32(1.0) / s).astype(f32)
        q0 = (w * r).astype(f32)
        en = (q0.astype(np.float64) * s.astype(np.float64) - w.astype(np.float64)).astype(f32)
        q = (-(en.astype(np.float64)) * r.astype(np.float64) + q0.astype(np.float64)).astype(f32)
        ex = (s.view(np.uint32) >> 23) & 0xFF
        fast = (ex >= 27) & (ex <= 227)
        return np.where(fast, q, (w / s).astype(f32))


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
def test_division_sequence_exhaustive(dt):
    """All 256 codes x every finite positive scale of T: RN_T(mirror) == RN_T(T(w) / T(s))."""
    w = fo.e4m3_table().astype(np.float32)
    if dt == "fp16":
        s = np.arange(1, 0x7C00, dtype=np.uint16).view(np.float16).astype(np.float32)
    else:
        s = (np.arange(1, 0x7F80, dtype=np.uint32) << 16).view(np.float32)
    ok = ~np.isnan(w)
    W, S = np.meshgrid(w[ok], s, indexing="ij")
    got = fo.round_to(_mirror(W.ravel(), S.ravel()), dt)
    ref = fo.div_t(W.ravel(), S.ravel(), dt)
    bad = ~(((got == ref) & (np.signbit(got) == np.signbit(ref))) | (np.isnan(got) & np.isnan(ref)))
    assert not bad.any(), f"{int(bad.sum())} mismatches, first w={W.ravel()[bad][0]} s={S.ravel()[bad][0]}"
    # the sequence itself is the correctly rounded fp32 quotient, not only after the rounding to T
    with np.errstate(all="ignore"):
        q32 = (W.ravel() / S.ravel()).astype(np.float32)
    m = _mirror(W.ravel(), S.ravel())
    assert np.array_equal(m[~np.isnan(q32)], q32[~np.isnan(q32)])


# ---- code packing -----------------------------------------------------------------------------------------------------
def test_pack_unpack_round_trip():
    g = torch.Generator().manual_seed(3)
    codes = torch.randint(0, 256, (96, 256), generator=g, dtype=torch.uint8)
    q = F.pack_fp8_codes(codes)
    assert q.shape == (64, 96) and q.dtype == torch.int32
    assert torch.equal(F.unpack_fp8_codes(q), codes)
    # byte j of word [i, n] is the code of row 4i + j
    for (i, n, j) in ((0, 0, 0), (5, 17, 3), (63, 95, 2)):
        assert (int(q[i, n]) >> (8 * j)) & 0xFF == int(codes[n, 4 * i + j])
    assert torch.equal(F.pack_fp8_codes(codes.view(torch.float8_e4m3fn)), q)


# ---- module envelope ----------------------------------------------------------------------------------------------------
def test_module_envelope():
    ok = dict(bits=8, group_size=-1, sym=True, desc_act=False, in_features=512, out_features=256)
    m = B200Fp8QuantLinear(**ok, bias=True, weight_scale_method="block", weight_block_size=[128, 128])
    assert m.weight.dtype == torch.float8_e4m3fn and m.weight.shape == (256, 512)
    assert m.weight_scale_inv.shape == (2, 4) and m.bias.shape == (256,)
    assert len(m.list_buffers()) == 3
    assert B200Fp8QuantLinear(**ok).weight_scale_inv.shape == (256,)
    assert B200Fp8QuantLinear(**ok, weight_scale_method="tensor").weight_scale_inv.shape == ()
    B200Fp8QuantLinear(**ok, weight_scale_method="block", weight_block_size=[1, 512])   # bc == K: per-channel table
    B200Fp8QuantLinear(**ok, weight_scale_method="block", weight_block_size=[32, 64])
    for kw in (dict(weight_block_size=[128, 32]), dict(weight_block_size=[128, 256]), dict(weight_block_size=[96, 128])):
        with pytest.raises(NotImplementedError):
            B200Fp8QuantLinear(**ok, weight_scale_method="block", **kw)
    for bad in (dict(in_features=500), dict(out_features=100), dict(bits=4)):
        with pytest.raises(NotImplementedError):
            B200Fp8QuantLinear(**{**ok, **bad})
    with pytest.raises(NotImplementedError):
        B200Fp8QuantLinear(**ok, format="e5m2")
    with pytest.raises(NotImplementedError):
        B200Fp8QuantLinear(**ok, weight_scale_semantics="direct")
    ok2, err = B200Fp8QuantLinear.validate(bits=8, in_features=512, out_features=256, dtype=torch.float32)
    assert not ok2 and isinstance(err, NotImplementedError)


def test_tp_helpers_refuse_fp8():
    from gptqmodel_b200 import tp

    layer = {"weight": torch.zeros(64, 128, dtype=torch.float8_e4m3fn), "weight_scale_inv": torch.ones(64)}
    for fn in (tp.shard_columns, tp.shard_rows):
        with pytest.raises(NotImplementedError, match="FP8"):
            fn(layer, 0, 2)
    m = B200Fp8QuantLinear(bits=8, group_size=-1, sym=True, desc_act=False, in_features=128, out_features=64)
    with pytest.raises(NotImplementedError, match="FP8"):
        tp.RowParallelLinear(m)


# ---- ABI argument checks (return -2 before any CUDA work) ---------------------------------------------------------------
def test_abi_argument_checks_without_gpu():
    assert lib.b2q_version() == 8
    P = 1 << 20  # any 16-byte aligned non-NULL value: a refused call never dereferences it
    good = dict(x=P, packed=P, scales=P, bias=None, out=P, M=4, K=256, N=128, g=128, dt=0)

    def mm(**kw):
        a = {**good, **kw}
        return lib.b2q_fp8_mm(a["x"], a["packed"], a["scales"], a["bias"], a["out"], a["M"], a["K"], a["N"], a["g"],
                              a["dt"], None, 0, None)

    for kw in (dict(packed=None), dict(scales=None), dict(out=None), dict(x=None), dict(dt=2), dict(M=-1),
               dict(K=100), dict(K=0), dict(N=48), dict(g=32), dict(g=256, K=512), dict(g=96), dict(K=192, g=128),
               dict(x=P + 8), dict(out=P + 2), dict(packed=P + 4)):
        assert mm(**kw) == -2, kw
        assert lib.b2q_last_error()
    assert mm(M=0) == 0  # an empty batch is a no-op
    assert mm(M=0, x=None) == 0
    for kw in (dict(g=256, K=256), dict(g=64)):
        assert mm(M=0, **kw) == 0

    def dq(**kw):
        a = {**good, **kw}
        return lib.b2q_fp8_dequant(a["packed"], a["scales"], a["out"], a["K"], a["N"], a["g"], a["dt"], None)

    for kw in (dict(packed=None), dict(scales=None), dict(out=None), dict(dt=-1), dict(K=96), dict(N=16), dict(g=32),
               dict(out=P + 8)):
        assert dq(**kw) == -2, kw
