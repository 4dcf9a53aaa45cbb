"""Checkpoint loader: config spellings, dynamic overrides, v1 -> v2 zero-points, sharded files.

Host-side only: tiny synthetic checkpoints are written with safetensors and loaded onto the CPU without post_init();
the tensors the modules end up holding are compared with the oracle (dequantised weights must survive the trip).
"""
import json
import os

import pytest
import torch
from safetensors.torch import save_file

import oracle
from gptqmodel_b200 import loader
from helpers import make_layer


def _write(tmp, layers, cfg, cfg_file="quantize_config.json", shards=1):
    names = sorted(layers)
    per = (len(names) + shards - 1) // shards
    wmap = {}
    for si in range(shards):
        blob = {}
        for n in names[si * per:(si + 1) * per]:
            for k, v in layers[n].items():
                if isinstance(v, torch.Tensor):
                    blob[f"{n}.{k}"] = v.contiguous()
        fn = "model.safetensors" if shards == 1 else f"model-{si + 1:05d}-of-{shards:05d}.safetensors"
        save_file(blob, os.path.join(tmp, fn))
        wmap.update({k: fn for k in blob})
    if shards > 1:
        json.dump({"weight_map": wmap}, open(os.path.join(tmp, "model.safetensors.index.json"), "w"))
    if cfg_file == "config.json":
        json.dump({"model_type": "llama", "quantization_config": cfg}, open(os.path.join(tmp, cfg_file), "w"))
    else:
        json.dump(cfg, open(os.path.join(tmp, cfg_file), "w"))


def _ckpt_tensors(L):
    d = {k: L[k] for k in ("qweight", "qzeros", "scales", "g_idx")}
    if L.get("bias") is not None:
        d["bias"] = L["bias"]
    return d


def test_config_spellings():
    s = loader.parse_quant_config({"bits": 4, "group_size": 64, "desc_act": True, "sym": False, "checkpoint_format": "gptq_v2",
                                   "quant_method": "gptq"})
    assert (s.bits, s.group_size, s.desc_act, s.sym, s.format, s.method) == (4, 64, True, False, "gptq_v2", "gptq")
    a = loader.parse_quant_config({"w_bit": 4, "q_group_size": 128, "zero_point": True, "version": "GEMM", "quant_method": "awq"})
    assert (a.bits, a.group_size, a.sym, a.format, a.method) == (4, 128, False, "gemm", "awq")
    assert loader.parse_quant_config({"bits": 8}).format == "gptq"           # default: v1 zero-points
    with pytest.raises(NotImplementedError):
        loader.parse_quant_config({"bits": 4, "quant_method": "gguf"})
    with pytest.raises(NotImplementedError):
        loader.parse_quant_config({"bits": 4, "quant_method": "awq", "version": "gemv"})
    with pytest.raises(ValueError):
        loader.parse_quant_config({"bits": 4, "is_marlin_format": True})
    with pytest.raises(NotImplementedError):
        loader.parse_quant_config({"bits": 4, "pack_dtype": "int16"})
    assert loader.parse_quant_config({"bits": 4, "pack_dtype": "torch.int32"}).bits == 4


def test_dynamic_overrides_first_match_wins():
    s = loader.parse_quant_config({"bits": 4, "group_size": 128, "dynamic": {
        r"-:.*\.mlp\.gate_proj$": {},
        r".*\.up_proj.*": {"bits": 8, "group_size": 32},
        r"+:.*layers\.1\..*": {"group_size": 64, "desc_act": True},
        r".*": {"group_size": -1},
    }})
    assert s.for_module("model.layers.0.mlp.gate_proj") is None
    up = s.for_module("model.layers.1.mlp.up_proj")
    assert (up.bits, up.group_size) == (8, 32)                                # earlier pattern beats the layers.1 one
    q1 = s.for_module("model.layers.1.self_attn.q_proj")
    assert (q1.bits, q1.group_size, q1.desc_act) == (4, 64, True)
    assert s.for_module("model.layers.0.self_attn.q_proj").group_size == -1
    assert loader.parse_quant_config({"bits": 4}).for_module("x").bits == 4


@pytest.mark.parametrize("cfg_file", ["quantize_config.json", "quant_config.json", "config.json"])
def test_load_v2_checkpoint_roundtrip(tmp_path, cfg_file):
    layers = {
        "model.layers.0.self_attn.q_proj": make_layer(256, 128, group_size=128, sym=True, seed=1),
        "model.layers.0.mlp.down_proj": make_layer(256, 64, group_size=64, sym=False, bias=True, seed=2),
        "model.layers.0.mlp.up_proj": make_layer(128, 64, bits=8, group_size=32, sym=False, seed=3),
        "model.layers.0.self_attn.o_proj": make_layer(256, 64, group_size=64, sym=False, desc_act=True, seed=4),
    }
    cfg = {"bits": 4, "group_size": 128, "sym": True, "desc_act": False, "checkpoint_format": "gptq_v2", "quant_method": "gptq",
           "dynamic": {r".*down_proj": {"group_size": 64, "sym": False}, r".*up_proj": {"bits": 8, "group_size": 32},
                       r".*o_proj": {"group_size": 64, "sym": False, "desc_act": True}}}
    _write(str(tmp_path), {n: _ckpt_tensors(L) for n, L in layers.items()}, cfg, cfg_file, shards=2)
    mods = loader.load_quantized_linears(str(tmp_path), device="cpu")
    assert set(mods) == set(layers)
    for n, L in layers.items():
        m = mods[n]
        assert (m.bits, m.in_features, m.out_features) == (L["bits"], L["K"], L["N"])
        assert m.qzero_format() == 2 and m.name == n
        W = oracle.dequantize_weight(m.qweight, m.qzeros, m.scales, m.g_idx, m.bits)
        assert torch.equal(W, oracle.dequantize_weight(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], L["bits"]))
        assert (m.bias is None) == (L["bias"] is None)
    only = loader.load_quantized_linears(str(tmp_path), device="cpu", only=["model.layers.0.mlp.up_proj"])
    assert list(only) == ["model.layers.0.mlp.up_proj"] and only["model.layers.0.mlp.up_proj"].bits == 8


def test_load_v1_checkpoint_adds_zero_offset(tmp_path):
    L = make_layer(256, 128, group_size=128, sym=True, seed=7)
    v1 = _ckpt_tensors(L)
    v1["qzeros"] = oracle.convert_v2_to_v1(L["qzeros"], 4)
    assert not torch.equal(v1["qzeros"], L["qzeros"])
    _write(str(tmp_path), {"m.q_proj": v1}, {"bits": 4, "group_size": 128, "sym": True})   # no format key: v1
    m = loader.load_quantized_linears(str(tmp_path), device="cpu")["m.q_proj"]
    assert m.qzero_format() == 2 and torch.equal(m.qzeros.data, L["qzeros"])                # utils/model.py:810-818


def test_asymmetric_v1_needs_a_trusted_quantizer(tmp_path):
    L = make_layer(256, 64, group_size=64, sym=False, seed=8)
    v1 = _ckpt_tensors(L)
    v1["qzeros"] = oracle.convert_v2_to_v1(L["qzeros"], 4)
    d1, d2 = tmp_path / "a", tmp_path / "b"
    d1.mkdir(), d2.mkdir()
    _write(str(d1), {"m.k_proj": v1}, {"bits": 4, "group_size": 64, "sym": False, "checkpoint_format": "gptq"})
    with pytest.raises(ValueError):
        loader.load_quantized_linears(str(d1), device="cpu")                                # models/loader.py:1659-1663
    _write(str(d2), {"m.k_proj": v1}, {"bits": 4, "group_size": 64, "sym": False, "checkpoint_format": "gptq",
                                       "meta": {"quantizer": ["gptqmodel:1.4.2"]}})
    m = loader.load_quantized_linears(str(d2), device="cpu")["m.k_proj"]
    W = oracle.dequantize_weight(m.qweight, m.qzeros, m.scales, m.g_idx, 4)
    assert torch.equal(W, oracle.dequantize_weight(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4))


def test_load_awq_checkpoint(tmp_path):
    gen = torch.Generator().manual_seed(11)
    K, N, gs = 256, 128, 64
    codes = torch.randint(0, 16, (K, N), generator=gen)
    zeros = torch.randint(0, 16, (K // gs, N), generator=gen)
    sc = (torch.rand(K // gs, N, generator=gen) * 0.01 + 0.002).to(torch.float16)
    t = {"qweight": oracle.awq_pack(codes), "qzeros": oracle.awq_pack(zeros), "scales": sc}
    _write(str(tmp_path), {"model.layers.3.mlp.gate_proj": t},
           {"w_bit": 4, "q_group_size": gs, "zero_point": True, "version": "gemm", "quant_method": "awq"}, "config.json")
    m = loader.load_quantized_linears(str(tmp_path), device="cpu")["model.layers.3.mlp.gate_proj"]
    assert type(m).__name__ == "B200AwqQuantLinear" and (m.in_features, m.out_features, m.group_size) == (K, N, gs)
    assert torch.equal(m.qweight.data, t["qweight"])        # AWQ layout until post_init() converts on the device
    with pytest.raises(FileNotFoundError):
        loader.read_quant_config(str(tmp_path / "missing"))


def test_load_lowbit_and_planar_checkpoints(tmp_path):
    """3-bit v1 file (zero-points straddle words: shifted in logical space, utils/model_dequant.py:900-907) and a planar
    5-bit gptq_p file (v2 zero-points on disk, quantization/config.py:112-114) built from reference-packed tensors."""
    import numpy as np
    from gptqmodel_b200 import layouts

    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "lowbit_cases.npz"))
    t = lambda n, k: torch.from_numpy(d[f"{n}.{k}"])  # noqa: E731
    v2 = {k: t("w3_g128_sym", k) for k in ("qweight", "qzeros", "scales", "g_idx")}
    v1 = dict(v2, qzeros=layouts.shift_zero_points(v2["qzeros"], 3, False, -1))
    assert not torch.equal(v1["qzeros"], v2["qzeros"])
    p3 = tmp_path / "w3"
    p3.mkdir()
    _write(str(p3), {"m.o_proj": v1}, {"bits": 3, "group_size": 128, "sym": True})
    m = loader.load_quantized_linears(str(p3), device="cpu")["m.o_proj"]
    assert m.bits == 3 and m.kbits == 4 and not m.planar and m.qzero_format() == 2
    assert torch.equal(m.qzeros.data, v2["qzeros"]) and m.qweight.shape == (256 * 3 // 32, 64)
    p5 = tmp_path / "w5"
    p5.mkdir()
    c5 = {k: t("w5_g64_asym", k) for k in ("qweight", "qzeros", "scales", "g_idx", "bias")}
    _write(str(p5), {"m.o_proj": c5}, {"bits": 5, "group_size": 64, "sym": False, "checkpoint_format": "gptq_p"})
    m = loader.load_quantized_linears(str(p5), device="cpu")["m.o_proj"]
    assert m.bits == 5 and m.kbits == 8 and m.planar and torch.equal(m.qzeros.data, c5["qzeros"])
    assert m.in_features == 128 and m.out_features == 64 and m.bias is not None
