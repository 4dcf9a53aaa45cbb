"""CPU: rotated (QuaRot / SpinQuant) checkpoints — the float64 oracle and the order rule against the reference's own
results (tests/golden/hadamard_cases.npz, make_golden_hadamard.py), had_K validation, b2q_hadamard's argument checks,
the loader's rotation handling and sibling fusion."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
from safetensors.torch import save_file

import gptqmodel_b200 as g
from gptqmodel_b200 import B200QuantLinear, fuse_siblings, loader, tp
from helpers import make_layer
from oracle.hadamard_oracle import hadamard_transform

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hadamard_cases.npz")
ORDERS = (12, 20, 28, 36, 40, 52, 60, 108, 140, 156, 172)


@pytest.fixture(scope="module")
def cases():
    return np.load(GOLDEN)


def test_oracle_matches_reference_matmul_hadU(cases):
    meta = json.loads(bytes(cases["__meta__"]).decode())
    assert len(meta["cases"]) >= 5
    for i, (K, n) in enumerate(meta["cases"]):
        x = torch.from_numpy(cases[f"case{i}.x"])
        # matmul_hadU divides by torch.tensor(n).sqrt(), a float32 value: undo that one rounding
        y = cases[f"case{i}.y"] * (float(np.sqrt(np.float32(n))) / np.sqrt(n))
        had = None if K == 1 else torch.from_numpy(cases[f"had{K}"])
        got = hadamard_transform(x, had, K).numpy()
        assert np.abs(got - y).max() <= 1e-12 * max(1.0, np.abs(y).max()), (K, n)


def test_order_rule_matches_reference_get_hadK(cases):
    for n, k in zip(cases["hadK.n"].tolist(), cases["hadK.K"].tolist()):
        if k < 0:
            with pytest.raises(ValueError):
                loader.hadamard_order(n)
        else:
            assert loader.hadamard_order(n) == k, n


def _module(K_in, N=64):
    return B200QuantLinear(bits=4, group_size=-1, desc_act=False, sym=True, in_features=K_in, out_features=N)


def test_set_had_K_accepts_reference_matrices_and_rejects_others(cases):
    for K in ORDERS:
        h = torch.from_numpy(cases[f"had{K}"]).to(torch.float32)
        m = _module(K * 64)
        m.online_full_had, m.K = True, K
        m.set_had_K(h)
        assert m.had_K is h and "had_K" in m._buffers and not m._buffers.get("had_K") is None
        assert m._had_dev is None  # the device copy is made by post_init()
        m.set_had_K(None)
        assert m.had_K is None
    h28 = torch.from_numpy(cases["had28"]).to(torch.float32)
    m = _module(28 * 64)
    m.online_full_had, m.K = True, 28
    bad = h28.clone()
    bad[3, 5] = 0.5
    with pytest.raises(ValueError, match="other than"):
        m.set_had_K(bad)
    bad = h28.clone()
    bad[3, 5] = -bad[3, 5]
    with pytest.raises(ValueError, match="not a Hadamard"):
        m.set_had_K(bad)
    with pytest.raises(ValueError, match="does not fit"):
        _module(4096).set_had_K(h28)  # 4096 is not 28 * 2^m
    assert m.had_K is None


def test_hadamard_abi_argument_validation_without_gpu():
    one = ctypes.c_void_p(16)
    two = ctypes.c_void_p(1 << 20)
    call = g.lib.b2q_hadamard
    assert call(one, one, 28, two, 1, 28 * 12, 0, None) == -2        # P = 12 is not a power of two
    assert b"power of two" in g.lib.b2q_last_error()
    assert call(one, one, 28, two, 1, 28 * 4, 0, None) == -2         # P = 4 < 8
    assert b"power of two" in g.lib.b2q_last_error()
    assert call(one, one, 257, two, 1, 257 * 8, 0, None) == -2       # K > 256
    assert b"K=257" in g.lib.b2q_last_error()
    assert call(one, None, 1, two, 1, 131072, 0, None) == -2         # n > 65536
    assert b"n=131072" in g.lib.b2q_last_error()
    assert call(one, None, 28, two, 1, 28 * 64, 0, None) == -2       # NULL had with K > 1
    assert b"NULL exactly when" in g.lib.b2q_last_error()
    assert call(one, one, 1, two, 1, 512, 0, None) == -2             # had given for K == 1
    assert b"NULL exactly when" in g.lib.b2q_last_error()
    assert call(one, one, 28, one, 1, 28 * 64, 0, None) == -2        # out == x
    assert b"overlap" in g.lib.b2q_last_error()
    assert call(one, one, 28, ctypes.c_void_p(16 + 64), 1, 28 * 64, 0, None) == -2  # out overlaps x
    assert b"overlap" in g.lib.b2q_last_error()
    assert call(one, one, 28, two, 1, 28 * 64, 2, None) == -2        # dtype
    assert b"dtype=2" in g.lib.b2q_last_error()
    assert call(ctypes.c_void_p(24), one, 28, two, 1, 28 * 64, 0, None) == -2  # misaligned
    assert b"aligned" in g.lib.b2q_last_error()
    assert call(one, one, 28, two, -1, 28 * 64, 0, None) == -2
    assert call(one, one, 28, two, 0, 28 * 64, 0, None) == 0         # rows == 0: no-op


def _write_ckpt(tmp, names, K_of, cfg):
    blob = {}
    for i, name in enumerate(names):
        L = make_layer(K_of(name), 64, bits=4, group_size=64, seed=i)
        for k in ("qweight", "qzeros", "scales", "g_idx"):
            blob[f"{name}.{k}"] = L[k].contiguous()
    save_file(blob, os.path.join(tmp, "model.safetensors"))
    json.dump(cfg, open(os.path.join(tmp, "quantize_config.json"), "w"))


NAMES = ("model.layers.0.mlp.down_proj", "model.layers.0.mlp.up_proj", "model.layers.0.self_attn.o_proj",
         "model.layers.1.mlp.down_proj", "model.layers.1.mlp.experts.0.down_proj")


def test_loader_rotation_flags_only_down_proj(tmp_path, cases):
    K_of = lambda n: 28 * 64 if n.endswith("mlp.down_proj") else 256  # noqa: E731
    _write_ckpt(str(tmp_path), NAMES, K_of, {"bits": 4, "group_size": 64, "format": "gptq_v2", "rotation": "hadamard"})
    h28 = torch.from_numpy(cases["had28"]).to(torch.float32)
    for tables in ({28: h28}, lambda n: (h28, 28) if n % 28 == 0 else (None, 1)):
        mods = loader.load_quantized_linears(str(tmp_path), device="cpu", hadamard=tables)
        for name, m in mods.items():
            rotated = name.endswith("mlp.down_proj")
            assert m.online_full_had == rotated and not m.online_partial_had, name
            assert m.K == (28 if rotated else 1)
            assert (m.had_K is not None) == rotated
            if rotated:
                assert torch.equal(m.had_K.float(), h28)
    assert loader.read_quant_config(str(tmp_path)).rotation == "hadamard"
    with pytest.raises(NotImplementedError, match="order 28"):
        loader.load_quantized_linears(str(tmp_path), device="cpu")
    with pytest.raises(NotImplementedError, match="order 28"):
        loader.load_quantized_linears(str(tmp_path), device="cpu", hadamard={172: h28})


def test_loader_rotation_power_of_two_needs_no_table(tmp_path):
    _write_ckpt(str(tmp_path), NAMES[:3], lambda n: 512, {"bits": 4, "group_size": 64, "rotation": "random"})
    mods = loader.load_quantized_linears(str(tmp_path), device="cpu")
    m = mods["model.layers.0.mlp.down_proj"]
    assert m.online_full_had and m.K == 1 and m.had_K is None
    assert not mods["model.layers.0.mlp.up_proj"].online_full_had


def test_loader_rotation_config_checks():
    assert loader.parse_quant_config({"bits": 4}).rotation is None
    assert loader.parse_quant_config({"bits": 4, "format": "gptq_v2", "rotation": "hadamard"}).rotation == "hadamard"
    with pytest.raises(ValueError, match="rotation"):
        loader.parse_quant_config({"bits": 4, "rotation": "givens"})
    with pytest.raises(NotImplementedError, match="rotation"):
        loader.parse_quant_config({"bits": 4, "quant_method": "awq", "version": "gemm", "rotation": "hadamard"})
    with pytest.raises(NotImplementedError, match="rotation"):
        loader.parse_quant_config({"bits": 3, "format": "gptq_p", "rotation": "hadamard"})


def _fake_prepacked(K_in):
    m = _module(K_in)
    m._prepacked, m.packed, m._is_sym = True, torch.empty(16, dtype=torch.uint8), True
    return m


def test_fuse_siblings_and_row_parallel_refuse_rotated_modules():
    a, b = _fake_prepacked(512), _fake_prepacked(512)
    assert fuse_siblings([a, b])  # control: the same pair without rotation shares a launch
    a, b = _fake_prepacked(512), _fake_prepacked(512)
    b.online_full_had = True
    assert not fuse_siblings([a, b]) and a._siblings is None and b._siblings is None
    with pytest.raises(NotImplementedError, match="row-sharded"):
        tp.RowParallelLinear(b)
    c = _fake_prepacked(512)
    c.online_partial_had, c.had_dim = True, 128
    with pytest.raises(NotImplementedError, match="row-sharded"):
        tp.RowParallelLinear(c)
