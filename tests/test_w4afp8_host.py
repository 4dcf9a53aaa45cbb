"""W4AFP8 on the host: the config parser's accept / refuse matrix, the checkpoint packing against compressed-tensors'
fixture, the numpy mirror of the kernel's tile layout, the ABI's argument checks and the MoE refusal."""
import copy
import json
import os

import numpy as np
import pytest
import torch

import w4afp8_mirror as wm
from gptqmodel_b200 import B200W4Fp8Linear, lib
from gptqmodel_b200.loader import load_w4afp8_linears, parse_fp8_w8a8_config, parse_int8_w8a8_config, \
    parse_w4afp8_config
from gptqmodel_b200.w4afp8 import tile_codes, unpack_codes

FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "w4afp8_cases.npz")
GOOD = {"quant_method": "compressed-tensors", "format": "pack-quantized", "ignore": ["lm_head", "re:.*gate$"],
        "kv_cache_scheme": {"num_bits": 8, "type": "float", "strategy": "tensor"},
        "config_groups": {"group_0": {"targets": ["Linear"],
                                      "weights": {"num_bits": 4, "type": "int", "symmetric": True, "strategy": "group",
                                                  "group_size": 128, "dynamic": False, "actorder": None},
                                      "input_activations": {"num_bits": 8, "type": "float", "symmetric": True,
                                                            "strategy": "token", "dynamic": True}}}}


def _cfg(**edits):
    """GOOD with edits: key "w.<k>" / "a.<k>" sets a weights / input_activations entry, other keys the group's."""
    c = copy.deepcopy(GOOD)
    g = c["config_groups"]["group_0"]
    for k, v in edits.items():
        if k.startswith("w."):
            g["weights"][k[2:]] = v
        elif k.startswith("a."):
            g["input_activations"][k[2:]] = v
        elif k == "top":
            c.update(v)
        else:
            g[k] = v
    return c


def test_parser_accepts():
    spec = parse_w4afp8_config(GOOD)
    assert spec.ignore == ("lm_head", "re:.*gate$") and spec.kv_cache_scheme == GOOD["kv_cache_scheme"]
    assert spec.ignores("lm_head") and spec.ignores("model.layers.0.mlp.gate") and not spec.ignores("x.q_proj")
    assert parse_w4afp8_config(_cfg(**{"w.actorder": "weight"})).ignore
    two = copy.deepcopy(GOOD)
    two["config_groups"]["group_1"] = copy.deepcopy(two["config_groups"]["group_0"])
    parse_w4afp8_config(two)


@pytest.mark.parametrize("edits", [
    {"w.group_size": 64}, {"w.group_size": 32}, {"w.strategy": "channel"}, {"w.strategy": "tensor"},
    {"w.num_bits": 8}, {"w.num_bits": 2}, {"w.symmetric": False}, {"w.actorder": "group"}, {"w.type": "float"},
    {"a.dynamic": False, "a.strategy": "tensor"}, {"a.strategy": "tensor"}, {"a.dynamic": False},
    {"a.type": "int"}, {"a.num_bits": 4}, {"output_activations": {"num_bits": 8}}, {"targets": ["Attention"]},
    {"input_activations": None}, {"top": {"format": "int-quantized"}}, {"top": {"quant_method": "gptq"}},
])
def test_parser_refuses_what_is_not_served(edits):
    with pytest.raises(NotImplementedError):
        parse_w4afp8_config(_cfg(**edits))


def test_parser_refuses_mixed_groups():
    mixed = copy.deepcopy(GOOD)
    g1 = copy.deepcopy(mixed["config_groups"]["group_0"])
    g1["weights"]["group_size"] = 64
    mixed["config_groups"]["group_1"] = g1
    with pytest.raises(NotImplementedError):
        parse_w4afp8_config(mixed)


@pytest.mark.parametrize("edits", [
    {"w.group_size": "128"}, {"w.group_size": None}, {"w.actorder": 1}, {"w.num_bits": "4"}, {"w.symmetric": "yes"},
    {"a.dynamic": "always"}, {"weights": "int4"}, {"targets": "Linear"}, {"top": {"ignore": "lm_head"}},
    {"top": {"ignore": ["re:("]}}, {"top": {"config_groups": {}}}, {"top": {"kv_cache_scheme": 8}},
])
def test_parser_rejects_malformed(edits):
    with pytest.raises(ValueError):
        parse_w4afp8_config(_cfg(**edits))
    with pytest.raises(ValueError):
        parse_w4afp8_config([GOOD])


def test_w8a8_parsers_still_refuse_pack_quantized():
    for parse in (parse_fp8_w8a8_config, parse_int8_w8a8_config):
        with pytest.raises(NotImplementedError, match="pack-quantized"):
            parse(GOOD)


def _fix():
    return np.load(FIX)


def test_unpack_equals_compressed_tensors():
    from compressed_tensors.compressors.pack_quantized.base import unpack_from_int32

    z = _fix()
    names = sorted({k.split(".")[0] for k in z.files})
    assert len(names) == 4
    for n in names:
        wp = z[f"{n}.weight_packed"]
        shape = torch.Size(z[f"{n}.weight_shape"].tolist())
        want = unpack_from_int32(torch.from_numpy(wp), 4, shape).numpy().astype(np.int32)
        assert np.array_equal(wm.unpack(wp).astype(np.int32) - 8, want), n
        assert np.array_equal(unpack_codes(torch.from_numpy(wp)).numpy().astype(np.int32) - 8, want), n
        assert np.array_equal(wm.pack(wm.unpack(wp)), wp), n


def test_prepack_layout_round_trips():
    rng = np.random.default_rng(0)
    for K, N in ((128, 128), (512, 256), (1024, 384)):
        c = rng.integers(0, 16, size=(N, K)).astype(np.uint8)
        tiles = wm.prepack(wm.pack(c))
        assert tiles.shape == (N // 128, K // 128, 4, 128, 4) and tiles.nbytes == lib.b2q_w4afp8_packed_bytes(K, N)
        assert np.array_equal(wm.unprepack(tiles, K, N), c)
        assert np.array_equal(tile_codes(torch.from_numpy(tiles.reshape(-1).view(np.uint8).copy()), K, N).numpy(), c)
        # word (nt, kb, quad, f, j), nibble p is k = 128 kb + 32 quad + 8 j + NIBBLE_K[p] of feature 128 nt + f
        nt, kb, quad, f, j = N // 128 - 1, K // 128 - 1, 2, 77, 3
        w = int(tiles[nt, kb, quad, f, j])
        for p in range(8):
            assert (w >> (4 * p)) & 15 == c[128 * nt + f, 128 * kb + 32 * quad + 8 * j + wm.NIBBLE_K[p]]


def test_dequantize_weight_on_host_equals_fixture():
    z = _fix()
    for n in sorted({k.split(".")[0] for k in z.files}):
        dtype = torch.bfloat16 if n.startswith("bf") else torch.float16
        ws = z[f"{n}.weight_scale"]
        ws = torch.from_numpy(ws.view(np.int16)).view(torch.bfloat16) if ws.dtype == np.uint16 else torch.from_numpy(ws)
        table = z[f"{n}.dq_table"]
        W = wm.table_weight(table, wm.unpack(z[f"{n}.weight_packed"]))
        W = torch.from_numpy(W.view(np.int16)).view(torch.bfloat16) if W.dtype == np.uint16 else torch.from_numpy(W)
        m = B200W4Fp8Linear.from_checkpoint_tensors(torch.from_numpy(z[f"{n}.weight_packed"]), ws,
                                                    weight_shape=torch.from_numpy(z[f"{n}.weight_shape"]),
                                                    device="cpu", post_init=False)
        assert torch.equal(m.dequantize_weight(dtype=dtype), W), n


def test_module_refuses_bad_tensors():
    wp, ws = torch.zeros(256, 64, dtype=torch.int32), torch.ones(256, 4, dtype=torch.bfloat16)
    mk = B200W4Fp8Linear.from_checkpoint_tensors
    with pytest.raises(NotImplementedError):  # K = 520 is outside the envelope
        mk(torch.zeros(256, 65, dtype=torch.int32), ws, device="cpu", post_init=False)
    with pytest.raises(NotImplementedError):  # N % 128 != 0
        mk(torch.zeros(192, 64, dtype=torch.int32), torch.ones(192, 4), device="cpu", post_init=False)
    with pytest.raises(ValueError):
        mk(wp, torch.ones(256, 2), device="cpu", post_init=False)
    with pytest.raises(ValueError):
        mk(wp.to(torch.int64), ws, device="cpu", post_init=False)
    with pytest.raises(ValueError):
        mk(wp, ws * float("nan"), device="cpu", post_init=False)
    with pytest.raises(ValueError):
        mk(wp, ws, weight_shape=torch.tensor([256, 1024]), device="cpu", post_init=False)
    with pytest.raises(NotImplementedError):
        B200W4Fp8Linear.validate_device("cpu")


def test_abi_argument_checks_without_gpu():
    P = 1 << 20  # any 16-byte aligned non-NULL value: a refused call never dereferences it
    assert lib.b2q_w4afp8_packed_bytes(4096, 1024) == 4096 * 1024 // 2
    assert lib.b2q_w4afp8_packed_bytes(100, 128) == 0 and lib.b2q_w4afp8_packed_bytes(128, 64) == 0
    assert lib.b2q_w4afp8_workspace_bytes(9, 4096) == lib.b2q_fp8ch_workspace_bytes(9, 4096) == 9 * 4096 + 48
    good = dict(x=P, p=P, s=P, bias=None, out=P, M=16, K=256, N=128, dt=0, ws=P, nws=1 << 30)

    def fwd(**kw):
        a = {**good, **kw}
        return lib.b2q_w4afp8_forward(a["x"], a["p"], a["s"], a["bias"], a["out"], a["M"], a["K"], a["N"], a["dt"],
                                      a["ws"], a["nws"], None)

    bad = (dict(p=None), dict(s=None), dict(out=None), dict(x=None), dict(dt=2), dict(M=-1), dict(K=64), dict(K=0),
           dict(K=65536 + 128), dict(N=64), dict(N=192), dict(N=0), dict(x=P + 8), dict(out=P + 2), dict(p=P + 4),
           dict(s=P + 4), dict(ws=None), dict(ws=P + 8), dict(nws=16 * 256), dict(M=1, ws=None))
    for kw in bad:
        assert fwd(**kw) == -2, kw
        assert lib.b2q_last_error()
    assert fwd(M=0) == 0 and fwd(M=0, x=None, ws=None) == 0  # an empty batch is a no-op

    def mm(**kw):
        a = {**good, "codes": P, "sx": P, "ks": 0, **kw}
        return lib.b2q_w4afp8_mm(a["codes"], a["sx"], a["p"], a["s"], a["bias"], a["out"], a["M"], a["K"], a["N"],
                                 a["dt"], a["ks"], None)

    for kw in (dict(codes=None), dict(sx=None), dict(codes=P + 4), dict(ks=9), dict(p=None), dict(K=192), dict(N=96),
               dict(dt=5), dict(K=65536 * 2)):
        assert mm(**kw) == -2, kw
        assert lib.b2q_last_error()
    assert mm(M=0) == 0

    def prepack(src=P, dst=P, K=256, N=128):
        return lib.b2q_w4afp8_prepack(src, dst, K, N, None)

    for kw in (dict(src=None), dict(dst=None), dict(dst=P + 8), dict(K=100), dict(N=64), dict(K=65536 + 128)):
        assert prepack(**kw) == -2, kw


def test_moe_grouped_refusal_names_the_reason():
    from gptqmodel_b200 import moe

    def mod(K, N):
        return B200W4Fp8Linear.from_checkpoint_tensors(torch.zeros(N, K // 8, dtype=torch.int32),
                                                       torch.ones(N, K // 128, dtype=torch.bfloat16), device="cpu",
                                                       post_init=False)

    w1, w3, w2 = [mod(256, 128)], [mod(256, 128)], [mod(128, 256)]
    assert moe.MoEExperts(w1, w3, w2)._stack is None  # the per-expert loop
    with pytest.raises(ValueError, match=r"grouped=True\): W4AFP8 experts \(B200W4Fp8Linear\) have no grouped kernels"):
        moe.MoEExperts(w1, w3, w2, grouped=True)


def _checkpoint(tmp_path, tensors, cfg=GOOD):
    from safetensors.torch import save_file

    with open(tmp_path / "config.json", "w") as f:
        json.dump({"model_type": "llama", "quantization_config": cfg}, f)
    save_file(tensors, str(tmp_path / "model.safetensors"))
    return str(tmp_path)


def test_loader_on_host(tmp_path):
    z = _fix()
    n = "bf_1024_128_48"
    wp = torch.from_numpy(z[f"{n}.weight_packed"])
    ws = torch.from_numpy(z[f"{n}.weight_scale"].view(np.int16)).view(torch.bfloat16)
    t = {"model.layers.0.self_attn.q_proj.weight_packed": wp, "model.layers.0.self_attn.q_proj.weight_scale": ws,
         "model.layers.0.mlp.gate.weight_packed": wp.clone(), "model.layers.0.mlp.gate.weight_scale": ws.clone(),
         "lm_head.weight": torch.zeros(128, 1024, dtype=torch.bfloat16)}
    path = _checkpoint(tmp_path, t)
    mods = load_w4afp8_linears(path, device="cpu")
    assert sorted(mods) == ["model.layers.0.self_attn.q_proj"]  # the gate is ignored by its pattern
    m = mods["model.layers.0.self_attn.q_proj"]
    assert m.in_features == 1024 and m.out_features == 128 and not m._ready
    assert torch.equal(m.weight_packed, wp) and torch.equal(m.weight_scale, ws)


@pytest.mark.parametrize("extra", ["zero_point", "g_idx"])
def test_loader_refuses_asymmetric_and_act_order(tmp_path, extra):
    K, N = 256, 128
    p = "model.layers.0.self_attn.q_proj"
    t = {f"{p}.weight_packed": torch.zeros(N, K // 8, dtype=torch.int32),
         f"{p}.weight_scale": torch.ones(N, K // 128, dtype=torch.bfloat16)}
    if extra == "zero_point":
        t[f"{p}.weight_zero_point"] = torch.zeros(N, K // 128, dtype=torch.int8)
        load_w4afp8_linears(_checkpoint(tmp_path, t), device="cpu")  # all zeros: symmetric
        t[f"{p}.weight_zero_point"][3, 1] = 2
    else:
        t[f"{p}.weight_g_idx"] = torch.arange(K, dtype=torch.int32) // 128
        load_w4afp8_linears(_checkpoint(tmp_path, t), device="cpu")  # contiguous groups
        t[f"{p}.weight_g_idx"] = torch.arange(K, dtype=torch.int32).flip(0) // 128
    with pytest.raises(NotImplementedError):
        load_w4afp8_linears(_checkpoint(tmp_path, t), device="cpu")
