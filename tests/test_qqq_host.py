"""CPU: QQQ (W4A8) checkpoints — un-permutation, oracle, loader and validation (no GPU needed).

The fixtures (tests/golden/qqq_cases.npz) come from the reference's own QQQTorchLinear (make_golden_qqq.py)."""
import json
import os

import numpy as np
import pytest
import torch
from safetensors.torch import save_file

import gptqmodel_b200 as g
from gptqmodel_b200 import B200QqqQuantLinear, loader
from gptqmodel_b200.qqq import unpermute_qqq
from oracle import qqq_oracle as qo

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, "golden", "qqq_cases.npz"))
CASES = sorted({k.split(".")[0] for k in GOLD.files})


def _case(c):
    t = lambda k: torch.from_numpy(GOLD[f"{c}.{k}"].copy())  # noqa: E731
    gs = -1 if GOLD[f"{c}.s_group"].size == 0 else 128
    return t, gs


def _x(t, tag):
    x = t("x" + tag)
    return x if tag == "16" else x.to(torch.bfloat16)


@pytest.mark.parametrize("c", CASES)
def test_unpermute_matches_reference_dequantize(c):
    t, gs = _case(c)
    codes, sc, sg = unpermute_qqq(t("B"), t("s_channel"), t("s_group") if gs == 128 else None, gs)
    assert torch.equal(codes, t("codes"))
    w = qo.weight_int8(codes, sg)
    assert torch.equal(w.to(torch.float32), t("weight").to(torch.float32))
    assert torch.equal(sc, t("weight_s_channel").reshape(-1))
    if gs == 128:
        assert torch.equal(sg, t("s_grp_canon"))
    # the oracle's independent statement of the format agrees
    c2, sc2, sg2 = qo.unpack_qqq(t("B"), t("s_channel"), t("s_group"))
    assert torch.equal(c2, codes) and torch.equal(sc2, sc)
    assert (sg2 is None) == (sg is None) and (sg is None or torch.equal(sg2, sg))


@pytest.mark.parametrize("gs", [-1, 128])
@pytest.mark.parametrize("KN", [(256, 128), (192, 256), (1024, 64)])
def test_pack_unpack_identity(gs, KN):
    K, N = KN
    if gs == 128 and K % 128:
        pytest.skip("group 128 needs K % 128 == 0")
    gen = torch.Generator().manual_seed(K * 7 + N + gs)
    codes = torch.randint(0, 16, (K, N), generator=gen).to(torch.uint8)
    sc = torch.rand(N, generator=gen) + 0.01
    sg = (torch.rand(K // 128, N, generator=gen) * 15 + 1).to(torch.float16) if gs == 128 else None
    B, sc_p, sg_p = qo.pack_qqq(codes, sc, sg)
    assert B.shape == (K // 16, 2 * N) and B.dtype == torch.int32
    c2, sc2, sg2 = qo.unpack_qqq(B, sc_p, sg_p)
    assert torch.equal(c2, codes) and torch.equal(sc2, sc)
    c3, sc3, sg3 = unpermute_qqq(B, sc_p, sg_p if gs == 128 else None, gs)
    assert torch.equal(c3, codes) and torch.equal(sc3, sc)
    if gs == 128:
        assert torch.equal(sg2, sg) and torch.equal(sg3, sg)


@pytest.mark.parametrize("c", CASES)
@pytest.mark.parametrize("tag", ["16", "bf"])
def test_oracle_dynamic_quant_bit_exact(c, tag):
    t, _ = _case(c)
    q, s = qo.quantize(_x(t, tag))
    assert torch.equal(q, t("q" + tag))
    assert torch.equal(s, t("s" + tag))
    zero = int((t("x" + tag).abs().amax(-1) == 0).nonzero()[0])
    assert s[zero] == 0 and not q[zero].any()


@pytest.mark.parametrize("c", CASES)
@pytest.mark.parametrize("tag", ["16", "bf"])
def test_oracle_forward_within_one_ulp_of_reference(c, tag):
    t, gs = _case(c)
    codes, sc, sg = unpermute_qqq(t("B"), t("s_channel"), t("s_group") if gs == 128 else None, gs)
    bias = t("bias") if t("bias").numel() else None
    x = _x(t, tag)
    y = qo.forward(x, codes, sc, sg, bias)
    ref = t("y" + tag).to(x.dtype)
    assert y.dtype == x.dtype and y.shape == ref.shape
    # the reference's torch path multiplies s_tok before s_channel: at most 1 fp16 ulp apart (then the cast)
    y16, r16 = y.to(torch.float16), ref.to(torch.float16)
    ulp = (r16.to(torch.float32).abs().clamp_min(2.0 ** -14).log2().floor() - 10).exp2()
    assert bool(((y16.to(torch.float32) - r16.to(torch.float32)).abs() <= ulp * (2 if tag == "bf" else 1)).all())
    assert (y16 == r16).float().mean() > 0.95


def test_oracle_group_range_rejected():
    codes = torch.zeros(128, 64, dtype=torch.uint8)
    sg = torch.full((1, 64), 17.0, dtype=torch.float16)  # (0 - 8) * 17 = -136
    with pytest.raises(ValueError):
        qo.weight_int8(codes, sg)
    from gptqmodel_b200.qqq import check_group_range
    with pytest.raises(ValueError):
        check_group_range(codes, sg)
    check_group_range(codes, torch.full((1, 64), 16.0, dtype=torch.float16))  # -128 fits


def test_validate_envelope():
    ok = [(128, 64), (256, 192), (64, 128), (192, 384), (4096, 14336), (14336, 4096), (65536, 64)]
    bad = [(64, 64), (192, 64), (128, 32), (64, 192), (32, 128), (96, 128), (65664, 128), (0, 128), (128, 0)]
    for K, N in ok:
        assert B200QqqQuantLinear.validate(bits=4, group_size=-1, in_features=K, out_features=N)[0], (K, N)
    for K, N in bad:
        okv, err = B200QqqQuantLinear.validate(bits=4, group_size=-1, in_features=K, out_features=N)
        assert not okv and isinstance(err, NotImplementedError), (K, N)
    for kw in ({"bits": 8}, {"group_size": 64}, {"sym": False}, {"dtype": torch.float32},
               {"group_size": 128, "in_features": 64, "out_features": 128}):
        args = {"bits": 4, "group_size": -1, "in_features": 256, "out_features": 128, **kw}
        okv, err = B200QqqQuantLinear.validate(**args)
        assert not okv and isinstance(err, NotImplementedError), kw
    assert B200QqqQuantLinear.validate(bits=4, group_size=128, desc_act=True, in_features=256, out_features=128)[0]
    with pytest.raises(NotImplementedError):
        B200QqqQuantLinear(bits=4, group_size=-1, desc_act=False, sym=True, in_features=64, out_features=64)


def test_abi_entry_points_without_gpu():
    assert g.lib.b2q_qqq_packed_bytes(4096, 4096) == 4096 * 4096 // 2
    assert g.lib.b2q_qqq_packed_bytes(320, 192) == 384 * 256 // 2   # padded to 128 k and 128 features
    assert g.lib.b2q_qqq_workspace_bytes(3, 320) == 128 + 3 * 384
    assert g.lib.b2q_qqq_workspace_bytes(0, 4096) == 0
    # shapes outside the envelope are refused before any CUDA work
    for K, N, gs in ((64, 64, -1), (192, 64, -1), (320, 128, 128), (4096, 4096, 64), (65664, 128, -1)):
        assert g.lib.b2q_qqq_mm(None, None, 16, 16, None, None, 16, 1, K, N, gs, 0, None) == -2, (K, N, gs)
        assert g.lib.b2q_qqq_forward(16, 16, 16, None, None, 16, 1, K, N, gs, 0, 0, 16, 1 << 20, None) == -2
    assert g.lib.b2q_qqq_forward(16, 16, 16, 16, None, 16, 1, 256, 128, -1, 0, 0, 16, 1 << 20, None) == -2  # s_group
    assert g.lib.b2q_qqq_forward(16, 16, 16, None, None, 16, 1, 256, 128, -1, 2, 0, 16, 1 << 20, None) == -2  # dtype
    assert g.lib.b2q_qqq_forward(16, 16, 16, None, None, 16, 4, 256, 128, -1, 0, 0, 16, 64, None) == -2  # workspace
    assert b"workspace" in g.lib.b2q_last_error()
    assert g.lib.b2q_qqq_quantize(16, 16, 16, 1, 96, 0, None) == -2
    assert g.lib.b2q_qqq_prepack(16, 16, 256, 96, -1, None) == -2


def _write_qqq_ckpt(tmp, layers, cfg):
    blob = {}
    for name, L in layers.items():
        for k, v in L.items():
            if v is not None and v.numel():
                blob[f"{name}.{k}"] = v.contiguous()
    save_file(blob, os.path.join(tmp, "model.safetensors"))
    json.dump(cfg, open(os.path.join(tmp, "quantize_config.json"), "w"))


def test_loader_reads_qqq_checkpoint(tmp_path):
    layers, want = {}, {}
    for c, name in (("ch", "model.layers.0.self_attn.q_proj"), ("g128_bias", "model.layers.0.mlp.up_proj")):
        t, gs = _case(c)
        layers[name] = {"B": t("B"), "s_channel": t("s_channel"), "s_group": t("s_group"),
                        "bias": t("bias") if t("bias").numel() else None}
        want[name] = (t, gs)
    cfg = {"bits": 4, "group_size": 128, "sym": True, "desc_act": False, "quant_method": "qqq",
           "checkpoint_format": "qqq", "dynamic": {r".*q_proj": {"group_size": -1}}}
    _write_qqq_ckpt(str(tmp_path), layers, cfg)
    mods = loader.load_quantized_linears(str(tmp_path), device="cpu", post_init=False)
    assert sorted(mods) == sorted(layers)
    for name, m in mods.items():
        t, gs = want[name]
        assert isinstance(m, B200QqqQuantLinear)
        assert m.requested_group_size == gs
        assert (m.in_features, m.out_features) == (t("codes").shape[0], t("codes").shape[1])
        assert torch.equal(m.B, t("B")) and torch.equal(m.s_channel, t("s_channel"))
        assert (m.bias is None) == (t("bias").numel() == 0)
        codes, _, _ = unpermute_qqq(m.B, m.s_channel, m.s_group if gs == 128 else None, gs)
        assert torch.equal(codes, t("codes"))


def test_parse_qqq_config():
    s = loader.parse_quant_config({"bits": 4, "group_size": 128, "quant_method": "qqq", "checkpoint_format": "qqq",
                                   "desc_act": True})
    assert (s.method, s.format, s.bits, s.group_size, s.desc_act) == ("qqq", "qqq", 4, 128, True)
    assert loader.parse_quant_config({"bits": 4, "group_size": -1, "quant_method": "qqq"}).format == "qqq"
    for bad in ({"bits": 8}, {"group_size": 64}, {"sym": False}, {"checkpoint_format": "gptq"},
                {"rotation": "hadamard"}):
        with pytest.raises(NotImplementedError):
            loader.parse_quant_config({"bits": 4, "group_size": 128, "quant_method": "qqq", **bad})
