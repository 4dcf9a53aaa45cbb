"""Block-FP8 (HF / DeepSeek-native, W8A8) host side: config parsing and refusals, the oracle and the module's
dequantiser against the reference's fixtures, the numpy quantiser against a torch restatement, the loader on a synthetic
checkpoint, the ABI's argument checks and the compiler's report on the new kernels.  No GPU needed."""
import json
import os
import re

import numpy as np
import pytest
import torch

from gptqmodel_b200 import B200BlockFp8Linear, lib
from gptqmodel_b200.loader import load_block_fp8_linears, load_quantized_linears, parse_block_fp8_config, \
    parse_quant_config
from oracle import fp8_block_oracle as fo

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = np.load(os.path.join(HERE, "golden", "fp8_block_cases.npz"))
NAMES = sorted({k.split(".")[0] for k in CASES.files})
HF = {"quant_method": "fp8", "fmt": "e4m3", "activation_scheme": "dynamic", "weight_block_size": [128, 128]}


# ---- config parsing ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("raw", [
    HF,
    {"quant_method": "fp8", "weight_block_size": [128, 128]},
    {"quant_method": "fp8", "fmt": "float8_e4m3fn", "weight_block_size": [128, 128]},
    {**HF, "modules_to_not_convert": ["lm_head"]},
])
def test_block_config_accepts(raw):
    s = parse_block_fp8_config(raw)
    assert (s.weight_block_size, s.activation_scheme) == ((128, 128), "dynamic")


@pytest.mark.parametrize("raw", [
    {**HF, "activation_scheme": "static"},
    {k: v for k, v in HF.items() if k != "weight_block_size"},
    {**HF, "weight_block_size": [64, 128]},
    {**HF, "weight_block_size": [128, 64]},
    {**HF, "fmt": "e5m2"},
    {**HF, "fmt": "e4m3fnuz"},
    {**HF, "fmt": "e8m0"},
    {"quant_method": "fp8", "format": "float8_e4m3fn", "weight_block_size": [128, 128]},
    {"quant_method": "fp8", "weight_scale_semantics": "inverse", "weight_block_size": [128, 128]},
    {"quant_method": "gptq", "bits": 4},
])
def test_block_config_refusals(raw):
    with pytest.raises(NotImplementedError):
        parse_block_fp8_config(raw)


def test_block_config_points_reference_format_to_its_loader():
    with pytest.raises(NotImplementedError, match="load_quantized_linears"):
        parse_block_fp8_config({"quant_method": "fp8", "format": "e4m3", "weight_block_size": [128, 128]})


@pytest.mark.parametrize("raw", [
    {**HF, "fmt": "bogus"},
    {**HF, "fmt": 3},
    {**HF, "activation_scheme": "sometimes"},
    {**HF, "weight_block_size": [128]},
    {**HF, "weight_block_size": [0, 128]},
    {**HF, "weight_block_size": "128x128"},
    {**HF, "modules_to_not_convert": "lm_head"},
])
def test_block_config_malformed(raw):
    with pytest.raises(ValueError):
        parse_block_fp8_config(raw)


def test_reference_loader_still_refuses_block_configs():
    with pytest.raises(NotImplementedError, match="load_block_fp8_linears"):
        parse_quant_config(HF)


# ---- fixtures -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("tag,dt", [("16", "fp16"), ("bf", "bf16")])
def test_dequantize_matches_reference(name, tag, dt):
    w, s = CASES[f"{name}.weight"], CASES[f"{name}.scale_inv"]
    ref = fo.unpack16(CASES[f"{name}.W{tag}"])
    assert np.array_equal(fo.dequantize_weight(w, s, dt).view(np.uint32), ref.view(np.uint32))
    m = B200BlockFp8Linear.from_checkpoint_tensors(torch.from_numpy(w).view(torch.float8_e4m3fn), torch.from_numpy(s),
                                                   device="cpu", post_init=False)
    got = m.dequantize_weight(dtype=torch.float16 if dt == "fp16" else torch.bfloat16).float().numpy()
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("tag", ["16", "bf"])
def test_fixture_outputs_within_activation_rounding(name, tag):
    """The e4m3 activations move x @ W_ref by at most 2^-4 relative of sum |x||W| (the GPU test's bound)."""
    w, s, x = CASES[f"{name}.weight"], CASES[f"{name}.scale_inv"], fo.unpack16(CASES[f"{name}.x{tag}"])
    codes, sx = fo.quantize(x)
    ref, _ = fo.reference(codes, sx, w, s)
    W = fo.unpack16(CASES[f"{name}.W{tag}"]).astype(np.float64)
    bound = np.abs(x.astype(np.float64)) @ np.abs(W) * 2.0 ** -4
    assert np.all(np.abs(ref - CASES[f"{name}.y{tag}"]) <= bound + 1e-6)


def _torch_quantize(x: torch.Tensor):
    """Independent restatement with torch's float8 cast (which gives NaN past 448: clamp first)."""
    M, K = x.shape
    g = x.float().reshape(M, K // 128, 128)
    s = g.abs().amax(dim=2).clamp_min(1e-10) / 448.0
    q = (g / s[:, :, None]).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    return q.reshape(M, K).view(torch.uint8).numpy(), s.numpy()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_quantiser_matches_torch(dtype):
    g = torch.Generator().manual_seed(5)
    x = torch.randn(12, 1024, generator=g) * torch.logspace(-3, 3, 12)[:, None]
    x[0, 5] = 3000.0  # an outlier: the rest of its group underflows to subnormals and zeros
    x[1, :128] = 0.0  # an all-zero group
    x[2, 128:256] = -65000.0 if dtype == torch.float16 else -1e30  # a saturating group of equal magnitudes
    x[3, 256:384] = 1e-7  # tiny values
    x[4, 384:512] *= 1e-4
    x = x.to(dtype)
    codes, s = fo.quantize(x.float().numpy())
    tc, ts = _torch_quantize(x)
    assert np.array_equal(codes, tc)
    assert np.array_equal(s.view(np.uint32), ts.view(np.uint32))
    assert not codes[1, :128].any() and np.isfinite(s).all()
    assert (codes[2, 128:256] == 0xFE).all()  # -448


def test_promotion_mirror_agrees_with_float64():
    rng = np.random.default_rng(3)
    M, K, N = 5, 512, 192
    x = (rng.standard_normal((M, K)) * 0.5).astype(np.float16).astype(np.float32)
    w = fo.e4m3_encode_rn_satfinite(rng.standard_normal((N, K)).astype(np.float32) * 50)
    s_w = (rng.random((2, K // 128)) * 1e-2 + 1e-3).astype(np.float32)
    codes, sx = fo.quantize(x)
    ref, mag = fo.reference(codes, sx, w, s_w)
    for ks in (1, 2, 4):
        acc = fo.promote(codes, sx, w, s_w, ks)
        assert np.all(np.abs(acc - ref) <= 2.0 ** -20 * mag + 1e-30)


# ---- loader -------------------------------------------------------------------------------------------------------------
def _write_ckpt(path, cfg, tensors):
    from safetensors.torch import save_file

    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump({"model_type": "llama", "quantization_config": cfg}, f)
    save_file(tensors, os.path.join(path, "model.safetensors"))


def _fp8(N, K, seed):
    return (torch.randn(N, K, generator=torch.Generator().manual_seed(seed)) * 30).to(torch.float8_e4m3fn)


def test_loader_reads_block_fp8(tmp_path):
    t = {"m.q.weight": _fp8(256, 512, 0), "m.q.weight_scale_inv": torch.rand(2, 4),
         "m.kv.weight": _fp8(576, 256, 1), "m.kv.weight_scale_inv": torch.rand(5, 2),
         "m.kv.bias": torch.zeros(576, dtype=torch.bfloat16),
         "lm_head.weight": torch.randn(64, 256, dtype=torch.bfloat16), "m.norm.weight": torch.ones(256)}
    _write_ckpt(str(tmp_path), {**HF, "modules_to_not_convert": ["lm_head"]}, t)
    mods = load_block_fp8_linears(str(tmp_path), device="cpu")
    assert sorted(mods) == ["m.kv", "m.q"]  # lm_head has no weight_scale_inv: it stays dense
    q, kv = mods["m.q"], mods["m.kv"]
    assert (q.in_features, q.out_features, q.bias) == (512, 256, None)
    assert (kv.in_features, kv.out_features, tuple(kv.weight_scale_inv.shape)) == (256, 576, (5, 2))
    assert torch.equal(q.weight.view(torch.uint8), t["m.q.weight"].view(torch.uint8))
    assert torch.equal(kv.weight_scale_inv, t["m.kv.weight_scale_inv"]) and kv.bias is not None
    assert set(load_block_fp8_linears(str(tmp_path), device="cpu", only=["m.q"])) == {"m.q"}
    with pytest.raises(NotImplementedError):  # the reference-format entry point keeps refusing these checkpoints
        load_quantized_linears(str(tmp_path), device="cpu")


@pytest.mark.parametrize("grid", [(4, 2), (5, 1), (5, 3), (6, 2)])
def test_loader_rejects_wrong_scale_grid(tmp_path, grid):
    t = {"m.kv.weight": _fp8(576, 256, 1), "m.kv.weight_scale_inv": torch.rand(*grid)}
    _write_ckpt(str(tmp_path), HF, t)
    with pytest.raises(ValueError, match="weight_scale_inv"):
        load_block_fp8_linears(str(tmp_path), device="cpu")


def test_loader_refuses_static_input_scales(tmp_path):
    t = {"m.q.weight": _fp8(128, 256, 0), "m.q.weight_scale_inv": torch.rand(1, 2), "m.q.input_scale": torch.ones(())}
    _write_ckpt(str(tmp_path), HF, t)
    with pytest.raises(NotImplementedError, match="input_scale"):
        load_block_fp8_linears(str(tmp_path), device="cpu")


def test_module_envelope():
    for K, N in ((192, 128), (256, 96), (0, 128), (65536 + 128, 128)):
        with pytest.raises(NotImplementedError):
            B200BlockFp8Linear(in_features=K, out_features=N)
    m = B200BlockFp8Linear(in_features=256, out_features=576, bias=True)
    assert tuple(m.weight_scale_inv.shape) == (5, 2) and m.weight.dtype == torch.float8_e4m3fn
    with pytest.raises(ValueError):
        B200BlockFp8Linear.from_checkpoint_tensors(_fp8(576, 256, 0), torch.rand(4, 2), device="cpu", post_init=False)


# ---- ABI argument checks (return -2 before any CUDA work) ---------------------------------------------------------------
def test_abi_argument_checks_without_gpu():
    P = 1 << 20  # any 16-byte aligned non-NULL value: a refused call never dereferences it
    assert lib.b2q_fp8blk_workspace_bytes(8, 4096) == 0  # decode quantises inside the GEMM
    assert lib.b2q_fp8blk_workspace_bytes(9, 4096) == 9 * 4096 + 32 * 12 * 4
    assert lib.b2q_fp8blk_workspace_bytes(300, 256) == 300 * 256 + 2 * 300 * 4

    good = dict(x=P, w=P, s=P, bias=None, out=P, M=16, K=256, N=128, dt=0, ws=P, nws=1 << 30)

    def fwd(**kw):
        a = {**good, **kw}
        return lib.b2q_fp8blk_forward(a["x"], a["w"], a["s"], a["bias"], a["out"], a["M"], a["K"], a["N"], a["dt"],
                                      a["ws"], a["nws"], None)

    bad = (dict(w=None), dict(s=None), dict(out=None), dict(x=None), dict(dt=2), dict(M=-1), dict(K=64), dict(K=0),
           dict(K=65536 + 128), dict(N=96), dict(N=0), dict(x=P + 8), dict(out=P + 2), dict(w=P + 4), dict(s=P + 4),
           dict(ws=None), dict(ws=P + 8), dict(nws=16 * 256))
    for kw in bad:
        assert fwd(**kw) == -2, kw
        assert lib.b2q_last_error()
    assert fwd(M=0) == 0 and fwd(M=0, x=None, ws=None) == 0  # an empty batch is a no-op

    def mm(**kw):
        a = {**good, "codes": P, "sx": P, "ks": 0, **kw}
        return lib.b2q_fp8blk_mm(a["codes"], a["sx"], a["w"], a["s"], a["bias"], a["out"], a["M"], a["K"], a["N"],
                                 a["dt"], a["ks"], None)

    for kw in (dict(codes=None), dict(sx=None), dict(codes=P + 1), dict(sx=P + 4), dict(ks=9), dict(w=None),
               dict(K=192), dict(N=32), dict(dt=-1)):
        assert mm(**kw) == -2, kw
    assert mm(M=0) == 0

    def quant(**kw):
        a = {"x": P, "codes": P, "sx": P, "M": 4, "K": 256, "dt": 1, **kw}
        return lib.b2q_fp8blk_quantize(a["x"], a["codes"], a["sx"], a["M"], a["K"], a["dt"], None)

    for kw in (dict(x=None), dict(codes=None), dict(sx=None), dict(x=P + 2), dict(K=100), dict(M=-2), dict(dt=3)):
        assert quant(**kw) == -2, kw
    assert quant(M=0) == 0


# ---- what the compiler made ---------------------------------------------------------------------------------------------
def test_new_kernels_do_not_spill():
    log = os.path.join(os.path.dirname(HERE), "gptqmodel_b200", "csrc", "b2q_fp8blk.o.log")
    if not os.path.exists(log):
        pytest.skip("b2q_fp8blk.o.log is written by the in-tree build")
    text = open(log).read()
    entries = re.findall(r"Compiling entry function '(\w+)'.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", text, flags=re.S)
    names = [e[0] for e in entries]
    assert sum("fp8blk_gemm_kernel" in n for n in names) == 7 and sum("fp8blk_quant_kernel" in n for n in names) == 2
    for name, stack, st, ld in entries:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), name
