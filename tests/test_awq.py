"""AWQ (FORMAT.GEMM) front-end: oracle pinned to the reference, exact layout conversion, GPU parity.

Fixtures: tests/golden/awq_cases.npz, produced by running the UNMODIFIED reference's `dequantize_gemm` and
`AwqTorchLinear.forward` (tests/golden/make_golden_awq.py).
"""
import json
import os

import numpy as np
import pytest
import torch

import oracle
from gptqmodel_b200 import B200AwqQuantLinear, awq_gemm_to_gptq
from helpers import assert_close_rel

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def awq_cases():
    z = np.load(os.path.join(HERE, "golden", "awq_cases.npz"))
    meta = json.loads(bytes(z["__meta__"]).decode())
    out = {}
    for name, m in meta.items():
        d = {k: torch.from_numpy(z[f"{name}.{k}"]) for k in ("qweight", "qzeros", "scales", "x", "W", "y_fp16", "y_bf16")}
        d.update({k: v for k, v in m.items() if k != "bias"})
        d["bias"] = torch.from_numpy(z[f"{name}.bias"]) if m["bias"] else None
        out[name] = d
    return out


def test_awq_oracle_matches_reference_bit_exact(awq_cases):
    # packing_utils.py:106-121 (dequantize_gemm) and torch_awq.py:157-197 (forward), outputs of the reference itself
    for name, c in awq_cases.items():
        W = oracle.awq_dequantize(c["qweight"], c["qzeros"], c["scales"], c["group_size"])
        assert W.dtype == torch.float16 and torch.equal(W, c["W"]), name
        y = oracle.awq_forward(c["x"], c["qweight"], c["qzeros"], c["scales"], c["group_size"], c["bias"])
        assert_close_rel(y, c["y_fp16"], 1e-3, name)
        ybf = oracle.awq_forward(c["x"].to(torch.bfloat16), c["qweight"], c["qzeros"], c["scales"], c["group_size"],
                                 c["bias"])
        assert_close_rel(ybf, c["y_bf16"], 1.6e-2, name + " bf16")  # 2 bf16 ulp: the reference rounds W to bf16 first
        assert torch.equal(oracle.awq_pack(oracle.awq_unpack(c["qweight"])), c["qweight"])


def test_scale_once_arithmetic_vs_per_weight_rounding(awq_cases):
    """Why GPU parity of the decode / GEMV tiers against the reference-rounded oracle carries `ref_rounding_slack`
    (VERDICT r01 next #1: "diagnose awq_gK").  The reference rounds EVERY dequantised weight to fp16 before the matmul; a
    kernel that applies the scale once per group to an exact integer dot product is the same sum without those K
    roundings.  On the reference's own fixture `awq_gK` (K = 128, one group, M = 2) even float64-exact arithmetic lands
    1.18x outside `1e-3*|ref| + 1e-3*rms(ref)` of the rounded-W oracle on one of the 256 outputs — the very element and
    ratio an earlier GPU run reported for the decode tier — so that miss was the reference's
    weight-rounding noise, not kernel arithmetic; with the 4-sigma noise term every case is inside."""
    from helpers import PARITY_LOG, ref_rounding_slack  # noqa: F401
    worst = {}
    for name, c in awq_cases.items():
        ye = oracle.awq_forward_exact(c["x"], c["qweight"], c["qzeros"], c["scales"], c["group_size"], c["bias"])
        yo = oracle.awq_forward(c["x"], c["qweight"], c["qzeros"], c["scales"], c["group_size"], c["bias"])
        r = yo.float()
        tol = 1e-3 * r.abs() + 1e-3 * r.pow(2).mean().sqrt()
        worst[name] = float(((ye.float() - r).abs() / tol).max())
        assert_close_rel(ye, yo, 1e-3, name, slack=ref_rounding_slack(c["W"], c["x"]))
    assert worst["awq_gK"] > 1.0 and abs(worst["awq_gK"] - 1.176) < 0.01, worst
    assert all(v < 1.0 for k, v in worst.items() if k != "awq_gK"), worst


def test_awq_to_gptq_conversion_is_exact(awq_cases):
    # the converted GPTQ v2 tensors must dequantise (GPTQ oracle, pinned to the reference's TorchLinear) to the very
    # weights the reference's AWQ path produces: the conversion is pure integer re-packing
    for name, c in awq_cases.items():
        g = awq_gemm_to_gptq(c["qweight"], c["qzeros"], c["scales"], c["group_size"])
        K, N = c["K"], c["N"]
        gs = c["group_size"] if c["group_size"] > 0 else K
        assert g["qweight"].shape == (K // 8, N) and g["qzeros"].shape == (K // gs, N // 8)
        assert g["qweight"].dtype == torch.int32 and g["qzeros"].dtype == torch.int32
        assert torch.equal(g["g_idx"], (torch.arange(K) // gs).to(torch.int32))
        W = oracle.dequantize_weight(g["qweight"], g["qzeros"], g["scales"], g["g_idx"], 4)
        assert torch.equal(W.to(torch.float16), c["W"]), name
        # code-level check against the AWQ oracle's own unpacking
        assert torch.equal(oracle.unpack_qweight(g["qweight"], 4).to(torch.int16), oracle.awq_unpack(c["qweight"]))
        assert torch.equal(oracle.unpack_qzeros(g["qzeros"], 4).to(torch.int16), oracle.awq_unpack(c["qzeros"]))


def test_awq_conversion_random_large_and_errors():
    gen = torch.Generator().manual_seed(5)
    K, N, gs = 1024, 512, 128
    codes = torch.randint(0, 16, (K, N), generator=gen)
    zeros = torch.randint(0, 16, (K // gs, N), generator=gen)
    qw, qz = oracle.awq_pack(codes), oracle.awq_pack(zeros)
    sc = (torch.rand(K // gs, N, generator=gen) * 0.01 + 0.001).to(torch.float16)
    g = awq_gemm_to_gptq(qw, qz, sc, gs)
    assert torch.equal(oracle.unpack_qweight(g["qweight"], 4).to(torch.int64), codes)
    assert torch.equal(oracle.unpack_qzeros(g["qzeros"], 4).to(torch.int64), zeros)
    with pytest.raises(ValueError):
        awq_gemm_to_gptq(qw, qz[:-1], sc, gs)
    with pytest.raises(NotImplementedError):
        awq_gemm_to_gptq(qw, qz, sc, gs, bits=8)
    with pytest.raises(ValueError):
        awq_gemm_to_gptq(qw.to(torch.int64), qz, sc, gs)


def test_awq_module_contract_without_gpu():
    m = B200AwqQuantLinear(bits=4, group_size=128, in_features=512, out_features=256, bias=True)
    # AWQ-shaped buffers for the loader (qlinear/__init__.py:1646-1668)
    assert m.qweight.shape == (512, 32) and m.qzeros.shape == (4, 32) and m.scales.shape == (4, 256)
    assert set(m.state_dict()) == {"qweight", "qzeros", "scales", "bias"}
    with pytest.raises(NotImplementedError):
        B200AwqQuantLinear(bits=8, group_size=128, in_features=512, out_features=256)
    with pytest.raises(NotImplementedError):
        B200AwqQuantLinear(bits=4, group_size=128, desc_act=True, in_features=512, out_features=256)
    from gptqmodel_b200 import B2QError
    with pytest.raises(B2QError):
        m.post_init()  # CPU tensors: converts, then fails loudly at the CUDA prepack (no CPU path)
