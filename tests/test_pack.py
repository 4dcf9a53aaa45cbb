"""Device-side packer against the reference's own packers.

tests/golden/ref_cases.npz holds, for every case, the float weights, the [N, G] scale / zero grids and the tensors the
reference's `pack_block` AND `pack_original` produced (asserted identical when the fixture was generated,
tests/golden/make_golden.py; the reference checks the same in tests/test_pack.py:114).
"""
import json
import os

import numpy as np
import pytest
import torch

import oracle
from gptqmodel_b200.pack import pack_gptq

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
META = json.loads(bytes(np.load(os.path.join(GOLDEN, "ref_cases.npz"))["__meta__"]).decode())


@pytest.mark.parametrize("name", list(META))
def test_pack_gptq_bit_exact_vs_reference(ref_cases, name):
    m = ref_cases.meta[name]
    bias = ref_cases.get(name, "lin_bias") if m["bias"] else None
    out = pack_gptq(ref_cases.get(name, "weight"), ref_cases.get(name, "in_scales"), ref_cases.get(name, "in_zeros"),
                    ref_cases.get(name, "g_idx"), m["bits"], bias=bias)
    assert torch.equal(out["qweight"], ref_cases.get(name, "qweight"))
    assert torch.equal(out["qzeros"], ref_cases.get(name, "qzeros"))
    assert torch.equal(out["scales"], ref_cases.get(name, "scales"))
    assert torch.equal(out["g_idx"], ref_cases.get(name, "g_idx"))
    if m["bias"]:
        assert torch.equal(out["bias"], ref_cases.get(name, "bias"))


def test_pack_gptq_matches_oracle_on_random_grids_and_rejects_bad_input():
    gen = torch.Generator().manual_seed(9)
    for bits, gs, sym in ((4, 64, False), (8, 128, True), (4, 128, True)):
        N, K = 96, 512
        W = torch.randn(N, K, generator=gen) * 0.3
        g_idx = torch.arange(K, dtype=torch.int32) // gs
        sc, ze = (oracle.quantize_sym if sym else oracle.quantize_asym)(W, bits, gs)[:2]
        a = pack_gptq(W, sc, ze, g_idx, bits)
        b = oracle.pack(W, sc, ze, g_idx, bits)
        assert torch.equal(a["qweight"], b[0]) and torch.equal(a["qzeros"], b[1]) and torch.equal(a["scales"], b[2])
    with pytest.raises(NotImplementedError):
        pack_gptq(W, sc, ze, g_idx, 9)
    with pytest.raises(ValueError):
        pack_gptq(W, sc[:-1], ze, g_idx, 4)


@pytest.mark.parametrize("name", list(META))
def test_module_pack_block_fills_reference_tensors(ref_cases, name):
    from gptqmodel_b200 import B200QuantLinear
    m = ref_cases.meta[name]
    lin = torch.nn.Linear(m["K"], m["N"], bias=m["bias"])
    with torch.no_grad():
        lin.weight.copy_(ref_cases.get(name, "weight"))
        if m["bias"]:
            lin.bias.copy_(ref_cases.get(name, "lin_bias"))
    if m["K"] % 64 or m["N"] % 32:
        pytest.skip("shape outside the B200 kernels' tiling")
    mod = B200QuantLinear(bits=m["bits"], group_size=m["group_size"], desc_act=m["desc_act"], sym=m["sym"],
                          in_features=m["K"], out_features=m["N"], bias=m["bias"])
    mod.pack_block(lin, ref_cases.get(name, "in_scales"), ref_cases.get(name, "in_zeros"), ref_cases.get(name, "g_idx"))
    for k in ("qweight", "qzeros", "scales", "g_idx"):
        assert torch.equal(getattr(mod, k).data, ref_cases.get(name, k)), k
    if m["bias"]:
        assert torch.equal(mod.bias.data, ref_cases.get(name, "bias"))
    assert mod.qzero_format() == 2 and set(mod.state_dict()) >= {"qweight", "qzeros", "scales", "g_idx"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(META))
def test_pack_gptq_on_the_gpu_bit_exact_vs_reference(ref_cases, name):
    # the quantiser-side contract on the device (the reference's pack_gpu, qlinear/__init__.py:1326-1498): same integer ops
    # on CUDA tensors must give the tensors the reference's CPU packers produced, and the packed module must then run
    m = ref_cases.meta[name]
    dev = "cuda"
    bias = ref_cases.get(name, "lin_bias").to(dev) if m["bias"] else None
    out = pack_gptq(ref_cases.get(name, "weight").to(dev), ref_cases.get(name, "in_scales").to(dev),
                    ref_cases.get(name, "in_zeros").to(dev), ref_cases.get(name, "g_idx").to(dev), m["bits"], bias=bias)
    for k in ("qweight", "qzeros", "scales", "g_idx"):
        assert out[k].is_cuda and torch.equal(out[k].cpu(), ref_cases.get(name, k)), k
    if m["K"] % 64 == 0 and m["N"] % 32 == 0:
        from gptqmodel_b200 import B200QuantLinear
        from helpers import assert_close_rel
        mod = B200QuantLinear.from_checkpoint_tensors(out["qweight"], out["qzeros"], out["scales"], out["g_idx"], m["bits"],
                                                      m["group_size"], bias=out.get("bias"), desc_act=m["desc_act"],
                                                      sym=m["sym"])
        x = ref_cases.get(name, "x")
        ref = oracle.forward(x, ref_cases.get(name, "qweight"), ref_cases.get(name, "qzeros"), ref_cases.get(name, "scales"),
                             ref_cases.get(name, "g_idx"), m["bits"], bias=ref_cases.get(name, "bias"))
        assert_close_rel(mod(x.to(dev)), ref, 1e-3, f"packed on the GPU: {name}")
