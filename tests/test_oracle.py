"""CPU: pin the oracle against the reference's golden vector and reference-generated fixtures."""
import json
import os

import numpy as np
import pytest
import torch

import oracle
from conftest import GOLDEN

META = json.loads(bytes(np.load(os.path.join(GOLDEN, "ref_cases.npz"))["__meta__"]).decode())


def test_q4_reference_golden_vector(q4_golden):
    # recipe: GPTQModel tests/test_q4_exllama_v2.py:32-87, vector: tests/q4_reference.py
    torch.manual_seed(42)
    qweight = torch.randint(-100, 100, size=(128, 1024), dtype=torch.int32)
    scales = torch.zeros(8, 1024, dtype=torch.float16) + 0.002
    qzeros = torch.full((8, 128), 0x11111111, dtype=torch.int32)
    g_idx = torch.arange(1024, dtype=torch.int32) // 128
    x = torch.rand(1, 1, 1024, dtype=torch.float16)
    y = oracle.forward(x, qweight, qzeros, scales, g_idx, 4)[0][0]
    ref = torch.tensor(q4_golden["reference"], dtype=torch.float16)
    assert y.shape == ref.shape
    assert torch.allclose(y, ref, rtol=3e-5, atol=2e-2)
    # far tighter than the reference's own tolerance: fp16 rounding of ~6.5 magnitudes
    assert (y.float() - ref.float()).abs().max().item() < 8e-3


@pytest.mark.parametrize("name", list(META))
def test_pack_bit_exact_vs_reference(ref_cases, name):
    m = ref_cases.meta[name]
    qw, qz, sc, gi = oracle.pack(
        ref_cases.get(name, "weight"), ref_cases.get(name, "in_scales"), ref_cases.get(name, "in_zeros"),
        ref_cases.get(name, "g_idx"), m["bits"])
    assert torch.equal(qw, ref_cases.get(name, "qweight"))
    assert torch.equal(qz, ref_cases.get(name, "qzeros"))
    assert torch.equal(sc, ref_cases.get(name, "scales"))
    assert torch.equal(gi, ref_cases.get(name, "g_idx"))


@pytest.mark.parametrize("name", list(META))
def test_dequant_bit_exact_vs_reference(ref_cases, name):
    m = ref_cases.meta[name]
    W = oracle.dequantize_weight(ref_cases.get(name, "qweight"), ref_cases.get(name, "qzeros"),
                                 ref_cases.get(name, "scales"), ref_cases.get(name, "g_idx"), m["bits"])
    Wr = ref_cases.get(name, "W")
    assert W.dtype == torch.float16 and W.shape == Wr.shape
    assert torch.equal(W, Wr)


@pytest.mark.parametrize("name", list(META))
def test_forward_vs_reference(ref_cases, name):
    m = ref_cases.meta[name]
    args = (ref_cases.get(name, "qweight"), ref_cases.get(name, "qzeros"), ref_cases.get(name, "scales"),
            ref_cases.get(name, "g_idx"), m["bits"])
    bias = ref_cases.get(name, "bias")
    x = ref_cases.get(name, "x")
    y = oracle.forward(x, *args, bias=bias)
    yr = ref_cases.get(name, "y_fp16")
    # the reference ran a CPU fp16 matmul; ours accumulates in fp32 (what cuBLAS does): <= 1-2 fp16 ulp
    assert torch.allclose(y.float(), yr.float(), rtol=2e-3, atol=2e-3)
    ybf = oracle.forward(x.to(torch.bfloat16), *args, bias=bias)
    assert torch.allclose(ybf.float(), ref_cases.get(name, "y_bf16"), rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("name", [n for n in META if META[n]["bits"] == 4 and META[n]["group_size"] > 0])
def test_cpu_fused_vs_reference(ref_cases, name):
    m = ref_cases.meta[name]
    lin = oracle.CpuFusedLinear(ref_cases.get(name, "qweight"), ref_cases.get(name, "qzeros"),
                                ref_cases.get(name, "scales"), ref_cases.get(name, "g_idx"), m["bits"],
                                m["group_size"], bias=ref_cases.get(name, "bias"))
    y = lin.forward(ref_cases.get(name, "x"))
    yr = ref_cases.get(name, "y_cpu_fused")
    assert torch.allclose(y.float(), yr, rtol=1e-2, atol=1e-2)
    # and the fused bf16 kernel agrees with the exact oracle at bf16 level
    yo = oracle.forward(ref_cases.get(name, "x"), ref_cases.get(name, "qweight"), ref_cases.get(name, "qzeros"),
                        ref_cases.get(name, "scales"), ref_cases.get(name, "g_idx"), m["bits"],
                        bias=ref_cases.get(name, "bias"))
    assert torch.allclose(y.float(), yo.float(), rtol=3e-2, atol=6e-2)


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("desc_act", [False, True])
def test_reference_closed_form(bits, desc_act):
    """tests/test_torch_kernel_accuracy.py:46-108 generator + `_reference_weight` closed form."""
    K, N, gs = 64, 32, 32
    torch.manual_seed((7 if desc_act else 0) + bits)
    maxq = (1 << bits) - 1
    lin = torch.nn.Linear(K, N, bias=True)
    scales = torch.rand(N, K // gs) * 0.01 + 0.005
    zeros = torch.randint(0, maxq + 1, (N, K // gs)).float()
    if desc_act:
        g_idx = (torch.randperm(K) // gs).to(torch.int32)
    else:
        g_idx = torch.arange(K, dtype=torch.int32) // gs
    sf, zf = scales[:, g_idx.long()], zeros[:, g_idx.long()]
    codes = torch.round((lin.weight.data + zf * sf) / sf).clamp(0, maxq)
    ref = ((codes - zf) * sf.to(torch.float16).float()).T.contiguous()
    qw, qz, sc, gi = oracle.pack(lin.weight.data, scales, zeros, g_idx, bits)
    W = oracle.dequantize_weight(qw, qz, sc, gi, bits)
    assert torch.allclose(W.float(), ref, atol=1e-4 if bits == 4 else 2e-3, rtol=0)
    assert torch.equal(oracle.unpack_qweight(qw, bits).float(), codes.T)
    x = (torch.randn(4, K) * 0.5).to(torch.float16)
    out = oracle.forward(x, qw, qz, sc, gi, bits, bias=lin.bias.data.to(torch.float16))
    ref_out = x.float() @ ref + lin.bias.data.float()
    assert torch.allclose(out.float(), ref_out, atol=5e-3, rtol=1e-2)


@pytest.mark.parametrize("bits", [4, 8])
def test_qzeros_v1_v2_roundtrip(bits):
    # utils/model.py:810-818; tests/test_qzero_offsets.py:145-163
    maxq = (1 << bits) - 1
    z = torch.randint(1, maxq + 1, (4, 64)).float()  # v1 stores zero-1, so zero>=1 round-trips
    _, qz, _, _ = oracle.pack(torch.zeros(64, 32), torch.ones(64, 4), z.T.contiguous(),
                              torch.arange(32, dtype=torch.int32) // 8, bits)
    v1 = oracle.convert_v2_to_v1(qz, bits)
    assert torch.equal(oracle.unpack_qzeros(v1, bits).float(), z - 1)
    assert torch.equal(oracle.convert_v1_to_v2(v1, bits), qz)


def test_negative_words_are_valid_codes():
    qw = torch.tensor([[-1], [-(2 ** 31)]], dtype=torch.int32)
    u = oracle.unpack_qweight(qw, 4)
    assert u[:8, 0].tolist() == [15] * 8
    assert u[8:, 0].tolist() == [0] * 7 + [8]
