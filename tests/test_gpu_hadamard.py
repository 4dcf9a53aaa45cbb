"""GPU: b2q_hadamard (the online Hadamard transform of rotated QuaRot / SpinQuant checkpoints) against the float64
oracle, and rotated QuantLinear modules end to end."""
import os

import numpy as np
import pytest
import torch

from helpers import assert_close_rel, assert_layer_close, make_layer
from oracle.hadamard_oracle import hadamard_transform

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hadamard_cases.npz")
ORDERS = (12, 20, 28, 36, 40, 52, 60, 108, 140, 156, 172)
ROWS = (1, 2, 7, 8, 9, 64, 133, 2048)
SHAPES = sorted({(K * P, K) for K in ORDERS for P in (8, 64, 512) if K * P <= 65536} |
                {(14336, 28), (28672, 28), (11008, 172), (8192, 1)})


def _had(K, device="cuda"):
    if K == 1:
        return None
    return torch.from_numpy(np.load(GOLDEN)[f"had{K}"]).to(device)


def _x(rows, n, dtype, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(rows, n, device="cuda", generator=gen)
    cols = torch.randperm(n, device="cuda", generator=gen)[: max(1, n // 100)]
    x[:, cols] *= 100.0  # outlier channels
    return x.to(dtype)


def _run(x, had, K):
    import gptqmodel_b200 as g

    y = torch.empty_like(x)
    g.check(g.lib.b2q_hadamard(x.data_ptr(), None if had is None else had.data_ptr(), K, y.data_ptr(), x.shape[0],
                               x.shape[1], 0 if x.dtype == torch.float16 else 1,
                               torch.cuda.current_stream().cuda_stream), "b2q_hadamard")
    return y


def _ulp(v, dtype):
    mant = 10 if dtype == torch.float16 else 7
    tiny = 2.0 ** -24 if dtype == torch.float16 else 2.0 ** -133
    _, e = torch.frexp(v.abs())
    return torch.clamp(torch.ldexp(torch.ones_like(v), (e - 1 - mant).to(torch.int32)), min=tiny)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("n,K", SHAPES, ids=[f"n{n}_K{K}" for n, K in SHAPES])
def test_hadamard_kernel_against_float64_oracle(n, K, dtype):
    had = _had(K)
    equal = total = 0
    for rows in ROWS:
        x = _x(rows, n, dtype, seed=rows * 7 + K)
        y = _run(x, had, K)
        exact = hadamard_transform(x.double(), None if had is None else had.double(), K)
        rn = exact.to(dtype)  # the correctly rounded result
        d = (y.double() - rn.double()).abs()
        ulp = _ulp(torch.maximum(rn.double().abs(), y.double().abs()), dtype)
        # fp32 accumulation: an output that cancels far below its row's magnitude (outlier channels of opposite sign)
        # carries the fp32 summation error bound, (log2 P + K + 2) * 2^-24 * sum|x| / sqrt(n), on top of the 1 ulp
        P = n // K
        acc = (P.bit_length() - 1 + K + 2) * 2.0 ** -24 * x.double().abs().sum(dim=1, keepdim=True) / n ** 0.5
        assert bool((d <= ulp + acc).all()), (rows, float((d / (ulp + acc)).max()))
        equal += int((y == rn).sum())
        total += y.numel()
    assert equal >= 0.999 * total, (equal, total)  # over all row counts of the case


@pytest.mark.gpu
def test_hadamard_is_deterministic():
    for n, K in ((14336, 28), (11008, 172), (8192, 1)):
        for rows in (1, 2048):
            x = _x(rows, n, torch.bfloat16, seed=5)
            a, b = _run(x, _had(K), K), _run(x, _had(K), K)
            assert torch.equal(a, b), (n, rows)


def _module(L, had=None, K=None, partial_dim=None, adapter=None):
    """K None: no rotation; else the full-row transform of order K (or rows of `partial_dim`)."""
    from gptqmodel_b200 import B200QuantLinear

    m = B200QuantLinear(bits=L["bits"], group_size=L["group_size"], desc_act=L["desc_act"], sym=L["sym"],
                        in_features=L["K"], out_features=L["N"], bias=L["bias"] is not None, register_buffers=False,
                        adapter=adapter)
    mk = lambda t: None if t is None else torch.nn.Parameter(t.clone().cuda(), requires_grad=False)  # noqa: E731
    m.qweight, m.qzeros, m.scales, m.g_idx, m.bias = (mk(L[k]) for k in ("qweight", "qzeros", "scales", "g_idx", "bias"))
    if partial_dim is not None:
        m.online_partial_had, m.had_dim, m.K = True, partial_dim, K
    elif K is not None:
        m.online_full_had, m.K = True, K
    if had is not None:
        m.set_had_K(had.float().cpu())
    m.post_init()
    return m


VARIANTS = {
    "4bit_g128_sym": dict(bits=4, group_size=128, sym=True),
    "4bit_g64_asym": dict(bits=4, group_size=64, sym=False),
    "8bit_g128": dict(bits=8, group_size=128, sym=True),
    "4bit_actorder": dict(bits=4, group_size=128, sym=True, desc_act=True),
    "4bit_bias": dict(bits=4, group_size=128, sym=True, bias=True),
}
KIN = 28 * 128  # Llama-3's order 28 at P = 128


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_rotated_module_against_oracle(variant):
    L = make_layer(KIN, 256, seed=11, **VARIANTS[variant])
    had = _had(28)
    rot = _module(L, had, 28)
    plain = _module(L)
    for dtype in (torch.float16, torch.bfloat16):
        for M in (1, 4, 8, 9, 64, 128, 129, 2048):
            x = _x(M, KIN, dtype, seed=M)
            y = rot(x)
            xr = _run(x, had, 28)
            assert torch.equal(y, plain(xr)), (variant, M)  # the rotated forward is the plain one on b2q_hadamard(x)
            xt = hadamard_transform(x.double(), had.double(), 28).to(dtype)
            rel = 1e-3 if dtype == torch.float16 else 1.6e-2  # bf16: 2 ulp, as the other bf16 parity tests
            assert_layer_close(y, L, xt, rel, f"{variant} {dtype} M={M}")


@pytest.mark.gpu
def test_rotated_module_power_of_two_and_partial():
    L = make_layer(4096, 128, seed=3)
    m = _module(L, None, 1)  # K = 1: pure Walsh-Hadamard, no had_K
    x = _x(5, 4096, torch.float16, seed=1)
    assert_layer_close(m(x), L, hadamard_transform(x.double(), None, 1).half(), 1e-3, "full K=1")
    L = make_layer(KIN, 128, seed=4)
    m = _module(L, None, 1, partial_dim=128)
    for M in (1, 9, 300):
        x = _x(M, KIN, torch.float16, seed=M)
        xt = hadamard_transform(x.double().reshape(-1, 128), None, 1).reshape(x.shape).half()
        assert_layer_close(m(x), L, xt, 1e-3, f"partial had_dim=128 M={M}")
    # the reference's quirk: had_K missing for K != 1 leaves x untouched
    q = _module(L)
    q.online_full_had, q.K = True, 28
    x = _x(3, KIN, torch.float16, seed=9)
    assert_layer_close(q(x), L, x, 1e-3, "had_K None, K=28")


@pytest.mark.gpu
def test_rotated_module_adapter_sees_rotated_input():
    from gptqmodel_b200 import Lora

    L = make_layer(KIN, 256, seed=21, bias=True)
    gen = torch.Generator().manual_seed(2)
    A = (torch.randn(KIN, 8, generator=gen) * 0.05).to(torch.float16)
    B = (torch.randn(8, 256, generator=gen) * 0.05).to(torch.float16)
    had = _had(28)
    m = _module(L, had, 28, adapter=Lora(rank=8, lora_A=A, lora_B=B))
    from helpers import oracle_forward
    for M in (1, 200):
        x = _x(M, KIN, torch.float16, seed=M)
        xt = hadamard_transform(x.double(), had.double(), 28).half().cpu()
        ref = oracle_forward(L, xt).float() + ((xt.float() @ A.float()).half().float() @ B.float())
        assert_close_rel(m(x), ref, 2e-3, f"rotated lora M={M}")


@pytest.mark.gpu
def test_pdl_chain_into_decode_is_bit_identical():
    import gptqmodel_b200 as g

    L = make_layer(14336, 512, seed=5)
    m = _module(L, _had(28), 28)
    xs = [_x(M, 14336, torch.float16, seed=M) for M in (1, 4, 8)]
    outs = {}
    try:
        for flag in ("1", "0"):
            os.environ["B2Q_DISABLE_PDL"] = flag
            g.lib.b2q_debug_reload_env()
            outs[flag] = [m(x) for x in xs]
            torch.cuda.synchronize()
    finally:
        os.environ.pop("B2Q_DISABLE_PDL", None)
        g.lib.b2q_debug_reload_env()
    for a, b in zip(outs["1"], outs["0"]):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_rotated_forward_in_cuda_graph():
    L = make_layer(KIN, 256, seed=8)
    m = _module(L, _had(28), 28)
    for M in (1, 64):
        x = _x(M, KIN, torch.float16, seed=M)
        want = m(x)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(x)  # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            y = m(x)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, want), M
        x.copy_(_x(M, KIN, torch.float16, seed=M + 100))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, m(x)), M
