"""GPU: QQQ (W4A8) tier — quantiser and GEMM bit-exact against the oracle, the reference's fixtures and kernel, graphs.

The accumulation is integer and the epilogue order is fixed, so the bar is torch.equal wherever the oracle applies."""
import os

import numpy as np
import pytest
import torch

from gptqmodel_b200 import B200QqqQuantLinear, Lora, lib
from gptqmodel_b200._lib import check
from oracle import qqq_oracle as qo

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = "cuda:0"
MS = (0, 1, 2, 7, 8, 9, 64, 127, 128, 129, 2048)
LLAMA = ((4096, 4096), (4096, 1024), (4096, 14336), (14336, 4096))
EDGES = ((128, 64), (64, 128), (192, 128), (256, 192), (320, 384))  # each edge of the envelope, 64-wide K tail, N%128=64


def _x(M, K, dtype, seed, halves=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g) * 0.7
    if M:
        x[:, 5 % K] *= 30.0                   # outlier columns
        x[:, K - 3] *= -45.0
        if M > 2:
            x[M // 2] = 0.0                   # an all-zero row
        if halves:
            # row 0: max |x| = 127 -> s_tok = 1, every other element on a .5 code boundary
            x[0] = (torch.arange(K) % 61 - 30).to(torch.float32) + 0.5
            x[0, 1] = 127.0
    return x.to(dtype).to(DEV)


def _quantize(x):
    M, K = x.shape
    Kp = (K + 127) // 128 * 128
    q = torch.full((M, Kp), 99, dtype=torch.int8, device=DEV)
    s = torch.full((M,), -1.0, dtype=torch.float32, device=DEV)
    check(lib.b2q_qqq_quantize(x.data_ptr(), q.data_ptr(), s.data_ptr(), M, K, 0 if x.dtype == torch.float16 else 1,
                               torch.cuda.current_stream().cuda_stream), "b2q_qqq_quantize")
    torch.cuda.synchronize()
    return q, s


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("K", [128, 320, 4096, 14336])
def test_quantiser_bit_exact(dtype, K):
    for M in MS:
        x = _x(M, K, dtype, seed=K + M)
        q, s = _quantize(x)
        rq, rs = qo.quantize(x.cpu())
        assert torch.equal(q[:, :K].cpu(), rq), (M, K)
        assert torch.equal(s.cpu(), rs), (M, K)
        assert not q[:, K:].any(), "padding codes must be 0"


def _layer(K, N, gs, seed):
    g = torch.Generator().manual_seed(seed)
    codes = torch.randint(0, 16, (K, N), generator=g).to(torch.uint8)
    sc = torch.rand(N, generator=g) * 2e-4 + 2e-5
    sg = (torch.rand(K // 128, N, generator=g) * 14.9 + 1.0).to(torch.float16) if gs == 128 else None
    bias = (torch.randn(N, generator=g) * 0.2).to(torch.float16)
    B, scp, sgp = qo.pack_qqq(codes, sc, sg)
    mod = B200QqqQuantLinear.from_checkpoint_tensors(B, scp, sgp if gs == 128 else None, gs, device=DEV)
    return mod, codes.to(DEV), sc.to(DEV), None if sg is None else sg.to(DEV), bias.to(DEV)


@pytest.mark.parametrize("KN", LLAMA + EDGES)
@pytest.mark.parametrize("gs", [-1, 128])
def test_forward_bit_exact(KN, gs):
    K, N = KN
    if gs == 128 and (K % 128 or K == 128):
        pytest.skip("group 128 needs K % 128 == 0 (and K == 128 is the per-channel format)")
    mod, codes, sc, sg, bias = _layer(K, N, gs, seed=K * 3 + N + gs)
    for use_bias in (False, True):
        mod.bias = bias if use_bias else None
        for dtype in (torch.float16, torch.bfloat16):
            for M in MS:
                x = _x(M, K, dtype, seed=M * 7 + K)
                y = mod(x)
                ref = qo.forward(x, codes, sc, sg, bias if use_bias else None)
                assert y.dtype == dtype and y.shape == (M, N)
                assert torch.equal(y, ref), (K, N, gs, use_bias, dtype, M,
                                             int((y != ref).sum()) if y.shape == ref.shape else None)


def test_forward_3d_noncontiguous_lora_and_determinism():
    K, N = 4096, 1024
    mod, codes, sc, sg, bias = _layer(K, N, 128, seed=11)
    mod.bias = bias
    base = _x(2 * 33, K * 2, torch.float16, seed=5, halves=False)
    x = base.view(2, 33, 2 * K)[..., ::2]              # 3-D, non-contiguous
    assert not x.is_contiguous()
    y = mod(x)
    assert y.shape == (2, 33, N)
    assert torch.equal(y, qo.forward(x.contiguous(), codes, sc, sg, bias))
    assert torch.equal(mod(x), y)                      # two runs, same bits
    xb = x.to(torch.bfloat16)
    assert torch.equal(mod(xb), qo.forward(xb.contiguous(), codes, sc, sg, bias))
    # LoRA on the fp16 output with the fp16 activations, then the cast (QQQLinear.forward)
    g = torch.Generator().manual_seed(3)
    la, lb = torch.randn(K, 8, generator=g) * 0.01, torch.randn(8, N, generator=g) * 0.01
    mod.adapter = Lora(rank=8)
    mod.adapter.post_init("x", DEV, lora_A=la, lora_B=lb)
    for xx in (x, xb):
        a16 = xx.reshape(-1, K).to(torch.float16)
        ref = qo.forward(xx.to(torch.float16).contiguous(), codes, sc, sg, bias).reshape(-1, N)
        ref = ref.add_((a16 @ la.to(DEV, torch.float16)) @ lb.to(DEV, torch.float16)).to(xx.dtype)
        assert torch.equal(mod(xx).reshape(-1, N), ref)
    mod.adapter = None


def test_empty_and_graph_capture():
    K, N = 4096, 4096
    mod, codes, sc, sg, bias = _layer(K, N, -1, seed=12)
    y0 = mod(torch.empty(0, K, dtype=torch.float16, device=DEV))
    assert y0.shape == (0, N) and y0.dtype == torch.float16
    y0 = mod(torch.empty(2, 0, K, dtype=torch.bfloat16, device=DEV))
    assert y0.shape == (2, 0, N) and y0.dtype == torch.bfloat16
    for M in (1, 2048):
        x = _x(M, K, torch.float16, seed=M)
        eager = mod(x)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            mod(x)  # warm-up outside the capture (tensor-map cache, shared-memory opt-in)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            yg = mod(x)
        x.copy_(_x(M, K, torch.float16, seed=M + 1))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, mod(x))
        x.copy_(_x(M, K, torch.float16, seed=M))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, eager)


def test_post_init_rejects_out_of_range_group_scale():
    K, N = 256, 128
    codes = torch.zeros(K, N, dtype=torch.uint8)                    # (0 - 8) * 16.5 = -132
    sg = torch.full((K // 128, N), 16.5, dtype=torch.float16)
    B, scp, sgp = qo.pack_qqq(codes, torch.ones(N), sg)
    with pytest.raises(ValueError):
        B200QqqQuantLinear.from_checkpoint_tensors(B, scp, sgp, 128, device=DEV)


GOLD = np.load(os.path.join(HERE, "golden", "qqq_cases.npz"))


@pytest.mark.parametrize("c", sorted({k.split(".")[0] for k in GOLD.files}))
def test_golden_reference_outputs(c):
    t = lambda k: torch.from_numpy(GOLD[f"{c}.{k}"].copy())  # noqa: E731
    gs = -1 if t("s_group").numel() == 0 else 128
    bias = t("bias") if t("bias").numel() else None
    mod = B200QqqQuantLinear.from_checkpoint_tensors(t("B"), t("s_channel"), t("s_group") if gs == 128 else None, gs,
                                                     bias=bias, device=DEV)
    for tag, dt in (("16", torch.float16), ("bf", torch.bfloat16)):
        x = t("x" + tag).to(dt).to(DEV)
        y = mod(x)
        ref = t("y" + tag).to(dt).to(DEV)
        y16, r16 = y.to(torch.float32), ref.to(torch.float32)
        ulp = (r16.abs().clamp_min(2.0 ** -14).log2().floor() - (10 if tag == "16" else 7)).exp2()
        assert bool(((y16 - r16).abs() <= ulp).all()), c
        codes = torch.from_numpy(GOLD[f"{c}.codes"].copy())
        sg = torch.from_numpy(GOLD[f"{c}.s_grp_canon"].copy()) if gs == 128 else None
        sc = torch.from_numpy(GOLD[f"{c}.s_ch_canon"].copy())
        assert torch.equal(y, qo.forward(x, codes, sc, sg, bias))


REF_SO = os.path.join(ROOT, "oracle", "_ref", "gptqmodel_qqq.so")


@pytest.mark.skipif(not os.path.exists(REF_SO), reason="the reference QQQ op was not built (oracle/build_qqq.py needs a "
                                                      "GPTQModel checkout at build time)")
@pytest.mark.parametrize("gs", [-1, 128])
def test_matches_reference_kernel(gs):
    torch.ops.load_library(REF_SO)
    for K, N in LLAMA:
        mod, codes, sc, sg, bias = _layer(K, N, gs, seed=K + 2 * N + gs)
        mod.bias = bias
        B, scp, sgp = qo.pack_qqq(codes.cpu(), sc.cpu(), None if sg is None else sg.cpu())
        B, scp, sgp = B.to(DEV), scp.to(DEV), sgp.to(DEV)
        for M in (1, 16, 64, 2048):
            x = _x(M, K, torch.float16, seed=M + K)
            q, s = _quantize(x)
            D = torch.empty(M, N, dtype=torch.float16, device=DEV)
            C = torch.zeros(16 * 64, N, dtype=torch.int32, device=DEV)
            ws = torch.zeros(N // 128 * 16, dtype=torch.int32, device=DEV)
            torch.ops.gptqmodel_qqq.qqq_gemm(q[:, :K].contiguous(), B, C, D, s.reshape(M, 1), scp, sgp, ws, -1, -1,
                                             -1, 16)
            D.add_(bias)
            assert torch.equal(mod(x), D), (K, N, gs, M)
