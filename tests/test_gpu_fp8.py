"""GPU: FP8 (e4m3fn, W8A16) layers on the 8-bit tiers — the exhaustive dequantisation, forward against the float64
oracle over every tier and tier boundary, determinism, CUDA graphs, LoRA, the fp16 scale overflow and the reference's
_scaled_mm arithmetic of tensor-scaled layers."""
import numpy as np
import pytest
import torch

from gptqmodel_b200 import B200Fp8QuantLinear, Lora, lib
from gptqmodel_b200._lib import check
from helpers import ref_rounding_slack
from oracle import fp8_oracle as fo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MS = (0, 1, 2, 8, 16, 33, 64, 127, 128, 129, 256, 2048)
LLAMA = ((4096, 4096), (4096, 1024), (4096, 14336), (14336, 4096))
LAYOUTS = (("tensor", None), ("row", None), ("block", (128, 128)), ("block", (64, 128)))
P = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}  # relative half-ulp bound x 2 of T


def _quantize(W, method, block):
    """fp32 W [N, K] -> (e4m3 codes, fp32 scale_inv): the reference's quantize_fp8_weight recipe, restated."""
    def sinv(amax):
        return torch.where(amax > 0, 448.0 / amax.clamp_min(torch.finfo(torch.float32).tiny), torch.ones_like(amax))
    N, K = W.shape
    if method == "tensor":
        s = sinv(W.abs().amax())
        return (W * s).clamp(-448, 448).to(torch.float8_e4m3fn), s
    if method == "row":
        s = sinv(W.abs().amax(dim=1))
        return (W * s[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn), s
    br, bc = block
    Wb = W.reshape(N // br, br, K // bc, bc)
    s = sinv(Wb.abs().amax(dim=(1, 3)))
    return (Wb * s[:, None, :, None]).clamp(-448, 448).to(torch.float8_e4m3fn).reshape(N, K), s


def _layer(K, N, method, block, bias, seed, device=DEV):
    g = torch.Generator(device=device).manual_seed(seed)
    W = torch.randn(N, K, generator=g, device=device) * 0.02
    W[:, 3] *= 20.0  # an outlier input column
    w, s = _quantize(W, method, block)
    b = (torch.randn(N, generator=g, device=device) * 0.1).to(torch.float16) if bias else None
    return w, s, b


def _x(M, K, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, K, generator=g, device=DEV)
    if M > 2:
        x[M // 2] = 0.0
    return x.to(dtype)


def _oracle_W(w, s, method, block, dtype):
    t = "fp16" if dtype == torch.float16 else "bf16"
    W = fo.dequantize(w.view(torch.uint8).cpu().numpy(), s.cpu().numpy(), method, block, t)
    return torch.from_numpy(W.astype(np.float32)).to(DEV).to(dtype)


def _check_forward(out, x, W, bias, gemv, what):
    """|out - ref| <= the fp32 summation bound (K 2^-24 |x| |W|) + the rounding of T at the matmul and at the bias, plus
    for the M = 1 GEMV (scale once per group) the per-weight rounding noise of the reference (helpers.ref_rounding_slack)."""
    dtype = x.dtype
    xd, Wd = x.double(), W.double()
    acc = xd @ Wd
    ref = acc.to(dtype)
    if bias is not None:
        ref = (ref.float() + bias.to(dtype).float()).to(dtype)
    K = x.shape[1]
    tol = K * 2.0 ** -24 * (xd.abs() @ Wd.abs()) + 2 * P[dtype] * (acc.abs() + ref.double().abs()) + 1e-30
    if gemv:
        tol = tol + ref_rounding_slack(W, x).to(DEV).double()
    err = (out.double() - ref.double()).abs()
    assert torch.isfinite(out).all(), what
    bad = err > tol
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} outside, worst {(err / tol).max().item():.2f}"


def _gemv(M, K):
    return M == 1 and K % 128 == 0


# ---- exhaustive dequantisation --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_dequant_exhaustive_codes_by_scales(dtype):
    """All 256 codes x every finite positive scale of T: b2q_fp8_dequant == T(w) / T(s) (torch's division)."""
    if dtype == torch.float16:
        sv = torch.arange(1, 0x7C00, dtype=torch.int32).to(torch.int16).view(torch.float16)
    else:
        sv = torch.arange(1, 0x7F80, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    N = (sv.numel() + 31) // 32 * 32
    s = torch.ones(N, dtype=dtype)
    s[: sv.numel()] = sv
    s = s.to(DEV)
    K = 256
    codes = torch.arange(256, dtype=torch.uint8, device=DEV).repeat(N, 1)  # w[n, k] = code k
    m = B200Fp8QuantLinear.from_checkpoint_tensors(codes.view(torch.float8_e4m3fn), s.float(), device=DEV)
    assert m._gs == K
    W = m.dequantize_weight(dtype=dtype)  # [K, N]
    ref = (codes.view(torch.float8_e4m3fn).to(dtype) / s.view(N, 1)).t()
    torch.cuda.synchronize()
    nan = torch.zeros(K, dtype=torch.bool)
    nan[0x7F] = nan[0xFF] = True
    assert torch.isnan(W[nan.to(DEV)]).all()
    assert torch.equal(W[~nan.to(DEV)].view(torch.int16), ref[~nan.to(DEV)].view(torch.int16))  # signed zeros too


@pytest.mark.parametrize("method,block", LAYOUTS + (("block", (64, 64)), ("block", (1, 128))))
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_dequant_equals_oracle(method, block, dtype):
    K, N = 512, 384
    w, s, _ = _layer(K, N, method, block, False, seed=11)
    m = B200Fp8QuantLinear.from_checkpoint_tensors(w, s, device=DEV)
    W = m.dequantize_weight(dtype=dtype)
    assert torch.equal(W.view(torch.int16), _oracle_W(w, s, method, block, dtype).view(torch.int16))


# ---- forward ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method,block", LAYOUTS)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("bias", [False, True])
def test_forward_every_tier(method, block, dtype, bias):
    K, N = 1024, 640
    w, s, b = _layer(K, N, method, block, bias, seed=K + N)
    m = B200Fp8QuantLinear.from_checkpoint_tensors(w, s, bias=b, device=DEV)
    W = _oracle_W(w, s, method, block, dtype)
    for M in MS:
        x = _x(M, K, dtype, seed=M)
        out = m(x)
        assert out.shape == (M, N) and out.dtype == dtype
        if M:
            _check_forward(out, x, W, b, _gemv(M, K), f"{method}{block} {dtype} bias={bias} M={M}")


@pytest.mark.parametrize("K,N", LLAMA)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_forward_llama_shapes(K, N, dtype):
    w, s, b = _layer(K, N, "block", (128, 128), True, seed=K ^ N)
    m = B200Fp8QuantLinear.from_checkpoint_tensors(w, s, bias=b, device=DEV)
    W = _oracle_W(w, s, "block", (128, 128), dtype)
    for M in (1, 16, 64, 128, 129, 2048):
        x = _x(M, K, dtype, seed=M + 1)
        _check_forward(m(x), x, W, b, _gemv(M, K), f"llama {K}x{N} {dtype} M={M}")


def test_forward_3d_and_non_contiguous_and_unaligned():
    K, N = 512, 256
    w, s, b = _layer(K, N, "block", (128, 128), True, seed=5)
    m = B200Fp8QuantLinear.from_checkpoint_tensors(w, s, bias=b, device=DEV)
    for dtype in (torch.float16, torch.bfloat16):
        W = _oracle_W(w, s, "block", (128, 128), dtype)
        x3 = _x(3 * 7, K, dtype, seed=9).reshape(3, 7, K)
        y3 = m(x3)
        assert y3.shape == (3, 7, N)
        _check_forward(y3.reshape(-1, N), x3.reshape(-1, K), W, b, False, "3-D")
        xt = _x(2 * K, 40, dtype, seed=10).t()[:, :K]  # [40, K] non-contiguous view
        _check_forward(m(xt), xt.contiguous(), W, b, False, "non-contiguous")
        xu = _x(1, K + 1, dtype, seed=12)[:, 1:]  # 2-byte offset: not 16-byte aligned
        _check_forward(m(xu), xu.contiguous(), W, b, True, "unaligned")
        assert m(torch.empty(2, 0, K, dtype=dtype, device=DEV)).shape == (2, 0, N)


def test_bit_identical_run_to_run():
    K, N = 4096, 1024
    w, s, b = _layer(K, N, "block", (128, 128), True, seed=77)
    m = B200Fp8QuantLinear.from_checkpoint_tensors(w, s, bias=b, device=DEV)
    for dtype in (torch.float16, torch.bfloat16):
        for M in (1, 8, 64, 129, 2048):
            x = _x(M, K, dtype, seed=M)
            a = m(x)
            for _ in range(3):
                assert torch.equal(m(x), a), (dtype, M)


def test_cuda_graph_capture_and_replay_across_m():
    K, N = 4096, 1024
    w, s, b = _layer(K, N, "row", None, True, seed=21)
    m = B200Fp8QuantLinear.from_checkpoint_tensors(w, s, bias=b, device=DEV)
    for dtype in (torch.float16, torch.bfloat16):
        for M in (1, 16, 100, 129):
            xs = _x(M, K, dtype, seed=1)
            m(xs)  # warm-up outside the capture (tensor-map cache, shared-memory opt-in)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                ys = m(xs)
            for seed in (2, 3):
                xs.copy_(_x(M, K, dtype, seed=seed))
                g.replay()
                torch.cuda.synchronize()
                assert torch.equal(ys, m(xs)), (dtype, M)


def test_lora_sees_x_and_the_output():
    K, N, r = 1024, 512, 16
    w, s, b = _layer(K, N, "block", (128, 128), True, seed=31)
    g = torch.Generator().manual_seed(4)
    A = (torch.randn(K, r, generator=g) * 0.05).to(torch.float16)
    B = (torch.randn(r, N, generator=g) * 0.05).to(torch.float16)
    base = B200Fp8QuantLinear.from_checkpoint_tensors(w, s, bias=b, device=DEV)
    m = B200Fp8QuantLinear.from_checkpoint_tensors(w, s, bias=b, device=DEV, adapter=Lora(lora_A=A, lora_B=B))
    for dtype in (torch.float16, torch.bfloat16):
        for M in (1, 33, 300):
            x = _x(M, K, dtype, seed=M).reshape(1, M, K)
            y0 = base(x)
            want = y0.reshape(M, N) + (x.reshape(M, K) @ A.to(DEV, dtype)) @ B.to(DEV, dtype)
            assert torch.equal(m(x).reshape(M, N), want), (dtype, M)


def test_fp16_scale_overflow_is_refused_bf16_served():
    K, N = 512, 256
    w, s, b = _layer(K, N, "block", (128, 128), False, seed=41)
    s = s.clone()
    s[0, 1] = 1.0e5  # > 65504: inf in fp16
    m = B200Fp8QuantLinear.from_checkpoint_tensors(w, s, device=DEV)
    with pytest.raises(ValueError, match="fp16"):
        m(_x(4, K, torch.float16, seed=1))
    W = _oracle_W(w, s, "block", (128, 128), torch.bfloat16)
    for M in (1, 4, 200):
        x = _x(M, K, torch.bfloat16, seed=M)
        _check_forward(m(x), x, W, None, _gemv(M, K), f"bf16 overflow layer M={M}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_tensor_scaled_layer_vs_scaled_mm(dtype):
    """The reference's CUDA path for tensor-scaled layers: per-tensor e4m3 activations and torch._scaled_mm.  This module
    keeps x in 16 bits, so the two differ by the activations' e4m3 rounding (half an ulp: 2^-4 relative, 2^-10 of the
    activation scale below the normal range) times |W|, plus the 16-bit roundings of W and of the outputs."""
    K, N = 4096, 1024
    w, s, _ = _layer(K, N, "tensor", None, False, seed=51)
    m = B200Fp8QuantLinear.from_checkpoint_tensors(w, s, device=DEV)
    Wd = m.dequantize_weight(dtype=dtype).double()
    for M in (16, 64, 256):
        x = _x(M, K, dtype, seed=M)
        xf = x.float()
        amax = xf.abs().amax()
        xs = torch.where(amax > 0, 448.0 / amax, torch.ones_like(amax))
        xq = (xf * xs).clamp(-448, 448).to(torch.float8_e4m3fn)
        y_sm = torch._scaled_mm(xq, w.t(), scale_a=torch.reciprocal(xs).reshape(()),
                                scale_b=torch.reciprocal(s.float()).reshape(()), out_dtype=dtype)
        ours = m(x)
        xd = x.double()
        act = (2.0 ** -4 * xd.abs() + 2.0 ** -10 / xs.double()) @ Wd.abs()
        tol = act + 2 * P[dtype] * (xd.abs() @ Wd.abs()) + 2 * P[dtype] * (ours.double().abs() + y_sm.double().abs())
        err = (ours.double() - y_sm.double()).abs()
        assert (err <= tol).all(), f"M={M}: worst {(err / tol).max().item():.2f}"


def test_abi_refuses_bad_arguments_on_the_device():
    K, N = 256, 128
    w, s, _ = _layer(K, N, "row", None, False, seed=1)
    m = B200Fp8QuantLinear.from_checkpoint_tensors(w, s, device=DEV)
    x = _x(4, K, torch.float16, seed=1)
    out = torch.empty(4, N, dtype=torch.float16, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    for g in (32, 96, 512):
        assert lib.b2q_fp8_mm(x.data_ptr(), m.packed.data_ptr(), m._scales[torch.float16].data_ptr(), None,
                              out.data_ptr(), 4, K, N, g, 0, None, 0, st) == -2
    check(lib.b2q_fp8_mm(x.data_ptr(), m.packed.data_ptr(), m._scales[torch.float16].data_ptr(), None, out.data_ptr(),
                         4, K, N, K, 0, None, 0, st), "b2q_fp8_mm")
    torch.cuda.synchronize()
    assert torch.equal(out, m(x))
