"""Per-channel / per-tensor FP8 (W8A8) on the GPU: the two quantisers and the e4m3 GEMM against tests/fp8_w8a8_mirror.py,
the fused decode path, compressed-tensors' fixture, torch's row-wise scaled_mm, B200ChannelFp8Linear end to end and
MoE experts over it."""
import os

import numpy as np
import pytest
import torch

import fp8_w8a8_mirror as fm
from gptqmodel_b200 import B200ChannelFp8Linear, Lora, lib
from gptqmodel_b200._lib import check
from oracle import fp8_block_oracle as fo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TNAME = {torch.float16: "fp16", torch.bfloat16: "bf16"}
DT = {torch.float16: 0, torch.bfloat16: 1}
EPS = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}  # 1 ulp(T) <= |y| * EPS
INF = float("inf")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def quantize_gpu(x, ub=INF):
    M, K = x.shape
    codes = torch.empty((M, K), dtype=torch.uint8, device=DEV)
    sx = torch.empty(M, dtype=torch.float32, device=DEV)
    check(lib.b2q_fp8ch_quantize(x.data_ptr(), codes.data_ptr(), sx.data_ptr(), M, K, ub, DT[x.dtype], _stream()),
          "b2q_fp8ch_quantize")
    return codes, sx


def quantize_static_gpu(x, s_in):
    M, K = x.shape
    codes = torch.empty((M, K), dtype=torch.uint8, device=DEV)
    sx = torch.empty(M, dtype=torch.float32, device=DEV)
    s = torch.tensor([s_in], dtype=torch.float32, device=DEV)
    check(lib.b2q_fp8ch_quantize_static(x.data_ptr(), s.data_ptr(), codes.data_ptr(), sx.data_ptr(), M, K, DT[x.dtype],
                                        _stream()), "b2q_fp8ch_quantize_static")
    return codes, sx


def mm_gpu(codes, sx, w, sw, bias, dtype, ks):
    M, K = codes.shape
    N = w.shape[0]
    out = torch.empty((M, N), dtype=dtype, device=DEV)
    check(lib.b2q_fp8ch_mm(codes.data_ptr(), sx.data_ptr(), w.data_ptr(), sw.data_ptr(),
                           None if bias is None else bias.data_ptr(), out.data_ptr(), M, K, N, DT[dtype], ks, _stream()),
          "b2q_fp8ch_mm")
    return out


def _x(M, K, dtype, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(M, K, generator=g) * scale).to(dtype).to(DEV)


def _layer(K, N, seed):
    """e4m3 codes [N, K] and per-channel scales [N, 1] with W = w * s of rms ~ 1 / sqrt(K)."""
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(N, K, generator=g) * 60).clamp(-448, 448).to(torch.float8_e4m3fn)
    s = (torch.rand(N, 1, generator=g) * 0.5 + 0.75) / (60 * K ** 0.5)
    return w, s


def _module(K, N, seed, kind="dynamic", ub=None, bias=None, adapter=None):
    w, s = _layer(K, N, seed)
    s_in = torch.tensor([0.05]) if kind == "static" else None
    return B200ChannelFp8Linear.from_checkpoint_tensors(w, s, input_scale=s_in, bias=bias, ub=ub, device=DEV,
                                                        adapter=adapter)


# ---- quantisers -----------------------------------------------------------------------------------------------------------
QSHAPES = [(1, 65536), (3, 14336), (8, 4096), (9, 4096), (64, 1024), (129, 4096), (2048, 512)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,K", QSHAPES)
def test_token_quantiser_equals_mirror(M, K, dtype):
    x = _x(M, K, dtype, seed=M + K) * torch.logspace(-2, 2, M, device=DEV)[:, None].to(dtype)
    x[0, 5] = 20000.0 if dtype == torch.float16 else 1e20  # an outlier: the rest of the row underflows
    if M > 1:
        x[1] = 0  # an all-zero row: zero codes, a finite scale
    for ub in (INF, 3.0):  # 3.0 clips the amax of most rows: codes of |x| > 3 saturate
        codes, sx = quantize_gpu(x, ub)
        want_c, want_s = fm.quantize_dynamic(x.float().cpu().numpy(), ub)
        assert torch.equal(codes.cpu(), torch.from_numpy(want_c)), ub
        assert torch.equal(sx.cpu(), torch.from_numpy(want_s)), ub
        if M > 1:
            assert not codes[1].any() and bool(torch.isfinite(sx).all())
    assert (codes[0, 5] == 0x7E).item()  # +448 under the clipping bound


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,K", QSHAPES)
def test_static_quantiser_equals_mirror(M, K, dtype):
    x = _x(M, K, dtype, seed=M * K, scale=4.0)
    x[0, :3] = torch.tensor([1000.0, -1000.0, 0.0], dtype=dtype)  # saturate at +-448
    for s_in in (0.05, 1.7e-3):
        codes, sx = quantize_static_gpu(x, s_in)
        want_c, want_s = fm.quantize_static(x.float().cpu().numpy(), np.float32(s_in))
        assert torch.equal(codes.cpu(), torch.from_numpy(want_c))
        assert torch.equal(sx.cpu(), torch.from_numpy(want_s))
        assert codes[0, :3].tolist() == [0x7E, 0xFE, 0x00]


# ---- integer-exact GEMM: the k-sum and the epilogue bit for bit -----------------------------------------------------------
INT_CODES = np.array([0x00, 0x38, 0x40, 0x44, 0x48, 0xB8, 0xC0, 0xC4, 0xC8], np.uint8)  # 0, +-1, +-2, +-3, +-4


@pytest.mark.parametrize("ks", [1, 2, 4])
@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 6, 7, 8, 9, 16, 17, 64, 128, 129, 300, 2048])
def test_mm_integer_exact(M, ks):
    K, N = 1024, 320  # 8 k-blocks; 2.5 feature tiles: the N tail
    rng = np.random.default_rng(M * 10 + ks)
    codes = INT_CODES[rng.integers(0, len(INT_CODES), (M, K))]
    w = INT_CODES[rng.integers(0, len(INT_CODES), (N, K))]
    sx = ((rng.random(M) * 3 + 0.01) * 2.0 ** -7).astype(np.float32)
    sw = ((rng.random(N) * 2 + 0.001) * 2.0 ** -9).astype(np.float32)
    acc = fm.promote(codes, w, ks)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(M)) * 0.5
    for dtype in (torch.float16, torch.bfloat16):
        b = bias.to(dtype)
        for bb in (None, b):
            want = fm.epilogue(acc, sx, sw, None if bb is None else bb.float().numpy(), TNAME[dtype])
            got = mm_gpu(torch.from_numpy(codes).to(DEV), torch.from_numpy(sx).to(DEV), torch.from_numpy(w).to(DEV),
                         torch.from_numpy(sw).to(DEV), None if bb is None else bb.to(DEV), dtype, ks)
            assert torch.equal(got.float().cpu(), torch.from_numpy(want)), (dtype, M, ks, bb is None)


# ---- random data against the float64 oracle ------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["dynamic", "static"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,K,N", [(1, 4096, 6144), (5, 4096, 4096), (16, 4096, 28672), (100, 14336, 4096),
                                   (300, 4096, 1024), (2048, 4096, 4096)])
def test_forward_random_within_accumulator_bound(M, K, N, dtype, kind):
    m = _module(K, N, seed=M + N, kind=kind)
    x = _x(M, K, dtype, seed=M)
    y = m(x).double().cpu().numpy()
    xf = x.float().cpu().numpy()
    codes, sx = fm.quantize_static(xf, np.float32(0.05)) if kind == "static" else fm.quantize_dynamic(xf)
    ref, mag = fm.reference(codes, sx, m.weight.view(torch.uint8).cpu().numpy(), m.weight_scale.cpu().numpy())
    tol = EPS[dtype] * np.abs(ref) + 2.0 ** -24 + 2.0 ** -10 * mag
    ratio = float((np.abs(y - ref) / tol).max())
    print(f"fp8 w8a8 {kind} M={M} K={K} N={N} {TNAME[dtype]}: worst |y - ref| / bound = {ratio:.4f}")
    assert ratio <= 1.0


@pytest.mark.parametrize("kind,ub", [("dynamic", None), ("dynamic", 2.5), ("static", None)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 6, 7, 8])
def test_fused_decode_equals_quantise_then_mm(M, dtype, kind, ub):
    for K, N in ((4096, 4096), (14336, 4096), (4096, 576), (512, 64)):
        m = _module(K, N, seed=K + N, kind=kind, ub=ub)
        x = _x(M, K, dtype, seed=M)
        codes, sx = quantize_static_gpu(x, 0.05) if kind == "static" else quantize_gpu(x, INF if ub is None else ub)
        want = mm_gpu(codes, sx, m.weight, m.weight_scale, None, dtype, 0)
        assert torch.equal(m(x), want), (K, N)


# ---- against compressed-tensors -------------------------------------------------------------------------------------------
CASES = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fp8_w8a8_cases.npz"))


def _t16(a, dtype):
    return torch.from_numpy(fo.unpack16(a)).to(dtype)


@pytest.mark.parametrize("name,dtype", [("dyn_bf", torch.bfloat16), ("dyn_16", torch.float16),
                                        ("static_bf", torch.bfloat16)])
def test_fixture_against_compressed_tensors(name, dtype):
    """y against compressed-tensors' fake-quantised layer: the two quantisers may pick codes one e4m3 step apart
    (compressed-tensors rounds the scale and the quotient to T first), which moves y by at most
    sum_k 2^-3 |x_k| |W_kn| (one step is <= 2^-3 of the code, plus the scale's own rounding), and the e4m3 GEMM adds the
    accumulator bound of the random-data test."""
    c = lambda k: CASES[f"{name}.{k}"]  # noqa: E731
    ws = _t16(c("weight_scale"), dtype)
    s_in = _t16(c("input_scale"), dtype) if f"{name}.input_scale" in CASES.files else None
    m = B200ChannelFp8Linear.from_checkpoint_tensors(torch.from_numpy(c("weight")).view(torch.float8_e4m3fn), ws,
                                                     input_scale=s_in, device=DEV)
    x = _t16(c("x"), dtype).to(DEV)
    y = m(x).double().cpu().numpy()
    W = fo.unpack16(c("W")).astype(np.float64)
    xd = np.abs(x.double().cpu().numpy())
    bound = 2.0 ** -3 * (xd @ np.abs(W)) + 2 * EPS[dtype] * np.abs(c("y")) + 2.0 ** -24
    assert np.all(np.abs(y - c("y")) <= bound)


def test_scaled_mm_rowwise_within_bound():
    """torch's row-wise scaled e4m3 GEMM on this module's codes and scales stays within the same float64 bound."""
    K, N, M, dtype = 4096, 1024, 64, torch.bfloat16
    m = _module(K, N, seed=5)
    x = _x(M, K, dtype, seed=6)
    codes, sx = quantize_gpu(x)
    try:
        y_t = torch._scaled_mm(codes.view(torch.float8_e4m3fn), m.weight.t(), scale_a=sx[:, None],
                               scale_b=m.weight_scale[None, :], out_dtype=dtype)
    except Exception as e:  # noqa: BLE001 (unsupported on this build / device)
        pytest.skip(f"row-wise scaled_mm unavailable here: {type(e).__name__}: {str(e)[:120]}")
    ref, mag = fm.reference(codes.cpu().numpy(), sx.cpu().numpy(), m.weight.view(torch.uint8).cpu().numpy(),
                            m.weight_scale.cpu().numpy())
    tol = EPS[dtype] * np.abs(ref) + 2.0 ** -24 + 2.0 ** -10 * mag
    assert np.all(np.abs(y_t.double().cpu().numpy() - ref) <= tol)
    assert np.all(np.abs(m(x).double().cpu().numpy() - ref) <= tol)


# ---- the module -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["dynamic", "static"])
def test_module_3d_non_contiguous_empty_deterministic_bias(kind):
    K, N = 1024, 576
    b = torch.randn(N, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16)
    m = _module(K, N, seed=3, kind=kind, bias=b)
    for dtype in (torch.float16, torch.bfloat16):
        x = _x(2 * 7, K, dtype, seed=2).reshape(2, 7, K)
        y = m(x)
        assert y.shape == (2, 7, N) and torch.equal(y.reshape(14, N), m(x.reshape(14, K)))
        xt = _x(K, 12, dtype, seed=4).t()  # non-contiguous
        assert torch.equal(m(xt), m(xt.contiguous()))
        assert m(torch.empty(0, K, dtype=dtype, device=DEV)).shape == (0, N)
        assert m(torch.empty(3, 0, K, dtype=dtype, device=DEV)).shape == (3, 0, N)
        for M in (1, 9, 700):
            x = _x(M, K, dtype, seed=M)
            assert torch.equal(m(x), m(x))
            xf = x.float().cpu().numpy()
            codes, sx = fm.quantize_static(xf, np.float32(0.05)) if kind == "static" else fm.quantize_dynamic(xf)
            got = quantize_static_gpu(x, 0.05) if kind == "static" else quantize_gpu(x)
            want = mm_gpu(*got, m.weight, m.weight_scale, b.to(dtype).to(DEV), dtype, 0)
            assert torch.equal(m(x), want), (dtype, M)


def test_module_lora():
    K, N, r = 1024, 512, 16
    g = torch.Generator().manual_seed(4)
    A = (torch.randn(K, r, generator=g) * 0.05).to(torch.float16)
    B = (torch.randn(r, N, generator=g) * 0.05).to(torch.float16)
    base = _module(K, N, seed=31)
    m = _module(K, N, seed=31, adapter=Lora(lora_A=A, lora_B=B))
    for dtype in (torch.float16, torch.bfloat16):
        for M in (1, 33, 300):
            x = _x(M, K, dtype, seed=M).reshape(1, M, K)
            want = base(x).reshape(M, N) + (x.reshape(M, K) @ A.to(DEV, dtype)) @ B.to(DEV, dtype)
            assert torch.equal(m(x).reshape(M, N), want), (dtype, M)


@pytest.mark.parametrize("kind", ["dynamic", "static"])
def test_cuda_graph_replay_equals_eager(kind):
    K, N = 4096, 1024
    m = _module(K, N, seed=21, kind=kind, bias=torch.randn(N).half())
    for dtype in (torch.float16, torch.bfloat16):
        for M in (1, 8, 16, 129):
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


# ---- MoE experts over the module: the per-expert loop ---------------------------------------------------------------------
def test_moe_experts_loop_and_grouped_refusal():
    from gptqmodel_b200 import moe

    E, H, I, T, top_k = 4, 1024, 512, 24, 2
    mods = lambda seed, K, N: [_module(K, N, seed=seed + e) for e in range(E)]  # noqa: E731
    w1, w3, w2 = mods(100, H, I), mods(200, H, I), mods(300, I, H)
    with pytest.raises(ValueError):
        moe.MoEExperts(w1, w3, w2, grouped=True)
    blk = moe.MoEExperts(w1, w3, w2)
    assert blk._stack is None  # the per-expert loop
    g = torch.Generator().manual_seed(7)
    ids = torch.stack([torch.randperm(E, generator=g)[:top_k] for _ in range(T)]).to(DEV)
    wts = torch.softmax(torch.randn(T, top_k, generator=g), -1).to(DEV)
    for dtype in (torch.float16, torch.bfloat16):
        x = _x(T, H, dtype, seed=9)
        y = blk(x, ids, wts).double()
        want = torch.zeros(T, H, dtype=torch.float64, device=DEV)
        for t in range(T):
            for j in range(top_k):
                e = int(ids[t, j])
                xt = x[t:t + 1]
                h = torch.nn.functional.silu(w1[e](xt)) * w3[e](xt)
                want[t] += float(wts[t, j]) * w2[e](h)[0].double()
        bound = 4 * EPS[dtype] * want.abs().max()  # the loop runs each expert's rows at another M: another k-split
        assert float((y - want).abs().max()) <= float(bound), dtype
