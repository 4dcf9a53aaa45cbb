"""Block-FP8 (HF / DeepSeek-native, W8A8) on the GPU: the quantiser and the e4m3 GEMM against oracle/fp8_block_oracle.py,
the fused decode path, the reference's dequantised weights, and B200BlockFp8Linear end to end."""
import numpy as np
import pytest
import torch

from gptqmodel_b200 import B200BlockFp8Linear, Lora, lib
from gptqmodel_b200._lib import check
from oracle import fp8_block_oracle as fo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TNAME = {torch.float16: "fp16", torch.bfloat16: "bf16"}
DT = {torch.float16: 0, torch.bfloat16: 1}
EPS = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}  # 1 ulp(T) <= |y| * EPS


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _mp(M):
    return (M + 3) // 4 * 4


def quantize_gpu(x):
    M, K = x.shape
    codes = torch.empty((M, K), dtype=torch.uint8, device=DEV)
    sx = torch.zeros((K // 128, _mp(M)), dtype=torch.float32, device=DEV)
    check(lib.b2q_fp8blk_quantize(x.data_ptr(), codes.data_ptr(), sx.data_ptr(), M, K, DT[x.dtype], _stream()),
          "b2q_fp8blk_quantize")
    return codes, sx


def mm_gpu(codes, sx, w, sw, bias, dtype, ks):
    M, K = codes.shape
    N = w.shape[0]
    out = torch.empty((M, N), dtype=dtype, device=DEV)
    check(lib.b2q_fp8blk_mm(codes.data_ptr(), sx.data_ptr(), w.data_ptr(), sw.data_ptr(),
                            None if bias is None else bias.data_ptr(), out.data_ptr(), M, K, N, DT[dtype], ks,
                            _stream()), "b2q_fp8blk_mm")
    return out


def _x(M, K, dtype, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(M, K, generator=g) * scale).to(dtype).to(DEV)


def _layer(K, N, seed):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(N, K, generator=g) * 60).clamp(-448, 448).to(torch.float8_e4m3fn)
    s = (torch.rand((N + 127) // 128, K // 128, generator=g) * 1e-3 + 2e-4) / K ** 0.5
    return w, s


# ---- quantiser ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,K", [(1, 4096), (3, 14336), (8, 256), (9, 4096), (64, 1024), (129, 4096), (2048, 512)])
def test_quantiser_equals_oracle(M, K, dtype):
    x = _x(M, K, dtype, seed=M + K) * torch.logspace(-2, 2, M, device=DEV)[:, None].to(dtype)
    x[0, :128] = 0  # all-zero group
    if K >= 512:
        x[0, 130] = 20000.0 if dtype == torch.float16 else 1e20  # the rest of the group: subnormal codes and zeros
        x[-1, 256:384] = -x[-1, 256:384].abs().max() - 1  # saturating: every |x| at or near the group max
    codes, sx = quantize_gpu(x)
    want_c, want_s = fo.quantize(x.float().cpu().numpy())
    assert torch.equal(codes.cpu(), torch.from_numpy(want_c))
    assert torch.equal(sx[:, :M].cpu(), torch.from_numpy(want_s.T.copy()))


# ---- integer-exact GEMM: the promotion chain bit for bit -----------------------------------------------------------------
INT_CODES = np.array([0x00, 0x38, 0x40, 0x44, 0x48, 0xB8, 0xC0, 0xC4, 0xC8], np.uint8)  # 0, +-1, +-2, +-3, +-4


def _int_problem(M, K, N, seed):
    rng = np.random.default_rng(seed)
    codes = INT_CODES[rng.integers(0, len(INT_CODES), (M, K))]
    w = INT_CODES[rng.integers(0, len(INT_CODES), (N, K))]
    sx = (rng.random((K // 128, _mp(M))) * 3 + 0.01).astype(np.float32) * np.float32(2.0 ** -7)
    sw = (rng.random(((N + 127) // 128, K // 128)) * 2 + 0.001).astype(np.float32) * np.float32(2.0 ** -9)
    return codes, sx, w, sw


@pytest.mark.parametrize("ks", [1, 2, 4])
@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 6, 7, 8, 9, 16, 17, 64, 128, 129, 300, 2048])
def test_mm_integer_exact(M, ks):
    K, N = 1024, 320  # 8 k-blocks; 2.5 feature tiles: the N tail
    codes, sx, w, sw = _int_problem(M, K, N, seed=M * 10 + ks)
    acc = fo.promote(codes, sx[:, :M].T, w, sw, ks)
    bias = (torch.randn(N, generator=torch.Generator().manual_seed(M)) * 0.5)
    for dtype in (torch.float16, torch.bfloat16):
        b = bias.to(dtype)
        y = fo.round_t(acc, TNAME[dtype])
        y = fo.round_t(y + b.float().numpy()[None, :], TNAME[dtype])
        got = mm_gpu(torch.from_numpy(codes).to(DEV), torch.from_numpy(sx).to(DEV),
                     torch.from_numpy(w).to(DEV), torch.from_numpy(sw).to(DEV), b.to(DEV), dtype, ks)
        assert torch.equal(got.float().cpu(), torch.from_numpy(y)), (dtype, M, ks)


# ---- random data against the float64 oracle ------------------------------------------------------------------------------
WORST = {}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,K,N", [(1, 4096, 4096), (5, 4096, 576), (16, 4096, 1024), (100, 14336, 512),
                                   (300, 1024, 4096), (2048, 4096, 576)])
def test_forward_random_within_accumulator_bound(M, K, N, dtype):
    w, s = _layer(K, N, seed=M + N)
    m = B200BlockFp8Linear.from_checkpoint_tensors(w, s, device=DEV)
    x = _x(M, K, dtype, seed=M)
    y = m(x).double().cpu().numpy()
    codes, sx = fo.quantize(x.float().cpu().numpy())
    ref, mag = fo.reference(codes, sx, w.view(torch.uint8).numpy(), s.numpy())
    tol = EPS[dtype] * np.abs(ref) + 2.0 ** -24 + 2.0 ** -10 * mag
    ratio = float((np.abs(y - ref) / tol).max())
    WORST[(M, K, N, TNAME[dtype])] = ratio
    print(f"block-fp8 M={M} K={K} N={N} {TNAME[dtype]}: worst |y - ref| / bound = {ratio:.4f}")
    assert ratio <= 1.0


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M", [1, 2, 3, 5, 8])
def test_fused_decode_equals_quantise_then_mm(M, dtype):
    for K, N in ((4096, 4096), (14336, 4096), (4096, 576), (512, 64)):
        w, s = _layer(K, N, seed=K + N)
        m = B200BlockFp8Linear.from_checkpoint_tensors(w, s, device=DEV)
        x = _x(M, K, dtype, seed=M)
        codes, sx = quantize_gpu(x)
        want = mm_gpu(codes, sx, m.weight, m.weight_scale_inv, None, dtype, 0)
        assert torch.equal(m(x), want), (K, N)


# ---- against the reference's dequantised weights --------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["small", "tall", "wide"])
@pytest.mark.parametrize("tag,dtype", [("16", torch.float16), ("bf", torch.bfloat16)])
def test_fixture_against_reference_dequantised_weight(name, tag, dtype):
    import os

    cases = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fp8_block_cases.npz"))
    w = torch.from_numpy(cases[f"{name}.weight"]).view(torch.float8_e4m3fn)
    m = B200BlockFp8Linear.from_checkpoint_tensors(w, torch.from_numpy(cases[f"{name}.scale_inv"]), device=DEV)
    x = torch.from_numpy(fo.unpack16(cases[f"{name}.x{tag}"])).to(dtype).to(DEV)
    W = fo.unpack16(cases[f"{name}.W{tag}"]).astype(np.float64)
    y = m(x).double().cpu().numpy()
    xd = x.double().cpu().numpy()
    bound = 2.0 ** -4 * (np.abs(xd) @ np.abs(W)) + EPS[dtype] * np.abs(cases[f"{name}.y{tag}"]) + 2.0 ** -24
    assert np.all(np.abs(y - cases[f"{name}.y{tag}"]) <= bound)


# ---- the module -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,N", [(4096, 4096), (4096, 1024), (4096, 14336), (14336, 4096),  # Llama-3-8B
                                 (4096, 12288), (12288, 4096), (4096, 576)])  # Qwen3-8B, DeepSeek kv_a_proj_with_mqa
def test_module_shapes_equal_quantise_then_mm(K, N):
    w, s = _layer(K, N, seed=K ^ N)
    g = torch.Generator().manual_seed(1)
    b = torch.randn(N, generator=g).to(torch.bfloat16)
    m = B200BlockFp8Linear.from_checkpoint_tensors(w, s, bias=b, device=DEV)
    for dtype in (torch.float16, torch.bfloat16):
        for M in (1, 16, 200):
            x = _x(M, K, dtype, seed=M)
            codes, sx = quantize_gpu(x)
            want = mm_gpu(codes, sx, m.weight, m.weight_scale_inv, b.to(dtype).to(DEV), dtype, 0)
            assert torch.equal(m(x), want), (dtype, M)


def test_module_3d_non_contiguous_empty_and_deterministic():
    K, N = 1024, 576
    w, s = _layer(K, N, seed=3)
    m = B200BlockFp8Linear.from_checkpoint_tensors(w, s, device=DEV)
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


def test_module_lora():
    K, N, r = 1024, 512, 16
    w, s = _layer(K, N, seed=31)
    g = torch.Generator().manual_seed(4)
    A = (torch.randn(K, r, generator=g) * 0.05).to(torch.float16)
    B = (torch.randn(r, N, generator=g) * 0.05).to(torch.float16)
    base = B200BlockFp8Linear.from_checkpoint_tensors(w, s, device=DEV)
    m = B200BlockFp8Linear.from_checkpoint_tensors(w, s, device=DEV, adapter=Lora(lora_A=A, lora_B=B))
    for dtype in (torch.float16, torch.bfloat16):
        for M in (1, 33, 300):
            x = _x(M, K, dtype, seed=M).reshape(1, M, K)
            want = base(x).reshape(M, N) + (x.reshape(M, K) @ A.to(DEV, dtype)) @ B.to(DEV, dtype)
            assert torch.equal(m(x).reshape(M, N), want), (dtype, M)


def test_cuda_graph_replay_equals_eager():
    K, N = 4096, 1024
    w, s = _layer(K, N, seed=21)
    m = B200BlockFp8Linear.from_checkpoint_tensors(w, s, bias=torch.randn(N).half(), device=DEV)
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


def test_blockwise_scaled_mm_if_available():
    """torch's own blockwise-scaled e4m3 GEMM (1 x 128 activations, 128 x 128 weights), where this build offers it."""
    F = torch.nn.functional
    if not hasattr(F, "scaled_mm") or not hasattr(F, "ScalingType"):
        pytest.skip("torch.nn.functional.scaled_mm with ScalingType is not available")
    K, N, M, dtype = 1024, 512, 64, torch.bfloat16
    w, s = _layer(K, N, seed=5)
    m = B200BlockFp8Linear.from_checkpoint_tensors(w, s, device=DEV)
    x = _x(M, K, dtype, seed=6)
    codes, sx = quantize_gpu(x)
    try:
        y_t = F.scaled_mm(codes.view(torch.float8_e4m3fn), m.weight.t(),
                          scale_a=sx[:, :M].t().contiguous().t(), scale_recipe_a=F.ScalingType.BlockWise1x128,
                          scale_b=m.weight_scale_inv.t().contiguous().t(), scale_recipe_b=F.ScalingType.BlockWise128x128,
                          output_dtype=dtype)
    except Exception as e:  # noqa: BLE001 (unsupported recipe / device)
        pytest.skip(f"blockwise scaled_mm unavailable here: {type(e).__name__}: {str(e)[:120]}")
    ref, mag = fo.reference(codes.cpu().numpy(), sx[:, :M].t().cpu().numpy(), w.view(torch.uint8).numpy(), s.numpy())
    tol = EPS[dtype] * np.abs(ref) + 2.0 ** -24 + 2.0 ** -10 * mag
    assert np.all(np.abs(y_t.double().cpu().numpy() - ref) <= tol)
    assert np.all(np.abs(m(x).double().cpu().numpy() - ref) <= tol)
