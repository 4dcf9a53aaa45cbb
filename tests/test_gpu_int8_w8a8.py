"""Per-channel / per-tensor INT8 (W8A8) on the GPU: the two quantisers and the s8 GEMM bit for bit against
tests/int8_w8a8_mirror.py (the k-sums are exact, so every split-K plan gives the same bits), negative controls of that
check, compressed-tensors' fixture, B200ChannelInt8Linear end to end, a Llama-3-8B-shaped checkpoint and MoE experts
over the module."""
import json
import os

import numpy as np
import pytest
import torch

import int8_w8a8_mirror as im
from gptqmodel_b200 import B200ChannelInt8Linear, Lora, lib
from gptqmodel_b200._lib import check
from oracle import fp8_block_oracle as fo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TNAME = {torch.float16: "fp16", torch.bfloat16: "bf16"}
DT = {torch.float16: 0, torch.bfloat16: 1}
EPS = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}  # 1 ulp(T) <= |y| * EPS


def _stream():
    return torch.cuda.current_stream().cuda_stream


def quantize_gpu(x):
    M, K = x.shape
    codes = torch.empty((M, K), dtype=torch.int8, device=DEV)
    sx = torch.empty(M, dtype=torch.float32, device=DEV)
    check(lib.b2q_int8ch_quantize(x.data_ptr(), codes.data_ptr(), sx.data_ptr(), M, K, DT[x.dtype], _stream()),
          "b2q_int8ch_quantize")
    return codes, sx


def quantize_static_gpu(x, s_in):
    M, K = x.shape
    codes = torch.empty((M, K), dtype=torch.int8, device=DEV)
    sx = torch.empty(M, dtype=torch.float32, device=DEV)
    s = torch.tensor([s_in], dtype=torch.float32, device=DEV)
    check(lib.b2q_int8ch_quantize_static(x.data_ptr(), s.data_ptr(), codes.data_ptr(), sx.data_ptr(), M, K,
                                         DT[x.dtype], _stream()), "b2q_int8ch_quantize_static")
    return codes, sx


def mm_gpu(codes, sx, w, sw, bias, dtype, ks):
    M, K = codes.shape
    N = w.shape[0]
    out = torch.empty((M, N), dtype=dtype, device=DEV)
    check(lib.b2q_int8ch_mm(codes.data_ptr(), sx.data_ptr(), w.data_ptr(), sw.data_ptr(),
                            None if bias is None else bias.data_ptr(), out.data_ptr(), M, K, N, DT[dtype], ks,
                            _stream()), "b2q_int8ch_mm")
    return out


def _x(M, K, dtype, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(M, K, generator=g) * scale).to(dtype).to(DEV)


def _i8(shape, seed):
    return torch.randint(-128, 128, shape, generator=torch.Generator().manual_seed(seed), dtype=torch.int8)


def _layer(K, N, seed):
    """int8 codes [N, K] and per-channel scales [N, 1] with W = w * s of rms ~ 1 / sqrt(K)."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randint(-128, 128, (N, K), generator=g, dtype=torch.int8)
    s = (torch.rand(N, 1, generator=g) * 0.5 + 0.75) / (74 * K ** 0.5)
    return w, s


def _module(K, N, seed, kind="dynamic", bias=None, adapter=None):
    w, s = _layer(K, N, seed)
    s_in = torch.tensor([0.05]) if kind == "static" else None
    return B200ChannelInt8Linear.from_checkpoint_tensors(w, s, input_scale=s_in, bias=bias, device=DEV,
                                                         adapter=adapter)


# ---- quantisers -----------------------------------------------------------------------------------------------------------
QSHAPES = [(1, 65536), (3, 14336), (8, 4096), (9, 4096), (64, 1024), (129, 4096), (2048, 512), (2048, 4096)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,K", QSHAPES)
def test_token_quantiser_equals_mirror(M, K, dtype):
    x = _x(M, K, dtype, seed=M + K) * torch.logspace(-2, 2, M, device=DEV)[:, None].to(dtype)
    x[0, 5] = 20000.0 if dtype == torch.float16 else 1e20  # an outlier row: the rest rounds to 0
    if M > 1:
        x[1] = 0  # an all-zero row: zero codes, a finite scale
    codes, sx = quantize_gpu(x)
    want_c, want_s = im.quantize_dynamic(x.float().cpu().numpy())
    assert torch.equal(codes.cpu(), torch.from_numpy(want_c))
    assert torch.equal(sx.cpu(), torch.from_numpy(want_s))
    assert codes[0, 5].item() == 127
    if M > 1:
        assert not codes[1].any() and bool(torch.isfinite(sx).all())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,K", QSHAPES)
def test_static_quantiser_equals_mirror(M, K, dtype):
    x = _x(M, K, dtype, seed=M * K, scale=4.0)
    x[0, :3] = torch.tensor([1000.0, -1000.0, 0.0], dtype=dtype)  # saturate at both ends
    for s_in in (0.05, 1.7e-3):
        codes, sx = quantize_static_gpu(x, s_in)
        want_c, want_s = im.quantize_static(x.float().cpu().numpy(), np.float32(s_in))
        assert torch.equal(codes.cpu(), torch.from_numpy(want_c))
        assert torch.equal(sx.cpu(), torch.from_numpy(want_s))
        assert codes[0, :3].tolist() == [127, -128, 0]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_quantisers_round_ties_to_even(dtype):
    """Quotients exactly k + 0.5 round to the even neighbour: with s = 0.5 (the static s_in, and the per-token scale of
    a row whose amax is 63.5, since 63.5 / 127 is exact) x = 0.25, 0.75, 1.25 give 0.5, 1.5, 2.5 -> 0, 2, 2."""
    K = 256
    x = torch.zeros(2, K)
    x[:, :6] = torch.tensor([0.25, 0.75, 1.25, -0.25, -0.75, -1.25])
    x[:, 6] = 63.5
    x[1] = -x[1]
    x = x.to(dtype).to(DEV)
    want = [0, 2, 2, 0, -2, -2, 127]
    for codes, sx in (quantize_static_gpu(x, 0.5), quantize_gpu(x)):
        assert sx.tolist() == [0.5, 0.5]
        assert codes[0, :7].tolist() == want and codes[1, :7].tolist() == [-c for c in want]
        assert not codes[:, 7:].any()


# ---- the GEMM: exact int32 sums, bit for bit for every split-K plan -------------------------------------------------------
MS = list(range(1, 17)) + [23, 64, 100, 128, 129, 200, 300, 2048]


@pytest.mark.parametrize("M", MS)
def test_mm_bit_exact_every_plan(M):
    K, N = 1024, 320  # 8 k-blocks; 2.5 feature tiles: the N tail
    rng = np.random.default_rng(M)
    codes = rng.integers(-128, 128, (M, K)).astype(np.int8)
    w = rng.integers(-128, 128, (N, K)).astype(np.int8)
    codes[0, :] = -128  # extremes: the largest sums of this K
    w[0, :] = -128
    sx = ((rng.random(M) * 3 + 0.01) * 2.0 ** -7).astype(np.float32)
    sw = ((rng.random(N) * 2 + 0.001) * 2.0 ** -9).astype(np.float32)
    acc = im.int_sums(codes, w)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(M)) * 0.5
    dc, dw = torch.from_numpy(codes).to(DEV), torch.from_numpy(w).to(DEV)
    dsx, dsw = torch.from_numpy(sx).to(DEV), torch.from_numpy(sw).to(DEV)
    if M >= 17:  # torch's int8 GEMM (M > 16) gives the same int32 sums
        try:
            ti = torch._int_mm(dc, dw.t())
        except RuntimeError as e:
            ti = None
            print(f"torch._int_mm unavailable at M={M}: {str(e)[:80]}")
        if ti is not None:
            assert torch.equal(ti.cpu().long(), torch.from_numpy(acc))
    for dtype in (torch.float16, torch.bfloat16):
        b = bias.to(dtype)
        for bb in (None, b):
            want = torch.from_numpy(im.epilogue(acc, sx, sw, None if bb is None else bb.float().numpy(), TNAME[dtype]))
            for ks in (1, 2, 4, 8, 0):
                got = mm_gpu(dc, dsx, dw, dsw, None if bb is None else bb.to(DEV), dtype, ks)
                assert torch.equal(got.float().cpu(), want), (dtype, ks, bb is None)


def test_mm_bit_exact_wide_k():
    """K = 65536: 512 k-blocks and sums up to 2^30 (float(acc) rounds)."""
    M, K, N = 5, 65536, 128
    rng = np.random.default_rng(1)
    codes = rng.integers(-128, 128, (M, K)).astype(np.int8)
    w = rng.integers(-128, 128, (N, K)).astype(np.int8)
    codes[0], w[0] = -128, -128  # acc[0, 0] = 2^30
    sx, sw = np.full(M, 2.0 ** -20, np.float32), np.full(N, 2.0 ** -9, np.float32)
    acc = im.int_sums(codes, w)
    assert acc[0, 0] == 2 ** 30
    want = torch.from_numpy(im.epilogue(acc, sx, sw, None, "bf16"))
    for ks in (1, 3, 8, 0):
        got = mm_gpu(torch.from_numpy(codes).to(DEV), torch.from_numpy(sx).to(DEV), torch.from_numpy(w).to(DEV),
                     torch.from_numpy(sw).to(DEV), None, torch.bfloat16, ks)
        assert torch.equal(got.float().cpu(), want), ks


def test_negative_controls_are_caught():
    """The bit-exact check must fail on a one-feature shift of s_w, a neighbour token's s_x and a dropped k-block."""
    M, K, N = 9, 1024, 256
    rng = np.random.default_rng(3)
    codes = rng.integers(-128, 128, (M, K)).astype(np.int8)
    w = rng.integers(-128, 128, (N, K)).astype(np.int8)
    sx = (rng.random(M) * 2 + 0.5).astype(np.float32) * np.float32(2.0 ** -8)
    sw = (rng.random(N) * 2 + 0.5).astype(np.float32) * np.float32(2.0 ** -12)
    got = mm_gpu(torch.from_numpy(codes).to(DEV), torch.from_numpy(sx).to(DEV), torch.from_numpy(w).to(DEV),
                 torch.from_numpy(sw).to(DEV), None, torch.float16, 0).float().cpu()
    acc = im.int_sums(codes, w)
    assert torch.equal(got, torch.from_numpy(im.epilogue(acc, sx, sw, None, "fp16")))
    wrong = (im.epilogue(acc, sx, np.roll(sw, 1), None, "fp16"),
             im.epilogue(acc, np.roll(sx, 1), sw, None, "fp16"),
             im.epilogue(im.int_sums(codes[:, :-128], w[:, :-128]), sx, sw, None, "fp16"))
    for bad in wrong:
        assert not torch.equal(got, torch.from_numpy(bad))


# ---- the layer ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["dynamic", "static"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_forward_equals_quantise_then_mm(kind, dtype):
    b = torch.randn(1024, generator=torch.Generator().manual_seed(2)).to(dtype)
    for K, N in ((4096, 1024), (14336, 512), (512, 64)):
        m = _module(K, N, seed=K + N, kind=kind, bias=b[:N])
        for M in (1, 2, 5, 8, 9, 16, 100, 300, 2048):
            x = _x(M, K, dtype, seed=M)
            codes, sx = quantize_static_gpu(x, 0.05) if kind == "static" else quantize_gpu(x)
            want = mm_gpu(codes, sx, m.weight, m.weight_scale, b[:N].to(DEV), dtype, 0)
            assert torch.equal(m(x), want), (K, N, M)
            xf = x.float().cpu().numpy()
            c, s = im.quantize_static(xf, np.float32(0.05)) if kind == "static" else im.quantize_dynamic(xf)
            ref = im.epilogue(im.int_sums(c, m.weight.cpu().numpy()), s, m.weight_scale.cpu().numpy(),
                              b[:N].float().numpy(), TNAME[dtype])
            assert torch.equal(want.float().cpu(), torch.from_numpy(ref)), (K, N, M)


CASES = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "int8_w8a8_cases.npz"))


def _t16(a, dtype):
    return torch.from_numpy(fo.unpack16(a)).to(dtype)


@pytest.mark.parametrize("name,dtype", [("dyn_bf", torch.bfloat16), ("dyn_16", torch.float16),
                                        ("static_bf", torch.bfloat16), ("static_16", torch.float16)])
def test_fixture_against_compressed_tensors(name, dtype):
    """y against compressed-tensors' fake-quantised layer: its activation codes may be one int8 step from this
    package's (scale amax / 127.5 against amax / 127, rounded to T), and its scale differs by at most that step, so
    |y - y_ct| <= sum_k step_m |W_kn| (one step of s_x per code, plus the scale's own change) + the output rounding."""
    c = lambda k: CASES[f"{name}.{k}"]  # noqa: E731
    ws = _t16(c("weight_scale"), dtype)
    s_in = _t16(c("input_scale"), dtype) if f"{name}.input_scale" in CASES.files else None
    m = B200ChannelInt8Linear.from_checkpoint_tensors(torch.from_numpy(c("weight")), ws, input_scale=s_in, device=DEV)
    x = _t16(c("x"), dtype).to(DEV)
    y = m(x).double().cpu().numpy()
    W = fo.unpack16(c("W")).astype(np.float64)
    xd = np.abs(x.double().cpu().numpy())
    step = (xd.max(axis=1) / 127.0)[:, None] if s_in is None else float(s_in.double()) * np.ones((x.shape[0], 1))
    bound = 1.01 * step * np.abs(W).sum(axis=0)[None, :] + 2.0 ** -9 * (xd @ np.abs(W)) \
        + 2 * EPS[dtype] * np.abs(c("y")) + 2.0 ** -24
    assert np.all(np.abs(y - c("y")) <= bound)


@pytest.mark.parametrize("kind", ["dynamic", "static"])
def test_module_3d_non_contiguous_empty_deterministic(kind):
    K, N = 1024, 576
    m = _module(K, N, seed=3, kind=kind, bias=torch.randn(N).to(torch.bfloat16))
    for dtype in (torch.float16, torch.bfloat16):
        x = _x(2 * 7, K, dtype, seed=2).reshape(2, 7, K)
        y = m(x)
        assert y.shape == (2, 7, N) and torch.equal(y.reshape(14, N), m(x.reshape(14, K)))
        xt = _x(K, 12, dtype, seed=4).t()  # non-contiguous
        assert torch.equal(m(xt), m(xt.contiguous()))
        assert m(torch.empty(0, K, dtype=dtype, device=DEV)).shape == (0, N)
        assert m(torch.empty(3, 0, K, dtype=dtype, device=DEV)).shape == (3, 0, N)
        x = _x(700, K, dtype, seed=5)
        assert torch.equal(m(x), m(x))


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


# ---- a Llama-3-8B-shaped checkpoint ---------------------------------------------------------------------------------------
def test_llama3_8b_layer_checkpoint(tmp_path):
    from safetensors.torch import save_file

    from gptqmodel_b200.loader import load_int8_w8a8_linears

    H, I, KV = 4096, 14336, 1024
    shapes = {"self_attn.q_proj": (H, H), "self_attn.k_proj": (KV, H), "self_attn.v_proj": (KV, H),
              "self_attn.o_proj": (H, H), "mlp.gate_proj": (I, H), "mlp.up_proj": (I, H), "mlp.down_proj": (H, I)}
    t = {}
    for i, (n, (N, K)) in enumerate(shapes.items()):
        w, s = _layer(K, N, seed=i)
        t[f"model.layers.0.{n}.weight"] = w
        t[f"model.layers.0.{n}.weight_scale"] = s.to(torch.bfloat16)
    t["lm_head.weight"] = torch.zeros(128, H, dtype=torch.bfloat16)
    cfg = {"quant_method": "compressed-tensors", "format": "int-quantized", "ignore": ["lm_head"],
           "config_groups": {"group_0": {"targets": ["Linear"],
                                         "weights": {"num_bits": 8, "type": "int", "symmetric": True,
                                                     "strategy": "channel", "dynamic": False},
                                         "input_activations": {"num_bits": 8, "type": "int", "symmetric": True,
                                                               "strategy": "token", "dynamic": True}}}}
    with open(tmp_path / "config.json", "w") as f:
        json.dump({"model_type": "llama", "quantization_config": cfg}, f)
    save_file(t, str(tmp_path / "model.safetensors"))
    mods = load_int8_w8a8_linears(str(tmp_path), device=DEV)
    assert sorted(mods) == sorted(f"model.layers.0.{n}" for n in shapes)
    for n, (N, K) in shapes.items():
        m = mods[f"model.layers.0.{n}"]
        for M in (1, 64):
            x = _x(M, K, torch.bfloat16, seed=M)
            c, s = im.quantize_dynamic(x.float().cpu().numpy())
            want = im.epilogue(im.int_sums(c, t[f"model.layers.0.{n}.weight"].numpy()), s,
                               t[f"model.layers.0.{n}.weight_scale"].float().reshape(-1).numpy(), None, "bf16")
            assert torch.equal(m(x).float().cpu(), torch.from_numpy(want)), (n, M)


# ---- MoE experts over the module: the per-expert loop ---------------------------------------------------------------------
def test_moe_experts_loop_matches_float64():
    from gptqmodel_b200 import moe

    E, H, I, T, top_k = 4, 1024, 512, 24, 2
    mods = lambda seed, K, N: [_module(K, N, seed=seed + e) for e in range(E)]  # noqa: E731
    w1, w3, w2 = mods(100, H, I), mods(200, H, I), mods(300, I, H)
    blk = moe.MoEExperts(w1, w3, w2)
    assert blk._stack is None  # the per-expert loop
    g = torch.Generator().manual_seed(7)
    ids = torch.stack([torch.randperm(E, generator=g)[:top_k] for _ in range(T)]).to(DEV)
    wts = torch.softmax(torch.randn(T, top_k, generator=g), -1).to(DEV)

    def ref_linear(m, xt):  # float64 s_x s_w sum_k q w of this package's codes, rounded to T as the layer does
        c, s = im.quantize_dynamic(xt.float().cpu().numpy())
        y = im.int_sums(c, m.weight.cpu().numpy()) * (s.astype(np.float64)[:, None]
                                                      * m.weight_scale.cpu().double().numpy()[None, :])
        return torch.from_numpy(y).to(xt.dtype).to(DEV)

    for dtype in (torch.float16, torch.bfloat16):
        x = _x(T, H, dtype, seed=9)
        y = blk(x, ids, wts).double()
        want = torch.zeros(T, H, dtype=torch.float64, device=DEV)
        for t in range(T):
            for j in range(top_k):
                e = int(ids[t, j])
                xt = x[t:t + 1]
                h = torch.nn.functional.silu(ref_linear(w1[e], xt)) * ref_linear(w3[e], xt)
                want[t] += float(wts[t, j]) * ref_linear(w2[e], h)[0].double()
        bound = 4 * EPS[dtype] * want.abs().max()  # per-token quantisation: one rounding of T apart at most per stage
        assert float((y - want).abs().max()) <= float(bound), dtype
