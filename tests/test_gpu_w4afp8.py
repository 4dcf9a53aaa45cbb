"""W4AFP8 tier on the GPU (b2q_w4afp8.cu): the GEMM bit for bit against the float32 mirror of its promotion chain on
small-integer codes, negative controls, a float64 bound on random data, the layer against quantise-then-mm, the
compressed-tensors fixtures, the module contract, a Llama-shaped checkpoint and MoE experts on the per-expert loop."""
import json
import os

import numpy as np
import pytest
import torch

import w4afp8_mirror as wm
from gptqmodel_b200 import B200W4Fp8Linear, Lora, lib
from gptqmodel_b200._lib import check

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
DT = {torch.float16: 0, torch.bfloat16: 1}
EPS = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}  # 1 ulp(T) <= |y| * EPS
FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "w4afp8_cases.npz")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def quantize_gpu(x):
    M, K = x.shape
    codes = torch.empty((M, K), dtype=torch.uint8, device=DEV)
    sx = torch.empty(M, dtype=torch.float32, device=DEV)
    check(lib.b2q_fp8ch_quantize(x.data_ptr(), codes.data_ptr(), sx.data_ptr(), M, K, float("inf"), DT[x.dtype],
                                 _stream()), "b2q_fp8ch_quantize")
    return codes, sx


def prepack_gpu(wp: np.ndarray, K: int, N: int):
    src = torch.from_numpy(wp).to(DEV)
    packed = torch.empty(int(lib.b2q_w4afp8_packed_bytes(K, N)), dtype=torch.uint8, device=DEV)
    check(lib.b2q_w4afp8_prepack(src.data_ptr(), packed.data_ptr(), K, N, _stream()), "b2q_w4afp8_prepack")
    return packed


def mm_gpu(codes, sx, packed, sw, bias, dtype, ks, N):
    M, K = codes.shape
    out = torch.empty((M, N), dtype=dtype, device=DEV)
    check(lib.b2q_w4afp8_mm(codes.data_ptr(), sx.data_ptr(), packed.data_ptr(), sw.data_ptr(),
                            None if bias is None else bias.data_ptr(), out.data_ptr(), M, K, N, DT[dtype], ks,
                            _stream()), "b2q_w4afp8_mm")
    return out


def _exact_case(M, K, N, seed):
    """Small-integer e4m3 codes in [-2, 2], weights q in [-8, 7], bf16-exact group scales (8 significant bits) and
    token scales: every k-block sum is an exact integer below 2^12 and every P * s_w is exact in float32."""
    rng = np.random.default_rng(seed)
    c = rng.integers(-2, 3, size=(M, K)).astype(np.float32)
    cq = rng.integers(0, 16, size=(N, K)).astype(np.uint8)
    sw = torch.from_numpy(rng.uniform(0.5, 2.0, size=(K // 128, N)).astype(np.float32) / 64).to(torch.bfloat16)
    sw = sw.float().numpy()
    sx = rng.uniform(0.01, 0.1, size=M).astype(np.float32)
    bias = (rng.standard_normal(N) * 0.1).astype(np.float32)
    return c, cq, sw, sx, bias


def _run_exact(M, K, N, ks, dtype, with_bias, seed=0):
    c, cq, sw, sx, bias = _exact_case(M, K, N, seed)
    wp = wm.pack(cq)
    packed = prepack_gpu(wp, K, N)
    codes = torch.from_numpy(c).to(torch.float8_e4m3fn).view(torch.uint8).to(DEV)
    tb = torch.from_numpy(bias).to(dtype).to(DEV) if with_bias else None
    out = mm_gpu(codes, torch.from_numpy(sx).to(DEV), packed, torch.from_numpy(sw).to(DEV), tb, dtype, ks, N)
    P = wm.block_sums(c, cq.astype(np.int32) - 8)
    kk = ks if ks > 0 else wm.plan_ks(M, K, N, _sms())
    want = wm.mm(P, sx, sw, None if tb is None else tb.float().cpu().numpy(), kk)
    return out, want, (c, cq, sw, sx, tb, P, kk)


def _as(want, dtype):
    return torch.from_numpy(want).to(dtype)


# ---- the GEMM bit for bit ---------------------------------------------------------------------------------------------------
EXACT_M = list(range(1, 17)) + [23, 64, 100, 129, 300, 2048]


@pytest.mark.parametrize("M", EXACT_M)
def test_mm_bit_exact_every_plan(M):
    K, N = 2048, 256
    for ks in (1, 2, 4, 8, 0):
        for dtype, with_bias in ((torch.float16, True), (torch.bfloat16, False), (torch.bfloat16, True)):
            out, want, _ = _run_exact(M, K, N, ks, dtype, with_bias, seed=M)
            assert torch.equal(out.cpu(), _as(want, dtype)), (M, ks, dtype, with_bias)


def test_mm_bit_exact_wide_layers():
    for M, K, N, ks in ((1, 14336, 4096, 0), (5, 4096, 14336, 0), (33, 65536, 128, 8)):
        out, want, _ = _run_exact(M, K, N, ks, torch.bfloat16, True, seed=K)
        assert torch.equal(out.cpu(), _as(want, torch.bfloat16)), (M, K, N)


def test_negative_controls_are_caught():
    """Each wrong ingredient changes the mirror's output, so the bit-exact comparisons would catch it."""
    M, K, N, ks, dtype = 12, 1024, 256, 2, torch.float16
    out, want, (c, cq, sw, sx, tb, P, kk) = _run_exact(M, K, N, ks, dtype, True, seed=5)
    got = out.cpu()
    assert torch.equal(got, _as(want, dtype))
    b = tb.float().cpu().numpy()
    wrong = {
        "s_w shifted by one group": wm.mm(P, sx, np.roll(sw, 1, axis=0), b, kk),
        "neighbouring token's s_x": wm.mm(P, np.roll(sx, 1), sw, b, kk),
        "last k-block dropped": wm.mm(P[:-1], sx, sw[:-1], b, kk),
    }
    sq = cq.copy()
    sq[:, [0, 1]] = sq[:, [1, 0]]
    sq[:, 0] = (sq[:, 0] + 1) % 16  # two nibbles swapped (made unequal) in every feature's first word
    sq[:, 1] = (sq[:, 1] + 3) % 16
    wrong["two nibbles swapped"] = wm.mm(wm.block_sums(c, sq.astype(np.int32) - 8), sx, sw, b, kk)
    for what, w in wrong.items():
        assert not torch.equal(got, _as(w, dtype)), what


# ---- random data: the float64 bound -------------------------------------------------------------------------------------
def test_random_data_within_float64_bound():
    worst = 0.0
    rng = np.random.default_rng(3)
    for M, K, N in ((1, 4096, 1024), (16, 4096, 512), (64, 14336, 256), (300, 1024, 4096), (2048, 4096, 128)):
        for dtype in (torch.float16, torch.bfloat16):
            x = torch.from_numpy(rng.standard_normal((M, K)).astype(np.float32) * 2).to(dtype).to(DEV)
            codes, sx = quantize_gpu(x)
            cq = rng.integers(0, 16, size=(N, K)).astype(np.uint8)
            sw = (rng.uniform(0.5, 1.5, size=(K // 128, N)) / (8 * K ** 0.5)).astype(np.float32)
            out = mm_gpu(codes, sx, prepack_gpu(wm.pack(cq), K, N), torch.from_numpy(sw).to(DEV), None, dtype, 0, N)
            c = codes.cpu().view(torch.float8_e4m3fn).double().numpy()
            q = cq.astype(np.float64) - 8
            s = sx.cpu().double().numpy()
            swk = np.repeat(sw.astype(np.float64), 128, axis=0)  # [K, N]
            ref = (c @ (q.T * swk)) * s[:, None]
            mag = (np.abs(c) @ (np.abs(q).T * swk)) * s[:, None]
            bound = EPS[dtype] * np.abs(ref) + 2.0 ** -24 + 2.0 ** -10 * mag
            err = np.abs(out.double().cpu().numpy() - ref)
            worst = max(worst, float((err / bound).max()))
            assert np.all(err <= bound), (M, K, N, dtype)
    print(f"worst error / bound: {worst:.3f}")


# ---- the layer ------------------------------------------------------------------------------------------------------------
def _module(K, N, seed, bias=None, adapter=None, dtype=torch.bfloat16):
    rng = np.random.default_rng(seed)
    wp = wm.pack(rng.integers(0, 16, size=(N, K)).astype(np.uint8))
    ws = torch.from_numpy(rng.uniform(0.5, 1.5, size=(N, K // 128)).astype(np.float32) / (8 * K ** 0.5)).to(dtype)
    return B200W4Fp8Linear.from_checkpoint_tensors(torch.from_numpy(wp), ws, weight_shape=torch.tensor([N, K]),
                                                   bias=bias, device=DEV, adapter=adapter), wp, ws


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_forward_equals_quantise_then_mm(dtype):
    K, N = 4096, 1024
    bias = torch.randn(N).to(dtype)
    m, _, _ = _module(K, N, seed=1, bias=bias)
    for M in (1, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 300, 2048):
        x = torch.randn(M, K, device=DEV).to(dtype)
        codes, sx = quantize_gpu(x)
        want = mm_gpu(codes, sx, m.packed, m.s_w, bias.to(DEV), dtype, 0, N)
        assert torch.equal(m(x), want), (M, dtype)


@pytest.mark.parametrize("name", ["bf_512_128_1", "bf_1024_128_48", "f16_512_256_48", "f16_512_128_1"])
def test_fixture_against_compressed_tensors(name):
    z = np.load(FIX)
    dtype = torch.bfloat16 if name.startswith("bf") else torch.float16

    def t(key):
        a = z[f"{name}.{key}"]
        return torch.from_numpy(a.view(np.int16)).view(torch.bfloat16) if a.dtype == np.uint16 else torch.from_numpy(a)

    wp, ws = t("weight_packed"), t("weight_scale")
    W = wm.table_weight(z[f"{name}.dq_table"], wm.unpack(z[f"{name}.weight_packed"]))
    W = torch.from_numpy(W.view(np.int16)).view(torch.bfloat16) if W.dtype == np.uint16 else torch.from_numpy(W)
    m = B200W4Fp8Linear.from_checkpoint_tensors(wp, ws, weight_shape=t("weight_shape"), device=DEV)
    assert torch.equal(m.dequantize_weight(dtype=dtype).cpu(), W)
    x = t("x").to(DEV)
    y = m(x).double().cpu().numpy()
    xd = x.double().cpu().numpy()
    Wd = W.double().numpy()
    # one e4m3 step (2^-3 relative, or the subnormal step 2^-9 s_x) per activation code, and the rounding of W to T
    sx = np.abs(xd).max(axis=1, keepdims=True) / 448
    dx = 2.0 ** -3 * np.abs(xd) + 2.0 ** -9 * sx
    bound = dx @ np.abs(Wd) + EPS[dtype] * (np.abs(xd) @ np.abs(Wd)) + EPS[dtype] * np.abs(z[f"{name}.y"]) + 1e-6
    assert np.all(np.abs(y - z[f"{name}.y"]) <= bound), name


def test_module_3d_non_contiguous_empty_deterministic():
    K, N = 1024, 640
    m, _, _ = _module(K, N, seed=3, bias=torch.randn(N).to(torch.bfloat16))
    assert m.list_buffers() and all(t.is_cuda for t in m.list_buffers())
    for dtype in (torch.float16, torch.bfloat16):
        x = torch.randn(14, K, device=DEV).to(dtype).reshape(2, 7, K)
        y = m(x)
        assert y.shape == (2, 7, N) and torch.equal(y.reshape(14, N), m(x.reshape(14, K)))
        xt = torch.randn(K, 12, device=DEV).to(dtype).t()  # non-contiguous
        assert torch.equal(m(xt), m(xt.contiguous()))
        assert m(torch.empty(0, K, dtype=dtype, device=DEV)).shape == (0, N)
        assert m(torch.empty(3, 0, K, dtype=dtype, device=DEV)).shape == (3, 0, N)
        x = torch.randn(700, K, device=DEV).to(dtype)
        assert torch.equal(m(x), m(x))


def test_module_lora():
    K, N, r = 1024, 512, 16
    g = torch.Generator().manual_seed(4)
    A = (torch.randn(K, r, generator=g) * 0.05).to(torch.float16)
    B = (torch.randn(r, N, generator=g) * 0.05).to(torch.float16)
    base, _, _ = _module(K, N, seed=31)
    m, _, _ = _module(K, N, seed=31, adapter=Lora(lora_A=A, lora_B=B))
    for dtype in (torch.float16, torch.bfloat16):
        for M in (1, 33, 300):
            x = torch.randn(1, M, K, device=DEV).to(dtype)
            want = base(x).reshape(M, N) + (x.reshape(M, K) @ A.to(DEV, dtype)) @ B.to(DEV, dtype)
            assert torch.equal(m(x).reshape(M, N), want), (dtype, M)


def test_cuda_graph_replay_equals_eager():
    K, N = 4096, 1024
    m, _, _ = _module(K, N, seed=21, bias=torch.randn(N).half())
    for dtype in (torch.float16, torch.bfloat16):
        for M in (1, 8, 16, 129):
            xs = torch.randn(M, K, device=DEV).to(dtype)
            m(xs)  # warm-up outside the capture (tensor-map cache, shared-memory opt-in)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                ys = m(xs)
            for _ in range(2):
                xs.copy_(torch.randn(M, K, device=DEV).to(dtype))
                g.replay()
                torch.cuda.synchronize()
                assert torch.equal(ys, m(xs)), (dtype, M)


# ---- a Llama-shaped checkpoint from the fixture tensors -------------------------------------------------------------------
def test_llama_checkpoint_from_fixture(tmp_path):
    from safetensors.torch import save_file

    from gptqmodel_b200.loader import load_w4afp8_linears

    z = np.load(FIX)

    def t(name, key):
        a = z[f"{name}.{key}"]
        return torch.from_numpy(a.view(np.int16)).view(torch.bfloat16) if a.dtype == np.uint16 else torch.from_numpy(a)

    names = {"self_attn.q_proj": "bf_1024_128_48", "self_attn.o_proj": "bf_512_128_1",
             "mlp.gate_proj": "bf_1024_128_48", "mlp.down_proj": "bf_512_128_1"}
    tensors = {}
    for n, case in names.items():
        for key in ("weight_packed", "weight_scale", "weight_shape"):
            tensors[f"model.layers.0.{n}.{key}"] = t(case, key).contiguous()
    tensors["lm_head.weight"] = torch.zeros(128, 512, dtype=torch.bfloat16)
    cfg = {"quant_method": "compressed-tensors", "format": "pack-quantized", "ignore": ["lm_head", "re:.*o_proj$"],
           "config_groups": {"group_0": {"targets": ["Linear"], "format": "pack-quantized",
                                         "weights": {"num_bits": 4, "type": "int", "symmetric": True,
                                                     "strategy": "group", "group_size": 128, "dynamic": False,
                                                     "actorder": None},
                                         "input_activations": {"num_bits": 8, "type": "float", "symmetric": True,
                                                               "strategy": "token", "dynamic": True}}}}
    with open(tmp_path / "config.json", "w") as f:
        json.dump({"model_type": "llama", "quantization_config": cfg}, f)
    save_file(tensors, str(tmp_path / "model.safetensors"))
    mods = load_w4afp8_linears(str(tmp_path), device=DEV)
    assert sorted(mods) == ["model.layers.0.mlp.down_proj", "model.layers.0.mlp.gate_proj",
                            "model.layers.0.self_attn.q_proj"]
    for n, m in mods.items():
        case = names[n.split("layers.0.")[1]]
        ref = B200W4Fp8Linear.from_checkpoint_tensors(t(case, "weight_packed"), t(case, "weight_scale"), device=DEV)
        assert torch.equal(m.packed, ref.packed) and torch.equal(m.s_w, ref.s_w)
        x = t(case, "x").to(DEV)
        assert torch.equal(m(x), ref(x)), n


# ---- MoE experts over the module: the per-expert loop ---------------------------------------------------------------------
def test_moe_experts_loop_equals_module_calls():
    from gptqmodel_b200 import moe

    E, H, I, T, top_k = 4, 1024, 512, 24, 2
    mods = lambda seed, K, N: [_module(K, N, seed=seed + e)[0] for e in range(E)]  # noqa: E731
    w1, w3, w2 = mods(100, H, I), mods(200, H, I), mods(300, I, H)
    blk = moe.MoEExperts(w1, w3, w2)
    assert blk._stack is None  # the per-expert loop
    with pytest.raises(ValueError, match="W4AFP8"):
        moe.MoEExperts(w1, w3, w2, grouped=True)
    g = torch.Generator().manual_seed(7)
    ids = torch.stack([torch.randperm(E, generator=g)[:top_k] for _ in range(T)]).to(DEV)
    wts = torch.softmax(torch.randn(T, top_k, generator=g), -1).to(DEV)
    for dtype in (torch.float16, torch.bfloat16):
        x = torch.randn(T, H, device=DEV).to(dtype)
        y = blk(x, ids, wts).double()
        want = torch.zeros(T, H, dtype=torch.float64, device=DEV)
        for t in range(T):
            for j in range(top_k):
                e = int(ids[t, j])
                xt = x[t:t + 1]
                h = torch.nn.functional.silu(w1[e](xt)) * w3[e](xt)
                want[t] += float(wts[t, j]) * w2[e](h)[0].double()
        assert torch.allclose(y, want, rtol=0, atol=float(4 * EPS[dtype] * want.abs().max())), dtype
