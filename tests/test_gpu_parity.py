"""GPU (B200): CUDA path vs the oracle, through the public module AND the raw C-ABI.  pytest -m gpu"""
import pytest
import torch

import oracle
from helpers import assert_close_rel, assert_layer_close, make_layer, oracle_forward, random_layer, ref_rounding_slack

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _module(layer, dtype=None):
    from gptqmodel_b200 import B200QuantLinear
    return B200QuantLinear.from_checkpoint_tensors(
        layer["qweight"], layer["qzeros"], layer["scales"], layer["g_idx"], layer["bits"], layer["group_size"],
        bias=layer["bias"], desc_act=layer["desc_act"], sym=layer["sym"], device=DEV, dtype=dtype)


def _abi_call(fn_name, mod, x, **kw):
    """Call b2q_gemv / b2q_gemm directly with raw pointers."""
    import gptqmodel_b200 as g
    M, K, N = x.shape[0], mod.in_features, mod.out_features
    out = torch.empty(M, N, dtype=x.dtype, device=x.device)
    code = 0 if x.dtype == torch.float16 else 1
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    st = torch.cuda.current_stream().cuda_stream
    if fn_name == "decode":
        g.check(g.lib.b2q_decode(p(x), p(mod.packed), p(mod._scales_for(x.dtype)), p(mod._zeros_dev), p(mod.perm),
                                 p(mod._bias_for(x.dtype)), p(out), M, K, N, mod.bits, mod.group_size, code,
                                 kw.get("ks", 0), kw.get("warps", 0), st), "b2q_decode")
    elif fn_name == "gemv":
        assert M == 1
        g.check(g.lib.b2q_gemv(p(x), p(mod.packed), p(mod._scales_for(x.dtype)), p(mod._zeros_dev), p(mod.perm),
                               p(mod._bias_for(x.dtype)), p(out), K, N, mod.bits, mod.group_size, code,
                               kw.get("ks", 0), kw.get("warps", 0), st), "b2q_gemv")
    else:
        nb = g.lib.b2q_workspace_bytes(max(M, 2), K, N, int(mod.perm is not None))
        ws = torch.empty(max(nb, 16), dtype=torch.uint8, device=x.device)
        g.check(g.lib.b2q_gemm(p(x), p(mod.packed), p(mod._scales_for(x.dtype)), p(mod._zeros_dev), p(mod.perm),
                               p(mod._bias_for(x.dtype)), p(out), M, K, N, mod.bits, mod.group_size, code,
                               p(ws), ws.numel(), st), "b2q_gemm")
    torch.cuda.synchronize()
    return out


# ---------------------------------------------------------------------------------------------------
def test_prepack_layout_bit_exact():
    """B2Q tiles hold exactly the checkpoint's codes.
    4-bit T4[K/64][N/16][32 lanes][4 words]: lane = 4g+t, word s, nibble p -> feature 16ft+g(+8 if p odd),
    k = 64kb + 16t + 4s + (2 if p&2) + (p>>2);  8-bit T8[K/32][N/32][2][32][4]: natural byte order."""
    for bits, desc in ((4, False), (4, True), (8, False), (8, True)):
        L = make_layer(256, 128, bits=bits, group_size=64, sym=False, desc_act=desc, seed=3)
        mod = _module(L)
        codes = oracle.unpack_qweight(L["qweight"], bits)  # [K, N]
        if mod.perm is not None:
            codes = codes[mod.perm[:256].cpu().long()]  # perm = [order | inverse] (ABI v3)
        K, N = 256, 128
        raw = torch.from_numpy(mod.packed.cpu().numpy().view("uint32").astype("int64"))
        got = torch.zeros(K, N, dtype=torch.int64)
        if bits == 4:
            raw = raw.reshape(K // 64, N // 16, 32, 4)  # [kb][ft][lane][word]
            for lane in range(32):
                g, t = lane >> 2, lane & 3
                for s_ in range(4):
                    for p_ in range(8):
                        k = torch.arange(K // 64) * 64 + 16 * t + 4 * s_ + (2 if p_ & 2 else 0) + (p_ >> 2)
                        n = torch.arange(N // 16) * 16 + g + (8 if p_ & 1 else 0)
                        got[k[:, None], n[None, :]] = (raw[:, :, lane, s_] >> (4 * p_)) & 0xF
        else:
            raw = raw.reshape(K // 32, N // 32, 2, 32, 4)  # [kc][nt][h][lane][word]
            for h in range(2):
                for j in range(4):
                    for b in range(4):
                        k = torch.arange(K // 32) * 32 + h * 16 + j * 4 + b
                        for lane in range(32):
                            n = torch.arange(N // 32) * 32 + lane
                            got[k[:, None], n[None, :]] = (raw[:, :, h, lane, j] >> (8 * b)) & 0xFF
        assert torch.equal(got, codes.long()), (bits, desc)


def test_q4_reference_golden_vector_on_gpu(q4_golden):
    """The reference's own KAT (tests/test_q4_exllama_v2.py:32-87 + tests/q4_reference.py), GEMV and GEMM tiers."""
    torch.manual_seed(42)
    qweight = torch.randint(-100, 100, size=(128, 1024), dtype=torch.int32)
    scales = torch.zeros(8, 1024, dtype=torch.float16) + 0.002
    qzeros = torch.full((8, 128), 0x11111111, dtype=torch.int32)
    g_idx = torch.arange(1024, dtype=torch.int32) // 128
    x = torch.rand(1, 1, 1024, dtype=torch.float16)
    from gptqmodel_b200 import B200QuantLinear
    mod = B200QuantLinear.from_checkpoint_tensors(qweight, qzeros, scales, g_idx, 4, 128, device=DEV)
    ref = torch.tensor(q4_golden["reference"], dtype=torch.float16)
    y = mod(x.to(DEV))[0][0].cpu()
    assert torch.allclose(y, ref, rtol=3e-5, atol=2e-2)
    assert (y.float() - ref.float()).abs().max().item() < 8e-3
    y2 = _abi_call("gemm", mod, x.to(DEV).reshape(1, 1024))[0].cpu()
    assert torch.allclose(y2, ref, rtol=3e-5, atol=2e-2)
    assert (y2.float() - ref.float()).abs().max().item() < 8e-3


def test_reference_generated_cases(ref_cases):
    """Fixtures produced by the reference's TorchLinear (tests/golden/make_golden.py)."""
    from gptqmodel_b200 import B200QuantLinear
    for name in ref_cases.names():
        m = ref_cases.meta[name]
        mod = B200QuantLinear.from_checkpoint_tensors(
            ref_cases.get(name, "qweight"), ref_cases.get(name, "qzeros"), ref_cases.get(name, "scales"),
            ref_cases.get(name, "g_idx"), m["bits"], m["group_size"], bias=ref_cases.get(name, "bias"),
            desc_act=m["desc_act"], sym=m["sym"], device=DEV)
        x = ref_cases.get(name, "x").to(DEV)
        y = mod(x)
        # reference CPU fp16 matmul differs from fp32-accumulate by <= ~1 fp16 ulp
        assert torch.allclose(y.float().cpu(), ref_cases.get(name, "y_fp16").float(), rtol=2e-3, atol=2e-3), name
        yo = oracle.forward(x.cpu(), ref_cases.get(name, "qweight"), ref_cases.get(name, "qzeros"),
                            ref_cases.get(name, "scales"), ref_cases.get(name, "g_idx"), m["bits"],
                            bias=ref_cases.get(name, "bias"))
        assert_close_rel(y, yo, 1e-3, name)
        Wr = oracle.dequantize_weight(ref_cases.get(name, "qweight"), ref_cases.get(name, "qzeros"),
                                      ref_cases.get(name, "scales"), ref_cases.get(name, "g_idx"), m["bits"])
        for i in range(x.shape[0]):  # every row through the M = 1 tier as well (scale-once tiers: + rounding noise)
            yi = mod(x[i:i + 1])
            assert_close_rel(yi, yo[i:i + 1], 1e-3, f"{name} row {i}", slack=ref_rounding_slack(Wr, x[i:i + 1].cpu()))
        ybf = mod(x.to(torch.bfloat16))
        assert torch.allclose(ybf.float().cpu(), ref_cases.get(name, "y_bf16"), rtol=2e-2, atol=3e-2), name


CASES = [
    # K, N, bits, group, sym, desc_act, bias
    (256, 512, 4, 128, True, False, False),
    (256, 512, 4, -1, True, False, False),
    (256, 512, 4, 64, True, True, False),
    (256, 512, 4, 128, True, True, True),
    (1024, 1024, 4, 32, False, False, True),
    (1024, 1024, 4, 64, False, True, False),
    (2048, 1024, 4, 128, False, False, False),
    (512, 256, 8, 128, True, False, False),
    (512, 256, 8, 32, False, True, True),
    (1024, 512, 8, 64, False, False, False),
    (4096, 4096, 4, 128, True, False, False),   # BASELINE configs[0] shape
    (4096, 1024, 4, 128, True, True, False),    # k/v proj with act-order (config 3)
    (3584, 4096, 4, 64, False, False, False),   # Mixtral TP-4 w2 shard, g64 asym (config 5)
    (1024, 96, 4, 128, True, False, False),     # N not a multiple of the 128-feature GEMM tile
    (1024, 512, 4, 32, True, True, False),      # 4-bit g32 + act-order: no decode tier, M = 1 needs the x[perm] workspace
    (1088, 160, 4, 64, False, False, True),     # K % 128 != 0 and a ragged last feature tile
]


@pytest.mark.parametrize("K,N,bits,gs,sym,desc,bias", CASES)
def test_forward_matches_oracle_fp16(K, N, bits, gs, sym, desc, bias):
    L = make_layer(K, N, bits=bits, group_size=gs, sym=sym, desc_act=desc, bias=bias, seed=42)
    mod = _module(L)
    gen = torch.Generator().manual_seed(43)
    for M in (1, 2, 7, 12, 20, 32, 64, 128, 129, 300):
        x = (torch.randn(M, K, generator=gen) * 0.5).to(torch.float16)
        out = mod(x.to(DEV))
        assert out.dtype == torch.float16 and out.shape == (M, N)
        assert_layer_close(out, L, x, 1e-3, f"M={M}")
    # every tier directly through the C-ABI on the same rows
    x8 = (torch.randn(8, K, generator=gen) * 0.5).to(torch.float16)
    ref8 = oracle_forward(L, x8)
    x1, ref1 = x8[:1].contiguous(), ref8[:1]
    assert_close_rel(_abi_call("gemm", mod, x1.to(DEV)), ref1, 1e-3, "abi gemm M=1")
    assert_close_rel(_abi_call("gemm", mod, x8.to(DEV)), ref8, 1e-3, "abi gemm M=8")
    has_m1_tier = (bits == 8 and K % 128 == 0) or (bits == 4 and K % 128 == 0 and gs in (64, 128, -1))
    # the scale-once tiers (decode / GEMV) against the per-weight-rounded oracle: + the reference's rounding noise
    W = oracle.dequantize_weight(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], bits)
    slack8 = ref_rounding_slack(W, x8)
    if has_m1_tier:
        assert_close_rel(_abi_call("gemv", mod, x1.to(DEV)), ref1, 1e-3, "abi gemv", slack=slack8[:1])
        combos = ((1, 8), (2, 4), (4, 8), (8, 4)) if bits == 4 else ((1, 8), (2, 4), (4, 2), (8, 1), (16, 4))
        for ks, warps in combos:
            if ks <= K // 128:
                assert_close_rel(_abi_call("gemv", mod, x1.to(DEV), ks=ks, warps=warps), ref1, 1e-3, f"ks={ks}",
                                 slack=slack8[:1])
    if bits == 4 and K % 128 == 0 and gs in (64, 128, -1):
        for M in (1, 2, 3, 5, 8):
            for ks, warps in ((0, 0), (1, 4), (2, 8), (4, 4), (8, 8)):
                if ks <= K // 128:
                    assert_close_rel(_abi_call("decode", mod, x8[:M].contiguous().to(DEV), ks=ks, warps=warps),
                                     ref8[:M], 1e-3, f"decode M={M} ks={ks} warps={warps}", slack=slack8[:M])


@pytest.mark.parametrize("K,N,bits,gs,sym,desc,bias", CASES[:10])
def test_forward_matches_oracle_bf16(K, N, bits, gs, sym, desc, bias):
    L = make_layer(K, N, bits=bits, group_size=gs, sym=sym, desc_act=desc, bias=bias, seed=7)
    L["scales"] = L["scales"].to(torch.bfloat16)  # model loaded in bf16: scales become bf16 (single rounding)
    if bias:
        L["bias"] = L["bias"].to(torch.bfloat16)
    mod = _module(L, dtype=torch.bfloat16)
    gen = torch.Generator().manual_seed(44)
    for M in (1, 5, 130):
        x = (torch.randn(M, K, generator=gen) * 0.5).to(torch.bfloat16)
        ref = oracle.forward(x, L["qweight"], L["qzeros"], L["scales"], L["g_idx"], bits, bias=L["bias"])
        out = mod(x.to(DEV))
        assert out.dtype == torch.bfloat16
        assert_close_rel(out, ref, 1.6e-2, f"bf16 M={M}")  # 2 bf16 ulp (ulp = 7.8e-3); the reference budgets 6e-3..8e-3
        # ABSOLUTE on |y|~1 with rtol 0.15 (tests/kernels/test_gptq.py:353-360)


SMALL_BATCH_CASES = [
    # K, N, bits, group, sym, desc_act, bias   (VERDICT r01 next #3: g32/g64/g128, sym/asym, 4/8-bit at every M below)
    (1024, 512, 4, 32, True, False, False), (1024, 512, 4, 32, False, False, True),
    (1024, 512, 4, 64, True, False, False), (2048, 384, 4, 64, False, True, False),
    (1024, 512, 4, 128, True, False, True), (2048, 384, 4, 128, False, False, False),
    (1024, 512, 8, 32, True, False, False), (1024, 512, 8, 32, False, False, True),
    (1024, 512, 8, 64, False, False, False), (2048, 384, 8, 128, True, True, False),
    (1024, 512, 8, 128, False, False, False), (512, 96, 4, -1, True, False, False),
]


@pytest.mark.parametrize("K,N,bits,gs,sym,desc,bias", SMALL_BATCH_CASES)
def test_small_batch_tier_matches_oracle(K, N, bits, gs, sym, desc, bias):
    """b2q_midm.cu (swapped wgmma operands + cluster split-K): every token-box width (16/32/64/128), partial boxes,
    every split-K cluster size, through the module and the raw ABI."""
    import gptqmodel_b200 as g
    import os
    L = make_layer(K, N, bits=bits, group_size=gs, sym=sym, desc_act=desc, bias=bias, seed=K + N + bits)
    mod = _module(L)
    gen = torch.Generator().manual_seed(45)
    xs = (torch.randn(128, K, generator=gen) * 0.5).to(torch.float16)
    ref = oracle_forward(L, xs)
    for M in (9, 16, 17, 33, 64, 127, 128):
        assert_close_rel(mod(xs[:M].to(DEV)), ref[:M], 1e-3, f"M={M}")
    try:
        for ks in (1, 2, 4, 8):
            os.environ["B2Q_MIDM_KS"] = str(ks)
            g.lib.b2q_debug_reload_env()
            for M in (5, 33, 100):
                assert_close_rel(_abi_call("gemm", mod, xs[:M].contiguous().to(DEV)), ref[:M], 1e-3, f"ks={ks} M={M}")
    finally:
        os.environ.pop("B2Q_MIDM_KS", None)
        g.lib.b2q_debug_reload_env()
    # determinism (no atomics: the split-K partials are summed in rank order)
    a = mod(xs[:40].to(DEV))
    assert torch.equal(a, mod(xs[:40].to(DEV)))
    # the round-1 padded single-CTA tier (B2Q_MIDM=0) computes the same exact-dequant products: agree within fp32
    # summation order
    try:
        os.environ["B2Q_MIDM"] = "0"
        g.lib.b2q_debug_reload_env()
        old = _abi_call("gemm", mod, xs[:40].contiguous().to(DEV))
    finally:
        os.environ.pop("B2Q_MIDM", None)
        g.lib.b2q_debug_reload_env()
    assert_close_rel(a, old, 1e-3, "midm vs padded tier")


def test_batched_and_empty_shapes():
    L = make_layer(256, 128, seed=5, bias=True)
    mod = _module(L)
    x = (torch.randn(2, 3, 256) * 0.5).to(torch.float16)
    out = mod(x.to(DEV))
    assert out.shape == (2, 3, 128)
    assert_close_rel(out.reshape(6, 128), oracle_forward(L, x.reshape(6, 256)), 1e-3)
    e = mod(torch.zeros(0, 256, dtype=torch.float16, device=DEV))  # qlinear/marlin.py:308-309
    assert e.shape == (0, 128)
    xs = torch.randn(4, 512, device=DEV).to(torch.float16)[:, ::2]  # non-contiguous input
    assert_close_rel(mod(xs), oracle_forward(L, xs.cpu()), 1e-3)


def test_nonuniform_g_idx_is_served():
    """One row moved to another group (63 / 65 rows instead of 64 / 64): round 1 refused such a layer; it is now regrouped
    (gptqmodel_b200/layouts.py::regroup) and must match the oracle, which walks g_idx directly like the reference."""
    L = make_layer(256, 128, group_size=64, seed=5)
    gi = L["g_idx"].clone()
    gi[0] = 3  # group 0 loses a row, group 3 gains one
    L["g_idx"] = gi
    mod = _module(L)
    assert mod._gather is not None and mod.perm is None
    for M in (1, 3, 40, 200):
        x = (torch.randn(M, 256, generator=torch.Generator().manual_seed(M)) * 0.5).to(torch.float16).to(DEV)
        assert_layer_close(mod(x), L, x, 1e-3, f"non-uniform g_idx M={M}")


@pytest.mark.parametrize("K,N", [(4096, 14336), (14336, 4096), (4096, 4096), (4096, 1024)])
def test_llama3_8b_shapes_full_size(K, N):
    """BASELINE configs[1] shapes at full size: oracle evaluated on the GPU in fp32 from the same rounded W."""
    L = random_layer(K, N, bits=4, group_size=128, sym=True, seed=K + N)
    mod = _module(L)
    W = oracle.dequantize_weight(L["qweight"].to(DEV), L["qzeros"].to(DEV), L["scales"].to(DEV),
                                 L["g_idx"].to(DEV), 4).float()
    torch.manual_seed(1)
    x = (torch.randn(2048, K, device=DEV) * 0.5).to(torch.float16)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ref = (x.float() @ W).to(torch.float16)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    out = mod(x)
    assert_close_rel(out, ref, 1e-3, "prefill M=2048")
    out1 = mod(x[5:6])
    assert_close_rel(out1, ref[5:6], 1e-3, "decode M=1", slack=ref_rounding_slack(W.half(), x[5:6]).cpu())
    for m in (16, 48, 128):  # small-batch tier at full size
        assert_close_rel(mod(x[:m]), ref[:m], 1e-3, f"small batch M={m}")
    # size-independent properties: determinism and tier agreement
    assert torch.equal(mod(x[5:6]), out1)
    assert torch.equal(mod(x), out)
    # linearity: scaling the input by 2 is exact in every operand, so only the tile shape (M=8 uses the
    # 128-row tile, M=2048 the 256-row one) and the accumulation order may differ: <= 1 fp16 ulp
    lin = mod((x[:8] * 2).to(torch.float16))
    assert_close_rel(lin, out[:8] * 2, 1e-3, "linearity")
    assert_close_rel(mod(x[:8]), out[:8], 1e-3, "tile-shape agreement")


def test_cuda_graph_capture_and_stream():
    L = make_layer(1024, 512, seed=9)
    mod = _module(L)
    x1 = (torch.randn(1, 1024, device=DEV) * 0.5).to(torch.float16)
    x8 = (torch.randn(8, 1024, device=DEV) * 0.5).to(torch.float16)
    ref1, ref8 = mod(x1).clone(), mod(x8).clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            mod(x1), mod(x8)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y1 = mod(x1)
        y8 = mod(x8)
    x1.copy_(x1 * 0 + x1)  # same values, replays must reproduce
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y1, ref1) and torch.equal(y8, ref8)


def _same_k_split(M, K, N_single, N_fused):
    """True if the decode planner cuts K identically (split-K ranks, warps per tile group, quads per CTA) for a single
    layer of width N_single and for the fused launch of total width N_fused."""
    import ctypes
    import os
    from gptqmodel_b200 import _lib as g
    ver = 2 if os.environ.get("B2Q_DECODE_V2") == "1" else 1
    a, b = (ctypes.c_int * 8)(), (ctypes.c_int * 8)()
    if g.lib.b2q_debug_decode_plan(ver, M, K, N_single, 0, 0, a) != 0 or \
            g.lib.b2q_debug_decode_plan(ver, M, K, N_fused, 0, 0, b) != 0:
        return False
    return (a[1], a[3], a[4]) == (b[1], b[3], b[4])


@pytest.mark.parametrize("sym,gs,bias", [(True, 128, False), (False, 64, True), (True, -1, False)])
def test_sibling_fusion_bit_identical(sym, gs, bias):
    """q/k/v-style siblings in ONE launch (b2q_decode_multi) == three separate forwards, bit for bit."""
    from gptqmodel_b200 import fuse_siblings
    K = 1024
    Ls = [make_layer(K, n, group_size=gs, sym=sym, bias=bias, seed=20 + i) for i, n in enumerate((1024, 256, 512))]
    mods = [_module(L) for L in Ls]
    gen = torch.Generator().manual_seed(3)
    for M in (1, 3, 8):
        x = (torch.randn(M, K, generator=gen) * 0.5).to(torch.float16).to(DEV)
        sep = [m(x).clone() for m in mods]
        assert fuse_siblings(mods)
        fused = [m(x) for m in mods]          # first call launches for all three, the others pick up
        for a, b, L in zip(sep, fused, Ls):
            # bit-identical whenever the fused launch splits K the same way as the single launches (the fp32 partial
            # sums are then added in the same order); otherwise only the summation order differs
            if _same_k_split(M, K, L["N"], sum(l["N"] for l in Ls)):
                assert torch.equal(a, b)
            else:
                assert_close_rel(b, a, 1e-3, f"fused vs separate M={M}")
            assert_layer_close(b, L, x, 1e-3, f"fused M={M}")
        # a different input invalidates the parked outputs; calling only one sibling still works
        x2 = (x * 0.5).to(torch.float16)
        assert torch.equal(mods[1](x2), mods[1].__class__.forward(mods[1], x2))
        big = (torch.randn(64, K, generator=gen) * 0.5).to(torch.float16).to(DEV)   # 9..128: per module (small-batch tier)
        assert_close_rel(mods[0](big), oracle_forward(Ls[0], big.cpu()), 1e-3, "fused M=64")
        pre = (torch.randn(300, K, generator=gen) * 0.5).to(torch.float16).to(DEV)  # > 128: ONE persistent prefill launch
        for m_, L_ in zip(mods, Ls):
            assert_close_rel(m_(pre), oracle_forward(L_, pre.cpu()), 1e-3, "fused prefill M=300")
        for m in mods:
            m._siblings = None
    # refused combinations
    ao = _module(make_layer(K, 256, group_size=64, desc_act=True, seed=30))
    assert not fuse_siblings([mods[0], ao])
    other_k = _module(make_layer(512, 256, seed=31))
    assert not fuse_siblings([mods[0], other_k])


def test_sibling_fusion_with_shared_act_order():
    """q/k/v of a GPTQ act-order checkpoint share g_idx (same input Hessian): one decode launch gathers x[perm] once."""
    from gptqmodel_b200 import fuse_siblings
    K = 1024
    Ls = [make_layer(K, n, group_size=128, sym=True, desc_act=True, seed=61) for n in (512, 256)]
    assert torch.equal(Ls[0]["g_idx"], Ls[1]["g_idx"])
    mods = [_module(L) for L in Ls]
    assert mods[0].perm is not None and fuse_siblings(mods)
    gen = torch.Generator().manual_seed(4)
    for M in (1, 5, 260):  # decode launch / prefill launch (x[:, perm] gathered once for both siblings)
        x = (torch.randn(M, K, generator=gen) * 0.5).to(torch.float16)
        for m, L in zip(mods, Ls):
            assert_layer_close(m(x.to(DEV)), L, x, 1e-3, f"act-order fused M={M}")
    other = _module(make_layer(K, 256, group_size=128, sym=True, desc_act=True, seed=62))  # a different permutation
    for m in mods:
        m._siblings = None
    assert not fuse_siblings([mods[0], other])


@pytest.mark.parametrize("K,N,kind", [
    (8192, 1024, "q_proj column shard"), (1024, 8192, "o_proj row shard"),
    (8192, 3584, "gate/up column shard"), (3584, 8192, "down_proj row shard"),
])
def test_llama3_70b_tp8_shard_shapes(K, N, kind):
    """BASELINE configs[3]: the per-rank QuantLinear shapes of Llama-3-70B under TP-8, decode + prefill."""
    L = random_layer(K, N, bits=4, group_size=128, sym=True, seed=K * 7 + N)
    mod = _module(L)
    W = oracle.dequantize_weight(L["qweight"].to(DEV), L["qzeros"].to(DEV), L["scales"].to(DEV),
                                 L["g_idx"].to(DEV), 4).float()
    torch.manual_seed(2)
    x = (torch.randn(300, K, device=DEV) * 0.5).to(torch.float16)
    ref = (x.float() @ W).to(torch.float16)
    assert_close_rel(mod(x), ref, 1e-3, f"{kind} M=300")
    sl = ref_rounding_slack(W.half(), x[:6]).cpu()
    assert_close_rel(mod(x[:1]), ref[:1], 1e-3, f"{kind} M=1", slack=sl[:1])
    assert_close_rel(mod(x[:6]), ref[:6], 1e-3, f"{kind} M=6", slack=sl)


def test_act_order_full_size_llama_layer():
    """BASELINE configs[2]: desc_act=True (random g_idx) on a full-size Llama-3-8B projection, decode and prefill."""
    K, N = 4096, 4096
    L = make_layer(K, N, bits=4, group_size=128, sym=True, desc_act=True, seed=77)
    mod = _module(L)
    assert mod.perm is not None
    gen = torch.Generator().manual_seed(5)
    x = (torch.randn(257, K, generator=gen) * 0.5).to(torch.float16)
    ref = oracle_forward(L, x)
    assert_close_rel(mod(x.to(DEV)), ref, 1e-3, "act-order M=257")
    assert_layer_close(mod(x[:1].to(DEV)), L, x[:1], 1e-3, "act-order M=1")
    assert_layer_close(mod(x[:8].to(DEV)), L, x[:8], 1e-3, "act-order M=8")
