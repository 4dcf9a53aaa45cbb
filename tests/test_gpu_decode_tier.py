"""The decode tier (4-bit weights, 1..8 tokens) at real launch shapes against a float64 oracle.  pytest -m gpu

Launches with more 32-feature tiles than the GPU has SMs (fused q|k|v and gate|up, single layers wider than 132 tiles)
run on decode2_kernel (b2q_decode2.cu) with one 16-warp group and no split-K; a launch whose decode2 plan does not fit
shared memory falls back to decode_kernel (b2q_decode.cu).  Each case records the kernel and instantiation that actually
ran (torch.profiler), and test_decode_tier_coverage checks that the cases reached every dense instantiation of
decode2_kernel with and without act-order, and the fallback.

Oracle.  The decode tier applies the scale once per (group, feature) to an exact integer dot product, so its reference is
the exact arithmetic: W = (q - z) * s in float64 with s the scale as the kernel reads it (the checkpoint's fp16 scale
converted to the run dtype), v = x @ W in float64, rounded once to the run dtype.  Kernel and oracle then differ by the
fp32 accumulation of the dot products (relative ~2^-24 * sqrt(K)) and by at most one rounding of the output across a
boundary: at most 2^-10 |y| in fp16 and 2^-7 |y| in bf16, inside rel = 1e-3 and 8e-3 of assert_close_rel.  The oracle is
evaluated on the GPU in blocks of output columns.  The kernel adds a bias after that rounding, RN(RN(v) + b), like the
reference; a one-ulp difference in RN(v) can then grow into two ulps of the sum, so the bias is checked exactly on the
kernel's own RN(v) (the same launch without bias), and RN(v) against the oracle.
"""
import os

import pytest
import torch

import oracle
from helpers import assert_close_rel, decode_k_split, decode_kernels_launched, random_layer, same_k_split

pytestmark = pytest.mark.gpu

DEV = "cuda"
F16, BF16 = torch.float16, torch.bfloat16
REL = {F16: 1e-3, BF16: 8e-3}
DTN = {F16: "__half", BF16: "__nv_bfloat16"}
MS = tuple(range(1, 9))


# ------------------------------------------------------------------------------------------------------------------------
# layers, oracle, module plumbing
# ------------------------------------------------------------------------------------------------------------------------
def _layers(K, Ns, dt, sym, gs, act, bias, seed):
    """Random 4-bit layers on the device sharing K (siblings).  act: one shuffled g_idx (arange(K) // gs)[randperm] for
    all of them, as the siblings of an act-order checkpoint share it.  bias: per layer, randn * 0.1 in dt."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    gi = None
    if act:
        perm = torch.randperm(K, generator=gen, device=DEV)
        gi = (torch.arange(K, dtype=torch.int32, device=DEV) // gs)[perm].to(torch.int32)
    Ls = []
    for i, N in enumerate(Ns):
        L = random_layer(K, N, bits=4, group_size=gs, sym=sym, seed=seed * 7 + i, device=DEV)
        if gi is not None:
            L["g_idx"], L["desc_act"] = gi.clone(), True
        if bias[i]:
            L["bias"] = (torch.randn(N, generator=gen, device=DEV) * 0.1).to(dt)
        Ls.append(L)
    return Ls


def _module(L, dt):
    from gptqmodel_b200 import B200QuantLinear
    return B200QuantLinear.from_checkpoint_tensors(
        L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, L["group_size"], bias=L["bias"], desc_act=L["desc_act"],
        sym=L["sym"], device=DEV, dtype=dt)


def _dequant(L, dt, n0, n1, qzeros=None, scales=None):
    """float64 W[:, n0:n1] = (q - z) * s, s exact in dt."""
    qz = L["qzeros"] if qzeros is None else qzeros
    sc = L["scales"] if scales is None else scales
    return oracle.dequantize_weight(L["qweight"][:, n0:n1], qz[:, n0 // 8:n1 // 8],
                                    sc[:, n0:n1].to(dt).to(torch.float64), L["g_idx"], 4)


def decode_oracle(L, x, bias=None, block=4096, **perturb):
    """x [M, K] (dt) -> [M, N] in dt: RN(x @ W) in float64, then RN(. + bias).  perturb: qzeros= / scales= replacing
    the layer's tensors (negative controls)."""
    dt = x.dtype
    xd = x.to(torch.float64)
    out = torch.empty(x.shape[0], L["N"], dtype=dt, device=x.device)
    for n0 in range(0, L["N"], block):
        n1 = min(L["N"], n0 + block)
        out[:, n0:n1] = (xd @ _dequant(L, dt, n0, n1, **perturb)).to(dt)
    if bias is not None:
        out = (out.to(torch.float64) + bias.to(torch.float64)).to(dt)
    return out


def _inputs(K, dt, seed):
    """Two sets of 8 token rows: randn * 0.5, and the same with 8 channels at 30x the others (a large sum_k x per group
    loads the (base + z) * sum_k x term of the fix-up, which cancels most of the raw accumulator)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(8, K, generator=gen, device=DEV) * 0.5
    xo = x.clone()
    ch = torch.randperm(K, generator=gen, device=DEV)[:8]
    xo[:, ch] *= 30
    return x.to(dt), xo.to(dt)


def _decode_multi(mods, x, biases):
    """b2q_decode_multi over the modules' weights with explicit bias pointers (None: that set has no bias)."""
    import ctypes
    import gptqmodel_b200 as g
    n, dt = len(mods), x.dtype
    M, K = x.shape
    outs = [torch.empty(M, m.out_features, dtype=dt, device=DEV) for m in mods]
    vp = ctypes.c_void_p * n
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    g.check(g.lib.b2q_decode_multi(
        x.data_ptr(), n, vp(*[m.packed.data_ptr() for m in mods]), vp(*[m._scales_for(dt).data_ptr() for m in mods]),
        vp(*[p(m._zeros_dev) for m in mods]), p(mods[0].perm), vp(*[p(b) for b in biases]), vp(*[o.data_ptr() for o in outs]),
        (ctypes.c_int * n)(*[m.out_features for m in mods]), M, K, 4, mods[0]._kgs, 0 if dt == F16 else 1,
        torch.cuda.current_stream().cuda_stream), "b2q_decode_multi")
    return outs


class _Env:
    """Sets decode switches for the duration of a block and restores the previous values (also on failure)."""

    def __init__(self, **kv):
        self.kv = kv

    def __enter__(self):
        import gptqmodel_b200 as g
        self.old = {k: os.environ.get(k) for k in self.kv}
        for k, v in self.kv.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
        g.lib.b2q_debug_reload_env()

    def __exit__(self, *exc):
        import gptqmodel_b200 as g
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        g.lib.b2q_debug_reload_env()
        return False


# ------------------------------------------------------------------------------------------------------------------------
# cases: (K, set widths, dtype, sym, group (-1: per channel), act-order, bias per set, token counts)
# ------------------------------------------------------------------------------------------------------------------------
QKV8B, GU8B = (4096, 1024, 1024), (14336, 14336)
CASES = {}
for _dt in (F16, BF16):
    _d = "fp16" if _dt == F16 else "bf16"
    for _sym in (True, False):
        for _gs in (64, 128, -1):
            CASES[f"llama3_8b_qkv-{_d}-{'sym' if _sym else 'asym'}-g{_gs}"] = (4096, QKV8B, _dt, _sym, _gs, False, (0, 0, 0), MS)
        for _gs in (64, 128):
            CASES[f"llama3_8b_qkv-{_d}-{'sym' if _sym else 'asym'}-g{_gs}-act"] = (4096, QKV8B, _dt, _sym, _gs, True, (0, 0, 0), MS)
    CASES[f"llama3_8b_gate_up-{_d}-sym-g128"] = (4096, GU8B, _dt, True, 128, False, (0, 0), MS)
    CASES[f"llama3_8b_gate_up-{_d}-sym-g128-act"] = (4096, GU8B, _dt, True, 128, True, (0, 0), MS)
    CASES[f"llama3_8b_gate_up-{_d}-asym-g64"] = (4096, GU8B, _dt, False, 64, False, (0, 0), MS)
    CASES[f"qwen25_7b_qkv_bias-{_d}-sym-g128"] = (3584, (3584, 512, 512), _dt, True, 128, False, (1, 1, 1), MS)
    CASES[f"one_quad-{_d}-asym-g128"] = (128, (8192,), _dt, False, 128, False, (0,), MS)
CASES["llama3_70b_tp8_gate_up-fp16-sym-g128"] = (8192, (3584, 3584), F16, True, 128, False, (0, 0), (1, 4, 8))
CASES["wide_4256-fp16-sym-g128-bias"] = (4096, (4256,), F16, True, 128, False, (1,), MS)
CASES["wide_4256-fp16-sym-g128"] = (4096, (4256,), F16, True, 128, False, (0,), MS)

SERVED = {}  # case -> {M: (kernel, dtype, asym, g64)} of the module call (filled by _run_case)


def _run_case(name):
    """Every token count of a case through the module (fused siblings for multi-set launches) and, for fused launches,
    through b2q_decode_multi with the middle set's bias dropped; oracle, determinism, instantiation and fused-vs-separate
    checks.  Returns {M: launched decode kernel}."""
    if name in SERVED:
        return SERVED[name]
    from gptqmodel_b200 import fuse_siblings
    K, Ns, dt, sym, gs, act, bias, Ms = CASES[name]
    rel = REL[dt]
    Ls = _layers(K, Ns, dt, sym, gs, act, bias, seed=list(CASES).index(name) + 11)
    mods = [_module(L, dt) for L in Ls]
    assert all((m.perm is not None) == act for m in mods)
    fused = len(mods) > 1
    if fused:
        assert fuse_siblings(mods)
    want = (DTN[dt], not sym, gs == 64)
    x, xo = _inputs(K, dt, seed=K + len(Ns))
    refs = {id(xs): [decode_oracle(L, xs) for L in Ls] for xs in (x, xo)}
    served = {}
    for M in Ms:
        for xs, tag in ((x, ""), (xo, " outliers")):
            xm = xs[:M].contiguous()
            ref = [r[:M] for r in refs[id(xs)]]
            if not tag:
                outs, ks = decode_kernels_launched(lambda: [m(xm).clone() for m in mods])
                assert len(ks) == 1 and ks[0][1:] == want, (name, M, ks)  # ONE launch, the instantiation of the layer
                served[M] = ks[0]
            else:
                outs = [m(xm).clone() for m in mods]
            again = [m(xm) for m in mods]
            assert all(torch.equal(a, b) for a, b in zip(outs, again)), f"{name} M={M}{tag}: not deterministic"
            # the same launch through b2q_decode_multi without bias against the oracle.  The bias is checked exactly on
            # the kernel's own RN(v): against the float64 oracle, RN(RN(v) + b) may sit one ulp of RN(v) plus one ulp
            # of the sum away (up to 2^-9 |y| in fp16), more than rel covers.
            plain = _decode_multi(mods, xm, [None] * len(mods))
            for i, (o, r) in enumerate(zip(plain, ref)):
                assert_close_rel(o, r, rel, f"{name} M={M} set {i}{tag}")
            with_bias = lambda v, b: v if b is None else (v.float() + b.float()).to(dt)  # noqa: E731
            for i, (o, v, m) in enumerate(zip(outs, plain, mods)):
                assert torch.equal(o, with_bias(v, m._bias_for(dt))), f"{name} M={M} set {i}{tag}: module != ABI"
            if fused:
                # bias pointers are per set: drop the middle set's, give set 0 one
                bs = [m._bias_for(dt) if i != 1 else None for i, m in enumerate(mods)]
                if bs[0] is None:
                    bs[0] = (torch.randn(Ns[0], generator=torch.Generator(device=DEV).manual_seed(M), device=DEV)
                             * 0.1).to(dt)
                direct = _decode_multi(mods, xm, bs)
                for i, (o, v, b) in enumerate(zip(direct, plain, bs)):
                    assert torch.equal(o, with_bias(v, b)), f"{name} M={M} set {i}{tag}: bias of set {i}"
        if fused:
            # fused vs separate launches: the same bits whenever both cut K the same way, whichever kernel ran
            xm = x[:M].contiguous()
            groups = [m._siblings for m in mods]
            for m in mods:
                m._siblings = None
            try:
                sep, ks_sep = decode_kernels_launched(lambda: [m(xm) for m in mods])
            finally:
                for m, g_ in zip(mods, groups):
                    m._siblings = g_
            assert len(ks_sep) == len(mods), ks_sep
            fo = [m(xm) for m in mods]
            for i, (s, k, f) in enumerate(zip(sep, ks_sep, fo)):
                if same_k_split(M, K, (Ns[i], k[0]), (sum(Ns), served[M][0])):
                    assert torch.equal(s, f), f"{name} M={M} set {i}: fused != separate ({k[0]} vs {served[M][0]})"
                    SAME_BITS.add((name, M, i, k[0], served[M][0]))
                else:
                    assert_close_rel(f, s, rel, f"{name} M={M} set {i} fused vs separate")
    # the planner's prediction (it sizes shared memory for sym g128) is what ran
    if sym and gs == 128:
        NT = sum(Ns) // 32
        for M, k in served.items():
            fits2 = decode_k_split(M, K, sum(Ns), "decode2_kernel") is not None
            assert k[0] == ("decode2_kernel" if NT > 132 and fits2 else "decode_kernel"), (name, M, k)
    SERVED[name] = served
    return served


SAME_BITS = set()  # (case, M, set, single launch's kernel, fused launch's kernel) pinned bit-identical


@pytest.mark.parametrize("name", list(CASES))
def test_decode_tier_matches_oracle(name):
    _run_case(name)


def test_decode_tier_coverage():
    """Which kernel served which case: decode2_kernel in all 8 dense instantiations with and without act-order, the
    decode_kernel fallback where decode2's shared memory does not fit, and the SiblingGroup bit-identity across kernels."""
    rows = []
    for name in CASES:
        for M, k in _run_case(name).items():
            rows.append((name, M) + k)
    print("\ncase | M | kernel | dtype | asym | g64")
    for r in rows:
        print(" | ".join(str(v) for v in r))
    inst = {(r[3], r[4], r[5], name_act) for r in rows if r[2] == "decode2_kernel"
            for name_act in [r[0].endswith("-act")]}
    for dt in DTN.values():
        for asym in (False, True):
            for g64 in (False, True):
                for act in (False, True):
                    assert (dt, asym, g64, act) in inst, (dt, asym, g64, act)
    # Llama-3-8B gate|up: decode2's parked partial sums outgrow shared memory from 6 tokens on
    for name in CASES:
        if name.startswith("llama3_8b_gate_up"):
            ks = {M: k[0] for M, k in SERVED[name].items()}
            assert ks == {M: "decode2_kernel" if M <= 5 else "decode_kernel" for M in MS}, (name, ks)
    assert SERVED["llama3_70b_tp8_gate_up-fp16-sym-g128"][8][0] == "decode_kernel"
    assert SERVED["wide_4256-fp16-sym-g128"][1][0] == "decode2_kernel"
    # the SiblingGroup docstring's claim across kernels: a fused decode2 launch and a single decode_kernel launch with
    # the same K split agree bit for bit (q of q|k|v, gate of gate|up)
    assert any(s[3] == "decode_kernel" and s[4] == "decode2_kernel" for s in SAME_BITS), SAME_BITS


# ------------------------------------------------------------------------------------------------------------------------
# forced plans: the split-K / warp-group plans the TP all-reduce path may take
# ------------------------------------------------------------------------------------------------------------------------
FORCED = [  # K, Ns, sym, group, act-order
    (4096, QKV8B, True, 128, False),
    (4096, QKV8B, False, 64, False),
    (4096, QKV8B, True, 128, True),
    (1024, (8192,), True, 128, False),
]


def test_decode2_forced_plans_match_oracle():
    """B2Q_DECODE_V2=1 (decode2_kernel chooses split-K ranks and warp groups freely) and B2Q_DECODE2_GW=1|2|4|8: every
    plan against the oracle and deterministic.  Together the plans cover cluster split-K with a DSMEM reduction, several
    warp groups per CTA (CTA-wide activation staging) and act-order staging."""
    import ctypes
    import gptqmodel_b200 as g
    from gptqmodel_b200 import fuse_siblings
    plans = set()
    for ci, (K, Ns, sym, gs, act) in enumerate(FORCED):
        Ls = _layers(K, Ns, F16, sym, gs, act, (0,) * len(Ns), seed=100 + ci)
        mods = [_module(L, F16) for L in Ls]
        if len(mods) > 1:
            assert fuse_siblings(mods)
        x, _ = _inputs(K, F16, seed=200 + ci)
        refs = [decode_oracle(L, x) for L in Ls]
        for gw in (None, 1, 2, 4, 8):
            with _Env(B2Q_DECODE_V2=1, B2Q_DECODE2_GW=gw):
                for M in (1, 3, 8):
                    xm = x[:M].contiguous()
                    outs, ks = decode_kernels_launched(lambda: [m(xm).clone() for m in mods])
                    assert len(ks) == 1, ks
                    what = f"K={K} N={Ns} sym={sym} g{gs} act={act} gw={gw} M={M}"
                    for i, (o, r) in enumerate(zip(outs, refs)):
                        assert_close_rel(o, r[:M], 1e-3, f"{what} set {i}")
                    assert all(torch.equal(a, m(xm)) for a, m in zip(outs, mods)), f"{what}: not deterministic"
                    if ks[0][0] == "decode2_kernel" and sym and gs == 128:
                        pl = (ctypes.c_int * 8)()
                        assert g.lib.b2q_debug_decode_plan(2, M, K, sum(Ns), 0, 0, pl) == 0
                        plans.add((pl[1], pl[2] // pl[3], act))  # (split-K ranks, warp groups per CTA, act-order)
    assert any(p[0] > 1 for p in plans), plans          # cluster split-K, DSMEM reduction
    assert any(p[1] > 1 for p in plans), plans          # several warp groups: CTA-wide staging
    assert any(p[0] > 1 and p[1] > 1 for p in plans), plans
    assert any(p[2] for p in plans), plans              # act-order staging


# ------------------------------------------------------------------------------------------------------------------------
# graph replay and a PDL chain
# ------------------------------------------------------------------------------------------------------------------------
def test_fused_gate_up_graph_replay():
    """One capture of the fused Llama-3-8B gate|up launch at M = 1 replays the eager bits."""
    from gptqmodel_b200 import fuse_siblings
    Ls = _layers(4096, GU8B, F16, True, 128, False, (0, 0), seed=300)
    mods = [_module(L, F16) for L in Ls]
    assert fuse_siblings(mods)
    x, _ = _inputs(4096, F16, seed=301)
    x1 = x[:1].contiguous()
    eager = [m(x1).clone() for m in mods]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            [m(x1) for m in mods]
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ys = [m(x1) for m in mods]
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(ys, eager):
        assert torch.equal(a, b)


def _chain(mods_qkv, mod_o, mods_gu, x):
    """q|k|v -> o (from q) -> gate|up (from o's output), enqueued with no host synchronisation."""
    q, k, v = [m(x) for m in mods_qkv]
    o = mod_o(q)
    g_, u = [m(o) for m in mods_gu]
    return q, k, v, o, g_, u


def test_pdl_chain_matches_stagewise_oracle():
    """Three dependent decode launches back to back (each may start its weight prefetch under the previous one): every
    stage against the oracle of its actual input, and bit-identical to the same chain without PDL."""
    from gptqmodel_b200 import fuse_siblings
    Lq = _layers(4096, QKV8B, F16, True, 128, False, (0, 0, 0), seed=400)
    Lo = _layers(4096, (4096,), F16, True, 128, False, (0,), seed=401)
    Lg = _layers(4096, GU8B, F16, True, 128, False, (0, 0), seed=402)
    mq, mo, mg = [_module(L, F16) for L in Lq], _module(Lo[0], F16), [_module(L, F16) for L in Lg]
    assert fuse_siblings(mq) and fuse_siblings(mg)
    x, _ = _inputs(4096, F16, seed=403)
    for M in (1, 5, 8):
        xm = x[:M].contiguous()
        outs = [t.clone() for t in _chain(mq, mo, mg, xm)]
        torch.cuda.synchronize()
        q = outs[0]
        for i, (o, L) in enumerate(zip(outs[:3], Lq)):
            assert_close_rel(o, decode_oracle(L, xm), 1e-3, f"chain M={M} qkv set {i}")
        assert_close_rel(outs[3], decode_oracle(Lo[0], q), 1e-3, f"chain M={M} o")
        for i, (o, L) in enumerate(zip(outs[4:], Lg)):
            assert_close_rel(o, decode_oracle(L, outs[3]), 1e-3, f"chain M={M} gate_up set {i}")
        with _Env(B2Q_DISABLE_PDL=1):
            plain = [t.clone() for t in _chain(mq, mo, mg, xm)]
            torch.cuda.synchronize()
        for a, b in zip(outs, plain):
            assert torch.equal(a, b), f"chain M={M}: PDL changed the result"


# ------------------------------------------------------------------------------------------------------------------------
# negative controls: the comparison above fails for each of these mistakes (applied to the oracle, never the kernel)
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", (F16, BF16), ids=["fp16", "bf16"])
def test_negative_controls(dt):
    from gptqmodel_b200 import fuse_siblings
    K = 4096
    Ls = _layers(K, QKV8B, dt, False, 64, False, (0, 0, 0), seed=500)
    mods = [_module(L, dt) for L in Ls]
    assert fuse_siblings(mods)
    x, _ = _inputs(K, dt, seed=501)
    outs, ks = decode_kernels_launched(lambda: [m(x).clone() for m in mods])
    assert ks[0][0] == "decode2_kernel"
    rel = REL[dt]
    refs = [decode_oracle(L, x) for L in Ls]
    for i in range(3):
        assert_close_rel(outs[i], refs[i], rel, f"control set {i}")
    L0 = Ls[0]

    def bites(ref, what, i=0):
        with pytest.raises(AssertionError, match="outside"):
            assert_close_rel(outs[i], ref, rel, f"negative control: {what}")

    # one (group, feature) zero point off by one, in the group with the largest activation sum (the size of the mistake)
    gmax = int(x.float().reshape(8, K // 64, 64).sum(2).abs().amax(0).argmax())
    qz = L0["qzeros"].clone()
    qz[gmax, 1] ^= 1 << 8  # feature 8 * 1 + 2: flips the zero's lowest bit
    bites(decode_oracle(L0, x, qzeros=qz), "zero point off by one")
    # the two 64-k scale rows of quad 3 exchanged (groups 6 and 7)
    sc = L0["scales"].clone()
    sc[[6, 7]] = sc[[7, 6]]
    bites(decode_oracle(L0, x, scales=sc), "G64 scale rows exchanged")
    # features g and g + 8 of tile 2 exchanged
    r = refs[0].clone()
    r[:, [64 + 3, 64 + 11]] = r[:, [64 + 11, 64 + 3]]
    bites(r, "features g, g + 8 exchanged")
    # the last quad's activations zeroed
    xz = x.clone()
    xz[:, K - 128:] = 0
    bites(decode_oracle(L0, xz), "last quad zeroed")
    # tokens 2t and 2t + 1 exchanged (t = 1)
    r = refs[0].clone()
    r[[2, 3]] = r[[3, 2]]
    bites(r, "tokens 2, 3 exchanged")
    # the first feature of set 1 taken from set 0
    r = refs[1].clone()
    r[:, 0] = refs[0][:, 0]
    bites(r, "set 1 feature 0 from set 0", i=1)
