"""The GPTQ tensor-core tiers against a float64 oracle: the prefill GEMM (gemm_kernel, b2q_gemm.cu: M > 128, and
b2q_gemm_multi for fused siblings) and the small-batch tier (midm_kernel MODE 0, b2q_midm.cu: M <= 128).  pytest -m gpu

Operand.  Both kernels feed the tensor cores W_T = RN_T((q - z) * s_T): s_T is the checkpoint scale converted to the run
dtype T, (q - z) is an exact integer, the product is exact in float64 (at most 11 + 8 significant bits) and is rounded
once to T.  The one-hot probes push rows of the identity through b2q_gemm: every output element is one weight times 1.0
plus exact zeros (under split-K the other ranks add exact +0), so the output must equal W_T bit for bit.  The probes use
launches of 16, 32, 64 and 128 rows (every token box of midm_kernel) and of 256 rows (gemm_kernel); row i of a launch
starting at k0 is e_k with k = (k0 + i) mod K, so every row of W_T is probed in every box.

Dense check.  acc = x @ W_T in float64 on the GPU (in blocks of 4096 columns), ref = RN_T(acc), and
    |out - ref| <= K 2^-24 (|x| @ |W_T|) + 2 P_T (|acc| + |ref|),   P_T = 2^-10 (fp16), 2^-7 (bf16):
the first term bounds any order of fp32 accumulation of K products that are exact in fp32 (T x T products have at most
22 significant bits), split-K partial sums included; the second covers the final rounding to T (half an ulp, 2^-11 |y|
in fp16 and 2^-8 |y| in bf16) with room for a double rounding of the oracle's float64 -> T conversion.  There is no
floor proportional to rms(ref): an all-zero input row must give exactly 0.  The bias is added after the rounding,
RN_T(RN_T(v) + b) (in fp32, like the epilogue), and is checked bit for bit on the kernel's own no-bias output v.

Each case records, through torch.profiler, which instantiation ran for every token count; test_wgmma_tier_coverage
asserts that the cases reached all 8 gemm_kernel and all 32 midm_kernel non-FP8 MODE-0 instantiations.  The negative
controls show that the checks fail for a one-ulp scale, two exchanged g32 scale rows and a zero-point off by one.
"""
import ctypes
import os
import re

import pytest
import torch

import oracle
from helpers import _record, random_layer

pytestmark = pytest.mark.gpu

DEV = "cuda"
F16, BF16 = torch.float16, torch.bfloat16
P = {F16: 2.0 ** -10, BF16: 2.0 ** -7}
DTN = {F16: "__half", BF16: "__nv_bfloat16"}
CODE = {F16: 0, BF16: 1}
SMALL = (1, 2, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128)
PREFILL = (129, 255, 256, 257, 300)
ZERO_ROW = 4  # the all-zero activation row of every input set
COL_BLOCK = 4096


# ------------------------------------------------------------------------------------------------------------------------
# layers, launches, oracle
# ------------------------------------------------------------------------------------------------------------------------
def _layer(K, N, bits, gs, sym, act, bias, dt, seed):
    """Random codes on the device (helpers.random_layer); act: g_idx = (arange(K) // gs)[randperm]; bias randn * 0.1 in dt."""
    L = random_layer(K, N, bits=bits, group_size=gs, sym=sym, seed=seed, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(seed + 1)
    if act:
        g = gs if gs > 0 else K
        perm = torch.randperm(K, generator=gen, device=DEV)
        L["g_idx"], L["desc_act"] = (torch.arange(K, dtype=torch.int32, device=DEV) // g)[perm].to(torch.int32), True
    if bias:
        L["bias"] = (torch.randn(N, generator=gen, device=DEV) * 0.1).to(dt)
    return L


def _module(L, dt):
    from gptqmodel_b200 import B200QuantLinear
    return B200QuantLinear.from_checkpoint_tensors(
        L["qweight"], L["qzeros"], L["scales"], L["g_idx"], L["bits"], L["group_size"], bias=L["bias"],
        desc_act=L["desc_act"], sym=L["sym"], device=DEV, dtype=dt)


def _p(t):
    return None if t is None else t.data_ptr()


def _gemm(m, x, bias=None, out=None):
    """b2q_gemm over the module's prepacked weights (never the decode tier or the GEMV); act-order layers get a workspace
    of exactly b2q_workspace_bytes(M, K, N, 1) = M*K*2 bytes.  The output starts as NaN, so an element no CTA writes
    cannot pass for a stale result of an earlier launch."""
    import gptqmodel_b200 as g
    M, K = x.shape
    N, dt = m.out_features, x.dtype
    if out is None:
        out = torch.full((M, N), float("nan"), dtype=dt, device=DEV)
    ws, wsb = None, 0
    if m.perm is not None:
        wsb = g.lib.b2q_workspace_bytes(M, K, N, 1)
        ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    g.check(g.lib.b2q_gemm(x.data_ptr(), m.packed.data_ptr(), m._scales_for(dt).data_ptr(), _p(m._zeros_dev), _p(m.perm),
                           _p(bias), out.data_ptr(), M, K, N, m.kbits, m._kgs, CODE[dt], _p(ws), wsb,
                           torch.cuda.current_stream().cuda_stream), "b2q_gemm")
    return out


def _w_t(L, dt, qzeros=None, scales=None):
    """W_T [K, N] in dt: RN_T((q - z) * s_T), the product exact in float64.  qzeros= / scales= replace the layer's
    tensors (negative controls)."""
    qz = L["qzeros"] if qzeros is None else qzeros
    sc = L["scales"] if scales is None else scales
    K, N, bits = L["K"], L["N"], L["bits"]
    c = 32 // bits  # features per zero word
    W = torch.empty(K, N, dtype=dt, device=DEV)
    for n0 in range(0, N, COL_BLOCK):
        n1 = min(N, n0 + COL_BLOCK)
        W[:, n0:n1] = oracle.dequantize_weight(L["qweight"][:, n0:n1], qz[:, n0 // c:n1 // c],
                                               sc[:, n0:n1].to(dt).to(torch.float64), L["g_idx"], bits).to(dt)
    return W


class _Ref:
    """acc = x @ W_T and K 2^-24 |x| @ |W_T| in float64 for all rows of x, evaluated in column blocks."""

    def __init__(self, x, W):
        xd = x.to(torch.float64)
        M, N = x.shape[0], W.shape[1]
        self.dt, self.K = x.dtype, x.shape[1]
        self.acc = torch.empty(M, N, dtype=torch.float64, device=DEV)
        self.bnd = torch.empty_like(self.acc)
        for n0 in range(0, N, COL_BLOCK):
            Wd = W[:, n0:n0 + COL_BLOCK].to(torch.float64)
            self.acc[:, n0:n0 + COL_BLOCK] = xd @ Wd
            self.bnd[:, n0:n0 + COL_BLOCK] = xd.abs() @ Wd.abs()
        self.bnd *= self.K * 2.0 ** -24


def _check(out, R, what):
    """out [M, N] (the first M rows of R's input) within the bound of the module docstring; returns the worst err/tol."""
    M = out.shape[0]
    acc = R.acc[:M]
    ref = acc.to(R.dt)
    tol = R.bnd[:M] + 2 * P[R.dt] * (acc.abs() + ref.to(torch.float64).abs())
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    err = (out.to(torch.float64) - ref.to(torch.float64)).abs()
    # a zero tolerance (an all-zero row: acc = 0) admits only an exact 0
    ratio = torch.where(tol > 0, err / tol.clamp_min(1e-300), torch.where(err > 0, torch.inf, torch.zeros_like(err)))
    worst = float(ratio.max())
    _record(what, P[R.dt], worst)
    if worst > 1:
        bad = ratio > 1
        i, j = [int(v) for v in bad.nonzero()[0]]
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} outside the bound, worst ratio {worst:.3g}; first "
                             f"[{i}, {j}]: out {float(out[i, j]):.6g} ref {float(ref[i, j]):.6g} tol {float(tol[i, j]):.3g}")
    if M > ZERO_ROW:
        assert not out[ZERO_ROW].to(torch.float32).abs().any(), f"{what}: the all-zero row is not exactly 0"
    return worst


def _with_bias(v, b):
    """RN_T(RN_T(v) + b), the sum in fp32 like the epilogues of both kernels."""
    return (v.float() + b.float()).to(v.dtype)


def _inputs(K, M, dt, seed):
    """randn * 0.5 and the same with 8 channels x 30; row ZERO_ROW all zero in both."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, K, generator=gen, device=DEV) * 0.5
    x[ZERO_ROW] = 0
    xo = x.clone()
    xo[:, torch.randperm(K, generator=gen, device=DEV)[:8]] *= 30
    return x.to(dt).contiguous(), xo.to(dt).contiguous()


def _probe(run, W, R, what):
    """One-hot probe: launches of R rows, row i of the launch at k0 = e_k with k = (k0 + i) mod K, for k0 = 0, R, 2R, ...
    < K.  run(x, out) writes out [R, N]; every output row must equal W_T's row k bit for bit."""
    K, N = W.shape
    n = (K + R - 1) // R
    outs = torch.full((n * R, N), float("nan"), dtype=W.dtype, device=DEV)
    rows = torch.arange(n * R, device=DEV) % K
    x = torch.zeros(n * R, K, dtype=W.dtype, device=DEV)
    x[torch.arange(n * R, device=DEV), rows] = 1
    for c in range(n):
        run(x[c * R:(c + 1) * R], outs[c * R:(c + 1) * R])
    ref = W[rows]
    bad = outs.view(torch.int16) != ref.view(torch.int16)
    if bad.any():
        i, j = [int(v) for v in bad.nonzero()[0]]
        raise AssertionError(f"{what}: one-hot probe ({R}-row launches) differs in {int(bad.sum())}/{bad.numel()} "
                             f"elements; first W[{int(rows[i])}, {j}]: out {float(outs[i, j]):.6g} W_T "
                             f"{float(ref[i, j]):.6g}")


# ------------------------------------------------------------------------------------------------------------------------
# which instantiation ran
# ------------------------------------------------------------------------------------------------------------------------
_GEMM = re.compile(r"\bgemm_kernel<(__half|__nv_bfloat16), (4|8), (true|false), 4, (true|false)>")
_MIDM = re.compile(r"\bmidm_kernel<(__half|__nv_bfloat16), (4|8), (true|false), (16|32|64|128), (\d+), (\d+), (\d+), "
                   r"(\d+), (true|false)>")


def _launched(fn):
    """Runs fn() (which launches ONE gemm_kernel / midm_kernel) three times under torch.profiler; returns (the last
    result, {instantiation}): ("gemm_kernel", dtype, bits, asym, None) or ("midm_kernel", dtype, bits, asym, token box).
    After many profiling sessions in one process a window can lose its first kernel records, so every window starts with
    filler kernels and repeats the launch; a window without any record is profiled again."""
    from torch.profiler import ProfilerActivity, profile
    pad = torch.zeros(1, device=DEV)
    for _ in range(5):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(64):
                pad.add_(1)
            torch.cuda.synchronize()
            for _ in range(3):
                res = fn()
            torch.cuda.synchronize()
        evs = [e for e in prof.events() if _GEMM.search(e.name) or _MIDM.search(e.name)]
        if evs:
            break
    out = set()
    for e in evs:
        m = _GEMM.search(e.name)
        if m:
            dt, bits, asym, fp8 = m.groups()
            out.add(("gemm_kernel", dt, int(bits), asym == "true", None))
        else:
            dt, bits, asym, ntok, _pst, _wst, mode, _dqg, fp8 = _MIDM.search(e.name).groups()
            assert mode == "0", e.name
            out.add(("midm_kernel", dt, int(bits), asym == "true", int(ntok)))
        assert fp8 == "false", e.name
    return res, out


def _box(M):
    return 16 if M <= 16 else 32 if M <= 32 else 64 if M <= 64 else 128


def _predict(dt, bits, sym, M, midm=True):
    """The instantiation b2q_gemm launches for M tokens (B2Q_MIDM=0: midm=False)."""
    if M <= 128 and midm:
        return ("midm_kernel", DTN[dt], bits, not sym, _box(M))
    return ("gemm_kernel", DTN[dt], bits, not sym, None)


class _Env:
    """Sets B2Q_* switches for the duration of a block and restores the previous values (also on failure)."""

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
# cases: (K, N, dtype, bits, group (-1: per channel), sym, act-order, bias, token counts)
# ------------------------------------------------------------------------------------------------------------------------
MS = SMALL + PREFILL
CASES = {
    # every (dtype, bits, symmetry) at every token box and above 128 tokens: the 40 instantiations
    "k4096_n4128-fp16-4b-sym-g128-bias": (4096, 4128, F16, 4, 128, True, False, True, MS + (2048,)),
    "k1088_n160-fp16-4b-asym-g32": (1088, 160, F16, 4, 32, False, False, False, MS),
    "k1088_n96-fp16-8b-sym-perchannel-bias": (1088, 96, F16, 8, -1, True, False, True, MS),
    "k4096_n4128-fp16-8b-asym-g64": (4096, 4128, F16, 8, 64, False, False, False, MS),
    "k4096_n4096-bf16-4b-sym-g64-act": (4096, 4096, BF16, 4, 64, True, True, False, MS),
    "k192_n320-bf16-4b-asym-perchannel-bias": (192, 320, BF16, 4, -1, False, False, True, MS),
    "k1088_n160-bf16-8b-sym-g32-act": (1088, 160, BF16, 8, 32, True, True, False, MS),
    "k4096_n4128-bf16-8b-asym-g128-bias": (4096, 4128, BF16, 8, 128, False, False, True, MS),
    # the rest of the shape / format space
    "k64_n32-fp16-4b-sym-g64": (64, 32, F16, 4, 64, True, False, False, MS),
    "k64_n96-bf16-8b-asym-g32": (64, 96, BF16, 8, 32, False, False, False, MS),
    "k4096_n1024-fp16-4b-asym-g128-act-bias": (4096, 1024, F16, 4, 128, False, True, True, MS),
    "k1088_n4128-fp16-8b-asym-g64-act": (1088, 4128, F16, 8, 64, False, True, False, MS),
    "k192_n4096-fp16-4b-sym-g32": (192, 4096, F16, 4, 32, True, False, False, MS),
    "k4096_n320-bf16-4b-sym-g128": (4096, 320, BF16, 4, 128, True, False, False, MS),
    "k14336_n4096-bf16-4b-asym-g128": (14336, 4096, BF16, 4, 128, False, False, False, (1, 16, 64, 128, 300)),
}
MODULE_MS = (9, 33, 128, 300)  # b2q_mm serves these on the same tier as b2q_gemm (above the decode tier and the GEMV)
SERVED = {}  # case -> {M: instantiation}
WORST = {}   # case -> worst err/tol of its dense checks


def _build(name):
    K, N, dt, bits, gs, sym, act, bias, Ms = CASES[name]
    L = _layer(K, N, bits, gs, sym, act, bias, dt, seed=list(CASES).index(name) * 13 + 5)
    m = _module(L, dt)
    assert (m.perm is not None) == act and (m._zeros_dev is None) == sym and m._kK == K
    return L, m


def _run_case(name):
    """Every token count of a case through b2q_gemm: the launched instantiation, the oracle on both input sets, the bias
    bit for bit, determinism, and the module (b2q_mm) equal to b2q_gemm where they share a tier."""
    if name in SERVED:
        return SERVED[name]
    K, N, dt, bits, gs, sym, act, bias, Ms = CASES[name]
    L, m = _build(name)
    W = _w_t(L, dt)
    b = m._bias_for(dt)
    x, xo = _inputs(K, max(Ms), dt, seed=K + N)
    refs = {id(x): _Ref(x, W), id(xo): _Ref(xo, W)}
    served, worst = {}, 0.0
    for M in Ms:
        for xs, tag in ((x, ""), (xo, " outliers")):
            xm = xs[:M].contiguous()
            what = f"{name} M={M}{tag}"
            if tag:
                v = _gemm(m, xm)
            else:
                v, ks = _launched(lambda: _gemm(m, xm))
                assert ks == {_predict(dt, bits, sym, M)}, (what, ks)
                served[M] = _predict(dt, bits, sym, M)
            worst = max(worst, _check(v, refs[id(xs)], what))
            assert torch.equal(v, _gemm(m, xm)), f"{what}: not deterministic"
            if b is not None:
                vb = _gemm(m, xm, b)
                assert torch.equal(vb, _with_bias(v, b)), f"{what}: bias is not RN(RN(v) + b)"
                if M > ZERO_ROW:
                    assert torch.equal(vb[ZERO_ROW], b), f"{what}: the zero row is not exactly the bias"
            if M in MODULE_MS:
                y = m(xm)
                assert torch.equal(y, _gemm(m, xm, b)), f"{what}: module (b2q_mm) != b2q_gemm"
    SERVED[name], WORST[name] = served, worst
    print(f"\n{name}: worst err/tol {worst:.3f}")
    return served


@pytest.mark.parametrize("name", list(CASES))
def test_wgmma_tier_matches_oracle(name):
    _run_case(name)


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c[0] <= 4096])
def test_one_hot_probes_exact(name):
    """Rows of the identity through b2q_gemm in every token box of midm_kernel and through gemm_kernel: the output is
    W_T bit for bit (with act-order, e_k returns row k of the original W)."""
    K, N, dt, bits, gs, sym, act, bias, Ms = CASES[name]
    L, m = _build(name)
    W = _w_t(L, dt)
    for R in (16, 32, 64, 128, 256):
        _, ks = _launched(lambda: _gemm(m, torch.eye(R, K, dtype=dt, device=DEV)))
        assert ks == {_predict(dt, bits, sym, R)}, (name, R, ks)
        _probe(lambda xr, o: _gemm(m, xr, out=o), W, R, f"{name} R={R}")


def test_wgmma_tier_coverage():
    """The cases reached all 8 gemm_kernel and all 32 midm_kernel non-FP8 MODE-0 instantiations."""
    rows = []
    for name in CASES:
        for M, k in _run_case(name).items():
            rows.append((name, M) + k)
    seen = {r[2:] for r in rows}
    print("\ncase | worst err/tol")
    for name in CASES:
        print(f"{name} | {WORST[name]:.3f}")
    want = set()
    for dt in DTN.values():
        for bits in (4, 8):
            for asym in (False, True):
                want.add(("gemm_kernel", dt, bits, asym, None))
                for ntok in (16, 32, 64, 128):
                    want.add(("midm_kernel", dt, bits, asym, ntok))
    assert len(want) == 40
    missing = want - seen
    assert not missing, sorted(missing, key=str)
    print(f"{len(want & seen)} of 40 instantiations ran")


# ------------------------------------------------------------------------------------------------------------------------
# gemm_kernel below 129 tokens, forced split-K of the small-batch tier
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["k1088_n160-fp16-4b-asym-g32", "k4096_n4128-bf16-8b-asym-g128-bias",
                                  "k4096_n1024-fp16-4b-asym-g128-act-bias"])
def test_midm_off_partial_token_tile(name):
    """B2Q_MIDM=0: b2q_gemm runs gemm_kernel with one partly filled 128-token tile at M = 1, 77, 128."""
    K, N, dt, bits, gs, sym, act, bias, _ = CASES[name]
    L, m = _build(name)
    W = _w_t(L, dt)
    b = m._bias_for(dt)
    x, xo = _inputs(K, 128, dt, seed=K + N + 1)
    with _Env(B2Q_MIDM=0):
        for xs, tag in ((x, ""), (xo, " outliers")):
            R = _Ref(xs, W)
            for M in (1, 77, 128):
                xm = xs[:M].contiguous()
                what = f"{name} B2Q_MIDM=0 M={M}{tag}"
                v, ks = _launched(lambda: _gemm(m, xm))
                assert ks == {_predict(dt, bits, sym, M, midm=False)}, (what, ks)
                _check(v, R, what)
                assert torch.equal(v, _gemm(m, xm)), f"{what}: not deterministic"
                if b is not None:
                    assert torch.equal(_gemm(m, xm, b), _with_bias(v, b)), f"{what}: bias"
        _probe(lambda xr, o: _gemm(m, xr, out=o), W, 77, f"{name} B2Q_MIDM=0")


def _ranks(K, ks):
    """k-blocks per split-K rank of midm_kernel for a requested ks (launch_midm: at most 8, halved until every rank owns
    a k-block; kpc = ceil(nkb / ks))."""
    nkb = K // 64
    ks = min(ks, 8)
    while ks > 1 and (ks - 1) * ((nkb + ks - 1) // ks) >= nkb:
        ks //= 2
    kpc = (nkb + ks - 1) // ks
    return [min(nkb, (r + 1) * kpc) - r * kpc for r in range(ks)]


FORCED = [  # K, N, dtype, bits, group, sym, act-order
    (64, 160, F16, 4, 32, False, False),
    (192, 96, BF16, 8, 64, True, False),
    (192, 4128, F16, 4, -1, True, True),
    (1088, 160, F16, 4, 32, False, False),
    (1088, 4096, BF16, 8, 64, False, True),
]


def test_forced_split_k():
    """B2Q_MIDM_KS = 1, 2, 4, 8 and the planner's choice on K = 64, 192 and 1088: the oracle, the one-hot probes (a
    dropped or doubled k-block of any rank changes a row) and determinism.  K = 1088 (17 k-blocks) at ks = 8 runs 4 ranks
    of 5, 5, 5 and 2 blocks; K = 192 at ks >= 2 runs 2 ranks of 2 and 1."""
    assert _ranks(1088, 8) == [5, 5, 5, 2] and _ranks(1088, 4) == [5, 5, 5, 2] and _ranks(1088, 2) == [9, 8]
    assert _ranks(192, 8) == [2, 1] and _ranks(192, 4) == [2, 1] and _ranks(64, 8) == [1]
    differ = 0
    for ci, (K, N, dt, bits, gs, sym, act) in enumerate(FORCED):
        L = _layer(K, N, bits, gs, sym, act, False, dt, seed=900 + ci)
        m = _module(L, dt)
        W = _w_t(L, dt)
        x, xo = _inputs(K, 128, dt, seed=901 + ci)
        Rs = {id(x): _Ref(x, W), id(xo): _Ref(xo, W)}
        first = {}
        for ks in (None, 1, 2, 4, 8):
            with _Env(B2Q_MIDM_KS=ks):
                for M in (1, 16, 33, 128):
                    for xs, tag in ((x, ""), (xo, " outliers")):
                        xm = xs[:M].contiguous()
                        what = f"K={K} N={N} {DTN[dt]} {bits}b g{gs} sym={sym} act={act} ks={ks} M={M}{tag}"
                        v = _gemm(m, xm)
                        _check(v, Rs[id(xs)], what)
                        assert torch.equal(v, _gemm(m, xm)), f"{what}: not deterministic"
                        key = (M, tag)
                        if key in first:
                            differ += not torch.equal(v, first[key])
                        else:
                            first[key] = v
                for R in (16, 128):
                    _probe(lambda xr, o: _gemm(m, xr, out=o), W, R, f"K={K} N={N} ks={ks}")
    # the switch takes effect: another split order changes some roundings of the fp32 sums
    assert differ > 0


# ------------------------------------------------------------------------------------------------------------------------
# b2q_gemm_multi through the raw ABI
# ------------------------------------------------------------------------------------------------------------------------
def _gemm_multi(mods, x, biases, **over):
    """b2q_gemm_multi over the modules' weights with explicit bias pointers; returns (rc, outs).  over: raw argument
    overrides for the refusal checks (nsets, qzeros, bits, M, ws)."""
    import gptqmodel_b200 as g
    n = over.get("nsets", len(mods))
    M, K = x.shape
    M = over.get("M", M)
    dt = x.dtype
    sets = [mods[i % len(mods)] for i in range(max(n, 1))]
    outs = [torch.full((M, s.out_features), 7.0, dtype=dt, device=DEV) for s in sets]
    vp = ctypes.c_void_p * len(sets)
    zeros = over.get("qzeros", [_p(s._zeros_dev) for s in sets])
    perm = mods[0].perm
    ws, wsb = None, 0
    if perm is not None and over.get("ws", True):
        wsb = M * K * 2
        ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    bs = [(biases[i] if i < len(biases) else None) for i in range(len(sets))]
    rc = g.lib.b2q_gemm_multi(
        x.data_ptr(), n, vp(*[s.packed.data_ptr() for s in sets]), vp(*[s._scales_for(dt).data_ptr() for s in sets]),
        vp(*zeros), _p(perm), vp(*[_p(b) for b in bs]), vp(*[o.data_ptr() for o in outs]),
        (ctypes.c_int * len(sets))(*[s.out_features for s in sets]), M, K, over.get("bits", 4), mods[0]._kgs, CODE[dt],
        _p(ws), wsb, torch.cuda.current_stream().cuda_stream)
    return rc, outs


MULTI = {  # K, set widths, dtype, group, sym, act-order, M
    "llama3_8b_qkv-fp16-sym-g128": (4096, (4096, 1024, 1024), F16, 128, True, False, 300),
    "ragged-bf16-asym-g32": (1088, (96, 32, 160), BF16, 32, False, False, 257),
    "two_sets-fp16-asym-perchannel": (192, (160, 4128), F16, -1, False, False, 129),
    "ragged-bf16-sym-g64-act": (1088, (96, 32, 160), BF16, 64, True, True, 300),
    "ragged-fp16-asym-g128-act": (4096, (4128, 32, 96), F16, 128, False, True, 256),
}


@pytest.mark.parametrize("name", list(MULTI))
def test_gemm_multi_matches_single_sets(name):
    """Each set of one b2q_gemm_multi launch equals a single-set b2q_gemm of that set (gemm_kernel, no split-K: the same
    arithmetic) and passes the oracle; the middle set has no bias, the others have one (bit for bit RN(RN(v) + b))."""
    import gptqmodel_b200 as g
    K, Ns, dt, gs, sym, act, M = MULTI[name]
    seed = 700 + list(MULTI).index(name) * 7
    Ls = [_layer(K, N, 4, gs, sym, act, True, dt, seed=seed + i) for i, N in enumerate(Ns)]
    if act:
        for L in Ls[1:]:
            L["g_idx"] = Ls[0]["g_idx"].clone()
    mods = [_module(L, dt) for L in Ls]
    if act:
        assert all(torch.equal(mm.perm, mods[0].perm) for mm in mods)
    x, xo = _inputs(K, M, dt, seed=seed)
    biases = [mm._bias_for(dt) if i != 1 else None for i, mm in enumerate(mods)]
    for xs, tag in ((x, ""), (xo, " outliers")):
        (rc, outs), ks = _launched(lambda: _gemm_multi(mods, xs, biases))
        g.check(rc, "b2q_gemm_multi")
        assert ks == {("gemm_kernel", DTN[dt], 4, not sym, None)}, ks
        (rc0, plain) = _gemm_multi(mods, xs, [None] * len(mods))
        g.check(rc0, "b2q_gemm_multi")
        for i, (mm, L) in enumerate(zip(mods, Ls)):
            what = f"{name} set {i}{tag}"
            assert torch.equal(outs[i], _gemm(mm, xs, biases[i])), f"{what}: fused != single-set b2q_gemm"
            assert torch.equal(plain[i], _gemm(mm, xs)), f"{what}: fused != single-set b2q_gemm (no bias)"
            _check(plain[i], _Ref(xs, _w_t(L, dt)), what)
            if biases[i] is not None:
                assert torch.equal(outs[i], _with_bias(plain[i], biases[i])), f"{what}: bias"
            else:
                assert torch.equal(outs[i], plain[i]), f"{what}: NULL bias"


def test_gemm_multi_refusals():
    """Bad b2q_gemm_multi calls return -2 with their reason before any CUDA work (the outputs stay untouched)."""
    import gptqmodel_b200 as g
    K = 1088
    Ls = [_layer(K, N, 4, 64, False, True, False, F16, seed=800 + i) for i, N in enumerate((96, 32, 160))]
    for L in Ls[1:]:
        L["g_idx"] = Ls[0]["g_idx"].clone()
    mods = [_module(L, F16) for L in Ls]
    x, _ = _inputs(K, 300, F16, seed=801)
    zs = [_p(mm._zeros_dev) for mm in mods]
    for over, text in ((dict(nsets=0), "nsets=0"), (dict(nsets=4), "nsets=4"),
                       (dict(qzeros=[zs[0], None, zs[2]]), "set 1 unsupported"), (dict(bits=8), "bits=8"),
                       (dict(M=128), "M=128"), (dict(ws=False), "workspace")):
        rc, outs = _gemm_multi(mods, x, [None] * 3, **over)
        err = g.lib.b2q_last_error()
        assert rc == -2 and text.encode() in err, (over, rc, err)
        torch.cuda.synchronize()
        assert all(bool((o == 7).all()) for o in outs), over


# ------------------------------------------------------------------------------------------------------------------------
# negative controls: each check fails when the oracle is wrong in the way a kernel could be
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", (F16, BF16), ids=["fp16", "bf16"])
def test_negative_controls(dt):
    K, N = 1088, 160
    L = _layer(K, N, 4, 32, False, False, False, dt, seed=1000)
    m = _module(L, dt)
    W = _w_t(L, dt)
    x, _ = _inputs(K, 300, dt, seed=1001)
    run = lambda xr, o: _gemm(m, xr, out=o)  # noqa: E731
    for R in (16, 256):
        _probe(run, W, R, "control")
    outs = {M: _gemm(m, x[:M].contiguous()) for M in (64, 300)}  # midm_kernel, gemm_kernel
    R0 = _Ref(x, W)
    for M, v in outs.items():
        _check(v, R0, f"control M={M}")

    # one scale of one (group, feature) one ulp of T higher: the probe fails (every box)
    sc = L["scales"].to(dt)
    bumped = sc.clone()
    bumped.view(torch.int16)[5, 77] += 1
    Wb = _w_t(L, dt, scales=bumped)
    assert not torch.equal(Wb, W)
    for R in (16, 256):
        with pytest.raises(AssertionError, match="one-hot probe"):
            _probe(run, Wb, R, "negative control: scale + 1 ulp")

    # the two g32 scale rows of k-block 7 (groups 14 and 15) exchanged: the dense check fails
    sw = sc.clone()
    sw[[14, 15]] = sw[[15, 14]]
    Rsw = _Ref(x, _w_t(L, dt, scales=sw))
    for M, v in outs.items():
        with pytest.raises(AssertionError, match="outside the bound"):
            _check(v, Rsw, f"negative control: g32 scale rows exchanged M={M}")

    # one zero-point off by one, in the (group, feature) whose activation sum is largest
    G = K // 32
    gsum = x[:64].float().reshape(64, G, 32).sum(2).abs().amax(0)
    gr = int(gsum.argmax())
    qz = L["qzeros"].clone()
    z = (int(qz[gr, 2]) >> 4) & 15  # feature 17 = word 2, nibble 1
    qz[gr, 2] = int(qz[gr, 2]) + ((1 << 4) if z < 15 else -(1 << 4))
    Rz = _Ref(x, _w_t(L, dt, qzeros=qz))
    for M, v in outs.items():
        with pytest.raises(AssertionError, match="outside the bound"):
            _check(v, Rz, f"negative control: zero-point off by one M={M}")
