"""Per-channel W8A8 MoE experts (FP8 and INT8, dynamic and static activations) on the grouped path of
gptqmodel_b200/moe.py: B200ChannelW8A8Experts.

Path: b2q_moe_align -> b2q_*ch_moe_gather (the layer quantiser over the sorted rows) -> *ch_moe_gemm_kernel GM 1 (gate|up,
SiLU-mul epilogue) -> the quantiser on h (b2q_*ch_quantize, or the gather over the sorted h with w2's input scales) ->
GM 2 (down, routing weight, scatter) -> b2q_moe_combine.  include/b2q.h states the rounding points; they are those of
the per-expert module loop.

The stages are checked bit for bit against the layer kernels: the gather against b2q_*ch_quantize[_static] of each token
(with the expert's own input_scale), the down launch against w * T(b2q_*ch_mm) on each expert's rows at ks = 1, 2, 4,
gate|up within one ulp of T(silu) of the layer kernels' g and u (__expf against torch's exp).

The block is checked against the chain of layer calls (assert_block_equals_chain).  INT8 sums are exact, so the chain
is the modules of the loop themselves; FP8 runs the layer kernels at the block's pinned ks.  The two differ only where
the exp of T(silu(g)) flipped an element of h, and then only through the requantisation of that row.  A coarse float64
oracle (dequantised weights, unquantised activations clipped to the quantisers' range) covers both formats.
"""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from helpers import _record
from test_gpu_moe import _route, _skewed, _ulp

DEV = "cuda"
DTYPES = (torch.float16, torch.bfloat16)
TNAME = {torch.float16: "fp16", torch.bfloat16: "bf16"}
DT = {torch.float16: 0, torch.bfloat16: 1}
INF = float("inf")
# (format, activation kind, ub): the kinds of the issue's matrix
KINDS = [("fp8", "dynamic", None), ("fp8", "static", None), ("fp8", "dynamic", 2.0), ("int8", "dynamic", None),
         ("int8", "static", None)]
KIND_IDS = ["fp8_dyn", "fp8_static", "fp8_ub", "int8_dyn", "int8_static"]
PRE = {"fp8": "b2q_fp8ch", "int8": "b2q_int8ch"}


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _lib():
    from gptqmodel_b200._lib import check, lib

    return check, lib


# ---- checkpoint tensors and blocks --------------------------------------------------------------------------------------
def _role(fmt, E, N, K, seed, per_tensor=False):
    """(codes [E, N, K], s_w fp32 [E, N] (per tensor: one value per expert, broadcast), the modules' weight_scale);
    W = w * s_w has about unit-variance dot products with unit activations."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    if fmt == "fp8":
        w = (torch.randn(E, N, K, device=DEV, generator=gen) * 60).clamp(-448, 448).to(torch.float8_e4m3fn)
        amp = 60.0
    else:
        w = torch.randint(-127, 128, (E, N, K), device=DEV, generator=gen, dtype=torch.int8)
        amp = 73.0
    s = (torch.rand(E, 1 if per_tensor else N, device=DEV, generator=gen) + 0.5) / (amp * K ** 0.5)
    return w, s.expand(E, N).contiguous(), s


def _s_in(fmt, E, seed):
    """Per-expert static input scales: about the range of unit-variance activations (amax ~ 4.5)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.rand(E, device=DEV, generator=gen) * 0.4 + 0.8) * (4.5 / (448.0 if fmt == "fp8" else 127.0))


def _cls(fmt):
    from gptqmodel_b200 import B200ChannelFp8Linear, B200ChannelInt8Linear

    return B200ChannelFp8Linear if fmt == "fp8" else B200ChannelInt8Linear


def _modules(fmt, kind, ub, w, ms, s_in, **kw):
    cls = _cls(fmt)
    return [cls.from_checkpoint_tensors(w[e], ms[e], input_scale=None if s_in is None else s_in[e:e + 1],
                                        activation=kind, ub=ub, device=DEV, **kw) for e in range(w.shape[0])]


def _problem(fmt, kind, ub, E, K, I, H, seed, per_tensor=False):
    """ck = {role: (codes, s_w [E, N], s_in [E] or None)} (w1 and w3 share their input scales) and the grouped block."""
    from gptqmodel_b200 import B200ChannelW8A8Experts

    static = kind == "static"
    s13, s2 = (_s_in(fmt, E, seed), _s_in(fmt, E, seed + 7)) if static else (None, None)
    ck, mods = {}, {}
    for r, (N, Kr, si, sd) in (("w1", (I, K, s13, 1)), ("w3", (I, K, s13, 2)), ("w2", (H, I, s2, 3))):
        w, s, ms = _role(fmt, E, N, Kr, seed + sd, per_tensor)
        ck[r] = (w, s, si)
        mods[r] = _modules(fmt, kind, ub, w, ms, si)
    blk = B200ChannelW8A8Experts(mods["w1"], mods["w3"], mods["w2"], grouped=True)
    assert blk._stack is not None and blk._stack["int8"] == (fmt == "int8")
    return ck, blk


def _x(T, K, dt, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(T, K, device=DEV, generator=gen).to(dt)


# ---- stages through the raw ABI -----------------------------------------------------------------------------------------
def _align(ids, E):
    check, lib = _lib()
    T, top_k = ids.shape
    ids = ids.to(torch.int32).contiguous()
    tables = torch.empty(2 * E + T * top_k, dtype=torch.int32, device=DEV)
    counts, offsets, pairs = tables[:E], tables[E:2 * E], tables[2 * E:]
    check(lib.b2q_moe_align(_p(ids), T, top_k, E, _p(counts), _p(offsets), _p(pairs), _st()), "b2q_moe_align")
    return counts, offsets, pairs


def _ub(fmt, ub):
    return () if fmt == "int8" else (INF if ub is None else ub,)


def _quantize(fmt, x, s_in=None, ub=None):
    """The layer quantiser: codes [M, K], s_x [M] (s_in: a one-element device tensor, static)."""
    check, lib = _lib()
    M, K = x.shape
    codes = torch.empty((M, K), dtype=torch.uint8, device=DEV)
    sx = torch.empty(M, dtype=torch.float32, device=DEV)
    if s_in is not None:
        check(getattr(lib, PRE[fmt] + "_quantize_static")(_p(x), _p(s_in), _p(codes), _p(sx), M, K, DT[x.dtype], _st()),
              "quantize_static")
    else:
        check(getattr(lib, PRE[fmt] + "_quantize")(_p(x), _p(codes), _p(sx), M, K, *_ub(fmt, ub), DT[x.dtype], _st()),
              "quantize")
    return codes, sx


def _gather(fmt, x, pairs, offsets, s_in, E, top_k, ub=None):
    """Sorted rows of x[pairs / top_k] (pairs None: x is already the sorted rows)."""
    check, lib = _lib()
    T, K = x.shape
    rows = T * top_k
    codes = torch.full((rows, K), 0x7F, dtype=torch.uint8, device=DEV)
    sx = torch.zeros(rows, dtype=torch.float32, device=DEV)
    check(getattr(lib, PRE[fmt] + "_moe_gather")(_p(x), _p(pairs), _p(offsets), _p(s_in), E, _p(codes), _p(sx), T, top_k,
                                                 K, *_ub(fmt, ub), DT[x.dtype], _st()), "moe_gather")
    return codes, sx


def _mm(fmt, codes, sx, w, s, dt, ks):
    check, lib = _lib()
    M, K = codes.shape
    N = w.shape[0]
    out = torch.empty((M, N), dtype=dt, device=DEV)
    check(getattr(lib, PRE[fmt] + "_mm")(_p(codes), _p(sx), _p(w), _p(s), None, _p(out), M, K, N, DT[dt], ks, _st()),
          "mm")
    return out


def _gate_up(fmt, codes, sx, w1, s1, w3, s3, counts, offsets, dt, ks):
    check, lib = _lib()
    rows, K = codes.shape
    E, N = w1.shape[:2]
    h = torch.full((rows, N), float("nan"), dtype=dt, device=DEV)
    check(getattr(lib, PRE[fmt] + "_moe_gate_up")(_p(codes), _p(sx), _p(w1), _p(s1), _p(w3), _p(s3), _p(h), _p(counts),
                                                  _p(offsets), E, rows, min(E, rows), K, N, DT[dt], ks, _st()),
          "moe_gate_up")
    return h


def _down(fmt, codes, sx, w2, s2, counts, offsets, pairs, wts, dt, ks):
    check, lib = _lib()
    rows, K = codes.shape
    E, N = w2.shape[:2]
    yp = torch.full((rows, N), float("nan"), dtype=torch.float32, device=DEV)
    check(getattr(lib, PRE[fmt] + "_moe_down")(_p(codes), _p(sx), _p(w2), _p(s2), _p(counts), _p(offsets), _p(pairs),
                                               _p(wts), _p(yp), E, rows, min(E, rows), K, N, DT[dt], ks, _st()),
          "moe_down")
    return yp


def _expert_rows(counts, offsets):
    c, o = counts.cpu().tolist(), offsets.cpu().tolist()
    return [(e, o[e], o[e] + c[e]) for e in range(len(c)) if c[e] > 0]


def _block_abi(fmt, x, ids, w, ck, ks, ub=None):
    """The six launches of B200ChannelW8A8Experts through the raw ABI with ks pinned (0 = the heuristic):
    (pairs, h [rows, I] sorted, ypair [rows, H] by pair, y [T, H])."""
    check, lib = _lib()
    T, top_k = ids.shape
    E = ck["w1"][0].shape[0]
    H, dt = ck["w2"][0].shape[1], x.dtype
    counts, offsets, pairs = _align(ids, E)
    codes, sx = _gather(fmt, x, pairs, offsets, ck["w1"][2], E, top_k, ub)
    h = _gate_up(fmt, codes, sx, *ck["w1"][:2], *ck["w3"][:2], counts, offsets, dt, ks)
    if ck["w2"][2] is not None:
        ch, sh = _gather(fmt, h, None, offsets, ck["w2"][2], E, 1, ub)
    else:
        ch, sh = _quantize(fmt, h, ub=ub)
    yp = _down(fmt, ch, sh, *ck["w2"][:2], counts, offsets, pairs, w.to(torch.float32).contiguous(), dt, ks)
    y = torch.empty((T, H), dtype=dt, device=DEV)
    check(lib.b2q_moe_combine(_p(yp), _p(y), T, top_k, H, DT[dt], _st()), "b2q_moe_combine")
    return pairs, h, yp, y


def _deq(w, s, e):
    """W_e^T [K, N] float64 = codes * s_w."""
    return (w[e].to(torch.float64) * s[e].to(torch.float64)[:, None]).t()


def _chain(fmt, x, ids, w, ck, ks, ub=None, mods=None, defect=None):
    """The per-expert loop on the layers: g, u = layer(x rows), h = T(T(silu(g)) * u) (torch), yp = w * T(layer(h)).
    mods = (w1, w3, w2) module lists: the loop's own modules (exact for INT8 at any split); else the layer kernels at
    ks.  Returns (h [rows, I] sorted, ypair [rows, H] by pair).  defect (negative controls): "next_sw" = the next
    expert's w2 scales, "next_sin" = the next expert's input_scale for w1 / w3, "no_q_h" = down on the unquantised h."""
    T, top_k = ids.shape
    E, inter = ck["w1"][0].shape[:2]
    H, dt = ck["w2"][0].shape[1], x.dtype
    counts, offsets, pairs = _align(ids, E)
    h = torch.empty((T * top_k, inter), dtype=dt, device=DEV)
    yp = torch.zeros(T * top_k, H, dtype=torch.float32, device=DEV)
    wf = w.to(torch.float32).reshape(-1).to(DEV)

    def layer(role, e, xe, s_role=None):
        wr, sr, si = ck[role]
        if mods is not None and s_role is None:
            return mods[("w1", "w3", "w2").index(role)][e](xe)
        if si is not None:
            en = (e + 1) % E if defect == "next_sin" and role != "w2" else e
            c, s = _quantize(fmt, xe, s_in=si[en:en + 1])
        else:
            c, s = _quantize(fmt, xe, ub=ub)
        return _mm(fmt, c, s, wr[e], sr[e] if s_role is None else s_role, dt, ks)

    for e, r0, r1 in _expert_rows(counts, offsets):
        p = pairs[r0:r1].long()
        xe = x[p // top_k].contiguous()
        g, u = layer("w1", e, xe), layer("w3", e, xe)
        he = F.silu(g) * u
        h[r0:r1] = he
        if defect == "no_q_h":
            ye = (he.double() @ _deq(ck["w2"][0], ck["w2"][1], e)).to(dt)
        elif defect == "next_sw":
            ye = layer("w2", e, he, ck["w2"][1][(e + 1) % E].contiguous())
        else:
            ye = layer("w2", e, he)
        yp[p] = wf[p][:, None] * ye.float()
    return h, yp


def assert_block_equals_chain(fmt, block, chain, ck, ids, w, what, ub=None):
    """Every pair whose h row equals the chain's has a bit-identical ypair row, and every token whose pairs all do has a
    bit-identical output (the fp32 slot sum rounded once).  At least half of the pairs must be such pairs.  The others
    differ only through the requantisation of h: with s the larger of the two row scales, each requantised element
    moves by at most s + |dh| (INT8) or 2^-4 (|h| + |h'|) + 2^-9 s + |dh| (e4m3), so yp moves by at most
    B = sum_k bound_k |W2[k, n]| plus two ulps of T and 2^-12 sum_k (|h_k| + s) |W2[k, n]| for the accumulation."""
    pairs, h, yp, y = block
    h_c, yp_c = chain
    T, top_k = w.shape
    dt, H = y.dtype, y.shape[1]
    same_sorted = (h == h_c).all(1)
    pl = pairs.long()
    same = torch.zeros_like(same_sorted)
    same[pl] = same_sorted
    n_same = int(same.sum())
    assert n_same * 2 >= same.numel(), (what, "too few pairs without an exp flip", n_same, same.numel())
    assert torch.equal(yp[same], yp_c[same]), (what, "ypair of pairs with identical h")
    tok_same = same.view(T, top_k).all(1)
    y_c = yp_c.view(T, top_k, H)[:, 0].clone()
    for j in range(1, top_k):
        y_c = y_c + yp_c.view(T, top_k, H)[:, j]
    assert torch.equal(y[tok_same], y_c.to(dt)[tok_same]), (what, "outputs of tokens with identical h")
    flat = ids.reshape(-1).to(DEV)
    wf = w.to(torch.float32).reshape(-1).to(DEV)
    s_in2 = ck["w2"][2]
    qmax = 448.0 if fmt == "fp8" else 127.0
    worst = 0.0
    for r in (~same_sorted).nonzero().squeeze(1).tolist():
        p, e = int(pl[r]), int(flat[int(pl[r])])
        a, b = h[r].double(), h_c[r].double()
        if s_in2 is not None:
            s = float(s_in2[e])
        else:
            amax = float(torch.maximum(a.abs().max(), b.abs().max()))
            s = max(min(amax, INF if ub is None else ub), 1e-10) / qmax
        dh = (a - b).abs()
        bound = s + dh if fmt == "int8" else 2.0 ** -4 * (a.abs() + b.abs()) + 2.0 ** -9 * s + dh
        W2 = _deq(ck["w2"][0], ck["w2"][1], e).abs()
        B = bound @ W2 + 2.0 ** -12 * ((a.abs() + s) @ W2)
        ye_c = yp_c[p] / wf[p] if float(wf[p]) != 0 else yp_c[p]
        tol = wf[p].abs().double() * (B + 2 * _ulp(ye_c, dt).double()) + 1e-30
        err = (yp[p] - yp_c[p]).abs().double()
        worst = max(worst, float((err / tol).max()))
        assert (err <= tol).all(), (what, "pair", p, float((err / tol).max()))
    _record(what + " requantised pairs", 0.0, worst)
    return n_same


def coarse_oracle(fmt, kind, ub, x, ids, w, ck):
    """float64 y = sum_j w_j (silu(x W1) * (x W3)) W2 with the dequantised weights and x, h clipped to the range the
    quantisers represent (dynamic FP8: ub; static: qmax * s_in)."""
    T, top_k = ids.shape
    qmax = 448.0 if fmt == "fp8" else 127.0
    H = ck["w2"][0].shape[1]
    y = torch.zeros(T, H, dtype=torch.float64, device=DEV)
    xd = x.double()

    def clip(v, role, e):
        si = ck[role][2]
        if si is not None:
            lim = qmax * float(si[e])
        elif fmt == "fp8" and ub is not None:
            lim = ub
        else:
            return v
        return v.clamp(-lim, lim)

    for t in range(T):
        for j in range(top_k):
            e = int(ids[t, j])
            xe = clip(xd[t], "w1", e)
            hh = F.silu(xe @ _deq(*ck["w1"][:2], e)) * (xe @ _deq(*ck["w3"][:2], e))
            y[t] += float(w[t, j]) * (clip(hh, "w2", e) @ _deq(*ck["w2"][:2], e))
    return y


def assert_coarse(fmt, y, ref, what):
    err = float((y.double() - ref).norm() / ref.norm())
    _record(what + " (relative Frobenius error)", 0.0, err)
    assert err < (0.05 if fmt == "int8" else 0.15), (what, err)


# ---- stages -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("fmt,kind,ub", KINDS, ids=KIND_IDS)
def test_gather_equals_layer_quantisers(fmt, kind, ub, dt):
    """Sorted row i holds the layer quantiser's codes and scale of token sorted_pairs[i] / top_k bit for bit (static:
    with its expert's input_scale), with an all-zero row and a saturating row; the sorted mode (sorted_pairs NULL) equals
    the layer quantiser of each row.  The next expert's input_scale does not."""
    for T, top_k, K, E in ((1, 1, 128, 4), (5, 3, 512, 8), (300, 8, 2048, 64)):
        x = _x(T, K, dt, seed=T) * torch.logspace(-1, 1, T, device=DEV)[:, None].to(dt)
        x[0] = 0
        if T > 1:
            x[-1, 5] = 3000.0
        ids, _ = _route(T, E, top_k, seed=T + K)
        counts, offsets, pairs = _align(ids, E)
        s_in = _s_in(fmt, E, seed=T) if kind == "static" else None
        codes, sx = _gather(fmt, x, pairs, offsets, s_in, E, top_k, ub)
        xs = x[pairs.long() // top_k].contiguous()
        sc, ss = _gather(fmt, xs, None, offsets, s_in, E, 1, ub)
        assert torch.equal(sc, codes) and torch.equal(ss, sx), (T, K)
        for e, r0, r1 in _expert_rows(counts, offsets):
            wc, ws = _quantize(fmt, xs[r0:r1].contiguous(), None if s_in is None else s_in[e:e + 1], ub)
            assert torch.equal(codes[r0:r1], wc) and torch.equal(sx[r0:r1], ws), (T, K, e)
            if s_in is not None and E > 1 and bool(xs[r0:r1].abs().max() > 0):
                nc, _ = _quantize(fmt, xs[r0:r1].contiguous(), s_in[(e + 1) % E:(e + 1) % E + 1])
                assert not torch.equal(codes[r0:r1], nc), ("next expert's input_scale", e)


STAGE_CASES = [(8, 512, 384, 320, 5, 2, False), (16, 1024, 640, 512, 64, 4, False), (32, 2048, 768, 1024, 300, 8, False),
               (8, 1024, 512, 704, 257, 2, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("ks", [1, 2, 4])
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("fmt", ["fp8", "int8"])
def test_down_equals_layer_kernel(fmt, dt, ks):
    """Every row of ypair is w * T(b2q_*ch_mm(codes_h[expert rows], ...)) bit for bit at the same ks, per-channel and
    per-tensor scales (N = 320 / 704 leave a 64-feature tail tile)."""
    for i, (E, K, I, H, T, top_k, skew) in enumerate(STAGE_CASES):
        w2, s2, _ = _role(fmt, E, H, I, seed=E + T, per_tensor=i % 2 == 1)
        ids, w = (_skewed if skew else _route)(T, E, top_k, seed=T)
        counts, offsets, pairs = _align(ids, E)
        ch, sh = _quantize(fmt, _x(T * top_k, I, dt, seed=T))
        wts = w.to(torch.float32).contiguous()
        yp = _down(fmt, ch, sh, w2, s2, counts, offsets, pairs, wts, dt, ks)
        for e, r0, r1 in _expert_rows(counts, offsets):
            want = _mm(fmt, ch[r0:r1], sh[r0:r1], w2[e], s2[e], dt, ks).float()
            p = pairs[r0:r1].long()
            assert torch.equal(yp[p], wts.reshape(-1)[p][:, None] * want), (E, T, e, ks)


@pytest.mark.gpu
@pytest.mark.parametrize("ks", [1, 2, 4])
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("fmt", ["fp8", "int8"])
def test_gate_up_within_one_ulp_of_layer_kernels(fmt, dt, ks):
    """h = T(a * u) with g and u from b2q_*ch_mm per expert at the same ks and a = T(silu(g)) or one of its two
    neighbours in T (__expf against torch's exp)."""
    flips = total = 0
    for i, (E, K, I, H, T, top_k, skew) in enumerate(STAGE_CASES):
        w1, s1, _ = _role(fmt, E, I, K, seed=3 * E + T, per_tensor=i % 2 == 0)
        w3, s3, _ = _role(fmt, E, I, K, seed=3 * E + T + 1)
        x = _x(T, K, dt, seed=T)
        ids, _ = (_skewed if skew else _route)(T, E, top_k, seed=T)
        counts, offsets, pairs = _align(ids, E)
        codes, sx = _quantize(fmt, x[pairs.long() // top_k].contiguous())
        h = _gate_up(fmt, codes, sx, w1, s1, w3, s3, counts, offsets, dt, ks)
        for e, r0, r1 in _expert_rows(counts, offsets):
            g = _mm(fmt, codes[r0:r1], sx[r0:r1], w1[e], s1[e], dt, ks).float()
            u = _mm(fmt, codes[r0:r1], sx[r0:r1], w3[e], s3[e], dt, ks).float()
            a = (g / (1 + torch.exp(-g))).to(dt)
            want = (a.float() * u).to(dt)
            got = h[r0:r1]
            ok = got == want
            for step in (-1, 1):
                an = (a.view(torch.int16) + step).view(dt)
                ok |= got == (an.float() * u).to(dt)
            assert ok.all(), (E, T, e, ks, int((~ok).sum()))
            flips += int((got != want).sum())
            total += got.numel()
    _record(f"w8a8 moe {fmt} gate_up {TNAME[dt]} ks={ks}: {flips} of {total} elements differ from the exp mirror", 0.0,
            flips / total)


# ---- the block end to end -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("fmt,kind,ub", KINDS, ids=KIND_IDS)
def test_block_equals_loop(fmt, kind, ub, dt):
    """The grouped block against the per-expert loop: INT8 against the loop's own modules (exact sums: any split),
    FP8 against the layer kernels at the block's pinned ks = 1, 2.  Per-channel and per-tensor weight scales; the module
    forward equals the raw-ABI block at the heuristic split; the coarse float64 oracle holds.  Negative controls fail:
    swapped slot weights, the next expert's w2 scales, the next expert's input_scale (static) and down fed the
    unquantised h."""
    E, K, I, H, top_k = 16, 1024, 512, 768, 4
    for per_tensor in (False, True):
        ck, blk = _problem(fmt, kind, ub, E, K, I, H, seed=11 + per_tensor, per_tensor=per_tensor)
        mods = (list(blk.w1), list(blk.w3), list(blk.w2))
        for T in (1, 17, 300):
            x = _x(T, K, dt, seed=7 * T)
            for routing, (ids, w) in (("softmax", _route(T, E, top_k, seed=T)), ("skewed", _skewed(T, E, top_k, T))):
                what = f"w8a8 moe {fmt} {kind} ub={ub} {TNAME[dt]} pt={per_tensor} T={T} {routing}"
                y = blk(x, ids, w)
                assert torch.equal(y, _block_abi(fmt, x, ids, w, ck, 0, ub)[3]), what
                for ks in ((0,) if fmt == "int8" else (1, 2)):
                    chain = _chain(fmt, x, ids, w, ck, ks, ub, mods=mods if fmt == "int8" else None)
                    assert_block_equals_chain(fmt, _block_abi(fmt, x, ids, w, ck, ks or 2, ub), chain, ck, ids, w,
                                              f"{what} ks={ks}", ub)
                if T == 17:
                    assert_coarse(fmt, y, coarse_oracle(fmt, kind, ub, x, ids, w, ck), what)
    T = 64
    x = _x(T, K, dt, seed=64)
    ids, w = _route(T, E, top_k, seed=64)
    block = _block_abi(fmt, x, ids, w, ck, 1, ub)
    defects = [("swapped", None), ("next_sw", "next_sw"), ("no_q_h", "no_q_h")]
    if kind == "static":
        defects.append(("next_sin", "next_sin"))
    for what, defect in defects:
        ww = w[:, [1, 0, 2, 3]] if what == "swapped" else w
        with pytest.raises(AssertionError):
            assert_block_equals_chain(fmt, block, _chain(fmt, x, ids, ww, ck, 1, ub, defect=defect), ck, ids, ww,
                                      f"control {what}", ub)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,kind,ub", [KINDS[0], KINDS[4]], ids=["fp8_dyn", "int8_static"])
def test_routing(fmt, kind, ub):
    """T = 1 .. 16, a sample to 300 and 2048; top_k 1, 2, 4, 8; softmax, skewed and sparse routing (most experts empty):
    the block (ks pinned to 1) against the loop chain at ks = 1."""
    E, K, I, H = 16, 512, 256, 384
    ck, blk = _problem(fmt, kind, ub, E, K, I, H, seed=5)
    blk.ks = 1
    mods = (list(blk.w1), list(blk.w3), list(blk.w2))
    for dt in DTYPES:
        for T in list(range(1, 17)) + [37, 100, 211, 300, 2048]:
            top_k = (1, 2, 4, 8)[T % 4]
            x = _x(T, K, dt, seed=T)
            ids, w = _route(T, E, top_k, seed=T)
            routings = {"softmax": (ids, w), "skewed": _skewed(T, E, top_k, seed=T)}
            if T in (16, 300):
                routings["sparse"] = (torch.where(ids % 4 == 0, ids, torch.full_like(ids, E - 1)), w)
            for r, (ids_r, w_r) in routings.items():
                what = f"w8a8 moe routing {fmt} {kind} {TNAME[dt]} T={T} top_k={top_k} {r}"
                block = _block_abi(fmt, x, ids_r, w_r, ck, 1, ub)
                assert torch.equal(blk(x, ids_r, w_r), block[3]), what
                chain = _chain(fmt, x, ids_r, w_r, ck, 1, ub, mods=mods if fmt == "int8" else None)
                assert_block_equals_chain(fmt, block, chain, ck, ids_r, w_r, what, ub)


@pytest.mark.gpu
def test_large_prefill_splits_the_grid():
    """E = 256, top_k = 8, T = 8192: 65536 rows in 128-row blocks give 256 * 512 (expert, token block) pairs, so both
    grouped launches are issued over several ranges of gridDim.z, with populated blocks past the first."""
    E, K, I, H, top_k, T = 256, 256, 128, 256, 8, 8192
    ids, w = _route(T, E, top_k, seed=5)
    counts = torch.bincount(ids.reshape(-1).cpu(), minlength=E)
    assert int(counts[E // 2:].sum()) > 0 and (E - 1) * 512 >= 65535
    for fmt, kind in (("int8", "dynamic"), ("fp8", "static")):
        ck, blk = _problem(fmt, kind, None, E, K, I, H, seed=9)
        mods = (list(blk.w1), list(blk.w3), list(blk.w2))
        x = _x(T, K, torch.bfloat16, seed=T)
        block = _block_abi(fmt, x, ids, w, ck, 0)
        assert torch.equal(blk(x, ids, w), block[3])
        # K = I = 256: every layer call and both grouped launches run ks = 1, so the modules are the chain for both
        assert_block_equals_chain(fmt, block, _chain(fmt, x, ids, w, ck, 1, mods=mods), ck, ids, w,
                                  f"w8a8 moe large prefill {fmt}")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,kind,ub", [KINDS[0], KINDS[4]], ids=["fp8_dyn", "int8_static"])
def test_graph_replay_equals_eager(fmt, kind, ub):
    """The six launches captured in a CUDA graph read the routing from the device: after new ids / weights are copied in,
    a replay equals an eager run bit for bit."""
    E, K, I, H, top_k, T = 32, 1024, 512, 1024, 8, 65
    ck, blk = _problem(fmt, kind, ub, E, K, I, H, seed=13)
    for dt in DTYPES:
        x = _x(T, K, dt, seed=65)
        ids, w = _route(T, E, top_k, seed=65)
        idc, wc = ids.clone(), w.clone()
        s_ = torch.cuda.Stream()
        s_.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s_):
            blk(x, idc, wc)
        torch.cuda.current_stream().wait_stream(s_)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            yg = blk(x, idc, wc)
        for what, (ids2, w2) in (("skewed", _skewed(T, E, top_k, seed=7)), ("softmax", _route(T, E, top_k, seed=66))):
            idc.copy_(ids2)
            wc.copy_(w2)
            gr.replay()
            torch.cuda.synchronize()
            assert torch.equal(yg, blk(x, ids2, w2)), (what, dt)
        del gr


@pytest.mark.gpu
def test_refused_stacks_take_the_loop():
    """Each disqualifying condition keeps the loop under grouped=None and raises under grouped=True; MoEExperts itself
    keeps the loop for a qualifying W8A8 stack."""
    from gptqmodel_b200 import B200ChannelW8A8Experts, Lora, moe

    E, K, I = 4, 256, 256

    def sets(fmt="fp8", kind="dynamic", ub=None, inter=I, seed=21):
        s13 = _s_in(fmt, E, seed) if kind == "static" else None
        s2 = _s_in(fmt, E, seed + 1) if kind == "static" else None
        out = []
        for N, Kr, si, sd in ((inter, K, s13, 1), (inter, K, s13, 2), (K, inter, s2, 3)):
            w, _, ms = _role(fmt, E, N, Kr, seed + sd)
            out.append(_modules(fmt, kind, ub, w, ms, si))
        return out

    good = sets()
    assert B200ChannelW8A8Experts(*good)._stack is not None
    assert moe.MoEExperts(*sets())._stack is None
    gen = torch.Generator().manual_seed(0)
    lora = Lora(lora_A=(torch.randn(K, 8, generator=gen) * 0.05).half(),
                lora_B=(torch.randn(8, I, generator=gen) * 0.05).half())
    cases = {}
    s = sets()
    s[2][1] = _cls("fp8").from_checkpoint_tensors(s[2][1].weight, s[2][1].weight_scale,
                                                  bias=torch.zeros(K, dtype=torch.float16), device=DEV)
    cases["bias"] = s
    s = sets()
    s[0][0] = _cls("fp8").from_checkpoint_tensors(s[0][0].weight, s[0][0].weight_scale, device=DEV, adapter=lora)
    cases["adapter"] = s
    s = sets()
    s[1][2] = sets(fmt="int8")[1][2]
    cases["mixed fp8 / int8"] = s
    s = sets()
    s[2] = sets(kind="static")[2]
    cases["activation kinds"] = s
    s = sets(ub=2.0)
    s[0][3] = sets(ub=3.0)[0][3]
    cases["ub"] = s
    s = sets(kind="static")
    s[1][1] = sets(kind="static", seed=40)[1][1]
    cases["w1 / w3 input_scale"] = s
    s = sets()
    s[2] = s[2][:3] + [_modules("fp8", "dynamic", None, *_role("fp8", 1, 128, I, 5)[::2], None)[0]]
    cases["w2 shape"] = s
    for what, st in cases.items():
        assert B200ChannelW8A8Experts(*st)._stack is None, what
        with pytest.raises(ValueError, match="B200ChannelW8A8Experts"):
            B200ChannelW8A8Experts(*st, grouped=True)
    T = 9
    x = _x(T, K, torch.float16, seed=9)
    ids, w = _route(T, E, 2, seed=9)
    assert B200ChannelW8A8Experts(*cases["bias"])(x, ids, w).shape == (T, K)  # the loop still runs
    blk = B200ChannelW8A8Experts(*sets(), grouped=True)
    for bad_x, bad_ids in ((x[:, :128], ids), (x[:8], ids), (x, ids[:8])):  # shapes that do not fit the block
        with pytest.raises(ValueError, match="does not fit"):
            blk(bad_x.contiguous(), bad_ids, w[:bad_ids.shape[0]])


# ---- checkpoints --------------------------------------------------------------------------------------------------------
def _ct_group(typ, w_strategy, a_strategy, dynamic):
    q = lambda strategy, dyn: {"num_bits": 8, "type": typ, "symmetric": True, "group_size": None,  # noqa: E731
                               "strategy": strategy, "block_structure": None, "dynamic": dyn, "actorder": None}
    return {"quant_method": "compressed-tensors", "format": "float-quantized" if typ == "float" else "int-quantized",
            "quantization_status": "compressed", "ignore": ["lm_head", "re:.*mlp\\.gate$"],
            "config_groups": {"group_0": {"targets": ["Linear"], "weights": q(w_strategy, False),
                                          "input_activations": q(a_strategy, dynamic), "output_activations": None}}}


CHECKPOINTS = {
    "fp8_dynamic": ("fp8", _ct_group("float", "channel", "token", True)),
    "fp8_static": ("fp8", _ct_group("float", "tensor", "tensor", False)),
    "int8_w8a8": ("int8", _ct_group("int", "channel", "token", True)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CHECKPOINTS))
def test_qwen3_moe_checkpoint_through_loader(tmp_path, name):
    """A tiny compressed-tensors checkpoint with Qwen3-MoE module names (router ignored), loaded by the existing W8A8
    loader into B200ChannelW8A8Experts: the block equals the loop over the same modules (K = I = 256, so every call runs
    ks = 1) and holds the coarse oracle."""
    from safetensors.torch import save_file

    from gptqmodel_b200 import B200ChannelW8A8Experts
    from gptqmodel_b200.loader import load_fp8_w8a8_linears, load_int8_w8a8_linears

    fmt, cfg = CHECKPOINTS[name]
    static = name == "fp8_static"
    E, K, I = 4, 256, 256
    proj = {"w1": "gate_proj", "w3": "up_proj", "w2": "down_proj"}
    tensors = {"model.layers.0.mlp.gate.weight": torch.randn(E, K).to(torch.bfloat16)}
    s13, s2 = _s_in(fmt, E, 3), _s_in(fmt, E, 4)
    for r, (N, Kr) in (("w1", (I, K)), ("w3", (I, K)), ("w2", (K, I))):
        w, _, ms = _role(fmt, E, N, Kr, seed=len(r) + ord(r[1]), per_tensor=static)
        for e in range(E):
            pre = f"model.layers.0.mlp.experts.{e}.{proj[r]}"
            tensors[pre + ".weight"] = w[e].cpu().contiguous()
            tensors[pre + ".weight_scale"] = (ms[e].reshape(1) if static else ms[e][:, None]).cpu().contiguous()
            if static:
                tensors[pre + ".input_scale"] = (s2 if r == "w2" else s13)[e:e + 1].cpu().contiguous()
    with open(os.path.join(tmp_path, "config.json"), "w") as f:
        json.dump({"model_type": "qwen3_moe", "quantization_config": cfg}, f)
    save_file(tensors, os.path.join(tmp_path, "model.safetensors"))
    mods = (load_fp8_w8a8_linears if fmt == "fp8" else load_int8_w8a8_linears)(str(tmp_path), device=DEV)
    assert len(mods) == 3 * E
    get = lambda r: [mods[f"model.layers.0.mlp.experts.{e}.{proj[r]}"] for e in range(E)]  # noqa: E731
    blk = B200ChannelW8A8Experts(get("w1"), get("w3"), get("w2"), grouped=True)
    st = blk._stack
    ck = {r: (st[r]["weight"], st[r]["scale"], st[r]["s_in"]) for r in ("w1", "w3", "w2")}
    assert (ck["w1"][2] is not None) == static
    chain_mods = (list(blk.w1), list(blk.w3), list(blk.w2))
    for dt in DTYPES:
        for T, top_k in ((9, 2), (64, 4)):
            x = _x(T, K, dt, seed=T)
            ids, w = _route(T, E, top_k, seed=T)
            what = f"w8a8 moe checkpoint {name} {TNAME[dt]} T={T}"
            block = _block_abi(fmt, x, ids, w, ck, 0)
            assert torch.equal(blk(x, ids, w), block[3]), what
            assert_block_equals_chain(fmt, block, _chain(fmt, x, ids, w, ck, 1, mods=chain_mods), ck, ids, w, what)
            assert_coarse(fmt, blk(x, ids, w), coarse_oracle(fmt, "static" if static else "dynamic", None, x, ids, w, ck),
                          what)
