"""Block-FP8 MoE experts (DeepSeek-V3, Qwen3-MoE FP8) on the grouped e4m3 path of gptqmodel_b200/moe.py.

Path: b2q_moe_align -> b2q_fp8blk_moe_gather (quantise the sorted rows) -> fp8blk_moe_gemm_kernel MODE 1 (gate|up, SiLU-mul
epilogue) -> b2q_fp8blk_quantize of h -> MODE 2 (down, routing weight, scatter) -> b2q_moe_combine.  The stages are
checked exactly against the layer kernels and oracle/fp8_block_oracle.py, the block end to end against the layer kernels and a float64 oracle.

Oracle.  T(.) rounds to the run dtype, Q(.) is the per-token-group quantiser (fo.quantize, bit-exact).  For every routed
pair (token t, slot j, expert e):
    (c, s_x) = Q(x_t),  g = T(sum_b s_x s_w1 P_b),  u = T(... W3_e ...),  a = T(silu(g)),  h = T(a * u)
    (c_h, s_h) = Q(h),  yp_j = T(sum_b s_h s_w2 P_b),  y_t = T(sum_j fp32(w_j * yp_j))
with the block sums P_b exact in float64 (products of e4m3 values are exact) and the oracle's own h re-quantised.

Two end-to-end checks.  The tight one is test_block_equals_layer_kernel_chain: the layer kernels share the e4m3 tensor
cores' accumulation, so the block must equal transformers' per-expert FP8Linear loop built from b2q_fp8blk_mm at the same
split bit for bit, except where torch's exp and __expf round T(silu(g)) differently (assert_block_equals_chain).  The
float64 oracle is the independent, coarse one.  Its tolerance cannot be tight: the e4m3 wgmma accumulates each 128-k
block with fewer bits than fp32.  On an H100, 30 % of fp16 and 6.6 % of bf16 outputs of b2q_fp8blk_mm (K = 2048,
random data) round to a different T value than the exact sum, with deviations up to 2^-14.2 of sum |s_x s_w q w|.  So g,
u and h differ from the oracle's in a large share of elements, and a changed element or group amax can move codes of
Q(h) by one e4m3 step (2^-3 |h_k| for normal codes, 2^-9 s_h for subnormal ones, plus the ulp of h).  Per group g of
pair j that moves yp_j before rounding by at most
    B_g = 9/64 sum_{k in g} (|h_k| + 2^-14 amax_g) |W2[k, n]|,
and the slack charges the two groups of largest B_g of every pair with the one-ulp flip of yp_j as in
tests/test_gpu_moe.py:
    slack_t = sum_j |w_j| (ulp(yp_j) + B_(1) + B_(2) + 2^-18 sum_k |c_h s_h| |W2|)
on top of rel * (|y| + rms(y)) with the rel of tests/test_gpu_moe.py.  This is of the order of |y| itself: it catches
wrong experts, routing, scales of the wrong order or garbage, not a deviation of a few percent.  Those are left to the
chain check, whose negative controls include down_proj on the unquantised h and w2 scales 2 % off.  The worst
err / tol of each comparison goes to parity.json.
"""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import _record, assert_close_rel
from oracle import fp8_block_oracle as fo
from test_gpu_moe import REL, _route, _skewed, _ulp

DEV = "cuda"
DTYPES = (torch.float16, torch.bfloat16)
TNAME = {torch.float16: "fp16", torch.bfloat16: "bf16"}
DT = {torch.float16: 0, torch.bfloat16: 1}

# experts E, hidden K, intermediate I, top_k of the model (the routing tests vary top_k)
STACKS = {
    "qwen3_30b_a3b": (128, 2048, 768, 8),
    "qwen3_235b_a22b": (128, 4096, 1536, 8),
    "deepseek_v3_ep8": (32, 7168, 2048, 8),  # the 256 routed experts over 8 GPUs of expert parallelism
    "edge_tail_top1": (4, 256, 640, 1),        # 10 paired gate|up tiles
    "edge_tail_top2": (4, 384, 384, 2),        # 3 down tiles
}
REAL = ("qwen3_30b_a3b", "qwen3_235b_a22b", "deepseek_v3_ep8")


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _mp(M):
    return (M + 3) // 4 * 4


# ---- checkpoint tensors -------------------------------------------------------------------------------------------------
def _role(E, N, K, seed):
    """Stacked e4m3 weights [E, N, K] and scales [E, ceil(N/128), K/128]; W = w * s has about unit-variance dot products."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    w = (torch.randn(E, N, K, device=DEV, generator=gen) * 60).clamp(-448, 448).to(torch.float8_e4m3fn)
    s = (torch.rand(E, (N + 127) // 128, K // 128, device=DEV, generator=gen) + 0.5) / (60 * K ** 0.5)
    return w, s


def _modules(w, s):
    from gptqmodel_b200 import B200BlockFp8Linear

    return [B200BlockFp8Linear.from_checkpoint_tensors(w[e], s[e], device=DEV) for e in range(w.shape[0])]


_BLOCKS = {}


@pytest.fixture(scope="module", autouse=True)
def _release_stacks():
    yield
    _BLOCKS.clear()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _stack(name):
    """(checkpoint {role: (w, s)}, grouped block, loop block over the same modules)."""
    if name not in _BLOCKS:
        from gptqmodel_b200 import moe

        _BLOCKS.clear()  # one real stack on the device at a time
        torch.cuda.empty_cache()
        E, K, I, _ = STACKS[name]
        ck = {"w1": _role(E, I, K, 1), "w3": _role(E, I, K, 2), "w2": _role(E, K, I, 3)}
        blk = moe.MoEExperts(*[_modules(*ck[r]) for r in ("w1", "w3", "w2")])
        assert blk._stack is not None and "fp8blk" in blk._stack, name
        loop = moe.MoEExperts(list(blk.w1), list(blk.w3), list(blk.w2), grouped=False)
        assert loop._stack is None
        _BLOCKS[name] = (ck, blk, loop)
    return _BLOCKS[name]


# ---- float64 oracle -----------------------------------------------------------------------------------------------------
def _deq_codes(codes, s, dev):
    """fo.quantize's (codes [M, K], s [M, K/128]) -> float64 [M, K] on dev."""
    v = torch.from_numpy(fo.e4m3_decode(codes)).to(dev)
    return v * torch.from_numpy(s.astype(np.float64)).to(dev).repeat_interleave(128, 1)


def _deq_w(w, s, e):
    """W_e^T [K, N] float64: e4m3 * s_w, exact."""
    N = w.shape[1]
    return (w[e].to(torch.float64) * s[e].to(torch.float64).repeat_interleave(128, 0)[:N].repeat_interleave(128, 1)).t()


def fp8_moe_oracle(x, ids, w, ck):
    """(y [T, H] in x.dtype, slack [T, H] float32) with the rounding points and the slack of the module docstring.
    ck[role] = (e4m3 [E, N, K], fp32 [E, ceil(N/128), K/128]) on x's device."""
    dt, dev = x.dtype, x.device
    T, top_k = ids.shape
    R = lambda v: v.to(dt).to(torch.float64)  # noqa: E731
    flat = ids.reshape(-1).to(dev)
    cx, sx = fo.quantize(x.float().cpu().numpy())
    xq = _deq_codes(cx, sx, dev)
    H = ck["w2"][0].shape[1]
    yp = torch.zeros(T * top_k, H, dtype=torch.float64, device=dev)
    sl = torch.zeros(T * top_k, H, dtype=torch.float32, device=dev)
    for e in torch.unique(flat).tolist():
        pairs = (flat == e).nonzero().squeeze(1)
        xe = xq.index_select(0, pairs // top_k)
        g, u = R(xe @ _deq_w(*ck["w1"], e)), R(xe @ _deq_w(*ck["w3"], e))
        h = R(R(F.silu(g)) * u)
        ch, sh = fo.quantize(h.float().cpu().numpy())
        W2 = _deq_w(*ck["w2"], e)
        hq = _deq_codes(ch, sh, dev)
        yp[pairs] = R(hq @ W2)
        # slack: the two groups of largest B_g, and the promotion chain
        hh, aw = h.abs().float(), W2.abs().float()
        amax = hh.view(hh.shape[0], -1, 128).amax(2)
        b1 = b2 = torch.zeros(hh.shape[0], H, device=dev)
        for gi in range(amax.shape[1]):
            k0 = 128 * gi
            bg = (9 / 64) * ((hh[:, k0:k0 + 128] + 2.0 ** -14 * amax[:, gi:gi + 1]) @ aw[k0:k0 + 128])
            b2 = torch.maximum(b2, torch.minimum(b1, bg))
            b1 = torch.maximum(b1, bg)
        mag = hq.abs().float() @ aw
        sl[pairs] = b1 + b2 + 2.0 ** -18 * mag
    yp = yp.to(torch.float32).view(T, top_k, -1)
    wf = w.to(device=dev, dtype=torch.float32)
    acc = torch.zeros(T, H, dtype=torch.float32, device=dev)
    for j in range(top_k):
        acc = acc + wf[:, j:j + 1] * yp[:, j]
    slack = (wf.abs()[:, :, None] * (_ulp(yp, dt) + sl.view(T, top_k, -1))).sum(1)
    return acc.to(dt), slack


def assert_fp8_moe_close(out, oracle_out, what):
    ref, slack = oracle_out
    assert out.shape == ref.shape and out.dtype == ref.dtype, (what, out.shape, out.dtype)
    assert_close_rel(out, ref, REL[ref.dtype], what, slack=slack.cpu())


def _x(T, K, dt, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(T, K, device=DEV, generator=gen).to(dt)


# ---- stages through the raw ABI -----------------------------------------------------------------------------------------
def _align(ids, E):
    from gptqmodel_b200._lib import check, lib

    T, top_k = ids.shape
    ids = ids.to(torch.int32).contiguous()
    tables = torch.empty(2 * E + T * top_k, dtype=torch.int32, device=DEV)
    counts, offsets, pairs = tables[:E], tables[E:2 * E], tables[2 * E:]
    check(lib.b2q_moe_align(_p(ids), T, top_k, E, _p(counts), _p(offsets), _p(pairs), _st()), "b2q_moe_align")
    return counts, offsets, pairs


def _gather(x, pairs, top_k):
    from gptqmodel_b200._lib import check, lib

    T, K = x.shape
    rows = T * top_k
    codes = torch.full((rows, K), 0x7F, dtype=torch.uint8, device=DEV)
    sx = torch.zeros((K // 128, _mp(rows)), dtype=torch.float32, device=DEV)
    check(lib.b2q_fp8blk_moe_gather(_p(x), _p(pairs), _p(codes), _p(sx), T, top_k, K, DT[x.dtype], _st()),
          "b2q_fp8blk_moe_gather")
    return codes, sx


def _quantize(x):
    from gptqmodel_b200._lib import check, lib

    M, K = x.shape
    codes = torch.empty((M, K), dtype=torch.uint8, device=DEV)
    sx = torch.zeros((K // 128, _mp(M)), dtype=torch.float32, device=DEV)
    check(lib.b2q_fp8blk_quantize(_p(x), _p(codes), _p(sx), M, K, DT[x.dtype], _st()), "b2q_fp8blk_quantize")
    return codes, sx


def _mm(codes, sx, w, s, dt, ks):
    from gptqmodel_b200._lib import check, lib

    M, K = codes.shape
    N = w.shape[0]
    out = torch.empty((M, N), dtype=dt, device=DEV)
    check(lib.b2q_fp8blk_mm(_p(codes), _p(sx), _p(w), _p(s), None, _p(out), M, K, N, DT[dt], ks, _st()), "b2q_fp8blk_mm")
    return out


def _gate_up(codes, sx, w1, s1, w3, s3, counts, offsets, dt, ks):
    from gptqmodel_b200._lib import check, lib

    rows, K = codes.shape
    E, N = w1.shape[:2]
    h = torch.full((rows, N), float("nan"), dtype=dt, device=DEV)
    check(lib.b2q_fp8blk_moe_gate_up(_p(codes), _p(sx), _p(w1), _p(s1), _p(w3), _p(s3), _p(h), _p(counts), _p(offsets),
                                     E, rows, min(E, rows), K, N, DT[dt], ks, _st()), "b2q_fp8blk_moe_gate_up")
    return h


def _down(codes, sx, w2, s2, counts, offsets, pairs, wts, dt, ks):
    from gptqmodel_b200._lib import check, lib

    rows, K = codes.shape
    E, N = w2.shape[:2]
    yp = torch.full((rows, N), float("nan"), dtype=torch.float32, device=DEV)
    check(lib.b2q_fp8blk_moe_down(_p(codes), _p(sx), _p(w2), _p(s2), _p(counts), _p(offsets), _p(pairs), _p(wts),
                                  _p(yp), E, rows, min(E, rows), K, N, DT[dt], ks, _st()), "b2q_fp8blk_moe_down")
    return yp


def _expert_rows(counts, offsets):
    c, o = counts.cpu().tolist(), offsets.cpu().tolist()
    return [(e, o[e], o[e] + c[e]) for e in range(len(c)) if c[e] > 0]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_gather_quantise_equals_oracle(dt):
    """Sorted row i holds fo.quantize(x)[sorted_pairs[i] / top_k] bit for bit, with an all-zero group, a group of one
    huge value among zeros and a saturating group."""
    for T, top_k, K, E in ((1, 1, 128, 4), (5, 3, 512, 8), (300, 8, 2048, 128), (33, 6, 7168, 32)):
        x = _x(T, K, dt, seed=T) * torch.logspace(-2, 2, T, device=DEV)[:, None].to(dt)
        x[0, :128] = 0
        if K >= 512:
            x[0, 130] = 20000.0 if dt == torch.float16 else 1e20
            x[-1, 256:384] = -x[-1, 256:384].abs().max() - 1
        ids, _ = _route(T, E, top_k, seed=T + K)
        _, _, pairs = _align(ids, E)
        codes, sx = _gather(x, pairs, top_k)
        want_c, want_s = fo.quantize(x.float().cpu().numpy())
        tok = (pairs.long() // top_k).cpu().numpy()
        assert torch.equal(codes.cpu(), torch.from_numpy(want_c[tok])), (T, top_k, K)
        assert torch.equal(sx[:, :T * top_k].cpu(), torch.from_numpy(want_s[tok].T.copy())), (T, top_k, K)


def _stage_problem(E, K, I, H, T, top_k, dt, seed, skew=False):
    ck = {"w1": _role(E, I, K, seed), "w3": _role(E, I, K, seed + 1), "w2": _role(E, H, I, seed + 2)}
    x = _x(T, K, dt, seed)
    ids, w = (_skewed if skew else _route)(T, E, top_k, seed)
    return ck, x, ids, w


STAGE_CASES = [(8, 512, 384, 320, 5, 2, False), (16, 1024, 640, 512, 64, 4, False), (32, 2048, 768, 1024, 300, 8, False),
               (8, 1024, 512, 704, 257, 2, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("ks", [1, 2, 4])
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_down_equals_layer_kernel(dt, ks):
    """Every row of ypair is w * T(b2q_fp8blk_mm(codes_h[expert rows], ...)) bit for bit at the same ks: the grouped mode
    runs the dense kernel's promotion chain (N = 320 / 704 leave a 64-feature tail tile)."""
    for E, K, I, H, T, top_k, skew in STAGE_CASES:
        ck, _, ids, w = _stage_problem(E, K, I, H, T, top_k, dt, seed=E + T, skew=skew)
        counts, offsets, pairs = _align(ids, E)
        h = _x(T * top_k, I, dt, seed=T)
        ch, sh = _quantize(h)
        wts = w.to(torch.float32).contiguous()
        yp = _down(ch, sh, *ck["w2"], counts, offsets, pairs, wts, dt, ks)
        for e, r0, r1 in _expert_rows(counts, offsets):
            ce, se = _quantize(h[r0:r1].contiguous())
            want = _mm(ce, se, ck["w2"][0][e], ck["w2"][1][e].clone(), dt, ks).float()
            p = pairs[r0:r1].long()
            want = wts.reshape(-1)[p][:, None] * want
            assert torch.equal(yp[p], want), (E, T, e, ks)


@pytest.mark.gpu
@pytest.mark.parametrize("ks", [1, 2, 4])
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_gate_up_within_one_ulp_of_layer_kernels(dt, ks):
    """h = T(a * u) with g and u from b2q_fp8blk_mm per expert at the same ks and a = T(silu(g)) or one of its two
    neighbours in T: the only difference allowed is __expf against torch's exp, which can flip a by one ulp (and h by up
    to two).  The flips of h are counted and recorded."""
    flips = total = 0
    for E, K, I, H, T, top_k, skew in STAGE_CASES:
        ck, x, ids, _ = _stage_problem(E, K, I, H, T, top_k, dt, seed=3 * E + T, skew=skew)
        counts, offsets, pairs = _align(ids, E)
        codes, sx = _gather(x, pairs, top_k)
        h = _gate_up(codes, sx, *ck["w1"], *ck["w3"], counts, offsets, dt, ks)
        for e, r0, r1 in _expert_rows(counts, offsets):
            ce, se = _quantize(x[pairs[r0:r1].long() // top_k].contiguous())
            g = _mm(ce, se, ck["w1"][0][e], ck["w1"][1][e].clone(), dt, ks).float()
            u = _mm(ce, se, ck["w3"][0][e], ck["w3"][1][e].clone(), dt, ks).float()
            a = (g / (1 + torch.exp(-g))).to(dt)
            want = (a.float() * u).to(dt)
            got = h[r0:r1]
            ok = got == want
            for step in (-1, 1):  # the neighbours of a in T (bit patterns of the same sign; a NaN never matches)
                an = (a.view(torch.int16) + step).view(dt)
                ok |= got == (an.float() * u).to(dt)
            assert ok.all(), (E, T, e, ks, int((~ok).sum()))
            flips += int((got != want).sum())
            total += got.numel()
    _record(f"fp8 moe gate_up {TNAME[dt]} ks={ks}: {flips} of {total} elements differ from the exp mirror", 0.0, flips / total)


INT_CODES = np.array([0x00, 0x38, 0x40, 0x44, 0x48, 0xB8, 0xC0, 0xC4, 0xC8], np.uint8)  # 0, +-1, +-2, +-3, +-4
POS_CODES = np.array([0x38, 0x40, 0x44, 0x48], np.uint8)  # 1, 2, 3, 4


@pytest.mark.gpu
@pytest.mark.parametrize("ks", [1, 2, 4])
def test_integer_problems_equal_promotion_mirror(ks):
    """The small-integer code problems of tests/test_gpu_fp8_block.py through both grouped modes: K = 1024, N = 320 (a
    64-feature tail), three experts with 0 / 37 / 91 / 2 rows.  Down: ypair = w * T(fo.promote) bit for bit.  Gate|up:
    the gate codes are positive with large scales, so g > 20 and silu(g) = g in fp32 whatever exp gives; then
    h = T(T(g) * T(u)) bit for bit."""
    rng = np.random.default_rng(ks)
    E, K, N = 4, 1024, 320
    cnt = [0, 37, 91, 2]
    rows = sum(cnt)
    ids = torch.tensor(sum(([e] * c for e, c in enumerate(cnt)), []), dtype=torch.int32)[torch.randperm(rows)]
    ids = ids.view(rows, 1).to(DEV)
    counts, offsets, pairs = _align(ids, E)
    KB, NS = K // 128, (N + 127) // 128
    xc = POS_CODES[rng.integers(0, 4, (rows, K))]
    sx = (rng.random((KB, _mp(rows))) * 3 + 0.01).astype(np.float32) * np.float32(2.0 ** -7)
    w1 = POS_CODES[rng.integers(0, 4, (E, N, K))]
    s1 = (rng.random((E, NS, KB)) * 2 + 1).astype(np.float32)
    w3 = INT_CODES[rng.integers(0, len(INT_CODES), (E, N, K))]
    s3 = (rng.random((E, NS, KB)) * 2 + 0.001).astype(np.float32) * np.float32(2.0 ** -9)
    wts = torch.rand(rows, generator=torch.Generator().manual_seed(ks)).to(DEV)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    for dt in DTYPES:
        h = _gate_up(d(xc), d(sx), d(w1), d(s1), d(w3), d(s3), counts, offsets, dt, ks)
        yp = _down(d(xc), d(sx), d(w3), d(s3), counts, offsets, pairs, wts, dt, ks)
        for e, r0, r1 in _expert_rows(counts, offsets):
            c, s = xc[r0:r1], sx[:, r0:r1].T
            g = fo.promote(c, s, w1[e], s1[e], ks)
            assert (g > 20).all()
            u = fo.promote(c, s, w3[e], s3[e], ks)
            want_h = fo.round_t(fo.round_t(g, TNAME[dt]) * fo.round_t(u, TNAME[dt]), TNAME[dt])
            assert torch.equal(h[r0:r1].float().cpu(), torch.from_numpy(want_h)), (dt, e, ks)
            p = pairs[r0:r1].long()
            want_y = wts[p].cpu()[:, None] * torch.from_numpy(fo.round_t(u, TNAME[dt]))
            assert torch.equal(yp[p].cpu(), want_y), (dt, e, ks)


# ---- the block end to end -----------------------------------------------------------------------------------------------
def _block_abi(x, ids, w, ck, ks):
    """The six launches of MoEExperts' grouped block-FP8 path through the raw ABI with ks pinned (0 = the heuristic the
    module runs): (sorted_pairs, h [rows, I] in sorted order, ypair [rows, H] by pair, y [T, H])."""
    from gptqmodel_b200._lib import check, lib

    T, top_k = ids.shape
    E = ck["w1"][0].shape[0]
    H, dt = ck["w2"][0].shape[1], x.dtype
    counts, offsets, pairs = _align(ids, E)
    codes, sx = _gather(x, pairs, top_k)
    h = _gate_up(codes, sx, *ck["w1"], *ck["w3"], counts, offsets, dt, ks)
    ch, sh = _quantize(h)
    yp = _down(ch, sh, *ck["w2"], counts, offsets, pairs, w.to(torch.float32).contiguous(), dt, ks)
    y = torch.empty((T, H), dtype=dt, device=DEV)
    check(lib.b2q_moe_combine(_p(yp), _p(y), T, top_k, H, DT[dt], _st()), "b2q_moe_combine")
    return pairs, h, yp, y


def _layer_chain(x, ids, w, ck, ks, defect=None):
    """transformers' per-expert FP8Linear loop on the layer kernels at the same ks: per expert g, u = b2q_fp8blk_mm(Q(x)),
    h = T(T(silu(g)) * u) with torch's exp, yp = w * T(b2q_fp8blk_mm(Q(h))).  Returns (h [rows, I] in sorted order,
    ypair [rows, H] by pair).  defect (negative controls): "no_q_h" = down_proj on the 16-bit h (float64 product,
    rounded once), "scale_2pct" = w2 scales 2 % high, "next_scales" = the next expert's w2 scales."""
    T, top_k = ids.shape
    E, inter = ck["w1"][0].shape[:2]
    H, dt = ck["w2"][0].shape[1], x.dtype
    counts, offsets, pairs = _align(ids, E)
    h = torch.empty((T * top_k, inter), dtype=dt, device=DEV)
    yp = torch.zeros(T * top_k, H, dtype=torch.float32, device=DEV)
    wf = w.to(torch.float32).reshape(-1)
    for e, r0, r1 in _expert_rows(counts, offsets):
        p = pairs[r0:r1].long()
        ce, se = _quantize(x[p // top_k].contiguous())
        g = _mm(ce, se, ck["w1"][0][e], ck["w1"][1][e].clone(), dt, ks).float()
        u = _mm(ce, se, ck["w3"][0][e], ck["w3"][1][e].clone(), dt, ks).float()
        he = ((g / (1 + torch.exp(-g))).to(dt).float() * u).to(dt)
        h[r0:r1] = he
        s2 = ck["w2"][1][(e + 1) % E if defect == "next_scales" else e].clone()
        if defect == "scale_2pct":
            s2 = s2 * 1.02
        if defect == "no_q_h":
            ye = (he.double() @ _deq_w(ck["w2"][0][e:e + 1], s2[None], 0)).to(dt).float()
        else:
            ch, sh = _quantize(he)
            ye = _mm(ch, sh, ck["w2"][0][e], s2, dt, ks).float()
        yp[p] = wf[p][:, None] * ye
    return h, yp


def assert_block_equals_chain(block, chain, ck, ids, w, what):
    """The block against _layer_chain.  The two differ only where the exp of T(silu(g)) flipped an element of h
    (test_gate_up_within_one_ulp_of_layer_kernels), and then only through Q(h) of the groups that hold such an element:
      * every pair whose h row equals the chain's has a bit-identical ypair row, and every token whose pairs all do has
        a bit-identical output;
      * the other pairs are within ulp(yp) + B_g summed over their groups that hold a flipped element (B_g of the module
        docstring, an upper bound on requantising one group), with the chain's own h.
    At least half of the pairs must be bit-identical, so the exact part of the check always bites."""
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
    for r in (~same_sorted).nonzero().squeeze(1).tolist():
        p = int(pl[r])
        e = int(flat[p])
        W2 = _deq_w(*ck["w2"], e).abs().float().contiguous()        # [I, H]
        hh = h_c[r].abs().float().view(-1, 128)                      # [groups, 128]
        flipped = (h[r] != h_c[r]).view(-1, 128).any(1)
        a = (hh + 2.0 ** -14 * hh.amax(1, keepdim=True))[flipped]    # the groups that hold a flipped element
        B = (9 / 64) * (a.reshape(1, -1) @ W2.reshape(-1, 128, H)[flipped].reshape(-1, H)).squeeze(0)
        ye_c = yp_c[p] / wf[p] if float(wf[p]) != 0 else yp_c[p]
        tol = wf[p].abs() * (B + 2 * _ulp(ye_c, dt)) + 1e-30
        err = (yp[p] - yp_c[p]).abs()
        _record(what + " flipped-h pairs", 0.0, float((err / tol).max()))
        assert (err <= tol).all(), (what, "pair", p, float((err / tol).max()))
    return n_same


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", ["qwen3_30b_a3b", "deepseek_v3_ep8", "edge_tail_top2"])
def test_block_equals_layer_kernel_chain(name, dt):
    """The tight end-to-end check: the grouped block against transformers' per-expert FP8Linear loop built from the
    layer kernels at the same split-K (assert_block_equals_chain), at ks = 1 and 2 over T = 1, 17 and 300 with softmax and
    skewed routing.  MoEExperts' own output equals the raw-ABI block at the heuristic split bit for bit.  Negative
    controls: down_proj on the unquantised h, w2 scales 2 % off and the next expert's w2 scales all fail."""
    ck, blk, _ = _stack(name)
    E, K, _, top_k = STACKS[name]
    for T in (1, 17, 300):
        x = _x(T, K, dt, seed=7 * T)
        for routing, (ids, w) in (("softmax", _route(T, E, top_k, seed=T)), ("skewed", _skewed(T, E, top_k, seed=T))):
            what = f"fp8 moe chain {name} {TNAME[dt]} T={T} {routing}"
            assert torch.equal(blk(x, ids, w), _block_abi(x, ids, w, ck, 0)[3]), what
            for ks in (1, 2):
                block = _block_abi(x, ids, w, ck, ks)
                assert_block_equals_chain(block, _layer_chain(x, ids, w, ck, ks), ck, ids, w, f"{what} ks={ks}")
    T = 64
    x = _x(T, K, dt, seed=64)
    ids, w = _route(T, E, top_k, seed=64)
    block = _block_abi(x, ids, w, ck, 1)
    for defect in ("no_q_h", "scale_2pct", "next_scales"):
        with pytest.raises(AssertionError):
            assert_block_equals_chain(block, _layer_chain(x, ids, w, ck, 1, defect), ck, ids, w, f"control {defect}")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", list(STACKS))
def test_block_against_float64_oracle(name, dt):
    """Softmax routing at T = 1 .. 2048 on every stack, then skewed, sparse (mostly empty experts), an expert twice in one
    token, and top_k 1 / 3 routings.  The grouped path is also compared with the loop over the same modules at a few T."""
    ck, blk, loop = _stack(name)
    E, K, _, top_k = STACKS[name]
    for T in (1, 2, 8, 17, 64, 300, 2048):
        x = _x(T, K, dt, seed=T)
        ids, w = _route(T, E, top_k, seed=1000 + T)
        ref = fp8_moe_oracle(x, ids, w, ck)
        y = blk(x, ids, w)
        assert_fp8_moe_close(y, ref, f"fp8 moe {name} {TNAME[dt]} T={T}")
        if T in (1, 17, 300):
            assert_fp8_moe_close(loop(x, ids, w), ref, f"fp8 moe {name} {TNAME[dt]} T={T} loop")
        if T == 300:
            assert torch.equal(blk(x, ids, w), y)
    T = 65
    x = _x(T, K, dt, seed=T)
    routings = {"skewed": _skewed(T, E, top_k, seed=T)}
    ids, w = _route(T, E, top_k, seed=T)
    routings["sparse"] = (torch.where(ids % 4 == 0, ids, torch.full_like(ids, E - 1)), w)
    if top_k > 1:
        dup = ids.clone()
        dup[:, 1] = dup[:, 0]
        routings["duplicate"] = (dup, w)
    for k2 in (1, 3):
        routings[f"top{k2}"] = _route(T, E, k2, seed=T + k2)
    for what, (ids, w) in routings.items():
        assert_fp8_moe_close(blk(x, ids, w), fp8_moe_oracle(x, ids, w, ck), f"fp8 moe {name} {TNAME[dt]} {what}")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_graph_replay_equals_eager(dt):
    """The six launches captured in a CUDA graph read the routing from the device: after new ids / weights are copied in,
    a replay equals an eager run bit for bit and matches the oracle."""
    name = "qwen3_30b_a3b"
    ck, blk, _ = _stack(name)
    E, K, _, top_k = STACKS[name]
    T = 65
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
        assert torch.equal(yg, blk(x, ids2, w2)), what
        assert_fp8_moe_close(yg, fp8_moe_oracle(x, ids2, w2, ck), f"fp8 moe graph replay {TNAME[dt]} {what}")
    del gr


@pytest.mark.gpu
def test_large_prefill_splits_the_grid():
    """E = 256, top_k = 8, T = 8192: 65536 rows in 128-row blocks give 256 * 512 (expert, token block) pairs, so both
    grouped launches are issued over several ranges of gridDim.z, with populated blocks past the first."""
    from gptqmodel_b200 import moe

    E, K, I, top_k, T = 256, 256, 128, 8, 8192
    ck = {"w1": _role(E, I, K, 11), "w3": _role(E, I, K, 12), "w2": _role(E, K, I, 13)}
    blk = moe.MoEExperts(*[_modules(*ck[r]) for r in ("w1", "w3", "w2")], grouped=True)
    ids, w = _route(T, E, top_k, seed=5)
    counts = torch.bincount(ids.reshape(-1).cpu(), minlength=E)
    assert int(counts[E // 2:].sum()) > 0 and (E - 1) * 512 >= 65535
    for dt in DTYPES:
        x = _x(T, K, dt, seed=T)
        assert_fp8_moe_close(blk(x, ids, w), fp8_moe_oracle(x, ids, w, ck), f"fp8 moe large prefill {TNAME[dt]}")


@pytest.mark.gpu
def test_negative_controls():
    """Stacks that do not qualify take the loop (grouped=None) or are refused (grouped=True): bias, an adapter, a mixed
    GPTQ / FP8 stack.  And the tolerance bites: the routing weights
    of slots 0 and 1 exchanged fail the comparison the tests above pass."""
    from gptqmodel_b200 import B200BlockFp8Linear, B200QuantLinear, Lora, moe
    from helpers import random_layer

    E, K, I = 4, 256, 256
    ck = {"w1": _role(E, I, K, 21), "w3": _role(E, I, K, 22), "w2": _role(E, K, I, 23)}
    mods = lambda: [_modules(*ck[r]) for r in ("w1", "w3", "w2")]  # noqa: E731
    good = moe.MoEExperts(*mods())
    assert good._stack is not None and "fp8blk" in good._stack
    biased = mods()
    biased[2][1] = B200BlockFp8Linear.from_checkpoint_tensors(ck["w2"][0][1], ck["w2"][1][1],
                                                              bias=torch.zeros(K, dtype=torch.float16), device=DEV)
    gen = torch.Generator().manual_seed(0)
    lora = Lora(lora_A=(torch.randn(K, 8, generator=gen) * 0.05).half(), lora_B=(torch.randn(8, I, generator=gen) * 0.05).half())
    adapted = mods()
    adapted[0][0] = B200BlockFp8Linear.from_checkpoint_tensors(ck["w1"][0][0], ck["w1"][1][0], device=DEV, adapter=lora)
    L = random_layer(K, I, group_size=128, sym=True, seed=1, device=DEV)
    mixed = mods()
    mixed[0][2] = B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, 128,
                                                          sym=True)
    for what, sets in (("bias", biased), ("adapter", adapted), ("mixed", mixed)):
        assert moe.MoEExperts(*sets, fuse=False)._stack is None, what
        with pytest.raises(ValueError, match="B200BlockFp8Linear"):
            moe.MoEExperts(*sets, grouped=True)
    T = 16
    x = _x(T, K, torch.float16, seed=16)
    ids, w = _route(T, E, 2, seed=16)
    y = good(x, ids, w)
    assert_fp8_moe_close(y, fp8_moe_oracle(x, ids, w, ck), "fp8 moe control: correct oracle")
    with pytest.raises(AssertionError, match="outside"):
        assert_fp8_moe_close(y, fp8_moe_oracle(x, ids, w[:, [1, 0]], ck), "fp8 moe control: slot weights swapped")
    for bad_x, bad_ids in ((x[:, :128], ids), (x[:8], ids), (x, ids[:8])):  # shapes that do not fit the block
        with pytest.raises(ValueError, match="does not fit"):
            good(bad_x.contiguous(), bad_ids, w[:bad_ids.shape[0]])
    # the loop over the biased experts still runs (and matches its own per-expert modules)
    assert moe.MoEExperts(*biased)(x, ids, w).shape == (T, K)


@pytest.mark.gpu
def test_qwen3_moe_checkpoint_through_loader(tmp_path):
    """A tiny safetensors checkpoint with Qwen3-MoE module names, loaded by load_block_fp8_linears, runs MoEExperts on
    the grouped path and matches the oracle."""
    from safetensors.torch import save_file

    from gptqmodel_b200 import moe
    from gptqmodel_b200.loader import load_block_fp8_linears

    E, K, I = 4, 256, 384
    ck = {"w1": _role(E, I, K, 31), "w3": _role(E, I, K, 32), "w2": _role(E, K, I, 33)}
    proj = {"w1": "gate_proj", "w3": "up_proj", "w2": "down_proj"}
    tensors = {}
    for r, (w, s) in ck.items():
        for e in range(E):
            pre = f"model.layers.0.mlp.experts.{e}.{proj[r]}"
            tensors[pre + ".weight"] = w[e].cpu().contiguous()
            tensors[pre + ".weight_scale_inv"] = s[e].cpu().contiguous()
    with open(os.path.join(tmp_path, "config.json"), "w") as f:
        json.dump({"model_type": "qwen3_moe", "quantization_config": {
            "quant_method": "fp8", "fmt": "e4m3", "activation_scheme": "dynamic", "weight_block_size": [128, 128]}}, f)
    save_file(tensors, os.path.join(tmp_path, "model.safetensors"))
    mods = load_block_fp8_linears(str(tmp_path), device=DEV)
    get = lambda r: [mods[f"model.layers.0.mlp.experts.{e}.{proj[r]}"] for e in range(E)]  # noqa: E731
    blk = moe.MoEExperts(get("w1"), get("w3"), get("w2"), grouped=True)
    for dt in DTYPES:
        x = _x(9, K, dt, seed=9)
        ids, w = _route(9, E, 2, seed=9)
        assert_fp8_moe_close(blk(x, ids, w), fp8_moe_oracle(x, ids, w, ck), f"fp8 moe checkpoint {TNAME[dt]}")


class _Fp8Dense(torch.nn.Module):
    """Stand-in block-FP8 expert: quantises its input like FP8Linear (fo.quantize), float64 product, output in T."""

    def __init__(self, w, s):
        super().__init__()
        self.w, self.s = w, s

    def forward(self, x):
        c, sx = fo.quantize(x.float().numpy())
        W = _deq_w(self.w[None], self.s[None], 0)
        return (_deq_codes(c, sx, "cpu") @ W).to(x.dtype)


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_oracle_matches_module_loop_on_cpu(dt):
    """CPU: fp8_moe_oracle's routing and rounding points against MoEExperts(grouped=False) over stand-in experts that
    quantise their input like transformers' FP8Linear.  Only the fp32 order of the final sum differs.  Routing covers
    empty experts, an expert twice in one token, unnormalised weights and top_k 1 / 3; exchanged slot weights fail."""
    from gptqmodel_b200 import moe

    gen = torch.Generator().manual_seed(7)
    E, K, I = 5, 256, 384

    def role(N, Kr):
        w = (torch.randn(E, N, Kr, generator=gen) * 60).clamp(-448, 448).to(torch.float8_e4m3fn)
        return w, (torch.rand(E, (N + 127) // 128, Kr // 128, generator=gen) + 0.5) / (60 * Kr ** 0.5)

    ck = {"w1": role(I, K), "w3": role(I, K), "w2": role(K, I)}
    experts = [[_Fp8Dense(ck[r][0][e], ck[r][1][e]) for e in range(E)] for r in ("w1", "w3", "w2")]
    blk = moe.MoEExperts(*experts, grouped=False)
    for T, top_k, routing in ((1, 1, "softmax"), (40, 3, "softmax"), (9, 3, "duplicate"), (40, 3, "sparse")):
        x = torch.randn(T, K, generator=gen).to(dt)
        ids, w = moe.route_topk(torch.randn(T, E, generator=gen), top_k)
        if routing == "duplicate":
            ids[:, 1] = ids[:, 0]
        elif routing == "sparse":
            ids[ids == 2] = 4
            w = torch.rand(T, top_k, generator=gen) * 1.5
            w[0, 0], w[1, 1] = 0.0, 1.75
        got = blk(x, ids, w)
        ref, slack = fp8_moe_oracle(x, ids, w, ck)
        what = f"cpu fp8 T={T} top_k={top_k} {routing}"
        assert got.dtype == dt and got.shape == (T, K)
        assert_close_rel(got, ref, REL[dt], what, slack=slack)
        if routing == "softmax" and top_k > 1:
            with pytest.raises(AssertionError, match="outside"):
                assert_close_rel(got, fp8_moe_oracle(x, ids, w[:, [1, 0, 2]], ck)[0], REL[dt], what + " swapped")
