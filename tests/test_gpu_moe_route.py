"""moe_route_kernel (b2q_moe_route, gptqmodel_b200/csrc/b2q_moe.cu) against transformers' fixtures and the float64 oracle
of oracle/moe_route_oracle.py.

Selection.  The softmax mode selects on the logits themselves, converted to fp32 exactly, so its choice and slot order
are exact: ids must equal the oracle's, ties included.  The grouped sigmoid mode selects on c = fp32(s) + bias with
s = 1 / (1 + expf(-l)).  With u = 2^-24: expf is within 2 ulp (<= 4u relative), which moves s by at most
4u * e / (1 + e) <= 4u relative; 1 + e and the division round once each (2u): |s - s64| <= 6u * s <= 3.6e-7.  The add rounds
once more, <= u |c|.  With |c| <= 2 (the sweep's biases stay below 1): TOL_C = 1e-6 for c and TOL_G = 3e-6 for a group
score (two c and one rounding).  On every row the chosen set must be a top-k within these: every selected c >= every c
left unselected in the kept groups - TOL_C, and every selected expert's group scores >= the topk_group-th group score -
TOL_G.  Rows whose oracle gaps at the group boundary and the k-th place both exceed the tolerance must have exactly the
oracle's ids as a set; slots must descend within TOL_C everywhere.

Weights.  Compared with the oracle's weights of the ids the kernel chose (route_weights), |w - w64| <= eps |w64|, from the
kernel's arithmetic (u = 2^-24, one rounding <= u relative, expf <= 2 ulp = 4u):
  softmax: p_j = expf(fl(l_j - m)) / S.  fl(l - m) = (l - m)(1 + d) changes exp by |l - m| u relative: at most D u with
    D = max - min of the row's logits, in the numerator and in every term of S.  expf adds 4u to each.  S sums NPER terms
    per lane then 5 shuffle levels: (NPER + 4) u.  The division: u.  eps_p = (2 D + 8 + NPER + 5) u.
  sigmoid: eps_s = 6u (above).
  renormalising: the k selected weights summed in slot order ((k - 1) u, plus the error of the terms) and one division:
    eps = 2 eps_p + (k + 1) u.  The scale multiply: u.
For the sweep's logits (|l| <~ 10) that is about 1e-5 relative at most.
"""
import pytest
import torch

from helpers import random_layer
from oracle import moe_route_oracle as ro

DEV = "cuda"
U = 2.0 ** -24
TOL_C, TOL_G = 1e-6, 3e-6
DTYPES = (torch.float32, torch.bfloat16, torch.float16)
TNAME = {torch.float32: "fp32", torch.bfloat16: "bf16", torch.float16: "fp16"}
GROUPS = ((1, 1), (4, 2), (8, 4), (16, 4))


def _moe():
    from gptqmodel_b200 import moe

    return moe


def weight_bound(logits, top_k, scoring, renormalize):
    """Per-row relative bound eps [T, 1] of the module docstring."""
    if scoring == "softmax":
        l = logits.double()
        D = (l.amax(-1) - l.amin(-1))[:, None]
        nper = (logits.shape[1] + 31) // 32
        eps = (2 * D + 8 + nper + 5) * U
    else:
        eps = torch.full((logits.shape[0], 1), 6 * U, dtype=torch.float64, device=logits.device)
    if renormalize:
        eps = 2 * eps + (top_k + 1) * U
    return eps + U


def assert_weights(w, logits, ids, top_k, scoring, renormalize, scale, what):
    ref = ro.route_weights(logits, ids, scoring, renormalize, scale)
    eps = weight_bound(logits, top_k, scoring, renormalize)
    err = (w.double() - ref).abs()
    bad = err > eps * ref.abs()
    assert not bad.any(), (what, int(bad.sum()), float((err / (eps * ref.abs())).max()))


def _logits(T, E, dt, seed, scale=2.0):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(T, E, device=DEV, generator=gen) * scale).to(dt)


def _bias(E, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(E, device=DEV, generator=gen) * 0.1


def _kth(v, k):
    """k-th largest per row ([T, 1]); -inf when k is 0."""
    return v.sort(dim=-1, descending=True).values[:, k - 1:k]


def check_softmax(logits, top_k, renormalize, what):
    ids, w = _moe().route_softmax_topk(logits, top_k, renormalize=renormalize)
    assert ids.dtype == torch.int32 and w.dtype == torch.float32 and ids.shape == w.shape == (logits.shape[0], top_k)
    o_ids = ro.route_softmax(logits, top_k, renormalize)[0]
    assert torch.equal(ids.long(), o_ids), what
    assert_weights(w, logits, ids, top_k, "softmax", renormalize, 1.0, what)
    return ids, w


def check_grouped(logits, bias, top_k, n_group, topk_group, renormalize, scale, what):
    T, E = logits.shape
    ids, w = _moe().route_grouped_sigmoid(logits, bias, top_k, n_group, topk_group, renormalize=renormalize, scale=scale)
    assert ids.dtype == torch.int32 and w.dtype == torch.float32 and ids.shape == w.shape == (T, top_k)
    li = ids.long()
    assert ((li >= 0) & (li < E)).all(), what
    assert (li.sort(-1).values.diff(dim=-1) > 0).all(), f"{what}: an expert twice in one row"
    o_ids, _, masked, _ = ro.route_grouped_sigmoid(logits, bias, top_k, n_group, topk_group, renormalize, scale)
    _, c = ro.sigmoid_scores(logits, bias)
    gs = E // n_group
    gsc = ro.group_scores(c, n_group)
    # group stage: every selected expert's group within TOL_G of the kept ones
    kth_g = _kth(gsc, topk_group)
    assert (gsc.gather(1, li // gs) >= kth_g - TOL_G).all(), f"{what}: expert of a dropped group"
    # expert stage, on rows where the kept groups are unambiguous
    if topk_group < n_group:
        g_gap = (kth_g - _kth(gsc, topk_group + 1)).squeeze(1)
    else:
        g_gap = torch.full((T,), float("inf"), dtype=torch.float64, device=DEV)
    clear_g = g_gap > TOL_G
    sel_c = c.gather(1, li)
    rest = masked.scatter(1, li, float("-inf"))
    ok = sel_c.amin(-1) >= rest.amax(-1) - TOL_C
    assert (ok | ~clear_g).all(), f"{what}: not a top-{top_k} of the kept groups on {int((~ok & clear_g).sum())} rows"
    assert (sel_c[:, :-1] >= sel_c[:, 1:] - TOL_C).all(), f"{what}: slots not in descending order"
    k_gap = (_kth(masked, top_k) - (_kth(masked, top_k + 1) if top_k < E else -float("inf"))).squeeze(1)
    clear = clear_g & (k_gap > TOL_C)
    same = (li.sort(-1).values == o_ids.sort(-1).values).all(-1)
    assert (same | ~clear).all(), f"{what}: ids differ from the oracle's on {int((~same & clear).sum())} clear rows"
    assert_weights(w, logits, ids, top_k, "sigmoid", renormalize, scale, what)
    return ids, w


# ---- 1. golden cases from transformers -----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_golden_cases():
    import os

    import numpy as np

    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "moe_route_cases.npz"))
    for name in z["names"]:
        c = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(f"{name}/")}
        logits = torch.from_numpy(c["logits"]).to(DEV)
        k, norm, scale = int(c["top_k"]), bool(c["renormalize"]), float(c["scale"])
        if int(c["scoring"]) == 0:
            ids, w = _moe().route_softmax_topk(logits, k, renormalize=norm, scale=scale)
            scoring = "softmax"
        else:
            ids, w = _moe().route_grouped_sigmoid(logits, torch.from_numpy(c["bias"]).to(DEV), k, int(c["n_group"]),
                                                  int(c["topk_group"]), renormalize=norm, scale=scale)
            scoring = "sigmoid"
        order = ids.long().argsort(-1)
        assert np.array_equal(ids.long().gather(1, order).cpu().numpy(), c["ids"]), name
        # transformers' fp32 weights, in the kernel's bound plus their own fp32 rounding (the oracle reproduces them to
        # 1e-6, tests/test_moe_route_host.py)
        ref = torch.from_numpy(c["weights"]).to(DEV).double()
        eps = weight_bound(logits, k, scoring, norm) + 1e-6
        err = (w.gather(1, order).double() - ref).abs()
        assert (err <= eps * ref.abs()).all(), (str(name), float((err / (eps * ref.abs())).max()))
        assert_weights(w, logits, ids, k, scoring, norm, scale, str(name))


# ---- 2. sweep against the float64 oracle ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=[TNAME[d] for d in DTYPES])
@pytest.mark.parametrize("E", [8, 16, 60, 64, 128, 160, 256])
def test_sweep_against_oracle(E, dt):
    """top_k 1 / 2 / 4 / 6 / 8 / 16 (<= E), T 1 / 2 / 7 / 33 / 1000 / 8193; softmax with and without renormalising, grouped
    sigmoid at every (n_group, topk_group) of GROUPS that divides E and holds top_k, with and without renormalising."""
    bias = _bias(E, seed=E)
    for top_k in (k for k in (1, 2, 4, 6, 8, 16) if k <= E):
        for T in (1, 2, 7, 33, 1000, 8193):
            seed = 100 * E + 10 * top_k + T
            logits = _logits(T, E, dt, seed)
            what = f"E={E} k={top_k} T={T} {TNAME[dt]}"
            check_softmax(logits, top_k, T % 2 == 1, f"softmax {what}")
            for n_group, topk_group in GROUPS:
                if E % n_group or E // n_group < 2 or top_k > topk_group * (E // n_group):
                    continue
                check_grouped(logits, bias, top_k, n_group, topk_group, T != 2, 2.5 if n_group == 8 else 1.0,
                              f"grouped {n_group}/{topk_group} {what}")


@pytest.mark.gpu
def test_weight_check_bites():
    """The weight bound is tight enough to catch a 3e-5 relative error, a weight of the wrong kind (p not renormalised)
    and the wrong scale."""
    logits = _logits(33, 64, torch.float32, seed=9)
    ids, w = _moe().route_softmax_topk(logits, 8)
    assert_weights(w, logits, ids, 8, "softmax", True, 1.0, "control")
    for bad, norm, scale in ((w * (1 + 3e-5), True, 1.0), (w, False, 1.0), (w, True, 1.0 + 1e-4)):
        with pytest.raises(AssertionError):
            assert_weights(bad, logits, ids, 8, "softmax", norm, scale, "control")


# ---- 3. exact ties ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=[TNAME[d] for d in DTYPES])
def test_exact_ties(dt):
    moe = _moe()
    for E in (8, 60, 256):
        for k in (1, 2, 8):
            ids, w = moe.route_softmax_topk(torch.full((3, E), 0.25, device=DEV, dtype=dt), k)
            assert ids.tolist() == [list(range(k))] * 3, (E, k)
            assert torch.allclose(w, torch.full_like(w, 1.0 / k), rtol=1e-6, atol=0)
    ids, _ = moe.route_grouped_sigmoid(torch.zeros(2, 256, device=DEV, dtype=dt), torch.zeros(256, device=DEV), 8, 8, 4)
    assert ids.tolist() == [list(range(8))] * 2
    # equal values straddling the k-th place resolve to the lower indices
    l = torch.zeros(1, 64, device=DEV)
    l[0, [40, 50]] = 3.0
    l[0, [7, 30, 60]] = 2.0
    ids, _ = moe.route_softmax_topk(l.to(dt), 4)
    assert ids.tolist() == [[40, 50, 7, 30]]
    bias = torch.zeros(64, device=DEV)
    bias[[40, 50]] = 0.5
    bias[[7, 30, 60]] = 0.25
    ids, _ = moe.route_grouped_sigmoid(torch.zeros(1, 64, device=DEV, dtype=dt), bias, 4, 1, 1)
    assert ids.tolist() == [[40, 50, 7, 30]]
    # tied group scores resolve to the lower group: groups of 4; groups 1, 2 and 3 tie above group 0, topk_group 2
    bias = torch.zeros(16, device=DEV)
    bias[[4, 5, 8, 9, 12, 13]] = 0.125
    ids, _ = moe.route_grouped_sigmoid(torch.zeros(1, 16, device=DEV, dtype=dt), bias, 4, 4, 2)
    assert ids.tolist() == [[4, 5, 8, 9]]
    bias[[13]] = 0.0
    bias[[14, 15]] = 0.0625  # group 3 now below groups 1 and 2 but above 0: the choice does not change
    assert moe.route_grouped_sigmoid(torch.zeros(1, 16, device=DEV, dtype=dt), bias, 4, 4, 2)[0].tolist() == [[4, 5, 8, 9]]


# ---- 4. masking of dropped groups ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_dropped_groups_never_chosen():
    """The kept group holds only negative biased scores.  Experts outside it count as -inf, so the kernel stays inside it;
    transformers' 0.0 fill would pick from the dropped group here."""
    moe = _moe()
    bias = torch.tensor([-0.9, -0.8, -2.0, -2.0, -2.0, -2.0, -2.0, -2.0], device=DEV)
    ids, w = moe.route_grouped_sigmoid(torch.zeros(1, 8, device=DEV), bias, 2, 2, 1)
    assert ids.tolist() == [[1, 0]]
    assert torch.allclose(w, torch.full_like(w, 0.5), rtol=1e-6, atol=0)
    # the DeepSeek-V3 shape: every biased score negative, logits random; all choices in the kept groups
    T, E = 257, 256
    logits = _logits(T, E, torch.float32, seed=4)
    bias = -1.5 - torch.rand(E, device=DEV)
    ids, _ = moe.route_grouped_sigmoid(logits, bias, 8, 8, 4, scale=2.5)
    _, _, _, kept = ro.route_grouped_sigmoid(logits, bias, 8, 8, 4)
    assert kept.gather(1, ids.long() // 32).all()
    check_grouped(logits, bias, 8, 8, 4, True, 2.5, "negative biased scores")


# ---- 5. end to end through MoEExperts --------------------------------------------------------------------------------------
def _gptq_block():
    from gptqmodel_b200 import B200QuantLinear

    E, K, I, gs = 64, 1024, 512, 128
    layers = [(random_layer(K, I, group_size=gs, seed=3 * e, device=DEV),
               random_layer(K, I, group_size=gs, seed=3 * e + 1, device=DEV),
               random_layer(I, K, group_size=gs, seed=3 * e + 2, device=DEV)) for e in range(E)]
    mk = lambda L: B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, gs,  # noqa: E731
                                                           sym=True)
    blk = _moe().MoEExperts([mk(L[0]) for L in layers], [mk(L[1]) for L in layers], [mk(L[2]) for L in layers])
    assert blk._stack is not None
    return layers, blk, E, K


@pytest.mark.gpu
@pytest.mark.parametrize("dt", (torch.float16, torch.bfloat16), ids=["fp16", "bf16"])
def test_end_to_end_gptq(dt):
    """Kernel routing into the grouped GPTQ stack equals the same experts routed by the oracle's ids and weights: one token
    on the decode path (top_k 2 / 4 / 8) and 64 tokens on the grouped path, softmax and grouped sigmoid."""
    from test_gpu_moe import assert_moe_close, moe_oracle, stack_weights

    layers, blk, E, K = _gptq_block()
    moe = _moe()
    bias = _bias(E, seed=5)
    for T in (1, 64):
        gen = torch.Generator(device=DEV).manual_seed(T)
        x = (torch.randn(T, K, device=DEV, generator=gen) * 0.5).to(dt)
        for top_k in (2, 4, 8):
            logits = _logits(T, E, dt, seed=T + top_k)
            form = "exact" if T == 1 and blk._decode_ok(top_k) else "rounded"
            for mode in ("softmax", "sigmoid"):
                if mode == "softmax":
                    ids, w = moe.route_softmax_topk(logits, top_k)
                    o_ids, o_w, _ = ro.route_softmax(logits, top_k)
                else:
                    ids, w = moe.route_grouped_sigmoid(logits, bias, top_k, 8, 4, scale=2.5)
                    o_ids, o_w, _, _ = ro.route_grouped_sigmoid(logits, bias, top_k, 8, 4, scale=2.5)
                assert torch.equal(ids.long(), o_ids), (mode, T, top_k)
                y = blk(x, ids, w)
                assert_moe_close(y, moe_oracle(x, o_ids, o_w.float(), stack_weights(layers, dt, form)),
                                 f"e2e gptq {mode} T={T} top_k={top_k} {dt}")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", (torch.float16, torch.bfloat16), ids=["fp16", "bf16"])
def test_end_to_end_block_fp8_grouped_sigmoid(dt):
    """A block-FP8 stack of 64 experts routed by grouped sigmoid (8 groups, 4 kept, scale 2.5) against the block-FP8
    oracle of tests/test_gpu_moe_fp8_block.py on the oracle's routing."""
    from test_gpu_moe_fp8_block import _modules, _role, assert_fp8_moe_close, fp8_moe_oracle

    E, K, I, top_k = 64, 1024, 512, 8
    ck = {"w1": _role(E, I, K, 1), "w3": _role(E, I, K, 2), "w2": _role(E, K, I, 3)}
    moe = _moe()
    blk = moe.MoEExperts(*[_modules(*ck[r]) for r in ("w1", "w3", "w2")])
    assert "fp8blk" in blk._stack
    bias = _bias(E, seed=6)
    for T in (1, 64):
        gen = torch.Generator(device=DEV).manual_seed(T)
        x = (torch.randn(T, K, device=DEV, generator=gen) * 0.5).to(dt)
        logits = _logits(T, E, torch.float32, seed=60 + T)
        ids, w = moe.route_grouped_sigmoid(logits, bias, top_k, 8, 4, scale=2.5)
        o_ids, o_w, _, _ = ro.route_grouped_sigmoid(logits, bias, top_k, 8, 4, scale=2.5)
        assert torch.equal(ids.long(), o_ids)
        assert_fp8_moe_close(blk(x, ids, w), fp8_moe_oracle(x, o_ids, o_w.float(), ck), f"e2e fp8blk T={T} {dt}")


# ---- 6. CUDA graph and host synchronisation --------------------------------------------------------------------------------
@pytest.mark.gpu
def test_graph_replay_and_no_host_sync():
    """Router + MoEExperts captured in one CUDA graph: replays with new logits equal eager runs bit for bit.  The router
    itself never synchronises with the host."""
    layers, blk, E, K = _gptq_block()
    moe = _moe()
    dt = torch.float16
    bias = _bias(E, seed=7)
    for T, top_k in ((1, 8), (64, 4)):
        x = (torch.randn(T, K, device=DEV) * 0.5).to(dt)
        lg = _logits(T, E, dt, seed=70 + T)

        def block():
            ids, w = moe.route_grouped_sigmoid(lg, bias, top_k, 8, 4, scale=2.5)
            return blk(x, ids, w), ids, w

        s_ = torch.cuda.Stream()
        s_.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s_):
            block()
        torch.cuda.current_stream().wait_stream(s_)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            yg, idg, wg = block()
        for seed in (1, 2):
            lg.copy_(_logits(T, E, dt, seed=700 + seed + T))
            gr.replay()
            torch.cuda.synchronize()
            ye, ide, we = block()
            assert torch.equal(idg, ide) and torch.equal(wg, we) and torch.equal(yg, ye), (T, seed)
        del gr
    lg = _logits(33, 256, torch.bfloat16, seed=8)
    b = _bias(256, seed=8)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        moe.route_grouped_sigmoid(lg, b, 8, 8, 4, scale=2.5)
        moe.route_softmax_topk(lg, 8)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
