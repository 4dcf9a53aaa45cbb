"""The MoE expert block (gptqmodel_b200/moe.py) against a float64 oracle that rounds where the kernels round.

Paths, all on stacks of random 4-bit experts with the per-rank shapes of real models:
  * grouped: b2q_moe_align -> b2q_moe_gather -> midm_kernel MODE 1 (gate|up, SiLU-mul epilogue) -> MODE 2 (down, routing
    weight, scatter) -> b2q_moe_combine (b2q_moe.cu, b2q_midm.cu);
  * loop (grouped=False): every expert's w1 / w3 / w2 module on its block of rows, through b2q_mm;
  * one token: b2q_moe_decode_gate_up / _act / _down for top_k 2 / 4 / 8, the grouped kernels for any other top_k.

Oracle.  T(.) rounds to the run dtype.  For every routed pair (token t, slot j, expert e = ids[t, j]):
    g = T(x_t W1_e),  u = T(x_t W3_e),  a = T(silu(g)),  h = T(a * u),  yp_j = T(h W2_e)
    y_t = T(sum_j fp32(w_j * yp_j))          (fp32 products, summed in j order)
These are the rounding points of the reference's per-expert module loop, where every module returns a 16-bit tensor.  They
are also the kernels' rounding points: MODE 1's epilogue and moe_decode_act_kernel, MODE 2's epilogue and the decode down
reduction, and moe_combine_kernel.  The oracle takes the dequantised weights in one of two forms:
  * ROUNDED, W = T((q - z) * s): what the tensor-core tiers feed the MMA (grouped path; loop-path experts on the
    small-batch or prefill tier);
  * EXACT, (q - z) * s in float64: the decode tier applies the scale once per group to an integer dot product (decode
    path; loop-path experts with at most 8 rows, see helpers.scale_once_tier).
bf16 runs use the fp16 checkpoint scales converted to bf16, which is what MoEExperts._scales and the modules hand the kernels.
The oracle runs on the GPU in float64 and dequantises only the experts that are routed to.

Tolerance, assert_close_rel: |out - ref| <= rel * |ref| + rel * rms(ref).  With the rounding points matched, kernel and
oracle differ only in how the fp32 dot products are accumulated (order, fused multiply-adds: relative ~2^-24 * sqrt(K)).
Such a difference can push a value across a rounding boundary of the run dtype, so any rounded quantity may come out one
ulp away from the oracle's.  A flip in g, u, a or h moves one of I terms of h W2 by one ulp of h: about 2^-p / sqrt(I) of
yp, far below one ulp of yp.  The flips that reach the output are those of yp_j and of y itself, so
one output element is off by at most
    ulp(y) + sum_j |w_j| ulp(yp_j).
The first term is at most 2^(1-p) |y| (p = 11 for fp16, 8 for bf16): 9.8e-4 |y| in fp16, 7.8e-3 |y| in bf16.  It is
covered by rel = 2e-3 (fp16) and 1.6e-2 (bf16), which leave room for both terms when the slots do not cancel
(sum_j |w_j| |yp_j| ~ |y|).  The second term is passed as an explicit per-element slack computed from the oracle's own yp_j.
rel * rms(ref) alone cannot carry it: where two slots of size ~3 rms(y) cancel, one flip of the larger slot is as large
as 2e-3 * (|y| + rms(y)).  Without the slack, the Mixtral stack's loop path at T = 17 in fp16 has exactly that case
on an H100: 1 element of 69632 at err / tol = 1.00.  parity.json records the worst err / tol ratio of every test.
"""
import os

import pytest
import torch
import torch.nn.functional as F

import oracle
from helpers import assert_close_rel, random_layer, scale_once_tier

DEV = "cuda"
DTYPES = (torch.float16, torch.bfloat16)
REL = {torch.float16: 2e-3, torch.bfloat16: 1.6e-2}

# per-rank expert stacks of real models: experts E, hidden K, intermediate I, group size (-1: per channel), symmetric
STACKS = {
    "mixtral_8x7b_tp4": (8, 4096, 3584, 64, False),
    "qwen1.5_moe_a2.7b": (60, 2048, 1408, 128, True),
    "deepseek_v2_lite": (64, 2048, 1408, 128, False),
    "qwen3_30b_a3b": (128, 2048, 768, 128, True),
    "edge_g32": (4, 256, 512, 32, False),
    "edge_per_channel": (4, 256, 512, -1, True),
}
CASES = [("mixtral_8x7b_tp4", 2), ("qwen1.5_moe_a2.7b", 4), ("deepseek_v2_lite", 6), ("qwen3_30b_a3b", 8),
         ("edge_g32", 1), ("edge_g32", 2), ("edge_per_channel", 1), ("edge_per_channel", 2)]
CASE_IDS = [f"{s}-top{k}" for s, k in CASES]


# ------------------------------------------------------------------------------------------------------------------------
# oracle (device-agnostic: the CPU test below checks its routing algebra against the module's loop path)
# ------------------------------------------------------------------------------------------------------------------------
def _ulp(v, dt):
    """One unit in the last place of dt at the (dt-representable) values v, float32."""
    p, tiny = (11, 2.0 ** -24) if dt == torch.float16 else (8, 2.0 ** -133)
    e = torch.floor(torch.log2(v.to(torch.float64).abs().clamp(min=tiny)))
    return torch.exp2(e - (p - 1)).clamp(min=tiny).to(torch.float32)


def moe_oracle(x, ids, w, weights):
    """(y [T, K_out] in x.dtype, slack [T, K_out] float32).  weights(e, rows) -> float64 (W1 [K, I], W3 [K, I],
    W2 [I, K_out]) of expert e, which receives `rows` pairs.  slack = sum_j |w_j| ulp(yp_j): the one-ulp flips of the
    expert outputs (module docstring)."""
    dt = x.dtype
    T, top_k = ids.shape
    R = lambda v: v.to(dt).to(torch.float64)  # noqa: E731
    flat = ids.reshape(-1).to(x.device)
    xd = x.to(torch.float64)
    yp = None
    for e in torch.unique(flat).tolist():
        pairs = (flat == e).nonzero().squeeze(1)
        W1, W3, W2 = weights(e, pairs.numel())
        xe = xd.index_select(0, pairs // top_k)
        g, u = R(xe @ W1), R(xe @ W3)
        h = R(R(F.silu(g)) * u)
        if yp is None:
            yp = torch.zeros(T * top_k, W2.shape[1], dtype=torch.float64, device=x.device)
        yp[pairs] = R(h @ W2)
    yp = yp.to(torch.float32).view(T, top_k, -1)
    wf = w.to(device=x.device, dtype=torch.float32)
    acc = torch.zeros(T, yp.shape[-1], dtype=torch.float32, device=x.device)
    for j in range(top_k):
        acc = acc + wf[:, j:j + 1] * yp[:, j]
    slack = (wf.abs()[:, :, None] * _ulp(yp, dt)).sum(1)
    return acc.to(dt), slack


def _dequant(L, dt, exact):
    sc = L["scales"].to(dt)  # bf16 runs: the fp16 checkpoint scales converted, as the module converts them
    if exact:
        return oracle.dequantize_weight(L["qweight"], L["qzeros"], sc.to(torch.float64), L["g_idx"], 4)
    return oracle.dequantize_weight(L["qweight"], L["qzeros"], sc, L["g_idx"], 4).to(torch.float64)


def stack_weights(layers, dt, form):
    """form: "rounded" (tensor-core tiers), "exact" (decode tier) or "loop": per matrix, exact where b2q_mm serves the
    expert's row count on a tier that applies the scale once per group."""
    def get(e, rows):
        return tuple(_dequant(L, dt, form == "exact" or (form == "loop" and scale_once_tier(L, rows))) for L in layers[e])
    return get


def _loop_form(layers, ids):
    counts = torch.bincount(ids.reshape(-1).cpu(), minlength=len(layers))
    return "loop" if any(scale_once_tier(L, int(c)) for Ls, c in zip(layers, counts) if c > 0 for L in Ls) else "rounded"


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the oracle's routing algebra
# ------------------------------------------------------------------------------------------------------------------------
class _Dense(torch.nn.Module):
    """Stand-in expert matrix: float64 product, output rounded to the input dtype like a QuantLinear's."""

    def __init__(self, W):
        super().__init__()
        self.W = W

    def forward(self, x):
        return (x.to(torch.float64) @ self.W).to(x.dtype)


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_oracle_matches_module_loop_on_cpu(dt):
    """The per-expert loop of MoEExperts with dense float64 stand-ins rounds at the same points as moe_oracle; only the
    fp32 order of the final sum differs (expert order there, slot order here).  Routing covers empty experts, an expert
    twice in one token, unnormalised weights with a 0.0 and a weight > 1, and top_k 1 / 3."""
    from gptqmodel_b200 import moe

    gen = torch.Generator().manual_seed(7)
    E, K, I = 5, 48, 80
    Ws = [tuple(torch.randn(a, b, generator=gen, dtype=torch.float64) * 0.2 for a, b in ((K, I), (K, I), (I, K)))
          for _ in range(E)]
    blk = moe.MoEExperts([_Dense(w[0]) for w in Ws], [_Dense(w[1]) for w in Ws], [_Dense(w[2]) for w in Ws], grouped=False)
    weights = lambda e, rows: Ws[e]  # noqa: E731
    for T, top_k, routing in ((1, 1, "softmax"), (40, 3, "softmax"), (9, 3, "duplicate"), (40, 3, "sparse")):
        x = (torch.randn(T, K, generator=gen) * 0.5).to(dt)
        ids, w = moe.route_topk(torch.randn(T, E, generator=gen), top_k)
        if routing == "duplicate":
            ids[:, 1] = ids[:, 0]                       # the same expert in two slots of every token
        elif routing == "sparse":
            ids[ids == 2] = 4                           # expert 2 empty (and some tokens on expert 4 twice)
            w = torch.rand(T, top_k, generator=gen) * 1.5
            w[0, 0], w[1, 1] = 0.0, 1.75
        got = blk(x, ids, w)
        assert got.dtype == dt and got.shape == (T, K)
        what = f"cpu T={T} top_k={top_k} {routing}"
        assert_close_rel(got, moe_oracle(x, ids, w, weights)[0], 1e-3, what)
        if routing == "softmax" and top_k > 1:  # the check bites: slots 0 and 1 with their weights exchanged
            with pytest.raises(AssertionError, match="outside"):
                assert_close_rel(got, moe_oracle(x, ids, w[:, [1, 0, 2]], weights)[0], 1e-3, what + " swapped")


# ------------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------------
_BLOCKS = {}


@pytest.fixture(scope="module", autouse=True)
def _release_stacks():
    """The expert stacks (about 1 GB on the device) are shared by the tests of this module only."""
    yield
    _BLOCKS.clear()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _stack(name):
    """(layers, grouped block, loop block) of one expert stack, built once per module run."""
    if name not in _BLOCKS:
        from gptqmodel_b200 import B200QuantLinear, moe

        E, K, I, gs, sym = STACKS[name]
        layers = [(random_layer(K, I, group_size=gs, sym=sym, seed=3 * e, device=DEV),
                   random_layer(K, I, group_size=gs, sym=sym, seed=3 * e + 1, device=DEV),
                   random_layer(I, K, group_size=gs, sym=sym, seed=3 * e + 2, device=DEV)) for e in range(E)]
        mk = lambda L: B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4,  # noqa: E731
                                                               gs, sym=sym)
        blk = moe.MoEExperts([mk(Ls[0]) for Ls in layers], [mk(Ls[1]) for Ls in layers], [mk(Ls[2]) for Ls in layers])
        assert blk._stack is not None, name
        loop = moe.MoEExperts(list(blk.w1), list(blk.w3), list(blk.w2), grouped=False)
        assert loop._stack is None
        _BLOCKS[name] = (layers, blk, loop)
    return _BLOCKS[name]


def _x(T, K, dt, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(T, K, device=DEV, generator=gen) * 0.5).to(dt)


def _route(T, E, top_k, seed):
    from gptqmodel_b200 import moe

    return moe.route_topk(torch.randn(T, E, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed)), top_k)


def _grouped(blk, x, ids, w, decode_path=False, fuse_act=False):
    blk.decode_path, blk.fuse_act = decode_path, fuse_act
    try:
        return blk(x, ids, w)
    finally:
        blk.decode_path, blk.fuse_act = True, False


def assert_moe_close(out, oracle_out, what):
    """out against moe_oracle's (y, slack) at the tolerance of the module docstring."""
    ref, slack = oracle_out
    assert out.shape == ref.shape and out.dtype == ref.dtype, (what, out.shape, out.dtype)
    assert_close_rel(out, ref, REL[ref.dtype], what, slack=slack.cpu())


def _check(layers, blk, loop, x, ids, w, what, paths=("grouped", "loop")):
    """Grouped and / or loop path against the oracle; returns the grouped output."""
    ref = moe_oracle(x, ids, w, stack_weights(layers, x.dtype, "rounded"))
    y = None
    if "grouped" in paths:
        y = _grouped(blk, x, ids, w)
        assert_moe_close(y, ref, f"{what} grouped")
    if "loop" in paths:
        form = _loop_form(layers, ids)
        ref_loop = ref if form == "rounded" else moe_oracle(x, ids, w, stack_weights(layers, x.dtype, form))
        assert_moe_close(loop(x, ids, w), ref_loop, f"{what} loop")
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name,top_k", CASES, ids=CASE_IDS)
def test_moe_token_counts(name, top_k, dt):
    """Softmax top-k routing at token counts on both sides of the 16 / 32 / 64 / 128-row token blocks.  One token also
    runs the decode path (top_k 2 / 4 / 8 with a group size the decode tier takes), where the SiLU-mul fused into the down
    launch must give the bits of the separate launch, or else the grouped fallback."""
    layers, blk, loop = _stack(name)
    E, K = STACKS[name][:2]
    for T in (1, 2, 8, 16, 17, 64, 65, 129, 300):
        x = _x(T, K, dt, seed=T)
        ids, w = _route(T, E, top_k, seed=1000 + T)
        y = _check(layers, blk, loop, x, ids, w, f"{name} {dt} T={T}")
        if T == 1:
            y_dec = _grouped(blk, x, ids, w, decode_path=True)
            if blk._decode_ok(top_k):
                assert torch.equal(_grouped(blk, x, ids, w, decode_path=True, fuse_act=True), y_dec)
                assert_moe_close(y_dec, moe_oracle(x, ids, w, stack_weights(layers, dt, "exact")), f"{name} {dt} decode path")
            else:
                assert torch.equal(y_dec, y)


def _skewed(T, E, top_k, seed):
    """Every token on the same top_k experts (a fixed random set), in a random slot order per token."""
    gen = torch.Generator().manual_seed(seed)
    sel = torch.randperm(E, generator=gen)[:top_k]
    ids = sel[torch.argsort(torch.rand(T, top_k, generator=gen), dim=1)]
    w = torch.rand(T, top_k, generator=gen) + 0.1
    return ids.to(DEV), (w / w.sum(-1, keepdim=True)).to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name,top_k", CASES, ids=CASE_IDS)
def test_moe_skewed_routing(name, top_k, dt):
    """Every token on the same top_k experts: each of them holds T rows, exactly on and one row past the 64-row (MODE 1)
    and 128-row (MODE 2) block boundaries, with several blocks of either mode for one expert at the larger T.  (The
    16 / 32-row blocks are only chosen when all T * top_k rows fit in one, so no expert spans two of them.)  The partial
    last block of an expert reads the next expert's rows.  Two runs are bit-identical."""
    layers, blk, loop = _stack(name)
    E, K = STACKS[name][:2]
    for T in (16, 17, 32, 33, 64, 65, 128, 129, 257):
        x = _x(T, K, dt, seed=T + 1)
        ids, w = _skewed(T, E, top_k, seed=T)
        y = _check(layers, blk, loop, x, ids, w, f"{name} {dt} skewed T={T}")
        if T in (65, 257):
            assert torch.equal(_grouped(blk, x, ids, w), y)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name,top_k", CASES, ids=CASE_IDS)
def test_moe_sparse_routing(name, top_k, dt):
    """Mostly empty experts (3 tokens), every token on the last expert, ids in descending order within each token, and
    routing weights that are not renormalised (one 0.0, one > 1)."""
    layers, blk, loop = _stack(name)
    E, K = STACKS[name][:2]
    gen = torch.Generator().manual_seed(11)
    x = _x(3, K, dt, seed=3)
    ids, w = _route(3, E, top_k, seed=3)
    _check(layers, blk, loop, x, ids, w, f"{name} {dt} 3 tokens")
    T = 33
    x = _x(T, K, dt, seed=33)
    ids, w = _route(T, E, top_k, seed=33)
    last = ids.clone()  # slot 0 of every token on expert E - 1, the other slots keep distinct experts
    last[:, 0] = E - 1
    for j in range(1, top_k):
        last[:, j] = torch.where(ids[:, j] == E - 1, ids[:, 0], ids[:, j])
    _check(layers, blk, loop, x, last, w, f"{name} {dt} all tokens on expert E-1")
    desc = torch.sort(ids, dim=1, descending=True).values
    _check(layers, blk, loop, x, desc, w, f"{name} {dt} descending ids")
    raw = (torch.rand(T, top_k, generator=gen) * 1.2).to(DEV)
    raw[0, 0], raw[1, top_k - 1] = 0.0, 1.5
    _check(layers, blk, loop, x, ids, raw, f"{name} {dt} unnormalised weights")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name,top_k", CASES, ids=CASE_IDS)
def test_moe_forced_split_k(name, top_k, dt):
    """Every split-K cluster size of the grouped launches (B2Q_MIDM_KS; the launch halves it while a rank would get no
    k-block)."""
    import gptqmodel_b200 as g

    layers, blk, loop = _stack(name)
    E, K = STACKS[name][:2]
    cases = []
    for T in (5, 129):
        x = _x(T, K, dt, seed=50 + T)
        ids, w = _route(T, E, top_k, seed=50 + T)
        cases.append((T, x, ids, w, moe_oracle(x, ids, w, stack_weights(layers, dt, "rounded"))))
    try:
        for ks in (1, 2, 4, 8):
            os.environ["B2Q_MIDM_KS"] = str(ks)
            g.lib.b2q_debug_reload_env()
            for T, x, ids, w, ref in cases:
                assert_moe_close(_grouped(blk, x, ids, w), ref, f"{name} {dt} ks={ks} T={T}")
    finally:
        os.environ.pop("B2Q_MIDM_KS", None)
        g.lib.b2q_debug_reload_env()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name,top_k", CASES, ids=CASE_IDS)
def test_moe_grouped_graph_replay(name, top_k, dt):
    """The grouped path captured in a CUDA graph reads the routing from the device: after new ids / weights are copied
    into the captured tensors (per-expert counts move across block boundaries) a replay matches the oracle and an eager
    run of the new routing bit for bit."""
    layers, blk, loop = _stack(name)
    E, K = STACKS[name][:2]
    T = 65
    x = _x(T, K, dt, seed=65)
    ids, w = _route(T, E, top_k, seed=65)
    idc, wc = ids.clone(), w.clone()
    blk.decode_path = False
    try:
        s_ = torch.cuda.Stream()
        s_.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s_):
            blk(x, idc, wc)
        torch.cuda.current_stream().wait_stream(s_)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            yg = blk(x, idc, wc)
    finally:
        blk.decode_path = True
    for what, (ids2, w2) in (("skewed", _skewed(T, E, top_k, seed=7)), ("softmax", _route(T, E, top_k, seed=66))):
        idc.copy_(ids2)
        wc.copy_(w2)
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, _grouped(blk, x, ids2, w2)), what
        assert_moe_close(yg, moe_oracle(x, ids2, w2, stack_weights(layers, dt, "rounded")),
                         f"{name} {dt} graph replay, {what} routing")
    del gr


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_moe_negative_controls(dt):
    """The tolerance bites: the Mixtral stack's grouped output against the oracle of slightly wrong blocks fails the same
    assertion the tests above pass — routing weights of slots 0 and 1 exchanged, and w1 / w3 of one routed expert
    exchanged."""
    name, top_k = CASES[0]
    layers, blk, _ = _stack(name)
    E, K = STACKS[name][:2]
    T = 16
    x = _x(T, K, dt, seed=16)
    ids, w = _route(T, E, top_k, seed=16)
    y = _grouped(blk, x, ids, w)
    good = stack_weights(layers, dt, "rounded")
    assert_moe_close(y, moe_oracle(x, ids, w, good), "control: correct oracle")
    with pytest.raises(AssertionError, match="outside"):
        assert_moe_close(y, moe_oracle(x, ids, w[:, [1, 0]], good), "control: slot weights swapped")
    e0 = int(ids[0, 0])

    def swapped(e, rows):
        W1, W3, W2 = good(e, rows)
        return (W3, W1, W2) if e == e0 else (W1, W3, W2)

    with pytest.raises(AssertionError, match="outside"):
        assert_moe_close(y, moe_oracle(x, ids, w, swapped), "control: w1 / w3 of one expert swapped")


MAX_GRID_Z = 65535  # gridDim.z limit of every CUDA device


def _populated_z(counts, rows, mode):
    """Largest (expert, token block) index z = e * tblocks + tb of a grouped launch that holds rows, with the token-block
    height launch_midm_grouped picks (b2q_midm.cu): 16 / 32 rows for small launches, else 64 (MODE 1) or 128 (MODE 2)."""
    ntok = 16 if rows <= 16 else 32 if rows <= 32 else 64 if (rows <= 64 or mode == 1) else 128
    tblocks = -(-rows // ntok)
    return max(e * tblocks + (-(-int(c) // ntok)) - 1 for e, c in enumerate(counts) if c > 0)


@pytest.mark.gpu
@pytest.mark.parametrize("E,top_k,T,later_chunks_work",
                         [(128, 8, 4096, False), (256, 8, 2048, False), (256, 8, 8192, True), (8, 2, 65536, False)])
def test_moe_large_prefill(E, top_k, T, later_chunks_work):
    """Prefill chunks whose grouped launches need more than 65535 (expert, token block) pairs, and more than 65535 tokens
    through b2q_moe_combine.  gridDim.z of one launch is at most 65535, so launch_midm_grouped splits such a grid into
    launches over ranges of z.  E = 128 / T = 4096 and E = 256 / T = 2048 are the smallest such prefills at top_k = 8, but
    only the last, always empty, token block lands past the first launch.  E = 256 / T = 8192 puts populated blocks of
    both modes into later launches (MODE 1: 4 launches + 4 z, experts 64.. onwards; MODE 2: experts 128..255 in the
    second launch).  Small K and I keep the oracle cheap."""
    from gptqmodel_b200 import B200QuantLinear, moe

    K, I, gs = 256, 128, 128
    layers = [(random_layer(K, I, group_size=gs, sym=False, seed=5 * e, device=DEV),
               random_layer(K, I, group_size=gs, sym=False, seed=5 * e + 1, device=DEV),
               random_layer(I, K, group_size=gs, sym=False, seed=5 * e + 2, device=DEV)) for e in range(E)]
    mk = lambda L: B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, gs,  # noqa: E731
                                                           sym=False)
    blk = moe.MoEExperts([mk(Ls[0]) for Ls in layers], [mk(Ls[1]) for Ls in layers], [mk(Ls[2]) for Ls in layers],
                         grouped=True)
    for dt in DTYPES:
        x = _x(T, K, dt, seed=T)
        ids, w = _route(T, E, top_k, seed=T + E)
        if later_chunks_work:
            counts = torch.bincount(ids.reshape(-1).cpu(), minlength=E)
            for mode in (1, 2):
                assert _populated_z(counts, T * top_k, mode) >= MAX_GRID_Z, (mode, "no work past the first launch")
        y = blk(x, ids, w)
        assert_moe_close(y, moe_oracle(x, ids, w, stack_weights(layers, dt, "rounded")), f"E={E} T={T} {dt}")


# ---- the routing kernels through the raw ABI: exact equality -------------------------------------------------------------
def _p(t):
    return t.data_ptr()


@pytest.mark.gpu
@pytest.mark.parametrize("E", [1, 8, 60, 128, 256])
def test_moe_align_matches_stable_sort(E):
    """counts = bincount, offsets = exclusive prefix sum, sorted_pairs = the stable argsort of the flattened ids."""
    from gptqmodel_b200._lib import check, lib

    gen = torch.Generator(device=DEV).manual_seed(E)
    st = torch.cuda.current_stream().cuda_stream
    for npairs in (1, 31, 32, 33, 1000, 32768):
        T, top_k = (npairs // 8, 8) if npairs % 8 == 0 and npairs >= 64 else (npairs, 1)
        for skew in (False, True):
            ids = torch.randint(0, E, (T, top_k), dtype=torch.int32, device=DEV, generator=gen)
            if skew:  # most pairs on the last expert
                ids = torch.where(torch.rand(T, top_k, device=DEV, generator=gen) < 0.9, E - 1, ids).to(torch.int32)
            tables = torch.full((2 * E + npairs,), -7, dtype=torch.int32, device=DEV)
            counts, offsets, pairs = tables[:E], tables[E:2 * E], tables[2 * E:]
            check(lib.b2q_moe_align(_p(ids), T, top_k, E, _p(counts), _p(offsets), _p(pairs), st), "b2q_moe_align")
            flat = ids.reshape(-1).long()
            ref = torch.bincount(flat, minlength=E)
            what = f"E={E} pairs={npairs} skew={skew}"
            assert torch.equal(counts.long(), ref), what
            assert torch.equal(offsets.long(), torch.cumsum(ref, 0) - ref), what
            assert torch.equal(pairs.long(), torch.argsort(flat, stable=True)), what


@pytest.mark.gpu
def test_moe_align_rejects_too_many_experts():
    from gptqmodel_b200._lib import lib

    ids = torch.zeros(4, 2, dtype=torch.int32, device=DEV)
    tables = torch.full((2 * 257 + 8,), -7, dtype=torch.int32, device=DEV)
    code = lib.b2q_moe_align(_p(ids), 4, 2, 257, _p(tables), _p(tables[257:]), _p(tables[514:]),
                             torch.cuda.current_stream().cuda_stream)
    assert code != 0
    assert b"at most 256 experts" in lib.b2q_last_error()
    torch.cuda.synchronize()
    assert (tables == -7).all()  # rejected before any launch


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_moe_gather_matches_index_select(dt):
    from gptqmodel_b200._lib import check, lib

    gen = torch.Generator(device=DEV).manual_seed(3)
    st = torch.cuda.current_stream().cuda_stream
    for T, top_k, K in ((1, 1, 8), (7, 2, 264), (300, 8, 2048), (33, 6, 4096)):
        x = torch.randn(T, K, device=DEV, generator=gen).to(dt)
        pairs = torch.randperm(T * top_k, device=DEV, generator=gen).to(torch.int32)
        xs = torch.full((T * top_k, K), float("nan"), dtype=dt, device=DEV)
        check(lib.b2q_moe_gather(_p(x), _p(pairs), _p(xs), T * top_k, top_k, K, st), "b2q_moe_gather")
        assert torch.equal(xs, x.index_select(0, pairs.long() // top_k)), (T, top_k, K)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_moe_combine_matches_fp32_sum(dt):
    """y[t] = T(sum_j ypair[t * top_k + j]): fp32 sum in slot order, one rounding; more than 65535 tokens in one call."""
    from gptqmodel_b200._lib import check, lib

    gen = torch.Generator(device=DEV).manual_seed(4)
    st = torch.cuda.current_stream().cuda_stream
    for T, top_k, N in ((1, 1, 4), (7, 2, 260), (300, 6, 2048), (33, 8, 4096), (70000, 2, 8)):
        ypair = torch.randn(T * top_k, N, device=DEV, generator=gen) * 3
        y = torch.full((T, N), float("nan"), dtype=dt, device=DEV)
        check(lib.b2q_moe_combine(_p(ypair), _p(y), T, top_k, N, 0 if dt == torch.float16 else 1, st), "b2q_moe_combine")
        v = ypair.view(T, top_k, N)
        acc = v[:, 0].clone()
        for j in range(1, top_k):
            acc = acc + v[:, j]
        assert torch.equal(y, acc.to(dt)), (T, top_k, N)
