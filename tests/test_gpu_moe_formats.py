"""8-bit, act-order, mixed-width and widened expert stacks on the grouped MoE path (gptqmodel_b200/moe.py).

Every stack here is grouped-eligible: 8-bit experts run the 8-bit arm of midm_kernel MODE 1 / 2 (b2q_midm.cu), act-order
experts read their activations through b2q_moe_gather_perm (b2q_moe.cu), and a w2 with act-order gets h permuted the same
way before the down launch.  The oracle and tolerance are those of tests/test_gpu_moe.py (see its docstring): act-order only
reorders the terms of the k sum and a wider code only changes the integers, so the derivation holds unchanged.  The oracle
dequantises every layer with its own bit width and g_idx (oracle.dequantize_weight), in the form the serving tier uses:
rounded for the tensor-core tiers, exact where the loop path's b2q_mm applies the scale once per group.
"""
import pytest
import torch

import oracle
from helpers import make_layer, random_layer, scale_once_tier
from test_gpu_moe import DTYPES, MAX_GRID_Z, _grouped, _populated_z, _route, _skewed, _x, assert_moe_close, moe_oracle

DEV = "cuda"

# experts E, hidden K, intermediate I, group size (-1: per channel), symmetric, bits of w1 / w3, bits of w2,
# act-order of w1 / w3 and of w2 ("all", "half" = even experts, None), top_k
STACKS = {
    "qwen1.5_moe_a2.7b_int8": (60, 2048, 1408, 128, True, 8, 8, None, None, 4),
    "edge_g32_int8": (4, 256, 512, 32, False, 8, 8, None, None, 2),
    "edge_per_channel_int8": (4, 256, 512, -1, True, 8, 8, None, None, 2),
    "mixtral_8x7b_tp4_act_order": (8, 4096, 3584, 64, False, 4, 4, "all", "all", 2),
    "mixtral_8x7b_tp4_half_act_order": (8, 4096, 3584, 64, False, 4, 4, "half", "half", 2),
    "gate_up_int4_down_int8": (16, 2048, 1408, 128, False, 4, 8, None, None, 4),
    "int8_act_order": (8, 2048, 1408, 128, False, 8, 8, "all", "all", 2),
    "edge_int2_act_order": (4, 256, 512, 32, False, 2, 2, "all", "all", 2),
}
NAMES = list(STACKS)


def _act_order(L, seed):
    """g_idx = (arange(K) // g)[randperm(K)]: the same codes, rows assigned to groups in a random order."""
    K, gs = L["K"], L["group_size"]
    gen = torch.Generator().manual_seed(seed)
    L["g_idx"] = ((torch.arange(K, dtype=torch.int32) // gs)[torch.randperm(K, generator=gen)]).to(L["qweight"].device)
    L["desc_act"] = True
    return L


def _layer(K, N, bits, gs, sym, seed):
    if bits == 2:  # quantised from a float matrix by the oracle's packer; post_init widens it to 4-bit fields
        L = make_layer(K, N, bits=2, group_size=gs, sym=sym, desc_act=True, seed=seed)
        return {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in L.items()}
    return random_layer(K, N, bits=bits, group_size=gs, sym=sym, seed=seed, device=DEV)


def build_layers(name):
    E, K, I, gs, sym, b13, b2, act13, act2 = STACKS[name][:9]
    on = lambda act, e: act == "all" or (act == "half" and e % 2 == 0)  # noqa: E731
    layers = []
    for e in range(E):
        w1 = _layer(K, I, b13, gs, sym, 3 * e)
        w3 = _layer(K, I, b13, gs, sym, 3 * e + 1)
        w2 = _layer(I, K, b2, gs, sym, 3 * e + 2)
        if on(act13, e):
            if b13 != 2:
                _act_order(w1, 100 + e)
            w3["g_idx"], w3["desc_act"] = w1["g_idx"].clone(), True  # w1 and w3 share the permutation
        if on(act2, e) and b2 != 2:
            _act_order(w2, 200 + e)
        layers.append((w1, w3, w2))
    return layers


def make_module(L):
    from gptqmodel_b200 import B200QuantLinear

    return B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], L["bits"],
                                                   L["group_size"], sym=L["sym"], desc_act=L["desc_act"])


def make_block(layers, **kw):
    from gptqmodel_b200 import moe

    return moe.MoEExperts([make_module(Ls[0]) for Ls in layers], [make_module(Ls[1]) for Ls in layers],
                          [make_module(Ls[2]) for Ls in layers], **kw)


def _scale_once(L, rows):
    """helpers.scale_once_tier for the container width b2q_mm sees (a 2-bit layer runs as 4-bit)."""
    return scale_once_tier({**L, "bits": 4 if L["bits"] <= 4 else 8}, rows)


def _dequant(L, dt, exact):
    sc = L["scales"].to(dt)  # bf16 runs: the fp16 checkpoint scales converted, as the module converts them
    if exact:
        return oracle.dequantize_weight(L["qweight"], L["qzeros"], sc.to(torch.float64), L["g_idx"], L["bits"])
    return oracle.dequantize_weight(L["qweight"], L["qzeros"], sc, L["g_idx"], L["bits"]).to(torch.float64)


def weights(layers, dt, loop=False):
    """moe_oracle's weights(e, rows) callback: every layer with its own bits and g_idx; rounded (tensor-core tiers), or
    for the loop path exact where b2q_mm serves the expert's row count on a scale-once tier."""
    def get(e, rows):
        return tuple(_dequant(L, dt, loop and _scale_once(L, rows)) for L in layers[e])
    return get


_BLOCKS = {}


@pytest.fixture(scope="module", autouse=True)
def _release_stacks():
    yield
    _BLOCKS.clear()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _stack(name):
    """(layers, grouped block, loop block), built once per module run."""
    if name not in _BLOCKS:
        from gptqmodel_b200 import moe

        E, K, I, gs, sym, b13, b2, act13, act2 = STACKS[name][:9]
        layers = build_layers(name)
        blk = make_block(layers)
        assert blk._stack is not None, name
        st = blk._stack
        assert (st["w1"]["bits"], st["w3"]["bits"], st["w2"]["bits"]) == (4 if b13 <= 4 else 8,) * 2 + (
            4 if b2 <= 4 else 8,), name
        assert (st["w1"]["perm"] is not None) == (act13 is not None), name
        assert (st["w2"]["perm"] is not None) == (act2 is not None), name
        loop = moe.MoEExperts(list(blk.w1), list(blk.w3), list(blk.w2), grouped=False)
        assert loop._stack is None
        _BLOCKS[name] = (layers, blk, loop)
    return _BLOCKS[name]


def _check(layers, blk, loop, x, ids, w, what):
    """Grouped and loop path against the oracle; returns the grouped output."""
    dt = x.dtype
    ref = moe_oracle(x, ids, w, weights(layers, dt))
    y = _grouped(blk, x, ids, w)
    assert_moe_close(y, ref, f"{what} grouped")
    counts = torch.bincount(ids.reshape(-1).cpu(), minlength=len(layers))
    loop_exact = any(_scale_once(L, int(c)) for Ls, c in zip(layers, counts) if c > 0 for L in Ls)
    ref_loop = moe_oracle(x, ids, w, weights(layers, dt, loop=True)) if loop_exact else ref
    assert_moe_close(loop(x, ids, w), ref_loop, f"{what} loop")
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", NAMES)
def test_moe_formats_token_counts(name, dt):
    """Softmax top-k routing on both sides of the 16 / 32 / 64 / 128-row token blocks.  One token takes the grouped kernels
    whenever the stack is outside the decode tier's envelope (8-bit or act-order), with or without the decode path."""
    layers, blk, loop = _stack(name)
    E, K, top_k = STACKS[name][0], STACKS[name][1], STACKS[name][9]
    for T in (1, 2, 16, 17, 64, 65, 129, 300):
        x = _x(T, K, dt, seed=T)
        ids, w = _route(T, E, top_k, seed=1000 + T)
        y = _check(layers, blk, loop, x, ids, w, f"{name} {dt} T={T}")
        if T == 1:
            assert not blk._decode_ok(top_k), name
            assert torch.equal(_grouped(blk, x, ids, w, decode_path=True), y)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", NAMES)
def test_moe_formats_skewed_routing(name, dt):
    """Every token on the same top_k experts: exactly on and one row past the 64-row (MODE 1) and 128-row (MODE 2) block
    boundaries.  Two runs are bit-identical."""
    layers, blk, loop = _stack(name)
    E, K, top_k = STACKS[name][0], STACKS[name][1], STACKS[name][9]
    for T in (64, 65, 128, 129):
        x = _x(T, K, dt, seed=T + 1)
        ids, w = _skewed(T, E, top_k, seed=T)
        y = _check(layers, blk, loop, x, ids, w, f"{name} {dt} skewed T={T}")
        if T in (65, 129):
            assert torch.equal(_grouped(blk, x, ids, w), y)


@pytest.mark.gpu
def test_moe_formats_large_prefill_int8():
    """8-bit Qwen3-30B-A3B per-rank stack (E 128, 2048 -> 768, g128, sym), top-8 at T = 8192: both grouped modes need more
    than 65535 (expert, token block) pairs and run as several launches; MODE 1 has populated blocks past the first."""
    from gptqmodel_b200 import moe

    E, K, I, top_k, T = 128, 2048, 768, 8, 8192
    layers = [tuple(random_layer(k, n, bits=8, group_size=128, sym=True, seed=3 * e + j, device=DEV)
                    for j, (k, n) in enumerate(((K, I), (K, I), (I, K)))) for e in range(E)]
    blk = make_block(layers, grouped=True)
    loop = moe.MoEExperts(list(blk.w1), list(blk.w3), list(blk.w2), grouped=False)
    rows = T * top_k
    for mode, ntok in ((1, 64), (2, 128)):
        assert E * (-(-rows // ntok)) > MAX_GRID_Z, (mode, "one launch")
    for dt in DTYPES:
        x = _x(T, K, dt, seed=T)
        ids, w = _route(T, E, top_k, seed=T + E)
        counts = torch.bincount(ids.reshape(-1).cpu(), minlength=E)
        assert _populated_z(counts, rows, 1) >= MAX_GRID_Z, "no MODE 1 work past the first launch"
        _check(layers, blk, loop, x, ids, w, f"qwen3 int8 T={T} {dt}")
    del blk, loop, layers
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_moe_act_order_graph_replay(dt):
    """The act-order grouped path (gather_perm, gate_up, gather_perm of h, down) captured in a CUDA graph: after new ids /
    weights are copied into the captured tensors, a replay matches the oracle and an eager run bit for bit."""
    name = "mixtral_8x7b_tp4_half_act_order"
    layers, blk, _ = _stack(name)
    E, K, top_k = STACKS[name][0], STACKS[name][1], STACKS[name][9]
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
        assert_moe_close(yg, moe_oracle(x, ids2, w2, weights(layers, dt)), f"{name} {dt} graph replay, {what}")
    del gr


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_moe_formats_negative_controls(dt):
    """The tolerance bites on the new paths: the grouped output against an oracle whose routed expert reads h in natural
    order instead of its w2 permutation (act-order stack), and against an oracle with w1 / w3 of one routed 8-bit expert
    exchanged, fails the assertion the tests above pass."""
    name = "mixtral_8x7b_tp4_act_order"
    layers, blk, _ = _stack(name)
    E, K, top_k = STACKS[name][0], STACKS[name][1], STACKS[name][9]
    T = 16
    x = _x(T, K, dt, seed=16)
    ids, w = _route(T, E, top_k, seed=16)
    y = _grouped(blk, x, ids, w)
    good = weights(layers, dt)
    assert_moe_close(y, moe_oracle(x, ids, w, good), "control: correct oracle (act-order)")
    e0 = int(ids[0, 0])
    order = torch.argsort(layers[e0][2]["g_idx"].long(), stable=True)

    def identity_p2(e, rows):  # P2 of e0 the identity: h W2[order] instead of h W2
        W1, W3, W2 = good(e, rows)
        return (W1, W3, W2[order]) if e == e0 else (W1, W3, W2)

    with pytest.raises(AssertionError, match="outside"):
        assert_moe_close(y, moe_oracle(x, ids, w, identity_p2), "control: w2 permutation of one expert the identity")

    name = "qwen1.5_moe_a2.7b_int8"
    layers, blk, _ = _stack(name)
    E, K, top_k = STACKS[name][0], STACKS[name][1], STACKS[name][9]
    x = _x(T, K, dt, seed=17)
    ids, w = _route(T, E, top_k, seed=17)
    y = _grouped(blk, x, ids, w)
    good = weights(layers, dt)
    assert_moe_close(y, moe_oracle(x, ids, w, good), "control: correct oracle (8-bit)")
    e0 = int(ids[0, 0])

    def swapped(e, rows):
        W1, W3, W2 = good(e, rows)
        return (W3, W1, W2) if e == e0 else (W1, W3, W2)

    with pytest.raises(AssertionError, match="outside"):
        assert_moe_close(y, moe_oracle(x, ids, w, swapped), "control: w1 / w3 of one 8-bit expert swapped")


@pytest.mark.gpu
def test_moe_unequal_w1_w3_permutations_stay_on_the_loop_path():
    """w1 and w3 of an expert read the same gathered activations, so a stack where one expert's w1 and w3 permutations
    differ is not grouped-eligible: it runs the per-expert loop, and grouped=True refuses it."""
    layers = build_layers("edge_g32_int8")
    for Ls in layers:
        _act_order(Ls[0], 7)
        _act_order(Ls[1], 7)
    _act_order(layers[1][1], 8)  # expert 1: w3 with a permutation of its own
    blk = make_block(layers)
    assert blk._stack is None
    with pytest.raises(ValueError, match="grouped=True"):
        make_block(layers, grouped=True)
    x = _x(9, 256, torch.float16, seed=9)
    ids, w = _route(9, 4, 2, seed=9)
    assert_moe_close(blk(x, ids, w), moe_oracle(x, ids, w, weights(layers, torch.float16, loop=True)),
                     "unequal w1 / w3 permutations, loop path")


# ---- b2q_moe_gather_perm through the raw ABI: exact equality ------------------------------------------------------------
def _p(t):
    return t.data_ptr()


def _gather_perm_ref(src, pairs, perms, offsets, top_k):
    """dst[i, k'] = src[r(i), perms[e(i), k']], e(i) = the last expert whose first row is <= i."""
    i = torch.arange(pairs.numel() if pairs is not None else src.shape[0], device=DEV)
    e = torch.searchsorted(offsets.long(), i, right=True) - 1
    r = pairs.long() // top_k if pairs is not None else i
    return torch.stack([src[r[j]].index_select(0, perms[e[j]].long()) for j in range(i.numel())])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_moe_gather_perm_matches_index_select(dt):
    """dst[i] = src[r(i)].index_select(0, perms[e(i)]) for the rows of every expert: experts without rows (at the start, in
    the middle and at the end), E = 256, a single expert, and the sorted_pairs == NULL form that permutes h."""
    from gptqmodel_b200._lib import check, lib

    gen = torch.Generator(device=DEV).manual_seed(5)
    st = torch.cuda.current_stream().cuda_stream
    for E, T, top_k, K in ((1, 5, 1, 8), (8, 7, 2, 264), (60, 300, 4, 2048), (256, 33, 8, 1408), (256, 2, 1, 64)):
        x = torch.randn(T, K, device=DEV, generator=gen).to(dt)
        ids = torch.randint(0, E, (T, top_k), device=DEV, generator=gen).to(torch.int32)
        if E >= 8:
            ids = torch.where(ids == 0, E - 2, ids).to(torch.int32)  # expert 0 empty, as may be others
        tables = torch.empty(2 * E + T * top_k, dtype=torch.int32, device=DEV)
        counts, offsets, pairs = tables[:E], tables[E:2 * E], tables[2 * E:]
        check(lib.b2q_moe_align(_p(ids), T, top_k, E, _p(counts), _p(offsets), _p(pairs), st), "b2q_moe_align")
        perms = torch.stack([torch.randperm(K, device=DEV, generator=gen) for _ in range(E)]).to(torch.int32)
        rows = T * top_k
        xs = torch.full((rows, K), float("nan"), dtype=dt, device=DEV)
        check(lib.b2q_moe_gather_perm(_p(x), _p(pairs), _p(perms), _p(offsets), E, _p(xs), rows, top_k, K, st),
              "b2q_moe_gather_perm")
        assert torch.equal(xs, _gather_perm_ref(x, pairs, perms, offsets, top_k)), (E, T, top_k, K)
        h2 = torch.full_like(xs, float("nan"))
        check(lib.b2q_moe_gather_perm(_p(xs), None, _p(perms), _p(offsets), E, _p(h2), rows, top_k, K, st),
              "b2q_moe_gather_perm")
        assert torch.equal(h2, _gather_perm_ref(xs, None, perms, offsets, top_k)), (E, T, top_k, K, "NULL pairs")
        assert int((counts == 0).sum()) >= (1 if E >= 8 else 0)


@pytest.mark.gpu
def test_moe_gather_perm_rejects_bad_arguments():
    """Rejected before any launch: more than 256 experts, K not a multiple of 8, a misaligned destination or permutation
    table, missing tables."""
    from gptqmodel_b200._lib import lib

    st = torch.cuda.current_stream().cuda_stream
    K, rows = 64, 4
    x = torch.zeros(rows, K, dtype=torch.float16, device=DEV)
    pairs = torch.arange(rows, dtype=torch.int32, device=DEV)
    offsets = torch.zeros(257, dtype=torch.int32, device=DEV)
    perms = torch.zeros(257 * K + 8, dtype=torch.int32, device=DEV)
    dst = torch.full((rows * K + 8,), -1.0, dtype=torch.float16, device=DEV)
    cases = [
        ("257 experts", (_p(x), _p(pairs), _p(perms), _p(offsets), 257, _p(dst), rows, 1, K), b"at most 256 experts"),
        ("K % 8", (_p(x), _p(pairs), _p(perms), _p(offsets), 4, _p(dst), rows, 1, K - 4), b"bad argument"),
        ("misaligned dst", (_p(x), _p(pairs), _p(perms), _p(offsets), 4, _p(dst) + 2, rows, 1, K), b"bad argument"),
        ("misaligned perms", (_p(x), _p(pairs), _p(perms) + 4, _p(offsets), 4, _p(dst), rows, 1, K), b"bad argument"),
        ("no perms", (_p(x), _p(pairs), None, _p(offsets), 4, _p(dst), rows, 1, K), b"bad argument"),
        ("no offsets", (_p(x), _p(pairs), _p(perms), None, 4, _p(dst), rows, 1, K), b"bad argument"),
        ("top_k 0", (_p(x), _p(pairs), _p(perms), _p(offsets), 4, _p(dst), rows, 0, K), b"bad argument"),
    ]
    for what, args, msg in cases:
        assert lib.b2q_moe_gather_perm(*args, st) != 0, what
        assert msg in lib.b2q_last_error(), (what, lib.b2q_last_error())
    torch.cuda.synchronize()
    assert (dst == -1.0).all()
