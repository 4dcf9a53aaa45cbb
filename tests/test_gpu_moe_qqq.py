"""QQQ (W4A8) MoE experts on the grouped int8 path of gptqmodel_b200/moe.py.

Path: b2q_moe_align -> b2q_qqq_moe_gather (quantise the sorted rows) -> qqq_moe_gemm_kernel MODE 1 (64 gate + 64 up
features per tile, SiLU-mul epilogue) -> b2q_qqq_quantize of h -> MODE 2 (down, routing weight, scatter) ->
b2q_moe_combine.  include/b2q.h states the rounding points; they are those of the per-expert loop over QQQLinear modules.

The accumulation is int32 and exact, so the stages are held to the layer kernel (b2q_qqq_mm, itself bit-exact to
oracle/qqq_oracle.py) bit for bit, except T(silu(g)), where __expf and torch's exp may round one ulp apart.  Such a flip
changes h, and then the down output only through the requantisation Q(h) of that row (assert_block_equals_chain).
"""
import json
import os

import pytest
import torch

from oracle import qqq_oracle as qo
from test_gpu_moe import _route, _skewed, _ulp

DEV = "cuda"
DTYPES = (torch.float16, torch.bfloat16)
TNAME = {torch.float16: "fp16", torch.bfloat16: "bf16"}
DT = {torch.float16: 0, torch.bfloat16: 1}


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _kp(K):
    return (K + 127) // 128 * 128


# ---- experts ------------------------------------------------------------------------------------------------------------
def _role(E, N, K, gs, seed):
    """E QQQ modules [K -> N] and their canonical tensors [(codes, s_channel, s_group)] on the device."""
    from gptqmodel_b200 import B200QqqQuantLinear

    g = torch.Generator().manual_seed(seed)
    mods, canon = [], []
    for _ in range(E):
        codes = torch.randint(0, 16, (K, N), generator=g).to(torch.uint8)
        # |w| ~ 74 on average: s_channel ~ 1 / (127 sqrt(K)) gives outputs of order one for unit-scale inputs
        sc = (torch.rand(N, generator=g) + 0.5) / (127 * K ** 0.5)
        sg = (torch.rand(K // 128, N, generator=g) * 14.9 + 1.0).to(torch.float16) if gs == 128 else None
        if sg is not None:
            sc = sc / 8
        B, scp, sgp = qo.pack_qqq(codes, sc, sg)
        mods.append(B200QqqQuantLinear.from_checkpoint_tensors(B, scp, sgp if gs == 128 else None, gs, device=DEV))
        canon.append((codes.to(DEV), sc.to(DEV), None if sg is None else sg.to(DEV)))
    return mods, canon


# E, hidden K, intermediate I, top_k, group size of w1 / w3, of w2
STACKS = {
    "small_g128": (8, 512, 256, 2, 128, 128),
    "tail_perchannel": (6, 256, 320, 4, -1, -1),    # I % 128 == 64: a half-filled packed tile in gate|up
    "mixed_kinds": (16, 384, 192, 8, 128, -1),      # w2 per-channel, w1 / w3 group 128
}
_BLOCKS = {}


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    _BLOCKS.clear()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _stack(name):
    if name not in _BLOCKS:
        from gptqmodel_b200 import moe

        E, K, I, _, g1, g2 = STACKS[name]
        roles = {"w1": _role(E, I, K, g1, 1), "w3": _role(E, I, K, g1, 2), "w2": _role(E, K, I, g2, 3)}
        blk = moe.MoEExperts(*[roles[r][0] for r in ("w1", "w3", "w2")], grouped=True)
        assert "qqq" in blk._stack
        _BLOCKS[name] = (roles, blk)
    return _BLOCKS[name]


def _x(T, K, dt, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(T, K, device=DEV, generator=gen)
    if T > 2:
        x[T // 2] = 0.0  # an all-zero token: s_tok = 0, codes 0
    return x.to(dt)


# ---- the raw ABI: the six launches and the layer kernel -----------------------------------------------------------------
def _align(ids, E):
    from gptqmodel_b200._lib import check, lib

    T, top_k = ids.shape
    tables = torch.empty(2 * E + T * top_k, dtype=torch.int32, device=DEV)
    ids32 = ids.to(torch.int32).contiguous()
    check(lib.b2q_moe_align(_p(ids32), T, top_k, E, _p(tables), _p(tables[E:]), _p(tables[2 * E:]), _st()), "align")
    return tables[:E], tables[E:2 * E], tables[2 * E:]


def _quantize(x):
    from gptqmodel_b200._lib import check, lib

    M, K = x.shape
    q = torch.empty((M, _kp(K)), dtype=torch.int8, device=DEV)
    s = torch.empty(M, dtype=torch.float32, device=DEV)
    check(lib.b2q_qqq_quantize(_p(x), _p(q), _p(s), M, K, DT[x.dtype], _st()), "b2q_qqq_quantize")
    return q, s


def _mm(q, s, m, dt, sc=None):
    """T(b2q_qqq_mm) of module m's prepacked tensors on codes q / scales s (sc: other channel scales)."""
    from gptqmodel_b200._lib import check, lib

    M = q.shape[0]
    out = torch.empty((M, m.out_features), dtype=dt, device=DEV)
    check(lib.b2q_qqq_mm(_p(q), _p(s), _p(m.packed), _p(m._sc if sc is None else sc), _p(m._sg), None, _p(out), M,
                         m.in_features, m.out_features, m._kgs, DT[dt], _st()), "b2q_qqq_mm")
    return out


def _block_abi(blk, x, ids, w):
    """(sorted_pairs, codes, s_x, h sorted, ypair by pair, y) of the grouped block through the raw ABI."""
    from gptqmodel_b200._lib import check, lib

    T, top_k = ids.shape
    s1, s3, s2 = blk._stack["w1"], blk._stack["w3"], blk._stack["w2"]
    E, K, I, H = len(blk.w1), s1["K"], s1["N"], s2["N"]
    rows, dt, code = T * top_k, x.dtype, DT[x.dtype]
    counts, offsets, pairs = _align(ids, E)
    codes = torch.empty((rows, _kp(K)), dtype=torch.int8, device=DEV)
    sx = torch.empty(rows, dtype=torch.float32, device=DEV)
    check(lib.b2q_qqq_moe_gather(_p(x), _p(pairs), _p(codes), _p(sx), T, top_k, K, code, _st()), "gather")
    h = torch.empty((rows, I), dtype=dt, device=DEV)
    active = min(E, rows)
    check(lib.b2q_qqq_moe_gate_up(_p(codes), _p(sx), _p(s1["packed"]), _p(s1["sc"]), _p(s1["sg"]), _p(s3["packed"]),
                                  _p(s3["sc"]), _p(s3["sg"]), _p(h), _p(counts), _p(offsets), E, rows, active, K, I,
                                  s1["group"], code, _st()), "gate_up")
    ch, sh = _quantize(h)
    yp = torch.empty((rows, H), dtype=torch.float32, device=DEV)
    wf = w.to(torch.float32).contiguous()
    check(lib.b2q_qqq_moe_down(_p(ch), _p(sh), _p(s2["packed"]), _p(s2["sc"]), _p(s2["sg"]), _p(counts), _p(offsets),
                               _p(pairs), _p(wf), _p(yp), E, rows, active, I, H, s2["group"], code, _st()), "down")
    y = torch.empty((T, H), dtype=dt, device=DEV)
    check(lib.b2q_moe_combine(_p(yp), _p(y), T, top_k, H, code, _st()), "combine")
    return pairs, codes, sx, h, yp, y


def _expert_rows(counts, offsets):
    c, o = counts.tolist(), offsets.tolist()
    return [(e, o[e], o[e] + c[e]) for e in range(len(c)) if c[e] > 0]


def _chain(blk, x, ids, w, defect=None):
    """The per-expert loop over the same modules, stage by stage: g = w1_e(x), u = w3_e(x), h = T(T(silu(g)) * u) with
    torch's exp, yp = w * w2_e(h).  Returns (h sorted, ypair by pair).  defect (negative controls): "no_q_h" = down on
    the unquantised h (float64 product, fp16 rounding), "next_scales" = the next expert's w2 channel scales."""
    T, top_k = ids.shape
    E, dt = len(blk.w1), x.dtype
    counts, offsets, pairs = _align(ids, E)
    I, H = blk.w1[0].out_features, blk.w2[0].out_features
    h = torch.empty((T * top_k, I), dtype=dt, device=DEV)
    yp = torch.zeros(T * top_k, H, dtype=torch.float32, device=DEV)
    wf = w.to(torch.float32).reshape(-1)
    for e, r0, r1 in _expert_rows(counts, offsets):
        p = pairs[r0:r1].long()
        xe = x[p // top_k].contiguous()
        g, u = blk.w1[e](xe).float(), blk.w3[e](xe).float()
        he = ((g / (1 + torch.exp(-g))).to(dt).float() * u).to(dt)
        h[r0:r1] = he
        m2 = blk.w2[e]
        if defect == "no_q_h":
            W2 = qo.weight_int8(*_canon_w2(blk, e)).double() * m2._sc.double()
            ye = (he.double() @ W2).to(torch.float16).to(dt).float()
        elif defect == "next_scales":
            ye = _mm(*_quantize(he), m2, dt, sc=blk.w2[(e + 1) % E]._sc).float()
        else:
            ye = m2(he).float()
        yp[p] = wf[p][:, None] * ye
    return h, yp


def _canon_w2(blk, e):
    return blk._canon_w2[e]


def assert_block_equals_chain(block, chain, blk, ids, w, what):
    """Every pair whose h row equals the chain's has a bit-identical ypair row (and a token whose pairs all do, a
    bit-identical output); at least half the pairs do.  Another pair differs only through Q(h): with both quantisations
    within s_h / 2 of their h, |dyp| <= |w| (sum_k (|dh_k| + (s_h + s_h') / 2) |W2[k, n]| + 2 ulp(yp))."""
    pairs, _, _, h, yp, y = block
    h_c, yp_c = chain
    T, top_k = ids.shape
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
    bad = (~same_sorted).nonzero().squeeze(1)
    if bad.numel():
        _, s_b = _quantize(h[bad].contiguous())
        _, s_c = _quantize(h_c[bad].contiguous())
    for i, r in enumerate(bad.tolist()):
        p, e = int(pl[r]), int(flat[pl[r]])
        W2 = (qo.weight_int8(*_canon_w2(blk, e)).double() * blk.w2[e]._sc.double()).abs()
        dh = (h[r].double() - h_c[r].double()).abs() + 0.5 * (float(s_b[i]) + float(s_c[i]))
        ye_c = yp_c[p] / wf[p] if float(wf[p]) != 0 else yp_c[p]
        tol = wf[p].abs() * ((dh @ W2).float() * (1 + 2 ** -10) + 2 * _ulp(ye_c, dt)) + 1e-30
        err = (yp[p] - yp_c[p]).abs()
        assert (err <= tol).all(), (what, "pair", p, float((err / tol).max()))
    return n_same


def _with_canon(name):
    roles, blk = _stack(name)
    blk._canon_w2 = [(c, sg) for c, _, sg in roles["w2"][1]]
    return roles, blk


# ---- stages -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_gather_quantise_equals_oracle(dt):
    """Sorted row i quantises token sorted_pairs[i] / top_k: codes and scale equal qqq_oracle.quantize bit for bit, and
    the padding codes up to 128 k are 0."""
    _, blk = _with_canon("tail_perchannel")
    E, K, *_ = STACKS["tail_perchannel"]
    for T, top_k in ((1, 1), (37, 4), (300, 8)):
        x = _x(T, K, dt, seed=T)
        ids, w = _route(T, E, min(top_k, E), seed=T)
        pairs, codes, sx, *_ = _block_abi(blk, x, ids, w)
        rq, rs = qo.quantize(x[pairs.long() // ids.shape[1]].cpu())
        assert torch.equal(codes[:, :K].cpu(), rq), (T, top_k)
        assert torch.equal(sx.cpu(), rs), (T, top_k)
        assert not codes[:, K:].any()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", list(STACKS))
def test_stages_equal_layer_kernel(name, dt):
    """Per expert's rows: down = w[pair] * T(b2q_qqq_mm) bit for bit; gate|up within one ulp of T of T(T(silu(g)) * u)
    with g, u = b2q_qqq_mm (bit-exact to the oracle); the gate / up values themselves are checked against the oracle."""
    roles, blk = _with_canon(name)
    E, K, I, top_k, *_ = STACKS[name]
    for T, routing in ((1, "softmax"), (9, "softmax"), (130, "skewed"), (300, "softmax")):
        x = _x(T, K, dt, seed=3 * T)
        ids, w = (_route if routing == "softmax" else _skewed)(T, E, top_k, seed=T)
        pairs, codes, sx, h, yp, _ = _block_abi(blk, x, ids, w)
        counts, offsets, _ = _align(ids, E)
        wf = w.to(torch.float32).reshape(-1)
        ch, sh = _quantize(h)
        flips = 0
        for e, r0, r1 in _expert_rows(counts, offsets):
            g = _mm(codes[r0:r1], sx[r0:r1], blk.w1[e], dt)
            u = _mm(codes[r0:r1], sx[r0:r1], blk.w3[e], dt)
            if e == 0 or r1 - r0 > 64:
                xe = x[pairs[r0:r1].long() // top_k]
                assert torch.equal(g, qo.forward(xe, *roles["w1"][1][e])), (name, e, "gate against the oracle")
            gf, uf = g.float(), u.float()
            ref = ((gf / (1 + torch.exp(-gf))).to(dt).float() * uf).to(dt)
            d = (h[r0:r1].float() - ref.float()).abs()
            assert (d <= _ulp(ref.float(), dt)).all(), (name, TNAME[dt], T, e, "gate|up")
            flips += int((d > 0).sum())
            y = _mm(ch[r0:r1], sh[r0:r1], blk.w2[e], dt).float()
            p = pairs[r0:r1].long()
            assert torch.equal(yp[p], wf[p][:, None] * y), (name, TNAME[dt], T, e, "down")
        assert flips <= h.numel() // 100, (name, "too many one-ulp flips", flips)


# ---- the block ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", list(STACKS))
def test_block_equals_module_loop(name, dt):
    """MoEExperts (grouped) against the loop over the same B200QqqQuantLinear modules at T = 1..300 (a sample below 17
    is every T) and 2048, top_k 1, 2, 4, 8, softmax / skewed / sparse routing; MoEExperts' output equals the raw-ABI
    block bit for bit."""
    _, blk = _with_canon(name)
    E, K, _, top_k, *_ = STACKS[name]
    Ts = list(range(1, 17)) + [31, 64, 65, 127, 128, 129, 200, 255, 300, 2048]
    for T in Ts:
        x = _x(T, K, dt, seed=T)
        k = [1, 2, 4, 8][T % 4] if T < 17 else top_k
        k = min(k, E)
        ids, w = (_skewed if T % 3 == 0 else _route)(T, E, k, seed=T)
        if T % 5 == 0:
            ids = torch.where(ids % 3 == 0, ids, torch.full_like(ids, E - 1))  # most experts empty
        what = f"qqq moe {name} {TNAME[dt]} T={T} top_k={k}"
        block = _block_abi(blk, x, ids, w)
        assert torch.equal(blk(x, ids, w), block[5]), what
        assert_block_equals_chain(block, _chain(blk, x, ids, w), blk, ids, w, what)


@pytest.mark.gpu
def test_negative_controls():
    """Each check above fails for: slot weights swapped, the next expert's w2 scales, down fed the unquantised h.
    Biased, adapted and mixed stacks take the loop, and grouped=True refuses them."""
    from gptqmodel_b200 import B200QqqQuantLinear, Lora, moe

    _, blk = _with_canon("small_g128")
    E, K, I, top_k, *_ = STACKS["small_g128"]
    T = 64
    x = _x(T, K, torch.float16, seed=64)
    ids, w = _route(T, E, top_k, seed=64)
    block = _block_abi(blk, x, ids, w)
    assert_block_equals_chain(block, _chain(blk, x, ids, w), blk, ids, w, "control: correct")
    for defect in ("no_q_h", "next_scales"):
        with pytest.raises(AssertionError):
            assert_block_equals_chain(block, _chain(blk, x, ids, w, defect), blk, ids, w, f"control {defect}")
    with pytest.raises(AssertionError):
        assert_block_equals_chain(block, _chain(blk, x, ids, w[:, [1, 0]]), blk, ids, w, "control: swapped weights")
    roles = {r: _role(2, n, k, 128, 40 + i) for i, (r, n, k) in enumerate((("w1", I, K), ("w3", I, K), ("w2", K, I)))}
    mods = lambda: [list(roles[r][0]) for r in ("w1", "w3", "w2")]  # noqa: E731
    assert "qqq" in moe.MoEExperts(*mods())._stack
    codes, sc, sg = roles["w2"][1][1]
    B, scp, sgp = qo.pack_qqq(codes, sc, sg)
    biased = mods()
    biased[2][1] = B200QqqQuantLinear.from_checkpoint_tensors(B, scp, sgp, 128, bias=torch.zeros(K), device=DEV)
    adapted = mods()
    gen = torch.Generator().manual_seed(0)
    lora = Lora(lora_A=(torch.randn(K, 8, generator=gen) * 0.05).half(),
                lora_B=(torch.randn(8, I, generator=gen) * 0.05).half())
    adapted[0][0] = B200QqqQuantLinear.from_checkpoint_tensors(*qo.pack_qqq(*roles["w1"][1][0]), 128, device=DEV)
    adapted[0][0].adapter = lora
    mixed = mods()
    mixed[1][0] = _role(1, I, K, -1, 50)[0][0]  # w3 per-channel, w1 group 128
    for what, sets in (("bias", biased), ("adapter", adapted), ("mixed group kinds", mixed)):
        assert moe.MoEExperts(*sets, fuse=False)._stack is None, what
        with pytest.raises(ValueError, match="B200QqqQuantLinear"):
            moe.MoEExperts(*sets, grouped=True)
    with pytest.raises(ValueError, match="does not fit"):
        blk(x[:, :128].contiguous(), ids, w)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_graph_replay_equals_eager(dt):
    """The six launches captured in a CUDA graph read the routing from the device: after new ids / weights are copied
    in, a replay equals an eager run bit for bit."""
    _, blk = _with_canon("small_g128")
    E, K, _, top_k, *_ = STACKS["small_g128"]
    T = 33
    x = _x(T, K, dt, seed=33)
    ids, w = _route(T, E, top_k, seed=33)
    idc, wc = ids.clone(), w.clone()
    s_ = torch.cuda.Stream()
    s_.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s_):
        blk(x, idc, wc)
    torch.cuda.current_stream().wait_stream(s_)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        yg = blk(x, idc, wc)
    for ids2, w2 in (_skewed(T, E, top_k, seed=7), _route(T, E, top_k, seed=34)):
        idc.copy_(ids2)
        wc.copy_(w2)
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, blk(x, ids2, w2))
    del gr


@pytest.mark.gpu
def test_large_prefill_splits_the_grid():
    """E = 256, top_k = 8, T = 8192: 65536 rows in 128-row blocks give 256 * 512 (expert, token block) pairs, so both
    grouped launches are issued over several ranges of gridDim.z; the block still equals the module loop."""
    from gptqmodel_b200 import moe

    E, K, I, top_k, T = 256, 256, 128, 8, 8192
    roles = {"w1": _role(E, I, K, 128, 61), "w3": _role(E, I, K, 128, 62), "w2": _role(E, K, I, -1, 63)}
    blk = moe.MoEExperts(*[roles[r][0] for r in ("w1", "w3", "w2")], grouped=True)
    blk._canon_w2 = [(c, sg) for c, _, sg in roles["w2"][1]]
    ids, w = _route(T, E, top_k, seed=5)
    counts = torch.bincount(ids.reshape(-1).cpu(), minlength=E)
    assert int(counts[E // 2:].sum()) > 0 and (E - 1) * 512 >= 65535
    x = _x(T, K, torch.bfloat16, seed=T)
    block = _block_abi(blk, x, ids, w)
    assert torch.equal(blk(x, ids, w), block[5])
    assert_block_equals_chain(block, _chain(blk, x, ids, w), blk, ids, w, "qqq moe large prefill")


@pytest.mark.gpu
def test_qwen3_moe_checkpoint_through_loader(tmp_path):
    """A tiny safetensors QQQ checkpoint with Qwen3-MoE module names goes through load_quantized_linears and runs
    grouped, equal to the module loop stage by stage."""
    from safetensors.torch import save_file

    from gptqmodel_b200 import moe
    from gptqmodel_b200.loader import load_quantized_linears

    E, K, I = 4, 256, 256
    proj = {"w1": ("gate_proj", I, K), "w3": ("up_proj", I, K), "w2": ("down_proj", K, I)}
    g = torch.Generator().manual_seed(3)
    tensors = {}
    for r, (name, n, k) in proj.items():
        for e in range(E):
            codes = torch.randint(0, 16, (k, n), generator=g).to(torch.uint8)
            sg = (torch.rand(k // 128, n, generator=g) * 14.9 + 1.0).to(torch.float16)
            B, scp, sgp = qo.pack_qqq(codes, (torch.rand(n, generator=g) + 0.5) / (127 * 64 * k ** 0.5), sg)
            pre = f"model.layers.0.mlp.experts.{e}.{name}"
            tensors.update({pre + ".B": B, pre + ".s_channel": scp, pre + ".s_group": sgp})
    with open(os.path.join(tmp_path, "config.json"), "w") as f:
        json.dump({"model_type": "qwen3_moe", "quantization_config": {
            "quant_method": "qqq", "bits": 4, "group_size": 128, "sym": True, "desc_act": False, "format": "qqq"}}, f)
    save_file(tensors, os.path.join(tmp_path, "model.safetensors"))
    mods = load_quantized_linears(str(tmp_path), device=DEV)
    get = lambda r: [mods[f"model.layers.0.mlp.experts.{e}.{proj[r][0]}"] for e in range(E)]  # noqa: E731
    blk = moe.MoEExperts(get("w1"), get("w3"), get("w2"), grouped=True)
    blk._canon_w2 = [_canon_from_ckpt(tensors, e) for e in range(E)]
    for dt in DTYPES:
        x = _x(9, K, dt, seed=9)
        ids, w = _route(9, E, 2, seed=9)
        block = _block_abi(blk, x, ids, w)
        assert torch.equal(blk(x, ids, w), block[5])
        assert_block_equals_chain(block, _chain(blk, x, ids, w), blk, ids, w, f"qqq checkpoint {TNAME[dt]}")


def _canon_from_ckpt(tensors, e):
    pre = f"model.layers.0.mlp.experts.{e}.down_proj"
    codes, _, sg = qo.unpack_qqq(tensors[pre + ".B"], tensors[pre + ".s_channel"], tensors[pre + ".s_group"])
    return codes.to(DEV), sg.to(DEV)
