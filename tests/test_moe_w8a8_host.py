"""CPU: the per-channel W8A8 MoE experts of B200ChannelW8A8Experts without a GPU.

  * the argument checks of the six grouped entry points (b2q_fp8ch_moe_* / b2q_int8ch_moe_*), which return -2 before
    any CUDA work;
  * the compiler's report: no spills and no stack frame in any new kernel;
  * the block oracle of include/b2q.h against MoEExperts(grouped=False) over dense stand-in experts that run the numpy
    mirrors of the layers (tests/fp8_w8a8_mirror.py, tests/int8_w8a8_mirror.py) bit for bit, so the loop and the oracle
    differ only in the order of the final sum over slots;
  * the stack qualification rules, on CPU modules marked ready.
"""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import fp8_w8a8_mirror as fm
import int8_w8a8_mirror as im
from gptqmodel_b200 import B200ChannelFp8Linear, B200ChannelInt8Linear, B200ChannelW8A8Experts, lib, moe
from gptqmodel_b200.fp8_channel import channel_scales
from helpers import assert_close_rel

HERE = os.path.dirname(os.path.abspath(__file__))
DTYPES = (torch.float16, torch.bfloat16)
TNAME = {torch.float16: "fp16", torch.bfloat16: "bf16"}
P = 1 << 20  # any 16-byte aligned non-NULL value: a refused call never dereferences it


# ---- ABI argument checks ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["fp8", "int8"])
def test_gather_argument_checks(fmt):
    fn = getattr(lib, f"b2q_{fmt}ch_moe_gather")

    def call(**kw):
        a = {"x": P, "pairs": P, "offsets": P, "s_in": None, "E": 8, "codes": P, "sx": P, "T": 4, "top_k": 2, "K": 256,
             "ub": float("inf"), "dt": 0, **kw}
        ub = () if fmt == "int8" else (a["ub"],)
        return fn(a["x"], a["pairs"], a["offsets"], a["s_in"], a["E"], a["codes"], a["sx"], a["T"], a["top_k"], a["K"],
                  *ub, a["dt"], None)

    bad = [dict(x=None), dict(codes=None), dict(sx=None), dict(x=P + 2), dict(codes=P + 8), dict(sx=P + 4), dict(T=0),
           dict(top_k=0), dict(K=100), dict(K=64), dict(K=0), dict(K=65536 + 128), dict(dt=2),
           dict(s_in=P, offsets=None), dict(s_in=P, E=0), dict(s_in=P, E=257)]
    if fmt == "fp8":
        bad += [dict(ub=0.0), dict(ub=-1.0), dict(ub=float("nan"))]
    for kw in bad:
        assert call(**kw) == -2, kw
        assert lib.b2q_last_error()


@pytest.mark.parametrize("fmt", ["fp8", "int8"])
def test_gate_up_and_down_argument_checks(fmt):
    gate_up, down = getattr(lib, f"b2q_{fmt}ch_moe_gate_up"), getattr(lib, f"b2q_{fmt}ch_moe_down")
    good = dict(codes=P, sx=P, w=P, s=P, w3=P, s3=P, out=P, counts=P, offsets=P, pairs=P, wts=P, E=8, rows=16, active=8,
                K=256, N=128, dt=1, ks=0)

    def gu(**kw):
        a = {**good, **kw}
        return gate_up(a["codes"], a["sx"], a["w"], a["s"], a["w3"], a["s3"], a["out"], a["counts"], a["offsets"], a["E"],
                       a["rows"], a["active"], a["K"], a["N"], a["dt"], a["ks"], None)

    def dn(**kw):
        a = {**good, **kw}
        return down(a["codes"], a["sx"], a["w"], a["s"], a["counts"], a["offsets"], a["pairs"], a["wts"], a["out"], a["E"],
                    a["rows"], a["active"], a["K"], a["N"], a["dt"], a["ks"], None)

    common = [dict(codes=None), dict(sx=None), dict(w=None), dict(s=None), dict(out=None), dict(counts=None),
              dict(offsets=None), dict(codes=P + 8), dict(sx=P + 4), dict(w=P + 4), dict(s=P + 4), dict(out=P + 2),
              dict(E=0), dict(E=257), dict(rows=0), dict(ks=9), dict(K=192), dict(K=64), dict(K=65536 + 128),
              dict(N=96), dict(N=0), dict(dt=2)]
    for kw in common + [dict(w3=None), dict(s3=None), dict(w3=P + 8), dict(s3=P + 4)]:
        assert gu(**kw) == -2, ("gate_up", kw)
    for kw in common + [dict(pairs=None), dict(wts=None)]:
        assert dn(**kw) == -2, ("down", kw)


def test_new_kernels_do_not_spill():
    log = os.path.join(os.path.dirname(HERE), "gptqmodel_b200", "csrc", "b2q_fp8ch.o.log")
    if not os.path.exists(log):
        pytest.skip("b2q_fp8ch.o.log is written by the in-tree build")
    entries = re.findall(r"Compiling entry function '(\w+)'.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", open(log).read(), flags=re.S)
    new = [e for e in entries if "ch_moe_" in e[0]]
    assert sum("fp8ch_moe_gemm_kernel" in e[0] for e in new) == 10  # 5 token widths x gate|up / down
    assert sum("int8ch_moe_gemm_kernel" in e[0] for e in new) == 10
    assert sum("fp8ch_moe_gather_kernel" in e[0] for e in new) == 2
    assert sum("int8ch_moe_gather_kernel" in e[0] for e in new) == 2
    for name, stack, st, ld in new:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), name


# ---- the block oracle against the loop ----------------------------------------------------------------------------------
class _Dense(torch.nn.Module):
    """Stand-in W8A8 expert: the numpy mirror of the layer (quantiser, k-sum, epilogue without bias), output in T."""

    def __init__(self, fmt, w, s_w, s_in=None, ub=np.inf):
        super().__init__()
        self.fmt, self.w, self.s_w, self.s_in, self.ub = fmt, w, s_w, s_in, ub

    def forward(self, x):
        dt = TNAME[x.dtype]
        xf = x.float().numpy()
        if self.fmt == "int8":
            c, s = im.quantize_dynamic(xf) if self.s_in is None else im.quantize_static(xf, self.s_in)
            y = im.epilogue(im.int_sums(c, self.w), s, self.s_w, None, dt)
        else:
            c, s = fm.quantize_dynamic(xf, self.ub) if self.s_in is None else fm.quantize_static(xf, self.s_in)
            y = fm.epilogue(fm.promote(c, self.w, 1), s, self.s_w, None, dt)
        return torch.from_numpy(np.asarray(y, np.float32)).to(x.dtype)


def w8a8_block_oracle(x, ids, w, roles):
    """include/b2q.h per routed pair (t, j, e): (c, s_x) = Q(x_t); g, u = the layers' values; h = T(T(silu(g)) * u);
    yp_j = the w2 layer on h (it quantises h itself); y_t = T(sum_j w_j * yp_j), the slot sum in float64."""
    dt = x.dtype
    T, top_k = ids.shape
    acc = torch.zeros(T, roles["w2"][0].w.shape[0], dtype=torch.float64)
    for t in range(T):
        for j in range(top_k):
            e = int(ids[t, j])
            xt = x[t:t + 1]
            g, u = roles["w1"][e](xt).float(), roles["w3"][e](xt).float()
            h = (F.silu(g).to(dt).float() * u).to(dt)
            acc[t] += float(w[t, j]) * roles["w2"][e](h)[0].double()
    return acc.to(dt)


def _dense_roles(fmt, kind, E, K, I, gen):
    def codes(N, Kr):
        if fmt == "int8":
            return torch.randint(-127, 128, (N, Kr), generator=gen, dtype=torch.int8).numpy()
        return (torch.randn(N, Kr, generator=gen) * 60).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8).numpy()

    qmax = 448.0 if fmt == "fp8" else 127.0
    roles = {}
    s13 = [float(v) for v in (torch.rand(E, generator=gen) * 0.4 + 0.8) * 4.5 / qmax]
    s2 = [float(v) for v in (torch.rand(E, generator=gen) * 0.4 + 0.8) * 4.5 / qmax]
    for r, (N, Kr, si) in (("w1", (I, K, s13)), ("w3", (I, K, s13)), ("w2", (K, I, s2))):
        roles[r] = [_Dense(fmt, codes(N, Kr), ((torch.rand(N, generator=gen) + 0.5) / (60 * Kr ** 0.5)).numpy(),
                           si[e] if kind == "static" else None) for e in range(E)]
    return roles


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("fmt,kind", [("fp8", "dynamic"), ("fp8", "static"), ("int8", "dynamic"), ("int8", "static")])
def test_oracle_matches_module_loop(fmt, kind, dt):
    gen = torch.Generator().manual_seed(5)
    E, K, I = 5, 256, 128
    roles = _dense_roles(fmt, kind, E, K, I, gen)
    blk = moe.MoEExperts(roles["w1"], roles["w3"], roles["w2"], grouped=False)
    for T, top_k, routing in ((1, 1, "softmax"), (23, 3, "softmax"), (9, 2, "duplicate"), (17, 3, "sparse")):
        x = torch.randn(T, K, generator=gen).to(dt)
        ids, w = moe.route_topk(torch.randn(T, E, generator=gen), top_k)
        if routing == "duplicate":
            ids[:, 1] = ids[:, 0]
        elif routing == "sparse":
            ids[ids == 2] = 4
        ref = w8a8_block_oracle(x, ids, w, roles)
        got = blk(x, ids, w)
        assert got.dtype == dt and got.shape == (T, K)
        # the only difference is the order of the slot sum (fp32 in expert order against float64): one ulp of T
        assert_close_rel(got, ref, 2.0 ** -8 if dt == torch.float16 else 2.0 ** -6, f"cpu {fmt} {kind} T={T} {routing}")
        if top_k > 1 and routing == "softmax":
            with pytest.raises(AssertionError, match="outside"):
                assert_close_rel(got, w8a8_block_oracle(x, ids, w[:, [1, 0, 2]], roles), 2.0 ** -8, "swapped")


# ---- stack qualification ------------------------------------------------------------------------------------------------
def _mods(cls, E, N, K, kind="dynamic", ub=None, bias=False, s_in=0.01, seed=0):
    """CPU modules with the state post_init leaves (fp32 [N] scales, fp32 [1] input scale), marked ready: the stack
    builder only reads that state."""
    gen = torch.Generator().manual_seed(seed)
    out = []
    for e in range(E):
        w = torch.randint(-127, 128, (N, K), generator=gen, dtype=torch.int8)
        if cls is B200ChannelFp8Linear:
            w = w.to(torch.float8_e4m3fn)
        m = cls.from_checkpoint_tensors(w, torch.rand(N, 1, generator=gen) + 0.5,
                                        input_scale=torch.tensor([s_in]) if kind == "static" else None,
                                        bias=torch.zeros(N, dtype=torch.float16) if bias else None, activation=kind,
                                        ub=ub, device="cpu", post_init=False)
        m.weight_scale = channel_scales(m.weight_scale, N)
        if m.input_scale is not None:
            m.input_scale = m.input_scale.float().reshape(1)
        m._ready = True
        out.append(m)
    return out


def _sets(cls=B200ChannelInt8Linear, E=3, K=256, inter=128, **kw):
    return [_mods(cls, E, inter, K, seed=1, **kw), _mods(cls, E, inter, K, seed=2, **kw),
            _mods(cls, E, K, inter, seed=3, **kw)]


@pytest.mark.parametrize("cls", [B200ChannelFp8Linear, B200ChannelInt8Linear], ids=["fp8", "int8"])
@pytest.mark.parametrize("kind", ["dynamic", "static"])
def test_qualifying_stack_views(cls, kind):
    """A qualifying stack is stacked once per role; the modules keep views into it; MoEExperts keeps the loop."""
    sets = _sets(cls, kind=kind)
    blk = B200ChannelW8A8Experts(*sets, grouped=True)
    st = blk._stack
    assert st["int8"] == (cls is B200ChannelInt8Linear) and st["static"] == (kind == "static")
    for r, mods in zip(("w1", "w3", "w2"), sets):
        assert st[r]["weight"].shape == (3, mods[0].out_features, mods[0].in_features)
        assert st[r]["weight"].dtype == cls.CODE_DTYPE and st[r]["scale"].shape == (3, mods[0].out_features)
        assert (st[r]["s_in"] is not None) == (kind == "static")
        for e, m in enumerate(mods):
            assert m.weight.data_ptr() == st[r]["weight"][e].data_ptr()
            assert m.weight_scale.data_ptr() == st[r]["scale"][e].data_ptr()
            if kind == "static":
                assert float(st[r]["s_in"][e]) == float(m.input_scale)
    assert moe.MoEExperts(*_sets(cls, kind=kind))._stack is None
    with pytest.raises(ValueError, match="B200ChannelW8A8Experts"):
        moe.MoEExperts(*_sets(cls, kind=kind), grouped=True)


def _refused():
    cases = {}
    s = _sets()
    s[0][1] = _mods(B200ChannelFp8Linear, 1, 128, 256)[0]
    cases["all be B200ChannelFp8Linear or all B200ChannelInt8Linear"] = s
    s = _sets()
    s[2][0] = torch.nn.Linear(128, 256)
    cases["all be B200ChannelFp8Linear or all B200ChannelInt8Linear "] = s
    s = _sets()
    s[1][2]._ready = False
    cases["post_init"] = s
    s = _sets()
    s[2][1] = _mods(B200ChannelInt8Linear, 1, 256, 128, bias=True)[0]
    cases["bias"] = s
    s = _sets()
    s[0][0].adapter = object()
    cases["adapter"] = s
    s = _sets()
    s[2] = _mods(B200ChannelInt8Linear, 3, 256, 128, kind="static")
    cases["activation kind"] = s
    s = _sets(cls=B200ChannelFp8Linear, ub=2.0)
    s[1][0] = _mods(B200ChannelFp8Linear, 1, 128, 256, ub=3.0)[0]
    cases["ub"] = s
    s = _sets(kind="static")
    s[1][1] = _mods(B200ChannelInt8Linear, 1, 128, 256, kind="static", s_in=0.02)[0]
    cases["input_scale"] = s
    s = _sets()
    s[1][0] = _mods(B200ChannelInt8Linear, 1, 192, 256)[0]
    cases["w1 and w3"] = s
    s = _sets()
    s[2][2] = _mods(B200ChannelInt8Linear, 1, 128, 128)[0]
    cases["w2 must"] = s
    cases["at most 256 experts"] = [m * 86 for m in _sets()]  # 258 experts (the same modules repeated)
    return cases


@pytest.mark.parametrize("why", list(_refused()))
def test_refused_stack_rules(why):
    """Each disqualifying condition keeps the loop under grouped=None and raises a ValueError naming it under
    grouped=True."""
    sets = _refused()[why]
    assert B200ChannelW8A8Experts(*sets, fuse=False)._stack is None
    with pytest.raises(ValueError, match=re.escape(why.strip())):
        B200ChannelW8A8Experts(*sets, grouped=True)
