"""CPU: the float64 routing oracle against transformers' routers, the Python wrappers' argument checks and the C-ABI of
b2q_moe_route (include/b2q.h)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from gptqmodel_b200 import moe
from gptqmodel_b200._lib import SYMBOLS, lib
from oracle import moe_route_oracle as ro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "moe_route_cases.npz")


def _cases():
    z = np.load(GOLDEN)
    for name in z["names"]:
        yield str(name), {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(f"{name}/")}


def _oracle(c):
    logits = torch.from_numpy(c["logits"])
    k, norm, scale = int(c["top_k"]), bool(c["renormalize"]), float(c["scale"])
    if int(c["scoring"]) == 0:
        return ro.route_softmax(logits, k, norm, scale)[:2]
    return ro.route_grouped_sigmoid(logits, torch.from_numpy(c["bias"]), k, int(c["n_group"]), int(c["topk_group"]), norm,
                                    scale)[:2]


def test_golden_cases_cover_every_family():
    names = [n for n, _ in _cases()]
    assert len(names) == 5
    scorings = {(int(c["scoring"]), int(c["n_group"]), bool(c["renormalize"])) for _, c in _cases()}
    assert scorings == {(0, 1, True), (0, 1, False), (1, 8, True), (1, 1, True)}


@pytest.mark.parametrize("name", [n for n, _ in _cases()])
def test_oracle_reproduces_transformers(name):
    """Same id set per row as transformers' router; weights to 1e-6 relative (transformers computes them in fp32)."""
    c = dict(_cases())[name]
    ids, w = _oracle(c)
    order = ids.argsort(dim=-1)
    ids_s, w_s = ids.gather(1, order).numpy(), w.gather(1, order).numpy()
    np.testing.assert_array_equal(ids_s, c["ids"], err_msg=name)
    np.testing.assert_allclose(w_s, c["weights"].astype(np.float64), rtol=1e-6, atol=0, err_msg=name)


def test_oracle_tie_and_order_rules():
    """Ties toward the lower index for experts and groups; slots in descending score."""
    ids, _, _ = ro.route_softmax(torch.zeros(2, 8), 3)
    assert ids.tolist() == [[0, 1, 2]] * 2
    l = torch.tensor([[0.0, 2.0, 1.0, 2.0, 1.0, 0.5]])
    assert ro.route_softmax(l, 3)[0].tolist() == [[1, 3, 2]]
    # groups {0,1}, {2,3}, {4,5}: groups 0 and 2 tie on score, group 1 is lower; topk_group 1 keeps group 0
    bias = torch.tensor([0.5, 0.5, 0.0, 0.0, 0.5, 0.5])
    ids, _, masked, kept = ro.route_grouped_sigmoid(torch.zeros(1, 6), bias, 2, 3, 1)
    assert kept.tolist() == [[True, False, False]] and ids.tolist() == [[0, 1]]
    assert torch.isinf(masked[0, 2:]).all()


def test_oracle_masks_dropped_groups_where_transformers_fills_zero():
    """A kept group whose biased scores are all negative: -inf masking still selects inside it; a 0.0 fill would not."""
    logits = torch.zeros(1, 8)
    bias = torch.tensor([-0.9, -0.8, -2.0, -2.0, -2.0, -2.0, -2.0, -2.0])  # group 0 = {0..3} wins, c < 0 everywhere
    ids, _, masked, kept = ro.route_grouped_sigmoid(logits, bias, 2, 2, 1)
    assert kept.tolist() == [[True, False]]
    assert ids.tolist() == [[1, 0]]
    zero_fill = torch.where(torch.isinf(masked), torch.zeros_like(masked), masked)
    assert set(zero_fill.topk(2).indices[0].tolist()) <= {4, 5, 6, 7}


def test_wrappers_reject_bad_arguments():
    l = torch.randn(4, 64)
    b = torch.zeros(64)
    with pytest.raises(ValueError, match="CUDA"):
        moe.route_softmax_topk(l, 2)
    with pytest.raises(ValueError, match="CUDA"):
        moe.route_grouped_sigmoid(l, b, 8, 8, 4)
    with pytest.raises(ValueError, match="CUDA"):
        moe.route_softmax_topk(l.numpy(), 2)
    bad_softmax = [(torch.randn(4, 64, dtype=torch.float64), 2), (torch.randn(4, 64).int(), 2), (torch.randn(64), 2),
                   (torch.randn(64, 4).t(), 2), (torch.randn(4, 257), 2), (torch.randn(4, 0), 1), (l, 0), (l, 17),
                   (torch.randn(4, 8), 9)]
    for x, k in bad_softmax:
        with pytest.raises(ValueError, match="contiguous|need"):
            moe.route_softmax_topk(x, k)
    bad_grouped = [(b.double(), 8, 8, 4), (torch.zeros(60), 8, 8, 4), (torch.zeros(64, 1), 8, 8, 4),
                   (torch.zeros(128)[::2], 8, 8, 4), (b, 8, 7, 4), (b, 8, 64, 4), (b, 8, 8, 0), (b, 8, 8, 9),
                   (b, 9, 8, 1), (b, 17, 8, 4), (b, 0, 8, 4)]
    for bias, k, ng, tg in bad_grouped:
        with pytest.raises(ValueError, match="correction_bias|need"):
            moe.route_grouped_sigmoid(l, bias, k, ng, tg)
    with pytest.raises(ValueError, match="correction_bias"):
        moe.route_grouped_sigmoid(l, None, 8, 8, 4)


def _ctype(decl):
    decl = decl.strip()
    if "*" in decl:
        return ctypes.c_void_p
    return {"int": ctypes.c_int, "float": ctypes.c_float}[decl.rsplit(" ", 1)[0]]


def test_ctypes_signature_matches_header():
    hdr = open(os.path.join(ROOT, "include", "b2q.h")).read()
    m = re.search(r"\bint\s+b2q_moe_route\s*\(([^)]*)\)\s*;", hdr)
    assert m, "b2q_moe_route is not declared in include/b2q.h"
    params = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S).split(",")
    assert [_ctype(p) for p in params] == SYMBOLS["b2q_moe_route"][1]
    assert SYMBOLS["b2q_moe_route"][0] is ctypes.c_int


def test_abi_argument_checks_without_gpu():
    P = 1 << 20  # any non-NULL value: a refused call never dereferences it
    good = dict(x=P, dt=2, bias=None, T=4, E=64, k=8, sc=0, ng=1, tg=1, ids=P, w=P)

    def route(**kw):
        a = {**good, **kw}
        return lib.b2q_moe_route(a["x"], a["dt"], a["bias"], a["T"], a["E"], a["k"], a["sc"], a["ng"], a["tg"], 1, 1.0,
                                 a["ids"], a["w"], None)

    grouped = dict(sc=1, bias=P, ng=8, tg=4)
    bad = [dict(E=0), dict(E=257), dict(k=0), dict(k=17), dict(E=8, k=9), dict(dt=3), dict(dt=-1), dict(sc=2),
           dict(T=-1), dict(ng=2), dict(tg=2), dict(bias=P),
           {**grouped, "bias": None}, {**grouped, "ng": 7}, {**grouped, "ng": 64}, {**grouped, "tg": 0},
           {**grouped, "tg": 9}, {**grouped, "ng": 8, "tg": 1, "k": 9}, {**grouped, "ng": 0},
           dict(x=None), dict(ids=None), dict(w=None)]
    for kw in bad:
        assert route(**kw) == -2, kw
        assert lib.b2q_last_error()
    assert route(T=0) == 0 and route(T=0, x=None, ids=None, w=None) == 0  # no tokens: nothing to do
    assert route(T=0, **grouped) == 0 and route(T=0, sc=1, bias=P, ng=1, tg=1, E=160) == 0
