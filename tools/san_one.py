"""Small-shape exercise of the decode, small-batch and prefill tiers (target for compute-sanitizer; also a quick parity
check).

    B2Q_DECODE_V2=1 compute-sanitizer --tool memcheck python tools/san_one.py
    ... --tool racecheck / --tool synccheck

Covers: decode v2 (sym / asym g64 / act-order, M = 1, 5, 8, single set and fused siblings, forced warp groups), the
small-batch tier's cluster split-K (M = 40, 128), and the prefill tier (M = 300: partial token and feature tiles) for single
layers and fused siblings.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import gptqmodel_b200 as _g  # noqa: E402
from gptqmodel_b200 import B200QuantLinear, fuse_siblings  # noqa: E402
from helpers import assert_close_rel, make_layer, oracle_forward  # noqa: E402


def mod(L):
    return B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], L["bits"],
                                                   L["group_size"], bias=L["bias"], desc_act=L["desc_act"], sym=L["sym"])


def check(m, L, M, what, rel=1e-3):
    x = (torch.randn(M, L["K"], generator=torch.Generator().manual_seed(M)) * 0.5).to(torch.float16)
    y = m(x.cuda())
    torch.cuda.synchronize()
    assert_close_rel(y, oracle_forward(L, x), rel, what)
    print("ok", what, flush=True)


layers = [make_layer(1024, 512, group_size=128, sym=True, seed=1),
          make_layer(1024, 256, group_size=64, sym=False, bias=True, seed=2),
          make_layer(512, 768, group_size=64, sym=False, desc_act=True, seed=3),
          make_layer(2048, 96, group_size=-1, sym=True, seed=4)]
for L in layers:
    m = mod(L)
    for M in (1, 5, 8):
        for gw in ("", "4", "16"):
            if gw:
                os.environ["B2Q_DECODE2_GW"] = gw
            else:
                os.environ.pop("B2Q_DECODE2_GW", None)
            _g.lib.b2q_debug_reload_env()
            check(m, L, M, f"decode K={L['K']} N={L['N']} g={L['group_size']} sym={L['sym']} act={L['desc_act']} M={M} gw={gw or 'auto'}")
    os.environ.pop("B2Q_DECODE2_GW", None)
    _g.lib.b2q_debug_reload_env()
    for M in (40, 128, 300):
        check(m, L, M, f"gemm K={L['K']} N={L['N']} M={M}")
# fused siblings through the multi-set path
Ls = [make_layer(1024, n, group_size=128, sym=True, seed=10 + i) for i, n in enumerate((512, 128, 256))]
ms = [mod(L) for L in Ls]
assert fuse_siblings(ms)
for M in (1, 6):
    x = (torch.randn(M, 1024, generator=torch.Generator().manual_seed(M)) * 0.5).to(torch.float16)
    for m, L in zip(ms, Ls):
        assert_close_rel(m(x.cuda()), oracle_forward(L, x), 1e-3, f"fused M={M}")
    print("ok fused siblings M =", M, flush=True)
# sibling-fused PREFILL launch (b2q_gemm_multi), incl. act-order siblings that share one gather of x
for desc in (False, True):
    Ls = [make_layer(512, n, group_size=64, sym=False, desc_act=desc, bias=True, seed=33) for n in (512, 96, 288)]
    ms = [mod(L) for L in Ls]
    assert fuse_siblings(ms)
    x = (torch.randn(300, 512, generator=torch.Generator().manual_seed(9)) * 0.5).to(torch.float16)
    for m, L in zip(ms, Ls):
        assert_close_rel(m(x.cuda()), oracle_forward(L, x), 1e-3, f"fused prefill act-order={desc}")
    print("ok fused prefill siblings, act-order =", desc, flush=True)
print("all ok")
