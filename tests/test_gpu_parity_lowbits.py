"""GPU parity of the widened layouts (2 / 3-bit, planar 3 / 5 / 6 / 7-bit), arbitrary g_idx and act-order row shards
(VERDICT r01 items 9 / 10).  Outputs are compared with (a) what the UNMODIFIED reference produced for
the same checkpoint tensors (tests/golden/lowbit_cases.npz) and (b) the oracle on larger layers at every kernel tier."""
import json
import os

import numpy as np
import pytest
import torch

import oracle
from gptqmodel_b200 import B200QuantLinear, layouts, tp
from gptqmodel_b200.pack import pack_gptq
from helpers import assert_close_rel, make_layer, ref_rounding_slack

_D = np.load(os.path.join(os.path.dirname(__file__), "golden", "lowbit_cases.npz"))
META = json.loads(bytes(_D["__meta__"]).decode())


def _t(name, key):
    return torch.from_numpy(_D[f"{name}.{key}"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(META))
def test_lowbit_module_matches_reference_outputs(name):
    m = META[name]
    qw, qz, sc, gi, W = (_t(name, k) for k in ("qweight", "qzeros", "scales", "g_idx", "W"))
    bias = _t(name, "bias") if m["bias"] else None
    mod = B200QuantLinear.from_checkpoint_tensors(qw, qz, sc, gi, m["bits"], m["group_size"], bias=bias,
                                                  desc_act=m["desc_act"], sym=m["sym"],
                                                  format="gptq_p" if m["planar"] else "gptq_v2")
    assert mod.kbits == (4 if m["bits"] <= 4 else 8) and mod.planar == m["planar"]
    x = _t(name, "x")
    y = mod(x.cuda())
    slack = ref_rounding_slack(W, x)  # M <= 8: decode / GEMV tiers apply the scale once per group (helpers.py)
    assert_close_rel(y, oracle.forward_any(x, qw, qz, sc, gi, m["bits"], m["planar"], bias=bias), 1e-3, name, slack=slack)
    # the reference's own CPU output (fp16-accumulating matmul: ~1 ulp, same bound as test_reference_generated_cases)
    assert torch.allclose(y.float().cpu(), _t(name, "y_fp16").float(), rtol=2e-3, atol=2e-3), name
    ybf = mod(x.cuda().to(torch.bfloat16))
    assert_close_rel(ybf, _t(name, "y_bf16"), 1.6e-2, name + " bf16")
    # dense weight through the exact-operand tensor-core tier: bit-identical to the reference's dequantize_weight()
    assert torch.equal(mod.dequantize_weight().cpu(), W), name


def _grid_layer(K, N, bits, gs, sym, planar, desc_act, seed):
    g = torch.Generator().manual_seed(seed)
    Wf = torch.randn(N, K, generator=g) * 0.5
    if desc_act:
        _, g_idx = oracle.make_act_order(K, gs, seed=seed)
    else:
        g_idx = torch.arange(K, dtype=torch.int32) // gs
    sc, ze = (oracle.quantize_sym if sym else oracle.quantize_asym)(Wf, bits, gs, g_idx)[:2]
    return pack_gptq(Wf, sc, ze, g_idx, bits, planar=planar)


@pytest.mark.gpu
@pytest.mark.parametrize("bits,planar,gs,sym,desc_act", [
    (2, False, 128, False, False), (3, False, 128, True, True), (3, True, 64, False, False),
    (5, True, 128, False, False), (6, True, 32, True, False), (7, True, 128, False, True)])
def test_lowbit_layers_at_every_tier(bits, planar, gs, sym, desc_act):
    K, N = 1024, 768
    L = _grid_layer(K, N, bits, gs, sym, planar, desc_act, seed=bits * 10 + gs)
    mod = B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], bits, gs,
                                                  desc_act=desc_act, sym=sym, format="gptq_p" if planar else "gptq_v2")
    W = oracle.dequantize_weight_any(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], bits, planar)
    gen = torch.Generator().manual_seed(bits)
    for M in (1, 5, 16, 100, 300):  # decode / GEMV, small-batch wgmma, prefill tiers
        x = (torch.randn(M, K, generator=gen) * 0.5).to(torch.float16)
        ref = oracle.forward_any(x, L["qweight"], L["qzeros"], L["scales"], L["g_idx"], bits, planar)
        assert_close_rel(mod(x.cuda()), ref, 1e-3, f"{bits}-bit planar={planar} g{gs} M={M}",
                         slack=ref_rounding_slack(W, x) if M <= 8 else None)


@pytest.mark.gpu
@pytest.mark.parametrize("bits,K,N,G", [(4, 1024, 512, 9), (8, 512, 256, 5), (3, 1024, 256, 12)])
def test_arbitrary_g_idx_on_gpu(bits, K, N, G):
    """Groups of unequal (and zero) size: rows sorted and padded per group by layouts.regroup, x gathered by forward()."""
    g = torch.Generator().manual_seed(K + G + bits)
    g_idx = torch.randint(0, G, (K,), generator=g, dtype=torch.int32)
    g_idx[g_idx == 2] = 0
    q = torch.randint(0, 1 << bits, (K, N), generator=g, dtype=torch.int32)
    z = torch.randint(0, 1 << bits, (G, N), generator=g, dtype=torch.int32)
    sc = (torch.rand(G, N, generator=g) * 0.02 + 0.005).to(torch.float16)
    qw, qz = layouts.pack_rows(q, bits), layouts.pack_cols(z, bits)
    mod = B200QuantLinear(bits=bits, group_size=128, desc_act=True, sym=False, in_features=K, out_features=N,
                          register_buffers=False)
    mk = lambda t: torch.nn.Parameter(t.cuda(), requires_grad=False)  # noqa: E731
    mod.qweight, mod.qzeros, mod.scales, mod.g_idx = mk(qw), mk(qz), mk(sc), mk(g_idx)
    mod.post_init()
    assert mod._gather is not None and mod._kK % 128 == 0 and mod._kgs in (32, 64, 128)
    W = oracle.dequantize_weight_any(qw, qz, sc, g_idx, bits)
    for M in (1, 4, 32, 200):
        x = (torch.randn(M, K, generator=g) * 0.5).to(torch.float16)
        ref = oracle.forward_any(x, qw, qz, sc, g_idx, bits)
        assert_close_rel(mod(x.cuda()), ref, 1e-3, f"ragged g_idx {bits}-bit M={M}",
                         slack=ref_rounding_slack(W, x) if M <= 8 else None)
    assert torch.equal(mod.dequantize_weight().cpu(), W)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 8])
def test_act_order_row_shards_on_gpu(world):
    """o_proj / down_proj of an act-order checkpoint, row-parallel: every rank's K-slice keeps the full scale tables
    (utils/marlin.py:300-305); the partial outputs of the shards sum to the unsharded layer's output."""
    K, N = 4096, 1024
    L = make_layer(K, N, group_size=128, desc_act=True, sym=False, seed=31)
    full = B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, 128, desc_act=True)
    shards = []
    for r in range(world):
        sh = tp.shard_rows(L, r, world)
        shards.append(B200QuantLinear.from_checkpoint_tensors(sh["qweight"], sh["qzeros"], sh["scales"], sh["g_idx"], 4, 128,
                                                              desc_act=True))
        assert shards[-1]._gather is not None
    g = torch.Generator().manual_seed(3)
    W = oracle.dequantize_weight(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4)
    for M in (1, 16, 300):
        x = (torch.randn(M, K, generator=g) * 0.5).to(torch.float16)
        xc = x.cuda()
        acc = torch.zeros(M, N, dtype=torch.float32, device="cuda")
        for r, s in enumerate(shards):
            acc += s(xc[:, r * K // world:(r + 1) * K // world].contiguous()).float()
        ref = oracle.forward(x, L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4)
        # P partial sums, each rounded to fp16 once: tolerance as in tests/test_tp_gpu.py
        assert_close_rel(acc, ref, 1e-3 * (1 + world ** 0.5 / 2), f"act-order row shards world={world} M={M}",
                         slack=ref_rounding_slack(W, x) if M <= 8 else None)
        assert_close_rel(full(xc), ref, 1e-3, f"unsharded M={M}", slack=ref_rounding_slack(W, x) if M <= 8 else None)
