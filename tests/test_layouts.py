"""2 / 3-bit continuous and planar 3 / 5 / 6 / 7-bit checkpoint layouts, exact widening, arbitrary g_idx (CPU).

Pinned against tensors packed, dequantised and multiplied by the UNMODIFIED reference (tests/golden/lowbit_cases.npz,
generator tests/golden/make_golden_lowbits.py): gptqmodel/nn_modules/qlinear/__init__.py:946-1003,
utils/planar_packing.py.  The oracle (numpy bit matrices) and the product (torch field tables) are independent
restatements; both must reproduce the reference bit for bit.
"""
import json
import os

import numpy as np
import pytest
import torch
from hypothesis import given, settings
from hypothesis import strategies as st

import oracle
from gptqmodel_b200 import layouts, tp
from gptqmodel_b200.pack import pack_gptq

GOLD = os.path.join(os.path.dirname(__file__), "golden", "lowbit_cases.npz")
_D = np.load(GOLD)
META = json.loads(bytes(_D["__meta__"]).decode())


def _t(name, key):
    return torch.from_numpy(_D[f"{name}.{key}"])


@pytest.mark.parametrize("name", sorted(META))
def test_unpack_matches_reference_bit_exact(name):
    m = META[name]
    qw, qz, sc, gi, W = (_t(name, k) for k in ("qweight", "qzeros", "scales", "g_idx", "W"))
    # oracle: dequantised weight identical to the reference's dequantize_weight()
    assert torch.equal(oracle.dequantize_weight_any(qw, qz, sc, gi, m["bits"], m["planar"]), W)
    # product field tables == oracle bit matrices, and packing is the exact inverse
    q = layouts.unpack_rows(qw, m["bits"], m["planar"])
    z = layouts.unpack_cols(qz, m["bits"], m["planar"])
    assert torch.equal(q, oracle.unpack_rows_any(qw, m["bits"], m["planar"]).int())
    assert torch.equal(z, oracle.unpack_cols_any(qz, m["bits"], m["planar"]).int())
    assert int(q.max()) < (1 << m["bits"]) and int(q.min()) >= 0
    assert torch.equal(layouts.pack_rows(q, m["bits"], m["planar"]), qw)
    assert torch.equal(layouts.pack_cols(z, m["bits"], m["planar"]), qz)


@pytest.mark.parametrize("name", sorted(META))
def test_packer_matches_reference_bit_exact(name):
    m = META[name]
    planar_fmt = m["planar"]
    out = pack_gptq(_t(name, "weight"), _t(name, "in_scales"), _t(name, "in_zeros"), _t(name, "g_idx"), m["bits"],
                    planar=planar_fmt)
    assert torch.equal(out["qweight"], _t(name, "qweight"))
    assert torch.equal(out["qzeros"], _t(name, "qzeros"))
    assert torch.equal(out["scales"], _t(name, "scales"))


@pytest.mark.parametrize("name", sorted(META))
def test_widening_is_exact(name):
    """The 4- / 8-bit container holds the same integers: the 4 / 8-bit oracle on the widened tensors reproduces the
    reference's dequantised weight and forward bit for bit."""
    m = META[name]
    qw, qz, sc, gi = (_t(name, k) for k in ("qweight", "qzeros", "scales", "g_idx"))
    wq, wz, kb = layouts.widen(qw, qz, m["bits"], m["planar"])
    assert kb == (4 if m["bits"] <= 4 else 8)
    assert wq.shape == (m["K"] * kb // 32, m["N"]) and wz.shape == (sc.shape[0], m["N"] * kb // 32)
    assert torch.equal(oracle.dequantize_weight(wq, wz, sc, gi, kb), _t(name, "W"))
    x = _t(name, "x")
    bias = _t(name, "bias") if m["bias"] else None
    y = oracle.forward(x, wq, wz, sc, gi, kb, bias=bias)
    ref = _t(name, "y_fp16")
    assert (y.float() - ref.float()).abs().max().item() <= 2e-3 * max(1.0, ref.float().abs().max().item())
    assert torch.equal(oracle.forward_any(x, qw, qz, sc, gi, m["bits"], m["planar"], bias=bias), y)


@settings(max_examples=40, deadline=None)
@given(bits=st.sampled_from([2, 3, 4, 5, 6, 7, 8]), planar=st.booleans(), blocks=st.integers(1, 3),
       cols=st.integers(1, 5), seed=st.integers(0, 2 ** 16))
def test_pack_unpack_round_trip(bits, planar, blocks, cols, seed):
    planar = planar or bits in layouts.PLANAR_ONLY_BITS
    g = torch.Generator().manual_seed(seed)
    codes = torch.randint(0, 1 << bits, (32 * blocks, cols), generator=g, dtype=torch.int32)
    words = layouts.pack_rows(codes, bits, planar)
    assert words.shape == (32 * blocks * bits // 32, cols) and words.dtype == torch.int32
    assert torch.equal(layouts.unpack_rows(words, bits, planar), codes)
    assert torch.equal(oracle.unpack_rows_any(words, bits, planar).int(), codes)
    if bits in (2, 4, 8):  # planar words of a single plane are the continuous words (utils/planar_packing.py:10-16)
        assert torch.equal(layouts.pack_rows(codes, bits, True), layouts.pack_rows(codes, bits, False))
    zc = codes.t().contiguous()
    assert torch.equal(layouts.unpack_cols(layouts.pack_cols(zc, bits, planar), bits, planar), zc)


@pytest.mark.parametrize("bits,planar", [(2, False), (3, False), (3, True), (4, False), (5, True), (7, True), (8, False)])
def test_zero_point_v1_v2_shift(bits, planar):
    g = torch.Generator().manual_seed(bits)
    z = torch.randint(0, 1 << bits, (3, 64), generator=g, dtype=torch.int32)
    v2 = layouts.pack_cols(z, bits, planar)
    v1 = layouts.shift_zero_points(v2, bits, planar, -1)
    assert torch.equal(layouts.unpack_cols(v1, bits, planar), (z - 1) & ((1 << bits) - 1))
    assert torch.equal(layouts.shift_zero_points(v1, bits, planar, +1), v2)
    assert torch.equal(oracle.shift_zero_points_any(v1, bits, planar, +1).int(), z)
    if bits in (2, 4, 8):  # without a wrapping field the reference adds a packed constant (utils/model.py:759-830)
        zz = z.clamp(min=1)
        v2 = layouts.pack_cols(zz, bits, planar)
        v1 = layouts.shift_zero_points(v2, bits, planar, -1)
        assert torch.equal(oracle.convert_v1_to_v2(v1, bits), v2)


def _ragged_layer(K, N, G, bits, seed):
    """A layer whose g_idx gives every group a different (possibly zero) number of rows."""
    g = torch.Generator().manual_seed(seed)
    g_idx = torch.randint(0, G, (K,), generator=g, dtype=torch.int32)
    g_idx[g_idx == 1] = 0  # group 1 stays empty
    q = torch.randint(0, 1 << bits, (K, N), generator=g, dtype=torch.int32)
    z = torch.randint(0, 1 << bits, (G, N), generator=g, dtype=torch.int32)
    s = (torch.rand(G, N, generator=g) * 0.02 + 0.005).to(torch.float16)
    return q, z, s, g_idx


@pytest.mark.parametrize("bits,K,N,G", [(4, 256, 64, 5), (8, 128, 32, 3), (4, 512, 32, 16)])
def test_regroup_arbitrary_g_idx_is_exact(bits, K, N, G):
    q, z, s, g_idx = _ragged_layer(K, N, G, bits, seed=K + G)
    r = layouts.regroup(q, z, s, g_idx)
    Kp, gran = r["gather"].numel(), r["granule"]
    assert Kp % 128 == 0 and gran in (32, 64, 128) and r["q"].shape == (Kp, N) and r["z"].shape == (Kp // gran, N)
    # dense weights: the regrouped layer (uniform groups of `gran` rows) against the original walked through g_idx
    W0 = (s[g_idx.long()].float() * (q - z[g_idx.long()]).float())                     # [K, N]
    gi2 = torch.arange(Kp) // gran
    W1 = (r["scales"][gi2].float() * (r["q"] - r["z"][gi2]).float())                   # [K', N]
    real = torch.zeros(Kp, dtype=torch.bool)
    # every input feature appears exactly once among the non-padding rows, with its own weight row
    nz = (r["q"] != r["z"][gi2]).any(dim=1)
    x = torch.randn(4, K, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    y0 = x @ W0.double()
    y1 = x[:, r["gather"]] @ W1.double()
    assert torch.equal(y0, y1) or (y0 - y1).abs().max().item() < 1e-9
    counts = torch.bincount(r["gather"][nz], minlength=K)
    assert int(counts.max()) <= 1
    # through the packed form the kernels read (and the 4 / 8-bit oracle)
    qw, qz = layouts.pack_rows(r["q"], bits), layouts.pack_cols(r["z"], bits)
    Wk = oracle.dequantize_weight(qw, qz, r["scales"], gi2.int(), bits)
    assert torch.equal(Wk.float(), W1.to(torch.float16).float()) or torch.allclose(Wk.float(), W1, rtol=1e-3, atol=0)
    del real


def test_act_order_row_shards_sum_to_the_full_layer():
    """tp.shard_rows on an act-order layer: K-slice + replicated tables; regrouped shards reproduce the layer."""
    from helpers import make_layer

    L = make_layer(512, 64, group_size=128, desc_act=True, sym=False, seed=9)
    x = (torch.randn(3, 512, generator=torch.Generator().manual_seed(2)) * 0.5).to(torch.float16)
    full = oracle.forward(x, L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4).double()
    for world in (2, 4):
        acc = torch.zeros_like(full)
        for r in range(world):
            sh = tp.shard_rows(L, r, world)
            assert sh["replicated_tables"] and sh["qweight"].shape == (512 // world * 4 // 32, 64)
            k0, k1 = r * 512 // world, (r + 1) * 512 // world
            rg = layouts.regroup(layouts.unpack_rows(sh["qweight"], 4), layouts.unpack_cols(sh["qzeros"], 4),
                                 sh["scales"], sh["g_idx"])
            gi2 = (torch.arange(rg["gather"].numel()) // rg["granule"]).int()
            W = oracle.dequantize_weight(layouts.pack_rows(rg["q"], 4), layouts.pack_cols(rg["z"], 4), rg["scales"], gi2, 4)
            acc += x[:, k0:k1][:, rg["gather"]].double() @ W.double()
        assert (acc - full).abs().max().item() <= 2e-3 * full.abs().max().item()


@settings(max_examples=30, deadline=None)
@given(kblocks=st.integers(1, 8), G=st.integers(1, 9), N=st.sampled_from([8, 32]), bits=st.sampled_from([4, 8]),
       seed=st.integers(0, 2 ** 16))
def test_regroup_property(kblocks, G, N, bits, seed):
    """Any assignment of rows to groups (empty groups, one giant group, ...) regroups to an exactly equivalent layer."""
    K = 32 * kblocks
    g = torch.Generator().manual_seed(seed)
    g_idx = torch.randint(0, G, (K,), generator=g, dtype=torch.int32)
    q = torch.randint(0, 1 << bits, (K, N), generator=g, dtype=torch.int32)
    z = torch.randint(0, 1 << bits, (G, N), generator=g, dtype=torch.int32)
    s = (torch.rand(G, N, generator=g) * 0.02 + 0.005).to(torch.float16)
    r = layouts.regroup(q, z, s, g_idx)
    Kp, gran = r["gather"].numel(), r["granule"]
    assert Kp % 128 == 0 and Kp >= K and gran in (32, 64, 128) and Kp % gran == 0
    assert r["q"].shape == (Kp, N) and r["z"].shape == (Kp // gran, N) and r["scales"].shape == (Kp // gran, N)
    gi2 = torch.arange(Kp) // gran
    W0 = s[g_idx.long()].double() * (q - z[g_idx.long()]).double()
    W1 = r["scales"][gi2].double() * (r["q"] - r["z"][gi2]).double()
    x = torch.randn(2, K, generator=g, dtype=torch.float64)
    assert torch.allclose(x @ W0, x[:, r["gather"]] @ W1, rtol=0, atol=1e-9)
    # every feature is placed exactly once; all other rows are exact zeros
    real = torch.zeros(Kp, dtype=torch.bool)
    nz_rows = (W1 != 0).any(dim=1)
    placed = torch.bincount(r["gather"][nz_rows], minlength=K)
    assert int(placed.max()) <= 1
    del real


def test_loader_round_trip_of_a_regrouped_act_order_row_shard(tmp_path):
    """A K-slice of an act-order layer written to a checkpoint (replicated tables) loads as a module whose tensors keep the
    reference's shapes for that slice; post_init (GPU) is what regroups it."""
    from helpers import make_layer

    L = make_layer(512, 64, group_size=128, desc_act=True, sym=False, seed=4)
    sh = tp.shard_rows(L, 1, 4)
    assert sh["qweight"].shape == (128 * 4 // 32, 64) and sh["scales"].shape == L["scales"].shape
    assert int(sh["g_idx"].max()) < L["scales"].shape[0] and sh["K"] == 128
    # the slice's dense weight equals the corresponding rows of the full layer's
    Wf = oracle.dequantize_weight(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4)
    Ws = oracle.dequantize_weight(sh["qweight"], sh["qzeros"], sh["scales"], sh["g_idx"], 4)
    assert torch.equal(Ws, Wf[128:256])
