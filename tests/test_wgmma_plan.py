"""CPU: the launch plans of the swapped-operand wgmma tiers (small-batch, QQQ, block-FP8), as b2q_debug_wgmma_plan
returns them, against the planner formulas written out here.  The split-K plan fixes the fp32 summation order of the
small-batch and block-FP8 outputs, so a planner that moves for some shape changes their bits.  Without a device the
library plans for 132 SMs (H100 SXM)."""
import ctypes

import pytest

import gptqmodel_b200 as g

SMS = 132
# Llama / Qwen / DeepSeek layer shapes (K, N) of bench.py and the tools, plus short and odd K
SHAPES = [(4096, 4096), (4096, 1024), (4096, 6144), (4096, 12288), (4096, 28672), (14336, 4096), (4096, 11008),
          (11008, 4096), (5120, 5120), (5120, 27648), (13824, 5120), (8192, 8192), (8192, 57344), (28672, 8192),
          (7168, 4096), (7168, 2048), (2048, 7168), (7168, 24576), (1536, 24576), (18432, 7168), (2048, 1536),
          (768, 2048), (4096, 1536), (64, 4096), (192, 4096), (1088, 4096), (128, 128), (256, 64)]
MS = list(range(1, 301)) + [2048]


def ntok(M, lo, hi):
    # the narrowest wgmma n that holds M
    n = lo
    while n < M and n < hi:
        n *= 2
    return n


def doubling(ctas, nkb, min_kb):
    ks = 1
    while ks < 8 and ctas * ks * 2 <= SMS and nkb // (ks * 2) >= min_kb:
        ks *= 2
    return ks


def trim(ks, nkb):
    while ks > 1 and (ks - 1) * -(-nkb // ks) >= nkb:
        ks >>= 1
    return ks


def midm_ref(mode, M, K, N, active, ks):
    # small-batch tier: 128-feature tiles, 64-k blocks, >= 4 k-blocks per rank; B2Q_MIDM_KS clamped to 8 and trimmed
    tiles, nkb = -(-N // 128), K // 64
    nt = ntok(M, 16, 64 if mode == 1 else 128)
    if ks <= 0:
        ks = doubling(tiles * (1 if mode == 0 else max(active, 1)), nkb, 4)
    ks = trim(min(ks, 8), nkb)
    return [nt, ks, -(-nkb // ks), -(-M // nt)]


def qqq_ref(M, K, N):
    kb, tiles = -(-K // 128), -(-N // 128)
    nt = ntok(M, 8, 128)
    tb = -(-M // nt)
    ks = trim(doubling(tiles * tb, kb, 2), kb)
    return [nt, ks, -(-kb // ks), tb]


def fp8blk_ref(mode, M, K, N, active, ks):
    # block-FP8: grouped gate|up tiles pair 64 gate with 64 up features; a pinned ks is taken as given
    kb, tiles = K // 128, -(-N // (64 if mode == 1 else 128))
    nt = ntok(M, 8, 128)
    tb = -(-M // nt)
    if ks <= 0:
        ks = trim(doubling(tiles * (tb if mode == 0 else max(tb, max(active, 1))), kb, 2), kb)
    return [nt, ks, -(-kb // ks), tb]


def plan(tier, mode, M, K, N, active=0, ks=0):
    out = (ctypes.c_int * 4)()
    rc = g.lib.b2q_debug_wgmma_plan(tier, mode, M, K, N, active, ks, out)
    assert rc == 0, (tier, mode, M, K, N, active, ks, g.lib.b2q_last_error())
    return list(out)


def test_small_batch_plan():
    for K, N in SHAPES:
        for M in range(1, 129):
            for ks in range(0, 9):
                assert plan(0, 0, M, K, N, 0, ks) == midm_ref(0, M, K, N, 1, ks), (M, K, N, ks)


@pytest.mark.parametrize("mode", [1, 2])
def test_small_batch_grouped_plan(mode):
    for K, N in SHAPES:
        for rows in MS:
            for active in (0, 1, 2, 8, 32, 128):
                assert plan(0, mode, rows, K, N, active) == midm_ref(mode, rows, K, N, active, 0), (rows, K, N, active)
        for rows in (1, 17, 65, 300, 2048):
            for ks in range(1, 9):
                assert plan(0, mode, rows, K, N, 8, ks) == midm_ref(mode, rows, K, N, 8, ks), (rows, K, N, ks)


def test_qqq_plan():
    for K, N in SHAPES:
        if not ((K % 128 == 0 and N % 64 == 0) or (K % 64 == 0 and N % 128 == 0)):
            continue
        for M in MS:
            assert plan(1, 0, M, K, N) == qqq_ref(M, K, N), (M, K, N)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_fp8blk_plan(mode):
    for K, N in SHAPES:
        if K % 128 or N % 64:
            continue
        for M in MS:
            for active in ((0,) if mode == 0 else (0, 1, 8, 64, 256)):
                assert plan(2, mode, M, K, N, active) == fp8blk_ref(mode, M, K, N, active, 0), (M, K, N, active)
            for ks in range(1, 9):
                assert plan(2, mode, M, K, N, 8, ks) == fp8blk_ref(mode, M, K, N, 8, ks), (M, K, N, ks)


def test_token_boxes():
    # the tokens per CTA of each tier and mode at the box boundaries
    for M, want in ((1, 16), (16, 16), (17, 32), (33, 64), (64, 64), (65, 128), (128, 128)):
        assert plan(0, 0, M, 4096, 4096)[0] == want
    for rows, want1, want2 in ((16, 16, 16), (64, 64, 64), (65, 64, 128), (2048, 64, 128)):
        assert plan(0, 1, rows, 4096, 4096)[0] == want1 and plan(0, 2, rows, 4096, 4096)[0] == want2
    for tier in (1, 2):
        for M, want in ((1, 8), (8, 8), (9, 16), (100, 128), (2048, 128)):
            assert plan(tier, 0, M, 4096, 4096)[0] == want


def test_bad_arguments():
    out = (ctypes.c_int * 4)()
    for args in ((3, 0, 16, 4096, 4096, 0, 0), (0, 0, 129, 4096, 4096, 0, 0), (0, 3, 16, 4096, 4096, 0, 0),
                 (0, 0, 0, 4096, 4096, 0, 0), (0, 0, 16, 4000, 4096, 0, 0), (0, 0, 16, 4096, 4016, 0, 0),
                 (1, 1, 16, 4096, 4096, 0, 0), (1, 0, 16, 4096, 4096, 0, 2), (1, 0, 16, 4096, 4000, 0, 0),
                 (2, 0, 16, 4032, 4096, 0, 0), (2, 0, 16, 4096, 4064, 0, 0), (2, 0, 16, 4096, 4096, 0, 9),
                 (2, 1, 16, 4096, 4096, -1, 0), (2, 0, 16, 131072, 4096, 0, 0)):
        assert g.lib.b2q_debug_wgmma_plan(*args, out) == -2, args
    assert g.lib.b2q_debug_wgmma_plan(0, 0, 16, 4096, 4096, 0, 0, None) == -2
