"""CPU model of the INDEX ARITHMETIC of the decode kernel v2 (gptqmodel_b200/csrc/b2q_decode2.cu).

The kernel cannot run without a GPU, but everything that is new in it relative to the GPU-validated v1 kernel is index
bookkeeping: which warp walks which (tile, k-quad) units, where it parks its partial sums in shared memory, how the
CTA / cluster reducers find them again, and how the shared-memory carve-up fits the size the host computes.  This file
restates those formulas (line by line from the kernel) and checks, for the launch plans the library's own planner
returns (`b2q_debug_decode_plan`), that
  * every (tile, quad) unit of the layer is processed exactly once,
  * every partial-sum slot the reducers read was written by exactly one warp, for the right (tile, token, feature),
  * every output element is emitted exactly once (by the CTA, or by exactly one rank of the cluster),
  * the shared-memory regions are disjoint and end inside the dynamic shared memory the host requests.
"""
import ctypes

import pytest

from gptqmodel_b200 import _lib as g

DEC_STAGES, QUAD = 4, 2048


def plan(M, K, N, ks=0, warps=0):
    out = (ctypes.c_int * 8)()
    rc = g.lib.b2q_debug_decode_plan(2, M, K, N, ks, warps, out)
    return None if rc != 0 else dict(zip(("C", "ks", "warps", "gw", "qpc", "max_tiles", "nst", "smem"), list(out)))


def smem_layout(p, M):
    """Byte offsets as computed by the kernel (ring | sx | xsum | wpart | cpart | bars | xbar)."""
    nw, nst, qpc, gw = p["warps"], p["nst"], p["qpc"], p["gw"]
    ngroups = nw // gw
    rows = ngroups * p["max_tiles"] * M
    off = {}
    off["ring"] = (0, nw * nst * QUAD)
    sx0 = off["ring"][1]
    off["sx"] = (sx0, sx0 + M * qpc * 128 * 2)
    xs0 = off["sx"][1]
    off["xsum"] = (xs0, xs0 + qpc * 2 * 8 * 4)
    wp0 = off["xsum"][1]
    off["wpart"] = (wp0, wp0 + rows * gw * 32 * 4)
    cp0 = off["wpart"][1]
    off["cpart"] = (cp0, cp0 + (rows * 32 * 4 if p["ks"] > 1 else 0))
    b0 = off["cpart"][1]
    off["bars"] = (b0, b0 + nw * DEC_STAGES * 8)
    off["xbar"] = (off["bars"][1], off["bars"][1] + 8)
    return off, rows


def simulate(M, K, N, p):
    TT, nquads = N // 32, K // 128
    C_cta, ks, nw, gw, qpc, max_tiles = p["C"], p["ks"], p["warps"], p["gw"], p["qpc"], p["max_tiles"]
    ngroups = nw // gw
    C = C_cta * ngroups
    off, rows = smem_layout(p, M)
    # --- shared memory: disjoint, 8/16-byte aligned where needed, inside what the host asks for
    prev_end = 0
    for name in ("ring", "sx", "xsum", "wpart", "cpart", "bars", "xbar"):
        a, b = off[name]
        assert a == prev_end and b >= a, (name, off)
        prev_end = b
    assert off["xbar"][1] <= p["smem"] <= 200 * 1024, (off, p)
    assert off["sx"][0] % 16 == 0 and off["bars"][0] % 8 == 0 and off["wpart"][0] % 4 == 0
    assert C_cta * ks <= 132

    units = {}    # (tile, quad) -> count
    emitted = {}  # (m, n) -> count
    for bx in range(C_cta):
        written = {}  # wpart float index -> (tile, m, feature, wg) per cluster rank
        for by in range(ks):
            q0 = by * qpc
            q1 = min(q0 + qpc, nquads)
            assert q1 > q0, "a cluster rank without k-quads"
            wslots = {}
            for warp in range(nw):
                grp, wg = divmod(warp, gw)
                tile0 = bx * ngroups + grp
                ntiles = (TT - tile0 + C - 1) // C if tile0 < TT else 0
                assert ntiles <= max_tiles
                nq = (q1 - q0 - wg + gw - 1) // gw if q0 + wg < q1 else 0
                for ti in range(ntiles):
                    tile = tile0 + ti * C
                    for qi in range(nq):
                        q = q0 + wg + qi * gw
                        assert q < q1
                        units[(tile, q)] = units.get((tile, q), 0) + 1
                        # activation-sum slot the main loop reads: (xs_a0 + qi * xs_qstep + kbl * 32) / 4 for t = 0
                        for kbl in range(2):
                            rd = (wg * 16) + qi * gw * 16 + kbl * 8
                            wr = ((wg + qi * gw) * 2 + kbl) * 8  # what the staging code writes for token 0
                            assert rd == wr and rd + 8 <= qpc * 2 * 8
                    # parking: wp = wpart + ((grp*max_tiles + ti) * M * gw + wg) * 32 ; + m*gw*32 + ((f + 8t) & 31)
                    for m in range(M):
                        t = m >> 1
                        for f in range(32):
                            idx = ((grp * max_tiles + ti) * M * gw + wg) * 32 + m * gw * 32 + ((f + 8 * t) & 31)
                            assert idx < rows * gw * 32
                            assert idx not in wslots, "two partial sums parked in the same slot"
                            wslots[idx] = (tile, m, f, wg)
            # CTA reducer: row = (g2 * max_tiles + ti) * M + m ; src = wpart + row*gw*32 + ((lane + 8*(m>>1)) & 31) + w*32
            cta_rows = {}
            for row in range(rows):
                m, r2 = row % M, row // M
                ti, g2 = r2 % max_tiles, r2 // max_tiles
                tile = bx * ngroups + g2 + ti * C
                if tile >= TT:
                    continue
                for lane in range(32):
                    for w in range(gw):
                        idx = row * gw * 32 + ((lane + 8 * (m >> 1)) & 31) + w * 32
                        assert wslots.get(idx) == (tile, m, lane, w), (idx, wslots.get(idx), (tile, m, lane, w))
                cta_rows[row] = (tile, m)
            written[by] = cta_rows
        # emission: ks == 1 -> the CTA itself; else rank r emits rows r*nw + warp, + ks*nw ...
        for by in range(ks):
            if ks == 1:
                mine = list(written[0])
            else:
                mine = [row for row in written[by] if (row // nw) % ks == by]
                # the kernel's loop: for (row = rank*nwarps + warp; row < rows; row += nrank*nwarps)
                loop = [row for warp in range(nw) for row in range(by * nw + warp, rows, ks * nw)]
                assert sorted(r for r in loop if r in written[by]) == sorted(mine)
            for row in mine:
                tile, m = written[by][row]
                for lane in range(32):
                    key = (m, tile * 32 + lane)
                    emitted[key] = emitted.get(key, 0) + 1
    assert len(units) == TT * nquads and set(units.values()) == {1}, "units missed or processed twice"
    assert len(emitted) == M * N and set(emitted.values()) == {1}, "outputs missed or written twice"


SHAPES = [(4096, 4096), (4096, 1024), (4096, 6144), (4096, 14336), (4096, 28672), (14336, 4096), (8192, 1280),
          (1792, 4096), (512, 4096), (128, 32), (256, 96), (1024, 32 * 149), (11008, 4096)]


@pytest.mark.parametrize("K,N", SHAPES)
def test_decode2_index_model(K, N):
    checked = 0
    big = N >= 14336  # keep the CPU suite short: the wide layers get the heuristic plan + two forced ones
    for M in ((1, 8) if big else (1, 2, 3, 5, 8)):
        for ks, warps in (((0, 0), (2, 16), (4, 8)) if big else ((0, 0), (1, 16), (2, 16), (4, 8), (8, 16), (2, 8))):
            p = plan(M, K, N, ks, warps)
            if p is None:
                continue
            simulate(M, K, N, p)
            checked += 1
    assert checked > 0


def test_decode2_index_model_forced_groups(monkeypatch):
    # B2Q_DECODE2_GW forces the warps-per-group split: exercise 1, 2, 4, 8-warp groups explicitly
    import gptqmodel_b200 as g
    for gw in (1, 2, 4, 8, 16):
        monkeypatch.setenv("B2Q_DECODE2_GW", str(gw))
        g.lib.b2q_debug_reload_env()  # the switches are read once at load, never on the call path
        for (K, N) in ((4096, 4096), (4096, 7168), (1024, 2048)):
            for M in (1, 4):
                for ks in (0, 2, 4):
                    p = plan(M, K, N, ks, 16)
                    if p is None:
                        continue
                    assert p["gw"] == gw
                    simulate(M, K, N, p)
    monkeypatch.delenv("B2Q_DECODE2_GW")
    g.lib.b2q_debug_reload_env()
