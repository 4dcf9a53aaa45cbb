"""GPU microbenchmarks used while tuning (not the contract bench; see bench.py).

  python tools/microbench.py gemv     sweep split-K cluster size / warps per Llama-3-8B shape (M=1)
  python tools/microbench.py gemv2    same sweep for the experimental decode kernel v2 (+ warps per tile group), vs v1
  python tools/microbench.py gemm     time the wgmma GEMM at M=2048 per shape
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import gptqmodel_b200 as g  # noqa: E402
from gptqmodel_b200 import B200QuantLinear  # noqa: E402
from helpers import random_layer  # noqa: E402
from oracle import algorithmic_bytes  # noqa: E402

PEAKS = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(
    os.path.join(ROOT, "MEASURED_PEAKS.json")) else {"hbm_gbs": 6650.0, "bf16_tflops": 1590.0}
SHAPES = [(4096, 4096), (4096, 1024), (4096, 14336), (14336, 4096)]


def build(K, N, copies, bits=4, gs=128, sym=True):
    mods = []
    for c in range(copies):
        L = random_layer(K, N, bits=bits, group_size=gs, sym=sym, seed=c, device="cuda")
        mods.append(B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"],
                                                            bits, gs, device="cuda"))
    return mods


def time_graph(fn, iters=20):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        fn()
    for _ in range(3):
        gr.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        gr.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3  # us per graph


def gemv(MB=1):
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    for K, N in SHAPES:
        nbytes = K * N // 2
        copies = max(2, int(300e6 // nbytes) + 1)  # rotate > L2 (50 MB) of distinct weights
        if os.environ.get("MB_L2") == "1":
            copies = 1  # weights stay L2-resident: measures latency chain + L2 streaming
        mods = build(K, N, copies)
        x = (torch.randn(MB, K, device="cuda") * 0.5).to(torch.float16)
        out = torch.empty(MB, N, dtype=torch.float16, device="cuda")
        alg = algorithmic_bytes(K, N, 128, 4, MB)
        res = []
        for ks in (0, 1, 2, 4, 8):
            for warps in ((0,) if ks == 0 else (8, 16)):
                quads = K // 128
                if ks > 0 and ks > quads:
                    continue

                def fn():
                    st = torch.cuda.current_stream().cuda_stream
                    for m in (mods * (16 if len(mods) == 1 else 1)):
                        g.check(g.lib.b2q_decode(p(x), p(m.packed), p(m.scales.data), None, None, None, p(out), MB, K,
                                                 N, 4, 128, 0, ks, warps, st), "decode")
                try:
                    us = time_graph(fn) / (16 if copies == 1 else copies)
                except Exception as e:  # noqa: BLE001
                    print("fail", K, N, ks, warps, e)
                    continue
                res.append((us, ks, warps))
        res.sort()
        print(f"GEMV K={K} N={N} alg={alg/1e6:.2f}MB copies={copies}")
        for us, ks, warps in res[:6]:
            print(f"   ks={ks:2d} warps={warps} {us:7.2f} us  {alg/us/1e3:7.0f} GB/s  frac={alg/us/1e3/PEAKS['hbm_gbs']:.3f}")
        heur = [r for r in res if r[1] == 0]
        if heur:
            print(f"   heuristic: {heur[0][0]:.2f} us")
        del mods
        torch.cuda.empty_cache()


def gemv2(MB=1):
    """Sweep (split-K ranks, warps, warps per tile group) of the experimental decode kernel v2 per shape, against v1's
    heuristic and v2's own planner choice: calibrates decode2_config's cost model (b2q_decode2.cu)."""
    import ctypes
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    plan = (ctypes.c_int * 8)()
    for K, N in SHAPES + [(4096, 6144), (4096, 28672)]:  # + the fused q|k|v and gate|up widths
        nbytes = K * N // 2
        copies = max(2, int(300e6 // nbytes) + 1)
        mods = build(K, N, copies)
        x = (torch.randn(MB, K, device="cuda") * 0.5).to(torch.float16)
        out = torch.empty(MB, N, dtype=torch.float16, device="cuda")
        alg = algorithmic_bytes(K, N, 128, 4, MB)

        def run(ks, warps):
            def fn():
                st = torch.cuda.current_stream().cuda_stream
                for m in mods:
                    g.check(g.lib.b2q_decode(p(x), p(m.packed), p(m.scales.data), None, None, None, p(out), MB, K, N, 4,
                                             128, 0, ks, warps, st), "decode")
            return time_graph(fn) / copies

        os.environ.pop("B2Q_DECODE2_GW", None)
        os.environ["B2Q_DECODE_V2"] = "0"
        g.lib.b2q_debug_reload_env()
        v1 = run(0, 0)
        os.environ["B2Q_DECODE_V2"] = "1"
        g.lib.b2q_debug_reload_env()
        v2 = run(0, 0)
        g.lib.b2q_debug_decode_plan(2, MB, K, N, 0, 0, plan)
        print(f"DECODE2 K={K} N={N} M={MB} alg={alg/1e6:.2f}MB  v1 {v1:.2f} us | v2 planner {v2:.2f} us "
              f"(C={plan[0]} ks={plan[1]} warps={plan[2]} gw={plan[3]} tiles/group={plan[5]})  roofline "
              f"{alg / PEAKS['hbm_gbs'] / 1e3:.2f} us")
        res = []
        for ks in (1, 2, 4, 8):
            for warps in (8, 16):
                for gw in (16, 8, 4, 2):
                    if gw > warps or g.lib.b2q_debug_decode_plan(2, MB, K, N, ks, warps, plan) != 0:
                        continue
                    os.environ["B2Q_DECODE2_GW"] = str(gw)
                    g.lib.b2q_debug_reload_env()
                    if g.lib.b2q_debug_decode_plan(2, MB, K, N, ks, warps, plan) != 0:
                        continue
                    try:
                        res.append((run(ks, warps), ks, warps, gw, plan[5]))
                    except Exception as e:  # noqa: BLE001
                        print("   fail", ks, warps, gw, e)
        os.environ.pop("B2Q_DECODE2_GW", None)
        g.lib.b2q_debug_reload_env()
        res.sort()
        for us, ks, warps, gw, mt in res[:5]:
            print(f"   ks={ks} warps={warps:2d} gw={gw:2d} tiles/group={mt:2d}  {us:7.2f} us  frac={alg/us/1e3/PEAKS['hbm_gbs']:.3f}")
        del mods
        torch.cuda.empty_cache()
    os.environ.pop("B2Q_DECODE_V2", None)
    g.lib.b2q_debug_reload_env()


def gemm(Ms=(2048,)):
    for K, N in SHAPES:
        mods = build(K, N, 2)
        for M in Ms:
            x = (torch.randn(M, K, device="cuda") * 0.5).to(torch.float16)

            def fn():
                for m in mods:
                    m(x)
            us = time_graph(fn, iters=10) / len(mods)
            fl = 2.0 * M * K * N
            print(f"GEMM M={M} K={K} N={N}: {us:8.1f} us  {fl/us/1e6:7.1f} TFLOP/s  frac={fl/us/1e6/PEAKS['bf16_tflops']:.3f}")
        W = torch.randn(K, N, device="cuda", dtype=torch.float16)
        x = (torch.randn(Ms[-1], K, device="cuda") * 0.5).to(torch.float16)
        us = time_graph(lambda: torch.matmul(x, W), iters=10)
        print(f"   cuBLAS fp16 dense M={Ms[-1]}: {us:8.1f} us  {2.0*Ms[-1]*K*N/us/1e6:7.1f} TFLOP/s")
        del mods
        torch.cuda.empty_cache()


def midm(Ms=(9, 16, 32, 64, 128)):
    """Small-batch tier (b2q_midm.cu) per Llama-3-8B shape with weights rotated > L2: heuristic split-K vs forced cluster
    sizes vs the round-1 paths (padded single-CTA tier; decode row blocks for M <= 16), + 8-bit and group_size 32."""
    def setenv(**kw):
        for k in ("B2Q_MIDM", "B2Q_MIDM_KS", "B2Q_DECODE_BLOCKS_M"):
            os.environ.pop(k, None)
        os.environ.update({k: str(v) for k, v in kw.items()})
        g.lib.b2q_debug_reload_env()

    for bits, gs in ((4, 128), (4, 32), (8, 128)):
        for K, N in SHAPES:
            nbytes = K * N * bits // 8
            copies = max(2, int(300e6 // nbytes) + 1)
            mods = build(K, N, copies, bits=bits, gs=gs)
            for M in ((1,) if (bits, gs) == (4, 32) else ()) + tuple(Ms) + ((2,) if bits == 8 else ()):
                x = (torch.randn(M, K, device="cuda") * 0.5).to(torch.float16)
                alg = algorithmic_bytes(K, N, gs, bits, M)

                def fn():
                    for m in mods:
                        m(x)
                row = {}
                variants = [("midm", {})] + [(f"ks{k}", {"B2Q_MIDM_KS": k}) for k in (1, 2, 4, 8)]
                if (bits, gs) == (4, 128):
                    variants.append(("padded_r1", {"B2Q_MIDM": 0}))
                    if M <= 16:
                        variants.append(("decode_x2_r1", {"B2Q_DECODE_BLOCKS_M": 16}))
                for name, envs in variants:
                    setenv(**envs)
                    try:
                        row[name] = time_graph(fn, iters=10) / copies
                    except Exception as e:  # noqa: BLE001
                        row[name] = float("nan")
                        print("   fail", name, e)
                setenv()
                best = row["midm"]
                print(f"MIDM bits={bits} g={gs} K={K} N={N} M={M}: " + "  ".join(f"{k} {v:6.2f}us" for k, v in row.items())
                      + f"  | heuristic {alg / best / 1e3:6.0f} GB/s frac={alg / best / 1e3 / PEAKS['hbm_gbs']:.3f}", flush=True)
            del mods
            torch.cuda.empty_cache()


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "gemv"
    if what == "gemv":
        gemv(int(sys.argv[2]) if len(sys.argv) > 2 else 1)
    elif what == "gemv2":
        gemv2(int(sys.argv[2]) if len(sys.argv) > 2 else 1)
    elif what == "midm":
        midm(tuple(int(a) for a in sys.argv[2:]) or (9, 16, 32, 64, 128))
    elif what == "gemm":
        gemm(tuple(int(a) for a in sys.argv[2:]) or (2048,))
