"""Per-launch cost of the 4-bit decode tier at batch 1: streaming slope and fixed intercept.

    python tools/decode_launch_cost.py [--out FILE.json] [--min-mb 640] [--iters 20]

For each shape (K, N) it builds enough DISTINCT layers to stream at least --min-mb of weights + scales (far more than
the 50 MB L2), captures one M = 1 forward of every layer in a CUDA graph (one b2q_mm launch per layer, consecutive
launches chained by programmatic dependent launch as in a decode step) and times replays with CUDA events.  A straight
line  t = intercept + bytes / slope  through the per-launch times of each K gives the streaming rate (TB/s) and the
fixed cost of a launch boundary (µs).  The fused q|k|v and gate|up launches of Llama-3-8B are timed the same way.
It also reports, for each dense decode kernel at the bench's launch shapes, how many CTAs the driver keeps resident per
SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor), with the card name, power limit and SM clock of the run.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import ClockSampler  # noqa: E402
from gptqmodel_b200 import B200QuantLinear, fuse_siblings  # noqa: E402
from gptqmodel_b200 import _lib as g  # noqa: E402
from helpers import random_layer  # noqa: E402

GS = 128
SINGLE = {4096: (1024, 2048, 3072, 4096), 14336: (1024, 2048, 3072, 4096)}  # <= 132 tiles: one decode_kernel launch
FUSED = {"qkv": (4096, (4096, 1024, 1024)), "gate_up": (4096, (14336, 14336))}
# (kernel version, K, N) of the bench's launches: o_proj, down_proj on decode_kernel; q|k|v, gate|up on decode2_kernel
BENCH_LAUNCHES = [(1, 4096, 4096), (1, 14336, 4096), (2, 4096, 6144), (2, 4096, 28672)]


def layer_bytes(K, N):
    return K * N // 2 + (K // GS) * N * 2


def make_mod(K, N, seed):
    L = random_layer(K, N, bits=4, group_size=GS, sym=True, seed=seed, device="cuda")
    return B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, GS,
                                                   device="cuda")


def time_graph(fn, iters):
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
    del gr
    return e0.elapsed_time(e1) / iters * 1e3  # µs per graph


def time_shape(Ns_of_set, K, min_mb, iters):
    """µs per launch over distinct copies of one launch (a single layer, or sibling layers fused into one launch)."""
    per = sum(layer_bytes(K, N) for N in Ns_of_set)
    copies = max(8, -(-int(min_mb * 2 ** 20) // per))
    sets = []
    for c in range(copies):
        mods = [make_mod(K, N, 1000 * c + i) for i, N in enumerate(Ns_of_set)]
        if len(mods) > 1 and not fuse_siblings(mods):
            raise RuntimeError("fuse_siblings refused the set")
        sets.append(mods)
    x = (torch.randn(1, K, device="cuda") * 0.5).to(torch.float16)

    def run():
        for mods in sets:
            for m in mods:
                m(x)

    us = time_graph(run, iters) / copies
    del sets
    torch.cuda.empty_cache()
    return {"us_per_launch": us, "bytes_per_launch": per, "copies": copies, "stream_mb": copies * per / 2 ** 20}


def fit(points):
    b = np.array([p["bytes_per_launch"] for p in points], dtype=np.float64)
    t = np.array([p["us_per_launch"] for p in points], dtype=np.float64)
    slope, icpt = np.polyfit(b, t, 1)  # µs per byte, µs
    return {"slope_tb_s": 1e-6 / slope if slope > 0 else None, "intercept_us": icpt}


def occupancy():
    fn = getattr(g.lib, "b2q_debug_decode_occupancy", None)
    if fn is None:
        return None
    out, plan = {}, (ctypes.c_int * 8)()
    blocks = ctypes.c_int(0)
    for ver, K, N in BENCH_LAUNCHES:
        # the library plans q|k|v and gate|up (more tiles than SMs) as one 16-warp group without split-K
        ks, warps = (1, 16) if ver == 2 else (0, 0)
        rc = g.lib.b2q_debug_decode_plan(ver, 1, K, N, ks, warps, plan)
        rc2 = fn(ver, 1, K, N, ks, warps, ctypes.byref(blocks))
        out[f"v{ver}_{K}x{N}"] = {"plan_rc": rc, "warps": plan[2], "smem_bytes": plan[7], "rc": rc2,
                                  "ctas_per_sm": blocks.value if rc2 == 0 else None}
    return out


def card():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        info["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        info["sm_clock_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception as e:  # noqa: BLE001
        info["nvml_error"] = f"{type(e).__name__}: {e}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    ap.add_argument("--min-mb", type=float, default=640.0, help="distinct weights + scales streamed per graph")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("decode_launch_cost: needs a CUDA GPU")
    torch.cuda.set_device(0)
    res = {"tool": "tools/decode_launch_cost.py", "M": 1, "group_size": GS, "dtype": "f16", **card()}
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    res["single"], res["fit"] = {}, {}
    allpts = []
    for K, Ns in SINGLE.items():
        pts = []
        for N in Ns:
            p = time_shape((N,), K, args.min_mb, args.iters)
            res["single"][f"{K}x{N}"] = p
            pts.append(p)
            print(f"[launch-cost] K={K} N={N}: {p['us_per_launch']:.2f} us/launch ({p['copies']} layers)",
                  file=sys.stderr, flush=True)
        res["fit"][f"K{K}"] = fit(pts)
        allpts += pts
    res["fit"]["all"] = fit(allpts)
    res["fused"] = {}
    for name, (K, Ns) in FUSED.items():
        res["fused"][name] = time_shape(Ns, K, args.min_mb, args.iters)
    sampler.stop_flag = True
    sampler.join()
    res["clocks"] = sampler.result()
    res["occupancy"] = occupancy()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
