#!/usr/bin/env python
"""Measure the online Hadamard transform of rotated (QuaRot / SpinQuant) checkpoints on one GPU.

    python tools/hadamard_bench.py --out results/h100_hadamard.json

1. b2q_hadamard alone: µs per launch from CUDA events over a CUDA graph of many launches, and the achieved bytes/s
   (4 * rows * n bytes: one 16-bit read and one 16-bit write per element) against the H100 SXM data-sheet 3.35 TB/s.
2. The Llama-3-8B linear stack of bench.py (`build_stack`, 32 layers, 4-bit g128) with the order-28 matrix on every
   down_proj, against the same stack unrotated: decode (1 token) tok/s and 2048-token prefill TFLOP/s.  The two are
   timed alternately in the same process, on the same weights (only the down_proj rotation flag differs).
3. A torch.profiler kernel summary of one rotated decode pass, to show where the extra time goes.
The card's name and power limit are read in the same run and stored with the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35  # H100 SXM data sheet
GOLDEN = os.path.join(ROOT, "tests", "golden", "hadamard_cases.npz")
SHAPES = ((11008, 172), (14336, 28), (28672, 28), (8192, 1))
ROWS = (1, 8, 64, 2048)


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = r.stdout.strip().splitlines()[0]
    except Exception as e:  # the number is still valid, the card's limit is then unknown
        info["power_limit_and_max_sm_clock"] = f"unavailable ({e})"
    return info


def had(K):
    return None if K == 1 else torch.from_numpy(np.load(GOLDEN)[f"had{K}"]).cuda()


def time_kernel(n, K, rows, launches=100, reps=5):
    import gptqmodel_b200 as g

    h = had(K)
    x = (torch.randn(rows, n, device="cuda")).half()
    y = torch.empty_like(x)
    s = torch.cuda.Stream()

    def launch():
        g.check(g.lib.b2q_hadamard(x.data_ptr(), None if h is None else h.data_ptr(), K, y.data_ptr(), rows, n, 0,
                                   torch.cuda.current_stream().cuda_stream), "b2q_hadamard")

    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            launch()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(launches):
            launch()
    graph.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / launches)
    us = statistics.median(times)
    tbs = 4.0 * rows * n / (us * 1e-6) / 1e12
    return {"n": n, "K": K, "rows": rows, "us_per_launch": round(us, 3), "TB_per_s": round(tbs, 3),
            "share_of_3.35TBs": round(tbs / HBM_TBS, 3)}


def set_rotation(stack, on, h28):
    for mods in stack:
        m = mods["down_proj"]
        if m.had_K is None:
            m.K = 28
            m.set_had_K(h28)
        m.online_full_had = on


def stack_arms(layers, rounds):
    import bench

    dev = torch.device("cuda:0")
    stack = bench.build_stack(dev, 0, 1, layers, fuse=True)
    h28 = had(28).float().cpu()
    _, weights = bench.stack_bytes_and_weights(bench.CFG, layers)
    res = {"layers": layers, "rounds": rounds, "decode_ms": {"plain": [], "rotated": []},
           "prefill2048_ms": {"plain": [], "rotated": []}}
    for _ in range(rounds):
        for arm in ("plain", "rotated"):
            set_rotation(stack, arm == "rotated", h28)
            ms, fin = bench.time_stack(stack, 1, 1, dev, 200, bench.CFG["hidden"])
            assert fin
            res["decode_ms"][arm].append(round(ms, 4))
            ms, fin = bench.time_stack(stack, 2048, 1, dev, 10, bench.CFG["hidden"])
            assert fin
            res["prefill2048_ms"][arm].append(round(ms, 4))
    med = {k: {a: statistics.median(v) for a, v in d.items()} for k, d in
           (("decode", res["decode_ms"]), ("prefill", res["prefill2048_ms"]))}
    res["decode_tok_s"] = {a: round(1e3 / ms, 1) for a, ms in med["decode"].items()}
    res["prefill_tflops"] = {a: round(2.0 * 2048 * weights / (ms * 1e-3) / 1e12, 1) for a, ms in med["prefill"].items()}
    res["decode_ratio_rotated_over_plain"] = round(med["decode"]["plain"] / med["decode"]["rotated"], 4)
    res["prefill_ratio_rotated_over_plain"] = round(med["prefill"]["plain"] / med["prefill"]["rotated"], 4)
    res["profile_rotated_decode"] = profile_decode(stack, h28)
    return res


def profile_decode(stack, h28):
    """GPU time per kernel name over 20 rotated decode passes (torch.profiler, CUDA activity)."""
    import bench
    from torch.profiler import ProfilerActivity, profile

    set_rotation(stack, True, h28)
    x = (torch.randn(1, bench.CFG["hidden"], device="cuda") * 0.5).half()
    for _ in range(3):
        bench.run_stack(stack, x, 1)
    torch.cuda.synchronize()
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                bench.run_stack(stack, x, 1)
            torch.cuda.synchronize()
    except Exception as e:
        return f"unavailable ({e})"
    rows = []
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t > 0:
            rows.append({"kernel": ev.key[:90], "calls": ev.count, "us_per_pass": round(t / 20, 2)})
    rows.sort(key=lambda r: -r["us_per_pass"])
    return rows[:10]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_hadamard.json"))
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("hadamard_bench: needs a CUDA device (no CPU timing is meaningful here)")
    torch.cuda.set_device(0)
    out = {"card": card(), "kernel": [time_kernel(n, K, r) for n, K in SHAPES for r in ROWS],
           "stack": stack_arms(args.layers, args.rounds),
           "competitor": "not measured (the reference's fast-hadamard-transform extension is not built)"}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
