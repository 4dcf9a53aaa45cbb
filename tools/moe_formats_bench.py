"""Grouped MoE path vs the per-expert loop (MoEExperts(grouped=False)) on 8-bit and act-order expert stacks.

    python tools/moe_formats_bench.py [--iters 50] [--rounds 5] [--out FILE.json]

Stacks (random codes, one GPU):
  * qwen1.5_moe_a2.7b_int8: E 60, 2048 -> 1408, 8-bit, g128, sym, top-4 (Qwen1.5-MoE-A2.7B-Chat-GPTQ-Int8 shape);
  * mixtral_8x7b_act_order: E 8, 4096 -> 14336, 4-bit, g128, asym, act-order (desc_act=True), top-2;
  * mixtral_8x7b: the same without act-order, as a control for what the permuting gathers cost.
At T in {1, 8, 64, 512} tokens both paths are warmed up, then timed with CUDA events over `iters` calls, alternating
grouped and loop for `rounds` rounds; the median per-call time of the rounds is reported.  The loop path's per-block host
synchronisation is part of its cost and lands inside the timed window.  The card's name and power limit are read in the
same run and written beside the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

STACKS = {  # E, K, I, bits, group size, sym, act-order, top_k
    "qwen1.5_moe_a2.7b_int8": (60, 2048, 1408, 8, 128, True, False, 4),
    "mixtral_8x7b_act_order": (8, 4096, 14336, 4, 128, False, True, 2),
    # control: the same stack without act-order (the grouped path as it was before 8-bit / act-order experts)
    "mixtral_8x7b": (8, 4096, 14336, 4, 128, False, False, 2),
}
TOKENS = (1, 8, 64, 512)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["?"])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(), "?")
    return {"name": name, "power_limit": power}


def build(name):
    from gptqmodel_b200 import B200QuantLinear, moe
    from helpers import random_layer

    E, K, I, bits, gs, sym, act, _ = STACKS[name]

    def mod(k, n, seed, perm_seed=None):
        L = random_layer(k, n, bits=bits, group_size=gs, sym=sym, seed=seed, device="cuda")
        g_idx = L["g_idx"]
        if perm_seed is not None:  # act-order: rows assigned to groups in a random order
            gen = torch.Generator().manual_seed(perm_seed)
            g_idx = (torch.arange(k, dtype=torch.int32) // gs)[torch.randperm(k, generator=gen)].cuda()
        m = B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], g_idx, bits, gs, sym=sym,
                                                    desc_act=act)
        del L
        return m

    w1 = [mod(K, I, 3 * e, e if act else None) for e in range(E)]
    w3 = [mod(K, I, 3 * e + 1, e if act else None) for e in range(E)]  # w1 and w3 share the permutation
    w2 = [mod(I, K, 3 * e + 2, 1000 + e if act else None) for e in range(E)]
    blk = moe.MoEExperts(w1, w3, w2, grouped=True)
    loop = moe.MoEExperts(list(blk.w1), list(blk.w3), list(blk.w2), grouped=False)
    return blk, loop


def time_call(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters  # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from gptqmodel_b200 import moe

    torch.cuda.set_device(0)
    res = {"device": card(), "iters": args.iters, "rounds": args.rounds, "unit": "us per MoE block call", "stacks": {}}
    for name in STACKS:
        E, K, I, bits, gs, sym, act, top_k = STACKS[name]
        blk, loop = build(name)
        rows = []
        for T in TOKENS:
            gen = torch.Generator(device="cuda").manual_seed(T)
            x = (torch.randn(T, K, device="cuda", generator=gen) * 0.5).to(torch.float16)
            ids, w = moe.route_topk(torch.randn(T, E, device="cuda", generator=gen), top_k)
            g = lambda: blk(x, ids, w)  # noqa: E731
            lp = lambda: loop(x, ids, w)  # noqa: E731
            yg, yl = g(), lp()
            rel = ((yg.float() - yl.float()).norm() / yl.float().norm()).item()
            for _ in range(args.warmup):
                g()
                lp()
            torch.cuda.synchronize()
            tg, tl = [], []
            for _ in range(args.rounds):
                tg.append(time_call(g, args.iters))
                tl.append(time_call(lp, args.iters))
            mg, ml = statistics.median(tg), statistics.median(tl)
            rows.append({"T": T, "grouped_us": round(mg, 2), "loop_us": round(ml, 2), "speedup": round(ml / mg, 3),
                         "grouped_us_rounds": [round(v, 2) for v in tg], "loop_us_rounds": [round(v, 2) for v in tl],
                         "grouped_vs_loop_rel_l2": rel})
            print(f"{name} T={T}: grouped {mg:.1f} us, loop {ml:.1f} us, x{ml / mg:.2f}", flush=True)
        res["stacks"][name] = {"E": E, "K": K, "I": I, "bits": bits, "group_size": gs, "sym": sym, "act_order": act,
                               "top_k": top_k, "dtype": "float16", "results": rows}
        del blk, loop
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
