"""Block-FP8 MoE experts: the grouped e4m3 path vs the per-expert loop, with the GPTQ W4A16 grouped path for context.

    python tools/moe_fp8_block_bench.py [--iters 20] [--rounds 3] [--out results/h100_moe_fp8_block.json]

Stacks (random e4m3 weights with 128 x 128 block scales, bf16 activations, softmax top-8 routing, one GPU):
  * qwen3_30b_a3b:   E 128, 2048 -> 768   (Qwen3-30B-A3B-FP8);
  * qwen3_235b_a22b: E 128, 4096 -> 1536  (Qwen3-235B-A22B-FP8);
  * deepseek_v3_ep8: E 32, 7168 -> 2048   (DeepSeek-V3 / R1, the 256 routed experts over 8 GPUs).
Arms, alternated over `rounds` rounds in one run and timed with CUDA events over `iters` calls (median of the rounds):
  * grouped: MoEExperts over B200BlockFp8Linear experts (six launches, no host synchronisation);
  * loop: the same modules with grouped=False (three module calls per routed expert; its per-block host synchronisation
    lands inside the timed window);
  * w4a16: MoEExperts over random 4-bit g128 symmetric GPTQ experts of the same shapes (grouped midm path).
Derived figures: at T <= 64 the distinct routed experts' weight bytes (e4m3 + scales, or 4-bit codes + fp16 scales) over
the time, as a share of the H100 SXM data sheet's 3.35 TB/s; at T >= 512 TFLOP/s from routed rows, 6 * T * top_k * K * I
over the time.  The card's name and power limit are read in the same run and written beside the numbers.
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

STACKS = {"qwen3_30b_a3b": (128, 2048, 768, 8), "qwen3_235b_a22b": (128, 4096, 1536, 8),
          "deepseek_v3_ep8": (32, 7168, 2048, 8)}  # E, K, I, top_k
TOKENS = (1, 8, 64, 512, 4096)
HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                       str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["?"])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(), "?")
    return {"name": name, "power_limit": power}


def build_fp8(E, K, I):
    from gptqmodel_b200 import B200BlockFp8Linear, moe

    gen = torch.Generator(device="cuda").manual_seed(0)

    def role(N, Kr):
        w = (torch.randn(E, N, Kr, device="cuda", generator=gen) * 60).clamp(-448, 448).to(torch.float8_e4m3fn)
        s = (torch.rand(E, (N + 127) // 128, Kr // 128, device="cuda", generator=gen) + 0.5) / (60 * Kr ** 0.5)
        return [B200BlockFp8Linear.from_checkpoint_tensors(w[e], s[e], device="cuda") for e in range(E)]

    blk = moe.MoEExperts(role(I, K), role(I, K), role(K, I), grouped=True)
    loop = moe.MoEExperts(list(blk.w1), list(blk.w3), list(blk.w2), grouped=False)
    return blk, loop


def build_w4a16(E, K, I):
    from gptqmodel_b200 import B200QuantLinear, moe
    from helpers import random_layer

    def mod(k, n, seed):
        L = random_layer(k, n, bits=4, group_size=128, sym=True, seed=seed, device="cuda")
        return B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, 128, sym=True)

    return moe.MoEExperts([mod(K, I, 3 * e) for e in range(E)], [mod(K, I, 3 * e + 1) for e in range(E)],
                          [mod(I, K, 3 * e + 2) for e in range(E)], grouped=True)


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
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--stacks", default=",".join(STACKS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from gptqmodel_b200 import moe

    torch.cuda.set_device(0)
    res = {"device": card(), "iters": args.iters, "rounds": args.rounds, "dtype": "bfloat16",
           "unit": "us per MoE block call", "hbm_peak_bytes_per_s": HBM, "stacks": {}}
    for name in args.stacks.split(","):
        E, K, I, top_k = STACKS[name]
        fp8, loop = build_fp8(E, K, I)
        w4 = build_w4a16(E, K, I)
        fp8_bytes = 3 * (K * I + 4 * (K // 128) * ((I + 127) // 128))  # one expert: e4m3 + fp32 block scales
        w4_bytes = 3 * (K * I // 2 + 2 * (K // 128) * I)
        rows = []
        for T in TOKENS:
            gen = torch.Generator(device="cuda").manual_seed(T)
            x = torch.randn(T, K, device="cuda", generator=gen).to(torch.bfloat16)
            ids, w = moe.route_topk(torch.randn(T, E, device="cuda", generator=gen), top_k)
            arms = {"grouped": lambda: fp8(x, ids, w), "loop": lambda: loop(x, ids, w), "w4a16": lambda: w4(x, ids, w)}
            yg, yl = arms["grouped"](), arms["loop"]()
            rel = ((yg.float() - yl.float()).norm() / yl.float().norm()).item()
            for _ in range(args.warmup):
                for f in arms.values():
                    f()
            torch.cuda.synchronize()
            iters = max(3, args.iters // (1 + T // 512))
            t = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, f in arms.items():
                    t[k].append(time_call(f, iters))
            med = {k: statistics.median(v) for k, v in t.items()}
            row = {"T": T, "iters": iters, "grouped_vs_loop_rel_l2": rel}
            for k in arms:
                row[f"{k}_us"] = round(med[k], 2)
                row[f"{k}_us_rounds"] = [round(v, 2) for v in t[k]]
            row["loop_over_grouped"] = round(med["loop"] / med["grouped"], 3)
            distinct = int(torch.unique(ids).numel())
            if T <= 64:
                row["distinct_experts"] = distinct
                row["grouped_hbm_share"] = round(distinct * fp8_bytes / (med["grouped"] * 1e-6) / HBM, 4)
                row["w4a16_hbm_share"] = round(distinct * w4_bytes / (med["w4a16"] * 1e-6) / HBM, 4)
            if T >= 512:
                flops = 6.0 * T * top_k * K * I
                row["grouped_tflops"] = round(flops / (med["grouped"] * 1e-6) / 1e12, 1)
                row["w4a16_tflops"] = round(flops / (med["w4a16"] * 1e-6) / 1e12, 1)
                row["grouped_over_w4a16_tflops"] = round(med["w4a16"] / med["grouped"], 3)
            rows.append(row)
            print(f"{name} T={T}: grouped {med['grouped']:.1f} us, loop {med['loop']:.1f} us, w4a16 "
                  f"{med['w4a16']:.1f} us", flush=True)
        res["stacks"][name] = {"E": E, "K": K, "I": I, "top_k": top_k, "results": rows}
        del fp8, loop, w4
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
