"""Per-channel W8A8 MoE experts: the grouped path of B200ChannelW8A8Experts against the per-expert loop over the same
modules, and against the grouped block-FP8 and W4A16 GPTQ paths on the same shapes -> results/h100_moe_w8a8.json.

Stacks: Qwen3-30B-A3B (E 128, 2048 -> 768, top-8), Qwen3-235B-A22B (E 128, 4096 -> 1536, top-8), Mixtral-8x7B (E 8,
4096 -> 14336, top-2) and DeepSeek-V2-Lite (E 64, 2048 -> 1408, top-6), at T = 1, 8, 64, 512 and 4096 tokens with
softmax routing of random logits, in fp16 and bf16.  Arms: grouped FP8 dynamic, FP8 static, INT8 dynamic and INT8
static; the loop of each; grouped block-FP8 and grouped W4A16 GPTQ (group 128) as references.  All arms of a stack
are resident at once and alternate within each of three rounds; the median is reported.  A grouped arm at T <= 64 is
timed as a captured CUDA graph of the block (the host cost of six launches is not the kernels'); a grouped arm above
and every loop arm (it synchronises with the host) eagerly, with CUDA events around several calls.  TFLOP/s count
2 * T * top_k * (2 K I + I K) flops.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

STACKS = {"qwen3_30b_a3b": (128, 2048, 768, 8), "qwen3_235b_a22b": (128, 4096, 1536, 8),
          "mixtral_8x7b": (8, 4096, 14336, 2), "deepseek_v2_lite": (64, 2048, 1408, 6)}
TS = (1, 8, 64, 512, 4096)
DEV = "cuda"
W8A8 = {"fp8_dynamic": ("fp8", "dynamic"), "fp8_static": ("fp8", "static"), "int8_dynamic": ("int8", "dynamic"),
        "int8_static": ("int8", "static")}


def _w8a8_role(fmt, kind, E, K, N, seed):
    from gptqmodel_b200 import B200ChannelFp8Linear, B200ChannelInt8Linear

    g = torch.Generator(device=DEV).manual_seed(seed)
    if fmt == "fp8":
        cls, w = B200ChannelFp8Linear, (torch.randn(E, N, K, device=DEV, generator=g) * 60).clamp(-448, 448)
        w, qmax = w.to(torch.float8_e4m3fn), 448.0
    else:
        cls, qmax = B200ChannelInt8Linear, 127.0
        w = torch.randint(-127, 128, (E, N, K), device=DEV, generator=g, dtype=torch.int8)
    s = (torch.rand(E, N, 1, device=DEV, generator=g) + 0.5) / (60 * K ** 0.5)
    s_in = (torch.rand(E, 1, device=DEV, generator=g) + 0.5) * (2.0 / qmax)
    return [cls.from_checkpoint_tensors(w[e], s[e], input_scale=s_in[e] if kind == "static" else None, device=DEV)
            for e in range(E)]


def _w8a8(name, E, K, I):
    from gptqmodel_b200 import B200ChannelW8A8Experts, moe

    fmt, kind = W8A8[name]
    roles = [_w8a8_role(fmt, kind, E, k, n, 100 * r + 1) for r, (k, n) in enumerate(((K, I), (K, I), (I, K)))]
    if kind == "static":  # gate and up quantise the same rows with one input_scale, as in real checkpoints
        for a, b in zip(roles[0], roles[1]):
            b.input_scale = a.input_scale
    blk = B200ChannelW8A8Experts(*roles, grouped=True)
    return blk, moe.MoEExperts(list(blk.w1), list(blk.w3), list(blk.w2), grouped=False)


def _fp8blk(E, K, I):
    from gptqmodel_b200 import B200BlockFp8Linear, moe

    def role(k, n, seed):
        g = torch.Generator(device=DEV).manual_seed(seed)
        w = (torch.randn(E, n, k, device=DEV, generator=g) * 60).clamp(-448, 448).to(torch.float8_e4m3fn)
        s = (torch.rand(E, (n + 127) // 128, k // 128, device=DEV, generator=g) + 0.5) / (60 * k ** 0.5)
        return [B200BlockFp8Linear.from_checkpoint_tensors(w[e], s[e], device=DEV) for e in range(E)]

    return moe.MoEExperts(*[role(k, n, 7 + r) for r, (k, n) in enumerate(((K, I), (K, I), (I, K)))], grouped=True)


def _gptq4(E, K, I):
    from gptqmodel_b200 import B200QuantLinear, moe
    from helpers import random_layer

    def make(k, n, seed):
        L = random_layer(k, n, bits=4, group_size=128, sym=True, seed=seed, device=DEV)
        return B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, 128,
                                                       sym=True, device=DEV)

    return moe.MoEExperts(*[[make(k, n, 1000 * r + e) for e in range(E)]
                            for r, (k, n) in enumerate(((K, I), (K, I), (I, K)))], grouped=True)


def _time(fn, graph, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    if graph:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fn()
        torch.cuda.current_stream().wait_stream(s)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            fn()
        run = gr.replay
        run()
    else:
        run = fn
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        run()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e3  # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_moe_w8a8.json"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--stacks", default=",".join(STACKS))
    ap.add_argument("--ts", default=",".join(map(str, TS)))
    args = ap.parse_args()
    from hadamard_bench import card
    from gptqmodel_b200 import moe

    torch.manual_seed(0)
    out = {"card": card(), "units": "us per block; tflops counts 2 T top_k (3 K I) flops", "stacks": {}}
    for name in args.stacks.split(","):
        E, K, I, top_k = STACKS[name]
        arms = {}
        for w in W8A8:
            arms[f"{w}_grouped"], arms[f"{w}_loop"] = _w8a8(w, E, K, I)
        arms["fp8_block_grouped"] = _fp8blk(E, K, I)
        arms["w4a16_grouped"] = _gptq4(E, K, I)
        res = {}
        for dt in (torch.float16, torch.bfloat16):
            dn = str(dt).replace("torch.", "")
            for T in map(int, args.ts.split(",")):
                x = (torch.randn(T, K, device=DEV) * 0.5).to(dt)
                ids, wts = moe.route_topk(torch.randn(T, E, device=DEV), top_k)
                flops = 2.0 * T * top_k * 3 * K * I
                samples = {a: [] for a in arms}
                for _ in range(args.rounds):
                    for a, m in arms.items():
                        graph = a.endswith("grouped") and T <= 64
                        reps = (20 if T <= 512 else 5) if a.endswith("grouped") else (5 if T <= 512 else 2)
                        samples[a].append(_time(lambda m=m: m(x, ids, wts), graph, reps))
                for a, v in samples.items():
                    med = statistics.median(v)
                    res.setdefault(dn, {}).setdefault(a, {})[str(T)] = {
                        "us": round(med, 2), "spread_us": round(max(v) - min(v), 2),
                        "tflops": round(flops / med / 1e6, 3),
                        "timing": "graph" if a.endswith("grouped") and T <= 64 else "eager"}
                    print(name, dn, a, T, res[dn][a][str(T)], flush=True)
        out["stacks"][name] = {"E": E, "K": K, "I": I, "top_k": top_k, "arms": res}
        del arms
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
