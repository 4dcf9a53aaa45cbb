"""QQQ (W4A8) and FP8 (W8A16) MoE experts: the grouped paths of MoEExperts against the per-expert loop, and against the
grouped 4-bit and 8-bit GPTQ paths on the same shapes -> results/h100_moe_qqq_fp8.json.

Stacks: Qwen3-30B-A3B (E 128, 2048 -> 768, top-8), Mixtral-8x7B (E 8, 4096 -> 14336, top-2), DeepSeek-V2-Lite (E 64,
2048 -> 1408, top-6), at T = 1, 8, 64, 512 and 4096 tokens with softmax routing of random logits.  Arms: grouped QQQ,
loop QQQ, grouped FP8, loop FP8, grouped W4A16 GPTQ (group 128) and grouped 8-bit GPTQ (the same bytes as FP8).  One
format's stack is resident at a time; the arms of a stack alternate within each of three rounds.  A grouped arm at
T <= 64 is timed as a captured CUDA graph of the block (the host cost of six launches is not the kernels'); a grouped
arm above and every loop arm (it synchronises with the host) eagerly, with CUDA events around 5..20 calls.  TFLOP/s
count 2 * T * top_k * (2 K I + I K) flops.  The card's name and power limit are read in the same run.
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

STACKS = {"qwen3_30b_a3b": (128, 2048, 768, 8), "mixtral_8x7b": (8, 4096, 14336, 2),
          "deepseek_v2_lite": (64, 2048, 1408, 6)}
TS = (1, 8, 64, 512, 4096)
DEV = "cuda"


def _qqq(K, N, seed):
    from gptqmodel_b200 import B200QqqQuantLinear, lib
    from gptqmodel_b200._lib import check

    g = torch.Generator(device=DEV).manual_seed(seed)
    m = B200QqqQuantLinear(bits=4, group_size=128, desc_act=False, sym=True, in_features=K, out_features=N,
                           register_buffers=False)
    codes = torch.randint(0, 16, (K, N), dtype=torch.uint8, device=DEV, generator=g)
    m.packed = torch.empty(lib.b2q_qqq_packed_bytes(K, N), dtype=torch.uint8, device=DEV)
    check(lib.b2q_qqq_prepack(codes.data_ptr(), m.packed.data_ptr(), K, N, 128, torch.cuda.current_stream().cuda_stream),
          "prepack")
    m._sc = (torch.rand(N, device=DEV, generator=g) + 0.5) / (127 * 8 * K ** 0.5)
    m._sg = (torch.rand(K // 128, N, device=DEV, generator=g) * 7 + 1).to(torch.float16)
    m._kgs, m._prepacked = 128, True
    return m


def _fp8(K, N, seed):
    from gptqmodel_b200 import B200Fp8QuantLinear

    g = torch.Generator(device=DEV).manual_seed(seed)
    w = (torch.randn(N, K, device=DEV, generator=g) * 100).clamp(-448, 448).to(torch.float8_e4m3fn)
    s = (torch.rand(N // 128, K // 128, device=DEV, generator=g) + 0.5) * 100 * K ** 0.5
    return B200Fp8QuantLinear.from_checkpoint_tensors(w, s, device=DEV)


def _gptq(bits):
    def make(K, N, seed):
        from gptqmodel_b200 import B200QuantLinear
        from helpers import random_layer

        L = random_layer(K, N, bits=bits, group_size=128, sym=True, seed=seed, device=DEV)
        return B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], bits, 128,
                                                       sym=True, device=DEV)
    return make


FORMATS = {"qqq": _qqq, "fp8": _fp8, "gptq4": _gptq(4), "gptq8": _gptq(8)}


def _block(fmt, E, K, I, grouped):
    from gptqmodel_b200 import moe

    make = FORMATS[fmt]
    roles = [[make(k, n, 1000 * r + e) for e in range(E)] for r, (k, n) in enumerate(((K, I), (K, I), (I, K)))]
    blk = moe.MoEExperts(*roles, grouped=True)
    loop = moe.MoEExperts(list(blk.w1), list(blk.w3), list(blk.w2), grouped=False) if grouped else None
    return blk, loop


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
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_moe_qqq_fp8.json"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--stacks", default=",".join(STACKS))
    args = ap.parse_args()
    from hadamard_bench import card
    from gptqmodel_b200 import moe

    torch.manual_seed(0)
    out = {"card": card(), "dtype": "float16", "units": "us per block; tflops counts 2 T top_k (3 K I) flops",
           "stacks": {}}
    for name in args.stacks.split(","):
        E, K, I, top_k = STACKS[name]
        res = {}
        for fmt in ("qqq", "fp8", "gptq4", "gptq8"):
            blk, loop = _block(fmt, E, K, I, grouped=fmt in ("qqq", "fp8"))
            arms = {f"{fmt}_grouped": blk}
            if loop is not None:
                arms[f"{fmt}_loop"] = loop
            for T in TS:
                x = (torch.randn(T, K, device=DEV) * 0.5).half()
                ids, w = moe.route_topk(torch.randn(T, E, device=DEV), top_k)
                flops = 2.0 * T * top_k * 3 * K * I
                samples = {a: [] for a in arms}
                for _ in range(args.rounds):
                    for a, m in arms.items():
                        graph = a.endswith("grouped") and T <= 64
                        reps = 20 if T <= 512 else 5
                        samples[a].append(_time(lambda m=m: m(x, ids, w), graph, reps))
                for a, v in samples.items():
                    med = statistics.median(v)
                    res.setdefault(a, {})[str(T)] = {"us": round(med, 2), "spread_us": round(max(v) - min(v), 2),
                                                     "tflops": round(flops / med / 1e6, 3),
                                                     "timing": "graph" if a.endswith("grouped") and T <= 64 else "eager"}
                    print(name, a, T, res[a][str(T)], flush=True)
            del blk, loop, arms
            torch.cuda.empty_cache()
        out["stacks"][name] = {"E": E, "K": K, "I": I, "top_k": top_k, "arms": res}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
