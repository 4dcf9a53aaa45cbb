"""MoE routing: transformers' routing function bodies in torch vs one b2q_moe_route launch.

    python tools/moe_route_bench.py [--iters 200] [--rounds 3] [--out results/h100_moe_route.json]

Configs (random logits; fp32 for the sigmoid routers, whose gate runs in fp32, bf16 for the softmax ones):
  * mixtral:        E 8,   top-2, softmax, renormalised      (MixtralTopKRouter)
  * qwen3_30b_a3b:  E 128, top-8, softmax, renormalised      (Qwen3MoeTopKRouter, norm_topk_prob)
  * olmoe:          E 64,  top-8, softmax, not renormalised
  * deepseek_v3:    E 256, top-8, grouped sigmoid, n_group 8, topk_group 4, routed_scaling_factor 2.5
                    (DeepseekV3MoE.route_tokens_to_experts)
  * glm4_5:         E 160, top-8, grouped sigmoid, n_group 1, routed_scaling_factor 2.5 (Glm4MoeMoE)
at T = 1, 16, 128, 1024, 8192.  Before timing, the two routings must choose the same expert set on every row (the torch
bodies select with topk(sorted=False), so sets are compared) except where the float64 scores tie within 1e-6 at the k-th
place or the group boundary, so that fp32 rounding decides; such rows are counted.  Both arms are timed eager and as a replayed CUDA graph of
one call, with CUDA events over `iters` calls, alternated over `rounds` rounds (median).  The kernel count of one eager
call comes from a separate torch.profiler run.  One end-to-end line: the qwen3_30b_a3b block-FP8 stack of
tools/moe_fp8_block_bench.py (E 128, 2048 -> 768, top-8) at T = 1 in bf16, router + experts graph-replayed, routed by the
torch body vs by the kernel.  The card's name and power limit are read in the same run and written beside the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# E, top_k, scoring, renormalize, n_group, topk_group, scale
CONFIGS = {
    "mixtral": (8, 2, "softmax", True, 1, 1, 1.0),
    "qwen3_30b_a3b": (128, 8, "softmax", True, 1, 1, 1.0),
    "olmoe": (64, 8, "softmax", False, 1, 1, 1.0),
    "deepseek_v3": (256, 8, "sigmoid", True, 8, 4, 2.5),
    "glm4_5": (160, 8, "sigmoid", True, 1, 1, 2.5),
}
TOKENS = (1, 16, 128, 1024, 8192)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                       str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["?"])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(), "?")
    return {"name": name, "power_limit": power}


def torch_softmax(logits, top_k, renormalize):
    """MixtralTopKRouter / Qwen3MoeTopKRouter after the gate's linear."""
    p = F.softmax(logits, dtype=torch.float, dim=-1)
    w, ids = torch.topk(p, top_k, dim=-1)
    if renormalize:
        w /= w.sum(dim=-1, keepdim=True)
    return ids, w


def torch_grouped(logits, bias, top_k, n_group, topk_group, renormalize, scale):
    """DeepseekV3MoE.route_tokens_to_experts (Glm4MoeMoE's is the same)."""
    E = logits.shape[-1]
    s = logits.sigmoid()
    c = s + bias
    group_scores = c.view(-1, n_group, E // n_group).topk(2, dim=-1)[0].sum(dim=-1)
    group_idx = torch.topk(group_scores, k=topk_group, dim=-1, sorted=False)[1]
    group_mask = torch.zeros_like(group_scores)
    group_mask.scatter_(1, group_idx, 1)
    score_mask = group_mask.unsqueeze(-1).expand(-1, n_group, E // n_group).reshape(-1, E)
    choice = c.masked_fill(~score_mask.bool(), 0.0)
    ids = torch.topk(choice, k=top_k, dim=-1, sorted=False)[1]
    w = s.gather(1, ids)
    if renormalize:
        w /= w.sum(dim=-1, keepdim=True) + 1e-20
    return ids, w * scale


def arms(cfg, logits, bias):
    from gptqmodel_b200 import moe

    E, k, scoring, norm, ng, tg, scale = cfg
    if scoring == "softmax":
        return {"torch": lambda: torch_softmax(logits, k, norm),
                "kernel": lambda: moe.route_softmax_topk(logits, k, renormalize=norm, scale=scale)}
    return {"torch": lambda: torch_grouped(logits, bias, k, ng, tg, norm, scale),
            "kernel": lambda: moe.route_grouped_sigmoid(logits, bias, k, ng, tg, renormalize=norm, scale=scale)}


def time_call(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters  # us per call


def graphed(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def kernel_count(fn):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def same_sets(a, b):
    return (a.long().sort(-1).values == b.long().sort(-1).values).all(-1)


def near_tie(cfg, logits, bias, gap=1e-6):
    """Rows whose float64 selection scores lie within `gap` at the k-th place or at the kept-group boundary."""
    from oracle import moe_route_oracle as ro

    E, k, scoring, norm, ng, tg, scale = cfg

    def close(v, n):
        if n >= v.shape[1]:
            return torch.zeros(v.shape[0], dtype=torch.bool, device=v.device)
        top = v.sort(dim=-1, descending=True).values
        return (top[:, n - 1] - top[:, n]) <= gap * top[:, n - 1].abs().clamp(min=1)

    if scoring == "softmax":
        return close(logits.double(), k)
    _, _, masked, _ = ro.route_grouped_sigmoid(logits, bias, k, ng, tg)
    _, c = ro.sigmoid_scores(logits, bias)
    return close(masked, k) | close(ro.group_scores(c, ng), tg)


def timed(fns, iters, rounds, warmup):
    for _ in range(warmup):
        for f in fns.values():
            f()
    torch.cuda.synchronize()
    t = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            t[k].append(time_call(f, iters))
    return {k: statistics.median(v) for k, v in t.items()}, t


def end_to_end(iters, rounds, warmup):
    """qwen3_30b_a3b block-FP8 experts at T = 1 in bf16, router + block graph-replayed."""
    from gptqmodel_b200 import B200BlockFp8Linear, moe

    E, K, I, k = 128, 2048, 768, 8
    gen = torch.Generator(device="cuda").manual_seed(0)

    def role(N, Kr):
        w = (torch.randn(E, N, Kr, device="cuda", generator=gen) * 60).clamp(-448, 448).to(torch.float8_e4m3fn)
        s = (torch.rand(E, (N + 127) // 128, Kr // 128, device="cuda", generator=gen) + 0.5) / (60 * Kr ** 0.5)
        return [B200BlockFp8Linear.from_checkpoint_tensors(w[e], s[e], device="cuda") for e in range(E)]

    blk = moe.MoEExperts(role(I, K), role(I, K), role(K, I), grouped=True)
    x = torch.randn(1, K, device="cuda", generator=gen).to(torch.bfloat16)
    logits = torch.randn(1, E, device="cuda", generator=gen).to(torch.bfloat16)
    fns = {"torch": lambda: blk(x, *torch_softmax(logits, k, True)),
           "kernel": lambda: blk(x, *moe.route_softmax_topk(logits, k))}
    y = {n: f() for n, f in fns.items()}
    assert torch.equal(y["torch"], y["kernel"]) or same_sets(torch_softmax(logits, k, True)[0],
                                                             moe.route_softmax_topk(logits, k)[0]).all()
    graphs = {n: graphed(f) for n, f in fns.items()}
    med, t = timed({n: g.replay for n, g in graphs.items()}, iters, rounds, warmup)
    yt, yk = fns["torch"](), fns["kernel"]()
    rel = ((yt.float() - yk.float()).norm() / yt.float().norm()).item()
    return {"stack": "qwen3_30b_a3b block-FP8", "E": E, "K": K, "I": I, "top_k": k, "T": 1, "dtype": "bfloat16",
            "mode": "graph", "torch_routed_us": round(med["torch"], 2), "kernel_routed_us": round(med["kernel"], 2),
            "torch_routed_us_rounds": [round(v, 2) for v in t["torch"]],
            "kernel_routed_us_rounds": [round(v, 2) for v in t["kernel"]],
            "saving_us": round(med["torch"] - med["kernel"], 2), "output_rel_l2": rel}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    torch.cuda.set_device(0)
    res = {"device": card(), "iters": args.iters, "rounds": args.rounds, "unit": "us per routing call", "configs": {}}
    for name in args.configs.split(","):
        cfg = CONFIGS[name]
        E, k, scoring = cfg[:3]
        rows = []
        for T in TOKENS:
            gen = torch.Generator(device="cuda").manual_seed(T + E)
            logits = torch.randn(T, E, device="cuda", generator=gen) * 2
            logits = logits if scoring == "sigmoid" else logits.to(torch.bfloat16)
            bias = torch.rand(E, device="cuda", generator=gen) * 0.1 if scoring == "sigmoid" else None
            fns = arms(cfg, logits, bias)
            ids_t, w_t = fns["torch"]()
            ids_k, w_k = fns["kernel"]()
            agree = same_sets(ids_t, ids_k)
            n_bad = int((~agree).sum())
            # the two may differ only where fp32 rounding decides: a gap of at most 1e-6 at the k-th place or the group
            # boundary (float64 scores)
            near = near_tie(cfg, logits, bias)
            assert not (~agree & ~near).any(), f"{name} T={T}: the routings choose different experts on {n_bad} rows"
            order_t, order_k = ids_t.argsort(-1), ids_k.long().argsort(-1)
            iters = max(20, args.iters // (1 + T // 1024))
            eager, eager_r = timed(fns, iters, args.rounds, args.warmup)
            graphs = {n: graphed(f) for n, f in fns.items()}
            graph, graph_r = timed({n: g.replay for n, g in graphs.items()}, iters, args.rounds, args.warmup)
            del graphs
            w_rel = ((w_t.gather(1, order_t) - w_k.gather(1, order_k)).abs() / w_t.gather(1, order_t).abs())[agree].max().item()
            row = {"T": T, "iters": iters, "rows_with_other_experts": n_bad, "weights_max_rel_diff": w_rel,
                   "kernels_torch": kernel_count(fns["torch"]), "kernels_kernel": kernel_count(fns["kernel"])}
            for n in fns:
                row[f"{n}_eager_us"] = round(eager[n], 2)
                row[f"{n}_graph_us"] = round(graph[n], 2)
                row[f"{n}_eager_us_rounds"] = [round(v, 2) for v in eager_r[n]]
                row[f"{n}_graph_us_rounds"] = [round(v, 2) for v in graph_r[n]]
            row["eager_speedup"] = round(eager["torch"] / eager["kernel"], 2)
            row["graph_speedup"] = round(graph["torch"] / graph["kernel"], 2)
            rows.append(row)
            print(f"{name} T={T}: eager torch {eager['torch']:.1f} / kernel {eager['kernel']:.1f} us, graph torch "
                  f"{graph['torch']:.1f} / kernel {graph['kernel']:.1f} us, kernels {row['kernels_torch']} / "
                  f"{row['kernels_kernel']}", flush=True)
        res["configs"][name] = {"E": E, "top_k": k, "scoring": scoring, "renormalize": cfg[3], "n_group": cfg[4],
                                "topk_group": cfg[5], "scale": cfg[6],
                                "logits_dtype": "float32" if scoring == "sigmoid" else "bfloat16", "results": rows}
    res["end_to_end"] = end_to_end(max(50, args.iters), args.rounds, args.warmup)
    print("end to end:", res["end_to_end"], flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
