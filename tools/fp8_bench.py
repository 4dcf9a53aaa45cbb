#!/usr/bin/env python
"""Measure FP8 (e4m3fn, block [128, 128]) layers on one GPU.

    python tools/fp8_bench.py --out results/h100_fp8.json

The 32-layer Llama-3-8B linear stack of bench.py (its shapes and run order, fp16 activations, no sibling fusion), three
arms built from weights of the same size (one byte per weight):
  * fp8_b200    : B200Fp8QuantLinear (b2q_fp8_mm);
  * gptq8_b200  : this project's 8-bit GPTQ g128 B200QuantLinear (b2q_mm), the same bytes with an integer dequant;
  * fp8_torch   : the reference's arithmetic in torch (TorchFP8Linear's dequantise-then-matmul path): every call expands
                  the scales, divides the weight and calls torch.matmul.
Decode tok/s (1 token), 16- and 64-token steps (tokens/s) and 2048-token prefill TFLOP/s counting 2*M*K*N; every pass is
one CUDA graph timed with CUDA events, the arms alternate within each round.  The card's name and power limit are read
in the same run and stored with the numbers.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

STEPS = ((1, 200), (16, 100), (64, 50), (2048, 5))  # (tokens, graph replays per timing)


def fp8_tensors(K, N, seed, dev):
    """e4m3 codes [N, K] and block-128 scale_inv with W = w / s of rms ~ 1 / sqrt(K) (the chained activations stay O(1))."""
    g = torch.Generator(device=dev).manual_seed(seed)
    w = (torch.randn(N, K, device=dev, generator=g) * 64.0).clamp(-448, 448).to(torch.float8_e4m3fn)
    s = (0.8 + 0.4 * torch.rand(N // 128, K // 128, device=dev, generator=g)) * 64.0 * K ** 0.5
    return w, s


def gptq8_tensors(K, N, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    qw = torch.randint(1, 256, (K, N), device=dev, generator=g, dtype=torch.int32)
    qw = qw.view(K // 4, 4, N)
    qw = qw[:, 0] | (qw[:, 1] << 8) | (qw[:, 2] << 16) | (qw[:, 3] << 24)
    qz = torch.full((K // 128, N // 4), 0x80808080 - (1 << 32), dtype=torch.int32, device=dev)
    sc = ((0.8 + 0.4 * torch.rand(K // 128, N, device=dev, generator=g)) / (5461.0 * K) ** 0.5).to(torch.float16)
    gi = torch.arange(K, dtype=torch.int32, device=dev) // 128
    return qw.contiguous(), qz, sc, gi


class TorchFp8(torch.nn.Module):
    """The reference's CUDA dequantise-then-matmul arithmetic (TorchFP8Linear._forward_dequant_matmul), restated."""

    def __init__(self, w, s):
        super().__init__()
        self.w, self.s = w, s

    def forward(self, x):
        sc = self.s.to(x.dtype).repeat_interleave(128, dim=0).repeat_interleave(128, dim=1)
        return torch.matmul(x, (self.w.to(x.dtype) / sc).t())


def build(arm, layers, dev):
    import bench
    from gptqmodel_b200 import B200Fp8QuantLinear, B200QuantLinear

    stack = []
    for li in range(layers):
        mods = {}
        for j, (name, kk, nn_, _) in enumerate(bench.LINEARS):
            K, N = bench.CFG[kk], bench.CFG[nn_]
            seed = li * 16 + j
            if arm == "gptq8_b200":
                qw, qz, sc, gi = gptq8_tensors(K, N, seed, dev)
                mods[name] = B200QuantLinear.from_checkpoint_tensors(qw, qz, sc, gi, 8, 128, device=dev)
            else:
                w, s = fp8_tensors(K, N, seed, dev)
                mods[name] = (B200Fp8QuantLinear.from_checkpoint_tensors(w, s, device=dev) if arm == "fp8_b200"
                              else TorchFp8(w, s))
        stack.append(mods)
    torch.cuda.empty_cache()
    return stack


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_fp8.json"))
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_bench: needs a CUDA device (no CPU timing is meaningful here)")
    torch.cuda.set_device(0)
    import bench
    from hadamard_bench import card

    dev = torch.device("cuda:0")
    _, weights = bench.stack_bytes_and_weights(bench.CFG, args.layers)
    arms = {}
    for a in ("fp8_b200", "gptq8_b200"):
        arms[a] = build(a, args.layers, dev)
    # the torch arm shares nothing with the others: one layer's weights per pass would not stream 6.5 GB; build it from
    # the fp8 arm's tensors instead (same bytes, same values)
    arms["fp8_torch"] = [{n: TorchFp8(m.weight, m.weight_scale_inv) for n, m in mods.items()} for mods in arms["fp8_b200"]]
    res = {"card": card(), "layers": args.layers, "rounds": args.rounds, "siblings_fused": False, "dtype": "fp16",
           "block": [128, 128], "ms": {str(M): {a: [] for a in arms} for M, _ in STEPS}}
    for _ in range(args.rounds):
        for M, iters in STEPS:
            for a, stack in arms.items():
                n = iters if a != "fp8_torch" else max(2, iters // 20)
                ms, fin = bench.time_stack(stack, M, 1, dev, n, bench.CFG["hidden"])
                assert fin, (a, M)
                res["ms"][str(M)][a].append(round(ms, 4))
                print(json.dumps({"M": M, "arm": a, "ms": round(ms, 4)}), flush=True)
    med = {M: {a: statistics.median(v) for a, v in d.items()} for M, d in res["ms"].items()}
    res["decode_tok_s"] = {a: round(1e3 / ms, 1) for a, ms in med["1"].items()}
    res["step16_tok_s"] = {a: round(16e3 / ms, 1) for a, ms in med["16"].items()}
    res["step64_tok_s"] = {a: round(64e3 / ms, 1) for a, ms in med["64"].items()}
    res["prefill2048_tflops"] = {a: round(2.0 * 2048 * weights / (ms * 1e-3) / 1e12, 1) for a, ms in med["2048"].items()}
    for M, key in (("1", "decode"), ("16", "step16"), ("64", "step64"), ("2048", "prefill2048")):
        res[f"{key}_ratio_fp8_over_gptq8"] = round(med[M]["gptq8_b200"] / med[M]["fp8_b200"], 3)
        res[f"{key}_speedup_fp8_over_torch"] = round(med[M]["fp8_torch"] / med[M]["fp8_b200"], 2)
    print(json.dumps({k: v for k, v in res.items() if k != "ms"}), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
