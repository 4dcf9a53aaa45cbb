#!/usr/bin/env python
"""Measure block-FP8 (HF / DeepSeek-native, W8A8) layers on one GPU.

    python tools/fp8_block_bench.py --out results/h100_fp8_block.json

The 32-layer Llama-3-8B linear stack of bench.py (its shapes and run order, fp16 activations, no sibling fusion), arms:
  * fp8blk_b200 : B200BlockFp8Linear (b2q_fp8blk_forward: e4m3 activations, e4m3 wgmma);
  * fp8_w8a16   : B200Fp8QuantLinear on the same e4m3 bytes and block-128 scales (16-bit activations, b2q_fp8_mm);
  * gptq4_b200  : this project's 4-bit GPTQ g128 B200QuantLinear (bench.py's layers, W4A16);
  * fp8_torch   : torch dequantise (w * s) + matmul every call;
  * scaled_mm   : torch.nn.functional.scaled_mm with BlockWise1x128 x BlockWise128x128 scales, where the build offers it
                  (activations quantised by b2q_fp8blk_quantize).
Decode tok/s (1 token), 16- and 64-token steps (tokens/s) and 2048-token prefill TFLOP/s counting 2*M*K*N; every pass is
one CUDA graph timed with CUDA events, the arms alternate within each round.  Per-shape kernel times of the four Llama
shapes at M = 1 / 16 / 2048 come from CUDA events around graphs of 20 calls.  The card's name and power limit are read
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
SHAPES = ((4096, 6144), (4096, 4096), (4096, 28672), (14336, 4096))  # qkv, o, gate+up, down (K, N)


def fp8_tensors(K, N, seed, dev):
    """e4m3 codes [N, K] and block-128 scales (multipliers) with W = w * s of rms ~ 1 / sqrt(K)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    w = (torch.randn(N, K, device=dev, generator=g) * 64.0).clamp(-448, 448).to(torch.float8_e4m3fn)
    s = (0.8 + 0.4 * torch.rand(N // 128, K // 128, device=dev, generator=g)) / (64.0 * K ** 0.5)
    return w, s


class TorchDequant(torch.nn.Module):
    def __init__(self, w, s):
        super().__init__()
        self.w, self.s = w, s

    def forward(self, x):
        sc = self.s.to(x.dtype).repeat_interleave(128, dim=0).repeat_interleave(128, dim=1)
        return torch.matmul(x, (self.w.to(x.dtype) * sc).t())


class ScaledMM(torch.nn.Module):
    def __init__(self, w, s):
        super().__init__()
        self.w, self.s = w, s.t().contiguous().t()

    def forward(self, x):
        from gptqmodel_b200 import lib

        M, K = x.shape
        codes = torch.empty((M, K), dtype=torch.uint8, device=x.device)
        mp = (M + 3) // 4 * 4
        sx = torch.empty((K // 128, mp), dtype=torch.float32, device=x.device)
        lib.b2q_fp8blk_quantize(x.data_ptr(), codes.data_ptr(), sx.data_ptr(), M, K, 0,
                                torch.cuda.current_stream().cuda_stream)
        F = torch.nn.functional
        return F.scaled_mm(codes.view(torch.float8_e4m3fn), self.w.t(), scale_a=sx[:, :M].t(),
                           scale_recipe_a=F.ScalingType.BlockWise1x128, scale_b=self.s,
                           scale_recipe_b=F.ScalingType.BlockWise128x128, output_dtype=x.dtype)


def make(arm, K, N, seed, dev):
    import bench
    from gptqmodel_b200 import B200BlockFp8Linear, B200Fp8QuantLinear, B200QuantLinear

    if arm == "gptq4_b200":
        L = bench.synth_layer(K, N, seed=seed, device=dev)
        return B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, 128,
                                                      device=dev)
    w, s = fp8_tensors(K, N, seed, dev)
    if arm == "fp8blk_b200":
        return B200BlockFp8Linear.from_checkpoint_tensors(w, s, device=dev)
    if arm == "fp8_w8a16":
        return B200Fp8QuantLinear.from_checkpoint_tensors(w, 1.0 / s, device=dev)
    return ScaledMM(w, s) if arm == "scaled_mm" else TorchDequant(w, s)


def scaled_mm_available(dev):
    try:
        m = make("scaled_mm", 256, 256, 0, dev)
        m(torch.randn(16, 256, device=dev, dtype=torch.float16))
        torch.cuda.synchronize()
        return True
    except Exception as e:  # noqa: BLE001
        print(json.dumps({"scaled_mm": f"unavailable: {type(e).__name__}: {str(e)[:200]}"}), flush=True)
        return False


def time_calls(mod, M, K, dev, calls=20, reps=5):
    x = (torch.randn(M, K, device=dev) * 0.5).to(torch.float16)
    for _ in range(2):
        mod(x)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            mod(x)
    g.replay()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) * 1e3 / calls)
    del g
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_fp8_block.json"))
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_block_bench: needs a CUDA device (no CPU timing is meaningful here)")
    torch.cuda.set_device(0)
    import bench
    from hadamard_bench import card

    dev = torch.device("cuda:0")
    _, weights = bench.stack_bytes_and_weights(bench.CFG, args.layers)
    names = ["fp8blk_b200", "fp8_w8a16", "gptq4_b200", "fp8_torch"] + (["scaled_mm"] if scaled_mm_available(dev) else [])
    res = {"card": card(), "layers": args.layers, "rounds": args.rounds, "siblings_fused": False, "dtype": "fp16",
           "block": [128, 128], "arms": names}
    # per-shape kernel times (one module per shape, CUDA events around a graph of 20 calls)
    res["shape_us"] = {}
    for K, N in SHAPES:
        for M in (1, 16, 2048):
            row = {}
            for a in names:
                if a == "fp8_torch" and M != 2048:
                    continue
                mod = make(a, K, N, seed=K + N, dev=dev)
                row[a] = round(time_calls(mod, M, K, dev), 2)
                del mod
            res["shape_us"][f"{K}x{N}@{M}"] = row
            print(json.dumps({"shape": f"{K}x{N}", "M": M, "us": row}), flush=True)
    torch.cuda.empty_cache()
    arms = {}
    for a in names:
        if a in ("fp8_torch", "scaled_mm"):
            continue
        arms[a] = [{n: make(a, bench.CFG[kk], bench.CFG[nn_], li * 16 + j, dev)
                    for j, (n, kk, nn_, _) in enumerate(bench.LINEARS)} for li in range(args.layers)]
    # the torch arms read the block arm's tensors (same bytes, same values)
    for a, cls in (("fp8_torch", TorchDequant), ("scaled_mm", ScaledMM)):
        if a in names:
            arms[a] = [{n: cls(m.weight, m.weight_scale_inv) for n, m in mods.items()} for mods in arms["fp8blk_b200"]]
    torch.cuda.empty_cache()
    res["ms"] = {str(M): {a: [] for a in arms} for M, _ in STEPS}
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
        res[f"{key}_ratio_over_w8a16"] = round(med[M]["fp8_w8a16"] / med[M]["fp8blk_b200"], 3)
        res[f"{key}_ratio_over_gptq4"] = round(med[M]["gptq4_b200"] / med[M]["fp8blk_b200"], 3)
    print(json.dumps({k: v for k, v in res.items() if k not in ("ms", "shape_us")}), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
