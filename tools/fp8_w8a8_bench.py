#!/usr/bin/env python
"""Measure per-channel / per-tensor FP8 (W8A8) layers on one GPU.

    python tools/fp8_w8a8_bench.py --out results/h100_fp8_w8a8.json

The 32-layer Llama-3-8B linear stack of bench.py (its shapes and run order, fp16 activations, no sibling fusion), arms:
  * ch_dynamic       : B200ChannelFp8Linear, per-channel weights, dynamic per-token activations (FP8_DYNAMIC);
  * ch_static        : B200ChannelFp8Linear, one per-tensor weight scale, a static input_scale (compressed-tensors FP8);
  * ch_fbgemm_ub     : B200ChannelFp8Linear, per-channel weights, per-token activations with ub = 1200 (fbgemm_fp8);
  * fp8blk_b200      : B200BlockFp8Linear on the same e4m3 bytes with 128 x 128 block scales;
  * fp8_w8a16        : B200Fp8QuantLinear on the same e4m3 bytes (16-bit activations);
  * gptq4_b200       : this project's 4-bit GPTQ g128 B200QuantLinear (bench.py's layers, W4A16);
  * scaled_mm_row    : torch._scaled_mm with row-wise scales (activations quantised by b2q_fp8ch_quantize), and
  * scaled_mm_tensor : torch._scaled_mm with tensor-wise scales (static activations, b2q_fp8ch_quantize_static),
                       where the build offers them.
Before any timing each new arm's output at every timed token count is checked against the float64 oracle (the bound of
tests/test_gpu_fp8_w8a8.py) on the 4096 x 4096 layer.  Decode tok/s (1 token), 16- and 64-token steps (tokens/s) and
2048-token prefill TFLOP/s counting 2*M*K*N; every pass is one CUDA graph timed with CUDA events, the arms alternate
within each round.  The card's name, power limit and SM clock are read in the same run and stored with the numbers.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

STEPS = ((1, 200), (16, 100), (64, 50), (2048, 5))  # (tokens, graph replays per timing)
SHAPES = ((4096, 6144), (4096, 4096), (4096, 28672), (14336, 4096))  # qkv, o, gate+up, down (K, N)
NEW = ("ch_dynamic", "ch_static", "ch_fbgemm_ub")
S_IN = 0.5 / 448 * 8  # static input scale: the bench's activations (randn * 0.5 through the stack) stay well inside it
UB = 1200.0


def card_now():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_sm_clock_max_sm_clock"] = r.stdout.strip().splitlines()[0]
    except Exception as e:  # the number is still valid, the card's limit is then unknown
        info["power_limit_sm_clock_max_sm_clock"] = f"unavailable ({e})"
    return info


def fp8_tensors(K, N, seed, dev):
    """e4m3 codes [N, K], per-channel scales [N, 1] and block-128 scales with W = w * s of rms ~ 1 / sqrt(K)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    w = (torch.randn(N, K, device=dev, generator=g) * 64.0).clamp(-448, 448).to(torch.float8_e4m3fn)
    s = (0.8 + 0.4 * torch.rand(N, 1, device=dev, generator=g)) / (64.0 * K ** 0.5)
    return w, s


class ScaledMM(torch.nn.Module):
    """torch._scaled_mm on codes of this project's quantisers: row-wise (per-token x per-channel) or tensor-wise."""

    def __init__(self, w, s, rowwise):
        super().__init__()
        self.w, self.rowwise = w, rowwise
        self.s = s.reshape(1, -1).float().contiguous() if rowwise else s.float().max().reshape(()).contiguous()
        self.s_in = torch.tensor([S_IN], dtype=torch.float32, device=w.device)

    def forward(self, x):
        from gptqmodel_b200 import lib

        M, K = x.shape
        codes = torch.empty((M, K), dtype=torch.uint8, device=x.device)
        sx = torch.empty(M, dtype=torch.float32, device=x.device)
        st = torch.cuda.current_stream().cuda_stream
        if self.rowwise:
            lib.b2q_fp8ch_quantize(x.data_ptr(), codes.data_ptr(), sx.data_ptr(), M, K, float("inf"), 0, st)
            return torch._scaled_mm(codes.view(torch.float8_e4m3fn), self.w.t(), scale_a=sx[:, None], scale_b=self.s,
                                    out_dtype=torch.bfloat16).to(x.dtype)
        lib.b2q_fp8ch_quantize_static(x.data_ptr(), self.s_in.data_ptr(), codes.data_ptr(), sx.data_ptr(), M, K, 0, st)
        return torch._scaled_mm(codes.view(torch.float8_e4m3fn), self.w.t(), scale_a=self.s_in.reshape(()),
                                scale_b=self.s, out_dtype=x.dtype)


def make(arm, K, N, seed, dev, w=None, s=None):
    import bench
    from gptqmodel_b200 import B200BlockFp8Linear, B200ChannelFp8Linear, B200Fp8QuantLinear, B200QuantLinear

    if arm == "gptq4_b200":
        L = bench.synth_layer(K, N, seed=seed, device=dev)
        return B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, 128,
                                                      device=dev)
    if w is None:
        w, s = fp8_tensors(K, N, seed, dev)
    if arm == "ch_dynamic":
        return B200ChannelFp8Linear.from_checkpoint_tensors(w, s, device=dev)
    if arm == "ch_fbgemm_ub":
        return B200ChannelFp8Linear.from_checkpoint_tensors(w, s, ub=UB, device=dev)
    if arm == "ch_static":
        return B200ChannelFp8Linear.from_checkpoint_tensors(w, s.max().reshape(1), device=dev,
                                                            input_scale=torch.tensor([S_IN], device=dev))
    # one scale per 128 x 128 block, drawn like the channel scales (an amax would grow the activations layer by layer)
    blk = s.reshape(N // 128, 128)[:, :1].expand(N // 128, K // 128).contiguous()
    if arm == "fp8blk_b200":
        return B200BlockFp8Linear.from_checkpoint_tensors(w, blk, device=dev)
    if arm == "fp8_w8a16":
        return B200Fp8QuantLinear.from_checkpoint_tensors(w, 1.0 / blk, device=dev)
    return ScaledMM(w, s, rowwise=arm == "scaled_mm_row")


def scaled_mm_available(arm, dev):
    try:
        make(arm, 256, 256, 0, dev)(torch.randn(16, 256, device=dev, dtype=torch.float16))
        torch.cuda.synchronize()
        return True
    except Exception as e:  # noqa: BLE001
        print(json.dumps({arm: f"unavailable: {type(e).__name__}: {str(e)[:200]}"}), flush=True)
        return False


def check_against_oracle(dev):
    """Each new arm at every timed M on the 4096 x 4096 layer within the float64 accumulator bound; worst ratios."""
    import fp8_w8a8_mirror as fm

    K = N = 4096
    w, s = fp8_tensors(K, N, 1, dev)
    out = {}
    for arm in NEW:
        m = make(arm, K, N, 1, dev, w, s)
        for M, _ in STEPS:
            x = (torch.randn(M, K, device=dev) * 0.5).to(torch.float16)
            y = m(x).double().cpu().numpy()
            xf = x.float().cpu().numpy()
            if arm == "ch_static":
                codes, sx = fm.quantize_static(xf, np.float32(S_IN))
            else:
                codes, sx = fm.quantize_dynamic(xf, UB if arm == "ch_fbgemm_ub" else np.inf)
            ref, mag = fm.reference(codes, sx, m.weight.view(torch.uint8).cpu().numpy(), m.weight_scale.cpu().numpy())
            tol = 2.0 ** -10 * np.abs(ref) + 2.0 ** -24 + 2.0 ** -10 * mag
            ratio = float((np.abs(y - ref) / tol).max())
            assert ratio <= 1.0, (arm, M, ratio)
            out[f"{arm}@{M}"] = round(ratio, 4)
    return out


def time_graph(fn, calls=20, reps=7):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            fn()
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
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_fp8_w8a8.json"))
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_w8a8_bench: needs a CUDA device (no CPU timing is meaningful here)")
    torch.cuda.set_device(0)
    import bench

    dev = torch.device("cuda:0")
    _, weights = bench.stack_bytes_and_weights(bench.CFG, args.layers)
    torch_arms = [a for a in ("scaled_mm_row", "scaled_mm_tensor") if scaled_mm_available(a, dev)]
    names = list(NEW) + ["fp8blk_b200", "fp8_w8a16", "gptq4_b200"] + torch_arms
    res = {"card": card_now(), "layers": args.layers, "rounds": args.rounds, "siblings_fused": False, "dtype": "fp16",
           "arms": names, "static_input_scale": S_IN, "fbgemm_ub": UB}
    res["oracle_worst_ratio"] = check_against_oracle(dev)
    print(json.dumps({"oracle_worst_ratio": res["oracle_worst_ratio"]}), flush=True)
    torch.cuda.empty_cache()
    arms = {a: [] for a in names}
    for li in range(args.layers):
        for a in names:
            arms[a].append({})
        for j, (n, kk, nn_, _) in enumerate(bench.LINEARS):
            K, N = bench.CFG[kk], bench.CFG[nn_]
            w, s = fp8_tensors(K, N, li * 16 + j, dev)  # every FP8 arm reads the same e4m3 bytes
            for a in names:
                arms[a][li][n] = make(a, K, N, li * 16 + j, dev, w, s)
    torch.cuda.empty_cache()
    res["ms"] = {str(M): {a: [] for a in arms} for M, _ in STEPS}
    for _ in range(args.rounds):
        for M, iters in STEPS:
            for a, stack in arms.items():
                ms, fin = bench.time_stack(stack, M, 1, dev, iters, bench.CFG["hidden"])
                assert fin, (a, M)
                res["ms"][str(M)][a].append(round(ms, 4))
                print(json.dumps({"M": M, "arm": a, "ms": round(ms, 4)}), flush=True)
    med = {M: {a: statistics.median(v) for a, v in d.items()} for M, d in res["ms"].items()}
    res["decode_tok_s"] = {a: round(1e3 / ms, 1) for a, ms in med["1"].items()}
    res["step16_tok_s"] = {a: round(16e3 / ms, 1) for a, ms in med["16"].items()}
    res["step64_tok_s"] = {a: round(64e3 / ms, 1) for a, ms in med["64"].items()}
    res["prefill2048_tflops"] = {a: round(2.0 * 2048 * weights / (ms * 1e-3) / 1e12, 1) for a, ms in med["2048"].items()}
    res["ratio_over_fp8blk"] = {a: {M: round(med[M]["fp8blk_b200"] / med[M][a], 3) for M in med} for a in NEW}
    if "scaled_mm_row" in names:
        res["prefill_ratio_over_scaled_mm_row"] = {a: round(med["2048"]["scaled_mm_row"] / med["2048"][a], 3)
                                                   for a in NEW}
    res["card_after"] = card_now()
    print(json.dumps({k: v for k, v in res.items() if k != "ms"}), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
