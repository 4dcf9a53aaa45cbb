#!/usr/bin/env python
"""Measure per-channel INT8 (W8A8) layers on one GPU.

    python tools/int8_w8a8_bench.py --out results/h100_int8_w8a8.json

The 32-layer Llama-3-8B linear stack of bench.py (its shapes and run order, fp16 activations, no sibling fusion), arms:
  * int8_dynamic : B200ChannelInt8Linear, per-channel weights, dynamic per-token activations (compressed-tensors W8A8);
  * int8_static  : B200ChannelInt8Linear, per-channel weights, a static per-tensor input_scale;
  * fp8_dynamic  : B200ChannelFp8Linear, per-channel e4m3 weights of the same size, dynamic per-token activations;
  * gptq4_b200   : this project's 4-bit GPTQ g128 B200QuantLinear (bench.py's layers, W4A16);
  * int_mm       : torch._int_mm on this package's int8 codes (b2q_int8ch_quantize) and weights, the scales applied in
                   torch; only at the token counts _int_mm accepts (M > 16).
Before any timing each int8 arm's output at every timed token count is checked bit for bit against
tests/int8_w8a8_mirror.py on the 4096 x 4096 layer.  Decode tok/s (1 token), 16- and 64-token steps (tokens/s) and
2048-token prefill TFLOP/s counting 2*M*K*N; every pass is one CUDA graph timed with CUDA events, the arms alternate
within each round and the medians of the rounds are reported.  The card's name, power limit and SM clock are read in the
same run and stored with the numbers.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from fp8_w8a8_bench import card_now, fp8_tensors  # noqa: E402

STEPS = ((1, 200), (16, 100), (64, 50), (2048, 5))  # (tokens, graph replays per timing)
NEW = ("int8_dynamic", "int8_static")
S_IN = 4.0 / 127  # static input scale: the bench's activations (randn * 0.5 through the stack) stay inside it


def int8_tensors(K, N, seed, dev):
    """int8 codes [N, K] and per-channel scales [N, 1] with W = w * s of rms ~ 1 / sqrt(K)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    w = torch.randint(-127, 128, (N, K), device=dev, generator=g, dtype=torch.int8)
    s = (0.8 + 0.4 * torch.rand(N, 1, device=dev, generator=g)) / (73.0 * K ** 0.5)
    return w, s


class IntMM(torch.nn.Module):
    """torch._int_mm on this package's per-token codes, y = (acc * s_x * s_w) in fp32, rounded to fp16."""

    def __init__(self, w, s):
        super().__init__()
        self.wt, self.s = w.t(), s.reshape(1, -1).float().contiguous()

    def forward(self, x):
        from gptqmodel_b200 import lib

        M, K = x.shape
        codes = torch.empty((M, K), dtype=torch.int8, device=x.device)
        sx = torch.empty(M, dtype=torch.float32, device=x.device)
        lib.b2q_int8ch_quantize(x.data_ptr(), codes.data_ptr(), sx.data_ptr(), M, K, 0,
                                torch.cuda.current_stream().cuda_stream)
        return (torch._int_mm(codes, self.wt).float() * (sx[:, None] * self.s)).to(x.dtype)


def make(arm, K, N, seed, dev, w8, s8, wf, sf):
    import bench
    from gptqmodel_b200 import B200ChannelFp8Linear, B200ChannelInt8Linear, B200QuantLinear

    if arm == "gptq4_b200":
        L = bench.synth_layer(K, N, seed=seed, device=dev)
        return B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, 128,
                                                      device=dev)
    if arm == "int8_dynamic":
        return B200ChannelInt8Linear.from_checkpoint_tensors(w8, s8, device=dev)
    if arm == "int8_static":
        return B200ChannelInt8Linear.from_checkpoint_tensors(w8, s8, device=dev,
                                                             input_scale=torch.tensor([S_IN], device=dev))
    if arm == "fp8_dynamic":
        return B200ChannelFp8Linear.from_checkpoint_tensors(wf, sf, device=dev)
    return IntMM(w8, s8)


def check_against_mirror(dev):
    """Each int8 arm at every timed M on the 4096 x 4096 layer equals the mirror bit for bit."""
    import int8_w8a8_mirror as im

    K = N = 4096
    w, s = int8_tensors(K, N, 1, dev)
    out = {}
    for arm in NEW:
        m = make(arm, K, N, 1, dev, w, s, None, None)
        for M, _ in STEPS:
            x = (torch.randn(M, K, device=dev) * 0.5).to(torch.float16)
            xf = x.float().cpu().numpy()
            codes, sx = im.quantize_static(xf, np.float32(S_IN)) if arm == "int8_static" else im.quantize_dynamic(xf)
            want = im.epilogue(im.int_sums(codes, w.cpu().numpy()), sx, m.weight_scale.cpu().numpy(), None, "fp16")
            assert torch.equal(m(x).float().cpu(), torch.from_numpy(want)), (arm, M)
            out[f"{arm}@{M}"] = "bit-exact"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_int8_w8a8.json"))
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("int8_w8a8_bench: needs a CUDA device (no CPU timing is meaningful here)")
    torch.cuda.set_device(0)
    import bench

    dev = torch.device("cuda:0")
    _, weights = bench.stack_bytes_and_weights(bench.CFG, args.layers)
    names = list(NEW) + ["fp8_dynamic", "gptq4_b200", "int_mm"]
    res = {"card": card_now(), "layers": args.layers, "rounds": args.rounds, "siblings_fused": False, "dtype": "fp16",
           "arms": names, "static_input_scale": S_IN, "int_mm_tokens": [M for M, _ in STEPS if M > 16]}
    res["mirror_check"] = check_against_mirror(dev)
    print(json.dumps({"mirror_check": res["mirror_check"]}), flush=True)
    torch.cuda.empty_cache()
    arms = {a: [] for a in names}
    for li in range(args.layers):
        for a in names:
            arms[a].append({})
        for j, (n, kk, nn_, _) in enumerate(bench.LINEARS):
            K, N = bench.CFG[kk], bench.CFG[nn_]
            w8, s8 = int8_tensors(K, N, li * 16 + j, dev)
            wf, sf = fp8_tensors(K, N, li * 16 + j, dev)
            for a in names:
                arms[a][li][n] = make(a, K, N, li * 16 + j, dev, w8, s8, wf, sf)
    torch.cuda.empty_cache()
    res["ms"] = {str(M): {a: [] for a in arms if a != "int_mm" or M > 16} for M, _ in STEPS}
    for _ in range(args.rounds):
        for M, iters in STEPS:
            for a in res["ms"][str(M)]:
                ms, fin = bench.time_stack(arms[a], M, 1, dev, iters, bench.CFG["hidden"])
                assert fin, (a, M)
                res["ms"][str(M)][a].append(round(ms, 4))
                print(json.dumps({"M": M, "arm": a, "ms": round(ms, 4)}), flush=True)
    med = {M: {a: statistics.median(v) for a, v in d.items()} for M, d in res["ms"].items()}
    res["decode_tok_s"] = {a: round(1e3 / ms, 1) for a, ms in med["1"].items()}
    res["step16_tok_s"] = {a: round(16e3 / ms, 1) for a, ms in med["16"].items()}
    res["step64_tok_s"] = {a: round(64e3 / ms, 1) for a, ms in med["64"].items()}
    res["prefill2048_tflops"] = {a: round(2.0 * 2048 * weights / (ms * 1e-3) / 1e12, 1) for a, ms in med["2048"].items()}
    # target: >= 0.95 at every token count (same bytes and tensor-core peak, no per-block promotion)
    res["ratio_over_fp8_dynamic"] = {a: {M: round(med[M]["fp8_dynamic"] / med[M][a], 3) for M in med} for a in NEW}
    # target: >= 1.0 at prefill
    res["ratio_over_int_mm"] = {a: {M: round(med[M]["int_mm"] / med[M][a], 3) for M in med if "int_mm" in med[M]}
                                for a in NEW}
    res["card_after"] = card_now()
    print(json.dumps({k: v for k, v in res.items() if k != "ms"}), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
