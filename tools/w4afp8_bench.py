#!/usr/bin/env python
"""Measure W4AFP8 layers on one GPU.

    python tools/w4afp8_bench.py --out results/h100_w4afp8.json

The 32-layer Llama-3-8B linear stack of bench.py (its shapes and run order, fp16 activations, no sibling fusion; one
module per linear, shared by the layers), arms:
  * w4afp8      : B200W4Fp8Linear, 4-bit group-128 weights, dynamic per-token e4m3 activations (compressed-tensors W4AFP8);
  * fp8_dynamic : B200ChannelFp8Linear, per-channel e4m3 weights, dynamic per-token activations (FP8_DYNAMIC);
  * gptq4_b200  : this project's 4-bit GPTQ g128 B200QuantLinear (bench.py's layers, W4A16);
  * qqq_g128    : B200QqqQuantLinear, 4-bit group-128 weights, per-token int8 activations (QQQ W4A8).
Before any timing the w4afp8 arm's output at every timed token count is checked bit for bit against the layer's two
launches (b2q_fp8ch_quantize + b2q_w4afp8_mm) on the 4096 x 4096 layer.  Decode tok/s (1 token), 16- and 64-token steps
(tokens/s) and 2048-token prefill TFLOP/s counting 2*M*K*N; every pass is one CUDA graph timed with CUDA events, the arms
alternate within each round and the medians of the rounds are reported.  The card's name, power limit and SM clock are
read in the same run and stored with the numbers.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from fp8_w8a8_bench import card_now, fp8_tensors  # noqa: E402
from qqq_bench import qqq_canonical  # noqa: E402

STEPS = ((1, 200), (16, 100), (64, 50), (2048, 5))  # (tokens, graph replays per timing)
ARMS = ("w4afp8", "fp8_dynamic", "gptq4_b200", "qqq_g128")
# The layers of the timed stack share one module per linear (see main), so a pass multiplies by the same matrices 32
# times and would overflow along their top singular vectors.  Every arm's weight scales are multiplied by GAIN < 1,
# which makes the pass decay instead; the kernels' time does not depend on the values.
GAIN = 0.25


def w4afp8_tensors(K, N, seed, dev):
    """weight_packed int32 [N, K/8] of codes uniform in q = -7..7 (zero mean, so no rank-one component grows through
    the stack) and bf16 group scales [N, K/128] with W of rms ~ GAIN / sqrt(K)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    c = torch.randint(1, 16, (N, K), device=dev, generator=g, dtype=torch.int32)
    wp = torch.zeros((N, K // 8), dtype=torch.int32, device=dev)
    for i in range(8):
        wp |= c[:, i::8] << (4 * i)
    ws = ((0.8 + 0.4 * torch.rand(N, K // 128, device=dev, generator=g)) * GAIN / (4.3 * K ** 0.5)).to(torch.bfloat16)
    return wp, ws


def make(arm, K, N, seed, dev, gain=GAIN):
    import bench
    from gptqmodel_b200 import B200ChannelFp8Linear, B200QqqQuantLinear, B200QuantLinear, B200W4Fp8Linear
    from oracle import qqq_oracle as qo

    if arm == "w4afp8":
        wp, ws = w4afp8_tensors(K, N, seed, dev)
        return B200W4Fp8Linear.from_checkpoint_tensors(wp, ws, device=dev)
    if arm == "fp8_dynamic":
        w, s = fp8_tensors(K, N, seed, dev)
        return B200ChannelFp8Linear.from_checkpoint_tensors(w, s * gain, device=dev)
    if arm == "gptq4_b200":
        L = bench.synth_layer(K, N, seed=seed, device=dev)
        return B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"] * gain, L["g_idx"], 4,
                                                      128, device=dev)
    codes, sc, sg = qqq_canonical(K, N, 128, seed, dev)
    B, scp, sgp = qo.pack_qqq(codes, sc * gain, sg)
    return B200QqqQuantLinear.from_checkpoint_tensors(B, scp, sgp, 128, device=dev)


def check_layer(dev):
    """The w4afp8 arm at every timed M on the 4096 x 4096 layer equals quantise + mm bit for bit."""
    from gptqmodel_b200 import lib
    from gptqmodel_b200._lib import check

    K = N = 4096
    m = make("w4afp8", K, N, 1, dev)
    out = {}
    st = torch.cuda.current_stream().cuda_stream
    for M, _ in STEPS:
        x = (torch.randn(M, K, device=dev) * 0.5).to(torch.float16)
        codes = torch.empty((M, K), dtype=torch.uint8, device=dev)
        sx = torch.empty(M, dtype=torch.float32, device=dev)
        want = torch.empty((M, N), dtype=torch.float16, device=dev)
        check(lib.b2q_fp8ch_quantize(x.data_ptr(), codes.data_ptr(), sx.data_ptr(), M, K, float("inf"), 0, st), "q")
        check(lib.b2q_w4afp8_mm(codes.data_ptr(), sx.data_ptr(), m.packed.data_ptr(), m.s_w.data_ptr(), None,
                                want.data_ptr(), M, K, N, 0, 0, st), "mm")
        assert torch.equal(m(x), want), M
        out[f"w4afp8@{M}"] = "bit-exact"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_w4afp8.json"))
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("w4afp8_bench: needs a CUDA device (no CPU timing is meaningful here)")
    torch.cuda.set_device(0)
    import bench

    dev = torch.device("cuda:0")
    _, weights = bench.stack_bytes_and_weights(bench.CFG, args.layers)
    res = {"card": card_now(), "layers": args.layers, "rounds": args.rounds, "siblings_fused": False, "dtype": "fp16",
           "arms": list(ARMS), "layers_share_modules": True, "weight_scale_gain": GAIN}
    res["layer_check"] = check_layer(dev)
    print(json.dumps({"layer_check": res["layer_check"]}), flush=True)
    torch.cuda.empty_cache()
    # one module per (arm, linear), shared by every layer of the stack: a layer's weights (>= 109 MB at 4 bits) exceed
    # the 50 MB L2, so the next layer's reads come from HBM as with distinct weights, and building 32 QQQ layers with
    # the host-side packer would take minutes
    arms = {a: [] for a in ARMS}
    for a in ARMS:
        mods = {n: make(a, bench.CFG[kk], bench.CFG[nn_], j, dev) for j, (n, kk, nn_, _) in enumerate(bench.LINEARS)}
        arms[a] = [mods] * args.layers
        print(json.dumps({"built": a}), flush=True)
    torch.cuda.empty_cache()
    res["ms"] = {str(M): {a: [] for a in ARMS} for M, _ in STEPS}
    for _ in range(args.rounds):
        for M, iters in STEPS:
            for a in ARMS:
                ms, fin = bench.time_stack(arms[a], M, 1, dev, iters, bench.CFG["hidden"])
                assert fin, (a, M)
                res["ms"][str(M)][a].append(round(ms, 4))
                print(json.dumps({"M": M, "arm": a, "ms": round(ms, 4)}), flush=True)
    med = {M: {a: statistics.median(v) for a, v in d.items()} for M, d in res["ms"].items()}
    res["decode_tok_s"] = {a: round(1e3 / ms, 1) for a, ms in med["1"].items()}
    res["step16_tok_s"] = {a: round(16e3 / ms, 1) for a, ms in med["16"].items()}
    res["step64_tok_s"] = {a: round(64e3 / ms, 1) for a, ms in med["64"].items()}
    res["prefill2048_tflops"] = {a: round(2.0 * 2048 * weights / (ms * 1e-3) / 1e12, 1) for a, ms in med["2048"].items()}
    res["w4afp8_speedup"] = {other: {M: round(med[M][other] / med[M]["w4afp8"], 3) for M in med}
                             for other in ARMS if other != "w4afp8"}
    # goals: decode >= 1.3x fp8_dynamic and > qqq_g128; 16 / 64 tokens >= fp8_dynamic; prefill >= 1.2x gptq4_b200
    # and >= 0.85x fp8_dynamic
    sp = res["w4afp8_speedup"]
    res["goals"] = {"decode_vs_fp8_dynamic>=1.3": sp["fp8_dynamic"]["1"] >= 1.3,
                    "decode_vs_qqq_g128>1": sp["qqq_g128"]["1"] > 1.0,
                    "step16_vs_fp8_dynamic>=1": sp["fp8_dynamic"]["16"] >= 1.0,
                    "step64_vs_fp8_dynamic>=1": sp["fp8_dynamic"]["64"] >= 1.0,
                    "prefill_vs_gptq4>=1.2": sp["gptq4_b200"]["2048"] >= 1.2,
                    "prefill_vs_fp8_dynamic>=0.85": sp["fp8_dynamic"]["2048"] >= 0.85}
    res["card_after"] = card_now()
    print(json.dumps({k: v for k, v in res.items() if k != "ms"}), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
