#!/usr/bin/env python
"""Measure the QQQ (W4A8) tier on one GPU.

    python tools/qqq_bench.py --out results/h100_qqq.json

1. Per-shape kernel times for the four Llama-3-8B linear shapes at M in {1, 8, 16, 64, 128, 2048}: the activation
   quantiser, the int8 GEMM and the two together (b2q_qqq_forward), against this project's W4A16 b2q_mm (4-bit g128)
   and, when oracle/build_qqq.py built it, the reference's own qqq_gemm.  Arms are timed alternately in the same
   process; each number is CUDA events over a CUDA graph of many launches.  For M <= 128 the launches cycle over enough
   copies of the weights to exceed the 50 MB L2, so every launch streams its weights from HBM.
2. The 32-layer Llama-3-8B linear stack of bench.py (its shapes and run order), QQQ (g128) against W4A16 (g128), both
   without sibling fusion: decode tok/s (1 token) and 2048-token prefill TFLOP/s counting 2*M*K*N.
The card's name and power limit are read in the same run and stored with the numbers.
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

SHAPES = ((4096, 4096), (4096, 1024), (4096, 14336), (14336, 4096))  # q/o, k/v, gate/up, down
MS = (1, 8, 16, 64, 128, 2048)
L2_BYTES = 50 * 2 ** 20
REF_SO = os.path.join(ROOT, "oracle", "_ref", "gptqmodel_qqq.so")


def graph_us(launch, ncopies, launches=60, reps=5):
    """µs per launch: CUDA events around the replay of a graph of `launches` calls cycling over the weight copies."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(2):
            launch(i % ncopies)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(launches):
            launch(i % ncopies)
    g.replay()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        t.append(e0.elapsed_time(e1) * 1e3 / launches)
    return statistics.median(t)


def qqq_canonical(K, N, gs, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    codes = torch.randint(1, 16, (K, N), device=dev, generator=g, dtype=torch.int32).to(torch.uint8)
    sg = (torch.rand(K // 128, N, device=dev, generator=g) * 14.9 + 1.0).to(torch.float16) if gs == 128 else None
    wrms = 40.0 if gs == 128 else 74.0  # rms of the int8 weights: keeps the chained activations O(1)
    sc = (0.8 + 0.4 * torch.rand(N, device=dev, generator=g)) / (wrms * K ** 0.5)
    return codes, sc.float(), sg


def qqq_module(K, N, gs, seed, dev):
    from gptqmodel_b200 import B200QqqQuantLinear
    from oracle import qqq_oracle as qo

    codes, sc, sg = qqq_canonical(K, N, gs, seed, dev)
    B, scp, sgp = qo.pack_qqq(codes, sc, sg)
    return B200QqqQuantLinear.from_checkpoint_tensors(B, scp, sgp if gs == 128 else None, gs, device=dev), (B, scp, sgp)


def shape_arms(K, N, M, gs, rounds, ref_op):
    import bench
    import gptqmodel_b200 as g
    from gptqmodel_b200 import B200QuantLinear

    dev = torch.device("cuda:0")
    stream = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731
    mod, (B, scp, sgp) = qqq_module(K, N, gs, K + N, dev)
    L = bench.synth_layer(K, N, seed=K * 3 + N, device=dev, gs=128)
    w16 = B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, 128, device=dev)
    ncopies = 1 if M > 128 else max(1, -(-3 * L2_BYTES // (K * N // 2)))
    qp = [mod.packed] + [mod.packed.clone() for _ in range(ncopies - 1)]
    wp = [w16.packed] + [w16.packed.clone() for _ in range(ncopies - 1)]
    x = (torch.randn(M, K, device=dev) * 0.5).half()
    y = torch.empty(M, N, dtype=torch.float16, device=dev)
    ws = torch.empty(g.lib.b2q_qqq_workspace_bytes(M, K), dtype=torch.uint8, device=dev)
    Kp = (K + 127) // 128 * 128
    st = ws[: (M * 4 + 127) // 128 * 128].view(torch.float32)[:M]
    q = ws[(M * 4 + 127) // 128 * 128:].view(torch.int8)
    sgp_ptr = None if mod._sg is None else mod._sg.data_ptr()

    def quant(i):
        g.check(g.lib.b2q_qqq_quantize(x.data_ptr(), q.data_ptr(), st.data_ptr(), M, K, 0, stream()), "quantize")

    def gemm(i):
        g.check(g.lib.b2q_qqq_mm(q.data_ptr(), st.data_ptr(), qp[i].data_ptr(), mod._sc.data_ptr(), sgp_ptr, None,
                                 y.data_ptr(), M, K, N, gs, 0, stream()), "qqq_mm")

    def total(i):
        g.check(g.lib.b2q_qqq_forward(x.data_ptr(), qp[i].data_ptr(), mod._sc.data_ptr(), sgp_ptr, None, y.data_ptr(),
                                      M, K, N, gs, 0, 0, ws.data_ptr(), ws.numel(), stream()), "qqq_forward")

    def w4a16(i):
        g.check(g.lib.b2q_mm(x.data_ptr(), wp[i].data_ptr(), w16.scales.data_ptr(), None, None, None, y.data_ptr(), M, K,
                             N, 4, 128, 0, None, 0, stream()), "b2q_mm")

    arms = {"qqq_quant": quant, "qqq_gemm": gemm, "qqq_total": total, "w4a16": w4a16}
    if ref_op is not None:
        rB = [B.to(dev)] + [B.to(dev) for _ in range(ncopies - 1)]
        rs2, rs3 = scp.to(dev), sgp.to(dev)
        C = torch.zeros(16 * 64, N, dtype=torch.int32, device=dev)
        rws = torch.zeros(N // 128 * 16, dtype=torch.int32, device=dev)
        qa = q[: M * Kp].view(M, Kp)[:, :K]
        qa = qa.contiguous() if Kp != K else qa
        s1 = st.view(M, 1)

        def ref(i):
            ref_op(qa, rB[i], C, y, s1, rs2, rs3, rws, -1, -1, -1, 16)

        quant(0)
        arms["reference_qqq_gemm"] = ref
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(graph_us(fn, ncopies))
    out = {"K": K, "N": N, "M": M, "group_size": gs, "weight_copies": ncopies}
    out.update({k + "_us": round(statistics.median(v), 3) for k, v in res.items()})
    out["speedup_total_vs_w4a16"] = round(out["w4a16_us"] / out["qqq_total_us"], 3)
    if "reference_qqq_gemm_us" in out:
        out["speedup_gemm_vs_reference"] = round(out["reference_qqq_gemm_us"] / out["qqq_gemm_us"], 3)
    out["qqq_total_tops"] = round(2.0 * M * K * N / (out["qqq_total_us"] * 1e-6) / 1e12, 1)
    return out


def qqq_stack(layers, gs, dev):
    import bench
    from gptqmodel_b200 import B200QqqQuantLinear

    base = {}
    for j, (name, kk, nn_, _) in enumerate(bench.LINEARS):
        K, N = bench.CFG[kk], bench.CFG[nn_]
        if (K, N) not in base:
            base[(K, N)] = qqq_module(K, N, gs, j, dev)[1]
    stack = []
    for _ in range(layers):  # distinct packed weights per layer (post_init repacks every module)
        mods = {}
        for name, kk, nn_, _ in bench.LINEARS:
            K, N = bench.CFG[kk], bench.CFG[nn_]
            B, scp, sgp = base[(K, N)]
            mods[name] = B200QqqQuantLinear.from_checkpoint_tensors(B, scp, sgp if gs == 128 else None, gs, device=dev)
        stack.append(mods)
    torch.cuda.empty_cache()
    return stack


def stack_arms(layers, rounds):
    import bench

    dev = torch.device("cuda:0")
    _, weights = bench.stack_bytes_and_weights(bench.CFG, layers)
    arms = {"w4a16": bench.build_stack(dev, 0, 1, layers, fuse=False), "qqq_g128": qqq_stack(layers, 128, dev)}
    res = {"layers": layers, "rounds": rounds, "siblings_fused": False,
           "decode_ms": {a: [] for a in arms}, "prefill2048_ms": {a: [] for a in arms}}
    for _ in range(rounds):
        for a, stack in arms.items():
            ms, fin = bench.time_stack(stack, 1, 1, dev, 200, bench.CFG["hidden"])
            assert fin, a
            res["decode_ms"][a].append(round(ms, 4))
            ms, fin = bench.time_stack(stack, 2048, 1, dev, 10, bench.CFG["hidden"])
            assert fin, a
            res["prefill2048_ms"][a].append(round(ms, 4))
    med = {k: {a: statistics.median(v) for a, v in res[k].items()} for k in ("decode_ms", "prefill2048_ms")}
    res["decode_tok_s"] = {a: round(1e3 / ms, 1) for a, ms in med["decode_ms"].items()}
    res["prefill_tflops"] = {a: round(2.0 * 2048 * weights / (ms * 1e-3) / 1e12, 1)
                             for a, ms in med["prefill2048_ms"].items()}
    res["decode_ratio_qqq_over_w4a16"] = round(med["decode_ms"]["w4a16"] / med["decode_ms"]["qqq_g128"], 3)
    res["prefill_ratio_qqq_over_w4a16"] = round(med["prefill2048_ms"]["w4a16"] / med["prefill2048_ms"]["qqq_g128"], 3)
    res["quantiser_us_per_layer_decode"] = "see kernel[].qqq_quant_us at M = 1 (7 launches per layer)"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_qqq.json"))
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-stack", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("qqq_bench: needs a CUDA device (no CPU timing is meaningful here)")
    torch.cuda.set_device(0)
    from hadamard_bench import card

    ref_op = None
    if os.path.exists(REF_SO):
        torch.ops.load_library(REF_SO)
        ref_op = torch.ops.gptqmodel_qqq.qqq_gemm
    out = {"card": card(), "reference_kernel": "built" if ref_op is not None else "not built (oracle/build_qqq.py)"}
    out["kernel"] = [shape_arms(K, N, M, gs, args.rounds, ref_op) for gs in (128, -1) for K, N in SHAPES for M in MS]
    for r in out["kernel"]:
        print(json.dumps(r), flush=True)
    if not args.skip_stack:
        out["stack"] = stack_arms(args.layers, args.rounds)
        print(json.dumps(out["stack"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
