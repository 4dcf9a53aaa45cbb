"""Competitor kernels on the SAME box, SAME packed checkpoint tensors (VERDICT r01 row g).

  python tools/competitors.py [--json gpurun_out/competitors.json] [--quick]

Arms (each reported as available / unavailable with the reason):
  * "marlin_ref"  — the reference's own Marlin (gptqmodel_ext/marlin) compiled by oracle/build_marlin.py from a GPTQModel
                    checkout into oracle/_ref/ (git-ignored); call sequence restates
                    MarlinLinear.post_init / forward (qlinear/marlin.py:246-337, utils/marlin.py:471-608).
  * "marlin_vllm" — vLLM 0.22's build of the same kernel family (torch.ops._C.marlin_gemm): library code in the image.
  * "cublas_fp16" — dense fp16 torch.matmul on the dequantised weights (context only: 4x the bytes at M=1).
  * "b2q"         — this repo, through B200QuantLinear.forward.
Every arm first checks its output against this repo's output on the same input (rtol/atol 2e-3 fp16: Marlin rounds
(q-8)*s per weight, like the oracle); a mismatching arm is reported as such and not timed.
Per-shape time is the mean over a CUDA graph that walks `copies` DISTINCT layers (weights >> L2 at M <= 64).
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gptqmodel_b200 import B200QuantLinear  # noqa: E402
from helpers import random_layer  # noqa: E402

SHAPES = [(4096, 4096), (4096, 1024), (4096, 14336), (14336, 4096)]
# Llama-3-8B per decoder layer: q, k, v, o, gate, up, down
STACK = [(4096, 4096), (4096, 1024), (4096, 1024), (4096, 4096), (4096, 14336), (4096, 14336), (14336, 4096)]


def time_graph(fn, iters=20):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        fn()
    for _ in range(3):
        gr.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        gr.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3  # us per graph replay


# ------------------------------------------------------------------------------------------------- arms
class MarlinVllm:
    name = "marlin_vllm"

    def __init__(self):
        t0 = time.time()
        from vllm import _custom_ops as ops
        from vllm.model_executor.layers.quantization.utils import marlin_utils as mu
        from vllm.scalar_type import scalar_types
        self.ops, self.mu, self.st = ops, mu, scalar_types
        self.ws = torch.zeros(132 * 4, dtype=torch.int32, device="cuda")
        self.empty = torch.empty(0, dtype=torch.int32, device="cuda")
        self.info = f"vllm {__import__('vllm').__version__} torch.ops._C.marlin_gemm (import {time.time() - t0:.0f}s)"

    def prepare(self, L):
        K, N, gs = L["K"], L["N"], L["group_size"]
        qw = self.ops.gptq_marlin_repack(L["qweight"].contiguous(), self.empty, K, N, 4)
        sc = self.mu.marlin_permute_scales(L["scales"].contiguous(), K, N, gs)
        return (qw, sc, K, N)

    def run(self, h, x):
        qw, sc, K, N = h
        return self.ops.marlin_gemm(x, None, qw, None, sc, None, None, self.empty, self.empty, self.empty, self.ws,
                                    self.st.uint4b8, x.shape[0], N, K, True, False, True, False)


class MarlinRef:
    """The reference's Marlin, built by oracle/build_marlin.py (op schema: marlin_torch_fp16.cpp)."""
    name = "marlin_ref"

    def __init__(self):
        so = os.path.join(ROOT, "oracle", "_ref", "gptqmodel_marlin_fp16.so")
        if not os.path.exists(so):
            raise RuntimeError(f"{so} not built (GPTQMODEL_SRC=<GPTQModel checkout> python oracle/build_marlin.py)")
        torch.ops.load_library(so)
        self.ns = torch.ops.gptqmodel_marlin_fp16
        # workspace: int32[max(SMs, 128)] zeros (utils/marlin.py:308-319)
        self.ws = torch.zeros(max(torch.cuda.get_device_properties(0).multi_processor_count, 128) * 4,
                              dtype=torch.int32, device="cuda")
        self.empty = torch.empty(0, dtype=torch.int32, device="cuda")
        self.info = "reference gptqmodel_ext/marlin compiled for sm_90a (oracle/build_marlin.py)"

    @staticmethod
    def _permute_scales(s, K, N, gs):
        # utils/marlin.py:373-399 (scale_perm: 8x8 interleave for grouped, single-row permutation for channelwise)
        scale_perm = [i + 8 * j for i in range(8) for j in range(8)]
        scale_perm_single = [2 * i + j for i in range(4) for j in (0, 1, 8, 9, 16, 17, 24, 25)]
        if gs < K and gs != -1:
            s = s.reshape(-1, 64)[:, scale_perm]
        else:
            s = s.reshape(-1, 32)[:, scale_perm_single]
        return s.reshape(-1, N).contiguous()

    def prepare(self, L):
        K, N, gs = L["K"], L["N"], L["group_size"]
        qw = self.ns.gptq_marlin_repack(L["qweight"].contiguous(), self.empty, K, N, 4)
        sc = self._permute_scales(L["scales"].contiguous(), K, N, gs)
        return (qw, sc, K, N)

    def run(self, h, x):
        qw, sc, K, N = h
        U4B8 = _scalar_type_id_u4b8()
        return self.ns.gptq_marlin_gemm_fp16(x, None, qw, None, sc, None, None, self.empty, self.empty, self.ws, U4B8,
                                             x.shape[0], N, K, True, False, True, False)


def _scalar_type_id_u4b8():
    # core/scalar_type.hpp ScalarType::id(): bit-packed {exponent:8, mantissa:8, signed:1, bias:32, finite_values_only:1,
    # nan_repr:8}; uint4b8 = ScalarType::uint(4, bias 8) -> exponent 0, mantissa 4, signed 0, bias 8, and the constructor's
    # DEFAULT nan_repr = NAN_IEEE_754 (1) also for integer types (scalar_type.hpp:37-40)
    exponent, mantissa, signed, bias = 0, 4, 0, 8
    v, off = 0, 0
    for val, width in ((exponent, 8), (mantissa, 8), (signed, 1), (bias, 32), (0, 1), (1, 8)):
        v |= (val & ((1 << width) - 1)) << off
        off += width
    return v


class B2Q:
    name = "b2q"
    info = "this repo (B200QuantLinear.forward -> b2q_mm)"

    def prepare(self, L):
        return B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4,
                                                       L["group_size"], device="cuda")

    def run(self, h, x):
        return h(x)


class Cublas:
    name = "cublas_fp16"
    info = "torch.matmul on the dense fp16 weights (dequantised once)"

    def prepare(self, L):
        m = B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4,
                                                    L["group_size"], device="cuda")
        return m.dequantize_weight().contiguous()

    def run(self, h, x):
        return x @ h


# ------------------------------------------------------------------------------------------------- driver
ARM_CLASSES = {}


def run(arm_names=("b2q", "marlin_ref", "marlin_vllm", "cublas_fp16"), Ms=(1, 16, 64, 2048), nlayers=32, stack=True,
        verbose=True):
    """-> dict: per-shape microseconds at every M and whole-stack decode tok/s / prefill TFLOP/s per arm (same box, same
    packed checkpoint tensors).  Used stand-alone and by bench.py's `competitors` block."""
    for cls in (B2Q, MarlinRef, MarlinVllm, Cublas):
        ARM_CLASSES[cls.name] = cls
    res = {"gpu": torch.cuda.get_device_name(torch.cuda.current_device()), "arms": {}, "per_shape_us": {}, "stack": {}}
    arms = []
    for name in arm_names:
        try:
            a = ARM_CLASSES[name]()
            arms.append(a)
            res["arms"][name] = {"available": True, "info": a.info}
        except Exception as e:  # noqa: BLE001
            res["arms"][name] = {"available": False, "why": f"{type(e).__name__}: {str(e)[:300]}"}
    if verbose:
        print(json.dumps(res["arms"], indent=1), flush=True)

    # ---- correctness of every arm against b2q on one layer, then per-shape timings
    for K, N in SHAPES:
        copies = max(2, min(24, int(600e6 // (K * N // 2))))  # >= 600 MB of distinct weights per graph
        layers = [random_layer(K, N, 4, 128, True, seed=c, device="cuda") for c in range(copies)]
        handles = {}
        for a in list(arms):
            try:
                handles[a.name] = [a.prepare(L) for L in layers]
            except Exception as e:  # noqa: BLE001
                res["arms"][a.name] = {"available": False, "why": f"prepare: {type(e).__name__}: {str(e)[:300]}"}
                arms.remove(a)
        for M in Ms:
            x = (torch.randn(M, K, device="cuda") * 0.5).to(torch.float16)
            yref = handles["b2q"][0](x) if "b2q" in handles else None
            for a in list(arms):
                key = f"{K}x{N}"
                try:
                    y = a.run(handles[a.name][0], x)
                    torch.cuda.synchronize()
                    if yref is not None and a.name != "b2q":
                        ok = torch.allclose(y.float(), yref.float(), rtol=4e-3, atol=4e-3 * yref.float().abs().max().item())
                        if not ok:
                            raise RuntimeError(f"output mismatch vs b2q: max abs diff "
                                               f"{(y.float() - yref.float()).abs().max().item():.3e}")
                    hs = handles[a.name]
                    us = time_graph(lambda: [a.run(h, x) for h in hs], iters=10) / len(hs)
                    res["per_shape_us"].setdefault(key, {}).setdefault(f"M{M}", {})[a.name] = round(us, 2)
                except Exception as e:  # noqa: BLE001
                    res["per_shape_us"].setdefault(key, {}).setdefault(f"M{M}", {})[a.name] = f"ERR {str(e)[:160]}"
            if verbose:
                print(K, N, M, res["per_shape_us"][f"{K}x{N}"][f"M{M}"], flush=True)
        del handles, layers
        torch.cuda.empty_cache()

    # ---- whole Llama-3-8B stack (32 x 7 QuantLinears, distinct weights): decode tok/s at M=1, prefill TFLOP/s at M=2048
    flops = 2 * 2048 * sum(k * n for k, n in STACK) * nlayers
    for a in (arms if stack else []):
        if a.name == "cublas_fp16":
            continue
        try:
            hs = []
            for li in range(nlayers):
                for j, (K, N) in enumerate(STACK):
                    hs.append((a.prepare(random_layer(K, N, 4, 128, True, seed=li * 7 + j, device="cuda")), K))
            out = {}
            for M, tag in ((1, "decode"), (2048, "prefill")):
                xs = {K: (torch.randn(M, K, device="cuda") * 0.5).to(torch.float16) for K in (4096, 14336)}
                us = time_graph(lambda: [a.run(h, xs[K]) for h, K in hs], iters=10 if M == 1 else 3)
                if tag == "decode":
                    out["decode_tok_s"] = round(1e6 / us * (32 / nlayers), 1)
                    out["decode_ms_per_token"] = round(us / 1e3 * (32 / nlayers), 4)
                else:
                    out["prefill_tflops"] = round(flops / (us * 1e-6) / 1e12, 1)
                    out["prefill_ms"] = round(us / 1e3 * (32 / nlayers), 3)
            out["note"] = "one launch per QuantLinear (224 per step), no sibling fusion, one CUDA graph"
            res["stack"][a.name] = out
            del hs
            torch.cuda.empty_cache()
        except Exception as e:  # noqa: BLE001
            res["stack"][a.name] = {"error": f"{type(e).__name__}: {str(e)[:300]}"}
        if verbose:
            print(a.name, res["stack"][a.name], flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=os.path.join(ROOT, "gpurun_out", "competitors.json"))
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--arms", default="b2q,marlin_ref,marlin_vllm,cublas_fp16")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    res = run(tuple(args.arms.split(",")), Ms=(1, 64) if args.quick else (1, 16, 64, 2048),
              nlayers=8 if args.quick else 32)
    os.makedirs(os.path.dirname(args.json), exist_ok=True)
    with open(args.json, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", args.json)


if __name__ == "__main__":
    main()
