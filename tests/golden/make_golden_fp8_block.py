#!/usr/bin/env python
"""Golden fixtures for HF / DeepSeek-native block-FP8 checkpoints.  Weights and scales come from transformers'
``Fp8Quantize`` (the FineGrainedFP8 quantiser, run on CPU), the dequantised weights from the UNMODIFIED reference's
``dequantize_fp8`` (gptqmodel/quantization/dtype.py, ``scale_inv=s, axis=None``).

Needs a GPTQModel source checkout ($GPTQMODEL_SRC, see make_golden.py) and transformers; the tests only read the
committed output:

    python tests/golden/make_golden_fp8_block.py

Output (committed): tests/golden/fp8_block_cases.npz, for every case name c:
  * c.weight (uint8 e4m3fn bit patterns [N, K]) / c.scale_inv (fp32 [N/128, K/128]) : Fp8Quantize of a random layer;
  * c.W16 / c.Wbf ([K, N]) : the reference's dequantize_fp8, transposed;
  * c.x16 / c.xbf ([M, K]) and c.y16 / c.ybf (x @ W in float64, stored as float32, [M, N]).
fp16 arrays are stored as float16, bf16 arrays as their uint16 bit patterns (numpy has no bf16): two bytes per value
keep the file small.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import _StubFinder, _shell, REF_ROOT  # noqa: E402

# (name, K, N, M)
CASES = (("small", 256, 128, 5), ("tall", 256, 256, 3), ("wide", 512, 128, 7))


def _store(t: torch.Tensor) -> np.ndarray:
    """fp16 -> float16 array, bf16 -> uint16 bit patterns."""
    return t.numpy() if t.dtype == torch.float16 else t.view(torch.int16).numpy().view(np.uint16)


def main():
    from transformers.integrations.finegrained_fp8 import Fp8Quantize

    sys.meta_path.append(_StubFinder())
    g = _shell("gptqmodel", REF_ROOT + "/gptqmodel")
    g.DEBUG_ON = False
    _shell("gptqmodel.quantization", REF_ROOT + "/gptqmodel/quantization")
    from gptqmodel.quantization.dtype import dequantize_fp8

    class _Q:  # the quantizer object Fp8Quantize reads its block size from
        quantization_config = {"weight_block_size": [128, 128]}

    out = {}
    gen = torch.Generator().manual_seed(20261017)
    for name, K, N, M in CASES:
        W = torch.randn(N, K, generator=gen) * 0.02
        W[:, 5] *= 40.0  # an outlier input column
        W[:128, 128:256] *= 1e-3  # a block with a tiny absmax: a small scale
        r = Fp8Quantize(_Q()).convert({"m.weight": [W]})
        q, s = r["m.weight"], r["m.weight_scale_inv"]
        assert bool((s <= 1).all()), "the fixtures keep every scale <= 1 (the reference multiplies there)"
        p = name + "."
        out[p + "weight"] = q.view(torch.uint8).numpy()
        out[p + "scale_inv"] = s.numpy()
        for tag, dt in (("16", torch.float16), ("bf", torch.bfloat16)):
            Wdq = dequantize_fp8(q, scale_inv=s, axis=None, target_dtype=dt).transpose(0, 1).contiguous()
            x = (torch.randn(M, K, generator=gen) * 0.5).to(dt)
            y = x.double() @ Wdq.double()
            out[p + "W" + tag] = _store(Wdq)
            out[p + "x" + tag] = _store(x)
            out[p + "y" + tag] = y.float().numpy()
        print(f"{name}: K={K} N={N} M={M}")
    np.savez_compressed(os.path.join(HERE, "fp8_block_cases.npz"), **out)
    print("wrote fp8_block_cases.npz")


if __name__ == "__main__":
    main()
