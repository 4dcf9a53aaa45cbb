#!/usr/bin/env python
"""Golden fixtures for FP8 (e4m3fn) checkpoints, produced by the UNMODIFIED reference's ``quantize_fp8_weight``,
``TorchFP8Linear`` and ``FP8Config`` (gptqmodel/nn_modules/qlinear/fp8.py, gptqmodel/quantization/config.py).

Needs a GPTQModel source checkout ($GPTQMODEL_SRC, see make_golden.py); the tests only read the committed output:

    python tests/golden/make_golden_fp8.py

Output (committed): tests/golden/fp8_cases.npz, for every case name c:
  * c.weight (uint8 e4m3fn bit patterns [N, K]) / c.scale_inv (fp32) : quantize_fp8_weight() of a random layer;
  * c.bias (fp16, empty without bias), c.method / c.block : the FP8Config-normalised scale layout;
  * c.W16 / c.Wbf (fp16 / bf16 as float32) : the CUDA branch of TorchFP8Linear.dequantize_weight (weight.to(T) /
    _expanded_scale_inv(T), transposed), run on CPU tensors;
  * c.x16 / c.xbf, c.y16 / c.ybf : inputs and torch.matmul(x, W) + bias in T (the reference's dequant-matmul forward).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import _StubFinder, _shell, REF_ROOT  # noqa: E402

# (name, config kwargs, K, N, M, bias)
CASES = (
    ("tensor", dict(weight_scale_method="tensor"), 256, 128, 5, True),
    ("row", dict(), 384, 96, 7, False),
    ("row_bias", dict(weight_scale_method="row"), 256, 64, 4, True),
    ("block128", dict(weight_scale_method="block", weight_block_size=[128, 128]), 512, 256, 6, True),
    ("block64", dict(weight_scale_method="block", weight_block_size=[64, 64]), 256, 192, 5, False),
)


def main():
    sys.meta_path.append(_StubFinder())
    g = _shell("gptqmodel", REF_ROOT + "/gptqmodel")
    g.DEBUG_ON = False
    _shell("gptqmodel.models", REF_ROOT + "/gptqmodel/models")
    from gptqmodel.nn_modules.qlinear.fp8 import TorchFP8Linear, quantize_fp8_weight
    from gptqmodel.quantization.config import FP8Config

    out = {}
    gen = torch.Generator().manual_seed(20261016)
    for name, kw, K, N, M, has_bias in CASES:
        cfg = FP8Config(format="e4m3", **kw)  # the reference's normalisation (alias, method, block size)
        block = tuple(cfg.weight_block_size) if cfg.weight_block_size is not None else None
        W = torch.randn(N, K, generator=gen) * 0.05
        W[:, 7] *= 30.0  # an outlier input column
        if block is not None:
            W[: block[0], : block[1]] *= 1e-3  # one block with a tiny absmax: a large scale_inv
        q, sinv = quantize_fp8_weight(W, format=cfg.format, weight_scale_method=cfg.weight_scale_method,
                                      weight_block_size=block)
        mod = TorchFP8Linear(bits=8, group_size=-1, sym=True, desc_act=False, in_features=K, out_features=N,
                             bias=has_bias, format=cfg.format, weight_scale_method=cfg.weight_scale_method,
                             weight_block_size=block, weight_scale_semantics=cfg.weight_scale_semantics)
        mod.weight = q
        mod.weight_scale_inv = sinv
        bias = (torch.randn(N, generator=gen) * 0.1).to(torch.float16) if has_bias else None
        p = name + "."
        out[p + "weight"] = q.view(torch.uint8).numpy()
        out[p + "scale_inv"] = sinv.numpy()
        out[p + "bias"] = bias.numpy() if has_bias else np.zeros((0,), np.float16)
        out[p + "method"] = np.array(cfg.weight_scale_method)
        out[p + "block"] = np.array(block if block is not None else (0, 0), np.int64)
        for tag, dt in (("16", torch.float16), ("bf", torch.bfloat16)):
            keep = torch.float16 if dt == torch.float16 else torch.float32  # (numpy has no bf16; exact in fp32)
            Wdq = (mod.weight.to(dt) / mod._expanded_scale_inv(target_device=torch.device("cpu"), target_dtype=dt))
            Wdq = Wdq.transpose(0, 1).contiguous()
            x = (torch.randn(M, K, generator=gen) * 0.5).to(dt)
            y = torch.matmul(x, Wdq)
            if has_bias:
                y = y + bias.to(dt)
            out[p + "W" + tag] = Wdq.to(keep).numpy()
            out[p + "x" + tag] = x.to(keep).numpy()
            out[p + "y" + tag] = y.to(keep).numpy()
        print(f"{name}: K={K} N={N} M={M} method={cfg.weight_scale_method} block={block} bias={has_bias}")
    np.savez_compressed(os.path.join(HERE, "fp8_cases.npz"), **out)
    print("wrote fp8_cases.npz")


if __name__ == "__main__":
    main()
