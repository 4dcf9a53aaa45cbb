#!/usr/bin/env python
"""Golden fixtures for QQQ (W4A8) checkpoints, produced by the UNMODIFIED reference's ``QQQTorchLinear``
(gptqmodel/nn_modules/qlinear/qqq.py).

Needs a GPTQModel source checkout ($GPTQMODEL_SRC, see make_golden.py); the tests only read the committed output:

    python tests/golden/make_golden_qqq.py

Output (committed): tests/golden/qqq_cases.npz, for every case name c:
  * c.B / c.s_channel / c.s_group / c.bias : the output of ``pack()`` (s_group empty for per-channel layers);
  * c.codes / c.s_ch_canon / c.s_grp_canon  : the canonical layer the case was built from (our fixture recipe);
  * c.weight / c.weight_s_channel           : ``_dequantize_weight_for_torch()`` (weight integer-valued, as int8);
  * c.x16 / c.xbf (fp16 / as float32)       : inputs with outlier columns and an all-zero row;
  * c.q16 / c.s16, c.qbf / c.sbf            : ``dynamic_quant()`` codes and scales of fp16(x16) and fp16(xbf);
  * c.y16 / c.ybf (fp16 / as float32)       : ``QQQTorchLinear.forward`` outputs for the fp16 and bf16 inputs.
K <= 1024 keeps every partial sum below 2^24, so the reference's fp32 matmul is exact.
"""
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import _StubFinder, _shell, REF_ROOT  # noqa: E402

# (name, group_size, K, N, M, bias)
CASES = (
    ("ch", -1, 512, 256, 9, False),
    ("ch_bias", -1, 320, 128, 6, True),
    ("g128", 128, 1024, 128, 9, False),
    ("g128_bias", 128, 512, 192, 5, True),
)


def _inputs(gen, M, K, dtype):
    x = torch.randn(M, K, generator=gen) * 0.5
    x[:, 3] *= 40.0    # outlier columns
    x[:, K - 5] *= -25.0
    x[M // 2] = 0.0    # an all-zero row
    return x.to(dtype)


def main():
    sys.meta_path.append(_StubFinder())
    g = _shell("gptqmodel", REF_ROOT + "/gptqmodel")
    g.DEBUG_ON = False
    _shell("gptqmodel.models", REF_ROOT + "/gptqmodel/models")
    from gptqmodel.nn_modules.qlinear.qqq import QQQTorchLinear

    out = {}
    gen = torch.Generator().manual_seed(20261016)
    for name, gs, K, N, M, has_bias in CASES:
        mod = QQQTorchLinear(bits=4, group_size=gs, desc_act=False, sym=True, in_features=K, out_features=N,
                             bias=has_bias)
        lin = nn.Linear(K, N, bias=has_bias)
        s_ch = (torch.rand(N, generator=gen) * 0.009 + 0.001)
        if gs == -1:
            c = torch.randint(-7, 8, (K, N), generator=gen)                       # signed codes
            scales = s_ch.to(torch.float16).reshape(N, 1)
            w = (c.to(torch.float32) * scales.to(torch.float32).reshape(1, N))
            lin.weight.data = w.t().contiguous().to(torch.float16)
            mod.pack(lin, scales)
            codes = (c & 0xF).to(torch.uint8)
            s_ch_canon = scales.to(torch.float32).reshape(N) / 16.0
            s_grp_canon = np.zeros((0,), np.float16)
        else:
            G = K // gs
            c = torch.randint(0, 16, (K, N), generator=gen)                      # unsigned codes, zero point 8
            u = torch.rand(N, G, generator=gen) * 14.9 + 1.0                      # s_group in [1, 15.9]
            scales = (s_ch.reshape(N, 1) * u).to(torch.float16)
            sgf = scales.to(torch.float32).t().repeat_interleave(gs, dim=0)       # [K, N]
            lin.weight.data = ((c.to(torch.float32) - 8.0) * sgf).t().contiguous().to(torch.float16)
            mod.pack(lin, scales, s_extra=s_ch.reshape(1, N))
            codes = c.to(torch.uint8)
            s_ch_canon = s_ch.to(torch.float32)
            s_grp_canon = (scales.to(torch.float32).t() / s_ch.reshape(1, N)).to(torch.float16).numpy()
        if has_bias:
            mod.bias = (torch.randn(N, generator=gen) * 0.1).to(torch.float16)
        weight, wsc = mod._dequantize_weight_for_torch()
        p = name + "."
        out[p + "B"] = mod.B.numpy()
        out[p + "s_channel"] = mod.s_channel.numpy()
        out[p + "s_group"] = mod.s_group.numpy()
        out[p + "bias"] = mod.bias.numpy() if has_bias else np.zeros((0,), np.float16)
        out[p + "codes"] = codes.numpy()
        out[p + "s_ch_canon"] = s_ch_canon.numpy()
        out[p + "s_grp_canon"] = s_grp_canon
        assert torch.equal(weight, weight.to(torch.int8).to(torch.float32))
        out[p + "weight"] = weight.to(torch.int8).numpy()      # integer-valued, stored exactly as int8
        out[p + "weight_s_channel"] = wsc.numpy()
        for tag, dt in (("16", torch.float16), ("bf", torch.bfloat16)):
            x = _inputs(gen, M, K, dt)
            q, s = mod.dynamic_quant(x.to(torch.float16))
            y = mod.forward(x)
            keep = torch.float16 if dt == torch.float16 else torch.float32  # (numpy has no bf16; exact in fp32)
            out[p + "x" + tag] = x.to(keep).numpy()
            out[p + "q" + tag] = q.numpy()
            out[p + "s" + tag] = s.reshape(-1).numpy()
            out[p + "y" + tag] = y.to(keep).numpy()
        print(f"{name}: K={K} N={N} M={M} group_size={gs} bias={has_bias}")
    np.savez_compressed(os.path.join(HERE, "qqq_cases.npz"), **out)
    print("wrote qqq_cases.npz")


if __name__ == "__main__":
    main()
