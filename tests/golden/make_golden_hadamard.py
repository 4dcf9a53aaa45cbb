#!/usr/bin/env python
"""Golden fixtures for the online Hadamard transform of rotated (QuaRot / SpinQuant) checkpoints, produced by the
UNMODIFIED reference.

Needs a GPTQModel source checkout ($GPTQMODEL_SRC, see make_golden.py); the tests only read the committed output:

    python tests/golden/make_golden_hadamard.py

Output (committed): tests/golden/hadamard_cases.npz with
  * had{K}            : the reference's +-1 matrices of order K (gptqmodel/quantization/rotation/hadamard_utils.py
                        get_had12 ... get_had172) as int8 [K, K];
  * hadK.n / hadK.K   : get_hadK(n)[1] for a list of n, K = -1 where get_hadK raises (n is not K times a power of two);
  * case{i}.x / .y    : float64 inputs and the reference's matmul_hadU(x) for a few small (K, n).
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import _StubFinder, _shell, REF_ROOT  # noqa: E402

ORDERS = (12, 20, 28, 36, 40, 52, 60, 108, 140, 156, 172)
# n for the order rule: the Llama / Qwen / Mistral intermediate sizes, powers of two, every order at small P, numbers
# divisible by two orders (the rule's precedence), and sizes no order serves
SIZES = (8192, 11008, 14336, 28672, 13824, 17920, 18944, 5632, 4096, 1024, 64, 96, 160, 224, 288, 320, 416, 480, 864,
         1120, 1248, 1376, 2240, 3440, 5120, 6144, 2560, 3072, 12288, 24, 48, 200, 1000, 4097, 14000, 100, 33)
CASES = ((12, 96), (36, 288), (28, 224), (172, 1376), (1, 64), (40, 320))


def main():
    sys.meta_path.append(_StubFinder())
    g = _shell("gptqmodel", REF_ROOT + "/gptqmodel")
    g.DEBUG_ON = False
    _shell("gptqmodel.models", REF_ROOT + "/gptqmodel/models")
    from gptqmodel.quantization.rotation import hadamard_utils as hu

    blobs = {}
    for K in ORDERS:
        m = getattr(hu, f"get_had{K}")()
        assert m.shape == (K, K) and bool(((m == 1) | (m == -1)).all())
        blobs[f"had{K}"] = m.to(torch.int8).numpy()
    ks = []
    for n in SIZES:
        try:
            ks.append(int(hu.get_hadK(n)[1]))
        except AssertionError:
            ks.append(-1)
    blobs["hadK.n"] = np.array(SIZES, dtype=np.int64)
    blobs["hadK.K"] = np.array(ks, dtype=np.int64)
    for i, (K, n) in enumerate(CASES):
        gen = torch.Generator().manual_seed(9100 + i)
        x = torch.randn(3, n, generator=gen, dtype=torch.float64)
        x[:, ::17] *= 100.0  # outlier channels
        assert hu.get_hadK(n)[1] == K
        y = hu.matmul_hadU(x)
        blobs[f"case{i}.x"] = x.numpy()
        blobs[f"case{i}.y"] = y.numpy()
    blobs["__meta__"] = np.frombuffer(json.dumps({"cases": CASES, "orders": ORDERS}).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(HERE, "hadamard_cases.npz"), **blobs)
    print("wrote hadamard_cases.npz", dict(zip(SIZES, ks)))


if __name__ == "__main__":
    main()
