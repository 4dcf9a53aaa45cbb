#!/usr/bin/env python
"""Generate golden fixtures by running the UNMODIFIED reference (read-only at /root/reference).

Run in the authoring container only (the GPU box has no /root/reference):

    python tests/golden/make_golden.py

Outputs (committed):
  tests/golden/q4_reference.json     the reference's own 1024-value golden vector
                                      (/root/reference/tests/q4_reference.py) + its recipe inputs
  tests/golden/ref_cases.npz         packed tensors, dequantised weights and forward outputs
                                      produced by the reference's TorchLinear / TorchAtenLinear

The reference package cannot be imported normally here (pcre, logbar, device_smi, tokenicer,
defuser, accelerate, torchao, parameterized are absent).  We import only the QuantLinear modules:
the missing third-party packages are satisfied by inert stub modules and the heavyweight
``gptqmodel/__init__.py`` and ``gptqmodel/models/__init__.py`` are skipped by registering
namespace shells for those two packages.  No reference code is modified or copied.
"""
import importlib
import importlib.machinery
import json
import os
import sys
import types

os.environ["CUDA_VISIBLE_DEVICES"] = ""
os.environ.setdefault("GPTQ_TORCH_TRITON_DEQUANT", "0")

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import transformers  # noqa: E402,F401
import transformers.modeling_utils  # noqa: E402,F401

from unittest.mock import MagicMock  # noqa: E402

REF_ROOT = os.environ.get("GPTQMODEL_SRC") or "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))


class _Stub(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return MagicMock(name=f"{self.__name__}.{name}")


class _StubFinder:
    PREFIXES = ("pcre", "logbar", "device_smi", "tokenicer", "defuser", "parameterized", "accelerate", "torchao")

    def find_spec(self, name, path=None, target=None):
        if name.split(".")[0] in self.PREFIXES:
            return importlib.machinery.ModuleSpec(name, self, is_package=True)
        return None

    def create_module(self, spec):
        m = _Stub(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, m):
        pass


def _shell(name, path):
    m = types.ModuleType(name)
    m.__path__ = [path]
    m.__spec__ = importlib.machinery.ModuleSpec(name, None, is_package=True)
    m.__spec__.submodule_search_locations = [path]
    sys.modules[name] = m
    return m


def import_reference():
    sys.meta_path.append(_StubFinder())
    g = _shell("gptqmodel", REF_ROOT + "/gptqmodel")
    g.DEBUG_ON = False
    _shell("gptqmodel.models", REF_ROOT + "/gptqmodel/models")
    from gptqmodel.nn_modules.qlinear.torch import TorchLinear
    from gptqmodel.nn_modules.qlinear.torch_aten_kernel import TorchAtenLinear

    return TorchLinear, TorchAtenLinear


def golden_q4_reference():
    """tests/q4_reference.py REFERENCE + the recipe of tests/test_q4_exllama_v2.py:32-87."""
    ns = {}
    with open(REF_ROOT + "/tests/q4_reference.py") as f:
        exec(compile(f.read(), "q4_reference.py", "exec"), ns)
    ref = ns["REFERENCE"]
    assert ref.numel() == 1024
    out = {
        "source": "ModelCloud/GPTQModel tests/q4_reference.py (REFERENCE), recipe tests/test_q4_exllama_v2.py:32-87",
        "recipe": {
            "seed": 42,
            "qweight": "torch.randint(-100, 100, (128, 1024), dtype=int32) after manual_seed(42)",
            "scales": 0.002,
            "qzeros_word": 0x11111111,
            "group_size": 128,
            "x": "torch.rand(1, 1, 1024, dtype=float16) drawn after qweight",
            "allclose": {"rtol": 3e-5, "atol": 2e-2},
        },
        "reference": [float(v) for v in ref.tolist()],
    }
    with open(os.path.join(HERE, "q4_reference.json"), "w") as f:
        json.dump(out, f)
    print("wrote q4_reference.json")


# (name, bits, group_size, sym, desc_act, K, N, M, bias)
CASES = [
    ("w4_g128_sym", 4, 128, True, False, 256, 128, 5, False),
    ("w4_g32_asym", 4, 32, False, False, 128, 64, 3, True),
    ("w4_g64_asym_act", 4, 64, False, True, 256, 64, 4, False),
    ("w4_g128_sym_act", 4, 128, True, True, 256, 128, 1, True),
    ("w4_gK_sym", 4, -1, True, False, 128, 64, 2, False),
    ("w8_g128_sym", 8, 128, True, False, 256, 64, 3, False),
    ("w8_g32_asym_act", 8, 32, False, True, 128, 64, 2, True),
]


def _quant_params(weight, bits, gs, sym, g_idx):
    """min/max grid quantiser (fixture generator, ours) -> scales/zeros [N, G] float."""
    N, K = weight.shape
    maxq = (1 << bits) - 1
    G = int(g_idx.max().item()) + 1
    scales = torch.zeros(N, G)
    zeros = torch.zeros(N, G)
    for g in range(G):
        blk = weight[:, g_idx == g]
        if sym:
            m = blk.abs().max(dim=1).values.clamp(min=1e-5)
            scales[:, g] = m / ((maxq + 1) // 2 - 1)
            zeros[:, g] = (maxq + 1) // 2
        else:
            lo = blk.min(dim=1).values.clamp(max=0)
            hi = blk.max(dim=1).values.clamp(min=0)
            sc = ((hi - lo) / maxq).clamp(min=1e-5)
            scales[:, g] = sc
            zeros[:, g] = torch.round(-lo / sc).clamp(0, maxq)
    return scales, zeros


def golden_ref_cases():
    TorchLinear, TorchAtenLinear = import_reference()
    blobs = {}
    meta = {}
    for i, (name, bits, gs, sym, desc_act, K, N, M, bias) in enumerate(CASES):
        torch.manual_seed(1000 + i)
        eff = gs if gs > 0 else K
        linear = nn.Linear(K, N, bias=bias)
        with torch.no_grad():
            linear.weight.copy_(torch.randn(N, K) * 0.5)
            if bias:
                linear.bias.copy_(torch.randn(N) * 0.1)
        if desc_act:
            perm = torch.randperm(K)
            g_idx = (torch.arange(K, dtype=torch.int32) // eff)[perm].contiguous()
        else:
            g_idx = torch.arange(K, dtype=torch.int32) // eff
        scales, zeros = _quant_params(linear.weight.data, bits, eff, sym, g_idx)

        def build(cls):
            m = cls(bits=bits, group_size=gs, sym=sym, desc_act=desc_act, in_features=K, out_features=N,
                    bias=bias, register_buffers=True)
            m.pack_block(linear, scales.clone(), zeros.clone(), g_idx.clone())
            return m

        mod = build(TorchLinear)
        # the two reference packers must agree bit-for-bit (tests/test_pack.py:114)
        mod2 = TorchLinear(bits=bits, group_size=gs, sym=sym, desc_act=desc_act, in_features=K, out_features=N,
                           bias=bias, register_buffers=True)
        mod2.pack_original(linear, scales.clone(), zeros.clone(), g_idx.clone())
        assert torch.equal(mod.qweight, mod2.qweight) and torch.equal(mod.qzeros, mod2.qzeros)
        # torch.compile of dequantize_weight (TorchLinear.optimize, torch.py:242-264) cannot build in this
        # container (no libgomp.spec) and does not change values: mark the instance as already optimised.
        mod.optimized = True
        mod.post_init()
        mod.eval()
        x16 = (torch.randn(M, K) * 0.5).to(torch.float16)
        xbf = x16.to(torch.bfloat16)
        with torch.inference_mode():
            W = mod.dequantize_weight().clone()
            y16 = mod(x16).clone()
            ybf = mod(xbf).clone()
        blobs[f"{name}.weight"] = linear.weight.data.numpy()
        if bias:
            blobs[f"{name}.lin_bias"] = linear.bias.data.numpy()
            blobs[f"{name}.bias"] = mod.bias.numpy()
        blobs[f"{name}.in_scales"] = scales.numpy()
        blobs[f"{name}.in_zeros"] = zeros.numpy()
        blobs[f"{name}.qweight"] = mod.qweight.numpy()
        blobs[f"{name}.qzeros"] = mod.qzeros.numpy()
        blobs[f"{name}.scales"] = mod.scales.numpy()
        blobs[f"{name}.g_idx"] = mod.g_idx.numpy()
        blobs[f"{name}.x"] = x16.numpy()
        blobs[f"{name}.W"] = W.numpy()
        blobs[f"{name}.y_fp16"] = y16.numpy()
        blobs[f"{name}.y_bf16"] = ybf.float().numpy()
        if bits == 4 and gs > 0:  # TorchAtenLinear supports group_size 16/32/64/128 only
            aten = build(TorchAtenLinear)
            aten.optimized = True
            aten.post_init()
            aten.eval()
            with torch.inference_mode():
                ya = aten(x16.clone()).clone()
            assert aten.linear_mode == "inference"
            blobs[f"{name}.y_cpu_fused"] = ya.float().numpy()
        meta[name] = dict(bits=bits, group_size=gs, sym=sym, desc_act=desc_act, K=K, N=N, M=M, bias=bias)
        print(name, "W", tuple(W.shape), W.dtype, "y", tuple(y16.shape))
    blobs["__meta__"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(HERE, "ref_cases.npz"), **blobs)
    print("wrote ref_cases.npz")


if __name__ == "__main__":
    golden_q4_reference()
    golden_ref_cases()
