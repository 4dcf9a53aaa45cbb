#!/usr/bin/env python
"""Golden fixtures for per-channel INT8 (W8A8) checkpoints, made with compressed-tensors (0.15) on the CPU: its
``calculate_qparams`` / ``quantize`` give the int8 weight codes and per-channel scales of the ``W8A8`` preset, its
``dequantize`` the dequantised weights, and its ``compute_dynamic_scales_and_zp`` / ``quantize`` the activation codes of
a dynamic per-token layer (the preset) or a static per-tensor one.  The tests only read the committed output:

    python tests/golden/make_golden_int8_w8a8.py

Output (committed): tests/golden/int8_w8a8_cases.npz, for every case name c (its dtype T = the model's dtype, in which
compressed-tensors stores the scales):
  * c.weight (int8 [N, K]) and c.weight_scale (T, [N, 1]);
  * c.input_scale (T, [1]) for the static cases;
  * c.W (T, [K, N]): compressed-tensors' dequantised weight, transposed;
  * c.x (T, [M, K]), c.codes (int8 [M, K]) and c.s_x (T, [M, 1] or [1]): compressed-tensors' activation codes and scales;
  * c.y (float32 [M, N]): compressed-tensors' fake-quantised layer dequant(codes, s_x) @ W in float64.
fp16 arrays are stored as float16, bf16 arrays as their uint16 bit patterns (numpy has no bf16).
"""
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))

# (name, activations, dtype, K, N, M)
CASES = (("dyn_bf", "dynamic", torch.bfloat16, 512, 128, 48),
         ("dyn_16", "dynamic", torch.float16, 512, 128, 48),
         ("static_bf", "static", torch.bfloat16, 256, 192, 16),
         ("static_16", "static", torch.float16, 256, 192, 16))


def _store(t: torch.Tensor) -> np.ndarray:
    """fp16 -> float16 array, bf16 -> uint16 bit patterns, other dtypes as they are."""
    if t.dtype == torch.bfloat16:
        return t.view(torch.int16).numpy().view(np.uint16)
    return t.numpy()


def main():
    from compressed_tensors.quantization import QuantizationArgs, preset_name_to_scheme
    from compressed_tensors.quantization.lifecycle.forward import compute_dynamic_scales_and_zp, dequantize, quantize
    from compressed_tensors.quantization.utils import calculate_qparams

    out = {}
    for name, act, dt, K, N, M in CASES:
        scheme = preset_name_to_scheme("W8A8", ["Linear"])
        wa, xa = scheme.weights, scheme.input_activations
        if act == "static":
            xa = QuantizationArgs(num_bits=8, type="int", symmetric=True, strategy="tensor", dynamic=False)
        g = torch.Generator().manual_seed(K + N + M)
        w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dt)
        x = (torch.randn(M, K, generator=g) * 3).to(dt)
        x[0] = 0  # an all-zero row
        zero = torch.zeros(())
        ws, wz = calculate_qparams(torch.minimum(w.amin(dim=1, keepdim=True), zero),
                                   torch.maximum(w.amax(dim=1, keepdim=True), zero), wa)
        ws, wz = ws.reshape(N, 1), wz.reshape(N, 1)
        wq = quantize(w, ws, wz, wa, dtype=torch.int8)
        W = dequantize(wq, ws, wz, wa, dtype=dt)
        if xa.dynamic:
            # token scales reduce the hidden dim of [batch, tokens, hidden] activations
            sx, zx = compute_dynamic_scales_and_zp(x[None], xa, module=torch.nn.Linear(K, N))
            sx, zx = sx[0], zx[0]
        else:
            sx, zx = calculate_qparams(torch.minimum(x.amin(), zero).reshape(1), torch.maximum(x.amax(), zero).reshape(1),
                                       xa)
            sx = sx.to(dt)  # a checkpoint stores it in the model's dtype
            out[f"{name}.input_scale"] = _store(sx)
        xq = quantize(x, sx, zx, xa, dtype=torch.int8)
        xd = dequantize(xq, sx, zx, xa, dtype=dt)
        y = xd.double() @ W.double().t()
        out[f"{name}.weight"] = wq.numpy()
        out[f"{name}.weight_scale"] = _store(ws.to(dt))
        out[f"{name}.W"] = _store(W.t().contiguous())
        out[f"{name}.x"] = _store(x)
        out[f"{name}.codes"] = xq.numpy()
        out[f"{name}.s_x"] = _store(sx)
        out[f"{name}.y"] = y.float().numpy()
        print(name, act, dt, tuple(ws.shape), ws.dtype, tuple(sx.shape), sx.dtype, wq.dtype, xq.dtype)
    np.savez_compressed(os.path.join(HERE, "int8_w8a8_cases.npz"), **out)


if __name__ == "__main__":
    main()
