#!/usr/bin/env python
"""Golden fixtures for per-channel / per-tensor FP8 (W8A8) checkpoints, made with compressed-tensors (0.15) on the CPU:
its ``calculate_qparams`` / ``quantize`` give the weight codes and scales of the FP8_DYNAMIC (channel) and FP8 (tensor)
presets, its ``dequantize`` the dequantised weights, and its ``compute_dynamic_scales_and_zp`` / ``quantize`` the
activation codes of a dynamic per-token or a static per-tensor layer.  The tests only read the committed output:

    python tests/golden/make_golden_fp8_w8a8.py

Output (committed): tests/golden/fp8_w8a8_cases.npz, for every case name c (its dtype T = the model's dtype, in which
compressed-tensors stores the scales):
  * c.weight (uint8 e4m3fn bit patterns [N, K]) and c.weight_scale (T, [N, 1] or [1]);
  * c.input_scale (T, [1]) for the static case;
  * c.W (T, [K, N]): compressed-tensors' dequantised weight, transposed;
  * c.x (T, [M, K]), c.codes (uint8 [M, K]) and c.s_x (T, [M, 1] or [1]): compressed-tensors' activation codes and scales;
  * c.y (float32 [M, N]): compressed-tensors' fake-quantised layer dequant(codes, s_x) @ W in float64.
fp16 arrays are stored as float16, bf16 arrays as their uint16 bit patterns (numpy has no bf16).
"""
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))

# (name, preset, dtype, K, N, M)
CASES = (("dyn_bf", "FP8_DYNAMIC", torch.bfloat16, 512, 128, 48),
         ("dyn_16", "FP8_DYNAMIC", torch.float16, 512, 128, 48),
         ("static_bf", "FP8", torch.bfloat16, 256, 192, 16))


def _store(t: torch.Tensor) -> np.ndarray:
    """fp16 -> float16 array, bf16 -> uint16 bit patterns, other dtypes as they are."""
    if t.dtype == torch.bfloat16:
        return t.view(torch.int16).numpy().view(np.uint16)
    return t.numpy()


def main():
    from compressed_tensors.quantization import preset_name_to_scheme
    from compressed_tensors.quantization.lifecycle.forward import compute_dynamic_scales_and_zp, dequantize, quantize
    from compressed_tensors.quantization.utils import calculate_qparams

    out = {}
    for name, preset, dt, K, N, M in CASES:
        scheme = preset_name_to_scheme(preset, ["Linear"])
        wa, xa = scheme.weights, scheme.input_activations
        g = torch.Generator().manual_seed(K + N + M)
        w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dt)
        x = (torch.randn(M, K, generator=g) * 3).to(dt)
        x[0] = 0  # an all-zero row
        dims = 1 if wa.strategy == "channel" else (0, 1)
        zero = torch.zeros(())
        ws, wz = calculate_qparams(torch.minimum(w.amin(dim=dims, keepdim=True), zero),
                                   torch.maximum(w.amax(dim=dims, keepdim=True), zero), wa)
        ws = ws.reshape(N, 1) if wa.strategy == "channel" else ws.reshape(1)
        wq = quantize(w, ws, wz.reshape(ws.shape), wa, dtype=torch.float8_e4m3fn)
        W = dequantize(wq, ws, wz.reshape(ws.shape), wa, dtype=dt)
        if xa.dynamic:
            # token scales reduce the hidden dim of [batch, tokens, hidden] activations
            sx, zx = compute_dynamic_scales_and_zp(x[None], xa, module=torch.nn.Linear(K, N))
            sx, zx = sx[0], zx[0]
        else:
            sx, zx = calculate_qparams(torch.minimum(x.amin(), zero).reshape(1), torch.maximum(x.amax(), zero).reshape(1),
                                       xa)
            sx = sx.to(dt)  # a checkpoint stores it in the model's dtype
            out[f"{name}.input_scale"] = _store(sx)
        xq = quantize(x, sx, zx, xa, dtype=torch.float8_e4m3fn)
        xd = dequantize(xq, sx, zx, xa, dtype=dt)
        y = xd.double() @ W.double().t()
        out[f"{name}.weight"] = wq.view(torch.uint8).numpy()
        out[f"{name}.weight_scale"] = _store(ws.to(dt))
        out[f"{name}.W"] = _store(W.t().contiguous())
        out[f"{name}.x"] = _store(x)
        out[f"{name}.codes"] = xq.view(torch.uint8).numpy()
        out[f"{name}.s_x"] = _store(sx)
        out[f"{name}.y"] = y.float().numpy()
        print(name, preset, dt, tuple(ws.shape), ws.dtype, tuple(sx.shape), sx.dtype)
    np.savez_compressed(os.path.join(HERE, "fp8_w8a8_cases.npz"), **out)


if __name__ == "__main__":
    main()
