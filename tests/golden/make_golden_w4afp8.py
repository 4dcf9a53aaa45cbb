#!/usr/bin/env python
"""Golden fixtures for W4AFP8 checkpoints, made with compressed-tensors (0.15) on the CPU: ``calculate_qparams`` gives
the group-128 scales of the ``W4AFP8`` preset's weights, ``PackedQuantizationCompressor.compress`` the checkpoint
tensors (``weight_packed``, ``weight_scale``, ``weight_shape``), ``dequantize`` the dequantised weights, and
``compute_dynamic_scales_and_zp`` / ``quantize`` the per-token e4m3 activation codes.

compressed-tensors dequantises each weight on its own, ``T(q * s[n, k / 128])``, so its dequantised weight is stored as
the table of the 16 values it gives each group (``dequantize`` on a code tensor that holds q = -8..7 in every group):
W[k, n] = table[n, k / 128, q[n, k] + 8].  The script asserts that identity against the full ``dequantize`` output, and
the table is an eighth of W's size.  The tests only read the committed output:

    python tests/golden/make_golden_w4afp8.py

Output (committed): tests/golden/w4afp8_cases.npz, for every case name c (its dtype T = the model's dtype, in which
compressed-tensors stores the scales):
  * c.weight_packed (int32 [N, K/8]), c.weight_scale (T, [N, K/128]) and c.weight_shape (int64 [2]);
  * c.dq_table (T, [N, K/128, 16]): compressed-tensors' dequantised weight as the table above;
  * c.x (T, [M, K]), c.codes (e4m3 bit patterns, uint8 [M, K]) and c.s_x (T, [M, 1]): compressed-tensors' activation
    codes and scales;
  * c.y (float32 [M, N]): compressed-tensors' fake-quantised layer dequant(codes, s_x) @ W in float64.
fp16 arrays are stored as float16, bf16 arrays as their uint16 bit patterns (numpy has no bf16).
"""
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))

# (name, dtype, K, N, M)
CASES = (("bf_512_128_1", torch.bfloat16, 512, 128, 1),
         ("bf_1024_128_48", torch.bfloat16, 1024, 128, 48),
         ("f16_512_256_48", torch.float16, 512, 256, 48),
         ("f16_512_128_1", torch.float16, 512, 128, 1))


def _store(t: torch.Tensor) -> np.ndarray:
    """fp16 -> float16 array, bf16 -> uint16 bit patterns, other dtypes as they are."""
    if t.dtype == torch.bfloat16:
        return t.view(torch.int16).numpy().view(np.uint16)
    return t.numpy()


def main():
    from compressed_tensors.compressors.pack_quantized.base import PackedQuantizationCompressor
    from compressed_tensors.quantization import preset_name_to_scheme
    from compressed_tensors.quantization.lifecycle.forward import compute_dynamic_scales_and_zp, dequantize, quantize
    from compressed_tensors.quantization.utils import calculate_qparams

    out = {}
    for name, dt, K, N, M in CASES:
        scheme = preset_name_to_scheme("W4AFP8", ["Linear"])
        wa, xa = scheme.weights, scheme.input_activations
        g = torch.Generator().manual_seed(K + N + M)
        w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dt)
        x = (torch.randn(M, K, generator=g) * 3).to(dt)
        zero = torch.zeros(())
        wg = w.reshape(N, K // 128, 128)
        ws, wz = calculate_qparams(torch.minimum(wg.amin(dim=2), zero), torch.maximum(wg.amax(dim=2), zero), wa)
        ws = ws.to(dt)  # a checkpoint stores the scales in the model's dtype
        sd = PackedQuantizationCompressor.compress({"weight": w, "weight_scale": ws, "weight_zero_point": wz}, scheme)
        wq = quantize(w, ws, wz, wa, dtype=torch.int8)
        W = dequantize(wq, ws, wz, wa, dtype=dt)
        grid = (torch.arange(K) % 16 - 8).to(torch.int8).expand(N, K).contiguous()  # q = -8..7 in every group
        table = dequantize(grid, ws, wz, wa, dtype=dt).reshape(N, K // 128, 128)[:, :, :16].contiguous()
        lookup = table.gather(2, (wq.to(torch.int64) + 8).reshape(N, K // 128, 128)).reshape(N, K)
        assert torch.equal(lookup, W), name
        sx, zx = compute_dynamic_scales_and_zp(x[None], xa, module=torch.nn.Linear(K, N))
        sx, zx = sx[0], zx[0]
        xq = quantize(x, sx, zx, xa, dtype=torch.float8_e4m3fn)
        xd = dequantize(xq, sx, zx, xa, dtype=dt)
        y = xd.double() @ W.double().t()
        assert "weight_zero_point" not in sd and sd["weight_scale"].dtype == dt
        out[f"{name}.weight_packed"] = sd["weight_packed"].numpy()
        out[f"{name}.weight_scale"] = _store(sd["weight_scale"])
        out[f"{name}.weight_shape"] = sd["weight_shape"].to(torch.int64).numpy()
        out[f"{name}.dq_table"] = _store(table)
        out[f"{name}.x"] = _store(x)
        out[f"{name}.codes"] = xq.view(torch.uint8).numpy()
        out[f"{name}.s_x"] = _store(sx)
        out[f"{name}.y"] = y.float().numpy()
        print(name, dt, tuple(sd["weight_packed"].shape), tuple(ws.shape), tuple(sx.shape), sx.dtype)
    np.savez_compressed(os.path.join(HERE, "w4afp8_cases.npz"), **out)


if __name__ == "__main__":
    main()
