"""Float64 restatement of the online Hadamard transform a rotated (QuaRot / SpinQuant) GPTQ layer applies to its input.

For a row v of length n = K * P (P a power of two), V = v viewed as [K, P] row-major:

    T(v) = vec(had_K . V . H_P) / sqrt(n),   H_P[i, j] = (-1)^popcount(i & j)

which is the reference's ``matmul_hadU`` (gptqmodel/quantization/rotation/hadamard_utils.py).  ``had_K`` is the
K x K +-1 matrix of the rotation's non-power-of-two factor; None for K == 1.
"""
import math

import torch

__all__ = ["hadamard_transform", "sylvester"]


def sylvester(P: int) -> torch.Tensor:
    """H_P in natural order, float64."""
    i = torch.arange(P)
    bits = torch.bitwise_and(i[:, None], i[None, :])
    pc = torch.zeros_like(bits)
    while bool(bits.any()):
        pc += bits & 1
        bits = bits >> 1
    return (1 - 2 * (pc & 1)).to(torch.float64)


def hadamard_transform(x: torch.Tensor, had_K, K: int) -> torch.Tensor:
    """T(x) along the last dimension, float64 (fast Walsh-Hadamard butterflies, then the had_K product)."""
    n = x.shape[-1]
    if n % K or (n // K) & (n // K - 1):
        raise ValueError(f"n={n} is not K={K} times a power of two")
    P = n // K
    v = x.to(torch.float64).reshape(-1, K, P).clone()
    h = 1
    while h < P:
        v = v.reshape(-1, K, P // (2 * h), 2, h)
        a, b = v[:, :, :, 0, :], v[:, :, :, 1, :]
        v = torch.stack((a + b, a - b), dim=3).reshape(-1, K, P)
        h *= 2
    if K > 1:
        v = torch.as_tensor(had_K).to(torch.float64) @ v
    return (v / math.sqrt(n)).reshape(x.shape)
