"""TEST INFRASTRUCTURE ONLY — restatement of the reference's QQQ (W4A8) serving arithmetic (QQQLinear.forward + qqq_gemm,
gptqmodel/nn_modules/qlinear/qqq.py, gptqmodel_ext/qqq/qqq_gemm.cu) with an exact integer accumulation, plus
``pack_qqq`` / ``unpack_qqq`` so tests can build large random QQQ layers.

The permutations are written here independently of ``gptqmodel_b200.qqq`` (numpy, from the format's description), so
the package's un-permutation is checked against a second statement of the format and against the reference's fixtures.
"""
from __future__ import annotations

import numpy as np
import torch

TILE = 16


def _perm(per_channel: bool) -> np.ndarray:
    # slot order of 1024 nibbles = 4 tiles of [16 x 16]; every word's 8 slots are interleaved at the end
    p = np.empty(1024, dtype=np.int64)
    o = 0
    for i in range(32):
        col, r0 = i // 4, 4 * (i % 4)
        run = np.array([16 * (r0 + r) + col + 8 * b for b in (0, 1) for r in range(4)])
        for j in range(4):
            p[o:o + 8] = run + 256 * j
            o += 8
    inter = np.array([4, 0, 5, 1, 6, 2, 7, 3] if per_channel else [0, 2, 4, 6, 1, 3, 5, 7])
    return p.reshape(-1, 8)[:, inter].reshape(-1)


def _scale_perm() -> np.ndarray:
    return np.arange(64).reshape(8, 8).T.reshape(-1)


def _scale_perm_single() -> np.ndarray:
    return np.array([2 * i + j for i in range(4) for j in (0, 1, 8, 9, 16, 17, 24, 25)])


def pack_qqq(codes: torch.Tensor, s_channel: torch.Tensor, s_group=None):
    """Canonical layer -> checkpoint tensors.  codes [K, N] nibbles 0..15 (per-channel layers: the two's complement
    nibble of the signed code); s_channel fp32 [N]; s_group fp16 [K/128, N] or None.  Returns (B, s_channel [1, N],
    s_group or an empty fp16 tensor)."""
    K, N = codes.shape
    per_channel = s_group is None
    c = codes.cpu().numpy().astype(np.int64) & 0xF
    t = c.reshape(K // TILE, TILE, N // TILE, TILE).transpose(0, 2, 1, 3).reshape(K // TILE, N * TILE)
    t = t.reshape(-1, 1024)[:, _perm(per_channel)].reshape(K // TILE, N * TILE)
    words = np.zeros((K // TILE, N * TILE // 8), dtype=np.int64)
    for i in range(8):
        words |= t[:, i::8] << (4 * i)
    B = torch.from_numpy(words.astype(np.uint32).view(np.int32).copy())
    sc = s_channel.detach().cpu().to(torch.float32).numpy().reshape(-1, 32)[:, _scale_perm_single()]
    sc = torch.from_numpy(np.ascontiguousarray(sc).reshape(1, N))
    if per_channel:
        return B, sc, torch.empty(0, dtype=torch.float16)
    sg = s_group.detach().cpu().to(torch.float16).numpy().reshape(-1, 64)[:, _scale_perm()]
    return B, sc, torch.from_numpy(np.ascontiguousarray(sg).reshape(K // 128, N))


def unpack_qqq(B: torch.Tensor, s_channel: torch.Tensor, s_group=None):
    """Checkpoint tensors -> (codes uint8 [K, N], s_channel fp32 [N], s_group fp16 [K/128, N] or None)."""
    K, N = B.shape[0] * TILE, B.shape[1] * 8 // TILE
    per_channel = s_group is None or s_group.numel() == 0
    w = B.detach().cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    t = np.empty((K // TILE, N * TILE), dtype=np.int64)
    for i in range(8):
        t[:, i::8] = (w >> (4 * i)) & 0xF
    perm = _perm(per_channel)
    u = np.empty_like(t.reshape(-1, 1024))
    u[:, perm] = t.reshape(-1, 1024)
    codes = u.reshape(K // TILE, N // TILE, TILE, TILE).transpose(0, 2, 1, 3).reshape(K, N)
    sc = np.empty((N // 32, 32), dtype=np.float32)
    sc[:, _scale_perm_single()] = s_channel.detach().cpu().to(torch.float32).numpy().reshape(-1, 32)
    sg = None
    if not per_channel:
        g = np.empty((K // 128 * N // 64, 64), dtype=np.float16)
        g[:, _scale_perm()] = s_group.detach().cpu().to(torch.float16).numpy().reshape(-1, 64)
        sg = torch.from_numpy(g.reshape(K // 128, N))
    return torch.from_numpy(codes.astype(np.uint8)), torch.from_numpy(sc.reshape(N)), sg


def weight_int8(codes: torch.Tensor, s_group=None) -> torch.Tensor:
    """int8 weights w [K, N] as int64: signed nibble * 16 (per-channel), round_half_even((c - 8) * s) (group 128).
    Raises ValueError outside [-128, 127] (the reference's two paths disagree there)."""
    c = codes.to(torch.int64)
    if s_group is None:
        return torch.where(c >= 8, c - 16, c) * 16
    K, N = c.shape
    s = s_group.to(torch.float32).to(c.device).repeat_interleave(128, dim=0)
    w = ((c - 8).to(torch.float32) * s).round()
    if float(w.min()) < -128 or float(w.max()) > 127:
        raise ValueError("group-128 weight outside int8")
    return w.to(torch.int64)


def quantize(x: torch.Tensor):
    """The reference's dynamic_quant on fp16(x): (codes int8 [M, K], s_tok fp32 [M])."""
    A = x if x.dtype == torch.float16 else x.to(torch.float16)
    Af = A.to(torch.float32)
    amax = Af.abs().amax(dim=-1)
    # a tensor divisor: torch turns division by a scalar into a reciprocal multiply on CUDA
    s = (amax / torch.full_like(amax, 127.0)).to(torch.float16).to(torch.float32)
    v = Af / s.unsqueeze(-1)
    q = torch.where(torch.isnan(v), torch.zeros_like(v), v.round().clamp(-128, 127))
    return q.to(torch.int8), s


def forward(x: torch.Tensor, codes: torch.Tensor, s_channel: torch.Tensor, s_group=None, bias=None) -> torch.Tensor:
    """y [..., N] in x's dtype.  The int32 accumulation is done in float64, exact for K <= 65536 (|sum| < 2^31), so this
    runs on any device; then fp16(fp32(acc) * s_channel * s_tok), fp16(y + bias), and the cast to x's dtype."""
    K = x.shape[-1]
    N = codes.shape[1]
    dev = x.device
    q, s = quantize(x.reshape(-1, K))
    w = weight_int8(codes.to(dev), None if s_group is None else s_group.to(dev))
    acc = (q.to(torch.float64) @ w.to(torch.float64)).to(torch.float32)
    y = ((acc * s_channel.to(dev, torch.float32).reshape(1, N)) * s.unsqueeze(-1)).to(torch.float16)
    if bias is not None:
        y = (y.to(torch.float32) + bias.to(dev, torch.float16).to(torch.float32)).to(torch.float16)
    return y.to(x.dtype).reshape(x.shape[:-1] + (N,))
