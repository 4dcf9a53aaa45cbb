"""Checkpoint bit layouts the kernels do not read natively, and their exact conversion into the ones they do.

The B200 kernels stream 4- and 8-bit codes.  The reference's GPTQ QuantLinear contract is wider
(gptqmodel/nn_modules/qlinear/__init__.py:766-785, :907-999; utils/planar_packing.py:1-52):

  * 2-bit                      16 codes per int32 word, LSB first (same scheme as 4 / 8-bit),
  * 3-bit "continuous"         32 codes = one 96-bit little-endian bit stream over 3 consecutive words
                               (codes 10 and 21 straddle a word boundary; :910-918, :976-999),
  * planar 3 / 5 / 6 / 7-bit   (`format = gptq_p`; 5-7 exist ONLY planar) 32 codes = `bits` consecutive words holding
                               word-aligned bit planes: a 4- (or 2-) bit low plane, then 2- and/or 1-bit high planes,
  * qzeros use the same layouts along N.

A b-bit code with a b-bit zero-point is the same integer in a wider container, and `(q - z) * s` does not depend on the
container: `widen()` re-packs such a layer into the 4-bit (b <= 4) or 8-bit (b >= 5) LSB-first layout, bit-exactly, once,
at `post_init()` time, on the device the checkpoint tensors live on (torch integer ops: load-time plumbing, not the hot
path).  The price is memory and bandwidth (a 2-bit layer streams 4 bits per weight, a 5-bit layer 8): the arithmetic is
the reference's, the footprint is the container's.

`regroup()` handles an ARBITRARY g_idx (groups of unequal size, e.g. a K-slice of an act-order layer whose scale table
is replicated across tensor-parallel ranks, utils/marlin.py:296-305): rows are sorted by group, every group's run is padded
to a multiple of a 32 / 64 / 128-row granule with rows whose code equals the group's zero-point (an exact zero weight),
and the scale / zero tables are re-indexed per granule, which yields a uniform-group layer the kernels serve as usual
plus the gather index for the activations' columns.
"""
from __future__ import annotations

from functools import lru_cache
from typing import Dict, List, Optional, Tuple

import torch

SUPPORTED_BITS = (2, 3, 4, 5, 6, 7, 8)
PLANAR_ONLY_BITS = (5, 6, 7)
# planes of the gptq_p layout, low to high: (width, first bit of the code it holds)
_PLANES = {2: ((2, 0),), 3: ((2, 0), (1, 2)), 4: ((4, 0),), 5: ((4, 0), (1, 4)), 6: ((4, 0), (2, 4)),
           7: ((4, 0), (2, 4), (1, 6)), 8: ((8, 0),)}


def is_planar(bits: int, fmt: Optional[str]) -> bool:
    """qlinear/__init__.py:773: 5/6/7-bit are always planar, 3-bit only under format gptq_p; planar 2/4/8 words are
    bit-identical to the continuous ones."""
    return bits in PLANAR_ONLY_BITS or (bits == 3 and str(getattr(fmt, "value", fmt)) == "gptq_p")


def container_bits(bits: int) -> int:
    if bits not in SUPPORTED_BITS:
        raise NotImplementedError(f"bits={bits} not supported (one of {SUPPORTED_BITS})")
    return 4 if bits <= 4 else 8


@lru_cache(maxsize=None)
def _fields(bits: int, planar: bool) -> Tuple[int, Tuple[Tuple[Tuple[int, int, int, int], ...], ...]]:
    """(codes per block, per code a tuple of bit fields (word, pos, width, dst)): code = sum(((word >> pos) & mask) << dst).

    A block is `codes * bits / 32` consecutive words.  Continuous layouts are one LSB-first bit stream over the block (for
    bits dividing 32 that degenerates to whole fields inside one word); planar layouts put plane p's word i after the
    words of the lower planes, holding codes [i * 32/w, (i+1) * 32/w) at shifts w * j."""
    if planar:
        per_code: List[List[Tuple[int, int, int, int]]] = [[] for _ in range(32)]
        base = 0
        for width, dst in _PLANES[bits]:
            per_word = 32 // width
            for c in range(32):
                per_code[c].append((base + c // per_word, width * (c % per_word), width, dst))
            base += width
        return 32, tuple(tuple(f) for f in per_code)
    if 32 % bits == 0:
        n = 32 // bits
        return n, tuple(((0, bits * c, bits, 0),) for c in range(n))
    out = []
    for c in range(32):
        lo, hi = c * bits, c * bits + bits
        fields, dst = [], 0
        while lo < hi:
            word, pos = divmod(lo, 32)
            width = min(hi - lo, 32 - pos)
            fields.append((word, pos, width, dst))
            lo += width
            dst += width
        out.append(tuple(fields))
    return 32, tuple(out)


def unpack_rows(words: torch.Tensor, bits: int, planar: bool = False) -> torch.Tensor:
    """int32 [R, C] -> codes int32 [R * 32 / bits, C] (codes packed along dim 0: qweight)."""
    if words.dtype != torch.int32 or words.dim() != 2:
        raise ValueError("unpack_rows: int32 [rows, cols] expected")
    codes, fields = _fields(bits, planar)
    wpb = codes * bits // 32
    R, C = words.shape
    if R % wpb != 0:
        raise ValueError(f"unpack_rows: {R} rows of {bits}-bit words do not hold whole {wpb}-word blocks")
    blk = words.view(R // wpb, wpb, C)
    out = torch.empty((R // wpb, codes, C), dtype=torch.int32, device=words.device)
    for c, fs in enumerate(fields):
        acc = None
        for word, pos, width, dst in fs:
            # arithmetic shift of a negative word fills with ones; the mask keeps the `width` wanted bits
            v = torch.bitwise_and(torch.bitwise_right_shift(blk[:, word, :], pos), (1 << width) - 1)
            if dst:
                v = torch.bitwise_left_shift(v, dst)
            acc = v if acc is None else torch.bitwise_or(acc, v)
        out[:, c, :] = acc
    return out.view(R // wpb * codes, C)


def pack_rows(codes_t: torch.Tensor, bits: int, planar: bool = False) -> torch.Tensor:
    """codes [K, C] (any integer dtype, values < 2^bits) -> int32 [K * bits / 32, C]; inverse of unpack_rows."""
    if codes_t.dim() != 2:
        raise ValueError("pack_rows: [rows, cols] expected")
    codes, fields = _fields(bits, planar)
    wpb = codes * bits // 32
    K, C = codes_t.shape
    if K % codes != 0:
        raise ValueError(f"pack_rows: {K} rows are not whole blocks of {codes} {bits}-bit codes")
    blk = codes_t.to(torch.int64).view(K // codes, codes, C)
    out = torch.zeros((K // codes, wpb, C), dtype=torch.int64, device=codes_t.device)
    for c, fs in enumerate(fields):
        for word, pos, width, dst in fs:
            v = torch.bitwise_and(torch.bitwise_right_shift(blk[:, c, :], dst), (1 << width) - 1)
            out[:, word, :] |= torch.bitwise_left_shift(v, pos)
    out = torch.where(out >= 2 ** 31, out - 2 ** 32, out).to(torch.int32)
    return out.view(K // codes * wpb, C)


def unpack_cols(words: torch.Tensor, bits: int, planar: bool = False) -> torch.Tensor:
    """int32 [G, N * bits / 32] -> codes int32 [G, N] (codes packed along dim 1: qzeros)."""
    return unpack_rows(words.t().contiguous(), bits, planar).t().contiguous()


def pack_cols(codes_t: torch.Tensor, bits: int, planar: bool = False) -> torch.Tensor:
    return pack_rows(codes_t.t().contiguous(), bits, planar).t().contiguous()


def shift_zero_points(qzeros: torch.Tensor, bits: int, planar: bool, delta: int) -> torch.Tensor:
    """v1 <-> v2 zero-points: every LOGICAL field +/- 1 modulo 2^bits (utils/model_dequant.py:900-907).  For 4 / 8-bit
    words without a wrapping field that equals adding 0x1111.. / 0x0101.. to the packed word (utils/model.py:813-830)."""
    z = unpack_cols(qzeros, bits, planar)
    return pack_cols(torch.bitwise_and(z + delta, (1 << bits) - 1), bits, planar)


def widen(qweight: torch.Tensor, qzeros: torch.Tensor, bits: int, planar: bool) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """(qweight, qzeros) of a b-bit layer (v2 zero-points) -> the same integers in the 4- or 8-bit LSB-first layout."""
    kb = container_bits(bits)
    if kb == bits and not planar:
        return qweight, qzeros, kb
    q = unpack_rows(qweight, bits, planar)
    z = unpack_cols(qzeros, bits, planar)
    return pack_rows(q, kb), pack_cols(z, kb), kb


def regroup(q: torch.Tensor, z: torch.Tensor, scales: torch.Tensor, g_idx: torch.Tensor,
            align: int = 128) -> Dict[str, torch.Tensor]:
    """Arbitrary g_idx -> uniform groups.

    q [K, N] codes, z [G, N] zero-points, scales [G, N], g_idx [K] with values in [0, G) ->
      q       [K', N]  rows sorted by group, each group's run padded to a multiple of `granule` with its zero-point
      z, scales [K'/granule, N]
      gather  int64 [K'] column of x feeding each row (padding rows read column 0: their weight is exactly zero)
      granule int      the new group_size (the one of 128 / 64 / 32 giving the smallest K')
    K' is a multiple of `align`."""
    K, N = q.shape
    G = z.shape[0]
    gi = g_idx.to(torch.int64)
    if gi.numel() != K or (K and (int(gi.min()) < 0 or int(gi.max()) >= G)):
        raise ValueError("regroup: g_idx must hold one group index in [0, G) per input feature")
    counts = torch.bincount(gi, minlength=G)
    best = None
    for granule in (128, 64, 32):
        padded = (counts + granule - 1) // granule * granule
        total = int(padded.sum())
        total = (total + align - 1) // align * align
        if best is None or total < best[0]:
            best = (total, granule, padded)
    Kp, granule, padded = best
    dev = q.device
    order = torch.argsort(gi, stable=True)
    gs_sorted = gi[order]
    first = torch.cumsum(counts, 0) - counts        # first sorted row of every group
    start = torch.cumsum(padded, 0) - padded        # first padded row of every group
    dest = start[gs_sorted] + (torch.arange(K, device=dev) - first[gs_sorted])
    # owner group of every padded row: groups in order, the alignment tail belongs to the last group
    owner = torch.repeat_interleave(torch.arange(G, device=dev), padded)
    if owner.numel() < Kp:
        owner = torch.cat([owner, owner.new_full((Kp - owner.numel(),), G - 1)])
    q2 = z.to(q.dtype)[owner]                       # padding: code == zero-point
    q2[dest] = q[order]
    gather = torch.zeros(Kp, dtype=torch.int64, device=dev)
    gather[dest] = order
    gmap = owner[::granule]
    return dict(q=q2.contiguous(), z=z[gmap].contiguous(), scales=scales[gmap].contiguous(), gather=gather,
                granule=granule)
