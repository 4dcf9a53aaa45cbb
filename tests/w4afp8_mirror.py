"""numpy mirrors of the W4AFP8 tier (include/b2q.h states the arithmetic): the checkpoint packing, the kernel's tile
layout and the float32 promotion chain of b2q_w4afp8_mm."""
import numpy as np

GROUP = 128
NIBBLE_K = (0, 1, 4, 5, 2, 3, 6, 7)  # nibble p of a tile word holds k0 + NIBBLE_K[p]


def pack(c: np.ndarray) -> np.ndarray:
    """codes c = q + 8 (uint8 [N, K], 0..15) -> weight_packed int32 [N, K/8] (compressed-tensors' pack_to_int32)."""
    N, K = c.shape
    w = np.zeros((N, K // 8), dtype=np.uint32)
    for i in range(8):
        w |= (c[:, i::8].astype(np.uint32) & 15) << (4 * i)
    return w.view(np.int32)


def unpack(wp: np.ndarray) -> np.ndarray:
    """weight_packed int32 [N, K/8] -> codes c uint8 [N, K]."""
    w = wp.view(np.uint32)
    return np.stack([(w >> (4 * i)) & 15 for i in range(8)], axis=-1).reshape(w.shape[0], -1).astype(np.uint8)


def prepack(wp: np.ndarray) -> np.ndarray:
    """b2q_w4afp8_prepack: weight_packed [N, K/8] -> tile words uint32 [N/128, K/128, 4 quads, 128 features, 4]."""
    c = unpack(wp)
    N, K = c.shape
    t = c.reshape(N // 128, 128, K // GROUP, 4, 4, 8)                 # [nt][f][kb][quad][word][k offset]
    t = t[..., list(NIBBLE_K)].astype(np.uint32)                      # [...][nibble p]
    words = np.zeros(t.shape[:-1], dtype=np.uint32)
    for p in range(8):
        words |= t[..., p] << (4 * p)
    return np.ascontiguousarray(words.transpose(0, 2, 3, 1, 4))       # [nt][kb][quad][f][word]


def unprepack(tiles: np.ndarray, K: int, N: int) -> np.ndarray:
    """The inverse of prepack: tile words -> codes c uint8 [N, K]."""
    w = tiles.reshape(N // 128, K // GROUP, 4, 128, 4).view(np.uint32)
    nib = np.stack([(w >> (4 * p)) & 15 for p in range(8)], axis=-1)[..., list(NIBBLE_K)]
    return nib.transpose(0, 3, 1, 2, 4, 5).reshape(N, K).astype(np.uint8)


def block_sums(c: np.ndarray, q: np.ndarray) -> np.ndarray:
    """P [KB, M, N] = sum over each 128-k block of c[m, k] q[n, k] in float64 (exact for the tests' small codes)."""
    M, K = c.shape
    cb = c.astype(np.float64).reshape(M, K // GROUP, GROUP)
    qb = q.astype(np.float64).reshape(q.shape[0], K // GROUP, GROUP)
    return np.einsum("mbk,nbk->bmn", cb, qb)


def mm(P: np.ndarray, s_x: np.ndarray, s_w: np.ndarray, bias, ks: int) -> np.ndarray:
    """The float32 chain of b2q_w4afp8_mm with ks split-K ranks (kpc = ceil(KB / ks) contiguous blocks per rank):
    acc = fma(P_b, s_w[b], acc) per rank in block order, the ranks summed in rank order, y = acc * s_x (+ bias), all in
    float32 (y before the rounding to the output dtype).  P_b * s_w[b] must be exact in float32, so an fma is one
    rounding of a float32 sum (computed in float64, whose rounding to float32 is then correct)."""
    KB = P.shape[0]
    kpc = -(-KB // ks)
    total = None
    for r in range(ks):
        acc = np.zeros(P.shape[1:], dtype=np.float32)
        for b in range(r * kpc, min(KB, (r + 1) * kpc)):
            prod = P[b] * s_w[b].astype(np.float64)[None, :]
            assert np.all(prod.astype(np.float32).astype(np.float64) == prod), "P * s_w must be exact in float32"
            acc = (prod + acc.astype(np.float64)).astype(np.float32)
        total = acc if total is None else (total + acc).astype(np.float32)
    y = (total * s_x.astype(np.float32)[:, None]).astype(np.float32)
    if bias is not None:
        y = (y + bias.astype(np.float32)[None, :]).astype(np.float32)
    return y


def plan_ks(M: int, K: int, N: int, sms: int) -> int:
    """The split-K ranks of the heuristic plan (fp8blk_plan, mode 0) on a device with `sms` SMs."""
    ntok = 8
    while ntok < M and ntok < 128:
        ntok *= 2
    blocks = (N // 128) * (-(-M // ntok))
    KB = K // GROUP
    ks = 1
    while ks < 8 and blocks * ks * 2 <= sms and KB // (ks * 2) >= 2:
        ks *= 2
    while ks > 1 and (ks - 1) * (-(-KB // ks)) >= KB:
        ks >>= 1
    return ks


def table_weight(table: np.ndarray, c: np.ndarray) -> np.ndarray:
    """A dequantised weight W [K, N] from a fixture's table [N, K/128, 16] (the 16 values of each group) and the codes
    c uint8 [N, K]: W[k, n] = table[n, k / 128, c[n, k]]."""
    N, K = c.shape
    w = np.take_along_axis(table, c.reshape(N, K // GROUP, GROUP).astype(np.int64), axis=2)
    return np.ascontiguousarray(w.reshape(N, K).T)
