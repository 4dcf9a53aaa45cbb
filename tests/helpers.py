"""Shared fixtures: synthetic quantised layers built with the oracle's packer (restated pack_original)."""
import re

import torch

import oracle


def make_layer(K, N, bits=4, group_size=128, sym=True, desc_act=False, bias=False, seed=42, dtype=torch.float16):
    """Returns dict of CPU checkpoint-layout tensors (v2 qzeros) quantised from randn weights.

    Recipe: W = randn(N, K, seed) * 0.5, sym grid of tests/kernels/test_swordfish.py:31-56
    or min/max asym, act-order g_idx = (arange // g)[randperm].
    """
    gen = torch.Generator().manual_seed(seed)
    W = torch.randn(N, K, generator=gen) * 0.5
    gs = group_size if group_size > 0 else K
    if desc_act:
        _, g_idx = oracle.make_act_order(K, gs, seed=seed)
    else:
        g_idx = torch.arange(K, dtype=torch.int32) // gs
    # vectorised min/max quantiser (same grid as oracle.quantize_sym / quantize_asym)
    G = K // gs
    order = torch.argsort(g_idx.long(), stable=True)
    Wg = W[:, order].reshape(N, G, gs)
    maxq = (1 << bits) - 1
    if sym:
        m = Wg.abs().amax(dim=2).clamp(min=1e-5)
        scales = m / ((maxq + 1) // 2 - 1)
        zeros = torch.full((N, G), float((maxq + 1) // 2))
    else:
        lo = Wg.amin(dim=2).clamp(max=0)
        hi = Wg.amax(dim=2).clamp(min=0)
        scales = ((hi - lo) / maxq).clamp(min=1e-5)
        zeros = torch.round(-lo / scales).clamp(0, maxq)
    qw, qz, sc, gi = oracle.pack(W, scales, zeros, g_idx, bits)
    b = None
    if bias:
        b = (torch.randn(N, generator=gen) * 0.1).to(torch.float16)
    return dict(qweight=qw, qzeros=qz, scales=sc, g_idx=gi, bias=b, bits=bits, group_size=group_size,
                sym=sym, desc_act=desc_act, K=K, N=N)


def random_layer(K, N, bits=4, group_size=128, sym=True, seed=0, device="cpu"):
    """Random codes (no quantiser): fast way to build LARGE layers for property tests / benchmarks."""
    gen = torch.Generator(device=device).manual_seed(seed)
    gs = group_size if group_size > 0 else K
    G = K // gs
    qw = torch.randint(-(2 ** 31), 2 ** 31 - 1, (K * bits // 32, N), dtype=torch.int32, device=device, generator=gen)
    if sym:
        zw = {4: 0x88888888 - (1 << 32), 8: 0x80808080 - (1 << 32)}[bits]
        qz = torch.full((G, N * bits // 32), zw, dtype=torch.int32, device=device)
    else:
        qz = torch.randint(-(2 ** 31), 2 ** 31 - 1, (G, N * bits // 32), dtype=torch.int32, device=device, generator=gen)
    sc = (torch.rand(G, N, device=device, generator=gen) * 0.01 + 0.005).to(torch.float16)
    if bits == 8:
        sc = sc / 16
    gi = (torch.arange(K, dtype=torch.int32, device=device) // gs)
    return dict(qweight=qw, qzeros=qz, scales=sc, g_idx=gi, bias=None, bits=bits, group_size=group_size,
                sym=sym, desc_act=False, K=K, N=N)


def oracle_forward(layer, x):
    xc = x.detach().cpu()
    return oracle.forward(xc, layer["qweight"].cpu(), layer["qzeros"].cpu(), layer["scales"].cpu().to(
        torch.float16 if x.dtype == torch.float16 else x.dtype), layer["g_idx"].cpu(), layer["bits"],
        bias=None if layer["bias"] is None else layer["bias"].cpu())


_DECODE_KERNEL = re.compile(r"\b(decode2?_kernel)<(__half|__nv_bfloat16), (true|false), (true|false), (true|false)>")


def decode_kernels_launched(fn):
    """Runs fn() under torch.profiler and returns (fn's result, [(kernel, dtype, asym, g64)] of the decode-tier
    kernels it launched, in launch order): kernel is "decode_kernel" or "decode2_kernel", dtype "__half" or
    "__nv_bfloat16" — the instantiation that actually ran, whatever the planner predicted."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):  # a profiling window this short now and then delivers no kernel record at all: profile again
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            res = fn()
            torch.cuda.synchronize()
        evs = sorted((e for e in prof.events() if _DECODE_KERNEL.search(e.name)), key=lambda e: e.time_range.start)
        if evs:
            break
    out = []
    for e in evs:
        k, dt, asym, g64, moe = _DECODE_KERNEL.search(e.name).groups()
        assert moe == "false", e.name
        out.append((k, dt, asym == "true", g64 == "true"))
    return res, out


def decode_k_split(M, K, N, kernel):
    """(split-K ranks, warps per tile group, quads per rank) of a decode launch of N features that ran on `kernel`, from
    that kernel's own planner (b2q_debug_decode_plan, which sizes shared memory for sym g128); None if it has no plan.
    decode2_kernel picked per launch shape runs one 16-warp group without split-K; B2Q_DECODE_V2=1 lets it choose."""
    import ctypes
    import os
    from gptqmodel_b200 import _lib as g
    out = (ctypes.c_int * 8)()
    if kernel == "decode2_kernel":
        free = os.environ.get("B2Q_DECODE_V2") == "1"
        rc = g.lib.b2q_debug_decode_plan(2, M, K, N, 0 if free else 1, 0 if free else 16, out)
    else:
        rc = g.lib.b2q_debug_decode_plan(1, M, K, N, 0, 0, out)
    return (out[1], out[3], out[4]) if rc == 0 else None


def same_k_split(M, K, single, fused):
    """True if two decode launches cut K identically; single / fused = (N, kernel that ran).  Both kernels give one
    warp of a group the same quads and sum the warps' and ranks' fp32 partials in the same order, so two launches with
    the same (ranks, group width, quads per rank) produce the same bits for a feature, whichever kernel ran."""
    a, b = decode_k_split(M, K, *single), decode_k_split(M, K, *fused)
    return a is not None and a == b


PARITY_LOG = {}  # test id -> worst err/tol ratio seen by assert_close_rel (dumped by conftest at session end)


def _record(what, rel, ratio):
    import os
    tid = os.environ.get("PYTEST_CURRENT_TEST", "?").split(" ")[0]
    e = PARITY_LOG.setdefault(tid, {"rel": rel, "worst_err_over_tol": 0.0, "worst_case": "", "checks": 0})
    e["checks"] += 1
    if ratio >= e["worst_err_over_tol"]:
        e["worst_err_over_tol"], e["worst_case"], e["rel"] = round(ratio, 4), what, rel


def ref_rounding_slack(W, x, sigmas=4.0):
    """Absolute deviation to be expected between an oracle that ROUNDS every dequantised weight to 16 bits (the
    reference: W = dtype((q - z) * s), one rounding per weight, qlinear/__init__.py:1001-1003) and arithmetic that does
    not (the decode / GEMV tiers apply the scale ONCE per group to an exact integer dot product — mathematically the
    same sum, closer to exact arithmetic, but not the reference's rounding points).  Every weight carries an independent
    relative rounding error uniform in +-2^-p (p = 11 for fp16, 8 for bf16): sigma = 2^-p / sqrt(3) per weight, so the two
    results differ by a random sum with standard deviation sigma * sqrt(sum_k (W[k, n] * x[m, k])^2).  Returns `sigmas`
    of those, [M, N].  tests/test_awq.py::test_scale_once_arithmetic_vs_per_weight_rounding shows on the reference's own
    AWQ fixture that EXACT float64 arithmetic sits 1.18x outside the plain 1e-3 criterion for this reason alone."""
    p = 11 if W.dtype == torch.float16 else 8
    sigma = 2.0 ** -p / 3 ** 0.5
    return sigmas * sigma * torch.sqrt((x.detach().float().cpu() ** 2) @ (W.detach().float().cpu() ** 2))


def scale_once_tier(layer, M):
    """True when b2q_mm serves (layer, M tokens) with a tier that applies the scale once per group to an exact integer dot
    product (decode tier: 4-bit, M <= 8, K % 128 == 0, group 64 / 128 / per-channel; 8-bit GEMV at M == 1) instead of feeding
    the tensor cores the reference's per-weight rounded operand."""
    K, gs, bits = layer["K"], layer["group_size"], layer["bits"]
    if bits == 4:
        return M <= 8 and K % 128 == 0 and gs in (64, 128, -1, K)
    return M == 1 and K % 128 == 0


def assert_layer_close(out, layer, x, rel=1e-3, what=""):
    """Module output against the oracle of the same checkpoint tensors: 1e-3 for the exact-operand tiers, 1e-3 plus the
    reference's own weight-rounding noise (ref_rounding_slack) for the scale-once tiers — see tests/test_awq.py."""
    xc = x.detach().cpu()
    ref = oracle_forward(layer, xc)
    slack = None
    if scale_once_tier(layer, xc.reshape(-1, xc.shape[-1]).shape[0]):
        W = oracle.dequantize_weight(layer["qweight"].cpu(), layer["qzeros"].cpu(), layer["scales"].cpu().to(xc.dtype),
                                     layer["g_idx"].cpu(), layer["bits"])
        slack = ref_rounding_slack(W, xc.reshape(-1, xc.shape[-1])).reshape(ref.shape)
    assert_close_rel(out, ref, rel, what, slack=slack)


def assert_close_rel(out, ref, rel=1e-3, what="", slack=None):
    """|out - ref| <= rel * |ref| + rel * rms(ref) (+ slack): the north-star's "1e-3 rel fp16" with an absolute floor
    for outputs that cancel to ~0.  `slack` ([M, N] or scalar, absolute): see ref_rounding_slack()."""
    o, r = out.detach().float().cpu(), ref.detach().float().cpu()
    assert o.shape == r.shape, (o.shape, r.shape)
    assert torch.isfinite(o).all(), f"{what}: non-finite output"
    rms = r.pow(2).mean().sqrt().item()
    err = (o - r).abs()
    tol = rel * r.abs() + rel * rms
    if slack is not None:
        tol = tol + slack
    bad = err > tol
    _record(what, rel, float((err / tol).max().item()) if err.numel() else 0.0)
    assert not bad.any(), (f"{what}: {int(bad.sum())}/{bad.numel()} outside {rel:g} rel; max abs err "
                           f"{err.max().item():.3e}, rms(ref) {rms:.3e}, worst ratio {(err / tol).max().item():.2f}")
