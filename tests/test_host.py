"""CPU: host-side logic and the C-ABI surface (no compute calls without a GPU)."""
import ctypes
import os
import re

import pytest
import torch

import gptqmodel_b200 as g
from gptqmodel_b200 import B200QuantLinear

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "b2q.h")).read()
    declared = set(re.findall(r"\b(b2q_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(g.SYMBOLS), (declared, set(g.SYMBOLS))
    raw = ctypes.CDLL(g.LIB_PATH)
    for name in declared:
        assert hasattr(raw, name), name
    assert g.lib.b2q_version() == g.ABI_VERSION


def test_abi_argument_validation_without_gpu():
    assert g.lib.b2q_packed_bytes(4096, 4096, 4) == 4096 * 4096 // 2
    assert g.lib.b2q_packed_bytes(256, 128, 8) == 256 * 128
    assert g.lib.b2q_workspace_bytes(1, 4096, 4096, 1) == 4096 * 2  # tier-independent bound: any act-order layer, any M
    # exact sizes for b2q_mm's own dispatch: the decode / GEMV tiers gather x[perm] themselves (ADVICE r01: a 4-bit g32
    # act-order layer at M = 1 has no decode tier and must get its workspace)
    assert g.lib.b2q_mm_workspace_bytes(1, 4096, 4096, 4, 128, 1) == 0
    assert g.lib.b2q_mm_workspace_bytes(8, 4096, 4096, 4, 64, 1) == 0
    assert g.lib.b2q_mm_workspace_bytes(1, 4096, 4096, 8, 128, 1) == 0
    assert g.lib.b2q_mm_workspace_bytes(1, 4096, 4096, 4, 32, 1) == 4096 * 2
    assert g.lib.b2q_mm_workspace_bytes(1, 4160, 4096, 4, 64, 1) == 4160 * 2   # K % 128 != 0
    assert g.lib.b2q_mm_workspace_bytes(9, 4096, 4096, 4, 128, 1) == 9 * 4096 * 2
    assert g.lib.b2q_mm_workspace_bytes(2, 4096, 4096, 8, 128, 1) == 2 * 4096 * 2
    assert g.lib.b2q_mm_workspace_bytes(300, 4096, 4096, 4, 128, 0) == 0
    assert g.lib.b2q_workspace_bytes(16, 4096, 4096, 1) == 16 * 4096 * 2
    assert g.lib.b2q_workspace_bytes(16, 4096, 4096, 0) == 0
    assert g.lib.b2q_prepack(None, None, None, 64, 64, 4, None) == -2
    assert b"null pointer" in g.lib.b2q_last_error()
    one = ctypes.c_void_p(16)
    assert g.lib.b2q_prepack(one, None, one, 60, 64, 4, None) == -2
    assert b"K=60" in g.lib.b2q_last_error()
    assert g.lib.b2q_mm(one, one, one, None, None, None, one, 1, 64, 64, 3, 32, 0, None, 0, None) == -2
    assert b"bits=3" in g.lib.b2q_last_error()
    assert g.lib.b2q_mm(one, one, one, None, None, None, one, 1, 64, 64, 4, 48, 0, None, 0, None) == -2
    assert b"group_size=48" in g.lib.b2q_last_error()
    assert g.lib.b2q_mm(one, one, one, None, None, None, one, 0, 64, 64, 4, 32, 0, None, 0, None) == 0  # M == 0
    with pytest.raises(g.B2QError):
        g.check(-2, "x")


def test_validate_follows_reference_convention():
    ok, err = B200QuantLinear.validate(bits=1, group_size=128, in_features=128, out_features=128)
    assert not ok and isinstance(err, NotImplementedError)
    for b in (2, 3, 5, 6, 7):  # widened exactly to 4- / 8-bit fields at post_init (gptqmodel_b200/layouts.py)
        ok, err = B200QuantLinear.validate(bits=b, group_size=128, in_features=128, out_features=128)
        assert ok and err is None
    ok, err = B200QuantLinear.validate(bits=4, group_size=16, in_features=128, out_features=128)
    assert not ok and isinstance(err, NotImplementedError)
    ok, err = B200QuantLinear.validate(bits=4, group_size=128, in_features=100, out_features=128)
    assert not ok
    ok, err = B200QuantLinear.validate(bits=4, group_size=128, in_features=4096, out_features=4096,
                                       pack_dtype=torch.int32, dtype=torch.bfloat16)
    assert ok and err is None
    with pytest.raises(NotImplementedError):
        B200QuantLinear(bits=16, group_size=128, desc_act=False, sym=True, in_features=128, out_features=128)
    for attr in ("SUPPORTS_BACKENDS", "SUPPORTS_METHODS", "SUPPORTS_FORMATS", "SUPPORTS_BITS", "SUPPORTS_GROUP_SIZE",
                 "SUPPORTS_DESC_ACT", "SUPPORTS_SYM", "SUPPORTS_SHARDS", "SUPPORTS_TRAINING", "SUPPORTS_AUTO_PADDING",
                 "SUPPORTS_IN_FEATURES_DIVISIBLE_BY", "SUPPORTS_OUT_FEATURES_DIVISIBLE_BY", "SUPPORTS_PACK_DTYPES",
                 "SUPPORTS_ADAPTERS", "SUPPORTS_DEVICES", "SUPPORTS_PLATFORM", "SUPPORTS_DTYPES"):
        assert getattr(B200QuantLinear, attr) is not None, attr  # verify_supports_params (qlinear/__init__.py:300-332)
    assert B200QuantLinear.REQUIRES_FORMAT_V2 is True


def test_checkpoint_buffer_shapes_match_reference_layout():
    # tests/kernels/test_qlinear_hierarchy.py:239-267 — qweight [K*bits/32, N], qzeros [G, N*bits/32], scales [G, N]
    m = B200QuantLinear(bits=4, group_size=128, desc_act=False, sym=True, in_features=512, out_features=256, bias=True)
    assert m.qweight.shape == (512 * 4 // 32, 256) and m.qweight.dtype == torch.int32
    assert m.qzeros.shape == (4, 256 * 4 // 32) and m.scales.shape == (4, 256) and m.scales.dtype == torch.float16
    assert m.g_idx.shape == (512,) and m.g_idx[127] == 0 and m.g_idx[128] == 1
    assert m.bias.shape == (256,)
    m8 = B200QuantLinear(bits=8, group_size=-1, desc_act=False, sym=True, in_features=256, out_features=64)
    assert m8.qweight.shape == (64, 64) and m8.qzeros.shape == (1, 16) and m8.group_size == 256
    sd = m.state_dict()
    assert set(sd) == {"qweight", "qzeros", "scales", "g_idx", "bias"}  # the wire format


def test_no_cpu_fallback():
    m = B200QuantLinear(bits=4, group_size=128, desc_act=False, sym=True, in_features=128, out_features=64)
    with pytest.raises(g.B2QError):
        m.forward(torch.zeros(1, 128, dtype=torch.float16))  # before post_init
    with pytest.raises(g.B2QError):
        m.post_init()  # CPU tensors: must fail loudly, never fall back


def test_v1_to_v2_conversion():
    m = B200QuantLinear(bits=4, group_size=128, desc_act=False, sym=True, in_features=128, out_features=64)
    m.qzeros.data.fill_(0x77777777)
    m.qzero_format(1)
    m.convert_gptq_v1_to_v2()
    assert m.qzero_format() == 2 and int(m.qzeros[0, 0]) == 0x88888888 - (1 << 32)


@pytest.mark.parametrize("version", [1, 2])
def test_decode_launch_plan_invariants(version):
    # host-side planner of the decode tier (b2q_decode.cu / b2q_decode2.cu): every plan must cover all 32-feature
    # tiles and all k-quads, fit one CTA (or one cluster) per SM and stay inside the shared-memory budget
    out = (ctypes.c_int * 8)()
    shapes = [(4096, 4096), (4096, 1024), (4096, 6144), (4096, 14336), (4096, 28672), (14336, 4096), (8192, 8192),
              (8192, 1280), (28672, 8192), (1024, 32), (128, 32), (256, 96), (11008, 4096), (4096, 32000)]
    for K, N in shapes:
        for M in range(1, 9):
            for ks, warps in ((0, 0), (2, 0), (0, 8)):
                rc = g.lib.b2q_debug_decode_plan(version, M, K, N, ks, warps, out)
                if rc != 0:
                    assert ks != 0 or warps != 0 or version == 2, (version, M, K, N)  # the v1 heuristic always finds one
                    continue
                C, pks, pw, gw, qpc, max_tiles, stages, smem = list(out)
                quads, tiles = K // 128, N // 32
                assert 1 <= C and C * pks <= 132 and pks in (1, 2, 4, 8) and pw in (4, 8, 16), list(out)
                assert pw % gw == 0 and stages in (2, 4) and smem <= 200 * 1024, list(out)
                assert qpc * pks >= quads and (pks - 1) * qpc < quads, list(out)  # every rank owns >= 1 quad
                ngroups = pw // gw
                if version == 2 or pks > 1:
                    assert C * ngroups * max_tiles >= tiles, list(out)
                if ks > 0:
                    assert pks == ks
                if warps > 0:
                    assert pw == warps
    assert g.lib.b2q_debug_decode_plan(3, 1, 4096, 4096, 0, 0, out) == -2
    assert g.lib.b2q_debug_decode_plan(2, 9, 4096, 4096, 0, 0, out) == -2


def test_decode_allreduce_argument_validation_without_gpu():
    # the fused row-parallel decode + all-reduce entry point: every bad call is refused before any CUDA work
    one = ctypes.c_void_p(16)
    peers = (ctypes.c_void_p * 2)(16, 16)
    fb = g.lib.b2q_decode_allreduce_flag_bytes()
    assert fb == 8 * 160 * 4
    ok_off = 2 * 2 * 4096 * 4

    def call(M=1, K=256, N=4096, bits=4, world=2, rank=0, peer=peers, off=ok_off, max_elems=4096, ctl=one):
        return g.lib.b2q_decode_allreduce(one, one, one, None, None, one, M, K, N, bits, 128, 0, rank, world, peer, off,
                                          max_elems, ctl, None)

    assert call(world=1) == -2 and b"world" in g.lib.b2q_last_error()
    assert call(world=9) == -2
    assert call(rank=2) == -2
    assert call(M=2) == -2 and b"max_elems" in g.lib.b2q_last_error()       # M*N > max_elems
    assert call(off=ok_off - 16) == -2                                        # flags would overlap the data rows
    assert call(ctl=None) == -2
    assert call(peer=(ctypes.c_void_p * 2)(16, None)) == -2 and b"peer buffer 1" in g.lib.b2q_last_error()
    assert call(bits=8) == -2 and b"bits=4" in g.lib.b2q_last_error()
    assert call(M=9, max_elems=9 * 4096, off=2 * 2 * 9 * 4096 * 4) == -2     # decode tier: <= 8 tokens


def test_row_parallel_wrapper_and_moe_block_single_process():
    # host logic without a process group: the wrappers fall through to the inner module / skip the collective
    from gptqmodel_b200 import moe, tp

    class Dense(torch.nn.Module):
        def __init__(self, K, N, seed):
            super().__init__()
            self.w = (torch.randn(K, N, generator=torch.Generator().manual_seed(seed)) * 0.1)
            self.perm, self.bits = None, 4

        def forward(self, x):
            return (x.float() @ self.w).to(x.dtype)

    x = torch.randn(3, 16).to(torch.float16)
    inner = Dense(16, 8, 0)
    assert torch.equal(tp.RowParallelLinear(inner)(x), inner(x))
    E = 3
    blk = moe.MoEExperts([Dense(16, 32, 10 + e) for e in range(E)], [Dense(16, 32, 20 + e) for e in range(E)],
                         [Dense(32, 16, 30 + e) for e in range(E)])
    ids, w = moe.route_topk(torch.randn(3, E, generator=torch.Generator().manual_seed(1)), 2)
    got = blk(x, ids, w)
    ref = torch.zeros(3, 16)
    for t in range(3):
        for j in range(2):
            e = int(ids[t, j])
            xt = x[t:t + 1]
            h = torch.nn.functional.silu(blk.w1[e](xt)) * blk.w3[e](xt)
            ref[t] += float(w[t, j]) * blk.w2[e](h)[0].float()
    assert torch.allclose(got.float(), ref, atol=2e-3, rtol=2e-2)
    with pytest.raises(ValueError):
        moe.MoEExperts([], [], [])


def test_lora_adapter_matches_reference_arithmetic(tmp_path):
    # adapter/adapter.py:150-178: out += (x @ lora_A) @ lora_B ; PEFT files hold the transposes
    from safetensors.torch import save_file
    from gptqmodel_b200.adapter import Lora
    gen = torch.Generator().manual_seed(0)
    K, N, r = 64, 32, 4
    A, B = torch.randn(K, r, generator=gen).to(torch.float16), torch.randn(r, N, generator=gen).to(torch.float16)
    x = torch.randn(2, 3, K, generator=gen).to(torch.float16)
    out = torch.randn(2, 3, N, generator=gen).to(torch.float16)
    ad = Lora(rank=r, lora_A=A, lora_B=B)
    ad.post_init("model.layers.0.self_attn.q_proj", "cpu")
    got = ad.apply(x=x, out=out.clone())
    assert torch.equal(got, out + ((x.reshape(-1, K) @ A) @ B).view(2, 3, N))
    save_file({"base_model.model.model.layers.0.self_attn.q_proj.lora_A.weight": A.T.contiguous(),
               "base_model.model.model.layers.0.self_attn.q_proj.lora_B.weight": B.T.contiguous()},
              str(tmp_path / "adapter_model.safetensors"))
    ad2 = Lora(path=str(tmp_path))
    ad2.post_init("model.layers.0.self_attn.q_proj", "cpu")
    assert ad2.rank == r and torch.equal(ad2.lora_A, A) and torch.equal(ad2.lora_B, B)
    assert ad2.apply(x=x.to(torch.bfloat16), out=out.to(torch.bfloat16).clone()).dtype == torch.bfloat16
    assert ad2.lora_A.dtype == torch.bfloat16      # moved to the activations' dtype on first use, like the reference
    with pytest.raises(KeyError):
        Lora(path=str(tmp_path)).post_init("model.layers.9.mlp.up_proj", "cpu")
    with pytest.raises(ValueError):
        Lora(rank=8, lora_A=A, lora_B=B).post_init("x", "cpu")
    assert Lora.name() == "lora" and Lora.parameter_keys() == ["lora_A", "lora_B"] and ad.to_dict()["rank"] == r
