"""GPU parity of the format front-ends: AWQ GEMM-format modules against outputs produced
by the reference's own AwqTorchLinear, full-size AWQ layers against the oracle, and a checkpoint loaded from safetensors.

Lives in its own file so that it is collected AFTER tests/test_gpu_parity.py (the hot path proper).
"""

import pytest
import torch

import oracle
from gptqmodel_b200 import B200AwqQuantLinear, loader
from helpers import assert_close_rel, make_layer, ref_rounding_slack
from test_awq import awq_cases  # noqa: F401  (fixture)
from test_loader import _ckpt_tensors, _write


@pytest.mark.gpu
def test_awq_module_matches_reference_outputs_on_gpu(awq_cases):
    for name, c in awq_cases.items():
        m = B200AwqQuantLinear.from_awq_tensors(c["qweight"], c["qzeros"], c["scales"], c["group_size"], bias=c["bias"])
        y = m(c["x"].cuda())
        # (a) kernel arithmetic: against the layer evaluated in EXACT arithmetic (unrounded W, float64 dot product, one
        # output rounding) at the north-star bar, no slack.  The tiers that serve these token counts apply the scale once
        # per group to an exact integer dot product, i.e. they converge to exactly this.
        ye = oracle.awq_forward_exact(c["x"], c["qweight"], c["qzeros"], c["scales"], c["group_size"], c["bias"])
        assert_close_rel(y, ye, 1e-3, name + " vs exact arithmetic")
        # (b) the oracle that is pinned bit-exact to the reference's dequantize_gemm (per-weight fp16 rounding of W,
        # fp32 accumulation): 1e-3 plus the reference's OWN weight-rounding noise (4 sigma; helpers.ref_rounding_slack —
        # exact arithmetic itself is 1.18x outside the plain criterion on `awq_gK`, tests/test_awq.py)
        yo = oracle.awq_forward(c["x"], c["qweight"], c["qzeros"], c["scales"], c["group_size"], c["bias"])
        assert_close_rel(y, yo, 1e-3, name, slack=ref_rounding_slack(c["W"], c["x"]))
        # (c) the reference's own output: AwqTorchLinear on the CPU accumulates the matmul in fp16 (torch_awq.py:157-197),
        # which differs from any fp32-accumulate result by up to ~1 fp16 ulp -> same bound as the GPTQ twin
        # (test_gpu_parity.py::test_reference_generated_cases)
        assert torch.allclose(y.float().cpu(), c["y_fp16"].float(), rtol=2e-3, atol=2e-3), name
        ybf = m(c["x"].cuda().to(torch.bfloat16))
        assert_close_rel(ybf, c["y_bf16"], 1.6e-2, name + " bf16")


@pytest.mark.gpu
@pytest.mark.parametrize("K,N,gs", [(4096, 4096, 128), (4096, 14336, 64), (14336, 4096, 128)])
def test_awq_full_size_layers_on_gpu(K, N, gs):
    gen = torch.Generator(device="cuda").manual_seed(K + N)
    qw = torch.randint(-(2 ** 31), 2 ** 31 - 1, (K, N // 8), dtype=torch.int32, device="cuda", generator=gen)
    qz = torch.randint(-(2 ** 31), 2 ** 31 - 1, (K // gs, N // 8), dtype=torch.int32, device="cuda", generator=gen)
    sc = (torch.rand(K // gs, N, device="cuda", generator=gen) * 0.01 + 0.005).to(torch.float16)
    m = B200AwqQuantLinear.from_awq_tensors(qw, qz, sc, gs)
    W = oracle.awq_dequantize(qw.cpu(), qz.cpu(), sc.cpu(), gs)
    for M in (1, 7, 64, 300):
        x = (torch.randn(M, K, device="cuda", generator=gen) * 0.5).to(torch.float16)
        ref = oracle.awq_forward(x.cpu(), qw.cpu(), qz.cpu(), sc.cpu(), gs)
        # M <= 8 runs on the decode tier (scale applied once per group): + the reference's own weight-rounding noise
        assert_close_rel(m(x), ref, 1e-3, f"awq K={K} N={N} M={M}", slack=ref_rounding_slack(W, x.cpu()) if M <= 8 else None)


@pytest.mark.gpu
def test_loaded_checkpoint_runs_on_gpu(tmp_path):
    from helpers import assert_close_rel, oracle_forward
    layers = {"m.q_proj": make_layer(512, 256, group_size=128, sym=True, seed=21),
              "m.o_proj": make_layer(512, 128, group_size=64, sym=False, desc_act=True, bias=True, seed=22)}
    cfg = {"bits": 4, "group_size": 128, "sym": True, "checkpoint_format": "gptq_v2",
           "dynamic": {r".*o_proj": {"group_size": 64, "sym": False, "desc_act": True}}}
    _write(str(tmp_path), {n: _ckpt_tensors(L) for n, L in layers.items()}, cfg)
    mods = loader.load_quantized_linears(str(tmp_path), device="cuda")
    x = (torch.randn(5, 512) * 0.5).to(torch.float16)
    from helpers import assert_layer_close
    for n, L in layers.items():
        assert_layer_close(mods[n](x.cuda()), L, x, 1e-3, n)


@pytest.mark.gpu
@pytest.mark.parametrize("bits,gs,sym,desc", [(4, 128, True, False), (4, 64, False, True), (8, 32, False, False)])
def test_dequantize_weight_bit_exact_on_gpu(bits, gs, sym, desc):
    # reference contract: dequantize_weight() (qlinear/__init__.py:947-1021); identity rows through the exact-dequant tier
    from gptqmodel_b200 import B200QuantLinear
    L = make_layer(640, 96, bits=bits, group_size=gs, sym=sym, desc_act=desc, bias=True, seed=40 + bits)
    m = B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], bits, gs,
                                                bias=L["bias"], desc_act=desc, sym=sym)
    W = m.dequantize_weight()
    ref = oracle.dequantize_weight(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], bits)
    assert W.shape == (640, 96) and W.dtype == torch.float16
    assert torch.equal(W.cpu(), ref)
    with pytest.raises(NotImplementedError):
        B200QuantLinear.validate_device("cpu")


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 3, 8, 40, 200])
def test_moe_block_on_gpu(T):
    # BASELINE configs[4] in miniature: g64 asymmetric experts, top-2 routing, tokens grouped per expert (decode tier for
    # small blocks with w1/w3 in one launch, tensor-core tier for larger ones); single GPU -> no collective
    import torch.nn.functional as F
    from gptqmodel_b200 import B200QuantLinear, moe
    from helpers import oracle_forward
    E, K, I, top_k = 4, 256, 512, 2
    layers = [(make_layer(K, I, group_size=64, sym=False, seed=200 + 3 * e),
               make_layer(K, I, group_size=64, sym=False, seed=201 + 3 * e),
               make_layer(I, K, group_size=64, sym=False, seed=202 + 3 * e)) for e in range(E)]
    mk = lambda L: B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, 64,  # noqa: E731
                                                           sym=False)
    blk = moe.MoEExperts([mk(l[0]) for l in layers], [mk(l[1]) for l in layers], [mk(l[2]) for l in layers])
    gen = torch.Generator().manual_seed(T)
    x = (torch.randn(T, K, generator=gen) * 0.5).to(torch.float16)
    ids, w = moe.route_topk(torch.randn(T, E, generator=gen), top_k)
    ref = torch.zeros(T, K)
    for t in range(T):
        for j in range(top_k):
            l1, l3, l2 = layers[int(ids[t, j])]
            xt = x[t:t + 1]
            h = (F.silu(oracle_forward(l1, xt).float()) * oracle_forward(l3, xt).float()).to(torch.float16)
            ref[t] += float(w[t, j]) * oracle_forward(l2, h)[0].float()
    assert blk._stack is not None  # the grouped kernels serve this block (4-bit B200 experts of one shape)
    got = blk(x.cuda(), ids.cuda(), w.cuda())
    assert got.shape == (T, K) and got.dtype == torch.float16
    assert_close_rel(got, ref, 4e-3, f"moe T={T}")   # two chained fp16 layers + fp16 silu: a few ulp on top of 1e-3
    # deterministic (no atomics), and the per-expert loop path (decode / small-batch / prefill tiers per expert block) agrees
    assert torch.equal(got, blk(x.cuda(), ids.cuda(), w.cuda()))
    loop = moe.MoEExperts(list(blk.w1), list(blk.w3), list(blk.w2), grouped=False)
    assert loop._stack is None
    assert_close_rel(loop(x.cuda(), ids.cuda(), w.cuda()), ref, 4e-3, f"moe loop path T={T}")
    # the grouped block has no host synchronisation: it can be captured in a CUDA graph
    xs, idc, wc = x.cuda(), ids.cuda(), w.cuda()
    s_ = torch.cuda.Stream()
    s_.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s_):
        blk(xs, idc, wc)
    torch.cuda.current_stream().wait_stream(s_)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        yg = blk(xs, idc, wc)
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, got)


@pytest.mark.gpu
@pytest.mark.parametrize("sym,gs", [(True, 128), (False, 64)])
def test_fused_gate_up_silu_epilogue_on_gpu(sym, gs):
    # act_fn(gate_proj(x)) * up_proj(x) in one launch, SiLU-mul in the epilogue, rounding at the module
    # boundaries of the reference's separate modules
    import torch.nn.functional as F
    from gptqmodel_b200 import B200QuantLinear
    from gptqmodel_b200.mlp import FusedGateUpSilu
    from helpers import oracle_forward
    K, I = 512, 768
    Lg, Lu = make_layer(K, I, group_size=gs, sym=sym, seed=91), make_layer(K, I, group_size=gs, sym=sym, seed=92)
    mk = lambda L: B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, gs,  # noqa: E731
                                                           sym=sym)
    fused = FusedGateUpSilu(mk(Lg), mk(Lu))
    for M in (1, 7, 40, 128, 200):
        x = (torch.randn(M, K, generator=torch.Generator().manual_seed(M)) * 0.5).to(torch.float16)
        ref = (F.silu(oracle_forward(Lg, x).float()).to(torch.float16).float() * oracle_forward(Lu, x).float()).to(torch.float16)
        got = fused(x.cuda())
        assert got.shape == (M, I) and got.dtype == torch.float16
        assert_close_rel(got, ref, 3e-3, f"gate/up silu M={M}")  # product of two 1e-3 factors + the fp16 silu rounding


@pytest.mark.gpu
def test_lora_adapter_epilogue_on_gpu():
    # forward() ends with adapter.apply(x=x, out=out) (reference contract, qlinear/marlin.py:333-335)
    from gptqmodel_b200 import B200QuantLinear, Lora
    from helpers import oracle_forward
    L = make_layer(512, 256, group_size=128, sym=True, bias=True, seed=77)
    gen = torch.Generator().manual_seed(1)
    A = (torch.randn(512, 8, generator=gen) * 0.05).to(torch.float16)
    B = (torch.randn(8, 256, generator=gen) * 0.05).to(torch.float16)
    m = B200QuantLinear(bits=4, group_size=128, desc_act=False, sym=True, in_features=512, out_features=256, bias=True,
                        adapter=Lora(rank=8, lora_A=A, lora_B=B), register_buffers=False)
    mk = lambda t: torch.nn.Parameter(t.clone().cuda(), requires_grad=False)  # noqa: E731
    m.qweight, m.qzeros, m.scales, m.g_idx, m.bias = (mk(L[k]) for k in ("qweight", "qzeros", "scales", "g_idx", "bias"))
    m.post_init()
    for shape in ((1, 512), (2, 5, 512), (200, 512)):
        x = (torch.randn(*shape, generator=gen) * 0.5).to(torch.float16)
        base = oracle_forward(L, x.reshape(-1, 512))
        ref = (base.float() + ((x.reshape(-1, 512).float() @ A.float()).to(torch.float16).float() @ B.float())).reshape(*shape[:-1], 256)
        assert_close_rel(m(x.cuda()), ref, 2e-3, f"lora {shape}")


@pytest.mark.gpu
def test_tiny_llama_with_b200_quantlinears_on_gpu():
    # the caller side of the hot path: every nn.Linear of a (random-init) HF Llama replaced by a B200QuantLinear, q|k|v and
    # gate|up fused into single decode launches; logits against the same model holding the dequantised dense weights
    import torch.nn as nn
    from gptqmodel_b200 import convert, fuse_siblings
    from test_convert import tiny_llama
    model, dense = tiny_llama(torch.float16), tiny_llama(torch.float16)
    dense_w = {}

    def factory(name, lin):
        q = convert.quantize_linear(lin, bits=4, group_size=128, sym=("mlp" in name), device="cpu", name=name)
        dense_w[name] = oracle.dequantize_weight(q.qweight.data, q.qzeros.data, q.scales.data, q.g_idx.data, 4).T.contiguous()
        for k in ("qweight", "qzeros", "scales", "g_idx"):
            setattr(q, k, nn.Parameter(getattr(q, k).data.cuda(), requires_grad=False))
        q.post_init()
        return q

    swapped = convert.replace_linears(model, factory)
    assert len(swapped) == 14
    for name, W in dense_w.items():
        dense.get_submodule(name).weight.data.copy_(W)
    model, dense = model.cuda(), dense.cuda()
    for layer in model.model.layers:
        assert fuse_siblings([layer.self_attn.q_proj, layer.self_attn.k_proj, layer.self_attn.v_proj])
        assert fuse_siblings([layer.mlp.gate_proj, layer.mlp.up_proj])
    gen = torch.Generator().manual_seed(3)
    for shape in ((2, 9), (1, 1), (3, 1)):     # prefill-like, single-token decode (fused launches), 3 sequences x 1 token
        ids = torch.randint(0, 1000, shape, generator=gen).cuda()
        with torch.inference_mode():
            a = model(ids).logits.float()
            b = dense(ids).logits.float()
        assert a.shape == shape + (1000,) and torch.isfinite(a).all()
        assert (a - b).abs().max().item() < 3e-2 * b.abs().max().item(), shape


@pytest.mark.gpu
@pytest.mark.parametrize("sym,gs", [(False, 64), (True, 128)])
def test_moe_one_token_decode_path(sym, gs):
    """Batch-1 decode through the experts on the decode tier (b2q_moe_decode_*): Mixtral TP-4 shard shapes (4096 x 3584 /
    3584 x 4096), top-2 of 8 experts, against the grouped small-batch kernels on the same stack and the oracle; the expert ids
    are read on the device, so a captured graph follows new routing decisions."""
    import torch.nn.functional as F
    from gptqmodel_b200 import B200QuantLinear, moe
    from helpers import random_layer
    E, K, I, top_k = 8, 4096, 3584, 2
    mk = lambda L: B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, gs,  # noqa: E731
                                                           sym=sym)
    Ls = [(random_layer(K, I, group_size=gs, sym=sym, seed=3 * e, device="cuda"),
           random_layer(K, I, group_size=gs, sym=sym, seed=3 * e + 1, device="cuda"),
           random_layer(I, K, group_size=gs, sym=sym, seed=3 * e + 2, device="cuda")) for e in range(E)]
    blk = moe.MoEExperts([mk(l[0]) for l in Ls], [mk(l[1]) for l in Ls], [mk(l[2]) for l in Ls])
    assert blk._stack is not None and blk._decode_ok(top_k)
    gen = torch.Generator().manual_seed(5)
    x = (torch.randn(1, K, generator=gen) * 0.2).to(torch.float16).cuda()

    def oracle_block(ids, w):
        ref = torch.zeros(1, K, dtype=torch.float64)
        for j in range(top_k):
            l1, l3, l2 = Ls[int(ids[0, j])]
            W1, W3, W2 = (oracle.dequantize_weight(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4).float() for L in (l1, l3, l2))
            g = (x.float() @ W1).to(torch.float16)
            u = (x.float() @ W3).to(torch.float16)
            h = (F.silu(g.float()).to(torch.float16).float() * u.float()).to(torch.float16)
            ref += float(w[0, j]) * (h.float() @ W2).to(torch.float16).double().cpu()
        return ref.float()

    for trial in range(3):
        ids, w = moe.route_topk(torch.randn(1, E, generator=gen), top_k)
        blk.decode_path, blk.fuse_act = True, True
        y_dec = blk(x, ids.cuda(), w.cuda())
        blk.fuse_act = False     # SiLU-mul as its own launch: the same arithmetic, hence the same bits
        assert torch.equal(blk(x, ids.cuda(), w.cuda()), y_dec)
        blk.fuse_act = True
        blk.decode_path = False
        y_grp = blk(x, ids.cuda(), w.cuda())
        ref = oracle_block(ids, w)
        assert_close_rel(y_dec, ref, 4e-3, f"moe decode path trial {trial}")
        assert_close_rel(y_grp, ref, 4e-3, f"moe grouped path trial {trial}")
        assert_close_rel(y_dec, y_grp, 4e-3, f"moe decode vs grouped trial {trial}")
    # CUDA graph: the routing tensors are inputs, not constants
    blk.decode_path = True
    idc, wc = ids.cuda(), w.cuda()
    s_ = torch.cuda.Stream()
    s_.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s_):
        blk(x, idc, wc)
    torch.cuda.current_stream().wait_stream(s_)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        yg = blk(x, idc, wc)
    ids2, w2 = moe.route_topk(torch.randn(1, E, generator=gen), top_k)
    idc.copy_(ids2)
    wc.copy_(w2)
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, blk(x, ids2.cuda(), w2.cuda()))
    assert_close_rel(yg, oracle_block(ids2, w2), 4e-3, "moe decode path, graph replay with new routing")
