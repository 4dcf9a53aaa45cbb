"""FP8 (e4m3fn, W8A16) MoE experts on the grouped small-batch kernels of gptqmodel_b200/moe.py.

Path: b2q_moe_align -> b2q_moe_gather -> midm_kernel MODE 1 with FP8 = true (gate|up, SiLU-mul epilogue) -> MODE 2
(down, routing weight, scatter) -> b2q_moe_combine.  The arithmetic is the GPTQ grouped path's with W the exact
b2q_fp8_dequant operand, so the block is checked against the float64 oracle of tests/test_gpu_moe.py (moe_oracle,
assert_moe_close: the same tolerance) built on each module's dequantize_weight().
"""
import json
import os

import pytest
import torch

from test_gpu_moe import _route, _skewed, assert_moe_close, moe_oracle

DEV = "cuda"
DTYPES = (torch.float16, torch.bfloat16)
TNAME = {torch.float16: "fp16", torch.bfloat16: "bf16"}


def _ckpt(E, N, K, method, seed, big=False):
    """E experts' checkpoint tensors [(weight e4m3 [N, K], weight_scale_inv)] with the reference's quantiser recipe;
    big: scales above 65504 (an fp16 table that overflows)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(E):
        W = torch.randn(N, K, generator=g) / K ** 0.5
        if method == "tensor":
            s = 448.0 / W.abs().amax()
            w = (W * s).clamp(-448, 448)
        elif method == "row":
            s = 448.0 / W.abs().amax(1)
            w = (W * s[:, None]).clamp(-448, 448)
        else:
            Wb = W.reshape(N // 128, 128, K // 128, 128)
            s = 448.0 / Wb.abs().amax(dim=(1, 3))
            w = (Wb * s[:, None, :, None]).clamp(-448, 448).reshape(N, K)
        if big:
            s = s * 1e4  # W = w / s: still finite weights in bf16, an inf scale in fp16
        out.append((w.to(torch.float8_e4m3fn), s.to(torch.float32)))
    return out


def _mods(ck):
    from gptqmodel_b200 import B200Fp8QuantLinear

    return [B200Fp8QuantLinear.from_checkpoint_tensors(w, s, device=DEV) for w, s in ck]


def _block(E, K, I, method, seed=1, big=False, grouped=True):
    from gptqmodel_b200 import moe

    mods = [_mods(_ckpt(E, n, k, method, seed + i, big)) for i, (n, k) in enumerate(((I, K), (I, K), (K, I)))]
    return moe.MoEExperts(*mods, grouped=grouped)


def _weights(blk, dt):
    """moe_oracle's weights(e, rows): W1, W3, W2 in float64 from the exact operand of b2q_fp8_dequant."""
    cache = {}

    def get(e, rows):
        if e not in cache:
            cache[e] = tuple(m[e].dequantize_weight(dtype=dt).double() for m in (blk.w1, blk.w3, blk.w2))
        return cache[e]
    return get


def _x(T, K, dt, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(T, K, device=DEV, generator=gen) * 0.5).to(dt)


STACKS = {  # E, K, I, top_k, scale layout
    "block_qwen_like": (16, 512, 384, 8, "block"),
    "row_mixtral_like": (8, 512, 1024, 2, "row"),
    "tensor_tail": (6, 256, 192, 4, "tensor"),  # I % 128 == 64: a partly filled feature tile
}
_BLOCKS = {}


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    _BLOCKS.clear()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _stack(name):
    if name not in _BLOCKS:
        E, K, I, _, method = STACKS[name]
        blk = _block(E, K, I, method)
        assert "fp8" in blk._stack
        _BLOCKS[name] = blk
    return _BLOCKS[name]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", list(STACKS))
def test_block_against_float64_oracle(name, dt):
    """T = 1..300 (every T below 17, a sample above) and 2048, top_k 1, 2, 4, 8, softmax / skewed / sparse routing: the
    grouped block against the float64 oracle on b2q_fp8_dequant's W; the loop over the same modules too at a few T."""
    blk = _stack(name)
    E, K, _, top_k, _ = STACKS[name]
    loop = type(blk)(list(blk.w1), list(blk.w3), list(blk.w2), grouped=False)
    W = _weights(blk, dt)
    for T in list(range(1, 17)) + [31, 64, 65, 127, 128, 129, 200, 255, 300, 2048]:
        k = min([1, 2, 4, 8][T % 4] if T < 17 else top_k, E)
        ids, w = (_skewed if T % 3 == 0 else _route)(T, E, k, seed=T)
        if T % 5 == 0:
            ids = torch.where(ids % 3 == 0, ids, torch.full_like(ids, E - 1))  # most experts empty
        x = _x(T, K, dt, seed=T)
        ref = moe_oracle(x, ids, w, W)
        y = blk(x, ids, w)
        assert_moe_close(y, ref, f"fp8 moe {name} {TNAME[dt]} T={T} top_k={k}")
        if T in (1, 17, 300):
            assert_moe_close(loop(x, ids, w), ref, f"fp8 moe {name} {TNAME[dt]} T={T} loop")
        if T == 300:
            assert torch.equal(blk(x, ids, w), y)


@pytest.mark.gpu
def test_fp16_refused_on_overflowing_scales():
    """A scale_inv above 65504 is inf in the fp16 table: fp16 input raises ValueError, as the layer does; bf16 is served
    and matches the oracle."""
    E, K, I = 4, 256, 128
    blk = _block(E, K, I, "row", seed=7, big=True)
    assert "fp8" in blk._stack
    ids, w = _route(5, E, 2, seed=5)
    with pytest.raises(ValueError, match="overflows fp16"):
        blk(_x(5, K, torch.float16, seed=5), ids, w)
    x = _x(5, K, torch.bfloat16, seed=5)
    assert_moe_close(blk(x, ids, w), moe_oracle(x, ids, w, _weights(blk, torch.bfloat16)), "fp8 moe big scales bf16")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_graph_replay_equals_eager(dt):
    """The five launches captured in a CUDA graph: after new ids / weights are copied in, a replay equals an eager run."""
    blk = _stack("block_qwen_like")
    E, K, _, top_k, _ = STACKS["block_qwen_like"]
    T = 65
    x = _x(T, K, dt, seed=65)
    ids, w = _route(T, E, top_k, seed=65)
    idc, wc = ids.clone(), w.clone()
    s_ = torch.cuda.Stream()
    s_.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s_):
        blk(x, idc, wc)
    torch.cuda.current_stream().wait_stream(s_)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        yg = blk(x, idc, wc)
    for ids2, w2 in (_skewed(T, E, top_k, seed=7), _route(T, E, top_k, seed=66)):
        idc.copy_(ids2)
        wc.copy_(w2)
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, blk(x, ids2, w2))
    del gr


@pytest.mark.gpu
def test_large_prefill_splits_the_grid():
    """E = 256, top_k = 8, T = 8192: 65536 rows give more than 65535 (expert, token block) pairs in both launches."""
    E, K, I, top_k, T = 256, 256, 128, 8, 8192
    blk = _block(E, K, I, "block", seed=11)
    ids, w = _route(T, E, top_k, seed=5)
    assert int(torch.bincount(ids.reshape(-1).cpu(), minlength=E)[E // 2:].sum()) > 0
    for dt in DTYPES:
        x = _x(T, K, dt, seed=T)
        assert_moe_close(blk(x, ids, w), moe_oracle(x, ids, w, _weights(blk, dt)), f"fp8 moe large {TNAME[dt]}")


@pytest.mark.gpu
def test_negative_controls():
    """Slot weights swapped and the next expert's scales fail the comparison; biased, adapted and mixed stacks take the
    loop, and grouped=True refuses them."""
    from gptqmodel_b200 import B200Fp8QuantLinear, Lora, moe
    from gptqmodel_b200._lib import check, lib

    blk = _stack("block_qwen_like")
    E, K, I, top_k, _ = STACKS["block_qwen_like"]
    T, dt = 40, torch.float16
    x = _x(T, K, dt, seed=40)
    ids, w = _route(T, E, top_k, seed=40)
    y = blk(x, ids, w)
    W = _weights(blk, dt)
    assert_moe_close(y, moe_oracle(x, ids, w, W), "control: correct")
    with pytest.raises(AssertionError, match="outside"):
        assert_moe_close(y, moe_oracle(x, ids, w[:, [1, 0] + list(range(2, top_k))], W), "control: swapped weights")

    def next_scales(e, rows):  # expert e's codes with expert e + 1's w2 scales
        W1, W3, _ = W(e, rows)
        m, nxt = blk.w2[e], blk.w2[(e + 1) % E]
        out = torch.empty((m.in_features, m.out_features), dtype=dt, device=DEV)
        check(lib.b2q_fp8_dequant(m.packed.data_ptr(), nxt._scales[dt].data_ptr(), out.data_ptr(), m.in_features,
                                  m.out_features, m._gs, 0, torch.cuda.current_stream().cuda_stream), "dequant")
        return W1, W3, out.double()
    with pytest.raises(AssertionError, match="outside"):
        assert_moe_close(y, moe_oracle(x, ids, w, next_scales), "control: next expert's scales")

    E2, K2, I2 = 2, 256, 128
    ck = [_ckpt(E2, n, k, "row", 30 + i) for i, (n, k) in enumerate(((I2, K2), (I2, K2), (K2, I2)))]
    mods = lambda: [_mods(c) for c in ck]  # noqa: E731
    assert "fp8" in moe.MoEExperts(*mods())._stack
    biased = mods()
    biased[2][1] = B200Fp8QuantLinear.from_checkpoint_tensors(*ck[2][1], bias=torch.zeros(K2), device=DEV)
    gen = torch.Generator().manual_seed(0)
    lora = Lora(lora_A=(torch.randn(K2, 8, generator=gen) * 0.05).half(),
                lora_B=(torch.randn(8, I2, generator=gen) * 0.05).half())
    adapted = mods()
    adapted[0][0] = B200Fp8QuantLinear.from_checkpoint_tensors(*ck[0][0], device=DEV, adapter=lora)
    mixed = mods()
    mixed[1][0] = _mods(_ckpt(1, I2, K2, "block", 50))[0]  # w3 with a 128-k scale group, w1 per-channel
    for what, sets in (("bias", biased), ("adapter", adapted), ("mixed scale groups", mixed)):
        assert moe.MoEExperts(*sets, fuse=False)._stack is None, what
        with pytest.raises(ValueError, match="B200Fp8QuantLinear"):
            moe.MoEExperts(*sets, grouped=True)
    assert moe.MoEExperts(*biased)(x[:, :K2].contiguous(), *_route(T, E2, 2, seed=1)).shape == (T, K2)


@pytest.mark.gpu
def test_qwen3_moe_checkpoint_through_loader(tmp_path):
    """A tiny FP8 safetensors checkpoint (the reference's FP8Config) with Qwen3-MoE module names goes through
    load_quantized_linears and runs grouped, matching the oracle."""
    from safetensors.torch import save_file

    from gptqmodel_b200 import moe
    from gptqmodel_b200.loader import load_quantized_linears

    E, K, I = 4, 256, 384
    proj = {"w1": ("gate_proj", I, K), "w3": ("up_proj", I, K), "w2": ("down_proj", K, I)}
    tensors = {}
    for i, (r, (name, n, k)) in enumerate(proj.items()):
        for e, (wq, s) in enumerate(_ckpt(E, n, k, "block", 70 + i)):
            pre = f"model.layers.0.mlp.experts.{e}.{name}"
            tensors[pre + ".weight"], tensors[pre + ".weight_scale_inv"] = wq, s
    with open(os.path.join(tmp_path, "config.json"), "w") as f:
        json.dump({"model_type": "qwen3_moe", "quantization_config": {
            "quant_method": "fp8", "format": "float8_e4m3fn", "weight_scale_method": "block",
            "weight_block_size": [128, 128]}}, f)
    save_file(tensors, os.path.join(tmp_path, "model.safetensors"))
    mods = load_quantized_linears(str(tmp_path), device=DEV)
    get = lambda r: [mods[f"model.layers.0.mlp.experts.{e}.{proj[r][0]}"] for e in range(E)]  # noqa: E731
    blk = moe.MoEExperts(get("w1"), get("w3"), get("w2"), grouped=True)
    for dt in DTYPES:
        x = _x(9, K, dt, seed=9)
        ids, w = _route(9, E, 2, seed=9)
        assert_moe_close(blk(x, ids, w), moe_oracle(x, ids, w, _weights(blk, dt)), f"fp8 checkpoint {TNAME[dt]}")
