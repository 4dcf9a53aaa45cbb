"""CPU: the block oracle of the QQQ MoE path (tests/test_gpu_moe_qqq.py states it stage by stage) against
MoEExperts(grouped=False) over dense stand-in QQQ experts, and the loader on tiny QQQ / FP8 checkpoints with Qwen3-MoE
module names.  The stand-ins run qqq_oracle.forward, the layer arithmetic bit for bit, so the loop and the oracle differ
only in the fp32 order of the final sum over slots."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from helpers import assert_close_rel
from oracle import qqq_oracle as qo

DTYPES = (torch.float16, torch.bfloat16)


class _QqqDense(torch.nn.Module):
    def __init__(self, codes, sc, sg):
        super().__init__()
        self.codes, self.sc, self.sg = codes, sc, sg

    def forward(self, x):
        return qo.forward(x, self.codes, self.sc, self.sg)


def _role(E, N, K, gs, gen):
    out = []
    for _ in range(E):
        codes = torch.randint(0, 16, (K, N), generator=gen).to(torch.uint8)
        sc = (torch.rand(N, generator=gen) + 0.5) / (127 * K ** 0.5)
        sg = (torch.rand(K // 128, N, generator=gen) * 14.9 + 1.0).to(torch.float16) if gs == 128 else None
        out.append(_QqqDense(codes, sc / 8 if sg is not None else sc, sg))
    return out


def qqq_block_oracle(x, ids, w, roles):
    """y_t = T(sum_j fp32(w_j * yp_j)) in slot order, yp_j = T(F(Q(h), W2_e)), h = T(T(silu(g)) * u),
    g / u = T(F(Q(x_t), W1_e / W3_e)) (include/b2q.h)."""
    dt = x.dtype
    T, top_k = ids.shape
    acc = torch.zeros(T, roles["w2"][0].codes.shape[1], dtype=torch.float32)
    for j in range(top_k):
        for t in range(T):
            e = int(ids[t, j])
            xt = x[t:t + 1]
            g, u = roles["w1"][e](xt).float(), roles["w3"][e](xt).float()
            h = (F.silu(g).to(dt).float() * u).to(dt)
            acc[t] += w[t, j].float() * roles["w2"][e](h)[0].float()
    return acc.to(dt)


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_qqq_oracle_matches_module_loop(dt):
    from gptqmodel_b200 import moe

    gen = torch.Generator().manual_seed(5)
    E, K, I = 5, 256, 192
    roles = {"w1": _role(E, I, K, 128, gen), "w3": _role(E, I, K, 128, gen), "w2": _role(E, K, I, -1, gen)}
    blk = moe.MoEExperts(roles["w1"], roles["w3"], roles["w2"], grouped=False)
    for T, top_k, routing in ((1, 1, "softmax"), (23, 3, "softmax"), (9, 2, "duplicate")):
        x = torch.randn(T, K, generator=gen).to(dt)
        ids, w = moe.route_topk(torch.randn(T, E, generator=gen), top_k)
        if routing == "duplicate":
            ids[:, 1] = ids[:, 0]
        ref = qqq_block_oracle(x, ids, w, roles)
        got = blk(x, ids, w)
        assert got.dtype == dt and got.shape == (T, K)
        # the only difference is the fp32 order of the slot sum: one ulp of T
        assert_close_rel(got, ref, 2.0 ** -8 if dt == torch.float16 else 2.0 ** -6, f"cpu qqq T={T} top_k={top_k}")
        if top_k > 1 and routing == "softmax":
            with pytest.raises(AssertionError, match="outside"):
                assert_close_rel(got, qqq_block_oracle(x, ids, w[:, [1, 0, 2]], roles), 2.0 ** -8, "swapped")


def _save(path, quant, tensors):
    from safetensors.torch import save_file

    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump({"model_type": "qwen3_moe", "quantization_config": quant}, f)
    save_file(tensors, os.path.join(path, "model.safetensors"))


def test_loader_reads_qwen3_moe_expert_checkpoints(tmp_path):
    """QQQ and FP8 expert tensors under Qwen3-MoE names load as B200QqqQuantLinear / B200Fp8QuantLinear modules."""
    from gptqmodel_b200 import B200Fp8QuantLinear, B200QqqQuantLinear
    from gptqmodel_b200.loader import load_quantized_linears

    gen = torch.Generator().manual_seed(1)
    names = ("gate_proj", "up_proj", "down_proj")
    q, f = {}, {}
    for e in range(2):
        for name in names:
            pre = f"model.layers.0.mlp.experts.{e}.{name}"
            codes = torch.randint(0, 16, (256, 128), generator=gen).to(torch.uint8)
            B, sc, sg = qo.pack_qqq(codes, torch.rand(128, generator=gen) * 1e-3,
                                    (torch.rand(2, 128, generator=gen) + 1).half())
            q.update({pre + ".B": B, pre + ".s_channel": sc, pre + ".s_group": sg})
            f.update({pre + ".weight": torch.randn(128, 256, generator=gen).to(torch.float8_e4m3fn),
                      pre + ".weight_scale_inv": torch.rand(1, 2, generator=gen) + 1})
    os.makedirs(tmp_path / "q")
    os.makedirs(tmp_path / "f")
    _save(str(tmp_path / "q"), {"quant_method": "qqq", "bits": 4, "group_size": 128, "sym": True, "desc_act": False,
                                "format": "qqq"}, q)
    _save(str(tmp_path / "f"), {"quant_method": "fp8", "format": "float8_e4m3fn", "weight_scale_method": "block",
                                "weight_block_size": [128, 128]}, f)
    for sub, cls in (("q", B200QqqQuantLinear), ("f", B200Fp8QuantLinear)):
        mods = load_quantized_linears(str(tmp_path / sub), device="cpu")
        assert len(mods) == 6 and all(isinstance(m, cls) for m in mods.values()), sub
