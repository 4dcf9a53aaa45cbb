"""Generate tests/golden/moe_route_cases.npz from transformers' own routing code (transformers 5.5).

  * softmax: MixtralTopKRouter and Qwen3MoeTopKRouter (norm_topk_prob on and off), fed the logits through an fp32 identity
    router weight with TF32 off, so x @ I is exact;
  * grouped sigmoid: DeepseekV3MoE.route_tokens_to_experts (n_group 8, topk_group 4, routed_scaling_factor 2.5) and
    Glm4MoeMoE.route_tokens_to_experts (n_group 1).  The correction biases are drawn >= 0, so every biased score is
    positive and transformers' 0.0 fill of dropped groups selects like -inf.

The grouped path uses topk(sorted=False), so each row's ids are stored sorted, with their weights.  A row whose k-th and
(k+1)-th scores (or, grouped, the topk_group-th and next group scores) lie within 1e-3 is redrawn: no case depends on
fp32 rounding at the selection boundary.

Usage: python tests/golden/make_golden_moe_route.py
"""
import os

import numpy as np
import torch

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
MARGIN = 1e-3
T = 48


def _gap(score, k):
    """Per row: k-th minus (k+1)-th largest score (inf when there is no (k+1)-th)."""
    v = score.sort(dim=-1, descending=True).values
    return v[:, k - 1] - v[:, k] if k < v.shape[1] else torch.full((v.shape[0],), float("inf"), dtype=v.dtype)


def _logits(gen, E, scale, ok):
    """[T, E] fp32 logits, rows redrawn until ok(row logits) holds."""
    x = torch.randn(T, E, generator=gen) * scale
    for _ in range(100):
        bad = ~ok(x)
        if not bad.any():
            return x
        x[bad] = torch.randn(int(bad.sum()), E, generator=gen) * scale
    raise RuntimeError("could not draw well-separated rows")


def softmax_case(name, router_cls, cfg, E, k, norm, gen):
    router = router_cls(cfg)
    with torch.no_grad():
        router.weight.copy_(torch.eye(E))
    x = _logits(gen, E, 2.0, lambda l: _gap(l, k) > MARGIN)  # softmax is monotonic: the logit gap decides
    with torch.no_grad():
        _, w, ids = router(x)
    order = ids.argsort(dim=-1)
    return dict(name=name, scoring=0, logits=x.numpy(), bias=np.zeros(E, np.float32), top_k=k, n_group=1, topk_group=1,
                renormalize=int(norm), scale=1.0, ids=ids.gather(1, order).numpy().astype(np.int32),
                weights=w.float().gather(1, order).numpy())


def sigmoid_case(name, moe, E, k, n_group, topk_group, scale, gen):
    bias = torch.rand(E, generator=gen) * 0.2
    with torch.no_grad():
        moe.gate.e_score_correction_bias.copy_(bias)

    def ok(l):
        c = torch.sigmoid(l.double()) + bias.double()
        gs = c.view(T, n_group, E // n_group).sort(-1, descending=True).values[..., :2].sum(-1)
        good = _gap(gs, topk_group) > MARGIN
        top = gs.sort(dim=-1, descending=True, stable=True).indices[:, :topk_group]
        kept = torch.zeros_like(gs, dtype=torch.bool).scatter_(1, top, True)
        masked = c.masked_fill(~kept.repeat_interleave(E // n_group, 1), float("-inf"))
        return good & (_gap(masked, k) > MARGIN)

    x = _logits(gen, E, 2.0, ok)
    with torch.no_grad():
        ids, w = moe.route_tokens_to_experts(x.clone())
    order = ids.argsort(dim=-1)
    return dict(name=name, scoring=1, logits=x.numpy(), bias=bias.numpy(), top_k=k, n_group=n_group,
                topk_group=topk_group, renormalize=int(moe.norm_topk_prob), scale=float(scale),
                ids=ids.gather(1, order).numpy().astype(np.int32), weights=w.float().gather(1, order).numpy())


def main():
    from transformers import DeepseekV3Config, Glm4MoeConfig, MixtralConfig, Qwen3MoeConfig
    from transformers.models.deepseek_v3.modeling_deepseek_v3 import DeepseekV3MoE
    from transformers.models.glm4_moe.modeling_glm4_moe import Glm4MoeMoE
    from transformers.models.mixtral.modeling_mixtral import MixtralTopKRouter
    from transformers.models.qwen3_moe.modeling_qwen3_moe import Qwen3MoeTopKRouter

    gen = torch.Generator().manual_seed(2026)
    cases = [
        softmax_case("mixtral_8_top2", MixtralTopKRouter,
                     MixtralConfig(num_local_experts=8, num_experts_per_tok=2, hidden_size=8), 8, 2, True, gen),
        softmax_case("qwen3_128_top8_norm", Qwen3MoeTopKRouter,
                     Qwen3MoeConfig(num_experts=128, num_experts_per_tok=8, hidden_size=128, norm_topk_prob=True),
                     128, 8, True, gen),
        softmax_case("qwen2_60_top4_nonorm", Qwen3MoeTopKRouter,
                     Qwen3MoeConfig(num_experts=60, num_experts_per_tok=4, hidden_size=60, norm_topk_prob=False),
                     60, 4, False, gen),
        sigmoid_case("deepseek_v3_256_top8_g8_4", DeepseekV3MoE(DeepseekV3Config(
            n_routed_experts=256, num_experts_per_tok=8, n_group=8, topk_group=4, routed_scaling_factor=2.5,
            hidden_size=16, moe_intermediate_size=4, n_shared_experts=1, norm_topk_prob=True)), 256, 8, 8, 4, 2.5, gen),
        sigmoid_case("glm4_moe_160_top8_g1", Glm4MoeMoE(Glm4MoeConfig(
            n_routed_experts=160, num_experts_per_tok=8, n_group=1, topk_group=1, routed_scaling_factor=2.5,
            hidden_size=16, moe_intermediate_size=4, n_shared_experts=1, norm_topk_prob=True)), 160, 8, 1, 1, 2.5, gen),
    ]
    out = {}
    for c in cases:
        for key, v in c.items():
            if key != "name":
                out[f"{c['name']}/{key}"] = np.asarray(v)
    out["names"] = np.array([c["name"] for c in cases])
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "moe_route_cases.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(cases)} cases of {T} tokens")


if __name__ == "__main__":
    main()
