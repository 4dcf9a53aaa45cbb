"""TEST INFRASTRUCTURE ONLY — float64 statement of the MoE routing of include/b2q.h (b2q_moe_route).

Both modes select by a score, break ties toward the lower index (groups and experts alike) and order the slots by
descending score, ties by lower index; NaN scores select as -inf.
  * softmax: score = the logit; p = exp(l - max) / sum exp(l - max); w = p (/ sum of the selected p) * scale.
  * grouped sigmoid: s = sigmoid(l), c = s + bias; group score = sum of the group's two largest c; the topk_group best
    groups are kept and experts of the others count as -inf; w = s (/ (sum of the selected s + 1e-20)) * scale.
Device-agnostic torch; every result is float64 except the int64 ids.
"""
import torch

__all__ = ["route_softmax", "route_grouped_sigmoid", "route_weights", "sigmoid_scores", "group_scores"]


def _desc_order(score):
    """Indices by descending score, ties to the lower index (NaN as -inf)."""
    score = torch.nan_to_num(score, nan=float("-inf"))
    return torch.sort(score, dim=-1, descending=True, stable=True).indices


def sigmoid_scores(logits, bias):
    """(s, c) in float64: s = sigmoid(l), c = s + bias."""
    s = torch.sigmoid(logits.to(torch.float64))
    return s, s + bias.to(device=s.device, dtype=torch.float64)


def group_scores(c, n_group):
    """[T, n_group]: the sum of the two largest c of each group of E / n_group consecutive experts."""
    T, E = c.shape
    return c.view(T, n_group, E // n_group).sort(dim=-1, descending=True).values[..., :2].sum(-1)


def route_weights(logits, ids, scoring, renormalize=True, scale=1.0):
    """The weights of experts `ids` [T, k] of each row: p (softmax) or s (sigmoid), renormalised over the row's ids."""
    l = logits.to(torch.float64)
    ids = ids.to(device=l.device, dtype=torch.int64)
    if scoring == "softmax":
        p = torch.softmax(l, dim=-1)
        w = p.gather(1, ids)
        if renormalize:
            w = w / w.sum(-1, keepdim=True)
    else:
        w = torch.sigmoid(l).gather(1, ids)
        if renormalize:
            w = w / (w.sum(-1, keepdim=True) + 1e-20)
    return w * scale


def route_softmax(logits, top_k, renormalize=True, scale=1.0):
    """(ids int64 [T, k], weights float64 [T, k], selection scores float64 [T, E])."""
    l = logits.to(torch.float64)
    ids = _desc_order(l)[:, :top_k]
    return ids, route_weights(l, ids, "softmax", renormalize, scale), l


def route_grouped_sigmoid(logits, bias, top_k, n_group, topk_group, renormalize=True, scale=1.0):
    """(ids int64 [T, k], weights float64 [T, k], masked selection scores float64 [T, E]: c in the kept groups, -inf
    elsewhere, kept groups bool [T, n_group])."""
    _, c = sigmoid_scores(logits, bias)
    T, E = c.shape
    gsc = group_scores(c, n_group)
    kept = torch.zeros(T, n_group, dtype=torch.bool, device=c.device)
    kept.scatter_(1, _desc_order(gsc)[:, :topk_group], True)
    masked = c.masked_fill(~kept.repeat_interleave(E // n_group, dim=1), float("-inf"))
    ids = _desc_order(masked)[:, :top_k]
    return ids, route_weights(logits, ids, "sigmoid", renormalize, scale), masked, kept
