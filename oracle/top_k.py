"""CPU statement of the top-k filter (sq_top_k_filter, csrc/sq_sampling.cu) -- TEST INFRASTRUCTURE, never imported by the
product.  The kernel selects with integer count histograms instead of a sort; counts are exact, so its result is the
sort's bit for bit and needs no separate restatement of the algorithm.
"""
import torch


def top_k_filter(logits: torch.Tensor, k: int) -> torch.Tensor:
    """A copy of the (n, V) fp16 `logits` in which only the k best of each row keep their value and every other one is
    -inf.  Ranking: a stable descending sort of the raw fp16 row (equal values by ascending index; -0 equals +0, NaN
    ranks first, -inf last).  k == 0 is off and k >= V filters nothing."""
    out = logits.clone()
    if k == 0 or k >= logits.shape[-1]:
        return out
    _, idx = torch.sort(logits, dim=-1, descending=True, stable=True)
    return out.scatter_(-1, idx[..., k:], float("-inf"))
