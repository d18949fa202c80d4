"""CPU statement of the min-p filter (sq_min_p_filter_per_seq, csrc/sq_sampling.cu) -- TEST INFRASTRUCTURE, never imported
by the product.  vLLM's rule softmax(x / T)_i >= min_p * max softmax(x / T) in logit space, with the kernel's fp32
roundings, so the two agree bit for bit without an exp or a log on the device.
"""
import math

import torch


def min_p_filter(logits: torch.Tensor, min_p: float, T: float) -> torch.Tensor:
    """A copy of the (..., V) fp16 `logits` in which every token whose probability at temperature T is below min_p times
    its row's largest becomes -inf.  With x the fp32 row, m its max over the non-NaN entries and thr = fp32(T) *
    fp32(ln min_p) (ln in double precision, one fp32 multiply), token i stays when x_i is NaN, x_i == m or fp32(x_i - m)
    >= thr.  min_p == 0 is off."""
    out = logits.clone()
    if min_p == 0:
        return out
    x = logits.float()
    nan = torch.isnan(x)
    m = torch.where(nan, float("-inf"), x).amax(-1, keepdim=True)
    thr = torch.tensor(T, dtype=torch.float32) * torch.tensor(math.log(min_p), dtype=torch.float32)
    keep = nan | (x == m) | ((x - m) >= thr)
    return out.masked_fill_(~keep, float("-inf"))
