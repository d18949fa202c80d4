"""CPU statement of the per-sequence allowed-token mask and logit bias (sq_logit_bias_rows_batch): float32 torch, row by
row.

Rows b*S .. b*S+S-1 belong to sequence b, and every one of them gets the same processing (the rule does not depend on the
tree).  1. Mask: with an allowed set, every entry whose id is not in it becomes -inf, NaN and +inf included; allowed
entries are left as they are.  2. Bias: for each (id, beta) in order, if the id is allowed and the fp16 logit x is finite,
x becomes fp16(clamp(float(x) + beta, -65504, 65504)), the add one fp32 round-to-nearest operation.  Non-finite logits,
frozen sequences and neutral ones (no allowed set, no entries) are left as they are."""
from typing import Optional, Sequence

import torch

F32 = torch.float32
FP16_MAX = 65504.0


def allowed_vector(allowed, V: int) -> Optional[torch.Tensor]:
    """(V,) bool of an allowed set (None: no mask)."""
    if allowed is None:
        return None
    ok = torch.zeros(V, dtype=torch.bool)
    ok[torch.as_tensor(list(allowed), dtype=torch.int64)] = True
    return ok


def process_row(row: torch.Tensor, ok: Optional[torch.Tensor], bias: Sequence) -> torch.Tensor:
    """One fp16 row after the mask ok ((V,) bool or None) and the (id, beta) entries of bias (beta fp32 values)."""
    return process_block(row.unsqueeze(0), ok, bias)[0]


def process_block(rows: torch.Tensor, ok: Optional[torch.Tensor], bias: Sequence) -> torch.Tensor:
    """(n, V) fp16 rows of one sequence, each processed by process_row's rule (column by column for the bias)."""
    V = rows.shape[1]
    out = rows.clone()
    if ok is not None:
        out[:, ~ok] = float("-inf")
    for t, beta in bias:
        t = int(t)
        if not 0 <= t < V or (ok is not None and not bool(ok[t])):
            continue
        x = out[:, t].to(F32)
        y = (x + torch.tensor(beta, dtype=F32)).clamp(-FP16_MAX, FP16_MAX).to(torch.float16)
        out[:, t] = torch.where(torch.isfinite(x), y, out[:, t])
    return out


def process_rows(logits: torch.Tensor, S: int, allowed: Sequence, bias: Sequence,
                 frozen: Optional[Sequence[bool]] = None) -> torch.Tensor:
    """The (>= B*S, V) fp16 logits after every sequence's mask and bias (a new tensor; rows from B*S on are copied).
    allowed: per sequence, None or a collection of ids; bias: per sequence, None or a sequence of (id, beta) pairs."""
    B, V = len(allowed), logits.shape[1]
    out = logits.clone()
    for b in range(B):
        if (frozen is not None and frozen[b]) or (allowed[b] is None and not bias[b]):
            continue
        out[b * S:(b + 1) * S] = process_block(logits[b * S:(b + 1) * S], allowed_vector(allowed[b], V), bias[b] or ())
    return out
