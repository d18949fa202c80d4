"""CPU statement of the per-sequence repetition / frequency / presence penalties (sq_penalize_rows_batch): float32 torch,
row by row from the growmap's ancestor-or-self matrix.

Row b*S + k is node k of sequence b.  Its context is the committed tokens[b, :P] (slot P-1 is node 0) and the tokens at
slots P-1+j of node k's ancestors-or-self j >= 1.  c_all(t) counts t in the context, c_out(t) only at slots >= L_b (the
prompt length); ids outside [0, V) are ignored.  Each finite logit x of a context token becomes, in fp32 with one rounding
per operation: x < 0 ? x * rho : x / rho (c_all > 0), then x - f * c_out, then - p (c_out > 0); clamped to +-65504 and
rounded to fp16.  Non-finite logits, frozen sequences and neutral ones (rho = 1, f = 0, p = 0) are left as they are."""
from typing import Optional, Sequence

import torch

F32 = torch.float32
FP16_MAX = 65504.0


def is_neutral(rep: float, freq: float, pres: float) -> bool:
    return rep == 1.0 and freq == 0.0 and pres == 0.0


def row_context(tokens_b: torch.Tensor, P: int, mask01: torch.Tensor, k: int):
    """-> (slots, ids) of row k's context: slots 0 .. P-1, then P-1+j for the ancestors-or-self j >= 1 of node k."""
    path = [P - 1 + j for j in range(1, mask01.shape[0]) if bool(mask01[k, j])]
    slots = torch.cat([torch.arange(P), torch.tensor(path, dtype=torch.long)])
    return slots, tokens_b[slots]


def penalize_row(row: torch.Tensor, ids: torch.Tensor, is_out: torch.Tensor, rep: float, freq: float,
                 pres: float) -> torch.Tensor:
    """One fp16 row penalised for the context ids (int64) with output flags is_out (bool)."""
    V = row.shape[0]
    ok = (ids >= 0) & (ids < V)
    ids, is_out = ids[ok], is_out[ok]
    c_all = torch.bincount(ids, minlength=V)
    c_out = torch.bincount(ids[is_out], minlength=V)
    x = row.to(F32)
    rho, f, p = (torch.tensor(v, dtype=F32) for v in (rep, freq, pres))
    y = torch.where(x < 0, x * rho, x / rho)
    y = torch.where(c_all > 0, y, x)
    z = (y - f * c_out.to(F32)) - p
    y = torch.where(c_out > 0, z, y)
    y = y.clamp(-FP16_MAX, FP16_MAX).to(torch.float16)
    return torch.where(torch.isfinite(x) & (c_all > 0), y, row)


def penalize_rows(logits: torch.Tensor, tokens: torch.Tensor, P: Sequence[int], prompt_len: Sequence[int],
                  mask01: torch.Tensor, rep: Sequence[float], freq: Sequence[float], pres: Sequence[float],
                  frozen: Optional[Sequence[bool]] = None) -> torch.Tensor:
    """The (>= B*S, V) fp16 logits after the penalties of every sequence (a new tensor; rows from B*S on are copied).
    tokens: (B, M) int64; P, prompt_len: per sequence; mask01: (S, S) ancestor-or-self; rep, freq, pres: per sequence,
    float32 values."""
    B, S = tokens.shape[0], mask01.shape[0]
    out = logits.clone()
    for b in range(B):
        if (frozen is not None and frozen[b]) or is_neutral(rep[b], freq[b], pres[b]):
            continue
        for k in range(S):
            slots, ids = row_context(tokens[b], int(P[b]), mask01, k)
            out[b * S + k] = penalize_row(logits[b * S + k], ids, slots >= int(prompt_len[b]), rep[b], freq[b], pres[b])
    return out
