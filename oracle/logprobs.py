"""CPU statement of the per-sequence logprobs of a verify step's committed tokens (sq_token_logprobs_batch), in float64.

For sequence b with P = state[b, P_OLD], n_new = state[b, N_NEW], a = P + n_new, the step committed positions P + j for
j < n_new and, when the walk wrote a bonus token (not terminal and a < M), for j = n_new.  Position P + j reads the target
row of the path node at depth j: node 0 for j = 0, else node accept_idx[b, j-1] - (P - 1); its token is tokens[b, P + j]
after the walk (an accepted node that lives at slot a is committed as the bonus token: SpecTree writes the bonus first).
Value: s = fp16(float32(x) * float32(1 / T)), T = 1 for a greedy sequence; the log-softmax of s at the token.  A row with
a +inf or NaN in s, or only -inf, gives NaN throughout.  Top entries: the n best ids by (raw fp16 value descending, -0 equal
to +0, NaN above +inf, equal values by ascending index) and their logprobs."""
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

ST_TERMINAL, ST_N_NEW, ST_P_OLD, ST_M, ST_FROZEN = 2, 3, 4, 8, 9
MAX_LOGPROBS = 20


def committed(state_b: torch.Tensor, M: int) -> int:
    """The number of positions the step committed for a sequence with state row state_b (M: the token row length)."""
    P, n_new = int(state_b[ST_P_OLD]), int(state_b[ST_N_NEW])
    m = int(state_b[ST_M]) if int(state_b[ST_M]) > 0 else M
    return n_new + (1 if not int(state_b[ST_TERMINAL]) and P + n_new < m else 0)


def path_node(state_b: torch.Tensor, accept_b: torch.Tensor, j: int) -> int:
    """The tree node whose target row position P_OLD + j was drawn from."""
    return 0 if j == 0 else int(accept_b[j - 1]) - (int(state_b[ST_P_OLD]) - 1)


def is_bonus_replacement(state_b: torch.Tensor, accept_b: torch.Tensor, j: int) -> bool:
    """Position P_OLD + j (j >= 1) holds the bonus token in place of the accepted node's: that node lived at slot a."""
    return j >= 1 and int(accept_b[j - 1]) == int(state_b[ST_P_OLD]) + int(state_b[ST_N_NEW])


def scaled(row: torch.Tensor, T: float, greedy: bool) -> np.ndarray:
    """The walk's fp16 scaled values s of an fp16 row, as float64."""
    inv = np.float32(1.0) if greedy else np.float32(1.0) / np.float32(T)
    with np.errstate(over="ignore", invalid="ignore"):
        return (row.numpy().astype(np.float32) * inv).astype(np.float16).astype(np.float64)


def log_softmax(s: np.ndarray) -> np.ndarray:
    """float64 log-softmax with the kernel's rules for non-finite rows."""
    m = s.max() if not np.isnan(s).any() else np.nan
    if np.isnan(m) or m == np.inf or m == -np.inf:
        return np.full_like(s, np.nan)
    with np.errstate(divide="ignore"):
        return (s - m) - np.log(np.exp(s - m).sum())


def rank_key(row: torch.Tensor) -> torch.Tensor:
    """int32 keys whose descending order is the ranking: NaN highest, -0 as +0, -inf lowest."""
    bits = row.view(torch.int16).to(torch.int32) & 0xFFFF
    key = torch.where(bits >= 0x8000, (~bits) & 0xFFFF, bits | 0x8000)
    key = torch.where(bits == 0x8000, torch.full_like(key, 0x8000), key)
    return torch.where((bits & 0x7FFF) > 0x7C00, torch.full_like(key, 0xFFFF), key)


def top_ids(row: torch.Tensor, n: int) -> torch.Tensor:
    """The n best ids of an fp16 row (stable descending sort of the keys: equal keys by ascending index)."""
    return torch.sort(rank_key(row), descending=True, stable=True).indices[:n]


def row_logprobs(row: torch.Tensor, token: int, T: float, greedy: bool, n: int) -> Tuple[float, List[int], List[float]]:
    """(token logprob, top ids, top logprobs) of one fp16 row."""
    lp = log_softmax(scaled(row, T, greedy))
    V = row.shape[0]
    ids = top_ids(row, min(n, V)).tolist()
    tok = float(lp[token]) if 0 <= token < V else float("nan")
    return tok, ids, [float(lp[i]) for i in ids]


def step_logprobs(logits: torch.Tensor, S: int, tokens: torch.Tensor, state: torch.Tensor, accept_idx: torch.Tensor,
                  T: Sequence[float], greedy: Sequence[bool], n_top: Sequence[Optional[int]]) -> dict:
    """Every value one step writes: {(b, pos): (token logprob, ids, logprobs)} for the sequences that are not frozen and
    have logprobs on (n_top[b] not None).  logits (>= B*S, V) fp16 as the walk read them; tokens (B, M) after the walk."""
    out = {}
    B, M = tokens.shape
    for b in range(B):
        if int(state[b, ST_FROZEN]) or n_top[b] is None:
            continue
        P = int(state[b, ST_P_OLD])
        for j in range(committed(state[b], M)):
            if P + j >= M:
                break
            k = path_node(state[b], accept_idx[b], j)
            out[(b, P + j)] = row_logprobs(logits[b * S + k], int(tokens[b, P + j]), T[b], greedy[b],
                                           min(n_top[b], MAX_LOGPROBS))
    return out
