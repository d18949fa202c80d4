"""CPU statement of guided decoding (sq_guide_*): the GuideState rules applied directly, never through the packed blob.

A state is anything with `edges` ({id: next}), `default` (None or a next state) and `banned` (ids), as
sequoia_b200.guide.GuideState holds them.  In a vocabulary of V ids:
  allowed(state, V)  = the keys of edges, plus every id in [0, V) outside banned when default is not None;
  step(state, t, V)  = edges[t] for a key, default for any other allowed id, None for an id that is not allowed.
A guide consumes the generated tokens in order from its start state; the first id it does not allow kills it (-1).
Row b*S + k of the target logits (node k of sequence b) is masked with the state of node k: the committed state walked
through the tokens of node k's path (slots P-1+j of its ancestors-or-self j >= 1, in slot order).  Every id that state
does not allow becomes -inf, NaN and +inf included, and a dead node's whole row does; allowed entries are unchanged."""
from typing import Optional, Sequence

import torch


def allowed_mask(state, V: int) -> torch.Tensor:
    """(V,) bool: the ids state allows."""
    keep = torch.full((V,), state.default is not None, dtype=torch.bool)
    ban = [int(t) for t in state.banned if 0 <= int(t) < V]
    if state.default is not None and ban:
        keep[torch.tensor(ban, dtype=torch.long)] = False
    ids = [int(t) for t in state.edges if 0 <= int(t) < V]
    if ids:
        keep[torch.tensor(ids, dtype=torch.long)] = True
    return keep


def allowed(state, V: int) -> set:
    """The ids state allows in [0, V)."""
    return set(torch.nonzero(allowed_mask(state, V)).flatten().tolist())


def step(state, t: int, V: int) -> Optional[int]:
    """The next state after id t, None when state does not allow it."""
    t = int(t)
    if not 0 <= t < V:
        return None
    if t in state.edges:
        return int(state.edges[t])
    if state.default is not None and t not in state.banned:
        return int(state.default)
    return None


def state_after(guide, ids: Sequence[int], V: int, start: Optional[int] = None) -> int:
    """The state after the ids from `start` (the guide's start by default), -1 once an id is not allowed."""
    s = guide.start if start is None else start
    for t in ids:
        if s < 0:
            return -1
        nx = step(guide.states[s], t, V)
        s = -1 if nx is None else nx
    return s


def accepted_prefix(guide, ids: Sequence[int], V: int) -> int:
    """The length of the longest prefix of ids the guide accepts."""
    s = guide.start
    for i, t in enumerate(ids):
        nx = step(guide.states[s], t, V)
        if nx is None:
            return i
        s = nx
    return len(ids)


def node_states(guide, root: int, tokens_b: torch.Tensor, P: int, mask01: torch.Tensor, V: int) -> list:
    """The state of every node: root walked through the tokens of the node's path."""
    S = mask01.shape[0]
    out = []
    for k in range(S):
        path = [int(tokens_b[P - 1 + j]) for j in range(1, S) if bool(mask01[k, j])]
        out.append(state_after(guide, path, V, start=root))
    return out


def process_rows(logits: torch.Tensor, tokens: torch.Tensor, P: Sequence[int], mask01: torch.Tensor,
                 guides: Sequence, roots: Sequence[int], frozen: Optional[Sequence[bool]] = None) -> torch.Tensor:
    """The (>= B*S, V) fp16 logits after every guided sequence's mask (a new tensor; rows from B*S on are copied).
    tokens: (B, M) int64; P, roots (committed states): per sequence; mask01: (S, S) ancestor-or-self; guides: per
    sequence, None or a guide (states, start)."""
    B, S, V = tokens.shape[0], mask01.shape[0], logits.shape[1]
    out = logits.clone()
    for b in range(B):
        if guides[b] is None or (frozen is not None and frozen[b]):
            continue
        keeps = {-1: torch.zeros(V, dtype=torch.bool)}
        for k, s in enumerate(node_states(guides[b], int(roots[b]), tokens[b], int(P[b]), mask01, V)):
            if s not in keeps:
                keeps[s] = allowed_mask(guides[b].states[s], V)
            out[b * S + k, ~keeps[s]] = float("-inf")
    return out
