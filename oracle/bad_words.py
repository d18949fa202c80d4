"""CPU statement of the per-sequence bad words and min_tokens (sq_ban_tokens_rows_batch): row by row from the growmap's
ancestor-or-self matrix.

Row b*S + k is node k of sequence b.  Its context is the committed tokens[b, :P] at positions 0 .. P-1, then the tokens at
slots P-1+j of node k's ancestors-or-self j >= 1, at positions P .. P+d-1 in slot order (d = depth[k]); the row's token
lands at position P + d.  The generated context is the part at positions >= L (the prompt length).
  Bad words (vLLM v1): a word w of n ids bans w[n-1] when the generated context has at least n - 1 tokens and its last
  n - 1 equal w[:n-1] (a one-token word bans its id in every row; a prefix never reaches into the prompt).
  min_tokens: with min_end = L + min_tokens (0 = off), every end id in [0, V) is banned while P + d < min_end.
A banned entry becomes -inf whatever it held (NaN and +inf included); nothing else changes.  Frozen sequences and neutral
ones (no words, min_end 0) are left as they are."""
from typing import Optional, Sequence

import torch

from oracle.penalty import row_context


def banned_ids(generated: Sequence[int], words: Sequence[Sequence[int]], position: int, min_end: int,
               end_ids: Sequence[int], V: int) -> set:
    """The ids banned in a row whose generated context is `generated` (oldest first) and whose token lands at
    absolute `position`."""
    gen = [int(t) if 0 <= int(t) < V else None for t in generated]      # (an id outside [0, V) matches no word)
    out = set()
    for w in words:
        n = len(w)
        if n - 1 <= len(gen) and [int(t) for t in w[:n - 1]] == gen[len(gen) - (n - 1):]:
            out.add(int(w[n - 1]))
    if position < min_end:
        out.update(int(t) for t in end_ids)
    return {t for t in out if 0 <= t < V}


def process_rows(logits: torch.Tensor, tokens: torch.Tensor, P: Sequence[int], prompt_len: Sequence[int],
                 mask01: torch.Tensor, depth: torch.Tensor, words: Sequence, min_end: Sequence[int],
                 end_ids: Sequence[Sequence[int]], frozen: Optional[Sequence[bool]] = None) -> torch.Tensor:
    """The (>= B*S, V) fp16 logits after every sequence's bans (a new tensor; rows from B*S on are copied).  tokens: (B, M)
    int64; P, prompt_len, min_end: per sequence; mask01: (S, S) ancestor-or-self; depth: (S,); words: per sequence, None or
    a sequence of words (sequences of ids); end_ids: per sequence, a sequence of ids."""
    B, S, V = tokens.shape[0], mask01.shape[0], logits.shape[1]
    out = logits.clone()
    for b in range(B):
        if (frozen is not None and frozen[b]) or (not words[b] and int(min_end[b]) <= 0):
            continue
        Pb, L = int(P[b]), int(prompt_len[b])
        for k in range(S):
            _, ids = row_context(tokens[b], Pb, mask01, k)     # positions 0 .. P+d-1 in order
            ban = banned_ids(ids[L:].tolist(), words[b] or (), Pb + int(depth[k]), int(min_end[b]), end_ids[b], V)
            if ban:
                out[b * S + k, sorted(ban)] = float("-inf")
    return out
