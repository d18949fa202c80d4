"""CPU statement of the prompt logprobs (sq_prompt_logprobs_ragged, BatchTree(prompt_logprobs=...)), in float64.

A prompt of P tokens has P - 1 scored positions.  Position i (1 <= i < P) reads the target's logits after prompt tokens
0 .. i-1, the row of its first verify's forward at prompt row i - 1, and scores prompt token i.  The rule is the logprobs
rule (oracle/logprobs.py) at T = 1 on the raw fp16 row: the log-softmax of the row's values, NaN throughout for a row with
+inf, NaN or only -inf, NaN for a token outside [0, V), and the n = min(n_top, 20, V) best ids by (raw value descending,
-0 equal to +0, NaN above +inf, equal values by ascending index) with their logprobs.  No temperature, filter, penalty,
bias, ban or guide applies.  Position 0 has no value."""
from typing import Dict, List, Sequence, Tuple

import torch

from oracle.logprobs import MAX_LOGPROBS, row_logprobs


def prompt_logprobs(logits: torch.Tensor, prompt: torch.Tensor, n_top: int) -> List[Tuple[float, List[int], List[float]]]:
    """logits: (>= P-1, V) fp16, row r the prediction after prompt tokens 0 .. r.  -> one (token logprob, top ids, top
    logprobs) per position 1 .. P-1."""
    n = min(n_top, MAX_LOGPROBS)
    return [row_logprobs(logits[r], int(prompt[r + 1]), 1.0, True, n) for r in range(len(prompt) - 1)]


def ragged_logprobs(logits: torch.Tensor, parts: Sequence[Tuple[int, int, int, int]],
                    tokens: torch.Tensor) -> Dict[Tuple[int, int], Tuple[float, List[int], List[float]]]:
    """Every value one sq_prompt_logprobs_ragged call writes: {(seq, pos): (token logprob, ids, logprobs)} for parts
    (seq, logits_row0, n_rows, n_top): row r scores tokens[seq, r + 1] on logits row logits_row0 + r."""
    out = {}
    for seq, row0, n_rows, n_top in parts:
        vals = prompt_logprobs(logits[row0:row0 + n_rows], tokens[seq, :n_rows + 1], n_top)
        for r, v in enumerate(vals):
            out[(seq, r + 1)] = v
    return out
