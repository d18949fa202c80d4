"""CPU statement of constrained drafting (sq_draft_rows_batch, SQ_ACCEPT_SKIP_DEAD).

Draft rows: in a tree with constrain_draft, the draft row of node k of sequence b (row row_base[k] + b * row_step[k])
is the distribution of the token after node k, the same context as target row b*S + k, so it gets exactly the processing
that target row gets: the allowed set and logit bias (oracle/logit_bias.py), then the bad words and min_tokens of node
k's context (oracle/bad_words.py), then the guide mask of node k's state (oracle/guide.py).  process_draft_rows applies
those three functions through the row tables.

Walk: a child of node k is dead when its token's entry in node k's processed draft row is -inf (0xFC00; the raw fp16
value, before any temperature).  The stochastic walk never accepts a dead child and leaves p (the running residual) and
q (the running draft row) as they were; a rejected live child's draft entry becomes -inf, as the kernel writes it.
A without-replacement draw from q returns a dead child only once q's live entries are used up, or when the key of a
zero-probability entry is NaN (log(1) / 0); in both cases p is already the distribution to continue from, so the first
committed token still follows p."""
from typing import Optional, Sequence

import torch

from oracle import bad_words as BW
from oracle import guide as G
from oracle import logit_bias as LB


def process_draft_rows(draft_logits: torch.Tensor, row_base: Sequence[int], row_step: Sequence[int], nodes: Sequence[int],
                       S: int, *, allowed=None, bias=None, tokens=None, P=None, prompt_len=None, mask01=None,
                       depth=None, words=None, min_end=None, end_ids=None, guides=None, roots=None,
                       frozen: Optional[Sequence[bool]] = None) -> torch.Tensor:
    """The draft logits after every sequence's processing of the rows of `nodes` (a new tensor; every other row is
    copied).  Each kind is applied when its arguments are given, with the target-row oracles' arguments: allowed / bias
    (logit_bias.process_rows); tokens, P, prompt_len, mask01, depth, words, min_end, end_ids (bad_words.process_rows);
    tokens, P, mask01, guides, roots (guide.process_rows)."""
    B = len(frozen) if frozen is not None else (len(allowed) if allowed is not None else
                                                  (tokens.shape[0] if tokens is not None else len(guides)))
    rows = [[int(row_base[k]) + b * int(row_step[k]) for k in range(S)] for b in range(B)]
    # the draft rows in the target rows' layout (row b*S + k = node k of sequence b)
    tgt = torch.stack([draft_logits[rows[b][k]] for b in range(B) for k in range(S)])
    if allowed is not None:
        tgt = LB.process_rows(tgt, S, allowed, bias, frozen=frozen)
    if words is not None:
        tgt = BW.process_rows(tgt, tokens, P, prompt_len, mask01, depth, words, min_end, end_ids, frozen=frozen)
    if guides is not None:
        tgt = G.process_rows(tgt, tokens, P, mask01, guides, roots, frozen=frozen)
    out = draft_logits.clone()
    for b in range(B):
        for k in nodes:
            out[rows[b][k]] = tgt[b * S + k]
    return out


def sample_children(draft_row: torch.Tensor, rand: torch.Tensor, k: int, T: float) -> torch.Tensor:
    """The k children a without-replacement draw takes from softmax(draft_row / T) with uniforms rand (..., V): the top k
    of log(rand) / q, a NaN key (log(1) / 0) first, as torch.topk orders it (Tree/SpecTree.py's sampler)."""
    q = torch.softmax(draft_row.to(rand.dtype) / T, dim=-1)
    return (rand.log() / q).topk(k, dim=-1).indices


def walk_first_token(target_row: torch.Tensor, draft_row: torch.Tensor, children: torch.Tensor, r: torch.Tensor,
                     noise: torch.Tensor, T: float, skip_dead: bool = True):
    """One parent node's stochastic accept step for N independent trials, in the dtype of r: p = softmax(target_row / T),
    children (N, K) token ids in order, r (N, K) uniforms, noise (N, V) Exp(1) draws for the bonus.  Child c with token t
    is accepted when p[t] > r * q[t], q = softmax(the working draft row / T); else p = relu(p - q) / sum and the working
    row's entry t becomes -inf.  With skip_dead a child whose entry in draft_row is -inf is skipped with p and q left as
    they were.  -> (first committed token (N,), accepted (N,) bool): the accepted child's token, else
    argmax(residual / noise)."""
    dt = r.dtype
    N, K = children.shape
    p = torch.softmax(target_row.to(dt) / T, dim=-1).expand(N, -1).clone()
    work = draft_row.to(dt).expand(N, -1).clone()
    raw_dead = torch.isneginf(draft_row.to(dt))
    first = torch.full((N,), -1, dtype=torch.long)
    done = torch.zeros(N, dtype=torch.bool)
    ar = torch.arange(N)
    for i in range(K):
        t = children[:, i]
        live = ~done
        if skip_dead:
            live &= ~raw_dead[t]
        q = torch.softmax(work / T, dim=-1)
        acc = live & (p[ar, t] > r[:, i] * q[ar, t])
        first[acc] = t[acc]
        done |= acc
        rej = live & ~acc
        res = (p - q).clamp_min(0)
        res = res / res.sum(-1, keepdim=True)
        p[rej] = res[rej]
        work[ar[rej], t[rej]] = float("-inf")
    bonus = torch.argmax(p / noise, dim=-1)
    return torch.where(done, first, bonus), done
