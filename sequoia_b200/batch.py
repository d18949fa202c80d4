"""Several prompts per decode step: B sequences that share the engines and the growmap (DESIGN.md §3a).

A steady step is the same two graph replays and one host sync as a single-sequence tree (sequoia_b200.tree), for all B
sequences together: every per-sequence kernel is one launch for the batch, the row-wise kernels and the GEMMs see B*n
rows.  Sequence b's device data: row b of state (B, 16), tokens / position_ids / storage_ids / r (B, M), rand (B, S, V),
noise (B, V), accept_idx (B, S), its temperature, top_p and log_min_p (B,) and top_k (B,) int32; rows b*S .. b*S+S-1 of
the target logits (B*S, V); the draft logits of node k at row_base[k] + b*row_step[k] (each tree level of all sequences
is one block, written by one lm_head GEMM).

A sequence that is terminal, or has no room for another tree in max_length, is frozen: its state word SQ_ST_FROZEN is
set and every batched kernel leaves its tokens, state and KV rows alone.  A frozen slot can take a new prompt with
admit(); the other sequences keep decoding.

Each sequence has its own policy, "spec" or "greedy".  While all are equal the tree launches the single-policy kernels;
once both are present (mixed mode, which then stays on) the sampler and the two walks are the *_mixed forms, which read
the (B,) int32 device array greedy_dev, and every sequence decodes as it would in a tree of its own policy.

A sampled sequence draws from softmax(top_p(top_k(min_p(logits))) / T): the accept walk filters the target rows first
to the tokens whose probability at T is at least min_p times the row's largest (0 = off, vLLM's min_p), then to the
top_k best raw logits (0 = off), then to top_p, and speculative sampling stays exact for the filtered distribution.
Each filter joins the captured graphs the first time a sampled sequence needs it (one recapture each); after that any
values run in the same graphs.

How a sequence ends: in default mode (every sequence with stop_tokens=None and max_new_tokens=None) the walks end it at
an accepted 0 or 2, the reference's rule.  Stop mode starts the first time a sequence has a stop set (any list, [] too)
or a token budget, and then stays on: the walks run without the fixed rule and then cut each sequence's committed tokens
at the first of its stop ids, or at its length limit len(prompt) + max_new_tokens, on the device (state words
SQ_ST_FINISH / SQ_ST_END).  The output is then exactly a prefix of the output without a stop rule.  finish_reason[b]
says why slot b ended: "stop", "length", "nan" or "room" (None while it decodes).

Penalties: each sequence has a repetition_penalty (1 = off), frequency_penalty and presence_penalty (0 = off), vLLM's
parameters.  Target row k of a sequence is penalised for the context it was computed from, the committed tokens plus the
tokens on the tree path to node k, before the greedy walk and the filters read it (sq_penalize_rows_batch; the draft is
not penalised, speculative sampling stays exact).  While every sequence is neutral nothing is launched; the first
non-neutral setting, at construction or admission, captures the steady and post graphs once more, and the penalty
kernels then stay in them.

Logprobs: each sequence has logprobs None (off) or n in 0..20, vLLM's parameter.  After the walk, inside the captured
graphs, sq_token_logprobs_batch writes the log-probability of every token the step committed and the n best ids of its
target row with theirs, from the rows as the walk read them (penalised, filtered) at the sequence's temperature (1 for a
greedy sequence), into (B, M) / (B, M, 20) device buffers at absolute positions; token_logprobs(b) copies slot b's
generated part to the host.  With T = 1 and no filter, penalty, logit bias or allowed set the values are the model's own
log-probabilities.  While every sequence is off nothing is allocated or launched; the first sequence with logprobs on, at
construction or admission, captures the steady and post graphs once more.

Prompt logprobs: each sequence has prompt_logprobs None (off) or n in 0..20, vLLM's parameter, for scoring a text.  The
first verify of a prompt of length P already runs its rows [0, P + S - 1) through every target layer in one ragged
forward; with the setting on, one lm_head GEMM per sequence turns its final-normed prompt rows 0 .. P-2 into logits (the
target runner's own logits buffer), and one sq_prompt_logprobs_ragged launch for all of them writes the log-probability of
each prompt token 1 .. P-1 given the tokens before it, and the n best ids of its row with theirs, into (B, M) /
(B, M, 20) device buffers; prompt_logprobs(b) copies slot b's to the host.  The values are the model's raw distribution:
the fp32 log-softmax of the fp16 logits at T = 1.  No temperature, filter, penalty, logit bias, allowed set, bad word or
guide applies, because no prompt token was drawn from a processed row (token_logprobs, in contrast, reads the processed
rows).  This is eager work in the first verify, outside every captured graph: graphs, captures and replayed launches are
the same with the setting on or off, and while every sequence is off nothing is allocated or launched.

Logit bias and allowed tokens: each sequence has a logit_bias {id: bias} and an allowed_token_ids set, vLLM's parameters.
Every target row of the sequence is processed alike, first of all in the accept step (sq_logit_bias_rows_batch): ids
outside the allowed set become -inf, then each bias is added to its finite logit; the penalties, the greedy walk and the
filters then read the processed rows (the draft is not processed, speculative sampling stays exact).  A stop id outside
the allowed set can never be generated, so it never ends the sequence.  While every sequence is neutral (no bias entries,
no allowed set) nothing is allocated or launched; the first non-neutral setting, at construction or admission, captures
the steady and post graphs once more, and the kernel then stays in them.

Bad words and min_tokens: each sequence has bad_words (token sequences its output must never contain) and min_tokens
(the tokens it must generate before it may end), vLLM's parameters.  Right after the logit bias, sq_ban_tokens_rows_batch
sets a few ids of each target row to -inf, for the context the row was computed from (the committed tokens plus the
tree path to its node): the last id of every word whose other ids end the row's generated context, and, while the row's
token would land before len(prompt) + min_tokens, the sequence's end ids (its stop ids in stop mode, 0 and 2 in default
mode).  The draft is not processed; speculative sampling stays exact, so no walk draws a banned id from the row that
bans it (on a branching tree the stochastic walk's bonus_first quirk can still commit the bonus token at an accepted
node's position, whose row did not draw it; DESIGN.md §3a).  A row can still lose every finite entry on some path
(settings that do so in every row are refused): a sampled sequence then ends by the walk's NaN flag (finish_reason
"nan"), a greedy one commits id 0, the argmax of an all -inf row.  While every sequence is neutral (no words,
min_tokens 0) nothing is allocated or launched; the first non-neutral setting, at construction or admission, captures
the steady and post graphs once more, and the kernel then stays in them.

Guided decoding (structured output): each sequence has a guide, a TokenGuide (sequoia_b200.guide) or None.  The guide's
state after the committed tokens lives in state word SQ_ST_GUIDE_STATE and advances on the device after each walk
(sq_guide_advance_batch).  In the accept step, after the ban, sq_guide_states_batch walks it down every tree path and
sq_guide_mask_rows_batch sets every id that a row's state does not allow to -inf, so the greedy walk and the filters
read the constrained rows.  A guided "spec" sequence gathers its accepted tokens before the walk writes the bonus token,
so each committed token is the one its row drew, on a branching tree too.  A sequence that still commits an id its
guide does not allow (a greedy one commits id 0 from a row with no finite entry) ends there with finish_reason "guide".
While no sequence has a guide nothing is allocated or launched; the first guide, at construction or admission,
allocates the (B,) table of blob addresses and captures the steady and post graphs once more.  Later admissions, with
guides of any size, rewrite one table entry.

Constrained drafting: with constrain_draft=True (tree-wide, default False) every draft row a sampler reads gets what its
target row gets above, up to and including the guide mask: the allowed set and logit bias, the bad words and min_tokens
of the node's context, and the guide mask of the node's state (sq_draft_rows_batch, in the draft graph: the root rows
first, then each level whose nodes have children, one launch each).  The draft then proposes only tokens the target rows
keep.  A child whose token is -inf in its parent's processed draft row is dead (a row with fewer finite entries than
children, an all -inf row, or a NaN sampling key); the stochastic walks never accept one and leave the residual as it was
(SQ_ACCEPT_SKIP_DEAD), so speculative sampling stays exact.  A seeded sequence commits a different, equally distributed
output than without it; greedy sequences commit the same.  While every slot is neutral nothing is launched; when a
constraint kind starts, the draft graph is captured once more along with the steady and post graphs.

Prefix reuse: admit(..., reuse_prefix=True) looks for the longest prefix of the new prompt (at most P - 1 tokens) that a
slot's ready prefix holds, the first target_kv_len[d] tokens of slot d, whose K/V both caches hold and no later step
rewrites.  Rows [0, L) are copied from the donor into the slot's rows of both caches (sq_kv_copy_prefix, one launch per
cache; none when the donor is the slot itself), and the draft prefill and first verify run rows [L, ...) only.  This is
eager admission work: the captured graphs are the same with or without it.  The copied rows are the donor's bytes, which
a forward of another shape computed, so the result matches a full prefill up to fp16 rounding, not bit for bit.
"""
from __future__ import annotations

import math
import numbers
import struct
from typing import Dict, List, Mapping, Optional, Sequence, Union

import torch

from . import _lib, ops
from .guide import TokenGuide
from .tree import _Static, check_vocab

F16 = torch.float16
ST_P, ST_M, ST_FROZEN = 0, 8, 9
ST_FINISH, ST_END = _lib.SQ_ST_FINISH, _lib.SQ_ST_END
ST_GUIDED, ST_GUIDE_STATE, ST_GUIDE_POS = _lib.SQ_ST_GUIDED, _lib.SQ_ST_GUIDE_STATE, _lib.SQ_ST_GUIDE_POS
MAX_STOP = _lib.SQ_MAX_STOP
PENALTY_MAX_LEN = _lib.SQ_PENALTY_MAX_LEN
MAX_LOGPROBS = _lib.SQ_MAX_LOGPROBS
MAX_LOGIT_BIAS = _lib.SQ_MAX_LOGIT_BIAS
LOGIT_BIAS_MAX = 100.0
MAX_BAD_WORDS, MAX_BAD_WORD_LEN = _lib.SQ_MAX_BAD_WORDS, _lib.SQ_MAX_BAD_WORD_LEN
DEFAULT_END_IDS = (0, 2)    # the ids the walks end a sequence on in default mode (the reference's fixed rule)
FP16_MAX = 65504.0
INT32_MAX = (1 << 31) - 1
POLICIES = ("spec", "greedy")
_PREVIOUS = object()        # admit(): keep the slot's previous stop set / budget / logprobs / prompt logprobs / logit
                            # bias / allowed set / bad words / min_tokens / guide


def draw_random(prompts: Sequence[torch.Tensor], M: int, S: int, V: int):
    """The CPU draws of each sequence, in prompt order, exactly as a lone SpecTree for that prompt makes them: r (M) in
    its constructor (Tree/SpecTree.py:60), then rand (S, V) after the draft prefill (:84).  -> (r (B, M), rand (B, S, V))"""
    rs, rands = [], []
    for _ in prompts:
        rs.append(torch.rand(M, dtype=F16))
        rands.append(torch.empty((S, V), dtype=F16).uniform_())
    return torch.stack(rs), torch.stack(rands)


def _h2d(t: torch.Tensor) -> torch.Tensor:
    """A copy source that does not block the host: device tensors as they are, host tensors pinned (the caching host
    allocator keeps the pinned block until the copy has run)."""
    return t if t.is_cuda else t.pin_memory()


def check_policy(policy) -> str:
    if not isinstance(policy, str) or policy not in POLICIES:
        raise ValueError(f"BatchTree policy {policy!r} is not supported (only {POLICIES}); greedys, specinfer and the "
                         "*TreeTest policies run one sequence at a time")
    return policy


def _policies(policy, B: int) -> List[str]:
    """One policy string for all B sequences, or a sequence of B strings."""
    if isinstance(policy, str) or not isinstance(policy, Sequence):
        return [check_policy(policy)] * B
    pols = [check_policy(p) for p in policy]
    if len(pols) != B:
        raise ValueError(f"policy: {len(pols)} values for {B} sequences")
    return pols


def check_sampling(temperature: float, top_p: float):
    """Refuse a temperature that is not a finite T > 0 and a top_p outside (0, 1]."""
    if not (math.isfinite(temperature) and temperature > 0):
        raise ValueError(f"temperature must be finite and > 0, got {temperature}")
    if not (math.isfinite(top_p) and 0 < top_p <= 1):
        raise ValueError(f"top_p must be in (0, 1], got {top_p}")


def check_top_k(top_k) -> int:
    """A top_k: an integer >= 0 (0 = off; a value >= the vocabulary size filters nothing)."""
    if isinstance(top_k, bool) or not isinstance(top_k, numbers.Integral) or top_k < 0:
        raise ValueError(f"top_k must be an integer >= 0 (0 = off), got {top_k!r}")
    return int(top_k)


def _top_ks(top_k, B: int) -> List[int]:
    """One top_k for all B sequences, or a sequence of B of them."""
    if isinstance(top_k, Sequence) and not isinstance(top_k, str):
        ks = [check_top_k(k) for k in top_k]
        if len(ks) != B:
            raise ValueError(f"top_k: {len(ks)} values for {B} sequences")
        return ks
    return [check_top_k(top_k)] * B


def check_min_p(min_p) -> float:
    """A min_p: a finite real number in [0, 1] (not a bool); 0 is off, 1 keeps only the tokens tied with the row's max."""
    if isinstance(min_p, bool) or not isinstance(min_p, numbers.Real) or not 0 <= min_p <= 1:
        raise ValueError(f"min_p must be a number in [0, 1] (0 = off), got {min_p!r}")
    return float(min_p)


def _min_ps(min_p, B: int) -> List[float]:
    """One min_p for all B sequences, or a sequence of B of them."""
    if _is_collection(min_p):
        vals = [check_min_p(v) for v in min_p]
        if len(vals) != B:
            raise ValueError(f"min_p: {len(vals)} values for {B} sequences")
        return vals
    return [check_min_p(min_p)] * B


def _log_min_p(policy: str, min_p: float) -> float:
    """A slot's device value: fp32(ln min_p) (ln in double precision), or -inf when the filter is off for it (min_p 0, or
    a greedy sequence)."""
    return float("-inf") if policy == "greedy" or min_p == 0.0 else _fp32(math.log(min_p))


def check_stop_tokens(stop_tokens, V: Optional[int] = None) -> Optional[tuple]:
    """A stop set: None (no stop ids), or a collection of at most MAX_STOP distinct integer ids in [0, V) (the upper bound
    is checked once V is given).  -> None or the sorted distinct ids."""
    if stop_tokens is None:
        return None
    if isinstance(stop_tokens, (str, bytes)) or not isinstance(stop_tokens, (Sequence, set, frozenset)):
        raise ValueError(f"stop_tokens must be None or a collection of token ids, got {stop_tokens!r}")
    ids = set()
    for t in stop_tokens:
        if isinstance(t, bool) or not isinstance(t, numbers.Integral) or t < 0 or (V is not None and t >= V):
            raise ValueError(f"stop_tokens: {t!r} is not a token id in [0, {V if V is not None else 'V'})")
        ids.add(int(t))
    if len(ids) > MAX_STOP:
        raise ValueError(f"stop_tokens: {len(ids)} distinct ids, at most {MAX_STOP}")
    return tuple(sorted(ids))


def _is_collection(x) -> bool:
    return isinstance(x, (Sequence, set, frozenset)) and not isinstance(x, (str, bytes))


def _stop_sets(stop_tokens, B: int) -> List[Optional[tuple]]:
    """One stop set (None or a collection of ids) for all B sequences, or a sequence of B of them (a non-empty sequence
    whose entries are all None or collections)."""
    if isinstance(stop_tokens, Sequence) and _is_collection(stop_tokens) and len(stop_tokens) > 0 \
            and all(t is None or _is_collection(t) for t in stop_tokens):
        sets = [check_stop_tokens(t) for t in stop_tokens]
        if len(sets) != B:
            raise ValueError(f"stop_tokens: {len(sets)} sets for {B} sequences")
        return sets
    return [check_stop_tokens(stop_tokens)] * B


def check_max_new_tokens(max_new_tokens) -> Optional[int]:
    """A token budget: None (no limit) or an integer >= 1."""
    if max_new_tokens is None:
        return None
    if isinstance(max_new_tokens, bool) or not isinstance(max_new_tokens, numbers.Integral) or max_new_tokens < 1:
        raise ValueError(f"max_new_tokens must be None or an integer >= 1, got {max_new_tokens!r}")
    return int(max_new_tokens)


def _budgets(max_new_tokens, B: int) -> List[Optional[int]]:
    """One budget for all B sequences, or a sequence of B of them."""
    if _is_collection(max_new_tokens):
        ns = [check_max_new_tokens(n) for n in max_new_tokens]
        if len(ns) != B:
            raise ValueError(f"max_new_tokens: {len(ns)} values for {B} sequences")
        return ns
    return [check_max_new_tokens(max_new_tokens)] * B


def _stop_row(ids: Optional[tuple]) -> List[int]:
    """A stop set as its device row: the ids padded with -1 to MAX_STOP."""
    ids = ids or ()
    return list(ids) + [-1] * (MAX_STOP - len(ids))


def _end_limit(prompt_len: int, budget: Optional[int]) -> int:
    """The absolute length limit len(prompt) + max_new_tokens the device holds (0 = none; clamped to int32)."""
    return 0 if budget is None else min(prompt_len + budget, INT32_MAX)


def _per_seq(value, B: int, name: str) -> List[float]:
    """One value (a Python, numpy or 0-d tensor scalar) for all B sequences, or a sequence of B values."""
    if isinstance(value, numbers.Real) or (isinstance(value, torch.Tensor) and value.dim() == 0):
        return [float(value)] * B
    vals = [float(v) for v in value]
    if len(vals) != B:
        raise ValueError(f"{name}: {len(vals)} values for {B} sequences")
    return vals


def _fp32(x: float) -> float:
    return struct.unpack("f", struct.pack("f", x))[0]


def check_penalty(name: str, value) -> float:
    """A repetition_penalty in (0, 65504], or a frequency_penalty / presence_penalty with |value| <= 65504: a finite real
    number (not a bool).  -> the value rounded to fp32, as the device holds it (a repetition penalty that rounds to 0 is
    refused).  The bounds keep f * count finite, so a penalised finite logit stays finite."""
    if isinstance(value, bool) or not isinstance(value, numbers.Real) or not math.isfinite(value):
        raise ValueError(f"{name} must be a finite number, got {value!r}")
    v = _fp32(float(value)) if abs(float(value)) <= FP16_MAX else float(value)
    if name == "repetition_penalty":
        if not 0 < v <= FP16_MAX:
            raise ValueError(f"repetition_penalty must be in (0, 65504], got {value!r}")
    elif not abs(v) <= FP16_MAX:
        raise ValueError(f"{name} must be in [-65504, 65504], got {value!r}")
    return v


def _penalties(name: str, value, B: int) -> List[float]:
    """One penalty for all B sequences, or a sequence of B of them."""
    if _is_collection(value):
        vals = [check_penalty(name, v) for v in value]
        if len(vals) != B:
            raise ValueError(f"{name}: {len(vals)} values for {B} sequences")
        return vals
    return [check_penalty(name, value)] * B


def is_neutral(rep: float, freq: float, pres: float) -> bool:
    """The penalties that leave a row as it is: repetition 1, frequency 0, presence 0."""
    return rep == 1.0 and freq == 0.0 and pres == 0.0


def check_logprobs(logprobs) -> Optional[int]:
    """A logprobs setting: None (off) or an integer in 0..20, the number of top alternatives per generated token."""
    if logprobs is None:
        return None
    if isinstance(logprobs, bool) or not isinstance(logprobs, numbers.Integral) or not 0 <= logprobs <= MAX_LOGPROBS:
        raise ValueError(f"logprobs must be None or an integer in 0..{MAX_LOGPROBS}, got {logprobs!r}")
    return int(logprobs)


def _logprobs(logprobs, B: int) -> List[Optional[int]]:
    """One logprobs setting for all B sequences, or a sequence of B of them."""
    if _is_collection(logprobs):
        vals = [check_logprobs(n) for n in logprobs]
        if len(vals) != B:
            raise ValueError(f"logprobs: {len(vals)} values for {B} sequences")
        return vals
    return [check_logprobs(logprobs)] * B


def check_prompt_logprobs(prompt_logprobs) -> Optional[int]:
    """A prompt_logprobs setting: None (off) or an integer in 0..20, the number of top alternatives per prompt token."""
    if prompt_logprobs is None:
        return None
    if isinstance(prompt_logprobs, bool) or not isinstance(prompt_logprobs, numbers.Integral) \
            or not 0 <= prompt_logprobs <= MAX_LOGPROBS:
        raise ValueError(f"prompt_logprobs must be None or an integer in 0..{MAX_LOGPROBS}, got {prompt_logprobs!r}")
    return int(prompt_logprobs)


def _prompt_logprobs(prompt_logprobs, B: int) -> List[Optional[int]]:
    """One prompt_logprobs setting for all B sequences, or a sequence of B of them."""
    if _is_collection(prompt_logprobs):
        vals = [check_prompt_logprobs(n) for n in prompt_logprobs]
        if len(vals) != B:
            raise ValueError(f"prompt_logprobs: {len(vals)} values for {B} sequences")
        return vals
    return [check_prompt_logprobs(prompt_logprobs)] * B


def check_logit_bias(logit_bias, V: Optional[int] = None) -> Optional[tuple]:
    """A logit bias: None, or a mapping {id: bias} of at most MAX_LOGIT_BIAS entries, each id an integer in [0, V) (the
    upper bound is checked once V is given) and each bias a finite real number in [-100, 100] (not a bool).  -> None, or
    the sorted tuple of (id, bias rounded to fp32, as the device holds it) without the entries whose bias is 0 (so {} and
    {5: 0.0} are both neutral: ())."""
    if logit_bias is None:
        return None
    if not isinstance(logit_bias, Mapping):
        raise ValueError(f"logit_bias must be None or a mapping {{token id: bias}}, got {logit_bias!r}")
    out = []
    for t, v in logit_bias.items():
        if isinstance(t, bool) or not isinstance(t, numbers.Integral) or t < 0 or (V is not None and t >= V):
            raise ValueError(f"logit_bias: {t!r} is not a token id in [0, {V if V is not None else 'V'})")
        if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v) \
                or not abs(float(v)) <= LOGIT_BIAS_MAX:
            raise ValueError(f"logit_bias: the bias of {int(t)} must be a finite number in [-100, 100], got {v!r}")
        v = _fp32(float(v))
        if v != 0.0:
            out.append((int(t), v))
    if len(out) > MAX_LOGIT_BIAS:
        raise ValueError(f"logit_bias: {len(out)} entries, at most {MAX_LOGIT_BIAS}")
    return tuple(sorted(out))


def _logit_biases(logit_bias, B: int) -> List[Optional[tuple]]:
    """One logit bias (None or a mapping) for all B sequences, or a sequence of B of them."""
    if _is_collection(logit_bias) and not isinstance(logit_bias, Mapping):
        vals = [check_logit_bias(v) for v in logit_bias]
        if len(vals) != B:
            raise ValueError(f"logit_bias: {len(vals)} values for {B} sequences")
        return vals
    return [check_logit_bias(logit_bias)] * B


def check_allowed_token_ids(allowed_token_ids, V: Optional[int] = None) -> Optional[tuple]:
    """An allowed set: None (every id), or a non-empty collection of distinct integer ids in [0, V) (the upper bound is
    checked once V is given).  -> None or the sorted ids; a set that covers all of [0, V) is None."""
    if allowed_token_ids is None:
        return None
    if not _is_collection(allowed_token_ids):
        raise ValueError(f"allowed_token_ids must be None or a collection of token ids, got {allowed_token_ids!r}")
    ids = set()
    for t in allowed_token_ids:
        if isinstance(t, bool) or not isinstance(t, numbers.Integral) or t < 0 or (V is not None and t >= V):
            raise ValueError(f"allowed_token_ids: {t!r} is not a token id in [0, {V if V is not None else 'V'})")
        if int(t) in ids:
            raise ValueError(f"allowed_token_ids: {int(t)} is listed twice")
        ids.add(int(t))
    if not ids:
        raise ValueError("allowed_token_ids must not be empty (None allows every id)")
    if V is not None and len(ids) == V:
        return None
    return tuple(sorted(ids))


def _allowed_sets(allowed_token_ids, B: int) -> List[Optional[tuple]]:
    """One allowed set (None or a collection of ids) for all B sequences, or a sequence of B of them (a non-empty sequence
    whose entries are all None or collections)."""
    if isinstance(allowed_token_ids, Sequence) and _is_collection(allowed_token_ids) and len(allowed_token_ids) > 0 \
            and all(t is None or _is_collection(t) for t in allowed_token_ids):
        sets = [check_allowed_token_ids(t) for t in allowed_token_ids]
        if len(sets) != B:
            raise ValueError(f"allowed_token_ids: {len(sets)} sets for {B} sequences")
        return sets
    return [check_allowed_token_ids(allowed_token_ids)] * B


def is_neutral_bias(logit_bias: Optional[tuple], allowed_token_ids: Optional[tuple]) -> bool:
    """The checked settings that leave a row as it is: no bias entries and no allowed set."""
    return not logit_bias and allowed_token_ids is None


def check_bad_words(bad_words, V: Optional[int] = None) -> Optional[tuple]:
    """Bad words: None, or a collection of words, each a non-empty sequence of at most MAX_BAD_WORD_LEN integer ids in
    [0, V) (not bools; the upper bound is checked once V is given), at most MAX_BAD_WORDS distinct words.  -> None, or the
    distinct words as tuples in first-seen order (duplicates dropped; an empty collection is ())."""
    if bad_words is None:
        return None
    if not _is_collection(bad_words):
        raise ValueError(f"bad_words must be None or a collection of words (sequences of token ids), got {bad_words!r}")
    out = {}
    for w in bad_words:
        if not isinstance(w, Sequence) or isinstance(w, (str, bytes)) or not 1 <= len(w) <= MAX_BAD_WORD_LEN:
            raise ValueError(f"bad_words: a word is a sequence of 1..{MAX_BAD_WORD_LEN} token ids, got {w!r}")
        for t in w:
            if isinstance(t, bool) or not isinstance(t, numbers.Integral) or t < 0 or (V is not None and t >= V):
                raise ValueError(f"bad_words: {t!r} is not a token id in [0, {V if V is not None else 'V'})")
        out.setdefault(tuple(int(t) for t in w), None)
    if len(out) > MAX_BAD_WORDS:
        raise ValueError(f"bad_words: {len(out)} distinct words, at most {MAX_BAD_WORDS}")
    return tuple(out)


def _is_word_set(x) -> bool:
    """None, or a collection whose entries are all collections: one prompt's set of words in the per-prompt form."""
    return x is None or (_is_collection(x) and all(_is_collection(w) for w in x))


def _bad_words(bad_words, B: int) -> List[Optional[tuple]]:
    """One set of words for all B sequences, or one per sequence.  The per-prompt form is a non-empty sequence whose every
    entry is None or a collection of collections (three levels of nesting: [None, [[2, 3]]]); anything else is one set
    for all prompts (two levels: [[1], [2, 3]] is one set of two words).  So [[], []] gives two prompts no words each."""
    if isinstance(bad_words, Sequence) and _is_collection(bad_words) and len(bad_words) > 0 \
            and all(_is_word_set(e) for e in bad_words):
        sets = [check_bad_words(e) for e in bad_words]
        if len(sets) != B:
            raise ValueError(f"bad_words: {len(sets)} sets for {B} sequences")
        return sets
    return [check_bad_words(bad_words)] * B


def check_min_tokens(min_tokens, max_new_tokens: Optional[int] = None) -> int:
    """A min_tokens: an integer >= 0 (not a bool; 0 = off), at most the sequence's max_new_tokens when it has one (vLLM
    refuses min_tokens > max_tokens)."""
    if isinstance(min_tokens, bool) or not isinstance(min_tokens, numbers.Integral) or min_tokens < 0:
        raise ValueError(f"min_tokens must be an integer >= 0 (0 = off), got {min_tokens!r}")
    if max_new_tokens is not None and min_tokens > max_new_tokens:
        raise ValueError(f"min_tokens={int(min_tokens)} exceeds max_new_tokens={max_new_tokens}")
    return int(min_tokens)


def _min_tokens(min_tokens, B: int) -> List[int]:
    """One min_tokens for all B sequences, or a sequence of B of them."""
    if _is_collection(min_tokens):
        vals = [check_min_tokens(m) for m in min_tokens]
        if len(vals) != B:
            raise ValueError(f"min_tokens: {len(vals)} values for {B} sequences")
        return vals
    return [check_min_tokens(min_tokens)] * B


def _min_end(prompt_len: int, min_tokens: int) -> int:
    """The absolute limit len(prompt) + min_tokens the device holds (0 = off; clamped to int32)."""
    return 0 if min_tokens == 0 else min(prompt_len + min_tokens, INT32_MAX)


def end_ids(stop_tokens: Optional[tuple], stop_mode: bool) -> tuple:
    """The ids that end a sequence, which min_tokens bans: its stop ids in stop mode (none without a stop set), else
    DEFAULT_END_IDS, the reference's fixed rule."""
    return (stop_tokens or ()) if stop_mode else DEFAULT_END_IDS


def check_bannable(V: int, bad_words: Optional[tuple], allowed_token_ids: Optional[tuple], min_tokens: int,
                   ends: tuple):
    """Refuse settings that ban every id a sequence may generate in every row: its one-token words, plus its end ids
    when min_tokens > 0, cover the vocabulary or its allowed set."""
    banned = {w[0] for w in bad_words or () if len(w) == 1}
    if min_tokens > 0:
        banned.update(ends)
    candidates = range(V) if allowed_token_ids is None else allowed_token_ids
    if len(banned) >= len(candidates) and all(t in banned for t in candidates):
        raise ValueError("bad_words" + (" and min_tokens" if min_tokens > 0 else "") + " ban every token id the "
                         "sequence may generate" + (" (its allowed_token_ids)" if allowed_token_ids is not None else ""))


def is_neutral_ban(bad_words: Optional[tuple], min_tokens: int) -> bool:
    """The checked settings that ban nothing: no words and min_tokens 0."""
    return not bad_words and min_tokens == 0


def check_guide(guide) -> Optional[TokenGuide]:
    """A guide: None or a TokenGuide."""
    if guide is not None and not isinstance(guide, TokenGuide):
        raise ValueError(f"guide must be None or a TokenGuide, got {guide!r}")
    return guide


def _guides(guide, B: int) -> List[Optional[TokenGuide]]:
    """One guide (None or a TokenGuide) for all B sequences, or a sequence of B of them."""
    if isinstance(guide, Sequence) and not isinstance(guide, (str, bytes)):
        vals = [check_guide(g) for g in guide]
        if len(vals) != B:
            raise ValueError(f"guide: {len(vals)} values for {B} sequences")
        return vals
    return [check_guide(guide)] * B


def check_reuse_prefix(reuse_prefix) -> bool:
    """admit()'s reuse_prefix: a bool."""
    if not isinstance(reuse_prefix, bool):
        raise ValueError(f"reuse_prefix must be a bool, got {reuse_prefix!r}")
    return reuse_prefix


def prefix_donor(prompt: torch.Tensor, rows: torch.Tensor, ready: Sequence[int], b: int,
                 prompt_logprobs: Optional[int] = None):
    """The prefix an admission into slot b reuses (host tensors): slot d offers its first ready[d] tokens rows[d] (whose
    K/V both caches hold); L is the longest common prefix of the prompt with any of them, capped at len(prompt) - 1 (the
    last prompt row always runs: it gives node 0's draft logits and the first verify's root).  The largest L wins; on a
    tie slot b itself (no copy), then the lowest index.  A slot with prompt_logprobs on reuses nothing (its rows below L
    would get no values).  -> (donor, L), or (None, 0)."""
    P = len(prompt)
    if prompt_logprobs is not None or P < 2:
        return None, 0
    best, best_len = None, 0
    for d in [b] + [d for d in range(len(ready)) if d != b]:
        m = min(int(ready[d]), P - 1)
        if m <= best_len:
            continue
        diff = (rows[d, :m] != prompt[:m]).nonzero()
        n = m if len(diff) == 0 else int(diff[0])
        if n > best_len:
            best, best_len = d, n
    return best, best_len


def check_seed(seed) -> int:
    """A per-sequence seed: an integer in [0, 2^64)."""
    if isinstance(seed, bool) or not isinstance(seed, numbers.Integral):
        raise ValueError(f"a seed must be an integer in [0, 2^64), got {seed!r}")
    seed = int(seed)
    if not 0 <= seed < 1 << 64:
        raise ValueError(f"a seed must be an integer in [0, 2^64), got {seed}")
    return seed


def _as_int64(seed: int) -> int:
    """The int64 with the bits of the uint64 `seed` (how the device arrays hold it)."""
    return seed - (1 << 64) if seed >= 1 << 63 else seed


class BatchTree:
    """Batched SpecTree ("spec") / GreedyTree ("greedy") over `len(prompts)` sequences.  The engines must have been built
    with batch_size == len(prompts).  verify() returns one (valid_tokens, accept_length, terminal) per sequence.
    policy: one of "spec" / "greedy" for all sequences, or one per sequence.
    temperature and top_p: one value for all sequences, or one per sequence; "greedy" sequences ignore both (their
    temperature must still be a valid one).
    top_k: one integer >= 0 for all sequences, or one per sequence: a sampled sequence keeps the top_k best target logits
    of each row (raw value descending, equal values by ascending index) before top_p and its softmax; 0, and any value
    >= the vocabulary size, is off.  "greedy" sequences ignore it.
    min_p: one number in [0, 1] for all sequences, or one per sequence: a sampled sequence keeps the target tokens whose
    probability at its temperature is at least min_p times the row's largest, before top_k, top_p and the softmax
    (vLLM's min_p; 0 is off).  "greedy" sequences ignore it.
    seeds: None (r and rand drawn with torch's CPU generator as a lone SpecTree draws them, the bonus noise with torch's
    CUDA generator), or one integer in [0, 2^64) per prompt: each sequence then draws all its random numbers on the
    device from a Philox stream keyed by its seed, so its output does not depend on its slot or its neighbours ("greedy"
    takes seeds and ignores them).
    stop_tokens: None, or a collection of at most 8 distinct ids in [0, V), for all sequences; or one such value per
    prompt.  max_new_tokens: None, or an integer >= 1, for all sequences or one per prompt.  Any stop set (an empty one
    too) or budget turns on stop mode (module docstring): sequence b then ends at the first of its stop ids that it
    commits, or when it holds len(prompt) + max_new_tokens tokens, whichever comes first, and verify() returns exactly
    the tokens up to there with terminal True.  Both policies honour them.
    repetition_penalty (in (0, 65504], 1 = off), frequency_penalty and presence_penalty (|value| <= 65504, 0 = off): one
    value for all sequences or one per prompt, vLLM's meaning (module docstring, include/sequoia_b200.h).  Both policies
    honour them.  Penalties count at most 4096 tokens: a tree with max_length > 4096 refuses a non-neutral setting.
    logprobs: None (off) or an integer in 0..20, for all sequences or one per prompt: token_logprobs(b) then gives the
    log-probability of each generated token and of the n best alternatives of its row (module docstring,
    include/sequoia_b200.h).  Both policies honour it; verify() returns what it returns without it.
    prompt_logprobs: None (off) or an integer in 0..20, for all sequences or one per prompt: prompt_logprobs(b) then gives
    the log-probability of each prompt token after the first, given the tokens before it, and the n best alternatives of
    its row, under the target's raw distribution (T = 1, no processing; module docstring).  It is computed in the first
    verify, outside the captured graphs; verify() returns what it returns without it.
    logit_bias: None or a mapping {id: bias} of at most 1024 ids in [0, V) with biases in [-100, 100] (-100 bans an id in
    practice), for all sequences or one per prompt.  allowed_token_ids: None or a non-empty collection of distinct ids in
    [0, V), for all sequences or one per prompt: every other id is -inf in the sequence's target rows.  Both policies
    honour both; a greedy sequence takes the argmax of the processed row (module docstring, include/sequoia_b200.h).
    bad_words: None, or a collection of at most 128 words, each a sequence of 1..16 ids in [0, V), for all sequences
    ([[1], [2, 3]]: two words); or one such value (or None) per prompt ([None, [[2, 3]]]: three levels of nesting).  The
    output then never contains a word: its last id is banned wherever its other ids end the generated tokens (a one-token
    word everywhere; a word never matches across the prompt).  min_tokens: an integer >= 0 (at most max_new_tokens), for
    all sequences or one per prompt: the sequence's end ids are banned until it has generated that many tokens.  Both
    policies honour both (module docstring, include/sequoia_b200.h).
    guide: None or a TokenGuide (sequoia_b200.guide), for all sequences or one per prompt: every generated token is one
    the guide allows in its current state.  The guide does not end a sequence; its end ids do.  A guide is refused when
    one of its states allows no id that the sequence may generate (within its allowed_token_ids and without its
    one-token bad_words).  Both policies honour it; guide_state(b) gives the slot's state after its committed tokens.
    constrain_draft: a bool (default False), for the whole tree: the draft rows get each sequence's allowed set, logit
    bias, bad words, min_tokens and guide as its target rows do, so the draft proposes only tokens the target rows keep,
    and the walks skip the children those rows set to -inf (module docstring).  A seeded "spec" sequence then commits a
    different, equally distributed output; admit() does not change it."""

    def __init__(self, draft, target, prompts: Sequence[torch.Tensor], grow_map: dict,
                 policy: Union[str, Sequence[str]] = "spec",
                 temperature: Union[float, Sequence[float]] = 0.6, top_p: Union[float, Sequence[float]] = 1.0,
                 max_length: int = 256, max_target_seq: Optional[int] = None,
                 seeds: Optional[Sequence[int]] = None, top_k: Union[int, Sequence[int]] = 0,
                 stop_tokens=None, max_new_tokens: Union[None, int, Sequence[Optional[int]]] = None,
                 repetition_penalty: Union[float, Sequence[float]] = 1.0,
                 frequency_penalty: Union[float, Sequence[float]] = 0.0,
                 presence_penalty: Union[float, Sequence[float]] = 0.0,
                 logprobs: Union[None, int, Sequence[Optional[int]]] = None,
                 prompt_logprobs: Union[None, int, Sequence[Optional[int]]] = None, logit_bias=None, allowed_token_ids=None, min_p: Union[float, Sequence[float]] = 0.0,
                 bad_words=None, min_tokens: Union[int, Sequence[int]] = 0, guide=None, constrain_draft: bool = False):
        if not isinstance(constrain_draft, bool):
            raise ValueError(f"constrain_draft must be a bool, got {constrain_draft!r}")
        B = len(prompts)
        guides = _guides(guide, B)
        policies = _policies(policy, B)
        min_ps = _min_ps(min_p, B)
        words, min_toks = _bad_words(bad_words, B), _min_tokens(min_tokens, B)
        biases, alloweds = _logit_biases(logit_bias, B), _allowed_sets(allowed_token_ids, B)
        lps = _logprobs(logprobs, B)
        plps = _prompt_logprobs(prompt_logprobs, B)
        reps = _penalties("repetition_penalty", repetition_penalty, B)
        freqs = _penalties("frequency_penalty", frequency_penalty, B)
        press = _penalties("presence_penalty", presence_penalty, B)
        use_penalty = not all(is_neutral(*v) for v in zip(reps, freqs, press))
        if use_penalty and max_length > PENALTY_MAX_LEN:
            raise ValueError(f"penalties count at most {PENALTY_MAX_LEN} tokens; max_length={max_length}")
        top_ks = _top_ks(top_k, B)
        stops, budgets = _stop_sets(stop_tokens, B), _budgets(max_new_tokens, B)
        temps, top_ps = _per_seq(temperature, B, "temperature"), _per_seq(top_p, B, "top_p")
        for t, p in zip(temps, top_ps):
            check_sampling(t, p)
        if seeds is not None:
            seeds = list(seeds)
            if len(seeds) != B:
                raise ValueError(f"seeds: {len(seeds)} values for {B} sequences")
            seeds = [check_seed(s) for s in seeds]
        for name, eng in (("draft", draft), ("target", target)):
            if eng.engine.batch_size != B:
                raise ValueError(f"{name} engine holds {eng.engine.batch_size} sequences, got {B} prompts")
            if eng.engine.max_length != max_length:
                raise ValueError(f"{name} engine max_length {eng.engine.max_length} != {max_length}")
        dev = torch.device(draft.device)
        if dev.type != "cuda":
            raise RuntimeError("sequoia_b200 trees run on a CUDA device only (there is no CPU path)")
        self.draft, self.target = draft, target
        self.policies = policies
        # mixed: both policies present (from here on, for the tree's life); greedy: every sequence greedy, never mixed
        self.mixed = len(set(policies)) > 1
        self.greedy = not self.mixed and policies[0] == "greedy"
        self.temps, self.top_ps, self.top_ks = temps, top_ps, top_ks
        self.B, self.M = B, max_length
        self.max_target_seq = max_target_seq or max_length
        self.st = st = _Static(grow_map, dev)
        S = self.S = st.S
        V = self.V = draft.engine.model_config.vocab_size
        for pol in set(policies):
            check_vocab(pol, V)
        stops = [check_stop_tokens(t, V) for t in stops]
        biases = [check_logit_bias(None if t is None else dict(t), V) for t in biases]
        alloweds = [check_allowed_token_ids(t, V) for t in alloweds]
        words = [check_bad_words(w, V) for w in words]
        stop_mode = any(t is not None for t in stops) or any(n is not None for n in budgets)
        for b in range(B):
            check_min_tokens(min_toks[b], budgets[b])
            check_bannable(V, words[b], alloweds[b], min_toks[b], end_ids(stops[b], stop_mode))
            if guides[b] is not None:
                guides[b].check(V, alloweds[b], words[b])
        M = max_length
        for p in prompts:
            if len(p) + S - 1 > M:
                raise ValueError(f"max_length={M} must hold the prompt ({len(p)}) + tree ({S}) - 1")
        self.device = dev
        # prefix reuse: (donor slot, L) of each slot's current prompt when its admission took rows [0, L) of K/V from a
        # slot's ready prefix (admit(reuse_prefix=True)), else None; the draft prefill and first verify start at row L
        self.reused_prefix: List[Optional[tuple]] = [None] * B
        # constrained drafting: every draft row a sampler reads gets its sequence's allowed set, logit bias, bad words and
        # guide, as its target row does, inside the draft graph; the walks then skip dead children (SQ_ACCEPT_SKIP_DEAD)
        self.constrain_draft = constrain_draft
        # guides: each slot's blob address in a (B,) device table (0 = none), read by the three guide kernels inside the
        # captured graphs, which they join the first time a slot has a guide; the host keeps the blobs alive
        self.guides = guides
        self.use_guide = False
        self.guide_table_dev = self.guide_scratch = None
        self.guide_blobs: List[Optional[torch.Tensor]] = [None] * B
        # sampling parameters live on the device, so the captured graphs serve any values an admission brings; the top-p
        # filter joins the steady / post graphs only once a sequence has had top_p < 1 (one recapture, see admit)
        # (a greedy sequence's top_p is 1 on the device, so the filter leaves its rows alone)
        self.T_dev = torch.tensor(temps, dtype=torch.float32, device=dev)
        self.top_p_dev = torch.tensor([1.0 if pol == "greedy" else p for pol, p in zip(policies, top_ps)],
                                      dtype=torch.float32, device=dev)
        self.greedy_dev = torch.tensor([pol == "greedy" for pol in policies], dtype=torch.int32, device=dev)
        self.use_top_p = any(pol == "spec" and p < 1.0 for pol, p in zip(policies, top_ps))
        # the same for top_k (0 for a greedy sequence; k >= V is off and held as V, which fits int32)
        self.top_k_dev = torch.tensor([0 if pol == "greedy" else min(k, V) for pol, k in zip(policies, top_ks)],
                                      dtype=torch.int32, device=dev)
        self.use_top_k = any(pol == "spec" and 0 < k < V for pol, k in zip(policies, top_ks))
        # the same for min_p, held as fp32(ln min_p) (-inf = off, and for a greedy sequence)
        self.min_ps = min_ps
        self.log_min_p_dev = torch.tensor([_log_min_p(pol, p) for pol, p in zip(policies, min_ps)], dtype=torch.float32,
                                          device=dev)
        self.use_min_p = any(pol == "spec" and p > 0.0 for pol, p in zip(policies, min_ps))
        # stop mode: each slot's stop ids (-1 padded) and absolute length limit (0 = none) on the device, read by the stop
        # walks inside the captured graphs, which replace the walks the first time a slot has either (one recapture)
        self.stop_tokens, self.max_new_tokens = stops, budgets
        self.stop_ids_dev = torch.tensor([_stop_row(t) for t in stops], dtype=torch.int32, device=dev)
        self.end_limit_dev = torch.tensor([_end_limit(len(p), n) for p, n in zip(prompts, budgets)], dtype=torch.int32,
                                          device=dev)
        self.use_stop = stop_mode
        # penalties: each slot's values and prompt length on the device, read by sq_penalize_rows_batch inside the
        # captured graphs, which it joins the first time a slot has a non-neutral setting (one recapture)
        self.repetition_penalty, self.frequency_penalty, self.presence_penalty = reps, freqs, press
        self.rep_dev = torch.tensor(reps, dtype=torch.float32, device=dev)
        self.freq_dev = torch.tensor(freqs, dtype=torch.float32, device=dev)
        self.pres_dev = torch.tensor(press, dtype=torch.float32, device=dev)
        self.prompt_len_dev = torch.tensor([len(p) for p in prompts], dtype=torch.int32, device=dev)
        self.use_penalty = False
        self.pen_scratch: Optional[torch.Tensor] = None
        if use_penalty:
            self._start_penalties()
        # logprobs: each slot's n on the device (-1 = off), read by sq_token_logprobs_batch inside the captured graphs,
        # which it joins the first time a slot has logprobs on (one recapture); the prompt lengths bound token_logprobs
        self.logprobs = lps
        self.prompt_lens = [len(p) for p in prompts]
        self.n_top_dev = torch.tensor([-1 if n is None else n for n in lps], dtype=torch.int32, device=dev)
        self.use_logprobs = False
        self.lp_token = self.lp_ids = self.lp_top = None
        # prompt logprobs: each slot's n (None = off) and whether its current prompt has had its first verify (the
        # buffers hold its values from then until the next admission); the (B, M) / (B, M, 20) buffers are allocated for
        # the first slot that turns it on
        self.prompt_logprobs_n = plps
        self.plp_ready = [False] * B
        self.plp_token = self.plp_ids = self.plp_top = None
        # bad words and min_tokens: each slot's word table and absolute limit L + min_tokens on the device, read by
        # sq_ban_tokens_rows_batch inside the captured graphs, which it joins the first time a slot is non-neutral
        self.bad_words, self.min_tokens = words, min_toks
        self.use_ban = False
        self.words_dev = self.word_len_dev = self.n_words_dev = self.min_end_dev = self.default_end_dev = None
        if not all(is_neutral_ban(*v) for v in zip(words, min_toks)):
            self._start_ban()
        # logit bias and allowed sets: each slot's bitmask row and sorted (id, bias) entries on the device, read by
        # sq_logit_bias_rows_batch inside the captured graphs, which it joins the first time a slot is non-neutral
        self.logit_bias, self.allowed_token_ids = biases, alloweds
        self.use_logit_bias = False
        self.allowed_dev = self.has_mask_dev = self.bias_ids_dev = self.bias_vals_dev = self.n_bias_dev = None
        if not all(is_neutral_bias(*v) for v in zip(biases, alloweds)):
            self._start_logit_bias()
        self.finish_reason: List[Optional[str]] = [None] * B
        i64 = dict(dtype=torch.int64, device=dev)
        self.tokens = torch.zeros(B, M, **i64)
        self.position_ids = torch.zeros(B, M, **i64)
        self.storage_ids = torch.arange(M, **i64).repeat(B, 1)
        self.state = torch.zeros(B, 16, dtype=torch.int32, device=dev)
        self.host_state = torch.zeros(B, 16, dtype=torch.int32).pin_memory()
        self.accept_idx = torch.zeros(B, max(S, 8), dtype=torch.int32, device=dev)
        self.draft_logits = torch.zeros(B * S, V, dtype=F16, device=dev)
        self.target_logits = torch.zeros(B * S, V, dtype=F16, device=dev)
        self.row_base, self.row_step = ops.draft_row_tables([(0, 1)] + [(lv["n0"], lv["tb"]) for lv in st.levels], S, B,
                                                            dev)
        self.noise = torch.ones(B, V, dtype=F16, device=dev)
        self.target_token = torch.zeros(B * S, **i64)
        self.external_noise: Optional[torch.Tensor] = None    # tests: (n_iter, B, V) Exp(1) rows
        self.graphs: Dict[str, torch.cuda.CUDAGraph] = {}
        self.graph_launches: Dict[str, int] = {}
        self.replays: Dict[str, int] = {}
        self.captures: Dict[str, int] = {}
        self.replayed_launches = 0
        self.use_graphs = True
        self.iter = 0
        self.frozen = [False] * B
        self.last: List[tuple] = [None] * B
        self.ground_truth_len = [len(p) for p in prompts]
        self.target_kv_len = [0] * B
        # seeded: each sequence draws r, rand and its bonus noise on the device from a counter-based stream of its own
        # (sq_rng.cu); steps[b] counts sequence b's verifies since it was seeded and advances inside the graphs
        self.seeded = seeds is not None
        if self.seeded:
            self.seeds = torch.tensor([_as_int64(s) for s in seeds], **i64)
            self.steps = torch.zeros(B, **i64)
        # r and rand: for every slot once any sequence samples (CPU draws for every prompt in prompt order, greedy ones
        # included, so a sampling sequence's numbers do not depend on its neighbours' policies)
        if self.greedy:
            self.r = self.rand = None
        elif self.seeded:
            self.r = torch.empty(B, M, dtype=F16, device=dev)
            self.rand = torch.empty(B, S, V, dtype=F16, device=dev)
            ops.rng_uniform_seqs(self.r, self.seeds, range(B), ops.RNG_R)
            ops.rng_uniform_seqs(self.rand, self.seeds, range(B), ops.RNG_RAND)
        else:
            r, rand = draw_random(prompts, M, S, V)
            self.r, self.rand = r.to(dev), rand.to(dev)
        if any(n is not None for n in lps):
            self._start_logprobs()
        if any(n is not None for n in plps):
            self._start_prompt_logprobs()
        if any(g is not None for g in guides):
            self._start_guide()
        for b, p in enumerate(prompts):
            self._load_prompt(b, p)
        with torch.inference_mode():
            self.op_draft_prefill(range(B))

    # ---- helpers ---------------------------------------------------------------------------------------------------------
    def _mask_kw(self):
        return dict(tree_bits=self.st.tree_bits, tree_words=self.st.tree_words, tree_size=self.S)

    def _start_penalties(self):
        """The penalty kernels join op_accept, with their scratch: a distinct-id list per sequence, rewritten every step
        before it is read, so not one of the captured buffers."""
        self.use_penalty = True
        self.pen_scratch = torch.zeros(ops.penalty_scratch_words(self.B, self.M), dtype=torch.int32, device=self.device)

    def _start_logprobs(self):
        """The logprobs kernel joins seq_post, with its (B, M) / (B, M, 20) output buffers (a position is written by the
        step that commits it)."""
        self.use_logprobs = True
        B, M, dev = self.B, self.M, self.device
        self.lp_token = torch.full((B, M), float("nan"), dtype=torch.float32, device=dev)
        self.lp_ids = torch.full((B, M, MAX_LOGPROBS), -1, dtype=torch.int32, device=dev)
        self.lp_top = torch.full((B, M, MAX_LOGPROBS), float("nan"), dtype=torch.float32, device=dev)

    def _start_prompt_logprobs(self):
        """The (B, M) / (B, M, 20) prompt-logprobs buffers, NaN / -1 filled (written eagerly by the first verify of each
        prompt with the setting on, outside the captured graphs)."""
        B, M, dev = self.B, self.M, self.device
        self.plp_token = torch.full((B, M), float("nan"), dtype=torch.float32, device=dev)
        self.plp_ids = torch.full((B, M, MAX_LOGPROBS), -1, dtype=torch.int32, device=dev)
        self.plp_top = torch.full((B, M, MAX_LOGPROBS), float("nan"), dtype=torch.float32, device=dev)

    def _start_logit_bias(self):
        """The mask-and-bias kernel joins op_accept, with every slot's device rows; it writes no scratch, so nothing joins
        the captured buffers."""
        self.use_logit_bias = True
        B, dev = self.B, self.device
        i32 = dict(dtype=torch.int32, device=dev)
        self.allowed_dev = torch.zeros(B, ops.mask_words(self.V), **i32)
        self.has_mask_dev = torch.zeros(B, **i32)
        self.n_bias_dev = torch.zeros(B, **i32)
        self.bias_ids_dev = torch.zeros(B, MAX_LOGIT_BIAS, **i32)
        self.bias_vals_dev = torch.zeros(B, MAX_LOGIT_BIAS, dtype=torch.float32, device=dev)
        for b in range(B):
            self._write_logit_bias(b)

    def _write_logit_bias(self, b: int):
        """Slot b's device rows from its host settings: the bitmask (zeros without a set) and the entries (zero padded)."""
        bias, allowed = self.logit_bias[b] or (), self.allowed_token_ids[b]
        mask = ops.pack_token_mask(allowed, self.V) if allowed is not None else torch.zeros(ops.mask_words(self.V),
                                                                                             dtype=torch.int32)
        ids = torch.zeros(MAX_LOGIT_BIAS, dtype=torch.int32)
        vals = torch.zeros(MAX_LOGIT_BIAS, dtype=torch.float32)
        if bias:
            ids[:len(bias)] = torch.tensor([t for t, _ in bias], dtype=torch.int32)
            vals[:len(bias)] = torch.tensor([v for _, v in bias], dtype=torch.float32)
        self.allowed_dev[b].copy_(_h2d(mask), non_blocking=True)
        self.bias_ids_dev[b].copy_(_h2d(ids), non_blocking=True)
        self.bias_vals_dev[b].copy_(_h2d(vals), non_blocking=True)
        self.has_mask_dev[b] = 0 if allowed is None else 1
        self.n_bias_dev[b] = len(bias)

    def _start_ban(self):
        """The ban kernel joins op_accept, with every slot's device rows; it writes no scratch, so nothing joins the
        captured buffers."""
        self.use_ban = True
        B, dev = self.B, self.device
        i32 = dict(dtype=torch.int32, device=dev)
        self.words_dev = torch.zeros(B, MAX_BAD_WORDS, MAX_BAD_WORD_LEN, **i32)
        self.word_len_dev = torch.zeros(B, MAX_BAD_WORDS, **i32)
        self.n_words_dev = torch.zeros(B, **i32)
        self.min_end_dev = torch.zeros(B, **i32)
        self.default_end_dev = torch.tensor([_stop_row(DEFAULT_END_IDS)] * B, **i32)
        for b in range(B):
            self._write_ban(b)

    def _write_ban(self, b: int):
        """Slot b's device rows from its host settings: the words (zero padded), their lengths and L + min_tokens."""
        words = self.bad_words[b] or ()
        table = torch.zeros(MAX_BAD_WORDS, MAX_BAD_WORD_LEN, dtype=torch.int32)
        lens = torch.zeros(MAX_BAD_WORDS, dtype=torch.int32)
        for i, w in enumerate(words):
            table[i, :len(w)] = torch.tensor(w, dtype=torch.int32)
            lens[i] = len(w)
        self.words_dev[b].copy_(_h2d(table), non_blocking=True)
        self.word_len_dev[b].copy_(_h2d(lens), non_blocking=True)
        self.n_words_dev[b] = len(words)
        self.min_end_dev[b] = _min_end(self.prompt_lens[b], self.min_tokens[b])

    def _ban_end_ids(self) -> torch.Tensor:
        """The (B, MAX_STOP) end-id rows the ban kernel reads: in stop mode the stop walks' own stop_ids_dev, so a slot's
        end ids are its stop ids with no copy to keep in step; in default mode DEFAULT_END_IDS for every slot.  Stop mode
        starts with a recapture, which takes the new array into the graphs."""
        return self.stop_ids_dev if self.use_stop else self.default_end_dev

    def _start_guide(self):
        """The guide kernels join op_accept and seq_post, with the blob table and the node-state scratch (rewritten every
        step before it is read, so not one of the captured buffers)."""
        self.use_guide = True
        self.guide_table_dev = torch.zeros(self.B, dtype=torch.int64, device=self.device)
        self.guide_scratch = torch.zeros(self.B, self.S, dtype=torch.int32, device=self.device)
        for b in range(self.B):
            self._write_guide(b)

    def _write_guide(self, b: int):
        """Slot b's blob and table entry from its host guide: a slot whose guide another slot already holds shares that
        slot's blob; the old blob is released (the stream orders its reuse after the kernels that read it)."""
        g = self.guides[b]
        blob = None
        if g is not None:
            blob = next((self.guide_blobs[o] for o in range(self.B) if o != b and self.guides[o] is g
                         and self.guide_blobs[o] is not None), None)
            if blob is None:
                blob = g.pack(self.V).to(self.device, non_blocking=False)
        self.guide_blobs[b] = blob
        self.guide_table_dev[b] = 0 if blob is None else blob.data_ptr()

    def guide_state(self, b: int) -> int:
        """Slot b's guide state after its committed tokens, from the host copy of the state words of its last verify()
        (the guide's start before its first one); -1 once a token has left the guide.  Refused for a slot without a
        guide."""
        if not 0 <= b < self.B:
            raise IndexError(f"slot {b} out of range for a batch of {self.B}")
        g = self.guides[b]
        if g is None:
            raise ValueError(f"slot {b} has no guide (guide=None)")
        return g.start if self.last[b] is None else int(self.host_state[b, ST_GUIDE_STATE])

    def _draft_processed(self) -> bool:
        """Whether the draft graph processes draft rows: a constrained tree with at least one constraint kind started."""
        return self.constrain_draft and (self.use_logit_bias or self.use_ban or self.use_guide)

    def _start_kind(self):
        """A constraint kind starts (its kernel joins op_accept): capture steady and post once more, and the draft graph
        too in a constrained tree (its processing and the walks' dead-child rule enter)."""
        for name in ("draft", "steady", "post") if self.constrain_draft else ("steady", "post"):
            self.graphs.pop(name, None)

    def _load_prompt(self, b: int, prompt: torch.Tensor):
        """Row b of tokens, position ids, state and accept_idx for a new prompt: nothing of an earlier occupant stays."""
        P, S, M = len(prompt), self.S, self.M
        pos = torch.zeros(M, dtype=torch.int64)
        pos[:P] = torch.arange(P)
        pos[P:P + S - 1] = self.st.depth_cpu[1:] + P - 1
        st0 = torch.zeros(16, dtype=torch.int32)
        st0[ST_P], st0[ST_M] = P, M
        g = self.guides[b]
        if g is not None:
            st0[ST_GUIDED], st0[ST_GUIDE_STATE], st0[ST_GUIDE_POS] = 1, g.start, P
        self.tokens[b].zero_()
        self.tokens[b, :P].copy_(_h2d(prompt), non_blocking=True)
        self.position_ids[b].copy_(_h2d(pos), non_blocking=True)
        self.state[b].copy_(_h2d(st0), non_blocking=True)
        self.accept_idx[b].zero_()

    def _prefill_start(self, b: int) -> int:
        """The first prompt row slot b's draft prefill and first verify run: L of a reused prefix, else 0."""
        reused = self.reused_prefix[b]
        return 0 if reused is None else reused[1]

    def op_draft_prefill(self, seqs):
        """Draft prefill of the sequences `seqs` (SpecTree.py:67-80) as one ragged forward: each one's rows [L, P) causal
        (L = 0 unless its admission reused a prefix), its last row's logits -> its node 0."""
        parts = []
        for b in seqs:
            P, L = self.ground_truth_len[b], self._prefill_start(b)
            parts.append((b, P - L, 1 - P + L, 1, 1, self.draft_logits[b:b + 1]))
        self.draft.engine.runner.forward_ragged(parts, self.tokens, self.position_ids, self.storage_ids, state=self.state,
                                                **self._mask_kw())

    def _reuse_prefix(self, b: int, prompt: torch.Tensor):
        """Find the prefix an admission of `prompt` into slot b reuses (prefix_donor over every slot's ready prefix
        tokens[d, :target_kv_len[d]], read back in one device-to-host copy) and copy its K/V rows from another slot into
        b's, in both caches.  Runs before slot b's token row is reloaded.  -> (donor, L) or None."""
        P = len(prompt)
        m = min(P - 1, max(self.target_kv_len))
        if m < 1 or self.prompt_logprobs_n[b] is not None:
            return None
        # (L <= m, so the prompt's first m + 1 tokens give the same donor and L as the whole prompt; on the device they
        # travel with the rows, in the same copy)
        if prompt.is_cuda:
            both = torch.cat([self.tokens[:, :m + 1], prompt[None, :m + 1].to(torch.int64)]).cpu()
            rows, head = both[:self.B], both[self.B]
        else:
            rows, head = self.tokens[:, :m].cpu(), prompt[:m + 1]
        donor, L = prefix_donor(head, rows, self.target_kv_len, b, self.prompt_logprobs_n[b])
        if L == 0:
            return None
        if donor != b:
            for eng in (self.draft, self.target):
                ops.kv_copy_prefix(eng.engine.kv_cache, donor, b, L)
        return donor, L

    def freeze(self, b: int):
        """Stop sequence b (the caller's length limit); it stays frozen until admit() gives the slot a new prompt."""
        self.frozen[b] = True
        self.state[b, ST_FROZEN] = 1

    @torch.inference_mode()
    def admit(self, b: int, prompt: torch.Tensor, temperature: Optional[float] = None, top_p: Optional[float] = None,
              seed: Optional[int] = None, policy: Optional[str] = None, top_k: Optional[int] = None,
              stop_tokens=_PREVIOUS, max_new_tokens=_PREVIOUS, repetition_penalty: Optional[float] = None,
              frequency_penalty: Optional[float] = None, presence_penalty: Optional[float] = None,
              logprobs=_PREVIOUS, logit_bias=_PREVIOUS, allowed_token_ids=_PREVIOUS, min_p: Optional[float] = None,
              bad_words=_PREVIOUS, min_tokens=_PREVIOUS, guide=_PREVIOUS, prompt_logprobs=_PREVIOUS,
              reuse_prefix: bool = False):
        """Start `prompt` in the frozen slot b (finished, out of room, or stopped with freeze), at its own policy,
        temperature, top_p and top_k (default: the slot's previous values).  The next verify() runs its first verify next
        to the steady sequences.  The slot draws r and rand as a lone SpecTree on the prompt would, and runs its draft
        prefill now.
        A seeded tree takes the prompt's `seed` (required there, refused otherwise): r and rand are then filled on the
        device from that seed's stream and the slot's noise counter restarts at 0.
        The first admission that puts both policies in the batch starts mixed mode: the draft, steady and post graphs are
        captured once more, on their next use.  A tree built all-greedy allocates r and rand at its first "spec"
        admission.  The first "spec" admission with 0 < top_k < V (in a tree that had none) captures the steady and post
        graphs once more: the top-k filter joins the accept step.
        min_p: the prompt's min_p (default: the slot's previous one).  The first "spec" admission with min_p > 0, in a tree
        that had none, captures the steady and post graphs once more: the min-p filter joins the accept step.
        stop_tokens / max_new_tokens: the prompt's stop set and token budget (default: the slot's previous ones; None is
        none).  The budget counts from this prompt.  The first admission that brings a stop set or a budget to a tree in
        default mode captures the steady and post graphs once more: the stop walks replace the walks.
        repetition_penalty / frequency_penalty / presence_penalty: the prompt's penalties (default: the slot's previous
        ones); they count this prompt and its output only.  The first non-neutral setting in a tree without one captures
        the steady and post graphs once more.
        logprobs: the prompt's logprobs setting (default: the slot's previous one; None is off).  The first one that is
        on, in a tree without one, captures the steady and post graphs once more.
        prompt_logprobs: the prompt's prompt_logprobs setting (default: the slot's previous one; None is off).  Its values
        come from the next verify(), the prompt's first; until then prompt_logprobs(b) is refused.  No recapture.
        logit_bias / allowed_token_ids: the prompt's logit bias and allowed set (default: the slot's previous ones; None is
        none).  The first non-neutral one, in a tree without one, captures the steady and post graphs once more.
        bad_words / min_tokens: the prompt's bad words (None is none) and min_tokens (default: the slot's previous ones);
        min_tokens counts from this prompt.  The first non-neutral one, in a tree without one, captures the steady and post
        graphs once more.
        guide: the prompt's guide (default: the slot's previous one; None is none), which starts at its start state.  The
        first guide, in a tree without one, captures the steady and post graphs once more.
        reuse_prefix: a bool (default False).  With True the prompt reuses the longest prefix whose K/V a slot already
        holds (prefix_donor): slot d offers its first target_kv_len[d] tokens, its ready prefix, which is 0 until its
        current prompt's first verify, then the committed length minus the bonus token after each verify that leaves it
        decoding, and unchanged by the verify that ends it (the rows below that step's start are never rewritten).  Slot
        b itself is a candidate: its previous occupant's rows are still there (multi-turn chat: the finished output plus
        a new turn).  With L >= 1 reused rows from another slot, sq_kv_copy_prefix copies them into b's rows of the draft
        and the target cache; the draft prefill then runs rows [L, P) and the first verify rows [L, P + S - 1).  L is at
        most P - 1, and 0 for a slot with prompt_logprobs on.  reused_prefix[b] reports (donor, L), or None.  A slot
        admitted since the last verify() is no donor (its ready length is 0): to fan one prompt out to several slots
        (parallel sampling), admit it once, run one verify(), then admit the copies with reuse_prefix=True.  The reused
        rows hold the donor's bytes, computed by a forward of another shape, so the admission matches a full prefill up
        to fp16 rounding, not bit for bit; a seeded "spec" slot may commit a different, equally distributed output.
        No graph is captured again."""
        check_reuse_prefix(reuse_prefix)
        if policy is not None:
            check_policy(policy)
        if top_k is not None:
            top_k = check_top_k(top_k)
        if min_p is not None:
            min_p = check_min_p(min_p)
        if stop_tokens is not _PREVIOUS:
            stop_tokens = check_stop_tokens(stop_tokens, self.V)
        if max_new_tokens is not _PREVIOUS:
            max_new_tokens = check_max_new_tokens(max_new_tokens)
        pens = [None if v is None else check_penalty(name, v) for name, v in
                (("repetition_penalty", repetition_penalty), ("frequency_penalty", frequency_penalty),
                 ("presence_penalty", presence_penalty))]
        if logprobs is not _PREVIOUS:
            logprobs = check_logprobs(logprobs)
        if prompt_logprobs is not _PREVIOUS:
            prompt_logprobs = check_prompt_logprobs(prompt_logprobs)
        if logit_bias is not _PREVIOUS:
            logit_bias = check_logit_bias(logit_bias, self.V)
        if allowed_token_ids is not _PREVIOUS:
            allowed_token_ids = check_allowed_token_ids(allowed_token_ids, self.V)
        if bad_words is not _PREVIOUS:
            bad_words = check_bad_words(bad_words, self.V)
        if min_tokens is not _PREVIOUS:
            min_tokens = check_min_tokens(min_tokens)
        if guide is not _PREVIOUS:
            guide = check_guide(guide)
        if not 0 <= b < self.B:
            raise IndexError(f"slot {b} out of range for a batch of {self.B}")
        if not self.frozen[b]:
            raise ValueError(f"slot {b} is still decoding; admit takes a finished or frozen slot")
        P = len(prompt)
        if P < 1 or P + self.S - 1 > self.M:
            raise ValueError(f"max_length={self.M} must hold the prompt ({P}) + tree ({self.S}) - 1")
        T = self.temps[b] if temperature is None else float(temperature)
        tp = self.top_ps[b] if top_p is None else float(top_p)
        check_sampling(T, tp)
        if self.seeded and seed is None:
            raise ValueError("this BatchTree was built with seeds: admit needs the prompt's seed=")
        if not self.seeded and seed is not None:
            raise ValueError("seed= needs a BatchTree built with seeds")
        if seed is not None:
            seed = check_seed(seed)
        pol = self.policies[b] if policy is None else policy
        k = self.top_ks[b] if top_k is None else top_k
        mp = self.min_ps[b] if min_p is None else min_p
        stop = self.stop_tokens[b] if stop_tokens is _PREVIOUS else stop_tokens
        budget = self.max_new_tokens[b] if max_new_tokens is _PREVIOUS else max_new_tokens
        rep, freq, pres = (old[b] if v is None else v for v, old in
                           zip(pens, (self.repetition_penalty, self.frequency_penalty, self.presence_penalty)))
        if not is_neutral(rep, freq, pres) and self.M > PENALTY_MAX_LEN:
            raise ValueError(f"penalties count at most {PENALTY_MAX_LEN} tokens; this tree's max_length={self.M}")
        words = self.bad_words[b] if bad_words is _PREVIOUS else bad_words
        m = self.min_tokens[b] if min_tokens is _PREVIOUS else min_tokens
        check_min_tokens(m, budget)
        allowed = self.allowed_token_ids[b] if allowed_token_ids is _PREVIOUS else allowed_token_ids
        check_bannable(self.V, words, allowed, m, end_ids(stop, self.use_stop or stop is not None or budget is not None))
        gd = self.guides[b] if guide is _PREVIOUS else guide
        if gd is not None:
            gd.check(self.V, allowed, words)
        # (every other slot holds the tree's one policy until then, so a different one means both are present; at B = 1
        # it is a switch, which the single-policy graphs do not serve either)
        enter_mixed = not self.mixed and pol != ("greedy" if self.greedy else "spec")
        self.temps[b], self.top_ps[b], self.policies[b] = T, tp, pol
        self.T_dev[b] = T
        self.top_p_dev[b] = 1.0 if pol == "greedy" else tp
        self.greedy_dev[b] = 1 if pol == "greedy" else 0
        self.top_ks[b] = k
        self.top_k_dev[b] = 0 if pol == "greedy" else min(k, self.V)
        if enter_mixed:
            self.mixed, self.greedy = True, False  # the mixed sampler and walks enter every graph: capture them once more
            for name in ("draft", "steady", "post"):
                self.graphs.pop(name, None)
        if tp < 1.0 and pol == "spec" and not self.use_top_p:
            self.use_top_p = True                  # the filter enters op_accept: capture steady and post once more
            for name in ("steady", "post"):
                self.graphs.pop(name, None)
        if 0 < k < self.V and pol == "spec" and not self.use_top_k:
            self.use_top_k = True                  # the same for the top-k filter
            for name in ("steady", "post"):
                self.graphs.pop(name, None)
        self.min_ps[b] = mp
        self.log_min_p_dev[b] = _log_min_p(pol, mp)
        if mp > 0.0 and pol == "spec" and not self.use_min_p:
            self.use_min_p = True                  # the same for the min-p filter
            for name in ("steady", "post"):
                self.graphs.pop(name, None)
        self.stop_tokens[b], self.max_new_tokens[b] = stop, budget
        self.stop_ids_dev[b] = torch.tensor(_stop_row(stop), dtype=torch.int32)
        self.end_limit_dev[b] = _end_limit(P, budget)
        if (stop is not None or budget is not None) and not self.use_stop:
            self.use_stop = True                   # the stop walks replace the walks: capture steady and post once more
            # (and the draft graph when it bans end ids: they become the stop ids, as in the target rows)
            for name in ("draft", "steady", "post") if self.constrain_draft and self.use_ban else ("steady", "post"):
                self.graphs.pop(name, None)
        self.repetition_penalty[b], self.frequency_penalty[b], self.presence_penalty[b] = rep, freq, pres
        self.rep_dev[b], self.freq_dev[b], self.pres_dev[b] = rep, freq, pres
        self.prompt_len_dev[b] = P
        if not is_neutral(rep, freq, pres) and not self.use_penalty:
            self._start_penalties()                # the penalty kernels enter op_accept: capture steady and post once more
            for name in ("steady", "post"):
                self.graphs.pop(name, None)
        n_lp = self.logprobs[b] if logprobs is _PREVIOUS else logprobs
        self.logprobs[b] = n_lp
        self.n_top_dev[b] = -1 if n_lp is None else n_lp
        self.prompt_lens[b] = P
        if n_lp is not None and not self.use_logprobs:
            self._start_logprobs()                 # the logprobs kernel enters seq_post: capture steady and post once more
            for name in ("steady", "post"):
                self.graphs.pop(name, None)
        if prompt_logprobs is not _PREVIOUS:
            self.prompt_logprobs_n[b] = prompt_logprobs
        self.plp_ready[b] = False                  # the earlier occupant's values are not this prompt's
        if self.prompt_logprobs_n[b] is not None and self.plp_token is None:
            self._start_prompt_logprobs()
        if logit_bias is not _PREVIOUS:
            self.logit_bias[b] = logit_bias
        if allowed_token_ids is not _PREVIOUS:
            self.allowed_token_ids[b] = allowed_token_ids
        if self.use_logit_bias:
            self._write_logit_bias(b)
        elif not is_neutral_bias(self.logit_bias[b], self.allowed_token_ids[b]):
            self._start_logit_bias()               # the bias kernel enters op_accept: capture steady and post once more
            self._start_kind()
        self.bad_words[b], self.min_tokens[b] = words, m
        if self.use_ban:
            self._write_ban(b)
        elif not is_neutral_ban(words, m):
            self._start_ban()                      # the ban kernel enters op_accept: capture steady and post once more
            self._start_kind()
        self.guides[b] = gd
        if self.use_guide:
            self._write_guide(b)
        elif gd is not None:
            self._start_guide()                    # the guide kernels enter the graphs: capture steady and post once more
            self._start_kind()
        if pol == "spec" and self.r is None:       # the first sampling sequence of a tree built all-greedy
            self.r = torch.zeros(self.B, self.M, dtype=F16, device=self.device)
            self.rand = torch.zeros(self.B, self.S, self.V, dtype=F16, device=self.device)
        self.reused_prefix[b] = self._reuse_prefix(b, prompt) if reuse_prefix else None   # (the copies first)
        self._load_prompt(b, prompt)
        self.frozen[b] = False
        self.finish_reason[b] = None
        self.last[b] = None
        self.ground_truth_len[b] = P
        self.target_kv_len[b] = 0
        if self.seeded:
            self.seeds[b] = _as_int64(seed)
            self.steps[b] = 0
            if pol == "spec":
                ops.rng_uniform_seqs(self.r, self.seeds, [b], ops.RNG_R)
                ops.rng_uniform_seqs(self.rand, self.seeds, [b], ops.RNG_RAND)
        elif self.r is not None:                   # (a greedy prompt of a mixed batch draws too: stream alignment)
            r, rand = draw_random([prompt], self.M, self.S, self.V)
            self.r[b].copy_(_h2d(r[0]), non_blocking=True)
            self.rand[b].copy_(_h2d(rand[0]), non_blocking=True)
        self.op_draft_prefill([b])

    # ---- the op sequences ------------------------------------------------------------------------------------------------
    def op_sample(self, i: int):
        lv = self.st.levels[i]
        if self.mixed:
            ops.sample_level_batch_mixed(self.draft_logits, self.row_base, self.row_step, self.rand, lv["n_parents"],
                                         lv["k"], self.T_dev, self.greedy_dev, parent_rows=lv["parents"],
                                         child_first=lv["first"], n_branch=lv["nb"], tokens=self.tokens, state=self.state)
            return
        ops.sample_level_batch_per_seq(self.draft_logits, self.row_base, self.row_step, self.rand, lv["n_parents"],
                                       lv["k"], self.T_dev, 1 if self.greedy else 0, parent_rows=lv["parents"],
                                       child_first=lv["first"], n_branch=lv["nb"], tokens=self.tokens, state=self.state)

    def op_draft_level(self, i: int):
        lv = self.st.levels[i]
        n0, tb, B = lv["n0"], lv["tb"], self.B
        self.draft.engine.runner.forward(tb, self.tokens, self.position_ids, self.storage_ids, state=self.state, n0=n0,
                                         kv_end=n0 + tb, batch=True, logits_out=self.draft_logits[B * n0:B * (n0 + tb)],
                                         **self._mask_kw())

    def op_target_steady(self):
        self.target.engine.runner.forward(self.S, self.tokens, self.position_ids, self.storage_ids, state=self.state,
                                          n0=0, kv_end=self.S, batch=True, logits_out=self.target_logits,
                                          **self._mask_kw())

    def op_target_first(self, seqs):
        """First verify of the sequences `seqs` (SpecTree.py:164-176) as one ragged forward: each one's rows [L, P+S-1)
        (L = 0 unless its admission reused a prefix), the logits of its S tree rows.  Then the prompt logprobs of those
        with the setting on (op_prompt_logprobs; their L is 0)."""
        S = self.S
        runner = self.target.engine.runner
        parts = []
        for b in seqs:
            P, L = self.ground_truth_len[b], self._prefill_start(b)
            parts.append((b, P - L + S - 1, 1 - P + L, S, S, self.target_logits[b * S:(b + 1) * S]))
        row0 = runner.forward_ragged(parts, self.tokens, self.position_ids, self.storage_ids, state=self.state,
                                     **self._mask_kw())
        self.op_prompt_logprobs(seqs, row0)

    def op_prompt_logprobs(self, seqs, row0):
        """Prompt logprobs of the first-verify sequences `seqs` with the setting on and P >= 2, whose ragged forward left
        the final-normed rows of sequence seqs[j] at the target runner's rows [row0[j], ...): one lm_head GEMM per
        sequence over its prompt rows [row0[j], row0[j] + P - 1), into the runner's logits at the same rows, then one
        sq_prompt_logprobs_ragged launch for all of them.  Eager (outside every graph); nothing when no sequence is on."""
        runner = self.target.engine.runner
        parts = [(b, r0, self.ground_truth_len[b] - 1, self.prompt_logprobs_n[b]) for b, r0 in zip(seqs, row0)
                 if self.prompt_logprobs_n[b] is not None and self.ground_truth_len[b] >= 2]
        if not parts:
            return
        for _, r0, n_rows, _ in parts:
            runner.lm_head_rows(r0, r0 + n_rows)
        ops.prompt_logprobs_ragged_(runner.logits, parts, self.tokens, self.plp_token, self.plp_ids, self.plp_top)

    def op_accept(self):
        st = self.st
        policy = ops.ACCEPT_SKIP_DEAD if self._draft_processed() else 0
        if self.use_guide:                         # the node states first: they read the tree tokens only
            ops.guide_states_batch(self.guide_table_dev, self.tokens, self.state, st.depth, st.tree_bits, st.tree_words,
                                   self.S, self.V, self.guide_scratch)
        if self.use_logit_bias:                    # first: a bias is in logit space, the penalties then scale it
            ops.logit_bias_rows_batch_(self.target_logits, self.S, self.state, self.allowed_dev, self.has_mask_dev,
                                       self.bias_ids_dev, self.bias_vals_dev, self.n_bias_dev)
        if self.use_ban:                           # -inf whatever the bias; the penalties leave -inf alone
            ops.ban_tokens_rows_batch_(self.target_logits, self.tokens, self.state, self.prompt_len_dev, st.depth,
                                       st.tree_bits, st.tree_words, self.S, self.words_dev, self.word_len_dev,
                                       self.n_words_dev, self.min_end_dev, self._ban_end_ids())
        if self.use_guide:                         # -inf whatever the bias and the ban; the penalties leave -inf alone
            ops.guide_mask_rows_batch_(self.target_logits, self.S, self.state, self.guide_table_dev, self.guide_scratch)
        if self.use_penalty:                       # first: the greedy walk and the filters rank the penalised rows
            ops.penalize_rows_batch_(self.target_logits, self.tokens, self.state, self.prompt_len_dev, st.tree_bits,
                                     st.tree_words, self.S, self.rep_dev, self.freq_dev, self.pres_dev, self.pen_scratch)
        if self.greedy:
            ops.argmax_rows(self.target_logits, self.target_token)
            if self.use_stop:
                ops.accept_greedy_batch_stop(self.target_token, st.succ_off, st.succ, st.depth, self.S, None,
                                             self.stop_ids_dev, self.end_limit_dev, self.tokens, self.position_ids,
                                             self.accept_idx, self.state, self.max_target_seq)
                return
            ops.accept_greedy_batch(self.target_token, st.succ_off, st.succ, st.depth, self.S, self.tokens,
                                    self.position_ids, self.accept_idx, self.state, self.max_target_seq)
            return
        if self.mixed:                             # the greedy sequences' walk; the sampling ones' follows below
            ops.argmax_rows(self.target_logits, self.target_token)
            if self.use_stop:
                ops.accept_greedy_batch_stop(self.target_token, st.succ_off, st.succ, st.depth, self.S, self.greedy_dev,
                                             self.stop_ids_dev, self.end_limit_dev, self.tokens, self.position_ids,
                                             self.accept_idx, self.state, self.max_target_seq)
            else:
                ops.accept_greedy_batch_mixed(self.target_token, st.succ_off, st.succ, st.depth, self.S, self.greedy_dev,
                                              self.tokens, self.position_ids, self.accept_idx, self.state,
                                              self.max_target_seq)
        if self.use_min_p:                         # vLLM's order: min_p, top_k, top_p (min_p and top_k commute)
            ops.min_p_filter_per_seq_(self.target_logits, self.log_min_p_dev, self.T_dev, self.S)
        if self.use_top_k:                         # top_k before top_p: top_p renormalises over the k survivors
            ops.top_k_filter_per_seq_(self.target_logits, self.top_k_dev, self.S)
        if self.use_top_p:
            ops.top_p_filter_per_seq_(self.target_logits, self.top_p_dev, self.T_dev, self.S)
        if self.external_noise is None:
            if self.seeded:
                ops.rng_exponential_batch(self.noise, self.seeds, self.steps, self.state)
            else:
                self.noise.exponential_(1.0)
        if self.use_stop:
            ops.accept_stochastic_batch_stop(self.target_logits, self.draft_logits, self.row_base, self.row_step, self.r,
                                             self.noise, st.succ_off, st.succ, st.depth, self.S, self.T_dev,
                                             self.greedy_dev if self.mixed else None, self.stop_ids_dev,
                                             self.end_limit_dev, self.tokens, self.position_ids, self.accept_idx,
                                             self.state, self.max_target_seq, policy)
            return
        if self.mixed:
            ops.accept_stochastic_batch_mixed(self.target_logits, self.draft_logits, self.row_base, self.row_step, self.r,
                                              self.noise, st.succ_off, st.succ, st.depth, self.S, self.T_dev,
                                              self.greedy_dev, self.tokens, self.position_ids, self.accept_idx, self.state,
                                              self.max_target_seq, policy)
            return
        ops.accept_stochastic_batch_per_seq(self.target_logits, self.draft_logits, self.row_base, self.row_step, self.r,
                                            self.noise, st.succ_off, st.succ, st.depth, self.S, self.T_dev, self.tokens,
                                            self.position_ids, self.accept_idx, self.state, self.max_target_seq, policy)

    def op_kv_gather(self):
        md = max(self.st.max_depth, 1)
        for eng in (self.draft, self.target):
            kv = eng.engine.kv_cache
            ops.kv_gather_batch(kv.k_cache, kv.v_cache, self.accept_idx, self.state, md)

    def op_bonus_forward(self):
        self.draft.engine.runner.forward(1, self.tokens, self.position_ids, self.storage_ids, state=self.state, n0=0,
                                         kv_end=1, batch=True, logits_out=self.draft_logits[0:self.B], **self._mask_kw())

    def op_draft_rows(self, k0: int, nk: int):
        """The draft rows of nodes [k0, k0 + nk) of every sequence get the processing their target rows get in op_accept,
        up to and including the guide mask (one launch)."""
        st = self.st
        ops.draft_rows_batch_(
            self.draft_logits, self.row_base, self.row_step, k0, nk, self.S, self.state,
            bias=(self.allowed_dev, self.has_mask_dev, self.bias_ids_dev, self.bias_vals_dev, self.n_bias_dev)
            if self.use_logit_bias else None,
            ban=(self.prompt_len_dev, st.depth, self.words_dev, self.word_len_dev, self.n_words_dev, self.min_end_dev,
                 self._ban_end_ids()) if self.use_ban else None,
            guide=(self.guide_table_dev, self.guide_scratch) if self.use_guide else None,
            tokens=self.tokens, tree_bits=st.tree_bits, tree_words=st.tree_words)

    def seq_draft(self):
        levels = self.st.levels
        processed = self._draft_processed()
        if processed:                              # the root row, from the bonus forward or an admission's draft prefill
            self.op_draft_rows(0, 1)
        for i in range(self.st.draft_step - 1):
            self.op_sample(i)
            self.op_draft_level(i)
            if processed and i + 1 < len(levels):  # a level whose nodes have children: before op_sample(i + 1) reads it
                self.op_draft_rows(levels[i]["n0"], levels[i]["tb"])

    def op_logprobs(self):
        ops.token_logprobs_batch_(self.target_logits, self.S, self.st.max_depth, self.tokens, self.state, self.accept_idx,
                                  self.T_dev, self.greedy_dev, self.n_top_dev, self.lp_token, self.lp_ids, self.lp_top)

    def seq_post(self):
        self.op_accept()
        if self.use_guide:                         # the committed tokens through the guide, before the host-state copy
            ops.guide_advance_batch(self.guide_table_dev, self.tokens, self.state, self.V)
        if self.use_logprobs:                      # the rows as the walk read them, before anything else writes them
            self.op_logprobs()
        self.op_kv_gather()
        self.op_bonus_forward()
        self.host_state.copy_(self.state, non_blocking=True)

    def seq_steady(self):
        self.op_target_steady()
        self.seq_post()

    # ---- graphs (as sequoia_b200.tree._Runtime) --------------------------------------------------------------------------
    def run(self, name: str, fn):
        if not self.use_graphs:
            fn()
            return
        g = self.graphs.get(name)
        if g is None:
            snap = self._snapshot()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                fn()
                s.synchronize()
            torch.cuda.current_stream().wait_stream(s)
            self._restore(snap)
            g = torch.cuda.CUDAGraph()
            c0 = _lib.launch_count()
            with torch.cuda.graph(g):
                fn()
            self.graph_launches[name] = _lib.launch_count() - c0
            self._restore(snap)
            self.graphs[name] = g
            self.captures[name] = self.captures.get(name, 0) + 1
        g.replay()
        self.replays[name] = self.replays.get(name, 0) + 1
        self.replayed_launches += self.graph_launches[name]      # per replay: a recapture changes the count

    def _caches(self):
        return [t for e in (self.draft, self.target) for t in (e.engine.kv_cache.k_cache, e.engine.kv_cache.v_cache)]

    def _captured_bufs(self):
        """The device buffers a graph's warm-up run writes (the noise counters of a seeded tree included, so that a
        sequence's noise does not depend on when the graphs were captured)."""
        bufs = [self.tokens, self.position_ids, self.state, self.draft_logits, self.target_logits, self.noise]
        if self.use_logprobs:
            bufs += [self.lp_token, self.lp_ids, self.lp_top]
        return bufs + [self.steps] if self.seeded else bufs

    def _snapshot(self):
        return dict(bufs=[t.clone() for t in self._captured_bufs()],
                    kv=[t.clone() for t in self._caches()], rng=torch.cuda.get_rng_state(self.device))

    def _restore(self, s):
        for t, c in zip(self._captured_bufs(), s["bufs"]):
            t.copy_(c)
        for t, c in zip(self._caches(), s["kv"]):
            t.copy_(c)
        torch.cuda.set_rng_state(s["rng"], self.device)

    def kernel_launches(self) -> int:
        """Kernels launched by graph replays so far, each replay counted with the launches of the graph it replayed."""
        return self.replayed_launches

    # ---- the reference-style steps ---------------------------------------------------------------------------------------
    @torch.inference_mode()
    def construct_grow_map(self):
        self.run("draft", self.seq_draft)

    @torch.inference_mode()
    def verify(self):
        """-> [(valid_tokens, accept_length, terminal)] per sequence; a frozen sequence repeats its last result."""
        if self.external_noise is not None and not self.greedy:
            self.noise.copy_(self.external_noise[self.iter])
        first = [b for b in range(self.B) if not self.frozen[b] and self.target_kv_len[b] != self.ground_truth_len[b] - 1]
        for b in range(self.B):                         # this step is every decoding prompt's first verify or a later one
            self.plp_ready[b] = self.plp_ready[b] or not self.frozen[b]
        if first:
            if len(first) + sum(self.frozen) < self.B:
                # steady sequences share the step with admitted ones: their tree rows first, the admitted slots frozen
                saved = self.state.clone()
                for b in first:
                    self.state[b, ST_FROZEN] = 1
                self.op_target_steady()
                self.state.copy_(saved)
            # prefill + tree rows of every first-verify sequence in one ragged forward (their row counts differ); the walk
            # and the rest batched
            self.op_target_first(first)
            self.run("post", self.seq_post)
        else:
            self.run("steady", self.seq_steady)
        torch.cuda.current_stream().synchronize()       # the one host sync of a verify step
        self.iter += 1
        hs = self.host_state
        out = []
        for b in range(self.B):
            if self.frozen[b]:
                out.append(self.last[b])
                continue
            a, terminal, skipped = int(hs[b, 1]), bool(hs[b, 2]), bool(hs[b, 7])
            finish = int(hs[b, ST_FINISH])          # (always 0 in default mode: only the stop walks write it)
            if self.guides[b] is not None and int(hs[b, ST_GUIDE_STATE]) < 0:
                valid = self.tokens[b, :int(hs[b, ST_GUIDE_POS])]     # the longest prefix the guide accepts
                terminal = True
                self.finish_reason[b] = "guide"
            elif finish:
                valid = self.tokens[b, :int(hs[b, ST_END])]
                terminal = True
                self.finish_reason[b] = "stop" if finish == 1 else "length"
            elif terminal:
                valid = self.tokens[b, :a]
                self.finish_reason[b] = "nan" if bool(hs[b, 6]) else "stop"
            elif skipped:
                valid = self.tokens[b, :min(a + 1, self.M)]
                self.finish_reason[b] = "room"
            else:
                valid = self.tokens[b, :a + 1]
                self.ground_truth_len[b] = a + 1
                self.target_kv_len[b] = a
            self.last[b] = (valid, a, terminal)
            if terminal or skipped:
                self.freeze(b)
            out.append(self.last[b])
        return out

    def token_logprobs(self, b: int):
        """Slot b's generated tokens so far (positions len(prompt) .. len(its last verify() tokens)), on the host:
        -> (token_lp (n,) float32, top_ids (n, k) int64, top_lp (n, k) float32), k = the slot's logprobs setting (at most
        V).  token_lp[i] is the log-probability of generated token i, top_ids[i] / top_lp[i] the k best ids of its row,
        best first, and theirs.  Refused for a slot whose logprobs are off."""
        if not 0 <= b < self.B:
            raise IndexError(f"slot {b} out of range for a batch of {self.B}")
        n_lp = self.logprobs[b]
        if n_lp is None:
            raise ValueError(f"slot {b} has logprobs off (logprobs=None)")
        L = self.prompt_lens[b]
        end = L if self.last[b] is None else max(L, len(self.last[b][0]))
        k = min(n_lp, self.V)
        return (self.lp_token[b, L:end].cpu(), self.lp_ids[b, L:end, :k].cpu().to(torch.int64),
                self.lp_top[b, L:end, :k].cpu())

    def prompt_logprobs(self, b: int):
        """Slot b's prompt scores, on the host: -> (token_lp (P-1,) float32, top_ids (P-1, k) int64, top_lp (P-1, k)
        float32), P = len(prompt), k = the slot's prompt_logprobs setting (at most V).  Row i is prompt position i + 1:
        token_lp[i] is the log-probability of prompt token i + 1 given tokens 0 .. i, top_ids[i] / top_lp[i] the k best ids
        of that row, best first, and theirs, all under the target's raw distribution (T = 1, no processing).  Position 0
        has no value; a prompt of length 1 gives empty arrays.  Refused for a slot whose setting is off and for a slot
        whose current prompt has not had its first verify() yet."""
        if not 0 <= b < self.B:
            raise IndexError(f"slot {b} out of range for a batch of {self.B}")
        n = self.prompt_logprobs_n[b]
        if n is None:
            raise ValueError(f"slot {b} has prompt logprobs off (prompt_logprobs=None)")
        if not self.plp_ready[b]:
            raise ValueError(f"slot {b}: its prompt has not had its first verify() yet")
        P, k = self.prompt_lens[b], min(n, self.V)
        return (self.plp_token[b, 1:P].cpu(), self.plp_ids[b, 1:P, :k].cpu().to(torch.int64),
                self.plp_top[b, 1:P, :k].cpu())
