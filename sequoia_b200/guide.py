"""Token guides for BatchTree's guided decoding (structured output): a token-level automaton per sequence.

A guide is a list of states.  State s allows a set of token ids; committing an allowed id t moves the sequence to the
next state.  A GuideState lists its transitions compactly:
  edges   {id: next state}: explicit transitions (the ids after '{', a node of a choice trie);
  default None, or the next state of every other id in [0, V) except the ids in `banned` (the inside of a JSON string:
          default = itself, the quote ids in edges, control ids banned).
So no state has to list V entries.  The guide consumes the generated tokens only, from position len(prompt) on, and
never ends a sequence itself: a sequence still ends through its end ids (its stop ids in stop mode, 0 and 2 in default
mode), so a guide whose sequences should be able to end allows such an id, for example in an accepting state.

On the device each guided slot holds one int32 blob (include/sequoia_b200.h): a header, default_next, the edges in CSR
form with ascending ids per state, and one allowed bitmask of ceil(V/32) words per state.  The masks dominate its size:
n_states * ceil(V/32) * 4 bytes, 16 KB per state at V = 128256 (64 MB for a guide of SQ_MAX_GUIDE_STATES = 4096
states)."""
from __future__ import annotations

import numbers
from typing import Collection, Dict, List, Mapping, Optional, Sequence

import numpy as np
import torch

from . import _lib

MAX_GUIDE_STATES, MAX_GUIDE_EDGES = _lib.SQ_MAX_GUIDE_STATES, _lib.SQ_MAX_GUIDE_EDGES
GUIDE_HEADER = _lib.SQ_GUIDE_HEADER


def _is_id(t) -> bool:
    return not isinstance(t, bool) and isinstance(t, numbers.Integral) and t >= 0


class GuideState:
    """One state of a TokenGuide.  Its allowed ids are the keys of `edges`, plus, when `default` is not None, every id in
    [0, V) that is not in `banned`.  An allowed id t moves to edges[t] when t is a key, else to `default`.
    Refused with ValueError: an id or a next state that is not an integer >= 0, `banned` without `default`, an id both in
    `banned` and in `edges`, and a state that allows no id (no edges and no default)."""

    __slots__ = ("edges", "default", "banned")

    def __init__(self, edges: Mapping[int, int] = {}, default: Optional[int] = None, banned: Collection[int] = ()):
        if not isinstance(edges, Mapping):
            raise ValueError(f"GuideState: edges must be a mapping {{token id: next state}}, got {edges!r}")
        out: Dict[int, int] = {}
        for t, n in edges.items():
            if not _is_id(t):
                raise ValueError(f"GuideState: {t!r} is not a token id (an integer >= 0)")
            if not _is_id(n):
                raise ValueError(f"GuideState: the next state of {int(t)} must be an integer >= 0, got {n!r}")
            out[int(t)] = int(n)
        if default is not None and not _is_id(default):
            raise ValueError(f"GuideState: default must be None or a state (an integer >= 0), got {default!r}")
        if isinstance(banned, (str, bytes)) or not isinstance(banned, Collection):
            raise ValueError(f"GuideState: banned must be a collection of token ids, got {banned!r}")
        ban = set()
        for t in banned:
            if not _is_id(t):
                raise ValueError(f"GuideState: banned {t!r} is not a token id (an integer >= 0)")
            ban.add(int(t))
        if ban and default is None:
            raise ValueError("GuideState: banned ids need a default (without one only the edges are allowed)")
        both = ban & out.keys()
        if both:
            raise ValueError(f"GuideState: ids both banned and in edges: {sorted(both)[:8]}")
        if not out and default is None:
            raise ValueError("GuideState: a state must allow some id (give it edges or a default)")
        self.edges: Dict[int, int] = dict(sorted(out.items()))
        self.default: Optional[int] = None if default is None else int(default)
        self.banned = frozenset(ban)

    def __repr__(self):
        return f"GuideState(edges={self.edges!r}, default={self.default!r}, banned={sorted(self.banned)!r})"


class TokenGuide:
    """A token automaton: `states` (GuideState, at most SQ_MAX_GUIDE_STATES = 4096 of them, at most SQ_MAX_GUIDE_EDGES =
    2^20 edges in all) and the `start` state.  Refused with ValueError: no states, too many states or edges, an entry that
    is not a GuideState, and a start or a next state outside [0, len(states))."""

    def __init__(self, states: Sequence[GuideState], start: int = 0):
        if isinstance(states, (str, bytes)) or not isinstance(states, Sequence):
            raise ValueError(f"TokenGuide: states must be a sequence of GuideState, got {states!r}")
        states = list(states)
        n = len(states)
        if not 1 <= n <= MAX_GUIDE_STATES:
            raise ValueError(f"TokenGuide: {n} states, must be 1..{MAX_GUIDE_STATES}")
        for s in states:
            if not isinstance(s, GuideState):
                raise ValueError(f"TokenGuide: {s!r} is not a GuideState")
        n_edges = sum(len(s.edges) for s in states)
        if n_edges > MAX_GUIDE_EDGES:
            raise ValueError(f"TokenGuide: {n_edges} edges, at most {MAX_GUIDE_EDGES}")
        if not _is_id(start) or start >= n:
            raise ValueError(f"TokenGuide: start {start!r} is not a state in [0, {n})")
        for i, s in enumerate(states):
            for nx in list(s.edges.values()) + ([] if s.default is None else [s.default]):
                if nx >= n:
                    raise ValueError(f"TokenGuide: state {i} moves to {nx}, outside [0, {n})")
        self.states: List[GuideState] = states
        self.start = int(start)
        self.n_edges = n_edges
        self._packed: Dict[int, torch.Tensor] = {}

    def __len__(self):
        return len(self.states)

    def check(self, V: int, allowed_token_ids: Optional[Collection[int]] = None,
              bad_words: Optional[Sequence[Sequence[int]]] = None):
        """Refuse (ValueError) a guide that does not fit a vocabulary of V ids, or that has a state whose allowed ids,
        within `allowed_token_ids` (None: every id) and without the one-token `bad_words`, are empty: a sequence in it
        could generate nothing."""
        excluded = {w[0] for w in bad_words or () if len(w) == 1}
        allowed = None if allowed_token_ids is None else set(allowed_token_ids)
        for i, s in enumerate(self.states):
            big = [t for t in s.edges if t >= V] + [t for t in s.banned if t >= V]
            if big:
                raise ValueError(f"TokenGuide: state {i} names id {big[0]}, outside [0, {V})")
            if any(t not in excluded and (allowed is None or t in allowed) for t in s.edges):
                continue
            if s.default is not None:
                gone = s.banned | excluded
                if allowed is None:
                    if len(gone) < V:
                        continue
                elif any(t not in gone for t in allowed):
                    continue
            raise ValueError(f"TokenGuide: state {i} allows no id the sequence may generate"
                             + (" (within its allowed_token_ids" if allowed is not None else " (")
                             + (" and without its one-token bad_words)" if excluded else ")"))

    def pack(self, V: int) -> torch.Tensor:
        """The guide's int32 device blob for a vocabulary of V ids, on the host (include/sequoia_b200.h; computed once per
        V).  The guide must fit V (check)."""
        blob = self._packed.get(V)
        if blob is None:
            blob = self._packed[V] = _pack(self, V)
        return blob


def _pack(guide: TokenGuide, V: int) -> torch.Tensor:
    n, W, E = len(guide.states), (V + 31) // 32, guide.n_edges
    default_next = np.array([-1 if s.default is None else s.default for s in guide.states], dtype=np.int32)
    edge_off = np.zeros(n + 1, dtype=np.int32)
    edge_off[1:] = np.cumsum([len(s.edges) for s in guide.states])
    edge_id = np.fromiter((t for s in guide.states for t in s.edges), dtype=np.int32, count=E)
    edge_next = np.fromiter((x for s in guide.states for x in s.edges.values()), dtype=np.int32, count=E)
    full = np.full(W, 0xFFFFFFFF, dtype=np.uint32)
    if V % 32:
        full[-1] = (1 << (V % 32)) - 1
    masks = np.zeros((n, W), dtype=np.uint32)
    for i, s in enumerate(guide.states):
        row = masks[i]
        if s.default is not None:
            row[:] = full
            if s.banned:
                b = np.fromiter(s.banned, dtype=np.int64)
                np.bitwise_and.at(row, b >> 5, ~(np.uint32(1) << (b & 31).astype(np.uint32)))
        if s.edges:
            e = np.fromiter(s.edges, dtype=np.int64)
            np.bitwise_or.at(row, e >> 5, np.uint32(1) << (e & 31).astype(np.uint32))
    header = np.array([n, W, E, V], dtype=np.int32)
    assert header.size == GUIDE_HEADER
    blob = np.concatenate([header, default_next, edge_off, edge_id, edge_next, masks.view(np.int32).ravel()])
    return torch.from_numpy(blob)


def guide_allowed_ids(blob: torch.Tensor, s: int) -> torch.Tensor:
    """Decode a packed blob: the allowed ids of state s, ascending (int64)."""
    n, W, E, V = (int(x) for x in blob[:GUIDE_HEADER])
    off = GUIDE_HEADER + 2 * n + 1 + 2 * E + s * W
    words = blob[off:off + W].numpy().view(np.uint32)
    bits = np.unpackbits(words.view(np.uint8), bitorder="little")[:V]
    return torch.from_numpy(np.nonzero(bits)[0].astype(np.int64))


def guide_next(blob: torch.Tensor, s: int, t: int) -> int:
    """Decode a packed blob: step(s, t) as the device computes it (-1 when t is not allowed in s)."""
    n, W, E, V = (int(x) for x in blob[:GUIDE_HEADER])
    if not (0 <= s < n and 0 <= t < V):
        return -1
    base = GUIDE_HEADER
    word = int(blob[base + 2 * n + 1 + 2 * E + s * W + (t >> 5)]) & 0xFFFFFFFF
    if not (word >> (t & 31)) & 1:
        return -1
    lo, hi = int(blob[base + n + s]), int(blob[base + n + s + 1])
    ids = blob[base + 2 * n + 1 + lo:base + 2 * n + 1 + hi]
    j = int(torch.searchsorted(ids, torch.tensor([t], dtype=torch.int32)))
    if j < hi - lo and int(ids[j]) == t:
        return int(blob[base + 2 * n + 1 + E + lo + j])
    return int(blob[base + s])
