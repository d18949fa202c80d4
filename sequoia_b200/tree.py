"""Sequoia tree speculation (Tree/Tree.py, Tree/SpecTree.py, Tree/GreedyTree.py) re-designed for the GPU.

Same constructor arguments, attributes and return values as the reference classes, but:
  * all per-iteration state (tokens, position ids, prefix length P, accept list) lives on the device; kernels read P
    from a state word, so one CUDA graph drafts the whole tree (construct_grow_map) and one graph runs the target
    forward, the accept/reject walk, both KV compactions and the 1-token draft forward of the bonus token (verify);
  * the tree-causal mask is the growmap's ancestor matrix packed to bits + P (no (2M,2M) fp16 tensor, no copies);
  * a verify step costs exactly one host synchronisation (to return accept_length / terminal as Python values),
    instead of one per tested child (Tree/SpecTree.py:152).
Random numbers follow the reference: r and rand are drawn on the CPU generator per prompt (SpecTree.py:60,84); the
bonus token uses an Exp(1) row drawn by torch on the device and argmax(residual / noise), i.e. torch.multinomial's
own n=1 algorithm (SpecTree.py:222).
"""
from __future__ import annotations

import os
import time
from typing import Dict, List, Optional

import torch

from . import _lib, ops
from .engine import GraphInferenceEngine, GraphInferenceEngineTG

F16 = torch.float16
FP16_MIN = torch.finfo(torch.float16).min


class Tree:
    """Tree/Tree.py:3-48."""

    def __init__(self, device: str = "cpu", max_length=512, dtype=torch.float16) -> None:
        self.tokens = None
        self.Successors: List[List[int]] = []
        self.num_nodes = 0
        self.device = device
        self.max_length = max_length
        self.dtype = dtype

    def initialize(self, attn_mask, sequence, new_tokens_buffer, parents_buffer, position_ids, active_mark):
        # The reference repeats the caller's (M,M) buffer into a (2M,2M) mask here (Tree.py:13-20); the kernels use
        # the packed tree mask instead, so the buffers are only kept for API compatibility.
        self.sequence = sequence
        self.new_tokens_buffer = new_tokens_buffer
        self.parents_buffer = parents_buffer
        self.active_mark = active_mark
        self._caller_attn_mask = attn_mask
        self._caller_position_ids = position_ids

    def verbose(self):
        print(self.tokens)
        print(self.Successors)


def pack_tree_mask(mask01: torch.Tensor) -> torch.Tensor:
    """(S,S) 0/1 ancestor-or-self matrix -> (S, ceil(S/32)) int32 words, bit j%32 of word j//32 = mask[i, j]."""
    S = mask01.shape[0]
    W = (S + 31) // 32
    m = torch.zeros(S, W * 32, dtype=torch.int64)
    m[:, :S] = (mask01 != 0).to(torch.int64)
    weights = (1 << torch.arange(32, dtype=torch.int64))
    words = (m.view(S, W, 32) * weights).sum(-1)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words)
    return words.to(torch.int32).contiguous()


class _Static:
    """Device-side tables of one growmap (Tree/SpecTree.py:39-48,62; tests/testbed.py:258-285)."""

    def __init__(self, grow_map: dict, device):
        self.S = S = int(grow_map["size"])
        roots, branches, succ = grow_map["roots"], grow_map["branches"], grow_map["Successors"]
        self.draft_step = len(roots)
        self.levels = []
        next_node = 1
        i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=device)
        for i in range(self.draft_step - 1):
            nb = [int(b) for b in branches[i]]
            parents = [int(x) for x in roots[i]]
            first = []
            for p, b in zip(parents, nb):
                first.append(next_node if b > 0 else 0)
                if b > 0:
                    assert list(succ[p]) == list(range(next_node, next_node + b)), "growmap children must be contiguous"
                next_node += b
            total = sum(nb)
            self.levels.append(dict(n0=next_node - total, tb=total, k=max(nb), n_parents=len(parents),
                                    parents=i32(parents), first=i32(first), nb=i32(nb)))
        assert next_node == S, (next_node, S)
        off = [0]
        flat: List[int] = []
        for k in range(S):
            flat.extend(int(c) for c in succ[k])
            off.append(len(flat))
        self.succ_off, self.succ = i32(off), i32(flat if flat else [0])
        depth = grow_map["depth"].to(torch.int64)
        self.depth_cpu = depth.clone()
        self.depth = depth.to(torch.int32).to(device)
        self.max_depth = int(depth.max())
        bits = pack_tree_mask(grow_map["mask"])
        self.tree_words = bits.shape[1]
        self.tree_bits = bits.to(device)
        self.mask01 = grow_map["mask"]


POLICIES = ("spec", "greedy", "greedys", "specinfer", "spec_test")


class _Runtime:
    """Static buffers + captured graphs for one (draft engine, target engine, growmap, policy) combination.
    Lives across prompts (the reference likewise captures its graphs once and reuses them, tests/testbed.py:256-285)."""

    def __init__(self, draft: GraphInferenceEngine, target: GraphInferenceEngineTG, grow_map: dict, policy: str,
                 T: float, top_p: float, M: int, max_target_seq: int, V: int, device):
        assert policy in POLICIES
        self.draft, self.target, self.grow_map = draft, target, grow_map
        self.policy = policy
        self.greedy = policy in ("greedy", "greedys")          # top-k drafting + token-match walk
        self.T, self.top_p, self.M, self.max_target_seq, self.V = float(T), float(top_p), M, max_target_seq, V
        self.device = torch.device(device)
        dev = self.device
        self.st = _Static(grow_map, dev)
        S = self.st.S
        self.tokens = torch.zeros(M, dtype=torch.int64, device=dev)
        self.position_ids = torch.zeros(M, dtype=torch.int64, device=dev)
        self.storage_ids = torch.arange(M, dtype=torch.int64, device=dev)
        self.draft_logits = torch.zeros((M, V), dtype=F16, device=dev)
        self.target_logits = torch.zeros((S, V), dtype=F16, device=dev)
        self.rand = torch.zeros((S, V), dtype=F16, device=dev)
        self.r = torch.zeros(M, dtype=F16, device=dev)
        self.noise = torch.ones(V, dtype=F16, device=dev)
        self.target_token = torch.zeros(S, dtype=torch.int64, device=dev)
        self.accept_idx = torch.zeros(max(S, 8), dtype=torch.int32, device=dev)
        self.state = torch.zeros(16, dtype=torch.int32, device=dev)
        self.host_state = torch.zeros(16, dtype=torch.int32).pin_memory()
        self.graphs: Dict[str, torch.cuda.CUDAGraph] = {}
        self.graph_launches: Dict[str, int] = {}
        self.replays: Dict[str, int] = {}
        self.use_graphs = True
        self.external_noise: Optional[torch.Tensor] = None   # tests: (n_iter, V) Exp(1) rows shared with the oracle
        # policy variants (SURVEY.md 8f.3)
        self.tuniform = torch.zeros((S, V), dtype=F16, device=dev) if policy == "greedys" else None
        self.external_tuniform: Optional[torch.Tensor] = None   # tests: (n_iter, S, V) uniforms shared with the oracle
        self.words = torch.zeros(S, dtype=torch.int64, device=dev) if policy == "specinfer" else None
        self.external_words: Optional[torch.Tensor] = None      # tests: (n_iter, S) int64 words in [0, 2^32)
        self.iter = 0

    # ---- the op sequences (captured into graphs, or run eagerly in benchmark mode) --------------------------------
    def _mask_kw(self):
        return dict(tree_bits=self.st.tree_bits, tree_words=self.st.tree_words, tree_size=self.st.S)

    def op_sample(self, i: int):
        lv = self.st.levels[i]
        if self.policy == "specinfer":                 # SpecInferTree.py:100-105: i.i.d. children, with replacement
            if i == 0 and self.external_words is None:
                self.words.random_(0, 1 << 32)         # one fresh uniform word per tree node and iteration
            ops.sample_replace(self.draft_logits, self.words, lv["n_parents"], lv["k"], self.T,
                               parent_rows=lv["parents"], child_first=lv["first"], n_branch=lv["nb"],
                               tokens=self.tokens, state=self.state)
            return
        ops.sample_level(self.draft_logits, None if self.greedy else self.rand, lv["n_parents"], lv["k"], self.T,
                         1 if self.greedy else 0, parent_rows=lv["parents"], child_first=lv["first"], n_branch=lv["nb"],
                         tokens=self.tokens, state=self.state)

    def op_draft_level(self, i: int):
        lv = self.st.levels[i]
        n0, tb = lv["n0"], lv["tb"]
        self.draft.engine.runner.forward(tb, self.tokens, self.position_ids, self.storage_ids, state=self.state, n0=n0,
                                         kv_end=n0 + tb, logits_out=self.draft_logits[n0:n0 + tb], **self._mask_kw())

    @property
    def tp(self):
        """TPDriver when the target is tensor-parallel over several ranks (sequoia_b200.tp), else None."""
        return getattr(self.target, "_tp_driver", None)

    def op_target_steady(self):
        S = self.st.S
        if self.tp is not None:
            self.tp.bcast_inputs(self)
        self.target.engine.runner.forward(S, self.tokens, self.position_ids, self.storage_ids, state=self.state, n0=0,
                                          kv_end=S, logits_out=self.target_logits, **self._mask_kw())

    def op_target_first(self, start: int, P: int):
        """First verify of a prompt (Tree/SpecTree.py:164-176): rows [start, P+S-1) in absolute addressing."""
        S = self.st.S
        end = P + S - 1
        n = end - start
        if self.tp is not None:
            self.tp.bcast_inputs(self)
        self.target.engine.runner.forward(n, self.tokens, self.position_ids, self.storage_ids, state=None, n0=start,
                                          kv_end=end, prefix_len=P, logits_out=self.target_logits, logits_from=n - S,
                                          **self._mask_kw())

    def op_accept(self):
        st = self.st
        if self.greedy:
            if self.policy == "greedys":                                                # GreedySTree.py:188-190
                if self.top_p < 1.0:
                    ops.top_p_filter_(self.target_logits, self.top_p, self.T)
                if self.external_tuniform is None:
                    self.tuniform.uniform_()
                # softmax(l/T).multinomial(1) per row == the k=1 exponential race of sampling_without_replacement
                ops.sample_level(self.target_logits, self.tuniform, st.S, 1, self.T, 0, positions=self.target_token)
            else:
                ops.argmax_rows(self.target_logits, self.target_token)                  # GreedyTree.py:186
            ops.accept_greedy(self.target_token, st.succ_off, st.succ, st.depth, st.S, self.tokens, self.position_ids,
                              self.accept_idx, self.state, self.max_target_seq)
        else:
            if self.top_p < 1.0:                                                        # utils.py:65-77 (off at P=1)
                ops.top_p_filter_(self.target_logits, self.top_p, self.T)
            if self.external_noise is None:
                self.noise.exponential_(1.0)                                            # torch.multinomial's draw
            ops.accept_stochastic(self.target_logits, self.draft_logits, self.r, self.noise, st.succ_off, st.succ,
                                  st.depth, st.S, self.T, self.tokens, self.position_ids, self.accept_idx, self.state,
                                  self.max_target_seq,
                                  policy={"specinfer": ops.ACCEPT_GE | ops.ACCEPT_KEEP_Q,
                                          "spec_test": ops.ACCEPT_GE}.get(self.policy, 0))

    def op_kv_gather(self):
        md = max(self.st.max_depth, 1)
        if self.tp is not None:
            self.tp.bcast_accept(self)
        self.draft.engine.kv_cache.gather_from_state(self.accept_idx, self.state, md)   # SpecTree.py:226-227
        self.target.engine.kv_cache.gather_from_state(self.accept_idx, self.state, md)

    def op_bonus_forward(self):
        """prepare_for_next_iter's 1-token draft forward (SpecTree.py:274-277): the bonus token is node 0 of the new P."""
        self.draft.engine.runner.forward(1, self.tokens, self.position_ids, self.storage_ids, state=self.state, n0=0,
                                         kv_end=1, logits_out=self.draft_logits[0:1], **self._mask_kw())

    def op_publish(self):
        self.host_state.copy_(self.state, non_blocking=True)

    def seq_draft(self):
        for i in range(self.st.draft_step - 1):
            self.op_sample(i)
            self.op_draft_level(i)

    def seq_post(self):
        self.op_accept()
        self.op_kv_gather()
        self.op_bonus_forward()
        self.op_publish()

    def seq_steady(self):
        self.op_target_steady()
        self.seq_post()

    # ---- graph management -----------------------------------------------------------------------------------------
    def run(self, name: str, fn):
        if not self.use_graphs:
            fn()
            return
        g = self.graphs.get(name)
        if g is None:
            g = self._capture(name, fn)
        g.replay()
        self.replays[name] = self.replays.get(name, 0) + 1

    def _capture(self, name: str, fn):
        # Warm-up on a side stream (cuBLAS handles / workspaces), restoring every buffer the sequence mutates so that
        # capture does not change the decode state.
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
        self._restore(snap)          # capture executes nothing, but keep the invariant explicit
        self.graphs[name] = g
        return g

    def _snapshot(self):
        dk, tk = self.draft.engine.kv_cache, self.target.engine.kv_cache
        return dict(tokens=self.tokens.clone(), pos=self.position_ids.clone(), state=self.state.clone(),
                    dl=self.draft_logits[:self.st.S].clone(), tl=self.target_logits.clone(),
                    dk=dk.k_cache.clone(), dv=dk.v_cache.clone(), tk=tk.k_cache.clone(), tv=tk.v_cache.clone(),
                    rng=torch.cuda.get_rng_state(self.device))

    def _restore(self, s):
        dk, tk = self.draft.engine.kv_cache, self.target.engine.kv_cache
        self.tokens.copy_(s["tokens"]); self.position_ids.copy_(s["pos"]); self.state.copy_(s["state"])
        self.draft_logits[:self.st.S].copy_(s["dl"]); self.target_logits.copy_(s["tl"])
        dk.k_cache.copy_(s["dk"]); dk.v_cache.copy_(s["dv"]); tk.k_cache.copy_(s["tk"]); tk.v_cache.copy_(s["tv"])
        torch.cuda.set_rng_state(s["rng"], self.device)

    def kernel_launches(self) -> int:
        """Kernels of libsequoia_b200.so launched through graph replays so far (for bench.py's gpu_launches)."""
        return sum(self.graph_launches.get(k, 0) * v for k, v in self.replays.items())


_RUNTIMES: Dict[tuple, _Runtime] = {}


SMALL_VOCAB = 32768       # largest vocabulary of the single-CTA kernels (sampling with replacement, SQ_ACCEPT_IMPL=0)
MAX_VOCAB = 131072        # largest vocabulary of the cluster kernels (the default decode path)


def check_vocab(policy: str, V: int):
    """Refuse, before any buffer is allocated, a vocabulary the policy's kernels cannot take."""
    if V > MAX_VOCAB or V % 8:
        raise ValueError(f"vocabulary {V}: the kernels take multiples of 8 up to {MAX_VOCAB}")
    if V <= SMALL_VOCAB:
        return
    if policy == "specinfer":
        raise ValueError(f"SpecInferTree supports vocabularies up to {SMALL_VOCAB} (sampling with replacement has no "
                         f"large-vocabulary kernel); this model has {V}")
    if policy in ("spec", "spec_test", "specinfer") and os.environ.get("SQ_ACCEPT_IMPL", "1") == "0":
        raise ValueError(f"SQ_ACCEPT_IMPL=0 (the single-CTA verification walk) supports vocabularies up to {SMALL_VOCAB}; "
                         f"this model has {V}")


def get_runtime(draft, target, grow_map, policy, T, top_p, M, max_target_seq, V, device) -> _Runtime:
    key = (id(draft), id(target), id(grow_map), policy, float(T), float(top_p), M, max_target_seq, V)
    rt = _RUNTIMES.get(key)
    if rt is None or rt.grow_map is not grow_map:
        rt = _Runtime(draft, target, grow_map, policy, T, top_p, M, max_target_seq, V, device)
        _RUNTIMES[key] = rt
    return rt


def clear_runtimes():
    _RUNTIMES.clear()


class _TreeBase(Tree):
    GREEDY = False          # top-k drafting, no random buffers (GreedyTree / GreedySTree)
    POLICY = "spec"

    def __init__(self, draft_model_engine: GraphInferenceEngine, target_model_engine: GraphInferenceEngineTG,
                 prefix: torch.LongTensor, temperature: float = 0.6, top_p: float = 0.9, draft_kv_len=0,
                 target_kv_len=0, max_length=256, device: str = "cpu", max_target_seq=256, vocab_size=32000,
                 grow_map=None, attn_mask=None, sequence=None, new_tokens_buffer=None, parents_buffer=None,
                 position_ids=None, residual_graph=None, sampling_callables=None, sample_gather_indices=None) -> None:
        super().__init__(device=device, max_length=max_length)
        assert self.max_length == draft_model_engine.engine.max_length
        if not str(device).startswith("cuda"):
            raise RuntimeError("sequoia_b200 trees run on a CUDA device only (there is no CPU path)")
        self.max_target_seq = max_target_seq
        self.draft_model_engine = draft_model_engine
        self.target_model_engine = target_model_engine
        self.temperature = temperature
        self.top_p = top_p
        # accepted for signature compatibility; the fused kernels replace these callables (utils.cuda_graph_for_*)
        self.residual_graph = residual_graph
        self.sampling_callables = sampling_callables
        self.sample_gather_indices = sample_gather_indices
        self.grow_map = grow_map
        # the buffers are sized by the engines' vocabulary (`vocab_size` is the reference's signature; 32000 = not given)
        V = draft_model_engine.engine.model_config.vocab_size
        if vocab_size not in (32000, V):
            raise ValueError(f"vocab_size={vocab_size} does not match the engines' vocabulary ({V})")
        check_vocab(self.POLICY, V)
        self.draft_step = len(grow_map["roots"])
        self.Successors = grow_map["Successors"]
        self.tree_size = grow_map["size"]
        self.initialize(attn_mask, sequence, new_tokens_buffer, parents_buffer, position_ids, None)
        rt = get_runtime(draft_model_engine, target_model_engine, grow_map, self.POLICY, temperature, top_p,
                         max_length, max_target_seq, V, device)
        self.rt = rt
        S, M = self.tree_size, max_length
        P = len(prefix)
        assert P + S - 1 <= M, "max_length must hold prefix + tree (README.md:47)"
        # Tree.set_prefix (Tree.py:21-27) + SpecTree.__init__ (:60-66)
        self.tokens = rt.tokens
        self.position_ids = rt.position_ids
        self.storage_ids = rt.storage_ids
        self.draft_logits = rt.draft_logits
        prefix_dev = prefix.to(self.device).clone()    # `prefix` may be a view of rt.tokens (a previous verify's valid_tokens)
        self.tokens.zero_()
        self.tokens[:P] = prefix_dev
        self.num_nodes = P
        self.ground_truth_len = P
        if not self.GREEDY:
            self.r = torch.rand(len(position_ids) if position_ids is not None else M, dtype=self.dtype)   # CPU draw
            rt.r[:min(M, self.r.numel())].copy_(self.r[:M])
            self.r = rt.r
        pos = torch.zeros(M, dtype=torch.int64)
        pos[:P] = torch.arange(P)
        pos[P:P + S - 1] = rt.st.depth_cpu[1:] + P - 1
        self.position_ids.copy_(pos)
        self.depth = rt.st.depth[1:]
        st0 = torch.zeros(16, dtype=torch.int32)
        st0[0] = P
        st0[8] = M                     # SQ_ST_M: the accept kernels bound their epilogue writes by the buffer length
        rt.state.copy_(st0)
        self._exhausted = False
        rt.iter = 0
        # draft prefill (SpecTree.py:67-80): eager, causal rows [draft_kv_len, P)
        start = draft_kv_len
        n = P - start
        dr = draft_model_engine.engine.runner
        dr.forward(n, self.tokens, self.position_ids, self.storage_ids, state=None, n0=start, kv_end=P, prefix_len=P,
                   logits_out=self.draft_logits[0:1], logits_from=n - 1)
        draft_model_engine.engine.kv_cache.kv_offset = P
        self.draft_kv_len = P
        self.target_kv_len = target_kv_len
        if not self.GREEDY:
            self.rand = torch.empty((S, self.draft_logits.shape[1]), dtype=self.dtype).uniform_()           # CPU draw
            rt.rand.copy_(self.rand)
            self.rand = rt.rand
        self.seq_to_use = list(range(self.max_length))

    # ---- reference-visible helpers ---------------------------------------------------------------------------------
    @property
    def attn_mask(self) -> torch.Tensor:
        """The (M,M) additive window the reference materialises (SpecTree.py:57-58,270-271), rebuilt on demand from
        the packed rule -- only for inspection / tests; no kernel reads it."""
        M, S, P = self.max_length, self.tree_size, self.ground_truth_len
        tot = P + S - 1
        m01 = self.rt.st.mask01
        r = torch.arange(M).view(-1, 1)
        c = torch.arange(M).view(1, -1)
        vis = (c <= torch.minimum(r, torch.tensor(P - 1))) & (r < tot)
        node_r = (r - (P - 1)).clamp(min=0, max=S - 1)
        node_c = (c - (P - 1)).clamp(min=0, max=S - 1)
        tree = m01.bool()[node_r.expand(M, M), node_c.expand(M, M)]
        vis = vis | ((r >= P) & (r < tot) & (c >= P - 1) & (c < tot) & tree)
        out = torch.full((M, M), FP16_MIN, dtype=F16)
        out[vis] = 0
        return out.to(self.device)

    @property
    def target_logits(self):
        return self.rt.target_logits

    # ---- drafting (Tree/SpecTree.py:88-134,245-259) ---------------------------------------------------------------
    @torch.inference_mode()
    def collective_grow_static(self, idx_list, n_branch_list, benchmark=False, grow_step=None):
        rt = self.rt
        x1 = x2 = 0.0
        if benchmark:
            torch.cuda.synchronize()
            t1 = time.time()
        rt.op_sample(grow_step)
        if benchmark:
            torch.cuda.synchronize()
            t2 = time.time()
            x1 = t2 - t1
        rt.op_draft_level(grow_step)
        total_branch = sum(n_branch_list)
        self.num_nodes += total_branch
        self.draft_kv_len = self.num_nodes
        self.draft_model_engine.engine.kv_cache.kv_offset = self.num_nodes
        if benchmark:
            torch.cuda.synchronize()
            x2 = time.time() - t2
            return n_branch_list, x1, x2
        return n_branch_list

    def _check_room(self):
        """The reference fails with an IndexError / shape error once prefix + tree no longer fit the M-long buffers
        (SpecTree.py:222,266); the device-side walk refuses to overrun them and flags ST_SKIPPED instead, so the next
        drafting step has nowhere to put its tree: raise here."""
        if self._exhausted or self.ground_truth_len + self.tree_size - 1 > self.max_length:
            raise RuntimeError(f"max_length={self.max_length} exhausted: sequence {self.ground_truth_len} + tree "
                               f"{self.tree_size} - 1 does not fit (README.md:47: M >= tree_size + max_target_seq)")

    def construct_grow_map(self, benchmark=False):
        rt = self.rt
        if benchmark:
            self._check_room()
            sample_time = compute_time = 0.0
            for i in range(self.draft_step - 1):
                _, t1, t2 = self.collective_grow_static(None, self.grow_map["branches"][i], benchmark=True, grow_step=i)
                sample_time += t1
                compute_time += t2
            return sample_time, compute_time
        self._check_room()
        if rt.external_words is not None and rt.words is not None:
            rt.words.copy_(rt.external_words[rt.iter])
        with torch.inference_mode():
            rt.run("draft", rt.seq_draft)
        self.num_nodes = self.ground_truth_len + self.tree_size - 1
        self.draft_kv_len = self.num_nodes
        self.draft_model_engine.engine.kv_cache.kv_offset = self.num_nodes
        return None

    # ---- verification (Tree/SpecTree.py:160-242, GreedyTree.py:151-223) ---------------------------------------------
    @torch.inference_mode()
    def verify(self, benchmark=False):
        rt = self.rt
        P, S = self.ground_truth_len, self.tree_size
        assert self.num_nodes == P + S - 1, "construct_grow_map() must run before verify()"
        steady = (self.target_kv_len == P - 1)
        if rt.external_noise is not None and not self.GREEDY:
            rt.noise.copy_(rt.external_noise[rt.iter])
        if rt.external_tuniform is not None and rt.tuniform is not None:
            rt.tuniform.copy_(rt.external_tuniform[rt.iter])
        if benchmark:
            torch.cuda.synchronize()
            t1 = time.time()
            if rt.tp is not None:
                rt.tp.send_ctrl(1 if steady else 2, self.target_kv_len, P, mode=1)      # MODE_EAGER: one execution
            if steady:
                rt.op_target_steady()
            else:
                rt.op_target_first(self.target_kv_len, P)
            torch.cuda.synchronize()
            t2 = time.time()
            rt.op_accept()
            torch.cuda.synchronize()
            t3 = time.time()
            rt.op_kv_gather()
            torch.cuda.synchronize()
            t4 = time.time()
            rt.op_bonus_forward()
            rt.op_publish()
        elif steady:
            if rt.tp is not None:                        # OP_STEADY + how this rank is about to execute it (tp.MODE_*)
                rt.tp.send_ctrl(1, mode=1 if not rt.use_graphs else (2 if "steady" not in rt.graphs else 0))
            rt.run("steady", rt.seq_steady)
        else:
            if rt.tp is not None:
                rt.tp.send_ctrl(2, self.target_kv_len, P)   # OP_FIRST; its post-processing stays eager so that the
                rt.op_target_first(self.target_kv_len, P)    # follower ranks see each collective exactly once
                rt.seq_post()
            else:
                rt.op_target_first(self.target_kv_len, P)
                rt.run("post", rt.seq_post)
        torch.cuda.current_stream().synchronize()       # the one host sync of a verify step
        rt.iter += 1
        hs = rt.host_state
        a, terminal = int(hs[1]), bool(hs[2])
        skipped = bool(hs[7])
        accept_length = a
        dkv, tkv = self.draft_model_engine.engine.kv_cache, self.target_model_engine.engine.kv_cache
        dkv.kv_offset = a
        tkv.kv_offset = a
        self.last_accept_len = a
        if not terminal:
            valid = self.tokens[:accept_length + 1]
            if not skipped:                             # prepare_for_next_iter ran on the device (SpecTree.py:261-281)
                self.ground_truth_len = a + 1
                self.num_nodes = a + 1
                self.draft_kv_len = a + 1
                self.target_kv_len = a
                dkv.kv_offset = a + 1
            else:
                self._exhausted = True
                valid = self.tokens[:min(accept_length + 1, self.max_length)]
        else:
            valid = self.tokens[:accept_length]
        if benchmark:
            return valid, accept_length, accept_length, t2 - t1, t3 - t2, t4 - t3, terminal
        return valid, accept_length, accept_length, terminal

    def accept_list(self) -> List[int]:
        """accept_list of the last verify (absolute slots), reconstructed from the device record."""
        hs = self.rt.host_state
        P_old, n_new = int(hs[4]), int(hs[3])
        return list(range(P_old)) + [int(x) for x in self.rt.accept_idx[:n_new].tolist()]

    def verbose(self):
        super().verbose()


class SpecTree(_TreeBase):
    """Tree/SpecTree.py:7-281 (stochastic Sequoia tree: sampling without replacement + residual verification)."""
    GREEDY = False
    POLICY = "spec"


class GreedyTree(_TreeBase):
    """Tree/GreedyTree.py:6-264 (top-k drafting, argmax verification)."""
    GREEDY = True
    POLICY = "greedy"


class GreedySTree(_TreeBase):
    """Tree/GreedySTree.py (top-k drafting verified against a target token SAMPLED from softmax(top_p(logits)/T),
    :188-190): the k=1 exponential race of `sq_sample_level` over the S target rows replaces the row argmax."""
    GREEDY = True
    POLICY = "greedys"


class SpecInferTree(_TreeBase):
    """Tree/SpecInferTree.py (the SpecInfer baseline policy on the same tree machinery): children drawn i.i.d. with
    replacement (`sq_sample_replace`), walk accepts on >= and never masks q (`sq_accept_stochastic` policy bits)."""
    GREEDY = False
    POLICY = "specinfer"


# ---- acceptance-rate measurement trees (Tree/SpecTree.py:284-483 SpecTreeTest, Tree/GreedyTree.py:264-456 GreedyTreeTest) ----
_STARS: Dict[int, dict] = {}


def star_grow_map(width: int) -> dict:
    """Root + `width` children: the one-level tree the reference's *TreeTest classes hard-code (`Successors =
    [list(range(1, W+1))] + [[]]*W`, SpecTree.py:312-313), as a growmap so that the same kernels / graphs serve it."""
    gm = _STARS.get(width)
    if gm is None:
        S = width + 1
        mask = torch.eye(S, dtype=torch.long)
        mask[:, 0] = 1
        gm = {"roots": [[0], list(range(1, S))], "branches": [[width], [0] * width],
              "Successors": [list(range(1, S))] + [[] for _ in range(width)], "mask": mask,
              "depth": torch.LongTensor([0] + [1] * width), "size": S}
        _STARS[width] = gm
    return gm


class _StarTest(_TreeBase):
    """One decode step of the acceptance-rate experiment (tests/test_accept.py:36-86): draft `max_width` children of the
    last committed token, verify, report WHICH child (rank b, or -1) was accepted.  Like the reference, a new object is
    built per step with the KV lengths the previous verify returned; its constructor already drafts the children."""

    def __init__(self, draft_model_engine, target_model_engine, prefix, temperature: float = 0.6, top_p: float = 0.9,
                 draft_kv_len=0, target_kv_len=0, max_length=256, max_width=32, device: str = "cpu", grow_map=None,
                 attn_mask=None, sequence=None, new_tokens_buffer=None, parents_buffer=None, position_ids=None) -> None:
        self.max_width = max_width
        super().__init__(draft_model_engine, target_model_engine, prefix, temperature=temperature, top_p=top_p,
                         draft_kv_len=draft_kv_len, target_kv_len=target_kv_len, max_length=max_length, device=device,
                         max_target_seq=max_length, vocab_size=draft_model_engine.engine.model_config.vocab_size,
                         grow_map=star_grow_map(max_width), attn_mask=attn_mask, sequence=sequence,
                         new_tokens_buffer=new_tokens_buffer, parents_buffer=parents_buffer, position_ids=position_ids)
        self.construct_grow_map()                       # SpecTree.py:342 / GreedyTree.py:322

    @torch.inference_mode()
    def verify(self, benchmark=False):
        """-> (valid_tokens, len(accept_list), len(accept_list), b, terminal)   (SpecTree.py:470-479)"""
        valid, a, _, terminal = super().verify(benchmark=False)
        hs = self.rt.host_state
        n_new, P_old = int(hs[3]), int(hs[4])
        b = int(self.rt.accept_idx[0]) - (P_old - 1) - 1 if n_new > 0 else -1     # successor order of the accepted child
        return valid, a, a, b, terminal


class SpecTreeTest(_StarTest):
    """Tree/SpecTree.py:284-483: children by sampling without replacement, accept on >= with the rejected token masked
    out of q.  Same estimator as the reference; arithmetic is the SpecTree kernels' fp16 chain (the reference's Test
    class happens to hold r / rand in fp32)."""
    GREEDY = False
    POLICY = "spec_test"


class GreedyTreeTest(_StarTest):
    """Tree/GreedyTree.py:264-456: top-`max_width` children, accept the one equal to the target's argmax."""
    GREEDY = True
    POLICY = "greedy"
