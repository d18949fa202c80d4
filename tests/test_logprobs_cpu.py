"""Host-side pieces of the per-sequence logprobs that need no GPU: the CPU statement (oracle/logprobs.py) against a
brute-force sort and log-softmax in Python floats, its row mapping against hand-walked paths, the refusals of
check_logprobs, ops.token_logprobs_batch_ and the C entry point, the device values a tree keeps per slot through
admissions, and testbed.py's --logprobs flag."""
import math

import numpy as np
import pytest
import torch

import cases
from oracle import logprobs as L
from test_stop_cpu import _cpu_tree

F16 = torch.float16
GM128 = "A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"   # config 2: 128 nodes
NAN, INF = float("nan"), float("inf")


def _brute(row, token, T, greedy, n):
    """One row in Python: each scaled value through numpy's fp16 one element at a time, the ranking by sorted() on
    (NaN first, value descending with -0 == +0, index), the log-softmax with math.fsum."""
    xs = [float(v) for v in row]
    inv = np.float32(1.0) if greedy else np.float32(1.0) / np.float32(T)
    with np.errstate(over="ignore", invalid="ignore"):
        s = [float(np.float16(np.float32(x) * inv)) for x in xs]
    finite_max = not any(math.isnan(v) or v == INF for v in s) and max(s) > -INF
    if finite_max:
        m = max(s)
        lse = m + math.log(math.fsum(math.exp(v - m) for v in s))
        lp = [v - lse for v in s]
    else:
        lp = [NAN] * len(s)
    order = sorted(range(len(xs)), key=lambda i: (0 if math.isnan(xs[i]) else 1,
                                                  0.0 if math.isnan(xs[i]) else -(xs[i] + 0.0), i))
    ids = order[:min(n, len(xs))]
    return lp[token], ids, [lp[i] for i in ids]


def _rows(V=96):
    g = torch.Generator().manual_seed(3)
    base = (torch.randn(V, generator=g) * 3).to(F16)
    ties = base.clone()
    ties[10:30] = 1.5                                   # a tie group across the top-n boundary
    ties[40], ties[41], ties[42] = 0.0, -0.0, 0.0       # -0 ranks with +0, by index
    runs = base.clone()
    runs[::2] = -INF                                    # filtered entries
    runs[5] = 7.0
    big = base.clone()
    big[7] = 4000.0                                     # scaled by 1 / 0.05 it overflows fp16: NaN row at T = 0.05
    pinf, nan = base.clone(), base.clone()
    pinf[9] = INF
    nan[11] = NAN
    all_ninf = torch.full((V,), -INF, dtype=F16)
    few = torch.full((V,), -INF, dtype=F16)
    few[[3, 50, 90]] = torch.tensor([1.0, 2.0, 1.0], dtype=F16)   # three survivors, the rest -inf ties by index
    return dict(base=base, ties=ties, runs=runs, big=big, pinf=pinf, nan=nan, all_ninf=all_ninf, few=few)


def _same(a, b, tol=1e-9):
    return (math.isnan(a) and math.isnan(b)) or a == b or abs(a - b) <= tol * (1 + abs(a))


@pytest.mark.parametrize("T", [0.05, 0.6, 1.0, 2.0])
@pytest.mark.parametrize("greedy", [False, True])
def test_oracle_matches_brute_force(T, greedy):
    for name, row in _rows().items():
        for token in (0, 5, 11, 40, 41, 95):
            for n in (0, 1, 5, 20):
                got = L.row_logprobs(row, token, T, greedy, n)
                want = _brute(row, token, T, greedy, n)
                assert got[1] == want[1], (name, n)
                assert _same(got[0], want[0]), (name, token, got[0], want[0])
                assert all(_same(a, b) for a, b in zip(got[2], want[2])), (name, got[2], want[2])


def test_oracle_row_rules():
    rows = _rows()
    tok, ids, top = L.row_logprobs(rows["runs"], 0, 1.0, False, 20)
    assert tok == -INF and ids[0] == 5 and math.isfinite(top[0])
    assert all(a >= b for a, b in zip(top, top[1:])), "non-increasing down the list"
    for name in ("pinf", "nan", "all_ninf"):
        tok, ids, top = L.row_logprobs(rows[name], 1, 0.6, False, 5)
        assert math.isnan(tok) and all(math.isnan(v) for v in top), name
    assert L.row_logprobs(rows["nan"], 0, 1.0, False, 1)[1] == [11], "NaN ranks first"
    assert L.row_logprobs(rows["pinf"], 0, 1.0, False, 1)[1] == [9]
    assert math.isnan(L.row_logprobs(rows["big"], 0, 0.05, False, 0)[0])
    assert math.isfinite(L.row_logprobs(rows["big"], 0, 0.05, True, 0)[0]), "greedy reads T as 1"
    _, ids, top = L.row_logprobs(rows["few"], 50, 1.0, False, 6)
    assert ids == [50, 3, 90, 0, 1, 2] and top[3:] == [-INF] * 3
    _, ids, _ = L.row_logprobs(rows["ties"], 0, 1.0, False, 20)
    assert ids[:20] == sorted(ids[:20], key=lambda i: (-float(rows["ties"][i]), i))
    assert L.row_logprobs(torch.zeros(8, dtype=F16), 0, 1.0, False, 20)[1] == list(range(8)), "n is capped at V"
    # the ids do not depend on T; with T = 1 the values are the fp16 row's own log-softmax
    assert L.row_logprobs(rows["base"], 0, 0.6, False, 20)[1] == L.row_logprobs(rows["base"], 0, 2.0, False, 20)[1]
    want = torch.log_softmax(rows["base"].double(), -1)
    assert abs(L.row_logprobs(rows["base"], 17, 1.0, False, 0)[0] - float(want[17])) < 1e-12


def _walk(gm, depth, pick):
    """A hand-walked path of `depth` nodes below the root: at each node the pick-th child (clamped)."""
    succ, node, path = gm["Successors"], 0, []
    for _ in range(depth):
        kids = list(succ[node])
        if not kids:
            break
        node = int(kids[min(pick, len(kids) - 1)])
        path.append(node)
    return path


def _state(P, n_new, terminal=0, M=512, frozen=0):
    st = torch.zeros(16, dtype=torch.int32)
    st[L.ST_P_OLD], st[L.ST_N_NEW], st[L.ST_TERMINAL], st[L.ST_M], st[L.ST_FROZEN] = P, n_new, terminal, M, frozen
    return st


@pytest.mark.parametrize("name", [GM128, "L40_growmaps/16-chain.pt", "L40_growmaps/128x1-tree.pt"])
def test_row_mapping_of_hand_walked_paths(name):
    gm = cases.load_growmap(name)
    P = 40
    for pick in (0, 1, 3):
        path = _walk(gm, int(gm["depth"].max()), pick)
        for n_new in range(len(path) + 1):
            acc = torch.tensor([P - 1 + k for k in path[:n_new]] + [0] * 8, dtype=torch.int32)
            st = _state(P, n_new)
            assert L.committed(st, 512) == n_new + 1
            assert [L.path_node(st, acc, j) for j in range(n_new + 1)] == [0] + path[:n_new]
            for j in range(1, n_new + 1):
                assert L.is_bonus_replacement(st, acc, j) == (path[j - 1] == n_new + 1)
    if name == "L40_growmaps/128x1-tree.pt":               # node 2 accepted alone sits at slot P + 1 = a
        acc = torch.tensor([P + 1] + [0] * 7, dtype=torch.int32)
        st = _state(P, 1)
        assert L.path_node(st, acc, 1) == 2 and L.is_bonus_replacement(st, acc, 1)
    if name == "L40_growmaps/16-chain.pt":                 # a chain never commits the bonus over an accepted node
        path = _walk(gm, 15, 0)
        assert path == list(range(1, 16))
        assert not any(L.is_bonus_replacement(_state(P, n), torch.tensor([P - 1 + k for k in path[:n]] + [0] * 8,
                                                                          dtype=torch.int32), n) for n in range(1, 16))


def test_committed_counts_and_step_logprobs():
    assert L.committed(_state(40, 3), 512) == 4
    assert L.committed(_state(40, 3, terminal=1), 512) == 3, "terminal: no bonus"
    assert L.committed(_state(40, 3, M=43), 512) == 3, "no room for the bonus"
    assert L.committed(_state(40, 3, M=0), 44) == 4, "M = 0 reads the token row length"
    g = torch.Generator().manual_seed(1)
    S, V, M = 4, 64, 64
    logits = (torch.randn(3 * S, V, generator=g) * 2).to(F16)
    tokens = torch.randint(0, V, (3, M), generator=g)
    state = torch.stack([_state(10, 2), _state(20, 1, frozen=1), _state(30, 0, terminal=1)])
    acc = torch.tensor([[10, 11, 0, 0], [0] * 4, [0] * 4], dtype=torch.int32)
    out = L.step_logprobs(logits, S, tokens, state, acc, [0.6, 1.0, 1.0], [False, False, True], [5, 5, 5])
    assert sorted(out) == [(0, 10), (0, 11), (0, 12)], "frozen and terminal-without-accepts write nothing"
    assert out[(0, 11)] == L.row_logprobs(logits[1], int(tokens[0, 11]), 0.6, False, 5)    # node 10 - (10 - 1) = 1
    assert out[(0, 12)] == L.row_logprobs(logits[2], int(tokens[0, 12]), 0.6, False, 5)
    assert L.step_logprobs(logits, S, tokens, state, acc, [0.6] * 3, [False] * 3, [None] * 3) == {}


# ------------------------------------------------------------------------------------------------ refusals
def test_check_logprobs():
    from sequoia_b200.batch import _logprobs, check_logprobs
    assert check_logprobs(None) is None
    for ok in (0, 1, 20, np.int64(5)):
        assert check_logprobs(ok) == int(ok)
    for bad in (-1, 21, True, False, 1.0, "3", [2]):
        with pytest.raises(ValueError, match="logprobs"):
            check_logprobs(bad)
    assert _logprobs(None, 3) == [None] * 3 and _logprobs(4, 2) == [4, 4]
    assert _logprobs([None, 0, 20], 3) == [None, 0, 20]
    with pytest.raises(ValueError, match="3 values for 2"):
        _logprobs([1, 2, 3], 2)
    with pytest.raises(ValueError):
        _logprobs([1, 21], 2)


def test_constructor_and_admit_refuse_bad_logprobs(monkeypatch):
    from sequoia_b200.batch import BatchTree
    prompts = [torch.zeros(3), torch.zeros(4)]
    for kw in (dict(logprobs=21), dict(logprobs=True), dict(logprobs=[1]), dict(logprobs=[1, -1]), dict(logprobs=2.0)):
        with pytest.raises(ValueError):
            BatchTree(None, None, prompts, {}, **kw)
    bt = _cpu_tree(monkeypatch, [torch.ones(n, dtype=torch.long) for n in (5, 7)])
    graphs = dict(bt.graphs)
    for bad in (21, -1, False, 0.5):
        with pytest.raises(ValueError, match="logprobs"):
            bt.admit(0, torch.ones(6, dtype=torch.long), logprobs=bad)
    assert bt.logprobs == [None, None] and not bt.use_logprobs and bt.graphs == graphs, "a refusal changes nothing"
    with pytest.raises(ValueError, match="logprobs off"):
        bt.token_logprobs(0)
    with pytest.raises(IndexError):
        bt.token_logprobs(2)


def test_ops_refuses_host_tensors():
    from sequoia_b200 import ops
    t = torch.zeros(8, 64, dtype=F16)
    i32 = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(TypeError, match="CUDA"):
        ops.token_logprobs_batch_(t, 4, 1, torch.zeros(2, 16, dtype=torch.long), torch.zeros(2, 16, dtype=torch.int32),
                                  torch.zeros(2, 8, dtype=torch.int32), torch.ones(2), i32, i32,
                                  torch.zeros(2, 16), torch.zeros(2, 16, 20, dtype=torch.int32), torch.zeros(2, 16, 20))


def test_entry_point_refuses_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    f = 256                                             # a non-null, 16-byte aligned address: refused before any launch

    def call(logits=f, ld=32000, V=32000, S=128, depth=7, tokens=f, ld_seq=384, state=f, acc=f, ld_acc=128, T=f,
             greedy=f, n_top=f, lp_token=f, lp_ids=f, lp_top=f, B=2):
        return lib.sq_token_logprobs_batch(logits, ld, V, S, depth, tokens, ld_seq, state, acc, ld_acc, T, greedy, n_top,
                                           lp_token, lp_ids, lp_top, B, None)
    c0 = lib.sq_launch_count()
    null = [dict(**{k: None}) for k in ("logits", "tokens", "state", "acc", "T", "greedy", "n_top", "lp_token", "lp_ids",
                                        "lp_top")]
    cases_ = [(kw, b"null array") for kw in null] + [
        (dict(B=0), b"B=0"), (dict(B=9), b"B=9"), (dict(V=32004, ld=32008), b"V=32004"),
        (dict(V=131080, ld=131080), b"V=131080"), (dict(V=0), b"V=0"), (dict(ld=31999), b"ld=31999"),
        (dict(ld=32004), b"ld=32004"), (dict(logits=264), b"aligned"), (dict(S=0, depth=0), b"S=0"),
        (dict(depth=128), b"max_depth=128"), (dict(depth=-1), b"max_depth=-1"), (dict(ld_seq=0), b"ld_seq=0"),
        (dict(ld_acc=6), b"ld_acc=6")]
    for kw, msg in cases_:
        assert call(**kw) == -1 and msg in lib.sq_last_error(), (kw, msg, lib.sq_last_error())
    assert lib.sq_launch_count() == c0, "refused before any launch"


# ------------------------------------------------------------------------------------------------ per-slot arrays
def test_device_logprobs_of_a_tree(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    assert bt.logprobs == [None] * 3 and not bt.use_logprobs and bt.lp_token is None
    assert bt.n_top_dev.tolist() == [-1] * 3 and bt.n_top_dev.dtype == torch.int32
    assert bt.prompt_lens == [5, 7, 9]
    bt = _cpu_tree(monkeypatch, prompts, logprobs=[None, 0, 20])
    assert bt.logprobs == [None, 0, 20] and bt.n_top_dev.tolist() == [-1, 0, 20]
    assert _cpu_tree(monkeypatch, prompts, logprobs=3).n_top_dev.tolist() == [3] * 3


def test_admissions_update_the_slots_and_recapture_once(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    bt.admit(0, torch.ones(6, dtype=torch.long))
    assert not bt.use_logprobs and bt.graphs == {"draft": 1, "steady": 2, "post": 3}, "off: no recapture"
    bt.admit(1, torch.ones(12, dtype=torch.long), logprobs=5)
    assert bt.use_logprobs and bt.graphs == {"draft": 1}, "the first admission with logprobs drops steady and post once"
    assert tuple(bt.lp_token.shape) == (3, 64) and bt.lp_token.dtype == torch.float32
    assert tuple(bt.lp_ids.shape) == (3, 64, 20) and bt.lp_ids.dtype == torch.int32
    assert tuple(bt.lp_top.shape) == (3, 64, 20) and bt.lp_top.dtype == torch.float32
    assert bt.n_top_dev.tolist() == [-1, 5, -1] and bt.prompt_lens == [6, 12, 9]
    bt.graphs = {"draft": 1, "steady": 4, "post": 5}
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long))
    assert bt.n_top_dev.tolist() == [-1, 5, -1] and bt.logprobs[1] == 5, "the previous value is kept"
    lp, ids, top = bt.token_logprobs(1)
    assert lp.shape == (0,) and ids.shape == (0, 5) and ids.dtype == torch.int64, "after admit: the new prompt only"
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long), logprobs=None)
    assert bt.n_top_dev.tolist() == [-1, -1, -1] and bt.logprobs[1] is None
    bt.admit(2, torch.ones(4, dtype=torch.long), logprobs=0)
    assert bt.graphs == {"draft": 1, "steady": 4, "post": 5} and bt.use_logprobs, "logprobs stay on, no recapture"
    assert bt.n_top_dev.tolist() == [-1, -1, 0]
    # token_logprobs: positions len(prompt) .. len(last tokens), k = the slot's n
    with torch.inference_mode():                        # (admit allocates under inference mode)
        bt.lp_token[2] = torch.arange(64, dtype=torch.float32)
        bt.lp_ids[2] = torch.arange(20, dtype=torch.int32)
    bt.last[2] = (torch.zeros(9, dtype=torch.long), 8, False)
    lp, ids, top = bt.token_logprobs(2)
    assert lp.tolist() == [4.0, 5.0, 6.0, 7.0, 8.0] and ids.shape == (5, 0) and top.shape == (5, 0)


# ------------------------------------------------------------------------------------------------ testbed
def test_logprobs_flag_parsing_and_refusals():
    import testbed
    ap = testbed.build_parser()
    assert testbed.batch_logprobs(ap.parse_args([])) is None
    assert testbed.batch_logprobs(ap.parse_args(["--logprobs", "5", "--batch", "2"])) == 5
    assert testbed.batch_logprobs(ap.parse_args(["--logprobs", "0", "--batch", "1", "--refill"])) == 0
    with pytest.raises(SystemExit, match="--batch"):
        testbed.batch_logprobs(ap.parse_args(["--logprobs", "5"]))
    for bad in ("21", "-1"):
        with pytest.raises(SystemExit, match="--logprobs"):
            testbed.batch_logprobs(ap.parse_args(["--logprobs", bad, "--batch", "2"]))


def test_batches_and_refill_report_the_mean_logprob(monkeypatch, capsys):
    import testbed
    import sequoia_b200.batch as batch
    built, admitted = [], []

    class Tree:
        def __init__(self, draft, target, chunk, gm, policy, **kw):
            built.append(kw.get("logprobs", "absent"))
            self.frozen = [False] * len(chunk)
            self.lens = [len(p) for p in chunk]

        def admit(self, b, prompt, **kw):
            admitted.append(kw)
            self.frozen[b] = False
            self.lens[b] = len(prompt)

        def construct_grow_map(self):
            pass

        def verify(self):
            out = [(torch.ones(300, dtype=torch.long), 0, True) for _ in self.frozen]
            self.frozen = [True] * len(self.frozen)
            return out

        def freeze(self, b):
            self.frozen[b] = True

        def token_logprobs(self, b):
            n = 300 - self.lens[b]
            return torch.full((n,), -0.5 * (b + 1)), torch.zeros(n, 3, dtype=torch.long), torch.zeros(n, 3)
    monkeypatch.setattr(batch, "BatchTree", Tree)
    monkeypatch.setattr(testbed.torch.cuda, "synchronize", lambda *a: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)

    class Eng:
        def clear_kv(self):
            pass
    prompts = [torch.tensor([i, 1]) for i in range(4)]
    res = testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, logprobs=3)
    assert res["mean_token_logprob"] == [-0.5, -1.0, -0.5, -1.0] and "prompt 3: mean token logprob -1.0000" in \
        capsys.readouterr().out
    res = testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2)
    assert "mean_token_logprob" not in res and built == [3, 3, "absent", "absent"]
    built.clear()
    res = testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, refill=True, logprobs=0)
    assert built == [0] and len(admitted) == 2 and not any("logprobs" in kw for kw in admitted)
    assert res["mean_token_logprob"] == [-0.5, -1.0, -0.5, -1.0]
