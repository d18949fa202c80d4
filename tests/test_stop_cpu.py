"""Host-side pieces of stop mode that need no GPU: the CPU statement of the cut (oracle/stop.py) against a brute-force
scan, the refusals of BatchTree's stop_tokens / max_new_tokens and of the C entry points, the device rows a tree keeps
per slot through construction and admissions, and testbed.py's --device-stop."""
import random

import pytest
import torch

import cases  # noqa: F401  (puts the repository root on sys.path)
from oracle.stop import cut


def _brute(tokens, P, n, stop_ids, end_limit):
    """Every candidate end, the stop ids' before the limit's, and the smallest wins (stable: a stop id on a tie)."""
    ends = [(j + 1, 1) for j in range(P, n) if tokens[j] in {t for t in stop_ids if t >= 0}]
    if 0 < end_limit <= n:
        ends.append((end_limit, 2))
    if not ends:
        return 0, 0
    end, finish = min(ends, key=lambda e: (e[0], e[1]))
    return finish, end


def test_cut_matches_brute_force():
    rnd = random.Random(5)
    for _ in range(3000):
        n_tok = rnd.randint(1, 40)
        tokens = [rnd.randint(0, 12) for _ in range(n_tok)]
        P = rnd.randint(0, n_tok - 1)
        n = rnd.randint(P, n_tok)
        ids = rnd.sample(range(13), rnd.randint(0, 8))
        row = ids + [-1] * (8 - len(ids))
        limit = rnd.choice([0, -3, rnd.randint(1, n_tok + 3), P + 1, n])
        assert cut(tokens, P, n, row, limit) == _brute(tokens, P, n, row, limit), (tokens, P, n, row, limit)


def test_cut_rules():
    t = [5, 5, 9, 7, 2, 0, 9]
    assert cut(t, 2, 7, [9], 0) == (1, 3), "the first stop id in [P, n)"
    assert cut(t, 3, 7, [9], 0) == (1, 7)
    assert cut(t, 3, 6, [9], 0) == (0, 0), "tokens at or past n are not output"
    assert cut(t, 3, 7, [], 5) == (2, 5) and cut(t, 3, 7, [], 7) == (2, 7) and cut(t, 3, 7, [], 8) == (0, 0)
    assert cut(t, 2, 7, [7], 4) == (1, 4), "a tie goes to the stop id"
    assert cut(t, 2, 7, [7], 3) == (2, 3)
    assert cut(t, 2, 7, [-1] * 8, 0) == (0, 0), "padding never matches"


# ------------------------------------------------------------------------------------------------ validation
def test_check_stop_tokens_and_budgets():
    import numpy as np
    from sequoia_b200.batch import _budgets, _stop_sets, check_max_new_tokens, check_stop_tokens
    assert check_stop_tokens(None) is None and check_stop_tokens([]) == ()
    assert check_stop_tokens([128009, 128001, 128009, np.int64(2)], 128256) == (2, 128001, 128009)
    assert check_stop_tokens(frozenset([1, 2])) == (1, 2) and check_stop_tokens(list(range(8)), 8) == tuple(range(8))
    for bad in ([-1], [1.5], [True], "12", 5, [None], list(range(9)), [[1]]):
        with pytest.raises(ValueError, match="stop_tokens"):
            check_stop_tokens(bad)
    with pytest.raises(ValueError, match="stop_tokens"):
        check_stop_tokens([32000], 32000)
    for ok in (None, 1, 1000, np.int32(4)):
        assert check_max_new_tokens(ok) == (None if ok is None else int(ok))
    for bad in (0, -1, 1.5, True, "3", [2]):
        with pytest.raises(ValueError, match="max_new_tokens"):
            check_max_new_tokens(bad)
    assert _stop_sets(None, 2) == [None, None] and _stop_sets([], 2) == [(), ()]
    assert _stop_sets([0, 2], 3) == [(0, 2)] * 3, "a list of ids is one set for all"
    assert _stop_sets([[3], None, []], 3) == [(3,), None, ()], "a list of sets is one per prompt"
    with pytest.raises(ValueError, match="3 sets for 2"):
        _stop_sets([[1], [2], [3]], 2)
    with pytest.raises(ValueError, match="stop_tokens"):
        _stop_sets([1, [2]], 2)
    assert _budgets(None, 2) == [None, None] and _budgets(7, 2) == [7, 7] and _budgets([None, 3], 2) == [None, 3]
    with pytest.raises(ValueError, match="3 values for 2"):
        _budgets([1, 2, 3], 2)


def test_constructor_and_admit_refuse_bad_stop_settings():
    from sequoia_b200.batch import BatchTree
    prompts = [torch.zeros(3), torch.zeros(4)]
    for kw in (dict(stop_tokens=[-1]), dict(stop_tokens=list(range(9))), dict(stop_tokens=[[1], [2], [3]]),
               dict(stop_tokens=[True]), dict(stop_tokens="2"), dict(max_new_tokens=0), dict(max_new_tokens=[1, 2, 3]),
               dict(max_new_tokens=True), dict(max_new_tokens=2.0)):
        with pytest.raises(ValueError):
            BatchTree(None, None, prompts, {}, **kw)
    bt = BatchTree.__new__(BatchTree)
    bt.B, bt.M, bt.S, bt.V, bt.seeded = 2, 64, 9, 32000, False
    bt.policies, bt.frozen = ["spec", "spec"], [True, False]
    bt.temps, bt.top_ps, bt.top_ks = [0.6] * 2, [1.0] * 2, [0, 0]
    bt.stop_tokens, bt.max_new_tokens = [None, (2,)], [None, 5]
    for kw in (dict(stop_tokens=[32000]), dict(stop_tokens=list(range(9))), dict(stop_tokens=[-2]),
               dict(max_new_tokens=0), dict(max_new_tokens=1.5), dict(max_new_tokens=False)):
        with pytest.raises(ValueError):
            bt.admit(0, torch.zeros(10, dtype=torch.long), **kw)
    assert bt.stop_tokens == [None, (2,)] and bt.max_new_tokens == [None, 5] and bt.frozen == [True, False], \
        "a refusal changes nothing"


def _cpu_tree(monkeypatch, prompts, **kw):
    """A BatchTree whose constructor stops at its first device allocation after the per-slot arrays (torch.tensor is
    redirected to the CPU), completed with the host state admit() reads."""
    import sequoia_b200.batch as batch
    real_tensor = torch.tensor

    class Stop(Exception):
        pass

    def stop(*a, **k):
        raise Stop
    monkeypatch.setattr(batch.torch, "tensor", lambda data, dtype=None, device=None: real_tensor(data, dtype=dtype))
    monkeypatch.setattr(batch.torch, "zeros", stop)
    monkeypatch.setattr(batch, "_Static", lambda gm, dev: type("St", (), dict(S=9))())
    monkeypatch.setattr(batch, "check_vocab", lambda pol, V: None)

    class Eng:
        def __init__(self):
            self.engine = type("E", (), dict(batch_size=len(prompts), max_length=64))()
            self.engine.model_config = type("C", (), dict(vocab_size=32000))()
            self.device = "cuda:0"
    bt = batch.BatchTree.__new__(batch.BatchTree)
    with pytest.raises(Stop):
        batch.BatchTree.__init__(bt, Eng(), Eng(), prompts, {}, max_length=64, **kw)
    monkeypatch.undo()
    monkeypatch.setattr(batch, "_h2d", lambda t: t)                 # (no pinned memory without a GPU)
    bt.device = torch.device("cpu")
    B = len(prompts)
    bt.frozen, bt.last, bt.r, bt.seeded = [True] * B, [None] * B, None, False
    bt.ground_truth_len, bt.target_kv_len = [len(p) for p in prompts], [0] * B
    bt.graphs = {"draft": 1, "steady": 2, "post": 3}
    bt._load_prompt = lambda b, p: None
    bt.op_draft_prefill = lambda seqs: None
    return bt


def test_device_stop_rows_of_a_tree(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    assert not bt.use_stop and bt.stop_tokens == [None] * 3 and bt.max_new_tokens == [None] * 3
    assert bt.stop_ids_dev.tolist() == [[-1] * 8] * 3 and bt.stop_ids_dev.dtype == torch.int32
    assert bt.end_limit_dev.tolist() == [0, 0, 0] and bt.end_limit_dev.dtype == torch.int32
    assert bt.finish_reason == [None] * 3
    bt = _cpu_tree(monkeypatch, prompts, stop_tokens=[[128 % 7, 3], None, []], max_new_tokens=[None, 4, 10 ** 12])
    assert bt.use_stop
    assert bt.stop_ids_dev.tolist() == [[2, 3] + [-1] * 6, [-1] * 8, [-1] * 8]
    assert bt.end_limit_dev.tolist() == [0, 11, (1 << 31) - 1], "len(prompt) + budget, clamped to int32"
    assert _cpu_tree(monkeypatch, prompts, stop_tokens=[]).use_stop, "an empty set is stop mode too"
    assert _cpu_tree(monkeypatch, prompts, max_new_tokens=3).end_limit_dev.tolist() == [8, 10, 12]


def test_admissions_update_the_rows_and_recapture_once(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    bt.admit(0, torch.ones(6, dtype=torch.long))
    assert not bt.use_stop and bt.graphs == {"draft": 1, "steady": 2, "post": 3}, "default mode: no recapture"
    bt.admit(1, torch.ones(12, dtype=torch.long), stop_tokens=[128009 % 32000, 7], max_new_tokens=20)
    assert bt.use_stop and bt.graphs == {"draft": 1}, "the first stop admission drops steady and post once"
    assert bt.stop_ids_dev[1].tolist() == [7, 128009 % 32000] + [-1] * 6 and int(bt.end_limit_dev[1]) == 32
    assert bt.finish_reason[1] is None
    bt.graphs = {"draft": 1, "steady": 4, "post": 5}
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long))
    assert bt.stop_ids_dev[1].tolist() == [7, 128009 % 32000] + [-1] * 6 and int(bt.end_limit_dev[1]) == 30, \
        "the previous set and budget, the budget counted from the new prompt"
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long), stop_tokens=None, max_new_tokens=None)
    assert bt.stop_ids_dev[1].tolist() == [-1] * 8 and int(bt.end_limit_dev[1]) == 0, "None clears"
    bt.admit(2, torch.ones(4, dtype=torch.long), stop_tokens=[1], max_new_tokens=1)
    assert bt.graphs == {"draft": 1, "steady": 4, "post": 5} and bt.use_stop, "stop mode stays on, no recapture"
    assert bt.stop_ids_dev.tolist()[0] == [-1] * 8 and int(bt.end_limit_dev[2]) == 5
    assert bt.stop_tokens == [None, None, (1,)] and bt.max_new_tokens == [None, None, 1]


# ------------------------------------------------------------------------------------------------ C entry points
def test_stop_entry_points_refuse_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    f = 256                                             # a non-null address: every case is refused before any launch

    def stoch(T=f, stop=f, end=f, S=9, V=32000, B=2, greedy=None, policy=0, ld_acc=9):
        return lib.sq_accept_stochastic_batch_stop(f, V, f, V, f, f, f, f, V, f, f, f, S, V, T, greedy, stop, end, f, f,
                                                   64, f, ld_acc, f, B, 64, policy, None)

    def greedy(stop=f, end=f, S=9, B=2, g=None):
        return lib.sq_accept_greedy_batch_stop(f, f, f, f, S, f, f, 64, f, 9, f, g, stop, end, B, 64, None)
    c0 = lib.sq_launch_count()
    for call, msg in ((lambda: stoch(stop=None), b"null stop_ids"), (lambda: stoch(end=None), b"null stop_ids"),
                      (lambda: stoch(T=None), b"null temperature"), (lambda: stoch(B=0), b"B=0"),
                      (lambda: stoch(B=9), b"B=9"), (lambda: stoch(S=0), b"S=0"), (lambda: stoch(S=1025), b"S=1025"),
                      (lambda: stoch(policy=4), b"policy"), (lambda: stoch(ld_acc=8), b"too short"),
                      (lambda: stoch(V=32004), b"V=32004"), (lambda: stoch(V=131080, greedy=f), b"V=131080"),
                      (lambda: greedy(stop=None), b"null stop_ids"), (lambda: greedy(end=None, g=f), b"null stop_ids"),
                      (lambda: greedy(B=0), b"B=0"), (lambda: greedy(B=9, g=f), b"B=9"), (lambda: greedy(S=0), b"S=0")):
        assert call() == -1 and msg in lib.sq_last_error(), (msg, lib.sq_last_error())
    assert lib.sq_launch_count() == c0, "refused before any launch"


# ------------------------------------------------------------------------------------------------ testbed --device-stop
def test_device_stop_flag_parsing_and_refusals():
    import testbed
    ap = testbed.build_parser()
    assert not ap.parse_args([]).device_stop and not testbed.batch_device_stop(ap.parse_args([]))
    assert testbed.batch_device_stop(ap.parse_args(["--device-stop", "--batch", "2"]))
    assert testbed.batch_device_stop(ap.parse_args(["--device-stop", "--batch", "1", "--refill"]))
    with pytest.raises(SystemExit, match="with --batch"):
        testbed.batch_device_stop(ap.parse_args(["--device-stop"]))


def test_device_stop_settings_end_where_the_host_loop_does():
    import testbed
    prompts = [torch.zeros(n, dtype=torch.long) for n in (10, 255, 256, 300)]
    stops, budgets = testbed.device_stop_settings(prompts, frozenset([128009, 128001, 128008]))
    assert stops == [[128001, 128008, 128009]] * 4
    assert budgets == [testbed.MAX_NEW_LEN - 10, 1, 1, 1]
    assert [len(p) + n for p, n in zip(prompts, budgets)][:2] == [testbed.MAX_NEW_LEN] * 2


class _FakeTree:
    """Finishes every slot after one step (as a device stop would) and records what each admission brought."""

    def __init__(self, prompts):
        self.frozen = [False] * len(prompts)
        self.rows = [p.clone() for p in prompts]
        self.admitted = []

    def admit(self, b, prompt, **kw):
        self.admitted.append((b, len(prompt), kw))
        self.rows[b] = prompt.clone()
        self.frozen[b] = False

    def construct_grow_map(self):
        pass

    def verify(self):
        out = []
        for b, row in enumerate(self.rows):
            out.append((torch.cat([row, torch.tensor([5])]), len(row), not self.frozen[b]))
            self.frozen[b] = True
        return out

    def freeze(self, b):
        self.frozen[b] = True


def test_refill_admissions_carry_each_prompts_stop_settings():
    import testbed
    prompts = [torch.zeros(n, dtype=torch.long) for n in (10, 20, 30, 40, 50)]
    dstop = testbed.device_stop_settings(prompts, frozenset([2, 0]))
    tree = _FakeTree(prompts[:2])
    testbed.decode_refill(tree, prompts, [testbed.MAX_NEW_LEN] * 5, device_stop=dstop)
    assert [(n, kw["stop_tokens"], kw["max_new_tokens"]) for _, n, kw in tree.admitted] == \
        [(n, [0, 2], testbed.MAX_NEW_LEN - n) for n in (30, 40, 50)]
    tree = _FakeTree(prompts[:2])
    testbed.decode_refill(tree, prompts, [testbed.MAX_NEW_LEN] * 5)
    assert all(kw == {} for _, _, kw in tree.admitted), "without the flag admissions keep each slot's settings"


def test_chunked_batches_get_the_stop_settings(monkeypatch):
    import testbed
    import sequoia_b200.batch as batch
    built = []

    class Tree:
        def __init__(self, draft, target, chunk, gm, policy, **kw):
            built.append((kw.get("stop_tokens"), kw.get("max_new_tokens")))
            self.frozen = [True] * len(chunk)
    monkeypatch.setattr(batch, "BatchTree", Tree)
    monkeypatch.setattr(testbed.torch.cuda, "synchronize", lambda *a: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)

    class Eng:
        def clear_kv(self):
            pass
    prompts = [torch.zeros(n, dtype=torch.long) for n in (10, 20, 30, 40)]
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, stop=frozenset([7]), device_stop=True)
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2)
    M = testbed.MAX_NEW_LEN
    assert built == [([[7], [7]], [M - 10, M - 20]), ([[7], [7]], [M - 30, M - 40]), (None, None), (None, None)]
