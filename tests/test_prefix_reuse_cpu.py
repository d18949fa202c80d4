"""Host-side pieces of prefix reuse that need no GPU: the reuse_prefix check, the donor rule (prefix_donor) with its cap,
ready-length limit, tie order and prompt_logprobs rule, the admissions' copies and prefill starts on a CPU tree, the
refusals of sq_kv_copy_prefix through the library, and testbed.py's --reuse-prefix flag."""
import pytest
import torch

from test_stop_cpu import _cpu_tree


def _t(xs):
    return torch.tensor(xs, dtype=torch.long)


def _rows(*rows, width=16):
    out = torch.full((len(rows), width), -1, dtype=torch.long)
    for d, r in enumerate(rows):
        out[d, :len(r)] = _t(r)
    return out


# ------------------------------------------------------------------------------------------------ donor rule
def test_longest_match_wins():
    from sequoia_b200.batch import prefix_donor
    prompt = _t([5, 6, 7, 8, 9, 10])
    rows = _rows([5, 6, 1], [5, 6, 7, 8], [5, 9], [1, 2, 3])
    assert prefix_donor(prompt, rows, [3, 4, 2, 3], b=3) == (1, 4)
    assert prefix_donor(prompt, rows, [3, 4, 2, 3], b=0) == (1, 4)
    assert prefix_donor(_t([4, 6, 7]), rows, [3, 4, 2, 3], b=0) == (None, 0), "no slot shares the first token"


def test_cap_at_prompt_length_minus_one():
    from sequoia_b200.batch import prefix_donor
    rows = _rows([5, 6, 7, 8, 9, 10], [5, 6])
    assert prefix_donor(_t([5, 6, 7, 8]), rows, [6, 2], b=1) == (0, 3), "the last prompt row always runs"
    assert prefix_donor(_t([5, 6, 7]), rows, [6, 2], b=1) == (1, 2), "capped at P - 1: a tie, slot b first"
    assert prefix_donor(_t([5]), rows, [6, 2], b=1) == (None, 0), "a one-token prompt reuses nothing"


def test_ready_length_limits_the_match():
    from sequoia_b200.batch import prefix_donor
    rows = _rows([5, 6, 7, 8, 9], [5, 6, 7, 8, 9])
    prompt = _t([5, 6, 7, 8, 9, 10, 11])
    assert prefix_donor(prompt, rows, [2, 4], b=0) == (1, 4), "tokens past R_d do not count"
    assert prefix_donor(prompt, rows, [0, 0], b=0) == (None, 0), "R_d = 0: no candidate"
    assert prefix_donor(prompt, rows, [5, 0], b=1) == (0, 5)


def test_tie_order_prefers_the_slot_then_the_lowest_index():
    from sequoia_b200.batch import prefix_donor
    rows = _rows([1, 2, 3], [1, 2, 3], [1, 2, 3], [1, 2, 3])
    prompt = _t([1, 2, 3, 4])
    assert prefix_donor(prompt, rows, [3, 3, 3, 3], b=2) == (2, 3)
    assert prefix_donor(prompt, rows, [3, 3, 3, 0], b=3) == (0, 3)
    assert prefix_donor(prompt, rows, [2, 3, 3, 2], b=3) == (1, 3)


def test_prompt_logprobs_forces_zero():
    from sequoia_b200.batch import prefix_donor
    rows = _rows([1, 2, 3], [1, 2, 3])
    assert prefix_donor(_t([1, 2, 3, 4]), rows, [3, 3], b=0, prompt_logprobs=0) == (None, 0)
    assert prefix_donor(_t([1, 2, 3, 4]), rows, [3, 3], b=0, prompt_logprobs=None) == (0, 3)


def test_reuse_prefix_must_be_a_bool():
    from sequoia_b200.batch import check_reuse_prefix
    assert check_reuse_prefix(True) is True and check_reuse_prefix(False) is False
    for bad in (1, 0, None, "yes", 1.0):
        with pytest.raises(ValueError, match="reuse_prefix must be a bool"):
            check_reuse_prefix(bad)


# ------------------------------------------------------------------------------------------------ admissions
def _tree(monkeypatch, prompts, **kw):
    import sequoia_b200.batch as batch
    bt = _cpu_tree(monkeypatch, prompts, **kw)
    copies = []
    monkeypatch.setattr(batch.ops, "kv_copy_prefix", lambda kv, src, dst, n: copies.append((kv, src, dst, n)))
    bt.draft.engine.kv_cache, bt.target.engine.kv_cache = "draft", "target"
    bt.tokens = torch.zeros(len(prompts), 64, dtype=torch.long)
    for b, p in enumerate(prompts):
        bt.tokens[b, :len(p)] = p
    return bt, copies


def test_admissions_copy_and_report(monkeypatch):
    prompts = [_t([3, 4, 5, 6, 7, 8]), _t([3, 4, 9, 9]), _t([1, 1])]
    bt, copies = _tree(monkeypatch, prompts)
    assert bt.reused_prefix == [None] * 3 and [bt._prefill_start(b) for b in range(3)] == [0, 0, 0]
    bt.target_kv_len = [5, 3, 1]
    with pytest.raises(ValueError, match="reuse_prefix must be a bool"):
        bt.admit(2, _t([3, 4, 5, 6, 7, 8, 1]), reuse_prefix=1)
    bt.admit(2, _t([3, 4, 5, 6, 7, 8, 1]), reuse_prefix=True)
    assert bt.reused_prefix[2] == (0, 5) and bt._prefill_start(2) == 5
    assert copies == [("draft", 0, 2, 5), ("target", 0, 2, 5)], "one copy per cache, draft first"
    assert bt.target_kv_len[2] == 0, "an admitted slot is no donor until its first verify"
    copies.clear()
    bt.admit(1, _t([3, 4, 9, 9, 2]), reuse_prefix=True)           # multi-turn: its own rows, no copy
    assert bt.reused_prefix[1] == (1, 3) and copies == []
    bt.frozen[1] = True
    bt.admit(1, _t([3, 4, 9, 9, 2]))
    assert bt.reused_prefix[1] is None and bt._prefill_start(1) == 0 and copies == []


def test_default_admission_reads_no_tokens(monkeypatch):
    prompts = [_t([3, 4, 5]), _t([3, 4, 5])]
    bt, copies = _tree(monkeypatch, prompts)
    bt.target_kv_len = [2, 2]

    class NoRead:
        def __getitem__(self, k):
            raise AssertionError("reuse_prefix=False read the token rows")
    bt.tokens = NoRead()
    bt.admit(0, _t([3, 4, 5, 6]))
    assert bt.reused_prefix == [None, None] and copies == []


def test_prompt_logprobs_admission_reuses_nothing(monkeypatch):
    prompts = [_t([3, 4, 5, 6]), _t([3, 4, 5, 6])]
    bt, copies = _tree(monkeypatch, prompts)
    bt.target_kv_len = [3, 3]
    bt._start_prompt_logprobs = lambda: None
    bt.admit(1, _t([3, 4, 5, 6, 7]), reuse_prefix=True, prompt_logprobs=2)
    assert bt.reused_prefix[1] is None and copies == []
    bt.frozen[1] = True
    bt.admit(1, _t([3, 4, 5, 6, 7]), reuse_prefix=True)             # the setting stays on (_PREVIOUS)
    assert bt.reused_prefix[1] is None
    bt.frozen[1] = True
    bt.admit(1, _t([3, 4, 5, 6, 7]), reuse_prefix=True, prompt_logprobs=None)
    assert bt.reused_prefix[1] == (0, 3) and copies == [("draft", 0, 1, 3), ("target", 0, 1, 3)]


def test_admission_keeps_the_graphs(monkeypatch):
    prompts = [_t([3, 4, 5, 6]), _t([3, 4, 5, 6])]
    bt, _ = _tree(monkeypatch, prompts)
    bt.target_kv_len = [3, 0]
    bt.admit(1, _t([3, 4, 5, 6, 7]), reuse_prefix=True)
    assert bt.graphs == {"draft": 1, "steady": 2, "post": 3}


# ------------------------------------------------------------------------------------------------ C entry point
def test_copy_prefix_refusals():
    from sequoia_b200 import _lib
    lib = _lib.load()
    k, v = 1 << 20, 1 << 21                                          # aligned, never dereferenced: refused first
    good = dict(k=k, v=v, L=2, B=4, Hkv=12, M=64, D=64, src=0, dst=1, n=8)
    bad = [dict(k=None), dict(v=None), dict(k=k + 2), dict(D=60), dict(D=0), dict(L=0), dict(Hkv=0), dict(B=0),
           dict(B=9), dict(src=-1), dict(src=4), dict(dst=4), dict(dst=-1), dict(dst=0), dict(n=0), dict(n=65),
           dict(n=-3)]
    for change in bad:
        a = dict(good, **change)
        rc = lib.sq_kv_copy_prefix(a["k"], a["v"], a["L"], a["B"], a["Hkv"], a["M"], a["D"], a["src"], a["dst"], a["n"],
                                   None)
        assert rc == -1, change
        assert b"sq_kv_copy_prefix" in lib.sq_last_error(), change


# ------------------------------------------------------------------------------------------------ testbed
def test_testbed_flag():
    import testbed
    ap = testbed.build_parser()
    assert testbed.batch_reuse_prefix(ap.parse_args([])) is False
    assert testbed.batch_reuse_prefix(ap.parse_args(["--reuse-prefix", "--batch", "2", "--refill"])) is True
    with pytest.raises(SystemExit, match="--refill"):
        testbed.batch_reuse_prefix(ap.parse_args(["--reuse-prefix", "--batch", "2"]))


def test_testbed_refill_passes_the_flag_and_counts(monkeypatch, capsys):
    import testbed
    import sequoia_b200.batch as batch
    admitted = []

    class Tree:
        def __init__(self, draft, target, chunk, gm, policy, **kw):
            assert "reuse_prefix" not in kw
            self.frozen = [False] * len(chunk)
            self.reused_prefix = [None] * len(chunk)

        def admit(self, b, prompt, **kw):
            admitted.append(kw)
            self.frozen[b] = False
            self.reused_prefix[b] = (0, len(prompt) - 1) if kw.get("reuse_prefix") else None

        def construct_grow_map(self):
            pass

        def verify(self):
            out = [(torch.ones(300, dtype=torch.long), 0, True) for _ in self.frozen]
            self.frozen = [True] * len(self.frozen)
            return out

        def freeze(self, b):
            self.frozen[b] = True
    monkeypatch.setattr(batch, "BatchTree", Tree)
    monkeypatch.setattr(testbed.torch.cuda, "synchronize", lambda *a: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)

    class Eng:
        def clear_kv(self):
            pass
    prompts = [torch.arange(n) for n in (4, 5, 6, 7)]
    res = testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, refill=True, reuse_prefix=True)
    assert [kw.get("reuse_prefix") for kw in admitted] == [True, True]
    assert res["reused_prompt_tokens"] == 5 + 6
    assert "reused prompt tokens: 11 in 2 admissions" in capsys.readouterr().out
    admitted.clear()
    res = testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, refill=True)
    assert admitted == [{}, {}] and "reused_prompt_tokens" not in res
