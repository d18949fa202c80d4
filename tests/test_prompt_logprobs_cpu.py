"""Host-side pieces of the prompt logprobs that need no GPU: the CPU statement (oracle/prompt_logprobs.py) against a
brute-force sort and log-softmax in Python floats, the refusals of check_prompt_logprobs, ops.prompt_logprobs_ragged_ and
the C entry point, the per-slot settings and the first-verify rule through admissions, and testbed.py's
--prompt-logprobs flag."""
import math

import numpy as np
import pytest
import torch

from oracle import prompt_logprobs as PL
from test_logprobs_cpu import _brute, _rows, _same
from test_stop_cpu import _cpu_tree

F16 = torch.float16
INF, NAN = float("inf"), float("nan")


def _logits_and_prompt(V=96):
    """Prompt rows with ties, -0 / +0, -inf runs, +inf and NaN (the logprobs CPU test's rows), and a prompt that scores
    ids inside them (an id outside V too)."""
    rows = _rows(V)
    logits = torch.stack(list(rows.values()))
    prompt = torch.tensor([7, 5, 11, 40, 41, 95, 0, 9, V + 2])
    return list(rows), logits, prompt


@pytest.mark.parametrize("n", [0, 1, 5, 20])
def test_oracle_matches_brute_force(n):
    names, logits, prompt = _logits_and_prompt()
    got = PL.prompt_logprobs(logits, prompt, n)
    assert len(got) == len(prompt) - 1 == len(names)
    for r, (tok, ids, top) in enumerate(got):
        t = int(prompt[r + 1])
        want = _brute(logits[r], t, 1.0, True, n) if t < logits.shape[1] else (NAN,) + _brute(logits[r], 0, 1.0, True, n)[1:]
        assert ids == want[1], (names[r], n)
        assert _same(tok, want[0]), (names[r], tok, want[0])
        assert all(_same(a, b) for a, b in zip(top, want[2])), (names[r], top, want[2])


def test_oracle_is_the_raw_log_softmax():
    g = torch.Generator().manual_seed(4)
    logits = (torch.randn(12, 64, generator=g) * 3).to(F16)
    prompt = torch.randint(0, 64, (13,), generator=g)
    want = torch.log_softmax(logits.double(), -1)
    for r, (tok, ids, top) in enumerate(PL.prompt_logprobs(logits, prompt, 20)):
        assert abs(tok - float(want[r, int(prompt[r + 1])])) < 1e-12
        assert ids == torch.sort(logits[r].float(), descending=True, stable=True).indices[:20].tolist()
        assert all(a >= b for a, b in zip(top, top[1:])) and tok <= top[0] + 1e-12
    assert PL.prompt_logprobs(logits, prompt[:1], 5) == [], "a one-token prompt has no scored position"
    names, logits, prompt = _logits_and_prompt()
    got = dict(zip(names, PL.prompt_logprobs(logits, prompt, 3)))
    for name in ("pinf", "nan", "all_ninf"):
        assert math.isnan(got[name][0]) and all(math.isnan(v) for v in got[name][2]), name
    assert got["runs"][1][0] == 5 and math.isfinite(got["runs"][2][0])


def test_ragged_maps_rows_to_positions():
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(40, 32, generator=g) * 2).to(F16)
    tokens = torch.randint(0, 32, (3, 24), generator=g)
    parts = [(2, 3, 5, 4), (0, 20, 1, 0)]
    out = PL.ragged_logprobs(logits, parts, tokens)
    assert sorted(out) == [(0, 1)] + [(2, i) for i in range(1, 6)], "position 0 and unlisted slots are never written"
    assert out[(2, 4)] == PL.prompt_logprobs(logits[3:8], tokens[2, :6], 4)[3]
    assert out[(0, 1)][1] == [] and out[(0, 1)][0] == PL.prompt_logprobs(logits[20:21], tokens[0, :2], 0)[0][0]


# ------------------------------------------------------------------------------------------------ refusals
def test_check_prompt_logprobs():
    from sequoia_b200.batch import _prompt_logprobs, check_prompt_logprobs
    assert check_prompt_logprobs(None) is None
    for ok in (0, 1, 20, np.int64(5)):
        assert check_prompt_logprobs(ok) == int(ok)
    for bad in (-1, 21, True, False, 1.0, "3", [2]):
        with pytest.raises(ValueError, match="prompt_logprobs"):
            check_prompt_logprobs(bad)
    assert _prompt_logprobs(None, 3) == [None] * 3 and _prompt_logprobs(4, 2) == [4, 4]
    assert _prompt_logprobs([None, 0, 20], 3) == [None, 0, 20]
    with pytest.raises(ValueError, match="3 values for 2"):
        _prompt_logprobs([1, 2, 3], 2)
    with pytest.raises(ValueError):
        _prompt_logprobs([1, 21], 2)


def test_constructor_and_admit_refuse_bad_settings(monkeypatch):
    from sequoia_b200.batch import BatchTree
    prompts = [torch.zeros(3), torch.zeros(4)]
    for kw in (dict(prompt_logprobs=21), dict(prompt_logprobs=True), dict(prompt_logprobs=[1]),
               dict(prompt_logprobs=[1, -1]), dict(prompt_logprobs=2.0)):
        with pytest.raises(ValueError):
            BatchTree(None, None, prompts, {}, **kw)
    bt = _cpu_tree(monkeypatch, [torch.ones(n, dtype=torch.long) for n in (5, 7)])
    graphs = dict(bt.graphs)
    for bad in (21, -1, False, 0.5):
        with pytest.raises(ValueError, match="prompt_logprobs"):
            bt.admit(0, torch.ones(6, dtype=torch.long), prompt_logprobs=bad)
    assert bt.prompt_logprobs_n == [None, None] and bt.plp_token is None and bt.graphs == graphs, \
        "a refusal changes nothing"
    with pytest.raises(ValueError, match="prompt logprobs off"):
        bt.prompt_logprobs(0)
    with pytest.raises(IndexError):
        bt.prompt_logprobs(2)


def test_ops_refuses_bad_tensors():
    from sequoia_b200 import ops
    t = torch.zeros(8, 64, dtype=F16)
    tok = torch.zeros(2, 16, dtype=torch.long)
    outs = (torch.zeros(2, 16), torch.zeros(2, 16, 20, dtype=torch.int32), torch.zeros(2, 16, 20))
    with pytest.raises(TypeError, match="CUDA"):
        ops.prompt_logprobs_ragged_(t, [(0, 0, 4, 1)], tok, *outs)


def test_entry_point_refuses_bad_arguments():
    import ctypes as C

    from sequoia_b200 import _lib, ops
    lib = _lib.load()
    f = 256                                             # a non-null, 16-byte aligned address: refused before any launch

    def call(logits=f, ld=32000, V=32000, rows=1024, parts=((0, 0, 99, 5), (1, 100, 299, 20)), n_parts=None, tokens=f,
             ld_seq=384, plp_token=f, plp_ids=f, plp_top=f, B=2):
        arr = (ops.PromptLpPart * len(parts))(*parts)
        return lib.sq_prompt_logprobs_ragged(logits, ld, V, rows, C.addressof(arr) if parts else None,
                                             len(parts) if n_parts is None else n_parts, tokens, ld_seq, plp_token,
                                             plp_ids, plp_top, B, None)
    c0 = lib.sq_launch_count()
    null = [dict(**{k: None}) for k in ("logits", "tokens", "plp_token", "plp_ids", "plp_top")]
    cases_ = [(kw, b"null array") for kw in null] + [
        (dict(parts=()), b"null array"), (dict(B=0), b"B=0"), (dict(B=9), b"B=9"),
        (dict(V=32004, ld=32008), b"V=32004"), (dict(V=131080, ld=131080), b"V=131080"), (dict(V=0), b"V=0"),
        (dict(ld=31999), b"ld=31999"), (dict(ld=32004), b"ld=32004"), (dict(logits=264), b"aligned"),
        (dict(n_parts=0), b"0 parts"), (dict(B=1), b"2 parts for 1"),
        (dict(parts=((0, 0, 9, 5), (2, 10, 9, 5)), B=2), b"sequence 2 of 2"),
        (dict(parts=((0, 0, 9, 5), (-1, 10, 9, 5))), b"sequence -1"),
        (dict(parts=((1, 0, 9, 5), (1, 10, 9, 5))), b"listed twice"),
        (dict(parts=((0, 0, 0, 5),)), b"n_rows=0"), (dict(parts=((0, 0, 384, 5),)), b"n_rows=384"),
        (dict(parts=((0, 1000, 30, 5),)), b"rows [1000, 1030) of 1024"),
        (dict(parts=((0, -1, 3, 5),)), b"rows [-1, 2)"),
        (dict(parts=((0, 0, 9, 21),)), b"n_top=21"), (dict(parts=((0, 0, 9, -1),)), b"n_top=-1")]
    for kw, msg in cases_:
        assert call(**kw) == -1 and msg in lib.sq_last_error(), (kw, msg, lib.sq_last_error())
    assert lib.sq_launch_count() == c0, "refused before any launch"


# ------------------------------------------------------------------------------------------------ per-slot settings
def test_settings_and_buffers_through_admissions(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    assert bt.prompt_logprobs_n == [None] * 3 and bt.plp_token is None and bt.plp_ready == [False] * 3
    bt = _cpu_tree(monkeypatch, prompts, prompt_logprobs=[None, 0, 20])
    assert bt.prompt_logprobs_n == [None, 0, 20]
    assert _cpu_tree(monkeypatch, prompts, prompt_logprobs=3).prompt_logprobs_n == [3] * 3
    bt = _cpu_tree(monkeypatch, prompts)
    graphs = dict(bt.graphs)
    bt.admit(0, torch.ones(6, dtype=torch.long))
    assert bt.plp_token is None, "off: nothing allocated"
    bt.admit(1, torch.ones(12, dtype=torch.long), prompt_logprobs=5)
    assert bt.graphs == graphs, "no recapture: the work is eager, outside the graphs"
    assert tuple(bt.plp_token.shape) == (3, 64) and bt.plp_token.dtype == torch.float32
    assert bool(bt.plp_token.isnan().all()) and bool((bt.plp_ids == -1).all()) and bool(bt.plp_top.isnan().all())
    assert tuple(bt.plp_ids.shape) == (3, 64, 20) and bt.plp_ids.dtype == torch.int32
    assert tuple(bt.plp_top.shape) == (3, 64, 20) and bt.plp_top.dtype == torch.float32
    assert bt.prompt_logprobs_n == [None, 5, None]
    with pytest.raises(ValueError, match="first verify"):
        bt.prompt_logprobs(1)
    # the first verify makes the values readable: positions 1 .. P-1, k = the slot's n
    with torch.inference_mode():
        bt.plp_token[1] = torch.arange(64, dtype=torch.float32)
        bt.plp_ids[1] = torch.arange(20, dtype=torch.int32)
    bt.plp_ready[1] = True
    lp, ids, top = bt.prompt_logprobs(1)
    assert lp.tolist() == [float(i) for i in range(1, 12)] and ids.shape == (11, 5) and ids.dtype == torch.int64
    assert ids[0].tolist() == [0, 1, 2, 3, 4] and top.shape == (11, 5)
    # an admission invalidates them, with the setting kept (_PREVIOUS), changed, or turned off
    buf = bt.plp_token
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long))
    assert bt.prompt_logprobs_n[1] == 5 and bt.plp_token is buf, "the previous value is kept, the buffers too"
    with pytest.raises(ValueError, match="first verify"):
        bt.prompt_logprobs(1)
    bt.plp_ready[1] = True
    assert bt.prompt_logprobs(1)[0].shape == (9,)
    bt.frozen[1] = True
    bt.admit(1, torch.ones(1, dtype=torch.long), prompt_logprobs=0)
    bt.plp_ready[1] = True
    lp, ids, top = bt.prompt_logprobs(1)
    assert lp.shape == (0,) and ids.shape == (0, 0) and top.shape == (0, 0), "a one-token prompt: empty arrays"
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long), prompt_logprobs=None)
    with pytest.raises(ValueError, match="prompt logprobs off"):
        bt.prompt_logprobs(1)


def test_first_verify_parts(monkeypatch):
    """op_prompt_logprobs: one lm_head per sequence with the setting on and P >= 2 over its prompt rows, then one kernel
    call for all of them; nothing at all when none is on."""
    from sequoia_b200 import batch
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 1, 9, 30)]
    bt = _cpu_tree(monkeypatch, prompts, prompt_logprobs=[3, 20, None, 0])
    calls = []

    class Runner:
        logits = "runner-logits"

        def lm_head_rows(self, start, end):
            calls.append(("lm_head", start, end))
    bt.target = type("T", (), dict(engine=type("E", (), dict(runner=Runner()))()))()
    bt.tokens = bt.plp_token = bt.plp_ids = bt.plp_top = None
    monkeypatch.setattr(batch.ops, "prompt_logprobs_ragged_",
                        lambda logits, parts, *a: calls.append(("kernel", logits, list(parts))))
    bt.op_prompt_logprobs([3, 1, 0, 2], [0, 36, 44, 56, 72])
    assert calls == [("lm_head", 0, 29), ("lm_head", 44, 48),
                     ("kernel", "runner-logits", [(3, 0, 29, 0), (0, 44, 4, 3)])]
    calls.clear()
    bt.op_prompt_logprobs([1, 2], [0, 8, 24])
    assert calls == [], "P = 1 and off: no GEMM, no launch"


# ------------------------------------------------------------------------------------------------ testbed
def test_prompt_logprobs_flag_parsing_and_refusals():
    import testbed
    ap = testbed.build_parser()
    assert testbed.batch_prompt_logprobs(ap.parse_args([])) is None
    assert testbed.batch_prompt_logprobs(ap.parse_args(["--prompt-logprobs", "5", "--batch", "2"])) == 5
    assert testbed.batch_prompt_logprobs(ap.parse_args(["--prompt-logprobs", "0", "--batch", "1", "--refill"])) == 0
    with pytest.raises(SystemExit, match="--batch"):
        testbed.batch_prompt_logprobs(ap.parse_args(["--prompt-logprobs", "5"]))
    for bad in ("21", "-1"):
        with pytest.raises(SystemExit, match="--prompt-logprobs"):
            testbed.batch_prompt_logprobs(ap.parse_args(["--prompt-logprobs", bad, "--batch", "2"]))


def test_batches_and_refill_report_prompt_perplexity(monkeypatch, capsys):
    import testbed
    import sequoia_b200.batch as batch
    built, admitted = [], []

    class Tree:
        def __init__(self, draft, target, chunk, gm, policy, **kw):
            built.append(kw.get("prompt_logprobs", "absent"))
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

        def prompt_logprobs(self, b):
            n = self.lens[b] - 1
            return torch.full((n,), -0.5 * (b + 1)), torch.zeros(n, 3, dtype=torch.long), torch.zeros(n, 3)
    monkeypatch.setattr(batch, "BatchTree", Tree)
    monkeypatch.setattr(testbed.torch.cuda, "synchronize", lambda *a: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)

    class Eng:
        def clear_kv(self):
            pass
    prompts = [torch.tensor([i, 1]) for i in range(4)]
    res = testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, prompt_logprobs=3)
    assert res["mean_prompt_logprob"] == [-0.5, -1.0, -0.5, -1.0]
    assert res["prompt_perplexity"] == pytest.approx([math.exp(0.5), math.e, math.exp(0.5), math.e])
    assert "prompt 3: mean prompt-token logprob -1.0000, perplexity 2.718" in capsys.readouterr().out
    res = testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2)
    assert "mean_prompt_logprob" not in res and built == [3, 3, "absent", "absent"]
    built.clear()
    res = testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, refill=True, prompt_logprobs=0)
    assert built == [0] and len(admitted) == 2 and not any("prompt_logprobs" in kw for kw in admitted)
    assert res["mean_prompt_logprob"] == [-0.5, -1.0, -0.5, -1.0]
