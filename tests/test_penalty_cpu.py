"""Host-side pieces of the per-sequence penalties that need no GPU: the CPU statement (oracle/penalty.py) against a
brute-force restatement with a dict of counts per row and float32 scalars, the refusals of BatchTree's penalties and of
the C entry point, the device values a tree keeps per slot through admissions, and testbed.py's penalty flags."""
import numpy as np
import pytest
import torch

import cases
from oracle.penalty import penalize_rows
from test_stop_cpu import _cpu_tree

F16 = torch.float16
GM128 = "A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"   # config 2: 128 nodes


def _brute_row(row, tokens_b, P, L, mask01, k, rep, freq, pres):
    """Row k in Python: a dict of (c_all, c_out) per id over the committed slots and node k's path, numpy float32
    arithmetic one operation at a time."""
    V = row.shape[0]
    slots = list(range(P)) + [P - 1 + j for j in range(1, mask01.shape[0]) if bool(mask01[k, j])]
    counts = {}
    for s in slots:
        t = int(tokens_b[s])
        if 0 <= t < V:
            ca, co = counts.get(t, (0, 0))
            counts[t] = (ca + 1, co + (s >= L))
    out = row.clone()
    rho, f, p = np.float32(rep), np.float32(freq), np.float32(pres)
    for t, (ca, co) in counts.items():
        x = np.float32(float(row[t]))
        if not np.isfinite(x):
            continue
        with np.errstate(over="ignore"):
            if ca > 0:
                x = np.float32(x * rho) if x < 0 else np.float32(x / rho)
            if co > 0:
                x = np.float32(x - np.float32(f * np.float32(co)))
                x = np.float32(x - p)
        x = min(max(x, np.float32(-65504.0)), np.float32(65504.0))
        out[t] = torch.tensor(float(np.float16(x)), dtype=F16)
    return out


def _case(gm, B, V, M, seed, P=None, L=None, vocab_hi=None):
    """Random logits (with -inf, +inf and NaN entries), tokens drawn from a small id range so ids repeat across the
    history and the path, and per-sequence P and L."""
    g = torch.Generator().manual_seed(seed)
    S = gm["size"]
    x = (torch.randn(B * S + 2, V, generator=g) * 4).to(F16)
    x[0, 3], x[1, 5], x[2, 7] = float("-inf"), float("inf"), float("nan")
    tokens = torch.randint(0, vocab_hi or min(V, 40), (B, M), generator=g)
    Ps = P or [int(torch.randint(2, M - S + 2, (1,), generator=g)) for _ in range(B)]
    Ls = L or [max(1, p - int(torch.randint(0, 30, (1,), generator=g))) for p in Ps]
    return x, tokens, Ps, Ls


def _check(gm, B, V, M, seed, reps, freqs, press, **kw):
    x, tokens, Ps, Ls = _case(gm, B, V, M, seed, **kw)
    got = penalize_rows(x, tokens, Ps, Ls, gm["mask"], reps, freqs, press)
    S = gm["size"]
    for b in range(B):
        for k in range(S):
            want = _brute_row(x[b * S + k], tokens[b], Ps[b], Ls[b], gm["mask"], k, reps[b], freqs[b], press[b])
            assert torch.equal(got[b * S + k].view(torch.int16), want.view(torch.int16)), (b, k)
    assert torch.equal(got[B * S:].view(torch.int16), x[B * S:].view(torch.int16)), "rows from B*S on untouched"
    return x, got


def _f32(v):
    return float(np.float32(v))


@pytest.mark.parametrize("gm_name", ["L40_growmaps/4x4-tree.pt", "L40_growmaps/2x8-tree.pt", "L40_growmaps/16-chain.pt",
                                     "L40_growmaps/1x16-tree.pt", GM128])
def test_oracle_matches_brute_force(gm_name):
    gm = cases.load_growmap(gm_name)
    reps, freqs, press = [_f32(1.3), _f32(0.5), 1.0], [_f32(0.7), 0.0, _f32(-0.7)], [_f32(0.5), _f32(-0.7), 0.0]
    V = 64
    x, got = _check(gm, 3, V, gm["size"] + 80, 5, reps, freqs, press)
    assert not torch.equal(got[:gm["size"]].view(torch.int16), x[:gm["size"]].view(torch.int16))


def test_oracle_saturates_and_keeps_non_finite():
    gm = cases.load_growmap("L40_growmaps/4x4-tree.pt")
    for reps, freqs, press in (([_f32(1e-30), 65504.0], [65504.0, -65504.0], [-65504.0, 65504.0]),
                               ([_f32(1e-45), _f32(0.5)], [_f32(-0.7), _f32(0.7)], [_f32(0.7), _f32(-0.7)])):
        x, got = _check(gm, 2, 64, 60, 7, reps, freqs, press)
        assert bool(torch.isfinite(got[torch.isfinite(x)]).all()), "a finite logit stays finite"
        assert torch.equal(got[0, 3].view(torch.int16), x[0, 3].view(torch.int16))
        assert torch.equal(got[1, 5].view(torch.int16), x[1, 5].view(torch.int16)) and bool(torch.isnan(got[2, 7]))


def test_oracle_no_output_yet_and_ids_outside_the_vocabulary():
    """P = L (nothing generated: only the path counts as output), and prompt ids >= V or < 0 (ignored)."""
    gm = cases.load_growmap("L40_growmaps/2x8-tree.pt")
    x, tokens, _, _ = _case(gm, 2, 64, 80, 9)
    tokens[0, :5] = torch.tensor([64, 70, 10 ** 6, -1, 63])
    Ps = [30, 41]
    got = penalize_rows(x, tokens, Ps, Ps, gm["mask"], [_f32(1.3)] * 2, [_f32(0.4)] * 2, [_f32(0.2)] * 2)
    S = gm["size"]
    for b in range(2):
        for k in range(S):
            want = _brute_row(x[b * S + k], tokens[b], Ps[b], Ps[b], gm["mask"], k, _f32(1.3), _f32(0.4), _f32(0.2))
            assert torch.equal(got[b * S + k].view(torch.int16), want.view(torch.int16))
    # row 0 of sequence 0 (the root: no path) has no output token, so only the repetition penalty applies
    t = int(tokens[0, 6])
    x0, rho = np.float32(float(x[0, t])), np.float32(_f32(1.3))
    assert float(got[0, t]) == float(np.float16(x0 * rho if x0 < 0 else x0 / rho))


def test_oracle_neutral_and_frozen_sequences_untouched():
    gm = cases.load_growmap("L40_growmaps/4x4-tree.pt")
    x, tokens, Ps, Ls = _case(gm, 3, 64, 60, 11)
    got = penalize_rows(x, tokens, Ps, Ls, gm["mask"], [1.0, _f32(1.3), _f32(1.3)], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0],
                        frozen=[False, True, False])
    S = gm["size"]
    assert torch.equal(got[:2 * S].view(torch.int16), x[:2 * S].view(torch.int16))
    assert not torch.equal(got[2 * S:3 * S].view(torch.int16), x[2 * S:3 * S].view(torch.int16))


# ------------------------------------------------------------------------------------------------ validation
def test_check_penalty():
    from sequoia_b200.batch import _penalties, check_penalty
    for ok in (1, 1.0, 0.5, 65504, 1e-30, np.float32(1.3), np.int64(2)):
        assert check_penalty("repetition_penalty", ok) == _f32(float(ok))
    for bad in (0, 0.0, -1.0, 65505.0, 1e-50, float("inf"), float("nan"), True, "1.2", None, [1.0]):
        with pytest.raises(ValueError, match="repetition_penalty"):
            check_penalty("repetition_penalty", bad)
    for name in ("frequency_penalty", "presence_penalty"):
        for ok in (0, -0.7, 0.7, 65504.0, -65504.0):
            assert check_penalty(name, ok) == _f32(ok)
        for bad in (65504.5, -70000.0, float("-inf"), float("nan"), False, "0", None, 1e300):
            with pytest.raises(ValueError, match=name):
                check_penalty(name, bad)
    assert _penalties("presence_penalty", 0.5, 3) == [0.5] * 3
    assert _penalties("repetition_penalty", [1.0, 1.5], 2) == [1.0, 1.5]
    with pytest.raises(ValueError, match="3 values for 2"):
        _penalties("frequency_penalty", [0.1, 0.2, 0.3], 2)


def test_constructor_refuses_bad_penalties():
    from sequoia_b200.batch import BatchTree
    prompts = [torch.zeros(3), torch.zeros(4)]
    for kw in (dict(repetition_penalty=0.0), dict(repetition_penalty=[1.0, -2.0]), dict(frequency_penalty=True),
               dict(presence_penalty=float("nan")), dict(presence_penalty=[0.1]), dict(frequency_penalty=1e5),
               dict(repetition_penalty=1.1, max_length=4097)):
        with pytest.raises(ValueError):
            BatchTree(None, None, prompts, {}, **kw)


def test_admit_refuses_bad_penalties(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7)]
    bt = _cpu_tree(monkeypatch, prompts)
    graphs = dict(bt.graphs)
    for kw in (dict(repetition_penalty=0.0), dict(repetition_penalty=False), dict(frequency_penalty=float("inf")),
               dict(presence_penalty=-65505.0), dict(presence_penalty="0.5")):
        with pytest.raises(ValueError):
            bt.admit(0, torch.ones(6, dtype=torch.long), **kw)
    bt.M = 4097                                         # a tree longer than the penalty kernels count
    with pytest.raises(ValueError, match="at most 4096"):
        bt.admit(0, torch.ones(6, dtype=torch.long), presence_penalty=0.5)
    assert bt.repetition_penalty == [1.0] * 2 and bt.presence_penalty == [0.0] * 2 and not bt.use_penalty
    assert bt.graphs == graphs and bt.frozen == [True, True], "a refusal changes nothing"
    bt.admit(0, torch.ones(6, dtype=torch.long))        # neutral: allowed at any length
    assert not bt.use_penalty


def test_device_penalties_of_a_tree(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    assert not bt.use_penalty and bt.pen_scratch is None
    assert bt.rep_dev.tolist() == [1.0] * 3 and bt.rep_dev.dtype == torch.float32
    assert bt.freq_dev.tolist() == [0.0] * 3 and bt.pres_dev.tolist() == [0.0] * 3
    assert bt.prompt_len_dev.tolist() == [5, 7, 9] and bt.prompt_len_dev.dtype == torch.int32
    bt = _cpu_tree(monkeypatch, prompts, repetition_penalty=[1.0, 1.3, 1.0], presence_penalty=0.5)
    assert bt.use_penalty
    assert bt.rep_dev.tolist() == [1.0, _f32(1.3), 1.0] and bt.pres_dev.tolist() == [0.5] * 3
    assert bt.repetition_penalty == [1.0, _f32(1.3), 1.0], "host values are the device's fp32 values"
    assert _cpu_tree(monkeypatch, prompts, frequency_penalty=-0.25).use_penalty
    assert not _cpu_tree(monkeypatch, prompts, frequency_penalty=-0.0).use_penalty, "-0 is neutral"


def test_admissions_update_the_rows_and_recapture_once(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    bt.admit(0, torch.ones(6, dtype=torch.long))
    assert not bt.use_penalty and bt.graphs == {"draft": 1, "steady": 2, "post": 3}, "neutral: no recapture"
    assert bt.prompt_len_dev.tolist() == [6, 7, 9]
    bt.admit(1, torch.ones(12, dtype=torch.long), repetition_penalty=1.2, frequency_penalty=0.3)
    assert bt.use_penalty and bt.graphs == {"draft": 1}, "the first non-neutral admission drops steady and post once"
    assert bt.pen_scratch.numel() == 3 * (3 * bt.M + 1) and bt.pen_scratch.dtype == torch.int32
    assert bt.rep_dev.tolist() == [1.0, _f32(1.2), 1.0] and bt.freq_dev.tolist() == [0.0, _f32(0.3), 0.0]
    assert bt.prompt_len_dev.tolist() == [6, 12, 9]
    bt.graphs = {"draft": 1, "steady": 4, "post": 5}
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long), presence_penalty=2.0)
    assert bt.rep_dev[1] == _f32(1.2) and bt.freq_dev[1] == _f32(0.3) and bt.pres_dev[1] == 2.0, "previous values kept"
    assert int(bt.prompt_len_dev[1]) == 10, "a re-admitted slot counts its new prompt only"
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long), repetition_penalty=1, frequency_penalty=0, presence_penalty=0)
    assert bt.rep_dev[1] == 1.0 and bt.freq_dev[1] == 0.0 and bt.pres_dev[1] == 0.0
    bt.admit(2, torch.ones(4, dtype=torch.long), repetition_penalty=3.0)
    assert bt.graphs == {"draft": 1, "steady": 4, "post": 5} and bt.use_penalty, "penalties stay on, no recapture"
    assert bt.repetition_penalty == [1.0, 1.0, 3.0] and bt.prompt_len_dev.tolist() == [6, 10, 4]


# ------------------------------------------------------------------------------------------------ C entry point
def test_penalty_entry_point_refuses_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    f = 256                                             # a non-null address: every case is refused before any launch

    def call(logits=f, ld=32000, V=32000, tokens=f, ld_seq=384, state=f, plen=f, bits=f, words=4, S=128, rep=f, freq=f,
             pres=f, scratch=f, words_scratch=10 ** 6, B=2):
        return lib.sq_penalize_rows_batch(logits, ld, V, tokens, ld_seq, state, plen, bits, words, S, rep, freq, pres,
                                          scratch, words_scratch, B, None)
    c0 = lib.sq_launch_count()
    cases_ = [(dict(logits=None), b"null array"), (dict(tokens=None), b"null array"), (dict(state=None), b"null array"),
              (dict(plen=None), b"null array"), (dict(bits=None), b"null array"), (dict(rep=None), b"null array"),
              (dict(freq=None), b"null array"), (dict(pres=None), b"null array"), (dict(scratch=None), b"null array"),
              (dict(B=0), b"B=0"), (dict(B=9), b"B=9"), (dict(V=32004, ld=32008), b"V=32004"),
              (dict(V=131080, ld=131080), b"V=131080"), (dict(V=0), b"V=0"), (dict(ld=31999), b"ld=31999"),
              (dict(S=0, words=0), b"S=0"), (dict(S=128, words=5), b"tree_words=5"),
              (dict(S=1025, words=33), b"S=1025"), (dict(ld_seq=4097), b"ld_seq=4097"), (dict(ld_seq=0), b"ld_seq=0"),
              (dict(words_scratch=2 * (3 * 384 + 1) - 1), b"scratch")]
    for kw, msg in cases_:
        assert call(**kw) == -1 and msg in lib.sq_last_error(), (kw, msg, lib.sq_last_error())
    assert lib.sq_launch_count() == c0, "refused before any launch"


# ------------------------------------------------------------------------------------------------ testbed flags
def test_penalty_flags_parsing_and_refusals():
    import testbed
    ap = testbed.build_parser()
    assert testbed.batch_penalties(ap.parse_args([])) == {}
    assert testbed.batch_penalties(ap.parse_args(["--repetition-penalty", "1", "--presence-penalty", "0"])) == {}
    got = testbed.batch_penalties(ap.parse_args(["--repetition-penalty", "1.1", "--presence-penalty", "0.5", "--batch",
                                                 "2"]))
    assert got == dict(repetition_penalty=_f32(1.1), frequency_penalty=0.0, presence_penalty=0.5)
    assert testbed.batch_penalties(ap.parse_args(["--frequency-penalty", "0.2", "--batch", "1", "--refill"]))
    for flag in ("--repetition-penalty", "--frequency-penalty", "--presence-penalty"):
        with pytest.raises(SystemExit, match="with --batch"):
            testbed.batch_penalties(ap.parse_args([flag, "0.5"]))
    with pytest.raises(SystemExit, match="repetition-penalty"):
        testbed.batch_penalties(ap.parse_args(["--repetition-penalty", "0", "--batch", "2"]))
    with pytest.raises(SystemExit, match="frequency-penalty"):
        testbed.batch_penalties(ap.parse_args(["--frequency-penalty", "nan", "--batch", "2"]))
    with pytest.raises(SystemExit, match="presence-penalty"):
        testbed.batch_penalties(ap.parse_args(["--presence-penalty", "1e6", "--batch", "2"]))


def test_batches_and_refill_get_the_penalties(monkeypatch):
    """Chunked batches are built with the penalties; refill admissions pass none, so each slot keeps its values."""
    import testbed
    import sequoia_b200.batch as batch
    built, admitted = [], []

    class Tree:
        def __init__(self, draft, target, chunk, gm, policy, **kw):
            built.append({k: v for k, v in kw.items() if k.endswith("_penalty")})
            self.frozen = [False] * len(chunk)

        def admit(self, b, prompt, **kw):
            admitted.append(kw)
            self.frozen[b] = False

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
    prompts = [torch.tensor([i, 1]) for i in range(4)]
    pen = dict(repetition_penalty=1.1, frequency_penalty=0.0, presence_penalty=0.5)
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, penalties=pen)
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2)
    assert built == [pen, pen, {}, {}]
    built.clear()
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, refill=True, penalties=pen)
    assert built == [pen] and len(admitted) == 2 and not any(k.endswith("_penalty") for kw in admitted for k in kw)
