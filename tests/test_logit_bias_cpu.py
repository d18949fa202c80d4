"""Host-side pieces of the per-sequence logit bias and allowed-token sets that need no GPU: the CPU statement
(oracle/logit_bias.py) against a brute-force numpy float32 restatement, the refusals of BatchTree's logit_bias /
allowed_token_ids and of the C entry point, the bitmask packing, the device rows a tree keeps per slot through admissions,
and testbed.py's --logit-bias / --allowed-token-ids."""
import numpy as np
import pytest
import torch

import cases  # noqa: F401  (puts the repository root on sys.path)
from oracle.logit_bias import process_rows
from test_stop_cpu import _cpu_tree

F16 = torch.float16


def _f32(v):
    return float(np.float32(v))


def _brute_row(row, allowed, bias):
    """One row in Python: the mask entry by entry, then each (id, bias) with numpy float32 scalars."""
    V = row.shape[0]
    out = row.clone()
    if allowed is not None:
        ok = set(int(t) for t in allowed)
        for t in range(V):
            if t not in ok:
                out[t] = float("-inf")
    for t, beta in bias or ():
        if not 0 <= t < V or (allowed is not None and t not in ok):
            continue
        x = np.float32(float(out[t]))
        if not np.isfinite(x):
            continue
        with np.errstate(over="ignore"):
            x = np.float32(x + np.float32(beta))
        x = min(max(x, np.float32(-65504.0)), np.float32(65504.0))
        out[t] = torch.tensor(float(np.float16(x)), dtype=F16)
    return out


def _rows(B, S, V, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B * S + 2, V, generator=g) * 4).to(F16)
    x[0, 3], x[0, 4], x[0, 5] = float("-inf"), float("inf"), float("nan")      # allowed below
    x[1, 6], x[1, 7], x[1, 8] = float("-inf"), float("inf"), float("nan")      # disallowed below
    x[:, 10] = 65500.0
    x[:, 11] = -65500.0
    return x


def _check(x, S, allowed, bias, frozen=None):
    got = process_rows(x, S, allowed, bias, frozen=frozen)
    B = len(allowed)
    for b in range(B):
        for k in range(S):
            r = b * S + k
            skip = (frozen is not None and frozen[b]) or (allowed[b] is None and not bias[b])
            want = x[r] if skip else _brute_row(x[r], allowed[b], bias[b])
            assert torch.equal(got[r].view(torch.int16), want.view(torch.int16)), (b, k)
    assert torch.equal(got[B * S:].view(torch.int16), x[B * S:].view(torch.int16)), "rows from B*S on untouched"
    return got


def test_oracle_matches_brute_force():
    V, S = 64, 5
    x = _rows(3, S, V, 1)
    allowed = [tuple(range(0, 6)) + (10, 11, 20, 63), None, (0, 63)]
    bias = [((0, _f32(0.3)), (3, 5.0), (4, -5.0), (5, 1.0), (6, 100.0), (10, 100.0), (11, -100.0), (63, _f32(-1e-3))),
            ((0, -100.0), (10, 100.0), (11, -100.0), (40, _f32(1e-30)), (63, 7.5)),
            ((1, 50.0), (63, 100.0))]
    got = _check(x, S, allowed, bias)
    assert float(got[0, 10]) == 65504.0 and float(got[0, 11]) == -65504.0, "65500 + 100 saturates to 65504"
    assert torch.isinf(got[1, 6]) and torch.isinf(got[1, 7]) and torch.isinf(got[1, 8]) and got[1, 7] < 0, \
        "disallowed -inf, +inf and NaN all become -inf"
    assert bool(torch.isnan(got[0, 5])) and float(got[0, 4]) == float("inf") and float(got[0, 3]) == float("-inf"), \
        "allowed non-finite entries are left alone by the mask and the bias"
    assert float(got[0, 6]) == float("-inf"), "a bias on a disallowed id does not apply"
    assert float(got[2 * S, 1]) == float("-inf"), "id 1 is outside sequence 2's set"
    assert float(got[S, 63]) == float(np.float16(np.float32(float(x[S, 63])) + np.float32(7.5))), "id V-1"


def test_oracle_neutral_frozen_and_ties():
    V, S = 48, 3
    x = _rows(3, S, V, 2)
    got = _check(x, S, [None, (1, 2), None], [(), ((1, 2.0),), ((2, 3.0),)], frozen=[False, True, False])
    assert torch.equal(got[:2 * S].view(torch.int16), x[:2 * S].view(torch.int16)), "neutral and frozen untouched"
    assert not torch.equal(got[2 * S:3 * S].view(torch.int16), x[2 * S:3 * S].view(torch.int16))
    # a tiny bias can round away in fp16: the add is exact in fp32, the fp16 rounding returns the old value
    y = torch.full((1, 16), 1000.0, dtype=F16)
    assert torch.equal(process_rows(y, 1, [None], [((3, _f32(1e-4)),)]), y)


# ------------------------------------------------------------------------------------------------ validation
def test_check_logit_bias():
    from sequoia_b200.batch import _logit_biases, check_logit_bias
    assert check_logit_bias(None) is None and check_logit_bias({}) == () and check_logit_bias({5: 0.0, 6: -0.0}) == ()
    assert check_logit_bias({9: 1, 3: -100, np.int64(5): np.float32(0.1)}, 10) == ((3, -100.0), (5, _f32(0.1)),
                                                                                   (9, 1.0))
    assert check_logit_bias({t: 1.0 for t in range(1024)}) is not None
    assert check_logit_bias({t: (1.0 if t < 1024 else 0.0) for t in range(2000)}) is not None, "zeros do not count"
    for bad in ({-1: 1.0}, {"5": 1.0}, {True: 1.0}, {1.5: 1.0}, {5: True}, {5: "1"}, {5: None}, {5: float("nan")},
                {5: float("inf")}, {5: 100.5}, {5: -101.0}, {t: 1.0 for t in range(1025)}, [(5, 1.0)], 5, "x"):
        with pytest.raises(ValueError, match="logit_bias"):
            check_logit_bias(bad)
    with pytest.raises(ValueError, match="logit_bias"):
        check_logit_bias({32000: 1.0}, 32000)
    assert _logit_biases({1: 2.0}, 2) == [((1, 2.0),)] * 2 and _logit_biases(None, 2) == [None, None]
    assert _logit_biases([{1: 2.0}, None], 2) == [((1, 2.0),), None]
    with pytest.raises(ValueError, match="3 values for 2"):
        _logit_biases([{}, {}, None], 2)


def test_check_allowed_token_ids():
    from sequoia_b200.batch import _allowed_sets, check_allowed_token_ids
    assert check_allowed_token_ids(None) is None
    assert check_allowed_token_ids([7, 3, np.int32(5)], 8) == (3, 5, 7)
    assert check_allowed_token_ids(range(8), 8) is None and check_allowed_token_ids(set(range(8)), 9) == tuple(range(8))
    assert check_allowed_token_ids(frozenset([1])) == (1,)
    for bad in ([], set(), "12", b"12", 5, [True], [1.5], [-1], [None], [1, 1], {1: 2}):
        with pytest.raises(ValueError, match="allowed_token_ids"):
            check_allowed_token_ids(bad)
    with pytest.raises(ValueError, match="allowed_token_ids"):
        check_allowed_token_ids([32000], 32000)
    assert _allowed_sets([1, 2], 3) == [(1, 2)] * 3 and _allowed_sets(None, 2) == [None, None]
    assert _allowed_sets([[2, 1], None], 2) == [(1, 2), None] and _allowed_sets(range(4), 2) == [(0, 1, 2, 3)] * 2
    with pytest.raises(ValueError, match="1 sets for 2"):
        _allowed_sets([[1]], 2)


def test_constructor_refuses_bad_settings(monkeypatch):
    from sequoia_b200.batch import BatchTree
    prompts = [torch.zeros(3), torch.zeros(4)]
    for kw in (dict(logit_bias={5: 101.0}), dict(logit_bias=[{5: 1.0}, {"a": 1.0}]), dict(logit_bias=[{}]),
               dict(logit_bias=5), dict(allowed_token_ids=[]), dict(allowed_token_ids=[[1], []]),
               dict(allowed_token_ids="ab"), dict(allowed_token_ids=[[1], [2], [3]]), dict(allowed_token_ids=[2, 2])):
        with pytest.raises(ValueError):
            BatchTree(None, None, prompts, {}, **kw)
    for kw in (dict(logit_bias={32000: 1.0}), dict(allowed_token_ids=[[5], [32000]])):      # V = 32000
        with pytest.raises(ValueError, match="32000"):
            _cpu_tree(monkeypatch, prompts, **kw)
        monkeypatch.undo()


def test_admit_refuses_bad_settings(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7)]
    bt = _cpu_tree(monkeypatch, prompts)
    graphs = dict(bt.graphs)
    for kw in (dict(logit_bias={32000: 1.0}), dict(logit_bias={5: float("nan")}), dict(logit_bias=[(5, 1.0)]),
               dict(allowed_token_ids=[]), dict(allowed_token_ids=[32000]), dict(allowed_token_ids=[True]),
               dict(allowed_token_ids="5")):
        with pytest.raises(ValueError):
            bt.admit(0, torch.ones(6, dtype=torch.long), **kw)
    assert bt.logit_bias == [None] * 2 and bt.allowed_token_ids == [None] * 2 and not bt.use_logit_bias
    assert bt.graphs == graphs and bt.frozen == [True, True], "a refusal changes nothing"


# ------------------------------------------------------------------------------------------------ bitmask and device rows
def test_pack_token_mask():
    from sequoia_b200 import ops
    for V in (8, 40, 64, 32000, 128256):
        ids = sorted({0, V - 1, V // 2, min(31, V - 1), min(32, V - 1)})
        m = ops.pack_token_mask(ids, V)
        assert m.dtype == torch.int32 and m.shape == (ops.mask_words(V),) and ops.mask_words(V) == -(-V // 32)
        u = m.numpy().view(np.uint32)
        bits = [(int(u[t >> 5]) >> (t & 31)) & 1 for t in range(len(u) * 32)]
        assert [t for t, v in enumerate(bits) if v] == ids, V
    assert ops.pack_token_mask([31], 32).tolist() == [-(1 << 31)], "bit 31 is the int32 sign bit"
    full = ops.pack_token_mask(range(40), 40)
    assert full.tolist() == [-1, 0xff], "the padding bits from V on stay clear"


def _rows_of(bt, b):
    return (bt.allowed_dev[b].clone(), int(bt.has_mask_dev[b]), bt.bias_ids_dev[b].clone(), bt.bias_vals_dev[b].clone(),
            int(bt.n_bias_dev[b]))


def _expect(bt, b, allowed, bias):
    from sequoia_b200 import ops
    mask, has, ids, vals, n = _rows_of(bt, b)
    want_mask = ops.pack_token_mask(allowed, bt.V) if allowed is not None else torch.zeros_like(mask)
    assert torch.equal(mask, want_mask) and has == (allowed is not None), b
    bias = bias or ()
    assert n == len(bias) and ids[:n].tolist() == [t for t, _ in bias] and vals[:n].tolist() == [v for _, v in bias]
    assert not bool(ids[n:].any()) and not bool(vals[n:].any()), "entries past n_bias are zero"


def test_device_rows_of_a_tree(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    assert not bt.use_logit_bias and bt.allowed_dev is None and bt.n_bias_dev is None
    assert bt.logit_bias == [None] * 3 and bt.allowed_token_ids == [None] * 3
    for kw in (dict(logit_bias={}), dict(logit_bias={5: 0.0, 9: -0.0}), dict(allowed_token_ids=range(32000)),
               dict(logit_bias=[None, {}, {3: 0}], allowed_token_ids=[None, set(range(32000)), None])):
        nb = _cpu_tree(monkeypatch, prompts, **kw)
        assert not nb.use_logit_bias and nb.allowed_dev is None, ("neutral settings allocate nothing", kw)
        assert nb.allowed_token_ids == [None] * 3
    bt = _cpu_tree(monkeypatch, prompts, logit_bias=[{7: 1.5, 2: -100}, None, {}], allowed_token_ids=[None, None, [4, 1]])
    assert bt.use_logit_bias and bt.logit_bias == [((2, -100.0), (7, 1.5)), None, ()]
    assert bt.allowed_token_ids == [None, None, (1, 4)]
    bt._start_logit_bias()                              # (the CPU constructor stops at its first device allocation)
    assert bt.allowed_dev.shape == (3, 1000) and bt.bias_ids_dev.shape == (3, 1024)
    assert bt.bias_vals_dev.dtype == torch.float32 and bt.has_mask_dev.dtype == torch.int32
    _expect(bt, 0, None, ((2, -100.0), (7, 1.5)))
    _expect(bt, 1, None, None)
    _expect(bt, 2, (1, 4), ())


def test_admissions_update_the_rows_and_recapture_once(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    bt.admit(0, torch.ones(6, dtype=torch.long), logit_bias={3: 0.0}, allowed_token_ids=range(32000))
    assert not bt.use_logit_bias and bt.graphs == {"draft": 1, "steady": 2, "post": 3}, "neutral: no recapture"
    assert bt.allowed_dev is None and bt.logit_bias[0] == ()
    bt.admit(1, torch.ones(12, dtype=torch.long), logit_bias={9: 2.0, 4: _f32(-0.3)})
    assert bt.use_logit_bias and bt.graphs == {"draft": 1}, "the first non-neutral admission drops steady and post once"
    _expect(bt, 1, None, ((4, _f32(-0.3)), (9, 2.0)))
    _expect(bt, 0, None, ())
    bt.graphs = {"draft": 1, "steady": 4, "post": 5}
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long), allowed_token_ids=[4, 31, 32, 31999])
    _expect(bt, 1, (4, 31, 32, 31999), ((4, _f32(-0.3)), (9, 2.0)))
    assert bt.logit_bias[1] == ((4, _f32(-0.3)), (9, 2.0)), "the default keeps the previous bias"
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long))
    _expect(bt, 1, (4, 31, 32, 31999), ((4, _f32(-0.3)), (9, 2.0)))
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long), logit_bias=None)
    _expect(bt, 1, (4, 31, 32, 31999), None)
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long), allowed_token_ids=None, logit_bias={31999: 100})
    _expect(bt, 1, None, ((31999, 100.0),))
    bt.admit(2, torch.ones(4, dtype=torch.long), allowed_token_ids=[0])
    _expect(bt, 2, (0,), None)
    assert bt.graphs == {"draft": 1, "steady": 4, "post": 5} and bt.use_logit_bias, "the kernel stays, no recapture"


# ------------------------------------------------------------------------------------------------ C entry point
def test_logit_bias_entry_point_refuses_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    f = 256                                             # a non-null address: every case is refused before any launch

    def call(logits=f, ld=32000, V=32000, S=128, state=f, allowed=f, words=1000, has=f, ids=f, vals=f, n=f, B=2):
        return lib.sq_logit_bias_rows_batch(logits, ld, V, S, state, allowed, words, has, ids, vals, n, B, None)
    c0 = lib.sq_launch_count()
    cases_ = [(dict(logits=None), b"null array"), (dict(state=None), b"null array"), (dict(allowed=None), b"null array"),
              (dict(has=None), b"null array"), (dict(ids=None), b"null array"), (dict(vals=None), b"null array"),
              (dict(n=None), b"null array"), (dict(B=0), b"B=0"), (dict(B=9), b"B=9"),
              (dict(V=32004, ld=32008, words=1001), b"V=32004"), (dict(V=131080, ld=131080, words=4097), b"V=131080"),
              (dict(V=0), b"V=0"), (dict(ld=31999), b"ld=31999"), (dict(S=0), b"S=0"), (dict(S=-1), b"S=-1"),
              (dict(words=999), b"allowed_words=999"), (dict(V=40, ld=40, words=1), b"allowed_words=1")]
    for kw, msg in cases_:
        assert call(**kw) == -1 and msg in lib.sq_last_error(), (kw, msg, lib.sq_last_error())
    assert lib.sq_launch_count() == c0, "refused before any launch"


# ------------------------------------------------------------------------------------------------ testbed flags
def test_logit_bias_flags_parsing_and_refusals():
    import testbed
    ap = testbed.build_parser()
    assert testbed.batch_logit_bias(ap.parse_args([])) == {}
    got = testbed.batch_logit_bias(ap.parse_args(["--logit-bias", "5:1.5,7:-100", "--allowed-token-ids", "0-3,9,12-12",
                                                  "--batch", "2"]))
    assert got == dict(logit_bias={5: 1.5, 7: -100.0}, allowed_token_ids=(0, 1, 2, 3, 9, 12))
    assert testbed.batch_logit_bias(ap.parse_args(["--logit-bias", "5:0", "--batch", "1", "--refill"])) == \
        dict(logit_bias={})
    for flag, val in (("--logit-bias", "5:1"), ("--allowed-token-ids", "1-4")):
        with pytest.raises(SystemExit, match="with --batch"):
            testbed.batch_logit_bias(ap.parse_args([flag, val]))
    for flag, val in (("--logit-bias", "5"), ("--logit-bias", "5:200"), ("--logit-bias", "a:1"),
                      ("--logit-bias", "-3:1"), ("--logit-bias", "5:nan"), ("--allowed-token-ids", "x"),
                      ("--allowed-token-ids", "5-1"), ("--allowed-token-ids", "1,1")):
        with pytest.raises(SystemExit, match=flag):
            testbed.batch_logit_bias(ap.parse_args([f"{flag}={val}", "--batch", "2"]))


def test_batches_and_refill_get_the_settings(monkeypatch):
    """Chunked batches are built with the settings; refill admissions pass none, so each slot keeps its values."""
    import testbed
    import sequoia_b200.batch as batch
    built, admitted = [], []

    class Tree:
        def __init__(self, draft, target, chunk, gm, policy, **kw):
            built.append({k: v for k, v in kw.items() if k in ("logit_bias", "allowed_token_ids")})
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
    kw = dict(logit_bias={5: 1.0}, allowed_token_ids=(1, 5, 9))
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, logit_bias=kw)
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2)
    assert built == [kw, kw, {}, {}]
    built.clear()
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, refill=True, logit_bias=kw)
    assert built == [kw] and len(admitted) == 2
    assert not any(k in ("logit_bias", "allowed_token_ids") for a in admitted for k in a)
