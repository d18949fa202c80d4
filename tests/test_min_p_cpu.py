"""Host-side pieces of the min-p filter that need no GPU: the CPU statement (oracle/min_p.py) against a float64 statement
of vLLM's rule and on its corner cases, the refusals of BatchTree's min_p and of the C entry point, the device values a
tree keeps per slot through admissions, and testbed.py's --min-p."""
import math
import struct

import numpy as np
import pytest
import torch

import cases  # noqa: F401  (puts the repository root on sys.path)
from oracle.min_p import min_p_filter
from test_stop_cpu import _cpu_tree

F16 = torch.float16
NEG_INF, POS_INF, NAN = float("-inf"), float("inf"), float("nan")


def _bits(x):
    return x.view(torch.int16)


def _fp32(x):
    return struct.unpack("f", struct.pack("f", x))[0]


def _kept(row):
    return (~torch.isneginf(row)).nonzero().flatten().tolist()


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("min_p", [1e-4, 0.05, 0.3, 0.9])
@pytest.mark.parametrize("T", [0.3, 0.6, 1.0, 1.7])
def test_oracle_matches_vllm_rule_away_from_the_boundary(min_p, T):
    """softmax(x / T) >= min_p * max in float64 (vLLM's statement), on entries whose log-ratio to the max is more than
    1e-3 away from ln(min_p) * T; every other entry agrees bit for bit with the input or is -inf."""
    g = torch.Generator().manual_seed(int(min_p * 1e4) + int(T * 10))
    x = (torch.randn(8, 4000, generator=g) * 3).to(F16)
    got = min_p_filter(x, min_p, T)
    xd = x.double()
    p = torch.softmax(xd / T, -1)
    want_keep = p >= min_p * p.amax(-1, keepdim=True)
    far = ((xd - xd.amax(-1, keepdim=True)) - T * math.log(min_p)).abs() > 1e-3
    keep = ~torch.isinf(got)
    assert torch.equal(keep[far], want_keep[far])
    assert torch.equal(_bits(got[keep]), _bits(x[keep])), "survivors keep their bits"
    assert bool(keep.any(-1).all()), "the max always survives"
    if min_p >= 0.05:
        assert int(keep.sum()) < keep.numel(), "the filter removes something"


def test_oracle_min_p_0_is_off():
    x = (torch.randn(4, 300, generator=torch.Generator().manual_seed(1)) * 5).to(F16)
    x[0, 3], x[1, 4] = NAN, POS_INF
    assert torch.equal(_bits(min_p_filter(x, 0.0, 0.6)), _bits(x))


def test_oracle_min_p_1_keeps_the_ties_with_the_max():
    g = torch.Generator().manual_seed(2)
    x = torch.randint(-5, 4, (6, 500), generator=g).to(F16)
    for T in (0.3, 1.0, 1.7):
        got = min_p_filter(x, 1.0, T)
        for r in range(x.shape[0]):
            assert _kept(got[r]) == (x[r] == x[r].max()).nonzero().flatten().tolist()
    z = torch.tensor([[0.0, -0.0, -1.0, 0.0]], dtype=F16)
    assert _kept(min_p_filter(z, 1.0, 0.6)[0]) == [0, 1, 3], "-0 ties with +0"


def test_oracle_non_finite_entries():
    x = torch.tensor([[1.0, NAN, NEG_INF, -20.0, 0.9],          # NaN stays, -inf stays, far entry dropped
                      [1.0, POS_INF, 3.0, NEG_INF, POS_INF],    # +inf stays, every finite entry dropped
                      [NAN, NAN, NEG_INF, NEG_INF, NEG_INF],    # no finite max: nothing changes
                      [NEG_INF] * 5], dtype=F16)
    got = min_p_filter(x, 0.1, 1.0)
    assert torch.isnan(got[0, 1]) and bool(torch.isneginf(got[0, [2, 3]]).all()) and _kept(got[0]) == [0, 1, 4]
    assert _kept(got[1]) == [1, 4] and bool(torch.isposinf(got[1, [1, 4]]).all())
    assert torch.equal(_bits(got[2:]), _bits(x[2:]))


@pytest.mark.parametrize("T,gap", [(1.0, 2.0), (0.5, 1.0)])
@pytest.mark.parametrize("m", [4.0, 5.5, -3.0])
def test_oracle_exact_boundary_is_kept(T, gap, m):
    """min_p = e^-2: thr = fp32(T) * fp32(ln e^-2) is exactly -2.0 at T = 1 and -1.0 at T = 0.5.  x = m - gap is on the
    boundary and stays; the next fp16 value below it is dropped."""
    min_p = math.exp(-2.0)
    assert _fp32(math.log(min_p)) == -2.0
    on = torch.tensor([m - gap], dtype=F16)
    below = (_bits(on) + (1 if m - gap < 0 else -1)).view(F16)             # the next fp16 value below (m - gap != 0)
    assert float(below) < float(on) and float(below.float().to(torch.float64)) < m - gap
    x = torch.cat([torch.tensor([m], dtype=F16), on, below, torch.tensor([m - gap / 2], dtype=F16)]).view(1, 4)
    assert _kept(min_p_filter(x, min_p, T)[0]) == [0, 1, 3]


# ------------------------------------------------------------------------------------------------ validation
def test_check_min_p():
    from sequoia_b200.batch import _min_ps, check_min_p
    for ok in (0, 0.0, 1e-300, 0.05, 1, 1.0, np.float32(0.25), np.float64(0.5)):
        assert check_min_p(ok) == float(ok)
    for bad in (True, False, NAN, POS_INF, NEG_INF, -1e-9, -0.5, 1.0000001, 2, "0.1", None, torch.tensor(0.1)):
        with pytest.raises(ValueError, match="min_p"):
            check_min_p(bad)
    assert _min_ps(0.1, 3) == [0.1] * 3 and _min_ps([0, 0.2], 2) == [0.0, 0.2]
    with pytest.raises(ValueError, match="3 values for 2"):
        _min_ps([0.1, 0.2, 0.3], 2)
    with pytest.raises(ValueError, match="min_p"):
        _min_ps([0.1, 1.5], 2)


def test_constructor_and_admit_refuse_bad_min_p(monkeypatch):
    from sequoia_b200.batch import BatchTree
    prompts = [torch.zeros(3), torch.zeros(4)]
    for bad in (True, NAN, POS_INF, -0.1, 1.5, [0.1], [0.1, NAN]):
        with pytest.raises(ValueError, match="min_p"):
            BatchTree(None, None, prompts, {}, min_p=bad)
    bt = _cpu_tree(monkeypatch, [torch.ones(n, dtype=torch.long) for n in (5, 7)])
    graphs = dict(bt.graphs)
    for bad in (True, NAN, NEG_INF, -0.1, 1.5, "0.1"):
        with pytest.raises(ValueError, match="min_p"):
            bt.admit(0, torch.ones(6, dtype=torch.long), min_p=bad)
    assert bt.min_ps == [0.0, 0.0] and not bt.use_min_p and bt.graphs == graphs and bt.frozen == [True, True], \
        "a refusal changes nothing"


# ------------------------------------------------------------------------------------------------ device values
def test_device_min_p_of_a_tree(monkeypatch):
    """log_min_p_dev is -inf for an off or greedy slot and fp32(math.log(min_p)) otherwise; the filter is needed only
    for a sampling slot with min_p > 0."""
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    assert bt.min_ps == [0.0] * 3 and not bt.use_min_p
    assert bt.log_min_p_dev.tolist() == [NEG_INF] * 3 and bt.log_min_p_dev.dtype == torch.float32
    bt = _cpu_tree(monkeypatch, prompts, policy=["greedy", "spec", "spec"], min_p=[0.2, 0.0, 0.05])
    assert bt.min_ps == [0.2, 0.0, 0.05] and bt.use_min_p
    assert bt.log_min_p_dev.tolist() == [NEG_INF, NEG_INF, _fp32(math.log(0.05))]
    assert not _cpu_tree(monkeypatch, prompts, policy=["greedy", "spec", "spec"], min_p=[0.2, 0.0, 0.0]).use_min_p, \
        "only a greedy slot has min_p > 0: no filter"
    bt = _cpu_tree(monkeypatch, prompts, min_p=1.0)
    assert bt.log_min_p_dev.tolist() == [0.0] * 3 and bt.use_min_p


def test_admissions_update_the_value_and_recapture_once(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts, policy=["spec", "greedy", "spec"])
    bt.mixed, bt.greedy = True, False
    base = {"draft": 1, "steady": 2, "post": 3}
    bt.admit(1, torch.ones(6, dtype=torch.long), min_p=0.3)
    assert not bt.use_min_p and bt.graphs == base, "a greedy admission never adds the filter"
    assert bt.min_ps[1] == 0.3 and bt.log_min_p_dev[1].item() == NEG_INF
    bt.admit(0, torch.ones(6, dtype=torch.long), min_p=0.0)
    assert not bt.use_min_p and bt.graphs == base, "min_p 0: no recapture"
    bt.admit(2, torch.ones(6, dtype=torch.long), min_p=0.1)
    assert bt.use_min_p and bt.graphs == {"draft": 1}, "the first spec admission with min_p > 0 drops steady and post"
    assert bt.log_min_p_dev[2].item() == _fp32(math.log(0.1))
    bt.graphs = {"draft": 1, "steady": 4, "post": 5}
    bt.frozen[2] = True
    bt.admit(2, torch.ones(6, dtype=torch.long))
    assert bt.min_ps[2] == 0.1 and bt.log_min_p_dev[2].item() == _fp32(math.log(0.1)), "the default keeps it"
    bt.frozen[2] = True
    bt.admit(2, torch.ones(6, dtype=torch.long), min_p=0.0)
    assert bt.log_min_p_dev[2].item() == NEG_INF
    bt.frozen[1] = True
    bt.admit(1, torch.ones(6, dtype=torch.long), policy="spec")
    assert bt.log_min_p_dev[1].item() == _fp32(math.log(0.3)), "a greedy slot's min_p applies once it samples"
    assert bt.graphs == {"draft": 1, "steady": 4, "post": 5}, "no recapture after the filter entered"


# ------------------------------------------------------------------------------------------------ C entry point
def test_min_p_entry_point_refuses_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    fake = 256                                          # a non-null address: every case is refused before any launch
    c0 = lib.sq_launch_count()
    f = lib.sq_min_p_filter_per_seq
    for call, msg in ((lambda: f(fake, 32000, 4, 32000, None, fake, 2, None), b"null log_min_p"),
                      (lambda: f(fake, 32000, 4, 32000, fake, None, 2, None), b"null log_min_p or temperature"),
                      (lambda: f(fake, 32000, 6, 32000, fake, fake, 4, None), b"does not divide"),
                      (lambda: f(fake, 32000, 4, 32000, fake, fake, 0, None), b"does not divide"),
                      (lambda: f(fake, 32000, -4, 32000, fake, fake, 2, None), b"does not divide"),
                      (lambda: f(fake, 32004, 4, 32004, fake, fake, 2, None), b"V=32004"),
                      (lambda: f(fake, 0, 4, 0, fake, fake, 2, None), b"V=0"),
                      (lambda: f(fake, 131080, 4, 131080, fake, fake, 2, None), b"V=131080")):
        assert call() == -1 and msg in lib.sq_last_error(), (msg, lib.sq_last_error())
    assert f(fake, 32000, 0, 32000, fake, fake, 2, None) == 0, "n == 0 is a no-op"
    assert lib.sq_launch_count() == c0, "refused or empty before any launch"


# ------------------------------------------------------------------------------------------------ testbed --min-p
def test_min_p_flag_parsing_and_refusals():
    import testbed
    ap = testbed.build_parser()
    assert ap.parse_args([]).min_p == 0.0 and testbed.batch_min_p(ap.parse_args([])) == 0.0
    assert testbed.batch_min_p(ap.parse_args(["--min-p", "0.1", "--batch", "2"])) == 0.1
    assert testbed.batch_min_p(ap.parse_args(["--min-p", "1", "--batch", "1", "--refill"])) == 1.0
    with pytest.raises(SystemExit, match="with --batch"):
        testbed.batch_min_p(ap.parse_args(["--min-p", "0.1"]))
    for bad in ("-0.1", "1.5", "nan", "inf"):
        with pytest.raises(SystemExit, match=r"\[0, 1\]"):
            testbed.batch_min_p(ap.parse_args(["--min-p", bad, "--batch", "2"]))


def test_chunked_batches_get_the_min_p(monkeypatch):
    import testbed
    import sequoia_b200.batch as batch
    built = []

    class Tree:
        def __init__(self, draft, target, chunk, gm, policy, min_p=0.0, **kw):
            built.append(min_p)
            self.frozen = [True] * len(chunk)
    monkeypatch.setattr(batch, "BatchTree", Tree)
    monkeypatch.setattr(testbed.torch.cuda, "synchronize", lambda *a: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)

    class Eng:
        def clear_kv(self):
            pass
    prompts = [torch.tensor([i, 1]) for i in range(4)]
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, min_p=0.1)
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2)
    assert built == [0.1, 0.1, 0.0, 0.0]
