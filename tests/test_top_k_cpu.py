"""Host-side pieces of the top-k filter that need no GPU: the CPU statement (oracle/top_k.py) against a brute-force
ranking, the refusals of BatchTree's top_k and of the C entry points, the device values a tree keeps per slot, and
testbed.py's --top-k."""
import pytest
import torch

import cases  # noqa: F401  (puts the repository root on sys.path)
from oracle.top_k import top_k_filter

NEG_INF = float("-inf")


def _brute(row: torch.Tensor, k: int) -> torch.Tensor:
    """Keep the k first of the indices ordered by (value descending, index ascending), in Python floats."""
    vals = [float(v) for v in row]
    order = sorted(range(len(vals)), key=lambda i: (-vals[i], i))
    out = torch.full_like(row, NEG_INF)
    for i in order[:k]:
        out[i] = row[i]
    return out


def _rows():
    g = torch.Generator().manual_seed(11)
    rand = (torch.randn(6, 200, generator=g) * 3).to(torch.float16)
    ties = torch.randint(-3, 4, (6, 200), generator=g).to(torch.float16)      # 7 values: big tie groups everywhere
    inf = rand.clone()
    inf[:, ::3] = NEG_INF                                                     # 67 of 200 already -inf
    inf[1, :190] = NEG_INF                                                    # 10 finite entries
    return {"random": rand, "ties": ties, "inf": inf}


@pytest.mark.parametrize("kind", ["random", "ties", "inf"])
@pytest.mark.parametrize("k", [1, 2, 7, 50, 133, 150, 199])
def test_oracle_matches_brute_force(kind, k):
    x = _rows()[kind]
    got = top_k_filter(x, k)
    for r in range(x.shape[0]):
        assert torch.equal(got[r], _brute(x[r], k)), (kind, k, r)
        assert int((got[r] == x[r]).sum()) == k or bool(torch.isinf(x[r]).any())
    finite = ~torch.isinf(x)
    assert bool((~torch.isinf(got[finite.sum(-1) <= k]) == finite[finite.sum(-1) <= k]).all()), \
        "a row with at most k finite entries loses nothing finite"


def test_oracle_k1_is_lowest_index_argmax():
    x = _rows()["ties"]
    got = top_k_filter(x, 1)
    for r in range(x.shape[0]):
        m = x[r].max()
        first = int((x[r] == m).nonzero()[0])
        assert (~torch.isinf(got[r])).nonzero().flatten().tolist() == [first]


@pytest.mark.parametrize("k", [0, 200, 201, 10 ** 6])
def test_oracle_off_values_leave_the_row(k):
    x = _rows()["random"]
    assert torch.equal(top_k_filter(x, k).view(torch.int16), x.view(torch.int16))


def test_oracle_signed_zeros_tie():
    """-0 and +0 are equal values: they rank by index, as in torch.sort."""
    x = torch.tensor([[-1.0, -0.0, 0.0, -0.0]], dtype=torch.float16)
    for k, kept in ((1, [1]), (2, [1, 2]), (3, [1, 2, 3])):
        got = top_k_filter(x, k)
        assert (~torch.isinf(got[0])).nonzero().flatten().tolist() == kept
        assert torch.equal(got.view(torch.int16)[0, kept], x.view(torch.int16)[0, kept])


# ------------------------------------------------------------------------------------------------ validation
def test_check_top_k():
    import numpy as np
    from sequoia_b200.batch import _top_ks, check_top_k
    for ok in (0, 1, 50, 131072, 10 ** 12, np.int64(7)):
        assert check_top_k(ok) == int(ok)
    for bad in (-1, 1.5, 2.0, True, False, "5", None):
        with pytest.raises(ValueError, match="top_k"):
            check_top_k(bad)
    assert _top_ks(5, 3) == [5, 5, 5] and _top_ks([0, 20], 2) == [0, 20]
    with pytest.raises(ValueError, match="3 values for 2"):
        _top_ks([1, 2, 3], 2)
    with pytest.raises(ValueError, match="top_k"):
        _top_ks([1, -2], 2)


def test_constructor_and_admit_refuse_bad_top_k():
    from sequoia_b200.batch import BatchTree
    prompts = [torch.zeros(3), torch.zeros(4)]
    for bad in (-1, 1.5, True, [1]):
        with pytest.raises(ValueError):
            BatchTree(None, None, prompts, {}, top_k=bad)
    bt = BatchTree.__new__(BatchTree)
    bt.B, bt.M, bt.S, bt.seeded = 2, 64, 9, False
    bt.policies, bt.frozen = ["spec", "spec"], [True, False]
    bt.temps, bt.top_ps, bt.top_ks = [0.6] * 2, [1.0] * 2, [0, 0]
    for bad in (-1, 1.5, True):
        with pytest.raises(ValueError, match="top_k"):
            bt.admit(0, torch.zeros(10, dtype=torch.long), top_k=bad)
    assert bt.top_ks == [0, 0] and bt.frozen == [True, False], "a refusal changes nothing"


def test_device_top_k_of_a_tree(monkeypatch):
    """The constructor's host-side values: top_k is 0 on the device for greedy slots and min(k, V) otherwise, and the
    filter is needed only for a sampling slot with 0 < top_k < V.  (torch.tensor(..., device=) is redirected to the
    CPU.)"""
    import sequoia_b200.batch as batch
    real_tensor = torch.tensor

    class Stop(Exception):
        pass

    def stop(*a, **k):
        raise Stop
    monkeypatch.setattr(batch.torch, "tensor", lambda data, dtype=None, device=None: real_tensor(data, dtype=dtype))
    monkeypatch.setattr(batch.torch, "zeros", stop)                  # the first device allocation after the arrays
    monkeypatch.setattr(batch, "_Static", lambda gm, dev: type("St", (), dict(S=9))())
    monkeypatch.setattr(batch, "check_vocab", lambda pol, V: None)

    class Eng:
        def __init__(self):
            self.engine = type("E", (), dict(batch_size=3, max_length=64))()
            self.engine.model_config = type("C", (), dict(vocab_size=32000))()
            self.device = "cuda:0"

    def build(policy, top_k):
        bt = batch.BatchTree.__new__(batch.BatchTree)
        with pytest.raises(Stop):
            batch.BatchTree.__init__(bt, Eng(), Eng(), [torch.ones(5, dtype=torch.long)] * 3, {}, policy=policy,
                                     top_k=top_k, max_length=64)
        return bt
    bt = build(["greedy", "spec", "spec"], [20, 0, 10 ** 9])
    assert bt.top_k_dev.tolist() == [0, 0, 32000] and bt.top_k_dev.dtype == torch.int32
    assert bt.top_ks == [20, 0, 10 ** 9]
    assert not bt.use_top_k, "only a greedy slot has 0 < top_k < V: no filter"
    bt = build("spec", 50)
    assert bt.use_top_k and bt.top_k_dev.tolist() == [50, 50, 50]
    assert not build("spec", 0).use_top_k and not build("spec", 32000).use_top_k


# ------------------------------------------------------------------------------------------------ C entry points
def test_top_k_entry_points_refuse_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    fake = 256                                          # a non-null address: every case is refused before any launch
    c0 = lib.sq_launch_count()
    for call, msg in ((lambda: lib.sq_top_k_filter(fake, 32000, 4, 32000, -1, None), b"k=-1"),
                      (lambda: lib.sq_top_k_filter(fake, 32004, 4, 32004, 5, None), b"V=32004"),
                      (lambda: lib.sq_top_k_filter(fake, 131080, 4, 131080, 5, None), b"V=131080"),
                      (lambda: lib.sq_top_k_filter_per_seq(fake, 32000, 4, 32000, None, 2, None), b"null top_k"),
                      (lambda: lib.sq_top_k_filter_per_seq(fake, 32000, 6, 32000, fake, 4, None), b"does not divide"),
                      (lambda: lib.sq_top_k_filter_per_seq(fake, 32000, 4, 32000, fake, 0, None), b"does not divide"),
                      (lambda: lib.sq_top_k_filter_per_seq(fake, 131080, 4, 131080, fake, 2, None), b"V=131080")):
        assert call() == -1 and msg in lib.sq_last_error(), (msg, lib.sq_last_error())
    for k in (0, 32000, 40000):                         # off: nothing to launch
        assert lib.sq_top_k_filter(fake, 32000, 4, 32000, k, None) == 0
    assert lib.sq_launch_count() == c0, "refused or off before any launch"


# ------------------------------------------------------------------------------------------------ testbed --top-k
def test_top_k_flag_parsing_and_refusals():
    import testbed
    ap = testbed.build_parser()
    assert ap.parse_args([]).top_k == 0 and testbed.batch_top_k(ap.parse_args([])) == 0
    assert testbed.batch_top_k(ap.parse_args(["--top-k", "20", "--batch", "2"])) == 20
    assert testbed.batch_top_k(ap.parse_args(["--top-k", "20", "--batch", "1", "--refill"])) == 20
    with pytest.raises(SystemExit, match="with --batch"):
        testbed.batch_top_k(ap.parse_args(["--top-k", "20"]))
    with pytest.raises(SystemExit, match=">= 0"):
        testbed.batch_top_k(ap.parse_args(["--top-k", "-3", "--batch", "2"]))


def test_chunked_batches_get_the_top_k(monkeypatch):
    import testbed
    import sequoia_b200.batch as batch
    built = []

    class Tree:
        def __init__(self, draft, target, chunk, gm, policy, top_k=0, **kw):
            built.append(top_k)
            self.frozen = [True] * len(chunk)
    monkeypatch.setattr(batch, "BatchTree", Tree)
    monkeypatch.setattr(testbed.torch.cuda, "synchronize", lambda *a: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)

    class Eng:
        def clear_kv(self):
            pass
    prompts = [torch.tensor([i, 1]) for i in range(4)]
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, top_k=20)
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2)
    assert built == [20, 20, 0, 0]
