"""Host-side pieces of constrained drafting that need no GPU: the exactness of the dead-child walk rule (chi-square of the
first committed token against softmax(processed target row / T) over 10^5 trials per case, in float64), the oracle's row
processing through the draft-row tables, BatchTree's constrain_draft refusals and graph bookkeeping, testbed.py's
--constrain-draft, and the refusals of sq_draft_rows_batch and of the SQ_ACCEPT_SKIP_DEAD policy bit before any launch."""
import numpy as np
import pytest
import torch

import cases  # noqa: F401  (puts the repository root on sys.path)
from oracle import constrained_draft as CD
from oracle import logit_bias as LB
from test_stop_cpu import _cpu_tree

F64 = torch.float64
N_TRIALS = 100_000


def _first_tokens(V, K, allowed, bias=(), T=0.6, seed=0, force_nan_key=False):
    """N_TRIALS draws of one node's first committed token: the draft and target rows (independent random logits) both
    get the same allowed set and bias, K children are drawn without replacement from the processed draft row, and the
    skip-rule walk runs.  -> (counts (V,), processed target row)."""
    g = torch.Generator().manual_seed(seed)
    ok = LB.allowed_vector(allowed, V)
    tgt = LB.process_row((torch.randn(V, generator=g, dtype=F64) * 2).to(torch.float16), ok, bias)
    drf = LB.process_row((torch.randn(V, generator=g, dtype=F64) * 2).to(torch.float16), ok, bias)
    rand = torch.rand(N_TRIALS, V, generator=g, dtype=F64)
    if force_nan_key:                                   # u = 1 at a masked id: key log(1) / 0 = NaN, drawn first
        masked = torch.nonzero(~ok).flatten()
        rand[torch.arange(N_TRIALS), masked[torch.randint(0, len(masked), (N_TRIALS,), generator=g)]] = 1.0
    children = CD.sample_children(drf, rand, K, T)
    if force_nan_key:
        assert bool(torch.isneginf(drf.to(F64)[children[:, 0]]).all()), "the NaN key puts a dead child first"
    r = torch.rand(N_TRIALS, K, generator=g, dtype=F64)
    noise = torch.empty(N_TRIALS, V, dtype=F64).exponential_(1.0, generator=g)
    first, _ = CD.walk_first_token(tgt, drf, children, r, noise, T)
    return torch.bincount(first, minlength=V), tgt


@pytest.mark.parametrize("case", ["support>K", "support=K", "support<K", "support1", "bias", "nan_key", "root19"])
def test_dead_child_rule_is_exact(case):
    from scipy.stats import chisquare
    V, T = 48, 0.6
    kw = {"support>K": dict(K=4, allowed=range(0, 24, 2)),
          "support=K": dict(K=6, allowed=[1, 5, 9, 20, 33, 47]),
          "support<K": dict(K=8, allowed=[3, 17, 40]),
          "support1": dict(K=4, allowed=[11]),
          "bias": dict(K=5, allowed=range(10), bias=((2, 3.0), (4, -2.5), (7, 1.25))),
          "nan_key": dict(K=6, allowed=[0, 8, 16, 30], force_nan_key=True),
          "root19": dict(K=19, allowed=[2, 6, 7, 12, 13, 21, 22], T=1.0, V=64)}[case]
    V, T = kw.pop("V", V), kw.pop("T", T)
    counts, tgt = _first_tokens(V, kw.pop("K"), kw.pop("allowed"), T=T, seed=sum(map(ord, case)), **kw)
    p = torch.softmax(tgt.to(F64) / T, 0)
    assert int(counts[p == 0].sum()) == 0, "no token outside the processed row's support"
    keep = p > 0
    obs, exp = counts[keep].double(), p[keep] * N_TRIALS
    if len(obs) == 1:
        assert int(obs[0]) == N_TRIALS
        return
    _, pval = chisquare(obs.numpy(), exp.numpy())
    assert pval > 1e-3, (case, pval, obs.tolist(), exp.tolist())


def test_without_the_rule_the_residual_turns_nan():
    """A node whose draft row has 2 live entries and 4 children, both live children rejected: with the rule the bonus
    comes from the finite residual; without it the walk reaches a dead child with an all -inf q and the residual turns
    NaN (the NaN flag's "nan" finish)."""
    V, T = 32, 0.6
    tgt = LB.process_row(torch.linspace(-2, 2, V).to(torch.float16), LB.allowed_vector([3, 9, 20], V), ())
    drf = LB.process_row(torch.linspace(2, -2, V).to(torch.float16), LB.allowed_vector([3, 9], V), ())
    children = torch.tensor([[3, 9, 0, 1]])
    r = torch.ones(1, 4, dtype=F64)                     # reject every live child
    noise = torch.ones(1, V, dtype=F64)
    with_rule, acc = CD.walk_first_token(tgt, drf, children, r, noise, T)
    assert not bool(acc[0]) and int(with_rule[0]) == 20
    p = torch.softmax(tgt.to(F64) / T, 0).unsqueeze(0)
    work = drf.to(F64).unsqueeze(0).clone()
    for t in children[0].tolist():
        q = torch.softmax(work / T, -1)
        res = (p - q).clamp_min(0)
        p = res / res.sum(-1, keepdim=True)
        work[0, t] = float("-inf")
    assert bool(torch.isnan(p).any())


def test_process_draft_rows_through_the_row_tables():
    from sequoia_b200.ops import draft_row_tables
    V, B, S = 64, 2, 5
    base, step = draft_row_tables([(0, 1), (1, 2), (3, 2)], S, B, "cpu")
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B * S + 2, V, generator=g).to(torch.float16)
    allowed, bias = [[1, 2, 3], None], [None, ((5, 2.0),)]
    out = CD.process_draft_rows(x, base.tolist(), step.tolist(), [1, 2], S, allowed=allowed, bias=bias)
    for b in range(B):
        for k in range(S):
            row = int(base[k]) + b * int(step[k])
            want = LB.process_row(x[row], LB.allowed_vector(allowed[b], V), bias[b] or ()) if k in (1, 2) else x[row]
            assert torch.equal(out[row].view(torch.int16), want.view(torch.int16)), (b, k)
    assert torch.equal(out[B * S:], x[B * S:])


# ------------------------------------------------------------------------------------------------ BatchTree
def test_constrain_draft_refusals():
    from sequoia_b200.batch import BatchTree
    for v in (1, 0, None, "yes", np.bool_(True)):
        with pytest.raises(ValueError, match="constrain_draft must be a bool"):
            BatchTree(None, None, [torch.ones(3, dtype=torch.long)], {}, constrain_draft=v)


def test_neutral_tree_and_the_draft_recapture(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7)]
    plain = _cpu_tree(monkeypatch, prompts)
    assert plain.constrain_draft is False and not plain._draft_processed()
    bt = _cpu_tree(monkeypatch, prompts, constrain_draft=True)
    assert bt.constrain_draft is True and not bt._draft_processed(), "every slot neutral: nothing to process"
    assert bt.allowed_dev is None and bt.words_dev is None and bt.guide_table_dev is None, "nothing allocated"
    bt.admit(0, prompts[0], allowed_token_ids=[4, 5, 6])
    assert bt._draft_processed() and bt.graphs == {}, "the first allowed set drops the draft graph too"
    bt.graphs = {"draft": 1, "steady": 2, "post": 3}
    bt.frozen[0] = True
    bt.admit(0, prompts[0], allowed_token_ids=[7])
    assert bt.graphs == {"draft": 1, "steady": 2, "post": 3}, "later admissions recapture nothing"
    bt.admit(1, prompts[1], bad_words=[[9]])
    assert bt.graphs == {}, "a second kind drops all three once"
    # an unconstrained tree keeps its draft graph when a kind starts
    un = _cpu_tree(monkeypatch, prompts)
    un.admit(0, prompts[0], allowed_token_ids=[4, 5, 6])
    assert un.graphs == {"draft": 1} and not un._draft_processed()


def test_stop_mode_recaptures_a_draft_graph_that_bans_end_ids(monkeypatch):
    """min_tokens bans the end ids, which become the stop ids when stop mode starts: a constrained tree that bans drops
    its draft graph with the steady and post graphs, so its draft rows keep banning what its target rows ban."""
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7)]

    def tree(**kw):
        t = _cpu_tree(monkeypatch, prompts, min_tokens=[3, 0], **kw)
        t._start_ban()                                   # (the CPU constructor stops at its first device allocation,
        t.logit_bias, t.allowed_token_ids = [None] * 2, [None] * 2   # before the rest of the host state)
        t.use_logit_bias, t.finish_reason = False, [None] * 2
        return t
    bt = tree(constrain_draft=True)
    assert bt._draft_processed()
    bt.admit(1, prompts[1], stop_tokens=[9])
    assert bt.use_stop and bt.graphs == {}
    un = tree()
    un.admit(1, prompts[1], stop_tokens=[9])
    assert un.graphs == {"draft": 1}, "an unconstrained tree keeps its draft graph"


def test_testbed_flag():
    import testbed
    ap = testbed.build_parser()
    assert testbed.batch_constrain_draft(ap.parse_args([])) is False
    assert testbed.batch_constrain_draft(ap.parse_args(["--constrain-draft", "--batch", "2"])) is True
    assert testbed.batch_constrain_draft(ap.parse_args(["--constrain-draft", "--refill"])) is True
    with pytest.raises(SystemExit, match="--constrain-draft runs with --batch"):
        testbed.batch_constrain_draft(ap.parse_args(["--constrain-draft"]))


# ------------------------------------------------------------------------------------------------ the C entry points
def test_draft_rows_entry_point_refuses_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    f = 256                                             # a non-null address: every case is refused before any launch
    ALL = _lib.SQ_DRAFT_BIAS | _lib.SQ_DRAFT_BAN | _lib.SQ_DRAFT_GUIDE

    def call(logits=f, ld=32000, V=32000, base=f, step=f, k0=1, nk=19, S=128, state=f, flags=ALL, allowed=f, aw=1000,
             has_mask=f, ids=f, vals=f, nb=f, tokens=f, ld_seq=384, bits=f, tw=4, L=f, depth=f, words=f, lens=f, nw=f,
             me=f, ends=f, table=f, node=f, B=2):
        return lib.sq_draft_rows_batch(logits, ld, V, base, step, k0, nk, S, state, flags, allowed, aw, has_mask, ids,
                                       vals, nb, tokens, ld_seq, bits, tw, L, depth, words, lens, nw, me, ends, table,
                                       node, B, None)
    c0 = lib.sq_launch_count()
    nulls = [(dict([(k, None)]), b"null") for k in ("logits", "base", "step", "state", "allowed", "has_mask", "ids",
                                                    "vals", "nb", "tokens", "bits", "L", "depth", "words", "lens", "nw",
                                                    "me", "ends", "table", "node")]
    cases_ = nulls + [(dict(flags=0), b"flags=0"), (dict(flags=8), b"flags=8"), (dict(B=0), b"B=0"),
                      (dict(B=9), b"B=9"), (dict(V=32004, ld=32008), b"V=32004"), (dict(V=131080, ld=131080), b"V=131080"),
                      (dict(V=0), b"V=0"), (dict(ld=31999), b"ld=31999"), (dict(S=0, tw=0), b"S=0"),
                      (dict(tw=3), b"tree_words=3"), (dict(S=1025, tw=33), b"S=1025"),
                      (dict(k0=0, nk=2), b"nodes [0, 2)"), (dict(k0=120, nk=9), b"nodes [120, 129)"),
                      (dict(nk=0), b"nodes [1, 1)"), (dict(k0=-1, nk=2), b"nodes [-1, 1)"), (dict(aw=999), b"allowed_words"),
                      (dict(ld_seq=0), b"ld_seq=0")]
    for kw, msg in cases_:
        assert call(**kw) == -1 and msg in lib.sq_last_error(), (kw, msg, lib.sq_last_error())
    # the arrays of a kind that is not selected are not read: a null bias array with flags = BAN is not refused for it
    assert call(flags=_lib.SQ_DRAFT_BAN, allowed=None, V=0) == -1 and b"V=0" in lib.sq_last_error()
    assert lib.sq_launch_count() == c0, "refused before any launch"


def test_skip_dead_policy_bit_refusals():
    """SQ_ACCEPT_SKIP_DEAD is taken by the per-sequence, mixed and stop batch walks only."""
    from sequoia_b200 import _lib, ops
    lib = _lib.load()
    f = 256
    c0 = lib.sq_launch_count()
    args = (f, 32000, f, 32000, f, f, f, f, 32000, f, f, f, 128, 32000)
    tail = (f, f, 384, f, 128, f, 2, 384)
    assert lib.sq_accept_stochastic_batch(*args, 0.6, *tail, ops.ACCEPT_SKIP_DEAD, None) == -1
    assert b"unknown policy bits 8" in lib.sq_last_error()
    assert lib.sq_accept_stochastic(f, 32000, f, 32000, f, f, f, f, f, 128, 32000, 0.6, f, f, f, f, 384,
                                    ops.ACCEPT_SKIP_DEAD, None) == -1
    assert b"unknown policy bits 8" in lib.sq_last_error()
    assert lib.sq_accept_stochastic_batch_per_seq(*args, f, *tail, ops.ACCEPT_SKIP_DEAD | 4, None) == -1
    assert b"unknown policy bits 12" in lib.sq_last_error()
    assert lib.sq_launch_count() == c0
