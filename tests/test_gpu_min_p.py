"""Min-p filtering on the device (sq_min_p_filter_per_seq, BatchTree(min_p=...)).

Kernel level: the filtered rows against oracle/min_p.py bit for bit, from single-CTA rows to clusters of 2 and 4 slices,
at min_p from 1e-4 to 1 and T from 0.3 to 1.7; a row max that lies only in the last slice; rows exactly on the boundary;
NaN and +inf rows; the per-sequence array against launches per group, with off rows untouched.  Composition: min-p and
top-k commute bit for bit, and min-p then top-p matches the oracle's composition.  Walk level: min_p = 1 turns the
sampled walk into the greedy one, with min_p = 0.2 every committed token passes the rule, and a NaN row still ends the
walk.  BatchTree level: a slot's output does not depend on its neighbours' min_p, min_p = 0 launches nothing, the filter
joins the graphs once, greedy slots ignore it, and the logprobs read the filtered rows."""
import math

import pytest
import torch

import cases
from oracle import sequoia_oracle as O
from oracle.min_p import min_p_filter
from oracle.top_k import top_k_filter
from test_gpu_mixed_policy import GM128, _walk_inputs
from test_gpu_refill import DEV, F16, GM, M, ST_N_NEW, ST_P, _draft_layout, _engines, _f32, _state, ops
from test_gpu_top_k import _rows

pytestmark = pytest.mark.gpu

VS = [32000, 32776, 49152, 128256, 131072]            # 1 CTA; clusters of 2, 2, 4, 4 slices (32776: a short 2nd slice)
SLICE = 32768
NEG_INF = float("-inf")


def _bits(x):
    return x.view(torch.int16)


def _lmp(min_ps):
    """The device array of log(min_p) values (-inf = off), rounded to fp32 from double precision as BatchTree does."""
    return _f32([NEG_INF if p == 0 else math.log(p) for p in min_ps])


def _filter(x, min_p, T, rows_per_seq=None):
    """The per-sequence kernel on all rows of x at one min_p and T (an all-equal array)."""
    R = rows_per_seq or x.shape[0]
    B = x.shape[0] // R
    return ops().min_p_filter_per_seq_(x, _lmp([min_p] * B), _f32([T] * B), R)


# ------------------------------------------------------------------------------------------------ kernel vs oracle
@pytest.mark.parametrize("V", VS)
@pytest.mark.parametrize("min_p", [1e-4, 0.05, 0.3, 1.0])
def test_min_p_filter_matches_oracle(V, min_p):
    for n in (1, 128, 1024):
        x = _rows(n, V, V + n + int(min_p * 1e4))
        xc = x.cpu()
        for T in (0.3, 0.6, 1.0, 1.7):
            got = _filter(x.clone(), min_p, T).cpu()
            want = min_p_filter(xc, min_p, T)
            assert torch.equal(_bits(got), _bits(want)), (V, min_p, T, n)
        if min_p >= 0.05:
            assert int(torch.isinf(got[0]).sum()) > int(torch.isinf(xc[0]).sum()), "a randn row loses tokens"


@pytest.mark.parametrize("V", [32776, 49152, 128256, 131072])
def test_min_p_row_max_only_in_the_last_slice(V):
    """The max of each row lies in the last slice, so the other slices learn it only through the cluster max."""
    g = torch.Generator(device=DEV).manual_seed(V)
    x = (torch.randn(6, V, generator=g, device=DEV) * 2).to(F16)
    last = (V - 1) // SLICE * SLICE
    for r in range(6):
        x[r, last + (r * 7) % (V - last)] = 20.0 + r
    got = _filter(x.clone(), 0.05, 1.0).cpu()
    want = min_p_filter(x.cpu(), 0.05, 1.0)
    assert torch.equal(_bits(got), _bits(want))
    assert bool(torch.isinf(got[:, :SLICE]).all()), "every first-slice entry lies far below the last slice's max"


@pytest.mark.parametrize("V", [32000, 128256])
def test_min_p_exact_boundary(V):
    """min_p = e^-2: thr is exactly -2.0 at T = 1 and -1.0 at T = 0.5.  x = m - 2 (m - 1) stays, the next fp16 value
    below it goes; rows of both sequences in one per-sequence launch."""
    x = torch.full((4, V), -30.0, dtype=F16)
    for r, (m, gap) in enumerate(((4.0, 2.0), (5.5, 2.0), (4.0, 1.0), (-3.0, 1.0))):
        on = torch.tensor([m - gap], dtype=F16)
        below = (_bits(on) + (1 if m - gap < 0 else -1)).view(F16)
        x[r, V - 1] = m
        x[r, 3], x[r, V // 2], x[r, V // 2 + 1] = on, below, on
    got = ops().min_p_filter_per_seq_(x.clone().to(DEV), _lmp([math.exp(-2.0)] * 2), _f32([1.0, 0.5]), 2).cpu()
    for r, T in enumerate((1.0, 1.0, 0.5, 0.5)):
        assert (~torch.isinf(got[r])).nonzero().flatten().tolist() == [3, V // 2 + 1, V - 1], r
        assert torch.equal(_bits(got[r]), _bits(min_p_filter(x[r:r + 1], math.exp(-2.0), T)[0]))


@pytest.mark.parametrize("V", [32000, 49152, 128256])
def test_min_p_rows_with_nan_and_inf(V):
    x = _rows(8, V, 5)
    x[0, 17] = float("nan")                              # NaN stays, the rest is filtered by the finite max
    x[1, V - 3] = float("nan")
    x[2, 5] = float("inf")                               # +inf stays, every finite entry goes
    x[3, V - 9], x[3, 2] = float("inf"), float("inf")
    x[4] = float("nan")
    x[5, :] = NEG_INF
    x[5, V // 3] = float("nan")
    got = _filter(x.clone(), 0.1, 0.8).cpu()
    want = min_p_filter(x.cpu(), 0.1, 0.8)
    assert torch.equal(_bits(got), _bits(want))
    assert torch.isnan(got[0, 17]) and torch.isnan(got[1, V - 3])
    assert (~torch.isinf(got[2]) | torch.isposinf(got[2])).nonzero().flatten().tolist() == [5]
    assert bool(torch.isneginf(got[3]).sum() == V - 2)


# ------------------------------------------------------------------------------------------------ per-sequence form
@pytest.mark.parametrize("V", [32000, 49152, 128256])
def test_min_p_filter_per_seq(V):
    B, R = 4, 16
    x = _rows(B * R, V, V + 9)
    got = _filter(x.clone(), 0.1, 0.7, R)
    torch.cuda.synchronize()
    for b in range(B):
        rows = slice(b * R, (b + 1) * R)
        want = _filter(x[rows].clone(), 0.1, 0.7)
        assert torch.equal(_bits(got[rows]), _bits(want)), "all-equal array == one launch per group"
    ps, Ts = [0.2, 0.0, 1e-3, 1.0, 0.0, 0.5], [0.6, 0.9, 1.3, 0.5, 1.0, 0.3]
    x = _rows(len(ps) * R, V, V + 10)
    got = ops().min_p_filter_per_seq_(x.clone(), _lmp(ps), _f32(Ts), R).cpu()
    xc = x.cpu()
    for b, (p, T) in enumerate(zip(ps, Ts)):
        rows = slice(b * R, (b + 1) * R)
        if p:
            assert torch.equal(_bits(got[rows]), _bits(min_p_filter(xc[rows], p, T))), (V, b)
        else:
            assert torch.equal(_bits(got[rows]), _bits(xc[rows])), f"sequence {b} is off: its rows are untouched"


# ------------------------------------------------------------------------------------------------ composition
@pytest.mark.parametrize("V", [32000, 128256])
@pytest.mark.parametrize("min_p,k,T", [(0.05, 50, 0.6), (0.3, 5, 1.0), (1e-3, 1000, 1.3), (1.0, 2, 0.7)])
def test_min_p_and_top_k_commute(V, min_p, k, T):
    x = _rows(64, V, V + k)
    a = ops().top_k_filter_(_filter(x.clone(), min_p, T), k)
    b = _filter(ops().top_k_filter_(x.clone(), k), min_p, T)
    want = top_k_filter(min_p_filter(x.cpu(), min_p, T), k)
    assert torch.equal(_bits(a), _bits(b)), "min_p -> top_k == top_k -> min_p"
    assert torch.equal(_bits(a.cpu()), _bits(want))


@pytest.mark.parametrize("min_p,top_p,T", [(0.05, 0.9, 0.6), (0.01, 0.5, 1.0), (0.2, 0.95, 0.7)])
def test_min_p_then_top_p_matches_oracle(min_p, top_p, T):
    """min-p then top-p against oracle.min_p_filter then top_p_filter_integer, within top-p's one-token tolerance (the
    kernel's softmax may move one fp16 probability by an ulp, which can move the top-p cut by one token)."""
    V = 32000
    x = (torch.randn(3, V, generator=torch.Generator().manual_seed(int(min_p * 100)), dtype=torch.float32) * 3).to(F16)
    mp = min_p_filter(x, min_p, T)
    want = O.top_p_filter_integer(mp, top_p, T)
    got = ops().top_p_filter_(_filter(x.clone().to(DEV), min_p, T), top_p, T).cpu()
    keep_g, keep_w = ~torch.isinf(got), ~torch.isinf(want)
    assert int((keep_g != keep_w).sum(-1).max()) <= 1
    assert not bool((keep_g & torch.isinf(mp)).any()) and torch.equal(got[keep_g], x[keep_g])
    assert bool((keep_g.sum(-1) >= 1).all())


# ------------------------------------------------------------------------------------------------ accept walks
@pytest.fixture(scope="module")
def tree():
    from sequoia_b200.tree import _Static
    return _Static(cases.load_growmap(GM), DEV)


def _unique_max(target):
    """Raise each row's first maximum by 1, so the max is unique and argmax_rows still picks it."""
    idx = ops().argmax_rows(target)
    rows = torch.arange(target.shape[0], device=DEV)
    target[rows, idx] = (target[rows, idx].float() + 1.0).to(F16)
    return target


@pytest.mark.parametrize("V", [32000, 128256])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_min_p_1_sampled_walk_commits_the_greedy_walk(V, seed, tree):
    """min_p = 1 on rows with a unique max keeps one token per row: accept_stochastic_batch_per_seq accepts the same
    slots as argmax_rows + accept_greedy_batch, with the same bonus token and state (committed tokens up to SpecTree's
    order of writes, as in the top-k test)."""
    B, S = 3, tree.S
    per_seq, target, tokens0, pos0, r, noise = _walk_inputs(tree, B, V, seed=V + seed)
    target = _unique_max(target)
    buf, base, step = _draft_layout(tree, per_seq, V)
    st0 = _state(B)
    Ts = _f32([0.6, 0.9, 1.3])

    def fresh():
        return [tokens0.clone(), pos0.clone(), torch.full((B, S), -1, dtype=torch.int32, device=DEV), st0.clone()]
    greedy, sampled = fresh(), fresh()
    ops().accept_greedy_batch(ops().argmax_rows(target), tree.succ_off, tree.succ, tree.depth, S, *greedy, M)
    filtered = ops().min_p_filter_per_seq_(target.clone(), _lmp([1.0] * B), Ts, S)
    assert bool(((~torch.isinf(filtered)).sum(-1) == 1).all()), "one token per row survives"
    ops().accept_stochastic_batch_per_seq(filtered, buf, base, step, r, noise, tree.succ_off, tree.succ, tree.depth, S,
                                          Ts, *sampled, M)
    torch.cuda.synchronize()
    greedy, sampled, tok0 = [t.cpu() for t in greedy], [t.cpu() for t in sampled], tokens0.cpu()
    for b in range(B):
        P, a, n, bonus = int(st0[b, ST_P]), int(greedy[3][b, 1]), int(greedy[3][b, ST_N_NEW]), int(greedy[3][b, 5])
        assert torch.equal(sampled[3][b, :6], greedy[3][b, :6]), (V, seed, b, sampled[3][b, :8], greedy[3][b, :8])
        acc = greedy[2][b, :n]
        assert torch.equal(sampled[2][b, :n], acc), (V, seed, b)
        assert not bool(greedy[3][b, 2]) and int(greedy[0][b, a]) == int(sampled[0][b, a]) == bonus
        assert torch.equal(sampled[0][b, P:a], torch.where(acc == a, bonus, tok0[b, acc.long()])), (V, seed, b)
    assert max(int(greedy[3][b, ST_N_NEW]) for b in range(B)) >= 2, "the walks should accept a path"


@pytest.mark.parametrize("V", [32000, 128256])
def test_min_p_walk_commits_only_kept_tokens(V, tree):
    """min_p = 0.2: the token of every accepted node passes the rule in its parent node's row, the bonus token in the last
    accepted node's row."""
    B, S = 3, tree.S
    succ_off, succ = tree.succ_off.cpu().tolist(), tree.succ.cpu().tolist()
    Ts = [0.6, 0.9, 1.3]
    deepest = 0
    for seed in (4, 5, 6):
        per_seq, target, tokens0, pos0, r, noise = _walk_inputs(tree, B, V, seed=V + seed)
        buf, base, step = _draft_layout(tree, per_seq, V)
        st0 = _state(B)
        bufs = [tokens0.clone(), pos0.clone(), torch.full((B, S), -1, dtype=torch.int32, device=DEV), st0.clone()]
        filtered = ops().min_p_filter_per_seq_(target.clone(), _lmp([0.2] * B), _f32(Ts), S)
        ops().accept_stochastic_batch_per_seq(filtered, buf, base, step, r, noise, tree.succ_off, tree.succ, tree.depth,
                                              S, _f32(Ts), *bufs, M)
        tc = target.cpu()
        kept = [set(min_p_filter(tc[i:i + 1], 0.2, Ts[i // S])[0].isfinite().nonzero().flatten().tolist())
                for i in range(B * S)]
        tok0, acc, st = tokens0.cpu(), bufs[2].cpu(), bufs[3].cpu()
        for b in range(B):
            n = int(st[b, ST_N_NEW])
            cur = 0
            for slot in acc[b, :n].tolist():                   # accepted slots, in path order
                node = slot - (int(st0[b, ST_P]) - 1)
                assert node in succ[succ_off[cur]:succ_off[cur + 1]], (V, seed, b, node)
                assert int(tok0[b, slot]) in kept[b * S + cur], (V, seed, b, node)
                cur = node
            if not bool(st[b, 2]):                             # (a terminal walk has no bonus token)
                assert int(st[b, 5]) in kept[b * S + cur], (V, seed, b, "bonus")
            deepest = max(deepest, n)
    assert deepest >= 2, "the walks should accept a path"


def test_nan_row_still_ends_the_walk(tree):
    B, S, V = 3, tree.S, 32000
    per_seq, target, tokens0, pos0, r, noise = _walk_inputs(tree, B, V, seed=77)
    target[0, 123] = float("nan")
    buf, base, step = _draft_layout(tree, per_seq, V)
    rows = ops().min_p_filter_per_seq_(target.clone(), _lmp([0.2] * B), _f32([0.6] * B), S)
    bufs = [tokens0.clone(), pos0.clone(), torch.full((B, S), -1, dtype=torch.int32, device=DEV), _state(B)]
    ops().accept_stochastic_batch_per_seq(rows, buf, base, step, r, noise, tree.succ_off, tree.succ, tree.depth, S,
                                          _f32([0.6] * B), *bufs, M)
    st = bufs[3].cpu()
    assert int(st[0, 6]) == 1 and int(st[0, 2]) == 1, "the filtered walk flags the NaN"
    assert not bool(st[1:, 6].any())


# ------------------------------------------------------------------------------------------------ BatchTree
def _run(engines, prompts, gm, min_p, seeds, iters=6, policy="spec", Mx=256, T=0.6, top_p=1.0, **kw):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    bt = BatchTree(d, t, prompts, gm, policy=policy, temperature=T, top_p=top_p, max_length=Mx, seeds=seeds,
                   **({} if min_p is None else dict(min_p=min_p)), **kw)
    steps = []
    for _ in range(iters):
        bt.construct_grow_map()
        steps.append([(v.cpu().clone(), a, term) for v, a, term in bt.verify()])
        if all(bt.frozen):
            break
    return steps, bt


def _same(got, want, slots, what):
    assert len(got) == len(want), what
    for it in range(len(got)):
        for b in slots:
            (v, a, term), (v0, a0, term0) = got[it][b], want[it][b]
            assert (a, term) == (a0, term0) and torch.equal(v, v0), (what, it, b)


def test_neighbours_min_p_does_not_matter_and_zero_is_off():
    gm = cases.load_growmap(GM)
    engines = _engines(3)
    prompts = [cases.make_prompt(400 + i, n).to(DEV) for i, n in enumerate((90, 64, 110))]
    seeds = [61, 62, 63]
    base, bt0 = _run(engines, prompts, gm, None, seeds)
    assert not bt0.use_min_p
    off, bt = _run(engines, prompts, gm, 0.0, seeds)
    assert not bt.use_min_p and bt.graph_launches == bt0.graph_launches
    _same(off, base, (0, 1, 2), "min_p = 0")
    nb, bt = _run(engines, prompts, gm, [0.0, 0.2, 0.2], seeds)
    assert bt.use_min_p and bt.graph_launches["steady"] == bt0.graph_launches["steady"] + 1
    _same(nb, base, (0,), "a min_p = 0 slot next to min_p = 0.2 neighbours")


def test_seeded_min_p_slot_decodes_as_alone():
    """A seeded min_p = 0.1 sequence at B = 1 and in slot 1 of a B = 3 batch: >= 95% of the committed positions agree
    (the GEMMs see other row counts, as in the admission tests)."""
    gm = cases.load_growmap(GM)
    prompts = [cases.make_prompt(410 + i, n).to(DEV) for i, n in enumerate((70, 100, 84))]
    lone, _ = _run(_engines(1), prompts[1:2], gm, 0.1, [72], iters=8)
    batch, bt = _run(_engines(3), prompts, gm, [0.0, 0.1, 0.3], [71, 72, 73], iters=8)
    assert bt.use_min_p
    got, want = batch[-1][1][0], lone[-1][0][0]
    P = len(prompts[1])
    k = min(len(got), len(want))
    same = int((got[:k] == want[:k]).sum()) - P
    total = max(len(got), len(want)) - P
    assert total > 0 and same >= 0.95 * total, (same, total)


def test_min_p_admissions_capture_once():
    """In a mixed batch: a greedy admission with min_p captures nothing; the first spec admission with min_p > 0 captures
    the steady and post graphs once more (one more launch per steady step); later values capture nothing."""
    gm = cases.load_growmap(GM)
    d, t = _engines(2)
    from sequoia_b200.batch import BatchTree
    bt = BatchTree(d, t, [cases.make_prompt(420, 60), cases.make_prompt(421, 70)], gm, policy=["spec", "greedy"],
                   temperature=0.7, max_length=256, seeds=[1, 2])

    def step():
        bt.construct_grow_map()
        bt.verify()

    def admission(b, seed, p, policy):
        bt.freeze(b)
        bt.admit(b, cases.make_prompt(seed, 50 + seed % 7), seed=seed, min_p=p, policy=policy)
        step()                                          # the first verify: the post graph
        step()                                          # a steady step
    step()
    step()
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}
    launches = bt.graph_launches["steady"]
    admission(1, 430, 0.2, "greedy")
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1} and not bt.use_min_p
    assert bt.log_min_p_dev.tolist() == [NEG_INF, NEG_INF] and bt.min_ps == [0.0, 0.2]
    admission(0, 431, 0.2, "spec")
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2} and bt.use_min_p
    assert bt.graph_launches["steady"] == launches + 1, "the min-p filter is one more launch"
    for seed, p in ((432, 0.05), (433, 0.0), (434, 1.0)):
        admission(0, seed, p, "spec")
        assert bt.log_min_p_dev[0].item() == (NEG_INF if p == 0 else _lmp([p])[0].item())
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2}, "no recapture after the filter entered"


def test_mixed_batch_greedy_slot_ignores_min_p():
    gm = cases.load_growmap(GM)
    engines = _engines(2)
    prompts = [cases.make_prompt(440 + i, n).to(DEV) for i, n in enumerate((80, 96))]
    with_p, bt = _run(engines, prompts, gm, [0.3, 0.3], [81, 82], policy=["spec", "greedy"])
    assert bt.mixed and bt.use_min_p and bt.log_min_p_dev[1].item() == NEG_INF
    without, _ = _run(engines, prompts, gm, 0.0, [81, 82], policy=["spec", "greedy"])
    _same(with_p, without, (1,), "greedy slot")


def test_logprobs_read_the_filtered_rows():
    """logprobs = 5 at T = 1 (the log-probabilities are then those of the filtered row itself) and min_p = 0.3: every
    generated token and every finite top alternative has lp >= lp_top[0] + ln 0.3 - 1e-3."""
    gm = cases.load_growmap(GM)
    prompts = [cases.make_prompt(450 + i, n).to(DEV) for i, n in enumerate((70, 90))]
    _, bt = _run(_engines(2), prompts, gm, 0.3, [5, 6], iters=6, T=1.0, logprobs=5)
    n_tok = 0
    for b in range(2):
        lp, ids, top = bt.token_logprobs(b)
        assert lp.shape[0] > 0 and ids.shape[1] == 5
        bound = top[:, 0] + math.log(0.3) - 1e-3
        assert bool((lp >= bound).all()), (b, lp, top[:, 0])
        fin = torch.isfinite(top)
        assert bool((top >= bound[:, None])[fin].all()), b
        n_tok += lp.shape[0]
    assert n_tok >= 4


def test_min_p_batch_llama3_vocab():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 2, seeded, min_p = 0.1 on slot 1: slot 0 commits what it commits
    in a batch without min_p, and slot 1 decodes."""
    import gc
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gc.collect()
    torch.cuda.empty_cache()
    gm, Mx = cases.load_growmap(GM128), 384
    engines = (GraphInferenceEngine(Mx, "random-init:llama-3.2-1b:1", device=DEV, batch_size=2),
               GraphInferenceEngineTG(Mx, "random-init:llama-3.1-8b:2", device=DEV, batch_size=2))
    g = torch.Generator().manual_seed(29)
    prompts = [torch.randint(3, 128256, (n,), generator=g).to(DEV) for n in (90, 128)]
    with_p, bt = _run(engines, prompts, gm, [0.0, 0.1], [91, 92], iters=4, Mx=Mx, top_p=[1.0, 0.95])
    assert bt.use_min_p and bt.V == 128256
    without, _ = _run(engines, prompts, gm, 0.0, [91, 92], iters=4, Mx=Mx, top_p=[1.0, 0.95])
    _same(with_p, without, (0,), "slot without min_p")
    assert len(with_p[-1][1][0]) >= len(prompts[1]) + len(with_p)
