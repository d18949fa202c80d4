"""Top-k filtering on the device (sq_top_k_filter, sq_top_k_filter_per_seq, BatchTree(top_k=...)).

Kernel level: the filtered rows against oracle/top_k.py (a stable descending torch.sort) bit for bit, from single-CTA
rows to clusters of 2, 3 and 4 slices, at k from 1 to V; boundary tie groups that span slices; the per-sequence form
against scalar launches; top-k then top-p against the oracle's composition.  Walk level: k = 1 turns the sampled walk into
the greedy one, and with k = 5 every committed token is among its row's 5 kept tokens.  BatchTree level: a slot's output
does not depend on its neighbours' top_k, k >= V is off, the filter joins the graphs once, and greedy slots ignore it."""
import pytest
import torch

import cases
from oracle import sequoia_oracle as O
from oracle.top_k import top_k_filter
from test_gpu_mixed_policy import GM128, _walk_inputs
from test_gpu_refill import DEV, F16, GM, M, ST_N_NEW, ST_P, _draft_layout, _engines, _f32, _state, ops

pytestmark = pytest.mark.gpu

VS = [32000, 32776, 49152, 128256, 131072]            # 1 CTA; clusters of 2, 2, 4, 4 slices (32776: a short 2nd slice)
SLICE = 32768
NEG_INF = float("-inf")


def _bits(x):
    return x.view(torch.int16)


def _i32(vals):
    return torch.tensor(vals, dtype=torch.int32, device=DEV)


def _rows(n, V, seed):
    """n rows of four kinds in turn: randn * 3 (fp16 ties at every k of interest), small integers (huge tie groups),
    randn with 90% -inf, and 20 finite entries in a row of -inf."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.randn(n, V, generator=g, device=DEV) * 3).to(F16)
    x[1::4] = torch.randint(-4, 5, (x[1::4].shape[0], V), generator=g, device=DEV).to(F16)
    x[2::4].masked_fill_(torch.rand(x[2::4].shape, generator=g, device=DEV) < 0.9, NEG_INF)
    sparse = x[3::4]
    keep = torch.rand(sparse.shape, generator=g, device=DEV).argsort(-1)[:, :20]
    x[3::4] = torch.full_like(sparse, NEG_INF).scatter_(-1, keep, sparse.gather(-1, keep))
    return x


# ------------------------------------------------------------------------------------------------ kernel vs oracle
@pytest.mark.parametrize("V", VS)
@pytest.mark.parametrize("kk", ["1", "2", "50", "1000", "V-1", "V"])
def test_top_k_filter_matches_oracle(V, kk):
    k = {"V-1": V - 1, "V": V}.get(kk) or int(kk)
    for n in (1, 128, 1024):
        x = _rows(n, V, V + n + k)
        got = ops().top_k_filter_(x.clone(), k)
        want = top_k_filter(x, k)
        torch.cuda.synchronize()
        assert torch.equal(_bits(got), _bits(want)), (V, k, n)
        if k < V:
            kept = (_bits(got) == _bits(x)) & ~torch.isinf(x)
            assert int(kept[0].sum()) == k, "a randn row keeps exactly k tokens"


@pytest.mark.parametrize("V", [32776, 49152, 128256, 131072])
def test_top_k_boundary_tie_group_across_slices_ranks_by_index(V):
    """Equal logits at 2.0, 32 in the first slice and up to 32 spread over the others, with the cut inside the later
    ones: the tie group keeps its lowest indices across slices.  Row 1 adds 10 larger logits, which stay, and the tie
    group keeps 10 fewer."""
    lg = torch.full((2, V), -30.0, dtype=F16)
    lo = torch.linspace(5, SLICE - 9, 32).long()
    hi = torch.linspace(SLICE, V - 1, 32).long().unique()
    idx = torch.cat([lo, hi])
    k = 32 + max(1, len(hi) // 2)
    top = idx[:10] + 1
    lg[:, idx] = 2.0
    lg[1, top] = 5.0
    got = ops().top_k_filter_(lg.clone().to(DEV), k).cpu()
    assert torch.equal((~torch.isinf(got[0])).nonzero().flatten(), idx[:k])
    assert torch.equal((~torch.isinf(got[1])).nonzero().flatten(), torch.cat([idx[:k - 10], top]).sort().values)


@pytest.mark.parametrize("V", [32000, 49152, 131072])
def test_top_k_all_equal_row_keeps_the_lowest_indices(V):
    lg = torch.full((3, V), 0.75, dtype=F16, device=DEV)
    for k in (1, 50, V - 1):
        got = ops().top_k_filter_(lg.clone(), k).cpu()
        assert bool((~torch.isinf(got)).sum(-1).eq(k).all())
        assert bool((~torch.isinf(got[:, :k])).all()), (V, k)


@pytest.mark.parametrize("V", [32000, 128256])
def test_top_k_row_with_nan_does_not_fault(V):
    """A NaN in a row: the launch completes and the other rows are filtered as usual (the NaN row is not compared; the
    accept walk's NaN flag ends such a sequence)."""
    x = _rows(8, V, 3)
    x[0, 17] = float("nan")
    x[5, V - 3] = float("nan")
    got = ops().top_k_filter_(x.clone(), 50)
    torch.cuda.synchronize()
    want = top_k_filter(x, 50)
    for r in (1, 2, 3, 4, 6, 7):
        assert torch.equal(_bits(got[r]), _bits(want[r])), r
    assert int((_bits(got[0]) == _bits(x[0])).sum()) == 50


# ------------------------------------------------------------------------------------------------ per-sequence form
@pytest.mark.parametrize("V", [32000, 49152, 128256])
def test_top_k_filter_per_seq(V):
    B, R = 4, 16
    x = _rows(B * R, V, V + 9)
    got = ops().top_k_filter_per_seq_(x.clone(), _i32([50] * B), R)
    want = ops().top_k_filter_(x.clone(), 50)
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want)), "all-equal array == the scalar call"
    ks = [7, 0, 1000, V, V + 5, 1]
    x = _rows(len(ks) * R, V, V + 10)
    got = ops().top_k_filter_per_seq_(x.clone(), _i32(ks), R)
    torch.cuda.synchronize()
    for b, k in enumerate(ks):
        rows = slice(b * R, (b + 1) * R)
        if 0 < k < V:
            want = ops().top_k_filter_(x[rows].clone(), k)
            torch.cuda.synchronize()
            assert torch.equal(_bits(got[rows]), _bits(want)), (V, b, k)
            assert bool(torch.isinf(got[rows]).sum() > torch.isinf(x[rows]).sum())
        else:
            assert torch.equal(_bits(got[rows]), _bits(x[rows])), f"k = {k}: rows untouched"


# ------------------------------------------------------------------------------------------------ composition
@pytest.mark.parametrize("k,top_p,T", [(50, 0.9, 0.6), (1000, 0.5, 1.0), (3, 0.95, 0.7)])
def test_top_k_then_top_p_matches_oracle(k, top_p, T):
    """top_k_filter_ then top_p_filter_ against oracle.top_k_filter then top_p_filter_integer.  As in the top-p tests the
    kernel's softmax may move one fp16 probability by an ulp, which can move the top-p cut by one token: at most one
    differing position per row, every survivor untouched and among the top-k set."""
    V = 32000
    x = (torch.randn(3, V, generator=torch.Generator().manual_seed(k), dtype=torch.float32) * 3).to(F16)
    topk = top_k_filter(x, k)
    want = O.top_p_filter_integer(topk, top_p, T)
    got = ops().top_p_filter_(ops().top_k_filter_(x.clone().to(DEV), k), top_p, T).cpu()
    keep_g, keep_w = ~torch.isinf(got), ~torch.isinf(want)
    assert int((keep_g != keep_w).sum(-1).max()) <= 1
    assert not bool((keep_g & torch.isinf(topk)).any()) and torch.equal(got[keep_g], x[keep_g])
    assert bool((keep_g.sum(-1) >= 1).all())


# ------------------------------------------------------------------------------------------------ accept walks
@pytest.fixture(scope="module")
def tree():
    from sequoia_b200.tree import _Static
    return _Static(cases.load_growmap(GM), DEV)


@pytest.mark.parametrize("V", [32000, 128256])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_k1_sampled_walk_commits_the_greedy_walk(V, seed, tree):
    """Target rows filtered to k = 1 make every sampled decision deterministic: accept_stochastic_batch_per_seq accepts
    the same tree slots as argmax_rows + accept_greedy_batch on the unfiltered rows, with the same bonus token and state.
    The committed tokens are the same too, up to SpecTree's order of writes (SpecTree.py:222-224, reproduced by the
    sampled walk): it writes the bonus at slot a before gathering the accepted slots, so an accepted slot equal to a
    commits the bonus token."""
    B, S = 3, tree.S
    per_seq, target, tokens0, pos0, r, noise = _walk_inputs(tree, B, V, seed=V + seed)
    buf, base, step = _draft_layout(tree, per_seq, V)
    st0 = _state(B)

    def fresh():
        return [tokens0.clone(), pos0.clone(), torch.full((B, S), -1, dtype=torch.int32, device=DEV), st0.clone()]
    greedy, sampled = fresh(), fresh()
    ops().accept_greedy_batch(ops().argmax_rows(target), tree.succ_off, tree.succ, tree.depth, S, *greedy, M)
    filtered = ops().top_k_filter_(target.clone(), 1)
    ops().accept_stochastic_batch_per_seq(filtered, buf, base, step, r, noise, tree.succ_off, tree.succ, tree.depth, S,
                                          _f32([0.6, 0.9, 1.3]), *sampled, M)
    torch.cuda.synchronize()
    greedy, sampled, tok0 = [t.cpu() for t in greedy], [t.cpu() for t in sampled], tokens0.cpu()
    for b in range(B):
        P, a, n, bonus = int(st0[b, ST_P]), int(greedy[3][b, 1]), int(greedy[3][b, ST_N_NEW]), int(greedy[3][b, 5])
        assert torch.equal(sampled[3][b, :6], greedy[3][b, :6]), (V, seed, b, sampled[3][b, :8], greedy[3][b, :8])
        acc = greedy[2][b, :n]
        assert torch.equal(sampled[2][b, :n], acc), (V, seed, b)
        assert not bool(greedy[3][b, 2]) and int(greedy[0][b, a]) == int(sampled[0][b, a]) == bonus
        assert torch.equal(greedy[0][b, :P], tok0[b, :P]) and torch.equal(sampled[0][b, :P], tok0[b, :P])
        assert torch.equal(greedy[0][b, P:a], tok0[b, acc.long()])
        assert torch.equal(sampled[0][b, P:a], torch.where(acc == a, bonus, tok0[b, acc.long()])), (V, seed, b)
    assert max(int(greedy[3][b, ST_N_NEW]) for b in range(B)) >= 2, "the walks should accept a path"


@pytest.mark.parametrize("V", [32000, 128256])
def test_k5_walk_commits_only_kept_tokens(V, tree):
    """k = 5: the token of every accepted node lies among the 5 kept tokens of its parent node's row, the bonus token
    among those of the last accepted node's row."""
    B, S = 3, tree.S
    succ_off, succ = tree.succ_off.cpu().tolist(), tree.succ.cpu().tolist()
    deepest = 0
    for seed in (4, 5, 6):
        per_seq, target, tokens0, pos0, r, noise = _walk_inputs(tree, B, V, seed=V + seed)
        buf, base, step = _draft_layout(tree, per_seq, V)
        st0 = _state(B)
        bufs = [tokens0.clone(), pos0.clone(), torch.full((B, S), -1, dtype=torch.int32, device=DEV), st0.clone()]
        filtered = ops().top_k_filter_(target.clone(), 5)
        ops().accept_stochastic_batch_per_seq(filtered, buf, base, step, r, noise, tree.succ_off, tree.succ, tree.depth,
                                              S, _f32([0.6, 0.9, 1.3]), *bufs, M)
        kept = [set(row.nonzero().flatten().tolist()) for row in (~torch.isinf(filtered)).cpu()]
        tok0, acc, st = tokens0.cpu(), bufs[2].cpu(), bufs[3].cpu()
        for b in range(B):
            P, n = int(st0[b, ST_P]), int(st[b, ST_N_NEW])
            cur = 0
            for slot in acc[b, :n].tolist():                   # accepted slots, in path order
                node = slot - (P - 1)
                assert node in succ[succ_off[cur]:succ_off[cur + 1]], (V, seed, b, node)
                assert int(tok0[b, slot]) in kept[b * S + cur], (V, seed, b, node)
                cur = node
            if not bool(st[b, 2]):                             # (a terminal walk has no bonus token)
                assert int(st[b, 5]) in kept[b * S + cur], (V, seed, b, "bonus")
            deepest = max(deepest, n)
    assert deepest >= 2, "the walks should accept a path"


def test_nan_row_still_ends_the_walk(tree):
    """A NaN in a sequence's root target row: after the k = 5 filter the walk still raises the NaN flag and ends that
    sequence, as it does on the unfiltered rows, and the other sequences walk as without the filter's NaN row."""
    B, S, V = 3, tree.S, 32000
    per_seq, target, tokens0, pos0, r, noise = _walk_inputs(tree, B, V, seed=77)
    target[0, 123] = float("nan")
    buf, base, step = _draft_layout(tree, per_seq, V)
    states = []
    for rows in (target, ops().top_k_filter_(target.clone(), 5)):
        bufs = [tokens0.clone(), pos0.clone(), torch.full((B, S), -1, dtype=torch.int32, device=DEV), _state(B)]
        ops().accept_stochastic_batch_per_seq(rows, buf, base, step, r, noise, tree.succ_off, tree.succ, tree.depth, S,
                                              _f32([0.6] * B), *bufs, M)
        states.append(bufs[3].cpu())
    unfiltered, filtered = states
    assert int(unfiltered[0, 6]) == 1 and int(unfiltered[0, 2]) == 1, "the unfiltered walk flags the NaN"
    assert int(filtered[0, 6]) == 1 and int(filtered[0, 2]) == 1, "the filtered walk flags it too"
    assert not bool(filtered[1:, 6].any())


# ------------------------------------------------------------------------------------------------ BatchTree
def _run(engines, prompts, gm, top_k, seeds, iters=6, policy="spec", Mx=256, T=0.6, top_p=1.0):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    bt = BatchTree(d, t, prompts, gm, policy=policy, temperature=T, top_p=top_p, max_length=Mx, seeds=seeds, top_k=top_k)
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


def test_neighbours_top_k_does_not_matter_and_large_k_is_off():
    gm = cases.load_growmap(GM)
    V = cases.V
    engines = _engines(3)
    prompts = [cases.make_prompt(300 + i, n).to(DEV) for i, n in enumerate((90, 64, 110))]
    seeds = [61, 62, 63]
    base, bt0 = _run(engines, prompts, gm, 0, seeds)
    assert not bt0.use_top_k
    nb, bt = _run(engines, prompts, gm, [0, 20, 20], seeds)
    assert bt.use_top_k and bt.top_k_dev.tolist() == [0, 20, 20]
    _same(nb, base, (0,), "a top_k = 0 slot next to top_k = 20 neighbours")
    for big in (V, 10 * V):
        off, bt = _run(engines, prompts, gm, big, seeds)
        assert not bt.use_top_k and bt.graph_launches == bt0.graph_launches
        _same(off, base, (0, 1, 2), f"top_k = {big}")
    # the filter changes what the filtered slots commit
    assert any(not torch.equal(nb[-1][b][0], base[-1][b][0]) for b in (1, 2))


def test_seeded_top_k_slot_decodes_as_alone():
    """A seeded top_k = 20 sequence at B = 1 and in slot 1 of a B = 3 batch: >= 95% of the committed positions agree
    (the GEMMs see other row counts, as in the admission tests)."""
    gm = cases.load_growmap(GM)
    prompts = [cases.make_prompt(310 + i, n).to(DEV) for i, n in enumerate((70, 100, 84))]
    lone, _ = _run(_engines(1), prompts[1:2], gm, 20, [72], iters=8)
    batch, bt = _run(_engines(3), prompts, gm, [0, 20, 5], [71, 72, 73], iters=8)
    assert bt.use_top_k
    got, want = batch[-1][1][0], lone[-1][0][0]
    P = len(prompts[1])
    k = min(len(got), len(want))
    same = int((got[:k] == want[:k]).sum()) - P
    total = max(len(got), len(want)) - P
    assert total > 0 and same >= 0.95 * total, (same, total)


def test_top_k_admissions_capture_once():
    """In a mixed batch: a greedy admission with top_k captures nothing; the first spec admission with 0 < top_k < V
    captures the steady and post graphs once more (one more launch per steady step); later spec admissions at other k
    (0, V and a new value) capture nothing."""
    gm = cases.load_growmap(GM)
    V = cases.V
    d, t = _engines(2)
    from sequoia_b200.batch import BatchTree
    bt = BatchTree(d, t, [cases.make_prompt(320, 60), cases.make_prompt(321, 70)], gm, policy=["spec", "greedy"],
                   temperature=0.7, max_length=256, seeds=[1, 2])

    def step():
        bt.construct_grow_map()
        bt.verify()

    def admission(b, seed, k, policy):
        bt.freeze(b)
        bt.admit(b, cases.make_prompt(seed, 50 + seed % 7), seed=seed, top_k=k, policy=policy)
        step()                                          # the first verify: the post graph
        step()                                          # a steady step
    step()
    step()
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}
    launches = bt.graph_launches["steady"]
    admission(1, 330, 20, "greedy")
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1} and not bt.use_top_k
    assert bt.top_k_dev.tolist() == [0, 0] and bt.top_ks == [0, 20]
    admission(0, 331, 20, "spec")
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2} and bt.use_top_k
    assert bt.graph_launches["steady"] == launches + 1, "the top-k filter is one more launch"
    for seed, k in ((332, 7), (333, 0), (334, V)):
        admission(0, seed, k, "spec")
        assert bt.top_k_dev.tolist() == [min(k, V), 0]
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2}, "no recapture after the filter entered"


def test_mixed_batch_greedy_slot_ignores_top_k():
    gm = cases.load_growmap(GM)
    engines = _engines(2)
    prompts = [cases.make_prompt(340 + i, n).to(DEV) for i, n in enumerate((80, 96))]
    with_k, bt = _run(engines, prompts, gm, [20, 20], [81, 82], policy=["spec", "greedy"])
    assert bt.mixed and bt.use_top_k and bt.top_k_dev.tolist() == [20, 0]
    without, _ = _run(engines, prompts, gm, 0, [81, 82], policy=["spec", "greedy"])
    _same(with_k, without, (1,), "greedy slot")


def test_top_k_batch_llama3_vocab():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 2, seeded, top_k = 40 on slot 1: slot 0 commits what it commits
    in a batch without top_k, and slot 1 decodes."""
    import gc
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gc.collect()
    torch.cuda.empty_cache()
    gm, Mx = cases.load_growmap(GM128), 384
    engines = (GraphInferenceEngine(Mx, "random-init:llama-3.2-1b:1", device=DEV, batch_size=2),
               GraphInferenceEngineTG(Mx, "random-init:llama-3.1-8b:2", device=DEV, batch_size=2))
    g = torch.Generator().manual_seed(23)
    prompts = [torch.randint(3, 128256, (n,), generator=g).to(DEV) for n in (90, 128)]
    with_k, bt = _run(engines, prompts, gm, [0, 40], [91, 92], iters=4, Mx=Mx, top_p=[1.0, 0.95])
    assert bt.use_top_k and bt.V == 128256
    without, _ = _run(engines, prompts, gm, 0, [91, 92], iters=4, Mx=Mx, top_p=[1.0, 0.95])
    _same(with_k, without, (0,), "slot without top_k")
    assert len(with_k[-1][1][0]) >= len(prompts[1]) + len(with_k)
