"""Greedy and sampled sequences in one batch (per-sequence policy, BatchTree(policy=[...])).

Kernel level: the three *_mixed entry points against the per-sequence / batched launches of one policy, bit for bit, and
byte-for-byte untouched rows of the other policy's and frozen sequences.  BatchTree level: each sequence of a mixed batch
decodes exactly as in a batch of its own policy (same prompts, seeds, T and top_p), at config 2 and Llama 3 shapes; a
mixing admission captures the draft, steady and post graphs once more, and a mixed steady step is still two replays and
one host sync."""
import pytest
import torch

import cases
from test_gpu_refill import DEV, F16, GM, M, ST_FROZEN, ST_N_NEW, ST_P, _draft_layout, _engines, _f32, _state, ops

pytestmark = pytest.mark.gpu

VOCABS = [32000, 49152, 128256]           # accept walk NCH = 1, 2, 4; sampling clusters of 1, 2, 4 CTAs
GM128 = "A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"   # config 2: 128 nodes


@pytest.fixture(scope="module")
def tree():
    from sequoia_b200.tree import _Static
    return _Static(cases.load_growmap(GM), DEV)


def _i32(vals):
    return torch.tensor(vals, dtype=torch.int32, device=DEV)


# ------------------------------------------------------------------------------------------------ sampler
def _sample(tree, buf, base, step, rand, T, mode, tokens, state, greedy=None):
    for lv in tree.levels:
        kw = dict(parent_rows=lv["parents"], child_first=lv["first"], n_branch=lv["nb"], tokens=tokens, state=state)
        if greedy is not None:
            ops().sample_level_batch_mixed(buf, base, step, rand, lv["n_parents"], lv["k"], T, greedy, **kw)
        else:
            ops().sample_level_batch_per_seq(buf, base, step, rand, lv["n_parents"], lv["k"], T, mode, **kw)
    torch.cuda.synchronize()


@pytest.mark.parametrize("V", VOCABS)
def test_sample_level_mixed(V, tree):
    """B = 4: sequences 0 and 1 greedy, 2 sampled, 3 frozen.  Greedy rows == a mode-1 launch, the sampled row == a mode-0
    launch at its own T, the frozen row untouched; all-zero / all-one greedy arrays == the mode-0 / mode-1 launches."""
    B, S = 4, tree.S
    g = torch.Generator(device=DEV).manual_seed(V + 3)
    per_seq = [(torch.randn(S, V, generator=g, device=DEV) * 2).to(F16) for _ in range(B)]
    rand = torch.rand(B, S, V, generator=g, device=DEV).to(F16)
    buf, base, step = _draft_layout(tree, per_seq, V)
    Ts = _f32([0.5, 0.8, 1.2, 0.7])
    state = _state(B, frozen=(3,))
    got = torch.full((B, M), -5, dtype=torch.int64, device=DEV)
    _sample(tree, buf, base, step, rand, Ts, None, got, state, greedy=_i32([1, 1, 0, 0]))
    want = {m: torch.full((B, M), -5, dtype=torch.int64, device=DEV) for m in (0, 1)}
    for m in (0, 1):
        _sample(tree, buf, base, step, rand, Ts, m, want[m], state)
    assert torch.equal(got[0], want[1][0]) and torch.equal(got[1], want[1][1])
    assert torch.equal(got[2], want[0][2])
    assert bool((got[3] == -5).all()), "frozen row untouched"
    P0 = int(state[0, ST_P])
    assert not torch.equal(got[0, P0:P0 + S - 1], want[0][0, P0:P0 + S - 1]), "greedy row must differ from a sampled one"
    state = _state(B)
    for flag in (0, 1):
        got = torch.full((B, M), -5, dtype=torch.int64, device=DEV)
        ref = torch.full((B, M), -5, dtype=torch.int64, device=DEV)
        _sample(tree, buf, base, step, rand, Ts, None, got, state, greedy=_i32([flag] * B))
        _sample(tree, buf, base, step, rand, Ts, flag, ref, state)
        assert torch.equal(got, ref), flag


# ------------------------------------------------------------------------------------------------ walks
def _walk_inputs(tree, B, V, seed):
    """Draft / target rows close enough that the sampled walks accept several nodes; the tree tokens of every sequence
    follow the target argmax along each node's first child, so the greedy walks accept a path down to a leaf."""
    S = tree.S
    g = torch.Generator(device=DEV).manual_seed(seed)
    per_seq, target = [], []
    for b in range(B):
        d = (torch.randn(S, V, generator=g, device=DEV) * 0.5).to(F16)
        per_seq.append(d)
        target.append((d.float() + 0.05 * torch.randn(S, V, generator=g, device=DEV)).to(F16))
    target = torch.cat(target)
    tokens = torch.randint(3, V, (B, M), generator=g, device=DEV)
    state = _state(B)
    tt = ops().argmax_rows(target).cpu().view(B, S)
    succ_off, succ = tree.succ_off.cpu().tolist(), tree.succ.cpu().tolist()
    for b in range(B):
        P = int(state[b, ST_P])
        for k in range(S):
            if succ_off[k] < succ_off[k + 1]:
                tokens[b, P - 1 + succ[succ_off[k]]] = int(tt[b, k])
    pos = torch.randint(0, M, (B, M), generator=g, device=DEV)
    r = torch.rand(B, M, generator=g, device=DEV).to(F16)
    noise = torch.empty(B, V, device=DEV).exponential_(1.0, generator=g).to(F16)
    return per_seq, target, tokens, pos, r, noise


@pytest.mark.parametrize("V", VOCABS)
def test_mixed_walks(V, tree):
    """B = 4, greedy = [1, 0, 1, 0], sequence 3 frozen.  Each mixed walk alone leaves every byte of the other policy's
    and the frozen sequences' tokens, position_ids, accept_idx and state rows as they were, and equals the per-sequence
    stochastic / batched greedy walk for its own sequences; both in sequence give the union."""
    B, S = 4, tree.S
    per_seq, target, tokens0, pos0, r, noise = _walk_inputs(tree, B, V, seed=V + 5)
    buf, base, step = _draft_layout(tree, per_seq, V)
    Ts = _f32([0.6, 0.9, 1.3, 0.7])
    greedy = _i32([1, 0, 1, 0])
    st0 = _state(B, frozen=(3,))
    target_token = ops().argmax_rows(target)

    def fresh():
        return [tokens0.clone(), pos0.clone(), torch.full((B, S), -1, dtype=torch.int32, device=DEV), st0.clone()]

    def stoch(bufs, mixed):
        args = (target, buf, base, step, r, noise, tree.succ_off, tree.succ, tree.depth, S, Ts)
        if mixed:
            ops().accept_stochastic_batch_mixed(*args, greedy, *bufs, M)
        else:
            ops().accept_stochastic_batch_per_seq(*args, *bufs, M)

    def greedy_walk(bufs, mixed):
        if mixed:
            ops().accept_greedy_batch_mixed(target_token, tree.succ_off, tree.succ, tree.depth, S, greedy, *bufs, M)
        else:
            ops().accept_greedy_batch(target_token, tree.succ_off, tree.succ, tree.depth, S, *bufs, M)

    ref_s, ref_g = fresh(), fresh()
    stoch(ref_s, False)
    greedy_walk(ref_g, False)
    sentinel = fresh()
    only_s, only_g, both = fresh(), fresh(), fresh()
    stoch(only_s, True)
    greedy_walk(only_g, True)
    greedy_walk(both, True)
    stoch(both, True)
    torch.cuda.synchronize()
    for b in range(B):
        own_s = b in (1,)
        own_g = b in (0, 2)
        for i, name in enumerate(("tokens", "position_ids", "accept_idx", "state")):
            want_s = ref_s[i][b] if own_s else sentinel[i][b]
            want_g = ref_g[i][b] if own_g else sentinel[i][b]
            assert torch.equal(only_s[i][b], want_s), (V, b, name, "stochastic")
            assert torch.equal(only_g[i][b], want_g), (V, b, name, "greedy")
            assert torch.equal(both[i][b], ref_s[i][b] if own_s else want_g), (V, b, name, "both")
    assert int(only_g[3][0, ST_N_NEW]) >= 2 and int(only_s[3][1, ST_N_NEW]) >= 1, "the walks should accept nodes"
    assert int(only_s[3][3, ST_FROZEN]) == 1


# ------------------------------------------------------------------------------------------------ BatchTree end to end
def _c2_engines(B, Mx=384):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    return (GraphInferenceEngine(Mx, "random-init:llama-68m:1", device=DEV, batch_size=B),
            GraphInferenceEngineTG(Mx, "random-init:llama-2-7b:2", device=DEV, batch_size=B))


def _decode(engines, prompts, gm, policy, Ts, tps, seeds, Mx, iters, torch_seed=None):
    """-> per step, per slot (valid tokens, accept_length, terminal), until every slot is frozen or `iters` steps"""
    from sequoia_b200.batch import BatchTree
    d, t = engines
    if torch_seed is not None:
        torch.manual_seed(torch_seed)
    bt = BatchTree(d, t, prompts, gm, policy=policy, temperature=Ts, top_p=tps, max_length=Mx, seeds=seeds)
    steps = []
    for _ in range(iters):
        bt.construct_grow_map()
        steps.append([(v.cpu().clone(), a, term) for v, a, term in bt.verify()])
        if all(bt.frozen):
            break
    return steps, bt


def _same_slots(got, want, slots, what):
    for it in range(min(len(got), len(want))):
        for b in slots:
            (v, a, term), (v0, a0, term0) = got[it][b], want[it][b]
            assert (a, term) == (a0, term0) and torch.equal(v, v0), (what, it, b)


@pytest.mark.parametrize("seeded", [True, False])
def test_mixed_batch_matches_single_policy_batches_config2(seeded):
    """Config 2 shapes (random-init llama-68m -> llama-2-7b, the 128-node tree, M 384), B = 4, policies [greedy, spec,
    spec, greedy], distinct T, top_p 0.9 for sequence 2, prompts of 4 lengths, 12 steps: every step's result of a greedy
    slot equals that slot of an all-greedy batch, of a spec slot that slot of an all-spec batch with the same seeds, T and
    top_p.  seeds=None: torch's generators are reset before each tree and the CPU draws stay stream-aligned."""
    gm = cases.load_growmap(GM128)
    engines = _c2_engines(4)
    prompts = [cases.make_prompt(200 + i, n).to(DEV) for i, n in enumerate((100, 64, 128, 80))]
    pols = ["greedy", "spec", "spec", "greedy"]
    Ts, tps = [0.5, 0.6, 0.9, 1.2], [1.0, 1.0, 0.9, 1.0]
    seeds = [11, 12, 13, 14] if seeded else None
    runs = {}
    for name, pol in (("mixed", pols), ("greedy", "greedy"), ("spec", "spec")):
        runs[name], bt = _decode(engines, prompts, gm, pol, Ts, tps, seeds, 384, 12, torch_seed=None if seeded else 7)
        if name == "mixed":
            assert bt.mixed and bt.use_top_p and bt.captures == {"draft": 1, "post": 1, "steady": 1}
    _same_slots(runs["mixed"], runs["greedy"], (0, 3), "greedy slots")
    _same_slots(runs["mixed"], runs["spec"], (1, 2), "spec slots")
    assert len(runs["mixed"]) >= 3


def test_mixed_batch_matches_single_policy_batches_llama3():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 2, one sequence per policy, 4 steps, seeded, compared as at
    config 2."""
    import gc
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gc.collect()
    torch.cuda.empty_cache()
    gm, Mx = cases.load_growmap(GM128), 384
    engines = (GraphInferenceEngine(Mx, "random-init:llama-3.2-1b:1", device=DEV, batch_size=2),
               GraphInferenceEngineTG(Mx, "random-init:llama-3.1-8b:2", device=DEV, batch_size=2))
    g = torch.Generator().manual_seed(21)
    prompts = [torch.randint(3, 128256, (n,), generator=g).to(DEV) for n in (90, 128)]
    Ts, tps, seeds = [0.7, 0.6], [1.0, 0.95], [31, 32]
    runs = {name: _decode(engines, prompts, gm, pol, Ts, tps, seeds, Mx, 4)[0]
            for name, pol in (("mixed", ["spec", "greedy"]), ("greedy", "greedy"), ("spec", "spec"))}
    _same_slots(runs["mixed"], runs["greedy"], (1,), "greedy slot")
    _same_slots(runs["mixed"], runs["spec"], (0,), "spec slot")


# ------------------------------------------------------------------------------------------------ admission
def _admission_run(policy0, admit_pol, iters=8, at=2, at2=5):
    """B = 3 seeded tree of `policy0`: slot 1 frozen after step at-1 and given a prompt of `admit_pol` at step `at`, slot 2
    frozen after step at2-1 and given a "spec" prompt (a "greedy" one in an all-greedy tree) at step at2."""
    from sequoia_b200.batch import BatchTree
    gm = cases.load_growmap(GM)
    d, t = _engines(3)
    prompts = [cases.make_prompt(140 + i, n) for i, n in enumerate((90, 64, 110))]
    bt = BatchTree(d, t, prompts, gm, policy=policy0, temperature=[0.6, 0.8, 0.7], top_p=1.0, max_length=256,
                   seeds=[41, 42, 43])
    assert (bt.r is None) == (policy0 == "greedy")
    steps, captures = [], {}
    for it in range(iters):
        if it == at:
            bt.admit(1, cases.make_prompt(150, 72), temperature=0.9, seed=51, policy=admit_pol)
            captures["first"] = dict(bt.captures)
        if it == at2:
            second = "greedy" if policy0 == admit_pol == "greedy" else "spec"
            bt.admit(2, cases.make_prompt(151, 66), temperature=0.75, seed=52, policy=second)
        bt.construct_grow_map()
        steps.append([(v.cpu().clone(), a, term) for v, a, term in bt.verify()])
        if it == at - 1:
            bt.freeze(1)
        if it == at2 - 1:
            bt.freeze(2)
    return steps, bt, captures


def test_mixing_admissions():
    """A greedy prompt admitted into a seeded spec batch, then a spec prompt into another slot: one recapture each of the
    draft, steady and post graphs; the greedy slot decodes as in an all-greedy batch with the same schedule; the other
    slots as in a run whose first admission was a spec prompt.  A spec prompt admitted into an all-greedy batch (r and
    rand allocated then) decodes as in the all-spec run."""
    mixed, bt, cap = _admission_run("spec", "greedy")
    assert cap["first"] == {"draft": 1, "post": 1, "steady": 1}
    assert bt.mixed and bt.captures == {"draft": 2, "post": 2, "steady": 2}, bt.captures
    greedy, _, _ = _admission_run("greedy", "greedy")
    spec, _, _ = _admission_run("spec", "spec")
    lazy, bt_lazy, _ = _admission_run("greedy", "spec")
    assert bt_lazy.mixed and bt_lazy.r is not None and bt_lazy.captures == {"draft": 2, "post": 2, "steady": 2}
    _same_slots(mixed[2:], greedy[2:], (1,), "admitted greedy slot")
    _same_slots(mixed, spec, (0, 2), "the other slots")
    _same_slots(lazy[2:], spec[2:], (1,), "a spec admission into an all-greedy batch")
    _same_slots(lazy[5:], spec[5:], (2,), "the second spec admission")
    _same_slots(lazy, greedy, (0,), "the all-greedy batch's remaining greedy slot")


# ------------------------------------------------------------------------------------------------ launches
def test_mixed_steady_step_launches(monkeypatch):
    """A mixed steady step is two graph replays and one host sync; its steady graph has the all-spec tree's launches plus
    argmax_rows and the greedy walk, its draft graph the same count.  A list of equal policies launches what the string
    does."""
    from sequoia_b200 import _lib
    from sequoia_b200.batch import BatchTree
    gm = cases.load_growmap(GM)
    launches = {}
    for name, pol in (("spec", "spec"), ("spec_list", ["spec", "spec"]), ("greedy", "greedy"),
                      ("greedy_list", ["greedy", "greedy"]), ("mixed", ["greedy", "spec"])):
        d, t = _engines(2)
        torch.manual_seed(1)
        bt = BatchTree(d, t, [cases.make_prompt(80, 60), cases.make_prompt(81, 70)], gm, policy=pol, temperature=0.6,
                       top_p=1.0, max_length=256)
        for _ in range(2):
            bt.construct_grow_map()
            bt.verify()
        syncs = []
        real_sync = torch.cuda.Stream.synchronize
        monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
        monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: syncs.append(1))
        r0, c0 = dict(bt.replays), _lib.launch_count()
        for _ in range(3):
            bt.construct_grow_map()
            bt.verify()
        monkeypatch.undo()
        torch.cuda.synchronize()
        assert not any(bt.frozen)
        assert bt.replays["draft"] - r0["draft"] == 3 and bt.replays["steady"] - r0["steady"] == 3, name
        assert len(syncs) == 3, "one host sync per step"
        assert _lib.launch_count() == c0, "a steady step launches only through graph replays"
        launches[name] = (bt.graph_launches["draft"], bt.graph_launches["steady"], bt.graph_launches["post"])
    assert launches["spec_list"] == launches["spec"] and launches["greedy_list"] == launches["greedy"], launches
    sd, ss, sp = launches["spec"]
    assert launches["mixed"] == (sd, ss + 2, sp + 2), launches
