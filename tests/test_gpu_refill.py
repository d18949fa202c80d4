"""Per-sequence sampling parameters and slot admission in a batch (BatchTree.admit).

Kernel level: the per-sequence entry points with all-equal arrays against the scalar batched ones, and with distinct
values against B = 1 launches at each sequence's own values, bit for bit.  BatchTree level: a reused slot decodes as a
fresh tree would, an admission leaves the other sequences' results alone, and new sampling values need no new graphs."""
import contextlib
import os

import pytest
import torch

import cases

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
F16 = torch.float16
GM = "L40_growmaps/8x8-tree.pt"
M = 640
ST_P, ST_N_NEW, ST_M, ST_FROZEN = 0, 3, 8, 9
VOCABS = [32000, 49152, 128256]           # accept walk NCH = 1, 2, 4; sampling and top-p clusters of 1, 2, 4 CTAs


def ops():
    from sequoia_b200 import ops as _ops
    return _ops


@contextlib.contextmanager
def _env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def tree():
    from sequoia_b200.tree import _Static
    return _Static(cases.load_growmap(GM), DEV)


def _f32(vals):
    return torch.tensor(vals, dtype=torch.float32, device=DEV)


def _state(B, frozen=()):
    st = torch.zeros(B, 16, dtype=torch.int32)
    for b in range(B):
        st[b, ST_P] = 40 + 37 * b
        st[b, ST_M] = M
    for b in frozen:
        st[b, ST_FROZEN] = 1
    return st.to(DEV)


def _draft_layout(tree, per_seq, V):
    """per-sequence (S, V) node-indexed draft logits -> the level-block layout of len(per_seq) sequences"""
    B = len(per_seq)
    levels = [(0, 1)] + [(lv["n0"], lv["tb"]) for lv in tree.levels]
    base, step = ops().draft_row_tables(levels, tree.S, B, DEV)
    buf = torch.full((B * tree.S, V), -7.0, dtype=F16, device=DEV)
    for b in range(B):
        buf[base.long() + b * step.long()] = per_seq[b]
    return buf, base, step


# ------------------------------------------------------------------------------------------------ sample_level
def _sample(tree, buf, base, step, rand, T, mode, tokens, state):
    for lv in tree.levels:
        kw = dict(parent_rows=lv["parents"], child_first=lv["first"], n_branch=lv["nb"], tokens=tokens, state=state)
        if isinstance(T, torch.Tensor):
            ops().sample_level_batch_per_seq(buf, base, step, rand, lv["n_parents"], lv["k"], T, mode, **kw)
        else:
            ops().sample_level_batch(buf, base, step, rand, lv["n_parents"], lv["k"], T, mode, **kw)
    torch.cuda.synchronize()


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("mode", [0, 1])
def test_sample_level_per_seq(V, mode, tree):
    B, S = 3, tree.S
    g = torch.Generator(device=DEV).manual_seed(V + mode)
    per_seq = [(torch.randn(S, V, generator=g, device=DEV) * 2).to(F16) for _ in range(B)]
    rand = torch.rand(B, S, V, generator=g, device=DEV).to(F16)
    buf, base, step = _draft_layout(tree, per_seq, V)
    # all-equal arrays == the scalar entry point
    state = _state(B)
    got, want = (torch.full((B, M), -5, dtype=torch.int64, device=DEV) for _ in range(2))
    _sample(tree, buf, base, step, rand, _f32([0.6] * B), mode, got, state)
    _sample(tree, buf, base, step, rand, 0.6, mode, want, state)
    assert torch.equal(got, want)
    # distinct values, sequence 1 frozen: each sequence == a B = 1 launch at its own T
    Ts = [0.45, 0.8, 1.3]
    state = _state(B, frozen=(1,))
    got = torch.full((B, M), -5, dtype=torch.int64, device=DEV)
    _sample(tree, buf, base, step, rand, _f32(Ts), mode, got, state)
    for b in range(B):
        want = torch.full((1, M), -5, dtype=torch.int64, device=DEV)
        if b != 1:
            buf1, base1, step1 = _draft_layout(tree, [per_seq[b]], V)
            _sample(tree, buf1, base1, step1, rand[b:b + 1], Ts[b], mode, want, state[b:b + 1].clone())
        assert torch.equal(got[b], want[0]), (V, mode, b)
    P0 = int(state[0, ST_P])
    assert bool((got[0, P0:P0 + S - 1] >= 0).all())


# ------------------------------------------------------------------------------------------------ accept walk
def _walk_inputs(tree, B, V, seed):
    S = tree.S
    g = torch.Generator(device=DEV).manual_seed(seed)
    per_seq, target = [], []
    for b in range(B):
        d = (torch.randn(S, V, generator=g, device=DEV) * 0.5).to(F16)
        per_seq.append(d)
        target.append((d.float() + [0.0, 0.3, 0.05][b] * torch.randn(S, V, generator=g, device=DEV)).to(F16))
    tokens = torch.randint(3, V, (B, M), generator=g, device=DEV)
    pos = torch.randint(0, M, (B, M), generator=g, device=DEV)
    r = torch.rand(B, M, generator=g, device=DEV).to(F16)
    noise = torch.empty(B, V, device=DEV).exponential_(1.0, generator=g).to(F16)
    return per_seq, torch.cat(target), tokens, pos, r, noise


def _walk(tree, target, buf, base, step, r, noise, T, tokens, pos, acc, state):
    args = (target, buf, base, step, r, noise, tree.succ_off, tree.succ, tree.depth, tree.S, T, tokens, pos, acc, state, M)
    if isinstance(T, torch.Tensor):
        ops().accept_stochastic_batch_per_seq(*args)
    else:
        ops().accept_stochastic_batch(*args)
    torch.cuda.synchronize()


@pytest.mark.parametrize("V", VOCABS)
def test_accept_stochastic_per_seq(V, tree):
    B, S = 3, tree.S
    per_seq, target, tokens0, pos0, r, noise = _walk_inputs(tree, B, V, seed=V + 1)
    buf, base, step = _draft_layout(tree, per_seq, V)

    def fresh(n, st):
        return tokens0[:n].clone(), pos0[:n].clone(), torch.full((n, S), -1, dtype=torch.int32, device=DEV), st.clone()

    st = _state(B)
    a, b_ = fresh(B, st), fresh(B, st)
    _walk(tree, target, buf, base, step, r, noise, _f32([0.6] * B), *a)
    _walk(tree, target, buf, base, step, r, noise, 0.6, *b_)
    for x, y in zip(a, b_):
        assert torch.equal(x, y)
    Ts = [0.5, 0.9, 1.4]
    st = _state(B, frozen=(1,))
    got = fresh(B, st)
    _walk(tree, target, buf, base, step, r, noise, _f32(Ts), *got)
    deepest = 0
    for b in range(B):
        tok, pos, acc, s = tokens0[b:b + 1].clone(), pos0[b:b + 1].clone(), torch.full((1, S), -1, dtype=torch.int32,
                                                                                      device=DEV), st[b:b + 1].clone()
        if b != 1:
            buf1, base1, step1 = _draft_layout(tree, [per_seq[b]], V)
            _walk(tree, target[b * S:(b + 1) * S], buf1, base1, step1, r[b:b + 1], noise[b:b + 1], Ts[b], tok, pos, acc,
                  s)
        for x, y in zip(got, (tok, pos, acc, s)):
            assert torch.equal(x[b], y[0]), (V, b)
        deepest = max(deepest, int(got[3][b, ST_N_NEW]))
    assert deepest >= 2, "the near-equal rows should accept a path of several nodes"


# ------------------------------------------------------------------------------------------------ top-p filter
@pytest.mark.parametrize("V", VOCABS)
def test_top_p_filter_per_seq(V):
    B, R = 3, 16
    g = torch.Generator(device=DEV).manual_seed(V + 2)
    logits0 = (torch.randn(B * R, V, generator=g, device=DEV) * 3).to(F16)
    got = logits0.clone()
    ops().top_p_filter_per_seq_(got, _f32([0.9] * B), _f32([0.6] * B), R)
    want = ops().top_p_filter_(logits0.clone(), 0.9, 0.6)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert bool(torch.isinf(got).any()), "the filter must remove tokens"
    tps, Ts = [0.8, 1.0, 0.95], [0.5, 0.7, 1.1]
    got = logits0.clone()
    ops().top_p_filter_per_seq_(got, _f32(tps), _f32(Ts), R)
    torch.cuda.synchronize()
    for b in range(B):
        rows = slice(b * R, (b + 1) * R)
        want = ops().top_p_filter_(logits0[rows].clone(), tps[b], Ts[b])
        torch.cuda.synchronize()
        assert torch.equal(got[rows], want), (V, b)
    assert torch.equal(got[R:2 * R].view(torch.int16), logits0[R:2 * R].view(torch.int16)), "top_p = 1: rows untouched"


# ------------------------------------------------------------------------------------------------ BatchTree admission
def _engines(B, Mx=256):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    dcfg, dw = cases.model_weights("draft")
    tcfg, tw = cases.model_weights("target")
    with _env(SQ_DRAFT_ATTN=0, SQ_ATTN_SPLITS=1):
        return (GraphInferenceEngine(Mx, {"config": dcfg, "state_dict": dw}, device=DEV, batch_size=B),
                GraphInferenceEngineTG(Mx, {"config": tcfg, "state_dict": tw}, device=DEV, batch_size=B))


def _caches(*engines):
    return [t for e in engines for t in (e.engine.kv_cache.k_cache, e.engine.kv_cache.v_cache)]


def test_reused_slot_decodes_like_a_fresh_tree():
    """B = 1: a prompt decodes until it runs out of room, then a second prompt is admitted into the slot and decoded 8
    steps.  Tokens, accept lengths and the KV rows [0, a) equal those of a fresh BatchTree on the second prompt with the
    same draws: nothing of the first prompt (longer, so its KV rows and tokens lie past the second's) is read."""
    from sequoia_b200.batch import BatchTree
    gm, Mx, iters = cases.load_growmap(GM), 256, 8
    S, V = gm["size"], cases.V
    first, second = cases.make_prompt(60, Mx - S - 4), cases.make_prompt(61, 90)
    noise = torch.empty(iters, 1, V, dtype=F16).exponential_(1.0, generator=torch.Generator().manual_seed(7)).to(DEV)
    d1, t1 = _engines(1)
    torch.manual_seed(5)
    bt = BatchTree(d1, t1, [first], gm, temperature=0.6, top_p=1.0, max_length=Mx)
    for _ in range(30):
        bt.construct_grow_map()
        bt.verify()
        if bt.frozen[0]:
            break
    assert bt.frozen[0], "the first prompt should run out of room"
    bt.external_noise = torch.cat([torch.ones(bt.iter, 1, V, dtype=F16, device=DEV), noise])
    torch.manual_seed(6)
    bt.admit(0, second, temperature=0.8, top_p=0.9)
    d2, t2 = _engines(1)
    torch.manual_seed(6)
    ref = BatchTree(d2, t2, [second], gm, temperature=0.8, top_p=0.9, max_length=Mx)
    ref.external_noise = noise
    for it in range(iters):
        out = []
        for tr in (bt, ref):
            tr.construct_grow_map()
            (v, a, term), = tr.verify()
            out.append((v.clone(), a, term))
        (v, a, term), (v_ref, a_ref, term_ref) = out
        assert (a, term) == (a_ref, term_ref) and torch.equal(v, v_ref), it
        for got, want in zip(_caches(d1, t1), _caches(d2, t2)):
            assert torch.equal(got[..., :a, :], want[..., :a, :]), it
        if term:
            break
    assert len(v) > len(second) + iters, "the admitted prompt keeps decoding"


def test_admission_leaves_the_other_sequences_alone():
    """B = 3: slot 1 is frozen after step 2 and given a new prompt at step 3, at its own T and top_p.  Slots 0 and 2
    match a run in which slot 1 stays frozen, bit for bit.  Slot 1 agrees with a lone SpecTree on its prompt at its T and
    top_p (same draws) on at least 95% of the committed positions (the batch's GEMMs see other row counts)."""
    from sequoia_b200.batch import BatchTree, draw_random
    from sequoia_b200.tree import SpecTree, clear_runtimes
    gm, Mx, iters, at = cases.load_growmap(GM), 256, 8, 3
    V = cases.V
    prompts = [cases.make_prompt(70 + i, n) for i, n in enumerate((100, 64, 120))]
    new = cases.make_prompt(73, 80)
    noise = torch.empty(iters, 3, V, dtype=F16).exponential_(1.0, generator=torch.Generator().manual_seed(8)).to(DEV)

    def run(admit):
        d, t = _engines(3)
        torch.manual_seed(4)
        bt = BatchTree(d, t, prompts, gm, temperature=0.6, top_p=1.0, max_length=Mx)
        bt.external_noise = noise
        steps = []
        for it in range(iters):
            if it == at and admit:
                torch.manual_seed(9)
                bt.admit(1, new, temperature=0.8, top_p=0.9)
            bt.construct_grow_map()
            steps.append([(v.clone(), a, term) for v, a, term in bt.verify()])
            if it == at - 1:
                bt.freeze(1)
        return steps, bt, (d, t)

    with_adm, bt, eng = run(True)
    without, bt0, eng0 = run(False)
    for it in range(iters):
        for b in (0, 2):
            (v, a, term), (v0, a0, term0) = with_adm[it][b], without[it][b]
            assert (a, term) == (a0, term0) and torch.equal(v, v0), (it, b)
    for b in (0, 2):
        a = with_adm[-1][b][1]
        for got, want in zip(_caches(*eng), _caches(*eng0)):
            assert torch.equal(got[:, b, ..., :a, :], want[:, b, ..., :a, :]), b
    torch.manual_seed(9)
    r, rand = draw_random([new], Mx, gm["size"], V)
    d1, t1 = _engines(1)
    clear_runtimes()
    lone = SpecTree(d1, t1, new.to(DEV), temperature=0.8, top_p=0.9, max_length=Mx, max_target_seq=Mx, device=DEV,
                    vocab_size=V, grow_map=gm)
    lone.rt.r.copy_(r[0].to(DEV))
    lone.rt.rand.copy_(rand[0].to(DEV))
    lone.rt.external_noise = noise[at:, 1].contiguous()
    for _ in range(iters - at):
        lone.construct_grow_map()
        v, _, _, term = lone.verify()
        if term:
            break
    lone.rt.external_noise = None
    got, want = with_adm[-1][1][0].cpu(), v.cpu()
    assert torch.equal(got[:len(new)], new)
    k = min(len(got), len(want))
    same = int((got[:k] == want[:k]).sum()) - len(new)
    total = max(len(got), len(want)) - len(new)
    assert total > 0 and same >= 0.95 * total, (same, total)


def test_admissions_reuse_the_graphs(monkeypatch):
    """New T and top_p values need no new graph; the first top_p < 1 captures the steady and post graphs once more
    (the filter joins op_accept).  A steady step is two replays and one host sync; an admission step (admit + draft +
    verify) has one host sync too, the verify's: admit's host-to-device copies are asynchronous."""
    from sequoia_b200 import _lib
    from sequoia_b200.batch import BatchTree
    gm = cases.load_growmap(GM)
    d, t = _engines(2)
    torch.manual_seed(1)
    bt = BatchTree(d, t, [cases.make_prompt(80, 60), cases.make_prompt(81, 70)], gm, temperature=[0.6, 0.7],
                   top_p=1.0, max_length=256)
    for _ in range(2):
        bt.construct_grow_map()
        bt.verify()
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}
    steady_launches = bt.graph_launches["steady"]

    syncs = []
    real_sync = torch.cuda.Stream.synchronize

    def count(fn):
        syncs.clear()
        monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
        monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: syncs.append(1))
        fn()
        monkeypatch.undo()
        return len(syncs)

    def step():
        bt.construct_grow_map()
        bt.verify()

    def steady_step():
        r0, c0, k0 = dict(bt.replays), _lib.launch_count(), bt.kernel_launches()
        assert count(step) == 1, "one host sync per steady step"
        assert bt.replays["draft"] == r0["draft"] + 1 and bt.replays["steady"] == r0["steady"] + 1
        assert _lib.launch_count() == c0, "a steady step launches only through graph replays"
        assert bt.kernel_launches() - k0 == bt.graph_launches["draft"] + bt.graph_launches["steady"]

    def admission(b, seed, T, tp, recapture=False):
        bt.freeze(b)
        assert count(lambda: bt.admit(b, cases.make_prompt(seed, 50 + seed % 7), temperature=T, top_p=tp)) == 0
        r0, k0 = dict(bt.replays), bt.kernel_launches()
        n = count(step)
        if not recapture:                               # (a capture synchronises its side stream)
            assert n == 1, "an admission step has one host sync, the verify's"
        assert bt.replays["post"] == r0["post"] + 1 and bt.replays["steady"] == r0["steady"]
        assert bt.kernel_launches() - k0 == bt.graph_launches["draft"] + bt.graph_launches["post"]

    steady_step()
    admission(0, 90, 0.9, 1.0)                          # new temperature: same graphs
    steady_step()
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}
    admission(1, 91, 0.5, 0.8, recapture=True)          # first top_p < 1: steady and post once more
    step()                                              # (the steady graph's capture)
    steady_step()
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2}
    assert bt.graph_launches["steady"] == steady_launches + 1, "the top-p filter is one more launch"
    admission(0, 92, 1.1, 0.7)
    steady_step()
    admission(1, 93, 0.7, 1.0)
    steady_step()
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2}, "no recapture after the filter entered"
    assert bt.T_dev.tolist() == pytest.approx([1.1, 0.7]) and bt.top_p_dev.tolist() == pytest.approx([0.7, 1.0])
