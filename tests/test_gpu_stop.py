"""Per-sequence stop ids and token budgets on the device (sq_accept_*_batch_stop, BatchTree(stop_tokens=...,
max_new_tokens=...)).

Kernel level: with an empty stop set and no limit each stop walk commits exactly what its walk commits, and leaves frozen
slots alone; with stop ids and limits its SQ_ST_FINISH / SQ_ST_END are oracle/stop.py's cut of the unstopped output; a
greedy path through the Llama-2 end ids 0 and 2 is walked through.  BatchTree level: each slot with a stop set or a
budget returns, step for step, the output of a run without a stop rule cut at its end; default mode launches what it
launched before; stop mode is captured once; refill admissions carry their own settings; one run at V = 128256."""
import pytest
import torch

import cases
from oracle.stop import cut
from test_gpu_mixed_policy import GM128, _walk_inputs
from test_gpu_refill import DEV, GM, M, ST_FROZEN, ST_N_NEW, ST_P, _draft_layout, _f32, _state, ops

pytestmark = pytest.mark.gpu

ST_ACCEPT_LEN, ST_TERMINAL, ST_FINISH, ST_END = 1, 2, 10, 11
VOCABS = [32000, 49152, 128256]           # accept walk NCH = 1, 2, 4


@pytest.fixture(scope="module")
def tree():
    from sequoia_b200.tree import _Static
    return _Static(cases.load_growmap(GM), DEV)


def _i32(vals):
    return torch.tensor(vals, dtype=torch.int32, device=DEV)


def _stop_rows(sets):
    return _i32([list(s) + [-1] * (8 - len(s)) for s in sets])


class _Walks:
    """One set of walk inputs for B sequences; run(kind, stop=None | (stop_ids, end_limit)) -> [tokens, position_ids,
    accept_idx, state] after the walk(s) of `kind` ("spec", "greedy" or "mixed"; mixed: even slots greedy)."""

    def __init__(self, tree, B, V, seed, frozen=()):
        self.tree, self.B, self.S = tree, B, tree.S
        per_seq, self.target, self.tokens0, self.pos0, self.r, self.noise = _walk_inputs(tree, B, V, seed)
        self.buf, self.base, self.step = _draft_layout(tree, per_seq, V)
        self.st0 = _state(B, frozen=frozen)
        for b in frozen:                                   # words 10 and 11 of a frozen slot must stay as they are
            self.st0[b, ST_FINISH], self.st0[b, ST_END] = 77, 88
        self.T = _f32([0.6 + 0.1 * (b % 5) for b in range(B)])
        self.greedy = _i32([1 - b % 2 for b in range(B)])
        self.target_token = ops().argmax_rows(self.target)

    def fresh(self):
        return [self.tokens0.clone(), self.pos0.clone(), torch.full((self.B, self.S), -1, dtype=torch.int32, device=DEV),
                self.st0.clone()]

    def run(self, kind, stop=None):
        t, S = self.tree, self.S
        bufs = self.fresh()
        sargs = (self.target, self.buf, self.base, self.step, self.r, self.noise, t.succ_off, t.succ, t.depth, S, self.T)
        gargs = (self.target_token, t.succ_off, t.succ, t.depth, S)
        g = self.greedy if kind == "mixed" else None
        if kind in ("greedy", "mixed"):
            if stop is not None:
                ops().accept_greedy_batch_stop(*gargs, g, *stop, *bufs, M)
            elif kind == "mixed":
                ops().accept_greedy_batch_mixed(*gargs, g, *bufs, M)
            else:
                ops().accept_greedy_batch(*gargs, *bufs, M)
        if kind in ("spec", "mixed"):
            if stop is not None:
                ops().accept_stochastic_batch_stop(*sargs, g, *stop, *bufs, M)
            elif kind == "mixed":
                ops().accept_stochastic_batch_mixed(*sargs, g, *bufs, M)
            else:
                ops().accept_stochastic_batch_per_seq(*sargs, *bufs, M)
        torch.cuda.synchronize()
        return [x.cpu() for x in bufs]


@pytest.mark.parametrize("kind", ["spec", "greedy", "mixed"])
@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("V", VOCABS)
def test_empty_stop_set_commits_what_the_walk_commits(V, B, kind, tree):
    """No stop id and no limit: tokens, position_ids, accept_idx and the whole state row (words 10 and 11 are 0 before
    and after) equal the current walk's, on paths without a 0 or 2; the frozen slot stays bit-identical."""
    frozen = (B - 1,) if B > 1 else ()
    w = _Walks(tree, B, V, seed=V + 10 * B + len(kind), frozen=frozen)
    ref = w.run(kind)
    got = w.run(kind, stop=(_stop_rows([()] * B), _i32([0] * B)))
    live = [b for b in range(B) if b not in frozen]
    assert not bool(ref[3][live, ST_TERMINAL].any()), "inputs must hold no accepted 0 or 2"
    for i, name in enumerate(("tokens", "position_ids", "accept_idx", "state")):
        assert torch.equal(got[i], ref[i]), (V, B, kind, name)
    sentinel = w.fresh()
    for b in frozen:
        for i in range(4):
            assert torch.equal(got[i][b], sentinel[i][b].cpu()), (V, B, kind, "frozen", i)
        assert int(got[3][b, ST_FINISH]) == 77 and int(got[3][b, ST_END]) == 88
    assert max(int(ref[3][b, ST_N_NEW]) for b in live) >= 1, "the walks should accept nodes"


@pytest.mark.parametrize("kind", ["spec", "greedy", "mixed"])
@pytest.mark.parametrize("V", [32000, 128256])
def test_cut_matches_the_oracle(V, kind, tree):
    """Stop ids taken from each newly committed position (the bonus included), then every budget from 1 to the committed
    count: FINISH, END, tokens[:END] (and everything the walk commits) equal oracle.stop.cut of the unstopped output."""
    B = 3
    w = _Walks(tree, B, V, seed=V + 77 + len(kind))
    free = w.run(kind, stop=(_stop_rows([()] * B), _i32([0] * B)))
    P = [int(w.st0[b, ST_P]) for b in range(B)]
    n = [int(free[3][b, ST_ACCEPT_LEN]) + 1 for b in range(B)]            # no NaN: the bonus is committed
    count = max(n[b] - P[b] for b in range(B))
    cases_run = 0
    for k in range(count):
        for mode in ("stop", "budget", "both"):
            sets, limits = [], []
            for b in range(B):
                j = min(P[b] + k, n[b] - 1)
                tok = int(free[0][b, j])
                sets.append((tok,) if mode != "budget" else ())
                limits.append(P[b] + k + 1 if mode != "stop" else 0)
            got = w.run(kind, stop=(_stop_rows(sets), _i32(limits)))
            for b in range(B):
                finish, end = cut(free[0][b].tolist(), P[b], n[b], sets[b], limits[b])
                assert (int(got[3][b, ST_FINISH]), int(got[3][b, ST_END])) == (finish, end), (V, kind, k, mode, b)
                assert finish != 0 or mode == "budget" and limits[b] > n[b]
                assert torch.equal(got[0][b, :end], free[0][b, :end])
                for i in range(3):
                    assert torch.equal(got[i][b], free[i][b]), (V, kind, k, mode, b, i)
                assert torch.equal(got[3][b, :10], free[3][b, :10])
                cases_run += 1
    assert count >= 2 and cases_run >= 18, "the walks should commit a path"


def test_llama3_ids_are_walked_through(tree):
    """V = 128256: a greedy path whose first two accepted tokens are 0 and 2.  The current walk ends at the 0; the stop
    walk with {128009} walks through both; with {2} it ends on the 2 with FINISH = 1."""
    B, V, S = 2, 128256, tree.S
    w = _Walks(tree, B, V, seed=5)
    succ_off, succ = tree.succ_off.cpu().tolist(), tree.succ.cpu().tolist()
    P = int(w.st0[0, ST_P])
    cur = 0
    for tok in (0, 2):                                       # slot 0: node cur's first child holds tok, its row's argmax
        child = succ[succ_off[cur]]
        w.tokens0[0, P - 1 + child] = tok
        w.target[cur, tok] = 60.0
        cur = child
    w.target_token = ops().argmax_rows(w.target)
    ref = w.run("greedy")
    assert int(ref[3][0, ST_TERMINAL]) == 1 and int(ref[3][0, ST_N_NEW]) == 1, "the fixed rule ends at the 0"
    through = w.run("greedy", stop=(_stop_rows([(128009,)] * B), _i32([0] * B)))
    assert int(through[3][0, ST_TERMINAL]) == 0 and int(through[3][0, ST_N_NEW]) >= 3
    assert through[0][0, P:P + 2].tolist() == [0, 2] and int(through[3][0, ST_FINISH]) == 0
    on_two = w.run("greedy", stop=(_stop_rows([(2,), (2,)]), _i32([0] * B)))
    assert (int(on_two[3][0, ST_FINISH]), int(on_two[3][0, ST_END])) == (1, P + 2)
    assert torch.equal(on_two[0][0], through[0][0])


# ------------------------------------------------------------------------------------------------ BatchTree
def _pair_engines(B, Mx=256):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    return (GraphInferenceEngine(Mx, "random-init:llama-68m:1", device=DEV, batch_size=B),
            GraphInferenceEngineTG(Mx, "random-init:llama-68m:2", device=DEV, batch_size=B))


def _run(engines, prompts, gm, seeds, iters=8, Mx=256, **kw):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    bt = BatchTree(d, t, prompts, gm, temperature=0.7, max_length=Mx, seeds=seeds, **kw)
    steps = []
    for _ in range(iters):
        bt.construct_grow_map()
        steps.append([(v.cpu().clone(), a, term) for v, a, term in bt.verify()])
        if all(bt.frozen):
            break
    return steps, bt


def _expect(free, b, plen, stop, budget):
    """(step, end, reason) at which slot b of the unstopped run `free` ends under (stop, budget); None if it does not."""
    prev = plen
    for it, step in enumerate(free):
        v, _, term = step[b]
        n = len(v)
        finish, end = cut(v.tolist(), prev, n, stop or (), plen + budget if budget else 0)
        if finish:
            return it, end, "stop" if finish == 1 else "length"
        if term:
            return None
        prev = n
    return None


def _check_prefix(free, got, bt, prompts, stops, budgets):
    """Every slot: the steps before its end equal the unstopped run's, the ending step returns that step's tokens cut at
    END with terminal True and the same accept length, and finish_reason says why."""
    ended = 0
    for b in range(len(prompts)):
        e = _expect(free, b, len(prompts[b]), stops[b], budgets[b])
        last = len(got) if e is None else e[0]
        for it in range(min(last, len(got))):
            (v, a, term), (v0, a0, term0) = got[it][b], free[it][b]
            assert (a, term) == (a0, term0) and torch.equal(v, v0), (b, it)
        if e is None:
            assert bt.finish_reason[b] in (None, "room"), (b, bt.finish_reason[b])
            continue
        it, end, reason = e
        (v, a, term), (v0, a0, _) = got[it][b], free[it][b]
        assert term and a == a0 and torch.equal(v, v0[:end]) and len(v) == end, (b, it, end, len(v))
        assert bt.finish_reason[b] == reason and bt.frozen[b], (b, bt.finish_reason[b], reason)
        ended += 1
    return ended


def _settings(free, B):
    """Per-slot stop sets (tokens the unstopped run commits, at several steps) and budgets, some slots with neither."""
    def tok(b, it, pos=-1):
        it = min(it, len(free) - 1)
        return int(free[it][b][0][pos])
    stops, budgets = [], []
    for b in range(B):
        r = b % 4
        stops.append([tok(b, 1 + b % 3)] if r == 0 else [tok(b, 2), 123] if r == 2 else [] if r == 3 else None)
        budgets.append(None if r in (0, 3) else 1 + 3 * b)
    return stops, budgets


@pytest.mark.parametrize("policy", ["spec", "greedy", "mixed"])
@pytest.mark.parametrize("B", [3, 8])
def test_batch_tree_outputs_are_prefixes(B, policy):
    """Seeded 68m pairs: each slot with a stop set or a budget returns the output of a stop_tokens=[] run step for step
    up to its end and that step's tokens cut at END; the other slots are unaffected."""
    gm = cases.load_growmap(GM)
    engines = _pair_engines(B)
    prompts = [cases.make_prompt(400 + i, 40 + 9 * i).to(DEV) for i in range(B)]
    seeds = [500 + i for i in range(B)]
    pol = ["greedy" if b % 2 == 0 else "spec" for b in range(B)] if policy == "mixed" else policy
    free, bt0 = _run(engines, prompts, gm, seeds, policy=pol, stop_tokens=[])
    assert bt0.use_stop and not any(bt0.finish_reason)
    stops, budgets = _settings(free, B)
    got, bt = _run(engines, prompts, gm, seeds, policy=pol, stop_tokens=stops, max_new_tokens=budgets)
    assert bt.graph_launches == bt0.graph_launches
    assert _check_prefix(free, got, bt, prompts, stops, budgets) >= 2


def test_default_mode_is_unchanged():
    """stop_tokens=None / max_new_tokens=None: the same graphs and outputs as a tree built without them; stop mode has
    the same launch counts (the stop walks replace the walks)."""
    gm = cases.load_growmap(GM)
    engines = _pair_engines(3)
    prompts = [cases.make_prompt(420 + i, n).to(DEV) for i, n in enumerate((50, 70, 90))]
    plain, bt0 = _run(engines, prompts, gm, [1, 2, 3], policy=["spec", "greedy", "spec"])
    none, bt1 = _run(engines, prompts, gm, [1, 2, 3], policy=["spec", "greedy", "spec"], stop_tokens=None,
                     max_new_tokens=None)
    assert not bt1.use_stop and bt1.graph_launches == bt0.graph_launches
    _, bt2 = _run(engines, prompts, gm, [1, 2, 3], iters=2, policy=["spec", "greedy", "spec"], stop_tokens=[])
    assert bt2.graph_launches == bt0.graph_launches
    assert len(plain) == len(none)
    for it in range(len(plain)):
        for b in range(3):
            (v, a, term), (v0, a0, term0) = none[it][b], plain[it][b]
            assert (a, term) == (a0, term0) and torch.equal(v, v0), (it, b)


def test_stop_admissions_capture_once():
    """The first admission with a stop set captures steady and post once more; later admissions with other sets and
    budgets capture nothing and the admitted slot ends at its budget exactly."""
    from sequoia_b200.batch import BatchTree
    gm = cases.load_growmap(GM)
    d, t = _pair_engines(2)
    bt = BatchTree(d, t, [cases.make_prompt(430, 60), cases.make_prompt(431, 70)], gm, policy=["spec", "greedy"],
                   temperature=0.7, max_length=256, seeds=[1, 2])

    def step():
        bt.construct_grow_map()
        return bt.verify()

    def admission(b, seed, **kw):
        bt.freeze(b)
        prompt = cases.make_prompt(seed, 50 + seed % 7)
        bt.admit(b, prompt, seed=seed, **kw)
        return len(prompt)
    step()
    step()
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1} and not bt.use_stop
    admission(1, 440)
    step()
    step()
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}, "a default-mode admission captures nothing"
    admission(0, 441, stop_tokens=[7, 9])
    step()
    step()
    assert bt.use_stop and bt.captures == {"draft": 1, "post": 2, "steady": 2}
    for seed, budget in ((442, 3), (443, 1), (444, 6)):
        plen = admission(0, seed, stop_tokens=[], max_new_tokens=budget)
        for _ in range(budget + 1):
            res = step()
            if bt.frozen[0]:
                break
        assert bt.finish_reason[0] == "length" and len(res[0][0]) == plen + budget, (seed, budget)
        assert bt.end_limit_dev[0].item() == plen + budget
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2}, "no recapture after stop mode started"


def test_refill_gives_each_prompt_its_own_settings():
    """testbed.decode_refill with per-prompt budgets and stop sets: every output ends at its own budget exactly or on its
    first stop id (no stop id earlier among its new tokens)."""
    import testbed
    from sequoia_b200.batch import BatchTree
    gm = cases.load_growmap(GM)
    d, t = _pair_engines(3)
    prompts = [cases.make_prompt(450 + i, 40 + 7 * i).to(DEV) for i in range(8)]
    budgets = [2, 5, 9, 3, 14, 1, 7, 4]
    stops = [[11 * i + 3, 17] for i in range(8)]
    seeds = [600 + i for i in range(8)]
    bt = BatchTree(d, t, prompts[:3], gm, temperature=0.7, max_length=256, seeds=seeds[:3], stop_tokens=stops[:3],
                   max_new_tokens=budgets[:3])
    outputs, _, _, order = testbed.decode_refill(bt, prompts, [10 ** 9] * 8, stop=frozenset(), seeds=seeds,
                                                 device_stop=(stops, budgets))
    assert sorted(order) == list(range(8))
    for i, out in enumerate(outputs):
        new = out[len(prompts[i]):].tolist()
        hits = [j for j, x in enumerate(new) if x in stops[i]]
        assert hits in ([], [len(new) - 1]), (i, new)
        assert len(new) == budgets[i] or (hits and len(new) <= budgets[i]), (i, len(new), budgets[i])


def test_stop_batch_llama3_vocab():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 2, seeded: the Llama 3 end ids plus a token the unstopped run
    commits on slot 0, a budget on slot 1; both are prefixes of the stop_tokens=[] run."""
    import gc
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gc.collect()
    torch.cuda.empty_cache()
    gm, Mx = cases.load_growmap(GM128), 384
    engines = (GraphInferenceEngine(Mx, "random-init:llama-3.2-1b:1", device=DEV, batch_size=2),
               GraphInferenceEngineTG(Mx, "random-init:llama-3.1-8b:2", device=DEV, batch_size=2))
    g = torch.Generator().manual_seed(29)
    prompts = [torch.randint(3, 128256, (n,), generator=g).to(DEV) for n in (90, 128)]
    free, bt0 = _run(engines, prompts, gm, [71, 72], iters=4, Mx=Mx, stop_tokens=[])
    assert bt0.V == 128256
    stops = [[128001, 128008, 128009, int(free[1][0][0][-1])], [128009]]
    budgets = [None, 3]
    got, bt = _run(engines, prompts, gm, [71, 72], iters=4, Mx=Mx, stop_tokens=stops, max_new_tokens=budgets)
    assert _check_prefix(free, got, bt, prompts, stops, budgets) >= 1
