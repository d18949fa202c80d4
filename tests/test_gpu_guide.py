"""Guided decoding on the device (sq_guide_states_batch, sq_guide_mask_rows_batch, sq_guide_advance_batch,
BatchTree(guide=...)).

Kernel level: the advance kernel followed by the states and mask kernels against oracle/guide.py bit for bit, at V in
{32000, 32776, 128256} and B in {1, 3, 8}, on the config-2, 16-chain and 16x8 trees, with committed states reached through
0 .. max_depth + 1 advanced tokens, paths through disallowed ids, dead sequences, and NaN and +inf at disallowed ids;
unguided and frozen sequences and the rows past B*S byte-identical; the advance kernel's stop cut and dead state; the
mask commutes with the logit bias, the ban and the penalties bit for bit.
The walk change: a one-level tree whose node 2 is accepted alone at slot a commits node 2's token and then the bonus
for a guided sequence, and the bonus twice (SpecTree's order) for an unguided one.
BatchTree level, on the branching config-2 and 16x8 trees: every generated token of every guided slot is accepted by its
guide; a chain guide forces an exact output and then a stop id; a choice trie ends in one of its choices; a refill
admission switches guides; V = 128256; logprobs; the "guide" finish of a greedy slot whose only allowed ids are banned;
the first generated token of a seeded guided "spec" slot follows softmax(masked row / T) (chi-square over 4000 seeds);
unguided slots commit what they commit without guides; graphs equal eager; one recapture at the first guide only."""
import random

import pytest
import torch

import cases
from oracle import guide as O
from oracle.bad_words import process_rows as ban_rows
from oracle.logit_bias import process_rows as bias_rows
from oracle.penalty import penalize_rows
from sequoia_b200.guide import GuideState, TokenGuide
from test_gpu_bad_words import _ban, _context, _decode, _same, _tree
from test_gpu_logit_bias import _device_rows as bias_device_rows
from test_gpu_mixed_policy import GM128
from test_gpu_refill import DEV, F16, _engines, ops

pytestmark = pytest.mark.gpu

ST_P, ST_ACCEPT_LEN, ST_TERMINAL, ST_M, ST_FROZEN, ST_FINISH, ST_END = 0, 1, 2, 8, 9, 10, 11
ST_GUIDED, ST_GUIDE_STATE, ST_GUIDE_POS = 12, 13, 14
GROWMAPS = {"config2": GM128, "chain": "L40_growmaps/16-chain.pt", "tree16x8": "L40_growmaps/16x8-tree.pt"}
ALPHA = list(range(3, 11))                                 # the small alphabet the kernel tests' tokens come from


def _bits16(x):
    return x.view(torch.int16)


def _random_guide(V, seed, n=6):
    """States over ALPHA (and a few large ids) that allow most of it, some with a default."""
    rnd = random.Random(seed)
    states = []
    for i in range(n):
        edges = {t: rnd.randrange(n) for t in rnd.sample(ALPHA, rnd.randint(3, 7))}
        edges.update({rnd.randrange(V): rnd.randrange(n) for _ in range(rnd.choice([0, 40, 3000]))})
        if i % 3 == 1:
            banned = set(rnd.sample(ALPHA, 3)) - edges.keys() | {V - 1} - edges.keys()
            states.append(GuideState(edges=edges, default=rnd.randrange(n), banned=banned))
        else:
            states.append(GuideState(edges=edges))
    return TokenGuide(states, start=rnd.randrange(n))


def _table(guides, V):
    blobs = [None if g is None else g.pack(V).to(DEV) for g in guides]
    table = torch.tensor([0 if b is None else b.data_ptr() for b in blobs], dtype=torch.int64, device=DEV)
    return table, blobs


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("V", [32000, 32776, 128256])
@pytest.mark.parametrize("tree", list(GROWMAPS))
def test_kernels_match_oracle(V, tree):
    from sequoia_b200.tree import _Static
    gm = cases.load_growmap(GROWMAPS[tree])
    st = _Static(gm, DEV)
    S, M, md = gm["size"], 640, int(gm["depth"].max())
    leaves = stays = False
    for B in (1, 3, 8):
        g = torch.Generator().manual_seed(V + B + S)
        tokens = torch.tensor(ALPHA)[torch.randint(0, len(ALPHA), (B, M), generator=g)]
        tokens[:, ::11] = torch.randint(0, V, (B, (M + 10) // 11), generator=g)   # ids most states do not allow
        guides = [_random_guide(V, V * 10 + B * 3 + b) for b in range(B)]
        P = [int(torch.randint(S + 40, M - S, (1,), generator=g)) for _ in range(B)]
        L = [P[b] - b % (md + 2) - 2 for b in range(B)]                     # n_adv + 2 generated tokens
        unguided, frozen = ((), ()) if B == 1 else ((1,), (B - 1,))
        for b in unguided:
            guides[b] = None
        for b in range(0, B, 2):                            # even sequences: committed tokens their guide accepts
            if guides[b] is None:
                continue
            s = guides[b].start
            for pos in range(L[b], P[b]):
                ok = [t for t in ALPHA if O.step(guides[b].states[s], t, V) is not None]
                if ok:
                    tokens[b, pos] = ok[int(torch.randint(0, len(ok), (1,), generator=g))]
                s = O.step(guides[b].states[s], int(tokens[b, pos]), V)
                if s is None:
                    break
        # committed state reached through n_adv advanced tokens: the oracle's state at P - n_adv, then the kernel
        state = torch.zeros(B, 16, dtype=torch.int32)
        state[:, ST_P] = torch.tensor(P)
        state[:, ST_ACCEPT_LEN] = torch.tensor(P) - 1                     # n = a + 1 = P
        state[:, ST_M] = M
        roots = []
        for b in range(B):
            n_adv = b % (md + 2)
            if guides[b] is not None:
                state[b, ST_GUIDED] = 1
                state[b, ST_GUIDE_STATE] = O.state_after(guides[b], tokens[b, L[b]:P[b] - n_adv].tolist(), V)
                state[b, ST_GUIDE_POS] = P[b] - n_adv
                roots.append(O.state_after(guides[b], tokens[b, L[b]:P[b]].tolist(), V))
            else:
                roots.append(0)
        for b in frozen:
            state[b, ST_FROZEN] = 1
        table, _blobs = _table(guides, V)
        state_d, tok_d = state.to(DEV), tokens.to(DEV)
        ops().guide_advance_batch(table, tok_d, state_d, V)
        got_state = state_d.cpu()
        for b in range(B):
            if guides[b] is None or b in frozen:
                assert torch.equal(got_state[b], state[b]), b
                continue
            assert int(got_state[b, ST_GUIDE_STATE]) == roots[b], (b, roots[b])
            want_pos = P[b] if roots[b] >= 0 else L[b] + O.accepted_prefix(guides[b], tokens[b, L[b]:P[b]].tolist(), V)
            if int(state[b, ST_GUIDE_STATE]) < 0:
                want_pos = int(state[b, ST_GUIDE_POS])                     # dead before: left alone
            assert int(got_state[b, ST_GUIDE_POS]) == want_pos, b
        x = (torch.randn(B * S + 3, V, generator=g) * 3).to(F16)
        x[:, 3] = float("nan")
        x[:, 4] = float("inf")
        x[:, V - 1] = float("nan")
        scratch = torch.full((B, S), -7, dtype=torch.int32, device=DEV)
        ops().guide_states_batch(table, tok_d, state_d, st.depth, st.tree_bits, st.tree_words, S, V, scratch)
        got = ops().guide_mask_rows_batch_(x.clone().to(DEV), S, state_d, table, scratch).cpu()
        want = O.process_rows(x, tokens, P, gm["mask"], guides, roots, frozen=[b in frozen for b in range(B)])
        assert torch.equal(_bits16(got), _bits16(want)), (V, tree, B, (_bits16(got) != _bits16(want)).nonzero()[:5])
        for b in set(unguided) | set(frozen):
            assert torch.equal(_bits16(got[b * S:(b + 1) * S]), _bits16(x[b * S:(b + 1) * S])), (b, "untouched")
        assert torch.equal(_bits16(got[B * S:]), _bits16(x[B * S:])), "sentinel rows untouched"
        live = [b for b in range(B) if guides[b] is not None and b not in frozen]
        ns = scratch.cpu()
        leaves |= any(int(ns[b, k]) < 0 for b in live for k in range(1, S))
        stays |= any(int(ns[b, k]) >= 0 for b in live for k in range(1, S))
    assert leaves and stays, "paths that leave their guide and paths that stay in it"


def test_advance_stop_cut_and_dead_state():
    V, M = 32000, 64
    g = TokenGuide([GuideState(edges={5: 1}), GuideState(edges={6: 0, 7: 1})])   # 5 (6 5 | 7)*
    tokens = torch.zeros(4, M, dtype=torch.long)
    tokens[:, 10:20] = torch.tensor([5, 7, 7, 6, 5, 9, 5, 6, 5, 7])
    state = torch.zeros(4, 16, dtype=torch.int32)
    state[:, ST_M] = M
    state[:, ST_GUIDED], state[:, ST_GUIDE_STATE], state[:, ST_GUIDE_POS] = 1, 0, 10
    state[0, ST_ACCEPT_LEN] = 14                                         # n = 15: all allowed
    state[1, ST_ACCEPT_LEN] = 18                                         # n = 19: 9 at 15 is not allowed
    state[2, ST_ACCEPT_LEN], state[2, ST_FINISH], state[2, ST_END] = 18, 1, 14   # the stop cut at 14
    state[3, ST_ACCEPT_LEN], state[3, ST_TERMINAL] = 15, 1               # terminal: n = a = 15
    table, _blobs = _table([g] * 4, V)
    s = state.to(DEV)
    ops().guide_advance_batch(table, tokens.to(DEV), s, V)
    got = s.cpu()
    for b, n in ((0, 15), (2, 14), (3, 15)):
        assert int(got[b, ST_GUIDE_STATE]) == O.state_after(g, tokens[b, 10:n].tolist(), V) >= 0, b
        assert int(got[b, ST_GUIDE_POS]) == n, b
    assert int(got[1, ST_GUIDE_STATE]) == -1 and int(got[1, ST_GUIDE_POS]) == 15
    ops().guide_advance_batch(table, tokens.to(DEV), s, V)                # a dead sequence is left alone
    assert torch.equal(s.cpu()[1], got[1])


def test_mask_commutes_with_bias_ban_and_penalties():
    from sequoia_b200.tree import _Static
    gm = cases.load_growmap("L40_growmaps/4x4-tree.pt")
    st = _Static(gm, DEV)
    S, V, B, M = gm["size"], 32000, 2, 384
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(B * S, V, generator=g) * 4).to(F16)
    tokens = torch.tensor(ALPHA)[torch.randint(0, len(ALPHA), (B, M), generator=g)]
    P, L = [M - S - 5, M - S - 40], [M - S - 60, M - S - 42]
    guides = [_random_guide(V, 11), _random_guide(V, 12)]
    roots = [O.state_after(guides[b], tokens[b, L[b]:P[b]].tolist(), V) for b in range(B)]
    if min(roots) < 0:
        roots = [guides[b].start for b in range(B)]
    state = torch.zeros(B, 16, dtype=torch.int32)
    state[:, ST_P] = torch.tensor(P)
    state[:, ST_GUIDED] = 1
    state[:, ST_GUIDE_STATE] = torch.tensor(roots)
    words = [_context(gm, (tokens, P, L, b, 40, g)) for b in range(B)]
    min_end, end_ids = [P[0] + 2, P[1] + 1], [(0, 2), (9, 11)]
    allowed, bias = [tuple(range(0, V, 2)), None], [tuple((t, 3.0) for t in range(0, 300, 4)),
                                                    tuple((t, -2.0) for t in range(1, 300, 3))]
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=DEV)  # noqa: E731
    reps, freqs, press = [1.25, 0.75], [0.5, -0.25], [0.5, 1.5]
    pen_scratch = torch.zeros(ops().penalty_scratch_words(B, M), dtype=torch.int32, device=DEV)
    table, _blobs = _table(guides, V)
    node = torch.zeros(B, S, dtype=torch.int32, device=DEV)
    sd = state.to(DEV)

    def run(order):
        out = x.clone().to(DEV)
        for op in order:
            if op == "bias":
                ops().logit_bias_rows_batch_(out, S, sd, *bias_device_rows(V, allowed, bias))
            elif op == "ban":
                _ban(out, tokens, P, L, gm, st, words, min_end, end_ids)
            elif op == "guide":
                ops().guide_states_batch(table, tokens.to(DEV), sd, st.depth, st.tree_bits, st.tree_words, S, V, node)
                ops().guide_mask_rows_batch_(out, S, sd, table, node)
            else:
                ops().penalize_rows_batch_(out, tokens.to(DEV), sd, torch.tensor(L, dtype=torch.int32, device=DEV),
                                           st.tree_bits, st.tree_words, S, f32(reps), f32(freqs), f32(press), pen_scratch)
        torch.cuda.synchronize()
        return out.cpu()
    ref = run(("bias", "ban", "guide", "pen"))
    for order in (("guide", "bias", "ban", "pen"), ("bias", "ban", "pen", "guide"), ("ban", "guide", "bias", "pen")):
        assert torch.equal(_bits16(run(order)), _bits16(ref)), order
    oracle = O.process_rows(
        penalize_rows(ban_rows(bias_rows(x, S, allowed, bias), tokens, P, L, gm["mask"], gm["depth"], words, min_end,
                               end_ids), tokens, P, L, gm["mask"], reps, freqs, press),
        tokens, P, gm["mask"], guides, roots)
    assert torch.equal(_bits16(ref), _bits16(oracle))
    assert int(torch.isinf(ref).sum()) > int(torch.isinf(run(("bias", "ban", "pen"))).sum()), "the guide masks"


# ------------------------------------------------------------------------------------------------ the walk change
@pytest.mark.parametrize("form", ["per_seq", "stop"])
def test_guided_walk_gathers_before_the_bonus(form):
    """One level: node 1 (token x) rejected, node 2 (token y) accepted alone, the bonus z from node 2's row."""
    V, M, S, P = 32000, 64, 3, 10
    x_id, y_id, z_id = 100, 200, 300
    tgt = torch.full((S, V), float("-inf"))
    tgt[0, y_id] = 0.0
    tgt[1, 7] = 0.0
    tgt[2, z_id] = 0.0
    drf = torch.full((S, V), float("-inf"))
    drf[0, x_id] = drf[0, y_id] = 5.0
    drf[1:, 7] = 0.0
    succ_off = torch.tensor([0, 2, 2, 2], dtype=torch.int32, device=DEV)
    succ = torch.tensor([1, 2], dtype=torch.int32, device=DEV)
    depth = torch.tensor([0, 1, 1], dtype=torch.int32, device=DEV)
    row_base = torch.tensor([0, 1, 2], dtype=torch.int32, device=DEV)
    row_step = torch.ones(3, dtype=torch.int32, device=DEV)
    results = {}
    for guided in (0, 1):
        tokens = torch.zeros(1, M, dtype=torch.long)
        tokens[0, P - 1:P + 2] = torch.tensor([42, x_id, y_id])
        state = torch.zeros(1, 16, dtype=torch.int32)
        state[0, ST_P], state[0, ST_M], state[0, ST_GUIDED] = P, M, guided
        t, s = tokens.to(DEV), state.to(DEV)
        pos = torch.arange(M, dtype=torch.long, device=DEV).unsqueeze(0)
        acc = torch.zeros(1, 8, dtype=torch.int32, device=DEV)
        r = torch.full((1, M), 0.5, dtype=F16, device=DEV)
        noise = torch.ones(1, V, dtype=F16, device=DEV)
        T = torch.ones(1, dtype=torch.float32, device=DEV)
        args = (tgt.to(F16).to(DEV), drf.to(F16).to(DEV), row_base, row_step, r, noise, succ_off, succ, depth, S, T)
        if form == "per_seq":
            ops().accept_stochastic_batch_per_seq(*args, t, pos, acc, s, M)
        else:
            ops().accept_stochastic_batch_stop(*args, None, torch.full((1, 8), -1, dtype=torch.int32, device=DEV),
                                               torch.zeros(1, dtype=torch.int32, device=DEV), t, pos, acc, s, M)
        torch.cuda.synchronize()
        results[guided] = (t.cpu()[0, P:P + 2].tolist(), int(s.cpu()[0, ST_ACCEPT_LEN]), int(acc.cpu()[0, 0]))
    assert results[1] == ([y_id, z_id], P + 1, P + 1), "guided: node 2's token, then the bonus"
    assert results[0] == ([z_id, z_id], P + 1, P + 1), "unguided: SpecTree's order, the bonus written first"


# ------------------------------------------------------------------------------------------------ BatchTree
POLICIES = {"spec": "spec", "greedy": "greedy", "mixed": ["spec", "greedy", "spec"]}


def _wide_guide(V, seed, n=5, width=1000):
    """States that allow `width` random ids each (one with a default instead), every id moving to a random state."""
    rnd = random.Random(seed)
    states = []
    for i in range(n):
        if i == 2:
            edges = {rnd.randrange(V): 0 for _ in range(50)}
            states.append(GuideState(edges=edges, default=3, banned=set(rnd.sample(range(V), 5000)) - edges.keys()))
        else:
            states.append(GuideState(edges={t: rnd.randrange(n) for t in rnd.sample(range(3, V), width)}))
    return TokenGuide(states)


def _gen(step, prompt):
    return step[0][len(prompt):].tolist()


@pytest.mark.parametrize("tree", ["config2", "tree16x8"])
@pytest.mark.parametrize("policy", list(POLICIES))
def test_output_follows_the_guide(policy, tree):
    gm, Mx = cases.load_growmap(GROWMAPS[tree]), 512
    S = gm["size"]
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(800 + i, n).to(DEV) for i, n in enumerate((40, 64, 50))]
    guides = [_wide_guide(cases.V, 1), _wide_guide(cases.V, 2), None]
    bt = _tree(engines, prompts, gm, Mx, policy=POLICIES[policy], seeds=[1, 2, 3], stop_tokens=[], temperature=1.0,
               guide=guides)
    steps = _decode(bt, 400)
    for b in range(2):
        gen = _gen(steps[-1][b], prompts[b])
        assert len(gen) >= min(100, Mx - S - len(prompts[b])), (policy, tree, b, len(gen))
        assert O.state_after(guides[b], gen, cases.V) >= 0, (policy, tree, b)
        assert bt.guide_state(b) == O.state_after(guides[b], gen, cases.V)
        assert bt.finish_reason[b] == "room"
    # a refill admission switches slot 1 to a choice trie and slot 2 to a guide
    trie = _trie([[11, 12, 13], [21, 22], [31]], 777)
    for b, gd in ((1, trie), (2, guides[0])):
        bt.freeze(b)
        bt.admit(b, cases.make_prompt(810 + b, 45).to(DEV), seed=20 + b, guide=gd, stop_tokens=[777])
    steps = _decode(bt, 200)
    gen1 = steps[-1][1][0][45:].tolist()
    assert bt.finish_reason[1] == "stop" and gen1 in ([11, 12, 13, 777], [21, 22, 777], [31, 777]), gen1
    gen2 = bt.last[2][0][45:].tolist()
    assert len(gen2) >= 50 and O.state_after(guides[0], gen2, cases.V) >= 0


def _trie(words, stop):
    nodes = [{}]
    for w in words:
        cur = 0
        for t in w:
            if t not in nodes[cur]:
                nodes.append({})
                nodes[cur][t] = len(nodes) - 1
            cur = nodes[cur][t]
    return TokenGuide([GuideState(edges=e if e else {stop: 0}) for e in nodes])


@pytest.mark.parametrize("policy", ["spec", "greedy"])
def test_chain_guide_forces_the_output(policy):
    gm, Mx = cases.load_growmap(GM128), 384
    prompts = [cases.make_prompt(820 + i, n).to(DEV) for i, n in enumerate((40, 64))]
    want = [5000 + 37 * i for i in range(30)]
    stop = 999
    chain = TokenGuide([GuideState(edges={t: i + 1}) for i, t in enumerate(want)] + [GuideState(edges={stop: 0})])
    bt = _tree(_engines(2, Mx), prompts, gm, Mx, policy=policy, seeds=[1, 2], stop_tokens=[stop], guide=chain)
    steps = _decode(bt, 100)
    assert bt.finish_reason == ["stop", "stop"]
    for b in range(2):
        assert _gen(steps[-1][b], prompts[b]) == want + [stop], b


def test_guide_finish_of_a_greedy_slot():
    """The start state allows only id 2, which min_tokens bans: the greedy slot commits 0 from an all -inf row, which the
    guide does not allow, and ends with finish_reason "guide" and no generated token."""
    gm, Mx = cases.load_growmap(GM128), 384
    prompts = [cases.make_prompt(830 + i, n).to(DEV) for i, n in enumerate((40, 64))]
    only2 = TokenGuide([GuideState(edges={2: 0})])
    bt = _tree(_engines(2, Mx), prompts, gm, Mx, policy="greedy", guide=[only2, None], min_tokens=[5, 0])
    steps = _decode(bt, 3)
    assert bt.finish_reason[0] == "guide" and bt.guide_state(0) == -1
    v, _, term = steps[0][0]
    assert term and torch.equal(v, prompts[0].cpu()), v[len(prompts[0]):]
    assert bt.finish_reason[1] is None and not bt.frozen[1]


def test_logprobs_with_a_guide():
    gm, Mx = cases.load_growmap(GM128), 384
    prompts = [cases.make_prompt(840 + i, n).to(DEV) for i, n in enumerate((50, 70))]
    small = TokenGuide([GuideState(edges={100: 1, 200: 0, 300: 1}), GuideState(edges={400: 0, 500: 0})])
    bt = _tree(_engines(2, Mx), prompts, gm, Mx, policy=["spec", "greedy"], seeds=[1, 2], logprobs=5, stop_tokens=[],
               guide=small)
    _decode(bt, 10)
    for b in range(2):
        lp, ids, top = bt.token_logprobs(b)
        assert lp.shape[0] >= 10 and bool(torch.isfinite(lp).all()), b
        fin = torch.isfinite(top)
        assert bool((fin.sum(1) <= 3).all()) and set(ids[fin].tolist()) <= {100, 200, 300, 400, 500}, b
        assert bool(torch.isneginf(top[:, 3:]).all()), "the disallowed top entries are -inf"


def test_first_token_follows_the_masked_row():
    """Seeded guided "spec" slots of the branching config-2 tree, one admission per seed on one prompt: the first
    generated token's frequencies against softmax(masked row 0 / T) (the root row, the same for every admission)."""
    from scipy.stats import chisquare
    gm, Mx, B, T = cases.load_growmap(GM128), 384, 4, 1.0
    S = gm["size"]
    prompt = cases.make_prompt(850, 40).to(DEV)
    engines = _engines(B, Mx)
    probe = _tree(engines, [prompt] * B, gm, Mx, seeds=list(range(B)), temperature=T, stop_tokens=[])
    probe.construct_grow_map()
    probe.verify()
    top = torch.topk(probe.target_logits[0].float(), 12).indices.tolist()
    allowed = top[::2] + [top[1]]                         # high-probability ids, so the draft proposes some of them
    gd = TokenGuide([GuideState(edges={t: 0 for t in allowed})])
    bt = _tree(engines, [prompt] * B, gm, Mx, seeds=list(range(B)), temperature=T, stop_tokens=[], guide=gd)
    counts = {t: 0 for t in allowed}
    row = None
    n_rounds = 1000
    for it in range(n_rounds):
        if it:
            for b in range(B):
                bt.freeze(b)
                bt.admit(b, prompt, seed=1000 + it * B + b)
        bt.construct_grow_map()
        out = bt.verify()
        if row is None:
            row = bt.target_logits[0].float().cpu()
        for b in range(B):
            counts[int(out[b][0][len(prompt)])] += 1
    p = torch.softmax(row.double() / T, 0)
    assert float(p.sum() - p[allowed].sum()) < 1e-12, "the row is masked to the allowed ids"
    obs = torch.tensor([counts[t] for t in allowed], dtype=torch.float64)
    exp = p[allowed] / p[allowed].sum() * obs.sum()
    keep = exp >= 5
    obs_k = torch.cat([obs[keep], obs[~keep].sum().view(1)]) if (~keep).any() else obs[keep]
    exp_k = torch.cat([exp[keep], exp[~keep].sum().view(1)]) if (~keep).any() else exp[keep]
    stat, pval = chisquare(obs_k.numpy(), exp_k.numpy())
    assert pval > 1e-3, (pval, obs.tolist(), exp.tolist())
    assert S == 128


def test_unguided_slots_graphs_and_captures():
    gm, Mx = cases.load_growmap(GM128), 384
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(860 + i, n).to(DEV) for i, n in enumerate((70, 100, 84))]
    kw = dict(seeds=[21, 22, 23], policy=["spec", "greedy", "spec"], stop_tokens=[])
    plain_bt = _tree(engines, prompts, gm, Mx, **kw)
    plain = _decode(plain_bt, 6)
    none_bt = _tree(engines, prompts, gm, Mx, guide=None, **kw)
    _same(_decode(none_bt, 6), plain, (0, 1, 2), "guide=None")
    assert not none_bt.use_guide and none_bt.guide_table_dev is None
    assert none_bt.graph_launches == plain_bt.graph_launches
    gd = _wide_guide(cases.V, 7)
    guided = _decode(_tree(engines, prompts, gm, Mx, guide=[gd, None, None], **kw), 6)
    _same(guided, plain, (1, 2), "unguided neighbours of a guided slot")
    eager_bt = _tree(engines, prompts, gm, Mx, guide=[gd, None, None], **kw)
    eager_bt.use_graphs = False
    _same(_decode(eager_bt, 6), guided, (0, 1, 2), "graphs == eager")
    # built without guides: the first guided admission recaptures steady and post once, later ones nothing
    bt = _tree(engines, prompts, gm, Mx, **kw)
    _decode(bt, 2)
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1} and not bt.use_guide
    launches = bt.graph_launches["steady"]

    def admission(b, seed, **akw):
        bt.freeze(b)
        bt.admit(b, cases.make_prompt(seed, 50 + seed % 7).to(DEV), seed=seed, **akw)
        _decode(bt, 2)
    admission(0, 870, guide=None)
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}, "no guide: nothing is captured"
    admission(1, 871, guide=gd)
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2} and bt.use_guide
    assert bt.graph_launches["steady"] == launches + 3, "three launches join the steady graph"
    big = TokenGuide([GuideState(default=i, banned=[5]) for i in range(300)])
    for seed, akw in ((872, dict(guide=big)), (873, dict(guide=None)), (874, {})):
        admission(seed % 3, seed, **akw)
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2}, "no recapture after the first guide"


def test_guide_llama3_vocab():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 3 of both policies: the output stays in its guide."""
    import gc
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gc.collect()
    torch.cuda.empty_cache()
    gm, Mx, V = cases.load_growmap(GM128), 384, 128256
    engines = (GraphInferenceEngine(Mx, "random-init:llama-3.2-1b:1", device=DEV, batch_size=3),
               GraphInferenceEngineTG(Mx, "random-init:llama-3.1-8b:2", device=DEV, batch_size=3))
    g = torch.Generator().manual_seed(29)
    prompts = [torch.randint(3, V, (n,), generator=g).to(DEV) for n in (90, 128, 100)]
    guides = [_wide_guide(V, 31), _wide_guide(V, 32), _wide_guide(V, 33)]
    bt = _tree(engines, prompts, gm, Mx, seeds=[31, 32, 33], policy=["spec", "greedy", "spec"], stop_tokens=[],
               temperature=1.0, guide=guides)
    steps = _decode(bt, 12)
    assert bt.V == V and bt.use_guide
    for b in range(3):
        gen = _gen(steps[-1][b], prompts[b])
        assert len(gen) >= 12 and O.state_after(guides[b], gen, V) >= 0, b
