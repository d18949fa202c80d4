"""Constrained drafting on the device (sq_draft_rows_batch, SQ_ACCEPT_SKIP_DEAD, BatchTree(constrain_draft=True)).

Row kernel: the root and every level of the config-2, 16-chain and 16x8 trees, at V in {32000, 32776, 128256} and B in
{1, 3, 8}, against oracle/constrained_draft.py bit for bit, with allowed sets, biases, bad words, min_tokens and guides
(paths that leave the guide, NaN and +inf at disallowed ids); neutral and frozen slots, the rows of other levels and the
rows past B*S byte-identical; the node states the kernel leaves for the next level.
Walk: hand-built one-level trees where the dead-child instance commits the oracle's token (both live children rejected,
an all -inf draft row, a dead child first), and the existing instance ends the same input by the NaN flag.
BatchTree: every guided slot's output stays in its guide, every token in its allowed set, no bad word occurs; a refill
admission switches a slot to a 3-choice trie, which ends in a choice with "stop"; greedy slots and neutral slots commit
what they commit without constrain_draft; the first generated token of seeded guided "spec" slots follows softmax(masked
row / T) with guides of 7 and 3 ids (chi-square over 4000 seeds each); graphs equal eager; one draft recapture; an
all-neutral constrained tree equals an unconstrained one in outputs and graph_launches; V = 128256."""
import random

import pytest
import torch

import cases
from oracle import constrained_draft as CD
from oracle import guide as O
from sequoia_b200.guide import GuideState, TokenGuide
from test_gpu_bad_words import _context, _decode, _device_rows as ban_device_rows, _occurs, _same, _tree
from test_gpu_guide import ALPHA, GROWMAPS, _random_guide, _table, _trie, _wide_guide
from test_gpu_logit_bias import _device_rows as bias_device_rows
from test_gpu_mixed_policy import GM128
from test_gpu_refill import DEV, F16, _engines, ops

pytestmark = pytest.mark.gpu

ST_P, ST_TERMINAL, ST_NAN, ST_M, ST_FROZEN = 0, 2, 6, 8, 9
ST_GUIDED, ST_GUIDE_STATE = 12, 13


def _bits16(x):
    return x.view(torch.int16)


# ------------------------------------------------------------------------------------------------ the row kernel
@pytest.mark.parametrize("V", [32000, 32776, 128256])
@pytest.mark.parametrize("tree", list(GROWMAPS))
def test_row_kernel_matches_oracle(V, tree):
    from sequoia_b200.tree import _Static
    gm = cases.load_growmap(GROWMAPS[tree])
    st = _Static(gm, DEV)
    S, M = gm["size"], 640
    levels = [(0, 1)] + [(lv["n0"], lv["tb"]) for lv in st.levels]
    leaves = stays = False
    for B in (1, 3, 8):
        g = torch.Generator().manual_seed(V + 7 * B + S)
        base, step = ops().draft_row_tables(levels, S, B, DEV)
        tokens = torch.tensor(ALPHA)[torch.randint(0, len(ALPHA), (B, M), generator=g)]
        tokens[:, ::13] = torch.randint(0, V, (B, (M + 12) // 13), generator=g)   # ids most states do not allow
        P = [int(torch.randint(S + 40, M - S, (1,), generator=g)) for _ in range(B)]
        L = [P[b] - 5 - 3 * b for b in range(B)]
        neutral, frozen = ((), ()) if B == 1 else ((1,), (B - 1,))
        guides = [None if b in neutral or b % 3 == 2 else _random_guide(V, V + 31 * B + b) for b in range(B)]
        allowed = [None if b in neutral or b % 2 else tuple(sorted(set(ALPHA[:6]) | set(range(0, V, 3)))) for b in range(B)]
        bias = [None if b in neutral else tuple((t, 2.5 - b) for t in range(1, 400, 7)) for b in range(B)]
        words = [None if b in neutral else _context(gm, (tokens, P, L, b, V, g)) for b in range(B)]
        min_end = [0 if b in neutral else P[b] + 1 + b % 3 for b in range(B)]
        end_ids = [(0, 2, 9) if b % 2 else (4, 6) for b in range(B)]
        roots = []
        for b in range(B):
            r = -1 if guides[b] is None else O.state_after(guides[b], tokens[b, L[b]:P[b]].tolist(), V)
            roots.append(guides[b].start if guides[b] is not None and r < 0 else max(r, 0))
        state = torch.zeros(B, 16, dtype=torch.int32)
        state[:, ST_P] = torch.tensor(P)
        state[:, ST_M] = M
        for b in range(B):
            if guides[b] is not None:
                state[b, ST_GUIDED], state[b, ST_GUIDE_STATE] = 1, roots[b]
        for b in frozen:
            state[b, ST_FROZEN] = 1
        table, _blobs = _table(guides, V)
        x = (torch.randn(B * S + 3, V, generator=g) * 3).to(F16)
        x[:, 3] = float("nan")                          # disallowed in most states and outside the allowed sets
        x[:, 4] = float("inf")
        x[:, V - 2] = float("nan")
        sd, td = state.to(DEV), tokens.to(DEV)
        node = torch.full((B, S), -7, dtype=torch.int32, device=DEV)
        kinds = dict(bias=bias_device_rows(V, allowed, bias),
                     ban=[torch.tensor(L, dtype=torch.int32, device=DEV), st.depth] + ban_device_rows(words, min_end,
                                                                                                     end_ids),
                     guide=(table, node), tokens=td, tree_bits=st.tree_bits, tree_words=st.tree_words)
        got = x.clone().to(DEV)
        ops().draft_rows_batch_(got, base, step, 0, 1, S, sd, **kinds)
        root_only = got.cpu()
        rows_of = lambda ks: {int(base[k]) + b * int(step[k]) for k in ks for b in range(B)}   # noqa: E731
        for rw in set(range(B * S + 3)) - rows_of([0]):
            assert torch.equal(_bits16(root_only[rw]), _bits16(x[rw])), ("rows outside the root", rw)
        for n0, tb in levels[1:]:
            ops().draft_rows_batch_(got, base, step, n0, tb, S, sd, **kinds)
        got = got.cpu()
        want = CD.process_draft_rows(x, base.tolist(), step.tolist(), range(S), S, allowed=allowed, bias=bias,
                                     tokens=tokens, P=P, prompt_len=L, mask01=gm["mask"], depth=gm["depth"], words=words,
                                     min_end=min_end, end_ids=end_ids, guides=guides, roots=roots,
                                     frozen=[b in frozen for b in range(B)])
        bad = (_bits16(got) != _bits16(want)).nonzero()[:5]
        assert torch.equal(_bits16(got), _bits16(want)), (V, tree, B, bad)
        for b in set(neutral) | set(frozen):
            for k in range(S):
                rw = int(base[k]) + b * int(step[k])
                assert torch.equal(_bits16(got[rw]), _bits16(x[rw])), (b, k, "untouched")
        assert torch.equal(_bits16(got[B * S:]), _bits16(x[B * S:])), "rows past B*S untouched"
        ns = node.cpu()
        for b in range(B):
            if guides[b] is None or b in frozen:
                assert bool((ns[b] == -7).all()), b
                continue
            want_states = O.node_states(guides[b], roots[b], tokens[b], P[b], gm["mask"], V)
            assert ns[b].tolist() == want_states, b
            leaves |= min(want_states) < 0
            stays |= max(want_states[1:] or [-1]) >= 0
    assert leaves and stays, "paths that leave their guide and paths that stay in it"


# ------------------------------------------------------------------------------------------------ the walk
def _one_level_walk(V, form, policy, tgt, drf, kids, r_val):
    """Root 0 with children 1..4 (tokens kids), leaves' rows all 0 at id 7.  -> (tokens[P:P+2], state row).  The sequence
    is marked guided so that the walk gathers the accepted slots before it writes the bonus (no guide kernel runs): an
    accepted node 2 at slot a would otherwise be overwritten by the bonus, SpecTree's order."""
    S, P, M = 5, 10, 64
    succ_off = torch.tensor([0, 4, 4, 4, 4, 4], dtype=torch.int32, device=DEV)
    succ = torch.tensor([1, 2, 3, 4], dtype=torch.int32, device=DEV)
    depth = torch.tensor([0, 1, 1, 1, 1], dtype=torch.int32, device=DEV)
    row_base = torch.arange(S, dtype=torch.int32, device=DEV)
    row_step = torch.ones(S, dtype=torch.int32, device=DEV)
    tokens = torch.zeros(1, M, dtype=torch.long)
    tokens[0, P - 1:P + 4] = torch.tensor([42] + kids)
    state = torch.zeros(1, 16, dtype=torch.int32)
    state[0, ST_P], state[0, ST_M], state[0, ST_GUIDED] = P, M, 1
    t, s = tokens.to(DEV), state.to(DEV)
    pos = torch.arange(M, dtype=torch.long, device=DEV).unsqueeze(0)
    acc = torch.zeros(1, 8, dtype=torch.int32, device=DEV)
    r = torch.full((1, M), r_val, dtype=F16, device=DEV)
    noise = torch.ones(1, V, dtype=F16, device=DEV)
    T = torch.ones(1, dtype=torch.float32, device=DEV)
    args = (tgt.to(DEV), drf.to(DEV), row_base, row_step, r, noise, succ_off, succ, depth, S, T)
    if form == "per_seq":
        ops().accept_stochastic_batch_per_seq(*args, t, pos, acc, s, M, policy)
    elif form == "mixed":
        ops().accept_stochastic_batch_mixed(*args, torch.zeros(1, dtype=torch.int32, device=DEV), t, pos, acc, s, M,
                                            policy)
    else:
        ops().accept_stochastic_batch_stop(*args, None, torch.full((1, 8), -1, dtype=torch.int32, device=DEV),
                                           torch.zeros(1, dtype=torch.int32, device=DEV), t, pos, acc, s, M, policy)
    torch.cuda.synchronize()
    return t.cpu()[0, P:P + 2].tolist(), s.cpu()[0]


@pytest.mark.parametrize("V", [32000, 128256])
@pytest.mark.parametrize("form", ["per_seq", "mixed", "stop"])
def test_walk_skips_dead_children(V, form):
    S, P = 5, 10
    x_id, y_id, z_id, d1, d2, d3 = 100, 200, V - 8, 300, 301, 302
    tgt = torch.full((S, V), float("-inf"))
    tgt[0, x_id], tgt[0, y_id], tgt[0, z_id] = -4.0, -4.0, 2.0        # most mass outside the draft's support
    tgt[1:, 7] = 0.0
    r1 = torch.ones(1, 4)
    noise = torch.ones(1, V)
    cases_ = {
        "two_live_both_rejected": ([x_id, y_id, d1, d2], {x_id: 3.0, y_id: 2.0}, 1.0),
        "all_dead": ([d1, d2, d3, x_id], {}, 1.0),
        "dead_first": ([d1, x_id, y_id, d2], {x_id: 3.0, y_id: 2.0}, 0.0),
    }
    for name, (kids, live, r_val) in cases_.items():
        drf = torch.full((S, V), float("-inf"))
        for t_, v in live.items():
            drf[0, t_] = v
        drf[1:, 7] = 0.0
        want, accepted = CD.walk_first_token(tgt[0].to(F16), drf[0].to(F16), torch.tensor([kids]),
                                             r1 * r_val, noise, 1.0)
        got, st = _one_level_walk(V, form, ops().ACCEPT_SKIP_DEAD, tgt.to(F16), drf.to(F16), kids, r_val)
        assert int(st[ST_NAN]) == 0 and int(st[ST_TERMINAL]) == 0, (name, st.tolist())
        assert got[0] == int(want[0]), (name, got, int(want[0]))
        if bool(accepted[0]):
            assert got == [int(want[0]), 7], (name, "the accepted child, then the bonus from its row")
        if name != "dead_first":
            # the existing instance on the same input: q runs out of support and the residual turns NaN
            _, st0 = _one_level_walk(V, form, 0, tgt.to(F16), drf.to(F16), kids, r_val)
            assert int(st0[ST_NAN]) == 1 and int(st0[ST_TERMINAL]) == 1, (name, st0.tolist())


# ------------------------------------------------------------------------------------------------ BatchTree
POLICIES = {"spec": "spec", "greedy": "greedy", "mixed": ["spec", "greedy", "spec"]}


@pytest.mark.parametrize("policy", list(POLICIES))
def test_constrained_output(policy):
    gm, Mx = cases.load_growmap(GM128), 512
    S = gm["size"]
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(900 + i, n).to(DEV) for i, n in enumerate((40, 64, 50))]
    guides = [_wide_guide(cases.V, 41), _wide_guide(cases.V, 42), None]
    allowed = [None, None, tuple(random.Random(5).sample(range(3, cases.V), 1000))]
    kw = dict(policy=POLICIES[policy], seeds=[1, 2, 3], stop_tokens=[], temperature=1.0, guide=guides,
              allowed_token_ids=allowed)
    bt = _tree(engines, prompts, gm, Mx, constrain_draft=True, **kw)
    steps = _decode(bt, 400)
    for b in range(2):
        gen = steps[-1][b][0][len(prompts[b]):].tolist()
        assert len(gen) >= min(100, Mx - S - len(prompts[b])), (policy, b, len(gen))
        assert O.state_after(guides[b], gen, cases.V) >= 0, (policy, b)
        assert bt.finish_reason[b] == "room"
    gen2 = steps[-1][2][0][len(prompts[2]):].tolist()
    assert set(gen2) <= set(allowed[2]) and bt.finish_reason[2] == "room"
    # greedy slots commit the argmax of their processed target rows whatever the draft proposes
    plain = _decode(_tree(engines, prompts, gm, Mx, **kw), 400)
    for b in [b for b, p in enumerate(bt.policies) if p == "greedy"]:
        assert torch.equal(steps[-1][b][0], plain[-1][b][0]), ("greedy slots do not depend on the draft", b)
    # a refill admission switches slot 1 to a choice trie of fewer ids than the root's 19 children
    trie = _trie([[11, 12, 13], [21, 22], [31]], 777)
    bt.freeze(1)
    bt.admit(1, cases.make_prompt(910, 45).to(DEV), seed=21, guide=trie, stop_tokens=[777], policy="spec")
    _decode(bt, 200)
    gen1 = bt.last[1][0][45:].tolist()
    assert bt.finish_reason[1] == "stop" and gen1 in ([11, 12, 13, 777], [21, 22, 777], [31, 777]), gen1


def test_no_bad_word_on_a_chain():
    gm, Mx = cases.load_growmap("L40_growmaps/16-chain.pt"), 384
    engines = _engines(2, Mx)
    prompts = [cases.make_prompt(920 + i, n).to(DEV) for i, n in enumerate((40, 64))]
    probe = _decode(_tree(engines, prompts, gm, Mx, seeds=[1, 2], stop_tokens=[]), 12)
    words = set()
    for b in range(2):
        gen = probe[-1][b][0][len(prompts[b]):].tolist()
        words |= {(gen[i],) for i in range(0, 12, 3)} | {tuple(gen[i:i + 2]) for i in range(1, 20, 4)}
    words = sorted(w for w in words if len(w) >= 1)
    bt = _tree(engines, prompts, gm, Mx, seeds=[1, 2], stop_tokens=[], bad_words=words, min_tokens=[20, 0],
               constrain_draft=True)
    steps = _decode(bt, 60)
    for b in range(2):
        gen = steps[-1][b][0][len(prompts[b]):].tolist()
        assert len(gen) >= 40 and not _occurs(gen, words), (b, _occurs(gen, words))


@pytest.mark.parametrize("n_allowed", [7, 3])
def test_first_token_follows_the_masked_row(n_allowed):
    from scipy.stats import chisquare
    gm, Mx, B, T = cases.load_growmap(GM128), 384, 4, 1.0
    S = gm["size"]
    prompt = cases.make_prompt(950, 40).to(DEV)
    engines = _engines(B, Mx)
    probe = _tree(engines, [prompt] * B, gm, Mx, seeds=list(range(B)), temperature=T, stop_tokens=[])
    probe.construct_grow_map()
    probe.verify()
    top = torch.topk(probe.target_logits[0].float(), 12).indices.tolist()
    allowed = (top[::2] + [top[1]])[:n_allowed]
    gd = TokenGuide([GuideState(edges={t: 0 for t in allowed})])
    bt = _tree(engines, [prompt] * B, gm, Mx, seeds=list(range(B)), temperature=T, stop_tokens=[], guide=gd,
               constrain_draft=True)
    counts = {t: 0 for t in allowed}
    row = None
    for it in range(1000):
        if it:
            for b in range(B):
                bt.freeze(b)
                bt.admit(b, prompt, seed=5000 + it * B + b)
        bt.construct_grow_map()
        out = bt.verify()
        if row is None:
            row = bt.target_logits[0].float().cpu()
        for b in range(B):
            assert bt.finish_reason[b] != "nan"
            counts[int(out[b][0][len(prompt)])] += 1
    p = torch.softmax(row.double() / T, 0)
    assert float(p.sum() - p[allowed].sum()) < 1e-12, "the row is masked to the allowed ids"
    obs = torch.tensor([counts[t] for t in allowed], dtype=torch.float64)
    exp = p[allowed] / p[allowed].sum() * obs.sum()
    keep = exp >= 5
    obs_k = torch.cat([obs[keep], obs[~keep].sum().view(1)]) if (~keep).any() else obs[keep]
    exp_k = torch.cat([exp[keep], exp[~keep].sum().view(1)]) if (~keep).any() else exp[keep]
    _, pval = chisquare(obs_k.numpy(), exp_k.numpy())
    assert pval > 1e-3, (pval, obs.tolist(), exp.tolist())
    assert S == 128 and int(gm["branches"][0][0]) == 19 > n_allowed


def test_neutral_slots_graphs_and_captures():
    gm, Mx = cases.load_growmap(GM128), 384
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(960 + i, n).to(DEV) for i, n in enumerate((70, 100, 84))]
    kw = dict(seeds=[21, 22, 23], policy=["spec", "greedy", "spec"], stop_tokens=[])
    plain_bt = _tree(engines, prompts, gm, Mx, **kw)
    plain = _decode(plain_bt, 6)
    neutral_bt = _tree(engines, prompts, gm, Mx, constrain_draft=True, **kw)
    _same(_decode(neutral_bt, 6), plain, (0, 1, 2), "all-neutral constrained tree")
    assert neutral_bt.graph_launches == plain_bt.graph_launches and neutral_bt.allowed_dev is None
    gd = _wide_guide(cases.V, 47)
    ckw = dict(guide=[gd, None, None], allowed_token_ids=[None, None, None], constrain_draft=True, **kw)
    guided = _decode(_tree(engines, prompts, gm, Mx, **ckw), 6)
    _same(guided, plain, (1, 2), "neutral neighbours of a constrained slot")
    eager_bt = _tree(engines, prompts, gm, Mx, **ckw)
    eager_bt.use_graphs = False
    _same(_decode(eager_bt, 6), guided, (0, 1, 2), "graphs == eager")
    # built neutral: the first guided admission recaptures draft, steady and post once, later ones nothing
    bt = _tree(engines, prompts, gm, Mx, constrain_draft=True, **kw)
    _decode(bt, 2)
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}
    draft_launches = bt.graph_launches["draft"]

    def admission(b, seed, **akw):
        bt.freeze(b)
        bt.admit(b, cases.make_prompt(seed, 50 + seed % 7).to(DEV), seed=seed, **akw)
        _decode(bt, 2)
    admission(1, 971, guide=gd)
    assert bt.captures == {"draft": 2, "post": 2, "steady": 2}
    levels = sum(1 for i in range(len(bt.st.levels)) if i + 1 < len(bt.st.levels))
    assert bt.graph_launches["draft"] == draft_launches + 1 + levels, "one launch for the root and per parent level"
    for seed, akw in ((972, dict(guide=_trie([[5, 6]], 9))), (973, dict(guide=None)), (974, {})):
        admission(seed % 3, seed, **akw)
    assert bt.captures == {"draft": 2, "post": 2, "steady": 2}, "no recapture after the first guide"
    admission(0, 975, allowed_token_ids=list(range(100, 1100)), guide=None)
    assert bt.captures == {"draft": 3, "post": 3, "steady": 3}, "the allowed sets start: one recapture more"
    assert bt.graph_launches["draft"] == draft_launches + 1 + levels, "still one launch per processed level"


def test_constrained_draft_llama3_vocab():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 3 of both policies: the output stays in its guide."""
    import gc
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gc.collect()
    torch.cuda.empty_cache()
    gm, Mx, V = cases.load_growmap(GM128), 384, 128256
    engines = (GraphInferenceEngine(Mx, "random-init:llama-3.2-1b:1", device=DEV, batch_size=3),
               GraphInferenceEngineTG(Mx, "random-init:llama-3.1-8b:2", device=DEV, batch_size=3))
    g = torch.Generator().manual_seed(39)
    prompts = [torch.randint(3, V, (n,), generator=g).to(DEV) for n in (90, 128, 100)]
    guides = [_wide_guide(V, 51), _trie([[700, 800, 900]] * 1 + [[1000 + i] for i in range(2)], 5), _wide_guide(V, 53)]
    bt = _tree(engines, prompts, gm, Mx, seeds=[31, 32, 33], policy=["spec", "greedy", "spec"], stop_tokens=[[], [5], []],
               temperature=1.0, guide=guides, constrain_draft=True)
    steps = _decode(bt, 12)
    assert bt.V == V and bt._draft_processed()
    for b in (0, 2):
        gen = steps[-1][b][0][len(prompts[b]):].tolist()
        assert len(gen) >= 12 and O.state_after(guides[b], gen, V) >= 0, b
    assert bt.finish_reason[1] == "stop" and "nan" not in bt.finish_reason
