"""Per-sequence bad words and min_tokens on the device (sq_ban_tokens_rows_batch, BatchTree(bad_words=...,
min_tokens=...)).

Kernel level: the processed rows against oracle/bad_words.py bit for bit, at V in {32000, 32776, 128256} and B in
{1, 3, 8}, on the config-2 tree, a chain and a 16x8 tree, with word prefixes planted in the committed tail, on tree paths
and across the two, words that would reach into the prompt, NaN and +inf at banned ids, and the min_tokens boundary
inside the tree; neutral and frozen sequences and the rows past B*S byte-identical.  The ban commutes with the logit bias
and the penalties bit for bit.
BatchTree level: +100 biases on t and u with the words [t, t] and [u, u] make the output alternate t, u; min_tokens holds
back a strongly biased stop id (stop mode) and the ids 0 and 2 (default mode) for exactly min_tokens tokens; words taken
from an unconstrained run's bigrams and trigrams never occur in the constrained output (three policies, refill
admissions, V = 128256); logprobs stay finite; a seeded slot does not depend on its neighbours' settings; graphs equal
eager; neutral settings launch and commit what a tree without them does; the graphs are captured once more at the first
non-neutral setting only; and a row left with no finite entry ends a sampled sequence by the NaN flag and makes a greedy
one commit id 0.  End-to-end properties of "spec" sequences use a chain growmap: on a branching tree the stochastic
walk's bonus_first quirk (SpecTree.py:222-224) can commit the bonus token at an accepted slot, a position whose row did
not draw it, so a word can appear there (DESIGN.md §3a)."""
import collections

import pytest
import torch

import cases
from oracle.bad_words import process_rows
from oracle.logit_bias import process_rows as bias_rows
from oracle.penalty import penalize_rows, row_context
from test_gpu_logit_bias import _device_rows as bias_device_rows
from test_gpu_mixed_policy import GM128
from test_gpu_refill import DEV, F16, _engines, ops

pytestmark = pytest.mark.gpu

ST_P, ST_FROZEN = 0, 9
NW, WL, NS = 128, 16, 8
GROWMAPS = {"config2": GM128, "chain": "L40_growmaps/16-chain.pt", "tree16x8": "L40_growmaps/16x8-tree.pt"}


def _bits16(x):
    return x.view(torch.int16)


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _device_rows(words, min_end, end_ids):
    B = len(words)
    table = torch.zeros(B, NW, WL, dtype=torch.int32)
    lens = torch.zeros(B, NW, dtype=torch.int32)
    for b, ws in enumerate(words):
        for i, w in enumerate(ws or ()):
            table[b, i, :len(w)] = torch.tensor(w, dtype=torch.int32)
            lens[b, i] = len(w)
    n = torch.tensor([len(ws or ()) for ws in words], dtype=torch.int32)
    ends = torch.tensor([list(e) + [-1] * (NS - len(e)) for e in end_ids], dtype=torch.int32)
    return [t.to(DEV) for t in (table, lens, n, torch.tensor(min_end, dtype=torch.int32), ends)]


def _ban(out, tokens, P, L, gm, st, words, min_end, end_ids, frozen=()):
    """sq_ban_tokens_rows_batch in place on the device tensor `out`."""
    B = len(words)
    state = torch.zeros(B, 16, dtype=torch.int32)
    state[:, ST_P] = torch.tensor(P)
    for b in frozen:
        state[b, ST_FROZEN] = 1
    ops().ban_tokens_rows_batch_(out, tokens.to(DEV), state.to(DEV), torch.tensor(L, dtype=torch.int32, device=DEV),
                                 st.depth, st.tree_bits, st.tree_words, gm["size"], *_device_rows(words, min_end, end_ids))
    return out


def _context(gm, setup):
    """Plant words: the generated context of a few rows (committed tail, path, both), cut to every length."""
    tokens, P, L, b, V, g = setup
    S = gm["size"]
    words = [(int(torch.randint(0, V, (1,), generator=g)),), (V - 1,)]            # one-token words
    depth = gm["depth"]
    deep = sorted(range(S), key=lambda k: -int(depth[k]))
    for k in [0, deep[0], deep[len(deep) // 3], deep[-1], S - 1]:
        _, ids = row_context(tokens[b], P[b], gm["mask"], k)
        gen = ids[L[b]:].tolist()
        for n in (2, 3, 5, 9, 16):
            if n - 1 <= len(gen):
                words.append(tuple(gen[len(gen) - (n - 1):]) + (int(torch.randint(0, V, (1,), generator=g)),))
        full = ids[max(0, L[b] - 2):].tolist()[-15:]         # reaches into the prompt when gen is short: no match
        words.append(tuple(full) + (7,))
    while len(words) < NW:                                   # small-alphabet words that match here and there
        n = int(torch.randint(2, 5, (1,), generator=g))
        words.append(tuple(torch.randint(3, 7, (n - 1,), generator=g).tolist()) + (int(torch.randint(0, V, (1,),
                                                                                                         generator=g)),))
    return list(dict.fromkeys(w for w in words if 1 <= len(w) <= WL))[:NW]


@pytest.mark.parametrize("V", [32000, 32776, 128256])
@pytest.mark.parametrize("tree", list(GROWMAPS))
def test_kernel_matches_oracle(V, tree):
    from sequoia_b200.tree import _Static
    gm = cases.load_growmap(GROWMAPS[tree])
    st = _Static(gm, DEV)
    S, M = gm["size"], 640
    for B in (1, 3, 8):
        g = torch.Generator().manual_seed(V + B + S)
        tokens = torch.randint(3, 7, (B, M), generator=g)                # a small alphabet: words match by chance too
        tokens[:, ::5] = torch.randint(0, V, (B, (M + 4) // 5), generator=g)
        P = [int(torch.randint(S + 20, M - S, (1,), generator=g)) for _ in range(B)]
        gens = [0, 3, 40, 1, 200, 7, 14, 2]                                 # committed generated tokens per sequence
        L = [max(1, P[b] - gens[b % 8]) for b in range(B)]
        words = [_context(gm, (tokens, P, L, b, V, g)) for b in range(B)]
        min_end = [P[b] + 2 if b % 3 == 0 else (P[b] + 100 if b % 3 == 1 else 0) for b in range(B)]
        end_ids = [(0, 2), (5, V - 1, 17), ()] * 3
        end_ids = end_ids[:B]
        neutral, frozen = ((), ()) if B == 1 else ((1,), (B - 1,))
        for b in neutral:
            words[b], min_end[b] = (), 0
        x = (torch.randn(B * S + 3, V, generator=g) * 3).to(F16)
        for b in range(B):                                   # non-finite entries at banned ids
            for i, w in enumerate(words[b][:6]):
                x[b * S:(b + 1) * S, w[-1]] = (float("nan"), float("inf"), float("-inf"))[i % 3]
        x[:, 0] = float("nan")
        got = _ban(x.clone().to(DEV), tokens, P, L, gm, st, words, min_end, end_ids, frozen).cpu()
        want = process_rows(x, tokens, P, L, gm["mask"], gm["depth"], words, min_end, end_ids,
                            frozen=[b in frozen for b in range(B)])
        assert torch.equal(_bits16(got), _bits16(want)), (V, tree, B, (_bits16(got) != _bits16(want)).nonzero()[:5])
        for b in set(neutral) | set(frozen):
            assert torch.equal(_bits16(got[b * S:(b + 1) * S]), _bits16(x[b * S:(b + 1) * S])), (b, "untouched")
        assert torch.equal(_bits16(got[B * S:]), _bits16(x[B * S:])), "sentinel rows untouched"
        changed = (_bits16(got[:S]) != _bits16(x[:S])).sum(1)
        assert int((changed > 0).sum()) > 0, "sequence 0 has bans"
        assert int((changed <= NW + NS).all()), "only banned ids change"


def test_kernel_all_neutral_launch_leaves_every_row():
    from sequoia_b200.tree import _Static
    gm = cases.load_growmap(GM128)
    st = _Static(gm, DEV)
    x = torch.randn(3 * 128, 32000).to(F16)
    tokens = torch.randint(0, 32000, (3, 384))
    got = _ban(x.clone().to(DEV), tokens, [200] * 3, [100] * 3, gm, st, [(), (), ()], [0] * 3, [(0, 2)] * 3).cpu()
    assert torch.equal(_bits16(got), _bits16(x))


def test_ban_commutes_with_logit_bias_and_penalties():
    from sequoia_b200.tree import _Static
    gm = cases.load_growmap("L40_growmaps/4x4-tree.pt")
    st = _Static(gm, DEV)
    S, V, B, M = gm["size"], 32000, 2, 384
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(B * S, V, generator=g) * 4).to(F16)
    tokens = torch.randint(3, 40, (B, M), generator=g)
    P, L = [M - S - 5, M - S - 40], [M - S - 60, M - S - 42]
    words = [_context(gm, (tokens, P, L, b, 40, g)) for b in range(B)]
    min_end, end_ids = [P[0] + 2, P[1] + 1], [(0, 2), (9, 11)]
    allowed, bias = [tuple(range(0, V, 2)), None], [tuple((t, 3.0) for t in range(0, 300, 4)),
                                                    tuple((t, -2.0) for t in range(1, 300, 3))]
    state = torch.zeros(B, 16, dtype=torch.int32)
    state[:, ST_P] = torch.tensor(P)
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=DEV)  # noqa: E731
    reps, freqs, press = [_f32(1.3), _f32(0.8)], [_f32(0.7), _f32(-0.3)], [_f32(0.5), _f32(1.5)]
    scratch = torch.zeros(ops().penalty_scratch_words(B, M), dtype=torch.int32, device=DEV)

    def run(order):
        out = x.clone().to(DEV)
        for op in order:
            if op == "bias":
                ops().logit_bias_rows_batch_(out, S, state.to(DEV), *bias_device_rows(V, allowed, bias))
            elif op == "ban":
                _ban(out, tokens, P, L, gm, st, words, min_end, end_ids)
            else:
                ops().penalize_rows_batch_(out, tokens.to(DEV), state.to(DEV),
                                           torch.tensor(L, dtype=torch.int32, device=DEV), st.tree_bits, st.tree_words,
                                           S, f32(reps), f32(freqs), f32(press), scratch)
        torch.cuda.synchronize()
        return out.cpu()
    ref = run(("bias", "ban", "pen"))
    for order in (("ban", "bias", "pen"), ("bias", "pen", "ban"), ("ban", "pen"), ("pen", "ban")):
        got = run(order)
        want = ref if "bias" in order else run(("ban", "pen"))
        assert torch.equal(_bits16(got), _bits16(want)), order
    oracle = process_rows(penalize_rows(bias_rows(x, S, allowed, bias), tokens, P, L, gm["mask"], reps, freqs, press),
                          tokens, P, L, gm["mask"], gm["depth"], words, min_end, end_ids)
    assert torch.equal(_bits16(ref), _bits16(oracle))
    assert int(torch.isinf(ref).sum()) > int(torch.isinf(run(("bias", "pen"))).sum()), "something is banned"


# ------------------------------------------------------------------------------------------------ BatchTree
def _tree(engines, prompts, gm, Mx, **kw):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    d.clear_kv()
    t.clear_kv()
    return BatchTree(d, t, prompts, gm, max_length=Mx, max_target_seq=Mx, **kw)


def _decode(bt, iters):
    steps = []
    for _ in range(iters):
        bt.construct_grow_map()
        steps.append([(v.cpu().clone(), a, term) for v, a, term in bt.verify()])
        if all(bt.frozen):
            break
    return steps


def _same(got, want, slots, what):
    assert len(got) == len(want), what
    for it in range(len(got)):
        for b in slots:
            (v, a, term), (v0, a0, term0) = got[it][b], want[it][b]
            assert (a, term) == (a0, term0) and torch.equal(v, v0), (what, it, b)


def _occurs(gen, words):
    """The words (tuples) that occur in the token list gen."""
    return [w for w in words if any(tuple(gen[i:i + len(w)]) == w for i in range(len(gen) - len(w) + 1))]


POLICIES = {"spec": "spec", "greedy": "greedy", "mixed": ["spec", "greedy", "spec"]}
CHAIN = "L40_growmaps/16-chain.pt"


def _growmap(policy):
    """A chain for any batch with a "spec" sequence (module docstring), the config-2 tree for an all-greedy one."""
    return cases.load_growmap(GM128 if policy == "greedy" else CHAIN)


@pytest.mark.parametrize("policy", list(POLICIES))
def test_bias_and_bad_words_alternate(policy):
    gm, Mx = _growmap(policy), 384
    prompts = [cases.make_prompt(700 + i, n).to(DEV) for i, n in enumerate((40, 64, 50))]
    t, u = 1234, 31999
    bt = _tree(_engines(3, Mx), prompts, gm, Mx, policy=POLICIES[policy], seeds=[1, 2, 3], stop_tokens=[],
               logit_bias={t: 100, u: 100}, bad_words=[[t, t], [u, u]])
    steps = _decode(bt, 300)
    for b in range(3):
        gen = steps[-1][b][0][len(prompts[b]):].tolist()
        assert len(gen) >= 100 and set(gen) == {t, u}, (policy, b, len(gen))
        assert all(gen[i] != gen[i + 1] for i in range(len(gen) - 1)), (policy, b)


@pytest.mark.parametrize("policy", ["spec", "greedy"])
def test_min_tokens_holds_back_the_stop_id(policy):
    gm, Mx = _growmap(policy), 384
    prompts = [cases.make_prompt(710 + i, n).to(DEV) for i, n in enumerate((40, 64, 50))]
    s, ms = 777, [1, 7, 40]
    bt = _tree(_engines(3, Mx), prompts, gm, Mx, policy=policy, seeds=[1, 2, 3], stop_tokens=[s], logit_bias={s: 100},
               min_tokens=ms)
    steps = _decode(bt, 100)
    assert bt.finish_reason == ["stop"] * 3
    for b in range(3):
        gen = steps[-1][b][0][len(prompts[b]):].tolist()
        assert len(gen) == ms[b] + 1 and gen[-1] == s and s not in gen[:-1], (policy, b, gen)


@pytest.mark.parametrize("policy", ["spec", "greedy"])
def test_min_tokens_holds_back_0_and_2_in_default_mode(policy):
    gm, Mx = _growmap(policy), 384
    prompts = [cases.make_prompt(720 + i, n).to(DEV) for i, n in enumerate((40, 64))]
    ms = [5, 30]
    bt = _tree(_engines(2, Mx), prompts, gm, Mx, policy=policy, seeds=[1, 2], logit_bias=[{0: 100}, {2: 100}],
               min_tokens=ms)
    assert not bt.use_stop
    steps = _decode(bt, 100)
    for b in range(2):
        gen = steps[-1][b][0][len(prompts[b]):].tolist()
        assert len(gen) > ms[b] and 0 not in gen[:ms[b]] and 2 not in gen[:ms[b]], (policy, b, gen[:ms[b] + 1])
        assert gen[ms[b]] == (0, 2)[b], (policy, b)


def _frequent_words(gens, n_bi=40, n_tri=20):
    bi, tri = collections.Counter(), collections.Counter()
    for gen in gens:
        bi.update(tuple(gen[i:i + 2]) for i in range(len(gen) - 1))
        tri.update(tuple(gen[i:i + 3]) for i in range(len(gen) - 2))
    return [w for w, _ in bi.most_common(n_bi)] + [w for w, _ in tri.most_common(n_tri)]


@pytest.mark.parametrize("policy", list(POLICIES))
def test_no_bad_word_in_any_output(policy):
    """Words from the unconstrained run's frequent bigrams and trigrams, so they would occur; a refill admission brings a
    new prompt with words of its own."""
    gm, Mx = _growmap(policy), 512
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(730 + i, n).to(DEV) for i, n in enumerate((40, 64, 50))]
    kw = dict(policy=POLICIES[policy], seeds=[4, 5, 6], stop_tokens=[], temperature=1.0)
    free = _decode(_tree(engines, prompts, gm, Mx, **kw), 40)
    gens = [free[-1][b][0][len(prompts[b]):].tolist() for b in range(3)]
    words = _frequent_words(gens)
    assert _occurs(sum(gens, []), words), "the words occur without the setting"
    bt = _tree(engines, prompts, gm, Mx, bad_words=words, **kw)
    steps = _decode(bt, 40)
    for b in range(3):
        gen = steps[-1][b][0][len(prompts[b]):].tolist()
        assert len(gen) >= 40 and not _occurs(gen, words), (policy, b, _occurs(gen, words)[:3])
    new_words = words[::2]
    bt.freeze(1)
    p_new = cases.make_prompt(739, 45).to(DEV)
    bt.admit(1, p_new, seed=9, bad_words=new_words)
    steps = _decode(bt, 40)
    gen = steps[-1][1][0][len(p_new):].tolist()
    assert len(gen) >= 40 and not _occurs(gen, new_words), policy
    assert bt.bad_words[1] == tuple(new_words) and bt.bad_words[0] == tuple(words)


def test_logprobs_stay_finite():
    gm, Mx = _growmap("mixed"), 384
    prompts = [cases.make_prompt(740 + i, n).to(DEV) for i, n in enumerate((50, 70))]
    bt = _tree(_engines(2, Mx), prompts, gm, Mx, policy=["spec", "greedy"], seeds=[1, 2], logprobs=5, stop_tokens=[],
               bad_words=[[t] for t in range(3, 60)] + [[5, 6], [7, 8, 9]], min_tokens=20)
    _decode(bt, 20)
    for b in range(2):
        lp, ids, _ = bt.token_logprobs(b)
        assert lp.shape[0] >= 20 and bool(torch.isfinite(lp).all()), b
        assert not set(ids[:, 0].tolist()) & set(range(3, 60)), "a banned id is never a top alternative's best"


def test_seeded_slot_ignores_neighbours_and_graphs_equal_eager():
    gm, Mx = cases.load_growmap(GM128), 384
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(750 + i, n).to(DEV) for i, n in enumerate((50, 70, 60))]
    mine = [[5, 6], [100], [7, 8, 9]]
    kw = dict(policy=["spec", "greedy", "spec"], seeds=[1, 2, 3], stop_tokens=[])
    a = _decode(_tree(engines, prompts, gm, Mx, bad_words=[mine, None, [[11]]], min_tokens=[3, 0, 9], **kw), 8)
    b = _decode(_tree(engines, prompts, gm, Mx, bad_words=[mine, [[1], [2, 3]], None], min_tokens=[3, 50, 0], **kw), 8)
    _same(a, b, (0,), "slot 0 with different neighbours")
    eager_bt = _tree(engines, prompts, gm, Mx, bad_words=[mine, None, [[11]]], min_tokens=[3, 0, 9], **kw)
    eager_bt.use_graphs = False
    _same(_decode(eager_bt, 8), a, (0, 1, 2), "graphs == eager")


def test_neutral_is_free_and_captures_once():
    gm, Mx = cases.load_growmap(GM128), 384
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(760 + i, n).to(DEV) for i, n in enumerate((70, 100, 84))]
    seeds = [21, 22, 23]
    plain_bt = _tree(engines, prompts, gm, Mx, seeds=seeds)
    plain = _decode(plain_bt, 6)
    neutral_bt = _tree(engines, prompts, gm, Mx, seeds=seeds, bad_words=[None, [], []], min_tokens=0)
    neutral = _decode(neutral_bt, 6)
    assert not neutral_bt.use_ban and neutral_bt.words_dev is None
    assert neutral_bt.graph_launches == plain_bt.graph_launches
    _same(neutral, plain, (0, 1, 2), "all-neutral tree")
    # built neutral; the first non-neutral admission recaptures steady and post once, later ones nothing
    bt = _tree(engines, prompts, gm, Mx, seeds=seeds, policy=["spec", "greedy", "spec"])

    def admission(b, seed, **kw):
        bt.freeze(b)
        bt.admit(b, cases.make_prompt(seed, 50 + seed % 7).to(DEV), seed=seed, **kw)
        _decode(bt, 2)
    _decode(bt, 2)
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1} and not bt.use_ban
    launches = bt.graph_launches["steady"]
    admission(0, 780, bad_words=[], min_tokens=0)
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}, "a neutral admission captures nothing"
    admission(1, 781, bad_words=[[5, 6]])
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2} and bt.use_ban
    assert bt.graph_launches["steady"] == launches + 1, "the kernel is one more launch"
    for seed, kw in ((782, dict(min_tokens=4)), (783, dict(bad_words=None)), (784, {})):
        admission(seed % 3, seed, **kw)
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2}, "no recapture after the kernel entered"


def test_a_row_with_no_finite_entry():
    """Allowed {a, c}, words [a, a] and [a, c], a strongly biased: after an a, the row has no finite entry.  The sampled
    sequence ends by the NaN flag; the greedy one commits id 0 there (the argmax of an all -inf row) and goes on."""
    gm, Mx = _growmap("mixed"), 384
    prompts = [cases.make_prompt(790 + i, n).to(DEV) for i, n in enumerate((40, 64))]
    a, c = 500, 600
    bt = _tree(_engines(2, Mx), prompts, gm, Mx, policy=["spec", "greedy"], seeds=[1, 2], stop_tokens=[],
               allowed_token_ids=(a, c), logit_bias={a: 100}, bad_words=[[a, a], [a, c]])
    steps = _decode(bt, 30)
    gen0 = steps[-1][0][0][len(prompts[0]):].tolist()
    assert bt.finish_reason[0] == "nan" and gen0 and set(gen0) == {a}, gen0
    gen1 = steps[-1][1][0][len(prompts[1]):].tolist()
    assert len(gen1) >= 20 and gen1[0::2] == [a] * len(gen1[0::2]) and gen1[1::2] == [0] * len(gen1[1::2]), gen1[:8]


def test_bad_words_batch_llama3_vocab():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 3 of the three policies: words from the unconstrained run's
    bigrams never occur in the constrained one."""
    import gc
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gc.collect()
    torch.cuda.empty_cache()
    gm, Mx = _growmap("mixed"), 384
    engines = (GraphInferenceEngine(Mx, "random-init:llama-3.2-1b:1", device=DEV, batch_size=3),
               GraphInferenceEngineTG(Mx, "random-init:llama-3.1-8b:2", device=DEV, batch_size=3))
    g = torch.Generator().manual_seed(29)
    prompts = [torch.randint(3, 128256, (n,), generator=g).to(DEV) for n in (90, 128, 100)]
    kw = dict(seeds=[31, 32, 33], policy=["spec", "greedy", "spec"], stop_tokens=[], temperature=1.0)
    free = _decode(_tree(engines, prompts, gm, Mx, **kw), 12)
    gens = [free[-1][b][0][len(prompts[b]):].tolist() for b in range(3)]
    words = _frequent_words(gens, 60, 0)
    assert _occurs(sum(gens, []), words)
    bt = _tree(engines, prompts, gm, Mx, bad_words=words + [[128255]], **kw)
    steps = _decode(bt, 12)
    assert bt.V == 128256 and bt.use_ban
    for b in range(3):
        gen = steps[-1][b][0][len(prompts[b]):].tolist()
        assert len(gen) >= 12 and not _occurs(gen, [tuple(w) for w in words] + [(128255,)]), b
