"""Per-sequence logit bias and allowed-token sets on the device (sq_logit_bias_rows_batch, BatchTree(logit_bias=...,
allowed_token_ids=...)).

Kernel level: the processed rows against oracle/logit_bias.py bit for bit, at V from 32000 to 131072, B in {1, 3, 8}, on
the config-2 tree, a chain and a one-level wide tree, with masks of 1, 5, V/2 and V-1 ids, biases of +-100, tiny ones and
ones on masked ids, and rows holding -inf, +inf and NaN; neutral and frozen sequences and rows past B*S untouched; rows
that are not 16-byte aligned.  Then bias, penalty, top-k and top-p in that order against the oracles' composition.
BatchTree level: greedy decoding commits the argmax of the oracle-processed row of each context, eagerly and with graphs;
every generated token lies in the allowed set; a bias of +100 on one id makes every generated token that id; neutral
settings launch and commit what a tree without them does; the graphs are captured once more at the first non-neutral
setting only; the top logprob ids lie in the allowed set; a stop id outside the set never ends a sequence; and one run
at V = 128256."""
import pytest
import torch

import cases
from oracle import sequoia_oracle as O
from oracle.logit_bias import allowed_vector, process_row, process_rows
from oracle.penalty import penalize_rows
from oracle.top_k import top_k_filter
from test_gpu_mixed_policy import GM128
from test_gpu_refill import DEV, F16, _engines, ops

pytestmark = pytest.mark.gpu

ST_P, ST_N_NEW, ST_FROZEN = 0, 3, 9
MAXB = 1024
GROWMAPS = {"config2": GM128, "chain": "L40_growmaps/16-chain.pt", "wide": "L40_growmaps/128x1-tree.pt"}


def _bits16(x):
    return x.view(torch.int16)


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _device_rows(V, allowed, bias):
    """The (B, ...) device arrays BatchTree keeps, from per-sequence allowed sets and (id, bias) tuples."""
    B = len(allowed)
    words = ops().mask_words(V)
    mask = torch.zeros(B, words, dtype=torch.int32)
    ids = torch.zeros(B, MAXB, dtype=torch.int32)
    vals = torch.zeros(B, MAXB, dtype=torch.float32)
    n = torch.zeros(B, dtype=torch.int32)
    for b in range(B):
        if allowed[b] is not None:
            mask[b] = ops().pack_token_mask(allowed[b], V)
        if bias[b]:
            n[b] = len(bias[b])
            ids[b, :n[b]] = torch.tensor([t for t, _ in bias[b]], dtype=torch.int32)
            vals[b, :n[b]] = torch.tensor([v for _, v in bias[b]], dtype=torch.float32)
    has = torch.tensor([a is not None for a in allowed], dtype=torch.int32)
    return [t.to(DEV) for t in (mask, has, ids, vals, n)]


def _launch(x, S, allowed, bias, frozen=(), logits=None):
    B = len(allowed)
    V = x.shape[1]
    state = torch.zeros(B, 16, dtype=torch.int32)
    for b in frozen:
        state[b, ST_FROZEN] = 1
    out = x.clone().to(DEV) if logits is None else logits
    ops().logit_bias_rows_batch_(out, S, state.to(DEV), *_device_rows(V, allowed, bias))
    torch.cuda.synchronize()
    return out.cpu()


def _rows(n, V, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, V, generator=g) * 4).to(F16)
    x[::5, 17] = float("-inf")
    x[1::7, 3] = float("inf")
    x[2::11, 5] = float("nan")
    x[::3, V - 1] = float("nan")
    x[:, 0] = 65500.0
    x[1::2, 8] = -65500.0
    return x, g


def _settings(V, B, g):
    """Per-sequence allowed sets (1, 5, V/2 and V-1 ids, none) and bias entries (+-100 at both ends of the vocabulary,
    tiny values, the full 1024 entries, entries on masked ids and on non-finite logits), cycled over the sequences."""
    perm = torch.randperm(V, generator=g).tolist()
    masks = [(17,), tuple(sorted(perm[:4] + [0])), tuple(sorted(perm[:V // 2] + [3, 5, 8, 17, V - 1])),
             tuple(sorted(set(range(V)) - {perm[0]})), None]
    masks = [m if m is None else tuple(sorted(set(m))) for m in masks]
    wide = sorted(set(torch.randint(0, V, (MAXB,), generator=g).tolist()))
    biases = [((0, 100.0), (3, -100.0), (5, 1.0), (17, 2.5), (V - 1, -100.0)),
              tuple((t, _f32(1e-3 * (i % 7 - 3))) for i, t in enumerate(wide) if i % 7 != 3),
              ((8, 100.0), (17, _f32(1e-30)), (perm[0], 50.0), (perm[1], -50.0)),
              tuple((t, float((-1) ** i * 100)) for i, t in enumerate(wide)),
              ((0, -100.0), (1, _f32(0.1)), (V - 1, 100.0), (V // 2, _f32(-7.3)))]
    return [masks[b % 5] for b in range(B)], [biases[(b * 2 + 1) % 5] for b in range(B)]


@pytest.mark.parametrize("V", [32000, 49152, 128256, 131072])
@pytest.mark.parametrize("tree", list(GROWMAPS))
def test_kernel_matches_oracle(V, tree):
    S = cases.load_growmap(GROWMAPS[tree])["size"]
    for B in (1, 3, 8):
        x, g = _rows(B * S + 3, V, V + B + S)
        allowed, bias = _settings(V, B, g)
        neutral, frozen = ((), ()) if B == 1 else ((1,), (B - 1,))
        for b in neutral:
            allowed[b], bias[b] = None, ()
        got = _launch(x, S, allowed, bias, frozen)
        want = process_rows(x, S, allowed, bias, frozen=[b in frozen for b in range(B)])
        assert torch.equal(_bits16(got), _bits16(want)), (V, tree, B, (_bits16(got) != _bits16(want)).nonzero()[:5])
        for b in set(neutral) | set(frozen):
            assert torch.equal(_bits16(got[b * S:(b + 1) * S]), _bits16(x[b * S:(b + 1) * S])), (b, "untouched")
        assert torch.equal(_bits16(got[B * S:]), _bits16(x[B * S:])), "sentinel rows untouched"
        assert not torch.equal(_bits16(got[:S]), _bits16(x[:S])), "sequence 0 is processed"


def test_kernel_rows_not_16_byte_aligned_and_every_mask_length():
    """A (rows, V) view at a 2-byte offset with pitch V + 8 (the element-wise path), and masks of every length pattern of
    one 8-id group (0..8 allowed ids in a group)."""
    V, S, B = 32000, 9, 3
    x, g = _rows(B * S, V, 3)
    allowed = [tuple(t for t in range(V) if (t // 8) % 9 > t % 8), tuple(range(1, V, 3)), None]
    bias = [((0, 1.0), (9, -2.0)), ((1, 100.0), (2, 100.0)), ((4, _f32(0.3)),)]
    big = torch.zeros(B * S, V + 8, dtype=F16, device=DEV)
    view = big[:, 1:V + 1]
    view.copy_(x.to(DEV))
    got = _launch(x, S, allowed, bias, logits=view)
    want = process_rows(x, S, allowed, bias)
    assert torch.equal(_bits16(got), _bits16(want))
    assert not bool(big[:, 0].any()) and not bool(big[:, V + 1:].any()), "nothing outside the view is written"
    got = _launch(x, S, allowed, bias)
    assert torch.equal(_bits16(got), _bits16(want))


def test_all_neutral_launch_leaves_every_row():
    x, _ = _rows(3 * 128, 32000, 1)
    got = _launch(x, 128, [None] * 3, [(), (), ()], frozen=())
    assert torch.equal(_bits16(got), _bits16(x))


# ------------------------------------------------------------------------------------------------ composition
@pytest.mark.parametrize("k,top_p,T", [(50, 0.9, 0.6), (1000, 0.5, 1.0)])
def test_bias_then_penalty_then_top_k_then_top_p_matches_oracle(k, top_p, T):
    """As in the penalty tests, the kernel's softmax may move one fp16 probability by an ulp and so the top-p cut by one
    token: at most one differing position per row, every survivor a processed value among the top-k set."""
    from sequoia_b200.tree import _Static
    gm = cases.load_growmap("L40_growmaps/4x4-tree.pt")
    st = _Static(gm, DEV)
    S, V, B, M = gm["size"], 32000, 2, 384
    g = torch.Generator().manual_seed(k)
    x = (torch.randn(B * S, V, generator=g) * 4).to(F16)
    tokens = torch.randint(0, 300, (B, M), generator=g)
    Ps, Ls = [M - S - 5, M - S - 40], [M - S - 60, M - S - 90]
    state = torch.zeros(B, 16, dtype=torch.int32)
    state[:, ST_P] = torch.tensor(Ps)
    allowed = [tuple(range(0, V, 2)), None]
    bias = [tuple((t, 3.0) for t in range(0, 300, 4)), tuple((t, -2.0) for t in range(1, 300, 3))]
    reps, freqs, press = [_f32(1.3), _f32(0.8)], [_f32(0.7), _f32(-0.3)], [_f32(0.5), _f32(1.5)]
    out = x.clone().to(DEV)
    ops().logit_bias_rows_batch_(out, S, state.to(DEV), *_device_rows(V, allowed, bias))
    scratch = torch.zeros(ops().penalty_scratch_words(B, M), dtype=torch.int32, device=DEV)
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=DEV)  # noqa: E731
    ops().penalize_rows_batch_(out, tokens.to(DEV), state.to(DEV), torch.tensor(Ls, dtype=torch.int32, device=DEV),
                               st.tree_bits, st.tree_words, S, f32(reps), f32(freqs), f32(press), scratch)
    want_pen = penalize_rows(process_rows(x, S, allowed, bias), tokens, Ps, Ls, gm["mask"], reps, freqs, press)
    assert torch.equal(_bits16(out.cpu()), _bits16(want_pen))
    topk = top_k_filter(want_pen, k)
    want = O.top_p_filter_integer(topk, top_p, T)
    got = ops().top_p_filter_(ops().top_k_filter_(out, k), top_p, T).cpu()
    keep_g, keep_w = ~torch.isinf(got), ~torch.isinf(want)
    assert int((keep_g != keep_w).sum(-1).max()) <= 1
    assert not bool((keep_g & torch.isinf(topk)).any()) and torch.equal(got[keep_g], want_pen[keep_g])


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


def _check_greedy_step(bt, snap, slots):
    """Every token a greedy slot committed in the step equals, in value, the maximum of the oracle-processed raw target
    row it was drawn from (node 0's row for the first, then the row of each accepted node in path order)."""
    raw, state = snap
    S = bt.S
    acc = bt.accept_idx.cpu()
    new_tokens, new_state = bt.tokens.cpu(), bt.state.cpu()
    n_checked = 0
    for b in slots:
        if int(state[b, ST_FROZEN]):
            continue
        P = int(state[b, ST_P])
        n_new, a = int(new_state[b, ST_N_NEW]), int(new_state[b, 1])
        nodes = [0] + [int(s) - (P - 1) for s in acc[b, :n_new]]
        end = a + 1 if not int(new_state[b, 2]) else a
        ok = allowed_vector(bt.allowed_token_ids[b], bt.V)
        for i, pos in enumerate(range(P, min(end, bt.M))):
            row = process_row(raw[b * S + nodes[i]], ok, bt.logit_bias[b] or ())
            t = int(new_tokens[b, pos])
            assert float(row[t]) == float(row.max()), (b, pos, nodes[i], t, int(row.argmax()))
            n_checked += 1
    return n_checked


def _snapshotting(bt, snaps):
    orig = bt.op_accept

    def op_accept():
        snaps.append((bt.target_logits.cpu(), bt.state.cpu()))
        orig()
    bt.op_accept = op_accept


def _set(lo, hi, step=1):
    return tuple(range(lo, hi, step))


@pytest.mark.parametrize("policy", ["greedy", "mixed"])
def test_greedy_commits_the_argmax_of_the_processed_rows(policy):
    gm, Mx = cases.load_growmap(GM128), 512
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(500 + i, n).to(DEV) for i, n in enumerate((60, 90, 75))]
    pol = "greedy" if policy == "greedy" else ["greedy", "spec", "greedy"]
    kw = dict(policy=pol, seeds=[5, 6, 7], stop_tokens=[], logit_bias=[{7: 5.0, 900: 3.0}, None, {12: -100.0, 40: 4.0}],
              allowed_token_ids=[None, _set(0, 32000, 3), _set(0, 20000)])
    slots = [0, 1, 2] if policy == "greedy" else [0, 2]
    readmit = dict(seed=9, logit_bias={5: 2.0}, allowed_token_ids=_set(100, 400))

    def run(bt, eager):
        out, checked, snaps = [], 0, []
        if eager:
            bt.use_graphs = False
            _snapshotting(bt, snaps)
        for it in range(8):
            if it == 4:                                 # a re-admitted slot takes its new settings
                bt.freeze(2)
                bt.admit(2, cases.make_prompt(599, 50).to(DEV), **readmit)
            out.extend(_decode(bt, 1))
            if eager:
                checked += _check_greedy_step(bt, snaps[-1], slots)
        return out, checked
    eager, checked = run(_tree(engines, prompts, gm, Mx, **kw), True)
    assert checked >= 8 * len(slots)
    bt2 = _tree(engines, prompts, gm, Mx, **kw)
    graphs, _ = run(bt2, False)
    assert bt2.use_logit_bias and bt2.captures["steady"] >= 1
    _same(graphs, eager, (0, 1, 2), "graphs == eager")


@pytest.mark.parametrize("policy,gm_name", [("spec", GM128), ("greedy", GM128), ("mixed", GM128),
                                            ("spec", "L40_growmaps/16-chain.pt")])
def test_every_generated_token_is_allowed(policy, gm_name):
    gm, Mx = cases.load_growmap(gm_name), 512
    B = 3
    prompts = [cases.make_prompt(520 + i, n).to(DEV) for i, n in enumerate((40, 64, 50))]
    pol = ["spec", "greedy", "spec"] if policy == "mixed" else policy
    allowed = [_set(3, 32000, 97), _set(1000, 1050), (5, 77, 31999)]
    bt = _tree(_engines(B, Mx), prompts, gm, Mx, policy=pol, seeds=[11, 12, 13], stop_tokens=[], temperature=0.8,
               allowed_token_ids=allowed, logit_bias=[None, {1010: 2.0, 5: 50.0}, {77: -3.0}])
    steps = _decode(bt, 400)
    for b in range(B):
        v, L = steps[-1][b][0], len(prompts[b])
        assert len(v) - L >= 100, (b, len(v) - L)
        assert set(v[L:].tolist()) <= set(allowed[b]), (policy, b, sorted(set(v[L:].tolist()) - set(allowed[b]))[:5])


@pytest.mark.parametrize("policy", ["spec", "greedy"])
def test_strong_bias_makes_every_token_the_biased_id(policy):
    gm, Mx = cases.load_growmap(GM128), 384
    prompts = [cases.make_prompt(540 + i, n).to(DEV) for i, n in enumerate((40, 64))]
    targets = [1234, 31999]
    bt = _tree(_engines(2, Mx), prompts, gm, Mx, policy=policy, seeds=[3, 4], stop_tokens=[],
               logit_bias=[{t: 100} for t in targets])
    steps = _decode(bt, 100)
    for b in range(2):
        v, L = steps[-1][b][0], len(prompts[b])
        assert len(v) - L >= 100 and set(v[L:].tolist()) == {targets[b]}, (policy, b)


def test_neutral_is_free():
    gm, Mx = cases.load_growmap(GM128), 384
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(560 + i, n).to(DEV) for i, n in enumerate((70, 100, 84))]
    seeds = [21, 22, 23]
    plain_bt = _tree(engines, prompts, gm, Mx, seeds=seeds)
    plain = _decode(plain_bt, 6)
    neutral_bt = _tree(engines, prompts, gm, Mx, seeds=seeds, logit_bias=[{}, {5: 0.0}, None],
                       allowed_token_ids=[None, range(32000), None])
    neutral = _decode(neutral_bt, 6)
    assert not neutral_bt.use_logit_bias and neutral_bt.graph_launches == plain_bt.graph_launches
    _same(neutral, plain, (0, 1, 2), "all-neutral tree")
    bias_bt = _tree(engines, prompts, gm, Mx, seeds=seeds, logit_bias=[None, {7: 5.0}, {9: -100.0}],
                    allowed_token_ids=[None, None, _set(0, 32000, 2)])
    biased = _decode(bias_bt, 6)
    assert bias_bt.use_logit_bias and bias_bt.graph_launches["steady"] == plain_bt.graph_launches["steady"] + 1
    _same(biased, plain, (0,), "a neutral slot next to biased neighbours")
    assert any(not torch.equal(biased[-1][b][0], plain[-1][b][0]) for b in (1, 2)), "the settings change the output"


def test_logit_bias_captures_once():
    """Built neutral: no launch.  The first non-neutral admission captures steady and post once more (one more launch per
    steady step); later admissions, neutral or not, capture nothing.  A tree built non-neutral captures each graph once."""
    gm, Mx = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256
    engines = _engines(2, Mx)
    bt = _tree(engines, [cases.make_prompt(570, 60).to(DEV), cases.make_prompt(571, 70).to(DEV)], gm, Mx,
               policy=["spec", "greedy"], seeds=[1, 2])

    def step():
        bt.construct_grow_map()
        bt.verify()

    def admission(b, seed, **kw):
        bt.freeze(b)
        bt.admit(b, cases.make_prompt(seed, 50 + seed % 7).to(DEV), seed=seed, **kw)
        step()
        step()
    step()
    step()
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1} and not bt.use_logit_bias
    launches = bt.graph_launches["steady"]
    admission(0, 580, logit_bias={}, allowed_token_ids=range(32000))
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}, "a neutral admission captures nothing"
    admission(1, 581, allowed_token_ids=_set(0, 5000))
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2} and bt.use_logit_bias
    assert bt.graph_launches["steady"] == launches + 1, "the kernel is one more launch"
    for seed, kw in ((582, dict(logit_bias={3: 1.0})), (583, dict(allowed_token_ids=None)), (584, {})):
        admission(seed % 2, seed, **kw)
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2}, "no recapture after the kernel entered"
    built = _tree(engines, [cases.make_prompt(590, 60).to(DEV), cases.make_prompt(591, 70).to(DEV)], gm, Mx,
                  seeds=[1, 2], logit_bias=[None, {4: 1.0}])
    _decode(built, 3)
    assert built.use_logit_bias and built.captures == {"draft": 1, "post": 1, "steady": 1}


def test_logprobs_top_ids_lie_in_the_allowed_set():
    gm, Mx = cases.load_growmap(GM128), 384
    prompts = [cases.make_prompt(600 + i, n).to(DEV) for i, n in enumerate((50, 70))]
    allowed = [_set(0, 32000, 5), (10, 11, 12)]
    bt = _tree(_engines(2, Mx), prompts, gm, Mx, policy=["spec", "greedy"], seeds=[1, 2], logprobs=5,
               allowed_token_ids=allowed, stop_tokens=[])
    _decode(bt, 10)
    for b in range(2):
        lp, ids, top = bt.token_logprobs(b)
        assert lp.shape[0] >= 10 and bool(torch.isfinite(lp).all())
        fin = torch.isfinite(top)
        assert set(ids[fin].tolist()) <= set(allowed[b]), b
        assert int(fin.sum(1).min()) == min(5, len(allowed[b])), "the allowed ids are the finite ones"


def test_stop_ids_outside_the_allowed_set_never_stop():
    """Stop ids that lie outside the set can never be generated: the sequences end by their budget only.  The control
    slot, whose stop id is allowed and strongly biased, ends by its stop id."""
    gm, Mx = cases.load_growmap(GM128), 512
    prompts = [cases.make_prompt(610 + i, n).to(DEV) for i, n in enumerate((50, 70, 60))]
    allowed = [_set(100, 200), _set(3, 32000, 2), _set(100, 200)]
    bt = _tree(_engines(3, Mx), prompts, gm, Mx, policy=["spec", "greedy", "spec"], seeds=[1, 2, 3],
               allowed_token_ids=allowed, stop_tokens=[[0, 2, 99, 250], [4, 6, 8], [150]], max_new_tokens=150,
               logit_bias=[None, None, {150: 100}])
    steps = _decode(bt, 300)
    assert bt.finish_reason[:2] == ["length", "length"] and bt.finish_reason[2] == "stop"
    for b in range(2):
        assert len(steps[-1][b][0]) == len(prompts[b]) + 150


def test_logit_bias_batch_llama3_vocab():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 2, seeded: slot 0 (neutral) commits what it commits in a batch
    without the settings, and slot 1 generates only allowed ids."""
    import gc
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gc.collect()
    torch.cuda.empty_cache()
    gm, Mx = cases.load_growmap(GM128), 384
    engines = (GraphInferenceEngine(Mx, "random-init:llama-3.2-1b:1", device=DEV, batch_size=2),
               GraphInferenceEngineTG(Mx, "random-init:llama-3.1-8b:2", device=DEV, batch_size=2))
    g = torch.Generator().manual_seed(29)
    prompts = [torch.randint(3, 128256, (n,), generator=g).to(DEV) for n in (90, 128)]
    kw = dict(seeds=[31, 32], policy=["spec", "greedy"])
    allowed = _set(64000, 128256)
    bias_bt = _tree(engines, prompts, gm, Mx, allowed_token_ids=[None, allowed], logit_bias=[None, {128255: 2.0}], **kw)
    biased = _decode(bias_bt, 4)
    assert bias_bt.use_logit_bias and bias_bt.V == 128256
    plain = _decode(_tree(engines, prompts, gm, Mx, **kw), 4)
    _same(biased, plain, (0,), "slot without settings")
    v = biased[-1][1][0]
    assert len(v) >= len(prompts[1]) + len(biased) and set(v[len(prompts[1]):].tolist()) <= set(allowed)
