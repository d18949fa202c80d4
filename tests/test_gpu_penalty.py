"""Per-sequence repetition / frequency / presence penalties on the device (sq_penalize_rows_batch, BatchTree(...)).

Kernel level: the penalised rows against oracle/penalty.py bit for bit, at V from 32000 to 131072, B in {1, 3, 8}, on the
config-2 tree, a chain and a one-level wide tree, with histories of 384 and 4096 tokens, saturating values and rows
holding -inf, +inf and NaN; neutral and frozen sequences and rows past B*S untouched.  Then penalty, top-k and top-p in
that order against the oracle's composition.  BatchTree level: greedy decoding commits the argmax of the oracle-penalised
row of each context, eagerly and with graphs; a presence penalty of 1000 never repeats a generated token; neutral
settings launch and commit what a tree without them does; the graphs are captured once more at the first non-neutral
setting only; and one run at V = 128256."""
import pytest
import torch

import cases
from oracle import sequoia_oracle as O
from oracle.penalty import penalize_row, penalize_rows, row_context
from oracle.top_k import top_k_filter
from test_gpu_mixed_policy import GM128
from test_gpu_refill import DEV, F16, _engines, ops

pytestmark = pytest.mark.gpu

ST_P, ST_N_NEW, ST_P_OLD, ST_FROZEN = 0, 3, 4, 9
TINY = float(torch.tensor(1e-30, dtype=torch.float32))
# (rho, f, p) per sequence, cycled: ordinary values, saturation both ways, and a tiny rho (x / rho overflows fp32)
VALUES = [(0.5, 0.7, -0.7), (1.3, -0.7, 0.7), (TINY, 65504.0, -65504.0), (65504.0, -65504.0, 65504.0), (1.3, 0.0, 0.0),
          (1.0, 0.7, 0.0), (1.0, 0.0, -65504.0), (TINY, 0.0, 0.0)]


def _f32(vals):
    return torch.tensor(vals, dtype=torch.float32, device=DEV)


def _bits16(x):
    return x.view(torch.int16)


def _inputs(gm, B, V, M, seed, values, neutral=(), frozen=()):
    """Rows (B*S + 3 sentinel rows) with -inf / +inf / NaN entries; tokens mixing a small id range (repeats across history
    and path), the whole vocabulary and ids outside it in the prompt; P near M, L a little below P."""
    g = torch.Generator().manual_seed(seed)
    S = gm["size"]
    x = (torch.randn(B * S + 3, V, generator=g) * 4).to(F16)
    x[::5, 17] = float("-inf")
    x[1::7, 3] = float("inf")
    x[2::11, 5] = float("nan")
    tokens = torch.randint(0, 300, (B, M), generator=g)
    wide = torch.rand(B, M, generator=g) < 0.5
    tokens[wide] = torch.randint(0, V, (int(wide.sum()),), generator=g)
    tokens[:, 0], tokens[:, 2] = V + 5, -3
    Ps = [M - S + 1 - 7 * b for b in range(B)]
    Ls = [max(1, p - 40 - 13 * b) for b, p in enumerate(Ps)]
    vals = [(1.0, 0.0, 0.0) if b in neutral else values[b % len(values)] for b in range(B)]
    state = torch.zeros(B, 16, dtype=torch.int32)
    for b in range(B):
        state[b, ST_P] = Ps[b]
        state[b, ST_FROZEN] = 1 if b in frozen else 0
    # the oracle reads the device's fp32 values
    reps, freqs, press = ([float(v) for v in torch.tensor(c, dtype=torch.float32)] for c in zip(*vals))
    return x, tokens, Ps, Ls, state, reps, freqs, press


def _launch(st, x, tokens, Ls, state, reps, freqs, press):
    B, M = tokens.shape
    out = x.clone().to(DEV)
    scratch = torch.full((ops().penalty_scratch_words(B, M),), -7, dtype=torch.int32, device=DEV)
    ops().penalize_rows_batch_(out, tokens.to(DEV), state.to(DEV), torch.tensor(Ls, dtype=torch.int32, device=DEV),
                               st.tree_bits, st.tree_words, st.S, _f32(reps), _f32(freqs), _f32(press), scratch)
    torch.cuda.synchronize()
    return out.cpu()


GROWMAPS = {"config2": GM128, "chain": "L40_growmaps/16-chain.pt", "wide": "L40_growmaps/128x1-tree.pt"}


@pytest.mark.parametrize("V", [32000, 49152, 128256, 131072])
@pytest.mark.parametrize("tree", list(GROWMAPS))
@pytest.mark.parametrize("M", [384, 4096])
def test_kernel_matches_oracle(V, tree, M):
    from sequoia_b200.tree import _Static
    gm = cases.load_growmap(GROWMAPS[tree])
    st = _Static(gm, DEV)
    S = gm["size"]
    for B in (1, 3, 8):
        neutral, frozen = ((), ()) if B == 1 else ((1,), (B - 1,))
        x, tokens, Ps, Ls, state, reps, freqs, press = _inputs(gm, B, V, M, V + M + B + S, VALUES, neutral, frozen)
        got = _launch(st, x, tokens, Ls, state, reps, freqs, press)
        want = penalize_rows(x, tokens, Ps, Ls, gm["mask"], reps, freqs, press, frozen=[b in frozen for b in range(B)])
        assert torch.equal(_bits16(got), _bits16(want)), (V, tree, M, B, (_bits16(got) != _bits16(want)).nonzero()[:5])
        for b in set(neutral) | set(frozen):
            assert torch.equal(_bits16(got[b * S:(b + 1) * S]), _bits16(x[b * S:(b + 1) * S])), (b, "untouched")
        assert torch.equal(_bits16(got[B * S:]), _bits16(x[B * S:])), "sentinel rows untouched"
        assert not torch.equal(_bits16(got[:S]), _bits16(x[:S])), "sequence 0 is penalised"
        fin = torch.isfinite(x)
        assert bool(torch.isfinite(got[fin]).all()) and bool(torch.isnan(got[~fin & torch.isnan(x)]).all())


def test_all_neutral_launch_leaves_every_row():
    from sequoia_b200.tree import _Static
    gm = cases.load_growmap(GM128)
    st = _Static(gm, DEV)
    x, tokens, Ps, Ls, state, reps, freqs, press = _inputs(gm, 3, 32000, 384, 1, VALUES, neutral=(0, 1, 2))
    got = _launch(st, x, tokens, Ls, state, reps, freqs, press)
    assert torch.equal(_bits16(got), _bits16(x))


# ------------------------------------------------------------------------------------------------ composition
@pytest.mark.parametrize("k,top_p,T", [(50, 0.9, 0.6), (1000, 0.5, 1.0)])
def test_penalty_then_top_k_then_top_p_matches_oracle(k, top_p, T):
    """As in the top-k tests, the kernel's softmax may move one fp16 probability by an ulp and so the top-p cut by one
    token: at most one differing position per row, every survivor a penalised value among the top-k set."""
    from sequoia_b200.tree import _Static
    gm = cases.load_growmap("L40_growmaps/4x4-tree.pt")
    st = _Static(gm, DEV)
    V = 32000
    x, tokens, Ps, Ls, state, reps, freqs, press = _inputs(gm, 2, V, 384, k, [(1.3, 0.7, 0.5), (0.8, -0.3, 1.5)])
    x = torch.nan_to_num(x, nan=0.0, posinf=0.0)
    pen = _launch(st, x, tokens, Ls, state, reps, freqs, press)
    want_pen = penalize_rows(x, tokens, Ps, Ls, gm["mask"], reps, freqs, press)
    assert torch.equal(_bits16(pen), _bits16(want_pen))
    topk = top_k_filter(want_pen, k)
    want = O.top_p_filter_integer(topk, top_p, T)
    got = ops().top_p_filter_(ops().top_k_filter_(pen.clone().to(DEV), k), top_p, T).cpu()
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


def _check_greedy_step(bt, snap, slots, gm):
    """Every token a greedy slot committed in the step equals, in value, the maximum of the oracle-penalised raw target
    row of its context (node 0's row for the first, then the row of each accepted node in path order)."""
    raw, tokens, state = snap
    S = bt.S
    acc = bt.accept_idx.cpu()
    new_tokens, new_state = bt.tokens.cpu(), bt.state.cpu()
    n_checked = 0
    for b in slots:
        if int(state[b, ST_FROZEN]):
            continue
        P = int(state[b, ST_P])
        L = int(bt.prompt_len_dev[b])
        n_new, a = int(new_state[b, ST_N_NEW]), int(new_state[b, 1])
        nodes = [0] + [int(s) - (P - 1) for s in acc[b, :n_new]]
        end = a + 1 if not int(new_state[b, 2]) else a           # (a terminal walk commits no bonus token)
        for i, pos in enumerate(range(P, min(end, bt.M))):
            k = nodes[i]
            slots_k, ids = row_context(tokens[b], P, gm["mask"], k)
            row = penalize_row(raw[b * S + k], ids, slots_k >= L, bt.repetition_penalty[b], bt.frequency_penalty[b],
                               bt.presence_penalty[b])
            t = int(new_tokens[b, pos])
            assert float(row[t]) == float(row.max()), (b, pos, k, t, int(row.argmax()))
            n_checked += 1
    return n_checked


def _snapshotting(bt, snaps):
    orig = bt.op_accept

    def op_accept():
        snaps.append((bt.target_logits.cpu(), bt.tokens.cpu(), bt.state.cpu()))
        orig()
    bt.op_accept = op_accept


@pytest.mark.parametrize("policy", ["greedy", "mixed"])
def test_greedy_commits_the_argmax_of_the_penalised_rows(policy):
    gm, Mx = cases.load_growmap(GM128), 512
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(400 + i, n).to(DEV) for i, n in enumerate((60, 90, 75))]
    pol = "greedy" if policy == "greedy" else ["greedy", "spec", "greedy"]
    kw = dict(policy=pol, seeds=[5, 6, 7], stop_tokens=[], repetition_penalty=[1.3, 1.2, 0.7],
              frequency_penalty=[0.4, 0.0, 1.5], presence_penalty=[0.5, 0.2, -0.3])
    slots = [0, 1, 2] if policy == "greedy" else [0, 2]
    bt = _tree(engines, prompts, gm, Mx, **kw)
    bt.use_graphs = False
    snaps = []
    _snapshotting(bt, snaps)
    eager, checked = [], 0
    for it in range(8):
        if it == 4:                                     # a re-admitted slot counts only its new prompt
            bt.freeze(2)
            bt.admit(2, cases.make_prompt(499, 50).to(DEV), seed=9, presence_penalty=3.0)
        bt.construct_grow_map()
        eager.append([(v.cpu().clone(), a, term) for v, a, term in bt.verify()])
        checked += _check_greedy_step(bt, snaps[-1], slots, gm)
    assert checked >= 8 * len(slots)
    bt2 = _tree(engines, prompts, gm, Mx, **kw)
    graphs = []
    for it in range(8):
        if it == 4:
            bt2.freeze(2)
            bt2.admit(2, cases.make_prompt(499, 50).to(DEV), seed=9, presence_penalty=3.0)
        graphs.extend(_decode(bt2, 1))
    assert bt2.use_penalty and bt2.captures["steady"] >= 1
    _same(graphs, eager, (0, 1, 2), "graphs == eager")


def _repeats(tokens, L):
    out = tokens[L:].tolist()
    return len(out) - len(set(out))


@pytest.mark.parametrize("policy,gm_name", [("greedy", GM128), ("spec", "L40_growmaps/16-chain.pt")])
def test_presence_penalty_never_repeats_a_generated_token(policy, gm_name):
    gm, Mx = cases.load_growmap(gm_name), 512
    B = 2
    prompts = [cases.make_prompt(420 + i, n).to(DEV) for i, n in enumerate((40, 64))]
    base = dict(policy=policy, seeds=[11, 12], stop_tokens=[], temperature=0.8)
    engines = _engines(B, Mx)
    free = _decode(_tree(engines, prompts, gm, Mx, **base), 400)
    bt = _tree(engines, prompts, gm, Mx, presence_penalty=1000.0, **base)
    steps = _decode(bt, 400)
    for b in range(B):
        v = steps[-1][b][0]
        L = len(prompts[b])
        assert len(v) - L >= 128, (b, len(v) - L)
        assert _repeats(v, L) == 0, (policy, b)
    assert sum(_repeats(free[-1][b][0], len(prompts[b])) for b in range(B)) > 0, "without the penalty tokens repeat"


def test_neutral_is_free():
    gm, Mx = cases.load_growmap(GM128), 384
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(440 + i, n).to(DEV) for i, n in enumerate((70, 100, 84))]
    seeds = [21, 22, 23]
    plain_bt = _tree(engines, prompts, gm, Mx, seeds=seeds)
    plain = _decode(plain_bt, 6)
    neutral_bt = _tree(engines, prompts, gm, Mx, seeds=seeds, repetition_penalty=[1.0] * 3, frequency_penalty=0.0,
                       presence_penalty=[0.0, -0.0, 0.0])
    neutral = _decode(neutral_bt, 6)
    assert not neutral_bt.use_penalty and neutral_bt.graph_launches == plain_bt.graph_launches
    _same(neutral, plain, (0, 1, 2), "all-neutral tree")
    pen_bt = _tree(engines, prompts, gm, Mx, seeds=seeds, repetition_penalty=[1.0, 1.3, 1.1],
                   presence_penalty=[0.0, 0.5, 2.0])
    pen = _decode(pen_bt, 6)
    assert pen_bt.use_penalty and pen_bt.graph_launches["steady"] == plain_bt.graph_launches["steady"] + 2
    _same(pen, plain, (0,), "a neutral slot next to penalised neighbours")
    assert any(not torch.equal(pen[-1][b][0], plain[-1][b][0]) for b in (1, 2)), "penalties change the output"


def test_penalties_capture_once():
    """Built neutral: no penalty launch.  The first non-neutral admission (here a greedy one) captures steady and post once
    more (two more launches per steady step); later admissions, neutral or not, capture nothing.  A tree built with
    penalties captures each graph once."""
    gm, Mx = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256
    engines = _engines(2, Mx)
    bt = _tree(engines, [cases.make_prompt(450, 60).to(DEV), cases.make_prompt(451, 70).to(DEV)], gm, Mx,
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
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1} and not bt.use_penalty
    launches = bt.graph_launches["steady"]
    admission(0, 460)
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}, "a neutral admission captures nothing"
    admission(1, 461, repetition_penalty=1.2)
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2} and bt.use_penalty
    assert bt.graph_launches["steady"] == launches + 2, "the penalty kernels are two more launches"
    for seed, kw in ((462, dict(presence_penalty=0.5)), (463, dict(repetition_penalty=1.0)), (464, {})):
        admission(seed % 2, seed, **kw)
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2}, "no recapture after the penalties entered"
    built = _tree(engines, [cases.make_prompt(470, 60).to(DEV), cases.make_prompt(471, 70).to(DEV)], gm, Mx,
                  seeds=[1, 2], frequency_penalty=[0.0, 0.3])
    _decode(built, 3)
    assert built.use_penalty and built.captures == {"draft": 1, "post": 1, "steady": 1}


def test_penalty_batch_llama3_vocab():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 2, seeded, penalties on slot 1: slot 0 commits what it commits in a
    batch without penalties, and slot 1 decodes."""
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
    pen_bt = _tree(engines, prompts, gm, Mx, repetition_penalty=[1.0, 1.3], presence_penalty=[0.0, 0.5], **kw)
    pen = _decode(pen_bt, 4)
    assert pen_bt.use_penalty and pen_bt.V == 128256
    plain = _decode(_tree(engines, prompts, gm, Mx, **kw), 4)
    _same(pen, plain, (0,), "slot without penalties")
    assert len(pen[-1][1][0]) >= len(prompts[1]) + len(pen)
