"""Per-sequence logprobs on the device (sq_token_logprobs_batch, BatchTree(logprobs=...)).

Kernel level: every value against oracle/logprobs.py (float64) at V from 32000 to 131072, B in {1, 3, 8}, on the
config-2 tree, a chain and a one-level wide tree, with synthetic steps covering every path depth, terminal, NaN, no-room,
frozen and off sequences, n in {0, 1, 5, 20} and T in {0.05, 0.6, 1, 2}; everything the kernel must not write is
untouched bit for bit.  BatchTree level: mixed batches with penalties, top-k and top-p against the oracle applied to each
step's post-walk rows, graphs against eager, the greedy / sampled invariants, a teacher-forced float32 forward of the
committed tokens (a dense causal pass that shares no code with the tree verify), the lifecycle (off is free, one
recapture, output lengths under stop ids and budgets, slot independence) and one run at V = 128256."""
import math

import numpy as np
import pytest
import torch

import cases
from oracle import logprobs as L
from oracle import sequoia_oracle as O
from test_gpu_mixed_policy import GM128
from test_gpu_refill import DEV, F16, _engines, ops

pytestmark = pytest.mark.gpu

NMAX = L.MAX_LOGPROBS
TOK_SENT, ID_SENT, TOP_SENT = 12345.0, -7, 777.0
GROWMAPS = {"config2": GM128, "chain": "L40_growmaps/16-chain.pt", "wide": "L40_growmaps/128x1-tree.pt"}
TEMPS = [0.05, 0.6, 1.0, 2.0]
NS = [0, 1, 5, 20]


def _walk(gm, depth, pick):
    succ, node, path = gm["Successors"], 0, []
    for _ in range(depth):
        kids = list(succ[node])
        if not kids:
            break
        node = int(kids[(pick * 7 + len(path)) % len(kids)])
        path.append(node)
    return path


def _deepest(gm):
    """The path from the root to the deepest node (its ancestors-or-self below the root, by depth)."""
    k = int(gm["depth"].argmax())
    return sorted((j for j in range(1, gm["size"]) if bool(gm["mask"][k, j])), key=lambda j: int(gm["depth"][j]))


def _inputs(gm, B, V, M, seed):
    """Rows with ties, -inf runs, a +inf row and a NaN row; per sequence a walked path of its own depth and a kind:
    0 normal, 1 terminal, 2 NaN end (terminal), 3 no room for the bonus, 4 frozen, 5 off, 6 greedy, 7 an id outside V."""
    g = torch.Generator().manual_seed(seed)
    S = gm["size"]
    D = int(gm["depth"].max())
    x = (torch.randn(B * S, V, generator=g) * 4).to(F16)
    x[::3, 100:140] = 2.5                               # a tie group
    x[1::4, ::2] = float("-inf")                        # filtered halves
    x[2::5, 10:20] = 0.0
    x[2::5, 20:30] = -0.0
    x[3, 7] = float("inf")
    x[min(4, B * S - 1), 9] = float("nan")
    tokens = torch.randint(0, V, (B, M), generator=g)
    state = torch.zeros(B, 16, dtype=torch.int32)
    acc = torch.zeros(B, max(S, 8), dtype=torch.int32)
    T, greedy, n_top = [], [], []
    for b in range(B):
        kind = b % 8 if B > 1 else 0
        depth = [D, 0, 1, max(D - 1, 0), D, 2, D, 1][b % 8] if B > 1 else D
        path = _deepest(gm) if depth == D else _walk(gm, depth, b)
        P = 60 + 5 * b
        n_new = len(path)
        acc[b, :n_new] = torch.tensor([P - 1 + k for k in path], dtype=torch.int32)
        state[b, L.ST_P_OLD], state[b, L.ST_N_NEW] = P, n_new
        state[b, L.ST_M] = P + n_new if kind == 3 else M
        state[b, L.ST_TERMINAL] = 1 if kind in (1, 2) else 0
        state[b, 6] = 1 if kind == 2 else 0
        state[b, L.ST_FROZEN] = 1 if kind == 4 else 0
        if kind == 7:
            tokens[b, P] = V + 3
        T.append(TEMPS[b % 4])
        greedy.append(kind == 6)
        n_top.append(None if kind == 5 else NS[(b + seed) % 4])
    return x, tokens, state, acc, T, greedy, n_top


def _launch(x, S, D, tokens, state, acc, T, greedy, n_top):
    B, M = tokens.shape
    lp_token = torch.full((B, M), TOK_SENT, dtype=torch.float32, device=DEV)
    lp_ids = torch.full((B, M, NMAX), ID_SENT, dtype=torch.int32, device=DEV)
    lp_top = torch.full((B, M, NMAX), TOP_SENT, dtype=torch.float32, device=DEV)
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=DEV)
    ops().token_logprobs_batch_(x.to(DEV), S, D, tokens.to(DEV), state.to(DEV), acc.to(DEV),
                                torch.tensor(T, dtype=torch.float32, device=DEV), i32([int(v) for v in greedy]),
                                i32([-1 if n is None else n for n in n_top]), lp_token, lp_ids, lp_top)
    torch.cuda.synchronize()
    return lp_token.cpu(), lp_ids.cpu(), lp_top.cpu()


def _lse(row, T, greedy):
    s = L.scaled(row, T, greedy)
    m = s.max()
    return float(m + np.log(np.exp(s - m).sum())) if np.isfinite(m) else 0.0


def _close(got, want, lse):
    if math.isnan(want) or math.isinf(want):
        return (math.isnan(got) and math.isnan(want)) or got == want
    return abs(got - want) <= 1e-4 * (1 + abs(lse))


def _check_step(x, S, tokens, state, acc, T, greedy, n_top, got):
    """Every written value against the oracle; every other element keeps its sentinel."""
    lp_token, lp_ids, lp_top = got
    want = L.step_logprobs(x, S, tokens, state, acc, T, greedy, n_top)
    B, M = tokens.shape
    tok_written = torch.zeros(B, M, dtype=torch.bool)
    top_written = torch.zeros(B, M, NMAX, dtype=torch.bool)
    for (b, pos), (t_lp, ids, tops) in want.items():
        j = pos - int(state[b, L.ST_P_OLD])
        row = x[b * S + L.path_node(state[b], acc[b], j)]
        lse = _lse(row, T[b], greedy[b])
        assert _close(float(lp_token[b, pos]), t_lp, lse), (b, pos, float(lp_token[b, pos]), t_lp)
        n = len(ids)
        assert lp_ids[b, pos, :n].tolist() == ids, (b, pos, lp_ids[b, pos, :n].tolist(), ids)
        for i in range(n):
            assert _close(float(lp_top[b, pos, i]), tops[i], lse), (b, pos, i, float(lp_top[b, pos, i]), tops[i])
        tok_written[b, pos] = True
        top_written[b, pos, :n] = True
    assert bool((lp_token[~tok_written] == TOK_SENT).all()), "an unwritten logprob changed"
    assert bool((lp_ids[~top_written] == ID_SENT).all()) and bool((lp_top[~top_written] == TOP_SENT).all()), \
        "an unwritten top entry changed"
    return len(want)


@pytest.mark.parametrize("V", [32000, 49152, 128256, 131072])
@pytest.mark.parametrize("tree", list(GROWMAPS))
def test_kernel_matches_oracle(V, tree):
    gm = cases.load_growmap(GROWMAPS[tree])
    S, D = gm["size"], int(gm["depth"].max())
    written = 0
    for B in (1, 3, 8):
        for seed in range(2):
            x, tokens, state, acc, T, greedy, n_top = _inputs(gm, B, V, 384, V + B + seed)
            got = _launch(x, S, D, tokens, state, acc, T, greedy, n_top)
            written += _check_step(x, S, tokens, state, acc, T, greedy, n_top, got)
    assert written >= 2 * D, "the steps commit positions"


def test_all_off_or_frozen_writes_nothing():
    gm = cases.load_growmap(GM128)
    x, tokens, state, acc, T, greedy, _ = _inputs(gm, 3, 32000, 384, 5)
    got = _launch(x, gm["size"], int(gm["depth"].max()), tokens, state, acc, T, greedy, [None] * 3)
    assert bool((got[0] == TOK_SENT).all()) and bool((got[1] == ID_SENT).all()) and bool((got[2] == TOP_SENT).all())


def test_ops_refusals_on_the_device():
    from sequoia_b200 import _lib
    B, S, M, V = 2, 4, 16, 64
    x = torch.zeros(B * S, V, dtype=F16, device=DEV)
    i32 = lambda *s: torch.zeros(*s, dtype=torch.int32, device=DEV)
    f32 = lambda *s: torch.zeros(*s, dtype=torch.float32, device=DEV)
    good = dict(target_logits=x, S=S, max_depth=1, tokens=torch.zeros(B, M, dtype=torch.long, device=DEV),
                state=i32(B, 16), accept_idx=i32(B, 8), T=torch.ones(B, device=DEV), greedy=i32(B), n_top=i32(B),
                lp_token=f32(B, M), lp_ids=i32(B, M, NMAX), lp_top=f32(B, M, NMAX))
    for bad, err in ((dict(target_logits=x[:B * S - 1]), ValueError), (dict(T=torch.ones(B, dtype=torch.float64,
                                                                                         device=DEV)), TypeError),
                     (dict(n_top=f32(B)), TypeError), (dict(greedy=i32(1)), TypeError),
                     (dict(lp_token=f32(B, M + 1)), ValueError), (dict(lp_ids=i32(B, M, 5)), ValueError),
                     (dict(lp_top=i32(B, M, NMAX)), TypeError), (dict(tokens=i32(B, M)), TypeError),
                     (dict(max_depth=S), _lib.SequoiaLibError)):
        with pytest.raises(err):
            ops().token_logprobs_batch_(**{**good, **bad})


# ------------------------------------------------------------------------------------------------ BatchTree
def _tree(engines, prompts, gm, Mx, **kw):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    d.clear_kv()
    t.clear_kv()
    return BatchTree(d, t, prompts, gm, max_length=Mx, max_target_seq=Mx, **kw)


def _snapshotting(bt, snaps):
    """Record each step's rows, tokens, state and accept_idx as the logprobs kernel reads them (after the walk)."""
    orig = bt.op_logprobs

    def op_logprobs():
        snaps.append((bt.target_logits.cpu(), bt.tokens.cpu(), bt.state.cpu(), bt.accept_idx.cpu()))
        orig()
    bt.op_logprobs = op_logprobs


def _buffers(bt):
    return bt.lp_token.cpu(), bt.lp_ids.cpu(), bt.lp_top.cpu()


MIXED = dict(policy=["spec", "greedy", "spec"], seeds=[5, 6, 7], temperature=[0.6, 1.0, 1.3], top_k=[50, 0, 50],
             top_p=[0.9, 1.0, 0.9], repetition_penalty=[1.2, 1.1, 1.0], presence_penalty=[0.3, 0.5, 0.0],
             stop_tokens=[], logprobs=[20, 5, 0])


def _mixed_prompts():
    return [cases.make_prompt(600 + i, n).to(DEV) for i, n in enumerate((60, 90, 75))]


def test_composition_invariants_and_graphs():
    """Eager: after every step, each written value equals the oracle applied to that step's post-walk rows (penalised,
    top-k and top-p filtered); the greedy and sampled invariants hold.  Graphs: identical logprob buffers."""
    gm, Mx = cases.load_growmap(GM128), 512
    engines = _engines(3, Mx)
    prompts = _mixed_prompts()
    bt = _tree(engines, prompts, gm, Mx, **MIXED)
    bt.use_graphs = False
    snaps = []
    _snapshotting(bt, snaps)
    S, greedy = bt.S, [p == "greedy" for p in bt.policies]
    checked = {"greedy": 0, "sampled": 0}
    for it in range(8):
        before = _buffers(bt)
        bt.construct_grow_map()
        bt.verify()
        x, tokens, state, acc = snaps[-1]
        want = L.step_logprobs(x, S, tokens, state, acc, bt.temps, greedy, bt.logprobs)
        lp_token, lp_ids, lp_top = _buffers(bt)
        for (b, pos), (t_lp, ids, tops) in want.items():
            j = pos - int(state[b, L.ST_P_OLD])
            lse = _lse(x[b * S + L.path_node(state[b], acc[b], j)], bt.temps[b], greedy[b])
            assert _close(float(lp_token[b, pos]), t_lp, lse), (it, b, pos)
            assert lp_ids[b, pos, :len(ids)].tolist() == ids, (it, b, pos)
            assert all(_close(float(lp_top[b, pos, i]), v, lse) for i, v in enumerate(tops)), (it, b, pos)
            if L.is_bonus_replacement(state[b], acc[b], j):
                continue
            if greedy[b]:
                assert int(lp_ids[b, pos, 0]) == int(tokens[b, pos]) and float(lp_token[b, pos]) == float(lp_top[b, pos, 0])
                checked["greedy"] += 1
            else:
                assert math.isfinite(float(lp_token[b, pos])), (it, b, pos, "a committed token was filtered")
                checked["sampled"] += 1
        unwritten = torch.ones_like(lp_token, dtype=torch.bool)
        for b, pos in want:
            unwritten[b, pos] = False
        assert torch.equal(lp_token.view(torch.int32)[unwritten], before[0].view(torch.int32)[unwritten]), \
            "only committed positions are written"
    assert checked["greedy"] >= 8 and checked["sampled"] >= 8, checked
    eager = _buffers(bt)
    bt2 = _tree(engines, prompts, gm, Mx, **MIXED)
    for _ in range(8):
        bt2.construct_grow_map()
        bt2.verify()
    assert bt2.captures["steady"] >= 1 and bt2.use_logprobs
    graphs = _buffers(bt2)
    for e, g in zip(eager, graphs):
        assert torch.equal(e.view(torch.int32), g.view(torch.int32)), "graphs == eager, bit for bit"
    for b in range(3):
        lp, ids, top = bt2.token_logprobs(b)
        assert lp.shape[0] == len(bt2.last[b][0]) - len(prompts[b]) and ids.shape == (lp.shape[0], bt2.logprobs[b])


def test_teacher_forced_float32_forward():
    """Greedy at T = 1, no filter, no penalty: token_logprobs(b) against log_softmax of a float32 causal forward of the
    same weights over the committed tokens (oracle.sequoia_oracle.LlamaOracle on the CPU, no code shared with the tree
    verify), position p read from the forward's row p - 1.
    Tolerance: |d logprob| <= |d x_t| + |d logsumexp(x)| <= 2 max_i |d x_i|.  The device's logits are fp16 (|x| < 4 for
    this random-init target: one rounding <= 2^-10) after fp16 activations through 3 layers, which the CPU fp16 path
    shows to move a logit by about 2e-3 from float32; 2^-8 = 3.9e-3 bounds d x with margin, so a token may differ by 2^-7
    and a sum of n tokens by n * 2^-7.  A row one position off moves a greedy token's logprob by about 2 (the argmax of
    one context is an ordinary token of the next), far outside."""
    gm, Mx = cases.load_growmap(GM128), 384
    B = 2
    engines = _engines(B, Mx)
    prompts = [cases.make_prompt(640 + i, n) for i, n in enumerate((50, 70))]
    bt = _tree(engines, [p.to(DEV) for p in prompts], gm, Mx, policy="greedy", temperature=1.0, stop_tokens=[],
               logprobs=3)
    for _ in range(6):
        bt.construct_grow_map()
        bt.verify()
    cfg, w = cases.model_weights("target")
    ref = O.EngineOracle(O.LlamaOracle(cfg, {k: v.float() for k, v in w.items()}, Mx, "TG", dtype=torch.float32))
    tol = 2.0 ** -7
    for b in range(B):
        seq = bt.last[b][0].cpu()
        Lp, n = len(prompts[b]), len(seq)
        assert n - Lp >= 6
        ref.model.kv_cache.clear()
        logits = ref.inference(seq[None], torch.arange(n), torch.arange(n)[None],
                               O.make_causal_mask(n, torch.float32)[None, None])[0].double()
        want = torch.log_softmax(logits, -1)[Lp - 1:n - 1].gather(1, seq[Lp:, None]).squeeze(1)
        lp, ids, _ = bt.token_logprobs(b)
        assert lp.shape == want.shape
        err = (lp.double() - want).abs()
        assert float(err.max()) <= tol, (b, float(err.max()), int(err.argmax()))
        assert abs(float(lp.double().sum() - want.sum())) <= tol * len(lp)
        assert torch.equal(ids[:, 0], seq[Lp:]), "greedy: the committed token is its row's best"


def _decode(bt, iters):
    out = []
    for _ in range(iters):
        bt.construct_grow_map()
        out.append([(v.cpu().clone(), a, term) for v, a, term in bt.verify()])
        if all(bt.frozen):
            break
    return out


def test_off_is_free():
    gm, Mx = cases.load_growmap(GM128), 384
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(660 + i, n).to(DEV) for i, n in enumerate((70, 100, 84))]
    kw = dict(seeds=[21, 22, 23], policy=["spec", "greedy", "spec"])
    plain_bt = _tree(engines, prompts, gm, Mx, **kw)
    plain = _decode(plain_bt, 6)
    off_bt = _tree(engines, prompts, gm, Mx, logprobs=[None] * 3, **kw)
    off = _decode(off_bt, 6)
    assert not off_bt.use_logprobs and off_bt.lp_token is None and off_bt.graph_launches == plain_bt.graph_launches
    assert off_bt.kernel_launches() == plain_bt.kernel_launches()
    on_bt = _tree(engines, prompts, gm, Mx, logprobs=[None, 2, 20], **kw)
    on = _decode(on_bt, 6)
    assert on_bt.graph_launches["steady"] == plain_bt.graph_launches["steady"] + 1
    for got in (off, on):
        for it in range(len(plain)):
            for b in range(3):
                assert torch.equal(got[it][b][0], plain[it][b][0]) and got[it][b][1:] == plain[it][b][1:], (it, b)


def test_first_request_recaptures_once():
    gm, Mx = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256
    engines = _engines(2, Mx)
    bt = _tree(engines, [cases.make_prompt(670, 60).to(DEV), cases.make_prompt(671, 70).to(DEV)], gm, Mx,
               policy=["spec", "greedy"], seeds=[1, 2])

    def admission(b, seed, **kw):
        bt.freeze(b)
        bt.admit(b, cases.make_prompt(seed, 50 + seed % 7).to(DEV), seed=seed, **kw)
        _decode(bt, 2)
    _decode(bt, 2)
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1} and not bt.use_logprobs
    launches = bt.graph_launches["steady"]
    admission(0, 680)
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}, "an admission with logprobs off captures nothing"
    admission(1, 681, logprobs=4)
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2} and bt.use_logprobs
    assert bt.graph_launches["steady"] == launches + 1, "the logprobs kernel is one more launch"
    lp, ids, top = bt.token_logprobs(1)
    assert lp.shape[0] == len(bt.last[1][0]) - len(cases.make_prompt(681, 50 + 681 % 7)) and ids.shape[1] == 4
    for seed, kw in ((682, dict(logprobs=20)), (683, dict(logprobs=None)), (684, {})):
        admission(seed % 2, seed, **kw)
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2}, "no recapture after the logprobs kernel entered"


def test_output_length_follows_stops_and_budgets():
    gm, Mx = cases.load_growmap(GM128), 384
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(690 + i, n).to(DEV) for i, n in enumerate((60, 80, 70))]
    # slot 0 stops at a frequent id of a plain run, slot 1 has a budget, slot 2 neither
    plain = _decode(_tree(engines, prompts, gm, Mx, seeds=[1, 2, 3], stop_tokens=[]), 8)
    stop_id = int(plain[-1][0][0][len(prompts[0]) + 3])
    bt = _tree(engines, prompts, gm, Mx, seeds=[1, 2, 3], stop_tokens=[[stop_id], [], []],
               max_new_tokens=[None, 13, None], logprobs=[1, 0, 5])
    for _ in range(40):
        bt.construct_grow_map()
        res = bt.verify()
        for b in range(3):
            lp, ids, top = bt.token_logprobs(b)
            assert lp.shape[0] == len(res[b][0]) - len(prompts[b]) == ids.shape[0] == top.shape[0], b
            assert bool(torch.isfinite(lp).all()), b
        if all(bt.frozen[:2]):
            break
    assert bt.finish_reason[0] == "stop" and bt.finish_reason[1] == "length"
    assert bt.token_logprobs(1)[0].shape[0] == 13


def test_seeded_sequence_same_logprobs_in_any_slot():
    gm, Mx = cases.load_growmap(GM128), 384
    engines = _engines(3, Mx)
    pairs = [(cases.make_prompt(700 + i, n).to(DEV), s) for i, (n, s) in enumerate(((70, 11), (95, 12), (82, 13)))]
    runs = []
    for order in ([0, 1, 2], [2, 0, 1]):
        bt = _tree(engines, [pairs[i][0] for i in order], gm, Mx, seeds=[pairs[i][1] for i in order],
                   temperature=0.8, top_k=40, logprobs=5)
        _decode(bt, 6)
        runs.append({i: bt.token_logprobs(b) for b, i in enumerate(order)})
    for i in range(3):
        for x, y in zip(runs[0][i], runs[1][i]):
            assert torch.equal(x, y), i


def test_logprobs_batch_llama3_vocab():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 2: slot 0 with 20 alternatives at T = 1, slot 1 off; both commit
    what they commit without logprobs."""
    import gc
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gc.collect()
    torch.cuda.empty_cache()
    gm, Mx = cases.load_growmap(GM128), 384
    engines = (GraphInferenceEngine(Mx, "random-init:llama-3.2-1b:1", device=DEV, batch_size=2),
               GraphInferenceEngineTG(Mx, "random-init:llama-3.1-8b:2", device=DEV, batch_size=2))
    g = torch.Generator().manual_seed(31)
    prompts = [torch.randint(3, 128256, (n,), generator=g).to(DEV) for n in (90, 128)]
    kw = dict(seeds=[41, 42], policy=["spec", "greedy"], temperature=1.0)
    lp_bt = _tree(engines, prompts, gm, Mx, logprobs=[20, None], **kw)
    got = _decode(lp_bt, 4)
    plain = _decode(_tree(engines, prompts, gm, Mx, **kw), 4)
    for it in range(len(plain)):
        for b in range(2):
            assert torch.equal(got[it][b][0], plain[it][b][0]), (it, b)
    lp, ids, top = lp_bt.token_logprobs(0)
    assert lp_bt.V == 128256 and lp.shape[0] == len(got[-1][0][0]) - len(prompts[0]) >= 4 and ids.shape[1] == 20
    assert bool(torch.isfinite(lp).all()) and bool(((ids >= 0) & (ids < 128256)).all())
    assert bool((top[:, :-1] >= top[:, 1:]).all()) and bool((lp <= top[:, 0] + 1e-6).all())
    assert float(torch.logsumexp(top.double(), -1).max()) <= 1e-6, "20 probabilities sum to at most 1"
    with pytest.raises(ValueError, match="off"):
        lp_bt.token_logprobs(1)
