"""Per-sequence counter-based random numbers on the device (csrc/sq_rng.cu) and the seeded BatchTree.

Kernel level: the filled r / rand rows and the bonus noise against the CPU restatement (oracle/philox.py) bit for bit, the
noise counters, and the distributions the sampler and the bonus draw make from them.  BatchTree level: a seeded tree draws
only from its seeds (buffers equal the restatement for (seed, step) at every step, graph captures included; torch's
generators untouched), a sequence's tokens do not depend on its slot, and a seeded steady step is still two replays and
one host sync."""
import contextlib
import os

import numpy as np
import pytest
import scipy.stats
import torch

import cases
from oracle import philox

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
F16 = torch.float16
GM = "L40_growmaps/8x8-tree.pt"
ST_P, ST_M, ST_FROZEN = 0, 8, 9
SEEDS = [0, 1, 0xFFFFFFFFFFFFFFFF, 0x8000000000000000, 0x0123456789ABCDEF, 17 << 32, (17 << 32) | 5, 0xDEADBEEF]


def ops():
    from sequoia_b200 import ops as _ops
    return _ops


def _seeds_dev(seeds):
    from sequoia_b200.batch import _as_int64
    return torch.tensor([_as_int64(s) for s in seeds], dtype=torch.int64, device=DEV)


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


def _state(B, frozen=()):
    st = torch.zeros(B, 16, dtype=torch.int32)
    st[:, ST_P] = 1
    st[:, ST_M] = 1024
    for b in frozen:
        st[b, ST_FROZEN] = 1
    return st.to(DEV)


# ------------------------------------------------------------------------------------------------ fill
@pytest.mark.parametrize("V", [32000, 128256])
@pytest.mark.parametrize("B,slots", [(1, [0]), (3, [2, 0]), (8, [7, 1, 4, 2, 5])])
def test_fill_matches_the_restatement(B, slots, V):
    """rand (B, S, V) and r (B, M) for a slot list, M = 384 (vector stores) and 389 (odd row pitch: element stores):
    every listed row equals the restatement for its seed; the sentinel rows of unlisted slots are unchanged."""
    S = 5
    seeds = SEEDS[:B]
    sd = _seeds_dev(seeds)
    for purpose, shape in ((philox.RAND, (B, S, V)), (philox.R, (B, 384)), (philox.R, (B, 389))):
        out = torch.full(shape, -3.0, dtype=F16, device=DEV)
        ops().rng_uniform_seqs(out, sd, slots, purpose)
        torch.cuda.synchronize()
        got = out.reshape(B, -1).cpu().numpy()
        n = got.shape[1]
        for b in range(B):
            if b in slots:
                want = philox.uniforms(seeds[b], purpose, n)
                assert np.array_equal(got[b].view(np.uint16), want.view(np.uint16)), (purpose, shape, b)
            else:
                assert bool((got[b] == -3.0).all()), (purpose, shape, b)


# ------------------------------------------------------------------------------------------------ noise
def _check_noise_row(got, seed, step, where):
    """got == fp16(-log(u)) restated in float64, except at fp16 rounding boundaries (1 ulp) -> number of such cases"""
    want, x = philox.noise(seed, step, got.shape[0])
    assert bool(np.isfinite(got).all()) and float(got.min()) > 0, where
    g, w = got.view(np.uint16).astype(np.int64), want.view(np.uint16).astype(np.int64)
    off = np.nonzero(g != w)[0]
    if off.size:
        assert int(np.abs(g[off] - w[off]).max()) == 1, where
        # each one lies within fp32 rounding of an fp16 half-way point: logf's error can only move it across one there
        lo = np.minimum(want[off], got[off]).astype(np.float64)
        hi = np.maximum(want[off], got[off]).astype(np.float64)
        mid = (lo + hi) / 2
        tol = 4 * np.spacing(x[off].astype(np.float32)).astype(np.float64)
        assert bool((np.abs(x[off] - mid) <= tol).all()), where
    return int(off.size)


@pytest.mark.parametrize("V", [32000, 128256])
def test_noise_matches_the_restatement_and_counts_steps(V):
    B = 4
    seeds = SEEDS[2:2 + B]
    sd = _seeds_dev(seeds)
    steps0 = [0, 5, (1 << 32) + 3, 7]                          # the counter word is step mod 2^32
    steps = torch.tensor(steps0, dtype=torch.int64, device=DEV)
    state = _state(B, frozen=(2,))
    noise = torch.full((B, V), -1.0, dtype=F16, device=DEV)
    boundary = 0
    for call in range(3):
        ops().rng_exponential_batch(noise, sd, steps, state)
        torch.cuda.synchronize()
        got = noise.cpu().numpy()
        for b in range(B):
            if b == 2:
                assert bool((got[b] == -1.0).all()), "a frozen row is untouched"
                continue
            boundary += _check_noise_row(got[b], seeds[b], (steps0[b] + call) & 0xFFFFFFFF, (V, call, b))
        assert steps.tolist() == [s + (call + 1) * (b != 2) for b, s in enumerate(steps0)]
    print(f"noise V={V}: {boundary} of {3 * (B - 1) * V} values 1 ulp off the float64 restatement (fp16 boundaries)")


# ------------------------------------------------------------------------------------------------ distributions
def test_sample_level_on_device_rand_draws_q():
    """sq_sample_level_batch with k = 1 on device-filled rand, over many seeds: the exponential race picks token v with
    frequency q_v = softmax(logits / T)."""
    B, S, V, T = 8, 256, 64, 1.0
    g = torch.Generator().manual_seed(3)
    row = (torch.randn(V, generator=g) * 0.8).to(F16)
    logits = row.to(DEV).repeat(B * S, 1).contiguous()
    base = torch.arange(S, dtype=torch.int32, device=DEV)
    step = torch.full((S,), S, dtype=torch.int32, device=DEV)        # node k of sequence b at row b * S + k
    parents = torch.arange(S, dtype=torch.int32, device=DEV)
    first = parents + 1
    nb = torch.ones(S, dtype=torch.int32, device=DEV)
    rand = torch.empty(B, S, V, dtype=F16, device=DEV)
    counts = np.zeros(V, dtype=np.int64)
    for rep in range(8):
        ops().rng_uniform_seqs(rand, _seeds_dev([1000 * rep + b for b in range(B)]), range(B), philox.RAND)
        tokens = torch.full((B, S + 2), -1, dtype=torch.int64, device=DEV)
        ops().sample_level_batch(logits, base, step, rand, S, 1, T, 0, parent_rows=parents, child_first=first,
                                 n_branch=nb, tokens=tokens, state=_state(B))
        torch.cuda.synchronize()
        picked = tokens[:, 1:S + 1].reshape(-1).cpu().numpy()
        assert picked.min() >= 0
        counts += np.bincount(picked, minlength=V)
    q = torch.softmax(row.float() / T, dim=-1).double().numpy()
    p = scipy.stats.chisquare(counts, q / q.sum() * counts.sum()).pvalue
    assert p > 1e-3, p


def test_bonus_draw_on_device_noise_draws_p():
    """argmax(fp16(p / noise)) over many steps of device noise picks v with frequency p_v."""
    B, V, steps_n = 8, 64, 400
    g = torch.Generator().manual_seed(4)
    p = torch.softmax(torch.randn(V, generator=g), dim=-1).to(F16)
    pd = p.to(DEV)
    sd = _seeds_dev([77 + b for b in range(B)])
    steps = torch.zeros(B, dtype=torch.int64, device=DEV)
    noise = torch.empty(B, V, dtype=F16, device=DEV)
    state = _state(B)
    picks = []
    for _ in range(steps_n):
        ops().rng_exponential_batch(noise, sd, steps, state)
        picks.append(torch.argmax(pd / noise, dim=-1))
    counts = np.bincount(torch.cat(picks).cpu().numpy(), minlength=V)
    assert int(counts.sum()) == B * steps_n and steps.tolist() == [steps_n] * B
    pv = p.double().numpy()
    pv = pv / pv.sum() * counts.sum()
    keep = pv >= 5                                               # merge the rare tokens into one bin
    obs = np.append(counts[keep], counts[~keep].sum())
    exp = np.append(pv[keep], pv[~keep].sum())
    assert scipy.stats.chisquare(obs, exp).pvalue > 1e-3


# ------------------------------------------------------------------------------------------------ seeded BatchTree
def _engines(B, Mx=256):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    dcfg, dw = cases.model_weights("draft")
    tcfg, tw = cases.model_weights("target")
    with _env(SQ_DRAFT_ATTN=0, SQ_ATTN_SPLITS=1):
        return (GraphInferenceEngine(Mx, {"config": dcfg, "state_dict": dw}, device=DEV, batch_size=B),
                GraphInferenceEngineTG(Mx, {"config": tcfg, "state_dict": tw}, device=DEV, batch_size=B))


def _check_draws(bt, seeds, slots):
    S, V, M = bt.S, bt.V, bt.M
    r, rand = bt.r.cpu().numpy(), bt.rand.reshape(bt.B, -1).cpu().numpy()
    for b in slots:
        assert np.array_equal(r[b].view(np.uint16), philox.uniforms(seeds[b], philox.R, M).view(np.uint16)), b
        assert np.array_equal(rand[b].view(np.uint16), philox.uniforms(seeds[b], philox.RAND, S * V).view(np.uint16)), b


def test_seeded_batch_tree_draws_only_from_its_seeds():
    """Construction, 2 steps, an admission with the first top_p < 1 (the steady and post graphs are captured again),
    3 more steps: every slot's r and rand, and each step's noise row, equal the restatement for (seed, step), also on
    the steps whose graphs were captured.  torch's CPU and CUDA generator states are unchanged."""
    from sequoia_b200.batch import BatchTree
    gm, B = cases.load_growmap(GM), 3
    seeds = [SEEDS[2], SEEDS[4], 5]
    d, t = _engines(B)
    cpu0, cuda0 = torch.get_rng_state(), torch.cuda.get_rng_state(DEV)
    bt = BatchTree(d, t, [cases.make_prompt(90 + b, 60 + 9 * b) for b in range(B)], gm, temperature=0.6, top_p=1.0,
                   max_length=256, seeds=seeds)
    torch.cuda.synchronize()
    _check_draws(bt, seeds, range(B))
    count = [0] * B
    boundary = 0

    def step():
        nonlocal boundary
        active = [not f for f in bt.frozen]
        bt.construct_grow_map()
        bt.verify()
        got = bt.noise.cpu().numpy()
        for b in range(B):
            if active[b]:
                boundary += _check_noise_row(got[b], seeds[b], count[b], (bt.iter, b))
                count[b] += 1
        assert bt.steps.tolist() == count

    for _ in range(2):
        step()
    assert bt.captures == {"draft": 1, "post": 1, "steady": 1}
    bt.freeze(1)
    seeds[1] = 0xFEEDFACECAFEBEEF
    bt.admit(1, cases.make_prompt(99, 70), temperature=0.8, top_p=0.9, seed=seeds[1])
    count[1] = 0
    torch.cuda.synchronize()
    _check_draws(bt, seeds, range(B))
    for _ in range(3):
        step()
    assert bt.captures == {"draft": 1, "post": 2, "steady": 2}
    assert torch.equal(torch.get_rng_state(), cpu0) and torch.equal(torch.cuda.get_rng_state(DEV), cuda0)
    print(f"seeded BatchTree: {boundary} noise values 1 ulp off the float64 restatement")


def _decode(order, pairs, iters=8):
    """Decode the (prompt, seed) pairs with pair order[b] in slot b; -> per pair: committed tokens per step, and the
    per-step draft / target logits rows of its slot."""
    from sequoia_b200.batch import BatchTree
    gm, B = cases.load_growmap(GM), len(order)
    d, t = _engines(B)
    bt = BatchTree(d, t, [pairs[i][0] for i in order], gm, temperature=0.6, top_p=1.0, max_length=256,
                   seeds=[pairs[i][1] for i in order])
    S = bt.S
    toks = {i: [] for i in order}
    logits = {i: [] for i in order}
    for _ in range(iters):
        bt.construct_grow_map()
        draft_rows = [(bt.row_base.long() + b * bt.row_step.long()) for b in range(B)]
        dl = [bt.draft_logits[draft_rows[b]].clone() for b in range(B)]
        res = bt.verify()
        for b, i in enumerate(order):
            toks[i].append(res[b][0].cpu().clone())
            logits[i].append((dl[b].cpu(), bt.target_logits[b * S:(b + 1) * S].cpu().clone()))
    return toks, logits


def test_slot_permutation_keeps_each_sequence_identical():
    """The same three (prompt, seed) pairs decoded 8 steps at B = 3 with the slots permuted: every GEMM sees the same row
    counts in both runs, so each sequence's committed tokens are identical.  On a difference the message names the first
    step and buffer (draft or target logits) whose rows depend on the slot."""
    pairs = [(cases.make_prompt(120 + i, n), s) for i, (n, s) in enumerate(((70, 11), (95, SEEDS[2]), (82, SEEDS[4])))]
    a_toks, a_log = _decode([0, 1, 2], pairs)
    b_toks, b_log = _decode([2, 0, 1], pairs)
    for i in range(3):
        for it in range(len(a_toks[i])):
            if torch.equal(a_toks[i][it], b_toks[i][it]):
                continue
            where = "tokens only"
            for jt in range(it + 1):
                for name, k in (("draft logits", 0), ("target logits", 1)):
                    x, y = a_log[i][jt][k], b_log[i][jt][k]
                    if not torch.equal(x, y):
                        where = f"{name} of step {jt} (max abs diff {float((x.float() - y.float()).abs().max())})"
                        break
                else:
                    continue
                break
            pytest.fail(f"pair {i} step {it}: committed tokens depend on the slot; first differing buffer: {where}")


def test_seeded_steady_step_is_two_replays_and_one_sync(monkeypatch):
    """A seeded steady step is two graph replays and one host sync; its steady graph has one launch more than an
    unseeded tree's (the noise kernel, in place of torch's exponential_), its draft graph the same launches."""
    from sequoia_b200 import _lib
    from sequoia_b200.batch import BatchTree
    gm = cases.load_growmap(GM)
    launches = {}
    for seeded in (False, True):
        d, t = _engines(2)
        torch.manual_seed(1)
        bt = BatchTree(d, t, [cases.make_prompt(80, 60), cases.make_prompt(81, 70)], gm, temperature=0.6, top_p=1.0,
                       max_length=256, seeds=[3, 4] if seeded else None)
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
        assert bt.replays["draft"] - r0["draft"] == 3 and bt.replays["steady"] - r0["steady"] == 3
        assert len(syncs) == 3, "one host sync per step"
        assert _lib.launch_count() == c0, "a steady step launches only through graph replays"
        launches[seeded] = (bt.graph_launches["draft"], bt.graph_launches["steady"])
        if seeded:
            assert bt.steps.tolist() == [5, 5]
    assert launches[True] == (launches[False][0], launches[False][1] + 1), launches
