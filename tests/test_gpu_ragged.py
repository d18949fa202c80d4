"""Ragged batched forward: a chosen set of the B sequences, each with its own row count (include/sequoia_b200.h, ragged
batches).

Kernel level, B = 8: the ragged embed, RoPE + KV append and tree attention against the _batch launch of each listed
sequence with every other sequence frozen, bit for bit, with parts in shuffled sequence order that mix prefill-like,
first-verify-like and steady-like shapes; attention also against the float64 reference.  Nothing of an unlisted
sequence is touched.  Runner level: forward_ragged against forward(batch=True) per sequence.  BatchTree level: the
constructor and an admission step run the row counts they need, in one forward."""
import contextlib
import os

import pytest
import torch

import cases
from test_gpu_full_batch import _attn_ref_seq
from test_gpu_kernels import _tree_vis

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
F16 = torch.float16
GM128 = "A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"   # config 2: 128 nodes
ST_P, ST_M, ST_FROZEN = 0, 8, 9
SENT = -7.0
B, MC = 8, 1024
REL_TOL = 4e-3              # logits of different GEMM row counts, relative to the row's max |logit| (test_gpu_fp8.py)


def ops():
    from sequoia_b200 import ops as _ops
    return _ops


def lib():
    from sequoia_b200 import _lib
    return _lib


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
    grow = cases.load_growmap(GM128)
    return _Static(grow, DEV), grow["mask"].bool().to(DEV)


# prefix lengths P of the 8 sequences; sequences 1, 4 and 6 are not listed
PS = [1, 77, 140, 200, 33, 300, 64, 40]


def _parts(S):
    """(seq, n, n0, kv_end) in shuffled sequence order: prefill-like (n0 = 1 - P, kv_end = 1), steady-like (n0 = 0,
    n = S, kv_end = S) and first-verify-like (n = P + S - 1, n0 = 1 - P, kv_end = S)."""
    return [(5, PS[5], 1 - PS[5], 1), (2, S, 0, S), (7, PS[7] + S - 1, 1 - PS[7], S), (0, PS[0], 1 - PS[0], 1),
            (3, S, 0, S)]


def _state(frozen=()):
    st = torch.zeros(B, 16, dtype=torch.int32)
    st[:, ST_P] = torch.tensor(PS, dtype=torch.int32)
    st[:, ST_M] = MC
    for b in frozen:
        st[b, ST_FROZEN] = 1
    return st.to(DEV)


def _frozen_copies(state, b):
    """sequence b alone: every other row a frozen copy of b's state row, so their kernels write nothing and read exactly
    the cache range b reads"""
    st = state[b:b + 1].repeat(state.shape[0], 1)
    st[:, ST_FROZEN] = 1
    st[b, ST_FROZEN] = 0
    return st


def _alone(b):
    return _frozen_copies(_state(), b)


def _row0(parts):
    r = [0]
    for p in parts:
        r.append(r[-1] + p[1])
    return r


def _one_launch(fn):
    c0 = lib().launch_count()
    fn()
    torch.cuda.synchronize()
    assert lib().launch_count() - c0 == 1, "a ragged op must be one launch for all parts"


# ------------------------------------------------------------------------------------------------ embed, RoPE + KV append
def test_embed_rows_ragged_b8(tree):
    st, _ = tree
    parts = _parts(st.S)
    row0 = _row0(parts)
    hidden, V = 4096, 32000
    g = torch.Generator(device=DEV).manual_seed(1)
    table = torch.randn(V, hidden, generator=g, device=DEV).to(F16)
    tokens = torch.randint(0, V, (B, MC), generator=g, device=DEV)
    state = _state()
    state0, tokens0 = state.clone(), tokens.clone()
    out = torch.full((row0[-1] + 8, hidden), SENT, dtype=F16, device=DEV)
    _one_launch(lambda: ops().embed_rows_ragged(table, tokens, parts, out, state))
    for j, (b, n, n0, _) in enumerate(parts):
        ref = torch.full((B * n, hidden), SENT, dtype=F16, device=DEV)
        ops().embed_rows_batch(table, tokens, n, ref, _alone(b), n0=n0)
        assert torch.equal(out[row0[j]:row0[j + 1]], ref[b * n:(b + 1) * n]), (j, b)
    assert bool((out[row0[-1]:] == SENT).all()), "rows past the parts were written"
    assert torch.equal(state, state0) and torch.equal(tokens, tokens0)


@pytest.mark.parametrize("H,Hkv,D", [(32, 8, 128), (12, 12, 64)], ids=str)
def test_rope_kv_append_ragged_b8(H, Hkv, D, tree):
    st, _ = tree
    parts = _parts(st.S)
    row0 = _row0(parts)
    L, layer, ld = 2, 1, (H + 2 * Hkv) * D
    g = torch.Generator(device=DEV).manual_seed(H + D)
    qkv0 = torch.randn(row0[-1] + 8, ld, generator=g, device=DEV).to(F16)
    cos = torch.randn(MC, D, generator=g, device=DEV).to(F16)
    sin = torch.randn(MC, D, generator=g, device=DEV).to(F16)
    pos = torch.randint(0, MC, (B, MC), generator=g, device=DEV)
    sto = torch.stack([torch.randperm(MC, device=DEV) for _ in range(B)])
    state = _state()
    state0 = state.clone()
    qkv = qkv0.clone()
    kc = torch.full((L, B, Hkv, MC, D), SENT, dtype=F16, device=DEV)
    vc = torch.full_like(kc, SENT)
    _one_launch(lambda: ops().rope_kv_append_ragged(qkv, H, Hkv, D, cos, sin, pos, sto, parts, kc[layer], vc[layer], MC,
                                                    state))
    listed = set()
    for j, (b, n, n0, _) in enumerate(parts):
        listed.add(b)
        q_ref = torch.zeros(B * n, ld, dtype=F16, device=DEV)
        q_ref[b * n:(b + 1) * n] = qkv0[row0[j]:row0[j + 1]]
        k_ref = torch.full((B, Hkv, MC, D), SENT, dtype=F16, device=DEV)
        v_ref = torch.full_like(k_ref, SENT)
        ops().rope_kv_append_batch(q_ref, H, Hkv, D, cos, sin, pos, sto, n, k_ref, v_ref, MC, _alone(b), n0=n0)
        assert torch.equal(qkv[row0[j]:row0[j + 1]], q_ref[b * n:(b + 1) * n]), (j, b)
        assert torch.equal(kc[layer, b], k_ref[b]) and torch.equal(vc[layer, b], v_ref[b]), (j, b)
    for b in set(range(B)) - listed:
        assert bool((kc[layer, b] == SENT).all()) and bool((vc[layer, b] == SENT).all()), f"unlisted sequence {b}"
    assert torch.equal(qkv[row0[-1]:], qkv0[row0[-1]:]), "rows past the parts were written"
    assert bool((kc[0] == SENT).all()) and bool((vc[0] == SENT).all()), "another layer was written"
    assert torch.equal(state, state0)


# ------------------------------------------------------------------------------------------------ tree attention
def _attn_bufs(H, Hkv, D, rows, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    kc = torch.randn(2, B, Hkv, MC, D, generator=g, device=DEV).to(F16)
    vc = torch.randn(2, B, Hkv, MC, D, generator=g, device=DEV).to(F16)
    qkv = torch.randn(rows + 16, (H + 2 * Hkv) * D, generator=g, device=DEV).to(F16)
    return kc, vc, qkv


def _attn_batch_ref(kc, vc, qkv_rows, b, n, n0, kv_end, H, Hkv, D, Z, st, layer):
    """the _batch launch with sequence b's rows at b*n (the other sequences' rows zero, frozen)"""
    q = torch.zeros(B * n, qkv_rows.shape[1], dtype=F16, device=DEV)
    q[b * n:(b + 1) * n] = qkv_rows
    out = torch.full((B * n, H * D), SENT, dtype=F16, device=DEV)
    with _env(SQ_ATTN_SPLITS=Z):
        plan = ops().AttnPlan(q, B * n, H, Hkv, D, kc, vc, out)
    ops().tree_attn_batch(plan, layer, n, state=_alone(b), n0=n0, kv_end=kv_end, tree_bits=st.tree_bits,
                          tree_words=st.tree_words, tree_size=st.S)
    torch.cuda.synchronize()
    assert plan.info()[1] == Z and plan.error() == 0
    return out[b * n:(b + 1) * n]


@pytest.mark.parametrize("H,Hkv,D", [(12, 12, 64), (32, 32, 128), (32, 8, 128)], ids=str)
def test_tree_attn_ragged_b8(H, Hkv, D, tree):
    """Each part's rows bit-identical to the _batch launch for its sequence at the same forced split count, and within the
    float64 reference's per-element bound; rows past the parts keep their sentinel; the caches are only read."""
    st, tmask = tree
    parts = _parts(st.S)
    row0 = _row0(parts)
    layer = 1
    kc, vc, qkv = _attn_bufs(H, Hkv, D, row0[-1], seed=H * Hkv + D)
    kc0, vc0 = kc.clone(), vc.clone()
    out = torch.full((row0[-1] + 16, H * D), SENT, dtype=F16, device=DEV)
    state = _state()
    kw = dict(state=state, tree_bits=st.tree_bits, tree_words=st.tree_words, tree_size=st.S)
    refs = []
    for j, (b, n, n0, kv_end) in enumerate(parts):
        P = PS[b]
        kv_len = P - 1 + kv_end
        vis = _tree_vis(torch.arange(P - 1 + n0, P - 1 + n0 + n), kv_len, P, tmask)
        refs.append(_attn_ref_seq(qkv[row0[j]:row0[j + 1], :H * D].view(n, H, D), kc[layer, b, :, :kv_len],
                                  vc[layer, b, :, :kv_len], vis, H, Hkv, D))
    for Z in (1, 2, 4, 8):
        with _env(SQ_ATTN_SPLITS=Z):
            plan = ops().AttnPlan(qkv, row0[-1] + 16, H, Hkv, D, kc, vc, out)
        out.fill_(SENT)
        _one_launch(lambda: ops().tree_attn_ragged(plan, layer, parts, **kw))
        assert plan.info()[1] == Z and plan.error() == 0, (Z, plan.info())
        assert bool((out[row0[-1]:] == SENT).all()), "rows past the parts were written"
        for j, (b, n, n0, kv_end) in enumerate(parts):
            got = out[row0[j]:row0[j + 1]]
            want = _attn_batch_ref(kc, vc, qkv[row0[j]:row0[j + 1]], b, n, n0, kv_end, H, Hkv, D, Z, st, layer)
            assert torch.equal(got, want), f"Z={Z} part {j} (sequence {b}) != its _batch launch"
            ref, tol = refs[j]
            nbad = int(((got.view(n, H, D).double() - ref).abs() > tol).sum())
            assert nbad == 0, f"Z={Z} part {j}: {nbad} elements outside the float64 bound"
    assert torch.equal(kc, kc0) and torch.equal(vc, vc0), "the attention wrote its caches"


def test_tree_attn_ragged_swapped_seqs_fail_the_comparison(tree):
    """Negative control: two parts with their seq fields swapped must not match the _batch launches of their sequences."""
    st, _ = tree
    H, Hkv, D, Z, layer = 32, 8, 128, 2, 1
    parts = [(2, st.S, 0, st.S), (3, st.S, 0, st.S)]
    swapped = [(3, st.S, 0, st.S), (2, st.S, 0, st.S)]
    row0 = _row0(parts)
    kc, vc, qkv = _attn_bufs(H, Hkv, D, row0[-1], seed=9)
    out = torch.full((row0[-1] + 16, H * D), SENT, dtype=F16, device=DEV)
    with _env(SQ_ATTN_SPLITS=Z):
        plan = ops().AttnPlan(qkv, row0[-1] + 16, H, Hkv, D, kc, vc, out)
    ops().tree_attn_ragged(plan, layer, swapped, state=_state(), tree_bits=st.tree_bits, tree_words=st.tree_words,
                           tree_size=st.S)
    torch.cuda.synchronize()
    for j, (b, n, n0, kv_end) in enumerate(parts):
        want = _attn_batch_ref(kc, vc, qkv[row0[j]:row0[j + 1]], b, n, n0, kv_end, H, Hkv, D, Z, st, layer)
        assert not torch.equal(out[row0[j]:row0[j + 1]], want), j


# ------------------------------------------------------------------------------------------------ refusals
def test_bad_part_lists_are_refused_before_any_launch(tree):
    st, _ = tree
    S, H, Hkv, D = st.S, 4, 4, 64
    rows = 64
    table = torch.zeros(100, 256, dtype=F16, device=DEV)
    tokens = torch.zeros(B, MC, dtype=torch.int64, device=DEV)
    hid = torch.zeros(rows, 256, dtype=F16, device=DEV)
    qkv = torch.zeros(rows, (H + 2 * Hkv) * D, dtype=F16, device=DEV)
    cos = torch.zeros(MC, D, dtype=F16, device=DEV)
    kc = torch.zeros(1, B, Hkv, MC, D, dtype=F16, device=DEV)
    out = torch.zeros(rows, H * D, dtype=F16, device=DEV)
    plan = ops().AttnPlan(qkv, rows, H, Hkv, D, kc, kc.clone(), out)
    state = _state()
    ok = (0, 4, 0, 4)
    bad = {"no parts": [], "nine parts": [ok] * 9, "seq = B": [(B, 4, 0, 4)], "seq < 0": [(-1, 4, 0, 4)],
           "seq twice": [ok, (0, 4, 0, 4)], "n = 0": [(1, 0, 0, 4)], "rows > n_max": [(0, 40, 0, 4), (1, 25, 0, 4)]}
    calls = {
        "embed": lambda p: ops().embed_rows_ragged(table, tokens, p, hid, state),
        "rope": lambda p: ops().rope_kv_append_ragged(qkv, H, Hkv, D, cos, cos, tokens, tokens, p, kc[0], kc[0], MC,
                                                      state),
        "attn": lambda p: ops().tree_attn_ragged(plan, 0, p, state=state, tree_bits=st.tree_bits,
                                                 tree_words=st.tree_words, tree_size=S),
    }
    torch.cuda.synchronize()
    for what, p in bad.items():
        for name, fn in calls.items():
            c0 = lib().launch_count()
            with pytest.raises(lib().SequoiaLibError):
                fn(p)
            assert lib().launch_count() == c0, f"{name}, {what}: refused after a launch"
    c0 = lib().launch_count()
    with pytest.raises(lib().SequoiaLibError):
        ops().tree_attn_ragged(plan, 0, [ok], state=state, tree_bits=st.tree_bits, tree_words=33, tree_size=S)
    assert lib().launch_count() == c0


# ------------------------------------------------------------------------------------------------ LlamaRunner
def _runner(Bn, M, weight_format="fp16"):
    from sequoia_b200.model import LlamaRunner
    cfg, w = cases.model_weights("target")
    return LlamaRunner({"config": cfg, "state_dict": w}, M, device=DEV, batch_size=Bn, weight_format=weight_format)


def _runner_inputs(Bn, M, Ps, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    tokens = torch.randint(0, cases.V, (Bn, M), generator=g, device=DEV)
    pos = torch.stack([torch.arange(M, device=DEV)] * Bn).contiguous()
    sto = torch.stack([torch.arange(M, device=DEV)] * Bn).contiguous()
    st = torch.zeros(Bn, 16, dtype=torch.int32)
    st[:, ST_P] = torch.tensor(Ps, dtype=torch.int32)
    st[:, ST_M] = M
    return tokens, pos, sto, st.to(DEV)


def _fill_caches(r, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    for c in (r.k_cache, r.v_cache):
        c.copy_(torch.randn(c.shape, generator=g, device=DEV).to(F16))


@pytest.mark.parametrize("weight_format", ["fp16", "fp8"])
def test_forward_ragged_vs_batched_forward(weight_format, tree):
    """B = 4, parts for sequences 3, 0 and 2 (a prefill, a first verify, a steady tree): logits within the repository's
    tolerance for different GEMM row counts of forward(batch=True) for each sequence with the others frozen, and
    sequence 1's KV planes byte-identical."""
    st, _ = tree
    S, M, Bn = st.S, 640, 4
    Ps = [100, 50, 180, 230]
    r = _runner(Bn, M, weight_format)
    tokens, pos, sto, state = _runner_inputs(Bn, M, Ps, seed=3)
    _fill_caches(r, 4)
    kv0 = [r.k_cache.clone(), r.v_cache.clone()]
    mk = dict(tree_bits=st.tree_bits, tree_words=st.tree_words, tree_size=S)
    geo = [(3, Ps[3], 1 - Ps[3], 1, 1), (0, Ps[0] + S - 1, 1 - Ps[0], S, S), (2, S, 0, S, S)]
    outs = [torch.full((m, cases.V), SENT, dtype=F16, device=DEV) for *_, m in geo]
    r.forward_ragged([g + (o,) for g, o in zip(geo, outs)], tokens, pos, sto, state=state, **mk)
    torch.cuda.synchronize()
    assert bool((r.k_cache[:, 1] == kv0[0][:, 1]).all()) and bool((r.v_cache[:, 1] == kv0[1][:, 1]).all()), \
        "the unlisted sequence's KV planes changed"
    for (b, n, n0, kv_end, m), got in zip(geo, outs):
        r.k_cache.copy_(kv0[0])
        r.v_cache.copy_(kv0[1])
        alone = _frozen_copies(state, b)
        want = torch.empty_like(got)
        r.forward(n, tokens, pos, sto, state=alone, n0=n0, kv_end=kv_end, batch=True, logits_from=b * n + n - m,
                  logits_to=b * n + n, logits_out=want, **mk)
        torch.cuda.synchronize()
        rel = ((got.float() - want.float()).abs() / want.float().abs().amax(-1, keepdim=True)).max().item()
        assert rel < REL_TOL, (weight_format, b, rel)
    assert r.gemm_err.tolist() == [0, 0, 0, 0]


def test_forward_ragged_one_part_at_b1_is_bit_identical(tree):
    st, _ = tree
    S, M = st.S, 512
    r = _runner(1, M)
    tokens, pos, sto, state = _runner_inputs(1, M, [150], seed=5)
    mk = dict(tree_bits=st.tree_bits, tree_words=st.tree_words, tree_size=S)
    n, n0 = 150 + S - 1, 1 - 150
    got, want = (torch.empty(S, cases.V, dtype=F16, device=DEV) for _ in range(2))
    _fill_caches(r, 6)
    r.forward_ragged([(0, n, n0, S, S, got)], tokens, pos, sto, state=state, **mk)
    kv = [r.k_cache.clone(), r.v_cache.clone()]
    _fill_caches(r, 6)
    r.forward(n, tokens, pos, sto, state=state, n0=n0, kv_end=S, batch=True, logits_from=n - S, logits_to=n,
              logits_out=want, **mk)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert torch.equal(kv[0], r.k_cache) and torch.equal(kv[1], r.v_cache)


# ------------------------------------------------------------------------------------------------ BatchTree
PROMPT_LENS8 = (20, 130, 64, 97, 33, 120, 75, 48)


def _bt_engines(Bn, Mx):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    dcfg, dw = cases.model_weights("draft")
    tcfg, tw = cases.model_weights("target")
    with _env(SQ_DRAFT_ATTN=0, SQ_ATTN_SPLITS=1):
        return (GraphInferenceEngine(Mx, {"config": dcfg, "state_dict": dw}, device=DEV, batch_size=Bn),
                GraphInferenceEngineTG(Mx, {"config": tcfg, "state_dict": tw}, device=DEV, batch_size=Bn))


def _record_rows(monkeypatch, runner):
    """the activation rows of every layer stack `runner` runs"""
    from sequoia_b200.model import LlamaRunner
    rows, real = [], LlamaRunner._layers

    def rec(self, n, attend):
        if self is runner:
            rows.append(n)
        return real(self, n, attend)
    monkeypatch.setattr(LlamaRunner, "_layers", rec)
    return rows


def test_batch_tree_runs_the_rows_it_needs(monkeypatch):
    """B = 8: the constructor's draft prefill is one forward of sum(P_b) rows and the first verify one target forward of
    sum(P_b + S - 1) rows.  An admission step runs B*S steady rows and P + S - 1 admitted rows in the target, with one
    host sync."""
    from sequoia_b200.batch import BatchTree
    gm, Mx = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256
    S = gm["size"]
    d, t = _bt_engines(B, Mx)
    prompts = [cases.make_prompt(190 + i, n) for i, n in enumerate(PROMPT_LENS8)]
    drows = _record_rows(monkeypatch, d.engine.runner)
    trows = _record_rows(monkeypatch, t.engine.runner)
    torch.manual_seed(3)
    bt = BatchTree(d, t, prompts, gm, temperature=0.6, top_p=1.0, max_length=Mx)
    assert drows == [sum(PROMPT_LENS8)]
    bt.construct_grow_map()
    bt.verify()
    assert trows == [sum(P + S - 1 for P in PROMPT_LENS8)]
    bt.construct_grow_map()
    bt.verify()
    bt.freeze(5)
    new = cases.make_prompt(199, 70)
    syncs = []
    real_sync = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: syncs.append(1))
    del drows[:], trows[:]
    bt.admit(5, new)
    assert drows == [len(new)]
    bt.construct_grow_map()
    bt.verify()
    assert len(syncs) == 1, "an admission step has one host sync"
    assert trows == [B * S, len(new) + S - 1]


def test_two_admissions_share_one_ragged_forward(monkeypatch):
    """B = 4: slots 1 and 3 are frozen after step 2 and both admitted at step 3.  Their first verifies run in one target
    forward; both decode, on at least 95% of the committed positions, like a fresh BatchTree on their two prompts with the
    same draws; slots 0 and 2 match a run without the admissions bit for bit."""
    from sequoia_b200.batch import BatchTree
    gm, Mx, iters, at, Bn = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256, 8, 3, 4
    S, V = gm["size"], cases.V
    prompts = [cases.make_prompt(200 + i, n) for i, n in enumerate((100, 64, 120, 90))]
    new = [cases.make_prompt(210, 80), cases.make_prompt(211, 45)]
    noise = torch.empty(iters, Bn, V, dtype=F16).exponential_(1.0, generator=torch.Generator().manual_seed(12)).to(DEV)

    def run(admit):
        d, t = _bt_engines(Bn, Mx)
        trows = _record_rows(monkeypatch, t.engine.runner)
        torch.manual_seed(4)
        bt = BatchTree(d, t, prompts, gm, temperature=0.6, top_p=1.0, max_length=Mx)
        bt.external_noise = noise
        steps = []
        for it in range(iters):
            if it == at and admit:
                torch.manual_seed(9)
                bt.admit(1, new[0], temperature=0.8, top_p=0.9)
                bt.admit(3, new[1], temperature=0.8, top_p=0.9)
                del trows[:]
            bt.construct_grow_map()
            steps.append([(v.clone(), a, term) for v, a, term in bt.verify()])
            if it == at and admit:
                assert trows == [Bn * S, sum(len(p) + S - 1 for p in new)], trows
            if it == at - 1:
                bt.freeze(1)
                bt.freeze(3)
        monkeypatch.undo()
        return steps

    with_adm = run(True)
    without = run(False)
    for it in range(iters):
        for b in (0, 2):
            (v, a, term), (v0, a0, term0) = with_adm[it][b], without[it][b]
            assert (a, term) == (a0, term0) and torch.equal(v, v0), (it, b)
    d2, t2 = _bt_engines(2, Mx)
    torch.manual_seed(9)
    fresh = BatchTree(d2, t2, new, gm, temperature=0.8, top_p=0.9, max_length=Mx)
    fresh.external_noise = noise[at:, [1, 3]].contiguous()
    for _ in range(iters - at):
        fresh.construct_grow_map()
        res = fresh.verify()
    for slot, k in ((1, 0), (3, 1)):
        got, want = with_adm[-1][slot][0].cpu(), res[k][0].cpu()
        assert torch.equal(got[:len(new[k])], new[k].cpu()) and len(got) > len(new[k]), slot
        n = min(len(got), len(want))
        same = int((got[:n] == want[:n]).sum()) - len(new[k])
        total = max(len(got), len(want)) - len(new[k])
        assert total > 0 and same >= 0.95 * total, (slot, same, total)
