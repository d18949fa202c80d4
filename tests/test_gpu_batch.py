"""Batched entry points (one launch for B sequences that share a growmap) against B launches of the single-sequence entry
points, bit for bit.  The sequences sit at different prefix lengths P; every buffer that a batched launch must not touch
(other sequences' rows, rows past the batch, other layers, a frozen sequence's tokens / state / KV) holds a sentinel or
a copy that is checked afterwards."""
import contextlib
import os

import pytest
import torch

import cases

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
F16 = torch.float16
GM = "A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"   # the 128-node config-2 tree
M = 640
V = cases.V
ST_P, ST_N_NEW, ST_P_OLD, ST_M, ST_FROZEN = 0, 3, 4, 8, 9
# kv_len = P - 1 + S of each sequence's full-tree verify: 128 j - 1, 128 j, 128 j + 1 (one KV tile is 128 keys) and M
KV_LENS = {2: [255, M], 3: [255, 256, 257], 4: [383, 384, 385, M]}
SENT = -7.0


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
    gm = cases.load_growmap(GM)
    return _Static(gm, DEV)


def _state(B, S, frozen=()):
    st = torch.zeros(B, 16, dtype=torch.int32)
    for b, kv in enumerate(KV_LENS[B]):
        st[b, ST_P] = kv + 1 - S
        st[b, ST_M] = M
    for b in frozen:
        st[b, ST_FROZEN] = 1
    return st.to(DEV)


def _one_launch(fn):
    c0 = lib().launch_count()
    fn()
    torch.cuda.synchronize()
    assert lib().launch_count() - c0 == 1, "a batched op must be one launch for all sequences"


B_VALUES = [2, 3, 4]


# ------------------------------------------------------------------------------------------------ embed, RoPE + KV append
@pytest.mark.parametrize("B", B_VALUES)
def test_embed_rows_batch(B, tree):
    S, h, n0, n = tree.S, 256, 1, 40
    g = torch.Generator(device=DEV).manual_seed(B)
    table = torch.randn(V, h, generator=g, device=DEV).to(F16)
    tokens = torch.randint(0, V, (B, M), generator=g, device=DEV)
    for frozen in ((), (1,)):
        state = _state(B, S, frozen)
        out = torch.full((B * n + 8, h), SENT, dtype=F16, device=DEV)
        _one_launch(lambda: ops().embed_rows_batch(table, tokens, n, out, state, n0=n0))
        for b in range(B):
            ref = torch.full((n, h), SENT, dtype=F16, device=DEV)
            if b not in frozen:
                ops().embed_rows(table, tokens[b], n, ref, state=state[b], n0=n0)
            assert torch.equal(out[b * n:(b + 1) * n], ref), (B, b, frozen)
        assert bool((out[B * n:] == SENT).all())


@pytest.mark.parametrize("B", B_VALUES)
@pytest.mark.parametrize("H,Hkv,D", [(8, 2, 128), (4, 4, 64)])
def test_rope_kv_append_batch(B, H, Hkv, D, tree):
    S, L, layer, n0, n = tree.S, 2, 1, 0, tree.S
    g = torch.Generator(device=DEV).manual_seed(10 * B + D)
    ld = (H + 2 * Hkv) * D
    qkv0 = torch.randn(B * n + 8, ld, generator=g, device=DEV).to(F16)
    cos = torch.randn(M, D, generator=g, device=DEV).to(F16)
    sin = torch.randn(M, D, generator=g, device=DEV).to(F16)
    pos = torch.randint(0, M, (B, M), generator=g, device=DEV)
    sto = torch.stack([torch.randperm(M, device=DEV) for _ in range(B)])
    for frozen in ((), (B - 1,)):
        state = _state(B, S, frozen)
        qkv = qkv0.clone()
        kc = torch.full((L, B, Hkv, M, D), SENT, dtype=F16, device=DEV)
        vc = torch.full_like(kc, SENT)
        _one_launch(lambda: ops().rope_kv_append_batch(qkv, H, Hkv, D, cos, sin, pos, sto, n, kc[layer], vc[layer], M,
                                                       state, n0=n0))
        for b in range(B):
            q_ref = qkv0[b * n:(b + 1) * n].clone()
            k_ref = torch.full((Hkv, M, D), SENT, dtype=F16, device=DEV)
            v_ref = torch.full_like(k_ref, SENT)
            if b not in frozen:
                ops().rope_kv_append(q_ref, H, Hkv, D, cos, sin, pos[b], sto[b], n, k_ref, v_ref, M, state=state[b], n0=n0)
            assert torch.equal(qkv[b * n:(b + 1) * n], q_ref), (B, b, frozen)
            assert torch.equal(kc[layer, b], k_ref) and torch.equal(vc[layer, b], v_ref), (B, b, frozen)
        assert torch.equal(qkv[B * n:], qkv0[B * n:])
        assert bool((kc[0] == SENT).all()) and bool((vc[0] == SENT).all())


# ------------------------------------------------------------------------------------------------ tree attention
def _attn_case(B, H, Hkv, D, tree, Z, seed):
    from sequoia_b200.tree import pack_tree_mask
    S, L = tree.S, 2
    n = S
    g = torch.Generator(device=DEV).manual_seed(seed)
    kc = torch.randn(L, B, Hkv, M, D, generator=g, device=DEV).to(F16)
    vc = torch.randn(L, B, Hkv, M, D, generator=g, device=DEV).to(F16)
    ld = (H + 2 * Hkv) * D
    qkv = torch.randn(B * n + 16, ld, generator=g, device=DEV).to(F16)
    out = torch.full((B * n + 16, H * D), SENT, dtype=F16, device=DEV)
    with _env(SQ_ATTN_SPLITS=Z):
        plan = ops().AttnPlan(qkv, B * n + 16, H, Hkv, D, kc, vc, out)
    return dict(kc=kc, vc=vc, qkv=qkv, out=out, plan=plan, n=n, L=L)


def _attn_single(c, b, H, Hkv, D, tree, Z, state_row, layer):
    n = c["n"]
    kc = c["kc"][:, b:b + 1].contiguous()
    vc = c["vc"][:, b:b + 1].contiguous()
    qkv = c["qkv"][b * n:(b + 1) * n].clone()
    out = torch.full((n, H * D), SENT, dtype=F16, device=DEV)
    with _env(SQ_ATTN_SPLITS=Z):
        plan = ops().AttnPlan(qkv, n, H, Hkv, D, kc, vc, out)
    ops().tree_attn(plan, layer, n, state=state_row, n0=0, kv_end=tree.S, tree_bits=tree.tree_bits,
                    tree_words=tree.tree_words, tree_size=tree.S)
    torch.cuda.synchronize()
    assert plan.info()[1] == min(Z, -(-M // 128))
    return out


@pytest.mark.parametrize("B", B_VALUES)
@pytest.mark.parametrize("Z", [1, 3])
@pytest.mark.parametrize("H,Hkv,D", [(8, 2, 128), (4, 4, 64)])
def test_tree_attn_batch(B, Z, H, Hkv, D, tree):
    layer = 1
    c = _attn_case(B, H, Hkv, D, tree, Z, seed=100 * B + Z + D)
    state = _state(B, tree.S)
    kc0, vc0 = c["kc"].clone(), c["vc"].clone()
    _one_launch(lambda: ops().tree_attn_batch(c["plan"], layer, c["n"], state=state, n0=0, kv_end=tree.S,
                                              tree_bits=tree.tree_bits, tree_words=tree.tree_words, tree_size=tree.S))
    assert c["plan"].info()[1] == min(Z, -(-M // 128))
    assert c["plan"].error() == 0
    n = c["n"]
    for b in range(B):
        ref = _attn_single(c, b, H, Hkv, D, tree, Z, state[b], layer)
        assert torch.equal(c["out"][b * n:(b + 1) * n], ref), (B, Z, b)
    assert bool((c["out"][B * n:] == SENT).all())
    assert torch.equal(c["kc"], kc0) and torch.equal(c["vc"], vc0)


def test_tree_attn_batch_swapped_states_fail_the_comparison(tree):
    """Negative control: with two sequences' state rows swapped, the batched outputs must differ from the single launches."""
    B, H, Hkv, D, Z, layer = 2, 8, 2, 128, 3, 1
    c = _attn_case(B, H, Hkv, D, tree, Z, seed=7)
    state = _state(B, tree.S)
    swapped = state[[1, 0]].contiguous()
    ops().tree_attn_batch(c["plan"], layer, c["n"], state=swapped, n0=0, kv_end=tree.S, tree_bits=tree.tree_bits,
                          tree_words=tree.tree_words, tree_size=tree.S)
    torch.cuda.synchronize()
    n = c["n"]
    for b in range(B):
        ref = _attn_single(c, b, H, Hkv, D, tree, Z, state[b], layer)
        assert not torch.equal(c["out"][b * n:(b + 1) * n], ref), b


# ------------------------------------------------------------------------------------------------ KV gather
@pytest.mark.parametrize("B", B_VALUES)
def test_kv_gather_batch(B, tree):
    S, L, Hkv, D = tree.S, 2, 2, 128
    md = tree.max_depth
    g = torch.Generator(device=DEV).manual_seed(B + 50)
    kc0 = torch.randn(L, B, Hkv, M, D, generator=g, device=DEV).to(F16)
    vc0 = torch.randn(L, B, Hkv, M, D, generator=g, device=DEV).to(F16)
    for frozen in ((), (0,)):
        state = _state(B, S, frozen)
        idx = torch.full((B, S), -1, dtype=torch.int32, device=DEV)
        for b in range(B):
            P = int(state[b, ST_P])
            nn_ = (b * 3 + 1) % (md + 1)                   # accepted nodes per sequence, 0 included
            sel = torch.sort(torch.randperm(S - 1, generator=torch.Generator().manual_seed(b))[:nn_])[0] + P
            idx[b, :nn_] = sel.to(torch.int32).to(DEV)
            state[b, ST_N_NEW] = nn_
            state[b, ST_P_OLD] = P
        kc, vc = kc0.clone(), vc0.clone()
        _one_launch(lambda: ops().kv_gather_batch(kc, vc, idx, state, md))
        for b in range(B):
            k_ref, v_ref = kc0[:, b:b + 1].contiguous(), vc0[:, b:b + 1].contiguous()
            if b not in frozen:
                ops().kv_gather(k_ref, v_ref, idx[b], 0, 0, state=state[b], max_n=md)
            assert torch.equal(kc[:, b:b + 1], k_ref) and torch.equal(vc[:, b:b + 1], v_ref), (B, b, frozen)


# ------------------------------------------------------------------------------------------------ draft sampling
def _draft_layout(tree, B, per_seq):
    """Pack per-sequence (S, V) node-indexed draft logits into the level-block layout; -> (buffer, row_base, row_step)."""
    levels = [(0, 1)] + [(lv["n0"], lv["tb"]) for lv in tree.levels]
    base, step = ops().draft_row_tables(levels, tree.S, B, DEV)
    buf = torch.full((B * tree.S + 4, V), SENT, dtype=F16, device=DEV)
    for b in range(B):
        rows = base.long() + b * step.long()
        buf[rows] = per_seq[b]
    return buf, base, step


@pytest.mark.parametrize("B", B_VALUES)
@pytest.mark.parametrize("mode", [0, 1])
def test_sample_level_batch(B, mode, tree):
    S = tree.S
    g = torch.Generator(device=DEV).manual_seed(B * 7 + mode)
    per_seq = [(torch.randn(S, V, generator=g, device=DEV) * 2).to(F16) for _ in range(B)]
    rand = torch.rand(B, S, V, generator=g, device=DEV).to(F16) if mode == 0 else None
    buf, base, step = _draft_layout(tree, B, per_seq)
    for frozen in ((), (B - 1,)):
        state = _state(B, S, frozen)
        tokens = torch.full((B, M), -5, dtype=torch.int64, device=DEV)
        ref = tokens.clone()
        for lv in tree.levels:
            _one_launch(lambda: ops().sample_level_batch(
                buf, base, step, rand, lv["n_parents"], lv["k"], 0.6, mode, parent_rows=lv["parents"],
                child_first=lv["first"], n_branch=lv["nb"], tokens=tokens, state=state))
            for b in range(B):
                if b not in frozen:
                    ops().sample_level(per_seq[b], rand[b] if rand is not None else None, lv["n_parents"], lv["k"], 0.6,
                                       mode, parent_rows=lv["parents"], child_first=lv["first"], n_branch=lv["nb"],
                                       tokens=ref[b], state=state[b])
        torch.cuda.synchronize()
        assert torch.equal(tokens, ref), (B, mode, frozen)
        for b in range(B):
            P = int(state[b, ST_P])
            written = tokens[b, P:P + S - 1]
            assert bool((written == -5).all()) if b in frozen else bool((written >= 0).all())


# ------------------------------------------------------------------------------------------------ verification walks
def _walk_inputs(tree, B, seed):
    S = tree.S
    g = torch.Generator(device=DEV).manual_seed(seed)
    per_seq, target = [], []
    for b in range(B):
        d = (torch.randn(S, V, generator=g, device=DEV) * 0.5).to(F16)
        eps = [0.0, 0.3, 3.0, 0.0][b]                  # equal rows accept deep paths; noisy rows reject early
        per_seq.append(d)
        target.append((d.float() + eps * torch.randn(S, V, generator=g, device=DEV)).to(F16))
    tokens = torch.randint(3, V, (B, M), generator=g, device=DEV)
    pos = torch.randint(0, M, (B, M), generator=g, device=DEV)
    r = torch.rand(B, M, generator=g, device=DEV).to(F16)
    noise = torch.empty(B, V, device=DEV).exponential_(1.0, generator=g).to(F16)
    return per_seq, torch.cat(target), tokens, pos, r, noise


@pytest.mark.parametrize("B", B_VALUES)
def test_accept_stochastic_batch(B, tree):
    S = tree.S
    per_seq, target, tokens0, pos0, r, noise = _walk_inputs(tree, B, seed=B + 200)
    buf, base, step = _draft_layout(tree, B, per_seq)
    for frozen in ((), (1,)):
        state = _state(B, S, frozen)
        st0 = state.clone()
        tokens, pos = tokens0.clone(), pos0.clone()
        acc = torch.full((B, S), -1, dtype=torch.int32, device=DEV)
        _one_launch(lambda: ops().accept_stochastic_batch(target, buf, base, step, r, noise, tree.succ_off, tree.succ,
                                                          tree.depth, S, 0.6, tokens, pos, acc, state, M))
        deepest = 0
        for b in range(B):
            t_ref, p_ref, a_ref, s_ref = tokens0[b].clone(), pos0[b].clone(), torch.full((S,), -1, dtype=torch.int32,
                                                                                         device=DEV), st0[b].clone()
            if b not in frozen:
                ops().accept_stochastic(target[b * S:(b + 1) * S], per_seq[b], r[b], noise[b], tree.succ_off, tree.succ,
                                        tree.depth, S, 0.6, t_ref, p_ref, a_ref, s_ref, M)
            torch.cuda.synchronize()
            assert torch.equal(tokens[b], t_ref) and torch.equal(pos[b], p_ref), (B, b, frozen)
            assert torch.equal(acc[b], a_ref) and torch.equal(state[b], s_ref), (B, b, frozen)
            deepest = max(deepest, int(state[b, ST_N_NEW]))
        assert deepest >= 3, "the equal-row sequence should accept a path of several nodes"


@pytest.mark.parametrize("B", B_VALUES)
def test_accept_greedy_batch(B, tree):
    S = tree.S
    _, _, tokens0, pos0, _, _ = _walk_inputs(tree, B, seed=B + 300)
    g = torch.Generator(device=DEV).manual_seed(B)
    target_token = torch.randint(3, V, (B * S,), generator=g, device=DEV)
    succ_off, succ = tree.succ_off.cpu(), tree.succ.cpu()
    st_host = _state(B, S).cpu()
    for b in range(0, B, 2):                           # even sequences: the target agrees with the first child everywhere
        P = int(st_host[b, ST_P])
        for k in range(S):
            c0, c1 = int(succ_off[k]), int(succ_off[k + 1])
            if c1 > c0:
                target_token[b * S + k] = tokens0[b, P - 1 + int(succ[c0])]
    for frozen in ((), (0,)):
        state = _state(B, S, frozen)
        st0 = state.clone()
        tokens, pos = tokens0.clone(), pos0.clone()
        acc = torch.full((B, S), -1, dtype=torch.int32, device=DEV)
        _one_launch(lambda: ops().accept_greedy_batch(target_token, tree.succ_off, tree.succ, tree.depth, S, tokens, pos,
                                                      acc, state, M))
        for b in range(B):
            t_ref, p_ref, s_ref = tokens0[b].clone(), pos0[b].clone(), st0[b].clone()
            a_ref = torch.full((S,), -1, dtype=torch.int32, device=DEV)
            if b not in frozen:
                ops().accept_greedy(target_token[b * S:(b + 1) * S], tree.succ_off, tree.succ, tree.depth, S, t_ref, p_ref,
                                    a_ref, s_ref, M)
            torch.cuda.synchronize()
            assert torch.equal(tokens[b], t_ref) and torch.equal(pos[b], p_ref), (B, b, frozen)
            assert torch.equal(acc[b], a_ref) and torch.equal(state[b], s_ref), (B, b, frozen)
        if not frozen:
            k, path = 0, 0
            while int(succ_off[k + 1]) > int(succ_off[k]):
                k, path = int(succ[int(succ_off[k])]), path + 1
            assert int(state[0, ST_N_NEW]) == path, "sequence 0 should accept its first-child path down to a leaf"


# ------------------------------------------------------------------------------------------------ BatchTree end to end
def _bt_engines(dkey, tkey, Mx, B):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    dcfg, dw = cases.model_weights(dkey)
    tcfg, tw = cases.model_weights(tkey)
    return (GraphInferenceEngine(Mx, {"config": dcfg, "state_dict": dw}, device=DEV, batch_size=B),
            GraphInferenceEngineTG(Mx, {"config": tcfg, "state_dict": tw}, device=DEV, batch_size=B))


@pytest.mark.parametrize("policy", ["spec", "greedy"])
def test_batch_tree_b1_is_bit_identical_to_the_single_tree(policy):
    """B = 1: BatchTree and SpecTree / GreedyTree on the same engines, seeds and bonus noise, 8 steps.  The draft attention
    phase is off in both, and the KV split count is forced to 1 so that the first verify (stateless in the single tree,
    tree-relative in the batch) launches the same attention."""
    from sequoia_b200.batch import BatchTree
    from sequoia_b200.tree import GreedyTree, SpecTree, clear_runtimes
    gm, Mx, iters = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256, 8
    prompt = cases.make_prompt(25, 100)
    noise = torch.empty(iters, V, dtype=F16).exponential_(1.0, generator=torch.Generator().manual_seed(5)).to(DEV)
    with _env(SQ_DRAFT_ATTN=0, SQ_ATTN_SPLITS=1):
        draft, target = _bt_engines("draft", "target", Mx, 1)
    cls = SpecTree if policy == "spec" else GreedyTree
    torch.manual_seed(17)
    single = cls(draft, target, prompt.to(DEV), temperature=0.6, top_p=1.0, max_length=Mx, max_target_seq=Mx,
                 device=DEV, vocab_size=V, grow_map=gm)
    single.rt.external_noise = noise if policy == "spec" else None
    ref = []
    for _ in range(iters):
        single.construct_grow_map()
        v, a, _, term = single.verify()
        ref.append((v.clone(), a, term, [t.clone() for e in (draft, target) for t in (e.engine.kv_cache.k_cache,)]))
        if term:
            break
    single.rt.external_noise = None
    clear_runtimes()
    torch.manual_seed(17)
    bt = BatchTree(draft, target, [prompt], gm, policy=policy, temperature=0.6, top_p=1.0, max_length=Mx)
    bt.external_noise = noise.view(iters, 1, V)
    for it, (v_ref, a_ref, t_ref, kv_ref) in enumerate(ref):
        bt.construct_grow_map()
        (v, a, term), = bt.verify()
        assert (a, term) == (a_ref, t_ref) and torch.equal(v, v_ref), (policy, it)
        for got, want in zip([e.engine.kv_cache.k_cache for e in (draft, target)], kv_ref):
            assert torch.equal(got[..., :a, :], want[..., :a, :]), (policy, it)


@pytest.mark.parametrize("policy", ["spec", "greedy"])
def test_batch_tree_three_prompts_lock_step(policy):
    """Three prompts of different lengths decoded together; each sequence against a lone single-sequence tree on that
    prompt (same random draws).  The batch's GEMMs run on 3x the rows, so cuBLAS may round differently: at least 95% of
    the committed tokens must agree position by position."""
    from sequoia_b200.batch import BatchTree
    from sequoia_b200.tree import GreedyTree, SpecTree, clear_runtimes
    gm, Mx, iters = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256, 5
    prompts = [cases.make_prompt(30 + i, n) for i, n in enumerate((100, 64, 120))]
    with _env(SQ_DRAFT_ATTN=0, SQ_ATTN_SPLITS=1):
        d1, t1 = _bt_engines("draft", "target", Mx, 1)
        d3, t3 = _bt_engines("draft", "target", Mx, 3)
    noise = torch.empty(iters, 3, V, dtype=F16).exponential_(1.0, generator=torch.Generator().manual_seed(9)).to(DEV)
    torch.manual_seed(4)
    bt = BatchTree(d3, t3, prompts, gm, policy=policy, temperature=0.6, top_p=1.0, max_length=Mx)
    bt.external_noise = noise
    for _ in range(iters):
        bt.construct_grow_map()
        res = bt.verify()
    torch.manual_seed(4)
    from sequoia_b200.batch import draw_random
    r, rand = draw_random(prompts, Mx, gm["size"], V)          # the batch's draws, reproduced per sequence below
    same = total = 0
    for b, p in enumerate(prompts):
        clear_runtimes()
        cls = SpecTree if policy == "spec" else GreedyTree
        tree = cls(d1, t1, p.to(DEV), temperature=0.6, top_p=1.0, max_length=Mx, max_target_seq=Mx, device=DEV,
                   vocab_size=V, grow_map=gm)
        if policy == "spec":
            tree.rt.r.copy_(r[b].to(DEV))
            tree.rt.rand.copy_(rand[b].to(DEV))
            tree.rt.external_noise = noise[:, b].contiguous()
        for _ in range(iters):
            tree.construct_grow_map()
            v, _, _, term = tree.verify()
            if term:
                break
        tree.rt.external_noise = None
        got = res[b][0].cpu()
        want = v.cpu()
        k = min(len(got), len(want))
        same += int((got[:k] == want[:k]).sum()) - len(p)
        total += max(len(got), len(want)) - len(p)
        assert torch.equal(got[:len(p)], p)
    assert total > 0 and same >= 0.95 * total, (policy, same, total)


def test_batch_tree_freeze_rule():
    """draft == target weights (deep acceptance).  Sequence 1 starts near max_length, so it runs out of room after a few
    steps; sequence 2 is stopped by the caller.  Once frozen, a sequence's tokens, state row and KV rows stay byte for
    byte while the others keep decoding."""
    from sequoia_b200.batch import BatchTree
    gm, Mx = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256
    S = gm["size"]
    prompts = [cases.make_prompt(40, 64), cases.make_prompt(41, Mx - S - 6), cases.make_prompt(42, 80)]
    draft, target = _bt_engines("draft", "draft", Mx, 3)
    torch.manual_seed(3)
    bt = BatchTree(draft, target, prompts, gm, policy="spec", temperature=0.6, top_p=1.0, max_length=Mx)
    snaps = {}
    grown = 0
    for it in range(8):
        bt.construct_grow_map()
        res = bt.verify()
        if it == 1:
            bt.freeze(2)
        for b in range(3):
            if bt.frozen[b]:
                cur = (bt.tokens[b].clone(), bt.state[b].clone(),
                       [t[:, b].clone() for e in (draft, target) for t in (e.engine.kv_cache.k_cache, e.engine.kv_cache.v_cache)])
                if b in snaps:
                    old = snaps[b]
                    assert torch.equal(cur[0], old[0]) and torch.equal(cur[1], old[1]), (it, b)
                    assert all(torch.equal(x, y) for x, y in zip(cur[2], old[2])), (it, b)
                else:
                    snaps[b] = cur
        if not bt.frozen[0]:
            grown = len(res[0][0])
    assert 1 in snaps and 2 in snaps, "sequence 1 must have run out of max_length, sequence 2 must be frozen"
    assert grown > 64 + 8, "sequence 0 keeps decoding"


def test_batch_tree_two_replays_one_sync_and_launches_independent_of_B(monkeypatch):
    from sequoia_b200.batch import BatchTree
    gm, Mx = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256
    launches = {}
    for B in (1, 2, 4):
        draft, target = _bt_engines("draft", "target", Mx, B)
        torch.manual_seed(1)
        bt = BatchTree(draft, target, [cases.make_prompt(50 + b, 60 + 7 * b) for b in range(B)], gm, policy="spec",
                       temperature=0.6, top_p=1.0, max_length=Mx)
        for _ in range(2):                            # first verify + graph captures
            bt.construct_grow_map()
            bt.verify()
        syncs = []
        real_sync = torch.cuda.Stream.synchronize
        monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
        monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: syncs.append(1))
        r0 = dict(bt.replays)
        c0 = lib().launch_count()
        for _ in range(3):
            bt.construct_grow_map()
            bt.verify()
        monkeypatch.undo()
        torch.cuda.synchronize()
        assert not any(bt.frozen)
        assert bt.replays["draft"] - r0["draft"] == 3 and bt.replays["steady"] - r0.get("steady", 0) == 3
        assert len(syncs) == 3, "one host sync per step"
        assert lib().launch_count() == c0, "a steady step launches only through graph replays"
        launches[B] = bt.graph_launches["draft"] + bt.graph_launches["steady"]
    assert launches[1] == launches[2] == launches[4], launches
