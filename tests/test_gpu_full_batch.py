"""The batched decode at full batch (B up to SQ_MAX_BATCH = 8) and at real model shapes.

Kernel level, B in {1, 5, 8}: every batched entry point with sequences at different prefix lengths, once with no sequence
frozen and once with the first and last slots frozen.  Attention is compared with the float64 reference and its
per-element bound, RoPE + KV append and the KV gather bit for bit with plain torch, sampling and the accept walks bit for
bit with B = 1 launches at each sequence's own values.  Per-row kernels (RMSNorm, SiLU * up) at every template instance and
at real widths, against the fp16-chain reference and a float64 bound.  BatchTree end to end at B = 8."""
import contextlib
import dataclasses
import os

import pytest
import torch

import cases
from oracle import sequoia_oracle as O
from test_gpu_kernels import _attn_reference, _tree_vis, ulp_close

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
F16 = torch.float16
GM128 = "A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"   # config 2: 128 nodes
GM768 = "L40_growmaps/L40-CNN-7b-70b-stochastic.pt"                     # config 4: 768 nodes
ST_P, ST_N_NEW, ST_P_OLD, ST_M, ST_FROZEN = 0, 3, 4, 8, 9
SENT = -7.0
B_VALUES = [1, 5, 8]
HEAD_LAYOUTS = [(32, 32, 128), (32, 8, 128), (40, 40, 128), (12, 12, 64)]    # 7B, Llama-3-8B, 13B, 68m draft


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


_static = {}


def _tree(gm):
    if gm not in _static:
        from sequoia_b200.tree import _Static
        grow = cases.load_growmap(gm)
        _static[gm] = (_Static(grow, DEV), grow["mask"].bool().to(DEV))
    return _static[gm]


def _cache_len(S):
    return 1024 if S <= 128 else 1152          # >= 8 KV tiles: Z = 8 is reachable


def _kv_lens(B, S, M):
    """kv_len = P - 1 + S of each sequence's full-tree verify: a prompt of one token (kv_len = S), 128 j - 1, 128 j,
    128 j + 1 (one KV tile is 128 keys), a tile-aligned and a mid-tile length, and the whole cache M."""
    j = -(-S // 128) + 1
    full = [S, 128 * j - 1, 128 * j, 128 * j + 1, 128 * (j + 1), M - 1, 128 * j + 64, M]
    return {1: [M], 5: full[:4] + [M], 8: full}[B]


def _frozen_sets(B):
    return ((), (0,) if B == 1 else (0, B - 1))


def _state(B, S, M, frozen=()):
    st = torch.zeros(B, 16, dtype=torch.int32)
    for b, kv in enumerate(_kv_lens(B, S, M)):
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


def _f32(vals):
    return torch.tensor(vals, dtype=torch.float32, device=DEV)


# ------------------------------------------------------------------------------------------------ tree attention
def _attn_ref_seq(q, kc, vc, vis, H, Hkv, D):
    """_attn_reference over groups of at most 8 query heads (the kv heads they read), so the float64 temporaries of a
    40-head layout stay small: -> (out, tol), each (n, H, D)."""
    rep = H // Hkv
    kvg = max(1, 8 // rep)
    outs, tols = [], []
    for hk in range(0, Hkv, kvg):
        hk1 = min(Hkv, hk + kvg)
        ref, tol, _ = _attn_reference(q[:, hk * rep:hk1 * rep], kc[hk:hk1], vc[hk:hk1], vis, (hk1 - hk) * rep, hk1 - hk, D)
        outs.append(ref)
        tols.append(tol)
    return torch.cat(outs, 1), torch.cat(tols, 1)


def _expected_z(B, H, Hkv, n, M, forced):
    G = H // Hkv
    GP = G if 128 % G == 0 else 1
    q_tiles = -(-n // (128 // GP))
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    z = forced if forced else n_sm // max(1, (H // GP) * q_tiles * B)
    return min(max(1, min(8, z)), -(-M // 128))


ATTN_CASES = [(H, Hkv, D, GM128) for H, Hkv, D in HEAD_LAYOUTS] + [(8, 1, 128, GM768)]


@pytest.mark.parametrize("B", B_VALUES)
@pytest.mark.parametrize("H,Hkv,D,gm", ATTN_CASES, ids=lambda v: str(v).split("/")[-1])
def test_tree_attn_batch_vs_float64(B, H, Hkv, D, gm):
    """Each sequence's rows against the float64 reference within its per-element bound, at the heuristic split count and
    at Z = 2 and 8.  A frozen sequence's attention rows are still computed (DESIGN.md, freeze rule): the launch with slots
    {0, B-1} frozen must give the same bytes everywhere.  Rows past the batch keep their sentinel, the caches are only
    read."""
    tree, tmask = _tree(gm)
    S, L, layer = tree.S, 2, 1
    M = _cache_len(S)
    n = S
    g = torch.Generator(device=DEV).manual_seed(1000 * B + H + Hkv + D)
    kc = torch.randn(L, B, Hkv, M, D, generator=g, device=DEV).to(F16)
    vc = torch.randn(L, B, Hkv, M, D, generator=g, device=DEV).to(F16)
    kc0, vc0 = kc.clone(), vc.clone()
    qkv = torch.randn(B * n + 16, (H + 2 * Hkv) * D, generator=g, device=DEV).to(F16)
    out = torch.full((B * n + 16, H * D), SENT, dtype=F16, device=DEV)
    live = _state(B, S, M)
    refs = []
    for b in range(B):
        P = int(live[b, ST_P])
        kv_len = P - 1 + S
        vis = _tree_vis(torch.arange(P - 1, P - 1 + n), kv_len, P, tmask)
        refs.append(_attn_ref_seq(qkv[b * n:(b + 1) * n, :H * D].view(n, H, D), kc[layer, b, :, :kv_len],
                                  vc[layer, b, :, :kv_len], vis, H, Hkv, D))
    kw = dict(n0=0, kv_end=S, tree_bits=tree.tree_bits, tree_words=tree.tree_words, tree_size=S)
    for Z in (0, 2, 8):
        with _env(SQ_ATTN_SPLITS=Z):
            plan = ops().AttnPlan(qkv, B * n + 16, H, Hkv, D, kc, vc, out)
        first = None
        for frozen in _frozen_sets(B):
            out.fill_(SENT)
            state = _state(B, S, M, frozen)
            _one_launch(lambda: ops().tree_attn_batch(plan, layer, n, state=state, **kw))
            assert plan.error() == 0, (B, Z, frozen)
            assert plan.info()[1] == _expected_z(B, H, Hkv, n, M, Z), (B, Z, plan.info())
            assert bool((out[B * n:] == SENT).all()), "rows past the batch were written"
            if first is None:
                first = out.clone()
                for b, (ref, tol) in enumerate(refs):
                    got = out[b * n:(b + 1) * n].view(n, H, D).double()
                    assert bool(torch.isfinite(got).all()), (B, Z, b)
                    nbad = int(((got - ref).abs() > tol).sum())
                    assert nbad == 0, f"B={B} Z={Z} seq {b}: {nbad} elements outside the float64 bound"
            else:
                assert torch.equal(out, first), (B, Z, frozen)
        if Z == 0 and B == 1:
            assert plan.info()[1] > 1, "B = 1 should split the KV range"
    assert torch.equal(kc, kc0) and torch.equal(vc, vc0), "the attention wrote its caches"


def test_tree_attn_batch_bound_rejects_a_swapped_state_row():
    """Negative control at B = 8: the last sequence reads the state row of sequence 0 (another prefix length); the
    float64 bound of the correct result must reject most of its rows."""
    H, Hkv, D = 32, 8, 128
    tree, tmask = _tree(GM128)
    B, S, L, layer = 8, tree.S, 2, 1
    M, n = _cache_len(S), tree.S
    g = torch.Generator(device=DEV).manual_seed(5)
    kc = torch.randn(L, B, Hkv, M, D, generator=g, device=DEV).to(F16)
    vc = torch.randn(L, B, Hkv, M, D, generator=g, device=DEV).to(F16)
    qkv = torch.randn(B * n, (H + 2 * Hkv) * D, generator=g, device=DEV).to(F16)
    out = torch.full((B * n, H * D), SENT, dtype=F16, device=DEV)
    state = _state(B, S, M)
    wrong = state.clone()
    wrong[B - 1] = state[0]
    plan = ops().AttnPlan(qkv, B * n, H, Hkv, D, kc, vc, out)
    ops().tree_attn_batch(plan, layer, n, state=wrong, n0=0, kv_end=S, tree_bits=tree.tree_bits,
                          tree_words=tree.tree_words, tree_size=S)
    torch.cuda.synchronize()
    b = B - 1
    P = int(state[b, ST_P])
    kv_len = P - 1 + S
    vis = _tree_vis(torch.arange(P - 1, P - 1 + n), kv_len, P, tmask)
    ref, tol = _attn_ref_seq(qkv[b * n:, :H * D].view(n, H, D), kc[layer, b, :, :kv_len], vc[layer, b, :, :kv_len], vis,
                             H, Hkv, D)
    outside = ((out[b * n:].view(n, H, D).double() - ref).abs() > tol).any(-1)
    assert outside.float().mean().item() >= 0.5, "a swapped state row stays within the bound"


# ------------------------------------------------------------------------------------------------ RoPE + KV append
def _rope_tables(H, Hkv, D, kind):
    from sequoia_b200 import model
    if kind == "default":
        cfg = model.LlamaConfigLite(H * D, 4 * H * D, 1, H, Hkv, max_position_embeddings=4096)
    else:
        cfg = dataclasses.replace(model.NAMED_CONFIGS["llama-3.1-8b"], hidden_size=H * D, num_attention_heads=H,
                                  num_key_value_heads=Hkv)
    return model.rope_cache(cfg, 8192, DEV)


@pytest.mark.parametrize("B", B_VALUES)
@pytest.mark.parametrize("H,Hkv,D", HEAD_LAYOUTS, ids=lambda v: str(v))
def test_rope_kv_append_batch_bit_exact(B, H, Hkv, D):
    """Each live sequence's q rows and K/V cache rows equal O.apply_rotary_pos_emb (the fp16 chain) on its rows, scattered
    through a storage_ids permutation, at positions up to 8191 with the default and the llama3 tables.  Every other cache
    row, plane and layer keeps its sentinel."""
    tree, _ = _tree(GM128)
    S, L, layer, n = tree.S, 2, 1, tree.S
    M = _cache_len(S)
    assert (H + Hkv) * D // 16 > 256 or D == 64, "the work loop must wrap"
    g = torch.Generator(device=DEV).manual_seed(100 * B + H + Hkv)
    qkv0 = torch.randn(B * n + 8, (H + 2 * Hkv) * D, generator=g, device=DEV).to(F16)
    pos = torch.randint(0, 8192, (B, M), generator=g, device=DEV)
    pos[:, :8] = 8191
    sto = torch.stack([torch.randperm(M, generator=g, device=DEV) for _ in range(B)])
    for kind in ("default", "llama3"):
        cos, sin = _rope_tables(H, Hkv, D, kind)
        for frozen in _frozen_sets(B):
            state = _state(B, S, M, frozen)
            qkv = qkv0.clone()
            kc = torch.full((L, B, Hkv, M, D), SENT, dtype=F16, device=DEV)
            vc = torch.full_like(kc, SENT)
            _one_launch(lambda: ops().rope_kv_append_batch(qkv, H, Hkv, D, cos, sin, pos, sto, n, kc[layer], vc[layer], M,
                                                           state))
            k_ref = torch.full_like(kc, SENT)
            v_ref = torch.full_like(kc, SENT)
            q_ref = qkv0.clone()
            for b in range(B):
                if b in frozen:
                    continue
                base = int(state[b, ST_P]) - 1
                rows = qkv0[b * n:(b + 1) * n]
                q = rows[:, :H * D].view(1, n, H, D).transpose(1, 2)
                k = rows[:, H * D:(H + Hkv) * D].view(1, n, Hkv, D).transpose(1, 2)
                v = rows[:, (H + Hkv) * D:].view(n, Hkv, D).transpose(0, 1)
                qe, ke = O.apply_rotary_pos_emb(q, k, cos, sin, pos[b, base:base + n].unsqueeze(0))
                q_ref[b * n:(b + 1) * n, :H * D] = qe[0].transpose(0, 1).reshape(n, H * D)
                slots = sto[b, base:base + n]
                k_ref[layer, b].index_copy_(1, slots, ke[0])
                v_ref[layer, b].index_copy_(1, slots, v)
            assert torch.equal(qkv, q_ref), (B, kind, frozen)
            assert torch.equal(kc, k_ref) and torch.equal(vc, v_ref), (B, kind, frozen)


def test_rope_kv_append_batch_tables_differ():
    """The llama3 tables must differ from the default ones at long positions, or the llama3 case above tests nothing new."""
    c0, _ = _rope_tables(32, 8, 128, "default")
    c1, _ = _rope_tables(32, 8, 128, "llama3")
    assert not torch.equal(c0[8000], c1[8000])


# ------------------------------------------------------------------------------------------------ embedding
@pytest.mark.parametrize("B", B_VALUES)
@pytest.mark.parametrize("hidden", [4096, 8192])
def test_embed_rows_batch_large_vocab(B, hidden):
    V = 128256
    tree, _ = _tree(GM128)
    S = tree.S
    M = _cache_len(S)
    n0, n = 1, S - 1
    g = torch.Generator(device=DEV).manual_seed(B + hidden)
    table = torch.randn(V, hidden, generator=g, device=DEV, dtype=F16)
    tokens = torch.randint(0, V, (B, M + S), generator=g, device=DEV)
    live = _state(B, S, M)
    for b in range(B):
        base = int(live[b, ST_P]) - 1 + n0
        tokens[b, base] = 0
        tokens[b, base + n - 1] = V - 1
    for frozen in _frozen_sets(B):
        state = _state(B, S, M, frozen)
        out = torch.full((B * n + 8, hidden), SENT, dtype=F16, device=DEV)
        _one_launch(lambda: ops().embed_rows_batch(table, tokens, n, out, state, n0=n0))
        for b in range(B):
            rows = out[b * n:(b + 1) * n]
            if b in frozen:
                assert bool((rows == SENT).all()), (B, b)
            else:
                base = int(state[b, ST_P]) - 1 + n0
                assert torch.equal(rows, table[tokens[b, base:base + n]]), (B, b, frozen)
        assert bool((out[B * n:] == SENT).all())


# ------------------------------------------------------------------------------------------------ KV gather
@pytest.mark.parametrize("B", B_VALUES)
def test_kv_gather_batch_vs_torch(B):
    """Against "gather into a temporary, then copy to [P_old, P_old + n)" on each live sequence's planes; every other
    byte of the caches (frozen sequences, rows outside the destination, both layers) is unchanged."""
    tree, _ = _tree(GM128)
    S, L, Hkv, D = tree.S, 2, 8, 128
    M = _cache_len(S)
    md = tree.max_depth
    g = torch.Generator(device=DEV).manual_seed(B + 70)
    kc0 = torch.randn(L, B, Hkv, M, D, generator=g, device=DEV).to(F16)
    vc0 = torch.randn(L, B, Hkv, M, D, generator=g, device=DEV).to(F16)
    n_new = [(0, md, 1, md - 1, 2, md, 0, 3)[b] for b in range(B)] if B > 1 else [md]
    for frozen in _frozen_sets(B):
        state = _state(B, S, M, frozen)
        idx = torch.full((B, S), -1, dtype=torch.int32, device=DEV)
        for b in range(B):
            P = int(state[b, ST_P])
            sel = torch.sort(torch.randperm(S - 1, generator=torch.Generator().manual_seed(b))[:n_new[b]])[0] + P
            idx[b, :n_new[b]] = sel.to(torch.int32).to(DEV)
            state[b, ST_N_NEW] = n_new[b]
            state[b, ST_P_OLD] = P
        kc, vc = kc0.clone(), vc0.clone()
        _one_launch(lambda: ops().kv_gather_batch(kc, vc, idx, state, md))
        k_ref, v_ref = kc0.clone(), vc0.clone()
        for b in range(B):
            if b in frozen or n_new[b] == 0:
                continue
            P, src = int(state[b, ST_P_OLD]), idx[b, :n_new[b]].long()
            for ref in (k_ref, v_ref):
                tmp = ref[:, b][:, :, src].clone()
                ref[:, b, :, P:P + n_new[b]] = tmp
        assert torch.equal(kc.view(torch.int16), k_ref.view(torch.int16)), (B, frozen)
        assert torch.equal(vc.view(torch.int16), v_ref.view(torch.int16)), (B, frozen)
        assert not torch.equal(kc, kc0) or all(b in frozen or n_new[b] == 0 for b in range(B))


# ------------------------------------------------------------------------------------------------ sampling and accept
TS = [0.45, 0.6, 0.8, 1.0, 1.3, 0.7, 0.5, 1.1]
TOP_PS = [0.9, 1.0, 0.8, 1.0, 0.95, 0.7, 1.0, 0.85]
BIG_VOCABS = [32000, 128256]


def _draft_layout(tree, per_seq, V):
    B = len(per_seq)
    levels = [(0, 1)] + [(lv["n0"], lv["tb"]) for lv in tree.levels]
    base, step = ops().draft_row_tables(levels, tree.S, B, DEV)
    buf = torch.full((B * tree.S, V), SENT, dtype=F16, device=DEV)
    for b in range(B):
        buf[base.long() + b * step.long()] = per_seq[b]
    return buf, base, step


@pytest.mark.parametrize("V", BIG_VOCABS)
@pytest.mark.parametrize("mode", [0, 1])
def test_sample_level_batch_per_seq_b8(V, mode):
    tree, _ = _tree(GM128)
    B, S = 8, tree.S
    M = _cache_len(S)
    g = torch.Generator(device=DEV).manual_seed(V + mode + 8)
    per_seq = [(torch.randn(S, V, generator=g, device=DEV) * 2).to(F16) for _ in range(B)]
    rand = torch.rand(B, S, V, generator=g, device=DEV).to(F16) if mode == 0 else None
    buf, base, step = _draft_layout(tree, per_seq, V)

    def sample(buf, base, step, rand, T, tokens, state):
        for lv in tree.levels:
            _one_launch(lambda: ops().sample_level_batch_per_seq(
                buf, base, step, rand, lv["n_parents"], lv["k"], T, mode, parent_rows=lv["parents"],
                child_first=lv["first"], n_branch=lv["nb"], tokens=tokens, state=state))

    for frozen in _frozen_sets(B):
        state = _state(B, S, M, frozen)
        got = torch.full((B, M), -5, dtype=torch.int64, device=DEV)
        sample(buf, base, step, rand, _f32(TS), got, state)
        for b in range(B):
            want = torch.full((1, M), -5, dtype=torch.int64, device=DEV)
            if b not in frozen:
                buf1, base1, step1 = _draft_layout(tree, [per_seq[b]], V)
                sample(buf1, base1, step1, rand[b:b + 1] if rand is not None else None, _f32([TS[b]]), want,
                       state[b:b + 1].clone())
                P = int(state[b, ST_P])
                assert bool((got[b, P:P + S - 1] >= 0).all()), (V, mode, b)
            assert torch.equal(got[b], want[0]), (V, mode, b, frozen)


def _walk_inputs(tree, B, V, M, seed):
    S = tree.S
    g = torch.Generator(device=DEV).manual_seed(seed)
    per_seq, target = [], []
    for b in range(B):
        d = (torch.randn(S, V, generator=g, device=DEV) * 0.5).to(F16)
        eps = [0.0, 0.3, 3.0, 0.0, 0.05, 0.5, 0.0, 1.0][b]       # equal rows accept deep paths; noisy rows reject early
        per_seq.append(d)
        target.append((d.float() + eps * torch.randn(S, V, generator=g, device=DEV)).to(F16))
    tokens = torch.randint(3, V, (B, M), generator=g, device=DEV)
    pos = torch.randint(0, M, (B, M), generator=g, device=DEV)
    r = torch.rand(B, M, generator=g, device=DEV).to(F16)
    noise = torch.empty(B, V, device=DEV).exponential_(1.0, generator=g).to(F16)
    return per_seq, torch.cat(target), tokens, pos, r, noise


@pytest.mark.parametrize("V", BIG_VOCABS)
def test_accept_stochastic_batch_per_seq_b8(V):
    tree, _ = _tree(GM128)
    B, S = 8, tree.S
    M = _cache_len(S)
    per_seq, target, tokens0, pos0, r, noise = _walk_inputs(tree, B, V, M, seed=V + 81)
    buf, base, step = _draft_layout(tree, per_seq, V)
    for frozen in _frozen_sets(B):
        st0 = _state(B, S, M, frozen)
        tokens, pos, acc, state = tokens0.clone(), pos0.clone(), torch.full((B, S), -1, dtype=torch.int32,
                                                                            device=DEV), st0.clone()
        _one_launch(lambda: ops().accept_stochastic_batch_per_seq(
            target, buf, base, step, r, noise, tree.succ_off, tree.succ, tree.depth, S, _f32(TS), tokens, pos, acc, state,
            M))
        deepest = 0
        for b in range(B):
            t1, p1, s1 = tokens0[b:b + 1].clone(), pos0[b:b + 1].clone(), st0[b:b + 1].clone()
            a1 = torch.full((1, S), -1, dtype=torch.int32, device=DEV)
            if b not in frozen:
                buf1, base1, step1 = _draft_layout(tree, [per_seq[b]], V)
                ops().accept_stochastic_batch_per_seq(target[b * S:(b + 1) * S], buf1, base1, step1, r[b:b + 1],
                                                      noise[b:b + 1], tree.succ_off, tree.succ, tree.depth, S,
                                                      _f32([TS[b]]), t1, p1, a1, s1, M)
                torch.cuda.synchronize()
            for x, y in zip((tokens, pos, acc, state), (t1, p1, a1, s1)):
                assert torch.equal(x[b], y[0]), (V, b, frozen)
            deepest = max(deepest, int(state[b, ST_N_NEW]))
        assert deepest >= 3, "the equal-row sequences should accept a path of several nodes"


def test_accept_greedy_batch_b8():
    tree, _ = _tree(GM128)
    B, S = 8, tree.S
    M = _cache_len(S)
    _, _, tokens0, pos0, _, _ = _walk_inputs(tree, B, cases.V, M, seed=390)
    g = torch.Generator(device=DEV).manual_seed(391)
    target_token = torch.randint(3, cases.V, (B * S,), generator=g, device=DEV)
    succ_off, succ = tree.succ_off.cpu(), tree.succ.cpu()
    st_host = _state(B, S, M).cpu()
    for b in range(1, B, 2):                           # odd sequences: the target agrees with the first child everywhere
        P = int(st_host[b, ST_P])
        for k in range(S):
            c0, c1 = int(succ_off[k]), int(succ_off[k + 1])
            if c1 > c0:
                target_token[b * S + k] = tokens0[b, P - 1 + int(succ[c0])]
    deep = 0
    for frozen in _frozen_sets(B):
        st0 = _state(B, S, M, frozen)
        tokens, pos, acc, state = tokens0.clone(), pos0.clone(), torch.full((B, S), -1, dtype=torch.int32,
                                                                            device=DEV), st0.clone()
        _one_launch(lambda: ops().accept_greedy_batch(target_token, tree.succ_off, tree.succ, tree.depth, S, tokens, pos,
                                                      acc, state, M))
        for b in range(B):
            t1, p1, s1 = tokens0[b:b + 1].clone(), pos0[b:b + 1].clone(), st0[b:b + 1].clone()
            a1 = torch.full((1, S), -1, dtype=torch.int32, device=DEV)
            if b not in frozen:
                ops().accept_greedy_batch(target_token[b * S:(b + 1) * S], tree.succ_off, tree.succ, tree.depth, S, t1,
                                          p1, a1, s1, M)
                torch.cuda.synchronize()
            for x, y in zip((tokens, pos, acc, state), (t1, p1, a1, s1)):
                assert torch.equal(x[b], y[0]), (b, frozen)
        deep = max(deep, int(state[B - 1, ST_N_NEW]))
    assert deep >= 3, "the last sequence should accept its first-child path while live"


@pytest.mark.parametrize("V", BIG_VOCABS)
def test_top_p_filter_per_seq_b8(V):
    B, R = 8, 32
    g = torch.Generator(device=DEV).manual_seed(V + 83)
    logits0 = (torch.randn(B * R, V, generator=g, device=DEV) * 3).to(F16)
    got = logits0.clone()
    _one_launch(lambda: ops().top_p_filter_per_seq_(got, _f32(TOP_PS), _f32(TS), R))
    for b in range(B):
        rows = slice(b * R, (b + 1) * R)
        if TOP_PS[b] >= 1.0:
            assert torch.equal(got[rows].view(torch.int16), logits0[rows].view(torch.int16)), f"top_p = 1: row {b} touched"
        else:
            want = ops().top_p_filter_(logits0[rows].clone(), TOP_PS[b], TS[b])
            torch.cuda.synchronize()
            assert torch.equal(got[rows], want), (V, b)
            assert bool(torch.isinf(got[rows]).any()), (V, b)


# ------------------------------------------------------------------------------------------------ RMSNorm
HIDDENS = [2048, 3072, 4096, 5120, 8192, 16384]        # rmsnorm_kernel MAXV = 1, 2, 2, 4, 4, 8 (5120: partial last pass)
ROW_KINDS = ("randn", "large", "small", "spike", "zero")


def _norm_rows(n, hidden, g, add):
    """(x, d) fp16 rows of kinds cycling through ROW_KINDS: randn; |x| up to 6e4 (the fp32 sum of squares near 2^45 at
    16384); randn * 3e-3 (mean square near eps, so eps matters); small values with a last 8-wide group ~ 30 (that group
    dominates the norm); all zero.  d (add_rmsnorm's delta) is None without add."""
    x = torch.randn(n, hidden, generator=g, device=DEV)
    d = torch.randn(n, hidden, generator=g, device=DEV) if add else None
    for r in range(n):
        kind = ROW_KINDS[r % len(ROW_KINDS)]
        if kind == "large":
            x[r] = (torch.rand(hidden, generator=g, device=DEV) * 2 - 1) * 6e4
        elif kind == "small":
            x[r] *= 3e-3
            if add:
                d[r] *= 1e-3
        elif kind == "spike":
            x[r] *= 0.01
            x[r, -8:] = 30.0
            if add:
                d[r] *= 0.01
        elif kind == "zero":
            x[r] = 0
            if add:
                d[r] = 0
    return x.to(F16), d.to(F16) if add else None


def _rms_f64(x, w, eps, drop_last_group=False):
    x64 = x.double()
    sq = x64[:, :-8] if drop_last_group else x64
    ms = (sq * sq).sum(-1, keepdim=True) / x.shape[-1]
    return w.double() * x64 / torch.sqrt(ms + eps)


def _rms_tol(exact, w, hidden):
    """Bound of |kernel - exact| for the fp16 chain fp16(w * fp16(x * rsqrtf(fp32 mean(x^2) + eps))):
      2 x 2^-11 relative   the fp16 roundings of xn = x * inv and of the product w * xn (w * xn itself is exact in fp32);
      (hidden/2 + 4) 2^-24 + 2^-22 relative   the fp32 sum of `hidden` non-negative squares (<= hidden 2^-24 relative
                           in any order, halved by the square root), the divide, the eps add, x * inv, and rsqrtf (2 ulp);
      (|w| + 1) 2^-25      xn or the output landing among the fp16 subnormals (absolute spacing 2^-24)."""
    rel = 2 * 2.0 ** -11 + (hidden / 2 + 4) * 2.0 ** -24 + 2.0 ** -22
    return rel * 1.01 * exact.abs() + (w.double().abs() + 1) * 2.0 ** -25


def _off_chain(got, src, w, eps):
    """Elements of `got` more than 1 fp16 ulp from the fp16-chain reference O.rmsnorm that the chain does not explain.
    The kernel sums the squares in fp32 in another order than torch, so where x * inv lies next to an fp16 rounding
    boundary its xn may round to the neighbouring fp16 value; a |w| < 1 can then put the product two output ulps away.
    Such an element must equal the chain's output at that neighbouring xn exactly."""
    nbad, bad = ulp_close(got, O.rmsnorm(src, w, eps), 1)
    if nbad == 0:
        return 0
    xf = src.float()
    bits = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(F16).view(torch.int16)
    near = (got == w * (bits + 1).view(F16)) | (got == w * (bits - 1).view(F16))
    return int((bad.to(DEV) & ~near).sum())


def _outside(got, exact, tol):
    return int(((got.double() - exact).abs() > tol).sum())


@pytest.mark.parametrize("add", [False, True], ids=["rmsnorm", "add_rmsnorm"])
@pytest.mark.parametrize("n", [1, 129, 1024])
@pytest.mark.parametrize("hidden", HIDDENS)
def test_rmsnorm_instances_vs_references(hidden, n, add):
    eps = 1e-5
    g = torch.Generator(device=DEV).manual_seed(hidden + n + int(add))
    x, d = _norm_rows(n, hidden, g, add)
    w = (1 + 0.1 * torch.randn(hidden, generator=g, device=DEV)).to(F16)
    out = torch.full((n + 2, hidden), SENT, dtype=F16, device=DEV)
    if add:
        resid = x.clone()
        _one_launch(lambda: ops().add_rmsnorm(resid, d, w, out, n, eps))
        assert torch.equal(resid, x + d), "resid must be x + d (one fp16 rounding)"
        src = x + d
    else:
        _one_launch(lambda: ops().rmsnorm(x, w, out, n, eps))
        src = x
    got = out[:n]
    assert bool((out[n:] == SENT).all())
    assert bool(torch.isfinite(got).all()), "non-finite outputs"
    nbad = _off_chain(got, src, w, eps)
    assert nbad == 0, f"{nbad} elements differ from the fp16 chain by more than 1 ulp (and not by one xn rounding)"
    exact = _rms_f64(src, w, eps)
    tol = _rms_tol(exact, w, hidden)
    assert _outside(got, exact, tol) == 0, "outside the float64 bound"
    zero = [r for r in range(n) if ROW_KINDS[r % len(ROW_KINDS)] == "zero"]
    if zero:
        assert bool((got[zero] == 0).all()), "an all-zero row must give 0"


@pytest.mark.parametrize("hidden", [4096, 16384])
def test_rmsnorm_bound_sees_errors(hidden):
    """Negative controls: fp16-chain outputs with eps off by 10x (seen on the rows whose mean square is near eps) and with
    the last 8-wide group left out of the sum of squares (seen on the rows where that group dominates) fall outside the
    float64 bound that the kernel meets."""
    eps, n = 1e-5, len(ROW_KINDS)
    g = torch.Generator(device=DEV).manual_seed(hidden)
    x, _ = _norm_rows(n, hidden, g, False)
    w = (1 + 0.1 * torch.randn(hidden, generator=g, device=DEV)).to(F16)
    exact = _rms_f64(x, w, eps)
    tol = _rms_tol(exact, w, hidden)
    small, spike = ROW_KINDS.index("small"), ROW_KINDS.index("spike")
    got = torch.empty(n, hidden, dtype=F16, device=DEV)
    ops().rmsnorm(x, w, got, n, eps)
    torch.cuda.synchronize()
    assert _outside(got, exact, tol) == 0
    wrong_eps = O.rmsnorm(x, w, 10 * eps)
    assert _outside(wrong_eps[small:small + 1], exact[small:small + 1], tol[small:small + 1]) > hidden // 2
    dropped = (w.double() * x.double() / torch.sqrt((x.double()[:, :-8] ** 2).sum(-1, keepdim=True) / hidden + eps)).to(F16)
    assert _outside(dropped[spike:spike + 1], exact[spike:spike + 1], tol[spike:spike + 1]) > hidden // 2


# ------------------------------------------------------------------------------------------------ SiLU * up
@pytest.mark.parametrize("n,inter", [(1024, 11008), (1024, 14336), (1, 688)])
def test_silu_mul_grid_stride(n, inter):
    """Plain within 1 ulp of torch's fp16 silu(gate) * up; the interleaved layout (blocks of 16 gate | 16 up) bit for bit
    against the plain call on the de-interleaved rows.  n * inter / 8 > 132 * 8 * 256 makes the grid-stride loop wrap."""
    g = torch.Generator(device=DEV).manual_seed(n + inter)
    gate = (torch.randn(n, inter, generator=g, device=DEV) * 3).to(F16)
    up = torch.randn(n, inter, generator=g, device=DEV).to(F16)
    gu = torch.cat([gate, up], 1)
    out = torch.full((n + 2, inter), SENT, dtype=F16, device=DEV)
    _one_launch(lambda: ops().silu_mul(gu, out, n))
    assert bool((out[n:] == SENT).all())
    nbad, _ = ulp_close(out[:n], torch.nn.functional.silu(gate) * up, 1)
    assert nbad == 0, f"{nbad} elements differ by more than 1 ulp"
    gu_i = torch.stack([gate.view(n, inter // 16, 16), up.view(n, inter // 16, 16)], 2).reshape(n, 2 * inter)
    out_i = torch.full_like(out, SENT)
    _one_launch(lambda: ops().silu_mul(gu_i, out_i, n, interleaved=True))
    assert torch.equal(out_i, out), "interleaved != plain"
    if n > 1:
        assert n * inter // 8 > 132 * 8 * 256


# ------------------------------------------------------------------------------------------------ refusals
def test_unsupported_calls_are_refused_before_any_launch():
    from sequoia_b200._lib import SequoiaLibError
    x = torch.zeros(4, 16392, dtype=F16, device=DEV)
    w = torch.ones(16392, dtype=F16, device=DEV)
    st9 = torch.zeros(9, 16, dtype=torch.int32, device=DEV)
    qkv = torch.zeros(8, 3 * 72, dtype=F16, device=DEV)
    cos = torch.zeros(16, 72, dtype=F16, device=DEV)
    ids = torch.zeros(1, 16, dtype=torch.int64, device=DEV)
    kl = torch.zeros(1, 1, 16, 72, dtype=F16, device=DEV)
    calls = {
        "rmsnorm hidden > 16384": lambda: ops().rmsnorm(x, w, x.clone(), 4, 1e-5),
        "add_rmsnorm hidden > 16384": lambda: ops().add_rmsnorm(x.clone(), x, w, x.clone(), 4, 1e-5),
        "rmsnorm hidden % 8": lambda: ops().rmsnorm(x[:, :4100], w[:4100], x.clone()[:, :4100], 4, 1e-5),
        "silu_mul inter % 8": lambda: ops().silu_mul(x[:, :8200], x.clone()[:, :4100], 4),
        "silu_mul interleaved inter % 16": lambda: ops().silu_mul(x[:, :8208], x.clone()[:, :4104], 4, interleaved=True),
        "embed_rows_batch B = 9": lambda: ops().embed_rows_batch(x, torch.zeros(9, 8, dtype=torch.int64, device=DEV), 1,
                                                                 x.clone(), st9),
        "rope_kv_append_batch D % 16": lambda: ops().rope_kv_append_batch(qkv, 1, 1, 72, cos, cos, ids, ids, 1, kl, kl, 16,
                                                                          st9[:1]),
        "kv_gather_batch B = 9": lambda: ops().kv_gather_batch(torch.zeros(1, 9, 1, 16, 64, dtype=F16, device=DEV),
                                                               torch.zeros(1, 9, 1, 16, 64, dtype=F16, device=DEV),
                                                               torch.zeros(9, 8, dtype=torch.int32, device=DEV), st9, 4),
    }
    torch.cuda.synchronize()
    for what, fn in calls.items():
        c0 = lib().launch_count()
        with pytest.raises(SequoiaLibError):
            fn()
        assert lib().launch_count() == c0, f"{what}: refused after a launch"


# ------------------------------------------------------------------------------------------------ BatchTree at B = 8
def _bt_engines(dkey, tkey, Mx, B):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    dcfg, dw = cases.model_weights(dkey)
    tcfg, tw = cases.model_weights(tkey)
    with _env(SQ_DRAFT_ATTN=0, SQ_ATTN_SPLITS=1):
        return (GraphInferenceEngine(Mx, {"config": dcfg, "state_dict": dw}, device=DEV, batch_size=B),
                GraphInferenceEngineTG(Mx, {"config": tcfg, "state_dict": tw}, device=DEV, batch_size=B))


PROMPT_LENS8 = (20, 130, 64, 97, 33, 120, 75, 48)


@pytest.mark.parametrize("policy", ["spec", "greedy"])
def test_batch_tree_eight_prompts_lock_step(policy):
    """Eight prompts of 20..130 tokens decoded together; each sequence against a lone SpecTree / GreedyTree on its prompt
    with the same draws.  The batch's GEMMs run on 8x the rows, so rounding may differ: at least 95% of each sequence's
    committed tokens must agree position by position, and every prompt is kept as it was."""
    from sequoia_b200.batch import BatchTree, draw_random
    from sequoia_b200.tree import GreedyTree, SpecTree, clear_runtimes
    gm, Mx, iters, B = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256, 5, 8
    V = cases.V
    prompts = [cases.make_prompt(130 + i, n) for i, n in enumerate(PROMPT_LENS8)]
    d1, t1 = _bt_engines("draft", "target", Mx, 1)
    d8, t8 = _bt_engines("draft", "target", Mx, B)
    noise = torch.empty(iters, B, V, dtype=F16).exponential_(1.0, generator=torch.Generator().manual_seed(19)).to(DEV)
    torch.manual_seed(14)
    bt = BatchTree(d8, t8, prompts, gm, policy=policy, temperature=0.6, top_p=1.0, max_length=Mx)
    bt.external_noise = noise
    for _ in range(iters):
        bt.construct_grow_map()
        res = bt.verify()
    torch.manual_seed(14)
    r, rand = draw_random(prompts, Mx, gm["size"], V)
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
        got, want = res[b][0].cpu(), v.cpu()
        assert torch.equal(got[:len(p)], p), (policy, b)
        k = min(len(got), len(want))
        same = int((got[:k] == want[:k]).sum()) - len(p)
        total = max(len(got), len(want)) - len(p)
        assert total > 0 and same >= 0.95 * total, (policy, b, same, total)


def test_batch_tree_b8_launches_syncs_and_replays(monkeypatch):
    """Steady steps at B = 8 launch as many kernels as at B = 1, through graph replays only, with one host sync each."""
    from sequoia_b200.batch import BatchTree
    gm, Mx = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256
    launches = {}
    for B in (1, 8):
        draft, target = _bt_engines("draft", "target", Mx, B)
        torch.manual_seed(1)
        bt = BatchTree(draft, target, [cases.make_prompt(150 + b, PROMPT_LENS8[b]) for b in range(B)], gm, policy="spec",
                       temperature=0.6, top_p=1.0, max_length=Mx)
        for _ in range(2):
            bt.construct_grow_map()
            bt.verify()
        syncs = []
        real_sync = torch.cuda.Stream.synchronize
        monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
        monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: syncs.append(1))
        r0, c0 = dict(bt.replays), lib().launch_count()
        for _ in range(3):
            bt.construct_grow_map()
            bt.verify()
        monkeypatch.undo()
        torch.cuda.synchronize()
        assert not any(bt.frozen), B
        assert bt.replays["draft"] - r0["draft"] == 3 and bt.replays["steady"] - r0.get("steady", 0) == 3, B
        assert len(syncs) == 3, f"B={B}: one host sync per step"
        assert lib().launch_count() == c0, f"B={B}: a steady step launches only through graph replays"
        launches[B] = bt.graph_launches["draft"] + bt.graph_launches["steady"]
    assert launches[1] == launches[8], launches


def test_batch_tree_b8_admission_into_the_last_slot():
    """B = 8: slot 7 is frozen after step 2 and given a new prompt at step 3 at its own T and top_p.  Slots 0..6 match a
    run in which slot 7 stays frozen, bit for bit: tokens, accept lengths and the KV rows of both engines."""
    from sequoia_b200.batch import BatchTree
    gm, Mx, iters, at, B = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256, 7, 3, 8
    V = cases.V
    prompts = [cases.make_prompt(170 + i, n) for i, n in enumerate(PROMPT_LENS8)]
    new = cases.make_prompt(180, 90)
    noise = torch.empty(iters, B, V, dtype=F16).exponential_(1.0, generator=torch.Generator().manual_seed(18)).to(DEV)

    def run(admit):
        d, t = _bt_engines("draft", "target", Mx, B)
        torch.manual_seed(4)
        bt = BatchTree(d, t, prompts, gm, temperature=0.6, top_p=1.0, max_length=Mx)
        bt.external_noise = noise
        steps = []
        for it in range(iters):
            if it == at and admit:
                torch.manual_seed(9)
                bt.admit(B - 1, new, temperature=0.9, top_p=0.85)
            bt.construct_grow_map()
            steps.append([(v.clone(), a, term) for v, a, term in bt.verify()])
            if it == at - 1:
                bt.freeze(B - 1)
        caches = [x for e in (d, t) for x in (e.engine.kv_cache.k_cache, e.engine.kv_cache.v_cache)]
        return steps, caches

    with_adm, caches = run(True)
    without, caches0 = run(False)
    for it in range(iters):
        for b in range(B - 1):
            (v, a, term), (v0, a0, term0) = with_adm[it][b], without[it][b]
            assert (a, term) == (a0, term0) and torch.equal(v, v0), (it, b)
    for b in range(B - 1):
        a = with_adm[-1][b][1]
        for got, want in zip(caches, caches0):
            assert torch.equal(got[:, b, ..., :a, :], want[:, b, ..., :a, :]), b
    v_new = with_adm[-1][B - 1][0].cpu()
    assert torch.equal(v_new[:len(new)], new) and len(v_new) > len(new), "the admitted prompt decodes"
