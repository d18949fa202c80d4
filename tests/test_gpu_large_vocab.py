"""Large-vocabulary (32768 < V <= 131072) instances of the sampling, top-p and accept kernels, the lm_head GEMM at
N = 128256, and decoding with 128K-vocabulary models.  References are float64 / torch-CPU restatements, or the V <= 32768
kernel instances the rest of the suite checks against the oracle."""
import pytest
import torch

import cases
from oracle import sequoia_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
F16 = torch.float16
VS = [32776, 128256, 131072]
SLICE = 32768


def ops():
    from sequoia_b200 import ops as _ops
    return _ops


def _ulp(x: torch.Tensor) -> torch.Tensor:
    mag = x.double().abs().clamp(min=2.0 ** -24)
    return torch.pow(2.0, torch.floor(torch.log2(mag)) - 10).clamp(min=2.0 ** -24)


def _logits(V, rows, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(rows, V, generator=g) * scale).to(F16)


def _topk_ref(x: torch.Tensor, k: int) -> torch.Tensor:
    """indices of the k largest values, ties to the lower index (a stable descending sort); NaN ranks above every number,
    as in torch.topk (a score log(u) / q is 0 / 0 when u rounds to 1 and q underflows to 0)"""
    return torch.sort(-torch.nan_to_num(x.double(), nan=float("inf")), stable=True).indices[:k]


# ------------------------------------------------------------------------------------------------ argmax / top-k
@pytest.mark.parametrize("V", VS)
def test_argmax_rows_large_vocab(V):
    x = _logits(V, 7, V)
    x[3, V - 5] = 30.0                       # a maximum in the last slice only
    x[4, 10] = 30.0
    x[4, V - 1] = 30.0                       # equal maxima in the first and last slice -> the lower index
    got = ops().argmax_rows(x.to(DEV)).cpu()
    ref = torch.stack([_topk_ref(r, 1)[0] for r in x])
    assert torch.equal(got, ref)
    assert int(got[3]) == V - 5 and int(got[4]) == 10
    # negative control: a reduction that skipped the last slice's exchange would have returned another index
    assert int(_topk_ref(x[3, :(V - 1) // SLICE * SLICE], 1)[0]) != V - 5


@pytest.mark.parametrize("V", VS)
@pytest.mark.parametrize("k", [1, 8, 32, 40])
def test_topk_sample_level_mode1_large_vocab(V, k):
    rows = 5
    x = _logits(V, rows, 7 * k + V)
    x[1, 3] = x[1, V - 3] = 25.0             # cross-slice tie at the top
    x[2, SLICE - 1] = x[2, SLICE] = 20.0     # tie straddling the first slice boundary
    pos = torch.full((rows, k), -1, dtype=torch.int64, device=DEV)
    ops().sample_level(x.to(DEV), None, rows, k, 1.0, 1, positions=pos)
    for r in range(rows):
        assert torch.equal(pos[r].cpu(), _topk_ref(x[r], k)), f"row {r}"
    assert int(pos[1, 0]) == 3 and int(pos[2, 0]) == SLICE - 1
    if k > 1:
        assert int(pos[1, 1]) == V - 3 and int(pos[2, 1]) == SLICE


@pytest.mark.parametrize("V", VS)
def test_sampling_without_replacement_large_vocab(V):
    """mode 0 (the exponential race): the fp16 scores fp16(fp16(log u) / q) restated on the CPU with q = fp16 of the
    float64 softmax of fp16(x * fp32(1/T)); positions bit-exact except where two scores are within 1 ulp (q may differ
    from the kernel's fp32 softmax by one ulp)."""
    rows, k, T = 4, 16, 0.6
    x = _logits(V, rows, V + 1)
    g = torch.Generator().manual_seed(V + 2)
    u = torch.rand(rows, V, generator=g).clamp(min=1e-4).to(F16)
    pos = torch.full((rows, k), -1, dtype=torch.int64, device=DEV)
    ops().sample_level(x.to(DEV), u.to(DEV), rows, k, T, 0, positions=pos)
    q = torch.softmax((x.float() * (1.0 / T)).half().double(), -1).half()
    score = (u.float().log().half().float() / q.float()).half()
    for r in range(rows):
        got, ref = pos[r].cpu(), _topk_ref(score[r], k)
        if not torch.equal(got, ref):
            a, b = score[r][got].double(), score[r][ref].double()
            ok = ((a - b).abs() <= 2 * _ulp(score[r][ref])) | (torch.isnan(a) & torch.isnan(b))
            assert bool(ok.all()), f"row {r}: {got.tolist()} vs {ref.tolist()}"


# ------------------------------------------------------------------------------------------------ softmax / residual
@pytest.mark.parametrize("V", VS)
def test_residual_large_vocab_within_one_ulp(V):
    g = torch.Generator().manual_seed(V + 4)
    p = torch.softmax(torch.randn(V, generator=g) * 3, -1).half()
    q = torch.softmax(torch.randn(V, generator=g) * 3, -1).half()
    got = ops().residual(p.to(DEV), q.to(DEV)).cpu().double()
    d = (p.float() - q.float()).half().float().clamp(min=0)
    tot = float(d.double().sum())
    ref = (d.double() / float(torch.tensor(tot).half())).half().double()
    assert bool(((got - ref).abs() <= _ulp(ref)).all())


# ------------------------------------------------------------------------------------------------ top-p
def _top_p_torch(logits, top_p, T):
    """utils.py:65-77 with the kernel's arithmetic: x * fp32(1/T) rounded to fp16, fp16 probabilities, and their
    cumulative sum taken exactly (float64: every fp16 probability is a multiple of 2^-24).  The kernel ranks by the scaled
    fp16 value xt (two logits that round to the same xt have equal probability and rank by index, as in the V <= 32768
    kernel), so the reference sorts by xt too."""
    xt_all = (logits.float() * (1.0 / T)).half()
    _, idx = torch.sort(xt_all, descending=True, stable=True)
    xt = torch.gather(xt_all, -1, idx).double()
    probs = torch.softmax(xt, dim=-1).half()
    cum = torch.cumsum(probs.double(), dim=-1).half()
    filt = cum > top_p
    filt[..., 1:] = filt[..., :-1].clone()
    filt[..., 0] = False
    return logits.masked_fill(filt.scatter(-1, idx, filt), float("-inf"))


@pytest.mark.parametrize("V", VS)
@pytest.mark.parametrize("top_p,scale", [(0.9, 3.0), (0.5, 8.0), (0.99, 1.0)])
def test_top_p_filter_large_vocab(V, top_p, scale):
    x = _logits(V, 4, V + int(100 * top_p), scale)
    got = ops().top_p_filter_(x.clone().to(DEV), top_p, 0.6).cpu()
    ref = _top_p_torch(x.clone(), top_p, 0.6)
    keep_g, keep_r = ~torch.isinf(got), ~torch.isinf(ref)
    assert int((keep_g.sum(-1) - keep_r.sum(-1)).abs().max()) <= 1     # identical up to one boundary token
    for r in range(x.shape[0]):
        diff = (keep_g[r] != keep_r[r]).nonzero().flatten()
        assert diff.numel() <= 1, f"row {r}: {diff.numel()} positions differ"
    assert torch.equal(got[keep_g], x[keep_g])                         # survivors untouched


@pytest.mark.parametrize("V", [32776, 128256])
def test_top_p_boundary_tie_group_across_slices_ranks_by_index(V):
    """64 equal logits spread over every slice at top_p = 0.5: the first 33 in index order stay."""
    lg = torch.full((1, V), -30.0, dtype=F16)
    idx = torch.linspace(5, V - 9, 64).long()
    lg[0, idx] = 2.0
    got = ops().top_p_filter_(lg.clone().to(DEV), 0.5, 1.0).cpu()
    assert torch.equal((~torch.isinf(got[0])).nonzero().flatten(), idx[:33])


# ------------------------------------------------------------------------------------------------ batched sampling
@pytest.mark.parametrize("V", [32776, 128256])
@pytest.mark.parametrize("mode", [0, 1])
def test_sample_level_batch_large_vocab_matches_single_launches(V, mode):
    B, S, P, k = 3, 3, 6, 4
    row_base, row_step = ops().draft_row_tables([(0, 1), (1, 2)], S, B, DEV)
    logits = _logits(V, S * B, V + mode).to(DEV)
    g = torch.Generator().manual_seed(11)
    rand = torch.rand(B, S, V, generator=g).clamp(min=1e-4).to(F16).to(DEV)
    parents = torch.tensor([1, 2], dtype=torch.int32, device=DEV)
    first = torch.tensor([3, 7], dtype=torch.int32, device=DEV)
    nb = torch.tensor([4, 3], dtype=torch.int32, device=DEV)
    M = 32
    state = torch.zeros(B, 16, dtype=torch.int32, device=DEV)
    state[:, 0] = P
    state[1, 9] = 1                                                     # sequence 1 frozen
    tokens = torch.full((B, M), -7, dtype=torch.int64, device=DEV)
    ops().sample_level_batch(logits, row_base, row_step, rand if mode == 0 else None, 2, k, 0.6, mode,
                             parent_rows=parents, child_first=first, n_branch=nb, tokens=tokens, state=state)
    rb, rs = row_base.cpu(), row_step.cpu()
    for b in range(B):
        if b == 1:
            assert bool((tokens[1] == -7).all())
            continue
        rows = torch.stack([logits[int(rb[n]) + b * int(rs[n])] for n in range(S)])
        tok = torch.full((M,), -7, dtype=torch.int64, device=DEV)
        st = state[b].clone()
        ops().sample_level(rows, rand[b] if mode == 0 else None, 2, k, 0.6, mode, parent_rows=parents,
                           child_first=first, n_branch=nb, tokens=tok, state=st)
        assert torch.equal(tokens[b], tok), f"sequence {b}"
        assert int((tok != -7).sum()) == 7 and bool((tok[:P - 1 + 3] == -7).all())   # sentinels outside the children


# ------------------------------------------------------------------------------------------------ accept walk
def _accept_case(seed, S_gm="L40_growmaps/8x8-tree.pt"):
    gm = cases.load_growmap(S_gm)
    S = gm["size"]
    g = torch.Generator().manual_seed(seed)
    tl = (torch.randn(S, cases.V, generator=g) * 2).to(F16)
    dl = (torch.randn(S, cases.V, generator=g) * 2).to(F16)
    dl[:, :64] += 4.0                                                    # drafts concentrated where the target is
    tl[:, :64] += 4.0
    P, M = 12, 128
    tokens = torch.zeros(M, dtype=torch.long)
    tokens[:P] = torch.randint(3, 1000, (P,), generator=g)
    tokens[P:P + S - 1] = torch.randint(3, 64, (S - 1,), generator=g)
    r = torch.rand(M, generator=g).half()
    noise = torch.empty(cases.V).exponential_(1.0, generator=g).half()
    return gm, S, tl, dl, tokens, r, noise, P, M


def _embed(x, V, off, fill=-float("inf")):
    out = torch.full(x.shape[:-1] + (V,), fill, dtype=x.dtype)
    out[..., off:off + x.shape[-1]] = x
    return out


@pytest.mark.parametrize("V", VS)
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_accept_stochastic_large_vocab_matches_small_instance(V, seed):
    """The same walk at V = 32000 (the instance checked against the oracle) and embedded at offset V - 32000 of a V-wide
    row (-inf elsewhere, so the softmax has the same terms): same accept list and bonus, shifted by the offset."""
    from sequoia_b200.tree import _Static
    gm, S, tl, dl, tokens, r, noise, P, M = _accept_case(seed)
    st = _Static(gm, DEV)
    off = V - cases.V
    res = []
    for (tl_, dl_, tok_, nz_) in ((tl, dl, tokens, noise),
                                  (_embed(tl, V, off), _embed(dl, V, off), torch.where(torch.arange(M) >= P, tokens + off,
                                                                                      tokens), _embed(noise, V, off, 1.0))):
        d_tok, d_pos = tok_.to(DEV), torch.arange(M).to(DEV)
        acc = torch.zeros(S, dtype=torch.int32, device=DEV)
        state = torch.zeros(16, dtype=torch.int32, device=DEV)
        state[0], state[8] = P, M
        ops().accept_stochastic(tl_.to(DEV), dl_.to(DEV), r.to(DEV), nz_.to(DEV), st.succ_off, st.succ, st.depth, S, 0.6,
                                d_tok, d_pos, acc, state, M)
        hs = state.cpu()
        res.append((hs.clone(), acc[:int(hs[3])].cpu().clone(), d_tok.cpu(), d_pos.cpu()))
    (h0, a0, t0, p0), (h1, a1, t1, p1) = res
    assert torch.equal(a0, a1) and torch.equal(h0[[0, 1, 2, 3, 4, 6, 7]], h1[[0, 1, 2, 3, 4, 6, 7]])
    if not bool(h0[2]):
        assert int(h1[5]) == int(h0[5]) + off
        a = int(h0[1])
        assert torch.equal(t1[P:a + 1], t0[P:a + 1] + off) and torch.equal(p0, p1)


@pytest.mark.parametrize("V", [32776, 128256])
def test_accept_stochastic_batch_large_vocab_matches_single(V):
    from sequoia_b200.tree import _Static
    B = 3
    gms = [_accept_case(s) for s in (4, 5, 6)]
    gm, S = gms[0][0], gms[0][1]
    st = _Static(gm, DEV)
    off = V - cases.V
    M, P = gms[0][8], gms[0][7]
    tl = torch.cat([_embed(c[2], V, off) for c in gms]).to(DEV)
    dl_rows = torch.stack([_embed(c[3], V, off) for c in gms], 1).reshape(S * B, V).to(DEV)   # node-major, B rows each
    row_base = torch.arange(S, dtype=torch.int32, device=DEV) * B
    row_step = torch.ones(S, dtype=torch.int32, device=DEV)
    tokens = torch.stack([torch.where(torch.arange(M) >= P, c[4] + off, c[4]) for c in gms]).to(DEV)
    r = torch.stack([c[5] for c in gms]).to(DEV)
    noise = torch.stack([_embed(c[6], V, off, 1.0) for c in gms]).to(DEV)
    pos = torch.arange(M).repeat(B, 1).to(DEV)
    acc = torch.full((B, S), -3, dtype=torch.int32, device=DEV)
    state = torch.zeros(B, 16, dtype=torch.int32, device=DEV)
    state[:, 0], state[:, 8] = P, M
    state[2, 9] = 1                                                       # frozen
    tok0, pos0, st0 = tokens.clone(), pos.clone(), state.clone()
    ops().accept_stochastic_batch(tl, dl_rows, row_base, row_step, r, noise, st.succ_off, st.succ, st.depth, S, 0.6, tokens,
                                  pos, acc, state, M)
    assert torch.equal(tokens[2], tok0[2]) and torch.equal(state[2], st0[2]) and bool((acc[2] == -3).all())
    for b in range(2):
        t1, p1 = tok0[b].clone(), pos0[b].clone()
        a1 = torch.zeros(S, dtype=torch.int32, device=DEV)
        s1 = st0[b].clone()
        ops().accept_stochastic(tl[b * S:(b + 1) * S], dl_rows[b::B], r[b], noise[b], st.succ_off, st.succ, st.depth, S, 0.6,
                                t1, p1, a1, s1, M)
        n = int(s1[3])
        assert torch.equal(state[b], s1) and torch.equal(tokens[b], t1) and torch.equal(pos[b], p1)
        assert torch.equal(acc[b, :n], a1[:n])


# ------------------------------------------------------------------------------------------------ refusals
def test_sample_replace_refuses_large_vocab():
    x = torch.zeros(2, 128256, dtype=F16, device=DEV)
    words = torch.zeros(8, dtype=torch.int64, device=DEV)
    pos = torch.zeros(2, 4, dtype=torch.int64, device=DEV)
    with pytest.raises(Exception, match="32768"):
        ops().sample_replace(x, words, 2, 4, 1.0, positions=pos)


def test_sampling_refuses_beyond_131072():
    x = torch.zeros(1, 131080, dtype=F16, device=DEV)
    with pytest.raises(Exception, match="131072"):
        ops().argmax_rows(x)


# ------------------------------------------------------------------------------------------------ lm_head GEMM
@pytest.mark.parametrize("K", [4096, 2048])
def test_lm_head_gemm_n128256_vs_float64(K):
    N = 128256
    g = torch.Generator(device=DEV).manual_seed(K)
    w = (torch.randn(N, K, device=DEV, generator=g) * 0.02).half()
    a = torch.randn(128, K, device=DEV, generator=g).half()
    c = torch.zeros(128, N, dtype=F16, device=DEV)
    plan = ops().GemmPlan(a, w, c)
    for n in (1, 19, 128):
        c.fill_(7.0)
        plan.run(n)
        torch.cuda.synchronize()
        ref = a[:n].double() @ w.double().t()
        bound = a[:n].double().abs() @ w.double().abs().t()
        err = (c[:n].double() - ref).abs()
        tol = _ulp(ref) + K * 2.0 ** -23 * bound
        assert bool((err <= tol).all()), f"n={n}: max err {float(err.max())}"
        assert bool((c[n:] == 7.0).all()), "rows beyond n written"
        del ref, bound, err, tol


# ------------------------------------------------------------------------------------------------ decoding
def _v128_models(M):
    from Engine.Engine import GraphInferenceEngine, GraphInferenceEngineTG
    V = 128256
    dcfg = O.LlamaCfg(hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, vocab_size=V)
    tcfg = O.LlamaCfg(hidden_size=512, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=4,
                      num_key_value_heads=4, vocab_size=V)
    dw, tw = O.init_llama_weights(dcfg, 501), O.init_llama_weights(tcfg, 502)
    draft = GraphInferenceEngine(M, {"config": dcfg, "state_dict": dw}, device=DEV)
    target = GraphInferenceEngineTG(M, {"config": tcfg, "state_dict": tw}, device=DEV)
    return dcfg, dw, tcfg, tw, draft, target


def _buf(M):
    return dict(attn_mask=torch.full((M, M), torch.finfo(F16).min, dtype=F16, device=DEV),
                sequence=torch.arange(M, device=DEV).unsqueeze(-1), new_tokens_buffer=torch.zeros(M, device=DEV).long(),
                parents_buffer=torch.zeros(M, device=DEV).long(), position_ids=torch.zeros(M, device=DEV).long())


@pytest.mark.parametrize("V", [32776, 128256, 131072])
@pytest.mark.parametrize("seed", [7, 8])
def test_accept_stochastic_large_vocab_spread_tokens_and_bonus_tie(V, seed):
    """The V = 32000 walk spread over the whole wide row by the increasing map i -> i * V // 32000 (-inf elsewhere): the
    drafted tokens land in every CTA and in chunks 1..3 of their threads, the first child of every node holds the draft
    maximum (so its rejection re-computes the draft statistics), and two tokens in different CTAs tie for the bonus."""
    from sequoia_b200.tree import _Static
    gm = cases.load_growmap("L40_growmaps/8x8-tree.pt")
    S, Vs, P, M = gm["size"], cases.V, 12, 128
    g = torch.Generator().manual_seed(seed)
    hot = torch.linspace(40, Vs - 40, 64).long()                          # spread over the small row
    tl = (torch.randn(S, Vs, generator=g) * 2).to(F16)
    dl = (torch.randn(S, Vs, generator=g) * 2).to(F16)
    tl[:, hot] += 4.0
    dl[:, hot] += 4.0
    tokens = torch.zeros(M, dtype=torch.long)
    tokens[:P] = torch.randint(3, 1000, (P,), generator=g)
    tokens[P:P + S - 1] = hot[torch.randint(0, 64, (S - 1,), generator=g)]
    for node, ch in enumerate(gm["Successors"]):
        if ch:
            dl[node, int(tokens[P - 1 + ch[0]])] = 12.0                   # the first child is the draft maximum
    a, b = 5, Vs - 7                                                      # bonus tie: equal p, never drafted, q ~ 0
    tl[:, a] = tl[:, b] = 16.0                                            # above every other target logit
    dl[:, a] = dl[:, b] = -20.0
    r = torch.rand(M, generator=g).half()
    noise = torch.empty(Vs).exponential_(1.0, generator=g).clamp(min=0.6).half()
    noise[a] = noise[b] = 0.25
    st = _Static(gm, DEV)
    mp = torch.arange(Vs) * V // Vs                                       # increasing: ties keep their order
    chunks = ((mp[hot] // 8) % ((V // 8 + 7) // 8)) // 512
    if V > 65536:
        assert set(chunks.tolist()) >= {0, 1, 2, 3}
    assert int(mp[a]) // ((V // 8 + 7) // 8 * 8) != int(mp[b]) // ((V // 8 + 7) // 8 * 8)

    def wide(x, fill):
        out = torch.full(x.shape[:-1] + (V,), fill, dtype=x.dtype)
        out[..., mp] = x
        return out

    res = []
    for (tl_, dl_, tok_, nz_) in ((tl, dl, tokens, noise),
                                  (wide(tl, -float("inf")), wide(dl, -float("inf")),
                                   torch.where(torch.arange(M) >= P, mp[tokens.clamp(max=Vs - 1)], tokens),
                                   wide(noise, 1.0))):
        d_tok, d_pos = tok_.to(DEV), torch.arange(M).to(DEV)
        acc = torch.zeros(S, dtype=torch.int32, device=DEV)
        state = torch.zeros(16, dtype=torch.int32, device=DEV)
        state[0], state[8] = P, M
        ops().accept_stochastic(tl_.to(DEV), dl_.to(DEV), r.to(DEV), nz_.to(DEV), st.succ_off, st.succ, st.depth, S, 0.6,
                                d_tok, d_pos, acc, state, M)
        hs = state.cpu()
        res.append((hs.clone(), acc[:int(hs[3])].cpu().clone(), d_tok.cpu(), d_pos.cpu()))
    (h0, a0, t0, p0), (h1, a1, t1, p1) = res
    assert torch.equal(a0, a1) and torch.equal(h0[[0, 1, 2, 3, 4, 6, 7]], h1[[0, 1, 2, 3, 4, 6, 7]])
    assert not bool(h0[2]) and int(h0[5]) == a                            # the lower index of the tie
    assert int(h1[5]) == int(mp[a])
    n = int(h0[1])
    assert torch.equal(t1[P:n + 1], mp[t0[P:n + 1]]) and torch.equal(p0, p1)


# ------------------------------------------------------------------------------------------------ decoding
V128 = 128256


def _v128_weights():
    """68m- and 160m-shaped layers (hidden 768, 12 heads of 64) with a 128256-token vocabulary"""
    dcfg = O.LlamaCfg(hidden_size=768, intermediate_size=3072, num_hidden_layers=2, num_attention_heads=12,
                      num_key_value_heads=12, vocab_size=V128)
    tcfg = O.LlamaCfg(hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                      num_key_value_heads=12, vocab_size=V128)
    return {"d128k": (dcfg, O.init_llama_weights(dcfg, 501)), "t128k": (tcfg, O.init_llama_weights(tcfg, 502))}


@pytest.fixture(scope="module")
def v128_weights():
    return _v128_weights()


@pytest.mark.parametrize("mode", ["spec", "greedy"])
def test_decode_128k_vocab_teacher_forced_vs_oracle(mode, v128_weights, monkeypatch):
    """tests/test_gpu_decode.py's teacher-forced lock-step with the CPU oracle (every level of every iteration compared,
    forks explained and repaired) on a 68m -> 160m-shaped pair with V = 128256: >= 95% identical drafted nodes."""
    import functools

    import test_gpu_decode as D
    monkeypatch.setattr(cases, "V", V128)
    for name in ("SpecTreeOracle", "GreedyTreeOracle"):
        monkeypatch.setattr(O, name, functools.partial(getattr(O, name), vocab_size=V128))
    monkeypatch.setattr(cases, "model_weights", lambda key: v128_weights[key])
    table = {"v128": ("L40_growmaps/8x8-tree.pt", mode, "d128k", "t128k", 256, 3, 64, 4, 11)}
    same, total, forks, done, worst = D._teacher_forced("v128", table)
    assert total > 0 and same / total >= D.MIN_IDENTICAL, (same, total, forks)
    # 12 target layers of width 768 against test_gpu_decode's 2-3 layers of 256-512: fp16 GEMM-order noise grows with
    # depth, so the logit bound is test_gpu_decode's REL_TOL rather than its DRAFT_LOGIT_TOL
    assert worst <= D.REL_TOL and done >= 1, (worst, done)


def _engines_v128(w, M, B=1, cfgs=("d128k", "t128k")):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    (dcfg, dw), (tcfg, tw) = w[cfgs[0]], w[cfgs[1]]
    return (GraphInferenceEngine(M, {"config": dcfg, "state_dict": dw}, device=DEV, batch_size=B),
            GraphInferenceEngineTG(M, {"config": tcfg, "state_dict": tw}, device=DEV, batch_size=B))


def test_batch_tree_b2_128k_vocab_matches_lone_spec_trees(v128_weights):
    """BatchTree at B = 2 (wide batched sampling and accept kernels inside the captured graphs) against two lone SpecTrees
    on the same prompts and random draws.  The batch's GEMMs run on twice the rows, so cuBLAS may round differently, as
    in tests/test_gpu_batch.py's lock-step: the first step must agree exactly and >= 95% of the committed tokens overall."""
    from sequoia_b200.batch import BatchTree, draw_random
    from sequoia_b200.tree import SpecTree, clear_runtimes
    gm, Mx, iters = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256, 5
    prompts = [cases.make_prompt(30 + i, n) for i, n in enumerate((100, 64))]
    import test_gpu_batch as TB
    with TB._env(SQ_DRAFT_ATTN=0, SQ_ATTN_SPLITS=1):
        d1, t1 = _engines_v128(v128_weights, Mx, 1)
        d2, t2 = _engines_v128(v128_weights, Mx, 2)
    noise = torch.empty(iters, 2, V128, dtype=F16).exponential_(1.0, generator=torch.Generator().manual_seed(9)).to(DEV)
    torch.manual_seed(4)
    bt = BatchTree(d2, t2, prompts, gm, policy="spec", temperature=0.6, top_p=1.0, max_length=Mx)
    bt.external_noise = noise
    steps = []
    for _ in range(iters):
        bt.construct_grow_map()
        steps.append([x[0].cpu().clone() for x in bt.verify()])
    assert bt.replays.get("steady", 0) >= iters - 1
    torch.manual_seed(4)
    r, rand = draw_random(prompts, Mx, gm["size"], V128)
    same = total = 0
    for b, p in enumerate(prompts):
        clear_runtimes()
        tree = SpecTree(d1, t1, p.to(DEV), temperature=0.6, top_p=1.0, max_length=Mx, max_target_seq=Mx, device=DEV,
                        grow_map=gm)
        tree.rt.r.copy_(r[b].to(DEV))
        tree.rt.rand.copy_(rand[b].to(DEV))
        tree.rt.external_noise = noise[:, b].contiguous()
        for it in range(iters):
            tree.construct_grow_map()
            v, _, _, term = tree.verify()
            if it == 0:
                assert torch.equal(v.cpu(), steps[0][b]), f"sequence {b}: first step differs"
            if term:
                break
        tree.rt.external_noise = None
        got, want = steps[-1][b], v.cpu()
        k = min(len(got), len(want))
        same += int((got[:k] == want[:k]).sum()) - len(p)
        total += max(len(got), len(want)) - len(p)
        d1.clear_kv()
        t1.clear_kv()
    assert total > 0 and same >= 0.95 * total, (same, total)


def _count_syncs(monkeypatch):
    syncs = []
    real = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real(self))[1])
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: syncs.append(1))
    return syncs


def test_llama3_1b_to_8b_real_shapes(monkeypatch):
    """random-init:llama-3.2-1b -> random-init:llama-3.1-8b with the 128-node c2 growmap: 8 decode steps through SpecTree
    and through BatchTree (B = 2); finite logits, tokens inside the vocabulary, and each steady step is two graph replays
    and one host sync with no launch outside the graphs."""
    from sequoia_b200 import _lib
    from sequoia_b200.batch import BatchTree
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    from sequoia_b200.tree import SpecTree, clear_runtimes
    gm = cases.load_growmap("A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt")
    assert gm["size"] == 128
    M, steps = 384, 8
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, V128, (128,), generator=g) for _ in range(2)]
    for B in (1, 2):
        clear_runtimes()
        draft = GraphInferenceEngine(M, "random-init:llama-3.2-1b:1", device=DEV, batch_size=B)
        target = GraphInferenceEngineTG(M, "random-init:llama-3.1-8b:2", device=DEV, batch_size=B)
        torch.manual_seed(5)
        if B == 1:
            tree = SpecTree(draft, target, prompts[0].to(DEV), temperature=0.6, top_p=1.0, max_length=M, max_target_seq=M,
                            device=DEV, grow_map=gm)
            replays, logits = tree.rt.replays, lambda: tree.rt.target_logits
            step = lambda: (tree.construct_grow_map(), [tree.verify()[0]])[1]
        else:
            tree = BatchTree(draft, target, [p.to(DEV) for p in prompts], gm, policy="spec", temperature=0.6, top_p=1.0,
                             max_length=M, max_target_seq=M)
            replays, logits = tree.replays, lambda: tree.target_logits
            step = lambda: [x[0] for x in (tree.construct_grow_map(), tree.verify())[1]]
        for it in range(steps):
            if it >= 2:
                syncs = _count_syncs(monkeypatch)
                r0, c0 = dict(replays), _lib.launch_count()
            out = step()
            if it >= 2:
                monkeypatch.undo()
                torch.cuda.synchronize()
                assert sum(replays.values()) - sum(r0.values()) == 2, (B, it, replays, r0)
                assert len(syncs) == 1, (B, it, len(syncs))
                assert _lib.launch_count() == c0, (B, it)
            assert bool(torch.isfinite(logits()).all()), (B, it)
            for v in out:
                assert int(v.max()) < V128 and int(v.min()) >= 0
        del tree, draft, target
        torch.cuda.empty_cache()
