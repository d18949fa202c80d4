"""Prompt logprobs on the device (sq_prompt_logprobs_ragged, BatchTree(prompt_logprobs=...)).

Kernel level: every written value against the rule of oracle/prompt_logprobs.py (float64) at V from 32000 to 131072, with
1, 3 and 8 parts of 1 to 1023 rows at gapped logits offsets, n in {0, 1, 5, 20}, on rows with ties, -inf runs, a +inf row
and a NaN row; everything the kernel must not write keeps its sentinel bit for bit.  BatchTree level: a teacher-forced
float32 forward of the prompts (a dense causal pass that shares no code with the ragged first verify), off and on change
nothing else (outputs, token logprobs, graphs, launches), the values ignore every per-sequence processing setting, the
admission rules, a full batch of prompt lengths 1 .. M - S + 1 and one run at V = 128256."""
import numpy as np
import pytest
import torch

import cases
from oracle import logprobs as L
from oracle import prompt_logprobs as PL
from oracle import sequoia_oracle as O
from test_gpu_mixed_policy import GM128
from test_gpu_refill import DEV, F16, _engines, ops

pytestmark = pytest.mark.gpu

NMAX = L.MAX_LOGPROBS
TOK_SENT, ID_SENT, TOP_SENT = 12345.0, -7, 777.0
NS = [0, 1, 5, 20]


def _lib():
    from sequoia_b200 import _lib as lib
    return lib


def _tree(engines, prompts, gm, Mx, **kw):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    d.clear_kv()
    t.clear_kv()
    return BatchTree(d, t, prompts, gm, max_length=Mx, max_target_seq=Mx, **kw)


# ------------------------------------------------------------------------------------------------ kernel
def _want_rows(x, toks, n):
    """The oracle's rule over many rows at once (float64): -> (token logprob (R,), ids (R, n), top logprobs (R, n)).
    Rows of x (R, V) fp16, toks (R,) the scored ids."""
    s = x.double()
    bad = torch.isnan(s).any(1) | (s == float("inf")).any(1)
    m = torch.where(torch.isnan(s), torch.full_like(s, -float("inf")), s).max(1).values
    ok = ~bad & (m > -float("inf"))
    m = torch.where(ok, m, torch.zeros_like(m))
    lse = m + torch.log(torch.exp(torch.where(ok[:, None], s - m[:, None], torch.zeros_like(s))).sum(1))
    lp = torch.where(ok[:, None], s - lse[:, None], torch.full_like(s, float("nan")))
    V = x.shape[1]
    inside = (toks >= 0) & (toks < V)
    tok_lp = torch.where(inside, lp.gather(1, toks.clamp(0, V - 1)[:, None])[:, 0], torch.full_like(lse, float("nan")))
    ids = torch.sort(L.rank_key(x), dim=1, descending=True, stable=True).indices[:, :min(n, V)]
    return tok_lp, ids, lp.gather(1, ids), torch.where(ok, lse, torch.zeros_like(lse))


def _close(got, want, lse):
    both_nan = torch.isnan(got) & torch.isnan(want)
    exact = got.double() == want
    near = (got.double() - want).abs() <= 1e-4 * (1 + lse.abs())
    return bool((both_nan | exact | near).all())


def _rows(R, V, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(R, V, generator=g) * 4).to(F16)
    x[::3, 100:140] = 2.5                               # a tie group across the top-n boundary
    x[1::4, ::2] = float("-inf")                        # -inf runs
    x[2::5, 10:20] = 0.0
    x[2::5, 20:30] = -0.0
    x[3::50, 7] = float("inf")                          # +inf rows, NaN rows and all -inf rows in every part set
    x[4::70, 9] = float("nan")
    x[5::90] = float("-inf")
    return x


PART_SETS = {1: [383], 3: [1, 17, 1023], 8: [2, 1, 17, 383, 2, 17, 1, 2]}


@pytest.mark.parametrize("V", [32000, 49152, 128256, 131072])
@pytest.mark.parametrize("n_parts", [1, 3, 8])
def test_kernel_matches_oracle(V, n_parts):
    B, Mx = 8, 1100
    sizes = PART_SETS[n_parts]
    g = torch.Generator().manual_seed(V + n_parts)
    seqs = torch.randperm(B, generator=g)[:n_parts].tolist()
    parts, r0 = [], 3                                   # gaps of 3 + j rows between the parts' logits rows
    for j, (seq, n_rows) in enumerate(zip(seqs, sizes)):
        parts.append((seq, r0, n_rows, NS[(j + n_parts) % 4]))
        r0 += n_rows + 3 + j
    x = _rows(r0, V, V + n_parts)
    tokens = torch.randint(0, V, (B, Mx), generator=g)
    tokens[seqs[0], 2] = V + 3                          # an id outside [0, V): NaN
    plp_token = torch.full((B, Mx), TOK_SENT, dtype=torch.float32, device=DEV)
    plp_ids = torch.full((B, Mx, NMAX), ID_SENT, dtype=torch.int32, device=DEV)
    plp_top = torch.full((B, Mx, NMAX), TOP_SENT, dtype=torch.float32, device=DEV)
    c0 = _lib().launch_count()
    ops().prompt_logprobs_ragged_(x.to(DEV), parts, tokens.to(DEV), plp_token, plp_ids, plp_top)
    torch.cuda.synchronize()
    assert _lib().launch_count() == c0 + 1, "one launch for all parts"
    got_tok, got_ids, got_top = plp_token.cpu(), plp_ids.cpu(), plp_top.cpu()
    tok_written = torch.zeros(B, Mx, dtype=torch.bool)
    top_written = torch.zeros(B, Mx, NMAX, dtype=torch.bool)
    for seq, row0, n_rows, n in parts:
        rows = x[row0:row0 + n_rows]
        toks = tokens[seq, 1:n_rows + 1]
        k = min(n, V)
        for c in range(0, n_rows, 128):                 # (in chunks: float64 copies of 128 rows at a time)
            e = min(c + 128, n_rows)
            w_tok, w_ids, w_top, lse = _want_rows(rows[c:e], toks[c:e], n)
            assert _close(got_tok[seq, c + 1:e + 1], w_tok, lse), (seq, n_rows, c)
            assert torch.equal(got_ids[seq, c + 1:e + 1, :k].long(), w_ids), (seq, n_rows, n, c)
            assert _close(got_top[seq, c + 1:e + 1, :k], w_top, lse[:, None]), (seq, n_rows, n, c)
        for r in {0, n_rows - 1, n_rows // 2}:          # the oracle itself, row by row
            t, ids, top = PL.prompt_logprobs(rows[r:r + 1], tokens[seq, r:r + 2], n)[0]
            lse = float(_want_rows(rows[r:r + 1], toks[r:r + 1], 0)[3][0])
            assert got_ids[seq, r + 1, :k].tolist() == ids
            assert np.allclose([float(got_tok[seq, r + 1])] + got_top[seq, r + 1, :k].tolist(), [t] + top,
                               rtol=0, atol=1e-4 * (1 + abs(lse)), equal_nan=True)
        tok_written[seq, 1:n_rows + 1] = True
        top_written[seq, 1:n_rows + 1, :k] = True
    assert bool((got_tok[~tok_written] == TOK_SENT).all()), "an unwritten logprob changed"
    assert bool((got_ids[~top_written] == ID_SENT).all()) and bool((got_top[~top_written] == TOP_SENT).all()), \
        "an unwritten top entry changed"


def test_ops_refusals_on_the_device():
    B, Mx, V = 2, 64, 32000
    x = torch.zeros(100, V, dtype=F16, device=DEV)
    tok = torch.zeros(B, Mx, dtype=torch.long, device=DEV)
    outs = [torch.zeros(B, Mx, device=DEV), torch.zeros(B, Mx, NMAX, dtype=torch.int32, device=DEV),
            torch.zeros(B, Mx, NMAX, device=DEV)]
    with pytest.raises(ValueError, match="plp_ids"):
        ops().prompt_logprobs_ragged_(x, [(0, 0, 4, 1)], tok, outs[0], outs[1][:, :, :5], outs[2])
    with pytest.raises(TypeError, match="int64"):
        ops().prompt_logprobs_ragged_(x, [(0, 0, 4, 1)], tok.int(), *outs)
    from sequoia_b200._lib import SequoiaLibError
    with pytest.raises(SequoiaLibError, match="rows"):
        ops().prompt_logprobs_ragged_(x, [(0, 90, 20, 1)], tok, *outs)


# ------------------------------------------------------------------------------------------------ BatchTree
def _reference_logprobs(prompt, Mx):
    """log_softmax of the float32 CPU oracle's causal forward over the prompt: (P-1, V) float64, row i = position i+1."""
    cfg, w = cases.model_weights("target")
    ref = O.EngineOracle(O.LlamaOracle(cfg, {k: v.float() for k, v in w.items()}, Mx, "TG", dtype=torch.float32))
    P = len(prompt)
    logits = ref.inference(prompt[None], torch.arange(P), torch.arange(P)[None],
                           O.make_causal_mask(P, torch.float32)[None, None])[0].double()
    return torch.log_softmax(logits, -1)[:P - 1]


def _check_teacher_forced(lp, ids, prompt, want):
    """Tolerance as in test_gpu_logprobs.test_teacher_forced_float32_forward: |d logprob| <= 2 max |d x| <= 2^-7 per
    position, n * 2^-7 for the sum; the top-1 id is the reference argmax wherever its margin exceeds 2^-6."""
    tol = 2.0 ** -7
    w_tok = want.gather(1, prompt[1:, None]).squeeze(1)
    assert lp.shape == w_tok.shape
    err = (lp.double() - w_tok).abs()
    assert float(err.max()) <= tol, (float(err.max()), int(err.argmax()))
    assert abs(float(lp.double().sum() - w_tok.sum())) <= tol * len(lp)
    top2 = want.topk(2, dim=1)
    clear = (top2.values[:, 0] - top2.values[:, 1]) > 2.0 ** -6
    assert bool(clear.any()) and torch.equal(ids[clear, 0], top2.indices[clear, 0])


def test_teacher_forced_float32_forward():
    gm, Mx = cases.load_growmap(GM128), 384
    prompts = [cases.make_prompt(740 + i, n) for i, n in enumerate((50, 70))]
    bt = _tree(_engines(2, Mx), [p.to(DEV) for p in prompts], gm, Mx, policy="greedy", temperature=1.0,
               prompt_logprobs=[20, 4])
    bt.construct_grow_map()
    bt.verify()
    for b, p in enumerate(prompts):
        lp, ids, top = bt.prompt_logprobs(b)
        assert ids.shape == (len(p) - 1, (20, 4)[b]) and top.shape == ids.shape
        _check_teacher_forced(lp, ids, p, _reference_logprobs(p, Mx))


def _decode(bt, iters):
    out = []
    for _ in range(iters):
        bt.construct_grow_map()
        out.append([(v.cpu().clone(), a, term) for v, a, term in bt.verify()])
        if all(bt.frozen):
            break
    return out


def test_off_and_on_change_nothing_else():
    gm, Mx = cases.load_growmap(GM128), 384
    engines = _engines(3, Mx)
    prompts = [cases.make_prompt(750 + i, n).to(DEV) for i, n in enumerate((70, 100, 84))]
    kw = dict(seeds=[31, 32, 33], policy=["spec", "greedy", "spec"], top_k=[40, 0, 0], repetition_penalty=[1.0, 1.0, 1.2],
              logprobs=[2, None, 5])
    runs = {}
    for setting in (None, 0, [20, None, 5]):
        bt = _tree(engines, prompts, gm, Mx, prompt_logprobs=setting, **kw)
        c0 = _lib().launch_count()
        out = _decode(bt, 6)
        runs[str(setting)] = (bt, out, _lib().launch_count() - c0)
    off_bt, off, off_launches = runs["None"]
    assert off_bt.plp_token is None, "off: nothing allocated"
    for name in ("0", "[20, None, 5]"):
        bt, out, launches = runs[name]
        assert len(out) == len(off)
        for it in range(len(off)):
            for b in range(3):
                assert torch.equal(out[it][b][0], off[it][b][0]) and out[it][b][1:] == off[it][b][1:], (name, it, b)
        assert bt.finish_reason == off_bt.finish_reason
        for b in (0, 2):
            for x, y in zip(bt.token_logprobs(b), off_bt.token_logprobs(b)):
                assert torch.equal(x, y), (name, b)
        assert bt.graph_launches == off_bt.graph_launches and bt.captures == off_bt.captures
        assert bt.kernel_launches() == off_bt.kernel_launches()
        # the first verify launches one more kernel, plus the lm_head GEMMs that run on sq_gemm (<= 128 rows with a plan)
        runner = bt.target.engine.runner
        on = [b for b in range(3) if (bt.prompt_logprobs_n[b] is not None)]
        gemms = sum(1 for b in on if runner.lm_plan is not None and len(prompts[b]) - 1 <= 128)
        assert launches == off_launches + 1 + gemms, (name, launches, off_launches)


def _guide():
    from sequoia_b200.guide import GuideState, TokenGuide
    return TokenGuide([GuideState(default=0, banned=(5, 6))])


def test_values_ignore_processing_settings():
    """Slot 0 with every processing setting, or none, next to the same neighbours: its prompt logprobs are the same
    bits (no prompt token was drawn from a processed row)."""
    gm, Mx = cases.load_growmap(GM128), 384
    engines = _engines(2, Mx)
    prompts = [cases.make_prompt(760 + i, n).to(DEV) for i, n in enumerate((60, 90))]
    base = dict(policy="spec", prompt_logprobs=[20, 3], seeds=[1, 2])
    plain = _tree(engines, prompts, gm, Mx, **base)
    plain.construct_grow_map()
    plain.verify()
    want = [plain.prompt_logprobs(b) for b in range(2)]
    settings = [dict(temperature=[0.3, 0.6]), dict(top_k=[5, 0]), dict(repetition_penalty=[1.5, 1.0]),
                dict(frequency_penalty=[0.7, 0.0]), dict(logit_bias=[{5: 20.0, 9: -100.0}, None]),
                dict(allowed_token_ids=[list(range(100, 900)), None]), dict(bad_words=[[[7], [8, 9]], None]),
                dict(guide=[_guide(), None]), dict(min_p=[0.2, 0.0])]
    for s in settings:
        bt = _tree(engines, prompts, gm, Mx, **base, **s)
        bt.construct_grow_map()
        bt.verify()
        for b in range(2):
            for x, y in zip(bt.prompt_logprobs(b), want[b]):
                assert torch.equal(x, y), (s, b)


def test_admission():
    gm, Mx = cases.load_growmap(GM128), 384
    prompts = [cases.make_prompt(770 + i, n).to(DEV) for i, n in enumerate((60, 80))]
    bt = _tree(_engines(2, Mx), prompts, gm, Mx, policy="greedy", temperature=1.0, prompt_logprobs=[5, None])
    with pytest.raises(ValueError, match="first verify"):
        bt.prompt_logprobs(0)
    _decode(bt, 2)
    steady = bt.prompt_logprobs(0)
    with pytest.raises(ValueError, match="off"):
        bt.prompt_logprobs(1)
    new = cases.make_prompt(780, 64)
    bt.freeze(1)
    bt.admit(1, new.to(DEV), prompt_logprobs=7)
    with pytest.raises(ValueError, match="first verify"):
        bt.prompt_logprobs(1)
    _decode(bt, 1)
    lp, ids, top = bt.prompt_logprobs(1)
    assert ids.shape == (63, 7)
    _check_teacher_forced(lp, ids, new, _reference_logprobs(new, Mx))
    for x, y in zip(bt.prompt_logprobs(0), steady):
        assert torch.equal(x, y), "a steady slot's values are not touched"
    again = cases.make_prompt(781, 40)
    bt.freeze(1)
    bt.admit(1, again.to(DEV))                          # _PREVIOUS: the setting stays 7
    with pytest.raises(ValueError, match="first verify"):
        bt.prompt_logprobs(1)
    _decode(bt, 1)
    lp, ids, _ = bt.prompt_logprobs(1)
    assert bt.prompt_logprobs_n[1] == 7 and ids.shape == (39, 7)
    _check_teacher_forced(lp, ids, again, _reference_logprobs(again, Mx))
    bt.freeze(1)
    bt.admit(1, new.to(DEV), prompt_logprobs=None)
    _decode(bt, 1)
    with pytest.raises(ValueError, match="off"):
        bt.prompt_logprobs(1)


def _check_shape_rules(lp, ids, top, P, k, V):
    assert lp.shape == (P - 1,) and ids.shape == (P - 1, k) and top.shape == (P - 1, k)
    if P == 1:
        return
    assert bool(torch.isfinite(lp).all()) and bool(torch.isfinite(top).all())
    if k == 0:
        return
    assert bool(((ids >= 0) & (ids < V)).all())
    assert bool((top[:, :-1] >= top[:, 1:]).all()), "top lists do not increase"
    assert float(torch.logsumexp(top.double(), -1).max()) <= 1e-6, "the top probabilities sum to at most 1"
    assert bool((lp <= top[:, 0]).all())


def test_full_batch():
    gm, Mx = cases.load_growmap(GM128), 384
    S = gm["size"]
    lens = [1, 2, 17, 60, 128, 129, 200, Mx - S + 1]
    prompts = [cases.make_prompt(790 + i, n).to(DEV) for i, n in enumerate(lens)]
    bt = _tree(_engines(8, Mx), prompts, gm, Mx, policy=["spec", "greedy"] * 4, seeds=list(range(8)),
               prompt_logprobs=[20, 1, 5, 0, 20, 3, 20, 20])
    _decode(bt, 2)
    for b, P in enumerate(lens):
        lp, ids, top = bt.prompt_logprobs(b)
        _check_shape_rules(lp, ids, top, P, bt.prompt_logprobs_n[b], bt.V)


def test_prompt_logprobs_llama3_vocab():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 2."""
    import gc
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gc.collect()
    torch.cuda.empty_cache()
    gm, Mx = cases.load_growmap(GM128), 384
    engines = (GraphInferenceEngine(Mx, "random-init:llama-3.2-1b:1", device=DEV, batch_size=2),
               GraphInferenceEngineTG(Mx, "random-init:llama-3.1-8b:2", device=DEV, batch_size=2))
    g = torch.Generator().manual_seed(37)
    prompts = [torch.randint(3, 128256, (n,), generator=g).to(DEV) for n in (90, 200)]
    bt = _tree(engines, prompts, gm, Mx, seeds=[41, 42], policy=["spec", "greedy"], prompt_logprobs=[20, 3])
    _decode(bt, 2)
    assert bt.V == 128256
    for b, p in enumerate(prompts):
        lp, ids, top = bt.prompt_logprobs(b)
        _check_shape_rules(lp, ids, top, len(p), (20, 3)[b], bt.V)
