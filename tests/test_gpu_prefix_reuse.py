"""Prefix reuse on the device (sq_kv_copy_prefix, BatchTree.admit(reuse_prefix=True)).

Kernel level: the copy against torch indexing, bit for bit, at the 68m, 7B and Llama-3.1-8B (GQA) cache shapes, B = 2 and
8, n from 1 to M; every byte outside dst's rows [0, n) keeps its random sentinel bits.  BatchTree level: a decoding donor
is untouched by a reusing admission next to it, one prompt fanned out to three slots at one seed gives three identical
outputs, a reusing first verify is close to a full one (a system prefix from another slot, and a multi-turn re-admission
of a slot's own output with no copy), nothing past a donor's ready length is read, the cases that reuse nothing, and one
run at V = 128256."""
import pytest
import torch

import cases
from test_gpu_refill import DEV, F16, _engines, ops

pytestmark = pytest.mark.gpu

GM = "L40_growmaps/8x8-tree.pt"
MX = 384


def _lib():
    from sequoia_b200 import _lib as lib
    return lib


# ------------------------------------------------------------------------------------------------ kernel
class _KV:
    def __init__(self, k, v):
        self.k_cache, self.v_cache = k, v


SHAPES = {"68m": (2, 12, 64, 640), "7b": (32, 32, 128, 512), "llama3_8b_gqa": (32, 8, 128, 512)}


@pytest.mark.parametrize("B", [2, 8])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_kernel_matches_torch_indexing(shape, B):
    L, Hkv, D, M = SHAPES[shape]
    g = torch.Generator(device=DEV).manual_seed(L * Hkv + B)
    bits = [torch.randint(-32768, 32768, (L, B, Hkv, M, D), generator=g, device=DEV, dtype=torch.int32).to(torch.int16)
            for _ in range(2)]                          # random sentinel bits, NaN patterns included
    kv = _KV(bits[0].view(F16), bits[1].view(F16))
    src, dst = (1, 0) if B == 2 else (5, 2)
    for n in (1, 7, 8, 9, 255, M):
        want = [t.clone() for t in bits]
        for w in want:
            w[:, dst, :, :n] = w[:, src, :, :n]
        c0 = _lib().launch_count()
        ops().kv_copy_prefix(kv, src, dst, n)
        torch.cuda.synchronize()
        assert _lib().launch_count() == c0 + 1, "one launch for K and V"
        for got, w, name in zip(bits, want, "KV"):
            assert torch.equal(got, w), (shape, B, n, name)


def test_ops_refusal_on_the_device():
    from sequoia_b200._lib import SequoiaLibError
    k = torch.zeros(2, 2, 4, 16, 64, dtype=F16, device=DEV)
    kv = _KV(k, k.clone())
    for src, dst, n in ((0, 0, 4), (0, 2, 4), (0, 1, 0), (0, 1, 17)):
        with pytest.raises(SequoiaLibError, match="sq_kv_copy_prefix"):
            ops().kv_copy_prefix(kv, src, dst, n)


# ------------------------------------------------------------------------------------------------ BatchTree
def _tree(engines, prompts, Mx=MX, gm=GM, **kw):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    d.clear_kv()
    t.clear_kv()
    return BatchTree(d, t, [p.to(DEV) for p in prompts], cases.load_growmap(gm), max_length=Mx, max_target_seq=Mx,
                     **kw)


def _step(bt):
    bt.construct_grow_map()
    return [(v.cpu().clone(), a, term) for v, a, term in bt.verify()]


def _instrument(bt):
    """-> a record of the S target logit rows of each first verify (as the ragged forward left them) and of the launches
    of each draft prefill."""
    rec = dict(first=[], prefill=[])
    first, prefill = bt.op_target_first, bt.op_draft_prefill

    def op_target_first(seqs):
        first(seqs)
        rec["first"].append({b: bt.target_logits[b * bt.S:(b + 1) * bt.S].clone() for b in seqs})

    def op_draft_prefill(seqs):
        c0 = _lib().launch_count()
        prefill(seqs)
        rec["prefill"].append(_lib().launch_count() - c0)
    bt.op_target_first, bt.op_draft_prefill = op_target_first, op_draft_prefill
    return rec


def _admit(bt, rec, b, prompt, **kw):
    """admit() -> the launches it made outside its draft prefill"""
    c0 = _lib().launch_count()
    bt.admit(b, prompt.to(DEV), **kw)
    return _lib().launch_count() - c0 - rec["prefill"][-1]


def test_donor_untouched():
    """B = 4, seeded: slot 3 reuses 80 tokens of decoding slot 0's prompt; every other slot's outputs are the bits of
    the run whose admission reuses nothing."""
    engines = _engines(4, MX)
    prompts = [cases.make_prompt(910 + i, n) for i, n in enumerate((100, 70, 90, 60))]
    new = torch.cat([prompts[0][:80], cases.make_prompt(915, 30)])
    runs = {}
    for reuse in (False, True):
        bt = _tree(engines, prompts, seeds=[11, 12, 13, 14])
        out = [_step(bt) for _ in range(2)]
        bt.freeze(3)
        bt.admit(3, new.to(DEV), seed=99, reuse_prefix=reuse)
        assert bt.reused_prefix[3] == ((0, 80) if reuse else None)
        out += [_step(bt) for _ in range(5)]
        runs[reuse] = out
    for it, (x, y) in enumerate(zip(runs[False], runs[True])):
        for b in range(3):
            assert torch.equal(x[b][0], y[b][0]) and x[b][1:] == y[b][1:], (it, b)


def test_fan_out_one_prompt_to_three_slots():
    engines = _engines(4, MX)
    p = cases.make_prompt(920, 96)
    bt = _tree(engines, [p] + [cases.make_prompt(921 + i, 50 + 10 * i) for i in range(3)], seeds=[1, 2, 3, 4])
    _step(bt)
    for b in (1, 2, 3):
        bt.freeze(b)
    for b in (1, 2, 3):
        bt.admit(b, p.to(DEV), seed=77, reuse_prefix=True)
        assert bt.reused_prefix[b] == (0, len(p) - 1)
    for it in range(6):
        res = _step(bt)
        for b in (2, 3):
            assert torch.equal(res[b][0], res[1][0]) and res[b][1:] == res[1][1:], (it, b)


def _nan_rows(bt, d, start):
    for eng in (bt.draft, bt.target):
        kv = eng.engine.kv_cache
        kv.k_cache[:, d, :, start:] = float("nan")
        kv.v_cache[:, d, :, start:] = float("nan")


def _system_prefix_run(engines, reuse, poison=False):
    """Slot 0 decodes a system prefix + its own question one step; then both slots are frozen and slot 1 takes the same
    system prefix + another question.  Greedy, so both runs draft the same tree.  -> (tree, first-verify rows of slot 1,
    admission launches outside the prefill)"""
    sys_p = cases.make_prompt(930, 100)
    p0 = torch.cat([sys_p, cases.make_prompt(931, 20)])
    new = torch.cat([sys_p, cases.make_prompt(933, 24)])
    bt = _tree(engines, [p0, cases.make_prompt(932, 60)], policy="greedy", temperature=1.0)
    rec = _instrument(bt)
    _step(bt)
    bt.freeze(0)
    bt.freeze(1)
    if poison:
        _nan_rows(bt, 0, bt.target_kv_len[0])
    launches = _admit(bt, rec, 1, new, reuse_prefix=reuse)
    _step(bt)
    return bt, rec["first"][-1][1], launches


def test_close_to_a_full_prefill_system_prefix():
    engines = _engines(2, MX)
    plain, want, plain_launches = _system_prefix_run(engines, False)
    bt, got, launches = _system_prefix_run(engines, True)
    assert plain.reused_prefix[1] is None and bt.reused_prefix[1] == (0, 100)
    assert launches == plain_launches + 2, "one copy launch per cache"
    P, S = 124, bt.S
    assert torch.equal(bt.tokens[1, :P + S - 1].cpu(), plain.tokens[1, :P + S - 1].cpu()), "the same drafted tree"
    err = float((got.float() - want.float()).abs().max())
    print(f"system prefix: max |reused - full| first-verify logit = {err}")
    assert bool(torch.isfinite(got).all()) and err <= 0.0625, err    # measured 0.0 on an H100 80GB HBM3
    # nothing of the donor past its ready length is read: the same bits with those rows NaN
    poisoned, got_p, _ = _system_prefix_run(engines, True, poison=True)
    assert bool(torch.isfinite(got_p).all()) and torch.equal(got_p, got)


def test_close_to_a_full_prefill_multi_turn():
    """Slot 0 decodes three steps and is stopped; its own output plus a new turn goes back into slot 0: L = R_0, no copy."""
    engines = _engines(2, MX)
    runs = {}
    for reuse in (False, True):
        bt = _tree(engines, [cases.make_prompt(940, 80), cases.make_prompt(941, 60)], policy="greedy", temperature=1.0)
        rec = _instrument(bt)
        for _ in range(3):
            _step(bt)
        assert not bt.frozen[0]
        bt.freeze(0)
        R0 = bt.target_kv_len[0]
        new = torch.cat([bt.last[0][0].cpu(), cases.make_prompt(942, 16)])
        launches = _admit(bt, rec, 0, new, reuse_prefix=reuse)
        _step(bt)
        runs[reuse] = (bt, rec["first"][-1][0], launches, R0, len(new))
    plain, want, plain_launches, R0, P = runs[False]
    bt, got, launches, R0_reuse, _ = runs[True]
    assert R0 == R0_reuse and R0 >= 80
    assert bt.reused_prefix[0] == (0, R0) and plain.reused_prefix[0] is None
    assert launches == plain_launches, "a slot's own rows: no copy"
    S = bt.S
    assert torch.equal(bt.tokens[0, :P + S - 1].cpu(), plain.tokens[0, :P + S - 1].cpu()), "the same drafted tree"
    err = float((got.float() - want.float()).abs().max())
    print(f"multi-turn: max |reused - full| first-verify logit = {err}")
    assert bool(torch.isfinite(got).all()) and err <= 0.0625, err    # measured 0.0 on an H100 80GB HBM3


def test_cases_that_reuse_nothing():
    engines = _engines(2, MX)
    p = cases.make_prompt(950, 90)
    bt = _tree(engines, [p, cases.make_prompt(951, 40)], seeds=[5, 6])
    rec = _instrument(bt)
    _step(bt)
    bt.freeze(0)
    bt.freeze(1)
    # slot 0 admitted in this gap has no first verify yet: no donor for slot 1
    _admit(bt, rec, 0, cases.make_prompt(952, 70), seed=7, reuse_prefix=True)
    assert bt.reused_prefix[0] is None
    with_flag = _admit(bt, rec, 1, cases.make_prompt(952, 70), seed=8, reuse_prefix=True)
    assert bt.reused_prefix[1] is None
    _step(bt)
    bt.freeze(1)
    # prompt_logprobs on: L = 0 although slot 0 now holds the prefix
    _admit(bt, rec, 1, cases.make_prompt(952, 70), seed=8, reuse_prefix=True, prompt_logprobs=0)
    assert bt.reused_prefix[1] is None
    _step(bt)
    bt.freeze(1)
    # reuse_prefix=False: the launches of an admission that finds nothing
    without = _admit(bt, rec, 1, cases.make_prompt(953, 70), seed=8, prompt_logprobs=None)
    assert bt.reused_prefix[1] is None and without == with_flag
    _step(bt)


def test_prefix_reuse_llama3_vocab():
    """V = 128256 (random-init Llama 3 1B -> 8B), B = 2: slot 1 takes slot 0's first 150 tokens."""
    import gc
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gc.collect()
    torch.cuda.empty_cache()
    engines = (GraphInferenceEngine(MX, "random-init:llama-3.2-1b:1", device=DEV, batch_size=2),
               GraphInferenceEngineTG(MX, "random-init:llama-3.1-8b:2", device=DEV, batch_size=2))
    g = torch.Generator().manual_seed(57)
    p0, p1 = (torch.randint(3, 128256, (n,), generator=g) for n in (180, 90))
    bt = _tree(engines, [p0, p1], seeds=[41, 42], policy=["spec", "greedy"])
    rec = _instrument(bt)
    _step(bt)
    bt.freeze(1)
    new = torch.cat([p0[:150], torch.randint(3, 128256, (40,), generator=g)])
    bt.admit(1, new.to(DEV), seed=43, reuse_prefix=True)
    assert bt.V == 128256 and bt.reused_prefix[1] == (0, 150)
    for _ in range(2):
        res = _step(bt)
    assert bool(torch.isfinite(rec["first"][-1][1]).all())
    assert torch.equal(res[1][0][:190], new) and len(res[1][0]) > 190
