"""FP8 (E4M3) target weights on the GPU.  By definition (ops.dequantize_fp8) the FP8 GEMM computes the fp16 GEMM of the
dequantized matrix W' = fp16(fp16(q) * s), so every check compares against the float64 product with W', the fp16
engine loaded with W', or the CPU oracle on W'."""
import contextlib
import os

import pytest
import torch

import cases
from oracle import sequoia_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16 = torch.float16
SENT = -1234.0

# every gemm_fp8_kernel instance sq_gemm_fp8.cu's run_tile can launch: (64-row weight tiles per CTA, K splits); each runs
# at R = 64 (tiles of <= 64 rows) and R = 128
FP8_INSTANCES = [(w, s) for w in (2, 3) for s in (1, 2, 3, 4)]
# (N, K) of the layer projections: Llama-2-7B qkv / o / gate_up / down, 13B down, Llama-3.1-8B qkv, the test targets
MODEL_SHAPES = [(12288, 4096), (4096, 4096), (22016, 4096), (4096, 11008), (5120, 13824), (6144, 4096),
                (1536, 512), (512, 512), (2048, 512), (512, 1024), (1024, 512)]
ROWS = (1, 7, 64, 65, 127, 128, 129, 300)


def ops():
    from sequoia_b200 import ops as _ops
    return _ops


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


def _fp16_ulp(x):
    return torch.pow(2.0, torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -14))) - 10)


def _reference(a, wd):
    """float64 A W'^T and the bound of an fp16-out GEMM with fp32 accumulation over K (as in test_gpu_kernels.py): 1 fp16
    ulp of the exact value plus K 2^-24 (|A| |W'|^T)."""
    a64, w64 = a.double(), wd.double()
    ref = a64 @ w64.t()
    return ref, _fp16_ulp(ref) + a.shape[1] * 2.0 ** -24 * (a64.abs() @ w64.abs().t())


def _assert_within(got, ref, tol, what):
    g = got.double()
    assert bool(torch.isfinite(g).all()), f"{what}: non-finite outputs"
    ratio = ((g - ref).abs() / tol).max().item()
    nbad = int(((g - ref).abs() > tol).sum())
    assert nbad == 0, f"{what}: {nbad}/{g.numel()} elements outside the bound (worst {ratio:.2f} x tol)"
    return ratio


def _assert_canary(buf, n, N, what):
    keep = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    keep[:n, :N] = False
    assert bool((buf[keep] == SENT).all()), f"{what}: wrote outside rows [0, {n}) x columns [0, {N})"


def _weights(N, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = torch.randn(N, K, generator=g, device=DEV) * 0.02
    w[::5] *= 8                                                          # channels of different ranges
    q, s = ops().quantize_fp8(w.to(F16))
    return q, s, ops().dequantize_fp8(q, s)


def _run_case(N, K, instance, seed, rows=ROWS):
    """One plan per case (forced instance or the default choice): a 300-row activation buffer, output at ldc = N + 64
    with sentinel rows and columns around it; every n of `rows` at row 0 into the plan's buffer, and at activation row
    37 into an output override."""
    q, s, wd = _weights(N, K, seed)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    n_max = 340
    a = (torch.randn(n_max, K, generator=g, device=DEV) * 0.5).to(F16)
    err = torch.zeros(4, dtype=torch.int32, device=DEV)
    c = torch.full((n_max + 8, N + 64), SENT, dtype=F16, device=DEV)
    env = {"SQ_GEMM_FP8_FORCE": "%d,%d" % instance} if instance else {}
    with _env(**env):
        plan = ops().GemmFp8Plan(a, q, s, c, err)
    if instance:
        assert plan.info()[:2] == instance, f"forced {instance}, plan {plan.info()}"
    worst = 0.0
    ref, tol = _reference(a, wd)
    for n in rows:
        what = f"fp8 gemm {plan.info()} N={N} K={K} n={n}"
        c.fill_(SENT)
        plan.run(n)
        torch.cuda.synchronize()
        assert err.tolist() == [0, 0, 0, 0], f"{what}: pipeline watchdog fired"
        worst = max(worst, _assert_within(c[:n, :N], ref[:n], tol[:n], what))
        _assert_canary(c, n, N, what)
    for n in (rows[0], rows[-1]):
        row0 = 37 if n + 37 <= n_max else 0
        out = torch.full((n + 8, N + 64), SENT, dtype=F16, device=DEV)
        c.fill_(SENT)
        plan.run(n, a_row0=row0, out=out)
        torch.cuda.synchronize()
        what = f"fp8 gemm {plan.info()} N={N} K={K} n={n} a_row0={row0}"
        assert err.tolist() == [0, 0, 0, 0], f"{what}: pipeline watchdog fired"
        worst = max(worst, _assert_within(out[:n, :N], ref[row0:row0 + n], tol[row0:row0 + n], what))
        _assert_canary(out, n, N, what)
        assert bool((c == SENT).all()), f"{what}: the plan's own buffer was written despite the output override"
    return worst, plan


@pytest.mark.parametrize("instance", FP8_INSTANCES, ids=lambda v: "nwg%d_split%d" % v)
def test_fp8_gemm_every_instance(instance):
    """Every instance, forced, at a ragged tile count (N / 64 not a multiple of NWG), at K with fewer K blocks per split than
    ring stages and with a ring that wraps several times, for every row count of ROWS."""
    nwg, split = instance
    worst = 0.0
    for N in (64 * (2 * nwg + 1), 64 * 4 * nwg):
        for K in (64 * split, 64 * split * 3, 64 * 40):
            w, _ = _run_case(N, K, instance, seed=N + K)
            worst = max(worst, w)
    cases.log_line("fp8_gemm.log", f"instance {instance}: worst err/bound {worst:.3f}")


@pytest.mark.parametrize("N,K", MODEL_SHAPES, ids=lambda v: str(v))
def test_fp8_gemm_model_shapes(N, K):
    worst, plan = _run_case(N, K, None, seed=N + 3 * K)
    cases.log_line("fp8_gemm.log", f"N={N} K={K} plan {plan.info()}: worst err/bound {worst:.3f}")


def test_fp8_gemm_dequantizes_bit_exactly():
    """With A = the identity, C = W'^T exactly (one nonzero product per sum): the kernel's cvt + HMUL2 gives the bit pattern
    of dequantize_fp8 for every weight, including subnormal products and the channels of the extreme scales."""
    N, K = 256, 128
    q, s, wd = _weights(N, K, 11)
    s[3] = 2.0 ** -24                                                    # subnormal products
    s[4] = 1.0
    q[5] = torch.arange(256, dtype=torch.int32).remainder(127).to(torch.uint8)[:K].view(torch.float8_e4m3fn).to(DEV)
    wd = ops().dequantize_fp8(q, s)
    a = torch.eye(K, dtype=F16, device=DEV)
    c = torch.zeros(K, N, dtype=F16, device=DEV)
    plan = ops().GemmFp8Plan(a, q.contiguous(), s, c)
    plan.run(K)
    torch.cuda.synchronize()
    assert torch.equal(c.t().contiguous().view(torch.int16), wd.view(torch.int16))


def test_fp8_gemm_bound_sees_a_wrong_scale_and_a_dropped_k_block():
    """Negative controls: the bound of the instance sweep rejects a reference with one channel's scale 6% off, and one
    without the last K block."""
    N, K, n = 512, 64 * 12, 128
    q, s, wd = _weights(N, K, 21)
    a = (torch.randn(n, K, generator=torch.Generator(device=DEV).manual_seed(5), device=DEV) * 0.5).to(F16)
    c = torch.zeros(n, N, dtype=F16, device=DEV)
    plan = ops().GemmFp8Plan(a, q, s, c)
    plan.run(n)
    torch.cuda.synchronize()
    ref, tol = _reference(a, wd)
    _assert_within(c, ref, tol, "exact reference")
    s_bad = s.clone()
    s_bad[77] = s_bad[77] * 1.0625
    bad, _ = _reference(a, ops().dequantize_fp8(q, s_bad))
    frac = ((c[:, 77].double() - bad[:, 77]).abs() > tol[:, 77]).float().mean().item()
    assert frac >= 0.9, f"a wrong channel scale: only {frac:.2%} of that channel's outputs leave the bound"
    dropped = ref - _reference(a[:, K - 64:], wd[:, K - 64:])[0]
    frac = ((c.double() - dropped).abs() > tol).float().mean().item()
    assert frac >= 0.9, f"a dropped K block: only {frac:.2%} of the outputs leave the bound"


def test_fp8_gemm_graph_replays_are_bit_identical():
    for instance in ((2, 4), (3, 1)):
        q, s, _ = _weights(4096, 4096, 31)
        a = (torch.randn(128, 4096, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV) * 0.5).to(F16)
        c = torch.zeros(128, 4096, dtype=F16, device=DEV)
        with _env(SQ_GEMM_FP8_FORCE="%d,%d" % instance):
            plan = ops().GemmFp8Plan(a, q, s, c)
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            plan.run(128)
        torch.cuda.current_stream().wait_stream(st)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            plan.run(100)
            plan.run(28, a_row0=100, out=c[100:])
        c.zero_()
        graph.replay()
        first = c.clone()
        c.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(first, c) and bool((first != 0).any()), instance


# ------------------------------------------------------------------------------------------------ engines
_PROJ = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


def _dequantized_state_dict(sd):
    """the state dict an FP8 engine computes with: every layer projection replaced by W' (quantized on the device, as the
    engine quantizes at load)"""
    out = {}
    for k, v in sd.items():
        if any(k.endswith(p + ".weight") for p in _PROJ):
            q, s = ops().quantize_fp8(v.to(DEV, F16))
            out[k] = ops().dequantize_fp8(q, s).cpu()
        else:
            out[k] = v
    return out


def test_fp8_runner_weights_resident_and_freed():
    from sequoia_b200.model import LlamaRunner
    cfg, w = cases.model_weights("target")
    r16 = LlamaRunner({"config": cfg, "state_dict": w}, 128, device=DEV)
    r8 = LlamaRunner({"config": cfg, "state_dict": w}, 128, device=DEV, weight_format="fp8")
    proj16 = sum(2 * ly[k].numel() for ly in r16.layers for k in r16.PROJECTIONS)
    rows = sum(ly[k].shape[0] for ly in r16.layers for k in r16.PROJECTIONS)
    assert r16.weight_bytes() - r8.weight_bytes() == proj16 // 2 - 2 * rows
    for ly in r8.layers:
        assert not any(k in ly for k in r8.PROJECTIONS), "no fp16 copy of a quantized projection stays resident"


@pytest.mark.parametrize("key", ["target", "target_gqa"])
def test_fp8_engine_logits_vs_fp16_engine_on_dequantized_weights(key):
    """A prefix forward then the tree rows of the 8x8 growmap: the FP8 engine against the fp16 engine loaded with W'
    (same arithmetic up to the fp32 summation order of the projections)."""
    from sequoia_b200.engine import GraphInferenceEngineTG
    cfg, w = cases.model_weights(key)
    M = 192
    gm = cases.load_growmap("L40_growmaps/8x8-tree.pt")
    S, P = gm["size"], 90
    tot = P + S - 1
    prompt = cases.make_prompt(77, tot)
    win = O.window_mask(O.build_full_attn_mask(M, gm["mask"]), M, tot)
    pos = torch.zeros(M, dtype=torch.long)
    pos[:P] = torch.arange(P)
    pos[P:tot] = gm["depth"][1:] + P - 1
    sto = torch.arange(M)
    e8 = GraphInferenceEngineTG(M, {"config": cfg, "state_dict": w}, device=DEV, weight_format="fp8")
    e16 = GraphInferenceEngineTG(M, {"config": cfg, "state_dict": _dequantized_state_dict(w)}, device=DEV)
    for (a, b) in ((0, P), (P, tot)):
        m = win[a:b, :b][None, None].to(DEV)
        args = (prompt[a:b].unsqueeze(0).to(DEV), sto[a:b].to(DEV), pos[a:b].unsqueeze(0).to(DEV), m)
        got, ref = e8.inference(*args).float(), e16.inference(*args).float()
        rel = ((got - ref).abs() / ref.abs().amax(-1, keepdim=True)).max().item()
        assert rel < 4e-3, f"{key} rows [{a},{b}): logits rel err {rel}"
    assert e8.engine.runner.gemm_err.tolist() == [0, 0, 0, 0]


def test_fp8_7b_shaped_layer_logits_vs_fp16_path_and_fp32():
    """test_gpu_kernels.py's 7B-shaped layer criterion, with the fp16 engine on W' as the reference path: the FP8 engine
    must be at least as close to the fp32 logits on W' as the fp16 path, and within the sum of both distances of it."""
    from sequoia_b200.engine import GraphInferenceEngineTG
    cfg = O.LlamaCfg(hidden_size=4096, intermediate_size=11008, num_hidden_layers=1, num_attention_heads=32,
                     num_key_value_heads=32, vocab_size=cases.V, rms_norm_eps=1e-5)
    w = O.init_llama_weights(cfg, 909)
    wd = _dequantized_state_dict(w)
    gm = cases.load_growmap("A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt")
    S, P, M = gm["size"], 64, 256
    tot = P + S - 1
    prompt = cases.make_prompt(78, tot)
    win = O.window_mask(O.build_full_attn_mask(M, gm["mask"]), M, tot)
    pos = torch.zeros(M, dtype=torch.long)
    pos[:P] = torch.arange(P)
    pos[P:tot] = gm["depth"][1:] + P - 1
    sto = torch.arange(M)
    orc32 = O.EngineOracle(O.LlamaOracle(cfg, {k: v.float() for k, v in wd.items()}, M, "TG", dtype=torch.float32))
    e16 = GraphInferenceEngineTG(M, {"config": cfg, "state_dict": wd}, device=DEV)
    e8 = GraphInferenceEngineTG(M, {"config": cfg, "state_dict": w}, device=DEV, weight_format="fp8")
    ours_vs_ref = ours_vs_32 = ref_vs_32 = 0.0
    for (a, b, m) in ((0, P, win[:P, :P][None, None]), (P, tot, win[P:tot, :tot][None, None])):
        ex = orc32.inference(prompt[a:b].unsqueeze(0), sto[a:b], pos[a:b].unsqueeze(0), m.float())
        args = (prompt[a:b].unsqueeze(0).to(DEV), sto[a:b].to(DEV), pos[a:b].unsqueeze(0).to(DEV), m.to(DEV))
        ref = e16.inference(*args).float().cpu()
        got = e8.inference(*args).float().cpu()
        scale = ex.abs().amax(dim=-1, keepdim=True)
        ours_vs_ref = max(ours_vs_ref, ((got - ref).abs() / scale).max().item())
        ours_vs_32 = max(ours_vs_32, ((got - ex).abs() / scale).max().item())
        ref_vs_32 = max(ref_vs_32, ((ref - ex).abs() / scale).max().item())
    cases.log_line("logit_err.log", f"FP8 7B-shaped layer, rows {tot}: ours vs fp16 path on W' {ours_vs_ref:.3e}; vs fp32 "
                   f"on W': ours {ours_vs_32:.3e}, fp16 path {ref_vs_32:.3e}")
    assert e8.engine.runner.gemm_err.tolist() == [0, 0, 0, 0]
    assert ours_vs_32 <= 1.05 * ref_vs_32, f"further from the exact logits ({ours_vs_32:.3e}) than the fp16 path ({ref_vs_32:.3e})"
    assert ours_vs_ref <= ours_vs_32 + ref_vs_32 and ours_vs_ref < 3e-3, ours_vs_ref


@pytest.mark.parametrize("name", ["spec_8x8", "greedy_4x4", "spec_a100_128"])
def test_fp8_target_teacher_forced_vs_oracle_on_dequantized_weights(name, monkeypatch):
    """test_gpu_decode.py's teacher-forced lock-step (same fork rule) with an FP8 target, the oracle's target on W'."""
    import test_gpu_decode as D
    from Engine.Engine import GraphInferenceEngine, GraphInferenceEngineTG
    gm_name, mode, dkey, tkey, M, pseed, plen, iters, rng_seed = cases.DECODE_CASES[name]
    tcfg, tw = cases.model_weights(tkey)
    fkey = tkey + "_fp8_dequantized"
    monkeypatch.setitem(cases._wcache, fkey, (tcfg, _dequantized_state_dict(tw)))

    def engines(dk, tk, M_):
        dcfg, dw = cases.model_weights(dk)
        return (GraphInferenceEngine(M_, {"config": dcfg, "state_dict": dw}, device=DEV),
                GraphInferenceEngineTG(M_, {"config": tcfg, "state_dict": tw}, device=DEV, weight_format="fp8"))

    monkeypatch.setattr(D, "_engines", engines)
    table = {name: (gm_name, mode, dkey, fkey, M, pseed, plen, iters, rng_seed)}
    same, total, forks, done, worst = D._teacher_forced(name, table)
    frac = same / max(total, 1)
    cases.log_line("teacher_forced.log", f"fp8 target {name} identical={same}/{total} frac={frac:.4f} "
                   f"accept_forks={forks} iters={done} logit_rel={worst:.3e}")
    assert frac >= D.MIN_IDENTICAL, f"{name}: only {frac:.3f} of the drafted nodes identical to the oracle"
    assert worst <= D.DRAFT_LOGIT_TOL, f"{name}: logits differ from the oracle's by {worst:.2e}"
    assert done >= 1


def _bt_engines(B, fmt="fp8"):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    dcfg, dw = cases.model_weights("draft")
    tcfg, tw = cases.model_weights("target")
    return (GraphInferenceEngine(256, {"config": dcfg, "state_dict": dw}, device=DEV, batch_size=B),
            GraphInferenceEngineTG(256, {"config": tcfg, "state_dict": tw}, device=DEV, batch_size=B, weight_format=fmt))


def test_fp8_batch_tree_b2_vs_lone_trees():
    """BatchTree at B = 2 on an FP8 target against a lone FP8 SpecTree per prompt (same draws): the first step identical,
    at least 95% of the committed tokens after that."""
    from sequoia_b200.batch import BatchTree, draw_random
    from sequoia_b200.tree import SpecTree, clear_runtimes
    gm, Mx, iters, V = cases.load_growmap("L40_growmaps/8x8-tree.pt"), 256, 5, cases.V
    prompts = [cases.make_prompt(60 + i, n) for i, n in enumerate((100, 72))]
    with _env(SQ_DRAFT_ATTN=0, SQ_ATTN_SPLITS=1):
        d1, t1 = _bt_engines(1)
        d2, t2 = _bt_engines(2)
    noise = torch.empty(iters, 2, V, dtype=F16).exponential_(1.0, generator=torch.Generator().manual_seed(9)).to(DEV)
    torch.manual_seed(4)
    bt = BatchTree(d2, t2, prompts, gm, policy="spec", temperature=0.6, top_p=1.0, max_length=Mx)
    bt.external_noise = noise
    steps = []
    for _ in range(iters):
        bt.construct_grow_map()
        steps.append([v.cpu() for v, _, _ in bt.verify()])
    torch.manual_seed(4)
    r, rand = draw_random(prompts, Mx, gm["size"], V)
    same = total = 0
    for b, p in enumerate(prompts):
        clear_runtimes()
        tree = SpecTree(d1, t1, p.to(DEV), temperature=0.6, top_p=1.0, max_length=Mx, max_target_seq=Mx, device=DEV,
                        vocab_size=V, grow_map=gm)
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
    assert total > 0 and same >= 0.95 * total, (same, total)
    assert t2.engine.runner.gemm_err.tolist() == [0, 0, 0, 0]


def test_fp8_batch_two_replays_one_sync(monkeypatch):
    from sequoia_b200 import _lib
    from sequoia_b200.batch import BatchTree
    gm = cases.load_growmap("L40_growmaps/8x8-tree.pt")
    draft, target = _bt_engines(2)
    torch.manual_seed(1)
    bt = BatchTree(draft, target, [cases.make_prompt(50, 60), cases.make_prompt(51, 67)], gm, policy="spec",
                   temperature=0.6, top_p=1.0, max_length=256)
    for _ in range(2):
        bt.construct_grow_map()
        bt.verify()
    syncs = []
    real_sync = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: syncs.append(1))
    r0 = dict(bt.replays)
    c0 = _lib.launch_count()
    for _ in range(3):
        bt.construct_grow_map()
        bt.verify()
    monkeypatch.undo()
    torch.cuda.synchronize()
    assert bt.replays["draft"] - r0["draft"] == 3 and bt.replays["steady"] - r0.get("steady", 0) == 3
    assert len(syncs) == 3, "one host sync per step"
    assert _lib.launch_count() == c0, "a steady step launches only through graph replays"
