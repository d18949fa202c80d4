"""The 7B verify projections that LlamaRunner runs on sq_gemm plans besides gate_up (model.VERIFY_PLANS: down_proj, on
the split-K tile of the deep ring, gemm_tn_deep_kernel): float64 bounds with sentinel canaries at 1, 97, 127 and 128
rows, graph-replay bit-identity, negative controls for the bound, both deep-ring instances at small shapes, and a
7B-shaped layer on those routes against the all-cuBLASLt route."""
import pytest
import torch

import cases
from oracle import sequoia_oracle as O
from sequoia_b200 import model
from test_gpu_kernels import DEV, F16, SENT, _assert_canary, _assert_within, _env, _gemm_reference, _log, ops

pytestmark = pytest.mark.gpu

# runner key: (N, K) of Llama-2-7B
SHAPES = {"wqkv": (12288, 4096), "wo": (4096, 4096), "wd": (4096, 11008)}
ROUTED = [k for k in SHAPES if k in model.VERIFY_PLANS]
ROWS = (1, 97, 127, 128)
DEEP_STAGES = {64: 8, 128: 6}     # ring depth of gemm_tn_deep_kernel per BN


def _inputs(N, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = (torch.randn(136, K, generator=g, device=DEV) * 0.5).to(F16)
    w = (torch.randn(N, K, generator=g, device=DEV) * 0.02).to(F16)
    return a, w


def test_routed_plans_run_the_measured_tile():
    """Each routed projection's plan runs the tile VERIFY_PLANS names; a split-K tile runs on the deep ring."""
    assert ROUTED, "no 7B verify projection is routed to sq_gemm"
    for k in ROUTED:
        N, K = SHAPES[k]
        a = torch.zeros(128, K, dtype=F16, device=DEV)
        plan = ops().GemmPlan(a, torch.zeros(N, K, dtype=F16, device=DEV), torch.zeros(128, N, dtype=F16, device=DEV))
        bn, split, st = plan.info()
        assert (bn, split) == model.VERIFY_PLANS[k], (k, plan.info())
        if split > 1:
            assert st % 100 == DEEP_STAGES[bn], (k, plan.info())


@pytest.mark.parametrize("key", ROUTED)
def test_routed_projection_within_float64_bound(key):
    """The plan's tile at n = 1, 97, 127, 128: every element within the float64 bound of an fp16-out, fp32-accumulate
    GEMM and nothing written outside [:n, :N]; likewise for n rows read at activation row 3 into an output override."""
    N, K = SHAPES[key]
    a, w = _inputs(N, K, 3 * N + K)
    err = torch.zeros(4, dtype=torch.int32, device=DEV)
    c = torch.full((136, N + 64), SENT, dtype=F16, device=DEV)
    plan = ops().GemmPlan(a, w, c, err)
    ref, tol = _gemm_reference(a[:128], w)
    worst = 0.0
    for n in ROWS:
        what = f"{key} {plan.info()} n={n}"
        c.fill_(SENT)
        plan.run(n)
        torch.cuda.synchronize()
        assert err.tolist() == [0, 0, 0, 0], f"{what}: pipeline watchdog fired"
        worst = max(worst, _assert_within(c[:n, :N], ref[:n], tol[:n], what))
        _assert_canary(c, n, N, what)
        out = torch.full((n + 8, N + 64), SENT, dtype=F16, device=DEV)
        plan.run(n, a_row0=3, out=out)
        torch.cuda.synchronize()
        _assert_within(out[:n, :N], *_gemm_reference(a[3:3 + n], w), what + " at row 3")
        _assert_canary(out, n, N, what + " at row 3")
    _log(f"verify route {key} (N={N} K={K}) tile {plan.info()}: worst {worst:.2f} x tol")


@pytest.mark.parametrize("key", ROUTED)
def test_routed_graph_replays_are_bit_identical(key):
    """Two replays of a captured plan run, and an eager run, give the same bits."""
    N, K = SHAPES[key]
    a, w = _inputs(N, K, 17)
    err = torch.zeros(4, dtype=torch.int32, device=DEV)
    c = torch.zeros(136, N, dtype=F16, device=DEV)
    plan = ops().GemmPlan(a, w, c, err)
    plan.run(128)
    torch.cuda.synchronize()
    eager = c.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.run(128)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.run(128)
    outs = []
    for _ in range(2):
        c.zero_()
        g.replay()
        torch.cuda.synchronize()
        outs.append(c.clone())
    assert err.tolist() == [0, 0, 0, 0]
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], eager) and bool(eager[:128].abs().sum() > 0)


@pytest.mark.parametrize("key", ROUTED)
def test_bound_rejects_a_dropped_k_block_or_split_partial(key):
    """Negative controls on the routed tile: against a reference missing one 64-wide k-block, and (split-K tile) one
    missing a whole split's partial sum, most outputs fall outside the bound."""
    N, K = SHAPES[key]
    a, w = _inputs(N, K, 23)
    err = torch.zeros(4, dtype=torch.int32, device=DEV)
    c = torch.zeros(136, N, dtype=F16, device=DEV)
    plan = ops().GemmPlan(a, w, c, err)
    plan.run(128)
    torch.cuda.synchronize()
    ref, tol = _gemm_reference(a[:128], w)
    _assert_within(c[:128], ref, tol, "control run")
    got = c[:128].double()
    _, split, _ = plan.info()
    drops = [(64 * 37, 64 * 38)]
    if split > 1:
        drops.append((K - K // split, K))
    for k0, k1 in drops:
        part = a[:128, k0:k1].double() @ w[:, k0:k1].double().t()
        bad = ((got - (ref - part)).abs() > tol).double().mean().item()
        assert bad > 0.5, f"{key}: dropping k [{k0}, {k1}) left {1 - bad:.1%} of the outputs inside the bound"


@pytest.mark.parametrize("bn", sorted(DEEP_STAGES))
@pytest.mark.parametrize("K", [128, 640, 4096 + 128])
def test_deep_ring_instances_within_float64_bound(bn, K):
    """Both gemm_tn_deep_kernel instances (forced "bn,2,1,1"), N = 4 BN: K splits of 1 k-block (shorter than the ring),
    5 and 33; row counts around the split's 64-row reduction share; canaries around the output; rows read at an
    activation offset into an output override."""
    N = 4 * bn
    a, w = _inputs(N, K, bn + K)
    err = torch.zeros(4, dtype=torch.int32, device=DEV)
    c = torch.full((136, N + 64), SENT, dtype=F16, device=DEV)
    with _env(SQ_GEMM_FORCE=f"{bn},2,1,1"):
        plan = ops().GemmPlan(a, w, c, err)
    assert plan.info() == (bn, 2, DEEP_STAGES[bn] + 100), plan.info()
    ref, tol = _gemm_reference(a[:128], w)
    for n in (1, 63, 64, 65, 128):
        what = f"deep bn={bn} K={K} n={n}"
        c.fill_(SENT)
        plan.run(n)
        torch.cuda.synchronize()
        assert err.tolist() == [0, 0, 0, 0], f"{what}: pipeline watchdog fired"
        _assert_within(c[:n, :N], ref[:n], tol[:n], what)
        _assert_canary(c, n, N, what)
        out = torch.full((n + 8, N + 64), SENT, dtype=F16, device=DEV)
        plan.run(n, a_row0=7, out=out)
        torch.cuda.synchronize()
        _assert_within(out[:n, :N], *_gemm_reference(a[7:7 + n], w), what + " at row 7")
        _assert_canary(out, n, N, what + " at row 7")


def test_7b_layer_on_the_routed_projections_is_as_close_to_fp32_as_cublas():
    """One 7B-shaped decoder layer (plus lm_head), prefix rows then the 127 tree rows of config 2, through the engine on
    its verify routes (gate_up and the VERIFY_PLANS projections on sq_gemm plans) and with every layer projection on
    cuBLASLt: the routed logits are no further from the fp32 exact result than the cuBLASLt route's."""
    from sequoia_b200.engine import GraphInferenceEngineTG
    cfg = O.LlamaCfg(hidden_size=4096, intermediate_size=11008, num_hidden_layers=1, num_attention_heads=32,
                     num_key_value_heads=32, vocab_size=cases.V, rms_norm_eps=1e-5)
    w = O.init_llama_weights(cfg, 911)
    gm = cases.load_growmap("A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt")
    S, P, M = gm["size"], 64, 256
    tot = P + S - 1
    prompt = cases.make_prompt(83, tot)
    win = O.window_mask(O.build_full_attn_mask(M, gm["mask"]), M, tot)
    pos = torch.zeros(M, dtype=torch.long)
    pos[:P] = torch.arange(P)
    pos[P:tot] = gm["depth"][1:] + P - 1
    sto = torch.arange(M)
    orc32 = O.EngineOracle(O.LlamaOracle(cfg, {k: v.float() for k, v in w.items()}, M, "TG", dtype=torch.float32))
    routed = GraphInferenceEngineTG(M, {"config": cfg, "state_dict": w}, device=DEV)
    plain = GraphInferenceEngineTG(M, {"config": cfg, "state_dict": w}, device=DEV)
    ly = routed.engine.runner.layers[0]
    for k in ROUTED + ["wgu"]:
        assert k + "_plan" in ly, f"the 7B verify route must run {k} on sq_gemm"
    for k in [k for k in plain.engine.runner.layers[0] if k.endswith("_plan")]:
        plain.engine.runner.layers[0].pop(k)
    d_routed = d_plain = 0.0
    for (a, b, m) in ((0, P, win[:P, :P][None, None]), (P, tot, win[P:tot, :tot][None, None])):
        ex = orc32.inference(prompt[a:b].unsqueeze(0), sto[a:b], pos[a:b].unsqueeze(0), m.float())
        args = (prompt[a:b].unsqueeze(0).to(DEV), sto[a:b].to(DEV), pos[a:b].unsqueeze(0).to(DEV), m.to(DEV))
        got_r = routed.inference(*args).float().cpu()
        got_p = plain.inference(*args).float().cpu()
        scale = ex.abs().amax(dim=-1, keepdim=True)
        d_routed = max(d_routed, ((got_r - ex).abs() / scale).max().item())
        d_plain = max(d_plain, ((got_p - ex).abs() / scale).max().item())
    _log(f"7B-shaped layer, {tot} rows, routes {ROUTED} + gate_up: max rel logit err vs fp32 {d_routed:.3e}, "
         f"cuBLASLt route {d_plain:.3e}")
    assert int(routed.engine.runner.gemm_err.abs().sum()) == 0
    assert d_routed <= 1.05 * d_plain, f"verify route further from fp32 ({d_routed:.3e}) than cuBLASLt ({d_plain:.3e})"
