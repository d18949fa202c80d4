"""The weight-streaming GEMM (csrc/sq_gemm.cu) at the Llama-2-7B verify shapes, on the tiles the library picks for them:
float64 bounds with sentinel canaries, the fused SwiGLU epilogue against the same kernel unfused + sq_silu_mul, graph
replay determinism, negative controls for the bound, and a 7B-shaped layer on the verify routes of LlamaRunner."""
import pytest
import torch

import cases
from oracle import sequoia_oracle as O
from test_gpu_kernels import DEV, F16, SENT, _assert_canary, _assert_within, _env, _gemm_reference, _log, ops

pytestmark = pytest.mark.gpu

# projection: (N, K, SwiGLU epilogue) of Llama-2-7B
SHAPES = {"qkv": (12288, 4096, False), "o_proj": (4096, 4096, False), "gate_up": (22016, 4096, True),
          "down_proj": (4096, 11008, False), "lm_head": (32000, 4096, False)}
ROWS = (1, 97, 127, 128)


def _inputs(N, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = (torch.randn(136, K, generator=g, device=DEV) * 0.5).to(F16)
    w = (torch.randn(N, K, generator=g, device=DEV) * 0.02).to(F16)
    return a, w


@pytest.mark.parametrize("name", list(SHAPES))
def test_verify_shape_within_float64_bound(name):
    """Each 7B verify projection on its picked tile, at n = 1, 97, 127, 128 rows: every element within the float64 bound
    of an fp16-out, fp32-accumulate GEMM, nothing written outside [:n, :N]; likewise for n rows read at activation row 5
    into an output override.  gate_up runs as the plain GEMM on [gate; up] here (its
    fused epilogue is checked against it below)."""
    N, K, _ = SHAPES[name]
    a, w = _inputs(N, K, N + K)
    err = torch.zeros(4, dtype=torch.int32, device=DEV)
    c = torch.full((136, N + 64), SENT, dtype=F16, device=DEV)
    plan = ops().GemmPlan(a, w, c, err)
    ref, tol = _gemm_reference(a[:128], w)
    for n in ROWS:
        what = f"{name} {plan.info()} n={n}"
        c.fill_(SENT)
        plan.run(n)
        torch.cuda.synchronize()
        assert err.tolist() == [0, 0, 0, 0], f"{what}: pipeline watchdog fired"
        worst = _assert_within(c[:n, :N], ref[:n], tol[:n], what)
        _assert_canary(c, n, N, what)
        out = torch.full((n + 8, N + 64), SENT, dtype=F16, device=DEV)
        plan.run(n, a_row0=5, out=out)
        torch.cuda.synchronize()
        _assert_within(out[:n, :N], *_gemm_reference(a[5:5 + n], w), what + " at row 5")
        _assert_canary(out, n, N, what + " at row 5")
    _log(f"verify GEMM {name} (N={N} K={K}) tile {plan.info()}: worst {worst:.2f} x tol")


def test_gate_up_fused_swiglu_is_bit_identical_to_unfused():
    """The 7B gate_up plan LlamaRunner builds (SwiGLU fused, interleaved weights) against the same tile run as a plain
    GEMM followed by sq_silu_mul: bit-identical at every verify row count, including into an output override at a row
    offset."""
    N, K, _ = SHAPES["gate_up"]
    I = N // 2
    a, w = _inputs(N, K, 7)
    wi = ops().interleave_gate_up(w[:I], w[I:])
    err = torch.zeros(4, dtype=torch.int32, device=DEV)
    act = torch.full((136, I + 64), SENT, dtype=F16, device=DEV)
    gu = torch.zeros(136, N, dtype=F16, device=DEV)
    want = torch.zeros(136, I, dtype=F16, device=DEV)
    fused = ops().GemmPlan(a, wi, act, err, swiglu=True)
    bn, split, st = fused.info()
    with _env(SQ_GEMM_FORCE=f"{bn},{split},{st // 100}"):
        plain = ops().GemmPlan(a, wi, gu, err)
    assert plain.info() == fused.info() and split == 1
    for n in ROWS:
        act.fill_(SENT)
        fused.run(n)
        plain.run(n)
        ops().silu_mul(gu, want, n, interleaved=True)
        torch.cuda.synchronize()
        assert err.tolist() == [0, 0, 0, 0]
        assert torch.equal(act[:n, :I], want[:n]), f"fused SwiGLU != GEMM + silu_mul at n={n}"
        _assert_canary(act, n, I, f"fused gate_up n={n}")
        out = torch.full((n + 4, I + 64), SENT, dtype=F16, device=DEV)
        fused.run(n, a_row0=3, out=out)
        plain.run(n + 3)
        ops().silu_mul(gu, want, n + 3, interleaved=True)
        torch.cuda.synchronize()
        assert torch.equal(out[:n, :I], want[3:3 + n]), f"fused SwiGLU at row 3 != GEMM + silu_mul, n={n}"
        _assert_canary(out, n, I, f"fused gate_up at row 3 n={n}")


@pytest.mark.parametrize("name", ["gate_up", "down_proj"])
def test_graph_replays_are_bit_identical(name):
    N, K, swiglu = SHAPES[name]
    a, w = _inputs(N, K, 11)
    if swiglu:
        w = ops().interleave_gate_up(w[:N // 2], w[N // 2:])
    err = torch.zeros(4, dtype=torch.int32, device=DEV)
    c = torch.zeros(136, N // 2 if swiglu else N, dtype=F16, device=DEV)
    plan = ops().GemmPlan(a, w, c, err, swiglu=swiglu)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.run(128)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.run(128)
    c.zero_()
    g.replay()
    torch.cuda.synchronize()
    first = c.clone()
    c.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert err.tolist() == [0, 0, 0, 0]
    assert torch.equal(first, c) and bool(first[:128].abs().sum() > 0)


@pytest.mark.parametrize("force", [None, "64,2,1"], ids=["picked", "split2"])
def test_bound_sees_a_dropped_k_block_and_a_dropped_split_partial(force):
    """Negative controls: the float64 bound must reject the kernel's output against a reference that drops one 64-wide
    k-block, and (split-K tile) against one that drops one split's whole partial sum."""
    N, K, _ = SHAPES["down_proj"]
    a, w = _inputs(N, K, 13)
    err = torch.zeros(4, dtype=torch.int32, device=DEV)
    c = torch.zeros(136, N, dtype=F16, device=DEV)
    if force:
        with _env(SQ_GEMM_FORCE=force):
            plan = ops().GemmPlan(a, w, c, err)
    else:
        plan = ops().GemmPlan(a, w, c, err)
    plan.run(128)
    torch.cuda.synchronize()
    got = c[:128].double()
    ref, tol = _gemm_reference(a[:128], w)
    _assert_within(c[:128], ref, tol, "control run")
    bn, split, _ = plan.info()
    drops = [(64 * 37, 64 * 38)]
    if split > 1:
        drops.append((0, K // split))
    for k0, k1 in drops:
        part = a[:128, k0:k1].double() @ w[:, k0:k1].double().t()
        bad = ((got - (ref - part)).abs() > tol).double().mean().item()
        assert bad > 0.5, f"dropping k [{k0}, {k1}) left {1 - bad:.1%} of the outputs inside the bound"


def test_7b_layer_on_the_verify_route_is_as_close_to_fp32_as_cublas():
    """One 7B-shaped decoder layer (plus lm_head), prefix rows then the 127 tree rows of config 2, through the engine on
    the verify routes (gate_up on the fused sq_gemm plan) and with every layer projection on cuBLASLt: the routed
    logits are no further from the fp32 exact result than the cuBLASLt route's."""
    from sequoia_b200.engine import GraphInferenceEngineTG
    cfg = O.LlamaCfg(hidden_size=4096, intermediate_size=11008, num_hidden_layers=1, num_attention_heads=32,
                     num_key_value_heads=32, vocab_size=cases.V, rms_norm_eps=1e-5)
    w = O.init_llama_weights(cfg, 910)
    gm = cases.load_growmap("A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt")
    S, P, M = gm["size"], 64, 256
    tot = P + S - 1
    prompt = cases.make_prompt(79, tot)
    win = O.window_mask(O.build_full_attn_mask(M, gm["mask"]), M, tot)
    pos = torch.zeros(M, dtype=torch.long)
    pos[:P] = torch.arange(P)
    pos[P:tot] = gm["depth"][1:] + P - 1
    sto = torch.arange(M)
    orc32 = O.EngineOracle(O.LlamaOracle(cfg, {k: v.float() for k, v in w.items()}, M, "TG", dtype=torch.float32))
    routed = GraphInferenceEngineTG(M, {"config": cfg, "state_dict": w}, device=DEV)
    plain = GraphInferenceEngineTG(M, {"config": cfg, "state_dict": w}, device=DEV)
    assert "wgu_plan" in routed.engine.runner.layers[0], "the 7B verify route must run gate_up on sq_gemm"
    plain.engine.runner.layers[0].pop("wgu_plan")
    d_routed = d_plain = 0.0
    for (a, b, m) in ((0, P, win[:P, :P][None, None]), (P, tot, win[P:tot, :tot][None, None])):
        ex = orc32.inference(prompt[a:b].unsqueeze(0), sto[a:b], pos[a:b].unsqueeze(0), m.float())
        args = (prompt[a:b].unsqueeze(0).to(DEV), sto[a:b].to(DEV), pos[a:b].unsqueeze(0).to(DEV), m.to(DEV))
        got_r = routed.inference(*args).float().cpu()
        got_p = plain.inference(*args).float().cpu()
        scale = ex.abs().amax(dim=-1, keepdim=True)
        d_routed = max(d_routed, ((got_r - ex).abs() / scale).max().item())
        d_plain = max(d_plain, ((got_p - ex).abs() / scale).max().item())
    _log(f"7B-shaped layer, {tot} rows: max rel logit err vs fp32: verify route {d_routed:.3e}, cuBLASLt route {d_plain:.3e}")
    assert int(routed.engine.runner.gemm_err.abs().sum()) == 0
    assert d_routed <= 1.05 * d_plain, f"verify route further from fp32 ({d_routed:.3e}) than cuBLASLt ({d_plain:.3e})"
