"""FP8 (E4M3) target weights without a GPU: the quantization format (ops.quantize_fp8 / dequantize_fp8), the C ABI's
refusals of unsupported FP8 GEMM shapes, and the engines' refusals of unsupported weight formats."""
import ctypes as C
import math

import pytest
import torch

F16, F8 = torch.float16, torch.float8_e4m3fn


def ops():
    from sequoia_b200 import ops as _ops
    return _ops


def _e4m3_value(code: int) -> float:
    """the value of an e4m3fn bit pattern from its fields: 1 sign, 4 exponent (bias 7), 3 mantissa bits"""
    sign = -1.0 if code & 0x80 else 1.0
    e, m = (code >> 3) & 0xF, code & 0x7
    return sign * (m * 2.0 ** -9 if e == 0 else (1 + m / 8) * 2.0 ** (e - 7))


def test_every_finite_e4m3_code_converts_exactly_to_fp16():
    codes = [c for c in range(256) if c & 0x7F != 0x7F]                  # 0x7F / 0xFF are the NaNs
    assert len(codes) == 254
    got = torch.tensor(codes, dtype=torch.uint8).view(F8).to(F16)
    want = torch.tensor([_e4m3_value(c) for c in codes], dtype=torch.float64)
    assert torch.equal(want.to(F16).double(), want), "every e4m3 value is representable in fp16"
    assert torch.equal(got.double(), want)
    assert torch.equal(torch.signbit(got), torch.tensor([bool(c & 0x80) for c in codes]))   # -0 stays -0
    assert float(got.abs().max()) == 448.0


def test_quantize_scales_clamp_zero_and_underflowing_rows():
    K = 128
    w = (torch.randn(6, K, generator=torch.Generator().manual_seed(1)) * 0.02).to(F16)
    w[1] = 0                                                             # all-zero row: s = 1, q = 0
    w[2] = 0
    w[2, 5] = 2.0 ** -24                                                 # max / 448 rounds to 0 in fp16: s = 2^-24
    w[2, 6] = -(2.0 ** -24)
    # a row whose rounded scale is below max / 448, so that W / s > 448 before the clamp
    amax = next(x for x in torch.arange(1000, 1200, dtype=torch.float64).tolist()
                if float(torch.tensor(x / 448, dtype=torch.float32).to(F16)) < x / 448)
    w[3] = 0.5
    w[3, 0], w[3, 1] = amax, -amax
    q, s = ops().quantize_fp8(w)
    assert q.dtype == F8 and s.dtype == F16 and q.shape == w.shape and s.shape == (6,)
    qf = q.to(torch.float32)
    assert bool(torch.isfinite(qf).all()) and float(qf.abs().max()) <= 448.0
    assert float(s[1]) == 1.0 and bool((qf[1] == 0).all())
    assert float(s[2]) == 2.0 ** -24 and float(qf[2, 5]) == 1.0 and float(qf[2, 6]) == -1.0
    assert float(s[3]) < amax / 448 and float(qf[3, 0]) == 448.0 and float(qf[3, 1]) == -448.0
    for j in (0, 4, 5):
        assert float(s[j]) == float(torch.tensor(float(w[j].float().abs().max()) / 448, dtype=torch.float32).to(F16))
    # the same result in row chunks of any size (load-time quantization works through chunks)
    q2, s2 = ops().quantize_fp8(w, rows_per_chunk=4)
    assert torch.equal(q2.view(torch.uint8), q.view(torch.uint8)) and torch.equal(s2, s)


def test_quantize_rounds_to_nearest_even():
    # 1 + 1/16 lies halfway between the e4m3 neighbours 1 and 1.125: it rounds to the even mantissa (1); 1 + 3/16 to 1.25
    w = torch.tensor([[448.0, 1 + 1 / 16, 1 + 3 / 16, -(1 + 1 / 16)]], dtype=F16)
    q, s = ops().quantize_fp8(w)
    assert float(s[0]) == 1.0
    assert q.to(torch.float32).tolist() == [[448.0, 1.0, 1.25, -1.0]]


def _random_weight(N, K, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g) * 0.02
    w[::7] *= 30                                                         # rows of very different ranges
    w[1::5, ::3] = 0
    return w.to(F16)


def test_dequantize_is_the_rounded_fp16_product():
    q, s = ops().quantize_fp8(_random_weight(96, 256, 3))
    wd = ops().dequantize_fp8(q, s)
    assert wd.dtype == F16
    assert torch.equal(wd, q.half() * s[:, None])
    exact = q.double() * s.double()[:, None]                             # exact: 4 + 11 significant bits
    assert torch.equal(wd.view(torch.int16), exact.to(F16).view(torch.int16))


def test_dequantized_error_bound():
    """|W - W'| <= 2^-4 |W| + 2^-10 s + ulp(W') per element: e4m3's relative rounding (half of 2^-3), half its subnormal
    step (2^-9 s), and the fp16 rounding of the product."""
    w = _random_weight(256, 512, 4)
    q, s = ops().quantize_fp8(w)
    wd = ops().dequantize_fp8(q, s).double()
    w64 = w.double()
    ulp = torch.pow(2.0, torch.floor(torch.log2(wd.abs().clamp(min=2.0 ** -14))) - 10)
    bound = 2.0 ** -4 * w64.abs() + 2.0 ** -10 * s.double()[:, None] + ulp
    err = (w64 - wd).abs()
    assert bool((err <= bound).all()), f"worst err/bound {(err / bound).max().item():.3f}"
    # and the bound is not vacuous: the typical error is a sizeable part of it
    assert (err / bound).max().item() > 0.3


def test_quantize_rejects_non_fp16():
    with pytest.raises(TypeError):
        ops().quantize_fp8(torch.zeros(4, 64))


def test_fp8_gemm_refusals_through_the_c_abi():
    from sequoia_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    fake = 4096                                                          # never dereferenced: refused before any use
    base = dict(a=fake, lda=4096, n_max=128, w=fake, s=fake, N=4096, K=4096, c=fake, ldc=4096)

    def create(**kw):
        a = {**base, **kw}
        return lib.sq_gemm_fp8_plan_create(C.byref(h), a["a"], a["lda"], a["n_max"], a["w"], a["s"], a["N"], a["K"],
                                           a["c"], a["ldc"], None)

    for kw, what in ((dict(K=4096 + 32), b"K % 64"), (dict(N=4096 + 32), b"N % 64"), (dict(n_max=0), b"n_max"),
                     (dict(w=None), b"null"), (dict(s=None), b"null"), (dict(a=None), b"null"), (dict(c=None), b"null"),
                     (dict(lda=4100), b"lda"), (dict(ldc=4000), b"ldc")):
        assert create(**kw) == -1, kw
        assert what in lib.sq_last_error(), (kw, lib.sq_last_error())
    assert lib.sq_gemm_fp8_tile_weights(fake, fake, 96, 64, None) == -1 and b"N % 64" in lib.sq_last_error()
    assert lib.sq_gemm_fp8_tile_weights(None, fake, 64, 64, None) == -1 and b"null" in lib.sq_last_error()
    assert lib.sq_gemm_fp8_run_at(None, 1, 0, None, 0, None) == -1 and b"null plan" in lib.sq_last_error()


def test_engines_refuse_tp_and_unknown_weight_formats():
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    from sequoia_b200.model import LlamaRunner
    with pytest.raises(ValueError, match="weight_format"):
        LlamaRunner("random-init:llama-68m", 64, device="cpu", weight_format="int8")
    with pytest.raises(NotImplementedError, match="tensor parallelism"):
        LlamaRunner("random-init:llama-68m", 64, device="cpu", tp_group=object(), weight_format="fp8")
    with pytest.raises(ValueError, match="weight_format"):
        GraphInferenceEngineTG(64, "random-init:llama-68m", device="cpu", weight_format="fp4")
    with pytest.raises(ValueError, match="weight_format"):
        GraphInferenceEngine(64, "random-init:llama-68m", device="cpu", weight_format="bf16")
    # the test draft's FFN (2I = 1376) is not a whole number of 64-row weight tiles
    import cases
    cfg, w = cases.model_weights("draft")
    with pytest.raises(ValueError, match="multiples of 64"):
        LlamaRunner({"config": cfg, "state_dict": w}, 64, device="cpu", weight_format="fp8")


def test_testbed_target_weights_flag():
    import testbed
    assert testbed.build_parser().parse_args([]).target_weights == "fp16"
    assert testbed.build_parser().parse_args(["--target-weights", "fp8"]).target_weights == "fp8"
    with pytest.raises(SystemExit):
        testbed.build_parser().parse_args(["--target-weights", "int8"])


def test_quantized_bytes_of_the_named_targets():
    """The four layer projections of a target in e4m3 plus one fp16 scale per output row: half the fp16 bytes (+ scales)."""
    from sequoia_b200.model import NAMED_CONFIGS
    for name, fp16_gb in (("llama-2-7b", 12.95), ("llama-2-13b", 25.4), ("llama-3.1-8b", 13.96)):
        c = NAMED_CONFIGS[name]
        h, I, L, D = c.hidden_size, c.intermediate_size, c.num_hidden_layers, c.head_dim
        shapes = [((c.num_attention_heads + 2 * c.num_key_value_heads) * D, h), (h, c.num_attention_heads * D), (2 * I, h),
                  (h, I)]
        elems = L * sum(n * k for n, k in shapes)
        rows = L * sum(n for n, _ in shapes)
        assert math.isclose(2 * elems / 1e9, fp16_gb, rel_tol=5e-3), name
        assert elems + 2 * rows < 0.501 * 2 * elems
        if name == "llama-2-7b":
            assert math.isclose(2 * rows / 1e6, 2.7, rel_tol=0.02)          # 2.7 MB of scales
