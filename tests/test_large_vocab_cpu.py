"""Host side of 128K-vocabulary models, on the CPU: llama3 RoPE scaling in rope_cache, rope_scaling parsing, the Llama 3
named configs, vocabulary refusals and the testbed's stop tokens."""
import json
import math

import pytest
import torch

from sequoia_b200 import model as M
from sequoia_b200 import tree as T

LLAMA3 = dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
              original_max_position_embeddings=8192)


def _cfg(**kw):
    base = dict(hidden_size=4096, intermediate_size=14336, num_hidden_layers=2, num_attention_heads=32,
                num_key_value_heads=8, vocab_size=128256, rope_theta=500000.0, max_position_embeddings=8192)
    base.update(kw)
    return base


def _llama3_inv_freq_f64(theta, d, rs):
    """The published transform restated element by element in float64."""
    out = []
    for i in range(0, d, 2):
        f = 1.0 / theta ** (i / d)
        wavelen = 2 * math.pi / f
        lo_w = rs["original_max_position_embeddings"] / rs["low_freq_factor"]
        hi_w = rs["original_max_position_embeddings"] / rs["high_freq_factor"]
        if wavelen < hi_w:
            out.append(f)
        elif wavelen > lo_w:
            out.append(f / rs["factor"])
        else:
            s = (rs["original_max_position_embeddings"] / wavelen - rs["low_freq_factor"]) / (
                rs["high_freq_factor"] - rs["low_freq_factor"])
            out.append((1 - s) * f / rs["factor"] + s * f)
    return torch.tensor(out, dtype=torch.float64)


@pytest.mark.parametrize("factor", [8.0, 32.0])
def test_llama3_inv_freq_matches_float64_restatement(factor):
    rs = dict(LLAMA3, factor=factor)
    d = 128
    inv = 1.0 / (500000.0 ** (torch.arange(0, d, 2, dtype=torch.float32) / d))
    got = M.llama3_inv_freq(inv, rs).double()
    ref = _llama3_inv_freq_f64(500000.0, d, rs)
    assert torch.allclose(got, ref, rtol=2e-6, atol=0)
    # all three bands occur at these parameters
    assert bool((got == inv.double()).any()) and bool((got < inv.double() / factor * 1.0001).any())


def test_llama3_inv_freq_matches_transformers():
    rope_utils = pytest.importorskip("transformers.modeling_rope_utils")
    from transformers import LlamaConfig
    hf = LlamaConfig(**_cfg(), rope_scaling=dict(LLAMA3))
    inv_hf, _ = rope_utils.ROPE_INIT_FUNCTIONS["llama3"](hf, "cpu")
    d = 128
    inv = 1.0 / (500000.0 ** (torch.arange(0, d, 2, dtype=torch.float32) / d))
    got = M.llama3_inv_freq(inv, M.parse_rope_scaling(LLAMA3))
    assert torch.allclose(got.float(), inv_hf.float(), rtol=1e-6, atol=0)


def test_rope_cache_llama3_tables():
    cfg = M.config_from(_cfg(rope_scaling=dict(LLAMA3)))
    cos, sin = M.rope_cache(cfg, 300, "cpu")
    inv = _llama3_inv_freq_f64(500000.0, 128, LLAMA3)
    t = torch.arange(300, dtype=torch.float64)
    emb = torch.cat([torch.outer(t, inv)] * 2, dim=-1)
    # fp32 table -> fp16: within one fp16 ulp of the float64 values
    assert torch.allclose(cos.double(), emb.cos(), atol=1e-3, rtol=0)
    assert torch.allclose(sin.double(), emb.sin(), atol=1e-3, rtol=0)
    unscaled = M.rope_cache(M.config_from(_cfg()), 300, "cpu")[0]
    assert not torch.equal(cos, unscaled)


def test_rope_scaling_none_keeps_tables_bit_identical():
    d, theta, n = 64, 10000.0, 2048
    for rs in (None, "absent"):
        c = _cfg(hidden_size=64 * 12, num_attention_heads=12, num_key_value_heads=12, rope_theta=theta,
                 max_position_embeddings=n)
        if rs is None:
            c["rope_scaling"] = None
        cfg = M.config_from(c)
        assert cfg.rope_scaling is None
        cos, sin = M.rope_cache(cfg, 384, "cpu")
        inv = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.float32) / d))   # the table as built before rope_scaling
        freqs = torch.outer(torch.arange(n, dtype=torch.float32), inv)
        emb = torch.cat((freqs, freqs), dim=-1)
        assert torch.equal(cos, emb.cos()[:384].half()) and torch.equal(sin, emb.sin()[:384].half())


@pytest.mark.parametrize("rs", [dict(type="linear", factor=2.0), dict(rope_type="dynamic", factor=2.0),
                                dict(rope_type="yarn", factor=4.0)])
def test_unknown_rope_scaling_raises(rs):
    with pytest.raises(ValueError, match="rope_scaling"):
        M.config_from(_cfg(rope_scaling=rs))


def test_rope_scaling_legacy_type_key():
    rs = dict(LLAMA3)
    rs["type"] = rs.pop("rope_type")
    assert M.config_from(_cfg(rope_scaling=rs)).rope_scaling["factor"] == 8.0


def test_named_llama3_configs():
    a, b = M.NAMED_CONFIGS["llama-3.2-1b"], M.NAMED_CONFIGS["llama-3.1-8b"]
    assert (a.hidden_size, a.intermediate_size, a.num_hidden_layers, a.num_attention_heads, a.num_key_value_heads) == \
        (2048, 8192, 16, 32, 8)
    assert (b.hidden_size, b.intermediate_size, b.num_hidden_layers, b.num_attention_heads, b.num_key_value_heads) == \
        (4096, 14336, 32, 32, 8)
    for c, f in ((a, 32.0), (b, 8.0)):
        assert c.vocab_size == 128256 and c.rope_theta == 500000.0 and c.rms_norm_eps == 1e-5
        assert c.rope_scaling["rope_type"] == "llama3" and c.rope_scaling["factor"] == f
        assert c.rope_scaling["original_max_position_embeddings"] == 8192


def test_vocabulary_refusals():
    T.check_vocab("spec", 128256)
    T.check_vocab("greedy", 131072)
    T.check_vocab("specinfer", 32000)
    with pytest.raises(ValueError, match="SpecInferTree"):
        T.check_vocab("specinfer", 128256)
    with pytest.raises(ValueError):
        T.check_vocab("spec", 131080)


def test_single_cta_walk_refuses_large_vocab(monkeypatch):
    monkeypatch.setenv("SQ_ACCEPT_IMPL", "0")
    with pytest.raises(ValueError, match="SQ_ACCEPT_IMPL=0"):
        T.check_vocab("spec", 128256)
    T.check_vocab("spec", 32000)
    T.check_vocab("greedy", 128256)           # the greedy walk never runs the stochastic kernel


def test_stop_tokens(tmp_path):
    import testbed
    assert testbed.stop_tokens("random-init:llama-68m") == frozenset([0, 2])
    for eos, want in ((128001, {128001}), ([128001, 128008, 128009], {128001, 128008, 128009}), (None, {0, 2})):
        d = tmp_path / f"m{len(want)}{eos is None}"
        d.mkdir()
        cfg = {"vocab_size": 128256} if eos is None else {"vocab_size": 128256, "eos_token_id": eos}
        (d / "config.json").write_text(json.dumps(cfg))
        assert testbed.stop_tokens(str(d)) == frozenset(want)


def test_rope_type_default_means_no_scaling():
    assert M.config_from(_cfg(rope_scaling=dict(rope_type="default", rope_theta=500000.0))).rope_scaling is None
    cfg = M.config_from(_cfg(rope_theta=None, rope_parameters=dict(rope_type="default", rope_theta=10000.0)))
    assert cfg.rope_scaling is None and cfg.rope_theta == 10000.0


def test_rope_parameters_of_transformers_5_configs():
    """transformers >= 5 writes theta and the scaling under `rope_parameters`: they must not be ignored."""
    c = _cfg(rope_theta=None, rope_parameters=dict(LLAMA3, rope_theta=500000.0))
    cfg = M.config_from(c)
    assert cfg.rope_theta == 500000.0 and cfg.rope_scaling == M.parse_rope_scaling(LLAMA3)
    with pytest.raises(ValueError, match="rope_scaling"):
        M.config_from(_cfg(rope_parameters=dict(rope_type="yarn", factor=4.0, rope_theta=1e4)))
    transformers = pytest.importorskip("transformers")
    hf = transformers.LlamaConfig(**_cfg(max_position_embeddings=131072), rope_scaling=dict(LLAMA3))
    assert M.config_from(hf).rope_scaling == M.parse_rope_scaling(LLAMA3)
    assert M.config_from(transformers.LlamaConfig(**_cfg())).rope_scaling is None
