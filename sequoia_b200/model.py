"""Tree-masked Llama forward on the sequoia_b200 kernels.

Replaces Engine/Llama_model.py + Engine/Llama_modules.py of the reference (LlamaForCausalLM_FI / _TG):
embed -> L x [RMSNorm, fused QKV GEMM, RoPE + KV append, tree attention, o_proj, residual+RMSNorm,
fused gate/up GEMM, SiLU*up, down_proj, residual+RMSNorm] -> lm_head.

* the dense weight GEMMs stay on cuBLASLt through torch.mm (SURVEY.md 2.2 K1: not a hand-written
  kernel on this path); everything else is a launch into libsequoia_b200.so;
* q/k/v and gate/up weights are concatenated at load time so one GEMM feeds each fused kernel;
* every buffer is preallocated for n_max rows, so a forward allocates nothing and is CUDA-graph
  capturable; dynamic quantities (prefix length, kv length) are read from the device state word;
* optional tensor parallelism (Megatron layout): column-parallel qkv / gate_up, row-parallel
  o_proj / down_proj followed by an NCCL sum-allreduce (2 per layer), KV cache sharded by kv head.
"""
from __future__ import annotations

import json
import math
import os
from dataclasses import dataclass
from typing import Dict, Optional

import torch

from . import ops

F16 = torch.float16


@dataclass
class LlamaConfigLite:
    hidden_size: int
    intermediate_size: int
    num_hidden_layers: int
    num_attention_heads: int
    num_key_value_heads: int
    vocab_size: int = 32000
    rms_norm_eps: float = 1e-6
    rope_theta: float = 10000.0
    max_position_embeddings: int = 2048
    rope_scaling: Optional[dict] = None    # None, or parse_rope_scaling()'s llama3 dict

    @property
    def head_dim(self):
        return self.hidden_size // self.num_attention_heads


# public HF configs of the model sizes BASELINE.json names (random-init weights of these shapes)
NAMED_CONFIGS = {
    "llama-68m": LlamaConfigLite(768, 3072, 2, 12, 12),
    "llama-160m": LlamaConfigLite(768, 3072, 12, 12, 12),
    "llama-2-7b": LlamaConfigLite(4096, 11008, 32, 32, 32, rms_norm_eps=1e-5, max_position_embeddings=4096),
    "llama-2-13b": LlamaConfigLite(5120, 13824, 40, 40, 40, rms_norm_eps=1e-5, max_position_embeddings=4096),
    "llama-2-70b": LlamaConfigLite(8192, 28672, 80, 64, 8, rms_norm_eps=1e-5, max_position_embeddings=4096),
    # the first 8 layers' worth of a 70B-shaped model: TP parity checks at the real head / FFN shapes where the
    # unsharded 138 GB model cannot sit next to a shard (bench.py tp_parity, tests/test_gpu_tp.py)
    "llama-2-70b-8l": LlamaConfigLite(8192, 28672, 8, 64, 8, rms_norm_eps=1e-5, max_position_embeddings=4096),
    # Llama 3 draft / target pair (128256-token vocabulary, llama3 RoPE scaling)
    "llama-3.2-1b": LlamaConfigLite(2048, 8192, 16, 32, 8, vocab_size=128256, rms_norm_eps=1e-5, rope_theta=500000.0,
                                    max_position_embeddings=131072,
                                    rope_scaling=dict(rope_type="llama3", factor=32.0, low_freq_factor=1.0,
                                                      high_freq_factor=4.0, original_max_position_embeddings=8192)),
    "llama-3.1-8b": LlamaConfigLite(4096, 14336, 32, 32, 8, vocab_size=128256, rms_norm_eps=1e-5, rope_theta=500000.0,
                                    max_position_embeddings=131072,
                                    rope_scaling=dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0,
                                                      high_freq_factor=4.0, original_max_position_embeddings=8192)),
}


def parse_rope_scaling(rs) -> Optional[dict]:
    """config.json's `rope_scaling` -> None (no scaling) or the llama3 parameters.  Any other type raises: decoding with
    unscaled frequencies would silently give wrong results."""
    if rs is None:
        return None
    kind = rs.get("rope_type", rs.get("type"))
    if kind in (None, "default"):          # transformers >= 5 writes {"rope_type": "default", "rope_theta": ...}
        return None
    if kind != "llama3":
        raise ValueError(f"rope_scaling type {kind!r} is not supported (supported: None, 'llama3')")
    return dict(rope_type="llama3", factor=float(rs["factor"]), low_freq_factor=float(rs["low_freq_factor"]),
                high_freq_factor=float(rs["high_freq_factor"]),
                original_max_position_embeddings=int(rs["original_max_position_embeddings"]))


def llama3_inv_freq(inv_freq: torch.Tensor, rs: dict) -> torch.Tensor:
    """The Llama 3 inverse-frequency transform: wavelengths longer than original_max / low_freq_factor are divided by
    `factor`, shorter than original_max / high_freq_factor kept, and the band between interpolated smoothly."""
    factor, lo, hi = rs["factor"], rs["low_freq_factor"], rs["high_freq_factor"]
    old = rs["original_max_position_embeddings"]
    wavelen = 2 * math.pi / inv_freq
    out = torch.where(wavelen > old / lo, inv_freq / factor, inv_freq)
    smooth = (old / wavelen - lo) / (hi - lo)
    smoothed = (1 - smooth) * out / factor + smooth * out
    medium = ~(wavelen < old / hi) & ~(wavelen > old / lo)
    return torch.where(medium, smoothed, out)


def config_from(obj) -> LlamaConfigLite:
    if isinstance(obj, LlamaConfigLite):
        return obj
    g = (lambda k, d=None: obj.get(k, d)) if isinstance(obj, dict) else (lambda k, d=None: getattr(obj, k, d))
    # transformers >= 5 keeps theta and the scaling under `rope_parameters`; older configs use the two top-level keys
    rp = g("rope_parameters", None) or {}
    theta = g("rope_theta", None) or rp.get("rope_theta")
    rs = g("rope_scaling", None) or (rp or None)
    return LlamaConfigLite(
        hidden_size=g("hidden_size"), intermediate_size=g("intermediate_size"),
        num_hidden_layers=g("num_hidden_layers"), num_attention_heads=g("num_attention_heads"),
        num_key_value_heads=g("num_key_value_heads") or g("num_attention_heads"), vocab_size=g("vocab_size", 32000),
        rms_norm_eps=g("rms_norm_eps", 1e-6), rope_theta=float(theta) if theta else 10000.0,
        max_position_embeddings=g("max_position_embeddings", 2048), rope_scaling=parse_rope_scaling(rs))


def _load_state_dict_dir(path: str) -> Dict[str, torch.Tensor]:
    sd: Dict[str, torch.Tensor] = {}
    files = sorted(os.listdir(path))
    st = [f for f in files if f.endswith(".safetensors")]
    if st:
        from safetensors.torch import load_file
        for f in st:
            sd.update(load_file(os.path.join(path, f)))
        return sd
    for f in files:                                    # HF shard names only (a model dir may also hold training_args.bin ...)
        if (f.startswith("pytorch_model") and f.endswith(".bin")) or (f.startswith("model") and f.endswith(".pt")):
            sd.update(torch.load(os.path.join(path, f), map_location="cpu"))
    if not sd:
        raise FileNotFoundError(f"no weight files (*.safetensors / *.bin) in {path}")
    return sd


class _RandomInit:
    """HF-default random init (normal std 0.02, norms = 1) generated on the device, tensor by tensor, from a seeded
    generator; the FULL tensor is always drawn and then sharded, so every TP degree sees the same model."""

    def __init__(self, cfg: LlamaConfigLite, seed: int, device):
        self.cfg, self.device = cfg, device
        self.g = torch.Generator(device=device)
        self.g.manual_seed(seed)

    def get(self, name: str, shape) -> torch.Tensor:
        if name.endswith("norm.weight") or "layernorm" in name:
            return torch.ones(shape, dtype=F16, device=self.device)
        t = torch.empty(shape, dtype=F16, device=self.device)
        t.normal_(0.0, 0.02, generator=self.g)
        return t


class _DictSource:
    def __init__(self, sd: Dict[str, torch.Tensor], device):
        self.sd, self.device = sd, device

    def get(self, name: str, shape) -> torch.Tensor:
        if name == "lm_head.weight" and name not in self.sd:          # tied embeddings: checkpoints omit lm_head
            name = "model.embed_tokens.weight"
        t = self.sd[name]
        assert tuple(t.shape) == tuple(shape), (name, t.shape, shape)
        return t.to(device=self.device, dtype=F16)


def resolve_model(model_name_or_path, device):
    """-> (LlamaConfigLite, weight source).  Accepted forms of `model_name_or_path`:
       * directory with config.json + *.safetensors / *.bin   (what from_pretrained took, Engine/Engine.py:18)
       * "random-init:<name>[:seed]" with <name> in NAMED_CONFIGS   (synthetic benchmarks, no network)
       * {"config": cfg, "state_dict": {...}}   (tests: weights shared with the oracle)."""
    if isinstance(model_name_or_path, dict):
        cfg = config_from(model_name_or_path["config"])
        return cfg, _DictSource(model_name_or_path["state_dict"], device)
    s = str(model_name_or_path)
    if s.startswith("random-init:"):
        parts = s.split(":")
        cfg = NAMED_CONFIGS[parts[1].lower()]
        seed = int(parts[2]) if len(parts) > 2 else 0
        return cfg, _RandomInit(cfg, seed, device)
    if os.path.isdir(s):
        with open(os.path.join(s, "config.json")) as f:
            cfg = config_from(json.load(f))
        return cfg, _DictSource(_load_state_dict_dir(s), device)
    raise FileNotFoundError(
        f"{s!r}: expected a local model directory or 'random-init:<{'|'.join(NAMED_CONFIGS)}>[:seed]' "
        "(there is no network access for hub downloads)")


def rope_cache(cfg: LlamaConfigLite, max_length: int, device):
    """LlamaRotaryEmbedding_FI (Engine/Llama_modules.py:16-45): fp32 tables, sliced [:max_length], cast to fp16."""
    d = cfg.head_dim
    inv_freq = 1.0 / (cfg.rope_theta ** (torch.arange(0, d, 2, dtype=torch.float32) / d))
    if cfg.rope_scaling is not None:
        inv_freq = llama3_inv_freq(inv_freq, parse_rope_scaling(cfg.rope_scaling))
    # the reference builds max_position_embeddings rows and slices [:max_length]; rows beyond that table would be an
    # out-of-bounds read in the RoPE kernel, so the table always covers max_length (identical values where both exist)
    t = torch.arange(max(cfg.max_position_embeddings, max_length), dtype=torch.float32)
    freqs = torch.outer(t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    return (emb.cos()[:max_length].to(F16).to(device).contiguous(), emb.sin()[:max_length].to(F16).to(device).contiguous())


class TPInfo:
    def __init__(self, group=None):
        import torch.distributed as dist
        self.group = group
        if group is None:
            self.rank, self.size = 0, 1
        else:
            self.rank, self.size = dist.get_rank(group), dist.get_world_size(group)

    def all_reduce(self, t: torch.Tensor):
        if self.size > 1:
            import torch.distributed as dist
            dist.all_reduce(t, group=self.group)


def full_state_dict(cfg: LlamaConfigLite, src) -> Dict[str, torch.Tensor]:
    """The whole model as an HF-named state dict, tensors requested from `src` in EXACTLY the order
    `load_sharded_weights` requests them -- so a seeded `_RandomInit` yields the same weights either way.  Used to hand
    the very same random-init model to the reference implementation / the CPU oracle in bench.py."""
    h, D, V = cfg.hidden_size, cfg.head_dim, cfg.vocab_size
    Hf, Hkvf, If = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.intermediate_size
    sd = {"model.embed_tokens.weight": src.get("model.embed_tokens.weight", (V, h))}
    for l in range(cfg.num_hidden_layers):
        p = f"model.layers.{l}."
        for name, shape in (("self_attn.q_proj.weight", (Hf * D, h)), ("self_attn.k_proj.weight", (Hkvf * D, h)),
                            ("self_attn.v_proj.weight", (Hkvf * D, h)), ("self_attn.o_proj.weight", (h, Hf * D)),
                            ("mlp.gate_proj.weight", (If, h)), ("mlp.up_proj.weight", (If, h)),
                            ("mlp.down_proj.weight", (h, If)), ("input_layernorm.weight", (h,)),
                            ("post_attention_layernorm.weight", (h,))):
            sd[p + name] = src.get(p + name, shape)
    sd["model.norm.weight"] = src.get("model.norm.weight", (h,))
    sd["lm_head.weight"] = src.get("lm_head.weight", (V, h))
    return sd


def load_sharded_weights(cfg: LlamaConfigLite, src, rank: int, tp: int) -> dict:
    """Megatron-style shard `rank` of `tp`: q/k/v and gate/up split by output rows (heads / FFN columns) and fused,
    o_proj / down_proj split by input columns (their partial products are summed by the allreduce)."""
    h, D, V = cfg.hidden_size, cfg.head_dim, cfg.vocab_size
    Hf, Hkvf, If = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.intermediate_size
    assert Hf % tp == 0 and Hkvf % tp == 0 and If % tp == 0, "heads / FFN width must divide the TP degree"
    H, Hkv, I, r = Hf // tp, Hkvf // tp, If // tp, rank
    out = {"embed": src.get("model.embed_tokens.weight", (V, h)), "layers": []}
    for l in range(cfg.num_hidden_layers):
        p = f"model.layers.{l}."
        wq = src.get(p + "self_attn.q_proj.weight", (Hf * D, h))[r * H * D:(r + 1) * H * D]
        wk = src.get(p + "self_attn.k_proj.weight", (Hkvf * D, h))[r * Hkv * D:(r + 1) * Hkv * D]
        wv = src.get(p + "self_attn.v_proj.weight", (Hkvf * D, h))[r * Hkv * D:(r + 1) * Hkv * D]
        wo = src.get(p + "self_attn.o_proj.weight", (h, Hf * D))[:, r * H * D:(r + 1) * H * D]
        wg = src.get(p + "mlp.gate_proj.weight", (If, h))[r * I:(r + 1) * I]
        wu = src.get(p + "mlp.up_proj.weight", (If, h))[r * I:(r + 1) * I]
        wd = src.get(p + "mlp.down_proj.weight", (h, If))[:, r * I:(r + 1) * I]
        out["layers"].append(dict(
            wqkv=torch.cat([wq, wk, wv], dim=0).contiguous(), wo=wo.contiguous(),
            wgu=torch.cat([wg, wu], dim=0).contiguous(), wd=wd.contiguous(),
            ln1=src.get(p + "input_layernorm.weight", (h,)), ln2=src.get(p + "post_attention_layernorm.weight", (h,))))
        del wq, wk, wv, wo, wg, wu, wd
    out["norm"] = src.get("model.norm.weight", (h,))
    out["lm_head"] = src.get("lm_head.weight", (V, h))
    return out


class LlamaRunner:
    """Weights + preallocated activations + attention plan of one engine."""

    PROJECTIONS = ("wqkv", "wo", "wgu", "wd")

    def __init__(self, model_name_or_path, max_length: int, device="cuda:0", tp_group=None, n_max: Optional[int] = None,
                 batch_size: int = 1, weight_format: str = "fp16"):
        """weight_format "fp8": the four layer projections are quantized to E4M3 with one fp16 scale per output channel
        at load (ops.quantize_fp8) and run on the FP8 GEMM at every row count; embedding, norms and lm_head stay fp16."""
        if weight_format not in ("fp16", "fp8"):
            raise ValueError(f"weight_format must be 'fp16' or 'fp8', got {weight_format!r}")
        if weight_format == "fp8" and tp_group is not None:
            raise NotImplementedError("FP8 target weights run on one GPU: tensor parallelism needs weight_format='fp16'")
        self.weight_format = weight_format
        self.device = torch.device(device)
        self.B = batch_size
        self.cfg, src = resolve_model(model_name_or_path, self.device)
        cfg = self.cfg
        self.tp = TPInfo(tp_group)
        tp, r = self.tp.size, self.tp.rank
        assert cfg.num_attention_heads % tp == 0 and cfg.num_key_value_heads % tp == 0 and cfg.intermediate_size % tp == 0
        self.M = max_length
        self.n_max = n_max or max_length * batch_size        # batch: B sequences' rows, sequence-major
        self.H, self.Hkv, self.D = cfg.num_attention_heads // tp, cfg.num_key_value_heads // tp, cfg.head_dim
        self.I = cfg.intermediate_size // tp
        h, D, V = cfg.hidden_size, self.D, cfg.vocab_size
        self.h, self.V, self.L = h, V, cfg.num_hidden_layers
        if weight_format == "fp8":
            shapes = (((self.H + 2 * self.Hkv) * D, h), (h, self.H * D), (2 * self.I, h), (h, self.I))
            if any(n % 64 or k % 64 for n, k in shapes):
                raise ValueError(f"weight_format='fp8' needs every layer projection (N, K) to be multiples of 64, got {shapes}")
        wts = load_sharded_weights(cfg, src, r, tp)
        self.embed, self.layers, self.norm, self.lm_head = wts["embed"], wts["layers"], wts["norm"], wts["lm_head"]
        self.cos, self.sin = rope_cache(cfg, max_length, self.device)
        self.eps = float(cfg.rms_norm_eps)
        n = self.n_max
        dev = self.device
        z = lambda *s: torch.zeros(*s, dtype=F16, device=dev)
        self.hidden, self.normed = z(n, h), z(n, h)
        self.qkv = z(n, (self.H + 2 * self.Hkv) * D)
        self.attn_out, self.proj = z(n, self.H * D), z(n, h)
        self.gate_up, self.act = z(n, 2 * self.I), z(n, self.I)
        self.logits = z(n, V)
        self.k_cache = torch.zeros(self.L, batch_size, self.Hkv, max_length, D, dtype=F16, device=dev)
        self.v_cache = torch.zeros_like(self.k_cache)
        self.plan = ops.AttnPlan(self.qkv, n, self.H, self.Hkv, D, self.k_cache, self.v_cache, self.attn_out)
        # Dense GEMMs.  The weight-streaming shapes go to the hand-written wgmma kernel (csrc/sq_gemm.cu) -- gate_up with the
        # SwiGLU epilogue fused (weights interleaved, `act` written directly: no gate_up round trip, no silu_mul launch)
        # and the target's lm_head -- for models whose layers are HBM-stream-sized (hidden >= 2048); q/k/v, o_proj and
        # down_proj stay on cuBLASLt (torch.mm), which is faster at those shapes.
        self.gemm_err = torch.zeros(4, dtype=torch.int32, device=dev)
        self.lm_plan = None
        if weight_format == "fp8":
            # each fp16 projection is dropped as soon as its plan holds the quantized, pre-tiled copy
            io = dict(wqkv=(self.normed, self.qkv), wo=(self.attn_out, self.proj), wgu=(self.normed, self.gate_up),
                      wd=(self.act, self.proj))
            for ly in self.layers:
                for k in self.PROJECTIONS:
                    q, s = ops.quantize_fp8(ly.pop(k))
                    ly[k + "_fp8"] = ops.GemmFp8Plan(io[k][0], q, s, io[k][1], self.gemm_err)
                    del q
            torch.cuda.empty_cache()
        stream_sized = h >= 2048
        # (a fused-epilogue plan cannot split K, so a narrow shard -- TP-4/8 of a 7B -- would leave most SMs idle: those
        # stay on cuBLASLt + sq_silu_mul).  The plans serve forwards of <= 128 rows; larger ones (prefill, the 768-row verify
        # of config 4: compute-bound, not a weight stream) go to cuBLASLt on the SAME weight tensor, which is why gate_up is
        # kept row-major in the interleaved order (16 gate rows | 16 up rows) rather than pre-tiled.
        gu_bn, gu_split, _ = ops.gemm_pick_tiles(2 * self.I, h, ops.GEMM_SWIGLU) if self.I % 16 == 0 and h % 64 == 0 else (0, 1, 1)
        gu_ctas = (-(-2 * self.I // gu_bn)) * gu_split if gu_bn else 0
        self.gu_interleaved = False
        if stream_sized and gu_ctas >= 120 and weight_format == "fp16":
            self.gu_interleaved = True
            for ly in self.layers:
                ly["wgu"] = ops.interleave_gate_up(ly["wgu"][:self.I], ly["wgu"][self.I:])
                ly["gu_plan"] = ops.GemmPlan(self.normed, ly["wgu"], self.act, self.gemm_err, swiglu=True)
        if stream_sized and V % 32 == 0 and h % 64 == 0:
            self.lm_plan = ops.GemmPlan(self.normed, self.lm_head, self.logits, self.gemm_err)
        # Small draft models (csrc/sq_draft.cu): a dedicated attention kernel replaces sq_tree_attn for the draft's
        # tree-relative forwards of <= 64 rows (SQ_DRAFT_ATTN=0 turns it off).
        self.draft_plan = None
        if (os.environ.get("SQ_DRAFT_ATTN", "1") != "0" and tp == 1 and batch_size == 1 and
                ops.draft_supported(h, self.H, self.Hkv, D, max_length)):
            self.draft_plan = ops.DraftPlan(h, self.L, self.H, max_length, self.k_cache, self.v_cache)
        self.peer = None
        if self.tp.size > 1 and os.environ.get("SQ_TP_MODE", "fused") == "fused":
            from .peer import PeerBuffers
            self.peer = PeerBuffers(tp_group, self.device, n, h)

    def _gate_up_act(self, ly, n: int):
        """act[:n] = silu(normed[:n] @ Wg.T) * (normed[:n] @ Wu.T)   (Engine/Llama_modules.py:272)"""
        plan = ly.get("gu_plan")
        # the plan's activation tile is always 128 rows: worth it when most of them are real (config 2: 128 rows); for the
        # 65-row tree of config 3 cuBLASLt's 64-row tiles ingest half as much activation per SM
        if plan is not None and 96 < n <= 128:
            plan.run(n)
            return
        self._project(ly, "wgu", self.normed, n, self.gate_up)
        ops.silu_mul(self.gate_up, self.act, n, interleaved=self.gu_interleaved)

    def _project(self, ly, k: str, a: torch.Tensor, n: int, out: torch.Tensor):
        """out[:n] = a[:n] @ W_k.T: torch.mm on an fp16 weight, the FP8 plan (bound to a / out) on a quantized one"""
        plan = ly.get(k + "_fp8")
        if plan is not None:
            plan.run(n)
        else:
            torch.mm(a[:n], ly[k].t(), out=out[:n])

    def weight_bytes(self) -> int:
        """bytes of the weights resident on the device (an FP8 projection: its e4m3 bytes and fp16 scales)"""
        b = 2 * (self.embed.numel() + self.lm_head.numel() + self.norm.numel())
        for ly in self.layers:
            b += 2 * (ly["ln1"].numel() + ly["ln2"].numel())
            b += sum(ly[k + "_fp8"].weight_bytes() if k + "_fp8" in ly else 2 * ly[k].numel() for k in self.PROJECTIONS)
        return b

    @torch.no_grad()
    def forward(self, n: int, tokens: torch.Tensor, position_ids: torch.Tensor, storage_ids: torch.Tensor, *,
                state=None, n0: int = 0, kv_end: int = 0, prefix_len: int = 0, dense_mask=None, mask_ld: int = 0,
                tree_bits=None, tree_words: int = 0, tree_size: int = 0, logits_out: Optional[torch.Tensor] = None,
                logits_from: int = 0, skip_lm_head: bool = False, batch: bool = False,
                logits_to: Optional[int] = None) -> Optional[torch.Tensor]:
        """Forward `n` rows.  Row r is token tokens[base+r] at position position_ids[base+r], written to cache slot
        storage_ids[base+r], base = (state ? P-1 : 0) + n0.  Attends slots [0, (state ? P-1 : 0) + kv_end).
        Logits of rows [logits_from, logits_to or n) are written to `logits_out` (default: the internal buffer) and
        returned.
        batch=True: `n` rows for each of the B sequences of the engine, in tree-relative addressing of each one's state
        row (state (B, 16), tokens / position_ids / storage_ids (B, M)); activation rows are sequence-major, so the
        row-wise ops and the GEMMs see B*n rows and logits_from / logits_to index those."""
        B = self.B if batch else 1
        N = n * B
        assert 0 < N <= self.n_max
        assert not batch or (state is not None and dense_mask is None)
        H, Hkv, D, M = self.H, self.Hkv, self.D, self.M
        small = (not batch and self.draft_plan is not None and state is not None and n <= ops.DraftPlan.MAX_ROWS
                 and dense_mask is None)
        if batch:
            ops.embed_rows_batch(self.embed, tokens, n, self.hidden, state, n0=n0)
        else:
            ops.embed_rows(self.embed, tokens, n, self.hidden, state=state, n0=n0)
        n_seq, n = n, N                                # from here on n counts the rows of all sequences
        ops.rmsnorm(self.hidden, self.layers[0]["ln1"], self.normed, n, self.eps)
        for l, ly in enumerate(self.layers):
            self._project(ly, "wqkv", self.normed, n, self.qkv)
            if batch:
                ops.rope_kv_append_batch(self.qkv, H, Hkv, D, self.cos, self.sin, position_ids, storage_ids, n_seq,
                                         self.k_cache[l], self.v_cache[l], M, state, n0=n0)
                ops.tree_attn_batch(self.plan, l, n_seq, state=state, n0=n0, kv_end=kv_end, tree_bits=tree_bits,
                                    tree_words=tree_words, tree_size=tree_size)
            else:
                ops.rope_kv_append(self.qkv, H, Hkv, D, self.cos, self.sin, position_ids, storage_ids, n,
                                   self.k_cache[l], self.v_cache[l], M, state=state, n0=n0)
                if small:
                    self.draft_plan.attention(l, n, self.qkv, self.attn_out, state, n0, kv_end, tree_bits, tree_words,
                                              tree_size)
                else:
                    ops.tree_attn(self.plan, l, n, state=state, n0=n0, kv_end=kv_end, prefix_len=prefix_len,
                                  dense_mask=dense_mask, mask_ld=mask_ld, tree_bits=tree_bits, tree_words=tree_words,
                                  tree_size=tree_size)
            nxt = self.layers[l + 1]["ln1"] if l + 1 < self.L else self.norm
            if self.peer is not None:
                torch.mm(self.attn_out[:n], ly["wo"].t(), out=self.peer.buf[0][:n])
                self.peer.allreduce_add_rmsnorm(0, self.hidden, ly["ln2"], self.normed, n, self.eps)
                self._gate_up_act(ly, n)
                torch.mm(self.act[:n], ly["wd"].t(), out=self.peer.buf[1][:n])
                self.peer.allreduce_add_rmsnorm(1, self.hidden, nxt, self.normed, n, self.eps)
                continue
            self._project(ly, "wo", self.attn_out, n, self.proj)
            self.tp.all_reduce(self.proj[:n])
            ops.add_rmsnorm(self.hidden, self.proj, ly["ln2"], self.normed, n, self.eps)
            self._gate_up_act(ly, n)
            self._project(ly, "wd", self.act, n, self.proj)
            self.tp.all_reduce(self.proj[:n])
            ops.add_rmsnorm(self.hidden, self.proj, nxt, self.normed, n, self.eps)
        if skip_lm_head:                               # TP follower ranks: only rank 0 consumes logits
            return None
        end = n if logits_to is None else logits_to
        m = end - logits_from
        out = logits_out if logits_out is not None else self.logits[:m]
        if self.lm_plan is not None and m <= 128 and out.stride(-1) == 1 and out.stride(0) % 8 == 0 and out.data_ptr() % 16 == 0:
            self.lm_plan.run(m, a_row0=logits_from, out=out)
        else:
            torch.mm(self.normed[logits_from:end], self.lm_head.t(), out=out)
        return out
