"""Seeded input generators shared by tests/golden/make_golden.py and the test-suite.

Inputs are regenerated from seeds at test time (same image => same torch CPU RNG stream);
only OUTPUTS of the reference are committed under tests/golden/.
"""
import hashlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.sequoia_oracle import LlamaCfg, init_llama_weights  # noqa: E402

V = 32000

# tiny Llama shapes that exercise both head dims the CUDA attention kernel is built for
CFG_DRAFT = LlamaCfg(hidden_size=256, intermediate_size=688, num_hidden_layers=2,
                     num_attention_heads=4, num_key_value_heads=4, vocab_size=V)          # D = 64
CFG_TARGET = LlamaCfg(hidden_size=512, intermediate_size=1024, num_hidden_layers=3,
                      num_attention_heads=4, num_key_value_heads=4, vocab_size=V)         # D = 128
CFG_TARGET_GQA = LlamaCfg(hidden_size=512, intermediate_size=1024, num_hidden_layers=2,
                          num_attention_heads=4, num_key_value_heads=2, vocab_size=V)     # D = 128, GQA

DRAFT_SEED, TARGET_SEED, GQA_SEED = 101, 202, 303


def log_line(name: str, line: str):
    """Append a measured number to <SEQUOIA_TEST_LOG_DIR or the temp dir>/sequoia_test_logs/<name> (outside the tree)."""
    import tempfile
    out = os.environ.get("SEQUOIA_TEST_LOG_DIR", os.path.join(tempfile.gettempdir(), "sequoia_test_logs"))
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, name), "a") as f:
        f.write(line + "\n")


def growmap_path(name: str) -> str:
    return os.path.join(ROOT, name)


def load_growmap(name: str) -> dict:
    return torch.load(growmap_path(name))


def make_prompt(seed: int, n: int = 128) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randint(3, V, (n,), generator=g)


def pack_mask(m: torch.Tensor) -> dict:
    """bool matrix -> bit-packed form for the golden files (an 895 x 895 mask is 100 KB instead of 800 KB)."""
    import numpy as np
    return {"shape": tuple(m.shape), "bits": torch.from_numpy(np.packbits(m.numpy().reshape(-1)))}


def unpack_mask(p) -> torch.Tensor:
    import numpy as np
    n = int(np.prod(p["shape"]))
    return torch.from_numpy(np.unpackbits(p["bits"].numpy())[:n].astype(bool)).view(*p["shape"])


def sha(t: torch.Tensor) -> str:
    t = t.detach().cpu().contiguous()
    return hashlib.sha256(t.view(torch.uint8).numpy().tobytes()).hexdigest()


def sampling_case(seed: int, rows: int, peaked: bool):
    """(logits fp16 (rows,V), rand fp16 (rows,V)) like SpecTree sees them."""
    g = torch.Generator().manual_seed(seed)
    scale = 4.0 if peaked else 0.5
    logits = (torch.randn(rows, V, generator=g) * scale).to(torch.float16)
    rand = torch.empty(rows, V, dtype=torch.float16).uniform_(generator=g)
    return logits, rand


def residual_case(seed: int):
    g = torch.Generator().manual_seed(seed)
    p = torch.softmax((torch.randn(V, generator=g) * 3).to(torch.float16) / 0.6, dim=-1)
    q = torch.softmax((torch.randn(V, generator=g) * 3).to(torch.float16) / 0.6, dim=-1)
    return p, q


DECODE_CASES = {
    # name: (growmap, mode, draft cfg/seed, target cfg/seed, M, prompt seed, prefix, iters, rng seed)
    "greedy_2chain": ("L40_growmaps/2-chain.pt", "greedy", "draft", "target", 256, 11, 96, 6, 17),
    "greedy_4x4": ("L40_growmaps/4x4-tree.pt", "greedy", "draft", "target", 256, 12, 64, 5, 17),
    "spec_8x8": ("L40_growmaps/8x8-tree.pt", "spec", "draft", "target", 256, 25, 100, 5, 17),
    "spec_a100_128": ("A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt", "spec", "draft", "target_gqa",
                      384, 22, 128, 4, 17),
    # draft == target weights: forces deep acceptance paths / multi-row KV gathers
    "spec_same_8x8": ("L40_growmaps/8x8-tree.pt", "spec", "draft", "draft", 256, 26, 80, 5, 17),
    "greedy_same_16chain": ("L40_growmaps/16-chain.pt", "greedy", "draft", "draft", 256, 16, 70, 4, 17),
    # config-4 tree shape (768 nodes, 18 levels, M=1024): 6 query tiles x 8 KV splits in the attention kernel
    "spec_l40_768": ("L40_growmaps/L40-CNN-7b-70b-stochastic.pt", "spec", "draft", "target_gqa", 1024, 31, 128, 2, 17),
}

# policy variants (SURVEY.md 8f.3): GreedySTree (sampled target token) and SpecInferTree (i.i.d. children, >=, no masking)
VARIANT_CASES = {
    "greedys_4x4": ("L40_growmaps/4x4-tree.pt", "greedys", "draft", "target", 256, 12, 64, 5, 17),
    "greedys_same_4x4": ("L40_growmaps/4x4-tree.pt", "greedys", "draft", "draft", 256, 13, 64, 5, 17),
    "specinfer_8x8": ("L40_growmaps/8x8-tree.pt", "specinfer", "draft", "target", 256, 25, 100, 5, 17),
    "specinfer_same_8x8": ("L40_growmaps/8x8-tree.pt", "specinfer", "draft", "draft", 256, 26, 80, 5, 17),
}

# reference sweep shapes (tests/run.sh: K chains of length L, driven there through SpecInferTree); oracle-vs-reference only
SWEEP_CASES = {
    "sweep_specinfer_8x1": ("L40_growmaps/8x1-tree.pt", "specinfer", "draft", "target", 256, 51, 64, 3, 17),
    "sweep_specinfer_1x8": ("L40_growmaps/1x8-tree.pt", "specinfer", "draft", "draft", 256, 52, 64, 3, 17),
    "sweep_specinfer_2x32": ("L40_growmaps/2x32-tree.pt", "specinfer", "draft", "draft", 256, 53, 64, 3, 17),
    "sweep_specinfer_128x1": ("L40_growmaps/128x1-tree.pt", "specinfer", "draft", "target", 384, 54, 64, 3, 17),
    "sweep_spec_16x8": ("L40_growmaps/16x8-tree.pt", "spec", "draft", "target", 384, 55, 64, 3, 17),
    # M = 512 as in tests/run.sh: draft == target accepts all 128 nodes per step, and 64 + 2 x 129 + 127 slots exceed 384
    "sweep_greedy_1x128": ("L40_growmaps/1x128-tree.pt", "greedy", "draft", "draft", 512, 56, 64, 2, 17),
    "sweep_greedys_5x8": ("L40_growmaps/5x8-tree.pt", "greedys", "draft", "draft", 256, 57, 64, 3, 17),
}

# Every instantiation of gemm_tn_kernel<BN, STAGES, SPLIT, MC> that sq_gemm.cu's run_tile can launch, in table order.
# test_gpu_kernels.py forces each one through SQ_GEMM_FORCE; test_cabi.py checks this list against the SQ_G(...) lines.
GEMM_VARIANTS = [
    (256, 4, 1, 1), (256, 4, 1, 2),
    (192, 5, 1, 1), (192, 5, 1, 2),
    (128, 6, 1, 1), (128, 6, 1, 2), (128, 4, 2, 1), (128, 4, 4, 1), (128, 4, 2, 2), (128, 4, 4, 2),
    (64, 8, 1, 1), (64, 8, 1, 2), (64, 4, 2, 1), (64, 4, 4, 1), (64, 4, 2, 2), (64, 4, 4, 2),
]

_MODELS = {"draft":(CFG_DRAFT, DRAFT_SEED), "target": (CFG_TARGET, TARGET_SEED),
           "target_gqa": (CFG_TARGET_GQA, GQA_SEED)}
_wcache = {}


def model_weights(key: str):
    if key not in _wcache:
        cfg, seed = _MODELS[key]
        _wcache[key] = (cfg, init_llama_weights(cfg, seed))
    return _wcache[key]
