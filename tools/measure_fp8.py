"""Cost of FP8 (E4M3) target weights on one GPU.

1. Projections: for the Llama-2-7B, Llama-2-13B and Llama-3.1-8B layer shapes (qkv, o, gate_up, down) at n = 1, 65, 128
   and 256 rows, the fp16 route LlamaRunner takes (torch.mm; gate_up: the fused SwiGLU sq_gemm plan for 96 < n <= 128
   where the runner builds one, torch.mm + sq_silu_mul otherwise) against the FP8 plan (+ sq_silu_mul for gate_up).
   CUDA-event time per call over many calls, and weight bytes/s of each against the H100 SXM data-sheet 3.35 TB/s.
2. Decode: configs c2 (68m -> 7B, 128-node tree) and c3 (68m -> 13B, 8x8 tree) of bench.py, random-init weights, T 0.6,
   M 384, 128-token prompts, SpecTree, with an fp16 and an FP8 target alternated in one process (--runs each): decode and
   verify ms per step (CUDA events around construct_grow_map() and verify() after warm-up steps that capture the graphs),
   accepted tokens per step, tokens/s, and the target's resident weight bytes.

The GPU name and power limit are read in the same run.

    python tools/measure_fp8.py --out result.json [--steps 30 --warmup 4 --runs 2] [--skip-decode]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
DEV = "cuda:0"
F16 = torch.float16
HBM_TBPS = 3.35
CONFIGS = {"c2": ("llama-68m", "llama-2-7b", "A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"),
           "c3": ("llama-68m", "llama-2-13b", "L40_growmaps/8x8-tree.pt")}
M, T, PREFIX = 384, 0.6, 128


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = [x.strip() for x in q.split(",")]
    return dict(gpu=name, power_limit=limit)


def per_call_us(fn, n=50, warmup=5):
    for _ in range(warmup):
        fn()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(n):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) * 1000.0 / n


def projections():
    from sequoia_b200 import ops
    from sequoia_b200.model import NAMED_CONFIGS
    out = {}
    for model in ("llama-2-7b", "llama-2-13b", "llama-3.1-8b"):
        c = NAMED_CONFIGS[model]
        h, I, D = c.hidden_size, c.intermediate_size, c.head_dim
        shapes = {"qkv": ((c.num_attention_heads + 2 * c.num_key_value_heads) * D, h), "o": (h, c.num_attention_heads * D),
                  "gate_up": (2 * I, h), "down": (h, I)}
        for proj, (N, K) in shapes.items():
            w = (torch.randn(N, K, device=DEV) * 0.02).half()
            a = torch.randn(256, K, device=DEV).half()
            c16 = torch.zeros(256, N, dtype=F16, device=DEV)
            act = torch.zeros(256, I, dtype=F16, device=DEV)
            q, s = ops.quantize_fp8(w)
            plan8 = ops.GemmFp8Plan(a, q, s, c16)
            del q
            gu_plan = None
            if proj == "gate_up":
                bn, split, _ = ops.gemm_pick_tiles(N, K, ops.GEMM_SWIGLU)
                if (-(-N // bn)) * split >= 120:                         # LlamaRunner's condition for the fused plan
                    gu_plan = ops.GemmPlan(a, ops.interleave_gate_up(w[:I], w[I:]), act, swiglu=True)
            for n in (1, 65, 128, 256):
                if proj != "gate_up":
                    f16 = lambda: torch.mm(a[:n], w.t(), out=c16[:n])
                    f8 = lambda: plan8.run(n)
                elif gu_plan is not None and 96 < n <= 128:
                    f16 = lambda: gu_plan.run(n)
                    f8 = lambda: (plan8.run(n), ops.silu_mul(c16, act, n))
                else:
                    f16 = lambda: (torch.mm(a[:n], w.t(), out=c16[:n]), ops.silu_mul(c16, act, n))
                    f8 = lambda: (plan8.run(n), ops.silu_mul(c16, act, n))
                us16, us8 = per_call_us(f16), per_call_us(f8)
                b16, b8 = N * K * 2, plan8.weight_bytes()
                r = dict(N=N, K=K, fp16_us=round(us16, 1), fp8_us=round(us8, 1), speedup=round(us16 / us8, 2),
                         fp16_TBps=round(b16 / us16 / 1e6, 2), fp8_TBps=round(b8 / us8 / 1e6, 2),
                         fp8_share_of_3p35=round(b8 / us8 / 1e6 / HBM_TBPS, 3), fp8_plan=plan8.info())
                out[f"{model}/{proj}/n{n}"] = r
                print(f"{model} {proj} n={n}: {r}", flush=True)
            del w, a, c16, act, plan8, gu_plan
            torch.cuda.empty_cache()
    return out


def decode_run(cfg, fmt, steps, warmup, seed):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    from sequoia_b200.tree import SpecTree, clear_runtimes
    dname, tname, gm_path = CONFIGS[cfg]
    gm = torch.load(os.path.join(ROOT, gm_path))
    clear_runtimes()
    draft = GraphInferenceEngine(M, f"random-init:{dname}:1", device=DEV)
    target = GraphInferenceEngineTG(M, f"random-init:{tname}:2", device=DEV, weight_format=fmt)
    prompt = torch.randint(3, 32000, (PREFIX,), generator=torch.Generator().manual_seed(seed))
    torch.manual_seed(seed)
    tree = SpecTree(draft, target, prompt.to(DEV), temperature=T, top_p=1.0, max_length=M, max_target_seq=M, device=DEV,
                    grow_map=gm)
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(3 * steps)]
    length = PREFIX
    for _ in range(warmup):
        tree.construct_grow_map()
        length = len(tree.verify()[0])
    tokens = 0
    for i in range(steps):
        evs[3 * i].record()
        tree.construct_grow_map()
        evs[3 * i + 1].record()
        v = tree.verify()[0]
        evs[3 * i + 2].record()
        tokens, length = tokens + len(v) - length, len(v)
    torch.cuda.synchronize()
    total = sum(evs[3 * i].elapsed_time(evs[3 * i + 2]) for i in range(steps))
    verify = sum(evs[3 * i + 1].elapsed_time(evs[3 * i + 2]) for i in range(steps))
    res = dict(config=cfg, target_weights=fmt, ms_per_step=round(total / steps, 3), verify_ms_per_step=round(verify / steps, 3),
               accepted_tokens_per_step=round(tokens / steps, 3), tokens_per_s=round(tokens / (total / 1e3), 1),
               target_weight_bytes=target.engine.runner.weight_bytes(),
               target_layer_weight_bytes=target.engine.runner.weight_bytes()
               - 2 * sum(t.numel() for t in (target.engine.runner.embed, target.engine.runner.lm_head)), steps=steps)
    del tree, draft, target
    clear_runtimes()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--skip-decode", action="store_true")
    ap.add_argument("--skip-projections", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("measure_fp8.py measures on a CUDA GPU; none is visible")
    res = dict(**gpu_info())
    print(res, flush=True)
    if not args.skip_projections:
        res["projections"] = projections()
    if not args.skip_decode:
        res["decode"] = []
        for cfg in ("c2", "c3"):
            for run in range(args.runs):
                for fmt in ("fp16", "fp8"):
                    r = decode_run(cfg, fmt, args.steps, args.warmup, seed=100 + run)
                    print(f"decode run {run}: {r}", flush=True)
                    res["decode"].append(r)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
