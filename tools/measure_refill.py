"""Keeping a batch full: chunked decoding against refill (BatchTree.admit) on the config-2 shapes (random-init
llama-68m -> llama-2-7b, A100-CNN-68m-7b-stochastic.pt, T 0.6, top_p 1, M 384).

16 prompts of 128 tokens, each with a new-token budget drawn from a seeded range: random-init weights rarely emit EOS,
so the budgets stand in for request lengths.  With M 384 and the 128-node tree a 128-token prompt has room for about 129
new tokens; past that the tree stops the sequence in both modes, so larger budgets would not bind and the budgets are
drawn from 32..128.  Per B (4 and 8), on the same engines, prompts and budgets:

* chunked: B prompts at a time (testbed.py --batch B), a chunk runs until its longest sequence stops;
* refill: one BatchTree whose finished slots take the next prompt (testbed.py --batch B --refill).

The two alternate `--reps` times in one process.  Reported: aggregate tokens/s (host clock around the whole decode of the
16 prompts, BatchTree construction included, ending in a device synchronise), and for refill the ms per steady step and
per admission step (admit + draft + verify; testbed.decode_refill's step timer, each step ends in verify's host sync).
The GPU name and power limit are read in the same run.

    python tools/measure_refill.py --out result.json [--reps 2 --batches 4,8]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
DEV = "cuda:0"
GROWMAP = "A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"
M, T, PREFIX, N_PROMPTS, BUDGET = 384, 0.6, 128, 16, (32, 128)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = [x.strip() for x in q.split(",")]
    return dict(gpu=name, power_limit=limit)


def run_chunked(draft, target, prompts, limits, gm, B):
    import testbed
    from sequoia_b200.batch import BatchTree
    decoded = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(0, len(prompts), B):
        tree = BatchTree(draft, target, prompts[i:i + B], gm, policy="spec", temperature=T, top_p=1.0, max_length=M)
        d, _ = testbed.decode_chunk(tree, prompts[i:i + B], limits[i:i + B])
        decoded += d
    torch.cuda.synchronize()
    return decoded, time.perf_counter() - t0


def run_refill(draft, target, prompts, limits, gm, B):
    import testbed
    from sequoia_b200.batch import BatchTree
    times = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tree = BatchTree(draft, target, prompts[:B], gm, policy="spec", temperature=T, top_p=1.0, max_length=M)
    _, decoded, _, _ = testbed.decode_refill(tree, prompts, limits, step_times=times)
    torch.cuda.synchronize()
    return decoded, time.perf_counter() - t0, times


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--batches", default="4,8")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_refill needs a CUDA device")
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(3, 32000, (PREFIX,), generator=g).to(DEV) for _ in range(N_PROMPTS)]
    rng = random.Random(11)
    budgets = [rng.randint(*BUDGET) for _ in range(N_PROMPTS)]
    limits = [PREFIX + n for n in budgets]
    out = dict(gpu_info(), workload="c2: llama-68m -> llama-2-7b (random init), 128-node tree, T 0.6, M 384, "
               f"{N_PROMPTS} prompts of {PREFIX} tokens", budgets=budgets, runs=[])
    for B in [int(x) for x in args.batches.split(",")]:
        draft = GraphInferenceEngine(M, "random-init:llama-68m:1", device=DEV, batch_size=B)
        target = GraphInferenceEngineTG(M, "random-init:llama-2-7b:2", device=DEV, batch_size=B)
        torch.manual_seed(0)
        run_refill(draft, target, prompts[:B], limits[:B], gm, B)          # warm-up: modules, allocator, algorithms
        res = dict(B=B, chunked=[], refill=[])
        steady, admission = [], []
        for _ in range(args.reps):
            torch.manual_seed(0)
            d, s = run_chunked(draft, target, prompts, limits, gm, B)
            res["chunked"].append(dict(tokens=d, seconds=s, tokens_per_s=d / s))
            torch.manual_seed(0)
            d, s, times = run_refill(draft, target, prompts, limits, gm, B)
            res["refill"].append(dict(tokens=d, seconds=s, tokens_per_s=d / s))
            steady += [t for k, t in times if k == "steady"]
            admission += [t for k, t in times if k == "admission"]
        res["refill_ms_per_steady_step"] = 1e3 * statistics.median(steady)
        res["refill_ms_per_admission_step"] = 1e3 * statistics.median(admission)
        res["steady_steps"], res["admission_steps"] = len(steady), len(admission)
        res["gain"] = (statistics.mean(r["tokens_per_s"] for r in res["refill"]) /
                       statistics.mean(r["tokens_per_s"] for r in res["chunked"]))
        out["runs"].append(res)
        print(json.dumps(res), flush=True)
        del draft, target
        torch.cuda.empty_cache()
    print(json.dumps(out))
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
