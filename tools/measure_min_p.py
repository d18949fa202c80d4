"""Cost of the min-p filter: the kernel alone, and a BatchTree decode step with and without it.

Kernels: device time per launch of sq_min_p_filter_per_seq (every sequence at min_p 0.05 and T 0.6, 128 rows per
sequence) on randn * 2 fp16 rows, from CUDA events around a CUDA graph of `--launches` launches.  The filter works in
place, so each launch is preceded by a copy of the unfiltered rows; the copy is timed alone and subtracted.  Shapes:
128 x 32000 (config 2, one sequence), 4*128 and 8*128 x 128256 (Llama 3, B = 4 and 8).

Steps: config 2 (random-init llama-68m -> llama-2-7b, V = 32000, the 128-node growmap A100-CNN-68m-7b-stochastic.pt,
T 0.6, top_p 1, M 384, seeded) as a BatchTree at B = 1 and 4, min_p 0 and 0.1 alternating `--reps` times in one process.
Each run builds the tree on 128-token prompts, runs 3 steps untimed (graph captures), then times `--steps` steps
(construct_grow_map + verify, which ends in the step's host sync) with a host clock; the median ms per step is reported.
The GPU name and power limit are read in the same run.

    python tools/measure_min_p.py [--out result.json] [--reps 3] [--steps 20] [--launches 200]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
DEV = "cuda:0"
GROWMAP = "A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"
M, T, PREFIX, S = 384, 0.6, 128, 128
DRAFT, TARGET = "random-init:llama-68m:1", "random-init:llama-2-7b:2"
KERNEL_CASES = [(128, 32000), (4 * 128, 128256), (8 * 128, 128256)]
MIN_P_KERNEL, MIN_P_STEP = 0.05, 0.1


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = [x.strip() for x in q.split(",")]
    return dict(gpu=name, power_limit=limit)


def per_launch(fn, n):
    """device time per call of fn: n calls captured in one CUDA graph, so the host's enqueue cost is not timed"""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    ev[0].record()
    g.replay()
    ev[1].record()
    torch.cuda.synchronize()
    return 1e3 * ev[0].elapsed_time(ev[1]) / n                  # us


def kernel_times(n_launch):
    from sequoia_b200 import ops
    out = []
    for rows, V in KERNEL_CASES:
        g = torch.Generator(device=DEV).manual_seed(rows + V)
        src = (torch.randn(rows, V, generator=g, device=DEV) * 2).to(torch.float16)
        x = src.clone()
        lmp = torch.full((rows // S,), math.log(MIN_P_KERNEL), dtype=torch.float32, device=DEV)
        temp = torch.full((rows // S,), T, dtype=torch.float32, device=DEV)
        copy = per_launch(lambda: x.copy_(src), n_launch)
        per_seq = per_launch(lambda: (x.copy_(src), ops.min_p_filter_per_seq_(x, lmp, temp, S)), n_launch) - copy
        kept = float((~torch.isinf(x)).float().mean())
        mb = rows * V * 2 / 1e6                                  # the row is read once; most 16-byte chunks are rewritten
        out.append(dict(rows=rows, V=V, min_p=MIN_P_KERNEL, T=T, copy_us=copy, min_p_filter_per_seq_us=per_seq,
                        row_MB=mb, kept_fraction=kept))
        print(json.dumps(out[-1]), flush=True)
    return out


def step_times(engines, prompts, gm, min_p, seeds, steps):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    tree = BatchTree(d, t, prompts, gm, policy="spec", temperature=T, top_p=1.0, max_length=M, seeds=seeds, min_p=min_p)
    for _ in range(3):
        tree.construct_grow_map()
        tree.verify()
    times = []
    for _ in range(steps):
        if any(tree.frozen):
            break
        t0 = time.perf_counter()
        tree.construct_grow_map()
        tree.verify()                                      # ends in the step's one host sync
        times.append(time.perf_counter() - t0)
    assert tree.use_min_p == (min_p > 0)
    return times


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_min_p needs a CUDA device")
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    out = dict(gpu_info())
    out["kernels"] = kernel_times(args.launches)
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(3, 32000, (PREFIX,), generator=g).to(DEV) for _ in range(4)]
    out["steps"] = {}
    for B in (1, 4):
        engines = (GraphInferenceEngine(M, DRAFT, device=DEV, batch_size=B),
                   GraphInferenceEngineTG(M, TARGET, device=DEV, batch_size=B))
        times = {0.0: [], MIN_P_STEP: []}
        for rep in range(args.reps):
            for p in times:
                times[p] += step_times(engines, prompts[:B], gm, p, [100 * rep + b for b in range(B)], args.steps)
        res = {f"min_p_{k}": dict(ms_per_step=1e3 * statistics.median(v), steps=len(v),
                                  ms_min=1e3 * min(v), ms_max=1e3 * max(v)) for k, v in times.items()}
        out["steps"][f"B{B}"] = res
        print(json.dumps({f"B{B}": res}), flush=True)
        del engines
        torch.cuda.empty_cache()
    out["workload"] = (f"config 2, 128-node tree, T {T}, top_p 1, M {M}, {PREFIX}-token prompts, seeded; "
                       f"{args.reps} alternating reps of {args.steps} steps")
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
