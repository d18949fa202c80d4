"""Cost of the per-sequence logprobs: the kernel alone, and a BatchTree decode step with logprobs off, n = 0 and n = 20.

Kernel: device time per sq_token_logprobs_batch call at B = 1 and 8, V = 32000 and 128256, n = 0 and 20, from CUDA events
around a CUDA graph of `--launches` calls.  Each sequence committed the deepest path of the config-2 growmap (128 nodes,
depth 5) and its bonus token: 6 positions, each one CTA that reads its row.  Reported with the bytes a step must read
(each committed position's row once, 2 bytes per entry) and the share of the H100 SXM's 3.35 TB/s HBM3 bandwidth that
reading them in the measured time would take (the kernel reads each row three times at n > 0 and twice at n = 0, the
later reads mostly from L2).

Steps: config 2 (random-init llama-68m -> llama-2-7b, V = 32000, the 128-node growmap A100-CNN-68m-7b-stochastic.pt,
T 0.6, top_p 1, M 384, seeded) as a BatchTree at B = 1 and 8, with logprobs off, 0 and 20, alternating `--reps` times in
one process.  Each run builds the tree on 128-token prompts, runs 3 steps untimed (graph captures), then times `--steps`
steps (construct_grow_map + verify, which ends in the step's host sync) with a host clock.  Reported: the median ms per
step with its range, and the tokens each sequence committed per step.  The GPU name and power limit are read in the
same run.

    python tools/measure_logprobs.py [--out result.json] [--reps 3] [--steps 20] [--launches 200]
"""
import argparse
import json
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
M, T, PREFIX = 384, 0.6, 128
DRAFT, TARGET = "random-init:llama-68m:1", "random-init:llama-2-7b:2"
HBM_BYTES_PER_S = 3.35e12                                      # H100 SXM data sheet


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


def kernel_times(gm, n_launch):
    from sequoia_b200 import ops
    S, D = gm["size"], int(gm["depth"].max())
    k = int(gm["depth"].argmax())
    path = sorted((j for j in range(1, S) if bool(gm["mask"][k, j])), key=lambda j: int(gm["depth"][j]))
    out = []
    for V in (32000, 128256):
        for B in (1, 8):
            g = torch.Generator(device=DEV).manual_seed(V + B)
            x = (torch.randn(B * S, V, generator=g, device=DEV) * 2).to(torch.float16)
            tokens = torch.randint(0, V, (B, M), generator=g, device=DEV)
            P = M - S
            state = torch.zeros(B, 16, dtype=torch.int32, device=DEV)
            state[:, 3], state[:, 4], state[:, 8] = len(path), P, M
            acc = torch.zeros(B, S, dtype=torch.int32, device=DEV)
            acc[:, :len(path)] = torch.tensor([P - 1 + j for j in path], dtype=torch.int32, device=DEV)
            Ts = torch.full((B,), T, dtype=torch.float32, device=DEV)
            greedy = torch.zeros(B, dtype=torch.int32, device=DEV)
            lp_token = torch.empty(B, M, dtype=torch.float32, device=DEV)
            lp_ids = torch.empty(B, M, 20, dtype=torch.int32, device=DEV)
            lp_top = torch.empty(B, M, 20, dtype=torch.float32, device=DEV)
            positions = B * (len(path) + 1)
            for n in (0, 20):
                n_top = torch.full((B,), n, dtype=torch.int32, device=DEV)
                us = per_launch(lambda: ops.token_logprobs_batch_(x, S, D, tokens, state, acc, Ts, greedy, n_top,
                                                                  lp_token, lp_ids, lp_top), n_launch)
                nbytes = positions * V * 2
                out.append(dict(V=V, B=B, n=n, positions=positions, us=us, bytes_per_step=nbytes,
                                hbm_bound_share=nbytes / HBM_BYTES_PER_S / (us * 1e-6)))
                print(json.dumps(out[-1]), flush=True)
    return out


def step_times(engines, prompts, gm, seeds, steps, n):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    d.clear_kv()
    t.clear_kv()
    tree = BatchTree(d, t, prompts, gm, policy="spec", temperature=T, top_p=1.0, max_length=M, seeds=seeds, logprobs=n)
    for _ in range(3):
        tree.construct_grow_map()
        res = tree.verify()
    lengths = [len(v) for v, _, _ in res]
    times, new = [], []
    for _ in range(steps):
        if any(tree.frozen):
            break
        t0 = time.perf_counter()
        tree.construct_grow_map()
        res = tree.verify()                                     # ends in the step's one host sync
        times.append(time.perf_counter() - t0)
        for b, (v, _, _) in enumerate(res):
            new.append(len(v) - lengths[b])
            lengths[b] = len(v)
    assert tree.use_logprobs == (n is not None)
    return times, new


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_logprobs needs a CUDA device")
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    out = dict(gpu_info())
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    out["kernels"] = kernel_times(gm, args.launches)
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(3, 32000, (PREFIX,), generator=g).to(DEV) for _ in range(8)]
    out["steps"] = {}
    settings = (None, 0, 20)
    name = {None: "off", 0: "n0", 20: "n20"}
    for B in (1, 8):
        engines = (GraphInferenceEngine(M, DRAFT, device=DEV, batch_size=B),
                   GraphInferenceEngineTG(M, TARGET, device=DEV, batch_size=B))
        times, new, per_rep = ({n: [] for n in settings} for _ in range(3))
        for rep in range(args.reps):
            for n in settings:
                t, k = step_times(engines, prompts[:B], gm, [100 * rep + b for b in range(B)], args.steps, n)
                times[n] += t
                new[n] += k
                per_rep[n].append(1e3 * statistics.median(t))
        res = {name[n]: dict(ms_per_step=1e3 * statistics.median(times[n]), ms_min=1e3 * min(times[n]),
                             ms_max=1e3 * max(times[n]), rep_medians_ms=per_rep[n], steps=len(times[n]),
                             tokens_per_step=statistics.mean(new[n])) for n in settings}
        out["steps"][f"B{B}"] = res
        print(json.dumps({f"B{B}": res}), flush=True)
        del engines
        torch.cuda.empty_cache()
    out["workload"] = (f"config 2, 128-node tree, T {T}, top_p 1, M {M}, {PREFIX}-token prompts, seeded; logprobs off, "
                       f"0 and 20; {args.reps} alternating reps of {args.steps} steps")
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
