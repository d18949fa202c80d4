"""Cost of the per-sequence logit bias and allowed-token sets: the kernel alone, and a BatchTree decode step with and
without them.

Kernel: device time per sq_logit_bias_rows_batch call on the config-2 growmap (128 nodes) at V = 32000 and 128256, B = 1,
4 and 8, from CUDA events around a CUDA graph of `--launches` calls.  The call works in place, so each one is preceded by
a copy of the unprocessed rows; the copy is timed alone and subtracted.  Cases: bias only (1024 entries), a mask of 100
allowed ids, a mask of V/2 allowed ids (random ids, so nearly every 8-id group is mixed).  Reported with each time: the
bytes the kernel reads and writes (mask words and entries included) and their share of the H100's 3.35 TB/s.

Steps: config 2 (random-init llama-68m -> llama-2-7b, V = 32000, the 128-node growmap A100-CNN-68m-7b-stochastic.pt,
T 0.6, top_p 1, M 384, seeded) as a BatchTree at B = 1 and 4, with three settings alternated `--reps` times in one
process: off, 64 bias entries, and an allowed set of 1000 ids.  Each run builds the tree on 128-token prompts, runs 3
steps untimed (graph captures), then times `--steps` steps (construct_grow_map + verify, which ends in the step's host
sync) with a host clock.  Reported: the median ms per step with its range, and the tokens each sequence committed per
step.  The GPU name and power limit are read in the same run.

    python tools/measure_logit_bias.py [--out result.json] [--reps 3] [--steps 20] [--launches 200]
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
HBM_BYTES_PER_S = 3.35e12
G = torch.Generator().manual_seed(7)
SETTINGS = {"off": {},
            "bias64": dict(logit_bias={int(t): 1.5 for t in torch.randperm(32000, generator=G)[:64]}),
            "allowed1000": dict(allowed_token_ids=sorted(torch.randperm(32000, generator=G)[:1000].tolist()))}


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


def _bytes(x, S, allowed, n_bias):
    """Bytes the kernel moves: per masked row, every 8-id group that is not all allowed is written (16 B), and read
    (16 B) unless it is all disallowed; its mask word reads (4 B per group); each bias entry's id, value and logit."""
    V = x.shape[1]
    total = 0
    for b, ids in enumerate(allowed):
        if ids is not None:
            ok = torch.zeros(V, dtype=torch.bool)
            ok[torch.tensor(ids)] = True
            n_ok = ok.view(-1, 8).sum(1)
            groups = n_ok.numel()
            total += S * (4 * groups + 16 * int((n_ok < 8).sum()) + 16 * int(((n_ok > 0) & (n_ok < 8)).sum()))
        total += S * n_bias[b] * (4 + 4 + 2 + 2)
    return total


def kernel_times(gm, n_launch):
    from sequoia_b200 import ops
    S = gm["size"]
    out = []
    for V in (32000, 128256):
        for B in (1, 4, 8):
            g = torch.Generator().manual_seed(V + B)
            src = (torch.randn(B * S, V, generator=g) * 2).to(torch.float16).to(DEV)
            x = src.clone()
            state = torch.zeros(B, 16, dtype=torch.int32, device=DEV)
            bias_ids = torch.stack([torch.randperm(V, generator=g)[:1024].sort().values for _ in range(B)])
            cases = {"bias1024": ([None] * B, [1024] * B),
                     "mask100": ([torch.randperm(V, generator=g)[:100].tolist() for _ in range(B)], [0] * B),
                     "maskV/2": ([torch.randperm(V, generator=g)[:V // 2].tolist() for _ in range(B)], [0] * B)}
            for name, (allowed, n_bias) in cases.items():
                mask = torch.stack([ops.pack_token_mask(a, V) if a is not None else
                                    torch.zeros(ops.mask_words(V), dtype=torch.int32) for a in allowed]).to(DEV)
                has = torch.tensor([a is not None for a in allowed], dtype=torch.int32, device=DEV)
                ids = bias_ids.to(torch.int32).to(DEV)
                vals = torch.full((B, 1024), 1.5, dtype=torch.float32, device=DEV)
                n = torch.tensor(n_bias, dtype=torch.int32, device=DEV)

                def call():
                    x.copy_(src)
                    ops.logit_bias_rows_batch_(x, S, state, mask, has, ids, vals, n)
                copy = per_launch(lambda: x.copy_(src), n_launch)
                us = per_launch(call, n_launch) - copy
                nbytes = _bytes(x, S, allowed, n_bias)
                out.append(dict(V=V, B=B, case=name, copy_us=copy, kernel_us=us, bytes=nbytes,
                                hbm_share=nbytes / (us * 1e-6) / HBM_BYTES_PER_S if us > 0 else None))
                print(json.dumps(out[-1]), flush=True)
    return out


def step_times(engines, prompts, gm, seeds, steps, kw):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    d.clear_kv()
    t.clear_kv()
    tree = BatchTree(d, t, prompts, gm, policy="spec", temperature=T, top_p=1.0, max_length=M, seeds=seeds, **kw)
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
    assert tree.use_logit_bias == bool(kw)
    return times, new


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_logit_bias needs a CUDA device")
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    out = dict(gpu_info())
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    out["kernels"] = kernel_times(gm, args.launches)
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(3, 32000, (PREFIX,), generator=g).to(DEV) for _ in range(4)]
    out["steps"] = {}
    for B in (1, 4):
        engines = (GraphInferenceEngine(M, DRAFT, device=DEV, batch_size=B),
                   GraphInferenceEngineTG(M, TARGET, device=DEV, batch_size=B))
        times = {k: [] for k in SETTINGS}
        new = {k: [] for k in SETTINGS}
        per_rep = {k: [] for k in SETTINGS}
        for rep in range(args.reps):
            for name, kw in SETTINGS.items():
                t, n = step_times(engines, prompts[:B], gm, [100 * rep + b for b in range(B)], args.steps, kw)
                times[name] += t
                new[name] += n
                per_rep[name].append(1e3 * statistics.median(t))
        res = {name: dict(ms_per_step=1e3 * statistics.median(times[name]), ms_min=1e3 * min(times[name]),
                          ms_max=1e3 * max(times[name]), rep_medians_ms=per_rep[name], steps=len(times[name]),
                          tokens_per_step=statistics.mean(new[name]), tokens_per_step_min=min(new[name]),
                          tokens_per_step_max=max(new[name]))
               for name in SETTINGS}
        out["steps"][f"B{B}"] = res
        print(json.dumps({f"B{B}": res}), flush=True)
        del engines
        torch.cuda.empty_cache()
    out["workload"] = (f"config 2, 128-node tree, T {T}, top_p 1, M {M}, {PREFIX}-token prompts, seeded; settings "
                       f"off / 64 bias entries of +1.5 / 1000 allowed ids; {args.reps} alternating reps of "
                       f"{args.steps} steps")
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
