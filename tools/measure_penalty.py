"""Cost of the per-sequence penalties: the kernels alone, and a BatchTree decode step with and without them.

Kernels: device time per sq_penalize_rows_batch call (its two launches) on the config-2 growmap (128 nodes) at V = 32000
and 128256, B = 1, 4 and 8, from CUDA events around a CUDA graph of `--launches` calls.  The call works in place, so each
one is preceded by a copy of the unpenalised rows; the copy is timed alone and subtracted.  Histories: M = 384 and the
cap M = 4096, each with P = M - 127 (the longest history a tree of 128 nodes leaves room for), prompt length P - 64,
token ids drawn from 0 .. 999 (many repeats) and uniformly from V (many distinct ids) in equal parts.

Steps: config 2 (random-init llama-68m -> llama-2-7b, V = 32000, the 128-node growmap A100-CNN-68m-7b-stochastic.pt,
T 0.6, top_p 1, M 384, seeded) as a BatchTree at B = 1 and 4, penalties off and then repetition_penalty 1.1 with
presence_penalty 0.5, alternating `--reps` times in one process.  Each run builds the tree on 128-token prompts, runs 3
steps untimed (graph captures), then times `--steps` steps (construct_grow_map + verify, which ends in the step's host
sync) with a host clock.  Reported: the median ms per step with its range, and the tokens each sequence committed per
step.  The GPU name and power limit are read in the same run.

    python tools/measure_penalty.py [--out result.json] [--reps 3] [--steps 20] [--launches 200]
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
PENALTY = dict(repetition_penalty=1.1, presence_penalty=0.5)


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
    from sequoia_b200.tree import _Static
    st = _Static(gm, DEV)
    S = st.S
    out = []
    for V in (32000, 128256):
        for B in (1, 4, 8):
            for Mx in (384, 4096):
                g = torch.Generator(device=DEV).manual_seed(V + B + Mx)
                src = (torch.randn(B * S, V, generator=g, device=DEV) * 2).to(torch.float16)
                x = src.clone()
                tokens = torch.where(torch.rand(B, Mx, generator=g, device=DEV) < 0.5,
                                     torch.randint(0, 1000, (B, Mx), generator=g, device=DEV),
                                     torch.randint(0, V, (B, Mx), generator=g, device=DEV))
                P = Mx - S + 1
                state = torch.zeros(B, 16, dtype=torch.int32, device=DEV)
                state[:, 0] = P
                plen = torch.full((B,), P - 64, dtype=torch.int32, device=DEV)
                rep, freq, pres = (torch.full((B,), v, dtype=torch.float32, device=DEV) for v in (1.1, 0.2, 0.5))
                scratch = torch.empty(ops.penalty_scratch_words(B, Mx), dtype=torch.int32, device=DEV)
                distinct = [len(set(tokens[b, :P].tolist())) for b in range(B)]

                def call():
                    x.copy_(src)
                    ops.penalize_rows_batch_(x, tokens, state, plen, st.tree_bits, st.tree_words, S, rep, freq, pres,
                                             scratch)
                copy = per_launch(lambda: x.copy_(src), n_launch)
                pen = per_launch(call, n_launch) - copy
                out.append(dict(V=V, B=B, M=Mx, P=P, distinct_ids=max(distinct), copy_us=copy, penalize_us=pen))
                print(json.dumps(out[-1]), flush=True)
    return out


def step_times(engines, prompts, gm, seeds, steps, pen):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    d.clear_kv()
    t.clear_kv()
    tree = BatchTree(d, t, prompts, gm, policy="spec", temperature=T, top_p=1.0, max_length=M, seeds=seeds,
                     **(PENALTY if pen else {}))
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
    assert tree.use_penalty == pen
    return times, new


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_penalty needs a CUDA device")
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
        times, new = {False: [], True: []}, {False: [], True: []}
        per_rep = {False: [], True: []}
        for rep in range(args.reps):
            for pen in (False, True):
                t, n = step_times(engines, prompts[:B], gm, [100 * rep + b for b in range(B)], args.steps, pen)
                times[pen] += t
                new[pen] += n
                per_rep[pen].append(1e3 * statistics.median(t))
        res = {("penalties" if pen else "off"): dict(ms_per_step=1e3 * statistics.median(times[pen]),
                                                     ms_min=1e3 * min(times[pen]), ms_max=1e3 * max(times[pen]),
                                                     rep_medians_ms=per_rep[pen], steps=len(times[pen]),
                                                     tokens_per_step=statistics.mean(new[pen]),
                                                     tokens_per_step_min=min(new[pen]),
                                                     tokens_per_step_max=max(new[pen]))
               for pen in (False, True)}
        out["steps"][f"B{B}"] = res
        print(json.dumps({f"B{B}": res}), flush=True)
        del engines
        torch.cuda.empty_cache()
    out["workload"] = (f"config 2, 128-node tree, T {T}, top_p 1, M {M}, {PREFIX}-token prompts, seeded; penalties "
                       f"{PENALTY}; {args.reps} alternating reps of {args.steps} steps")
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
