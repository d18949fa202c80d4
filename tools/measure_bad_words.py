"""Cost of the per-sequence bad words and min_tokens: the kernel alone, and a BatchTree decode step with and without them.

Kernel: device time per sq_ban_tokens_rows_batch call on the config-2 growmap (128 nodes) at V = 32000 and 128256 and
B = 1, 4 and 8, from CUDA events around a CUDA graph of `--launches` calls.  Every sequence has the full 128 words of 16
ids each and min_tokens on (every row bans its end ids), the worst case the kernel meets.  The call only writes -inf, so
repeating it in place is the same work each time and needs no copy of the rows.

Steps: config 2 (random-init llama-68m -> llama-2-7b, V = 32000, the 128-node growmap A100-CNN-68m-7b-stochastic.pt,
T 0.6, top_p 1, M 384, seeded) as a BatchTree at B = 1, with two settings alternated `--reps` times in one process:
off, and 128 words of 2-16 ids plus min_tokens 200.  Each run builds the tree on a 128-token prompt, runs 3 steps untimed
(graph captures), then times `--steps` steps (construct_grow_map + verify, which ends in the step's host sync) with a
host clock.  Reported: the median ms per step with its range, and the tokens committed per step.  The GPU name and
power limit are read in the same run.

    python tools/measure_bad_words.py [--out result.json] [--reps 3] [--steps 20] [--launches 200]
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
NW, WL, NS = 128, 16, 8
G = torch.Generator().manual_seed(7)
WORDS = [torch.randint(3, 32000, (2 + i % 15,), generator=G).tolist() for i in range(NW)]
SETTINGS = {"off": {}, "words128_min200": dict(bad_words=WORDS, min_tokens=200)}


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
    S = gm["size"]
    out = []
    for V in (32000, 128256):
        for B in (1, 4, 8):
            g = torch.Generator().manual_seed(V + B)
            x = (torch.randn(B * S, V, generator=g) * 2).to(torch.float16).to(DEV)
            tokens = torch.randint(3, V, (B, M), generator=g).to(DEV)
            state = torch.zeros(B, 16, dtype=torch.int32)
            state[:, 0] = 200
            state = state.to(DEV)
            L = torch.full((B,), 100, dtype=torch.int32, device=DEV)
            words = torch.randint(0, V, (B, NW, WL), generator=g).to(torch.int32).to(DEV)
            lens = torch.full((B, NW), WL, dtype=torch.int32, device=DEV)
            n = torch.full((B,), NW, dtype=torch.int32, device=DEV)
            min_end = torch.full((B,), 100000, dtype=torch.int32, device=DEV)
            ends = torch.tensor([[0, 2, 5, 7, 11, 13, 17, 19]] * B, dtype=torch.int32, device=DEV)

            def call():
                ops.ban_tokens_rows_batch_(x, tokens, state, L, st.depth, st.tree_bits, st.tree_words, S, words, lens,
                                           n, min_end, ends)
            us = per_launch(call, n_launch)
            # per CTA: the word table and lengths of its sequence, the row's path bits and tokens; 8 halves written
            nbytes = B * S * (NW * WL * 4 + NW * 4 + NS * 2)
            out.append(dict(V=V, B=B, kernel_us=us, bytes_per_launch=nbytes))
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
    assert tree.use_ban == bool(kw)
    return times, new


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_bad_words needs a CUDA device")
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    out = dict(gpu_info())
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    out["kernels"] = kernel_times(gm, args.launches)
    g = torch.Generator().manual_seed(3)
    prompt = [torch.randint(3, 32000, (PREFIX,), generator=g).to(DEV)]
    engines = (GraphInferenceEngine(M, DRAFT, device=DEV, batch_size=1),
               GraphInferenceEngineTG(M, TARGET, device=DEV, batch_size=1))
    times = {k: [] for k in SETTINGS}
    new = {k: [] for k in SETTINGS}
    per_rep = {k: [] for k in SETTINGS}
    for rep in range(args.reps):
        for name, kw in SETTINGS.items():
            t, n = step_times(engines, prompt, gm, [100 * rep], args.steps, kw)
            times[name] += t
            new[name] += n
            per_rep[name].append(1e3 * statistics.median(t))
    out["steps_B1"] = {name: dict(ms_per_step=1e3 * statistics.median(times[name]), ms_min=1e3 * min(times[name]),
                                  ms_max=1e3 * max(times[name]), rep_medians_ms=per_rep[name], steps=len(times[name]),
                                  tokens_per_step=statistics.mean(new[name]), tokens_per_step_min=min(new[name]),
                                  tokens_per_step_max=max(new[name]))
                       for name in SETTINGS}
    out["workload"] = (f"config 2, 128-node tree, B 1, T {T}, top_p 1, M {M}, {PREFIX}-token prompt, seeded; settings "
                       f"off / 128 random words of 2-16 ids and min_tokens 200; {args.reps} alternating reps of "
                       f"{args.steps} steps")
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
