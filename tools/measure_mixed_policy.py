"""Greedy and sampled sequences in one BatchTree (per-sequence policy) against the two single-policy batches.

Config 2 (random-init llama-68m -> llama-2-7b, V = 32000), B = 4, M 384, the 128-node growmap
A100-CNN-68m-7b-stochastic.pt, T 0.6, top_p 1.  On the same engines and prompts, three runs alternate `--reps` times in one
process:

* spec:   BatchTree(policy="spec");
* greedy: BatchTree(policy="greedy");
* mixed:  policies alternating spec, greedy by prompt (2 + 2 in the batch).

Each run is a refill decode (testbed.decode_refill) of a queue of 16 prompts of 128 tokens, budgets drawn from 32..128; in
the mixed run prompt i has policy ("spec", "greedy")[i % 2], and each admitted prompt brings its own.  Reported per run:
median ms per steady step and per admission step (decode_refill's step timer), refill tokens/s (construction included)
and accepted tokens per target step per sequence.

Kernels (first, unless --skip-kernels): device time per launch (CUDA events around a CUDA graph of 200 launches) of
argmax_rows on B*S target rows (S = 128), of the mixed greedy walk and of the mixed stochastic walk (half of the batch
greedy), at B = 4 and 8 and V = 32000 and 128256.  The GPU name and power limit are read in the same run.

    python tools/measure_mixed_policy.py --out result.json [--reps 3] [--skip-kernels] [--skip-decode]
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
M, T, PREFIX, N_PROMPTS, BUDGET, B = 384, 0.6, 128, 16, (32, 128), 4
DRAFT, TARGET = "random-init:llama-68m:1", "random-init:llama-2-7b:2"
RUNS = {"spec": "spec", "greedy": "greedy", "mixed": None}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = [x.strip() for x in q.split(",")]
    return dict(gpu=name, power_limit=limit)


def kernel_times(gm):
    from sequoia_b200 import ops
    from sequoia_b200.tree import _Static
    st = _Static(gm, DEV)
    S = st.S
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def per_launch(fn, n=200):
        """device time per launch: n launches captured in one CUDA graph, so the host's enqueue cost is not timed"""
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

    out = []
    for V in (32000, 128256):
        for Bk in (4, 8):
            g = torch.Generator(device=DEV).manual_seed(V + Bk)
            logits = (torch.randn(Bk * S, V, generator=g, device=DEV) * 2).to(torch.float16)
            draft = logits.clone()
            target_token = torch.empty(Bk * S, dtype=torch.int64, device=DEV)
            row_base, row_step = ops.draft_row_tables([(0, 1)] + [(lv["n0"], lv["tb"]) for lv in st.levels], S, Bk, DEV)
            tokens0 = torch.randint(3, V, (Bk, M), generator=g, device=DEV)
            pos0 = torch.zeros(Bk, M, dtype=torch.int64, device=DEV)
            state0 = torch.zeros(Bk, 16, dtype=torch.int32, device=DEV)
            state0[:, 0], state0[:, 8] = 100, M
            tokens, pos, state = tokens0.clone(), pos0.clone(), state0.clone()
            acc = torch.zeros(Bk, S, dtype=torch.int32, device=DEV)
            r = torch.rand(Bk, M, generator=g, device=DEV).to(torch.float16)
            noise = torch.ones(Bk, V, dtype=torch.float16, device=DEV)
            Ts = torch.full((Bk,), T, dtype=torch.float32, device=DEV)
            greedy = torch.tensor([b % 2 for b in range(Bk)], dtype=torch.int32, device=DEV)

            def reset():
                # every walk restarts from the same tokens and state (a walk moves P on): the copies are timed with it
                tokens.copy_(tokens0)
                pos.copy_(pos0)
                state.copy_(state0)

            copies = per_launch(reset)
            argmax = per_launch(lambda: ops.argmax_rows(logits, target_token))
            gwalk = per_launch(lambda: (reset(), ops.accept_greedy_batch_mixed(
                target_token, st.succ_off, st.succ, st.depth, S, greedy, tokens, pos, acc, state, M)))
            swalk = per_launch(lambda: (reset(), ops.accept_stochastic_batch_mixed(
                logits, draft, row_base, row_step, r, noise, st.succ_off, st.succ, st.depth, S, Ts, greedy, tokens, pos,
                acc, state, M)))
            out.append(dict(V=V, B=Bk, rows=Bk * S, argmax_rows_us=argmax, reset_copies_us=copies,
                            greedy_walk_mixed_us=gwalk - copies, stochastic_walk_mixed_us=swalk - copies))
            print(json.dumps(out[-1]), flush=True)
    return out


def run(draft, target, prompts, limits, gm, kind):
    """One refill decode of the whole queue -> (total s, decoded tokens, target steps, step times)"""
    import testbed
    from sequoia_b200.batch import BatchTree
    policies = [("spec", "greedy")[i % 2] for i in range(len(prompts))] if kind == "mixed" else None
    times = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tree = BatchTree(draft, target, prompts[:B], gm, policy=RUNS[kind] or policies[:B], temperature=T, top_p=1.0,
                     max_length=M)
    _, decoded, steps, _ = testbed.decode_refill(tree, prompts, limits, step_times=times, policies=policies)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, decoded, steps, times


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-kernels", action="store_true")
    ap.add_argument("--skip-decode", action="store_true")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_mixed_policy needs a CUDA device")
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    rng = random.Random(11)
    budgets = [rng.randint(*BUDGET) for _ in range(N_PROMPTS)]
    limits = [PREFIX + n for n in budgets]
    out = dict(gpu_info(), workload=f"config 2, B = {B}, {N_PROMPTS} prompts of {PREFIX} tokens, 128-node tree, T {T}, "
                                    f"top_p 1, M {M}", budgets=budgets)
    if not args.skip_kernels:
        out["kernels"] = kernel_times(gm)
    if not args.skip_decode:
        g = torch.Generator().manual_seed(3)
        prompts = [torch.randint(3, 32000, (PREFIX,), generator=g).to(DEV) for _ in range(N_PROMPTS)]
        draft = GraphInferenceEngine(M, DRAFT, device=DEV, batch_size=B)
        target = GraphInferenceEngineTG(M, TARGET, device=DEV, batch_size=B)
        for kind in RUNS:                                   # warm-up: modules, allocator, algorithms
            torch.manual_seed(100)
            run(draft, target, prompts[:B + 2], limits[:B + 2], gm, kind)
        res = {kind: dict(tokens_per_s=[], tokens_per_step=[], steady=[], admission=[]) for kind in RUNS}
        for k in range(args.reps):
            for kind in RUNS:
                torch.manual_seed(k)
                total, decoded, steps, times = run(draft, target, prompts, limits, gm, kind)
                r = res[kind]
                r["tokens_per_s"].append(decoded / total)
                r["tokens_per_step"].append(decoded / max(steps, 1))
                r["steady"] += [t for kd, t in times if kd == "steady"]
                r["admission"] += [t for kd, t in times if kd == "admission"]
        for kind in RUNS:
            r = res[kind]
            steady, admission = r.pop("steady"), r.pop("admission")
            r["ms_per_steady_step"] = 1e3 * statistics.median(steady)
            r["ms_per_admission_step"] = 1e3 * statistics.median(admission)
            r["steady_steps"], r["admission_steps"] = len(steady), len(admission)
        out["runs"] = res
        print(json.dumps(res), flush=True)
    print(json.dumps(out))
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
