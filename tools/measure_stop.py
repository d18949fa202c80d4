"""Cost of stop mode (per-sequence stop ids and token budgets applied by the accept walks).

Kernels: device time per launch (CUDA events around a CUDA graph of 200 launches, each after the copies that restore the
walk's tokens, position ids and state; the copies' own time is subtracted) of the stop walks against the walks they
replace, on the 128-node growmap A100-CNN-68m-7b-stochastic.pt, at V = 32000 and 128256 and B = 1, 4 and 8:
sq_accept_stochastic_batch_stop (greedy NULL) against sq_accept_stochastic_batch_per_seq, and sq_accept_greedy_batch_stop
against sq_accept_greedy_batch.  Every sequence has 3 stop ids and a length limit, neither reached, so the cut scans
every committed token.

Steps: config 2 (random-init llama-68m -> llama-2-7b), B = 4, M 384, seeded, T 0.6, prompts of 128 tokens.  A tree in
default mode and one in stop mode (stop_tokens=[], which stops nothing, so both decode the same tokens unless an accepted
0 or 2 ends a default-mode sequence) alternate `--reps` times in one process; each times `--steps` steady steps
(construct_grow_map + verify, which ends in the step's host sync) after `--warmup` steps.  The GPU name and power limit
are read in the same run.

    python tools/measure_stop.py --out result.json [--reps 3] [--steps 40] [--warmup 5] [--skip-kernels] [--skip-steps]
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
M, T, PREFIX, B = 384, 0.6, 128, 4
DRAFT, TARGET = "random-init:llama-68m:1", "random-init:llama-2-7b:2"


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
        for Bk in (1, 4, 8):
            g = torch.Generator(device=DEV).manual_seed(V + Bk)
            draft = (torch.randn(Bk * S, V, generator=g, device=DEV) * 0.5).to(torch.float16)
            # target rows close to the draft rows (as tests/test_gpu_mixed_policy.py's walk inputs): several accepts
            logits = (draft.float() + 0.05 * torch.randn(Bk * S, V, generator=g, device=DEV)).to(torch.float16)
            target_token = ops.argmax_rows(logits)
            row_base, row_step = ops.draft_row_tables([(0, 1)] + [(lv["n0"], lv["tb"]) for lv in st.levels], S, Bk, DEV)
            tokens0 = torch.randint(3, V, (Bk, M), generator=g, device=DEV)
            tt = target_token.cpu()
            succ_off, succ = st.succ_off.cpu().tolist(), st.succ.cpu().tolist()
            for b in range(Bk):                               # the greedy walk accepts a path down to a leaf
                for k in range(S):
                    if succ_off[k] < succ_off[k + 1]:
                        tokens0[b, 100 - 1 + succ[succ_off[k]]] = int(tt[b * S + k])
            pos0 = torch.zeros(Bk, M, dtype=torch.int64, device=DEV)
            state0 = torch.zeros(Bk, 16, dtype=torch.int32, device=DEV)
            state0[:, 0], state0[:, 8] = 100, M
            tokens, pos, state = tokens0.clone(), pos0.clone(), state0.clone()
            acc = torch.zeros(Bk, S, dtype=torch.int32, device=DEV)
            r = torch.rand(Bk, M, generator=g, device=DEV).to(torch.float16)
            noise = torch.empty(Bk, V, device=DEV).exponential_(1.0, generator=g).to(torch.float16)
            Ts = torch.full((Bk,), T, dtype=torch.float32, device=DEV)
            stop_ids = torch.tensor([[1, 5, 7] + [-1] * 5] * Bk, dtype=torch.int32, device=DEV)
            end_limit = torch.full((Bk,), M, dtype=torch.int32, device=DEV)

            def reset():
                tokens.copy_(tokens0)
                pos.copy_(pos0)
                state.copy_(state0)
            sargs = (logits, draft, row_base, row_step, r, noise, st.succ_off, st.succ, st.depth, S, Ts)
            gargs = (target_token, st.succ_off, st.succ, st.depth, S)
            copies = per_launch(reset)
            res = dict(V=V, B=Bk, reset_copies_us=copies)
            res["stochastic_walk_us"] = per_launch(lambda: (reset(), ops.accept_stochastic_batch_per_seq(
                *sargs, tokens, pos, acc, state, M))) - copies
            res["stochastic_walk_stop_us"] = per_launch(lambda: (reset(), ops.accept_stochastic_batch_stop(
                *sargs, None, stop_ids, end_limit, tokens, pos, acc, state, M))) - copies
            res["greedy_walk_us"] = per_launch(lambda: (reset(), ops.accept_greedy_batch(
                *gargs, tokens, pos, acc, state, M))) - copies
            res["greedy_walk_stop_us"] = per_launch(lambda: (reset(), ops.accept_greedy_batch_stop(
                *gargs, None, stop_ids, end_limit, tokens, pos, acc, state, M))) - copies
            reset()
            ops.accept_stochastic_batch_stop(*sargs, None, stop_ids, end_limit, tokens, pos, acc, state, M)
            res["stochastic_new_tokens"] = (state[:, 3] + 1).tolist()
            reset()
            ops.accept_greedy_batch_stop(*gargs, None, stop_ids, end_limit, tokens, pos, acc, state, M)
            res["greedy_new_tokens"] = (state[:, 3] + 1).tolist()
            out.append(res)
            print(json.dumps(res), flush=True)
    return out


def steady_steps(draft, target, prompts, gm, stop_mode, steps, warmup):
    from sequoia_b200.batch import BatchTree
    kw = dict(stop_tokens=[]) if stop_mode else {}
    tree = BatchTree(draft, target, prompts, gm, temperature=T, top_p=1.0, max_length=M,
                     seeds=[900 + i for i in range(len(prompts))], **kw)
    times, tokens = [], 0
    for it in range(warmup + steps):
        t0 = time.perf_counter()
        tree.construct_grow_map()
        res = tree.verify()                                    # ends in the step's host sync
        if it >= warmup:
            times.append(1e3 * (time.perf_counter() - t0))
        if any(tree.frozen):
            break
    tokens = sum(len(v) - len(p) for (v, _, _), p in zip(res, prompts))
    return times, tokens


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--skip-kernels", action="store_true")
    ap.add_argument("--skip-steps", action="store_true")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_stop needs a CUDA device")
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    out = dict(gpu_info(), workload=f"config 2, B = {B}, prompts of {PREFIX} tokens, 128-node tree, T {T}, top_p 1, "
                                    f"M {M}, seeded")
    if not args.skip_kernels:
        out["kernels"] = kernel_times(gm)
    if not args.skip_steps:
        from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
        g = torch.Generator().manual_seed(3)
        prompts = [torch.randint(3, 32000, (PREFIX,), generator=g).to(DEV) for _ in range(B)]
        draft = GraphInferenceEngine(M, DRAFT, device=DEV, batch_size=B)
        target = GraphInferenceEngineTG(M, TARGET, device=DEV, batch_size=B)
        runs = {"default": [], "stop": []}
        for rep in range(args.reps):
            for name in ("default", "stop"):
                times, tokens = steady_steps(draft, target, prompts, gm, name == "stop", args.steps, args.warmup)
                runs[name].append(dict(median_ms=statistics.median(times), min_ms=min(times), max_ms=max(times),
                                       n=len(times), new_tokens=tokens))
                print(name, rep, json.dumps(runs[name][-1]), flush=True)
                draft.clear_kv()
                target.clear_kv()
        out["steps"] = runs
    out.update(gpu_info_after=gpu_info())
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
