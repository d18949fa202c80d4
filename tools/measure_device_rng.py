"""Seeded BatchTree (random numbers drawn on the device, per-sequence Philox streams) against the CPU draws it replaces.

Per model pair and B (4 and 8), on the same engines, prompts and new-token budgets, the two modes alternate `--reps` times
in one process:

* cpu:    BatchTree(seeds=None): r and rand drawn with torch's CPU generator per prompt (at construction and at every
          admit), the bonus noise with torch's exponential_;
* device: BatchTree(seeds=...): r and rand filled on the device from each prompt's seed, the noise by the noise kernel.

Reported per mode: BatchTree construction time (host clock, ending in a device synchronise), ms per admission step and
per steady step of a refill decode (testbed.decode_refill's step timer, as tools/measure_refill.py), refill tokens/s
(construction included) and accepted tokens per target step per sequence.  Repetition k draws other numbers in both
modes (torch.manual_seed(k) for cpu, seeds (k + 11) << 32 | prompt index for device), so the spread of the accepted tokens
per step between repetitions is the spread between streams, against which the two modes are compared.  Pairs: config 2
(random-init llama-68m -> llama-2-7b) and Llama 3 (random-init llama-3.2-1b -> llama-3.1-8b, V = 128256), both on
A100-CNN-68m-7b-stochastic.pt, T 0.6, top_p 1, M 384, prompts of 128 tokens with budgets drawn from 32..128.

Kernels (first, unless --skip-kernels): device time per launch (CUDA events around a CUDA graph of 200 launches) of the
bonus noise of B sequences, sq_rng_exponential_batch against torch's exponential_ on the same (B, V) buffer, and of one
slot's rand fill (S = 128), sq_rng_uniform_seqs against the CPU draw + pinned copy it replaces (host clock, ending in a
device synchronise), at V = 32000 and 128256.  The GPU name and power limit are read in the same run.

    python tools/measure_device_rng.py --out result.json [--reps 3 --batches 4,8 --pairs c2,llama3] [--skip-decode]
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
M, T, PREFIX, N_PROMPTS, BUDGET = 384, 0.6, 128, 12, (32, 128)
PAIRS = {"c2": ("random-init:llama-68m:1", "random-init:llama-2-7b:2", 32000),
         "llama3": ("random-init:llama-3.2-1b:1", "random-init:llama-3.1-8b:2", 128256)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = [x.strip() for x in q.split(",")]
    return dict(gpu=name, power_limit=limit)


def kernel_times(batches):
    from sequoia_b200 import ops
    from sequoia_b200.batch import draw_random
    out = []
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

    for V in (32000, 128256):
        for B in batches:
            noise = torch.empty(B, V, dtype=torch.float16, device=DEV)
            seeds = torch.arange(B, dtype=torch.int64, device=DEV)
            steps = torch.zeros(B, dtype=torch.int64, device=DEV)
            state = torch.zeros(B, 16, dtype=torch.int32, device=DEV)
            kern = per_launch(lambda: ops.rng_exponential_batch(noise, seeds, steps, state))
            ref = per_launch(lambda: noise.exponential_(1.0))
            out.append(dict(V=V, B=B, noise_kernel_us=kern, torch_exponential_us=ref))
            print(json.dumps(out[-1]), flush=True)
        rand = torch.empty(1, 128, V, dtype=torch.float16, device=DEV)
        seeds = torch.zeros(1, dtype=torch.int64, device=DEV)
        fill = per_launch(lambda: ops.rng_uniform_seqs(rand, seeds, [0], ops.RNG_RAND), 50)
        cpu = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, r = draw_random([None], M, 128, V)
            rand[0].copy_(r[0].pin_memory(), non_blocking=True)
            torch.cuda.synchronize()
            cpu.append(1e3 * (time.perf_counter() - t0))
        out.append(dict(V=V, S=128, rand_fill_kernel_us=fill, rand_cpu_draw_and_copy_ms=statistics.median(cpu)))
        print(json.dumps(out[-1]), flush=True)
    return out


def run(draft, target, prompts, limits, gm, B, seeds):
    """One refill decode of the whole queue -> (construction s, total s, decoded tokens, target steps, step times)"""
    import testbed
    from sequoia_b200.batch import BatchTree
    times = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tree = BatchTree(draft, target, prompts[:B], gm, policy="spec", temperature=T, top_p=1.0, max_length=M,
                     seeds=None if seeds is None else seeds[:B])
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    _, decoded, steps, _ = testbed.decode_refill(tree, prompts, limits, step_times=times, seeds=seeds)
    torch.cuda.synchronize()
    return t1 - t0, time.perf_counter() - t0, decoded, steps, times


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batches", default="4,8")
    ap.add_argument("--pairs", default="c2,llama3")
    ap.add_argument("--skip-kernels", action="store_true")
    ap.add_argument("--skip-decode", action="store_true")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_device_rng needs a CUDA device")
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    rng = random.Random(11)
    budgets = [rng.randint(*BUDGET) for _ in range(N_PROMPTS)]
    limits = [PREFIX + n for n in budgets]

    def seeds(k):
        return [((k + 11) << 32) | i for i in range(N_PROMPTS)]

    out = dict(gpu_info(), workload=f"{N_PROMPTS} prompts of {PREFIX} tokens, 128-node tree, T 0.6, top_p 1, M {M}",
               budgets=budgets, runs=[])
    batches = [int(x) for x in args.batches.split(",")]
    if not args.skip_kernels:
        out["kernels"] = kernel_times(batches)
    for pair in ([] if args.skip_decode else args.pairs.split(",")):
        dname, tname, V = PAIRS[pair]
        g = torch.Generator().manual_seed(3)
        prompts = [torch.randint(3, V, (PREFIX,), generator=g).to(DEV) for _ in range(N_PROMPTS)]
        for B in batches:
            draft = GraphInferenceEngine(M, dname, device=DEV, batch_size=B)
            target = GraphInferenceEngineTG(M, tname, device=DEV, batch_size=B)
            for sd in (None, seeds(100)):                     # warm-up: modules, allocator, algorithms
                torch.manual_seed(100)
                run(draft, target, prompts[:B], limits[:B], gm, B, None if sd is None else sd[:B])
            res = dict(pair=pair, draft=dname, target=tname, V=V, B=B)
            for mode in ("cpu", "device"):
                res[mode] = dict(construction_ms=[], tokens_per_s=[], tokens_per_step=[], steady=[], admission=[])
            for k in range(args.reps):
                for mode, sd in (("cpu", None), ("device", seeds(k))):
                    torch.manual_seed(k)
                    cons, total, decoded, steps, times = run(draft, target, prompts, limits, gm, B, sd)
                    r = res[mode]
                    r["construction_ms"].append(1e3 * cons)
                    r["tokens_per_s"].append(decoded / total)
                    r["tokens_per_step"].append(decoded / max(steps, 1))
                    r["steady"] += [t for kind, t in times if kind == "steady"]
                    r["admission"] += [t for kind, t in times if kind == "admission"]
            for mode in ("cpu", "device"):
                r = res[mode]
                steady, admission = r.pop("steady"), r.pop("admission")
                r["ms_per_steady_step"] = 1e3 * statistics.median(steady)
                r["ms_per_admission_step"] = 1e3 * statistics.median(admission)
                r["steady_steps"], r["admission_steps"] = len(steady), len(admission)
            out["runs"].append(res)
            print(json.dumps(res), flush=True)
            del draft, target
            torch.cuda.empty_cache()
    print(json.dumps(out))
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
