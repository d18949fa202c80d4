"""Cost of the prompt logprobs: the kernel alone, and a BatchTree first verify with the setting off and on.

Kernel: device time per sq_prompt_logprobs_ragged call at V = 32000 and 128256, n = 0 and 20, over 128, 1024 and 8192
prompt rows in all (8 parts of equal size), from CUDA events around a CUDA graph of `--launches` calls.  Reported with
the bytes one pass over the rows reads (2 bytes per entry; the kernel makes three passes at n > 0 and two at n = 0, the
later ones mostly from L2) and the share of the H100 SXM's 3.35 TB/s HBM3 bandwidth that one pass in the measured time
would take.

First verify: config 2 (random-init llama-68m -> llama-2-7b, V = 32000, the 128-node growmap
A100-CNN-68m-7b-stochastic.pt, T 0.6, top_p 1, M 512, seeded) as a BatchTree at B = 1 and 4 with prompts of 100 and 300
tokens.  Every slot is admitted again before each timed step, alternating prompt_logprobs None and 20 `--reps` times in
the same tree (graphs captured in an untimed step first), and the step's verify() (the ragged first verify, the walk and
the host sync) is timed with a host clock after a device synchronize.  Reported: the median ms with its range.  The GPU
name and power limit are read in the same run.

    python tools/measure_prompt_logprobs.py [--out result.json] [--reps 10] [--launches 50]
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
M, T = 512, 0.6
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


def kernel_times(n_launch):
    from sequoia_b200 import ops
    B, Mx = 8, 1100
    out = []
    for V in (32000, 128256):
        for rows in (128, 1024, 8192):
            g = torch.Generator(device=DEV).manual_seed(V + rows)
            x = (torch.randn(rows, V, generator=g, device=DEV) * 2).to(torch.float16)
            tokens = torch.randint(0, V, (B, Mx), generator=g, device=DEV)
            plp_token = torch.empty(B, Mx, dtype=torch.float32, device=DEV)
            plp_ids = torch.empty(B, Mx, 20, dtype=torch.int32, device=DEV)
            plp_top = torch.empty(B, Mx, 20, dtype=torch.float32, device=DEV)
            per = rows // B
            for n in (0, 20):
                parts = [(b, b * per, per, n) for b in range(B)]
                us = per_launch(lambda: ops.prompt_logprobs_ragged_(x, parts, tokens, plp_token, plp_ids, plp_top),
                                n_launch)
                nbytes = rows * V * 2
                out.append(dict(V=V, rows=rows, n=n, us=us, bytes_per_pass=nbytes,
                                hbm_bound_share=nbytes / HBM_BYTES_PER_S / (us * 1e-6)))
                print(json.dumps(out[-1]), flush=True)
            del x
            torch.cuda.empty_cache()
    return out


def first_verify_times(engines, prompts, gm, reps):
    """-> {"off": [s, ...], "on": [s, ...]}: verify() of a first verify of every slot, alternating the setting"""
    from sequoia_b200.batch import BatchTree
    d, t = engines
    d.clear_kv()
    t.clear_kv()
    B = len(prompts)
    tree = BatchTree(d, t, prompts, gm, policy="spec", temperature=T, top_p=1.0, max_length=M, max_target_seq=M,
                     seeds=list(range(B)), prompt_logprobs=20)
    tree.construct_grow_map()
    tree.verify()                                               # captures the draft and post graphs
    times = {"off": [], "on": []}
    for rep in range(reps):
        for name, n in (("off", None), ("on", 20)):
            for b in range(B):
                tree.freeze(b)
                tree.admit(b, prompts[b], seed=1000 * rep + b, prompt_logprobs=n)
            tree.construct_grow_map()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tree.verify()                                       # ends in the step's one host sync
            times[name].append(time.perf_counter() - t0)
            if n is not None:
                assert tree.prompt_logprobs(0)[0].shape[0] == len(prompts[0]) - 1
    return times


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=50)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_prompt_logprobs needs a CUDA device")
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    out = dict(gpu_info())
    print(json.dumps(out), flush=True)
    out["kernels"] = kernel_times(args.launches)
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    g = torch.Generator().manual_seed(3)
    out["first_verify"] = {}
    for B in (1, 4):
        engines = (GraphInferenceEngine(M, DRAFT, device=DEV, batch_size=B),
                   GraphInferenceEngineTG(M, TARGET, device=DEV, batch_size=B))
        for P in (100, 300):
            prompts = [torch.randint(3, 32000, (P,), generator=g).to(DEV) for _ in range(B)]
            times = first_verify_times(engines, prompts, gm, args.reps)
            res = {k: dict(ms_median=1e3 * statistics.median(v), ms_min=1e3 * min(v), ms_max=1e3 * max(v), n=len(v))
                   for k, v in times.items()}
            out["first_verify"][f"B{B}_P{P}"] = res
            print(json.dumps({f"B{B}_P{P}": res}), flush=True)
        del engines
        torch.cuda.empty_cache()
    out["workload"] = (f"config 2, 128-node tree, T {T}, top_p 1, M {M}, seeded; first verify of every slot, prompt_logprobs "
                       f"None and 20 alternating, {args.reps} reps each")
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
