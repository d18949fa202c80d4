"""Cost and gain of prefix reuse (BatchTree.admit(reuse_prefix=True)): the copy kernel alone, an admission step, and a
refill queue, with and without reuse.

Kernel: device time per sq_kv_copy_prefix call (K and V of every layer, one launch) at the 68m draft, 7B and Llama-3.1-8B
cache shapes with M = 2048, B = 8, for n = 1 .. 2047 rows, from CUDA events around a CUDA graph of `--launches` calls;
the same copy done with torch's strided copy_ of the same K and V slices, timed the same way, is the baseline.  Bytes
are 2 (K, V) x 2 (read + write) x L x Hkv x n x D x 2, reported against the H100 SXM's 3.35 TB/s HBM3 data-sheet
bandwidth.

Admission step: config 2 (random-init llama-68m -> llama-2-7b, V = 32000, the 128-node growmap, T 0.6, top_p 1, M 2048,
seeded) at B = 4 and 8.  Every slot holds a prompt made of a shared prefix of 0 / 512 / 1024 / 1536 tokens plus 64
distinct tokens.  Before each timed admission the last slot gets an unrelated prompt and one untimed step, so the timed
admission of another shared-prefix prompt into it copies the prefix from a neighbour.  The step is timed with a host
clock from the admit() call to the end of its verify() (which ends in the step's host sync), alternating reuse off and on
`--reps` times in one tree.  One Llama-3.2-1B -> Llama-3.1-8B line (V = 128256) at B = 4 and a 1024-token prefix.

Refill: the same config-2 trees decode one queue of 3B such prompts, each to 64 new tokens, through testbed.decode_refill
(each finished slot takes the next prompt), twice without and twice with reuse, alternating; reported as committed tokens
per second over the whole queue.  The GPU name and power limit are read in the same run.

    python tools/measure_prefix_reuse.py [--out result.json] [--reps 5] [--launches 20]
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
M, T = 2048, 0.6
CONFIG2 = ("random-init:llama-68m:1", "random-init:llama-2-7b:2", 32000)
LLAMA3 = ("random-init:llama-3.2-1b:1", "random-init:llama-3.1-8b:2", 128256)
HBM_BYTES_PER_S = 3.35e12                                      # H100 SXM data sheet
PREFIXES = (0, 512, 1024, 1536)
DISTINCT = 64


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


class _KV:
    def __init__(self, k, v):
        self.k_cache, self.v_cache = k, v


def kernel_times(n_launch):
    from sequoia_b200 import ops
    B, src, dst = 8, 5, 2
    out = []
    for name, (L, Hkv, D) in (("68m", (2, 12, 64)), ("7b", (32, 32, 128)), ("llama3_8b", (32, 8, 128))):
        kv = _KV(torch.randn(L, B, Hkv, M, D, device=DEV).half(), torch.randn(L, B, Hkv, M, D, device=DEV).half())
        for n in (1, 64, 512, 1024, 1536, 2047):
            def torch_copy():
                kv.k_cache[:, dst, :, :n].copy_(kv.k_cache[:, src, :, :n])
                kv.v_cache[:, dst, :, :n].copy_(kv.v_cache[:, src, :, :n])
            us = per_launch(lambda: ops.kv_copy_prefix(kv, src, dst, n), n_launch)
            us_torch = per_launch(torch_copy, n_launch)
            nbytes = 2 * 2 * L * Hkv * n * D * 2
            out.append(dict(cache=name, n=n, us=us, GBps=nbytes / us * 1e-3, hbm_share=nbytes / HBM_BYTES_PER_S / (us * 1e-6),
                            torch_us=us_torch, torch_GBps=nbytes / us_torch * 1e-3, bytes=nbytes))
            print(json.dumps(out[-1]), flush=True)
        del kv
        torch.cuda.empty_cache()
    return out


def _engines(cfg, B):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    return (GraphInferenceEngine(M, cfg[0], device=DEV, batch_size=B),
            GraphInferenceEngineTG(M, cfg[1], device=DEV, batch_size=B))


def _prompts(g, V, prefix, k):
    shared = torch.randint(3, V, (prefix,), generator=g)
    return [torch.cat([shared, torch.randint(3, V, (DISTINCT,), generator=g)]).to(DEV) for _ in range(k)]


def admission_times(engines, V, B, prefix, reps, gm, g):
    """-> {"off": [s, ...], "on": [s, ...]}, reused L per admission with reuse on"""
    from sequoia_b200.batch import BatchTree
    d, t = engines
    d.clear_kv()
    t.clear_kv()
    prompts = _prompts(g, V, prefix, B + 2 * reps)
    tree = BatchTree(d, t, prompts[:B], gm, policy="spec", temperature=T, top_p=1.0, max_length=M, max_target_seq=M,
                     seeds=list(range(B)))
    tree.construct_grow_map()
    tree.verify()
    times, reused, b, nxt = {"off": [], "on": []}, [], B - 1, B
    for rep in range(reps):
        for name in ("off", "on"):
            tree.freeze(b)                                      # an unrelated prompt first: the timed one copies
            tree.admit(b, torch.randint(3, V, (prefix + DISTINCT,), generator=g).to(DEV), seed=7 + rep)
            tree.construct_grow_map()
            tree.verify()
            tree.freeze(b)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tree.admit(b, prompts[nxt], seed=1000 + nxt, reuse_prefix=name == "on")
            tree.construct_grow_map()
            tree.verify()
            times[name].append(time.perf_counter() - t0)
            if name == "on":
                reused.append(0 if tree.reused_prefix[b] is None else tree.reused_prefix[b][1])
            nxt += 1
    return times, reused


def refill_rate(engines, prompts, gm, reuse):
    import testbed
    from sequoia_b200.batch import BatchTree
    d, t = engines
    d.clear_kv()
    t.clear_kv()
    B = d.engine.batch_size
    limits = [len(p) + 64 for p in prompts]
    tree = BatchTree(d, t, prompts[:B], gm, policy="spec", temperature=T, top_p=1.0, max_length=M, max_target_seq=M,
                     seeds=list(range(3 * B))[:B])
    reused = [] if reuse else None
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _, decoded, _, _ = testbed.decode_refill(tree, prompts, limits, stop=frozenset(), seeds=list(range(3 * B)),
                                             reused=reused)
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    return dict(tokens_per_s=decoded / sec, decoded=decoded, seconds=sec, reused_tokens=sum(reused or []))


def _stats(v):
    return dict(ms_median=1e3 * statistics.median(v), ms_min=1e3 * min(v), ms_max=1e3 * max(v), n=len(v))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_prefix_reuse needs a CUDA device")
    out = dict(gpu_info())
    print(json.dumps(out), flush=True)
    out["kernel"] = kernel_times(args.launches)
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    g = torch.Generator().manual_seed(3)
    out["admission"], out["refill"] = {}, {}
    for cfg, Bs, prefixes in ((CONFIG2, (4, 8), PREFIXES), (LLAMA3, (4,), (1024,))):
        V = cfg[2]
        for B in Bs:
            engines = _engines(cfg, B)
            for prefix in prefixes:
                key = f"V{V}_B{B}_prefix{prefix}"
                times, reused = admission_times(engines, V, B, prefix, args.reps, gm, g)
                out["admission"][key] = dict(off=_stats(times["off"]), on=_stats(times["on"]), reused_L=reused)
                print(json.dumps({key: out["admission"][key]}), flush=True)
                if V == 32000:
                    runs, queue = {}, _prompts(g, V, prefix, 3 * B)
                    for reuse in (False, True, False, True):
                        runs.setdefault("on" if reuse else "off", []).append(refill_rate(engines, queue, gm, reuse))
                    out["refill"][key] = runs
                    print(json.dumps({key: runs}), flush=True)
            del engines
            torch.cuda.empty_cache()
    out["workload"] = (f"M {M}, 128-node tree, T {T}, top_p 1, seeded; prompts = shared prefix + {DISTINCT} distinct "
                       f"tokens; admission timed from admit() to the end of verify(), off / on alternating {args.reps} "
                       "times; refill: 3B prompts to 64 new tokens each")
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
