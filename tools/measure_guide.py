"""Cost of guided decoding: the three guide kernels alone, and a BatchTree decode step with and without a guide.

Kernels: device time per call of sq_guide_states_batch, sq_guide_mask_rows_batch and sq_guide_advance_batch on the
config-2 growmap (128 nodes) at V = 32000 and 128256 and B = 1, 4 and 8, from CUDA events around a CUDA graph of
`--launches` calls.  Every sequence has a 16-state guide whose states each allow the same 1000 ids (each id moving to a
random state) and its tokens are drawn from those ids, so every node of every path is alive: each of the 127 node
transitions and the max_depth + 1 = 11 committed transitions searches 1000 edges, and each row keeps 1000 ids.  The
states and mask calls do not change their inputs, so repeating them in place is the same work each time.  The advance
call moves the state words, so its graph restores them before each call; the restore's own time, measured the same way,
is subtracted.

Steps: config 2 (random-init llama-68m -> llama-2-7b, V = 32000, the 128-node growmap A100-CNN-68m-7b-stochastic.pt,
T 0.6, top_p 1, M 384, seeded, stop mode without stop ids) as a BatchTree at B = 1, with two settings alternated
`--reps` times in one process: no guide, and an 8-state guide whose states allow 1000 random ids each.  Each run builds
the tree on a 128-token prompt, runs 3 steps untimed (graph captures), then times `--steps` steps (construct_grow_map +
verify, which ends in the step's host sync) with a host clock.  Reported: the median ms per step with its range, and the
tokens committed per step.  The GPU name and power limit are read in the same run.

    python tools/measure_guide.py [--out result.json] [--reps 3] [--steps 20] [--launches 200]
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
M, T, PREFIX = 384, 0.6, 128
DRAFT, TARGET = "random-init:llama-68m:1", "random-init:llama-2-7b:2"
WIDTH = 1000


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


def wide_guide(V, n_states, seed, shared_ids=False):
    from sequoia_b200.guide import GuideState, TokenGuide
    rnd = random.Random(seed)
    ids = rnd.sample(range(3, V), WIDTH)
    states = []
    for _ in range(n_states):
        own = ids if shared_ids else rnd.sample(range(3, V), WIDTH)
        states.append(GuideState(edges={t: rnd.randrange(n_states) for t in own}))
    return TokenGuide(states), ids


def kernel_times(gm, n_launch):
    from sequoia_b200 import ops
    from sequoia_b200.tree import _Static
    st = _Static(gm, DEV)
    S, md = gm["size"], int(gm["depth"].max())
    out = []
    for V in (32000, 128256):
        guide, ids = wide_guide(V, 16, V, shared_ids=True)
        blob = guide.pack(V).to(DEV)
        for B in (1, 4, 8):
            g = torch.Generator().manual_seed(V + B)
            x = (torch.randn(B * S, V, generator=g) * 2).to(torch.float16).to(DEV)
            pool = torch.tensor(ids)
            tokens = pool[torch.randint(0, WIDTH, (B, M), generator=g)].to(DEV)
            P = 200
            state0 = torch.zeros(B, 16, dtype=torch.int32)
            state0[:, 0], state0[:, 1], state0[:, 8] = P, P + md, M         # a step that committed max_depth + 1
            state0[:, 12], state0[:, 13], state0[:, 14] = 1, 0, P
            state0 = state0.to(DEV)
            state = state0.clone()
            table = torch.full((B,), blob.data_ptr(), dtype=torch.int64, device=DEV)
            node = torch.zeros(B, S, dtype=torch.int32, device=DEV)

            def states():
                ops.guide_states_batch(table, tokens, state0, st.depth, st.tree_bits, st.tree_words, S, V, node)

            def mask():
                ops.guide_mask_rows_batch_(x, S, state0, table, node)

            def restore():
                state.copy_(state0)

            def advance():
                state.copy_(state0)
                ops.guide_advance_batch(table, tokens, state, V)
            us_states, us_mask = per_launch(states, n_launch), per_launch(mask, n_launch)
            us_adv = per_launch(advance, n_launch) - per_launch(restore, n_launch)
            assert int(node.min()) >= 0 and int(state[:, 13].min()) >= 0, "every path stays in the guide"
            out.append(dict(V=V, B=B, states_us=us_states, mask_us=us_mask, advance_us=us_adv,
                            total_us=us_states + us_mask + us_adv))
            print(json.dumps(out[-1]), flush=True)
    return out


def step_times(engines, prompts, gm, seeds, steps, kw):
    from sequoia_b200.batch import BatchTree
    d, t = engines
    d.clear_kv()
    t.clear_kv()
    tree = BatchTree(d, t, prompts, gm, policy="spec", temperature=T, top_p=1.0, max_length=M, seeds=seeds,
                     stop_tokens=[], **kw)
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
    assert tree.use_guide == bool(kw)
    return times, new


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_guide needs a CUDA device")
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    out = dict(gpu_info())
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    out["kernels"] = kernel_times(gm, args.launches)
    g = torch.Generator().manual_seed(3)
    prompt = [torch.randint(3, 32000, (PREFIX,), generator=g).to(DEV)]
    engines = (GraphInferenceEngine(M, DRAFT, device=DEV, batch_size=1),
               GraphInferenceEngineTG(M, TARGET, device=DEV, batch_size=1))
    settings = {"off": {}, "guide1000": dict(guide=wide_guide(32000, 8, 5)[0])}
    times = {k: [] for k in settings}
    new = {k: [] for k in settings}
    per_rep = {k: [] for k in settings}
    for rep in range(args.reps):
        for name, kw in settings.items():
            t, n = step_times(engines, prompt, gm, [100 * rep], args.steps, kw)
            times[name] += t
            new[name] += n
            per_rep[name].append(1e3 * statistics.median(t))
    out["steps_B1"] = {name: dict(ms_per_step=1e3 * statistics.median(times[name]), ms_min=1e3 * min(times[name]),
                                  ms_max=1e3 * max(times[name]), rep_medians_ms=per_rep[name], steps=len(times[name]),
                                  tokens_per_step=statistics.mean(new[name]), tokens_per_step_min=min(new[name]),
                                  tokens_per_step_max=max(new[name]))
                       for name in settings}
    out["workload"] = (f"config 2, 128-node tree, B 1, T {T}, top_p 1, M {M}, {PREFIX}-token prompt, seeded, stop mode "
                       f"without stop ids; no guide / an 8-state guide of {WIDTH} random ids per state; {args.reps} "
                       f"alternating reps of {args.steps} steps")
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
