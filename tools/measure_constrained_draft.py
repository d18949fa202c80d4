"""Cost and effect of constrained drafting: the draft-row processing alone, and BatchTree decode steps with the draft
constrained and unconstrained.

Kernels: device time of one step's draft-row processing (sq_draft_rows_batch on the root and on each tree level whose
nodes have children, 1 + 8 = 9 calls on the config-2 growmap, 128 nodes) at V = 32000 and 128256 and B = 1, 4 and 8,
from CUDA events around a CUDA graph of `--launches` such steps, for two settings: a 1000-id allowed set with 16 bias
entries (SQ_DRAFT_BIAS), and a 16-state guide whose states each allow the same 1000 ids with the tokens drawn from them
(SQ_DRAFT_GUIDE), so every path stays alive and every transition searches 1000 edges.  The calls rewrite only -inf over
-inf, an unchanged bias sum aside, so repeating them in place is the same work each time (the bias is 0 here).

Steps: config 2 (random-init llama-68m -> llama-2-7b, V = 32000, the 128-node growmap A100-CNN-68m-7b-stochastic.pt,
T 0.6, top_p 1, M 384, seeded, stop mode without stop ids) as a BatchTree at B = 1 and B = 4, with seven settings
alternated `--reps` times in one process: no constraint; 1000 allowed ids with the draft unconstrained / constrained; an
8-state guide of 1000 ids per state unconstrained / constrained; an 8-state guide of 3 ids per state unconstrained /
constrained.  Each run builds the tree on 128-token prompts, runs 3 steps untimed (graph captures), then times `--steps`
steps (construct_grow_map + verify, which ends in the step's host sync) with a host clock.  Reported: the median ms per
step with its range, and the tokens committed per sequence per step.  The GPU name and power limit are read in the same
run.

    python tools/measure_constrained_draft.py [--out result.json] [--reps 3] [--steps 20] [--launches 50]
"""
import argparse
import gc
import json
import os
import random
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from measure_guide import DEV, DRAFT, GROWMAP, M, PREFIX, T, TARGET, WIDTH, gpu_info, per_launch, wide_guide  # noqa: E402


def narrow_guide(V, n_states, width, seed):
    """A guide whose states each allow `width` random ids, each moving to a random state."""
    from sequoia_b200.guide import GuideState, TokenGuide
    rnd = random.Random(seed)
    return TokenGuide([GuideState(edges={t: rnd.randrange(n_states) for t in rnd.sample(range(3, V), width)})
                       for _ in range(n_states)])


def kernel_times(gm, n_launch):
    from sequoia_b200 import ops
    from sequoia_b200.tree import _Static
    st = _Static(gm, DEV)
    S = gm["size"]
    levels = [(0, 1)] + [(lv["n0"], lv["tb"]) for i, lv in enumerate(st.levels) if i + 1 < len(st.levels)]
    out = []
    for V in (32000, 128256):
        guide, ids = wide_guide(V, 16, V, shared_ids=True)
        blob = guide.pack(V).to(DEV)
        for B in (1, 4, 8):
            g = torch.Generator().manual_seed(V + B)
            x = (torch.randn(B * S, V, generator=g) * 2).to(torch.float16).to(DEV)
            base, step = ops.draft_row_tables([(0, 1)] + [(lv["n0"], lv["tb"]) for lv in st.levels], S, B, DEV)
            tokens = torch.tensor(ids)[torch.randint(0, WIDTH, (B, M), generator=g)].to(DEV)
            state = torch.zeros(B, 16, dtype=torch.int32)
            state[:, 0], state[:, 8] = 200, M
            state[:, 12], state[:, 13], state[:, 14] = 1, 0, 200
            state = state.to(DEV)
            table = torch.full((B,), blob.data_ptr(), dtype=torch.int64, device=DEV)
            node = torch.zeros(B, S, dtype=torch.int32, device=DEV)
            mask = ops.pack_token_mask(ids, V).to(DEV).repeat(B, 1)
            bias_ids = torch.zeros(B, ops._lib.SQ_MAX_LOGIT_BIAS, dtype=torch.int32)
            bias_ids[:, :16] = torch.tensor(sorted(ids)[:16], dtype=torch.int32)
            bias = (mask, torch.ones(B, dtype=torch.int32, device=DEV), bias_ids.to(DEV),
                    torch.zeros(B, ops._lib.SQ_MAX_LOGIT_BIAS, dtype=torch.float32, device=DEV),
                    torch.full((B,), 16, dtype=torch.int32, device=DEV))
            common = dict(tokens=tokens, tree_bits=st.tree_bits, tree_words=st.tree_words)

            def allowed_step():
                for k0, nk in levels:
                    ops.draft_rows_batch_(x, base, step, k0, nk, S, state, bias=bias, **common)

            def guide_step():
                for k0, nk in levels:
                    ops.draft_rows_batch_(x, base, step, k0, nk, S, state, guide=(table, node), **common)
            us_allowed, us_guide = per_launch(allowed_step, n_launch), per_launch(guide_step, n_launch)
            assert int(node.min()) >= 0, "every path stays in the guide"
            out.append(dict(V=V, B=B, calls_per_step=len(levels), allowed_us_per_step=us_allowed,
                            guide_us_per_step=us_guide))
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
    assert tree._draft_processed() == bool(kw.get("constrain_draft")), kw.keys()
    assert "nan" not in tree.finish_reason
    return times, new


def steps_table(B, gm, reps, steps):
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    g = torch.Generator().manual_seed(3 + B)
    prompts = [torch.randint(3, 32000, (PREFIX,), generator=g).to(DEV) for _ in range(B)]
    engines = (GraphInferenceEngine(M, DRAFT, device=DEV, batch_size=B),
               GraphInferenceEngineTG(M, TARGET, device=DEV, batch_size=B))
    allowed = random.Random(7).sample(range(3, 32000), WIDTH)
    g1000, g3 = wide_guide(32000, 8, 5)[0], narrow_guide(32000, 8, 3, 9)
    settings = {"off": {}}
    for name, kw in (("allowed1000", dict(allowed_token_ids=allowed)), ("guide1000", dict(guide=g1000)),
                     ("guide3", dict(guide=g3))):
        settings[name] = kw
        settings[name + "_constrained"] = dict(kw, constrain_draft=True)
    times = {k: [] for k in settings}
    new = {k: [] for k in settings}
    per_rep = {k: [] for k in settings}
    for rep in range(reps):
        for name, kw in settings.items():
            t, n = step_times(engines, prompts, gm, [100 * rep + b for b in range(B)], steps, kw)
            times[name] += t
            new[name] += n
            per_rep[name].append(1e3 * statistics.median(t))
    del engines
    gc.collect()
    torch.cuda.empty_cache()
    return {name: dict(ms_per_step=1e3 * statistics.median(times[name]), ms_min=1e3 * min(times[name]),
                       ms_max=1e3 * max(times[name]), rep_medians_ms=per_rep[name], steps=len(times[name]),
                       tokens_per_seq_step=statistics.mean(new[name]), tokens_min=min(new[name]),
                       tokens_max=max(new[name]))
            for name in settings}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=50)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_constrained_draft needs a CUDA device")
    out = dict(gpu_info())
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    out["kernels"] = kernel_times(gm, args.launches)
    for B in (1, 4):
        out[f"steps_B{B}"] = steps_table(B, gm, args.reps, args.steps)
        print(json.dumps({f"steps_B{B}": out[f"steps_B{B}"]}), flush=True)
    out["workload"] = (f"config 2, 128-node tree, B 1 and 4, T {T}, top_p 1, M {M}, {PREFIX}-token prompts, seeded, "
                       f"stop mode without stop ids; no constraint / {WIDTH} allowed ids / an 8-state guide of {WIDTH} "
                       f"random ids per state / an 8-state guide of 3 ids per state, each with the draft unconstrained "
                       f"and constrained; {args.reps} alternating reps of {args.steps} steps")
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
