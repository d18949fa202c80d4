"""Cost of batched verification: config-2 shapes (random-init llama-68m -> llama-2-7b, A100-CNN-68m-7b-stochastic.pt,
T 0.6, top_p 1, M 384, 128-token prompts) decoded B = 1, 2 and 4 prompts at a time with sequoia_b200.batch.BatchTree.

Per B: ms per step (CUDA events around construct_grow_map() + verify() of the timed steps, after warm-up steps that
capture the graphs), accepted tokens per step per sequence, and aggregate tokens/s.  At B = 1 the single-sequence
SpecTree runs on the same engines for comparison.  The GPU name and power limit are read in the same run.

    python tools/measure_batch.py --out result.json [--steps 20 --warmup 5 --batches 1,2,4]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
DEV = "cuda:0"
GROWMAP = "A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"
M, T, PREFIX = 384, 0.6, 128


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = [x.strip() for x in q.split(",")]
    return dict(gpu=name, power_limit=limit)


def _timed(step, n):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    tokens = 0
    for _ in range(n):
        tokens += step()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1), tokens


def measure_batch(B, prompts, gm, steps, warmup, with_single):
    from sequoia_b200.batch import BatchTree
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    draft = GraphInferenceEngine(M, "random-init:llama-68m:1", device=DEV, batch_size=B)
    target = GraphInferenceEngineTG(M, "random-init:llama-2-7b:2", device=DEV, batch_size=B)
    torch.manual_seed(0)
    tree = BatchTree(draft, target, prompts[:B], gm, policy="spec", temperature=T, top_p=1.0, max_length=M)
    length = [len(p) for p in prompts[:B]]

    def step():
        tree.construct_grow_map()
        new = 0
        for b, (valid, _, _) in enumerate(tree.verify()):
            new += valid.shape[0] - length[b]
            length[b] = valid.shape[0]
        return new

    _timed(step, warmup)                              # first verify (eager prefill) + graph captures
    assert not any(tree.frozen), "a sequence finished during warm-up; use fewer steps"
    ms, tokens = _timed(step, steps)
    assert not any(tree.frozen), "a sequence finished inside the timed window; use fewer steps"
    res = dict(B=B, ms_per_step=ms / steps, tokens_per_step_per_sequence=tokens / (steps * B),
               aggregate_tokens_per_s=tokens / (ms / 1e3),
               launches_per_step=tree.graph_launches["draft"] + tree.graph_launches["steady"])
    if with_single:
        from sequoia_b200.tree import SpecTree
        torch.manual_seed(0)
        st = SpecTree(draft, target, prompts[0].to(DEV), temperature=T, top_p=1.0, max_length=M, max_target_seq=M,
                      device=DEV, vocab_size=32000, grow_map=gm)
        n = [len(prompts[0])]

        def step1():
            st.construct_grow_map()
            valid, _, _, _ = st.verify()
            new = valid.shape[0] - n[0]
            n[0] = valid.shape[0]
            return new

        _timed(step1, warmup)
        ms1, tok1 = _timed(step1, steps)
        res["spectree"] = dict(ms_per_step=ms1 / steps, tokens_per_step=tok1 / steps, tokens_per_s=tok1 / (ms1 / 1e3))
    del tree, draft, target
    torch.cuda.empty_cache()
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batches", default="1,2,4")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_batch needs a CUDA device")
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    g = torch.Generator().manual_seed(3)
    batches = [int(x) for x in args.batches.split(",")]
    prompts = [torch.randint(3, 32000, (PREFIX,), generator=g) for _ in range(max(batches))]
    out = dict(gpu_info(), workload="c2: llama-68m -> llama-2-7b (random init), 128-node tree, T 0.6, M 384",
               steps=args.steps, warmup=args.warmup, runs=[])
    for B in batches:
        r = measure_batch(B, prompts, gm, args.steps, args.warmup, with_single=(B == 1))
        out["runs"].append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps(out))
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
