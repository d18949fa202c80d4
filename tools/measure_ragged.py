"""Ragged batched forward against the per-sequence path on the config-2 shapes (random-init llama-68m -> llama-2-7b,
A100-CNN-68m-7b-stochastic.pt (128 nodes), T 0.6, top_p 1, M 384).

Two BatchTree variants on the same engines:

* ragged: BatchTree as it is -- the draft prefill and the target first verify of the sequences that need them run as one
  LlamaRunner.forward_ragged each, at sum(P_b) and sum(P_b + S - 1) rows;
* per-sequence: the same steps restated here as one forward(batch=True) per sequence, every other sequence given a frozen
  copy of its state row, so each runs B*P (draft) and B*(P + S - 1) (target) rows.

Per B (4 and 8), alternating the two variants `--reps` times in one process (host clock around work that ends in a
device synchronise):

* construction: BatchTree construction through the first construct_grow_map + verify, with B prompts of 128 tokens and
  with B prompts of mixed lengths drawn from 20..250;
* admission: one step that admits a 128-token prompt into a frozen slot (admit + construct_grow_map + verify), after two
  steady steps.

The first-verify target logits of the two variants are compared on the same inputs (same drafted tree, same KV state):
the max abs difference per sequence.  The GPU name and power limit are read in the same run.

    python tools/measure_ragged.py --out result.json [--reps 3 --batches 4,8]
"""
import argparse
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
DEV = "cuda:0"
GROWMAP = "A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"
M, T, PREFIX, MIXED = 384, 0.6, 128, (20, 250)
ST_FROZEN = 9


def _alone(bt, b, fn):
    """Run fn for sequence b only: every other sequence gets a frozen copy of b's state row (writes nothing of its own,
    reads the cache range b reads); the state rows are restored afterwards."""
    saved = bt.state.clone()
    tmp = saved[b:b + 1].repeat(bt.B, 1)
    tmp[:, ST_FROZEN] = 1
    tmp[b] = saved[b]
    bt.state.copy_(tmp)
    fn()
    bt.state.copy_(saved)


def per_sequence_class():
    from sequoia_b200.batch import BatchTree

    class PerSequence(BatchTree):
        """BatchTree with the draft prefill and first verify as one forward(batch=True) per sequence"""

        def op_draft_prefill(self, seqs):
            for b in seqs:
                P = self.ground_truth_len[b]
                _alone(self, b, lambda: self.draft.engine.runner.forward(
                    P, self.tokens, self.position_ids, self.storage_ids, state=self.state, n0=1 - P, kv_end=1,
                    batch=True, logits_from=b * P + P - 1, logits_to=b * P + P, logits_out=self.draft_logits[b:b + 1],
                    **self._mask_kw()))

        def op_target_first(self, seqs):
            S = self.S
            for b in seqs:
                P = self.ground_truth_len[b]
                n = P + S - 1
                _alone(self, b, lambda: self.target.engine.runner.forward(
                    n, self.tokens, self.position_ids, self.storage_ids, state=self.state, n0=1 - P, kv_end=S,
                    batch=True, logits_from=b * n + n - S, logits_to=b * n + n,
                    logits_out=self.target_logits[b * S:(b + 1) * S], **self._mask_kw()))

    return PerSequence


def time_construction(cls, draft, target, prompts, gm):
    torch.manual_seed(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    bt = cls(draft, target, prompts, gm, policy="spec", temperature=T, top_p=1.0, max_length=M)
    bt.construct_grow_map()
    bt.verify()                                  # ends in the step's host sync
    return time.perf_counter() - t0


def time_admission(cls, draft, target, prompts, new, gm):
    torch.manual_seed(0)
    bt = cls(draft, target, prompts, gm, policy="spec", temperature=T, top_p=1.0, max_length=M)
    for _ in range(2):
        bt.construct_grow_map()
        bt.verify()
    b = bt.B - 1
    bt.freeze(b)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    bt.admit(b, new)
    bt.construct_grow_map()
    bt.verify()
    return time.perf_counter() - t0


def compare_first_verify(cls_per_seq, draft, target, prompts, gm):
    """Max abs difference of the first-verify target logits per sequence, both paths from the same drafted tree and KV."""
    from sequoia_b200.batch import BatchTree
    torch.manual_seed(0)
    bt = BatchTree(draft, target, prompts, gm, policy="spec", temperature=T, top_p=1.0, max_length=M)
    bt.use_graphs = False
    with torch.inference_mode():
        bt.construct_grow_map()
        seqs = list(range(bt.B))
        snap = bt._snapshot()
        bt.op_target_first(seqs)
        ragged = bt.target_logits.clone()
        bt._restore(snap)
        cls_per_seq.op_target_first(bt, seqs)
        per_seq = bt.target_logits.clone()
    S = bt.S
    return [float((ragged[b * S:(b + 1) * S].float() - per_seq[b * S:(b + 1) * S].float()).abs().max())
            for b in range(bt.B)]


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batches", default="4,8")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("measure_ragged needs a CUDA device")
    from measure_refill import gpu_info
    from sequoia_b200.batch import BatchTree
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    PerSequence = per_sequence_class()
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    g = torch.Generator().manual_seed(3)
    rng = random.Random(5)
    out = dict(gpu_info(), workload="c2: llama-68m -> llama-2-7b (random init), 128-node tree, T 0.6, M 384", runs=[])
    variants = (("ragged", BatchTree), ("per_sequence", PerSequence))
    for B in [int(x) for x in args.batches.split(",")]:
        draft = GraphInferenceEngine(M, "random-init:llama-68m:1", device=DEV, batch_size=B)
        target = GraphInferenceEngineTG(M, "random-init:llama-2-7b:2", device=DEV, batch_size=B)
        sets = {"prompts_128": [torch.randint(3, 32000, (PREFIX,), generator=g).to(DEV) for _ in range(B)],
                "prompts_mixed": [torch.randint(3, 32000, (rng.randint(*MIXED),), generator=g).to(DEV)
                                  for _ in range(B)]}
        new = torch.randint(3, 32000, (PREFIX,), generator=g).to(DEV)
        res = dict(B=B, mixed_lengths=[len(p) for p in sets["prompts_mixed"]])
        for _, cls in variants:                                    # warm-up: modules, allocator, GEMM algorithms
            for prompts in sets.values():
                time_construction(cls, draft, target, prompts, gm)
            time_admission(cls, draft, target, sets["prompts_128"], new, gm)
        times = {(k, name): [] for k in list(sets) + ["admission"] for name, _ in variants}
        for _ in range(args.reps):
            for name, cls in variants:
                for k, prompts in sets.items():
                    times[(k, name)].append(time_construction(cls, draft, target, prompts, gm))
                times[("admission", name)].append(time_admission(cls, draft, target, sets["prompts_128"], new, gm))
        for k in list(sets) + ["admission"]:
            ms = {name: 1e3 * statistics.median(times[(k, name)]) for name, _ in variants}
            res[k] = dict(ragged_ms=ms["ragged"], per_sequence_ms=ms["per_sequence"],
                          speedup=ms["per_sequence"] / ms["ragged"],
                          ragged_all_ms=[1e3 * t for t in times[(k, "ragged")]],
                          per_sequence_all_ms=[1e3 * t for t in times[(k, "per_sequence")]])
        res["first_verify_logits_max_abs_diff"] = {k: compare_first_verify(PerSequence, draft, target, p, gm)
                                                   for k, p in sets.items()}
        out["runs"].append(res)
        print(json.dumps(res), flush=True)
        del draft, target
        torch.cuda.empty_cache()
    print(json.dumps(out))
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
