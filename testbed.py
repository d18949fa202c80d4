"""End-to-end driver with the command line of the reference's tests/testbed.py (tree speculative decoding of a prompt
set, reporting accepted tokens per target step and wall time), running on the sequoia_b200 engines.

    python testbed.py --model <draft> --target <target> --growmap A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt \
        --T 0.6 --P 1.0 --M 384 --Mode greedy --dataset synthetic --start 0 --end 20

Same flags and modes as the reference (tests/testbed.py:21-33):
  --Mode greedy      simulation_fast (:45-95): the metric loop (BASELINE.md), tree policy chosen by --tree
  --Mode benchmark   simulation_benchmark (:138-213): the same loop with per-phase timers (eager, synchronised)
  --Mode baseline    simulation_baseline (:98-137): plain autoregressive sampling from the target, 32 tokens per prompt
Models are local directories or `random-init:<name>[:seed]` (no hub access); `--dataset` is `synthetic` or a JSON-lines /
JSON file of token-id lists (`input_tokens` / `input_ids` keys, e.g. the reference's dataset/c4_small.json) — no
tokenizer is needed.  `--tree {spec,greedy,specinfer,greedys}` selects the tree class (the reference edits the import).
"""
from __future__ import annotations

import argparse
import json
import os
import random
import sys
import time
from typing import List

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
DEV = "cuda:0"
PREFIX = 128            # tests/testbed.py:59 — prompts are cut to 128 tokens
MAX_NEW_LEN = 256       # :80 — decode until the sequence holds 256 tokens


def load_prompts(spec: str, start: int, end: int, seed: int, vocab_size: int = 32000) -> List[torch.Tensor]:
    """`synthetic` -> random ids in [3, vocab); else a file of token-id lists (JSON lines or one JSON array)."""
    if spec == "synthetic":
        from data_converter import synthetic_prompts
        return synthetic_prompts(end, PREFIX, vocab_size, seed)[start:end]
    rows = []
    with open(spec) as f:
        text = f.read().strip()
    try:
        data = json.loads(text)
        rows = data if isinstance(data, list) else [data]
    except json.JSONDecodeError:
        rows = [json.loads(line) for line in text.splitlines() if line.strip()]
    out = []
    for r in rows[start:end]:
        ids = r.get("input_tokens", r.get("input_ids")) if isinstance(r, dict) else r
        ids = [int(t) for t in ids][:PREFIX]
        if len(ids) == PREFIX:                       # the reference skips padded (short) rows, :62
            out.append(torch.tensor(ids, dtype=torch.long))
    return out


def setup_seed(seed: int):
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)
    np.random.seed(seed)
    random.seed(seed)


def _buffers(M: int):
    dtype = torch.float16
    return dict(attn_mask=torch.full((M, M), torch.finfo(dtype).min, dtype=dtype, device=DEV),
                sequence=torch.arange(M, device=DEV).long().unsqueeze(-1),
                new_tokens_buffer=torch.zeros(M, device=DEV).long(), parents_buffer=torch.zeros(M, device=DEV).long(),
                position_ids=torch.zeros(M, device=DEV).long())


def _tree_class(name: str):
    if name == "spec":
        from Tree.SpecTree import SpecTree as cls
    elif name == "greedy":
        from Tree.GreedyTree import GreedyTree as cls
    elif name == "specinfer":
        from Tree.SpecInferTree import SpecInferTree as cls
    else:
        from Tree.GreedySTree import GreedySTree as cls
    return cls


def stop_tokens(model_name_or_path) -> frozenset:
    """Token ids that end a generation: `eos_token_id` (an int or a list) of the model directory's config.json when it has
    one, else 2 and 0 (the Llama-2 eos and pad ids, what the reference stops on)."""
    path = os.path.join(str(model_name_or_path), "config.json")
    if os.path.isfile(path):
        with open(path) as f:
            eos = json.load(f).get("eos_token_id")
        if isinstance(eos, int):
            return frozenset([eos])
        if isinstance(eos, (list, tuple)) and eos:
            return frozenset(int(t) for t in eos)
    return DEFAULT_STOP


DEFAULT_STOP = frozenset([0, 2])


@torch.inference_mode()
def simulation(target, draft, prompts, grow_map, tree_cls, T, top_p, M, benchmark: bool, stop=DEFAULT_STOP):
    """simulation_fast / simulation_benchmark."""
    bufs = _buffers(M)
    steps = decoded = 0
    total_time = 0.0
    phase = dict(speculate=0.0, verify=0.0, sample=0.0, small=0.0, large=0.0, accept=0.0, kv=0.0)
    for prompt in prompts:
        input_ids = prompt.view(1, -1).to(DEV)
        bufs["attn_mask"].fill_(torch.finfo(torch.float16).min)
        tree = tree_cls(prefix=input_ids[0], device=DEV, temperature=T, top_p=top_p, draft_kv_len=0, target_kv_len=0,
                        draft_model_engine=draft, target_model_engine=target, max_length=M, max_target_seq=M,
                        grow_map=grow_map, residual_graph=None, sampling_callables=None, sample_gather_indices=None,
                        **bufs)
        terminate = False
        torch.cuda.synchronize()
        t1 = time.time()
        while input_ids.shape[1] < MAX_NEW_LEN and not terminate:
            n0 = input_ids.shape[1]
            if benchmark:
                t2 = time.time()
                a, b = tree.construct_grow_map(benchmark=True)
                torch.cuda.synchronize()
                t3 = time.time()
                valid, _, _, x, y, z, terminate = tree.verify(benchmark=True)
                torch.cuda.synchronize()
                t4 = time.time()
            else:
                tree.construct_grow_map()
                valid, _, _, terminate = tree.verify()
            input_ids = valid.unsqueeze(0)
            last = int(input_ids[0, -1])
            if last in stop:
                terminate = True
            if benchmark:
                if any(int(t) in stop for t in input_ids[0].tolist()) or input_ids.shape[1] >= MAX_NEW_LEN:
                    terminate = True
                if terminate:                          # the reference drops the last step from the phase averages
                    continue
                for k, v in (("sample", a), ("small", b), ("large", x), ("accept", y), ("kv", z),
                             ("speculate", t3 - t2), ("verify", t4 - t3)):
                    phase[k] += v
            decoded += valid.shape[0] - n0
            steps += 1
        torch.cuda.synchronize()
        total_time += time.time() - t1
        draft.clear_kv()
        target.clear_kv()
    steps = max(steps, 1)
    print("total time :{:.5f}s, latency :{:.5f}s, decoding step: {}, large model step: {}, {}".format(
        total_time, total_time / max(decoded, 1), decoded, steps, decoded / steps))
    if benchmark:
        print("speculate time: {}".format(phase["speculate"] / steps), "verify time: {}".format(phase["verify"] / steps))
        print("large model run: {}".format(phase["large"] / steps), "accept loop: {}".format(phase["accept"] / steps),
              "kv select: {}".format(phase["kv"] / steps))
        print("small model run: {}".format(phase["small"] / steps), "sample time: {}".format(phase["sample"] / steps))
    return dict(decoded_tokens=decoded, target_steps=steps, tokens_per_step=decoded / steps, seconds=total_time,
                tokens_per_second=decoded / total_time if total_time > 0 else 0.0)


@torch.inference_mode()          # engine outputs are inference tensors; the nucleus filter edits them in place
def simulation_baseline(target, prompts, T, top_p, M, new_tokens: int = 32, stop=DEFAULT_STOP):
    """Autoregressive sampling from the target alone (tests/testbed.py:98-137)."""
    from utils import _make_causal_mask, get_sampling_logits
    position_ids = torch.arange(M, device=DEV).unsqueeze(0)
    storage_ids = torch.arange(M, device=DEV)
    mask = _make_causal_mask((M, M), target.dtype, target.device)
    total_time, decoded = 0.0, 0
    for prompt in prompts:
        ids = prompt.view(1, -1).to(DEV)
        n0 = ids.shape[1]
        torch.cuda.synchronize()
        t1 = time.time()
        for i in range(new_tokens):
            lo, hi = (0, n0) if i == 0 else (n0 + i - 1, n0 + i)
            logits = target.inference(input_ids=ids, storage_ids=storage_ids[lo:hi], position_ids=position_ids[..., lo:hi],
                                      attn_mask=mask[lo:hi, :hi][None, None, :, :])[0][-1]
            logits = get_sampling_logits(logits=logits, top_p=top_p, T=T)
            ids = torch.softmax(logits / T, dim=-1).multinomial(num_samples=1).unsqueeze(0)
            decoded += 1
            if int(ids[0, -1]) in stop - {0}:      # (the baseline loop only ever stopped on eos)
                break
        torch.cuda.synchronize()
        total_time += time.time() - t1
        target.clear_kv()
    print("total time :{:.5f}s, latency :{:.5f}s, decoding step: {}".format(total_time, total_time / max(decoded, 1), decoded))
    return dict(decoded_tokens=decoded, seconds=total_time, latency=total_time / max(decoded, 1))


@torch.inference_mode()
def simulation_batch(target, draft, prompts, grow_map, policy, T, top_p, M, B: int, stop=DEFAULT_STOP):
    """--batch B: the same metric loop with B prompts decoded together (sequoia_b200.batch.BatchTree)."""
    from sequoia_b200.batch import BatchTree
    steps = decoded = 0                          # steps: target steps summed over sequences (per-sequence tokens / step)
    total_time = 0.0
    for i in range(0, len(prompts), B):
        chunk = [p.to(DEV) for p in prompts[i:i + B]]
        tree = BatchTree(draft, target, chunk, grow_map, policy=policy, temperature=T, top_p=top_p, max_length=M,
                         max_target_seq=M)
        length = [len(p) for p in chunk]
        done = set()
        torch.cuda.synchronize()
        t1 = time.time()
        while not all(tree.frozen):
            tree.construct_grow_map()
            for b, (valid, _, terminate) in enumerate(tree.verify()):
                if b in done:
                    continue
                decoded += valid.shape[0] - length[b]
                steps += 1
                length[b] = valid.shape[0]
                last = int(valid[-1]) if valid.shape[0] else 0
                if terminate or last in stop or length[b] >= MAX_NEW_LEN:
                    done.add(b)
                    if not tree.frozen[b]:
                        tree.freeze(b)
        torch.cuda.synchronize()
        total_time += time.time() - t1
        draft.clear_kv()
        target.clear_kv()
    steps = max(steps, 1)
    print("total time :{:.5f}s, latency :{:.5f}s, decoding step: {}, large model step: {}, {}".format(
        total_time, total_time / max(decoded, 1), decoded, steps, decoded / steps))
    print("batch {}: aggregate {:.2f} tokens/s".format(B, decoded / total_time if total_time > 0 else 0.0))
    return dict(decoded_tokens=decoded, target_steps=steps, tokens_per_step=decoded / steps, seconds=total_time,
                tokens_per_second=decoded / total_time if total_time > 0 else 0.0, batch=B)


def build_parser():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--model", type=str, default="random-init:llama-68m", help="draft model")
    ap.add_argument("--target", type=str, default="random-init:llama-68m:2", help="target model")
    ap.add_argument("--dataset", type=str, default="synthetic", help="'synthetic' or a JSON(-lines) file of token ids")
    ap.add_argument("--growmap", type=str, default="L40_growmaps/8x8-tree.pt", help="growmap path")
    ap.add_argument("--start", type=int, default=0)
    ap.add_argument("--end", type=int, default=20)
    ap.add_argument("--T", type=float, default=0.6, help="temperature")
    ap.add_argument("--P", type=float, default=0.9, help="top_p")
    ap.add_argument("--M", type=int, default=384, help="max length (>= 256 + tree size)")
    ap.add_argument("--seed", type=int, default=17)
    ap.add_argument("--Mode", type=str, default="greedy", choices=["greedy", "benchmark", "baseline"])
    ap.add_argument("--tree", type=str, default="spec", choices=["spec", "greedy", "specinfer", "greedys"])
    ap.add_argument("--offloading", action="store_true", help="use OffloadEngine for the target (weights stay resident)")
    ap.add_argument("--batch", type=int, default=1,
                    help="decode this many prompts together (--Mode greedy, --tree spec|greedy; the prompt count must divide)")
    ap.add_argument("--target-weights", type=str, default="fp16", choices=["fp16", "fp8"],
                    help="fp8: the target's layer projections quantized to E4M3 with per-channel scales at load")
    return ap


def main(argv=None):
    args = build_parser().parse_args(argv)
    print(args)
    setup_seed(args.seed)
    from Engine.Engine import GraphInferenceEngine, GraphInferenceEngineTG
    from Engine.offload_engine import OffloadEngine
    prompts = load_prompts(args.dataset, args.start, args.end, args.seed)
    tcls = OffloadEngine if args.offloading else GraphInferenceEngineTG
    stop = stop_tokens(args.target)
    if args.target_weights != "fp16" and args.offloading:
        raise SystemExit("--target-weights fp8 runs without --offloading")
    if args.batch != 1:
        if args.Mode != "greedy" or args.tree not in ("spec", "greedy") or args.offloading:
            raise SystemExit("--batch runs --Mode greedy with --tree spec or greedy, without --offloading")
        if len(prompts) % args.batch:
            raise SystemExit(f"--batch {args.batch} must divide the {len(prompts)} prompts")
        target = GraphInferenceEngineTG(max_length=args.M, model_name_or_path=args.target, dtype=torch.float16,
                                        device=DEV, batch_size=args.batch, weight_format=args.target_weights)
        draft = GraphInferenceEngine(max_length=args.M, model_name_or_path=args.model, dtype=torch.float16, device=DEV,
                                     batch_size=args.batch)
        path = args.growmap if os.path.isabs(args.growmap) or os.path.exists(args.growmap) else os.path.join(ROOT, args.growmap)
        grow_map = torch.load(path)
        assert args.M >= MAX_NEW_LEN + grow_map["size"], "--M must hold 256 tokens + the tree (README.md:47 of the reference)"
        res = simulation_batch(target, draft, prompts, grow_map, args.tree, args.T, args.P, args.M, args.batch,
                               stop=stop)
        print(json.dumps({k: (round(v, 5) if isinstance(v, float) else v) for k, v in res.items()}))
        return res
    target = (tcls(max_length=args.M, model_name_or_path=args.target, dtype=torch.float16, device=DEV)
              if args.offloading else
              tcls(max_length=args.M, model_name_or_path=args.target, dtype=torch.float16, device=DEV,
                   weight_format=args.target_weights))
    if args.Mode == "baseline":
        res = simulation_baseline(target, prompts, args.T, args.P, args.M, stop=stop)
    else:
        draft = GraphInferenceEngine(max_length=args.M, model_name_or_path=args.model, dtype=torch.float16, device=DEV)
        path = args.growmap if os.path.isabs(args.growmap) or os.path.exists(args.growmap) else os.path.join(ROOT, args.growmap)
        grow_map = torch.load(path)
        assert args.M >= MAX_NEW_LEN + grow_map["size"], "--M must hold 256 tokens + the tree (README.md:47 of the reference)"
        res = simulation(target, draft, prompts, grow_map, _tree_class(args.tree), args.T, args.P, args.M,
                         benchmark=(args.Mode == "benchmark"), stop=stop)
    print(json.dumps({k: (round(v, 5) if isinstance(v, float) else v) for k, v in res.items()}))
    return res


if __name__ == "__main__":
    main()
