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
import math
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


def device_stop_settings(prompts, stop):
    """--device-stop: prompt i's (stop_tokens, max_new_tokens) lists for BatchTree / admit: the stop ids of the target's
    config, and the budget that ends it at MAX_NEW_LEN tokens, where the host loop stops it (at least 1)."""
    ids = sorted(stop)
    return [ids] * len(prompts), [max(1, MAX_NEW_LEN - len(p)) for p in prompts]


def _record_logprobs(tree, b: int, i: int, means):
    """means[i] = the mean logprob of the tokens slot b generated for prompt i (a tree with logprobs; means None: off)."""
    if means is not None:
        lp = tree.token_logprobs(b)[0]
        means[i] = float(lp.double().mean()) if len(lp) else float("nan")


def _record_prompt_logprobs(tree, b: int, i: int, means):
    """means[i] = the mean logprob of prompt i's tokens after the first, scored in slot b (a tree with prompt logprobs;
    means None: off; NaN for a one-token prompt)."""
    if means is not None:
        lp = tree.prompt_logprobs(b)[0]
        means[i] = float(lp.double().mean()) if len(lp) else float("nan")


def decode_refill(tree, prompts, limits, stop=DEFAULT_STOP, step_times=None, seeds=None, policies=None,
                  device_stop=None, logprob_means=None, prompt_logprob_means=None, reused=None):
    """Decode every prompt of a queue on a BatchTree whose B slots start with prompts[:B]: each slot that finishes (a stop
    token, its length limit `limits[i]`, or out of room) takes the next prompt, until the queue is empty.
    -> (outputs, decoded tokens, per-sequence target steps, admission order); outputs[i] = prompt i's committed tokens.
    step_times: a list that receives ("steady" | "admission", seconds) per step; an admission step is timed from the
    first admit() of the step to the end of its verify.  seeds: for a seeded tree, prompt i's seed is seeds[i].
    policies: prompt i decodes with policies[i] ("spec" / "greedy"); None keeps each slot's policy.
    device_stop: (stop_tokens, max_new_tokens) per prompt (device_stop_settings), passed to each admission; None keeps
    each slot's.  logprob_means: a list that receives prompt i's mean token logprob at index i (--logprobs).
    prompt_logprob_means: the same for the mean logprob of prompt i's own tokens (--prompt-logprobs).
    reused: a list that receives the prompt tokens each admission reused from a slot's cached prefix; admissions then
    pass reuse_prefix=True (--reuse-prefix).  None: admit without it."""
    B = len(tree.frozen)
    slot = list(range(B))                        # prompt index decoding in each slot (None: the queue ran out)
    length = [len(p) for p in prompts[:B]]
    order, pending, nxt = list(range(B)), [], B
    outputs = [None] * len(prompts)
    decoded = steps = 0
    while any(i is not None for i in slot):
        t0 = time.perf_counter()
        for b in pending:
            kw = {}
            if seeds is not None:
                kw["seed"] = seeds[slot[b]]
            if policies is not None:
                kw["policy"] = policies[slot[b]]
            if device_stop is not None:
                kw["stop_tokens"], kw["max_new_tokens"] = device_stop[0][slot[b]], device_stop[1][slot[b]]
            if reused is not None:
                kw["reuse_prefix"] = True
            tree.admit(b, prompts[slot[b]], **kw)
            if reused is not None:
                reused.append(0 if tree.reused_prefix[b] is None else tree.reused_prefix[b][1])
        kind = "admission" if pending else "steady"
        pending = []
        tree.construct_grow_map()
        res = tree.verify()
        if step_times is not None:
            step_times.append((kind, time.perf_counter() - t0))
        for b, (valid, _, terminate) in enumerate(res):
            i = slot[b]
            if i is None:
                continue
            decoded += valid.shape[0] - length[b]
            steps += 1
            length[b] = valid.shape[0]
            last = int(valid[-1]) if valid.shape[0] else 0
            # tree.frozen[b] without `terminate`: the tree stopped the slot itself (no room for another tree)
            if terminate or tree.frozen[b] or last in stop or length[b] >= limits[i]:
                outputs[i] = valid.clone()           # the slot's token row is reused by the next prompt
                _record_logprobs(tree, b, i, logprob_means)
                _record_prompt_logprobs(tree, b, i, prompt_logprob_means)
                if not tree.frozen[b]:
                    tree.freeze(b)
                if nxt < len(prompts):
                    slot[b], length[b] = nxt, len(prompts[nxt])
                    order.append(nxt)
                    pending.append(b)
                    nxt += 1
                else:
                    slot[b] = None
    return outputs, decoded, steps, order


def decode_chunk(tree, chunk, limits, stop=DEFAULT_STOP, logprob_means=None, i0: int = 0, prompt_logprob_means=None):
    """Decode a BatchTree built on `chunk` until every sequence has finished.  -> (decoded tokens, per-sequence steps)
    logprob_means: a list that receives the mean token logprob of chunk[b] at index i0 + b (--logprobs);
    prompt_logprob_means the same for the mean logprob of chunk[b]'s own tokens (--prompt-logprobs)."""
    length = [len(p) for p in chunk]
    done = set()
    decoded = steps = 0
    while not all(tree.frozen):
        tree.construct_grow_map()
        for b, (valid, _, terminate) in enumerate(tree.verify()):
            if b in done:
                continue
            decoded += valid.shape[0] - length[b]
            steps += 1
            length[b] = valid.shape[0]
            last = int(valid[-1]) if valid.shape[0] else 0
            if terminate or tree.frozen[b] or last in stop or length[b] >= limits[b]:
                done.add(b)
                _record_logprobs(tree, b, i0 + b, logprob_means)
                _record_prompt_logprobs(tree, b, i0 + b, prompt_logprob_means)
                if not tree.frozen[b]:
                    tree.freeze(b)
    return decoded, steps


@torch.inference_mode()
def simulation_batch(target, draft, prompts, grow_map, policy, T, top_p, M, B: int, stop=DEFAULT_STOP,
                     refill: bool = False, seeds=None, policies=None, top_k: int = 0, device_stop: bool = False,
                     penalties=None, logprobs=None, logit_bias=None, min_p: float = 0.0, bad_words=None,
                     constrain_draft: bool = False, prompt_logprobs=None, reuse_prefix: bool = False):
    """--batch B: the same metric loop with B prompts decoded together (sequoia_b200.batch.BatchTree).  Chunked: B
    prompts at a time, each chunk until its last sequence stops.  refill: one batch whose finished slots take the next
    prompt (BatchTree.admit).  seeds: one per prompt (--device-rng): each sequence draws its random numbers on the device
    from its own seed.  policies: one per prompt (--policies), in place of `policy` for all.  top_k: every sampled
    prompt's top-k filter (--top-k, 0 = off).  device_stop: each sequence ends on the device at the stop ids and the
    length limit the host loop applies (--device-stop), without overshoot.  penalties: every prompt's
    repetition_penalty / frequency_penalty / presence_penalty keywords (--repetition-penalty ..., batch_penalties); refill
    admissions keep them.  logprobs: every prompt's logprobs setting (--logprobs, None = off); the mean logprob of each
    prompt's generated tokens is printed and returned.  logit_bias: every prompt's logit_bias / allowed_token_ids keywords
    (--logit-bias / --allowed-token-ids, batch_logit_bias); refill admissions keep them.  min_p: every sampled prompt's
    min-p filter (--min-p, 0 = off); refill admissions keep it.  bad_words: every prompt's bad_words / min_tokens
    keywords (--bad-words / --min-tokens, batch_bad_words); refill admissions keep them.  constrain_draft: BatchTree's
    constrain_draft (--constrain-draft): the draft rows get the allowed set, bias, bad words and guide too.
    prompt_logprobs: every prompt's prompt_logprobs setting (--prompt-logprobs, None = off); the mean logprob of each
    prompt's own tokens after the first and its perplexity exp(-mean) are printed and returned; refill admissions keep
    it.  reuse_prefix: every refill admission reuses the longest cached prefix of its prompt (--reuse-prefix); the total
    of reused prompt tokens is printed and returned."""
    from sequoia_b200.batch import BatchTree
    steps = decoded = 0                          # steps: target steps summed over sequences (per-sequence tokens / step)
    total_time = 0.0
    limits = [MAX_NEW_LEN] * len(prompts)
    prompts = [p.to(DEV) for p in prompts]
    chunks = [prompts[:B]] if refill else [prompts[i:i + B] for i in range(0, len(prompts), B)]
    dstop = device_stop_settings(prompts, stop) if device_stop else None
    means = None if logprobs is None else [float("nan")] * len(prompts)
    pmeans = None if prompt_logprobs is None else [float("nan")] * len(prompts)
    reused = [] if reuse_prefix else None
    for c, chunk in enumerate(chunks):
        i0 = c * B
        pol = policy if policies is None else policies[i0:i0 + len(chunk)]
        kw = dict(penalties or {})
        kw.update(logit_bias or {})
        kw.update(bad_words or {})
        if logprobs is not None:
            kw["logprobs"] = logprobs
        if prompt_logprobs is not None:
            kw["prompt_logprobs"] = prompt_logprobs
        if dstop is not None:
            kw.update(stop_tokens=dstop[0][i0:i0 + len(chunk)], max_new_tokens=dstop[1][i0:i0 + len(chunk)])
        tree = BatchTree(draft, target, chunk, grow_map, policy=pol, temperature=T, top_p=top_p, max_length=M,
                         max_target_seq=M, seeds=None if seeds is None else seeds[i0:i0 + len(chunk)], top_k=top_k, min_p=min_p,
                         constrain_draft=constrain_draft, **kw)
        torch.cuda.synchronize()
        t1 = time.time()
        if refill:
            _, d, s, _ = decode_refill(tree, prompts, limits, stop, seeds=seeds, policies=policies, device_stop=dstop,
                                       logprob_means=means, prompt_logprob_means=pmeans, reused=reused)
        else:
            d, s = decode_chunk(tree, chunk, limits[:len(chunk)], stop, logprob_means=means, i0=i0,
                                prompt_logprob_means=pmeans)
        decoded += d
        steps += s
        torch.cuda.synchronize()
        total_time += time.time() - t1
        draft.clear_kv()
        target.clear_kv()
    steps = max(steps, 1)
    print("total time :{:.5f}s, latency :{:.5f}s, decoding step: {}, large model step: {}, {}".format(
        total_time, total_time / max(decoded, 1), decoded, steps, decoded / steps))
    print("batch {}{}: aggregate {:.2f} tokens/s".format(B, " (refill)" if refill else "",
                                                         decoded / total_time if total_time > 0 else 0.0))
    res = dict(decoded_tokens=decoded, target_steps=steps, tokens_per_step=decoded / steps, seconds=total_time,
               tokens_per_second=decoded / total_time if total_time > 0 else 0.0, batch=B, refill=refill)
    if means is not None:
        for i, m in enumerate(means):
            print(f"prompt {i}: mean token logprob {m:.4f}")
        res["mean_token_logprob"] = means
    if pmeans is not None:
        ppl = [math.exp(-m) for m in pmeans]
        for i, (m, p) in enumerate(zip(pmeans, ppl)):
            print(f"prompt {i}: mean prompt-token logprob {m:.4f}, perplexity {p:.3f}")
        res["mean_prompt_logprob"], res["prompt_perplexity"] = pmeans, ppl
    if reused is not None:
        print(f"reused prompt tokens: {sum(reused)} in {len(reused)} admissions")
        res["reused_prompt_tokens"] = sum(reused)
    return res


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
                    help="decode this many prompts together (--Mode greedy, --tree spec|greedy; without --refill the "
                         "prompt count must divide)")
    ap.add_argument("--refill", action="store_true",
                    help="with --batch: keep the batch full, each finished slot takes the next prompt of the queue")
    ap.add_argument("--device-rng", action="store_true",
                    help="with --batch: each prompt draws its random numbers on the device from a stream of its own, "
                         "seeded (seed << 32) | prompt index, so its output does not depend on its slot or its neighbours")
    ap.add_argument("--policies", type=str, default=None,
                    help="with --batch and --tree spec: a comma-separated list of spec / greedy; prompt i decodes with "
                         "policies[i %% len], greedy and sampled prompts in one batch")
    ap.add_argument("--top-k", type=int, default=0,
                    help="with --batch: keep the K best target logits of each row before top_p (0 = off)")
    ap.add_argument("--bad-words", type=str, default=None,
                    help="with --batch: ID,ID,...;ID;... token sequences no prompt's output may contain")
    ap.add_argument("--min-tokens", type=int, default=None,
                    help="with --batch: the tokens every prompt generates before a stop id (or 0 / 2) may end it")
    ap.add_argument("--constrain-draft", action="store_true",
                    help="with --batch: apply the allowed ids, logit bias and bad words to the draft rows too, so the "
                         "draft proposes only tokens the target rows keep")
    ap.add_argument("--min-p", type=float, default=0.0,
                    help="with --batch: keep the target tokens whose probability is at least P times the row's largest, "
                         "before top_k and top_p (0 = off)")
    ap.add_argument("--device-stop", action="store_true",
                    help="with --batch: each sequence ends on the device at the target's stop ids (anywhere in an "
                         "accepted path) and at the length limit, exactly, instead of after the step")
    ap.add_argument("--repetition-penalty", type=float, default=1.0,
                    help="with --batch: HF's repetition penalty of every prompt (1 = off), on the target rows")
    ap.add_argument("--frequency-penalty", type=float, default=0.0,
                    help="with --batch: vLLM's frequency penalty of every prompt (0 = off), on the target rows")
    ap.add_argument("--presence-penalty", type=float, default=0.0,
                    help="with --batch: vLLM's presence penalty of every prompt (0 = off), on the target rows")
    ap.add_argument("--logprobs", type=int, default=None,
                    help="with --batch: the top alternatives per token (0..20); prints each prompt's mean token logprob")
    ap.add_argument("--prompt-logprobs", type=int, default=None,
                    help="with --batch: the top alternatives per prompt token (0..20); prints each prompt's mean "
                         "prompt-token logprob and perplexity under the target")
    ap.add_argument("--reuse-prefix", action="store_true",
                    help="with --batch --refill: each admission copies the longest prefix of its prompt whose K/V a "
                         "slot already holds and prefills only the rest; prints the reused prompt tokens")
    ap.add_argument("--logit-bias", type=str, default=None,
                    help="with --batch: ID:BIAS[,ID:BIAS...], added to every prompt's target logits (bias in [-100, 100])")
    ap.add_argument("--allowed-token-ids", type=str, default=None,
                    help="with --batch: LO-HI|ID[,...] (ranges inclusive), the only ids every prompt may generate")
    ap.add_argument("--target-weights", type=str, default="fp16", choices=["fp16", "fp8"],
                    help="fp8: the target's layer projections quantized to E4M3 with per-channel scales at load")
    return ap


def check_batch_args(args, n_prompts: int) -> int:
    """Refuse --batch / --refill combinations the batched path does not run; -> the engines' batch size."""
    if args.Mode != "greedy" or args.tree not in ("spec", "greedy") or args.offloading:
        raise SystemExit("--batch runs --Mode greedy with --tree spec or greedy, without --offloading")
    if args.batch < 1 or n_prompts < 1:
        raise SystemExit(f"--batch {args.batch} with {n_prompts} prompts")
    if args.refill:
        return min(args.batch, n_prompts)
    if n_prompts % args.batch:
        raise SystemExit(f"--batch {args.batch} must divide the {n_prompts} prompts (or use --refill)")
    return args.batch


def device_rng_seeds(args, n_prompts: int):
    """--device-rng: prompt i's seed (args.seed << 32) | i; None without the flag.  Refused without --batch."""
    if not args.device_rng:
        return None
    if args.batch == 1 and not args.refill:
        raise SystemExit("--device-rng runs with --batch (the batched tree); the lone trees keep the reference's draws")
    if not 0 <= args.seed < 1 << 32:
        raise SystemExit(f"--device-rng needs --seed in [0, 2^32), got {args.seed}")
    return [(args.seed << 32) | i for i in range(n_prompts)]


def prompt_policies(args, n_prompts: int):
    """--policies: prompt i's policy policies[i % len]; None without the flag.  Refused without --batch, with a --tree
    other than spec, and with an entry other than spec / greedy."""
    if args.policies is None:
        return None
    if args.batch == 1 and not args.refill:
        raise SystemExit("--policies runs with --batch (the batched tree)")
    if args.tree != "spec":
        raise SystemExit(f"--policies takes the place of --tree spec, got --tree {args.tree}")
    pols = [p.strip() for p in args.policies.split(",")]
    bad = [p for p in pols if p not in ("spec", "greedy")]
    if bad:
        raise SystemExit(f"--policies: entries must be spec or greedy, got {args.policies!r}")
    return [pols[i % len(pols)] for i in range(n_prompts)]


def batch_top_k(args) -> int:
    """--top-k: every prompt's top_k (0 = off).  Refused below 0, and without --batch: the lone trees keep the
    reference's sampling."""
    if args.top_k < 0:
        raise SystemExit(f"--top-k must be >= 0, got {args.top_k}")
    if args.top_k and args.batch == 1 and not args.refill:
        raise SystemExit("--top-k runs with --batch (the batched tree); the lone trees keep the reference's sampling")
    return args.top_k


def batch_min_p(args) -> float:
    """--min-p: every prompt's min_p (0 = off).  Refused outside [0, 1], and without --batch: the lone trees keep the
    reference's sampling."""
    if not 0.0 <= args.min_p <= 1.0:
        raise SystemExit(f"--min-p must be in [0, 1], got {args.min_p}")
    if args.min_p and args.batch == 1 and not args.refill:
        raise SystemExit("--min-p runs with --batch (the batched tree); the lone trees keep the reference's sampling")
    return args.min_p


def batch_device_stop(args) -> bool:
    """--device-stop: refused without --batch / --refill (the lone trees keep the reference's end rule)."""
    if args.device_stop and args.batch == 1 and not args.refill:
        raise SystemExit("--device-stop runs with --batch (the batched tree); the lone trees keep the reference's end rule")
    return args.device_stop


def batch_penalties(args) -> dict:
    """--repetition-penalty / --frequency-penalty / --presence-penalty: BatchTree's keywords for every prompt ({} when all
    are off).  Refused outside the ranges BatchTree takes, and without --batch: the lone trees keep the reference's
    sampling."""
    from sequoia_b200.batch import check_penalty, is_neutral
    vals = {}
    for name in ("repetition_penalty", "frequency_penalty", "presence_penalty"):
        try:
            vals[name] = check_penalty(name, getattr(args, name))
        except ValueError as e:
            raise SystemExit(f"--{name.replace('_', '-')}: {e}")
    if is_neutral(*vals.values()):
        return {}
    if args.batch == 1 and not args.refill:
        raise SystemExit("--repetition-penalty / --frequency-penalty / --presence-penalty run with --batch (the batched "
                         "tree); the lone trees keep the reference's sampling")
    return vals


def batch_prompt_logprobs(args):
    """--prompt-logprobs N: every prompt's prompt_logprobs setting (None = off).  Refused outside 0..20, and without
    --batch: the lone trees score no prompt."""
    if args.prompt_logprobs is None:
        return None
    from sequoia_b200.batch import check_prompt_logprobs
    try:
        n = check_prompt_logprobs(args.prompt_logprobs)
    except ValueError as e:
        raise SystemExit(f"--prompt-logprobs: {e}")
    if args.batch == 1 and not args.refill:
        raise SystemExit("--prompt-logprobs runs with --batch (the batched tree); the lone trees score no prompt")
    return n


def batch_logprobs(args):
    """--logprobs N: every prompt's logprobs setting (None = off).  Refused outside 0..20, and without --batch: the lone
    trees compute no logprobs."""
    if args.logprobs is None:
        return None
    from sequoia_b200.batch import check_logprobs
    try:
        n = check_logprobs(args.logprobs)
    except ValueError as e:
        raise SystemExit(f"--logprobs: {e}")
    if args.batch == 1 and not args.refill:
        raise SystemExit("--logprobs runs with --batch (the batched tree); the lone trees compute no logprobs")
    return n


def _parse_logit_bias(text: str) -> dict:
    out = {}
    for item in text.split(","):
        t, sep, v = item.partition(":")
        if not sep:
            raise ValueError(f"{item!r} is not ID:BIAS")
        out[int(t)] = float(v)
    return out


def _parse_token_ids(text: str) -> list:
    out = []
    for item in text.split(","):
        lo, sep, hi = item.strip().partition("-")
        out.extend(range(int(lo), int(hi) + 1) if sep else [int(lo)])
    return out


def batch_logit_bias(args) -> dict:
    """--logit-bias ID:BIAS[,...] / --allowed-token-ids LO-HI|ID[,...]: BatchTree's logit_bias / allowed_token_ids for
    every prompt ({} when neither is given).  Refused when malformed or outside what BatchTree takes (ids are checked
    against the vocabulary when the tree is built), and without --batch: the lone trees keep the reference's sampling."""
    from sequoia_b200.batch import check_allowed_token_ids, check_logit_bias
    kw = {}
    for flag, attr, parse, check in (("--logit-bias", "logit_bias", _parse_logit_bias, check_logit_bias),
                                     ("--allowed-token-ids", "allowed_token_ids", _parse_token_ids,
                                      check_allowed_token_ids)):
        text = getattr(args, attr)
        if text is None:
            continue
        try:
            val = check(parse(text))
        except ValueError as e:
            raise SystemExit(f"{flag}: {e}")
        kw[attr] = dict(val) if attr == "logit_bias" else val     # (a mapping: a sequence would be one per prompt)
    if kw and args.batch == 1 and not args.refill:
        raise SystemExit("--logit-bias / --allowed-token-ids run with --batch (the batched tree); the lone trees keep the "
                         "reference's sampling")
    return kw


def batch_constrain_draft(args) -> bool:
    """--constrain-draft: BatchTree's constrain_draft.  Refused without --batch: the lone trees process no draft rows."""
    if args.constrain_draft and args.batch == 1 and not args.refill:
        raise SystemExit("--constrain-draft runs with --batch (the batched tree); the lone trees process no draft rows")
    return bool(args.constrain_draft)


def batch_reuse_prefix(args) -> bool:
    """--reuse-prefix: admit(reuse_prefix=True) for every refill admission.  Refused without --refill: only admissions
    reuse a prefix (a tree's first prompts have none cached)."""
    if args.reuse_prefix and not args.refill:
        raise SystemExit("--reuse-prefix runs with --refill (admissions reuse cached prefixes; a new tree has none)")
    return bool(args.reuse_prefix)


def batch_bad_words(args) -> dict:
    """--bad-words ID,ID,...;ID;... / --min-tokens N: BatchTree's bad_words / min_tokens for every prompt ({} when
    neither is given).  Refused when malformed or outside what BatchTree takes (ids are checked against the vocabulary
    when the tree is built), and without --batch: the lone trees keep the reference's sampling."""
    from sequoia_b200.batch import check_bad_words, check_min_tokens
    kw = {}
    try:
        if args.bad_words is not None:
            words = [[int(t) for t in w.split(",")] for w in args.bad_words.split(";")]
            check_bad_words(words)
            kw["bad_words"] = words
    except ValueError as e:
        raise SystemExit(f"--bad-words: {e}")
    try:
        if args.min_tokens is not None:
            kw["min_tokens"] = check_min_tokens(args.min_tokens)
    except ValueError as e:
        raise SystemExit(f"--min-tokens: {e}")
    if kw and args.batch == 1 and not args.refill:
        raise SystemExit("--bad-words / --min-tokens run with --batch (the batched tree); the lone trees keep the "
                         "reference's sampling")
    return kw


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
    seeds = device_rng_seeds(args, len(prompts))
    policies = prompt_policies(args, len(prompts))
    top_k = batch_top_k(args)
    min_p = batch_min_p(args)
    device_stop = batch_device_stop(args)
    penalties = batch_penalties(args)
    logprobs = batch_logprobs(args)
    prompt_logprobs = batch_prompt_logprobs(args)
    logit_bias = batch_logit_bias(args)
    bad_words = batch_bad_words(args)
    constrain_draft = batch_constrain_draft(args)
    reuse_prefix = batch_reuse_prefix(args)
    if args.batch != 1 or args.refill:
        B = check_batch_args(args, len(prompts))
        target = GraphInferenceEngineTG(max_length=args.M, model_name_or_path=args.target, dtype=torch.float16,
                                        device=DEV, batch_size=B, weight_format=args.target_weights)
        draft = GraphInferenceEngine(max_length=args.M, model_name_or_path=args.model, dtype=torch.float16, device=DEV,
                                     batch_size=B)
        path = args.growmap if os.path.isabs(args.growmap) or os.path.exists(args.growmap) else os.path.join(ROOT, args.growmap)
        grow_map = torch.load(path)
        assert args.M >= MAX_NEW_LEN + grow_map["size"], "--M must hold 256 tokens + the tree (README.md:47 of the reference)"
        res = simulation_batch(target, draft, prompts, grow_map, args.tree, args.T, args.P, args.M, B, stop=stop,
                               refill=args.refill, seeds=seeds, policies=policies, top_k=top_k,
                               device_stop=device_stop, penalties=penalties, logprobs=logprobs,
                               logit_bias=logit_bias, min_p=min_p, bad_words=bad_words,
                               constrain_draft=constrain_draft, prompt_logprobs=prompt_logprobs,
                               reuse_prefix=reuse_prefix)
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
