"""Cost of 128K-vocabulary decoding on one GPU.

1. Decode: random-init llama-3.2-1b -> llama-3.1-8b (V = 128256), A100-CNN-68m-7b-stochastic.pt (128-node tree), T 0.6,
   top_p 1, M 384, 128-token prompts, through SpecTree (B = 1) and BatchTree (B = 2): ms per step (CUDA events around
   construct_grow_map() + verify() after warm-up steps that capture the graphs), accepted tokens per step per sequence
   and aggregate tokens/s.
2. Kernels: per-launch time (CUDA events over many launches) of sq_sample_level (mode 0, 16 rows, k 8),
   sq_top_p_filter (128 rows), sq_argmax_rows (128 rows) and sq_accept_stochastic (128-node tree) at V = 128256 against
   V = 32000, with achieved bytes/s from the algorithmic bytes of DESIGN.md section 4 (sampling: logits + rand read;
   top-p and argmax: one logits read; accept: target + draft row of every visited parent, counted as the root's two rows).
3. lm_head: sq_gemm (the route LlamaRunner takes for <= 128 rows) against torch.mm at N = 128256, K = 4096 and 2048, for
   1, 19 and 128 rows, with achieved bytes/s of the weight stream.

The GPU name and power limit are read in the same run.

    python tools/measure_large_vocab.py --out result.json [--steps 20 --warmup 4] [--skip-decode]
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
F16 = torch.float16


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = [x.strip() for x in q.split(",")]
    return dict(gpu=name, power_limit=limit)


def per_launch_us(fn, n=200, warmup=10):
    for _ in range(warmup):
        fn()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(n):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) * 1000.0 / n


def decode(steps, warmup):
    from sequoia_b200.batch import BatchTree
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG
    from sequoia_b200.tree import SpecTree, clear_runtimes
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(0, 128256, (PREFIX,), generator=g) for _ in range(2)]
    out = {}
    for B in (1, 2):
        clear_runtimes()
        draft = GraphInferenceEngine(M, "random-init:llama-3.2-1b:1", device=DEV, batch_size=B)
        target = GraphInferenceEngineTG(M, "random-init:llama-3.1-8b:2", device=DEV, batch_size=B)
        torch.manual_seed(0)
        if B == 1:
            tree = SpecTree(draft, target, prompts[0].to(DEV), temperature=T, top_p=1.0, max_length=M, max_target_seq=M,
                            device=DEV, grow_map=gm)
            lens = [PREFIX]

            def step():
                tree.construct_grow_map()
                v = tree.verify()[0]
                n, lens[0] = len(v) - lens[0], len(v)
                return n
        else:
            tree = BatchTree(draft, target, [p.to(DEV) for p in prompts], gm, policy="spec", temperature=T, top_p=1.0,
                             max_length=M, max_target_seq=M)
            lens = [PREFIX] * B

            def step():
                tree.construct_grow_map()
                n = 0
                for b, (v, _, _) in enumerate(tree.verify()):
                    n, lens[b] = n + len(v) - lens[b], len(v)
                return n
        for _ in range(warmup):
            step()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        tokens = sum(step() for _ in range(steps))
        ev1.record()
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1)
        out[f"B{B}"] = dict(ms_per_step=round(ms / steps, 3), accepted_tokens_per_step=round(tokens / steps / B, 3),
                            tokens_per_s=round(tokens / (ms / 1000.0), 1), steps=steps)
        print(f"decode B={B}: {out[f'B{B}']}", flush=True)
        del tree, draft, target
        torch.cuda.empty_cache()
    clear_runtimes()
    return out


def kernels():
    from sequoia_b200 import ops
    from sequoia_b200.tree import _Static
    gm = torch.load(os.path.join(ROOT, GROWMAP))
    S = gm["size"]
    st = _Static(gm, DEV)
    out = {}
    for V in (32000, 128256):
        g = torch.Generator(device=DEV).manual_seed(V)
        lg = (torch.randn(S, V, device=DEV, generator=g) * 3).half()
        rand = torch.rand(S, V, device=DEV, generator=g).clamp(min=1e-4).half()
        pos = torch.zeros(16, 8, dtype=torch.int64, device=DEV)
        am = torch.zeros(S, dtype=torch.int64, device=DEV)
        work = lg.clone()
        tokens = torch.randint(0, V, (M,), device=DEV)
        r = torch.rand(M, device=DEV).half()
        noise = torch.empty(V, device=DEV).exponential_(1.0).half()
        acc = torch.zeros(S, dtype=torch.int32, device=DEV)
        state = torch.zeros(16, dtype=torch.int32, device=DEV)

        def accept():
            state.zero_()
            state[0], state[8] = PREFIX, M
            ops.accept_stochastic(lg, lg, r, noise, st.succ_off, st.succ, st.depth, S, T, tokens, torch.arange(M, device=DEV),
                                  acc, state, M)

        t_state = per_launch_us(lambda: (state.zero_(), state.__setitem__(0, PREFIX), state.__setitem__(8, M)))
        row = V * 2
        res = {
            "sample_level(16 rows, k 8)": (per_launch_us(lambda: ops.sample_level(lg, rand, 16, 8, T, 0, positions=pos)),
                                           16 * 2 * row),
            "top_p_filter(128 rows)": (per_launch_us(lambda: (work.copy_(lg), ops.top_p_filter_(work, 0.9, T)))
                                       - per_launch_us(lambda: work.copy_(lg)), S * row),
            "argmax_rows(128 rows)": (per_launch_us(lambda: ops.argmax_rows(lg, am)), S * row),
            "accept_stochastic(128-node tree)": (per_launch_us(accept) - t_state, 2 * row),
        }
        out[f"V{V}"] = {k: dict(us=round(us, 2), GBps=round(b / us / 1e3, 1)) for k, (us, b) in res.items()}
        print(f"kernels V={V}: {out[f'V{V}']}", flush=True)
    return out


def lm_head():
    from sequoia_b200 import ops
    out = {}
    N = 128256
    for K in (4096, 2048):
        w = (torch.randn(N, K, device=DEV) * 0.02).half()
        a = torch.randn(128, K, device=DEV).half()
        c = torch.zeros(128, N, dtype=F16, device=DEV)
        plan = ops.GemmPlan(a, w, c)
        for n in (1, 19, 128):
            us_g = per_launch_us(lambda: plan.run(n), n=50)
            us_t = per_launch_us(lambda: torch.mm(a[:n], w.t(), out=c[:n]), n=50)
            wb = N * K * 2
            out[f"K{K}_n{n}"] = dict(sq_gemm_us=round(us_g, 1), torch_mm_us=round(us_t, 1),
                                     sq_gemm_GBps=round(wb / us_g / 1e3, 1), torch_mm_GBps=round(wb / us_t / 1e3, 1))
            print(f"lm_head K={K} n={n}: {out[f'K{K}_n{n}']}", flush=True)
        del w, a, c, plan
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--skip-decode", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("measure_large_vocab.py measures on a CUDA GPU; none is visible")
    res = dict(**gpu_info())
    print(res, flush=True)
    res["kernels"] = kernels()
    res["lm_head"] = lm_head()
    if not args.skip_decode:
        res["decode"] = decode(args.steps, args.warmup)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
