"""Per-projection device times of the 128-row verify GEMMs of a Llama-2-7B target, and of one whole 7B layer.

For each projection of the c2 verify (rows n = 128, 97, 127 by default) it times
  * cuBLASLt: torch.mm (plus sq_silu_mul for gate_up),
  * the weight-streaming wgmma GEMM (csrc/sq_gemm.cu) with the tile the library picks,
  * with --sweep: every legal (bn, split, mc) tile of that kernel (forced through SQ_GEMM_FORCE at plan creation).
Every timing is a CUDA graph that cycles over COPIES weight copies (>= 6, 2+ GB in all), so the weights come from HBM and
not from the 50 MB L2.  It reports us per call, weight GB/s and that rate's share of the H100 SXM data-sheet 3.35 TB/s.

--layer also times one 7B-shaped decoder layer as the model runs it (rmsnorm, qkv, RoPE + KV append, attention, o_proj,
add_rmsnorm, gate_up (+ silu_mul), down_proj, add_rmsnorm) on a 4-layer LlamaRunner, on each route of --routes:
programmatic dependent launch only shows up in such a chain.  A route is "model" (the runner's own routes), "cublas"
(every projection on torch.mm + sq_silu_mul), or "+"-joined projections on sq_gemm plans, each with the tile the library
picks or a forced one: "gu+qkv+o=64:2:1+down=128:4:1" (gu = the fused gate_up plan; the others stay on cuBLASLt).

Prints the card and its power limit first; --json writes every number.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from sequoia_b200 import ops  # noqa: E402

HBM_PEAK_GBS = 3350.0            # H100 SXM data sheet (HBM3), for a card allowed up to 700 W
SHAPES = {                       # projection: (N, K, SwiGLU epilogue) of Llama-2-7B
    "qkv": (12288, 4096, False),
    "o_proj": (4096, 4096, False),
    "gate_up": (22016, 4096, True),
    "down_proj": (4096, 11008, False),
    "lm_head": (32000, 4096, False),
    "gate_up_13b": (27648, 5120, True),              # Llama-2-13B (not in the default set: --only gate_up_13b)
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                   # the numbers below still stand, without the limit beside them
        q = f"power limit unknown ({e})"
    return f"{name}, {torch.cuda.get_device_properties(0).multi_processor_count} SMs, power limit / max SM clock: {q}"


def graph_time_us(fn, copies, reps):
    """Median over `reps` replays of a graph of 4 * copies calls fn(i % copies), in us per call."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(copies):
            fn(i)
    s.synchronize()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(4 * copies):
            fn(i % copies)
    g.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / (4 * copies))
    times.sort()
    return times[len(times) // 2]


def make_plan(a, w, c, err, swiglu, force):
    if force:
        os.environ["SQ_GEMM_FORCE"] = force
    try:
        return ops.GemmPlan(a, w, c, err, swiglu=swiglu)
    finally:
        os.environ.pop("SQ_GEMM_FORCE", None)


def tile_candidates(N, K, swiglu):
    kb = K // 64
    out = []
    for bn in (64, 128, 192, 256):
        for split in (1, 2, 4):
            if kb % split or (split > 1 and (swiglu or bn > 128 or N % bn)):
                continue
            if split == 2:
                out.append((bn, 2, 1, 1))                    # split-K on the deep ring (gemm_tn_deep_kernel)
            for mc in (1, 2, 4):
                tiles = -(-N // bn)
                if tiles % mc:
                    continue
                out.append((bn, split, mc))
    return out


def measure_shapes(ns, copies, reps, sweep, only):
    dev = "cuda:0"
    err = torch.zeros(4, dtype=torch.int32, device=dev)
    rows = []
    for name, (N, K, swiglu) in SHAPES.items():
        if (only and name not in only) or (not only and name.endswith("_13b")):
            continue
        gen = torch.Generator(device=dev).manual_seed(0)
        a = (torch.randn(128, K, device=dev, generator=gen) * 0.5).half()
        ws = [(torch.randn(N, K, device=dev, generator=gen) * 0.02).half() for _ in range(copies)]
        nout = N // 2 if swiglu else N
        c = torch.zeros(128, N, device=dev, dtype=torch.float16)
        act = torch.zeros(128, nout, device=dev, dtype=torch.float16)
        wi = [ops.interleave_gate_up(w[:N // 2], w[N // 2:]) for w in ws] if swiglu else ws
        gb = N * K * 2 / 1e9
        ref = a.double() @ ws[0].double().t()
        if swiglu:
            g_, u_ = ref[:, :N // 2], ref[:, N // 2:]
            ref = g_ / (1 + torch.exp(-g_)) * u_
        scale = ref.abs().max().item()

        def cublas(i, n):
            torch.mm(a[:n], ws[i].t(), out=c[:n])
            if swiglu:
                ops.silu_mul(c, act, n)

        variants = [("default", None)]
        if sweep:
            variants += [(",".join(map(str, t)), ",".join(map(str, t))) for t in tile_candidates(N, K, swiglu)]
        plans = {}
        for label, force in variants:
            ps = [make_plan(a, w, act if swiglu else c, err, swiglu, force) for w in wi]
            info = ps[0].info()
            if force and (info[0], info[1], info[2] // 100) != tuple(int(x) for x in force.split(",")[:3]):
                continue                                         # the library rejected the forced tile
            plans[label] = ps
        for n in ns:
            out = act if swiglu else c
            res = {"projection": name, "N": N, "K": K, "n": n, "weight_GB": round(gb, 4)}
            t = graph_time_us(lambda i: cublas(i, n), copies, reps)
            cublas(0, n)
            torch.cuda.synchronize()
            e = (out[:n].double() - ref[:n]).abs().max().item() / scale
            res["cublas"] = dict(us=round(t, 2), GBs=round(gb / t * 1e6, 1), share=round(gb / t * 1e6 / HBM_PEAK_GBS, 3), rel_err=e)
            for label, ps in plans.items():
                t = graph_time_us(lambda i: ps[i].run(n), copies, reps)
                out.zero_()
                ps[0].run(n)
                torch.cuda.synchronize()
                e = (out[:n].double() - ref[:n]).abs().max().item() / scale
                bn, sp, st = ps[0].info()
                res["sq_gemm " + label] = dict(tile=f"bn={bn} split={sp} mc={st // 100} stages={st % 100}", us=round(t, 2),
                                               GBs=round(gb / t * 1e6, 1), share=round(gb / t * 1e6 / HBM_PEAK_GBS, 3),
                                               rel_err=e)
            rows.append(res)
            best = min((k for k in res if k.startswith("sq_gemm")), key=lambda k: res[k]["us"])
            print(f"{name:9s} n={n:3d} cuBLASLt {res['cublas']['us']:7.2f} us ({res['cublas']['GBs']:6.0f} GB/s "
                  f"{res['cublas']['share']:.0%})  sq_gemm default {res['sq_gemm default']['us']:7.2f} us "
                  f"({res['sq_gemm default']['GBs']:6.0f} GB/s, {res['sq_gemm default']['tile']})  best {best[8:]} "
                  f"{res[best]['us']:7.2f} us  err cublas {res['cublas']['rel_err']:.1e} sq {res['sq_gemm default']['rel_err']:.1e}",
                  flush=True)
            if sweep:
                for k in sorted((k for k in res if k.startswith("sq_gemm ")), key=lambda k: res[k]["us"]):
                    print(f"    {k[8:]:12s} {res[k]['tile']:34s} {res[k]['us']:7.2f} us {res[k]['GBs']:6.0f} GB/s", flush=True)
        if any(err.tolist()):
            raise RuntimeError(f"sq_gemm watchdog flag set: {err.tolist()}")
        del ws, wi, plans
        torch.cuda.empty_cache()
    return rows


def measure_layer(ns, reps, routes):
    """One 7B-shaped decoder layer per call (a 4-layer runner, so each layer's 405 MB of weights comes from HBM).  Also
    compares each route's logits (4 layers + lm_head, same inputs and cache) with the first route's."""
    from sequoia_b200 import model
    cfg = model.NAMED_CONFIGS["llama-2-7b"]
    model.NAMED_CONFIGS["llama-2-7b-4l"] = model.LlamaConfigLite(cfg.hidden_size, cfg.intermediate_size, 4,
                                                                 cfg.num_attention_heads, cfg.num_key_value_heads,
                                                                 rms_norm_eps=cfg.rms_norm_eps,
                                                                 max_position_embeddings=cfg.max_position_embeddings)
    M, P = 384, 128
    dev = "cuda:0"
    r = model.LlamaRunner("random-init:llama-2-7b-4l:2", max_length=M, device=dev)
    ids = torch.randint(0, 32000, (M,), device=dev)
    pos = torch.arange(M, device=dev)
    mask = torch.zeros(128, M, dtype=torch.float16, device=dev)
    out, first = [], {}
    for route in routes:
        restore = route_set(r, route)
        for n in ns:
            sto = torch.arange(P, P + n, device=dev)
            fn = lambda i: r.forward(n, ids, pos[P:P + n], sto, kv_end=P + n, dense_mask=mask, mask_ld=M, skip_lm_head=True)
            t = graph_time_us(fn, 1, reps) / r.L
            logits = r.forward(n, ids, pos[P:P + n], sto, kv_end=P + n, dense_mask=mask, mask_ld=M).double()
            ref = first.setdefault(n, logits.clone())
            d = ((logits - ref).abs().max() / ref.abs().max()).item()
            out.append({"route": route, "n": n, "us_per_layer": round(t, 2), "logit_rel_diff_vs_first_route": d})
            print(f"layer  route {route:40s} n={n:3d}  {t:8.2f} us per 7B layer   logits vs route {routes[0]}: "
                  f"max |diff| / max |logit| = {d:.2e}", flush=True)
        restore()
    if any(r.gemm_err.tolist()):
        raise RuntimeError(f"sq_gemm watchdog flag set: {r.gemm_err.tolist()}")
    return out


ROUTE_KEYS = {"gu": "wgu", "qkv": "wqkv", "o": "wo", "down": "wd"}


def route_set(r, route):
    """Install `route` (see the module docstring) on runner r; returns the function that puts the runner's own back."""
    from sequoia_b200 import ops
    if route == "model":
        return lambda: None
    saved = [{k: ly.pop(k) for k in list(ly) if k.endswith("_plan")} for ly in r.layers]
    io = dict(wqkv=(r.normed, r.qkv), wo=(r.attn_out, r.proj), wd=(r.act, r.proj))
    for part in ([] if route == "cublas" else route.split("+")):
        name, _, tile = part.partition("=")
        k = ROUTE_KEYS[name]
        for ly, s in zip(r.layers, saved):
            if k == "wgu":
                if "wgu_plan" not in s:
                    raise ValueError("the runner built no fused gate_up plan")
                ly["wgu_plan"] = s["wgu_plan"]
            else:
                ly[k + "_plan"] = make_plan(io[k][0], ly[k], io[k][1], r.gemm_err, False, tile.replace(":", ","))
                if tile and ly[k + "_plan"].info()[:2] != tuple(int(x) for x in tile.split(":")[:2]):
                    raise ValueError(f"tile {tile} refused for {k}")

    def restore():
        for ly, s in zip(r.layers, saved):
            for k in [k for k in ly if k.endswith("_plan")]:
                del ly[k]
            ly.update(s)
    return restore


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--n", default="128,97,127", help="row counts")
    ap.add_argument("--copies", type=int, default=6, help="weight copies cycled through (>= 6 keeps them out of L2)")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--only", default="", help="comma-separated projections")
    ap.add_argument("--sweep", action="store_true", help="also time every legal sq_gemm tile")
    ap.add_argument("--layer", action="store_true", help="also time a whole 7B layer on each route")
    ap.add_argument("--routes", default="cublas,model", help="comma-separated layer routes (see above)")
    ap.add_argument("--json", default=None, help="write the results here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("measure_verify_gemms: needs a CUDA device")
    ns = [int(x) for x in args.n.split(",")]
    info = card()
    print(info, flush=True)
    res = {"card": info, "shapes": measure_shapes(ns, max(args.copies, 6), args.reps, args.sweep,
                                                  [x for x in args.only.split(",") if x])}
    if args.layer:
        res["layer"] = measure_layer(ns, args.reps, args.routes.split(","))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
