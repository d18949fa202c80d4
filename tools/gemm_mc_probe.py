"""Where the 2-CTA activation multicast of sq_gemm loses its time: each tile against the same tile without multicast.

Compiles csrc/sq_gemm.cu once more with -DSQ_GEMM_STAMPS into a probe library in a temporary directory (the library
proper never defines that macro: its kernels are untouched).  For each (N, K, tile) it reports
  * cudaOccupancyMaxActiveClusters of the (MC, SPLIT) cluster at the instance's shared-memory size, against the
    clusters the grid needs: fewer means a second wave;
  * the device time per call (CUDA graph cycling over 6 weight copies, so the weights come from HBM);
  * from one stamped run, per CTA %globaltimer at the first TMA issue, the first and the last full ring slot, and the
    exit: how late CTAs start (launch skew), how long the first slot takes to land, the k-loop, and the tail;
    plus how many distinct SMs the CTAs ran on.

    python tools/gemm_mc_probe.py [--json out.json]

Prints the card and its power limit first.  Needs a GPU and nvcc."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from sequoia_b200 import _lib  # noqa: E402
from measure_verify_gemms import card, graph_time_us  # noqa: E402

CSRC = os.path.join(ROOT, "sequoia_b200", "csrc")
# (label, N, K, tiles): the 7B verify shapes whose picked tile used multicast, and gate_up at BN 256 where it can;
# "bn,2,1,1" is the split-K tile on the deep ring (gemm_tn_deep_kernel)
CASES = [
    ("qkv", 12288, 4096, ["128,1,2", "128,1,1"]),
    ("o_proj", 4096, 4096, ["128,4,2", "128,4,1", "64,2,2", "64,2,1", "64,2,1,1"]),
    ("down_proj", 4096, 11008, ["128,4,2", "128,4,1", "64,2,1", "64,2,1,1"]),
    ("gate_up@256", 22016 - 22016 % 512, 4096, ["256,1,2", "256,1,1"]),
]


def build_probe(out_dir):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    so = os.path.join(out_dir, "libsq_gemm_probe.so")
    subprocess.run([nvcc, "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a",
                    "--expt-relaxed-constexpr", "-DSQ_GEMM_STAMPS", "-shared", "-o", so,
                    os.path.join(CSRC, "sq_gemm.cu"), os.path.join(CSRC, "sq_capi.cu"), "-lcudart"], check=True)
    lib = C.CDLL(so)
    for name, (res, args) in _lib._SIGNATURES.items():
        if name.startswith("sq_gemm_") and not name.startswith("sq_gemm_fp8") or name == "sq_last_error":
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    lib.sq_gemm_probe_set_stamps.restype, lib.sq_gemm_probe_set_stamps.argtypes = C.c_int, [C.c_void_p, C.c_void_p]
    lib.sq_gemm_probe_max_clusters.restype = C.c_int
    lib.sq_gemm_probe_max_clusters.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    return lib


def check(lib, rc, what):
    if rc != 0:
        raise RuntimeError(f"{what}: {lib.sq_last_error().decode()}")


def plan(lib, a, w, c, err, force):
    os.environ["SQ_GEMM_FORCE"] = force
    try:
        h = C.c_void_p()
        check(lib, lib.sq_gemm_plan_create_ex(C.byref(h), a.data_ptr(), a.stride(0), a.shape[0], w.data_ptr(), w.shape[0],
                                              w.shape[1], c.data_ptr(), c.stride(0), err.data_ptr(), 0), "plan")
    finally:
        os.environ.pop("SQ_GEMM_FORCE")
    bn, sp, st = C.c_int(), C.c_int(), C.c_int()
    lib.sq_gemm_plan_info(h, C.byref(bn), C.byref(sp), C.byref(st))
    if (bn.value, sp.value, st.value // 100) != tuple(int(x) for x in force.split(",")[:3]):
        raise RuntimeError(f"tile {force} refused for N={w.shape[0]} K={w.shape[1]}")
    return h


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(q * len(xs)))]


def probe_case(lib, label, N, K, force, copies=6, reps=7):
    dev = "cuda:0"
    g = torch.Generator(device=dev).manual_seed(0)
    a = (torch.randn(128, K, device=dev, generator=g) * 0.5).half()
    ws = [(torch.randn(N, K, device=dev, generator=g) * 0.02).half() for _ in range(copies)]
    c = torch.zeros(128, N, device=dev, dtype=torch.float16)
    err = torch.zeros(4, dtype=torch.int32, device=dev)
    hs = [plan(lib, a, w, c, err, force) for w in ws]
    bn, split, mc = (int(x) for x in force.split(",")[:3])
    ctas = -(-N // bn) * split
    mx = C.c_int()
    check(lib, lib.sq_gemm_probe_max_clusters(hs[0], C.byref(mx)), "max clusters")
    stream = lambda: torch.cuda.current_stream().cuda_stream
    t = graph_time_us(lambda i: check(lib, lib.sq_gemm_run(hs[i], 128, C.c_void_p(stream())), "run"), copies, reps)
    ref = a.double() @ ws[1].double().t()
    stamps = torch.zeros(ctas * 5, dtype=torch.int64, device=dev)
    lib.sq_gemm_probe_set_stamps(hs[1], stamps.data_ptr())
    check(lib, lib.sq_gemm_run(hs[0], 128, C.c_void_p(stream())), "run")     # another copy first: weights of hs[1] cold
    torch.cuda.synchronize()                                                   # and no launch overlapping the stamped one
    check(lib, lib.sq_gemm_run(hs[1], 128, C.c_void_p(stream())), "run")
    torch.cuda.synchronize()
    rel = ((c.double() - ref).abs().max() / ref.abs().max()).item()
    s = stamps.view(ctas, 5).cpu().tolist()
    t0 = min(r[1] for r in s)
    start = [(r[1] - t0) / 1e3 for r in s]
    first = [(r[2] - r[1]) / 1e3 for r in s]
    loop = [(r[3] - r[2]) / 1e3 for r in s]
    tail = [(r[4] - r[3]) / 1e3 for r in s]
    span = (max(r[4] for r in s) - t0) / 1e3
    res = dict(label=label, N=N, K=K, tile=force, ctas=ctas, clusters=ctas // (mc * split), max_active_clusters=mx.value,
               us=round(t, 2), GBs=round(N * K * 2 / t / 1e3, 1), stamped_span_us=round(span, 2),
               distinct_sms=len({r[0] for r in s}), rel_err=rel, watchdog=err.tolist())
    for name, xs in (("start", start), ("first_slot", first), ("k_loop", loop), ("tail", tail)):
        res[name + "_us"] = [round(pct(xs, q), 2) for q in (0.0, 0.5, 0.9, 1.0)]
    for h in hs:
        lib.sq_gemm_plan_destroy(h)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--json", default=None, help="write the results here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_mc_probe: needs a CUDA device")
    print(card(), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_probe(tmp)
        out = []
        for label, N, K, tiles in CASES:
            for force in tiles:
                r = probe_case(lib, label, N, K, force)
                out.append(r)
                print(f"{label:12s} tile {force:8s} ctas {r['ctas']:3d} clusters {r['clusters']:3d} (max active "
                      f"{r['max_active_clusters']:3d}) sms {r['distinct_sms']:3d}  {r['us']:7.2f} us {r['GBs']:6.0f} GB/s  "
                      f"stamped span {r['stamped_span_us']:7.2f} us  start {r['start_us']}  first slot {r['first_slot_us']}"
                      f"  k-loop {r['k_loop_us']}  tail {r['tail_us']}  (min/med/p90/max)  err {r['rel_err']:.1e}"
                      f" wd {r['watchdog']}", flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
