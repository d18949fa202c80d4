"""The tensor-parallel all-reduce + residual + RMSNorm kernels and the driver -> follower message kernels of
csrc/sq_tp.cu on ONE GPU: every protocol at N = 2..8 ranks, the ranks emulated in sequence.

Emulation.  A peer is only a device pointer, so N emulated ranks are N blocks on one GPU, carved by peer.peer_layout
exactly as PeerBuffers carves its block; each rank also has its own resid and out.
* The ranks' kernels run one after another on one stream, in a chosen order.
* Forward traffic is real: whatever rank a's kernel writes for rank b, a running before b, stays as a wrote it and b
  consumes it.
* Backward traffic is pre-published by the host: whatever b needs from a rank that runs after it (flags, row flags and
  reduced rows, push slots and push flags, LL words) is written into b's block before the launches, from the
  restatement below, tagged with the epoch of this reduction.  The later rank then writes the same bytes again.
* Every case runs in order 0..N-1 and in order N-1..0, so between the two runs every directed (producer, consumer) pair
  is exercised for real.
* No rank is launched with an input unpublished, so no wait spins.  The watchdog word (epoch[2], the consume call's
  `err`) is read after every launch; a non-zero value fails the test at once.
Not covered: anything that needs two kernels running at the same time (NVLink ordering across GPUs, a reader racing a
writer, rejection of a stale word under a race).  test_gpu_tp.py runs the protocols across real GPUs.

Restatement.  x[r] = the fp16 rounding of the fp32 sum of the partials proj_s[r], s = 0..N-1 in rank order from +0.0;
resid' = fp16(resid + x).  Every byte of every emulated block is predicted after each launch: the blocks start from a
random fill (flag words from an epoch older than any used), and only the writes the protocol makes are applied, epoch
words included.  resid must be bit-identical to the restatement; out bit-identical to sq_add_rmsnorm(resid, x, w) for the
pulls and push (same element-to-thread mapping and expression as rmsnorm_kernel), and for LL (which sums the squares of
4-half pairs in another order) within the fp16-chain and float64 criteria of test_gpu_full_batch.  All ranks and all
protocols that the shapes allow must agree bit for bit."""
import ctypes as C

import pytest
import torch

from test_gpu_full_batch import ROW_KINDS, _norm_rows, _off_chain, _outside, _rms_f64, _rms_tol

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
F16, I32 = torch.float16, torch.int32
EPS = 1e-5
SENT = -7.0
FLAG_FILL = 0xA5A5A5A5            # older than every epoch used here under the kernels' signed comparison
E0 = 0xFFFFFFFE                   # first reductions cross the 2^32 wrap: e = 0xFFFFFFFF, 0, 1
TINY = 2.0 ** -15                 # below half the fp32 ulp of 2^10 (2^-13)
PULLS = ("one_shot", "two_shot")
PROTOS = ("one_shot", "two_shot", "push", "ll2", "ll1")     # ll2: LL two-shot, ll1: LL one-shot


def _lib():
    from sequoia_b200 import _lib as L
    return L


def _peer():
    from sequoia_b200 import peer
    return peer


def _i32(u):
    u &= 0xFFFFFFFF
    return u - (1 << 32) if u >= 1 << 31 else u


def _v(b, off, count, dtype):
    """`count` elements of `dtype` at byte `off` of block b (a view)."""
    isz = torch.empty(0, dtype=dtype).element_size()
    return b[off:off + count * isz].view(dtype)


def _bits(t):
    return t.contiguous().view(torch.int16)


def _llw(rows, e):
    """LL wire words of fp16 rows (m, hidden): per 4 halfs one 16-byte word (pair.lo, e, pair.hi, e)."""
    m, h = rows.shape
    u = rows.contiguous().view(I32).view(m, h // 4, 2)
    w = torch.empty(m, h // 4, 4, dtype=I32, device=DEV)
    w[..., 0], w[..., 2] = u[..., 0], u[..., 1]
    w[..., 1] = w[..., 3] = _i32(e)
    return w


def _fits(proto, hidden):
    if proto.startswith("ll"):
        return hidden % 4 == 0 and hidden <= 8192
    return hidden % 8 == 0 and hidden <= 16384


class World:
    """N emulated ranks: a block per rank on the production layout, its expected contents, resid / out per rank."""

    def __init__(self, N, n_max, hidden, ll_oneshot, seed):
        P = _peer()
        self.N, self.n_max, self.hidden = N, n_max, hidden
        self.L = L = P.peer_layout(N, n_max, hidden, ll_oneshot=ll_oneshot)
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.blk = [torch.randint(0, 256, (L.total,), dtype=torch.uint8, device=DEV, generator=g) for _ in range(N)]
        for b in self.blk:
            for off, nb in [(L.flags, P.FLAG_BYTES), (L.rowflags[0], L.rowflag_bytes), (L.rowflags[1], L.rowflag_bytes),
                            (L.pflags, L.pflag_bytes)]:
                _v(b, off, nb // 4, I32).fill_(_i32(FLAG_FILL))
            _v(b, L.epoch, 3, I32).copy_(torch.tensor([_i32(E0), 0, 0], dtype=I32))
        self.exp = [b.clone() for b in self.blk]
        self.w = (1 + 0.1 * torch.randn(hidden, generator=g, device=DEV)).to(F16)
        self.resid = [torch.empty(n_max + 1, hidden, dtype=F16, device=DEV) for _ in range(N)]
        self.out = [torch.empty(n_max + 1, hidden, dtype=F16, device=DEV) for _ in range(N)]

    def base(self, k):
        return self.blk[k].data_ptr()

    def peers(self, off):
        return (C.c_void_p * 8)(*[self.base(k) + off for k in range(self.N)] + [None] * (8 - self.N))

    def epoch(self, b):
        return _v(b, self.L.epoch, 3, I32)

    def proj(self, b, w):
        return _v(b, self.L.proj[w], self.n_max * self.hidden, F16).view(self.n_max, self.hidden)

    def ll1(self, b, w):
        L = self.L
        return _v(b, L.ll1[w], L.ll1_bytes // 4, I32).view(self.N, L.ll_own, self.hidden // 4, 4)

    def ll2(self, b, w):
        L = self.L
        return _v(b, L.ll2[w], L.ll2_bytes // 4, I32).view(L.push_rows, self.hidden // 4, 4)

    def next_epoch(self):
        eps = {int(self.epoch(b)[0]) & 0xFFFFFFFF for b in self.blk}
        assert len(eps) == 1, f"ranks at different epochs: {eps}"
        return (eps.pop() + 1) & 0xFFFFFFFF

    def diff(self):
        """[(rank, first differing region)] of blocks that differ from their expected contents."""
        ne = torch.stack([(a != b).any() for a, b in zip(self.blk, self.exp)]).tolist()
        bad = []
        for k, d in enumerate(ne):
            if d:
                i = int((self.blk[k] != self.exp[k]).nonzero()[0])
                name = [nm for nm, off, sz in self.L.regions() if off <= i < off + sz] or ["(padding)"]
                bad.append((k, name[0], i))
        return bad


def _writes(W, proto, k, w, n, e, P, X):
    """The restated writes of rank k's kernel: [(destination rank, fn(block), shared)]; `shared` marks the flag and push
    flag words, which buffers A and B share."""
    L, N, h = W.L, W.N, W.hidden
    ei = _i32(e)
    peers = [s for s in range(N) if s != k]
    out = []
    if proto in PULLS:
        out += [(s, lambda b: _v(b, L.flags, N, I32).__setitem__(k, ei), True) for s in peers]     # flags[s][rank]
    if proto == "two_shot" and k < n:
        def red(b):
            _v(b, L.red[w], W.n_max * h, F16).view(W.n_max, h)[k:n:N] = X[k:n:N]                 # red[s][r], r % N == k
            _v(b, L.rowflags[w], W.n_max, I32)[k:n:N] = ei                                         # rowflags[s][r]
        out += [(s, red, False) for s in peers]
    if proto == "push":
        rows = L.push_rows

        def push(b):
            _v(b, L.recv[w], N * rows * h, F16).view(N, rows, h)[k, :n] = P[k]                     # recv[s][rank][r]

        def pflag(b):
            _v(b, L.pflags, N * rows, I32).view(N, rows)[k, :n] = ei                               # pflags[s][rank][r]
        out += [(s, push, False) for s in peers] + [(s, pflag, True) for s in peers]
    if proto.startswith("ll"):
        if L.ll_oneshot:
            words = _llw(P[k], e)
            out += [(s, lambda b: W.ll1(b, w)[k, :n].copy_(words), False) for s in peers]          # ll1[s][rank][r]
        else:
            for o in peers:                                                                        # ll1[owner][rank][r/N]
                if o < n:
                    words = _llw(P[k][o:n:N], e)
                    out.append((o, lambda b, words=words: W.ll1(b, w)[k, :words.shape[0]].copy_(words), False))
            if k < n:
                red_words = _llw(X[k:n:N], e)
                out += [(s, lambda b: W.ll2(b, w)[k:n:N].copy_(red_words), False) for s in peers]  # ll2[s][r]
    return out


def _launch(W, proto, k, w, n):
    lb, L, N, h = _lib().load(), W.L, W.N, W.hidden
    resid, out, wt = W.resid[k].data_ptr(), W.out[k].data_ptr(), W.w.data_ptr()
    ep, st = W.base(k) + L.epoch, torch.cuda.current_stream().cuda_stream
    local = W.base(k) + L.proj[w]
    if proto == "one_shot":
        rc = lb.sq_tp_allreduce_add_rmsnorm(resid, W.peers(L.proj[w]), W.peers(L.flags), ep, k, N, wt, out, n, h, EPS, st)
    elif proto == "two_shot":
        rc = lb.sq_tp_allreduce2_add_rmsnorm(resid, W.peers(L.proj[w]), W.peers(L.red[w]), W.peers(L.flags),
                                             W.peers(L.rowflags[w]), ep, k, N, wt, out, n, h, EPS, st)
    elif proto == "push":
        rc = lb.sq_tp_allreduce3_add_rmsnorm(resid, local, W.peers(L.recv[w]), W.peers(L.pflags), ep, k, N, L.push_rows,
                                             wt, out, n, h, EPS, st)
    else:
        assert L.ll_oneshot == (proto == "ll1")
        rc = lb.sq_tp_allreduce_ll_add_rmsnorm(resid, local, W.peers(L.ll1[w]), W.peers(L.ll2[w]), ep, k, N, L.push_rows,
                                               L.ll_own, wt, out, n, h, EPS, st)
    assert rc == 0, _lib().load().sq_last_error()


def _restate(P, resid_in, order=None, drop=None):
    """x = fp16(fp32 sum of the partials in `order` from +0.0), resid' = fp16(resid + x)."""
    acc = torch.zeros(P[0].shape, dtype=torch.float32, device=DEV)
    for s in (order if order is not None else range(len(P))):
        if s != drop:
            acc = acc + P[s].float()
    x = acc.to(F16)
    return x, (resid_in.float() + x.float()).to(F16)


def _sens_cols(hidden):
    return torch.arange(3, hidden, 8, device=DEV)


def _data(N, hidden, n, step, seed):
    """Replicated residual rows of every ROW_KINDS kind and N partials; every 8th column is order-sensitive: +2^10 at
    rank a, -2^10 at rank b, 2^-15 at the others, (a, b) cycling over the columns."""
    g = torch.Generator(device=DEV).manual_seed(seed * 1000 + n * 10 + step)
    resid_in, _ = _norm_rows(n, hidden, g, False)
    P = [(0.5 * torch.randn(n, hidden, generator=g, device=DEV)).to(F16) for _ in range(N)]
    cols = _sens_cols(hidden)
    i = torch.arange(len(cols))
    a = i % N
    b = (a + 1 + (i // N) % (N - 1)) % N
    for s in range(N):
        pat = torch.full((len(cols),), TINY)
        pat[a == s], pat[b == s] = 1024.0, -1024.0
        P[s][:, cols] = pat.to(F16).to(DEV)
    return resid_in, P


def _reduce(W, proto, w, n, resid_in, P, order, want):
    """One reduction on buffer w: pre-publish the backward traffic, launch the ranks in `order`, check every block, the
    watchdog word, resid and out after each launch.  Returns (resid, out) of the ranks (identical)."""
    N, h = W.N, W.hidden
    e = W.next_epoch()
    x, R, out_ref = want
    for k in range(N):                                   # the row-parallel GEMM outputs and the replicated residual stream
        for blks in (W.blk, W.exp):
            W.proj(blks[k], w)[:n] = P[k]
        W.resid[k].fill_(SENT)
        W.resid[k][:n] = resid_in
        W.out[k].fill_(SENT)
    pos = {k: i for i, k in enumerate(order)}
    writes = {k: _writes(W, proto, k, w, n, e, P, x) for k in range(N)}
    for k in range(N):
        for dst, fn, _ in writes[k]:
            if dst != k and pos[k] > pos[dst]:           # backward: rank dst runs first and needs it
                fn(W.blk[dst])
                fn(W.exp[dst])
    sent = _bits(torch.full((1, h), SENT, dtype=F16, device=DEV))
    first = None
    for k in order:
        _launch(W, proto, k, w, n)
        err = int(W.epoch(W.blk[k])[2])
        assert err == 0, f"{proto} N={N} rank {k} n={n}: watchdog word {err}"
        for dst, fn, _ in writes[k]:
            fn(W.exp[dst])
        W.epoch(W.exp[k]).copy_(torch.tensor([_i32(e), 0, 0], dtype=I32))
        bad = W.diff()
        assert not bad, f"{proto} N={N} rank {k} n={n} e={e:#x}: blocks differ from the restatement at {bad}"
        got_r, got_o = W.resid[k][:n], W.out[k][:n]
        assert torch.equal(_bits(got_r), _bits(R)), f"{proto} N={N} rank {k} n={n}: resid differs from the restatement"
        assert bool((_bits(W.resid[k][n:]) == sent).all() & (_bits(W.out[k][n:]) == sent).all()), "row >= n written"
        if first is None:
            if proto.startswith("ll"):
                assert bool(torch.isfinite(got_o).all())
                assert _off_chain(got_o, R, W.w, EPS) == 0, f"{proto} N={N} n={n}: out off the fp16 chain"
                exact = _rms_f64(R, W.w, EPS)
                assert _outside(got_o, exact, _rms_tol(exact, W.w, h)) == 0, f"{proto} N={N} n={n}: outside float64 bound"
            else:
                assert torch.equal(_bits(got_o), _bits(out_ref)), f"{proto} N={N} rank {k} n={n}: out != sq_add_rmsnorm"
            first = (got_r.clone(), got_o.clone())
        else:
            assert torch.equal(_bits(got_r), _bits(first[0])) and torch.equal(_bits(got_o), _bits(first[1])), \
                f"{proto} N={N} rank {k} n={n}: ranks diverge"
    return first


def _want(W, resid_in, P, n):
    from sequoia_b200 import ops
    x, R = _restate(P, resid_in)
    if W.hidden % 8:                                     # LL-only width: sq_add_rmsnorm holds multiples of 8
        return x, R, None
    r2 = resid_in.clone()
    out_ref = torch.empty(n, W.hidden, dtype=F16, device=DEV)
    ops.add_rmsnorm(r2, x, W.w, out_ref, n, EPS)
    assert torch.equal(_bits(r2), _bits(R))
    return x, R, out_ref


# (N, hidden): every protocol at every N, every MAXV (pull / push: 2048 -> 1, 2056 / 4096 -> 2, 4104 / 5120 / 8192 -> 4,
# 8200 / 16384 -> 8) and MAXP (LL: 1024 -> 1, 1028 / 2048 -> 2, 2052 / 2056 / 4096 -> 4, 4100 / 4104 / 5120 / 8192 -> 8)
WORLDS = [(2, 2048), (2, 1028), (3, 2056), (3, 2052), (4, 4096), (4, 4100), (5, 4104), (5, 1024), (6, 8192), (6, 5120),
          (7, 8200), (7, 2048), (8, 16384), (8, 8192)]


def _n_values(N, hidden):
    ns = sorted({1, N - 1, N + 1, 127, 256})
    return ns + [768] if (N, hidden) == (8, 8192) else ns     # 768 x 8192: config 4's verify (the two pulls)


def _protos(N, hidden, n):
    ps = [p for p in PROTOS if _fits(p, hidden) and (n <= 256 or p in PULLS)]
    lead = PULLS[N % 2]                                        # the world's first reductions cross the epoch wrap
    return sorted(ps, key=lambda p: p != lead)


@pytest.mark.parametrize("N,hidden", WORLDS, ids=[f"N{N}-h{h}" for N, h in WORLDS])
def test_allreduce_protocols_emulated(N, hidden):
    """Every protocol the shapes allow at n = 1, N-1, N+1, 127, 256 (and 768 at config 4's width for the pulls), three
    reductions each on buffers A, B, A, in both launch orders; resid / out identical across protocols, orders and ranks."""
    n_max = 768 if (N, hidden) == (8, 8192) else 256
    results, ran, data = {}, set(), {}
    for oneshot in (N <= 3, N > 3):                            # the production LL form first, then the other one
        W = World(N, n_max, hidden, oneshot, seed=N * 100000 + hidden)
        for n in _n_values(N, hidden):
            for proto in _protos(N, hidden, n):
                if proto.startswith("ll") and (proto == "ll1") != W.L.ll_oneshot:
                    continue
                if oneshot != (N <= 3) and not proto.startswith("ll"):
                    continue
                ran.add(proto)
                for order in (list(range(N)), list(range(N - 1, -1, -1))):
                    for step, w in enumerate((0, 1, 0)):
                        if (n, step) not in data:
                            resid_in, P = _data(N, hidden, n, step, seed=N + hidden)
                            data[n, step] = resid_in, P, _want(W, resid_in, P, n)
                        resid_in, P, want = data[n, step]
                        got = _reduce(W, proto, w, n, resid_in, P, order, want)
                        key = (n, step)
                        if key not in results:
                            results[key] = (proto, got)
                        else:
                            p0, (r0, o0) = results[key]
                            assert torch.equal(_bits(got[0]), _bits(r0)), f"resid of {proto} != {p0} at n={n}"
                            if not proto.startswith("ll") and not p0.startswith("ll"):
                                assert torch.equal(_bits(got[1]), _bits(o0)), f"out of {proto} != {p0} at n={n}"
        del W
        torch.cuda.empty_cache()
    assert ran == {p for p in PROTOS if _fits(p, hidden)}


def test_order_sensitive_columns_see_rank_order():
    """The order-sensitive columns change x under a reversed-order sum at every N >= 3 (two fp32 addends commute)."""
    for N in range(3, 9):
        resid_in, P = _data(N, 4096, 5, 0, seed=1)
        cols = _sens_cols(4096)
        x, _ = _restate(P, resid_in)
        xr, _ = _restate(P, resid_in, order=range(N - 1, -1, -1))
        assert bool((_bits(x[:, cols]) != _bits(xr[:, cols])).any(dim=1).all()), N


@pytest.mark.parametrize("proto", ["two_shot", "ll2"])
def test_negative_controls(proto):
    """The comparisons that the kernels pass fail for a restatement that sums in reversed rank order, drops one rank's
    partial, or takes a peer's row r+1 for row r, and the block comparison fails for an LL word with a stale tag."""
    N, hidden, n = 4, 4096, 10
    W = World(N, 256, hidden, False, seed=7)
    resid_in, P = _data(N, hidden, n, 0, seed=7)
    got_r, _ = _reduce(W, proto, 0, n, resid_in, P, list(range(N)), _want(W, resid_in, P, n))
    zero = [r for r in range(n) if ROW_KINDS[r % len(ROW_KINDS)] == "zero"]
    cols = _sens_cols(hidden)
    _, rev = _restate(P, resid_in, order=range(N - 1, -1, -1))
    assert not torch.equal(_bits(rev[zero][:, cols]), _bits(got_r[zero][:, cols])), "reversed rank order not seen"
    _, dropped = _restate(P, resid_in, drop=2)
    assert not torch.equal(_bits(dropped), _bits(got_r)), "a dropped partial not seen"
    shifted = [p.clone() for p in P]
    shifted[1][:-1] = P[1][1:]
    _, sh = _restate(shifted, resid_in)
    assert not torch.equal(_bits(sh[:-1]), _bits(got_r[:-1])), "a shifted peer row not seen"
    if proto == "ll2":
        # rank 1's gather slot from rank 0 (row 1) holds a word tagged with this epoch; a stale tag must be seen
        tag = W.ll1(W.exp[1], 0)[0, 0, 0, 1]
        assert int(tag) == _i32(W.next_epoch() - 1)
        tag -= 2
        assert W.diff() and W.diff()[0][:2] == (1, "ll1_a")
        tag += 2
        assert not W.diff()


@pytest.mark.parametrize("proto,N", [("one_shot", 3), ("two_shot", 5), ("push", 4), ("ll2", 6), ("ll1", 2)])
def test_graph_replay_matches_eager(proto, N):
    """The N ranks' launches on A and then B captured as one CUDA graph, replayed three times with new partials, each
    replay bit-identical (blocks, resid, out) to the eager launches on the same data.  The backward traffic of each replay
    is pre-published from the device epoch before it.  Flags and push flags are shared by A and B, so A's launches would
    overwrite B's pre-published ones: the graph re-publishes those from a staging buffer with one copy just before each
    rank's B launch (no copies for LL, whose areas are all per buffer)."""
    hidden, n = 4096, 37
    order = list(range(N))
    oneshot = proto == "ll1"
    WE, WG = (World(N, 64, hidden, oneshot, seed=11) for _ in range(2))
    L = WG.L
    shared = proto in PULLS or proto == "push"
    stage = torch.zeros(N, N, L.push_rows, dtype=I32, device=DEV)     # [consumer][source][row] flag words for B

    def flag_view(b):
        return (_v(b, L.flags, N, I32).view(N, 1) if proto in PULLS
                else _v(b, L.pflags, N * L.push_rows, I32).view(N, L.push_rows))

    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            for k in order:
                _launch(WG, proto, k, 0, n)
            for k in order:
                if shared:
                    cols = 1 if proto in PULLS else n
                    flag_view(WG.blk[k])[k + 1:, :cols].copy_(stage[k, k + 1:, :cols])
                _launch(WG, proto, k, 1, n)
    torch.cuda.current_stream().wait_stream(side)
    for rep in range(3):
        data = [_data(N, hidden, n, 10 * rep + w, seed=11) for w in range(2)]
        # eager, fully checked launch by launch
        resid_in, P = data[0]
        wa = _want(WE, resid_in, P, n)
        ra, _ = _reduce(WE, proto, 0, n, resid_in, P, order, wa)
        wb = _want(WE, ra, data[1][1], n)
        _reduce(WE, proto, 1, n, ra, data[1][1], order, wb)
        # the same data through the graph
        e = WG.next_epoch()
        for k in range(N):
            for w in range(2):
                WG.proj(WG.blk[k], w)[:n] = data[w][1][k]
            WG.resid[k].fill_(SENT)
            WG.resid[k][:n] = resid_in
            WG.out[k].fill_(SENT)
        stage.zero_()
        for w, (ew, xw) in enumerate(((e, wa[0]), ((e + 1) & 0xFFFFFFFF, wb[0]))):
            for k in range(N):
                for dst, fn, sh in _writes(WG, proto, k, w, n, ew, data[w][1], xw):
                    if dst < k:                                        # backward in order 0..N-1
                        if w == 1 and sh:
                            stage[dst, k, :n if proto == "push" else 1] = _i32(ew)
                        else:
                            fn(WG.blk[dst])
        g.replay()
        torch.cuda.synchronize()
        for k in range(N):
            err = int(WG.epoch(WG.blk[k])[2])
            assert err == 0, f"graph replay {rep}, rank {k}: watchdog word {err}"
        for k in range(N):
            assert torch.equal(WG.blk[k], WE.blk[k]), f"replay {rep}: block of rank {k} differs from the eager run"
            assert torch.equal(_bits(WG.resid[k]), _bits(WE.resid[k])) and torch.equal(_bits(WG.out[k]), _bits(WE.out[k]))
    del g


# ------------------------------------------------------------------------------------------------ messages
def _msg_segments(cap, g):
    sets = [(0, 1, 255), (256, 257, 0), (257, 0, 256), (cap - 513, 256, 257)]
    segs = [[torch.randint(-2 ** 31, 2 ** 31 - 1, (c,), dtype=I32, device=DEV, generator=g) for c in s] for s in sets]
    M = 1024                                              # the real message: int64 tokens and position ids, 16 state words
    segs.append([torch.randint(0, 128256, (M,), dtype=torch.int64, device=DEV, generator=g),
                 torch.arange(M, dtype=torch.int64, device=DEV) + 4000,
                 torch.randint(-2 ** 31, 2 ** 31 - 1, (16,), dtype=I32, device=DEV, generator=g)])
    return segs


@pytest.mark.parametrize("n_peers", range(1, 8))
def test_ll_messages(n_peers):
    """sq_tp_ll_publish to n_peers mailboxes then sq_tp_ll_consume on each, epochs 1..4 per message shape: dst equals src
    bit for bit, each mailbox holds (word, e) in half e & 1 and nothing else changed, consumer sentinels past each
    segment are untouched, both epoch counters advanced and err == 0."""
    from sequoia_b200.peer import MBOX_WORDS as cap
    lb = _lib().load()
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device=DEV).manual_seed(n_peers)
    guard = 64
    box = torch.randint(-2 ** 31, 2 ** 31 - 1, (n_peers, 4 * cap + guard), dtype=I32, device=DEV, generator=g)
    exp_box = box.clone()
    boxes = (C.c_void_p * 8)(*[box[p].data_ptr() for p in range(n_peers)] + [None] * (8 - n_peers))
    for segs in _msg_segments(cap, g):
        words = [t.numel() * t.element_size() // 4 for t in segs]
        assert sum(words) <= cap
        src = torch.cat([t.view(I32) for t in segs]) if sum(words) else torch.empty(0, dtype=I32, device=DEV)
        ep_drv = torch.zeros(1, dtype=I32, device=DEV)
        ep_f = torch.zeros(n_peers, 4, dtype=I32, device=DEV)          # [peer]: epoch, err
        for e in range(1, 5):
            before = [t.clone() for t in segs]
            a = [(t.data_ptr() if t.numel() else None, c) for t, c in zip(segs, words)]
            rc = lb.sq_tp_ll_publish(boxes, n_peers, cap, ep_drv.data_ptr(), a[0][0], a[0][1], a[1][0], a[1][1], a[2][0],
                                     a[2][1], st)
            assert rc == 0
            half = (e & 1) * cap
            mb = exp_box[:, :4 * cap].view(n_peers, 2 * cap, 2)
            mb[:, half:half + len(src), 0] = src
            mb[:, half:half + len(src), 1] = e
            assert torch.equal(box, exp_box), (words, e)
            assert int(ep_drv[0]) == e
            assert all(torch.equal(x, y) for x, y in zip(segs, before)), "publish changed its source"
            for p in range(n_peers):
                dst = [torch.full((c + 8,), -0x5A5A5A5B, dtype=I32, device=DEV) for c in words]
                rc = lb.sq_tp_ll_consume(box[p].data_ptr(), cap, ep_f[p].data_ptr(), ep_f[p, 1:].data_ptr(),
                                         dst[0].data_ptr(), words[0], dst[1].data_ptr(), words[1], dst[2].data_ptr(),
                                         words[2], st)
                assert rc == 0
                assert int(ep_f[p, 1]) == 0, f"consume watchdog {int(ep_f[p, 1])}"
                assert int(ep_f[p, 0]) == e
                for t, d, c in zip(segs, dst, words):
                    assert torch.equal(d[:c], t.view(I32)), (words, e, p)
                    assert bool((d[c:] == -0x5A5A5A5B).all()), "consumer wrote past its segment"
            assert torch.equal(box, exp_box), "consume changed a mailbox"


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals():
    """Arguments outside what the kernels hold return SQ_ERR_INVALID_ARG before any launch."""
    L = _lib()
    lb = L.load()
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    p = buf.data_ptr()
    arr = (C.c_void_p * 8)(*[p] * 8)
    st = torch.cuda.current_stream().cuda_stream
    calls = []
    for N, rank, h in [(1, 0, 4096), (9, 0, 4096), (4, -1, 4096), (4, 4, 4096), (4, 0, 4100), (4, 0, 16392)]:
        calls += [lambda N=N, rank=rank, h=h: lb.sq_tp_allreduce_add_rmsnorm(p, arr, arr, p, rank, N, p, p, 1, h, EPS, st),
                  lambda N=N, rank=rank, h=h: lb.sq_tp_allreduce2_add_rmsnorm(p, arr, arr, arr, arr, p, rank, N, p, p, 1, h,
                                                                              EPS, st),
                  lambda N=N, rank=rank, h=h: lb.sq_tp_allreduce3_add_rmsnorm(p, p, arr, arr, p, rank, N, 8, p, p, 1, h, EPS,
                                                                              st)]
    for N, rank, h in [(1, 0, 4096), (9, 0, 4096), (4, -1, 4096), (4, 4, 4096), (4, 0, 1026), (4, 0, 8196)]:
        calls.append(lambda N=N, rank=rank, h=h: lb.sq_tp_allreduce_ll_add_rmsnorm(p, p, arr, arr, p, rank, N, 8, 2, p, p, 1,
                                                                                   h, EPS, st))
    calls += [lambda: lb.sq_tp_allreduce3_add_rmsnorm(p, p, arr, arr, p, 0, 4, 8, p, p, 9, 4096, EPS, st),        # n > rows
              lambda: lb.sq_tp_allreduce_ll_add_rmsnorm(p, p, arr, arr, p, 0, 4, 8, 8, p, p, 9, 4096, EPS, st),   # one-shot
              lambda: lb.sq_tp_allreduce_ll_add_rmsnorm(p, p, arr, arr, p, 0, 4, 256, 10, p, p, 41, 4096, EPS, st)]
    cap = 64
    calls += [lambda: lb.sq_tp_ll_publish(arr, 2, cap, p, p, 30, p, 30, p, 5, st),
              lambda: lb.sq_tp_ll_publish(arr, 0, cap, p, p, 1, None, 0, None, 0, st),
              lambda: lb.sq_tp_ll_publish(arr, 8, cap, p, p, 1, None, 0, None, 0, st),
              lambda: lb.sq_tp_ll_publish(arr, 2, cap, p, p, -1, None, 0, None, 0, st),
              lambda: lb.sq_tp_ll_consume(p, cap, p, p, p, 64, p, 1, None, 0, st),
              lambda: lb.sq_tp_ll_consume(p, cap, p, p, p, -1, None, 0, None, 0, st)]
    for i, call in enumerate(calls):
        before = L.launch_count()
        assert call() == -1, i
        assert L.launch_count() == before, i
    # the edges themselves are accepted (not launched here: n = 0 returns before any launch)
    assert lb.sq_tp_allreduce_add_rmsnorm(p, arr, arr, p, 7, 8, p, p, 0, 16384, EPS, st) == 0
    assert lb.sq_tp_allreduce_ll_add_rmsnorm(p, p, arr, arr, p, 0, 4, 256, 64, p, p, 0, 8192, EPS, st) == 0
    torch.cuda.synchronize()
