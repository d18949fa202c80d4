"""N > 1 host logic on CPU (gloo, world_size 2): Megatron sharding arithmetic of the target weights and the
driver / follower control protocol of sequoia_b200.tp (the CUDA kernels themselves need a GPU and are stubbed)."""
import os
import socket
import sys
import types

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _init(rank, world, port):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)


def _shard_worker(rank, world, port, q):
    import cases
    from sequoia_b200.model import _DictSource, config_from, load_sharded_weights
    _init(rank, world, port)
    cfg_o, w = cases.model_weights("target_gqa")                # H=4, Hkv=2 -> 2 ranks: 2 q heads + 1 kv head each
    cfg = config_from(cfg_o)
    src = _DictSource({k: v.float() for k, v in w.items()}, "cpu")
    src.get = lambda name, shape, _s=src: _s.sd[name]            # keep fp32 on CPU for an exact comparison
    full = load_sharded_weights(cfg, src, 0, 1)["layers"][0]
    mine = load_sharded_weights(cfg, src, rank, world)["layers"][0]
    g = torch.Generator().manual_seed(3)
    x = torch.randn(5, cfg.hidden_size, generator=g)
    D, H, Hkv, I = cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.intermediate_size
    # column-parallel qkv: my rows are the matching slices of the full projection
    qkv_full = x @ full["wqkv"].t()
    qkv_mine = x @ mine["wqkv"].t()
    h2, k2 = H // world, Hkv // world
    exp = torch.cat([qkv_full[:, rank * h2 * D:(rank + 1) * h2 * D],
                     qkv_full[:, H * D + rank * k2 * D: H * D + (rank + 1) * k2 * D],
                     qkv_full[:, (H + Hkv) * D + rank * k2 * D:(H + Hkv) * D + (rank + 1) * k2 * D]], dim=1)
    ok = torch.allclose(qkv_mine, exp, atol=1e-5)
    # row-parallel o_proj / down_proj: partial products summed by the allreduce equal the full product
    a_full = torch.randn(5, H * D, generator=g)
    part = a_full[:, rank * h2 * D:(rank + 1) * h2 * D] @ mine["wo"].t()
    dist.all_reduce(part)
    ok &= torch.allclose(part, a_full @ full["wo"].t(), atol=1e-4)
    gu_full = x @ full["wgu"].t()
    act_full = torch.nn.functional.silu(gu_full[:, :I]) * gu_full[:, I:]
    gu = x @ mine["wgu"].t()
    Ir = I // world
    act = torch.nn.functional.silu(gu[:, :Ir]) * gu[:, Ir:]
    ok &= torch.allclose(act, act_full[:, rank * Ir:(rank + 1) * Ir], atol=1e-5)
    down = act @ mine["wd"].t()
    dist.all_reduce(down)
    ok &= torch.allclose(down, act_full @ full["wd"].t(), atol=1e-4)
    q.put((rank, bool(ok)))
    dist.destroy_process_group()


def test_megatron_sharding_math_gloo():
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_shard_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in range(2))
    [p.join(60) for p in procs]
    assert res == [(0, True), (1, True)]


class _StubEngine:
    """Records what a follower rank would run on its target shard."""

    def __init__(self, log):
        self.log = log
        outer = self

        class _Runner:
            def forward(self, n, tokens, position_ids, storage_ids, **kw):
                outer.log.append(("forward", n, int(tokens[:4].sum()), kw.get("n0"), kw.get("kv_end"),
                                  kw.get("prefix_len", 0), kw.get("skip_lm_head")))

        class _KV:
            def gather_from_state(self, idx, state, max_n, zero_tail=False):
                outer.log.append(("gather", int(state[3]), int(state[4]), idx[:2].tolist()))

        self.engine = types.SimpleNamespace(runner=_Runner(), kv_cache=_KV())

    def clear_kv(self):
        self.log.append(("clear",))


def _proto_worker(rank, world, port, q):
    import cases
    from sequoia_b200 import tp
    _init(rank, world, port)
    gm = cases.load_growmap("L40_growmaps/8x8-tree.pt")
    S, M = gm["size"], 256
    if rank == 0:
        drv = tp.TPDriver(dist.group.WORLD, "cpu")
        rt = types.SimpleNamespace(tokens=torch.arange(M), position_ids=torch.arange(M), state=torch.zeros(16, dtype=torch.int32),
                                   accept_idx=torch.zeros(S, dtype=torch.int32))
        drv.send_ctrl(tp.OP_CLEAR)
        rt.state[0] = 100
        drv.send_ctrl(tp.OP_FIRST, 0, 100)
        drv.bcast_inputs(rt)
        rt.state[3], rt.state[4] = 2, 100
        rt.accept_idx[:2] = torch.tensor([101, 109], dtype=torch.int32)
        drv.bcast_accept(rt)
        for step in range(2):
            rt.tokens += 1
            drv.send_ctrl(tp.OP_STEADY)
            drv.bcast_inputs(rt)
            rt.state[3], rt.state[4] = step, 103 + step
            drv.bcast_accept(rt)
        drv.send_ctrl(tp.OP_STOP)
        q.put((0, "done"))
    else:
        log = []
        f = tp.TPFollower(_StubEngine(log), gm, False, M, "cpu", dist.group.WORLD)
        f.use_graphs = False
        f.serve()
        q.put((1, log))
    dist.destroy_process_group()


def test_tp_driver_follower_protocol_gloo():
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_proto_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = dict(q.get(timeout=120) for _ in range(2))
    [p.join(60) for p in procs]
    log = res[1]
    S = 65
    assert log[0] == ("clear",)
    assert log[1] == ("forward", 100 + S - 1, 0 + 1 + 2 + 3, 0, 100 + S - 1, 100, True)      # OP_FIRST: rows [0, P+S-1)
    assert log[2] == ("gather", 2, 100, [101, 109])
    assert log[3] == ("forward", S, 1 + 2 + 3 + 4, 0, S, 0, True) and log[4] == ("gather", 0, 103, [101, 109])
    assert log[5] == ("forward", S, 2 + 3 + 4 + 5, 0, S, 0, True) and log[6] == ("gather", 1, 104, [101, 109])
    assert len(log) == 7


# ------------------------------------------------------------------------------------------------ peer block layout
def _ll_accepts(N, n, rows_max, own_max):
    """sq_tp_allreduce_ll_add_rmsnorm's size check (own_max == rows_max is its one-shot form)."""
    return n <= rows_max and (own_max == rows_max or (n + N - 1) // N <= own_max)


def _layout_cases():
    return [(N, n_max, hidden) for N in range(2, 9)
            for n_max, hidden in [(1, 4096), (N - 1 or 1, 2048), (N + 1, 1028), (128, 4096), (257, 8192), (768, 8192),
                                  (1024, 5120), (300, 16384)]]


def test_peer_layout_regions_hold_every_kernel_access():
    """The regions of PeerBuffers' block do not overlap, fit in `total`, and hold the highest byte each kernel in sq_tp.cu
    can touch for any n <= n_max it accepts (indexing restated from the kernels)."""
    from sequoia_b200.peer import FLAG_BYTES, MBOX_WORDS, peer_layout
    for N, n_max, hidden in _layout_cases():
        for form in (None, True, False):
            L = peer_layout(N, n_max, hidden, ll_oneshot=form)
            regs = L.regions()
            # 16-byte words everywhere; at hidden % 8 == 4 (LL only) the partials are read 8 bytes at a time
            assert regs[0][1] == 0 and all(off % (16 if hidden % 8 == 0 or name not in ("proj_b", "red_a", "red_b") else 8) == 0
                                           for name, off, _ in regs), (N, n_max, hidden, regs)
            for (a, oa, sa), (b, ob, _) in zip(regs, regs[1:]):
                assert oa + sa <= ob, (N, n_max, hidden, a, b)
            assert regs[-1][1] + regs[-1][2] <= L.total
            size = {name: sz for name, _, sz in regs}
            rows = L.push_rows
            assert rows == min(n_max, 256)
            # highest byte + 1 touched, per region
            assert n_max * hidden * 2 <= size["proj_a"] and n_max * hidden * 2 <= size["red_a"]    # pull partials / red rows
            assert 4 * N <= size["flags"] and 4 * 3 <= size["epoch"]                               # flags[s], epoch[0..2]
            assert 4 * n_max <= size["rowflags_a"]                                                  # rowflags[r], r < n
            assert (((N - 1) * rows + rows - 1) * hidden + hidden) * 2 <= size["recv_a"]            # recv[(rank*rows_max+r)*hidden]
            assert 4 * N * rows <= size["pflags"]                                                   # pflags[src*rows_max + r]
            oneshot = L.ll_own == rows
            lrow_max = max((n - 1) if oneshot else (n - 1) // N for n in range(1, n_max + 1)
                           if _ll_accepts(N, n, rows, L.ll_own))
            assert lrow_max < L.ll_own
            assert (((N - 1) * L.ll_own + lrow_max) * (hidden // 4) + hidden // 4) * 16 <= size["ll1_a"]
            assert ((rows - 1) * (hidden // 4) + hidden // 4) * 16 <= size["ll2_a"]                 # ll2[r * hidden/4 + p]
            assert 2 * MBOX_WORDS * 8 == size["mbox_0"] == size["mbox_1"]
            assert FLAG_BYTES == 1024
            assert size["proj_b"] == size["proj_a"] and size["recv_b"] == size["recv_a"] and size["ll1_b"] == size["ll1_a"]


def test_peer_layout_ll_form():
    """own_max == rows_max (the LL kernel's one-shot form) exactly where the one-shot form is intended: below 4 ranks, or
    a single row (where the two-shot gather area of one row per source is the one-shot area).  Forcing the form gives
    own_max = rows_max or ceil(rows_max / N)."""
    from sequoia_b200.peer import peer_layout
    for N, n_max, hidden in _layout_cases():
        L = peer_layout(N, n_max, hidden)
        intended = N <= 3 or L.push_rows == 1
        assert (L.ll_own == L.push_rows) == intended == L.ll_oneshot, (N, n_max)
        assert L.ll_own == (L.push_rows if N <= 3 else -(-L.push_rows // N))
        assert peer_layout(N, n_max, hidden, ll_oneshot=True).ll_own == L.push_rows
        two = peer_layout(N, n_max, hidden, ll_oneshot=False)
        assert two.ll_own == -(-two.push_rows // N) and two.ll_oneshot == (two.push_rows == 1)


def test_tp_protocol_table():
    """The all-reduce kernel chosen for (N, n, hidden) under the defaults and each SQ_TP_SHOT."""
    from sequoia_b200.peer import tp_protocol
    P, T, O, LL = "push", "two_shot", "one_shot", "ll"
    points = [(1, 4096), (128, 4096), (256, 8192), (257, 4096), (129, 8192), (128, 16384), (256, 16384), (768, 8192),
              (64, 1028)]
    for N in range(2, 9):
        for n, h in points:
            ll_fits = n <= 256 and n * h * 2 <= 4 << 20 and h <= 8192
            pull = T if N >= 4 else O
            want = {"": LL if (4 <= N <= 7 and ll_fits) else pull,
                    "1": O, "2": T,
                    "3": P if (n <= 256 and (N - 1) * n * h * 2 <= 8 << 20) else pull,
                    "4": LL if ll_fits else pull}
            for shot, w in want.items():
                assert tp_protocol(N, n, h, shot) == w, (N, n, h, shot)
    # literal spot checks of the defaults: config 2 (128 rows x 4096) and config 4 (768 rows x 8192)
    assert [tp_protocol(N, 128, 4096) for N in range(2, 9)] == [O, O, LL, LL, LL, LL, T]
    assert [tp_protocol(N, 768, 8192) for N in range(2, 9)] == [O, O, T, T, T, T, T]
    assert [tp_protocol(N, 128, 16384) for N in range(2, 9)] == [O, O, T, T, T, T, T]      # LL holds hidden <= 8192 only
    assert tp_protocol(2, 256, 16384, "3") == P and tp_protocol(3, 256, 16384, "3") == O
