"""NVLink peer-memory buffers for the fused TP all-reduce kernel (csrc/sq_tp.cu).

Each rank cudaMalloc's one block (layout: `peer_layout`), exports it with CUDA IPC, and maps every
peer's block (cudaIpcOpenMemHandle, peer access over NVLink / NVSwitch).  torch sees the two partial buffers as ordinary
fp16 tensors (zero-copy via __cuda_array_interface__), so the row-parallel GEMMs write their outputs straight into
peer-visible memory with `torch.mm(..., out=...)`."""
from __future__ import annotations

import ctypes as C
import dataclasses
import os

import torch
import torch.distributed as dist

from . import _lib
from ._lib import check, ptr, stream_ptr


class _CudaArray:
    def __init__(self, address: int, shape, typestr="<f2"):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (address, False), "version": 2}


FLAG_BYTES = 1024
MBOX_WORDS = 8192              # 4-byte payload words per message (tokens + position ids of M <= 2040 plus the state word)
PUSH_ROWS_MAX = 256            # rows of the push receive slots and of the LL areas
LL_BYTES_MAX = 4 << 20         # LL: payload (n x hidden fp16) at most this
LL_HIDDEN_MAX = 256 * 4 * 8    # LL kernel: 256 threads x 8 16-byte pairs x 4 halfs
PUSH_BYTES_MAX = 8 << 20       # push: bytes pushed per rank ((N - 1) x payload) at most this


@dataclasses.dataclass(frozen=True)
class PeerLayout:
    """Byte offsets of the regions of one rank's peer block (every rank's block has the same layout).  Pairs are
    (buffer A, buffer B); `mbox` is (channel 0, channel 1), each 2 parities x MBOX_WORDS 8-byte LL words."""
    N: int
    n_max: int
    hidden: int
    push_rows: int             # rows_max of the push and LL kernels
    ll_own: int                # own_max of the LL kernel; == push_rows selects its one-shot form
    ll_oneshot: bool           # the LL form these areas are sized for
    part: int                  # bytes of one partial / reduced buffer (n_max, hidden) fp16
    rowflag_bytes: int
    recv_bytes: int
    pflag_bytes: int
    ll1_bytes: int
    ll2_bytes: int
    mbox_bytes: int
    proj: tuple
    red: tuple
    flags: int
    epoch: int
    rowflags: tuple
    recv: tuple
    pflags: int
    ll1: tuple
    ll2: tuple
    mbox: tuple
    total: int

    def regions(self):
        """(name, offset, bytes) of every region, in address order."""
        r = [("proj_a", self.proj[0], self.part), ("proj_b", self.proj[1], self.part), ("red_a", self.red[0], self.part),
             ("red_b", self.red[1], self.part), ("flags", self.flags, FLAG_BYTES), ("epoch", self.epoch, FLAG_BYTES)]
        r += [(f"rowflags_{'ab'[w]}", self.rowflags[w], self.rowflag_bytes) for w in range(2)]
        r += [(f"recv_{'ab'[w]}", self.recv[w], self.recv_bytes) for w in range(2)]
        r += [("pflags", self.pflags, self.pflag_bytes)]
        for w in range(2):
            r += [(f"ll1_{'ab'[w]}", self.ll1[w], self.ll1_bytes), (f"ll2_{'ab'[w]}", self.ll2[w], self.ll2_bytes)]
        r += [(f"mbox_{ch}", self.mbox[ch], self.mbox_bytes // 2) for ch in range(2)]
        return r


def peer_layout(N: int, n_max: int, hidden: int, ll_oneshot=None) -> PeerLayout:
    """The layout of one rank's block [partial A | partial B | reduced A | reduced B | flags | epoch | row flags A | row
    flags B | push slots A | push slots B | push flags | LL A | LL B | mailboxes].  ll_oneshot=None picks the LL form
    PeerBuffers uses: one-shot below 4 ranks."""
    part = n_max * hidden * 2
    rowflag_bytes = ((n_max * 4 + 1023) // 1024) * 1024
    # one-shot PUSH (small payloads): receive slots for <= push_rows rows from each source, per buffer parity
    push_rows = min(n_max, PUSH_ROWS_MAX)
    recv_bytes = N * push_rows * hidden * 2
    pflag_bytes = ((N * push_rows * 4 + 1023) // 1024) * 1024
    # LL (small payloads): gather area (N sources x own_max rows) and reduced-row area, 2 bytes of slot per byte of payload,
    # per buffer parity.  One-shot form (N <= 3): every row from every source, one NVLink trip, own_max = rows_max; two-shot:
    # rows owned by rank r % N, two trips, own_max = ceil(rows_max / N).  The kernel reads own_max == rows_max as the
    # one-shot form, so a single row (rows_max = 1, where the two areas coincide) always runs one-shot.
    if ll_oneshot is None:
        ll_oneshot = N <= 3
    ll_own = push_rows if ll_oneshot else (push_rows + N - 1) // N
    ll_oneshot = ll_own == push_rows
    ll1_bytes = N * ll_own * hidden * 4
    ll2_bytes = push_rows * hidden * 4
    # mailboxes for the driver -> follower messages: 2 channels x 2 parities x MBOX_WORDS 8-byte LL words
    mbox_bytes = 2 * 2 * MBOX_WORDS * 8
    flags = 4 * part
    rf0 = flags + 2 * FLAG_BYTES
    rv0 = rf0 + 2 * rowflag_bytes
    pflags = rv0 + 2 * recv_bytes
    ll0 = pflags + pflag_bytes
    mb0 = ll0 + 2 * (ll1_bytes + ll2_bytes)
    return PeerLayout(
        N=N, n_max=n_max, hidden=hidden, push_rows=push_rows, ll_own=ll_own, ll_oneshot=ll_oneshot, part=part,
        rowflag_bytes=rowflag_bytes, recv_bytes=recv_bytes, pflag_bytes=pflag_bytes, ll1_bytes=ll1_bytes,
        ll2_bytes=ll2_bytes, mbox_bytes=mbox_bytes, proj=(0, part), red=(2 * part, 3 * part), flags=flags,
        epoch=flags + FLAG_BYTES, rowflags=(rf0, rf0 + rowflag_bytes), recv=(rv0, rv0 + recv_bytes), pflags=pflags,
        ll1=tuple(ll0 + w * (ll1_bytes + ll2_bytes) for w in range(2)),
        ll2=tuple(ll0 + w * (ll1_bytes + ll2_bytes) + ll1_bytes for w in range(2)),
        mbox=(mb0, mb0 + 2 * MBOX_WORDS * 8), total=mb0 + mbox_bytes)


def tp_protocol(N: int, n: int, hidden: int, shot: str = "") -> str:
    """The all-reduce kernel PeerBuffers.allreduce_add_rmsnorm runs for n rows (n <= n_max): 'll', 'push', 'two_shot' or
    'one_shot' (pull).  `shot` is SQ_TP_SHOT: '1' one-shot pull, '2' two-shot pull, '3' allows push, '4' allows LL; ''
    the defaults (not measured on H100 multi-GPU boxes): one-shot pull below 4 ranks, LL for 4..7 ranks and two-shot pull
    at 8, LL and push only for payloads that fit their areas and byte limits."""
    # shot 4 = LL (data and epoch in one 8-byte store, readers poll).  LL doubles the bytes, and at 8 ranks each owner
    # gathers 7 x 256 KB of a c2 payload (128 rows x 4096).
    ll_ok = shot == "4" or (shot == "" and 4 <= N < 8)
    if ll_ok and n <= PUSH_ROWS_MAX and n * hidden * 2 <= LL_BYTES_MAX and hidden <= LL_HIDDEN_MAX:
        return "ll"
    # shot 3 = one-shot PUSH for small payloads.  Opt-in: the system fence between the remote stores and the flag costs the
    # round trip that the pull spends on its loads.
    if shot == "3" and n <= PUSH_ROWS_MAX and (N - 1) * n * hidden * 2 <= PUSH_BYTES_MAX:
        return "push"
    # one-shot (every rank pulls all partials) below 4 ranks, two-shot (reduce-scatter + all-gather in one kernel) from 4
    if shot == "2" or (shot != "1" and N >= 4):
        return "two_shot"
    return "one_shot"


class PeerBuffers:
    FLAG_BYTES = FLAG_BYTES
    MBOX_WORDS = MBOX_WORDS

    def __init__(self, group, device, n_max: int, hidden: int):
        lib = _lib.load()
        self.group, self.device = group, torch.device(device)
        self.N, self.rank = dist.get_world_size(group), dist.get_rank(group)
        assert 2 <= self.N <= 8
        self.n_max, self.hidden = n_max, hidden
        L = self.layout = peer_layout(self.N, n_max, hidden)
        self.push_rows, self.ll_own = L.push_rows, L.ll_own
        self.shot = os.environ.get("SQ_TP_SHOT", "")
        base = C.c_void_p()
        check(lib.sq_tp_alloc(C.byref(base), L.total), "sq_tp_alloc")
        self.base = base.value
        handle = (C.c_uint8 * 64)()
        check(lib.sq_tp_ipc_export(base, handle), "sq_tp_ipc_export")
        handles = [None] * self.N
        dist.all_gather_object(handles, bytes(handle), group=group)
        self.bases = []
        self._opened = []
        for r in range(self.N):
            if r == self.rank:
                self.bases.append(self.base)
                continue
            p = C.c_void_p()
            h = (C.c_uint8 * 64).from_buffer_copy(handles[r])
            check(lib.sq_tp_ipc_open(h, C.byref(p)), "sq_tp_ipc_open")
            self.bases.append(p.value)
            self._opened.append(p.value)
        arr = C.c_void_p * 8

        def peers(off):
            return arr(*[b + off for b in self.bases] + [None] * (8 - self.N))

        self.proj_ptrs = [peers(L.proj[w]) for w in range(2)]
        self.red_ptrs = [peers(L.red[w]) for w in range(2)]
        self.flag_ptrs = peers(L.flags)
        self.epoch_ptr = self.base + L.epoch
        self.rowflag_ptrs = [peers(L.rowflags[w]) for w in range(2)]
        self.recv_ptrs = [peers(L.recv[w]) for w in range(2)]
        self.pflag_ptrs = peers(L.pflags)
        self.ll1_ptrs = [peers(L.ll1[w]) for w in range(2)]
        self.ll2_ptrs = [peers(L.ll2[w]) for w in range(2)]
        self.mbox_local = [self.base + L.mbox[ch] for ch in range(2)]
        self.mbox_peers = [arr(*([b + L.mbox[ch] for i, b in enumerate(self.bases) if i != self.rank]
                                 + [None] * (8 - (self.N - 1)))) for ch in range(2)]
        self.msg_epoch = torch.zeros(4, dtype=torch.int32, device=self.device)      # [channel] message counters of this rank
        self.msg_on = os.environ.get("SQ_TP_MSG", "ll") == "ll"                      # SQ_TP_MSG=nccl keeps the NCCL broadcasts
        self.buf = [torch.as_tensor(_CudaArray(self.base + L.proj[w], (n_max, hidden)), device=self.device) for w in range(2)]
        assert self.buf[0].data_ptr() == self.base and self.buf[0].dtype == torch.float16
        dist.barrier(group=group)                      # every rank has mapped every peer before the first kernel runs

    def allreduce_add_rmsnorm(self, which: int, resid: torch.Tensor, weight: torch.Tensor, out: torch.Tensor, n: int,
                              eps: float):
        """resid += sum over ranks of partial buffer `which`; out = rmsnorm(resid) * weight  (one kernel per rank)."""
        proto = tp_protocol(self.N, n, self.hidden, self.shot)
        if proto == "ll":
            check(_lib.load().sq_tp_allreduce_ll_add_rmsnorm(ptr(resid), self.buf[which].data_ptr(), self.ll1_ptrs[which],
                                                             self.ll2_ptrs[which], self.epoch_ptr, self.rank, self.N,
                                                             self.push_rows, self.ll_own, ptr(weight), ptr(out), n, self.hidden,
                                                             eps, stream_ptr()), "sq_tp_allreduce_ll_add_rmsnorm")
            return
        if proto == "push":
            check(_lib.load().sq_tp_allreduce3_add_rmsnorm(ptr(resid), self.buf[which].data_ptr(), self.recv_ptrs[which],
                                                           self.pflag_ptrs, self.epoch_ptr, self.rank, self.N, self.push_rows,
                                                           ptr(weight), ptr(out), n, self.hidden, eps, stream_ptr()),
                  "sq_tp_allreduce3_add_rmsnorm")
            return
        if proto == "two_shot":
            check(_lib.load().sq_tp_allreduce2_add_rmsnorm(ptr(resid), self.proj_ptrs[which], self.red_ptrs[which],
                                                           self.flag_ptrs, self.rowflag_ptrs[which], self.epoch_ptr,
                                                           self.rank, self.N, ptr(weight), ptr(out), n, self.hidden, eps,
                                                           stream_ptr()), "sq_tp_allreduce2_add_rmsnorm")
            return
        check(_lib.load().sq_tp_allreduce_add_rmsnorm(ptr(resid), self.proj_ptrs[which], self.flag_ptrs, self.epoch_ptr,
                                                      self.rank, self.N, ptr(weight), ptr(out), n, self.hidden, eps,
                                                      stream_ptr()), "sq_tp_allreduce_add_rmsnorm")

    @staticmethod
    def _words(t):
        assert t.is_contiguous() and (t.numel() * t.element_size()) % 4 == 0
        return t.numel() * t.element_size() // 4

    def fits(self, tensors) -> bool:
        """True if the message fits a mailbox (else the caller keeps the NCCL broadcasts; both sides see the same sizes)."""
        return sum(self._words(t) for t in tensors) <= self.MBOX_WORDS

    def publish(self, channel: int, tensors):
        """Rank 0: write `tensors` (<= 3) as LL words into every follower's mailbox of `channel` (one kernel)."""
        ts = list(tensors) + [None] * (3 - len(tensors))
        a = [(ptr(t), self._words(t)) if t is not None else (None, 0) for t in ts]
        check(_lib.load().sq_tp_ll_publish(self.mbox_peers[channel], self.N - 1, self.MBOX_WORDS,
                                           self.msg_epoch.data_ptr() + 4 * channel, a[0][0], a[0][1], a[1][0], a[1][1], a[2][0],
                                           a[2][1], stream_ptr()), "sq_tp_ll_publish")

    def consume(self, channel: int, tensors):
        """Followers: poll the mailbox of `channel` and scatter the words into `tensors` (one kernel)."""
        ts = list(tensors) + [None] * (3 - len(tensors))
        a = [(ptr(t), self._words(t)) if t is not None else (None, 0) for t in ts]
        check(_lib.load().sq_tp_ll_consume(self.mbox_local[channel], self.MBOX_WORDS, self.msg_epoch.data_ptr() + 4 * channel,
                                           self.epoch_ptr + 8, a[0][0], a[0][1], a[1][0], a[1][1], a[2][0], a[2][1], stream_ptr()),
              "sq_tp_ll_consume")

    def error(self) -> int:
        t = torch.as_tensor(_CudaArray(self.epoch_ptr, (4,), "<i4"), device=self.device)
        return int(t[2])
