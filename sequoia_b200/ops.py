"""Tensor-level wrappers over the C ABI (one function per exported kernel).

Everything here launches on torch's current CUDA stream, never allocates on the hot path unless
an output tensor is not supplied, and raises on any error (no fallback).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import check, ptr, stream_ptr

F16 = torch.float16


def _need(t: torch.Tensor, dtype, name: str):
    if t.dtype != dtype or not t.is_cuda:
        raise TypeError(f"{name}: expected CUDA tensor of {dtype}, got {t.dtype} on {t.device}")


def embed_rows(table, tokens, n, out, state=None, n0=0):
    lib = _lib.load()
    check(lib.sq_embed_rows(ptr(table), ptr(tokens), ptr(state), n0, n, table.shape[1], ptr(out), stream_ptr()),
          "sq_embed_rows")


def rmsnorm(x, weight, out, n, eps):
    lib = _lib.load()
    check(lib.sq_rmsnorm(ptr(x), ptr(weight), ptr(out), n, x.shape[-1], eps, stream_ptr()), "sq_rmsnorm")


def add_rmsnorm(resid, delta, weight, out, n, eps):
    lib = _lib.load()
    check(lib.sq_add_rmsnorm(ptr(resid), ptr(delta), ptr(weight), ptr(out), n, resid.shape[-1], eps, stream_ptr()),
          "sq_add_rmsnorm")


def silu_mul(gate_up, out, n, interleaved=False):
    """out = silu(gate) * up; interleaved: gate_up columns in blocks of 32 = 16 gate | 16 up (interleave_gate_up order)."""
    lib = _lib.load()
    check(lib.sq_silu_mul_ex(ptr(gate_up), ptr(out), n, out.shape[-1], 1 if interleaved else 0, stream_ptr()), "sq_silu_mul_ex")


def rope_kv_append(qkv, H, Hkv, D, cos, sin, position_ids, storage_ids, n, k_layer, v_layer, M, state=None, n0=0):
    lib = _lib.load()
    check(lib.sq_rope_kv_append(ptr(qkv), qkv.shape[-1], H, Hkv, D, ptr(cos), ptr(sin), ptr(position_ids),
                                ptr(storage_ids), ptr(state), n0, n, ptr(k_layer), ptr(v_layer), M, stream_ptr()),
          "sq_rope_kv_append")


def kv_gather(k_cache, v_cache, idx, n, offset, state=None, max_n=0, zero_tail=False):
    """k_cache/v_cache (L,1,Hkv,M,D); idx int32 device tensor."""
    lib = _lib.load()
    L, _, Hkv, M, D = k_cache.shape
    check(lib.sq_kv_gather(ptr(k_cache), ptr(v_cache), L, Hkv, M, D, ptr(idx), n, offset, ptr(state), max_n,
                           1 if zero_tail else 0, stream_ptr()), "sq_kv_gather")


def kv_gather_big(k_cache, v_cache, idx, n, offset, zero_tail=False):
    """Index lists too long for the on-chip staging of `kv_gather` (host-known n / offset): through a global scratch."""
    lib = _lib.load()
    L, _, Hkv, M, D = k_cache.shape
    nbytes = lib.sq_kv_gather_scratch_bytes(L, Hkv, D, n)
    scratch = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=k_cache.device)
    check(lib.sq_kv_gather_big(ptr(k_cache), ptr(v_cache), L, Hkv, M, D, ptr(idx), n, offset, ptr(scratch), nbytes,
                               1 if zero_tail else 0, stream_ptr()), "sq_kv_gather_big")


class AttnPlan:
    """TMA descriptors + split-KV workspace for one (qkv buffer, KV cache, output buffer) triple.  A (L, B, Hkv, M, D) cache
    with B > 1 makes a batch plan, launched through `tree_attn_batch` (n_max then counts the rows of all B sequences)."""

    def __init__(self, qkv: torch.Tensor, n_max: int, H: int, Hkv: int, D: int, k_cache, v_cache, out):
        lib = _lib.load()
        L, B, hk, M, d = k_cache.shape
        assert hk == Hkv and d == D
        nbytes = lib.sq_attn_workspace_bytes(n_max, H, D, M)
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=qkv.device)
        self.handle = C.c_void_p()
        self._keep = (qkv, k_cache, v_cache, out)
        check(lib.sq_attn_plan_create_batch(C.byref(self.handle), ptr(qkv), qkv.shape[-1], n_max, H, Hkv, D, ptr(k_cache),
                                            ptr(v_cache), L, B, M, ptr(out), ptr(self.workspace), nbytes),
              "sq_attn_plan_create_batch")
        self.n_max, self.M, self.B = n_max, M, B

    def error(self) -> int:
        return _lib.load().sq_attn_plan_error(self.handle)

    def info(self):
        """(query heads per 128-row tile, KV splits of the last tensor-core launch)"""
        gp, z = C.c_int(), C.c_int()
        check(_lib.load().sq_attn_plan_info(self.handle, C.byref(gp), C.byref(z)), "sq_attn_plan_info")
        return gp.value, z.value

    def __del__(self):
        try:
            if self.handle:
                _lib.load().sq_attn_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


def tree_attn(plan: AttnPlan, layer, n, *, state=None, n0=0, kv_end=0, prefix_len=0, dense_mask=None, mask_ld=0,
              tree_bits=None, tree_words=0, tree_size=0, impl=0):
    lib = _lib.load()
    check(lib.sq_tree_attn(plan.handle, layer, n, ptr(state), n0, kv_end, prefix_len, ptr(dense_mask), mask_ld,
                           ptr(tree_bits), tree_words, tree_size, impl, stream_ptr()), "sq_tree_attn")


def softmax_T(logits: torch.Tensor, T: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need(logits, F16, "softmax_T")
    lg = logits.reshape(-1, logits.shape[-1])
    assert lg.stride(-1) == 1
    if out is None:
        out = torch.empty((lg.shape[0], lg.shape[1]), dtype=F16, device=logits.device)
    lib = _lib.load()
    check(lib.sq_softmax_T(ptr(lg), lg.stride(0), ptr(out), out.stride(0), lg.shape[0], lg.shape[1], T, stream_ptr()),
          "sq_softmax_T")
    return out.view(logits.shape) if out.numel() == logits.numel() else out


def sample_level(logits, rand, n_parents, k_max, T, mode, *, parent_rows=None, child_first=None, n_branch=None,
                 positions=None, tokens=None, state=None):
    lib = _lib.load()
    V = logits.shape[-1]
    check(lib.sq_sample_level(ptr(logits), logits.stride(-2), ptr(rand), rand.stride(-2) if rand is not None else 0,
                              ptr(parent_rows), ptr(child_first), ptr(n_branch), n_parents, k_max, V, T, mode,
                              ptr(positions), ptr(tokens), ptr(state), stream_ptr()), "sq_sample_level")


def sample_replace(logits, words, n_parents, k_max, T, *, parent_rows=None, child_first=None, n_branch=None,
                   positions=None, tokens=None, state=None):
    """i.i.d. draws with replacement from softmax(logits/T) rows (SpecInferTree.py:100-105); words: int64 in [0, 2^32)."""
    lib = _lib.load()
    if words.dtype != torch.int64:
        raise TypeError("sample_replace: words must be int64")
    check(lib.sq_sample_replace(ptr(logits), logits.stride(-2), ptr(words), ptr(parent_rows), ptr(child_first),
                                ptr(n_branch), n_parents, k_max, logits.shape[-1], T, ptr(positions), ptr(tokens),
                                ptr(state), stream_ptr()), "sq_sample_replace")


def residual(p, q, out=None):
    _need(p, F16, "residual")
    if out is None:
        out = torch.empty_like(p)
    check(_lib.load().sq_residual(ptr(p), ptr(q), ptr(out), p.shape[-1], stream_ptr()), "sq_residual")
    return out


def top_p_filter_(logits, top_p: float, T: float):
    """get_sampling_logits (utils.py:65-77), in place on (n, V) fp16 logits."""
    _need(logits, F16, "top_p_filter_")
    n, V = logits.shape
    check(_lib.load().sq_top_p_filter(ptr(logits), logits.stride(0), n, V, float(top_p), float(T), stream_ptr()),
          "sq_top_p_filter")
    return logits


def top_k_filter_(logits, k: int):
    """Top-k filter in place on (n, V) fp16 logits: the k best of each row (raw logit descending, equal values by
    ascending index) keep their value, every other one becomes -inf.  k == 0 is off, k >= V filters nothing."""
    _need(logits, F16, "top_k_filter_")
    n, V = logits.shape
    check(_lib.load().sq_top_k_filter(ptr(logits), logits.stride(0), n, V, int(k), stream_ptr()), "sq_top_k_filter")
    return logits


def argmax_rows(logits, out=None):
    n, V = logits.shape
    if out is None:
        out = torch.empty(n, dtype=torch.int64, device=logits.device)
    check(_lib.load().sq_argmax_rows(ptr(logits), logits.stride(0), n, V, ptr(out), stream_ptr()), "sq_argmax_rows")
    return out


ACCEPT_GE, ACCEPT_KEEP_Q = 1, 2          # sq_accept_stochastic policy bits (include/sequoia_b200.h)
ACCEPT_SKIP_DEAD = 8                     # the per-sequence, mixed and stop batch walks only: skip dead children


def accept_stochastic(target_logits, draft_logits, r, noise, succ_off, succ, depth, S, T, tokens, position_ids,
                      accept_idx, state, max_target_seq, policy=0):
    V = target_logits.shape[-1]
    check(_lib.load().sq_accept_stochastic(ptr(target_logits), target_logits.stride(0), ptr(draft_logits),
                                           draft_logits.stride(0), ptr(r), ptr(noise), ptr(succ_off), ptr(succ),
                                           ptr(depth), S, V, T, ptr(tokens), ptr(position_ids), ptr(accept_idx),
                                           ptr(state), max_target_seq, policy, stream_ptr()), "sq_accept_stochastic")


def accept_greedy(target_token, succ_off, succ, depth, S, tokens, position_ids, accept_idx, state, max_target_seq):
    check(_lib.load().sq_accept_greedy(ptr(target_token), ptr(succ_off), ptr(succ), ptr(depth), S, ptr(tokens),
                                       ptr(position_ids), ptr(accept_idx), ptr(state), max_target_seq, stream_ptr()),
          "sq_accept_greedy")


GEMM_TILED, GEMM_SWIGLU = 1, 2          # sq_gemm_plan_create_ex flags (include/sequoia_b200.h)


def gemm_pick_tiles(N: int, K: int, flags: int = 0):
    bn, sp, mc = C.c_int(), C.c_int(), C.c_int()
    check(_lib.load().sq_gemm_pick_tiles_ex(N, K, flags, C.byref(bn), C.byref(sp), C.byref(mc)), "sq_gemm_pick_tiles_ex")
    return bn.value, sp.value, mc.value


def tile_weights(w: torch.Tensor, flags: int = 0) -> torch.Tensor:
    """(N, K) row-major -> (ceil(N/BN), K/64, BN, 64) contiguous, rows beyond N zero (BN = the plan's tile width)."""
    N, K = w.shape
    bn, _, _ = gemm_pick_tiles(N, K, flags)
    tiles = (N + bn - 1) // bn
    if tiles * bn != N:
        pad = torch.zeros(tiles * bn, K, dtype=w.dtype, device=w.device)
        pad[:N] = w
        w = pad
    return w.view(tiles, bn, K // 64, 64).permute(0, 2, 1, 3).contiguous()


def interleave_gate_up(wg: torch.Tensor, wu: torch.Tensor) -> torch.Tensor:
    """(I, K) gate and up weights -> (2I, K) with rows 32b..32b+15 = gate[16b..], rows 32b+16..32b+31 = up[16b..]: the
    row order the fused SwiGLU epilogue of sq_gemm expects."""
    I, K = wg.shape
    assert I % 16 == 0 and wu.shape == wg.shape
    return torch.stack([wg.reshape(I // 16, 16, K), wu.reshape(I // 16, 16, K)], dim=1).reshape(2 * I, K).contiguous()


class GemmPlan:
    """C[:n] = A[:n] @ W.T on the weight-streaming wgmma kernel (csrc/sq_gemm.cu); n > 128 runs one launch per 128 rows."""

    def __init__(self, a: torch.Tensor, w: torch.Tensor, c: torch.Tensor, err_flag: Optional[torch.Tensor] = None,
                 tiled: bool = False, swiglu: bool = False):
        """tiled=True: `w` (N, K) is re-laid out once into the plan's own HBM-friendly copy (`self.w_tiled`, tile (n-tile,
        k-block) = one contiguous BN x 64 block) and the plan streams that copy.
        swiglu=True: `w` = interleave_gate_up(gate, up); the output (n, N/2) is silu(gate) * up (fused epilogue)."""
        lib = _lib.load()
        assert a.dtype == F16 and w.dtype == F16 and c.dtype == F16 and w.is_contiguous()
        assert a.stride(-1) == 1 and c.stride(-1) == 1 and a.shape[1] == w.shape[1]
        assert c.shape[1] >= (w.shape[0] // 2 if swiglu else w.shape[0])
        self.handle = C.c_void_p()
        self.w_tiled = None
        self.N, self.K, self.swiglu = w.shape[0], w.shape[1], swiglu
        flags = (GEMM_TILED if tiled else 0) | (GEMM_SWIGLU if swiglu else 0)
        if tiled:
            self.w_tiled = w = tile_weights(w, flags)
        self._keep = (a, w, c, err_flag)
        check(lib.sq_gemm_plan_create_ex(C.byref(self.handle), ptr(a), a.stride(0), a.shape[0], ptr(w), self.N, self.K,
                                         ptr(c), c.stride(0), ptr(err_flag), flags), "sq_gemm_plan_create_ex")

    def info(self):
        bn, sp, st = C.c_int(), C.c_int(), C.c_int()
        _lib.load().sq_gemm_plan_info(self.handle, C.byref(bn), C.byref(sp), C.byref(st))
        return bn.value, sp.value, st.value

    def run(self, n: int, a_row0: int = 0, out: Optional[torch.Tensor] = None):
        """rows [a_row0, a_row0+n) of the activation buffer -> `out[:n]` (default: the plan's output buffer, same rows)."""
        if a_row0 == 0 and out is None:
            check(_lib.load().sq_gemm_run(self.handle, n, stream_ptr()), "sq_gemm_run")
            return
        if out is not None:
            assert out.dtype == F16 and out.stride(-1) == 1 and out.shape[0] >= n
        check(_lib.load().sq_gemm_run_at(self.handle, n, a_row0, ptr(out), out.stride(0) if out is not None else 0,
                                         stream_ptr()), "sq_gemm_run_at")

    def __del__(self):
        try:
            if self.handle:
                _lib.load().sq_gemm_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


# ---- FP8 (E4M3) weights (csrc/sq_gemm_fp8.cu) --------------------------------------------------------------------------------
FP8_MAX = 448.0                          # largest finite e4m3 magnitude
F8 = torch.float8_e4m3fn


def quantize_fp8(w: torch.Tensor, rows_per_chunk: int = 4096):
    """(N, K) fp16 weight -> (q (N, K) float8_e4m3fn, s (N) fp16), on w's device:
    s[j] = fp16(max|W[j,:]| / 448) (1 for an all-zero row, the smallest positive fp16 where that rounds to 0) and
    q = e4m3(clamp(W / s, -448, 448)), rounded to nearest even.  Works through `rows_per_chunk` rows at a time, so the
    fp32 temporaries stay small next to the weight."""
    if w.dtype != F16 or w.dim() != 2:
        raise TypeError(f"quantize_fp8: expected a 2-D float16 tensor, got {w.dtype} {tuple(w.shape)}")
    N, K = w.shape
    q = torch.empty(N, K, dtype=F8, device=w.device)
    s = torch.empty(N, dtype=F16, device=w.device)
    tiny = torch.finfo(F16).smallest_normal * 2.0 ** -10          # 2^-24, the smallest positive (subnormal) fp16
    for r0 in range(0, N, rows_per_chunk):
        blk = w[r0:r0 + rows_per_chunk].float()
        amax = blk.abs().amax(dim=1)
        sc = (amax / FP8_MAX).to(F16)
        sc = torch.where(amax == 0, torch.ones_like(sc), torch.where(sc == 0, torch.full_like(sc, tiny), sc))
        q[r0:r0 + rows_per_chunk] = (blk / sc.float()[:, None]).clamp_(-FP8_MAX, FP8_MAX).to(F8)
        s[r0:r0 + rows_per_chunk] = sc
    return q, s


def dequantize_fp8(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """W'[j, k] = fp16(fp16(q[j, k]) * s[j]): the fp16 matrix the FP8 GEMM multiplies by (exact e4m3 -> fp16, one
    rounding of the product)."""
    return q.to(F16) * s.to(F16)[:, None]


def fp8_tile_weights(q: torch.Tensor) -> torch.Tensor:
    """(N, K) float8_e4m3fn row-major -> the FP8 GEMM's pre-tiled copy (N * K bytes, layout in include/sequoia_b200.h)."""
    if q.dtype != F8 or not q.is_cuda or not q.is_contiguous():
        raise TypeError("fp8_tile_weights: expected a contiguous CUDA float8_e4m3fn tensor")
    N, K = q.shape
    out = torch.empty(N * K, dtype=torch.uint8, device=q.device)
    check(_lib.load().sq_gemm_fp8_tile_weights(ptr(q), ptr(out), N, K, stream_ptr(q.device)), "sq_gemm_fp8_tile_weights")
    return out


class GemmFp8Plan:
    """C[:n] = A[:n] @ W'.T on the FP8 weight-streaming kernel, W' = dequantize_fp8(q, s).  The plan keeps the pre-tiled
    copy of q and the scales (the only resident form of the weight); n > 128 runs one launch per 128 rows."""

    def __init__(self, a: torch.Tensor, q: torch.Tensor, s: torch.Tensor, c: torch.Tensor,
                 err_flag: Optional[torch.Tensor] = None):
        assert a.dtype == F16 and c.dtype == F16 and s.dtype == F16 and q.dtype == F8
        assert a.stride(-1) == 1 and c.stride(-1) == 1 and a.shape[1] == q.shape[1] and c.shape[1] >= q.shape[0]
        assert s.shape == (q.shape[0],) and s.is_contiguous()
        self.N, self.K = q.shape
        self.w_tiled = fp8_tile_weights(q)
        self.scale = s
        self.handle = C.c_void_p()
        self._keep = (a, c, err_flag)
        check(_lib.load().sq_gemm_fp8_plan_create(C.byref(self.handle), ptr(a), a.stride(0), a.shape[0], ptr(self.w_tiled),
                                                  ptr(s), self.N, self.K, ptr(c), c.stride(0), ptr(err_flag)),
              "sq_gemm_fp8_plan_create")

    def info(self):
        """(64-row weight tiles per CTA, K splits, ring stages of the 128-row instance)"""
        w, sp, st = C.c_int(), C.c_int(), C.c_int()
        check(_lib.load().sq_gemm_fp8_plan_info(self.handle, C.byref(w), C.byref(sp), C.byref(st)), "sq_gemm_fp8_plan_info")
        return w.value, sp.value, st.value

    def weight_bytes(self) -> int:
        return self.w_tiled.numel() + 2 * self.scale.numel()

    def run(self, n: int, a_row0: int = 0, out: Optional[torch.Tensor] = None):
        """rows [a_row0, a_row0+n) of the activation buffer -> `out[:n]` (default: the plan's output buffer, same rows)."""
        if out is not None:
            assert out.dtype == F16 and out.stride(-1) == 1 and out.shape[0] >= n
        check(_lib.load().sq_gemm_fp8_run_at(self.handle, n, a_row0, ptr(out), out.stride(0) if out is not None else 0,
                                             stream_ptr()), "sq_gemm_fp8_run_at")

    def __del__(self):
        try:
            if self.handle:
                _lib.load().sq_gemm_fp8_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


# ---- draft attention (csrc/sq_draft.cu) -----------------------------------------------------------------------------------
def draft_supported(hidden, n_heads, n_kv_heads, head_dim, max_length) -> bool:
    return bool(_lib.load().sq_draft_supported(hidden, n_heads, n_kv_heads, head_dim, max_length))


class DraftPlan:
    """Tree-masked attention of the small draft model's forwards of <= 64 rows, K/V read from the engine's caches."""
    MAX_ROWS = 64

    def __init__(self, hidden, n_layers, n_heads, max_length, k_cache, v_cache):
        for t in (k_cache, v_cache):
            assert t.dtype == F16 and t.is_contiguous()
        self._keep = (k_cache, v_cache)
        self.handle = C.c_void_p()
        check(_lib.load().sq_draft_plan_create(C.byref(self.handle), hidden, n_layers, n_heads, max_length, ptr(k_cache),
                                               ptr(v_cache)), "sq_draft_plan_create")

    def attention(self, layer, n, qkv, attn_out, state, n0, kv_end, tree_bits, tree_words, tree_size):
        check(_lib.load().sq_draft_attention(self.handle, layer, n, ptr(qkv), ptr(attn_out), ptr(state), n0, kv_end,
                                             ptr(tree_bits), tree_words, tree_size, stream_ptr()), "sq_draft_attention")

    def __del__(self):
        try:
            if self.handle:
                _lib.load().sq_draft_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


# ---- batches of B sequences sharing one growmap (include/sequoia_b200.h, "batches") ------------------------------------------
# Per-sequence buffers are (B, ...) tensors: state (B, 16) int32, tokens / position_ids / storage_ids / r (B, M), accept_idx
# (B, >= S) int32, noise (B, >= V); activation rows are sequence-major (sequence b's n rows start at row b * n).  Draft logits:
# node k of sequence b at row row_base[k] + b * row_step[k] (see draft_row_tables).
def _rows(t, name):
    if t.dim() != 2 or t.stride(-1) != 1:
        raise ValueError(f"{name}: expected a (B, ...) tensor with contiguous rows, got {tuple(t.shape)}")
    return t.stride(0)


def draft_row_tables(levels, S: int, B: int, device):
    """(row_base, row_step) int32 tables of S entries for a draft-logit buffer holding each tree level (n0, tb) as one block
    of B * tb rows at row B * n0: row of node k of sequence b = row_base[k] + b * row_step[k].  Node 0 (the root) is
    level (0, 1)."""
    base, step = [0] * S, [1] * S
    for n0, tb in levels:
        for k in range(n0, n0 + tb):
            base[k], step[k] = B * n0 + (k - n0), tb
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=device)
    return i32(base), i32(step)


def embed_rows_batch(table, tokens, n, out, state, n0=0):
    B = state.shape[0]
    check(_lib.load().sq_embed_rows_batch(ptr(table), ptr(tokens), _rows(tokens, "tokens"), ptr(state), n0, n, B,
                                          table.shape[1], ptr(out), stream_ptr()), "sq_embed_rows_batch")


def rope_kv_append_batch(qkv, H, Hkv, D, cos, sin, position_ids, storage_ids, n, k_layer, v_layer, M, state, n0=0):
    """k_layer / v_layer: (B, Hkv, M, D) = one layer of a (L, B, Hkv, M, D) cache."""
    B = state.shape[0]
    ld = _rows(position_ids, "position_ids")
    assert _rows(storage_ids, "storage_ids") == ld and k_layer.shape[0] == B
    check(_lib.load().sq_rope_kv_append_batch(ptr(qkv), qkv.shape[-1], H, Hkv, D, ptr(cos), ptr(sin), ptr(position_ids),
                                              ptr(storage_ids), ld, ptr(state), n0, n, B, ptr(k_layer), ptr(v_layer), M,
                                              stream_ptr()), "sq_rope_kv_append_batch")


def kv_gather_batch(k_cache, v_cache, accept_idx, state, max_n):
    L, B, Hkv, M, D = k_cache.shape
    assert state.shape[0] == B and accept_idx.dtype == torch.int32
    check(_lib.load().sq_kv_gather_batch(ptr(k_cache), ptr(v_cache), L, B, Hkv, M, D, ptr(accept_idx),
                                         _rows(accept_idx, "accept_idx"), ptr(state), max_n, stream_ptr()),
          "sq_kv_gather_batch")


def kv_copy_prefix(kv_cache, src: int, dst: int, n: int):
    """Rows [0, n) of sequence src's K and V, every layer, into sequence dst's of the same (L, B, Hkv, M, D) cache
    (an object with k_cache / v_cache, as KV_Cache); one launch."""
    k, v = kv_cache.k_cache, kv_cache.v_cache
    assert k.shape == v.shape and k.dtype == v.dtype == torch.float16 and k.is_contiguous() and v.is_contiguous()
    L, B, Hkv, M, D = k.shape
    check(_lib.load().sq_kv_copy_prefix(ptr(k), ptr(v), L, B, Hkv, M, D, int(src), int(dst), int(n), stream_ptr()),
          "sq_kv_copy_prefix")


def tree_attn_batch(plan: AttnPlan, layer, n, *, state, n0=0, kv_end=0, tree_bits=None, tree_words=0, tree_size=0):
    check(_lib.load().sq_tree_attn_batch(plan.handle, layer, n, state.shape[0], ptr(state), n0, kv_end, ptr(tree_bits),
                                         tree_words, tree_size, stream_ptr()), "sq_tree_attn_batch")


class RaggedPart(C.Structure):
    """sq_ragged_part: n rows of sequence seq, nodes [n0, n0 + n) in its tree-relative addressing, attending slots
    [0, base + kv_end)"""
    _fields_ = [("seq", C.c_int32), ("n", C.c_int32), ("n0", C.c_int32), ("kv_end", C.c_int32)]


def ragged_parts(parts):
    """(seq, n, n0, kv_end) tuples -> the host array the *_ragged calls take (an array built here is passed through)."""
    if isinstance(parts, C.Array):
        return parts
    parts = [tuple(int(x) for x in p) for p in parts]
    return (RaggedPart * len(parts))(*parts)


def ragged_layout(parts, B: int, n_max: int, rows_per_tile: int = 1):
    """-> (row0, tile0): lists of len(parts) + 1 prefix sums of the packed rows and of the q tiles of rows_per_tile rows.
    Raises SequoiaLibError on a part list the ragged calls refuse."""
    arr = ragged_parts(parts)
    k = len(arr)
    row0, tile0 = (C.c_int32 * (k + 1))(), (C.c_int32 * (k + 1))()
    check(_lib.load().sq_ragged_layout(C.addressof(arr), k, B, n_max, rows_per_tile, C.addressof(row0),
                                       C.addressof(tile0)), "sq_ragged_layout")
    return list(row0), list(tile0)


def embed_rows_ragged(table, tokens, parts, out, state):
    """Rows of the listed sequences packed in list order into out (n_max = out's rows); tokens (B, M), state (B, 16)."""
    arr = ragged_parts(parts)
    check(_lib.load().sq_embed_rows_ragged(ptr(table), ptr(tokens), _rows(tokens, "tokens"), ptr(state), C.addressof(arr),
                                           len(arr), state.shape[0], out.shape[0], table.shape[1], ptr(out),
                                           stream_ptr()), "sq_embed_rows_ragged")


def rope_kv_append_ragged(qkv, H, Hkv, D, cos, sin, position_ids, storage_ids, parts, k_layer, v_layer, M, state):
    """k_layer / v_layer: (B, Hkv, M, D) = one layer of a (L, B, Hkv, M, D) cache; qkv rows packed in list order."""
    B = state.shape[0]
    ld = _rows(position_ids, "position_ids")
    assert _rows(storage_ids, "storage_ids") == ld and k_layer.shape[0] == B
    arr = ragged_parts(parts)
    check(_lib.load().sq_rope_kv_append_ragged(ptr(qkv), qkv.shape[-1], H, Hkv, D, ptr(cos), ptr(sin), ptr(position_ids),
                                               ptr(storage_ids), ld, ptr(state), C.addressof(arr), len(arr), B,
                                               qkv.shape[0], ptr(k_layer), ptr(v_layer), M, stream_ptr()),
          "sq_rope_kv_append_ragged")


def tree_attn_ragged(plan: AttnPlan, layer, parts, *, state, tree_bits=None, tree_words=0, tree_size=0):
    arr = ragged_parts(parts)
    check(_lib.load().sq_tree_attn_ragged(plan.handle, layer, C.addressof(arr), len(arr), ptr(state), ptr(tree_bits),
                                          tree_words, tree_size, stream_ptr()), "sq_tree_attn_ragged")


def sample_level_batch(logits, row_base, row_step, rand, n_parents, k_max, T, mode, *, parent_rows, child_first, n_branch,
                       tokens, state):
    """rand: (B, S, V) (mode 0) or None (mode 1, top-k)."""
    if rand is not None:
        assert rand.dim() == 3 and rand.stride(-1) == 1
    check(_lib.load().sq_sample_level_batch(
        ptr(logits), logits.stride(0), ptr(row_base), ptr(row_step), ptr(rand), rand.stride(1) if rand is not None else 0,
        rand.stride(0) if rand is not None else 0, ptr(parent_rows), ptr(child_first), ptr(n_branch), n_parents, k_max,
        logits.shape[-1], T, mode, ptr(tokens), _rows(tokens, "tokens"), ptr(state), state.shape[0], stream_ptr()),
        "sq_sample_level_batch")


def accept_stochastic_batch(target_logits, draft_logits, row_base, row_step, r, noise, succ_off, succ, depth, S, T, tokens,
                            position_ids, accept_idx, state, max_target_seq, policy=0):
    """target_logits (B*S, V); r, tokens, position_ids (B, M); noise (B, V); accept_idx (B, >= S)."""
    V = target_logits.shape[-1]
    ld = _rows(tokens, "tokens")
    assert _rows(position_ids, "position_ids") == ld and _rows(r, "r") == ld
    check(_lib.load().sq_accept_stochastic_batch(
        ptr(target_logits), target_logits.stride(0), ptr(draft_logits), draft_logits.stride(0), ptr(row_base),
        ptr(row_step), ptr(r), ptr(noise), _rows(noise, "noise"), ptr(succ_off), ptr(succ), ptr(depth), S, V, T,
        ptr(tokens), ptr(position_ids), ld, ptr(accept_idx), _rows(accept_idx, "accept_idx"), ptr(state), state.shape[0],
        max_target_seq, policy, stream_ptr()), "sq_accept_stochastic_batch")


def _seq_params(name, B, **arrays):
    for k, t in arrays.items():
        if t is None or t.dtype != torch.float32 or not t.is_cuda or t.dim() != 1 or t.shape[0] < B or t.stride(0) != 1:
            raise TypeError(f"{name}: {k} must be a contiguous ({B},) float32 CUDA tensor")


def sample_level_batch_per_seq(logits, row_base, row_step, rand, n_parents, k_max, T, mode, *, parent_rows, child_first,
                               n_branch, tokens, state):
    """sample_level_batch with the temperature of sequence b read from T[b] ((B,) float32 on the device)."""
    _seq_params("sample_level_batch_per_seq", state.shape[0], T=T)
    if rand is not None:
        assert rand.dim() == 3 and rand.stride(-1) == 1
    check(_lib.load().sq_sample_level_batch_per_seq(
        ptr(logits), logits.stride(0), ptr(row_base), ptr(row_step), ptr(rand), rand.stride(1) if rand is not None else 0,
        rand.stride(0) if rand is not None else 0, ptr(parent_rows), ptr(child_first), ptr(n_branch), n_parents, k_max,
        logits.shape[-1], ptr(T), mode, ptr(tokens), _rows(tokens, "tokens"), ptr(state), state.shape[0], stream_ptr()),
        "sq_sample_level_batch_per_seq")


def accept_stochastic_batch_per_seq(target_logits, draft_logits, row_base, row_step, r, noise, succ_off, succ, depth, S, T,
                                    tokens, position_ids, accept_idx, state, max_target_seq, policy=0):
    """accept_stochastic_batch with the temperature of sequence b read from T[b] ((B,) float32 on the device)."""
    _seq_params("accept_stochastic_batch_per_seq", state.shape[0], T=T)
    V = target_logits.shape[-1]
    ld = _rows(tokens, "tokens")
    assert _rows(position_ids, "position_ids") == ld and _rows(r, "r") == ld
    check(_lib.load().sq_accept_stochastic_batch_per_seq(
        ptr(target_logits), target_logits.stride(0), ptr(draft_logits), draft_logits.stride(0), ptr(row_base),
        ptr(row_step), ptr(r), ptr(noise), _rows(noise, "noise"), ptr(succ_off), ptr(succ), ptr(depth), S, V, ptr(T),
        ptr(tokens), ptr(position_ids), ld, ptr(accept_idx), _rows(accept_idx, "accept_idx"), ptr(state), state.shape[0],
        max_target_seq, policy, stream_ptr()), "sq_accept_stochastic_batch_per_seq")


def top_p_filter_per_seq_(logits, top_p, T, rows_per_seq: int):
    """top_p_filter_ in place on (n, V) fp16 logits whose row r belongs to sequence r // rows_per_seq, at that sequence's
    top_p[b] and T[b] ((B,) float32 on the device); rows of a sequence with top_p >= 1 are left untouched."""
    _need(logits, F16, "top_p_filter_per_seq_")
    n, V = logits.shape
    B = n // rows_per_seq if rows_per_seq > 0 else 0
    _seq_params("top_p_filter_per_seq_", B, top_p=top_p, T=T)
    check(_lib.load().sq_top_p_filter_per_seq(ptr(logits), logits.stride(0), n, V, ptr(top_p), ptr(T), rows_per_seq,
                                              stream_ptr()), "sq_top_p_filter_per_seq")
    return logits


def top_k_filter_per_seq_(logits, top_k, rows_per_seq: int):
    """top_k_filter_ in place on (n, V) fp16 logits whose row r belongs to sequence r // rows_per_seq, at that sequence's
    top_k[b] ((B,) int32 on the device); rows of a sequence with top_k <= 0 or >= V are left untouched."""
    _need(logits, F16, "top_k_filter_per_seq_")
    n, V = logits.shape
    B = n // rows_per_seq if rows_per_seq > 0 else 0
    if top_k is None or top_k.dtype != torch.int32 or not top_k.is_cuda or top_k.dim() != 1 or top_k.shape[0] < B \
            or top_k.stride(0) != 1:
        raise TypeError(f"top_k_filter_per_seq_: top_k must be a contiguous ({B},) int32 CUDA tensor")
    check(_lib.load().sq_top_k_filter_per_seq(ptr(logits), logits.stride(0), n, V, ptr(top_k), rows_per_seq,
                                              stream_ptr()), "sq_top_k_filter_per_seq")
    return logits


def min_p_filter_per_seq_(logits, log_min_p, T, rows_per_seq: int):
    """Min-p filter in place on (n, V) fp16 logits whose row r belongs to sequence b = r // rows_per_seq: a token keeps its
    logit when its probability at T[b] is at least min_p times the row's largest, else it becomes -inf (the exact rule in
    include/sequoia_b200.h).  log_min_p and T are (B,) float32 on the device, log_min_p[b] = fp32(ln min_p) or -inf (off:
    the rows are left untouched)."""
    _need(logits, F16, "min_p_filter_per_seq_")
    n, V = logits.shape
    B = n // rows_per_seq if rows_per_seq > 0 else 0
    _seq_params("min_p_filter_per_seq_", B, log_min_p=log_min_p, T=T)
    check(_lib.load().sq_min_p_filter_per_seq(ptr(logits), logits.stride(0), n, V, ptr(log_min_p), ptr(T), rows_per_seq,
                                              stream_ptr()), "sq_min_p_filter_per_seq")
    return logits


# ---- per-sequence counter-based random numbers (csrc/sq_rng.cu; stream layout in include/sequoia_b200.h) -------------------
RNG_R, RNG_RAND, RNG_NOISE = 0, 1, 2     # purposes: r (M), rand (S*V, node-major), bonus noise (V, one step per verify)


def _seeds(seeds, B, name):
    if seeds.dtype != torch.int64 or not seeds.is_cuda or seeds.dim() != 1 or seeds.shape[0] < B or seeds.stride(0) != 1:
        raise TypeError(f"{name}: seeds must be a contiguous ({B},) int64 CUDA tensor (the uint64 seeds' bits)")


def rng_uniform_seqs(out, seeds, slots, purpose: int):
    """Fill row b of `out` ((B, ...) fp16, each row contiguous) with the uniforms of `purpose` (RNG_R or RNG_RAND) of the
    stream keyed by seeds[b], for every slot b in `slots` (host list), in one launch.  seeds: (B,) int64 on the device."""
    _need(out, F16, "rng_uniform_seqs")
    B = out.shape[0]
    _seeds(seeds, B, "rng_uniform_seqs")
    row = out[0]
    if not row.is_contiguous():
        raise ValueError(f"rng_uniform_seqs: rows of out must be contiguous, got strides {tuple(out.stride())}")
    slots = [int(b) for b in slots]
    arr = (C.c_int32 * max(len(slots), 1))(*slots)
    check(_lib.load().sq_rng_uniform_seqs(ptr(out), out.stride(0), row.numel(), ptr(seeds), C.addressof(arr), len(slots),
                                          B, purpose, stream_ptr()), "sq_rng_uniform_seqs")
    return out


def rng_exponential_batch(noise, seeds, steps, state):
    """Row b of the (B, V) fp16 noise = the Exp(1) draws of step steps[b] of seeds[b]'s stream, for every sequence not
    frozen in `state`; then steps[b] += 1 on the device.  seeds, steps: (B,) int64 on the device."""
    _need(noise, F16, "rng_exponential_batch")
    B = state.shape[0]
    _seeds(seeds, B, "rng_exponential_batch")
    if steps.dtype != torch.int64 or not steps.is_cuda or steps.dim() != 1 or steps.shape[0] < B or steps.stride(0) != 1:
        raise TypeError(f"rng_exponential_batch: steps must be a contiguous ({B},) int64 CUDA tensor")
    if noise.shape[0] < B:
        raise ValueError(f"rng_exponential_batch: {noise.shape[0]} noise rows for {B} sequences")
    check(_lib.load().sq_rng_exponential_batch(ptr(noise), _rows(noise, "noise"), noise.shape[-1], ptr(seeds), ptr(steps),
                                               ptr(state), B, stream_ptr()), "sq_rng_exponential_batch")


def accept_greedy_batch(target_token, succ_off, succ, depth, S, tokens, position_ids, accept_idx, state, max_target_seq):
    """target_token (B*S) int64."""
    ld = _rows(tokens, "tokens")
    assert _rows(position_ids, "position_ids") == ld
    check(_lib.load().sq_accept_greedy_batch(ptr(target_token), ptr(succ_off), ptr(succ), ptr(depth), S, ptr(tokens),
                                             ptr(position_ids), ld, ptr(accept_idx), _rows(accept_idx, "accept_idx"),
                                             ptr(state), state.shape[0], max_target_seq, stream_ptr()),
          "sq_accept_greedy_batch")


# ---- per-sequence policy: greedy and sampled sequences in one batch (include/sequoia_b200.h) -----------------------------
def _greedy_arg(greedy, B, name):
    if greedy is None or greedy.dtype != torch.int32 or not greedy.is_cuda or greedy.dim() != 1 or greedy.shape[0] < B \
            or greedy.stride(0) != 1:
        raise TypeError(f"{name}: greedy must be a contiguous ({B},) int32 CUDA tensor (nonzero = greedy)")


def sample_level_batch_mixed(logits, row_base, row_step, rand, n_parents, k_max, T, greedy, *, parent_rows, child_first,
                             n_branch, tokens, state):
    """sample_level_batch_per_seq with sequence b drawing as mode 1 (top-k) when greedy[b] != 0, else as mode 0 at T[b].
    rand: (B, S, V), required (its rows of greedy sequences are not read)."""
    B = state.shape[0]
    _seq_params("sample_level_batch_mixed", B, T=T)
    _greedy_arg(greedy, B, "sample_level_batch_mixed")
    if rand is not None:
        assert rand.dim() == 3 and rand.stride(-1) == 1
    check(_lib.load().sq_sample_level_batch_mixed(
        ptr(logits), logits.stride(0), ptr(row_base), ptr(row_step), ptr(rand), rand.stride(1) if rand is not None else 0,
        rand.stride(0) if rand is not None else 0, ptr(parent_rows), ptr(child_first), ptr(n_branch), n_parents, k_max,
        logits.shape[-1], ptr(T), ptr(greedy), ptr(tokens), _rows(tokens, "tokens"), ptr(state), B, stream_ptr()),
        "sq_sample_level_batch_mixed")


def accept_greedy_batch_mixed(target_token, succ_off, succ, depth, S, greedy, tokens, position_ids, accept_idx, state,
                              max_target_seq):
    """accept_greedy_batch for the sequences with greedy[b] != 0 only."""
    B = state.shape[0]
    _greedy_arg(greedy, B, "accept_greedy_batch_mixed")
    ld = _rows(tokens, "tokens")
    assert _rows(position_ids, "position_ids") == ld
    check(_lib.load().sq_accept_greedy_batch_mixed(ptr(target_token), ptr(succ_off), ptr(succ), ptr(depth), S, ptr(tokens),
                                                   ptr(position_ids), ld, ptr(accept_idx), _rows(accept_idx, "accept_idx"),
                                                   ptr(state), ptr(greedy), B, max_target_seq, stream_ptr()),
          "sq_accept_greedy_batch_mixed")


def accept_stochastic_batch_mixed(target_logits, draft_logits, row_base, row_step, r, noise, succ_off, succ, depth, S, T,
                                  greedy, tokens, position_ids, accept_idx, state, max_target_seq, policy=0):
    """accept_stochastic_batch_per_seq for the sequences with greedy[b] == 0 only."""
    B = state.shape[0]
    _seq_params("accept_stochastic_batch_mixed", B, T=T)
    _greedy_arg(greedy, B, "accept_stochastic_batch_mixed")
    V = target_logits.shape[-1]
    ld = _rows(tokens, "tokens")
    assert _rows(position_ids, "position_ids") == ld and _rows(r, "r") == ld
    check(_lib.load().sq_accept_stochastic_batch_mixed(
        ptr(target_logits), target_logits.stride(0), ptr(draft_logits), draft_logits.stride(0), ptr(row_base),
        ptr(row_step), ptr(r), ptr(noise), _rows(noise, "noise"), ptr(succ_off), ptr(succ), ptr(depth), S, V, ptr(T),
        ptr(greedy), ptr(tokens), ptr(position_ids), ld, ptr(accept_idx), _rows(accept_idx, "accept_idx"), ptr(state), B,
        max_target_seq, policy, stream_ptr()), "sq_accept_stochastic_batch_mixed")


# ---- stop mode: per-sequence stop ids and length limits, applied by the walks (include/sequoia_b200.h) -------------------
def _stop_args(stop_ids, end_limit, B, name):
    if stop_ids is None or stop_ids.dtype != torch.int32 or not stop_ids.is_cuda or stop_ids.dim() != 2 \
            or stop_ids.shape[0] < B or stop_ids.shape[1] != _lib.SQ_MAX_STOP or not stop_ids.is_contiguous():
        raise TypeError(f"{name}: stop_ids must be a contiguous ({B}, {_lib.SQ_MAX_STOP}) int32 CUDA tensor (-1 = unused)")
    if end_limit is None or end_limit.dtype != torch.int32 or not end_limit.is_cuda or end_limit.dim() != 1 \
            or end_limit.shape[0] < B or end_limit.stride(0) != 1:
        raise TypeError(f"{name}: end_limit must be a contiguous ({B},) int32 CUDA tensor (<= 0 = no limit)")


def accept_stochastic_batch_stop(target_logits, draft_logits, row_base, row_step, r, noise, succ_off, succ, depth, S, T,
                                 greedy, stop_ids, end_limit, tokens, position_ids, accept_idx, state, max_target_seq,
                                 policy=0):
    """accept_stochastic_batch_per_seq (greedy None) or accept_stochastic_batch_mixed (greedy set) without the fixed 0 / 2
    end rule; then each walked sequence's committed tokens are cut at its stop ids (stop_ids (B, 8) int32, -1 padded) and
    its absolute length limit (end_limit (B,) int32, <= 0 = none): state words SQ_ST_FINISH / SQ_ST_END."""
    B = state.shape[0]
    _seq_params("accept_stochastic_batch_stop", B, T=T)
    if greedy is not None:
        _greedy_arg(greedy, B, "accept_stochastic_batch_stop")
    _stop_args(stop_ids, end_limit, B, "accept_stochastic_batch_stop")
    V = target_logits.shape[-1]
    ld = _rows(tokens, "tokens")
    assert _rows(position_ids, "position_ids") == ld and _rows(r, "r") == ld
    check(_lib.load().sq_accept_stochastic_batch_stop(
        ptr(target_logits), target_logits.stride(0), ptr(draft_logits), draft_logits.stride(0), ptr(row_base),
        ptr(row_step), ptr(r), ptr(noise), _rows(noise, "noise"), ptr(succ_off), ptr(succ), ptr(depth), S, V, ptr(T),
        ptr(greedy), ptr(stop_ids), ptr(end_limit), ptr(tokens), ptr(position_ids), ld, ptr(accept_idx),
        _rows(accept_idx, "accept_idx"), ptr(state), B, max_target_seq, policy, stream_ptr()),
        "sq_accept_stochastic_batch_stop")


def accept_greedy_batch_stop(target_token, succ_off, succ, depth, S, greedy, stop_ids, end_limit, tokens, position_ids,
                             accept_idx, state, max_target_seq):
    """accept_greedy_batch (greedy None) or accept_greedy_batch_mixed (greedy set) with the stop rule of
    accept_stochastic_batch_stop."""
    B = state.shape[0]
    if greedy is not None:
        _greedy_arg(greedy, B, "accept_greedy_batch_stop")
    _stop_args(stop_ids, end_limit, B, "accept_greedy_batch_stop")
    ld = _rows(tokens, "tokens")
    assert _rows(position_ids, "position_ids") == ld
    check(_lib.load().sq_accept_greedy_batch_stop(ptr(target_token), ptr(succ_off), ptr(succ), ptr(depth), S, ptr(tokens),
                                                  ptr(position_ids), ld, ptr(accept_idx), _rows(accept_idx, "accept_idx"),
                                                  ptr(state), ptr(greedy), ptr(stop_ids), ptr(end_limit), B,
                                                  max_target_seq, stream_ptr()), "sq_accept_greedy_batch_stop")


# ---- per-sequence repetition / frequency / presence penalties (csrc/sq_penalty.cu; semantics in include/sequoia_b200.h) --
def penalty_scratch_words(B: int, ld_seq: int) -> int:
    """int32 words of the scratch penalize_rows_batch_ needs: a distinct-id list of ld_seq entries per sequence."""
    return B * (3 * ld_seq + 1)


def penalize_rows_batch_(logits, tokens, state, prompt_len, tree_bits, tree_words: int, S: int, rep, freq, pres,
                         scratch):
    """Apply sequence b's repetition (rep[b]), frequency (freq[b]) and presence (pres[b]) penalties in place to its S
    target rows b*S .. b*S+S-1 of the (>= B*S, V) fp16 logits: row b*S + k counts the committed tokens[b, :P] and the tokens
    of node k's ancestors-or-self on the tree (tree_bits), output from slot prompt_len[b] on.  rep, freq, pres: (B,) float32
    and prompt_len: (B,) int32 on the device; tokens (B, ld_seq) int64; scratch: int32 of penalty_scratch_words(B, ld_seq).
    Frozen sequences and sequences with rep = 1, freq = 0, pres = 0 are left untouched."""
    _need(logits, F16, "penalize_rows_batch_")
    if logits.dim() != 2 or logits.stride(-1) != 1:
        raise ValueError(f"penalize_rows_batch_: logits must be (rows, V) with contiguous rows, got {tuple(logits.shape)}")
    B = state.shape[0]
    if logits.shape[0] < B * S:
        raise ValueError(f"penalize_rows_batch_: {logits.shape[0]} logit rows for {B} sequences of {S}")
    _seq_params("penalize_rows_batch_", B, rep=rep, freq=freq, pres=pres)
    if prompt_len is None or prompt_len.dtype != torch.int32 or not prompt_len.is_cuda or prompt_len.dim() != 1 \
            or prompt_len.shape[0] < B or prompt_len.stride(0) != 1:
        raise TypeError(f"penalize_rows_batch_: prompt_len must be a contiguous ({B},) int32 CUDA tensor")
    _need(tokens, torch.int64, "penalize_rows_batch_")
    _need(state, torch.int32, "penalize_rows_batch_")
    _need(tree_bits, torch.int32, "penalize_rows_batch_")
    _need(scratch, torch.int32, "penalize_rows_batch_")
    if not tree_bits.is_contiguous() or not scratch.is_contiguous() or not state.is_contiguous():
        raise ValueError("penalize_rows_batch_: tree_bits, scratch and state must be contiguous")
    if tokens.shape[0] < B:
        raise ValueError(f"penalize_rows_batch_: {tokens.shape[0]} token rows for {B} sequences")
    check(_lib.load().sq_penalize_rows_batch(ptr(logits), logits.stride(0), logits.shape[1], ptr(tokens),
                                             _rows(tokens, "tokens"), ptr(state), ptr(prompt_len), ptr(tree_bits),
                                             tree_words, S, ptr(rep), ptr(freq), ptr(pres), ptr(scratch), scratch.numel(),
                                             B, stream_ptr()), "sq_penalize_rows_batch")
    return logits


# ---- per-sequence logprobs of the committed tokens (csrc/sq_logprobs.cu; semantics in include/sequoia_b200.h) -----------
def token_logprobs_batch_(target_logits, S: int, max_depth: int, tokens, state, accept_idx, T, greedy, n_top, lp_token,
                          lp_ids, lp_top):
    """After the walk: for each sequence b with n_top[b] >= 0 that is not frozen, the logprob of every token the step
    committed (positions state[b, P_OLD] + j, j <= the path depth, the bonus included) into lp_token[b, pos], and the
    min(n_top[b], 20) best ids of its target row with their logprobs into lp_ids / lp_top[b, pos, :n].  target_logits:
    (>= B*S, V) fp16 as the walk read it (row b*S + k = node k of sequence b); T: (B,) float32, greedy / n_top: (B,) int32
    on the device; tokens: (B, M) int64; accept_idx: (B, >= max_depth) int32; lp_token: (B, M) float32; lp_ids: (B, M, 20)
    int32; lp_top: (B, M, 20) float32.  Nothing else of the outputs is written."""
    name = "token_logprobs_batch_"
    _need(target_logits, F16, name)
    if target_logits.dim() != 2 or target_logits.stride(-1) != 1:
        raise ValueError(f"{name}: target_logits must be (rows, V) with contiguous rows, got {tuple(target_logits.shape)}")
    _need(tokens, torch.int64, name)
    _need(state, torch.int32, name)
    _need(accept_idx, torch.int32, name)
    if not state.is_contiguous():
        raise ValueError(f"{name}: state must be contiguous")
    B = state.shape[0]
    if target_logits.shape[0] < B * S:
        raise ValueError(f"{name}: {target_logits.shape[0]} logit rows for {B} sequences of {S}")
    _seq_params(name, B, T=T)
    for k, t in (("greedy", greedy), ("n_top", n_top)):
        if t is None or t.dtype != torch.int32 or not t.is_cuda or t.dim() != 1 or t.shape[0] < B or t.stride(0) != 1:
            raise TypeError(f"{name}: {k} must be a contiguous ({B},) int32 CUDA tensor")
    M = tokens.shape[1] if tokens.dim() == 2 else -1
    if tokens.dim() != 2 or tokens.shape[0] < B or accept_idx.dim() != 2 or accept_idx.shape[0] < B:
        raise ValueError(f"{name}: tokens and accept_idx must be (B, ...) with B = {B}")
    for k, t, dt, shape in (("lp_token", lp_token, torch.float32, (B, M)),
                            ("lp_ids", lp_ids, torch.int32, (B, M, _lib.SQ_MAX_LOGPROBS)),
                            ("lp_top", lp_top, torch.float32, (B, M, _lib.SQ_MAX_LOGPROBS))):
        _need(t, dt, name)
        if tuple(t.shape) != shape or not t.is_contiguous():
            raise ValueError(f"{name}: {k} must be a contiguous {shape} tensor, got {tuple(t.shape)}")
    check(_lib.load().sq_token_logprobs_batch(ptr(target_logits), target_logits.stride(0), target_logits.shape[1], S,
                                              max_depth, ptr(tokens), _rows(tokens, "tokens"), ptr(state), ptr(accept_idx),
                                              _rows(accept_idx, "accept_idx"), ptr(T), ptr(greedy), ptr(n_top),
                                              ptr(lp_token), ptr(lp_ids), ptr(lp_top), B, stream_ptr()),
          "sq_token_logprobs_batch")


class PromptLpPart(C.Structure):
    """sq_prompt_lp_part: rows [0, n_rows) of sequence seq's prompt scores, on logits rows logits_row0 + r, n_top best"""
    _fields_ = [("seq", C.c_int32), ("logits_row0", C.c_int32), ("n_rows", C.c_int32), ("n_top", C.c_int32)]


def prompt_logprobs_ragged_(logits, parts, tokens, plp_token, plp_ids, plp_top):
    """Prompt logprobs at T = 1 for the listed sequences, one launch: parts is (seq, logits_row0, n_rows, n_top) per
    sequence; row r of a part (logits row logits_row0 + r, the prediction after prompt tokens 0 .. r) scores tokens[seq,
    r + 1] into plp_token[seq, r + 1], and its min(n_top, V) best ids with their logprobs into plp_ids / plp_top[seq, r + 1,
    :n].  logits: (rows, V) fp16 with contiguous rows; tokens: (B, M) int64; plp_token: (B, M) float32; plp_ids: (B, M, 20)
    int32; plp_top: (B, M, 20) float32.  Nothing else of the outputs is written."""
    name = "prompt_logprobs_ragged_"
    _need(logits, F16, name)
    if logits.dim() != 2 or logits.stride(-1) != 1:
        raise ValueError(f"{name}: logits must be (rows, V) with contiguous rows, got {tuple(logits.shape)}")
    _need(tokens, torch.int64, name)
    if tokens.dim() != 2:
        raise ValueError(f"{name}: tokens must be (B, M), got {tuple(tokens.shape)}")
    B, M = tokens.shape
    for k, t, dt, shape in (("plp_token", plp_token, torch.float32, (B, M)),
                            ("plp_ids", plp_ids, torch.int32, (B, M, _lib.SQ_MAX_LOGPROBS)),
                            ("plp_top", plp_top, torch.float32, (B, M, _lib.SQ_MAX_LOGPROBS))):
        _need(t, dt, name)
        if tuple(t.shape) != shape or not t.is_contiguous():
            raise ValueError(f"{name}: {k} must be a contiguous {shape} tensor, got {tuple(t.shape)}")
    arr = (PromptLpPart * len(parts))(*[tuple(int(x) for x in p) for p in parts])
    check(_lib.load().sq_prompt_logprobs_ragged(ptr(logits), logits.stride(0), logits.shape[1], logits.shape[0],
                                                C.addressof(arr), len(arr), ptr(tokens), _rows(tokens, "tokens"),
                                                ptr(plp_token), ptr(plp_ids), ptr(plp_top), B, stream_ptr()),
          "sq_prompt_logprobs_ragged")


# ---- per-sequence allowed-token mask and logit bias (csrc/sq_logit_bias.cu; semantics in include/sequoia_b200.h) ----------
def mask_words(V: int) -> int:
    """int32 words of one allowed-token bitmask row: ceil(V / 32)."""
    return (V + 31) // 32


def pack_token_mask(ids, V: int) -> torch.Tensor:
    """The (mask_words(V),) int32 bitmask of a collection of ids in [0, V) on the host: bit t & 31 of word t >> 5 set for
    every id t; the padding bits from V on are clear."""
    words = mask_words(V)
    bits = torch.zeros(words * 32, dtype=torch.bool)
    bits[torch.as_tensor(list(ids), dtype=torch.int64)] = True
    w = (bits.view(words, 32).to(torch.int64) << torch.arange(32, dtype=torch.int64)).sum(1)
    return torch.where(w >= 1 << 31, w - (1 << 32), w).to(torch.int32)


def logit_bias_rows_batch_(logits, S: int, state, allowed, has_mask, bias_ids, bias_vals, n_bias):
    """Apply sequence b's allowed-token mask (when has_mask[b]) and then its logit bias entries in place to its S target
    rows b*S .. b*S+S-1 of the (>= B*S, V) fp16 logits.  allowed: (B, >= mask_words(V)) int32 bitmask rows; has_mask,
    n_bias: (B,) int32; bias_ids / bias_vals: (B, SQ_MAX_LOGIT_BIAS) int32 / float32, each row's first n_bias[b] ids
    ascending; all on the device.  Frozen sequences and sequences with no mask and no entries are left untouched."""
    name = "logit_bias_rows_batch_"
    _need(logits, F16, name)
    if logits.dim() != 2 or logits.stride(-1) != 1:
        raise ValueError(f"{name}: logits must be (rows, V) with contiguous rows, got {tuple(logits.shape)}")
    _need(state, torch.int32, name)
    if not state.is_contiguous():
        raise ValueError(f"{name}: state must be contiguous")
    B = state.shape[0]
    if logits.shape[0] < B * S:
        raise ValueError(f"{name}: {logits.shape[0]} logit rows for {B} sequences of {S}")
    for k, t in (("has_mask", has_mask), ("n_bias", n_bias)):
        if t is None or t.dtype != torch.int32 or not t.is_cuda or t.dim() != 1 or t.shape[0] < B or t.stride(0) != 1:
            raise TypeError(f"{name}: {k} must be a contiguous ({B},) int32 CUDA tensor")
    nmax = _lib.SQ_MAX_LOGIT_BIAS
    for k, t, dt, cols in (("allowed", allowed, torch.int32, mask_words(logits.shape[1])),
                           ("bias_ids", bias_ids, torch.int32, nmax), ("bias_vals", bias_vals, torch.float32, nmax)):
        _need(t, dt, name)
        if t.dim() != 2 or t.shape[0] < B or t.shape[1] < cols or not t.is_contiguous():
            raise ValueError(f"{name}: {k} must be a contiguous ({B}, >= {cols}) tensor, got {tuple(t.shape)}")
    if bias_ids.shape[1] != nmax or bias_vals.shape[1] != nmax:
        raise ValueError(f"{name}: bias_ids and bias_vals must have {nmax} columns")
    check(_lib.load().sq_logit_bias_rows_batch(ptr(logits), logits.stride(0), logits.shape[1], S, ptr(state), ptr(allowed),
                                               allowed.shape[1], ptr(has_mask), ptr(bias_ids), ptr(bias_vals),
                                               ptr(n_bias), B, stream_ptr()), "sq_logit_bias_rows_batch")
    return logits


# ---- per-sequence bad words and min_tokens (csrc/sq_ban.cu; semantics in include/sequoia_b200.h) ---------------------
def ban_tokens_rows_batch_(logits, tokens, state, prompt_len, depth, tree_bits, tree_words: int, S: int, words, word_len,
                           n_words, min_end, end_ids):
    """Write -inf in place at the banned ids of sequence b's S target rows b*S .. b*S+S-1 of the (>= B*S, V) fp16 logits:
    the last id of each bad word whose prefix ends the row's generated context (the committed tokens from slot
    prompt_len[b] on, then node k's path on the tree), and the end ids while the row's position P + depth[k] is below
    min_end[b].  words: (B, SQ_MAX_BAD_WORDS, SQ_MAX_BAD_WORD_LEN) int32; word_len: (B, SQ_MAX_BAD_WORDS) int32; n_words,
    min_end, prompt_len: (B,) int32; end_ids: (B, SQ_MAX_STOP) int32, -1 padded; depth: (S,) int32; all on the device.
    Frozen sequences and sequences with no words and min_end 0 are left untouched."""
    name = "ban_tokens_rows_batch_"
    _need(logits, F16, name)
    if logits.dim() != 2 or logits.stride(-1) != 1:
        raise ValueError(f"{name}: logits must be (rows, V) with contiguous rows, got {tuple(logits.shape)}")
    _need(state, torch.int32, name)
    _need(tokens, torch.int64, name)
    _need(tree_bits, torch.int32, name)
    if not state.is_contiguous() or not tree_bits.is_contiguous():
        raise ValueError(f"{name}: state and tree_bits must be contiguous")
    B = state.shape[0]
    if logits.shape[0] < B * S:
        raise ValueError(f"{name}: {logits.shape[0]} logit rows for {B} sequences of {S}")
    if tokens.shape[0] < B:
        raise ValueError(f"{name}: {tokens.shape[0]} token rows for {B} sequences")
    for k, t, n in (("prompt_len", prompt_len, B), ("n_words", n_words, B), ("min_end", min_end, B), ("depth", depth, S)):
        if t is None or t.dtype != torch.int32 or not t.is_cuda or t.dim() != 1 or t.shape[0] < n or t.stride(0) != 1:
            raise TypeError(f"{name}: {k} must be a contiguous ({n},) int32 CUDA tensor")
    nw, wl, ns = _lib.SQ_MAX_BAD_WORDS, _lib.SQ_MAX_BAD_WORD_LEN, _lib.SQ_MAX_STOP
    for k, t, shape in (("words", words, (nw, wl)), ("word_len", word_len, (nw,)), ("end_ids", end_ids, (ns,))):
        _need(t, torch.int32, name)
        if tuple(t.shape[1:]) != shape or t.shape[0] < B or not t.is_contiguous():
            raise ValueError(f"{name}: {k} must be a contiguous ({B}, {', '.join(map(str, shape))}) tensor, got "
                             f"{tuple(t.shape)}")
    check(_lib.load().sq_ban_tokens_rows_batch(ptr(logits), logits.stride(0), logits.shape[1], ptr(tokens),
                                               _rows(tokens, "tokens"), ptr(state), ptr(prompt_len), ptr(depth),
                                               ptr(tree_bits), tree_words, S, ptr(words), ptr(word_len), ptr(n_words),
                                               ptr(min_end), ptr(end_ids), B, stream_ptr()), "sq_ban_tokens_rows_batch")
    return logits


# ---- guided decoding: per-sequence token automata (csrc/sq_guide.cu; semantics in include/sequoia_b200.h) ----------------
def _guide_table(guide_table, B, name):
    if guide_table is None or guide_table.dtype != torch.int64 or not guide_table.is_cuda or guide_table.dim() != 1 \
            or guide_table.shape[0] < B or guide_table.stride(0) != 1:
        raise TypeError(f"{name}: guide_table must be a contiguous ({B},) int64 CUDA tensor of guide blob addresses")


def guide_states_batch(guide_table, tokens, state, depth, tree_bits, tree_words: int, S: int, V: int, node_state):
    """node_state[b, k] = the guide state of node k of every guided sequence b: its committed state (state word
    SQ_ST_GUIDE_STATE) walked through the tokens of node k's path on the tree (tree_bits), -1 from a disallowed id on.
    guide_table: (B,) int64 blob addresses (0 = none); tokens (B, ld_seq) int64; depth (S,) int32; node_state (B, S)
    int32; all on the device.  Unguided and frozen sequences' entries are not written."""
    name = "guide_states_batch"
    _need(state, torch.int32, name)
    _need(tokens, torch.int64, name)
    _need(tree_bits, torch.int32, name)
    _need(node_state, torch.int32, name)
    if not state.is_contiguous() or not tree_bits.is_contiguous():
        raise ValueError(f"{name}: state and tree_bits must be contiguous")
    B = state.shape[0]
    _guide_table(guide_table, B, name)
    if tokens.shape[0] < B:
        raise ValueError(f"{name}: {tokens.shape[0]} token rows for {B} sequences")
    if depth is None or depth.dtype != torch.int32 or not depth.is_cuda or depth.dim() != 1 or depth.shape[0] < S \
            or depth.stride(0) != 1:
        raise TypeError(f"{name}: depth must be a contiguous ({S},) int32 CUDA tensor")
    if tuple(node_state.shape) != (B, S) or not node_state.is_contiguous():
        raise ValueError(f"{name}: node_state must be a contiguous ({B}, {S}) tensor, got {tuple(node_state.shape)}")
    check(_lib.load().sq_guide_states_batch(ptr(guide_table), ptr(tokens), _rows(tokens, "tokens"), ptr(state),
                                            ptr(depth), ptr(tree_bits), tree_words, S, V, ptr(node_state), B,
                                            stream_ptr()), "sq_guide_states_batch")
    return node_state


def guide_mask_rows_batch_(logits, S: int, state, guide_table, node_state):
    """Write -inf in place at every id the node's guide state does not allow (every id for a dead node, -1) in the S
    target rows b*S .. b*S+S-1 of every guided sequence b of the (>= B*S, V) fp16 logits; allowed entries are not
    touched.  node_state: (B, S) int32 from guide_states_batch."""
    name = "guide_mask_rows_batch_"
    _need(logits, F16, name)
    if logits.dim() != 2 or logits.stride(-1) != 1:
        raise ValueError(f"{name}: logits must be (rows, V) with contiguous rows, got {tuple(logits.shape)}")
    _need(state, torch.int32, name)
    _need(node_state, torch.int32, name)
    if not state.is_contiguous():
        raise ValueError(f"{name}: state must be contiguous")
    B = state.shape[0]
    _guide_table(guide_table, B, name)
    if logits.shape[0] < B * S:
        raise ValueError(f"{name}: {logits.shape[0]} logit rows for {B} sequences of {S}")
    if tuple(node_state.shape) != (B, S) or not node_state.is_contiguous():
        raise ValueError(f"{name}: node_state must be a contiguous ({B}, {S}) tensor, got {tuple(node_state.shape)}")
    check(_lib.load().sq_guide_mask_rows_batch(ptr(logits), logits.stride(0), logits.shape[1], S, ptr(state),
                                               ptr(guide_table), ptr(node_state), B, stream_ptr()),
          "sq_guide_mask_rows_batch")
    return logits


def guide_advance_batch(guide_table, tokens, state, V: int):
    """After the walk: move every guided sequence's committed guide state (state word SQ_ST_GUIDE_STATE) through the
    tokens the step committed, from position SQ_ST_GUIDE_POS on; a disallowed id kills it (-1) and leaves its position in
    SQ_ST_GUIDE_POS."""
    name = "guide_advance_batch"
    _need(state, torch.int32, name)
    _need(tokens, torch.int64, name)
    if not state.is_contiguous():
        raise ValueError(f"{name}: state must be contiguous")
    B = state.shape[0]
    _guide_table(guide_table, B, name)
    if tokens.shape[0] < B:
        raise ValueError(f"{name}: {tokens.shape[0]} token rows for {B} sequences")
    check(_lib.load().sq_guide_advance_batch(ptr(guide_table), ptr(tokens), _rows(tokens, "tokens"), ptr(state), V, B,
                                             stream_ptr()), "sq_guide_advance_batch")


# ---- constrained drafting: the target-row processing on draft rows (csrc/sq_draft_rows.cu; include/sequoia_b200.h) ----
def draft_rows_batch_(draft_logits, row_base, row_step, k0: int, nk: int, S: int, state, *, bias=None, ban=None,
                      guide=None, tokens=None, tree_bits=None, tree_words: int = 0):
    """Apply, in place, sequence b's allowed set and logit bias, bad words and min_tokens, and guide mask to the draft rows
    of nodes [k0, k0 + nk) (row row_base[k] + b * row_step[k] of the fp16 draft logits), exactly as logit_bias_rows_batch_,
    ban_tokens_rows_batch_ and guide_mask_rows_batch_ process target row k.  Each kind is None (not applied) or a tuple:
      bias  = (allowed, has_mask, bias_ids, bias_vals, n_bias)                    as logit_bias_rows_batch_ takes them;
      ban   = (prompt_len, depth, words, word_len, n_words, min_end, end_ids)    as ban_tokens_rows_batch_ takes them;
      guide = (guide_table, node_state): node_state (B, S) int32 holds the parents' states from earlier calls and
              receives the states of nodes [k0, k0 + nk).
    tokens (B, ld_seq) int64 and tree_bits / tree_words are needed by ban and guide.  The node range is the root alone
    (0, 1) or a range in [1, S) whose nodes' parents lie below k0."""
    name = "draft_rows_batch_"
    _need(draft_logits, F16, name)
    if draft_logits.dim() != 2 or draft_logits.stride(-1) != 1:
        raise ValueError(f"{name}: draft_logits must be (rows, V) with contiguous rows, got {tuple(draft_logits.shape)}")
    _need(state, torch.int32, name)
    if not state.is_contiguous():
        raise ValueError(f"{name}: state must be contiguous")
    B, V = state.shape[0], draft_logits.shape[1]
    for k, t in (("row_base", row_base), ("row_step", row_step)):
        if t is None or t.dtype != torch.int32 or not t.is_cuda or t.dim() != 1 or t.shape[0] < S or t.stride(0) != 1:
            raise TypeError(f"{name}: {k} must be a contiguous ({S},) int32 CUDA tensor")
    flags = 0
    args_bias = [None, 0, None, None, None, None]
    if bias is not None:
        flags |= _lib.SQ_DRAFT_BIAS
        allowed, has_mask, bias_ids, bias_vals, n_bias = bias
        _need(allowed, torch.int32, name)
        if allowed.dim() != 2 or allowed.shape[0] < B or allowed.shape[1] < mask_words(V) or not allowed.is_contiguous():
            raise ValueError(f"{name}: allowed must be a contiguous ({B}, >= {mask_words(V)}) tensor")
        for k, t, dt in (("has_mask", has_mask, torch.int32), ("n_bias", n_bias, torch.int32)):
            if t is None or t.dtype != dt or not t.is_cuda or t.dim() != 1 or t.shape[0] < B or t.stride(0) != 1:
                raise TypeError(f"{name}: {k} must be a contiguous ({B},) int32 CUDA tensor")
        nmax = _lib.SQ_MAX_LOGIT_BIAS
        for k, t, dt in (("bias_ids", bias_ids, torch.int32), ("bias_vals", bias_vals, torch.float32)):
            _need(t, dt, name)
            if t.dim() != 2 or t.shape[0] < B or t.shape[1] != nmax or not t.is_contiguous():
                raise ValueError(f"{name}: {k} must be a contiguous ({B}, {nmax}) tensor")
        args_bias = [ptr(allowed), allowed.shape[1], ptr(has_mask), ptr(bias_ids), ptr(bias_vals), ptr(n_bias)]
    args_ban = [None] * 7
    if ban is not None:
        flags |= _lib.SQ_DRAFT_BAN
        prompt_len, depth, words, word_len, n_words, min_end, end_ids = ban
        for k, t, n in (("prompt_len", prompt_len, B), ("n_words", n_words, B), ("min_end", min_end, B),
                        ("depth", depth, S)):
            if t is None or t.dtype != torch.int32 or not t.is_cuda or t.dim() != 1 or t.shape[0] < n or t.stride(0) != 1:
                raise TypeError(f"{name}: {k} must be a contiguous ({n},) int32 CUDA tensor")
        nw, wl, ns = _lib.SQ_MAX_BAD_WORDS, _lib.SQ_MAX_BAD_WORD_LEN, _lib.SQ_MAX_STOP
        for k, t, shape in (("words", words, (nw, wl)), ("word_len", word_len, (nw,)), ("end_ids", end_ids, (ns,))):
            _need(t, torch.int32, name)
            if tuple(t.shape[1:]) != shape or t.shape[0] < B or not t.is_contiguous():
                raise ValueError(f"{name}: {k} must be a contiguous ({B}, {', '.join(map(str, shape))}) tensor")
        args_ban = [ptr(prompt_len), ptr(depth), ptr(words), ptr(word_len), ptr(n_words), ptr(min_end), ptr(end_ids)]
    args_guide = [None, None]
    if guide is not None:
        flags |= _lib.SQ_DRAFT_GUIDE
        guide_table, node_state = guide
        _guide_table(guide_table, B, name)
        _need(node_state, torch.int32, name)
        if tuple(node_state.shape) != (B, S) or not node_state.is_contiguous():
            raise ValueError(f"{name}: node_state must be a contiguous ({B}, {S}) tensor")
        args_guide = [ptr(guide_table), ptr(node_state)]
    ld_seq = 0
    if ban is not None or guide is not None:
        _need(tokens, torch.int64, name)
        _need(tree_bits, torch.int32, name)
        if tokens.shape[0] < B or not tree_bits.is_contiguous():
            raise ValueError(f"{name}: tokens must hold {B} rows and tree_bits must be contiguous")
        ld_seq = _rows(tokens, "tokens")
    check(_lib.load().sq_draft_rows_batch(
        ptr(draft_logits), draft_logits.stride(0), V, ptr(row_base), ptr(row_step), k0, nk, S, ptr(state), flags,
        *args_bias, ptr(tokens) if ld_seq else None, ld_seq, ptr(tree_bits) if ld_seq else None, tree_words, *args_ban,
        *args_guide, B, stream_ptr()), "sq_draft_rows_batch")
    return draft_logits
