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


def argmax_rows(logits, out=None):
    n, V = logits.shape
    if out is None:
        out = torch.empty(n, dtype=torch.int64, device=logits.device)
    check(_lib.load().sq_argmax_rows(ptr(logits), logits.stride(0), n, V, ptr(out), stream_ptr()), "sq_argmax_rows")
    return out


ACCEPT_GE, ACCEPT_KEEP_Q = 1, 2          # sq_accept_stochastic policy bits (include/sequoia_b200.h)


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


def tree_attn_batch(plan: AttnPlan, layer, n, *, state, n0=0, kv_end=0, tree_bits=None, tree_words=0, tree_size=0):
    check(_lib.load().sq_tree_attn_batch(plan.handle, layer, n, state.shape[0], ptr(state), n0, kv_end, ptr(tree_bits),
                                         tree_words, tree_size, stream_ptr()), "sq_tree_attn_batch")


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


def accept_greedy_batch(target_token, succ_off, succ, depth, S, tokens, position_ids, accept_idx, state, max_target_seq):
    """target_token (B*S) int64."""
    ld = _rows(tokens, "tokens")
    assert _rows(position_ids, "position_ids") == ld
    check(_lib.load().sq_accept_greedy_batch(ptr(target_token), ptr(succ_off), ptr(succ), ptr(depth), S, ptr(tokens),
                                             ptr(position_ids), ld, ptr(accept_idx), _rows(accept_idx, "accept_idx"),
                                             ptr(state), state.shape[0], max_target_seq, stream_ptr()),
          "sq_accept_greedy_batch")
