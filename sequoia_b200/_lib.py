"""ctypes binding of libsequoia_b200.so (the C ABI declared in include/sequoia_b200.h).

The product path has NO fallback: if the shared library is missing or a call fails, an exception
is raised.  Build with ``python -c "import __graft_entry__ as g; g.build()"`` (or ``make -C
sequoia_b200/csrc``).
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsequoia_b200.so")

_lib = None

i32, i64, f32, vp = C.c_int, C.c_int64, C.c_float, C.c_void_p

_SIGNATURES = {
    "sq_last_error": (C.c_char_p, []),
    "sq_version": (i32, []),
    "sq_launch_count": (C.c_uint64, []),
    "sq_embed_rows": (i32, [vp, vp, vp, i32, i32, i32, vp, vp]),
    "sq_rmsnorm": (i32, [vp, vp, vp, i32, i32, f32, vp]),
    "sq_add_rmsnorm": (i32, [vp, vp, vp, vp, i32, i32, f32, vp]),
    "sq_silu_mul": (i32, [vp, vp, i32, i32, vp]),
    "sq_silu_mul_ex": (i32, [vp, vp, i32, i32, i32, vp]),
    "sq_rope_kv_append": (i32, [vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, i32, i32, vp, vp, i32, vp]),
    "sq_kv_gather": (i32, [vp, vp, i32, i32, i32, i32, vp, i32, i32, vp, i32, i32, vp]),
    "sq_kv_gather_scratch_bytes": (i64, [i32, i32, i32, i32]),
    "sq_kv_gather_big": (i32, [vp, vp, i32, i32, i32, i32, vp, i32, i32, vp, i64, i32, vp]),
    "sq_attn_workspace_bytes": (i64, [i32, i32, i32, i32]),
    "sq_attn_plan_create": (i32, [C.POINTER(vp), vp, i32, i32, i32, i32, i32, vp, vp, i32, i32, vp, vp, i64]),
    "sq_attn_plan_destroy": (i32, [vp]),
    "sq_attn_plan_error": (i32, [vp]),
    "sq_attn_plan_info": (i32, [vp, C.POINTER(i32), C.POINTER(i32)]),
    "sq_attn_plan_debug_times": (i32, [vp, vp]),
    "sq_tree_attn": (i32, [vp, i32, i32, vp, i32, i32, i32, vp, i64, vp, i32, i32, i32, vp]),
    "sq_softmax_T": (i32, [vp, i64, vp, i64, i32, i32, f32, vp]),
    "sq_sample_level": (i32, [vp, i64, vp, i64, vp, vp, vp, i32, i32, i32, f32, i32, vp, vp, vp, vp]),
    "sq_sample_replace": (i32, [vp, i64, vp, vp, vp, vp, i32, i32, i32, f32, vp, vp, vp, vp]),
    "sq_residual": (i32, [vp, vp, vp, i32, vp]),
    "sq_argmax_rows": (i32, [vp, i64, i32, i32, vp, vp]),
    "sq_top_p_filter": (i32, [vp, i64, i32, i32, f32, f32, vp]),
    "sq_accept_stochastic": (i32, [vp, i64, vp, i64, vp, vp, vp, vp, vp, i32, i32, f32, vp, vp, vp, vp, i32, i32, vp]),
    "sq_accept_greedy": (i32, [vp, vp, vp, vp, i32, vp, vp, vp, vp, i32, vp]),
    "sq_gemm_plan_create": (i32, [C.POINTER(vp), vp, i32, i32, vp, i32, i32, vp, i32, vp]),
    "sq_gemm_pick_tiles": (i32, [i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]),
    "sq_gemm_pick_tiles_ex": (i32, [i32, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]),
    "sq_gemm_plan_create_ex": (i32, [C.POINTER(vp), vp, i32, i32, vp, i32, i32, vp, i32, vp, i32]),
    "sq_gemm_plan_create_tiled": (i32, [C.POINTER(vp), vp, i32, i32, vp, i32, i32, vp, i32, vp]),
    "sq_gemm_plan_set_epilogue": (i32, [vp, i32, i32]),
    "sq_gemm_plan_destroy": (i32, [vp]),
    "sq_gemm_plan_info": (i32, [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]),
    "sq_gemm_run": (i32, [vp, i32, vp]),
    "sq_gemm_run_at": (i32, [vp, i32, i32, vp, i32, vp]),
    "sq_gemm_fp8_tile_weights": (i32, [vp, vp, i32, i32, vp]),
    "sq_gemm_fp8_plan_create": (i32, [C.POINTER(vp), vp, i32, i32, vp, vp, i32, i32, vp, i32, vp]),
    "sq_gemm_fp8_plan_info": (i32, [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]),
    "sq_gemm_fp8_plan_destroy": (i32, [vp]),
    "sq_gemm_fp8_run_at": (i32, [vp, i32, i32, vp, i32, vp]),
    "sq_tp_alloc": (i32, [C.POINTER(vp), i64]),
    "sq_tp_free": (i32, [vp]),
    "sq_tp_ipc_export": (i32, [vp, vp]),
    "sq_tp_ipc_open": (i32, [vp, C.POINTER(vp)]),
    "sq_tp_ipc_close": (i32, [vp]),
    "sq_tp_allreduce_add_rmsnorm": (i32, [vp, vp, vp, vp, i32, i32, vp, vp, i32, i32, f32, vp]),
    "sq_tp_allreduce2_add_rmsnorm": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, i32, i32, f32, vp]),
    "sq_tp_allreduce3_add_rmsnorm": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, vp, vp, i32, i32, f32, vp]),
    "sq_tp_allreduce_ll_add_rmsnorm": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, i32, vp, vp, i32, i32, f32, vp]),
    "sq_tp_ll_publish": (i32, [vp, i32, i32, vp, vp, i32, vp, i32, vp, i32, vp]),
    "sq_tp_ll_consume": (i32, [vp, i32, vp, vp, vp, i32, vp, i32, vp, i32, vp]),
    "sq_draft_supported": (i32, [i32, i32, i32, i32, i32]),
    "sq_draft_plan_create": (i32, [C.POINTER(vp), i32, i32, i32, i32, vp, vp]),
    "sq_draft_plan_destroy": (i32, [vp]),
    "sq_draft_attention": (i32, [vp, i32, i32, vp, vp, vp, i32, i32, vp, i32, i32, vp]),
    "sq_embed_rows_batch": (i32, [vp, vp, i64, vp, i32, i32, i32, i32, vp, vp]),
    "sq_rope_kv_append_batch": (i32, [vp, i32, i32, i32, i32, vp, vp, vp, vp, i64, vp, i32, i32, i32, vp, vp, i32, vp]),
    "sq_kv_gather_batch": (i32, [vp, vp, i32, i32, i32, i32, i32, vp, i32, vp, i32, vp]),
    "sq_attn_plan_create_batch": (i32, [C.POINTER(vp), vp, i32, i32, i32, i32, i32, vp, vp, i32, i32, i32, vp, vp, i64]),
    "sq_tree_attn_batch": (i32, [vp, i32, i32, i32, vp, i32, i32, vp, i32, i32, vp]),
    "sq_sample_level_batch": (i32, [vp, i64, vp, vp, vp, i64, i64, vp, vp, vp, i32, i32, i32, f32, i32, vp, i64, vp, i32,
                                    vp]),
    "sq_accept_stochastic_batch": (i32, [vp, i64, vp, i64, vp, vp, vp, vp, i64, vp, vp, vp, i32, i32, f32, vp, vp, i64, vp,
                                         i64, vp, i32, i32, i32, vp]),
    "sq_accept_greedy_batch": (i32, [vp, vp, vp, vp, i32, vp, vp, i64, vp, i64, vp, i32, i32, vp]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


class SequoiaLibError(RuntimeError):
    pass


def load():
    """Load the shared library (once).  Raises if it has not been built -- never falls back."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SequoiaLibError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
                "sequoia_b200 has no CPU / PyTorch fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().sq_last_error()
        raise SequoiaLibError(f"{what} failed (rc={rc}): {msg.decode() if msg else ''}")


def ptr(t):
    """Device pointer of a tensor (or None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


def stream_ptr(device=None):
    return torch.cuda.current_stream(device).cuda_stream


def launch_count() -> int:
    return int(load().sq_launch_count())
