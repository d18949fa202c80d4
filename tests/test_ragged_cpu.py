"""Ragged part lists on the host (no GPU): the packed row and q-tile layout, the refusals of the C entry points before
any launch, and the runner's Python-side refusals."""
import types

import pytest

from sequoia_b200 import _lib, ops


def test_layout_prefix_sums():
    parts = [(5, 300, -299, 1), (2, 128, 0, 128), (7, 167, -39, 128), (0, 1, 0, 1)]
    assert ops.ragged_layout(parts, 8, 4096) == ([0, 300, 428, 595, 596], [0, 300, 428, 595, 596])
    # q tiles of 128 rows (GP = 1) and of 16 rows (GP = 8)
    assert ops.ragged_layout(parts, 8, 4096, 128)[1] == [0, 3, 4, 6, 7]
    assert ops.ragged_layout(parts, 8, 4096, 16)[1] == [0, 19, 27, 38, 39]
    assert ops.ragged_layout([(0, 129, 0, 1)], 1, 129, 128) == ([0, 129], [0, 2])
    # the host array is passed through as built
    arr = ops.ragged_parts(parts)
    assert ops.ragged_parts(arr) is arr
    assert [(p.seq, p.n, p.n0, p.kv_end) for p in arr] == parts


BAD = {
    "no parts": ([], 8, 100),
    "more parts than sequences": ([(0, 1, 0, 1), (1, 1, 0, 1)], 1, 100),
    "seq = B": ([(8, 1, 0, 1)], 8, 100),
    "seq < 0": ([(-1, 1, 0, 1)], 8, 100),
    "seq twice": ([(3, 1, 0, 1), (3, 2, 0, 1)], 8, 100),
    "n = 0": ([(0, 0, 0, 1)], 8, 100),
    "n < 0": ([(0, -4, 0, 1)], 8, 100),
    "rows > n_max": ([(0, 60, 0, 1), (1, 41, 0, 1)], 8, 100),
}


@pytest.mark.parametrize("what", list(BAD))
def test_bad_part_lists_are_refused(what):
    parts, B, n_max = BAD[what]
    with pytest.raises(_lib.SequoiaLibError):
        ops.ragged_layout(parts, B, n_max)


@pytest.mark.parametrize("what", list(BAD))
def test_entry_points_refuse_before_any_launch(what):
    """The C calls check the part list before touching a pointer or launching (null device pointers here)."""
    parts, B, n_max = BAD[what]
    lib = _lib.load()
    arr = ops.ragged_parts(parts)
    ap = ops.C.addressof(arr)
    c0 = _lib.launch_count()
    assert lib.sq_embed_rows_ragged(None, None, 1024, 16, ap, len(arr), B, n_max, 256, None, None) == -1
    assert lib.sq_rope_kv_append_ragged(None, 768, 4, 4, 64, None, None, None, None, 1024, 16, ap, len(arr), B, n_max,
                                        None, None, 1024, None) == -1
    assert _lib.launch_count() == c0
    assert lib.sq_last_error()


def test_entry_points_refuse_null_state_and_bad_shapes():
    lib = _lib.load()
    arr = ops.ragged_parts([(0, 4, 0, 4)])
    ap = ops.C.addressof(arr)
    assert lib.sq_embed_rows_ragged(None, None, 1024, None, ap, 1, 1, 8, 256, None, None) == -1
    assert lib.sq_embed_rows_ragged(None, None, 1024, 16, ap, 1, 1, 8, 260, None, None) == -1
    assert lib.sq_rope_kv_append_ragged(None, 768, 4, 4, 72, None, None, None, None, 1024, 16, ap, 1, 1, 8, None, None,
                                        1024, None) == -1
    assert lib.sq_tree_attn_ragged(None, 0, ap, 1, None, None, 0, 0, None) == -1


def _bare_runner(tp_size=1):
    from sequoia_b200.model import LlamaRunner
    r = LlamaRunner.__new__(LlamaRunner)
    r.tp = types.SimpleNamespace(size=tp_size)
    r.B, r.n_max, r.V = 4, 1000, 10
    return r


def test_forward_ragged_refuses_tensor_parallel_engines():
    with pytest.raises(NotImplementedError):
        _bare_runner(tp_size=2).forward_ragged([(0, 4, 0, 4, 1, None)], None, None, None, state=None)


@pytest.mark.parametrize("part", [(0, 4, 0, 4, 0, "out"), (0, 4, 0, 4, 5, "out"), (0, 4, 0, 4, 1, None),
                                  (0, 4, 0, 4, 2, "out")])
def test_forward_ragged_refuses_bad_logit_requests(part):
    """n_logits outside 1..n, or a logits_out that is not (n_logits, V)"""
    import torch
    out = torch.empty(1, 10) if part[5] == "out" else None
    with pytest.raises(ValueError):
        _bare_runner().forward_ragged([part[:5] + (out,)], None, None, None, state=None)


def test_forward_ragged_refuses_bad_part_lists():
    with pytest.raises(_lib.SequoiaLibError):
        _bare_runner().forward_ragged([(4, 4, 0, 4, 1, None)], None, None, None, state=None)
    with pytest.raises(_lib.SequoiaLibError):
        _bare_runner().forward_ragged([(0, 600, 0, 4, 1, None), (1, 401, 0, 4, 1, None)], None, None, None, state=None)
