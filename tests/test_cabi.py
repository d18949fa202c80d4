"""CPU-side checks of the drop-in boundary: the shared library loads and exports every symbol include/*.h
declares; the Python host mirrors the reference's module paths and signatures.  No compute (no GPU here)."""
import inspect
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from sequoia_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "sequoia_b200.h")).read()
    declared = set(re.findall(r"\b(sq_[a-z_A-Z0-9]+)\s*\(", hdr))
    assert len(declared) >= 20
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/sequoia_b200.h but not exported"
    assert declared == set(_lib.EXPORTED_SYMBOLS), declared ^ set(_lib.EXPORTED_SYMBOLS)
    assert lib.sq_version() >= 100
    assert lib.sq_last_error() is not None


def test_argument_errors_are_reported_not_crashes():
    from sequoia_b200 import _lib
    lib = _lib.load()
    rc = lib.sq_rmsnorm(None, None, None, 1, 7, 1e-5, None)          # hidden % 8 != 0 -> rejected before any launch
    assert rc == -1 and b"hidden" in lib.sq_last_error()
    rc = lib.sq_softmax_T(None, 0, None, 0, 1, 100000, 0.6, None)    # V too large
    assert rc == -1


def test_reference_module_paths_and_signatures():
    """tests/testbed.py:12-18 imports, and the constructor keyword sets of Tree/SpecTree.py:8-28 / Engine.py."""
    from Engine.Engine import GraphInferenceEngine, GraphInferenceEngineTG
    from Engine.Llama_KV import KV_Cache
    from Engine.offload_engine import OffloadEngine
    from Tree.GreedyTree import GreedyTree
    from Tree.SpecTree import SpecTree
    import data_converter
    import utils
    for fn in ("get_sampling_logits", "_make_causal_mask", "cuda_graph_for_residual",
               "cuda_graph_for_sampling_without_replacement", "cuda_graph_for_sampling_argmax", "get_residual",
               "sampling_without_replacement", "sampling_argmax", "ChildrenAccept"):
        assert hasattr(utils, fn)
    for fn in ("convert_wiki_dataset", "convert_cnn_dataset", "convert_c4_dataset_eval", "convert_wikimqa_dataset"):
        assert hasattr(data_converter, fn)
    want = ["draft_model_engine", "target_model_engine", "prefix", "temperature", "top_p", "draft_kv_len",
            "target_kv_len", "max_length", "device", "max_target_seq", "vocab_size", "grow_map", "attn_mask", "sequence",
            "new_tokens_buffer", "parents_buffer", "position_ids", "residual_graph", "sampling_callables",
            "sample_gather_indices"]
    for cls in (SpecTree, GreedyTree):
        assert list(inspect.signature(cls.__init__).parameters)[1:] == want
        for m in ("construct_grow_map", "verify", "collective_grow_static"):
            assert hasattr(cls, m)
    assert list(inspect.signature(GraphInferenceEngine.__init__).parameters)[1:5] == ["max_length", "model_name_or_path", "dtype", "device"]
    assert list(inspect.signature(GraphInferenceEngineTG.__init__).parameters)[1:6] == ["max_length", "model_name_or_path", "dtype", "device", "offloading"]
    for m in ("initialize_cuda_graph", "graph_inference", "inference", "clear_kv", "gather_kv", "initialize_kv", "get_kv_cache"):
        assert hasattr(GraphInferenceEngine, m)
    for m in ("inference", "clear_kv", "set_kv_len", "gather_kv", "initialize_kv", "get_kv_cache"):
        assert hasattr(GraphInferenceEngineTG, m) and hasattr(OffloadEngine, m)
    for m in ("initialize_kv", "gather_kv", "gather_kv_incremental", "update_kv_cache", "clear", "get_usable_length", "set_kv_len"):
        assert hasattr(KV_Cache, m)


def test_gemm_dispatch_table_is_swept():
    """Every gemm_tn_kernel instantiation run_tile can launch is in the GPU variant sweep (cases.GEMM_VARIANTS), so a
    variant added to the table cannot go untested.  (The sweep also checks that each forced plan records the table's
    stage count.)"""
    import cases
    src = open(os.path.join(ROOT, "sequoia_b200", "csrc", "sq_gemm.cu")).read()
    body = src[src.index("static int run_tile("):]
    body = body[:body.index("#undef SQ_G")]
    table = [tuple(int(x) for x in m) for m in re.findall(r"\bSQ_G\(\s*(\d+),\s*(\d+),\s*(\d+),\s*(\d+)\s*\)", body)]
    assert len(table) == 16, table
    assert table == cases.GEMM_VARIANTS


def test_draft_attention_supported_shapes():
    """The draft attention keeps the whole K/V of a head in shared memory: for the 68m draft shape (h = 768, 12 heads of
    64) 640 is the longest max_length that fits, and 672 (the next multiple of 32) must be refused.  A 7B shape (head_dim
    128) is refused at any length."""
    from sequoia_b200 import ops
    assert ops.draft_supported(768, 12, 12, 64, 640)
    assert not ops.draft_supported(768, 12, 12, 64, 672)
    assert not ops.draft_supported(4096, 32, 32, 128, 384)


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "sequoia_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("the oracle", "").replace("CPU oracle", ""), f"{f} mentions oracle"


def test_growmap_static_tables():
    import torch
    from sequoia_b200.tree import _Static, pack_tree_mask
    import cases
    for name in ("A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt", "L40_growmaps/8x8-tree.pt",
                 "L40_growmaps/2-chain.pt", "L40_growmaps/L40-CNN-7b-70b-stochastic.pt", "L40_growmaps/1x128-tree.pt"):
        gm = cases.load_growmap(name)
        st = _Static(gm, "cpu")
        S = gm["size"]
        assert sum(l["tb"] for l in st.levels) == S - 1
        bits = pack_tree_mask(gm["mask"]).to(torch.int64) & 0xFFFFFFFF
        j = torch.arange(S)
        unpacked = (bits[:, j // 32] >> (j % 32)) & 1
        assert torch.equal(unpacked, gm["mask"].to(torch.int64))
        # CSR == Successors
        for k in range(S):
            assert st.succ[st.succ_off[k]:st.succ_off[k + 1]].tolist() == list(gm["Successors"][k])
