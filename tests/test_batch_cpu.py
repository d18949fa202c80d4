"""Host-side pieces of the batched entry points that need no GPU."""
import os
import re

import torch

import cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_draft_row_tables_pack_each_level_of_all_sequences_in_one_block():
    from sequoia_b200 import ops
    from sequoia_b200.tree import _Static
    st = _Static(cases.load_growmap("A100_growmaps/68m_7b/growmaps/A100-CNN-68m-7b-stochastic.pt"), "cpu")
    levels = [(0, 1)] + [(lv["n0"], lv["tb"]) for lv in st.levels]
    for B in (1, 2, 3, 8):
        base, step = ops.draft_row_tables(levels, st.S, B, "cpu")
        rows = base.long().view(1, -1) + torch.arange(B).view(-1, 1) * step.long().view(1, -1)   # (B, S)
        assert sorted(rows.flatten().tolist()) == list(range(B * st.S)), "every (sequence, node) has its own row"
        for n0, tb in levels:                          # a level of all B sequences is the contiguous block [B*n0, B*(n0+tb))
            blk = rows[:, n0:n0 + tb]
            assert blk.min().item() == B * n0 and blk.max().item() == B * (n0 + tb) - 1
            assert torch.equal(blk.flatten(), torch.arange(B * n0, B * (n0 + tb))), "sequence-major inside a level"
        if B == 1:
            assert torch.equal(rows[0], torch.arange(st.S)), "B = 1 is the node-indexed layout of the single-sequence path"


def test_batched_entry_points_refuse_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    assert lib.sq_embed_rows_batch(None, None, 0, None, 0, 1, 9, 256, None, None) == -1          # B > SQ_MAX_BATCH
    assert b"B=9" in lib.sq_last_error()
    assert lib.sq_embed_rows_batch(None, None, 0, None, 0, 1, 2, 256, None, None) == -1          # no state array
    assert lib.sq_kv_gather_batch(None, None, 2, 2, 2, 64, 64, None, 8, None, 4, None) == -1
    assert lib.sq_accept_greedy_batch(None, None, None, None, 16, None, None, 64, None, 8, None, 2, 64, None) == -1
    assert b"rows of 8" in lib.sq_last_error()                                                   # accept_idx rows < S
    assert lib.sq_tree_attn_batch(None, 0, 1, 1, None, 0, 1, None, 0, 0, None) == -1


def test_state_word_of_the_freeze_flag_matches_the_kernels():
    hdr = open(os.path.join(ROOT, "include", "sequoia_b200.h")).read()
    cuh = open(os.path.join(ROOT, "sequoia_b200", "csrc", "sq_common.cuh")).read()
    assert re.search(r"#define SQ_ST_FROZEN (\d+)", hdr).group(1) == re.search(r"ST_FROZEN = (\d+)", cuh).group(1)


def test_per_sequence_random_draws_follow_a_lone_spectree_in_prompt_order():
    from sequoia_b200.batch import draw_random
    M, S, V = 64, 9, 40
    prompts = [torch.zeros(5), torch.zeros(7), torch.zeros(3)]
    torch.manual_seed(123)
    r, rand = draw_random(prompts, M, S, V)
    torch.manual_seed(123)
    for b in range(len(prompts)):               # SpecTree: r in the constructor, rand after the draft prefill
        assert torch.equal(r[b], torch.rand(M, dtype=torch.float16))
        assert torch.equal(rand[b], torch.empty((S, V), dtype=torch.float16).uniform_())


def test_batch_refusals():
    import pytest
    from sequoia_b200.batch import BatchTree
    from sequoia_b200.engine import GraphInferenceEngine, GraphInferenceEngineTG, InferenceEngine
    from sequoia_b200.kv import KV_Cache
    for pol in ("greedys", "specinfer", "spec_test"):
        with pytest.raises(ValueError, match="not supported"):
            BatchTree(None, None, [torch.zeros(3)], {}, policy=pol)
    for cls in (GraphInferenceEngine, GraphInferenceEngineTG):
        with pytest.raises(NotImplementedError, match="tensor parallelism"):
            cls(256, "random-init:llama-68m", device="cpu", tp_group=object(), batch_size=2)
    with pytest.raises(ValueError):
        GraphInferenceEngine(256, "random-init:llama-68m", device="cpu", batch_size=9)
    eng = InferenceEngine.__new__(InferenceEngine)            # the dense-mask API of a 2-sequence engine
    eng.batch_size = 2
    with pytest.raises(RuntimeError, match="dense mask"):
        eng.model_run(torch.zeros(1, 4, dtype=torch.long), torch.arange(4))
    with pytest.raises(RuntimeError, match="dense mask"):
        eng.gather_kv([0, 1])
    kv = KV_Cache(cases.CFG_DRAFT, batch_size=2, max_length=32, device="cpu")
    assert tuple(kv.k_cache.shape)[:2] == (cases.CFG_DRAFT.num_hidden_layers, 2)
    for call in (lambda: kv.gather_kv([0]), lambda: kv.gather_kv_incremental([0], 1),
                 lambda: kv.initialize_kv(kv.k_cache, kv.v_cache, 1)):
        with pytest.raises(RuntimeError, match="holds 2"):
            call()
    one = KV_Cache(cases.CFG_DRAFT, batch_size=1, max_length=32, device="cpu")
    assert tuple(one.k_cache.shape) == (cases.CFG_DRAFT.num_hidden_layers, 1, cases.CFG_DRAFT.num_key_value_heads, 32,
                                        cases.CFG_DRAFT.hidden_size // cases.CFG_DRAFT.num_attention_heads)
