"""Host-side pieces of slot admission that need no GPU: argument refusals of BatchTree.admit and of the per-sequence C
entry points, testbed.py's --refill flag, and its queue logic against a fake tree."""
import math

import pytest
import torch

import cases  # noqa: F401  (puts the repository root on sys.path)


def _bare_tree(B=2, M=64, S=9, frozen=(True, False)):
    """A BatchTree with only the host fields admit() checks before it touches the device."""
    from sequoia_b200.batch import BatchTree
    bt = BatchTree.__new__(BatchTree)
    bt.B, bt.M, bt.S, bt.greedy = B, M, S, False
    bt.frozen = list(frozen)
    bt.temps, bt.top_ps = [0.6] * B, [1.0] * B
    return bt


def test_admit_refusals():
    bt = _bare_tree()
    p = torch.zeros(10, dtype=torch.long)
    with pytest.raises(IndexError):
        bt.admit(2, p)
    with pytest.raises(ValueError, match="still decoding"):
        bt.admit(1, p)
    with pytest.raises(ValueError, match="must hold the prompt"):
        bt.admit(0, torch.zeros(64 - 9 + 2, dtype=torch.long))          # len + S - 1 > M
    with pytest.raises(ValueError, match="must hold the prompt"):
        bt.admit(0, torch.zeros(0, dtype=torch.long))
    for T in (0.0, -1.0, math.inf, math.nan):
        with pytest.raises(ValueError, match="temperature"):
            bt.admit(0, p, temperature=T)
    for tp in (0.0, -0.1, 1.0001, math.nan, math.inf):
        with pytest.raises(ValueError, match="top_p"):
            bt.admit(0, p, top_p=tp)
    assert bt.frozen == [True, False] and bt.temps == [0.6, 0.6] and bt.top_ps == [1.0, 1.0], "a refusal changes nothing"


def test_constructor_refuses_bad_per_sequence_values():
    from sequoia_b200.batch import BatchTree
    prompts = [torch.zeros(3), torch.zeros(4)]
    with pytest.raises(ValueError, match="3 values for 2"):
        BatchTree(None, None, prompts, {}, temperature=[0.5, 0.6, 0.7])
    with pytest.raises(ValueError, match="temperature"):
        BatchTree(None, None, prompts, {}, temperature=[0.5, 0.0])
    with pytest.raises(ValueError, match="top_p"):
        BatchTree(None, None, prompts, {}, top_p=[1.0, 1.5])


def test_per_sequence_entry_points_refuse_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    # null temperature array
    assert lib.sq_sample_level_batch_per_seq(None, 0, None, None, None, 0, 0, None, None, None, 1, 2, 32000, None, 1,
                                             None, 256, None, 2, None) == -1
    assert b"null temperature" in lib.sq_last_error()
    assert lib.sq_accept_stochastic_batch_per_seq(None, 0, None, 0, None, None, None, None, 32000, None, None, None, 16,
                                                  32000, None, None, None, 256, None, 16, None, 2, 256, 0, None) == -1
    assert b"null temperature" in lib.sq_last_error()
    fake = 256                                          # a non-null address: refused before any launch
    assert lib.sq_top_p_filter_per_seq(None, 32000, 8, 32000, None, fake, 4, None) == -1
    assert b"null top_p" in lib.sq_last_error()
    assert lib.sq_top_p_filter_per_seq(None, 32000, 8, 32000, fake, None, 4, None) == -1
    assert b"null top_p" in lib.sq_last_error()
    for rows in (3, 0, -1):                             # rows_per_seq must divide n
        assert lib.sq_top_p_filter_per_seq(None, 32000, 8, 32000, fake, fake, rows, None) == -1
        assert b"does not divide" in lib.sq_last_error()
    # the checks shared with the scalar entry points still apply
    assert lib.sq_sample_level_batch_per_seq(None, 0, None, None, None, 0, 0, None, None, None, 1, 2, 32000, fake, 1,
                                             None, 256, None, 9, None) == -1
    assert b"B=9" in lib.sq_last_error()


# ------------------------------------------------------------------------------------------------ testbed --refill
def test_refill_flag_and_batch_checks():
    import testbed
    ap = testbed.build_parser()
    assert ap.parse_args([]).refill is False
    a = ap.parse_args(["--batch", "4", "--refill"])
    assert (a.batch, a.refill) == (4, True)
    assert testbed.check_batch_args(a, 10) == 4                       # any prompt count
    assert testbed.check_batch_args(a, 3) == 3                        # engines sized min(B, prompts)
    with pytest.raises(SystemExit, match="must divide"):
        testbed.check_batch_args(ap.parse_args(["--batch", "4"]), 10)
    assert testbed.check_batch_args(ap.parse_args(["--batch", "4"]), 8) == 4
    for extra in (["--Mode", "benchmark"], ["--tree", "specinfer"], ["--offloading"]):
        with pytest.raises(SystemExit):
            testbed.check_batch_args(ap.parse_args(["--batch", "2", "--refill"] + extra), 4)


class FakeTree:
    """Each step appends one token per active slot (`stop_at`: the prompt whose slot emits a stop token at its 3rd
    step; `room_at`: the prompts whose slot runs out of room at its 2nd step, which the tree freezes itself and reports
    with terminal = False, as BatchTree does).  A frozen slot repeats its last result.  admit() records the order and
    checks the slot was frozen.  verify() raises after `max_verifies` calls, so a loop that never ends fails."""

    def __init__(self, prompts, stop_token=None, stop_at=None, room_at=(), max_verifies=200):
        self.rows = [list(p.tolist()) for p in prompts]
        self.frozen = [False] * len(prompts)
        self.admitted = []
        self.ids = list(range(len(prompts)))
        self.stop_token, self.stop_at, self.room_at = stop_token, stop_at, set(room_at)
        self.ages = [0] * len(prompts)
        self.last = [None] * len(prompts)
        self.verifies, self.max_verifies = 0, max_verifies

    def construct_grow_map(self):
        pass

    def verify(self):
        self.verifies += 1
        assert self.verifies <= self.max_verifies, "the decode loop does not end"
        out = []
        for b, row in enumerate(self.rows):
            if not self.frozen[b]:
                self.ages[b] += 1
                tok = 1000 * (self.ids[b] + 1) + self.ages[b]
                if self.ids[b] == self.stop_at and self.ages[b] == 3:
                    tok = self.stop_token
                row.append(tok)
                self.last[b] = (torch.tensor(row), len(row) - 1, False)
                if self.ids[b] in self.room_at and self.ages[b] == 2:
                    self.frozen[b] = True                 # out of room: frozen by the tree, not terminal
            out.append(self.last[b])
        return out

    def freeze(self, b):
        self.frozen[b] = True

    def admit(self, b, prompt):
        assert self.frozen[b], "admit takes a frozen slot"
        self.rows[b] = list(prompt.tolist())
        self.frozen[b], self.ages[b] = False, 0
        self.ids[b] = int(prompt[0]) // 100
        self.admitted.append(self.ids[b])


@pytest.mark.parametrize("n,B", [(7, 3), (4, 4), (9, 2), (2, 3), (5, 1)])
def test_refill_queue_decodes_every_prompt_once(n, B):
    import testbed
    B0 = min(B, n)
    prompts = [torch.tensor([100 * i + j for j in range(5 + i % 3)]) for i in range(n)]
    limits = [len(p) + 2 + (3 * i) % 5 for i, p in enumerate(prompts)]        # 2..6 new tokens per prompt
    tree = FakeTree(prompts[:B0], stop_token=2, stop_at=n - 1)
    outputs, decoded, steps, order = testbed.decode_refill(tree, prompts, limits, stop=frozenset([2]))
    assert order == list(range(n)), "prompts are admitted in queue order"
    assert tree.admitted == list(range(B0, n))
    assert all(tree.frozen), "every slot ends frozen"
    for i, (p, out) in enumerate(zip(prompts, outputs)):
        assert out is not None and torch.equal(out[:len(p)], p), i
        new = out[len(p):].tolist()
        if i == n - 1 and limits[i] - len(p) >= 3:
            assert new == [1000 * (i + 1) + 1, 1000 * (i + 1) + 2, 2], "a stop token ends the prompt"
        else:
            assert new == [1000 * (i + 1) + k for k in range(1, limits[i] - len(p) + 1)], i
    assert decoded == sum(len(o) - len(p) for o, p in zip(outputs, prompts))
    assert steps == decoded                                                   # one token per step in the fake


@pytest.mark.parametrize("n,B", [(6, 2), (3, 3), (5, 1)])
def test_refill_takes_over_a_slot_the_tree_froze_for_lack_of_room(n, B):
    """Prompts 0 and 2 run out of room (frozen by the tree, terminal = False) before any limit or stop token: their
    slots are refilled, every prompt is decoded once, and the loop ends."""
    import testbed
    prompts = [torch.tensor([100 * i, 7, 7]) for i in range(n)]
    limits = [len(p) + 5 for p in prompts]
    tree = FakeTree(prompts[:B], room_at=(0, 2))
    outputs, decoded, steps, order = testbed.decode_refill(tree, prompts, limits)
    assert order == list(range(n)) and tree.admitted == list(range(B, n))
    assert all(tree.frozen)
    for i, (p, out) in enumerate(zip(prompts, outputs)):
        n_new = 2 if i in (0, 2) else 5
        assert out.tolist() == p.tolist() + [1000 * (i + 1) + k for k in range(1, n_new + 1)], i
    assert decoded == steps == sum(len(o) - len(p) for o, p in zip(outputs, prompts))


def test_chunk_counts_no_step_for_a_slot_the_tree_froze():
    import testbed
    prompts = [torch.tensor([100 * i, 7]) for i in range(2)]
    tree = FakeTree(prompts, room_at=(0,))
    decoded, steps = testbed.decode_chunk(tree, prompts, [len(p) + 6 for p in prompts])
    assert (decoded, steps) == (2 + 6, 2 + 6)


def test_scalar_sampling_values_of_any_numeric_type_broadcast():
    import numpy as np
    from sequoia_b200.batch import _per_seq
    for v in (0.7, 1, np.float32(0.7), np.float64(0.7), torch.tensor(0.7)):
        assert _per_seq(v, 3, "temperature") == [float(v)] * 3
    assert _per_seq(np.array([0.5, 0.6], dtype=np.float32), 2, "top_p") == [float(np.float32(0.5)), float(np.float32(0.6))]
    assert _per_seq(torch.tensor([0.5, 0.25]), 2, "top_p") == [0.5, 0.25]
    with pytest.raises(ValueError, match="1 values for 2"):
        _per_seq(torch.tensor([0.5]), 2, "top_p")


def test_refill_records_steady_and_admission_steps():
    import testbed
    prompts = [torch.tensor([100 * i, 1]) for i in range(3)]
    limits = [3, 5, 3]
    tree = FakeTree(prompts[:2])
    times = []
    testbed.decode_refill(tree, prompts, limits, step_times=times)
    # step 1: both decode (slot 0 hits its limit), step 2: admission of prompt 2 into slot 0, step 3: steady
    assert [k for k, _ in times] == ["steady", "admission", "steady"]
    assert all(s >= 0 for _, s in times)
