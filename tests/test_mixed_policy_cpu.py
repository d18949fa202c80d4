"""Host-side pieces of the per-sequence policy that need no GPU: refusals of policy lists and of admit(policy=), the C
entry points' argument refusals, the host values a mixed tree keeps per slot, and testbed.py's --policies."""
import pytest
import torch

import cases  # noqa: F401  (puts the repository root on sys.path)


def _bare_tree(B=2, M=64, S=9, policies=("spec", "spec"), frozen=(True, False)):
    """A BatchTree with only the host fields admit() checks before it touches the device."""
    from sequoia_b200.batch import BatchTree
    bt = BatchTree.__new__(BatchTree)
    bt.B, bt.M, bt.S, bt.seeded = B, M, S, False
    bt.policies = list(policies)
    bt.mixed = len(set(policies)) > 1
    bt.greedy = not bt.mixed and policies[0] == "greedy"
    bt.frozen = list(frozen)
    bt.temps, bt.top_ps = [0.6] * B, [1.0] * B
    return bt


def test_policy_lists_are_checked():
    from sequoia_b200.batch import _policies
    assert _policies("spec", 3) == ["spec"] * 3
    assert _policies(["greedy", "spec"], 2) == ["greedy", "spec"]
    assert _policies(("spec", "spec"), 2) == ["spec", "spec"]
    with pytest.raises(ValueError, match="3 values for 2"):
        _policies(["spec", "greedy", "spec"], 2)
    with pytest.raises(ValueError, match="1 values for 2"):
        _policies(["spec"], 2)
    for bad in ("greedys", "specinfer", "bogus", "Spec", None, 1):
        with pytest.raises(ValueError, match="not supported"):
            _policies(bad, 2)
        with pytest.raises(ValueError, match="not supported"):
            _policies(["spec", bad], 2)


def test_constructor_refuses_bad_policies():
    from sequoia_b200.batch import BatchTree
    prompts = [torch.zeros(3), torch.zeros(4)]
    for pol in (["spec"], ["spec", "greedy", "greedy"], ["spec", "greedys"], ["specinfer", "greedy"], "greedys"):
        with pytest.raises(ValueError):
            BatchTree(None, None, prompts, {}, policy=pol)
    with pytest.raises(ValueError, match="temperature"):           # T = 0 stays refused, for a greedy sequence too
        BatchTree(None, None, prompts, {}, policy=["greedy", "spec"], temperature=[0.0, 0.6])


def test_admit_refuses_unknown_policies():
    p = torch.zeros(10, dtype=torch.long)
    bt = _bare_tree()
    for bad in ("bogus", "greedys", "specinfer", 3):
        with pytest.raises(ValueError, match="not supported"):
            bt.admit(0, p, policy=bad)
    with pytest.raises(ValueError, match="temperature"):
        bt.admit(0, p, temperature=0.0, policy="greedy")
    assert bt.policies == ["spec", "spec"] and not bt.mixed and not bt.greedy, "a refusal changes nothing"
    assert bt.frozen == [True, False] and bt.temps == [0.6, 0.6] and bt.top_ps == [1.0, 1.0]


def test_mixed_entry_points_refuse_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    fake = 256                                          # a non-null address: every case is refused before any launch
    c0 = lib.sq_launch_count()

    def sample(T, greedy, B=2, rand=fake):
        return lib.sq_sample_level_batch_mixed(fake, 32000, fake, fake, rand, 32000, 8 * 32000, fake, fake, fake, 1, 2,
                                               32000, T, greedy, fake, 256, fake, B, None)

    def walk_g(greedy, B=2):
        return lib.sq_accept_greedy_batch_mixed(fake, fake, fake, fake, 16, fake, fake, 256, fake, 16, fake, greedy, B,
                                                256, None)

    def walk_s(T, greedy, B=2):
        return lib.sq_accept_stochastic_batch_mixed(fake, 32000, fake, 32000, fake, fake, fake, fake, 32000, fake, fake,
                                                    fake, 16, 32000, T, greedy, fake, fake, 256, fake, 16, fake, B, 256, 0,
                                                    None)

    null = b"null temperature or greedy"
    for call, msg in ((lambda: sample(None, fake), null), (lambda: sample(fake, None), null),
                      (lambda: sample(fake, fake, B=9), b"B=9"), (lambda: sample(fake, fake, B=0), b"B=0"),
                      (lambda: sample(fake, fake, rand=None), b"rand required"),
                      (lambda: walk_g(None), b"null greedy"), (lambda: walk_g(fake, B=9), b"B=9"),
                      (lambda: walk_s(None, fake), null), (lambda: walk_s(fake, None), null),
                      (lambda: walk_s(fake, fake, B=9), b"B=9")):
        assert call() == -1 and msg in lib.sq_last_error(), (msg, lib.sq_last_error())
    assert lib.sq_launch_count() == c0, "refused before any launch"


def test_cpu_draws_are_stream_aligned_for_greedy_prompts():
    """With seeds=None every prompt draws r and rand in prompt order, greedy ones included: a sampling prompt's numbers
    are those it gets in an all-spec batch."""
    from sequoia_b200.batch import draw_random
    prompts = [torch.zeros(5)] * 4
    torch.manual_seed(3)
    r, rand = draw_random(prompts, 32, 3, 16)
    torch.manual_seed(3)
    r1, rand1 = draw_random(prompts, 32, 3, 16)
    assert torch.equal(r, r1) and torch.equal(rand, rand1)
    torch.manual_seed(3)
    r2, rand2 = draw_random(prompts[:2], 32, 3, 16)
    assert torch.equal(r[:2], r2) and torch.equal(rand[:2], rand2), "slot b's draws depend only on the prompts before it"


def test_device_parameter_arrays_of_a_mixed_tree(monkeypatch):
    """The constructor's host-side values: top_p is 1 on the device for greedy slots, greedy_dev marks them, and the
    filter is needed only for a sampling slot with top_p < 1.  (torch.tensor(..., device=) is redirected to the CPU.)"""
    import sequoia_b200.batch as batch
    made = {}
    real_tensor = torch.tensor

    def cpu_tensor(data, dtype=None, device=None):
        return real_tensor(data, dtype=dtype)

    class Stop(Exception):
        pass

    def stop(*a, **k):
        raise Stop
    prompts = [torch.ones(5, dtype=torch.long)] * 3
    monkeypatch.setattr(batch.torch, "tensor", cpu_tensor)
    monkeypatch.setattr(batch.torch, "zeros", stop)                  # the first device allocation after the arrays

    class Eng:
        def __init__(self):
            self.engine = type("E", (), dict(batch_size=3, max_length=64))()
            self.device = "cuda:0"
    monkeypatch.setattr(batch, "_Static", lambda gm, dev: type("St", (), dict(S=9))())
    monkeypatch.setattr(batch, "check_vocab", lambda pol, V: made.setdefault("vocab", []).append(pol))
    d = Eng()
    d.engine.model_config = type("C", (), dict(vocab_size=32000))()
    bt = batch.BatchTree.__new__(batch.BatchTree)
    with pytest.raises(Stop):
        batch.BatchTree.__init__(bt, d, d, prompts, {}, policy=["greedy", "spec", "spec"],
                                 temperature=[0.5, 0.7, 0.9], top_p=[0.8, 1.0, 1.0], max_length=64)
    assert bt.mixed and not bt.greedy and bt.policies == ["greedy", "spec", "spec"]
    assert sorted(made["vocab"]) == ["greedy", "spec"]
    assert bt.top_p_dev.tolist() == [1.0, 1.0, 1.0], "a greedy slot's top_p is 1 on the device"
    assert bt.greedy_dev.tolist() == [1, 0, 0] and bt.greedy_dev.dtype == torch.int32
    assert bt.T_dev.tolist() == pytest.approx([0.5, 0.7, 0.9])
    assert not bt.use_top_p, "only a greedy slot has top_p < 1: no filter"
    bt2 = batch.BatchTree.__new__(batch.BatchTree)
    with pytest.raises(Stop):
        batch.BatchTree.__init__(bt2, d, d, prompts, {}, policy=["greedy", "spec", "greedy"],
                                 top_p=[1.0, 0.9, 1.0], max_length=64)
    assert bt2.use_top_p and bt2.top_p_dev.tolist() == pytest.approx([1.0, 0.9, 1.0])
    for pols, mixed, greedy in ((["spec"] * 3, False, False), (["greedy"] * 3, False, True), ("greedy", False, True)):
        bt3 = batch.BatchTree.__new__(batch.BatchTree)
        with pytest.raises(Stop):
            batch.BatchTree.__init__(bt3, d, d, prompts, {}, policy=pols, max_length=64)
        assert (bt3.mixed, bt3.greedy) == (mixed, greedy), pols


# ------------------------------------------------------------------------------------------------ testbed --policies
def test_policies_flag_parsing_and_refusals():
    import testbed
    ap = testbed.build_parser()
    assert ap.parse_args([]).policies is None
    assert testbed.prompt_policies(ap.parse_args(["--batch", "2"]), 5) is None
    a = ap.parse_args(["--batch", "2", "--policies", "spec,greedy"])
    assert testbed.prompt_policies(a, 5) == ["spec", "greedy", "spec", "greedy", "spec"]
    a = ap.parse_args(["--batch", "4", "--refill", "--policies", "greedy, greedy,spec"])
    assert testbed.prompt_policies(a, 4) == ["greedy", "greedy", "spec", "greedy"]
    with pytest.raises(SystemExit, match="with --batch"):
        testbed.prompt_policies(ap.parse_args(["--policies", "spec,greedy"]), 4)
    for tree in ("greedy", "specinfer", "greedys"):
        with pytest.raises(SystemExit, match="--tree"):
            testbed.prompt_policies(ap.parse_args(["--batch", "2", "--tree", tree, "--policies", "spec,greedy"]), 4)
    for bad in ("spec,greedys", "specinfer", "", "spec,,greedy"):
        with pytest.raises(SystemExit, match="spec or greedy"):
            testbed.prompt_policies(ap.parse_args(["--batch", "2", "--policies", bad]), 4)


class PolicyTree:
    """test_refill_cpu.FakeTree's step logic with a policy per slot: admit() records each admitted prompt's policy."""

    def __init__(self, prompts, policies):
        from test_refill_cpu import FakeTree
        self.fake = FakeTree(prompts)
        self.frozen = self.fake.frozen
        self.policies = list(policies)
        self.admitted = []

    def construct_grow_map(self):
        pass

    def verify(self):
        return self.fake.verify()

    def freeze(self, b):
        self.fake.freeze(b)

    def admit(self, b, prompt, policy):
        self.fake.admit(b, prompt)
        self.policies[b] = policy
        self.admitted.append((self.fake.ids[b], policy))


@pytest.mark.parametrize("n,B", [(7, 3), (5, 2), (4, 4)])
def test_refill_passes_each_prompts_policy(n, B):
    import testbed
    prompts = [torch.tensor([100 * i + j for j in range(4)]) for i in range(n)]
    limits = [len(p) + 2 + i % 3 for i, p in enumerate(prompts)]
    pols = ["spec", "greedy", "greedy"]
    policies = [pols[i % 3] for i in range(n)]
    tree = PolicyTree(prompts[:B], policies[:B])
    outputs, decoded, steps, order = testbed.decode_refill(tree, prompts, limits, policies=policies)
    assert order == list(range(n))
    assert tree.admitted == [(i, policies[i]) for i in range(B, n)], "each admission brings its prompt's policy"
    assert all(o is not None for o in outputs)


def test_chunked_batches_get_round_robin_policies(monkeypatch):
    import testbed
    import sequoia_b200.batch as batch
    built = []

    class Tree:
        def __init__(self, draft, target, chunk, gm, policy, **kw):
            built.append(policy)
            self.frozen = [True] * len(chunk)
    monkeypatch.setattr(batch, "BatchTree", Tree)
    monkeypatch.setattr(testbed.torch.cuda, "synchronize", lambda *a: None)

    class Eng:
        def clear_kv(self):
            pass
    prompts = [torch.tensor([i, 1]) for i in range(6)]
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)
    args = testbed.build_parser().parse_args(["--batch", "3", "--policies", "spec,greedy"])
    policies = testbed.prompt_policies(args, len(prompts))
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 3, policies=policies)
    assert built == [["spec", "greedy", "spec"], ["greedy", "spec", "greedy"]]
    built.clear()
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "greedy", 0.6, 1.0, 64, 3)
    assert built == ["greedy", "greedy"], "without --policies the tree policy is passed as before"
