"""Per-sequence counter-based random numbers, the parts that need no GPU: the CPU restatement of the generator
(oracle/philox.py) against Random123's philox4x32-10 known answers and the uniform grid, the seed refusals of BatchTree
and admit, the C entry points' argument refusals, and testbed.py's --device-rng flag."""
import numpy as np
import pytest
import scipy.stats
import torch

import cases  # noqa: F401  (puts the repository root on sys.path)
from oracle import philox

MASK = 0xFFFFFFFF


@pytest.mark.parametrize("ctr,key,want", [
    ([0, 0, 0, 0], [0, 0], "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
    ([MASK] * 4, [MASK] * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0], "d16cfe09 94fdcceb 5001e420 24126ea1"),
])
def test_philox_known_answers(ctr, key, want):
    got = philox.philox4x32_10(ctr, key)
    assert " ".join("%08x" % int(x) for x in got) == want


def test_stream_layout():
    """Element e is word e % 4 of counter (e // 4, 0, purpose, step); the key is the seed's two halves."""
    seed = 0x0123456789ABCDEF
    w = philox.words(seed, 2, 7, 10)
    for e in (0, 3, 4, 9):
        blk = philox.philox4x32_10([e // 4, 0, 2, 7], [seed & MASK, seed >> 32])
        assert int(w[e]) == int(blk[e % 4])
    # purposes, steps and seeds are separate streams
    a = philox.words(seed, 0, 0, 64)
    for other in (philox.words(seed, 1, 0, 64), philox.words(seed, 0, 1, 64), philox.words(seed + 1, 0, 0, 64),
                  philox.words(seed ^ (1 << 40), 0, 0, 64)):
        assert not np.array_equal(a, other)


def test_uniforms_lie_on_the_2048_grid_and_are_uniform():
    """u = k/2048, k in [0, 2048) (zero included, one excluded): the values torch's CPU fp16 uniform_ takes.  A
    chi-square over 2^20 draws across the 2048 values passes at p > 1e-3."""
    u = philox.uniforms(0xC0FFEE, philox.RAND, 1 << 20)
    assert u.dtype == np.float16
    k = u.astype(np.float64) * 2048
    assert np.array_equal(k, np.round(k)) and k.min() == 0 and k.max() == 2047
    counts = np.bincount(k.astype(np.int64), minlength=2048)
    p = scipy.stats.chisquare(counts).pvalue
    assert p > 1e-3, p
    torch_grid = torch.unique(torch.empty(1 << 20, dtype=torch.float16).uniform_()).double().numpy() * 2048
    assert set(torch_grid.astype(np.int64).tolist()) <= set(range(2048))


def test_noise_is_positive_and_exponential():
    h, x = philox.noise(42, 3, 1 << 16)
    assert h.dtype == np.float16 and bool(np.isfinite(h).all()) and float(h.min()) >= 2.0 ** -24
    assert abs(float(x.mean()) - 1.0) < 0.02 and abs(float(x.var()) - 1.0) < 0.05
    assert scipy.stats.kstest(x, "expon").pvalue > 1e-3
    # the largest word gives u = 1 after the fp32 rounding: clamped to the smallest positive fp16
    assert philox.noise_u(np.array([MASK], dtype=np.uint32))[0] == 1.0


# ------------------------------------------------------------------------------------------------ BatchTree seeds
def test_constructor_refuses_bad_seeds():
    from sequoia_b200.batch import BatchTree
    prompts = [torch.zeros(3), torch.zeros(4)]
    with pytest.raises(ValueError, match="seeds: 3 values for 2"):
        BatchTree(None, None, prompts, {}, seeds=[1, 2, 3])
    for bad in ([1, -1], [1, 1 << 64], [1, 2.0], [True, 2], [1, "7"]):
        with pytest.raises(ValueError, match="seed"):
            BatchTree(None, None, prompts, {}, seeds=bad)


def test_seed_bits():
    from sequoia_b200.batch import _as_int64, check_seed
    assert check_seed(np.uint64((1 << 64) - 1)) == (1 << 64) - 1
    assert _as_int64((1 << 64) - 1) == -1 and _as_int64(1 << 63) == -(1 << 63) and _as_int64(5) == 5
    t = torch.tensor([_as_int64((1 << 64) - 2)], dtype=torch.int64)
    assert int(t.numpy().view(np.uint64)[0]) == (1 << 64) - 2


def _bare_tree(seeded, B=2, M=64, S=9):
    from sequoia_b200.batch import BatchTree
    bt = BatchTree.__new__(BatchTree)
    bt.B, bt.M, bt.S, bt.greedy, bt.seeded = B, M, S, False, seeded
    bt.frozen = [True, False]
    bt.temps, bt.top_ps = [0.6] * B, [1.0] * B
    return bt


def test_admit_seed_refusals():
    p = torch.zeros(10, dtype=torch.long)
    bt = _bare_tree(seeded=True)
    with pytest.raises(ValueError, match="needs the prompt's seed"):
        bt.admit(0, p)
    for bad in (-1, 1 << 64, 0.5, None):
        with pytest.raises(ValueError, match="seed"):
            bt.admit(0, p, temperature=0.9, seed=bad)
    bt = _bare_tree(seeded=False)
    with pytest.raises(ValueError, match="built with seeds"):
        bt.admit(0, p, seed=3)
    assert bt.frozen == [True, False] and bt.temps == [0.6, 0.6], "a refusal changes nothing"


# ------------------------------------------------------------------------------------------------ C entry points
def test_rng_entry_points_refuse_bad_arguments():
    import ctypes as C
    from sequoia_b200 import _lib
    lib = _lib.load()
    fake = 256                                          # a non-null address: every case is refused before any launch
    c0 = lib.sq_launch_count()

    keep = []                                           # the host slot lists stay alive until the calls have run

    def slots(*b):
        keep.append((C.c_int32 * max(len(b), 1))(*b))
        return C.addressof(keep[-1])

    arr = slots(0, 1)
    cases_ = [
        ((None, 64, 64, fake, arr, 2, 2, 0), b"null"),
        ((fake, 64, 64, None, arr, 2, 2, 0), b"null"),
        ((fake, 64, 64, fake, None, 2, 2, 0), b"null"),
        ((fake, 64, 64, fake, arr, 2, 0, 0), b"B=0"),
        ((fake, 64, 64, fake, arr, 2, 9, 0), b"B=9"),
        ((fake, 64, 64, fake, arr, 2, 2, 2), b"purpose 2"),
        ((fake, 64, 64, fake, arr, 2, 2, -1), b"purpose -1"),
        ((fake, 64, 64, fake, arr, 3, 2, 0), b"3 slots"),
        ((fake, 64, 64, fake, arr, 0, 2, 0), b"0 slots"),
        ((fake, 64, 64, fake, slots(0, 2), 2, 2, 0), b"slot 2 of 2"),
        ((fake, 64, 64, fake, slots(1, -1), 2, 2, 0), b"slot -1"),
        ((fake, 64, 64, fake, slots(1, 1), 2, 3, 1), b"listed twice"),
        ((fake, 32, 64, fake, arr, 2, 2, 0), b"count=64"),
        ((fake, 64, 0, fake, arr, 2, 2, 0), b"count=0"),
    ]
    for args, msg in cases_:
        assert lib.sq_rng_uniform_seqs(*args, None) == -1, args
        assert msg in lib.sq_last_error(), (args, lib.sq_last_error())
    bad_noise = [
        ((None, 32000, 32000, fake, fake, fake, 2), b"null"),
        ((fake, 32000, 32000, fake, None, fake, 2), b"null"),
        ((fake, 32000, 32000, fake, fake, None, 2), b"null"),
        ((fake, 32000, 32000, fake, fake, fake, 0), b"B=0"),
        ((fake, 32000, 32000, fake, fake, fake, 9), b"B=9"),
        ((fake, 32000, 31999, fake, fake, fake, 2), b"multiples of 8"),
        ((fake, 31992, 32000, fake, fake, fake, 2), b"multiples of 8"),
        ((fake + 8, 32000, 32000, fake, fake, fake, 2), b"aligned"),
    ]
    for args, msg in bad_noise:
        assert lib.sq_rng_exponential_batch(*args, None) == -1, args
        assert msg in lib.sq_last_error(), (args, lib.sq_last_error())
    assert lib.sq_launch_count() == c0, "a refused call launches nothing"


# ------------------------------------------------------------------------------------------------ testbed --device-rng
def test_testbed_device_rng_flag():
    import testbed
    ap = testbed.build_parser()
    assert ap.parse_args([]).device_rng is False
    a = ap.parse_args(["--batch", "4", "--device-rng", "--seed", "5"])
    assert a.device_rng and testbed.device_rng_seeds(a, 3) == [(5 << 32) | i for i in range(3)]
    a = ap.parse_args(["--batch", "2", "--refill", "--device-rng"])
    assert testbed.device_rng_seeds(a, 2) == [(17 << 32), (17 << 32) | 1]
    assert testbed.device_rng_seeds(ap.parse_args(["--batch", "4"]), 4) is None
    for argv in (["--device-rng"], ["--device-rng", "--batch", "1"]):
        with pytest.raises(SystemExit, match="--batch"):
            testbed.device_rng_seeds(ap.parse_args(argv), 4)
    with pytest.raises(SystemExit, match="--batch"):
        testbed.main(["--device-rng"])                  # refused before any model is built
    with pytest.raises(SystemExit, match="seed"):
        testbed.device_rng_seeds(ap.parse_args(["--batch", "2", "--device-rng", "--seed", "-1"]), 2)


class _SeedTree:
    """admit() records (slot, prompt id, seed)."""

    def __init__(self, B):
        self.frozen, self.admits, self.n = [False] * B, [], 0

    def construct_grow_map(self):
        pass

    def verify(self):
        self.n += 1
        out = [(torch.tensor([7] * (3 + self.n)), 0, False)] * len(self.frozen)
        return out

    def freeze(self, b):
        self.frozen[b] = True

    def admit(self, b, prompt, seed=None):
        self.frozen[b] = False
        self.admits.append((b, int(prompt[0]), seed))


def test_refill_passes_each_prompt_its_own_seed():
    import testbed
    prompts = [torch.tensor([i, 7, 7]) for i in range(5)]
    tree = _SeedTree(2)
    seeds = [1000 + i for i in range(5)]
    testbed.decode_refill(tree, prompts, [4] * 5, seeds=seeds)
    assert [(p, s) for _, p, s in tree.admits] == [(i, 1000 + i) for i in range(2, 5)]
