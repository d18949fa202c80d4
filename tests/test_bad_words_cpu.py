"""Host-side pieces of the per-sequence bad words and min_tokens that need no GPU: the CPU statement
(oracle/bad_words.py) against an independent restatement of vLLM's rules on explicit token lists, the refusals of
BatchTree's bad_words / min_tokens and of the C entry point, the per-prompt and shared input forms, the device rows a
tree keeps per slot through admissions (the end ids when stop mode starts included), and testbed.py's --bad-words /
--min-tokens."""
import pytest
import torch

import cases  # noqa: F401  (puts the repository root on sys.path)
from oracle.bad_words import banned_ids, process_rows
from test_stop_cpu import _cpu_tree

F16 = torch.float16


def _vllm_bad_words(logits, bad_words, past_tokens):
    """vLLM v1's _apply_bad_words_single_batch: past_tokens are the output tokens only."""
    for w in bad_words:
        if len(w) > len(past_tokens) + 1:
            continue
        prefix = len(w) - 1
        actual = past_tokens[-prefix:] if prefix > 0 else []
        if list(actual) == list(w[:prefix]):
            logits[w[-1]] = float("-inf")


def _vllm_min_tokens(logits, n_output, min_tokens, stop_ids):
    """vLLM's min-tokens processor: the stop ids are -inf while fewer than min_tokens tokens have been generated."""
    if n_output < min_tokens:
        for t in stop_ids:
            logits[t] = float("-inf")


# ------------------------------------------------------------------------------------------------ oracle
def test_banned_ids_on_explicit_lists():
    V = 50
    words = [(7,), (3, 4), (9, 3, 4, 5), (1, 2, 8), (20, 21, 22, 23, 24, 25)]
    for gen in ([], [3], [9, 3, 4], [2, 9, 3, 4], [1, 2], [2], [20, 21, 22, 23, 24], [21, 22, 23, 24]):
        row = torch.zeros(V)
        _vllm_bad_words(row, words, gen)
        assert banned_ids(gen, words, 0, 0, (), V) == set(torch.isinf(row).nonzero().flatten().tolist()), gen
    assert banned_ids([], words, 0, 0, (), V) == {7}, "one-token words everywhere; longer ones need a context"
    assert banned_ids([9, 3, 4], words, 0, 0, (), V) == {7, 5}
    assert banned_ids([21, 22, 23, 24], words, 0, 0, (), V) == {7}, "a word longer than the generated context"
    assert banned_ids([3], words, 0, 0, (), 4) == set(), "ids outside [0, V) are not banned"


def _setup(V=64):
    """One sequence on a 4-node tree 0 -> 1 -> 2, 0 -> 3: prompt of L = 5, committed P = 8 (3 generated)."""
    mask = torch.tensor([[1, 0, 0, 0], [1, 1, 0, 0], [1, 1, 1, 0], [1, 0, 0, 1]], dtype=torch.bool)
    depth = torch.tensor([0, 1, 2, 1])
    tokens = torch.zeros(1, 16, dtype=torch.long)
    tokens[0, :8] = torch.tensor([10, 11, 12, 13, 14, 20, 21, 22])        # prompt 10..14, generated 20 21 22
    tokens[0, 8:11] = torch.tensor([30, 31, 40])                          # nodes 1, 2, 3 at slots P-1+j
    return tokens, mask, depth, V


def test_oracle_rows_against_vllm_on_tree_contexts():
    tokens, mask, depth, V = _setup()
    P, L = 8, 5
    contexts = {0: [20, 21, 22], 1: [20, 21, 22, 30], 2: [20, 21, 22, 30, 31], 3: [20, 21, 22, 40]}
    words = [(22, 30, 50), (30, 31, 51), (21, 22, 52), (14, 20, 53), (13, 14, 20, 21, 22, 54), (22, 40, 55), (6,),
             (20, 21, 22, 30, 31, 56), (19, 20, 21, 22, 30, 31, 57)]
    g = torch.Generator().manual_seed(1)
    x = torch.randn(4 + 1, V, generator=g).to(F16)
    x[:, 51], x[:, 52], x[:, 6] = float("nan"), float("inf"), float("-inf")
    got = process_rows(x, tokens, [P], [L], mask, depth, [words], [0], [()])
    for k, gen in contexts.items():
        want = x[k].clone()
        _vllm_bad_words(want, words, gen)
        assert torch.equal(got[k].view(torch.int16), want.view(torch.int16)), k
    assert bool(torch.isinf(got[0, 52])) and got[0, 52] < 0, "+inf at a banned id becomes -inf"
    assert bool(torch.isinf(got[2, 51])) and got[2, 51] < 0, "NaN at a banned id becomes -inf"
    assert not bool(torch.isinf(got[1, 51])), "a path word matches only its own path"
    assert bool(torch.isinf(got[0, 53])) is False and bool(torch.isinf(got[1, 53])) is False, "no match across the prompt"
    assert float(got[2, 56]) == float("-inf") and not bool(torch.isinf(got[2, 57])), "committed tail + path, no prompt"
    assert torch.equal(got[4].view(torch.int16), x[4].view(torch.int16)), "rows from B*S on are copied"


@pytest.mark.parametrize("m", [1, 3, 4, 5])
def test_min_tokens_boundary(m):
    """P + d = L + m - 1 is banned, P + d = L + m is not (vLLM: fewer than m output tokens so far)."""
    tokens, mask, depth, V = _setup()
    P, L = 8, 5
    x = torch.zeros(5, V, dtype=F16)
    x[:, 2] = float("nan")
    got = process_rows(x, tokens, [P], [L], mask, depth, [()], [L + m], [(0, 2, 63)])
    for k in range(4):
        n_out = P + int(depth[k]) - L
        want = x[k].clone()
        _vllm_min_tokens(want, n_out, m, (0, 2, 63))
        assert torch.equal(got[k].view(torch.int16), want.view(torch.int16)), (m, k)
        assert bool(torch.isinf(got[k, 0])) == (P + int(depth[k]) <= L + m - 1), (m, k)


def test_oracle_neutral_and_frozen():
    tokens, mask, depth, V = _setup()
    tokens = tokens.repeat(3, 1)
    x = torch.randn(12, V).to(F16)
    got = process_rows(x, tokens, [8] * 3, [5] * 3, mask, depth, [None, ((6,),), ((7,),)], [0, 0, 20], [(0,)] * 3,
                       frozen=[False, True, False])
    assert torch.equal(got[:8].view(torch.int16), x[:8].view(torch.int16)), "neutral and frozen untouched"
    assert bool(torch.isinf(got[8:, 7]).all()) and bool(torch.isinf(got[8:, 0]).all())


# ------------------------------------------------------------------------------------------------ validation
def test_check_bad_words():
    import numpy as np
    from sequoia_b200.batch import check_bad_words
    assert check_bad_words(None) is None and check_bad_words([]) == () and check_bad_words(set()) == ()
    assert check_bad_words([[5], (1, 2), [5], [np.int64(1), 2]]) == ((5,), (1, 2)), "duplicates dropped, order kept"
    assert check_bad_words({(3, 4), (3, 4)}) == ((3, 4),)
    assert len(check_bad_words([[t] for t in range(128)])) == 128
    assert check_bad_words([list(range(16))], 16) == (tuple(range(16)),)
    assert len(check_bad_words([[t % 100] for t in range(300)])) == 100, "the limit counts distinct words"
    for bad in ([[]], [[1, True]], [[1.0]], [["1"]], [[-1]], [list(range(17))], [[t] for t in range(129)], [5], 5, "ab",
                [{1, 2}], ["ab"], [b"ab"], [[None]]):
        with pytest.raises(ValueError, match="bad_words"):
            check_bad_words(bad)
    with pytest.raises(ValueError, match="32000"):
        check_bad_words([[1, 32000]], 32000)


def test_shared_and_per_prompt_forms():
    from sequoia_b200.batch import _bad_words
    assert _bad_words(None, 2) == [None, None] and _bad_words([], 2) == [(), ()]
    assert _bad_words([[1], [2, 3]], 2) == [((1,), (2, 3))] * 2, "two levels: one set of two words for all"
    assert _bad_words([[1, 2]], 3) == [((1, 2),)] * 3
    assert _bad_words([None, [[2, 3]]], 2) == [None, ((2, 3),)], "three levels: one set per prompt"
    assert _bad_words([[[1]], [[2, 3], [4]]], 2) == [((1,),), ((2, 3), (4,))]
    assert _bad_words([[], []], 2) == [(), ()], "an empty entry is an empty set of words, not an empty word"
    assert _bad_words([[[1]]], 1) == [((1,),)]
    with pytest.raises(ValueError, match="3 sets for 2"):
        _bad_words([None, None, [[1]]], 2)
    with pytest.raises(ValueError, match="bad_words"):
        _bad_words([[[1]], [2, 3]], 2)                 # mixed depths: the shared form, whose word [[1]] is refused


def test_check_min_tokens():
    import numpy as np
    from sequoia_b200.batch import _min_tokens, check_min_tokens
    assert check_min_tokens(0) == 0 and check_min_tokens(np.int32(7)) == 7 and check_min_tokens(5, 5) == 5
    for bad in (-1, 1.0, True, None, "3"):
        with pytest.raises(ValueError, match="min_tokens"):
            check_min_tokens(bad)
    with pytest.raises(ValueError, match="exceeds max_new_tokens=4"):
        check_min_tokens(5, 4)
    assert _min_tokens(3, 2) == [3, 3] and _min_tokens([1, 0], 2) == [1, 0]
    with pytest.raises(ValueError, match="1 values for 2"):
        _min_tokens([1], 2)


def test_check_bannable():
    from sequoia_b200.batch import check_bannable
    check_bannable(8, tuple((t,) for t in range(7)), None, 0, (0, 2))
    with pytest.raises(ValueError, match="every token id"):
        check_bannable(8, tuple((t,) for t in range(8)), None, 0, ())
    with pytest.raises(ValueError, match="min_tokens"):
        check_bannable(8, tuple((t,) for t in range(1, 8) if t != 2), None, 1, (0, 2))
    check_bannable(8, tuple((t,) for t in range(1, 8) if t != 2), None, 0, (0, 2))
    with pytest.raises(ValueError, match="allowed_token_ids"):
        check_bannable(32000, ((5,), (9, 7)), (5,), 0, ())
    check_bannable(32000, ((5,), (7, 9)), (5, 9), 0, ())          # a path-dependent ban is not refused
    with pytest.raises(ValueError, match="allowed_token_ids"):
        check_bannable(32000, ((5,),), (2, 5), 3, (2,))


def test_constructor_refuses_bad_settings(monkeypatch):
    from sequoia_b200.batch import BatchTree
    prompts = [torch.zeros(3), torch.zeros(4)]
    for kw in (dict(bad_words=[[]]), dict(bad_words=[None, [[1]], None]), dict(bad_words=5), dict(min_tokens=-1),
               dict(min_tokens=[1, 2, 3]), dict(min_tokens=True)):
        with pytest.raises(ValueError):
            BatchTree(None, None, prompts, {}, **kw)
    for kw, msg in ((dict(bad_words=[[32000]]), "32000"), (dict(min_tokens=5, max_new_tokens=[4, 9]), "exceeds"),
                    (dict(allowed_token_ids=[7, 8], bad_words=[[7], [8]]), "every token id"),
                    (dict(allowed_token_ids=[7, 0], bad_words=[[7]], min_tokens=[0, 1]), "every token id")):
        with pytest.raises(ValueError, match=msg):
            _cpu_tree(monkeypatch, prompts, **kw)
        monkeypatch.undo()
    _cpu_tree(monkeypatch, prompts, allowed_token_ids=[7, 0], bad_words=[[7]], min_tokens=[0, 1], stop_tokens=[])
    monkeypatch.undo()                                   # (stop mode without stop ids: min_tokens bans nothing)


def test_admit_refuses_bad_settings(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7)]
    bt = _cpu_tree(monkeypatch, prompts, max_new_tokens=[10, None], allowed_token_ids=[None, [4, 2]])
    graphs = dict(bt.graphs)
    for kw in (dict(bad_words=[[32000]]), dict(bad_words=[[]]), dict(bad_words=[(1,)] * 2 + [(t,) for t in range(129)]),
               dict(min_tokens=None), dict(min_tokens=-2), dict(min_tokens=11), dict(min_tokens=3, max_new_tokens=2)):
        with pytest.raises(ValueError):
            bt.admit(0, torch.ones(6, dtype=torch.long), **kw)
    for kw in (dict(bad_words=[[4], [2]]), dict(bad_words=[[4]], min_tokens=1, stop_tokens=[2]),
               dict(bad_words=[[4]], min_tokens=1, allowed_token_ids=[4, 2], stop_tokens=[2])):
        with pytest.raises(ValueError, match="every token id"):
            bt.admit(1, torch.ones(6, dtype=torch.long), **kw)
    assert bt.bad_words == [None] * 2 and bt.min_tokens == [0] * 2 and not bt.use_ban
    assert bt.graphs == graphs and bt.frozen == [True, True] and bt.stop_tokens == [None, None], "a refusal changes nothing"
    bt._start_logit_bias()                              # (the CPU constructor stopped at its first device allocation)
    bt.finish_reason = [None] * 2
    bt.admit(0, torch.ones(6, dtype=torch.long), min_tokens=10)            # = the slot's budget
    assert bt.min_tokens[0] == 10 and bt.use_ban


# ------------------------------------------------------------------------------------------------ device rows
def _expect(bt, b, words, min_end):
    n = len(words or ())
    assert int(bt.n_words_dev[b]) == n and int(bt.min_end_dev[b]) == min_end, b
    for i, w in enumerate(words or ()):
        assert int(bt.word_len_dev[b, i]) == len(w) and bt.words_dev[b, i, :len(w)].tolist() == list(w), (b, i)
        assert not bool(bt.words_dev[b, i, len(w):].any())
    assert not bool(bt.word_len_dev[b, n:].any()) and not bool(bt.words_dev[b, n:].any()), "rows past n_words are zero"


def test_device_rows_of_a_tree(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    assert not bt.use_ban and bt.words_dev is None and bt.bad_words == [None] * 3 and bt.min_tokens == [0] * 3
    for kw in (dict(bad_words=[]), dict(min_tokens=0), dict(bad_words=[None, [], []], min_tokens=[0, 0, 0])):
        nb = _cpu_tree(monkeypatch, prompts, **kw)
        assert not nb.use_ban and nb.words_dev is None, ("neutral settings allocate nothing", kw)
    bt = _cpu_tree(monkeypatch, prompts, bad_words=[[[5, 6], [7]], None, [[31999] * 16]], min_tokens=[0, 3, 10 ** 12])
    assert bt.use_ban and bt.bad_words == [((5, 6), (7,)), None, ((31999,) * 16,)]
    bt._start_ban()                                      # (the CPU constructor stops at its first device allocation)
    assert bt.words_dev.shape == (3, 128, 16) and bt.word_len_dev.shape == (3, 128) and bt.words_dev.dtype == torch.int32
    _expect(bt, 0, ((5, 6), (7,)), 0)
    _expect(bt, 1, None, 10)
    _expect(bt, 2, ((31999,) * 16,), (1 << 31) - 1)
    assert bt._ban_end_ids().tolist() == [[0, 2] + [-1] * 6] * 3, "default mode: the reference's 0 and 2"


def test_admissions_update_the_rows_and_the_end_ids(monkeypatch):
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    bt.admit(0, torch.ones(6, dtype=torch.long), bad_words=[], min_tokens=0)
    assert not bt.use_ban and bt.graphs == {"draft": 1, "steady": 2, "post": 3}, "neutral: no recapture"
    assert bt.bad_words[0] == ()
    bt.admit(1, torch.ones(12, dtype=torch.long), bad_words=[[9, 8], [3]], min_tokens=4)
    assert bt.use_ban and bt.graphs == {"draft": 1}, "the first non-neutral admission drops steady and post once"
    _expect(bt, 1, ((9, 8), (3,)), 16)
    _expect(bt, 0, (), 0)
    assert bt._ban_end_ids().tolist() == [[0, 2] + [-1] * 6] * 3 and not bt.use_stop
    bt.graphs = {"draft": 1, "steady": 4, "post": 5}
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long))
    _expect(bt, 1, ((9, 8), (3,)), 14)                   # the default keeps both; min_tokens counts from the new prompt
    bt.frozen[1] = True
    bt.admit(1, torch.ones(10, dtype=torch.long), bad_words=None, min_tokens=0)
    _expect(bt, 1, None, 0)
    assert bt.graphs == {"draft": 1, "steady": 4, "post": 5} and bt.use_ban, "the kernel stays, no recapture"
    bt.admit(2, torch.ones(4, dtype=torch.long), stop_tokens=[7, 31999], min_tokens=2)
    assert bt.use_stop and bt.graphs == {"draft": 1}, "stop mode starts: steady and post recaptured"
    ends = bt._ban_end_ids()
    assert ends is bt.stop_ids_dev, "stop mode: the kernel reads each slot's stop ids"
    assert ends.tolist() == [[-1] * 8, [-1] * 8, [7, 31999] + [-1] * 6]
    _expect(bt, 2, None, 6)


# ------------------------------------------------------------------------------------------------ C entry point
def test_ban_entry_point_refuses_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    f = 256                                             # a non-null address: every case is refused before any launch

    def call(logits=f, ld=32000, V=32000, tokens=f, ld_seq=384, state=f, L=f, depth=f, bits=f, tw=4, S=128, words=f,
             lens=f, n=f, me=f, ends=f, B=2):
        return lib.sq_ban_tokens_rows_batch(logits, ld, V, tokens, ld_seq, state, L, depth, bits, tw, S, words, lens, n,
                                            me, ends, B, None)
    c0 = lib.sq_launch_count()
    nulls = [(dict([(k, None)]), b"null array") for k in ("logits", "tokens", "state", "L", "depth", "bits", "words",
                                                          "lens", "n", "me", "ends")]
    cases_ = nulls + [(dict(B=0), b"B=0"), (dict(B=9), b"B=9"), (dict(V=32004, ld=32008), b"V=32004"),
                      (dict(V=131080, ld=131080), b"V=131080"), (dict(V=0), b"V=0"), (dict(ld=31999), b"ld=31999"),
                      (dict(S=0, tw=0), b"S=0"), (dict(tw=3), b"tree_words=3"), (dict(S=1025, tw=33), b"tree_words=33"),
                      (dict(ld_seq=0), b"ld_seq=0")]
    for kw, msg in cases_:
        assert call(**kw) == -1 and msg in lib.sq_last_error(), (kw, msg, lib.sq_last_error())
    assert lib.sq_launch_count() == c0, "refused before any launch"


# ------------------------------------------------------------------------------------------------ testbed flags
def test_flags_parsing_and_refusals():
    import testbed
    ap = testbed.build_parser()
    assert testbed.batch_bad_words(ap.parse_args([])) == {}
    got = testbed.batch_bad_words(ap.parse_args(["--bad-words", "5,6;7; 8 ,9,10", "--min-tokens", "4", "--batch", "2"]))
    assert got == dict(bad_words=[[5, 6], [7], [8, 9, 10]], min_tokens=4)
    assert testbed.batch_bad_words(ap.parse_args(["--min-tokens", "0", "--batch", "1", "--refill"])) == \
        dict(min_tokens=0)
    for flag, val in (("--bad-words", "5"), ("--min-tokens", "3")):
        with pytest.raises(SystemExit, match="with --batch"):
            testbed.batch_bad_words(ap.parse_args([flag, val]))
    for flag, val in (("--bad-words", "a"), ("--bad-words", "5;;6"), ("--bad-words", "-1"), ("--bad-words", ",".join(
            ["1"] * 17)), ("--min-tokens", "-1")):
        with pytest.raises(SystemExit, match=flag):
            testbed.batch_bad_words(ap.parse_args([f"{flag}={val}", "--batch", "2"]))


def test_batches_and_refill_get_the_settings(monkeypatch):
    """Chunked batches are built with the settings; refill admissions pass none, so each slot keeps its values."""
    import testbed
    import sequoia_b200.batch as batch
    built, admitted = [], []

    class Tree:
        def __init__(self, draft, target, chunk, gm, policy, **kw):
            built.append({k: v for k, v in kw.items() if k in ("bad_words", "min_tokens")})
            self.frozen = [False] * len(chunk)

        def admit(self, b, prompt, **kw):
            admitted.append(kw)
            self.frozen[b] = False

        def construct_grow_map(self):
            pass

        def verify(self):
            out = [(torch.ones(300, dtype=torch.long), 0, True) for _ in self.frozen]
            self.frozen = [True] * len(self.frozen)
            return out

        def freeze(self, b):
            self.frozen[b] = True
    monkeypatch.setattr(batch, "BatchTree", Tree)
    monkeypatch.setattr(testbed.torch.cuda, "synchronize", lambda *a: None)
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)

    class Eng:
        def clear_kv(self):
            pass
    prompts = [torch.tensor([i, 1]) for i in range(4)]
    kw = dict(bad_words=[[5, 6]], min_tokens=3)
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, bad_words=kw)
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2)
    assert built == [kw, kw, {}, {}]
    built.clear()
    testbed.simulation_batch(Eng(), Eng(), prompts, {}, "spec", 0.6, 1.0, 64, 2, refill=True, bad_words=kw)
    assert built == [kw] and len(admitted) == 2
    assert not any(k in ("bad_words", "min_tokens") for a in admitted for k in a)
