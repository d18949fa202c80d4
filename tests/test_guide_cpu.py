"""Host-side pieces of guided decoding that need no GPU: the CPU statement (oracle/guide.py) against an independent
hand-written statement on small explicit guides (a choice trie, a JSON-string-like default/banned state, the dead
state), every refusal of GuideState, TokenGuide, BatchTree(guide=...), admit(guide=...) and the three C entry points,
the shared and per-prompt forms, the table and blobs a tree keeps through admissions, and the packed blob decoded back to
the oracle's allowed ids and transitions at V = 32000 and 128256."""
import random

import pytest
import torch

import cases  # noqa: F401  (puts the repository root on sys.path)
from oracle import guide as O
from sequoia_b200.guide import GuideState, TokenGuide, guide_allowed_ids, guide_next
from test_stop_cpu import _cpu_tree

V = 32000


def _trie(words, end_id):
    """A choice trie over token sequences: after a whole word only end_id is allowed, into an accepting sink."""
    nodes = [{}]
    for w in words:
        cur = 0
        for t in w:
            if t not in nodes[cur]:
                nodes.append({})
                nodes[cur][t] = len(nodes) - 1
            cur = nodes[cur][t]
    sink = len(nodes)
    states = [GuideState(edges=e if e else {end_id: sink}) for e in nodes]
    states.append(GuideState(edges={end_id: sink}))
    return TokenGuide(states)


def _string_guide():
    """'"' opens a string; inside it every id but the control ids 0..31 stays inside, '"' (34) closes it; then 2 ends."""
    quote, end = 34, 2
    return TokenGuide([GuideState(edges={quote: 1}),
                       GuideState(edges={quote: 2}, default=1, banned=set(range(32))),
                       GuideState(edges={end: 2})])


# ------------------------------------------------------------------------------------------------ oracle
def _hand_trie(words, ids):
    """Independent statement of the trie: the ids must spell a prefix of a word, then only end ids after it."""
    def valid(pre):
        return any(pre == list(w[:len(pre)]) or (pre[:len(w)] == list(w) and set(pre[len(w):]) <= {2}) for w in words)
    return max(n for n in range(len(ids) + 1) if valid(list(ids[:n])))


def test_trie_against_hand_statement():
    words = [(10, 11, 12), (10, 13), (20,)]
    g = _trie(words, 2)
    for ids in ([10, 11, 12, 2, 2], [10, 13, 2], [20, 2], [10, 11, 13], [11], [10, 13, 13], [20, 20], [], [10]):
        assert O.accepted_prefix(g, ids, V) == _hand_trie(words, ids), ids
        s = O.state_after(g, ids, V)
        assert (s < 0) == (O.accepted_prefix(g, ids, V) < len(ids)), ids
    assert O.allowed(g.states[0], V) == {10, 20}
    assert O.allowed(g.states[O.state_after(g, [10], V)], V) == {11, 13}
    assert O.allowed(g.states[O.state_after(g, [10, 13], V)], V) == {2}


def test_string_state_against_hand_statement():
    g = _string_guide()
    inside = g.states[1]
    allowed = O.allowed(inside, V)
    assert allowed == set(range(32, V)) and O.step(inside, 34, V) == 2 and O.step(inside, 500, V) == 1
    assert O.step(inside, 5, V) is None and O.step(inside, V, V) is None and O.step(inside, -1, V) is None
    rnd = random.Random(3)
    for _ in range(200):
        ids = [34] + [rnd.choice([34, 2, 5, 40, 31999, 1000]) for _ in range(rnd.randint(0, 8))]
        # hand statement: after the opening quote, ids >= 32 other than 34 stay inside; 34 closes; then only 2
        s, n = 0, 0
        for t in ids:
            nxt = {0: {34: 1}.get(t), 1: (2 if t == 34 else (1 if t >= 32 else None)), 2: {2: 2}.get(t)}[s]
            if nxt is None:
                break
            s, n = nxt, n + 1
        assert O.accepted_prefix(g, ids, V) == n, ids
        assert O.state_after(g, ids, V) == (s if n == len(ids) else -1), ids


def test_process_rows_masks_by_node_state_and_kills_the_subtree():
    g = _trie([(5, 6), (7,)], 2)
    S = 4                                                  # node 1 and 2 children of 0, node 3 child of 1
    mask01 = torch.tensor([[1, 0, 0, 0], [1, 1, 0, 0], [1, 0, 1, 0], [1, 1, 0, 1]], dtype=torch.bool)
    P, Vs = 10, 64
    tokens = torch.zeros(1, 20, dtype=torch.long)
    tokens[0, P:P + 3] = torch.tensor([5, 9, 6])           # node 1 = 5 (ok), node 2 = 9 (dead), node 3 = 6 (ok)
    x = torch.randn(S, Vs).to(torch.float16)
    x[:, 5] = float("nan")
    x[:, 40] = float("inf")
    out = O.process_rows(x, tokens, [P], mask01, [g], [g.start])
    fin = [set(torch.nonzero(out[k] != float("-inf")).flatten().tolist()) for k in range(S)]
    assert fin[0] == {5, 7}                                # (5 still holds its NaN: an allowed entry is unchanged)
    assert bool(torch.isnan(out[0, 5])) and bool(torch.isinf(out[0, 40])) and out[0, 40] < 0
    assert fin[1] == {6} and fin[2] == set() and fin[3] == {2}
    bits = x.view(torch.int16)
    assert O.process_rows(x, tokens, [P], mask01, [None], [0]).view(torch.int16).equal(bits)
    assert O.process_rows(x, tokens, [P], mask01, [g], [0], frozen=[True]).view(torch.int16).equal(bits)
    dead = O.process_rows(x, tokens, [P], mask01, [g], [-1])
    assert bool(torch.isneginf(dead).all())


# ------------------------------------------------------------------------------------------------ refusals
def test_guide_state_and_token_guide_refusals():
    for kw in (dict(edges={-1: 0}), dict(edges={True: 0}), dict(edges={3: -1}), dict(edges={3: 1.5}),
               dict(edges=[(3, 0)]), dict(default=-1), dict(default=0, banned=[-2]), dict(edges={3: 0}, banned=[4]),
               dict(edges={3: 0}, default=0, banned=[3]), dict(), dict(edges={}), dict(default=0, banned="ab")):
        with pytest.raises(ValueError):
            GuideState(**kw)
    ok = GuideState(edges={3: 0})
    for args in (([],), ([ok] * 4097,), ([ok, "x"],), ([ok], 1), ([ok], -1), ([GuideState(edges={3: 5})],),
                 ([GuideState(default=2)],), ("ab",)):
        with pytest.raises(ValueError):
            TokenGuide(*args)
    TokenGuide([ok] * 4096)
    big = GuideState(edges={t: 0 for t in range(1 << 19)})
    TokenGuide([big, big])
    with pytest.raises(ValueError, match="edges"):
        TokenGuide([big, big, GuideState(edges={1: 0})])


def test_guide_check_against_the_vocabulary_and_the_slot():
    g = TokenGuide([GuideState(edges={5: 1}), GuideState(default=1, banned=range(10))])
    g.check(V)
    with pytest.raises(ValueError, match="outside"):
        TokenGuide([GuideState(edges={V: 0})]).check(V)
    with pytest.raises(ValueError, match="outside"):
        TokenGuide([GuideState(default=0, banned=[V])]).check(V)
    with pytest.raises(ValueError, match="allows no id"):
        TokenGuide([GuideState(default=0, banned=range(16))]).check(16)
    with pytest.raises(ValueError, match="allowed_token_ids"):
        g.check(V, allowed_token_ids=(6, 7))               # state 0 allows only 5
    with pytest.raises(ValueError, match="bad_words"):
        g.check(V, bad_words=((5,), (6, 7)))
    g.check(V, bad_words=((6, 5),))                        # a path-dependent word is not counted
    with pytest.raises(ValueError, match="allowed_token_ids"):
        g.check(V, allowed_token_ids=(5, 3), bad_words=())  # state 1 bans 0..9
    g.check(V, allowed_token_ids=(5, 30))


def test_constructor_and_admit_refusals(monkeypatch):
    from sequoia_b200.batch import BatchTree
    ok = TokenGuide([GuideState(edges={5: 0})])
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7)]
    for kw in (dict(guide=5), dict(guide=[ok]), dict(guide=[ok, ok, None]), dict(guide=[ok, "x"])):
        with pytest.raises(ValueError):
            BatchTree(None, None, prompts, {}, **kw)
    for kw, msg in ((dict(guide=TokenGuide([GuideState(edges={V: 0})])), "outside"),
                    (dict(guide=[None, ok], allowed_token_ids=[None, [6]]), "allows no id"),
                    (dict(guide=ok, bad_words=[[5]]), "allows no id")):
        with pytest.raises(ValueError, match=msg):
            _cpu_tree(monkeypatch, prompts, **kw)
        monkeypatch.undo()
    bt = _cpu_tree(monkeypatch, prompts, allowed_token_ids=[None, [4, 2]])
    graphs = dict(bt.graphs)
    for b, kw in ((0, dict(guide="x")), (0, dict(guide=TokenGuide([GuideState(edges={V: 0})]))), (1, dict(guide=ok)),
                  (0, dict(guide=ok, bad_words=[[5]])), (0, dict(guide=ok, allowed_token_ids=[6]))):
        with pytest.raises(ValueError):
            bt.admit(b, torch.ones(6, dtype=torch.long), **kw)
    assert bt.guides == [None, None] and not bt.use_guide and bt.graphs == graphs, "a refusal changes nothing"
    with pytest.raises(ValueError, match="no guide"):
        bt.guide_state(0)


def test_shared_and_per_prompt_forms(monkeypatch):
    g, h = _trie([(10, 11)], 2), _string_guide()
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    assert _cpu_tree(monkeypatch, prompts, guide=g).guides == [g, g, g]
    monkeypatch.undo()
    assert _cpu_tree(monkeypatch, prompts, guide=[None, h, g]).guides == [None, h, g]
    monkeypatch.undo()
    assert _cpu_tree(monkeypatch, prompts, guide=(None, None, None)).guides == [None] * 3
    monkeypatch.undo()
    assert _cpu_tree(monkeypatch, prompts).guides == [None] * 3


def test_table_and_blobs_through_admissions(monkeypatch):
    g, h = _trie([(10, 11)], 2), _string_guide()
    prompts = [torch.ones(n, dtype=torch.long) for n in (5, 7, 9)]
    bt = _cpu_tree(monkeypatch, prompts)
    assert not bt.use_guide and bt.guide_table_dev is None
    bt.admit(0, torch.ones(6, dtype=torch.long), guide=None)
    assert not bt.use_guide and bt.graphs == {"draft": 1, "steady": 2, "post": 3}, "no guide: nothing changes"
    bt.admit(1, torch.ones(6, dtype=torch.long), guide=g)
    assert bt.use_guide and bt.graphs == {"draft": 1}, "the first guide drops steady and post once"
    assert bt.guide_table_dev.dtype == torch.int64 and bt.guide_scratch.shape == (3, 9)
    assert bt.guide_table_dev.tolist() == [0, bt.guide_blobs[1].data_ptr(), 0]
    assert torch.equal(bt.guide_blobs[1], g.pack(V)) and bt.guide_state(1) == g.start
    bt.graphs = {"draft": 1, "steady": 4, "post": 5}
    bt.frozen[2] = True
    bt.admit(2, torch.ones(6, dtype=torch.long), guide=g)
    assert bt.guide_blobs[2] is bt.guide_blobs[1], "slots with one guide share its blob"
    bt.frozen[1] = True
    bt.admit(1, torch.ones(6, dtype=torch.long), guide=h)
    assert torch.equal(bt.guide_blobs[1], h.pack(V)) and bt.guide_blobs[2] is not bt.guide_blobs[1]
    bt.frozen[1] = True
    bt.admit(1, torch.ones(6, dtype=torch.long))                          # the default keeps the slot's guide
    assert bt.guides[1] is h
    bt.frozen[2] = True
    bt.admit(2, torch.ones(6, dtype=torch.long), guide=None)
    assert bt.guide_table_dev.tolist() == [0, bt.guide_blobs[1].data_ptr(), 0] and bt.guide_blobs[2] is None
    assert bt.graphs == {"draft": 1, "steady": 4, "post": 5}, "no recapture after the first guide"


# ------------------------------------------------------------------------------------------------ the packed blob
@pytest.mark.parametrize("Vs", [32000, 128256])
def test_blob_decodes_to_the_oracle(Vs):
    rnd = random.Random(Vs)
    states = []
    n = 12
    for i in range(n):
        kind = i % 4
        edges = {rnd.randrange(Vs): rnd.randrange(n) for _ in range(rnd.choice([1, 3, 31, 32, 33, 700, 5000]))}
        if kind == 0:
            states.append(GuideState(edges=edges))
        elif kind == 1:
            banned = {rnd.randrange(Vs) for _ in range(50)} - edges.keys()
            states.append(GuideState(edges=edges, default=rnd.randrange(n), banned=banned))
        elif kind == 2:
            states.append(GuideState(default=i, banned=range(0, Vs, 7)))
        else:
            states.append(GuideState(edges={Vs - 1: 0, 0: 1}))
    g = TokenGuide(states, start=3)
    g.check(Vs)
    blob = g.pack(Vs)
    W = (Vs + 31) // 32
    assert blob.dtype == torch.int32 and blob[:4].tolist() == [n, W, g.n_edges, Vs]
    assert blob.numel() == 4 + 2 * n + 1 + 2 * g.n_edges + n * W
    for s in range(n):
        want = O.allowed_mask(g.states[s], Vs)
        got = torch.zeros(Vs, dtype=torch.bool)
        got[guide_allowed_ids(blob, s)] = True
        assert torch.equal(got, want), s
        probes = list(g.states[s].edges)[:40] + [rnd.randrange(Vs) for _ in range(40)] + [0, Vs - 1, Vs, -1]
        probes += list(g.states[s].banned)[:5]
        for t in probes:
            nx = O.step(g.states[s], t, Vs)
            assert guide_next(blob, s, t) == (-1 if nx is None else nx), (s, t)


# ------------------------------------------------------------------------------------------------ C entry points
def test_guide_entry_points_refuse_bad_arguments():
    from sequoia_b200 import _lib
    lib = _lib.load()
    f = 256                                             # a non-null address: every case is refused before any launch
    c0 = lib.sq_launch_count()

    def states(table=f, tokens=f, ld_seq=384, state=f, depth=f, bits=f, tw=4, S=128, V=32000, out=f, B=2):
        return lib.sq_guide_states_batch(table, tokens, ld_seq, state, depth, bits, tw, S, V, out, B, None)

    def mask(logits=f, ld=32000, V=32000, S=128, state=f, table=f, ns=f, B=2):
        return lib.sq_guide_mask_rows_batch(logits, ld, V, S, state, table, ns, B, None)

    def advance(table=f, tokens=f, ld_seq=384, state=f, V=32000, B=2):
        return lib.sq_guide_advance_batch(table, tokens, ld_seq, state, V, B, None)
    common = [(dict(B=0), b"B=0"), (dict(B=9), b"B=9"), (dict(V=32004), b"V=32004"), (dict(V=131080), b"V=131080"),
              (dict(V=0), b"V=0")]
    for fn, nulls, extra in (
            (states, ("table", "tokens", "state", "depth", "bits", "out"),
             [(dict(S=0, tw=0), b"S=0"), (dict(tw=3), b"tree_words=3"), (dict(S=1025, tw=33), b"S=1025"),
              (dict(ld_seq=0), b"ld_seq=0")]),
            (mask, ("logits", "state", "table", "ns"), [(dict(ld=31999), b"ld=31999"), (dict(S=0), b"S=0")]),
            (advance, ("table", "tokens", "state"), [(dict(ld_seq=0), b"ld_seq=0")])):
        for kw, msg in [(dict([(k, None)]), b"null array") for k in nulls] + common + extra:
            if fn is mask and "V" in kw:
                kw = dict(kw, ld=max(kw["V"], 8))
            assert fn(**kw) == -1 and msg in lib.sq_last_error(), (fn.__name__, kw, msg, lib.sq_last_error())
    assert lib.sq_launch_count() == c0, "refused before any launch"
