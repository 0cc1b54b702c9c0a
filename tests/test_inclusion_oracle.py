"""CPU tests of the allow-list oracle (tests/inclusion_oracle.py) on a small hand-made corpus, against brute force over the corpus
rows and hand-worked cases: colliding tuples of dedup ranks 0..3, repeats and -1 padding, unretrievable rows, ids outside
[-1, N), combination with an exclusion, one level of the beam search with fillers and the retrieval."""
import itertools

import numpy as np
import pytest

import exclusion_oracle as X
import inclusion_oracle as I
import item_oracle as IO

K, H = 4, 3
CORPUS = np.array([
    [0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0],       # rows 0..3: one tuple, dedup ranks 0..3
    [0, 1, 2], [0, 1, 3],                             # rows 4, 5
    [1, 0, 0], [1, 0, 1], [1, 2, 3],                  # rows 6..8
    [2, 0, 0], [2, K, 0], [2, 0, 1],                  # rows 9..11: row 10 is not retrievable
    [3, 3, 3],                                        # row 12
], dtype=np.int64)


def key(*t):
    return X.tuple_key(t, K)


def table():
    return IO.build(CORPUS, K)


def padded(rows, M=16):
    return np.array([list(rows) + [-1] * (M - len(rows))], dtype=np.int64)


CASES = {
    # name: (allowed, excluded, eligible rows, valid keys per level 1..H, bad)
    "one_item": ([5], [], {5}, ([key(0)], [key(0, 1)], [key(0, 1, 3)]), 0),
    "dedup_ranks": ([2, 0], [], {0, 2}, ([key(0)], [key(0, 0)], [key(0, 0, 0)]), 0),
    "repeats_and_padding": ([-1, 7, 7, -1, 12], [], {7, 12},
                            ([key(1), key(3)], [key(1, 0), key(3, 3)], [key(1, 0, 1), key(3, 3, 3)]), 0),
    "unretrievable": ([10, 9], [], {9}, ([key(2)], [key(2, 0)], [key(2, 0, 0)]), 0),
    "only_unretrievable": ([10, -1], [], set(), ([], [], []), 0),
    "out_of_range": ([13, -2, 8, 99], [], {8}, ([key(1)], [key(1, 2)], [key(1, 2, 3)]), 3),
    "with_exclusion": ([0, 1, 6, 7], [1, 7, 12], {0, 6}, ([key(0), key(1)], [key(0, 0), key(1, 0)],
                                                          [key(0, 0, 0), key(1, 0, 0)]), 0),
    "all_excluded": ([4, 5], [4, 5], set(), ([], [], []), 0),
    "empty": ([], [], set(), ([], [], []), 0),
}


def build_case(name):
    allowed, excluded = CASES[name][:2]
    t = table()
    excls = X.build(t, padded(excluded)) if excluded else None
    return I.build(t, padded(allowed), excls)[0]


@pytest.mark.parametrize("name", sorted(CASES))
def test_eligible_and_valid_prefixes(name):
    _, _, eligible, keys, bad = CASES[name]
    incl = build_case(name)
    t = table()
    assert incl["eligible"] == eligible
    assert incl["bad"] == bad
    inv = {int(r): p for p, r in enumerate(t["row"])}
    assert incl["pos"] == sorted(inv[r] for r in eligible)
    for l in range(1, H + 1):
        assert incl["keys"][l] == sorted(keys[l - 1]), l


@pytest.mark.parametrize("name", sorted(CASES))
def test_valid_prefix_equals_brute_force(name):
    incl = build_case(name)
    t = table()
    for l in range(1, H + 1):
        for prefix in itertools.product(range(-1, K + 1), repeat=l):
            assert I.valid_prefix(incl, prefix, K) == I.valid_prefix_brute(CORPUS, t, incl["eligible"], prefix), prefix


def test_positions_are_ascending_keys_distinct():
    rs = np.random.RandomState(0)
    corpus = rs.randint(0, 5, size=(200, H)).astype(np.int64)
    t = IO.build(corpus, 5)
    items = rs.randint(-1, 200, size=(6, 60))
    excls = X.build(t, rs.randint(-1, 200, size=(6, 30)))
    for incl, ex in zip(I.build(t, items, excls), excls):
        assert incl["pos"] == sorted(set(incl["pos"]))
        assert not incl["eligible"] & ex["excluded"]
        for l in range(1, H + 1):
            want = sorted(set(X.tuple_key(corpus[r, :l], 5) for r in incl["eligible"]))
            assert incl["keys"][l] == want


def test_beam_level_with_fillers():
    """Two valid first codes for the history: the two best valid extensions, then -inf fillers by ascending code."""
    incl = build_case("repeats_and_padding")
    logits = np.array([[0.0, 1.0, 2.0, 3.0]])
    gen, lp, parent = I.beam_topk(CORPUS, K, [incl], logits, None, None, 4)
    assert gen[0, :, 0].tolist() == [3, 1, 0, 2]
    assert np.isfinite(lp[0, :2]).all() and np.isneginf(lp[0, 2:]).all()
    assert parent[0].tolist() == [0, 0, 0, 0]
    gen2, lp2, parent2 = I.beam_topk(CORPUS, K, [incl], np.zeros((4, K)), gen, lp, 3)
    assert gen2[0].tolist() == [[3, 3], [1, 0], [3, 0]]                    # (3, 3) and (1, 0), then filler e = 0
    assert parent2[0].tolist() == [0, 1, 0] and np.isneginf(lp2[0, 2])


def test_beam_level_equals_brute_force():
    rs = np.random.RandomState(1)
    incls = [build_case(n) for n in sorted(CASES)]
    B = len(incls)
    logits = rs.randn(B, K)
    scores = I.candidate_scores(CORPUS, K, incls, logits, None, None)
    for b in range(B):
        for c in range(K):
            ok = I.valid_prefix_brute(CORPUS, table(), incls[b]["eligible"], [c])
            assert np.isfinite(scores[b, c]) == ok


def test_sample_scores():
    incl = build_case("with_exclusion")
    samples = np.array([[0, 1, 2, 3]])
    samp_log_p = np.log(np.full((1, 4), 0.25))
    s = I.sample_scores([incl], K, samples, samp_log_p, None, None)
    assert np.isfinite(s[0]).tolist() == [True, True, False, False]


def test_retrieve():
    t = table()
    incl = build_case("dedup_ranks")
    other = build_case("with_exclusion")
    gen = np.array([[[0, 0, 0], [0, 0, 0], [1, 0, 0], [3, 3, 3]]] * 2)
    lp = np.array([[-1.0, -2.0, -3.0, -np.inf]] * 2)
    items, beam, count = I.retrieve(t, [incl, other], gen, lp, 5)
    assert items[0].tolist() == [0, 2, -1, -1, -1] and beam[0].tolist() == [0, 0, -1, -1, -1] and count[0] == 2
    assert items[1].tolist() == [0, 6, -1, -1, -1] and beam[1].tolist() == [0, 2, -1, -1, -1] and count[1] == 2
    items, _, count = I.retrieve(t, [build_case("empty")] * 2, gen, lp, 5)
    assert (count == 0).all() and (items == -1).all()
