"""CPU tests of the exclusion oracle (tests/exclusion_oracle.py) on a small hand-made corpus whose blocked prefixes, retrieved
items and ranks are worked out by hand: colliding tuples of dedup ranks 0..3, part and all of a tuple excluded, a whole level-1
subtree, repeats and -1 padding, unretrievable rows, ids outside [-1, N) and a history that excludes every item."""
import numpy as np
import pytest

import exclusion_oracle as X
import item_oracle as IO

K, H = 4, 3
CORPUS = np.array([
    [0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0],       # rows 0..3: one tuple, dedup ranks 0..3
    [0, 1, 2], [0, 1, 3],                             # rows 4, 5
    [1, 0, 0], [1, 0, 1], [1, 2, 3],                  # rows 6..8: the level-1 subtree (1,)
    [2, 0, 0], [2, K, 0], [2, 0, 1],                  # rows 9..11: row 10 is not retrievable
    [3, 3, 3],                                        # row 12
], dtype=np.int64)


def key(*t):
    return X.tuple_key(t, K)


def table():
    return IO.build(CORPUS, K)


CASES = {
    # name: (items, excluded rows, blocked keys per level 1..H, bad)
    "part_of_tuple": ([0, 1], {0, 1}, ([], [], []), 0),
    "all_of_tuple": ([3, 1, 0, 2], {0, 1, 2, 3}, ([], [key(0, 0)], [key(0, 0, 0)]), 0),
    "level1_subtree": ([6, 7, 8], {6, 7, 8}, ([key(1)], [key(1, 0), key(1, 2)], [key(1, 0, 0), key(1, 0, 1), key(1, 2, 3)]), 0),
    "repeats_and_padding": ([-1, 6, 6, -1, 7], {6, 7}, ([], [key(1, 0)], [key(1, 0, 0), key(1, 0, 1)]), 0),
    # row 10 (2, K, 0) is not retrievable: it is ignored, and (2,) is blocked once its retrievable rows 9 and 11 are excluded
    "unretrievable": ([10, 9, 11], {9, 11}, ([key(2)], [key(2, 0)], [key(2, 0, 0), key(2, 0, 1)]), 0),
    "only_unretrievable": ([10, -1], set(), ([], [], []), 0),
    "out_of_range": ([13, -2, 5, 99], {5}, ([], [], [key(0, 1, 3)]), 3),
    "everything": (list(range(13)), set(range(13)) - {10},
                   ([key(0), key(1), key(2), key(3)],
                    [key(0, 0), key(0, 1), key(1, 0), key(1, 2), key(2, 0), key(3, 3)],
                    [key(0, 0, 0), key(0, 1, 2), key(0, 1, 3), key(1, 0, 0), key(1, 0, 1), key(1, 2, 3), key(2, 0, 0),
                     key(2, 0, 1), key(3, 3, 3)]), 0),
}


def build_case(name):
    items = CASES[name][0]
    return X.build(table(), np.array([items + [-1] * (13 - len(items))], dtype=np.int64))[0]


@pytest.mark.parametrize("name", sorted(CASES))
def test_blocked_prefixes(name):
    _, excluded, blocked, bad = CASES[name]
    ex = build_case(name)
    t = table()
    assert ex["excluded"] == excluded
    assert ex["bad"] == bad
    for l in range(1, H + 1):
        assert ex["blocked"][l] == sorted(blocked[l - 1]), l
    inv = {int(r): p for p, r in enumerate(t["row"])}
    assert ex["pos"] == sorted(inv[r] for r in excluded)
    assert all(p < t["start"][-1] for p in ex["pos"])           # only retrievable rows have positions


def test_prefix_validity():
    ex = build_case("all_of_tuple")
    assert not X.valid_prefix(CORPUS, K, ex, [0, 0])
    assert not X.valid_prefix(CORPUS, K, ex, [0, 0, 0])
    assert X.valid_prefix(CORPUS, K, ex, [0]) and X.valid_prefix(CORPUS, K, ex, [0, 1])
    ex = build_case("unretrievable")
    assert not X.valid_prefix(CORPUS, K, ex, [2])
    assert X.valid_prefix(CORPUS, K, build_case("part_of_tuple"), [2, K])   # a corpus prefix of an unretrievable row
    assert not X.valid_prefix(CORPUS, K, build_case("part_of_tuple"), [2, 3])   # not a corpus prefix at all
    none = build_case("only_unretrievable")
    for t in map(tuple, CORPUS):
        for l in range(1, H + 1):
            assert X.valid_prefix(CORPUS, K, none, t[:l])


def test_candidate_scores_mask_blocked_extensions():
    excls = [build_case("level1_subtree"), build_case("only_unretrievable")]
    logits = np.zeros((2, K), dtype=np.float32)
    s = X.candidate_scores(CORPUS, K, excls, logits, None, None)
    assert np.isneginf(s[0, 1]) and np.isfinite(s[0, [0, 2, 3]]).all()
    assert np.isfinite(s[1]).all()
    generated = np.array([[[0, 0]], [[0, 0]]], dtype=np.int64)
    excls = [build_case("all_of_tuple"), build_case("part_of_tuple")]
    s = X.candidate_scores(CORPUS, K, excls, logits, generated, np.zeros((2, 1)))
    assert np.isneginf(s[0]).all()                                  # (0, 0, 0) is blocked, (0, 0, c > 0) not in the corpus
    assert np.isfinite(s[1, 0]) and np.isneginf(s[1, 1:]).all()


def test_retrieve():
    t = table()
    generated = np.array([[[0, 0, 0], [1, 0, 0], [0, 0, 0], [3, 3, 3]]] * 3, dtype=np.int64)
    log_probas = np.array([[-1.0, -2.0, -3.0, -4.0]] * 3)
    excls = [build_case("part_of_tuple"), build_case("all_of_tuple"), build_case("everything")]
    items, beam, count = X.retrieve(t, excls, generated, log_probas, 6)
    assert items[0].tolist() == [2, 3, 6, 12, -1, -1] and beam[0].tolist() == [0, 0, 1, 3, -1, -1] and count[0] == 4
    assert items[1].tolist() == [6, 12, -1, -1, -1, -1] and beam[1].tolist() == [1, 3, -1, -1, -1, -1] and count[1] == 2
    assert count[2] == 0 and (items[2] == -1).all()
    ref = IO.retrieve(t, generated, log_probas, 6)                  # an empty set is item_oracle.retrieve
    got = X.retrieve(t, [build_case("only_unretrievable")] * 3, generated, log_probas, 6)
    for a, b in zip(ref, got):
        np.testing.assert_array_equal(a, b)


def test_rank_select():
    t = table()
    U = len(t["keys"])                                              # 9 leaves: (0,0,0) (0,1,2) (0,1,3) (1,0,0) (1,0,1) ...
    assert U == 9
    scores = np.array([[-1.0, -5.0, -2.0, -3.0, np.nan, -4.0, -6.0, -7.0, -8.0]] * 4, dtype=np.float32)
    excls = [build_case("only_unretrievable"), build_case("part_of_tuple"), build_case("all_of_tuple"), build_case("everything")]
    t_leaf = np.array([0, 0, 2, 0])
    t_dedup = np.array([2, 0, 0, 0])
    items, s, rank = X.rank_select(t, excls, scores, t_leaf, t_dedup, 7)
    # leaf order: 0 (rows 0..3), 2 (row 5), 3 (row 6), 5 (row 8), 1 (row 4), 6 (row 9), 7 (row 11), 8 (row 12), 4 (NaN, row 7)
    assert items[0].tolist() == [0, 1, 2, 3, 5, 6, 8] and rank[0] == 2
    assert items[1].tolist() == [2, 3, 5, 6, 8, 4, 9] and rank[1] == -1      # the target, row 0, is excluded
    assert items[2].tolist() == [5, 6, 8, 4, 9, 11, 12] and rank[2] == 0
    np.testing.assert_array_equal(s[2], np.array([-2, -3, -4, -5, -6, -7, -8], dtype=np.float32))
    assert (items[3] == -1).all() and np.isneginf(s[3]).all() and rank[3] == -1
    t_dedup[1] = 3
    assert X.rank_select(t, excls, scores, t_leaf, t_dedup, 7)[2][1] == 1     # row 3 follows row 2 once rows 0, 1 are gone


@pytest.mark.parametrize("K,H,accepted", [(2048, 6, False), (256, 8, False), (1024, 6, True), (2048, 5, True)])
def test_filter_entry_points_take_keys_of_at_most_62_bits(K, H, accepted):
    """rqb200_sid_exclusion_build and rqb200_sid_inclusion_build refuse H * bits(K - 1) > 62 (66 and 64 bits here) before
    reading any pointer, and take 60 and 55 bits (B = 0: nothing to launch)."""
    from rq_vae_recommender_b200 import _lib
    lib = _lib.load()
    calls = {"sid_exclusion_build": lambda B: lib.rqb200_sid_exclusion_build(0, B, 4, 10, 0, 0, 0, 5, H, K, 0, 0, 0, 0),
             "sid_inclusion_build": lambda B: lib.rqb200_sid_inclusion_build(0, B, 4, 10, 0, 0, 0, 5, H, K, 0, 0, 0, 0, 0, 0, 0,
                                                                             0, 0)}
    for name, call in calls.items():
        if accepted:
            assert call(0) == 0
            assert call(1) == 1 and b"null pointer" in lib.rqb200_last_error()
        else:
            assert call(1) == 3
            msg = lib.rqb200_last_error().decode()
            assert msg.startswith(name) and "H * bits(K - 1) <= 62" in msg and f"H = {H}, K = {K}" in msg
