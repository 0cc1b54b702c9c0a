"""CPU tests of the corpus trie's numpy restatement (trie_oracle) against oracle.rq_oracle.check_valid_prefix on random corpora
with duplicated rows and ids outside [0, K), and of the rule by which ops.SidPrefixIndex picks its index."""
import numpy as np
import pytest

import trie_oracle as T


def random_corpus(rs, N, C, K):
    corpus = rs.randint(0, K, size=(N, C)).astype(np.int64)
    if N > 4:
        corpus[: N // 4, : max(1, C // 2)] = rs.randint(0, min(K, 4), size=(N // 4, max(1, C // 2)))   # shared prefixes
        corpus[N // 3: N // 3 + N // 5] = corpus[: N // 5]                                            # duplicated rows
        bad = rs.rand(N, C) < 0.05                                                                     # ids outside [0, K)
        corpus[bad] = rs.choice([-1, K, K + 7, -(1 << 40)], size=int(bad.sum()))
    return corpus


def prefixes(rs, corpus, l, K, n=300):
    """corpus prefixes, corpus prefixes with one id changed, random prefixes and prefixes holding ids outside [0, K)"""
    parts = [rs.randint(0, K, size=(n, l))]
    if len(corpus):
        rows = corpus[rs.randint(0, len(corpus), size=n), :l]
        changed = rows.copy()
        changed[np.arange(n), rs.randint(0, l, size=n)] = rs.randint(0, K, size=n)
        parts += [rows, changed]
    odd = rs.randint(0, K, size=(n // 4, l))
    odd[np.arange(n // 4), rs.randint(0, l, size=n // 4)] = rs.choice([-1, K, K + 3], size=n // 4)
    return np.concatenate(parts + [odd]).astype(np.int64)


@pytest.mark.parametrize("K", [16, 256, 2048])
@pytest.mark.parametrize("C", range(1, 9))
@pytest.mark.parametrize("N", [0, 1, 600])
def test_trie_lookup_equals_check_valid_prefix(K, C, N):
    rs = np.random.RandomState(K * 100 + C * 10 + N)
    corpus = random_corpus(rs, N, C, K)
    trie = T.build(corpus, K)
    for l in range(1, C + 1):
        p = prefixes(rs, corpus, l, K)
        want = T.valid_prefixes(corpus, p, K)
        assert np.array_equal(T.lookup(trie, p), want), l
        if N > 1 and l == 1:
            assert want.any() and not want.all()
    # the structure: n[l] distinct valid l-prefixes, children contiguous and sorted by code
    depth = np.cumprod((corpus >= 0) & (corpus < K), axis=1).sum(axis=1)
    for l in range(1, C + 1):
        distinct = {tuple(r[:l]) for r, d in zip(corpus.tolist(), depth) if d >= l}
        assert trie["n"][l] == len(distinct) == len(trie["codes"][l])
    for l in range(C):
        ch = trie["child"][l]
        assert len(ch) == trie["n"][l] + 1 and ch[0] == 0 and ch[-1] == trie["n"][l + 1] and (np.diff(ch) >= 0).all()
        codes = trie["codes"][l + 1]
        for i in range(trie["n"][l]):
            assert (np.diff(codes[ch[i]:ch[i + 1]]) > 0).all()


def test_duplicates_only_and_invalid_first_ids():
    K = 16
    corpus = np.array([[3, 4, 5]] * 5 + [[-1, 2, 2], [16, 0, 0], [3, 99, 1]], dtype=np.int64)
    trie = T.build(corpus, K)
    assert trie["n"] == [1, 1, 1, 1]
    assert T.lookup(trie, [[3], [2], [16], [-1]]).tolist() == [True, False, False, False]
    assert T.lookup(trie, [[3, 4], [3, 99], [-1, 2]]).tolist() == [True, False, False]
    assert T.lookup(trie, [[3, 4, 5], [3, 99, 1]]).tolist() == [True, False]


@pytest.mark.parametrize("K", [16, 256, 512, 1024, 2048])
@pytest.mark.parametrize("C", range(1, 9))
def test_index_choice_follows_bitmap_limit(K, C):
    """The bitmap wherever K^C fits its 2^33 bits (every shape that had an index before keeps it), the trie elsewhere."""
    from rq_vae_recommender_b200 import ops
    assert ops.SidPrefixIndex.kind_for(C, K) == ("bitmap" if K ** C <= 1 << 33 else "trie")


def test_index_choice_at_the_named_shapes():
    from rq_vae_recommender_b200 import ops
    kind = ops.SidPrefixIndex.kind_for
    assert [kind(3, 256), kind(4, 256), kind(3, 2048), kind(8, 16)] == ["bitmap"] * 4
    assert [kind(5, 256), kind(8, 256), kind(4, 512), kind(4, 2048), kind(8, 2048)] == ["trie"] * 5


def test_index_rejects_cpu_tensors_and_unknown_kinds():
    import torch
    from rq_vae_recommender_b200 import _lib, ops
    with pytest.raises(_lib.Rqb200Error):
        ops.SidPrefixIndex(torch.zeros((4, 5), dtype=torch.int64), 256)
    with pytest.raises(_lib.Rqb200Error):
        ops.SidPrefixIndex(torch.zeros((4, 5), dtype=torch.int64), 256, kind="trie")
