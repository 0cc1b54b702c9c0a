"""CPU tests of the corpus trie's numpy restatement (trie_oracle) against oracle.rq_oracle.check_valid_prefix on random corpora
with duplicated rows and ids outside [0, K), and of the trie's size and index construction without a device."""
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


def test_trie_bytes_without_a_device_below_the_corpus_table():
    """The trie's persistent bytes are arithmetic (no device is queried) and, at the shipped shape and at a million rows, fewer
    than those of the int64 corpus table [N, C] it indexes."""
    from rq_vae_recommender_b200 import _lib
    lib = _lib.load()
    for N, C, K in ((12101, 3, 256), (1 << 20, 3, 256)):
        nbytes = lib.rqb200_sid_trie_workspace_bytes(N, C, K)
        assert 0 < nbytes < N * C * 8, (N, nbytes)
    assert lib.rqb200_sid_trie_workspace_bytes(0x7fffffff, 3, 256) == 0                 # outside the trie's limits


def test_index_rejects_cpu_tensors():
    import torch
    from rq_vae_recommender_b200 import _lib, ops
    with pytest.raises(_lib.Rqb200Error):
        ops.SidPrefixIndex(torch.zeros((4, 5), dtype=torch.int64), 256)
