"""Numpy restatement of the corpus trie (csrc/sid.cu: rqb200_sid_trie_build and the SidTrie lookups).  Level l = 1..C holds the
distinct l-prefixes of the corpus rows, each row cut at its first id outside [0, K), in lexicographic order: codes[l][i] is node
i's last code, and for l < C its children are nodes [child[l][i], child[l][i + 1]) of level l + 1 (level 0 is the root:
child[0] = [0, n[1]])."""
import numpy as np


def build(corpus_ids, K):
    corpus = np.asarray(corpus_ids, dtype=np.int64)
    N, C = corpus.shape
    depth = np.cumprod((corpus >= 0) & (corpus < K), axis=1).sum(axis=1)
    enc = np.where(np.arange(C)[None, :] < depth[:, None], corpus, K)        # the rest of a row sorts after every code
    order = np.lexsort(enc.T[::-1]) if N else np.zeros(0, dtype=np.int64)
    enc, depth = enc[order], depth[order]
    lcp = np.zeros(N, dtype=np.int64)
    if N > 1:
        lcp[1:] = np.minimum(np.cumprod(enc[1:] == enc[:-1], axis=1).sum(axis=1), np.minimum(depth[1:], depth[:-1]))
    level = np.arange(1, C + 1)[None, :]
    flag = (level > lcp[:, None]) & (level <= depth[:, None])                # [N, C]: row r starts a node of level l
    before = np.cumsum(flag, axis=0) - flag                                  # nodes of each level started before row r
    n = [1] + [int(flag[:, l].sum()) for l in range(C)]
    codes = [None] + [enc[flag[:, l], l] for l in range(C)]
    child = [np.array([0, n[1]], dtype=np.int64)]
    for l in range(1, C):
        child.append(np.append(before[flag[:, l - 1], l], n[l + 1]))
    return dict(C=C, K=K, n=n, codes=codes, child=child)


def lookup(trie, prefix):
    """bool [P]: prefix[p] ([P, l], l <= C) is a corpus prefix -- a walk of l binary searches."""
    prefix = np.asarray(prefix, dtype=np.int64)
    K = trie["K"]
    out = np.zeros(prefix.shape[0], dtype=bool)
    for p, ids in enumerate(prefix):
        lo, hi = trie["child"][0]
        for j, v in enumerate(ids):
            if not 0 <= v < K:
                break
            codes = trie["codes"][j + 1]
            i = lo + int(np.searchsorted(codes[lo:hi], v))
            if i >= hi or codes[i] != v:
                break
            if j + 1 == len(ids):
                out[p] = True
            else:
                lo, hi = trie["child"][j + 1][i], trie["child"][j + 1][i + 1]
    return out


def valid_prefixes(corpus_ids, prefix, K):
    """The prefix indexes' semantics from oracle.rq_oracle.check_valid_prefix: a corpus prefix holding no id outside [0, K)."""
    from oracle import rq_oracle as O
    prefix = np.asarray(prefix, dtype=np.int64)
    return O.check_valid_prefix(np.asarray(corpus_ids), prefix) & ((prefix >= 0) & (prefix < K)).all(axis=1)
