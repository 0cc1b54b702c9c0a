"""The rule of generate(search="exact") stated in numpy (no GPU): on a trie whose child scores are the parent's plus a
log-probability <= 0, decoding level by level only the nodes with score >= tau that the filter allows, then selecting the w best
leaves (score descending, leaf ascending, NaN and blocked leaves left out), gives the dense sort's top w for every tau at or
below the true w-th score.  Random tries with shared prefixes, single-child chains and K not a power of two; ties at tau; -inf
log-probabilities; blocked (exclusion) and allowed (allow-list) prefix sets."""
import numpy as np
import pytest


def trie(corpus):
    """levels[l]: the sorted distinct l-prefixes (tuples), l = 0..H; parent[l][i]: node i's node in level l - 1."""
    H = corpus.shape[1]
    levels = [[()]] + [sorted({tuple(r[:l]) for r in corpus.tolist()}) for l in range(1, H + 1)]
    index = [{p: i for i, p in enumerate(lv)} for lv in levels]
    parent = [None] + [np.array([index[l - 1][p[:-1]] for p in levels[l]]) for l in range(1, H + 1)]
    return levels, parent


def node_scores(rs, levels, parent, ties):
    """fp32 score of every node, level by level: parent + a log-probability <= 0 (some -inf, some from a small set: ties)."""
    scores = [np.zeros(1, dtype=np.float32)]
    for l in range(1, len(levels)):
        n = len(levels[l])
        lp = -rs.exponential(1.0, size=n).astype(np.float32)
        lp[rs.rand(n) < 0.3] = np.float32(-0.5)              # equal log-probabilities give equal leaf scores
        if ties:
            lp[rs.rand(n) < 0.3] = np.float32(0.0)
        lp[rs.rand(n) < 0.05] = -np.inf
        scores.append((scores[l - 1][parent[l]] + lp).astype(np.float32))
    return scores


def allowed_mask(levels, prefixes, mode):
    """Per level, whether each node is valid: exclusion -- not under a blocked prefix; allow-list -- under an allowed one."""
    out = []
    for l in range(len(levels)):
        if mode == "exclude":
            out.append(np.array([not any(p[:len(q)] == q for q in prefixes) for p in levels[l]]))
        elif mode == "include":
            out.append(np.array([any(p[:len(q)] == q or q[:len(p)] == p for q in prefixes) for p in levels[l]]))
        else:
            out.append(np.ones(len(levels[l]), dtype=bool))
    return out


def dense_top(scores, valid, w):
    s = scores[-1]
    idx = np.nonzero(valid[-1] & ~np.isnan(s))[0]
    return idx[np.lexsort((idx, -s[idx]))][:w]


def pruned_top(scores, parent, valid, w, tau):
    """Level by level from the root: the children of the kept nodes, kept when score >= tau and valid; then the selection."""
    H = len(scores) - 1
    kept = np.array([0])
    rows = 1
    for l in range(1, H + 1):
        children = np.nonzero(np.isin(parent[l], kept))[0]       # in trie order
        if l < H:
            kept = children[(scores[l][children] >= tau) & valid[l][children]]
            rows += len(kept)
    s = scores[H][children]
    ok = valid[H][children] & ~np.isnan(s)
    cand, s = children[ok], s[ok]
    return cand[np.lexsort((cand, -s))][:w], rows


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("mode", ["none", "exclude", "include"])
def test_pruned_decode_equals_dense_sort(seed, mode):
    rs = np.random.RandomState(seed)
    K, H = [(7, 3), (5, 4), (13, 2), (3, 5)][seed % 4]
    N = rs.randint(5, 120)
    corpus = rs.randint(0, K, size=(N, H))
    corpus[: N // 4, : H - 1] = corpus[N // 4, : H - 1]          # shared prefixes
    corpus[N // 2] = corpus[0]                                    # a duplicate
    chain = rs.randint(0, K, size=H)
    chain[0] = K - 1
    corpus = np.concatenate([corpus, chain[None]], 0)             # a single-child chain under a fresh first code
    corpus = corpus[(corpus[:, 0] != K - 1) | (np.arange(len(corpus)) == len(corpus) - 1)]
    levels, parent = trie(corpus)
    scores = node_scores(rs, levels, parent, ties=seed % 2 == 0)
    prefixes = [tuple(corpus[rs.randint(len(corpus))][: rs.randint(1, H + 1)]) for _ in range(3)]
    valid = allowed_mask(levels, prefixes, mode)
    U = len(levels[H])
    for w in sorted({1, 2, 5, U, U + 3}):
        want = dense_top(scores, valid, w)
        finite = np.sort(scores[H][valid[H] & np.isfinite(scores[H])])[::-1]
        true_tau = finite[w - 1] if len(finite) >= w else -np.inf
        for tau in {true_tau, np.float32(true_tau - 0.25), np.float32(true_tau - 3.0), -np.inf}:
            got, rows = pruned_top(scores, parent, valid, w, tau)
            assert np.array_equal(got, want), (w, tau)
            assert rows <= sum(len(lv) for lv in levels[:H])

