"""The exact search's kernel statements (tests/exact_oracle.py) composed as generate(search="exact") composes the kernels: the
frontier level by level from the root, then the selection, equal the dense sort of tests/test_exact_search_model.py (dense_top)
for every tau at or below the true w-th score, and for a chunk of the batch (b0 > 0).  Random tries with K not a power of two,
shared prefixes and single-child chains; exact ties at tau; -inf scores; exclusion and allow-list filters.  No GPU."""
import numpy as np
import pytest

import exact_oracle as EO
import trie_oracle as TO
from exclusion_oracle import tuple_key
from test_exact_search_model import allowed_mask, dense_top, node_scores, trie


def random_corpus(rs, K, H):
    N = rs.randint(5, 120)
    corpus = rs.randint(0, K, size=(N, H))
    corpus[: N // 4, : H - 1] = corpus[N // 4, : H - 1]          # shared prefixes
    chain = rs.randint(0, K, size=H)
    chain[0] = K - 1
    corpus = corpus[corpus[:, 0] != K - 1]
    return np.concatenate([corpus, chain[None]], 0)               # a single-child chain under a fresh first code


def composed(tr, scores, valid, tau, w, b0):
    """The frontier statement from the root to level H - 1, then the selection, for histories b0 .. B - 1 (chunk-local b)."""
    H = tr["C"]
    Bc = len(scores) - b0
    ch = EO.root_children(np.stack([scores[b0 + b][1] for b in range(Bc)]), tr["codes"][1])
    rows, ties = 0, 0
    for l in range(1, H):
        out = EO.frontier(ch, tau[b0:], tr["child"][l], tr["codes"][l + 1], tr["K"], l, valid, b0)
        rows += len(out["code"])
        ties += int(out["at_tau"].sum())
        hist = np.repeat(np.arange(Bc), out["counts"][1])           # each next child's history
        nxt = np.array([scores[b0 + b][l + 1][n] for b, n in zip(hist, out["nnode"])], dtype=np.float32)
        ch = EO.next_children(out, nxt)
    return EO.select(ch, w, tr["codes"], [None] + tr["parents"][1:], tr["leaf_key"], valid, b0), rows, ties


@pytest.mark.parametrize("seed", range(10))
@pytest.mark.parametrize("mode", ["none", "exclude", "include"])
def test_composed_statements_equal_dense_top(seed, mode):
    rs = np.random.RandomState(100 + seed)
    K, H = [(7, 3), (5, 4), (13, 2), (3, 5), (6, 3)][seed % 5]
    corpus = random_corpus(rs, K, H)
    levels, parent = trie(corpus)
    tr = TO.build(corpus, K)
    for l in range(1, H + 1):                                     # the two statements of the trie agree on node order
        assert [p[-1] for p in levels[l]] == tr["codes"][l].tolist()
    tr["parents"] = parent
    keys = [None] + [np.array([tuple_key(p, K) for p in levels[l]], dtype=np.int64) for l in range(1, H + 1)]
    tr["leaf_key"] = keys[H]
    B = 4
    scores, valid_keys = [], []
    for b in range(B):
        scores.append(node_scores(rs, levels, parent, ties=(seed + b) % 2 == 0))
        prefixes = [tuple(corpus[rs.randint(len(corpus))][: rs.randint(1, H + 1)]) for _ in range(2 + b)]
        ok = allowed_mask(levels, prefixes, mode)
        valid_keys.append([None] + [keys[l][ok[l]] for l in range(1, H + 1)])
    valid = None if mode == "none" else (lambda bg, l, k: np.isin(k, valid_keys[bg][l]))
    U = len(levels[H])
    ties = 0
    for w in sorted({1, 2, 5, U, U + 3}):
        want_leaf, true_tau = [], np.zeros(B, dtype=np.float32)
        for b in range(B):
            ok = [np.ones(1, dtype=bool)] + [np.isin(keys[l], valid_keys[b][l]) for l in range(1, H + 1)]
            want_leaf.append(dense_top(scores[b], ok, w))
            finite = np.sort(scores[b][H][ok[H] & np.isfinite(scores[b][H])])[::-1]
            true_tau[b] = finite[w - 1] if len(finite) >= w else -np.inf
        for shift in (0.0, 0.25, 3.0, np.inf):
            tau = (true_tau - np.float32(shift)).astype(np.float32)
            for b0 in (0, 1):
                (gen, lp), rows, at_tau = composed(tr, scores, valid, tau, w, b0)
                ties += at_tau if shift == 0.0 else 0
                assert rows <= (B - b0) * sum(len(lv) for lv in levels[1:H])
                for b in range(b0, B):
                    want = want_leaf[b]
                    n = len(want)
                    assert np.array_equal(gen[b - b0, :n], np.array(levels[H], dtype=np.int64).reshape(-1, H)[want]), (w, b)
                    assert np.array_equal(lp[b - b0, :n].view(np.int32), scores[b][H][want].view(np.int32)), (w, b)
                    assert (gen[b - b0, n:] == -1).all() and (lp[b - b0, n:] == -np.inf).all()
    if seed % 2 == 0:
        assert ties > 0                                           # node_scores' 0.0 log-probabilities tie a path node at tau


def test_statement_edges():
    """The frontier keeps -inf under tau = -inf and never NaN; its tile table and child ranges at 63 / 64 / 65 / 129 rows; an
    empty history in the middle and at the end; the selection folds -0.0 into +0.0 and pads past the valid candidates."""
    K, n1 = 300, 300
    child1 = np.arange(n1 + 1, dtype=np.int64) * 2                 # two children per level-1 node
    code2 = np.arange(2 * n1, dtype=np.int64) % K
    first = np.full((7, n1), np.float32(-1.0))
    first[0, :5] = [np.nan, -np.inf, 0.0, -0.0, np.nan]
    tau = np.array([-np.inf, 0, 0, 0, np.inf, 0, np.inf], dtype=np.float32)
    for b, k in zip((1, 2, 3, 5), (63, 64, 65, 129)):
        first[b, :k] = 0.5
    out = EO.frontier(EO.root_children(first, np.arange(n1) % K), tau, child1, code2, K, 1)
    assert out["counts"][0].tolist() == [n1 - 2, 63, 64, 65, 0, 129, 0]
    assert out["counts"][2].tolist() == [5, 1, 1, 2, 0, 3, 0]
    assert -np.inf in out["score"][:n1 - 2] and not np.isnan(out["score"]).any()
    assert [t[2] for t in out["tiles"] if t[0] == 3] == [64, 1] and [t[2] for t in out["tiles"] if t[0] == 5] == [64, 64, 1]
    assert out["child"][-1] == len(out["nnode"]) == 2 * out["counts"][0].sum()
    assert (out["npar"][out["child"][:-1]] == np.arange(len(out["code"]))).all()
    ch = dict(scores=np.array([-0.0, 0.0, np.nan, -np.inf, -0.0], dtype=np.float32), offsets=np.array([0, 5, 5]),
              node=np.arange(5), code=None, parent=None, pkey=None)
    codes, parents = [None, np.arange(5) + 10], [None, np.zeros(5, dtype=np.int64)]
    gen, lp = EO.select(ch, 6, codes, parents)
    assert gen[0, :, 0].tolist() == [10, 11, 14, 13, -1, -1] and gen[1].ravel().tolist() == [-1] * 6
    assert lp[0].view(np.int32).tolist() == np.array([-0.0, 0.0, -0.0, -np.inf, -np.inf, -np.inf], np.float32).view(np.int32).tolist()
