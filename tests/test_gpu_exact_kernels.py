"""GPU tests of the exact top-k search's kernels (csrc/t5rank.cu t5exact_frontier_kernel<FILTER, WRITE> and
t5exact_select_kernel<KEYS_IN_SMEM, FILTER>, behind ops.t5exact_frontier_count / _write and ops.t5exact_select) against the
numpy statement of tests/exact_oracle.py, bit for bit, and under the model (generate(search="exact")).

Frontier: the count pass, the host scan and the write pass as FusedT5Exact.run drives them, walked from the root over tries of
K = 300 / 2048 with H = 3 / 5 and K = 128 with H = 8, chunks of 1, 7 and 300 histories at b0 = 0 and b0 > 0, each filter mode;
then targeted inputs: 0, 1, 255, 256, 257 and 3000 children per history, tau -inf / +inf / on a shared score / keeping exactly 63,
64, 65 and 129 rows, empty frontiers in the middle and at the end of the chunk, NaN / -inf / +-0.0 scores.  Select: 0, 1, w - 1, w,
w + 1, 24 576, 24 577 and 60 000 candidates per history (both sides of RK_SEL_SMEM_KEYS), w = 1 / 10 / 1024, all-equal and random
scores, each filter mode, b0 > 0, and the root's children of a one-column corpus.  Model: more than 24 576 leaf candidates per
history, chunk reruns with each filter, and each level's frontier on sharpened heads, where nodes tie tau exactly.
`pytest -m gpu`."""
import functools

import numpy as np
import pytest
import torch

import exact_oracle as EO
import exclusion_oracle as X
import inclusion_oracle as I
import item_oracle as IO
import trie_oracle as TO
from test_gpu_exact_search import dense_topw, leaf_tuples, sharpen
from test_gpu_exclusion import built as excl_built
from test_gpu_exclusion import corpus_with_subtrees, exclusion_sets
from test_gpu_generate import history, realistic_corpus
from test_gpu_inclusion import allow_lists
from test_gpu_inclusion import built as incl_built
from test_gpu_rank import batch_for, model_for

pytestmark = pytest.mark.gpu

SMEM_KEYS = 24 * 1024                # RK_SEL_SMEM_KEYS: above it t5exact_select recomputes every key on each radix pass
FILTERS = ("none", "exclude", "include")
SHARED = np.float32(1.5)             # a score several children share


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def assert_ints(got, want, what):
    got = host(got).astype(np.int64)
    want = np.asarray(want, dtype=np.int64).reshape(got.shape)
    assert np.array_equal(got, want), what


def assert_bits(got, want, what):
    assert np.array_equal(host(got).view(np.int32), np.asarray(want, dtype=np.float32).view(np.int32)), what


class Trie:
    """A corpus's trie as the search reads it (ops.SidPrefixIndex(...).levels(counts())), its numpy copy and each node's
    packed prefix key."""

    def __init__(self, corpus, K):
        from rq_vae_recommender_b200 import ops
        self.corpus, self.K, self.H = corpus, K, corpus.shape[1]
        self.index = ops.SidPrefixIndex(dev(corpus), K)
        self.levels = self.index.levels(self.index.counts().tolist())
        H = self.H
        self.n = list(self.levels.n)
        self.code = [None] + [host(self.levels.code[l]).astype(np.int64) for l in range(1, H + 1)]
        self.parent = [None] + [host(self.levels.parent[l]).astype(np.int64) for l in range(1, H + 1)]
        self.child = [host(c).astype(np.int64) for c in self.levels.child[:H]]
        self.key = [None, self.code[1]]
        for l in range(2, H + 1):
            self.key.append(self.key[l - 1][self.parent[l]] * K + self.code[l])
        self.leaf_key = dev(self.key[H])


@functools.lru_cache(maxsize=None)
def trie_of(K, H, N, seed=0, kind="subtrees"):
    rs = np.random.RandomState(seed)
    if kind == "subtrees":
        corpus = corpus_with_subtrees(rs, N, H, K)
    elif kind == "distinct":                                    # one column, N distinct codes
        corpus = rs.permutation(K)[:N, None].astype(np.int64)
    else:
        corpus = realistic_corpus(rs, N, H, K)
    return Trie(corpus, K)


@functools.lru_cache(maxsize=None)
def filters_of(K, H, N, B, M, seed=0, kind="subtrees"):
    """{mode: (the statement's valid(), the kernels' filter kwargs)} for B histories of trie_of's corpus: exclusion_sets /
    allow_lists (heavy sets, a subtree, an empty set), built by sid_exclusion_build / sid_inclusion_build and by the oracles."""
    corpus = trie_of(K, H, N, seed, kind).corpus
    rs = np.random.RandomState(seed + 1)
    ex_items = exclusion_sets(rs, corpus, B, M)
    _, ref, ex = excl_built(corpus, K, ex_items)
    in_items = allow_lists(rs, corpus, B, M)
    _, ref, inc, incls = incl_built(corpus, K, in_items)
    return {"none": (None, {}), "exclude": (EO.exclusion_valid(X.build(ref, ex_items)), {"exclude": ex}),
            "include": (EO.inclusion_valid(incls), {"include": inc})}


def test_trie_levels_match_trie_oracle():
    for K, H, N in ((300, 3, 3000), (2048, 5, 4000), (128, 8, 1500)):
        tr = trie_of(K, H, N)
        want = TO.build(tr.corpus, K)
        assert tr.n == want["n"]
        for l in range(1, H + 1):
            assert np.array_equal(tr.code[l], want["codes"][l]), (K, H, l)
            assert np.array_equal(tr.child[l - 1], want["child"][l - 1]), (K, H, l)
            assert np.array_equal(tr.parent[l], np.repeat(np.arange(tr.n[l - 1]), np.diff(want["child"][l - 1]))), (K, H, l)


# ---------------------------------------------------------------------------------------------------------------- frontier
def child_scores(rs, n, distinct=False):
    """fp32 [n]: distinct multiples of 1/8 with NaN and -inf among them, and unless ``distinct`` the shared value, +0.0 and
    -0.0 as well."""
    s = ((rs.permutation(n) - n // 2) * 0.125).astype(np.float32)
    r = rs.rand(n)
    s[r < 0.04] = np.nan
    s[(r >= 0.04) & (r < 0.07)] = -np.inf
    if not distinct:
        s[(r >= 0.07) & (r < 0.13)] = SHARED
        s[(r >= 0.13) & (r < 0.16)] = 0.0
        s[(r >= 0.16) & (r < 0.19)] = -0.0
    return s


def pick_tau(ch, plan, valid, K, l, b0):
    """tau fp32 [Bc] per plan entry: "-inf", "+inf", "shared", "mid" (the median allowed score) or k (the k-th best allowed
    score: exactly k rows kept when the history's scores are distinct)."""
    keys = EO.child_keys(ch, K)
    tau = np.zeros(len(plan), dtype=np.float32)
    for b, p in enumerate(plan):
        j = np.arange(ch["offsets"][b], ch["offsets"][b + 1])
        s = ch["scores"][j]
        ok = ~np.isnan(s)
        if valid is not None and len(j):
            ok &= valid(b0 + b, l, keys[j])
        v = np.sort(s[ok])[::-1]
        if p == "-inf":
            tau[b] = -np.inf
        elif p == "+inf":
            tau[b] = np.inf
        elif p == "shared":
            tau[b] = SHARED
        elif p == "mid":
            tau[b] = v[len(v) // 2] if len(v) else 0.0
        else:
            tau[b] = v[p - 1] if len(v) >= p else -np.inf
    return tau


def to_device(ch, n_root, with_key):
    from rq_vae_recommender_b200 import ops
    if n_root is not None:                                      # the root's children: history b's are b * n_root ..
        return ops.ExactChildren(dev(ch["scores"]), n_root)
    i32 = lambda a: dev(np.asarray(a, dtype=np.int32))
    return ops.ExactChildren(dev(ch["scores"]), 0, i32(ch["offsets"]), i32(ch["node"]), i32(ch["code"]), i32(ch["parent"]),
                             dev(np.asarray(ch["pkey"], dtype=np.int64)) if with_key else None)


def check_frontier(tr, ch, n_root, tau, l, b0, filt):
    """The count pass, the host scan and the write pass (as FusedT5Exact.run drives them) against EO.frontier, bit for bit;
    returns the statement's output."""
    from rq_vae_recommender_b200 import ops
    valid, kw = filt
    want = EO.frontier(ch, tau, tr.child[l], tr.code[l + 1], tr.K, l, valid, b0)
    Bc = len(tau)
    dch = to_device(ch, n_root, bool(kw))
    tau_d = dev(np.asarray(tau, dtype=np.float32))
    counts = ops.t5exact_frontier_count(dch, tr.levels.code[1], tau_d, tr.K, l, tr.levels.child[l], b0, **kw)
    assert_ints(counts, want["counts"], "counts")
    scan = torch.zeros((3, Bc + 1), dtype=torch.int32, device="cuda")
    scan[:, 1:] = counts.cumsum(1)
    totals = scan[:, -1].tolist()
    if totals[0] == 0:                                          # every frontier empty: FusedT5Exact.run stops before the write
        return want
    nxt =ops.t5exact_frontier_write(dch, tr.levels.code[1], tau_d, tr.K, l, tr.levels.child[l], tr.levels.code[l + 1], scan,
                                     totals, b0, **kw)
    assert_ints(nxt.code, want["code"], "row codes")
    assert_ints(nxt.parent, want["parent"], "row parents")
    assert_bits(nxt.score, want["score"], "row scores")
    if kw:
        assert_ints(nxt.key, want["key"], "row keys")
    assert_ints(nxt.tiles, want["tiles"], "tiles")
    assert_ints(nxt.child, want["child"], "child ranges")
    assert_ints(nxt.children.offsets, np.concatenate([[0], np.cumsum(want["counts"][1])]), "child offsets")
    assert_ints(nxt.children.node, want["nnode"], "next nodes")
    assert_ints(nxt.children.code, want["ncode"], "next codes")
    assert_ints(nxt.children.parent, want["npar"], "next parents")
    return want


PLAN = ["-inf", "shared", 63, 64, "mid", 65, 129, "+inf"]


def walk(tr, rs, b0, Bc, filt, stats):
    """From the root's children to level H - 1, each written level's children scored afresh."""
    H = tr.H
    first = np.stack([child_scores(rs, tr.n[1], distinct=(b0 + b) % 2 == 1) for b in range(Bc)])
    ch, n_root = EO.root_children(first, tr.code[1]), tr.n[1]
    for l in range(1, H):
        plan = [PLAN[(b0 + b + l) % len(PLAN)] for b in range(Bc)]
        tau = pick_tau(ch, plan, filt[0], tr.K, l, b0)
        want = check_frontier(tr, ch, n_root, tau, l, b0, filt)
        stats["filtered"] += int(want["filtered"].sum())
        stats["levels"] += 1
        if want["counts"][0].sum() == 0:
            break
        nxt = np.concatenate([child_scores(rs, int(c), distinct=(b0 + b) % 2 == 1) for b, c in enumerate(want["counts"][1])])
        ch, n_root = EO.next_children(want, nxt), None


WALK = {"k300_h3": (300, 3, 3000), "k300_h5": (300, 5, 3000), "k2048_h3": (2048, 3, 4000), "k2048_h5": (2048, 5, 4000),
        "k128_h8": (128, 8, 1500)}


@pytest.mark.parametrize("mode", FILTERS)
@pytest.mark.parametrize("shape", list(WALK))
def test_frontier_walk(shape, mode):
    K, H, N = WALK[shape]
    tr = trie_of(K, H, N)
    filt = filters_of(K, H, N, 10, 1024)[mode]
    rs = np.random.RandomState(K + H)
    stats = dict(filtered=0, levels=0)
    for b0, Bc in ((0, 7), (3, 7), (9, 1)):                     # the filter holds the whole batch of 10
        walk(tr, rs, b0, Bc, filt, stats)
    assert stats["levels"] >= 2 * (H - 1)                     # the walk reaches the last frontier level
    if mode != "none":
        assert stats["filtered"] > 0


@pytest.mark.parametrize("mode", FILTERS)
def test_frontier_wide_chunk(mode):
    K, H, N = 300, 3, 2000
    tr = trie_of(K, H, N, seed=1)
    filt = filters_of(K, H, N, 310, 512, seed=1)[mode]
    rs = np.random.RandomState(5)
    stats = dict(filtered=0, levels=0)
    for b0 in (0, 10):
        walk(tr, rs, b0, 300, filt, stats)
    assert stats["levels"] == 2 * (H - 1)
    if mode != "none":
        assert stats["filtered"] > 0


@pytest.mark.parametrize("mode", FILTERS)
def test_frontier_edges(mode):
    """Level 2 of a K = 2048 trie, chunk b0 = 4 of 16 histories: the children counts and tau of each history pick an edge."""
    K, H, N = 2048, 3, 20000
    tr = trie_of(K, H, N, seed=2)
    filt = filters_of(K, H, N, 16, 4096, seed=2)[mode]
    valid = filt[0]
    rs = np.random.RandomState(6)
    b0, l = 4, 2
    # (children, tau plan, distinct scores)
    cases = [(0, "-inf", False), (1, "-inf", False), (255, "-inf", False), (256, "-inf", False), (257, "-inf", False),
             (3000, "shared", False), (0, "-inf", False), (400, 63, True), (400, 64, True), (400, 65, True),
             (400, 129, True), (300, "+inf", False)]
    n2 = tr.n[2]
    nodes, par, pkey, scores = [], [], [], []
    for b, (c, _, distinct) in enumerate(cases):
        pool = np.arange(n2) if valid is None else np.flatnonzero(valid(b0 + b, 2, tr.key[2]))
        half = rs.choice(pool, min((c + 1) // 2, len(pool)), replace=False)
        rest = rs.choice(np.setdiff1d(np.arange(n2), half), c - len(half), replace=False)
        nd = np.sort(np.concatenate([half, rest]).astype(np.int64))
        rows, inv = np.unique(tr.parent[2][nd], return_inverse=True)   # the history's rows: its children's parents
        par.append(len(pkey) + inv)
        pkey.extend(tr.key[1][rows].tolist())
        nodes.append(nd)
        scores.append(child_scores(rs, c, distinct))
    nd = np.concatenate(nodes)
    ch = dict(scores=np.concatenate(scores), offsets=np.concatenate([[0], np.cumsum([c for c, _, _ in cases])]), node=nd,
              code=tr.code[2][nd], parent=np.concatenate(par), pkey=np.asarray(pkey, dtype=np.int64))
    tau = pick_tau(ch, [p for _, p, _ in cases], valid, K, l, b0)
    want = check_frontier(tr, ch, None, tau, l, b0, filt)
    kept = want["counts"][0]
    assert kept[7:11].tolist() == [63, 64, 65, 129]           # the tile table at 63 / 64 / 65 / 129 rows
    assert kept[0] == kept[6] == kept[-1] == 0 and kept[2:6].all()   # empty frontiers in the middle and at the end
    assert want["at_tau"][5] >= 2                              # several rows tie at tau
    assert np.isnan(ch["scores"]).any() and np.isneginf(want["score"]).any()   # NaN never kept, -inf kept under tau = -inf
    zeros = want["score"][want["score"] == 0].view(np.int32)
    assert (zeros == 0).any() and (zeros != 0).any()           # +0.0 and -0.0 kept with their bits
    if mode != "none":
        assert want["filtered"].sum() > 0                       # rows at or above tau that the filter alone dropped
    tau_all = np.full(len(cases), np.inf, dtype=np.float32)     # nothing kept anywhere: the closing range entry alone
    want = check_frontier(tr, ch, None, tau_all, l, b0, filt)
    assert want["counts"].sum() == 0


# ---------------------------------------------------------------------------------------------------------------- select
def select_scores(rs, U, kind):
    if kind == "equal":
        return np.full(U, np.float32(-2.5))
    if kind == "nan":                                           # NaN but for a few: fewer valid candidates than w
        s = np.full(U, np.nan, dtype=np.float32)
        s[rs.choice(U, min(U, 100), replace=False)] = rs.randn(min(U, 100)).astype(np.float32)
        return s
    return child_scores(rs, U)


def run_select(tr, counts, kinds, w, b0, filt, rs):
    """One t5exact_select launch over leaf candidates (sorted random leaves) of len(counts) histories, against EO.select."""
    from rq_vae_recommender_b200 import ops
    valid, kw = filt
    H = tr.H
    nodes = [np.sort(rs.choice(tr.n[H], U, replace=False)) for U in counts]
    ch = dict(scores=np.concatenate([select_scores(rs, U, k) for U, k in zip(counts, kinds)]),
              offsets=np.concatenate([[0], np.cumsum(counts)]), node=np.concatenate(nodes).astype(np.int64))
    want = EO.select(ch, w, tr.code, tr.parent, tr.key[H], valid, b0)
    Bc, max_u = len(counts), max(counts)                        # always the true largest count
    gen = torch.full((Bc, w, H), -7, dtype=torch.int64, device="cuda")
    lp = torch.full((Bc, w), 7.0, dtype=torch.float32, device="cuda")
    i32 = lambda a: dev(np.asarray(a, dtype=np.int32))
    dch = ops.ExactChildren(dev(ch["scores"]), 0, i32(ch["offsets"]), i32(ch["node"]))
    ops.t5exact_select(dch, max_u, tr.levels, H, tr.leaf_key, w, gen, lp, b0, **kw)
    assert_ints(gen, want[0], "tuples")
    assert_bits(lp, want[1], "scores")
    n_valid, n_blocked = [], 0                                  # per history: candidates neither NaN nor blocked
    for b in range(Bc):
        j = np.arange(ch["offsets"][b], ch["offsets"][b + 1])
        ok = ~np.isnan(ch["scores"][j])
        if valid is not None and len(j):
            allowed = valid(b0 + b, H, tr.key[H][ch["node"][j]])
            n_blocked += int((ok & ~allowed).sum())
            ok &= allowed
        n_valid.append(int(ok.sum()))
    return want, n_valid, n_blocked


@pytest.mark.parametrize("w", [1, 10, 1024])
@pytest.mark.parametrize("mode", FILTERS)
def test_select(mode, w):
    K, H, N = 256, 3, 66000
    tr = trie_of(K, H, N, kind="realistic")
    assert tr.n[H] > 60000
    filt = filters_of(K, H, N, 16, 1500, kind="realistic")[mode]
    rs = np.random.RandomState(w)
    small = [0, 1, max(w - 1, 0), w, w + 1, SMEM_KEYS, SMEM_KEYS, 3000]
    large = [SMEM_KEYS + 1, 60000, 0, 1, w, SMEM_KEYS + 1, 30000, 40000]
    for b0, counts, kinds in ((0, small, ["random"] * 6 + ["equal", "random"]),
                              (8, large, ["random"] * 5 + ["equal", "nan", "random"])):
        assert (max(counts) <= SMEM_KEYS) == (b0 == 0)         # chunk 0 keeps its keys in shared memory, chunk 8 recomputes
        (gen, lp), n_valid, n_blocked = run_select(tr, counts, kinds, w, b0, filt, rs)
        b = kinds.index("equal")                                # all equal: the tie at the w-th score spans 512-thread rounds
        assert (lp[b] == np.float32(-2.5)).sum() == min(w, n_valid[b])
        if mode == "none":
            assert n_valid[b] > w                               # equal candidates left out at the w-th score
        else:
            assert n_blocked > 0                                # candidates the filter alone left out
        if w == 1024:                                           # fewer valid candidates than w: padded
            assert any(0 < n_valid[i] < w and counts[i] > SMEM_KEYS for i in range(len(counts))) or b0 == 0
            assert all((gen[i, n_valid[i]:] == -1).all() for i in range(len(counts)) if n_valid[i] < w)


@pytest.mark.parametrize("mode", FILTERS)
def test_select_root(mode):
    """The root's children as candidates (ch.node None: history b's are b * n_root ..), one-column corpora of 1 500 and 30 000
    codes, on both sides of the shared-memory bound."""
    from rq_vae_recommender_b200 import ops
    for K, N in ((2048, 1500), (40000, 30000)):
        tr = trie_of(K, 1, N, kind="distinct")
        n1 = tr.n[1]
        assert n1 == N and (n1 > SMEM_KEYS) == (N == 30000)
        valid, kw = filters_of(K, 1, N, 6, 2048, kind="distinct")[mode]
        rs = np.random.RandomState(N)
        Bc, b0 = 4, 2
        first = np.stack([select_scores(rs, n1, k) for k in ("random", "equal", "nan", "random")])
        ch = EO.root_children(first, tr.code[1])
        for w in (1, 10, 1024):
            want = EO.select(ch, w, tr.code, tr.parent, tr.key[1], valid, b0)
            gen = torch.full((Bc, w, 1), -7, dtype=torch.int64, device="cuda")
            lp = torch.full((Bc, w), 7.0, dtype=torch.float32, device="cuda")
            ops.t5exact_select(ops.ExactChildren(dev(first.reshape(-1)), n1), n1, tr.levels, 1, tr.leaf_key, w, gen, lp, b0,
                               **kw)
            assert_ints(gen, want[0], (K, w))
            assert_bits(lp, want[1], (K, w))


def test_argument_errors():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200._lib import Rqb200Error
    tr = trie_of(300, 3, 3000)
    Bc = 2
    scores = torch.zeros(Bc * tr.n[1], device="cuda")
    root = ops.ExactChildren(scores, tr.n[1])
    gen = torch.empty((Bc, 1025, 3), dtype=torch.int64, device="cuda")
    lp = torch.empty((Bc, 1025), dtype=torch.float32, device="cuda")
    offsets = dev(np.array([0, 3, 6], dtype=np.int32))
    ch = ops.ExactChildren(torch.zeros(6, device="cuda"), 0, offsets, *(dev(np.zeros(6, dtype=np.int32)) for _ in range(3)))
    with pytest.raises(Rqb200Error, match="w <= 1024"):
        ops.t5exact_select(ch, 3, tr.levels, 3, tr.leaf_key, 1025, gen, lp)
    tau = torch.zeros(Bc, device="cuda")
    with pytest.raises(ValueError, match="root_code"):
        ops.t5exact_frontier_count(root, None, tau, 300, 1, tr.levels.child[1])
    counts = ops.t5exact_frontier_count(root, tr.levels.code[1], tau, 300, 1, tr.levels.child[1])
    for bad in (torch.zeros((3, Bc), dtype=torch.int32, device="cuda"), torch.zeros((3, Bc + 1), device="cuda"),
                torch.zeros((Bc + 1, 3), dtype=torch.int32, device="cuda").t()):
        with pytest.raises(ValueError, match="offsets"):
            ops.t5exact_frontier_write(root, tr.levels.code[1], tau, 300, 1, tr.levels.child[1], tr.levels.code[2], bad,
                                       (0, 0, 0))
    assert counts.shape == (3, Bc)


# ---------------------------------------------------------------------------------------------------------------- model
def fat_corpus(rs, K, H, prefixes, leaves):
    """``prefixes`` distinct (H - 1)-prefixes, each with ``leaves`` distinct last codes (one item per tuple), rows shuffled."""
    keys = rs.choice(K ** (H - 1), prefixes, replace=False)
    pre = np.stack([(keys // K ** (H - 2 - h)) % K for h in range(H - 1)], 1)
    rows = [np.concatenate([np.repeat(p[None], leaves, 0), rs.choice(K, leaves, replace=False)[:, None]], 1) for p in pre]
    corpus = np.concatenate(rows).astype(np.int64)
    return corpus[rs.permutation(len(corpus))]


def valid_leaves(m, corpus, K, H, mode, items, B):
    """bool [B, U]: each leaf's validity for each history under the call's filter (the oracles), None without one."""
    if mode == "none":
        return None
    leaf_key = host(m._rank_levels(torch.device("cuda"))[1])
    ref = IO.build(corpus, K)
    assert np.array_equal(X.leaf_keys(ref), leaf_key)
    if mode == "exclude":
        lists = [e["blocked"][H] for e in X.build(ref, items)]
        return torch.from_numpy(np.stack([~np.isin(leaf_key, v) for v in lists])).cuda()
    lists = [e["keys"][H] for e in I.build(ref, items)]
    return torch.from_numpy(np.stack([np.isin(leaf_key, v) for v in lists])).cuda()


def record_select(monkeypatch):
    """ops.t5exact_select wrapped: each launch's max_u, b0 and filter."""
    from rq_vae_recommender_b200 import ops
    orig, seen = ops.t5exact_select, []

    def wrapped(ch, max_u, levels, H, leaf_key, w, out_gen, out_lp, b0=0, **kw):
        seen.append((max_u, b0, tuple(kw)))
        return orig(ch, max_u, levels, H, leaf_key, w, out_gen, out_lp, b0, **kw)

    monkeypatch.setattr(ops, "t5exact_select", wrapped)
    return seen


FAT = {"k2048_h2": (2048, 2, 20, 2000), "k256_h3": (256, 3, 120, 250)}


@pytest.mark.parametrize("mode", FILTERS)
@pytest.mark.parametrize("shape", list(FAT))
def test_model_many_leaf_candidates(shape, mode, monkeypatch):
    """Random init (nothing pruned: a prefix scores far above any leaf), so each history's candidates are all the leaves."""
    from rq_vae_recommender_b200.modules import model as M
    K, H, P, L = FAT[shape]
    B = 3
    rs = np.random.RandomState(K + H)
    corpus = fat_corpus(rs, K, H, P, L)
    m = model_for(M, corpus, K, H)
    mask, ids, users = history(rs, B, 6, H, K)
    prefix_rows = [np.flatnonzero((corpus[:, :H - 1] == p).all(1)) for p in np.unique(corpus[:, :H - 1], axis=0)]
    kwargs, items = {}, None
    if mode == "exclude":
        items = np.full((B, 2 * L), -1, dtype=np.int64)
        items[0, :L] = prefix_rows[0]                            # a whole fat prefix
        items[1, :300] = rs.choice(len(corpus), 300, replace=False)
        kwargs = dict(exclude_items=torch.from_numpy(items).cuda())
    elif mode == "include":                                      # one item under each fat prefix: every prefix survives
        items = np.stack([[rs.choice(r) for r in prefix_rows] for _ in range(B)]).astype(np.int64)
        kwargs = dict(include_items=torch.from_numpy(items).cuda())
    dense = m.rank_sem_ids(mask, ids, users)
    tuples = leaf_tuples(m, H, K)
    valid = valid_leaves(m, corpus, K, H, mode, items, B)
    seen = record_select(monkeypatch)
    for w in (w for w in (1, 100, 256, 1024) if w <= K):
        got = m.generate(mask, ids, users, search="exact", num_beams=w, **kwargs)
        want = dense_topw(dense, tuples, w, valid)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), w
        if mode == "include" and w >= 256:
            assert (got[0][:, -1] == -1).all()                   # fewer valid leaves than w
    assert seen and all(max_u > SMEM_KEYS for max_u, _, _ in seen)   # the recompute path
    assert all(kw == (() if mode == "none" else (mode,)) for _, _, kw in seen)


def record_runs(monkeypatch, M):
    run, runs = M.FusedT5Exact.run, []

    def counted(self, b0, b1, *a, **kw):
        out = run(self, b0, b1, *a, **kw)
        runs.append((b0, b1, out is None))
        return out

    monkeypatch.setattr(M.FusedT5Exact, "run", counted)
    return runs


def test_model_chunk_reruns_with_filters(monkeypatch):
    """A one-level row budget forces reruns and chunks with b0 > 0; with each filter the result is the unchunked call's bits."""
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, w = 256, 3, 9, 32
    rs = np.random.RandomState(21)
    corpus = corpus_with_subtrees(rs, 2000, H, K)
    m = model_for(M, corpus, K, H)
    mask, ids, users = history(rs, B, 8, H, K)
    ex_items = exclusion_sets(rs, corpus, B, 600)
    in_items = allow_lists(rs, corpus, B, 1500)
    calls = {"exclude": dict(exclude_items=torch.from_numpy(ex_items).cuda()),
             "include": dict(include_items=torch.from_numpy(in_items).cuda())}
    dense = m.rank_sem_ids(mask, ids, users)
    tuples = leaf_tuples(m, H, K)
    batch = batch_for(rs, corpus, B, 6, H, K)
    ref = {mode: m.generate(mask, ids, users, search="exact", num_beams=w, **kw) for mode, kw in calls.items()}
    ref_hist = m.generate_next_sem_id(batch, search="exact", num_beams=w, exclude_history=True)
    levels = m._rank_levels(dense.device)[0]
    monkeypatch.setattr(M, "RANK_BYTE_BUDGET", max(levels.n[:H]) * M.FusedT5Rank.row_bytes(m))
    runs = record_runs(monkeypatch, M)
    for mode, kw in calls.items():
        runs.clear()
        got = m.generate(mask, ids, users, search="exact", num_beams=w, **kw)
        assert any(r for _, _, r in runs) and any(b0 > 0 and not r for b0, _, r in runs), runs
        assert torch.equal(got[0], ref[mode][0]) and torch.equal(got[1], ref[mode][1]), mode
        items = ex_items if mode == "exclude" else in_items
        want = dense_topw(dense, tuples, w, valid_leaves(m, corpus, K, H, mode, items, B))
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), mode
    runs.clear()
    got = m.generate_next_sem_id(batch, search="exact", num_beams=w, exclude_history=True)
    assert any(r for _, _, r in runs) and any(b0 > 0 and not r for b0, _, r in runs), runs
    assert torch.equal(got.sem_ids, ref_hist.sem_ids) and torch.equal(got.log_probas, ref_hist.log_probas)


def record_frontier(monkeypatch, levels):
    """ops.t5exact_frontier_count / _write wrapped: each level's children, tau, level and b0 (numpy, the statement's form)."""
    from rq_vae_recommender_b200 import ops
    count, write, seen = ops.t5exact_frontier_count, ops.t5exact_frontier_write, []

    def counted(ch, root_code, tau, K, l, lchild, b0=0, **kw):
        Bc = tau.shape[0]
        if ch.node is None:
            c = EO.root_children(host(ch.scores).reshape(Bc, ch.n_root), host(root_code))
        else:
            c = dict(scores=host(ch.scores), offsets=host(ch.offsets), node=host(ch.node), code=host(ch.code),
                     parent=host(ch.parent), pkey=None if ch.key is None else host(ch.key))
        seen.append(dict(ch=c, tau=host(tau), l=l, b0=b0, kw=kw))
        return count(ch, root_code, tau, K, l, lchild, b0, **kw)

    def written(ch, root_code, tau, K, l, lchild, lcode_next, offsets, totals, b0=0, **kw):
        nxt = write(ch, root_code, tau, K, l, lchild, lcode_next, offsets, totals, b0, **kw)
        seen[-1]["next"] = nxt
        return nxt

    monkeypatch.setattr(ops, "t5exact_frontier_count", counted)
    monkeypatch.setattr(ops, "t5exact_frontier_write", written)
    return seen


def tie_corpus(rs, K):
    """Level-2 nodes holding every last code, so that the most probable leaf under them exists (its log-probability can be
    exactly 0.0 and the node ties it), and one first code holding every second code."""
    rows = []
    for a in rs.choice(K, 4, replace=False):
        for c in rs.choice(K, 16, replace=False):
            rows.append(np.stack([np.full(K, a), np.full(K, c), np.arange(K)], 1))
    a = rows[0][0, 0]
    rows.append(np.stack([np.full(K, a), np.arange(K), rs.randint(0, K, K)], 1))
    return np.unique(np.concatenate(rows), axis=0)


def test_model_frontier_ties_at_tau(monkeypatch):
    """Sharpened heads until some log-probabilities are exactly 0.0: each level's frontier, recorded under the model, equals
    the statement; some kept node scores exactly tau; the result is the dense top w; the decoder rows are Bc plus the kept rows."""
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 6
    rs = np.random.RandomState(22)
    corpus = tie_corpus(rs, K)
    mask, ids, users = history(rs, B, 8, H, K)
    ties, checked = 0, 0
    for scale in (32, 128, 512):
        m = sharpen(model_for(M, corpus, K, H), scale)
        levels = m._rank_levels(torch.device("cuda"))[0]
        child = [host(c).astype(np.int64) for c in levels.child[:H]]
        code = [None] + [host(c).astype(np.int64) for c in levels.code[1:]]
        dense = m.rank_sem_ids(mask, ids, users)
        tuples = leaf_tuples(m, H, K)
        for w in (1, 2, 5, 10, 32):
            seen = record_frontier(monkeypatch, levels)
            got = m.generate(mask, ids, users, search="exact", num_beams=w)
            monkeypatch.undo()
            want = dense_topw(dense, tuples, w)
            assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), (scale, w)
            rows = 0
            for s in seen:
                assert s["b0"] == 0 and not s["kw"]
                out = EO.frontier(s["ch"], s["tau"], child[s["l"]], code[s["l"] + 1], K, s["l"])
                if "next" in s:                                  # a level with kept rows: its written layout
                    nxt = s["next"]
                    assert_ints(nxt.code, out["code"], "row codes")
                    assert_ints(nxt.parent, out["parent"], "row parents")
                    assert_bits(nxt.score, out["score"], "row scores")
                    assert_ints(nxt.tiles, out["tiles"], "tiles")
                    assert_ints(nxt.child, out["child"], "child ranges")
                    assert_ints(nxt.children.node, out["nnode"], "next nodes")
                    assert_ints(nxt.children.parent, out["npar"], "next parents")
                else:
                    assert out["counts"][0].sum() == 0
                rows += len(out["code"])
                ties += int(out["at_tau"][np.isfinite(s["tau"])].sum())
                checked += 1
            assert M.EXACT_DECODER_ROWS == B + rows, (scale, w)
        if ties:
            break
    assert checked >= 2 and ties > 0
