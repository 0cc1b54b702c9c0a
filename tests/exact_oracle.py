"""Numpy statement of the exact top-k search's two kernel families (csrc/t5rank.cu t5exact_frontier_kernel and
t5exact_select_kernel, behind ops.t5exact_frontier_count / _write and ops.t5exact_select), in float64 and int64: no torch, no GPU.

Children of one decoder level, for a chunk of Bc histories whose first is history b0 of the batch, are flat arrays ("ch"):
scores fp32 [C]; offsets int [Bc + 1] (history b's children are offsets[b] .. offsets[b + 1] - 1); node / code / parent int [C]
(node id in trie level l, its last code, its parent row in the level above); pkey int64 [rows] (each parent row's prefix key; None
at level 1, where a child's key is its code).  ``root_children`` gives the root's children in that form.

A filter is a predicate valid(b_global, l, keys) -> bool array: is each packed l-prefix key (level 0 most significant, K-ary) valid
for history b_global of the batch.  ``exclusion_valid`` / ``inclusion_valid`` state it for tests/exclusion_oracle.py's and
tests/inclusion_oracle.py's builds: an exclusion blocks its listed prefixes, an allow-list admits only its listed ones."""
import numpy as np

QTILE = 64                                                   # query rows per cross-attention tile (RK_QTILE)


def root_children(first, code1):
    """The root's children (level 1) of a chunk: first fp32 [Bc, n1] (history b's score of each level-1 node) and code1 [n1]."""
    Bc, n1 = first.shape
    return dict(scores=np.asarray(first, dtype=np.float32).reshape(-1), offsets=np.arange(Bc + 1, dtype=np.int64) * n1,
                node=np.tile(np.arange(n1, dtype=np.int64), Bc), code=np.tile(np.asarray(code1, dtype=np.int64), Bc),
                parent=np.repeat(np.arange(Bc, dtype=np.int64), n1), pkey=None)


def exclusion_valid(excls):
    """valid() of exclusion_oracle.build's histories: an l-prefix is valid unless it is among the history's blocked ones."""
    lists = [{l: np.asarray(v, dtype=np.int64) for l, v in e["blocked"].items()} for e in excls]
    return lambda bg, l, keys: ~np.isin(keys, lists[bg][l])


def inclusion_valid(incls):
    """valid() of inclusion_oracle.build's histories: an l-prefix is valid when it is among the history's valid ones."""
    lists = [{l: np.asarray(v, dtype=np.int64) for l, v in e["keys"].items()} for e in incls]
    return lambda bg, l, keys: np.isin(keys, lists[bg][l])


def child_keys(ch, K):
    """int64 [C]: each child's prefix key, pkey[parent] * K + code (its code at level 1)."""
    code = np.asarray(ch["code"], dtype=np.int64)
    if ch["pkey"] is None:
        return code
    return np.asarray(ch["pkey"], dtype=np.int64)[np.asarray(ch["parent"], dtype=np.int64)] * K + code


def frontier(ch, tau, child_l, code_next, K, l, valid=None, b0=0):
    """One level of the frontier, count and write passes together.  A child is kept when score >= tau[b] (NaN never is) and
    the filter allows its key.  child_l: the trie's child ranges of level l ([n_l + 1]); code_next: its codes of level l + 1.
    Returns a dict:
      counts int64 [3, Bc]   kept rows, their children, their 64-row tiles, per history;
      code, parent, score, key, node [R]   the next level's rows in trie order, history by history (score fp32, as given);
      tiles int64 [T, 3]     (b, first row, min(64, rest)) per history, in order;
      child int64 [R + 1]    each row's first child in the next children, global across the chunk, last entry C;
      nnode, ncode, npar [C] the next children: node (level l + 1), code, parent row;
      at_tau [Bc]            kept rows that score exactly tau[b];  filtered [Bc]  rows score >= tau[b] that the filter dropped."""
    scores = np.asarray(ch["scores"], dtype=np.float32)
    offsets = np.asarray(ch["offsets"], dtype=np.int64)
    node = np.asarray(ch["node"], dtype=np.int64)
    child_l = np.asarray(child_l, dtype=np.int64)
    keys = child_keys(ch, K)
    tau = np.asarray(tau, dtype=np.float32).astype(np.float64)
    Bc = len(offsets) - 1
    counts = np.zeros((3, Bc), dtype=np.int64)
    at_tau = np.zeros(Bc, dtype=np.int64)
    filtered = np.zeros(Bc, dtype=np.int64)
    kept = []
    for b in range(Bc):
        j = np.arange(offsets[b], offsets[b + 1])
        s = scores[j].astype(np.float64)
        with np.errstate(invalid="ignore"):
            keep = s >= tau[b]
        if valid is not None and len(j):
            ok = np.asarray(valid(b0 + b, l, keys[j]), dtype=bool)
            filtered[b] = int((keep & ~ok).sum())
            keep &= ok
        j = j[keep]
        kept.append(j)
        at_tau[b] = int((scores[j].astype(np.float64) == tau[b]).sum())
        counts[0, b] = len(j)
        counts[1, b] = int((child_l[node[j] + 1] - child_l[node[j]]).sum())
        counts[2, b] = -(-len(j) // QTILE)
    rows = np.concatenate(kept) if kept else np.zeros(0, dtype=np.int64)
    nch = child_l[node[rows] + 1] - child_l[node[rows]]
    child = np.concatenate([[0], np.cumsum(nch)]).astype(np.int64)
    tiles, roff = [], 0
    for b in range(Bc):
        for t0 in range(0, int(counts[0, b]), QTILE):
            tiles.append((b, roff + t0, min(QTILE, int(counts[0, b]) - t0)))
        roff += int(counts[0, b])
    nnode = np.concatenate([np.arange(child_l[n], child_l[n + 1]) for n in node[rows]] or [np.zeros(0)]).astype(np.int64)
    npar = np.repeat(np.arange(len(rows), dtype=np.int64), nch)
    ncode = np.asarray(code_next, dtype=np.int64)[nnode] if code_next is not None else np.zeros(0, dtype=np.int64)
    return dict(counts=counts, code=np.asarray(ch["code"], dtype=np.int64)[rows],
                parent=np.asarray(ch["parent"], dtype=np.int64)[rows], score=scores[rows], key=keys[rows], node=node[rows],
                tiles=np.asarray(tiles, dtype=np.int64).reshape(-1, 3), child=child, nnode=nnode, ncode=ncode, npar=npar,
                at_tau=at_tau, filtered=filtered)


def next_children(out, scores):
    """The next level's children (``ch``) of a frontier() output, with their scores fp32 [C]."""
    return dict(scores=np.asarray(scores, dtype=np.float32),
                offsets=np.concatenate([[0], np.cumsum(out["counts"][1])]).astype(np.int64),
                node=out["nnode"], code=out["ncode"], parent=out["npar"], pkey=out["key"])


def select(ch, w, codes, parents, leaf_key=None, valid=None, b0=0):
    """Each history's w best leaf candidates: score descending (-0.0 equal to +0.0), then candidate index ascending; NaN and
    leaves the filter blocks (valid(b0 + b, H, leaf_key[node])) left out, -inf kept.  codes / parents: the trie's levels
    1..H (index 0 unused), H = len(codes) - 1.  Returns (gen int64 [Bc, w, H], each leaf's tuple along its path, -1 past the
    valid candidates; lp fp32 [Bc, w], each leaf's score, -inf past them)."""
    scores = np.asarray(ch["scores"], dtype=np.float32)
    offsets = np.asarray(ch["offsets"], dtype=np.int64)
    node = np.asarray(ch["node"], dtype=np.int64)
    H = len(codes) - 1
    Bc = len(offsets) - 1
    gen = np.full((Bc, w, H), -1, dtype=np.int64)
    lp = np.full((Bc, w), -np.inf, dtype=np.float32)
    for b in range(Bc):
        s = scores[offsets[b]:offsets[b + 1]]
        nd = node[offsets[b]:offsets[b + 1]]
        ok = ~np.isnan(s)
        if valid is not None and len(s):
            ok &= np.asarray(valid(b0 + b, H, np.asarray(leaf_key, dtype=np.int64)[nd]), dtype=bool)
        u = np.flatnonzero(ok)
        order = u[np.lexsort((u, -s[u].astype(np.float64)))][:w]
        lp[b, :len(order)] = s[order]
        n = nd[order]
        for lv in range(H, 0, -1):
            gen[b, :len(order), lv - 1] = np.asarray(codes[lv], dtype=np.int64)[n]
            n = np.asarray(parents[lv], dtype=np.int64)[n]
    return gen, lp
