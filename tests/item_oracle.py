"""Numpy restatement of the corpus item table (csrc/sid.cu: rqb200_sid_items_build, _lookup, _retrieve) and of the rank rule of
rqb200_sid_topk_rank_hist.  Row n of the corpus table [N, C] is item n; a row holding an id outside [0, K) is never retrievable.
The build orders the retrievable rows by tuple, equal tuples by ascending row (a stable sort); row[start[u] .. start[u + 1]) are
the rows of the u-th distinct tuple, keys[u]."""
import numpy as np


def build(corpus_ids, K):
    corpus = np.asarray(corpus_ids, dtype=np.int64)
    N, C = corpus.shape
    ok = ((corpus >= 0) & (corpus < K)).all(axis=1) if N else np.zeros(0, dtype=bool)
    enc = np.where(ok[:, None], corpus, K)                                  # unretrievable rows sort last
    order = np.lexsort(enc.T[::-1]) if N else np.zeros(0, dtype=np.int64)   # np.lexsort is stable
    valid = order[ok[order]]
    vals = corpus[valid]
    new = np.ones(len(valid), dtype=bool)
    if len(valid) > 1:
        new[1:] = (vals[1:] != vals[:-1]).any(axis=1)
    start = np.append(np.flatnonzero(new), len(valid))
    return dict(C=C, K=K, row=order, keys=vals[new], start=start)


def _find(table, t):
    """Position of tuple t among the table's distinct tuples, or -1."""
    if "index" not in table:
        table["index"] = {tuple(int(v) for v in key): u for u, key in enumerate(table["keys"])}
    t = tuple(int(v) for v in t)
    return table["index"].get(t, -1) if len(t) == table["C"] else -1


def items_of(table, t):
    """The items of tuple t in dedup-rank order (empty when it is not in the corpus)."""
    u = _find(table, t)
    return [] if u < 0 else [int(r) for r in table["row"][table["start"][u]:table["start"][u + 1]]]


def lookup(table, ids, with_dedup=False):
    ids = np.asarray(ids, dtype=np.int64)
    C = table["C"]
    out = np.full(ids.shape[0], -1, dtype=np.int64)
    for p, t in enumerate(ids):
        items = items_of(table, t[:C])
        d = int(t[C]) if with_dedup else 0
        if 0 <= d < len(items):
            out[p] = items[d]
    return out


def retrieve(table, generated, log_probas, n):
    generated = np.asarray(generated, dtype=np.int64)
    B, k, _ = generated.shape
    items = np.full((B, n), -1, dtype=np.int64)
    beam = np.full((B, n), -1, dtype=np.int32)
    count = np.zeros(B, dtype=np.int32)
    for b in range(B):
        got, seen = [], set()
        for j in range(k):
            if log_probas is not None and not log_probas[b, j] > -np.inf:
                continue
            for it in items_of(table, generated[b, j]):
                if it not in seen:
                    seen.add(it)
                    got.append((it, j))
        got = got[:n]
        count[b] = len(got)
        for o, (it, j) in enumerate(got):
            items[b, o], beam[b, o] = it, j
    return items, beam, count


def rank_hist(actual, candidates, item_mode=False):
    """int64 [k + 1]: hist[r] rows whose first candidate equal to actual in all D columns is r, hist[k] rows with none."""
    actual = np.asarray(actual, dtype=np.int64)
    candidates = np.asarray(candidates, dtype=np.int64)
    B, k, D = candidates.shape
    match = (candidates == actual[:, None, :]).all(axis=-1)
    if item_mode:
        match &= (actual != -1).all(axis=-1)[:, None]
    rank = np.where(match.any(axis=1), match.argmax(axis=1), k)
    return np.bincount(rank, minlength=k + 1).astype(np.int64)
