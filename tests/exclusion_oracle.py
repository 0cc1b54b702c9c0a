"""Numpy statement of the per-history exclusion sets (csrc/sid.cu rqb200_sid_exclusion_build and its four consumers), on the
item table of tests/item_oracle.py.

An exclusion set is a list of corpus rows (-1 pads, repeats allowed).  Rows outside [-1, N) are counted and otherwise ignored;
rows that are not retrievable are ignored.  A trie prefix is blocked when at least one excluded item lies under it and every
retrievable item under it is excluded.  The searches treat an extension to a blocked prefix as one the corpus lacks; the item
retrieval and the exact ranking's selection skip excluded items."""
import numpy as np

import beam_search_oracle as BS


def tuple_key(t, K):
    """The K-ary packed key of a tuple (level 0 most significant): modules/model.py's _tuple_key."""
    key = 0
    for v in t:
        key = key * K + int(v)
    return key


def leaf_keys(table):
    """int64 [U]: the packed keys of the table's distinct retrievable tuples, ascending (the order of table["keys"])."""
    return np.array([tuple_key(t, table["K"]) for t in table["keys"]], dtype=np.int64)


def build(table, items):
    """items [B, M] -> one dict per history: excluded (the set of excluded retrievable rows), pos (their positions in
    table["row"], ascending), blocked ({l: sorted keys of the blocked l-prefixes}, l = 1..H) and bad (entries outside [-1, N))."""
    items = np.asarray(items, dtype=np.int64)
    row, start, H, K = table["row"], table["start"], table["C"], table["K"]
    N = len(row)
    n_items = int(start[-1])
    inv = np.empty(N, dtype=np.int64)
    inv[row] = np.arange(N)
    retrievable = set(int(r) for r in row[:n_items])
    tuples = {}                                                    # retrievable row -> its tuple
    for u, key in enumerate(table["keys"]):
        for r in row[start[u]:start[u + 1]]:
            tuples[int(r)] = tuple(int(v) for v in key)
    out = []
    for hist in items:
        bad = int(((hist < -1) | (hist >= N)).sum())
        excluded = set(int(i) for i in hist if 0 <= i < N and int(i) in retrievable)
        blocked = {}
        for l in range(1, H + 1):
            under = {}
            for r, t in tuples.items():
                under.setdefault(t[:l], set()).add(r)
            blocked[l] = sorted(tuple_key(p, K) for p, rows in under.items() if rows & excluded and rows <= excluded)
        out.append(dict(excluded=excluded, pos=sorted(int(inv[i]) for i in excluded), blocked=blocked, bad=bad))
    return out


def is_blocked(excl, prefix, K):
    """Is the l-prefix `prefix` blocked for the history of excl (one entry of build())?"""
    return tuple_key(prefix, K) in set(excl["blocked"].get(len(prefix), []))


def valid_prefix(corpus_ids, K, excl, prefix):
    """The searches' validity of an id prefix for one history: a corpus prefix (beam_search_oracle's check) that is not
    blocked."""
    corpus_ok = bool(BS.O.check_valid_prefix(np.asarray(corpus_ids), np.asarray(prefix, dtype=np.int64)[None])[0])
    in_range = all(0 <= int(v) < K for v in prefix)
    return corpus_ok and not (in_range and is_blocked(excl, prefix, K))


def candidate_scores(corpus_ids, K, excls, logits, generated, log_probas):
    """[B, kp * K] float64: beam_search_oracle.candidate_scores with the extensions to a blocked prefix at -inf as well."""
    scores = BS.candidate_scores(corpus_ids, logits, generated, log_probas)
    B = scores.shape[0]
    for b in range(B):
        for e in range(scores.shape[1]):
            beam, c = divmod(e, K)
            prefix = ([] if generated is None else [int(v) for v in generated[b, beam]]) + [c]
            if scores[b, e] > -np.inf and is_blocked(excls[b], prefix, K):
                scores[b, e] = -np.inf
    return scores


def retrieve(table, excls, generated, log_probas, n):
    """item_oracle.retrieve with each history's excluded items skipped."""
    from item_oracle import items_of
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
            t = tuple(int(v) for v in generated[b, j])
            if t in seen:                                          # a tuple an earlier beam carries
                continue
            seen.add(t)
            got += [(it, j) for it in items_of(table, t) if it not in excls[b]["excluded"]]
        got = got[:n]
        count[b] = len(got)
        for o, (it, j) in enumerate(got):
            items[b, o], beam[b, o] = it, j
    return items, beam, count


def rank_select(table, excls, scores, t_leaf, t_dedup, n):
    """The exact ranking's selection with exclusions: per history every item that is not excluded, leaves by score descending
    (NaN last), then leaf, then dedup rank; the first n (items -1 / scores -inf pad) and the target's position among them all
    (-1 when the target leaf or dedup rank is out of range, or the target is excluded)."""
    scores = np.asarray(scores, dtype=np.float32)
    row, start = table["row"], table["start"]
    B, U = scores.shape
    items = np.full((B, n), -1, dtype=np.int64)
    item_scores = np.full((B, n), -np.inf, dtype=np.float32)
    rank = np.full(B, -1, dtype=np.int64)
    for b in range(B):
        s = scores[b]
        order = sorted(range(U), key=lambda u: (np.isnan(s[u]), -s[u] if not np.isnan(s[u]) else 0.0, u))
        ranked = [(int(r), u) for u in order for r in row[start[u]:start[u + 1]] if int(r) not in excls[b]["excluded"]]
        for o, (it, u) in enumerate(ranked[:n]):
            items[b, o], item_scores[b, o] = it, s[u]
        tl, td = int(t_leaf[b]), int(t_dedup[b])
        if 0 <= tl < U and 0 <= td < start[tl + 1] - start[tl]:
            target = int(row[start[tl] + td])
            pos = [it for it, _ in ranked]
            rank[b] = pos.index(target) if target in pos else -1
    return items, item_scores, rank
