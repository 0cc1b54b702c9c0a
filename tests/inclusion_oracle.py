"""Numpy statement of the per-history allow-lists (csrc/sid.cu rqb200_sid_inclusion_build and its three consumers), on the item
table of tests/item_oracle.py.

An allow-list is a list of corpus rows (-1 pads, repeats allowed).  Rows outside [-1, N) are counted and otherwise ignored.  An
item is eligible for the history when it is in the allow-list, retrievable and not excluded (tests/exclusion_oracle.py).  A trie
prefix is valid for the history when at least one eligible item lies under it.  The searches treat an extension to a prefix that
is not valid as one the corpus lacks; the item retrieval returns eligible items only."""
import numpy as np

import beam_search_oracle as BS
from exclusion_oracle import tuple_key


def build(table, items, excls=None):
    """items [B, M] (and optionally the exclusion_oracle.build of the same histories) -> one dict per history: eligible (the
    set of eligible rows), pos (their positions in table["row"], ascending), keys ({l: sorted keys of the valid l-prefixes},
    l = 1..H) and bad (entries of items outside [-1, N))."""
    items = np.asarray(items, dtype=np.int64)
    row, start, H, K = table["row"], table["start"], table["C"], table["K"]
    N = len(row)
    inv = np.empty(N, dtype=np.int64)
    inv[row] = np.arange(N)
    tuples = {}                                                    # retrievable row -> its tuple
    for u, key in enumerate(table["keys"]):
        for r in row[start[u]:start[u + 1]]:
            tuples[int(r)] = tuple(int(v) for v in key)
    out = []
    for b, hist in enumerate(items):
        bad = int(((hist < -1) | (hist >= N)).sum())
        excluded = set() if excls is None else excls[b]["excluded"]
        eligible = set(int(i) for i in hist if 0 <= i < N and int(i) in tuples and int(i) not in excluded)
        keys = {l: sorted(set(tuple_key(tuples[r][:l], K) for r in eligible)) for l in range(1, H + 1)}
        out.append(dict(eligible=eligible, pos=sorted(int(inv[i]) for i in eligible), keys=keys, bad=bad))
    return out


def valid_prefix(incl, prefix, K):
    """Is the id prefix valid for the history of incl (one entry of build())?"""
    if not all(0 <= int(v) < K for v in prefix):
        return False
    sets = incl.setdefault("key_sets", {l: set(v) for l, v in incl["keys"].items()})
    return tuple_key(prefix, K) in sets[len(prefix)]


def valid_prefix_brute(corpus_ids, table, eligible, prefix):
    """valid_prefix by brute force over the corpus rows: some eligible row's first len(prefix) ids equal prefix."""
    corpus = np.asarray(corpus_ids)
    prefix = [int(v) for v in prefix]
    return any(corpus[r, :len(prefix)].tolist() == prefix for r in eligible)


def candidate_scores(corpus_ids, K, incls, logits, generated, log_probas):
    """[B, kp * K] float64: beam_search_oracle.candidate_scores' score of every extension, -inf where the extended prefix is
    not valid for the history (valid prefixes are corpus prefixes, so the corpus needs no separate test)."""
    logp = BS.log_softmax64(logits)
    logp = np.where(np.isnan(logp), -np.inf, logp)
    B = len(incls)
    if generated is None:
        kp, h = 1, 0
        scores = logp.reshape(B, 1, K)
        pkey, ok = np.zeros((B, 1), dtype=np.int64), np.ones((B, 1), dtype=bool)
    else:
        generated = np.asarray(generated, dtype=np.int64)
        _, kp, h = generated.shape
        scores = logp.reshape(B, kp, K) + np.asarray(log_probas, dtype=np.float64)[:, :, None]
        ok = ((generated >= 0) & (generated < K)).all(axis=2)
        pkey = np.zeros((B, kp), dtype=np.int64)
        for j in range(h):
            pkey = pkey * K + np.clip(generated[:, :, j], 0, K - 1)
    keys = pkey[:, :, None] * K + np.arange(K, dtype=np.int64)
    valid = np.stack([np.isin(keys[b], np.asarray(incls[b]["keys"][h + 1], dtype=np.int64)) for b in range(B)])
    valid &= ok[:, :, None]
    return np.where(valid, scores, -np.inf).reshape(B, kp * K)


def beam_topk(corpus_ids, K, incls, logits, generated, log_probas, k):
    """One level of the exhaustive beam search with allow-lists: the k best candidates of candidate_scores, equal scores
    (the -inf fillers among them) by ascending beam * K + code.  Returns (generated [B, k, h + 1], log_probas [B, k] float64,
    parent beam [B, k])."""
    scores = candidate_scores(corpus_ids, K, incls, logits, generated, log_probas)
    B = scores.shape[0]
    h = 0 if generated is None else generated.shape[2]
    order = np.argsort(-scores, axis=1, kind="stable")[:, :k]
    parent, code = order // K, order % K
    gen = np.zeros((B, k, h + 1), dtype=np.int64)
    for b in range(B):
        if h:
            gen[b, :, :h] = generated[b, parent[b]]
        gen[b, :, h] = code[b]
    return gen, np.take_along_axis(scores, order, axis=1), parent


def sample_scores(incls, K, samples, samp_log_p, generated, log_probas):
    """[B, kp * nc] float64: each sampled candidate's score in the sampled search, -inf when its prefix is not valid."""
    samples = np.asarray(samples)
    rows, nc = samples.shape
    B = len(incls)
    kp = rows // B
    out = np.full((B, kp * nc), -np.inf)
    for b in range(B):
        for beam in range(kp):
            plp = 0.0 if log_probas is None else float(log_probas[b, beam])
            prefix = [] if generated is None else [int(v) for v in generated[b, beam]]
            for r in range(nc):
                tok = int(samples[b * kp + beam, r])
                if valid_prefix(incls[b], prefix + [tok], K):
                    out[b, beam * nc + r] = float(samp_log_p[b * kp + beam, r]) + plp
    return out


def retrieve(table, incls, generated, log_probas, n):
    """item_oracle.retrieve returning only each history's eligible items."""
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
            got += [(it, j) for it in items_of(table, t) if it in incls[b]["eligible"]]
        got = got[:n]
        count[b] = len(got)
        for o, (it, j) in enumerate(got):
            items[b, o], beam[b, o] = it, j
    return items, beam, count
