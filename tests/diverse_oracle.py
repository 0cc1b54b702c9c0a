"""numpy statement of one level of the generative-retrieval search under a per-prefix cap (max_per_prefix beams per
prefix_len-prefix), for the exhaustive "beam" search and the sampled "sample" search.

A candidate's group is its parent beam's first prefix_len ids, named by the lowest beam of the history with an equal prefix.
The kept set is the greedy walk down the uncapped order (score descending, lowest flat index first) that accepts a candidate
unless its group already holds max_per_prefix accepted ones; NaN scores count as -inf and -inf candidates are not beams.
Equivalently every finite candidate outside its group's max_per_prefix best drops to -inf, and the uncapped selection then
takes the k best, the -inf fillers by lowest flat index."""
import numpy as np

import beam_search_oracle as O


def groups(generated, prefix_len):
    """int [B, kp]: each beam's group, the lowest beam of its history whose first prefix_len ids equal its own."""
    g = np.asarray(generated)
    B, kp = g.shape[:2]
    out = np.empty((B, kp), dtype=np.int64)
    for b in range(B):
        seen = {}
        for j in range(kp):
            out[b, j] = seen.setdefault(tuple(g[b, j, :prefix_len].tolist()), j)
    return out


def capped_scores(scores, grp, per_beam, m):
    """scores [B, kp * per_beam] (any float dtype) with every finite candidate outside its group's m best (score descending,
    lowest flat index first) set to -inf; NaN becomes -inf.  grp [B, kp] from ``groups``."""
    s = np.where(np.isnan(scores), -np.inf, scores).astype(scores.dtype)
    out = s.copy()
    B, E = s.shape
    for b in range(B):
        beam_group = np.repeat(grp[b], per_beam)
        for g in np.unique(grp[b]):
            idx = np.nonzero(beam_group == g)[0]
            order = idx[np.lexsort((idx, -s[b, idx].astype(np.float64)))]   # score descending, then index ascending
            drop = order[m:]
            out[b, drop] = -np.inf
    return out


def select(scores, k):
    """(flat indices [B, k], scores [B, k]): the k best by score descending, lowest flat index first (-0 equal to +0)."""
    s = np.where(np.isnan(scores), -np.inf, scores)
    idx = np.argsort(-s.astype(np.float64), axis=1, kind="stable")[:, :k]
    return idx, np.take_along_axis(s, idx, 1)


def greedy_walk(scores, grp, per_beam, m, k):
    """The statement's walk itself, one candidate at a time (the reference for ``capped_scores`` + ``select``): flat indices
    [B, k] and their scores, the unfilled slots then taken by the lowest flat indices not yet kept, at -inf."""
    s = np.where(np.isnan(scores), -np.inf, scores)
    B, E = s.shape
    idx = np.empty((B, k), dtype=np.int64)
    val = np.empty((B, k), dtype=s.dtype)
    for b in range(B):
        held, kept = {}, []
        fin = np.nonzero(np.isfinite(s[b]))[0]
        for e in fin[np.lexsort((fin, -s[b, fin].astype(np.float64)))]:
            if len(kept) == k:
                break
            g = grp[b, e // per_beam]
            if held.get(g, 0) < m:
                held[g] = held.get(g, 0) + 1
                kept.append(int(e))
        taken = set(kept)
        fill = [e for e in range(min(E, k + len(kept))) if e not in taken][:k - len(kept)]
        idx[b] = kept + fill
        val[b] = [s[b, e] for e in kept] + [-np.inf] * len(fill)
    return idx, val


def beam_topk_capped(corpus_ids, logits, generated, log_probas, k, prefix_len, m):
    """The capped "beam" level on ``beam_search_oracle.candidate_scores`` (float64): (generated [B, k, h + 1], log_probas
    [B, k], parent_global [B, k]) as ``beam_search_oracle.beam_topk`` returns them."""
    scores = O.candidate_scores(corpus_ids, logits, generated, log_probas)
    B, kp, h = np.asarray(generated).shape
    K = np.asarray(logits).shape[1]
    idx, val = select(capped_scores(scores, groups(generated, prefix_len), K, m), k)
    beam, code = idx // K, idx % K
    gen = np.concatenate([np.take_along_axis(np.asarray(generated), beam[:, :, None], 1), code[:, :, None]], axis=2)
    return gen, val, np.arange(B)[:, None] * kp + beam


def sample_order_scores(samples, samp_log_p, corpus_ids, generated, log_probas, valid=None):
    """[B, kp * nc] fp32 candidate scores of the sampled level in its flat order (beam * nc + slot): samp_log_p + the parent's,
    -inf where the extended prefix is invalid (``valid(b, prefix)``, default: a corpus prefix) or the score is NaN --
    ``sample_oracle``'s order, on which the capped walk runs."""
    generated = np.asarray(generated)
    B, kp, h = generated.shape
    nc = samples.shape[1]
    prefixes = {tuple(r[:h + 1]) for r in np.asarray(corpus_ids).tolist()}
    valid = valid or (lambda b, prefix: tuple(prefix) in prefixes)
    lp = np.asarray(samp_log_p, dtype=np.float32).reshape(B, kp, nc) + np.asarray(log_probas, dtype=np.float32)[:, :, None]
    out = lp.astype(np.float32)
    for b in range(B):
        for j in range(kp):
            for r in range(nc):
                if not valid(b, list(generated[b, j]) + [int(samples[b * kp + j, r])]) or np.isnan(out[b, j, r]):
                    out[b, j, r] = -np.inf
    return out.reshape(B, kp * nc)

