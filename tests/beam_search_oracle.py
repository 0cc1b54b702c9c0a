"""Numpy oracle of one level of the exhaustive beam search (ops.SidPrefixIndex.beam_topk), built on oracle.rq_oracle.beam_select."""
import numpy as np

from oracle import rq_oracle as O


def log_softmax64(logits):
    """float64 log_softmax per row, x - (m + log(sum(exp(x - m)))); rows holding NaN or +inf, or all -inf, become all NaN."""
    x = np.asarray(logits, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        m = x.max(axis=1, keepdims=True)
        return x - (m + np.log(np.exp(x - m).sum(axis=1, keepdims=True)))


def beam_topk(corpus_ids, logits, generated, log_probas, k):
    """Every code of every beam is a candidate: candidates tile(arange(K)), scored by the float64 log_softmax of the beam's
    logits (NaN -> -inf) plus the parent's log-probability, prefixes absent from the corpus -inf, the k best by beam_select's
    stable sort (equal scores: lowest beam * K + code).  logits [B * kp, K]; generated [B, kp, h] or None; log_probas [B, kp]
    or None.  Returns (generated [B, k, h + 1], log_probas [B, k], parent_global [B, k])."""
    logits = np.asarray(logits)
    rows, K = logits.shape
    logp = log_softmax64(logits)
    logp = np.where(np.isnan(logp), -np.inf, logp)
    candidates = np.tile(np.arange(K, dtype=np.int64), (rows, 1))
    lp = None if log_probas is None else np.asarray(log_probas, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        return O.beam_select(corpus_ids, candidates, logp, generated, lp, k)


def candidate_scores(corpus_ids, logits, generated, log_probas):
    """[B, kp * K] float64 score of every candidate as beam_topk ranks them (-inf where the prefix is not in the corpus)."""
    logp = log_softmax64(logits)
    logp = np.where(np.isnan(logp), -np.inf, logp)
    rows, K = logp.shape
    codes = np.tile(np.arange(K, dtype=np.int64), rows)[:, None]
    if generated is None:
        B, prefix, scores = rows, codes, logp
    else:
        B, kp, h = generated.shape
        prefix = np.concatenate([np.repeat(generated.reshape(-1, h), K, axis=0), codes], axis=1)
        scores = logp.reshape(B, kp * K) + np.repeat(np.asarray(log_probas, dtype=np.float64), K, axis=1)
    return np.where(O.check_valid_prefix(corpus_ids, prefix).reshape(B, -1), scores.reshape(B, -1), -np.inf)
