"""Numpy oracle of the sampled beam-search level (ops.SidPrefixIndex.sample_select), built on oracle.rq_oracle.beam_select."""
import numpy as np

from oracle import rq_oracle as O


def topk_order_key(v: np.ndarray) -> np.ndarray:
    """int64 image of fp32 values in the order torch.topk ranks them: NaN largest, -0 below +0."""
    x = np.ascontiguousarray(v, dtype=np.float32).view(np.uint32).astype(np.int64)
    key = np.where(x & 0x80000000, 0xFFFFFFFF - x, x | 0x80000000)
    return np.where(np.isnan(v), 0xFFFFFFFF, key)


def sample_select(corpus_ids, probas, noise, generated, log_probas, k, nc):
    """Sampling step + selection step of the constrained beam search, modules/model.py:345-388.  torch.multinomial(probas, nc)
    without replacement is topk(probas / noise, nc) with noise = empty_like(probas).exponential_(1) from the same generator:
    the samples are the nc largest fp32 ratios, descending (stable: equal ratios by ascending index), samp_log_p their log
    probabilities; then beam_select.  probas / noise [B * kp, K]; generated [B, kp, h] or None; log_probas [B, kp] or None.
    Returns (generated, log_probas, parent_global, samples, samp_log_p)."""
    probas = np.asarray(probas, dtype=np.float32)
    ratio = (probas / np.asarray(noise, dtype=np.float32)).astype(np.float32)
    samples = np.argsort(-topk_order_key(ratio), axis=1, kind="stable")[:, :nc]
    with np.errstate(divide="ignore", invalid="ignore"):
        samp_log_p = np.log(np.take_along_axis(probas, samples, 1))
    gen, lp, parent = O.beam_select(corpus_ids, samples, samp_log_p, generated, log_probas, k)
    return gen, lp, parent, samples, samp_log_p
