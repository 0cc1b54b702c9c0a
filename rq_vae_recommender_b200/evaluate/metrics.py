"""evaluate/metrics.py of the reference: ``TopKAccumulator`` with the same names, methods and reduced keys, accumulated on the
device.

The reference builds a [B, k, D] compare for every evaluation batch and waits on the host for the NDCG sum and once more per
entry of ``ks``.  Here ``accumulate`` adds every row's rank -- its first candidate equal to the actual ids in all D columns, k when
none is -- to an int64 histogram on the device in one launch (``ops.sid_topk_rank_hist``) and never waits on the host.
``reduce`` copies the histograms once and computes from them
    ndcg = sum_r hist[r] / log2(r + 2) / total,    h@j = sum_{r < j} hist[r] / total.
``accumulate_items`` is an addition: it scores lists of corpus items (``EncoderDecoderRetrievalModel.generate_items``) against the
true next item (``EncoderDecoderRetrievalModel.item_of``) in separate histograms, reported as ``item_ndcg`` and ``item_h@{k}``.
There a -1 (padding, an item that could not be resolved) never matches.  ``accumulate_ranks`` is another addition: exact ranks
(``EncoderDecoderRetrievalModel.rank_items``' target_rank, -1 a miss) in a third histogram, reported as ``exact_ndcg`` and
``exact_h@{k}``.  The reference's keys are unchanged.
"""
from typing import Dict
from typing import Sequence

import numpy as np
import torch
from torch import Tensor

from .. import ops


def metrics_from_hist(hist, total: int, ks: Sequence[int], prefix: str = "") -> Dict[str, float]:
    """The reduced metrics of a rank histogram over ``total`` rows: hist[r] rows of rank r < k, hist[k] rows without a match.
    Keys in the reference's order: ``prefix + "ndcg"``, then ``prefix + f"h@{j}"`` for each j in ks."""
    h = np.asarray(hist, dtype=np.float64)
    k = h.shape[0] - 1
    out = {prefix + "ndcg": float((h[:k] / np.log2(np.arange(k) + 2.0)).sum()) / total}
    for j in ks:
        out[f"{prefix}h@{j}"] = float(h[:max(0, min(j, k))].sum()) / total
    return out


class TopKAccumulator:
    def __init__(self, ks=[1, 5, 10]):
        self.ks = ks
        self.reset()

    def reset(self):
        self.total = 0
        self.item_total = 0
        self.exact_total = 0
        self._hists = {}                                     # (mode, k, device) -> int64 [k + 1] device histogram

    def _add(self, actual: Tensor, candidates: Tensor, item_mode: bool) -> None:
        key = (item_mode, candidates.shape[1], candidates.device)
        hist = self._hists.get(key)
        if hist is None:
            hist = self._hists[key] = torch.zeros(candidates.shape[1] + 1, dtype=torch.int64, device=candidates.device)
        ops.sid_topk_rank_hist(actual, candidates, hist, item_mode=item_mode)

    def accumulate(self, actual: Tensor, top_k: Tensor) -> None:
        """actual [B, D] ids, top_k [B, k, D] candidates (generate's beams): one launch, no host synchronisation."""
        B, D = actual.shape
        self._add(actual, top_k, False)
        self.total += B

    def accumulate_items(self, actual_items: Tensor, retrieved_items: Tensor) -> None:
        """actual_items [B] item ids (-1: unknown), retrieved_items [B, n] item lists (-1 pads): one launch, no host
        synchronisation."""
        actual = actual_items.reshape(-1, 1)
        self._add(actual, retrieved_items.reshape(actual.shape[0], -1).unsqueeze(-1), True)
        self.item_total += actual.shape[0]

    def accumulate_ranks(self, rank: Tensor, num_items: int) -> None:
        """rank [B] int64: exact 0-based ranks among num_items ranked items (-1: a miss), e.g. ``rank_items``' target_rank and
        num_items.  One launch into a histogram of num_items + 1 bins, no host synchronisation."""
        rank = rank.reshape(-1)
        key = ("exact", max(1, int(num_items)), rank.device)
        hist = self._hists.get(key)
        if hist is None:
            hist = self._hists[key] = torch.zeros(key[1] + 1, dtype=torch.int64, device=rank.device)
        ops.sid_rank_hist(rank, hist)
        self.exact_total += rank.shape[0]

    def reduce(self) -> dict:
        if not self._hists:
            return {}
        keys = list(self._hists)
        dev = keys[0][2]
        flat = torch.cat([self._hists[key].to(dev) for key in keys]).cpu().numpy()   # the one wait on the device
        out = {}
        for item_mode, prefix, total in ((False, "", self.total), (True, "item_", self.item_total),
                                         ("exact", "exact_", self.exact_total)):
            parts, at = [], 0
            for key in keys:
                k = key[1]
                if key[0] == item_mode:
                    parts.append((k, flat[at:at + k + 1]))
                at += k + 1
            if not parts:
                continue
            kmax = max(k for k, _ in parts)
            hist = np.zeros(kmax + 1, dtype=np.int64)
            for k, h in parts:                               # histograms of batches with fewer candidates: ranks, then no match
                hist[:k] += h[:k]
                hist[kmax] += h[k]
            out.update(metrics_from_hist(hist, total, self.ks, prefix))
        return out
