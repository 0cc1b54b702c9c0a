"""init/kmeans.py of the reference (:8-72) on the fused assign+accumulate kernel.

Per Lloyd iteration the reference builds a [B,K,D] broadcast tensor and loops over the K clusters in Python;
here one kernel launch does the assignment (same direct (x-c)^2 distance) and the per-cluster fp64 sums/counts,
a second one writes the means.  RNG draws stay on the host in the reference's order: ``np.random.choice`` once
(kmeans.py:35), ``torch.randint`` once per empty cluster in cluster order (kmeans.py:53).

``group``: when a torch.distributed process group is given, ``x`` is this rank's shard of the rows and the
sums/counts are all-reduced every iteration; see parallel.py for the driver."""
from typing import NamedTuple, Optional

import numpy as np
import torch

from .. import ops


def kmeans_init_(tensor: torch.Tensor, x: torch.Tensor):
    assert tensor.dim() == 2
    assert x.dim() == 2

    with torch.no_grad():
        k, _ = tensor.shape
        kmeans_out = Kmeans(k=k).run(x)
        tensor.data.copy_(kmeans_out.centroids)


class KmeansOutput(NamedTuple):
    centroids: torch.Tensor
    assignment: torch.Tensor


class Kmeans:
    def __init__(self, k: int, max_iters: int = None, stop_threshold: float = 1e-10) -> None:
        self.k = k
        self.iters = max_iters
        self.stop_threshold = stop_threshold
        self.centroids = None
        self.assignment = None
        self.n_iters = 0

    def _init_centroids(self, x: torch.Tensor) -> None:
        B, D = x.shape
        init_idx = np.random.choice(B, self.k, replace=False)
        self.centroids = x[torch.as_tensor(init_idx, device=x.device), :].contiguous()
        self.assignment = None

    def _draw_reseed_rows(self, counts_host: torch.Tensor, n_rows: int, device) -> Optional[torch.Tensor]:
        empty = torch.nonzero(counts_host == 0).flatten().tolist()
        if not empty:
            return None
        if n_rows <= 0:
            raise ValueError("Can not choose random element from x, x is empty")
        rows = torch.full((self.k,), -1, dtype=torch.int64)
        for c in empty:                                    # cluster order, one draw each (kmeans.py:48-54)
            rows[c] = torch.randint(0, n_rows, (1,)).item()
        return rows.to(device)

    def _update_centroids(self, x, buf) -> float:
        ops.kmeans_assign_accumulate(x, self.centroids, buf)
        reseed = self._draw_reseed_rows(buf["counts"].cpu(), x.size(0), x.device)
        ops.kmeans_finalize(x, self.centroids, buf, reseed)
        self.assignment = buf["assign"]
        return float(buf["shift"].item())

    @torch.no_grad()
    def run(self, x):
        x = x.detach()
        if x.dtype != torch.float32:
            x = x.float()
        if x.stride(-1) != 1:
            x = x.contiguous()
        self._init_centroids(x)
        buf = ops.kmeans_workspace(x, self.k)

        i = 0
        while self.iters is None or i < self.iters:
            shift = self._update_centroids(x, buf)
            self.n_iters = i + 1
            if shift < self.stop_threshold:
                break
            i += 1

        return KmeansOutput(centroids=self.centroids, assignment=self.assignment)
