"""Multi-GPU and host-facing drivers of the hot path.

* ``CorpusTokenizer``: items -> semantic ids.  Rows are independent, so a corpus is cut into contiguous shards,
  one per rank, tokenised with no data-path collective, and only the [N/G, L] id blocks are all-gathered.
* ``sharded_kmeans_init_``: k-means codebook init over row shards; per Lloyd iteration one all-reduce of the
  [K, D] fp64 sums + [K] counts (one flat buffer), identical centroid update on every rank.
* ``codebook_usage``: [L,K] usage counts, all-reduced.

torch.distributed is the plumbing (NCCL on GPUs; the same code runs on gloo for the CPU logic tests with the
kernel calls injected).
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from . import ops


def shard_bounds(n: int, world: int, rank: int):
    """Contiguous shard [lo, hi) of n rows for `rank` (first n % world ranks get one extra row)."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class CorpusTokenizer:
    """Frozen codebooks -> ids.  ``use_tc`` selects the wgmma filter + exact re-rank kernel (state prepared once; its margin is
    a deterministic bound, so the result contract is the exact kernel's).  Default: on whenever the shape allows it (K = 256 m
    with m = 1..8, D <= 768; widths that are not a multiple of 64 are zero-padded)."""

    def __init__(self, codebooks: Sequence[torch.Tensor], use_tc: Optional[bool] = None,
                 encoder: Optional[Callable[[torch.Tensor], torch.Tensor]] = None, chunk_rows: int = 16384):
        self.codebooks = [c.detach() for c in codebooks]
        self.K, self.D = self.codebooks[0].shape
        self.L = len(self.codebooks)
        if use_tc is None:
            use_tc = bool(ops.tc_padded_dim(self.D, self.K, self.L))
        self.use_tc = bool(use_tc)
        self._state = ops.TcState(self.codebooks) if self.use_tc else None
        self._state_build = ops.StreamBuild(self._state.buf) if self.use_tc else None
        self.encoder = encoder
        self.chunk_rows = chunk_rows
        self._copy_stream = None
        self._host_out = None
        self._ring = None

    @property
    def state(self) -> Optional[ops.TcState]:
        """The prepared codebooks of the tensor-core tokeniser (None without it), with the current stream ordered after their
        preparation (``ops.StreamBuild``)."""
        if self._state_build is not None:
            self._state_build.ready()
        return self._state

    # ---- device resident rows
    @torch.no_grad()
    def tokenize_device(self, x: torch.Tensor, stats=None) -> torch.Tensor:
        if self.encoder is not None:
            x = self.encoder(x)
        if self.use_tc:
            return ops.rq_tokenize_tc(x, state=self.state, stats=stats)
        return ops.rq_tokenize(x, self.codebooks)

    # ---- host rows in, host ids out (the reference's semids.py:93 copies every 512-row batch H->D)
    RING = 3

    @torch.no_grad()
    def tokenize_host(self, x_host: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Pipelined over ``chunk_rows`` chunks with a ring of RING device buffers: chunk i+1 (and i+2) are copied host->device
        on a side stream while chunk i is quantised, and a buffer is refilled only after the kernel that read it has finished,
        so at most RING chunks (not the corpus) are resident.  ``x_host`` should be pinned for the copies to overlap.
        Returns ``out`` if given; otherwise the tokenizer's own pinned result buffer, which the NEXT call with the same row
        count overwrites -- pass ``out=`` (or clone) to keep a result across calls."""
        n = x_host.shape[0]
        dev = self.codebooks[0].device
        if out is None:                       # pinned result buffer, allocated once per size (cudaHostAlloc is slow)
            if self._host_out is None or self._host_out.shape[0] != n:
                self._host_out = torch.empty((n, self.L), dtype=torch.int64).pin_memory()
            out = self._host_out
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=dev)
        width = x_host.shape[1]
        if self._ring is None or self._ring[0].shape[1] != width or self._ring[0].dtype != x_host.dtype:
            self._ring = [torch.empty((self.chunk_rows, width), dtype=x_host.dtype, device=dev) for _ in range(self.RING)]
        main = torch.cuda.current_stream(dev)
        cs = self._copy_stream
        cs.wait_stream(main)
        starts = list(range(0, n, self.chunk_rows))
        copied = [None] * len(starts)         # event: chunk i landed in ring[i % RING]
        consumed = [None] * len(starts)       # event: the kernel that read chunk i has finished

        def issue_copy(i):
            if i >= len(starts):
                return
            if i >= self.RING:
                cs.wait_event(consumed[i - self.RING])
            s = starts[i]
            rows = min(self.chunk_rows, n - s)
            with torch.cuda.stream(cs):
                self._ring[i % self.RING][:rows].copy_(x_host[s:s + rows], non_blocking=True)
                copied[i] = torch.cuda.Event()
                copied[i].record(cs)

        for i in range(min(self.RING, len(starts))):
            issue_copy(i)
        for i, s in enumerate(starts):
            rows = min(self.chunk_rows, n - s)
            main.wait_event(copied[i])
            ids = self.tokenize_device(self._ring[i % self.RING][:rows])
            consumed[i] = torch.cuda.Event()
            consumed[i].record(main)
            out[s:s + rows].copy_(ids, non_blocking=True)
            issue_copy(i + self.RING)
        main.synchronize()
        return out

    # ---- corpus sharded over the ranks of `group`
    @torch.no_grad()
    def tokenize_sharded(self, x_local: torch.Tensor, n_total: int, group=None) -> torch.Tensor:
        """x_local = rows shard_bounds(n_total, world, rank) of the corpus; returns the full [n_total, L] table on
        every rank (all-gather of int32 id blocks, corpus order)."""
        import torch.distributed as dist
        ids_local = self.tokenize_device(x_local)
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return ids_local
        return all_gather_rows(ids_local.to(torch.int32), n_total, group).to(torch.int64)


def all_gather_rows(block: torch.Tensor, n_total: int, group=None) -> torch.Tensor:
    """Concatenate per-rank row blocks (sizes given by shard_bounds) in rank order on every rank."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    sizes = [shard_bounds(n_total, world, r) for r in range(world)]
    mx = max(hi - lo for lo, hi in sizes)
    pad = torch.zeros((mx,) + tuple(block.shape[1:]), dtype=block.dtype, device=block.device)
    pad[: block.shape[0]] = block
    gathered = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(gathered, pad, group=group)
    return torch.cat([g[: hi - lo] for g, (lo, hi) in zip(gathered, sizes)], dim=0)


def codebook_usage(sem_ids_local: torch.Tensor, K: int, group=None, hist_fn=None) -> torch.Tensor:
    """[L,K] int64 usage counts over all shards (train_rqvae.py:285-289 semantics), all-reduced."""
    import torch.distributed as dist
    hist = (hist_fn or ops.sid_histogram)(sem_ids_local, K)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(hist, group=group)
    return hist


# ------------------------------------------------------------------------------------------------ sharded k-means
def _default_assign_accumulate(x, centroids, buf):
    ops.kmeans_assign_accumulate(x, centroids, buf)


def _default_finalize(x, centroids, buf, reseed):
    ops.kmeans_finalize(x, centroids, buf, reseed)


@torch.no_grad()
def sharded_kmeans(x_local: torch.Tensor, k: int, n_total: int, group=None, max_iters: Optional[int] = None,
                   stop_threshold: float = 1e-10, assign_accumulate=None, finalize=None, make_buf=None,
                   check_every: int = 4):
    """init/kmeans.py semantics over a row-sharded x (every rank holds shard_bounds(n_total, world, rank)).

    Per Lloyd iteration: local assign + fp64 accumulate (one kernel), the [k, D] fp64 sums and the [k] int32 counts are
    all-reduced IN PLACE (two NCCL calls on the kernel's own buffers, no staging copy), identical centroid update on every
    rank.  The host is consulted once every ``check_every`` iterations, not twice per iteration: the per-iteration shift and
    an "a cluster came up empty" flag are recorded on the device.  Empty clusters are rare (every initial centroid is a data
    row) and need the reference's host RNG draw in THAT iteration (kmeans.py:48-54), so a window that saw one is rolled back to
    its snapshot and replayed with per-iteration host checks -- results are those of the reference's loop either way.  A window
    may run up to ``check_every - 1`` iterations past convergence; with the reference's threshold (1e-10: a fixed point) they
    change nothing.

    RNG: every rank draws the SAME global ``np.random.choice(n_total, k)`` (seed numpy identically on all ranks, as for a
    single process) and, for empty clusters, rank 0 draws ``torch.randint(0, n_total)`` and broadcasts.  Rows named by a
    global index are fetched from their owners with ONE sum all-reduce of a one-hot-masked [k, D] buffer (init and re-seed
    only; k rows with k different owners: a single small collective beats k broadcasts).
    Returns (centroids [k,D], local assignment, n_iters)."""
    import torch.distributed as dist
    distributed = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
    world = dist.get_world_size(group) if distributed else 1
    rank = dist.get_rank(group) if distributed else 0
    lo, hi = shard_bounds(n_total, world, rank)
    assert x_local.shape[0] == hi - lo, (x_local.shape, lo, hi)
    dev = x_local.device
    D = x_local.shape[1]
    assign_accumulate = assign_accumulate or _default_assign_accumulate
    finalize = finalize or _default_finalize
    buf = (make_buf or ops.kmeans_workspace)(x_local, k)

    def fetch_rows(global_idx: torch.Tensor) -> torch.Tensor:
        """rows x[global_idx] ([m] int64 on host; -1 = none) gathered from their owners -> [m, D] on every rank"""
        out = torch.zeros((len(global_idx), D), dtype=torch.float32, device=dev)
        mine = (global_idx >= lo) & (global_idx < hi)
        if mine.any():
            sel = torch.nonzero(mine).flatten()
            out[sel.to(dev)] = x_local[(global_idx[sel] - lo).to(dev)]
        if distributed:
            dist.all_reduce(out, group=group)
        return out

    def accumulate(centroids):
        assign_accumulate(x_local, centroids, buf)
        if distributed:                                    # in place, on the buffers the kernel wrote
            dist.all_reduce(buf["sums"], group=group)
            dist.all_reduce(buf["counts"], group=group)

    def reseed_empty(centroids, counts_h):
        empty = torch.nonzero(counts_h == 0).flatten()
        if len(empty):
            if n_total <= 0:
                raise ValueError("Can not choose random element from x, x is empty")
            draws = torch.tensor([int(torch.randint(0, n_total, (1,))) for _ in empty.tolist()], dtype=torch.int64)
            if distributed:
                d = draws.to(dev)
                dist.broadcast(d, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
                draws = d.cpu()
            centroids[empty.to(dev)] = fetch_rows(draws)

    init_idx = torch.from_numpy(np.random.choice(n_total, k, replace=False).astype(np.int64))
    centroids = fetch_rows(init_idx).contiguous()
    check_every = max(1, int(check_every))
    rec = torch.zeros((2, check_every), dtype=torch.float32, device=dev)     # [shift, any-empty] per iteration of the window
    i = 0
    n_iters = 0
    done = False
    while not done and (max_iters is None or i < max_iters):
        snapshot, i0 = centroids.clone(), i
        w = 0
        while w < check_every and (max_iters is None or i < max_iters):      # ---- a window without host contact
            accumulate(centroids)
            old = centroids.clone()
            finalize(x_local, centroids, buf, None)         # means; an empty cluster keeps its old centroid
            rec[0, w] = (centroids - old).norm(dim=1).max()
            rec[1, w] = (buf["counts"] == 0).any().float()
            w += 1
            i += 1
        h = rec[:, :w].cpu()                                # the window's only synchronisation
        if bool((h[1] > 0).any()):
            # an empty cluster: replay this window the reference's way (host RNG draw in the iteration that needs it)
            centroids.copy_(snapshot)
            i = i0
            for _ in range(w):
                accumulate(centroids)
                counts_h = buf["counts"].cpu()
                old = centroids.clone()
                finalize(x_local, centroids, buf, None)
                reseed_empty(centroids, counts_h)
                shift = float((centroids - old).norm(dim=1).max().item())
                i += 1
                n_iters = i
                if shift < stop_threshold:
                    done = True
                    break
        else:
            n_iters = i
            below = torch.nonzero(h[0] < stop_threshold).flatten()
            if len(below):
                n_iters = i0 + int(below[0]) + 1
                done = True
    return centroids, buf["assign"], n_iters


@torch.no_grad()
def sharded_kmeans_init_(weight: torch.Tensor, x_local: torch.Tensor, n_total: int, group=None, **kw) -> None:
    """kmeans_init_(tensor, x) (init/kmeans.py:8-15) for a row-sharded x: every rank ends with the same codebook."""
    centroids, _, _ = sharded_kmeans(x_local, weight.shape[0], n_total, group, **kw)
    weight.data.copy_(centroids)
