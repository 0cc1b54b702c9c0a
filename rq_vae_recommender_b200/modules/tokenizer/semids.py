"""modules/tokenizer/semids.py of the reference (:22-146) on the fused tokeniser kernels.

Same class name, constructor and methods.  ``precompute_corpus_ids`` differs underneath:
  * the corpus goes through ``RqVae.tokenize`` in 65 536-row batches -> ``ops.rq_tokenize_auto``: the wgmma candidate
    filter + exact re-rank (prepared state cached on the codebooks; D = 32 / 64 quantisers zero-padded to 64) when K is
    256, 512, ..., 2048 and the batch has >= 1 024 rows, else the exact CUDA-core kernel -- instead of 512-row batches of
    full RqVae forwards;
  * the dedup column -- the number of EARLIER corpus rows with the same id tuple, which the reference finds with an
    O(N^2) compare against everything seen so far (semids.py:94-108, 90-97 % of its wall time, SURVEY 8f-1) -- is the
    rank inside a stable sort of packed tuples: identical values, O(N log N).
"""
from typing import List
from typing import Optional

import torch
from torch import nn
from torch import Tensor

from .. import utils as _utils
from ... import ops
from ...data.schemas import SeqBatch
from ...data.schemas import TokenizedSeqBatch
from ..rqvae import RqVae

BATCH_SIZE = 16
eval_mode = _utils.eval_mode


def dedup_rank(sem_ids: Tensor, codebook_size: int) -> Tensor:
    """[N] int64: for every row, how many earlier rows carry the identical id tuple (semids.py:94-108)."""
    N, L = sem_ids.shape
    if N == 0:
        return torch.zeros(0, dtype=torch.int64, device=sem_ids.device)
    if sem_ids.is_cuda:
        res = ops.sid_dedup_rank(sem_ids, codebook_size)       # direct-table kernel: no sort, O(N) on near-unique tables
        if res is not None:
            return res[0]
    if codebook_size ** L < 2 ** 62:
        key = sem_ids[:, 0].clone()
        for l in range(1, L):
            key = key * codebook_size + sem_ids[:, l]
    else:
        _, key = torch.unique(sem_ids, dim=0, return_inverse=True)
    skey, order = torch.sort(key, stable=True)
    pos = torch.arange(N, device=key.device)
    is_start = torch.ones(N, dtype=torch.bool, device=key.device)
    is_start[1:] = skey[1:] != skey[:-1]
    start = torch.cummax(torch.where(is_start, pos, torch.zeros_like(pos)), dim=0).values
    rank = torch.empty(N, dtype=torch.int64, device=key.device)
    rank[order] = pos - start
    return rank


def corpus_id_stats(cached_ids: Tensor, codebook_size: int) -> dict:
    """The ID-diversity numbers train_rqvae.py:276-292 logs after ``precompute_corpus_ids`` -- ``max_id_duplicates``,
    ``rqvae_entropy`` and ``codebook_usage_{l}`` -- as 0-d device tensors from three kernel launches (dedup/entropy pass +
    per-level usage histogram) instead of ``torch.unique(dim=0)`` + a Python loop over levels."""
    n = cached_ids.shape[0]
    sem_ids = cached_ids[:, :-1].contiguous()
    L = sem_ids.shape[1]
    out = {}
    res = ops.sid_dedup_rank(sem_ids, codebook_size) if cached_ids.is_cuda else None
    if res is not None:
        _, st = res
        out["rqvae_entropy"] = st["entropy"].to(torch.float32)
    else:
        _, counts = torch.unique(sem_ids, dim=0, return_counts=True)
        p = counts / n
        out["rqvae_entropy"] = -(p * torch.log(p)).sum()
    out["max_id_duplicates"] = cached_ids[:, -1].max() / n
    hist = ops.sid_histogram(sem_ids, codebook_size)
    for l in range(L):
        out[f"codebook_usage_{l}"] = (hist[l] > 0).sum() / codebook_size
    return out


class SemanticIdTokenizer(nn.Module):
    """
    Tokenizes a batch of sequences of item features into a batch of sequences of semantic ids.
    """

    def __init__(
        self,
        input_dim: int,
        output_dim: int,
        hidden_dims: List[int],
        codebook_size: int,
        n_layers: int = 3,
        n_cat_feats: int = 18,
        commitment_weight: float = 0.25,
        rqvae_weights_path: Optional[str] = None,
        rqvae_codebook_normalize: bool = False,
        rqvae_sim_vq: bool = False,
    ) -> None:
        super().__init__()

        self.rq_vae = RqVae(
            input_dim=input_dim,
            embed_dim=output_dim,
            hidden_dims=hidden_dims,
            codebook_size=codebook_size,
            codebook_kmeans_init=False,
            codebook_normalize=rqvae_codebook_normalize,
            codebook_sim_vq=rqvae_sim_vq,
            n_layers=n_layers,
            n_cat_features=n_cat_feats,
            commitment_weight=commitment_weight,
        )

        if rqvae_weights_path is not None:
            self.rq_vae.load_pretrained(rqvae_weights_path)

        self.rq_vae.eval()

        self.codebook_size = codebook_size
        self.n_layers = n_layers
        self.corpus_batch = 65536
        self.reset()

    def _get_hits(self, query: Tensor, key: Tensor) -> Tensor:
        return (key.unsqueeze(0) == query.unsqueeze(1)).all(axis=-1)

    def reset(self):
        self.cached_ids = None

    @property
    def sem_ids_dim(self):
        return self.n_layers + 1

    @torch.no_grad
    @eval_mode
    def precompute_corpus_ids(self, movie_dataset) -> Tensor:
        n = len(movie_dataset)
        device = self.rq_vae.device
        blocks = []
        for s in range(0, n, self.corpus_batch):
            idx = list(range(s, min(n, s + self.corpus_batch)))
            batch = movie_dataset[idx]
            x = batch.x.to(device)
            tok = getattr(self.rq_vae, "tokenize", None)
            blocks.append(tok(x) if tok is not None else self.rq_vae.get_semantic_ids(x).sem_ids)
        sem_ids = torch.cat(blocks, dim=0) if blocks else torch.zeros((0, self.n_layers), dtype=torch.int64, device=device)
        dedup = dedup_rank(sem_ids, self.codebook_size)
        self.cached_ids = torch.cat([sem_ids, dedup.unsqueeze(1)], dim=1)
        return self.cached_ids

    def _tokenize_seq_batch_from_cached(self, ids: Tensor) -> Tensor:
        return ops.sid_gather(self.cached_ids, ids, None, want_token_type=False)[0]

    @torch.no_grad
    @eval_mode
    def forward(self, batch: SeqBatch) -> TokenizedSeqBatch:
        if self.cached_ids is None or batch.ids.max() >= self.cached_ids.shape[0]:
            B, N = batch.ids.shape
            sem_ids = self.rq_vae.get_semantic_ids(batch.x).sem_ids
            D = sem_ids.shape[-1]
            seq_mask, sem_ids_fut = None, None
        else:
            B, N = batch.ids.shape
            _, D = self.cached_ids.shape
            # one kernel: gather + -1 under the padding mask + token_type_ids (reference: index, repeat_interleave, masked
            # assignment, arange().repeat())
            sem_ids, token_type_ids = ops.sid_gather(self.cached_ids, batch.ids, batch.seq_mask)
            seq_mask = batch.seq_mask.repeat_interleave(D, dim=1)
            sem_ids_fut, token_type_ids_fut = ops.sid_gather(self.cached_ids, batch.ids_fut, None)

        if seq_mask is None:
            token_type_ids = torch.arange(D, device=sem_ids.device).repeat(B, N)
            token_type_ids_fut = torch.arange(D, device=sem_ids.device).repeat(B, 1)
        return TokenizedSeqBatch(
            user_ids=batch.user_ids,
            sem_ids=sem_ids,
            sem_ids_fut=sem_ids_fut,
            seq_mask=seq_mask,
            token_type_ids=token_type_ids,
            token_type_ids_fut=token_type_ids_fut,
        )
