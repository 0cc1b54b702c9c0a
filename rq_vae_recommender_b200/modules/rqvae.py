"""modules/rqvae.py of the reference (:37-175) on the fused sm_90a kernels.

Same class / NamedTuple names, constructor signature, state-dict keys and HF-hub mixin, so the reference's
train_rqvae.py, train_decoder.py and SemanticIdTokenizer use it unchanged.  What differs is underneath:
``get_semantic_ids`` runs the L chained Quantize levels (distance, argmin, gather, STE / rotation output, loss,
residual update) in ONE kernel launch with the residual tile held on chip; ``forward`` uses the lean variant
that never materialises the [B,D,L] embeddings/residuals stacks (it needs only sum_l emb, ||emb_l|| and the loss),
and replaces the O(B^2) p_unique_ids compare by a sort of packed id tuples."""
from functools import cached_property
from typing import List
from typing import NamedTuple

import torch
from torch import nn
from torch import Tensor

from huggingface_hub import PyTorchModelHubMixin

from .. import ops
from ..data.schemas import SeqBatch
from .encoder import MLP
from .loss import CategoricalReconstuctionLoss
from .loss import ReconstructionLoss
from .loss import QuantizeLoss  # noqa: F401  (re-exported like the reference module)
from .normalize import l2norm
from .quantize import Quantize
from .quantize import QuantizeForwardMode

torch.set_float32_matmul_precision("high")


class RqVaeOutput(NamedTuple):
    embeddings: Tensor
    residuals: Tensor
    sem_ids: Tensor
    quantize_loss: Tensor


class RqVaeComputedLosses(NamedTuple):
    loss: Tensor
    reconstruction_loss: Tensor
    rqvae_loss: Tensor
    embs_norm: Tensor
    p_unique_ids: Tensor


@torch.compiler.disable      # ctypes call into librqb200: opaque to Dynamo
def count_unique_id_tuples(sem_ids: Tensor, codebook_size: int) -> Tensor:
    """#distinct rows of a [B,L] id table as a 0-d DEVICE tensor (no host sync in the training step).  Equals the reference's
    [B,B,L] triangular compare (rqvae.py:159-167: rows with no later duplicate) without the O(B^2) memory: the direct-table
    dedup kernel counts the groups (ops.sid_dedup_rank); key spaces beyond 2^26 sort the packed keys on the device."""
    if sem_ids.is_cuda:
        res = ops.sid_dedup_rank(sem_ids, codebook_size)
        if res is not None:
            return res[1]["n_unique"]
    L = sem_ids.shape[1]
    if codebook_size ** L < 2 ** 62:
        key = sem_ids[:, 0].clone()
        for l in range(1, L):
            key = key * codebook_size + sem_ids[:, l]
        skey = torch.sort(key).values
        return (skey[1:] != skey[:-1]).sum() + 1 if len(skey) else torch.zeros((), dtype=torch.int64, device=sem_ids.device)
    return torch.as_tensor(torch.unique(sem_ids, dim=0).shape[0], device=sem_ids.device)


class RqVae(nn.Module, PyTorchModelHubMixin):
    def __init__(
        self,
        input_dim: int,
        embed_dim: int,
        hidden_dims: List[int],
        codebook_size: int,
        codebook_kmeans_init: bool = True,
        codebook_normalize: bool = False,
        codebook_sim_vq: bool = False,
        codebook_mode: QuantizeForwardMode = QuantizeForwardMode.GUMBEL_SOFTMAX,
        n_layers: int = 3,
        commitment_weight: float = 0.25,
        n_cat_features: int = 18,
    ) -> None:
        self._config = locals()

        super().__init__()

        self.input_dim = input_dim
        self.embed_dim = embed_dim
        self.hidden_dims = hidden_dims
        self.n_layers = n_layers
        self.codebook_size = codebook_size
        self.commitment_weight = commitment_weight
        self.n_cat_feats = n_cat_features

        self.layers = nn.ModuleList(
            modules=[
                Quantize(
                    embed_dim=embed_dim,
                    n_embed=codebook_size,
                    forward_mode=codebook_mode,
                    do_kmeans_init=codebook_kmeans_init,
                    codebook_normalize=i == 0 and codebook_normalize,
                    sim_vq=codebook_sim_vq,
                    commitment_weight=commitment_weight,
                )
                for i in range(n_layers)
            ]
        )

        self.encoder = MLP(
            input_dim=input_dim,
            hidden_dims=hidden_dims,
            out_dim=embed_dim,
            normalize=codebook_normalize,
        )

        self.decoder = MLP(
            input_dim=embed_dim,
            hidden_dims=hidden_dims[-1::-1],
            out_dim=input_dim,
            normalize=False,
        )

        self.reconstruction_loss = (
            CategoricalReconstuctionLoss(n_cat_features)
            if n_cat_features != 0
            else ReconstructionLoss()
        )

    @cached_property
    def config(self) -> dict:
        return self._config

    @property
    def device(self) -> torch.device:
        return next(self.encoder.parameters()).device

    def load_pretrained(self, path: str) -> None:
        state = torch.load(path, map_location=self.device, weights_only=False)
        self.load_state_dict(state["model"])
        print(f"---Loaded RQVAE Iter {state['iter']}---")

    def encode(self, x: Tensor) -> Tensor:
        return self.encoder(x)

    def decode(self, x: Tensor) -> Tensor:
        return self.decoder(x)

    # ------------------------------------------------------------------ fused chain
    def _fusable(self) -> bool:
        """All levels can go through one launch: no pending k-means init, no Gumbel training level, same mode."""
        modes = {layer.kernel_mode() for layer in self.layers}
        pending_init = any(l.do_kmeans_init and not l.kmeans_initted for l in self.layers)
        betas = {l.quantize_loss.commitment_weight for l in self.layers}
        return (not pending_init and len(modes) == 1 and ops.MODE_GUMBEL not in modes and len(betas) == 1
                and len(self.layers) <= 8)

    def _chain(self, res: Tensor, gumbel_t: float, lean: bool):
        if torch.compiler.is_compiling():
            # inside torch.compile (the reference compiles forward, rqvae.py:141): the kernels are custom-operator nodes of the
            # captured graph (library.py); everything else in here is plain torch and Python that Dynamo traces
            from .. import library
            if self._fusable():
                mode = self.layers[0].kernel_mode()
                beta = self.layers[0].quantize_loss.commitment_weight
                return library.rq_chain(res, mode, beta, lean, [layer.codebook() for layer in self.layers])
            return self._chain_levels(res, gumbel_t, lean)
        return self._chain_eager(res, gumbel_t, lean)

    @torch.compiler.disable      # librqb200 is called through ctypes: opaque to Dynamo
    def _chain_eager(self, res: Tensor, gumbel_t: float, lean: bool):
        if self._fusable():
            mode = self.layers[0].kernel_mode()
            beta = self.layers[0].quantize_loss.commitment_weight
            codebooks = [layer.codebook() for layer in self.layers]
            return ops.RqChainFunction.apply(res, mode, beta, lean, *codebooks)
        return self._chain_levels(res, gumbel_t, lean)

    def _chain_levels(self, res: Tensor, gumbel_t: float, lean: bool):
        # level-by-level (first call with k-means init pending, or GUMBEL_SOFTMAX training): rqvae.py:122-132
        quantize_loss = 0
        embs, residuals, sem_ids = [], [], []
        for layer in self.layers:
            residuals.append(res)
            quantized = layer(res, temperature=gumbel_t)
            quantize_loss = quantize_loss + quantized.loss
            emb, id = quantized.embeddings, quantized.ids
            res = res - emb
            sem_ids.append(id)
            embs.append(emb)
        ids = torch.stack(sem_ids, dim=1)
        if lean:
            e = torch.stack(embs, dim=0)
            return e.sum(dim=0), e.detach().norm(dim=2).transpose(0, 1), ids, quantize_loss
        return torch.stack(embs, dim=0), torch.stack(residuals, dim=0), ids, quantize_loss

    def get_semantic_ids(self, x: Tensor, gumbel_t: float = 0.001) -> RqVaeOutput:
        x = x.to(next(self.encoder.parameters()).dtype)
        res = self.encode(x)
        embs, residuals, sem_ids, quantize_loss = self._chain(res, gumbel_t, lean=False)
        return RqVaeOutput(
            embeddings=embs.permute(1, 2, 0),      # [B,D,L] view of the kernel's [L,B,D] (rqvae.py:135)
            residuals=residuals.permute(1, 2, 0),
            sem_ids=sem_ids,
            quantize_loss=quantize_loss,
        )

    @torch.compiler.disable
    @torch.no_grad()
    def tokenize(self, x: Tensor, mlp_precision: str = None) -> Tensor:
        """sem_ids [B,L] only: what SemanticIdTokenizer consumes (semids.py:125).  Large batches of a model whose codebook
        size is 256 m (m = 1..8) go through the wgmma candidate filter + exact re-rank (prepared codebook state cached on the
        codebooks' identity and version; the shipped D = 32 quantiser is zero-padded to 64), everything else through the exact
        CUDA-core kernel: ops.rq_tokenize_auto.
        ``mlp_precision="bf16"`` runs the encoder on the bf16 wgmma GEMMs (faster, NOT index-exact vs fp32)."""
        x = x.to(next(self.encoder.parameters()).dtype)
        if mlp_precision is not None:
            old, self.encoder.precision = self.encoder.precision, mlp_precision
            try:
                res = self.encode(x)
            finally:
                self.encoder.precision = old
        else:
            res = self.encode(x)
        return ops.rq_tokenize_auto(res, [layer.codebook() for layer in self.layers])

    def forward(self, batch: SeqBatch, gumbel_t: float) -> RqVaeComputedLosses:
        x = batch.x
        xin = x.to(next(self.encoder.parameters()).dtype)
        res = self.encode(xin)
        emb_sum, embs_norm, sem_ids, rqvae_loss = self._chain(res, gumbel_t, lean=True)
        x_hat = self.decode(emb_sum)
        if self.n_cat_feats != 0:   # with n_cat_feats == 0 the reference's [:-0] slice is empty: no-op
            x_hat = torch.cat(
                [l2norm(x_hat[..., : -self.n_cat_feats]), x_hat[..., -self.n_cat_feats:]],
                axis=-1,
            )

        reconstuction_loss = self.reconstruction_loss(x_hat, x)
        loss = (reconstuction_loss + rqvae_loss).mean()

        with torch.no_grad():
            # Compute debug ID statistics
            if torch.compiler.is_compiling():
                from .. import library
                n_unique = library.count_unique_id_tuples(sem_ids, self.codebook_size)
            else:
                n_unique = count_unique_id_tuples(sem_ids, self.codebook_size)
            p_unique_ids = (n_unique / sem_ids.shape[0]).to(torch.float32)

        return RqVaeComputedLosses(
            loss=loss,
            reconstruction_loss=reconstuction_loss.mean(),
            rqvae_loss=rqvae_loss.mean(),
            embs_norm=embs_norm,
            p_unique_ids=p_unique_ids,
        )
