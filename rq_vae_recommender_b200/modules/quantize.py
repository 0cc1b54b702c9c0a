"""modules/quantize.py of the reference (:16-163) on the fused sm_90a kernels.

Same public names, constructor signature, state-dict keys (``embedding.weight``, ``out_proj.0.weight``) and
forward contract ``Quantize.forward(x, temperature) -> QuantizeOutput(embeddings, ids, loss)``.
Eval / STE / ROTATION_TRICK levels run as a single-level call of the fused chain kernel (distance, first-index
argmin, gather, mode-specific output and QuantizeLoss in one launch); GUMBEL_SOFTMAX runs GEMM -> fused
noise+softmax -> GEMM.  ``RqVae`` chains all its levels in ONE launch instead of calling this per level."""
from enum import Enum
from typing import NamedTuple

import torch
from torch import nn
from torch import Tensor

try:  # gin-config is not in this image; the shim keeps `%modules.quantize.QuantizeForwardMode.X` macros working
    import gin
except ImportError:  # pragma: no cover
    from .. import gin_compat as gin

from .. import ops
from ..distributions import gumbel as _gumbel
from ..init.kmeans import kmeans_init_
from .loss import QuantizeLoss
from .normalize import L2NormalizationLayer


@gin.constants_from_enum
class QuantizeForwardMode(Enum):
    GUMBEL_SOFTMAX = 1
    STE = 2
    ROTATION_TRICK = 3


class QuantizeDistance(Enum):
    L2 = 1
    COSINE = 2


class QuantizeOutput(NamedTuple):
    embeddings: Tensor
    ids: Tensor
    loss: Tensor


_KERNEL_MODE = {QuantizeForwardMode.STE: ops.MODE_STE, QuantizeForwardMode.ROTATION_TRICK: ops.MODE_ROTATION}


def efficient_rotation_trick_transform(u, q, e):
    """4.2 in https://arxiv.org/abs/2410.06424 -- stand-alone API (reference quantize.py:34-50); the fused
    kernels evaluate the same expression in their epilogue."""
    w = torch.nn.functional.normalize(u + q, p=2, dim=1, eps=1e-6).detach()
    ew = (e * w).sum(dim=1, keepdim=True)
    eu = (e * u.detach()).sum(dim=1, keepdim=True)
    return (e - 2 * (ew * w) + 2 * (eu * q.detach())).squeeze()


class Quantize(nn.Module):
    def __init__(
        self,
        embed_dim: int,
        n_embed: int,
        do_kmeans_init: bool = True,
        codebook_normalize: bool = False,
        sim_vq: bool = False,  # https://arxiv.org/pdf/2411.02038
        commitment_weight: float = 0.25,
        forward_mode: QuantizeForwardMode = QuantizeForwardMode.GUMBEL_SOFTMAX,
        distance_mode: QuantizeDistance = QuantizeDistance.L2,
    ) -> None:
        super().__init__()

        self.embed_dim = embed_dim
        self.n_embed = n_embed
        self.embedding = nn.Embedding(n_embed, embed_dim)
        self.forward_mode = forward_mode
        self.distance_mode = distance_mode
        self.do_kmeans_init = do_kmeans_init
        self.kmeans_initted = False

        self.out_proj = nn.Sequential(
            nn.Linear(embed_dim, embed_dim, bias=False) if sim_vq else nn.Identity(),
            L2NormalizationLayer(dim=-1) if codebook_normalize else nn.Identity(),
        )

        self.quantize_loss = QuantizeLoss(commitment_weight)
        self._init_weights()

    @property
    def weight(self) -> Tensor:
        return self.embedding.weight

    @property
    def device(self) -> torch.device:
        return self.embedding.weight.device

    @property
    def commitment_weight(self) -> float:
        return self.quantize_loss.commitment_weight

    def _init_weights(self) -> None:
        for m in self.modules():
            if isinstance(m, nn.Embedding):
                nn.init.uniform_(m.weight)

    @torch.no_grad
    def _kmeans_init(self, x) -> None:
        kmeans_init_(self.embedding.weight, x=x)
        self.kmeans_initted = True

    def codebook(self) -> Tensor:
        """out_proj(embedding.weight) (reference quantize.py:110); plain weight when out_proj is the identity."""
        w = self.embedding.weight
        for m in self.out_proj:
            if isinstance(m, nn.Linear):
                if torch.compiler.is_compiling():
                    from .. import library
                    w = library.mlp(w, False, [m.weight])
                else:
                    w = ops.MLPFunction.apply(w, False, m.weight)
            elif not isinstance(m, nn.Identity):
                w = m(w)
        return w

    def get_item_embeddings(self, item_ids) -> Tensor:
        return self.codebook()[item_ids] if not self._plain() else self.embedding(item_ids)

    def _plain(self) -> bool:
        return all(isinstance(m, nn.Identity) for m in self.out_proj)

    def kernel_mode(self) -> int:
        """Mode id of the fused kernels for the CURRENT train/eval state (GUMBEL has no fused-chain mode)."""
        if not self.training:
            return ops.MODE_EVAL
        if self.forward_mode == QuantizeForwardMode.GUMBEL_SOFTMAX:
            return ops.MODE_GUMBEL
        if self.forward_mode in _KERNEL_MODE:
            return _KERNEL_MODE[self.forward_mode]
        raise Exception("Unsupported Quantize forward mode.")

    def forward(self, x, temperature) -> QuantizeOutput:
        if (torch.compiler.is_compiling() and not (self.do_kmeans_init and not self.kmeans_initted)
                and self.distance_mode == QuantizeDistance.L2):
            # inside torch.compile: the level is one custom-operator node (library.py); the lazy k-means init is data dependent
            # (host-side convergence check) and stays a graph break on the one call that runs it
            from .. import library
            codebook = self.codebook()
            mode = self.kernel_mode()
            beta = self.quantize_loss.commitment_weight
            if mode == ops.MODE_GUMBEL:
                uniform = _gumbel.draw_uniform((x.shape[0], self.n_embed), self.device)
                emb_out, ids, loss = library.gumbel_level(x, codebook, uniform, temperature, beta)
            else:
                embs, _res, ids, loss = library.rq_chain(x, mode, beta, False, [codebook])
                emb_out, ids = embs[0], ids[:, 0]
            return QuantizeOutput(embeddings=emb_out, ids=ids, loss=loss)
        return self._forward_eager(x, temperature)

    @torch.compiler.disable      # ctypes call into librqb200: opaque to Dynamo
    def _forward_eager(self, x, temperature) -> QuantizeOutput:
        assert x.shape[-1] == self.embed_dim

        if self.do_kmeans_init and not self.kmeans_initted:
            self._kmeans_init(x=x)

        if self.distance_mode != QuantizeDistance.L2:
            if self.distance_mode == QuantizeDistance.COSINE:
                raise NotImplementedError("QuantizeDistance.COSINE is never selected by a reference caller "
                                          " and is not built")
            raise Exception("Unsupported Quantize distance mode.")

        codebook = self.codebook()
        mode = self.kernel_mode()
        beta = self.quantize_loss.commitment_weight

        if mode == ops.MODE_GUMBEL:
            uniform = _gumbel.draw_uniform((x.shape[0], self.n_embed), self.device)
            emb_out, ids, loss = ops.GumbelQuantizeFunction.apply(x, codebook, uniform, temperature, beta)
        else:
            embs, _res, ids, loss = ops.RqChainFunction.apply(x, mode, beta, False, codebook)
            emb_out, ids = embs[0], ids[:, 0]

        return QuantizeOutput(embeddings=emb_out, ids=ids, loss=loss)
