"""modules/encoder.py of the reference (:7-38): bias-free Linear+ReLU stack, optional final L2 norm.

The module tree (``self.mlp`` Sequential with Linear at indices 0,2,4,6) is kept so state-dict keys match the
shipped checkpoints; forward() bypasses it and runs the whole stack as one autograd node on the fp32 GEMM kernel
with the ReLU fused in its epilogue (ops.MLPFunction)."""
from typing import List

import torch
from torch import nn
from torch import Tensor

from .. import ops
from .normalize import L2NormalizationLayer


class MLP(nn.Module):
    def __init__(self, input_dim: int, hidden_dims: List[int], out_dim: int, dropout: float = 0.0,
                 normalize: bool = False) -> None:
        super().__init__()
        self.input_dim = input_dim
        self.hidden_dims = hidden_dims
        self.out_dim = out_dim
        self.dropout = dropout
        self.normalize = normalize

        dims = [self.input_dim] + list(self.hidden_dims) + [self.out_dim]
        self.mlp = nn.Sequential()
        for i, (in_d, out_d) in enumerate(zip(dims[:-1], dims[1:])):
            self.mlp.append(nn.Linear(in_d, out_d, bias=False))
            if i != len(dims) - 2:
                self.mlp.append(nn.ReLU())
                if dropout != 0:
                    self.mlp.append(nn.Dropout(dropout))
        self.mlp.append(L2NormalizationLayer() if normalize else nn.Identity())

    # ---- default precision: fp32-accurate.  From ops.SPLIT_MIN_ROWS rows on every Linear (forward and dgrad) runs on the fp16
    # tensor cores as a split-precision GEMM (three wgmma products per k-step, as close to float64 as a plain fp32 GEMM:
    # csrc/gemm_tc.cu gs_gemm_kernel, tests/test_gpu_gemm_split.py); smaller batches use the CUDA-core SGEMM.
    # ---- reduced-precision path: bf16 wgmma GEMMs (gt_gemm_kernel).  Opt-in and forward-only: chosen when no
    # gradient is needed AND (self.precision == "bf16" OR a bf16 torch.autocast region is active -- the reference runs
    # these Linears in bf16 under accelerator.autocast(), train_rqvae.py:36,69).
    precision = "fp32"

    def _bf16_wanted(self, x: Tensor) -> bool:
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            return False
        want = self.precision == "bf16" or (torch.is_autocast_enabled() and torch.get_autocast_dtype("cuda") == torch.bfloat16)
        dims = [self.input_dim] + list(self.hidden_dims) + [self.out_dim]
        return bool(want) and x.is_cuda and ops.bf16_supported(dims)

    def _weight_images(self, weights):
        key = tuple((w.data_ptr(), w._version) for w in weights)
        cache = getattr(self, "_wimg_cache", None)
        if cache is None or cache[0] != key:
            images = [ops.to_bf16_image(w.detach()) for w in weights]
            cache = (key, images, ops.StreamBuild(*images))
            object.__setattr__(self, "_wimg_cache", cache)
        cache[2].ready()
        return cache[1]

    def forward(self, x: Tensor) -> Tensor:
        assert x.shape[-1] == self.input_dim, f"Invalid input dim: Expected {self.input_dim}, found {x.shape[-1]}"
        if torch.compiler.is_compiling() and self.precision == "fp32" and not (self.dropout != 0 and self.training):
            # inside torch.compile (the reference compiles RqVae.forward, rqvae.py:141): one custom-operator node, no graph break
            from .. import library
            weights = [m.weight for m in self.mlp if isinstance(m, nn.Linear)]
            norm = bool(getattr(self, "normalize", False)) or isinstance(self.mlp[-1], L2NormalizationLayer)
            return library.mlp(x.reshape(-1, self.input_dim), norm, weights).reshape(*x.shape[:-1], self.out_dim)
        return self._forward_eager(x)

    @torch.compiler.disable      # ctypes call into librqb200: opaque to Dynamo
    def _forward_eager(self, x: Tensor) -> Tensor:
        if self._bf16_wanted(x):
            weights = [m.weight for m in self.mlp if isinstance(m, nn.Linear)]
            lead = x.shape[:-1]
            y = ops.mlp_forward_bf16(x.reshape(-1, self.input_dim), weights,
                                     bool(getattr(self, "normalize", False)) or isinstance(self.mlp[-1], L2NormalizationLayer),
                                     weight_images=self._weight_images(weights))
            return y.reshape(*lead, self.out_dim)
        if self.dropout != 0 and self.training:
            raise NotImplementedError("MLP dropout > 0 in training is not built (no reference caller sets it)")
        weights = [m.weight for m in self.mlp if isinstance(m, nn.Linear)]
        lead = x.shape[:-1]
        y = ops.MLPFunction.apply(x.reshape(-1, self.input_dim), bool(getattr(self, "normalize", False)) or
                                  isinstance(self.mlp[-1], L2NormalizationLayer), *weights)
        return y.reshape(*lead, self.out_dim)
