"""H100-native RQ-VAE residual-quantisation hot path behind the reference's module API.

Layout (only what the path needs):
  csrc/            hand-written sm_90a CUDA kernels + the C ABI (include/rqb200.h) -> librqb200.so
  _lib.py          ctypes binding (fails loudly when the library is missing -- no fallback)
  ops.py           torch.Tensor <-> C ABI marshalling, autograd Functions
  modules/ init/ distributions/ data/ evaluate/   mirrors of the reference modules with identical public names
  parallel.py      item-sharded tokenisation + all-reduced k-means over torch.distributed (NCCL / gloo)
  dropin.py        makes the UNMODIFIED reference train_rqvae.py / train_decoder.py import these modules
"""
__version__ = "0.1.0"
