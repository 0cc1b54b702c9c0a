"""torch.Tensor <-> librqb200 C-ABI marshalling and the autograd Functions built on it.

PyTorch is plumbing here: it owns device memory, streams and the autograd tape; every FLOP of the hot path
runs in the hand-written kernels of csrc/.  CUDA tensors only -- CPU tensors raise (no fallback).
"""
from __future__ import annotations

import ctypes
import weakref
from typing import List, NamedTuple, Optional, Sequence, Tuple

import torch

from . import _lib

MODE_EVAL, MODE_GUMBEL, MODE_STE, MODE_ROTATION = 0, 1, 2, 3

#: count of librqb200 kernel launches issued through this module (bench.py reports it as `gpu_launches`)
LAUNCHES = 0
#: calls of the tensor-core tokeniser / prepared-state builds (tests assert the module API really routes there)
TC_CALLS = 0
TC_PREPARES = 0


def _count(n: int) -> None:
    global LAUNCHES
    LAUNCHES += n


def _p(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _live(live: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """A device-counted launch's live count: an int32 CUDA tensor whose first entry the kernels read (None: host-counted)."""
    if live is not None and (live.dtype != torch.int32 or not live.is_cuda or live.numel() < 1 or not live.is_contiguous()):
        raise ValueError("live must be a contiguous int32 CUDA tensor")
    return live


def _need_cuda(*ts) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.Rqb200Error("rq_vae_recommender_b200 runs on CUDA tensors only (no CPU fallback); got a "
                                   f"{t.device} tensor")


def _f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def _rows(t: torch.Tensor) -> torch.Tensor:
    """fp32 2-D tensor whose last dim is unit-stride (row stride may exceed the width)."""
    if t.dtype != torch.float32:
        t = t.float()
    if t.dim() != 2:
        raise ValueError(f"expected a 2-D tensor, got {tuple(t.shape)}")
    if t.stride(1) != 1 or t.stride(0) < t.shape[1]:
        t = t.contiguous()
    return t


def _ptr_array(ts: Sequence[Optional[torch.Tensor]]):
    arr = (ctypes.c_void_p * len(ts))()
    for i, t in enumerate(ts):
        arr[i] = _p(t)
    return arr


class StreamBuild:
    """The build of cached device state (prepared codebooks, operand images, tries, item tables): kernels enqueued on the stream
    current at construction, with no host sync.  Later calls reuse the state from whatever stream is current then, so each reuse
    goes through ``ready()``: it orders the current stream after the build (an event wait, no host sync; nothing on the build
    stream or on a stream that already waited) and marks the state's tensors as used on that stream, so that freeing them -- a
    cache evicting the entry -- also waits for the work that stream has queued.  Inside a CUDA-graph capture it does nothing:
    capture starts from a synchronised device, and the caches rebuild their entries in a captured stream anyway."""

    __slots__ = ("tensors", "event", "streams")

    def __init__(self, *tensors: torch.Tensor):
        stream = torch.cuda.current_stream(tensors[0].device)
        self.tensors = tensors
        self.event = torch.cuda.Event()
        self.event.record(stream)
        self.streams = {stream.cuda_stream}

    def ready(self) -> None:
        stream = torch.cuda.current_stream(self.tensors[0].device)
        # streams are told apart by their handle: torch's pooled streams live as long as the process, but a destroyed external
        # stream whose handle the driver hands out again would be taken for the one that waited; and the capture check is that of
        # the current device's stream, the one the library's launches go to
        if stream.cuda_stream in self.streams or torch.cuda.is_current_stream_capturing():
            return
        stream.wait_event(self.event)
        for t in self.tensors:
            t.record_stream(stream)
        self.streams.add(stream.cuda_stream)


def _check_codebooks(cbs: Sequence[torch.Tensor], D: int) -> List[torch.Tensor]:
    out = [_f32c(c) for c in cbs]
    K = out[0].shape[0]
    for c in out:
        if c.shape != (K, D):
            raise ValueError(f"codebook shape {tuple(c.shape)} != ({K}, {D})")
    return out


# ---------------------------------------------------------------------------------------------- fused RQ chain
def rq_forward(x: torch.Tensor, codebooks: Sequence[torch.Tensor], mode: int, beta: float, *,
               want_ids=True, want_embeddings=False, want_residuals=False, want_sum=False, want_norms=False,
               want_loss=False):
    """All L Quantize levels in one launch (csrc/rq_simt.cu).  Returns a dict of the requested outputs;
    embeddings / residuals come back as [L,B,D] (permute to the reference's [B,D,L] is a view)."""
    _need_cuda(x, *codebooks)
    lib = _lib.load()
    x = _rows(x)
    B, D = x.shape
    cbs = _check_codebooks(codebooks, D)
    K, L = cbs[0].shape[0], len(cbs)
    dev = x.device
    out = {}
    ids = torch.empty((B, L), dtype=torch.int64, device=dev) if want_ids else None
    emb = torch.empty((L, B, D), dtype=torch.float32, device=dev) if want_embeddings else None
    res = torch.empty((L, B, D), dtype=torch.float32, device=dev) if want_residuals else None
    esum = torch.empty((B, D), dtype=torch.float32, device=dev) if want_sum else None
    norms = torch.empty((B, L), dtype=torch.float32, device=dev) if want_norms else None
    loss = torch.empty((B,), dtype=torch.float32, device=dev) if want_loss else None
    if (B >= TC_MIN_ROWS and tc_padded_dim(D, K, L)
            and (want_embeddings or want_residuals or want_sum or want_norms or want_loss)):
        # large batch: ids from the tensor-core tokeniser (those of the exact kernel), everything else from the streaming
        # pass over the given ids -- same outputs bit for bit, HBM-bound instead of CUDA-core-FLOP-bound
        tids = rq_tokenize_tc(x, state=tc_state_for(cbs))
        with torch.cuda.device(dev):
            _lib.check(lib.rqb200_rq_forward_from_ids(mode, _p(x), x.stride(0), _ptr_array(cbs), _p(tids), B, D, K, L,
                                                      float(beta), _p(emb), _p(res), _p(esum), _p(norms), _p(loss), _stream()),
                       "rq_forward_from_ids")
        _count(1)
        out.update(ids=tids if want_ids else None, embeddings=emb, residuals=res, emb_sum=esum, emb_norms=norms, loss=loss)
        return out
    ws_bytes = lib.rqb200_rq_workspace_bytes(D, K, L)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.rqb200_rq_forward(mode, _p(x), x.stride(0), _ptr_array(cbs), B, D, K, L, float(beta),
                                         _p(ids), _p(emb), _p(res), _p(esum), _p(norms), _p(loss),
                                         _p(ws), ws_bytes, _stream()), "rq_forward")
    _count(3)
    out.update(ids=ids, embeddings=emb, residuals=res, emb_sum=esum, emb_norms=norms, loss=loss)
    return out


def rq_tokenize(x: torch.Tensor, codebooks: Sequence[torch.Tensor]) -> torch.Tensor:
    """sem_ids [B,L] int64 -- eval-mode hard argmin chain, exact fp32 kernel."""
    return rq_forward(x, codebooks, MODE_EVAL, 0.0, want_ids=True)["ids"]


class RqChainFunction(torch.autograd.Function):
    """Differentiable fused chain (eval / STE / rotation-trick).

    lean=True  -> (emb_sum [B,D], emb_norms [B,L], ids [B,L], loss [B])     what RqVae.forward consumes
    lean=False -> (embeddings [L,B,D], residuals [L,B,D], ids [B,L], loss [B])   what get_semantic_ids returns
    """

    @staticmethod
    def forward(ctx, x, mode, beta, lean, *codebooks):
        xr = _rows(x)
        cbs = _check_codebooks(codebooks, xr.shape[1])
        o = rq_forward(xr, cbs, mode, beta, want_ids=True, want_embeddings=not lean, want_residuals=not lean,
                       want_sum=lean, want_norms=lean, want_loss=True)
        ctx.mode, ctx.beta, ctx.lean = mode, beta, lean
        ctx.save_for_backward(xr, o["ids"], *cbs)
        ctx.mark_non_differentiable(o["ids"])
        if lean:
            ctx.mark_non_differentiable(o["emb_norms"])
            return o["emb_sum"], o["emb_norms"], o["ids"], o["loss"]
        return o["embeddings"], o["residuals"], o["ids"], o["loss"]

    @staticmethod
    def backward(ctx, g_a, g_b, _g_ids, g_loss):
        xr, ids, *cbs = ctx.saved_tensors
        lib = _lib.load()
        B, D = xr.shape
        K, L = cbs[0].shape[0], len(cbs)
        dev = xr.device

        def f32(g):
            return None if g is None else (g if g.dtype == torch.float32 else g.float())

        g_a, g_loss = f32(g_a), f32(g_loss)
        if ctx.lean:
            g_emb, g_res = g_a, None
            ge = (g_emb.stride(0), g_emb.stride(1), 0) if g_emb is not None else (0, 0, 0)
            gr = (0, 0, 0)
        else:
            g_emb, g_res = g_a, f32(g_b)
            ge = (g_emb.stride(1), g_emb.stride(2), g_emb.stride(0)) if g_emb is not None else (0, 0, 0)
            gr = (g_res.stride(1), g_res.stride(2), g_res.stride(0)) if g_res is not None else (0, 0, 0)
        g_x = torch.empty((B, D), dtype=torch.float32, device=dev)
        need_cb = [ctx.needs_input_grad[4 + l] for l in range(L)]
        g_cbs = [torch.zeros_like(c) if n else None for c, n in zip(cbs, need_cb)]
        with torch.cuda.device(dev):
            _lib.check(lib.rqb200_rq_backward(ctx.mode, _p(xr), xr.stride(0), _ptr_array(cbs), _p(ids), B, D, K, L,
                                              float(ctx.beta), _p(g_emb), *ge, _p(g_res), *gr, _p(g_loss),
                                              g_loss.stride(0) if g_loss is not None else 0, _p(g_x),
                                              _ptr_array(g_cbs), _stream()), "rq_backward")
        _count(1)
        return (g_x if ctx.needs_input_grad[0] else None, None, None, None, *g_cbs)


# ---------------------------------------------------------------------------------------------- dense helpers
def sgemm(a: torch.Tensor, b: torch.Tensor, *, trans_a=False, trans_b=False, relu=False,
          mask: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, alpha=1.0, beta=0.0):
    """out = epi(alpha * op(a) @ op(b) + beta*out) with the fp32 CUDA-core GEMM of csrc/dense.cu."""
    lib = _lib.load()
    a, b = _rows(a), _rows(b)
    M, Ka = (a.shape[1], a.shape[0]) if trans_a else a.shape
    Kb, N = (b.shape[1], b.shape[0]) if trans_b else b.shape
    if Ka != Kb:
        raise ValueError(f"sgemm inner dims differ: {Ka} vs {Kb}")
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    if mask is not None:
        mask = _rows(mask)
    with torch.cuda.device(a.device):
        _lib.check(lib.rqb200_sgemm(int(trans_a), int(trans_b), M, N, Ka, float(alpha), _p(a), a.stride(0), _p(b),
                                    b.stride(0), float(beta), _p(out), out.stride(0), int(relu), _p(mask),
                                    mask.stride(0) if mask is not None else 0, _stream()), "sgemm")
    _count(1)
    return out


# ---------------------------------------------------------------------------------------------- split-precision tensor-core GEMM
#: rows of the A operand from which the dense GEMMs of the MLPs / the Gumbel level run on the tensor cores (three fp16
#: products per k-step, fp32-accurate: csrc/gemm_tc.cu); below it one launch of the CUDA-core SGEMM is as fast
SPLIT_MIN_ROWS = 512
SPLIT_CALLS = 0


class SplitOperand:
    """One GEMM operand [rows, K] as hi + lo fp16 images with power-of-two row scales (rqb200_f32_to_split_image).
    ``transposed=True`` builds the operand of t.T without materialising the transpose.  ``live`` (int32 on the device; row-major
    only, rqb200_f32_to_split_image_counted): t's rows are a capacity and only the first live[0] are converted."""

    def __init__(self, t: torch.Tensor, transposed: bool = False, live: Optional[torch.Tensor] = None):
        _need_cuda(t)
        lib = _lib.load()
        t = _rows(t.detach())
        self.rows, self.K = (t.shape[1], t.shape[0]) if transposed else (t.shape[0], t.shape[1])
        self.device = t.device
        nbytes = lib.rqb200_split_image_bytes(self.rows, self.K)
        self.buf = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=t.device)
        with torch.cuda.device(t.device):
            if live is None:
                _lib.check(lib.rqb200_f32_to_split_image(_p(t), t.stride(0), self.rows, self.K, int(transposed), _p(self.buf),
                                                         _stream()), "f32_to_split_image")
            else:
                if transposed:
                    raise ValueError("SplitOperand: a device row count needs a row-major operand")
                _lib.check(lib.rqb200_f32_to_split_image_counted(_p(t), t.stride(0), self.rows, self.K, _p(_live(live)),
                                                                 _p(self.buf), _stream()), "f32_to_split_image_counted")
        _count(1)


# operands that do not change between calls (weights, codebooks): keyed on identity AND version like the tokeniser state
_SPLIT_CACHE: "dict[tuple, tuple]" = {}
_SPLIT_CACHE_MAX = 32


_NO_OPERAND_CACHE = 0


class no_operand_cache:
    """Inside this context prepared operands are rebuilt on every use and never stored.  The torch.library operators run under
    it: a compiled caller (mode="reduce-overhead") executes them inside a CUDA-graph memory pool -- warm-up run included -- where
    a cached buffer would be an allocation the graph does not own, and a replay must see the weights of that moment."""

    def __enter__(self):
        global _NO_OPERAND_CACHE
        _NO_OPERAND_CACHE += 1

    def __exit__(self, *a):
        global _NO_OPERAND_CACHE
        _NO_OPERAND_CACHE -= 1


def split_operand_cached(t: torch.Tensor, transposed: bool = False) -> SplitOperand:
    # the entry remembers the tensor OBJECT (weak reference): a temporary that died and whose address the allocator handed to
    # another tensor of the same shape must not hit
    if _NO_OPERAND_CACHE or torch.cuda.is_current_stream_capturing():
        return SplitOperand(t, transposed)       # inside a CUDA-graph capture the split kernel must be PART of the graph (replays
                                                 # see the weights of that moment, not the images of capture time)
    key = (t.data_ptr(), t._version, tuple(t.shape), tuple(t.stride()), t.device.index, bool(transposed))
    hit = _SPLIT_CACHE.get(key)
    if hit is not None and hit[0]() is t:
        hit[2].ready()
        return hit[1]
    if len(_SPLIT_CACHE) >= _SPLIT_CACHE_MAX:
        _SPLIT_CACHE.pop(next(iter(_SPLIT_CACHE)))
    op = SplitOperand(t, transposed)
    _SPLIT_CACHE[key] = (weakref.ref(t), op, StreamBuild(op.buf))
    return op


def gemm_split(a, b, *, relu: bool = False, mask: Optional[torch.Tensor] = None,
               out: Optional[torch.Tensor] = None, live: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[M, N] = act(A[M, K] @ B[N, K]^T) on the fp16 tensor cores with fp32 accuracy; a, b: SplitOperand or fp32 tensor.
    ``live`` (int32 on the device, rqb200_gemm_split_counted): M is a capacity and only rows below live[0] are computed and
    written (a tensor ``a`` is converted with the same count)."""
    global SPLIT_CALLS
    lib = _lib.load()
    if not isinstance(a, SplitOperand):
        a = SplitOperand(a, live=live)
    if not isinstance(b, SplitOperand):
        b = SplitOperand(b)
    if a.K != b.K:
        raise ValueError(f"gemm_split inner dims differ: {a.K} vs {b.K}")
    M, N = a.rows, b.rows
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    if mask is not None:
        mask = _rows(mask)
    with torch.cuda.device(a.device):
        if live is None:
            _lib.check(lib.rqb200_gemm_split(_p(a.buf), _p(b.buf), M, N, a.K, int(relu), _p(mask),
                                             mask.stride(0) if mask is not None else 0, _p(out), out.stride(0), _stream()),
                       "gemm_split")
        else:
            _lib.check(lib.rqb200_gemm_split_counted(_p(a.buf), _p(b.buf), M, N, a.K, int(relu), _p(mask),
                                                     mask.stride(0) if mask is not None else 0, _p(_live(live)), _p(out),
                                                     out.stride(0), _stream()), "gemm_split_counted")
    _count(1)
    SPLIT_CALLS += 1
    return out


def gemm_tn(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a^T @ b for a [B, M], b [B, N]: the contraction runs over the (long) batch dimension -- weight / codebook gradients.
    Tensor cores with a split-K schedule from SPLIT_MIN_ROWS batch rows on (both operands are split transposed, partial sums are
    reduced in a fixed order), the CUDA-core SGEMM below."""
    global SPLIT_CALLS
    B = a.shape[0]
    if B < SPLIT_MIN_ROWS:
        return sgemm(a, b, trans_a=True)
    lib = _lib.load()
    ao, bo = SplitOperand(a, transposed=True), SplitOperand(b, transposed=True)
    M, N = ao.rows, bo.rows
    out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        slices = lib.rqb200_gemm_split_k_slices(M, N, B)
        ws = torch.empty((slices, M, N), dtype=torch.float32, device=a.device) if slices > 1 else None
        _lib.check(lib.rqb200_gemm_split_k(_p(ao.buf), _p(bo.buf), M, N, B, slices, _p(ws), _p(out), out.stride(0), _stream()),
                   "gemm_split_k")
    _count(2 if slices > 1 else 1)
    SPLIT_CALLS += 1
    return out


def linear_nt(a: torch.Tensor, w: torch.Tensor, *, relu: bool = False, mask: Optional[torch.Tensor] = None,
              w_transposed: bool = False) -> torch.Tensor:
    """a[M, K] @ op(w)^T with a static second operand (weight / codebook): op(w) = w [N, K], or w^T for w [K, N] when
    ``w_transposed``.  Tensor cores from SPLIT_MIN_ROWS rows on, the CUDA-core SGEMM below (same result to ~1e-7)."""
    if a.shape[0] >= SPLIT_MIN_ROWS:
        return gemm_split(a, split_operand_cached(w, transposed=w_transposed), relu=relu, mask=mask)
    return sgemm(a, w, trans_b=not w_transposed, relu=relu, mask=mask)


class MLPFunction(torch.autograd.Function):
    """modules/encoder.py:23-38 as one autograd node: bias-free Linear+ReLU stack (ReLU fused in the GEMM
    epilogue), optional final L2 normalisation (modules/normalize.py)."""

    @staticmethod
    def forward(ctx, x, normalize, *weights):
        _need_cuda(x, *weights)
        lib = _lib.load()
        h = _rows(x)
        ws = [_f32c(w) for w in weights]
        acts = [h]
        n = len(ws)
        for i, w in enumerate(ws):
            h = linear_nt(h, w, relu=(i != n - 1))
            acts.append(h)
        norms = None
        if normalize:
            y = torch.empty_like(h)
            norms = torch.empty(h.shape[0], dtype=torch.float32, device=h.device)
            with torch.cuda.device(h.device):
                _lib.check(lib.rqb200_l2norm_fwd(_p(h), _p(y), _p(norms), h.shape[0], h.shape[1], 1e-12, _stream()),
                           "l2norm_fwd")
            _count(1)
            acts.append(y)
            h = y
        ctx.normalize = normalize
        ctx.n = n
        ctx.save_for_backward(*acts, *ws, *([norms] if normalize else []))
        return h

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        n = ctx.n
        saved = ctx.saved_tensors
        n_act = n + 1 + (1 if ctx.normalize else 0)
        acts, ws = saved[:n_act], saved[n_act:n_act + n]
        g = _f32c(g)
        if ctx.normalize:
            norms, y = saved[-1], acts[-1]
            gx = torch.empty_like(g)
            with torch.cuda.device(g.device):
                _lib.check(lib.rqb200_l2norm_bwd(_p(g), _p(y), _p(norms), _p(gx), g.shape[0], g.shape[1], 1e-12,
                                                 _stream()), "l2norm_bwd")
            _count(1)
            g = gx
        g_ws = [None] * n
        for i in range(n - 1, -1, -1):
            h_in = acts[i]
            if ctx.needs_input_grad[2 + i]:
                g_ws[i] = gemm_tn(g, h_in)                                 # [out,B] @ [B,in]
            if i > 0 or ctx.needs_input_grad[0]:
                g = linear_nt(g, ws[i], mask=h_in if i > 0 else None, w_transposed=True)   # [B,out] @ [out,in], ReLU' of layer i-1
        return (g if ctx.needs_input_grad[0] else None, None, *g_ws)


def l2norm_rows(x: torch.Tensor, eps: float = 1e-12) -> torch.Tensor:
    """F.normalize(x, p=2, dim=-1) forward only (no autograd)."""
    lib = _lib.load()
    shp = x.shape
    x2 = _f32c(x.reshape(-1, shp[-1]))
    y = torch.empty_like(x2)
    with torch.cuda.device(x2.device):
        _lib.check(lib.rqb200_l2norm_fwd(_p(x2), _p(y), 0, x2.shape[0], x2.shape[1], float(eps), _stream()), "l2norm")
    _count(1)
    return y.reshape(shp)


class L2NormFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, eps):
        lib = _lib.load()
        shp = x.shape
        x2 = _f32c(x.reshape(-1, shp[-1]))
        y = torch.empty_like(x2)
        norms = torch.empty(x2.shape[0], dtype=torch.float32, device=x2.device)
        with torch.cuda.device(x2.device):
            _lib.check(lib.rqb200_l2norm_fwd(_p(x2), _p(y), _p(norms), x2.shape[0], x2.shape[1], float(eps), _stream()),
                       "l2norm_fwd")
        _count(1)
        ctx.eps, ctx.shp = eps, shp
        ctx.save_for_backward(y, norms)
        return y.reshape(shp)

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        y, norms = ctx.saved_tensors
        g2 = _f32c(g.reshape(y.shape))
        gx = torch.empty_like(g2)
        with torch.cuda.device(g2.device):
            _lib.check(lib.rqb200_l2norm_bwd(_p(g2), _p(y), _p(norms), _p(gx), y.shape[0], y.shape[1], float(ctx.eps),
                                             _stream()), "l2norm_bwd")
        _count(1)
        return gx.reshape(ctx.shp), None


# ---------------------------------------------------------------------------------------------- Gumbel-softmax level
class GumbelQuantizeFunction(torch.autograd.Function):
    """One training-mode GUMBEL_SOFTMAX Quantize level (modules/quantize.py:113-136,157): returns
    (emb [B,D], ids [B], loss [B]).  The uniform draw U is an input (the caller draws it with torch.rand on the
    device, exactly where distributions/gumbel.py:10 does)."""

    @staticmethod
    def forward(ctx, x, codebook, uniform, temperature, beta):
        _need_cuda(x, codebook, uniform)
        lib = _lib.load()
        x, cb, u = _rows(x), _f32c(codebook), _f32c(uniform)
        B, D = x.shape
        K = cb.shape[0]
        dev = x.device
        cc = torch.empty(K, dtype=torch.float32, device=dev)
        ids = torch.empty(B, dtype=torch.int64, device=dev)
        loss = torch.empty(B, dtype=torch.float32, device=dev)
        w = torch.empty((B, K), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            st = _stream()
            _lib.check(lib.rqb200_row_sqnorm(_p(cb), K, D, _p(cc), st), "row_sqnorm")
            dist = linear_nt(x, cb)                                              # x @ C^T
            _lib.check(lib.rqb200_dist_finish(_p(dist), _p(x), x.stride(0), _p(cc), B, D, K, _p(ids), st), "dist")
            _lib.check(lib.rqb200_gumbel_softmax_fwd(_p(dist), _p(u), _p(w), B, K, float(temperature), st), "softmax")
            emb = linear_nt(w, cb, w_transposed=True)                            # W @ C   (quantize.py:135)
            _lib.check(lib.rqb200_gumbel_row_finish(_p(x), x.stride(0), _p(emb), B, D, float(beta), _p(loss), st),
                       "row_finish")
        _count(4)
        ctx.temperature, ctx.beta = float(temperature), float(beta)
        ctx.save_for_backward(x, cb, w, emb)
        ctx.mark_non_differentiable(ids)
        return emb, ids, loss

    @staticmethod
    def backward(ctx, g_emb, _g_ids, g_loss):
        lib = _lib.load()
        x, cb, w, emb = ctx.saved_tensors
        B, D = x.shape
        K = cb.shape[0]
        dev = x.device
        g_emb = None if g_emb is None else (g_emb if g_emb.dtype == torch.float32 else g_emb.float())
        g_loss = None if g_loss is None else (g_loss if g_loss.dtype == torch.float32 else g_loss.float())
        gl_s = g_loss.stride(0) if g_loss is not None else 0
        gE = torch.empty((B, D), dtype=torch.float32, device=dev)
        rowsum = torch.empty(B, dtype=torch.float32, device=dev)
        colsum = torch.empty(K, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            st = _stream()
            _lib.check(lib.rqb200_gumbel_bwd_ge(_p(g_emb), g_emb.stride(0) if g_emb is not None else 0,
                                                g_emb.stride(1) if g_emb is not None else 0, _p(g_loss), gl_s,
                                                _p(x), x.stride(0), _p(emb), _p(gE), B, D, st), "bwd_ge")
            gw = linear_nt(gE, cb)                                               # gW = gE @ C^T   [B,K]
            _lib.check(lib.rqb200_gumbel_bwd_softmax(_p(w), _p(gw), B, K, ctx.temperature, _p(rowsum), _p(colsum), st),
                       "bwd_softmax")                                            # gw now holds gdist
            gx = linear_nt(gw, cb, w_transposed=True)                            # gdist @ C       [B,D]
            _lib.check(lib.rqb200_gumbel_bwd_gx(_p(gx), _p(x), x.stride(0), _p(emb), _p(g_loss), gl_s, _p(rowsum),
                                                ctx.beta, B, D, st), "bwd_gx")
            gc = None
            if ctx.needs_input_grad[1]:
                if B >= SPLIT_MIN_ROWS:
                    gc = gemm_tn(w, gE)                                          # W^T @ gE        [K,D]
                    gc.add_(gemm_tn(gw, x), alpha=-2.0)                          # - 2 gdist^T @ x
                else:
                    gc = sgemm(w, gE, trans_a=True)
                    sgemm(gw, x, trans_a=True, out=gc, alpha=-2.0, beta=1.0)
                _lib.check(lib.rqb200_gumbel_bwd_gc(_p(gc), _p(cb), _p(colsum), K, D, st), "bwd_gc")
        _count(5)
        return (gx if ctx.needs_input_grad[0] else None, gc, None, None, None)


# ---------------------------------------------------------------------------------------------- k-means
def kmeans_workspace(x: torch.Tensor, K: int):
    lib = _lib.load()
    D = x.shape[1]
    dev = x.device
    ws_bytes = lib.rqb200_rq_workspace_bytes(D, K, 1)
    return dict(ws=torch.empty(ws_bytes, dtype=torch.uint8, device=dev), ws_bytes=ws_bytes,
                assign=torch.empty(x.shape[0], dtype=torch.int64, device=dev),
                sums=torch.empty((K, D), dtype=torch.float64, device=dev),
                counts=torch.empty(K, dtype=torch.int32, device=dev),
                shift=torch.empty(1, dtype=torch.float32, device=dev))


def kmeans_assign_accumulate(x: torch.Tensor, centroids: torch.Tensor, buf) -> None:
    lib = _lib.load()
    B, D = x.shape
    K = centroids.shape[0]
    with torch.cuda.device(x.device):
        _lib.check(lib.rqb200_kmeans_assign_accumulate(_p(x), x.stride(0), _p(centroids), B, D, K, _p(buf["assign"]),
                                                       _p(buf["sums"]), _p(buf["counts"]), _p(buf["ws"]),
                                                       buf["ws_bytes"], _stream()), "kmeans_assign_accumulate")
    _count(3)


def kmeans_finalize(x: torch.Tensor, centroids: torch.Tensor, buf, reseed_rows: Optional[torch.Tensor]) -> None:
    lib = _lib.load()
    K, D = centroids.shape
    with torch.cuda.device(x.device):
        _lib.check(lib.rqb200_kmeans_finalize(_p(buf["sums"]), _p(buf["counts"]), _p(x), x.stride(0), _p(reseed_rows),
                                              _p(centroids), K, D, _p(buf["shift"]), _stream()), "kmeans_finalize")
    _count(1)


# ---------------------------------------------------------------------------------------------- id statistics
def sid_histogram(ids: torch.Tensor, K: int) -> torch.Tensor:
    """[L,K] int64 code-usage counts of a [B,L] int64 id table (train_rqvae.py:285-289)."""
    _need_cuda(ids)
    lib = _lib.load()
    ids = ids.contiguous()
    B, L = ids.shape
    hist = torch.empty((L, K), dtype=torch.int64, device=ids.device)
    with torch.cuda.device(ids.device):
        _lib.check(lib.rqb200_sid_histogram(_p(ids), B, L, K, _p(hist), _stream()), "sid_histogram")
    _count(1)
    return hist


def sid_dedup_rank(ids: torch.Tensor, K: int):
    """Dedup column + diversity statistics of a corpus id table (semids.py:94-108, train_rqvae.py:276-283) in two launches.
    Returns (rank [N] int64, stats) with stats = dict(max_rank, n_unique: 0-d int32 tensors, entropy: 0-d float64 tensor), all on
    the device (no host sync), or None when the key space K^L is too large for the direct table (the caller sorts instead)."""
    _need_cuda(ids)
    lib = _lib.load()
    ids = ids.contiguous()
    N, L = ids.shape
    ws_bytes = lib.rqb200_sid_dedup_workspace_bytes(N, L, K)
    if ws_bytes == 0:
        return None
    dev = ids.device
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    rank = torch.empty(N, dtype=torch.int64, device=dev)
    stats = torch.empty(2, dtype=torch.int32, device=dev)
    entropy = torch.empty(1, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.rqb200_sid_dedup_rank(_p(ids), N, L, K, _p(rank), _p(stats), _p(entropy), _p(ws), ws_bytes, _stream()),
                   "sid_dedup_rank")
    _count(2)
    return rank, dict(max_rank=stats[0], n_unique=stats[1], entropy=entropy[0])


class SidPrefixIndex:
    """Valid-prefix index of a corpus id table [N, C] (modules/model.py:169-182), built once per corpus: a trie of the corpus's
    distinct prefixes (rqb200_sid_trie_build, O(N C) bytes for any K^C).  ``check`` is the reference's `_check_valid_prefix`;
    ``beam_select`` one selection step of its constrained beam search (model.py:340-376)."""

    def __init__(self, cached_ids: torch.Tensor, codebook_size: int):
        _need_cuda(cached_ids)
        lib = _lib.load()
        ids = cached_ids.to(torch.int64).contiguous()
        self.N, self.C = ids.shape
        self.K = int(codebook_size)
        self.device = ids.device
        with torch.cuda.device(ids.device):
            nbytes = lib.rqb200_sid_trie_workspace_bytes(self.N, self.C, self.K)
            scratch_bytes = lib.rqb200_sid_trie_scratch_bytes(self.N, self.C, self.K)
            if nbytes == 0 or scratch_bytes == 0:
                raise _lib.Rqb200Error(f"prefix index: a trie of {self.N} rows of {self.C} ids over {self.K} codes is outside "
                                       "its limits (N < 2^31 - 1, C <= 8, K <= 65536)")
            #: device bytes the index holds (the build's scratch is freed after the build)
            self.nbytes = int(nbytes)
            self.ws = torch.empty(nbytes, dtype=torch.uint8, device=ids.device)
            scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=ids.device)   # the allocator reuses it in stream order
            _lib.check(lib.rqb200_sid_trie_build(_p(ids), self.N, self.C, self.K, _p(self.ws), nbytes, _p(scratch), scratch_bytes,
                                                 _stream()), "sid_trie_build")
        _count(1)                                             # one build call (the trie's sort and scans are several kernels)
        self._build = StreamBuild(self.ws)

    def ready(self) -> "SidPrefixIndex":
        """This index, with the current stream ordered after its build and that of its cached levels (``StreamBuild``)."""
        self._build.ready()
        return self

    def check(self, prefix: torch.Tensor) -> torch.Tensor:
        """bool [P]: does some corpus row start with prefix[p] ([P, l], l <= C)."""
        _need_cuda(prefix)
        if prefix.dtype != torch.int64:
            prefix = prefix.to(torch.int64)
        if prefix.stride(-1) != 1:
            prefix = prefix.contiguous()
        P, l = prefix.shape
        if l > self.C:
            raise ValueError(f"prefix length {l} exceeds the id tuple length {self.C}")
        valid = torch.empty(P, dtype=torch.bool, device=prefix.device)
        with torch.cuda.device(prefix.device):
            _lib.check(_lib.load().rqb200_sid_trie_check(_p(prefix), prefix.stride(0), P, l, self.C, self.K, _p(self.ws), _p(valid),
                                                         _stream()), "sid_trie_check")
        _count(1)
        return valid

    def beam_select(self, samples: torch.Tensor, samp_log_p: torch.Tensor, generated: Optional[torch.Tensor],
                    log_probas: Optional[torch.Tensor], k: int):
        """samples / samp_log_p [B * kp, nc] (kp = 1 on the first level), generated [B, kp, h] or None, log_probas [B, kp] or None
        -> (generated [B, k, h + 1], log_probas [B, k], parent_global [B * k]) exactly as model.py:353-388 computes them."""
        _need_cuda(samples, samp_log_p)
        if generated is None:
            B, kp, h = samples.shape[0], 1, 0
        else:
            B, kp, h = generated.shape
            generated = generated.to(torch.int64).contiguous()
        nc = samples.shape[-1]
        samples = samples.to(torch.int64).reshape(B * kp, nc).contiguous()
        samp_log_p = samp_log_p.to(torch.float32).reshape(B * kp, nc).contiguous()
        if log_probas is not None:
            log_probas = log_probas.to(torch.float32).reshape(B, kp).contiguous()
        dev = samples.device
        out_g = torch.empty((B, k, h + 1), dtype=torch.int64, device=dev)
        out_p = torch.empty((B, k), dtype=torch.float32, device=dev)
        out_parent = torch.empty((B * k,), dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().rqb200_sid_trie_beam_select(_p(samples), _p(samp_log_p), _p(generated), _p(log_probas), B, kp,
                                                               nc, h, k, self.C, self.K, _p(self.ws), _p(out_g), _p(out_p),
                                                               _p(out_parent), _stream()), "sid_trie_beam_select")
        _count(1)
        return out_g, out_p, out_parent

    def sample_select(self, probas: torch.Tensor, noise: torch.Tensor, generated: Optional[torch.Tensor],
                      log_probas: Optional[torch.Tensor], k: int, nc: int, want_samples: bool = False,
                      reject: Optional[torch.Tensor] = None, exclude: Optional["SidExclusion"] = None,
                      include: Optional["SidInclusion"] = None, cap: Optional[Tuple[int, int]] = None):
        """The sampling step fused with ``beam_select`` (rqb200_sid_trie_sample_select), one launch.  probas / noise [B * kp, K]
        (kp = 1 on the first level; noise = the Exp(1) draw torch.multinomial makes, ``torch.empty_like(probas).exponential_(1)``),
        generated [B, kp, h] or None, log_probas [B, kp] or None -> (generated [B, k, h + 1], log_probas [B, k],
        parent_global [B * k]), plus (samples [B * kp, nc], samp_log_p [B * kp, nc]) when ``want_samples``: the samples are
        ``torch.multinomial(probas, nc)``'s under the same generator state.  ``reject``, an int32 [2] device tensor, is ADDED the
        number of rows torch.multinomial would reject: [0] with a NaN, +-inf or negative entry, [1] otherwise all zero.
        ``exclude`` (``sid_exclusion_build``, one set per history): extensions to a prefix blocked for the history are invalid,
        exactly like prefixes the corpus lacks; the samples do not change.  ``include`` (``sid_inclusion_build``, one allow-list
        per history, any exclusion folded in; not with ``exclude``): extensions to a prefix without an eligible item of the
        history are invalid alike.  ``cap`` = (prefix_len, max_per_prefix) caps the selection as ``beam_topk``'s ``cap``, in
        the candidates' order (score descending, lowest beam * nc + slot first); the samples do not change."""
        return self._sample_select("sid_trie_sample_select", probas, noise, generated, log_probas, k, nc, want_samples, reject,
                                   exclude, include, cap=cap)

    def sample_select_wide(self, probas: torch.Tensor, noise: torch.Tensor, generated: Optional[torch.Tensor],
                           log_probas: Optional[torch.Tensor], k: int, nc: int, want_samples: bool = False,
                           reject: Optional[torch.Tensor] = None, exclude: Optional["SidExclusion"] = None,
                           include: Optional["SidInclusion"] = None, cluster: int = 0):
        """``sample_select`` for up to 1024 beams per history (rqb200_sid_trie_sample_select_wide): one thread-block cluster per
        history, one launch.  Same arguments and results, bit for bit wherever both run; kp <= 1024, k <= 1024, nc <= 64.  When
        k > kp * nc the slots past kp * nc repeat candidate 0 with -inf.  ``cluster``: CTAs per history (1, 2, 4 or 8; 0
        chooses); no result depends on it."""
        return self._sample_select("sid_trie_sample_select_wide", probas, noise, generated, log_probas, k, nc, want_samples,
                                   reject, exclude, include, int(cluster))

    def sample_select_warped(self, logits: torch.Tensor, noise: torch.Tensor, generated: Optional[torch.Tensor],
                             log_probas: Optional[torch.Tensor], k: int, nc: int, temperature: float, top_p: float,
                             want_samples: bool = False, bad: Optional[torch.Tensor] = None,
                             exclude: Optional["SidExclusion"] = None, include: Optional["SidInclusion"] = None,
                             cap: Optional[Tuple[int, int]] = None):
        """``sample_select`` drawn from the head's logits at ``temperature`` and within a ``top_p`` nucleus
        (rqb200_sid_trie_sample_select_warped), one launch.  logits / noise [B * kp, K].  Per beam row x:
        p_T = softmax(x / T) in fp32; the nucleus N = the codes with p_T >= t, t the largest p_T whose codes at or above it
        hold at least top_p of the mass (fixed-point sums; ties at t all in; top_p = 1: every code); the beam draws the
        min(nc, |N+|) largest p_T / noise over N+ (the codes of N with p_T > 0), equal ratios by ascending code, and fills the
        other slots with -inf.  A drawn code scores its model log-probability x[c] - lse (``beam_topk``'s lse, bit for bit)
        plus the parent's, -inf off the trie or blocked by the filter; ``samp_log_p`` holds x[c] - lse (-inf for a filler).
        ``bad``, an int32 device tensor, is ADDED the number of beam rows holding a NaN or +inf or all -inf (their slots are
        fillers).  T finite and > 0, 0 < top_p <= 1, else ``Rqb200Error``.  ``exclude`` / ``include`` / ``cap`` as in
        ``sample_select``."""
        return self._sample_select("sid_trie_sample_select_warped", logits, noise, generated, log_probas, k, nc, want_samples,
                                   bad, exclude, include, warp=(float(temperature), float(top_p)), cap=cap)

    def sample_select_warped_wide(self, logits: torch.Tensor, noise: torch.Tensor, generated: Optional[torch.Tensor],
                                  log_probas: Optional[torch.Tensor], k: int, nc: int, temperature: float, top_p: float,
                                  want_samples: bool = False, bad: Optional[torch.Tensor] = None,
                                  exclude: Optional["SidExclusion"] = None, include: Optional["SidInclusion"] = None,
                                  cluster: int = 0):
        """``sample_select_warped`` on the cluster kernel (rqb200_sid_trie_sample_select_warped_wide), with
        ``sample_select_wide``'s limits and ``cluster``; bit for bit wherever both run, and no result depends on the cluster
        size."""
        return self._sample_select("sid_trie_sample_select_warped_wide", logits, noise, generated, log_probas, k, nc,
                                   want_samples, bad, exclude, include, int(cluster), warp=(float(temperature), float(top_p)))

    def _sample_select(self, entry: str, probas, noise, generated, log_probas, k: int, nc: int, want_samples: bool, reject,
                       exclude, include, cluster: Optional[int] = None, warp: Optional[tuple] = None,
                       cap: Optional[Tuple[int, int]] = None):
        _need_cuda(probas, noise, reject)
        if generated is None:
            B, kp, h = probas.shape[0], 1, 0
        else:
            B, kp, h = generated.shape
            generated = generated.to(torch.int64).contiguous()
            if log_probas is None:
                raise ValueError("log_probas is required with generated")
            log_probas = log_probas.to(torch.float32).reshape(B, kp).contiguous()
        probas, noise = _rows(probas), _rows(noise)
        if probas.shape != noise.shape or probas.shape[0] != B * kp:
            raise ValueError(f"probas {tuple(probas.shape)} / noise {tuple(noise.shape)} must both be [B * kp = {B * kp}, K]")
        if probas.shape[1] != self.K:
            raise ValueError(f"probas has {probas.shape[1]} codes, the prefix index {self.K}")
        if warp is not None:
            if reject is not None and (reject.dtype != torch.int32 or reject.numel() < 1 or not reject.is_contiguous()):
                raise ValueError("bad must be a contiguous int32 tensor")
        elif reject is not None and (reject.dtype != torch.int32 or reject.numel() < 2 or not reject.is_contiguous()):
            raise ValueError("reject must be a contiguous int32 tensor of 2 elements")
        dev = probas.device
        out_g = torch.empty((B, k, h + 1), dtype=torch.int64, device=dev)
        out_p = torch.empty((B, k), dtype=torch.float32, device=dev)
        out_parent = torch.empty((B * k,), dtype=torch.int64, device=dev)
        samples = torch.empty((B * kp, nc), dtype=torch.int64, device=dev) if want_samples else None
        samp_log_p = torch.empty((B * kp, nc), dtype=torch.float32, device=dev) if want_samples else None
        name, filt = _filter_entry(entry, exclude, include, B, h + 1, entry[9:], cap)
        lib = _lib.load()
        wide = ()
        if cluster is not None:                               # the wide entry: its workspace and the cluster size
            ws_bytes = lib.rqb200_sid_trie_sample_select_wide_workspace_bytes(B, kp, nc)
            ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
            wide = (_p(ws), ws_bytes, cluster)
        warp = () if warp is None else warp                   # the warped entries: temperature, top_p
        with torch.cuda.device(dev):
            _lib.check(getattr(lib, "rqb200_" + name)(
                _p(probas), probas.stride(0), _p(noise), noise.stride(0), _p(generated), _p(log_probas), B, kp, nc, h, k, self.C,
                self.K, _p(self.ws), _p(out_g), _p(out_p), _p(out_parent), _p(samples), _p(samp_log_p), _p(reject), *wide, *warp,
                *filt, _stream()), name)
        _count(1)
        if want_samples:
            return out_g, out_p, out_parent, samples, samp_log_p
        return out_g, out_p, out_parent

    def beam_topk(self, logits: torch.Tensor, generated: Optional[torch.Tensor], log_probas: Optional[torch.Tensor], k: int,
                  bad: Optional[torch.Tensor] = None, exclude: Optional["SidExclusion"] = None,
                  include: Optional["SidInclusion"] = None, cap: Optional[Tuple[int, int]] = None):
        """One level of the exhaustive constrained beam search from the head's logits (rqb200_sid_trie_beam_topk), one launch.
        logits [B * kp, K] (kp = 1 on the first level), generated [B, kp, h] or None, log_probas [B, kp] or None ->
        (generated [B, k, h + 1], log_probas [B, k], parent_global [B * k]): of all kp * K extensions of each history, scored
        log_softmax(logits)[code] + the parent's log-probability (-inf when the extended prefix is not in the corpus), the k
        best in descending order, equal scores by ascending beam * K + code.  Deterministic.  ``bad``, an int32 device tensor,
        is ADDED the number of beam rows whose logits hold a NaN or +inf or are all -inf.  ``exclude`` / ``include`` as in
        ``sample_select``: extensions to a prefix blocked for the history, or without an eligible item of it, score -inf.
        ``cap`` = (prefix_len, max_per_prefix), 1 <= prefix_len <= h and max_per_prefix >= 1 (rqb200_sid_trie_beam_topk_capped):
        walking down that order, a candidate is kept unless max_per_prefix candidates whose parents share its parent's first
        prefix_len ids were kept before it; the dropped ones score -inf and rank among the -inf fillers by beam * K + code.
        None (or max_per_prefix >= k, which cannot bind) gives the uncapped result."""
        return self._beam_topk("sid_trie_beam_topk", logits, generated, log_probas, k, bad, exclude, include, cap=cap)

    def beam_topk_wide(self, logits: torch.Tensor, generated: Optional[torch.Tensor], log_probas: Optional[torch.Tensor], k: int,
                       bad: Optional[torch.Tensor] = None, exclude: Optional["SidExclusion"] = None,
                       include: Optional["SidInclusion"] = None, cluster: int = 0):
        """``beam_topk`` for up to 1024 beams per history (rqb200_sid_trie_beam_topk_wide): one thread-block cluster per history,
        one launch.  Same arguments and results, bit for bit wherever both run; kp <= 1024, k <= min(1024, K).  ``cluster``:
        CTAs per history (1, 2, 4 or 8; 0 chooses); no result depends on it."""
        return self._beam_topk("sid_trie_beam_topk_wide", logits, generated, log_probas, k, bad, exclude, include, int(cluster))

    def _beam_topk(self, entry: str, logits, generated, log_probas, k: int, bad, exclude, include,
                   cluster: Optional[int] = None, cap: Optional[Tuple[int, int]] = None):
        _need_cuda(logits, bad)
        if generated is None:
            B, kp, h = logits.shape[0], 1, 0
        else:
            B, kp, h = generated.shape
            generated = generated.to(torch.int64).contiguous()
            if log_probas is None:
                raise ValueError("log_probas is required with generated")
            log_probas = log_probas.to(torch.float32).reshape(B, kp).contiguous()
        logits = _rows(logits)
        if logits.shape[0] != B * kp:
            raise ValueError(f"logits {tuple(logits.shape)} must be [B * kp = {B * kp}, K]")
        if logits.shape[1] != self.K:
            raise ValueError(f"logits has {logits.shape[1]} codes, the prefix index {self.K}")
        if bad is not None and (bad.dtype != torch.int32 or bad.numel() < 1 or not bad.is_contiguous()):
            raise ValueError("bad must be a contiguous int32 tensor")
        dev = logits.device
        out_g = torch.empty((B, k, h + 1), dtype=torch.int64, device=dev)
        out_p = torch.empty((B, k), dtype=torch.float32, device=dev)
        out_parent = torch.empty((B * k,), dtype=torch.int64, device=dev)
        name, filt = _filter_entry(entry, exclude, include, B, h + 1, entry[9:], cap)
        wide = () if cluster is None else (cluster,)
        with torch.cuda.device(dev):
            _lib.check(getattr(_lib.load(), "rqb200_" + name)(
                _p(logits), logits.stride(0), _p(generated), _p(log_probas), B, kp, h, k, self.C, self.K, _p(self.ws), _p(out_g),
                _p(out_p), _p(out_parent), _p(bad), *wide, *filt, _stream()), name)
        _count(1)
        return out_g, out_p, out_parent

    def counts(self) -> torch.Tensor:
        """int32 [C + 1] on the device: the node count of every level (the root's 1 first), one launch, no host read."""
        counts = torch.empty(self.C + 1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().rqb200_sid_trie_counts(_p(self.ws), _p(counts), _stream()), "sid_trie_counts")
        _count(1)
        return counts

    def levels(self, n: Sequence[int]) -> "SidTrieLevels":
        """The level arrays of levels 1..C as device tensors, given the node counts n = ``counts()`` read on the host; one launch
        per level.  Built once and cached on the index."""
        self.ready()
        if getattr(self, "_levels", None) is None:
            n = [int(v) for v in n]
            if len(n) != self.C + 1 or n[0] != 1:
                raise ValueError(f"levels: n must be the {self.C + 1} node counts of counts(), got {n}")
            child0 = torch.zeros(2, dtype=torch.int32, device=self.device)
            child0[1:].fill_(n[1])                            # not torch.tensor(..., device=): that copy synchronises the stream
            code, parent, child = [None], [None], [child0]
            lib = _lib.load()
            for l in range(1, self.C + 1):
                c = torch.empty(n[l], dtype=torch.int32, device=self.device)
                p = torch.empty(n[l], dtype=torch.int32, device=self.device)
                ch = torch.zeros(n[l] + 1, dtype=torch.int32, device=self.device) if l < self.C else None
                if n[l] > 0:
                    with torch.cuda.device(self.device):
                        _lib.check(lib.rqb200_sid_trie_level(_p(self.ws), self.C, l, n[l], n[l - 1], _p(c), _p(p), _p(ch),
                                                             _stream()), "sid_trie_level")
                    _count(1)
                code.append(c)
                parent.append(p)
                child.append(ch)
            self._levels = SidTrieLevels(n, code, parent, child)
            self._build = StreamBuild(self.ws, *(t for t in code + parent + child if t is not None))
        return self._levels


class SidTrieLevels(NamedTuple):
    """A trie's levels: n[l] nodes in level l (n[0] = 1, the root); for l >= 1 code[l] / parent[l] int32 [n[l]] (each node's last
    id and its node in level l - 1); child[l] int32 [n[l] + 1] for l < C (node i's children in level l + 1 are child[l][i] ..
    child[l][i + 1] - 1; child[0] = [0, n[1]]).  Nodes of one level are in lexicographic order of their prefixes."""
    n: List[int]
    code: List[Optional[torch.Tensor]]
    parent: List[Optional[torch.Tensor]]
    child: List[Optional[torch.Tensor]]


class SidItemTable:
    """Item table of a corpus id table [N, C] (rqb200_sid_items_build): maps generated id tuples back to the corpus items (rows)
    that carry them.  Row n is item n; the items of one tuple come in ascending row order, which is dedup rank 0, 1, 2, ....
    A row holding an id outside [0, codebook_size) is never retrieved.  Built once per corpus, one launch per call."""

    MAX_K, MAX_N = 1024, 4096

    def __init__(self, cached_ids: torch.Tensor, codebook_size: int):
        _need_cuda(cached_ids)
        lib = _lib.load()
        ids = cached_ids.to(torch.int64).contiguous()
        self.N, self.C = ids.shape
        self.K = int(codebook_size)
        self.device = ids.device
        nbytes = lib.rqb200_sid_items_workspace_bytes(self.N, self.C, self.K)
        if nbytes == 0:
            raise _lib.Rqb200Error(f"item table: {self.N} rows of {self.C} ids over {self.K} codes is outside its limits "
                                   "(N < 2^31 - 1, C <= 8, K <= 65536)")
        #: device bytes the table holds (its build scratch included)
        self.nbytes = int(nbytes)
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=ids.device)
        with torch.cuda.device(ids.device):
            _lib.check(lib.rqb200_sid_items_build(_p(ids), self.N, self.C, self.K, _p(self.ws), nbytes, _stream()),
                       "sid_items_build")
        _count(1)                                             # one build call (the sort and the scan are several kernels)
        self._build = StreamBuild(self.ws)

    def ready(self) -> "SidItemTable":
        """This table, with the current stream ordered after its build and that of its cached positions (``StreamBuild``)."""
        self._build.ready()
        return self

    def lookup(self, ids: torch.Tensor, with_dedup: bool = False) -> torch.Tensor:
        """int64 [...]: the item of each tuple ids[..., :C] -- its first item, or with ``with_dedup`` the item of dedup rank
        ids[..., C] -- or -1 when the tuple is not in the corpus or the rank is outside [0, count)."""
        _need_cuda(ids)
        width = self.C + (1 if with_dedup else 0)
        if ids.shape[-1] != width:
            raise ValueError(f"lookup: expected {width} columns (C = {self.C}{' + the dedup rank' if with_dedup else ''}), "
                             f"got {ids.shape[-1]}")
        lead = ids.shape[:-1]
        rows = ids.to(torch.int64).reshape(-1, width)
        if rows.stride(-1) != 1 or (rows.shape[0] > 1 and rows.stride(0) < width):
            rows = rows.contiguous()
        P = rows.shape[0]
        out = torch.empty(P, dtype=torch.int64, device=ids.device)
        with torch.cuda.device(ids.device):
            _lib.check(_lib.load().rqb200_sid_items_lookup(_p(self.ws), _p(rows), max(rows.stride(0), 1), P, int(with_dedup),
                                                           _p(out), _stream()), "sid_items_lookup")
        _count(1)
        return out.reshape(lead)

    def retrieve(self, generated: torch.Tensor, log_probas: Optional[torch.Tensor], n: int,
                 exclude: Optional["SidExclusion"] = None, include: Optional["SidInclusion"] = None):
        """generated [B, k, C], log_probas [B, k] or None -> (items [B, n] int64, beam [B, n] int32, count [B] int32): per
        history, in beam order, the items of every beam whose log-probability is above -inf and whose tuple is in the corpus,
        each beam's in dedup-rank order, no item twice, cut off at n; -1 pads items and beam.  k <= 1024, n <= 4096.
        ``exclude`` (``sid_exclusion_build`` on this table): the history's excluded items are skipped.  ``include``
        (``sid_inclusion_build`` on this table; not with ``exclude``): only the history's eligible items are taken."""
        _need_cuda(generated, log_probas)
        B, k, C = generated.shape
        if C != self.C:
            raise ValueError(f"retrieve: generated has {C} ids per beam, the item table {self.C}")
        n = int(n)
        generated = generated.to(torch.int64).contiguous()
        if log_probas is not None:
            log_probas = log_probas.to(torch.float32).reshape(B, k).contiguous()
        dev = generated.device
        items = torch.empty((B, n), dtype=torch.int64, device=dev)
        beam = torch.empty((B, n), dtype=torch.int32, device=dev)
        count = torch.empty((B,), dtype=torch.int32, device=dev)
        name, filt = _filter_entry("sid_items_retrieve", exclude, include, B, 0, "retrieve")
        with torch.cuda.device(dev):
            _lib.check(getattr(_lib.load(), "rqb200_" + name)(_p(self.ws), _p(generated), _p(log_probas), B, k, C, n, _p(items),
                                                              _p(beam), _p(count), *filt, _stream()), name)
        _count(1)
        return items, beam, count

    def arrays(self):
        """(row int32 [N], start int32 [N + 1]): views of the table's workspace.  Tuple u's items are row[start[u] .. start[u + 1])
        in dedup order; only the first U + 1 entries of start are written (U: the distinct retrievable tuples)."""
        self.ready()
        row_off, start_off = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(_lib.load().rqb200_sid_items_offsets(self.N, self.C, self.K, ctypes.byref(row_off), ctypes.byref(start_off)),
                   "sid_items_offsets")
        row = self.ws[row_off.value:row_off.value + 4 * self.N].view(torch.int32)
        start = self.ws[start_off.value:start_off.value + 4 * (self.N + 1)].view(torch.int32)
        return row, start

    def positions(self) -> torch.Tensor:
        """int32 [N]: each item's position in the table's row array (the inverse permutation of ``arrays()[0]``), built once
        and cached on the table."""
        if getattr(self, "_positions", None) is None:
            row, _ = self.arrays()
            inv = torch.empty(self.N, dtype=torch.int32, device=self.device)
            inv[row.long()] = torch.arange(self.N, dtype=torch.int32, device=self.device)
            self._positions = inv
            self._build = StreamBuild(self.ws, inv)
        self.ready()
        return self._positions


#: most entries per history an exclusion set takes (sid_exclusion_build sorts them in shared memory)
EXCLUDE_MAX_ITEMS = 4096
#: most entries per history an allow-list takes (sid_inclusion_build, the same kernel)
INCLUDE_MAX_ITEMS = EXCLUDE_MAX_ITEMS


def _filter_args(f, kind: str, B: int, levels: int, what: str):
    """The filter arguments (pos, keys, count, M, H) of the *_excluding / *_including entry points, for B histories and a level
    up to ``levels``."""
    _need_cuda(f.pos)
    H = f[1].shape[1]
    if f.pos.shape[0] != B:
        raise ValueError(f"{what}: the {kind} holds {f.pos.shape[0]} histories, the call {B}")
    if levels > H:
        raise ValueError(f"{what}: level {levels} is deeper than the {kind}'s {H} levels")
    return _p(f.pos), _p(f[1]), _p(f.count), f.pos.shape[1], H


def _filter_entry(entry: str, exclude, include, B: int, levels: int, what: str, cap: Optional[Tuple[int, int]] = None):
    """(entry point name, filter arguments) of a consumer call: ``entry`` without a filter, ``entry``_excluding /
    ``entry``_including with one.  An inclusion has the exclusion folded in, so a call takes at most one.  With a ``cap``
    (prefix_len, max_per_prefix): ``entry``_capped, whose arguments are the cap, the filter mode and the filter's arrays."""
    if exclude is not None and include is not None:
        raise ValueError(f"{what}: pass exclude or include, not both (sid_inclusion_build folds an exclusion into the "
                         "inclusion)")
    if cap is not None:
        prefix_len, max_per_prefix = (int(c) for c in cap)
        if include is not None:
            return entry + "_capped", (prefix_len, max_per_prefix, 2) + include.args(B, levels, what)
        if exclude is not None:
            return entry + "_capped", (prefix_len, max_per_prefix, 1) + exclude.args(B, levels, what)
        return entry + "_capped", (prefix_len, max_per_prefix, 0, None, None, None, 0, 0)
    if include is not None:
        return entry + "_including", include.args(B, levels, what)
    if exclude is not None:
        return entry + "_excluding", exclude.args(B, levels, what)
    return entry, ()


class SidExclusion(NamedTuple):
    """Each history's exclusion set (``sid_exclusion_build``).  pos int32 [B, M]: the distinct excluded retrievable items as
    positions in the item table's row array, ascending; blocked int64 [B, H, M]: per level l = 1..H the keys (``_tuple_key``
    of the prefix) of the blocked l-prefixes, ascending -- prefixes holding an excluded item under which every retrievable
    item is excluded; count int32 [B, H + 2]: [0] the positions, [l] the blocked l-prefixes, [H + 1] the entries outside
    [-1, N).  Entries past a count are -1."""
    pos: torch.Tensor
    blocked: torch.Tensor
    count: torch.Tensor

    def args(self, B: int, levels: int, what: str):
        """The exclusion arguments of the *_excluding entry points, for B histories and a level up to ``levels``."""
        return _filter_args(self, "exclusion", B, levels, what)


class SidInclusion(NamedTuple):
    """Each history's allow-list (``sid_inclusion_build``), in ``SidExclusion``'s layout.  pos int32 [B, M]: the distinct
    eligible items (allowed, retrievable, not excluded) as positions in the item table's row array, ascending; keys int64
    [B, H, M]: per level l = 1..H the keys (``_tuple_key`` of the prefix) of the valid l-prefixes -- those with an eligible item
    under them -- ascending; count int32 [B, H + 2]: [0] the positions, [l] the valid l-prefixes, [H + 1] the allowed ids
    outside [-1, N).  Entries past a count are -1."""
    pos: torch.Tensor
    keys: torch.Tensor
    count: torch.Tensor

    def args(self, B: int, levels: int, what: str):
        """The inclusion arguments of the *_including entry points, for B histories and a level up to ``levels``."""
        return _filter_args(self, "inclusion", B, levels, what)


def _filter_items(items: torch.Tensor, kind: str, limit: int):
    """items as a contiguous int64 [B, max(M, 1)] (an empty row is one -1), after the checks of a filter build."""
    if items.dim() != 2 or items.dtype.is_floating_point or items.dtype.is_complex or items.dtype == torch.bool:
        raise ValueError(f"{kind}: items must be an integer [B, M] tensor, got {items.dtype} {tuple(items.shape)}")
    B, M = items.shape
    if M > limit:
        raise ValueError(f"{kind}: M = {M} items per history exceeds {limit}")
    if M == 0:
        return torch.full((B, 1), -1, dtype=torch.int64, device=items.device)
    return items.to(torch.int64).contiguous()


def sid_inclusion_build(items: torch.Tensor, table: SidItemTable, leaf_key: torch.Tensor,
                        exclude: Optional[SidExclusion] = None) -> SidInclusion:
    """Each history's allow-list (rqb200_sid_inclusion_build), one launch, no host read.  items integer [B, M] (corpus rows,
    -1 pads, repeats allowed, M <= ``INCLUDE_MAX_ITEMS``), table and leaf_key as in ``sid_exclusion_build``, exclude an
    exclusion of the same B histories on the same table, folded in: an item is eligible when it is allowed, retrievable and
    not excluded.  Ids outside [-1, N) are counted in count[:, H + 1]."""
    _need_cuda(items, leaf_key)
    items = _filter_items(items, "inclusion", INCLUDE_MAX_ITEMS)
    B, M = items.shape
    dev = items.device
    leaf_key = leaf_key.to(torch.int64).contiguous()
    H, U = table.C, leaf_key.shape[0]
    if exclude is not None and exclude.blocked.shape[1] != H:
        raise ValueError(f"inclusion: the exclusion has {exclude.blocked.shape[1]} levels, the item table {H}")
    filt = (None, None, None, 0, 0) if exclude is None else exclude.args(B, H, "inclusion")
    _, start = table.arrays()
    pos = torch.empty((B, M), dtype=torch.int32, device=dev)
    keys = torch.empty((B, H, M), dtype=torch.int64, device=dev)
    count = torch.empty((B, H + 2), dtype=torch.int32, device=dev)
    inv = table.positions()
    with torch.cuda.device(dev):
        _lib.check(_lib.load().rqb200_sid_inclusion_build(_p(items), B, M, table.N, _p(inv), _p(start), _p(leaf_key), U, H,
                                                          table.K, _p(pos), _p(keys), _p(count), *filt, _stream()),
                   "sid_inclusion_build")
    _count(1)
    return SidInclusion(pos, keys, count)


def sid_exclusion_build(items: torch.Tensor, table: SidItemTable, leaf_key: torch.Tensor) -> SidExclusion:
    """Each history's exclusion set (rqb200_sid_exclusion_build), one launch, no host read.  items integer [B, M] (corpus rows,
    -1 pads, repeats allowed, M <= ``EXCLUDE_MAX_ITEMS``), table the corpus's ``SidItemTable`` (H = its C ids per tuple),
    leaf_key int64 [U]: the table's U distinct retrievable tuples packed K-ary (level 0 most significant), ascending.  Rows
    that are not retrievable are ignored; ids outside [-1, N) are counted in count[:, H + 1]."""
    _need_cuda(items, leaf_key)
    items = _filter_items(items, "exclusion", EXCLUDE_MAX_ITEMS)
    B, M = items.shape
    dev = items.device
    leaf_key = leaf_key.to(torch.int64).contiguous()
    H, U = table.C, leaf_key.shape[0]
    _, start = table.arrays()
    pos = torch.empty((B, M), dtype=torch.int32, device=dev)
    blocked = torch.empty((B, H, M), dtype=torch.int64, device=dev)
    count = torch.empty((B, H + 2), dtype=torch.int32, device=dev)
    inv = table.positions()
    with torch.cuda.device(dev):
        _lib.check(_lib.load().rqb200_sid_exclusion_build(_p(items), B, M, table.N, _p(inv), _p(start), _p(leaf_key), U, H,
                                                          table.K, _p(pos), _p(blocked), _p(count), _stream()),
                   "sid_exclusion_build")
    _count(1)
    return SidExclusion(pos, blocked, count)


def sid_rank_hist(rank: torch.Tensor, hist: torch.Tensor) -> None:
    """Adds exact ranks (int64 [B], -1: not ranked) to hist (int64 [k + 1]): hist[rank] for rank < k, hist[k] otherwise.  One
    launch; never waits on the host."""
    _need_cuda(rank, hist)
    if hist.dtype != torch.int64 or hist.dim() != 1 or hist.numel() < 2 or not hist.is_contiguous():
        raise ValueError("rank histogram: hist must be a contiguous int64 tensor of k + 1 >= 2 elements")
    rank = rank.reshape(-1).to(torch.int64).contiguous()
    with torch.cuda.device(hist.device):
        _lib.check(_lib.load().rqb200_sid_rank_hist(_p(rank), rank.numel(), hist.numel() - 1, _p(hist), _stream()),
                   "sid_rank_hist")
    _count(1)


def sid_topk_rank_hist(actual: torch.Tensor, candidates: torch.Tensor, hist: torch.Tensor, item_mode: bool = False) -> None:
    """Adds the rank of every row to hist (int64 [k + 1], on the device): the first candidate candidates[b, j] ([B, k, D]) equal
    to actual[b] ([B, D]) in all D columns, k when none is (evaluate/metrics.py's rule).  ``item_mode``: -1 never matches.
    One launch; never waits on the host."""
    _need_cuda(actual, candidates, hist)
    if candidates.dim() != 3 or actual.dim() != 2 or actual.shape[0] != candidates.shape[0] or \
            actual.shape[1] != candidates.shape[2]:
        raise ValueError(f"rank histogram: actual {tuple(actual.shape)} must be [B, D] and candidates "
                         f"{tuple(candidates.shape)} [B, k, D]")
    B, k, D = candidates.shape
    if hist.dtype != torch.int64 or hist.numel() < k + 1 or not hist.is_contiguous():
        raise ValueError(f"rank histogram: hist must be a contiguous int64 tensor of at least k + 1 = {k + 1} elements")
    actual = actual.to(torch.int64)
    if actual.stride(1) != 1 or actual.stride(0) < D:
        actual = actual.contiguous()
    candidates = candidates.to(torch.int64)
    if candidates.stride(2) != 1 or candidates.stride(1) != D or candidates.stride(0) < k * D:
        candidates = candidates.contiguous()
    with torch.cuda.device(hist.device):
        _lib.check(_lib.load().rqb200_sid_topk_rank_hist(_p(actual), max(actual.stride(0), D), _p(candidates),
                                                         max(candidates.stride(0), k * D), B, k, D, int(item_mode), _p(hist),
                                                         _stream()), "sid_topk_rank_hist")
    _count(1)


def sid_gather(cached_ids: torch.Tensor, item_ids: torch.Tensor, seq_mask: Optional[torch.Tensor] = None,
               want_token_type: bool = True):
    """cached_ids[item_ids] -> [B, S*C] with -1 under the padding mask, and token_type_ids (semids.py:112-146), one launch."""
    _need_cuda(cached_ids, item_ids)
    lib = _lib.load()
    cached_ids = cached_ids.contiguous()
    if item_ids.stride(-1) != 1:
        item_ids = item_ids.contiguous()
    B, S = item_ids.shape
    C = cached_ids.shape[1]
    dev = cached_ids.device
    out = torch.empty((B, S * C), dtype=torch.int64, device=dev)
    tt = torch.empty((B, S * C), dtype=torch.int64, device=dev) if want_token_type else None
    m = None
    if seq_mask is not None:
        m = seq_mask.to(torch.uint8) if seq_mask.dtype != torch.uint8 else seq_mask
        if m.stride(-1) != 1:
            m = m.contiguous()
    with torch.cuda.device(dev):
        _lib.check(lib.rqb200_sid_gather(_p(cached_ids), cached_ids.shape[0], C, _p(item_ids), item_ids.stride(0), _p(m),
                                         m.stride(0) if m is not None else 0, B, S, _p(out), _p(tt), _stream()), "sid_gather")
    _count(1)
    return out, tt


# ---------------------------------------------------------------------------------------------- fused T5 decoder step
T5_DKV = 64       # d_kv the decoder-step kernels are built for (csrc/t5dec.cu)


def _rows_of(t: torch.Tensor, width: int, what: str) -> torch.Tensor:
    t = _rows(t)
    if t.shape[1] != width:
        raise ValueError(f"{what}: expected {width} columns, got {tuple(t.shape)}")
    return t


def t5dec_cross_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, mask: Optional[torch.Tensor], nq: int,
                          heads: int) -> torch.Tensor:
    """T5 cross-attention over keys/values stored once per history (rqb200_t5dec_cross_attention), one launch.
    q [B * nq, heads * 64] (history b owns rows b * nq ...), k / v [B * S, heads * 64] (any row stride), mask [B, S] (0 masks a
    key: -FLT_MAX is added to its score, as HF's eager mask) or None -> [B * nq, heads * 64]."""
    _need_cuda(q, k, v, mask)
    inner = heads * T5_DKV
    q, k, v = _rows_of(q, inner, "q"), _rows_of(k, inner, "k"), _rows_of(v, inner, "v")
    if q.shape[0] % nq:
        raise ValueError(f"q has {q.shape[0]} rows, not a multiple of nq = {nq}")
    B = q.shape[0] // nq
    if B == 0 or k.shape != v.shape or k.shape[0] == 0 or k.shape[0] % B:
        raise ValueError(f"k {tuple(k.shape)} / v {tuple(v.shape)} must both be [B * S, {inner}] with B = {B} > 0, S > 0")
    if k.stride(0) != v.stride(0):
        k, v = k.contiguous(), v.contiguous()
    S = k.shape[0] // B
    if mask is not None:
        mask = _f32c(mask)
        if mask.shape != (B, S):
            raise ValueError(f"mask {tuple(mask.shape)} must be [B, S] = [{B}, {S}]")
    out = torch.empty((q.shape[0], inner), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        _lib.check(_lib.load().rqb200_t5dec_cross_attention(_p(q), q.stride(0), _p(k), _p(v), k.stride(0), _p(mask), B, nq, S,
                                                            heads, _p(out), out.stride(0), _stream()), "t5dec_cross_attention")
    _count(1)
    return out


def t5dec_self_attention(qkv: torch.Tensor, cache_k: torch.Tensor, cache_v: torch.Tensor, bias: torch.Tensor, h: int,
                         anc_in: Optional[torch.Tensor], parent: Optional[torch.Tensor] = None,
                         anc_out: Optional[torch.Tensor] = None, live: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The causal T5 self-attention of query position h for R beam rows (rqb200_t5dec_self_attention), one launch.
    qkv [R, 3 * heads * 64] (q | k | v); cache_k / cache_v [H, rows, heads * 64] contiguous, rows >= R: the rows' k / v are written
    to slot h, position j < h of row r is read from row anc[r, j] of slot j; bias [heads, H, H] (HF's compute_bias(H, H)[0]).
    anc = anc_in (int32 [*, H]) when parent is None; with parent (int64 [R]) anc[r] = anc_in[parent[r]] with position h - 1 set
    to parent[r], written to anc_out (int32 [R', H], R' >= R, not anc_in).  Returns [R, heads * 64].  ``live`` (int32 on the
    device, rqb200_t5dec_self_attention_counted): R is a capacity and only rows below live[0] are computed and written."""
    _need_cuda(qkv, cache_k, cache_v, bias, anc_in, parent, anc_out)
    H, rows, inner = cache_k.shape
    heads = inner // T5_DKV
    qkv = _rows_of(qkv, 3 * inner, "qkv")
    R = qkv.shape[0]
    if cache_v.shape != cache_k.shape or not (cache_k.is_contiguous() and cache_v.is_contiguous()) or rows < R or \
            cache_k.dtype != torch.float32 or cache_v.dtype != torch.float32:
        raise ValueError(f"cache_k / cache_v must be contiguous fp32 [H, rows >= {R}, {inner}]")
    bias = _f32c(bias)
    if bias.shape != (heads, H, H):
        raise ValueError(f"bias {tuple(bias.shape)} must be [{heads}, {H}, {H}]")
    for name, t in (("anc_in", anc_in), ("anc_out", anc_out)):
        if t is not None and (t.dtype != torch.int32 or t.dim() != 2 or t.shape[1] != H or not t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous int32 [rows, {H}] tensor")
    if parent is not None:
        parent = parent.to(torch.int64).contiguous()
        if parent.shape != (R,) or anc_out is None or anc_out.shape[0] < R or (anc_in is not None and
                                                                               anc_out.data_ptr() == anc_in.data_ptr()):
            raise ValueError("parent must be [R] and comes with an anc_out of at least R rows that is not anc_in")
    elif anc_in is not None and anc_in.shape[0] < R:
        raise ValueError(f"anc_in has {anc_in.shape[0]} rows, fewer than R = {R}")
    out = torch.empty((R, inner), dtype=torch.float32, device=qkv.device)
    with torch.cuda.device(qkv.device):
        if live is None:
            _lib.check(_lib.load().rqb200_t5dec_self_attention(_p(qkv), qkv.stride(0), _p(cache_k), _p(cache_v), rows * inner,
                                                               _p(bias), _p(anc_in), _p(parent), _p(anc_out), R, heads, int(h), H,
                                                               _p(out), out.stride(0), _stream()), "t5dec_self_attention")
        else:
            _lib.check(_lib.load().rqb200_t5dec_self_attention_counted(
                _p(qkv), qkv.stride(0), _p(cache_k), _p(cache_v), rows * inner, _p(bias), _p(anc_in), _p(parent), _p(anc_out), R,
                _p(_live(live)), heads, int(h), H, _p(out), out.stride(0), _stream()), "t5dec_self_attention_counted")
    _count(1)
    return out


def t5dec_add_norm(x: torch.Tensor, delta: Optional[torch.Tensor], weight: torch.Tensor, out: torch.Tensor, eps: float,
                   emb: Optional[torch.Tensor] = None, ids: Optional[torch.Tensor] = None, offset: int = 0,
                   live: Optional[torch.Tensor] = None) -> torch.Tensor:
    """A T5 sublayer boundary (rqb200_t5dec_add_norm), one launch: x += delta in place -- or, with emb [V, D], x = emb[ids + offset]
    (ids int64 [R], any stride; emb[0] for every row when ids is None) -- then out = T5LayerNorm(x) * weight.  x, out [R, D]
    contiguous fp32.  Returns out.  ``live`` (int32 on the device, rqb200_t5dec_add_norm_counted): R is a capacity and only rows
    below live[0] are read and written."""
    _need_cuda(x, delta, weight, out, emb, ids)
    R, D = x.shape
    for name, t in (("x", x), ("out", out)):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.shape != (R, D):
            raise ValueError(f"{name} must be a contiguous fp32 [{R}, {D}] tensor")
    weight = _f32c(weight)
    if weight.shape != (D,):
        raise ValueError(f"weight {tuple(weight.shape)} must be [{D}]")
    if delta is not None:
        delta = _rows_of(delta, D, "delta")
        if delta.shape[0] != R:
            raise ValueError(f"delta has {delta.shape[0]} rows, x {R}")
    if emb is not None:
        emb = _f32c(emb)
        if emb.dim() != 2 or emb.shape[1] != D:
            raise ValueError(f"emb {tuple(emb.shape)} must be [V, {D}]")
    if ids is not None:
        if ids.dtype != torch.int64 or ids.shape != (R,):
            raise ValueError(f"ids must be int64 [{R}]")
    args = (_p(x), _p(delta), delta.stride(0) if delta is not None else 0, _p(emb), _p(ids), ids.stride(0) if ids is not None else 0,
            int(offset), emb.shape[0] if emb is not None else 0, _p(weight), R)
    with torch.cuda.device(x.device):
        if live is None:
            _lib.check(_lib.load().rqb200_t5dec_add_norm(*args, D, float(eps), _p(out), _stream()), "t5dec_add_norm")
        else:
            _lib.check(_lib.load().rqb200_t5dec_add_norm_counted(*args, _p(_live(live)), D, float(eps), _p(out), _stream()),
                       "t5dec_add_norm_counted")
    _count(1)
    return out


# ---------------------------------------------------------------------------------------------- exact ranking (csrc/t5rank.cu)
def _int32_vec(t: torch.Tensor, n: int, what: str) -> torch.Tensor:
    if t.dtype != torch.int32 or t.dim() != 1 or t.shape[0] < n or not t.is_contiguous():
        raise ValueError(f"{what} must be a contiguous int32 vector of at least {n} entries")
    return t


def t5rank_cross_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, offsets: torch.Tensor,
                           key_mask: Optional[torch.Tensor], Q: int, heads: int, tf32: bool = False) -> torch.Tensor:
    """T5 cross-attention of Q queries per history (rqb200_t5rank_cross_attention, fp32 on the CUDA cores, or with ``tf32``
    rqb200_t5rank_cross_attention_tc, the products on the TF32 tensor cores), one launch.  q [B * Q, heads * 64] (history b
    owns rows b * Q ...), k / v [rows, heads * 64] (any row stride, equal), history b's keys rows offsets[b] .. offsets[b + 1] - 1
    (int32 [B + 1], absolute), key_mask fp32 [rows] added to the scores (None: 0) -> [B * Q, heads * 64]."""
    _need_cuda(q, k, v, offsets, key_mask)
    inner = heads * T5_DKV
    q, k, v = _rows_of(q, inner, "q"), _rows_of(k, inner, "k"), _rows_of(v, inner, "v")
    if Q <= 0 or q.shape[0] % Q:
        raise ValueError(f"q has {q.shape[0]} rows, not a multiple of Q = {Q}")
    B = q.shape[0] // Q
    _int32_vec(offsets, B + 1, "offsets")
    if k.shape != v.shape:
        raise ValueError(f"k {tuple(k.shape)} and v {tuple(v.shape)} must have one shape")
    if k.stride(0) != v.stride(0):
        k, v = k.contiguous(), v.contiguous()
    if key_mask is not None:
        key_mask = _f32c(key_mask)
        if key_mask.dim() != 1 or key_mask.shape[0] != k.shape[0]:
            raise ValueError(f"key_mask {tuple(key_mask.shape)} must be [{k.shape[0]}], one entry per key row")
    if tf32 and any(t.data_ptr() % 16 or t.stride(0) % 4 for t in (q, k)):
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
    out = torch.empty((q.shape[0], inner), dtype=torch.float32, device=q.device)
    name = "t5rank_cross_attention_tc" if tf32 else "t5rank_cross_attention"
    with torch.cuda.device(q.device):
        _lib.check(getattr(_lib.load(), "rqb200_" + name)(_p(q), q.stride(0), _p(k), _p(v), k.stride(0), _p(offsets), _p(key_mask),
                                                          B, Q, heads, _p(out), out.stride(0), _stream()), name)
    _count(1)
    return out


def t5rank_children(logits: torch.Tensor, parent: Optional[torch.Tensor], child: torch.Tensor, code: torch.Tensor, n_h: int,
                    out: torch.Tensor, bad: Optional[torch.Tensor] = None, live: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Child scores of one trie level (rqb200_t5rank_children), one launch: logits [B * n_h, K] of the level's node rows, parent
    fp32 [B * n_h] (the nodes' scores; None: 0), child int32 [n_h + 1], code int32 [n_next] -> out fp32 [B, n_next] (written):
    out[b, j] = (logits[b * n_h + i, code[j]] - lse) + parent[b * n_h + i] for every child j of node i.  ``bad`` (int32, on the
    device) is ADDED the rows holding a NaN or +inf logit or all -inf; their children score NaN.  ``live`` (int32 [2] on the
    device, rqb200_t5rank_children_counted): one group (n_h = R) of capacity R whose rows are the first live[0], with live[1] <=
    n_next children."""
    _need_cuda(logits, parent, child, code, out, bad)
    logits = _rows(logits)
    R, K = logits.shape
    if n_h <= 0 or R % n_h:
        raise ValueError(f"logits has {R} rows, not a multiple of n_h = {n_h}")
    B = R // n_h
    _int32_vec(child, n_h + 1, "child")
    n_next = code.shape[0]
    _int32_vec(code, n_next, "code")
    if out.dtype != torch.float32 or out.shape != (B, n_next) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous fp32 [{B}, {n_next}] tensor")
    if parent is not None:
        parent = _f32c(parent).reshape(-1)
        if parent.shape[0] != R:
            raise ValueError(f"parent has {parent.shape[0]} entries, logits {R} rows")
    if bad is not None and (bad.dtype != torch.int32 or bad.numel() < 1 or not bad.is_contiguous()):
        raise ValueError("bad must be a contiguous int32 tensor")
    with torch.cuda.device(logits.device):
        if live is None:
            _lib.check(_lib.load().rqb200_t5rank_children(_p(logits), logits.stride(0), R, K, n_h, _p(parent), _p(child), _p(code),
                                                          n_next, _p(out), _p(bad), _stream()), "t5rank_children")
        else:
            if n_h != R or _live(live).numel() < 2:
                raise ValueError("t5rank_children: a device count takes one group (n_h = R) and live [rows, children]")
            _lib.check(_lib.load().rqb200_t5rank_children_counted(_p(logits), logits.stride(0), R, K, _p(parent), _p(child), _p(code),
                                                                  n_next, _p(live), _p(out), _p(bad), _stream()),
                       "t5rank_children_counted")
    _count(1)
    return out


def t5rank_select(scores: torch.Tensor, row: torch.Tensor, start: torch.Tensor, t_leaf: torch.Tensor, t_dedup: torch.Tensor,
                  n: int, exclude: Optional[SidExclusion] = None):
    """The n best items of each history from its leaf scores (rqb200_t5rank_select), one launch.  scores fp32 [B, U] (leaf u =
    item-table tuple u), (row, start) = ``SidItemTable.arrays()``, t_leaf / t_dedup int64 [B] (the target's tuple, -1 when it has
    none, and dedup rank) -> (items int64 [B, n], item scores fp32 [B, n], target rank int64 [B]): items by score descending, then
    tuple, then dedup rank, NaN last; -1 / -inf pad; rank -1 when the target is not ranked.  n <= 1024.  ``exclude``
    (``sid_exclusion_build`` on the same table): the history's excluded items are skipped and the rank counts only the items
    that are not excluded (-1 when the target is excluded)."""
    _need_cuda(scores, row, start, t_leaf, t_dedup)
    scores = _f32c(scores)
    if scores.dim() != 2:
        raise ValueError(f"scores {tuple(scores.shape)} must be [B, U]")
    B, U = scores.shape
    _int32_vec(start, U + 1, "start")
    _int32_vec(row, 0, "row")
    t_leaf = t_leaf.to(torch.int64).reshape(-1).contiguous()
    t_dedup = t_dedup.to(torch.int64).reshape(-1).contiguous()
    if t_leaf.shape[0] != B or t_dedup.shape[0] != B:
        raise ValueError(f"t_leaf / t_dedup must have B = {B} entries")
    n = int(n)
    dev = scores.device
    items = torch.empty((B, n), dtype=torch.int64, device=dev)
    item_scores = torch.empty((B, n), dtype=torch.float32, device=dev)
    rank = torch.empty((B,), dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        if exclude is None:
            _lib.check(_lib.load().rqb200_t5rank_select(_p(scores), B, U, _p(row), _p(start), _p(t_leaf), _p(t_dedup), n,
                                                        _p(items), _p(item_scores), _p(rank), _stream()), "t5rank_select")
        else:
            _lib.check(_lib.load().rqb200_t5rank_select_excluding(_p(scores), B, U, _p(row), _p(start), _p(t_leaf), _p(t_dedup), n,
                                                                  _p(items), _p(item_scores), _p(rank),
                                                                  *exclude.args(B, 0, "t5rank_select"), _stream()),
                       "t5rank_select_excluding")
    _count(1)
    return items, item_scores, rank


#: most candidate tuples per history t5score_trie_build takes (its block sort holds them in shared memory)
SCORE_MAX_CANDIDATES = 4096


class CandidateTrie(NamedTuple):
    """The trie of each history's own candidate tuples (``t5score_trie_build``).  counts int32 [B, H]: entry l - 1 the node count
    n_l of level l; code / parent int32 [B, H, C]: entry (l - 1, i) node i's last id and its node in level l - 1 (0, 0 for
    i >= n_l); child int32 [B, H, C + 1]: entry (l, i) for l < H the start of node i's children in level l + 1 (n_{l + 1} for
    i >= n_l, so node i's children are child[l][i] .. child[l][i + 1] - 1); leaf int32 [B, C]: each candidate's node in level H,
    -1 when it holds an id outside [0, K).  Nodes of one level are in lexicographic order of their prefixes."""
    counts: torch.Tensor
    code: torch.Tensor
    parent: torch.Tensor
    child: torch.Tensor
    leaf: torch.Tensor


def t5score_trie_build(ids: torch.Tensor, K: int) -> CandidateTrie:
    """The candidate trie of every history (rqb200_t5score_trie_build), one launch: ids integer [B, C, H] (C candidate tuples per
    history) over K codes per level.  C <= ``SCORE_MAX_CANDIDATES``, H <= 8, H * bits(K - 1) <= 62."""
    _need_cuda(ids)
    if ids.dim() != 3 or ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
        raise ValueError(f"ids must be an integer [B, C, H] tensor, got {ids.dtype} {tuple(ids.shape)}")
    B, C, H = ids.shape
    ids = ids.to(torch.int64).contiguous()
    dev = ids.device
    counts = torch.empty((B, H), dtype=torch.int32, device=dev)
    code = torch.empty((B, H, C), dtype=torch.int32, device=dev)
    parent = torch.empty((B, H, C), dtype=torch.int32, device=dev)
    child = torch.empty((B, H, C + 1), dtype=torch.int32, device=dev)
    leaf = torch.empty((B, C), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().rqb200_t5score_trie_build(_p(ids), B, C, H, int(K), _p(counts), _p(code), _p(parent), _p(child),
                                                         _p(leaf), _stream()), "t5score_trie_build")
    _count(1)
    return CandidateTrie(counts, code, parent, child, leaf)


# ---------------------------------------------------------------------------------------------- fused T5 encoder pass
def t5enc_len(n: int, H: int, sep: bool, user: bool) -> int:
    """Positions of the encoder input of n = items * H ids: the user row, then per item its H ids and a separator."""
    return int(user) + n // H * (H + int(sep))


def t5enc_offsets(mask: torch.Tensor, H: int, sep: bool, user: bool):
    """The kept positions of each history (rqb200_t5enc_offsets), one launch.  mask [B, n] (nonzero keeps the id; a separator
    follows the mask of its item's last id, the user row is always kept; a history with nothing kept keeps every position) ->
    (offsets int32 [B + 1], history b owning packed rows offsets[b] .. offsets[b + 1] - 1, and key_mask fp32 [B]: 0, or
    -FLT_MAX for a history without an unmasked position)."""
    _need_cuda(mask)
    mask = _f32c(mask)
    if mask.dim() != 2 or mask.shape[1] % H:
        raise ValueError(f"mask {tuple(mask.shape)} must be [B, items * {H}]")
    B, n = mask.shape
    offsets = torch.empty(B + 1, dtype=torch.int32, device=mask.device)
    key_mask = torch.empty(B, dtype=torch.float32, device=mask.device)
    with torch.cuda.device(mask.device):
        _lib.check(_lib.load().rqb200_t5enc_offsets(_p(mask), B, n, H, int(sep), int(user), _p(offsets), _p(key_mask), _stream()),
                   "t5enc_offsets")
    _count(1)
    return offsets, key_mask


def t5enc_assemble(mask: torch.Tensor, ids: torch.Tensor, user_ids: Optional[torch.Tensor], item_table: torch.Tensor,
                   sep_row: Optional[torch.Tensor], user_table: Optional[torch.Tensor], K: int, H: int, offsets: torch.Tensor,
                   n_kept: int, weight: torch.Tensor, eps: float):
    """The packed encoder input and its first T5LayerNorm (rqb200_t5enc_assemble), one launch.  mask / ids [B, n] (ids int64, any
    row stride), user_ids int64 [B, *] (column 0 is read) with user_table [U, D], or both None; item_table [V, D]; sep_row [D] or
    None; offsets from ``t5enc_offsets`` with n_kept = offsets[B].  Returns x, out [n_kept, D] (the input rows and
    T5LayerNorm(x) * weight), src int32 [n_kept] (b * S + p of each packed row) and slot int32 [B, S] (packed row or -1)."""
    return _t5enc_assemble("t5enc_assemble", mask, ids, user_ids, item_table, sep_row, user_table, K, H, offsets, n_kept, weight,
                           eps)


def t5enc_assemble_capacity(mask: torch.Tensor, ids: torch.Tensor, user_ids: Optional[torch.Tensor], item_table: torch.Tensor,
                            sep_row: Optional[torch.Tensor], user_table: Optional[torch.Tensor], K: int, H: int,
                            offsets: torch.Tensor, weight: torch.Tensor, eps: float):
    """``t5enc_assemble`` without N (rqb200_t5enc_assemble_capacity), one launch, for a pass that cannot read offsets[B] on the
    host (a CUDA-graph capture): x, out and src hold B * S rows, rows offsets[B] .. B * S - 1 being x = out = 0 and src = -1.
    The attention kernels neither read nor write those rows, and ``t5dec_add_norm`` keeps a zero row zero."""
    B, n = mask.shape
    rows = B * t5enc_len(n, H, sep_row is not None, user_table is not None)
    return _t5enc_assemble("t5enc_assemble_capacity", mask, ids, user_ids, item_table, sep_row, user_table, K, H, offsets, rows,
                           weight, eps)


def _t5enc_assemble(name, mask, ids, user_ids, item_table, sep_row, user_table, K, H, offsets, n_kept, weight, eps):
    _need_cuda(mask, ids, user_ids, item_table, sep_row, user_table, offsets, weight)
    if (user_ids is None) != (user_table is None):
        raise ValueError("user_ids and user_table go together")
    mask = _f32c(mask)
    B, n = mask.shape
    if ids.dtype != torch.int64 or ids.shape != (B, n) or ids.stride(1) != 1:
        ids = ids.to(torch.int64).contiguous()
        if ids.shape != (B, n):
            raise ValueError(f"ids {tuple(ids.shape)} must be [{B}, {n}] like the mask")
    item_table = _f32c(item_table)
    D = item_table.shape[1]
    if user_ids is not None:
        if user_ids.dtype != torch.int64:
            user_ids = user_ids.to(torch.int64)
        if user_ids.dim() != 2 or user_ids.shape[0] != B:
            raise ValueError(f"user_ids {tuple(user_ids.shape)} must be [{B}, *]")
        user_table = _f32c(user_table)
        if user_table.dim() != 2 or user_table.shape[1] != D:
            raise ValueError(f"user_table {tuple(user_table.shape)} must be [U, {D}]")
    if sep_row is not None:
        sep_row = _f32c(sep_row).reshape(-1)
        if sep_row.shape != (D,):
            raise ValueError(f"sep_row must hold {D} values")
    weight = _f32c(weight)
    if weight.shape != (D,):
        raise ValueError(f"weight {tuple(weight.shape)} must be [{D}]")
    if offsets.dtype != torch.int32 or offsets.shape != (B + 1,):
        raise ValueError(f"offsets must be int32 [{B + 1}]")
    S = t5enc_len(n, H, sep_row is not None, user_table is not None)
    x = torch.empty((n_kept, D), dtype=torch.float32, device=mask.device)
    out = torch.empty_like(x)
    src = torch.empty(n_kept, dtype=torch.int32, device=mask.device)
    slot = torch.empty((B, S), dtype=torch.int32, device=mask.device)
    with torch.cuda.device(mask.device):
        _lib.check(getattr(_lib.load(), "rqb200_" + name)(
            _p(mask), _p(ids), ids.stride(0), _p(user_ids), user_ids.stride(0) if user_ids is not None else 0, _p(item_table),
            item_table.shape[0], _p(sep_row), _p(user_table), user_table.shape[0] if user_table is not None else 0, int(K), B, n, H,
            D, _p(offsets), _p(weight), float(eps), _p(x), _p(out), _p(src), _p(slot), _stream()), name)
    _count(1)
    return x, out, src, slot


def t5enc_rel_bias(bias: torch.Tensor) -> torch.Tensor:
    """[heads, 2S - 1] from HF's compute_bias(S, S)[0] ([heads, S, S], a function of key - query position only): entry t is the
    bias of distance t - (S - 1)."""
    return torch.cat([bias[:, 1:, 0].flip(1), bias[:, 0, :]], dim=1).contiguous()


def t5enc_attention(qkv: torch.Tensor, src: torch.Tensor, offsets: torch.Tensor, key_mask: torch.Tensor, rel: torch.Tensor,
                    S: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Bidirectional T5 self-attention among each history's packed rows (rqb200_t5enc_attention), one launch.  qkv [N, 3 inner]
    (q | k | v), src / offsets / key_mask as ``t5enc_assemble`` / ``t5enc_offsets`` give them, rel [heads, 2S - 1] from
    ``t5enc_rel_bias`` -> [N, inner].  ``out``: a contiguous fp32 [N, inner] tensor to write instead of a new one; its rows past
    offsets[B] (``t5enc_assemble_capacity``'s) are not written and keep their values."""
    return _t5enc_attention_eval("t5enc_attention", qkv, src, offsets, key_mask, rel, S, out)


def t5enc_attention_tc(qkv: torch.Tensor, src: torch.Tensor, offsets: torch.Tensor, key_mask: torch.Tensor, rel: torch.Tensor,
                       S: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``t5enc_attention`` with its products on TF32 tensor cores (rqb200_t5enc_attention_tc, csrc/t5enc_tc.cu), one launch."""
    return _t5enc_attention_eval("t5enc_attention_tc", qkv, src, offsets, key_mask, rel, S, out)


def _rows_of16(t: torch.Tensor, width: int, what: str) -> torch.Tensor:
    """``_rows_of`` for the encoder attention kernels' 16-byte row loads: a copy when the row pitch or the base is not aligned."""
    t = _rows_of(t, width, what)
    return t.contiguous() if t.stride(0) % 4 or t.data_ptr() % 16 else t


def _t5enc_attention_eval(name, qkv, src, offsets, key_mask, rel, S, out=None):
    _need_cuda(qkv, src, offsets, key_mask, rel, out)
    rel = _f32c(rel)
    heads = rel.shape[0]
    if rel.shape != (heads, 2 * S - 1):
        raise ValueError(f"rel {tuple(rel.shape)} must be [heads, {2 * S - 1}]")
    inner = heads * T5_DKV
    qkv = _rows_of16(qkv, 3 * inner, "qkv")
    B = offsets.shape[0] - 1
    if offsets.dtype != torch.int32 or src.dtype != torch.int32 or src.shape != (qkv.shape[0],) or key_mask.shape != (B,):
        raise ValueError("src must be int32 [N] with N = qkv rows, offsets int32 [B + 1], key_mask [B]")
    key_mask = _f32c(key_mask)
    if out is None:
        out = torch.empty((qkv.shape[0], inner), dtype=torch.float32, device=qkv.device)
    elif out.dtype != torch.float32 or out.shape != (qkv.shape[0], inner) or not out.is_contiguous() or out.data_ptr() % 16:
        raise ValueError(f"out must be a contiguous, 16-byte aligned fp32 [{qkv.shape[0]}, {inner}] tensor")
    with torch.cuda.device(qkv.device):
        _lib.check(getattr(_lib.load(), "rqb200_" + name)(_p(qkv), qkv.stride(0), _p(src), _p(offsets), _p(key_mask), _p(rel), B,
                                                         S, heads, _p(out), out.stride(0), _stream()), name)
    _count(1)
    return out


def t5enc_scatter(rows: torch.Tensor, slot: torch.Tensor) -> torch.Tensor:
    """[B, S, D]: row slot[b, s] of rows [N, D], zeros where slot is -1 (rqb200_t5enc_scatter), one launch."""
    _need_cuda(rows, slot)
    rows = _f32c(rows)
    if slot.dtype != torch.int32 or slot.dim() != 2 or not slot.is_contiguous():
        raise ValueError("slot must be a contiguous int32 [B, S] tensor")
    B, S = slot.shape
    D = rows.shape[1]
    out = torch.empty((B, S, D), dtype=torch.float32, device=rows.device)
    with torch.cuda.device(rows.device):
        _lib.check(_lib.load().rqb200_t5enc_scatter(_p(rows), _p(slot), B * S, D, _p(out), _stream()), "t5enc_scatter")
    _count(1)
    return out


# ---------------------------------------------------------------------------------------------- training the T5 encoder pass
def t5enc_dropout_seed(device) -> torch.Tensor:
    """int64 [1] on the device: a fresh attention-dropout seed drawn from torch's generator of that device (no host read), so
    ``torch.manual_seed`` reproduces the keep bits."""
    return torch.empty(1, dtype=torch.int64, device=device).random_()


def _check_p(p: float) -> float:
    if not 0.0 <= p < 1.0:
        raise ValueError(f"dropout probability {p} must be in [0, 1)")
    return float(p)


def _check_seed(seed: torch.Tensor) -> None:
    if seed.dtype != torch.int64 or seed.numel() != 1:
        raise ValueError("seed must be an int64 tensor of one element")


def t5enc_dropout_keep(seed: torch.Tensor, p: float, B: int, heads: int, S: int) -> torch.Tensor:
    """uint8 [B, heads, S, S]: the attention-dropout keep bits (rqb200_t5enc_dropout_keep) that ``t5enc_attention_train`` applies
    with this seed, indexed by (history, head, query position, key position), one launch."""
    _need_cuda(seed)
    _check_seed(seed)
    keep = torch.empty((B, heads, S, S), dtype=torch.uint8, device=seed.device)
    with torch.cuda.device(seed.device):
        _lib.check(_lib.load().rqb200_t5enc_dropout_keep(_p(seed), _check_p(p), B, heads, S, _p(keep), _stream()),
                   "t5enc_dropout_keep")
    _count(1)
    return keep


def t5enc_attention_train(qkv: torch.Tensor, src: torch.Tensor, offsets: torch.Tensor, key_mask: torch.Tensor, rel: torch.Tensor,
                          S: int, seed: torch.Tensor, p: float):
    """``t5enc_attention`` with HF's attention-weight dropout (probability p, keep bits from ``seed``) that also returns the
    log-sum-exp the backward needs (rqb200_t5enc_attention_train), one launch -> (out [N, inner], lse [N, heads])."""
    return _t5enc_attention_train("t5enc_attention_train", qkv, src, offsets, key_mask, rel, S, seed, p)


def t5enc_attention_tc_train(qkv: torch.Tensor, src: torch.Tensor, offsets: torch.Tensor, key_mask: torch.Tensor,
                             rel: torch.Tensor, S: int, seed: torch.Tensor, p: float):
    """``t5enc_attention_train`` with its products on TF32 tensor cores (rqb200_t5enc_attention_tc_train), one launch; the same
    keep bits under the same seed."""
    return _t5enc_attention_train("t5enc_attention_tc_train", qkv, src, offsets, key_mask, rel, S, seed, p)


def _t5enc_attention_train(name, qkv, src, offsets, key_mask, rel, S, seed, p):
    _need_cuda(qkv, src, offsets, key_mask, rel, seed)
    rel = _f32c(rel)
    heads = rel.shape[0]
    if rel.shape != (heads, 2 * S - 1):
        raise ValueError(f"rel {tuple(rel.shape)} must be [heads, {2 * S - 1}]")
    qkv = _rows_of16(qkv, 3 * heads * T5_DKV, "qkv")
    B = offsets.shape[0] - 1
    if offsets.dtype != torch.int32 or src.dtype != torch.int32 or src.shape != (qkv.shape[0],) or key_mask.shape != (B,):
        raise ValueError("src must be int32 [N] with N = qkv rows, offsets int32 [B + 1], key_mask [B]")
    _check_seed(seed)
    key_mask = _f32c(key_mask)
    N = qkv.shape[0]
    out = torch.empty((N, heads * T5_DKV), dtype=torch.float32, device=qkv.device)
    lse = torch.empty((N, heads), dtype=torch.float32, device=qkv.device)
    with torch.cuda.device(qkv.device):
        _lib.check(getattr(_lib.load(), "rqb200_" + name)(_p(qkv), qkv.stride(0), _p(src), _p(offsets), _p(key_mask), _p(rel), B,
                                                         S, heads, _p(seed), _check_p(p), _p(out), out.stride(0), _p(lse),
                                                         _stream()), name)
    _count(1)
    return out, lse


def t5enc_attention_backward(qkv: torch.Tensor, out: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor, src: torch.Tensor,
                             offsets: torch.Tensor, key_mask: torch.Tensor, rel: torch.Tensor, S: int, seed: torch.Tensor, p: float):
    """The backward of ``t5enc_attention_train`` (rqb200_t5enc_attention_backward), two launches and one fixed-order sum ->
    (d_qkv [N, 3 inner], d_rel [heads, 2S - 1]).  Bit-reproducible."""
    return _t5enc_attention_backward("t5enc_attention_backward", qkv, out, dout, lse, src, offsets, key_mask, rel, S, seed, p)


def t5enc_attention_tc_backward(qkv: torch.Tensor, out: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor, src: torch.Tensor,
                                offsets: torch.Tensor, key_mask: torch.Tensor, rel: torch.Tensor, S: int, seed: torch.Tensor,
                                p: float):
    """The backward of ``t5enc_attention_tc_train`` on TF32 tensor cores (rqb200_t5enc_attention_tc_backward), two launches and
    one fixed-order sum -> (d_qkv [N, 3 inner], d_rel [heads, 2S - 1]).  Bit-reproducible."""
    return _t5enc_attention_backward("t5enc_attention_tc_backward", qkv, out, dout, lse, src, offsets, key_mask, rel, S, seed, p)


def _t5enc_attention_backward(name, qkv, out, dout, lse, src, offsets, key_mask, rel, S, seed, p):
    _need_cuda(qkv, out, dout, lse, src, offsets, key_mask, rel, seed)
    heads = rel.shape[0]
    inner = heads * T5_DKV
    qkv, out, dout = _rows_of16(qkv, 3 * inner, "qkv"), _rows_of16(out, inner, "out"), _rows_of16(dout, inner, "dout")
    lse, rel, key_mask = _f32c(lse), _f32c(rel), _f32c(key_mask)
    B, N = offsets.shape[0] - 1, qkv.shape[0]
    if out.shape[0] != N or dout.shape[0] != N or lse.shape != (N, heads) or rel.shape != (heads, 2 * S - 1):
        raise ValueError("out / dout [N, inner], lse [N, heads] and rel [heads, 2S - 1] must match qkv [N, 3 inner]")
    lib = _lib.load()
    tiles = getattr(lib, "rqb200_" + name + "_tiles")(S)
    delta = torch.empty((N, heads), dtype=torch.float32, device=qkv.device)
    dqkv = torch.empty((N, 3 * inner), dtype=torch.float32, device=qkv.device)
    part = torch.empty((B * tiles, heads, 2 * S - 1), dtype=torch.float32, device=qkv.device)
    with torch.cuda.device(qkv.device):
        _lib.check(getattr(lib, "rqb200_" + name)(_p(qkv), qkv.stride(0), _p(out), out.stride(0), _p(dout), dout.stride(0),
                                                 _p(lse), _p(src), _p(offsets), _p(key_mask), _p(rel), B, S, heads, _p(seed),
                                                 _check_p(p), _p(delta), _p(dqkv), dqkv.stride(0), _p(part), _stream()), name)
    _count(2)
    return dqkv, part.sum(0)


def t5enc_add_norm_fwd(x: torch.Tensor, delta: Optional[torch.Tensor], weight: torch.Tensor, eps: float):
    """Out-of-place add + T5LayerNorm (rqb200_t5enc_add_norm_fwd), one launch: x [R, D] and delta [R, D] or None ->
    (x_out = x + delta, out = T5LayerNorm(x_out) * weight, inv_rms [R])."""
    _need_cuda(x, delta, weight)
    x = _f32c(x)
    R, D = x.shape
    weight = _f32c(weight)
    if weight.shape != (D,):
        raise ValueError(f"weight {tuple(weight.shape)} must be [{D}]")
    if delta is not None:
        delta = _rows_of(delta, D, "delta")
        if delta.shape[0] != R:
            raise ValueError(f"delta has {delta.shape[0]} rows, x {R}")
    x_out, out = torch.empty_like(x), torch.empty_like(x)
    inv = torch.empty(R, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().rqb200_t5enc_add_norm_fwd(_p(x), _p(delta), delta.stride(0) if delta is not None else 0, _p(weight),
                                                         R, D, float(eps), _p(x_out), _p(out), _p(inv), _stream()),
                   "t5enc_add_norm_fwd")
    _count(1)
    return x_out, out, inv


def t5enc_add_norm_bwd(d_out: torch.Tensor, d_res: Optional[torch.Tensor], x_out: torch.Tensor, inv_rms: torch.Tensor,
                       weight: torch.Tensor):
    """The backward of ``t5enc_add_norm_fwd`` (rqb200_t5enc_add_norm_bwd), one launch and one fixed-order sum: d_out [R, D] (the
    norm output's gradient) and d_res [R, D] or None (x_out's own) -> (dx [R, D], the gradient of x and delta, d_weight [D])."""
    _need_cuda(d_out, d_res, x_out, inv_rms, weight)
    x_out, d_out, inv_rms, weight = _f32c(x_out), _f32c(d_out), _f32c(inv_rms), _f32c(weight)
    R, D = x_out.shape
    if d_res is not None:
        d_res = _f32c(d_res)
    for name, t in (("d_out", d_out), ("d_res", d_res)):
        if t is not None and t.shape != (R, D):
            raise ValueError(f"{name} {tuple(t.shape)} must be [{R}, {D}]")
    lib = _lib.load()
    dx = torch.empty_like(x_out)
    part = torch.empty((lib.rqb200_t5enc_add_norm_bwd_parts(R), D), dtype=torch.float32, device=x_out.device)
    with torch.cuda.device(x_out.device):
        _lib.check(lib.rqb200_t5enc_add_norm_bwd(_p(d_out), _p(d_res), _p(x_out), _p(inv_rms), _p(weight), R, D, _p(dx), _p(part),
                                                 _stream()), "t5enc_add_norm_bwd")
    _count(1)
    return dx, part.sum(0)


def _t5enc_attention_function(name: str, train, backward, doc: str):
    """The autograd.Function class ``name`` of a training attention whose kernels are the wrappers ``train`` and ``backward``."""

    def forward_(ctx, qkv, rel, src, offsets, key_mask, S, seed, p):
        qkv = qkv.contiguous()
        out, lse = train(qkv, src, offsets, key_mask, rel, S, seed, p)
        ctx.save_for_backward(qkv, rel, src, offsets, key_mask, seed, out, lse)
        ctx.S, ctx.p = S, p
        return out

    def backward_(ctx, dout):
        qkv, rel, src, offsets, key_mask, seed, out, lse = ctx.saved_tensors
        dqkv, drel = backward(qkv, out, dout, lse, src, offsets, key_mask, rel, ctx.S, seed, ctx.p)
        return dqkv, drel, None, None, None, None, None, None

    return type(name, (torch.autograd.Function,), {"forward": staticmethod(forward_), "backward": staticmethod(backward_),
                                                   "__doc__": doc, "__module__": __name__})


T5EncAttentionFunction = _t5enc_attention_function(
    "T5EncAttentionFunction", t5enc_attention_train, t5enc_attention_backward,
    "Autograd of the training attention: ``apply(qkv, rel, src, offsets, key_mask, S, seed, p)`` -> out [N, inner]; gradients "
    "for qkv and rel.")
T5EncAttentionTCFunction = _t5enc_attention_function(
    "T5EncAttentionTCFunction", t5enc_attention_tc_train, t5enc_attention_tc_backward,
    "``T5EncAttentionFunction`` on the TF32 tensor-core kernels (``t5enc_attention_tc_train`` / ``_tc_backward``), the same "
    "arguments and gradients.")


class T5EncAddNormFunction(torch.autograd.Function):
    """Autograd of the training add + norm: ``apply(x, delta, weight, eps)`` (delta may be None) -> (x_out, out)."""

    @staticmethod
    def forward(ctx, x, delta, weight, eps):
        x_out, out, inv = t5enc_add_norm_fwd(x, delta, weight, eps)
        ctx.save_for_backward(x_out, inv, weight)
        ctx.has_delta = delta is not None
        return x_out, out

    @staticmethod
    def backward(ctx, d_x_out, d_out):
        x_out, inv, weight = ctx.saved_tensors
        if d_out is None:
            d_out = torch.zeros_like(x_out)
        dx, dw = t5enc_add_norm_bwd(d_out, d_x_out, x_out, inv, weight)
        return dx, dx if ctx.has_delta else None, dw, None


# ---------------------------------------------------------------------------------------------- training the T5 decoder pass
def t5dec_self_attention_train(qkv: torch.Tensor, rel: torch.Tensor, T: int, seed: torch.Tensor, p: float):
    """Causal T5 self-attention of T decoder positions per history with HF's attention-weight dropout
    (rqb200_t5dec_self_attention_train), one launch.  qkv [B * T, 3 inner] (row b * T + t: position t of history b; q | k | v),
    rel [heads, 2T - 1] (``t5enc_rel_bias`` layout) -> (out [B * T, inner], lse [B * T, heads])."""
    _need_cuda(qkv, rel, seed)
    _check_seed(seed)
    rel = _f32c(rel)
    heads = rel.shape[0]
    if rel.shape != (heads, 2 * T - 1):
        raise ValueError(f"rel {tuple(rel.shape)} must be [heads, {2 * T - 1}]")
    qkv = _rows_of(qkv, 3 * heads * T5_DKV, "qkv")
    if qkv.shape[0] % T:
        raise ValueError(f"qkv has {qkv.shape[0]} rows, not a multiple of T = {T}")
    B = qkv.shape[0] // T
    out = torch.empty((B * T, heads * T5_DKV), dtype=torch.float32, device=qkv.device)
    lse = torch.empty((B * T, heads), dtype=torch.float32, device=qkv.device)
    with torch.cuda.device(qkv.device):
        _lib.check(_lib.load().rqb200_t5dec_self_attention_train(_p(qkv), qkv.stride(0), _p(rel), B, T, heads, _p(seed), _check_p(p),
                                                                 _p(out), out.stride(0), _p(lse), _stream()),
                   "t5dec_self_attention_train")
    _count(1)
    return out, lse


def t5dec_self_attention_backward(qkv: torch.Tensor, out: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor, rel: torch.Tensor,
                                  T: int, seed: torch.Tensor, p: float):
    """The backward of ``t5dec_self_attention_train`` (rqb200_t5dec_self_attention_backward), one launch and one fixed-order sum ->
    (d_qkv [B * T, 3 inner], d_rel [heads, 2T - 1]).  Bit-reproducible."""
    _need_cuda(qkv, out, dout, lse, rel, seed)
    _check_seed(seed)
    rel = _f32c(rel)
    heads = rel.shape[0]
    inner = heads * T5_DKV
    qkv, out, dout, lse = _rows_of(qkv, 3 * inner, "qkv"), _rows_of(out, inner, "out"), _rows_of(dout, inner, "dout"), _f32c(lse)
    N = qkv.shape[0]
    if N % T or out.shape[0] != N or dout.shape[0] != N or lse.shape != (N, heads) or rel.shape != (heads, 2 * T - 1):
        raise ValueError("qkv [B * T, 3 inner], out / dout [B * T, inner], lse [B * T, heads] and rel [heads, 2T - 1] must match")
    B = N // T
    dqkv = torch.empty((N, 3 * inner), dtype=torch.float32, device=qkv.device)
    part = torch.empty((B, heads, 2 * T - 1), dtype=torch.float32, device=qkv.device)
    with torch.cuda.device(qkv.device):
        _lib.check(_lib.load().rqb200_t5dec_self_attention_backward(
            _p(qkv), qkv.stride(0), _p(out), out.stride(0), _p(dout), dout.stride(0), _p(lse), _p(rel), B, T, heads, _p(seed),
            _check_p(p), _p(dqkv), dqkv.stride(0), _p(part), _stream()), "t5dec_self_attention_backward")
    _count(1)
    return dqkv, part.sum(0)


def _cross_layout(q, kv, offsets, key_mask, src, T, heads):
    inner = heads * T5_DKV
    q, kv = _rows_of(q, inner, "q"), _rows_of(kv, 2 * inner, "kv")
    if q.shape[0] % T:
        raise ValueError(f"q has {q.shape[0]} rows, not a multiple of T = {T}")
    B = q.shape[0] // T
    if offsets.dtype != torch.int32 or offsets.shape != (B + 1,):
        raise ValueError(f"offsets must be int32 [{B + 1}]")
    key_mask = _f32c(key_mask)
    if key_mask.shape != (kv.shape[0],):
        raise ValueError(f"key_mask {tuple(key_mask.shape)} must hold one value per key row ({kv.shape[0]})")
    if src is not None and (src.dtype != torch.int32 or src.shape != (kv.shape[0],) or not src.is_contiguous()):
        raise ValueError(f"src must be a contiguous int32 [{kv.shape[0]}] tensor")
    return q, kv, key_mask, B


def t5dec_cross_attention_train(q: torch.Tensor, kv: torch.Tensor, offsets: torch.Tensor, key_mask: torch.Tensor,
                                src: Optional[torch.Tensor], S: int, T: int, seed: torch.Tensor, p: float):
    """T5 cross-attention of T decoder positions per history over its encoder rows, with HF's attention-weight dropout
    (rqb200_t5dec_cross_attention_train), one launch.  q [B * T, inner]; kv [rows, 2 inner] (k | v); history b's keys are rows
    offsets[b] .. offsets[b + 1] - 1 (int32 [B + 1]) with additive key_mask [rows] (0 or finfo(float32).min); a key's position in
    the dropout bits is src[row] - b * S (packed encoder rows) or row - offsets[b] (src None: [B * S] rows).
    -> (out [B * T, inner], lse [B * T, heads])."""
    _need_cuda(q, kv, offsets, key_mask, src, seed)
    _check_seed(seed)
    heads = q.shape[1] // T5_DKV
    q, kv, key_mask, B = _cross_layout(q, kv, offsets, key_mask, src, T, heads)
    inner = heads * T5_DKV
    out = torch.empty((B * T, inner), dtype=torch.float32, device=q.device)
    lse = torch.empty((B * T, heads), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        _lib.check(_lib.load().rqb200_t5dec_cross_attention_train(
            _p(q), q.stride(0), _p(kv), kv.data_ptr() + 4 * inner, kv.stride(0), _p(offsets), _p(key_mask), _p(src), B, int(S), T,
            heads, _p(seed), _check_p(p), _p(out), out.stride(0), _p(lse), _stream()), "t5dec_cross_attention_train")
    _count(1)
    return out, lse


def t5dec_cross_attention_backward(q: torch.Tensor, kv: torch.Tensor, out: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor,
                                   offsets: torch.Tensor, key_mask: torch.Tensor, src: Optional[torch.Tensor], S: int, T: int,
                                   seed: torch.Tensor, p: float):
    """The backward of ``t5dec_cross_attention_train`` (rqb200_t5dec_cross_attention_backward), one launch -> (d_q [B * T, inner],
    d_kv [rows, 2 inner], zero in rows no history owns).  Bit-reproducible."""
    _need_cuda(q, kv, out, dout, lse, offsets, key_mask, src, seed)
    _check_seed(seed)
    heads = q.shape[1] // T5_DKV
    q, kv, key_mask, B = _cross_layout(q, kv, offsets, key_mask, src, T, heads)
    inner = heads * T5_DKV
    out, dout, lse = _rows_of(out, inner, "out"), _rows_of(dout, inner, "dout"), _f32c(lse)
    if out.shape[0] != B * T or dout.shape[0] != B * T or lse.shape != (B * T, heads):
        raise ValueError("out / dout [B * T, inner] and lse [B * T, heads] must match q")
    dq = torch.empty_like(out)
    dkv = torch.zeros((kv.shape[0], 2 * inner), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        _lib.check(_lib.load().rqb200_t5dec_cross_attention_backward(
            _p(q), q.stride(0), _p(kv), kv.data_ptr() + 4 * inner, kv.stride(0), _p(out), out.stride(0), _p(dout), dout.stride(0),
            _p(lse), _p(offsets), _p(key_mask), _p(src), B, int(S), T, heads, _p(seed), _check_p(p), _p(dq), dq.stride(0), _p(dkv),
            dkv.data_ptr() + 4 * inner, dkv.stride(0), _stream()), "t5dec_cross_attention_backward")
    _count(1)
    return dq, dkv


class T5DecSelfAttentionFunction(torch.autograd.Function):
    """Autograd of the decoder's training self-attention: ``apply(qkv, rel, T, seed, p)`` -> out [B * T, inner]; gradients for
    qkv and rel."""

    @staticmethod
    def forward(ctx, qkv, rel, T, seed, p):
        qkv = qkv.contiguous()
        out, lse = t5dec_self_attention_train(qkv, rel, T, seed, p)
        ctx.save_for_backward(qkv, rel, seed, out, lse)
        ctx.T, ctx.p = T, p
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, rel, seed, out, lse = ctx.saved_tensors
        dqkv, drel = t5dec_self_attention_backward(qkv, out, dout, lse, rel, ctx.T, seed, ctx.p)
        return dqkv, drel, None, None, None


class T5DecCrossAttentionFunction(torch.autograd.Function):
    """Autograd of the decoder's training cross-attention: ``apply(q, kv, offsets, key_mask, src, S, T, seed, p)`` -> out
    [B * T, inner]; gradients for q and kv."""

    @staticmethod
    def forward(ctx, q, kv, offsets, key_mask, src, S, T, seed, p):
        q, kv = q.contiguous(), kv.contiguous()
        out, lse = t5dec_cross_attention_train(q, kv, offsets, key_mask, src, S, T, seed, p)
        ctx.save_for_backward(q, kv, offsets, key_mask, src, seed, out, lse)
        ctx.S, ctx.T, ctx.p = S, T, p
        return out

    @staticmethod
    def backward(ctx, dout):
        q, kv, offsets, key_mask, src, seed, out, lse = ctx.saved_tensors
        dq, dkv = t5dec_cross_attention_backward(q, kv, out, dout, lse, offsets, key_mask, src, ctx.S, ctx.T, seed, ctx.p)
        return dq, dkv, None, None, None, None, None, None, None


# ---------------------------------------------------------------------------------------------- tensor-core tokeniser
def tc_supported(D: int, K: int, L: int) -> bool:
    return bool(_lib.load().rqb200_tokenize_tc_supported(D, K, L))


TC_PAD = 64   # the wgmma tokeniser wants D % 64 == 0: narrower / odd widths are zero-padded (exact for every dot product)


def tc_padded_dim(D: int, K: int, L: int) -> int:
    """Width the tensor-core tokeniser runs a D-wide quantiser at (D itself, or D zero-padded to the next multiple of 64);
    0 when the shape cannot use it at all (K not one of 256, 512, ..., 2048; D > 768; L > 8)."""
    Dp = (D + TC_PAD - 1) // TC_PAD * TC_PAD
    return Dp if tc_supported(Dp, K, L) else 0


class TcState:
    """Device-side prepared codebooks for the wgmma tokeniser (fp16 images, measured rounding norms, float64 Gram
    tables, an fp32 copy for the exact re-rank).  Owns everything it needs: the caller's tensors are not referenced after
    construction.  Codebooks narrower than a multiple of 64 are zero-padded (``self.D`` is the padded width,
    ``self.D_in`` the caller's)."""

    def __init__(self, codebooks: Sequence[torch.Tensor]):
        lib = _lib.load()
        cbs = _check_codebooks(codebooks, codebooks[0].shape[1])
        _need_cuda(*cbs)
        self.K, self.D_in = cbs[0].shape
        self.L = len(cbs)
        self.D = tc_padded_dim(self.D_in, self.K, self.L)
        if not self.D:
            raise _lib.Rqb200Error(f"wgmma tokeniser does not support D={self.D_in} K={self.K} L={self.L}")
        if self.D != self.D_in:
            cbs = [torch.nn.functional.pad(c, (0, self.D - self.D_in)) for c in cbs]
        self.device = cbs[0].device
        nbytes = lib.rqb200_tokenize_tc_state_bytes(self.D, self.K, self.L)
        self.buf = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        self.nbytes = nbytes
        with torch.cuda.device(self.device):
            _lib.check(lib.rqb200_tokenize_tc_prepare(_ptr_array(cbs), self.D, self.K, self.L, _p(self.buf), nbytes,
                                                      _stream()), "tokenize_tc_prepare")
        _count(7 + self.L * (self.L - 1) // 2)
        global TC_PREPARES
        TC_PREPARES += 1


def rq_tokenize_tc(x: torch.Tensor, codebooks=None, state: Optional[TcState] = None, stats=None) -> torch.Tensor:
    """sem_ids [B,L] int64 via the wgmma candidate filter + exact fp32 re-rank (csrc/rq_tcx.cu).  Same result contract as
    ``rq_tokenize``: the filter's margin is a deterministic bound on the fp16 rounding, every row with more
    than one candidate inside it is re-scored with the exact kernel's fp32 arithmetic."""
    _need_cuda(x)
    lib = _lib.load()
    if state is None:
        state = TcState(codebooks)
    x = _rows(x)
    B, D = x.shape
    if D != state.D_in:
        raise _lib.Rqb200Error(f"rq_tokenize_tc: x has {D} columns, the prepared state was built for {state.D_in}")
    if x.device != state.device:
        raise _lib.Rqb200Error(f"rq_tokenize_tc: x is on {x.device}, the prepared state on {state.device}")
    if D != state.D:
        x = torch.nn.functional.pad(x, (0, state.D - D))
    if x.data_ptr() % 16 or x.stride(0) % 4:        # the kernel bulk-copies x's rows: 16-byte aligned base and row pitch
        x = x.contiguous()
    ids = torch.empty((B, state.L), dtype=torch.int64, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(lib.rqb200_tokenize_tc_run(_p(x), x.stride(0), B, _p(state.buf), state.D, state.K, state.L, _p(ids),
                                              _p(stats), _stream()), "tokenize_tc_run")
    _count(1)
    global TC_CALLS
    TC_CALLS += 1
    return ids


# frozen-codebook cache of prepared states behind the module API (RqVae.tokenize / SemanticIdTokenizer): keyed on the
# identity AND version of every codebook tensor, so an optimiser step (in-place update bumps ._version) or a reloaded
# checkpoint re-prepares; a handful of entries is plenty (one model per process in the reference's scripts)
_TC_CACHE: "dict[tuple, tuple]" = {}
_TC_CACHE_MAX = 4
#: rows below which the exact CUDA-core kernel is used even when the tensor-core path is available (one 128-row tile keeps
#: 2 of 132 SMs busy; the prepare step runs again whenever the cache misses)
TC_MIN_ROWS = 1024


def _tc_cache_key(codebooks: Sequence[torch.Tensor]):
    return tuple((c.data_ptr(), c._version, tuple(c.shape), c.device.index) for c in codebooks)


def tc_state_for(codebooks: Sequence[torch.Tensor]) -> TcState:
    # an entry also remembers the tensor OBJECTS (weak references): a derived codebook (sim_vq projection, normalised rows) is a
    # temporary whose address the allocator may hand to the next call's temporary with the same version counter
    if _NO_OPERAND_CACHE or torch.cuda.is_current_stream_capturing():
        return TcState(codebooks)                # a captured graph re-prepares on every replay (see split_operand_cached)
    key = _tc_cache_key(codebooks)
    hit = _TC_CACHE.get(key)
    if hit is not None and all(r() is c for r, c in zip(hit[0], codebooks)):
        hit[2].ready()
        return hit[1]
    if len(_TC_CACHE) >= _TC_CACHE_MAX:
        _TC_CACHE.pop(next(iter(_TC_CACHE)))
    st = TcState(codebooks)
    _TC_CACHE[key] = ([weakref.ref(c) for c in codebooks], st, StreamBuild(st.buf))
    return st


def rq_tokenize_auto(x: torch.Tensor, codebooks: Sequence[torch.Tensor], stats=None) -> torch.Tensor:
    """What the module API calls (RqVae.tokenize, SemanticIdTokenizer.precompute_corpus_ids, modules/rqvae.py:118-139 ids
    only): the tensor-core tokeniser with a cached prepared state whenever the shape allows (K = 256 m with m = 1..8,
    D <= 768 after zero-padding to a multiple of 64) and the batch is large enough to fill the GPU, else the exact CUDA-core
    kernel."""
    K, D = codebooks[0].shape
    if x.shape[0] >= TC_MIN_ROWS and not torch.is_grad_enabled() and tc_padded_dim(D, K, len(codebooks)):
        return rq_tokenize_tc(x, state=tc_state_for(codebooks), stats=stats)
    return rq_tokenize(x, codebooks)


# ---------------------------------------------------------------------------------------------- bf16 tensor-core MLP
def bf16_supported(dims) -> bool:
    """Every contraction dim (all but the last entry of [in, hidden..., out]) must be a multiple of 64."""
    return all(d % 64 == 0 for d in dims[:-1])


def to_bf16_image(x: torch.Tensor) -> torch.Tensor:
    """fp32 [rows, K] -> bf16 operand image (csrc/gemm_tc.cu); used for activations and for weights W[N, K]."""
    _need_cuda(x)
    lib = _lib.load()
    x = _rows(x)
    rows, K = x.shape
    nbytes = lib.rqb200_bf16_image_bytes(rows, K)
    if nbytes == 0 and rows:
        raise _lib.Rqb200Error(f"bf16 image needs K % 64 == 0, got K={K}")
    img = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(lib.rqb200_f32_to_bf16_image(_p(x), x.stride(0), rows, K, _p(img), _stream()), "f32_to_bf16_image")
    _count(1)
    return img


@torch.no_grad()
def mlp_forward_bf16(x: torch.Tensor, weights: Sequence[torch.Tensor], normalize: bool = False,
                     weight_images: Optional[Sequence[torch.Tensor]] = None) -> torch.Tensor:
    """modules/encoder.py:23-38 with bf16 wgmma GEMMs (fp32 accumulate, ReLU fused; activations stay in the bf16
    operand-image layout between layers).  Forward only, reduced precision: NOT index-exact vs the fp32 reference."""
    _need_cuda(x, *weights)
    lib = _lib.load()
    x = _rows(x)
    M = x.shape[0]
    dims = [x.shape[1]] + [w.shape[0] for w in weights]
    if not bf16_supported(dims):
        raise _lib.Rqb200Error(f"bf16 MLP needs every contraction dim to be a multiple of 64, got {dims}")
    if weight_images is None:
        weight_images = [to_bf16_image(w.detach()) for w in weights]
    a = to_bf16_image(x)
    n = len(weights)
    out = None
    with torch.cuda.device(x.device):
        for i, (w, wi) in enumerate(zip(weights, weight_images)):
            N, K = w.shape
            last = i == n - 1
            nxt = None
            if not last:
                nxt = torch.empty(lib.rqb200_bf16_image_bytes(M, N), dtype=torch.uint8, device=x.device)
            else:
                out = torch.empty((M, N), dtype=torch.float32, device=x.device)
            _lib.check(lib.rqb200_gemm_bf16(_p(a), _p(wi), M, N, K, int(not last), _p(nxt), _p(out) if last else 0,
                                            N if last else 0, _stream()), "gemm_bf16")
            _count(1)
            a = nxt
    return l2norm_rows(out) if normalize else out


# ---------------------------------------------------------------------------------------------- exact top-k search (csrc/t5rank.cu)
def t5rank_cross_attention_ragged(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, offsets: torch.Tensor,
                                  key_mask: Optional[torch.Tensor], tiles: torch.Tensor, heads: int,
                                  live: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``t5rank_cross_attention`` (fp32) over a ragged level (rqb200_t5rank_cross_attention_ragged), one launch: q [R, heads * 64]
    the level's query rows, tiles int32 [T, 3] (history b, first query row, query count <= 64; ``t5exact_frontier_write``), each
    tile's queries over history b's keys (k, v, offsets, key_mask as ``t5rank_cross_attention``) -> [R, heads * 64].  Each row
    gets the bits the uniform kernel gives it.  ``live`` (int32 on the device, rqb200_t5rank_cross_attention_ragged_counted): T is
    a capacity and only the first live[0] tiles run."""
    _need_cuda(q, k, v, offsets, key_mask, tiles)
    inner = heads * T5_DKV
    q, k, v = _rows_of(q, inner, "q"), _rows_of(k, inner, "k"), _rows_of(v, inner, "v")
    if tiles.dtype != torch.int32 or tiles.dim() != 2 or tiles.shape[1] != 3 or not tiles.is_contiguous():
        raise ValueError(f"tiles must be a contiguous int32 [T, 3] tensor, got {tiles.dtype} {tuple(tiles.shape)}")
    if offsets.dtype != torch.int32 or offsets.dim() != 1 or not offsets.is_contiguous():
        raise ValueError("offsets must be a contiguous int32 vector")
    if k.shape != v.shape:
        raise ValueError(f"k {tuple(k.shape)} and v {tuple(v.shape)} must have one shape")
    if k.stride(0) != v.stride(0):
        k, v = k.contiguous(), v.contiguous()
    if key_mask is not None:
        key_mask = _f32c(key_mask)
        if key_mask.dim() != 1 or key_mask.shape[0] != k.shape[0]:
            raise ValueError(f"key_mask {tuple(key_mask.shape)} must be [{k.shape[0]}], one entry per key row")
    out = torch.empty((q.shape[0], inner), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        if live is None:
            _lib.check(_lib.load().rqb200_t5rank_cross_attention_ragged(_p(q), q.stride(0), _p(k), _p(v), k.stride(0), _p(offsets),
                                                                        _p(key_mask), _p(tiles), tiles.shape[0], heads, _p(out),
                                                                        out.stride(0), _stream()), "t5rank_cross_attention_ragged")
        else:
            _lib.check(_lib.load().rqb200_t5rank_cross_attention_ragged_counted(
                _p(q), q.stride(0), _p(k), _p(v), k.stride(0), _p(offsets), _p(key_mask), _p(tiles), tiles.shape[0], _p(_live(live)),
                heads, _p(out), out.stride(0), _stream()), "t5rank_cross_attention_ragged_counted")
    _count(1)
    return out


class ExactChildren(NamedTuple):
    """The scored children of one decoder level of the exact search, history by history, as ``t5exact_frontier_*`` and
    ``t5exact_select`` read them.  scores fp32 [C]; for the root's children (level 1) offsets, node, code and parent are None and
    history b's children are the n_root entries from b * n_root, child i being node i of level 1.  Otherwise offsets int32
    [Bc + 1] (history b's children are offsets[b] .. offsets[b + 1] - 1), node / code / parent int32 [C] (node id, last code,
    parent row) and key int64 [rows] (each parent row's prefix key; None without a filter)."""
    scores: torch.Tensor
    n_root: int
    offsets: Optional[torch.Tensor] = None
    node: Optional[torch.Tensor] = None
    code: Optional[torch.Tensor] = None
    parent: Optional[torch.Tensor] = None
    key: Optional[torch.Tensor] = None


class ExactLevel(NamedTuple):
    """The next decoder level of the exact search (``t5exact_frontier_write``): rows in trie order (history b's are offsets[0][b]
    .. offsets[0][b + 1] - 1), their last codes and parent rows (int64 [R], ``_T5DecoderLevels.level``'s ids / parent), scores
    fp32 [R], prefix keys int64 [R] (None without a filter), query tiles int32 [T, 3], and the rows' children: child ranges
    int32 [R + 1] (one group) and ``children`` (scores not yet written)."""
    code: torch.Tensor
    parent: torch.Tensor
    score: torch.Tensor
    key: Optional[torch.Tensor]
    tiles: torch.Tensor
    child: torch.Tensor
    children: ExactChildren


def _exact_children_args(ch: ExactChildren):
    return (_p(ch.scores), _p(ch.offsets), int(ch.n_root), _p(ch.node), _p(ch.code), _p(ch.parent), _p(ch.key))


def t5exact_frontier_count(ch: ExactChildren, root_code: Optional[torch.Tensor], tau: torch.Tensor, K: int, l: int,
                           lchild: torch.Tensor, b0: int = 0, exclude: Optional[SidExclusion] = None,
                           include: Optional[SidInclusion] = None) -> torch.Tensor:
    """The count pass of the exact search's frontier (rqb200_t5exact_frontier[_excluding/_including]), one launch: per history
    of the chunk, its children (nodes of level l) with score >= tau[b] (fp32 [Bc]) that the filter (of the whole batch; the
    chunk's first history is b0) does not block -> int32 [3, Bc]: kept rows, their children (lchild = SidTrieLevels.child[l]),
    their 64-query tiles.  root_code: SidTrieLevels.code[1] for the root's children (``ch.node`` None)."""
    Bc = tau.shape[0]
    counts = torch.empty((3, Bc), dtype=torch.int32, device=tau.device)
    _t5exact_frontier(ch, root_code, tau, K, l, lchild, None, b0, counts, None, (None,) * 10, exclude, include)
    return counts


def t5exact_frontier_write(ch: ExactChildren, root_code: Optional[torch.Tensor], tau: torch.Tensor, K: int, l: int,
                           lchild: torch.Tensor, lcode_next: torch.Tensor, offsets: torch.Tensor, totals: Sequence[int],
                           b0: int = 0, exclude: Optional[SidExclusion] = None,
                           include: Optional[SidInclusion] = None) -> ExactLevel:
    """The write pass (the same entry points), one launch: offsets int32 [3, Bc + 1] the exclusive scans of the count pass,
    totals their last column (R rows, C children, T tiles, read on the host by the caller) -> the next level (``ExactLevel``);
    lcode_next = SidTrieLevels.code[l + 1]."""
    R, C, T = (int(t) for t in totals[:3])
    Bc, dev = tau.shape[0], tau.device
    filt = exclude is not None or include is not None
    code, parent = (torch.empty(R, dtype=torch.int64, device=dev) for _ in range(2))
    score = torch.empty(R, dtype=torch.float32, device=dev)
    key = torch.empty(R, dtype=torch.int64, device=dev) if filt else None
    node = torch.empty(max(R, 1), dtype=torch.int32, device=dev)
    tiles = torch.empty((T, 3), dtype=torch.int32, device=dev)
    child = torch.empty(R + 1, dtype=torch.int32, device=dev)
    nnode, ncode, npar = (torch.empty(C, dtype=torch.int32, device=dev) for _ in range(3))
    nxt = ExactChildren(torch.empty(C, dtype=torch.float32, device=dev), 0, offsets[1], nnode, ncode, npar, key)
    _t5exact_frontier(ch, root_code, tau, K, l, lchild, lcode_next, b0, None, offsets,
                      (code, parent, score, key, node, tiles, child, nnode, ncode, npar), exclude, include)
    return ExactLevel(code, parent, score, key, tiles, child, nxt)


def t5exact_frontier_capacity(ch: ExactChildren, root_code: Optional[torch.Tensor], tau: torch.Tensor, K: int, l: int,
                              lchild: torch.Tensor, lcode_next: torch.Tensor, offsets: torch.Tensor, caps: Sequence[int],
                              overflow: torch.Tensor, b0: int = 0, exclude: Optional[SidExclusion] = None,
                              include: Optional[SidInclusion] = None):
    """The write pass at fixed capacities (rqb200_t5exact_frontier_capacity[_excluding/_including]), one launch, for a caller that
    cannot read the totals on the host: caps = (R, C, T) size the outputs, and the kernel reads the totals offsets[:, Bc] itself.
    -> (the next level, ``ExactLevel`` at those capacities with ``children.offsets`` the kernel's copy of offsets[1]; live int32
    [3], the level's rows, children and tiles).  When a total exceeds its capacity nothing is written, live and the children's
    offsets are 0 and overflow[0] (int32, on the device) is set to 1."""
    R, C, T = (int(t) for t in caps)
    if min(R, C, T) < 1:
        raise ValueError(f"t5exact_frontier_capacity: capacities {(R, C, T)} must be >= 1")
    Bc, dev = tau.shape[0], tau.device
    filt = exclude is not None or include is not None
    code, parent = (torch.empty(R, dtype=torch.int64, device=dev) for _ in range(2))
    score = torch.empty(R, dtype=torch.float32, device=dev)
    key = torch.empty(R, dtype=torch.int64, device=dev) if filt else None
    node = torch.empty(R, dtype=torch.int32, device=dev)
    tiles = torch.empty((T, 3), dtype=torch.int32, device=dev)
    child = torch.empty(R + 1, dtype=torch.int32, device=dev)
    nnode, ncode, npar = (torch.empty(C, dtype=torch.int32, device=dev) for _ in range(3))
    live = torch.empty(3, dtype=torch.int32, device=dev)
    noff = torch.empty(Bc + 1, dtype=torch.int32, device=dev)
    nxt = ExactChildren(torch.empty(C, dtype=torch.float32, device=dev), 0, noff, nnode, ncode, npar, key)
    _t5exact_frontier(ch, root_code, tau, K, l, lchild, lcode_next, b0, None, offsets,
                      (code, parent, score, key, node, tiles, child, nnode, ncode, npar), exclude, include,
                      (R, C, T, _p(live), _p(_live(overflow)), _p(noff)))
    return ExactLevel(code, parent, score, key, tiles, child, nxt), live


def _t5exact_frontier(ch, root_code, tau, K, l, lchild, lcode_next, b0, counts, offsets, outs, exclude, include, cap=None):
    _need_cuda(ch.scores, tau, lchild)
    if ch.node is None and root_code is None:
        raise ValueError("t5exact_frontier: the root's children need root_code (SidTrieLevels.code[1])")
    if offsets is not None and (offsets.dtype != torch.int32 or offsets.shape != (3, tau.shape[0] + 1) or not offsets.is_contiguous()):
        raise ValueError(f"t5exact_frontier: offsets must be a contiguous int32 [3, {tau.shape[0] + 1}] tensor")
    ch_args = list(_exact_children_args(ch))
    if ch.node is None:
        ch_args[4] = _p(root_code)
    entry = "t5exact_frontier" if cap is None else "t5exact_frontier_capacity"
    name, filt = _filter_entry(entry, exclude, include, _filter_rows(exclude, include), l, entry)
    pass_args = (_p(counts), _p(offsets)) if cap is None else (_p(offsets),)
    with torch.cuda.device(tau.device):
        _lib.check(getattr(_lib.load(), "rqb200_" + name)(*ch_args, _p(tau), tau.shape[0], int(K), int(l), _p(lchild),
                                                          _p(lcode_next), int(b0), *pass_args, *(_p(t) for t in outs),
                                                          *(cap or ()), *filt, _stream()), name)
    _count(1)


def _filter_rows(exclude, include) -> int:
    """The histories a filter holds (the whole batch; a chunk indexes it from its first history)."""
    f = include if include is not None else exclude
    return 0 if f is None else f.pos.shape[0]


def t5exact_select(ch: ExactChildren, max_u: int, levels: SidTrieLevels, H: int, leaf_key: torch.Tensor, w: int,
                   out_gen: torch.Tensor, out_lp: torch.Tensor, b0: int = 0, exclude: Optional[SidExclusion] = None,
                   include: Optional[SidInclusion] = None) -> None:
    """The exact search's selection (rqb200_t5exact_select[_excluding/_including]), one launch: per history of the chunk, the w
    best of its leaf candidates ``ch`` (leaf ids in ``ch.node``; max_u the largest count of a history) by score descending,
    then leaf ascending, NaN and blocked leaves left out -> out_gen int64 [Bc, w, H] (written: each leaf's tuple, from
    ``levels``' codes and parents) and out_lp fp32 [Bc, w]; -1 / -inf past the valid candidates.  leaf_key int64 [U]: the
    leaves' ``_tuple_key`` (read with a filter)."""
    _need_cuda(ch.scores, out_gen, out_lp, leaf_key)
    Bc = out_lp.shape[0]
    if out_gen.dtype != torch.int64 or out_gen.shape != (Bc, w, H) or not out_gen.is_contiguous():
        raise ValueError(f"out_gen must be a contiguous int64 [{Bc}, {w}, {H}] tensor")
    if out_lp.dtype != torch.float32 or out_lp.shape != (Bc, w) or not out_lp.is_contiguous():
        raise ValueError(f"out_lp must be a contiguous fp32 [{Bc}, {w}] tensor")
    name, filt = _filter_entry("t5exact_select", exclude, include, _filter_rows(exclude, include), H, "t5exact_select")
    args = _exact_children_args(ch)
    codes = _ptr_array([None] + [levels.code[l] for l in range(1, H + 1)])
    parents = _ptr_array([None] + [levels.parent[l] for l in range(1, H + 1)])
    with torch.cuda.device(out_lp.device):
        _lib.check(getattr(_lib.load(), "rqb200_" + name)(args[0], args[1], args[2], args[3], int(max_u), _p(leaf_key), codes,
                                                          parents, Bc, int(H), int(w), int(b0), _p(out_gen), _p(out_lp), *filt,
                                                          _stream()), name)
    _count(1)
