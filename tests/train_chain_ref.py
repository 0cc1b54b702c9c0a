"""Float64 reference of the training-mode quantiser, as plain differentiable torch (test infrastructure only).

It restates, on GIVEN ids, the L-level residual chain of modules/rqvae.py:122-132 over the eval, STE and rotation-trick
levels of modules/quantize.py:104-163, and the Gumbel-softmax level with given uniforms (quantize.py:113-136,
distributions/gumbel.py:8-20).  Every output is row-major: ``embeddings`` / ``residuals`` [B, L, D], ``emb_sum`` [B, D],
``emb_norms`` [B, L], ``loss`` [B].  ``evaluate`` runs one of these chains in any dtype on any device, optionally in row chunks
(codebook gradients are summed across chunks), so a 65 536 x 768 float64 reference fits in a few hundred MB of GPU memory.
"""
import contextlib

import torch
import torch.nn.functional as F

EVAL, GUMBEL, STE, ROT = 0, 1, 2, 3          # the kernels' mode numbers (ops.MODE_*)


def level(res, cb, ids, mode, beta):
    """One eval / STE / rotation-trick level on the given ids -> (emb_out [B, D], loss [B])."""
    e = cb[ids]
    if mode == EVAL:
        eo = e
    elif mode == STE:
        eo = res + (e - res).detach()
    elif mode == ROT:
        u = res / (res.norm(dim=-1, keepdim=True) + 1e-8)
        q = e / (e.norm(dim=-1, keepdim=True) + 1e-8)
        w = F.normalize(u + q, p=2, dim=1, eps=1e-6).detach()
        rot = res - 2 * (res * w).sum(1, keepdim=True) * w + 2 * (res * u.detach()).sum(1, keepdim=True) * q.detach()
        eo = rot * (e.norm(dim=1, keepdim=True) / (res.norm(dim=1, keepdim=True) + 1e-6)).detach()
    else:
        raise ValueError(f"mode {mode}")
    loss = ((res.detach() - e) ** 2).sum(-1) + beta * ((res - e.detach()) ** 2).sum(-1)
    return eo, loss


def gumbel_level(res, cb, u, temperature, beta):
    """One Gumbel-softmax level with the uniform draw ``u`` [B, K] given -> (emb [B, D], loss [B], dist [B, K])."""
    u = u.to(res.dtype)
    dist = (res ** 2).sum(1, keepdim=True) + (cb ** 2).sum(1)[None] - 2 * res @ cb.t()
    g = -torch.log(-torch.log(u + 1e-20) + 1e-20)
    w = torch.softmax((-dist + g) / temperature, dim=-1)
    emb = w @ cb
    loss = ((res.detach() - emb) ** 2).sum(-1) + beta * ((res - emb.detach()) ** 2).sum(-1)
    return emb, loss, dist


def _pack(embs, ress, loss):
    E = torch.stack(embs, 1)
    return dict(embeddings=E, residuals=torch.stack(ress, 1), emb_sum=E.sum(1), emb_norms=E.norm(dim=-1), loss=loss)


def chain(mode, beta):
    """fn(x, codebooks, ids [B, L]) of the L-level eval / STE / rotation chain, for ``evaluate``."""
    def fn(x, codebooks, ids):
        res, embs, ress, loss = x, [], [], 0
        for l, cb in enumerate(codebooks):
            ress.append(res)
            eo, lo = level(res, cb, ids[:, l], mode, beta)
            embs.append(eo)
            loss = loss + lo
            res = res - eo
        return _pack(embs, ress, loss)
    return fn


def gumbel_chain(temperature, beta):
    """fn(x, codebooks, uniforms [B, L, K]) of L chained Gumbel-softmax levels (res <- res - emb), for ``evaluate``.
    Besides the chain's outputs it returns ``ids`` [B, L], the first-index argmin of each level's distances."""
    def fn(x, codebooks, uniforms):
        res, embs, ress, ids, loss = x, [], [], [], 0
        for l, cb in enumerate(codebooks):
            ress.append(res)
            emb, lo, dist = gumbel_level(res, cb, uniforms[:, l], temperature, beta)
            ids.append(dist.argmin(1))
            embs.append(emb)
            loss = loss + lo
            res = res - emb
        out = _pack(embs, ress, loss)
        out["ids"] = torch.stack(ids, 1)
        return out
    return fn


def evaluate(fn, x, codebooks, row_args=(), upstream=None, chunk=None, on_chunk=None, dtype=torch.float64):
    """Run ``fn(x, codebooks, *row_args)`` in ``dtype`` on the device of ``x``, ``chunk`` rows at a time.

    ``upstream`` maps output names to the gradient of the objective with respect to that output (row-major, any dtype); with
    it the gradients of sum_k <output_k, upstream_k> with respect to ``x`` and every codebook are returned as well.
    ``on_chunk(rows, outputs)`` receives each chunk's outputs (a slice and a dict); without it they are concatenated.
    Returns (outputs or None, g_x or None, [g_codebook] or None)."""
    B = x.shape[0]
    chunk = chunk or max(B, 1)
    grad = upstream is not None
    cbs = [c.detach().to(dtype).requires_grad_(grad) for c in codebooks]
    gx = torch.empty(x.shape, dtype=dtype, device=x.device) if grad else None
    pieces = {}
    for s in range(0, B, chunk):
        rows = slice(s, min(B, s + chunk))
        xc = x[rows].detach().to(dtype).requires_grad_(grad)
        with torch.enable_grad():
            out = fn(xc, cbs, *[a[rows] for a in row_args])
            if grad:
                obj = sum((out[k] * g[rows].to(dtype)).sum() for k, g in upstream.items() if g is not None)
                obj.backward()
                gx[rows] = 0 if xc.grad is None else xc.grad        # None: the objective does not depend on x
        out = {k: v.detach() for k, v in out.items()}
        if on_chunk is not None:
            on_chunk(rows, out)
        else:
            for k, v in out.items():
                pieces.setdefault(k, []).append(v)
    outputs = None if on_chunk is not None else {k: torch.cat(v) for k, v in pieces.items()}
    return outputs, gx, ([torch.zeros_like(c) if c.grad is None else c.grad for c in cbs] if grad else None)


@contextlib.contextmanager
def highest_matmul_precision():
    """fp32 torch matmuls in full fp32 (modules/rqvae.py sets "high", i.e. TF32, on import), restored afterwards."""
    old = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("highest")
    try:
        yield
    finally:
        torch.set_float32_matmul_precision(old)
