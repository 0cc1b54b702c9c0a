"""CPU oracle for the RQ-VAE residual-quantization hot path  --  TEST INFRASTRUCTURE ONLY.

This file is a plain-numpy restatement of the reference algorithm
(EdoardoBotta/RQ-VAE-Recommender @ /root/reference).  Every function cites the
reference file:line it follows.  It is the *checker*: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline / ``--impl reference``
legs may import it.  Nothing under ``rq_vae_recommender_b200/`` imports it, and
the product path has no CPU fallback.

Parity pinning: the reference ships no tests / golden vectors, so the oracle is
pinned against the reference ITSELF, executed in the build container from
/root/reference (see ``tests/golden/make_golden.py``, which imports the
unmodified reference modules and writes ``tests/golden/*.npz``).
``tests/test_oracle_golden.py`` checks every function below against those
fixtures, so on the GPU box (where /root/reference does not exist) the oracle
stands in for the reference.

All functions are dtype-generic: pass float32 arrays for the canonical oracle,
float64 arrays for the tie classifier (``top2_gap``).
"""
from __future__ import annotations

from typing import Callable, List, NamedTuple, Optional, Sequence

import numpy as np

# forward modes, numbering of modules/quantize.py:16-20
GUMBEL_SOFTMAX = 1
STE = 2
ROTATION_TRICK = 3


# --------------------------------------------------------------------------- helpers
def l2norm(x: np.ndarray, eps: float = 1e-12) -> np.ndarray:
    """modules/normalize.py:6-7 -> F.normalize(p=2): x / max(||x||_2, eps)."""
    n = np.sqrt((x * x).sum(axis=-1, keepdims=True))
    return x / np.maximum(n, x.dtype.type(eps))


def mlp_forward(x: np.ndarray, weights: Sequence[np.ndarray], normalize: bool = False,
                act: str = "relu") -> np.ndarray:
    """modules/encoder.py:23-38: bias-free Linear (+ReLU between layers), optional final L2 norm.

    ``weights[i]`` has the nn.Linear layout [out, in].  ``act="silu"`` reproduces the
    activation pickled inside the shipped Amazon checkpoints."""
    h = x
    n = len(weights)
    for i, w in enumerate(weights):
        h = h @ w.T
        if i != n - 1:
            if act == "relu":
                h = np.maximum(h, h.dtype.type(0))
            elif act == "silu":
                h = h / (1 + np.exp(-h))
            else:
                raise ValueError(act)
    return l2norm(h) if normalize else h


def quantize_dist(x: np.ndarray, codebook: np.ndarray) -> np.ndarray:
    """modules/quantize.py:113-117: (x**2).sum(1) + (c.T**2).sum(0) - 2*x @ c.T  -> [B,K]."""
    return ((x ** 2).sum(axis=1, keepdims=True)
            + (codebook.T ** 2).sum(axis=0, keepdims=True)
            - (2 * x) @ codebook.T)


def argmin_first(dist: np.ndarray) -> np.ndarray:
    """modules/quantize.py:128: dist.min(axis=1).indices -- first minimal index on ties."""
    return np.argmin(dist, axis=1).astype(np.int64)


def quantize_loss(query: np.ndarray, value: np.ndarray, beta: float) -> np.ndarray:
    """modules/loss.py:38-41: ||sg(q)-v||^2 + beta*||q-sg(v)||^2 per row (two separately rounded terms)."""
    emb_loss = ((query - value) ** 2).sum(axis=-1)
    query_loss = ((query - value) ** 2).sum(axis=-1)
    return emb_loss + query.dtype.type(beta) * query_loss


def sample_gumbel_from_uniform(u: np.ndarray, eps: float = 1e-20) -> np.ndarray:
    """distributions/gumbel.py:8-11 with the uniform draw U injected: -log(-log(U+eps)+eps)."""
    e = u.dtype.type(eps)
    return -np.log(-np.log(u + e) + e)


def gumbel_softmax_from_uniform(logits: np.ndarray, temperature: float, u: np.ndarray) -> np.ndarray:
    """distributions/gumbel.py:14-20: softmax((logits + G)/T, dim=-1)."""
    y = (logits + sample_gumbel_from_uniform(u)) / logits.dtype.type(temperature)
    y = y - y.max(axis=-1, keepdims=True)
    e = np.exp(y)
    return e / e.sum(axis=-1, keepdims=True)


def rotation_trick(u: np.ndarray, q: np.ndarray, e: np.ndarray) -> np.ndarray:
    """modules/quantize.py:34-50: e - 2 (e.w) w + 2 (e.u) q  with w = normalize(u+q, eps=1e-6)."""
    w = u + q
    w = w / np.maximum(np.sqrt((w * w).sum(axis=1, keepdims=True)), e.dtype.type(1e-6))
    ew = (e * w).sum(axis=1, keepdims=True)
    eu = (e * u).sum(axis=1, keepdims=True)
    return e - 2 * (ew * w) + 2 * (eu * q)


# --------------------------------------------------------------------------- one level
class QuantizeOut(NamedTuple):
    embeddings: np.ndarray   # emb_out [B,D]
    ids: np.ndarray          # [B] int64
    loss: np.ndarray         # [B]
    emb: np.ndarray          # the (pre-STE) quantised vector used in the loss [B,D]


def quantize_forward(x: np.ndarray, codebook: np.ndarray, mode: int = STE, training: bool = False,
                     temperature: float = 0.2, beta: float = 0.25,
                     gumbel_uniform: Optional[np.ndarray] = None) -> QuantizeOut:
    """modules/quantize.py:104-163 (L2 distance).  ``codebook`` is out_proj(embedding.weight)."""
    dist = quantize_dist(x, codebook)
    ids = argmin_first(dist)
    if training:
        if mode == GUMBEL_SOFTMAX:                                    # :131-136
            w = gumbel_softmax_from_uniform(-dist, temperature, gumbel_uniform)
            emb = w @ codebook
            emb_out = emb
        elif mode == STE:                                             # :137-139
            emb = codebook[ids]
            emb_out = x + (emb - x)
        elif mode == ROTATION_TRICK:                                  # :140-153
            emb = codebook[ids]
            t = x.dtype.type
            xn = np.sqrt((x * x).sum(axis=-1, keepdims=True))
            en = np.sqrt((emb * emb).sum(axis=-1, keepdims=True))
            rot = rotation_trick(x / (xn + t(1e-8)), emb / (en + t(1e-8)), x)
            emb_out = rot * (en / (xn + t(1e-6)))
        else:
            raise ValueError("Unsupported Quantize forward mode.")
        loss = quantize_loss(x, emb, beta)                             # :157
    else:                                                             # :159-161
        emb = codebook[ids]
        emb_out = emb
        loss = quantize_loss(x, emb_out, beta)
    return QuantizeOut(emb_out, ids, loss, emb)


# --------------------------------------------------------------------------- L chained levels
class RqOut(NamedTuple):
    embeddings: np.ndarray   # [B,D,L]
    residuals: np.ndarray    # [B,D,L]
    sem_ids: np.ndarray      # [B,L] int64
    quantize_loss: np.ndarray  # [B]


def rq_forward(res: np.ndarray, codebooks: Sequence[np.ndarray], mode: int = STE,
               training: bool = False, temperature: float = 0.2, beta: float = 0.25,
               gumbel_uniform: Optional[Sequence[np.ndarray]] = None) -> RqOut:
    """modules/rqvae.py:122-139: residual chain over the L Quantize levels (input = encoder output)."""
    embs, residuals, ids = [], [], []
    loss = np.zeros(res.shape[0], dtype=res.dtype)
    for l, cb in enumerate(codebooks):
        residuals.append(res)
        q = quantize_forward(res, cb, mode, training, temperature, beta,
                             None if gumbel_uniform is None else gumbel_uniform[l])
        loss = loss + q.loss
        res = res - q.embeddings
        ids.append(q.ids)
        embs.append(q.embeddings)
    return RqOut(np.stack(embs, axis=-1), np.stack(residuals, axis=-1), np.stack(ids, axis=-1), loss)


def rq_tokenize(res: np.ndarray, codebooks: Sequence[np.ndarray]) -> np.ndarray:
    """Eval-mode sem_ids only (what modules/tokenizer/semids.py:125 consumes)."""
    ids = []
    for cb in codebooks:
        i = argmin_first(quantize_dist(res, cb))
        res = res - cb[i]
        ids.append(i)
    return np.stack(ids, axis=-1)


def top2_gap(res64: np.ndarray, codebooks64: Sequence[np.ndarray], ids: Optional[np.ndarray] = None,
             return_abs: bool = False):
    """float64 tie classifier.

    Returns (ids64 [B,L], best2 [B,L], relgap [B,L]) where the chain follows ``ids`` if given
    (so level l is judged on the residual the implementation under test actually saw),
    best2 is the runner-up code and relgap = (d2 - d1) / max(d1, tiny).
    With ``return_abs`` also (d2 - d1) / (||res||^2 + ||c_best||^2): the gap in units of the OPERANDS of
    quantize.py:113-117's  xx + cc - 2 x.c  -- when a row all but coincides with a code, d1 is a cancellation
    residue of terms ~1 and fp32 cannot resolve differences below a few 2^-24 of those terms, whatever d1 is."""
    assert res64.dtype == np.float64
    B = res64.shape[0]
    L = len(codebooks64)
    ids64 = np.zeros((B, L), np.int64)
    second = np.zeros((B, L), np.int64)
    gap = np.zeros((B, L), np.float64)
    absgap = np.zeros((B, L), np.float64)
    res = res64
    for l, cb in enumerate(codebooks64):
        d = quantize_dist(res, cb)
        order = np.argsort(d, axis=1, kind="stable")[:, :2]
        d1 = np.take_along_axis(d, order[:, :1], axis=1)[:, 0]
        d2 = np.take_along_axis(d, order[:, 1:2], axis=1)[:, 0]
        ids64[:, l] = order[:, 0]
        second[:, l] = order[:, 1]
        gap[:, l] = (d2 - d1) / np.maximum(np.abs(d1), 1e-30)
        scale = (res * res).sum(1) + (cb * cb).sum(1)[order[:, 0]]
        absgap[:, l] = (d2 - d1) / np.maximum(scale, 1e-30)
        follow = ids64[:, l] if ids is None else ids[:, l]
        res = res - cb[follow]
    if return_abs:
        return ids64, second, gap, absgap
    return ids64, second, gap


# --------------------------------------------------------------------------- full model
class RqVaeLosses(NamedTuple):
    loss: np.ndarray
    reconstruction_loss: np.ndarray
    rqvae_loss: np.ndarray
    embs_norm: np.ndarray
    p_unique_ids: np.ndarray


def reconstruction_loss(x_hat: np.ndarray, x: np.ndarray, n_cat: int = 0) -> np.ndarray:
    """modules/loss.py:9-10 (n_cat == 0) and :19-30 (SSE on the first D-n_cat dims + BCE-with-logits)."""
    if n_cat == 0:
        return ((x_hat - x) ** 2).sum(axis=-1)
    rec = ((x_hat[:, :-n_cat] - x[:, :-n_cat]) ** 2).sum(axis=-1)
    z, y = x_hat[:, -n_cat:], x[:, -n_cat:]
    bce = np.maximum(z, 0) - z * y + np.log1p(np.exp(-np.abs(z)))
    return rec + bce.sum(axis=-1)


def p_unique_ids(sem_ids: np.ndarray) -> float:
    """modules/rqvae.py:159-167: fraction of rows that have no LATER identical row == n_unique / B."""
    return np.unique(sem_ids, axis=0).shape[0] / sem_ids.shape[0]


def rqvae_forward(x: np.ndarray, enc_w: Sequence[np.ndarray], codebooks: Sequence[np.ndarray],
                  dec_w: Sequence[np.ndarray], mode: int = STE, training: bool = False,
                  temperature: float = 0.2, beta: float = 0.25, n_cat: int = 0,
                  codebook_normalize: bool = False, act: str = "relu",
                  gumbel_uniform=None) -> RqVaeLosses:
    """modules/rqvae.py:141-175."""
    res = mlp_forward(x, enc_w, normalize=codebook_normalize, act=act)
    q = rq_forward(res, codebooks, mode, training, temperature, beta, gumbel_uniform)
    x_hat = mlp_forward(q.embeddings.sum(axis=-1), dec_w, act=act)
    if n_cat != 0:     # rqvae.py:147-150; with n_cat == 0 the [:-0] slice is empty -> no normalisation
        x_hat = np.concatenate([l2norm(x_hat[..., :-n_cat]), x_hat[..., -n_cat:]], axis=-1)
    rec = reconstruction_loss(x_hat, x, n_cat)
    loss = (rec + q.quantize_loss).mean()
    embs_norm = np.sqrt((q.embeddings ** 2).sum(axis=1))
    return RqVaeLosses(loss, rec.mean(), q.quantize_loss.mean(), embs_norm,
                       np.asarray(p_unique_ids(q.sem_ids), dtype=x.dtype))


# --------------------------------------------------------------------------- backward
def quantize_backward(mode: int, x: np.ndarray, codebook: np.ndarray, ids: np.ndarray,
                      g_out: np.ndarray, g_loss: np.ndarray, beta: float = 0.25,
                      temperature: float = 0.2, gumbel_uniform: Optional[np.ndarray] = None):
    """Analytic gradients of (emb_out, loss) of one training-mode Quantize level w.r.t. (x, codebook).

    These are the autograd results of modules/quantize.py:130-157 + modules/loss.py:38-41;
    checked against the reference's own autograd in tests/golden (grad fixtures)."""
    t = x.dtype.type
    K = codebook.shape[0]
    gl = g_loss[:, None]
    if mode in (STE, ROTATION_TRICK):
        e = codebook[ids]
        gx = 2 * t(beta) * gl * (x - e)
        ge = 2 * gl * (e - x)
        if mode == STE:
            gx = gx + g_out
        else:
            xn = np.sqrt((x * x).sum(axis=-1, keepdims=True))
            en = np.sqrt((e * e).sum(axis=-1, keepdims=True))
            u = x / (xn + t(1e-8))
            q = e / (en + t(1e-8))
            w = u + q
            w = w / np.maximum(np.sqrt((w * w).sum(axis=1, keepdims=True)), t(1e-6))
            gh = g_out * (en / (xn + t(1e-6)))
            gx = gx + gh - 2 * (gh * w).sum(axis=1, keepdims=True) * w \
                + 2 * (gh * q).sum(axis=1, keepdims=True) * u
        gc = np.zeros_like(codebook)
        np.add.at(gc, ids, ge)
        return gx, gc
    if mode == GUMBEL_SOFTMAX:
        dist = quantize_dist(x, codebook)
        w = gumbel_softmax_from_uniform(-dist, temperature, gumbel_uniform)
        E = w @ codebook
        gE = g_out + 2 * gl * (E - x)
        gW = gE @ codebook.T
        gY = w * (gW - (w * gW).sum(axis=1, keepdims=True)) / t(temperature)
        gd = -gY
        gx = 2 * t(beta) * gl * (x - E) + 2 * x * gd.sum(axis=1, keepdims=True) - 2 * gd @ codebook
        gc = w.T @ gE + 2 * codebook * gd.sum(axis=0)[:, None] - 2 * gd.T @ x
        return gx, gc
    raise ValueError(mode)


# --------------------------------------------------------------------------- k-means init
class KmeansOut(NamedTuple):
    centroids: np.ndarray
    assignment: np.ndarray
    n_iters: int


def kmeans_run(x: np.ndarray, k: int, init_idx: np.ndarray,
               randint: Callable[[int], int], max_iters: Optional[int] = None,
               stop_threshold: float = 1e-10) -> KmeansOut:
    """init/kmeans.py:33-72 with the two RNG draws injected.

    ``init_idx`` is what ``np.random.choice(B, k, replace=False)`` returned (kmeans.py:35);
    ``randint(n)`` stands for ``torch.randint(0, n, (1,))`` (kmeans.py:53), called once per
    empty cluster in cluster order.  Distances are the broadcast (x-c)**2 sum of kmeans.py:40-43."""
    c = x[init_idx, :].copy()
    assignment = None
    i = 0
    while max_iters is None or i < max_iters:
        old = c.copy()
        # (x[:,None,:]-c[None,:,:])**2 summed over d, chunked over rows to bound memory (same arithmetic per element)
        idx = np.empty(x.shape[0], np.int64)
        step = max(1, (1 << 24) // max(1, k * x.shape[1]))
        for s in range(0, x.shape[0], step):
            d = ((x[s:s + step, None, :] - c[None, :, :]) ** 2).sum(axis=2)
            idx[s:s + step] = np.argmin(d, axis=1)
        for cluster in range(k):                                      # kmeans.py:48-58 (in-place, sequential)
            m = idx == cluster
            if not m.any():
                c[cluster, :] = x[randint(x.shape[0])]
            else:
                c[cluster, :] = x[m, :].mean(axis=0)
        assignment = idx
        i += 1
        if np.sqrt(((c - old) ** 2).sum(axis=1)).max() < stop_threshold:   # kmeans.py:68
            break
    return KmeansOut(c, assignment, i)


# --------------------------------------------------------------------------- tokenizer helpers
def dedup_rank(sem_ids: np.ndarray) -> np.ndarray:
    """modules/tokenizer/semids.py:94-108: number of EARLIER corpus rows with the identical id tuple."""
    N = sem_ids.shape[0]
    out = np.zeros(N, np.int64)
    seen = {}
    for i in range(N):
        key = tuple(int(v) for v in sem_ids[i])
        out[i] = seen.get(key, 0)
        seen[key] = out[i] + 1
    return out


def codebook_usage(sem_ids: np.ndarray, K: int) -> np.ndarray:
    """train_rqvae.py:285-289: per-level histogram of used codes -> [L,K] int64."""
    L = sem_ids.shape[1]
    return np.stack([np.bincount(sem_ids[:, l], minlength=K) for l in range(L)]).astype(np.int64)


# --------------------------------------------------------------------------- reduced-precision (AMP-like) MLP
def round_bf16(a: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even to bfloat16, returned as float32 (what cvt.rn.bf16.f32 does)."""
    b = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32).reshape(a.shape)


def mlp_forward_bf16(x: np.ndarray, weights: Sequence[np.ndarray], normalize: bool = False) -> np.ndarray:
    """modules/encoder.py:23-38 as the reference computes it under bf16 autocast (train_rqvae.py:36,69): operands rounded
    to bf16, products accumulated in higher precision, ReLU, activations re-rounded to bf16 between layers; the last
    layer's output stays fp32."""
    h = round_bf16(x)
    n = len(weights)
    for i, w in enumerate(weights):
        y = (h.astype(np.float64) @ round_bf16(w).astype(np.float64).T).astype(np.float32)
        if i != n - 1:
            h = round_bf16(np.maximum(y, 0))
        else:
            h = y
    return l2norm(h) if normalize else h


def check_valid_prefix(corpus_ids: np.ndarray, prefix: np.ndarray) -> np.ndarray:
    """modules/model.py:169-182 `_check_valid_prefix`: bool [P], prefix p occurs as the first l ids of some corpus row."""
    trimmed = corpus_ids[:, : prefix.shape[1]]
    l = prefix.shape[1]
    if trimmed.size * prefix.shape[0] > (1 << 26) and l <= 4 and trimmed.min(initial=0) >= 0 and trimmed.max(initial=0) < (1 << 15):
        # large cases: the same predicate through packed keys (row equality <=> key equality for ids in [0, 2^15)); a prefix
        # holding an id outside that range equals no corpus row
        inside = ((prefix >= 0) & (prefix < (1 << 15))).all(axis=1)
        w = (1 << 15) ** np.arange(l - 1, -1, -1, dtype=np.int64)
        keys = (np.where(inside[:, None], prefix, 0).astype(np.int64) * w).sum(axis=1)
        return inside & np.isin(keys, np.unique((trimmed.astype(np.int64) * w).sum(axis=1)))
    out = np.zeros(prefix.shape[0], dtype=bool)
    for i in range(0, prefix.shape[0], 4096):
        batch = prefix[i:i + 4096]
        out[i:i + 4096] = (trimmed[:, None, :] == batch[None, :, :]).all(axis=2).any(axis=0)
    return out


def beam_select(corpus_ids, samples, samp_log_p, generated, log_probas, k):
    """One selection step of the constrained beam search, modules/model.py:353-388 (numpy restatement; stable sort, so equal
    scores keep candidate order -- torch.sort there is unstable: compare ids only where the k-th score is not tied).
    samples / samp_log_p [B * kp, nc]; generated [B, kp, h] or None; log_probas [B, kp] or None."""
    nc = samples.shape[1]
    if generated is None:
        B = samples.shape[0]
        valid = check_valid_prefix(corpus_ids, samples.reshape(-1, 1)).reshape(B, nc)
        scores = np.where(valid, samp_log_p, -np.inf)
        idx = np.argsort(-scores, axis=1, kind="stable")[:, :k]
        gen = np.take_along_axis(samples, idx, 1)[:, :, None]
        return gen, np.take_along_axis(scores, idx, 1), np.zeros((B, k), dtype=np.int64) + np.arange(B)[:, None]
    B, kp, h = generated.shape
    prev = np.repeat(generated.reshape(-1, h), nc, axis=0)
    prefix = np.concatenate([prev, samples.reshape(-1, 1)], axis=1)
    valid = check_valid_prefix(corpus_ids, prefix).reshape(B, kp * nc)
    scores = np.where(valid, samp_log_p.reshape(B, kp * nc) + np.repeat(log_probas, nc, axis=1), -np.inf)
    idx = np.argsort(-scores, axis=1, kind="stable")[:, :k]
    parent = idx // nc
    parent_ids = np.take_along_axis(generated, parent[:, :, None].repeat(h, 2), 1)
    new_ids = np.take_along_axis(samples.reshape(B, kp * nc), idx, 1)[:, :, None]
    return (np.concatenate([parent_ids, new_ids], axis=2), np.take_along_axis(scores, idx, 1),
            parent + np.arange(B)[:, None] * kp)
