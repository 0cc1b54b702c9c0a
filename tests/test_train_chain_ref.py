"""The float64 training-chain reference (tests/train_chain_ref.py) against the numpy oracle, on the CPU."""
import numpy as np
import pytest
import torch

import inputs as I
import train_chain_ref as R
from oracle import rq_oracle as O

T, BETA = 0.2, 0.25
OMODE = {R.EVAL: O.STE, R.STE: O.STE, R.ROT: O.ROTATION_TRICK, R.GUMBEL: O.GUMBEL_SOFTMAX}
MODES = [R.EVAL, R.STE, R.ROT, R.GUMBEL]


def problem(B, D, K, L, seed):
    x, cbs = I.rq_problem(max(B, K), D, K, L, seed=seed)
    u = I.rand(seed + 7, B, L, K)
    return x[:B].astype(np.float64), [c.astype(np.float64) for c in cbs], u.astype(np.float64)


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def oracle(mode, x, cbs, u):
    return O.rq_forward(x, cbs, OMODE[mode], mode != R.EVAL, T, BETA, gumbel_uniform=[u[:, l] for l in range(len(cbs))])


def reference(mode, x, cbs, u, ids=None, upstream=None, chunk=None):
    if mode == R.GUMBEL:
        return R.evaluate(R.gumbel_chain(T, BETA), t(x), [t(c) for c in cbs], (t(u),), upstream, chunk)
    return R.evaluate(R.chain(mode, BETA), t(x), [t(c) for c in cbs], (t(ids),), upstream, chunk)


@pytest.mark.parametrize("B,D,K,L", [(1, 5, 3, 1), (37, 16, 10, 3), (200, 24, 40, 4)])
@pytest.mark.parametrize("mode", MODES)
def test_forward_matches_oracle(mode, B, D, K, L):
    x, cbs, u = problem(B, D, K, L, seed=B + D)
    so = oracle(mode, x, cbs, u)
    out, _, _ = reference(mode, x, cbs, u, ids=so.sem_ids)
    assert rel(out["embeddings"].numpy(), so.embeddings.transpose(0, 2, 1)) < 1e-12
    assert rel(out["residuals"].numpy(), so.residuals.transpose(0, 2, 1)) < 1e-12
    assert rel(out["loss"].numpy(), so.quantize_loss) < 1e-12
    assert rel(out["emb_sum"].numpy(), so.embeddings.sum(-1)) < 1e-12
    assert rel(out["emb_norms"].numpy(), np.sqrt((so.embeddings ** 2).sum(1))) < 1e-12
    if mode == R.GUMBEL:
        assert np.array_equal(out["ids"].numpy(), so.sem_ids)


def single_level_backward(mode, x, cb, ids, g_out, g_loss, u):
    """Analytic gradients of one level: the oracle's quantize_backward, and for eval mode (emb_out = codebook[ids], the loss
    of loss.py:38-41) the two lines it amounts to."""
    if mode != R.EVAL:
        return O.quantize_backward(OMODE[mode], x, cb, ids, g_out, g_loss, BETA, T, u)
    e = cb[ids]
    gc = np.zeros_like(cb)
    np.add.at(gc, ids, g_out + 2 * g_loss[:, None] * (e - x))
    return 2 * BETA * g_loss[:, None] * (x - e), gc


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("L", [1, 3])
def test_backward_is_l_single_level_backwards(mode, L):
    """Gradients of the whole chain (autograd) equal L analytic single-level backwards walked from the last level to the
    first, with the upstream gradient of every output (embeddings, residuals, loss)."""
    B, D, K = 150, 12, 20
    x, cbs, u = problem(B, D, K, L, seed=40 + L)
    rs = np.random.RandomState(3)
    ge, gr, gl = rs.randn(B, L, D), rs.randn(B, L, D), rs.rand(B)
    so = oracle(mode, x, cbs, u)
    up = dict(embeddings=t(ge), residuals=t(gr), loss=t(gl))
    out, gx, gcs = reference(mode, x, cbs, u, ids=so.sem_ids, upstream=up)
    res = so.residuals.transpose(0, 2, 1)                       # [B, L, D], the residual entering each level
    g_next = np.zeros((B, D))                                   # gradient w.r.t. the residual leaving level l
    gcs_ref = [None] * L
    for l in range(L - 1, -1, -1):
        # res_{l+1} = res_l - emb_out_l: emb_out_l sees ge_l - g_next, res_l sees g_next directly
        gxl, gcs_ref[l] = single_level_backward(mode, res[:, l], cbs[l], so.sem_ids[:, l], ge[:, l] - g_next, gl, u[:, l])
        g_next = g_next + gxl + gr[:, l]
    assert rel(gx.numpy(), g_next) < 1e-12
    for a, b in zip(gcs, gcs_ref):
        assert rel(a.numpy(), b) < 1e-12


@pytest.mark.parametrize("mode", MODES)
def test_chain_is_l_single_levels(mode):
    """The L-level chain's forward equals L calls of the single-level functions on the running residual."""
    B, D, K, L = 64, 10, 16, 3
    x, cbs, u = problem(B, D, K, L, seed=9)
    ids = oracle(mode, x, cbs, u).sem_ids
    out, _, _ = reference(mode, x, cbs, u, ids=ids)
    res, loss = t(x), 0
    for l in range(L):
        assert torch.equal(out["residuals"][:, l], res)
        if mode == R.GUMBEL:
            emb, lo, _ = R.gumbel_level(res, t(cbs[l]), t(u[:, l]), T, BETA)
        else:
            emb, lo = R.level(res, t(cbs[l]), t(ids[:, l]), mode, BETA)
        assert torch.equal(out["embeddings"][:, l], emb)
        loss = loss + lo
        res = res - emb
    assert torch.equal(out["loss"], loss)


@pytest.mark.parametrize("mode", MODES)
def test_row_chunks_sum_codebook_gradients(mode):
    """Row chunks change nothing: outputs and gradients equal up to float64 summation order."""
    B, D, K, L = 301, 8, 12, 2
    x, cbs, u = problem(B, D, K, L, seed=21)
    ids = oracle(mode, x, cbs, u).sem_ids
    rs = np.random.RandomState(5)
    up = dict(emb_sum=t(rs.randn(B, D)), loss=t(rs.rand(B)))
    whole, gx, gcs = reference(mode, x, cbs, u, ids=ids, upstream=up)
    seen = []
    parts = R.evaluate(R.gumbel_chain(T, BETA) if mode == R.GUMBEL else R.chain(mode, BETA), t(x), [t(c) for c in cbs],
                       (t(u),) if mode == R.GUMBEL else (t(ids),), up, chunk=64,
                       on_chunk=lambda rows, o: seen.append((rows, o)))
    assert parts[0] is None and [r.start for r, _ in seen] == [0, 64, 128, 192, 256]
    for rows, o in seen:
        for k, v in o.items():
            assert rel(v.numpy(), whole[k][rows].numpy()) < 1e-13, k
    assert rel(parts[1].numpy(), gx.numpy()) < 1e-13
    for a, b in zip(parts[2], gcs):
        assert rel(a.numpy(), b.numpy()) < 1e-13
