"""CPU model of the tensor-core tokeniser's blocked candidate selection for K = 512 .. 2048 codes
(tests/tc_blocked_model.py restates rq_tcx_blocked_kernel in csrc/rq_tcx.cu): the kept set always contains the unblocked filter's set,
which contains the float64 argmin, and blocking adds (almost) no rows to the exact re-rank."""
import numpy as np
import pytest

import inputs as I
import tc_blocked_model as MB
import tc_filter_model as M
from oracle import rq_oracle as O

SLACK = 0.002       # rows per level that may go to the re-rank because of the blocking alone


def _check(x, cbs):
    ids = O.rq_tokenize(x, cbs)
    lv = M.filter_levels(x, cbs, ids)
    bl = MB.filter_levels_blocked(x, cbs, ids, levels=lv)
    rows = np.arange(len(x))
    fracs = []
    for l, (u, b) in enumerate(zip(lv, bl)):
        assert not (u["cand"] & ~b["cand"]).any(), f"level {l}: the blocked selection lost a candidate of the unblocked filter"
        assert b["cand"][rows, ids[:, l]].all(), f"level {l}: the oracle's fp32 argmin was filtered out"
        true = M.true_half_distances(x, cbs, ids, l)
        fin = np.isfinite(u["eps"]) & np.isfinite(true).all(1)
        assert u["cand"][rows[fin], true[fin].argmin(1)].all(), f"level {l}: the float64 argmin was filtered out"
        fu, fb = float((u["cand"].sum(1) > 1).mean()), float((b["cand"].sum(1) > 1).mean())
        assert fb <= fu + SLACK, (l, fu, fb)
        fracs.append((fu, fb))
    return fracs


@pytest.mark.parametrize("K", [512, 1024, 2048])
@pytest.mark.parametrize("D,L", [(768, 3), (64, 3)])
def test_blocked_selection_keeps_the_unblocked_set(K, D, L):
    x, cbs = I.rq_problem(4096, D, K, L, seed=K + D)
    fracs = _check(x, cbs)
    assert max(fb for _, fb in fracs) < 0.2, fracs


@pytest.mark.parametrize("K", [512, 1024, 2048])
@pytest.mark.parametrize("kind", M.ADVERSARIAL_KINDS)
def test_blocked_selection_on_coherent_rounding(kind, K):
    x, cbs = M.adversarial_problem(kind, D=128, K=K, L=2, n=96)
    _check(x, cbs)


def test_true_minimum_in_the_last_block_drops_the_first():
    """Rows whose best code is in the last block, with a runner-up in block 0 that is outside the final margin: block 0 is
    kept while it is scored (its own minimum sets the running threshold) and dropped at the end, so the row has one candidate."""
    D, K = 128, 1024
    rs = np.random.RandomState(3)
    cb = (rs.randn(K, D) / np.sqrt(D)).astype(np.float32)
    x = (cb[K - 5] + 1e-3 * rs.randn(64, D)).astype(np.float32)
    cb[7] = (cb[K - 5] + 0.05 * rs.randn(D) / np.sqrt(D)).astype(np.float32)       # near, but far outside eps
    ids = O.rq_tokenize(x, [cb])
    assert (ids[:, 0] == K - 5).all()
    u = M.filter_levels(x, [cb], ids)[0]
    b = MB.filter_levels_blocked(x, [cb], ids)[0]
    assert (u["cand"].sum(1) == 1).all() and np.array_equal(u["cand"], b["cand"])


def test_single_block_is_the_unblocked_filter():
    """K = 256: one block, nothing to drop -- the selection is the unblocked filter's exactly."""
    x, cbs = I.rq_problem(1024, 128, 256, 3, seed=8)
    ids = O.rq_tokenize(x, cbs)
    for u, b in zip(M.filter_levels(x, cbs, ids), MB.filter_levels_blocked(x, cbs, ids)):
        assert np.array_equal(u["cand"], b["cand"])
