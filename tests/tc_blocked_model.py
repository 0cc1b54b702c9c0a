"""numpy model of the blocked candidate selection of the tensor-core tokeniser for K = 512 .. 2048 codes
(rq_tcx_blocked_kernel in csrc/rq_tcx.cu) -- test infrastructure, built on the unblocked filter model of tests/tc_filter_model.py.

The codes of a level are scored one 256-code block at a time.  Block b keeps {k in b : h[k] <= M_b + margin}, with M_b the
running row minimum over blocks 0..b and margin = 2 eps (1 + 2^-16).  At the end of the level every block whose minimum is
above the final threshold M + margin is dropped; a block holding a NaN score never is.  Since M_b >= M, every block keeps a
superset of its share of the unblocked candidate set, and a row whose unblocked set is one code ends with exactly that code.
"""
import numpy as np

import tc_filter_model as M

BLOCK = 256


def filter_levels_blocked(x, cbs, ids, levels=None, block=BLOCK):
    """`levels`: tc_filter_model.filter_levels' output on the same inputs (recomputed when None).
    Returns per level: cand [B, K], eps [B], h [B, K]."""
    if levels is None:
        levels = M.filter_levels(x, cbs, ids)
    out = []
    for r in levels:
        h, eps = r["h"], r["eps"]
        B, K = h.shape
        margin = 2.0 * eps * (1 + 2.0 ** -16)
        hn = np.where(np.isnan(h), np.float32(np.inf), h)
        run = np.full(B, np.inf, np.float32)
        cand = np.zeros(h.shape, bool)
        keys = []
        with np.errstate(over="ignore", invalid="ignore"):
            for b0 in range(0, K, block):
                bmin = hn[:, b0:b0 + block].min(1)
                run = np.minimum(run, bmin)
                cand[:, b0:b0 + block] = ~(h[:, b0:b0 + block] > (run + margin)[:, None])
                keys.append(np.where(np.isnan(h[:, b0:b0 + block]).any(1), np.nan, bmin))
            thr = run + margin
            if K > block:
                for i, b0 in enumerate(range(0, K, block)):
                    cand[keys[i] > thr, b0:b0 + block] = False
        out.append(dict(cand=cand, eps=eps, h=h))
    return out
