"""Parity protocol helpers shared by the CPU and GPU tests."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


# ---- the parity protocol of SURVEY 8(c): ids exact except on float64-classified near ties -------------
TAU = 1e-5
TAU_ABS = 1e-6      # ~16 fp32 ulps of the operands xx + cc: below that the reference's own fp32 distances are summation-order noise


def assert_ids_match(ids, ref_ids, res, codebooks, what=""):
    """ids/ref_ids [B,L].  Rows may differ from the fp32 reference only where the float64 oracle says BOTH answers are
    near-tied with the float64 minimum at the first differing level: distance excess (d - d_min) <= TAU * d_min, or, for rows
    that all but coincide with a code (d_min is then a cancellation residue of terms ~1), (d - d_min) <= TAU_ABS (xx + cc).
    (Several codes can be tied at once -- near-duplicate codes -- so membership in {best, runner-up} is not required.)
    Returns the number of such near-tie rows."""
    from oracle import rq_oracle as O
    ids = np.asarray(ids).astype(np.int64).reshape(len(ids), -1)
    ref_ids = np.asarray(ref_ids).astype(np.int64).reshape(len(ref_ids), -1)
    bad = np.nonzero((ids != ref_ids).any(axis=1))[0]
    if len(bad) == 0:
        return 0
    cbs64 = [np.asarray(c, np.float64) for c in codebooks]
    r64 = np.asarray(res, np.float64)[bad]
    for r in range(len(bad)):
        a, b = ids[bad[r]], ref_ids[bad[r]]
        l = int(np.nonzero(a != b)[0][0])
        resid = r64[r].copy()
        for j in range(l):                       # both chains are identical up to the first differing level
            resid -= cbs64[j][a[j]]
        d = O.quantize_dist(resid[None, :], cbs64[l])[0]
        dmin = d.min()
        scale = (resid * resid).sum() + (cbs64[l][int(d.argmin())] ** 2).sum()
        for k, who in ((int(a[l]), "impl"), (int(b[l]), "ref")):
            exc = d[k] - dmin
            assert exc <= TAU * max(abs(dmin), 1e-30) or exc <= TAU_ABS * max(scale, 1e-30), (
                f"{what}: row {bad[r]} level {l}: impl {a} vs ref {b}; {who}'s code {k} is {exc:.3e} above the float64 "
                f"minimum {dmin:.3e} (code {int(d.argmin())}; operand scale {scale:.3e})")
    return len(bad)


def assert_no_worse_than(ids, ref, x, cbs, what=""):
    """Rows where ids differ from ref: at the first differing level, the float64 distance of ids' code exceeds that of ref's
    code by at most the near-tie tolerance above.  The exact CUDA-core kernel sums each dot product sequentially, the
    tensor-core tokeniser's re-rank in lane order; on near-duplicate codes either one can land a few ulps past that tolerance
    from the float64 minimum, so this is the comparison that holds between the two kernels.  Returns the number of differing
    rows."""
    bad = np.nonzero((ids != ref).any(1))[0]
    c64 = [np.asarray(c, np.float64) for c in cbs]
    for r in bad:
        l = int(np.nonzero(ids[r] != ref[r])[0][0])
        res = x[r].astype(np.float64) - sum(c64[j][ids[r, j]] for j in range(l))
        d = ((res[None, :] - c64[l]) ** 2).sum(1)
        scale = (res * res).sum() + (c64[l][int(d.argmin())] ** 2).sum()
        exc = d[ids[r, l]] - d[ref[r, l]]
        assert exc <= max(TAU * abs(d.min()), TAU_ABS * scale), (
            f"{what}: row {r} level {l}: code {ids[r, l]} is {exc:.3e} further than {ref[r, l]} (scale {scale:.3e})")
    return len(bad)


def rel_err(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))
