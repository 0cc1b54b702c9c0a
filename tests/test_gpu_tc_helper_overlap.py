"""The wgmma tokeniser's hand-offs between its scoring warpgroup and its helper warpgroup (conversion and exact re-rank),
under the heaviest load they can carry: every row of every level goes to the exact re-rank, and every CTA runs several tiles,
so the helper re-ranks the last level of one tile while the scorer runs the first level of the next.  Each level's
codebook repeats code 17 at codes 90, 200 and K - 1, and every row sits next to the sum of the codes 17 of all levels, so
each level's candidates always include the four equal codes.  The batch of 3 x 132 x 64 + 17 rows gives 3 or 4 tiles per
CTA on a 132-SM H100.  Ids must equal the exact CUDA-core kernel's, and the re-rank counters must add up over row slices of
the batch.  All of it is `pytest -m gpu`."""
import numpy as np
import pytest
import torch

import inputs as I

pytestmark = pytest.mark.gpu

TX_R = 64                                       # rows per tile of the kernel
N = 3 * 132 * TX_R + 17
D = 768
TIE = 17


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def ops():
    from rq_vae_recommender_b200 import ops as _ops
    return _ops


def tied_problem(n, K, L, seed):
    """Level-l codes are gaussian of norm about 4^-l; codes 90, 200 and K - 1 repeat code 17.  Rows are the sum of the codes
    17 of all levels plus jitter far below the last level's code spacing, so the nearest code of every level is code 17 and
    its three copies, an exact four-way tie that the first index wins."""
    cbs = []
    for l in range(L):
        c = I.randn(seed + l, K, D) * np.float32(0.25 ** l / np.sqrt(D))
        for k in (90, 200, K - 1):
            c[k] = c[TIE]
        cbs.append(c)
    base = sum(c[TIE].astype(np.float64) for c in cbs)
    jitter = I.randn(seed + 100, n, D).astype(np.float64) * (0.01 * 0.25 ** (L - 1) / np.sqrt(D))
    return (base[None, :] + jitter).astype(np.float32), cbs


def run(ops, xd, state):
    stats = torch.zeros(4, dtype=torch.int32, device="cuda")
    ids = ops.rq_tokenize_tc(xd, state=state, stats=stats)
    torch.cuda.synchronize()
    return ids.cpu().numpy(), stats.cpu().numpy()


@pytest.mark.parametrize("K", [256, 1280])
@pytest.mark.parametrize("L", [1, 2, 8])
def test_tc_every_row_reranked_over_several_tiles(ops, K, L):
    """K = 256 runs the single-accumulator kernel on a 4-stage ring, K = 1280 the blocked kernel (five 256-code blocks per
    level) on a 3-stage ring."""
    from rq_vae_recommender_b200 import _lib
    assert _lib.load().rqb200_tokenize_tc_ring_stages(D, K, L) == (4 if K == 256 else 3)
    x, cbs = tied_problem(N, K, L, seed=K + L)
    cds = [dev(c) for c in cbs]
    state = ops.TcState(cds)
    xd = dev(x)
    ids, stats = run(ops, xd, state)
    assert stats[0] == N * L, (stats.tolist(), N * L)          # every row-level re-ranked
    assert stats[1] >= 4 * N * L and stats[2] == N * L, stats.tolist()
    ref = ops.rq_tokenize(xd, cds).cpu().numpy()
    assert np.array_equal(ids, ref), int((ids != ref).any(1).sum())
    assert (ids == TIE).all()
    # the same rows as consecutive slices: single rows, partial tiles, fewer tiles than SMs, one to two tiles per CTA
    total = np.zeros(3, dtype=np.int64)
    a = 0
    for size in [1, 63, 65, 129, 61 * TX_R + 5, 200 * TX_R - 23]:
        part, st = run(ops, xd[a:a + size], state)
        assert np.array_equal(part, ids[a:a + size]), (a, size)
        total += st[:3]
        a += size
    part, st = run(ops, xd[a:], state)
    assert np.array_equal(part, ids[a:]), (a, N - a)
    total += st[:3]
    assert total.tolist() == stats[:3].tolist(), (total.tolist(), stats[:3].tolist())
