"""The wgmma tokeniser's result for a row may not depend on where the row lands: which tile, which row of the tile, which CTA,
or how far round the codebook ring that CTA is.  A seeded batch is tokenised whole and then as consecutive row slices of
awkward sizes (single rows, tiles of 63 / 64 / 65 rows, an odd tile count, fewer tiles than SMs, a persistent grid whose last
tile is partial); the ids must be bit-identical and the re-rank counters must add up to the whole batch's.  Deep hierarchies
(L = 8, up to 7 Gram tables summed per score) are checked against the exact CUDA-core kernel.  All of it is `pytest -m gpu`."""
import numpy as np
import pytest
import torch

import inputs as I
from parity import assert_ids_match

TX_R = 64                                       # rows per tile of the kernel


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def ops():
    from rq_vae_recommender_b200 import ops as _ops
    return _ops


def run(ops, xd, state):
    stats = torch.zeros(4, dtype=torch.int32, device="cuda")
    ids = ops.rq_tokenize_tc(xd, state=state, stats=stats)
    torch.cuda.synchronize()
    return ids.cpu().numpy(), stats.cpu().numpy()


def slice_sizes(n):
    """Consecutive slices covering n rows; the last one takes what is left."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = [1, 63, 64, 65, 129, 7 * TX_R, (sms // 4) * TX_R - 5, (2 * sms + 1) * TX_R - 23]
    assert sum(sizes) < n
    return sizes + [n - sum(sizes)]


def problem(n, D, K, L, seed):
    x = I.unit_rows(seed, n, D)
    m = max(8192, K)
    _, cbs = I.rq_problem(m, D, K, L, seed=seed, x=I.unit_rows(seed, m, D))
    return x, cbs


@pytest.mark.gpu
@pytest.mark.parametrize("n,D,K,L", [(65536, 768, 256, 3), (24576, 768, 1280, 3)])
def test_tc_row_slices_give_the_batch_ids(ops, n, D, K, L):
    """(768, 256, 3) is the benchmark's shape (4-stage ring); (768, 1280, 3) is scored in five 256-code blocks per level on
    a 3-stage ring.  A second run on the same state gives the same ids and counters."""
    x, cbs = problem(n, D, K, L, seed=D + K + L)
    state = ops.TcState([dev(c) for c in cbs])
    xd = dev(x)
    ids, stats = run(ops, xd, state)
    ids2, stats2 = run(ops, xd, state)
    assert np.array_equal(ids, ids2) and np.array_equal(stats, stats2), (stats.tolist(), stats2.tolist())
    total = np.zeros(3, dtype=np.int64)
    a = 0
    for size in slice_sizes(n):
        part, st = run(ops, xd[a:a + size], state)
        assert np.array_equal(part, ids[a:a + size]), (a, size, int((part != ids[a:a + size]).any(1).sum()))
        total += st[:3]
        a += size
    assert a == n
    assert total.tolist() == stats[:3].tolist(), (total.tolist(), stats[:3].tolist())
    print(f"slices D={D} K={K} L={L} n={n}: stats {stats.tolist()}")


@pytest.mark.gpu
@pytest.mark.parametrize("D,K", [(128, 256), (128, 512), (768, 256)])
def test_tc_eight_levels_vs_exact_kernel(ops, D, K):
    """L = 8: the level-7 score sums 7 Gram rows per code; ids against the exact kernel on every row of a multi-tile batch."""
    L, n = 8, 4096
    x, cbs = problem(n, D, K, L, seed=3 * D + K)
    state = ops.TcState([dev(c) for c in cbs])
    ids, stats = run(ops, dev(x), state)
    ref = ops.rq_tokenize(dev(x), [dev(c) for c in cbs]).cpu().numpy()
    n_tie = assert_ids_match(ids, ref, x, cbs, f"tc L=8 D={D} K={K} vs exact kernel")
    assert n_tie <= max(2, n // 2000), n_tie
    print(f"L=8 D={D} K={K}: near-ties {n_tie}, stats {stats.tolist()}")
