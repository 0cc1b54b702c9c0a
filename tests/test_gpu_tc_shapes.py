"""The wgmma tokeniser (csrc/rq_tcx.cu, prepared by csrc/rq_tc.cu) across the shapes rqb200_tokenize_tc_supported accepts:
every width D = 64 .. 768 with every codebook size K = 256 .. 2048, every 3-stage codebook ring whose stages per tile are
not a multiple of 3 (a CTA's next tile then starts partway round the ring, with the mbarrier phase flipped), adversarial
inputs at such a ring, and zero-padded widths.  Ids are checked against the exact CUDA-core kernel on every row and against
the fp32 oracle on a sample.  The ring-depth query test needs no GPU; the rest is `pytest -m gpu`."""
import numpy as np
import pytest
import torch

import tc_blocked_model as MB
import tc_filter_model as M
from oracle import rq_oracle as O
from parity import assert_ids_match, assert_no_worse_than

TX_R = 64                                       # rows per tile of the kernel
WIDTHS = list(range(64, 769, 64))
SIZES = list(range(256, 2049, 256))
SUPPORTED = [(D, K, L) for D in WIDTHS for K in SIZES for L in range(1, 9)]


def stages_per_tile(D, K, L):
    """32 KB ring stages a tile consumes: one per (level, 256-code block, 64-wide k chunk)."""
    return (D // 64) * (K // 256) * L


def _uneven_three_stage_shapes():
    """Every supported shape whose ring has 3 stages and whose stages per tile are not a multiple of 3, from the library's
    own ring-depth query (empty if the library is not built; the ring-depth test then fails)."""
    from rq_vae_recommender_b200 import _lib
    try:
        lib = _lib.load()
    except (_lib.Rqb200Error, OSError):
        return []
    return [s for s in SUPPORTED if lib.rqb200_tokenize_tc_ring_stages(*s) == 3 and stages_per_tile(*s) % 3]


UNEVEN = _uneven_three_stage_shapes()
# plus 3 stages with an even split, and 4 stages with 3 or 11 stages per tile
RING = UNEVEN + [(768, 1280, 3), (704, 1536, 2), (192, 256, 1), (704, 256, 1)]


def test_ring_stages_of_every_supported_shape():
    """rqb200_tokenize_tc_ring_stages (the depth rq_tcx.cu's launcher uses) on all 768 supported shapes: 3 or 4 stages, 4 at
    K = 256, 3 exactly where 4 stages do not fit beside the x image and the candidate words."""
    from rq_vae_recommender_b200 import _lib
    _lib.build()
    lib = _lib.load()
    assert len(SUPPORTED) == 768 and all(lib.rqb200_tokenize_tc_supported(*s) for s in SUPPORTED)
    nb = {s: lib.rqb200_tokenize_tc_ring_stages(*s) for s in SUPPORTED}
    assert set(nb.values()) == {3, 4}
    assert all(nb[s] == 4 for s in SUPPORTED if s[1] == 256)
    three = {s for s in SUPPORTED if nb[s] == 3}
    expect = ({(768, K, L) for K in SIZES if K >= 512 for L in range(1, 9)} |
              {(704, K, L) for K in SIZES if K >= 1280 for L in range(1, 9)} |
              {(640, 2048, L) for L in range(5, 9)})
    assert three == expect and len(three) == 92
    uneven = [s for s in SUPPORTED if nb[s] == 3 and stages_per_tile(*s) % 3]
    assert UNEVEN == uneven and len(uneven) == 21
    assert {s[0] for s in uneven} == {640, 704}
    for s in [(32, 256, 3), (700, 256, 1), (832, 256, 3), (768, 128, 3), (768, 2304, 3), (768, 384, 3), (768, 256, 0),
              (768, 256, 9)]:
        assert lib.rqb200_tokenize_tc_ring_stages(*s) == 0, s


# ---------------------------------------------------------------------------------------------------------------- GPU
def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def ops():
    from rq_vae_recommender_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def problem():
    """make(n, D, K, L, seed) -> (x [n, D], L codebooks [K, D]): seeded unit rows, and codebooks whose level-l codes are rows
    of the level-l residual of the first m = min(max(n, K, 4096), 8192) rows plus 0.5 / sqrt(D) gaussian jitter, so every code
    attracts rows and near-ties are realistic (like inputs.rq_problem).  The walk's argmin is torch fp32 on the GPU: a float64
    walk on the host is too slow at K = 2048, L = 8, D = 768, and the walk need not be the exact chain."""
    def make(n, D, K, L, seed):
        m = min(max(n, K, 4096), 8192)
        rng = np.random.default_rng(seed)
        x = rng.standard_normal((max(n, m), D))
        x = (x / np.sqrt((x * x).sum(1, keepdims=True))).astype(np.float32)
        res = dev(x[:m])
        cbs = []
        for _ in range(L):
            idx = torch.from_numpy(rng.choice(m, K, replace=False)).cuda()
            cb = res[idx] + dev(rng.standard_normal((K, D), dtype=np.float32) * np.float32(0.5 / np.sqrt(D)))
            cbs.append(cb)
            res = res - cb[((cb * cb).sum(1)[None, :] - 2.0 * (res @ cb.t())).argmin(1)]
        return x[:n], [host(c) for c in cbs]
    return make


def run_tc(ops, x, cbs=None, state=None):
    stats = torch.zeros(4, dtype=torch.int32, device="cuda")
    ids = ops.rq_tokenize_tc(x if torch.is_tensor(x) else dev(x), None if cbs is None else [dev(c) for c in cbs],
                             state=state, stats=stats)
    torch.cuda.synchronize()
    return host(ids), host(stats)


def exact(ops, x, cbs):
    return host(ops.rq_tokenize(dev(x), [dev(c) for c in cbs]))


def ring_batch():
    """Rows for (2 SMs + 1) tiles, the last one partial: every CTA of the persistent grid converts at least two tiles."""
    return (2 * torch.cuda.get_device_properties(0).multi_processor_count + 1) * TX_R - 23


def check(ops, ids, x, cbs, what):
    """The yardsticks of every sweep case: ids in range; the exact kernel on all rows (at most max(2, B / 2000) rows differ,
    only on float64-classified near-ties); the fp32 oracle on the first 256 rows and every row of the last tile.  Returns
    the number of rows that differ from the exact kernel."""
    B, L, K = len(x), len(cbs), cbs[0].shape[0]
    assert ids.shape == (B, L) and ids.min() >= 0 and ids.max() < K, (what, ids.shape, ids.min(), ids.max())
    n_tie = assert_ids_match(ids, exact(ops, x, cbs), x, cbs, f"{what} vs exact kernel")
    assert n_tie <= max(2, B // 2000), (what, n_tie)
    rows = np.union1d(np.arange(min(256, B)), np.arange((B - 1) // TX_R * TX_R, B))
    assert_ids_match(ids[rows], O.rq_tokenize(x[rows], cbs), x[rows], cbs, f"{what} vs oracle")
    return n_tie


@pytest.mark.gpu
@pytest.mark.parametrize("D,K,L", [(D, K, 1 + (D // 64 + K // 256) % 8) for D in WIDTHS for K in SIZES])
def test_tc_every_width_and_codebook_size(ops, problem, D, K, L):
    """All 96 (D, K) pairs, L cycling so every L meets every D and every K; 1 000 rows end in a partial tile."""
    B = 1000
    x, cbs = problem(B, D, K, L, seed=D * 10000 + K + L)
    ids, stats = run_tc(ops, x, cbs)
    n_tie = check(ops, ids, x, cbs, f"tc D={D} K={K} L={L}")
    print(f"sweep D={D} K={K} L={L}: near-ties {n_tie}, stats {stats.tolist()}")


@pytest.mark.gpu
@pytest.mark.parametrize("D,K,L", RING)
def test_tc_ring_phase_across_tiles(ops, problem, D, K, L):
    """Shapes where a CTA's tiles start on different ring slots (or, for the last four, reference rings that do not), at
    enough rows that every CTA converts two or more tiles.  Two runs on one prepared state agree on every id and every
    stats word."""
    B = ring_batch()
    x, cbs = problem(B, D, K, L, seed=D * 10000 + K + 7 * L)
    state = ops.TcState([dev(c) for c in cbs])
    xd = dev(x)
    ids, stats = run_tc(ops, xd, state=state)
    ids2, stats2 = run_tc(ops, xd, state=state)
    assert np.array_equal(ids, ids2) and np.array_equal(stats, stats2), (stats.tolist(), stats2.tolist())
    n_tie = check(ops, ids, x, cbs, f"tc ring D={D} K={K} L={L}")
    print(f"ring D={D} K={K} L={L} B={B} ({stages_per_tile(D, K, L)} stages per tile): near-ties {n_tie}, "
          f"stats {stats.tolist()}")


@pytest.mark.gpu
@pytest.mark.parametrize("D,K,L", [(704, 1280, 2), (640, 2048, 5)])
def test_tc_rerank_count_at_an_uneven_ring(ops, problem, D, K, L):
    """stats[0] (rows re-ranked) against the CPU model of the blocked selection, with the slack of
    test_gpu_tc_large_k.py::test_tc_rerank_count_matches_the_cpu_model.  A stale or misplaced ring stage can leave the ids
    right (the re-rank repairs them) and still show as a wrong candidate count."""
    n = 1024
    x, cbs = problem(n, D, K, L, seed=D + K + L)
    ids, stats = run_tc(ops, x, cbs)
    ref = O.rq_tokenize(x, cbs)
    assert_ids_match(ids, ref, x, cbs, f"tc/rerank D={D} K={K} L={L}")
    model = sum(int((lv["cand"].sum(1) > 1).sum()) for lv in MB.filter_levels_blocked(x, cbs, ref))
    print(f"rerank D={D} K={K} L={L}: kernel {int(stats[0])} rows, CPU model {model} of {n * L} row-levels")
    assert abs(int(stats[0]) - model) <= 0.01 * n * L + 16, (int(stats[0]), model)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", M.ADVERSARIAL_KINDS)
def test_tc_adversarial_rounding_at_an_uneven_ring(ops, kind):
    D, K, L = 704, 1280, 2
    x, cbs = M.adversarial_problem(kind, D=D, K=K, L=L, n=300)
    ids, stats = run_tc(ops, x, cbs)
    assert ids.shape == (300, L) and ids.min() >= 0 and ids.max() < K
    assert_ids_match(ids, O.rq_tokenize(x, cbs), x, cbs, f"tc/adversarial/{kind} D={D} K={K} L={L}")
    assert_no_worse_than(ids, exact(ops, x, cbs), x, cbs, f"tc-vs-simt/adversarial/{kind} D={D} K={K} L={L}")


@pytest.mark.gpu
def test_tc_overflow_rows_fill_the_rerank_queue_on_multi_tile_ctas(ops):
    """tiny_and_huge rows tiled to the ring sweep's batch at D = 704, K = 1280, L = 2 (110 stages per tile on a 3-stage
    ring).  The first 100 of every 300 rows are rescaled to overflow fp16, so every code of theirs is re-ranked and most
    tiles queue all 64 rows.  A row's ids may not depend on which tile, CTA or ring slot it met."""
    D, K, L, n = 704, 1280, 2, 300
    x0, cbs = M.adversarial_problem("tiny_and_huge", D=D, K=K, L=L, n=n)
    x0[:100] *= np.float32(1e5) / np.abs(x0[:100]).max(1, keepdims=True)
    with np.errstate(over="ignore"):
        over = np.isinf(x0.astype(np.float16)).any(1)
    assert over[:100].all() and not over[100:].any()
    B = ring_batch()
    rep = np.arange(B) % n
    x = x0[rep]
    ids, stats = run_tc(ops, x, cbs)
    assert ids.shape == (B, L) and ids.min() >= 0 and ids.max() < K
    assert np.array_equal(ids, ids[:n][rep])
    assert_ids_match(ids[:n], O.rq_tokenize(x0, cbs), x0, cbs, "tc/tiled tiny_and_huge vs oracle")
    n_diff = assert_no_worse_than(ids, exact(ops, x, cbs), x, cbs, "tc-vs-simt/tiled tiny_and_huge")
    n_over = int(over[rep].sum())
    print(f"tiled tiny_and_huge B={B}: {n_over} overflow rows, {n_diff} rows differ from the exact kernel, "
          f"stats {stats.tolist()}")
    assert stats[0] >= n_over * L and stats[1] >= n_over * L * K, (stats.tolist(), n_over)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 63, 65, 700])
def test_tc_zero_padded_widths(ops, problem, D):
    """Widths that TcState zero-pads to the next multiple of 64, against the exact kernel at the caller's width."""
    B, K, L = 2000, 512, 3
    x, cbs = problem(B, D, K, L, seed=D + 4242)
    state = ops.TcState([dev(c) for c in cbs])
    assert state.D_in == D and state.D == (D + 63) // 64 * 64
    ids, stats = run_tc(ops, x, state=state)
    n_tie = check(ops, ids, x, cbs, f"tc padded D={D}")
    print(f"padded D={D} -> {state.D}: near-ties {n_tie}, stats {stats.tolist()}")
