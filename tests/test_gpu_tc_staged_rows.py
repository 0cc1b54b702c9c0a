"""The wgmma tokeniser stages each tile's fp32 rows in its shared-memory ring with one bulk copy per row and 128 columns per
stage, ahead of the tile.  These cases exercise what that staging depends on: the caller's row stride (ldx = D, D + 4,
D + 64), widths whose last stage is half full (D = 64, 192, 704), a last tile of 1 or 63 rows or a 65-row remainder, and
CTAs that convert three or more tiles, at a 3-stage ring and at a 4-stage ring whose stages per tile (x stages plus
codebook stages) are not a multiple of its depth.  Ids are checked against the exact CUDA-core kernel; a strided view must
give the same ids and stats words as its contiguous copy.  All of it is `pytest -m gpu`."""
import numpy as np
import pytest
import torch

from parity import assert_ids_match

TX_R = 64                                       # rows per tile of the kernel


@pytest.fixture(scope="module")
def ops():
    from rq_vae_recommender_b200 import ops as _ops
    return _ops


def problem(n, D, K, L, seed):
    """Seeded unit rows and L codebooks drawn from the level residuals of the first rows plus a little jitter, so every
    code attracts rows and near-ties are realistic (the walk is torch fp32 on the device)."""
    m = min(max(n, K, 4096), 8192)
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((max(n, m), D))
    x = (x / np.sqrt((x * x).sum(1, keepdims=True))).astype(np.float32)
    res = torch.from_numpy(x[:m]).cuda()
    cbs = []
    for _ in range(L):
        idx = torch.from_numpy(rng.choice(m, K, replace=False)).cuda()
        cb = res[idx] + torch.from_numpy(rng.standard_normal((K, D), dtype=np.float32) * np.float32(0.5 / np.sqrt(D))).cuda()
        cbs.append(cb)
        res = res - cb[((cb * cb).sum(1)[None, :] - 2.0 * (res @ cb.t())).argmin(1)]
    return x[:n], cbs


def strided(x, ldx):
    """x as a [B, D] view of a [B, ldx] buffer whose padding columns hold NaN: a kernel that read them would show it."""
    buf = torch.full((x.shape[0], ldx), float("nan"), device="cuda")
    buf[:, :x.shape[1]] = torch.from_numpy(x).cuda()
    view = buf[:, :x.shape[1]]
    assert view.stride(0) == ldx
    return view


def run(ops, xd, state):
    stats = torch.zeros(4, dtype=torch.int32, device="cuda")
    ids = ops.rq_tokenize_tc(xd, state=state, stats=stats)
    torch.cuda.synchronize()
    return ids.cpu().numpy(), stats.cpu().numpy()


def check_case(ops, x, cbs, ldx, what):
    """Contiguous x against the exact kernel (at most max(2, B / 2000) rows differ, only on float64-classified near-ties),
    then the strided view against the contiguous run: same ids and stats words."""
    state = ops.TcState(cbs)
    xd = torch.from_numpy(x).cuda()
    ids, stats = run(ops, xd, state)
    ref = ops.rq_tokenize(xd, cbs).cpu().numpy()
    cbs_h = [c.cpu().numpy() for c in cbs]
    n_tie = assert_ids_match(ids, ref, x, cbs_h, f"{what} vs exact kernel")
    assert n_tie <= max(2, len(x) // 2000), (what, n_tie)
    ids_s, stats_s = run(ops, strided(x, ldx), state)
    assert np.array_equal(ids_s, ids), (what, int((ids_s != ids).any(1).sum()))
    assert np.array_equal(stats_s, stats), (what, stats_s.tolist(), stats.tolist())
    print(f"{what}: near-ties {n_tie}, stats {stats.tolist()}")


@pytest.mark.gpu
@pytest.mark.parametrize("D", [64, 192, 704, 768])
@pytest.mark.parametrize("pad", [0, 4, 64])
def test_tc_row_stride(ops, D, pad):
    """ldx = D + pad; D = 64, 192 and 704 end in a half-full x stage.  1 000 rows end in a partial tile."""
    K, L, B = 256, 3, 1000
    x, cbs = problem(B, D, K, L, seed=17 * D + pad)
    check_case(ops, x, cbs, D + pad, f"D={D} ldx={D + pad}")


@pytest.mark.gpu
@pytest.mark.parametrize("tail", [1, 63, 65])
@pytest.mark.parametrize("D", [192, 768])
def test_tc_last_tile_rows(ops, D, tail):
    """A batch of 2 SMs' worth of full tiles plus `tail` rows: the last tile holds 1 or 63 rows, or a full tile is followed
    by one of a single row."""
    K, L = 256, 2
    B = 2 * torch.cuda.get_device_properties(0).multi_processor_count * TX_R + tail
    x, cbs = problem(B, D, K, L, seed=D + tail)
    check_case(ops, x, cbs, D + 4, f"D={D} B={B} (tail {tail})")


@pytest.mark.gpu
@pytest.mark.parametrize("D,K,L", [(768, 512, 3), (704, 256, 1)])
def test_tc_three_tiles_per_cta(ops, D, K, L):
    """Every CTA converts three or more tiles.  (768, 512, 3) runs on a 3-stage ring; (704, 256, 1) on a 4-stage ring with
    6 x stages + 11 codebook stages = 17 stages per tile, so consecutive tiles start on different slots and phases."""
    from rq_vae_recommender_b200 import _lib
    nb = _lib.load().rqb200_tokenize_tc_ring_stages(D, K, L)
    per_tile = (D + 127) // 128 + (D // 64) * (K // 256) * L
    assert (nb, per_tile % nb != 0) == ((3, False) if K == 512 else (4, True)), (nb, per_tile)
    B = (3 * torch.cuda.get_device_properties(0).multi_processor_count + 1) * TX_R - 5
    x, cbs = problem(B, D, K, L, seed=D * K + L)
    check_case(ops, x, cbs, D + 64, f"D={D} K={K} L={L} B={B} ({nb}-stage ring, {per_tile} stages per tile)")
