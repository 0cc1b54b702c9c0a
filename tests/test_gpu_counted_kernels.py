"""GPU tests of the device-counted launches (include/rqb200.h "device-counted launches"): each against its host-counted call on
the same inputs.  Rows (tiles) below the live count get the host-counted call's bits; outputs at and past it keep their sentinel
fill.  Live counts 0, inside the capacity and equal to it.  The frontier's capacity write pass against the plain write pass, at
every filter mode and a chunk offset b0 > 0, with room to spare, exactly full, and one row, child or tile short (overflow flag
set, live counts 0, no children offsets for the next level).  `pytest -m gpu`."""
import numpy as np
import pytest
import torch

import exact_oracle as EO
from test_gpu_exact_kernels import FILTERS, child_scores, filters_of, pick_tau, to_device, trie_of

pytestmark = pytest.mark.gpu

SENTINEL = -12345.0


def live_of(n):
    return torch.tensor([n], dtype=torch.int32, device="cuda")


def filled(shape, dtype=torch.float32):
    return torch.full(shape, SENTINEL, dtype=dtype, device="cuda")


def check_rows(got, want, live, what):
    """got[:live] bit-equal to want[:live], got[live:] still the sentinel."""
    assert torch.equal(got[:live].view(torch.int32) if got.dtype == torch.float32 else got[:live],
                       want[:live].view(torch.int32) if want.dtype == torch.float32 else want[:live]), what
    assert bool((got[live:] == SENTINEL).all()), what + " past the live count"


CAP = 300


@pytest.mark.parametrize("live", [0, 1, 129, CAP])
@pytest.mark.parametrize("K", [64, 200, 3100])
def test_split_gemm(live, K):
    from rq_vae_recommender_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(K + live)
    a = torch.randn((CAP, K), device="cuda", generator=g)
    b = torch.randn((96, K), device="cuda", generator=g)
    n = live_of(live)
    out = filled((CAP, 96))
    got = ops.gemm_split(a, ops.SplitOperand(b), out=out, live=n, relu=True)
    want = ops.gemm_split(a[:live], ops.SplitOperand(b), relu=True) if live else torch.empty((0, 96), device="cuda")
    check_rows(got, want, live, "gemm_split")


@pytest.mark.parametrize("live", [0, 5, 64])
def test_add_norm_and_self_attention(live):
    from rq_vae_recommender_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(live)
    R, D, heads, H, h = 64, 96, 2, 4, 2
    inner = heads * 64
    emb = torch.randn((50, D), device="cuda", generator=g)
    ids = torch.randint(0, 20, (R,), device="cuda", generator=g)
    w = torch.rand(D, device="cuda", generator=g)
    n = live_of(live)
    x_g, o_g = filled((R, D)), filled((R, D))
    ops.t5dec_add_norm(x_g, None, w, o_g, 1e-6, emb=emb, ids=ids, offset=7, live=n)
    x_w, o_w = torch.empty((live, D), device="cuda"), torch.empty((live, D), device="cuda")
    if live:
        ops.t5dec_add_norm(x_w, None, w, o_w, 1e-6, emb=emb, ids=ids[:live], offset=7)
    check_rows(x_g, x_w, live, "gather")
    check_rows(o_g, o_w, live, "gather norm")
    delta = torch.randn((R, D), device="cuda", generator=g)
    ops.t5dec_add_norm(x_g, delta, w, o_g, 1e-6, live=n)
    if live:
        ops.t5dec_add_norm(x_w, delta[:live], w, o_w, 1e-6)
    check_rows(x_g, x_w, live, "residual")
    check_rows(o_g, o_w, live, "residual norm")

    qkv = torch.randn((R, 3 * inner), device="cuda", generator=g)
    bias = torch.randn((heads, H, H), device="cuda", generator=g)
    base_k = torch.randn((H, 40, inner), device="cuda", generator=g)
    base_v = torch.randn((H, 40, inner), device="cuda", generator=g)
    anc_in = torch.randint(0, 40, (40, H), dtype=torch.int32, device="cuda", generator=g)
    parent = torch.randint(0, 40, (R,), device="cuda", generator=g)
    cache_k, cache_v = [torch.cat([c, torch.full((H, R, inner), SENTINEL, device="cuda")], 1)[:, :R].contiguous()
                        for c in (base_k, base_v)]
    cache_k[:, :40], cache_v[:, :40] = base_k, base_v
    ck2, cv2 = cache_k.clone(), cache_v.clone()
    anc_g = torch.full((R, H), -7, dtype=torch.int32, device="cuda")
    anc_w = torch.full((R, H), -7, dtype=torch.int32, device="cuda")
    got = ops.t5dec_self_attention(qkv, cache_k, cache_v, bias, h, anc_in, parent, anc_g, live=n)
    got[live:] = SENTINEL                                        # out is a fresh tensor: only rows below live are defined
    if live:
        want = ops.t5dec_self_attention(qkv[:live], ck2, cv2, bias, h, anc_in, parent[:live], anc_w)
        assert torch.equal(got[:live], want)
    assert torch.equal(cache_k, ck2) and torch.equal(cache_v, cv2)
    assert torch.equal(anc_g[:, :h], anc_w[:, :h]) and bool((anc_g[live:] == -7).all())


@pytest.mark.parametrize("live_tiles", [0, 3, 7])
def test_ragged_cross_attention_and_children(live_tiles):
    from rq_vae_recommender_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(live_tiles)
    heads, inner, B = 2, 128, 3
    offsets = torch.tensor([0, 20, 20, 57], dtype=torch.int32, device="cuda")
    k = torch.randn((57, inner), device="cuda", generator=g)
    v = torch.randn((57, inner), device="cuda", generator=g)
    tiles = torch.tensor([[0, 0, 64], [0, 64, 10], [1, 74, 5], [2, 79, 64], [2, 143, 64], [2, 207, 1], [2, 208, 12]],
                         dtype=torch.int32, device="cuda")
    R = 220
    q = torch.randn((R, inner), device="cuda", generator=g)
    rows = int(tiles[live_tiles - 1, 1] + tiles[live_tiles - 1, 2]) if live_tiles else 0
    got = ops.t5rank_cross_attention_ragged(q, k, v, offsets, None, tiles, heads, live=live_of(live_tiles))
    want = ops.t5rank_cross_attention_ragged(q, k, v, offsets, None, tiles[:live_tiles].contiguous(), heads)
    assert torch.equal(got[:rows], want[:rows])

    Kc, n_next = 40, 700                                         # >= 3 R: every child range fits
    logits = torch.randn((R, Kc), device="cuda", generator=g)
    logits[3, 5] = float("nan")
    parent = torch.randn(R, device="cuda", generator=g)
    child = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"),
                       torch.randint(0, 4, (R,), device="cuda", generator=g).cumsum(0)]).int()
    code = torch.randint(0, Kc, (n_next,), dtype=torch.int32, device="cuda", generator=g)
    live = torch.tensor([rows, int(child[rows])], dtype=torch.int32, device="cuda")
    out, bad = filled((1, n_next)), torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.t5rank_children(logits, parent, child, code, R, out, bad, live=live)
    want, want_bad = filled((1, n_next)), torch.zeros(1, dtype=torch.int32, device="cuda")
    if rows:
        ops.t5rank_children(logits[:rows], parent[:rows], child[:rows + 1].contiguous(), code, rows, want, want_bad)
    assert torch.equal(out.view(torch.int32), want.view(torch.int32)) and torch.equal(bad, want_bad)


def frontier_case(mode, b0, Bc=7):
    """A level-1 frontier and a level-2 one of the K = 300, H = 3 trie, with scores, tau and filters as the kernel tests."""
    K, H, N = 300, 3, 3000
    tr = trie_of(K, H, N)
    filt = filters_of(K, H, N, 10, 1024)[mode]
    rs = np.random.RandomState(b0 + 17)
    first = np.stack([child_scores(rs, tr.n[1]) for _ in range(Bc)])
    ch = EO.root_children(first, tr.code[1])
    tau = pick_tau(ch, ["mid", 64, "-inf", 65, "shared", "+inf", 129][:Bc], filt[0], K, 1, b0)
    return tr, to_device(ch, tr.n[1], bool(filt[1])), torch.from_numpy(tau).cuda(), filt[1]


@pytest.mark.parametrize("b0", [0, 3])
@pytest.mark.parametrize("mode", FILTERS)
def test_frontier_capacity(mode, b0):
    from rq_vae_recommender_b200 import ops
    tr, ch, tau, kw = frontier_case(mode, b0)
    counts = ops.t5exact_frontier_count(ch, tr.levels.code[1], tau, tr.K, 1, tr.levels.child[1], b0, **kw)
    scan = torch.zeros((3, 8), dtype=torch.int32, device="cuda")
    scan[:, 1:] = counts.cumsum(1)
    R, C, T = scan[:, -1].tolist()
    assert R > 0
    want = ops.t5exact_frontier_write(ch, tr.levels.code[1], tau, tr.K, 1, tr.levels.child[1], tr.levels.code[2], scan, (R, C, T),
                                      b0, **kw)
    for caps, over in [((R + 9, C + 9, T + 2), False), ((R, C, T), False), ((R - 1, C, T), True), ((R, C - 1, T), True),
                       ((R, C, T - 1), True)]:
        overflow = torch.zeros(1, dtype=torch.int32, device="cuda")
        got2, live2 = ops.t5exact_frontier_capacity(ch, tr.levels.code[1], tau, tr.K, 1, tr.levels.child[1], tr.levels.code[2],
                                                    scan, caps, overflow, b0, **kw)
        if over:
            assert overflow.item() == 1 and live2.tolist() == [0, 0, 0]
            assert not bool((got2.children.offsets != 0).any())
            continue
        assert overflow.item() == 0 and live2.tolist() == [R, C, T]
        assert torch.equal(got2.children.offsets, scan[1])
        pairs = [(got2.code, want.code, R), (got2.parent, want.parent, R), (got2.score.view(torch.int32),
                 want.score.view(torch.int32), R), (got2.tiles, want.tiles, T), (got2.child, want.child, R + 1),
                 (got2.children.node, want.children.node, C), (got2.children.code, want.children.code, C),
                 (got2.children.parent, want.children.parent, C)] + ([(got2.key, want.key, R)] if kw else [])
        for g, w, n in pairs:
            assert torch.equal(g[:n], w[:n])
