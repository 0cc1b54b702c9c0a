"""GPU tests of the corpus item table (ops.SidItemTable), the device-side rank histogram (ops.sid_topk_rank_hist), the
device-side TopKAccumulator and EncoderDecoderRetrievalModel.generate_items / item_of, against the numpy oracle item_oracle
and the UNMODIFIED reference's TopKAccumulator (tests/golden/metrics.npz)."""
import numpy as np
import pytest
import torch

import item_oracle as I
from test_gpu_generate import dev, history, small_model
from test_item_oracle import corpus, golden_cases, queries

pytestmark = pytest.mark.gpu

HEADER = np.dtype([("C", "<i4"), ("K", "<i4"), ("N", "<i8"), ("U", "<i4"), ("G", "<i4"), ("width", "<i4"), ("cols", "<i4"),
                   ("row", "<u8"), ("key", "<u8"), ("start", "<u8")])


def table_arrays(t):
    """The header, row [N] and start [U + 1] arrays of a built table, read from its workspace."""
    ws = t.ws.cpu().numpy()
    h = np.frombuffer(ws[:HEADER.itemsize].tobytes(), dtype=HEADER)[0]
    N, U = int(h["N"]), int(h["U"])
    row = np.frombuffer(ws[int(h["row"]):int(h["row"]) + 4 * N].tobytes(), dtype=np.int32)
    start = np.frombuffer(ws[int(h["start"]):int(h["start"]) + 4 * (U + 1)].tobytes(), dtype=np.int32)
    return h, row, start


@pytest.mark.parametrize("N,C,K", [(0, 3, 256), (1, 3, 256), (600, 1, 16), (600, 5, 2048), (600, 8, 256), (12101, 3, 256),
                                   (1 << 20, 3, 256), (1 << 20, 4, 65536)])
def test_build_matches_stable_argsort(N, C, K):
    from rq_vae_recommender_b200 import ops
    ids = corpus(N, C, K, seed=N + C)
    if N >= 12101:
        rng = np.random.default_rng(N)
        ids = rng.integers(0, K, size=(N, C))
        ids[::7] = ids[1::7][: len(ids[::7])]                                   # collisions
        ids[::97, C - 1] = K                                                   # unretrievable rows
    t = ops.SidItemTable(dev(ids), K)
    o = I.build(ids, K)
    h, row, start = table_arrays(t)
    assert (int(h["C"]), int(h["K"]), int(h["N"]), int(h["U"])) == (C, K, N, len(o["keys"]))
    assert np.array_equal(row, o["row"]) and np.array_equal(start, o["start"])
    assert t.nbytes == ops._lib.load().rqb200_sid_items_workspace_bytes(N, C, K)


@pytest.mark.parametrize("K", [16, 256, 2048])
@pytest.mark.parametrize("C", [1, 3, 5, 8])
def test_lookup_vs_oracle(K, C):
    from rq_vae_recommender_b200 import ops
    ids = corpus(600, C, K, seed=K * C)
    table, o = ops.SidItemTable(dev(ids), K), I.build(ids, K)
    q = queries(ids, K, C, np.random.default_rng(K + C), P=2000)
    assert np.array_equal(table.lookup(dev(q[:, :C])).cpu().numpy(), I.lookup(o, q[:, :C]))
    assert np.array_equal(table.lookup(dev(q), with_dedup=True).cpu().numpy(), I.lookup(o, q, with_dedup=True))
    strided = dev(np.concatenate([q, q], axis=1))[:, :C + 1]                   # a row stride wider than the tuple
    assert np.array_equal(table.lookup(strided, with_dedup=True).cpu().numpy(), I.lookup(o, q, with_dedup=True))
    assert table.lookup(dev(q[:0, :C])).shape == (0,)


def crafted_beams(ids, K, C, B, k, rng):
    """Beams drawn from corpus tuples, absent tuples and tuples with out-of-range ids; two beams with one tuple, descending
    log-probabilities with -inf fillers at the tail and a NaN."""
    q = queries(ids, K, C, rng, P=400)[:, :C]
    gen = q[rng.integers(0, len(q), size=(B, k))]
    if k > 3:
        gen[:, 3] = gen[:, 1]
    lp = -np.sort(rng.exponential(size=(B, k)).astype(np.float32), axis=1)
    lp[:, k - k // 4:] = -np.inf
    if k > 2:
        lp[0, 2] = np.nan
    return gen, lp


RETRIEVE = [(B, k, n) for i, (B, k) in enumerate([(B, k) for B in (1, 7, 640) for k in (1, 10, 32, 1024)])
            for n in ((1, 10, 100, 4096)[i % 4],)] + [(7, k, n) for k in (1, 10, 32, 1024) for n in (1, 10, 100, 4096)]


@pytest.mark.parametrize("B,k,n", sorted(set(RETRIEVE)))
def test_retrieve_crafted_vs_oracle(B, k, n):
    from rq_vae_recommender_b200 import ops
    K, C = 16, 3
    ids = corpus(600, C, K, seed=B + k)
    table, o = ops.SidItemTable(dev(ids), K), I.build(ids, K)
    gen, lp = crafted_beams(ids, K, C, B, k, np.random.default_rng(B * k + n))
    for log_probas in (lp, None):
        items, beam, count = table.retrieve(dev(gen), None if log_probas is None else dev(log_probas), n)
        wi, wb, wc = I.retrieve(o, gen, log_probas, n)
        assert items.dtype == torch.int64 and beam.dtype == torch.int32 and count.dtype == torch.int32
        assert np.array_equal(items.cpu().numpy(), wi) and np.array_equal(beam.cpu().numpy(), wb)
        assert np.array_equal(count.cpu().numpy(), wc)


def test_retrieve_limits_and_arguments():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200._lib import Rqb200Error
    ids = corpus(600, 3, 16, seed=3)
    table = ops.SidItemTable(dev(ids), 16)
    gen = dev(ids[:8].reshape(2, 4, 3))
    with pytest.raises(Rqb200Error):
        table.retrieve(gen, None, 4097)
    with pytest.raises(Rqb200Error):
        table.retrieve(dev(np.zeros((1, 1025, 3), dtype=np.int64)), None, 10)
    with pytest.raises(ValueError):
        table.retrieve(gen[:, :, :2], None, 10)
    with pytest.raises(Rqb200Error):
        ops.SidItemTable(torch.from_numpy(ids), 16)
    with pytest.raises(Rqb200Error):
        ops.SidItemTable(dev(np.zeros((4, 9), dtype=np.int64)), 16)
    empty = table.retrieve(gen[:0], None, 10)
    assert [tuple(t.shape) for t in empty] == [(0, 10), (0, 10), (0,)]
    before = ops.LAUNCHES
    table.retrieve(gen, None, 10)
    table.lookup(gen[0])
    assert ops.LAUNCHES - before == 2


@pytest.mark.parametrize("item_mode", [False, True])
@pytest.mark.parametrize("B,k,D", [(1, 1, 1), (640, 10, 3), (333, 100, 1), (5000, 10, 8)])
def test_rank_hist_vs_oracle(B, k, D, item_mode):
    from rq_vae_recommender_b200 import ops
    rng = np.random.default_rng(B + k + D)
    actual = rng.integers(-1, 3, size=(B, D))
    cand = rng.integers(-1, 3, size=(B, k, D))
    hist = torch.full((k + 1,), 5, dtype=torch.int64, device="cuda")
    ops.sid_topk_rank_hist(dev(actual), dev(cand), hist, item_mode=item_mode)
    assert np.array_equal(hist.cpu().numpy(), I.rank_hist(actual, cand, item_mode) + 5)   # added to, never cleared
    wide = dev(np.concatenate([cand, cand], axis=2))[:, :, :D]                 # strided candidates are copied
    ops.sid_topk_rank_hist(dev(actual), wide, hist, item_mode=item_mode)
    assert np.array_equal(hist.cpu().numpy(), 2 * I.rank_hist(actual, cand, item_mode) + 5)


@pytest.mark.parametrize("case", ["tuples", "wide_ks", "items"])
def test_topk_accumulator_vs_reference(case):
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.evaluate.metrics import TopKAccumulator
    name, ks, batches, keys, values = next(c for c in golden_cases() if c[0] == case)
    acc = TopKAccumulator(ks=ks)
    assert acc.reduce() == {}
    for a, t in batches:
        a, t = dev(a), dev(t)
        before = ops.LAUNCHES
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            acc.accumulate(actual=a, top_k=t)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert ops.LAUNCHES - before == 1
    assert acc.total == sum(a.shape[0] for a, _ in batches)
    got = acc.reduce()
    assert list(got) == keys
    for key, v in zip(keys, values):
        if key == "ndcg":
            assert got[key] == pytest.approx(v, rel=1e-6)
        else:
            assert got[key] == v
    acc.reset()
    assert acc.reduce() == {} and acc.total == 0


def test_topk_accumulator_items_and_varying_candidates():
    from rq_vae_recommender_b200.evaluate.metrics import TopKAccumulator, metrics_from_hist
    rng = np.random.default_rng(8)
    acc = TopKAccumulator(ks=[1, 5, 10])
    tuples_hist, items_hist = np.zeros(11, dtype=np.int64), np.zeros(21, dtype=np.int64)
    for k in (10, 4):                                                          # batches with different candidate counts
        a, t = rng.integers(0, 3, size=(50, 3)), rng.integers(0, 3, size=(50, k, 3))
        acc.accumulate(dev(a), dev(t))
        h = I.rank_hist(a, t)
        tuples_hist[:k] += h[:k]
        tuples_hist[10] += h[k]
    for n in (20, 7):
        a, r = rng.integers(-1, 30, size=60), rng.integers(-1, 30, size=(60, n))
        da, dr = dev(a), dev(r)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            acc.accumulate_items(da, dr)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        h = I.rank_hist(a[:, None], r[:, :, None], item_mode=True)
        items_hist[:n] += h[:n]
        items_hist[20] += h[n]
    got = acc.reduce()
    want = metrics_from_hist(tuples_hist, 100, [1, 5, 10])
    want.update(metrics_from_hist(items_hist, 120, [1, 5, 10], "item_"))
    assert list(got) == list(want) and got == pytest.approx(want, rel=1e-12)
    assert list(got)[:4] == ["ndcg", "h@1", "h@5", "h@10"]


def collision_corpus(rs, N, H, K):
    """Corpus ids over few codes, so most tuples carry several items."""
    return rs.randint(0, 6, size=(N, H)).astype(np.int64) % K


def fut_batch(rs, corpus, B, items, H):
    """A TokenizedSeqBatch of B histories of corpus items (ids plus the dedup column) and their next items."""
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    o = I.build(corpus, 1 << 16)
    dedup = np.zeros(len(corpus), dtype=np.int64)
    for u in range(len(o["keys"])):
        rows = o["row"][o["start"][u]:o["start"][u + 1]]
        dedup[rows] = np.arange(len(rows))
    full = np.concatenate([corpus, dedup[:, None]], axis=1)
    hist = rs.randint(0, len(corpus), size=(B, items))
    nxt = rs.randint(0, len(corpus), size=B)
    sem_ids = full[hist].reshape(B, -1)
    mask = np.ones_like(sem_ids, dtype=bool)
    mask[: B // 2, : H + 1] = False
    return TokenizedSeqBatch(user_ids=dev(rs.randint(0, 100, size=(B, 1))), sem_ids=dev(sem_ids), sem_ids_fut=dev(full[nxt]),
                             seq_mask=dev(mask), token_type_ids=dev(np.tile(np.arange(H + 1), (B, items))),
                             token_type_ids_fut=dev(np.tile(np.arange(H + 1), (B, 1)))), nxt


@pytest.mark.parametrize("search", ["sample", "beam"])
def test_generate_items(search):
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, k = 256, 3, 64, 10
    rs = np.random.RandomState(31)
    cb = collision_corpus(rs, 3000, H, K)
    m = small_model(M, cb, K, H, k=k)
    batch, nxt = fut_batch(rs, cb, B, 12, H)
    o = I.build(cb, K)
    torch.manual_seed(4)
    before = ops.LAUNCHES
    out = m.generate_items(batch, n=4096, search=search)
    first = ops.LAUNCHES - before
    torch.manual_seed(4)
    ref = m.generate_next_sem_id(batch, search=search)
    assert torch.equal(out.sem_ids, ref.sem_ids) and torch.equal(out.log_probas, ref.log_probas)    # generate unchanged
    gen, lp = out.sem_ids.cpu().numpy(), out.log_probas.cpu().numpy()
    items, beam, count = I.retrieve(o, gen, lp, 4096)
    assert np.array_equal(out.item_ids.cpu().numpy(), items) and np.array_equal(out.beams.cpu().numpy(), beam)
    assert np.array_equal(out.count.cpu().numpy(), count)
    assert search == "sample" or int(count.min()) > 0                          # the sampled search can miss every code
    # item_of: the true next item, and it is among the items whenever its tuple is among the finite beams
    truth = m.item_of(batch.sem_ids_fut).cpu().numpy()
    assert np.array_equal(truth, nxt)
    for b in range(B):
        finite = {tuple(g) for g, p in zip(gen[b].tolist(), lp[b]) if p > -np.inf}
        assert (tuple(cb[nxt[b]].tolist()) in finite) == (nxt[b] in items[b].tolist())
    # n defaults to top_k_for_generation and truncates the same list; one extra launch per call after the first
    torch.manual_seed(4)
    before = ops.LAUNCHES
    short = m.generate_items(batch, search=search)
    again = ops.LAUNCHES - before
    assert np.array_equal(short.item_ids.cpu().numpy(), items[:, :k])
    before = ops.LAUNCHES
    m.generate_next_sem_id(batch, search=search)
    assert again == ops.LAUNCHES - before + 1
    assert first == again + 2                                                  # the prefix index and the item table builds
    # load_state_dict writes into the codebooks buffer: the table is rebuilt (item n becomes item N - 1 - n)
    sd = {name: v.clone() for name, v in m.state_dict().items()}
    sd["codebooks"] = sd["codebooks"].flip(0).contiguous()
    m.load_state_dict(sd)
    torch.manual_seed(4)
    before = ops.LAUNCHES
    flipped = m.generate_items(batch, n=4096, search=search)
    assert ops.LAUNCHES - before == first
    o2 = I.build(cb[::-1], K)
    want, _, _ = I.retrieve(o2, flipped.sem_ids.cpu().numpy(), flipped.log_probas.cpu().numpy(), 4096)
    assert np.array_equal(flipped.item_ids.cpu().numpy(), want)
    assert np.array_equal(m.item_of(batch.sem_ids_fut).cpu().numpy(), I.lookup(o2, batch.sem_ids_fut.cpu().numpy(), True))


@pytest.mark.parametrize("search", ["sample", "beam"])
def test_retrieve_on_search_outputs(search):
    """retrieve on both searches' real beams at B = 640, top-k 10 (fillers included where the corpus runs out)."""
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, k = 256, 3, 640, 10
    rs = np.random.RandomState(7)
    cb = np.concatenate([collision_corpus(rs, 2000, H, K), rs.randint(0, K, size=(40, H))])
    m = small_model(M, cb, K, H, k=k)
    mask, ids, users = history(rs, B, 10, H, K)
    torch.manual_seed(9)
    gen, lp = m.generate(mask, ids, users, search=search)
    table, o = ops.SidItemTable(dev(cb), K), I.build(cb, K)
    for n in (1, 10, 100, 4096):
        items, beam, count = table.retrieve(gen, lp, n)
        wi, wb, wc = I.retrieve(o, gen.cpu().numpy(), lp.cpu().numpy(), n)
        assert np.array_equal(items.cpu().numpy(), wi) and np.array_equal(beam.cpu().numpy(), wb)
        assert np.array_equal(count.cpu().numpy(), wc)
