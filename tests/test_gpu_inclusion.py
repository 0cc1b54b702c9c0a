"""GPU tests of the per-history allow-lists (csrc/sid.cu rqb200_sid_inclusion_build and the inclusion input of
sid_trie_sample_select, sid_trie_beam_topk and sid_items_retrieve; modules/model.py include_items).  The build and each consumer
equal tests/inclusion_oracle.py; a history's search equals, bit for bit, the same search on the corpus of its eligible rows; an
allow-list of every item changes no bit; generate_items returns eligible items only; no host read is added.  `pytest -m gpu`."""
import warnings

import numpy as np
import pytest
import torch

import exclusion_oracle as X
import inclusion_oracle as I
import item_oracle as IO
from test_gpu_exclusion import corpus_with_subtrees, item_batch
from test_gpu_rank import model_for

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def allow_lists(rs, corpus, B, M):
    """[B, M] items, -1 padded: random rows with repeats, a whole level-1 subtree, a whole tuple of colliding rows, one history
    with a single item and one with none."""
    N = len(corpus)
    items = np.full((B, M), -1, dtype=np.int64)
    for b in range(B):
        pick = list(rs.randint(0, N, size=max(M // 2, 1))) + [int(rs.randint(0, N))] * 2
        if b % 3 == 0:
            pick += list(np.flatnonzero(corpus[:, 0] == corpus[b, 0]))
        if b % 3 == 1:
            pick += list(np.flatnonzero((corpus == corpus[N // 4]).all(1)))
        pick = pick[:M]
        items[b, :len(pick)] = pick
    items[1] = -1
    items[1, 0] = rs.randint(0, N)
    items[B - 1] = -1
    return items


def built(corpus, K, items, ex_items=None):
    from rq_vae_recommender_b200 import ops
    table = ops.SidItemTable(dev(corpus), K)
    ref = IO.build(corpus, K)
    keys = dev(X.leaf_keys(ref))
    ex = None if ex_items is None else ops.sid_exclusion_build(dev(ex_items), table, keys)
    inc = ops.sid_inclusion_build(dev(items), table, keys, exclude=ex)
    incls = I.build(ref, items, None if ex_items is None else X.build(ref, ex_items))
    return table, ref, inc, incls


@pytest.mark.parametrize("excluding", [False, True])
@pytest.mark.parametrize("K,H", [(256, 3), (2048, 3), (256, 5), (2048, 5)])
@pytest.mark.parametrize("M", [1, 511, 512, 513, 1024, 1025, 2048, 2049, 4096])
def test_build_matches_oracle(M, K, H, excluding):
    rs = np.random.RandomState(M + K + H)
    B, N = 5, 3000
    corpus = corpus_with_subtrees(rs, N, H, K)
    corpus[7, 1] = K                                                   # unretrievable rows
    corpus[9, H - 1] = -1
    items = allow_lists(rs, corpus, B, M)
    items[0, :min(M, 3)] = [7, 9, 7][:min(M, 3)]                      # allowed rows that are not retrievable
    if M > 4:
        items[2, -2:] = [N, -5]                                       # ids outside [-1, N)
    ex_items = None
    if excluding:
        ex_items = np.where(rs.rand(B, M) < 0.3, items, -1)            # part of each allow-list excluded
        ex_items[3] = items[3]                                        # all of one
    _, _, inc, incls = built(corpus, K, items, ex_items)
    pos, keys, count = inc.pos.cpu().numpy(), inc.keys.cpu().numpy(), inc.count.cpu().numpy()
    for b, w in enumerate(incls):
        assert count[b, 0] == len(w["pos"]) and pos[b, :count[b, 0]].tolist() == w["pos"], b
        assert (pos[b, count[b, 0]:] == -1).all()
        for l in range(1, H + 1):
            assert count[b, l] == len(w["keys"][l]) and keys[b, l - 1, :count[b, l]].tolist() == w["keys"][l], (b, l)
            assert (keys[b, l - 1, count[b, l]:] == -1).all()
        assert count[b, H + 1] == w["bad"]
    assert count[B - 1, 0] == 0
    if excluding:
        assert count[3, 0] == 0


def _reduced_index(corpus, K, incl):
    from rq_vae_recommender_b200 import ops
    rows = sorted(incl["eligible"])
    return ops.SidPrefixIndex(dev(corpus[rows]), K) if rows else None


@pytest.mark.parametrize("K,H", [(256, 3), (2048, 3), (256, 5), (2048, 5)])
@pytest.mark.parametrize("search", ["beam", "sample"])
def test_search_matches_eligible_corpus_and_oracle(K, H, search):
    """Per history, each level with its allow-list is the same level on the corpus of its eligible rows, bit for bit, and the
    oracle's: beams and fillers for the beam search, the valid sampled candidates for the sampled search."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K * H)
    B, k = 6, 32 if search == "beam" else 16
    corpus = corpus_with_subtrees(rs, 800, H, K)
    items = allow_lists(rs, corpus, B, 300)
    ex_items = np.full((B, 4), -1, dtype=np.int64)
    ex_items[2, :2] = items[2, :2]
    index = ops.SidPrefixIndex(dev(corpus), K)
    _, ref, inc, incls = built(corpus, K, items, ex_items)
    reduced = [_reduced_index(corpus, K, w) for w in incls]
    assert reduced[B - 1] is None
    gen, lp = None, None
    for h in range(H):
        kp = 1 if gen is None else k
        logits = torch.randn(B * kp, K, device="cuda") * 3
        probas = torch.softmax(logits, -1)
        noise = torch.empty_like(probas).exponential_(1)
        if search == "sample":
            out = index.sample_select(probas, noise, gen, lp, k, 64, want_samples=True, include=inc)
            base = index.sample_select(probas, noise, gen, lp, k, 64, want_samples=True)
            assert torch.equal(out[3], base[3]) and torch.equal(out[4], base[4])   # the same noise draws the same samples
            scores = I.sample_scores(incls, K, out[3].cpu().numpy(), out[4].cpu().numpy(),
                                     None if gen is None else gen.cpu().numpy(), None if lp is None else lp.cpu().numpy())
            want = -np.sort(-scores, axis=1)[:, :k]
            np.testing.assert_allclose(out[1].cpu().numpy(), want, rtol=0, atol=1e-4)
        else:
            out = index.beam_topk(logits, gen, lp, k, include=inc)
            w_gen, w_lp, w_parent = I.beam_topk(corpus, K, incls, logits.cpu().numpy(), None if gen is None else gen.cpu().numpy(),
                                                None if lp is None else lp.cpu().numpy(), k)
            np.testing.assert_array_equal(out[0].cpu().numpy(), w_gen)
            np.testing.assert_array_equal(out[2].view(B, k).cpu().numpy() - np.arange(B)[:, None] * kp, w_parent)
            np.testing.assert_allclose(out[1].cpu().numpy(), w_lp, rtol=0, atol=1e-4)
        for b in range(B):
            if reduced[b] is None:
                assert torch.isneginf(out[1][b]).all()
                continue
            rows = slice(b * kp, (b + 1) * kp)
            g = None if gen is None else gen[b:b + 1]
            p = None if lp is None else lp[b:b + 1]
            if search == "sample":
                want = reduced[b].sample_select(probas[rows], noise[rows], g, p, k, 64)
            else:
                want = reduced[b].beam_topk(logits[rows], g, p, k)
            assert torch.equal(out[0][b], want[0][0]), (h, b)
            assert torch.equal(out[1][b], want[1][0]), (h, b)
            assert torch.equal(out[2].view(B, k)[b] - b * kp, want[2]), (h, b)
        for b in range(B):
            for j in range(k):
                if out[1][b, j] > -np.inf:
                    assert I.valid_prefix(incls[b], out[0][b, j].tolist(), K)
        gen, lp = out[0], out[1]
    if search == "beam":
        assert (lp[1] > -np.inf).sum() == 1                           # one allowed item: one finite beam


def test_retrieve_matches_oracle():
    rs = np.random.RandomState(2)
    K, H, B = 256, 3, 7
    corpus = corpus_with_subtrees(rs, 500, H, K)
    corpus[11, 0] = K                                                 # an unretrievable row
    items = allow_lists(rs, corpus, B, 200)
    items[2, -2:] = [11, 11]
    ex_items = np.full((B, 8), -1, dtype=np.int64)
    ex_items[0, :5] = items[0, :5]
    table, ref, inc, incls = built(corpus, K, items, ex_items)
    k = 40                                                           # beams: corpus tuples, some repeated, some not in it
    gen = corpus[rs.randint(0, len(corpus), size=(B, k))]
    gen[:, 1] = corpus[len(corpus) // 4]
    gen[:, 2] = gen[:, 0]
    gen[:, 3] = [K - 1, K - 1, K - 1]
    gen[0, 5:15] = corpus[items[0, 5:15]]                             # beams holding allowed items
    lp = -np.sort(rs.rand(B, k), axis=1).astype(np.float32)
    lp[:, -2:] = -np.inf
    for n in (1, 5, 64, 600):
        got = table.retrieve(dev(gen), dev(lp), n, include=inc)
        want = I.retrieve(ref, incls, gen, lp, n)
        for a, w in zip(got, want):
            np.testing.assert_array_equal(a.cpu().numpy(), w)
    assert got[2][0] > 0 and got[2][B - 1] == 0


def test_every_item_allowed_changes_nothing():
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(1)
    K, H, B, k = 256, 3, 5, 16
    corpus = corpus_with_subtrees(rs, 3000, H, K)
    corpus[5, 2] = K                                                  # allowed but not retrievable: ignored
    index = ops.SidPrefixIndex(dev(corpus), K)
    items = np.tile(np.arange(len(corpus)), (B, 1))
    for b in range(B):
        items[b] = rs.permutation(items[b])
    table, _, inc, _ = built(corpus, K, items)
    for beam in (True, False):
        gen, lp = None, None
        for h in range(H):
            rows = B if gen is None else B * k
            logits = torch.randn(rows, K, device="cuda") * 3
            if beam:
                base = index.beam_topk(logits, gen, lp, k)
                out = index.beam_topk(logits, gen, lp, k, include=inc)
            else:
                probas = torch.softmax(logits, -1)
                noise = torch.empty_like(probas).exponential_(1)
                base = index.sample_select(probas, noise, gen, lp, k, 64, want_samples=True)
                out = index.sample_select(probas, noise, gen, lp, k, 64, want_samples=True, include=inc)
            for a, c in zip(base, out):
                assert torch.equal(a, c)
            gen, lp = base[0], base[1]
        for a, c in zip(table.retrieve(gen, lp, 40), table.retrieve(gen, lp, 40, include=inc)):
            assert torch.equal(a, c)


@pytest.mark.parametrize("decoder", ["hf", "fused"])
@pytest.mark.parametrize("search", ["beam", "sample"])
def test_generate_items_returns_eligible_items(search, decoder):
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(4)
    K, H, B = 256, 3, 5
    corpus = corpus_with_subtrees(rs, 400, H, K)
    m = model_for(M, corpus, K, H, k=10)
    batch, hist, _ = item_batch(rs, corpus, B, 20, H)
    items = allow_lists(rs, corpus, B, 30)
    items[0, :3] = hist[0, -3:]                                       # allowed items the history holds: excluded below
    ref = IO.build(corpus, K)
    incls = I.build(ref, items, X.build(ref, hist))
    kw = dict(search=search, decoder=decoder, encoder="fused")
    got = m.generate_items(batch, n=40, include_items=dev(items), exclude_history=True, **kw)
    for b in range(B):
        returned = got.item_ids[b, :got.count[b]].cpu().numpy().tolist()
        assert set(returned) <= incls[b]["eligible"] and len(set(returned)) == len(returned)
        assert (got.item_ids[b, got.count[b]:] == -1).all()
        for j in range(got.sem_ids.shape[1]):
            if got.log_probas[b, j] > -np.inf:
                assert set(IO.items_of(ref, got.sem_ids[b, j].tolist())) & incls[b]["eligible"], (b, j)
    assert got.count[B - 1] == 0 and torch.isneginf(got.log_probas[B - 1]).all()
    if search == "beam":
        assert got.count[0] > 0
    torch.manual_seed(3)
    sem = m.generate_next_sem_id(batch, include_items=dev(items), exclude_history=True, **kw)
    torch.manual_seed(3)
    again = m.generate_next_sem_id(batch, include_items=dev(items), exclude_history=True, **kw)
    assert torch.equal(sem.sem_ids, again.sem_ids) and torch.equal(sem.log_probas, again.log_probas)


@pytest.mark.parametrize("search", ["beam", "sample"])
def test_generate_with_every_item_allowed_is_unfiltered(search):
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(8)
    K, H, B = 256, 3, 4
    corpus = corpus_with_subtrees(rs, 300, H, K)
    m = model_for(M, corpus, K, H, k=10)
    batch, _, _ = item_batch(rs, corpus, B, 8, H)
    everything = dev(np.tile(np.arange(len(corpus)), (B, 1)))
    kw = dict(search=search, decoder="fused", encoder="fused")
    torch.manual_seed(5)
    base = m.generate_items(batch, n=30, **kw)
    torch.manual_seed(5)
    got = m.generate_items(batch, n=30, include_items=everything, **kw)
    for f in ("item_ids", "beams", "count", "sem_ids", "log_probas"):
        assert torch.equal(getattr(base, f), getattr(got, f)), f
    empty = m.generate_items(batch, n=30, include_items=torch.full((B, 3), -1, dtype=torch.int64, device="cuda"), **kw)
    assert (empty.count == 0).all() and torch.isneginf(empty.log_probas).all() and (empty.item_ids == -1).all()


def test_inclusion_adds_no_host_sync():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(6)
    K, H, B, k = 256, 3, 8, 10
    corpus = corpus_with_subtrees(rs, 500, H, K)
    items = dev(allow_lists(rs, corpus, B, 50))
    table = ops.SidItemTable(dev(corpus), K)
    index = ops.SidPrefixIndex(dev(corpus), K)
    keys = dev(X.leaf_keys(IO.build(corpus, K)))
    ex = ops.sid_exclusion_build(items[:, :5].contiguous(), table, keys)
    table.positions()
    logits = torch.randn(B, K, device="cuda")
    probas = torch.softmax(logits, -1)
    noise = torch.empty_like(probas).exponential_(1)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")                           # the build and every consumer, no host read
    try:
        inc = ops.sid_inclusion_build(items, table, keys, exclude=ex)
        gen, lp, _ = index.beam_topk(logits, None, None, k, include=inc)
        index.sample_select(probas, noise, None, None, k, 64, include=inc)
        table.retrieve(gen.repeat(1, 1, H), lp, 20, include=inc)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    m = model_for(M, corpus, K, H)
    batch, _, _ = item_batch(rs, corpus, B, 10, H)
    mask = M._strip_dedup_col(batch.seq_mask.long(), H + 1, H)
    ids = M._strip_dedup_col(batch.sem_ids, H + 1, H)

    def syncs(**kw):
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                for search in ("beam", "sample"):
                    m.generate(mask, ids, batch.user_ids, search=search, decoder="fused", **kw)
            finally:
                torch.cuda.set_sync_debug_mode(0)
        return sum("called a synchronizing CUDA operation" in str(x.message) for x in w)

    m.generate(mask, ids, batch.user_ids, include_items=items)       # warm: _rank_levels' one read, the item table
    assert syncs(include_items=items) == syncs()
    assert syncs(include_items=items, exclude_items=items[:, :5]) == syncs()


def test_argument_errors():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(7)
    K, H, B = 256, 3, 3
    corpus = corpus_with_subtrees(rs, 200, H, K)
    m = model_for(M, corpus, K, H)
    batch, _, _ = item_batch(rs, corpus, B, 6, H)
    mask = M._strip_dedup_col(batch.seq_mask.long(), H + 1, H)
    ids = M._strip_dedup_col(batch.sem_ids, H + 1, H)
    bad = torch.full((B, 4), -1, dtype=torch.int64, device="cuda")
    bad[1, 2] = 200                                                   # = N
    with pytest.raises(ValueError, match="allowed item id.*outside"):
        m.generate(mask, ids, batch.user_ids, include_items=bad)
    with pytest.raises(ValueError, match="outside"):
        m.generate_items(batch, include_items=bad, search="sample")
    table = m._item_table(torch.device("cuda"))
    leaf_key = m._rank_levels(torch.device("cuda"))[1]
    launches = ops.LAUNCHES
    with pytest.raises(ValueError, match="4096"):
        ops.sid_inclusion_build(torch.zeros((B, 4097), dtype=torch.int64, device="cuda"), table, leaf_key)
    assert ops.LAUNCHES == launches                                   # raised before any launch
    with pytest.raises(ValueError, match="4096"):
        m.generate_items(batch, include_items=torch.zeros((B, 4097), dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError, match="include_items"):
        m.generate(mask, ids, batch.user_ids, include_items=torch.zeros((B + 1, 2), dtype=torch.int64, device="cuda"))
    inc = ops.sid_inclusion_build(torch.zeros((B, 2), dtype=torch.int64, device="cuda"), table, leaf_key)
    ex = ops.sid_exclusion_build(torch.zeros((B, 2), dtype=torch.int64, device="cuda"), table, leaf_key)
    index = m._prefix_index(torch.device("cuda"))
    with pytest.raises(ValueError, match="not both"):
        index.beam_topk(torch.zeros(B, K, device="cuda"), None, None, 4, exclude=ex, include=inc)
    with pytest.raises(ValueError, match="histories"):
        table.retrieve(torch.zeros((B + 1, 2, H), dtype=torch.int64, device="cuda"), None, 4, include=inc)
