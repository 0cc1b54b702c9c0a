"""GPU tests of the per-history exclusion sets (csrc/sid.cu rqb200_sid_exclusion_build and the exclusion input of
sid_trie_sample_select, sid_trie_beam_topk, sid_items_retrieve and t5rank_select; modules/model.py exclude_items /
exclude_history).  Empty sets change no bit; the searches with a history's set equal the same search on the corpus without that
history's excluded rows, bit for bit; the build, the retrieval and the selection equal tests/exclusion_oracle.py exactly;
rank_items equals the unexcluded ranking filtered; generate adds no host read.  `pytest -m gpu`."""
import warnings

import numpy as np
import pytest
import torch

import exclusion_oracle as X
import item_oracle as IO
from test_gpu_rank import model_for

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def corpus_with_subtrees(rs, N, H, K):
    """Random rows, with a few first codes shared by many rows (whole level-1 subtrees to exclude) and colliding tuples."""
    corpus = rs.randint(0, K, size=(N, H)).astype(np.int64)
    corpus[: N // 4, 0] = rs.randint(0, 3, size=N // 4)
    corpus[N // 4: N // 4 + 12] = corpus[N // 4]                       # one tuple with 13 items
    corpus[N // 2: N // 2 + 4, :H - 1] = corpus[N // 2, :H - 1]        # siblings under one (H - 1)-prefix
    return corpus


def exclusion_sets(rs, corpus, B, M):
    """[B, M] items, -1 padded: random rows, repeats, a whole level-1 subtree, a whole tuple, one history excluding everything
    when the corpus is small enough, one empty history."""
    N = len(corpus)
    items = np.full((B, M), -1, dtype=np.int64)
    for b in range(B - 1):
        pick = list(rs.randint(0, N, size=8)) + [int(rs.randint(0, N))] * 2
        if b % 3 == 0:
            pick += list(np.flatnonzero(corpus[:, 0] == corpus[b, 0]))   # the subtree of history b's first code
        if b % 3 == 1:
            pick += list(np.flatnonzero((corpus == corpus[N // 4]).all(1)))
        if b % 3 == 2:
            pick += list(np.flatnonzero((corpus[:, :-1] == corpus[N // 2, :-1]).all(1)))
        pick = pick[:M]
        items[b, :len(pick)] = pick
    if N <= M:
        items[0, :N] = rs.permutation(N)
    return items


def built(corpus, K, items):
    from rq_vae_recommender_b200 import ops
    table = ops.SidItemTable(dev(corpus), K)
    ref = IO.build(corpus, K)
    ex = ops.sid_exclusion_build(dev(items), table, dev(X.leaf_keys(ref)))
    return table, ref, ex


def test_build_matches_oracle():
    rs = np.random.RandomState(0)
    K, H = 256, 3
    corpus = corpus_with_subtrees(rs, 400, H, K)
    corpus[7, 1] = K                                                   # unretrievable rows
    corpus[9, 2] = -1
    items = exclusion_sets(rs, corpus, 7, 120)
    items[1, -3:] = [7, 9, 7]                                          # excluded rows that are not retrievable
    items[2, -2:] = [400, -5]                                          # ids outside [-1, N)
    _, ref, ex = built(corpus, K, items)
    want = X.build(ref, items)
    pos, blocked, count = ex.pos.cpu().numpy(), ex.blocked.cpu().numpy(), ex.count.cpu().numpy()
    for b, w in enumerate(want):
        assert count[b, 0] == len(w["pos"]) and pos[b, :count[b, 0]].tolist() == w["pos"]
        assert (pos[b, count[b, 0]:] == -1).all()
        for l in range(1, H + 1):
            assert blocked[b, l - 1, :count[b, l]].tolist() == w["blocked"][l], (b, l)
        assert count[b, H + 1] == w["bad"]
    assert count[2, H + 1] == 2 and count[:, 1].sum() > 0 and count[:, H].sum() > 0


def test_empty_sets_change_nothing():
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(1)
    K, H, B, k = 256, 3, 5, 16
    corpus = corpus_with_subtrees(rs, 3000, H, K)
    index = ops.SidPrefixIndex(dev(corpus), K)
    table, ref, _ = built(corpus, K, np.full((B, 1), -1))
    keys = dev(X.leaf_keys(ref))
    empties = [ops.sid_exclusion_build(torch.full((B, 6), -1, dtype=torch.int64, device="cuda"), table, keys),
               ops.sid_exclusion_build(torch.zeros((B, 0), dtype=torch.int64, device="cuda"), table, keys)]
    for beam in (True, False):
        gen, lp = None, None
        for h in range(H):
            rows = B if gen is None else B * k
            logits = torch.randn(rows, K, device="cuda") * 3
            if beam:
                base = index.beam_topk(logits, gen, lp, k)
                outs = [index.beam_topk(logits, gen, lp, k, exclude=e) for e in empties]
            else:
                probas = torch.softmax(logits, -1)
                noise = torch.empty_like(probas).exponential_(1)
                base = index.sample_select(probas, noise, gen, lp, k, 64, want_samples=True)
                outs = [index.sample_select(probas, noise, gen, lp, k, 64, want_samples=True, exclude=e) for e in empties]
            for out in outs:
                for a, c in zip(base, out):
                    assert torch.equal(a, c)
            gen, lp = base[0], base[1]
    base = table.retrieve(gen, lp, 40)
    for e in empties:
        for a, c in zip(base, table.retrieve(gen, lp, 40, exclude=e)):
            assert torch.equal(a, c)
    U = len(ref["keys"])
    scores = torch.randn(B, U, device="cuda").round(decimals=1)       # ties
    scores[0, :5] = float("nan")
    row, start = table.arrays()
    t_leaf = torch.randint(-1, U, (B,), device="cuda")
    t_dedup = torch.randint(0, 2, (B,), device="cuda")
    base = ops.t5rank_select(scores, row, start, t_leaf, t_dedup, 50)
    for e in empties:
        for a, c in zip(base, ops.t5rank_select(scores, row, start, t_leaf, t_dedup, 50, exclude=e)):
            assert torch.equal(a, c)


@pytest.mark.parametrize("K,H", [(256, 3), (2048, 3), (256, 5), (2048, 5)])
@pytest.mark.parametrize("search", ["beam", "sample"])
def test_search_equals_reduced_corpus(K, H, search):
    """Per history, the search with its exclusion set is the search on the corpus without its excluded rows, bit for bit."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K + H)
    B, k = 6, 32 if search == "beam" else 16
    corpus = corpus_with_subtrees(rs, 600, H, K)
    items = exclusion_sets(rs, corpus, B, 700)
    index = ops.SidPrefixIndex(dev(corpus), K)
    _, _, ex = built(corpus, K, items)
    reduced = []
    for b in range(B):
        keep = np.setdiff1d(np.arange(len(corpus)), items[b][items[b] >= 0])
        reduced.append(ops.SidPrefixIndex(dev(corpus[keep]), K))
    gen, lp = None, None
    for h in range(H):
        kp = 1 if gen is None else k
        logits = torch.randn(B * kp, K, device="cuda") * 3
        if h == 0:
            logits[torch.arange(B), dev(corpus[:B, 0])] += 8               # the excluded subtree would lead
        probas, noise = torch.softmax(logits, -1), None
        if search == "sample":
            noise = torch.empty_like(probas).exponential_(1)
            out = index.sample_select(probas, noise, gen, lp, k, 64, exclude=ex)
        else:
            out = index.beam_topk(logits, gen, lp, k, exclude=ex)
        for b in range(B):
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
        gen, lp = out[0], out[1]
    assert torch.isneginf(lp[0]).all()                                # history 0 excludes the whole corpus


def test_search_with_unretrievable_rows_matches_oracle():
    """Unretrievable rows keep their prefixes valid in the index but not under the blocking rule: the oracle states it."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(5)
    K, H, B, k = 256, 3, 4, 8
    corpus = corpus_with_subtrees(rs, 300, H, K)
    first = np.flatnonzero(corpus[:, 0] == corpus[0, 0])
    corpus[first[0], 2] = K                                           # an unretrievable row under the excluded subtree
    items = np.full((B, 80), -1, dtype=np.int64)
    items[0, :len(first)] = first
    items[1, :3] = [first[0], 5, 6]
    index = ops.SidPrefixIndex(dev(corpus), K)
    table, ref, ex = built(corpus, K, items)
    excls = X.build(ref, items)
    assert excls[0]["blocked"][1] == [int(corpus[0, 0])]
    logits = torch.randn(B, K, device="cuda")
    logits[:, int(corpus[0, 0])] += 20
    gen, lp, _ = index.beam_topk(logits, None, None, k, exclude=ex)
    scores = X.candidate_scores(corpus, K, excls, logits.cpu().numpy(), None, None)
    want = -np.sort(-scores, axis=1)[:, :k]
    np.testing.assert_allclose(lp.cpu().numpy(), want, rtol=0, atol=1e-5)
    for b in range(B):
        for j in range(k):
            if lp[b, j] > -np.inf:
                assert X.valid_prefix(corpus, K, excls[b], gen[b, j].tolist())


def test_retrieve_and_select_match_oracle():
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(2)
    K, H, B = 256, 3, 7
    corpus = corpus_with_subtrees(rs, 500, H, K)
    corpus[11, 0] = K                                                 # unretrievable rows
    items = exclusion_sets(rs, corpus, B, 200)
    items[2, -2:] = [11, 11]
    table, ref, ex = built(corpus, K, items)
    excls = X.build(ref, items)
    k = 40                                                           # beams: corpus tuples, some repeated, some not in it
    gen = corpus[rs.randint(0, len(corpus), size=(B, k))]
    gen[:, 1] = corpus[len(corpus) // 4]
    gen[:, 2] = gen[:, 0]
    gen[:, 3] = [K - 1, K - 1, K - 1]
    lp = -np.sort(rs.rand(B, k), axis=1).astype(np.float32)
    lp[:, -2:] = -np.inf
    for n in (5, 64, 600):
        got = table.retrieve(dev(gen), dev(lp), n, exclude=ex)
        want = X.retrieve(ref, excls, gen, lp, n)
        for a, w in zip(got, want):
            np.testing.assert_array_equal(a.cpu().numpy(), w)
    U = len(ref["keys"])
    row, start = table.arrays()
    for U_scores in ("smem", "global"):
        scores = rs.randn(B, U).round(1).astype(np.float32)
        scores[1, :30] = np.nan
        t_leaf = rs.randint(-1, U, size=B)
        t_dedup = rs.randint(0, 3, size=B)
        t_leaf[3] = np.searchsorted(X.leaf_keys(ref), X.tuple_key(corpus[len(corpus) // 4], K))
        t_dedup[3] = 2
        for n in (1, 20, 700):
            got = ops.t5rank_select(dev(scores), row, start, dev(t_leaf), dev(t_dedup), n, exclude=ex)
            want = X.rank_select(ref, excls, scores, t_leaf, t_dedup, n)
            for a, w in zip(got, want):
                np.testing.assert_array_equal(a.cpu().numpy(), w)
        if U_scores == "smem":                                        # the select's keys beyond shared memory: a larger corpus
            corpus = corpus_with_subtrees(rs, 40000, H, K)
            items = exclusion_sets(rs, corpus, B, 300)
            table, ref, ex = built(corpus, K, items)
            excls = X.build(ref, items)
            U = len(ref["keys"])
            assert U > 24 * 1024
            row, start = table.arrays()


def dedup_ranks(corpus):
    seen, out = {}, np.zeros(len(corpus), dtype=np.int64)
    for i, t in enumerate(map(tuple, corpus)):
        out[i] = seen.get(t, 0)
        seen[t] = out[i] + 1
    return out


def item_batch(rs, corpus, B, S, H):
    """A batch whose histories are corpus items (H ids + dedup rank per item), some padded, with corpus items as targets.
    Returns the batch, its items [B, S] (-1 where padded) and the targets [B]."""
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    full = np.concatenate([corpus, dedup_ranks(corpus)[:, None]], axis=1)
    hist = rs.randint(0, len(corpus), size=(B, S))
    mask = np.ones((B, S), dtype=bool)
    mask[0, :3] = False
    fut = rs.randint(0, len(corpus), size=B)
    fut[1] = hist[1, -1]                                              # a target among its history's items
    w = H + 1
    sem = full[hist].reshape(B, S * w)
    seq = np.repeat(mask, w, axis=1)
    tt = np.tile(np.arange(w), (B, S))
    batch = TokenizedSeqBatch(user_ids=dev(rs.randint(0, 100, size=(B, 1))), sem_ids=dev(sem), sem_ids_fut=dev(full[fut]),
                              seq_mask=dev(seq), token_type_ids=dev(tt), token_type_ids_fut=dev(np.tile(np.arange(w), (B, 1))))
    return batch, np.where(mask, hist, -1), fut


def test_rank_items_equals_filtered_ranking():
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(3)
    K, H, B = 256, 3, 5
    corpus = corpus_with_subtrees(rs, 300, H, K)
    m = model_for(M, corpus, K, H)
    batch, hist, fut = item_batch(rs, corpus, B, 12, H)
    np.testing.assert_array_equal(m.history_items(batch).cpu().numpy(), hist)
    seen = [set(h[h >= 0].tolist()) for h in hist]
    full = m.rank_items(batch, n=300)
    got = m.rank_items(batch, n=300, exclude_history=True)
    assert full.num_items == got.num_items == 300
    for b in range(B):
        items, scores = full.item_ids[b].cpu().numpy(), full.scores[b].cpu().numpy()
        keep = np.array([it not in seen[b] for it in items])
        n_kept = int(keep.sum())
        assert got.item_ids[b, :n_kept].cpu().numpy().tolist() == items[keep].tolist()
        assert (got.item_ids[b, n_kept:] == -1).all()
        np.testing.assert_array_equal(got.scores[b, :n_kept].cpu().numpy().view(np.int32), scores[keep].view(np.int32))
        filtered = items[keep].tolist()
        want = filtered.index(fut[b]) if fut[b] in filtered else -1
        assert got.target_rank[b].item() == want, b
    assert got.target_rank[1].item() == -1
    M.DEFAULT_EXCLUDE_HISTORY = True
    try:
        again = m.rank_items(batch, n=300)
    finally:
        M.DEFAULT_EXCLUDE_HISTORY = False
    assert torch.equal(again.item_ids, got.item_ids) and torch.equal(again.target_rank, got.target_rank)


@pytest.mark.parametrize("search", ["beam", "sample"])
def test_generate_items_excluding_history(search):
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(4)
    K, H, B = 256, 3, 4
    corpus = corpus_with_subtrees(rs, 400, H, K)
    m = model_for(M, corpus, K, H, k=10)
    batch, hist, _ = item_batch(rs, corpus, B, 20, H)
    seen = [set(h[h >= 0].tolist()) for h in hist]
    kw = dict(search=search, decoder="fused", encoder="fused")
    torch.manual_seed(11)
    got = m.generate_items(batch, n=40, exclude_history=True, **kw)
    for b in range(B):
        items = got.item_ids[b, :got.count[b]].cpu().numpy().tolist()
        assert not set(items) & seen[b] and -1 not in items
    for b in range(B):                                                # the same search on the corpus without history b's items
        keep = np.setdiff1d(np.arange(len(corpus)), sorted(seen[b]))
        r = model_for(M, corpus[keep], K, H, k=10)
        r.load_state_dict({n: v for n, v in m.state_dict().items() if n != "codebooks"}, strict=False)
        torch.manual_seed(11)
        want = r.generate_next_sem_id(batch, **kw)
        assert torch.equal(got.sem_ids[b], want.sem_ids[b]), b
        assert torch.equal(got.log_probas[b], want.log_probas[b]), b


def test_generate_exclusion_adds_no_host_sync():
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(6)
    K, H, B = 256, 3, 8
    corpus = corpus_with_subtrees(rs, 500, H, K)
    m = model_for(M, corpus, K, H)
    batch, _, _ = item_batch(rs, corpus, B, 10, H)
    mask = M._strip_dedup_col(batch.seq_mask.long(), H + 1, H)
    ids = M._strip_dedup_col(batch.sem_ids, H + 1, H)
    exclude = m.history_items(batch)

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

    m.generate(mask, ids, batch.user_ids, exclude_items=exclude)     # warm: _rank_levels' one read, the item table
    assert syncs(exclude_items=exclude) == syncs()


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
    bad[1, 2] = 200
    with pytest.raises(ValueError, match="outside"):
        m.generate(mask, ids, batch.user_ids, exclude_items=bad)
    with pytest.raises(ValueError, match="outside"):
        m.rank_items(batch, exclude_items=bad)
    table = m._item_table(torch.device("cuda"))
    leaf_key = m._rank_levels(torch.device("cuda"))[1]
    launches = ops.LAUNCHES
    with pytest.raises(ValueError, match="4096"):
        ops.sid_exclusion_build(torch.zeros((B, 4097), dtype=torch.int64, device="cuda"), table, leaf_key)
    assert ops.LAUNCHES == launches                                   # raised before any launch
    with pytest.raises(ValueError, match="4096"):
        m.generate_items(batch, exclude_items=torch.zeros((B, 4097), dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError, match="exclude_items"):
        m.generate(mask, ids, batch.user_ids, exclude_items=torch.zeros((B + 1, 2), dtype=torch.int64, device="cuda"))
