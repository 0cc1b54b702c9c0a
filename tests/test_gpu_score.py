"""GPU tests of the exact scoring of given tuples (csrc/t5rank.cu t5score_trie_build, modules/model.py FusedT5Rank.run_candidates,
score_sem_ids / score_items): the trie build against the host statement of tests/test_score_ref.py, scores bit-identical to
rank_sem_ids on corpus tuples and near the float64 statement elsewhere, chunking, the target's rank against a torch sort, the
per-row cross-entropy of forward, host reads and modes.  `pytest -m gpu`."""
import numpy as np
import pytest
import torch

from test_gpu_decode import highest
from test_gpu_generate import history, realistic_corpus
from test_gpu_rank import batch_for, model_for
from test_score_ref import candidate_trie, candidates_with_edges, score_decompose

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("C", [1, 7, 101, 512, 513, 1024, 1025, 2048, 2049, 4096])
@pytest.mark.parametrize("K", [256, 300, 2048])
@pytest.mark.parametrize("H", [3, 5])
def test_trie_build_matches_host_statement(C, K, H):
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(C + K + H)
    ids = rs.randint(0, K, size=(4, C, H)).astype(np.int64)
    ids[0, :, 0] = rs.randint(0, 3, size=C)                                  # shared prefixes
    ids[0, rs.rand(C) < 0.1, H - 1] = K                                      # invalid ids
    ids[0, rs.rand(C) < 0.1] = -1                                            # padding
    ids[1] = ids[1, 0]                                                       # every tuple the same
    ids[2] = -1                                                              # every tuple padding
    ids[3, ::2] = ids[3, 0]                                                  # duplicates among distinct tuples
    trie = ops.t5score_trie_build(torch.from_numpy(ids).cuda(), K)
    got = [t.cpu().numpy() for t in trie]
    for b in range(ids.shape[0]):
        want = candidate_trie(ids[b], K)
        for name, g, w in zip(("counts", "code", "parent", "child", "leaf"), got, want):
            assert np.array_equal(g[b], w), (b, name)
    again = ops.t5score_trie_build(torch.from_numpy(ids).cuda(), K)
    assert all(torch.equal(a, b) for a, b in zip(trie, again))


def candidates(rs, corpus, B, C, H, K):
    """Corpus tuples in every slot but the edge slots of candidates_with_edges (out of corpus, duplicate, invalid, padding)."""
    cand = candidates_with_edges(rs, corpus, B, C, H, K)
    cand[:, 1, 0] = K - 1                                                    # surely not a corpus tuple's id pattern alone
    return torch.from_numpy(cand).cuda()


@pytest.mark.parametrize("encoder", ["hf", "fused"])
@pytest.mark.parametrize("attention", ["fp32", "tf32"])
def test_corpus_tuples_bit_identical_to_rank_sem_ids(encoder, attention):
    """Each kernel computes a row from that row's inputs alone, so a corpus tuple's score does not depend on which trie it sits in."""
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, C = 256, 3, 7, 101
    rs = np.random.RandomState(11)
    corpus = realistic_corpus(rs, 1500, H, K)
    corpus[:40, :2] = corpus[40, :2]                                         # shared prefixes
    m = model_for(M, corpus, K, H)
    mask, ids, users = history(rs, B, 20, H, K)
    mask[-1] = 0
    cand = candidates(rs, corpus, B, C, H, K)
    kw = dict(encoder=encoder, attention=attention)
    got = m.score_sem_ids(mask, ids, users, sem_ids=cand, **kw)
    dense = m.rank_sem_ids(mask, ids, users, **kw)
    _, leaf_key, _ = m._rank_levels(dense.device)
    leaf = m._leaf_of(cand.reshape(-1, H), leaf_key).reshape(B, C)
    inside = leaf >= 0
    assert inside.float().mean() > 0.9
    assert torch.equal(got[inside], dense.gather(1, leaf.clamp(min=0))[inside])
    valid = ((cand >= 0) & (cand < K)).all(2)
    assert torch.isfinite(got[valid]).all() and (got[~valid] == float("-inf")).all()
    assert torch.equal(got[:, 0], got[:, 2])
    own = max(1 + (H - 1) * C, 1)
    chunked = m.score_sem_ids(mask, ids, users, sem_ids=cand, max_rows=own, **kw)
    assert torch.equal(chunked, got)
    with pytest.raises(ValueError, match="max_rows = 2 is below"):
        m.score_sem_ids(mask, ids, users, sem_ids=cand, max_rows=2, **kw)


@pytest.mark.parametrize("K,H", [(256, 3), (2048, 5)])
def test_scores_match_float64(K, H):
    from rq_vae_recommender_b200.modules import model as M
    B, C = 5, 12
    rs = np.random.RandomState(K + H)
    corpus = realistic_corpus(rs, 300, H, K)
    m = model_for(M, corpus, K, H)
    mask, ids, users = history(rs, B, 10, H, K)
    cand = candidates(rs, corpus, B, C, H, K)
    with highest():
        got = m.score_sem_ids(mask, ids, users, sem_ids=cand)
        enc_out, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
    ref = M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), num_hierarchies=H, num_embeddings_per_hierarchy=K,
                                         t5_d_model=64, t5_num_heads=2, t5_d_ff=128, t5_num_layers=2, top_k_for_generation=10,
                                         should_add_sep_token=True, num_user_bins=11)
    ref.load_state_dict(m.state_dict())
    ref = ref.double().eval()
    with torch.no_grad():
        want = score_decompose(ref, enc_out.double().cpu(), enc_mask.cpu(), cand.cpu().numpy())
    fin = torch.isfinite(want)
    assert torch.equal(fin, torch.isfinite(got.cpu()))
    assert (got.double().cpu()[fin] - want[fin]).abs().max().item() <= 1e-5


def sorted_rank(scores, tuples, items, target, K):
    """The target's position among the row's valid items by a torch sort: NaN last, score descending, tuple, item id."""
    ok = items >= 0
    s, t, it = scores[ok], tuples[ok], items[ok]
    key = torch.zeros_like(it)
    for h in range(t.shape[1]):
        key = key * K + t[:, h]
    nan = s.isnan()
    order = sorted(range(len(s)), key=lambda i: (bool(nan[i]), 0.0 if nan[i] else -float(s[i]), int(key[i]), int(it[i])))
    ranked = [int(it[i]) for i in order]
    return ranked.index(int(target)) if int(target) in ranked else -1


def test_score_items_target_rank_and_metrics():
    from rq_vae_recommender_b200.evaluate.metrics import TopKAccumulator
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, C = 256, 3, 9, 101
    rs = np.random.RandomState(13)
    corpus = realistic_corpus(rs, 2000, H, K)
    corpus[100:104] = corpus[105]                                            # one tuple, several items
    m = model_for(M, corpus, K, H)
    batch = batch_for(rs, corpus, B, 6, H, K)
    batch.sem_ids_fut[1:, H] = 0                                              # dedup rank 0: every target but row 0's exists
    target = m.item_of(batch.sem_ids_fut)
    items = torch.from_numpy(rs.randint(0, len(corpus), size=(B, C))).cuda()
    items[:, 0] = target
    items[1, :5] = torch.tensor([100, 101, 102, 103, 105])                   # items sharing a tuple: ordered by item id
    items[1, 5] = target[1]
    items[2, 1:3] = items[2, 0]                                              # the target three times
    items[3, -10:] = -1                                                      # padding
    items[4] = torch.where(items[4] == target[4], (target[4] + 1) % len(corpus), items[4])   # the target is not a candidate
    out = m.score_items(batch, items)
    tuples = torch.from_numpy(corpus).cuda()[items.clamp(min=0)]
    want = m.score_sem_ids(M._strip_dedup_col(batch.seq_mask.long(), H + 1, H), M._strip_dedup_col(batch.sem_ids, H + 1, H),
                           batch.user_ids, sem_ids=torch.where(items[..., None] >= 0, tuples, -1))
    assert torch.equal(out.scores, want)
    assert (out.scores[3, -10:] == float("-inf")).all()
    ranks = [sorted_rank(out.scores[b].cpu(), tuples[b].cpu(), items[b].cpu(), target[b].cpu(), K) for b in range(B)]
    assert out.target_rank.tolist() == ranks
    assert out.target_rank[0] == -1 and out.target_rank[4] == -1           # not retrievable; not a candidate
    acc = TopKAccumulator([1, 5, 10, 50])
    acc.accumulate_ranks(out.target_rank, C)
    r = np.array(ranks)
    res = acc.reduce()
    for k in (1, 5, 10, 50):
        assert res[f"exact_h@{k}"] == pytest.approx(float(((r >= 0) & (r < k)).sum()) / B, abs=1e-15)
    hand = TopKAccumulator([1, 2])
    hand.accumulate_ranks(torch.tensor([0, 1, 2, -1], device="cuda"), 3)
    assert hand.reduce()["exact_h@1"] == 0.25 and hand.reduce()["exact_h@2"] == 0.5


def test_single_target_is_forward_cross_entropy():
    """With C = 1 and the target item, -score is the sum over levels of forward's per-row cross-entropy."""
    import torch.nn.functional as F
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 8
    rs = np.random.RandomState(14)
    corpus = realistic_corpus(rs, 500, H, K)
    m = model_for(M, corpus, K, H)
    batch = batch_for(rs, corpus, B, 6, H, K)
    fut = batch.sem_ids_fut[1:].clone()                                      # row 0's target is not retrievable
    fut[:, H] = 0
    batch = batch._replace(sem_ids_fut=fut, sem_ids=batch.sem_ids[1:], seq_mask=batch.seq_mask[1:],
                           user_ids=batch.user_ids[1:], token_type_ids=batch.token_type_ids[1:],
                           token_type_ids_fut=batch.token_type_ids_fut[1:])
    target = m.item_of(batch.sem_ids_fut)
    assert (target >= 0).all()
    with highest(), torch.no_grad():
        out = m.score_items(batch, target[:, None])
        fwd = m(batch)
        mask = M._strip_dedup_col(batch.seq_mask.long(), H + 1, H)
        enc, enc_mask = m.encoder_forward_pass(mask, M._strip_dedup_col(batch.sem_ids, H + 1, H), batch.user_ids)
        fut = batch.sem_ids_fut[:, :H]
        dec = m.decoder_forward_pass(future_ids=fut, encoder_output=enc, attention_mask_for_encoder=enc_mask)[:, :-1]
        ce = torch.stack([F.cross_entropy(m.decoder_mlp[h](dec[:, h]), fut[:, h].long(), reduction="none") for h in range(H)], 1)
    assert (ce.mean(0) - fwd.loss_d).abs().max().item() < 1e-6
    assert (-out.scores[:, 0] - ce.sum(1)).abs().max().item() < 1e-5
    assert (out.target_rank == 0).all()


def test_host_reads_modes_and_errors():
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, C = 256, 3, 5, 30
    rs = np.random.RandomState(15)
    corpus = realistic_corpus(rs, 800, H, K)
    m = model_for(M, corpus, K, H)
    batch = batch_for(rs, corpus, B, 5, H, K)
    items = torch.from_numpy(rs.randint(0, len(corpus), size=(B, C))).cuda()
    first = m.score_items(batch, items, encoder="fused")                      # builds the item table
    reads = []

    def documented(fn):
        def wrapped(*a, **kw):
            reads.append(fn.__name__)
            mode = torch.cuda.get_sync_debug_mode()
            torch.cuda.set_sync_debug_mode(0)
            try:
                return fn(*a, **kw)
            finally:
                torch.cuda.set_sync_debug_mode(mode)
        return wrapped

    orig_err, orig_kept, orig_counts = M.EncoderDecoderRetrievalModel._raise_score_errors, M._read_n_kept, M._read_node_counts
    M.EncoderDecoderRetrievalModel._raise_score_errors = staticmethod(documented(orig_err))
    M._read_n_kept, M._read_node_counts = documented(orig_kept), documented(orig_counts)
    state = torch.cuda.get_rng_state()
    try:
        torch.cuda.set_sync_debug_mode("error")
        again = m.score_items(batch, items, encoder="fused")
    finally:
        torch.cuda.set_sync_debug_mode(0)
        M.EncoderDecoderRetrievalModel._raise_score_errors = staticmethod(orig_err)
        M._read_n_kept, M._read_node_counts = orig_kept, orig_counts
    assert reads == ["_read_node_counts", "_read_n_kept", "_raise_score_errors"]
    assert torch.equal(torch.cuda.get_rng_state(), state)
    assert torch.equal(first.scores, again.scores) and torch.equal(first.target_rank, again.target_rank)
    with pytest.raises(ValueError, match="eval mode"):
        m.train().score_items(batch, items)
    m.eval()
    with pytest.raises(ValueError, match="autocast"), torch.autocast("cuda", dtype=torch.bfloat16):
        m.score_items(batch, items)
    bad = items.clone()
    bad[0, 0], bad[2, 3], bad[1, 1] = len(corpus), -2, -1
    with pytest.raises(ValueError, match=r"score_items: 2 item id\(s\) outside \[-1, N\)"):
        m.score_items(batch, bad)
    with torch.no_grad():
        m.decoder_mlp[1].weight[3, 0] = float("nan")
    with pytest.raises(RuntimeError, match=r"score_items: \d+ decoder row"):
        m.score_items(batch, items)
