"""GPU tests of the exact ranking (csrc/t5rank.cu, modules/model.py FusedT5Rank, rank_sem_ids / rank_items): leaf scores against
the float64 statement of tests/t5_rank_ref.py at "highest" precision, against the beam search's log-probabilities, the selection
against a torch sort of the dense scores, chunking and repeat bit-identity, host reads, modes and the exact-rank metrics.
`pytest -m gpu`."""
import numpy as np
import pytest
import torch

import t5_rank_ref as RR
import t5_step_ref as T
from test_gpu_decode import highest
from test_gpu_generate import history, realistic_corpus

pytestmark = pytest.mark.gpu


def model_for(M, corpus, K, H, k=10, seed=0, d=64):
    torch.manual_seed(seed)
    return M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), num_hierarchies=H, num_embeddings_per_hierarchy=K,
                                          t5_d_model=d, t5_num_heads=2, t5_d_ff=128, t5_num_layers=2, top_k_for_generation=k,
                                          should_add_sep_token=True, num_user_bins=11).cuda().eval()


def batch_for(rs, corpus, B, items, H, K):
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    mask, ids, users = history(rs, B, items, H, K)
    mask[-1] = 0                                                              # a history with every position masked
    fut = corpus[rs.randint(0, len(corpus), size=B)]
    fut = np.concatenate([fut[:, :H], rs.randint(0, 2, size=(B, 1))], axis=1)
    fut[0, 0] = K                                                             # a target that is not retrievable
    w = H + 1
    sem = torch.zeros(B, items * w, dtype=torch.int64, device="cuda")
    seq = torch.zeros(B, items * w, dtype=torch.bool, device="cuda")
    sem.view(B, items, w)[:, :, :H] = ids.view(B, items, H)
    seq.view(B, items, w)[:, :, :H] = mask.view(B, items, H).bool()
    seq.view(B, items, w)[:, :, H] = mask.view(B, items, H)[:, :, -1].bool()
    tt = torch.arange(items * w, device="cuda").remainder(w).expand(B, -1)
    return TokenizedSeqBatch(user_ids=users, sem_ids=sem, sem_ids_fut=torch.from_numpy(fut).cuda(), seq_mask=seq,
                             token_type_ids=tt, token_type_ids_fut=torch.arange(w, device="cuda").expand(B, -1))


def expected_items(scores, corpus, H, K, n):
    """Per history: every (item, score) by a torch sort of the dense leaf scores (NaN last, then tuple, then dedup)."""
    levels, _ = RR.trie_levels(corpus, H, K)
    rows = RR.items_of_leaves(corpus, levels[H])
    counts = np.array([len(r) for r in rows])
    out = []
    for s in scores.cpu().numpy():
        pairs = RR.sort_items(s, counts)
        out.append(pairs)
    return out, rows


@pytest.mark.parametrize("encoder", ["hf", "fused"])
def test_leaf_scores_match_float64(encoder):
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 7
    rs = np.random.RandomState(1)
    corpus = realistic_corpus(rs, 500, H, K)
    corpus[:40, 1] = corpus[40:80, 1] = 3                                      # shared prefixes
    corpus[5] = corpus[6]
    corpus[7, 2] = K                                                         # a row that is never a leaf
    m = model_for(M, corpus, K, H)
    mask, ids, users = history(rs, B, 20, H, K)
    mask[-1] = 0
    with highest():
        got = m.rank_sem_ids(mask, ids, users, encoder=encoder)
        enc_out, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
    levels, parents = RR.trie_levels(corpus, H, K)
    ref = M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), num_hierarchies=H, num_embeddings_per_hierarchy=K,
                                         t5_d_model=64, t5_num_heads=2, t5_d_ff=128, t5_num_layers=2, top_k_for_generation=10,
                                         should_add_sep_token=True, num_user_bins=11)
    ref.load_state_dict(m.state_dict())
    ref = ref.double().eval()
    with torch.no_grad():
        want = RR.rank_decompose(ref, enc_out.double().cpu(), enc_mask.cpu(), levels, parents)
    assert got.shape == (B, len(levels[H]))
    err = (got.double().cpu() - want).abs().max().item()
    assert err <= 1e-5, err


def test_exact_scores_agree_with_beam_search():
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 16
    rs = np.random.RandomState(2)
    corpus = realistic_corpus(rs, 2000, H, K)
    m = model_for(M, corpus, K, H, k=10)
    mask, ids, users = history(rs, B, 20, H, K)
    with highest():
        gen, lp = m.generate(mask, ids, users, search="beam", decoder="fused")
        scores = m.rank_sem_ids(mask, ids, users)
    _, leaf_key, _ = m._rank_levels(scores.device)
    leaf = m._leaf_of(gen.reshape(-1, H), leaf_key).reshape(B, -1)
    finite = torch.isfinite(lp)
    assert finite.any() and (leaf[finite] >= 0).all()
    exact = scores.gather(1, leaf.clamp(min=0))
    assert (exact - lp)[finite].abs().max().item() <= 1e-5
    assert (scores.max(1).values >= lp[:, 0] - 1e-5).all()


@pytest.mark.parametrize("K,H,B,N", [(256, 3, 7, 1500), (1024, 3, 1, 3000), (2048, 5, 7, 2500), (256, 3, 640, 300)])
def test_rank_items_match_sort_and_chunking(K, H, B, N):
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(K + H + B)
    corpus = realistic_corpus(rs, N, H, K)
    corpus[10:14] = corpus[20]                                               # a tuple with several items
    m = model_for(M, corpus, K, H)
    batch = batch_for(rs, corpus, B, 6, H, K)
    with highest():
        out = m.rank_items(batch, n=1024)
        scores = m.rank_sem_ids(M._strip_dedup_col(batch.seq_mask.long(), H + 1, H),
                                M._strip_dedup_col(batch.sem_ids, H + 1, H), batch.user_ids)
        levels = m._rank_levels(scores.device)[0]
        per_history = sum(levels.n[:H])
        chunked = m.rank_items(batch, n=1024, max_rows=per_history)
        again = m.rank_items(batch, n=1024)
    ok = ((corpus >= 0) & (corpus < K)).all(1)
    assert out.num_items == int(ok.sum())
    for o in (chunked, again):
        assert torch.equal(o.item_ids, out.item_ids) and torch.equal(o.scores, out.scores)
        assert torch.equal(o.target_rank, out.target_rank)
    full, rows = expected_items(scores, corpus, H, K, 1024)
    target = m.item_of(batch.sem_ids_fut).cpu().numpy()
    items, sc, rank = out.item_ids.cpu().numpy(), out.scores.cpu().numpy(), out.target_rank.cpu().numpy()
    s_np = scores.cpu().numpy()
    for b in range(B):
        want = [int(rows[u][d]) for u, d in full[b][:1024]]
        assert items[b, :len(want)].tolist() == want and (items[b, len(want):] == -1).all()
        assert np.array_equal(sc[b, :len(want)], s_np[b, [u for u, _ in full[b][:1024]]])
        flat = [int(rows[u][d]) for u, d in full[b]]
        assert rank[b] == (flat.index(target[b]) if target[b] >= 0 else -1)
    assert rank[0] == -1
    for n in (1, 10):
        with highest():
            small = m.rank_items(batch, n=n)
        assert torch.equal(small.item_ids, out.item_ids[:, :n]) and torch.equal(small.target_rank, out.target_rank)


def test_empty_corpus():
    from rq_vae_recommender_b200.modules import model as M
    K, H = 256, 3
    rs = np.random.RandomState(4)
    corpus = np.full((5, H), K, dtype=np.int64)                              # no retrievable row
    m = model_for(M, corpus, K, H)
    batch = batch_for(rs, realistic_corpus(rs, 10, H, K), 3, 4, H, K)
    out = m.rank_items(batch, n=5)
    assert out.num_items == 0 and (out.item_ids == -1).all() and (out.target_rank == -1).all()
    assert m.rank_sem_ids(torch.ones(2, 6, device="cuda"), torch.zeros(2, 6, dtype=torch.int64, device="cuda")).shape == (2, 0)


def test_host_reads_rng_modes_and_nan():
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 5
    rs = np.random.RandomState(5)
    corpus = realistic_corpus(rs, 800, H, K)
    m = model_for(M, corpus, K, H)
    batch = batch_for(rs, corpus, B, 5, H, K)
    m.rank_items(batch)                                                      # builds and caches the trie levels (one read)
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

    orig_bad, orig_kept = M.EncoderDecoderRetrievalModel._raise_bad, M._read_n_kept
    M.EncoderDecoderRetrievalModel._raise_bad = staticmethod(documented(orig_bad))
    M._read_n_kept = documented(orig_kept)
    state = torch.cuda.get_rng_state()
    try:
        a = m.rank_items(batch, encoder="hf")                               # HF's encoder is not this project's to audit
        torch.cuda.set_sync_debug_mode("error")
        b = m.rank_items(batch, encoder="fused")
    finally:
        torch.cuda.set_sync_debug_mode(0)
        M.EncoderDecoderRetrievalModel._raise_bad, M._read_n_kept = staticmethod(orig_bad), orig_kept
    assert reads == ["_raise_bad", "_read_n_kept", "_raise_bad"]           # hf: the NaN count; fused: the row count, the NaN count
    assert torch.equal(torch.cuda.get_rng_state(), state)
    assert (a.target_rank == b.target_rank).float().mean() > 0.5
    with pytest.raises(ValueError, match="eval mode"):
        m.train().rank_items(batch)
    m.eval()
    with pytest.raises(ValueError, match="autocast"), torch.autocast("cuda", dtype=torch.bfloat16):
        m.rank_items(batch)
    with pytest.raises(ValueError, match="n = 1025"):
        m.rank_items(batch, n=1025)
    with torch.no_grad():
        m.decoder_mlp[1].weight[3, 0] = float("nan")
    with pytest.raises(RuntimeError, match=r"rank_items: \d+ decoder row"):
        m.rank_items(batch)


def test_accumulate_ranks_metrics():
    from rq_vae_recommender_b200.evaluate.metrics import TopKAccumulator
    rs = np.random.RandomState(6)
    ks = [1, 5, 10, 50, 100]
    ranks = [rs.randint(-1, 300, size=B) for B in (40, 17)]
    actual = torch.from_numpy(rs.randint(0, 4, size=(40, 3))).cuda()
    cands = torch.from_numpy(rs.randint(0, 4, size=(40, 10, 3))).cuda()
    plain, acc = TopKAccumulator(ks), TopKAccumulator(ks)
    for a in (plain, acc):
        a.accumulate(actual, cands)
    acc.accumulate_ranks(torch.from_numpy(ranks[0]).cuda(), 300)
    acc.accumulate_ranks(torch.from_numpy(ranks[1]).cuda(), 250)              # ranks >= 250 are misses there
    out, base = acc.reduce(), plain.reduce()
    assert {k: v for k, v in out.items() if not k.startswith("exact_")} == base
    r = np.concatenate([ranks[0], np.where(ranks[1] >= 250, -1, ranks[1])]).astype(np.float64)
    hit = r >= 0
    assert abs(out["exact_ndcg"] - float((1.0 / np.log2(r[hit] + 2)).sum()) / len(r)) < 1e-12
    for k in ks:
        assert out[f"exact_h@{k}"] == pytest.approx(float(((r >= 0) & (r < k)).sum()) / len(r), abs=1e-15)


def cross_reference(q, k, v, offsets, key_mask, Q, heads, dtype):
    """The cross-attention statement per history, in dtype (float32 products at the current matmul precision)."""
    out = []
    off = offsets.tolist()
    for b in range(len(off) - 1):
        kb, vb, mb = k[off[b]:off[b + 1]].to(dtype), v[off[b]:off[b + 1]].to(dtype), key_mask[off[b]:off[b + 1]].to(dtype)
        qb = q[b * Q:(b + 1) * Q].to(dtype).reshape(Q, heads, 64).transpose(0, 1)
        s = qb @ kb.reshape(-1, heads, 64).permute(1, 2, 0) + mb
        w = torch.softmax(s, dim=-1)
        out.append((w @ vb.reshape(-1, heads, 64).transpose(0, 1)).transpose(0, 1).reshape(Q, heads * 64))
    return torch.cat(out)


@pytest.mark.parametrize("S,Q,heads", [(1, 1, 1), (81, 257, 6), (7, 64, 2), (200, 1000, 6), (64, 65, 8)])
def test_cross_attention_kernels_against_float64(S, Q, heads):
    """fp32 kernel within 1e-5 of float64; the TF32 kernel's error at most twice that of the float32 statement at "high" (never
    below twice one TF32 unit of the largest entry), the bound tests/test_gpu_encode_tc.py uses."""
    from rq_vae_recommender_b200 import ops
    B, inner = 5, heads * 64
    g = torch.Generator(device="cuda").manual_seed(S + Q + heads)
    lens = torch.tensor([S, max(1, S // 2), S, 1, S])
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), lens.cumsum(0)]).to(torch.int32).cuda()
    rows = int(lens.sum())
    q = torch.randn(B * Q, inner, device="cuda", generator=g) * 0.4
    kv = torch.randn(rows, 3 * inner, device="cuda", generator=g) * 0.4             # strided views of a wider tensor
    k, v = kv[:, :inner], kv[:, 2 * inner:]
    key_mask = torch.where(torch.rand(rows, device="cuda", generator=g) < 0.3, T.NEG, 0.0)
    key_mask[offsets[2]:offsets[3]] = T.NEG                                          # every key masked: the mean of the values
    want = cross_reference(q, k, v, offsets, key_mask, Q, heads, torch.float64)
    top = want.abs().max().item()
    got = ops.t5rank_cross_attention(q, k, v, offsets, key_mask, Q, heads)
    assert (got.double() - want).abs().max().item() <= 1e-5 * max(1.0, top)
    saved = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("high")
    try:
        cmp = cross_reference(q, k, v, offsets, key_mask, Q, heads, torch.float32)
    finally:
        torch.set_float32_matmul_precision(saved)
    tc = ops.t5rank_cross_attention(q, k, v, offsets, key_mask, Q, heads, tf32=True)
    e_tc, e_cmp = (tc.double() - want).abs().max().item(), (cmp.double() - want).abs().max().item()
    assert e_tc <= 2 * max(e_cmp, 2 ** -11 * top), (e_tc, e_cmp)
    assert torch.equal(ops.t5rank_cross_attention(q, k, v, offsets, key_mask, Q, heads, tf32=True), tc)


def test_tf32_attention_rank_items():
    """attention="tf32": scores near the fp32 attention's, bit-identical chunked and repeated."""
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 7
    rs = np.random.RandomState(8)
    corpus = realistic_corpus(rs, 1500, H, K)
    m = model_for(M, corpus, K, H)
    batch = batch_for(rs, corpus, B, 6, H, K)
    ref = m.rank_items(batch, n=100)
    tf = m.rank_items(batch, n=100, attention="tf32")
    per_history = sum(m._rank_levels(ref.scores.device)[0].n[:H])
    chunked = m.rank_items(batch, n=100, attention="tf32", max_rows=2 * per_history)
    assert torch.equal(chunked.item_ids, tf.item_ids) and torch.equal(chunked.scores, tf.scores)
    assert torch.equal(chunked.target_rank, tf.target_rank)
    finite = torch.isfinite(ref.scores)
    assert (tf.scores - ref.scores)[finite].abs().max().item() < 1e-2
    with pytest.raises(ValueError, match="attention must be one of"):
        m.rank_items(batch, attention="bf16")


def test_trie_leaves_are_the_item_table_tuples():
    """The device trie's level-H leaves, in order, are the device item table's tuples: each leaf's key, unpacked, looks up to a
    corpus item, and the leaves' item ranges cover every retrievable row exactly once in the table's order."""
    from rq_vae_recommender_b200.modules import model as M
    K, H = 256, 3
    rs = np.random.RandomState(9)
    corpus = realistic_corpus(rs, 3000, H, K)
    corpus[:50, :2] = corpus[50, :2]                                          # deep shared prefixes
    corpus[60:70] = corpus[70]                                                # duplicates
    corpus[80, 1] = K                                                         # a cut row
    m = model_for(M, corpus, K, H)
    levels, leaf_key, n_items = m._rank_levels(torch.device("cuda"))
    tuples = torch.stack([(leaf_key // K ** (H - 1 - h)) % K for h in range(H)], 1)
    ok = ((corpus >= 0) & (corpus < K)).all(1)
    want = np.unique(corpus[ok], axis=0)
    assert np.array_equal(tuples.cpu().numpy(), want) and levels.n[H] == len(want)
    table = m._item_table(tuples.device)
    row, start = table.arrays()
    first = table.lookup(tuples)
    assert torch.equal(first, row[start[:-1][:len(want)].long()].long())
    assert int(start[len(want)]) == n_items == int(ok.sum())
