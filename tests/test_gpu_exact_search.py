"""GPU tests of the exact top-k search (generate(search="exact"): modules/model.py FusedT5Exact, csrc/t5rank.cu
t5exact_frontier / t5exact_select / t5rank_cross_attention_ragged): bit-identity with the dense top-w of rank_sem_ids at random
init and with sharpened heads that prune, generate_items against rank_items, allow-lists, chunk reruns, decoders, encoders,
repeats, side streams, the ragged cross-attention against the uniform kernel, and the errors.  `pytest -m gpu`."""
import numpy as np
import pytest
import torch

from test_gpu_decode import highest
from test_gpu_generate import history, realistic_corpus
from test_gpu_rank import batch_for, model_for

pytestmark = pytest.mark.gpu

WIDTHS = (1, 10, 32, 257, 1024)


def sharpen(m, scale):
    """The heads' weights times scale: a stand-in for a trained, more confident model, under which the search prunes."""
    with torch.no_grad():
        for mlp in m.decoder_mlp:
            mlp.weight.mul_(scale)
    return m


def leaf_tuples(m, H, K):
    _, leaf_key, _ = m._rank_levels(torch.device("cuda"))
    return torch.stack([(leaf_key // K ** (H - 1 - h)) % K for h in range(H)], 1)


def dense_topw(scores, tuples, w, valid=None):
    """The w best leaves per history of the dense scores [B, U] by score descending, then tuple (leaf) ascending, NaN and
    invalid leaves left out, -1 / -inf past them."""
    B, U = scores.shape
    H = tuples.shape[1]
    s = scores.cpu().numpy()
    ok = ~np.isnan(s) if valid is None else (~np.isnan(s) & valid.cpu().numpy())
    gen = np.full((B, w, H), -1, dtype=np.int64)
    lp = np.full((B, w), -np.inf, dtype=np.float32)
    t = tuples.cpu().numpy()
    for b in range(B):
        idx = np.nonzero(ok[b])[0]
        order = idx[np.lexsort((idx, -s[b, idx]))][:w]
        gen[b, :len(order)] = t[order]
        lp[b, :len(order)] = s[b, order]
    return torch.from_numpy(gen).cuda(), torch.from_numpy(lp).cuda()


def assert_same(got, want):
    assert torch.equal(got[0], want[0]), "tuples differ"
    assert torch.equal(got[1], want[1]), "scores differ"


SHAPES = {                                                   # K, H, corpus rows, histories
    "k256_h3": (256, 3, 2000, 6),
    "k300_h5": (300, 5, 1200, 5),
    "k2048_h3": (2048, 3, 3000, 3),
    "k128_h8": (128, 8, 800, 4),                             # H = 8 packs into 62 bits up to K = 128
}


@pytest.mark.parametrize("scale", [1, 8, 32])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_exact_equals_dense_topw(shape, scale):
    from rq_vae_recommender_b200.modules import model as M
    K, H, N, B = SHAPES[shape]
    rs = np.random.RandomState(K + H + scale)
    corpus = realistic_corpus(rs, N, H, K)
    corpus[:30, :H - 1] = corpus[30, :H - 1]                 # a deep shared prefix
    m = sharpen(model_for(M, corpus, K, H), scale)
    mask, ids, users = history(rs, B, 10, H, K)
    dense = m.rank_sem_ids(mask, ids, users)
    tuples = leaf_tuples(m, H, K)
    levels = m._rank_levels(dense.device)[0]
    full = sum(levels.n[:H]) * B
    for w in (w for w in WIDTHS if w <= K):
        got = m.generate(mask, ids, users, search="exact", num_beams=w)
        assert got[0].shape == (B, w, H) and got[1].shape == (B, w)
        assert_same(got, dense_topw(dense, tuples, w))
        if scale > 1 and w <= 32:
            assert M.EXACT_DECODER_ROWS < full, (M.EXACT_DECODER_ROWS, full)


def test_fewer_leaves_than_width():
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 300, 3, 4
    rs = np.random.RandomState(11)
    corpus = realistic_corpus(rs, 200, H, K)                 # fewer than 257 distinct tuples
    m = model_for(M, corpus, K, H)
    mask, ids, users = history(rs, B, 8, H, K)
    dense = m.rank_sem_ids(mask, ids, users)
    for w in (257, 256):
        got = m.generate(mask, ids, users, search="exact", num_beams=w)
        assert_same(got, dense_topw(dense, leaf_tuples(m, H, K), w))
        assert (got[0][:, dense.shape[1]:] == -1).all() and torch.isinf(got[1][:, dense.shape[1]:]).all()


@pytest.mark.parametrize("exclude_history", [False, True])
def test_generate_items_equals_rank_items(exclude_history):
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 7
    rs = np.random.RandomState(12)
    corpus = realistic_corpus(rs, 1500, H, K)
    corpus[10:14] = corpus[20]                               # a tuple with several items
    m = sharpen(model_for(M, corpus, K, H), 8)
    batch = batch_for(rs, corpus, B, 6, H, K)
    batch.sem_ids.view(B, 6, H + 1)[:, :3, :H] = torch.from_numpy(corpus[20:23]).cuda()   # seen items the search must skip
    for n in (1, 10, 100):
        got = m.generate_items(batch, n=n, num_beams=n, search="exact", exclude_history=exclude_history)
        want = m.rank_items(batch, n=n, exclude_history=exclude_history)
        assert torch.equal(got.item_ids, want.item_ids)
        scores = torch.where(got.item_ids >= 0, got.log_probas.gather(1, got.beams.clamp(min=0).long()), float("-inf"))
        assert torch.equal(scores, want.scores)


def test_allow_lists():
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, w = 256, 3, 5, 20
    rs = np.random.RandomState(13)
    corpus = realistic_corpus(rs, 1500, H, K)
    m = sharpen(model_for(M, corpus, K, H), 8)
    mask, ids, users = history(rs, B, 8, H, K)
    allowed = rs.randint(-1, len(corpus), size=(B, 300))
    allowed[1] = -1                                          # a history with no eligible item
    allowed[2, :5] = 7                                       # repeats
    dense = m.rank_sem_ids(mask, ids, users)
    _, leaf_key, _ = m._rank_levels(dense.device)
    valid = torch.zeros_like(dense, dtype=torch.bool)
    for b in range(B):
        rows = allowed[b][allowed[b] >= 0]
        leaf = m._leaf_of(torch.from_numpy(corpus[rows]).cuda(), leaf_key)
        valid[b, leaf[leaf >= 0]] = True
    got = m.generate(mask, ids, users, search="exact", num_beams=w, include_items=torch.from_numpy(allowed).cuda())
    assert_same(got, dense_topw(dense, leaf_tuples(m, H, K), w, valid))
    assert (got[0][1] == -1).all()


def test_same_result_across_settings(monkeypatch):
    """At random init (nearly nothing pruned) so that a one-level budget forces chunk reruns."""
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, w = 256, 3, 9, 32
    rs = np.random.RandomState(14)
    corpus = realistic_corpus(rs, 2000, H, K)
    m = model_for(M, corpus, K, H)
    mask, ids, users = history(rs, B, 8, H, K)
    ref = m.generate(mask, ids, users, search="exact", num_beams=w, decoder="fused")
    rows = M.EXACT_DECODER_ROWS
    assert_same(m.generate(mask, ids, users, search="exact", num_beams=w, decoder="fused"), ref)    # repeated
    assert_same(m.generate(mask, ids, users, search="exact", num_beams=w, decoder="hf"), ref)       # the bound's decoder
    levels = m._rank_levels(ref[0].device)[0]
    monkeypatch.setattr(M, "RANK_BYTE_BUDGET", max(levels.n[:H]) * M.FusedT5Rank.row_bytes(m))   # chunk reruns
    run, reruns = M.FusedT5Exact.run, []

    def counted(self, *a, **kw):
        out = run(self, *a, **kw)
        reruns.append(out is None)
        return out

    monkeypatch.setattr(M.FusedT5Exact, "run", counted)
    assert_same(m.generate(mask, ids, users, search="exact", num_beams=w), ref)
    assert any(reruns) and M.EXACT_DECODER_ROWS == rows
    monkeypatch.undo()
    for encoder in ("hf", "fused"):                          # each encoder: its own dense ranking, bit for bit
        with highest():
            dense = m.rank_sem_ids(mask, ids, users, encoder=encoder)
            got = m.generate(mask, ids, users, search="exact", num_beams=w, encoder=encoder)
        assert_same(got, dense_topw(dense, leaf_tuples(m, H, K), w))


def test_side_stream():
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, w = 256, 3, 6, 10
    rs = np.random.RandomState(15)
    corpus = realistic_corpus(rs, 1500, H, K)
    m = sharpen(model_for(M, corpus, K, H), 8)
    mask, ids, users = history(rs, B, 8, H, K)
    ref = m.generate(mask, ids, users, search="exact", num_beams=w, encoder="fused", decoder="fused")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = m.generate(mask, ids, users, search="exact", num_beams=w, encoder="fused", decoder="fused")
    torch.cuda.current_stream().wait_stream(s)
    assert_same(got, ref)


def test_ragged_cross_attention_equals_uniform():
    from rq_vae_recommender_b200 import ops
    B, Q, heads = 5, 150, 3
    inner = heads * 64
    g = torch.Generator(device="cuda").manual_seed(3)
    lens = torch.tensor([9, 1, 130, 40, 77])
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), lens.cumsum(0)]).to(torch.int32).cuda()
    kv = torch.randn(int(lens.sum()), 2 * inner, device="cuda", generator=g) * 0.4
    key_mask = torch.where(torch.rand(kv.shape[0], device="cuda", generator=g) < 0.3, -3.4e38, 0.0)
    q = torch.randn(B * Q, inner, device="cuda", generator=g) * 0.4
    uniform = ops.t5rank_cross_attention(q, kv[:, :inner], kv[:, inner:], offsets, key_mask, Q, heads)
    counts = [0, 1, 64, 65, 150]                             # queries per history: none, one, one tile, a tile and one, all
    pick = torch.cat([torch.arange(b * Q, b * Q + c) for b, c in enumerate(counts)]).cuda()
    tiles, row = [], 0
    for b, c in enumerate(counts):
        for t0 in range(0, c, 64):
            tiles.append((b, row + t0, min(64, c - t0)))
        row += c
    tiles = torch.tensor(tiles, dtype=torch.int32).cuda()
    got = ops.t5rank_cross_attention_ragged(q[pick], kv[:, :inner], kv[:, inner:], offsets, key_mask, tiles, heads)
    assert torch.equal(got, uniform[pick])


def test_errors():
    from rq_vae_recommender_b200._lib import Rqb200Error
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 3
    rs = np.random.RandomState(16)
    corpus = realistic_corpus(rs, 500, H, K)
    m = model_for(M, corpus, K, H)
    mask, ids, users = history(rs, B, 5, H, K)
    with pytest.raises(ValueError, match="eval mode"):
        m.train().generate(mask, ids, users, search="exact")
    m.eval()
    with pytest.raises(ValueError, match="autocast"), torch.autocast("cuda", dtype=torch.bfloat16):
        m.generate(mask, ids, users, search="exact")
    for w in (0, K + 1, 1025):
        with pytest.raises(Rqb200Error, match="exact search's limits"):
            m.generate(mask, ids, users, search="exact", num_beams=w)
    deep = model_for(M, realistic_corpus(rs, 50, 8, K), K, 8)   # 8 levels of 256 codes: 64 bits
    with pytest.raises(Rqb200Error, match="64-bit tuple key"):
        deep.generate(torch.ones(2, 16, device="cuda"), torch.zeros(2, 16, dtype=torch.int64, device="cuda"), search="exact")
    with torch.no_grad():
        m.decoder_mlp[2].weight[5, 0] = float("nan")         # every level-2 row holds a NaN logit
    with pytest.raises(RuntimeError, match=r"generate: \d+ beam row"):
        m.generate(mask, ids, users, search="exact", num_beams=4)
    m._finish_search = lambda *a: None                       # past the bound's own check: the exact pass counts its rows
    with pytest.raises(RuntimeError, match=r"generate\(search=\"exact\"\): \d+ decoder row"):
        m.generate(mask, ids, users, search="exact", num_beams=4)


def test_dropin_default_search():
    import sys
    import rq_vae_recommender_b200.dropin as dropin
    from rq_vae_recommender_b200.modules import model as M
    saved = {name: sys.modules.get(name) for name in ("gin", "modules.model", "init", "distributions")}
    try:
        dropin.install(replace_model=True, search="exact")
        assert M.DEFAULT_SEARCH == "exact"
        K, H, B = 256, 3, 3
        rs = np.random.RandomState(17)
        corpus = realistic_corpus(rs, 500, H, K)
        m = model_for(M, corpus, K, H, k=5)
        mask, ids, users = history(rs, B, 5, H, K)
        assert_same(m.generate(mask, ids, users), dense_topw(m.rank_sem_ids(mask, ids, users), leaf_tuples(m, H, K), 5))
    finally:
        dropin.uninstall()
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod
    assert M.DEFAULT_SEARCH == "sample"
