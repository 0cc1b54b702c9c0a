"""GPU tests of EncoderDecoderRetrievalModel.capture_exact_items: generate_items(search="exact", encoder="fused", decoder="fused")
replayed as one CUDA graph whose pruned levels are sized on the device.  A replay equals the eager call bit for bit on unpadded
histories (items, beams, count, sem_ids, log_probas) at B = 1 and B > 1, w = n and n > w, head scales 1 and 8, a 4-level model,
with no filter, with exclude_history and with allow-lists; to 1e-5 with the same beams on padded histories.  A max_rows that one
batch exceeds falls back to the eager search; in-place weight updates are followed, a replaced corpus recaptures, side streams
work, a non-finite head row raises the eager error and only the counter read synchronises.  `pytest -m gpu`."""
import re

import numpy as np
import pytest
import torch

from test_gpu_exact_search import sharpen
from test_gpu_generate import dev, realistic_corpus, small_model
from test_gpu_generate_graph import assert_same, batch_of, highest
from test_gpu_inclusion import allow_lists

pytestmark = pytest.mark.gpu

K, N_CORPUS = 256, 12101


@pytest.fixture(scope="module")
def corpus():
    return realistic_corpus(np.random.RandomState(12101), N_CORPUS, 3, K)


def model_of(corpus, H=3, scale=1, seed=0):
    from rq_vae_recommender_b200.modules import model as M
    return sharpen(small_model(M, corpus[:, :H], K, H, seed=seed), scale)


def eager(m, batch, **kw):
    return m.generate_items(batch, search="exact", encoder="fused", decoder="fused", **kw)


@pytest.mark.parametrize("scale", [1, 8])
@pytest.mark.parametrize("B,w,n", [(1, 10, 10), (7, 10, 25), (16, 32, 32)])
def test_replay_equals_eager(corpus, scale, B, w, n):
    from rq_vae_recommender_b200.modules import model as M
    m = model_of(corpus, scale=scale)
    rs = np.random.RandomState(B * 100 + w + scale)
    for filt in ("none", "exclude_history", "include"):
        batch = batch_of(rs, corpus, B, padded=False)
        kw = dict(num_beams=w, n=n, exclude_history=filt == "exclude_history")
        inc = dict(include_items=dev(allow_lists(rs, corpus, max(B, 2), 256)[:B])) if filt == "include" else {}
        g = m.capture_exact_items(batch, **kw, **inc)
        want = eager(m, batch, **kw, **inc)
        rows = M.EXACT_DECODER_ROWS
        got = g(batch, **inc)
        assert got.sem_ids.shape == (B, w, 3) and got.item_ids.shape == (B, n)
        assert_same(got, want)
        assert g.rows == rows and g.fallbacks == 0
        batch2 = batch_of(rs, corpus, B, padded=False)
        assert_same(g(batch2, **inc), eager(m, batch2, **kw, **inc))


def test_four_levels(corpus):
    rs = np.random.RandomState(4)
    c4 = np.concatenate([corpus, rs.randint(0, K, size=(N_CORPUS, 1))], axis=1)
    m = model_of(c4, H=4, scale=8)
    from test_gpu_exclusion import dedup_ranks
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    full = np.concatenate([c4, dedup_ranks(c4)[:, None]], axis=1)
    hist = rs.randint(0, N_CORPUS, size=(5, 6))
    batch = TokenizedSeqBatch(user_ids=None, sem_ids=dev(full[hist].reshape(5, -1)), sem_ids_fut=None,
                              seq_mask=dev(np.ones((5, 6 * 5), dtype=bool)), token_type_ids=None, token_type_ids_fut=None)
    g = m.capture_exact_items(batch, num_beams=10)
    assert_same(g(batch), eager(m, batch, num_beams=10))


def test_padded_histories(corpus):
    m = model_of(corpus, scale=8)
    rs = np.random.RandomState(5)
    batch = batch_of(rs, corpus, 7, padded=True)
    with highest():
        g = m.capture_exact_items(batch, num_beams=10, exclude_history=True)
        assert_same(g(batch), eager(m, batch, num_beams=10, exclude_history=True), exact=False)


def test_small_max_rows_falls_back_to_eager(corpus):
    m = model_of(corpus, scale=1)
    rs = np.random.RandomState(6)
    batch = batch_of(rs, corpus, 7, padded=False)
    want = eager(m, batch, num_beams=10)
    g = m.capture_exact_items(batch, num_beams=10, max_rows=64)
    assert_same(g(batch), want)
    assert g.fallbacks == 1
    big = m.capture_exact_items(batch, num_beams=10, max_rows=1 << 20)
    assert_same(big(batch), want)
    assert big.fallbacks == 0


def test_weights_in_place_and_replaced_corpus(corpus):
    m = model_of(corpus, scale=8)
    rs = np.random.RandomState(7)
    batch = batch_of(rs, corpus, 7, padded=False)
    g = m.capture_exact_items(batch, num_beams=10)
    graph = g._graph
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn_like(p), alpha=0.01)
    assert_same(g(batch), eager(m, batch, num_beams=10))
    assert g._graph is graph
    m.codebooks = m.codebooks.clone()
    m.codebooks[:50] = m.codebooks[50:100].clone()
    assert_same(g(batch), eager(m, batch, num_beams=10))
    assert g._graph is not graph


def test_side_stream(corpus):
    m = model_of(corpus, scale=8)
    rs = np.random.RandomState(8)
    batch = batch_of(rs, corpus, 7, padded=False)
    want = eager(m, batch, num_beams=10)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        g = m.capture_exact_items(batch, num_beams=10)
        got = g(batch)
    torch.cuda.current_stream().wait_stream(side)
    assert_same(got, want)


def test_non_finite_head_row_raises_the_eager_error(corpus):
    m = model_of(corpus, scale=1, seed=8)
    batch = batch_of(np.random.RandomState(9), corpus, 7, padded=False)
    g = m.capture_exact_items(batch, num_beams=10)
    with torch.no_grad():
        m.decoder_mlp[2].weight[0] = float("nan")
    with pytest.raises(RuntimeError) as err:
        eager(m, batch, num_beams=10)
    with pytest.raises(RuntimeError, match=re.escape(str(err.value))):
        g(batch)


def test_only_the_counter_read_synchronises(corpus):
    from rq_vae_recommender_b200.modules import model as M
    m = model_of(corpus, scale=8)
    rs = np.random.RandomState(10)
    batch = batch_of(rs, corpus, 7, padded=False)
    g = m.capture_exact_items(batch, num_beams=10, exclude_history=True)
    g(batch)
    read = M._read_search_counters
    reads = []

    def allowed(values):
        reads.append(1)
        torch.cuda.set_sync_debug_mode(0)
        try:
            return read(values)
        finally:
            torch.cuda.set_sync_debug_mode("error")

    torch.cuda.synchronize()
    M._read_search_counters = allowed
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = g(batch)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        M._read_search_counters = read
    assert reads == [1] and out.item_ids.shape == (7, 10)
