"""GPU tests of the wide beam searches: the cluster selection kernels of csrc/sid.cu (ops.SidPrefixIndex.beam_topk_wide /
sample_select_wide) against the numpy oracles, a torch composition and today's one-CTA kernels, at every cluster size and on
both sides of the shared-memory key capacity; the decode cross-attention at any number of queries; and the model's
generate(num_beams=...).  `pytest -m gpu`."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import beam_search_oracle as BO
import sample_oracle as SO
from oracle import rq_oracle as O
from test_gpu_beam_search import assert_matches, oracle_level, torch_level
from test_gpu_exclusion import built as built_exclusion, corpus_with_subtrees, exclusion_sets
from test_gpu_generate import dev, history, level_logits, realistic_corpus, small_model
from test_gpu_inclusion import allow_lists, built as built_inclusion

pytestmark = pytest.mark.gpu

NC = 64
SMEM_KEYS = 16 * 1024                                         # SID_WIDE_SMEM_KEYS: score keys a CTA holds in shared memory


def _levels(rs, corpus, B, k, K, n_levels=3, clip=60):
    """Yields (h, kp, logits) of n_levels levels; the caller feeds each level's beams back through send()."""
    generated = None
    for h in range(n_levels):
        kp = 1 if h == 0 else k
        logits = level_logits(rs, corpus, None if h == 0 else generated.reshape(-1, h).cpu().numpy(), B * kp, K)
        generated = yield h, kp, dev(np.clip(logits, -clip, clip))


def _run_levels(rs, corpus, B, k, K, step, n_levels=3):
    """Runs step(logits, generated, log_probas) -> (generated, log_probas, parent) over n_levels levels; returns every level's
    (logits, generated in, log_probas in, out)."""
    out, generated, log_probas = [], None, None
    gen = _levels(rs, corpus, B, k, K, n_levels)
    h, kp, logits = next(gen)
    while True:
        got = step(logits, generated, log_probas)
        out.append((logits, generated, log_probas, got))
        generated, log_probas = got[0], got[1]
        try:
            h, kp, logits = gen.send(generated)
        except StopIteration:
            return out


def _equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------------- exhaustive, oracle
@pytest.mark.parametrize("k,K", [(1, 256), (33, 256), (64, 1000), (100, 256), (256, 1000), (33, 2048), (1024, 2048)])
def test_beam_topk_wide_vs_oracle(k, K):
    """Three levels against the float64 numpy oracle (small shapes) or the torch composition (large ones), with the gap rule
    of test_gpu_beam_search.assert_matches."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(k * 7 + K)
    corpus = realistic_corpus(rs, 12101, 3, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    B = 3 if k * K >= 256 * 1000 else 5
    for logits, generated, log_probas, got in _run_levels(rs, corpus, B, k, K,
                                                          lambda lg, g, p: idx.beam_topk_wide(lg, g, p, k)):
        h = 0 if generated is None else generated.shape[2]
        assert got[0].shape == (B, k, h + 1) and got[1].shape == (B, k) and got[2].shape == (B * k,)
        E = logits.shape[0] // B * K
        if E <= 64 * 1024:
            assert_matches(*oracle_level(corpus, logits, generated, log_probas, k), got, k)
        else:
            ref = (t.cpu().numpy() for t in torch_level(idx, logits, generated, log_probas, min(k, E - 1)))
            assert_matches(*ref, got, k, exact_ties=False, min_checked=0.3)


def test_beam_topk_wide_exact_ties_fillers_and_bad_rows():
    """Integer logits tie exactly: equal scores come out lowest beam * K + code first, bit-identical to the oracle's order; a
    sparse corpus fills with -inf in index order; NaN / +inf / all -inf rows are counted and complete."""
    from rq_vae_recommender_b200 import ops
    K, C, B, kp, k = 64, 2, 3, 40, 60
    corpus = np.stack(np.meshgrid(np.arange(K), np.arange(K), indexing="ij"), -1).reshape(-1, C).astype(np.int64)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    rs = np.random.RandomState(3)
    generated = rs.randint(0, K, size=(B, kp, 1)).astype(np.int64)
    log_probas = rs.randint(-2, 1, size=(B, kp)).astype(np.float32)
    logits = rs.randint(0, 3, size=(B * kp, K)).astype(np.float32)
    g, p, par = idx.beam_topk_wide(dev(logits), dev(generated), dev(log_probas), k)
    og, op, opar = BO.beam_topk(corpus, logits, generated, log_probas, k)
    assert np.array_equal(g.cpu().numpy(), og) and np.array_equal(par.cpu().numpy().reshape(B, k), opar)
    np.testing.assert_allclose(p.cpu().numpy(), op, rtol=1e-5, atol=1e-5)
    assert (op[:, 1:] == op[:, :-1]).sum() > B * 50
    # sparse corpus: 3 valid extensions at level 0, then -inf fillers in ascending code order
    sparse = np.array([[5, 1], [5, 2], [60, 7]], dtype=np.int64)
    sidx = ops.SidPrefixIndex(dev(sparse), K)
    lg0 = rs.randn(B, K).astype(np.float32)
    g, p, par = sidx.beam_topk_wide(dev(lg0), None, None, 40)
    og, op, opar = BO.beam_topk(sparse, lg0, None, None, 40)
    assert np.array_equal(g.cpu().numpy(), og) and np.isneginf(p.cpu().numpy()[:, 2:]).all()
    # bad rows
    bad_logits = logits.copy()
    bad_logits[1, 3] = np.nan
    bad_logits[7, 0] = np.inf
    bad_logits[50] = -np.inf
    bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    g, p, par = idx.beam_topk_wide(dev(bad_logits), dev(generated), dev(log_probas), k, bad=bad)
    assert int(bad) == 3 and bool(torch.isfinite(p[:, 0]).all())


# ---------------------------------------------------------------------------------------------------------- sampled, oracle
@pytest.mark.parametrize("kp,k,K", [(1, 33, 256), (33, 64, 1000), (33, 1024, 256), (256, 100, 2048), (1024, 1024, 256),
                                    (1, 1024, 256), (256, 256, 1000)])
def test_sample_select_wide_vs_oracle(kp, k, K):
    """One level of kp beams (level 1 from a random beam set, or level 0) against sample_oracle.sample_select: the samples
    bit for bit, the kept beams as the oracle's stable sort, including k > kp * 64 (entry 0 repeated with -inf)."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(kp + k + K)
    corpus = realistic_corpus(rs, 12101, 3, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    B = 3
    if kp == 1:
        generated, log_probas = None, None
    else:
        generated = corpus[rs.randint(0, len(corpus), size=B * kp), :1].reshape(B, kp, 1)
        log_probas = -np.abs(rs.randn(B, kp)).astype(np.float32)
    logits = level_logits(rs, corpus, None if generated is None else generated.reshape(-1, 1), B * kp, K)
    probas = F.softmax(dev(logits), dim=-1)
    noise = torch.empty_like(probas).exponential_(1)
    g, p, par, s, lp = idx.sample_select_wide(probas, noise, None if generated is None else dev(generated),
                                              None if log_probas is None else dev(log_probas), k, NC, want_samples=True)
    n = min(k, kp * NC)
    osamp, olp = SO.sample_select(corpus, probas.cpu().numpy(), noise.cpu().numpy(), generated, log_probas, n, NC)[3:]
    assert np.array_equal(s.cpu().numpy(), osamp)
    np.testing.assert_allclose(lp.cpu().numpy(), olp, rtol=1e-6, atol=0)
    # the selection from the kernel's own draws: the oracle's stable sort of the same fp32 scores, bit for bit
    og, op, opar = O.beam_select(corpus, s.cpu().numpy(), lp.cpu().numpy(), generated, log_probas, n)
    assert np.array_equal(p.cpu().numpy()[:, :n], op) and np.array_equal(g.cpu().numpy()[:, :n], og)
    assert np.array_equal(par.cpu().numpy().reshape(B, k)[:, :n], opar)
    if k > n:                                                    # the rest repeat candidate 0 with -inf
        assert np.isneginf(p.cpu().numpy()[:, n:]).all()
        assert (par.cpu().numpy().reshape(B, k)[:, n:] == (np.arange(B) * kp)[:, None]).all()
        assert (g.cpu().numpy()[:, n:, -1] == s.cpu().numpy().reshape(B, kp * NC)[:, :1]).all()


def test_sample_select_wide_rejected_rows_complete_and_are_counted():
    from rq_vae_recommender_b200 import ops
    B, K, kp, k = 4, 256, 40, 64
    rs = np.random.RandomState(3)
    corpus = realistic_corpus(rs, 5000, 3, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    probas = F.softmax(dev(rs.randn(B * kp, K).astype(np.float32)), dim=-1)
    noise = torch.empty_like(probas).exponential_(1)
    generated = dev(corpus[rs.randint(0, 5000, size=B * kp), :1].reshape(B, kp, 1))
    lp = torch.zeros((B, kp), device="cuda")
    bad = probas.clone()
    bad[1, 7] = float("nan")
    bad[2, 0] = -1e-3
    bad[4, 200] = float("inf")
    bad[8] = 0.0
    reject = torch.zeros(2, dtype=torch.int32, device="cuda")
    out = idx.sample_select_wide(bad, noise, generated, lp, k, NC, reject=reject)
    torch.cuda.synchronize()
    assert reject.tolist() == [3, 1] and out[0].shape == (B, k, 2)


# ------------------------------------------------------------------------------------------------ bit for bit, cluster sizes
def _filters(kind, corpus, K, B, rs):
    if kind == "none":
        return {}
    if kind == "exclude":
        _, _, ex = built_exclusion(corpus, K, exclusion_sets(rs, corpus, B, 64))
        return {"exclude": ex}
    _, _, inc, _ = built_inclusion(corpus, K, allow_lists(rs, corpus, B, 256))
    return {"include": inc}


@pytest.mark.parametrize("kind", ["none", "exclude", "include"])
@pytest.mark.parametrize("K", [256, 2048])
def test_wide_equals_narrow_where_both_run(kind, K):
    """At every shape both kernels take (k <= 32; sampled kp * 64 <= 1024) the wide kernels give the narrow kernels' bits."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K + len(kind))
    B, H = 64, 3
    corpus = corpus_with_subtrees(rs, 6000, H, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    filt = _filters(kind, corpus, K, B, rs)
    for k in (1, 10, 32):
        bad_n, bad_w = (torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(2))
        levels = _run_levels(rs, corpus, B, k, K, lambda lg, g, p: idx.beam_topk(lg, g, p, k, bad=bad_n, **filt))
        for logits, generated, log_probas, got in levels:
            assert _equal(idx.beam_topk_wide(logits, generated, log_probas, k, bad=bad_w, **filt), got)
        assert torch.equal(bad_n, bad_w)
    for k in (1, 10, 16):
        generated, log_probas = None, None
        for h in range(H):
            kp = 1 if h == 0 else k
            logits = level_logits(rs, corpus, None if h == 0 else generated.reshape(-1, h).cpu().numpy(), B * kp, K)
            probas = F.softmax(dev(logits), dim=-1)
            noise = torch.empty_like(probas).exponential_(1)
            rn, rw = (torch.zeros(2, dtype=torch.int32, device="cuda") for _ in range(2))
            a = idx.sample_select(probas, noise, generated, log_probas, k, NC, want_samples=True, reject=rn, **filt)
            b = idx.sample_select_wide(probas, noise, generated, log_probas, k, NC, want_samples=True, reject=rw, **filt)
            assert _equal(a, b) and torch.equal(rn, rw)
            generated, log_probas = a[0], a[1]


@pytest.mark.parametrize("search", ["beam", "sample"])
@pytest.mark.parametrize("kind", ["none", "exclude", "include"])
def test_cluster_size_does_not_matter(search, kind):
    """Bit-identical results for cluster = 1, 2, 4, 8 and the launcher's choice, over the shared-memory key capacity: at
    K = 256 a CTA keeps its exhaustive keys for at most 64 beams, its sampled keys for at most 256."""
    from rq_vae_recommender_b200 import ops
    K, B, H = 256, 4, 3
    rs = np.random.RandomState(5 + len(kind))
    corpus = corpus_with_subtrees(rs, 12101, H, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    filt = _filters(kind, corpus, K, B, rs)
    kp, k = 1024, 256
    generated = dev(corpus[rs.randint(0, len(corpus), size=B * kp), :1].reshape(B, kp, 1))
    log_probas = dev(-np.abs(rs.randn(B, kp)).astype(np.float32))
    logits = dev(np.clip(level_logits(rs, corpus, generated.reshape(-1, 1).cpu().numpy(), B * kp, K), -60, 60))
    if search == "beam":
        run = lambda c: idx.beam_topk_wide(logits, generated, log_probas, k, cluster=c, **filt)
    else:
        probas = F.softmax(logits, dim=-1)
        noise = torch.empty_like(probas).exponential_(1)
        run = lambda c: idx.sample_select_wide(probas, noise, generated, log_probas, k, NC, want_samples=True, cluster=c, **filt)
    ref = run(1)
    for c in (2, 4, 8, 0):
        assert _equal(run(c), ref), c


@pytest.mark.parametrize("search", ["beam", "sample"])
def test_key_capacity_edges(search):
    """A CTA's slice at the shared-memory key capacity -1, 0 and +1 (cluster = 1: keys stored, stored, recomputed / re-read)
    gives the bits of the same level split over 8 CTAs (keys stored)."""
    from rq_vae_recommender_b200 import ops
    K, B = 256, 3
    per = SMEM_KEYS // (K if search == "beam" else NC)
    rs = np.random.RandomState(17)
    corpus = realistic_corpus(rs, 12101, 3, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    for kp in (per - 1, per, per + 1):
        generated = dev(corpus[rs.randint(0, len(corpus), size=B * kp), :1].reshape(B, kp, 1))
        log_probas = dev(-np.abs(rs.randn(B, kp)).astype(np.float32))
        logits = dev(np.clip(level_logits(rs, corpus, generated.reshape(-1, 1).cpu().numpy(), B * kp, K), -60, 60))
        k = min(kp, 100)
        if search == "beam":
            a, b = (idx.beam_topk_wide(logits, generated, log_probas, k, cluster=c) for c in (1, 8))
        else:
            probas = F.softmax(logits, dim=-1)
            noise = torch.empty_like(probas).exponential_(1)
            a, b = (idx.sample_select_wide(probas, noise, generated, log_probas, k, NC, cluster=c) for c in (1, 8))
        assert _equal(a, b), kp


def test_wide_argument_limits_raise():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200._lib import Rqb200Error
    rs = np.random.RandomState(13)
    idx = ops.SidPrefixIndex(dev(realistic_corpus(rs, 500, 3, 256)), 256)
    lg = dev(rs.randn(2, 256).astype(np.float32))
    with pytest.raises(Rqb200Error, match="k <= K"):
        idx.beam_topk_wide(lg, None, None, 257)
    with pytest.raises(Rqb200Error, match="cluster = 3"):
        idx.beam_topk_wide(lg, None, None, 10, cluster=3)
    p = F.softmax(lg, dim=-1)
    with pytest.raises(Rqb200Error, match="k = 1025"):
        idx.sample_select_wide(p, torch.empty_like(p).exponential_(1), None, None, 1025, NC)


# ------------------------------------------------------------------------------------------------------------ cross-attention
@pytest.mark.parametrize("nq", [33, 256, 1024])
def test_cross_attention_any_nq(nq):
    """Within 1e-5 of T.cross_attention-style float64 maths, and bit-identical to the same queries in slices of <= 32."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(nq)
    B, S, heads = 3, 21, 2
    inner = heads * 64
    q = dev(rs.randn(B * nq, inner).astype(np.float32))
    k = dev(rs.randn(B * S, inner).astype(np.float32) * 0.3)
    v = dev(rs.randn(B * S, inner).astype(np.float32))
    mask = torch.ones((B, S), device="cuda")
    mask[0, 5:] = 0
    out = ops.t5dec_cross_attention(q, k, v, mask, nq, heads)
    qd = q.double().view(B, nq, heads, 64).transpose(1, 2)
    kd = k.double().view(B, S, heads, 64).transpose(1, 2)
    vd = v.double().view(B, S, heads, 64).transpose(1, 2)
    bias = torch.where(mask == 0, torch.finfo(torch.float32).min, 0.0).double()[:, None, None, :]
    ref = torch.softmax(qd @ kd.transpose(-1, -2) + bias, -1) @ vd
    ref = ref.transpose(1, 2).reshape(B * nq, inner)
    assert (out.double() - ref).abs().max().item() < 1e-5
    qb = q.view(B, nq, inner)
    for i0 in range(0, nq, 32):
        part = qb[:, i0:i0 + 32].reshape(-1, inner).contiguous()
        n = min(32, nq - i0)
        assert torch.equal(ops.t5dec_cross_attention(part, k, v, mask, n, heads).view(B, n, inner), out.view(B, nq, inner)[:, i0:i0 + 32])


# ---------------------------------------------------------------------------------------------------------------------- model
@pytest.mark.parametrize("search", ["beam", "sample"])
@pytest.mark.parametrize("w", [33, 64, 256])
def test_generate_wide_fused_equals_hf(search, w):
    """generate(num_beams=w): shapes [B, w, H]; under "highest" precision the fused and HF decoders give identical beams."""
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 6
    rs = np.random.RandomState(w)
    m = small_model(M, realistic_corpus(rs, 3000, H, K), K, H)
    mask, ids, users = history(rs, B, 10, H, K)
    prev = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("highest")
    try:
        torch.manual_seed(3)
        g_f, p_f = m.generate(mask, ids, users, search=search, decoder="fused", num_beams=w)
        torch.manual_seed(3)
        g_h, p_h = m.generate(mask, ids, users, search=search, decoder="hf", num_beams=w)
    finally:
        torch.set_float32_matmul_precision(prev)
    assert g_f.shape == (B, w, H) and p_f.shape == (B, w)
    fin = torch.isfinite(p_h)
    assert torch.equal(torch.isfinite(p_f), fin) and torch.equal(g_f[fin], g_h[fin])
    torch.testing.assert_close(p_f[fin], p_h[fin], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("search,w", [("beam", 1), ("beam", 32), ("sample", 5), ("sample", 16)])
def test_generate_narrow_widths_equal_default(search, w):
    """num_beams inside today's limits runs today's kernels: the bits and launch count of top_k_for_generation = w."""
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 8
    rs = np.random.RandomState(40 + w)
    corpus = realistic_corpus(rs, 3000, H, K)
    m = small_model(M, corpus, K, H, k=w)
    mask, ids, users = history(rs, B, 10, H, K)
    m.generate(mask, ids, users, search=search)                               # builds the index
    torch.manual_seed(8)
    n0 = ops.LAUNCHES
    a = m.generate(mask, ids, users, search=search)
    n1 = ops.LAUNCHES
    torch.manual_seed(8)
    m.top_k_for_generation = 10
    b = m.generate(mask, ids, users, search=search, num_beams=w)
    assert _equal(a, b) and ops.LAUNCHES - n1 == n1 - n0


@pytest.mark.parametrize("w", [20, 64])
def test_generate_sampled_wide_equals_composition(w):
    """The sampled search at width w equals the reference's per-level loop (torch.multinomial + beam_select) under one seed."""
    from rq_vae_recommender_b200.modules import model as M

    class Composed(M.EncoderDecoderRetrievalModel):
        def _sample_and_select(self, index, probas, generated, log_probas, k, n_cands, reject, wide=False):
            samples = torch.multinomial(probas, n_cands)
            samp_log_p = torch.log(torch.gather(probas, 1, samples))
            kp = 1 if generated is None else generated.shape[1]
            B = probas.shape[0] // kp
            scores = samp_log_p.view(B, kp * n_cands) + (0 if log_probas is None else log_probas.repeat_interleave(n_cands, 1))
            h = 0 if generated is None else generated.shape[2]
            prefix = samples.reshape(-1, 1) if h == 0 else torch.cat(
                [generated.reshape(-1, h).repeat_interleave(n_cands, 0), samples.reshape(-1, 1)], 1)
            scores = scores.masked_fill(~index.check(prefix).view(B, -1) | torch.isnan(scores), float("-inf"))
            s, order = scores.sort(dim=-1, descending=True, stable=True)
            top, s = order[:, :k], s[:, :k]
            parent = top // n_cands
            tok = torch.gather(samples.view(B, -1), 1, top).unsqueeze(-1)
            gen = tok if h == 0 else torch.cat([torch.gather(generated, 1, parent.unsqueeze(-1).expand(-1, -1, h)), tok], -1)
            return gen, s, (parent + torch.arange(B, device=probas.device)[:, None] * kp).reshape(-1)

    K, H, B = 256, 3, 8
    rs = np.random.RandomState(60 + w)
    corpus = realistic_corpus(rs, 3000, H, K)
    fused = small_model(M, corpus, K, H)
    composed = small_model(M, corpus, K, H, seed=1)
    composed.load_state_dict(fused.state_dict())
    mask, ids, users = history(rs, B, 10, H, K)
    torch.manual_seed(5)
    g_f, p_f = fused.generate(mask, ids, users, search="sample", num_beams=w)
    torch.manual_seed(5)
    g_c, p_c = composed.generate(mask, ids, users, search="sample", num_beams=w)
    fin = torch.isfinite(p_c)
    assert torch.equal(torch.isfinite(p_f), fin) and torch.equal(g_f[fin], g_c[fin]) and torch.equal(p_f[fin], p_c[fin])


@pytest.mark.parametrize("search", ["beam", "sample"])
def test_generate_items_wide_filters(search):
    """generate_items(num_beams=256) under exclude_history and under include_items returns only eligible items."""
    from rq_vae_recommender_b200.modules import model as M
    from test_gpu_exclusion import item_batch
    K, H, B = 256, 3, 6
    rs = np.random.RandomState(70)
    corpus = corpus_with_subtrees(rs, 3000, H, K)
    m = small_model(M, corpus, K, H)
    batch = item_batch(rs, corpus, B, 8, H)[0]
    out = m.generate_items(batch, search=search, num_beams=256, n=400, exclude_history=True)
    assert out.item_ids.shape == (B, 400) and out.sem_ids.shape == (B, 256, H)
    hist = m.history_items(batch).cpu().numpy()
    items = out.item_ids.cpu().numpy()
    for b in range(B):
        got = items[b][items[b] >= 0]
        assert len(got) > 0 and not set(got) & set(hist[b][hist[b] >= 0])
    allow = allow_lists(rs, corpus, B, 512)
    out = m.generate_items(batch, search=search, num_beams=256, include_items=dev(allow), exclude_history=False)
    items = out.item_ids.cpu().numpy()
    assert out.item_ids.shape == (B, 256)
    for b in range(B):
        got = items[b][items[b] >= 0]
        assert set(got) <= set(allow[b][allow[b] >= 0])


def test_exhaustive_wide_search_is_the_exact_ranking():
    """Every trie level has <= w nodes: the exhaustive search at width w drops no prefix and returns every leaf with a finite
    score in rank_sem_ids' order (log-probabilities within 1e-5, order free only among scores that close)."""
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, w = 256, 3, 5, 256
    rs = np.random.RandomState(80)
    corpus = np.unique(realistic_corpus(rs, 200, H, K), axis=0)
    m = small_model(M, corpus, K, H)
    mask, ids, users = history(rs, B, 6, H, K)
    prev = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("highest")
    try:
        g, p = m.generate(mask, ids, users, search="beam", num_beams=w)
        scores = m.rank_sem_ids(mask, ids, users).cpu().numpy()          # [B, U], the tuples in lexicographic order
    finally:
        torch.set_float32_matmul_precision(prev)
    g, p = g.cpu().numpy(), p.cpu().numpy()
    for b in range(B):
        order = np.argsort(-scores[b], kind="stable")
        ref_lp, ref_ids = scores[b][order], corpus[order]
        n = int(np.isfinite(ref_lp).sum())
        assert n > 0 and int(np.isfinite(p[b]).sum()) == n
        np.testing.assert_allclose(p[b][:n], ref_lp[:n], rtol=1e-5, atol=1e-5)
        assert {tuple(t) for t in g[b][:n].tolist()} == {tuple(t) for t in ref_ids[:n].tolist()}
        for j in range(n):
            near = np.abs(ref_lp[:n] - ref_lp[j]) <= 1e-5 + 1e-5 * abs(ref_lp[j])
            if near.sum() == 1:
                assert tuple(g[b][j]) == tuple(ref_ids[j])
