"""GPU tests of the warped sampled search: SidPrefixIndex.sample_select_warped[_wide] against the float64 oracle
(warp_sample_oracle) at every filter mode, the level-0 scores against search="beam" bit for bit, cluster-size independence, the
default controls against the untempered path, a chi-square check of the first draw, bad rows, graph replays and both decoders.
`pytest -m gpu`."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import exclusion_oracle as X
import warp_sample_oracle as WO
from test_gpu_exclusion import built as built_exclusion, corpus_with_subtrees, exclusion_sets
from test_gpu_generate import dev, level_logits, realistic_corpus, small_model
from test_gpu_generate_graph import assert_same, batch_of, eager, highest, replay
from test_gpu_inclusion import allow_lists, built as built_inclusion
import inclusion_oracle as I

pytestmark = pytest.mark.gpu

NC = 64
# Closeness of two ratios (relative), of a nucleus mass to its target (absolute, of a total 1) or of t to the next p_T
# (relative) within which the kernel's fp32 p_T (a few 1e-7 relative, plus the row's exponent rounding) may decide otherwise
TOL = 5e-6
H3 = 3


def _filter(kind, corpus, K, B, rs):
    """(kwargs of the kernel call, valid(b, prefix) of the oracle) of a filter mode."""
    prefixes = {tuple(r[:l]) for r in corpus.tolist() for l in range(1, corpus.shape[1] + 1)}
    if kind == "none":
        return {}, lambda b, prefix: tuple(prefix) in prefixes
    if kind == "exclude":
        items = exclusion_sets(rs, corpus, B, 64)
        _, ref, ex = built_exclusion(corpus, K, items)
        excls = X.build(ref, items)
        return {"exclude": ex}, lambda b, prefix: tuple(prefix) in prefixes and not X.is_blocked(excls[b], prefix, K)
    _, _, inc, incls = built_inclusion(corpus, K, allow_lists(rs, corpus, B, 256))
    return {"include": inc}, lambda b, prefix: I.valid_prefix(incls[b], prefix, K)


def _select(idx, kp, k, wide):
    if wide or not (k <= 32 and kp * NC <= 1024):
        return idx.sample_select_warped_wide
    return idx.sample_select_warped


def _check_level(idx, corpus, logits, generated, log_probas, k, T, top_p, filt, valid, wide=False):
    """One level against the oracle: draws equal outside ambiguous rows, model log-probabilities to 1e-6 of the row's scale,
    and the kept beams exactly the oracle's selection from the kernel's own fp32 draws.  Returns (out, ambiguous rows)."""
    B = logits.shape[0] if generated is None else generated.shape[0]
    kp = logits.shape[0] // B
    noise = torch.empty_like(logits).exponential_(1)
    bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = _select(idx, kp, k, wide)(logits, noise, generated, log_probas, k, NC, T, top_p, want_samples=True, bad=bad, **filt)
    g, p, par, s, lp = (t.cpu().numpy() for t in out)
    x = logits.cpu().numpy()
    os_, olp, amb, obad = WO.warped_level(x, noise.cpu().numpy(), T, top_p, NC, tol=TOL)
    assert int(bad) == int(obad.sum())
    ok = ~amb
    assert np.array_equal(s[ok], os_[ok])
    assert np.array_equal(np.isfinite(lp[ok]), np.isfinite(olp[ok]))
    scale = np.broadcast_to(np.maximum(1.0, np.abs(x).max(1))[:, None], lp.shape)
    fin = np.isfinite(olp) & ok[:, None]
    assert (np.abs(lp[fin] - olp[fin]) <= 1e-6 * scale[fin]).all()
    gen_in = None if generated is None else generated.cpu().numpy()
    lp_in = None if log_probas is None else log_probas.cpu().numpy()
    og, op, opar = WO.keep_best(s, lp, gen_in, lp_in, k, valid, dtype=np.float32)
    assert np.array_equal(p, op) and np.array_equal(g, og) and np.array_equal(par.reshape(B, k), opar)
    return out, int(amb.sum())


@pytest.mark.parametrize("K,kp,k", [(256, 1, 10), (300, 10, 10), (2048, 10, 10), (256, 32, 32), (300, 64, 64),
                                    (2048, 64, 100), (256, 1024, 256)])
@pytest.mark.parametrize("T,top_p", [(0.25, 0.9), (0.7, 0.05), (1.0, 0.9), (3.0, 1.0), (0.7, 1.0)])
def test_warped_level_vs_oracle(K, kp, k, T, top_p):
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K + kp + int(T * 100) + int(top_p * 100))
    corpus = realistic_corpus(rs, 12101, H3, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    B = 3
    filt, valid = _filter("none", corpus, K, B, rs)
    if kp == 1:
        generated, log_probas = None, None
    else:
        generated = dev(corpus[rs.randint(0, len(corpus), size=B * kp), :1].reshape(B, kp, 1))
        log_probas = dev(-np.abs(rs.randn(B, kp)).astype(np.float32))
    beams = None if generated is None else generated.reshape(-1, 1).cpu().numpy()
    logits = dev(np.clip(level_logits(rs, corpus, beams, B * kp, K), -60, 60))
    _, n_amb = _check_level(idx, corpus, logits, generated, log_probas, k, T, top_p, filt, valid)
    print(f"K={K} kp={kp} T={T} top_p={top_p}: {n_amb} of {B * kp} rows within {TOL} of a tie, not compared")
    assert n_amb <= max(4, 0.05 * B * kp)


@pytest.mark.parametrize("kind", ["none", "exclude", "include"])
@pytest.mark.parametrize("w", [1, 10, 64])
def test_filters_and_per_level_values(kind, w):
    """Three levels, each at its own (T, top_p), with each filter mode: every level against the oracle, fed the kernel's beams."""
    from rq_vae_recommender_b200 import ops
    K, B = 256, 6
    rs = np.random.RandomState(w + len(kind))
    corpus = corpus_with_subtrees(rs, 6000, H3, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    filt, valid = _filter(kind, corpus, K, B, rs)
    controls = [(0.5, 0.9), (2.0, 0.05), (1.0, 0.7)]
    generated, log_probas, n_amb, rows = None, None, 0, 0
    for h, (T, top_p) in enumerate(controls):
        beams = None if h == 0 else generated.reshape(-1, h).cpu().numpy()
        logits = dev(np.clip(level_logits(rs, corpus, beams, B * (1 if h == 0 else w), K), -60, 60))
        out, a = _check_level(idx, corpus, logits, generated, log_probas, w, T, top_p, filt, valid)
        n_amb, rows = n_amb + a, rows + logits.shape[0]
        generated, log_probas = out[0], out[1]
    print(f"{kind} w={w}: {n_amb} of {rows} rows within {TOL} of a tie, not compared")
    assert n_amb <= max(4, 0.05 * rows)


def test_level0_scores_are_the_beam_searchs():
    """A level-0 candidate scores bit for bit what search="beam" gives the same code (beam_topk_wide ranks every code)."""
    from rq_vae_recommender_b200 import ops
    K, B = 256, 8
    rs = np.random.RandomState(4)
    corpus = np.stack([np.arange(K), rs.randint(0, K, K), rs.randint(0, K, K)], 1).astype(np.int64)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    logits = dev((rs.randn(B, K) * 3).astype(np.float32))
    g, p, _ = idx.beam_topk_wide(logits, None, None, K)
    beam = torch.full((B, K), float("nan"), device="cuda").scatter_(1, g[:, :, 0], p)
    for T, top_p in [(0.5, 1.0), (2.0, 0.9), (1.0, 0.3)]:
        noise = torch.empty_like(logits).exponential_(1)
        s, lp = idx.sample_select_warped(logits, noise, None, None, 10, NC, T, top_p, want_samples=True)[3:]
        drawn = torch.isfinite(lp)
        assert drawn.any(1).all()
        assert torch.equal(lp[drawn], beam.gather(1, s)[drawn])


@pytest.mark.parametrize("kind", ["none", "exclude", "include"])
def test_cluster_size_does_not_matter_and_narrow_equals_wide(kind):
    from rq_vae_recommender_b200 import ops
    K, B = 256, 4
    rs = np.random.RandomState(9 + len(kind))
    corpus = corpus_with_subtrees(rs, 12101, H3, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    filt, _ = _filter(kind, corpus, K, B, rs)
    kp, k = 1024, 256
    generated = dev(corpus[rs.randint(0, len(corpus), size=B * kp), :1].reshape(B, kp, 1))
    log_probas = dev(-np.abs(rs.randn(B, kp)).astype(np.float32))
    logits = dev(np.clip(level_logits(rs, corpus, generated.reshape(-1, 1).cpu().numpy(), B * kp, K), -60, 60))
    noise = torch.empty_like(logits).exponential_(1)
    run = lambda c: idx.sample_select_warped_wide(logits, noise, generated, log_probas, k, NC, 0.7, 0.9, want_samples=True,
                                                  cluster=c, **filt)
    ref = run(1)
    for c in (2, 4, 8, 0):
        assert all(torch.equal(a, b) for a, b in zip(run(c), ref)), c
    for k in (1, 10, 16):                                       # both kernels run kp * 64 <= 1024
        kp = k
        g = dev(corpus[rs.randint(0, len(corpus), size=B * kp), :1].reshape(B, kp, 1))
        lp = dev(-np.abs(rs.randn(B, kp)).astype(np.float32))
        lg = dev(level_logits(rs, corpus, g.reshape(-1, 1).cpu().numpy(), B * kp, K))
        q = torch.empty_like(lg).exponential_(1)
        a = idx.sample_select_warped(lg, q, g, lp, k, NC, 1.3, 0.8, want_samples=True, **filt)
        b = idx.sample_select_warped_wide(lg, q, g, lp, k, NC, 1.3, 0.8, want_samples=True, **filt)
        assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_first_draw_follows_the_tempered_nucleus():
    """Seeded chi-square: over 40 000 rows of the same logits, the first draw's codes follow p_T restricted to N."""
    from scipy import stats
    from rq_vae_recommender_b200 import ops
    K, R, T, top_p = 32, 40000, 0.7, 0.8
    corpus = np.stack([np.arange(K), np.zeros(K, dtype=np.int64)], 1)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    torch.manual_seed(0)
    x = torch.randn(K, device="cuda") * 1.5
    logits = x.expand(R, K).contiguous()
    noise = torch.empty_like(logits).exponential_(1)
    s = idx.sample_select_warped(logits, noise, None, None, 1, NC // 2, T, top_p, want_samples=True)[3]
    p = WO.tempered(x.cpu().numpy()[None].astype(np.float64), T)[0]
    N, _ = WO.nucleus(p, top_p)
    want = np.where(N, p, 0) / p[N].sum()
    got = np.bincount(s[:, 0].cpu().numpy(), minlength=K)
    assert got[~N].sum() == 0 and 1 < N.sum() < K
    chi = stats.chisquare(got[N], want[N] * R)
    assert chi.pvalue > 1e-4, chi


# ------------------------------------------------------------------------------------------------------------------ model
@pytest.fixture(scope="module")
def corpus():
    return realistic_corpus(np.random.RandomState(12101), 12101, H3, 256)


@pytest.fixture(scope="module")
def model(corpus):
    from rq_vae_recommender_b200.modules import model as M
    return small_model(M, corpus, 256, H3)


@pytest.mark.parametrize("w", [None, 64])
def test_default_controls_are_the_untempered_search(model, corpus, w):
    """T = 1, top_p = 1 (floats or per level): the call without the arguments, bit for bit, with the same generator state."""
    from rq_vae_recommender_b200 import ops
    batch = batch_of(np.random.RandomState(1), corpus, 16)
    model.generate_items(batch, num_beams=w, decoder="fused", encoder="fused")   # the corpus caches' first-use builds
    outs, states, launches = [], [], []
    for kw in ({}, dict(temperature=1.0, top_p=1.0), dict(temperature=[1, 1, 1], top_p=(1.0, 1.0, 1.0))):
        torch.manual_seed(3)
        before = ops.LAUNCHES
        outs.append(model.generate_items(batch, num_beams=w, decoder="fused", encoder="fused", **kw))
        launches.append(ops.LAUNCHES - before)
        states.append(torch.cuda.get_rng_state())
    for o, st in zip(outs[1:], states[1:]):
        assert_same(o, outs[0])
        assert torch.equal(st, states[0])
    assert launches[1] == launches[0] == launches[2]


def test_warped_search_consumes_the_generator_as_the_untempered_one(model, corpus):
    batch = batch_of(np.random.RandomState(2), corpus, 8)
    torch.manual_seed(5)
    model.generate_items(batch, decoder="fused", encoder="fused")
    plain = torch.cuda.get_rng_state()
    torch.manual_seed(5)
    model.generate_items(batch, decoder="fused", encoder="fused", temperature=0.6, top_p=0.9)
    assert torch.equal(torch.cuda.get_rng_state(), plain)


def test_bad_head_rows_raise_after_the_search(model, corpus):
    from rq_vae_recommender_b200 import ops
    batch = batch_of(np.random.RandomState(3), corpus, 4)
    w = model.decoder_mlp[1].weight
    saved = w.detach().clone()
    try:
        with torch.no_grad():
            w[7, 0] = float("nan")
        with pytest.raises(RuntimeError, match=r"generate: \d+ beam row\(s\) of the decoder head's logits hold a NaN"):
            model.generate_items(batch, decoder="fused", encoder="fused", temperature=0.5)
    finally:
        with torch.no_grad():
            w.copy_(saved)


@pytest.mark.parametrize("w", [10, 64])
@pytest.mark.parametrize("side", [False, True])
def test_graph_replay_equals_eager(model, corpus, w, side):
    rs = np.random.RandomState(w)
    batch = batch_of(rs, corpus, 16, padded=False)
    kw = dict(temperature=[0.5, 1.0, 2.0], top_p=0.9, num_beams=w)
    stream = torch.cuda.Stream() if side else torch.cuda.current_stream()
    with torch.cuda.stream(stream):
        g = model.capture_generate_items(batch, **kw)
        for seed in (1, 2):
            assert_same(replay(g, batch, seed), eager(model, batch, seed, **kw))
    torch.cuda.synchronize()


@pytest.mark.parametrize("w", [10, 64])
def test_decoders_agree(model, corpus, w):
    """The HF and fused decoders give the same beams under "highest" precision, with each level's own controls."""
    batch = batch_of(np.random.RandomState(7 + w), corpus, 8)
    kw = dict(temperature=[0.7, 1.5, 1.0], top_p=[0.9, 1.0, 0.5], num_beams=w, encoder="fused")
    with highest():
        torch.manual_seed(9)
        a = model.generate_next_sem_id(batch, decoder="hf", **kw)
        torch.manual_seed(9)
        b = model.generate_next_sem_id(batch, decoder="fused", **kw)
    assert torch.equal(a.sem_ids, b.sem_ids)
    fin = torch.isfinite(b.log_probas)
    assert torch.equal(torch.isfinite(a.log_probas), fin)
    torch.testing.assert_close(a.log_probas[fin], b.log_probas[fin], rtol=0, atol=1e-5)


def test_deterministic_searches_ignore_generate_next_sem_id_temperature(model, corpus):
    batch = batch_of(np.random.RandomState(11), corpus, 4)
    a = model.generate_next_sem_id(batch, search="beam", temperature=0.3, decoder="fused", encoder="fused")
    b = model.generate_next_sem_id(batch, search="beam", decoder="fused", encoder="fused")
    assert torch.equal(a.sem_ids, b.sem_ids) and torch.equal(a.log_probas, b.log_probas)
