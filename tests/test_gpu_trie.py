"""GPU tests of the corpus trie index (csrc/sid.cu: rqb200_sid_trie_*, ops.SidPrefixIndex): check against
oracle.rq_oracle.check_valid_prefix up to K^C = 2^88, the three searches against their oracles and against each other (the
sampled search's child masks against beam_select's walk), the sampled and exhaustive searches at K^C above 2^33, and the
drop-in model at five hierarchy levels.  `pytest -m gpu`."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import trie_oracle as T
from oracle import rq_oracle as O
import beam_search_oracle as BO
import sample_oracle as SO
from test_gpu_beam_search import TOL, assert_matches, oracle_level, torch_level
from test_gpu_generate import composition, dev, history, level_logits, realistic_corpus, small_model
from test_trie_oracle import prefixes, random_corpus

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("K,C", [(16, 8), (256, 5), (512, 4), (2048, 4), (2048, 8)])
def test_check_matches_check_valid_prefix(K, C):
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K + C)
    corpus = random_corpus(rs, 2000, C, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    for l in range(1, C + 1):
        p = prefixes(rs, corpus, l, K, n=1000)
        want = T.valid_prefixes(corpus, p, K)
        assert want.any() and not want.all()
        assert np.array_equal(idx.check(dev(p)).cpu().numpy(), want), l
        strided = dev(np.concatenate([p, p[:, :1]], axis=1))[:, :l]             # a row stride above l
        assert np.array_equal(idx.check(strided).cpu().numpy(), want), l


@pytest.mark.parametrize("N", [0, 1, 2])
def test_check_on_tiny_corpora(N):
    from rq_vae_recommender_b200 import ops
    K, C = 256, 5
    corpus = np.array([[1, 2, 3, 4, 5], [1, 2, 300, 4, 5]], dtype=np.int64)[:N]
    idx = ops.SidPrefixIndex(dev(corpus.reshape(N, C)), K)
    rs = np.random.RandomState(N)
    for l in range(1, C + 1):
        p = np.concatenate([np.array([[1, 2, 3, 4, 5], [1, 2, 300, 4, 5]])[:, :l], rs.randint(0, 4, size=(50, l))])
        assert np.array_equal(idx.check(dev(p)).cpu().numpy(), T.valid_prefixes(corpus.reshape(N, C), p, K)), l


def same(a, b):
    """bit-identical tensors (a NaN equals the same NaN)"""
    bits = lambda t: t.view(torch.int32) if t.dtype == torch.float32 else t
    return all(torch.equal(bits(u), bits(v)) for u, v in zip(a, b))


CASES = [(B, k, K) for B in (1, 7, 640) for k in (1, 10, 32) for K in (16, 256, 2048) if k <= K]


@pytest.mark.parametrize("B,k,K", CASES)
def test_searches_agree_with_oracles_and_each_other(B, k, K):
    """Three levels of each search on one corpus, each level fed the search's own beams.  Logit rows with NaN, all -inf, and
    probability rows with a NaN or a zero sum are mixed in; at k = 32, K = 2048 beam_topk recomputes its keys (65 536
    candidates).  sample_select (its candidates tested against a K-bit child mask per beam) is bit-identical to beam_select
    (a binary search per candidate) over its own samples, which are sample_oracle's; check of every extension is
    trie_oracle's; beam_topk matches beam_search_oracle and returns as many finite beams as there are valid finite
    extensions, up to k.  The reject and bad counts are numpy's."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(B * 7 + k * 131 + K)
    C = 3
    corpus = realistic_corpus(rs, 3000 if K == 16 else 12101, C, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    nc = min(64, K, 1024 // k)
    n = lambda t: None if t is None else t.cpu().numpy()
    gen_b = gen_s = lp_b = lp_s = None
    for h in range(C):
        kp = 1 if h == 0 else k
        beams = None if h == 0 else n(gen_b).reshape(-1, h)
        logits = dev(np.clip(level_logits(rs, corpus, beams, B * kp, K), -60, 60))    # clipped as in test_beam_topk_vs_oracle
        if B * kp > 3:
            logits[1, 5] = float("nan")
            logits[2] = -float("inf")
        bad = torch.zeros(1, dtype=torch.int32, device="cuda")
        out = idx.beam_topk(logits, gen_b, lp_b, k, bad=bad)
        x = n(logits)
        assert int(bad) == int((np.isnan(x).any(1) | np.isposinf(x).any(1) | np.isneginf(x).all(1)).sum())
        ref = oracle_level(corpus, logits, gen_b, lp_b, k)
        assert_matches(*ref, out, k)
        finite = np.isfinite(n(out[1]))
        assert np.array_equal(finite.sum(1), np.minimum(k, np.isfinite(ref[3]).sum(1)))
        assert T.valid_prefixes(corpus, n(out[0])[finite], K).all()

        probas = F.softmax(logits.nan_to_num(0.0), dim=-1)
        if B * kp > 3:
            probas[3] = 0.0
            probas[1, 2] = float("nan")
        noise = torch.empty_like(probas).exponential_(1)
        reject = torch.zeros(2, dtype=torch.int32, device="cuda")
        samp = idx.sample_select(probas, noise, gen_s, lp_s, k, nc, want_samples=True, reject=reject)
        p = n(probas)
        bad_rows = ~(p >= 0).all(1) | np.isinf(p).any(1)
        assert n(reject).tolist() == [int(bad_rows.sum()), int((~bad_rows & (p == 0).all(1)).sum())]
        assert np.array_equal(n(samp[3]), SO.sample_select(corpus, p, n(noise), n(gen_s), n(lp_s), k, nc)[3])
        assert same(samp[:3], idx.beam_select(samp[3], samp[4], gen_s, lp_s, k))
        ext = samp[3].reshape(-1, 1) if h == 0 else torch.cat([gen_s.reshape(-1, h).repeat_interleave(nc, 0),
                                                                samp[3].reshape(-1, 1)], 1)
        assert np.array_equal(n(idx.check(ext)), T.valid_prefixes(corpus, n(ext), K))
        gen_b, lp_b = out[0], out[1]
        gen_s, lp_s = samp[0], samp[1]


def test_sparse_corpus_fillers_in_oracle_order():
    """Fewer valid extensions than k on all three levels: the valid ones first, then the -inf fillers in ascending flat index
    (beam * K + code) with their parents and ids, exactly as beam_search_oracle has them."""
    from rq_vae_recommender_b200 import ops
    K, k, B = 256, 10, 6
    corpus = np.array([[5, 1, 0], [5, 2, 0], [200, 7, 1]], dtype=np.int64)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    rs = np.random.RandomState(22)
    g = lp = None
    for h in range(3):
        logits = rs.randn(B * (1 if h == 0 else k), K).astype(np.float32)
        out = idx.beam_topk(dev(logits), g, lp, k)
        og, op, opar = BO.beam_topk(corpus, logits, None if g is None else g.cpu().numpy(),
                                    None if lp is None else lp.cpu().numpy(), k)
        assert np.isneginf(op[:, -1]).all()
        assert np.array_equal(out[0].cpu().numpy(), og) and np.array_equal(out[2].cpu().numpy().reshape(B, k), opar)
        np.testing.assert_allclose(out[1].cpu().numpy(), op, rtol=TOL, atol=TOL)
        g, lp = out[0], out[1]


def test_sample_select_five_levels_vs_oracle():
    """K = 256, C = 5 (a 2^40-bit key space): per level the samples are torch.multinomial's under the same seed, and the
    selection is sample_oracle's (oracle.rq_oracle.beam_select over the samples and their log-probabilities)."""
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules.model import draw_exponential
    K, C, B, k, nc = 256, 5, 24, 10, 64
    rs = np.random.RandomState(31)
    corpus = realistic_corpus(rs, 3000, C, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    generated = log_probas = None
    n_valid = 0
    for h in range(C):
        kp = 1 if h == 0 else k
        logits = level_logits(rs, corpus, None if h == 0 else generated.reshape(-1, h).cpu().numpy(), B * kp, K)
        probas = F.softmax(dev(logits), dim=-1)
        torch.cuda.manual_seed(2000 + h)
        want = torch.multinomial(probas, nc)
        torch.cuda.manual_seed(2000 + h)
        noise = draw_exponential(probas)
        g, p, par, samples, samp_log_p = idx.sample_select(probas, noise, generated, log_probas, k, nc, want_samples=True)
        assert torch.equal(samples, want)
        assert torch.equal(samp_log_p, torch.log(torch.gather(probas, 1, want)))
        n = lambda t: None if t is None else t.cpu().numpy()
        o_samples = SO.sample_select(corpus, n(probas), n(noise), n(generated), n(log_probas), k, nc)[3]
        assert np.array_equal(o_samples, n(samples))
        og, op, opar = O.beam_select(corpus, n(samples), n(samp_log_p), n(generated), n(log_probas), k)
        assert np.array_equal(n(g), og) and np.array_equal(n(p), op)
        assert np.array_equal(n(par).reshape(B, k), opar)
        n_valid += int(np.isfinite(op).sum())
        generated, log_probas = g, p
    assert n_valid > 0


def test_beam_topk_65536_candidates_four_levels_vs_oracle():
    """K = 2048, k = 32, C = 4 (2^44 keys): all four levels against beam_search_oracle, 65 536 candidates per history."""
    from rq_vae_recommender_b200 import ops
    K, C, B, k = 2048, 4, 7, 32
    rs = np.random.RandomState(32)
    corpus = realistic_corpus(rs, 12101, C, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    generated, log_probas = None, None
    for h in range(C):
        kp = 1 if h == 0 else k
        logits = dev(np.clip(level_logits(rs, corpus, None if h == 0 else generated.reshape(-1, h).cpu().numpy(), B * kp, K),
                             -60, 60))
        got = idx.beam_topk(logits, generated, log_probas, k)
        assert_matches(*oracle_level(corpus, logits, generated, log_probas, k), got, k)
        generated, log_probas = got[0], got[1]


def test_generate_five_levels_sample_and_beam():
    """The drop-in model at five hierarchy levels (K = 256, 2^40 keys): one build then one launch per level, deterministic,
    the exhaustive search leaves the CUDA RNG state alone and agrees with the torch composition on hook-recorded logits, the
    sampled search equals torch.multinomial + beam_select under the same seed, and load_state_dict rebuilds the index."""
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, k = 256, 5, 32, 10
    rs = np.random.RandomState(33)
    corpus = realistic_corpus(rs, 3000, H, K)
    m = small_model(M, corpus, K, H, k=k)
    mask, ids, users = history(rs, B, 10, H, K)
    before = ops.LAUNCHES
    torch.manual_seed(1)
    rng = torch.cuda.get_rng_state()
    g1, p1 = m.generate(mask, ids, users, search="beam")
    assert ops.LAUNCHES - before == 1 + H
    assert torch.equal(torch.cuda.get_rng_state(), rng)
    assert g1.shape == (B, k, H) and bool(torch.isfinite(p1).all())
    assert bool(torch.from_numpy(T.valid_prefixes(corpus, g1.reshape(-1, H).cpu().numpy(), K)).all())
    before = ops.LAUNCHES
    g2, p2 = m.generate(mask, ids, users, search="beam")
    assert ops.LAUNCHES - before == H and torch.equal(g1, g2) and torch.equal(p1, p2)
    logits, levels = [], []
    hooks = [mlp.register_forward_hook(lambda mod, inp, out: logits.append(out.detach().clone())) for mlp in m.decoder_mlp]
    index = m._prefix_index(ids.device)                                      # the cached index (ids are on the model's device)

    class Recording:
        def beam_topk(self, lg, generated, log_probas, k, bad=None):
            out = index.beam_topk(lg, generated, log_probas, k, bad=bad)
            levels.append((generated, log_probas, out))
            return out

    m._prefix_index = lambda device: Recording()
    try:
        g3, _ = m.generate(mask, ids, users, search="beam")
    finally:
        for hk in hooks:
            hk.remove()
        del m._prefix_index
    assert torch.equal(g3, g1) and len(logits) == H
    for lg, (generated, log_probas, out) in zip(logits, levels):
        ref_g, ref_p, ref_par, scores = (t.cpu().numpy() for t in torch_level(index, lg, generated, log_probas, k))
        assert_matches(ref_g, ref_p, ref_par, scores, out, k, exact_ties=False, min_checked=0.9)

    class Composed(M.EncoderDecoderRetrievalModel):
        def _sample_and_select(self, index, probas, generated, log_probas, k, n_cands, reject):
            return composition(index, probas, generated, log_probas, k, n_cands)[:3]

    composed = small_model(M, corpus, K, H, k=k, seed=1)
    composed.__class__ = Composed
    composed.load_state_dict(m.state_dict())
    before = ops.LAUNCHES
    torch.manual_seed(5)
    g_f, p_f = m.generate(mask, ids, users, search="sample")
    assert ops.LAUNCHES - before == H
    torch.manual_seed(5)
    g_c, p_c = composed.generate(mask, ids, users, search="sample")
    assert torch.equal(g_f, g_c) and torch.equal(p_f, p_c)
    torch.manual_seed(5)
    g_f2, p_f2 = m.generate(mask, ids, users, search="sample")
    assert torch.equal(g_f, g_f2) and torch.equal(p_f, p_f2)
    sd = m.state_dict()
    corpus2 = realistic_corpus(rs, 3000, H, K)
    corpus2[:, 0] = corpus2[:, 0] % 5
    sd["codebooks"] = torch.from_numpy(corpus2)
    m.load_state_dict(sd)
    for search in ("beam", "sample"):
        before = ops.LAUNCHES
        g4, p4 = m.generate(mask, ids, users, search=search)
        assert ops.LAUNCHES - before == (1 if search == "beam" else 0) + H
        finite = torch.isfinite(p4)
        assert finite.any() and bool((g4[..., 0][finite] < 5).all())
