"""GPU tests of the fused sampling + selection kernel (csrc/sid.cu: sid_sample_select_kernel) and of the drop-in model's
generate: against the UNMODIFIED reference's run (tests/golden/beam.npz), against the device composition torch.multinomial +
log/gather + SidPrefixIndex.beam_select under the same CUDA seed, on rows torch.multinomial rejects, and at the argument
limits.  `pytest -m gpu`."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from parity import load_golden
from test_generate_oracle import beam_levels_from_seed

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("K", [16, 256, 2048])
@pytest.mark.parametrize("n", [1, 64])
@pytest.mark.parametrize("rows", [64, 6400])
def test_multinomial_is_exponential_race_cuda(K, n, rows):
    """The identity the kernel's parity rests on, on the installed torch's CUDA path (both topk code paths: 6400 rows of
    2048 take the multi-block one), with peaked rows whose softmax is 0 for most codes."""
    n = min(n, K)
    g = torch.Generator(device="cuda").manual_seed(K * n + rows)
    logits = torch.randn(rows, K, device="cuda", generator=g) * 4
    logits[::3] *= 40
    p = F.softmax(logits, dim=-1)
    torch.cuda.manual_seed(77)
    want = torch.multinomial(p, n, replacement=False)
    torch.cuda.manual_seed(77)
    got = torch.topk(p / torch.empty_like(p).exponential_(1), n).indices
    assert torch.equal(want, got)


def test_sample_select_vs_reference_fixture():
    """The reference run's logits (softmax on the device) and its seed-902 exponential draws: samples, beams and parents equal
    the reference's generate."""
    from rq_vae_recommender_b200 import ops
    g = load_golden("beam")
    B, k, H, K, N = (int(v) for v in g["shape"])
    nc = min(64, K)
    idx = ops.SidPrefixIndex(dev(g["corpus"]), K)
    generated, log_probas = None, None
    for h, _, noise in beam_levels_from_seed(g):
        probas = F.softmax(dev(g[f"logits{h}"]), dim=-1)
        generated, log_probas, parent, samples, _ = idx.sample_select(probas, dev(noise), generated, log_probas, k, nc,
                                                                       want_samples=True)
        assert np.array_equal(samples.cpu().numpy().reshape(-1), g[f"prefix{h}"][:, -1])
        if h > 0:
            assert np.array_equal(parent.cpu().numpy(), g[f"parent{h}"])
        if h + 1 < H:
            assert np.array_equal(generated.reshape(-1, h + 1).cpu().numpy(), g[f"future{h + 1}"])
    assert np.array_equal(generated.cpu().numpy(), g["generated"])
    np.testing.assert_allclose(log_probas.cpu().numpy(), g["log_probas"], rtol=2e-5, atol=1e-6)


def realistic_corpus(rs, N, C, K):
    corpus = rs.randint(0, K, size=(N, C)).astype(np.int64)
    if C == 4:
        corpus[:, 3] = rs.randint(0, 3, size=N)                               # the dedup column is small
    return corpus


def level_logits(rs, corpus, beams, rows, K):
    """Logits per beam row: random, a boost on tokens that continue the beam's prefix in the corpus, and every third row
    peaked so that its softmax is 0 for most codes (zero-probability ties, fewer than k finite candidates)."""
    logits = rs.randn(rows, K).astype(np.float32) * 2
    h = 0 if beams is None else beams.shape[1]
    if h == 0:
        logits[:, np.unique(corpus[:, 0])] += 3
    else:
        w = K ** np.arange(h - 1, -1, -1, dtype=np.int64)
        order = np.argsort((corpus[:, :h] * w).sum(1), kind="stable")
        ckeys = (corpus[order, :h] * w).sum(1)
        bkeys = (beams * w).sum(1)
        lo, hi = np.searchsorted(ckeys, bkeys, "left"), np.searchsorted(ckeys, bkeys, "right")
        for r in np.nonzero(hi > lo)[0]:
            logits[r, corpus[order[rs.randint(lo[r], hi[r], size=8)], h]] += 4
    logits[::3] *= 40
    return logits


def composition(idx, probas, generated, log_probas, k, nc):
    """The reference's sampling with the selection kernel (INTEGRATION.md §3 before the drop-in)."""
    samples = torch.multinomial(probas, nc)
    samp_log_p = torch.log(torch.gather(probas, 1, samples))
    return idx.beam_select(samples, samp_log_p, generated, log_probas, k) + (samples, samp_log_p)


@pytest.mark.parametrize("K,C", [(256, 3), (256, 4), (2048, 3)])
def test_sample_select_vs_device_composition_at_evaluation_sizes(K, C):
    from rq_vae_recommender_b200 import ops
    B, k, nc, N = 640, 10, 64, 12101
    rs = np.random.RandomState(K + C)
    corpus = realistic_corpus(rs, N, C, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    generated, log_probas = None, None
    n_zero_ties = n_short = 0
    for h in range(C):
        kp = 1 if h == 0 else k
        logits = level_logits(rs, corpus, None if h == 0 else generated.reshape(-1, h).cpu().numpy(), B * kp, K)
        probas = F.softmax(dev(logits), dim=-1)
        torch.cuda.manual_seed(1000 + h)
        g_c, p_c, par_c, s_c, l_c = composition(idx, probas, generated, log_probas, k, nc)
        torch.cuda.manual_seed(1000 + h)
        from rq_vae_recommender_b200.modules.model import draw_exponential
        g_f, p_f, par_f, s_f, l_f = idx.sample_select(probas, draw_exponential(probas), generated, log_probas, k, nc,
                                                      want_samples=True)
        assert torch.equal(s_f, s_c)
        assert torch.equal(l_f, l_c)
        n_zero_ties += int((l_c == -np.inf).sum(1).gt(1).sum())
        finite = torch.isfinite(p_c)
        n_short += int((finite.sum(1) < k).sum())
        assert torch.equal(torch.isfinite(p_f), finite)
        assert torch.equal(p_f[finite], p_c[finite])
        assert torch.equal(g_f[finite], g_c[finite])
        assert torch.equal(par_f.view(B, k)[finite], par_c.view(B, k)[finite])
        generated, log_probas = g_c, p_c
    assert n_zero_ties > 0 and n_short > 0


def test_rejected_rows_complete_and_are_counted():
    from rq_vae_recommender_b200 import ops
    B, K, k, nc = 12, 256, 10, 64
    rs = np.random.RandomState(3)
    corpus = realistic_corpus(rs, 5000, 3, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    probas = F.softmax(dev(rs.randn(B, K).astype(np.float32)), dim=-1)
    noise = torch.empty_like(probas).exponential_(1)
    bad = probas.clone()
    bad[1, 7] = float("nan")
    bad[2, 0] = -1e-3
    bad[4, 200] = float("inf")
    bad[5, 9] = -float("inf")
    bad[8] = 0.0
    reject = torch.zeros(2, dtype=torch.int32, device="cuda")
    out_bad = idx.sample_select(bad, noise, None, None, k, nc, want_samples=True, reject=reject)
    out_ok = idx.sample_select(probas, noise, None, None, k, nc, want_samples=True)
    torch.cuda.synchronize()
    assert reject.tolist() == [4, 1]
    keep = torch.tensor([r not in (1, 2, 4, 5, 8) for r in range(B)], device="cuda")
    for a, b in zip(out_bad, out_ok):
        rows = keep if a.shape[0] == B else keep.repeat_interleave(k)
        assert torch.equal(a[rows], b[rows])
    assert int(out_bad[3].min()) >= 0 and int(out_bad[3].max()) < K            # samples of rejected rows stay in range
    # reject accumulates over calls
    idx.sample_select(bad, noise, None, None, k, nc, reject=reject)
    assert reject.tolist() == [8, 2]


def small_model(M, corpus, K, H, k=10, seed=0):
    torch.manual_seed(seed)
    return M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), num_hierarchies=H, num_embeddings_per_hierarchy=K,
                                          t5_d_model=64, t5_num_heads=2, t5_d_ff=128, t5_num_layers=2, top_k_for_generation=k,
                                          should_add_sep_token=True, num_user_bins=11).cuda().eval()


def history(rs, B, items, H, K):
    ids = torch.from_numpy(rs.randint(0, K, size=(B, items * H))).cuda()
    mask = torch.ones_like(ids)
    mask[: B // 2, : H] = 0                                                   # some histories are padded
    return mask, ids, torch.from_numpy(rs.randint(0, 100, size=(B, 1))).cuda()


def test_generate_matches_composition_and_counts_launches():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M

    class Composed(M.EncoderDecoderRetrievalModel):
        def _sample_and_select(self, index, probas, generated, log_probas, k, n_cands, reject):
            return composition(index, probas, generated, log_probas, k, n_cands)[:3]

    K, H, B = 256, 3, 48
    rs = np.random.RandomState(11)
    corpus = realistic_corpus(rs, 3000, H, K)
    fused = small_model(M, corpus, K, H)
    composed = small_model(M, corpus, K, H, seed=1)
    composed.load_state_dict(fused.state_dict())
    mask, ids, users = history(rs, B, 20, H, K)
    before = ops.LAUNCHES
    torch.manual_seed(5)
    g_f, p_f = fused.generate(mask, ids, users)
    assert ops.LAUNCHES - before == 1 + H                                     # the index build, then one launch per level
    torch.manual_seed(5)
    g_c, p_c = composed.generate(mask, ids, users)
    assert g_f.shape == (B, 10, H)
    assert torch.equal(g_f, g_c) and torch.equal(p_f, p_c)
    before = ops.LAUNCHES
    torch.manual_seed(6)
    fused.generate(mask, ids, users)
    assert ops.LAUNCHES - before == H
    # load_state_dict writes a new corpus into the codebooks buffer: the index is rebuilt and the beams follow the new corpus
    sd = fused.state_dict()
    corpus2 = realistic_corpus(rs, 3000, H, K)
    corpus2[:, 0] = corpus2[:, 0] % 5
    sd["codebooks"] = torch.from_numpy(corpus2)
    fused.load_state_dict(sd)
    before = ops.LAUNCHES
    torch.manual_seed(5)
    g2, p2 = fused.generate(mask, ids, users)
    assert ops.LAUNCHES - before == 1 + H
    finite = torch.isfinite(p2)
    assert finite.any() and bool((g2[..., 0][finite] < 5).all())


def test_generate_raises_torch_multinomial_error():
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 8
    rs = np.random.RandomState(12)
    m = small_model(M, realistic_corpus(rs, 2000, H, K), K, H)
    with torch.no_grad():
        m.decoder_mlp[1].weight[3, 0] = float("nan")
    mask, ids, users = history(rs, B, 5, H, K)
    with pytest.raises(RuntimeError) as want:                                 # torch's text (its CUDA path asserts on the device)
        torch.multinomial(torch.full((2, K), float("nan")), 64)
    with pytest.raises(RuntimeError) as got:
        m.generate(mask, ids, users)
    assert str(got.value) == str(want.value)


def test_argument_limits_raise():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200._lib import Rqb200Error
    rs = np.random.RandomState(13)
    idx = ops.SidPrefixIndex(dev(realistic_corpus(rs, 500, 3, 256)), 256)
    B = 4
    p = F.softmax(dev(rs.randn(B * 32, 256).astype(np.float32)), dim=-1)
    q = torch.empty_like(p).exponential_(1)
    gen = torch.zeros((B, 32, 1), dtype=torch.int64, device="cuda")
    lp = torch.zeros((B, 32), device="cuda")
    with pytest.raises(Rqb200Error, match="kp \\* nc"):
        idx.sample_select(p, q, gen, lp, 10, 64)                              # kp * nc = 2048
    with pytest.raises(Rqb200Error, match="k = 33"):
        idx.sample_select(p[:B], q[:B], None, None, 33, 64)
    small = ops.SidPrefixIndex(dev(realistic_corpus(rs, 500, 3, 16)), 16)
    p16 = F.softmax(dev(rs.randn(B, 16).astype(np.float32)), dim=-1)
    with pytest.raises(Rqb200Error, match="nc = 17"):
        small.sample_select(p16, torch.empty_like(p16).exponential_(1), None, None, 4, 17)
    big = ops.SidPrefixIndex(dev(rs.randint(0, 4096, size=(500, 2)).astype(np.int64)), 4096)
    p4k = F.softmax(dev(rs.randn(B, 4096).astype(np.float32)), dim=-1)
    with pytest.raises(Rqb200Error, match="K = 4096"):
        big.sample_select(p4k, torch.empty_like(p4k).exponential_(1), None, None, 10, 64)
    from rq_vae_recommender_b200.modules import model as M
    m = small_model(M, realistic_corpus(rs, 500, 3, 256), 256, 3, k=20)          # 20 beams x 64 candidates > 1024
    mask, ids, users = history(rs, 2, 3, 3, 256)
    with pytest.raises(Rqb200Error, match="top_k_for_generation"):
        m.generate(mask, ids, users)
