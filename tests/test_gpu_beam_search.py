"""GPU tests of the exhaustive beam-search kernel (csrc/sid.cu: sid_beam_topk_kernel, ops.SidPrefixIndex.beam_topk) against the
numpy oracle beam_search_oracle.beam_topk, on exact ties, sparse corpora and bad rows, and of the drop-in model's
generate(search="beam") against a torch composition.  `pytest -m gpu`."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import beam_search_oracle as BO
from test_gpu_generate import dev, history, level_logits, realistic_corpus, small_model

pytestmark = pytest.mark.gpu

TOL = 1e-5


def assert_matches(ref_g, ref_p, ref_par, scores, got, k, exact_ties=True, min_checked=0.5):
    """ref_*: a reference's k + 1 best (k when there is no (k + 1)-th candidate), parents global [B, k(+1)]; scores: its score of
    every candidate [B, E]; got: the kernel's (generated, log_probas, parent_global).  Log-probabilities within
    rtol = atol = TOL everywhere.  The gap rule: on rows where no candidate scores within the tolerance of the k-th score the
    kept set is the reference's, and there every position whose score is farther than the tolerance from each other kept
    score holds the reference's beam and parent.  Equal scores count as apart: -inf fillers always, other equal scores when
    ``exact_ties`` (a float64 reference: equal only for the same logit of the same row and parent, which ties in fp32 too)."""
    g, p, par = (t.cpu().numpy() for t in got)
    B = g.shape[0]
    par = par.reshape(B, k)
    np.testing.assert_allclose(p, ref_p[:, :k], rtol=TOL, atol=TOL)
    same = (lambda a, b: a == b) if exact_ties else (lambda a, b: np.isneginf(a) & np.isneginf(b))

    def near(a, b):                                           # |a - b| within the tolerance, not an exact tie
        with np.errstate(invalid="ignore"):
            return (np.abs(a - b) <= TOL + TOL * np.abs(np.where(np.isfinite(b), b, 0))) & ~same(a, b)

    sk = ref_p[:, k - 1:k]
    rows = near(scores, sk).sum(1) <= (0 if exact_ties else 1)                   # (not exact_ties: the k-th itself)
    assert rows.mean() >= min_checked, rows.mean()
    v = ref_p[:, :k]
    alone = ~(near(v[:, None, :], v[:, :, None]) & ~np.eye(k, dtype=bool)).any(2)       # [B, k]: apart from the other kept
    for b in np.nonzero(rows)[0]:
        want = {(int(ref_par[b, j]),) + tuple(ref_g[b, j].tolist()) for j in range(k)}
        have = {(int(par[b, j]),) + tuple(g[b, j].tolist()) for j in range(k)}
        assert have == want, b
        for j in np.nonzero(alone[b])[0]:
            assert par[b, j] == ref_par[b, j] and np.array_equal(g[b, j], ref_g[b, j]), (b, j)


def oracle_level(corpus, logits, generated, log_probas, k):
    """The oracle's k + 1 best (k when the history has only k candidates) and every candidate's score, inputs as the kernel
    got them."""
    n = lambda t: None if t is None else t.cpu().numpy()
    E = logits.shape[1] * (1 if generated is None else generated.shape[1])
    return BO.beam_topk(corpus, n(logits), n(generated), n(log_probas), min(k + 1, E)) + (
        BO.candidate_scores(corpus, n(logits), n(generated), n(log_probas)),)


CASES = [(B, k, K) for B in (1, 7, 640) for k in (1, 10, 32) for K in (16, 256, 2048) if k <= K]


@pytest.mark.parametrize("B,k,K", CASES)
def test_beam_topk_vs_oracle(B, k, K):
    """Three levels (h = 0, 1, 2), each fed the kernel's beams of the level before.  At k = 32, K = 2048 a history has
    E = 65 536 candidates, more than the kernel keeps in shared memory: its keys are recomputed on every pass.
    The fp32 log-sum-exp is off by up to half an ulp of the row maximum (1.5e-5 at 400), so the logits of level_logits'
    peaked rows are clipped to +-60 for the 1e-5 tolerance; clipped codes tie exactly."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(B * 7 + k * 131 + K)
    corpus = realistic_corpus(rs, 3000 if K == 16 else 12101, 3, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    generated, log_probas = None, None
    for h in range(3):
        kp = 1 if h == 0 else k
        logits = dev(np.clip(level_logits(rs, corpus, None if h == 0 else generated.reshape(-1, h).cpu().numpy(), B * kp, K),
                             -60, 60))
        got = idx.beam_topk(logits, generated, log_probas, k)
        assert got[0].shape == (B, k, h + 1) and got[1].shape == (B, k) and got[2].shape == (B * k,)
        assert_matches(*oracle_level(corpus, logits, generated, log_probas, k), got, k)
        again = idx.beam_topk(logits, generated, log_probas, k)
        assert all(torch.equal(a, b) for a, b in zip(got, again))
        generated, log_probas = got[0], got[1]


def test_exact_ties_lowest_flat_index_first():
    """Duplicated logits inside a row, and beams with identical ids, log-probabilities and logits rows: the kernel keeps equal
    scores in ascending flat index (beam * K + code), exactly as the oracle's stable sort, with bit-identical scores."""
    from rq_vae_recommender_b200 import ops
    K, C, B, kp = 16, 2, 5, 4
    corpus = np.stack(np.meshgrid(np.arange(K), np.arange(K), indexing="ij"), -1).reshape(-1, C).astype(np.int64)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    rs = np.random.RandomState(21)
    logits0 = rs.randint(0, 3, size=(B, K)).astype(np.float32)
    for k in (10, 16):
        g, p, par = idx.beam_topk(dev(logits0), None, None, k)
        og, op, opar = BO.beam_topk(corpus, logits0, None, None, k)
        assert np.array_equal(g.cpu().numpy(), og) and np.array_equal(par.cpu().numpy().reshape(B, k), opar)
    generated = rs.randint(0, K, size=(B, kp, 1)).astype(np.int64)
    generated[:, 2] = generated[:, 0]                                         # beam 2 repeats beam 0 ...
    log_probas = np.tile(np.float32([-0.25, -1.5, -0.25, -0.75]), (B, 1))
    logits1 = rs.randint(0, 3, size=(B, kp, K)).astype(np.float32)
    logits1[:, 2] = logits1[:, 0]                                             # ... with the same logits row
    logits1 = logits1.reshape(B * kp, K)
    for k in (10, 16):
        g, p, par = idx.beam_topk(dev(logits1), dev(generated), dev(log_probas), k)
        og, op, opar = BO.beam_topk(corpus, logits1, generated, log_probas, k)
        g, p, par = g.cpu().numpy(), p.cpu().numpy(), par.cpu().numpy().reshape(B, k)
        assert np.array_equal(g, og) and np.array_equal(par, opar)
        np.testing.assert_allclose(p, op, rtol=TOL, atol=TOL)
        tied = op[:, 1:] == op[:, :-1]
        assert tied.sum() > B * 3
        assert np.array_equal(p[:, 1:].view(np.uint32)[tied], p[:, :-1].view(np.uint32)[tied])
        flat = (par - np.arange(B)[:, None] * kp) * K + g[:, :, 1]
        assert (flat[:, 1:][tied] > flat[:, :-1][tied]).all()


def test_sparse_corpus_fills_with_minus_inf_in_index_order():
    """Fewer than k valid extensions: the valid ones first, then -inf fillers in ascending flat index with their parents and
    ids, as the oracle has them."""
    from rq_vae_recommender_b200 import ops
    K, k, B = 256, 10, 6
    corpus = np.array([[5, 1, 0], [5, 2, 0], [200, 7, 1]], dtype=np.int64)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    rs = np.random.RandomState(22)
    logits0 = rs.randn(B, K).astype(np.float32)
    g0, p0, par0 = idx.beam_topk(dev(logits0), None, None, k)
    og, op, opar = BO.beam_topk(corpus, logits0, None, None, k)
    assert np.array_equal(g0.cpu().numpy(), og) and np.array_equal(par0.cpu().numpy().reshape(B, k), opar)
    np.testing.assert_allclose(p0.cpu().numpy(), op, rtol=TOL, atol=TOL)
    assert np.isfinite(op[:, :2]).all() and np.isneginf(op[:, 2:]).all()
    assert (og[:, 2:, 0] == [0, 1, 2, 3, 4, 6, 7, 8]).all()                  # fillers: the lowest codes not already kept
    logits1 = rs.randn(B * k, K).astype(np.float32)
    g1, p1, par1 = idx.beam_topk(dev(logits1), g0, p0, k)
    og, op, opar = BO.beam_topk(corpus, logits1, g0.cpu().numpy(), p0.cpu().numpy(), k)
    assert np.array_equal(g1.cpu().numpy(), og) and np.array_equal(par1.cpu().numpy().reshape(B, k), opar)
    np.testing.assert_allclose(p1.cpu().numpy(), op, rtol=TOL, atol=TOL)
    assert np.isfinite(op[:, :3]).all() and np.isneginf(op[:, 3:]).all()


def test_bad_rows_complete_and_are_counted():
    from rq_vae_recommender_b200 import ops
    B, K, k = 12, 256, 10
    rs = np.random.RandomState(23)
    corpus = realistic_corpus(rs, 5000, 3, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    good = dev(rs.randn(B, K).astype(np.float32))
    bad = good.clone()
    bad[1, 7] = float("nan")
    bad[4, 200] = float("inf")
    bad[5] = -float("inf")
    bad[8, 3] = -float("inf")                                                 # one -inf logit is a valid row
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    out_bad = idx.beam_topk(bad, None, None, k, bad=counter)
    out_ok = idx.beam_topk(good, None, None, k)
    assert counter.tolist() == [3]
    keep = torch.tensor([r not in (1, 4, 5, 8) for r in range(B)], device="cuda")
    for a, b in zip(out_bad, out_ok):
        rows = keep if a.shape[0] == B else keep.repeat_interleave(k)
        assert torch.equal(a[rows], b[rows])
    for r in (1, 4, 5):                                                      # every candidate of a bad row scores -inf
        assert bool(torch.isneginf(out_bad[1][r]).all())
        assert out_bad[0][r, :, 0].tolist() == list(range(k))
    assert bool(torch.isfinite(out_bad[1][8]).any())
    idx.beam_topk(bad, None, None, k, bad=counter)
    assert counter.tolist() == [6]                                            # the count accumulates over calls
    # h = 1: a bad beam row touches its own history only
    gen, lp, _ = out_ok
    logits1 = dev(rs.randn(B * k, K).astype(np.float32))
    bad1 = logits1.clone()
    bad1[2 * k + 3, 11] = float("nan")
    counter.zero_()
    out_bad = idx.beam_topk(bad1, gen, lp, k, bad=counter)
    out_ok = idx.beam_topk(logits1, gen, lp, k)
    assert counter.tolist() == [1]
    keep = torch.arange(B, device="cuda") != 2
    for a, b in zip(out_bad, out_ok):
        rows = keep if a.shape[0] == B else keep.repeat_interleave(k)
        assert torch.equal(a[rows], b[rows])
    assert not bool((out_bad[2].view(B, k)[2] == 2 * k + 3).any())


def test_op_arguments():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200._lib import Rqb200Error
    rs = np.random.RandomState(24)
    idx = ops.SidPrefixIndex(dev(realistic_corpus(rs, 500, 3, 16)), 16)
    x = dev(rs.randn(4, 16).astype(np.float32))
    with pytest.raises(Rqb200Error, match="k = 33"):
        idx.beam_topk(x, None, None, 33)
    with pytest.raises(Rqb200Error, match="k = 17"):
        idx.beam_topk(x, None, None, 17)
    with pytest.raises(ValueError, match="codes"):
        idx.beam_topk(dev(rs.randn(4, 32).astype(np.float32)), None, None, 4)
    with pytest.raises(ValueError, match="B \\* kp"):
        idx.beam_topk(x, torch.zeros((4, 2, 1), dtype=torch.int64, device="cuda"), torch.zeros((4, 2), device="cuda"), 4)
    big = ops.SidPrefixIndex(dev(rs.randint(0, 4096, size=(500, 2)).astype(np.int64)), 4096)
    with pytest.raises(Rqb200Error, match="K = 4096"):
        big.beam_topk(dev(rs.randn(4, 4096).astype(np.float32)), None, None, 10)
    empty = idx.beam_topk(torch.empty((0, 16), device="cuda"), None, None, 4)
    assert empty[0].shape == (0, 4, 1)
    strided = dev(rs.randn(4, 40).astype(np.float32))[:, 3:19]                  # a row stride above K, and fp64 input
    a = idx.beam_topk(strided, None, None, 4)
    b = idx.beam_topk(strided.double().contiguous(), None, None, 4)
    assert all(torch.equal(u, v) for u, v in zip(a, b))


def torch_level(index, logits, generated, log_probas, k):
    """One level in torch: log_softmax, SidPrefixIndex.check, masked_fill, a stable descending sort and gathers.  Returns
    (generated [B, k + 1, h + 1], log_probas [B, k + 1], parent_global [B, k + 1]) -- one entry more, for the gap rule -- and
    every candidate's score [B, kp * K]."""
    K = logits.shape[1]
    B, kp, h = (logits.shape[0], 1, 0) if generated is None else generated.shape
    codes = torch.arange(K, device=logits.device).repeat(B * kp).unsqueeze(1)
    prefix = codes if h == 0 else torch.cat([generated.reshape(-1, h).repeat_interleave(K, dim=0), codes], dim=1)
    scores = F.log_softmax(logits.float(), dim=-1).reshape(B, kp * K)
    if h:
        scores = scores + log_probas.repeat_interleave(K, dim=1)
    scores = scores.masked_fill(~index.check(prefix).reshape(B, kp * K), float("-inf"))
    s, order = scores.sort(dim=-1, descending=True, stable=True)
    top = order[:, : k + 1]
    parent = top // K
    new_ids = (top % K).unsqueeze(-1)
    gen = new_ids if h == 0 else torch.cat([torch.gather(generated, 1, parent.unsqueeze(-1).expand(-1, -1, h)), new_ids], -1)
    return gen, s[:, : k + 1], parent + torch.arange(B, device=logits.device).unsqueeze(1) * kp, scores


def test_generate_beam_search():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    K, H, B, k = 256, 3, 48, 10
    rs = np.random.RandomState(25)
    m = small_model(M, realistic_corpus(rs, 3000, H, K), K, H, k=k)
    mask, ids, users = history(rs, B, 20, H, K)
    before = ops.LAUNCHES
    torch.manual_seed(1)
    rng = torch.cuda.get_rng_state()
    g1, p1 = m.generate(mask, ids, users, search="beam")
    assert ops.LAUNCHES - before == 1 + H                                     # the index build, then one launch per level
    assert torch.equal(torch.cuda.get_rng_state(), rng)
    assert g1.shape == (B, k, H) and bool(torch.isfinite(p1).all())
    torch.manual_seed(2)
    before = ops.LAUNCHES
    g2, p2 = m.generate(mask, ids, users, search="beam")
    assert ops.LAUNCHES - before == H
    assert torch.equal(g1, g2) and torch.equal(p1, p2)
    # against the torch composition on the logits the model's head produced at each level (recorded by hooks) and the beams
    # the kernel returned for the level before
    logits, levels = [], []
    hooks = [mlp.register_forward_hook(lambda mod, inp, out: logits.append(out.detach().clone())) for mlp in m.decoder_mlp]
    index = m._prefix_index(torch.device("cuda"))

    class Recording:
        def beam_topk(self, lg, generated, log_probas, k, bad=None):
            out = index.beam_topk(lg, generated, log_probas, k, bad=bad)
            levels.append((generated, log_probas, out))
            return out

    m._prefix_index = lambda device: Recording()
    try:
        g3, p3 = m.generate(mask, ids, users, search="beam")
    finally:
        for hk in hooks:
            hk.remove()
        del m._prefix_index
    assert torch.equal(g3, g1) and len(logits) == H
    for lg, (generated, log_probas, out) in zip(logits, levels):
        ref_g, ref_p, ref_par, scores = (t.cpu().numpy() for t in torch_level(index, lg, generated, log_probas, k))
        assert_matches(ref_g, ref_p, ref_par, scores, out, k, exact_ties=False, min_checked=0.9)


def test_generate_beam_search_raises_on_nan_head_and_limits():
    from rq_vae_recommender_b200._lib import Rqb200Error
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 256, 3, 8
    rs = np.random.RandomState(26)
    corpus = realistic_corpus(rs, 2000, H, K)
    m = small_model(M, corpus, K, H)
    with torch.no_grad():
        m.decoder_mlp[1].weight[3, 0] = float("nan")
    mask, ids, users = history(rs, B, 5, H, K)
    with pytest.raises(RuntimeError, match="NaN"):
        m.generate(mask, ids, users, search="beam")
    with pytest.raises(Rqb200Error, match="top_k_for_generation = 33"):
        small_model(M, corpus, K, H, k=33).generate(mask, ids, users, search="beam")
    with pytest.raises(Rqb200Error, match="top_k_for_generation = 20"):
        small_model(M, realistic_corpus(rs, 500, H, 16), 16, H, k=20).generate(mask % 16, ids % 16, users, search="beam")
    m20 = small_model(M, corpus, K, H, k=20)                                  # the sampled search rejects 20 x 64 candidates
    g, p = m20.generate(mask, ids, users, search="beam")
    assert g.shape == (B, 20, H) and bool(torch.isfinite(p[:, 0]).all())
