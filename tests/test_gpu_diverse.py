"""GPU tests of the per-prefix cap on the generative-retrieval search: SidPrefixIndex.beam_topk / sample_select /
sample_select_warped with ``cap`` against the numpy statement (diverse_oracle), beams, parents and log-probabilities bit for bit,
then the model end to end on both decoders.

The statement runs on the kernels' own fp32 scores.  Each group's max_per_prefix best are among its beams' max_per_prefix best
(max_per_prefix < k <= 32), so one uncapped launch over the beams as single-beam histories (the same rows, noise and filter,
the 32 best of each) gives every score the capped walk can keep, with the bits the uncapped kernel gives that extension.
`pytest -m gpu`."""
import numpy as np
import pytest
import torch

import diverse_oracle as D
from test_gpu_exclusion import built as built_exclusion, exclusion_sets
from test_gpu_generate import dev, level_logits, realistic_corpus, small_model
from test_gpu_generate_graph import assert_same, batch_of
from test_gpu_inclusion import allow_lists, built as built_inclusion

pytestmark = pytest.mark.gpu


def _beams(rs, corpus, B, kp, h, K, sparse_ids=True):
    """[B, kp, h] beams: corpus prefixes drawn from a few first codes (groups of several beams), some not in the corpus."""
    rows = corpus[rs.randint(0, len(corpus), size=(B, kp))]
    gen = rows[:, :, :h].copy()
    heads = corpus[rs.randint(0, len(corpus), size=(B, 3)), 0]                 # three level-0 codes per history, shared
    gen[:, :, 0] = np.take_along_axis(heads, rs.randint(0, 3, size=(B, kp)), 1)
    if sparse_ids:
        gen[rs.rand(B, kp) < 0.1, -1] = rs.randint(0, K)
    return gen


def _filters(kind, rs, corpus, K, B, kp):
    """(filter of the B histories, the same filter for the B * kp single-beam histories)."""
    if kind == "none":
        return {}, {}
    if kind == "exclude":
        items = exclusion_sets(rs, corpus, B, 64)
        return ({"exclude": built_exclusion(corpus, K, items)[2]},
                {"exclude": built_exclusion(corpus, K, np.repeat(items, kp, 0))[2]})
    items = allow_lists(rs, corpus, max(B, 2), 256)[:B]
    return ({"include": built_inclusion(corpus, K, items)[2]},
            {"include": built_inclusion(corpus, K, np.repeat(items, kp, 0))[2]})


def _known_scores(g1, p1, B, kp, per_beam, slot_of):
    """[B, kp * per_beam] fp32: the single-beam launch's scores at their flat index, -inf elsewhere."""
    S = np.full((B, kp * per_beam), -np.inf, dtype=np.float32)
    for r in range(B * kp):
        b, beam = divmod(r, kp)
        for tok, v in zip(g1[r, :, -1], p1[r]):
            if np.isfinite(v):
                S[b, beam * per_beam + slot_of(r, int(tok))] = v
    return S


def _expect(S, generated, prefix_len, m, k, per_beam, tok_of):
    idx, val = D.greedy_walk(S, D.groups(generated, prefix_len), per_beam, m, k)
    B, kp, h = generated.shape
    beam = idx // per_beam
    toks = np.array([[tok_of(b, int(e)) for e in row] for b, row in enumerate(idx)], dtype=np.int64).reshape(B, k)
    gen = np.concatenate([np.take_along_axis(generated, beam[:, :, None], 1), toks[:, :, None]], axis=2)
    return gen, val, (np.arange(B)[:, None] * kp + beam).reshape(-1)


def _check(out, want):
    g, p, par = (t.cpu().numpy() for t in out[:3])
    wg, wp, wpar = want
    assert np.array_equal(p.view(np.uint32), wp.astype(np.float32).view(np.uint32))
    assert np.array_equal(g, wg) and np.array_equal(par, wpar)


def _bits_equal(a, b):
    """Equal tensors, floats bit for bit (a NaN equals the same NaN)."""
    if a.dtype.is_floating_point:
        return torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


def _assert_cap(generated, log_probas, prefix_len, m):
    g, p = generated.cpu().numpy(), log_probas.cpu().numpy()
    for b in range(g.shape[0]):
        fin = np.isfinite(p[b])
        _, counts = np.unique(g[b][fin][:, :prefix_len], axis=0, return_counts=True)
        assert counts.max(initial=0) <= m


# ------------------------------------------------------------------------------------------------------------ beam top-k
# (K, H, kp, k, B): k = kp at a level past the first; 2048 x 32 = 65 536 > 49 152 candidates takes the recomputed keys
BEAM_CASES = [(256, 3, 10, 10, 640), (300, 3, 10, 10, 7), (2048, 3, 10, 10, 7), (256, 5, 32, 32, 7), (300, 5, 2, 2, 7),
              (2048, 5, 32, 32, 7), (2048, 3, 25, 1, 1), (256, 3, 32, 32, 640), (300, 3, 32, 32, 1)]


@pytest.mark.parametrize("filt", ["none", "exclude", "include"])
@pytest.mark.parametrize("K,H,kp,k,B", BEAM_CASES)
def test_beam_topk_capped(K, H, kp, k, B, filt):
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K + H + kp + k + B + len(filt))
    corpus = realistic_corpus(rs, 12101, H, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    f_cap, f_one = _filters(filt, rs, corpus, K, B, kp)
    for h, prefix_len in [(1, 1), (2, 1), (2, 2), (H - 1, 2)]:
        gen = _beams(rs, corpus, B, kp, h, K)
        lp = (-rs.rand(B, kp) * 4).astype(np.float32)
        logits = level_logits(rs, corpus, gen.reshape(B * kp, h), B * kp, K)
        logits[rs.rand(B * kp) < 0.02] = np.nan                                 # bad rows: all their candidates -inf
        gen_d, lp_d, logits_d = dev(gen), dev(lp), dev(logits)
        bad1 = torch.zeros(1, dtype=torch.int32, device="cuda")
        one = idx.beam_topk(logits_d, gen_d.reshape(B * kp, 1, h), lp_d.reshape(B * kp, 1), min(32, K), bad=bad1, **f_one)
        S = _known_scores(one[0].cpu().numpy(), one[1].cpu().numpy(), B, kp, K, lambda r, tok: tok)
        plain = idx.beam_topk(logits_d, gen_d, lp_d, k, **f_cap)
        for m in sorted({1, 2, 3, k}):
            bad = torch.zeros(1, dtype=torch.int32, device="cuda")
            out = idx.beam_topk(logits_d, gen_d, lp_d, k, bad=bad, cap=(prefix_len, m), **f_cap)
            assert int(bad) == int(bad1)
            if m >= k:                                                          # cannot bind: the uncapped result
                for a, b in zip(out, plain):
                    assert _bits_equal(a, b)
                continue
            _check(out, _expect(S, gen, prefix_len, m, k, K, lambda b, e: e % K))
            _assert_cap(out[0], out[1], prefix_len, m)


def test_beam_topk_capped_ties_and_fillers():
    """Exact score ties across groups (integer logits, equal parents) and a 40-row corpus that leaves fillers."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(5)
    K, H, kp, k, B = 300, 3, 12, 12, 7
    for corpus in (realistic_corpus(rs, 12101, H, K), realistic_corpus(rs, 40, H, K)):
        idx = ops.SidPrefixIndex(dev(corpus), K)
        gen = _beams(rs, corpus, B, kp, 2, K, sparse_ids=False)
        lp = np.zeros((B, kp), dtype=np.float32)
        logits = rs.randint(0, 3, size=(B * kp, K)).astype(np.float32)
        one = idx.beam_topk(dev(logits), dev(gen).reshape(B * kp, 1, 2), dev(lp).reshape(B * kp, 1), 32)
        S = _known_scores(one[0].cpu().numpy(), one[1].cpu().numpy(), B, kp, K, lambda r, tok: tok)
        for prefix_len in (1, 2):
            for m in (1, 2, 3):
                out = idx.beam_topk(dev(logits), dev(gen), dev(lp), k, cap=(prefix_len, m))
                _check(out, _expect(S, gen, prefix_len, m, k, K, lambda b, e: e % K))


# ----------------------------------------------------------------------------------------------------------- sampling
SAMPLE_CASES = [(256, 3, 10, 10, 640), (300, 5, 10, 10, 7), (2048, 3, 16, 16, 7), (256, 3, 1, 1, 7), (300, 3, 16, 16, 1),
                (2048, 5, 10, 10, 1)]


@pytest.mark.parametrize("warp", [None, (0.7, 0.9)])
@pytest.mark.parametrize("filt", ["none", "exclude", "include"])
@pytest.mark.parametrize("K,H,kp,k,B", SAMPLE_CASES)
def test_sample_select_capped(K, H, kp, k, B, filt, warp):
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K + H + kp + k + B + len(filt) + (warp is not None))
    nc = 64
    corpus = realistic_corpus(rs, 12101, H, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    f_cap, f_one = _filters(filt, rs, corpus, K, B, kp)
    for h, prefix_len in [(1, 1), (2, 2), (H - 1, 1)]:
        gen = _beams(rs, corpus, B, kp, h, K)
        lp = (-rs.rand(B, kp) * 4).astype(np.float32)
        logits = dev(level_logits(rs, corpus, gen.reshape(B * kp, h), B * kp, K) * 3)
        logits[0] = float("nan")
        x = logits if warp else torch.softmax(logits, -1)
        noise = torch.empty_like(x).exponential_(1)
        gen_d, lp_d = dev(gen), dev(lp)

        def run(g, p, kk, f, **kw):
            cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
            if warp:
                o = idx.sample_select_warped(x, noise, g, p, kk, nc, *warp, want_samples=True, bad=cnt, **f, **kw)
            else:
                o = idx.sample_select(x, noise, g, p, kk, nc, want_samples=True, reject=cnt, **f, **kw)
            return o, cnt

        one, cnt1 = run(gen_d.reshape(B * kp, 1, h), lp_d.reshape(B * kp, 1), min(32, nc), f_one)
        samples = one[3].cpu().numpy()
        slot = [{int(t): r for r, t in enumerate(row)} for row in samples]
        S = _known_scores(one[0].cpu().numpy(), one[1].cpu().numpy(), B, kp, nc, lambda r, tok: slot[r][tok])
        plain, _ = run(gen_d, lp_d, k, f_cap)
        for m in sorted({1, 2, 3, k}):
            out, cnt = run(gen_d, lp_d, k, f_cap, cap=(prefix_len, m))
            assert torch.equal(cnt, cnt1) and _bits_equal(out[3], one[3]) and _bits_equal(out[4], one[4])
            if m >= k:
                for a, b in zip(out, plain):
                    assert _bits_equal(a, b)
                continue
            _check(out, _expect(S, gen, prefix_len, m, k, nc, lambda b, e: int(samples[b * kp + e // nc, e % nc])))
            _assert_cap(out[0], out[1], prefix_len, m)


# ------------------------------------------------------------------------------------------------------------ end to end
K_M, H_M = 256, 3


@pytest.fixture(scope="module")
def corpus():
    return realistic_corpus(np.random.RandomState(12101), 12101, H_M, K_M)


@pytest.fixture(scope="module")
def model(corpus):
    from rq_vae_recommender_b200.modules import model as M
    m = small_model(M, corpus, K_M, H_M)
    with torch.no_grad():
        for head in m.decoder_mlp:                                              # sharpened heads: beams crowd into few prefixes
            for p in head.parameters():
                p.mul_(8)
    return m


@pytest.mark.parametrize("decoder", ["fused", "hf"])
@pytest.mark.parametrize("search", ["beam", "sample"])
def test_generate_respects_the_cap(model, corpus, decoder, search):
    rs = np.random.RandomState(3)
    batch = batch_of(rs, corpus, 7, padded=False)
    for prefix_len, m, w in [(1, 1, 10), (1, 2, 10), (2, 3, 16), (1, 5, 16)]:
        torch.manual_seed(0)
        out = model.generate_next_sem_id(batch, search=search, decoder=decoder, encoder="fused", num_beams=w,
                                         max_per_prefix=m, prefix_len=prefix_len, exclude_history=False)
        _assert_cap(out.sem_ids, out.log_probas, prefix_len, m)
        assert torch.isfinite(out.log_probas).any()
    for m in (10, 11):                                                          # max_per_prefix >= w: the uncapped call
        torch.manual_seed(1)
        want = model.generate_next_sem_id(batch, search=search, decoder=decoder, encoder="fused", num_beams=10)
        torch.manual_seed(1)
        got = model.generate_next_sem_id(batch, search=search, decoder=decoder, encoder="fused", num_beams=10,
                                         max_per_prefix=m)
        assert torch.equal(got.sem_ids, want.sem_ids) and torch.equal(got.log_probas, want.log_probas)


@pytest.mark.parametrize("search", ["beam", "sample"])
def test_items_come_from_capped_beams(model, corpus, search):
    rs = np.random.RandomState(4)
    batch = batch_of(rs, corpus, 7, padded=False)
    torch.manual_seed(0)
    out = model.generate_items(batch, n=20, search=search, decoder="fused", encoder="fused", num_beams=10,
                               max_per_prefix=2, prefix_len=1)
    _assert_cap(out.sem_ids, out.log_probas, 1, 2)
    items, beams = out.item_ids.cpu().numpy(), out.beams.cpu().numpy()
    fin = np.isfinite(out.log_probas.cpu().numpy())
    for b in range(items.shape[0]):
        for it, be in zip(items[b], beams[b]):
            if it >= 0:
                assert fin[b, be] and np.array_equal(corpus[it], out.sem_ids[b, be].cpu().numpy())


@pytest.mark.parametrize("search", ["beam", "sample"])
@pytest.mark.parametrize("B", [1, 7, 640])
def test_replay_with_cap_equals_eager(model, corpus, search, B):
    rs = np.random.RandomState(B)
    batch = batch_of(rs, corpus, B, padded=False)
    kw = dict(n=10, search=search, num_beams=10, max_per_prefix=2, prefix_len=1)
    g = model.capture_generate_items(batch, **kw)
    assert g.cap == (1, 2)
    torch.manual_seed(7)
    got = g(batch)
    torch.manual_seed(7)
    want = model.generate_items(batch, encoder="fused", decoder="fused", **kw)
    assert_same(got, want)
    side = torch.cuda.Stream()                                                  # and on a side stream
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.manual_seed(7)
        got2 = g(batch)
        torch.manual_seed(7)
        want2 = model.generate_items(batch, encoder="fused", decoder="fused", **kw)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert_same(got2, want)
    assert_same(want2, want)
