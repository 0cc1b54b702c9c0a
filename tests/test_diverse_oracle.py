"""CPU-only: the capped search's statement (diverse_oracle) against brute force -- its kept set dominates every feasible set
rank by rank, it is the greedy walk, and a cap of k or more is the uncapped selection -- and the cap's argument rules, which
raise before any launch."""
import itertools

import numpy as np
import pytest
import torch

import beam_search_oracle as O
import diverse_oracle as D
from test_generate_graph_args import H, K, _batch, _fake_graph_class, _model


def _feasible_sets(s, grp, per_beam, m, k):
    """Every set of at most k finite candidates holding at most m of any group."""
    fin = [e for e in range(len(s)) if np.isfinite(s[e])]
    for n in range(min(k, len(fin)) + 1):
        for chosen in itertools.combinations(fin, n):
            held = {}
            for e in chosen:
                held[grp[e // per_beam]] = held.get(grp[e // per_beam], 0) + 1
            if max(held.values(), default=0) <= m:
                yield chosen


@pytest.mark.parametrize("seed", range(12))
def test_kept_set_dominates_every_feasible_set(seed):
    rs = np.random.RandomState(seed)
    kp, per_beam = rs.randint(1, 4), rs.randint(1, 4)
    E = kp * per_beam
    k, m = rs.randint(1, min(E, 5) + 1), rs.randint(1, 3)
    s = rs.randint(-3, 3, size=(1, E)).astype(np.float64)              # exact ties within and across groups
    s[0, rs.rand(E) < 0.2] = -np.inf
    s[0, rs.rand(E) < 0.1] = np.nan
    grp = D.groups(rs.randint(0, 2, size=(1, kp, 2)), rs.randint(1, 3))
    idx, val = D.select(D.capped_scores(s, grp, per_beam, m), k)
    kept = np.sort(val[0][np.isfinite(val[0])])[::-1]
    clean = np.where(np.isnan(s[0]), -np.inf, s[0])
    for chosen in _feasible_sets(clean, grp[0], per_beam, m, k):
        other = np.sort(clean[list(chosen)])[::-1]
        assert len(kept) >= len(other) and (kept[:len(other)] >= other).all(), (s, grp, chosen)
    # the walk itself gives the same indices and scores, fillers included
    widx, wval = D.greedy_walk(s, grp, per_beam, m, k)
    assert np.array_equal(idx, widx) and np.array_equal(val, wval)
    # the guarantee
    held = {}
    for e, v in zip(idx[0], val[0]):
        if np.isfinite(v):
            held[grp[0, e // per_beam]] = held.get(grp[0, e // per_beam], 0) + 1
    assert max(held.values(), default=0) <= m


@pytest.mark.parametrize("prefix_len", [1, 2])
def test_cap_of_k_or_more_is_the_uncapped_level(prefix_len):
    rs = np.random.RandomState(prefix_len)
    Kc, h, kp, B, k = 12, 2, 5, 4, 6
    corpus = rs.randint(0, Kc, size=(300, 3)).astype(np.int64)
    generated = corpus[rs.randint(0, 300, size=(B, kp)), :h]
    log_probas = -rs.rand(B, kp).astype(np.float32)
    logits = rs.randn(B * kp, Kc).astype(np.float32)
    want = O.beam_topk(corpus, logits, generated, log_probas, k)
    for m in (k, k + 3):
        got = D.beam_topk_capped(corpus, logits, generated, log_probas, k, prefix_len, m)
        for a, b in zip(got, want):
            assert np.array_equal(np.asarray(a).reshape(np.shape(b)), b)
    got = D.beam_topk_capped(corpus, logits, generated, log_probas, k, prefix_len, 1)
    grp = D.groups(generated, prefix_len)
    for b in range(B):
        fin = np.isfinite(got[1][b])
        lead = [grp[b, p - b * kp] for p in got[2][b][fin]]
        assert len(lead) == len(set(lead))


# ------------------------------------------------------------------------------------------------------------- arguments
@pytest.mark.parametrize("kw,err,match", [
    (dict(max_per_prefix=0), ValueError, "max_per_prefix must be an integer >= 1"),
    (dict(max_per_prefix=-2), ValueError, "max_per_prefix must be"),
    (dict(max_per_prefix=1.5), ValueError, "max_per_prefix must be"),
    (dict(max_per_prefix=1, prefix_len=0), ValueError, r"prefix_len must be an integer in \[1, 2\]"),
    (dict(max_per_prefix=1, prefix_len=H), ValueError, "prefix_len must be"),
    (dict(max_per_prefix=1, search="exact"), ValueError, "exact"),
    (dict(max_per_prefix=1, search="beam", num_beams=33), "Rqb200Error", "cluster kernels"),
    (dict(max_per_prefix=1, search="sample", num_beams=17), "Rqb200Error", "cluster kernels"),
    (dict(max_per_prefix=2, search="sample", num_beams=33), "Rqb200Error", "cluster kernels")])
@pytest.mark.parametrize("entry", ["generate", "generate_next_sem_id", "generate_items", "capture_generate_items"])
def test_bad_caps_raise_before_any_launch(entry, kw, err, match):
    from rq_vae_recommender_b200 import ops
    if err == "Rqb200Error":
        from rq_vae_recommender_b200._lib import Rqb200Error as err
    m = _model()
    batch = _batch()
    launches = ops.LAUNCHES
    with pytest.raises(err, match=match):
        if entry == "generate":
            m.generate(batch.seq_mask.long(), batch.sem_ids, **kw)
        else:
            getattr(m, entry)(batch, **kw)
    assert ops.LAUNCHES == launches


def test_cap_controls():
    from rq_vae_recommender_b200.modules import model as M
    assert M._prefix_cap_controls("beam", None, 0, H, "t") is None              # no cap: prefix_len is not read
    assert M._prefix_cap_controls("sample", 2, 2, H, "t") == (2, 2)
    m = _model()                                                                # top_k_for_generation = 3
    assert m._capping("beam", 3, 1, None, "t") is None                          # max_per_prefix >= w cannot bind
    assert m._capping("beam", 40, 1, 40, "t") is None                           # ... at any width
    assert m._capping("beam", 2, 1, None, "t") == (1, 2)
    assert m._capping("sample", 1, 2, 16, "t") == (2, 1)                        # 16 beams x 64 candidates: one CTA


def test_capture_fixes_the_cap():
    m = _model()
    Fake = _fake_graph_class()
    g = Fake(m, _batch(), None, "beam", 10, None, None, None, None, "fused", "fused", 1.0, 1.0, 2, 2)
    assert g.cap == (2, 2)
    assert Fake(m, _batch(), None, "beam", 10, None, None, None, None, "fused", "fused", 1.0, 1.0, 10, 1).cap is None
    assert Fake(m, _batch(), None, "sample", None, None, None, None, None).cap is None
    assert K >= 10
