"""CPU-only: the warped-draw oracle (warp_sample_oracle) against brute-force statements of its rules, and the sampling
controls' argument rules -- bad temperatures and nucleus masses, wrong sequence lengths and the deterministic searches raise
ValueError before any launch, and capture_generate_items fixes the values it is given."""
import math

import numpy as np
import pytest
import torch

import warp_sample_oracle as WO
from test_generate_graph_args import B, H, _batch, _fake_graph_class, _model


# ------------------------------------------------------------------------------------------------------------------- oracle
def _brute_nucleus(p, top_p):
    """N by its definition: the largest t among the p with mass(p >= t) >= top_p * total."""
    if top_p >= 1:
        return np.ones(p.shape, dtype=bool)
    total = p.sum()
    best = None
    for t in np.unique(p):
        if p[p >= t].sum() >= top_p * total and (best is None or t > best):
            best = t
    return p >= best


def test_nucleus_is_its_definition():
    rs = np.random.RandomState(0)
    skipped = 0
    for _ in range(200):
        K = rs.randint(1, 40)
        p = rs.randint(0, 6, size=K).astype(np.float64)           # many exact ties
        if p.sum() == 0:
            p[0] = 1
        p /= p.sum()
        top_p = rs.choice([0.05, 0.3, 0.5, 0.9, 0.999, 1.0])
        N, amb = WO.nucleus(p, top_p, tol=1e-12)
        skipped += amb                                          # the mass meets the target to rounding: either side is right
        assert amb or np.array_equal(N, _brute_nucleus(p, top_p)), (p, top_p)
    assert skipped < 40


def test_boundary_ties_are_all_in():
    p = np.array([0.4, 0.2, 0.2, 0.2])
    N, amb = WO.nucleus(p, 0.5, tol=1e-9)
    assert N.tolist() == [True, True, True, True] and not amb    # 0.4 < 0.5: t = 0.2, and every 0.2 is in
    N, _ = WO.nucleus(p, 0.4)
    assert N.tolist() == [True, False, False, False]
    N, amb = WO.nucleus(np.array([0.5, 0.25, 0.25]), 0.5, tol=1e-9)
    assert N.tolist() == [True, False, False] and amb          # the mass at t meets the target exactly: reported ambiguous


def test_tiny_top_p_keeps_one_code():
    rs = np.random.RandomState(1)
    x = rs.randn(20, 300) * 3
    p = WO.tempered(x, 0.7)
    for r in range(20):
        N, _ = WO.nucleus(p[r], 1e-6)
        assert N.sum() == 1 and N[np.argmax(p[r])]
    s, lp, amb, bad = WO.warped_level(x, rs.exponential(size=x.shape), 0.7, 1e-6, 8)
    assert (s[:, 0] == x.argmax(1)).all() and np.isfinite(lp[:, 0]).all() and np.isneginf(lp[:, 1:]).all()
    for r in range(20):                                         # the fillers: the other codes, ascending
        assert s[r, 1:].tolist() == [c for c in range(8) if c != s[r, 0]][:7]


def test_small_temperature_underflow_leaves_fillers():
    x = np.zeros((1, 64))
    x[0, :3] = [10.0, 9.0, -5.0]                                # at T = 0.05: exp(-20), exp(-300) -> 0 in fp32, ...
    p = WO.tempered(x, 0.05)
    assert p[0, 0] > 0 and p[0, 1] > 0 and p[0, 2] == 0 and (p[0, 3:] == 0).all()
    s, lp, _, _ = WO.warped_level(x, np.ones_like(x), 0.05, 1.0, 4)
    assert s[0].tolist() == [0, 1, 2, 3] and np.isfinite(lp[0, :2]).all() and np.isneginf(lp[0, 2:]).all()


def test_nucleus_smaller_than_nc_and_draw_is_a_multinomial_race():
    rs = np.random.RandomState(2)
    x = rs.randn(50, 256) * 4
    q = rs.exponential(size=x.shape)
    s, lp, _, _ = WO.warped_level(x, q, 1.5, 0.3, 64)
    p = WO.tempered(x, 1.5)
    lse = x.max(1) + np.log(np.exp(x - x.max(1, keepdims=True)).sum(1))
    for r in range(50):
        N = _brute_nucleus(p[r], 0.3)
        n = min(64, N.sum())
        ratio = np.where(N, p[r] / q[r], -1)
        assert n < 64 and list(s[r, :n]) == list(np.argsort(-ratio, kind="stable")[:n])
        np.testing.assert_allclose(lp[r, :n], x[r, s[r, :n]] - lse[r])
        assert np.isneginf(lp[r, n:]).all() and list(s[r, n:]) == list(np.nonzero(~N)[0][:64 - n])


def test_bad_rows_and_keep_best():
    x = np.random.RandomState(3).randn(4, 16)
    x[1, 2], x[2, 5], x[3] = np.nan, np.inf, -np.inf
    s, lp, _, bad = WO.warped_level(x, np.ones_like(x), 1.0, 0.9, 4)
    assert bad.tolist() == [False, True, True, True] and np.isneginf(lp[1:]).all()
    g, sc, par = WO.keep_best(s, lp, None, None, 3, lambda b, prefix: prefix[-1] % 2 == 0)
    assert all(int(t) % 2 == 0 for t, v in zip(g[0, :, 0], sc[0]) if v > -np.inf)
    assert (np.diff(sc[0]) <= 0).all() and np.isneginf(sc[1:]).all()


# ------------------------------------------------------------------------------------------------------------- arguments
@pytest.mark.parametrize("kw,match", [
    (dict(temperature=0.0), "temperature must be finite and > 0"), (dict(temperature=-1.0), "temperature must be"),
    (dict(temperature=math.inf), "temperature must be"), (dict(temperature=math.nan), "temperature must be"),
    (dict(top_p=0.0), r"top_p must be in \(0, 1\]"), (dict(top_p=1.5), "top_p must be in"), (dict(top_p=math.nan), "top_p"),
    (dict(temperature=[1.0, 2.0]), "temperature has 2 values"), (dict(top_p=[0.9] * (H + 1)), f"top_p has {H + 1} values"),
    (dict(temperature="hot"), "temperature"),
    (dict(search="beam", temperature=0.5), "deterministic"), (dict(search="beam", top_p=0.9), "deterministic"),
    (dict(search="exact", top_p=[1.0, 1.0, 0.5]), "deterministic")])
@pytest.mark.parametrize("entry", ["generate", "generate_items", "capture_generate_items"])
def test_bad_controls_raise_before_any_launch(entry, kw, match):
    from rq_vae_recommender_b200 import ops
    m = _model()
    batch = _batch()
    launches = ops.LAUNCHES
    with pytest.raises(ValueError, match=match):
        if entry == "generate":
            m.generate(batch.seq_mask.long(), batch.sem_ids, **kw)
        else:
            getattr(m, entry)(batch, **kw)
    assert ops.LAUNCHES == launches


@pytest.mark.parametrize("kw,match", [(dict(temperature=0.0), "temperature must be"), (dict(top_p=2.0), "top_p must be"),
                                      (dict(search="beam", top_p=0.5), "deterministic"),
                                      (dict(search="exact", top_p=0.5), "deterministic"),
                                      (dict(temperature=[0.5, 1.0]), "temperature has 2 values")])
def test_generate_next_sem_id_controls(kw, match):
    m = _model()
    with pytest.raises(ValueError, match=match):
        m.generate_next_sem_id(_batch(), **kw)


def test_controls_per_level_and_the_default_path():
    from rq_vae_recommender_b200.modules import model as M
    assert M._sampling_controls("sample", 1, 1.0, H, "t") is None
    assert M._sampling_controls("sample", [1.0] * H, (1, 1, 1), H, "t") is None
    assert M._sampling_controls("sample", 0.5, 1.0, H, "t") == [(0.5, 1.0)] * H
    assert M._sampling_controls("sample", [2.0, 1.0, 1.0], 0.9, H, "t") == [(2.0, 0.9), (1.0, 0.9), (1.0, 0.9)]
    assert M._sampling_controls("sample", torch.tensor([0.5, 1.0, 3.0]), 1.0, H, "t") == [(0.5, 1.0), (1.0, 1.0), (3.0, 1.0)]
    # generate_next_sem_id's temperature is ignored by the deterministic searches, whatever its value
    assert M._sampling_controls("beam", 0.0, 1.0, H, "t", ignore_temperature=True) is None
    assert M._sampling_controls("exact", [7.0, 1.0], 1.0, H, "t", ignore_temperature=True) is None
    with pytest.raises(ValueError, match="deterministic"):
        M._sampling_controls("beam", 0.3, 0.5, H, "t", ignore_temperature=True)


def test_capture_fixes_the_controls():
    m = _model()
    Fake = _fake_graph_class()
    g = Fake(m, _batch(), None, "sample", None, None, None, None, None, "fused", "fused", [0.5, 1.0, 2.0], 0.9)
    assert g.warp == [(0.5, 0.9), (1.0, 0.9), (2.0, 0.9)]
    assert Fake(m, _batch(), None, "sample", None, None, None, None, None).warp is None
    assert Fake(m, _batch(), None, "beam", None, None, None, None, None, "fused", "fused", 1.0, 1.0).warp is None


def test_warped_graph_errors_are_the_beam_searchs(monkeypatch):
    """A warped search counts bad head rows as the beam search does, and raises its error after the replay."""
    m = _model()
    Fake = _fake_graph_class()

    class Warped(Fake):
        def _capture(self):
            super()._capture()
            self.counters = torch.zeros(1, dtype=torch.int32)
            self._captured = (self._captured[0], torch.zeros(1, dtype=torch.int32), 1, [])

    g = Warped(m, _batch(), None, "sample", None, None, None, None, None, "fused", "fused", 0.7, 1.0)
    g.counters.fill_(2)
    with pytest.raises(RuntimeError, match="generate: 2 beam row"):
        g(_batch())
    g.counters.zero_()
    assert g(_batch()).item_ids.shape[0] == B
