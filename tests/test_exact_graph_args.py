"""CPU-only: capture_exact_items refuses what its graph cannot run (training mode, autocast, widths outside the exact search's
limits, a bad max_rows) before any launch, and ExactItemsGraph's bookkeeping on a fake graph: the eager errors from its one
counter read, the decoder rows it reports, and the eager fallback a capacity overflow takes."""
import pytest
import torch

from test_generate_graph_args import H, _batch, _model


@pytest.mark.parametrize("kw,error,match", [
    (dict(num_beams=0), "Rqb200Error", "num_beams = 0"),
    (dict(num_beams=65), "Rqb200Error", "num_beams = 65"),
    (dict(max_rows=0), "ValueError", "max_rows = 0"),
    (dict(max_rows=2.5), "ValueError", "max_rows = 2.5"),
    (dict(encoder_attention="bf16"), "ValueError", "encoder_attention must be")])
def test_refused_arguments(kw, error, match):
    from rq_vae_recommender_b200 import _lib, ops
    m = _model()
    launches = ops.LAUNCHES
    with pytest.raises(_lib.Rqb200Error if error == "Rqb200Error" else ValueError, match=match):
        m.capture_exact_items(_batch(), **kw)
    assert ops.LAUNCHES == launches


def test_training_mode_and_autocast_are_refused(monkeypatch):
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    m = _model().train()
    launches = ops.LAUNCHES
    with pytest.raises(ValueError, match="eval mode only"):
        m.capture_exact_items(_batch())
    m.eval()
    monkeypatch.setattr(M.torch, "is_autocast_enabled", lambda *a: True)
    with pytest.raises(ValueError, match="autocast"):
        m.capture_exact_items(_batch())
    assert ops.LAUNCHES == launches


def test_generate_graph_still_refuses_exact_and_names_the_exact_graph():
    with pytest.raises(ValueError, match="capture_exact_items"):
        _model().capture_generate_items(_batch(), search="exact")


def _fake_exact_class():
    """ExactItemsGraph with the capture replaced by a fake graph: a replay writes sem_ids[:, :n] to item_ids and the read values
    set in ``values`` ([beam counter, filter counts..., bad rows, overflow, rows])."""
    from rq_vae_recommender_b200.modules import model as M

    class Replay:
        def __init__(self, g):
            self.g, self.replays = g, 0

        def replay(self):
            self.replays += 1
            out, values = self.g._captured[:2]
            out.item_ids.copy_(self.g._static[0][:, :self.g.n])
            values.copy_(self.g.values)

    class Fake(M.ExactItemsGraph):
        captures = 0
        filters = []

        def _capture(self):
            self.captures += 1
            self.values = torch.zeros(1 + len(self.filters) + 3, dtype=torch.int32)
            b = self._static[0].shape[0]
            out = M.ItemGenerationOutput(item_ids=torch.zeros((b, self.n), dtype=torch.int64),
                                         beams=torch.zeros((b, self.n), dtype=torch.int32), count=torch.zeros(b, dtype=torch.int32),
                                         sem_ids=torch.zeros((b, self.k, H), dtype=torch.int64),
                                         log_probas=torch.zeros((b, self.k)))
            self._graph = Replay(self)
            self._captured = (out, torch.zeros_like(self.values), 1, self.filters)
            self._key = self._state_key()

    return Fake


@pytest.mark.parametrize("values,error,match", [
    ([2, 0, 0, 5], RuntimeError, "generate: 2 beam row"),
    ([0, 3, 0, 0, 5], ValueError, "generate: 3 excluded item id"),
    ([0, 4, 0, 0, 5], ValueError, "generate: 4 allowed item id"),
    ([0, 7, 0, 5], RuntimeError, r"generate\(search=\"exact\"\): 7 ")])
def test_counter_errors_are_the_eager_ones(monkeypatch, values, error, match):
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    Fake = _fake_exact_class()
    empty = torch.zeros(0)
    n_filters = len(values) - 4
    kinds = [ops.SidExclusion(empty, empty, empty), ops.SidInclusion(empty, empty, empty)]
    Fake.filters = kinds[:1] if n_filters == 1 and "excluded" in match else kinds[1:] if n_filters == 1 else []
    g = Fake(_model(), _batch())
    reads = []
    monkeypatch.setattr(M, "_read_search_counters", lambda v: reads.append(1) or v.tolist())
    g.values.copy_(torch.tensor(values))
    with pytest.raises(error, match=match):
        g(_batch())
    g.values.zero_()
    g.values[-1] = 9
    out = g(_batch(seed=4))
    assert torch.equal(out.item_ids, _batch(seed=4).sem_ids[:, :3])
    assert reads == [1, 1] and g.rows == 9 and g.fallbacks == 0


def test_overflow_falls_back_to_the_eager_search(monkeypatch):
    from rq_vae_recommender_b200.modules import model as M
    m = _model()
    g = _fake_exact_class()(m, _batch(), n=2, num_beams=3, exclude_history=True)
    calls = []
    eager = M.ItemGenerationOutput(*(torch.full((1,), i) for i in range(5)))
    monkeypatch.setattr(m, "generate_items", lambda batch, **kw: calls.append((batch, kw)) or eager)
    g.values.copy_(torch.tensor([0, 0, 1, 40]))
    batch = _batch(seed=5)
    assert g(batch) is eager
    assert g.fallbacks == 1 and g.rows == 40
    (got, kw), = calls
    assert got is batch
    assert kw == dict(n=2, search="exact", encoder="fused", decoder="fused", encoder_attention=g.attention, exclude_items=None,
                      exclude_history=True, include_items=None, num_beams=3)
    g.values[2] = 0                                            # a replay that fits is returned, not rerun
    g(batch)
    assert g.fallbacks == 1 and len(calls) == 1
