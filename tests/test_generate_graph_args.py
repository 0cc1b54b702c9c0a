"""CPU-only: capture_generate_items refuses what a CUDA graph cannot run (search="exact", HF passes, training mode, autocast)
before any launch, and GenerateItemsGraph's bookkeeping -- input checks before any replay, copies into the static buffers,
results the caller owns, recapture when the corpus changes, and the eager errors from its one counter read -- on a fake graph."""
import numpy as np
import pytest
import torch

K, H, B, ITEMS = 64, 3, 2, 4


def _model():
    from rq_vae_recommender_b200.modules import model as M
    corpus = np.random.RandomState(0).randint(0, K, size=(50, H)).astype(np.int64)
    torch.manual_seed(0)
    return M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), num_hierarchies=H, num_embeddings_per_hierarchy=K,
                                          t5_d_model=64, t5_num_heads=2, t5_d_ff=128, t5_num_layers=2, top_k_for_generation=3,
                                          should_add_sep_token=True, num_user_bins=11).eval()


def _batch(b=B, items=ITEMS, users=True, seed=0):
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    g = torch.Generator().manual_seed(seed)
    sem = torch.randint(0, K, (b, items * (H + 1)), generator=g)
    return TokenizedSeqBatch(user_ids=torch.zeros((b, 1), dtype=torch.int64) if users else None, sem_ids=sem, sem_ids_fut=None,
                             seq_mask=torch.ones_like(sem, dtype=torch.bool), token_type_ids=None, token_type_ids_fut=None)


@pytest.mark.parametrize("kw,match", [(dict(search="exact"), "exact"), (dict(encoder="hf"), "fused encoder and decoder"),
                                      (dict(decoder="hf"), "fused encoder and decoder"), (dict(search="greedy"), "search must be"),
                                      (dict(encoder_attention="bf16"), "encoder_attention must be")])
def test_refused_arguments(kw, match):
    from rq_vae_recommender_b200 import ops
    m = _model()
    launches = ops.LAUNCHES
    with pytest.raises(ValueError, match=match):
        m.capture_generate_items(_batch(), **kw)
    assert ops.LAUNCHES == launches


def test_training_mode_and_autocast_are_refused(monkeypatch):
    from rq_vae_recommender_b200.modules import model as M
    m = _model().train()
    with pytest.raises(ValueError, match="eval mode only"):
        m.capture_generate_items(_batch())
    m.eval()
    monkeypatch.setattr(M.torch, "is_autocast_enabled", lambda *a: True)
    with pytest.raises(ValueError, match="autocast"):
        m.capture_generate_items(_batch())


def test_width_limits_are_the_searchs():
    from rq_vae_recommender_b200._lib import Rqb200Error
    m = _model()
    with pytest.raises(Rqb200Error, match="num_beams = 65"):
        m.capture_generate_items(_batch(), search="beam", num_beams=65)


def _fake_graph_class():
    """GenerateItemsGraph with the capture replaced by a fake graph: a replay writes sem_ids[:, :n] to item_ids and the counters
    set in ``counters``."""
    from rq_vae_recommender_b200.modules import model as M

    class Replay:
        def __init__(self, g):
            self.g, self.replays = g, 0

        def replay(self):
            self.replays += 1
            out, values = self.g._captured[:2]
            out.item_ids.copy_(self.g._static[0][:, :self.g.n])
            values.copy_(self.g.counters)

    class Fake(M.GenerateItemsGraph):
        captures = 0
        filters = []

        def _capture(self):
            self.captures += 1
            n_counters = 1 if self.search == "beam" else 2
            self.counters = torch.zeros(n_counters + len(self.filters), dtype=torch.int32)
            b = self._static[0].shape[0]
            out = M.ItemGenerationOutput(item_ids=torch.zeros((b, self.n), dtype=torch.int64),
                                         beams=torch.zeros((b, self.n), dtype=torch.int32), count=torch.zeros(b, dtype=torch.int32),
                                         sem_ids=torch.zeros((b, self.k, H), dtype=torch.int64),
                                         log_probas=torch.zeros((b, self.k)))
            self._graph = Replay(self)
            self._captured = (out, torch.zeros_like(self.counters), n_counters, self.filters)
            self._key = self._state_key()

    return Fake


def test_inputs_are_checked_before_any_replay():
    m = _model()
    Fake = _fake_graph_class()
    g = Fake(m, _batch(), None, "beam", None, None, torch.zeros((B, 5), dtype=torch.int64), None, None)
    for batch, kw in [(_batch(b=B + 1), dict(exclude_items=torch.zeros((B + 1, 5), dtype=torch.int64))),
                      (_batch(items=ITEMS + 1), dict(exclude_items=torch.zeros((B, 5), dtype=torch.int64))),
                      (_batch(users=False), dict(exclude_items=torch.zeros((B, 5), dtype=torch.int64))),
                      (_batch(), dict(exclude_items=torch.zeros((B, 6), dtype=torch.int64))),
                      (_batch(), dict(exclude_items=torch.zeros((B, 5), dtype=torch.int32))),
                      (_batch(), {}),
                      (_batch(), dict(exclude_items=torch.zeros((B, 5), dtype=torch.int64),
                                      include_items=torch.zeros((B, 5), dtype=torch.int64)))]:
        with pytest.raises(ValueError, match="must match the captured call"):
            g(batch, **kw)
    assert g._graph.replays == 0 and g.captures == 1


def test_inputs_are_copied_and_results_are_the_callers():
    m = _model()
    g = _fake_graph_class()(m, _batch(seed=1), None, "beam", None, None, None, None, None)
    a, b = _batch(seed=2), _batch(seed=3)
    out_a = g(a)
    assert torch.equal(out_a.item_ids, a.sem_ids[:, :3])
    out_b = g(b)
    assert torch.equal(out_a.item_ids, a.sem_ids[:, :3]) and torch.equal(out_b.item_ids, b.sem_ids[:, :3])
    assert out_a.item_ids.data_ptr() != g._captured[0].item_ids.data_ptr()
    assert g.captures == 1 and g._graph.replays == 2


def test_changed_corpus_or_moved_parameter_recaptures():
    m = _model()
    g = _fake_graph_class()(m, _batch(), None, "beam", None, None, None, None, None)
    g(_batch())
    with torch.no_grad():
        m.decoder_mlp[0].weight.mul_(2)                       # in place: followed by the graph, no recapture
    g(_batch())
    assert g.captures == 1
    m.codebooks.add_(0)                                       # written to
    g(_batch())
    assert g.captures == 2
    m.codebooks = m.codebooks.clone()                         # replaced
    g(_batch())
    assert g.captures == 3
    m.decoder_mlp[0].weight.data = m.decoder_mlp[0].weight.data.clone()   # storage moved
    g(_batch())
    assert g.captures == 4
    g(_batch())
    assert g.captures == 4


@pytest.mark.parametrize("search,counters,error,match", [
    ("beam", [2], RuntimeError, "generate: 2 beam row"),
    ("sample", [1, 0], RuntimeError, "probability tensor contains"),
    ("sample", [0, 3], RuntimeError, "invalid multinomial distribution"),
    ("beam", [0, 4], ValueError, "generate: 4 excluded item id"),
    ("sample", [1, 0, 0, 2], ValueError, "generate: 2 allowed item id")])
def test_counter_errors_are_the_eager_ones(monkeypatch, search, counters, error, match):
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    m = _model()
    Fake = _fake_graph_class()
    n_filters = len(counters) - (1 if search == "beam" else 2)
    empty = torch.zeros(0)
    Fake.filters = [ops.SidExclusion(empty, empty, empty), ops.SidInclusion(empty, empty, empty)][:n_filters]
    g = Fake(m, _batch(), None, search, None, None, None, None, None)
    reads = []
    monkeypatch.setattr(M, "_read_search_counters", lambda v: reads.append(1) or v.tolist())
    g.counters.copy_(torch.tensor(counters))
    with pytest.raises(error, match=match):
        g(_batch())
    g.counters.zero_()
    g(_batch())
    assert reads == [1, 1]
