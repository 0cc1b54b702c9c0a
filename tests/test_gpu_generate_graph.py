"""GPU tests of EncoderDecoderRetrievalModel.capture_generate_items: generate_items(encoder="fused", decoder="fused") replayed as
one CUDA graph.  A replay equals the eager call bit for bit when every history position is unmasked, and to 1e-5 in log_probas
with the same beams when histories are padded (the encoder's GEMMs then run B * S capacity rows instead of N).  Sampled replays
consume the generator as eager calls do; in-place weight updates are followed; a changed corpus recaptures; errors come from one
host read with the eager texts; capture and replay run on side streams; the capacity rows of the encoder stay zero.
A small random model on a 12 101-row corpus.  `pytest -m gpu`."""
import contextlib
import re

import numpy as np
import pytest
import torch

from test_gpu_exclusion import dedup_ranks
from test_gpu_generate import dev, realistic_corpus, small_model
from test_gpu_inclusion import allow_lists

pytestmark = pytest.mark.gpu

K, H, N_CORPUS, ITEMS = 256, 3, 12101, 10


@pytest.fixture(scope="module")
def corpus():
    return realistic_corpus(np.random.RandomState(12101), N_CORPUS, H, K)


@pytest.fixture(scope="module")
def model(corpus):
    from rq_vae_recommender_b200.modules import model as M
    return small_model(M, corpus, K, H)


def batch_of(rs, corpus, B, users=True, padded=True, items=ITEMS):
    """B histories of corpus items (H ids + dedup rank each).  padded: leading items masked, a different count per history,
    and (B > 1) one history with every position masked."""
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    full = np.concatenate([corpus, dedup_ranks(corpus)[:, None]], axis=1)
    hist = rs.randint(0, len(corpus), size=(B, items))
    mask = np.ones((B, items), dtype=bool)
    if padded:
        for b in range(B):
            mask[b, :rs.randint(1, items)] = False
        if B > 1:
            mask[B - 1] = False
    w = H + 1
    return TokenizedSeqBatch(user_ids=dev(rs.randint(0, 100, size=(B, 1))) if users else None,
                             sem_ids=dev(full[hist].reshape(B, items * w)), sem_ids_fut=dev(full[hist[:, -1]]),
                             seq_mask=dev(np.repeat(mask, w, axis=1)), token_type_ids=dev(np.tile(np.arange(w), (B, items))),
                             token_type_ids_fut=dev(np.tile(np.arange(w), (B, 1))))


def eager(m, batch, seed=None, **kw):
    if seed is not None:
        torch.manual_seed(seed)
    return m.generate_items(batch, encoder="fused", decoder="fused", **kw)


def replay(g, batch, seed=None, **kw):
    if seed is not None:
        torch.manual_seed(seed)
    return g(batch, **kw)


def assert_same(got, want, exact=True):
    for name in ("item_ids", "beams", "count", "sem_ids"):
        assert torch.equal(getattr(got, name), getattr(want, name)), name
    if exact:
        assert torch.equal(got.log_probas, want.log_probas)
    else:
        fin = torch.isfinite(want.log_probas)
        assert torch.equal(torch.isfinite(got.log_probas), fin)
        torch.testing.assert_close(got.log_probas[fin], want.log_probas[fin], rtol=0, atol=1e-5)


@contextlib.contextmanager
def highest(on=True):
    """fp32 GEMMs (no TF32) while padded histories are compared: the capacity rows change the encoder GEMMs' row count."""
    prev = torch.get_float32_matmul_precision()
    if on:
        torch.set_float32_matmul_precision("highest")
    try:
        yield
    finally:
        torch.set_float32_matmul_precision(prev)


# (filter, user rows, padded histories)
VARIANTS = [("none", True, False), ("exclude_history", False, False), ("include", True, True), ("none", False, True),
            ("exclude_history", True, True)]


@pytest.mark.parametrize("search", ["beam", "sample"])
@pytest.mark.parametrize("w", [1, 10, 64])
@pytest.mark.parametrize("B", [1, 7, 64])
def test_replay_equals_eager(model, corpus, B, w, search):
    """Full histories: every output bit for bit.  Padded ones, under "highest" precision: the same beams and items, log_probas
    within 1e-5.  w = 64 runs the cluster selection kernels."""
    rs = np.random.RandomState(B * 100 + w)
    for filt, users, padded in VARIANTS:
        batch = batch_of(rs, corpus, B, users=users, padded=padded)
        kw = dict(search=search, num_beams=w, exclude_history=filt == "exclude_history")
        inc = dict(include_items=dev(allow_lists(rs, corpus, max(B, 2), 256)[:B])) if filt == "include" else {}
        with highest(padded):
            g = model.capture_generate_items(batch, **kw, **inc)
            want = eager(model, batch, seed=7, **kw, **inc)
            got = replay(g, batch, seed=7, **inc)
        assert got.sem_ids.shape == (B, w, H) and got.item_ids.shape == (B, w)
        assert_same(got, want, exact=not padded)
        # a second batch of the same shapes through the same graph
        batch2 = batch_of(rs, corpus, B, users=users, padded=padded)
        with highest(padded):
            assert_same(replay(g, batch2, seed=8, **inc), eager(model, batch2, seed=8, **kw, **inc), exact=not padded)


def test_results_are_the_callers(model, corpus):
    """A later call does not overwrite an earlier result."""
    rs = np.random.RandomState(1)
    a, b = batch_of(rs, corpus, 7, padded=False), batch_of(rs, corpus, 7, padded=False)
    g = model.capture_generate_items(a, search="beam")
    out_a = g(a)
    keep = out_a.item_ids.clone()
    out_b = g(b)
    assert torch.equal(out_a.item_ids, keep) and not torch.equal(out_a.item_ids, out_b.item_ids)


@pytest.mark.parametrize("w", [10, 64])
def test_sampled_replays_follow_the_generator(model, corpus, w):
    """After manual_seed(s), three consecutive replays equal three consecutive eager calls; capturing does not move the
    generator."""
    rs = np.random.RandomState(2)
    batch = batch_of(rs, corpus, 7, padded=False)
    torch.manual_seed(11)
    state = torch.cuda.get_rng_state()
    g = model.capture_generate_items(batch, search="sample", num_beams=w)
    assert torch.equal(torch.cuda.get_rng_state(), state)
    torch.manual_seed(4)
    want = [eager(model, batch, search="sample", num_beams=w) for _ in range(3)]
    torch.manual_seed(4)
    got = [g(batch) for _ in range(3)]
    for a, b in zip(got, want):
        assert_same(a, b)
    assert not torch.equal(want[0].sem_ids, want[1].sem_ids)


def test_in_place_weight_updates_are_followed(model, corpus):
    """An in-place change of a concatenated weight (encoder q, decoder cross k) and of a head, and a load_state_dict, are
    followed without recapture."""
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(3)
    m = small_model(M, corpus, K, H, seed=5)
    other = small_model(M, corpus, K, H, seed=6)
    batch = batch_of(rs, corpus, 7, padded=False)
    g = m.capture_generate_items(batch, search="beam")
    before = g(batch)
    key = g._key
    with torch.no_grad():
        m.encoder.encoder.block[0].layer[0].SelfAttention.q.weight.mul_(3)
        m.t5_decoder.block[1].layer[1].EncDecAttention.k.weight.add_(0.5)
        m.decoder_mlp[2].weight.mul_(4)
    after = g(batch)
    assert g._key is key                                                      # no recapture
    assert_same(after, eager(m, batch, search="beam"))
    assert not torch.equal(after.log_probas, before.log_probas)
    weights = {k: v for k, v in other.state_dict().items() if k != "codebooks"}
    m.load_state_dict(weights, strict=False)
    assert_same(g(batch), eager(m, batch, search="beam"))
    assert g._key is key


def test_changed_corpus_recaptures(model, corpus):
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(4)
    m = small_model(M, corpus, K, H, seed=7)
    batch = batch_of(rs, corpus, 7, padded=False)
    g = m.capture_generate_items(batch, search="beam", exclude_history=True)
    g(batch)
    key = g._key
    new = realistic_corpus(np.random.RandomState(99), N_CORPUS, H, K)
    m.codebooks.copy_(torch.from_numpy(new))                                  # written to: _version moves
    got = g(batch)
    assert g._key != key
    assert_same(got, eager(m, batch, search="beam", exclude_history=True))
    m.codebooks = torch.from_numpy(corpus).cuda()                             # replaced
    got = g(batch)
    assert_same(got, eager(m, batch, search="beam", exclude_history=True))


def test_only_the_counter_read_synchronises(model, corpus):
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(5)
    batch = batch_of(rs, corpus, 7)
    exclude = dev(rs.randint(-1, N_CORPUS, size=(7, 5)))
    g = model.capture_generate_items(batch, search="sample", num_beams=64, exclude_items=exclude, exclude_history=True)
    g(batch, exclude_items=exclude)                                                 # warm
    read = M._read_search_counters
    reads = []

    def allowed(values):
        reads.append(1)
        torch.cuda.set_sync_debug_mode(0)
        try:
            return read(values)
        finally:
            torch.cuda.set_sync_debug_mode("error")

    torch.cuda.synchronize()
    M._read_search_counters = allowed
    torch.cuda.set_sync_debug_mode("error")
    try:
        with pytest.raises(RuntimeError):
            read(torch.zeros(2, dtype=torch.int32, device="cuda"))                 # the mode is on: an unmarked read raises
        out = g(batch, exclude_items=exclude)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        M._read_search_counters = read
    assert reads == [1] and out.item_ids.shape == (7, 64)


def _eager_error(fn, kind):
    with pytest.raises(kind) as err:
        fn()
    return str(err.value)


@pytest.mark.parametrize("search", ["beam", "sample"])
def test_non_finite_head_row_raises_the_eager_error(corpus, search):
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(6)
    m = small_model(M, corpus, K, H, seed=8)
    batch = batch_of(rs, corpus, 7)
    g = m.capture_generate_items(batch, search=search)
    with torch.no_grad():
        m.decoder_mlp[1].weight[0] = float("nan")                              # every level-1 row's logit of code 0
    text = _eager_error(lambda: eager(m, batch, search=search), RuntimeError)
    with pytest.raises(RuntimeError, match=re.escape(text)):
        g(batch)


@pytest.mark.parametrize("kind", ["exclude_items", "include_items"])
def test_filter_id_out_of_range_raises_the_eager_error(model, corpus, kind):
    rs = np.random.RandomState(7)
    batch = batch_of(rs, corpus, 7, padded=False)
    items = dev(rs.randint(-1, N_CORPUS, size=(7, 6)))
    g = model.capture_generate_items(batch, search="beam", **{kind: items})
    bad = items.clone()
    bad[2, 3] = N_CORPUS + 5
    bad[4, 0] = -7
    text = _eager_error(lambda: eager(model, batch, search="beam", **{kind: bad}), ValueError)
    with pytest.raises(ValueError, match=re.escape(text)):
        g(batch, **{kind: bad})
    assert_same(g(batch, **{kind: items}), eager(model, batch, search="beam", **{kind: items}))


def test_mismatched_inputs_raise_before_any_launch(model, corpus):
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(8)
    batch = batch_of(rs, corpus, 7)
    g = model.capture_generate_items(batch, search="beam", exclude_items=dev(rs.randint(0, N_CORPUS, size=(7, 4))))

    class NoReplay:
        def replay(self):
            raise AssertionError("replayed")

    g._graph = NoReplay()
    launches = ops.LAUNCHES
    wrong = [(batch_of(rs, corpus, 6), dict(exclude_items=dev(rs.randint(0, N_CORPUS, size=(6, 4))))),
             (batch_of(rs, corpus, 7, items=ITEMS + 1), dict(exclude_items=dev(rs.randint(0, N_CORPUS, size=(7, 4))))),
             (batch_of(rs, corpus, 7, users=False), dict(exclude_items=dev(rs.randint(0, N_CORPUS, size=(7, 4))))),
             (batch, dict(exclude_items=dev(rs.randint(0, N_CORPUS, size=(7, 5))))),
             (batch, dict(exclude_items=dev(rs.randint(0, N_CORPUS, size=(7, 4))).int())),
             (batch, {}),
             (batch, dict(exclude_items=dev(rs.randint(0, N_CORPUS, size=(7, 4))),
                          include_items=dev(rs.randint(0, N_CORPUS, size=(7, 4)))))]
    for b, kw in wrong:
        with pytest.raises(ValueError, match="must match the captured call"):
            g(b, **kw)
    assert ops.LAUNCHES == launches


@pytest.mark.parametrize("search,w", [("beam", 10), ("sample", 64)])
def test_side_stream(model, corpus, search, w):
    """Capture and replay on a side stream; and a graph captured on the default stream replayed on a side stream."""
    rs = np.random.RandomState(9)
    batch = batch_of(rs, corpus, 7, padded=False)
    want = eager(model, batch, seed=3, search=search, num_beams=w)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        g = model.capture_generate_items(batch, search=search, num_beams=w)
        got = replay(g, batch, seed=3)
    torch.cuda.current_stream().wait_stream(side)
    assert_same(got, want)
    g2 = model.capture_generate_items(batch, search=search, num_beams=w)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = replay(g2, batch, seed=3)
    torch.cuda.current_stream().wait_stream(side)
    assert_same(got, want)


@pytest.mark.parametrize("attention", ["fp32", "tf32"])
@pytest.mark.parametrize("users", [True, False])
def test_capacity_rows_are_zero(model, corpus, attention, users):
    """FusedT5Encode(capacity=True): B * S packed rows; rows past N are exactly zero with src -1; rows below N are the eager
    pass's (to GEMM rounding), and the scattered [B, S, d] output likewise."""
    from rq_vae_recommender_b200.modules import model as M
    from rq_vae_recommender_b200.modules.model import _strip_dedup_col
    rs = np.random.RandomState(10)
    batch = batch_of(rs, corpus, 9, users=users)
    mask, ids = _strip_dedup_col(batch.seq_mask.long(), H + 1, H), _strip_dedup_col(batch.sem_ids, H + 1, H)
    with torch.no_grad(), highest():
        cap = M.FusedT5Encode(model, attention, capacity=True).packed(mask, ids, batch.user_ids)
        ref = M.FusedT5Encode(model, attention).packed(mask, ids, batch.user_ids)
        out_cap = M.FusedT5Encode(model, attention, capacity=True)(mask, ids, batch.user_ids)[0]
        out_ref = M.FusedT5Encode(model, attention)(mask, ids, batch.user_ids)[0]
    B, S = cap.slot.shape
    N = int(ref.offsets[-1])
    assert cap.rows.shape == (B * S, model.t5_decoder.config.d_model) and N < B * S
    assert torch.equal(cap.offsets, ref.offsets) and torch.equal(cap.slot, ref.slot)
    assert torch.equal(cap.src[:N], ref.src) and bool((cap.src[N:] == -1).all())
    assert bool(torch.isfinite(cap.rows).all()) and bool((cap.rows[N:] == 0).all())
    # TF32 attention rounds its inputs to 10-bit mantissas, so the GEMMs' last-bit differences can move its products by 1e-4
    atol = 1e-5 if attention == "fp32" else 1e-3
    torch.testing.assert_close(cap.rows[:N], ref.rows, rtol=0, atol=atol)
    torch.testing.assert_close(out_cap, out_ref, rtol=0, atol=atol)
