"""Every entry point as one stream-ordered op on the caller's stream.  Serving code and data loaders call the library on side
streams; on the default stream a launch on the wrong stream still runs in order, so only a side stream can show one.

A. Late inputs: each case's inputs are filled on a side stream s with a valid decoy, then overwritten with the real inputs behind a
   ~75 ms ``torch.cuda._sleep`` on s; the call runs under ``torch.cuda.stream(s)``.  A launch on any other stream reads the decoy
   and returns another (valid) answer.  Results must equal the default-stream run: bit for bit where two default-stream runs are
   bit-identical, integers always, and otherwise within the bound of the case's float64 test.
B. Cached device state (prepared codebooks, operand images, tries, item tables) built on one stream and fetched from another:
   the getter must order the fetching stream after the build, and an evicted entry's memory must not be reused while a
   stream that fetched it still reads it.  No consumer kernel ever runs on an entry that may be unbuilt.
C. Inputs on cuda:1 while cuda:0 is current with a side stream (two GPUs; skipped otherwise).
D. ``CorpusTokenizer.tokenize_host``: the host-in, host-out pipeline against ``tokenize_device`` and the float64 oracle.
`pytest -m gpu`."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import inputs as I
from oracle import rq_oracle as O
from parity import assert_ids_match

pytestmark = pytest.mark.gpu
SEED = 1234
SLEEP_MS = 75


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def cycles():
    """``torch.cuda._sleep`` cycles of about SLEEP_MS, measured once with CUDA events on the default stream."""
    torch.cuda._sleep(1000)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    probe = 10_000_000
    e0.record()
    torch.cuda._sleep(probe)
    e1.record()
    torch.cuda.synchronize()
    return max(int(probe * SLEEP_MS / e0.elapsed_time(e1)), probe)


def late_inputs(s, real, decoy, cycles):
    """Buffers allocated on s holding ``decoy`` (synchronised), then overwritten on s with ``real`` behind a sleep."""
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        late = [d.clone() for d in decoy]
    s.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(cycles)
        for t, r in zip(late, real):
            t.copy_(r)
    return late


class Atomic(list):
    """A case's floating-point outputs that are sums in atomic order (atomicAdd in csrc/: the codebook gradients of the chain
    and of the Gumbel level, k-means' fp64 sums, the dedup entropy): their last bits change from run to run."""


def tensors_of(out, atomic=False):
    """[(tensor, atomic)] of a case's outputs, in order."""
    if isinstance(out, torch.Tensor):
        return [(out, atomic)]
    atomic = atomic or isinstance(out, Atomic)
    if isinstance(out, dict):
        return [p for v in out.values() for p in tensors_of(v, atomic)]
    if isinstance(out, (tuple, list)):
        return [p for v in out for p in tensors_of(v, atomic)]
    assert out is None or isinstance(out, (int, float, bool)), type(out)
    return []


def run(fn, inputs):
    torch.manual_seed(SEED)
    return [(t.detach().clone(), atomic) for t, atomic in tensors_of(fn(*inputs))]


def rel(a, b):
    a, b = a.double(), b.double()
    fin = torch.isfinite(b)
    assert torch.equal(fin, torch.isfinite(a)) and torch.equal(a[~fin], b[~fin])
    return ((a[fin] - b[fin]).abs().max() / b[fin].abs().max().clamp_min(1e-30)).item() if fin.any() else 0.0


#: bounds of the float64 tests, relative to the largest entry, for the ``Atomic`` outputs: k-means' fp64 sums (1e-12,
#: test_gpu_train_chain's k-means test) and the training chain's fp32 gradients (2e-5, its ``close``).  Reordering an n-term fp32
#: sum moves it by at most 2 (n - 1) u sum|terms| (u = 2^-24); these sums take at most a few hundred terms of one sign pattern, a
#: few ulps in practice -- far inside 2e-5 -- while a read of the decoy changes them at the first digit.
TOL = {torch.float64: 1e-12, torch.float32: 2e-5}


def assert_stream_ordered(fn, make, cycles):
    """fn(*make(0)) under a side stream whose inputs arrive late equals fn(*make(0)) on the default stream: bit for bit, except
    the outputs the case marks ``Atomic``, which are within TOL.  Every other output must repeat bit for bit on the default
    stream too."""
    real, decoy = make(0), make(1)
    want, again = run(fn, real), run(fn, real)
    other = run(fn, decoy)
    assert any(not torch.equal(a, b) for (a, _), (b, _) in zip(want, other)), "the decoy must change the result"
    s = torch.cuda.Stream()
    late = late_inputs(s, real, decoy, cycles)
    with torch.cuda.stream(s):
        got = run(fn, late)
    s.synchronize()
    assert len(got) == len(want)
    for i, ((g, _), (w, atomic), (w2, _)) in enumerate(zip(got, want, again)):
        assert g.shape == w.shape and g.dtype == w.dtype, i
        if atomic:
            assert w.is_floating_point(), f"output {i}: integer outputs are exact"
            assert rel(w2, w) <= TOL[w.dtype] and rel(g, w) <= TOL[w.dtype], f"output {i} differs on the side stream"
        else:
            assert torch.equal(w, w2), f"output {i} differs between two default-stream runs and is not marked Atomic"
            assert torch.equal(g, w), f"output {i} differs on the side stream"


def test_negative_control_default_stream_reads_the_decoy(cycles):
    """The sleep covers the window: a plain torch op enqueued on the default stream while the inputs are late sees the decoy,
    the same op on the side stream the real inputs."""
    real = torch.arange(4096, dtype=torch.float32, device="cuda")
    real * 2                                                                   # loads the kernel: a module load syncs the device
    s = torch.cuda.Stream()
    late = late_inputs(s, [real], [-real], cycles)[0]
    early = late * 2
    with torch.cuda.stream(s):
        ordered = late * 2
    torch.cuda.synchronize()
    assert torch.equal(early, -2 * real) and torch.equal(ordered, 2 * real)


# ------------------------------------------------------------------------------------------------ A. late inputs, per family
def rq_inputs(n, d, k, L):
    def make(seed):
        x, cbs = I.rq_problem(n, d, k, L, seed=seed + 40)
        return [dev(x)] + [dev(c) for c in cbs]
    return make


def grads(*ts):
    return [t.grad for t in ts]


def chain_fn(mode):
    def fn(x, *cbs):
        from rq_vae_recommender_b200 import ops
        x = x.detach().requires_grad_()
        cs = [c.detach().requires_grad_() for c in cbs]
        esum, norms, ids, loss = ops.RqChainFunction.apply(x, mode, 0.25, True, *cs)
        (esum.square().sum() + loss.sum()).backward()
        return esum, norms, ids, loss, x.grad, Atomic(grads(*cs))
    return fn


def gumbel_fn(x, cb, u):
    from rq_vae_recommender_b200 import ops
    x, cb = x.detach().requires_grad_(), cb.detach().requires_grad_()
    emb, ids, loss = ops.GumbelQuantizeFunction.apply(x, cb, u, 0.5, 0.25)
    (emb.square().sum() + loss.sum()).backward()
    return emb, ids, loss, x.grad, Atomic([cb.grad])


def gumbel_make(seed):
    rs = np.random.RandomState(seed)
    B, D, K = 640, 64, 128
    return [dev(rs.randn(B, D).astype(np.float32)), dev(rs.randn(K, D).astype(np.float32) * 0.3),
            dev(0.01 + 0.98 * rs.rand(B, K).astype(np.float32))]


def l2norm_fn(x, g):
    from rq_vae_recommender_b200 import ops
    x = x.detach().requires_grad_()
    y = ops.L2NormFunction.apply(x, 1e-12)
    (y * g).sum().backward()
    return y, x.grad, ops.l2norm_rows(g)


def mlp_make(seed):
    rs = np.random.RandomState(seed)
    return [dev(rs.randn(640, 96).astype(np.float32))] + [dev(w) for w in I.mlp_weights(seed + 7, [96, 128, 64])]


def mlp_fn(x, *ws):
    from rq_vae_recommender_b200 import ops
    x = x.detach().requires_grad_()
    ws = [w.detach().requires_grad_() for w in ws]
    y = ops.MLPFunction.apply(x, True, *ws)
    y2 = ops.MLPFunction.apply(x[:100], False, *ws)                              # below SPLIT_MIN_ROWS: the CUDA-core GEMMs
    (y.square().sum() + y2.sum()).backward()
    return y, y2, grads(x, *ws)


def gemm_make(seed):
    rs = np.random.RandomState(seed)
    return [dev(rs.randn(600, 80).astype(np.float32)), dev(rs.randn(200, 80).astype(np.float32)),
            dev(rs.randn(600, 48).astype(np.float32))]


def gemm_fn(a, b, c):
    from rq_vae_recommender_b200 import ops
    return (ops.sgemm(a, b, trans_b=True, relu=True), ops.gemm_split(a, b), ops.gemm_tn(a, c), ops.gemm_tn(a[:100], c[:100]),
            ops.linear_nt(a, b), ops.linear_nt(a, b.t(), w_transposed=True))


def bf16_make(seed):
    rs = np.random.RandomState(seed)
    return [dev(rs.randn(300, 128).astype(np.float32))] + [dev(w) for w in I.mlp_weights(seed + 3, [128, 128, 64])]


def bf16_fn(x, *ws):
    from rq_vae_recommender_b200 import ops
    return ops.mlp_forward_bf16(x, ws, normalize=True)


def kmeans_make(seed):
    rs = np.random.RandomState(seed)
    x = rs.randn(700, 32).astype(np.float32)
    return [dev(x), dev(x[rs.choice(700, 64, replace=False)])]


def kmeans_fn(x, cent):
    from rq_vae_recommender_b200 import ops
    buf = ops.kmeans_workspace(x, 64)
    ops.kmeans_assign_accumulate(x, cent, buf)
    c = cent.clone()
    ops.kmeans_finalize(x, c, buf, None)
    return buf["assign"], buf["counts"], Atomic([buf["sums"], c, buf["shift"]])


def sid_stats_make(seed):
    rs = np.random.RandomState(seed)
    return [dev(rs.randint(0, 16, size=(500, 3))), dev(rs.randint(0, 500, size=(6, 9))), dev(rs.rand(6, 9) > 0.3)]


def sid_stats_fn(ids, items, mask):
    from rq_vae_recommender_b200 import ops
    rank, stats = ops.sid_dedup_rank(ids, 16)
    return (ops.sid_histogram(ids, 16), rank, stats["max_rank"], stats["n_unique"], Atomic([stats["entropy"]]),
            ops.sid_gather(ids, items, mask))


K_SEARCH, H_SEARCH, B_SEARCH, BEAMS = 256, 3, 8, 10


def search_make(seed):
    from test_gpu_generate import realistic_corpus
    rs = np.random.RandomState(seed + 60)
    corpus = realistic_corpus(rs, 3000, H_SEARCH, K_SEARCH)
    logits0 = rs.randn(B_SEARCH, K_SEARCH).astype(np.float32) * 2
    logits0[:, np.unique(corpus[:, 0])] += 3
    logits1 = rs.randn(B_SEARCH * BEAMS, K_SEARCH).astype(np.float32) * 4
    noise = rs.exponential(size=(B_SEARCH, K_SEARCH)).astype(np.float32)
    prefix = corpus[rs.randint(0, 3000, size=200), :2].copy()
    prefix[::3, 1] = rs.randint(0, K_SEARCH, size=len(prefix[::3]))
    ok = ((corpus >= 0) & (corpus < K_SEARCH)).all(1)
    leaf_key = np.unique((corpus[ok, 0] * K_SEARCH + corpus[ok, 1]) * K_SEARCH + corpus[ok, 2])
    gen = corpus[rs.randint(0, 3000, size=(B_SEARCH, BEAMS))]
    gen[:, ::4, 2] = rs.randint(0, K_SEARCH, size=gen[:, ::4, 2].shape)
    lp = -np.sort(rs.rand(B_SEARCH, BEAMS).astype(np.float32), axis=1)
    lp[:, -1] = -np.inf
    excl = rs.randint(-1, 3000, size=(B_SEARCH, 40))
    excl[:, :10] = rs.randint(0, 3000, size=(B_SEARCH, BEAMS))
    incl = rs.randint(-1, 3000, size=(B_SEARCH, 300))
    return [dev(a) for a in (corpus, prefix, logits0, logits1, noise, leaf_key, gen, lp, excl, incl)]


def prefix_index_fn(corpus, prefix, logits0, logits1, noise, *_):
    from rq_vae_recommender_b200 import ops
    idx = ops.SidPrefixIndex(corpus, K_SEARCH)
    valid = idx.check(prefix)
    g, p, par = idx.beam_topk(logits0, None, None, BEAMS)
    g1, p1, par1 = idx.beam_topk(logits1, g, p, BEAMS)
    sel = idx.sample_select(F.softmax(logits0, -1), noise, None, None, BEAMS, 64, want_samples=True)
    sel1 = idx.sample_select(F.softmax(logits1, -1), noise.repeat(BEAMS, 1), g, p, BEAMS, 16)
    bsel = idx.beam_select(sel[3], sel[4], None, None, BEAMS)
    n = idx.counts()
    return valid, g, p, par, g1, p1, par1, sel, sel1, bsel, n


def item_table_fn(corpus, prefix, logits0, logits1, noise, leaf_key, gen, lp, *_):
    from rq_vae_recommender_b200 import ops
    table = ops.SidItemTable(corpus, K_SEARCH)
    ded = torch.cat([gen, (gen[..., :1] % 3)], -1)
    return table.lookup(gen), table.lookup(ded, with_dedup=True), table.retrieve(gen, lp, 30), table.arrays()[0], table.positions()


def filters_fn(corpus, prefix, logits0, logits1, noise, leaf_key, gen, lp, excl, incl):
    from rq_vae_recommender_b200 import ops
    table, idx = ops.SidItemTable(corpus, K_SEARCH), ops.SidPrefixIndex(corpus, K_SEARCH)
    ex = ops.sid_exclusion_build(excl, table, leaf_key)
    inc = ops.sid_inclusion_build(incl, table, leaf_key, exclude=ex)
    out = [ex, inc]
    for f in ({"exclude": ex}, {"include": inc}):
        g, p, par = idx.beam_topk(logits0, None, None, BEAMS, **f)
        out += [g, p, par, idx.beam_topk(logits1, g, p, BEAMS, **f)]
        out.append(idx.sample_select(F.softmax(logits0, -1), noise, None, None, BEAMS, 64, **f))
        out.append(table.retrieve(gen, lp, 30, **f))
    return out


def rank_hist_make(seed):
    rs = np.random.RandomState(seed)
    cand = rs.randint(0, 4, size=(50, 10, 3))
    actual = cand[np.arange(50), rs.randint(0, 12, size=50) % 10].copy()
    actual[::5] = 9
    cand[::7, 2] = -1
    return [dev(actual), dev(cand), dev(rs.randint(-1, 14, size=50))]


def rank_hist_fn(actual, cand, rank):
    from rq_vae_recommender_b200 import ops
    h1, h2, h3 = (torch.zeros(11, dtype=torch.int64, device=rank.device) for _ in range(3))
    ops.sid_topk_rank_hist(actual, cand, h1)
    ops.sid_topk_rank_hist(actual, cand, h2, item_mode=True)
    ops.sid_rank_hist(rank, h3)
    return h1, h2, h3


def tc_fn(x, *cbs):
    from rq_vae_recommender_b200 import ops
    stats = torch.zeros(4, dtype=torch.int32, device=x.device)
    return ops.rq_tokenize_tc(x, list(cbs), stats=stats), stats


def auto_fn(x, *cbs):
    from rq_vae_recommender_b200 import ops
    with torch.no_grad():
        return ops.rq_tokenize_auto(x, list(cbs)), ops.rq_tokenize_auto(x[:300], list(cbs))


def simt_fn(x, *cbs):
    from rq_vae_recommender_b200 import ops
    return ops.rq_tokenize(x, list(cbs)), ops.rq_forward(x, list(cbs), ops.MODE_EVAL, 0.25, want_embeddings=True,
                                                         want_residuals=True, want_loss=True)


KERNEL_CASES = {
    "rq_tokenize": (simt_fn, rq_inputs(300, 96, 64, 3)),
    "rq_tokenize_tc_k256": (tc_fn, rq_inputs(700, 96, 256, 3)),
    "rq_tokenize_tc_k1024": (tc_fn, rq_inputs(1100, 64, 1024, 2)),
    "rq_tokenize_auto": (auto_fn, rq_inputs(1200, 128, 256, 3)),
    "rq_chain_ste": (chain_fn(2), rq_inputs(300, 64, 64, 3)),
    "rq_chain_rot": (chain_fn(3), rq_inputs(600, 64, 128, 2)),
    "gumbel": (gumbel_fn, gumbel_make),
    "l2norm": (l2norm_fn, lambda seed: [dev(I.randn(seed + 5, 300, 48)), dev(I.randn(seed + 6, 300, 48))]),
    "mlp": (mlp_fn, mlp_make),
    "gemm": (gemm_fn, gemm_make),
    "mlp_bf16": (bf16_fn, bf16_make),
    "kmeans": (kmeans_fn, kmeans_make),
    "sid_stats": (sid_stats_fn, sid_stats_make),
    "prefix_index": (prefix_index_fn, search_make),
    "item_table": (item_table_fn, search_make),
    "filters": (filters_fn, search_make),
    "rank_hist": (rank_hist_fn, rank_hist_make),
}


@pytest.mark.parametrize("case", list(KERNEL_CASES))
def test_kernel_entry_points_run_on_the_callers_stream(case, cycles):
    assert_stream_ordered(*KERNEL_CASES[case], cycles)


# ------------------------------------------------------------------------------------------------ A. model level
@pytest.mark.parametrize("mode", ["ste", "rot", "gumbel"])
def test_rqvae_forward_backward_and_tokenize_on_the_callers_stream(mode, cycles):
    from test_gpu_modules import batch_of, build
    m = build(mode, 0)[0]

    def fn(x):
        m.zero_grad(set_to_none=True)
        fo = m(batch_of(x), 0.2)
        fo.loss.backward()
        with torch.no_grad():
            ids = m.tokenize(x)
        codebooks = [layer.embedding.weight for layer in m.layers]
        others = [p.grad for p in m.parameters() if p.grad is not None and all(p is not c for c in codebooks)]
        return tuple(fo), ids, others, Atomic([c.grad for c in codebooks])

    assert_stream_ordered(fn, lambda seed: [dev(I.randn(seed + 70, 640, 64))], cycles)


def retrieval_model():
    from rq_vae_recommender_b200.modules import model as M
    from test_gpu_generate import realistic_corpus
    from test_gpu_rank import model_for
    corpus = realistic_corpus(np.random.RandomState(21), 3000, 3, 256)
    corpus[100:104] = corpus[105]
    return model_for(M, corpus, 256, 3), corpus


def batch_make(corpus, B=12, items=6):
    from test_gpu_rank import batch_for

    def make(seed):
        rs = np.random.RandomState(seed + 80)
        b = batch_for(rs, corpus, B, items, 3, 256)
        return list(b) + [dev(rs.randint(-1, len(corpus), size=(B, 40)))]
    return make


def batch_of_inputs(t):
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    return TokenizedSeqBatch(*t[:6]), t[6]


@pytest.mark.parametrize("search", ["sample", "beam"])
@pytest.mark.parametrize("encoder,decoder,attention", [("hf", "fused", None), ("fused", "hf", "fp32"), ("fused", "fused", "tf32")])
def test_generate_on_the_callers_stream(search, encoder, decoder, attention, cycles):
    from test_gpu_generate import history
    m, _ = retrieval_model()

    def fn(mask, ids, users):
        return m.generate(mask, ids, users, search=search, decoder=decoder, encoder=encoder, encoder_attention=attention)

    assert_stream_ordered(fn, lambda seed: list(history(np.random.RandomState(seed + 90), 12, 6, 3, 256)), cycles)


def test_generate_items_rank_and_score_on_the_callers_stream(cycles):
    m, corpus = retrieval_model()

    def fn(*t):
        batch, items = batch_of_inputs(t)
        ex = m.generate_items(batch, n=20, search="beam", decoder="fused", encoder="fused", exclude_history=True)
        inc = m.generate_items(batch, n=20, search="sample", decoder="fused", encoder="hf", exclude_history=True,
                               include_items=items)
        rank = m.rank_items(batch, n=20, encoder="fused", exclude_history=True)
        score = m.score_items(batch, items)
        rank32 = m.rank_items(batch, n=20, encoder="fused", encoder_attention="tf32", attention="tf32")
        score32 = m.score_items(batch, items, encoder="fused", encoder_attention="tf32", attention="tf32")
        return ex, inc, rank, score, rank32, score32

    assert_stream_ordered(fn, batch_make(corpus), cycles)


def test_fused_training_pass_under_dropout_on_the_callers_stream(cycles):
    from test_gpu_encode_train import amazon, set_dropout, train_batch
    m = amazon()
    set_dropout(m, 0.1)

    def make(seed):
        rs = np.random.RandomState(seed + 100)
        return list(train_batch(rs, 24, 12, 3, 256, rs.randint(1, 13, size=24)))

    def fn(*t):
        from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
        m.zero_grad(set_to_none=True)
        loss = m(TokenizedSeqBatch(*t), encoder="fused", decoder="fused").loss
        loss.backward()
        return loss, [p.grad for p in m.parameters() if p.grad is not None]

    assert_stream_ordered(fn, make, cycles)


# ------------------------------------------------------------------------------------------------ B. cached state between streams
def assert_fetch_waits_for_build(cycles, warm, build, fetch, gate=True):
    """build() under stream B (behind a sleep when ``gate``), then fetch(built) -- a getter only, no consumer kernel -- under an
    idle stream C: C must not pass an event before B's build is done.  warm() first runs the same build on other objects under B:
    the first launch of a kernel loads its module, and the first allocations on a stream take new device memory; either may
    synchronise the device and finish B's build early."""
    b, c = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(b):
        warm()
    torch.cuda.synchronize()
    with torch.cuda.stream(b):
        if gate:
            torch.cuda._sleep(cycles)
        built = build()
    with torch.cuda.stream(c):
        fetch(built)
        ev = torch.cuda.Event()
        ev.record(c)
    waited = not ev.query()
    building = not b.query()
    torch.cuda.synchronize()
    assert building, "the build finished before the fetch: the case does not test anything"
    assert waited, "the fetching stream does not wait for the build on another stream"


def test_tc_state_cache_orders_a_fetching_stream_after_the_prepare(cycles):
    from rq_vae_recommender_b200 import ops
    cbs = rq_inputs(300, 96, 256, 3)(0)[1:]
    assert_fetch_waits_for_build(cycles, lambda: ops.TcState(cbs), lambda: ops.tc_state_for(cbs), lambda _: ops.tc_state_for(cbs))


def test_split_operand_cache_orders_a_fetching_stream_after_the_split(cycles):
    from rq_vae_recommender_b200 import ops
    w = dev(I.randn(3, 200, 80))
    assert_fetch_waits_for_build(cycles, lambda: ops.SplitOperand(w), lambda: ops.split_operand_cached(w),
                                 lambda _: ops.split_operand_cached(w))


def test_bf16_weight_image_cache_orders_a_fetching_stream_after_the_conversion(cycles):
    from test_gpu_modules import build
    enc = build("ste", 0, Din=128, hidden=(128,))[0].encoder
    ws = [mod.weight for mod in enc.mlp if isinstance(mod, torch.nn.Linear)]
    from rq_vae_recommender_b200 import ops
    assert_fetch_waits_for_build(cycles, lambda: [ops.to_bf16_image(w.detach()) for w in ws], lambda: enc._weight_images(ws),
                                 lambda _: enc._weight_images(ws))


def test_corpus_tokenizer_state_orders_a_fetching_stream_after_the_prepare(cycles):
    from rq_vae_recommender_b200 import parallel
    cbs = rq_inputs(300, 96, 256, 3)(0)[1:]
    make = lambda: parallel.CorpusTokenizer(cbs, use_tc=True)                  # noqa: E731
    assert_fetch_waits_for_build(cycles, make, make, lambda tok: tok.state)


@pytest.mark.parametrize("getter", ["_prefix_index", "_item_table"])
def test_model_corpus_caches_order_a_fetching_stream_after_the_build(getter, cycles):
    m, _ = retrieval_model()
    dv = torch.device("cuda", torch.cuda.current_device())
    assert_fetch_waits_for_build(cycles, lambda: getattr(retrieval_model()[0], getter)(dv), lambda: getattr(m, getter)(dv),
                                 lambda _: getattr(m, getter)(dv))


def test_rank_levels_order_a_fetching_stream_after_their_build(cycles, monkeypatch):
    """_rank_levels reads the host once in its build; the sleep gates the build after that read, in SidPrefixIndex.levels."""
    from rq_vae_recommender_b200 import ops
    (m, _), (m2, _) = retrieval_model(), retrieval_model()
    dv = torch.device("cuda", torch.cuda.current_device())
    index = m._prefix_index(dv)
    levels = ops.SidPrefixIndex.levels

    def late_levels(self, n):
        if self is index:
            torch.cuda._sleep(cycles)
        return levels(self, n)

    monkeypatch.setattr(ops.SidPrefixIndex, "levels", late_levels)
    assert_fetch_waits_for_build(cycles, lambda: m2._rank_levels(dv), lambda: m._rank_levels(dv), lambda _: m._rank_levels(dv),
                                 gate=False)


def test_index_levels_order_a_fetching_stream_after_their_build(cycles):
    from rq_vae_recommender_b200 import ops
    idx, idx2 = ops.SidPrefixIndex(search_make(0)[0], K_SEARCH), ops.SidPrefixIndex(search_make(1)[0], K_SEARCH)
    n, n2 = idx.counts().tolist(), idx2.counts().tolist()
    assert_fetch_waits_for_build(cycles, lambda: idx2.levels(n2), lambda: idx.levels(n), lambda _: idx.levels(n))


def test_item_table_and_its_positions_order_a_fetching_stream_after_their_build(cycles):
    from rq_vae_recommender_b200 import ops
    corpus, other = search_make(0)[0], search_make(1)[0]
    table, table2 = ops.SidItemTable(corpus, K_SEARCH), ops.SidItemTable(other, K_SEARCH)
    assert_fetch_waits_for_build(cycles, table2.positions, table.positions, lambda _: table.positions())
    make = lambda: ops.SidItemTable(corpus, K_SEARCH)                          # noqa: E731
    assert_fetch_waits_for_build(cycles, make, make, lambda t: t.arrays())


def test_evicted_split_operand_is_not_reused_while_a_stream_reads_it(cycles):
    """linear_nt behind a sleep on C takes a cached weight image built on B; the entry is evicted and B allocates and fills
    tensors of its size.  C's product must still be the default-stream one: the eviction may not hand the image's memory to B
    while C's GEMM has yet to read it."""
    from rq_vae_recommender_b200 import ops
    a, w = dev(I.randn(11, 640, 96)), dev(I.randn(12, 160, 96))
    want = ops.gemm_split(a, ops.SplitOperand(w))
    torch.empty(16, dtype=torch.uint8, device="cuda").fill_(0x3c)             # loads the fill kernel ahead of the window
    ops._SPLIT_CACHE.clear()
    torch.cuda.synchronize()
    b, c = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(b):
        nbytes = ops.split_operand_cached(w).buf.numel()
    b.synchronize()
    with torch.cuda.stream(c):
        torch.cuda._sleep(cycles)
        got = ops.linear_nt(a, w)
    others = [dev(I.randn(13 + i, 64, 64)) for i in range(ops._SPLIT_CACHE_MAX)]
    with torch.cuda.stream(b):
        for o in others:
            ops.split_operand_cached(o)
        assert not any(r() is w for r, *_ in ops._SPLIT_CACHE.values())          # evicted
        fill = [torch.empty(nbytes, dtype=torch.uint8, device="cuda").fill_(0x3c) for _ in range(32)]
    running = not c.query()
    torch.cuda.synchronize()
    assert running, "C's GEMM finished before the eviction: the case does not test anything"
    assert torch.equal(got, want)
    del fill


# ------------------------------------------------------------------------------------------------ C. a second device
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("case", ["rq_tokenize", "rq_tokenize_tc_k256", "gumbel", "mlp", "prefix_index", "filters"])
def test_inputs_on_a_second_device_while_the_first_has_a_side_stream(case):
    fn, make = KERNEL_CASES[case]
    real = [t.to("cuda:1") for t in make(0)]
    with torch.cuda.device(1):
        want = run(fn, real)
    with torch.cuda.device(0):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            got = run(fn, real)
        s.synchronize()
    torch.cuda.synchronize(1)
    for (g, _), (w, atomic) in zip(got, want):
        assert g.device == w.device == torch.device("cuda", 1)
        assert torch.equal(g, w) or (atomic and rel(g, w) <= TOL[w.dtype])


# ------------------------------------------------------------------------------------------------ D. host-fed tokeniser
D_HOST, K_HOST, L_HOST = 96, 256, 3


@pytest.fixture(scope="module")
def host_problem():
    x, cbs = I.rq_problem(4 * 16384 + 5, D_HOST, K_HOST, L_HOST, seed=55)
    return x, cbs, [dev(c) for c in cbs]


def device_ids(tok, x):
    return tok.tokenize_device(dev(x)).cpu()


@pytest.mark.parametrize("use_tc", [True, False])
@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 768, 769, 2577])
def test_tokenize_host_chunks_and_ring_cycles(host_problem, use_tc, n):
    from rq_vae_recommender_b200 import parallel
    x, _, cbs = host_problem
    tok = parallel.CorpusTokenizer(cbs, use_tc=use_tc, chunk_rows=256)
    got = tok.tokenize_host(torch.from_numpy(x[:n]).pin_memory())
    assert got.shape == (n, L_HOST) and got.dtype == torch.int64 and (got.is_pinned() or n == 0)
    assert torch.equal(got, device_ids(tok, x[:n]) if n else torch.empty((0, L_HOST), dtype=torch.int64))


@pytest.mark.parametrize("use_tc", [True, False])
def test_tokenize_host_default_chunks_against_float64(host_problem, use_tc):
    from rq_vae_recommender_b200 import parallel
    x, cbs_h, cbs = host_problem
    tok = parallel.CorpusTokenizer(cbs, use_tc=use_tc)
    assert tok.chunk_rows == 16384 and x.shape[0] == 4 * 16384 + 5
    got = tok.tokenize_host(torch.from_numpy(x))                                 # pageable rows
    assert torch.equal(got, device_ids(tok, x))
    if use_tc:
        assert_ids_match(got.numpy(), O.rq_tokenize(x, cbs_h), x, cbs_h, "tokenize_host")


def test_tokenize_host_outputs_reuse_and_reallocation(host_problem):
    from rq_vae_recommender_b200 import parallel
    x, _, cbs = host_problem
    wide = np.concatenate([x[:3000], I.randn(56, 3000, 64)], axis=1)               # host rows wider than D
    tok = parallel.CorpusTokenizer(cbs, encoder=lambda r: r[:, :D_HOST], chunk_rows=512)
    want = device_ids(tok, x[:3000])
    first = tok.tokenize_host(torch.from_numpy(wide).pin_memory())
    assert torch.equal(first, want) and first.is_pinned()
    again = tok.tokenize_host(torch.from_numpy(wide[:, :D_HOST + 8]))             # same size: the same pinned buffer, new width
    assert again is first and torch.equal(again, want)
    half = tok.tokenize_host(torch.from_numpy(x[:1500]).half())                    # another size and dtype: new buffer and ring
    assert half is not first and torch.equal(half, device_ids(tok, x[:1500].astype(np.float16)))
    for out in (torch.full((3000, L_HOST), -7, dtype=torch.int64), torch.full((3000, L_HOST), -7, dtype=torch.int64).pin_memory()):
        got = tok.tokenize_host(torch.from_numpy(wide), out=out)
        assert got is out and torch.equal(out, want)


def test_tokenize_host_on_a_side_stream_and_with_late_kernels(host_problem, cycles):
    """A side stream current; then every chunk's kernel starts late (a sleep before it), so only the 'consumed' events keep chunk
    i + RING's copy from overwriting the ring slot chunk i's kernel has yet to read."""
    from rq_vae_recommender_b200 import parallel
    x, _, cbs = host_problem
    tok = parallel.CorpusTokenizer(cbs, chunk_rows=256)
    xh = torch.from_numpy(x[:2577]).pin_memory()
    want = device_ids(tok, x[:2577])
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = tok.tokenize_host(xh).clone()
    assert torch.equal(got, want)
    tokenize = tok.tokenize_device

    def late(rows, stats=None):
        torch.cuda._sleep(cycles // 8)
        return tokenize(rows, stats)

    tok.tokenize_device = late
    assert torch.equal(tok.tokenize_host(xh), want)
    with torch.cuda.stream(s):
        assert torch.equal(tok.tokenize_host(xh), want)
