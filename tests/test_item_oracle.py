"""CPU tests of the corpus item table and the device-side metrics: the numpy oracle ``item_oracle`` against a brute-force tuple
dictionary, the histogram-to-metrics reduction against the UNMODIFIED reference TopKAccumulator (tests/golden/metrics.npz),
``dropin.install(replace_metrics=True)`` and the plumbing of ``generate_items`` / ``item_of`` with the oracle in place of the
kernels."""
import sys

import numpy as np
import pytest
import torch

import item_oracle as I
from parity import load_golden


def corpus(N, C, K, seed):
    """N rows over a small id range (many duplicate tuples), a few rows exactly duplicated, a few with an id outside [0, K)."""
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, min(K, 3), size=(N, C))
    if N > 10:
        ids[rng.integers(0, N, size=N // 10)] = ids[rng.integers(0, N, size=N // 10)]
        bad = rng.integers(0, N, size=N // 20)
        ids[bad, rng.integers(0, C, size=bad.size)] = rng.choice([-1, K, K + 7], size=bad.size)
    return ids


def brute(ids, K):
    d = {}
    for n, row in enumerate(ids):
        if ((row >= 0) & (row < K)).all():
            d.setdefault(tuple(int(v) for v in row), []).append(n)
    return d


def queries(ids, K, C, rng, P=200):
    """Corpus tuples, tuples absent from the corpus and tuples with out-of-range ids, each with a dedup rank in [-1, 3]."""
    rows = [ids[rng.integers(0, len(ids))] if len(ids) else np.zeros(C, dtype=np.int64) for _ in range(P // 2)]
    rows += [rng.integers(0, min(K, 3) + 1, size=C) for _ in range(P // 4)]
    rows += [np.where(rng.random(C) < 0.3, rng.choice([-1, K]), rng.integers(0, min(K, 3), size=C)) for _ in range(P // 4)]
    q = np.stack(rows).astype(np.int64)
    return np.concatenate([q, rng.integers(-1, 4, size=(len(q), 1))], axis=1)


@pytest.mark.parametrize("K", [16, 256, 2048])
@pytest.mark.parametrize("C", [1, 3, 5, 8])
@pytest.mark.parametrize("N", [0, 1, 600])
def test_item_oracle_vs_tuple_dictionary(K, C, N):
    rng = np.random.default_rng(K * 100 + C * 10 + N)
    ids = corpus(N, C, K, seed=K + C + N)
    table = I.build(ids, K)
    d = brute(ids, K)
    assert len(table["keys"]) == len(d) and table["start"][-1] == sum(len(v) for v in d.values())
    for t, rows in d.items():
        assert I.items_of(table, t) == rows                                 # ascending row order = dedup rank order
    q = queries(ids, K, C, rng)
    want = np.array([d.get(tuple(int(v) for v in t[:C]), [-1])[0] for t in q])
    assert np.array_equal(I.lookup(table, q[:, :C]), want)
    rows = [d.get(tuple(int(v) for v in t[:C]), []) for t in q]
    want = np.array([r[t[C]] if 0 <= t[C] < len(r) else -1 for t, r in zip(q, rows)])
    assert np.array_equal(I.lookup(table, q, with_dedup=True), want)
    # retrieve: 7 histories of k = 12 beams, -inf fillers, the same tuple on two beams, truncation at n
    B, k = 7, 12
    gen = q[rng.integers(0, len(q), size=(B, k)), :C]
    gen[:, 5] = gen[:, 2]
    lp = np.sort(rng.normal(size=(B, k)).astype(np.float32), axis=1)[:, ::-1].copy()
    lp[:, 9:] = -np.inf
    lp[0, 3] = np.nan
    for n in (1, 4, 100):
        items, beam, count = I.retrieve(table, gen, lp, n)
        for b in range(B):
            got = []
            for j in range(k):
                if lp[b, j] > -np.inf:
                    got += [(it, j) for it in d.get(tuple(int(v) for v in gen[b, j]), []) if it not in [g[0] for g in got]]
            got = got[:n]
            assert count[b] == len(got)
            assert items[b].tolist() == [g[0] for g in got] + [-1] * (n - len(got))
            assert beam[b].tolist() == [g[1] for g in got] + [-1] * (n - len(got))
    items_all, _, _ = I.retrieve(table, gen, None, 100)                     # no log-probabilities: every beam contributes
    assert (items_all >= 0).sum() >= (I.retrieve(table, gen, lp, 100)[0] >= 0).sum()


def test_item_oracle_order_is_stable_argsort():
    ids = corpus(600, 3, 16, seed=5)
    table = I.build(ids, 16)
    ok = ((ids >= 0) & (ids < 16)).all(1)
    enc = np.where(ok[:, None], ids, 16)
    want = np.argsort(enc[:, 0] * 17 * 17 + enc[:, 1] * 17 + enc[:, 2], kind="stable")
    assert np.array_equal(table["row"], want)


def golden_cases():
    g = load_golden("metrics")
    for name in ("tuples", "wide_ks", "items"):
        batches = [(g[f"{name}/actual{i}"].astype(np.int64), g[f"{name}/top_k{i}"].astype(np.int64))
                   for i in range(int(g[f"{name}/batches"]))]
        yield name, [int(k) for k in g[f"{name}/ks"]], batches, list(g[f"{name}/keys"]), g[f"{name}/values"]


@pytest.mark.parametrize("case", ["tuples", "wide_ks", "items"])
def test_metrics_from_hist_vs_reference(case):
    from rq_vae_recommender_b200.evaluate.metrics import metrics_from_hist
    name, ks, batches, keys, values = next(c for c in golden_cases() if c[0] == case)
    hist = sum(I.rank_hist(a, t) for a, t in batches)
    total = sum(a.shape[0] for a, _ in batches)
    got = metrics_from_hist(hist, total, ks)
    assert list(got) == keys
    for key, v in zip(keys, values):
        if key == "ndcg":
            assert got[key] == pytest.approx(v, rel=1e-6)
        else:
            assert got[key] == v                                             # exact: integer counts over the same total


def test_rank_hist_oracle_item_mode():
    actual = np.array([[3], [-1], [5], [7]])
    cand = np.array([[[1], [3], [3]], [[-1], [-1], [2]], [[-1], [5], [-1]], [[-1], [-1], [-1]]])
    assert I.rank_hist(actual, cand).tolist() == [1, 2, 0, 1]               # tuple mode: -1 == -1 matches
    assert I.rank_hist(actual, cand, item_mode=True).tolist() == [0, 2, 0, 2]


def test_topk_accumulator_interface_on_cpu():
    from rq_vae_recommender_b200._lib import Rqb200Error
    from rq_vae_recommender_b200.evaluate.metrics import TopKAccumulator
    acc = TopKAccumulator()
    assert acc.ks == [1, 5, 10] and acc.total == 0 and acc.reduce() == {}
    with pytest.raises(Rqb200Error):
        acc.accumulate(actual=torch.zeros(2, 3, dtype=torch.long), top_k=torch.zeros(2, 4, 3, dtype=torch.long))
    acc.reset()
    assert acc.reduce() == {} and acc.total == 0


def test_install_replace_metrics():
    import rq_vae_recommender_b200.dropin as dropin
    names = ("gin", "evaluate", "evaluate.metrics", "init", "distributions", "modules.model")
    saved = {name: sys.modules.get(name) for name in names}
    try:
        default = dropin.install()
        assert "evaluate.metrics" not in default
        assert default == sorted(list(dropin._ALIASES) + ["modules.tokenizer.semids"])
        installed = dropin.install(replace_metrics=True)
        assert installed == sorted(default + ["evaluate.metrics"])
        from rq_vae_recommender_b200.evaluate import metrics
        assert sys.modules["evaluate.metrics"] is metrics
        from evaluate.metrics import TopKAccumulator
        assert TopKAccumulator is metrics.TopKAccumulator
    finally:
        dropin.uninstall()
        assert "evaluate.metrics" not in sys.modules
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod


class OracleTable:
    """CPU stand-in for ops.SidItemTable built on item_oracle."""
    def __init__(self, corpus, K):
        self.table = I.build(corpus.numpy(), K)
        self.calls = 0

    def retrieve(self, generated, log_probas, n):
        self.calls += 1
        items, beam, count = I.retrieve(self.table, generated.numpy(), None if log_probas is None else log_probas.numpy(), n)
        return torch.from_numpy(items), torch.from_numpy(beam), torch.from_numpy(count)

    def lookup(self, ids, with_dedup=False):
        return torch.from_numpy(I.lookup(self.table, ids.numpy(), with_dedup))


def test_generate_items_plumbing_with_oracle():
    """generate_items on the CPU, with the oracles in place of the kernels: generate's beams unchanged, then the table's items."""
    from test_generate_oracle import OracleIndex, decoder_batch, decoder_model
    from rq_vae_recommender_b200.modules import model as M
    g = load_golden("decoder")
    m = decoder_model(M, g)
    index = OracleIndex(m.codebooks)
    K = m.num_embeddings_per_hierarchy
    table = OracleTable(m.codebooks, K)
    m._prefix_index = lambda device: index
    m._item_table = lambda device: table
    batch = decoder_batch(g)
    torch.manual_seed(1002)
    out = m.generate_items(batch)
    assert table.calls == 1
    assert np.array_equal(out.sem_ids.numpy(), g["gen_sem_ids"])
    np.testing.assert_allclose(out.log_probas.numpy(), g["gen_log_probas"], rtol=2e-5, atol=1e-6)
    items, beam, count = I.retrieve(table.table, out.sem_ids.numpy(), out.log_probas.numpy(), m.top_k_for_generation)
    assert np.array_equal(out.item_ids.numpy(), items) and np.array_equal(out.beams.numpy(), beam)
    assert np.array_equal(out.count.numpy(), count)
    torch.manual_seed(1002)
    wide = m.generate_items(batch, n=50)
    assert wide.item_ids.shape == (batch.sem_ids.shape[0], 50)
    assert np.array_equal(wide.item_ids.numpy()[:, :m.top_k_for_generation], items)
    H = m.num_hierarchies
    fut = batch.sem_ids_fut
    want = I.lookup(table.table, fut[:, :H + 1].numpy(), with_dedup=True)
    assert np.array_equal(m.item_of(fut).numpy(), want)
    assert isinstance(out, M.ItemGenerationOutput)
