"""GPU parity of the wgmma tokeniser at K = 512 .. 2048 codes per level (256-code blocks, blocked candidate selection)
against the oracle and the exact CUDA-core kernel, plus the routing of the module API and the training forward.  `pytest -m gpu`."""
import numpy as np
import pytest
import torch

import inputs as I
import tc_blocked_model as MB
import tc_filter_model as M
from oracle import rq_oracle as O
from parity import assert_ids_match, assert_no_worse_than

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def ops():
    from rq_vae_recommender_b200 import ops as _ops
    return _ops


def problem(n, D, K, L, seed):
    """Unit rows + L live codebooks drawn from a residual walk of the first max(n, K, 4096) rows (capped at 8192), the walk's
    argmin by the fp32 oracle: like inputs.rq_problem, without its float64 walk (slow at K = 2048)."""
    m = min(max(n, K, 4096), 8192)
    x = I.unit_rows(seed, max(n, m), D)
    rs = np.random.RandomState(seed + 1)
    cbs, res = [], x[:m].copy()
    for _ in range(L):
        idx = rs.choice(m, K, replace=False)
        cb = (res[idx] + (rs.randn(K, D) * (0.5 / np.sqrt(D))).astype(np.float32)).astype(np.float32)
        cbs.append(cb)
        res = res - cb[O.rq_tokenize(res, [cb])[:, 0]]
    return x[:n], cbs


def run_tc(ops, x, cbs):
    stats = torch.zeros(4, dtype=torch.int32, device="cuda")
    ids = ops.rq_tokenize_tc(dev(x), [dev(c) for c in cbs], stats=stats)
    torch.cuda.synchronize()
    return host(ids), host(stats)


def exact(ops, x, cbs):
    return host(ops.rq_tokenize(dev(x), [dev(c) for c in cbs]))


def test_tc_supported_large_k(ops):
    assert all(ops.tc_supported(768, 256 * m, 3) for m in range(1, 9))
    assert not ops.tc_supported(768, 2304, 3) and not ops.tc_supported(768, 384, 3) and not ops.tc_supported(768, 128, 3)
    assert ops.tc_padded_dim(32, 1024, 3) == 64 and ops.tc_padded_dim(32, 1000, 3) == 0


@pytest.mark.parametrize("K,B,D,L", [(512, 1, 768, 3), (512, 100, 768, 3), (512, 129, 128, 1), (512, 5000, 64, 3),
                                      (512, 600, 64, 8), (1024, 1, 64, 1), (1024, 100, 128, 3), (1024, 129, 768, 1),
                                      (1024, 5000, 768, 3), (2048, 1, 128, 3), (2048, 100, 64, 3), (2048, 129, 768, 3),
                                      (2048, 5000, 128, 1), (2048, 5000, 768, 3), (1536, 777, 256, 2)])
def test_tc_large_k_vs_oracle(ops, K, B, D, L):
    x, cbs = problem(B, D, K, L, seed=K + B + D + L)
    ids, stats = run_tc(ops, x, cbs)
    assert ids.shape == (B, L) and ids.min() >= 0 and ids.max() < K
    n_tie = assert_ids_match(ids, O.rq_tokenize(x, cbs), x, cbs, f"tc K={K} B={B} D={D} L={L}")
    assert n_tie <= max(2, B // 2000)
    ex = exact(ops, x, cbs)
    assert_ids_match(ids, ex, x, cbs, f"tc-vs-simt K={K} B={B} D={D} L={L}")
    assert (ids != ex).any(1).sum() <= max(2, B // 2000)


@pytest.mark.parametrize("D", [64, 768])
def test_tc_large_k_full_size_vs_exact_kernel(ops, D):
    """65 536 rows at K = 1024, L = 3: the exact CUDA-core kernel is the reference (the fp32 oracle is too slow on the host)."""
    n, K, L = 65536, 1024, 3
    x, cbs = problem(n, D, K, L, seed=31 + D)
    ids, stats = run_tc(ops, x, cbs)
    n_tie = assert_ids_match(ids, exact(ops, x, cbs), x, cbs, f"tc-vs-simt full K={K} D={D}")
    assert n_tie <= n // 2000, n_tie
    assert stats[0] < 0.2 * n * L, stats


def test_tc_ties_across_blocks_pick_first_index(ops):
    """Code 17 duplicated as 17 + 256 (block 1) and 17 + 1792 (block 7): every row must get 17."""
    D, K, L = 128, 2048, 2
    _, cbs = problem(4096, D, K, L, seed=5)
    cbs[0][17 + 256] = cbs[0][17]
    cbs[0][17 + 1792] = cbs[0][17]
    x = np.repeat(cbs[0][17:18], 256, axis=0) + 1e-4 * I.randn(4, 256, D)
    ids, stats = run_tc(ops, x, cbs)
    assert (ids[:, 0] == 17).all(), np.unique(ids[:, 0], return_counts=True)
    assert stats[0] >= 256          # every row needed the exact re-rank at level 0
    assert_ids_match(ids, O.rq_tokenize(x, cbs), x, cbs, "tc/ties across blocks")


@pytest.mark.parametrize("gap", ["near", "far"])
def test_tc_true_minimum_in_the_last_block(ops, gap):
    """Rows whose best code is in the last block while block 0 holds the runner-up.  'near': the runner-up is inside the filter
    margin, the exact re-rank must pick the last-block code.  'far': it is outside; block 0 is kept while it is scored (its own
    minimum sets the running threshold) and dropped at the end of the level, so no row is re-ranked."""
    D, K = 128, 1024
    rs = np.random.RandomState(11)
    cb = (rs.randn(K, D) / np.sqrt(D)).astype(np.float32)
    best = K - 5
    delta = rs.randn(D) / np.sqrt(D)
    cb[7] = (cb[best] + (3e-3 if gap == "near" else 0.1) * delta).astype(np.float32)
    x = (cb[best] + 1e-4 * rs.randn(512, D) / np.sqrt(D)).astype(np.float32)
    ids, stats = run_tc(ops, x, [cb])
    ref = O.rq_tokenize(x, [cb])
    assert (ref[:, 0] == best).all()
    assert (ids[:, 0] == best).all(), np.unique(ids[:, 0], return_counts=True)
    if gap == "near":
        assert stats[0] == 512 and stats[1] >= 2 * 512, stats
    else:
        assert stats[0] == 0, stats


def test_tc_large_k_scaled_and_extreme_inputs(ops):
    """Rows at very different scales, rows that overflow fp16, exact duplicates of codes in several blocks, zero rows, a
    non-finite row (the cases of test_gpu_tc.py::test_tc_scaled_and_extreme_inputs at K = 1024)."""
    D, K, L = 768, 1024, 3
    x, cbs = problem(2048, D, K, L, seed=99)
    x = x[:512].copy()
    x[0:64] *= 1e-3
    x[64:128] *= 37.0
    x[128:132] *= 1e6            # fp16 overflow -> every code re-ranked exactly
    x[132:136] = 0.0
    x[136:140] = cbs[0][[10, 300, 700, 1020]]   # exact hits, one per block 0, 1, 2, 3
    x[140, 5] = np.inf
    ids, stats = run_tc(ops, x[:140], cbs)
    ref = O.rq_tokenize(x[:140], cbs)
    assert_ids_match(ids, ref, x[:140], cbs, "tc/extreme K=1024")
    assert (ids[136:140, 0] == [10, 300, 700, 1020]).all()
    ids2, _ = run_tc(ops, x[:141], cbs)          # a non-finite row must not disturb its neighbours
    assert (ids2[:140] == ids).all()
    assert (ids2[140] >= 0).all() and (ids2[140] < K).all()


@pytest.mark.parametrize("kind", M.ADVERSARIAL_KINDS)
@pytest.mark.parametrize("D,L", [(768, 1), (768, 3), (128, 2)])
def test_tc_large_k_adversarial_rounding(ops, kind, D, L):
    x, cbs = M.adversarial_problem(kind, D=D, K=1024, L=L, n=300)
    ids, stats = run_tc(ops, x, cbs)
    assert_ids_match(ids, O.rq_tokenize(x, cbs), x, cbs, f"tc/adversarial/{kind} K=1024 D={D} L={L}")
    assert_no_worse_than(ids, exact(ops, x, cbs), x, cbs, f"tc-vs-simt/adversarial/{kind} K=1024")


@pytest.mark.parametrize("K", [512, 2048])
def test_tc_rerank_count_matches_the_cpu_model(ops, K):
    """stats[0] (rows re-ranked) against the CPU model of the blocked selection on the same inputs.  The model's scores are a
    float64 product rounded once, the kernel's an fp32 tensor-core accumulation, so rows right at a threshold may fall either
    way: slack 1 % of the row-levels + 16."""
    n, D, L = 4096, 128, 3
    x, cbs = problem(n, D, K, L, seed=17 + K)
    ids, stats = run_tc(ops, x, cbs)
    ref = O.rq_tokenize(x, cbs)
    assert_ids_match(ids, ref, x, cbs, f"tc/rerank K={K}")
    model = sum(int((lv["cand"].sum(1) > 1).sum()) for lv in MB.filter_levels_blocked(x, cbs, ref))
    assert abs(int(stats[0]) - model) <= 0.01 * n * L + 16, (int(stats[0]), model)


def test_module_api_routes_large_k_to_the_tensor_core_tokeniser(ops):
    """SemanticIdTokenizer.precompute_corpus_ids -> RqVae.tokenize at K = 1024, D = 64 runs the wgmma tokeniser (one prepare,
    one launch per batch), returns get_semantic_ids' ids, and a codebook update re-prepares."""
    from rq_vae_recommender_b200.data.schemas import SeqBatch
    from rq_vae_recommender_b200.modules.rqvae import RqVae
    from rq_vae_recommender_b200.modules.quantize import QuantizeForwardMode
    from rq_vae_recommender_b200.modules.tokenizer.semids import SemanticIdTokenizer
    Din, D, K, L, N = 768, 64, 1024, 3, 5000
    torch.manual_seed(0)
    m = RqVae(input_dim=Din, embed_dim=D, hidden_dims=[128], codebook_size=K, codebook_kmeans_init=False,
              codebook_mode=QuantizeForwardMode.STE, n_layers=L, n_cat_features=0).cuda()
    x = I.unit_rows(4242, N, Din)
    with torch.no_grad():          # live codebooks: residual rows of the encoder output, like a k-means-initialised model
        res = m.encode(dev(x))
        for l, layer in enumerate(m.layers):
            layer.embedding.weight.copy_(res[torch.randperm(N, generator=torch.Generator().manual_seed(l))[:K].cuda()])
            res = res - layer.embedding.weight[ops.rq_tokenize(res, [layer.embedding.weight])[:, 0]]
    tok = SemanticIdTokenizer(input_dim=Din, output_dim=D, hidden_dims=[128], codebook_size=K, n_layers=L, n_cat_feats=0).cuda()
    tok.rq_vae = m.eval()
    tok.corpus_batch = 1700         # three batches (1700, 1700, 1600; all >= ops.TC_MIN_ROWS)

    class Items:
        def __len__(self):
            return N

        def __getitem__(self, idx):
            idx = torch.as_tensor(idx)
            return SeqBatch(user_ids=-torch.ones_like(idx), ids=idx.unsqueeze(0), ids_fut=-torch.ones_like(idx),
                            x=torch.from_numpy(x)[idx], x_fut=-torch.ones_like(idx), seq_mask=torch.ones_like(idx, dtype=bool))
    calls, preps = ops.TC_CALLS, ops.TC_PREPARES
    cached = host(tok.precompute_corpus_ids(Items()))
    assert ops.TC_CALLS - calls == 3 and ops.TC_PREPARES - preps == 1, (ops.TC_CALLS - calls, ops.TC_PREPARES - preps)
    with torch.no_grad():
        out = m.get_semantic_ids(dev(x))
        z = m.encode(dev(x))
        cbs = [host(layer.codebook()) for layer in m.layers]
    assert_ids_match(cached[:, :L], host(out.sem_ids), host(z), cbs, "module-api/tc K=1024")
    assert np.array_equal(cached[:, :L], host(m.tokenize(dev(x))))
    preps = ops.TC_PREPARES
    with torch.no_grad():           # an optimiser step (in-place update) must invalidate the cached state
        m.layers[0].embedding.weight.mul_(1.01)
    m.tokenize(dev(x))
    assert ops.TC_PREPARES - preps == 1


@pytest.mark.parametrize("D", [64, 768])
@pytest.mark.parametrize("mode_name", ["eval", "ste", "rot"])
def test_large_k_forward_is_tokenise_plus_replay_and_bit_identical(ops, D, mode_name):
    """K = 1024, B = 3000: the training-mode forward takes its ids from the tensor-core tokeniser and replays the chain over
    them; every output equals the fused CUDA-core chain's bit for bit, and the gradients agree."""
    mode = {"eval": ops.MODE_EVAL, "ste": ops.MODE_STE, "rot": ops.MODE_ROTATION}[mode_name]
    B, K, L = 3000, 1024, 3
    x, cbs = problem(B, D, K, L, seed=7 * D + K)
    xd, cd = dev(x), [dev(c) for c in cbs]
    kw = dict(want_ids=True, want_embeddings=True, want_residuals=True, want_sum=True, want_norms=True, want_loss=True)
    calls0 = ops.TC_CALLS
    new = ops.rq_forward(xd, cd, mode, 0.25, **kw)
    assert ops.TC_CALLS == calls0 + 1, "the large-batch forward must go through the tensor-core tokeniser"
    old_min, ops.TC_MIN_ROWS = ops.TC_MIN_ROWS, 1 << 62
    try:
        ref = ops.rq_forward(xd, cd, mode, 0.25, **kw)
    finally:
        ops.TC_MIN_ROWS = old_min
    for k in ("ids", "embeddings", "residuals", "emb_sum", "emb_norms", "loss"):
        assert torch.equal(new[k], ref[k]), f"{mode_name} D={D} K={K}: {k} differs"

    def grads():
        xt = xd.clone().requires_grad_(True)
        ct = [c.clone().requires_grad_(True) for c in cd]
        e, n, ids, loss = ops.RqChainFunction.apply(xt, mode, 0.25, True, *ct)
        (e.sum() + loss.sum()).backward()
        return [xt.grad] + [c.grad for c in ct]
    g_new = grads()
    ops.TC_MIN_ROWS = 1 << 62
    try:
        g_ref = grads()
    finally:
        ops.TC_MIN_ROWS = old_min
    for a, b in zip(g_new, g_ref):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6 * b.abs().max().item())      # codebook grads: fp32 atomics, order varies
