"""GPU parity of the wgmma tokeniser (fp16 candidate filter + exact fp32 re-rank) against the oracle, the
reference-generated fixtures and the exact CUDA-core kernel.  `pytest -m gpu`."""
import numpy as np
import pytest
import torch

import inputs as I
from oracle import rq_oracle as O
from parity import assert_ids_match, load_golden

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def ops():
    from rq_vae_recommender_b200 import ops as _ops
    return _ops


def run_tc(ops, x, cbs):
    stats = torch.zeros(4, dtype=torch.int32, device="cuda")
    ids = ops.rq_tokenize_tc(dev(x), [dev(c) for c in cbs], stats=stats)
    torch.cuda.synchronize()
    return ids.cpu().numpy(), stats.cpu().numpy()


def test_tc_supported(ops):
    assert ops.tc_supported(768, 256, 3) and ops.tc_supported(64, 256, 1)
    assert not ops.tc_supported(32, 256, 3) and not ops.tc_supported(768, 128, 3) and not ops.tc_supported(800, 256, 3)


def test_tc_ns_vs_reference(ops):
    g = load_golden("rq_ns2048")
    n, D, K, L = (int(v) for v in g["shape"])
    x, cbs = I.rq_problem(n, D, K, L, seed=1234)
    ids, stats = run_tc(ops, x, cbs)
    n_tie = assert_ids_match(ids, g["eval_ids"], x, cbs, "tc/ns2048")
    assert n_tie <= 2
    assert stats[0] < 0.2 * n * L, stats      # the filter decides most rows alone


@pytest.mark.parametrize("B,D,L", [(1, 768, 3), (100, 768, 3), (128, 768, 1), (129, 768, 2), (1000, 64, 3),
                                    (777, 128, 4), (5000, 256, 3), (4096, 512, 2), (20000, 768, 3)])
def test_tc_vs_oracle_shapes(ops, B, D, L):
    K = 256
    x, cbs = I.rq_problem(max(B, 1024), D, K, L, seed=B + D + L)
    x = x[:B]
    ids, stats = run_tc(ops, x, cbs)
    ref = O.rq_tokenize(x, cbs)
    n_tie = assert_ids_match(ids, ref, x, cbs, f"tc B={B} D={D} L={L}")
    assert n_tie <= max(2, B // 2000)
    exact = ops.rq_tokenize(dev(x), [dev(c) for c in cbs]).cpu().numpy()
    assert (ids != exact).any(1).sum() <= max(2, B // 2000)


def test_tc_scaled_and_extreme_inputs(ops):
    """Rows at very different scales, rows that overflow fp16, exact duplicates of codes, zero rows."""
    D, K, L = 768, 256, 3
    x, cbs = I.rq_problem(2048, D, K, L, seed=99)
    x = x[:512].copy()
    x[0:64] *= 1e-3
    x[64:128] *= 37.0
    x[128:132] *= 1e6            # fp16 overflow -> every code re-ranked exactly
    x[132:136] = 0.0
    x[136:140] = cbs[0][10:14]   # exact hits
    x[140, 5] = np.inf
    ids, stats = run_tc(ops, x[:140], cbs)
    ref = O.rq_tokenize(x[:140], cbs)
    assert_ids_match(ids, ref, x[:140], cbs, "tc/extreme")
    assert (ids[136:140, 0] == np.arange(10, 14)).all()
    ids2, _ = run_tc(ops, x[:141], cbs)          # a non-finite row must not disturb its neighbours
    assert (ids2[:140] == ids).all()


def test_tc_exact_ties_pick_first_index(ops):
    D, K, L = 128, 256, 2
    x, cbs = I.rq_problem(1024, D, K, L, seed=5)
    cbs[0][200] = cbs[0][17]
    cbs[0][90] = cbs[0][17]
    x = np.repeat(cbs[0][17:18], 256, axis=0) + 1e-4 * I.randn(4, 256, D)
    ids, stats = run_tc(ops, x, cbs)
    assert (ids[:, 0] == 17).all()
    assert stats[0] >= 256          # every row needed the exact re-rank at level 0


def test_tc_strided_rows_and_state_reuse(ops):
    D, K, L = 768, 256, 3
    x, cbs = I.rq_problem(1024, D, K, L, seed=21)
    state = ops.TcState([dev(c) for c in cbs])
    big = torch.zeros(1024, 1024, device="cuda")
    big[:, 128:128 + D] = dev(x)
    a = ops.rq_tokenize_tc(big[:, 128:128 + D], state=state).cpu().numpy()
    b = ops.rq_tokenize_tc(dev(x), state=state).cpu().numpy()
    assert np.array_equal(a, b)
    assert_ids_match(b, O.rq_tokenize(x, cbs), x, cbs)


def test_tc_misaligned_rows_are_copied_by_the_host_side(ops):
    """x whose base is not 16-byte aligned (and whose row stride is not a multiple of 4): the kernel reads x through TMA, so
    ops.rq_tokenize_tc hands it an aligned copy; the C entry point itself rejects such a view (INTEGRATION.md)."""
    from rq_vae_recommender_b200 import _lib
    D, K, L = 128, 256, 3
    x, cbs = I.rq_problem(1024, D, K, L, seed=33)
    big = torch.zeros(700, D + 7, device="cuda")
    big[:, 3:3 + D] = dev(x[:700])
    view = big[:, 3:3 + D]                         # offset 3 floats, row stride D+7
    assert view.data_ptr() % 16 != 0 and view.stride(0) % 4 != 0
    state = ops.TcState([dev(c) for c in cbs])
    a = ops.rq_tokenize_tc(view, state=state).cpu().numpy()
    b = ops.rq_tokenize_tc(dev(x[:700]), state=state).cpu().numpy()
    assert np.array_equal(a, b)
    assert_ids_match(b, O.rq_tokenize(x[:700], cbs), x[:700], cbs)
    lib = _lib.load()
    ids = torch.empty((700, L), dtype=torch.int64, device="cuda")
    rc = lib.rqb200_tokenize_tc_run(view.data_ptr(), view.stride(0), 700, state.buf.data_ptr(), D, K, L, ids.data_ptr(), 0, 0)
    assert rc != 0 and b"16-byte aligned" in lib.rqb200_last_error()


def test_tc_max_levels(ops):
    """L = 8 (RQB_MAX_LEVELS): 28 Gram tables, the serial j >= 2 correction path, all 8 bytes of the packed ids."""
    D, K, L = 64, 256, 8
    x, cbs = I.rq_problem(1024, D, K, L, seed=44)
    ids, stats = run_tc(ops, x[:600], cbs)
    assert ids.shape == (600, 8)
    n_tie = assert_ids_match(ids, O.rq_tokenize(x[:600], cbs), x[:600], cbs, "tc L=8")
    assert n_tie <= 2
    assert not ops.tc_supported(64, 256, 9)


# ---------------------------------------------------------------------------------------------------------------------
# Round-2 additions (VERDICT r1, "next round" item 1): inputs whose fp16 rounding errors are COHERENT (they defeat a z-sigma
# margin; the deterministic bound of tc_eps must flag them), and parity at the full bench / corpus sizes.
import tc_filter_model as M


@pytest.mark.parametrize("kind", M.ADVERSARIAL_KINDS)
@pytest.mark.parametrize("D,L", [(768, 1), (768, 3), (128, 2)])
def test_tc_adversarial_rounding_vs_oracle(ops, kind, D, L):
    x, cbs = M.adversarial_problem(kind, D=D, L=L, n=300)
    ids, stats = run_tc(ops, x, cbs)
    ref = O.rq_tokenize(x, cbs)
    assert_ids_match(ids, ref, x, cbs, f"tc/adversarial/{kind} D={D} L={L}")
    exact = ops.rq_tokenize(dev(x), [dev(c) for c in cbs]).cpu().numpy()
    assert_ids_match(ids, exact, x, cbs, f"tc-vs-simt/adversarial/{kind}")


def test_tc_judge_counterexample(ops):
    """fp32 / fp64 say code 10; the fp16 scores alone say 200 (tests/test_tc_filter_model.py checks that on the CPU model)."""
    x, cbs = M.adversarial_problem("judge_r1", D=768, L=1, n=256)
    ids, stats = run_tc(ops, x, cbs)
    assert (ids[:, 0] == 10).all(), np.unique(ids[:, 0], return_counts=True)
    assert stats[0] >= 256          # every row was re-ranked exactly


def big_problem(n, D, K, L, seed):
    """Like inputs.rq_problem (live residual codebooks) but with the fp32 oracle doing the residual walk: the float64 walk of
    rq_problem takes 15 s per 65 536 x 768 x 3 problem on the build container."""
    x = I.unit_rows(seed, n, D)
    rs = np.random.RandomState(seed + 1)
    cbs, res = [], x.copy()
    for _ in range(L):
        idx = rs.choice(n, K, replace=False)
        cb = (res[idx] + (rs.randn(K, D) * (0.5 / np.sqrt(D))).astype(np.float32)).astype(np.float32)
        cbs.append(cb)
        res = res - cb[O.rq_tokenize(res, [cb])[:, 0]]
    return x, cbs


@pytest.mark.parametrize("n", [65536, 12101, 84000])
@pytest.mark.parametrize("seed", [1234, 77, 2026])
def test_tc_full_size_vs_oracle(ops, n, seed):
    """NS (65 536), C2 (12 101) and C3 (84 000) rows x 768, K=256, L=3 against the fp32 oracle and the exact CUDA-core kernel."""
    D, K, L = 768, 256, 3
    x, cbs = big_problem(n, D, K, L, seed)
    ids, stats = run_tc(ops, x, cbs)
    ref = O.rq_tokenize(x, cbs)
    n_tie = assert_ids_match(ids, ref, x, cbs, f"tc/full n={n} seed={seed}")
    assert n_tie <= max(2, n // 2000), n_tie
    exact = ops.rq_tokenize(dev(x), [dev(c) for c in cbs]).cpu().numpy()
    assert_ids_match(ids, exact, x, cbs, f"tc-vs-simt/full n={n}")
    assert stats[0] < 0.12 * n * L, stats          # deterministic margin: a few % of row-levels are re-ranked


def test_tc_beauty_codebooks_zero_padded_to_64(ops):
    """The shipped Beauty checkpoint's quantiser is D = 32: zero-padding x and the codebooks to 64 columns is exact for every
    dot product, so the tensor-core path must return the exact kernel's ids (reference-generated golden)."""
    g = load_golden("beauty_ckpt")
    z = g["res"].astype(np.float32)
    cbs = [np.ascontiguousarray(c, np.float32) for c in g["codebooks"]]
    pad = lambda a: np.concatenate([a, np.zeros((a.shape[0], 64 - a.shape[1]), np.float32)], axis=1)
    ids, stats = run_tc(ops, pad(z), [pad(c) for c in cbs])
    assert_ids_match(ids, g["sem_ids"], z, cbs, "tc/beauty padded")


@pytest.mark.parametrize("D,L", [(768, 3), (32, 3), (256, 4)])
@pytest.mark.parametrize("mode_name", ["eval", "ste", "rot"])
def test_large_batch_forward_is_tokenise_plus_replay_and_bit_identical(D, L, mode_name):
    """From ops.TC_MIN_ROWS rows on, the training-mode forward takes its ids from the tensor-core tokeniser and computes embeddings,
    residuals, sums, norms and the loss in a streaming pass over the given ids (rq_replay_kernel).  Every output must equal the
    fused CUDA-core chain's bit for bit (same ids, same loops), and the backward must not notice."""
    from rq_vae_recommender_b200 import ops
    mode = {"eval": ops.MODE_EVAL, "ste": ops.MODE_STE, "rot": ops.MODE_ROTATION}[mode_name]
    B = 3000
    x, cbs = I.rq_problem(B, D, 256, L, seed=7 * D + L)
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
        assert torch.equal(new[k], ref[k]), f"{mode_name} D={D} L={L}: {k} differs"
    # autograd through the new route: gradients equal the fused route's
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
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6 * b.abs().max().item())      # codebook grads: fp32 atomics, order varies run to run
