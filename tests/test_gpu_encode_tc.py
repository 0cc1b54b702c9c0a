"""GPU tests of the TF32 tensor-core self-attention of the fused T5 encoder (csrc/t5enc_tc.cu, ops.t5enc_attention_tc*,
ops.T5EncAttentionTCFunction, encoder_attention="tf32").  `pytest -m gpu`.

Accuracy contract: no worse than HF's attention at the module's default matmul precision.  The comparator is the packed statement
tests/t5_enc_train_ref.attention_train evaluated in float32 on the GPU at "high", where its `@` products are cuBLAS TF32 GEMMs as
in HF's eager attention.  Against float64 autograd of the same statement, the kernels' largest error of out, dq, dk, dv and d_rel
must be at most 2x the comparator's, and below 1e-2 of the tensor's largest entry.

Measured on an H100 80GB HBM3 (700 W), kernel error over comparator error:
  * with 1 head, S = 20, 81, 300, 800, p = 0 and 0.1: 0.65 - 1.73;
  * with 6 heads: 0.71 - 1.42 at S = 300 and 800, 0.95 - 2.47 at S = 81 (d_rel), 1.66 - 3.12 at S = 20.  There the comparator's
    error is far below TF32 rounding (out 1.3e-4 of a 0.86 entry, against 3.9e-4 with 1 head): cuBLAS does not run those small
    batched products as TF32.  The kernels' own errors stay under 2^-10 of the largest entry, the floor of the bound below;
  * S = 5120, 1 head: 0.74 - 1.0;  tile-edge histories: 0.96 - 1.9."""
import numpy as np
import pytest
import torch

import t5_enc_train_ref as TR
from test_gpu_decode import amazon_model, candidate_scores, highest, rel_err
from test_gpu_encode_train import loss_grads, packed_histories, set_dropout, train_batch
from test_gpu_generate import history, realistic_corpus
import t5_step_ref as T

pytestmark = pytest.mark.gpu


class high:
    """matmul precision "high" (TF32) for the block, the module's default."""

    def __enter__(self):
        self.old = torch.get_float32_matmul_precision()
        torch.set_float32_matmul_precision("high")

    def __exit__(self, *exc):
        torch.set_float32_matmul_precision(self.old)


def attention_errors(qkv, rel, dout, src, offs, key_mask, S, seed, p, B):
    """{name: (kernel error, comparator error, largest entry)} for out, dq, dk, dv and d_rel, errors as max |x - float64|."""
    from rq_vae_recommender_b200 import ops
    heads = rel.shape[0]
    inner = heads * 64
    keep = ops.t5enc_dropout_keep(seed, p, B, heads, S) if p > 0 else None
    q64, r64 = qkv.double().requires_grad_(), rel.double().requires_grad_()
    want = TR.attention_train(q64, src, offs, key_mask.double(), r64, S, keep, p)
    want.backward(dout.double())
    with high():
        q32, r32 = qkv.clone().requires_grad_(), rel.clone().requires_grad_()
        cmp = TR.attention_train(q32, src, offs, key_mask, r32, S, keep, p)
        cmp.backward(dout)
    out, lse = ops.t5enc_attention_tc_train(qkv, src, offs, key_mask, rel, S, seed, p)
    dqkv, drel = ops.t5enc_attention_tc_backward(qkv, out, dout, lse, src, offs, key_mask, rel, S, seed, p)
    cols = {"dq": slice(0, inner), "dk": slice(inner, 2 * inner), "dv": slice(2 * inner, 3 * inner)}
    res = {"out": (out, cmp.detach(), want.detach())}
    for name, c in cols.items():
        res[name] = (dqkv[:, c], q32.grad[:, c], q64.grad[:, c])
    res["drel"] = (drel, r32.grad, r64.grad)
    return {k: ((a.double() - w).abs().max().item(), (b.double() - w).abs().max().item(), w.abs().max().item())
            for k, (a, b, w) in res.items()}


def assert_contract(errs, what):
    """The kernel's error at most twice the comparator's.  For some small batched shapes (an H100 measured it at S = 20 with 6
    heads) cuBLAS runs the comparator's products in full fp32 rather than TF32 at "high"; its error then falls below TF32's own
    rounding, so the bound never drops below twice one TF32 unit (2^-11) of the largest entry."""
    for name, (e_tc, e_cmp, top) in errs.items():
        print(f"{what} {name}: kernel {e_tc:.3e}, TF32 matmuls {e_cmp:.3e}, ratio {e_tc / max(e_cmp, 1e-30):.2f}, "
              f"largest entry {top:.3e}")
        assert e_tc <= 2 * max(e_cmp, 2 ** -11 * top), (what, name, e_tc, e_cmp)
        assert e_tc < 1e-2 * top, (what, name, e_tc, top)


def inputs(N, heads, S, seed):
    g = torch.Generator().manual_seed(seed)
    inner = heads * 64
    qkv = (torch.randn(N, 3 * inner, generator=g) * 0.3).cuda()
    rel = torch.randn(heads, 2 * S - 1, generator=g).cuda()
    dout = torch.randn(N, inner, generator=g).cuda()
    return qkv, rel, dout


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("S", [20, 81, 300, 800])
@pytest.mark.parametrize("heads", [1, 6])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_accuracy_no_worse_than_tf32_matmuls(S, heads, p):
    from rq_vae_recommender_b200 import ops
    offs, src, key_mask, B = packed_histories(S, S + heads)
    qkv, rel, dout = inputs(src.shape[0], heads, S, S * 10 + heads)
    seed = torch.tensor([1234567 + S], dtype=torch.int64, device="cuda")
    assert_contract(attention_errors(qkv, rel, dout, src, offs, key_mask, S, seed, p, B), f"S={S} heads={heads} p={p}")
    if p == 0:                                                  # the eval kernel is the training kernel without dropout
        out, _ = ops.t5enc_attention_tc_train(qkv, src, offs, key_mask, rel, S, seed, 0.0)
        assert torch.equal(out, ops.t5enc_attention_tc(qkv, src, offs, key_mask, rel, S))


def test_longest_histories():
    """S = 5120 (MAX_TRAIN_ENCODER_LEN) with one head: the same contract, and the backward's shared memory at its largest."""
    S, heads = 5120, 1
    offs, src, key_mask, B = packed_histories(S, 3)
    qkv, rel, dout = inputs(src.shape[0], heads, S, 4)
    seed = torch.tensor([99], dtype=torch.int64, device="cuda")
    assert_contract(attention_errors(qkv, rel, dout, src, offs, key_mask, S, seed, 0.1, B), "S=5120")


def test_tile_edges_match_the_fp32_kernels():
    """Histories of 1, 63, 64, 65 and 128 kept rows (plus 0, 2 and 130); the last one ends at the allocation's last row."""
    from rq_vae_recommender_b200 import ops
    S, heads = 130, 2
    counts = [1, 63, 64, 0, 65, 128, 2, 130]
    g = torch.Generator().manual_seed(8)
    src, offs = [], [0]
    for b, c in enumerate(counts):
        pos = torch.randperm(S, generator=g)[:c].sort().values
        src.append(pos + b * S)
        offs.append(offs[-1] + c)
    src = torch.cat(src).to(torch.int32).cuda()
    offs = torch.tensor(offs, dtype=torch.int32, device="cuda")
    key_mask = torch.zeros(len(counts), device="cuda")
    key_mask[2] = T.NEG
    qkv, rel, dout = inputs(src.shape[0], heads, S, 9)
    seed = torch.tensor([5], dtype=torch.int64, device="cuda")
    for p in (0.0, 0.1):
        o32, l32 = ops.t5enc_attention_train(qkv, src, offs, key_mask, rel, S, seed, p)
        otc, ltc = ops.t5enc_attention_tc_train(qkv, src, offs, key_mask, rel, S, seed, p)
        assert rel_err(otc, o32) < 1e-2 and rel_err(ltc, l32) < 1e-3
        d32 = ops.t5enc_attention_backward(qkv, o32, dout, l32, src, offs, key_mask, rel, S, seed, p)
        dtc = ops.t5enc_attention_tc_backward(qkv, otc, dout, ltc, src, offs, key_mask, rel, S, seed, p)
        inner = heads * 64
        for i in range(3):
            assert rel_err(dtc[0][:, i * inner:(i + 1) * inner], d32[0][:, i * inner:(i + 1) * inner]) < 1e-2, (p, i)
        assert rel_err(dtc[1], d32[1]) < 1e-2, p
        assert_contract(attention_errors(qkv, rel, dout, src, offs, key_mask, S, seed, p, len(counts)), f"edges p={p}")


def test_backward_is_bit_reproducible():
    from rq_vae_recommender_b200 import ops
    S, heads = 300, 6
    offs, src, key_mask, B = packed_histories(S, 5)
    qkv, rel, dout = inputs(src.shape[0], heads, S, 4)
    seed = ops.t5enc_dropout_seed("cuda")
    out, lse = ops.t5enc_attention_tc_train(qkv, src, offs, key_mask, rel, S, seed, 0.1)
    out2, lse2 = ops.t5enc_attention_tc_train(qkv, src, offs, key_mask, rel, S, seed, 0.1)
    assert torch.equal(out, out2) and torch.equal(lse, lse2)
    a = ops.t5enc_attention_tc_backward(qkv, out, dout, lse, src, offs, key_mask, rel, S, seed, 0.1)
    b = ops.t5enc_attention_tc_backward(qkv, out, dout, lse, src, offs, key_mask, rel, S, seed, 0.1)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ------------------------------------------------------------------------------------------------ whole model
def amazon(seed=0):
    from rq_vae_recommender_b200.modules import model as M
    m = amazon_model(M, realistic_corpus(np.random.RandomState(seed), 3000, 3, 256)).train()
    set_dropout(m, 0.0)
    return m


def tf32_loss_grads(m, batch, fn=None):
    m.zero_grad(set_to_none=True)
    loss = (m if fn is None else fn)(batch, encoder="fused", encoder_attention="tf32").loss
    loss.backward()
    return loss.detach(), {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}


def assert_tf32_matches_hf(m, batch, fn=None):
    """Loss within 1e-3 relative of HF's at "high", and every gradient within 1e-2 of its parameter's largest entry -- or, where
    the pass with the fp32 attention kernels is itself farther from HF at "high", within twice its largest distance.  At "high"
    every GEMM of both passes rounds to TF32 in different shapes, so a relu flip in the decoder moves whole rows of a wi
    gradient, in whichever block it happens: an H100 measured up to 1.1e-1 for either pass (decoder wi, 64 histories of 20
    items), varying from run to run with HF's own atomic embedding backward."""
    with high():
        lh, gh = loss_grads(m, batch, "hf", fn)
        _, g32 = loss_grads(m, batch, "fused", fn)
        lf, gf = tf32_loss_grads(m, batch, fn)
    assert abs(lf.item() - lh.item()) <= 1e-3 * abs(lh.item()), (lf.item(), lh.item())
    assert set(gf) == set(gh) == set(g32)

    def err(g):
        return {name: (g[name] - gh[name]).abs().max().item() / max(gh[name].abs().max().item(), 1e-30) for name in gh}
    e_tf, e_32 = err(gf), err(g32)
    worst = max(e_tf, key=e_tf.get)
    print(f"loss {lf.item():.6f} vs HF {lh.item():.6f}; largest gradient difference {e_tf[worst]:.2e} ({worst}), with the fp32 "
          f"attention {e_32[worst]:.2e}; largest with the fp32 attention {max(e_32.values()):.2e}")
    for name in gh:
        assert e_tf[name] <= max(1e-2, 2 * max(e_32.values())), (name, e_tf[name], e_32[name])


@pytest.mark.parametrize("lengths", ["full", "uniform"])
def test_forward_matches_hf_at_high_precision(lengths):
    rs = np.random.RandomState(3)
    m = amazon().eval()
    B = 64
    batch = train_batch(rs, B, 20, 3, 256, None if lengths == "full" else rs.randint(1, 21, size=B))
    assert_tf32_matches_hf(m, batch)


def test_forward_matches_hf_through_torch_compile():
    rs = np.random.RandomState(5)
    m = amazon().eval()
    batch = train_batch(rs, 32, 20, 3, 256, rs.randint(1, 21, size=32))
    assert_tf32_matches_hf(m, batch, fn=torch.compile(m))


def test_dropout_step_is_reproducible_under_the_seed():
    rs = np.random.RandomState(7)
    m = amazon()
    set_dropout(m, 0.1)
    batch = train_batch(rs, 48, 20, 3, 256, rs.randint(2, 21, size=48))
    runs = []
    for _ in range(2):
        torch.manual_seed(11)
        m.zero_grad(set_to_none=True)
        loss = m(batch, encoder="fused", decoder="fused", encoder_attention="tf32").loss
        loss.backward()
        runs.append((loss.detach(), {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}))
    (l1, g1), (l2, g2) = runs
    assert torch.equal(l1, l2)
    assert set(g1) == set(g2)
    for name in g1:
        assert torch.equal(g1[name], g2[name]), name
    torch.manual_seed(11)
    l32 = m(batch, encoder="fused", decoder="fused", encoder_attention="fp32").loss.detach()
    assert not torch.equal(l1, l32) and abs(l1.item() - l32.item()) <= 1e-3 * abs(l32.item())   # same keep bits, other rounding


def test_generate_tf32_against_fp32_near_ties_only():
    """The near-tie rule of tests/test_gpu_encode.py, with the fp32 kernel's encoder output in HF's place."""
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(12)
    K, H, k, B = 256, 3, 10, 64
    m = amazon_model(M, realistic_corpus(rs, 3000, H, K))
    mask, ids, users = history(rs, B, 20, H, K)
    with high(), torch.no_grad():
        enc_f, mask_f = m._fused_encoder("fp32")(mask, ids, users)
        enc_t, _ = m._fused_encoder("tf32")(mask, ids, users)
        beams = T.random_beams(B, k, H, K, seed=16, device="cuda")
        want = T.hf_level_logits(m, enc_f, mask_f, beams, k)
        got = T.hf_level_logits(m, enc_t, mask_f, beams, k)
        D = max((a - b).abs().max().item() for a, b in zip(got, want))
        print(f"largest |logit difference| between the fp32 and tf32 attention: {D:.3e}")
        assert D < 1e-2
        runs = {}
        for att in ("fp32", "tf32"):
            runs[att] = captured_run(m, mask, ids, users, att)
    (lf, (gf, pf)), (_, (gt, pt)) = runs["fp32"], runs["tf32"]
    index = m._prefix_index(torch.device("cuda"))
    same_rows = (gt == gf).reshape(B, -1).all(1)
    near_tie = torch.zeros(B, dtype=torch.bool, device="cuda")
    generated, log_probas = None, None
    for h in range(H):
        top = candidate_scores(index, lf[h], generated, log_probas, k).topk(k + 1, dim=1).values
        gaps = (top[:, :-1] - top[:, 1:]).nan_to_num(nan=float("inf"))
        near_tie |= (gaps < 2 * D * (h + 1)).any(1)
        generated, log_probas, _ = index.beam_topk(lf[h], generated, log_probas, k)
    assert torch.equal(generated, gf)
    print(f"histories with different beams: {int((~same_rows).sum())} of {B}, near-tied: {int(near_tie.sum())}")
    assert bool((same_rows | near_tie).all())
    assert (pt[same_rows] - pf[same_rows]).nan_to_num(neginf=0.0).abs().max().item() <= 2 * D * H


def captured_run(m, mask, ids, users, att):
    from test_gpu_decode import captured_logits
    return captured_logits(m, lambda: m.generate(mask, ids, users, search="beam", encoder="fused", encoder_attention=att))


# ------------------------------------------------------------------------------------------------ launches, host sync, errors
def test_launches_and_synchronisation():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(19)
    m = amazon()
    set_dropout(m, 0.1)
    L = len(m.encoder.encoder.block)
    batch = train_batch(rs, 16, 10, 3, 256, rs.randint(1, 11, size=16))
    mask = M._strip_dedup_col(batch.seq_mask.long(), 4, 3)
    ids = M._strip_dedup_col(batch.sem_ids, 4, 3)
    m.eval()
    with torch.no_grad():
        m._fused_encoder("tf32")(mask, ids, batch.user_ids)
        before = ops.LAUNCHES
        m._fused_encoder("tf32")(mask, ids, batch.user_ids)
        assert ops.LAUNCHES - before == 3 + 3 * L
    m.train()
    out, _ = m._fused_train_encoder_pass(mask, ids, batch.user_ids, "tf32")      # warm-up
    out.square().sum().backward()
    read = M._read_n_kept
    reads = []

    def allowed(offsets):
        reads.append(1)
        torch.cuda.set_sync_debug_mode(0)
        try:
            return read(offsets)
        finally:
            torch.cuda.set_sync_debug_mode("error")

    torch.cuda.synchronize()
    M._read_n_kept = allowed
    try:
        m.zero_grad(set_to_none=True)
        torch.cuda.set_sync_debug_mode("error")
        out, _ = m._fused_train_encoder_pass(mask, ids, batch.user_ids, "tf32")
        out.square().sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
        M._read_n_kept = read
    assert reads == [1]


def test_tf32_errors():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200._lib import Rqb200Error
    rs = np.random.RandomState(23)
    m = amazon()
    batch = train_batch(rs, 4, 3, 3, 256)
    with pytest.raises(ValueError, match="encoder_attention"):
        m(batch, encoder="hf", encoder_attention="tf32")
    with pytest.raises(ValueError, match="encoder_attention must be one of"):
        m(batch, encoder="fused", encoder_attention="bf16")
    with torch.autocast("cuda", dtype=torch.bfloat16), pytest.raises(ValueError, match="autocast"):
        m(batch, encoder="fused", encoder_attention="tf32")
    long = train_batch(rs, 2, 1300, 3, 256)
    with pytest.raises(Rqb200Error, match="exceed"):
        m(long, encoder="fused", encoder_attention="tf32")
    offs, src, key_mask, B = packed_histories(20, 1)
    qkv, rel, dout = inputs(src.shape[0], 1, 20, 1)
    with pytest.raises(ValueError, match="rel"):
        ops.t5enc_attention_tc(qkv, src, offs, key_mask, rel[:, 1:], 20)
    with pytest.raises(ValueError, match="probability"):
        ops.t5enc_attention_tc_train(qkv, src, offs, key_mask, rel, 20, torch.zeros(1, dtype=torch.int64, device="cuda"), 1.0)
