"""GPU tests of the trainable fused T5 encoder pass (csrc/t5enc.cu training kernels, ops.T5EncAttentionFunction /
T5EncAddNormFunction, modules/model.py FusedT5EncodeTrain, forward(encoder="fused")): each kernel against torch autograd of a
float64 statement (tests/t5_enc_train_ref.py, with the keep bits the kernels export), bit-reproducibility, the keep rate, and
the whole training pass against HF's.  `pytest -m gpu`."""
import math

import numpy as np
import pytest
import torch

import t5_enc_ref as E
import t5_enc_train_ref as TR
import t5_step_ref as T
from test_gpu_decode import amazon_model, highest, rel_err
from test_gpu_generate import realistic_corpus

pytestmark = pytest.mark.gpu

MASKS = ("full", "end", "front", "holes", "empty")


def packed_histories(S, seed):
    """offsets, src, key_mask of histories of S positions kept by every mask kind (one history with nothing unmasked)."""
    keep = torch.cat([E.masks(kind, 2, S, 1, seed) for kind in MASKS]).bool()
    empty = ~keep.any(1)
    keep[empty] = True
    key_mask = torch.where(empty, T.NEG, 0.0).float().cuda()
    counts = keep.sum(1)
    offs = torch.cat([counts.new_zeros(1), counts.cumsum(0)]).to(torch.int32).cuda()
    src = keep.reshape(-1).nonzero().squeeze(1).to(torch.int32).cuda()
    return offs, src, key_mask, keep.shape[0]


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("S", [20, 81, 300, 800])
@pytest.mark.parametrize("heads", [1, 6])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_attention_forward_and_backward(S, heads, p):
    """S below 32, not a multiple of 32, above 128 (several query tiles) and 800 (200-item histories)."""
    from rq_vae_recommender_b200 import ops
    g = torch.Generator().manual_seed(S * 10 + heads)
    offs, src, key_mask, B = packed_histories(S, S + heads)
    N, inner = src.shape[0], heads * 64
    qkv = (torch.randn(N, 3 * inner, generator=g) * 0.3).cuda()
    rel = torch.randn(heads, 2 * S - 1, generator=g).cuda()
    dout = torch.randn(N, inner, generator=g).cuda()
    seed = torch.tensor([1234567 + S], dtype=torch.int64, device="cuda")
    keep = ops.t5enc_dropout_keep(seed, p, B, heads, S) if p > 0 else None

    q64, r64 = qkv.double().requires_grad_(), rel.double().requires_grad_()
    want = TR.attention_train(q64, src, offs, key_mask.double(), r64, S, keep, p)
    want.backward(dout.double())
    out, lse = ops.t5enc_attention_train(qkv, src, offs, key_mask, rel, S, seed, p)
    assert rel_err(out.double(), want.detach()) < 1e-5
    dqkv, drel = ops.t5enc_attention_backward(qkv, out, dout, lse, src, offs, key_mask, rel, S, seed, p)
    for got, ref, what in ((dqkv[:, :inner], q64.grad[:, :inner], "dq"), (dqkv[:, inner:2 * inner], q64.grad[:, inner:2 * inner], "dk"),
                           (dqkv[:, 2 * inner:], q64.grad[:, 2 * inner:], "dv"), (drel, r64.grad, "drel")):
        assert rel_err(got.double(), ref) < 2e-5, what
    if p == 0:
        assert torch.equal(out, ops.t5enc_attention(qkv, src, offs, key_mask, rel, S))   # the eval kernel's output exactly


def test_backward_and_add_norm_are_bit_reproducible():
    from rq_vae_recommender_b200 import ops
    S, heads = 300, 6
    g = torch.Generator().manual_seed(4)
    offs, src, key_mask, B = packed_histories(S, 5)
    N, inner = src.shape[0], heads * 64
    qkv = torch.randn(N, 3 * inner, generator=g).cuda() * 0.3
    rel = torch.randn(heads, 2 * S - 1, generator=g).cuda()
    dout = torch.randn(N, inner, generator=g).cuda()
    seed = ops.t5enc_dropout_seed("cuda")
    out, lse = ops.t5enc_attention_train(qkv, src, offs, key_mask, rel, S, seed, 0.1)
    a = ops.t5enc_attention_backward(qkv, out, dout, lse, src, offs, key_mask, rel, S, seed, 0.1)
    b = ops.t5enc_attention_backward(qkv, out, dout, lse, src, offs, key_mask, rel, S, seed, 0.1)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    x, w = torch.randn(5000, 384, device="cuda"), torch.rand(384, device="cuda") + 0.5
    xo, _, inv = ops.t5enc_add_norm_fwd(x, None, w, 1e-6)
    g_out = torch.randn(5000, 384, device="cuda")
    d1 = ops.t5enc_add_norm_bwd(g_out, x, xo, inv, w)
    d2 = ops.t5enc_add_norm_bwd(g_out, x, xo, inv, w)
    assert torch.equal(d1[0], d2[0]) and torch.equal(d1[1], d2[1])


@pytest.mark.parametrize("R,D", [(1, 64), (70, 384), (4099, 128)])
@pytest.mark.parametrize("with_delta", [True, False])
def test_add_norm_forward_and_backward(R, D, with_delta):
    from rq_vae_recommender_b200 import ops
    g = torch.Generator().manual_seed(R + D)
    x, delta = torch.randn(R, D, generator=g).cuda(), torch.randn(R, D, generator=g).cuda() if with_delta else None
    w, eps = (torch.rand(D, generator=g) + 0.5).cuda(), 1e-6
    g_out, g_res = torch.randn(R, D, generator=g).cuda(), torch.randn(R, D, generator=g).cuda()
    x64, w64 = x.double().requires_grad_(), w.double().requires_grad_()
    d64 = delta.double().requires_grad_() if with_delta else None
    xo64 = x64 + d64 if with_delta else x64 * 1
    out64 = TR.t5_norm(xo64, w64, eps)
    torch.autograd.backward([out64, xo64], [g_out.double(), g_res.double()])
    xo, out, inv = ops.t5enc_add_norm_fwd(x, delta, w, eps)
    assert rel_err(xo.double(), xo64.detach()) < 1e-6 and rel_err(out.double(), out64.detach()) < 1e-6
    dx, dw = ops.t5enc_add_norm_bwd(g_out, g_res, xo, inv, w)
    assert rel_err(dx.double(), x64.grad) < 1e-5
    assert rel_err(dw.double(), w64.grad) < 1e-5
    # the autograd Function routes the same gradient to x and delta
    xa, da, wa = x.clone().requires_grad_(), delta.clone().requires_grad_() if with_delta else None, w.clone().requires_grad_()
    xo_a, out_a = ops.T5EncAddNormFunction.apply(xa, da, wa, eps)
    torch.autograd.backward([out_a, xo_a], [g_out, g_res])
    assert torch.equal(xa.grad, dx) and torch.equal(wa.grad, dw)
    if with_delta:
        assert torch.equal(da.grad, dx)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_rate_is_binomial(p):
    from rq_vae_recommender_b200 import ops
    torch.manual_seed(0)
    B, heads, S = 64, 6, 81
    keep = ops.t5enc_dropout_keep(ops.t5enc_dropout_seed("cuda"), p, B, heads, S)
    n = keep.numel()
    kept = int(keep.sum())
    sd = math.sqrt(n * p * (1 - p))
    assert abs(kept - n * (1 - p)) < 6 * sd, (kept, n * (1 - p), sd)
    assert set(keep.unique().tolist()) <= {0, 1}
    # the bits depend on the seed and differ between heads and histories
    other = ops.t5enc_dropout_keep(ops.t5enc_dropout_seed("cuda"), p, B, heads, S)
    assert not torch.equal(keep, other) and not torch.equal(keep[0, 0], keep[0, 1]) and not torch.equal(keep[0], keep[1])


# ------------------------------------------------------------------------------------------------ whole training pass
def train_batch(rs, B, items, H, K, lengths=None):
    """A TokenizedSeqBatch of end-padded histories (lengths in items, default all ``items``)."""
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    W = H + 1
    sem = torch.from_numpy(rs.randint(0, K, size=(B, items * W))).cuda()
    sem.view(B, items, W)[:, :, H] = torch.from_numpy(rs.randint(0, 3, size=(B, items))).cuda()
    L = torch.full((B,), items) if lengths is None else torch.as_tensor(lengths)
    seq_mask = (torch.arange(items * W)[None, :] < (L[:, None] * W)).cuda()
    fut = torch.from_numpy(rs.randint(0, K, size=(B, W))).cuda()
    users = torch.from_numpy(rs.randint(0, 100, size=(B, 1))).cuda()
    zeros = torch.zeros_like(sem)
    return TokenizedSeqBatch(user_ids=users, sem_ids=sem, sem_ids_fut=fut, seq_mask=seq_mask, token_type_ids=zeros,
                             token_type_ids_fut=torch.zeros_like(fut))


def set_dropout(m, p):
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = p
        if type(mod).__name__ == "T5Attention":
            mod.dropout = p


def loss_grads(m, batch, encoder, fn=None):
    m.zero_grad(set_to_none=True)
    loss = (m if fn is None else fn)(batch, encoder=encoder).loss
    loss.backward()
    return loss.detach(), {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}


def assert_matches_hf(m, batch, fn=None):
    with highest():
        lh, gh = loss_grads(m, batch, "hf", fn)
        lf, gf = loss_grads(m, batch, "fused", fn)
    assert abs(lf.item() - lh.item()) <= 1e-5, (lf.item(), lh.item())
    assert set(gf) == set(gh)
    errs = {name: (gf[name] - gh[name]).abs().max().item() / max(gh[name].abs().max().item(), 1e-30) for name in gh}
    worst = max(errs, key=errs.get)
    print(f"largest gradient difference, relative to the parameter's largest entry: {errs[worst]:.2e} ({worst})")
    # The two passes round differently in fp32, so a feed-forward pre-activation within rounding of 0 can pass relu on one side
    # only, and that moves a whole row of wi's gradient.  At 64 x 81 positions an H100 measured up to 3.5e-3 of the largest
    # entry, in block 0's wi; through torch.compile at 32 histories, 1.9e-6.  The loss agrees within 1e-5.  Measured against
    # the float64 statement at 64 full 20-item histories (tests/test_gpu_train_statement.py, an H100 at 700 W), the fused pass
    # flips 3 relus, each within 1.6 fp32 units of its layer's largest pre-activation; they move encoder block 3's wi gradient
    # by 1.2e-3 of its largest entry, and with its relu decisions followed the statement is within 2e-6.
    for name, err in errs.items():
        assert err <= 1e-2, (name, err)


def amazon(seed=0):
    from rq_vae_recommender_b200.modules import model as M
    m = amazon_model(M, realistic_corpus(np.random.RandomState(seed), 3000, 3, 256)).train()
    set_dropout(m, 0.0)
    return m


@pytest.mark.parametrize("lengths", ["full", "uniform"])
def test_forward_equals_hf_without_dropout(lengths):
    rs = np.random.RandomState(3)
    m = amazon()
    B = 64
    batch = train_batch(rs, B, 20, 3, 256, None if lengths == "full" else rs.randint(1, 21, size=B))
    assert_matches_hf(m, batch)
    m.eval()
    assert_matches_hf(m, batch)                                  # eval mode: no dropout either, gradients still flow


def test_forward_equals_hf_through_torch_compile():
    rs = np.random.RandomState(5)
    m = amazon()
    batch = train_batch(rs, 32, 20, 3, 256, rs.randint(1, 21, size=32))
    compiled = torch.compile(m)
    assert_matches_hf(m, batch, fn=compiled)


def test_dropout_pass_is_reproducible_under_the_seed():
    rs = np.random.RandomState(7)
    m = amazon()
    set_dropout(m, 0.1)
    batch = train_batch(rs, 48, 20, 3, 256, rs.randint(2, 21, size=48))
    runs = []
    for _ in range(2):
        torch.manual_seed(11)
        runs.append(loss_grads(m, batch, "fused"))
    (l1, g1), (l2, g2) = runs
    assert torch.equal(l1, l2)
    # every gradient of the encoder pass; the tables the decoder also reads (item_sid_embedding_table) and the decoder's own
    # parameters go through torch's embedding backward, which sums with atomics
    for name in g1:
        if name.startswith("encoder.") or name == "sep_token":
            assert torch.equal(g1[name], g2[name]), name
    torch.manual_seed(12)
    l3, _ = loss_grads(m, batch, "fused")
    assert not torch.equal(l1, l3)
    set_dropout(m, 0.0)
    torch.manual_seed(11)
    l0, _ = loss_grads(m, batch, "fused")
    assert not torch.equal(l0, l1)                               # dropout really changed the pass


def test_only_the_kept_count_read_synchronises():
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(19)
    m = amazon()
    set_dropout(m, 0.1)
    batch = train_batch(rs, 16, 10, 3, 256, rs.randint(1, 11, size=16))
    loss_grads(m, batch, "fused")                                # warm-up
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
        enc_mask = M._strip_dedup_col(batch.seq_mask.long(), 4, 3)
        ids = M._strip_dedup_col(batch.sem_ids, 4, 3)
        torch.cuda.set_sync_debug_mode("error")
        out, _ = m._fused_train_encoder_pass(enc_mask, ids, batch.user_ids)
        out.square().sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
        M._read_n_kept = read
    assert reads == [1]


def test_forward_encoder_errors():
    from rq_vae_recommender_b200._lib import Rqb200Error
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(23)
    m = amazon()
    batch = train_batch(rs, 4, 3, 3, 256)
    with pytest.raises(ValueError, match="encoder must be one of"):
        m(batch, encoder="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16), pytest.raises(ValueError, match="autocast"):
        m(batch, encoder="fused")
    long = train_batch(rs, 2, 1300, 3, 256)                      # 1300 items * 4 = 5200 positions > 5120
    with pytest.raises(Rqb200Error, match="exceed"):
        m(long, encoder="fused")
    M.DEFAULT_FORWARD_ENCODER = "fused"
    try:
        with highest():
            torch.manual_seed(1)
            a = m(batch).loss
            torch.manual_seed(1)
            b = m(batch, encoder="fused").loss
        assert torch.equal(a, b)
    finally:
        M.DEFAULT_FORWARD_ENCODER = "hf"
