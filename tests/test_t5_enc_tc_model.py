"""CPU model of the TF32 tensor-core encoder attention (csrc/t5enc_tc.cu) and its switch (encoder_attention).

``TileModel`` restates the kernels' tiling in plain torch: 64-row query and key tiles clipped at each history's edges and
zero-filled past them, the online softmax in key-tile order, the register A operand built from the accumulator layout with the
0,2,4,6,1,3,5,7 key order of the transposed B staging, the backward's lse recompute, the d_rel bins (two halves of the query
tile, one query row per round, key columns in parallel), and TF32 operand rounding by masking mantissa bits (cvt.rna).  Against
float64 autograd of tests/t5_enc_train_ref.attention_train it must match to fp32 rounding with the TF32 rounding off (so the
tiling itself is exact), and within 1e-2 of each tensor's largest entry with it on."""
import sys

import pytest
import torch

import t5_enc_ref as E
import t5_enc_train_ref as TR
import t5_step_ref as T

TILE = 64
MASKS = ("full", "end", "front", "holes", "empty")


def tf32(x):
    """cvt.rna.tf32.f32: round to the nearest 10-bit mantissa, ties away from zero (the low 13 bits zero)."""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def perm_row(k):
    """K position k of a transposed tile -> the row it holds (tc_perm_row): 0,2,4,6,1,3,5,7 in each group of 8."""
    k = torch.as_tensor(k)
    return (k & ~7) | torch.where((k & 4) != 0, 2 * (k & 3) + 1, 2 * (k & 3))


def a_fragment(acc):
    """The TF32 A fragment of each k8 step as the kernels pass it: thread t of a quad hands its accumulator columns 2t and 2t + 1
    of the 8-column block as A's columns t and t + 4."""
    a = torch.empty_like(acc)
    for blk in range(0, acc.shape[1], 8):
        for t in range(4):
            a[:, blk + t] = acc[:, blk + 2 * t]
            a[:, blk + t + 4] = acc[:, blk + 2 * t + 1]
    return a


def staged_t(rows):
    """The transposing staging copy: tile[d, k] = rows[perm_row(k), d] (64 rows, zero-filled past the history)."""
    return rows[perm_row(torch.arange(rows.shape[0]))].t()


def mma(a, b, rnd):
    """D = A B^T with fp32 accumulation of the (optionally TF32-rounded) operands."""
    if rnd:
        a, b = tf32(a), tf32(b)
    return (a.double() @ b.double().t()).float()


def mma_rs(acc, rows, rnd):
    """D = P . rows for P in the accumulator layout: the A fragment against the permuted transposed staging of rows."""
    return mma(a_fragment(acc), staged_t(rows), rnd)


class TileModel:
    def __init__(self, qkv, src, offs, key_mask, rel, S, keep=None, p=0.0, rnd=True):
        self.qkv, self.src, self.offs, self.km, self.rel, self.S = qkv.float(), src.long(), offs.long(), key_mask.float(), rel.float(), S
        self.heads = rel.shape[0]
        self.keep, self.scale, self.rnd = keep, (1.0 / (1.0 - p) if p > 0 else 1.0), rnd

    def tile(self, b, t0, col):
        """rows t0 .. t0 + 63 of history b, columns col .. col + 63 of `col`'s tensor, zero past the history; positions (-1 past)."""
        tensor, c0 = col
        lo, hi = int(self.offs[b]), int(self.offs[b + 1])
        n = max(0, min(TILE, hi - lo - t0))
        out = torch.zeros(TILE, 64)
        out[:n] = tensor[lo + t0:lo + t0 + n, c0:c0 + 64]
        pos = torch.full((TILE,), -1, dtype=torch.long)
        pos[:n] = self.src[lo + t0:lo + t0 + n] - b * self.S
        return out, pos

    def z(self, b, n, pi, pj):
        if self.keep is None:
            return torch.ones(pi.shape[0], pj.shape[0])
        return self.keep[b, n][pi.clamp_min(0)][:, pj.clamp_min(0)].float() * self.scale

    def scores(self, a, bt, n, b, pi, pj):
        """a . bt^T + (rel[pj - pi] + key_mask): the tile's scores, -inf where the key or the query is past the history."""
        s = mma(a, bt, self.rnd)
        bias = self.rel[n][(pj[None, :] - pi[:, None]).clamp(-(self.S - 1), self.S - 1) + self.S - 1]
        s = s + (bias + self.km[b])
        return s.masked_fill((pj[None, :] < 0) | (pi[:, None] < 0), float("-inf"))

    def forward(self):
        N, inner = self.qkv.shape[0], self.heads * 64
        out, lse = torch.zeros(N, inner), torch.zeros(N, self.heads)
        for b in range(self.offs.shape[0] - 1):
            lo, cnt = int(self.offs[b]), int(self.offs[b + 1] - self.offs[b])
            for n in range(self.heads):
                for q0 in range(0, cnt, TILE):
                    Q, pi = self.tile(b, q0, (self.qkv, n * 64))
                    m, l, o = torch.full((TILE,), float("-inf")), torch.zeros(TILE), torch.zeros(TILE, 64)
                    for t0 in range(0, cnt, TILE):
                        K, pj = self.tile(b, t0, (self.qkv, inner + n * 64))
                        V, _ = self.tile(b, t0, (self.qkv, 2 * inner + n * 64))
                        s = self.scores(Q, K, n, b, pi.clamp_min(0), pj)
                        m_new = torch.maximum(m, s.max(1).values)
                        alpha = torch.exp(m - m_new)
                        pr = torch.exp(s - m_new[:, None])
                        l = l * alpha + pr.sum(1)
                        pr = pr * (self.z(b, n, pi, pj) > 0)
                        o = o * alpha[:, None] + mma_rs(pr, V, self.rnd)
                        m = m_new
                    rows = slice(lo + q0, lo + min(cnt, q0 + TILE))
                    k = rows.stop - rows.start
                    out[rows, n * 64:(n + 1) * 64] = (o / l[:, None] * self.scale)[:k]
                    lse[rows, n] = ((m - self.km[b]) + torch.log(l))[:k]
        return out, lse

    def backward(self, out, dout, lse):
        N, inner = self.qkv.shape[0], self.heads * 64
        dqkv, drel = torch.zeros(N, 3 * inner), torch.zeros(self.heads, 2 * self.S - 1)
        delta = torch.zeros(N, self.heads)
        for n in range(self.heads):
            delta[:, n] = (dout[:, n * 64:(n + 1) * 64] * out[:, n * 64:(n + 1) * 64]).sum(1)
        for b in range(self.offs.shape[0] - 1):
            lo, cnt = int(self.offs[b]), int(self.offs[b + 1] - self.offs[b])
            for n in range(self.heads):
                for q0 in range(0, cnt, TILE):                # the query-major pass: dQ and the d_rel bins
                    Q, pi = self.tile(b, q0, (self.qkv, n * 64))
                    G, _ = self.tile(b, q0, (dout, n * 64))
                    Li, _ = self.tile(b, q0, (torch.nn.functional.pad(lse[:, n:n + 1], (0, 63)), 0))
                    Di, _ = self.tile(b, q0, (torch.nn.functional.pad(delta[:, n:n + 1], (0, 63)), 0))
                    li, di = Li[:, 0], Di[:, 0]
                    dq = torch.zeros(TILE, 64)
                    bins = torch.zeros(2, 2 * self.S - 1)
                    for t0 in range(0, cnt, TILE):
                        K, pj = self.tile(b, t0, (self.qkv, inner + n * 64))
                        V, _ = self.tile(b, t0, (self.qkv, 2 * inner + n * 64))
                        s = self.scores(Q, K, n, b, pi, pj)
                        pr = torch.exp((s - self.km[b]) - li[:, None])     # recomputed from the saved lse
                        ds = pr * (mma(G, V, self.rnd) * self.z(b, n, pi, pj) - di[:, None])
                        dq = dq + mma_rs(ds, K, self.rnd)
                        for half in range(2):                     # one query row per round, the key columns in parallel
                            for i in range(32 * half, 32 * half + 32):
                                ok = (pj >= 0) & (pi[i] >= 0)
                                bins[half].index_add_(0, (pj - pi[i] + self.S - 1)[ok], ds[i][ok])
                    k = min(cnt - q0, TILE)
                    dqkv[lo + q0:lo + q0 + k, n * 64:(n + 1) * 64] = dq[:k]
                    drel[n] += bins[0] + bins[1]
                for k0 in range(0, cnt, TILE):                # the key-major pass: dK and dV
                    K, pj = self.tile(b, k0, (self.qkv, inner + n * 64))
                    V, _ = self.tile(b, k0, (self.qkv, 2 * inner + n * 64))
                    dk, dv = torch.zeros(TILE, 64), torch.zeros(TILE, 64)
                    for t0 in range(0, cnt, TILE):
                        Q, pi = self.tile(b, t0, (self.qkv, n * 64))
                        G, _ = self.tile(b, t0, (dout, n * 64))
                        Li, _ = self.tile(b, t0, (torch.nn.functional.pad(lse[:, n:n + 1], (0, 63)), 0))
                        Di, _ = self.tile(b, t0, (torch.nn.functional.pad(delta[:, n:n + 1], (0, 63)), 0))
                        bias = self.rel[n][(pj[:, None] - pi[None, :]).clamp(-(self.S - 1), self.S - 1) + self.S - 1]
                        st = mma(K, Q, self.rnd) + (bias + self.km[b])    # keys as rows: S^T = K Q^T
                        st = st.masked_fill((pj[:, None] < 0) | (pi[None, :] < 0), float("-inf"))
                        pr = torch.exp((st - self.km[b]) - Li[:, 0][None, :])
                        zt = self.z(b, n, pi, pj).t()
                        ds = pr * (mma(V, G, self.rnd) * zt - Di[:, 0][None, :])
                        dv = dv + mma_rs(pr * zt, G, self.rnd)
                        dk = dk + mma_rs(ds, Q, self.rnd)
                    k = min(cnt - k0, TILE)
                    dqkv[lo + k0:lo + k0 + k, inner + n * 64:inner + (n + 1) * 64] = dk[:k]
                    dqkv[lo + k0:lo + k0 + k, 2 * inner + n * 64:2 * inner + (n + 1) * 64] = dv[:k]
        return dqkv, drel


def packed(S, seed, kinds=MASKS):
    keep = torch.cat([E.masks(kind, 2, S, 1, seed) for kind in kinds]).bool()
    empty = ~keep.any(1)
    keep[empty] = True
    key_mask = torch.where(empty, T.NEG, 0.0).float()
    counts = keep.sum(1)
    offs = torch.cat([counts.new_zeros(1), counts.cumsum(0)]).to(torch.int32)
    src = keep.reshape(-1).nonzero().squeeze(1).to(torch.int32)
    return offs, src, key_mask, keep.shape[0]


def rel_err(a, b):
    return ((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("S", [20, 81, 300, 800])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_tile_model_against_float64(S, p):
    offs, src, key_mask, B = packed(S, S)
    heads = 1 if S >= 300 else 2
    g = torch.Generator().manual_seed(S)
    N, inner = src.shape[0], heads * 64
    qkv = torch.randn(N, 3 * inner, generator=g) * 0.3
    rel = torch.randn(heads, 2 * S - 1, generator=g)
    dout = torch.randn(N, inner, generator=g)
    keep = (torch.rand(B, heads, S, S, generator=g) >= p).to(torch.uint8) if p > 0 else None
    q64, r64 = qkv.double().requires_grad_(), rel.double().requires_grad_()
    want = TR.attention_train(q64, src, offs, key_mask.double(), r64, S, keep, p)
    want.backward(dout.double())
    refs = {"out": want.detach(), "dq": q64.grad[:, :inner], "dk": q64.grad[:, inner:2 * inner], "dv": q64.grad[:, 2 * inner:],
            "drel": r64.grad}
    for rnd, bound in ((False, 1e-5), (True, 1e-2)):
        model = TileModel(qkv, src, offs, key_mask, rel, S, keep, p, rnd)
        out, lse = model.forward()
        dqkv, drel = model.backward(out, dout, lse)
        got = {"out": out, "dq": dqkv[:, :inner], "dk": dqkv[:, inner:2 * inner], "dv": dqkv[:, 2 * inner:], "drel": drel}
        for name, ref in refs.items():
            assert rel_err(got[name], ref) < bound, (S, p, rnd, name, rel_err(got[name], ref))


def test_k_permutation_makes_the_accumulator_the_a_fragment():
    g = torch.Generator().manual_seed(1)
    acc, v = torch.randn(64, 64, generator=g), torch.randn(64, 64, generator=g)
    assert sorted(perm_row(torch.arange(8)).tolist()) == list(range(8))
    assert perm_row(torch.arange(8)).tolist() == [0, 2, 4, 6, 1, 3, 5, 7]
    assert torch.allclose(mma_rs(acc, v, False), (acc.double() @ v.double()).float(), atol=1e-4)
    # without the permutation the fragment pairs the wrong keys
    assert not torch.allclose(mma(a_fragment(acc), v.t(), False), (acc.double() @ v.double()).float(), atol=1e-2)


def test_tf32_rounding_keeps_ten_mantissa_bits():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 2 ** -10, -(1.0 + 3 * 2 ** -12), 3.0e-3])
    r = tf32(x)
    assert r[0] == 1.0 and r[1] == 1.0 + 2 ** -10 and r[2] == 1.0 + 2 ** -10 and r[3] == -(1.0 + 2 ** -10)
    assert ((r.view(torch.int32) & 0x1FFF) == 0).all()
    assert ((r - x).abs() <= x.abs() * 2 ** -11).all()


# ------------------------------------------------------------------------------------------------ the switch
def test_encoder_attention_switch():
    from rq_vae_recommender_b200.modules import model as M
    from test_t5_enc_ref import random_model
    assert M.ENCODERS == ("hf", "fused") and M.DECODERS == ("hf", "fused")
    assert M.DEFAULT_ENCODER_ATTENTION == "fp32" and M.ENCODER_ATTENTIONS == ("fp32", "tf32")
    assert M._encoder_attention("fused", None, "x") == "fp32"
    assert M._encoder_attention("fused", "tf32", "x") == "tf32"
    assert M._encoder_attention("hf", None, "x") == "fp32"
    with pytest.raises(ValueError, match="encoder_attention must be one of"):
        M._encoder_attention("fused", "bf16", "x")
    with pytest.raises(ValueError, match="tf32"):
        M._encoder_attention("hf", "tf32", "x")
    m = random_model(M)
    mask = torch.ones(2, 6, dtype=torch.long)
    ids = torch.zeros(2, 6, dtype=torch.long)
    with pytest.raises(ValueError, match="encoder_attention"):
        m.generate(mask, ids, encoder="hf", encoder_attention="tf32")
    with pytest.raises(ValueError, match="encoder_attention must be one of"):
        m.generate(mask, ids, encoder="fused", encoder_attention="fp16")
    with pytest.raises(ValueError):
        M.FusedT5Encode(m, "fp16")
    with pytest.raises(ValueError):
        M.FusedT5EncodeTrain(m.train(), "fp16")
    from rq_vae_recommender_b200 import ops
    assert M.FusedT5Encode(m).attention is ops.t5enc_attention
    assert M.FusedT5Encode(m, "tf32").attention is ops.t5enc_attention_tc
    assert M.FusedT5EncodeTrain(m).attention is ops.T5EncAttentionFunction
    assert M.FusedT5EncodeTrain(m, "tf32").attention is ops.T5EncAttentionTCFunction
    M.DEFAULT_ENCODER_ATTENTION = "bf16"
    try:
        with pytest.raises(ValueError, match="encoder_attention must be one of"):
            m.eval().generate(mask, ids, encoder="fused")
    finally:
        M.DEFAULT_ENCODER_ATTENTION = "fp32"


def test_dropin_encoder_attention():
    import rq_vae_recommender_b200.dropin as dropin
    from rq_vae_recommender_b200.modules import model as M
    saved = {name: sys.modules.get(name) for name in ("gin", "modules.model", "init", "distributions")}
    try:
        dropin.install(replace_model=True, encoder_attention="tf32")
        assert sys.modules["modules.model"].DEFAULT_ENCODER_ATTENTION == "tf32"
        assert (M.DEFAULT_ENCODER, M.DEFAULT_FORWARD_ENCODER) == ("hf", "hf")
        dropin.install(replace_model=True)
        assert M.DEFAULT_ENCODER_ATTENTION == "fp32"
        dropin.install(replace_model=True, encoder="fused", forward_encoder="fused", encoder_attention="tf32")
        assert (M.DEFAULT_ENCODER, M.DEFAULT_FORWARD_ENCODER, M.DEFAULT_ENCODER_ATTENTION) == ("fused", "fused", "tf32")
        with pytest.raises(ValueError, match="replace_model"):
            dropin.install(encoder_attention="tf32")
        with pytest.raises(ValueError, match="encoder_attention must be"):
            dropin.install(replace_model=True, encoder_attention="bf16")
    finally:
        dropin.uninstall()
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod
    assert M.DEFAULT_ENCODER_ATTENTION == "fp32" and M.DEFAULT_ENCODER == "hf"
