"""GPU tests of the fused T5 decode (csrc/t5dec.cu, modules/model.py FusedT5Decode, generate(decoder="fused")): each kernel
against the plain-torch statement of tests/t5_step_ref.py at "highest" matmul precision, and whole generate against
decoder="hf".  `pytest -m gpu`.

Near-tie rule at the module's "high" (TF32) precision: the two decoders compute the same T5 maths with different GEMM shapes,
so their logits differ by TF32 rounding.  The test measures the largest logit difference D over the same beams and bounds a
candidate's score change by 2 D per level (log_softmax moves by at most 2 D, and each level adds its parent's change).  Beams of
a history may then differ only at a level where HF's own sorted candidate scores hold two neighbours among the first top_k + 1
closer than that bound (a beam swapped in, or two beams swapped in order); every other history's beams must be identical."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import t5_step_ref as T
from parity import load_golden
from test_beam_search_oracle import torch_beam_search
from test_generate_oracle import decoder_batch, decoder_model
from test_gpu_generate import history, realistic_corpus, small_model

pytestmark = pytest.mark.gpu


class highest:
    """torch.set_float32_matmul_precision("highest") inside, the previous setting restored afterwards."""

    def __enter__(self):
        self.saved = torch.get_float32_matmul_precision()
        torch.set_float32_matmul_precision("highest")

    def __exit__(self, *a):
        torch.set_float32_matmul_precision(self.saved)


def rel_err(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("S", [1, 7, 64, 80, 81, 257, 1024])
@pytest.mark.parametrize("nq", [1, 10, 32])
@pytest.mark.parametrize("heads", [1, 2, 6, 8])
def test_cross_attention_kernel(S, nq, heads):
    from rq_vae_recommender_b200 import ops
    B, inner = 5, heads * 64
    g = torch.Generator(device="cuda").manual_seed(S * 100 + nq * 10 + heads)
    q = torch.randn(B * nq, inner, device="cuda", generator=g) * 0.4
    kv = torch.randn(B * S, 3 * inner, device="cuda", generator=g) * 0.4          # k and v are strided views of a wider tensor
    k, v = kv[:, :inner], kv[:, 2 * inner:]
    mask = torch.ones(B, S, device="cuda")
    mask[1, : S // 2] = 0                                                           # padded history
    mask[2] = 0                                                                     # every key masked: the mean of the values
    mask[3] = (torch.rand(S, device="cuda", generator=g) > 0.3).float()
    mask[3, -1] = 1
    with highest():
        want = T.cross_attention(q, k.contiguous(), v.contiguous(), mask, nq, heads)
        want_nomask = T.cross_attention(q, k.contiguous(), v.contiguous(), None, nq, heads)
    got = ops.t5dec_cross_attention(q, k, v, mask, nq, heads)
    assert rel_err(got, want) < 1e-5
    assert rel_err(ops.t5dec_cross_attention(q, k, v, None, nq, heads), want_nomask) < 1e-5
    mean_v = v.reshape(B, S, inner)[2].mean(0)
    assert rel_err(got.reshape(B, nq, inner)[2], mean_v.expand(nq, -1)) < 1e-5


@pytest.mark.parametrize("H", [1, 2, 3, 5, 8])
def test_self_attention_kernel(H):
    from rq_vae_recommender_b200 import ops
    heads, rows = 6, 60
    inner = heads * 64
    g = torch.Generator(device="cuda").manual_seed(H)
    bias = torch.randn(heads, H, H, device="cuda", generator=g)
    for h in range(H):
        R = rows if h else rows // 4
        ck = torch.randn(H, rows, inner, device="cuda", generator=g) * 0.3
        cv = torch.randn(H, rows, inner, device="cuda", generator=g)
        qkv = torch.randn(R, 3 * inner, device="cuda", generator=g) * 0.3
        anc_in = torch.randint(0, R, (rows, H), device="cuda", generator=g, dtype=torch.int32)
        ref_k, ref_v = ck.clone(), cv.clone()
        with highest():
            want = T.self_attention(qkv, ref_k, ref_v, bias, h, anc_in[:R])
        got = ops.t5dec_self_attention(qkv, ck, cv, bias, h, anc_in)
        assert rel_err(got, want) < 1e-5
        assert torch.equal(ck, ref_k) and torch.equal(cv, ref_v)                    # slot h written, nothing else touched
        if h == 0:
            continue
        parent = torch.randint(0, rows, (R,), device="cuda", generator=g)
        anc_out = torch.full((rows, H), -7, dtype=torch.int32, device="cuda")
        adv = T.advance_ancestors(anc_in, parent, h)
        with highest():
            want = T.self_attention(qkv, ref_k, ref_v, bias, h, adv)
        got = ops.t5dec_self_attention(qkv, ck, cv, bias, h, anc_in, parent, anc_out)
        assert rel_err(got, want) < 1e-5
        assert torch.equal(anc_out[:R, :h], adv[:, :h])


def test_add_norm_kernel():
    from rq_vae_recommender_b200 import ops
    R, D, eps = 300, 384, 1e-6
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(R, D, device="cuda", generator=g)
    wide = torch.randn(R, D + 16, device="cuda", generator=g)
    delta = wide[:, :D]
    w = torch.rand(D, device="cuda", generator=g) + 0.5
    x_ref = x.clone()
    with highest():
        want = T.add_norm(x_ref, delta, w, eps)
    out = torch.empty_like(x)
    ops.t5dec_add_norm(x, delta, w, out, eps)
    assert torch.equal(x, x_ref)                                                     # the residual add is one fp32 add
    assert rel_err(out, want) < 1e-6
    # the input embedding: row ids[r] + offset of the table (ids a strided column of generated), and the BOS row for all rows
    table = torch.randn(3 * 256, D, device="cuda", generator=g)
    generated = torch.randint(0, 256, (R // 10, 10, 2), device="cuda", generator=g)
    ids = generated.reshape(R, 2)[:, 1]
    ops.t5dec_add_norm(x, None, w, out, eps, emb=table, ids=ids, offset=256)
    assert torch.equal(x, table[ids + 256])
    assert rel_err(out, T.add_norm(table[ids + 256].clone(), None, w, eps)) < 1e-6
    bos = torch.randn(1, D, device="cuda", generator=g)
    ops.t5dec_add_norm(x, None, w, out, eps, emb=bos)
    assert torch.equal(x, bos.expand(R, -1))
    from rq_vae_recommender_b200._lib import Rqb200Error
    with pytest.raises(Rqb200Error):
        ops.t5dec_add_norm(x.cpu(), None, w.cpu(), out.cpu(), eps)


# ------------------------------------------------------------------------------------------------ whole generate
def amazon_model(M, corpus, seed=0):
    """The T5 shape of configs/decoder_amazon.gin: d_model 384, 6 heads, d_ff 1024, 4 layers, top_k 10, K = 256, 3 levels."""
    torch.manual_seed(seed)
    return M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), num_hierarchies=3, num_embeddings_per_hierarchy=256,
                                          t5_d_model=384, t5_num_heads=6, t5_d_ff=1024, t5_num_layers=4, top_k_for_generation=10,
                                          should_add_sep_token=True, num_user_bins=None).cuda().eval()


def captured_logits(m, fn):
    """Run fn() and return the head logits of every level (forward hooks on decoder_mlp) and fn's result."""
    got = []
    hooks = [mlp.register_forward_hook(lambda mod, inp, out: got.append(out.detach().clone())) for mlp in m.decoder_mlp]
    try:
        res = fn()
    finally:
        for hk in hooks:
            hk.remove()
    return got, res


def both_decoders(m, mask, ids, users, search, seed=5):
    out = {}
    for dec in ("hf", "fused"):
        torch.manual_seed(seed)
        out[dec] = captured_logits(m, lambda: m.generate(mask, ids, users, search=search, decoder=dec))
    return out


# name: (model of a corpus, seed, histories, items per history, K); K = 300 leaves a partial last word in the child masks
SHAPES = {"small": (lambda M, corpus: small_model(M, corpus, 256, 3), 11, 48, 20, 256),
          "decoder_amazon": (amazon_model, 12, 64, 20, 256),
          "small_k300": (lambda M, corpus: small_model(M, corpus, 300, 3), 13, 48, 20, 300)}


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("search", ["sample", "beam"])
def test_generate_fused_equals_hf_at_highest(shape, search):
    from rq_vae_recommender_b200.modules import model as M
    make, seed, B, items, K = SHAPES[shape]
    rs = np.random.RandomState(seed)
    H = 3
    m = make(M, realistic_corpus(rs, 3000, H, K))
    mask, ids, users = history(rs, B, items, H, K)
    with highest():
        runs = both_decoders(m, mask, ids, users, search)
    (lh, (gh, ph)), (lf, (gf, pf)) = runs["hf"], runs["fused"]
    assert len(lh) == len(lf) == H
    for h in range(H):
        err = (lf[h] - lh[h]).abs().max().item()
        assert err <= 1e-5, (h, err)
    assert torch.equal(gf, gh)
    fin = torch.isfinite(ph)
    assert torch.equal(torch.isfinite(pf), fin) and fin.any()
    assert (pf[fin] - ph[fin]).abs().max().item() <= 1e-5


def test_fused_logits_for_given_beams_at_highest():
    """FusedT5Decode against HF's T5Stack for random beams (parents repeated and skipped), levels 0..4 of a 5-level model."""
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(14)
    H, K, B = 5, 64, 40
    m = small_model(M, realistic_corpus(rs, 2000, H, K), K, H)
    mask, ids, users = history(rs, B, 6, H, K)
    with torch.no_grad(), highest():
        enc_out, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
        beams = T.random_beams(B, 10, H, K, seed=15, device="cuda")
        want = T.hf_level_logits(m, enc_out, enc_mask, beams, 10)
        got = T.fused_level_logits(m, enc_out, enc_mask, beams, 10, decode_cls=M.FusedT5Decode)
    for h in range(H):
        assert (got[h] - want[h]).abs().max().item() <= 1e-5, h


def candidate_scores(index, logits, generated, log_probas, k):
    """HF's candidates of one level of the exhaustive search: [B, kp * K] scores, -inf for prefixes absent from the corpus."""
    Kc = logits.shape[1]
    B, kp, h = (logits.shape[0], 1, 0) if generated is None else generated.shape
    codes = torch.arange(Kc, device=logits.device).repeat(B * kp).unsqueeze(1)
    prefix = codes if h == 0 else torch.cat([generated.reshape(-1, h).repeat_interleave(Kc, dim=0), codes], dim=1)
    scores = F.log_softmax(logits, dim=-1).reshape(B, kp * Kc)
    if h:
        scores = scores + log_probas.repeat_interleave(Kc, dim=1)
    return scores.masked_fill(~index.check(prefix).reshape(B, kp * Kc), float("-inf"))


def test_generate_fused_at_high_precision_near_ties_only():
    from rq_vae_recommender_b200.modules import model as M
    assert torch.get_float32_matmul_precision() == "high"
    rs = np.random.RandomState(12)
    K, H, k, B = 256, 3, 10, 64
    m = amazon_model(M, realistic_corpus(rs, 3000, H, K))
    mask, ids, users = history(rs, B, 20, H, K)
    with torch.no_grad():
        enc_out, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
        beams = T.random_beams(B, k, H, K, seed=16, device="cuda")
        want = T.hf_level_logits(m, enc_out, enc_mask, beams, k)
        got = T.fused_level_logits(m, enc_out, enc_mask, beams, k, decode_cls=M.FusedT5Decode)
    D = max((a - b).abs().max().item() for a, b in zip(got, want))
    print(f"largest |logit difference| between the decoders at matmul precision 'high': {D:.3e}")
    assert D < 1e-2
    runs = both_decoders(m, mask, ids, users, "beam")
    (lh, (gh, ph)), (_, (gf, pf)) = runs["hf"], runs["fused"]
    index = m._prefix_index(torch.device("cuda"))
    same_rows = (gf == gh).reshape(B, -1).all(1)
    near_tie = torch.zeros(B, dtype=torch.bool, device="cuda")
    generated, log_probas = None, None
    for h in range(H):
        top = candidate_scores(index, lh[h], generated, log_probas, k).topk(k + 1, dim=1).values
        gaps = (top[:, :-1] - top[:, 1:]).nan_to_num(nan=float("inf"))               # -inf next to -inf: both keep index order
        near_tie |= (gaps < 2 * D * (h + 1)).any(1)
        generated, log_probas, _ = index.beam_topk(lh[h], generated, log_probas, k)  # HF's beams entering the next level
    assert torch.equal(generated, gh)
    print(f"histories with different beams: {int((~same_rows).sum())} of {B}, near-tied: {int(near_tie.sum())}")
    assert bool((same_rows | near_tie).all())
    assert (pf[same_rows] - ph[same_rows]).nan_to_num(neginf=0.0).abs().max().item() <= 2 * D * H


def test_generate_beam_fused_equals_torch_search_on_decoder_golden():
    from rq_vae_recommender_b200.modules import model as M
    g = load_golden("decoder")
    cpu = decoder_model(M, g)
    H = cpu.num_hierarchies
    batch = decoder_batch(g)
    with torch.no_grad():
        want_g, want_p = torch_beam_search(cpu, M._strip_dedup_col(batch.seq_mask.long(), H + 1, H),
                                           M._strip_dedup_col(batch.sem_ids, H + 1, H), batch.user_ids)
    m = decoder_model(M, g).cuda()
    with highest():
        out = m.generate_next_sem_id(decoder_batch(g, "cuda"), search="beam", decoder="fused")
    assert torch.equal(out.sem_ids.cpu(), want_g)
    np.testing.assert_allclose(out.log_probas.cpu().numpy(), want_p.numpy(), rtol=1e-5, atol=1e-5)


def test_generate_items_fused_equals_hf():
    from rq_vae_recommender_b200.modules import model as M
    g = load_golden("decoder")
    m = decoder_model(M, g).cuda()
    batch = decoder_batch(g, "cuda")
    with highest():
        for search in ("sample", "beam"):
            torch.manual_seed(9)
            a = m.generate_items(batch, n=6, search=search, decoder="hf")
            torch.manual_seed(9)
            b = m.generate_items(batch, n=6, search=search, decoder="fused")
            for x, y in zip(a[:4], b[:4]):
                assert torch.equal(x, y)
            fin = torch.isfinite(a.log_probas)
            assert torch.equal(torch.isfinite(b.log_probas), fin)
            assert (a.log_probas[fin] - b.log_probas[fin]).abs().max().item() <= 1e-5


def test_fused_state_is_per_history_and_launches_per_level_are_fixed():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(17)
    K, k = 256, 10
    for H in (3, 5):
        m = small_model(M, realistic_corpus(rs, 3000, H, K), K, H, k=k)
        mask, ids, users = history(rs, 24, 5, H, K)
        states = []
        make = m._fused_decoder
        m._fused_decoder = lambda *a: states.append(make(*a)) or states[-1]
        m.generate(mask, ids, users, decoder="fused")                              # builds the prefix index
        L = len(m.t5_decoder.block)
        for search in ("sample", "beam"):
            before = ops.LAUNCHES
            m.generate(mask, ids, users, search=search, decoder="fused")
            # per level: the input embedding + norm, per layer self-attention, cross-attention and three add + norm, the search
            assert ops.LAUNCHES - before == H * (1 + 5 * L + 1)
        st = states[-1]
        B, S = st.B, st.mask.shape[1]
        assert B == 24
        assert st.cross_kv.shape == (B * S, L * 2 * st.inner)                       # B rows of cross K/V, not B * k
        assert st.cache.shape == (L, 2, H, B * k, st.inner)
        before = ops.LAUNCHES
        m.generate(mask, ids, users, decoder="hf")
        assert ops.LAUNCHES - before == H                                          # the HF path's count is unchanged


def test_fused_errors_on_the_device():
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(18)
    m = small_model(M, realistic_corpus(rs, 500, 3, 256), 256, 3)
    mask, ids, users = history(rs, 4, 3, 3, 256)
    with pytest.raises(ValueError, match="decoder must be one of"):
        m.generate(mask, ids, users, decoder="cuda")
    m.train()
    with pytest.raises(ValueError, match="eval mode only"):
        m.generate(mask, ids, users, decoder="fused")
