"""GPU tests of the fused T5 encoder pass (csrc/t5enc.cu, modules/model.py FusedT5Encode, generate(encoder="fused")): each kernel
against the plain-torch statement of tests/t5_enc_ref.py at "highest" matmul precision, the whole pass against
encoder_forward_pass, and whole generate against the all-HF path.  `pytest -m gpu`.

Near-tie rule at the module's "high" (TF32) precision, as in tests/test_gpu_decode.py: the two encoders compute the same T5 maths
with different GEMM shapes, so the decoder's logits differ by TF32 rounding.  The test measures the largest logit difference D
over the same beams and bounds a candidate's score change by 2 D per level.  Beams of a history may then differ only at a level
where HF's own sorted candidate scores hold two neighbours among the first top_k + 1 closer than that bound."""
import numpy as np
import pytest
import torch

import t5_enc_ref as E
import t5_step_ref as T
from parity import load_golden
from test_generate_oracle import decoder_batch, decoder_model
from test_gpu_decode import SHAPES, amazon_model, candidate_scores, captured_logits, highest, rel_err
from test_gpu_generate import history, realistic_corpus, small_model

pytestmark = pytest.mark.gpu

MASKS = ("full", "end", "front", "holes", "empty")


def masked_batch(items, H, K, seed, B_per_kind=3):
    """One batch holding every mask kind of t5_enc_ref.masks (B_per_kind histories each) and negative user ids."""
    mask = torch.cat([E.masks(kind, B_per_kind, items, H, seed) for kind in MASKS]).cuda()
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, K, mask.shape, generator=g).cuda()
    users = torch.randint(-500, 500, (mask.shape[0], 1), generator=g).cuda()
    return mask, ids, users


def model_of(M, H, K, sep, user_bins, d=64, heads=2, layers=2, seed=0):
    torch.manual_seed(seed)
    corpus = torch.randint(0, K, (200, H))
    return M.EncoderDecoderRetrievalModel(codebooks=corpus, num_hierarchies=H, num_embeddings_per_hierarchy=K, t5_d_model=d,
                                          t5_num_heads=heads, t5_d_ff=2 * d, t5_num_layers=layers, top_k_for_generation=4,
                                          should_add_sep_token=sep, num_user_bins=user_bins).cuda().eval()


def kept_rows(enc_mask):
    kept = enc_mask != 0
    kept[~kept.any(1)] = True
    return kept


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("sep", [True, False])
@pytest.mark.parametrize("user", [True, False])
def test_offsets_and_assembly_kernels(sep, user):
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    H, K, items = 3, 64, 7
    m = model_of(M, H, K, sep, 11 if user else None, d=96, seed=1)
    mask, ids, users = masked_batch(items, H, K, seed=2)
    users = users if user else None
    eps, w = 1e-6, torch.rand(96, device="cuda") + 0.5
    table, sep_row = m.item_sid_embedding_table.weight.detach(), m.sep_token.detach() if sep else None
    utab = m.user_embedding.weight.detach() if user else None
    offs, key_mask = ops.t5enc_offsets(mask, H, sep, user)
    want_offs, want_km = E.offsets(mask, H, sep, user)
    assert torch.equal(offs, want_offs) and torch.equal(key_mask, want_km)
    N = int(offs[-1])
    x, out, src, slot = ops.t5enc_assemble(mask, ids, users, table, sep_row, utab, K, H, offs, N, w, eps)
    want_x, want_src, want_slot = E.assemble(mask, ids, users, table, sep_row, utab, K, H)
    assert torch.equal(x, want_x)                                                    # gathered rows: bit-exact
    assert torch.equal(src, want_src) and torch.equal(slot, want_slot)
    with highest():
        assert rel_err(out, T.add_norm(want_x.clone(), None, w, eps)) < 1e-6
    # an id outside the table gives a NaN row (the mask keeps it), like t5dec_add_norm
    bad = ids.clone()
    bad[0, 0] = K * H
    x, out, src, _ = ops.t5enc_assemble(mask, bad, users, table, sep_row, utab, K, H, offs, N, w, eps)
    row = int(slot[0, 1 if user else 0])
    assert mask[0, 0] != 0 and torch.isnan(x[row]).all() and torch.isnan(out[row]).all()
    assert not torch.isnan(x[row + 1:]).any()


@pytest.mark.parametrize("S", [1, 7, 80, 81, 257, 800])
@pytest.mark.parametrize("heads", [1, 2, 6, 8])
def test_attention_kernel(S, heads):
    """Histories of S positions kept by every mask kind (one with nothing unmasked: all kept, every key at -FLT_MAX)."""
    from rq_vae_recommender_b200 import ops
    g = torch.Generator().manual_seed(S * 10 + heads)
    keep = torch.cat([E.masks(kind, 2, S, 1, S + heads) for kind in MASKS]).bool()
    B = keep.shape[0]
    empty = ~keep.any(1)
    keep[empty] = True
    key_mask = torch.where(empty, T.NEG, 0.0).float().cuda()
    counts = keep.sum(1)
    offs = torch.cat([counts.new_zeros(1), counts.cumsum(0)]).to(torch.int32).cuda()
    src = keep.reshape(-1).nonzero().squeeze(1).to(torch.int32).cuda()
    N, inner = src.shape[0], heads * 64
    qkv = (torch.randn(N, 3 * inner, generator=g) * 0.3).cuda()
    rel = torch.randn(heads, 2 * S - 1, generator=g).cuda()
    with highest():
        want = E.attention(qkv, src, offs, key_mask, rel, S)
    got = ops.t5enc_attention(qkv, src, offs, key_mask, rel, S)
    assert rel_err(got, want) < 1e-5
    # the fully masked histories average every value
    for b in empty.nonzero().squeeze(1).tolist():
        lo, hi = int(offs[b]), int(offs[b + 1])
        assert rel_err(got[lo:hi], qkv[lo:hi, 2 * inner:].mean(0).expand(hi - lo, -1)) < 1e-5
    assert empty.any()


def test_scatter_kernel():
    from rq_vae_recommender_b200 import ops
    rows = torch.randn(50, 96, device="cuda")
    slot = torch.full((6, 20), -1, dtype=torch.int32, device="cuda")
    slot.view(-1)[torch.randperm(120, device="cuda")[:50]] = torch.arange(50, dtype=torch.int32, device="cuda")
    assert torch.equal(ops.t5enc_scatter(rows, slot), E.scatter(rows, slot))


# ------------------------------------------------------------------------------------------------ whole encoder pass
CASES = [(sep, bins) for sep in (True, False) for bins in (None, 11)]


@pytest.mark.parametrize("sep,user_bins", CASES)
@pytest.mark.parametrize("items", [1, 20, 200])
def test_encoder_equals_hf_at_highest(sep, user_bins, items):
    from rq_vae_recommender_b200.modules import model as M
    H, K = 3, 64
    m = model_of(M, H, K, sep, user_bins, d=128, heads=2, seed=items)
    mask, ids, users = masked_batch(items, H, K, seed=items, B_per_kind=2 if items == 200 else 4)
    with torch.no_grad(), highest():
        want, want_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
        got, got_mask = m._fused_encoder()(mask, ids, users)
    assert torch.equal(got_mask, want_mask) and got_mask.dtype == want_mask.dtype
    kept = kept_rows(got_mask)
    if items < 200:
        assert (got[kept] - want[kept]).abs().max().item() <= 1e-5
    else:
        # 800 keys: fp32 sums in cuBLAS's order and the kernel's differ by up to ~1.3e-5 at outputs of magnitude ~4, so the
        # bound is relative to the largest output
        assert rel_err(got[kept], want[kept]) < 1e-5
    assert torch.equal(got[~kept], torch.zeros_like(got[~kept]))


def test_encoder_equals_hf_on_decoder_amazon_shape():
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(3)
    m = amazon_model(M, realistic_corpus(rs, 3000, 3, 256))
    mask, ids, users = history(rs, 64, 20, 3, 256)                   # the first item of half the histories is masked: a hole
    with torch.no_grad(), highest():
        want, want_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
        got, got_mask = m._fused_encoder()(mask, ids, users)
    kept = kept_rows(got_mask)
    assert torch.equal(got_mask, want_mask) and not kept.all()
    assert (got[kept] - want[kept]).abs().max().item() <= 1e-5
    assert (got[~kept] == 0).all()


# ------------------------------------------------------------------------------------------------ whole generate
def encoder_runs(m, mask, ids, users, search, decoder, seed=5):
    out = {}
    for enc in ("hf", "fused"):
        torch.manual_seed(seed)
        out[enc] = captured_logits(m, lambda: m.generate(mask, ids, users, search=search,
                                                         decoder="hf" if enc == "hf" else decoder, encoder=enc))
    return out


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("search", ["sample", "beam"])
@pytest.mark.parametrize("decoder", ["hf", "fused"])
def test_generate_fused_encoder_equals_hf_at_highest(shape, search, decoder):
    from rq_vae_recommender_b200.modules import model as M
    make, seed, B, items, K = SHAPES[shape]
    rs = np.random.RandomState(seed)
    H = 3
    m = make(M, realistic_corpus(rs, 3000, H, K))
    mask, ids, users = history(rs, B, items, H, K)
    mask[-3:, : 12 * H] = 0                                                         # some shorter histories too
    with highest():
        runs = encoder_runs(m, mask, ids, users, search, decoder)
    (lh, (gh, ph)), (lf, (gf, pf)) = runs["hf"], runs["fused"]
    for h in range(H):
        assert (lf[h] - lh[h]).abs().max().item() <= 1e-5, h
    assert torch.equal(gf, gh)
    fin = torch.isfinite(ph)
    assert torch.equal(torch.isfinite(pf), fin) and fin.any()
    assert (pf[fin] - ph[fin]).abs().max().item() <= 1e-5


def test_generate_items_fused_encoder_equals_hf():
    from rq_vae_recommender_b200.modules import model as M
    g = load_golden("decoder")
    m = decoder_model(M, g).cuda()
    batch = decoder_batch(g, "cuda")
    with highest():
        for search in ("sample", "beam"):
            for decoder in ("hf", "fused"):
                torch.manual_seed(9)
                a = m.generate_items(batch, n=6, search=search)
                torch.manual_seed(9)
                b = m.generate_items(batch, n=6, search=search, decoder=decoder, encoder="fused")
                for x, y in zip(a[:4], b[:4]):
                    assert torch.equal(x, y)
                fin = torch.isfinite(a.log_probas)
                assert torch.equal(torch.isfinite(b.log_probas), fin)
                assert (a.log_probas[fin] - b.log_probas[fin]).abs().max().item() <= 1e-5


def test_generate_fused_encoder_at_high_precision_near_ties_only():
    from rq_vae_recommender_b200.modules import model as M
    assert torch.get_float32_matmul_precision() == "high"
    rs = np.random.RandomState(12)
    K, H, k, B = 256, 3, 10, 64
    m = amazon_model(M, realistic_corpus(rs, 3000, H, K))
    mask, ids, users = history(rs, B, 20, H, K)
    with torch.no_grad():
        enc_h, mask_h = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
        enc_f, _ = m._fused_encoder()(mask, ids, users)
        beams = T.random_beams(B, k, H, K, seed=16, device="cuda")
        want = T.hf_level_logits(m, enc_h, mask_h, beams, k)
        got = T.hf_level_logits(m, enc_f, mask_h, beams, k)
    D = max((a - b).abs().max().item() for a, b in zip(got, want))
    print(f"largest |logit difference| between the encoders at matmul precision 'high': {D:.3e}")
    assert D < 1e-2
    runs = encoder_runs(m, mask, ids, users, "beam", "hf")
    (lh, (gh, ph)), (_, (gf, pf)) = runs["hf"], runs["fused"]
    index = m._prefix_index(torch.device("cuda"))
    same_rows = (gf == gh).reshape(B, -1).all(1)
    near_tie = torch.zeros(B, dtype=torch.bool, device="cuda")
    generated, log_probas = None, None
    for h in range(H):
        top = candidate_scores(index, lh[h], generated, log_probas, k).topk(k + 1, dim=1).values
        gaps = (top[:, :-1] - top[:, 1:]).nan_to_num(nan=float("inf"))
        near_tie |= (gaps < 2 * D * (h + 1)).any(1)
        generated, log_probas, _ = index.beam_topk(lh[h], generated, log_probas, k)
    assert torch.equal(generated, gh)
    print(f"histories with different beams: {int((~same_rows).sum())} of {B}, near-tied: {int(near_tie.sum())}")
    assert bool((same_rows | near_tie).all())
    assert (pf[same_rows] - ph[same_rows]).nan_to_num(neginf=0.0).abs().max().item() <= 2 * D * H


# ------------------------------------------------------------------------------------------------ launches, host sync, errors
def test_launches_are_fixed_and_state_is_packed():
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(17)
    K, H = 256, 3
    m = small_model(M, realistic_corpus(rs, 3000, H, K), K, H)
    L, Ld = len(m.encoder.encoder.block), len(m.t5_decoder.block)
    states = []
    make = m._fused_encoder
    m._fused_encoder = lambda: states.append(make()) or states[-1]
    m.generate(*history(rs, 8, 5, H, K), encoder="fused")                          # builds the prefix index
    for items in (1, 5, 20):
        mask, ids, users = history(rs, 24, items, H, K)
        mask[:6, H:] = 0                                                            # a few one-item histories
        before = ops.LAUNCHES
        _, enc_mask = m._fused_encoder()(mask, ids, users)
        # offsets, assembly + first norm, per layer attention and two add + norm, the scatter
        assert ops.LAUNCHES - before == 3 + 3 * L
        kept = kept_rows(enc_mask)
        assert states[-1].n_kept == int(kept.sum()) < kept.numel()
        for search in ("sample", "beam"):
            for decoder, per_level in (("hf", 1), ("fused", 1 + 5 * Ld + 1)):
                before = ops.LAUNCHES
                m.generate(mask, ids, users, search=search, decoder=decoder, encoder="fused")
                assert ops.LAUNCHES - before == 3 + 3 * L + H * per_level


def test_only_the_kept_count_read_synchronises():
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(19)
    m = small_model(M, realistic_corpus(rs, 500, 3, 256), 256, 3)
    mask, ids, users = history(rs, 16, 10, 3, 256)
    m._fused_encoder()(mask, ids, users)                                            # warm-up: module loads, cuBLAS handles
    read = M._read_n_kept
    reads = []

    def allowed(offsets):                                                           # the one documented synchronisation
        reads.append(1)
        torch.cuda.set_sync_debug_mode(0)
        try:
            return read(offsets)
        finally:
            torch.cuda.set_sync_debug_mode("error")

    torch.cuda.synchronize()
    M._read_n_kept = allowed
    torch.cuda.set_sync_debug_mode("error")
    try:
        with pytest.raises(RuntimeError):
            read(torch.zeros(2, dtype=torch.int32, device="cuda"))                 # the mode is on: an unmarked read raises
        with torch.no_grad():
            out, _ = m._fused_encoder()(mask, ids, users)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        M._read_n_kept = read
    assert reads == [1]
    assert out.shape[0] == 16


def test_fused_encoder_errors():
    from rq_vae_recommender_b200._lib import Rqb200Error
    from rq_vae_recommender_b200.modules import model as M
    rs = np.random.RandomState(18)
    m = small_model(M, realistic_corpus(rs, 500, 3, 256), 256, 3)
    mask, ids, users = history(rs, 4, 3, 3, 256)
    with pytest.raises(ValueError, match="encoder must be one of"):
        m.generate(mask, ids, users, encoder="cuda")
    with pytest.raises(Rqb200Error, match="CUDA tensors only"):
        m._fused_encoder()(mask.cpu(), ids.cpu(), users.cpu())
    m.train()
    with pytest.raises(ValueError, match="eval mode only"):
        m.generate(mask, ids, users, encoder="fused")
