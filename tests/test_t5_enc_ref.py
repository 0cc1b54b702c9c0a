"""CPU proof that the packed encoder pass of ``generate(encoder="fused")`` is exact: the plain-torch decomposition of
tests/t5_enc_ref.py (kept positions only, packed, HF's relative bias at the original positions) gives an encoder output within
1e-5 of transformers' T5EncoderModel run through ``encoder_forward_pass`` at every kept position, zeros at the dropped ones, and
the same mask."""
import pytest
import torch

import t5_enc_ref as E
from parity import load_golden
from test_generate_oracle import decoder_batch, decoder_model

MASKS = ("full", "end", "front", "holes", "empty")


def random_model(M, H=3, K=32, sep=True, user_bins=None, seed=0, heads=3, ff="relu"):
    from transformers.models.t5.modeling_t5 import T5Config
    from transformers import T5EncoderModel
    torch.manual_seed(seed)
    m = M.EncoderDecoderRetrievalModel(codebooks=torch.randint(0, K, (100, H)), num_hierarchies=H, num_embeddings_per_hierarchy=K,
                                       t5_d_model=64, t5_num_heads=heads, t5_d_ff=96, t5_num_layers=2, top_k_for_generation=4,
                                       should_add_sep_token=sep, num_user_bins=user_bins)
    if ff != "relu":
        m.encoder = T5EncoderModel(T5Config(vocab_size=H * K, d_model=64, num_heads=heads, d_ff=96, num_layers=2,
                                            feed_forward_proj=ff, is_decoder=False))
    return m.eval()


def inputs(kind, B, items, H, K, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, K, (B, items * H), generator=g)
    users = torch.randint(-60, 60, (B, 1), generator=g)                 # negative ids too: torch.remainder's sign rule
    return E.masks(kind, B, items, H, seed), ids, users


def assert_encoder_matches(m, mask, ids, users):
    with torch.no_grad():
        want, want_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
        got, got_mask = E.encode(m, mask, ids, users)
    assert got.shape == want.shape
    assert torch.equal(got_mask, want_mask) and got_mask.dtype == want_mask.dtype
    kept = got_mask != 0
    kept[~kept.any(1)] = True                                           # a history with nothing unmasked keeps every position
    err = (got[kept] - want[kept]).abs().max().item()
    assert err <= 1e-5, err
    assert torch.equal(got[~kept], torch.zeros_like(got[~kept]))
    return kept


@pytest.mark.parametrize("kind", MASKS)
@pytest.mark.parametrize("sep", [True, False])
@pytest.mark.parametrize("user_bins", [None, 7])
def test_packed_encoder_equals_hf(kind, sep, user_bins):
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, sep=sep, user_bins=user_bins, seed=len(kind) + 10 * sep)
    mask, ids, users = inputs(kind, 6, 5, 3, 32, seed=3)
    kept = assert_encoder_matches(m, mask, ids, users)
    if kind != "full":
        assert not kept.all()
    if kind == "empty":
        # history 0 has no unmasked id: with a user row only that row is kept, without one every position is
        assert int(kept[0].sum()) == (1 if user_bins else kept.shape[1])


def test_fully_masked_history_averages_every_position():
    """Without a user token, HF gives every key of a fully masked history the same score (finfo.min swamps the bias), so each
    output row is the same; keeping all positions reproduces it."""
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, user_bins=None, seed=5)
    mask, ids, users = inputs("full", 3, 4, 3, 32, seed=6)
    mask[1] = 0
    assert_encoder_matches(m, mask, ids, None)
    with torch.no_grad():
        out, _ = E.encode(m, mask, ids, None)
    assert (out[1] != 0).all(1).all()


def test_user_id_without_user_bins_and_user_bins_without_user_id():
    from rq_vae_recommender_b200.modules import model as M
    mask, ids, users = inputs("holes", 4, 3, 3, 32, seed=8)
    assert_encoder_matches(random_model(M, user_bins=None, seed=9), mask, ids, users)
    assert_encoder_matches(random_model(M, user_bins=5, seed=9), mask, ids, None)


def test_decoder_golden_model():
    from rq_vae_recommender_b200.modules import model as M
    g = load_golden("decoder")
    m = decoder_model(M, g)
    batch = decoder_batch(g)
    H = m.num_hierarchies
    mask = M._strip_dedup_col(batch.seq_mask.long(), H + 1, H)
    ids = M._strip_dedup_col(batch.sem_ids, H + 1, H)
    assert (mask == 0).any()
    assert_encoder_matches(m, mask, ids, batch.user_ids)


def test_relative_bias_slice_is_hf_table():
    """rel[n, j - i + S - 1] is compute_bias(S, S)[0, n, i, j] for every query i and key j."""
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, heads=4, seed=12)
    att = m.encoder.encoder.block[0].layer[0].SelfAttention
    for S in (1, 2, 7, 81):
        with torch.no_grad():
            full = att.compute_bias(S, S)[0]
            rel = E.rel_bias(full)
        assert rel.shape == (4, 2 * S - 1)
        i, j = torch.meshgrid(torch.arange(S), torch.arange(S), indexing="ij")
        assert torch.equal(rel[:, j - i + S - 1], full)


def test_packing_order_and_offsets():
    mask = torch.tensor([[1, 1, 0, 0, 1, 1], [0, 0, 0, 0, 0, 0], [0, 0, 1, 1, 1, 1]])
    offs, key_mask = E.offsets(mask, 2, True, False)                    # S = 3 items * 3 = 9
    assert offs.tolist() == [0, 6, 15, 21]                               # 4 ids + 2 separators, all 9, 4 + 2
    assert key_mask[1].item() == torch.finfo(torch.float32).min and key_mask[0].item() == 0
    table = torch.arange(12, dtype=torch.float32)[:, None].repeat(1, 2)
    x, src, slot = E.assemble(mask, torch.ones_like(mask), None, table, torch.full((2,), -1.0), None, 6, 2)
    assert src[:6].tolist() == [0, 1, 2, 6, 7, 8]
    assert x[:6, 0].tolist() == [1, 7, -1, 1, 7, -1]                     # id 1 at levels 0 and 1, then the separator
    assert x[6:15, 0].tolist() == [0, 0, -1] * 3                         # masked ids read row 0
    assert slot[0].tolist() == [0, 1, 2, -1, -1, -1, 3, 4, 5]


def test_encoder_argument_errors():
    """An unknown encoder name, encoder="fused" in training mode, a gated feed-forward and CPU tensors raise."""
    from rq_vae_recommender_b200._lib import Rqb200Error
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M)
    mask, ids, users = inputs("end", 2, 2, 3, 32, seed=41)
    with pytest.raises(ValueError, match="encoder must be one of"):
        m.generate(mask, ids, users, encoder="eager")
    with pytest.raises(Rqb200Error, match="CUDA tensors only"):
        m.generate(mask, ids, users, encoder="fused")
    m.train()
    with pytest.raises(ValueError, match="eval mode only"):
        m.generate(mask, ids, users, encoder="fused")
    with pytest.raises(Rqb200Error, match="relu feed-forward"):
        M.FusedT5Encode(random_model(M, ff="gated-gelu"))
    assert M.ENCODERS == ("hf", "fused") and M.DEFAULT_ENCODER == "hf"


def test_install_encoder_switch():
    import sys

    import rq_vae_recommender_b200.dropin as dropin
    from rq_vae_recommender_b200.modules import model as M
    saved = {name: sys.modules.get(name) for name in ("gin", "modules.model", "init", "distributions")}
    try:
        dropin.install(replace_model=True, encoder="fused")
        assert sys.modules["modules.model"].DEFAULT_ENCODER == "fused"
        assert (M.DEFAULT_SEARCH, M.DEFAULT_DECODER) == ("sample", "hf")
        dropin.install(replace_model=True)
        assert M.DEFAULT_ENCODER == "hf"
        dropin.install(replace_model=True, search="beam", decoder="fused", encoder="fused")
        assert (M.DEFAULT_SEARCH, M.DEFAULT_DECODER, M.DEFAULT_ENCODER) == ("beam", "fused", "fused")
        with pytest.raises(ValueError, match="replace_model"):
            dropin.install(encoder="fused")
        with pytest.raises(ValueError, match="encoder must be"):
            dropin.install(replace_model=True, encoder="eager")
    finally:
        dropin.uninstall()
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod
    assert (M.DEFAULT_SEARCH, M.DEFAULT_DECODER, M.DEFAULT_ENCODER) == ("sample", "hf", "hf")
