"""CPU proof that the fused training decoder pass of ``forward(decoder="fused")`` is exact: the float64 statement of
tests/t5_dec_train_ref.py (the H positions the loss reads, either key layout), with explicit keep masks, gives the same loss and
the same gradient for every parameter as ``forward(encoder="hf", decoder="hf")`` in training mode when HF's dropout calls apply
the same masks in call order.  Also the argument errors and the ``dropin`` switch of the training decoder."""
import copy

import pytest
import torch

import t5_dec_train_ref as DR
import t5_enc_train_ref as TR
from test_t5_enc_ref import inputs, random_model
from test_t5_enc_train_ref import _cuda_autocast_flag, loss_and_grads


def batch_of(mask, ids, users, H, K, seed):
    """A TokenizedSeqBatch whose stripped ids and mask are ids and mask (the dedup column copies the item's last id's mask)."""
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    B, n = ids.shape
    g = torch.Generator().manual_seed(seed)
    sem = torch.cat([ids.view(B, n // H, H), torch.randint(0, 3, (B, n // H, 1), generator=g)], dim=2).reshape(B, -1)
    m = mask.view(B, n // H, H)
    seq_mask = torch.cat([m, m[:, :, -1:]], dim=2).reshape(B, -1).bool()
    fut = torch.randint(0, K, (B, H + 1), generator=g)
    return TokenizedSeqBatch(user_ids=users, sem_ids=sem, sem_ids_fut=fut, seq_mask=seq_mask, token_type_ids=torch.zeros_like(sem),
                             token_type_ids_fut=torch.zeros_like(fut))


def set_dropout(m, p):
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = p
        if type(mod).__name__ == "T5Attention":
            mod.dropout = p


def compare(m, batch, layout, p, seed):
    """HF's fp32 forward in training mode against the encoder (HF's, or the packed statement) plus the float64 decoder statement
    on a float64 copy: loss within 1e-5 relative, each parameter's gradient within 1e-5 of its largest entry."""
    from rq_vae_recommender_b200.modules import model as M
    m = m.float().train()
    set_dropout(m, p)
    H = m.num_hierarchies
    mask = M._strip_dedup_col(batch.seq_mask.long(), H + 1, H)
    ids = M._strip_dedup_col(batch.sem_ids, H + 1, H)
    fut = batch.sem_ids_fut[:, :H]
    sep, user = m.sep_token is not None, m.user_embedding is not None
    with torch.no_grad():
        _, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=batch.user_ids)
    B, S = enc_mask.shape
    enc_masks = TR.random_masks(m, B, S, p, seed)
    dec_masks = DR.random_masks(m, B, H, S, p, seed + 100)
    m64 = copy.deepcopy(m).double()

    def patched(masks, fn):
        fake = TR.hf_dropout_from(masks)
        real = torch.nn.functional.dropout
        torch.nn.functional.dropout = fake
        try:
            out = fn()
        finally:
            torch.nn.functional.dropout = real
        assert not fake.queue
        return out

    def hf():
        return patched(enc_masks + dec_masks, lambda: m(batch, encoder="hf", decoder="hf").loss)

    def statement():
        # the encoder statement of tests/t5_enc_train_ref.py (HF's own float64 encoder overflows finfo(float64).min for a fully
        # masked history); its [B, S, d] output is HF's at the kept positions and 0 at the others, which get weight 0
        out, em = TR.encode_train(m64, mask, ids, batch.user_ids, enc_masks, p)
        keys = DR.packed_layout(out, mask, H, sep, user) if layout == "packed" else DR.padded_layout(out, em)
        return DR.level_loss(m64, DR.decode_train(m64, fut, *keys, dec_masks, p), fut)

    want_loss, want = loss_and_grads(m, hf)
    got_loss, got = loss_and_grads(m64, statement)
    assert torch.isfinite(want_loss)
    assert abs(got_loss.item() - want_loss.item()) <= 1e-5 * max(1.0, abs(want_loss.item()))
    for name in want:
        scale = max(want[name].abs().max().item(), 1e-30)
        err = (got[name] - want[name].double()).abs().max().item()
        assert err <= 1e-5 * scale, (name, err, scale)
    return want


@pytest.mark.parametrize("layout", ["packed", "padded"])
@pytest.mark.parametrize("kind", ["full", "end", "holes", "empty"])
@pytest.mark.parametrize("sep,user_bins", [(True, None), (False, 7), (True, 7)])
def test_decoder_statement_equals_hf(layout, kind, sep, user_bins):
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, sep=sep, user_bins=user_bins, seed=len(kind) + 10 * sep)
    mask, ids, users = inputs(kind, 5, 4, 3, 32, seed=3)
    grads = compare(m, batch_of(mask, ids, users, 3, 32, seed=1), layout, p=0.1, seed=len(kind))
    assert grads["t5_decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"].abs().max() > 0
    assert grads["item_sid_embedding_table.weight"].abs().max() > 0 and grads["bos_token"].abs().max() > 0


@pytest.mark.parametrize("layout", ["packed", "padded"])
def test_five_levels_and_fully_masked_histories(layout):
    """H = 5, and histories with nothing unmasked and no user row: their cross-attention averages every encoder position."""
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, H=5, user_bins=None, seed=5)
    mask, ids, users = inputs("holes", 4, 3, 5, 32, seed=6)
    mask[1] = 0
    compare(m, batch_of(mask, ids, users, 5, 32, seed=2), layout, p=0.1, seed=2)
    mask[:] = 0
    compare(m, batch_of(mask, ids, users, 5, 32, seed=3), layout, p=0.0, seed=3)


def gated_decoder_model(M):
    from transformers.models.t5.modeling_t5 import T5Config, T5Stack
    m = random_model(M)
    m.t5_decoder = T5Stack(T5Config(vocab_size=96, d_model=64, num_heads=3, d_ff=96, num_layers=2, feed_forward_proj="gated-gelu",
                                    is_decoder=True, is_encoder_decoder=False))
    return m


def test_forward_decoder_argument_errors():
    from rq_vae_recommender_b200._lib import Rqb200Error
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M)
    assert M.DEFAULT_FORWARD_DECODER == "hf"
    with pytest.raises(ValueError, match="decoder must be one of"):
        m.forward(None, decoder="eager")
    with pytest.raises(Rqb200Error, match="relu feed-forward"):
        M.FusedT5DecodeTrain(gated_decoder_model(M))
    with pytest.raises(Rqb200Error, match="levels exceed"):
        M.FusedT5DecodeTrain(random_model(M, H=9))
    with pytest.raises(Rqb200Error, match="fp32 parameters"):
        M.FusedT5DecodeTrain(random_model(M).double())
    B, S = 2, 5
    fut = torch.zeros(B, 3, dtype=torch.long)
    rows, offs = torch.zeros(B * S, 64), torch.arange(0, (B + 1) * S, S, dtype=torch.int32)
    with pytest.raises(Rqb200Error, match="CUDA tensors only"):
        M.FusedT5DecodeTrain(m)(fut, rows, offs, torch.zeros(B * S), None, S)
    with _cuda_autocast_flag(), pytest.raises(ValueError, match="autocast"):
        M.FusedT5DecodeTrain(m)(fut, rows, offs, torch.zeros(B * S), None, S)


def test_encoder_rows_layout():
    """``PackedEncoderOutput.keys``: the rows, offsets and per-row key mask the offsets-based cross-attentions read, from HF's
    padded output (every position a row) and from a packed pass (a row takes its history's key mask)."""
    from rq_vae_recommender_b200.modules import model as M
    B, S, d = 3, 4, 5
    fmin = torch.finfo(torch.float32).min
    enc_out = torch.arange(B * S * d, dtype=torch.float32).view(B, S, d)
    enc_mask = torch.tensor([[1., 1, 0, 1], [0, 0, 0, 0], [1, 1, 1, 1]])
    rows, offsets, key_mask, src, S_ = M.PackedEncoderOutput.of_padded(enc_out, enc_mask).keys()
    assert src is None and S_ == S
    assert torch.equal(rows, enc_out.reshape(B * S, d))                             # history b's rows: b * S .. b * S + S - 1
    assert offsets.dtype == torch.int32 and offsets.tolist() == [0, 4, 8, 12]
    assert key_mask.dtype == torch.float32 and key_mask.tolist() == [0, 0, fmin, 0] + [fmin] * 4 + [0] * 4
    packed = M.PackedEncoderOutput(rows[:5], torch.tensor([0, 2, 4, 5], dtype=torch.int32), torch.tensor([0., fmin, 0.]),
                                   torch.tensor([0, 3, 4, 5, 8], dtype=torch.int32), None, S, enc_mask)
    assert packed.keys()[2].tolist() == [0, 0, fmin, fmin, 0] and packed.keys()[3] is packed.src


def test_install_forward_decoder_switch():
    import sys

    import rq_vae_recommender_b200.dropin as dropin
    from rq_vae_recommender_b200.modules import model as M
    saved = {name: sys.modules.get(name) for name in ("gin", "modules.model", "init", "distributions")}
    try:
        names = dropin.install(replace_model=True, forward_decoder="fused")
        assert names == dropin.install(replace_model=True)           # the returned list does not depend on it
        dropin.install(replace_model=True, forward_decoder="fused")
        assert sys.modules["modules.model"].DEFAULT_FORWARD_DECODER == "fused"
        assert (M.DEFAULT_SEARCH, M.DEFAULT_DECODER, M.DEFAULT_ENCODER, M.DEFAULT_FORWARD_ENCODER) == ("sample", "hf", "hf", "hf")
        dropin.install(replace_model=True)
        assert M.DEFAULT_FORWARD_DECODER == "hf"
        dropin.install(replace_model=True, forward_decoder="fused")
        with pytest.raises(ValueError, match="replace_model"):
            dropin.install(forward_decoder="fused")
        with pytest.raises(ValueError, match="forward_decoder must be"):
            dropin.install(replace_model=True, forward_decoder="eager")
    finally:
        dropin.uninstall()
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod
    assert M.DEFAULT_FORWARD_DECODER == "hf"
