"""CPU proof that the trainable packed encoder pass of ``forward(encoder="fused")`` is exact: the float64 packed statement of
tests/t5_enc_train_ref.py, with explicit keep masks, gives the same loss and the same gradient for every parameter as
transformers' T5EncoderModel in training mode (run through ``encoder_forward_pass``) when HF's dropout calls apply the same masks
in call order.  Also the argument errors and the ``dropin`` switch of the training encoder."""
import copy

import pytest
import torch

import t5_enc_train_ref as TR
from test_t5_enc_ref import MASKS, inputs, random_model


def loss_and_grads(m, fn):
    m.zero_grad(set_to_none=True)
    loss = fn()
    loss.backward()
    return loss.detach(), {name: (p.grad.clone() if p.grad is not None else torch.zeros_like(p))
                           for name, p in m.named_parameters()}


def weighted_loss(out, enc_mask, W):
    kept = enc_mask != 0
    kept[~kept.any(1)] = True                                # a history with nothing unmasked keeps every position
    return (out * W * kept[..., None].to(out.dtype)).sum()


def compare(m, mask, ids, users, p, seed):
    """HF's fp32 model in training mode against the float64 packed statement on a float64 copy: loss within 1e-5 relative, each
    parameter's gradient within 1e-5 of its largest entry (fp32 rounding of HF's pass)."""
    m = m.float().train()
    with torch.no_grad():
        _, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
    B, S = enc_mask.shape
    masks = TR.random_masks(m, B, S, p, seed)
    W = torch.randn(B, S, m.encoder.config.d_model, generator=torch.Generator().manual_seed(seed + 1), dtype=torch.float64)
    for mod in m.encoder.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = p
        if type(mod).__name__ == "T5Attention":
            mod.dropout = p

    m64 = copy.deepcopy(m).double()

    def hf():
        fake = TR.hf_dropout_from(masks)
        real = torch.nn.functional.dropout
        torch.nn.functional.dropout = fake
        try:
            out, em = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
        finally:
            torch.nn.functional.dropout = real
        assert not fake.queue
        return weighted_loss(out, em, W.float())

    def packed():
        out, em = TR.encode_train(m64, mask, ids, users, masks, p)
        return weighted_loss(out, em, W)

    want_loss, want = loss_and_grads(m, hf)
    got_loss, got = loss_and_grads(m64, packed)
    assert torch.isfinite(want_loss)
    assert abs(got_loss.item() - want_loss.item()) <= 1e-5 * max(1.0, abs(want_loss.item()))
    for name in want:
        scale = max(want[name].abs().max().item(), 1e-30)
        err = (got[name] - want[name].double()).abs().max().item()
        assert err <= 1e-5 * scale, (name, err, scale)
    return want


@pytest.mark.parametrize("kind", MASKS)
@pytest.mark.parametrize("sep", [True, False])
@pytest.mark.parametrize("user_bins", [None, 7])
def test_packed_training_pass_equals_hf(kind, sep, user_bins):
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, sep=sep, user_bins=user_bins, seed=len(kind) + 10 * sep)
    mask, ids, users = inputs(kind, 6, 5, 3, 32, seed=3)
    grads = compare(m, mask, ids, users, p=0.1, seed=len(kind))
    assert grads["encoder.encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"].abs().max() > 0
    assert grads["item_sid_embedding_table.weight"].abs().max() > 0


def test_fully_masked_history_without_user_row_passes_gradient():
    """A history with no unmasked position and no user row: every score rounds to finfo.min, the softmax is uniform and HF's
    autograd still passes dS into q, k and the relative bias; the packed statement does the same."""
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, user_bins=None, seed=5)
    mask, ids, _ = inputs("full", 3, 4, 3, 32, seed=6)
    mask[1] = 0
    compare(m, mask, ids, None, p=0.1, seed=2)
    mask[:] = 0                                              # every history fully masked
    compare(m, mask, ids, None, p=0.0, seed=3)


def test_without_dropout_equals_eval_pass():
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, user_bins=5, seed=7)
    mask, ids, users = inputs("holes", 4, 3, 3, 32, seed=8)
    compare(m, mask, ids, users, p=0.0, seed=4)


def test_forward_encoder_argument_errors():
    from rq_vae_recommender_b200._lib import Rqb200Error
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M)
    assert M.DEFAULT_FORWARD_ENCODER == "hf"
    with pytest.raises(ValueError, match="encoder must be one of"):
        m.forward(None, encoder="eager")
    with pytest.raises(Rqb200Error, match="relu feed-forward"):
        M.FusedT5EncodeTrain(random_model(M, ff="gated-gelu"))
    with pytest.raises(Rqb200Error, match="fp32 parameters"):
        M.FusedT5EncodeTrain(random_model(M).double())
    mask, ids, users = inputs("end", 2, 2, 3, 32, seed=41)
    with pytest.raises(Rqb200Error, match="CUDA tensors only"):
        M.FusedT5EncodeTrain(m)(mask, ids, users)
    with _cuda_autocast_flag(), pytest.raises(ValueError, match="autocast"):
        M.FusedT5EncodeTrain(m)(mask, ids, users)


class _cuda_autocast_flag:
    """torch.is_autocast_enabled("cuda") is True inside, without a device."""

    def __enter__(self):
        self.prev = torch.is_autocast_enabled("cuda")
        torch.set_autocast_enabled("cuda", True)

    def __exit__(self, *exc):
        torch.set_autocast_enabled("cuda", self.prev)


def test_install_forward_encoder_switch():
    import sys

    import rq_vae_recommender_b200.dropin as dropin
    from rq_vae_recommender_b200.modules import model as M
    saved = {name: sys.modules.get(name) for name in ("gin", "modules.model", "init", "distributions")}
    try:
        dropin.install(replace_model=True, forward_encoder="fused")
        assert sys.modules["modules.model"].DEFAULT_FORWARD_ENCODER == "fused"
        assert (M.DEFAULT_SEARCH, M.DEFAULT_DECODER, M.DEFAULT_ENCODER) == ("sample", "hf", "hf")
        dropin.install(replace_model=True)
        assert M.DEFAULT_FORWARD_ENCODER == "hf"
        dropin.install(replace_model=True, forward_encoder="fused")
        with pytest.raises(ValueError, match="replace_model"):
            dropin.install(forward_encoder="fused")
        with pytest.raises(ValueError, match="forward_encoder must be"):
            dropin.install(replace_model=True, forward_encoder="eager")
    finally:
        dropin.uninstall()
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod
    assert M.DEFAULT_FORWARD_ENCODER == "hf"
