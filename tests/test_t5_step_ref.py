"""CPU proof that the fused decode of ``generate(decoder="fused")`` is exact: the plain-torch decomposition of tests/t5_step_ref.py
(cross keys/values once per history, BOS from level 0, the ancestor table, HF's bias table) gives per-level head logits within
1e-5 of transformers' T5Stack run with its cache the way ``generate(decoder="hf")`` runs it, for the same beams."""
import numpy as np
import pytest
import torch

import t5_step_ref as T
from parity import load_golden
from test_generate_oracle import decoder_batch, decoder_model


def random_model(M, H, K=32, user_bins=None, seed=0, k=4):
    torch.manual_seed(seed)
    corpus = torch.randint(0, K, (200, H))
    return M.EncoderDecoderRetrievalModel(codebooks=corpus, num_hierarchies=H, num_embeddings_per_hierarchy=K, t5_d_model=64,
                                          t5_num_heads=3, t5_d_ff=96, t5_num_layers=2, top_k_for_generation=k,
                                          should_add_sep_token=True, num_user_bins=user_bins).eval()


def history(B, items, H, K, seed, pad=True):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, K, (B, items * H), generator=g)
    mask = torch.ones_like(ids)
    if pad:
        for b in range(B):
            mask[b, :H * (b % items)] = 0                                    # 0 .. items - 1 padded items
    return mask, ids, torch.randint(0, 50, (B, 1), generator=g)


def assert_levels_match(m, mask, ids, users, seed):
    k = m.top_k_for_generation
    with torch.no_grad():
        enc_out, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
        beams = T.random_beams(enc_out.shape[0], k, m.num_hierarchies, m.num_embeddings_per_hierarchy, seed)
        want = T.hf_level_logits(m, enc_out, enc_mask, beams, k)
        got = T.fused_level_logits(m, enc_out, enc_mask, beams, k)
    assert len(got) == m.num_hierarchies
    for h, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape
        err = (a - b).abs().max().item()
        assert err <= 1e-5, (h, err)


def test_decoder_golden_model():
    from rq_vae_recommender_b200.modules import model as M
    g = load_golden("decoder")
    m = decoder_model(M, g)
    batch = decoder_batch(g)
    H = m.num_hierarchies
    mask = M._strip_dedup_col(batch.seq_mask.long(), H + 1, H)
    ids = M._strip_dedup_col(batch.sem_ids, H + 1, H)
    assert_levels_match(m, mask, ids, batch.user_ids, 1)


@pytest.mark.parametrize("H", [1, 3, 5, 8])
def test_random_models_at_every_depth(H):
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, H, user_bins=7, seed=H)
    assert_levels_match(m, *history(6, 4, H, 32, seed=H), seed=10 + H)


@pytest.mark.parametrize("user_bins", [None, 5])
def test_padded_histories(user_bins):
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, 3, user_bins=user_bins, seed=21, k=5)
    mask, ids, users = history(8, 6, 3, 32, seed=22)
    assert (mask == 0).any()
    assert_levels_match(m, mask, ids, users, seed=23)


def test_history_with_every_key_masked():
    """Without a user token every encoder key of history 0 is masked: HF adds finfo.min to all its scores and averages the
    values; the decomposition does the same."""
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, 3, user_bins=None, seed=31)
    mask, ids, users = history(4, 3, 3, 32, seed=32, pad=False)
    mask[0] = 0
    assert_levels_match(m, mask, ids, users, seed=33)


def test_ancestor_table_follows_parents():
    """The table after two levels names, for every beam, the level-0 row (its history) and the level-1 row it descends from."""
    beams = T.random_beams(3, 4, 3, 16, seed=5)
    anc = torch.zeros((12, 3), dtype=torch.int32)
    anc = T.advance_ancestors(anc[:3], beams[0][1], 1)
    anc = T.advance_ancestors(anc, beams[1][1], 2)
    parent2 = beams[1][1]
    assert torch.equal(anc[:, 1].long(), parent2)
    assert torch.equal(anc[:, 0].long(), parent2 // 4)
    assert torch.equal(anc[:, 0].long(), torch.arange(3).repeat_interleave(4))
    # the beams' ids agree with their ancestry: level-1 beam anc[r, 1] carries the same first id
    assert np.array_equal(beams[1][0].reshape(12, 2)[:, 0].numpy(), beams[0][0].reshape(12)[parent2].numpy())


def test_decoder_argument_errors():
    """An unknown decoder name and decoder="fused" in training mode raise before any pass runs."""
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, 3)
    mask, ids, users = history(2, 2, 3, 32, seed=41)
    with pytest.raises(ValueError, match="decoder must be one of"):
        m.generate(mask, ids, users, decoder="triton")
    m.train()
    with pytest.raises(ValueError, match="eval mode only"):
        m.generate(mask, ids, users, decoder="fused")
    assert M.DECODERS == ("hf", "fused") and M.DEFAULT_DECODER == "hf"


def test_install_decoder_switch():
    import sys

    import rq_vae_recommender_b200.dropin as dropin
    from rq_vae_recommender_b200.modules import model as M
    saved = {name: sys.modules.get(name) for name in ("gin", "modules.model", "init", "distributions")}
    try:
        assert dropin.install() == sorted(list(dropin._ALIASES) + ["modules.tokenizer.semids"])
        assert M.DEFAULT_DECODER == "hf"
        dropin.install(replace_model=True, decoder="fused")
        assert sys.modules["modules.model"].DEFAULT_DECODER == "fused" and M.DEFAULT_SEARCH == "sample"
        dropin.install(replace_model=True)
        assert M.DEFAULT_DECODER == "hf"
        dropin.install(replace_model=True, search="beam", decoder="fused")
        assert (M.DEFAULT_SEARCH, M.DEFAULT_DECODER) == ("beam", "fused")
        with pytest.raises(ValueError, match="replace_model"):
            dropin.install(decoder="fused")
        with pytest.raises(ValueError, match="decoder must be"):
            dropin.install(replace_model=True, decoder="eager")
    finally:
        dropin.uninstall()
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod
    assert (M.DEFAULT_SEARCH, M.DEFAULT_DECODER) == ("sample", "hf")
