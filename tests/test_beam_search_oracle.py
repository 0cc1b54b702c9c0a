"""CPU tests of the exhaustive beam search (``generate(search="beam")``): the numpy oracle ``beam_search_oracle.beam_topk`` finds
the true top-k of a two-level search, the drop-in model's generate plumbing against a plain-torch beam search on the
tests/golden/decoder.npz model, the per-search limits and ``dropin.install(search=...)``."""
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import beam_search_oracle as BO
from parity import load_golden
from test_generate_oracle import decoder_batch, decoder_model


def test_oracle_two_level_search_is_exhaustive():
    """H = 2, K = k = 16 and fixed logits per prefix: keeping all 16 first codes and scoring every extension, the oracle
    search returns exactly the 16 best valid complete sequences, as enumerating every sequence finds them."""
    K, k, B = 16, 16, 3
    rs = np.random.RandomState(0)
    corpus = np.unique(rs.randint(0, K, size=(70, 2)), axis=0).astype(np.int64)
    logits0 = rs.randn(B, K).astype(np.float32) * 2                  # the "model": level-0 logits per history ...
    logits1 = rs.randn(B, K, K).astype(np.float32) * 2               # ... and level-1 logits per history and first code
    gen0, lp0, _ = BO.beam_topk(corpus, logits0, None, None, k)
    assert np.array_equal(np.sort(gen0[:, :, 0], axis=1), np.tile(np.arange(K), (B, 1)))
    gen, lp, parent = BO.beam_topk(corpus, logits1[np.arange(B)[:, None], gen0[:, :, 0]].reshape(B * k, K), gen0, lp0, k)
    ls0, ls1 = BO.log_softmax64(logits0), BO.log_softmax64(logits1.reshape(B * K, K)).reshape(B, K, K)
    valid = np.zeros((K, K), dtype=bool)
    valid[corpus[:, 0], corpus[:, 1]] = True
    assert valid.sum() >= k
    for b in range(B):
        total = np.where(valid, ls0[b][:, None] + ls1[b], -np.inf).reshape(-1)
        best = np.argsort(-total, kind="stable")[:k]
        assert np.array_equal(gen[b], np.stack([best // K, best % K], axis=1))
        np.testing.assert_allclose(lp[b], total[best], rtol=1e-12, atol=1e-12)
        assert np.array_equal(gen0[b, parent[b] - b * k, 0], gen[b, :, 0])


class OracleBeamIndex:
    """CPU stand-in for ops.SidPrefixIndex.beam_topk built on beam_search_oracle.beam_topk (the test exercises generate's
    plumbing: the beams it feeds back and the decoder cache it keeps)."""
    def __init__(self, corpus):
        self.corpus = corpus.numpy()

    def beam_topk(self, logits, generated, log_probas, k, bad=None):
        n = lambda t: None if t is None else t.numpy()
        gen, lp, parent = BO.beam_topk(self.corpus, n(logits), n(generated), n(log_probas), k)
        return torch.from_numpy(gen), torch.from_numpy(lp.astype(np.float32)), torch.from_numpy(parent.reshape(-1))


def torch_beam_search(m, attention_mask, input_ids, user_id):
    """The exhaustive constrained beam search in plain torch: generate's T5 calls and cache handling, log_softmax over every
    code, the reference's prefix compare, masked_fill, a stable descending sort and gathers."""
    from transformers.cache_utils import DynamicCache, EncoderDecoderCache
    k, K, H = m.top_k_for_generation, m.num_embeddings_per_hierarchy, m.num_hierarchies
    B = input_ids.shape[0]
    enc_out, enc_mask = m.encoder_forward_pass(attention_mask=attention_mask, input_ids=input_ids, user_id=user_id)
    rep_enc, rep_mask = enc_out.repeat_interleave(k, dim=0), enc_mask.repeat_interleave(k, dim=0)
    generated, log_probas = None, None
    past_kv = EncoderDecoderCache(DynamicCache(), DynamicCache())
    for h in range(H):
        first = generated is None
        dec_out, past_kv = m.decoder_forward_pass(
            future_ids=None if first else generated.reshape(-1, h), encoder_output=enc_out if first else rep_enc,
            attention_mask_for_encoder=enc_mask if first else rep_mask, use_cache=True, past_key_values=past_kv)
        logp = F.log_softmax(m.decoder_mlp[h](dec_out[:, -1, :]), dim=-1)
        kp = 1 if first else k
        codes = torch.arange(K).repeat(B * kp).unsqueeze(1)
        prefix = codes if first else torch.cat([generated.reshape(-1, h).repeat_interleave(K, dim=0), codes], dim=1)
        valid = (m.codebooks[:, : h + 1].unsqueeze(1) == prefix.unsqueeze(0)).all(dim=2).any(dim=0)
        scores = logp.reshape(B, kp * K) + (0 if first else log_probas.repeat_interleave(K, dim=1))
        scores, idx = scores.masked_fill(~valid.reshape(B, kp * K), float("-inf")).sort(dim=-1, descending=True, stable=True)
        top = idx[:, :k]
        parent = top // K
        new_ids = (top % K).unsqueeze(-1)
        generated = new_ids if first else torch.cat([torch.gather(generated, 1, parent.unsqueeze(-1).expand(-1, -1, h)), new_ids],
                                                    dim=-1)
        log_probas = scores[:, :k]
        if first:
            past_kv = EncoderDecoderCache(DynamicCache(), DynamicCache())
        else:
            past_kv.reorder_cache((parent + torch.arange(B).unsqueeze(1) * kp).flatten())
    return generated, log_probas


def test_dropin_generate_beam_plumbing_vs_torch_search():
    """generate(search="beam") on the CPU with the oracle in place of the kernel equals the plain-torch search: beams exactly,
    log-probabilities to fp32 rounding; it draws nothing from the generator."""
    from rq_vae_recommender_b200.modules import model as M
    g = load_golden("decoder")
    m = decoder_model(M, g)
    index = OracleBeamIndex(m.codebooks)
    m._prefix_index = lambda device: index
    batch = decoder_batch(g)
    rng = torch.get_rng_state()
    out = m.generate_next_sem_id(batch, search="beam")
    assert torch.equal(torch.get_rng_state(), rng)
    H = m.num_hierarchies
    with torch.no_grad():
        want_g, want_p = torch_beam_search(m, M._strip_dedup_col(batch.seq_mask.long(), H + 1, H),
                                           M._strip_dedup_col(batch.sem_ids, H + 1, H), batch.user_ids)
    assert out.sem_ids.shape == (g["sem_ids"].shape[0], 4, H)
    assert torch.isfinite(out.log_probas).any()
    assert torch.equal(out.sem_ids, want_g)
    np.testing.assert_allclose(out.log_probas.numpy(), want_p.numpy(), rtol=1e-5, atol=1e-6)
    # DEFAULT_SEARCH is read at call time
    saved = M.DEFAULT_SEARCH
    try:
        M.DEFAULT_SEARCH = "beam"
        again = m.generate_next_sem_id(batch)
    finally:
        M.DEFAULT_SEARCH = saved
    assert torch.equal(again.sem_ids, out.sem_ids) and torch.equal(again.log_probas, out.log_probas)


def small_cpu_model(M, K, k, H=3):
    corpus = torch.from_numpy(np.random.RandomState(0).randint(0, K, size=(50, H)))
    return M.EncoderDecoderRetrievalModel(codebooks=corpus, num_hierarchies=H, num_embeddings_per_hierarchy=K, t5_d_model=16,
                                          t5_num_heads=2, t5_d_ff=32, t5_num_layers=1, top_k_for_generation=k).eval()


def test_generate_search_limits():
    from rq_vae_recommender_b200._lib import Rqb200Error
    from rq_vae_recommender_b200.modules import model as M
    ids = torch.zeros((2, 6), dtype=torch.int64)
    mask = torch.ones_like(ids)
    with pytest.raises(Rqb200Error, match="beam search kernel"):
        small_cpu_model(M, 256, 33).generate(mask, ids, search="beam")
    with pytest.raises(Rqb200Error, match="beam search kernel"):
        small_cpu_model(M, 16, 20).generate(mask, ids, search="beam")
    with pytest.raises(Rqb200Error, match="beam search kernel"):
        small_cpu_model(M, 4096, 10, H=2).generate(mask, ids, search="beam")
    with pytest.raises(Rqb200Error, match="sampling kernel"):
        small_cpu_model(M, 256, 20).generate(mask, ids, search="sample")
    with pytest.raises(ValueError, match="search must be"):
        small_cpu_model(M, 256, 10).generate(mask, ids, search="greedy")


def test_install_search_switch():
    import rq_vae_recommender_b200.dropin as dropin
    from rq_vae_recommender_b200.modules import model as M
    saved = {name: sys.modules.get(name) for name in ("gin", "modules.model", "init", "distributions")}
    try:
        default = dropin.install()
        assert default == sorted(list(dropin._ALIASES) + ["modules.tokenizer.semids"])
        assert M.DEFAULT_SEARCH == "sample"
        assert "modules.model" in dropin.install(replace_model=True)
        assert M.DEFAULT_SEARCH == "sample"
        assert dropin.install(replace_model=True, search="beam") == sorted(
            list(dropin._ALIASES) + ["modules.tokenizer.semids", "modules.model"])
        assert sys.modules["modules.model"].DEFAULT_SEARCH == "beam"
        dropin.install(replace_model=True)
        assert M.DEFAULT_SEARCH == "sample"
        dropin.install(replace_model=True, search="beam")
        with pytest.raises(ValueError, match="replace_model"):
            dropin.install(search="beam")
        with pytest.raises(ValueError, match="search must be"):
            dropin.install(replace_model=True, search="greedy")
    finally:
        dropin.uninstall()
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod
    assert M.DEFAULT_SEARCH == "sample"
