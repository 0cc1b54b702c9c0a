"""CPU tests of the sampled beam search: the multinomial = exponential-race identity the fused kernel relies on, the numpy
oracle ``sample_oracle.sample_select`` against the UNMODIFIED reference's generate (tests/golden/beam.npz), the drop-in model's
forward and generate against the reference model (tests/golden/decoder.npz) and ``dropin.install(replace_model=...)``."""
import sys

import numpy as np
import pytest
import torch

from oracle import rq_oracle as O
import sample_oracle as S
from parity import load_golden


@pytest.mark.parametrize("K", [16, 256, 2048])
@pytest.mark.parametrize("n", [1, 64])
def test_multinomial_is_exponential_race_cpu(K, n):
    """torch.multinomial(p, n) without replacement == topk(p / exponential_(1), n) under the same seed (bit for bit)."""
    n = min(n, K)
    g = torch.Generator().manual_seed(K + n)
    p = torch.softmax(torch.randn(64, K, generator=g) * 4, dim=-1)
    torch.manual_seed(31)
    want = torch.multinomial(p, n, replacement=False)
    torch.manual_seed(31)
    got = torch.topk(p / torch.empty_like(p).exponential_(1), n).indices
    assert torch.equal(want, got)


def beam_levels_from_seed(g):
    """The reference run's per-level probabilities (F.softmax of the recorded logits) and the Exp(1) draws its multinomial
    calls made under torch.manual_seed(902)."""
    B, k, H, K, N = (int(v) for v in g["shape"])
    torch.manual_seed(902)
    for h in range(H):
        probas = torch.softmax(torch.from_numpy(g[f"logits{h}"]), dim=-1)
        yield h, probas.numpy(), torch.empty_like(probas).exponential_(1).numpy()


def test_sample_select_oracle_vs_reference_generate():
    g = load_golden("beam")
    B, k, H, K, N = (int(v) for v in g["shape"])
    nc = min(64, K)
    corpus = g["corpus"]
    generated, log_probas = None, None
    for h, probas, noise in beam_levels_from_seed(g):
        if h > 0:
            assert np.array_equal(generated.reshape(-1, h), g[f"future{h}"])
        prev = generated
        generated, log_probas, parent, samples, samp_log_p = S.sample_select(corpus, probas, noise, generated, log_probas, k, nc)
        assert np.array_equal(samples.reshape(-1), g[f"prefix{h}"][:, -1])                       # the reference's samples
        prefix = samples.reshape(-1, 1) if h == 0 else np.concatenate(
            [np.repeat(prev.reshape(-1, h), nc, axis=0), samples.reshape(-1, 1)], axis=1)
        assert np.array_equal(O.check_valid_prefix(corpus, prefix), g[f"valid{h}"])
        if h > 0:
            assert np.array_equal(parent.reshape(-1), g[f"parent{h}"])
    assert np.array_equal(generated, g["generated"])
    np.testing.assert_allclose(log_probas, g["log_probas"], rtol=2e-5, atol=1e-6)


def test_oracle_sample_order_on_ties():
    """The oracle's sample order: descending, NaN first, equal ratios (zero probabilities) by ascending index, -0 after +0."""
    v = np.array([[0.0, 3.0, 0.0, -0.0, np.nan, 3.0, 1.0, 0.0]], dtype=np.float32)
    order = np.argsort(-S.topk_order_key(v), axis=1, kind="stable")
    assert order[0].tolist() == [4, 1, 5, 6, 0, 2, 7, 3]


def decoder_model(M, g):
    B, items, H, K, N, users = (int(v) for v in g["shape"])
    sd = {name[3:]: torch.from_numpy(g[name]) for name in g.files if name.startswith("sd/")}
    m = M.EncoderDecoderRetrievalModel(codebooks=sd["codebooks"].clone(), num_hierarchies=H, num_embeddings_per_hierarchy=K,
                                       t5_d_model=32, t5_num_heads=2, t5_d_ff=64, t5_num_layers=2, top_k_for_generation=4,
                                       should_add_sep_token=True, num_user_bins=users)
    m.load_state_dict(sd, strict=True)
    return m.eval()


def decoder_batch(g, device="cpu"):
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    B = g["sem_ids"].shape[0]
    return TokenizedSeqBatch(user_ids=t(g["user_ids"]), sem_ids=t(g["sem_ids"]), sem_ids_fut=t(g["sem_ids_fut"]),
                             seq_mask=t(g["seq_mask"]), token_type_ids=t(g["token_type_ids"]),
                             token_type_ids_fut=t(np.arange(g["sem_ids_fut"].shape[1])[None].repeat(B, 0)))


def test_dropin_model_forward_vs_reference():
    from rq_vae_recommender_b200.modules import model as M
    g = load_golden("decoder")
    m = decoder_model(M, g)
    assert sorted(m.state_dict()) == sorted(name[3:] for name in g.files if name.startswith("sd/"))
    with torch.no_grad():
        out = m(decoder_batch(g))
    assert out.logits is None
    np.testing.assert_allclose(out.loss.numpy(), g["loss"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(out.loss_d.numpy(), g["loss_d"], rtol=1e-5, atol=1e-5)


class OracleIndex:
    """CPU stand-in for ops.SidPrefixIndex.sample_select built on sample_oracle.sample_select (the test exercises generate's plumbing:
    the draws it makes, the beams it feeds back, the decoder cache it keeps)."""
    def __init__(self, corpus):
        self.corpus = corpus.numpy()

    def sample_select(self, probas, noise, generated, log_probas, k, nc, reject=None):
        n = lambda t: None if t is None else t.numpy()
        gen, lp, parent, _, _ = S.sample_select(self.corpus, n(probas), n(noise), n(generated), n(log_probas), k, nc)
        return torch.from_numpy(gen), torch.from_numpy(lp.astype(np.float32)), torch.from_numpy(parent.reshape(-1))


def test_dropin_generate_plumbing_vs_reference():
    """generate on the CPU with the oracle in place of the kernel reproduces the reference's generate_next_sem_id under the
    same seed: beams exactly, log-probabilities to fp32 rounding."""
    from rq_vae_recommender_b200.modules import model as M
    g = load_golden("decoder")
    m = decoder_model(M, g)
    index = OracleIndex(m.codebooks)
    m._prefix_index = lambda device: index
    torch.manual_seed(1002)
    out = m.generate_next_sem_id(decoder_batch(g))
    assert np.array_equal(out.sem_ids.numpy(), g["gen_sem_ids"])
    np.testing.assert_allclose(out.log_probas.numpy(), g["gen_log_probas"], rtol=2e-5, atol=1e-6)


def test_model_module_sets_matmul_precision_like_the_reference():
    from rq_vae_recommender_b200.modules import model as M  # noqa: F401
    assert torch.get_float32_matmul_precision() == "high"


def test_install_replace_model():
    import rq_vae_recommender_b200.dropin as dropin
    saved = {name: sys.modules.get(name) for name in ("gin", "modules.model", "init", "distributions")}
    try:
        default = dropin.install()
        assert default == sorted(list(dropin._ALIASES) + ["modules.tokenizer.semids"])
        assert "modules.model" not in default
        assert "modules.model" in dropin.install(replace_model=True)
        from rq_vae_recommender_b200.modules import model as M
        assert sys.modules["modules.model"] is M
        from modules.model import EncoderDecoderRetrievalModel
        assert EncoderDecoderRetrievalModel is M.EncoderDecoderRetrievalModel
    finally:
        dropin.uninstall()
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod
    assert "modules.model" not in sys.modules or sys.modules["modules.model"] is saved["modules.model"]
