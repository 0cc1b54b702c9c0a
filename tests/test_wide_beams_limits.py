"""CPU-only: generate(num_beams=...) checks its limits before any launch (modules/model.py _check_search_limits), and keeps
today's top_k_for_generation limits when num_beams is not given."""
import numpy as np
import pytest
import torch


def _model(K, H=3, k=10):
    from rq_vae_recommender_b200.modules import model as M
    corpus = np.random.RandomState(0).randint(0, K, size=(50, H)).astype(np.int64)
    torch.manual_seed(0)
    return M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), num_hierarchies=H, num_embeddings_per_hierarchy=K,
                                          t5_d_model=64, t5_num_heads=2, t5_d_ff=128, t5_num_layers=2, top_k_for_generation=k,
                                          should_add_sep_token=True, num_user_bins=11).eval()


def _inputs(K, H=3, B=2):
    ids = torch.randint(0, K, (B, 4 * H))
    return torch.ones_like(ids), ids, torch.zeros((B, 1), dtype=torch.int64)


@pytest.mark.parametrize("search,K,w", [("beam", 256, 0), ("beam", 256, 257), ("beam", 2048, 1025), ("sample", 256, 0),
                                        ("sample", 256, 1025), ("sample", 16, 2000)])
def test_num_beams_outside_limits_raises_before_launch(search, K, w):
    from rq_vae_recommender_b200._lib import Rqb200Error
    m = _model(K)
    with pytest.raises(Rqb200Error, match=f"num_beams = {w}"):
        m.generate(*_inputs(K), search=search, num_beams=w)


def test_num_beams_limits_at_the_edges():
    """The widest accepted widths pass the check; more than 2048 codes per level is refused at any width."""
    from rq_vae_recommender_b200._lib import Rqb200Error
    m = _model(256)
    m._check_search_limits("beam", 256, 64, 256)
    m._check_search_limits("sample", 1024, 64, 1024)
    m = _model(4096)
    with pytest.raises(Rqb200Error, match="num_beams = 10"):
        m._check_search_limits("beam", 10, 64, 10)


@pytest.mark.parametrize("search,k", [("beam", 33), ("sample", 20)])
def test_default_width_keeps_todays_limits(search, k):
    from rq_vae_recommender_b200._lib import Rqb200Error
    m = _model(256, k=k)
    with pytest.raises(Rqb200Error, match=f"top_k_for_generation = {k}"):
        m.generate(*_inputs(256), search=search)


def test_narrow_kernels_serve_todays_widths():
    from rq_vae_recommender_b200.modules import model as M
    narrow = M.EncoderDecoderRetrievalModel._narrow_search
    assert narrow("beam", 32, 64) and not narrow("beam", 33, 64)
    assert narrow("sample", 16, 64) and not narrow("sample", 17, 64) and narrow("sample", 32, 16)
    assert not narrow("sample", 33, 16)
