"""CPU tests of the exact ranking (rank_sem_ids / rank_items): in float64, one decoder row per corpus-trie node per history gives
every tuple the log-probability HF's T5Stack gives it teacher-forced alone; the selection rule of t5rank_select against a plain
sort; the new C entry points' argument checks."""
import numpy as np
import pytest
import torch

import t5_rank_ref as RR


def tiny_model(M, corpus, K, H, sep, users, seed):
    torch.manual_seed(seed)
    return M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), num_hierarchies=H, num_embeddings_per_hierarchy=K,
                                          t5_d_model=32, t5_num_heads=2, t5_d_ff=48, t5_num_layers=2, top_k_for_generation=4,
                                          should_add_sep_token=sep, num_user_bins=users).eval()


def corpus_with_edges(rs, N, H, K):
    """Random rows over few codes (shared prefixes), duplicated tuples, and rows holding an id outside [0, K) (prefix nodes that
    are never leaves)."""
    corpus = rs.randint(0, min(K, 3), size=(N, H)).astype(np.int64)
    corpus[1] = corpus[0]
    corpus[2] = corpus[0]
    corpus[3, H - 1] = K
    corpus[4, 1] = -1
    return corpus


@pytest.mark.parametrize("H", [3, 5])
@pytest.mark.parametrize("sep", [True, False])
@pytest.mark.parametrize("users", [None, 7])
def test_trie_decomposition_equals_teacher_forcing_float64(H, sep, users):
    from rq_vae_recommender_b200.modules import model as M
    K, B, items = 5, 4, 3
    rs = np.random.RandomState(H * 10 + sep * 2 + (users or 0))
    corpus = corpus_with_edges(rs, 24, H, K)
    m = tiny_model(M, corpus, K, H, sep, users, seed=H)
    ids = torch.from_numpy(rs.randint(0, K, size=(B, items * H)))
    mask = torch.ones_like(ids)
    mask[1, :H] = 0                                                         # a padded history
    mask[2, H:2 * H] = 0                                                    # a masked hole
    mask[3] = 0                                                             # every position masked
    user_ids = torch.from_numpy(rs.randint(0, 50, size=(B, 1)))
    levels, parents = RR.trie_levels(corpus, H, K)
    assert len(levels[H]) < len(corpus)                                     # duplicates and cut rows are not leaves
    with torch.no_grad():
        # the encoder in fp32 (HF's float64 mask of a fully masked history overflows to NaN), the decoders in float64
        enc_out, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=user_ids)
        enc_out = enc_out.double()
        m.double()
        got = RR.rank_decompose(m, enc_out, enc_mask, levels, parents)
        want = RR.rank_teacher_forced(m, enc_out, enc_mask, levels[H])
    assert got.dtype == torch.float64 and got.shape == (B, len(levels[H]))
    # HF's float64 cross-attention mask (finfo(float64).min) overflows for the fully masked history; it is checked in fp32 below
    assert (got[:3] - want[:3]).abs().max().item() < 1e-10
    assert torch.isfinite(got).all()
    m.float()
    with torch.no_grad():
        got = RR.rank_decompose(m, enc_out[3:].float(), enc_mask[3:], levels, parents)
        want = RR.rank_teacher_forced(m, enc_out[3:].float(), enc_mask[3:], levels[H])
    assert (got - want).abs().max().item() < 1e-5


def test_trie_levels_leaves_are_the_item_tuples():
    """Level H holds the distinct tuples of the rows whose ids are all in [0, K), in lexicographic order: the item table's."""
    rs = np.random.RandomState(3)
    H, K = 3, 4
    corpus = corpus_with_edges(rs, 40, H, K)
    levels, _ = RR.trie_levels(corpus, H, K)
    ok = ((corpus >= 0) & (corpus < K)).all(1)
    assert np.array_equal(levels[H], np.unique(corpus[ok], axis=0))
    packed = (levels[H] * K ** np.arange(H - 1, -1, -1)).sum(1)
    assert np.all(np.diff(packed) > 0)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("n", [1, 10, 200])
def test_select_model_matches_plain_sort(seed, n):
    rs = np.random.RandomState(seed)
    U = int(rs.randint(1, 80))
    scores = np.round(rs.randn(U), 1).astype(np.float32)                   # many equal scores
    scores[rs.rand(U) < 0.1] = np.nan
    scores[rs.rand(U) < 0.1] = -np.inf
    scores[rs.rand(U) < 0.05] = -0.0
    counts = rs.randint(1, 4, size=U)
    full = RR.sort_items(scores, counts)
    for t_leaf in range(U):
        for t_dedup in range(-1, int(counts[t_leaf]) + 1):
            got, rank = RR.select_model(scores, counts, n, t_leaf, t_dedup)
            assert got == full[:n]
            want = full.index((t_leaf, t_dedup)) if 0 <= t_dedup < counts[t_leaf] else -1
            assert rank == want
    assert RR.select_model(scores, counts, n, -1, 0)[1] == -1
    assert RR.select_model(scores[:0], counts[:0], n, -1, 0) == ([], -1)


def test_rank_entry_points_report_argument_errors():
    from rq_vae_recommender_b200 import _lib
    lib = _lib.load()
    assert lib.rqb200_t5rank_cross_attention(0, 64, 0, 0, 64, 0, 0, -1, 1, 1, 0, 64, 0) == 1
    assert b"t5rank_cross_attention: bad argument" in lib.rqb200_last_error()
    assert lib.rqb200_t5rank_cross_attention(0, 64, 0, 0, 64, 0, 0, 70000, 1, 1, 0, 64, 0) == 3
    assert lib.rqb200_t5rank_cross_attention(0, 64, 0, 0, 64, 0, 0, 1, 1, 1, 0, 64, 0) == 1
    assert b"null pointer" in lib.rqb200_last_error()
    assert lib.rqb200_t5rank_children(0, 8, 6, 8, 4, 0, 0, 0, 3, 0, 0, 0) == 1              # R not a multiple of n_h
    assert b"t5rank_children: bad argument" in lib.rqb200_last_error()
    assert lib.rqb200_t5rank_children(0, 8, 8, 8, 4, 0, 0, 0, 3, 0, 0, 0) == 1
    assert b"null pointer" in lib.rqb200_last_error()
    assert lib.rqb200_t5rank_select(0, 1, 10, 0, 0, 0, 0, 1025, 0, 0, 0, 0) == 3
    assert b"n <= 1024" in lib.rqb200_last_error()
    assert lib.rqb200_t5rank_select(0, 1, 10, 0, 0, 0, 0, 0, 0, 0, 0, 0) == 1
    assert lib.rqb200_t5rank_select(0, 0, 10, 0, 0, 0, 0, 5, 0, 0, 0, 0) == 0              # B = 0: no-op
    assert lib.rqb200_sid_trie_level(0, 3, 4, 1, 1, 0, 0, 0, 0) == 1                       # level above C
    assert b"sid_trie_level: bad argument" in lib.rqb200_last_error()
    assert lib.rqb200_sid_trie_counts(0, 0, 0) == 1
    assert lib.rqb200_sid_rank_hist(0, 4, 0, 0, 0) == 1
    assert b"sid_rank_hist: bad argument" in lib.rqb200_last_error()
    import ctypes
    a, b = ctypes.c_size_t(), ctypes.c_size_t()
    assert lib.rqb200_sid_items_offsets(100, 9, 16, ctypes.byref(a), ctypes.byref(b)) == 3
    assert lib.rqb200_sid_items_offsets(100, 3, 16, ctypes.byref(a), ctypes.byref(b)) == 0
    assert a.value % 256 == 0 and b.value > a.value


def test_rank_calls_refuse_cpu_tensors_and_bad_modes():
    from rq_vae_recommender_b200 import _lib, ops
    from rq_vae_recommender_b200.modules import model as M
    with pytest.raises(_lib.Rqb200Error):
        ops.t5rank_cross_attention(torch.zeros(2, 64), torch.zeros(3, 64), torch.zeros(3, 64),
                                   torch.zeros(3, dtype=torch.int32), None, 1, 1)
    m = tiny_model(M, np.zeros((4, 3), dtype=np.int64), 4, 3, True, None, 0).train()
    with pytest.raises(ValueError, match="eval mode"):
        m.rank_sem_ids(torch.ones(1, 3), torch.zeros(1, 3, dtype=torch.int64))
