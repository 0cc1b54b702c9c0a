"""CPU tests of the exact scoring of given tuples (score_sem_ids / score_items): the host statement of the per-history candidate
trie that csrc/t5rank.cu's t5score_trie_build writes, its decomposition against HF's T5Stack teacher-forced on each candidate in
float64, and the argument and mode errors of both entry points."""
import numpy as np
import pytest
import torch

import t5_rank_ref as RR
from test_rank_ref import tiny_model


def candidate_trie(ids: np.ndarray, K: int):
    """One history's candidate trie as t5score_trie_build writes it, from ids [C, H]: (counts [H], code [H, C], parent [H, C],
    child [H, C + 1], leaf [C]).  Only tuples whose ids are all in [0, K) make nodes; padding entries are code 0, parent 0 and
    child n_{l + 1}."""
    C, H = ids.shape
    ok = ((ids >= 0) & (ids < K)).all(1)
    levels, parents = RR.trie_levels(ids[ok], H, K)
    n = [len(lv) for lv in levels]
    counts = np.array(n[1:], dtype=np.int32)
    code = np.zeros((H, C), dtype=np.int32)
    parent = np.zeros((H, C), dtype=np.int32)
    child = np.zeros((H, C + 1), dtype=np.int32)
    for l in range(1, H + 1):
        code[l - 1, :n[l]] = levels[l][:, l - 1]
        parent[l - 1, :n[l]] = parents[l]
    for l in range(H):                                                       # parents ascend: a node's first child by bisection
        child[l] = n[l + 1]
        child[l, :n[l]] = np.searchsorted(parents[l + 1], np.arange(n[l])) if l > 0 else 0
    leaf = np.full(C, -1, dtype=np.int32)
    for c in np.nonzero(ok)[0]:
        leaf[c] = np.nonzero((levels[H] == ids[c]).all(1))[0][0]
    return counts, code, parent, child, leaf


def score_decompose(model, enc_out, enc_mask, ids: np.ndarray):
    """[B, C]: each history's candidates scored by decoding the trie of its own candidates (one row per node), -inf for a tuple
    holding an id outside [0, K)."""
    H, K = model.num_hierarchies, model.num_embeddings_per_hierarchy
    B, C, _ = ids.shape
    out = torch.full((B, C), float("-inf"), dtype=enc_out.dtype)
    for b in range(B):
        _, _, _, _, leaf = candidate_trie(ids[b], K)
        if (leaf < 0).all():
            continue
        ok = leaf >= 0
        levels, parents = RR.trie_levels(ids[b][ok], H, K)
        leaves = RR.rank_decompose(model, enc_out[b:b + 1], enc_mask[b:b + 1], levels, parents)[0]
        out[b, torch.from_numpy(np.nonzero(ok)[0])] = leaves[torch.from_numpy(leaf[ok]).long()]
    return out


def candidates_with_edges(rs, corpus, B, C, H, K):
    """Per history: corpus tuples, tuples the corpus does not hold, duplicates, ids outside [0, K) and -1 padding rows."""
    ids = corpus[rs.randint(0, len(corpus), size=(B, C))].copy()
    ids[:, 1] = rs.randint(0, K, size=(B, H))
    ids[:, 2] = ids[:, 0]
    ids[:, 3, H - 1] = K
    ids[:, 4, 0] = -3
    ids[:, -2:] = -1
    return ids


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("H,K", [(3, 4), (5, 3), (3, 256)])
def test_candidate_trie_statement(seed, H, K):
    """Levels are the sorted distinct prefixes of the valid candidates; every node's children are a contiguous range of the next
    level under it; each valid candidate's leaf holds its tuple."""
    rs = np.random.RandomState(seed)
    C = int(rs.randint(1, 40))
    ids = rs.randint(0, min(K, 3), size=(C, H)).astype(np.int64)
    ids[rs.rand(C) < 0.2, H - 1] = K
    ids[rs.rand(C) < 0.2] = -1
    counts, code, parent, child, leaf = candidate_trie(ids, K)
    ok = ((ids >= 0) & (ids < K)).all(1)
    for l in range(1, H + 1):
        prefixes = np.unique(ids[ok][:, :l], axis=0) if ok.any() else np.zeros((0, l), dtype=np.int64)
        assert counts[l - 1] == len(prefixes)
        assert np.array_equal(code[l - 1, :counts[l - 1]], prefixes[:, l - 1] if len(prefixes) else [])
        assert (code[l - 1, counts[l - 1]:] == 0).all() and (parent[l - 1, counts[l - 1]:] == 0).all()
    n = [1] + counts.tolist()
    for l in range(H):
        assert np.all(np.diff(child[l]) >= 0) and (child[l, n[l]:] == n[l + 1]).all()
        for i in range(n[l]):
            kids = np.arange(child[l, i], child[l, i + 1])
            assert (len(kids) > 0 or n[l + 1] == 0) and (parent[l, kids] == i).all()   # an empty root: no valid tuple
    for c in range(C):
        if not ok[c]:
            assert leaf[c] == -1
            continue
        node = leaf[c]
        for l in range(H, 0, -1):                                            # walk up: the path spells the tuple
            assert code[l - 1, node] == ids[c, l - 1]
            node = parent[l - 1, node]
    equal = [(a, b) for a in range(C) for b in range(C) if ok[a] and ok[b] and (ids[a] == ids[b]).all()]
    assert all(leaf[a] == leaf[b] for a, b in equal)


@pytest.mark.parametrize("H", [3, 5])
@pytest.mark.parametrize("sep", [True, False])
@pytest.mark.parametrize("users", [None, 7])
def test_candidate_decomposition_equals_teacher_forcing_float64(H, sep, users):
    from rq_vae_recommender_b200.modules import model as M
    K, B, items, C = 5, 4, 3, 9
    rs = np.random.RandomState(H * 10 + sep * 2 + (users or 0) + 1)
    corpus = rs.randint(0, min(K, 3), size=(12, H)).astype(np.int64)
    m = tiny_model(M, corpus, K, H, sep, users, seed=H + 1)
    cand = candidates_with_edges(rs, corpus, B, C, H, K)
    ids = torch.from_numpy(rs.randint(0, K, size=(B, items * H)))
    mask = torch.ones_like(ids)
    mask[1, :H] = 0                                                         # a padded history
    mask[2, H:2 * H] = 0                                                    # a masked hole
    mask[3] = 0                                                             # every position masked
    user_ids = torch.from_numpy(rs.randint(0, 50, size=(B, 1)))
    valid = ((cand >= 0) & (cand < K)).all(2)
    with torch.no_grad():
        enc_out, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=user_ids)
        enc_out = enc_out.double()
        m.double()
        got = score_decompose(m, enc_out, enc_mask, cand)
        want = torch.full((B, C), float("-inf"), dtype=torch.float64)
        for b in range(B):
            want[b, valid[b]] = RR.rank_teacher_forced(m, enc_out[b:b + 1], enc_mask[b:b + 1], cand[b][valid[b]])[0]
    assert torch.equal(torch.isinf(got), torch.from_numpy(~valid))
    assert torch.equal(got[:, 0], got[:, 2])                                 # duplicates score the same
    # HF's float64 mask of the fully masked history overflows (as in test_rank_ref); it is checked in fp32 below
    fin = torch.from_numpy(valid[:3])
    assert (got[:3][fin] - want[:3][fin]).abs().max().item() < 1e-10
    m.float()
    with torch.no_grad():
        got = score_decompose(m, enc_out[3:].float(), enc_mask[3:], cand[3:])
        want = RR.rank_teacher_forced(m, enc_out[3:].float(), enc_mask[3:], cand[3][valid[3]])
    assert (got[0, torch.from_numpy(valid[3])] - want[0]).abs().max().item() < 1e-5


def test_score_entry_point_reports_argument_errors():
    from rq_vae_recommender_b200 import _lib
    lib = _lib.load()
    assert lib.rqb200_t5score_trie_build(0, 1, 0, 3, 256, 0, 0, 0, 0, 0, 0) == 1
    assert b"t5score_trie_build: bad argument" in lib.rqb200_last_error()
    assert lib.rqb200_t5score_trie_build(0, 1, 4097, 3, 256, 0, 0, 0, 0, 0, 0) == 3
    assert b"C <= 4096" in lib.rqb200_last_error()
    assert lib.rqb200_t5score_trie_build(0, 1, 5, 9, 4, 0, 0, 0, 0, 0, 0) == 3                 # H > 8
    assert lib.rqb200_t5score_trie_build(0, 1, 5, 8, 256, 0, 0, 0, 0, 0, 0) == 3               # 64 key bits
    assert lib.rqb200_t5score_trie_build(0, 1, 5, 3, 256, 0, 0, 0, 0, 0, 0) == 1
    assert b"null pointer" in lib.rqb200_last_error()
    assert lib.rqb200_t5score_trie_build(0, 0, 5, 3, 256, 0, 0, 0, 0, 0, 0) == 0               # B = 0: no-op


def test_score_calls_refuse_cpu_tensors_and_bad_arguments():
    from rq_vae_recommender_b200 import _lib, ops
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    from rq_vae_recommender_b200.modules import model as M
    H, K = 3, 4
    m = tiny_model(M, np.zeros((4, H), dtype=np.int64), K, H, True, None, 0)
    mask, ids = torch.ones(2, 3), torch.zeros(2, 3, dtype=torch.int64)
    with pytest.raises(_lib.Rqb200Error, match="CUDA tensors only"):
        ops.t5score_trie_build(torch.zeros(2, 3, H, dtype=torch.int64), K)
    with pytest.raises(_lib.Rqb200Error, match="CUDA tensors only"):
        m.score_sem_ids(mask, ids, sem_ids=torch.zeros(2, 5, H, dtype=torch.int64))
    for bad in (torch.zeros(2, 0, H, dtype=torch.int64), torch.zeros(2, 4097, H, dtype=torch.int64)):
        with pytest.raises(ValueError, match=r"candidates per history must be in \[1, 4096\]"):
            m.score_sem_ids(mask, ids, sem_ids=bad)
    for bad in (torch.zeros(3, 5, H, dtype=torch.int64), torch.zeros(2, 5, H + 1, dtype=torch.int64), torch.zeros(2, 5)):
        with pytest.raises(ValueError, match="sem_ids"):
            m.score_sem_ids(mask, ids, sem_ids=bad)
    with pytest.raises(ValueError, match="sem_ids"):
        m.score_sem_ids(mask, ids)
    with pytest.raises(ValueError, match="encoder must be one of"):
        m.score_sem_ids(mask, ids, sem_ids=torch.zeros(2, 5, H, dtype=torch.int64), encoder="x")
    with pytest.raises(ValueError, match="attention must be one of"):
        m.score_sem_ids(mask, ids, sem_ids=torch.zeros(2, 5, H, dtype=torch.int64), attention="bf16")
    wide = tiny_model(M, np.zeros((4, 5), dtype=np.int64), 1 << 13, 5, True, None, 0)        # 5 x 13 key bits
    with pytest.raises(_lib.Rqb200Error, match="64-bit tuple key"):
        wide.score_sem_ids(torch.ones(2, 5), torch.zeros(2, 5, dtype=torch.int64), sem_ids=torch.zeros(2, 5, 5, dtype=torch.int64))
    w = H + 1
    batch = TokenizedSeqBatch(user_ids=None, sem_ids=torch.zeros(2, w, dtype=torch.int64), sem_ids_fut=torch.zeros(2, w),
                              seq_mask=torch.ones(2, w, dtype=torch.bool), token_type_ids=None, token_type_ids_fut=None)
    with pytest.raises(_lib.Rqb200Error, match="CUDA tensors only"):
        m.score_items(batch, torch.zeros(2, 5, dtype=torch.int64))
    m.train()
    with pytest.raises(ValueError, match="eval mode"):
        m.score_sem_ids(mask, ids, sem_ids=torch.zeros(2, 5, H, dtype=torch.int64))
