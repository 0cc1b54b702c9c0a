"""GPU tests of the semantic-id stack (csrc/sid.cu, csrc/sid_excl.cuh, csrc/t5rank.cu) along the axes its other tests leave power
of two or sparse: codebook sizes K that are not powers of two (a partial last child-mask word, trie widths next to a power of
two, trie keys over two 64-bit words), every width of the per-history block sorts of the filter builds and the candidate trie
on dense rows (the profiler confirms every instantiation ran), consumers of exclusions of 4096 items and of allow-lists of 4096
items under one prefix, and the widest accepted keys (H * bits(K - 1) = 60).  Every output is compared with the exact numpy
statements of tests/ (trie_oracle, beam_search_oracle, sample_oracle, item_oracle, exclusion_oracle, inclusion_oracle,
test_score_ref.candidate_trie) or the float64 statements of the exact ranking and scoring.  `pytest -m gpu`."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import exclusion_oracle as X
import inclusion_oracle as I
import item_oracle as IO
import sample_oracle as SO
import t5_rank_ref as RR
import trie_oracle as T
from test_gpu_beam_search import assert_matches, oracle_level
from test_gpu_decode import highest
from test_gpu_exclusion import corpus_with_subtrees
from test_gpu_generate import dev, history, level_logits
from test_gpu_rank import batch_for, expected_items, model_for
from test_gpu_score import candidates
from test_gpu_trie import same
from test_score_ref import candidate_trie, score_decompose
from test_trie_oracle import prefixes, random_corpus

pytestmark = pytest.mark.gpu


def key_bits(K):
    """bits(K - 1), at least 1: the width of one id in the filters' and the candidate trie's keys"""
    return max(1, (K - 1).bit_length())


def tail(K):
    """the codes of the last child-mask word, 32 floor(K / 32) .. K - 1 (all of the last word's codes when K % 32 == 0)"""
    return np.arange(32 * ((K - 1) // 32), K)


def tail_corpus(rs, N, H, K):
    """corpus_with_subtrees, with a fifth of its rows made of codes of the last mask word only"""
    corpus = corpus_with_subtrees(rs, N, H, K)
    t = tail(K)
    corpus[N - N // 5:] = t[rs.randint(0, len(t), size=(N // 5, H))]
    return corpus


# (K, H): one bit past a mask word; a partial last word (trie width 9, 7 ids per 64-bit word) and eight levels over two words;
# trie width 10 and seven levels over two words; the largest searchable K below 2048 (trie width 11, 2048's is 12)
SHAPES = [(33, 3), (33, 5), (300, 3), (300, 8), (1000, 3), (1000, 7), (2047, 3)]
# the filters and the candidate trie take H * bits(K - 1) <= 62: these, a K only the item table and filters accept, and 60 bits
FILTER_SHAPES = [(K, H) for K, H in SHAPES if H * key_bits(K) <= 62] + [(40000, 3), (1024, 6)]


@pytest.mark.parametrize("K,H", SHAPES + [(1024, 6)])
def test_check_matches_valid_prefixes(K, H):
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K + H)
    corpus = random_corpus(rs, 3000, H, K)
    t = tail(K)
    corpus[:300] = t[rs.randint(0, len(t), size=(300, H))]
    idx = ops.SidPrefixIndex(dev(corpus), K)
    for l in range(1, H + 1):
        p = prefixes(rs, corpus, l, K, n=600)
        near = corpus[rs.randint(0, 600, size=300), :l].copy()            # tail-code prefixes, one id changed within the tail
        near[np.arange(300), rs.randint(0, l, size=300)] = t[rs.randint(0, len(t), size=300)]
        p = np.concatenate([p, near, np.full((1, l), K - 1), np.full((1, l), K)])
        want = T.valid_prefixes(corpus, p, K)
        assert want.any() and not want.all()
        assert np.array_equal(idx.check(dev(p)).cpu().numpy(), want), l
        assert np.array_equal(T.lookup(T.build(corpus, K), p), want), l


@pytest.mark.parametrize("K,H", SHAPES)
def test_searches_agree_with_oracles_and_each_other(K, H):
    """As test_gpu_trie.py's test of the same name, over min(H, 5) levels, with logits that favour the codes of the last mask
    word: beam_topk matches beam_search_oracle, sample_select's samples are sample_oracle's and its beams beam_select's over
    them, and check of every sampled extension is trie_oracle's."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K * 10 + H)
    B, k = 7, 10
    corpus = tail_corpus(rs, 3000, H, K)
    idx = ops.SidPrefixIndex(dev(corpus), K)
    nc = min(64, K)
    n = lambda t: None if t is None else t.cpu().numpy()
    gen_b = gen_s = lp_b = lp_s = None
    n_tail = 0
    for h in range(min(H, 5)):
        kp = 1 if h == 0 else k
        lg = level_logits(rs, corpus, None if h == 0 else n(gen_b).reshape(-1, h), B * kp, K)
        lg[:, tail(K)] += 4
        logits = dev(np.clip(lg, -60, 60))
        logits[1, 5] = float("nan")
        logits[2] = -float("inf")
        bad = torch.zeros(1, dtype=torch.int32, device="cuda")
        out = idx.beam_topk(logits, gen_b, lp_b, k, bad=bad)
        x = n(logits)
        assert int(bad) == int((np.isnan(x).any(1) | np.isposinf(x).any(1) | np.isneginf(x).all(1)).sum())
        ref = oracle_level(corpus, logits, gen_b, lp_b, k)
        assert_matches(*ref, out, k)
        finite = np.isfinite(n(out[1]))
        assert np.array_equal(finite.sum(1), np.minimum(k, np.isfinite(ref[3]).sum(1)))
        assert T.valid_prefixes(corpus, n(out[0])[finite], K).all()
        n_tail += int(np.isin(n(out[0])[finite][:, -1], tail(K)).sum())

        probas = F.softmax(logits.nan_to_num(0.0), dim=-1)
        probas[3] = 0.0
        probas[1, 2] = float("nan")
        noise = torch.empty_like(probas).exponential_(1)
        samp = idx.sample_select(probas, noise, gen_s, lp_s, k, nc, want_samples=True)
        p = n(probas)
        assert np.array_equal(n(samp[3]), SO.sample_select(corpus, p, n(noise), n(gen_s), n(lp_s), k, nc)[3])
        assert same(samp[:3], idx.beam_select(samp[3], samp[4], gen_s, lp_s, k))
        ext = samp[3].reshape(-1, 1) if h == 0 else torch.cat([gen_s.reshape(-1, h).repeat_interleave(nc, 0),
                                                                samp[3].reshape(-1, 1)], 1)
        assert np.array_equal(n(idx.check(ext)), T.valid_prefixes(corpus, n(ext), K))
        gen_b, lp_b = out[0], out[1]
        gen_s, lp_s = samp[0], samp[1]
    assert n_tail > 0                                                    # beams ended in the last mask word


def leaf_of(ref, item):
    """(leaf, dedup rank) of a retrievable item in the item table"""
    inv = np.empty(len(ref["row"]), dtype=np.int64)
    inv[ref["row"]] = np.arange(len(ref["row"]))
    u = int(np.searchsorted(ref["start"], inv[item], side="right") - 1)
    return u, int(inv[item] - ref["start"][u])


@pytest.mark.parametrize("K,H", SHAPES + [(40000, 3), (1024, 6)])
def test_item_table_matches_oracle(K, H):
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K + 3 * H)
    N, B, k = 3000, 5, 40
    corpus = tail_corpus(rs, N, H, K)
    corpus[5, H - 1] = K                                                 # unretrievable rows
    corpus[6, 0] = -1
    table = ops.SidItemTable(dev(corpus), K)
    ref = IO.build(corpus, K)
    row, start = table.arrays()
    U = len(ref["keys"])
    assert np.array_equal(row.cpu().numpy(), ref["row"]) and np.array_equal(start[:U + 1].cpu().numpy(), ref["start"])
    ids = np.concatenate([corpus[rs.randint(0, N, size=500)], rs.randint(0, K, size=(100, H)), corpus[5:7]])
    ids[-3, 0] = K
    dedup = rs.randint(-1, 14, size=(len(ids), 1))
    assert np.array_equal(table.lookup(dev(ids)).cpu().numpy(), IO.lookup(ref, ids))
    with_d = np.concatenate([ids, dedup], 1)
    assert np.array_equal(table.lookup(dev(with_d), with_dedup=True).cpu().numpy(), IO.lookup(ref, with_d, with_dedup=True))
    gen = corpus[rs.randint(0, N, size=(B, k))]
    gen[:, 1] = corpus[N // 4]                                            # 13 items
    gen[:, 2] = gen[:, 0]
    gen[:, 3] = K - 1
    lp = -np.sort(rs.rand(B, k), axis=1).astype(np.float32)
    lp[:, -2:] = -np.inf
    for n in (1, 20, 600):
        got = table.retrieve(dev(gen), dev(lp), n)
        for a, w in zip(got, IO.retrieve(ref, gen, lp, n)):
            assert np.array_equal(a.cpu().numpy(), w)


def assert_exclusion(ex, want, H):
    pos, blocked, count = ex.pos.cpu().numpy(), ex.blocked.cpu().numpy(), ex.count.cpu().numpy()
    for b, w in enumerate(want):
        assert count[b, 0] == len(w["pos"]) and pos[b, :count[b, 0]].tolist() == w["pos"], b
        assert (pos[b, count[b, 0]:] == -1).all(), b
        for l in range(1, H + 1):
            assert count[b, l] == len(w["blocked"][l]) and blocked[b, l - 1, :count[b, l]].tolist() == w["blocked"][l], (b, l)
            assert (blocked[b, l - 1, count[b, l]:] == -1).all(), (b, l)
        assert count[b, H + 1] == w["bad"], b


def assert_inclusion(inc, want, H):
    pos, keys, count = inc.pos.cpu().numpy(), inc.keys.cpu().numpy(), inc.count.cpu().numpy()
    for b, w in enumerate(want):
        assert count[b, 0] == len(w["pos"]) and pos[b, :count[b, 0]].tolist() == w["pos"], b
        assert (pos[b, count[b, 0]:] == -1).all(), b
        for l in range(1, H + 1):
            assert count[b, l] == len(w["keys"][l]) and keys[b, l - 1, :count[b, l]].tolist() == w["keys"][l], (b, l)
            assert (keys[b, l - 1, count[b, l]:] == -1).all(), (b, l)
        assert count[b, H + 1] == w["bad"], b


def filters(corpus, K, items, ex_items):
    """The device exclusion of ex_items and inclusion of items (ex_items folded in), and the oracles'."""
    from rq_vae_recommender_b200 import ops
    table = ops.SidItemTable(dev(corpus), K)
    ref = IO.build(corpus, K)
    keys = dev(X.leaf_keys(ref))
    ex = ops.sid_exclusion_build(dev(ex_items), table, keys)
    inc = ops.sid_inclusion_build(dev(items), table, keys, exclude=ex)
    excls = X.build(ref, ex_items)
    return table, ref, ex, inc, excls, I.build(ref, items, excls)


def search_level(index, search, logits, noise, gen, lp, k, **filt):
    if search == "beam":
        return index.beam_topk(logits, gen, lp, k, **filt)
    return index.sample_select(torch.softmax(logits, -1), noise, gen, lp, k, min(64, logits.shape[1]), **filt)


def assert_search_equals_reduced(H, index, reduced, logits_of, search, k, **filt):
    """Per history, each level of the search with the filter is the same level on history b's reduced corpus, bit for bit
    (reduced[b] None: no eligible row, every beam -inf)."""
    B = len(reduced)
    gen, lp = None, None
    for h in range(H):
        kp = 1 if gen is None else k
        logits = logits_of(h, B * kp)
        noise = torch.empty_like(logits).exponential_(1)
        out = search_level(index, search, logits, noise, gen, lp, k, **filt)
        for b in range(B):
            if reduced[b] is None:
                assert torch.isneginf(out[1][b]).all()
                continue
            rows = slice(b * kp, (b + 1) * kp)
            g = None if gen is None else gen[b:b + 1]
            p = None if lp is None else lp[b:b + 1]
            want = search_level(reduced[b], search, logits[rows], noise[rows], g, p, k)
            assert torch.equal(out[0][b], want[0][0]), (h, b)
            assert torch.equal(out[1][b], want[1][0]), (h, b)
            assert torch.equal(out[2].view(B, k)[b] - b * kp, want[2]), (h, b)
        gen, lp = out[0], out[1]
    return lp


def tail_logits(K):
    def logits_of(h, rows):
        logits = torch.randn(rows, K, device="cuda") * 3
        logits[:, dev(tail(K))] += 2
        return logits
    return logits_of


@pytest.mark.parametrize("K,H", FILTER_SHAPES)
def test_filters_match_oracles_and_reduced_corpus_search(K, H):
    """Both filter builds against their oracles; then, where the searches take K, both searches with each filter equal the
    unfiltered search on the history's reduced (exclusion) or eligible (inclusion) corpus."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K + H + 1)
    N, B = 1500, 4
    corpus = tail_corpus(rs, N, H, K)
    bad_row = N // 2 + 100                                               # an unretrievable row outside the excluded subtrees
    corpus[bad_row, :2] = [K - 1, K]
    items = np.full((B, 300), -1, dtype=np.int64)
    ex_items = np.full((B, 200), -1, dtype=np.int64)
    for b in range(B):
        sub = np.flatnonzero(corpus[:, 0] == corpus[b, 0])              # a whole level-1 subtree
        items[b, :300] = np.concatenate([sub, rs.randint(0, N, size=300)])[:300]
        cut = len(sub) if b == 0 else 120                                # history 0 excludes all of it, the others part
        ex_items[b, :len(sub[:cut])] = sub[:cut]
        ex_items[b, -10:] = rs.randint(N - N // 5, N, size=10)           # tail rows
    ex_items[1, -12:-10] = [N, -3]                                       # ids outside [-1, N)
    items[2, -3:] = [bad_row, N + 1, bad_row]
    items[3] = -1
    _, ref, ex, inc, excls, incls = filters(corpus, K, items, ex_items)
    assert_exclusion(ex, excls, H)
    assert_inclusion(inc, incls, H)
    assert sum(len(w["blocked"][1]) for w in excls) > 0 and sum(len(w["blocked"][H]) for w in excls) > 0
    if K > 2048:
        return
    index = ops.SidPrefixIndex(dev(corpus), K)
    without = [ops.SidPrefixIndex(dev(np.delete(corpus, sorted(w["excluded"]), 0)), K) for w in excls]
    eligible = [ops.SidPrefixIndex(dev(corpus[sorted(w["eligible"])]), K) if w["eligible"] else None for w in incls]
    levels = min(H, 4)
    for search in ("beam", "sample"):
        assert_search_equals_reduced(levels, index, without, tail_logits(K), search, 16, exclude=ex)
        assert_search_equals_reduced(levels, index, eligible, tail_logits(K), search, 16, include=inc)


@pytest.mark.parametrize("K,H", FILTER_SHAPES)
def test_candidate_trie_matches_host_statement(K, H):
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(K + H + 2)
    C = 300
    corpus = tail_corpus(rs, 1000, H, K)
    ids = corpus[rs.randint(0, len(corpus), size=(3, C))].copy()
    ids[0, ::7, H - 1] = K                                               # invalid tuples
    ids[0, 3::11] = -1                                                   # padding
    ids[1, ::2] = ids[1, 1]                                              # duplicates
    ids[2, :, 0] = K - 1
    trie = [t.cpu().numpy() for t in ops.t5score_trie_build(dev(ids), K)]
    for b in range(ids.shape[0]):
        for name, g, w in zip(("counts", "code", "parent", "child", "leaf"), trie, candidate_trie(ids[b], K)):
            assert np.array_equal(g[b], w), (b, name)


def rank_targets(rs, ref, excls, B):
    """t_leaf / t_dedup [B]: an excluded item of history 0, an item of history 1 that is not excluded, one of a leaf with several
    items (its last dedup rank), a dedup rank past its leaf's items, and out-of-range leaves."""
    U = len(ref["keys"])
    t_leaf, t_dedup = rs.randint(0, U, size=B), np.zeros(B, dtype=np.int64)
    t_leaf[0], t_dedup[0] = leaf_of(ref, sorted(excls[0]["excluded"])[len(excls[0]["excluded"]) // 2])
    kept = [r for r in ref["row"][:ref["start"][-1]] if int(r) not in excls[1]["excluded"]]
    t_leaf[1], t_dedup[1] = leaf_of(ref, int(kept[len(kept) // 3]))
    if B > 2:
        sizes = np.diff(ref["start"])
        t_leaf[2] = int(np.argmax(sizes))
        t_dedup[2] = sizes[t_leaf[2]] - 1
    if B > 3:
        t_dedup[3] = 99
    if B > 4:
        t_leaf[4] = -1
    return t_leaf, t_dedup


@pytest.mark.parametrize("N", [3000, 40000])
def test_rank_select_matches_oracle(N):
    """t5rank_select at K = 300 with and without an exclusion, U <= 24 576 leaf keys in shared memory (N = 3000) and above."""
    from rq_vae_recommender_b200 import ops
    K, H, B = 300, 3, 5
    rs = np.random.RandomState(N)
    corpus = tail_corpus(rs, N, H, K)
    corpus[N // 3: N // 3 + 40] = corpus[N // 3]                        # one tuple of 41 items
    ex_items = np.full((B, 500), -1, dtype=np.int64)
    for b in range(B):
        sub = np.flatnonzero(corpus[:, 0] == corpus[b, 0])
        ex_items[b] = np.concatenate([sub[:300], rs.randint(0, N, size=500)])[:500]
    ex_items[2, :20] = np.arange(N // 3, N // 3 + 20)                    # half of the large tuple
    table, ref, ex, _, excls, _ = filters(corpus, K, ex_items, ex_items)
    U = len(ref["keys"])
    assert (U <= 24 * 1024) == (N == 3000)
    row, start = table.arrays()
    scores = rs.randn(B, U).round(1).astype(np.float32)                 # ties
    scores[1, :30] = np.nan
    scores[3, -5:] = -np.inf
    t_leaf, t_dedup = rank_targets(rs, ref, excls, B)
    none = [dict(excluded=set())] * B
    for n in (1, 700, 1024):
        for exclude, e in ((None, none), (ex, excls)):
            got = ops.t5rank_select(dev(scores), row, start, dev(t_leaf), dev(t_dedup), n, exclude=exclude)
            want = X.rank_select(ref, e, scores, t_leaf, t_dedup, n)
            for a, w in zip(got, want):
                np.testing.assert_array_equal(a.cpu().numpy(), w)
    assert got[2][0] == -1 and got[2][1] >= 0


def test_model_ranks_and_scores_match_float64_at_k300():
    """rank_sem_ids and score_sem_ids of a K = 300 model (t5rank_children over ten 32-code words and a partial one) against the
    float64 statements of test_gpu_rank.py and test_gpu_score.py, and rank_items against a sort of the dense scores."""
    from rq_vae_recommender_b200.modules import model as M
    K, H, B = 300, 3, 6
    rs = np.random.RandomState(300)
    corpus = tail_corpus(rs, 500, H, K)
    corpus[:40, 1] = 299
    corpus[7, 2] = K                                                     # a row that is never a leaf
    m = model_for(M, corpus, K, H)
    mask, ids, users = history(rs, B, 12, H, K)
    mask[-1] = 0
    cand = candidates(rs, corpus, B, 12, H, K)
    with highest():
        ranked = m.rank_sem_ids(mask, ids, users, encoder="fused")
        scored = m.score_sem_ids(mask, ids, users, sem_ids=cand)
        enc_out, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=users)
    ref = M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), num_hierarchies=H, num_embeddings_per_hierarchy=K,
                                         t5_d_model=64, t5_num_heads=2, t5_d_ff=128, t5_num_layers=2, top_k_for_generation=10,
                                         should_add_sep_token=True, num_user_bins=11)
    ref.load_state_dict(m.state_dict())
    ref = ref.double().eval()
    levels, parents = RR.trie_levels(corpus, H, K)
    with torch.no_grad():
        want = RR.rank_decompose(ref, enc_out.double().cpu(), enc_mask.cpu(), levels, parents)
        want_s = score_decompose(ref, enc_out.double().cpu(), enc_mask.cpu(), cand.cpu().numpy())
    assert ranked.shape == (B, len(levels[H]))
    assert (ranked.double().cpu() - want).abs().max().item() <= 1e-5
    fin = torch.isfinite(want_s)
    assert torch.equal(fin, torch.isfinite(scored.cpu()))
    assert (scored.double().cpu()[fin] - want_s[fin]).abs().max().item() <= 1e-5
    batch = batch_for(rs, corpus, B, 6, H, K)
    with highest():
        out = m.rank_items(batch, n=600)
        scores = m.rank_sem_ids(M._strip_dedup_col(batch.seq_mask.long(), H + 1, H),
                                M._strip_dedup_col(batch.sem_ids, H + 1, H), batch.user_ids)
    full, rows = expected_items(scores, corpus, H, K, 600)
    items = out.item_ids.cpu().numpy()
    for b in range(B):
        got = [int(rows[u][d]) for u, d in full[b][:600]]
        assert items[b, :len(got)].tolist() == got and (items[b, len(got):] == -1).all()


# ------------------------------------------------------------------------------------------------ every sort width
WIDTHS = [512, 513, 1024, 1025, 2048, 2049, 4096]
REPEAT = 9                                                               # IPT + 1 copies straddle a thread boundary at any IPT


def dense_rows(rs, corpus, B, M):
    """[B, M] items, 94 % valid in every row but 2 and 3: one item REPEAT times, whole level-1 subtrees and a long 2-prefix run
    (runs of positions across thread boundaries), random rows with repeats, unretrievable rows, and -1 pads and ids outside
    [-1, N) interleaved; row 2 is one item M times, row 3 all -1."""
    N = len(corpus)
    items = np.empty((B, M), dtype=np.int64)
    for b in range(B):
        sub = np.flatnonzero(corpus[:, 0] == corpus[b % 3, 0])
        run = np.arange(N // 2, N // 2 + 64)
        rep = int(rs.randint(N // 4, N))
        pick = np.concatenate([np.full(REPEAT, rep), sub[:M // 2], run, [5, 6], rs.randint(0, N, size=M)])[:M]
        pick = rs.permutation(pick)
        holes = (rs.rand(M) < 0.06) & (pick != rep) & ~np.isin(pick, sub) & ~np.isin(pick, run)
        pick[holes] = rs.choice([-1, -1, -1, N, N + 7, -2, -(1 << 40)], size=int(holes.sum()))
        items[b] = pick
    items[2] = rs.randint(N // 4, N)
    items[3] = -1
    return items


def sort_corpus(rs, M, K, H):
    N = max(2000, 2 * M)
    corpus = corpus_with_subtrees(rs, N, H, K)
    corpus[N // 2: N // 2 + 64, :2] = corpus[N // 2, :2]                # a 2-prefix of 64 items
    corpus[5, 1] = K                                                     # unretrievable rows
    corpus[6, H - 1] = -1
    return corpus


def assert_straddles(ref, items, M):
    """the REPEAT copies of row 0's repeated item take sorted slots c .. c + REPEAT - 1 with t IPT - 1 and t IPT among them"""
    ipt = 1 if M <= 512 else 2 if M <= 1024 else 4 if M <= 2048 else 8
    n_items = int(ref["start"][-1])
    inv = np.empty(len(ref["row"]), dtype=np.int64)
    inv[ref["row"]] = np.arange(len(ref["row"]))
    row = items[0]
    ok = (row >= 0) & (row < len(ref["row"]))
    pos = np.sort(inv[row[ok]])
    pos = pos[pos < n_items]
    vals, counts = np.unique(pos, return_counts=True)
    c = int(np.searchsorted(pos, vals[counts >= REPEAT][0]))
    assert any((c <= t * ipt - 1) and (t * ipt <= c + REPEAT - 1) for t in range(1, M // ipt + 1))


@pytest.mark.parametrize("M", WIDTHS)
def test_filter_builds_on_dense_rows(M):
    rs = np.random.RandomState(M)
    K, H, B = (300, 1000)[M % 2], 3, 5
    corpus = sort_corpus(rs, M, K, H)
    items = dense_rows(rs, corpus, B, M)
    ex_items = dense_rows(rs, corpus, B, M)
    ex_items[0] = np.where(rs.rand(M) < 0.5, items[0], ex_items[0])      # part of an allow-list excluded
    ex_items[4] = items[4]                                               # all of one
    _, ref, ex, inc, excls, incls = filters(corpus, K, items, ex_items)
    assert_straddles(ref, items, M)
    assert_exclusion(ex, excls, H)
    assert_inclusion(inc, incls, H)
    assert inc.count[4, 0] == 0 and inc.count[3, 0] == 0 and inc.count[2, 0] == 1
    assert len(excls[1]["blocked"][1]) > 0 and len(excls[1]["blocked"][2]) > 0


@pytest.mark.parametrize("M,ex_M", [(100, 4096), (4096, 100)])
def test_inclusion_with_exclusion_of_another_width(M, ex_M):
    rs = np.random.RandomState(M + 7)
    K, H, B = 300, 3, 5
    corpus = sort_corpus(rs, 4096, K, H)
    items = dense_rows(rs, corpus, B, M)
    ex_items = dense_rows(rs, corpus, B, ex_M)
    w = min(M, ex_M)
    ex_items[1, :w] = items[1, :w]                                       # part of history 1's allow-list excluded
    _, ref, ex, inc, excls, incls = filters(corpus, K, items, ex_items)
    assert_exclusion(ex, excls, H)
    assert_inclusion(inc, incls, H)
    assert len(incls[1]["eligible"]) < len(I.build(ref, items[1:2])[0]["eligible"])


def dense_candidates(rs, corpus, B, C, H, K):
    """[B, C, H]: corpus tuples of a small pool (duplicates and shared prefixes across thread boundaries), one tuple REPEAT
    times, and invalid tuples and -1 padding rows interleaved; history 2 is one tuple C times, history 3 all padding."""
    pool = corpus[rs.randint(0, len(corpus), size=max(C // 3, 1))]
    ids = pool[rs.randint(0, len(pool), size=(B, C))]
    for b in range(B):
        ids[b, rs.choice(C, size=REPEAT, replace=False)] = pool[0]
        holes = rs.choice(C, size=C // 15, replace=False)
        ids[b, holes[::3]] = -1
        ids[b, holes[1::3], rs.randint(0, H)] = K
        ids[b, holes[2::3], 0] = -5
    ids[2] = ids[2, 0]
    ids[3] = -1
    return ids


@pytest.mark.parametrize("C", WIDTHS)
def test_candidate_trie_on_dense_rows(C):
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(C + 1)
    K, H, B = (300, 1000)[C % 2], 3, 5
    ids = dense_candidates(rs, corpus_with_subtrees(rs, 2000, H, K), B, C, H, K)
    trie = [t.cpu().numpy() for t in ops.t5score_trie_build(dev(ids), K)]
    for b in range(B):
        for name, g, w in zip(("counts", "code", "parent", "child", "leaf"), trie, candidate_trie(ids[b], K)):
            assert np.array_equal(g[b], w), (b, name)


def kernel_names(run):
    """Names of the CUDA kernels run() launched, from torch.profiler.  A fill kernel launched after run() tells a complete trace
    from one the profiler did not deliver whole, which is profiled again (as in test_gpu_train_chain.py)."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
            torch.full((1,), 7.0, device="cuda")
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        if any("FillFunctor" in n for n in names):
            return names
    raise AssertionError("three profiler traces in a row hold no record of the marker kernel")


def test_every_sort_instantiation_runs():
    """The widths above launch all eight sid_filter_kernel<IPT, INCLUDE> and all four t5score_trie_kernel<IPT>."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(12)
    K, H, B = 300, 3, 2
    corpus = sort_corpus(rs, 4096, K, H)
    table = ops.SidItemTable(dev(corpus), K)
    keys = dev(X.leaf_keys(IO.build(corpus, K)))
    table.positions()

    def run():
        for M in WIDTHS:
            items = dev(dense_rows(rs, corpus, 5, M)[:B])
            ex = ops.sid_exclusion_build(items, table, keys)
            ops.sid_inclusion_build(items, table, keys, exclude=ex)
            ops.t5score_trie_build(dev(corpus[rs.randint(0, len(corpus), size=(B, M))]), K)

    names = kernel_names(run)
    found = lambda pattern: [m.groups() for m in map(re.compile(pattern).search, names) if m]
    filt = {(int(ipt), inc == "true") for ipt, inc in found(r"sid_filter_kernel<(\d+), (true|false)>")}
    trie = {int(ipt) for (ipt,) in found(r"t5score_trie_kernel<(\d+)>")}
    assert filt == {(ipt, inc) for ipt in (1, 2, 4, 8) for inc in (False, True)}, filt
    assert trie == {1, 2, 4, 8}, trie


# ------------------------------------------------------------------------------------------------ consumers at full filters
def full_exclusion(rs, corpus, B):
    """[B, 4096] of 4096 distinct items per history, shuffled: whole level-1 subtrees while they fit in 3500, then scattered
    rows."""
    N = len(corpus)
    out = np.empty((B, 4096), dtype=np.int64)
    firsts = np.unique(corpus[:, 0])
    for b in range(B):
        pick = []
        for c in rs.permutation(firsts):
            sub = np.flatnonzero(corpus[:, 0] == c)
            if len(pick) + len(sub) <= 3500:
                pick += sub.tolist()
        pick = np.array(pick + rs.permutation(np.setdiff1d(np.arange(N), pick)).tolist())[:4096]
        out[b] = rs.permutation(pick)
    return out


@pytest.mark.parametrize("N", [12101, 40000])
def test_consumers_of_a_4096_item_exclusion(N):
    """4096 excluded items per history: t5rank_select in the key path of its U (n = 1 and 1024, targets inside and outside the
    excluded set), retrieve with n = 4096, and on the smaller corpus both searches against the reduced-corpus search."""
    from rq_vae_recommender_b200 import ops
    K, H, B = 300, 3, 3
    rs = np.random.RandomState(N + 1)
    corpus = corpus_with_subtrees(rs, N, H, K)
    reps = corpus[rs.randint(0, N, size=min(1000, N // 25))]             # tuples of 10 items each
    corpus[N // 2: N // 2 + 10 * len(reps)] = np.repeat(reps, 10, axis=0)
    ex_items = full_exclusion(rs, corpus, B)
    table, ref, ex, _, excls, _ = filters(corpus, K, ex_items, ex_items)
    assert (ex.count[:, 0] == 4096).all() and all(len(w["blocked"][1]) > 0 for w in excls)
    U = len(ref["keys"])
    assert (U <= 24 * 1024) == (N == 12101)
    row, start = table.arrays()
    scores = rs.randn(B, U).round(1).astype(np.float32)
    scores[1, :50] = np.nan
    t_leaf, t_dedup = rank_targets(rs, ref, excls, B)
    for n in (1, 1024):
        got = ops.t5rank_select(dev(scores), row, start, dev(t_leaf), dev(t_dedup), n, exclude=ex)
        for a, w in zip(got, X.rank_select(ref, excls, scores, t_leaf, t_dedup, n)):
            np.testing.assert_array_equal(a.cpu().numpy(), w)
    assert got[2][0] == -1 and got[2][1] >= 0
    k = 1024                                                             # beams: every repeated tuple, then corpus rows
    gen = np.stack([np.concatenate([reps[rs.permutation(len(reps))], corpus[rs.randint(0, N, size=k - len(reps))]])
                    for _ in range(B)])
    lp = -np.sort(rs.rand(B, k), axis=1).astype(np.float32)
    lp[:, -3:] = -np.inf
    got = table.retrieve(dev(gen), dev(lp), 4096, exclude=ex)
    want = X.retrieve(ref, excls, gen, lp, 4096)
    for a, w in zip(got, want):
        np.testing.assert_array_equal(a.cpu().numpy(), w)
    assert (want[2] > 2048).all() and (N == 12101 or (want[2] == 4096).all())
    if N > 12101:
        return
    index = ops.SidPrefixIndex(dev(corpus), K)
    without = [ops.SidPrefixIndex(dev(np.delete(corpus, sorted(w["excluded"]), 0)), K) for w in excls]
    for search in ("beam", "sample"):
        assert_search_equals_reduced(H, index, without, tail_logits(K), search, 32 if search == "beam" else 16,
                                     exclude=ex)


def test_searches_with_4096_allowed_items_under_one_prefix():
    """K = 2048: each history allows 4096 items under the level-1 prefix 7, so the mask of the beam (7,) is built from up to 2048
    allowed level-2 keys; both searches equal the search on the eligible corpus."""
    from rq_vae_recommender_b200 import ops
    K, H, B = 2048, 3, 3
    rs = np.random.RandomState(2048)
    corpus = corpus_with_subtrees(rs, 12101, H, K)
    corpus[:6000, 0] = 7
    items = np.stack([rs.permutation(rs.permutation(6000)[:4096]) for _ in range(B)])
    ex_items = np.full((B, 1), -1, dtype=np.int64)
    ex_items[1, 0] = items[1, 0]
    _, ref, _, inc, _, incls = filters(corpus, K, items, ex_items)
    assert len(incls[0]["keys"][2]) > 1500 and (inc.count[:, 1] == 1).all()
    index = ops.SidPrefixIndex(dev(corpus), K)
    eligible = [ops.SidPrefixIndex(dev(corpus[sorted(w["eligible"])]), K) for w in incls]

    def logits_of(h, rows):
        logits = torch.randn(rows, K, device="cuda") * 3
        if h == 0:
            logits[:, 7] += 5                                            # the only valid first code: sampled too
        return logits

    for search in ("beam", "sample"):
        assert_search_equals_reduced(H, index, eligible, logits_of, search, 32 if search == "beam" else 16,
                                     include=inc)


# ------------------------------------------------------------------------------------------------ key-width limits
@pytest.mark.parametrize("K,H", [(2048, 6), (256, 8), (300, 8), (1000, 7)])
def test_filter_builds_refuse_keys_above_62_bits(K, H):
    from rq_vae_recommender_b200 import _lib, ops
    rs = np.random.RandomState(K + H)
    corpus = rs.randint(0, K, size=(50, H)).astype(np.int64)
    table = ops.SidItemTable(dev(corpus), K)
    keys = torch.zeros(50, dtype=torch.int64, device="cuda")             # refused before the keys are read
    items = dev(rs.randint(0, 50, size=(2, 8)))
    launches = ops.LAUNCHES
    with pytest.raises(_lib.Rqb200Error, match=r"H \* bits\(K - 1\) <= 62"):
        ops.sid_exclusion_build(items, table, keys)
    with pytest.raises(_lib.Rqb200Error, match=r"H \* bits\(K - 1\) <= 62"):
        ops.sid_inclusion_build(items, table, keys)
    assert ops.LAUNCHES == launches
