"""Plain-torch statement of the exact ranking of ``EncoderDecoderRetrievalModel.rank_sem_ids`` / ``rank_items`` (modules/model.py
``FusedT5Rank``, csrc/t5rank.cu), and the statements it is checked against.

The decomposition: items that share an l-prefix share the causal decoder's state at positions 0..l, so one decoder row per node of
the corpus trie per history (level h: the distinct h-prefixes; level 0: BOS) gives each child's log-probability, and a tuple's
score is the sum along its path.  ``trie_levels`` builds the levels on the host, ``rank_decompose`` decodes them with the kernel-level
functions of t5_step_ref (ancestors through an advanced table, cross keys and values shared by a history's rows), and
``rank_teacher_forced`` runs HF's T5Stack on BOS + the first H - 1 ids of each tuple alone."""
import numpy as np
import torch
import torch.nn.functional as F

import t5_step_ref as T


def trie_levels(corpus: np.ndarray, H: int, K: int):
    """Per level l = 1..H: the sorted distinct l-prefixes of the rows whose first l ids are in [0, K) ([n_l, l] int64) and each
    node's parent in level l - 1.  Level H is the item table's tuple order."""
    levels, parents = [np.zeros((1, 0), dtype=np.int64)], [None]
    for l in range(1, H + 1):
        rows = corpus[:, :l]
        ok = ((rows >= 0) & (rows < K)).all(1)
        nodes = np.unique(rows[ok], axis=0) if ok.any() else np.zeros((0, l), dtype=np.int64)
        prev = levels[-1]
        parent = np.array([np.nonzero((prev == nd[:l - 1]).all(1))[0][0] for nd in nodes], dtype=np.int64)
        levels.append(nodes)
        parents.append(parent)
    return levels, parents


def items_of_leaves(corpus: np.ndarray, leaves: np.ndarray):
    """Each leaf's corpus rows in ascending row order (dedup rank 0, 1, ...)."""
    return [np.nonzero((corpus[:, :leaves.shape[1]] == t).all(1))[0] for t in leaves]


def rank_decompose(model, enc_out, enc_mask, levels, parents):
    """[B, U] leaf scores: one decoder row per trie node per history, as FusedT5Rank computes them, in the model's dtype."""
    dec = model.t5_decoder
    H, K = model.num_hierarchies, model.num_embeddings_per_hierarchy
    heads, eps = dec.config.num_heads, dec.config.layer_norm_epsilon
    blocks = [blk.layer for blk in dec.block]
    inner = heads * T.DKV
    B, S, d = enc_out.shape
    bias = blocks[0][0].SelfAttention.compute_bias(H, H)[0]
    n = [len(lv) for lv in levels]
    width = max(n[:H])
    cache = torch.zeros((len(blocks), 2, H, B * width, inner), dtype=enc_out.dtype)
    anc = torch.zeros((B * width, H), dtype=torch.int64)
    score = torch.zeros((B, 1), dtype=enc_out.dtype)
    for h in range(H):
        R = B * n[h]
        if h == 0:
            x = model.bos_token.expand(R, -1).clone()
        else:
            code = torch.from_numpy(levels[h][:, h - 1]).repeat(B)
            x = model.item_sid_embedding_table.weight[code + (h - 1) * K].clone()
            parent = (torch.arange(B)[:, None] * n[h - 1] + torch.from_numpy(parents[h])[None]).reshape(-1)
            anc = T.advance_ancestors(anc, parent, h)
        nrm = T.add_norm(x, None, blocks[0][0].layer_norm.weight, eps)
        for l, lay in enumerate(blocks):
            att = lay[0].SelfAttention
            qkv = F.linear(nrm, torch.cat([att.q.weight, att.k.weight, att.v.weight]))
            a = T.self_attention(qkv, cache[l, 0], cache[l, 1], bias, h, anc[:R])
            nrm = T.add_norm(x, F.linear(a, att.o.weight), lay[1].layer_norm.weight, eps)
            xatt = lay[1].EncDecAttention
            k, v = F.linear(enc_out.reshape(B * S, d), xatt.k.weight), F.linear(enc_out.reshape(B * S, d), xatt.v.weight)
            a = T.cross_attention(F.linear(nrm, xatt.q.weight), k, v, enc_mask, n[h], heads)
            nrm = T.add_norm(x, F.linear(a, xatt.o.weight), lay[2].layer_norm.weight, eps)
            ff = lay[2].DenseReluDense
            nxt = blocks[l + 1][0].layer_norm.weight if l + 1 < len(blocks) else dec.final_layer_norm.weight
            nrm = T.add_norm(x, F.linear(F.relu(F.linear(nrm, ff.wi.weight)), ff.wo.weight), nxt, eps)
        logp = torch.log_softmax(model.decoder_mlp[h](nrm), dim=-1).reshape(B, n[h], K)
        child = torch.from_numpy(levels[h + 1][:, h])
        par = torch.from_numpy(parents[h + 1])
        score = score[:, par] + logp[:, par, child]
    return score


def rank_teacher_forced(model, enc_out, enc_mask, leaves):
    """[B, U]: each tuple's log-probability from HF's T5Stack run on BOS + its first H - 1 ids alone."""
    H = model.num_hierarchies
    B, U = enc_out.shape[0], leaves.shape[0]
    t = torch.from_numpy(leaves)
    fut = t[:, :H - 1].repeat(B, 1)
    out = model.decoder_forward_pass(future_ids=fut, encoder_output=enc_out.repeat_interleave(U, 0),
                                     attention_mask_for_encoder=enc_mask.repeat_interleave(U, 0))
    total = torch.zeros(B * U, dtype=enc_out.dtype)
    for h in range(H):
        logp = torch.log_softmax(model.decoder_mlp[h](out[:, h]), dim=-1)
        total = total + logp.gather(1, t[:, h].repeat(B)[:, None])[:, 0]
    return total.reshape(B, U)


def select_model(scores: np.ndarray, counts: np.ndarray, n: int, t_leaf: int, t_dedup: int):
    """The selection rule of t5rank_select for one history, stated the way the kernel computes it: the n-th best 32-bit score key
    T (NaN lowest, -0 = +0), every leaf above T and the lowest-index leaves at T, ranked by (score, leaf), expanded to items;
    the target's rank is the count of items of the leaves before it plus its dedup rank.  Returns ((leaf, dedup) pairs [<= n],
    target rank)."""
    U = scores.shape[0]
    key = np.where(np.isnan(scores), -np.inf, scores)
    nan = np.isnan(scores)
    order_key = [(0 if nan[u] else 1, key[u], -u) for u in range(U)]
    nsel = min(n, U)
    chosen = sorted(range(U), key=lambda u: order_key[u], reverse=True)[:nsel]
    threshold = order_key[chosen[-1]][:2] if nsel else None
    above = [u for u in range(U) if nsel and order_key[u][:2] > threshold]
    ties = [u for u in range(U) if nsel and order_key[u][:2] == threshold][:nsel - len(above)]
    kept = sorted(above + ties, key=lambda u: order_key[u], reverse=True)
    out = [(u, d) for u in kept for d in range(counts[u])][:n]
    rank = -1
    if 0 <= t_leaf < U and 0 <= t_dedup < counts[t_leaf]:
        rank = int(sum(counts[u] for u in range(U) if order_key[u] > order_key[t_leaf])) + t_dedup
    return out, rank


def sort_items(scores: np.ndarray, counts: np.ndarray):
    """Every (leaf, dedup) pair by a plain sort: score descending (NaN last), then leaf, then dedup."""
    leaf = np.repeat(np.arange(scores.shape[0]), counts)
    dedup = np.concatenate([np.arange(c) for c in counts]) if len(counts) else np.zeros(0, dtype=np.int64)
    s = scores[leaf]
    nan = np.isnan(s)
    order = np.lexsort((dedup, leaf, -np.where(nan, 0, s), nan))
    return list(zip(leaf[order].tolist(), dedup[order].tolist()))
