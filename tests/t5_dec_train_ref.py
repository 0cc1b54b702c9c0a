"""Plain-torch statement of the fused training decoder pass of ``forward(decoder="fused")`` (modules/model.py
``FusedT5DecodeTrain``), with its dropout given as explicit keep masks.

The decomposition it states:
  * only the T = H positions the loss reads run: row b * T + t holds position t of history b, its input ``bos_token`` at t = 0
    and ``item_sid_embedding_table[fut_ids[b, t - 1] + (t - 1) K]`` after.  HF runs one more position (the last future id), which
    causality keeps out of every earlier position;
  * self-attention is causal with block 0's unidirectional relative-position bias (``compute_bias(T, T)``);
  * cross-attention reads history b's encoder rows offsets[b] .. offsets[b + 1] - 1 with an additive per-key mask: the packed kept
    rows of the fused encoder (a history's key_mask on each of its rows) or the [B * S] rows of HF's encoder (finfo.min where its
    mask is 0).  Either layout gives HF's output: a dropped position has weight exactly 0 in HF's softmax;
  * HF's nine dropout sites in HF's call order: the embedding output, per layer the self-attention weights and output, the
    cross-attention weights and output, the feed-forward inner activation and output, and the final norm's output.
Masks are given at HF's shapes (T + 1 positions); the statement reads the first T positions of each and, for cross-attention, the
key's ORIGINAL encoder position, so one list drives HF (through a patched ``F.dropout``) and this statement.  Run it on a float64
copy of the model; finfo(float32).min stays the mask value, and the scores of a fully masked history round to it in float64 as in
fp32, so its softmax is uniform as HF's is."""
import torch
import torch.nn.functional as F

import t5_enc_ref as E
from t5_enc_train_ref import t5_norm
from t5_step_ref import DKV, NEG


def dropout_shapes(model, B, T, S):
    """The shapes of HF's dropout calls in one decoder pass over BOS and T future ids (T + 1 positions), in call order."""
    cfg = model.t5_decoder.config
    d, h, ff, P = cfg.d_model, cfg.num_heads, cfg.d_ff, T + 1
    per_layer = [(B, h, P, P), (B, P, d), (B, h, P, S), (B, P, d), (B, P, ff), (B, P, d)]
    return [(B, P, d)] + per_layer * cfg.num_layers + [(B, P, d)]


def random_masks(model, B, T, S, p, seed, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    return [(torch.rand(shape, generator=g) >= p).to(dtype) for shape in dropout_shapes(model, B, T, S)]


def self_attention_train(qkv, rel, T, keep=None, p=0.0):
    """Causal self-attention of T positions per history: qkv [B * T, 3 inner] -> [B * T, inner].  rel [heads, 2T - 1]; keep
    [B, heads, >= T, >= T] or None."""
    heads = rel.shape[0]
    inner = heads * DKV
    B = qkv.shape[0] // T
    q, k, v = (qkv[:, i * inner:(i + 1) * inner].reshape(B, T, heads, DKV).transpose(1, 2) for i in range(3))
    pos = torch.arange(T, device=qkv.device)
    bias = rel[:, pos[None, :] - pos[:, None] + T - 1]                       # [heads, query, key]
    causal = torch.where(pos[None, :] > pos[:, None], NEG, 0.0).to(qkv.dtype)
    w = torch.softmax(q @ k.transpose(-1, -2) + (bias + causal), dim=-1)     # HF's order: scores += (bias + mask)
    if keep is not None:
        w = w * keep[:, :, :T, :T].to(w.dtype) / (1 - p)
    return (w @ v).transpose(1, 2).reshape(B * T, inner)


def cross_attention_train(q, kv, offs, key_mask, kpos, T, keep=None, p=0.0):
    """q [B * T, inner] over key rows offs[b] .. offs[b + 1] - 1 of kv [rows, 2 inner] (k | v) with additive key_mask [rows];
    kpos [rows] is each key's original encoder position, the column of keep [B, heads, >= T, S] it reads."""
    inner = q.shape[1]
    heads = inner // DKV
    outs = []
    for b in range(offs.shape[0] - 1):
        lo, hi = int(offs[b]), int(offs[b + 1])
        qb = q[b * T:(b + 1) * T].reshape(T, heads, DKV).transpose(0, 1)
        k, v = (kv[lo:hi, i * inner:(i + 1) * inner].reshape(hi - lo, heads, DKV).transpose(0, 1) for i in range(2))
        w = torch.softmax(qb @ k.transpose(1, 2) + key_mask[lo:hi], dim=-1)
        if keep is not None:
            w = w * keep[b][:, :T][:, :, kpos[lo:hi].long()].to(w.dtype) / (1 - p)
        outs.append((w @ v).transpose(0, 1).reshape(T, inner))
    return torch.cat(outs)


def decode_train(model, fut_ids, rows, offs, key_mask, kpos, masks=None, p=0.0, relu=None, pre=None):
    """The decoder pass: [B, T, d] (the final norm's output after its dropout), differentiable in every parameter and in rows.
    masks: HF-order keep masks (``random_masks``) or None for no dropout.  relu: one [B, T + 1, d_ff] mask per feed-forward, in
    call order, nonzero where its relu passes (the first T positions are read): the pass computes ``pre * mask`` in place of
    ``F.relu(pre)``; None uses F.relu.  pre: a list each feed-forward's pre-activation [B * T, d_ff] is appended to, or None."""
    dec = model.t5_decoder
    T, K, eps = model.num_hierarchies, model.num_embeddings_per_hierarchy, dec.config.layer_norm_epsilon
    B, d = fut_ids.shape[0], model.bos_token.shape[1]
    table = model.item_sid_embedding_table.weight
    idx = fut_ids[:, :T - 1].long() + torch.arange(T - 1, device=fut_ids.device) * K
    x = torch.cat([model.bos_token.expand(B, 1, d), table[idx]], dim=1).reshape(B * T, d)
    queue = list(masks) if masks is not None else None

    def drop(t):                                            # a token-wise site: the first T positions of the next [B, T + 1, *] mask
        if queue is None:
            return t
        return t * queue.pop(0)[:, :T].reshape(B * T, -1).to(t.dtype) / (1 - p)

    def keep():
        return queue.pop(0) if queue is not None else None

    relus = list(relu) if relu is not None else None

    def act(t):                                             # a feed-forward relu: F.relu, or the first T positions of the next mask
        if pre is not None:
            pre.append(t.detach())
        if relus is None:
            return F.relu(t)
        return t * relus.pop(0)[:, :T].reshape(B * T, -1).to(t.dtype)

    blocks = [blk.layer for blk in dec.block]
    rel = E.rel_bias(blocks[0][0].SelfAttention.compute_bias(T, T)[0])
    x = drop(x)
    for lay in blocks:
        att = lay[0].SelfAttention
        qkv = F.linear(t5_norm(x, lay[0].layer_norm.weight, eps), torch.cat([att.q.weight, att.k.weight, att.v.weight]))
        x = x + drop(F.linear(self_attention_train(qkv, rel, T, keep(), p), att.o.weight))
        ca = lay[1].EncDecAttention
        q = F.linear(t5_norm(x, lay[1].layer_norm.weight, eps), ca.q.weight)
        kv = F.linear(rows, torch.cat([ca.k.weight, ca.v.weight]))
        x = x + drop(F.linear(cross_attention_train(q, kv, offs, key_mask, kpos, T, keep(), p), ca.o.weight))
        ff = lay[2].DenseReluDense
        h = drop(act(F.linear(t5_norm(x, lay[2].layer_norm.weight, eps), ff.wi.weight)))
        x = x + drop(F.linear(h, ff.wo.weight))
    out = drop(t5_norm(x, dec.final_layer_norm.weight, eps))
    assert not queue and not relus
    return out.reshape(B, T, d)


def padded_layout(enc_out, enc_mask):
    """HF's encoder output as decoder key rows: (rows [B * S, d], offsets, key_mask [B * S], kpos [B * S])."""
    B, S, d = enc_out.shape
    offs = torch.arange(0, (B + 1) * S, S, dtype=torch.int32, device=enc_out.device)
    key_mask = torch.where(enc_mask == 0, NEG, 0.0).to(enc_out.dtype).reshape(B * S)
    return enc_out.reshape(B * S, d), offs, key_mask, torch.arange(S, device=enc_out.device).repeat(B)


def packed_layout(enc_out, attention_mask, H, sep, user):
    """The kept rows of the fused encoder's [B, S, d] output, packed: (rows [N, d], offsets, key_mask [N], kpos [N])."""
    B, S, d = enc_out.shape
    keep, km = E.kept_positions(attention_mask, H, sep, user)
    src = keep.reshape(-1).nonzero().squeeze(1)
    offs, _ = E.offsets(attention_mask, H, sep, user)
    return enc_out.reshape(B * S, d)[src], offs, km.to(enc_out.dtype)[src // S], src % S


def level_loss(model, dec, fut_ids):
    """``forward``'s loss: the sum over levels of the cross-entropy of head h on position h."""
    return sum(F.cross_entropy(model.decoder_mlp[h](dec[:, h]), fut_ids[:, h].long()) for h in range(model.num_hierarchies))
