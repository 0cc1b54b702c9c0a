"""Plain-torch statement of the trainable packed encoder pass of ``forward(encoder="fused")`` (modules/model.py
``FusedT5EncodeTrain``), with its dropout given as explicit keep masks.

It is tests/t5_enc_ref.py's packed pass with HF's six dropout sites, in HF's call order:
  * the embedding output (T5Stack.dropout), [B, S, d];
  * per layer: the attention weights (T5Attention.dropout), [B, heads, S, S]; the attention output (T5LayerSelfAttention.dropout),
    [B, S, d]; the feed-forward inner activation (T5DenseActDense.dropout), [B, S, d_ff]; the feed-forward output
    (T5LayerFF.dropout), [B, S, d];
  * the final norm's output (T5Stack.dropout), [B, S, d].
Masks are given at HF's full shapes; the packed pass reads each kept row's (and each kept query/key pair's) entry, so the same
list drives both HF (through a patched ``F.dropout``) and this statement.  Gradients come from torch autograd.  Run it on a
float64 copy of the model: every step, the softmax included, is then float64 (HF casts scores to fp32 for its softmax, so HF
itself is only an fp32 reference).  The mask value stays HF's finfo(float32).min; scores of a fully masked history round to it in
float64 as they do in fp32."""
import torch
import torch.nn.functional as F

import t5_enc_ref as E
from t5_step_ref import DKV


def dropout_shapes(model, B, S):
    """The shapes of HF's dropout calls in one encoder pass, in call order."""
    cfg = model.encoder.config
    d, h, ff = cfg.d_model, cfg.num_heads, cfg.d_ff
    per_layer = [(B, h, S, S), (B, S, d), (B, S, ff), (B, S, d)]
    return [(B, S, d)] + per_layer * cfg.num_layers + [(B, S, d)]


def random_masks(model, B, S, p, seed, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    return [(torch.rand(shape, generator=g) >= p).to(dtype) for shape in dropout_shapes(model, B, S)]


def hf_dropout_from(masks):
    """A stand-in for ``torch.nn.functional.dropout`` that applies the given masks in call order."""
    queue = list(masks)

    def dropout(x, p=0.5, training=True, inplace=False):
        if not training:
            return x
        mask = queue.pop(0)
        assert mask.shape == x.shape, (mask.shape, x.shape)
        return x * mask.to(x.dtype) / (1 - p)
    dropout.queue = queue
    return dropout


def attention_train(qkv, src, offs, key_mask, rel, S, keep=None, p=0.0):
    """Packed self-attention with HF's attention-weight dropout: qkv [N, 3 inner] -> [N, inner].  keep [B, heads, S, S] (at the
    original positions) or None; key_mask [B] holds finfo(float32).min for a history without an unmasked position."""
    heads = rel.shape[0]
    inner = heads * DKV
    outs = []
    for b in range(offs.shape[0] - 1):
        lo, hi = int(offs[b]), int(offs[b + 1])
        if hi == lo:
            continue
        pos = src[lo:hi].long() - b * S
        q, k, v = (qkv[lo:hi, i * inner:(i + 1) * inner].reshape(hi - lo, heads, DKV).transpose(0, 1) for i in range(3))
        bias = rel[:, pos[None, :] - pos[:, None] + S - 1]
        scores = q @ k.transpose(1, 2) + (bias + key_mask[b])
        w = torch.softmax(scores, dim=-1)
        if keep is not None:
            w = w * keep[b][:, pos][:, :, pos].to(w.dtype) / (1 - p)
        outs.append((w @ v).transpose(0, 1).reshape(hi - lo, inner))
    return torch.cat(outs)


def t5_norm(x, weight, eps):
    return weight * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def encode_train(model, attention_mask, input_ids, user_id=None, masks=None, p=0.0, relu=None, pre=None):
    """The packed training pass: (enc_out [B, S, d] with dropped rows 0, enc_mask [B, S]), differentiable in every parameter.
    masks: HF-order keep masks (``random_masks``) or None for no dropout.  relu: one [B, S, d_ff] mask per feed-forward, in call
    order, nonzero where its relu passes: the pass computes ``pre * mask`` in place of ``F.relu(pre)``, so it can follow another
    pass's relu decisions; None uses F.relu.  pre: a list each feed-forward's pre-activation [N, d_ff] is appended to, or None."""
    enc = model.encoder.encoder
    H, eps = model.num_hierarchies, enc.config.layer_norm_epsilon
    sep = model.sep_token is not None
    user = user_id is not None and model.user_embedding is not None
    B, n = attention_mask.shape
    enc_mask = attention_mask
    if sep:
        items = enc_mask.view(B, n // H, H)
        enc_mask = torch.cat([items, items[:, :, -1:]], dim=2).reshape(B, -1)
    if user:
        enc_mask = torch.cat([torch.ones(B, 1, device=enc_mask.device), enc_mask], dim=1)
    offs, key_mask = E.offsets(attention_mask, H, sep, user)
    x, src, slot = E.assemble(attention_mask, input_ids, user_id if user else None, model.item_sid_embedding_table.weight,
                              model.sep_token if sep else None, model.user_embedding.weight if user else None,
                              model.num_embeddings_per_hierarchy, H)
    dtype = x.dtype
    key_mask = key_mask.to(dtype)                          # finfo(float32).min, HF's value for its fp32 model, exact in float64
    S = slot.shape[1]
    queue = list(masks) if masks is not None else None
    rows = src.long()

    def drop(t):                                           # a token-wise site: the kept rows of the next [B, S, *] mask
        if queue is None:
            return t
        m = queue.pop(0)
        return t * m.reshape(B * S, -1)[rows].to(t.dtype) / (1 - p)

    relus = list(relu) if relu is not None else None

    def act(t):                                            # a feed-forward relu: F.relu, or the kept rows of the next relu mask
        if pre is not None:
            pre.append(t.detach())
        if relus is None:
            return F.relu(t)
        return t * relus.pop(0).reshape(B * S, -1)[rows].to(t.dtype)

    blocks = [blk.layer for blk in enc.block]
    rel = E.rel_bias(blocks[0][0].SelfAttention.compute_bias(S, S)[0])
    x = drop(x)
    for lay in blocks:
        att = lay[0].SelfAttention
        qkv = F.linear(t5_norm(x, lay[0].layer_norm.weight, eps), torch.cat([att.q.weight, att.k.weight, att.v.weight]))
        keep = queue.pop(0) if queue is not None else None
        a = attention_train(qkv, src, offs, key_mask, rel, S, keep, p)
        x = x + drop(F.linear(a, att.o.weight))
        ff = lay[1].DenseReluDense
        h = drop(act(F.linear(t5_norm(x, lay[1].layer_norm.weight, eps), ff.wi.weight)))
        x = x + drop(F.linear(h, ff.wo.weight))
    out = drop(t5_norm(x, enc.final_layer_norm.weight, eps))
    assert not queue and not relus
    return E.scatter(out, slot), enc_mask
