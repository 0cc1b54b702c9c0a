"""Plain-torch statement of the fused T5 decode of ``generate(decoder="fused")`` (modules/model.py ``FusedT5Decode``), and the
drivers that compare it with transformers' T5Stack run the way ``generate(decoder="hf")`` runs it.

The decomposition it states:
  * cross-attention keys/values projected once per history (B rows, never B * k), every beam of history b reads history b's;
  * self-attention keys/values of position j kept in slot j, each beam reading its earlier positions through an ancestor table
    anc [rows, H] that the search's parent_global advances: anc'[r] = anc[parent[r]], anc'[r][h - 1] = parent[r];
  * level 1 reuses level 0's BOS keys/values (HF re-runs [BOS, tok0] on B * k rows);
  * the relative-position bias is HF's own ``block[0].layer[0].SelfAttention.compute_bias(H, H)``.
The kernel-level functions (``cross_attention``, ``self_attention``, ``add_norm``) follow the C ABI's contracts in
include/rqb200.h, so the GPU tests compare each kernel with them."""
import torch
import torch.nn.functional as F

DKV = 64
NEG = torch.finfo(torch.float32).min


def cross_attention(q, k, v, mask, nq, heads):
    """q [B * nq, inner], k / v [B * S, inner], mask [B, S] or None -> [B * nq, inner]."""
    B = q.shape[0] // nq
    S = k.shape[0] // B
    qh = q.reshape(B, nq, heads, DKV).transpose(1, 2)                         # [B, heads, nq, 64]
    kh = k.reshape(B, S, heads, DKV).transpose(1, 2)
    vh = v.reshape(B, S, heads, DKV).transpose(1, 2)
    scores = qh @ kh.transpose(2, 3)                                           # no 1/sqrt(d) scaling
    if mask is not None:
        scores = scores + torch.where(mask != 0, 0.0, NEG).to(scores.dtype)[:, None, None, :]
    w = torch.softmax(scores.float(), dim=-1).to(scores.dtype)
    return (w @ vh).transpose(1, 2).reshape(B * nq, heads * DKV)


def self_attention(qkv, cache_k, cache_v, bias, h, anc):
    """qkv [R, 3 inner], cache_k / cache_v [H, rows, inner] (slot h of rows 0..R-1 is written), bias [heads, H, H], anc [R, H]
    (positions j < h) -> [R, inner]."""
    R = qkv.shape[0]
    H, _, inner = cache_k.shape
    heads = inner // DKV
    q, k, v = qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:]
    cache_k[h, :R] = k
    cache_v[h, :R] = v
    keys = torch.stack([cache_k[j, anc[:, j].long()] for j in range(h)] + [k], dim=1)    # [R, h + 1, inner]
    vals = torch.stack([cache_v[j, anc[:, j].long()] for j in range(h)] + [v], dim=1)
    qh = q.reshape(R, heads, 1, DKV)
    kh = keys.reshape(R, h + 1, heads, DKV).permute(0, 2, 3, 1)              # [R, heads, 64, h + 1]
    scores = (qh @ kh)[:, :, 0, :] + bias[:, h, :h + 1][None]                # [R, heads, h + 1]
    w = torch.softmax(scores.float(), dim=-1).to(scores.dtype)
    vh = vals.reshape(R, h + 1, heads, DKV).transpose(1, 2)                  # [R, heads, h + 1, 64]
    return (w[:, :, None, :] @ vh)[:, :, 0, :].reshape(R, inner)


def advance_ancestors(anc, parent, h):
    """The ancestor table of level h's rows from level h - 1's table and the search's parent_global."""
    out = anc[parent.long()].clone()
    out[:, h - 1] = parent.to(out.dtype)
    return out


def add_norm(x, delta, weight, eps):
    """x + delta (in place, delta None: x unchanged) and T5LayerNorm(x) * weight."""
    if delta is not None:
        x += delta
    var = x.float().pow(2).mean(-1, keepdim=True)
    return weight * (x * torch.rsqrt(var + eps))


class FusedDecodeRef:
    """FusedT5Decode in plain torch (same constructor and ``step``)."""

    def __init__(self, model, enc_out, enc_mask, k):
        dec = model.t5_decoder
        self.model, self.k, self.H = model, k, model.num_hierarchies
        self.heads, self.eps = dec.config.num_heads, dec.config.layer_norm_epsilon
        self.blocks = [blk.layer for blk in dec.block]
        B, S, d = enc_out.shape
        self.B, inner = B, self.heads * DKV
        self.inner = inner
        w_kv = torch.cat([w for lay in self.blocks for w in (lay[1].EncDecAttention.k.weight, lay[1].EncDecAttention.v.weight)])
        self.cross_kv = F.linear(enc_out.reshape(B * S, d), w_kv)
        self.mask = enc_mask.float()
        self.bias = dec.block[0].layer[0].SelfAttention.compute_bias(self.H, self.H)[0]
        self.cache = torch.zeros((len(self.blocks), 2, self.H, B * k, inner), dtype=enc_out.dtype, device=enc_out.device)
        self.anc = torch.zeros((B * k, self.H), dtype=torch.int32, device=enc_out.device)
        self.final = dec.final_layer_norm.weight

    def step(self, h, generated, parent):
        m, eps, inner = self.model, self.eps, self.inner
        nq = 1 if h == 0 else self.k
        R = self.B * nq
        if h == 0:
            x = m.bos_token.expand(R, -1).clone()
        else:
            self.anc = advance_ancestors(self.anc, parent, h)
            x = m.item_sid_embedding_table.weight[generated.reshape(R, h)[:, h - 1] + (h - 1) * m.num_embeddings_per_hierarchy].clone()
        nrm = add_norm(x, None, self.blocks[0][0].layer_norm.weight, eps)
        for l, lay in enumerate(self.blocks):
            att = lay[0].SelfAttention
            qkv = F.linear(nrm, torch.cat([att.q.weight, att.k.weight, att.v.weight]))
            a = self_attention(qkv, self.cache[l, 0], self.cache[l, 1], self.bias, h, self.anc[:R])
            nrm = add_norm(x, F.linear(a, att.o.weight), lay[1].layer_norm.weight, eps)
            kv = self.cross_kv[:, 2 * l * inner:(2 * l + 2) * inner]
            xatt = lay[1].EncDecAttention
            a = cross_attention(F.linear(nrm, xatt.q.weight), kv[:, :inner], kv[:, inner:], self.mask, nq, self.heads)
            nrm = add_norm(x, F.linear(a, xatt.o.weight), lay[2].layer_norm.weight, eps)
            ff = lay[2].DenseReluDense
            nxt = self.blocks[l + 1][0].layer_norm.weight if l + 1 < len(self.blocks) else self.final
            nrm = add_norm(x, F.linear(F.relu(F.linear(nrm, ff.wi.weight)), ff.wo.weight), nxt, eps)
        return nrm


def random_beams(B, k, H, K, seed, device="cpu"):
    """Per level h < H - 1: (generated [B, k, h + 1] int64, parent_global [B * k] int64) as a search would hand them on -- every
    beam's parent in its own history, parents repeated and skipped at random."""
    g = torch.Generator().manual_seed(seed)
    out, gen = [], None
    for h in range(H - 1):
        if h == 0:
            parent = torch.arange(B).repeat_interleave(k)
            gen = torch.randint(0, K, (B, k, 1), generator=g)
        else:
            beam = torch.randint(0, k, (B, k), generator=g)
            parent = (beam + torch.arange(B)[:, None] * k).reshape(-1)
            gen = torch.cat([gen.reshape(B * k, h)[parent].reshape(B, k, h), torch.randint(0, K, (B, k, 1), generator=g)], dim=2)
        out.append((gen.to(device), parent.to(device)))
    return out


def hf_level_logits(model, enc_out, enc_mask, beams, k):
    """Per-level head logits of T5Stack driven exactly as generate(decoder="hf") drives it, fed the given beams."""
    from transformers.cache_utils import DynamicCache, EncoderDecoderCache
    rep_enc, rep_mask = enc_out.repeat_interleave(k, dim=0), enc_mask.repeat_interleave(k, dim=0)
    past_kv = EncoderDecoderCache(DynamicCache(), DynamicCache())
    out, generated = [], None
    for h in range(model.num_hierarchies):
        first = generated is None
        dec_out, past_kv = model.decoder_forward_pass(
            future_ids=None if first else generated.reshape(-1, h), encoder_output=enc_out if first else rep_enc,
            attention_mask_for_encoder=enc_mask if first else rep_mask, use_cache=True, past_key_values=past_kv)
        out.append(model.decoder_mlp[h](dec_out[:, -1, :]))
        if h + 1 < model.num_hierarchies:
            generated, parent = beams[h]
            if first:
                past_kv = EncoderDecoderCache(DynamicCache(), DynamicCache())
            else:
                past_kv.reorder_cache(parent)
    return out


def fused_level_logits(model, enc_out, enc_mask, beams, k, decode_cls=FusedDecodeRef):
    """Per-level head logits of a fused decode (``decode_cls``: this module's FusedDecodeRef or the model's FusedT5Decode)."""
    dec = decode_cls(model, enc_out, enc_mask, k)
    out, generated, parent = [], None, None
    for h in range(model.num_hierarchies):
        out.append(model.decoder_mlp[h](dec.step(h, generated, parent)))
        if h + 1 < model.num_hierarchies:
            generated, parent = beams[h]
    return out
