"""Plain-torch statement of the packed encoder pass of ``generate(encoder="fused")`` (modules/model.py ``FusedT5Encode``).

The decomposition it states:
  * position p of a history's encoder input is the user row (p = 0 with a user token), an item id, or the separator after an
    item (carrying the mask of the item's last id), exactly as ``encoder_forward_pass`` lays them out;
  * a position is kept when its mask is nonzero (the user row always is); a history with no such position keeps all of them and
    adds finfo(float32).min to every key, which is what HF's eager mask does (its softmax then averages every position);
  * kept rows are packed history by history in position order, and every token-wise step (embedding gather, T5LayerNorm, the
    GEMMs, the residual adds) runs on the packed rows;
  * self-attention runs among each history's packed rows, with HF's relative-position bias taken at the ORIGINAL positions:
    ``compute_bias(S, S)`` of block 0 depends only on key - query position, so its [heads, 2S - 1] slice holds every value;
  * the output is scattered back to [B, S, d] with the rows of dropped positions set to 0.
The kernel-level functions (``offsets``, ``assemble``, ``rel_bias``, ``attention``, ``scatter``) follow the C ABI's contracts in
include/rqb200.h, so the GPU tests compare each kernel with them."""
import torch
import torch.nn.functional as F

from t5_step_ref import DKV, NEG, add_norm


def layout(n, H, sep, user, device="cpu"):
    """Per encoder position: kind (0 user, 1 item id, 2 separator), the column of the [B, n] inputs it reads (the item's last id
    for a separator) and the id's level."""
    W = H + int(sep)
    q = torch.arange(n // H * W, device=device)
    item, j = q // W, q % W
    kind = torch.where(j < H, 1, 2)
    col = item * H + torch.clamp(j, max=H - 1)
    lvl = torch.where(j < H, j, 0)
    if user:
        zero = torch.zeros(1, dtype=torch.long, device=device)
        kind, col, lvl = torch.cat([zero, kind]), torch.cat([zero, col]), torch.cat([zero, lvl])
    return kind, col, lvl


def kept_positions(mask, H, sep, user):
    """bool [B, S]: the kept positions, and key_mask [B] (0, or NEG for a history without an unmasked position)."""
    kind, col, _ = layout(mask.shape[1], H, sep, user, mask.device)
    keep = (kind == 0)[None, :] | (mask[:, col] != 0)
    empty = ~keep.any(1)
    keep[empty] = True
    return keep, torch.where(empty, NEG, 0.0).float()


def offsets(mask, H, sep, user):
    """int32 [B + 1] (history b owns packed rows offsets[b] .. offsets[b + 1] - 1) and key_mask fp32 [B]."""
    keep, key_mask = kept_positions(mask, H, sep, user)
    counts = keep.sum(1)
    return torch.cat([counts.new_zeros(1), counts.cumsum(0)]).to(torch.int32), key_mask


def assemble(mask, ids, user_ids, item_table, sep_row, user_table, K, H):
    """x [N, D] (the packed input rows), src int32 [N] (b * S + p) and slot int32 [B, S] (packed row or -1)."""
    B, n = mask.shape
    sep, user = sep_row is not None, user_table is not None
    kind, col, lvl = layout(n, H, sep, user, mask.device)
    keep, _ = kept_positions(mask, H, sep, user)
    S = kind.shape[0]
    flat = keep.reshape(-1).nonzero().squeeze(1)                       # row-major: history by history, in position order
    b, p = flat // S, flat % S
    rows = torch.empty((flat.shape[0], item_table.shape[1]), dtype=item_table.dtype, device=item_table.device)
    k = kind[p]
    c = col[p]
    item_id = (ids[b, c] + lvl[p] * K) * mask[b, c].long()
    rows[k == 1] = item_table[item_id[k == 1]]
    if sep:
        rows[k == 2] = sep_row.reshape(1, -1).to(rows.dtype)
    if user:
        rows[k == 0] = user_table[torch.remainder(user_ids[b[k == 0], 0], user_table.shape[0])]
    slot = torch.full((B * S,), -1, dtype=torch.int32, device=mask.device)
    slot[flat] = torch.arange(flat.shape[0], dtype=torch.int32, device=mask.device)
    return rows, flat.to(torch.int32), slot.reshape(B, S)


def rel_bias(bias):
    """[heads, 2S - 1] from HF's compute_bias(S, S)[0] ([heads, S, S]): entry t is the bias of key - query position t - (S - 1)."""
    return torch.cat([bias[:, 1:, 0].flip(1), bias[:, 0, :]], dim=1)


def attention(qkv, src, offs, key_mask, rel, S):
    """Self-attention among each history's packed rows: qkv [N, 3 inner] -> [N, inner]."""
    heads = rel.shape[0]
    inner = heads * DKV
    out = torch.empty((qkv.shape[0], inner), dtype=qkv.dtype, device=qkv.device)
    for b in range(offs.shape[0] - 1):
        lo, hi = int(offs[b]), int(offs[b + 1])
        if hi == lo:
            continue
        pos = src[lo:hi].long() - b * S
        q, k, v = (qkv[lo:hi, i * inner:(i + 1) * inner].reshape(hi - lo, heads, DKV).transpose(0, 1) for i in range(3))
        bias = rel[:, pos[None, :] - pos[:, None] + S - 1]                 # [heads, queries, keys]
        scores = q @ k.transpose(1, 2) + (bias + key_mask[b])           # no 1/sqrt(d) scaling; HF's order
        w = torch.softmax(scores.float(), dim=-1).to(scores.dtype)
        out[lo:hi] = (w @ v).transpose(0, 1).reshape(hi - lo, inner)
    return out


def scatter(rows, slot):
    """[B, S, D]: rows[slot], zeros where slot is -1."""
    B, S = slot.shape
    out = torch.zeros((B * S, rows.shape[1]), dtype=rows.dtype, device=rows.device)
    s = slot.reshape(-1).long()
    out[s >= 0] = rows[s[s >= 0]]
    return out.reshape(B, S, -1)


def encode(model, attention_mask, input_ids, user_id=None):
    """The packed encoder pass: (enc_out [B, S, d] with dropped rows 0, enc_mask [B, S]) like ``encoder_forward_pass``."""
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
    offs, key_mask = offsets(attention_mask, H, sep, user)
    x, src, slot = assemble(attention_mask, input_ids, user_id if user else None, model.item_sid_embedding_table.weight,
                            model.sep_token if sep else None, model.user_embedding.weight if user else None,
                            model.num_embeddings_per_hierarchy, H)
    S = slot.shape[1]
    blocks = [blk.layer for blk in enc.block]
    rel = rel_bias(blocks[0][0].SelfAttention.compute_bias(S, S)[0])
    x = x.clone()
    nrm = add_norm(x, None, blocks[0][0].layer_norm.weight, eps)
    for l, lay in enumerate(blocks):
        att = lay[0].SelfAttention
        a = attention(F.linear(nrm, torch.cat([att.q.weight, att.k.weight, att.v.weight])), src, offs, key_mask, rel, S)
        nrm = add_norm(x, F.linear(a, att.o.weight), lay[1].layer_norm.weight, eps)
        ff = lay[1].DenseReluDense
        nxt = blocks[l + 1][0].layer_norm.weight if l + 1 < len(blocks) else enc.final_layer_norm.weight
        nrm = add_norm(x, F.linear(F.relu(F.linear(nrm, ff.wi.weight)), ff.wo.weight), nxt, eps)
    return scatter(nrm, slot), enc_mask


def masks(kind, B, items, H, seed=0):
    """[B, items * H] attention masks of one kind: "full", "end" (end-padded like SeqData), "front" (front-padded), "holes"
    (random masked ids), "empty" (history 0 fully masked, the rest end-padded)."""
    g = torch.Generator().manual_seed(seed)
    mask = torch.ones((B, items * H), dtype=torch.long)
    lengths = torch.randint(1, items + 1, (B,), generator=g)
    for b in range(B):
        L = int(lengths[b])
        if kind == "end":
            mask[b, L * H:] = 0
        elif kind == "front":
            mask[b, :(items - L) * H] = 0
        elif kind == "holes":
            mask[b] = (torch.rand(items * H, generator=g) > 0.4).long()
        elif kind == "empty":
            mask[b, L * H:] = 0
    if kind == "empty":
        mask[0] = 0
    return mask
