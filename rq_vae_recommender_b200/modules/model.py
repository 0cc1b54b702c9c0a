"""modules/model.py of the reference: the T5 encoder-decoder generative-retrieval model, with its constrained beam search on
the semantic-id kernels.

Same names (``EncoderDecoderRetrievalModel``, ``ModelOutput``, ``GenerationOutput``, ``_strip_dedup_col``), constructor
signature and ``state_dict`` keys, so decoder checkpoints load with ``strict=True``.  ``forward`` and the encoder / decoder
passes are plain torch on HF T5 unless a call (or the ``DEFAULT_*`` switch it falls back to, which ``dropin.install`` sets)
picks a fused pass.  Shapes outside a kernel's limits raise ``Rqb200Error``; nothing falls back to the reference's code.

The search (``generate``, ``generate_items``):
  * ``_check_valid_prefix`` is a lookup in a trie of the corpus's id prefixes (``ops.SidPrefixIndex``), built on first use and
    rebuilt when the ``codebooks`` buffer is replaced, written to (``load_state_dict``) or moved;
  * ``search="sample"``: per level the head, the softmax, ``draw_exponential`` and ONE kernel that samples, checks the prefixes,
    scores and keeps the k best.  ``torch.multinomial(p, n)`` without replacement is ``topk(p / q, n)`` with
    ``q = draw_exponential(p)`` from the same generator, so under the same seed the samples, beams and log-probabilities are the
    reference's.  Nothing in the level loop waits for the device: rows ``torch.multinomial`` would reject are counted on the
    device and raise its error after the last level.  ``temperature`` / ``top_p`` (per call, per level) draw instead from
    softmax(logits / T) within a top-p nucleus, in the same kernel's warped mode (``SidPrefixIndex.sample_select_warped``);
  * ``search="beam"``: an exhaustive, deterministic beam search over every code (``SidPrefixIndex.beam_topk``), no sampling;
  * ``search="exact"``: the w valid corpus tuples of highest exact log-probability (``rank_sem_ids``' score, bit for bit): a beam
    search of width w bounds the w-th best score, and ``FusedT5Exact`` decodes only the trie nodes that reach the bound;
  * ``generate_items`` resolves the beams to corpus items with one more launch (``ops.SidItemTable.retrieve``); ``item_of``
    resolves ``sem_ids_fut`` to the true next item;
  * ``exclude_items`` / ``exclude_history`` leave given items (or each history's own) out of the search, the retrieval and
    ``rank_items``: a prefix under which every retrievable item is excluded is invalid for that history, like one the corpus
    lacks (``ops.sid_exclusion_build``);
  * ``include_items`` restricts the search and the retrieval to each history's allowed items: a prefix without an eligible item
    (allowed, retrievable, not excluded) under it is invalid for that history (``ops.sid_inclusion_build``).

The fused T5 passes, each HF's maths as GEMMs between this project's kernels, described once by ``_T5Weights``:
  * ``FusedT5Decode`` (``generate(decoder="fused")``) and ``FusedT5Rank`` (exact scoring) run the incremental decoder of
    ``_T5DecoderLevels``; ``FusedT5Encode`` (``generate(encoder="fused")``) runs the unpadded positions of each history only;
  * ``FusedT5EncodeTrain`` / ``FusedT5DecodeTrain`` (``forward(encoder="fused")`` / ``forward(decoder="fused")``) are the same
    passes with a backward and HF's dropout;
  * ``PackedEncoderOutput`` is the one layout of encoder rows that every offsets-based cross-attention reads.

``rank_items`` / ``rank_sem_ids`` are an evaluation tool with no search: every corpus item is scored by its exact
log-probability, one decoder row per corpus-trie node per history, and ranked.  ``score_items`` / ``score_sem_ids`` give the same
exact log-probability for items the caller chooses, decoding per history the trie of its own candidates with the same kernels.
"""
import functools
import math
from typing import List
from typing import NamedTuple
from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn
from torch import Tensor
from transformers import T5EncoderModel
from transformers.cache_utils import DynamicCache
from transformers.cache_utils import EncoderDecoderCache
from transformers.models.t5.modeling_t5 import T5Config
from transformers.models.t5.modeling_t5 import T5Stack

from .. import ops
from .._lib import Rqb200Error
from ..data.schemas import TokenizedSeqBatch

# The reference module sets this on import; the T5 passes of a script that imports this module instead run with TF32 as before.
torch.set_float32_matmul_precision("high")

MAX_CANDIDATES = 64
#: the widest beam generate(num_beams=...) takes (the cluster selection kernels keep at most 1024 beams per history)
MAX_NUM_BEAMS = 1024
#: the search generate() runs when it is not given one: "sample" (the reference's sampled beam search), "beam" (exhaustive) or
#: "exact" (the w most probable corpus tuples, no search error)
DEFAULT_SEARCH = "sample"
SEARCHES = ("sample", "beam", "exact")
#: the decoder passes generate() runs when it is not given a decoder: "hf" (transformers' T5Stack with its cache, as the
#: reference) or "fused" (FusedT5Decode: cross keys/values once per history, the decoder-step kernels of csrc/t5dec.cu)
DEFAULT_DECODER = "hf"
DECODERS = ("hf", "fused")
#: the encoder pass generate() runs when it is not given an encoder: "hf" (transformers' T5EncoderModel over every padded
#: position, as the reference) or "fused" (FusedT5Encode: the kept positions of each history only, the kernels of csrc/t5enc.cu)
DEFAULT_ENCODER = "hf"
ENCODERS = ("hf", "fused")
#: the encoder pass forward() (the training pass) runs when it is not given an encoder: "hf" (transformers' T5EncoderModel) or
#: "fused" (FusedT5EncodeTrain: the kept positions only, with the training kernels of csrc/t5enc.cu and HF's dropout)
DEFAULT_FORWARD_ENCODER = "hf"
#: the decoder pass forward() runs when it is not given a decoder: "hf" (transformers' T5Stack) or "fused" (FusedT5DecodeTrain:
#: the H positions the loss reads, with the training kernels of csrc/t5dec.cu and HF's dropout)
DEFAULT_FORWARD_DECODER = "hf"
#: the precision of the fused encoder's self-attention when a call gives none (read at call time): "fp32" (csrc/t5enc.cu, fp32 on
#: the CUDA cores) or "tf32" (csrc/t5enc_tc.cu: scores, P.V and the gradient products on TF32 tensor cores, softmax in fp32).  It
#: applies to encoder="fused" passes only; HF's encoder follows torch's matmul precision.
DEFAULT_ENCODER_ATTENTION = "fp32"
ENCODER_ATTENTIONS = ("fp32", "tf32")
#: whether generate_next_sem_id, generate_items and rank_items leave out the items of each history (``exclude_history``) when a
#: call does not say (read at call time)
DEFAULT_EXCLUDE_HISTORY = False
_MULTINOMIAL_ERRORS = ("probability tensor contains either `inf`, `nan` or element < 0",
                       "invalid multinomial distribution (sum of probabilities <= 0)")


class ModelOutput(NamedTuple):
    loss: Tensor
    logits: Tensor
    loss_d: Tensor


class GenerationOutput(NamedTuple):
    sem_ids: Tensor
    log_probas: Tensor


class ItemGenerationOutput(NamedTuple):
    """generate_items: the corpus items of the beams (item_ids [B, n] int64 and the source beam of each, beams [B, n] int32,
    both -1 past count [B] int32), and generate's own beams (sem_ids [B, top_k, H], log_probas [B, top_k])."""
    item_ids: Tensor
    beams: Tensor
    count: Tensor
    sem_ids: Tensor
    log_probas: Tensor


def draw_exponential(probas: Tensor) -> Tensor:
    """The Exp(1) draw ``torch.multinomial(probas, n)`` (without replacement) makes from the default generator: sampling is
    then ``topk(probas / draw, n)``.  Patch this function to inject noise."""
    return torch.empty_like(probas).exponential_(1)


def dropout_rows(x: Tensor, p: float) -> Tensor:
    """HF's nn.Dropout at the token-wise sites of the fused training encoder (embedding, attention output, feed-forward inner
    and output, final output), drawn from torch's generator.  Patch this function to inject masks."""
    return F.dropout(x, p, training=True) if p > 0 else x


def _strip_dedup_col(tensor: Tensor, sem_ids_dim: int, n_layers: int) -> Tensor:
    """[B, N * sem_ids_dim] token rows (each item: n_layers ids + the tokenizer's dedup column) -> [B, N * n_layers]."""
    B, width = tensor.shape
    items = width // sem_ids_dim
    return tensor.view(B, items, sem_ids_dim)[:, :, :n_layers].contiguous().view(B, items * n_layers)



def _choice(value: Optional[str], default: Optional[str], allowed, what: str, name: str) -> str:
    """An option string of one call: ``value``, else ``default``; ``ValueError`` when it is not one of ``allowed``."""
    value = default if value is None else value
    if value not in allowed:
        raise ValueError(f"{what}: {name} must be one of {allowed}, got {value!r}")
    return value


def _check_no_autocast(what: str) -> None:
    if torch.is_autocast_enabled("cuda"):
        raise ValueError(f"{what} runs fp32 kernels: it cannot run inside an autocast region")


class _T5Weights:
    """One T5 stack (``model.t5_decoder`` or ``model.encoder.encoder``) as the fused passes read it: ``blocks`` (each block's
    sub-layers), ``norms`` (every sub-layer's T5LayerNorm weight in pass order, then the final norm's), ``heads``, ``eps`` and
    ``inner`` = heads * d_kv.  The kernels are built for d_kv = 64 and a relu feed-forward: any other config raises."""

    def __init__(self, stack, what: str):
        cfg = stack.config
        if cfg.d_kv != ops.T5_DKV or cfg.is_gated_act or cfg.dense_act_fn != "relu":
            raise Rqb200Error(f"{what} needs d_kv = {ops.T5_DKV} and a relu feed-forward (d_kv = {cfg.d_kv}, "
                              f"feed_forward_proj = {cfg.feed_forward_proj!r})")
        self.stack = stack
        self.blocks = [blk.layer for blk in stack.block]
        self.norms = [sub.layer_norm.weight for lay in self.blocks for sub in lay] + [stack.final_layer_norm.weight]
        self.heads, self.eps, self.inner = cfg.num_heads, cfg.layer_norm_epsilon, cfg.num_heads * ops.T5_DKV

    def qkv(self, l: int) -> Tensor:
        """Layer l's q | k | v self-attention weight, concatenated here: a training pass calls this per step, so autograd reaches
        the three parameters."""
        att = self.blocks[l][0].SelfAttention
        return torch.cat([att.q.weight, att.k.weight, att.v.weight])

    def layer(self, l: int) -> tuple:
        """Layer l's GEMM weights in pass order: q|k|v, self-attention o, (decoders: cross-attention q, o), wi, wo."""
        lay = self.blocks[l]
        cross = (lay[1].EncDecAttention.q.weight, lay[1].EncDecAttention.o.weight) if len(lay) == 3 else ()
        ff = lay[-1].DenseReluDense
        return (self.qkv(l), lay[0].SelfAttention.o.weight, *cross, ff.wi.weight, ff.wo.weight)


def _linear(x: Tensor, w: Tensor, relu: bool = False) -> Tensor:
    """x w^T on cuBLAS, the feed-forward's relu in place."""
    y = F.linear(x, w)
    return y.relu_() if relu else y


class _T5DecoderLevels:
    """The incremental T5 decoder (eval mode, no 1/sqrt(d), block 0's relative bias) that ``FusedT5Decode`` and ``FusedT5Rank``
    share: one query position per call of ``level``, between the decoder-step kernels of csrc/t5dec.cu.  The two differ in the
    GEMM (``linear(x, w, relu=False)`` over weights wrapped by ``operand``) and in the cross-attention kernel, and in nothing
    else.  Cross keys and values are projected here ONCE from the encoder ``rows``, for every layer in one GEMM: ``cross_kv``
    [rows, layers * 2 * inner], layer l's keys at columns 2 l inner, its values at (2 l + 1) inner."""

    def __init__(self, model: "EncoderDecoderRetrievalModel", what: str, rows: Tensor, linear, operand=lambda w: w):
        self.model, self.H, self.linear = model, model.num_hierarchies, linear
        self.t5 = t5 = _T5Weights(model.t5_decoder, what)
        self.w = [tuple(operand(w) for w in t5.layer(l)) for l in range(len(t5.blocks))]
        w_kv = torch.cat([w for lay in t5.blocks for w in (lay[1].EncDecAttention.k.weight, lay[1].EncDecAttention.v.weight)])
        self.cross_kv = linear(rows, operand(w_kv))
        self.bias = t5.blocks[0][0].SelfAttention.compute_bias(self.H, self.H)[0].contiguous()

    def level(self, h: int, R: int, ids: Optional[Tensor], parent: Optional[Tensor], cache: Tensor, anc: List[Tensor],
              cross, live: Optional[Tensor] = None) -> Tensor:
        """The final-layer-normed hidden state [R, d_model] of query position h for R rows.  ids [R] are the rows' last codes
        (None at h = 0: BOS).  Self-attention keys/values of position j live in slot j of ``cache`` [layers, 2, H, >= R, inner];
        a row reads its past through the int32 ancestor table anc[0] [>= R, H], which this call advances from ``parent`` [R]
        (each row's row at level h - 1) into anc[1] and then swaps the pair, so no level copies the cache.
        ``cross(q, k, v)`` is the cross-attention of the R queries over one layer's keys and values.  ``live`` (int32 on the
        device; ``ops.gemm_split`` levels only): R is a capacity and every launch runs the first live[0] rows."""
        m, linear, eps, norms, inner = self.model, self.linear, self.t5.eps, self.t5.norms, self.t5.inner
        if live is not None:
            linear = functools.partial(linear, live=live)
        x = torch.empty((R, m.bos_token.shape[1]), dtype=torch.float32, device=self.cross_kv.device)
        nrm = torch.empty_like(x)
        if ids is None:
            ops.t5dec_add_norm(x, None, norms[0], nrm, eps, emb=m.bos_token, live=live)
        else:
            ops.t5dec_add_norm(x, None, norms[0], nrm, eps, emb=m.item_sid_embedding_table.weight, ids=ids,
                               offset=(h - 1) * m.num_embeddings_per_hierarchy, live=live)
        for l, (w_qkv, w_o, w_q, w_xo, w_i, w_fo) in enumerate(self.w):
            advance = h > 0 and l == 0
            a = ops.t5dec_self_attention(linear(nrm, w_qkv), cache[l, 0], cache[l, 1], self.bias, h, anc[0],
                                         parent if advance else None, anc[1] if advance else None, live=live)
            if advance:
                anc.reverse()
            ops.t5dec_add_norm(x, linear(a, w_o), norms[3 * l + 1], nrm, eps, live=live)
            kv = self.cross_kv[:, 2 * l * inner:(2 * l + 2) * inner]
            a = cross(linear(nrm, w_q), kv[:, :inner], kv[:, inner:])
            ops.t5dec_add_norm(x, linear(a, w_xo), norms[3 * l + 2], nrm, eps, live=live)
            ops.t5dec_add_norm(x, linear(linear(nrm, w_i, relu=True), w_fo), norms[3 * l + 3], nrm, eps, live=live)
        return nrm


class FusedT5Decode(_T5DecoderLevels):
    """The decoder passes of one ``generate(decoder="fused")`` call: HF's T5Stack (eval mode, relu FFN, d_kv 64) restated as
    cuBLAS GEMMs (``F.linear``) between the decoder-step kernels, with the key/value state laid out so that no level copies it:
      * cross-attention keys/values are projected once from the encoder output of the B histories (``cross_kv`` [B * S, ...]),
        and each history's are read once per level for all of its beams (``t5dec_cross_attention``);
      * ``cache`` [layers, 2, H, B * k, inner] and the ancestor tables live across the levels; ``step`` advances the tables from
        the search's parent_global (no reorder copy);
      * level 1 reuses level 0's BOS keys/values: the BOS position depends only on the history.
    ``step(h, generated, parent)`` returns the final-layer-normed hidden state [rows, d_model] of query position h."""

    def __init__(self, model: "EncoderDecoderRetrievalModel", enc_out: Tensor, enc_mask: Tensor, k: int):
        B, S, d = enc_out.shape
        super().__init__(model, "decoder=\"fused\"", enc_out.reshape(B * S, d), _linear)
        self.k, self.B, self.S, self.inner = k, B, S, self.t5.inner
        self.mask = enc_mask.to(torch.float32).contiguous()
        self.cache = torch.empty((len(self.w), 2, self.H, B * k, self.inner), dtype=torch.float32, device=enc_out.device)
        self.anc = [torch.empty((B * k, self.H), dtype=torch.int32, device=enc_out.device) for _ in range(2)]

    def step(self, h: int, generated: Optional[Tensor], parent: Optional[Tensor]) -> Tensor:
        nq = 1 if h == 0 else self.k
        R = self.B * nq
        return self.level(h, R, None if h == 0 else generated.reshape(R, h)[:, h - 1], parent, self.cache, self.anc,
                          lambda q, k, v: ops.t5dec_cross_attention(q, k, v, self.mask, nq, self.t5.heads))

class ItemRankingOutput(NamedTuple):
    """rank_items: the n best corpus items of each history by exact log-probability (item_ids [B, n] int64, -1 past the corpus),
    their log-probabilities (scores [B, n] fp32, -inf past the corpus), the true next item's 0-based rank among every retrievable
    item (target_rank [B] int64, -1 when it is not retrievable) and the number of retrievable items ranked (num_items)."""
    item_ids: Tensor
    scores: Tensor
    target_rank: Tensor
    num_items: int


class ItemScoreOutput(NamedTuple):
    """score_items: the exact log-probability of each given item (scores [B, C] fp32, -inf for padding and for items whose
    tuple holds an id outside [0, K)) and the 0-based position of the true next item among the row's items in rank_items' order
    (target_rank [B] int64, -1 when it is not among them)."""
    scores: Tensor
    target_rank: Tensor


#: device bytes one chunk of histories of rank_sem_ids / rank_items / score_sem_ids is sized to when max_rows is not given
RANK_BYTE_BUDGET = 4 << 30
#: most items rank_items returns per history
MAX_RANK_ITEMS = 1024


class FusedT5Rank(_T5DecoderLevels):
    """The decoder passes of ``rank_sem_ids``: one decoder row per node of the corpus trie per history.  Items that share an
    l-prefix share the causal decoder's state at positions 0..l, so level h's rows (one per h-prefix node; the root at h = 0) give
    every child's log-probability, and a leaf's score is the sum along its path.  The maths are ``FusedT5Decode``'s, with
      * node rows' ids and parents taken from the trie, and cache slots sized to the largest level of the chunk;
      * every GEMM on the split-precision tensor-core GEMM (``ops.gemm_split``: fp32-accurate, each output row a function of its
        input row alone), so the chunking of histories does not change a bit; the weights' split images are built once per call;
      * ``t5rank_cross_attention`` for the level's n_h queries per history over the encoder rows given by offsets and an additive
        per-row key mask, fp32 on the CUDA cores or (``attention="tf32"``) its products on the TF32 tensor cores;
      * after each level's head, ``t5rank_children`` (log-sum-exp as the beam search, child score = parent + log-probability)."""

    def __init__(self, model: "EncoderDecoderRetrievalModel", rows: Tensor, offsets: Tensor, key_mask: Tensor,
                 attention: str = "fp32"):
        super().__init__(model, "rank_sem_ids", rows, ops.gemm_split, ops.SplitOperand)
        self.tf32 = _choice(attention, None, ENCODER_ATTENTIONS, "FusedT5Rank", "attention") == "tf32"
        self.heads_w = [ops.SplitOperand(mlp.weight) for mlp in model.decoder_mlp]
        self.offsets, self.key_mask = offsets, key_mask

    @staticmethod
    def row_bytes(model: "EncoderDecoderRetrievalModel") -> int:
        """Device bytes one node row of the widest level holds while a chunk runs: its self-attention cache (layers x k, v x H
        slots x inner fp32), the activations of one layer (x, norm, qkv, attention, projection, feed-forward, head logits) and
        its ids, parent and ancestor entries."""
        cfg = model.t5_decoder.config
        inner, d, H = cfg.num_heads * ops.T5_DKV, cfg.d_model, model.num_hierarchies
        floats = cfg.num_layers * 2 * H * inner + 3 * d + 5 * inner + cfg.d_ff + model.num_embeddings_per_hierarchy + 1
        return 4 * floats + 16 + 8 * H

    def run(self, b0: int, b1: int, levels: ops.SidTrieLevels, out: Tensor, bad: Tensor) -> None:
        """Leaf scores of histories b0 .. b1 - 1 over the corpus trie into out[b0:b1] ([B, U]): every history decodes every node."""
        H, Bc, dev = self.H, b1 - b0, self.cross_kv.device
        first = torch.arange(Bc, device=dev)[:, None]
        ids = [None] + [levels.code[h].long().repeat(Bc) for h in range(1, H)]
        parent = [None] + [(first * levels.n[h - 1] + levels.parent[h].long()[None, :]).reshape(-1) for h in range(1, H)]
        nxt = [torch.empty((Bc, levels.n[h + 1]), dtype=torch.float32, device=dev) for h in range(H - 1)] + [out[b0:b1]]
        self.decode(b0, b1, levels.n[:H], ids, parent, levels.child[:H], levels.code[1:H + 1], nxt, bad)

    def run_candidates(self, b0: int, b1: int, n: List[int], trie: ops.CandidateTrie, out: Tensor, bad: Tensor) -> None:
        """Candidate scores of histories b0 .. b1 - 1 over their own tries (``ops.t5score_trie_build``) into out[b0:b1] ([B, C];
        -inf for a candidate holding an id outside [0, K)).  Level h is padded to n[h] rows per history, the chunk's largest
        count (at least 1).  A padding row decodes code 0 under its history's row 0 of the level above, so its values are finite;
        it has no children, except that the last row of a history owns the padding slots of the level below it, which keeps the
        chunk's child ranges one ascending array.  No padding score is read."""
        H, Bc, dev = self.H, b1 - b0, self.cross_kv.device
        first = torch.arange(Bc, device=dev)[:, None]
        ids = [None] + [trie.code[b0:b1, h - 1, :n[h]].reshape(-1).long() for h in range(1, H)]
        parent = [None] + [(first * n[h - 1] + trie.parent[b0:b1, h - 1, :n[h]]).reshape(-1) for h in range(1, H)]
        # the chunk as one group of Bc * n[h] rows: child ranges offset to the chunk's slots of level h + 1
        child = [torch.cat([(first * n[h + 1] + trie.child[b0:b1, h, :n[h]]).reshape(-1),
                            torch.full((1,), Bc * n[h + 1], dtype=torch.int64, device=dev)]).to(torch.int32) for h in range(H)]
        code = [trie.code[b0:b1, h, :n[h + 1]].reshape(-1).contiguous() for h in range(H)]
        nxt = [torch.empty((1, Bc * n[h + 1]), dtype=torch.float32, device=dev) for h in range(H)]
        self.decode(b0, b1, n[:H], ids, parent, child, code, nxt, bad)
        leaf = trie.leaf[b0:b1].long()
        out[b0:b1] = torch.where(leaf >= 0, nxt[H - 1].view(-1)[first * n[H] + leaf.clamp(min=0)], float("-inf"))

    def decode(self, b0: int, b1: int, n: List[int], ids: List[Optional[Tensor]], parent: List[Optional[Tensor]],
               child: List[Tensor], code: List[Tensor], nxt: List[Tensor], bad: Tensor) -> None:
        """The level loop of histories b0 .. b1 - 1 over given trie levels.  Level h runs n[h] decoder rows per history (row
        b * n[h] + i; n[0] = 1, BOS); for h >= 1 ids[h] / parent[h] (int64 [Bc * n[h]]) are each row's last code and its row in
        level h - 1.  After the level's head, ``t5rank_children`` writes the children's scores to nxt[h] ([G, n_next]: the level's
        rows as G equal groups, child[h] int32 the child ranges of one group's rows, code[h] int32 [n_next] the children's last
        codes, nxt[h - 1] the rows' own scores)."""
        Bc, dev = b1 - b0, self.cross_kv.device
        rows = Bc * max(n)
        cache = torch.empty((len(self.w), 2, self.H, rows, self.t5.inner), dtype=torch.float32, device=dev)
        anc = [torch.zeros((rows, self.H), dtype=torch.int32, device=dev)]
        anc.append(torch.empty_like(anc[0]))
        offsets = self.offsets[b0:b1 + 1]
        score = None
        for h in range(self.H):
            n_h = n[h]
            R = Bc * n_h
            nrm = self.level(h, R, ids[h], parent[h], cache, anc,
                             lambda q, k, v: ops.t5rank_cross_attention(q, k, v, offsets, self.key_mask, n_h, self.t5.heads,
                                                                        tf32=self.tf32))
            ops.t5rank_children(ops.gemm_split(nrm, self.heads_w[h]), score, child[h], code[h], R // nxt[h].shape[0], nxt[h], bad)
            score = nxt[h]


#: decoder rows the pruned decode of the last generate(search="exact") call ran, summed over its chunks (neither the bound's beam
#: search and rescoring nor a level abandoned for a smaller chunk counts); observation only
EXACT_DECODER_ROWS = 0


def _read_frontier(offsets: Tensor, counts: Tensor) -> List[int]:
    """The totals of the next level of one chunk of generate(search="exact"): its decoder rows, their children, their query tiles
    and the most children of one history, read on the host to size the level: one read per level per chunk."""
    return torch.cat([offsets[:, -1], counts[1].max().view(1)]).tolist()


def _grow_rows(t: Tensor, dim: int, rows: int) -> Tensor:
    """t with dimension ``dim`` enlarged to ``rows``, the existing entries copied."""
    shape = list(t.shape)
    shape[dim] = rows
    out = t.new_empty(shape)
    out.narrow(dim, 0, t.shape[dim]).copy_(t)
    return out


class FusedT5Exact(FusedT5Rank):
    """The pruned exact decode of ``generate(search="exact")``: ``FusedT5Rank``'s maths over the corpus trie, decoding per history
    only the nodes whose exact score is at least tau[b], a score some valid leaf of the history reaches.  A child never scores
    above its parent (``t5rank_children`` adds a log-probability <= 0), so no pruned node has a descendant in the history's
    exact top w, and the nodes kept get ``rank_sem_ids``' bits: every GEMM is row-wise, and the ragged cross-attention gives a
    query the uniform kernel's arithmetic.  Per level, after the head and ``t5rank_children``:
      * ``t5exact_frontier_count`` counts each history's kept children (score >= tau[b], allowed by the filter), a scan gives the
        offsets, ``_read_frontier`` reads the totals on the host, and ``t5exact_frontier_write`` lays out the next level's rows --
        ragged, history b's contiguous with no padding -- their query tiles, and their children as one group;
      * the level's rows run ``_T5DecoderLevels.level`` with ``t5rank_cross_attention_ragged``; level 0 is each history's BOS row.
    ``t5exact_select`` then takes each history's w best leaves among the last level's children."""

    def run(self, b0: int, b1: int, levels: ops.SidTrieLevels, tau: Tensor, w: int, leaf_key: Tensor, filt: dict, max_rows: int,
            gen: Tensor, lp: Tensor, bad: Tensor) -> Optional[int]:
        """The w best leaves of histories b0 .. b1 - 1 into gen [b1 - b0, w, H] / lp [b1 - b0, w]; returns the decoder rows run,
        or None (nothing written) when a level of two or more histories would exceed ``max_rows`` rows."""
        H, Bc, dev = self.H, b1 - b0, self.cross_kv.device
        K = self.model.num_embeddings_per_hierarchy
        offsets, tau_c, heads = self.offsets[b0:b1 + 1], tau[b0:b1], self.t5.heads
        cap = Bc                                             # cache and ancestor rows, grown with the levels
        cache = torch.empty((len(self.w), 2, H, cap, self.t5.inner), dtype=torch.float32, device=dev)
        anc = [torch.zeros((cap, H), dtype=torch.int32, device=dev), torch.empty((cap, H), dtype=torch.int32, device=dev)]
        nrm = self.level(0, Bc, None, None, cache, anc,
                         lambda q, k, v: ops.t5rank_cross_attention(q, k, v, offsets, self.key_mask, 1, heads))
        first = torch.empty((Bc, levels.n[1]), dtype=torch.float32, device=dev)
        ops.t5rank_children(ops.gemm_split(nrm, self.heads_w[0]), None, levels.child[0], levels.code[1], 1, first, bad)
        children, max_u, rows = ops.ExactChildren(first.view(-1), levels.n[1]), levels.n[1], Bc
        for l in range(1, H):
            counts = ops.t5exact_frontier_count(children, levels.code[1], tau_c, K, l, levels.child[l], b0, **filt)
            scan = torch.zeros((3, Bc + 1), dtype=torch.int32, device=dev)
            scan[:, 1:] = counts.cumsum(1)
            R, C, T, max_u = _read_frontier(scan, counts)
            if R > max_rows and Bc > 1:
                return None
            if R == 0:                                       # every history's frontier is empty: no valid leaf reaches tau
                gen.fill_(-1)
                lp.fill_(float("-inf"))
                return rows
            nxt = ops.t5exact_frontier_write(children, levels.code[1], tau_c, K, l, levels.child[l], levels.code[l + 1], scan,
                                             (R, C, T), b0, **filt)
            if R > cap:
                cap = min(max(R, 2 * cap), max(R, max_rows))
                cache = _grow_rows(cache, 3, cap)
                anc = [_grow_rows(anc[0], 0, cap), torch.empty((cap, H), dtype=torch.int32, device=dev)]
            nrm = self.level(l, R, nxt.code, nxt.parent, cache, anc,
                             lambda q, k, v: ops.t5rank_cross_attention_ragged(q, k, v, offsets, self.key_mask, nxt.tiles, heads))
            ops.t5rank_children(ops.gemm_split(nrm, self.heads_w[l]), nxt.score, nxt.child, nxt.children.code, R,
                                nxt.children.scores.view(1, -1), bad)
            children, rows = nxt.children, rows + R
        ops.t5exact_select(children, max_u, levels, H, leaf_key, w, gen, lp, b0, **filt)
        return rows

    @staticmethod
    def capacities(n: List[int], B: int, K: int, max_rows: int) -> List[tuple]:
        """(rows, children, tiles) capacities of pruned levels l = 1 .. H - 1 of a ``run_capacity`` of B histories over trie levels
        of n[l] nodes: R_l = min(B n[l], max_rows), C_l = min(B n[l + 1], K R_l), T_l = ceil(R_l / 64) + B."""
        caps = []
        for l in range(1, len(n) - 1):
            R = min(B * n[l], max_rows)
            caps.append((R, min(B * n[l + 1], K * R), -(-R // 64) + B))
        return caps

    def run_capacity(self, levels: ops.SidTrieLevels, tau: Tensor, w: int, leaf_key: Tensor, filt: dict, max_rows: int,
                     gen: Tensor, lp: Tensor, bad: Tensor, overflow: Tensor) -> Tensor:
        """``run`` of the whole batch at fixed capacities (``capacities``), reading nothing on the host, for a CUDA-graph capture:
        the cache, the ancestor tables and every level's buffers are sized once, and each pruned level's launches read its live
        counts from the device (``ops.t5exact_frontier_capacity`` and the ``live`` launches).  The rows kept get ``run``'s bits.
        A level whose frontier exceeds a capacity sets overflow[0] = 1 and leaves every later level empty, so gen / lp are then
        not the search's result.  Returns the decoder rows run (int32 [1], on the device)."""
        H, B, dev = self.H, tau.shape[0], self.cross_kv.device
        K = self.model.num_embeddings_per_hierarchy
        offsets, heads = self.offsets, self.t5.heads
        caps = self.capacities(levels.n[:H + 1], B, K, max_rows)
        cap = max([B] + [c[0] for c in caps])
        cache = torch.empty((len(self.w), 2, H, cap, self.t5.inner), dtype=torch.float32, device=dev)
        anc = [torch.zeros((cap, H), dtype=torch.int32, device=dev), torch.empty((cap, H), dtype=torch.int32, device=dev)]
        nrm = self.level(0, B, None, None, cache, anc,
                         lambda q, k, v: ops.t5rank_cross_attention(q, k, v, offsets, self.key_mask, 1, heads))
        first = torch.empty((B, levels.n[1]), dtype=torch.float32, device=dev)
        ops.t5rank_children(ops.gemm_split(nrm, self.heads_w[0]), None, levels.child[0], levels.code[1], 1, first, bad)
        children, max_u = ops.ExactChildren(first.view(-1), levels.n[1]), levels.n[1]
        rows = torch.full((1,), B, dtype=torch.int32, device=dev)
        for l in range(1, H):
            R, C, T = caps[l - 1]
            counts = ops.t5exact_frontier_count(children, levels.code[1], tau, K, l, levels.child[l], 0, **filt)
            scan = torch.zeros((3, B + 1), dtype=torch.int32, device=dev)
            scan[:, 1:] = counts.cumsum(1)
            nxt, live = ops.t5exact_frontier_capacity(children, levels.code[1], tau, K, l, levels.child[l], levels.code[l + 1], scan,
                                                      (R, C, T), overflow, 0, **filt)
            nrm = self.level(l, R, nxt.code, nxt.parent, cache, anc,
                             lambda q, k, v: ops.t5rank_cross_attention_ragged(q, k, v, offsets, self.key_mask, nxt.tiles, heads,
                                                                               live=live[2:]), live=live)
            ops.t5rank_children(ops.gemm_split(nrm, self.heads_w[l], live=live), nxt.score, nxt.child, nxt.children.code, R,
                                nxt.children.scores.view(1, -1), bad, live=live)
            children, max_u = nxt.children, min(levels.n[H], C)
            rows += live[:1]
        ops.t5exact_select(children, max_u, levels, H, leaf_key, w, gen, lp, 0, **filt)
        return rows


def _encoder_attention(encoder: str, encoder_attention: Optional[str], what: str) -> str:
    """The fused encoder's attention precision of one call: ``encoder_attention``, else ``DEFAULT_ENCODER_ATTENTION``.  An explicit
    "tf32" with encoder="hf" raises: HF's attention runs at torch's matmul precision, and the switch would be ignored."""
    att = _choice(encoder_attention, DEFAULT_ENCODER_ATTENTION, ENCODER_ATTENTIONS, what, "encoder_attention")
    if encoder_attention == "tf32" and encoder != "fused":
        raise ValueError(f"{what}: encoder_attention=\"tf32\" selects the fused encoder's attention kernels; with "
                         f"encoder={encoder!r} the attention follows torch.get_float32_matmul_precision()")
    return att


def _read_n_kept(offsets: Tensor) -> int:
    """The packed row count offsets[B], read on the host to size the encoder's GEMMs: the one host synchronisation of an
    encoder="fused" pass."""
    return int(offsets[-1])


def _read_node_counts(counts: Tensor) -> List[List[int]]:
    """The candidate tries' node counts [B, H], read on the host to size the padded levels and the chunks: the first of the two
    host reads of score_sem_ids / score_items."""
    return counts.tolist()


class PackedEncoderOutput(NamedTuple):
    """An encoder pass as rows: rows [N, d_model] (history b's are rows offsets[b] .. offsets[b + 1] - 1, in position order),
    offsets int32 [B + 1], S encoder positions per history and enc_mask [B, S], the mask ``encoder_forward_pass`` returns.
    ``packed`` of the fused encoders keeps only some positions and adds key_mask fp32 [B] (finfo(float32).min for a history
    without an unmasked position), src int32 [N] (b * S + position of each row) and slot int32 [B, S] (row of each position or
    -1); ``of_padded`` (every position a row) leaves the three None."""
    rows: Tensor
    offsets: Tensor
    key_mask: Optional[Tensor]
    src: Optional[Tensor]
    slot: Optional[Tensor]
    S: int
    enc_mask: Tensor

    @classmethod
    def of_padded(cls, enc_out: Tensor, enc_mask: Tensor) -> "PackedEncoderOutput":
        """HF's encoder output [B, S, d_model] and its mask [B, S]: history b's rows are b * S .. b * S + S - 1."""
        B, S, d = enc_out.shape
        offsets = torch.arange(0, (B + 1) * S, S, dtype=torch.int32, device=enc_out.device)
        return cls(enc_out.reshape(B * S, d), offsets, None, None, None, S, enc_mask)

    def keys(self):
        """(rows, offsets, additive key mask fp32 [N], src, S): what the offsets-based cross-attentions take.  A padded layout
        masks the rows whose enc_mask is 0; a packed one holds kept positions only, so a row takes its history's key_mask."""
        if self.src is None:
            key_mask = torch.where(self.enc_mask == 0, torch.finfo(torch.float32).min, 0.0).to(torch.float32).reshape(-1)
        else:
            key_mask = self.key_mask.index_select(0, torch.div(self.src, self.S, rounding_mode="floor").long())
        return self.rows, self.offsets, key_mask, self.src, self.S


def _encoder_mask(model: "EncoderDecoderRetrievalModel", attention_mask: Tensor, user: bool) -> Tensor:
    """``encoder_forward_pass``'s mask [B, S] of the ids' mask [B, n]: each item's separator takes the mask of the item's last
    id, and the user column is ones."""
    B, n = attention_mask.shape
    H = model.num_hierarchies
    enc_mask = attention_mask
    if model.sep_token is not None:
        items = enc_mask.view(B, n // H, H)
        enc_mask = torch.cat([items, items[:, :, -1:]], dim=2).reshape(B, n // H * (H + 1))
    if user:
        enc_mask = torch.cat([torch.ones(B, 1, device=enc_mask.device), enc_mask], dim=1)
    return enc_mask


class FusedT5Encode:
    """The encoder pass of ``generate(encoder="fused")``: ``encoder_forward_pass`` (HF's T5EncoderModel in eval mode, relu FFN,
    d_kv 64) restated over the KEPT positions of each history only, as cuBLAS GEMMs (``F.linear``) between the kernels of
    csrc/t5enc.cu and the decoder's ``t5dec_add_norm``:
      * a position is kept when its mask is nonzero (the user row always is); a history with no unmasked position keeps all of
        them, so HF's uniform average over its positions is reproduced.  Everywhere else a dropped position changes nothing:
        HF's softmax gives a masked key the weight 0, and both decoders mask it again;
      * kept rows are packed history by history; the GEMMs run on the packed [N, d_model] rows and self-attention adds HF's
        relative-position bias at each row's ORIGINAL position (``compute_bias(S, S)`` of block 0, once per call);
      * ``__call__`` returns what ``encoder_forward_pass`` returns: enc_out [B, S, d_model] with the rows of dropped positions
        set to 0, and enc_mask [B, S] with the same values.
    N is read on the host once per call (``_read_n_kept``) to size the GEMMs; it is the pass's only host synchronisation, and
    ``n_kept`` keeps the last call's.  ``attention`` picks the self-attention kernel: "fp32" (``ops.t5enc_attention``) or "tf32"
    (``ops.t5enc_attention_tc``).
    ``capacity=True`` reads nothing on the host, for a CUDA-graph capture: the packed rows are B * S, rows N .. B * S - 1 zero
    (``ops.t5enc_assemble_capacity``, and one zero-filled attention output that the attention kernels never write past N), so
    the GEMMs run B * S rows and rows 0 .. N - 1 differ from the eager pass only by the GEMMs' rounding at another row count."""

    def __init__(self, model: "EncoderDecoderRetrievalModel", attention: str = "fp32", capacity: bool = False):
        self.model = model
        self.t5 = _T5Weights(model.encoder.encoder, "encoder=\"fused\"")
        tf32 = _choice(attention, None, ENCODER_ATTENTIONS, "FusedT5Encode", "attention") == "tf32"
        self.attention = ops.t5enc_attention_tc if tf32 else ops.t5enc_attention
        self.w = [self.t5.layer(l) for l in range(len(self.t5.blocks))]
        self.capacity = capacity
        self.n_kept = None

    def __call__(self, attention_mask: Tensor, input_ids: Tensor, user_id: Optional[Tensor] = None):
        out = self.packed(attention_mask, input_ids, user_id)
        return ops.t5enc_scatter(out.rows, out.slot), out.enc_mask

    def packed(self, attention_mask: Tensor, input_ids: Tensor, user_id: Optional[Tensor] = None) -> PackedEncoderOutput:
        """The pass without the scatter: the kept rows [N, d_model] and their layout."""
        m, eps, norms = self.model, self.t5.eps, self.t5.norms
        H = m.num_hierarchies
        sep = m.sep_token is not None
        user = user_id is not None and m.user_embedding is not None
        enc_mask = _encoder_mask(m, attention_mask, user)
        offsets, key_mask = ops.t5enc_offsets(attention_mask, H, sep, user)
        inputs = (attention_mask, input_ids, user_id if user else None, m.item_sid_embedding_table.weight,
                  m.sep_token if sep else None, m.user_embedding.weight if user else None, m.num_embeddings_per_hierarchy, H, offsets)
        a_out = None
        if self.capacity:
            x, nrm, src, slot = ops.t5enc_assemble_capacity(*inputs, norms[0], eps)
            a_out = x.new_zeros((x.shape[0], self.t5.inner))
        else:
            self.n_kept = _read_n_kept(offsets)
            x, nrm, src, slot = ops.t5enc_assemble(*inputs, self.n_kept, norms[0], eps)
        S = slot.shape[1]
        rel = ops.t5enc_rel_bias(self.t5.blocks[0][0].SelfAttention.compute_bias(S, S)[0])
        for l, (w_qkv, w_o, w_i, w_fo) in enumerate(self.w):
            a = self.attention(F.linear(nrm, w_qkv), src, offsets, key_mask, rel, S, a_out)
            ops.t5dec_add_norm(x, F.linear(a, w_o), norms[2 * l + 1], nrm, eps)
            ops.t5dec_add_norm(x, F.linear(_linear(nrm, w_i, relu=True), w_fo), norms[2 * l + 2], nrm, eps)
        return PackedEncoderOutput(nrm, offsets, key_mask, src, slot, S, enc_mask)

def _encoder_layout(n: int, H: int, sep: bool, user: bool, device) -> Tensor:
    """[3, S] per encoder position: kind (0 user row, 1 item id, 2 separator), the column of the [B, n] inputs it reads and the id's
    level -- the layout encoder_forward_pass builds."""
    W = H + int(sep)
    q = torch.arange(n // H * W, device=device)
    item, j = q // W, q % W
    kind = torch.where(j < H, 1, 2)
    col = item * H + torch.clamp(j, max=H - 1)
    lvl = torch.where(j < H, j, 0)
    out = torch.stack([kind, col, lvl])
    if user:
        out = torch.cat([torch.zeros((3, 1), dtype=out.dtype, device=device), out], dim=1)
    return out


class _AssembleFunction(torch.autograd.Function):
    """The packed input rows x [N, D] of ``ops.t5enc_assemble``, with the backward of the gather: each packed row's gradient is
    added (``index_put_`` with accumulate, a sorted and therefore deterministic sum) to the table row it was read from."""

    @staticmethod
    def forward(ctx, item_w, sep_row, user_w, mask, ids, user_ids, K, H, offsets, n_kept, norm_w, eps):
        x, _, src, slot = ops.t5enc_assemble(mask, ids, user_ids, item_w, sep_row, user_w, K, H, offsets, n_kept, norm_w, eps)
        ctx.save_for_backward(src, mask, ids, user_ids)
        ctx.K, ctx.H, ctx.S, ctx.sep, ctx.user = K, H, slot.shape[1], sep_row is not None, user_w is not None
        ctx.shapes = (item_w.shape[0], user_w.shape[0] if user_w is not None else 0)
        ctx.mark_non_differentiable(src, slot)
        return x, src, slot

    @staticmethod
    def backward(ctx, dx, _src, _slot):
        src, mask, ids, user_ids = ctx.saved_tensors
        V, U = ctx.shapes
        lay = _encoder_layout(mask.shape[1], ctx.H, ctx.sep, ctx.user, dx.device)
        src = src.long()
        b, pos = src // ctx.S, src % ctx.S
        kind, col, lvl = lay[0, pos], lay[1, pos], lay[2, pos]
        d_item = d_sep = d_user = None
        if ctx.needs_input_grad[0]:
            row = (ids[b, col].long() + lvl * ctx.K) * mask[b, col].float().long()   # the kernel's id: masked ids read row 0
            row = torch.where((kind == 1) & (row >= 0) & (row < V), row, V)
            d_item = dx.new_zeros((V + 1, dx.shape[1])).index_put_((row,), dx, accumulate=True)[:V]
        if ctx.sep and ctx.needs_input_grad[1]:
            d_sep = (dx * (kind == 2).to(dx.dtype)[:, None]).sum(0, keepdim=True)
        if ctx.user and ctx.needs_input_grad[2]:
            row = torch.where(kind == 0, torch.remainder(user_ids[b, 0], U), U)
            d_user = dx.new_zeros((U + 1, dx.shape[1])).index_put_((row,), dx, accumulate=True)[:U]
        return d_item, d_sep, d_user, None, None, None, None, None, None, None, None, None


class _ScatterFunction(torch.autograd.Function):
    """``ops.t5enc_scatter`` with its backward: the packed rows' gradient is the output's gradient gathered at src."""

    @staticmethod
    def forward(ctx, rows, slot, src):
        ctx.save_for_backward(src)
        return ops.t5enc_scatter(rows, slot)

    @staticmethod
    def backward(ctx, dout):
        (src,) = ctx.saved_tensors
        return dout.reshape(-1, dout.shape[-1]).index_select(0, src.long()), None, None


class _RelBiasFunction(torch.autograd.Function):
    """``t5enc_rel_bias(compute_bias(S, S)[0])`` of a bidirectional T5Attention: rel [heads, 2S - 1] = table[bucket(t - (S - 1))]^T,
    the same values.  Its backward adds d_rel into the table with ``index_put_`` (accumulate, a sorted sum), so the table's
    gradient is bit-reproducible; compute_bias's embedding backward is not."""

    @staticmethod
    def forward(ctx, table, buckets):
        ctx.save_for_backward(buckets)
        ctx.rows = table.shape[0]
        return table.index_select(0, buckets).t().contiguous()

    @staticmethod
    def backward(ctx, drel):
        (buckets,) = ctx.saved_tensors
        return drel.new_zeros((ctx.rows, drel.shape[0])).index_put_((buckets,), drel.t(), accumulate=True), None


def _rel_bias(att, S: int) -> Tensor:
    dist = torch.arange(-(S - 1), S, device=att.relative_attention_bias.weight.device)
    buckets = att._relative_position_bucket(dist, bidirectional=not att.is_decoder, num_buckets=att.relative_attention_num_buckets,
                                            max_distance=att.relative_attention_max_distance)
    return _RelBiasFunction.apply(att.relative_attention_bias.weight, buckets.long())


#: longest encoder sequence the training attention's backward takes (one shared-memory bin array of 2S - 1 floats per warp)
MAX_TRAIN_ENCODER_LEN = 5120


# What the two training passes share.  Dropout follows HF: each site's probability is read at call time from its module when that
# module is in training mode (0 else), and the draws come from torch's generator in HF's order.
def _p(mod) -> float:
    return float(mod.p) if mod.training else 0.0


def _attention_dropout(att, device):
    """(p, seed) of one attention site: the attention-weight dropout's probability and, when it is on, a fresh seed for the
    kernel's Philox stream drawn from torch's generator."""
    p = float(att.dropout) if att.training else 0.0
    return p, ops.t5enc_dropout_seed(device) if p > 0 else torch.zeros(1, dtype=torch.int64, device=device)


def _train_sublayer(x: Tensor, out: Tensor, sub, weight: Tensor, eps: float):
    """The end of sub-layer ``sub``: x + dropout(out), then the next T5LayerNorm -> (x, nrm)."""
    return ops.T5EncAddNormFunction.apply(x, dropout_rows(out, _p(sub.dropout)), weight, eps)


def _train_feed_forward(x: Tensor, nrm: Tensor, sub, weight: Tensor, eps: float):
    """The feed-forward sub-layer ``sub``: wi, relu, dropout, wo, then ``_train_sublayer``."""
    ff = sub.DenseReluDense
    h = dropout_rows(F.relu(F.linear(nrm, ff.wi.weight)), _p(ff.dropout))
    return _train_sublayer(x, F.linear(h, ff.wo.weight), sub, weight, eps)


def _check_fp32_parameters(model: nn.Module, what: str) -> None:
    if any(t.dtype != torch.float32 for t in model.parameters()):
        raise Rqb200Error(f"{what} needs fp32 parameters")


class FusedT5EncodeTrain:
    """The encoder pass of ``forward(encoder="fused")``: ``FusedT5Encode``'s packed pass (kept positions only, HF's relative bias
    at the original positions) made trainable.  Autograd runs through
      * ``_AssembleFunction`` (gradient into ``item_sid_embedding_table``, ``sep_token`` and ``user_embedding``),
      * ``ops.T5EncAddNormFunction`` at every norm (out of place: the residual row and its inverse RMS are saved),
      * ``ops.T5EncAttentionFunction`` (attention-weight dropout from a Philox stream keyed on a seed drawn per layer from torch's
        generator, log-sum-exp saved; the backward recomputes P),
      * ``F.linear`` for every GEMM and ``_ScatterFunction`` back to [B, S, d_model];
    ``rel`` holds the values of ``t5enc_rel_bias(compute_bias(S, S)[0])`` of block 0 (``_rel_bias``: a gather of
    ``relative_attention_bias`` at the buckets of distances -(S - 1) .. S - 1), so its gradient reaches that table summed over the
    layers, as in HF, through a deterministic sum.  Dropout sites: embedding, attention weights, attention output, feed-forward
    inner and output, final output.  The token-wise sites call ``dropout_rows``.  fp32 parameters only; an active autocast region
    raises ``ValueError``.  ``attention`` picks the attention kernels: "fp32" (``ops.T5EncAttentionFunction``) or "tf32"
    (``ops.T5EncAttentionTCFunction``, the same keep bits under the same seed)."""

    def __init__(self, model: "EncoderDecoderRetrievalModel", attention: str = "fp32"):
        self.model = model
        self.t5 = _T5Weights(model.encoder.encoder, "encoder=\"fused\"")
        _check_fp32_parameters(model, "forward(encoder=\"fused\")")
        tf32 = _choice(attention, None, ENCODER_ATTENTIONS, "FusedT5EncodeTrain", "attention") == "tf32"
        self.attention = ops.T5EncAttentionTCFunction if tf32 else ops.T5EncAttentionFunction

    def __call__(self, attention_mask: Tensor, input_ids: Tensor, user_id: Optional[Tensor] = None):
        """(enc_out [B, S, d_model] with the rows of dropped positions 0, enc_mask [B, S]), as ``encoder_forward_pass``."""
        out = self.packed(attention_mask, input_ids, user_id)
        return _ScatterFunction.apply(out.rows, out.slot, out.src), out.enc_mask

    def packed(self, attention_mask: Tensor, input_ids: Tensor, user_id: Optional[Tensor] = None) -> PackedEncoderOutput:
        """The pass without the scatter: the kept rows [N, d_model] (the encoder's final dropout applied) and their layout."""
        _check_no_autocast("forward(encoder=\"fused\")")
        m, t5, eps, norms = self.model, self.t5, self.t5.eps, self.t5.norms
        enc = t5.stack
        H = m.num_hierarchies
        sep = m.sep_token is not None
        user = user_id is not None and m.user_embedding is not None
        S = ops.t5enc_len(attention_mask.shape[1], H, sep, user)
        if S > MAX_TRAIN_ENCODER_LEN:
            raise Rqb200Error(f"forward(encoder=\"fused\"): {S} encoder positions exceed {MAX_TRAIN_ENCODER_LEN}")
        offsets, key_mask = ops.t5enc_offsets(attention_mask, H, sep, user)
        n_kept = _read_n_kept(offsets)
        x, src, slot = _AssembleFunction.apply(
            m.item_sid_embedding_table.weight, m.sep_token if sep else None, m.user_embedding.weight if user else None,
            attention_mask, input_ids, user_id if user else None, m.num_embeddings_per_hierarchy, H, offsets, n_kept,
            norms[0], eps)
        x, nrm = ops.T5EncAddNormFunction.apply(dropout_rows(x, _p(enc.dropout)), None, norms[0], eps)
        rel = _rel_bias(t5.blocks[0][0].SelfAttention, S)
        for l, lay in enumerate(t5.blocks):
            p_att, seed = _attention_dropout(lay[0].SelfAttention, x.device)
            a = self.attention.apply(F.linear(nrm, t5.qkv(l)), rel, src, offsets, key_mask, S, seed, p_att)
            x, nrm = _train_sublayer(x, F.linear(a, lay[0].SelfAttention.o.weight), lay[0], norms[2 * l + 1], eps)
            x, nrm = _train_feed_forward(x, nrm, lay[1], norms[2 * l + 2], eps)
        return PackedEncoderOutput(dropout_rows(nrm, _p(enc.dropout)), offsets, key_mask, src, slot, S,
                                   _encoder_mask(m, attention_mask, user))

class _DecoderInputFunction(torch.autograd.Function):
    """The decoder's input rows x [B * T, d]: row b * T + t is bos for t = 0 and table[ids[b, t - 1] + (t - 1) K] after.  The
    backward adds each row's gradient to the table row it was read from with ``index_put_`` (accumulate, a sorted and therefore
    deterministic sum) and sums bos's rows in order."""

    @staticmethod
    def forward(ctx, table, bos, ids, K, T):
        B, d = ids.shape[0], table.shape[1]
        rows = ids[:, :T - 1].long() + torch.arange(T - 1, device=ids.device) * K
        x = torch.cat([bos.expand(B, 1, d), table.index_select(0, rows.reshape(-1)).view(B, T - 1, d)], dim=1)
        ctx.save_for_backward(rows)
        ctx.V, ctx.T = table.shape[0], T
        return x.reshape(B * T, d)

    @staticmethod
    def backward(ctx, dx):
        (rows,) = ctx.saved_tensors
        dx = dx.view(-1, ctx.T, dx.shape[1])
        d_table = d_bos = None
        if ctx.needs_input_grad[0]:
            d_table = dx.new_zeros((ctx.V, dx.shape[2])).index_put_((rows.reshape(-1),), dx[:, 1:].reshape(-1, dx.shape[2]),
                                                                    accumulate=True)
        if ctx.needs_input_grad[1]:
            d_bos = dx[:, 0].sum(0, keepdim=True)
        return d_table, d_bos, None, None, None


#: most decoder positions (hierarchy levels) the decoder's training kernels take
MAX_TRAIN_DECODER_LEN = 8


class FusedT5DecodeTrain:
    """The decoder pass of ``forward(decoder="fused")``: HF's T5Stack decoder (relu FFN, d_kv 64) over the T = H positions the loss
    reads (causality makes them independent of HF's extra last position), as cuBLAS GEMMs (``F.linear``) between the training
    kernels of csrc/t5dec.cu.  Autograd runs through
      * ``_DecoderInputFunction`` (gradient into ``item_sid_embedding_table`` and ``bos_token``, deterministic),
      * ``ops.T5EncAddNormFunction`` at every norm,
      * ``ops.T5DecSelfAttentionFunction`` (causal, block 0's unidirectional relative bias from ``_rel_bias``) and
        ``ops.T5DecCrossAttentionFunction`` over the encoder rows of ``PackedEncoderOutput.keys``: the packed rows of
        ``FusedT5EncodeTrain.packed`` or the [B * S] rows of HF's encoder.  Cross keys and values are one GEMM per layer on
        those rows.  Attention-weight dropout draws one seed per attention site and layer from torch's generator, the bits keyed
        on the key's ORIGINAL encoder position, so both encoders give the same bits under one seed;
      * HF's token-wise dropout sites through ``dropout_rows``.
    ``__call__`` returns the final-normed, dropped-out hidden state [B, T, d_model].  fp32 parameters only; an active autocast
    region raises ``ValueError``."""

    def __init__(self, model: "EncoderDecoderRetrievalModel"):
        self.model = model
        self.t5 = _T5Weights(model.t5_decoder, "decoder=\"fused\"")
        if model.num_hierarchies > MAX_TRAIN_DECODER_LEN:
            raise Rqb200Error(f"forward(decoder=\"fused\"): {model.num_hierarchies} levels exceed {MAX_TRAIN_DECODER_LEN}")
        _check_fp32_parameters(model, "forward(decoder=\"fused\")")

    def __call__(self, fut_ids: Tensor, rows: Tensor, offsets: Tensor, key_mask: Tensor, src: Optional[Tensor], S: int) -> Tensor:
        """fut_ids [B, >= T - 1]; rows [*, d_model] the encoder rows, history b's keys rows offsets[b] .. offsets[b + 1] - 1 with
        additive key_mask [rows]; src [rows] (b * S + position) or None (row - offsets[b] is the position)."""
        _check_no_autocast("forward(decoder=\"fused\")")
        m, t5, eps, norms = self.model, self.t5, self.t5.eps, self.t5.norms
        dec = t5.stack
        T, B = m.num_hierarchies, fut_ids.shape[0]
        x = _DecoderInputFunction.apply(m.item_sid_embedding_table.weight, m.bos_token, fut_ids, m.num_embeddings_per_hierarchy, T)
        x, nrm = ops.T5EncAddNormFunction.apply(dropout_rows(x, _p(dec.dropout)), None, norms[0], eps)
        rel = _rel_bias(t5.blocks[0][0].SelfAttention, T)
        for l, lay in enumerate(t5.blocks):
            p_att, seed = _attention_dropout(lay[0].SelfAttention, x.device)
            a = ops.T5DecSelfAttentionFunction.apply(F.linear(nrm, t5.qkv(l)), rel, T, seed, p_att)
            x, nrm = _train_sublayer(x, F.linear(a, lay[0].SelfAttention.o.weight), lay[0], norms[3 * l + 1], eps)
            ca = lay[1].EncDecAttention
            p_ca, seed = _attention_dropout(ca, x.device)
            kv = F.linear(rows, torch.cat([ca.k.weight, ca.v.weight]))
            a = ops.T5DecCrossAttentionFunction.apply(F.linear(nrm, ca.q.weight), kv, offsets, key_mask, src, S, T, seed, p_ca)
            x, nrm = _train_sublayer(x, F.linear(a, ca.o.weight), lay[1], norms[3 * l + 2], eps)
            x, nrm = _train_feed_forward(x, nrm, lay[2], norms[3 * l + 3], eps)
        return dropout_rows(nrm, _p(dec.dropout)).view(B, T, -1)


def _tuple_key(tuples: Tensor, K: int) -> Tensor:
    """int64 [...]: the ids of tuples [..., H] packed into one key, level 0 most significant, so keys order as the tuples do
    (lexicographically).  Ids outside [0, K) are clamped: the caller tracks which tuples are valid."""
    key = torch.zeros(tuples.shape[:-1], dtype=torch.int64, device=tuples.device)
    for h in range(tuples.shape[-1]):
        key = key * K + tuples[..., h].clamp(0, K - 1)
    return key


def _check_tuple_key(H: int, K: int, what: str, max_levels: Optional[int] = None) -> None:
    """``_tuple_key`` of H levels of K codes must fit in 62 bits (and H in max_levels, when the caller's kernels bound it)."""
    if H * max(1, (K - 1).bit_length()) > 62 or (max_levels is not None and H > max_levels):
        raise Rqb200Error(f"{what}: {H} levels of {K} codes do not pack into a 64-bit tuple key"
                          + (f" (at most {max_levels} levels)" if max_levels is not None else ""))


def _level_values(value, H: int, name: str, what: str) -> List[float]:
    """A sampling control given as one float or as a sequence of H floats (one per level) -> H floats."""
    if isinstance(value, (int, float)) and not isinstance(value, bool):
        return [float(value)] * H
    try:
        values = [float(v) for v in value]
    except (TypeError, ValueError):
        raise ValueError(f"{what}: {name} must be a float or a sequence of {H} floats (one per level), got {value!r}") from None
    if len(values) != H:
        raise ValueError(f"{what}: {name} has {len(values)} values; it takes one float or one per level ({H})")
    return values


def _sampling_controls(search: str, temperature, top_p, H: int, what: str, ignore_temperature: bool = False):
    """The per-level (temperature, top_p) of a search, checked before any launch: None for the untempered search (T = 1 and
    top_p = 1 at every level, or a deterministic search).  T must be finite and > 0 and top_p in (0, 1], else ``ValueError``;
    so must anything but the defaults with search "beam" or "exact", except a temperature ``ignore_temperature`` drops (the
    reference's ``generate_next_sem_id`` argument, which those searches ignore)."""
    deterministic = search != "sample"
    temps = [1.0] * H if deterministic and ignore_temperature else _level_values(temperature, H, "temperature", what)
    ps = _level_values(top_p, H, "top_p", what)
    for t in temps:
        if not (math.isfinite(t) and t > 0):
            raise ValueError(f"{what}: temperature must be finite and > 0, got {t}")
    for p in ps:
        if not 0 < p <= 1:
            raise ValueError(f"{what}: top_p must be in (0, 1], got {p}")
    if all(t == 1 for t in temps) and all(p == 1 for p in ps):
        return None
    if deterministic:
        raise ValueError(f"{what}: temperature and top_p shape the sampled search only; search={search!r} is deterministic "
                         "(use search=\"sample\", or leave them at 1)")
    return list(zip(temps, ps))


def _prefix_cap_controls(search: str, max_per_prefix: Optional[int], prefix_len: int, H: int, what: str):
    """The (prefix_len, max_per_prefix) of a capped search, checked before any launch: None without ``max_per_prefix``.
    prefix_len must be in [1, H - 1] and max_per_prefix >= 1, else ``ValueError``; search="exact" raises ``ValueError``."""
    if max_per_prefix is None:
        return None
    if isinstance(max_per_prefix, bool) or isinstance(prefix_len, bool):
        raise ValueError(f"{what}: max_per_prefix and prefix_len must be integers")
    if int(max_per_prefix) != max_per_prefix or max_per_prefix < 1:
        raise ValueError(f"{what}: max_per_prefix must be an integer >= 1, got {max_per_prefix!r}")
    if int(prefix_len) != prefix_len or not 1 <= prefix_len <= H - 1:
        raise ValueError(f"{what}: prefix_len must be an integer in [1, {H - 1}] (the id tuple has {H} levels), got "
                         f"{prefix_len!r}")
    if search == "exact":
        raise ValueError(f"{what}: max_per_prefix caps the \"beam\" and \"sample\" searches only; search=\"exact\" takes no cap")
    return int(prefix_len), int(max_per_prefix)


def _non_finite_error(what: str, n_bad: int) -> RuntimeError:
    return RuntimeError(f"{what}: {n_bad} decoder row(s) of the head's logits "
                        "hold a NaN or +inf or are all -inf; the items below them score NaN")

class EncoderDecoderRetrievalModel(nn.Module):
    """T5 encoder over the history's semantic ids, T5 decoder stack plus one Linear head per hierarchy level for the next
    item's ids; ``generate`` is a sampled beam search restricted to id prefixes that occur in the corpus (``codebooks``)."""

    def __init__(self, codebooks: Tensor, num_hierarchies: int, num_embeddings_per_hierarchy: int, t5_d_model: int = 128,
                 t5_num_heads: int = 6, t5_d_ff: int = 1024, t5_num_layers: int = 4, top_k_for_generation: int = 10,
                 should_add_sep_token: bool = True, num_user_bins: Optional[int] = None):
        super().__init__()
        self.num_hierarchies = num_hierarchies
        self.num_embeddings_per_hierarchy = num_embeddings_per_hierarchy
        self.top_k_for_generation = top_k_for_generation
        self.register_buffer("codebooks", codebooks)
        vocab = num_embeddings_per_hierarchy * num_hierarchies
        shape = dict(vocab_size=vocab, d_model=t5_d_model, num_heads=t5_num_heads, d_ff=t5_d_ff, num_layers=t5_num_layers)
        self.encoder = T5EncoderModel(T5Config(**shape, is_decoder=False))
        self.t5_decoder = T5Stack(T5Config(**shape, is_decoder=True, is_encoder_decoder=False))
        self.bos_token = nn.Parameter(torch.randn(1, t5_d_model), requires_grad=True)
        self.decoder_mlp = nn.ModuleList(
            [nn.Linear(t5_d_model, num_embeddings_per_hierarchy, bias=False) for _ in range(num_hierarchies)])
        # one table for all levels: token t of level h is row h * num_embeddings_per_hierarchy + t
        self.item_sid_embedding_table = nn.Embedding(vocab, t5_d_model)
        self.user_embedding = nn.Embedding(num_user_bins, t5_d_model) if num_user_bins else None
        self.sep_token = nn.Parameter(torch.randn(1, t5_d_model), requires_grad=True) if should_add_sep_token else None
        self._prefix_index_cache = None
        self._item_table_cache = None

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    # ------------------------------------------------------------------------------------------------ transformer passes
    def _level_offsets(self, ids: Tensor, mask: Optional[Tensor] = None) -> Tensor:
        """Column c of a [B, n] id row belongs to level c % num_hierarchies: shift it into that level's rows of the table;
        padded positions (mask 0) become 0."""
        if ids.ndim != 2:
            raise ValueError("Input tensor must be 2-dimensional.")
        level = torch.arange(ids.shape[1], device=ids.device) % self.num_hierarchies
        out = ids + level * self.num_embeddings_per_hierarchy
        return out if mask is None else out * mask

    def _append_sep_tokens(self, emb: Tensor, mask: Tensor):
        """Insert sep_token after every item's num_hierarchies embeddings; the separator inherits the mask of the item's last id."""
        B, n, d = emb.shape
        H = self.num_hierarchies
        items = n // H
        sep = self.sep_token.view(1, 1, 1, d).expand(B, items, 1, d)
        emb = torch.cat([emb.view(B, items, H, d), sep], dim=2).reshape(B, items * (H + 1), d)
        mask = mask.view(B, items, H)
        mask = torch.cat([mask, mask[:, :, -1:]], dim=2).reshape(B, items * (H + 1))
        return emb, mask

    def encoder_forward_pass(self, attention_mask, input_ids, user_id=None):
        inputs_embeds = self.item_sid_embedding_table(self._level_offsets(input_ids, attention_mask))
        if self.sep_token is not None:
            inputs_embeds, attention_mask = self._append_sep_tokens(inputs_embeds, attention_mask)
        if user_id is not None and self.user_embedding is not None:
            user = self.user_embedding(torch.remainder(user_id[:, 0], self.user_embedding.num_embeddings))
            inputs_embeds = torch.cat([user.unsqueeze(1), inputs_embeds], dim=1)
            attention_mask = torch.cat([torch.ones(attention_mask.shape[0], 1, device=attention_mask.device), attention_mask],
                                       dim=1)
        out = self.encoder(inputs_embeds=inputs_embeds, attention_mask=attention_mask).last_hidden_state
        return out, attention_mask

    @staticmethod
    def _cache_holds_steps(past_key_values) -> bool:
        if isinstance(past_key_values, (EncoderDecoderCache, DynamicCache)):
            return len(past_key_values) > 0
        return isinstance(past_key_values, tuple)

    def decoder_forward_pass(self, attention_mask=None, future_ids=None, encoder_output=None, attention_mask_for_encoder=None,
                             use_cache=False, past_key_values=None):
        if future_ids is None:
            inputs_embeds = self.bos_token.unsqueeze(0).expand(encoder_output.shape[0], 1, -1)
        else:
            mask = torch.ones_like(future_ids) if attention_mask is None else attention_mask
            inputs_embeds = self.item_sid_embedding_table(self._level_offsets(future_ids, mask))
            if self._cache_holds_steps(past_key_values):
                inputs_embeds = inputs_embeds[:, -1:, :]          # the cache holds every earlier step
            else:
                B = future_ids.shape[0]
                inputs_embeds = torch.cat([self.bos_token.unsqueeze(0).expand(B, 1, -1), inputs_embeds], dim=1)
                if attention_mask is not None:
                    attention_mask = torch.cat([torch.ones(B, 1, device=future_ids.device), attention_mask], dim=1)
        out = self.t5_decoder(inputs_embeds=inputs_embeds, attention_mask=attention_mask, encoder_hidden_states=encoder_output,
                              encoder_attention_mask=attention_mask_for_encoder, use_cache=use_cache,
                              past_key_values=past_key_values)
        if use_cache:
            return out.last_hidden_state, out.past_key_values
        return out.last_hidden_state

    @torch.compiler.disable
    def _fused_train_encoder_pass(self, attention_mask, input_ids, user_id, attention="fp32"):
        """FusedT5EncodeTrain runs outside torch.compile's graphs (ctypes launches): a graph break, with backward through it."""
        return FusedT5EncodeTrain(self, attention)(attention_mask, input_ids, user_id)

    @torch.compiler.disable
    def _fused_train_passes(self, attention_mask, input_ids, user_id, fut_ids, attention="fp32"):
        """Both fused passes in one graph break: the decoder attends to the encoder's packed rows (no scatter to [B, S, d])."""
        enc = FusedT5EncodeTrain(self, attention).packed(attention_mask, input_ids, user_id)
        return FusedT5DecodeTrain(self)(fut_ids, *enc.keys())

    @torch.compiler.disable
    def _fused_train_decoder_pass(self, fut_ids, enc_out, enc_mask):
        """The fused decoder pass over HF's encoder output, every position a key row."""
        return FusedT5DecodeTrain(self)(fut_ids, *PackedEncoderOutput.of_padded(enc_out, enc_mask).keys())

    def forward(self, batch: TokenizedSeqBatch, encoder: Optional[str] = None, decoder: Optional[str] = None,
                encoder_attention: Optional[str] = None) -> ModelOutput:
        """The training loss.  ``encoder`` (default: the module's ``DEFAULT_FORWARD_ENCODER``, read at call time):
          "hf"      ``encoder_forward_pass``: transformers' T5EncoderModel over every position, as the reference;
          "fused"   ``FusedT5EncodeTrain``: the kept positions only, with HF's dropout in training mode and none in eval mode;
                    gradients in both.  It reads the packed row count on the host once.
        ``decoder`` (default: the module's ``DEFAULT_FORWARD_DECODER``, read at call time):
          "hf"      ``decoder_forward_pass``: transformers' T5Stack over BOS and the H future ids, as the reference;
          "fused"   ``FusedT5DecodeTrain``: the H positions the loss reads, with HF's dropout in training mode and none in eval
                    mode; gradients in both.  With encoder="fused" it attends to the encoder's packed rows directly.
        ``encoder_attention`` (default: the module's ``DEFAULT_ENCODER_ATTENTION``, read at call time) picks the fused encoder's
        attention kernels: "fp32" or "tf32" (TF32 tensor-core products, the same dropout bits).  "tf32" needs encoder="fused"."""
        encoder = _choice(encoder, DEFAULT_FORWARD_ENCODER, ENCODERS, "forward", "encoder")
        decoder = _choice(decoder, DEFAULT_FORWARD_DECODER, DECODERS, "forward", "decoder")
        att = _encoder_attention(encoder, encoder_attention, "forward")
        H = self.num_hierarchies
        input_ids = _strip_dedup_col(batch.sem_ids, H + 1, H)
        attention_mask = _strip_dedup_col(batch.seq_mask.long(), H + 1, H)
        fut_ids = batch.sem_ids_fut[:, :H]
        if encoder == "fused" and decoder == "fused":
            dec = self._fused_train_passes(attention_mask, input_ids, batch.user_ids, fut_ids, att)
        else:
            if encoder == "fused":
                enc, enc_mask = self._fused_train_encoder_pass(attention_mask, input_ids, batch.user_ids, att)
            else:
                enc, enc_mask = self.encoder_forward_pass(attention_mask=attention_mask, input_ids=input_ids,
                                                          user_id=batch.user_ids)
            if decoder == "fused":
                dec = self._fused_train_decoder_pass(fut_ids, enc, enc_mask)
            else:
                dec = self.decoder_forward_pass(future_ids=fut_ids, encoder_output=enc, attention_mask_for_encoder=enc_mask,
                                                use_cache=False)[:, :-1]
        loss = torch.tensor(0.0, device=dec.device)
        per_level = []
        for h in range(H):
            level_loss = F.cross_entropy(self.decoder_mlp[h](dec[:, h]), fut_ids[:, h].long())
            loss = loss + level_loss
            per_level.append(level_loss.detach())
        return ModelOutput(loss=loss, logits=None, loss_d=torch.stack(per_level))

    # ------------------------------------------------------------------------------------------------ constrained search
    def _prefix_index(self, device: torch.device) -> ops.SidPrefixIndex:
        """The corpus prefix index, built on first use and again whenever the codebooks buffer is another tensor, has been
        written to (load_state_dict copies into it) or the search runs on another device."""
        cb = self.codebooks
        key = (id(cb), cb._version, cb.device, torch.device(device))
        if self._prefix_index_cache is None or self._prefix_index_cache[0] != key:
            index = ops.SidPrefixIndex(cb.to(device), self.num_embeddings_per_hierarchy)
            self._prefix_index_cache = (key, index)
        return self._prefix_index_cache[1].ready()

    def _item_table(self, device: torch.device) -> ops.SidItemTable:
        """The corpus item table (row n of codebooks is item n), cached on the same key as the prefix index."""
        cb = self.codebooks
        key = (id(cb), cb._version, cb.device, torch.device(device))
        if self._item_table_cache is None or self._item_table_cache[0] != key:
            table = ops.SidItemTable(cb[:, :self.num_hierarchies].to(device), self.num_embeddings_per_hierarchy)
            self._item_table_cache = (key, table)
        return self._item_table_cache[1].ready()

    def _check_valid_prefix(self, prefix: Tensor, batch_size: int = 100000) -> Tensor:
        """bool [P]: some corpus row starts with prefix[p] (batch_size is accepted for the reference's signature)."""
        return self._prefix_index(prefix.device).check(prefix)

    def _sample_and_select(self, index: ops.SidPrefixIndex, probas: Tensor, generated: Optional[Tensor],
                           log_probas: Optional[Tensor], k: int, n_cands: int, reject: Tensor,
                           exclude: Optional[ops.SidExclusion] = None, include: Optional[ops.SidInclusion] = None,
                           wide: bool = False, cap: Optional[tuple] = None):
        """One level of the search after the softmax: n_cands samples per beam, prefix check, scores, the k best beams
        (``wide``: on the cluster kernel, ``SidPrefixIndex.sample_select_wide``)."""
        filt = {} if exclude is None else {"exclude": exclude}
        if include is not None:
            filt["include"] = include
        if cap is not None:
            filt["cap"] = cap
        select = index.sample_select_wide if wide else index.sample_select
        return select(probas, draw_exponential(probas), generated, log_probas, k, n_cands, reject=reject, **filt)

    @staticmethod
    def _warped_sample_and_select(index: ops.SidPrefixIndex, logits: Tensor, generated: Optional[Tensor],
                                  log_probas: Optional[Tensor], k: int, n_cands: int, bad: Tensor, control: tuple,
                                  wide: bool, filt: dict, cap: Optional[tuple] = None):
        """One level of the search from the head's logits at this level's (temperature, top_p): the noise is drawn as the
        untempered level draws it (``draw_exponential`` of a [B * kp, K] tensor), then one launch of
        ``SidPrefixIndex.sample_select_warped`` (``_wide`` on the cluster kernel)."""
        select = index.sample_select_warped_wide if wide else index.sample_select_warped
        if cap is not None:
            filt = dict(filt, cap=cap)
        return select(logits, draw_exponential(logits), generated, log_probas, k, n_cands, *control, bad=bad, **filt)

    @staticmethod
    def _narrow_search(search: str, k: int, n_cands: int) -> bool:
        """A search of beam width k fits the one-CTA-per-history selection kernels (``beam_topk`` / ``sample_select``)."""
        return k <= 32 and (search == "beam" or k * n_cands <= 1024)

    def _search_cap(self, cap: Optional[tuple], search: str, k: int, n_cands: int, what: str) -> Optional[tuple]:
        """A checked cap (``_prefix_cap_controls``) at beam width k: None when max_per_prefix >= k (it cannot bind; the
        uncapped path runs), else ``Rqb200Error`` when only the cluster kernels take the width (they have no capped mode)."""
        if cap is None or cap[1] >= k:
            return None
        if not self._narrow_search(search, k, n_cands):
            raise Rqb200Error(f"{what}: max_per_prefix = {cap[1]} caps the one-CTA selection kernels only; num_beams = {k} "
                              f"(with {n_cands} candidates per beam for \"sample\") runs on the cluster kernels, which take no "
                              "cap (need num_beams <= 32, and num_beams * candidates <= 1024 for \"sample\")")
        return cap

    def _check_search_limits(self, search: str, k: int, n_cands: int, num_beams: Optional[int] = None) -> None:
        K = self.num_embeddings_per_hierarchy
        if num_beams is not None:
            top = MAX_NUM_BEAMS if search == "sample" else min(MAX_NUM_BEAMS, K)
            if not 1 <= num_beams <= top or K > 2048:
                raise Rqb200Error(f"generate: num_beams = {num_beams} with {K} codes per level is outside the {search} search's "
                                  f"limits (1 <= num_beams <= {top}, at most 2048 codes per level)")
            return
        if search == "sample":
            if k > 32 or k * n_cands > 1024 or K > 2048:
                raise Rqb200Error(f"generate: top_k_for_generation = {k} (at most 32, and top_k * {n_cands} candidates at most "
                                  f"1024) with {K} codes per level (at most 2048) is outside the sampling kernel's limits")
        elif k > 32 or k > K or K > 2048:
            raise Rqb200Error(f"generate: top_k_for_generation = {k} (at most 32 and at most the number of codes) with {K} "
                              "codes per level (at most 2048) is outside the beam search kernel's limits")

    def _fused_decoder(self, enc_out: Tensor, enc_mask: Tensor, k: int) -> FusedT5Decode:
        return FusedT5Decode(self, enc_out, enc_mask, k)

    def _fused_encoder(self, attention: str = "fp32") -> FusedT5Encode:
        return FusedT5Encode(self, attention)

    def _excluded_items(self, batch: TokenizedSeqBatch, exclude_items: Optional[Tensor],
                        exclude_history: Optional[bool]) -> Optional[Tensor]:
        """int64 [B, M]: exclude_items joined with the batch's own items when ``exclude_history`` (default
        ``DEFAULT_EXCLUDE_HISTORY``); None when there is nothing to exclude."""
        exclude_history = DEFAULT_EXCLUDE_HISTORY if exclude_history is None else exclude_history
        parts = [] if exclude_items is None else [exclude_items]
        if exclude_history:
            parts.append(self.history_items(batch))
        if not parts:
            return None
        B = batch.sem_ids.shape[0]
        return torch.cat([self._check_exclude_items(t, B) for t in parts], dim=1)

    @staticmethod
    def _check_exclude_items(items: Tensor, B: int, name: str = "exclude_items") -> Tensor:
        ops._need_cuda(items)
        if items.dim() != 2 or items.shape[0] != B or items.dtype.is_floating_point or items.dtype == torch.bool:
            raise ValueError(f"{name} must be an integer [B = {B}, M] tensor of corpus rows, got {items.dtype} "
                             f"{tuple(items.shape)}")
        return items.long()

    def _exclusion(self, items: Optional[Tensor], B: int, device: torch.device) -> Optional[ops.SidExclusion]:
        """The exclusion sets of one call (``ops.sid_exclusion_build`` on the corpus item table), None without items."""
        if items is None:
            return None
        items = self._check_exclude_items(items, B)
        _, leaf_key, _ = self._rank_levels(device)
        return ops.sid_exclusion_build(items.to(device), self._item_table(device), leaf_key)

    def _filters(self, exclude_items: Optional[Tensor], include_items: Optional[Tensor], B: int,
                 device: torch.device) -> list:
        """The item filters of one call, in build order: the exclusion (``_exclusion``), then the allow-list built on it
        (``ops.sid_inclusion_build``); empty without either.  The consumers take the last one (``_filter_kwargs``)."""
        exclusion = self._exclusion(exclude_items, B, device)
        filters = [] if exclusion is None else [exclusion]
        if include_items is not None:
            items = self._check_exclude_items(include_items, B, "include_items")
            _, leaf_key, _ = self._rank_levels(device)
            filters.append(ops.sid_inclusion_build(items.to(device), self._item_table(device), leaf_key, exclude=exclusion))
        return filters

    @staticmethod
    def _filter_kwargs(filters: list) -> dict:
        """The filter argument of the search and retrieval calls: an allow-list holds the exclusion folded in."""
        if not filters:
            return {}
        return {"include" if isinstance(filters[-1], ops.SidInclusion) else "exclude": filters[-1]}

    @staticmethod
    def _counter_values(counters: Tensor, filters: list) -> Tensor:
        """int32 on the device: the counters, then each filter's count of ids outside [-1, N) -- what ``_read_counters`` reads."""
        if not filters:
            return counters
        return torch.cat([counters.int()] + [f.count[:, -1].sum(dtype=torch.int32).view(1) for f in filters])

    @staticmethod
    def _read_counters(counters: Tensor, filters: list, what: str) -> List[int]:
        """The one host read at the end of a call: its counters, after which the excluded or allowed ids outside [-1, N) of
        the call's filters (``_filters``) raise."""
        if not filters:
            return counters.tolist()
        values = EncoderDecoderRetrievalModel._counter_values(counters, filters).tolist()
        return EncoderDecoderRetrievalModel._check_filter_counts(values, counters.numel(), filters, what)

    @staticmethod
    def _check_filter_counts(values: List[int], n_counters: int, filters: list, what: str) -> List[int]:
        """values as read from ``_counter_values``: the ``ValueError`` of a filter id outside [-1, N), else the counters."""
        values, n_ids = values[:n_counters], values[n_counters:]
        for f, n in zip(filters, n_ids):
            if n:
                kind = "allowed" if isinstance(f, ops.SidInclusion) else "excluded"
                raise ValueError(f"{what}: {n} {kind} item id(s) outside [-1, N) where N is the number of corpus rows")
        return values

    @torch.no_grad()
    def history_items(self, batch: TokenizedSeqBatch) -> Tensor:
        """int64 [B, S]: the corpus item of each (H ids, dedup) group of ``batch.sem_ids`` (``item_of``), -1 where the group is
        masked or does not resolve."""
        H = self.num_hierarchies
        B = batch.sem_ids.shape[0]
        groups = batch.sem_ids.reshape(B, -1, H + 1)
        items = self.item_of(groups.reshape(-1, H + 1)).view(B, -1)
        return torch.where(batch.seq_mask.reshape(B, -1, H + 1)[:, :, :H].bool().all(-1), items, -1)

    @torch.no_grad()
    def generate(self, attention_mask, input_ids, user_id=None, search: Optional[str] = None, decoder: Optional[str] = None,
                 encoder: Optional[str] = None, encoder_attention: Optional[str] = None, exclude_items: Optional[Tensor] = None,
                 include_items: Optional[Tensor] = None, num_beams: Optional[int] = None, temperature=1.0, top_p=1.0,
                 max_per_prefix: Optional[int] = None, prefix_len: int = 1):
        """Top-k semantic ids by beam search restricted to id prefixes of the corpus.  ``search`` (default: the module's
        ``DEFAULT_SEARCH``, read at call time):
          "sample"  per level, n_cands = min(64, K) tokens sampled without replacement per beam, scored by cumulative
                    log-probability, prefixes absent from the corpus scored -inf, the k best kept (the reference's search);
          "beam"    per level, every code of every beam scored by cumulative log-probability, the k best valid extensions kept
                    (equal scores: lowest beam * K + code first); deterministic, draws no random numbers.
        ``decoder`` (default: the module's ``DEFAULT_DECODER``, read at call time):
          "hf"      transformers' T5Stack with an EncoderDecoderCache, as the reference drives it;
          "fused"   ``FusedT5Decode``: the same T5 maths with cross keys/values once per history and the decoder-step kernels of
                    csrc/t5dec.cu; eval mode only (HF would apply dropout in training mode).
        ``encoder`` (default: the module's ``DEFAULT_ENCODER``, read at call time), independent of ``decoder`` and ``search``:
          "hf"      ``encoder_forward_pass``: transformers' T5EncoderModel over every position, padded ones included;
          "fused"   ``FusedT5Encode``: the same encoder output at every unpadded position (padded rows are 0) from the unpadded
                    positions only; eval mode only.  It reads the packed row count on the host once, before the first level.
        ``encoder_attention`` (default: the module's ``DEFAULT_ENCODER_ATTENTION``, read at call time) picks the fused encoder's
        attention kernel: "fp32" or "tf32" (TF32 tensor-core products).  "tf32" needs encoder="fused".
        ``exclude_items`` (integer [B, M], corpus rows, -1 pads, M <= ``ops.EXCLUDE_MAX_ITEMS``): no beam leads only to excluded
        items of its history; an extension under which every retrievable item is excluded is invalid, like a prefix the corpus
        lacks.  It adds one launch and no host read; ids outside [-1, N) raise ``ValueError`` after the search.
        ``include_items`` (integer [B, M], corpus rows, -1 pads, M <= ``ops.INCLUDE_MAX_ITEMS``): every beam leads to an eligible
        item of its history -- one in its allow-list, retrievable and not excluded; an extension without one under it is
        invalid, like a prefix the corpus lacks.  None means no restriction; a row without an eligible item gets -inf fillers
        only.  It adds one launch and no host read; ids outside [-1, N) raise ``ValueError`` after the search.
        ``num_beams`` (default None: ``top_k_for_generation``, with its limits) is the beam width w of this call:
        1 <= w <= min(1024, K) for "beam", 1 <= w <= 1024 for "sample" (still n_cands samples per beam), K <= 2048; outside
        them ``Rqb200Error`` before any launch.  Widths the one-CTA-per-history selection kernels take (w <= 32, and
        w * n_cands <= 1024 for "sample") run on them; wider ones select each level on one thread-block cluster per history
        (``SidPrefixIndex.beam_topk_wide`` / ``sample_select_wide``), with the same rules.  The fused decoder's self-attention
        cache is [layers, 2, H, B * w, inner] fp32; the HF decoder repeats the encoder output w times per history.
        ``temperature`` / ``top_p`` (default 1: the untempered search above, launch for launch) shape the "sample" search's
        draw, each a float or one float per level: level h draws from softmax(logits / T_h) restricted to its top-p_h nucleus
        (``SidPrefixIndex.sample_select_warped``); the beams still score and return the model's own log-probabilities.  T
        finite and > 0, 0 < top_p <= 1; anything else, or anything but 1 with "beam" or "exact", raises ``ValueError``
        before any launch.  Bad head rows then raise the "beam" search's ``RuntimeError``.
        ``max_per_prefix`` (default None: no cap) / ``prefix_len`` (default 1) cap how many beams share a prefix: among a
        history's returned beams with a finite log-probability, at most max_per_prefix share their first prefix_len ids (the
        -inf fillers are not beams and are exempt).  The cap binds at the levels h >= prefix_len (0-based; after level h a beam
        holds h + 1 ids); earlier levels run unchanged.  There a candidate's group is its parent's first prefix_len ids, and the
        level keeps what a walk down the search's own order (score descending, then lowest beam * K + code for "beam", the
        sampled order for "sample") keeps when it skips a candidate whose group already holds max_per_prefix: each group's
        max_per_prefix best, with the uncapped log-probability bits; the rest of the w slots are -inf fillers as before.  The
        cap composes with the item filters (a blocked extension is invalid before the cap counts it) and, for "sample", with
        temperature and top_p (the draws do not change).  "beam" stays deterministic.  prefix_len in [1, H - 1] and
        max_per_prefix >= 1, else ``ValueError``; search="exact" raises ``ValueError``.  max_per_prefix >= w cannot bind and runs
        the uncapped search, bit for bit; a cap that can bind on a width only the cluster kernels take (w > 32, or
        w * n_cands > 1024 for "sample") raises ``Rqb200Error``.  All before any launch.
        Returns generated [B, w, num_hierarchies] and log_probas [B, w]."""
        warp = self._sampling(search, temperature, top_p, "generate")
        cap = self._capping(search, max_per_prefix, prefix_len, num_beams, "generate")
        return self._generate(attention_mask, input_ids, user_id, search, decoder, encoder, encoder_attention,
                              self._filters(exclude_items, include_items, attention_mask.shape[0], attention_mask.device),
                              num_beams, warp, cap)

    def _sampling(self, search: Optional[str], temperature, top_p, what: str, ignore_temperature: bool = False):
        """``_sampling_controls`` of a call's search (default ``DEFAULT_SEARCH``, read at call time)."""
        search = _choice(search, DEFAULT_SEARCH, SEARCHES, what, "search")
        return _sampling_controls(search, temperature, top_p, self.num_hierarchies, what, ignore_temperature)

    def _capping(self, search: Optional[str], max_per_prefix: Optional[int], prefix_len: int, num_beams: Optional[int],
                 what: str):
        """The cap of a call (``_prefix_cap_controls``, then ``_search_cap`` at its beam width), checked on the host before any
        launch; search defaults to ``DEFAULT_SEARCH``, read at call time."""
        search = _choice(search, DEFAULT_SEARCH, SEARCHES, what, "search")
        cap = _prefix_cap_controls(search, max_per_prefix, prefix_len, self.num_hierarchies, what)
        if cap is None:
            return None
        k = self.top_k_for_generation if num_beams is None else int(num_beams)
        return self._search_cap(cap, search, k, min(MAX_CANDIDATES, self.num_embeddings_per_hierarchy), what)

    def _generate(self, attention_mask, input_ids, user_id, search, decoder, encoder, encoder_attention, filters: list,
                  num_beams: Optional[int] = None, warp: Optional[list] = None, cap: Optional[tuple] = None):
        decoder = _choice(decoder, DEFAULT_DECODER, DECODERS, "generate", "decoder")
        if decoder == "fused" and self.training:
            raise ValueError("generate: decoder=\"fused\" runs the decoder in eval mode only; call model.eval() first (in "
                             "training mode HF's decoder applies dropout)")
        encoder = _choice(encoder, DEFAULT_ENCODER, ENCODERS, "generate", "encoder")
        att = _encoder_attention(encoder, encoder_attention, "generate")
        if encoder == "fused" and self.training:
            raise ValueError("generate: encoder=\"fused\" runs the encoder in eval mode only; call model.eval() first (in "
                             "training mode HF's encoder applies dropout)")
        search = _choice(search, DEFAULT_SEARCH, SEARCHES, "generate", "search")
        num_beams = None if num_beams is None else int(num_beams)
        if search == "exact":
            return self._generate_exact(attention_mask, input_ids, user_id, decoder, encoder, encoder_attention, filters,
                                        num_beams)
        k = self.top_k_for_generation if num_beams is None else num_beams
        n_cands = min(MAX_CANDIDATES, self.num_embeddings_per_hierarchy)
        self._check_search_limits(search, k, n_cands, num_beams)
        if encoder == "fused":
            # "fp32" without an argument: a caller may have replaced _fused_encoder with a function of none
            fused_encoder = self._fused_encoder() if att == "fp32" else self._fused_encoder(att)
            enc_out, enc_mask = fused_encoder(attention_mask, input_ids, user_id)
        else:
            enc_out, enc_mask = self.encoder_forward_pass(attention_mask=attention_mask, input_ids=input_ids, user_id=user_id)
        generated, log_probas, reject = self._search_levels(enc_out, enc_mask, search, decoder, k, filters, warp, cap)
        self._finish_search(_counter_kind(search, warp), reject, filters)
        return generated, log_probas

    def _search_levels(self, enc_out: Tensor, enc_mask: Tensor, search: str, decoder: str, k: int, filters: list,
                       warp: Optional[list] = None, cap: Optional[tuple] = None):
        """The level loop of a "sample" or "beam" search of width k over the encoder output: (generated [B, k, H], log_probas
        [B, k], the device counters ``_finish_search`` reads).  ``warp``: the per-level (temperature, top_p) of a warped
        "sample" search (``_sampling_controls``), whose counter is the "beam" search's count of bad head rows.  ``cap``: the
        (prefix_len, max_per_prefix) of a capped search (``_search_cap``), applied at the levels h >= prefix_len."""
        n_cands = min(MAX_CANDIDATES, self.num_embeddings_per_hierarchy)
        beam = search == "beam"
        wide = not self._narrow_search(search, k, n_cands)
        index = self._prefix_index(enc_out.device)
        fused = self._fused_decoder(enc_out, enc_mask, k) if decoder == "fused" else None
        if fused is None:
            rep_enc, rep_mask = enc_out.repeat_interleave(k, dim=0), enc_mask.repeat_interleave(k, dim=0)
            past_kv = EncoderDecoderCache(DynamicCache(), DynamicCache())
        reject = torch.zeros(1 if beam or warp is not None else 2, dtype=torch.int32, device=enc_out.device)
        filt = self._filter_kwargs(filters)
        generated, log_probas, parent_global = None, None, None
        for h in range(self.num_hierarchies):
            first = generated is None
            if fused is not None:
                logits = self.decoder_mlp[h](fused.step(h, generated, parent_global))
            else:
                dec_out, past_kv = self.decoder_forward_pass(
                    future_ids=None if first else generated.reshape(-1, h), encoder_output=enc_out if first else rep_enc,
                    attention_mask_for_encoder=enc_mask if first else rep_mask, use_cache=True, past_key_values=past_kv)
                logits = self.decoder_mlp[h](dec_out[:, -1, :])
            level_cap = cap if cap is not None and h >= cap[0] else None
            if level_cap is not None:                         # a cap binds on the one-CTA kernels only (_search_cap)
                if beam:
                    generated, log_probas, parent_global = index.beam_topk(logits, generated, log_probas, k, bad=reject,
                                                                           cap=level_cap, **filt)
                elif warp is not None:
                    generated, log_probas, parent_global = self._warped_sample_and_select(
                        index, logits, generated, log_probas, k, n_cands, reject, warp[h], False, filt, level_cap)
                else:
                    generated, log_probas, parent_global = self._sample_and_select(
                        index, F.softmax(logits, dim=-1), generated, log_probas, k, n_cands, reject, cap=level_cap, **filt)
            elif beam:
                topk = index.beam_topk_wide if wide else index.beam_topk
                generated, log_probas, parent_global = topk(logits, generated, log_probas, k, bad=reject, **filt)
            elif warp is not None:
                generated, log_probas, parent_global = self._warped_sample_and_select(index, logits, generated, log_probas, k,
                                                                                      n_cands, reject, warp[h], wide, filt)
            elif wide:
                generated, log_probas, parent_global = self._sample_and_select(index, F.softmax(logits, dim=-1), generated,
                                                                               log_probas, k, n_cands, reject, wide=True, **filt)
            else:
                generated, log_probas, parent_global = self._sample_and_select(index, F.softmax(logits, dim=-1), generated,
                                                                               log_probas, k, n_cands, reject, **filt)
            if fused is not None:
                continue
            if first:
                past_kv = EncoderDecoderCache(DynamicCache(), DynamicCache())   # level 1 re-runs the decoder on B * k rows
            else:
                past_kv.reorder_cache(parent_global)
        return generated, log_probas, reject

    def _finish_search(self, search: str, reject: Tensor, filters: list) -> None:
        """The one host read after a "sample" or "beam" search's levels: its counters, then the errors they report (``search``:
        whose counters, ``_counter_kind``)."""
        if search == "beam" and not filters:
            counters = [int(reject[0])]
        else:
            counters = self._read_counters(reject, filters, "generate")
        self._raise_search_errors(search, counters)

    @staticmethod
    def _raise_search_errors(search: str, counters: List[int]) -> None:
        """The errors of a "sample" or "beam" search's counters, as read on the host."""
        if search == "beam":
            n_bad = counters[0]
            if n_bad:
                raise RuntimeError(f"generate: {n_bad} beam row(s) of the decoder head's logits hold a NaN or +inf or are all "
                                   "-inf; the beam search cannot rank them")
            return
        bad, zero_sum = counters
        if bad:
            raise RuntimeError(_MULTINOMIAL_ERRORS[0])
        if zero_sum:
            raise RuntimeError(_MULTINOMIAL_ERRORS[1])

    def _generate_exact(self, attention_mask, input_ids, user_id, decoder, encoder, encoder_attention, filters: list,
                        num_beams: Optional[int]):
        """generate(search="exact"): the bound (the beam search of width w with the call's filters and decoder, its leaves
        rescored exactly; tau[b] the w-th largest exact score when all w are finite, else -inf), then ``FusedT5Exact`` in
        chunks of histories sized by ``RANK_BYTE_BUDGET`` (a chunk whose level would not fit reruns with half its
        histories)."""
        global EXACT_DECODER_ROWS
        what = "generate(search=\"exact\")"
        encoder, att, _ = self._check_rank_call(encoder, encoder_attention, None, what)
        H, K, B = self.num_hierarchies, self.num_embeddings_per_hierarchy, attention_mask.shape[0]
        w = self.top_k_for_generation if num_beams is None else num_beams
        if not 1 <= w <= min(MAX_NUM_BEAMS, K) or K > 2048:
            raise Rqb200Error(f"{what}: num_beams = {w} with {K} codes per level is outside the exact search's limits "
                              f"(1 <= num_beams <= min({MAX_NUM_BEAMS}, K), at most 2048 codes per level)")
        _check_tuple_key(H, K, what, max_levels=8)
        dev = attention_mask.device
        levels, leaf_key, _ = self._rank_levels(dev)
        if encoder == "fused":
            packed = self._fused_encoder(att).packed(attention_mask, input_ids, user_id)
            enc_out, enc_mask = ops.t5enc_scatter(packed.rows, packed.slot), packed.enc_mask
        else:
            enc_out, enc_mask = self.encoder_forward_pass(attention_mask=attention_mask, input_ids=input_ids, user_id=user_id)
            packed = PackedEncoderOutput.of_padded(enc_out, enc_mask)
        beams, beam_lp, reject = self._search_levels(enc_out, enc_mask, "beam", decoder, w, filters)
        self._finish_search("beam", reject, filters)
        gen = torch.full((B, w, H), -1, dtype=torch.int64, device=dev)
        lp = torch.full((B, w), float("-inf"), dtype=torch.float32, device=dev)
        EXACT_DECODER_ROWS = 0
        if B == 0 or levels.n[H] == 0:
            return gen, lp
        ranker = FusedT5Exact(self, *packed.keys()[:3])
        bad = torch.zeros(1, dtype=torch.int32, device=dev)
        exact = self._score_candidates(lambda: ranker, beams, None, bad, what)
        bounded = (torch.isfinite(beam_lp) & torch.isfinite(exact)).all(1)
        tau = torch.where(bounded, exact.min(1).values, float("-inf")).contiguous()
        max_rows = max(max(levels.n[:H]), RANK_BYTE_BUDGET // FusedT5Rank.row_bytes(self))
        filt = self._filter_kwargs(filters)
        rows, b0, chunk = 0, 0, min(B, max_rows)
        while b0 < B:
            b1 = min(B, b0 + chunk)
            ran = ranker.run(b0, b1, levels, tau, w, leaf_key, filt, max_rows, gen[b0:b1], lp[b0:b1], bad)
            if ran is None:
                chunk = max(1, (b1 - b0) // 2)
                continue
            rows, b0 = rows + ran, b1
        EXACT_DECODER_ROWS = rows
        self._raise_bad(bad, what)
        return gen, lp

    def _batch_exclusion(self, batch: TokenizedSeqBatch, exclude_items, exclude_history) -> Optional[ops.SidExclusion]:
        return self._exclusion(self._excluded_items(batch, exclude_items, exclude_history), batch.sem_ids.shape[0],
                               batch.sem_ids.device)

    def _batch_filters(self, batch: TokenizedSeqBatch, exclude_items, exclude_history, include_items) -> list:
        return self._filters(self._excluded_items(batch, exclude_items, exclude_history), include_items, batch.sem_ids.shape[0],
                             batch.sem_ids.device)

    def _generate_batch(self, batch: TokenizedSeqBatch, search, decoder, encoder, encoder_attention,
                        filters: list, num_beams: Optional[int] = None, warp: Optional[list] = None,
                        cap: Optional[tuple] = None) -> GenerationOutput:
        H = self.num_hierarchies
        generated, log_probas = self._generate(_strip_dedup_col(batch.seq_mask.long(), H + 1, H),
                                               _strip_dedup_col(batch.sem_ids, H + 1, H), batch.user_ids, search, decoder,
                                               encoder, encoder_attention, filters, num_beams, warp, cap)
        return GenerationOutput(sem_ids=generated, log_probas=log_probas)

    @torch.no_grad()
    def generate_next_sem_id(self, batch: TokenizedSeqBatch, top_k: bool = True, temperature: int = 1,
                             search: Optional[str] = None, decoder: Optional[str] = None,
                             encoder: Optional[str] = None, encoder_attention: Optional[str] = None,
                             exclude_items: Optional[Tensor] = None, exclude_history: Optional[bool] = None,
                             include_items: Optional[Tensor] = None, num_beams: Optional[int] = None,
                             top_p=1.0, max_per_prefix: Optional[int] = None, prefix_len: int = 1) -> GenerationOutput:
        """``generate`` on the batch's histories.  ``exclude_items``, ``include_items``, ``num_beams``, ``temperature`` and
        ``top_p`` as in ``generate``, except that "beam" and "exact" ignore ``temperature`` (the reference ignores it for every
        search; ``top_p`` < 1 still raises with them); ``exclude_history`` (default ``DEFAULT_EXCLUDE_HISTORY``, read at call
        time) also excludes each history's own items (``history_items``).  ``max_per_prefix`` / ``prefix_len`` as in
        ``generate``.  ``top_k`` is accepted for the reference's signature."""
        warp = self._sampling(search, temperature, top_p, "generate_next_sem_id", ignore_temperature=True)
        cap = self._capping(search, max_per_prefix, prefix_len, num_beams, "generate_next_sem_id")
        return self._generate_batch(batch, search, decoder, encoder, encoder_attention,
                                    self._batch_filters(batch, exclude_items, exclude_history, include_items), num_beams, warp,
                                    cap)

    @torch.no_grad()
    def generate_items(self, batch: TokenizedSeqBatch, n: Optional[int] = None, search: Optional[str] = None,
                       decoder: Optional[str] = None, encoder: Optional[str] = None,
                       encoder_attention: Optional[str] = None, exclude_items: Optional[Tensor] = None,
                       exclude_history: Optional[bool] = None, include_items: Optional[Tensor] = None,
                       num_beams: Optional[int] = None, temperature=1.0, top_p=1.0, max_per_prefix: Optional[int] = None,
                       prefix_len: int = 1) -> ItemGenerationOutput:
        """The top corpus items for each history: ``generate_next_sem_id``'s beams, unchanged, then one launch that takes the
        items of every finite beam whose ids are in the corpus, beam by beam in descending score order, each beam's items by
        dedup rank, no item twice, at most n (default: the call's beam width, ``num_beams`` or else top_k_for_generation; at
        most ``ops.SidItemTable.MAX_N``) per history.  ``exclude_items`` / ``exclude_history`` as in
        ``generate_next_sem_id``: the search and the retrieval both leave the excluded items out.  ``include_items`` as in
        ``generate``: the search and the retrieval both return only each history's eligible items.  ``num_beams`` as in
        ``generate``: a wider search yields more candidate items (``n`` up to 4096).  ``temperature`` / ``top_p`` and
        ``max_per_prefix`` / ``prefix_len`` as in ``generate``: with a cap, the items come from the capped beams only."""
        warp = self._sampling(search, temperature, top_p, "generate_items")
        cap = self._capping(search, max_per_prefix, prefix_len, num_beams, "generate_items")
        filters = self._batch_filters(batch, exclude_items, exclude_history, include_items)
        out = self._generate_batch(batch, search, decoder, encoder, encoder_attention, filters, num_beams, warp, cap)
        table = self._item_table(out.sem_ids.device)
        width = self.top_k_for_generation if num_beams is None else num_beams
        items, beams, count = table.retrieve(out.sem_ids, out.log_probas, width if n is None else n,
                                             **self._filter_kwargs(filters))
        return ItemGenerationOutput(item_ids=items, beams=beams, count=count, sem_ids=out.sem_ids, log_probas=out.log_probas)

    def capture_generate_items(self, batch: TokenizedSeqBatch, n: Optional[int] = None, search: Optional[str] = None,
                               num_beams: Optional[int] = None, encoder_attention: Optional[str] = None,
                               exclude_items: Optional[Tensor] = None, exclude_history: Optional[bool] = None,
                               include_items: Optional[Tensor] = None, encoder: str = "fused",
                               decoder: str = "fused", temperature=1.0, top_p=1.0, max_per_prefix: Optional[int] = None,
                               prefix_len: int = 1) -> "GenerateItemsGraph":
        """``generate_items(batch, ..., encoder="fused", decoder="fused")`` captured as one CUDA graph, for serving: calling the
        returned ``GenerateItemsGraph`` with a batch of the same shapes is one graph replay and one host read of the error
        counters.  The example batch fixes every shape: B, the history width, whether ``user_ids`` is given, and the widths of
        ``exclude_items`` / ``include_items`` (and whether each is given).  ``search`` is "sample" or "beam" at any width those
        searches take; ``search``, ``n``, ``num_beams``, ``encoder_attention``, ``exclude_history``, ``temperature``,
        ``top_p``, ``max_per_prefix`` and ``prefix_len`` are read once, here, with ``generate_items``' defaults and checks.  Raises ``ValueError`` for search="exact" (one host read per level), an HF encoder or
        decoder, training mode and an active autocast region.  See ``GenerateItemsGraph`` for what a replay follows."""
        return GenerateItemsGraph(self, batch, n, search, num_beams, encoder_attention, exclude_items, exclude_history,
                                  include_items, encoder, decoder, temperature, top_p, max_per_prefix, prefix_len)

    def capture_exact_items(self, batch: TokenizedSeqBatch, n: Optional[int] = None, num_beams: Optional[int] = None,
                            max_rows: Optional[int] = None, encoder_attention: Optional[str] = None,
                            exclude_items: Optional[Tensor] = None, exclude_history: Optional[bool] = None,
                            include_items: Optional[Tensor] = None) -> "ExactItemsGraph":
        """``generate_items(batch, ..., search="exact", encoder="fused", decoder="fused")`` captured as one CUDA graph, for serving
        exact top-w results: calling the returned ``ExactItemsGraph`` with a batch of the same shapes is one graph replay and one
        host read.  The example batch fixes every shape, as ``capture_generate_items``.  ``n``, ``num_beams``,
        ``encoder_attention``, ``exclude_history`` are read once, here, with ``generate_items``' defaults, limits and errors.
        ``max_rows`` bounds the decoder rows of one pruned level (default: ``RANK_BYTE_BUDGET`` bytes of decoder state, the eager
        search's budget; the graph holds that memory while it lives).  A batch whose frontier exceeds it is answered by the eager
        search (``ExactItemsGraph.fallbacks``).  Raises ``ValueError`` in training mode and in an active autocast region, before
        any launch.  See ``ExactItemsGraph`` for what a replay follows."""
        return ExactItemsGraph(self, batch, n, num_beams, max_rows, encoder_attention, exclude_items, exclude_history, include_items)

    @torch.no_grad()
    def item_of(self, sem_ids_fut: Tensor) -> Tensor:
        """int64 [B]: the corpus item of each row of ``TokenizedSeqBatch.sem_ids_fut`` (its H ids and the dedup column), -1
        when the tuple is not in the corpus or the dedup rank exceeds its items."""
        H = self.num_hierarchies
        return self._item_table(sem_ids_fut.device).lookup(sem_ids_fut[:, :H + 1], with_dedup=True)

    # ------------------------------------------------------------------------------------------------ exact ranking
    def _rank_levels(self, device: torch.device):
        """(trie levels, leaf keys int64 [U], retrievable items) of the prefix index, built once per index and cached on it.  The
        node counts and the item count are read on the host here, in one read.  The leaves of level H are the item table's U
        tuples in the same (lexicographic) order: both hold the distinct tuples of the rows whose first H ids are in [0, K)."""
        index = self._prefix_index(device)
        H, K = self.num_hierarchies, self.num_embeddings_per_hierarchy
        state = getattr(index, "_rank_state", None)
        if state is None or state[0] != H:
            if index.C < H:
                raise Rqb200Error(f"rank_sem_ids: the corpus table has {index.C} id columns, fewer than {H} levels")
            _check_tuple_key(H, K, "rank_sem_ids")
            cb = self.codebooks[:, :H].to(device)
            n_items = ((cb >= 0) & (cb < K)).all(1).sum()
            host = torch.cat([index.counts().long(), n_items.view(1)]).tolist()   # the one host read of the ranking
            levels = index.levels(host[:-1])
            key = levels.code[1].long()                                           # _tuple_key of each leaf, along its path
            for l in range(2, H + 1):
                key = key[levels.parent[l].long()] * K + levels.code[l]
            state = index._rank_state = (H, levels, key, int(host[-1]), ops.StreamBuild(key))
        state[4].ready()
        return state[1:4]

    def _leaf_of(self, tuples: Tensor, leaf_key: Tensor) -> Tensor:
        """int64 [B]: the leaf (item-table tuple) of each row of tuples [B, H], -1 when it holds an id outside [0, K) or is not in
        the corpus."""
        K, U = self.num_embeddings_per_hierarchy, leaf_key.shape[0]
        t = tuples.long()
        if U == 0:
            return torch.full((t.shape[0],), -1, dtype=torch.int64, device=t.device)
        valid = ((t >= 0) & (t < K)).all(1)
        key = _tuple_key(t, K)
        idx = torch.searchsorted(leaf_key, key).clamp_(max=U - 1)
        return torch.where(valid & (leaf_key[idx] == key), idx, -1)

    def _check_rank_call(self, encoder, encoder_attention, attention, what: str):
        """(encoder, its attention, the decoder's cross-attention) of an exact-scoring call, after its mode checks."""
        if self.training:
            raise ValueError(f"{what} runs the model in eval mode only; call model.eval() first (in training mode HF's passes "
                             "apply dropout)")
        _check_no_autocast(what)
        encoder = _choice(encoder, DEFAULT_ENCODER, ENCODERS, what, "encoder")
        att = _encoder_attention(encoder, encoder_attention, what)
        return encoder, att, _choice(attention, "fp32", ENCODER_ATTENTIONS, what, "attention")

    def _rank_encoder(self, attention_mask, input_ids, user_id, encoder: str, att: str):
        """The encoder rows the exact scoring attends to: (rows [*, d_model], offsets int32 [B + 1], additive key mask [*])."""
        if encoder == "fused":
            enc = self._fused_encoder(att).packed(attention_mask, input_ids, user_id)
        else:
            enc = PackedEncoderOutput.of_padded(*self.encoder_forward_pass(attention_mask=attention_mask, input_ids=input_ids,
                                                                           user_id=user_id))
        return enc.keys()[:3]

    def _row_budget(self, max_rows: Optional[int], per_history: int, what: str) -> int:
        """Most decoder rows one chunk of histories runs: ``max_rows`` (at least one history's), else what ``RANK_BYTE_BUDGET``
        bytes of decoder state hold."""
        if max_rows is None:
            return max(per_history, RANK_BYTE_BUDGET // FusedT5Rank.row_bytes(self))
        if max_rows < per_history:
            raise ValueError(f"{what}: max_rows = {max_rows} is below the {per_history} decoder rows of one history")
        return max_rows

    def _leaf_scores(self, attention_mask, input_ids, user_id, encoder, encoder_attention, attention, max_rows, what: str):
        encoder, att, attention = self._check_rank_call(encoder, encoder_attention, attention, what)
        dev = attention_mask.device
        levels, leaf_key, n_items = self._rank_levels(dev)
        H, B = self.num_hierarchies, attention_mask.shape[0]
        U = levels.n[H]
        per_history = sum(levels.n[:H])
        max_rows = self._row_budget(max_rows, per_history, what)
        bad = torch.zeros(1, dtype=torch.int32, device=dev)
        scores = torch.empty((B, U), dtype=torch.float32, device=dev)
        if B == 0 or U == 0:
            return scores, bad, leaf_key, n_items
        ranker = FusedT5Rank(self, *self._rank_encoder(attention_mask, input_ids, user_id, encoder, att), attention)
        chunk = max_rows // per_history
        for b0 in range(0, B, chunk):
            ranker.run(b0, min(B, b0 + chunk), levels, scores, bad)
        return scores, bad, leaf_key, n_items

    @staticmethod
    def _raise_bad(bad: Tensor, what: str) -> None:
        n_bad = int(bad[0])
        if n_bad:
            raise _non_finite_error(what, n_bad)

    @torch.no_grad()
    def rank_sem_ids(self, attention_mask, input_ids, user_id=None, encoder: Optional[str] = None,
                     encoder_attention: Optional[str] = None, attention: Optional[str] = None,
                     max_rows: Optional[int] = None) -> Tensor:
        """fp32 [B, U]: the exact log-probability of every retrievable corpus tuple (U distinct tuples, in the item table's
        lexicographic order) for each history: sum over levels of log_softmax(decoder_mlp[h](dec_h))[c_h], with the per-row
        log-sum-exp of the beam search.  One decoder row per corpus-trie node per history (``FusedT5Rank``), histories in chunks of
        at most ``max_rows`` decoder rows (default: ``RANK_BYTE_BUDGET`` bytes of decoder state); chunking does not change a bit.
        ``encoder`` / ``encoder_attention`` as in ``generate``; ``attention`` the cross-attention's precision: "fp32" (default) or
        "tf32" (its products on the TF32 tensor cores).  The GEMMs are fp32-accurate whatever torch's matmul precision.  Eval mode only, no autocast, no random draws.  Raises
        ``RuntimeError`` after the pass when some head row was not finite (its items score NaN).  An evaluation tool: it runs a
        decoder row per trie node, thousands of times ``generate``'s work."""
        scores, bad, _, _ = self._leaf_scores(attention_mask, input_ids, user_id, encoder, encoder_attention, attention,
                                               max_rows, "rank_sem_ids")
        self._raise_bad(bad, "rank_sem_ids")
        return scores

    @torch.no_grad()
    def rank_items(self, batch: TokenizedSeqBatch, n: Optional[int] = None, encoder: Optional[str] = None,
                   encoder_attention: Optional[str] = None, attention: Optional[str] = None,
                   max_rows: Optional[int] = None, exclude_items: Optional[Tensor] = None,
                   exclude_history: Optional[bool] = None) -> ItemRankingOutput:
        """Every retrievable corpus item ranked for each history by the model's exact log-probability (``rank_sem_ids``): the n
        best (default top_k_for_generation, at most ``MAX_RANK_ITEMS``) and the rank of ``item_of(batch.sem_ids_fut)``.  Order:
        score descending, then tuple (lexicographic), then dedup rank; NaN last.  One selection launch after the decoder.
        ``exclude_items`` / ``exclude_history`` as in ``generate_next_sem_id``: excluded items are not returned and the target's
        rank counts only the items that are not excluded (-1 when the target itself is excluded), the masked full-ranking
        protocol; ``num_items`` stays the corpus's count."""
        n = self.top_k_for_generation if n is None else int(n)
        if not 1 <= n <= MAX_RANK_ITEMS:
            raise ValueError(f"rank_items: n = {n} must be in [1, {MAX_RANK_ITEMS}]")
        H = self.num_hierarchies
        exclusion = self._batch_exclusion(batch, exclude_items, exclude_history)
        scores, bad, leaf_key, n_items = self._leaf_scores(
            _strip_dedup_col(batch.seq_mask.long(), H + 1, H), _strip_dedup_col(batch.sem_ids, H + 1, H), batch.user_ids,
            encoder, encoder_attention, attention, max_rows, "rank_items")
        fut = batch.sem_ids_fut
        row, start = self._item_table(scores.device).arrays()
        items, item_scores, rank = ops.t5rank_select(scores, row, start, self._leaf_of(fut[:, :H], leaf_key), fut[:, H], n,
                                                     exclude=exclusion)
        if exclusion is None:
            self._raise_bad(bad, "rank_items")
        else:
            n_bad, = self._read_counters(bad, [exclusion], "rank_items")
            if n_bad:
                raise _non_finite_error("rank_items", n_bad)
        return ItemRankingOutput(item_ids=items, scores=item_scores, target_rank=rank, num_items=n_items)

    # ------------------------------------------------------------------------------------------------ scoring given items
    def _candidate_scores(self, attention_mask, input_ids, user_id, sem_ids: Tensor, encoder, encoder_attention, attention,
                          max_rows, bad: Tensor, what: str) -> Tensor:
        """fp32 [B, C]: each candidate tuple's exact log-probability, decoding per history the trie of its own candidates
        (``ops.t5score_trie_build``, ``FusedT5Rank.run_candidates``); NaN-row counts are added to bad[0]."""
        encoder, att, attention = self._check_rank_call(encoder, encoder_attention, attention, what)
        H, K = self.num_hierarchies, self.num_embeddings_per_hierarchy
        _check_tuple_key(H, K, what, max_levels=8)
        B = attention_mask.shape[0]
        if sem_ids.dim() != 3 or sem_ids.shape[0] != B or sem_ids.shape[2] != H:
            raise ValueError(f"{what}: sem_ids {tuple(sem_ids.shape)} must be [B = {B}, C, H = {H}]")
        C = sem_ids.shape[1]
        if not 1 <= C <= ops.SCORE_MAX_CANDIDATES:
            raise ValueError(f"{what}: C = {C} candidates per history must be in [1, {ops.SCORE_MAX_CANDIDATES}]")
        return self._score_candidates(
            lambda: FusedT5Rank(self, *self._rank_encoder(attention_mask, input_ids, user_id, encoder, att), attention), sem_ids,
            max_rows, bad, what)

    def _score_candidates(self, make_ranker, sem_ids: Tensor, max_rows, bad: Tensor, what: str) -> Tensor:
        """fp32 [B, C]: the candidate tuples sem_ids [B, C, H] scored on the ranker ``make_ranker()`` returns (built once the
        tries are, and only when there are histories)."""
        H, K = self.num_hierarchies, self.num_embeddings_per_hierarchy
        B, C = sem_ids.shape[0], sem_ids.shape[1]
        trie = ops.t5score_trie_build(sem_ids, K)
        need = [[1] + [max(1, c) for c in row] for row in _read_node_counts(trie.counts)]   # rows per level, n[0] = 1 (BOS)
        max_rows = self._row_budget(max_rows, max((sum(n[:H]) for n in need), default=0), what)
        scores = torch.empty((B, C), dtype=torch.float32, device=sem_ids.device)
        if B == 0:
            return scores
        chunks, b0 = [], 0                  # histories in order, each chunk as long as its padded levels fit in max_rows
        while b0 < B:
            n, b1 = need[b0], b0 + 1
            while b1 < B:
                wider = [max(a, c) for a, c in zip(n, need[b1])]
                if (b1 + 1 - b0) * sum(wider[:H]) > max_rows:
                    break
                n, b1 = wider, b1 + 1
            chunks.append((b0, b1, n))
            b0 = b1
        ranker = make_ranker()
        for b0, b1, n in chunks:
            ranker.run_candidates(b0, b1, n, trie, scores, bad)
        return scores

    @staticmethod
    def _raise_score_errors(counters: Tensor, what: str) -> None:
        """The one host read at the end of score_sem_ids / score_items: counters[0] the head rows that were not finite,
        counters[1] the item ids outside [-1, N)."""
        n_bad, n_items = counters.tolist()
        if n_items:
            raise ValueError(f"{what}: {n_items} item id(s) outside [-1, N) where N is the number of corpus rows")
        if n_bad:
            raise _non_finite_error(what, n_bad)

    @torch.no_grad()
    def score_sem_ids(self, attention_mask, input_ids, user_id=None, sem_ids: Optional[Tensor] = None,
                      encoder: Optional[str] = None, encoder_attention: Optional[str] = None, attention: Optional[str] = None,
                      max_rows: Optional[int] = None) -> Tensor:
        """fp32 [B, C]: the exact log-probability of each of the C candidate tuples (sem_ids integer [B, C, H]) of each history,
        the quantity ``rank_sem_ids`` gives a corpus tuple (the same kernels, the same log-sum-exp, bit for bit).  A tuple whose
        ids are all in [0, K) is scored whether or not the corpus holds it; one holding an id outside [0, K) (-1 pads ragged
        candidate lists) scores -inf; equal tuples score the same.  Each history decodes the trie of its own candidates, one decoder
        row per node: at most 1 + C (H - 1) rows per history.  ``encoder``, ``encoder_attention``, ``attention`` and ``max_rows``
        as in ``rank_sem_ids``; C <= ``ops.SCORE_MAX_CANDIDATES``.  Two host reads: the tries' node counts after their build, and
        the non-finite row count at the end (``RuntimeError`` when some head row was not finite)."""
        if sem_ids is None:
            raise ValueError("score_sem_ids: sem_ids [B, C, H] is required")
        counters = torch.zeros(2, dtype=torch.int32, device=attention_mask.device)
        scores = self._candidate_scores(attention_mask, input_ids, user_id, sem_ids, encoder, encoder_attention, attention,
                                        max_rows, counters, "score_sem_ids")
        self._raise_score_errors(counters, "score_sem_ids")
        return scores

    @torch.no_grad()
    def score_items(self, batch: TokenizedSeqBatch, item_ids: Tensor, encoder: Optional[str] = None,
                    encoder_attention: Optional[str] = None, attention: Optional[str] = None,
                    max_rows: Optional[int] = None) -> ItemScoreOutput:
        """The exact log-probability of given corpus items (item_ids int64 [B, C], corpus rows, -1 pads) for each history,
        through their tuples codebooks[item, :H] (``score_sem_ids``), and the position of ``item_of(batch.sem_ids_fut)`` among the
        row's items in ``rank_items``' order: score descending, then tuple, then item id (dedup order), NaN last; -1 when the
        target is not among them.  With the target among C sampled items, ``TopKAccumulator.accumulate_ranks(target_rank, C)``
        gives the sampled-candidate metrics.  Item ids outside [-1, N) are counted on the device and raise ``ValueError`` after
        the pass; the host reads are those of ``score_sem_ids``."""
        ops._need_cuda(item_ids)
        H, K = self.num_hierarchies, self.num_embeddings_per_hierarchy
        B = batch.sem_ids.shape[0]
        if item_ids.dim() != 2 or item_ids.shape[0] != B or item_ids.dtype.is_floating_point or item_ids.dtype == torch.bool:
            raise ValueError(f"score_items: item_ids must be an integer [B = {B}, C] tensor, got {item_ids.dtype} "
                             f"{tuple(item_ids.shape)}")
        items = item_ids.long()
        cb = self.codebooks[:, :H].to(items.device).long()
        N = cb.shape[0]
        ok = (items >= 0) & (items < N)
        counters = torch.zeros(2, dtype=torch.int32, device=items.device)
        counters[1:] = (~ok & (items != -1)).sum().view(1)
        tuples = torch.where(ok[..., None], cb[items.clamp(0, max(N - 1, 0))], -1)
        scores = self._candidate_scores(
            _strip_dedup_col(batch.seq_mask.long(), H + 1, H), _strip_dedup_col(batch.sem_ids, H + 1, H), batch.user_ids, tuples,
            encoder, encoder_attention, attention, max_rows, counters, "score_items")
        target = self.item_of(batch.sem_ids_fut)[:, None]
        key = _tuple_key(tuples, K)
        match = ok & (items == target)
        pos = match.int().argmax(1, keepdim=True)
        s_t, key_t = scores.gather(1, pos), key.gather(1, pos)
        nan, nan_t = scores.isnan(), s_t.isnan()
        tie = (scores == s_t) | (nan & nan_t)
        before = ok & ((~nan & nan_t) | (scores > s_t) | (tie & ((key < key_t) | ((key == key_t) & (items < target)))))
        rank = torch.where(match.any(1), before.sum(1), -1)
        self._raise_score_errors(counters, "score_items")
        return ItemScoreOutput(scores=scores, target_rank=rank)


_EXACT = "generate(search=\"exact\")"


def _counter_kind(search: str, warp: Optional[list]) -> str:
    """Whose counters and errors a "sample" or "beam" search reports: a warped "sample" search counts bad head rows as "beam"
    does (it reads the logits, not a softmax ``torch.multinomial`` would check)."""
    return "beam" if warp is not None else search


def _read_search_counters(values: Tensor) -> List[int]:
    """The one host read of a ``GenerateItemsGraph`` call, after its replay: the search's counters, then each filter's count of
    ids outside [-1, N) (``EncoderDecoderRetrievalModel._counter_values``)."""
    return values.tolist()


def _input_spec(t: Optional[Tensor]):
    return None if t is None else (tuple(t.shape), t.dtype, t.device)


class GenerateItemsGraph:
    """One ``generate_items(..., encoder="fused", decoder="fused")`` call captured as a CUDA graph
    (``EncoderDecoderRetrievalModel.capture_generate_items``).  ``graph(batch, exclude_items=None, include_items=None)`` copies
    ``batch.sem_ids``, ``batch.seq_mask``, ``batch.user_ids`` and the item lists into the graph's static buffers, replays the
    graph on the current stream, reads the counters once and returns an ``ItemGenerationOutput`` of new tensors (a later call
    does not overwrite them).  Inputs must match the captured ones in shape, dtype, device and presence, else ``ValueError``
    before any launch: pad histories with masked rows and shorter histories with mask zeros, as ``SeqData`` does.
      * Results: the eager call's on the same inputs, with the decoder at the eager B * w rows.  The encoder runs at a fixed
        capacity of B * S packed rows (``FusedT5Encode(capacity=True)``, no host read of N): with every position unmasked it is
        the eager pass; with padding its GEMMs run B * S rows instead of N, which changes only their rounding.  "sample" draws
        its noise from torch's CUDA generator through the graph-safe Philox offsets, so consecutive replays consume the generator
        as consecutive eager calls do.  Capturing leaves the generator's state as it found it.
      * Weights: a replay reads the live parameters (the q|k|v and cross k|v concatenations are copies inside the graph), so an
        in-place update (``optimizer.step()``, ``load_state_dict``) is followed without recapture.  A parameter whose storage
        moved (``model.to``, a replaced tensor) makes the next call recapture.
      * Corpus: the graph bakes in the prefix index, the item table and the trie levels; when the ``codebooks`` buffer is
        replaced, written to or moved, the next call recaptures before replaying.
      * Errors: the eager ``RuntimeError``s (non-finite head rows, rows ``torch.multinomial`` rejects) and ``ValueError`` (filter
        ids outside [-1, N)) with the same texts, from the one host read after the replay (``_read_search_counters``).
      * Streams: capture and replay order with the caller's current stream (capture runs on torch's side stream when that is
        the default stream, which cannot capture)."""

    def __init__(self, model: EncoderDecoderRetrievalModel, batch: TokenizedSeqBatch, n: Optional[int], search: Optional[str],
                 num_beams: Optional[int], encoder_attention: Optional[str], exclude_items: Optional[Tensor],
                 exclude_history: Optional[bool], include_items: Optional[Tensor], encoder: str = "fused",
                 decoder: str = "fused", temperature=1.0, top_p=1.0, max_per_prefix: Optional[int] = None,
                 prefix_len: int = 1):
        what = "capture_generate_items"
        if encoder != "fused" or decoder != "fused":
            raise ValueError(f"{what}: a CUDA graph runs the fused encoder and decoder only (encoder={encoder!r}, "
                             f"decoder={decoder!r}); HF's passes are host-driven")
        self._check_mode(model, what)
        self.search = _choice(search, DEFAULT_SEARCH, SEARCHES, what, "search")
        #: the per-level (temperature, top_p) of a warped "sample" search, fixed at capture (None: untempered)
        self.warp = _sampling_controls(self.search, temperature, top_p, model.num_hierarchies, what)
        if self.search == "exact" and max_per_prefix is not None:
            _prefix_cap_controls(self.search, max_per_prefix, prefix_len, model.num_hierarchies, what)
        if self.search == "exact":
            raise ValueError(f"{what}: search=\"exact\" reads its frontier's size on the host once per level; it cannot be "
                             "captured here (use \"sample\" or \"beam\", or capture_exact_items for the exact search)")
        self.attention = _encoder_attention("fused", encoder_attention, what)
        self.k = model.top_k_for_generation if num_beams is None else int(num_beams)
        n_cands = min(MAX_CANDIDATES, model.num_embeddings_per_hierarchy)
        model._check_search_limits(self.search, self.k, n_cands, None if num_beams is None else self.k)
        #: the (prefix_len, max_per_prefix) of a capped search, fixed at capture (None: uncapped, or a cap that cannot bind)
        self.cap = model._capping(self.search, max_per_prefix, prefix_len, num_beams, what)
        self.n = self.k if n is None else int(n)
        self.exclude_history = DEFAULT_EXCLUDE_HISTORY if exclude_history is None else bool(exclude_history)
        self._store(model, batch, exclude_items, include_items, what)

    def _store(self, model: EncoderDecoderRetrievalModel, batch: TokenizedSeqBatch, exclude_items: Optional[Tensor],
               include_items: Optional[Tensor], what: str) -> None:
        """Keep the example inputs' specs and static copies, then capture."""
        self.model = model
        self.device = model.device
        inputs = (batch.sem_ids, batch.seq_mask, batch.user_ids, exclude_items, include_items)
        for t in inputs:
            if t is not None and t.device != self.device:
                raise ValueError(f"{what}: every input must be on the model's device {self.device}, got {t.device}")
        self._spec = tuple(_input_spec(t) for t in inputs)
        self._static = tuple(None if t is None else t.clone() for t in inputs)
        self._graph = None
        self._capture()

    @staticmethod
    def _check_mode(model: EncoderDecoderRetrievalModel, what: str) -> None:
        if model.training:
            raise ValueError(f"{what}: the fused passes run in eval mode only; call model.eval() first")
        _check_no_autocast(what)

    def _state_key(self):
        """What the captured graph bakes in: the corpus (the prefix index's cache key) and every parameter's storage."""
        cb = self.model.codebooks
        return (id(cb), cb._version, cb.device), tuple(p.data_ptr() for p in self.model.parameters())

    def _run(self):
        """The captured work on the static inputs: (outputs, the device counters, the counter count, the filters)."""
        m, H = self.model, self.model.num_hierarchies
        sem, seq, users, exclude_items, include_items = self._static
        batch = TokenizedSeqBatch(user_ids=users, sem_ids=sem, sem_ids_fut=None, seq_mask=seq, token_type_ids=None,
                                  token_type_ids_fut=None)
        filters = m._batch_filters(batch, exclude_items, self.exclude_history, include_items)
        enc_out, enc_mask = FusedT5Encode(m, self.attention, capacity=True)(
            _strip_dedup_col(seq.long(), H + 1, H), _strip_dedup_col(sem, H + 1, H), users)
        generated, log_probas, reject = m._search_levels(enc_out, enc_mask, self.search, "fused", self.k, filters, self.warp,
                                                         self.cap)
        items, beams, count = m._item_table(sem.device).retrieve(generated, log_probas, self.n, **m._filter_kwargs(filters))
        out = ItemGenerationOutput(item_ids=items, beams=beams, count=count, sem_ids=generated, log_probas=log_probas)
        return out, m._counter_values(reject, filters), reject.numel(), filters

    @torch.no_grad()
    def _capture(self) -> None:
        """Warm up on the capture stream (module loads, cuBLAS handles, the corpus caches and their host reads), restore the
        generator, capture."""
        self._graph = self._captured = self._key = None       # the previous graph's memory goes back before the new capture
        dev = self.device
        caller = torch.cuda.current_stream(dev)
        stream = caller if caller != torch.cuda.default_stream(dev) else torch.cuda.Stream(dev)
        stream.wait_stream(caller)
        rng = torch.cuda.get_rng_state(dev)
        with torch.cuda.stream(stream):
            self._run()
        torch.cuda.set_rng_state(rng, dev)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            captured = self._run()
        caller.wait_stream(stream)
        self._graph, self._captured, self._key = graph, captured, self._state_key()

    def _check_inputs(self, batch: TokenizedSeqBatch, exclude_items: Optional[Tensor], include_items: Optional[Tensor]):
        inputs = (batch.sem_ids, batch.seq_mask, batch.user_ids, exclude_items, include_items)
        names = ("batch.sem_ids", "batch.seq_mask", "batch.user_ids", "exclude_items", "include_items")
        for name, t, spec in zip(names, inputs, self._spec):
            if _input_spec(t) != spec:
                want = "None" if spec is None else f"{spec[1]} {list(spec[0])} on {spec[2]}"
                got = "None" if t is None else f"{t.dtype} {list(t.shape)} on {t.device}"
                raise ValueError(f"{type(self).__name__}: {name} must match the captured call ({want}), got {got}")
        return inputs

    def _replay(self, batch: TokenizedSeqBatch, exclude_items: Optional[Tensor], include_items: Optional[Tensor]) -> None:
        """Check the inputs, copy them into the static buffers, recapture when the corpus or a parameter moved, replay."""
        self._check_mode(self.model, type(self).__name__)
        inputs = self._check_inputs(batch, exclude_items, include_items)
        for dst, src in zip(self._static, inputs):
            if dst is not None:
                dst.copy_(src)
        if self._state_key() != self._key:
            self._capture()
        self._graph.replay()

    @torch.no_grad()
    def __call__(self, batch: TokenizedSeqBatch, exclude_items: Optional[Tensor] = None,
                 include_items: Optional[Tensor] = None) -> ItemGenerationOutput:
        self._replay(batch, exclude_items, include_items)
        out, values, n_counters, filters = self._captured
        counters = EncoderDecoderRetrievalModel._check_filter_counts(_read_search_counters(values), n_counters, filters,
                                                                     "generate")
        EncoderDecoderRetrievalModel._raise_search_errors(_counter_kind(self.search, self.warp), counters)
        return ItemGenerationOutput(*(t.clone() for t in out))


class ExactItemsGraph(GenerateItemsGraph):
    """One ``generate_items(..., search="exact", encoder="fused", decoder="fused")`` call captured as a CUDA graph
    (``EncoderDecoderRetrievalModel.capture_exact_items``).  Calls, input checks, static buffers, recapture rules, streams and
    caller-owned results are ``GenerateItemsGraph``'s; what differs is what the graph runs and what its one read returns.
      * The graph: the encoder at a fixed capacity (``FusedT5Encode(capacity=True)``), the width-w beam search of the bound, its
        rescoring over each history's candidate trie at fixed level sizes [1, min(w, K), min(w, K^2), ...], and the pruned decode
        of the whole batch as one chunk at fixed capacities (``FusedT5Exact.run_capacity``): pruned level l holds at most
        R_l = min(B n_l, max_rows) decoder rows, n_l the corpus trie's nodes at level l.  No launch reads a count on the host.
      * Results: the eager call's on the same inputs, bit for bit with unpadded histories; with padded histories the encoder's
        GEMMs run B * S rows instead of N, which changes only their rounding (as ``GenerateItemsGraph``).
      * Overflow: a replay whose frontier exceeds a level's capacity is not returned.  The call runs the eager exact search on
        the same inputs instead, returns its result and counts the event in ``fallbacks``.
      * The one read after the replay (``_read_search_counters``): the bound's beam counters and the filters' id counts (the
        eager errors, with the eager texts), the non-finite head rows (the eager ``RuntimeError``), the overflow flag and the
        decoder rows the replay ran, kept in ``rows`` (as ``EXACT_DECODER_ROWS``: the pruned decode's rows, level 0 included).
      * What a replay follows: in-place weight updates, without recapture; a replaced, written or moved ``codebooks`` buffer
        recaptures before the next replay.  The exact search draws no random numbers: the generator is never touched.
      * Memory: the graph holds the decoder state of max_rows rows (default ``RANK_BYTE_BUDGET`` bytes of it, the eager search's
        budget) plus each level's buffers at its capacity, for as long as it lives."""

    def __init__(self, model: EncoderDecoderRetrievalModel, batch: TokenizedSeqBatch, n: Optional[int] = None,
                 num_beams: Optional[int] = None, max_rows: Optional[int] = None, encoder_attention: Optional[str] = None,
                 exclude_items: Optional[Tensor] = None, exclude_history: Optional[bool] = None,
                 include_items: Optional[Tensor] = None):
        what = "capture_exact_items"
        self._check_mode(model, what)
        self.search, self.warp = "exact", None
        self.attention = _encoder_attention("fused", encoder_attention, what)
        H, K = model.num_hierarchies, model.num_embeddings_per_hierarchy
        self.k = model.top_k_for_generation if num_beams is None else int(num_beams)
        if not 1 <= self.k <= min(MAX_NUM_BEAMS, K) or K > 2048:
            raise Rqb200Error(f"{_EXACT}: num_beams = {self.k} with {K} codes per level is outside the exact search's limits "
                              f"(1 <= num_beams <= min({MAX_NUM_BEAMS}, K), at most 2048 codes per level)")
        _check_tuple_key(H, K, _EXACT, max_levels=8)
        if max_rows is not None and (isinstance(max_rows, bool) or int(max_rows) != max_rows or max_rows < 1):
            raise ValueError(f"{what}: max_rows = {max_rows!r} must be a positive integer")
        #: most decoder rows of one pruned level (None: RANK_BYTE_BUDGET bytes of decoder state, at least the trie's widest level)
        self.max_rows = None if max_rows is None else int(max_rows)
        self.n = self.k if n is None else int(n)
        self.exclude_history = DEFAULT_EXCLUDE_HISTORY if exclude_history is None else bool(exclude_history)
        #: replays that overflowed a capacity and were answered by the eager search
        self.fallbacks = 0
        #: decoder rows the last replay ran (None before the first call)
        self.rows = None
        self._store(model, batch, exclude_items, include_items, what)

    def _run(self):
        m, H, K = self.model, self.model.num_hierarchies, self.model.num_embeddings_per_hierarchy
        sem, seq, users, exclude_items, include_items = self._static
        batch = TokenizedSeqBatch(user_ids=users, sem_ids=sem, sem_ids_fut=None, seq_mask=seq, token_type_ids=None,
                                  token_type_ids_fut=None)
        filters = m._batch_filters(batch, exclude_items, self.exclude_history, include_items)
        filt = m._filter_kwargs(filters)
        dev, B, w = sem.device, sem.shape[0], self.k
        levels, leaf_key, _ = m._rank_levels(dev)
        packed = FusedT5Encode(m, self.attention, capacity=True).packed(_strip_dedup_col(seq.long(), H + 1, H),
                                                                        _strip_dedup_col(sem, H + 1, H), users)
        beams, beam_lp, reject = m._search_levels(ops.t5enc_scatter(packed.rows, packed.slot), packed.enc_mask, "beam", "fused",
                                                  w, filters)
        gen = torch.full((B, w, H), -1, dtype=torch.int64, device=dev)
        lp = torch.full((B, w), float("-inf"), dtype=torch.float32, device=dev)
        bad, overflow, rows = (torch.zeros(1, dtype=torch.int32, device=dev) for _ in range(3))
        if B and levels.n[H]:
            # rows past N (src -1) belong to no history's key range: any history's mask does for them
            key_mask = packed.key_mask.index_select(0, torch.div(packed.src.clamp(min=0), packed.S, rounding_mode="floor").long())
            ranker = FusedT5Exact(m, packed.rows, packed.offsets, key_mask)
            exact = torch.empty((B, w), dtype=torch.float32, device=dev)
            ranker.run_candidates(0, B, [1] + [min(w, K ** h) for h in range(1, H + 1)], ops.t5score_trie_build(beams, K), exact,
                                  bad)
            bounded = (torch.isfinite(beam_lp) & torch.isfinite(exact)).all(1)
            tau = torch.where(bounded, exact.min(1).values, float("-inf")).contiguous()
            max_rows = self.max_rows or max(max(levels.n[:H]), RANK_BYTE_BUDGET // FusedT5Rank.row_bytes(m))
            rows = ranker.run_capacity(levels, tau, w, leaf_key, filt, max_rows, gen, lp, bad, overflow)
        items, item_beams, count = m._item_table(dev).retrieve(gen, lp, self.n, **filt)
        out = ItemGenerationOutput(item_ids=items, beams=item_beams, count=count, sem_ids=gen, log_probas=lp)
        return out, torch.cat([m._counter_values(reject, filters), bad, overflow, rows]), reject.numel(), filters

    @torch.no_grad()
    def __call__(self, batch: TokenizedSeqBatch, exclude_items: Optional[Tensor] = None,
                 include_items: Optional[Tensor] = None) -> ItemGenerationOutput:
        self._replay(batch, exclude_items, include_items)
        out, values, n_counters, filters = self._captured
        values = _read_search_counters(values)
        counters = EncoderDecoderRetrievalModel._check_filter_counts(values[:-3], n_counters, filters, "generate")
        EncoderDecoderRetrievalModel._raise_search_errors("beam", counters)
        n_bad, overflow, self.rows = values[-3:]
        if overflow:
            self.fallbacks += 1
            return self.model.generate_items(batch, n=self.n, search="exact", encoder="fused", decoder="fused",
                                             encoder_attention=self.attention, exclude_items=exclude_items,
                                             exclude_history=self.exclude_history, include_items=include_items, num_beams=self.k)
        if n_bad:
            raise _non_finite_error(_EXACT, n_bad)
        return ItemGenerationOutput(*(t.clone() for t in out))
