#!/usr/bin/env python
"""bench_score.py -- exact scores of given items (EncoderDecoderRetrievalModel.score_items) against rank_items and generate.

    python bench_score.py [--corpora 12101,1048576] [--negatives 100] [--reference-histories 4]

At the configs/decoder_amazon.gin shape (640 histories of 20 items, K = 256, 3 levels, d_model 384, 6 heads, d_ff 1024, 4 layers,
randomly initialised) on a corpus of uniformly random id tuples, each history's candidates are its true next item and
--negatives items drawn uniformly from the corpus (the sampled-candidate protocol).  For each corpus size:
  * ms per call, alternating after a warm-up call: score_items with the fp32 and with the TF32 cross-attention, rank_items(n=100)
    (every corpus item, fp32 attention) and generate_items(search="beam", decoder="fused");
  * decoder rows per call: score_items' padded rows (one per candidate-trie node, each level padded to the batch's largest count)
    and rank_items' (one per corpus-trie node per history);
  * torch.cuda.max_memory_allocated during one call of each scoring arm;
  * a split of one score_items call per attention from torch.profiler's CUDA kernel times (the groups of bench_rank.py, plus the
    trie build);
  * whether score_items' scores equal rank_items' dense scores at the candidates, bit for bit, and the sampled h@10 / NDCG.
On the smaller corpus also HF's T5Stack teacher-forced on the same candidates (the plain torch statement) for
--reference-histories histories, as ms per history.
Prints the card's name, power limit and max SM clock, read in the same run, and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_generate import _card  # noqa: E402
from bench_rank import B, H, K, SHAPE, inputs  # noqa: E402


def split(torch, fn):
    """ms of one call's CUDA kernels by group, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    groups = dict(gemm=0.0, cross_attention=0.0, children=0.0, trie_build=0.0, other=0.0)
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
        name = e.key
        if "t5rank_cross_attention" in name:
            groups["cross_attention"] += us
        elif "t5rank_children" in name:
            groups["children"] += us
        elif "t5score_trie" in name:
            groups["trie_build"] += us
        elif "gemm" in name.lower() or "split_image" in name or "sm90_xmma" in name or "cutlass" in name.lower():
            groups["gemm"] += us
        else:
            groups["other"] += us
    return {k: round(v / 1e3, 2) for k, v in groups.items()}


def torch_statement_ms(torch, m, batch, tuples, histories):
    """HF's T5Stack teacher-forced on each candidate tuple of the first `histories` histories, ms per history."""
    from rq_vae_recommender_b200.modules.model import _strip_dedup_col
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        for b in range(histories):
            mask = _strip_dedup_col(batch.seq_mask[b:b + 1].long(), H + 1, H)
            ids = _strip_dedup_col(batch.sem_ids[b:b + 1], H + 1, H)
            enc, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids)
            t = tuples[b]
            out = m.decoder_forward_pass(future_ids=t[:, :H - 1], encoder_output=enc.expand(t.shape[0], -1, -1),
                                         attention_mask_for_encoder=enc_mask.expand(t.shape[0], -1))
            sum(torch.log_softmax(m.decoder_mlp[h](out[:, h]), -1).gather(1, t[:, h:h + 1]) for h in range(H))
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / histories


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corpora", default="12101,1048576")
    ap.add_argument("--negatives", type=int, default=100)
    ap.add_argument("--reference-histories", type=int, default=4)
    args = ap.parse_args()
    import numpy as np
    import torch
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.evaluate.metrics import TopKAccumulator
    from rq_vae_recommender_b200.modules import model as M
    assert torch.cuda.is_available(), "bench_score.py needs a CUDA device"
    card = _card()
    print(f"card: {card}")
    result = dict(card=card, histories=B, candidates=1 + args.negatives, shape=SHAPE, corpora={})
    for N in (int(v) for v in args.corpora.split(",")):
        corpus, batch = inputs(torch, np, N, seed=N)
        torch.manual_seed(0)
        m = M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), **SHAPE).cuda().eval()
        target = m.item_of(batch.sem_ids_fut)
        rs = np.random.RandomState(N + 1)
        items = torch.cat([target[:, None], torch.from_numpy(rs.randint(0, N, size=(B, args.negatives))).cuda()], 1)
        tuples = m.codebooks[:, :H].cuda()[items]
        arms = {"score_fp32": lambda: m.score_items(batch, items),
                "score_tf32": lambda: m.score_items(batch, items, attention="tf32"),
                "rank_items": lambda: m.rank_items(batch, n=100),
                "generate": lambda: m.generate_items(batch, n=10, search="beam", decoder="fused")}
        first = {name: fn() for name, fn in arms.items()}
        torch.cuda.synchronize()
        counts = ops.t5score_trie_build(tuples, K).counts.clamp(min=1)
        score_rows = B * (1 + int(counts[:, :H - 1].max(0).values.sum()))
        levels = m._rank_levels(torch.device("cuda"))[0]
        times = {name: [] for name in arms}
        for _ in range(3):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                times[name].append(round((time.perf_counter() - t0) * 1e3, 2))
        peak = {}
        for name in ("score_fp32", "score_tf32", "rank_items"):
            torch.cuda.reset_peak_memory_stats()
            arms[name]()
            torch.cuda.synchronize()
            peak[name] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
        fp, tf = first["score_fp32"], first["score_tf32"]
        dense = m.rank_sem_ids(M._strip_dedup_col(batch.seq_mask.long(), H + 1, H), M._strip_dedup_col(batch.sem_ids, H + 1, H),
                               batch.user_ids)
        _, leaf_key, _ = m._rank_levels(dense.device)
        leaf = m._leaf_of(tuples.reshape(-1, H), leaf_key).reshape(B, -1)
        acc = TopKAccumulator([1, 5, 10])
        acc.accumulate_ranks(fp.target_rank, items.shape[1])
        metrics = acc.reduce()
        entry = dict(ms=times, decoder_rows=dict(score_items=score_rows, rank_items=B * sum(levels.n[:H])), peak_gib=peak,
                     split_ms={name: split(torch, arms[name]) for name in ("score_fp32", "score_tf32")},
                     equals_rank_sem_ids=bool(torch.equal(fp.scores, dense.gather(1, leaf))),
                     tf32_vs_fp32_max_score_diff=float((tf.scores - fp.scores).abs().max()),
                     sampled_exact_h10=metrics["exact_h@10"], sampled_exact_ndcg=round(metrics["exact_ndcg"], 5))
        del dense
        if args.reference_histories and N <= 20000:
            entry["torch_statement_ms_per_history"] = round(torch_statement_ms(torch, m, batch, tuples,
                                                                               args.reference_histories), 1)
        result["corpora"][N] = entry
        print(f"N={N}: {entry}")
        del m, first, arms, fp, tf
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
