#!/usr/bin/env python
"""bench_rank.py -- exact ranking of every corpus item (EncoderDecoderRetrievalModel.rank_items) against generate.

    python bench_rank.py [--corpora 12101,1048576] [--reference-histories 2]

At the configs/decoder_amazon.gin shape (640 histories of 20 items, K = 256, 3 levels, d_model 384, 6 heads, d_ff 1024, 4 layers,
randomly initialised) on a corpus of uniformly random id tuples (not a tokenised catalogue), for each corpus size:
  * ms per rank_items call (n = 100) with the fp32 and with the TF32 cross-attention (attention="fp32" / "tf32"), and per
    generate(search="beam", decoder="fused") call (the module's matmul precision, "high"), alternating, after a warm-up call;
  * the largest |score difference| between the two attentions over the returned items;
  * decoder rows per call (one per trie node per history) and torch.cuda.max_memory_allocated during one rank_items call;
  * a split of one rank_items call per attention from torch.profiler's CUDA kernel times: GEMMs, the new cross-attention, the
    children scores, the selection, and the rest (add-norm, self-attention, encoder);
  * the share of histories whose exact top-10 items differ from the items of search="beam"'s top-10 beams.  This is a property
    of the randomly initialised model, not of a trained one.
On the smaller corpus also the plain torch statement (HF's T5Stack teacher-forced on every corpus tuple, in chunks) for
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

B, K, H, ITEMS = 640, 256, 3, 20
SHAPE = dict(num_hierarchies=H, num_embeddings_per_hierarchy=K, t5_d_model=384, t5_num_heads=6, t5_d_ff=1024, t5_num_layers=4,
             top_k_for_generation=10, should_add_sep_token=True)


def inputs(torch, np, N, seed):
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    rs = np.random.RandomState(seed)
    corpus = rs.randint(0, K, size=(N, H)).astype(np.int64)
    ids = torch.from_numpy(rs.randint(0, K, size=(B, ITEMS * H))).cuda()
    w = H + 1
    sem = torch.zeros(B, ITEMS * w, dtype=torch.int64, device="cuda")
    sem.view(B, ITEMS, w)[:, :, :H] = ids.view(B, ITEMS, H)
    seq = torch.ones(B, ITEMS * w, dtype=torch.bool, device="cuda")
    fut = torch.from_numpy(np.concatenate([corpus[rs.randint(0, N, size=B)], np.zeros((B, 1), dtype=np.int64)], 1)).cuda()
    tt = torch.arange(ITEMS * w, device="cuda").remainder(w).expand(B, -1)
    batch = TokenizedSeqBatch(user_ids=None, sem_ids=sem, sem_ids_fut=fut, seq_mask=seq, token_type_ids=tt,
                              token_type_ids_fut=torch.arange(w, device="cuda").expand(B, -1))
    return corpus, batch


def split(torch, fn):
    """ms of one call's CUDA kernels by group, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    groups = dict(gemm=0.0, cross_attention=0.0, children=0.0, select=0.0, other=0.0)
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
        name = e.key
        if "t5rank_cross_attention" in name:
            groups["cross_attention"] += us
        elif "t5rank_children" in name:
            groups["children"] += us
        elif "t5rank_select" in name:
            groups["select"] += us
        elif "gemm" in name.lower() or "split_image" in name or "sm90_xmma" in name or "cutlass" in name.lower():
            groups["gemm"] += us
        else:
            groups["other"] += us
    return {k: round(v / 1e3, 2) for k, v in groups.items()}


def torch_statement_ms(torch, m, batch, corpus, histories):
    """HF's T5Stack teacher-forced on every retrievable tuple for the first `histories` histories, ms per history."""
    from rq_vae_recommender_b200.modules.model import _strip_dedup_col
    tuples = torch.from_numpy(__import__("numpy").unique(corpus, axis=0)).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        for b in range(histories):
            mask = _strip_dedup_col(batch.seq_mask[b:b + 1].long(), H + 1, H)
            ids = _strip_dedup_col(batch.sem_ids[b:b + 1], H + 1, H)
            enc, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids)
            for c in range(0, tuples.shape[0], 4096):
                t = tuples[c:c + 4096]
                out = m.decoder_forward_pass(future_ids=t[:, :H - 1], encoder_output=enc.expand(t.shape[0], -1, -1),
                                             attention_mask_for_encoder=enc_mask.expand(t.shape[0], -1))
                s = sum(torch.log_softmax(m.decoder_mlp[h](out[:, h]), -1).gather(1, t[:, h:h + 1]) for h in range(H))
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / histories


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corpora", default="12101,1048576")
    ap.add_argument("--reference-histories", type=int, default=2)
    args = ap.parse_args()
    import numpy as np
    import torch
    from rq_vae_recommender_b200.modules import model as M
    assert torch.cuda.is_available(), "bench_rank.py needs a CUDA device"
    card = _card()
    print(f"card: {card}")
    result = dict(card=card, histories=B, items=ITEMS, shape=SHAPE, corpora={})
    for N in (int(v) for v in args.corpora.split(",")):
        corpus, batch = inputs(torch, np, N, seed=N)
        torch.manual_seed(0)
        m = M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), **SHAPE).cuda().eval()
        arms = {"rank_fp32": lambda: m.rank_items(batch, n=100),
                "rank_tf32": lambda: m.rank_items(batch, n=100, attention="tf32"),
                "generate": lambda: m.generate_items(batch, n=10, search="beam", decoder="fused")}
        first = {name: fn() for name, fn in arms.items()}
        torch.cuda.synchronize()
        levels = m._rank_levels(torch.device("cuda"))[0]
        rows = B * sum(levels.n[:H])
        times = {name: [] for name in arms}
        for _ in range(3):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                times[name].append(round((time.perf_counter() - t0) * 1e3, 2))
        peak = {}
        for name in ("rank_fp32", "rank_tf32"):
            torch.cuda.reset_peak_memory_stats()
            arms[name]()
            torch.cuda.synchronize()
            peak[name] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
        out, tf, g = first["rank_fp32"], first["rank_tf32"], first["generate"]
        fin = torch.isfinite(out.scores)
        differs = float((out.item_ids[:, :10] != g.item_ids).any(1).float().mean())
        entry = dict(ms=times, decoder_rows=rows, leaves=levels.n[H], peak_gib=peak,
                     split_ms={name: split(torch, arms[name]) for name in ("rank_fp32", "rank_tf32")},
                     tf32_vs_fp32_max_score_diff=float((tf.scores - out.scores)[fin].abs().max()),
                     tf32_same_top10=float((tf.item_ids[:, :10] == out.item_ids[:, :10]).all(1).float().mean()),
                     top10_differs_from_beam=round(differs, 4), num_items=out.num_items)
        if args.reference_histories and N <= 20000:
            entry["torch_statement_ms_per_history"] = round(torch_statement_ms(torch, m, batch, corpus,
                                                                               args.reference_histories), 1)
        result["corpora"][N] = entry
        print(f"N={N}: {entry}")
        del m, out, tf, g, first, arms
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
