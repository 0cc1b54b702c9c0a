#!/usr/bin/env python
"""bench_include.py -- the cost of per-history allow-lists (ops.sid_inclusion_build and the include= input of the searches and
the item retrieval).

    python bench_include.py [--corpora 12101,1048576] [--sizes 100,1000,4096] [--reps 20]

At bench_generate.py's shape (640 histories, top-k 10, K = 256, 3 levels) on corpora of uniformly random id tuples, for each
corpus size and allow-list size (items per history, drawn uniformly from the corpus: a candidate pool of an upstream retriever),
median ms over --reps repetitions with the arms alternated (CUDA events, one warm-up):
  * the build of the 640 allow-lists;
  * per level, SidPrefixIndex.beam_topk and sample_select (64 candidates per beam) with and without the allow-list;
  * SidItemTable.retrieve of the top-10 beams with and without.
The beams of the next level come from the beam search with the allow-list, so every level and the retrieval see beams that
lead to allowed items.  Prints the card's name, power limit and max SM clock, read in the same run, and one JSON line; writes
nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_generate import _card  # noqa: E402

B, K, H, TOP_K, NC = 640, 256, 3, 10, 64


def timed(torch, arms, reps):
    """Median ms of each arm (a dict of name -> fn), the arms alternated within every repetition."""
    for fn in arms.values():
        fn()
    times = {name: [] for name in arms}
    for _ in range(reps):
        for name, fn in arms.items():
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            fn()
            end.record()
            end.synchronize()
            times[name].append(start.elapsed_time(end))
    return {name: round(sorted(t)[len(t) // 2], 4) for name, t in times.items()}


def run(N, sizes, reps):
    import numpy as np
    import torch
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(N)
    corpus = rs.randint(0, K, size=(N, H)).astype(np.int64)
    ids = torch.from_numpy(corpus).cuda()
    index, table = ops.SidPrefixIndex(ids, K), ops.SidItemTable(ids, K)
    tuples = np.unique(corpus, axis=0)                          # the table's leaves, in its lexicographic order
    leaf_key = torch.from_numpy((tuples[:, 0] * K + tuples[:, 1]) * K + tuples[:, 2]).cuda()
    out = dict(corpus_rows=N, leaves=leaf_key.shape[0], allow_lists=[])
    for M in sizes:
        items = torch.from_numpy(rs.randint(0, N, size=(B, M))).cuda()
        inc = ops.sid_inclusion_build(items, table, leaf_key)
        res = dict(items_per_history=M)
        res["build_ms"] = timed(torch, {"build": lambda: ops.sid_inclusion_build(items, table, leaf_key)}, reps)["build"]
        gen, lp = None, None
        for h in range(H):
            rows = B if gen is None else B * TOP_K
            logits = torch.randn(rows, K, device="cuda") * 3
            probas = torch.softmax(logits, -1)
            noise = torch.empty_like(probas).exponential_(1)
            g, p = gen, lp
            res[f"level{h}_ms"] = timed(torch, {
                "beam_topk": lambda: index.beam_topk(logits, g, p, TOP_K),
                "beam_topk_including": lambda: index.beam_topk(logits, g, p, TOP_K, include=inc),
                "sample_select": lambda: index.sample_select(probas, noise, g, p, TOP_K, NC),
                "sample_select_including": lambda: index.sample_select(probas, noise, g, p, TOP_K, NC, include=inc),
            }, reps)
            gen, lp, _ = index.beam_topk(logits, g, p, TOP_K, include=inc)
        res["retrieve_ms"] = timed(torch, {"retrieve": lambda: table.retrieve(gen, lp, TOP_K),
                                           "retrieve_including": lambda: table.retrieve(gen, lp, TOP_K, include=inc)}, reps)
        res["finite_beams"] = int((lp > -float("inf")).sum())
        out["allow_lists"].append(res)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corpora", default="12101,1048576")
    ap.add_argument("--sizes", default="100,1000,4096")
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    sizes = [int(m) for m in args.sizes.split(",")]
    import torch
    card = _card()
    print(f"card: {card}")
    res = dict(card=card, histories=B, top_k=TOP_K, K=K, levels=H,
               corpora=[run(int(n), sizes, args.reps) for n in args.corpora.split(",")])
    torch.cuda.synchronize()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
