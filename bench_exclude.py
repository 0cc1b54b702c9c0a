#!/usr/bin/env python
"""bench_exclude.py -- the cost of per-history exclusion sets (ops.sid_exclusion_build and the exclude= input of the searches,
the item retrieval and the exact ranking's selection).

    python bench_exclude.py [--corpora 12101,1048576] [--reps 20]

At bench_generate.py's shape (640 histories of 20 items excluded each, top-k 10, K = 256, 3 levels) on corpora of uniformly
random id tuples, for each corpus size, median ms over --reps repetitions with the arms alternated (CUDA events, one warm-up):
  * the build of the 640 exclusion sets;
  * per level, SidPrefixIndex.beam_topk and sample_select (64 candidates per beam) with and without the exclusion;
  * SidItemTable.retrieve of the top-10 beams with and without;
  * ops.t5rank_select (n = 100) over the corpus's U leaves (bench_rank.py's U) with and without.
The excluded items are each history's 20 items, drawn from the corpus.  Prints the card's name, power limit and max SM clock,
read in the same run, and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_generate import _card  # noqa: E402

B, K, H, ITEMS, TOP_K, NC = 640, 256, 3, 20, 10, 64


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


def run(N, reps):
    import numpy as np
    import torch
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(N)
    corpus = rs.randint(0, K, size=(N, H)).astype(np.int64)
    ids = torch.from_numpy(corpus).cuda()
    index, table = ops.SidPrefixIndex(ids, K), ops.SidItemTable(ids, K)
    tuples = np.unique(corpus, axis=0)                          # the table's leaves, in its lexicographic order
    leaf_key = torch.from_numpy((tuples[:, 0] * K + tuples[:, 1]) * K + tuples[:, 2]).cuda()
    U = leaf_key.shape[0]
    items = torch.from_numpy(rs.randint(0, N, size=(B, ITEMS))).cuda()
    ex = ops.sid_exclusion_build(items, table, leaf_key)
    out = dict(corpus_rows=N, leaves=U)
    out["build_ms"] = timed(torch, {"build": lambda: ops.sid_exclusion_build(items, table, leaf_key)}, reps)["build"]
    gen, lp = None, None
    for h in range(H):
        rows = B if gen is None else B * TOP_K
        logits = torch.randn(rows, K, device="cuda") * 3
        probas = torch.softmax(logits, -1)
        noise = torch.empty_like(probas).exponential_(1)
        g, p = gen, lp
        t = timed(torch, {
            "beam_topk": lambda: index.beam_topk(logits, g, p, TOP_K),
            "beam_topk_excluding": lambda: index.beam_topk(logits, g, p, TOP_K, exclude=ex),
            "sample_select": lambda: index.sample_select(probas, noise, g, p, TOP_K, NC),
            "sample_select_excluding": lambda: index.sample_select(probas, noise, g, p, TOP_K, NC, exclude=ex),
        }, reps)
        out[f"level{h}_ms"] = t
        gen, lp, _ = index.beam_topk(logits, g, p, TOP_K, exclude=ex)
    out["retrieve_ms"] = timed(torch, {"retrieve": lambda: table.retrieve(gen, lp, TOP_K),
                                       "retrieve_excluding": lambda: table.retrieve(gen, lp, TOP_K, exclude=ex)}, reps)
    scores = torch.randn(B, U, device="cuda")
    row, start = table.arrays()
    t_leaf = torch.randint(0, U, (B,), device="cuda")
    t_dedup = torch.zeros(B, dtype=torch.int64, device="cuda")
    out["t5rank_select_ms"] = timed(torch, {
        "select": lambda: ops.t5rank_select(scores, row, start, t_leaf, t_dedup, 100),
        "select_excluding": lambda: ops.t5rank_select(scores, row, start, t_leaf, t_dedup, 100, exclude=ex)}, reps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corpora", default="12101,1048576")
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    card = _card()
    print(f"card: {card}")
    res = dict(card=card, histories=B, excluded_per_history=ITEMS, top_k=TOP_K, K=K, levels=H,
               corpora=[run(int(n), args.reps) for n in args.corpora.split(",")])
    torch.cuda.synchronize()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
