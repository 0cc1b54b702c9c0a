#!/usr/bin/env python
"""bench_exact.py -- the exact top-k search (generate_items(search="exact")) against the beam search and the full exact ranking.

    python bench_exact.py [--corpora 12101,1048576] [--scales 1,8,32] [--repeats 2]

At the configs/decoder_amazon.gin shape (640 histories of 20 items, K = 256, 3 levels, d_model 384, 6 heads, d_ff 1024, 4 layers)
on a corpus of uniformly random id tuples, for each corpus size and head scale s (decoder_mlp weights times s: s = 1 is the
randomly initialised model, whose leaf scores lie within about 1e-3 of each other, the worst case for pruning; s = 8 and 32 are
a stand-in for a trained, more confident model -- how much a trained model prunes is NOT measured here):
  * ms per call, alternating the arms after a warm-up call of each: generate_items(search="exact", decoder="fused": the bound's
    beam search on the fused decoder) at w = 10 and w = 100 (n = w),
    generate_items(search="beam", decoder="fused", n = 10) and rank_items(n = 10);
  * decoder rows per history of the pruned decode (mean / max; EXACT_DECODER_ROWS and the per-level counts) against the full
    trie's rows per history (what rank_items decodes);
  * a split of one exact call into the bound (beam search + exact rescoring), the pruned decode and the selection, each timed
    between device synchronisations in an instrumented call of its own;
  * torch.cuda.max_memory_allocated during one call of each arm;
  * the share of histories whose beam top-10 items differ from the exact top-10 (w = 10) items.
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
from bench_rank import B, H, SHAPE, inputs  # noqa: E402


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def instrumented(torch, M, fn):
    """One exact call with its phases timed between synchronisations, and each history's decoder rows."""
    phases = dict(bound=0.0, decode=0.0, select=0.0)
    rows = torch.zeros(B, dtype=torch.int64)
    chunk = []
    orig = (M.EncoderDecoderRetrievalModel._search_levels, M.EncoderDecoderRetrievalModel._score_candidates, M.FusedT5Exact.run,
            M.ops.t5exact_select, M._read_frontier)

    def clocked(name, f):
        def wrapped(*a, **kw):
            out, ms = timed(torch, lambda: f(*a, **kw))
            phases[name] += ms
            return out
        return wrapped

    def run(self, b0, b1, *a, **kw):
        chunk.clear()
        out, ms = timed(torch, lambda: orig[2](self, b0, b1, *a, **kw))
        phases["decode"] += ms
        if out is not None:
            rows[b0:b1] += 1 + sum(c.cpu().long() for c in chunk) if chunk else 1
        return out

    def read(offsets, counts):
        chunk.append(counts[0].clone())
        return orig[4](offsets, counts)

    M.EncoderDecoderRetrievalModel._search_levels = clocked("bound", orig[0])
    M.EncoderDecoderRetrievalModel._score_candidates = clocked("bound", orig[1])
    M.FusedT5Exact.run = run
    M.ops.t5exact_select = clocked("select", orig[3])
    M._read_frontier = read
    try:
        fn()
    finally:
        (M.EncoderDecoderRetrievalModel._search_levels, M.EncoderDecoderRetrievalModel._score_candidates, M.FusedT5Exact.run,
         M.ops.t5exact_select, M._read_frontier) = orig
    phases["decode"] -= phases["select"]                      # run() includes the selection
    return {k: round(v, 1) for k, v in phases.items()}, rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corpora", default="12101,1048576")
    ap.add_argument("--scales", default="1,8,32")
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    import numpy as np
    import torch
    from rq_vae_recommender_b200.modules import model as M
    assert torch.cuda.is_available(), "bench_exact.py needs a CUDA device"
    card = _card()
    print(f"card: {card}")
    result = dict(card=card, histories=B, shape=SHAPE, trained_model_pruning="not measured", runs={})
    for N in (int(v) for v in args.corpora.split(",")):
        corpus, batch = inputs(torch, np, N, seed=N)
        for s in (float(v) for v in args.scales.split(",")):
            torch.manual_seed(0)
            m = M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), **SHAPE).cuda().eval()
            with torch.no_grad():
                for mlp in m.decoder_mlp:
                    mlp.weight.mul_(s)
            arms = {"exact_w10": lambda: m.generate_items(batch, n=10, num_beams=10, search="exact", decoder="fused"),
                    "exact_w100": lambda: m.generate_items(batch, n=100, num_beams=100, search="exact", decoder="fused"),
                    "beam_w10": lambda: m.generate_items(batch, n=10, search="beam", decoder="fused"),
                    "rank_n10": lambda: m.rank_items(batch, n=10)}
            first, rows = {}, {}
            for name, fn in arms.items():
                first[name] = fn()
                if name.startswith("exact"):
                    rows[name] = M.EXACT_DECODER_ROWS
            levels = m._rank_levels(torch.device("cuda"))[0]
            full = sum(levels.n[:H])
            times = {name: [] for name in arms}
            for _ in range(args.repeats):
                for name, fn in arms.items():
                    times[name].append(round(timed(torch, fn)[1], 1))
            peak = {}
            for name, fn in arms.items():
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                fn()
                torch.cuda.synchronize()
                peak[name] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
            split, per_history = {}, {}
            for name in ("exact_w10", "exact_w100"):
                split[name], r = instrumented(torch, M, arms[name])
                assert int(r.sum()) == rows[name], (int(r.sum()), rows[name])
                per_history[name] = dict(mean=round(float(r.float().mean()), 1), max=int(r.max()))
            ex, bm, rk = first["exact_w10"], first["beam_w10"], first["rank_n10"]
            entry = dict(ms=times, full_trie_rows_per_history=full, rows_per_history=per_history, split_ms=split, peak_gib=peak,
                         beam_top10_differs=round(float((bm.item_ids != ex.item_ids).any(1).float().mean()), 4),
                         exact_equals_rank=bool(torch.equal(ex.item_ids, rk.item_ids)), leaves=levels.n[H])
            result["runs"][f"N={N},s={s:g}"] = entry
            print(f"N={N} s={s:g}: {entry}", flush=True)
            del m, arms, first, ex, bm, rk
            torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
