#!/usr/bin/env python
"""bench_serve_exact.py -- serving latency of the exact top-k search: the eager generate_items(search="exact") against one
CUDA-graph replay of capture_exact_items, beside the beam replay of capture_generate_items.

    python bench_serve_exact.py [--corpora 12101,1048576] [--batches 1,8,64,640] [--windows 5] [--window-s 0.25]

At the configs/decoder_amazon.gin T5 shape of bench_serve.py / bench_exact.py (K = 256, 3 levels) on corpora of uniformly
random id tuples, B histories of 20 unmasked items, encoder="fused", decoder="fused".  The heads are scaled by s in {1, 8} (the
stand-in for a trained, more confident model of bench_exact.py, under which the search prunes), w = n = 10, and at s = 8 also
w = n = 100.  Per case:
  * ms per call, host clock around the call and the read of its item ids, for the arms "eager" (generate_items(search="exact")),
    "exact_graph" (a replay of capture_exact_items) and "beam_graph" (a replay of capture_generate_items(search="beam") at the
    same w); each arm warmed up, then alternated over --windows windows of about --window-s seconds: median and min..max;
  * capture ms and the capture's peak memory above what was allocated before;
  * decoder rows per history of the pruned decode (``ExactItemsGraph.rows / B``), the graph's fallbacks to the eager search over
    the timed calls, and whether every checked replay equalled its eager call (items, beams, count, sem_ids, log_probas);
  * empty CTAs, at the largest --batches value when its replay did not fall back: the replay at the default max_rows (the
    largest capacity) against a graph captured with max_rows just above the rows its pruned levels ran, same inputs.
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
from bench_rank import H, K, SHAPE  # noqa: E402
from bench_serve import compare, make_batch  # noqa: E402


def capture(torch, make):
    """(graph, capture ms, peak GiB above the memory before)."""
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    g = make()
    torch.cuda.synchronize()
    return g, round((time.perf_counter() - t0) * 1e3, 1), round((torch.cuda.max_memory_allocated() - before) / 2 ** 30, 3)


def same(a, b):
    return all(__import__("torch").equal(x, y) for x, y in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corpora", default="12101,1048576")
    ap.add_argument("--batches", default="1,8,64,640")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--window-s", type=float, default=0.25)
    args = ap.parse_args()
    import numpy as np
    import torch
    from rq_vae_recommender_b200.modules import model as M
    assert torch.cuda.is_available(), "bench_serve_exact.py needs a CUDA device"
    card = _card()
    print(f"card: {card}", flush=True)
    result = dict(card=card, shape=SHAPE, clock="host, call + item ids read", runs={})
    batches = [int(v) for v in args.batches.split(",")]
    for N in (int(v) for v in args.corpora.split(",")):
        rs = np.random.RandomState(N)
        corpus = rs.randint(0, K, size=(N, H)).astype(np.int64)
        for scale, w in [(1, 10), (8, 10), (8, 100)]:
            torch.manual_seed(0)
            m = M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), **SHAPE).cuda().eval()
            with torch.no_grad():
                for mlp in m.decoder_mlp:
                    mlp.weight.mul_(scale)
            for B in batches:
                batch = make_batch(torch, np, rs, corpus, B, padded=False)
                kw = dict(num_beams=w, n=w)
                eager = lambda: m.generate_items(batch, search="exact", encoder="fused", decoder="fused", **kw)  # noqa: E731
                want = eager()
                g, cap_ms, peak_gib = capture(torch, lambda: m.capture_exact_items(batch, **kw))
                beam, _, _ = capture(torch, lambda: m.capture_generate_items(batch, search="beam", **kw))
                got = g(batch)
                equal = same(got, want)
                rows = g.rows
                ms = compare(torch, {"eager": eager, "exact_graph": lambda: g(batch), "beam_graph": lambda: beam(batch)},
                             args.windows, args.window_s)
                equal = equal and same(g(batch), want)
                entry = dict(ms=ms, capture_ms=cap_ms, capture_peak_gib=peak_gib, rows_per_history=round(rows / B, 1),
                             fallbacks=g.fallbacks, replay_equals_eager=equal)
                if g.fallbacks == 0 and B == max(batches):
                    # the pruned levels' rows bound a capacity just above what this batch runs
                    tight_rows = max(1, rows - B) + 1
                    tight, _, tight_gib = capture(torch, lambda: m.capture_exact_items(batch, max_rows=tight_rows, **kw))
                    t = compare(torch, {"default_max_rows": lambda: g(batch), "tight_max_rows": lambda: tight(batch)},
                                args.windows, args.window_s)
                    entry["empty_ctas"] = dict(ms=t, tight_max_rows=tight_rows, tight_capture_peak_gib=tight_gib,
                                               tight_fallbacks=tight.fallbacks)
                    del tight
                name = f"N={N},s={scale},B={B},w=n={w}"
                result["runs"][name] = entry
                print(f"{name}: {entry}", flush=True)
                del g, beam, got, want
                torch.cuda.empty_cache()
            del m
            torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
