#!/usr/bin/env python
"""bench_serve.py -- serving latency of generate_items: the eager call against one CUDA-graph replay (capture_generate_items).

    python bench_serve.py [--corpora 12101,1048576] [--batches 1,8,64,640] [--windows 5] [--window-s 0.25]

At the configs/decoder_amazon.gin T5 shape (K = 256, 3 levels, d_model 384, 6 heads, d_ff 1024, 4 layers) on corpora of uniformly
random id tuples, for B histories of 20 items each (every position unmasked, so N = B * S and the graph's encoder does the eager
work), encoder="fused", decoder="fused":
  * ms per call, host clock around the call and the read of its item ids (``.cpu()``), for the arms "eager"
    (``generate_items``) and "graph" (a replay of ``capture_generate_items``' graph), search "beam" and "sample" at w = 10, and
    at w = 64 for B <= 64.  Each arm is warmed up, then the arms alternate over --windows windows of about --window-s seconds;
    the median window and the spread (min..max) are printed;
  * librqb200 launches of one eager call (``ops.LAUNCHES``; cuBLAS and torch launches come on top);
  * the one-time capture cost (ms, with its warm-up call) and the graph's memory: the peak of max_memory_allocated during the
    capture above what was allocated before, and what the graph keeps allocated after it;
  * at B = 640 (when in --batches): histories of a uniform 1..20 items, where the graph's encoder GEMMs run B * S capacity rows
    against the eager N: the ratio B * S / N (the extra GEMM rows) and the two arms' times.
Whether a replay equals the eager call (search "beam", full histories) is checked once per shape.  Prints the card's name, power
limit and max SM clock, read in the same run, and one JSON line; writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_generate import _card  # noqa: E402
from bench_rank import H, ITEMS, K, SHAPE  # noqa: E402


def make_batch(torch, np, rs, corpus, B, padded):
    """B histories of ITEMS random corpus items; padded: the first 0..ITEMS - 1 items of each masked (1..ITEMS kept)."""
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    w = H + 1
    sem = np.zeros((B, ITEMS, w), dtype=np.int64)
    sem[:, :, :H] = corpus[rs.randint(0, len(corpus), size=(B, ITEMS))]
    mask = np.ones((B, ITEMS), dtype=bool)
    if padded:
        keep = rs.randint(1, ITEMS + 1, size=B)
        mask = np.arange(ITEMS)[None, :] >= (ITEMS - keep)[:, None]
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    return TokenizedSeqBatch(user_ids=None, sem_ids=cuda(sem.reshape(B, ITEMS * w)), sem_ids_fut=cuda(sem[:, -1]),
                             seq_mask=cuda(np.repeat(mask, w, axis=1)), token_type_ids=None, token_type_ids_fut=None)


def per_call_ms(torch, fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn().item_ids.cpu()
    return (time.perf_counter() - t0) * 1e3 / reps


def compare(torch, arms, windows, window_s):
    """{arm: (median ms, min ms, max ms)} over alternated windows, after a warm-up sized from one timed call."""
    reps = {}
    for name, fn in arms.items():
        for _ in range(3):
            fn()
        ms = per_call_ms(torch, fn, 3)
        reps[name] = max(3, int(window_s * 1e3 / max(ms, 1e-3)))
    times = {name: [] for name in arms}
    for _ in range(windows):
        for name, fn in arms.items():
            times[name].append(per_call_ms(torch, fn, reps[name]))
    return {name: (round(statistics.median(t), 3), round(min(t), 3), round(max(t), 3)) for name, t in times.items()}


def capture(torch, m, batch, **kw):
    """(graph, capture ms, peak GiB above the memory before, GiB the graph keeps)."""
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    g = m.capture_generate_items(batch, **kw)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    gib = 2 ** 30
    return g, round(ms, 1), round((torch.cuda.max_memory_allocated() - before) / gib, 3), \
        round((torch.cuda.memory_allocated() - before) / gib, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corpora", default="12101,1048576")
    ap.add_argument("--batches", default="1,8,64,640")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--window-s", type=float, default=0.25)
    args = ap.parse_args()
    import numpy as np
    import torch
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    assert torch.cuda.is_available(), "bench_serve.py needs a CUDA device"
    card = _card()
    print(f"card: {card}", flush=True)
    result = dict(card=card, shape=SHAPE, items=ITEMS, clock="host, call + item ids read", runs={})
    batches = [int(v) for v in args.batches.split(",")]
    for N in (int(v) for v in args.corpora.split(",")):
        rs = np.random.RandomState(N)
        corpus = rs.randint(0, K, size=(N, H)).astype(np.int64)
        torch.manual_seed(0)
        m = M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus), **SHAPE).cuda().eval()
        for B in batches:
            for search, w in [("beam", 10), ("sample", 10)] + ([("beam", 64), ("sample", 64)] if B <= 64 else []):
                batch = make_batch(torch, np, rs, corpus, B, padded=False)
                kw = dict(search=search, num_beams=w)
                eager = lambda: m.generate_items(batch, encoder="fused", decoder="fused", **kw)  # noqa: E731
                eager()
                n0 = ops.LAUNCHES
                want = eager()
                launches = ops.LAUNCHES - n0
                g, cap_ms, peak_gib, kept_gib = capture(torch, m, batch, **kw)
                got = g(batch)
                equal = None if search == "sample" else all(torch.equal(a, b) for a, b in zip(got, want))
                ms = compare(torch, {"eager": eager, "graph": lambda: g(batch)}, args.windows, args.window_s)
                entry = dict(ms=ms, speedup=round(ms["eager"][0] / ms["graph"][0], 2), lib_launches=launches,
                             capture_ms=cap_ms, capture_peak_gib=peak_gib, graph_gib=kept_gib, replay_equals_eager=equal)
                name = f"N={N},B={B},{search},w={w}"
                result["runs"][name] = entry
                print(f"{name}: {entry}", flush=True)
                del g, got, want
        if 640 in batches:
            batch = make_batch(torch, np, rs, corpus, 640, padded=True)
            kw = dict(search="beam", num_beams=10)
            H_ = m.num_hierarchies
            offsets, _ = ops.t5enc_offsets(M._strip_dedup_col(batch.seq_mask.long(), H_ + 1, H_), H_, True, False)
            n_kept = int(offsets[-1])
            rows = 640 * ops.t5enc_len(ITEMS * H_, H_, True, False)
            g, cap_ms, peak_gib, kept_gib = capture(torch, m, batch, **kw)
            got, want = g(batch), m.generate_items(batch, encoder="fused", decoder="fused", **kw)
            ms = compare(torch, {"eager": lambda: m.generate_items(batch, encoder="fused", decoder="fused", **kw),
                                 "graph": lambda: g(batch)}, args.windows, args.window_s)
            entry = dict(ms=ms, packed_rows_eager=n_kept, capacity_rows=rows, extra_gemm_rows=round(rows / n_kept, 3),
                         capture_ms=cap_ms, capture_peak_gib=peak_gib, graph_gib=kept_gib,
                         same_items=bool(torch.equal(got.item_ids, want.item_ids)),
                         max_log_proba_diff=float((got.log_probas - want.log_probas).abs().nan_to_num(0).max()))
            name = f"N={N},B=640,beam,w=10,histories of 1..{ITEMS} items"
            result["runs"][name] = entry
            print(f"{name}: {entry}", flush=True)
            del g, got, want
        del m
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
