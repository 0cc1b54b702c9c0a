"""Benchmark of the corpus item table and the device-side evaluation metrics (no reference run needed).

    python bench_retrieve.py [--min-window-s 1.0]

Arms:
  * build_ms / build_bytes  ops.SidItemTable over corpora of K = 256, 3 levels: 12 101 random rows (the shipped Beauty corpus
                            size), 1 048 576 random rows, and 1 048 576 rows over 8 codes per level (512 tuples, ~2 000 items each);
  * retrieve_ms             SidItemTable.retrieve at batch 640, top-k 10, n = 10 and 100, beams drawn from the corpus with
                            descending log-probabilities, on the 12 101-row corpus and on 12 101 rows over 6 codes per level;
  * accumulate_ms           TopKAccumulator.accumulate per evaluation batch (640 x top-k 10 x 3 levels) against a plain-torch
                            statement of the same rule (the [B, k, D] compare, .all(-1).max(-1), the NDCG sum and h@k for
                            ks = 1, 5, 10 read back per batch), with the host synchronisations each makes per call, counted with
                            torch.cuda.set_sync_debug_mode("warn").
Every shape is warmed up and every timed window lasts at least --min-window-s seconds (CUDA events).  Prints the card's name,
power limit and max SM clock, and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys
import warnings

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_generate import _card, timed_ms  # noqa: E402

B, TOP_K, K, H = 640, 10, 256, 3
KS = [1, 5, 10]


def torch_accumulate(torch, metrics, actual, top_k):
    """The reference's TopKAccumulator.accumulate rule in plain torch."""
    match = (actual.unsqueeze(1) == top_k).all(dim=-1)
    found, rank = match.max(dim=-1)
    matched = rank[found]
    metrics["ndcg"] += (1.0 / torch.log2(matched.float() + 2.0)).sum().item()
    for k in KS:
        metrics[f"h@{k}"] += int((matched < k).sum())


def host_syncs(torch, fn):
    """Host synchronisations one call of fn makes."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("called a synchronizing CUDA operation" in str(w.message) for w in caught)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-window-s", type=float, default=1.0)
    args = ap.parse_args()
    import torch
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.evaluate.metrics import TopKAccumulator
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    corpora = {
        "12101": torch.randint(0, K, (12101, H), device=dev, generator=g),
        "1048576": torch.randint(0, K, (1 << 20, H), device=dev, generator=g),
        "1048576_8codes": torch.randint(0, 8, (1 << 20, H), device=dev, generator=g),
        "12101_6codes": torch.randint(0, 6, (12101, H), device=dev, generator=g),
    }
    out = {"card": _card(), "batch": B, "top_k": TOP_K, "K": K, "levels": H}
    for name in ("12101", "1048576", "1048576_8codes"):
        cb = corpora[name]
        out[f"build_ms/{name}"] = round(timed_ms(torch, lambda: ops.SidItemTable(cb, K), args.min_window_s), 4)
        out[f"build_bytes/{name}"] = ops.SidItemTable(cb, K).nbytes
    for name in ("12101", "12101_6codes"):
        cb = corpora[name]
        table = ops.SidItemTable(cb, K)
        gen = cb[torch.randint(0, cb.shape[0], (B, TOP_K), device=dev, generator=g)]
        lp = -torch.rand(B, TOP_K, device=dev, generator=g).sort(dim=1).values
        for n in (10, 100):
            out[f"retrieve_ms/{name}/n{n}"] = round(timed_ms(torch, lambda: table.retrieve(gen, lp, n), args.min_window_s), 4)
            items, _, count = table.retrieve(gen, lp, n)
            out[f"retrieve_mean_count/{name}/n{n}"] = round(float(count.float().mean()), 2)
    actual = corpora["12101"][torch.randint(0, 12101, (B,), device=dev, generator=g)]
    top_k = corpora["12101"][torch.randint(0, 12101, (B, TOP_K), device=dev, generator=g)]
    top_k[::3, 4] = actual[::3]
    acc, metrics = TopKAccumulator(ks=KS), {"ndcg": 0.0, **{f"h@{k}": 0 for k in KS}}
    out["accumulate_ms"] = round(timed_ms(torch, lambda: acc.accumulate(actual, top_k), args.min_window_s), 4)
    out["accumulate_torch_ms"] = round(timed_ms(torch, lambda: torch_accumulate(torch, metrics, actual, top_k),
                                                args.min_window_s), 4)
    out["accumulate_host_syncs"] = host_syncs(torch, lambda: acc.accumulate(actual, top_k))
    out["accumulate_torch_host_syncs"] = host_syncs(torch, lambda: torch_accumulate(torch, metrics, actual, top_k))
    acc.reset()
    acc.accumulate(actual, top_k)
    check = {"ndcg": 0.0, **{f"h@{k}": 0 for k in KS}}
    torch_accumulate(torch, check, actual, top_k)
    red = acc.reduce()
    out["accumulate_agrees"] = all(abs(red[k] - check[k] / B) <= 1e-6 * max(1.0, abs(check[k] / B)) for k in check)
    print(f"card: {out['card']}")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
