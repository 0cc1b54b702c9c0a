"""Generate tests/golden/metrics.npz by running the UNMODIFIED reference evaluate.metrics.TopKAccumulator.

Run where the reference tree is available (RQ_REFERENCE_PATH, see ref_harness.py):   python tests/golden/make_golden_metrics.py
The GPU box never runs this; it consumes the committed .npz file.

Three cases, each several batches of (actual [B, D], top_k [B, k, D]) accumulated into one TopKAccumulator, then reduce():
rows with no match, rows with several matching candidates (the first counts), batches of different sizes and ``ks`` wider than
the candidate list.  Stored: the batches, ks, and the reduced keys and values in the reference's order.
"""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_harness          # noqa: E402

CASES = {                   # name: (ks, k candidates, D columns, id range, batch sizes)
    "tuples": ([1, 5, 10], 10, 3, 4, [64, 37, 128]),
    "wide_ks": ([1, 3, 8, 20, 50], 8, 3, 3, [50, 50, 1]),
    "items": ([1, 5, 10, 100], 10, 1, 12, [200, 33]),
}


def batch(rng, B, k, D, hi):
    actual = rng.integers(0, hi, size=(B, D))
    top_k = rng.integers(0, hi, size=(B, k, D))
    plant = rng.random(B) < 0.5                              # half the rows get the actual tuple planted at a random rank
    top_k[plant, rng.integers(0, k, size=B)[plant]] = actual[plant]
    again = rng.random(B) < 0.2                              # some get it twice more, so several candidates match
    for _ in range(2):
        top_k[again, rng.integers(0, k, size=B)[again]] = actual[again]
    top_k[: max(1, B // 10)] = hi + 1                        # rows that match nothing
    return actual, top_k


def main():
    ref_harness.load()
    metrics = importlib.import_module("evaluate.metrics")
    rng = np.random.default_rng(2024)
    out = {}
    for name, (ks, k, D, hi, sizes) in CASES.items():
        acc = metrics.TopKAccumulator(ks=ks)
        out[f"{name}/ks"] = np.array(ks, dtype=np.int64)
        out[f"{name}/batches"] = np.array(len(sizes))
        for i, B in enumerate(sizes):
            actual, top_k = batch(rng, B, k, D, hi)
            out[f"{name}/actual{i}"], out[f"{name}/top_k{i}"] = actual.astype(np.int16), top_k.astype(np.int16)
            acc.accumulate(actual=torch.from_numpy(actual), top_k=torch.from_numpy(top_k))
        red = acc.reduce()
        out[f"{name}/keys"] = np.array(list(red))
        out[f"{name}/values"] = np.array(list(red.values()), dtype=np.float64)
        acc.reset()
        assert acc.reduce() == {}
    np.savez(os.path.join(HERE, "metrics.npz"), **out)
    print({k: v for k, v in out.items() if k.endswith(("keys", "values"))})


if __name__ == "__main__":
    main()
