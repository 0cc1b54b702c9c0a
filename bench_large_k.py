#!/usr/bin/env python
"""bench_large_k.py -- the tensor-core tokeniser with codebooks of 512, 1024 and 2048 codes.

    python bench_large_k.py [--rows N]

For K in {512, 1024, 2048}, L = 3 and D = 768 and D = 64 (the ml-32m quantiser width), 65 536 unit-norm rows by default:
device-timed ms of ops.rq_tokenize_tc with a prepared state against the exact CUDA-core kernel ops.rq_tokenize at the same
shape, the fraction of row-levels that go to the exact re-rank, prepare ms, state MB, and the number of rows whose ids
differ from the exact kernel's.  Codebooks are drawn from an 8 192-row residual walk, as bench.py's make_problem does
(the float64 walk over all rows is too slow at large K).  Prints one JSON line; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

L = 3


def _event_ms(torch, fn, n=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def _card():
    """Name, power limit and max SM clock of GPU 0 (read-only query); the numbers are only meaningful beside them."""
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    args = ap.parse_args()
    import torch
    import inputs as I
    from rq_vae_recommender_b200 import ops
    n = args.rows
    out = {"rows": n, "levels": L, "card": _card()}
    for d in (768, 64):
        x_h = I.unit_rows(555 + d, n, d)
        x = torch.from_numpy(x_h).cuda()
        for k in (512, 1024, 2048):
            _, cbs_h = I.rq_problem(max(8192, k), d, k, L, seed=555 + d, x=I.unit_rows(555 + d, max(8192, k), d))
            cbs = [torch.from_numpy(c).cuda() for c in cbs_h]
            prep_ms = _event_ms(torch, lambda: ops.TcState(cbs), n=3, warm=1)
            st = ops.TcState(cbs)
            stats = torch.zeros(4, dtype=torch.int32, device="cuda")
            with torch.no_grad():
                tc_ms = _event_ms(torch, lambda: ops.rq_tokenize_tc(x, state=st), n=10)
                ex_ms = _event_ms(torch, lambda: ops.rq_tokenize(x, cbs), n=3, warm=1)
                ids_tc = ops.rq_tokenize_tc(x, state=st, stats=stats)
                ids_ex = ops.rq_tokenize(x, cbs)
            s_h = stats.cpu().tolist()
            out[f"K{k}_D{d}"] = {
                "tc_ms": tc_ms, "exact_ms": ex_ms, "speedup_vs_exact": ex_ms / tc_ms,
                "rerank_fraction_of_row_levels": s_h[0] / float(n * L),
                "candidates_per_reranked_row": s_h[1] / max(s_h[0], 1),
                "prepare_ms": prep_ms, "state_mb": st.nbytes / 1e6,
                "rows_differing_from_exact": int((ids_tc != ids_ex).any(1).sum().item())}
            del st, cbs
        del x
    out["timed"] = "ops.rq_tokenize_tc (prepared state) and ops.rq_tokenize (exact CUDA-core kernel), device resident, CUDA events"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
