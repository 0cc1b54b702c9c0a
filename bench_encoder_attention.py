#!/usr/bin/env python
"""bench_encoder_attention.py -- the fused T5 encoder's self-attention in fp32 (csrc/t5enc.cu) against TF32 tensor cores
(csrc/t5enc_tc.cu, encoder_attention="tf32").

    python bench_encoder_attention.py [--min-window-s 1.0] [--windows 3] [--parts train,generate,kernels]

At the configs/decoder_amazon.gin T5 shape (d_model 384, 6 heads, d_ff 1024, 4 layers, K = 256, 3 levels, random init, matmul
precision "high"), it reports:
  * train:    bench_train_decoder.py's history sets (uniform, full, ml1m; training mode, dropout 0.1): ms per training step for
              hf/hf, fused/fused with "fp32" and fused/fused with "tf32" attention, the arms alternated over --windows windows of
              at least --min-window-s seconds (CUDA events); peak memory of one step; the step split of
              bench_train_decoder.step_split (encoder forward / backward among others);
  * generate: the encoder pass of generate on bench_decode.py --part encoder's history sets (64 x 20 items full and uniform,
              64 x 200 items full), encoder="hf", "fused" + "fp32" and "fused" + "tf32", alternated;
  * kernels:  the attention forward (training, dropout 0.1) and backward at the training sets' packed shapes, fp32 against tf32
              (CUDA events), beside the TF32 FLOP floor at the data sheet's 495 TFLOP/s: the useful products (2 forward, 7
              backward) over each history's kept rows, and the same with every history padded to 64-row tiles.
Prints the card's name, power limit and max SM clock, read in the same run, and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench_decode  # noqa: E402
import bench_train_decoder as btd  # noqa: E402
from bench_generate import _card, corpus_of, timed_ms  # noqa: E402

TF32_PEAK = 495e12                      # dense TF32 FLOP/s of the H100 SXM data sheet (700 W)
TRAIN_ARMS = [("hf/hf", "hf", "fp32"), ("fused/fused fp32", "fused", "fp32"), ("fused/fused tf32", "fused", "tf32")]


def train_step(m, opt, batch, encoder, attention):
    def step():
        kw = {"encoder_attention": attention} if encoder == "fused" else {}
        m(batch, encoder=encoder, decoder=encoder, **kw).loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
    return step


def floors(counts, heads):
    """TF32 FLOPs of the attention's products: (useful, tile-padded) for one forward (2 products) and one backward (7)."""
    useful = sum(c * c for c in counts) * heads * 64 * 2
    padded = sum((-(-c // 64) * 64) ** 2 for c in counts) * heads * 64 * 2
    return {"forward": (2 * useful, 2 * padded), "backward": (7 * useful, 7 * padded)}


def run_train(torch, np, M, ops, args, kernels):
    out = {}
    for name, (B, items, lengths) in btd.SETS.items():
        rs = np.random.RandomState(0)
        torch.manual_seed(0)
        m = M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus_of(np, 3000, 1, btd.K, btd.H)), **btd.SHAPE).cuda().train()
        opt = torch.optim.AdamW(m.parameters(), lr=1e-4)
        batch = btd.batch_of(torch, rs, B, items, lengths)
        steps = {arm: train_step(m, opt, batch, enc, att) for arm, enc, att in TRAIN_ARMS}
        mem = {}
        for arm, fn in steps.items():
            fn()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            fn()
            torch.cuda.synchronize()
            mem[arm] = torch.cuda.max_memory_allocated() / 2 ** 20
        times = {arm: [] for arm in steps}
        for _ in range(args.windows):
            for arm, fn in steps.items():
                times[arm].append(timed_ms(torch, fn, args.min_window_s))
        split = {arm: btd.step_split(torch, M, m, opt, batch, enc, enc, attention=att) for arm, enc, att in TRAIN_ARMS}
        row = {"batch": B, "items": items, "lengths": "uniform %d..%d" % lengths if lengths else "all %d" % items,
               "step_ms": {a: [round(t, 2) for t in ts] for a, ts in times.items()},
               "speedup_median_vs_hf": {a: round(float(np.median(times["hf/hf"]) / np.median(ts)), 3) for a, ts in times.items()},
               "peak_mib": {a: round(v, 1) for a, v in mem.items()},
               "split_ms": {a: {k: round(v, 2) for k, v in sp.items()} for a, sp in split.items()}}
        print(f"train {name}: B={B} items={items} {row['lengths']}")
        for arm in steps:
            print(f"  {arm:18s} step ms {row['step_ms'][arm]} (x{row['speedup_median_vs_hf'][arm]} vs hf/hf), peak MiB "
                  f"{row['peak_mib'][arm]}, split {row['split_ms'][arm]}")
        out[name] = row
        if kernels:
            with torch.no_grad():
                H = m.num_hierarchies
                packed = M.FusedT5EncodeTrain(m).packed(M._strip_dedup_col(batch.seq_mask.long(), H + 1, H),
                                                       M._strip_dedup_col(batch.sem_ids, H + 1, H), batch.user_ids)
            out[name]["kernels"] = kernel_times(torch, ops, packed, m.encoder.encoder.config.num_heads, args)
        del m, opt, batch, steps
        torch.cuda.empty_cache()
    return out


def kernel_times(torch, ops, packed, heads, args):
    offs, src, key_mask, S = packed.offsets, packed.src, packed.key_mask, packed.S
    N, inner = src.shape[0], heads * 64
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv = torch.randn(N, 3 * inner, device="cuda", generator=g) * 0.3
    rel = torch.randn(heads, 2 * S - 1, device="cuda", generator=g)
    dout = torch.randn(N, inner, device="cuda", generator=g)
    seed = torch.tensor([7], dtype=torch.int64, device="cuda")
    fns = {}
    for att, fwd, bwd in (("fp32", ops.t5enc_attention_train, ops.t5enc_attention_backward),
                          ("tf32", ops.t5enc_attention_tc_train, ops.t5enc_attention_tc_backward)):
        o, lse = fwd(qkv, src, offs, key_mask, rel, S, seed, 0.1)
        fns[f"forward_{att}"] = (lambda fwd=fwd: fwd(qkv, src, offs, key_mask, rel, S, seed, 0.1))
        fns[f"backward_{att}"] = (lambda bwd=bwd, o=o, lse=lse: bwd(qkv, o, dout, lse, src, offs, key_mask, rel, S, seed, 0.1))
    times = {k: [] for k in fns}
    for _ in range(args.windows):
        for k, fn in fns.items():
            times[k].append(timed_ms(torch, fn, args.min_window_s / 4))
    counts = (offs[1:] - offs[:-1]).tolist()
    fl = floors(counts, heads)
    res = {"S": S, "rows": N, "ms": {k: [round(t, 4) for t in ts] for k, ts in times.items()}}
    for part in ("forward", "backward"):
        useful, padded = fl[part]
        best = min(times[f"{part}_tf32"])
        res[f"{part}_tf32_floor_ms"] = round(useful / TF32_PEAK * 1e3, 4)
        res[f"{part}_tf32_padded_floor_ms"] = round(padded / TF32_PEAK * 1e3, 4)
        res[f"{part}_tf32_share_of_floor"] = round(useful / TF32_PEAK * 1e3 / best, 3)
        res[f"{part}_tf32_faster_in_every_window"] = all(t < f for t, f in zip(times[f"{part}_tf32"], times[f"{part}_fp32"]))
    print(f"  kernels S={S}: {res}")
    return res


def run_generate(torch, np, M, args):
    corpus = torch.from_numpy(corpus_of(np, 12101, 12101, bench_decode.K, 3))
    torch.manual_seed(0)
    m = M.EncoderDecoderRetrievalModel(codebooks=corpus, num_hierarchies=3, **bench_decode.SHAPE).cuda().eval()
    out = []
    for kind, B, items in (("full", bench_decode.B, bench_decode.ITEMS), ("uniform", bench_decode.B, bench_decode.ITEMS),
                           ("full", bench_decode.LONG_B, bench_decode.LONG_ITEMS)):
        mask, ids = bench_decode.history_set(torch, np, kind, B, items, 3)
        fns = {"hf": lambda: m.encoder_forward_pass(attention_mask=mask, input_ids=ids),
               "fused_fp32": lambda: m._fused_encoder("fp32")(mask, ids),
               "fused_tf32": lambda: m._fused_encoder("tf32")(mask, ids)}
        times = {k: [] for k in fns}
        with torch.no_grad():
            enc32, _ = fns["fused_fp32"]()
            enctc, _ = fns["fused_tf32"]()
            for _ in range(args.windows):
                for k, fn in fns.items():
                    times[k].append(timed_ms(torch, fn, args.min_window_s))
        row = {"history_set": kind, "batch": B, "items": items, "encoder_ms": {k: [round(t, 3) for t in ts] for k, ts in times.items()},
               "max_abs_enc_out_diff_tf32_vs_fp32": float((enc32 - enctc).abs().max())}
        print(f"generate encoder {kind} {B}x{items}: {row['encoder_ms']}")
        out.append(row)
    del m
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-window-s", type=float, default=1.0)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--parts", default="train,generate,kernels")
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_encoder_attention.py measures on a CUDA device; none is visible")
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    parts = args.parts.split(",")
    card = _card()
    print(f"card: {card}")
    result = {"card": card, "precision": torch.get_float32_matmul_precision()}
    if "train" in parts or "kernels" in parts:
        result["train"] = run_train(torch, np, M, ops, args, "kernels" in parts)
    if "generate" in parts:
        result["generate"] = run_generate(torch, np, M, args)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
