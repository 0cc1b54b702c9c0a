#!/usr/bin/env python
"""bench_train_decoder.py -- the generative-retrieval model's training step for every (encoder, decoder) pair of HF's passes and the
fused ones.

    python bench_train_decoder.py [--min-window-s 1.0] [--windows 3]

At the configs/decoder_amazon.gin T5 shape (d_model 384, 6 heads, d_ff 1024, 4 layers, K = 256, 3 levels, randomly initialised,
training mode with HF's dropout 0.1, the module's matmul precision "high", TF32), for three history sets:
  * "uniform": batch 640, lengths uniform over 2..20 items, end-padded to 20 (SeqData's subsample=True windows);
  * "full":    batch 640, every history 20 items;
  * "ml1m":    batch 64, every history 200 items (ML-1M's max_seq_len; 801 encoder positions);
it reports:
  * ms per training step -- ``model(batch, encoder=..., decoder=...)``, ``loss.backward()``, ``AdamW.step()`` and ``zero_grad`` --
    for the four arms (encoder, decoder) in {hf, fused}^2, alternating the arms, --windows windows of at least --min-window-s
    seconds each (CUDA events);
  * torch.cuda.max_memory_allocated during one step of each arm (model, optimizer state and inputs included);
  * a CUDA-event split of each arm's step: encoder forward, decoder + heads forward, decoder + heads backward, encoder backward
    (the encoder output's gradient through the encoder) and optimizer.  The split cuts the step at the encoder output, so it
    runs the fused pair as two graph breaks instead of one;
Prints the card's name, power limit and max SM clock, read in the same run, and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_generate import _card, corpus_of, timed_ms  # noqa: E402

K, H = 256, 3
SHAPE = dict(num_hierarchies=H, num_embeddings_per_hierarchy=K, t5_d_model=384, t5_num_heads=6, t5_d_ff=1024, t5_num_layers=4,
             top_k_for_generation=10, should_add_sep_token=True)
SETS = {"uniform": (640, 20, (2, 20)), "full": (640, 20, None), "ml1m": (64, 200, None)}


def batch_of(torch, rs, B, items, lengths):
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch
    W = H + 1
    sem = torch.from_numpy(rs.randint(0, K, size=(B, items * W))).cuda()
    sem.view(B, items, W)[:, :, H] = torch.from_numpy(rs.randint(0, 3, size=(B, items))).cuda()
    L = torch.full((B,), items) if lengths is None else torch.from_numpy(rs.randint(lengths[0], lengths[1] + 1, size=B))
    seq_mask = (torch.arange(items * W)[None, :] < (L[:, None] * W)).cuda()
    fut = torch.from_numpy(rs.randint(0, K, size=(B, W))).cuda()
    users = torch.from_numpy(rs.randint(0, 100, size=(B, 1))).cuda()
    return TokenizedSeqBatch(user_ids=users, sem_ids=sem, sem_ids_fut=fut, seq_mask=seq_mask,
                             token_type_ids=torch.zeros_like(sem), token_type_ids_fut=torch.zeros_like(fut))


ARMS = [("hf", "hf"), ("fused", "hf"), ("hf", "fused"), ("fused", "fused")]


def step_fn(m, opt, batch, encoder, decoder):
    def step():
        out = m(batch, encoder=encoder, decoder=decoder)
        out.loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
    return step


def step_split(torch, M, m, opt, batch, encoder, decoder, reps=10, attention="fp32"):
    """Mean ms of the step's encoder forward, decoder + heads forward, decoder + heads backward, encoder backward and optimizer,
    over reps steps with CUDA events; ``attention`` is the fused encoder's attention precision."""
    Hh = m.num_hierarchies
    names = ("encoder_forward_ms", "decoder_forward_ms", "decoder_backward_ms", "encoder_backward_ms", "optimizer_ms")
    tot = [0.0] * len(names)
    for rep in range(reps + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
        ev[0].record()
        mask = M._strip_dedup_col(batch.seq_mask.long(), Hh + 1, Hh)
        ids = M._strip_dedup_col(batch.sem_ids, Hh + 1, Hh)
        fut = batch.sem_ids_fut[:, :Hh]
        if encoder == "fused" and decoder == "fused":
            packed = M.FusedT5EncodeTrain(m, attention).packed(mask, ids, batch.user_ids)
            out = packed.rows
        elif encoder == "fused":
            out, enc_mask = m._fused_train_encoder_pass(mask, ids, batch.user_ids, attention)
        else:
            out, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids, user_id=batch.user_ids)
        ev[1].record()
        leaf = out.detach().requires_grad_()
        if encoder == "fused" and decoder == "fused":
            key_mask = packed.key_mask.index_select(0, torch.div(packed.src, packed.S, rounding_mode="floor").long())
            dec = M.FusedT5DecodeTrain(m)(fut, leaf, packed.offsets, key_mask, packed.src, packed.S)
        elif decoder == "fused":
            dec = m._fused_train_decoder_pass(fut, leaf, enc_mask)
        else:
            dec = m.decoder_forward_pass(future_ids=fut, encoder_output=leaf, attention_mask_for_encoder=enc_mask)[:, :-1]
        loss = sum(torch.nn.functional.cross_entropy(m.decoder_mlp[h](dec[:, h]), fut[:, h].long()) for h in range(Hh))
        ev[2].record()
        loss.backward()
        ev[3].record()
        out.backward(leaf.grad)
        ev[4].record()
        opt.step()
        opt.zero_grad(set_to_none=True)
        ev[5].record()
        torch.cuda.synchronize()
        if rep:
            for i in range(len(names)):
                tot[i] += ev[i].elapsed_time(ev[i + 1])
    return {name: t / reps for name, t in zip(names, tot)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-window-s", type=float, default=1.0)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--sets", default=",".join(SETS))
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_decoder.py measures on a CUDA device; none is visible")
    from rq_vae_recommender_b200.modules import model as M
    card = _card()
    print(f"card: {card}")
    result = {"card": card, "precision": torch.get_float32_matmul_precision(), "sets": {}}
    for name in args.sets.split(","):
        B, items, lengths = SETS[name]
        rs = np.random.RandomState(0)
        torch.manual_seed(0)
        m = M.EncoderDecoderRetrievalModel(codebooks=torch.from_numpy(corpus_of(np, 3000, 1, K, H)), **SHAPE).cuda().train()
        opt = torch.optim.AdamW(m.parameters(), lr=1e-4)
        batch = batch_of(torch, rs, B, items, lengths)
        steps = {f"{enc}/{dec}": step_fn(m, opt, batch, enc, dec) for enc, dec in ARMS}
        mem = {}
        for enc, fn in steps.items():
            fn()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            fn()
            torch.cuda.synchronize()
            mem[enc] = torch.cuda.max_memory_allocated() / 2 ** 20
        times = {enc: [] for enc in steps}
        for _ in range(args.windows):
            for enc, fn in steps.items():
                times[enc].append(timed_ms(torch, fn, args.min_window_s))
        split = {f"{enc}/{dec}": step_split(torch, M, m, opt, batch, enc, dec) for enc, dec in ARMS}
        kept = float(batch.seq_mask.float().mean())
        row = {"batch": B, "items": items, "lengths": "uniform %d..%d" % lengths if lengths else "all %d" % items,
               "kept_fraction_of_ids": round(kept, 3),
               "step_ms": {enc: [round(t, 2) for t in ts] for enc, ts in times.items()},
               "peak_mib": {enc: round(v, 1) for enc, v in mem.items()},
               "split_ms": {arm: {k: round(v, 2) for k, v in sp.items()} for arm, sp in split.items()}}
        row["speedup_median_vs_hf"] = {arm: round(float(np.median(times["hf/hf"]) / np.median(ts)), 3) for arm, ts in times.items()}
        print(f"{name}: B={B} items={items} {row['lengths']}")
        for arm in steps:
            print(f"  {arm:12s} step ms {row['step_ms'][arm]} (x{row['speedup_median_vs_hf'][arm]} vs hf/hf), peak MiB "
                  f"{row['peak_mib'][arm]}, split {row['split_ms'][arm]}")
        result["sets"][name] = row
        del m, opt, batch, steps
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
