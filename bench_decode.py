#!/usr/bin/env python
"""bench_decode.py -- whole generate of the generative-retrieval model with HF's decoder passes against the fused decode.

    python bench_decode.py [--min-window-s 1.0]

At the configs/decoder_amazon.gin evaluation shape (batch 640, top_k_for_generation 10, K = 256, d_model 384, 6 heads, d_ff 1024,
4 layers, randomly initialised, 20-item histories, a 12 101-row corpus), with 3 hierarchy levels and again with 5:
  * ms per generate call for four arms, decoder "hf" / "fused" x search "sample" / "beam", alternating, three windows of at least
    --min-window-s seconds each (CUDA events, after warm-up), at the module's matmul precision ("high", TF32);
  * torch.cuda.max_memory_allocated during one call of each arm (the model and inputs included);
  * for the fused arms, a per-level split from CUDA events: the encoder pass (with the one cross key/value projection and the
    prefix index lookup), then per level the decoder step and the head + search;
  * whether the two decoders return equal beams (same seed for "sample"), the fraction of histories whose beams are all equal,
    and the largest |log-probability difference| over beams finite under both, at every position and at positions where both
    decoders returned the same ids.
Prints the card's name, power limit and max SM clock, read in the same run, and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_generate import _card, corpus_of, timed_ms  # noqa: E402

B, TOP_K, K, ITEMS = 640, 10, 256, 20
SHAPE = dict(num_embeddings_per_hierarchy=K, t5_d_model=384, t5_num_heads=6, t5_d_ff=1024, t5_num_layers=4,
             top_k_for_generation=TOP_K, should_add_sep_token=True)


def fused_split(torch, F, M, m, mask, ids, search, reps=20):
    """Mean ms of the encoder pass (+ cross K/V projection) and, per level, of the decoder step and of head + search, over reps
    calls of generate's fused loop restated with CUDA events between its parts."""
    H, k = m.num_hierarchies, m.top_k_for_generation
    n_cands = min(M.MAX_CANDIDATES, K)
    totals = None
    for rep in range(reps + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 + 2 * H)]
        ev[0].record()
        with torch.no_grad():
            enc_out, enc_mask = m.encoder_forward_pass(attention_mask=mask, input_ids=ids)
            index = m._prefix_index(enc_out.device)
            fused = m._fused_decoder(enc_out, enc_mask, k)
            ev[1].record()
            generated, log_probas, parent = None, None, None
            reject = torch.zeros(2, dtype=torch.int32, device="cuda")
            for h in range(H):
                hid = fused.step(h, generated, parent)
                ev[2 + 2 * h].record()
                logits = m.decoder_mlp[h](hid)
                if search == "beam":
                    generated, log_probas, parent = index.beam_topk(logits, generated, log_probas, k, bad=reject)
                else:
                    generated, log_probas, parent = m._sample_and_select(index, F.softmax(logits, dim=-1), generated, log_probas,
                                                                         k, n_cands, reject)
                ev[3 + 2 * h].record()
        torch.cuda.synchronize()
        if rep == 0:                                          # warm-up
            continue
        t = [ev[0].elapsed_time(ev[1])] + [ev[i].elapsed_time(ev[i + 1]) for i in range(1, 1 + 2 * H)]
        totals = t if totals is None else [a + b for a, b in zip(totals, t)]
    t = [x / reps for x in totals]
    return {"encoder_ms": t[0], "levels": [{"decoder_step_ms": t[1 + 2 * h], "head_search_ms": t[2 + 2 * h]} for h in range(H)]}


def run_shape(torch, F, np, M, levels, w):
    corpus = torch.from_numpy(corpus_of(np, 12101, 12101, K, levels))
    torch.manual_seed(0)
    m = M.EncoderDecoderRetrievalModel(codebooks=corpus, num_hierarchies=levels, **SHAPE).cuda().eval()
    rs = np.random.RandomState(1)
    ids = torch.from_numpy(rs.randint(0, K, size=(B, ITEMS * levels))).cuda()
    mask = torch.ones_like(ids)
    arms = [(dec, search) for search in ("sample", "beam") for dec in ("hf", "fused")]
    res = {"levels": levels}
    outs = {}
    for dec, search in arms:
        m.generate(mask, ids, search=search, decoder=dec)    # warm-up (builds the index)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        torch.manual_seed(3)
        outs[dec, search] = m.generate(mask, ids, search=search, decoder=dec)
        torch.cuda.synchronize()
        res[f"{dec}_{search}_peak_bytes"] = torch.cuda.max_memory_allocated()
    for search in ("sample", "beam"):
        (gh, ph), (gf, pf) = outs["hf", search], outs["fused", search]
        fin = torch.isfinite(ph) & torch.isfinite(pf)
        res[f"{search}_beams_equal"] = bool(torch.equal(gh, gf))
        res[f"{search}_rows_with_equal_beams"] = float((gh == gf).reshape(B, -1).all(1).float().mean())
        res[f"{search}_max_abs_log_proba_diff"] = float((ph[fin] - pf[fin]).abs().max()) if fin.any() else None
        same = fin & (gh == gf).all(-1)
        res[f"{search}_max_abs_log_proba_diff_equal_beams"] = float((ph[same] - pf[same]).abs().max()) if same.any() else None
    times = {f"{dec}_{search}_ms": [] for dec, search in arms}
    for _ in range(3):                                        # alternate the arms: clock drift hits all alike
        for dec, search in arms:
            times[f"{dec}_{search}_ms"].append(timed_ms(torch, lambda: m.generate(mask, ids, search=search, decoder=dec), w))
    res.update(times)
    res["fused_faster_in_every_pair"] = {
        search: all(f < h for f, h in zip(times[f"fused_{search}_ms"], times[f"hf_{search}_ms"])) for search in ("sample", "beam")}
    res["fused_split"] = {search: fused_split(torch, F, M, m, mask, ids, search) for search in ("sample", "beam")}
    del m
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-window-s", type=float, default=1.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import torch.nn.functional as F
    from rq_vae_recommender_b200.modules import model as M
    assert torch.cuda.is_available(), "bench_decode.py measures on a CUDA device"
    out = {"card": _card(), "batch": B, "top_k": TOP_K, "codes": K, "history_items": ITEMS,
           "t5": "d_model 384, 6 heads, d_ff 1024, 4 layers, random init, matmul precision " + torch.get_float32_matmul_precision()}
    out["levels3"] = run_shape(torch, F, np, M, 3, args.min_window_s)
    out["levels5"] = run_shape(torch, F, np, M, 5, args.min_window_s)
    out["timed"] = "CUDA events, windows >= %.1f s after warm-up, arms alternated" % args.min_window_s
    print(out["card"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
