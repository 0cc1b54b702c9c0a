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
The encoder part, at the same T5 shape with 3 levels and the fused decoder, for two history sets of batch 640 (every history 20
items, and seeded lengths uniform over 1..20 items, end-padded) and for 64 histories of 200 items (encoder pass only):
  * a CUDA-event split of HF's encoder pass into its nn.Linear calls (the GEMMs) and the rest;
  * ms per encoder pass, encoder "hf" against "fused", alternating, and ms per generate call for encoder "hf" / "fused" x search
    "sample" / "beam" with decoder "fused", alternating;
  * the largest |encoder output difference| at kept positions, and whether the beams agree (same seed for "sample").
``--part decoder`` / ``--part encoder`` runs one part only.
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


def hf_encoder_split(torch, m, mask, ids, reps=20):
    """Mean ms of HF's encoder pass and the part of it spent in the encoder's nn.Linear calls (the GEMMs), from CUDA events
    recorded around every Linear by forward hooks; the rest is the eager attention, norms, residual adds and input assembly."""
    linears = [mod for mod in m.encoder.modules() if isinstance(mod, torch.nn.Linear)]
    pairs = []
    pre = lambda mod, inp: pairs.append([torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)]) or \
        pairs[-1][0].record()
    post = lambda mod, inp, out: pairs[-1][1].record()
    hooks = [h for mod in linears for h in (mod.register_forward_pre_hook(pre), mod.register_forward_hook(post))]
    total = gemm = 0.0
    try:
        for rep in range(reps + 1):
            pairs.clear()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            with torch.no_grad():
                m.encoder_forward_pass(attention_mask=mask, input_ids=ids)
            b.record()
            torch.cuda.synchronize()
            if rep == 0:
                continue
            total += a.elapsed_time(b)
            gemm += sum(s.elapsed_time(e) for s, e in pairs)
    finally:
        for h in hooks:
            h.remove()
    return {"encoder_ms": total / reps, "gemm_ms": gemm / reps, "rest_ms": (total - gemm) / reps, "linear_calls": len(pairs)}


def history_set(torch, np, kind, batch, items, levels, seed=1):
    """ids [batch, items * levels] and the mask: "full" (every item), or "uniform" (lengths uniform over 1..items, end-padded
    like the reference's SeqData, whose padded ids are -1: masked ids read table row 0 either way)."""
    rs = np.random.RandomState(seed)
    ids = torch.from_numpy(rs.randint(0, K, size=(batch, items * levels))).cuda()
    mask = torch.ones_like(ids)
    if kind == "uniform":
        lengths = rs.randint(1, items + 1, size=batch)
        for b, n in enumerate(lengths):
            mask[b, n * levels:] = 0
            ids[b, n * levels:] = -1
    return mask, ids


def encoder_arms(torch, np, M, m, kind, batch, items, w, generate_arms=True):
    """Encoder pass alone, HF against fused, and (generate_arms) whole generate with decoder="fused" for both encoders and both
    searches, every group of arms alternated; output agreement at the module's matmul precision."""
    levels = m.num_hierarchies
    mask, ids = history_set(torch, np, kind, batch, items, levels)
    res = {"history_set": kind, "batch": batch, "items": items}
    with torch.no_grad():
        enc_h, mask_h = m.encoder_forward_pass(attention_mask=mask, input_ids=ids)
        st = m._fused_encoder()
        enc_f, mask_f = st(mask, ids)
    kept = mask_h != 0
    kept[~kept.any(1)] = True
    res["positions"] = int(mask_h.numel())
    res["kept_positions"] = st.n_kept
    res["enc_masks_equal"] = bool(torch.equal(mask_h, mask_f))
    res["max_abs_enc_out_diff_kept"] = float((enc_h[kept] - enc_f[kept]).abs().max())
    res["dropped_rows_zero"] = bool((enc_f[~kept] == 0).all())
    res["hf_encoder_split"] = hf_encoder_split(torch, m, mask, ids)
    fns = {"hf": lambda: m.encoder_forward_pass(attention_mask=mask, input_ids=ids), "fused": lambda: m._fused_encoder()(mask, ids)}
    times = {f"encoder_{e}_ms": [] for e in fns}
    with torch.no_grad():
        for _ in range(3):
            for e, fn in fns.items():
                times[f"encoder_{e}_ms"].append(timed_ms(torch, fn, w))
    res.update(times)
    res["encoder_fused_faster_in_every_pair"] = all(f < h for f, h in zip(times["encoder_fused_ms"], times["encoder_hf_ms"]))
    if not generate_arms:
        return res
    arms = [(enc, search) for search in ("sample", "beam") for enc in ("hf", "fused")]
    outs = {}
    for enc, search in arms:
        torch.manual_seed(3)
        outs[enc, search] = m.generate(mask, ids, search=search, decoder="fused", encoder=enc)
    for search in ("sample", "beam"):
        (gh, ph), (gf, pf) = outs["hf", search], outs["fused", search]
        fin = torch.isfinite(ph) & torch.isfinite(pf)
        same = fin & (gh == gf).all(-1)
        res[f"{search}_beams_equal"] = bool(torch.equal(gh, gf))
        res[f"{search}_rows_with_equal_beams"] = float((gh == gf).reshape(batch, -1).all(1).float().mean())
        res[f"{search}_max_abs_log_proba_diff_equal_beams"] = float((ph[same] - pf[same]).abs().max()) if same.any() else None
    gt = {f"generate_{enc}_{search}_ms": [] for enc, search in arms}
    for _ in range(3):
        for enc, search in arms:
            gt[f"generate_{enc}_{search}_ms"].append(
                timed_ms(torch, lambda: m.generate(mask, ids, search=search, decoder="fused", encoder=enc), w))
    res.update(gt)
    res["generate_fused_encoder_faster_in_every_pair"] = {
        search: all(f < h for f, h in zip(gt[f"generate_fused_{search}_ms"], gt[f"generate_hf_{search}_ms"]))
        for search in ("sample", "beam")}
    return res


def run_encoder(torch, np, M, w):
    corpus = torch.from_numpy(corpus_of(np, 12101, 12101, K, 3))
    torch.manual_seed(0)
    m = M.EncoderDecoderRetrievalModel(codebooks=corpus, num_hierarchies=3, **SHAPE).cuda().eval()
    m.generate(*history_set(torch, np, "full", 8, ITEMS, 3), decoder="fused")     # builds the prefix index
    out = [encoder_arms(torch, np, M, m, kind, B, ITEMS, w) for kind in ("full", "uniform")]
    out.append(encoder_arms(torch, np, M, m, "full", LONG_B, LONG_ITEMS, w, generate_arms=False))
    del m
    torch.cuda.empty_cache()
    return out


LONG_B, LONG_ITEMS = 64, 200           # MovieLens-length histories (S = 800 encoder positions)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-window-s", type=float, default=1.0)
    ap.add_argument("--part", choices=("all", "decoder", "encoder"), default="all",
                    help="decoder: HF against fused decoder passes at 3 and 5 levels; encoder: HF against fused encoder pass")
    args = ap.parse_args()
    import numpy as np
    import torch
    import torch.nn.functional as F
    from rq_vae_recommender_b200.modules import model as M
    assert torch.cuda.is_available(), "bench_decode.py measures on a CUDA device"
    out = {"card": _card(), "batch": B, "top_k": TOP_K, "codes": K, "history_items": ITEMS,
           "t5": "d_model 384, 6 heads, d_ff 1024, 4 layers, random init, matmul precision " + torch.get_float32_matmul_precision()}
    if args.part in ("all", "decoder"):
        out["levels3"] = run_shape(torch, F, np, M, 3, args.min_window_s)
        out["levels5"] = run_shape(torch, F, np, M, 5, args.min_window_s)
    if args.part in ("all", "encoder"):
        out["encoder"] = run_encoder(torch, np, M, args.min_window_s)
    out["timed"] = "CUDA events, windows >= %.1f s after warm-up, arms alternated" % args.min_window_s
    print(out["card"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
