#!/usr/bin/env python
"""bench_generate.py -- the prefix-constrained beam searches of the generative-retrieval model, sampled and exhaustive.

    python bench_generate.py [--min-window-s 1.0]

At the shipped evaluation settings (configs/decoder_amazon.gin: batch 640, top_k_for_generation 10, 64 sampled candidates per
beam, K = 256 codes, 3 hierarchy levels), on a 12 101-row corpus (Amazon Beauty's size) and a 1 M-row synthetic one:
  * ms per level h = 0, 1, 2 for three arms that all start from the level's probabilities:
      reference   torch.multinomial, log/gather, the reference's prefix check (every prefix against every corpus row, in
                  100 000-prefix chunks), masked_fill, sort and gathers (modules/model.py's expression);
      composed    torch.multinomial, log/gather, then SidPrefixIndex.beam_select (one kernel);
      fused       draw_exponential, then SidPrefixIndex.sample_select (one kernel);
    the reference arm is not run on the 1 M-row corpus: one chunk would need 100 000 x 1 M x l bytes of bool temporaries;
    and two arms of the exhaustive search (generate(search="beam")) that start from the level's logits:
      beam            SidPrefixIndex.beam_topk (one kernel);
      beam_composed   torch: log_softmax, SidPrefixIndex.check of every extension, masked_fill, a stable descending sort,
                      gathers;
  * the two exhaustive arms again at top-k 32 and K = 2048 (65 536 candidates per history) on a 12 101-row corpus;
  * the corpus prefix index (the trie): build ms, the device bytes it keeps and the bytes of its build scratch, on a
    12 101-row corpus at K = 256, C = 3 (the shipped shape), K = 2048, C = 3 and K = 256, C = 4, and on a 1 048 576-row
    corpus at K = 256, C = 3;
  * per-level ms of sample_select (top-k 10, 64 candidates) and beam_topk (top-k 10) at deeper hierarchies and larger
    codebooks: K = 256 with C = 5 and 8, K = 1024 and 2048 with C = 4, and beam_topk at top-k 32 with K = 2048, C = 4 (65 536
    candidates per history), each on a 12 101-row corpus;
  * whole-generate ms of the drop-in EncoderDecoderRetrievalModel at the decoder_amazon.gin T5 shape (d_model 384, 6 heads,
    d_ff 1024, 4 layers, randomly initialised) on 20-item histories, of the same model with the composed arm in place of
    sample_select, under the same seed (their beams are compared), and of generate(search="beam"); three alternating windows
    each; and generate(search="sample") and generate(search="beam") of the same T5 shape with 5 hierarchy levels at K = 256.  Also the fraction of returned beams with a finite log-probability under each search (of this randomly
    initialised model: it says how often a search runs out of valid prefixes, not how good its beams are).
Every shape is warmed up, every timed window lasts at least --min-window-s seconds (CUDA events).  Prints the card's name,
power limit and max SM clock, and one JSON line; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

B, TOP_K, NC, K, H, ITEMS = 640, 10, 64, 256, 3, 20


def _card():
    """Name, power limit and max SM clock of GPU 0 (read-only query); the numbers are only meaningful beside them."""
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or None
    except Exception:
        return None


def timed_ms(torch, fn, min_window_s):
    """ms per call over a window of at least min_window_s seconds, after warm-up calls."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 1
    while True:
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b)
        if ms >= min_window_s * 1e3:
            return ms / n
        n = max(n * 2, int(n * min_window_s * 1e3 / max(ms, 1e-3) * 1.2) + 1)


def reference_level(torch, corpus, probas, generated, log_probas, k, nc):
    """modules/model.py's sampling and selection step, as the reference computes it."""
    samples = torch.multinomial(probas, num_samples=nc)
    samp_log_p = torch.log(torch.gather(probas, 1, samples))
    if generated is None:
        prefix = samples.reshape(-1, 1)
    else:
        h = generated.shape[2]
        prefix = torch.cat([generated.reshape(-1, h).repeat_interleave(nc, dim=0), samples.reshape(-1, 1)], dim=1)
    trimmed = corpus[:, : prefix.shape[1]]
    valid = torch.cat([(trimmed.unsqueeze(1) == prefix[i:i + 100000].unsqueeze(0)).all(dim=2).any(dim=0)
                       for i in range(0, prefix.shape[0], 100000)])
    Bn = probas.shape[0] if generated is None else generated.shape[0]
    if generated is None:
        scores, idx = samp_log_p.masked_fill(~valid.reshape(Bn, nc), float("-inf")).sort(-1, descending=True)
        return torch.gather(samples, 1, idx[:, :k]).unsqueeze(-1), scores[:, :k], None
    kp, h = generated.shape[1], generated.shape[2]
    total = samp_log_p.reshape(Bn, kp * nc) + log_probas.repeat_interleave(nc, dim=1)
    scores, idx = total.masked_fill(~valid.reshape(Bn, kp * nc), float("-inf")).sort(-1, descending=True)
    top = idx[:, :k]
    parent = top // nc
    parent_global = (parent + torch.arange(Bn, device=parent.device).unsqueeze(1) * kp).flatten()
    parent_ids = torch.gather(generated, 1, parent.unsqueeze(-1).expand(-1, -1, h))
    new_ids = torch.gather(samples.reshape(Bn, kp * nc), 1, top).unsqueeze(-1)
    return torch.cat([parent_ids, new_ids], dim=-1), scores[:, :k], parent_global


def composed_level(torch, index, probas, generated, log_probas, k, nc):
    samples = torch.multinomial(probas, num_samples=nc)
    samp_log_p = torch.log(torch.gather(probas, 1, samples))
    return index.beam_select(samples, samp_log_p, generated, log_probas, k)


def beam_composed_level(torch, F, index, logits, generated, log_probas, k):
    """One level of the exhaustive search in torch: log_softmax, the prefix check of every extension, masked_fill, a stable
    descending sort and gathers."""
    Kc = logits.shape[1]
    Bn, kp, h = (logits.shape[0], 1, 0) if generated is None else generated.shape
    codes = torch.arange(Kc, device=logits.device).repeat(Bn * kp).unsqueeze(1)
    prefix = codes if h == 0 else torch.cat([generated.reshape(-1, h).repeat_interleave(Kc, dim=0), codes], dim=1)
    scores = F.log_softmax(logits, dim=-1).reshape(Bn, kp * Kc)
    if h:
        scores = scores + log_probas.repeat_interleave(Kc, dim=1)
    scores = scores.masked_fill(~index.check(prefix).reshape(Bn, kp * Kc), float("-inf"))
    scores, idx = scores.sort(dim=-1, descending=True, stable=True)
    top = idx[:, :k]
    parent = top // Kc
    new_ids = (top % Kc).unsqueeze(-1)
    if h:
        new_ids = torch.cat([torch.gather(generated, 1, parent.unsqueeze(-1).expand(-1, -1, h)), new_ids], dim=-1)
    return new_ids, scores[:, :k], (parent + torch.arange(Bn, device=logits.device).unsqueeze(1) * kp).flatten()


def corpus_of(np, rows, seed, codes=K, levels=H):
    rs = np.random.RandomState(seed)
    return rs.randint(0, codes, size=(rows, levels)).astype(np.int64)


def level_inputs(torch, F, index, seed, codes=K, levels=H):
    """Per level: probabilities (softmax of random logits), the logits, and the beams entering it (from the fused chain)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out, generated, log_probas = [], None, None
    from rq_vae_recommender_b200.modules.model import draw_exponential
    for h in range(levels):
        rows = B if h == 0 else B * TOP_K
        logits = torch.randn(rows, codes, device="cuda", generator=g) * 3
        probas = F.softmax(logits, dim=-1)
        out.append((probas, logits, generated, log_probas))
        generated, log_probas, _ = index.sample_select(probas, draw_exponential(probas), generated, log_probas, TOP_K, NC)
    return out


def beam_level_inputs(torch, index, k, codes, seed, levels=H):
    """Per level: random logits and the beams entering it (from the exhaustive chain)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out, generated, log_probas = [], None, None
    for h in range(levels):
        logits = torch.randn(B if h == 0 else B * k, codes, device="cuda", generator=g) * 3
        out.append((logits, generated, log_probas))
        generated, log_probas, _ = index.beam_topk(logits, generated, log_probas, k)
    return out


def build_ms(torch, ops, corpus, codes, reps=5):
    """Median ms of building the prefix index (host clock around the build and a device synchronise), the bytes it keeps and
    the bytes of its build scratch."""
    import time
    from rq_vae_recommender_b200 import _lib
    times = []
    for _ in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        index = ops.SidPrefixIndex(corpus, codes)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
        nbytes = index.nbytes
        del index
    times = sorted(times[1:])                                  # the first build loads the module
    rows, levels = corpus.shape
    return {"build_ms": times[len(times) // 2], "bytes": nbytes,
            "scratch_bytes": _lib.load().rqb200_sid_trie_scratch_bytes(rows, levels, codes)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-window-s", type=float, default=1.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import torch.nn.functional as F
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    assert torch.cuda.is_available(), "bench_generate.py measures on a CUDA device"
    w = args.min_window_s
    out = {"card": _card(), "batch": B, "top_k": TOP_K, "candidates": NC, "codes": K, "levels": H}
    for name, rows in (("corpus_12101", 12101), ("corpus_1M", 1 << 20)):
        corpus = torch.from_numpy(corpus_of(np, rows, rows)).cuda()
        index = ops.SidPrefixIndex(corpus, K)
        res = {}
        for h, (probas, logits, generated, log_probas) in enumerate(level_inputs(torch, F, index, 7)):
            arms = {"composed_ms": lambda: composed_level(torch, index, probas, generated, log_probas, TOP_K, NC),
                    "fused_ms": lambda: index.sample_select(probas, M.draw_exponential(probas), generated, log_probas, TOP_K, NC),
                    "beam_ms": lambda: index.beam_topk(logits, generated, log_probas, TOP_K),
                    "beam_composed_ms": lambda: beam_composed_level(torch, F, index, logits, generated, log_probas, TOP_K)}
            if rows < 100000:
                arms["reference_ms"] = lambda: reference_level(torch, corpus, probas, generated, log_probas, TOP_K, NC)
            res[f"level{h}"] = {arm: timed_ms(torch, fn, w) for arm, fn in arms.items()}
        out[name] = res
        del index, corpus
        torch.cuda.empty_cache()
    big_k, big_codes = 32, 2048                               # 65 536 candidates per history
    corpus = torch.from_numpy(corpus_of(np, 12101, 12101, big_codes)).cuda()
    index = ops.SidPrefixIndex(corpus, big_codes)
    res = {}
    for h, (logits, generated, log_probas) in enumerate(beam_level_inputs(torch, index, big_k, big_codes, 8)):
        want = index.beam_topk(logits, generated, log_probas, big_k)
        got = beam_composed_level(torch, F, index, logits, generated, log_probas, big_k)
        res[f"level{h}"] = {
            "beam_ms": timed_ms(torch, lambda: index.beam_topk(logits, generated, log_probas, big_k), w),
            "beam_composed_ms": timed_ms(torch, lambda: beam_composed_level(torch, F, index, logits, generated, log_probas, big_k), w),
            "rows_with_equal_beams": float((want[0] == got[0]).reshape(B, -1).all(1).float().mean()),
            "log_probas_max_abs_diff": float((want[1] - got[1]).nan_to_num(posinf=0, neginf=0).abs().max())}
    out["beam_top_k32_codes2048_corpus_12101"] = res
    del index, corpus
    torch.cuda.empty_cache()
    builds = {}
    for codes, levels in ((K, 3), (2048, 3), (K, 4)):
        corpus = torch.from_numpy(corpus_of(np, 12101, 12101, codes, levels)).cuda()
        builds[f"codes{codes}_levels{levels}"] = build_ms(torch, ops, corpus, codes)
        torch.cuda.empty_cache()
    out["index_build_corpus_12101"] = builds
    corpus = torch.from_numpy(corpus_of(np, 1 << 20, 1 << 20)).cuda()
    out["index_build_corpus_1M"] = {f"codes{K}_levels{H}": build_ms(torch, ops, corpus, K)}
    del corpus
    torch.cuda.empty_cache()
    deep = {}
    for codes, levels in ((K, 5), (K, 8), (1024, 4), (2048, 4)):
        corpus = torch.from_numpy(corpus_of(np, 12101, 12101, codes, levels)).cuda()
        trie = ops.SidPrefixIndex(corpus, codes)
        res = {}
        for h, (probas, logits, generated, log_probas) in enumerate(level_inputs(torch, F, trie, 9, codes, levels)):
            res[f"level{h}"] = {
                "fused_ms": timed_ms(torch, lambda: trie.sample_select(probas, M.draw_exponential(probas), generated, log_probas,
                                                                       TOP_K, NC), w),
                "beam_ms": timed_ms(torch, lambda: trie.beam_topk(logits, generated, log_probas, TOP_K), w)}
        if codes == 2048:
            for h, (logits, generated, log_probas) in enumerate(beam_level_inputs(torch, trie, big_k, codes, 10, levels)):
                res[f"level{h}"]["beam_top_k32_ms"] = timed_ms(torch, lambda: trie.beam_topk(logits, generated, log_probas, big_k), w)
        deep[f"codes{codes}_levels{levels}"] = res
        del trie, corpus
        torch.cuda.empty_cache()
    out["trie_corpus_12101"] = deep

    class Composed(M.EncoderDecoderRetrievalModel):
        def _sample_and_select(self, index, probas, generated, log_probas, k, n_cands, reject):
            return composed_level(torch, index, probas, generated, log_probas, k, n_cands)

    corpus = torch.from_numpy(corpus_of(np, 12101, 12101))
    shape = dict(num_hierarchies=H, num_embeddings_per_hierarchy=K, t5_d_model=384, t5_num_heads=6, t5_d_ff=1024,
                 t5_num_layers=4, top_k_for_generation=TOP_K, should_add_sep_token=True)
    torch.manual_seed(0)
    fused = M.EncoderDecoderRetrievalModel(codebooks=corpus.clone(), **shape).cuda().eval()
    composed = Composed(codebooks=corpus.clone(), **shape).cuda().eval()
    composed.load_state_dict(fused.state_dict())
    rs = np.random.RandomState(1)
    ids = torch.from_numpy(rs.randint(0, K, size=(B, ITEMS * H))).cuda()
    mask = torch.ones_like(ids)
    torch.manual_seed(3)
    g_f, p_f = fused.generate(mask, ids)
    torch.manual_seed(3)
    g_c, p_c = composed.generate(mask, ids)
    g_b, p_b = fused.generate(mask, ids, search="beam")
    fused_ms, composed_ms, beam_ms = [], [], []
    for _ in range(3):                                        # alternate the models: clock drift hits all alike
        fused_ms.append(timed_ms(torch, lambda: fused.generate(mask, ids), w))
        composed_ms.append(timed_ms(torch, lambda: composed.generate(mask, ids), w))
        beam_ms.append(timed_ms(torch, lambda: fused.generate(mask, ids, search="beam"), w))
    out["generate"] = {
        "fused_ms": fused_ms, "composed_ms": composed_ms, "beam_ms": beam_ms,
        "beams_equal": bool(torch.equal(g_f, g_c)), "log_probas_equal": bool(torch.equal(p_f, p_c)),
        "finite_beam_fraction_random_init_model": {"sample": float(torch.isfinite(p_f).float().mean()),
                                                   "beam": float(torch.isfinite(p_b).float().mean())},
        "history_items": ITEMS, "t5": "d_model 384, 6 heads, d_ff 1024, 4 layers, random init, TF32 matmuls"}
    del fused, composed
    deep_h = 5
    corpus5 = torch.from_numpy(corpus_of(np, 12101, 12101, K, deep_h))
    torch.manual_seed(0)
    model5 = M.EncoderDecoderRetrievalModel(codebooks=corpus5, **dict(shape, num_hierarchies=deep_h)).cuda().eval()
    ids5 = torch.from_numpy(rs.randint(0, K, size=(B, ITEMS * deep_h))).cuda()
    mask5 = torch.ones_like(ids5)
    g_s5, p_s5 = model5.generate(mask5, ids5)
    g_b5, p_b5 = model5.generate(mask5, ids5, search="beam")
    sample5, beam5 = [], []
    for _ in range(3):
        sample5.append(timed_ms(torch, lambda: model5.generate(mask5, ids5), w))
        beam5.append(timed_ms(torch, lambda: model5.generate(mask5, ids5, search="beam"), w))
    out["generate_levels5"] = {
        "sample_ms": sample5, "beam_ms": beam5,
        "finite_beam_fraction_random_init_model": {"sample": float(torch.isfinite(p_s5).float().mean()),
                                                   "beam": float(torch.isfinite(p_b5).float().mean())}}
    out["timed"] = ("CUDA events, windows >= %.1f s after warm-up; per-level arms start from the level's probabilities (beam arms: "
                    "its logits)" % w)
    print(out["card"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
