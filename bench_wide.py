#!/usr/bin/env python
"""bench_wide.py -- the wide beam searches of the generative-retrieval model (generate(num_beams=w), w up to 1024).

    python bench_wide.py [--min-window-s 1.0]

On a 12 101-row corpus (Amazon Beauty's size), 3 hierarchy levels, per-level ms of one level h = 1 (w beams in, w out):
  * narrow: SidPrefixIndex.beam_topk (one CTA per history) against beam_topk_wide (one thread-block cluster per history) at
    the shapes both take: B = 640, k = 10 and 32, K = 256 and 2048.  The model runs the narrow kernel at these widths; the
    pair shows what that choice is worth;
  * wide: beam_topk_wide and sample_select_wide at w = 64, 128, 256, 1024 (w <= K), K = 256 and 2048, B = 1, 8, 64, 640,
    beside torch compositions: log_softmax, SidPrefixIndex.check of every extension, masked_fill, a stable descending sort
    and gathers (exhaustive); torch.multinomial, log/gather, check, masked_fill, a stable sort and gathers (sampled).  A
    torch arm whose temporaries would exceed 2^28 candidates is not run (null);
  * whole generate_items(num_beams=w, decoder="fused", encoder="fused") of the drop-in model at the decoder_amazon.gin T5 shape
    (d_model 384, 6 heads, d_ff 1024, 4 layers, random init) on 640 20-item histories, w in 10, 32, 64, 128, 256, both
    searches: ms and torch.cuda.max_memory_allocated; and decoder="hf" at w = 64 on 64 histories beside the fused decoder on
    the same 64.
Every shape is warmed up, every timed window lasts at least --min-window-s seconds (CUDA events), arms alternate.  Prints the
card's name, power limit and max SM clock, and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_generate import _card, beam_composed_level, corpus_of, timed_ms  # noqa: E402

N_CORPUS, NC, H, ITEMS = 12101, 64, 3, 20
MAX_TORCH_CANDIDATES = 1 << 28


def sample_composed_level(torch, index, probas, generated, log_probas, k, nc):
    """One sampled level in torch: multinomial, log/gather, the prefix check, masked_fill, a stable sort and gathers."""
    Bn, kp, h = generated.shape
    samples = torch.multinomial(probas, nc)
    scores = torch.log(torch.gather(probas, 1, samples)).view(Bn, kp * nc) + log_probas.repeat_interleave(nc, 1)
    prefix = torch.cat([generated.reshape(-1, h).repeat_interleave(nc, 0), samples.reshape(-1, 1)], 1)
    scores = scores.masked_fill(~index.check(prefix).view(Bn, -1), float("-inf"))
    s, order = scores.sort(dim=-1, descending=True, stable=True)
    top = order[:, :k]
    parent = top // nc
    tok = torch.gather(samples.view(Bn, -1), 1, top).unsqueeze(-1)
    return torch.cat([torch.gather(generated, 1, parent.unsqueeze(-1).expand(-1, -1, h)), tok], -1), s[:, :k], parent


def level1_inputs(torch, F, corpus, Bn, w, Kc, seed):
    """Level h = 1 of w beams per history: beams on corpus first codes, random logits, their softmax."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rows = torch.randint(0, corpus.shape[0], (Bn * w,), device="cuda", generator=g)
    generated = corpus[rows, :1].reshape(Bn, w, 1).contiguous()
    log_probas = -torch.rand((Bn, w), device="cuda", generator=g)
    logits = torch.randn((Bn * w, Kc), device="cuda", generator=g) * 3
    return logits, F.softmax(logits, dim=-1), generated, log_probas


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-window-s", type=float, default=1.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import torch.nn.functional as F
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    assert torch.cuda.is_available(), "bench_wide.py measures on a CUDA device"
    win = args.min_window_s
    out = {"card": _card(), "corpus_rows": N_CORPUS, "levels": H, "candidates_per_beam": NC}
    narrow, wide = {}, {}
    for Kc in (256, 2048):
        corpus = torch.from_numpy(corpus_of(np, N_CORPUS, N_CORPUS, Kc)).cuda()
        index = ops.SidPrefixIndex(corpus, Kc)
        for k in (10, 32):
            logits, _, generated, log_probas = level1_inputs(torch, F, corpus, 640, k, Kc, k)
            a = index.beam_topk(logits, generated, log_probas, k)
            b = index.beam_topk_wide(logits, generated, log_probas, k)
            arms = {"beam_topk_ms": lambda: index.beam_topk(logits, generated, log_probas, k),
                    "beam_topk_wide_ms": lambda: index.beam_topk_wide(logits, generated, log_probas, k)}
            res = {name: [] for name in arms}
            for _ in range(2):
                for name, fn in arms.items():
                    res[name].append(timed_ms(torch, fn, win))
            res["bit_identical"] = all(torch.equal(x, y) for x, y in zip(a, b))
            narrow[f"B640_k{k}_K{Kc}"] = res
        for w in (64, 128, 256, 1024):
            if w > Kc:
                continue
            for Bn in (1, 8, 64, 640):
                logits, probas, generated, log_probas = level1_inputs(torch, F, corpus, Bn, w, Kc, w + Bn)
                noise = M.draw_exponential(probas)
                arms = {"beam_topk_wide_ms": lambda: index.beam_topk_wide(logits, generated, log_probas, w),
                        "sample_select_wide_ms": lambda: index.sample_select_wide(probas, noise, generated, log_probas, w, NC)}
                if Bn * w * Kc <= MAX_TORCH_CANDIDATES:
                    arms["beam_torch_ms"] = lambda: beam_composed_level(torch, F, index, logits, generated, log_probas, w)
                    arms["sample_torch_ms"] = lambda: sample_composed_level(torch, index, probas, generated, log_probas, w, NC)
                res = {name: timed_ms(torch, fn, win) for name, fn in arms.items()}
                res.setdefault("beam_torch_ms", None)
                res.setdefault("sample_torch_ms", None)
                wide[f"w{w}_K{Kc}_B{Bn}"] = res
                print(f"w{w}_K{Kc}_B{Bn}", json.dumps(res), file=sys.stderr, flush=True)
                del logits, probas, generated, log_probas, noise
                torch.cuda.empty_cache()
        del index, corpus
        torch.cuda.empty_cache()
    out["level1_narrow_shapes"] = narrow
    out["level1_wide"] = wide

    Kc = 256
    corpus = torch.from_numpy(corpus_of(np, N_CORPUS, N_CORPUS, Kc))
    shape = dict(num_hierarchies=H, num_embeddings_per_hierarchy=Kc, t5_d_model=384, t5_num_heads=6, t5_d_ff=1024,
                 t5_num_layers=4, top_k_for_generation=10, should_add_sep_token=True)
    torch.manual_seed(0)
    model = M.EncoderDecoderRetrievalModel(codebooks=corpus, **shape).cuda().eval()
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch

    def batch_of(Bn, seed):
        rs = np.random.RandomState(seed)
        full = np.concatenate([corpus.numpy(), np.zeros((N_CORPUS, 1), dtype=np.int64)], 1)       # dedup rank 0
        hist = rs.randint(0, N_CORPUS, size=(Bn, ITEMS))
        cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        return TokenizedSeqBatch(user_ids=cuda(rs.randint(0, 100, size=(Bn, 1))), sem_ids=cuda(full[hist].reshape(Bn, -1)),
                                 sem_ids_fut=cuda(full[rs.randint(0, N_CORPUS, size=Bn)]),
                                 seq_mask=cuda(np.ones((Bn, ITEMS * (H + 1)), dtype=bool)),
                                 token_type_ids=cuda(np.tile(np.arange(H + 1), (Bn, ITEMS))),
                                 token_type_ids_fut=cuda(np.tile(np.arange(H + 1), (Bn, 1))))

    def items_call(batch, w, search, decoder="fused"):
        return lambda: model.generate_items(batch, num_beams=w, search=search, decoder=decoder, encoder="fused")

    def measured(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated()
        return {"ms": timed_ms(torch, fn, win), "max_memory_allocated_bytes": int(peak)}

    batch = batch_of(640, 1)
    gen = {}
    with torch.no_grad():
        for w in (10, 32, 64, 128, 256):
            for search in ("sample", "beam"):
                torch.manual_seed(3)
                gen[f"w{w}_{search}"] = measured(items_call(batch, w, search))
                print(f"generate_items w{w}_{search}", json.dumps(gen[f"w{w}_{search}"]), file=sys.stderr, flush=True)
        small = batch_of(64, 2)
        hf = {"hf": measured(items_call(small, 64, "beam", "hf")), "fused": measured(items_call(small, 64, "beam"))}
    out["generate_items_B640"] = gen
    out["generate_items_B64_w64_beam_decoders"] = hf
    out["t5"] = "d_model 384, 6 heads, d_ff 1024, 4 layers, random init, TF32 matmuls, 20-item histories"
    out["timed"] = "CUDA events, windows >= %.1f s after warm-up" % win
    print(out["card"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
