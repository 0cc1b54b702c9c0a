#!/usr/bin/env python
"""bench_diverse.py -- the per-prefix cap on the generative-retrieval search (max_per_prefix beams per prefix_len-prefix).

    python bench_diverse.py [--min-window-s 0.5]

  * One level at B = 640 histories (level h = 1 of w beams whose first codes come from three per history, random logits times
    3, a 12 101-row corpus): capped (prefix_len = 1, max_per_prefix in {1, 2, 5}) against uncapped, for "beam"
    (SidPrefixIndex.beam_topk) and "sample" (sample_select, the softmax included), at w in {10, 32} and K in {256, 2048}.
    "sample" at w = 32 takes the cluster kernel (32 x 64 candidates > 1024), which has no capped mode: it is not timed.
  * Whole generate_items(encoder="fused", decoder="fused", w = 10) at the configs/decoder_amazon.gin shape (K = 256, 3 levels,
    d_model 384, 6 heads, d_ff 1024, 4 layers, 20-item histories), eager and as a CUDA-graph replay, uncapped and capped
    (max_per_prefix = 2, prefix_len = 1), at B = 1, 64 and 640.
  * Diversity at B = 640, w = 10, with the heads scaled by 8 as a stand-in for a trained, more confident model (a RANDOM model:
    what the cap does to a trained model's recall is not measured): distinct level-0 codes among each history's w beams,
    distinct items per history, and the mean finite returned log-probability, uncapped and at max_per_prefix in {1, 2, 3}.
Every arm is warmed up; arms alternate over two rounds, timed with CUDA events over windows of at least --min-window-s.
Prints the card's name, power limit and max SM clock, read in the same run, and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_generate import _card, corpus_of  # noqa: E402
from bench_sample_warp import alternated  # noqa: E402

N_CORPUS, NC, H, ITEMS, B = 12101, 64, 3, 20, 640


def level_inputs(torch, corpus, Bn, w, Kc, seed):
    """Level h = 1 of w beams per history, their first codes drawn from three of the corpus per history."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    heads = corpus[torch.randint(0, corpus.shape[0], (Bn, 3), device="cuda", generator=g), 0]
    generated = torch.gather(heads, 1, torch.randint(0, 3, (Bn, w), device="cuda", generator=g)).unsqueeze(-1).contiguous()
    log_probas = -torch.rand((Bn, w), device="cuda", generator=g)
    logits = torch.randn((Bn * w, Kc), device="cuda", generator=g) * 3
    return logits, generated, log_probas


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-window-s", type=float, default=0.5)
    args = ap.parse_args()
    import numpy as np
    import torch
    import torch.nn.functional as F
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    assert torch.cuda.is_available(), "bench_diverse.py measures on a CUDA device"
    win = args.min_window_s
    out = {"card": _card(), "corpus_rows": N_CORPUS, "candidates_per_beam": NC, "prefix_len": 1}

    levels = {}
    with torch.no_grad():
        for Kc in (256, 2048):
            corpus = torch.from_numpy(corpus_of(np, N_CORPUS, N_CORPUS, Kc)).cuda()
            index = ops.SidPrefixIndex(corpus, Kc)
            for w in (10, 32):
                logits, generated, log_probas = level_inputs(torch, corpus, B, w, Kc, w + Kc)
                noise = M.draw_exponential(logits)
                arms = {"beam_ms": lambda: index.beam_topk(logits, generated, log_probas, w)}
                for m in (1, 2, 5):
                    arms[f"beam_cap{m}_ms"] = lambda m=m: index.beam_topk(logits, generated, log_probas, w, cap=(1, m))
                if w * NC <= 1024:
                    arms["sample_ms"] = lambda: index.sample_select(F.softmax(logits, dim=-1), noise, generated, log_probas, w, NC)
                    for m in (1, 2, 5):
                        arms[f"sample_cap{m}_ms"] = lambda m=m: index.sample_select(F.softmax(logits, dim=-1), noise, generated,
                                                                                    log_probas, w, NC, cap=(1, m))
                res = alternated(torch, arms, win)
                levels[f"w{w}_K{Kc}"] = res
                print(f"level w{w}_K{Kc}", json.dumps(res), file=sys.stderr, flush=True)
                del logits, generated, log_probas, noise
                torch.cuda.empty_cache()
            del index, corpus
            torch.cuda.empty_cache()
    out["level_B640"] = levels

    Kc = 256
    corpus = torch.from_numpy(corpus_of(np, N_CORPUS, N_CORPUS, Kc))
    shape = dict(num_hierarchies=H, num_embeddings_per_hierarchy=Kc, t5_d_model=384, t5_num_heads=6, t5_d_ff=1024,
                 t5_num_layers=4, top_k_for_generation=10, should_add_sep_token=True)
    torch.manual_seed(0)
    model = M.EncoderDecoderRetrievalModel(codebooks=corpus, **shape).cuda().eval()
    from rq_vae_recommender_b200.data.schemas import TokenizedSeqBatch

    def batch_of(Bn, seed):
        rs = np.random.RandomState(seed)
        full = np.concatenate([corpus.numpy(), np.zeros((N_CORPUS, 1), dtype=np.int64)], 1)
        hist = rs.randint(0, N_CORPUS, size=(Bn, ITEMS))
        cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        return TokenizedSeqBatch(user_ids=cuda(rs.randint(0, 100, size=(Bn, 1))), sem_ids=cuda(full[hist].reshape(Bn, -1)),
                                 sem_ids_fut=cuda(full[rs.randint(0, N_CORPUS, size=Bn)]),
                                 seq_mask=cuda(np.ones((Bn, ITEMS * (H + 1)), dtype=bool)),
                                 token_type_ids=cuda(np.tile(np.arange(H + 1), (Bn, ITEMS))),
                                 token_type_ids_fut=cuda(np.tile(np.arange(H + 1), (Bn, 1))))

    calls = {}
    for Bn in (1, 64, 640):
        batch = batch_of(Bn, Bn)
        arms = {}
        for name, kw in (("uncapped", {}), ("cap2", dict(max_per_prefix=2, prefix_len=1))):
            graph = model.capture_generate_items(batch, search="beam", **kw)
            arms[f"{name}_eager_ms"] = (lambda kw=kw: model.generate_items(batch, search="beam", encoder="fused", decoder="fused",
                                                                           **kw))
            arms[f"{name}_replay_ms"] = (lambda g=graph: g(batch))
        calls[f"B{Bn}"] = alternated(torch, arms, win)
        print(f"generate_items B{Bn}", json.dumps(calls[f"B{Bn}"]), file=sys.stderr, flush=True)
        del arms
        torch.cuda.empty_cache()
    out["generate_items_beam_w10"] = calls

    with torch.no_grad():
        for head in model.decoder_mlp:
            head.weight.mul_(8)
    batch = batch_of(B, 7)
    diversity = {}
    for search in ("beam", "sample"):
        for m in (None, 1, 2, 3):
            torch.manual_seed(1)
            r = model.generate_items(batch, search=search, encoder="fused", decoder="fused", max_per_prefix=m)
            first = r.sem_ids[:, :, 0]
            distinct0 = torch.tensor([len(set(row)) for row in first.tolist()], dtype=torch.float64)
            items = [len({i for i in row if i >= 0}) for row in r.item_ids.tolist()]
            lp = r.log_probas[torch.isfinite(r.log_probas)]
            diversity[f"{search}_cap{m}"] = {"distinct_level0_codes": round(distinct0.mean().item(), 3),
                                             "distinct_items": round(float(np.mean(items)), 3),
                                             "mean_log_proba": round(lp.mean().item(), 4)}
    out["diversity_B640_w10_heads_x8"] = diversity
    out["t5"] = "d_model 384, 6 heads, d_ff 1024, 4 layers, random init, TF32 matmuls, 20-item histories"
    out["timed"] = "CUDA events, two alternated rounds, windows >= %.1f s after warm-up" % win
    print(out["card"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
