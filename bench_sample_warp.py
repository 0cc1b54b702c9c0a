#!/usr/bin/env python
"""bench_sample_warp.py -- the sampled search at a temperature and within a top-p nucleus (the warped draw).

    python bench_sample_warp.py [--min-window-s 0.5]

  * One level at B = 640 histories (level h = 1 of w beams, random logits times 3, a 12 101-row corpus): the warped kernel
    (SidPrefixIndex.sample_select_warped[_wide], T = 0.7, top_p = 0.9) against the untempered kernel of the same width
    (sample_select[_wide] from a softmax, the softmax included) and against a torch composition of the warped level (division,
    softmax, sort, cumsum, nucleus mask, the Exp(1) top-n, log_softmax gather, prefix check, stable sort), at w = 10 with
    K = 256 and 2048 (one-CTA kernels) and w = 64, 256, 1024 with K = 256 and 2048 (cluster kernels; the torch arm only where
    its [B w, K] tensors stay under 2^28 elements).
  * Whole generate_items(encoder="fused", decoder="fused", w = 10) at the configs/decoder_amazon.gin shape (K = 256, 3 levels,
    d_model 384, 6 heads, d_ff 1024, 4 layers, 20-item histories), eager and as a CUDA-graph replay, untempered and warped
    (T = 0.7, top_p = 0.9), at B = 1, 64 and 640.
  * Diversity at B = 640, w = 10, with the heads scaled by 8 as a stand-in for a trained, more confident model (a RANDOM model:
    what a trained model gains is not measured): distinct level-0 codes among each history's w beams, distinct items per
    history, and the mean finite returned log-probability, at T in {0.5, 1, 2} and top_p in {0.9, 1}.
Every arm is warmed up; arms alternate over two rounds, timed with CUDA events over windows of at least --min-window-s.
Prints the card's name, power limit and max SM clock, read in the same run, and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_generate import _card, corpus_of, timed_ms  # noqa: E402
from bench_wide import level1_inputs  # noqa: E402

N_CORPUS, NC, H, ITEMS, B = 12101, 64, 3, 20, 640
T, TOP_P = 0.7, 0.9
MAX_TORCH_ELEMENTS = 1 << 28


def warped_composed_level(torch, F, index, logits, generated, log_probas, k, nc, temp, top_p):
    """One warped level in torch, with torch.multinomial's Exp(1) race written out."""
    Bn, kp, h = generated.shape
    p = F.softmax(logits / temp, dim=-1)
    ps, order = p.sort(dim=-1, descending=True)
    keep_sorted = (ps.cumsum(-1) - ps) < top_p * ps.sum(-1, keepdim=True)
    keep = torch.zeros_like(keep_sorted).scatter_(1, order, keep_sorted) & (p > 0)
    ratio = torch.where(keep, p / torch.empty_like(p).exponential_(1), -1.0)
    samples = ratio.topk(nc, dim=-1).indices
    lp = torch.gather(F.log_softmax(logits, dim=-1), 1, samples)
    lp = torch.where(torch.gather(keep, 1, samples), lp, float("-inf"))
    scores = lp.view(Bn, kp * nc) + log_probas.repeat_interleave(nc, 1)
    prefix = torch.cat([generated.reshape(-1, h).repeat_interleave(nc, 0), samples.reshape(-1, 1)], 1)
    scores = scores.masked_fill(~index.check(prefix).view(Bn, -1), float("-inf"))
    s, top = scores.sort(dim=-1, descending=True, stable=True)
    top = top[:, :k]
    parent = top // nc
    tok = torch.gather(samples.view(Bn, -1), 1, top).unsqueeze(-1)
    return torch.cat([torch.gather(generated, 1, parent.unsqueeze(-1).expand(-1, -1, h)), tok], -1), s[:, :k], parent


def alternated(torch, arms, win):
    res = {name: [] for name in arms}
    for _ in range(2):
        for name, fn in arms.items():
            res[name].append(round(timed_ms(torch, fn, win), 4))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-window-s", type=float, default=0.5)
    args = ap.parse_args()
    import numpy as np
    import torch
    import torch.nn.functional as F
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    assert torch.cuda.is_available(), "bench_sample_warp.py measures on a CUDA device"
    win = args.min_window_s
    out = {"card": _card(), "corpus_rows": N_CORPUS, "candidates_per_beam": NC, "temperature": T, "top_p": TOP_P}

    levels = {}
    with torch.no_grad():
        for Kc in (256, 2048):
            corpus = torch.from_numpy(corpus_of(np, N_CORPUS, N_CORPUS, Kc)).cuda()
            index = ops.SidPrefixIndex(corpus, Kc)
            for w in (10, 64, 256, 1024):
                logits, _, generated, log_probas = level1_inputs(torch, F, corpus, B, w, Kc, w + Kc)
                noise = M.draw_exponential(logits)
                narrow = w * NC <= 1024 and w <= 32
                warped = index.sample_select_warped if narrow else index.sample_select_warped_wide
                plain = index.sample_select if narrow else index.sample_select_wide
                arms = {"warped_ms": lambda: warped(logits, noise, generated, log_probas, w, NC, T, TOP_P),
                        "untempered_ms": lambda: plain(F.softmax(logits, dim=-1), noise, generated, log_probas, w, NC)}
                if B * w * Kc <= MAX_TORCH_ELEMENTS:
                    arms["torch_ms"] = lambda: warped_composed_level(torch, F, index, logits, generated, log_probas, w, NC, T,
                                                                     TOP_P)
                res = alternated(torch, arms, win)
                res["kernel"] = "one-CTA" if narrow else "cluster"
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
        for name, kw in (("untempered", {}), ("warped", dict(temperature=T, top_p=TOP_P))):
            graph = model.capture_generate_items(batch, **kw)
            arms[f"{name}_eager_ms"] = (lambda kw=kw: model.generate_items(batch, encoder="fused", decoder="fused", **kw))
            arms[f"{name}_replay_ms"] = (lambda g=graph: g(batch))
        calls[f"B{Bn}"] = alternated(torch, arms, win)
        print(f"generate_items B{Bn}", json.dumps(calls[f"B{Bn}"]), file=sys.stderr, flush=True)
        del arms
        torch.cuda.empty_cache()
    out["generate_items_w10"] = calls

    with torch.no_grad():
        for head in model.decoder_mlp:
            head.weight.mul_(8)
    batch = batch_of(B, 7)
    diversity = {}
    for temp in (0.5, 1.0, 2.0):
        for top_p in (0.9, 1.0):
            torch.manual_seed(1)
            r = model.generate_items(batch, encoder="fused", decoder="fused", temperature=temp, top_p=top_p)
            first = r.sem_ids[:, :, 0]
            distinct0 = torch.tensor([len(set(row)) for row in first.tolist()], dtype=torch.float64)
            items = [len({i for i in row if i >= 0}) for row in r.item_ids.tolist()]
            lp = r.log_probas[torch.isfinite(r.log_probas)]
            diversity[f"T{temp}_p{top_p}"] = {"distinct_level0_codes": round(distinct0.mean().item(), 3),
                                              "distinct_items": round(float(np.mean(items)), 3),
                                              "mean_log_proba": round(lp.mean().item(), 4)}
    out["diversity_B640_w10_heads_x8"] = diversity
    out["t5"] = "d_model 384, 6 heads, d_ff 1024, 4 layers, random init, TF32 matmuls, 20-item histories"
    out["timed"] = "CUDA events, two alternated rounds, windows >= %.1f s after warm-up" % win
    print(out["card"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
