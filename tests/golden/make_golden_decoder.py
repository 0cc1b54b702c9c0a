"""Generate tests/golden/decoder.npz by running the UNMODIFIED reference EncoderDecoderRetrievalModel (modules/model.py).

Run where the reference tree is available (RQ_REFERENCE_PATH, see ref_harness.py):   python tests/golden/make_golden_decoder.py
The GPU box never runs this; it consumes the committed .npz file.

A tiny T5 on the CPU, in eval mode (no dropout): the model's state_dict, one TokenizedSeqBatch (padding, the dedup column, user
ids), forward's loss and loss_d, and the beams and log-probabilities of generate_next_sem_id under torch.manual_seed(1002).
"""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_harness          # noqa: E402


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def main():
    torch.set_num_threads(8)
    ref = ref_harness.load()
    stub = sys.modules.pop("accelerate", None)              # transformers probes the real package: the harness stub has no spec
    try:
        M = importlib.import_module("modules.model")
    finally:
        if stub is not None:
            sys.modules["accelerate"] = stub
    B, items, H, K, N, users = 8, 5, 3, 16, 200, 7
    rs = np.random.RandomState(1000)
    corpus = rs.randint(0, K, size=(N, H)).astype(np.int64)
    torch.manual_seed(1001)
    m = M.EncoderDecoderRetrievalModel(codebooks=t(corpus), num_hierarchies=H, num_embeddings_per_hierarchy=K, t5_d_model=32,
                                       t5_num_heads=2, t5_d_ff=64, t5_num_layers=2, top_k_for_generation=4,
                                       should_add_sep_token=True, num_user_bins=users).eval()
    lengths = rs.randint(1, items + 1, size=B)
    mask = np.arange(items)[None, :] < lengths[:, None]                  # [B, items], padding at the end
    sem = np.concatenate([rs.randint(0, K, size=(B, items, H)), rs.randint(0, 3, size=(B, items, 1))], axis=2)
    sem = np.where(mask[:, :, None], sem, -1).reshape(B, items * (H + 1)).astype(np.int64)
    seq_mask = np.repeat(mask, H + 1, axis=1)
    fut = np.concatenate([corpus[rs.randint(0, N, size=B)], rs.randint(0, 3, size=(B, 1))], axis=1).astype(np.int64)
    user_ids = rs.randint(0, 1000, size=(B, 1)).astype(np.int64)
    tt = np.tile(np.arange(H + 1), (B, items)).astype(np.int64)
    batch = ref.schemas.TokenizedSeqBatch(user_ids=t(user_ids), sem_ids=t(sem), sem_ids_fut=t(fut), seq_mask=t(seq_mask),
                                          token_type_ids=t(tt), token_type_ids_fut=t(np.arange(H + 1)[None].repeat(B, 0)))
    with torch.no_grad():
        o = m(batch)
    torch.manual_seed(1002)                                   # torch.multinomial inside generate
    gen = m.generate_next_sem_id(batch)
    out = {"sd/" + name: v.numpy() for name, v in m.state_dict().items()}
    out.update(shape=np.array([B, items, H, K, N, users]), user_ids=user_ids, sem_ids=sem, sem_ids_fut=fut, seq_mask=seq_mask,
               token_type_ids=tt, loss=o.loss.numpy(), loss_d=o.loss_d.numpy(), gen_sem_ids=gen.sem_ids.numpy(),
               gen_log_probas=gen.log_probas.numpy())
    path = os.path.join(HERE, "decoder.npz")
    np.savez_compressed(path, **out)
    print(f"decoder: {os.path.getsize(path) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
