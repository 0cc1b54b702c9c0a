"""GPU tests of the module-level mirrors (Quantize / RqVae / MLP / Kmeans / SemanticIdTokenizer) against outputs of
the unmodified reference modules (tests/golden/rqvae_c1.npz, tokenizer.npz) and the oracle.  `pytest -m gpu`."""
import numpy as np
import pytest
import torch

import inputs as I
from oracle import rq_oracle as O
from parity import assert_ids_match, load_golden, rel_err

pytestmark = pytest.mark.gpu
T, BETA = 0.2, 0.25


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.detach().cpu().numpy()


def build(mode_name, n_cat, Din=64, D=16, hidden=(32,), K=32, L=2, seed=320):
    from rq_vae_recommender_b200.modules.rqvae import RqVae
    from rq_vae_recommender_b200.modules.quantize import QuantizeForwardMode as M
    mode = {"ste": M.STE, "rot": M.ROTATION_TRICK, "gumbel": M.GUMBEL_SOFTMAX}[mode_name]
    m = RqVae(input_dim=Din, embed_dim=D, hidden_dims=list(hidden), codebook_size=K, codebook_kmeans_init=False,
              codebook_mode=mode, n_layers=L, commitment_weight=BETA, n_cat_features=n_cat).cuda()
    enc = I.mlp_weights(seed, [Din] + list(hidden) + [D])
    dec = I.mlp_weights(seed + 1, [D] + list(hidden)[::-1] + [Din])
    cbs = [(I.rand(seed + 10 + l, K, D) * (0.6 ** l) - (0.25 if l else 0.0)).astype(np.float32) for l in range(L)]
    with torch.no_grad():
        for lin, w in zip([mm for mm in m.encoder.mlp if isinstance(mm, torch.nn.Linear)], enc):
            lin.weight.copy_(dev(w))
        for lin, w in zip([mm for mm in m.decoder.mlp if isinstance(mm, torch.nn.Linear)], dec):
            lin.weight.copy_(dev(w))
        for layer, c in zip(m.layers, cbs):
            layer.embedding.weight.copy_(dev(c))
    return m, enc, dec, cbs


def c1_inputs(n_cat):
    g = load_golden("rqvae_c1")
    B, Din, D, H, K, L = (int(v) for v in g["shape"])
    x = I.randn(300, B, Din)
    if n_cat:
        x[:, -n_cat:] = (I.rand(301, B, n_cat) > 0.5).astype(np.float32)
    us = [I.rand(310 + l, B, K) for l in range(L)]
    return g, x, us


def batch_of(x):
    from rq_vae_recommender_b200.data.schemas import SeqBatch
    return SeqBatch(user_ids=None, ids=None, ids_fut=None, x=x, x_fut=None, seq_mask=None)


@pytest.mark.parametrize("n_cat", [0, 4])
def test_rqvae_eval_outputs_vs_reference(n_cat):
    g, x, _ = c1_inputs(n_cat)
    m, enc, dec, cbs = build("ste", n_cat)
    m.eval()
    with torch.no_grad():
        so = m.get_semantic_ids(dev(x), T)
        fo = m(batch_of(dev(x)), T)
        tok = m.tokenize(dev(x))
    res = O.mlp_forward(x, enc)
    ids = host(so.sem_ids)
    assert so.embeddings.shape == (x.shape[0], 16, 2) and so.residuals.shape == (x.shape[0], 16, 2)
    assert so.sem_ids.dtype == torch.int64 and np.array_equal(ids, host(tok))
    assert_ids_match(ids, g[f"cat{n_cat}_eval_sem_ids"], res, cbs)
    same = (ids == g[f"cat{n_cat}_eval_sem_ids"]).all(1)
    assert same.mean() > 0.995
    assert rel_err(host(so.embeddings)[same], g[f"cat{n_cat}_eval_embeddings"][same]) < 1e-5
    assert np.abs(host(so.residuals)[same] - g[f"cat{n_cat}_eval_residuals"][same]).max() < 1e-5
    assert rel_err(host(so.quantize_loss)[same], g[f"cat{n_cat}_eval_qloss"][same]) < 1e-4
    if same.all():
        ref = g[f"cat{n_cat}_eval_losses"]
        got = np.array([fo.loss.item(), fo.reconstruction_loss.item(), fo.rqvae_loss.item(), fo.p_unique_ids.item()])
        assert np.allclose(got, ref, rtol=1e-5), (got, ref)
        assert rel_err(host(fo.embs_norm), g[f"cat{n_cat}_eval_embs_norm"]) < 1e-5


@pytest.mark.parametrize("n_cat", [0, 4])
@pytest.mark.parametrize("mname", ["ste", "rot", "gumbel"])
def test_rqvae_train_step_vs_reference(n_cat, mname, monkeypatch):
    """forward() losses and the gradient of EVERY parameter against the reference's autograd."""
    g, x, us = c1_inputs(n_cat)
    m, *_ = build(mname, n_cat)
    m.train()
    if mname == "gumbel":
        from rq_vae_recommender_b200.distributions import gumbel
        queue = [dev(u) for u in us]
        monkeypatch.setattr(gumbel, "draw_uniform", lambda shape, device: queue.pop(0))
    fo = m(batch_of(dev(x)), T)
    fo.loss.backward()
    tag = f"cat{n_cat}_{mname}"
    ref = g[f"{tag}_losses"]
    got = np.array([fo.loss.item(), fo.reconstruction_loss.item(), fo.rqvae_loss.item(), fo.p_unique_ids.item()])
    tol = 1e-4 if mname == "gumbel" else 2e-5
    assert np.allclose(got, ref, rtol=tol), (got, ref)
    assert rel_err(host(fo.embs_norm), g[f"{tag}_embs_norm"]) < (5e-4 if mname == "gumbel" else 1e-5)
    gtol = 2e-3 if mname == "gumbel" else 1e-4
    for name, p in m.named_parameters():
        assert p.grad is not None, name
        assert rel_err(host(p.grad), g[f"{tag}_grad_{name}"]) < gtol, name


def test_state_dict_keys_and_checkpoint_roundtrip(tmp_path):
    m, *_ = build("ste", 0, Din=768, D=32, hidden=(512, 256, 128), K=256, L=3)
    keys = sorted(m.state_dict().keys())
    assert keys == sorted([f"layers.{i}.embedding.weight" for i in range(3)] +
                          [f"encoder.mlp.{i}.weight" for i in (0, 2, 4, 6)] +
                          [f"decoder.mlp.{i}.weight" for i in (0, 2, 4, 6)])       # SURVEY 5.4 drop-in constraint
    path = str(tmp_path / "ckpt.pt")
    torch.save({"iter": 7, "model": m.state_dict(), "model_config": m.config}, path)
    m2, *_ = build("ste", 0, Din=768, D=32, hidden=(512, 256, 128), K=256, L=3, seed=999)
    m2.load_pretrained(path)
    x = dev(I.unit_rows(5, 300, 768))
    m.eval(); m2.eval()
    assert torch.equal(m.tokenize(x), m2.tokenize(x))


def test_quantize_module_api_and_kmeans_first_call():
    from rq_vae_recommender_b200.modules.quantize import Quantize, QuantizeForwardMode, QuantizeOutput
    from rq_vae_recommender_b200.init.kmeans import Kmeans
    x = dev(I.randn(600, 4096, 16))
    q = Quantize(embed_dim=16, n_embed=32, do_kmeans_init=True, forward_mode=QuantizeForwardMode.STE).cuda().train()
    np.random.seed(610); torch.manual_seed(611)
    out = q(x, temperature=T)
    assert isinstance(out, QuantizeOutput) and q.kmeans_initted
    np.random.seed(610); torch.manual_seed(611)
    ref = Kmeans(k=32).run(x)
    assert torch.allclose(q.embedding.weight, ref.centroids, atol=1e-6)
    g = load_golden("kmeans")
    assert np.abs(host(q.embedding.weight) - g["a_centroids"]).max() < 2e-5     # = the reference's k-means result
    o = O.quantize_forward(host(x), host(q.embedding.weight), O.STE, True, T, BETA)
    assert_ids_match(host(out.ids), o.ids, host(x), [host(q.embedding.weight)])
    assert rel_err(host(out.loss), o.loss) < 1e-5
    with pytest.raises(NotImplementedError):
        from rq_vae_recommender_b200.modules.quantize import QuantizeDistance
        Quantize(16, 32, do_kmeans_init=False, distance_mode=QuantizeDistance.COSINE).cuda()(x, T)


def test_sim_vq_and_codebook_normalize_paths():
    """out_proj = Linear (sim_vq) + L2 norm (codebook_normalize): gradients flow to embedding AND projection."""
    from rq_vae_recommender_b200.modules.rqvae import RqVae
    from rq_vae_recommender_b200.modules.quantize import QuantizeForwardMode
    torch.manual_seed(0)
    m = RqVae(input_dim=64, embed_dim=16, hidden_dims=[32], codebook_size=32, codebook_kmeans_init=False,
              codebook_normalize=True, codebook_sim_vq=True, codebook_mode=QuantizeForwardMode.ROTATION_TRICK,
              n_layers=2, n_cat_features=0).cuda().train()
    assert "layers.0.out_proj.0.weight" in m.state_dict()
    x = dev(I.randn(1, 256, 64))
    fo = m(batch_of(x), T)
    fo.loss.backward()
    for name, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
    # float64 torch re-statement of the same forward on the kernel's ids
    so = m.get_semantic_ids(x, T)
    # (float64: rqvae.py sets float32 matmul precision "high" like the reference, so a float32 `@` here would be TF32)
    w64 = m.layers[0].embedding.weight.double() @ m.layers[0].out_proj[0].weight.double().T
    cb0 = torch.nn.functional.normalize(w64, dim=-1)
    assert torch.allclose(m.layers[0].codebook().double(), cb0, atol=1e-6)
    assert so.sem_ids.shape == (256, 2)


def test_tokenizer_corpus_pass_vs_reference():
    from rq_vae_recommender_b200.modules.tokenizer.semids import SemanticIdTokenizer, dedup_rank
    from rq_vae_recommender_b200.data.schemas import SeqBatch
    g = load_golden("tokenizer")
    N, Din, D, H, K, L = (int(v) for v in g["shape"])
    x = I.randn(801, N, Din)
    m, enc, dec, cbs = build("gumbel", 0, Din=Din, D=D, hidden=(H,), K=K, L=L, seed=800)
    tok = SemanticIdTokenizer(input_dim=Din, output_dim=D, hidden_dims=[H], codebook_size=K, n_layers=L, n_cat_feats=0).cuda()
    tok.rq_vae = m
    tok.corpus_batch = 700          # ragged last batch

    class Items:
        def __len__(self):
            return N
        def __getitem__(self, idx):
            idx = torch.as_tensor(idx)
            return SeqBatch(user_ids=-torch.ones_like(idx), ids=idx.unsqueeze(0), ids_fut=-torch.ones_like(idx),
                            x=torch.from_numpy(x)[idx], x_fut=-torch.ones_like(idx), seq_mask=torch.ones_like(idx, dtype=bool))
    cached = host(tok.precompute_corpus_ids(Items()))
    ref = g["cached_ids"].astype(np.int64)
    assert cached.shape == ref.shape == (N, L + 1) and tok.sem_ids_dim == L + 1
    res = O.mlp_forward(x, enc)
    assert_ids_match(cached[:, :L], ref[:, :L], res, cbs)
    if np.array_equal(cached[:, :L], ref[:, :L]):
        assert np.array_equal(cached[:, L], ref[:, L])           # dedup column == the reference's O(N^2) result
    assert np.array_equal(host(dedup_rank(dev(ref[:, :L]), K)), ref[:, L])
    # sequence tokenisation from the cache (semids.py:112-146)
    ids = torch.tensor([[3, 5, 7], [9, 11, 2]]).cuda()
    b = SeqBatch(user_ids=torch.zeros(2).cuda(), ids=ids, ids_fut=torch.tensor([[1], [4]]).cuda(), x=None, x_fut=None,
                 seq_mask=torch.tensor([[True, True, False], [True, True, True]]).cuda())
    out = tok(b)
    assert out.sem_ids.shape == (2, 3 * (L + 1)) and (out.sem_ids[0, -(L + 1):] == -1).all()
    assert torch.equal(out.sem_ids[1, : L + 1], tok.cached_ids[9])
    assert out.sem_ids_fut.shape == (2, L + 1) and out.token_type_ids.shape == (2, 3 * (L + 1))


@pytest.mark.parametrize("D,hidden", [(768, ()), (64, (128,)), (32, (512, 256, 128))])
def test_module_api_routes_to_the_tensor_core_tokeniser(D, hidden):
    """VERDICT r1 item 3: SemanticIdTokenizer.precompute_corpus_ids -> RqVae.tokenize must run the wgmma tokeniser (prepared
    state cached across batches) for K = 256 models -- D = 768, D = 64 and the shipped D = 32 (zero-padded to 64) -- and return
    the exact kernel's ids (modules/tokenizer/semids.py:76-125)."""
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules.tokenizer.semids import SemanticIdTokenizer
    from rq_vae_recommender_b200.data.schemas import SeqBatch
    Din, K, L, N = 768, 256, 3, 5000
    m, enc, dec, _ = build("ste", 0, Din=Din, D=D, hidden=hidden, K=K, L=L, seed=4000 + D)
    x = I.unit_rows(4100 + D, N, Din)
    with torch.no_grad():          # live codebooks: residual rows of the encoder output, like a k-means-initialised model
        res = m.encode(dev(x))
        for l, layer in enumerate(m.layers):
            layer.embedding.weight.copy_(res[torch.randperm(N, generator=torch.Generator().manual_seed(l))[:K].cuda()])
            res = res - layer.embedding.weight[ops.rq_tokenize(res, [layer.embedding.weight])[:, 0]]
    tok = SemanticIdTokenizer(input_dim=Din, output_dim=D, hidden_dims=list(hidden), codebook_size=K, n_layers=L, n_cat_feats=0).cuda()
    tok.rq_vae = m.eval()
    tok.corpus_batch = 1700         # three batches (1700, 1700, 1600; all >= ops.TC_MIN_ROWS) -> one prepare, three tensor-core launches

    class Items:
        def __len__(self):
            return N
        def __getitem__(self, idx):
            idx = torch.as_tensor(idx)
            return SeqBatch(user_ids=-torch.ones_like(idx), ids=idx.unsqueeze(0), ids_fut=-torch.ones_like(idx),
                            x=torch.from_numpy(x)[idx], x_fut=-torch.ones_like(idx), seq_mask=torch.ones_like(idx, dtype=bool))
    calls, preps = ops.TC_CALLS, ops.TC_PREPARES
    cached = host(tok.precompute_corpus_ids(Items()))
    assert ops.TC_CALLS - calls == 3 and ops.TC_PREPARES - preps == 1, (ops.TC_CALLS - calls, ops.TC_PREPARES - preps)
    with torch.no_grad():
        z = m.encode(dev(x))
        cbs = [layer.codebook() for layer in m.layers]
        exact = host(ops.rq_tokenize(z, cbs))
    assert_ids_match(cached[:, :L], exact, host(z), [host(c) for c in cbs], f"module-api/tc D={D}")
    assert np.array_equal(cached[:, :L], host(m.tokenize(dev(x))))
    # an optimiser step (in-place update) must invalidate the cached state
    with torch.no_grad():
        m.layers[0].embedding.weight.mul_(1.01)
    m.tokenize(dev(x))
    assert ops.TC_PREPARES - preps == 2


def test_training_loop_like_train_rqvae():
    """The call sequence of train_rqvae.py:136-292 (k-means warm-up call, AdamW steps, eval, corpus ids + diversity
    stats) on synthetic item features: the loss must fall and the id statistics must be well formed."""
    from rq_vae_recommender_b200.modules.rqvae import RqVae
    from rq_vae_recommender_b200.modules.quantize import QuantizeForwardMode
    from rq_vae_recommender_b200.modules.tokenizer.semids import SemanticIdTokenizer
    from rq_vae_recommender_b200 import parallel
    np.random.seed(0); torch.manual_seed(0)
    N, Din = 6000, 768
    centers = I.unit_rows(40, 64, Din)
    items = centers[np.random.RandomState(1).randint(0, 64, N)] + 0.3 * I.unit_rows(41, N, Din)
    items = dev((items / np.linalg.norm(items, axis=1, keepdims=True)).astype(np.float32))
    model = RqVae(input_dim=Din, embed_dim=32, hidden_dims=[512, 256, 128], codebook_size=256,
                  codebook_kmeans_init=True, codebook_mode=QuantizeForwardMode.STE, n_layers=3, n_cat_features=0).cuda()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3, weight_decay=1e-4)
    model.train()
    model(batch_of(items[:4000]), 0.2)                      # train_rqvae.py:178-183: lazy k-means init of all levels
    assert all(l.kmeans_initted for l in model.layers)
    losses = []
    for it in range(40):
        idx = torch.randint(0, N, (640,), device="cuda")
        opt.zero_grad()
        out = model(batch_of(items[idx]), gumbel_t=0.2)
        out.loss.backward()
        opt.step()
        losses.append(out.loss.item())
    assert np.isfinite(losses).all() and np.mean(losses[-5:]) < np.mean(losses[:5])
    model.eval()
    with torch.no_grad():
        ev = model(batch_of(items[:640]), gumbel_t=0.2)
    assert 0 < ev.p_unique_ids.item() <= 1 and ev.embs_norm.shape == (640, 3)
    tok = SemanticIdTokenizer(input_dim=Din, output_dim=32, hidden_dims=[512, 256, 128], codebook_size=256, n_layers=3,
                              n_cat_feats=0).cuda()
    tok.rq_vae = model

    class Items:
        def __len__(self):
            return N
        def __getitem__(self, idx):
            return batch_of(items[torch.as_tensor(idx).cuda()])
    corpus = tok.precompute_corpus_ids(Items())
    assert corpus.shape == (N, 4)
    usage = parallel.codebook_usage(corpus[:, :3].contiguous(), 256)
    assert usage.shape == (3, 256) and usage.sum(1).tolist() == [N] * 3
    _, counts = torch.unique(corpus[:, :-1], dim=0, return_counts=True)        # train_rqvae.py:279-283
    assert counts.max().item() - 1 == corpus[:, -1].max().item()


def test_mlp_bf16_path_is_opt_in_and_forward_only():
    """precision="bf16" / bf16 autocast selects the wgmma GEMMs only when no gradient is needed; default stays exact."""
    from rq_vae_recommender_b200.modules.encoder import MLP
    torch.manual_seed(0)
    mlp = MLP(input_dim=768, hidden_dims=[512, 256, 128], out_dim=32).cuda()
    x = dev(I.unit_rows(3, 500, 768))
    ws = [host(m.weight) for m in mlp.mlp if isinstance(m, torch.nn.Linear)]
    exact = mlp(x)                                           # grad enabled, params require grad -> exact fp32 path
    assert exact.requires_grad and rel_err(host(exact), O.mlp_forward(host(x), ws)) < 1e-5
    with torch.no_grad():
        assert torch.equal(mlp(x), exact.detach())           # default precision: still exact
        mlp.precision = "bf16"
        y16 = mlp(x)
        ref16 = O.mlp_forward_bf16(host(x), ws)
        err = np.abs(host(y16).astype(np.float64) - ref16) / np.abs(ref16).max()
        assert np.median(err) < 1e-6 and err.max() < 1e-2
        assert not torch.equal(y16, exact.detach())
        y16b = mlp(x)
        assert torch.equal(y16, y16b)                        # weight-image cache reused, deterministic
        mlp.mlp[0].weight.mul_(1.5)                          # in-place update bumps _version -> cache rebuilt
        assert not torch.equal(mlp(x), y16)
    mlp.precision = "fp32"
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        ya = mlp(x)                                          # bf16 autocast region (the reference's AMP mode) -> bf16 GEMMs
    with torch.no_grad():
        mlp.precision = "bf16"
        assert torch.equal(ya, mlp(x))
    mlp.precision = "bf16"
    assert mlp(x).requires_grad                              # gradient needed -> falls to the exact, differentiable path


@pytest.mark.parametrize("N,L,K,dup", [(5000, 3, 256, 0.3), (1, 3, 256, 0.0), (777, 2, 32, 0.9), (3000, 4, 256, 0.5)])
def test_corpus_dedup_rank_and_id_statistics(N, L, K, dup):
    """(f)-1: the dedup column (semids.py:94-108: rows j < i with the same tuple) and the diversity statistics of
    train_rqvae.py:276-292 from the direct-table kernels, against the reference's own expressions (O(N^2) compare, torch.unique)."""
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules.tokenizer.semids import corpus_id_stats, dedup_rank
    rs = np.random.RandomState(N + L)
    ids = rs.randint(0, K, size=(N, L)).astype(np.int64)
    ndup = int(dup * N)
    if ndup:
        ids[rs.choice(N, ndup, replace=False)] = ids[rs.choice(max(N // 10, 1), ndup)]     # many copies of a few tuples
    ref_rank = (np.tril((ids[:, None, :] == ids[None, :, :]).all(-1), -1)).sum(1) if N <= 5000 else None
    rank = dedup_rank(dev(ids), K)
    assert np.array_equal(host(rank), ref_rank)
    cached = torch.cat([dev(ids), rank.unsqueeze(1)], 1)
    st = corpus_id_stats(cached, K)
    t = torch.from_numpy(ids)
    _, counts = torch.unique(t, dim=0, return_counts=True)                                # train_rqvae.py:279-283
    p = counts / N
    assert abs(float(st["rqvae_entropy"]) - float(-(p * torch.log(p)).sum())) < 1e-5
    assert float(st["max_id_duplicates"]) == pytest.approx(ref_rank.max() / N)
    for l in range(L):
        assert float(st[f"codebook_usage_{l}"]) == pytest.approx(len(torch.unique(t[:, l])) / K)
    if K ** L <= 2 ** 26:
        r2, s2 = ops.sid_dedup_rank(dev(ids), K)
        assert int(s2["n_unique"]) == len(counts) and int(s2["max_rank"]) == ref_rank.max()
    else:
        assert ops.sid_dedup_rank(dev(ids), K) is None           # 256^4 keys: the sort path answered above


def test_sequence_gather_kernel_vs_reference_indexing():
    """(f)-2: cached_ids[ids] with -1 under the padding mask and token_type_ids (semids.py:112-146) in one launch."""
    from rq_vae_recommender_b200 import ops
    rs = np.random.RandomState(3)
    ncorp, C, B, S = 999, 4, 37, 20
    cached = dev(rs.randint(0, 256, size=(ncorp, C)).astype(np.int64))
    item = rs.randint(0, ncorp, size=(B, S)).astype(np.int64)
    mask = rs.rand(B, S) > 0.3
    item[~mask] = -1                                             # padded positions carry -1 like the reference's batches
    out, tt = ops.sid_gather(cached, dev(item), dev(mask))
    ref = cached[dev(item).flatten(), :].reshape(B, S * C)        # reference: index (wraps -1), then mask
    m = dev(mask).repeat_interleave(C, dim=1)
    ref[~m] = -1
    assert torch.equal(out, ref)
    assert torch.equal(tt, torch.arange(C, device="cuda").repeat(B, S))
    fut, ttf = ops.sid_gather(cached, dev(item[:, :1].clip(0)), None)
    assert torch.equal(fut, cached[dev(item[:, 0].clip(0))]) and torch.equal(ttf, torch.arange(C, device="cuda").repeat(B, 1))


def _grads(m):
    return {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("mode_name", ["ste", "rot", "gumbel"])
def test_forward_compiles_to_one_graph_with_custom_operators(mode_name):
    """SURVEY 8(b): the reference decorates RqVae.forward with torch.compile (rqvae.py:141).  The kernels are registered with
    torch.library (rq_vae_recommender_b200/library.py): the whole training forward traces into ONE graph (fullgraph=True raises
    on any graph break) whose losses and parameter gradients equal the eager path's."""
    import rq_vae_recommender_b200.library  # noqa: F401  (registration)
    g, x, _ = c1_inputs(4)
    m, enc, dec, cbs = build(mode_name, 4)
    m.train()
    batch = batch_of(dev(x))
    torch.manual_seed(7)
    eager = m(batch, T)
    eager.loss.backward()
    g_eager = _grads(m)
    m.zero_grad(set_to_none=True)
    compiled = torch.compile(lambda b, t: m(b, t), backend="aot_eager", fullgraph=True)
    torch.manual_seed(7)                                      # the Gumbel level draws its uniforms with torch.rand inside forward
    out = compiled(batch, T)
    assert torch.allclose(out.loss, eager.loss, rtol=1e-6), (out.loss.item(), eager.loss.item())
    assert torch.allclose(out.rqvae_loss, eager.rqvae_loss, rtol=1e-6)
    assert torch.allclose(out.embs_norm, eager.embs_norm, rtol=1e-6) and torch.equal(out.p_unique_ids, eager.p_unique_ids)
    out.loss.backward()
    g_comp = _grads(m)
    assert g_comp.keys() == g_eager.keys() and len(g_comp) > 0
    for n in g_eager:
        assert torch.allclose(g_comp[n], g_eager[n], rtol=1e-5, atol=1e-7 * g_eager[n].abs().max().item() + 1e-12), n


@pytest.mark.parametrize("mode_name", ["STE", "GUMBEL_SOFTMAX"])
def test_compiled_forward_with_projected_normalised_codebooks(mode_name):
    """sim_vq projection + row-normalised first codebook + an L2-normalising decoder input path: compiled (one graph) == eager."""
    import rq_vae_recommender_b200.library  # noqa: F401
    from rq_vae_recommender_b200.modules.rqvae import RqVae
    from rq_vae_recommender_b200.modules.quantize import QuantizeForwardMode as M
    g, x, _ = c1_inputs(4)
    torch.manual_seed(11)
    m = RqVae(input_dim=x.shape[1], embed_dim=16, hidden_dims=[32], codebook_size=32, codebook_kmeans_init=False,
              codebook_mode=getattr(M, mode_name), n_layers=2, commitment_weight=BETA, n_cat_features=4,
              codebook_sim_vq=True, codebook_normalize=True).cuda()
    m.train()
    batch = batch_of(dev(x))
    torch.manual_seed(7)
    eager = m(batch, T)
    eager.loss.backward()
    g_eager = _grads(m)
    m.zero_grad(set_to_none=True)
    compiled = torch.compile(lambda b, t: m(b, t), backend="aot_eager", fullgraph=True)
    torch.manual_seed(7)
    out = compiled(batch, T)
    assert torch.allclose(out.loss, eager.loss, rtol=1e-6), (out.loss.item(), eager.loss.item())
    out.loss.backward()
    g_comp = _grads(m)
    assert g_comp.keys() == g_eager.keys() and len(g_comp) > 0
    for n in g_eager:
        # codebook gradients are fp32 atomics (order varies run to run) and pass through the projection / normalisation backward
        err = (g_comp[n] - g_eager[n]).abs().max().item() / (g_eager[n].abs().max().item() + 1e-30)
        assert err <= 2e-5, (n, err)


def test_reduce_overhead_graph_follows_weight_updates():
    """mode="reduce-overhead" (the reference's setting) replays a CUDA graph: nothing prepared on the host at capture time may go
    stale when the optimiser updates the weights in place between replays."""
    import rq_vae_recommender_b200.library  # noqa: F401
    g, x, _ = c1_inputs(0)
    m, enc, dec, cbs = build("ste", 0)
    m.train()
    batch = batch_of(dev(x))
    compiled = torch.compile(lambda b, t: m(b, t).loss, mode="reduce-overhead", fullgraph=True)
    opt = torch.optim.SGD(m.parameters(), lr=0.05)
    for step in range(4):
        loss_c = compiled(batch, T)
        loss_c.backward()
        gc = _grads(m)
        m.zero_grad(set_to_none=True)
        loss_e = m(batch, T).loss
        loss_e.backward()
        ge = _grads(m)
        assert torch.allclose(loss_c, loss_e, rtol=1e-5), (step, loss_c.item(), loss_e.item())
        for n in ge:
            assert torch.allclose(gc[n], ge[n], rtol=1e-4, atol=1e-6 * ge[n].abs().max().item() + 1e-12), (step, n)
        opt.step()
        m.zero_grad(set_to_none=True)


def test_forward_inside_a_compiled_caller_with_pending_kmeans_init():
    """The lazy k-means initialisation (train_rqvae.py:178-183) is data dependent: on the call that runs it the compiled caller
    breaks the graph around it and still returns the eager result."""
    g, x, _ = c1_inputs(0)
    from rq_vae_recommender_b200.modules.rqvae import RqVae
    from rq_vae_recommender_b200.modules.quantize import QuantizeForwardMode as M
    torch.manual_seed(3)
    m = RqVae(input_dim=x.shape[1], embed_dim=16, hidden_dims=[32], codebook_size=32, codebook_kmeans_init=True,
              codebook_mode=M.STE, n_layers=2, commitment_weight=BETA, n_cat_features=0).cuda()
    m.train()
    batch = batch_of(dev(x))
    compiled = torch.compile(lambda b, t: m(b, t), backend="eager")
    out = compiled(batch, T)
    assert all(l.kmeans_initted for l in m.layers)
    eager = m(batch, T)                                       # codebooks are initialised now: same weights, same result
    assert torch.allclose(out.loss, eager.loss, rtol=1e-5)
    out.loss.backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())
