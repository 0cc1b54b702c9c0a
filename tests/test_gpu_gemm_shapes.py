"""GPU tests of csrc/gemm_tc.cu (and the id histogram of csrc/dense.cu) at the operand widths, tile edges and layouts where the
kernels take different code: every instantiation of the row splitter and its scalar load path, the transposed splitter with a
row pitch, the epilogues at ragged N, every regime of the split-K schedule, the bf16 GEMM's persistent loop over several work
items per CTA, and sid_histogram's large-table and out-of-range paths.

The yardstick of the split-precision GEMM is tests/test_gpu_gemm_split.py's: error against the float64 product relative to
|a_i||b_j|, bounded by twice what plain fp32 torch makes on the same inputs.  Inputs are drawn on the device from fixed seeds.
`pytest -m gpu`."""
import numpy as np
import pytest
import torch

from test_gpu_gemm_split import _err_vs_f64

pytestmark = pytest.mark.gpu

# K = 1 .. 64 covers the row splitter <1,8>, then <1,16> to 128, <1,32> to 256, <2,32> to 512, <3,32> to 768, <4,32> to 1024,
# <12,32> to 3072 and the two-pass wide splitter above
KS = [1, 7, 8, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 513, 767, 768, 769, 1023, 1024, 1025, 1536, 2047, 3071,
      3072, 3073, 4096, 8192]
EDGE_MN = [(383, 129), (129, 383), (128, 127), (1, 383), (127, 1)]     # 128-row tiles and 128-column blocks: full, ragged, one


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(g, *shape):
    return torch.randn(*shape, device="cuda", generator=g)


def _floor(K):
    # Below one 64-wide k chunk a result sums too few products for their rounding errors to average out, and a plain fp32 GEMM
    # is nearly exact there; the bound is then the format's worst case per product: 2^-23 of the row maximum for hi + lo of each
    # operand, 2^-22 for the dropped lo.lo and the tensor core's truncating accumulation, 3 x 2^-22 in all
    return 3e-7 if K >= 64 else 3 * 2.0 ** -22


def _check(out, a, b_t, what, act=None):
    """out vs act(a @ b_t) in float64: the split GEMM's yardstick (a [M, K], b_t [K, N], both fp32 as the kernel read them)."""
    a64, b64 = a.double(), b_t.double()
    e_32, ref = _err_vs_f64(a @ b_t, a64, b64)
    if act is not None:
        ref = act(ref)
    scale = a64.norm(dim=1, keepdim=True) * b64.norm(dim=0, keepdim=True)
    e_tc = ((out.double() - ref).abs() / scale.clamp_min(1e-300)).max().item()
    bound = max(2.0 * e_32, _floor(a.shape[1]))
    assert e_tc <= bound, f"{what}: split GEMM error {e_tc:.3e} > {bound:.3e} (fp32 GEMM {e_32:.3e}, relative to |a||b|)"
    assert torch.allclose(out.double(), ref, rtol=1e-5, atol=1e-5 * ref.abs().max().item()), what
    return e_tc, e_32


def _layout(t, layout):
    """t [rows, K] as a contiguous tensor, as a view with row pitch K + 3, or as a view starting one float into its allocation
    (the last two are read by the row splitter's scalar loads)."""
    rows, K = t.shape
    if layout == "contiguous":
        return t.contiguous()
    if layout == "pitch":
        buf = torch.full((rows, K + 3), float("nan"), device="cuda")
        buf[:, :K] = t
        return buf[:, :K]
    buf = torch.full((rows * K + 1,), float("nan"), device="cuda")
    v = buf[1:].view(rows, K)
    v.copy_(t)
    return v


@pytest.mark.parametrize("layout", ["contiguous", "pitch", "offset"])
@pytest.mark.parametrize("K", KS)
def test_row_splitter_every_width_and_layout(K, layout):
    from rq_vae_recommender_b200 import ops
    M, N = EDGE_MN[KS.index(K) % len(EDGE_MN)]
    g = _gen(K)
    a = _layout(_randn(g, M, K) * torch.exp(_randn(g, M, 1)), layout)      # rows of very different norms
    b = _randn(g, N, K) * 0.05
    if layout == "offset":
        assert a.data_ptr() % 16 == 4
    calls = ops.SPLIT_CALLS
    out = ops.gemm_split(a, b)
    assert ops.SPLIT_CALLS == calls + 1 and out.shape == (M, N)
    e_tc, e_32 = _check(out, a, b.t(), f"K={K} {layout}")
    print(f"M={M} N={N} K={K} {layout}: split {e_tc:.3e}, fp32 {e_32:.3e}")


@pytest.mark.parametrize("pitch", [0, 5])
@pytest.mark.parametrize("K", KS)
def test_transposed_splitter_every_width_with_row_pitch(K, pitch):
    """Both operands given as [K, rows] (gs_colmax / gs_split_cols), ragged row counts, row pitch = rows + pitch."""
    from rq_vae_recommender_b200 import ops
    M, N = EDGE_MN[(KS.index(K) + 2) % len(EDGE_MN)]
    g = _gen(10_000 + K)

    def cols(rows, scale):
        buf = torch.full((K, rows + pitch), float("nan"), device="cuda")
        buf[:, :rows] = _randn(g, K, rows) * scale
        return buf[:, :rows]

    a_t = cols(M, torch.exp(_randn(g, 1, M)))                # image row i = column i: columns of very different norms
    b_t = cols(N, 0.05)
    out = ops.gemm_split(ops.SplitOperand(a_t, transposed=True), ops.SplitOperand(b_t, transposed=True))
    _check(out, a_t.t(), b_t, f"transposed K={K} pitch {pitch}")


@pytest.mark.parametrize("N", [1, 33, 129, 255])
def test_epilogues_at_ragged_n(N):
    """relu, mask (row pitch > N) and out= (ld > N) at column counts that end inside a 128-column block and inside a column
    pair; nothing is written past N."""
    from rq_vae_recommender_b200 import ops
    M, K = 300, 200
    g = _gen(20_000 + N)
    a = _randn(g, M, K)
    b = _randn(g, N, K) * 0.1
    mask_buf = _randn(g, M, N + 7)
    mask = mask_buf[:, :N]
    _check(ops.gemm_split(a, b, relu=True), a, b.t(), f"relu N={N}", act=lambda r: r.clamp_min(0))
    _check(ops.gemm_split(a, b, mask=mask), a, b.t(), f"mask N={N}", act=lambda r: r * (mask > 0))
    _check(ops.gemm_split(a, b, relu=True, mask=mask), a, b.t(), f"relu+mask N={N}",
           act=lambda r: r.clamp_min(0) * (mask > 0))
    big = torch.full((M, N + 9), 7.0, device="cuda")
    out = ops.gemm_split(a, b, out=big[:, :N])
    assert out.data_ptr() == big.data_ptr()
    assert torch.equal(big[:, N:], torch.full((M, 9), 7.0, device="cuda")), "written past N"
    _check(big[:, :N], a, b.t(), f"out= N={N}")


# (B, M, N): B on both sides of SPLIT_MIN_ROWS and ragged; (M, N) such that the slice count is 1 (>= 132 output tiles), the
# nkc / 4 cap (few tiles) or in between
SPLIT_K = [(511, 130, 70), (512, 130, 70), (513, 130, 70), (4095, 32, 128), (4095, 1536, 1536), (65537, 512, 768),
           (65537, 1, 33)]


@pytest.mark.parametrize("B,M,N", SPLIT_K)
def test_gemm_tn_split_k_regimes(B, M, N):
    from rq_vae_recommender_b200 import _lib, ops
    g = _gen(30_000 + B + M)
    a = _randn(g, B, M) * torch.exp(0.5 * _randn(g, 1, M))
    b = _randn(g, B, N) * 0.05
    calls = ops.SPLIT_CALLS
    out = ops.gemm_tn(a, b)
    assert ops.SPLIT_CALLS - calls == (B >= ops.SPLIT_MIN_ROWS), "tensor cores from SPLIT_MIN_ROWS batch rows on"
    slices = _lib.load().rqb200_gemm_split_k_slices(M, N, B)
    e_tc, e_32 = _check(out, a.t(), b, f"gemm_tn B={B} M={M} N={N}")
    print(f"B={B} M={M} N={N}: {slices} slices, split-K {e_tc:.3e}, fp32 {e_32:.3e}")
    assert torch.equal(out, ops.gemm_tn(a, b)), "fixed-order reduction: run-to-run identical"


def test_split_k_cases_cover_every_slice_regime():
    from rq_vae_recommender_b200 import _lib, ops
    lib = _lib.load()
    seen = set()
    for B, M, N in SPLIT_K:
        if B < ops.SPLIT_MIN_ROWS:
            continue
        nkc = (B + 63) // 64
        s = lib.rqb200_gemm_split_k_slices(M, N, B)
        kc_per = -(-nkc // max(1, nkc // 4))
        cap = -(-nkc // kc_per)                               # the slice count of the nkc / 4 cap, empty slices dropped
        assert 1 <= s <= cap and (s - 1) * -(-nkc // s) < nkc, (B, M, N, s)
        seen.add("one" if s == 1 else "cap" if s == cap else "middle")
    assert seen == {"one", "cap", "middle"}, seen


def _bf16_ref_layer(h, w):
    """Step (1) of test_gpu_parity.test_gemm_bf16_mlp_vs_bf16_oracle on the device: the layer's bf16-rounded input and weight
    multiplied in float64."""
    return h.to(torch.bfloat16).double() @ w.to(torch.bfloat16).double().t()


@pytest.mark.parametrize("M,dims", [(1, [64, 192, 1]), (127, [4096, 320, 33]), (129, [64, 64, 192, 70]),
                                    (129, [4096, 64, 1]), (65536, [512, 512, 512, 33]), (65536, [64, 320, 70])])
def test_bf16_mlp_layer_by_layer(M, dims):
    """gt_gemm_kernel: hidden widths with N % 128 = 64 (a group of one 128-column block), final N of 1 / 33 / 70, K = 64 and
    4096; 65 536 rows give up to 1024 work items, ~8 per CTA of the persistent loop."""
    from rq_vae_recommender_b200 import ops
    g = _gen(40_000 + M + sum(dims))
    x = _randn(g, M, dims[0]) * 0.3
    ws = [(torch.rand(o, i, device="cuda", generator=g) * 2 - 1) / i ** 0.5 for i, o in zip(dims[:-1], dims[1:])]
    prev = None
    for k in range(1, len(ws) + 1):
        yk = ops.mlp_forward_bf16(x, ws[:k])
        assert yk.shape == (M, dims[k])
        # the kernel's epilogue rounds relu(previous output) to bf16 for layer k: feed the reference exactly that
        expect = _bf16_ref_layer(x if prev is None else prev.clamp_min(0), ws[k - 1])
        err = (yk.double() - expect).abs().max().item() / max(expect.abs().max().item(), 1e-30)
        assert err < 1e-5, (M, dims, k, err)
        prev = yk


@pytest.mark.parametrize("L", [1, 3, 8])
@pytest.mark.parametrize("K", [1, 5, 256, 2048])
def test_sid_histogram_vs_bincount(K, L):
    """Ids of -1 and K are skipped; 10^6 rows run the grid-stride loop; K = 2048, L = 8 needs 64 KB of shared memory."""
    from rq_vae_recommender_b200 import ops
    g = _gen(50_000 + 16 * K + L)
    for B in (0, 1000, 1_000_000):
        ids = torch.randint(-1, K + 1, (B, L), device="cuda", generator=g)
        h = ops.sid_histogram(ids, K).cpu().numpy()
        host = ids.cpu().numpy()
        assert h.shape == (L, K) and h.dtype == np.int64
        for l in range(L):
            col = host[:, l]
            assert np.array_equal(h[l], np.bincount(col[(col >= 0) & (col < K)], minlength=K)), (B, l)


def test_sid_histogram_table_limit():
    """The [L, K] table lives in shared memory: up to 160 KB (K = 2048, L = 20) it runs, past it the call raises."""
    from rq_vae_recommender_b200 import _lib, ops
    ids = torch.randint(0, 2048, (5000, 20), device="cuda", generator=_gen(60_000))
    h = ops.sid_histogram(ids, 2048)
    host = ids.cpu().numpy()
    assert all(np.array_equal(h[l].cpu().numpy(), np.bincount(host[:, l], minlength=2048)) for l in range(20))
    with pytest.raises(_lib.Rqb200Error):
        ops.sid_histogram(torch.zeros((10, 21), dtype=torch.int64, device="cuda"), 2048)


def test_rqvae_4096_wide_items_match_the_cuda_core_path(monkeypatch):
    """An RqVae over 4096-wide item embeddings: a train step at 640 rows (encoder input, decoder output and its dgrad on the
    split GEMM) and tokenize at 640 and 4096 rows equal the same model run on the CUDA-core SGEMM (SPLIT_MIN_ROWS raised)."""
    from rq_vae_recommender_b200 import ops
    from parity import assert_ids_match, rel_err
    from test_gpu_modules import batch_of, build
    import inputs as I
    Din, D, K, L, N = 4096, 32, 256, 3, 4096
    m, *_ = build("ste", 0, Din=Din, D=D, hidden=(512, 256, 128), K=K, L=L, seed=700)
    x = torch.from_numpy(I.unit_rows(701, N, Din)).cuda()
    with torch.no_grad():          # live codebooks: residual rows of the encoder output, like a k-means-initialised model
        res = m.encode(x)
        for l, layer in enumerate(m.layers):
            layer.embedding.weight.copy_(res[torch.randperm(N, generator=torch.Generator().manual_seed(l))[:K].cuda()])
            res = res - layer.embedding.weight[ops.rq_tokenize(res, [layer.embedding.weight])[:, 0]]

    def run():
        m.train()
        m.zero_grad()
        fo = m(batch_of(x[:640]), 0.2)
        fo.loss.backward()
        m.eval()
        with torch.no_grad():
            out = [m.tokenize(x[:640]), m.tokenize(x), m.encode(x)]
        return ([fo.loss.item(), fo.reconstruction_loss.item(), fo.rqvae_loss.item()],
                {n: p.grad.clone() for n, p in m.named_parameters()}, out)

    calls = ops.SPLIT_CALLS
    losses, grads, (ids640, ids, z) = run()
    assert ops.SPLIT_CALLS > calls
    monkeypatch.setattr(ops, "SPLIT_MIN_ROWS", 1 << 62)
    calls = ops.SPLIT_CALLS
    losses_sg, grads_sg, (ids640_sg, ids_sg, z_sg) = run()
    assert ops.SPLIT_CALLS == calls
    assert np.allclose(losses, losses_sg, rtol=1e-5), (losses, losses_sg)
    for n in grads:
        assert rel_err(grads[n].cpu().numpy(), grads_sg[n].cpu().numpy()) < 1e-4, n
    assert rel_err(z.cpu().numpy(), z_sg.cpu().numpy()) < 1e-5
    cbs = [layer.codebook().detach().cpu().numpy() for layer in m.layers]
    zh = z_sg.double().cpu().numpy()
    assert_ids_match(ids640.cpu().numpy(), ids640_sg.cpu().numpy(), zh[:640], cbs, "tokenize 640 rows")
    assert_ids_match(ids.cpu().numpy(), ids_sg.cpu().numpy(), zh, cbs, "tokenize 4096 rows")
    assert len(np.unique(ids_sg.cpu().numpy(), axis=0)) > N // 4, "live codebooks"
