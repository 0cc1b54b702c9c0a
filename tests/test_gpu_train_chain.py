"""The training-mode quantiser kernels against the float64 reference (tests/train_chain_ref.py) at every row-tile height of the
fused chain and at training batch sizes: rq_fused_kernel, rq_replay_kernel, rq_bwd_kernel, the Gumbel-softmax row kernels,
the k-means kernels and the L2 norm.  Ids come from the kernel under test and are checked with the near-tie protocol; every
value is then compared with the reference evaluated on those same ids.  `pytest -m gpu`."""
import re

import pytest
import torch
import torch.nn.functional as F

import train_chain_ref as R
from parity import assert_ids_match

pytestmark = pytest.mark.gpu

BETA, T = 0.25, 0.2
MODES = {"eval": R.EVAL, "ste": R.STE, "rot": R.ROT}
OUTS = ("ids", "embeddings", "residuals", "emb_sum", "emb_norms", "loss")
WANT = dict(zip(OUTS, ("want_ids", "want_embeddings", "want_residuals", "want_sum", "want_norms", "want_loss")))
ALL = {w: True for w in WANT.values()}


@pytest.fixture(scope="module")
def ops():
    from rq_vae_recommender_b200 import ops as _ops
    return _ops


# ------------------------------------------------------------------ inputs and comparisons
def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def argmin64(res, cb):
    cc = (cb.double() ** 2).sum(1)
    out = torch.empty(res.shape[0], dtype=torch.int64, device=res.device)
    for s in range(0, res.shape[0], 8192):
        out[s:s + 8192] = (cc[None] - 2 * res[s:s + 8192].double() @ cb.double().t()).argmin(1)
    return out


def problem(B, D, K, L, seed):
    """Unit rows and L live codebooks (level-l codes are level-l residual rows plus jitter), generated on the device."""
    g = gen(seed)
    x = torch.randn(B, D, generator=g, device="cuda", dtype=torch.float64)
    x = (x / x.norm(dim=1, keepdim=True)).float()
    res, cbs = x.double(), []
    for _ in range(L):
        idx = torch.randint(0, B, (K,), generator=g, device="cuda")
        jitter = torch.randn(K, D, generator=g, device="cuda", dtype=torch.float64) * (0.5 / D ** 0.5)
        cb = (res[idx] + jitter).float()
        cbs.append(cb)
        res = res - cb.double()[argmin64(res, cb)]
    return x, cbs


def check_ids(ids, x, cbs, what=""):
    """Kernel ids [B, L] against the float64 chain's own argmins, through the near-tie protocol."""
    res, ref = x.double(), []
    for cb in cbs:
        i = argmin64(res, cb)
        ref.append(i)
        res = res - cb.double()[i]
    return assert_ids_match(ids.cpu().numpy(), torch.stack(ref, 1).cpu().numpy(), x.cpu().numpy(),
                            [c.cpu().numpy() for c in cbs], what)


def rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-300)).item()


def close(what, got, ref64, ref32=None, tol=2e-5):
    """rel_err(got, float64) < tol.  Where fp32 itself drifts further (deep chains, Gumbel softmax at T = 0.2), an fp32 torch
    restatement ``ref32`` sets the bound instead: at most twice its own error against float64."""
    err = rel(got, ref64)
    bound = tol if ref32 is None else max(tol, 2.0 * rel(ref32, ref64))
    assert err < bound, f"{what}: rel err {err:.3e} >= {bound:.3e}" + ("" if ref32 is None else " (2 x fp32 torch's, or tol)")


def row_major(o):
    """Kernel outputs ([L, B, D] embeddings / residuals) in the reference's row-major layout."""
    return {k: (v.permute(1, 0, 2) if k in ("embeddings", "residuals") else v) for k, v in o.items() if v is not None}


def compare_forward(o, x, cbs, mode, what, ref32=False):
    """Every requested output of ops.rq_forward against the float64 chain on the kernel's ids."""
    check_ids(o["ids"], x, cbs, what)
    fn = R.chain(mode, BETA)
    ref, _, _ = R.evaluate(fn, x, cbs, (o["ids"],), chunk=16384)
    r32 = R.evaluate(fn, x, cbs, (o["ids"],), chunk=16384, dtype=torch.float32)[0] if ref32 else {}
    for k, v in row_major(o).items():
        if k != "ids":
            close(f"{what} {k}", v, ref[k], r32.get(k))


# ------------------------------------------------------------------ the fused kernel's tile geometry (csrc/rq_simt.cu)
def tile_n(K):
    return 1 if K <= 32 else 2 if K <= 64 else 4 if K <= 128 else 8


def heights(K, D):
    """Row-tile heights TM whose shared-memory tile fits 200 KB (fused_smem_bytes); RQB200_TM is ignored for the others."""
    Dp = -(-D // 16) * 16
    return [tm for tm in (8, 4, 2, 1) if (3 * 16 * 32 * tile_n(K) + 8 * tm * (Dp + 4)) * 4 + 3 * 8 + 64 <= 200 * 1024]


def fused_instantiations(run):
    """(TM, TN, DIRECT) of every rq_fused_kernel launched by run(), from torch.profiler's CUDA activity.  A fill kernel launched
    after run() tells a complete trace from one whose kernel records the profiler did not deliver (it happens, rarely, between
    back-to-back sessions); such a trace says nothing about what ran, so run() is profiled again."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
            torch.full((1,), 7.0, device="cuda")
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        if any("FillFunctor" in n for n in names):
            break
    else:
        raise AssertionError("three profiler traces in a row hold no record of the marker kernel")
    found = set()
    for name in names:
        m = re.search(r"rq_fused_kernel<(\d+), (\d+), (true|false)>", name)
        if m:
            found.add((int(m.group(1)), int(m.group(2)), m.group(3) == "true"))
    return found


# ------------------------------------------------------------------ 1. tile-height sweep of the fused forward
SWEEP = [(1003, 20, 5, 3), (515, 1536, 5, 1), (777, 128, 50, 8), (1001, 768, 100, 3), (71, 1536, 100, 8),
         (999, 128, 256, 3), (1003, 768, 256, 1), (333, 20, 300, 8), (517, 1536, 300, 3), (301, 128, 2048, 3),
         (123, 768, 2048, 8), (1021, 20, 2048, 1)]


@pytest.mark.parametrize("B,D,K,L", SWEEP)
@pytest.mark.parametrize("mname", ["eval", "ste", "rot"])
def test_fused_forward_is_identical_at_every_tile_height(ops, monkeypatch, B, D, K, L, mname):
    """A row's arithmetic does not depend on how many rows a warp holds: every output is bit-identical at every height TM that
    fits, and matches the float64 chain once.  The profiler confirms which instantiation ran."""
    x, cbs = problem(B, D, K, L, seed=B + D + K + L)
    mode = MODES[mname]
    tms = heights(K, D)
    outs = {}
    for tm in tms:
        monkeypatch.setenv("RQB200_TM", str(tm))
        run = lambda: outs.__setitem__(tm, ops.rq_forward(x, cbs, mode, BETA, **ALL))
        if mname == "eval":
            assert fused_instantiations(run) == {(tm, tile_n(K), False)}, f"TM={tm} did not run"
        else:
            run()
    for tm in tms[1:]:
        for k in OUTS:
            assert torch.equal(outs[tm][k], outs[tms[0]][k]), f"{k} differs between TM={tms[0]} and TM={tm}"
    compare_forward(outs[tms[0]], x, cbs, mode, f"{mname} B={B} D={D} K={K} L={L}", ref32=L == 8)


# ------------------------------------------------------------------ 2. optional outputs and row strides
@pytest.mark.parametrize("B,D,K,L", [(1003, 20, 5, 3), (999, 128, 256, 3), (3001, 64, 256, 3), (2050, 20, 2048, 2)])
@pytest.mark.parametrize("mname", ["eval", "ste", "rot"])
def test_each_output_alone_and_strided_rows(ops, B, D, K, L, mname):
    """Requesting one output gives bit for bit what requesting all gives; a column slice of a wider tensor (16-byte aligned
    start: vector loads; misaligned: scalar loads) gives bit for bit what its contiguous copy gives."""
    x, cbs = problem(B, D, K, L, seed=3 * B + K)
    mode = MODES[mname]
    full = ops.rq_forward(x, cbs, mode, BETA, **ALL)
    for k in OUTS:
        alone = ops.rq_forward(x, cbs, mode, BETA, **{WANT[j]: j == k for j in OUTS})
        assert torch.equal(alone[k], full[k]), f"{k} alone differs"
        assert all(alone[j] is None for j in OUTS if j != k)
    wide = torch.randn(B, D + 12, generator=gen(B), device="cuda")
    for off in (4, 3):
        wide[:, off:off + D] = x
        xs = wide[:, off:off + D]
        assert xs.stride(0) == D + 12 and (xs.data_ptr() % 16 == 0) == (off == 4)
        strided = ops.rq_forward(xs, cbs, mode, BETA, **ALL)
        for k in OUTS:
            assert torch.equal(strided[k], full[k]), f"offset {off}: {k} differs"


# ------------------------------------------------------------------ 3. training batch sizes
@pytest.mark.parametrize("mname", ["eval", "ste", "rot"])
def test_fused_route_at_its_natural_height(ops, monkeypatch, mname):
    """20 000 rows at D = 128, K = 300 (no tensor-core tokeniser for K = 300): the fused kernel picks TM = 8 itself."""
    monkeypatch.delenv("RQB200_TM", raising=False)
    B, D, K, L = 20000, 128, 300, 3
    x, cbs = problem(B, D, K, L, seed=11)
    o = {}
    ran = fused_instantiations(lambda: o.update(ops.rq_forward(x, cbs, MODES[mname], BETA, **ALL)))
    assert ran == {(8, 8, False)}, ran
    compare_forward(o, x, cbs, MODES[mname], f"{mname} fused TM=8")


@pytest.mark.parametrize("D,L", [(32, 3), (64, 8)])
@pytest.mark.parametrize("mname", ["eval", "ste", "rot"])
def test_tensor_core_and_replay_route_at_training_batch(ops, mname, D, L):
    """20 000 rows: ids from the tensor-core tokeniser, every other output from rq_replay_kernel (rows past its grid cap of
    132 x 8 CTAs x 8 warps go through the grid-stride loop).  Bit-identical to the fused route, and right against float64."""
    B, K = 20000, 256
    x, cbs = problem(B, D, K, L, seed=D + L)
    mode = MODES[mname]
    calls = ops.TC_CALLS
    new = ops.rq_forward(x, cbs, mode, BETA, **ALL)
    assert ops.TC_CALLS == calls + 1
    old_min, ops.TC_MIN_ROWS = ops.TC_MIN_ROWS, 1 << 62
    try:
        ref = ops.rq_forward(x, cbs, mode, BETA, **ALL)
    finally:
        ops.TC_MIN_ROWS = old_min
    for k in OUTS:
        assert torch.equal(new[k], ref[k]), f"{k} differs from the fused route"
    compare_forward(new, x, cbs, mode, f"{mname} replay D={D} L={L}", ref32=L == 8)


@pytest.mark.parametrize("mname", ["eval", "ste", "rot"])
def test_replay_with_fewer_warps_per_cta(ops, mname):
    """rq_forward_from_ids at D = 4096 runs 4 warps per CTA (and 5 000 rows loop past its grid cap): every output equals the
    fused kernel's on the fused kernel's ids."""
    from rq_vae_recommender_b200 import _lib
    B, D, K, L = 5000, 4096, 64, 2
    x, cbs = problem(B, D, K, L, seed=4096)
    mode = MODES[mname]
    fused = ops.rq_forward(x, cbs, mode, BETA, **ALL)
    out = {k: torch.full_like(fused[k], float("nan")) for k in OUTS[1:]}
    lib = _lib.load()
    _lib.check(lib.rqb200_rq_forward_from_ids(mode, x.data_ptr(), x.stride(0), ops._ptr_array(cbs), fused["ids"].data_ptr(),
                                              B, D, K, L, BETA, *(out[k].data_ptr() for k in OUTS[1:]),
                                              torch.cuda.current_stream().cuda_stream), "rq_forward_from_ids")
    for k in OUTS[1:]:
        assert torch.equal(out[k], fused[k]), f"{k} differs"
    compare_forward(fused, x, cbs, mode, f"{mname} D=4096")


# ------------------------------------------------------------------ 4. backward against float64 autograd
BWD = {"20000x768 L3": (20000, 768, 256, 3), "5000x768 L8": (5000, 768, 300, 8), "3000x1536 L8": (3000, 1536, 64, 8),
       "B1": (1, 64, 32, 3), "D20": (777, 20, 40, 3)}
VARIANTS = ("dense", "expanded", "permuted", "unused", "frozen", "strided")
_PROBLEMS = {}


def bwd_problem(name):
    if name not in _PROBLEMS:
        _PROBLEMS[name] = problem(*BWD[name], seed=len(name) + BWD[name][0])
    return _PROBLEMS[name]


def run_backward(ops, x, cbs, mode, lean, variant, seed):
    """Kernel gradients of one objective, and the upstream gradients (row-major) the float64 reference needs for it.

    dense:    random upstream gradients of every differentiable output;
    expanded: out.sum() (stride-0 gradients);
    permuted: the [B, D, L] permute of the non-lean outputs (lean: the transpose of emb_sum), non-contiguous gradients;
    unused:   non-lean: the residual output unused (no gradient); lean: the loss unused;
    frozen:   levels 0, 2, 4, ... frozen (no codebook gradient);
    strided:  x a column slice of a wider tensor."""
    B, D = x.shape
    L = len(cbs)
    g = gen(seed)
    rnd = lambda *s: torch.randn(*s, generator=g, device="cuda")
    if variant == "strided":
        wide = torch.zeros(B, D + 5, device="cuda")
        wide[:, 3:3 + D] = x
        wide.requires_grad_(True)
        xt = wide[:, 3:3 + D]
    else:
        xt = x.clone().requires_grad_(True)
    cts = [c.clone().requires_grad_(variant != "frozen" or l % 2 == 1) for l, c in enumerate(cbs)]
    a, b, ids, loss = ops.RqChainFunction.apply(xt, mode, BETA, lean, *cts)
    gl = torch.rand(B, generator=g, device="cuda")
    up = {}
    if variant == "expanded":
        obj = a.sum() + loss.sum() + (0 if lean else b.sum())
        up = {"emb_sum" if lean else "embeddings": torch.ones(B, *(() if lean else (L,)), D, device="cuda"),
              "loss": torch.ones(B, device="cuda")}
        if not lean:
            up["residuals"] = torch.ones(B, L, D, device="cuda")
    elif variant == "permuted":
        if lean:
            ga = rnd(D, B)
            obj = (a.t() * ga).sum() + (loss * gl).sum()
            up = {"emb_sum": ga.t(), "loss": gl}
        else:
            ga, gb = rnd(B, D, L), rnd(B, D, L)
            obj = (a.permute(1, 2, 0) * ga).sum() + (b.permute(1, 2, 0) * gb).sum() + (loss * gl).sum()
            up = {"embeddings": ga.permute(0, 2, 1), "residuals": gb.permute(0, 2, 1), "loss": gl}
    else:
        ga = rnd(*a.shape)
        obj = (a * ga).sum()
        up = {"emb_sum": ga} if lean else {"embeddings": ga.permute(1, 0, 2)}
        if not (lean and variant == "unused"):
            obj = obj + (loss * gl).sum()
            up["loss"] = gl
        if not lean and variant != "unused":
            gb = rnd(*b.shape)
            obj = obj + (b * gb).sum()
            up["residuals"] = gb.permute(1, 0, 2)
    obj.backward()
    gx = wide.grad if variant == "strided" else xt.grad
    return ids, a, loss, gx, [c.grad for c in cts], up


@pytest.mark.parametrize("shape", list(BWD))
@pytest.mark.parametrize("lean", [True, False])
@pytest.mark.parametrize("mname", ["eval", "ste", "rot"])
def test_backward_vs_float64_autograd(ops, shape, lean, mname):
    """rq_bwd_kernel for every upstream-gradient layout RqChainFunction accepts, against float64 autograd on the same ids.
    5 000 x 768 at L = 8 runs 4 warps per CTA and 3 000 x 1536 at L = 8 runs 2; both, and 20 000 rows, loop past the grid cap
    of 132 x 8 CTAs."""
    x, cbs = bwd_problem(shape)
    B, D, K, L = BWD[shape]
    mode = MODES[mname]
    fn = R.chain(mode, BETA)
    for i, variant in enumerate(VARIANTS):
        what = f"{mname} {shape} lean={lean} {variant}"
        ids, a, loss, gx, gcs, up = run_backward(ops, x, cbs, mode, lean, variant, seed=100 + i)
        if i == 0:
            check_ids(ids, x, cbs, what)
        ref, rgx, rgcs = R.evaluate(fn, x, cbs, (ids,), upstream=up, chunk=8192)
        r32 = R.evaluate(fn, x, cbs, (ids,), upstream=up, chunk=8192, dtype=torch.float32) if L == 8 else (None,) * 3
        if variant == "dense":
            k = "emb_sum" if lean else "embeddings"
            close(f"{what} fwd", a if lean else a.permute(1, 0, 2), ref[k], None if r32[0] is None else r32[0][k])
            close(f"{what} loss", loss, ref["loss"], None if r32[0] is None else r32[0]["loss"])
        if variant == "strided":
            assert not gx[:, :3].any() and not gx[:, 3 + D:].any()
            gx = gx[:, 3:3 + D]
        close(f"{what} g_x", gx, rgx, r32[1])
        for l in range(L):
            if variant == "frozen" and l % 2 == 0:
                assert gcs[l] is None
            else:
                close(f"{what} g_codebook[{l}]", gcs[l], rgcs[l], None if r32[2] is None else r32[2][l])


class MaxRel:
    """rel_err accumulated over row chunks: max |a - b| / max |b|."""

    def __init__(self):
        self.num, self.den = 0.0, 0.0

    def add(self, a, b):
        self.num = max(self.num, (a.double() - b).abs().max().item())
        self.den = max(self.den, b.abs().max().item())

    def value(self):
        return self.num / max(self.den, 1e-300)


def test_rotation_at_the_benchmark_shape(ops):
    """65 536 x 768, K = 256, L = 3 rotation trick (the benchmark's c4 arm): every forward output and every gradient, with the
    float64 reference run on the device in row chunks."""
    B, D, K, L = 65536, 768, 256, 3
    x, cbs = problem(B, D, K, L, seed=65536)
    o = ops.rq_forward(x, cbs, R.ROT, BETA, **ALL)
    check_ids(o["ids"], x, cbs, "c4")
    fwd = row_major(o)
    errs = {k: MaxRel() for k in OUTS[1:]}
    xt = x.clone().requires_grad_(True)
    cts = [c.clone().requires_grad_(True) for c in cbs]
    esum, _norms, ids, loss = ops.RqChainFunction.apply(xt, R.ROT, BETA, True, *cts)
    assert torch.equal(ids, o["ids"]) and torch.equal(esum, o["emb_sum"]) and torch.equal(loss, o["loss"])
    ge = torch.randn(B, D, generator=gen(1), device="cuda")
    gl = torch.rand(B, generator=gen(2), device="cuda")
    ((esum * ge).sum() + (loss * gl).sum()).backward()

    def on_chunk(rows, out):
        for k in errs:
            errs[k].add(fwd[k][rows], out[k])
    _, rgx, rgcs = R.evaluate(R.chain(R.ROT, BETA), x, cbs, (o["ids"],), upstream={"emb_sum": ge, "loss": gl}, chunk=8192,
                              on_chunk=on_chunk)
    for k, e in errs.items():
        assert e.value() < 2e-5, f"{k}: {e.value():.3e}"
    close("g_x", xt.grad, rgx)
    for l in range(L):
        close(f"g_codebook[{l}]", cts[l].grad, rgcs[l])


# ------------------------------------------------------------------ 5. Gumbel-softmax
def gumbel_kernel_chain(ops, x, cbs, U):
    res, embs, ids, loss = x, [], [], 0
    for l, cb in enumerate(cbs):
        e, i, lo = ops.GumbelQuantizeFunction.apply(res, cb, U[:, l], T, BETA)
        embs.append(e)
        ids.append(i)
        loss = loss + lo
        res = res - e
    return torch.stack(embs, 1), torch.stack(ids, 1), loss


@pytest.mark.parametrize("B,D,K,L", [(300, 64, 256, 3), (5000, 128, 256, 3), (65536, 768, 256, 3), (64, 16, 8448, 1)])
def test_gumbel_chain_vs_float64(ops, B, D, K, L):
    """L chained GumbelQuantizeFunction levels (the gradient flows back through the residual) with fixed uniforms, against
    float64 autograd: B = 300 runs the CUDA-core SGEMM, 5 000 the split-precision GEMMs with rows past the softmax backward's
    grid cap, 65 536 x 768 the benchmark shape, K = 8 448 the softmax backward's global column sums.  Softmax at T = 0.2
    amplifies fp32 rounding, so the bound is twice an fp32 torch restatement's error against float64."""
    x, cbs = problem(B, D, K, L, seed=B + K)
    U = torch.rand(B, L, K, generator=gen(B), device="cuda")
    xt = x.clone().requires_grad_(True)
    cts = [c.clone().requires_grad_(True) for c in cbs]
    E, ids, loss = gumbel_kernel_chain(ops, xt, cts, U)
    ge = torch.randn(B, L, D, generator=gen(3), device="cuda")
    gl = torch.rand(B, generator=gen(4), device="cuda")
    ((E * ge).sum() + (loss * gl).sum()).backward()
    up = {"embeddings": ge, "loss": gl}
    fn = R.gumbel_chain(T, BETA)
    chunk = 8192
    ref, rgx, rgcs = R.evaluate(fn, x, cbs, (U,), upstream=up, chunk=chunk)
    with R.highest_matmul_precision():
        r32, sgx, sgcs = R.evaluate(fn, x, cbs, (U,), upstream=up, chunk=chunk, dtype=torch.float32)
    # level 0 sees the same input: its ids must be the float64 argmin wherever float64 does not call a near-tie
    d64 = (x.double() ** 2).sum(1, keepdim=True) + (cbs[0].double() ** 2).sum(1)[None] - 2 * x.double() @ cbs[0].double().t()
    top2 = d64.topk(2, dim=1, largest=False)
    clear = (top2.values[:, 1] - top2.values[:, 0]) > 1e-5 * top2.values[:, 0].abs()
    assert clear.float().mean() > 0.9 and torch.equal(ids[clear, 0], ref["ids"][clear, 0])
    close("embeddings", E, ref["embeddings"], r32["embeddings"])
    close("loss", loss, ref["loss"], r32["loss"])
    close("g_x", xt.grad, rgx, sgx)
    for l in range(L):
        close(f"g_codebook[{l}]", cts[l].grad, rgcs[l], sgcs[l])


# ------------------------------------------------------------------ 6. k-means kernels
def kmeans_problem(B, D, K, seed, strided):
    g = gen(seed)
    x = torch.randn(B, D + 7, generator=g, device="cuda")
    x = x[:, 2:2 + D] if strided else x[:, :D].contiguous()
    if B:
        cent = x[torch.randint(0, B, (K,), generator=g, device="cuda")] + 0.1 * torch.randn(K, D, generator=g, device="cuda")
    else:
        cent = torch.randn(K, D, generator=g, device="cuda")
    cent[::7] = 1e3 + torch.randn(cent[::7].shape, generator=g, device="cuda")    # far from every row: empty clusters
    return x, cent.contiguous()


def direct_dist64(x, cent, rows):
    x64, c64 = x[rows].double(), cent.double()
    out = torch.empty(x64.shape[0], c64.shape[0], dtype=torch.float64, device="cuda")
    step = max(1, (1 << 25) // (c64.numel()))
    for s in range(0, x64.shape[0], step):
        out[s:s + step] = ((x64[s:s + step, None, :] - c64[None]) ** 2).sum(-1)
    return out


KM = [(1000, 3, 5), (2000, 16, 32), (777, 33, 100), (1500, 768, 300), (5000, 16, 2048), (900, 768, 2048), (0, 16, 32)]


@pytest.mark.parametrize("B,D,K", KM)
@pytest.mark.parametrize("strided", [False, True])
def test_kmeans_kernels(ops, monkeypatch, B, D, K, strided):
    """kmeans_assign_accumulate at every tile height (assignments and counts bit-identical across heights), against a float64
    direct-distance argmin, its own bincount and a float64 sum over its own assignment; then kmeans_finalize: means, reseeded
    empty clusters, -1 and NULL reseeds, and the max shift."""
    x, cent = kmeans_problem(B, D, K, seed=B + D + K + strided, strided=strided)
    assert B == 0 or x.is_contiguous() != strided
    runs = {}
    for tm in heights(K, D):
        monkeypatch.setenv("RQB200_TM", str(tm))
        buf = ops.kmeans_workspace(x, K)
        buf["sums"].fill_(float("nan"))
        buf["counts"].fill_(-1)
        ops.kmeans_assign_accumulate(x, cent, buf)
        runs[tm] = buf
    tms = list(runs)
    buf = runs[tms[0]]
    for tm in tms[1:]:
        assert torch.equal(runs[tm]["assign"], buf["assign"]) and torch.equal(runs[tm]["counts"], buf["counts"]), tm
        assert rel(runs[tm]["sums"], buf["sums"]) < 1e-12
    assign, counts, sums = buf["assign"], buf["counts"], buf["sums"]
    assert torch.equal(counts.long(), torch.bincount(assign, minlength=K))
    ref_sums = torch.zeros(K, D, dtype=torch.float64, device="cuda").index_add_(0, assign, x.double())
    if B:
        assert rel(sums, ref_sums) < 1e-12
        d = direct_dist64(x, cent, slice(None))
        dmin = d.min(1).values
        excess = d.gather(1, assign[:, None])[:, 0] - dmin
        assert (excess <= 1e-5 * dmin).all(), f"{int((excess > 1e-5 * dmin).sum())} rows off the float64 argmin"
        assert (counts[::7] == 0).all()
    else:
        assert not sums.any() and not counts.any()

    # finalize: reseed half of the empty clusters from a row, the rest with -1; then the same with a NULL reseed table
    empty = torch.nonzero(counts == 0).flatten()
    for with_table in (True, False):
        c = cent.clone()
        reseed = None
        if with_table:
            reseed = torch.full((K,), -1, dtype=torch.int64, device="cuda")
            if B:
                reseed[empty[::2]] = torch.randint(0, B, (len(empty[::2]),), generator=gen(7), device="cuda")
        ops.kmeans_finalize(x, c, buf, reseed)
        expect = cent.clone()
        full = counts > 0
        expect[full] = (sums[full] / counts[full, None].double()).float()
        if reseed is not None:
            r = reseed >= 0
            expect[r] = x[reseed[r]]
        assert torch.equal(c, expect), f"finalize (reseed table: {with_table})"
        shift = (c.double() - cent.double()).norm(dim=1).max()
        assert abs(buf["shift"].item() - shift.item()) <= 1e-6 * shift.item()


# ------------------------------------------------------------------ 7. L2 norm
@pytest.mark.parametrize("D", [1, 31, 32, 33, 768])
@pytest.mark.parametrize("B", [1, 9, 4097])
def test_l2norm_vs_float64_autograd(ops, B, D):
    """L2NormFunction forward and backward against float64 F.normalize autograd, with zero rows and rows of norm below eps
    (the only rows where the clamp changes the gradient: gx = gy / eps)."""
    eps = 1e-12
    g = gen(B * 1000 + D)
    x = torch.randn(B, D, generator=g, device="cuda")
    if B > 1:
        x[1] = 0
        x[2] = 1e-14
        x[3:5] *= 0.5 * eps / x[3:5].double().norm(dim=1, keepdim=True).float()   # 0 < ||x|| = eps / 2
        x[5] *= 1e3
    gy = torch.randn(B, D, generator=g, device="cuda")
    xt = x.clone().requires_grad_(True)
    y = ops.L2NormFunction.apply(xt, eps)
    (y * gy).sum().backward()
    x64 = x.double().requires_grad_(True)
    y64 = F.normalize(x64, p=2, dim=-1, eps=eps)
    (y64 * gy.double()).sum().backward()

    den = x.double().norm(dim=1).clamp_min(eps)

    def rowwise(a, b, scale):     # per-row error in units of the row's own scale: rows at 1 / eps must not hide the others
        return ((a.double() - b).abs().max(1).values / scale).max().item()
    assert rowwise(y, y64, x.double().abs().max(1).values.clamp_min(1e-300) / den) < 2e-5
    assert rowwise(xt.grad, x64.grad, gy.double().abs().max(1).values / den) < 2e-5
