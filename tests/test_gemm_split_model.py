"""CPU model of the split-precision tensor-core GEMM (csrc/gemm_tc.cu: gs_split_* / gs_gemm_kernel): the operand representation
and the accumulation scheme restated in numpy, checked against float64.  It pins the two design claims of DESIGN.md 5.3 without a
GPU: (1) hi + lo fp16 images of a power-of-two scaled row carry the operand to ~2^-22, so three products reproduce the fp32
product; (2) with an fp32 accumulator that truncates after every MMA (the behaviour tensor-core measurements match), ONE accumulator
loses ~3x more than hi.hi and the cross terms kept apart -- the reason the products are kept in short tensor-core sums (the kernel promotes every 64 k into an fp32 total)."""
import numpy as np
import pytest


def split_rows(a):
    """gs_split_rows_kernel: scale 2^e puts the row maximum into [2^14, 2^15); hi = fp16(v 2^e), lo = fp16(v 2^e - hi)."""
    mx = np.abs(a).max(axis=1, keepdims=True)
    _, ex = np.frexp(np.where(mx > 0, mx, 1.0))
    s = np.where(mx > 0, np.exp2(np.clip(15 - ex, -120, 120)), 1.0).astype(np.float32)
    t = (a * s).astype(np.float32)
    hi = t.astype(np.float16)
    lo = (t - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64), s.astype(np.float64)


def trunc24(x):
    m, e = np.frexp(x)
    return np.ldexp(np.trunc(m * 2.0 ** 24) / 2.0 ** 24, e)


def model_gemm(a, b, separate):
    ah, al, sa = split_rows(a)
    bh, bl, sb = split_rows(b)
    main = np.zeros((a.shape[0], b.shape[0]))
    cross = np.zeros_like(main)
    for k0 in range(0, a.shape[1], 16):                       # one MMA = 16 k: products exact, accumulator truncated
        sl = slice(k0, k0 + 16)
        if separate:
            main = trunc24(main + ah[:, sl] @ bh[:, sl].T)
            cross = trunc24(cross + al[:, sl] @ bh[:, sl].T)
            cross = trunc24(cross + ah[:, sl] @ bl[:, sl].T)
        else:
            for x, y in ((ah, bh), (al, bh), (ah, bl)):
                main = trunc24(main + x[:, sl] @ y[:, sl].T)
    tot = (main.astype(np.float32) + cross.astype(np.float32)).astype(np.float64)
    return tot / sa / sb.T


def problem(M, N, K, seed):
    rng = np.random.default_rng(seed)
    a = (rng.standard_normal((M, K)) * np.exp(rng.standard_normal((M, 1)))).astype(np.float32)
    b = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    ref = a.astype(np.float64) @ b.astype(np.float64).T
    scale = np.linalg.norm(a.astype(np.float64), axis=1)[:, None] * np.linalg.norm(b.astype(np.float64), axis=1)[None, :]
    return a, b, ref, scale


def test_split_representation_carries_22_bits():
    rng = np.random.default_rng(0)
    a = (rng.standard_normal((64, 768)) * np.exp(3 * rng.standard_normal((64, 1)))).astype(np.float32)
    a[3] = 0.0
    a[4, 7] = 1e6                                             # one dominant element: the small ones get a subnormal lo
    hi, lo, s = split_rows(a)
    assert np.abs(hi).max() <= 2.0 ** 15 and np.isfinite(hi).all()      # (a maximum just below 2^15 may round up to it)
    rec = (hi + lo) / s
    rowmax = np.abs(a).max(axis=1, keepdims=True).astype(np.float64)
    # per element: 2^-22 relative, or 2^-25 absolute in scaled units (= 2^-39 of the row maximum) when lo is subnormal
    bound = np.maximum(2.0 ** -22 * np.abs(a.astype(np.float64)), 2.0 ** -39 * rowmax)
    assert (np.abs(rec - a.astype(np.float64)) <= bound + 1e-300).all()


@pytest.mark.parametrize("K", [64, 256, 768])
def test_three_products_match_float64_and_two_accumulators_pay(K):
    a, b, ref, scale = problem(96, 96, K, seed=K)
    e_two = (np.abs(model_gemm(a, b, separate=True) - ref) / scale).max()
    e_one = (np.abs(model_gemm(a, b, separate=False) - ref) / scale).max()
    e_f32 = (np.abs((a @ b.T).astype(np.float64) - ref) / scale).max()
    assert e_two <= 3e-7, e_two                               # the level of a plain fp32 GEMM
    assert e_two <= max(3.0 * e_f32, 2.5e-7)
    if K >= 256:
        assert e_one >= 1.8 * e_two, (e_one, e_two)           # one shared accumulator
