"""Float64 numpy statement of the warped sampled level (ops.SidPrefixIndex.sample_select_warped[_wide]): the sampled search's
draw at a temperature T and within a top-p nucleus, scored by the model's own log-probability.

Per beam row x [K] of the head's logits and its Exp(1) noise q [K]:
  1. p_T = exp((x - max x) / T) / sum exp((x - max x) / T);
  2. N = {c : p_T[c] >= t}, t the largest p_T with sum_{p_T >= t} p_T >= top_p * sum p_T (ties at t all in; top_p = 1: all);
  3. N+ = the codes of N with p_T > 0; the beam draws the n = min(nc, |N+|) largest p_T / q over N+ (equal ratios by ascending
     code); the other nc - n slots are fillers: the codes outside N+ in ascending order, scored -inf;
  4. a drawn code scores (x[c] - lse) + the parent's log-probability, lse = max x + log sum exp(x - max x); -inf when the
     extended prefix is invalid for the history; the k best are kept, equal scores by ascending candidate index.
The kernel evaluates p_T in fp32, so a p_T below fp32's smallest subnormal is 0 there: the oracle flushes it too.  Where a
result rests on a comparison that fp32 rounding could flip (two ratios or two masses within `tol` of each other, a p_T at
the underflow edge), the row is reported ambiguous rather than decided."""
import numpy as np

FP32_TINY = 2.0 ** -149                                      # smallest positive fp32: p_T below half of it rounds to 0


def tempered(x, T):
    """float64 [R, K]: p_T of rows x (rule 1), flushed to 0 where fp32 underflows; bad rows (NaN, +inf, all -inf) are NaN."""
    x = np.asarray(x, dtype=np.float64)
    m = x.max(1, keepdims=True)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        e = np.exp((x - m) / T)
        p = e / e.sum(1, keepdims=True)
    p[(p < FP32_TINY / 2) & ~np.isnan(p)] = 0.0
    return p


def bad_rows(x):
    """bool [R]: rows holding a NaN or +inf, or all -inf (counted, drawn as fillers only)."""
    x = np.asarray(x, dtype=np.float64)
    return np.isnan(x).any(1) | np.isposinf(x).any(1) | np.isneginf(x).all(1)


def nucleus(p, top_p, tol=0.0):
    """(N bool [K], ambiguous bool) of one row of p_T (rule 2).  Ambiguous: the mass at or above t, or strictly above it, is
    within tol of the target, or the next smaller p_T is within relative tol of t (fp32 could tie or split them)."""
    K = p.shape[0]
    if top_p >= 1:
        return np.ones(K, dtype=bool), False
    order = np.argsort(-p, kind="stable")
    ps = p[order]
    cum = np.cumsum(ps)
    last = np.searchsorted(-ps, -ps, side="right") - 1         # end of each run of equal values (ties count together)
    mass = cum[last]
    target = top_p * cum[-1]
    j = int(np.argmax(mass >= target))                       # the largest value whose mass reaches the target
    t = ps[j]
    first = int(np.searchsorted(-ps, -t, side="left"))
    above = cum[first - 1] if first > 0 else 0.0               # the mass strictly above t
    nxt = ps[last[j] + 1] if last[j] + 1 < K else -1.0
    amb = bool(abs(mass[j] - target) <= tol or abs(above - target) <= tol or (nxt > 0 and t - nxt <= tol * t))
    return p >= t, amb


def draw(p, q, top_p, nc, tol=0.0):
    """(samples int64 [nc], drawn bool [nc], ambiguous bool) of one row (rules 2-3)."""
    N, amb = nucleus(p, top_p, tol)
    ok = N & (p > 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(ok, p / np.asarray(q, dtype=np.float64), -1.0)
    drawable = np.nonzero(ok)[0]
    order = drawable[np.argsort(-ratio[drawable], kind="stable")]
    n = min(nc, len(order))
    fillers = np.nonzero(~ok)[0][:nc - n]
    samples = np.concatenate([order[:n], fillers]).astype(np.int64)
    if tol > 0:
        r = ratio[order[:n + 1]]
        amb |= bool((np.abs(np.diff(r)) <= tol * np.abs(r[:-1])).any())
        amb |= bool(n > 0 and (p[order[:n]] < 2.0 ** -100).any())   # fp32 subnormal p_T: few significant bits
        amb |= bool(n < nc and (N & (p > FP32_TINY / 8) & (p < FP32_TINY * 8)).any())   # at the underflow edge
    return samples, np.arange(nc) < n, amb


def warped_level(logits, noise, T, top_p, nc, tol=0.0):
    """Rules 1-3 and the model log-probabilities over rows [R, K]: (samples int64 [R, nc], samp_log_p float64 [R, nc] (-inf for
    fillers and bad rows), ambiguous bool [R], bad bool [R])."""
    x = np.asarray(logits, dtype=np.float64)
    R, K = x.shape
    bad = bad_rows(x)
    p = tempered(x, T)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        m = x.max(1, keepdims=True)
        lse = m + np.log(np.exp(x - m).sum(1, keepdims=True))
    samples = np.zeros((R, nc), dtype=np.int64)
    lp = np.full((R, nc), -np.inf)
    amb = np.zeros(R, dtype=bool)
    for r in range(R):
        if bad[r]:
            samples[r] = np.arange(nc)
            continue
        s, drawn, amb[r] = draw(p[r], noise[r], top_p, nc, tol)
        samples[r] = s
        lp[r, drawn] = x[r, s[drawn]] - lse[r, 0]
    return samples, lp, amb, bad


def keep_best(samples, samp_log_p, generated, log_probas, k, valid, dtype=np.float64):
    """Rule 4's selection from given draws: scores [B, kp * nc] = samp_log_p + the parent's (in `dtype`: float32 restates the
    kernel's own rounding), -inf where valid(b, prefix) is False; the k best by a stable descending sort.  Returns (generated
    [B, k, h + 1], log_probas [B, k], parent_global [B, k])."""
    samples = np.asarray(samples)
    rows, nc = samples.shape
    B = rows if generated is None else generated.shape[0]
    kp = rows // B
    h = 0 if generated is None else generated.shape[2]
    scores = np.full((B, kp * nc), -np.inf, dtype=dtype)
    for b in range(B):
        for beam in range(kp):
            prefix = [] if generated is None else [int(v) for v in generated[b, beam]]
            plp = dtype(0) if log_probas is None else dtype(log_probas[b, beam])
            for r in range(nc):
                lp = dtype(samp_log_p[b * kp + beam, r])
                tok = int(samples[b * kp + beam, r])
                if lp > -np.inf and valid(b, prefix + [tok]):
                    scores[b, beam * nc + r] = lp + plp
    idx = np.argsort(-scores, axis=1, kind="stable")[:, :k]
    parent = idx // nc
    new = np.take_along_axis(samples.reshape(B, kp * nc), idx, 1)[:, :, None]
    if h:
        gen = np.concatenate([np.take_along_axis(generated, parent[:, :, None].repeat(h, 2), 1), new], axis=2)
    else:
        gen = new
    return gen, np.take_along_axis(scores, idx, 1), parent + np.arange(B)[:, None] * kp
