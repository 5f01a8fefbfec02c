"""Exact reference of the split scan (k_scan, k_scan_wide, k_scan_wide_cat, k_presort_*) and of the selection.

Everything starts from integers: per-row gradient codes (tests/util.quantize_q24, unbiased) and second-plane codes
(quantize_second) with the tree's scales, summed per bucket in int64.  A node's buckets, in scan order (bucket order for a
numerical column, ascending (key, category) for a categorical one, distinct values for a presorted one), are scored at
every boundary:

- variance gain, unweighted: d = S_pos*n_neg - S_neg*n_pos as a Python int and score = d^2 ginv^2 / (n_pos n_neg c0^2)
  as a Fraction; the candidates are pre-screened in float64 and only those near the top are decided exactly.
- hessian gain: the engine's double formula (splitter_accumulator.h's Score) in float64; its rounding is the
  reference's own kind of noise, so choices inside a band of BAND times the magnitude of the terms are left free.

A verdict lists the boundaries a correct scan may choose (one, unless exact scores tie within BAND) and whether a split
must, must not, or may be found."""
from fractions import Fraction

import numpy as np

MIN_HESSIAN = 0.001   # kMinHessianForNewtonStep
BAND = 2.0 ** -45


def mid_threshold(a, b) -> np.float32:
    """MidThreshold (learner/decision_tree/utils.h:103-109) in float32."""
    a, b = np.float32(a), np.float32(b)
    t = np.float32(a + np.float32((b - a) / np.float32(2)))
    return b if t <= a else t


def l1_threshold(v, l1):
    if l1 == 0:
        return v
    return np.sign(v) * np.maximum(0.0, np.abs(v) - l1)


def prescreen(cnt, s, h, order, use_hessian, min_obs=1, l2=1.0, weight=None, subtract_parent=False, l1=0.0):
    """float64 scores of the boundaries after sorted positions 0..B-2 (-1 where not valid) and the positive counts.
    `weight`: per-bucket weight sums, which take the place of the counts in the variance score (the counts keep deciding
    min_obs).  subtract_parent: the hessian score less the parent's term; else the parent's term is the minimum score."""
    c = np.asarray(cnt, np.float64)[order]
    cs = np.cumsum(c)
    ws = None if weight is None else np.cumsum(np.asarray(weight, np.float64)[order])
    ss = np.cumsum(np.asarray(s, np.float64)[order])
    hs = np.cumsum(np.asarray(h, np.float64)[order])
    tc, ts, th = cs[-1], ss[-1], hs[-1]
    nn, npos = cs[:-1], tc - cs[:-1]
    valid = (nn >= min_obs) & (npos >= min_obs)
    with np.errstate(invalid="ignore", divide="ignore"):
        if not use_hessian:
            c0, wn, wp = (tc, nn, npos) if ws is None else (ws[-1], ws[:-1], ws[-1] - ws[:-1])
            valid &= (wn > 0) & (wp > 0)
            d = (ts - ss[:-1]) * wn - ss[:-1] * wp
            sc = (d / wp) * (d / wn) / (c0 * c0)
            valid &= sc > 0
        else:
            g0 = l1_threshold(ts, l1)
            parent = g0 * g0 / (max(th, MIN_HESSIAN) + l2)
            gn, gp = l1_threshold(ss[:-1], l1), l1_threshold(ts - ss[:-1], l1)
            hn = np.maximum(hs[:-1], MIN_HESSIAN) + l2
            hp = np.maximum(th - hs[:-1], MIN_HESSIAN) + l2
            sc = gp * gp / hp + gn * gn / hn - (parent if subtract_parent else 0.0)
            valid &= sc > (0.0 if subtract_parent else parent)
    return np.where(valid, sc, -1.0), npos


class Verdict:
    """found: True (a split must be found), False (none may be), None (either).  accept: the boundaries (sorted
    positions) a correct scan may choose; first: the first exact maximum; exact: its exact score (Fraction, unweighted
    variance gain only); n_pos: the positive count at every boundary."""

    def __init__(self, found, accept, first, exact, n_pos):
        self.found, self.accept, self.first, self.exact, self.n_pos = found, accept, first, exact, n_pos


def verdict(cnt, s, h, *, use_hessian, min_obs=1, l1=0.0, l2=0.0, subtract_parent=False, ginv=1.0, hinv=1.0, w=None,
            w_inv=None):
    """Scan of one node's buckets, already in scan order: cnt row counts, s unbiased gradient-code sums, h second-plane
    code sums (int arrays); ginv / hinv the units of one code (P / 2^23, V / 2^24).  Boundaries 0..len-2.
    `w` (variance gain with example weights): per-bucket weight-code sums in units of w_inv; they take the place of the
    counts in the score, and |d| at or below the engine's floor of half a unit per row counts as 0 (boundaries within
    BAND of that floor are free)."""
    cnt = [int(x) for x in cnt]
    s = [int(x) for x in s]
    h = [int(x) for x in h]
    B = len(cnt)
    cs, ss, hs = np.cumsum(cnt, dtype=object), np.cumsum(s, dtype=object), np.cumsum(h, dtype=object)
    tc, ts, th = int(cs[-1]), int(ss[-1]), int(hs[-1])
    n_pos = [tc - int(cs[b]) for b in range(B - 1)]
    valid = [cs[b] >= min_obs and n_pos[b] >= min_obs for b in range(B - 1)]
    if not use_hessian:
        ws = cs if w is None else np.cumsum([int(x) for x in w], dtype=object)
        tw = int(ws[-1])
        wn = [int(ws[b]) for b in range(B - 1)]
        wp = [tw - x for x in wn]
        valid = [valid[b] and wn[b] > 0 and wp[b] > 0 for b in range(B - 1)]
        d = [(ts - int(ss[b])) * wn[b] - int(ss[b]) * wp[b] if valid[b] else 0 for b in range(B - 1)]
        strict = maybe = [b for b in range(B - 1) if valid[b] and d[b] != 0]
        if w is not None:   # boundary_score's floor, in units of the weight codes times w_inv
            floor = {b: 0.5 * (n_pos[b] * wn[b] * w_inv + int(cs[b]) * wp[b] * w_inv +
                               (abs(ts - int(ss[b])) * int(cs[b]) + abs(int(ss[b])) * n_pos[b]) * w_inv) for b in maybe}
            strict = [b for b in maybe if abs(d[b]) * w_inv > floor[b] * (1 + BAND)]
            maybe = [b for b in maybe if abs(d[b]) * w_inv > floor[b] * (1 - BAND)]
        if not maybe:
            return Verdict(False, [], None, None, n_pos)
        approx = {b: float(d[b]) ** 2 / (float(wp[b]) * float(wn[b])) for b in maybe}
        top = max(approx.values())
        near = [b for b in maybe if approx[b] >= top * (1 - 1e-9)]
        exact = {b: Fraction(d[b] * d[b], wp[b] * wn[b]) for b in near}
        best = max(exact.values())
        first = min(b for b in near if exact[b] == best)
        # (an exact tie is no license: the first maximum is the answer; only near-ties are free)
        accept = [b for b in near if exact[b] >= best * (1 - Fraction(BAND)) and (exact[b] != best or b == first)]
        scale = Fraction(ginv) ** 2 / Fraction(tw) ** 2
        if w is not None:   # the weight sums in real units: w codes times w_inv
            scale /= Fraction(w_inv) ** 2
        return Verdict(True if strict else None, accept, first, best * scale, n_pos)
    g = lambda v: l1_threshold(float(v) * ginv, l1)   # noqa: E731 (exact products: ginv is a power of two)
    g0 = g(ts)
    parent = g0 * g0 / (max(th * hinv, MIN_HESSIAN) + l2)
    min_score = 0.0 if subtract_parent else parent
    sc, mag = {}, {}
    for b in range(B - 1):
        if not valid[b]:
            continue
        gn, gp = g(int(ss[b])), g(ts - int(ss[b]))
        hn = max(int(hs[b]) * hinv, MIN_HESSIAN) + l2
        hp = max((th - int(hs[b])) * hinv, MIN_HESSIAN) + l2
        sc[b] = gp * gp / hp + gn * gn / hn - (parent if subtract_parent else 0.0)
        mag[b] = gp * gp / hp + gn * gn / hn + parent
    if not sc:
        return Verdict(False, [], None, None, n_pos)
    band = BAND * max(mag.values())
    strict = [b for b in sc if sc[b] > min_score + band]
    maybe = [b for b in sc if sc[b] > min_score - band]
    if not maybe:
        return Verdict(False, [], None, None, n_pos)
    best = max(sc[b] for b in maybe)
    accept = [b for b in maybe if sc[b] >= best - band]
    first = min(b for b in maybe if sc[b] == best)
    return Verdict(True if strict else None, accept, first, None, n_pos)


def bucket_sums(codes, rows, q, hq, num_bins):
    """(count, unbiased gradient-code sum, second-plane sum) per bucket of the node's rows (codes[rows]), int64."""
    c = np.asarray(codes)[rows].astype(np.int64)
    cnt = np.bincount(c, minlength=num_bins)
    s = np.bincount(c, weights=q[rows] - 2 ** 23, minlength=num_bins)
    h = np.bincount(c, weights=hq[rows], minlength=num_bins)
    assert (len(rows) + 1) * 2 ** 24 < 2 ** 53   # float64 sums of integers stay exact
    return cnt, s.astype(np.int64), h.astype(np.int64)


def numerical_expect(cnt, b, B, values=None, wide=False):
    """Threshold of a numerical split at boundary b (bucket interpolation, splitter_scanner.h:993-1000, and the exact
    rule with bucket `values`): -> (threshold_bin, lo, hi, threshold_value)."""
    nz = np.flatnonzero(np.asarray(cnt)[b + 1:B] > 0)
    hi = int(b + 1 + nz[0]) if len(nz) else None
    if values is None:
        idx = b
        if hi is not None and hi <= B - 2 and hi != b + 1:
            idx = (b + hi) // 2
        return idx + 1, -1, -1, np.float32(np.nan)
    t = mid_threshold(values[b], values[hi])
    k = b + 1
    while k < hi and values[k] < t:
        k += 1
    return (k, -1, -1, t) if wide else (k, b, hi, t)


def category_keys(cnt, s, h, use_hessian, ginv, hinv, l1=0.0, l2_categorical=1.0, w_inv=None):
    """category_key in float64: the label mean (with example weights, `h` holds the weight codes and the mean is over
    their sum h * w_inv), or the float32 hessian priority; 0 for an empty bucket.  Every step is one correctly rounded
    operation, so numpy reproduces the device's keys bit for bit."""
    cnt = np.asarray(cnt, np.int64)
    sg = np.asarray(s, np.float64) * ginv
    with np.errstate(invalid="ignore", divide="ignore"):
        if not use_hessian:
            den = cnt.astype(np.float64) if w_inv is None else np.asarray(h, np.float64) * w_inv
            return np.where((cnt > 0) & (den != 0), sg / np.where(den != 0, den, 1.0), 0.0)
        H = np.asarray(h, np.float64) * hinv
        k = (l1_threshold(sg, l1) / (H + l2_categorical)).astype(np.float32).astype(np.float64)
    return np.where(H > 0, k, 0.0)


def category_order(keys):
    """Ascending (key, category index); -0.0 == +0.0."""
    return np.lexsort((np.arange(len(keys)), keys))
