"""Numpy CART reference of one node of a categorical feature with any number of categories (DESIGN.md §21), and
helpers shared by the wide categorical tests.

The rule is the byte scan's (scan_node_categorical) written out: per category the key (label mean, or the float
hessian priority with l2_categorical), categories sorted ascending by (key, index), every boundary between sorted
positions scored, the first maximum kept; the categories after it form the positive set."""
import numpy as np

MIN_HESSIAN = 0.001   # kMinHessianForNewtonStep


def keys(cnt, s, h, use_hessian, l2_categorical=1.0, weight=None):
    cnt, s, h = (np.asarray(a, np.float64) for a in (cnt, s, h))
    if not use_hessian:
        den = cnt if weight is None else np.asarray(weight, np.float64)   # a weighted mean: the weight sum
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where((cnt > 0) & (den != 0), s / np.where(den != 0, den, 1), 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        k = (s / (h + l2_categorical)).astype(np.float32).astype(np.float64)
    return np.where(h > 0, k, 0.0)


def scores(cnt, s, h, order, use_hessian, min_obs=1, l2_categorical=1.0, weight=None, subtract_parent=False):
    """Scores of the boundaries after sorted positions 0..B-2 (-1 where not valid) and the positive counts.  `weight`:
    per-category weight sums, which take the place of the counts in the variance score (the counts keep deciding
    min_obs).  subtract_parent: the hessian score less the parent's term; else the parent's term is the minimum score
    (hessian_split_score_subtract_parent)."""
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
            parent = ts * ts / (max(th, MIN_HESSIAN) + l2_categorical)
            gn, gp = ss[:-1], ts - ss[:-1]
            hn = np.maximum(hs[:-1], MIN_HESSIAN) + l2_categorical
            hp = np.maximum(th - hs[:-1], MIN_HESSIAN) + l2_categorical
            sc = gp * gp / hp + gn * gn / hn - (parent if subtract_parent else 0.0)
            valid &= sc > (0.0 if subtract_parent else parent)
    return np.where(valid, sc, -1.0), npos


def best_split(cnt, s, h, use_hessian, min_obs=1, l2_categorical=1.0, weight=None, subtract_parent=False):
    """-> (score, sorted positive categories, n_pos) of the node, or None when no split is valid."""
    k = keys(cnt, s, h, use_hessian, l2_categorical, weight)
    order = np.lexsort((np.arange(len(k)), k))   # ascending key, then index; -0.0 == +0.0
    sc, npos = scores(cnt, s, h, order, use_hessian, min_obs, l2_categorical, weight, subtract_parent)
    if len(sc) == 0 or sc.max() < 0:
        return None
    b = int(np.argmax(sc))   # the first maximum
    return float(sc[b]), np.sort(order[b + 1:]), int(npos[b])


def set_of_words(words, num_bins):
    """Categories whose bit is set in uint32 words."""
    c = np.arange(num_bins)
    return c[((np.asarray(words, np.uint32)[c >> 5] >> (c & 31).astype(np.uint32)) & 1) != 0]


def zipf_codes(rng, n, num_bins, a=1.2, missing=0.05, na_bin=0):
    """Categories 0..num_bins-1 with Zipf(a) frequencies (category 1 the most frequent, 0 rare), missing rows folded
    into na_bin; -> (codes, missing mask)."""
    ranks = np.arange(1, num_bins, dtype=np.float64)
    p = ranks ** -a
    p /= p.sum()
    codes = (rng.choice(num_bins - 1, size=n, p=p) + 1).astype(np.uint16)
    codes[rng.random(n) < 0.002] = 0
    miss = rng.random(n) < missing
    codes[miss] = na_bin
    return codes, miss
