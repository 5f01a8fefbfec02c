"""Numpy CART reference of one node of a categorical feature with any number of categories (DESIGN.md §21), and
helpers shared by the wide categorical tests.

The rule is the byte scan's (scan_node_categorical) written out: per category the key (label mean, or the float
hessian priority with l2_categorical), categories sorted ascending by (key, index), every boundary between sorted
positions scored, the first maximum kept; the categories after it form the positive set."""
import numpy as np

from tests.scan_ref import MIN_HESSIAN, prescreen as scores  # noqa: F401 (the scores are the scan reference's)


def keys(cnt, s, h, use_hessian, l2_categorical=1.0, weight=None):
    cnt, s, h = (np.asarray(a, np.float64) for a in (cnt, s, h))
    if not use_hessian:
        den = cnt if weight is None else np.asarray(weight, np.float64)   # a weighted mean: the weight sum
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where((cnt > 0) & (den != 0), s / np.where(den != 0, den, 1), 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        k = (s / (h + l2_categorical)).astype(np.float32).astype(np.float64)
    return np.where(h > 0, k, 0.0)


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
