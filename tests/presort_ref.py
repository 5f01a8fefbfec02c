"""Numpy reference of the exact numerical splitter on one node (DESIGN.md §22), shared by the presorted column tests.

The node's rows are grouped by distinct value (missing values already replaced by the column mean), every boundary
between two consecutive distinct values is scored with the byte and wide scans' formulas (tests/scan_ref.prescreen
over the values in ascending order), and the first maximum wins.  The threshold is MidThreshold of the two values
around the cut (learner/decision_tree/utils.h:103-109) in float32."""
import numpy as np

from tests import scan_ref as S
from tests import wide_cat_ref as W


mid_threshold = S.mid_threshold


def best_split(values, g_units, h_units=None, use_hessian=False, min_obs=1, w_units=None, subtract_parent=False, l2=0.0):
    """-> (score, float32 threshold, n_pos) of the node's rows, or None when no boundary is a valid split.  `*_units`:
    per-row quantised values in the engine's units (their sums are exact)."""
    v = np.asarray(values, np.float32)
    distinct, inv = np.unique(v, return_inverse=True)   # (-0.0 == +0.0: one value)
    if len(distinct) < 2:
        return None
    cnt = np.bincount(inv, minlength=len(distinct)).astype(np.float64)
    s = np.bincount(inv, weights=g_units, minlength=len(distinct))
    h = np.bincount(inv, weights=h_units, minlength=len(distinct)) if use_hessian else cnt
    w = None if w_units is None else np.bincount(inv, weights=w_units, minlength=len(distinct))
    sc, npos = S.prescreen(cnt, s, h, np.arange(len(distinct)), use_hessian, min_obs, l2, w, subtract_parent)
    if sc.max() < 0:
        return None
    b = int(np.argmax(sc))   # the first maximum in ascending value order
    return float(sc[b]), mid_threshold(distinct[b], distinct[b + 1]), int(npos[b])


def brute_force(values, g, h=None, use_hessian=False, min_obs=1):
    """The same split by trying every threshold between two consecutive distinct values on the rows themselves (no
    grouping, no prefix sums): variance reduction of the row sums, or the hessian gain with the parent as minimum."""
    v = np.asarray(values, np.float32)
    g = np.asarray(g, np.float64)
    h = np.ones_like(g) if h is None else np.asarray(h, np.float64)
    distinct = np.unique(v)
    best = None
    for lo, hi in zip(distinct[:-1], distinct[1:]):
        t = mid_threshold(lo, hi)
        pos = v >= t
        n_pos, n_neg = int(pos.sum()), int((~pos).sum())
        if n_pos < min_obs or n_neg < min_obs:
            continue
        if use_hessian:
            gp, gn, hp, hn = g[pos].sum(), g[~pos].sum(), h[pos].sum(), h[~pos].sum()
            parent = g.sum() ** 2 / max(h.sum(), W.MIN_HESSIAN)
            score = gp * gp / max(hp, W.MIN_HESSIAN) + gn * gn / max(hn, W.MIN_HESSIAN)
            if not score > parent:
                continue
        else:
            score = np.var(g) - n_pos / len(g) * np.var(g[pos]) - n_neg / len(g) * np.var(g[~pos])
            if not score > 0:
                continue
        if best is None or score > best[0] * (1 + 1e-12):
            best = (float(score), t, n_pos)
    return best
