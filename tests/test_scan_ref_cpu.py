"""The exact scan reference (tests/scan_ref.py) against brute force over the rows, the failure of a double-precision
variance numerator on large pure nodes, and the refusals of the candidate-capture seam without a device."""
import ctypes as C
import itertools
from fractions import Fraction

import numpy as np
import pytest

import ydf_b200
from tests import scan_ref as S


def exact_variance_gain(codes, pos):
    """Between-group sum of squares over the node's count, exact: (mean_pos - mean_neg)^2 n_pos n_neg / c0^2."""
    sp, sn = sum(int(x) for x in codes[pos]), sum(int(x) for x in codes[~pos])
    np_, nn = int(pos.sum()), int((~pos).sum())
    c0 = np_ + nn
    return (Fraction(sp, np_) - Fraction(sn, nn)) ** 2 * np_ * nn / (c0 * c0)


@pytest.mark.parametrize("seed", range(12))
def test_numerical_verdict_matches_brute_force_over_rows(seed):
    rng = np.random.default_rng(seed)
    B = int(rng.choice([2, 3, 7, 30]))
    n = int(rng.integers(5, 400))
    bins = rng.integers(0, B, size=n)
    bins[bins == B // 2] = 0                       # an empty bucket in the middle
    codes = rng.integers(-50, 50, size=n) * (1 if seed % 3 else 0) + (7 if seed % 4 == 0 else 0)
    min_obs = int(rng.choice([1, 5]))
    cnt = np.bincount(bins, minlength=B)
    s = np.bincount(bins, weights=codes, minlength=B).astype(np.int64)
    v = S.verdict(cnt, s, cnt, use_hessian=False, min_obs=min_obs)
    best, first = Fraction(0), None
    for t in range(1, B):
        pos = bins >= t
        if pos.sum() < min_obs or (~pos).sum() < min_obs:
            continue
        sc = exact_variance_gain(codes, pos)
        if sc > best:
            best, first = sc, t - 1
    assert v.found == (first is not None)
    if first is not None:
        assert v.first == first and v.exact == best
        assert v.n_pos[first] == int((bins > first).sum())


@pytest.mark.parametrize("seed", range(8))
def test_categorical_verdict_is_the_best_subset(seed):
    """Sorting categories by mean and scanning finds the best of all two-way partitions (variance gain, Breiman)."""
    rng = np.random.default_rng(100 + seed)
    B = int(rng.choice([3, 4, 6]))
    n = int(rng.integers(20, 300))
    cats = rng.integers(0, B, size=n)
    codes = rng.integers(-30, 30, size=n) + cats * int(rng.integers(-5, 5))
    cnt = np.bincount(cats, minlength=B)
    s = np.bincount(cats, weights=codes, minlength=B).astype(np.int64)
    order = S.category_order(S.category_keys(cnt, s, cnt, False, 1.0, 1.0))
    v = S.verdict(cnt[order], s[order], cnt[order], use_hessian=False)
    best = Fraction(0)
    for r in range(1, B):
        for pos_set in itertools.combinations(range(B), r):
            pos = np.isin(cats, pos_set)
            if 0 < pos.sum() < n:
                best = max(best, exact_variance_gain(codes, pos))
    assert (v.found is True) == (best > 0)
    if best > 0:
        assert v.exact == best


@pytest.mark.parametrize("subtract_parent", [False, True])
def test_hessian_verdict_matches_row_sums(subtract_parent):
    rng = np.random.default_rng(7)
    B, n = 20, 500
    bins = rng.integers(0, B, size=n)
    g = rng.integers(-2 ** 22, 2 ** 22, size=n)
    h = rng.integers(0, 2 ** 24, size=n)
    ginv, hinv, l2 = 2.0 ** -23, 0.25 * 2.0 ** -24, 1.5
    cnt = np.bincount(bins, minlength=B)
    s = np.bincount(bins, weights=g, minlength=B).astype(np.int64)
    hs = np.bincount(bins, weights=h, minlength=B).astype(np.int64)
    v = S.verdict(cnt, s, hs, use_hessian=True, l2=l2, subtract_parent=subtract_parent, ginv=ginv, hinv=hinv)
    G, H = g.sum() * ginv, h.sum() * hinv
    parent = G * G / (max(H, S.MIN_HESSIAN) + l2)
    scores = []
    for t in range(1, B):
        pos = bins >= t
        gp, gn = g[pos].sum() * ginv, g[~pos].sum() * ginv
        hp, hn = h[pos].sum() * hinv, h[~pos].sum() * hinv
        scores.append(gp * gp / (max(hp, S.MIN_HESSIAN) + l2) + gn * gn / (max(hn, S.MIN_HESSIAN) + l2) -
                      (parent if subtract_parent else 0.0))
    scores = np.array(scores)
    ok = scores > (0.0 if subtract_parent else parent)
    assert v.found == bool(ok.any())
    if ok.any():
        assert int(np.argmax(np.where(ok, scores, -np.inf))) in v.accept


def contracted_numerator(s_pos, n_neg, s_neg, n_pos):
    """dq as an FMA-contracted double expression computes it: fma(S_pos, n_neg, -round(S_neg * n_pos)).  The operands
    are integers below 2^53, so the exact product and one rounding of the sum give the FMA's result."""
    return float(s_pos * n_neg - int(float(s_neg * n_pos)))


def test_double_numerator_splits_a_large_pure_node():
    """A pure node of 300K rows (g = 0.7, P = 1): the exact numerator is 0 at every boundary and the reference finds no
    split, while the contracted double numerator leaves the rounding error of u n_pos n_neg > 2^53 at many boundaries:
    a score of ~1e-33 that a strict '> 0' accepts."""
    n, u = 300000, int(np.rint(np.float32(0.7) * np.float32(2.0 ** 23)))
    cuts = np.linspace(1, n - 1, 200).astype(np.int64)
    noisy = [c for c in cuts if contracted_numerator(u * (n - c), int(c), u * int(c), n - int(c)) != 0.0]
    assert len(noisy) > 20
    c = int(noisy[0])
    dq = contracted_numerator(u * (n - c), c, u * c, n - c)
    d = dq * 2.0 ** -23
    assert 0 < (d / (n - c)) * (d / c) / (float(n) * n) < 1e-30
    cnt = np.diff(np.concatenate([[0], cuts, [n]]))
    v = S.verdict(cnt, cnt * u, cnt, use_hessian=False)
    assert v.found is False


def test_capture_seam_refuses_without_handle():
    L = ydf_b200.lib()
    assert L.ygg_debug_capture_candidates(None, 1) == 1
    assert "null" in L.ygg_last_error().decode()
    n = C.c_int32()
    scales = (C.c_float * 3)()
    nodes = np.zeros(4, ydf_b200._capi.LEVEL_NODE_DTYPE)
    cands = np.zeros(4, ydf_b200._capi.CANDIDATE_DTYPE)
    assert L.ygg_debug_level_candidates(None, 0, 4, nodes.ctypes.data_as(C.c_void_p), cands.ctypes.data_as(C.c_void_p),
                                        None, 0, C.byref(n), scales) == 1
    assert "null" in L.ygg_last_error().decode()
