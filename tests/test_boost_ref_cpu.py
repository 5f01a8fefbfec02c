"""tests/boost_ref.py pinned without a device: node sums and leaf values against brute force with Fractions, gradients
against the oracle, the exp ambiguity detector, the quantisers against tests/util.py, and the row samplers against the
oracle's."""
from fractions import Fraction

import numpy as np
import pytest

import ydf_b200
from oracle import oracle as O
from tests import boost_ref as R
from tests.util import quantize_q24, quantize_second

F32 = np.float32


def small_tree():
    """root: feature 0 >= 3; its negative child: feature 1 in {1, 4}; leaves elsewhere."""
    t = np.zeros(5, ydf_b200.NODE_DTYPE)
    t["feature"] = [0, 1, -1, -1, -1]
    t["threshold_bin"] = [3, 0, 0, 0, 0]
    t["condition_type"] = [0, 1, 0, 0, 0]
    t["cat_mask"][1, 0] = (1 << 1) | (1 << 4)
    t["neg_child"] = [1, 2, -1, -1, -1]
    t["pos_child"] = [4, 3, -1, -1, -1]
    return t


def brute_node(rows, g, h, sel, P, V):
    """Fractions, one row at a time: sum_g, sum of squares and sum of hessians of the node's selected rows, as the
    quantised values the kernels add up."""
    sg = sg2 = sh = Fraction(0)
    n = 0
    for r in rows:
        if not sel[r]:
            continue
        n += 1
        sg += Fraction(int(np.rint(float(g[r]) * 2 ** 30 / P))) * Fraction(P) / 2 ** 30
        sq = float(F32(g[r]) * F32(g[r]))
        sg2 += Fraction(min(int(np.rint(sq * 2 ** 31 / (P * P))), 2 ** 31)) * Fraction(P * P) / 2 ** 31
        sh += Fraction(min(int(np.rint(float(h[r]) * 2 ** 31 / V)), 2 ** 31)) * Fraction(V) / 2 ** 31
    return n, sg, sg2, sh


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_node_sums_and_leaves_match_brute_force(seed):
    rng = np.random.default_rng(seed)
    n = 300
    cols = [("num", rng.integers(0, 6, n).astype(np.uint8), 6, None), ("cat", rng.integers(0, 6, n).astype(np.uint8), 6, None)]
    tree = small_tree()
    g = rng.uniform(-0.9, 0.9, n).astype(F32)
    h = rng.uniform(0.0, 0.25, n).astype(F32)
    sel = rng.random(n) < 0.7
    rows_of = R.route(tree, cols)
    assert sorted(np.concatenate([rows_of[i] for i in (2, 3, 4)]).tolist()) == list(range(n))
    rows = R.Rows(g, h, sel, 1.0, 0.25)
    cfg = ydf_b200.default_config(shrinkage=0.1, l1_regularization=0.05, l2_regularization=0.5, clamp_leaf_logit=5.0,
                             use_hessian_gain=1)
    for i in range(len(tree)):
        s = rows.sums(rows_of[i])
        m, sg, sg2, sh = brute_node(rows_of[i], g, h, sel, 1.0, 0.25)
        assert s["n"] == m
        stat, sum_h = R.expected_stats(s, rows, cfg, logit=True)
        assert stat[0][0] == stat[0][1] == float(sg)
        assert sum_h[0] == float(sh)
        assert Fraction(s["sg2"][0]) / 2 ** 31 == sg2
        # the leaf: shrinkage * l1(sum_g) / (max(sum_h, 1e-3) + l2), rounded once to float (the double quotient is within
        # an ulp of the exact one, far below a float's half ulp except on a midpoint)
        num = max(Fraction(0), abs(sg) - Fraction(float(F32(0.05))))
        num = num if sg > 0 else -num
        exact = Fraction(float(F32(0.1))) * num / (max(sh, Fraction(1, 1000)) + Fraction(float(F32(0.5))))
        assert abs(float(R.leaf_value(float(sg), float(sh), cfg, True)) - float(exact)) <= R.ulp32(float(exact)) / 2


def test_exact_scores_restate_the_kernels_in_fractions():
    # variance: d = (sp nn - sn np) P / 2^30; weighted: weight sums for the counts
    assert R.split_score_variance(3 * 2 ** 30, -2 ** 30, 4, 4, 1.0) == Fraction(16 * 16, 4 * 4 * 64)
    assert R.split_score_variance(2 ** 30, 2 ** 30, 5, 5, 2.0) == 0
    w = 2 ** 30   # weight 0.5 at w_pow2 = 1
    assert R.split_score_weighted(2 ** 30, 2 ** 30, w, w, 1.0, 1.0) == 0
    assert R.split_score_weighted(2 ** 30, 0, w, w, 1.0, 1.0) == 1   # d = 1 * 0.5, d^2 / (0.5 * 0.5 * 1^2)
    assert R.split_score_weighted(2 ** 30, 0, 0, w, 1.0, 1.0) is None


def test_gradients_match_the_oracle_within_one_ulp():
    rng = np.random.default_rng(3)
    n = 20000
    pred = rng.normal(scale=3.0, size=n).astype(F32)
    labels = rng.integers(1, 3, n).astype(np.int32)
    g, h, _ = R.binomial_gradients(pred, labels == 2)
    og, oh = O.update_gradients(O.LOSS_BINOMIAL, labels, pred)
    # glibc's expf and the double exp rounded once may differ by an ulp; h = p (1 - p) carries p's ulp twice
    for a, b, ulps in ((g, og, 1), (h, oh, 2)):
        assert np.all(np.abs(a.astype(np.float64) - b) <= ulps * np.spacing(np.abs(b).astype(F32)).astype(np.float64))
    y = rng.normal(scale=100, size=n).astype(F32)
    g, h, _ = R.squared_error_gradients(pred, y)
    og, oh = O.update_gradients(1, y, pred)
    assert np.array_equal(g, og) and np.array_equal(h, oh)
    K = 5
    mp = rng.normal(scale=2.0, size=(K, n)).astype(F32)
    ml = rng.integers(1, K + 1, n).astype(np.int32)
    g, h, _ = R.mc_gradients(mp, ml - 1)
    og, oh = O.mc_update_gradients(ml, K, np.ascontiguousarray(mp.T))
    # the oracle rounds e * norm before the subtraction, the device does not (FFMA), and glibc's expf may differ from
    # the double exp by an ulp: the difference is an ulp or two of the terms (<= 1), whatever the cancellation
    for a, b in ((g, og), (h, oh)):
        assert np.abs(a.astype(np.float64) - b).max() <= 2 * float(np.spacing(F32(1)))


def test_single_rounding_of_the_contracted_difference():
    rng = np.random.default_rng(4)
    e = rng.uniform(0, 1, 5000).astype(F32)
    m = rng.uniform(0, 1, 5000).astype(F32)
    ind = (rng.random(5000) < 0.5).astype(np.float64)
    got = R.sub_round_f32(ind, e.astype(np.float64) * m.astype(np.float64))
    for i in range(5000):
        exact = Fraction(float(ind[i])) - Fraction(float(e[i])) * Fraction(float(m[i]))
        f = F32(float(exact))   # float(Fraction) rounds once to double; check against both float neighbours
        cands = [f, np.nextafter(f, F32(np.inf)), np.nextafter(f, F32(-np.inf))]
        best = min(cands, key=lambda c: (abs(Fraction(float(c)) - exact), int(np.float32(c).view(np.uint32)) & 1))
        assert got[i] == best, (i, got[i], best)
    # a double result exactly on a float midpoint, with the exact value just above it: rounds up, not to even
    a, b = 1.0, 2.0 ** -25 - 2.0 ** -60
    assert R.sub_round_f32(np.array([a]), np.array([b]))[0] == F32(1.0)
    assert R.sub_round_f32(np.array([a]), np.array([2.0 ** -25 + 2.0 ** -60]))[0] == np.nextafter(F32(1), F32(0))


def test_ambiguity_detector_on_midpoints():
    f = F32(1.5)
    up = np.nextafter(f, F32(2))
    mid = (float(f) + float(up)) / 2
    e = np.array([mid, np.nextafter(mid, 2.0), np.nextafter(mid, 0.0), mid + 3 * np.spacing(mid), float(f),
                  mid + 100 * np.spacing(mid)])
    val, alt, amb = R.f32_candidates(e)
    assert amb.tolist() == [True, True, True, True, False, False]
    assert {float(val[0]), float(alt[0])} == {float(f), float(up)}
    assert val[4] == alt[4] == f
    # random inputs: ambiguous rows are rare
    x = np.random.default_rng(5).normal(size=100000).astype(F32)
    assert R.exp_f32(x)[2].sum() <= 2


def test_quantisers_match_tests_util():
    rng = np.random.default_rng(6)
    P = 4.0
    g = rng.uniform(-P, P, 10000).astype(F32)
    g[:2] = [0.0, -P]
    # quant_stat_signed at 2^7 P is the 24-bit code without its bias (the 24-bit code clamps at 2^24 - 1, below P)
    g = g[np.abs(g) < np.float32(P - P / 2 ** 23)]
    assert np.array_equal(R.quant_signed(g, 128 * P), quantize_q24(g, P) - 2 ** 23)
    v = rng.uniform(0, 0.25, 10000).astype(F32)
    v[:2] = [0.0, 0.25]
    assert np.array_equal(R.quant_unsigned(v, 128 * 0.25), quantize_second(v, 0.25))
    assert R.quant_unsigned(np.array([0.25], F32), 0.25)[0] == 2 ** 31
    assert R.quant_signed(np.array([P, -P], F32), P).tolist() == [2 ** 30, -2 ** 30]
    assert R.pow2_cover(0.0) == 1.0 and R.pow2_cover(0.25) == 0.25 and R.pow2_cover(0.3) == 0.5


def test_subsample_matches_the_oracle_sampler():
    from tests.util import synth
    n = 6000
    bins, nb, na, y = synth(n, 4, seed=3, bins=16)
    ref = O.gbt_train(bins, nb, na, y, O.default_config(num_trees=3, max_depth=3, subsample=0.5), 3)
    rng = O.Rng(123456)
    for t in range(3):
        assert int(ref["trees"][t][0]["num_examples"]) == int(R.subsample_mask(rng, n, 0.5).sum())


@pytest.mark.parametrize("alpha,beta", [(0.2, 0.1), (0.3, 0.15), (0.0, 0.5)])
def test_goss_selection_matches_the_oracle_sampler(alpha, beta):
    rng = np.random.default_rng(7)
    g = np.round(rng.normal(size=5000), 2).astype(F32)   # ties in |g|
    O.set_goss_stable_sort(True)
    try:
        ids, w = O.goss_sample(g, alpha, beta, O.Rng(99))
    finally:
        O.set_goss_stable_sort(False)
    sel, ww = R.goss_selection(g, alpha, beta, O.Rng(99))
    assert sorted(ids.tolist()) == np.flatnonzero(sel).tolist()
    assert np.array_equal(ww[sel], w[sel])
    assert (ww[~sel] == 1).all()
