"""Every split candidate of every tree level against the exact scan reference (tests/scan_ref.py).

The level loop's candidate tables are captured (Gbt.capture_candidates) and, for every level node and every feature,
compared with the reference computed from the node's rows (found by routing every row through the emitted tree) and the
per-row integer codes at the tree's captured scales.  Rules:

- Unweighted variance gain: `found`, the boundary, threshold_bin, n_pos and the category mask match exactly, with "not
  found" exactly when no boundary has an exact score > 0.  Boundaries whose exact scores differ by less than 2^-45
  relative are interchangeable.  The float score is within 1 ulp of the exact score rounded to float.
- Hessian gain: within a band of 2^-45 times the magnitude of the terms (gp^2/hp + gn^2/hn + parent), `found` and the
  boundary are free; outside it they match exactly.
- Selection: a node splits on the first maximum of the float candidate scores in feature order, if it is > 0.
- k_node_stats: with the unweighted variance gain, every split's stored score is within 1 float ulp of the exact score
  from its children's 31-bit sums.
"""
from fractions import Fraction

import numpy as np
import pytest

import ydf_b200
from tests import scan_ref as S
from tests.boost_ref import route
from tests.util import quantize_q24, quantize_second

pytestmark = pytest.mark.gpu


def byte_cols(bins, num_bins, ftypes, bucket_values=None):
    """Column descriptions of byte columns: (kind, codes, buckets, bucket values or None)."""
    bucket_values = bucket_values or {}
    return [("cat" if ftypes[f] == 1 else "num", bins[f], int(num_bins[f]), bucket_values.get(f)) for f in range(len(bins))]


def ulp32(x):
    x = np.float32(abs(x))
    return float(np.nextafter(x, np.float32(np.inf)) - x)


def same_f32(a, b):
    a, b = np.float32(a), np.float32(b)
    return (np.isnan(a) and np.isnan(b)) or a == b


def check_scan(gbt, cfg, tree, cols, g, h, w=None, tree_index=-1, sel=None, select=None, hist_of=None):
    """Compares every captured candidate of the tree with the reference; -> number of (node, feature) pairs checked.
    `cols`: per feature (kind, codes or stored values, buckets, bucket values), kind 'num' / 'cat' (byte), 'wide_num' /
    'wide_cat' (uint16), 'pre' (presorted).  `w`: example weights (the rows then carry w*g in `g`).  `sel`: the rows the
    tree was trained on (subsample / GOSS; None: all).  `select(level, j, cap)`: the feature node j of the level must
    split on (-1: none), in place of the first maximum in feature order (candidate sampling).  `hist_of(level, cap,
    rows_of, q, hq)`: the level's bucket sums in one pass (tests/level_hist_ref.LevelHist), a function (j, f) -> (cnt,
    s, hs) or None (then, and without a provider, scan_ref.bucket_sums per node and feature)."""
    wide = list(getattr(gbt.dataset, "wide", {}))
    sets = gbt.get_category_sets(tree_index, tree) if any(c[0] == "wide_cat" for c in cols) else {}
    rows_of = route(tree, cols, sets)
    if sel is not None:
        rows_of = {i: r[sel[r]] for i, r in rows_of.items()}
    min_obs = cfg.min_examples if cfg.in_split_min_examples_check else 1
    use_h = bool(cfg.use_hessian_gain)
    checked, derived_seen = 0, 0
    for level in range(cfg.max_depth - 1):
        cap = gbt.level_candidates(level)
        P = cap["P"]
        ginv = P / 2.0 ** 23
        q = quantize_q24(g, P)
        w_inv = None
        if w is not None:
            w_inv = cap["w_pow2"] / 2.0 ** 24
            hq, hinv = quantize_second(w, cap["w_pow2"]), w_inv
        elif h is not None:
            V = cap["h_pow2"]
            hq, hinv = quantize_second(h, V), V / 2.0 ** 24
        else:
            hq, hinv = np.full(len(g), 2 ** 24, np.int64), cap["h_pow2"] / 2.0 ** 24
        if level == 0 or not cfg.sibling_subtraction:
            assert not cap["derived"].any(), f"level {level}: derived nodes"
        derived_seen += int(cap["derived"].sum())
        level_sums = hist_of(level, cap, rows_of, q, hq) if hist_of is not None else None
        for j in range(len(cap["node"])):
            pre = int(cap["node"][j])
            rows = rows_of[pre]
            assert len(rows) == cap["num_examples"][j], (level, j)
            if not cap["candidate"][j]:
                assert not cap["found"][j].any()
                continue
            for f, (kind, codes, B, values) in enumerate(cols):
                if kind == "pre":
                    distinct, inv = np.unique(codes[rows], return_inverse=True)   # -0.0 == +0.0: one value
                    B = len(distinct)
                    cnt, s, hs = S.bucket_sums(inv, np.arange(len(rows)), q[rows], hq[rows], B)
                else:
                    sums = level_sums(j, f) if level_sums is not None else None
                    cnt, s, hs = sums if sums is not None else S.bucket_sums(codes, rows, q, hq, B)
                cat = kind in ("cat", "wide_cat")
                l2 = cfg.l2_regularization_categorical if cat else cfg.l2_regularization
                order = np.arange(B)
                if cat:
                    order = S.category_order(S.category_keys(cnt, s, hs, use_h, ginv, hinv, cfg.l1_regularization, l2,
                                                             w_inv=w_inv))
                v = S.verdict(cnt[order], s[order], hs[order], use_hessian=use_h, min_obs=min_obs,
                              l1=cfg.l1_regularization, l2=l2, subtract_parent=bool(cfg.hessian_split_score_subtract_parent),
                              ginv=ginv, hinv=hinv, w=None if w is None else hs[order], w_inv=w_inv)
                found = bool(cap["found"][j, f])
                where = f"level {level} node {pre} feature {f} ({kind}, {B} buckets)"
                if v.found is not None:
                    assert found == v.found, f"{where}: found {found}, reference {v.found}"
                checked += 1
                if not found:
                    continue
                c = {k: int(cap[k][j, f]) for k in ("threshold_bin", "lo", "hi", "num_pos_examples")}
                match = []
                for b in v.accept:
                    if c["num_pos_examples"] != v.n_pos[b]:
                        continue
                    if cat:
                        want = np.zeros(max(8, (B + 31) // 32), np.uint32)
                        for k in order[b + 1:]:
                            want[k >> 5] |= np.uint32(1) << np.uint32(k & 31)
                        if kind == "cat":
                            ok = np.array_equal(want[:8], cap["cat_mask"][j, f])
                        else:
                            # (the captured row is as wide as the widest wide categorical column)
                            got = cap["sets"][j, wide.index(f)]
                            m = max(len(want), len(got))
                            ok = np.array_equal(np.pad(want, (0, m - len(want))), np.pad(got, (0, m - len(got))))
                        ok = ok and np.isnan(cap["threshold_value"][j, f])
                    else:
                        if kind == "pre":
                            want = (1, -1, -1, S.mid_threshold(distinct[b], distinct[b + 1]))
                        else:
                            want = S.numerical_expect(cnt, b, B, values, wide=kind == "wide_num")
                        ok = (c["threshold_bin"], c["lo"], c["hi"]) == want[:3] and \
                            same_f32(cap["threshold_value"][j, f], want[3])
                    if ok:
                        match.append(b)
                assert match, (f"{where}: thr {c['threshold_bin']} lo/hi {c['lo']}/{c['hi']} n_pos {c['num_pos_examples']} "
                               f"value {cap['threshold_value'][j, f]} is none of the reference's boundaries {v.accept} "
                               f"(first {v.first})")
                if v.exact is not None:
                    want = np.float32(float(v.exact))
                    got = float(cap["score"][j, f])
                    assert abs(got - float(want)) <= ulp32(want), f"{where}: score {got} vs exact {float(v.exact)}"
            # the selection: the first maximum of the float scores in feature order, if > 0
            if select is not None:
                want = select(level, j, cap)
            else:
                sc = np.where(cap["found"][j] != 0, cap["score"][j], 0.0).astype(np.float32)
                best = int(np.argmax(sc))
                want = best if sc[best] > 0 else -1
            assert tree[pre]["feature"] == want, f"level {level} node {pre}: selection"
    if cfg.sibling_subtraction and cfg.max_depth > 2 and (tree["depth"] >= 3).any():
        assert derived_seen > 0
    return checked


def node_stats_check(tree, rows_of, g, P):
    """Unweighted variance gain: every split's score within 1 float ulp of the exact score from the children's 31-bit
    sums (quant_stat_signed)."""
    t = np.clip(np.rint(np.asarray(g, np.float32) * np.float32(2.0 ** 30 / P)), -2 ** 30, 2 ** 30).astype(np.int64)
    for i in np.flatnonzero(tree["feature"] >= 0):
        rp, rn = rows_of[int(tree["pos_child"][i])], rows_of[int(tree["neg_child"][i])]
        sp, sn = int(t[rp].sum()), int(t[rn].sum())
        np_, nn = len(rp), len(rn)
        d = Fraction(sp * nn - sn * np_) * Fraction(P) / 2 ** 30
        exact = d * d / (np_ * nn * (np_ + nn) ** 2)
        want = np.float32(float(exact))
        assert abs(float(tree["split_score"][i]) - float(want)) <= ulp32(want), (i, tree["split_score"][i], float(exact))


def mixed_bins(rng, n, layout):
    """Byte columns: layout = list of (kind, B) with kind 'num' or 'cat'; skewed codes with empty buckets."""
    bins, nb, ft = [], [], []
    for kind, B in layout:
        if kind == "num":
            x = rng.normal(size=n)
            c = np.clip(((x + 3) / 6 * B).astype(np.int64), 0, B - 1)
            if B > 8:   # runs of empty buckets, and empty trailing buckets
                c = np.where((c % 7 == 3) | (c >= B - 3), np.maximum(c - 1, 0), c)
        else:
            p = 1.0 / np.arange(1, B + 1) ** 1.1
            if B > 4:
                p[rng.choice(B, size=B // 5, replace=False)] = 0.0
            p /= p.sum()
            c = rng.choice(B, size=n, p=p)
        bins.append(c.astype(np.uint8))
        nb.append(B)
        ft.append(1 if kind == "cat" else 0)
    return np.stack(bins), np.array(nb, np.int32), np.array(ft, np.int32)


LAYOUT = [("num", 255), ("cat", 3), ("num", 2), ("num", 3), ("cat", 256), ("num", 256), ("cat", 17), ("num", 40)]

CASES = {
    "variance": dict(loss=1),
    "variance_binomial": dict(loss=0),
    "variance_min40": dict(loss=1, min_examples=40),
    "variance_min5_no_in_split": dict(loss=1, min_examples=5, in_split_min_examples_check=0),
    "variance_min1_no_sibling": dict(loss=1, min_examples=1, sibling_subtraction=0),
    "variance_depth2": dict(loss=1, max_depth=2),
    "hessian": dict(loss=0, use_hessian_gain=1),
    "hessian_subtract_parent": dict(loss=0, use_hessian_gain=1, hessian_split_score_subtract_parent=1),
    "hessian_l1_l2": dict(loss=0, use_hessian_gain=1, l1_regularization=0.5, l2_regularization=2.0,
                          l2_regularization_categorical=3.0),
    "hessian_squared_error_l2": dict(loss=1, use_hessian_gain=1, l2_regularization=1.0),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_every_candidate_matches_the_exact_scan(case):
    kw = dict(CASES[case])
    rng = np.random.default_rng(sorted(CASES).index(case) + 11)
    n = 60000
    bins, nb, ft = mixed_bins(rng, n, LAYOUT)
    ds = ydf_b200.Dataset(bins, nb, np.zeros(len(nb), np.int32), feature_types=ft)
    cfg = ydf_b200.default_config(**{"max_depth": 8, **kw})
    gbt = ydf_b200.Gbt(ds, cfg)
    effect = rng.normal(size=(len(nb), 256))
    m = sum(effect[f][bins[f]] for f in (0, 1, 4, 6)) + rng.normal(scale=0.5, size=n)
    if cfg.loss == 0:
        g = (0.9 * m / np.abs(m).max()).astype(np.float32)
        h = rng.uniform(0.01, 0.25, size=n).astype(np.float32)
        gbt.set_labels((m > 0).astype(np.int32) + 1)
    else:
        g = m.astype(np.float32)
        h = None
        gbt.set_labels(m.astype(np.float32))
    gbt.capture_candidates(True)
    tree = gbt.train_tree_on_gradients(g, h)
    assert (tree["feature"] >= 0).sum() >= min(3, 2 ** (cfg.max_depth - 1) - 1)
    assert check_scan(gbt, cfg, tree, byte_cols(bins, nb, ft), g, h) > 0
    if not cfg.use_hessian_gain:
        node_stats_check(tree, route(tree, byte_cols(bins, nb, ft)), g, gbt.level_candidates(0)["P"])


def test_exact_rule_and_many_features_deep_tree():
    """41 features (k_select_local's lanes loop), lossless-bucket features under the exact threshold rule (hi = B-1 among
    them), depth 10: the deepest split level holds up to 256 nodes, k_select_global's whole chunk."""
    rng = np.random.default_rng(5)
    n = 200000
    layout = [("num", 64)] * 30 + [("cat", 9)] * 6 + [("num", 255)] * 5
    bins, nb, ft = mixed_bins(rng, n, layout)
    # feature 40: 5 % of the rows in the last bucket, the rest in 0..99: its best boundary's next non-empty bucket is B-1
    bins[40] = np.where(rng.random(n) < 0.05, 254, rng.integers(0, 100, size=n)).astype(np.uint8)
    ds = ydf_b200.Dataset(bins, nb, np.zeros(len(nb), np.int32), feature_types=ft)
    values = {}
    for f in range(36, 41):
        v = np.cumsum(rng.uniform(0.1, 1.0, size=255)).astype(np.float32)
        ds.set_bucket_values(f, v, v[0])
        values[f] = v
    cfg = ydf_b200.default_config(loss=1, max_depth=10, min_examples=1)
    gbt = ydf_b200.Gbt(ds, cfg)
    g = (rng.normal(size=n) + sum(bins[f] * 0.01 for f in range(0, 41, 5)) + 3.0 * (bins[40] == 254)).astype(np.float32)
    gbt.set_labels(g)
    gbt.capture_candidates(True)
    tree = gbt.train_tree_on_gradients(g)
    assert len(gbt.level_candidates(8)["node"]) > 200
    assert check_scan(gbt, cfg, tree, byte_cols(bins, nb, ft, values), g, None) > 0
    cap = gbt.level_candidates(0)
    assert cap["found"][0, 40] and cap["hi"][0, 40] == 254
    node_stats_check(tree, route(tree, byte_cols(bins, nb, ft)), g, gbt.level_candidates(0)["P"])


@pytest.mark.parametrize("l2", [0.0, 1.0])
def test_pure_node_of_300k_rows_is_a_leaf(l2):
    """g = 0.7 on every row: every boundary's exact score is 0, so no split may be found (in doubles the two products
    of the numerator exceed 2^53 on such nodes and their rounding leaves a score of ~1e-33)."""
    rng = np.random.default_rng(0)
    n = 300000
    bins, nb, ft = mixed_bins(rng, n, [("num", 255), ("cat", 40), ("num", 16)])
    ds = ydf_b200.Dataset(bins, nb, np.zeros(3, np.int32), feature_types=ft)
    cfg = ydf_b200.default_config(loss=1, max_depth=4, min_examples=1, l2_regularization=l2)
    gbt = ydf_b200.Gbt(ds, cfg)
    g = np.full(n, 0.7, np.float32)
    gbt.set_labels(g)
    gbt.capture_candidates(True)
    tree = gbt.train_tree_on_gradients(g)
    cap = gbt.level_candidates(0)
    assert not cap["found"].any(), f"scores {cap['score'][cap['found'] != 0]}"
    assert len(tree) == 1


@pytest.mark.parametrize("near", [False, True])
def test_large_nodes_with_pure_and_near_pure_regions(near):
    """2M rows.  Pure: two regions of constant gradient (0.7 and 0.3) split once, then every node is pure.  Near pure:
    the gradients of one region differ by a few code units between halves, so exact scores are tiny but not zero."""
    rng = np.random.default_rng(1)
    n = 2000000
    bins, nb, ft = mixed_bins(rng, n, [("num", 255), ("num", 2), ("cat", 12)])
    ds = ydf_b200.Dataset(bins, nb, np.zeros(3, np.int32), feature_types=ft)
    cfg = ydf_b200.default_config(loss=1, max_depth=4, min_examples=1)
    gbt = ydf_b200.Gbt(ds, cfg)
    g = np.where(bins[1] == 1, np.float32(0.7), np.float32(0.3)).astype(np.float32)
    if near:
        g = np.where((bins[1] == 0) & (bins[0] >= 128), np.float32(0.3) + np.float32(3 * 2.0 ** -23), g).astype(np.float32)
    gbt.set_labels(g)
    gbt.capture_candidates(True)
    tree = gbt.train_tree_on_gradients(g)
    assert check_scan(gbt, cfg, tree, byte_cols(bins, nb, ft), g, None) > 0
    node_stats_check(tree, route(tree, byte_cols(bins, nb, ft)), g, gbt.level_candidates(0)["P"])
    splits = int((tree["feature"] >= 0).sum())
    assert splits == 1 if not near else splits >= 2


def test_capture_refusals_and_no_change_when_off():
    rng = np.random.default_rng(3)
    n = 20000
    bins, nb, ft = mixed_bins(rng, n, [("num", 64), ("cat", 5)])
    ds = ydf_b200.Dataset(bins, nb, np.zeros(2, np.int32), feature_types=ft)
    g = rng.normal(size=n).astype(np.float32)
    cfg = ydf_b200.default_config(loss=1, max_depth=5, num_trees=3)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(g)
    with pytest.raises(ydf_b200.YggError) as e:
        gbt.level_candidates(0)
    assert e.value.code == 1 and "not enabled" in str(e.value)
    gbt.capture_candidates(True)
    with pytest.raises(ydf_b200.YggError) as e:
        gbt.level_candidates(0)
    assert e.value.code == 1
    a = gbt.train_tree_on_gradients(g)
    for bad in (-1, cfg.max_depth - 1):
        with pytest.raises(ydf_b200.YggError) as e:
            gbt.level_candidates(bad)
        assert e.value.code == 1
    gbt.capture_candidates(False)
    b = gbt.train_tree_on_gradients(g)
    assert a.tobytes() == b.tobytes()
    # training: the same launches and the same trees with capture on and off
    runs = []
    for on in (False, True):
        h = ydf_b200.Gbt(ds, cfg)
        h.set_labels(g)
        h.capture_candidates(on)
        launches = h.train_timed(3)[1]
        runs.append((launches, [h.get_tree(t).tobytes() for t in range(3)]))
    assert runs[0] == runs[1]
    shuffled = ydf_b200.Gbt(ds, ydf_b200.default_config(loss=1, max_depth=3, candidate_shuffle=2))
    with pytest.raises(ydf_b200.YggError) as e:
        shuffled.capture_candidates(True)
    assert e.value.code == 1


def wide_codes(rng, n, B):
    """Wide numerical codes whose best boundary is the last bucket of the first 256-bucket tile (B > 257): the rows are in
    buckets 0..255 or in the top third, so the next non-empty bucket is in a later tile, several empty tiles away for
    B = 65535; for B = 257 the step is at bucket 200."""
    if B == 257:
        return rng.integers(0, B, size=n), 200
    return np.where(rng.random(n) < 0.5, rng.integers(0, 256, size=n), rng.integers(B - B // 3, B, size=n)), 256


@pytest.mark.parametrize("B_num,B_cat", [(257, 257), (513, 4096), (65535, 65535)])
def test_wide_columns_match_the_exact_scan(B_num, B_cat):
    """k_scan_wide (tiles of 256 buckets with a running carry, hi past the tile) and k_scan_wide_cat (B = 257: 255 +inf
    pads in the sort; 4096: none; 65535), at every level of a depth-5 tree with derived planes."""
    rng = np.random.default_rng(B_num + B_cat)
    n = 150000
    bins, nb, ft = mixed_bins(rng, n, [("num", 64), ("cat", 9), ("num", 1), ("cat", 1)])
    ds = ydf_b200.Dataset(bins, nb, np.zeros(4, np.int32), feature_types=ft)
    wn, step = wide_codes(rng, n, B_num)
    values = np.cumsum(rng.uniform(0.5, 1.5, size=B_num)).astype(np.float32)
    ds.set_wide_column(2, wn.astype(np.uint16), B_num, 0, values, values[0])
    p = 1.0 / np.arange(1, B_cat + 1) ** 1.05
    p /= p.sum()
    wc = rng.choice(B_cat, size=n, p=p)
    ds.set_wide_categorical_column(3, wc.astype(np.uint16), B_cat, 1)
    effect = rng.normal(size=B_cat) * (np.arange(B_cat) < 60)
    g = (1.5 * (wn >= step) + effect[wc] + 0.3 * (bins[0] > 30) + rng.normal(scale=0.5, size=n)).astype(np.float32)
    cfg = ydf_b200.default_config(loss=1, max_depth=5, min_examples=5)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(g)
    gbt.capture_candidates(True)
    tree = gbt.train_tree_on_gradients(g)
    cols = byte_cols(bins, nb, ft)
    cols[2] = ("wide_num", wn, B_num, values)
    cols[3] = ("wide_cat", wc, B_cat, None)
    assert check_scan(gbt, cfg, tree, cols, g, None) > 0
    assert {2, 3} <= set(tree["feature"][tree["feature"] >= 0].tolist())
    cap = gbt.level_candidates(0)
    k, t = int(cap["threshold_bin"][0, 2]), cap["threshold_value"][0, 2]
    assert cap["num_pos_examples"][0, 2] == int((wn >= step).sum()) and values[step - 1] < t <= values[k]
    assert (k == step) if B_num == 257 else (k > 256)   # past the first tile: the buckets after 255 are empty


def test_presorted_columns_match_the_exact_scan():
    """k_presort_scan / k_presort_candidates: tied values, -0.0 and +0.0 (one value), NaN replaced by the mean, and a column
    whose two boundaries have exactly equal scores at the root (the first must be kept)."""
    rng = np.random.default_rng(21)
    n = 120000
    sym = rng.choice(3, size=n, p=[0.3, 0.4, 0.3])
    sym[:36000], sym[36000:84000], sym[84000:] = 0, 1, 2          # counts 36000 / 48000 / 36000: mirror images
    a = np.round(rng.normal(size=n), 2).astype(np.float32)        # ties
    a[rng.random(n) < 0.1] = np.float32(-0.0)
    a[rng.random(n) < 0.1] = np.float32(0.0)
    a[rng.random(n) < 0.05] = np.nan
    b = rng.normal(size=n).astype(np.float32)
    bins, nb, ft = mixed_bins(rng, n, [("num", 1)] * 3 + [("num", 32)])
    ds = ydf_b200.Dataset(bins, nb, np.zeros(4, np.int32))
    ds.set_numerical_column(0, sym.astype(np.float32), 1.0)
    ds.set_numerical_column(1, a, float(np.nanmean(a)))
    ds.set_numerical_column(2, b, 0.0)
    cols = byte_cols(bins, nb, ds.feature_types)
    for f in range(3):
        cols[f] = ("pre", ds.get_numerical_column(f), 0, None)
    assert (cols[1][1] == 0).sum() > 0.15 * n and not np.isnan(cols[1][1]).any()
    # the root: g = +0.3 / 0 / -0.3 by `sym` (codes of equal magnitude: P = 0.5, no clamp), so its two boundaries tie
    # exactly; below, noise plus `a`
    g = np.where(sym == 0, 0.3, np.where(sym == 2, -0.3, 0.0)).astype(np.float32)
    g2 = (g + 0.2 * np.nan_to_num(a) * (sym == 1) + 0.1 * rng.normal(size=n) * (sym != 1)).astype(np.float32)
    for gg, first_split_on_sym in ((g, True), (g2, False)):
        cfg = ydf_b200.default_config(loss=1, max_depth=5, min_examples=3)
        gbt = ydf_b200.Gbt(ds, cfg)
        gbt.set_labels(gg)
        gbt.capture_candidates(True)
        tree = gbt.train_tree_on_gradients(gg)
        assert check_scan(gbt, cfg, tree, cols, gg, None) > 0
        if first_split_on_sym:
            cap = gbt.level_candidates(0)
            assert tree[0]["feature"] == 0 and cap["num_pos_examples"][0, 0] == 84000   # the first of the two boundaries


@pytest.mark.parametrize("pure_region", [False, True])
def test_weighted_variance_gain_matches_the_exact_scan(pure_region):
    """Example weights (squared error, the first tree of training): weight sums in place of the counts, the floor of half
    a unit per row, weighted category means; byte, wide and presorted columns."""
    rng = np.random.default_rng(31 + pure_region)
    n = 80000
    bins, nb, ft = mixed_bins(rng, n, [("num", 255), ("cat", 17), ("num", 1), ("num", 1)])
    ds = ydf_b200.Dataset(bins, nb, np.zeros(4, np.int32), feature_types=ft)
    wn = rng.integers(0, 300, size=n)
    values = np.arange(300, dtype=np.float32)
    ds.set_wide_column(2, wn.astype(np.uint16), 300, 0, values, 0.0)
    pv = np.round(rng.normal(size=n), 1).astype(np.float32)
    ds.set_numerical_column(3, pv, 0.0)
    cols = byte_cols(bins, nb, ds.feature_types)
    cols[2] = ("wide_num", wn, 300, values)
    cols[3] = ("pre", ds.get_numerical_column(3), 0, None)
    w = rng.uniform(0.2, 3.0, size=n).astype(np.float32)
    w[rng.random(n) < 0.02] = 0.0
    y = (np.sin(bins[0] / 40.0) + 0.5 * (bins[1] % 3) + 0.002 * wn + 0.3 * pv + rng.normal(scale=0.3, size=n))
    if pure_region:
        y = np.where(bins[1] < 4, 1.25, y)   # a constant region: weighted pure nodes
    y = y.astype(np.float32)
    cfg = ydf_b200.default_config(loss=1, max_depth=5, num_trees=1, min_examples=5)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_weights(w)
    gbt.set_labels(y)
    gbt.capture_candidates(True)
    gbt.train(1)
    tree = gbt.get_tree(0)
    init = np.float32(gbt.initial_prediction())
    wg = ((y - init).astype(np.float32) * w).astype(np.float32)   # k_pred_grad: (label - prediction) * weight
    assert check_scan(gbt, cfg, tree, cols, wg, None, w=w, tree_index=0) > 0
