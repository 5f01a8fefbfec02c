"""Wide categorical columns (257..65535 categories, uint16 codes; DESIGN.md §21) on the GPU: k_hist_wide's category
histograms against numpy (`==`), the CART split of k_scan_wide_cat against the numpy reference on the same integer
histograms, the pooled positive sets through partition / prediction / the model files, and the learner end to end."""
import os
import tempfile

import numpy as np
import pytest

import ydf_b200
from ydf_b200 import dataspec, model_io
from ydf_b200.model import GradientBoostedTreesModel
from tests import wide_cat_ref as W
from tests.util import pow2_cover, quantize_q24, quantize_second

pytestmark = pytest.mark.gpu


def cat_dataset(byte, byte_bins, byte_types, wide):
    """Byte columns, then the wide categorical columns `wide` = [(codes, num_bins, na_bin)] attached after them."""
    F = byte.shape[0] + len(wide)
    n = byte.shape[1]
    b = np.zeros((F, n), np.uint8)
    b[:byte.shape[0]] = byte
    types = list(byte_types) + [1] * len(wide)
    ds = ydf_b200.Dataset(b, list(byte_bins) + [1] * len(wide), [0] * F, feature_types=types)
    for i, (codes, B, na) in enumerate(wide):
        ds.set_wide_categorical_column(byte.shape[0] + i, codes, B, na)
        got, nb, nab = ds.get_wide_column(byte.shape[0] + i)
        assert (got == codes).all() and nb == B and nab == na
    return ds


@pytest.mark.parametrize("B", [257, 2001, 65535])
def test_category_histograms_are_exact(B):
    n = 90000
    rng = np.random.default_rng(B)
    codes, _ = W.zipf_codes(rng, n, B, na_bin=1)
    byte = rng.integers(0, 16, size=(2, n)).astype(np.uint8)
    ds = cat_dataset(byte, [16, 16], [0, 1], [(codes, B, 1)])
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=6))
    g = (rng.normal(size=n) * 0.3).astype(np.float32)
    slots = rng.integers(-1, 2, size=n).astype(np.int32)
    _, _, _, (P, _) = gbt.level_histogram(2, g, slots, 2)
    s, c, _ = gbt.wide_histogram(2)
    q = quantize_q24(g, P)
    rs = np.zeros((2, B), np.uint64)
    rc = np.zeros((2, B), np.uint32)
    rows = np.nonzero(slots >= 0)[0]
    np.add.at(rs.reshape(-1), slots[rows] * B + codes[rows], q[rows].astype(np.uint64))
    np.add.at(rc.reshape(-1), slots[rows] * B + codes[rows], np.uint32(1))
    assert (c == rc).all() and (s == rs).all()


def root_case(n, B, seed, pure=False):
    rng = np.random.default_rng(seed)
    codes, _ = W.zipf_codes(rng, n, B, na_bin=2)
    effect = rng.normal(size=B)
    if pure:   # many categories whose rows all carry one label: equal keys, ordered by index
        effect = np.where(rng.random(B) < 0.5, 9.0, -9.0) * (np.arange(B) % 3 != 0) + effect * (np.arange(B) % 3 == 0)
    y = (effect[codes] + rng.normal(scale=0.7, size=n) > 0).astype(np.int32) + 1
    return codes, y


@pytest.mark.parametrize("hessian", [0, 1])
@pytest.mark.parametrize("B,pure", [(257, False), (2001, False), (5000, False), (65535, False), (3000, True)])
def test_root_split_matches_the_numpy_cart(B, pure, hessian):
    """One split (max_depth 2: the root is the only histogrammed level, whose planes wide_histogram reads back after
    training): feature, full positive set, na_value and positive count exact, score within 1e-5 of the numpy CART on the
    same integer sums."""
    n = 120000
    codes, y = root_case(n, B, seed=B + 7 * hessian + pure, pure=pure)
    rng = np.random.default_rng(1)
    byte = rng.integers(0, 4, size=(1, n)).astype(np.uint8)   # a weak byte feature next to the wide one
    ds = cat_dataset(byte, [4], [0], [(codes, B, 2)])
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=2, num_trees=1, use_hessian_gain=hessian))
    gbt.set_labels(y)
    gbt.train(1)
    tree = gbt.get_tree(0)
    s, c, h2 = gbt.wide_histogram(1)
    p0 = 1 / (1 + np.exp(-np.float64(gbt.initial_prediction())))
    sq = s[0].astype(np.float64) - c[0].astype(np.float64) * 2.0 ** 23   # P = 1 on the binomial loss
    g = sq / 2.0 ** 23
    if hessian:
        V = float(pow2_cover(np.float32(p0 * (1 - p0))))
        h = h2[0].astype(np.float64) * V / 2.0 ** 24
    else:
        h = c[0].astype(np.float64)
    ref = W.best_split(c[0], g, h, bool(hessian), min_obs=5, subtract_parent=bool(gbt.cfg.hessian_split_score_subtract_parent))
    assert ref is not None
    root = tree[0]
    assert root["feature"] == 1 and root["condition_type"] == 1
    assert (root["cat_mask"] == 0).all()
    sets = gbt.get_category_sets(0, tree)
    got = W.set_of_words(sets[0], B)
    score, positive, n_pos = ref
    assert np.array_equal(got, positive)
    assert root["num_pos_examples"] == n_pos
    assert bool(root["na_value"]) == (2 in set(positive.tolist()))
    np.testing.assert_allclose(root["split_score"], score, rtol=1e-5)
    assert root["num_pos_examples"] == int(np.isin(codes, positive).sum())


def mixed_table(n, seed, task="binary", wide_cat=(2001, 300)):
    """Byte numerical, byte categorical, wide numerical and wide categorical columns (Zipf(1.2), 5% missing)."""
    rng = np.random.default_rng(seed)
    margin = np.zeros(n)
    cols, bins = [], []
    x = rng.normal(size=n).astype(np.float32)
    c = dataspec.infer_column("num", x, 64)
    cols.append(c); bins.append(c.encode(x).astype(np.uint16)); margin += x
    k = 20
    cc = rng.integers(0, k, size=n)
    cols.append(dataspec.CategoricalColumn("small", ["<OOD>"] + [str(i) for i in range(1, k)], [0] * k, k, 1))
    bins.append(cc.astype(np.uint16)); margin += rng.normal(size=k)[cc]
    grid = np.sort(rng.choice(100000, size=900, replace=False)).astype(np.float32)
    xw = grid[rng.integers(0, 900, size=n)]
    xw[rng.random(n) < 0.05] = np.nan
    cw = dataspec.infer_column_lossless("wide_num", xw, max_distinct=65535)
    cols.append(cw); bins.append(cw.encode16(xw)); margin += np.sin(np.nan_to_num(xw) / 9000.0)
    for j, B in enumerate(wide_cat):
        codes, _ = W.zipf_codes(rng, n, B, na_bin=1)
        cols.append(dataspec.CategoricalColumn(f"wc{j}", ["<OOD>"] + [str(i) for i in range(1, B)], [0] * B, B, 1))
        bins.append(codes); margin += 1.5 * rng.normal(size=B)[codes]
    margin += rng.normal(scale=0.5, size=n)
    if task == "binary":
        y = (margin > np.median(margin)).astype(np.int32) + 1
    elif task == "multi":
        y = np.digitize(margin, np.quantile(margin, [1 / 3, 2 / 3])).astype(np.int32) + 1
    else:
        y = margin.astype(np.float32)
    return cols, np.stack(bins), y


def routed_counts(tree, sets, bins):
    """Rows reaching every node of a pre-order tree, routed on the host with the pooled sets."""
    n = bins.shape[1]
    node = np.zeros(n, np.int64)
    counts = np.zeros(len(tree), np.int64)
    active = np.ones(n, bool)
    while active.any():
        np.add.at(counts, node[active], 1)
        idx = np.nonzero(active)[0]
        nd = node[idx]
        leaf = tree["feature"][nd] < 0
        active[idx[leaf]] = False
        idx, nd = idx[~leaf], nd[~leaf]
        b = bins[tree["feature"][nd], idx].astype(np.int64)
        pos = np.zeros(len(idx), bool)
        for i in np.unique(nd):
            at = nd == i
            t = tree[i]
            if t["condition_type"] == 1:
                words = sets[int(i)] if int(i) in sets else t["cat_mask"]
                pos[at] = ((words[b[at] >> 5] >> (b[at] & 31).astype(np.uint32)) & 1) != 0
            else:
                pos[at] = b[at] >= t["threshold_bin"]
        node[idx] = np.where(pos, tree["pos_child"][nd], tree["neg_child"][nd])
    return counts


CASES = {
    "variance": dict(),
    "hessian": dict(use_hessian_gain=1),
    "regression": dict(loss=1),
    "multinomial": dict(loss=2, num_classes=3),
    "depth2": dict(max_depth=2),
    "depth10": dict(max_depth=10, min_examples=5),
    "min_examples_400": dict(min_examples=400, max_depth=8),
    "subsample": dict(subsample=0.6),
    "goss": dict(goss_alpha=0.2, goss_beta=0.1),
    "best_first": dict(growing_strategy=1, max_num_nodes=20),
    "no_sibling_subtraction": dict(sibling_subtraction=0),
    "weights": dict(),
    "tie_shuffle": dict(candidate_shuffle=2, split_jobs_draw_seeds=1),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_trees_route_by_their_sets_and_predictions_agree(case):
    """Every split of every tree sends exactly its recorded positive count through the host routing of the pooled sets
    (so partition, the stored sets and the counts agree), and ygg_gbt_predict equals the host model on held-out rows,
    out-of-dictionary codes and NA rows."""
    kw = dict(CASES[case])
    task = "multi" if kw.get("loss") == 2 else ("reg" if kw.get("loss") == 1 else "binary")
    cols, bins, y = mixed_table(60000, seed=100 + sorted(CASES).index(case), task=task)
    train = np.arange(len(y)) < 50000
    cfg = ydf_b200.default_config(max_depth=kw.pop("max_depth", 6), num_trees=4, **kw)
    ds = dataspec.device_dataset(bins[:, train], cols)
    held = bins[:, ~train].copy()
    held[3, :50] = 0        # out-of-dictionary
    held[4, 50:100] = 1     # the NA replacement
    dsv = dataspec.device_dataset(held, cols)
    gbt = ydf_b200.Gbt(ds, cfg)
    if case == "weights":
        gbt.set_weights(np.random.default_rng(5).random(int(train.sum())).astype(np.float32) * 2)
    gbt.set_labels(y[train])
    gbt.train(4)
    trees = [gbt.get_tree(i) for i in range(gbt.num_trees())]
    sets = [gbt.get_category_sets(i, t) for i, t in enumerate(trees)]
    assert any(sets), "no split on a wide categorical column"
    if case not in ("subsample", "goss"):   # (sampled trees count the sampled rows only)
        for t, s in zip(trees, sets):
            counts = routed_counts(t, s, bins[:, train])
            for i in np.nonzero(t["feature"] >= 0)[0]:
                assert counts[t["pos_child"][i]] == t["num_pos_examples"][i]
                assert counts[i] == t["num_examples"][i]
    for t, s in zip(trees, sets):
        for i, words in s.items():
            f = int(t["feature"][i])
            assert len(words) == (cols[f].num_bins + 31) // 32
            assert bool(t["na_value"][i]) == bool((words[1 >> 5] >> 1) & 1)   # na_bin = 1
    spec = dataspec.DataSpec(columns=cols, label="y", task="CLASSIFICATION" if task != "reg" else "REGRESSION")
    if task == "multi":
        spec.label_classes = [1, 2, 3]
    loss = {0: "BINOMIAL_LOG_LIKELIHOOD", 1: "SQUARED_ERROR", 2: "MULTINOMIAL_LOG_LIKELIHOOD"}[cfg.loss]
    model = GradientBoostedTreesModel(spec, trees, gbt.initial_prediction(), loss, category_sets=sets)
    np.testing.assert_allclose(gbt.predict(dsv), model._raw(held), rtol=0, atol=1e-5)


def test_held_out_split_with_early_stopping():
    """The random hold-out (ygg_dataset_split_rows carries the wide categorical columns), validation losses through
    k_valid_update and early stopping; the engine's predictions on the held-out rows equal the host model's."""
    cols, bins, y = mixed_table(50000, seed=77, task="reg")
    ds = dataspec.device_dataset(bins, cols)
    sel = (np.random.default_rng(2).random(len(y)) < 0.8).astype(np.uint8)
    tr, va = ds.split_rows(sel)
    for f in (3, 4):
        assert (tr.get_wide_column(f)[0] == bins[f, sel == 1]).all()
        assert (va.get_wide_column(f)[0] == bins[f, sel == 0]).all()
    cfg = ydf_b200.default_config(loss=1, max_depth=6, num_trees=30, early_stopping=2,
                                  early_stopping_num_trees_look_ahead=3, early_stopping_initial_iteration=2)
    gbt = ydf_b200.Gbt(tr, cfg)
    gbt.set_labels(y[sel == 1])
    gbt.set_validation(va, y[sel == 0])
    gbt.train(30)
    trees = [gbt.get_tree(i) for i in range(gbt.num_trees())]
    sets = [gbt.get_category_sets(i, t) for i, t in enumerate(trees)]
    assert any(sets)
    spec = dataspec.DataSpec(columns=cols, label="y", task="REGRESSION")
    model = GradientBoostedTreesModel(spec, trees, gbt.initial_prediction(), "SQUARED_ERROR", category_sets=sets)
    np.testing.assert_allclose(gbt.predict(va), model._raw(bins[:, sel == 0]), rtol=0, atol=1e-5)
    losses = [gbt.validation_loss(i)[0] for i in range(gbt.num_iterations())]
    assert np.isfinite(losses).all() and losses[-1] < losses[0]


def test_learner_end_to_end_with_2001_categories():
    """A string column with 2001 dictionary entries (option raised): the learner trains, and model.predict, the saved
    model read back by the generic reader, and the engine agree on held-out rows, unknown strings and missing values,
    including categories absent from the node that splits on them."""
    rng = np.random.default_rng(11)
    n = 80000
    B = 2001
    codes, miss = W.zipf_codes(rng, n, B, missing=0.05, na_bin=0)
    codes = np.maximum(codes, 1)
    codes[:B - 1] = np.arange(1, B)   # every category present: 2000 entries + <OOD>
    words = np.array([f"k{i:05d}" for i in range(B + 50)], dtype=object)
    col = words[codes].copy()
    col[miss] = ""
    effect = rng.normal(size=B + 50)
    x = rng.integers(-20, 20, size=n).astype(np.float32) / 10   # 40 values: the exact splitter's byte buckets
    y = np.where(effect[codes] + 0.5 * x + rng.normal(scale=0.5, size=n) > 0, "a", "b")
    data = {"c": col, "x": x, "y": y}
    L = ydf_b200.GradientBoostedTreesLearner
    with pytest.raises(NotImplementedError, match="categorical_arity_limit_for_random"):
        L(label="y", min_vocab_frequency=1, num_trees=3).train(data)
    model = L(label="y", min_vocab_frequency=1, max_vocab_count=-1, categorical_arity_limit_for_random=65536,
              num_trees=12, validation_ratio=0.1).train(data)
    c = model.data_spec.columns[0]
    assert c.num_bins > 256 and c.wide
    assert any(model.category_sets)
    probe = {"c": np.concatenate([col[:3000], words[B:B + 50], np.array([""] * 20, object)]),
             "x": np.concatenate([x[:3000], np.zeros(70, np.float32)])}
    p_host = model.predict(probe)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "m")
        model.save(path)
        m = model_io.read_ydf_model(path)
        assert m["columns"][1]["number_of_unique_values"] == c.num_bins
        assert len(m["columns"][1]["vocabulary"]) == c.num_bins
        raw_io = model_io.predict_ydf_model(m, probe)
    np.testing.assert_allclose(1 / (1 + np.exp(-raw_io.astype(np.float64))), p_host, rtol=0, atol=1e-6)


# ---- every wide categorical split against the numpy CART on its node's own histogram -------------------------------

def rows_of_nodes(tree, sets, bins):
    """Training rows of every node of a pre-order tree (parents come before their children)."""
    rows = [None] * len(tree)
    rows[0] = np.arange(bins.shape[1])
    for i in range(len(tree)):
        t = tree[i]
        if t["feature"] < 0:
            continue
        r = rows[i]
        b = bins[t["feature"], r].astype(np.int64)
        if t["condition_type"] == 1:
            words = sets.get(i, t["cat_mask"])
            pos = ((words[b >> 5] >> (b & 31).astype(np.uint32)) & 1) != 0
        else:
            pos = b >= t["threshold_bin"]
        rows[t["pos_child"]], rows[t["neg_child"]] = r[pos], r[~pos]
    return rows


def check_against_reference(tree, sets, cols, bins, g_units, h_units, use_hessian, min_obs, w_units=None, subtract_parent=False):
    """Every split node: a split on a wide categorical feature has the numpy CART's positive set, positive count,
    na_value and score (1e-5) on the node's own per-category sums; a split on another feature scores at least the best
    wide categorical split of the node.  `*_units`: per-row quantised values in the engine's units (exact sums).
    -> number of wide categorical splits checked."""
    rows = rows_of_nodes(tree, sets, bins)
    wide = [f for f, c in enumerate(cols) if c.feature_type == 1 and c.num_bins > 256]
    checked = 0
    for i in np.nonzero(tree["feature"] >= 0)[0]:
        t, r = tree[i], rows[i]
        assert len(r) == t["num_examples"]
        best = None
        for f in wide:
            B = cols[f].num_bins
            code = bins[f, r].astype(np.int64)
            cnt = np.bincount(code, minlength=B).astype(np.float64)
            s = np.bincount(code, weights=g_units[r], minlength=B)
            h = np.bincount(code, weights=h_units[r], minlength=B) if use_hessian else cnt
            w = None if w_units is None else np.bincount(code, weights=w_units[r], minlength=B)
            ref = W.best_split(cnt, s, h, use_hessian, min_obs=min_obs, weight=w, subtract_parent=subtract_parent)
            if t["feature"] == f:
                assert ref is not None
                score, positive, n_pos = ref
                got = W.set_of_words(sets[int(i)], B)
                assert np.array_equal(got, positive), f"node {i}: positive set differs"
                assert t["num_pos_examples"] == n_pos
                assert bool(t["na_value"]) == (cols[f].na_bin in set(positive.tolist()))
                np.testing.assert_allclose(t["split_score"], score, rtol=1e-5)
                checked += 1
            elif ref is not None:
                best = max(best or 0.0, ref[0])
        if t["feature"] not in wide and best is not None:
            assert best <= t["split_score"] * (1 + 1e-5) + 1e-12, f"node {i}: a better wide categorical split was missed"
    return checked


TREE_CASES = {
    "variance": dict(loss=1),
    "hessian": dict(loss=0, use_hessian_gain=1),
    "depth2": dict(loss=1, max_depth=2),
    "depth10": dict(loss=1, max_depth=10, min_examples=5),
    "min_examples_400": dict(loss=1, max_depth=8, min_examples=400),
    "no_sibling_subtraction": dict(loss=1, sibling_subtraction=0),
    "hessian_no_sibling_subtraction": dict(loss=0, use_hessian_gain=1, sibling_subtraction=0, max_depth=8),
    "hessian_subtract_parent": dict(loss=0, use_hessian_gain=1, hessian_split_score_subtract_parent=1),
}


@pytest.mark.parametrize("case", sorted(TREE_CASES))
def test_every_split_of_a_tree_matches_the_numpy_cart(case):
    """ygg_tree_train_on_gradients on known gradients (their sets read back with tree -1): derived (parent - direct) and
    direct nodes at every depth, both gains; the leaves of the variance gain are the nodes' mean gradients."""
    kw = dict(TREE_CASES[case])
    cols, bins, y = mixed_table(70000, seed=300 + sorted(TREE_CASES).index(case), task="reg")
    rng = np.random.default_rng(sorted(TREE_CASES).index(case))
    ds = dataspec.device_dataset(bins, cols)
    cfg = ydf_b200.default_config(max_depth=kw.pop("max_depth", 6), **kw)
    gbt = ydf_b200.Gbt(ds, cfg)
    m = (y - y.mean()) / np.abs(y - y.mean()).max()
    if cfg.loss == 0:   # binomial: |g| < 1 on the fixed scale P = 1, 0 < h <= 0.25 on V = 0.25
        g = (0.98 * m).astype(np.float32)
        h = (rng.uniform(0.01, 0.25, size=len(y))).astype(np.float32)
        gbt.set_labels((m > 0).astype(np.int32) + 1)
        P, V = 1.0, 0.25
    else:
        g = (3.0 * m + rng.normal(scale=0.2, size=len(y))).astype(np.float32)
        h = None
        gbt.set_labels(y)
        P, V = float(pow2_cover(np.abs(g).max())), 1.0
    tree = gbt.train_tree_on_gradients(g, h)
    sets = gbt.get_category_sets(-1, tree)
    assert sets, "no split on a wide categorical column"
    g_units = (quantize_q24(g, P) - 2 ** 23).astype(np.float64) * P / 2.0 ** 23
    h_units = None if h is None else quantize_second(h, V).astype(np.float64) * V / 2.0 ** 24
    assert check_against_reference(tree, sets, cols, bins, g_units, h_units, bool(cfg.use_hessian_gain), cfg.min_examples,
                                   subtract_parent=bool(cfg.hessian_split_score_subtract_parent)) > 0
    if not cfg.use_hessian_gain:
        rows = rows_of_nodes(tree, sets, bins)
        leaves = np.nonzero(tree["feature"] < 0)[0]
        means = np.array([g[rows[i]].astype(np.float64).mean() for i in leaves])
        # (the leaf of the tree trainer: the mean gradient, times the shrinkage when the trainer applies it)
        assert any(np.allclose(tree["leaf_value"][leaves], k * means, rtol=1e-5, atol=1e-6) for k in (cfg.shrinkage, 1.0))


def test_weighted_splits_match_the_numpy_cart():
    """Example weights (variance gain, squared error): the key is the weighted mean and the score uses the weight sums.
    The quantised w*g and weights are first pinned `==` against the engine's own root histogram (max_depth 2), then
    every wide categorical split of a depth-6 tree is checked on them."""
    cols, bins, y = mixed_table(60000, seed=411, task="reg")
    w = np.random.default_rng(4).uniform(0.2, 3.0, size=len(y)).astype(np.float32)
    trees = {}
    for depth in (2, 6):
        gbt = ydf_b200.Gbt(dataspec.device_dataset(bins, cols), ydf_b200.default_config(loss=1, max_depth=depth, num_trees=1))
        gbt.set_weights(w)
        gbt.set_labels(y)
        gbt.train(1)
        tree = gbt.get_tree(0)
        trees[depth] = (tree, gbt.get_category_sets(0, tree), np.float32(gbt.initial_prediction()), gbt)
    tree, sets, init, gbt2 = trees[2]
    wg = (y.astype(np.float32) - init) * w
    P, WP = float(pow2_cover(np.abs(wg).max())), float(pow2_cover(w.max()))
    q, qw = quantize_q24(wg, P), quantize_second(w, WP)
    s, c, s2 = gbt2.wide_histogram(1)
    offs = np.concatenate([[0], np.cumsum([cols[f].num_bins for f in (2, 3, 4)])])
    for k, f in enumerate((2, 3, 4)):
        B = cols[f].num_bins
        assert (c[0, offs[k]:offs[k] + B] == np.bincount(bins[f], minlength=B)).all()
        assert (s[0, offs[k]:offs[k] + B] == np.bincount(bins[f], weights=q, minlength=B).astype(np.uint64)).all()
        assert (s2[0, offs[k]:offs[k] + B] == np.bincount(bins[f], weights=qw, minlength=B).astype(np.uint64)).all()
    g_units = (q - 2 ** 23).astype(np.float64) * P / 2.0 ** 23
    w_units = qw.astype(np.float64) * WP / 2.0 ** 24
    for depth in (2, 6):
        tree, sets, _, _ = trees[depth]
        assert check_against_reference(tree, sets, cols, bins, g_units, None, False, 5, w_units=w_units) > 0


# ---- tie-break replay ------------------------------------------------------------------------------------------------

def tie_table(n, B, seed):
    rng = np.random.default_rng(seed)
    codes, _ = W.zipf_codes(rng, n, B, missing=0.0, na_bin=1)
    group = (rng.random(B) < 0.5).astype(np.int32)
    group[0], group[1] = 0, 1
    y = group[codes] + 1   # the label is a function of the category's group: the group partition is a pure split
    return codes, group, y


def test_a_tied_wide_categorical_alternative_is_counted_unresolved():
    """Two identical wide categorical columns: the second is recorded without its set (n_pos = -1), so whenever the
    reference's shuffle puts it first the node keeps the first column and counts as unresolved."""
    n, B = 40000, 700
    codes, _, y = tie_table(n, B, seed=21)
    noise = np.random.default_rng(3).integers(0, 8, size=(1, n)).astype(np.uint8)
    ds = cat_dataset(noise, [8], [0], [(codes, B, 1), (codes.copy(), B, 1)])
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=3, num_trees=12, candidate_shuffle=2, split_jobs_draw_seeds=1))
    gbt.set_labels(y)
    gbt.train(12)
    renamed, unresolved = gbt.tie_stats()
    assert unresolved > 0 and renamed == 0
    trees = [gbt.get_tree(i) for i in range(gbt.num_trees())]
    sets = [gbt.get_category_sets(i, t) for i, t in enumerate(trees)]
    assert all(t["feature"][0] == 1 for t in trees)   # the engine's choice stays
    bins = np.stack([noise[0].astype(np.uint16), codes, codes])
    cols = [dataspec.CategoricalColumn("n", [str(i) for i in range(8)], [0] * 8, 8, 0)] + \
           [dataspec.CategoricalColumn(f"c{j}", [str(i) for i in range(B)], [0] * B, B, 1) for j in range(2)]
    model = GradientBoostedTreesModel(dataspec.DataSpec(columns=cols, label="y", task="CLASSIFICATION"), trees,
                                      gbt.initial_prediction(), "BINOMIAL_LOG_LIKELIHOOD", category_sets=sets)
    np.testing.assert_allclose(gbt.predict(ds), model._raw(bins), rtol=0, atol=1e-5)
    for t, s in zip(trees, sets):
        counts = routed_counts(t, s, bins)
        for i in np.nonzero(t["feature"] >= 0)[0]:
            assert counts[t["pos_child"][i]] == t["num_pos_examples"][i]


def test_a_wide_categorical_split_is_renamed_to_a_verified_byte_twin():
    """A byte categorical column holding each row's group cuts the root exactly like the wide column's best split (a
    pure partition, equal float scores).  The wide column comes first and wins the level-wise tie-break; when the
    reference's shuffle puts the byte column first the node is renamed to it and routes by its byte mask."""
    n, B = 40000, 700
    codes, group, y = tie_table(n, B, seed=22)
    twin = (group[codes] + 1).astype(np.uint8)[None, :]     # categories 1 / 2 of a 3-category byte column
    ds = ydf_b200.Dataset(np.concatenate([np.zeros((1, n), np.uint8), twin]), [1, 3], [0, 1], feature_types=[1, 1])
    ds.set_wide_categorical_column(0, codes, B, 1)
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=2, num_trees=12, candidate_shuffle=2, split_jobs_draw_seeds=1))
    gbt.set_labels(y)
    gbt.train(12)
    renamed, unresolved = gbt.tie_stats()
    trees = [gbt.get_tree(i) for i in range(gbt.num_trees())]
    sets = [gbt.get_category_sets(i, t) for i, t in enumerate(trees)]
    roots = [int(t["feature"][0]) for t in trees]
    assert renamed > 0 and unresolved == 0
    assert roots.count(1) == renamed and roots.count(0) == len(trees) - renamed
    present = np.unique(codes)
    for t, s in zip(trees, sets):
        if t["feature"][0] == 1:   # renamed: routed by the byte mask, no pooled set
            assert 0 not in s and t["cat_mask"][0].any()
        else:                      # the categories present in the positive set are one group
            pos = np.intersect1d(W.set_of_words(s[0], B), present)
            assert len(np.unique(group[pos])) == 1 and len(pos) == int((group[present] == group[pos[0]]).sum())
    bins = np.stack([codes, twin[0].astype(np.uint16)])
    cols = [dataspec.CategoricalColumn("c", [str(i) for i in range(B)], [0] * B, B, 1),
            dataspec.CategoricalColumn("t", ["0", "1", "2"], [0] * 3, 3, 1)]
    model = GradientBoostedTreesModel(dataspec.DataSpec(columns=cols, label="y", task="CLASSIFICATION"), trees,
                                      gbt.initial_prediction(), "BINOMIAL_LOG_LIKELIHOOD", category_sets=sets)
    np.testing.assert_allclose(gbt.predict(ds), model._raw(bins), rtol=0, atol=1e-5)
