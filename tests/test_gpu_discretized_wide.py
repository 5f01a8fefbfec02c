"""Discretized wide columns (257..65535 bins, uint16 codes; DESIGN.md §25) on the GPU: the 16-bit binning step against the
host rule, the wide histograms against an integer reference, every split candidate against the exact scan reference
with the discretized threshold rule (across 256-bucket tiles), trees against the oracle on the same uint16 codes, the
saved model, the learner end to end and the memory refusal."""
import os
import tempfile

import numpy as np
import pytest

import ydf_b200
from ydf_b200 import dataspec, model_io
from tests import scan_ref as S
from tests.test_discretized_wide_cpu import _columns
from tests.test_gpu_scan_exact import byte_cols, check_scan, mixed_bins
from tests.test_gpu_wide_columns import _oracle_cfg, oracle_train as _oracle_train, wide_hist_ref
from tests.util import compare_trees, quantize_q24
from oracle import oracle as O

pytestmark = pytest.mark.gpu


# ---- binning ---------------------------------------------------------------------------------------------------------

def _check_builder_column(b, f, x, max_bins, n_stats=0):
    bounds, mean, na_bin, missing = b.get_numerical(f)
    sample = x if n_stats <= 0 else x[:n_stats]
    want = dataspec.infer_column16("x", sample, max_bins)
    np.testing.assert_array_equal(bounds, want.boundaries)
    # (the device sums in a fixed compensated order, the host in long double: the same float32 mean, as the byte path)
    assert mean == pytest.approx(want.mean, rel=1e-14, abs=1e-300) and np.float32(mean) == np.float32(want.mean)
    assert na_bin == want.na_bin and missing == int(np.isnan(sample).sum())
    return want


@pytest.mark.parametrize("max_bins", [257, 1024, 4096, 65535])
@pytest.mark.parametrize("n", [3000, 1000000])
def test_binning_matches_the_host_rule(max_bins, n):
    """Boundaries, mean, NA bin and every uint16 code, bit for bit, on ties, NaN, -0, heavy values, constants and fewer
    distinct values than bins; columns that end with at most 256 bins become byte columns with the same codes."""
    cols = _columns(n, seed=max_bins + n)
    names = list(cols)
    b = ydf_b200.DatasetBuilder(n, len(names))
    for f, name in enumerate(names):
        b.add_numerical16_async(f, cols[name], max_bins, 3)
    want = [_check_builder_column(b, f, cols[name], max_bins) for f, name in enumerate(names)]
    ds = b.finish()
    for f, name in enumerate(names):
        codes = want[f].encode16(cols[name])
        if want[f].num_bins > 256:
            got, nb, na = ds.get_wide_column(f)
            assert nb == want[f].num_bins and na == want[f].na_bin
        else:
            got = ds.get_bins(f)
        np.testing.assert_array_equal(got.astype(np.uint16), codes, err_msg=name)
    if n >= 1000000 and max_bins >= 1024:
        assert want[0].num_bins > 256 and want[1].num_bins > 256   # the continuous and the tied columns are wide
    ds.close()


def test_binning_at_full_size_and_with_a_statistics_sample():
    """10M rows at 65535 and 1024 bins, the boundaries from the first rows only (n_stats_rows), every row encoded."""
    n = 10_000_000
    rng = np.random.default_rng(7)
    x = rng.normal(size=n).astype(np.float32)
    x[rng.random(n) < 0.01] = np.nan
    t = np.round(rng.exponential(size=n) * 2000).astype(np.float32)
    b = ydf_b200.DatasetBuilder(n, 3)
    b.add_numerical16_async(0, x, 65535, 3)
    b.add_numerical16_async(1, t, 1024, 3)
    b.add_numerical16_async(2, x, 4096, 3, n_stats_rows=500000)
    want = [_check_builder_column(b, 0, x, 65535), _check_builder_column(b, 1, t, 1024),
            _check_builder_column(b, 2, x, 4096, n_stats=500000)]
    ds = b.finish()
    for f, v in enumerate((x, t, x)):
        got, nb, _ = ds.get_wide_column(f)
        assert nb == want[f].num_bins
        np.testing.assert_array_equal(got, want[f].encode16(v))
    assert want[0].num_bins > 60000
    ds.close()


def test_builder_refusals():
    b = ydf_b200.DatasetBuilder(1000, 1)
    x = np.arange(1000, dtype=np.float32)
    for bad in (256, 65536):
        with pytest.raises(ydf_b200.YggError, match="257, 65535"):
            b.add_numerical16_async(0, x, bad, 3)
    with pytest.raises(ydf_b200.YggError):
        b.add_numerical_async(0, x, 300, 3)   # the byte path keeps its bound
    b.close()


# ---- histograms ------------------------------------------------------------------------------------------------------

def test_wide_histograms_are_exact():
    n = 70000
    rng = np.random.default_rng(3)
    x = rng.normal(size=n).astype(np.float32)
    col = dataspec.infer_column16("x", x, 4096)
    codes = col.encode16(x)
    byte = rng.integers(0, 32, size=(3, n)).astype(np.uint8)
    ds = ydf_b200.Dataset(byte, [32] * 3, [0] * 3)
    ds.set_wide_discretized_column(2, codes, col.num_bins, col.na_bin)
    got, nb, na = ds.get_wide_column(2)
    assert (got == codes).all() and nb == col.num_bins and na == col.na_bin
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=6))
    g = (rng.normal(size=n) * 0.3).astype(np.float32)
    slots = rng.integers(-1, 3, size=n).astype(np.int32)
    _, _, _, (P, _) = gbt.level_histogram(3, g, slots, 3)
    s, c, _ = gbt.wide_histogram(3)
    rs, rc, _ = wide_hist_ref([codes], np.array([0, col.num_bins]), col.num_bins, slots, 3, quantize_q24(g, P))
    assert (c == rc).all() and (s == rs).all()


# ---- candidates ------------------------------------------------------------------------------------------------------

def _tile_codes(rng, n, B, step):
    """Rows in buckets [0, step) or in the top third: the first non-empty bucket after `step - 1` is tiles away."""
    return np.where(rng.random(n) < 0.5, rng.integers(0, step, size=n), rng.integers(B - B // 3, B, size=n))


@pytest.mark.parametrize("B,step", [(257, 200), (300, 256), (4096, 255), (4096, 257), (65535, 256), (65535, 1000)])
def test_candidates_match_the_exact_scan(B, step):
    """Every candidate of every level of a depth-5 tree, with the discretized rule: bucket interpolation across runs of
    empty buckets that start before, at and after a 256-bucket tile edge."""
    rng = np.random.default_rng(B + step)
    n = 150000
    bins, nb, ft = mixed_bins(rng, n, [("num", 64), ("cat", 9), ("num", 1)])
    ds = ydf_b200.Dataset(bins, nb, np.zeros(3, np.int32), feature_types=ft)
    wn = _tile_codes(rng, n, B, step)
    ds.set_wide_discretized_column(2, wn.astype(np.uint16), B, B // 2)
    g = (1.5 * (wn >= step) + 0.3 * (bins[0] > 30) + 0.2 * (wn % 5) + rng.normal(scale=0.5, size=n)).astype(np.float32)
    cfg = ydf_b200.default_config(loss=1, max_depth=5, min_examples=5)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(g)
    gbt.capture_candidates(True)
    tree = gbt.train_tree_on_gradients(g)
    cols = byte_cols(bins, nb, ft)
    cols[2] = ("wide_num", wn, B, None)
    assert check_scan(gbt, cfg, tree, cols, g, None) > 0
    cap = gbt.level_candidates(0)
    want = S.numerical_expect(np.bincount(wn, minlength=B), step - 1, B)[0]
    assert tree[0]["feature"] == 2 and int(cap["threshold_bin"][0, 2]) == want
    if B >= 4096:
        assert want > 512   # the interpolation reached buckets tiles away
    assert np.isnan(cap["threshold_value"][0, 2]) and cap["lo"][0, 2] == -1 and cap["hi"][0, 2] == -1
    assert cap["num_pos_examples"][0, 2] == int((wn >= step).sum())


# ---- trees against the oracle ----------------------------------------------------------------------------------------

def oracle_train(*args, **kw):
    """tests/test_gpu_wide_columns.oracle_train with the oracle's categories of EQUAL sort keys in index order, as the
    engine sorts them (DESIGN.md §9).  A node below a categorical split holds some categories with no rows, whose keys
    are all 0: the reference's std::sort (libstdc++ above 16 elements) may order them differently, which changes the
    positive set on categories the node does not hold, not the node's partition."""
    O.set_stable_category_sort(True)
    try:
        return _oracle_train(*args, **kw)
    finally:
        O.set_stable_category_sort(False)


def disc_table(n, seed, task="binary", sizes=(1024, 4096)):
    """Byte discretized, 16-bit discretized (missing values), wide exact and two byte categorical columns (12 and 40
    categories).
    -> (columns, uint16 bins [F, n], feature types, labels, raw values)."""
    rng = np.random.default_rng(seed)
    raw, cols, margin = [], [], np.zeros(n)
    x = rng.normal(size=n).astype(np.float32)
    raw.append(x)
    cols.append(dataspec.infer_column("b0", x, 64))
    margin += 0.5 * np.tanh(x)
    for j, B in enumerate(sizes):
        x = (rng.normal(size=n) * (1 + j)).astype(np.float32)
        x[rng.random(n) < 0.05] = np.nan
        raw.append(x)
        cols.append(dataspec.infer_column16(f"d{j}", x, B))
        margin += 1.5 * np.sin(np.nan_to_num(x, nan=0.3) * (2.0 + j))
    grid = np.sort(rng.choice(100000, size=2000, replace=False)).astype(np.float32) / 7.0
    x = grid[rng.integers(0, 2000, size=n)]
    raw.append(x)
    cols.append(dataspec.infer_column_lossless("e0", x, max_distinct=65535))
    margin += 0.8 * np.cos(x / grid.max() * 5.0)
    bins = [c.encode16(v) for c, v in zip(cols, raw)]
    types = [0] * len(cols)
    for name, k in (("c0", 12), ("c1", 40)):
        c = rng.integers(0, k, size=n)
        margin += 0.7 * rng.normal(size=k)[c]
        cols.append(dataspec.CategoricalColumn(name=name, vocabulary=["<OOD>"] + [str(i) for i in range(1, k)],
                                               counts=[0] * k, num_bins=k, na_bin=1))
        bins.append(c.astype(np.uint16))
        raw.append(c)
        types.append(1)
    margin += rng.normal(scale=0.5, size=n)
    if task == "binary":
        y = (margin > np.median(margin)).astype(np.int32) + 1
    elif task == "multi":
        y = np.digitize(margin, np.quantile(margin, [1 / 3, 2 / 3])).astype(np.int32) + 1
    else:
        y = margin.astype(np.float32)
    assert all(cols[1 + j].num_bins > 256 for j in range(len(sizes)))
    return cols, np.stack(bins), np.array(types, np.int32), y, raw


def engine_dataset(cols, bins):
    ds = dataspec.device_dataset(bins, cols)
    for f, c in enumerate(cols):
        if getattr(c, "bucket_values", None) is not None and not c.wide:
            ds.set_bucket_values(f, c.bucket_values, c.mean)
    return ds


CASES = {
    "variance": dict(),
    "hessian": dict(use_hessian_gain=1),
    "regression": dict(loss=1),
    "regression_hessian": dict(loss=1, use_hessian_gain=1),
    "subsample": dict(subsample=0.6),
    "goss": dict(goss_alpha=0.2, goss_beta=0.1),
    "no_sibling_subtraction": dict(sibling_subtraction=0),
    "depth8": dict(max_depth=8),
}


def _assert_trees(gbt, ref, n_trees, disc):
    used = 0
    for i in range(n_trees):
        got, want = gbt.get_tree(i), ref["trees"][i]
        errs = compare_trees(got, want)
        assert not errs, (i, errs[:5])
        used += sum(int(f in disc) for f in want["feature"][want["feature"] >= 0])
        sp = np.isin(got["feature"], list(disc))
        assert np.isnan(got["threshold_value"][sp]).all()
    assert used > 0, "no split on a discretized wide column"


@pytest.mark.parametrize("case", sorted(CASES))
def test_trees_match_oracle(case):
    kw = dict(max_depth=6, num_trees=4)
    kw.update(CASES[case])
    cols, bins, types, y, _ = disc_table(60000, seed=len(case), task="regression" if kw.get("loss") == 1 else "binary")
    ds = engine_dataset(cols, bins)
    assert list(ds.feature_types) == list(types)
    cfg = ydf_b200.default_config(**kw)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(y)
    gbt.train(cfg.num_trees)
    ref = oracle_train(cols, bins, types, y, cfg, cfg.num_trees)
    _assert_trees(gbt, ref, cfg.num_trees, {1, 2})
    for i in range(cfg.num_trees):
        assert abs(gbt.train_loss(i)[0] - ref["loss"][i]) <= 1e-5 * max(1.0, abs(ref["loss"][i]))


def test_weighted_trees_match_oracle():
    cols, bins, types, y, _ = disc_table(60000, seed=41)
    w = np.random.default_rng(5).random(len(y)).astype(np.float32) * 2 + 0.1
    cfg = ydf_b200.default_config(max_depth=6, num_trees=3)
    gbt = ydf_b200.Gbt(engine_dataset(cols, bins), cfg)
    gbt.set_weights(w)
    gbt.set_labels(y)
    gbt.train(3)
    _assert_trees(gbt, oracle_train(cols, bins, types, y, cfg, 3, weights=w), 3, {1, 2})


def test_multinomial_trees_match_oracle():
    for hess in (0, 1):
        cols, bins, types, y, _ = disc_table(50000, seed=43 + hess, task="multi")
        cfg = ydf_b200.default_config(loss=2, num_classes=3, max_depth=5, num_trees=2, use_hessian_gain=hess)
        gbt = ydf_b200.Gbt(engine_dataset(cols, bins), cfg)
        gbt.set_labels(y)
        gbt.train(2)
        _assert_trees(gbt, oracle_train(cols, bins, types, y, cfg, 2), 6, {1, 2})


def test_best_first_trees_match_oracle():
    cols, bins, types, y, _ = disc_table(60000, seed=47)
    cfg = ydf_b200.default_config(max_depth=6, num_trees=3, growing_strategy=1, max_num_nodes=20)
    gbt = ydf_b200.Gbt(engine_dataset(cols, bins), cfg)
    gbt.set_labels(y)
    gbt.train(3)
    _assert_trees(gbt, oracle_train(cols, bins, types, y, cfg, 3, best_first=20), 3, {1, 2})


# ---- model, prediction, learner --------------------------------------------------------------------------------------

def test_saved_model_and_predictions_agree():
    """The learner at 1024 bins: the saved model's dataspec holds the wide column's boundaries, its splits are
    DiscretizedHigher bin thresholds, and the model file, model.predict and ygg_gbt_predict on a held-out dataset (the
    validation walk's codes, NaN in the mean's bin) give the same scores."""
    cols, bins, types, y, raw = disc_table(40000, seed=53)
    names = [c.name for c in cols]
    data = {nm: v for nm, v, c in zip(names, raw, cols) if c.feature_type != 1}
    data["y"] = np.where(y == 2, "a", "b")
    rng = np.random.default_rng(3)
    train = rng.random(len(y)) < 0.8
    tr = {k: v[train] for k, v in data.items()}
    te = {k: v[~train] for k, v in data.items()}
    model = ydf_b200.GradientBoostedTreesLearner(label="y", discretize_numerical_columns=True,
                                                 num_discretized_numerical_bins=1024, num_trees=15,
                                                 validation_ratio=0.0).train(tr, valid=te)
    wide = [i for i, c in enumerate(model.data_spec.columns) if c.wide]
    assert wide and all(model.data_spec.columns[i].bucket_values is None for i in wide)
    assert any(int(f) in wide for t in model.trees for f in t["feature"][t["feature"] >= 0])
    p_host = model.predict(te)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "m")
        model.save(path)
        m = model_io.read_ydf_model(path)
        raw_io = model_io.predict_ydf_model(m, {k: v for k, v in te.items() if k != "y"})
        spec = [model_io.pb_decode(v) for f, _, v in model_io.pb_decode(open(os.path.join(path, "data_spec.pb"), "rb").read())
                if f == 1]
    for i in wide:   # DiscretizedNumericalSpec.maximum_num_bins: the budget asked for
        assert model_io._one(model_io.pb_decode(model_io._one(spec[i + 1], 8)), 3) == 1024
    for i in wide:   # column 0 is the label
        np.testing.assert_array_equal(m["columns"][i + 1]["boundaries"], model.data_spec.columns[i].boundaries)
    on_wide = [nd for nd in m["nodes"] if nd.get("attribute", 0) - 1 in wide]
    assert on_wide and all("discretized_threshold" in nd for nd in on_wide)
    assert max(nd["discretized_threshold"] for nd in on_wide) > 255
    np.testing.assert_allclose(1 / (1 + np.exp(-raw_io.astype(np.float64))), p_host, rtol=0, atol=1e-6)
    # the engine's own prediction walk over the same held-out rows
    vb = dataspec.encode_features(te, model.data_spec.columns)
    vds = dataspec.device_dataset(vb, model.data_spec.columns)
    full = dataspec.device_dataset(dataspec.encode_features(tr, model.data_spec.columns), model.data_spec.columns)
    gbt = ydf_b200.Gbt(full, ydf_b200.default_config(max_depth=6, num_trees=5))
    gbt.set_labels(np.where(tr["y"] == "a", 2, 1).astype(np.int32))
    gbt.train(5)
    host = ydf_b200.model.GradientBoostedTreesModel(model.data_spec, [gbt.get_tree(i) for i in range(5)],
                                                    gbt.initial_prediction(), "BINOMIAL_LOG_LIKELIHOOD")
    np.testing.assert_allclose(gbt.predict(vds), host._raw(vb), rtol=0, atol=1e-5)


def test_learner_on_adult_at_1024_bins_matches_the_oracle():
    """The learner end to end on the Adult numerical columns with num_discretized_numerical_bins=1024 (fnlwgt becomes a
    discretized wide column): the trees the oracle grows on the same dataspec and hold-out, tree for tree."""
    data = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "adult_numerical.npz"))
    names = ("age", "fnlwgt", "capital_gain", "capital_loss", "hours_per_week")
    cols = {nm: data[f"train_{nm}"].astype(np.float32) for nm in names}
    cols["income"] = data["train_income"]
    kw = dict(num_trees=8, validation_ratio=0.0, max_depth=5)
    model = ydf_b200.GradientBoostedTreesLearner(label="income", discretize_numerical_columns=True,
                                                 num_discretized_numerical_bins=1024, **kw).train(cols)
    spec = model.data_spec.columns
    assert spec[1].wide and spec[1].num_bins > 256
    bins = np.stack([c.encode16(cols[c.name]) for c in spec])
    want_cols = [dataspec.infer_column16(c.name, cols[c.name], 1024) for c in spec]
    for c, w in zip(spec, want_cols):
        np.testing.assert_array_equal(c.boundaries, w.boundaries)
    y = np.array([model.data_spec.label_classes.index(v) + 1 for v in cols["income"].tolist()], np.int32)
    cfg = ydf_b200.default_config()
    for k, _ in cfg._fields_:
        if k != "reserved":
            setattr(cfg, k, model.config[k])
    ref = oracle_train(spec, bins, np.zeros(len(spec), np.int32), y, cfg, cfg.num_trees)
    assert model.num_trees() == cfg.num_trees
    used = 0
    for i in range(model.num_trees()):
        errs = compare_trees(model.trees[i], ref["trees"][i])
        assert not errs, (i, errs[:5])
        used += int((model.trees[i]["feature"] == 1).sum())
    assert used > 0


# ---- memory ----------------------------------------------------------------------------------------------------------

def test_oversize_configuration_returns_the_allocation_error():
    """200 discretized wide columns of 65535 bins at depth 10: (512 slots + 2 x 512 nodes) x 13.1 M buckets x 12 B is far
    beyond the card; ygg_gbt_create reports the size instead of faulting."""
    n, F = 4096, 200
    ds = ydf_b200.Dataset(np.zeros((F, n), np.uint8), [1] * F, [0] * F)
    codes = (np.arange(n) % 65535).astype(np.uint16)
    for f in range(F):
        ds.set_wide_discretized_column(f, codes, 65535, 0)
    with pytest.raises(ydf_b200.YggError, match="GB of histogram planes"):
        ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=10))
    ds.close()


# ---- validation, early stopping and DART against the oracle's training loop ----------------------------------------

def oracle_validated(cols, bins, types, y, cfg, dart=None):
    """oracle.gbt_train_validated on the uint16 codes (the oracle's hold-out draw: 0.2 of the rows), exact-rule columns
    with their bucket values, categories of equal keys in index order, DART when `dart` is a rate."""
    O.set_bucket_values([getattr(c, "bucket_values", None) for c in cols], [getattr(c, "mean", 0.0) for c in cols])
    O.set_stable_category_sort(True)
    if dart is not None:
        O.set_dart(dart)
    try:
        return O.gbt_train_validated(bins, [c.num_bins for c in cols], [c.na_bin for c in cols], y, _oracle_cfg(cfg), 0.2,
                                     num_threads=4, feature_type=types)
    finally:
        O.set_dart(None)
        O.set_stable_category_sort(False)
        O.set_bucket_values(None)


def noisy_labels(y, seed):
    """Labels a depth-6 model overfits within a few dozen iterations: 30 % flipped classes, or heavy noise."""
    rng = np.random.default_rng(seed)
    if y.dtype.kind == "f":
        return (y + rng.normal(scale=3.0, size=len(y))).astype(np.float32)
    return np.where(rng.random(len(y)) < 0.3, 3 - y, y).astype(np.int32)


def leaf_nodes(tree, bins):
    """The leaf every column of `bins` ([F, n] codes, byte or uint16) reaches in `tree`."""
    rows = np.arange(bins.shape[1])
    node = np.zeros(bins.shape[1], np.int64)
    while True:
        f = tree["feature"][node]
        act = np.nonzero(f >= 0)[0]
        if len(act) == 0:
            return node
        nd = node[act]
        v = bins[f[act], rows[act]].astype(np.int64)
        go = v >= tree["threshold_bin"][nd]
        cat = tree["condition_type"][nd] == 1
        vc = v[cat]
        go[cat] = ((tree["cat_mask"][nd[cat], vc >> 5] >> (vc & 31).astype(np.uint32)) & 1) != 0
        node[act] = np.where(go, tree["pos_child"][nd], tree["neg_child"][nd])


def engine_validated(cols, bins, y, cfg, dart=None):
    full = engine_dataset(cols, bins)
    m = ydf_b200.validation_split_mask(cfg.random_seed, len(y), 0.2)
    tr, va = full.split_rows(m)
    full.close()
    gbt = ydf_b200.Gbt(tr, cfg)
    if dart is not None:
        gbt.set_dart(dart)
    gbt.set_labels(y[m])
    gbt.set_validation(va, y[~m])
    gbt.train(cfg.num_trees)
    return gbt, m, tr, va


def _assert_run(gbt, ref, disc):
    assert gbt.num_iterations() == ref["num_entries"] and gbt.num_trees() == len(ref["trees"])
    _assert_trees(gbt, ref, gbt.num_trees(), disc)
    for i in range(gbt.num_iterations()):
        tl, _ = gbt.train_loss(i)
        vl, vs = gbt.validation_loss(i)
        assert abs(tl - ref["train_loss"][i]) <= 1e-5 * abs(ref["train_loss"][i])
        assert abs(vl - ref["valid_loss"][i]) <= 1e-5 * abs(ref["valid_loss"][i])
        assert abs(vs - ref["valid_secondary"][i]) <= 1e-5 * max(1.0, abs(ref["valid_secondary"][i]))
    fv, trig = gbt.final_validation()
    assert trig == ref["early_stopping_triggered"]
    assert abs(fv - ref["validation_loss"]) <= 1e-5 * abs(ref["validation_loss"])


@pytest.mark.parametrize("loss,policy", [(0, 0), (0, 1), (0, 2), (1, 2)])
def test_validation_and_early_stopping_match_oracle(loss, policy):
    """The validation walk (k_valid_update on the held-out rows' uint16 codes), its losses, the early-stopping decision
    and the truncated model against the oracle's training loop, for each policy (0 NONE, 1 MIN_LOSS_FINAL, 2
    LOSS_INCREASE)."""
    n = 12000
    cols, bins, types, y, _ = disc_table(n, seed=70 + 3 * loss + policy, task="regression" if loss == 1 else "binary")
    y = noisy_labels(y, n + policy)
    cfg = ydf_b200.default_config(loss=loss, num_trees=40, max_depth=6, shrinkage=0.3, min_examples=2,
                                  early_stopping=policy, early_stopping_num_trees_look_ahead=12,
                                  early_stopping_initial_iteration=4, rng_words_consumed=n)
    ref = oracle_validated(cols, bins, types, y, cfg)
    gbt, m, tr, va = engine_validated(cols, bins, y, cfg)
    np.testing.assert_array_equal(m, ref["in_training"])
    _assert_run(gbt, ref, {1, 2})
    if policy == 2:
        assert gbt.num_iterations() < cfg.num_trees, "the problem is meant to stop early"
    # ygg_gbt_predict on the held-out rows: the host walk of the kept trees over the same codes
    host = ydf_b200.model.GradientBoostedTreesModel(
        dataspec.DataSpec(columns=cols, label="y", task="CLASSIFICATION" if loss == 0 else "REGRESSION"),
        [gbt.get_tree(i) for i in range(gbt.num_trees())], gbt.initial_prediction(),
        "BINOMIAL_LOG_LIKELIHOOD" if loss == 0 else "SQUARED_ERROR")
    np.testing.assert_allclose(gbt.predict(va), host._raw(bins[:, ~m]), rtol=0, atol=1e-5)
    for d in (gbt, tr, va):
        d.close()


@pytest.mark.parametrize("loss,rate,policy", [(0, 0.1, 2), (1, 0.5, 0), (0, 1.0, 1)])
def test_dart_matches_oracle(loss, rate, policy):
    """DART (per-iteration dropout, rescaled trees) on the mixed table against the oracle's DART loop: every tree,
    dropped set, weight (bitwise), loss and stopping point, and the scaled model's held-out scores."""
    from tests import dart_ref as D
    n = 10000
    cols, bins, types, y, _ = disc_table(n, seed=90 + loss, task="regression" if loss == 1 else "binary")
    y = noisy_labels(y, n)
    cfg = ydf_b200.default_config(loss=loss, num_trees=40, max_depth=6, shrinkage=0.3, min_examples=2,
                                  early_stopping=policy, early_stopping_num_trees_look_ahead=12,
                                  early_stopping_initial_iteration=4, rng_words_consumed=n, split_jobs_draw_seeds=1)
    ref = oracle_validated(cols, bins, types, y, cfg, dart=rate)
    gbt, m, tr, va = engine_validated(cols, bins, y, cfg, dart=rate)
    for i in range(min(gbt.num_iterations(), ref["num_entries"])):
        assert gbt.dart_dropped(i).tolist() == ref["dart_dropped"][i], i
    _assert_run(gbt, ref, {1, 2})
    assert np.array_equal(gbt.dart_weights(), ref["dart_weights"])
    vbins = bins[:, ~m]
    nodes = [leaf_nodes(ref["trees"][t], vbins) for t in range(len(ref["trees"]))]
    want = D.scaled_sum(np.float32(gbt.initial_prediction()),
                        np.stack([gbt.get_tree(t)["leaf_value"][nd] for t, nd in enumerate(nodes)]), ref["dart_weights"], 1)
    assert np.array_equal(gbt.predict(va)[None], want)
    for d in (gbt, tr, va):
        d.close()


def test_builder_dataset_takes_a_held_out_dataset_made_in_feature_order():
    """The GPU binning step attaches its 16-bit columns when the builder finishes, so a wide column set on the finished
    dataset comes after them in its wide order.  A held-out dataset made column by column in feature order has the
    same features: set_validation and predict() accept it and route its rows by its own codes; a dataset whose wide
    column at a feature is of another kind is still refused."""
    from tests import boost_ref as R
    rng = np.random.default_rng(61)
    n, nv = 20000, 3000
    x = rng.normal(size=n + nv).astype(np.float32)
    codes = rng.integers(0, 600, size=n + nv).astype(np.uint16)
    values = np.arange(600, dtype=np.float32)
    b = ydf_b200.DatasetBuilder(n, 2)
    b.add_bins(0, np.zeros(n, np.uint8), 1, 0)
    b.add_numerical16_async(1, x[:n], 4096, 3)
    col = dataspec.infer_column16("x", x[:n], 4096)
    ds = b.finish()
    ds.set_wide_column(0, codes[:n], 600, 0, values, 0.0)
    assert col.wide and ds.wide == {1: (col.num_bins, col.na_bin), 0: (600, 0)}
    enc = col.encode16(x[n:])
    va = ydf_b200.Dataset(np.zeros((2, nv), np.uint8), [1, 1], [0, 0])
    va.set_wide_column(0, codes[n:], 600, 0, values, 0.0)
    va.set_wide_discretized_column(1, enc, col.num_bins, col.na_bin)
    y = ((np.sin(2 * x) + codes / 300.0 + rng.normal(scale=0.3, size=n + nv)) > 1).astype(np.int32) + 1
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=4, num_trees=3))
    gbt.set_labels(y[:n])
    gbt.set_validation(va, y[n:])
    gbt.train(3)
    cols = [("wide_num", codes[n:], 600, values), ("wide_num", enc, col.num_bins, None)]
    want = np.full(nv, np.float32(gbt.initial_prediction()), np.float32)
    for t in range(3):
        tree = gbt.get_tree(t)
        want = (want + tree["leaf_value"][R.leaf_of_rows(tree, R.route(tree, cols), nv)]).astype(np.float32)
    assert {0, 1} <= set(np.concatenate([gbt.get_tree(t)["feature"] for t in range(3)]).tolist())
    assert np.array_equal(gbt.predict(va), want)
    other = ydf_b200.Dataset(np.zeros((2, nv), np.uint8), [1, 1], [0, 0])
    other.set_wide_column(0, codes[n:], 600, 0, values, 0.0)
    other.set_wide_column(1, enc, col.num_bins, 0, np.arange(col.num_bins, dtype=np.float32), 0.0)
    with pytest.raises(ydf_b200.YggError, match="features / binning"):
        gbt.predict(other)
    for d in (gbt, ds, va, other):
        d.close()


# ---- mixed with wide categorical and presorted columns; candidate sampling ---------------------------------------------

def mixed_wide(rng, n):
    """Byte numerical and categorical columns, a discretized wide column of 4096 bins (feature 2), a wide categorical one
    of 300 categories (3), a presorted float column (4) and a wide exact column of 600 buckets (5).
    -> (dataset, route column descriptions, gradients)."""
    bins, nb, ft = mixed_bins(rng, n, [("num", 64), ("cat", 9), ("num", 1), ("cat", 1), ("num", 1), ("num", 1)])
    ds = ydf_b200.Dataset(bins, nb, np.zeros(6, np.int32), feature_types=ft)
    x = rng.normal(size=n).astype(np.float32)
    x[rng.random(n) < 0.05] = np.nan
    col = dataspec.infer_column16("d", x, 4096)
    dn = col.encode16(x)
    ds.set_wide_discretized_column(2, dn, col.num_bins, col.na_bin)
    wc = rng.integers(0, 300, size=n).astype(np.uint16)
    ds.set_wide_categorical_column(3, wc, 300, 0)
    pv = np.round(rng.normal(size=n), 2).astype(np.float32)
    ds.set_numerical_column(4, pv, float(pv.mean()))
    wn = np.minimum(rng.geometric(0.01, size=n) - 1, 599).astype(np.uint16)
    values = np.arange(600, dtype=np.float32)
    ds.set_wide_column(5, wn, 600, 0, values, 0.0)
    cols = byte_cols(bins, nb, ds.feature_types)
    cols[2] = ("wide_num", dn, col.num_bins, None)
    cols[3] = ("wide_cat", wc, 300, None)
    cols[4] = ("pre", ds.get_numerical_column(4), 0, None)
    cols[5] = ("wide_num", wn, 600, values)
    effect = rng.normal(size=300) * (np.arange(300) < 40)
    g = (bins[0] / 64.0 + 1.2 * np.sin(3 * np.nan_to_num(x)) + effect[wc] + 0.5 * pv + 0.004 * wn +
         rng.normal(scale=0.5, size=n)).astype(np.float32)
    return ds, cols, g


@pytest.mark.parametrize("hessian", [0, 1])
def test_mixed_wide_kinds_match_the_exact_scan(hessian):
    """Every candidate of every level with discretized wide, wide categorical, presorted and wide exact columns in one
    table, against the exact scan reference."""
    rng = np.random.default_rng(101 + hessian)
    ds, cols, g = mixed_wide(rng, 120000)
    cfg = ydf_b200.default_config(loss=1, max_depth=6, min_examples=5, use_hessian_gain=hessian)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(g)
    gbt.capture_candidates(True)
    tree = gbt.train_tree_on_gradients(g)
    assert check_scan(gbt, cfg, tree, cols, g, None) > 0
    used = set(tree["feature"][tree["feature"] >= 0].tolist())
    assert {2, 3} <= used and used & {4, 5}


def test_candidate_sampling_with_discretized_wide_columns():
    """Candidate feature sampling: every level's selection among the sampled features and every validity flag against
    the restatement (tests/test_gpu_candidate_sampling.check_levels), with the mixed wide table."""
    from tests.test_gpu_candidate_sampling import check_levels, k_valid
    rng = np.random.default_rng(103)
    ds, cols, g = mixed_wide(rng, 60000)
    cfg = ydf_b200.default_config(loss=1, max_depth=6, min_examples=1, candidate_shuffle=0)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(g)
    gbt.set_candidate_sampling(3, None)
    gbt.capture_candidates(True)
    tree = gbt.train_tree_on_gradients(g)
    assert 2 in set(tree["feature"][tree["feature"] >= 0].tolist())
    nodes, flags, _ = check_levels(gbt, cfg, tree, 0, k_valid(cfg, ds.n_features, 3), cols, g)
    assert nodes >= 7 and flags > 0
