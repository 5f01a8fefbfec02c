"""Presorted numerical columns (DESIGN.md §22) on the GPU: the reference's known answers for the exact numerical
splitter, trees equal to the byte / wide bucket paths (and the oracle) on columns of at most 65535 values, every split of
trees on continuous columns far beyond 65535 values against a numpy exact splitter, the learner end to end, prediction
and model files, the refusals and the lists' memory."""
import os
import tempfile

import numpy as np
import pytest

import ydf_b200
from ydf_b200 import _capi, dataspec, model_io
from tests import presort_ref as PR
from tests import reference_replay as R
from tests import test_gpu_wide_columns as WC
from tests.util import compare_trees, pow2_cover, prune_noise_splits, quantize_q24, quantize_second

pytestmark = pytest.mark.gpu

NAN = np.float32(np.nan)


def presorted_dataset(values, na_replacements, byte=None, byte_bins=()):
    """Presorted columns 0..len(values)-1, then the byte columns `byte` [k, n] with `byte_bins` buckets."""
    n = len(values[0])
    F = len(values) + (0 if byte is None else len(byte))
    bins = np.zeros((F, n), np.uint8)
    if byte is not None:
        bins[len(values):] = byte
    ds = ydf_b200.Dataset(bins, [1] * len(values) + list(byte_bins), [0] * F)
    for f, (v, na) in enumerate(zip(values, na_replacements)):
        ds.set_numerical_column(f, v, na)
    return ds


# ---- the reference's known answers ------------------------------------------------------------------------------------

KA_X = np.array([2, 3, 0, 1, NAN, NAN], np.float32)   # decision_tree_test.cc:947-995, NA replacement 2
KA_Y = np.array([1, 1, 0, 0, 1, 0], np.float32)


def test_known_answer_unweighted():
    ds = presorted_dataset([KA_X], [2.0])
    np.testing.assert_array_equal(ds.get_numerical_column(0), [2, 3, 0, 1, 2, 2])
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(loss=1, max_depth=2, min_examples=1))
    gbt.set_labels(KA_Y)
    t = gbt.train_tree_on_gradients(KA_Y)   # the labels as gradients
    root = t[0]
    assert (root["feature"], root["condition_type"], root["threshold_bin"]) == (0, 2, -1)
    assert root["threshold_value"] == np.float32(1.5)
    assert (root["num_examples"], root["num_pos_examples"], root["na_value"]) == (6, 4, 1)
    np.testing.assert_allclose(root["split_score"], 0.125, rtol=1e-5)


def test_known_answer_weighted():
    """Weights 1..6 through one iteration of a weighted squared-error handle: g = y - weighted mean, whose variance score
    is the labels'."""
    ds = presorted_dataset([KA_X], [2.0])
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(loss=1, max_depth=2, min_examples=1, num_trees=1))
    gbt.set_weights(np.arange(1, 7, dtype=np.float32))
    gbt.set_labels(KA_Y)
    gbt.train(1)
    root = gbt.get_tree(0)[0]
    assert (root["feature"], root["condition_type"], root["threshold_value"]) == (0, 2, np.float32(1.5))
    assert (root["num_examples"], root["num_pos_examples"], root["na_value"]) == (6, 4, 1)
    np.testing.assert_allclose(root["split_score"], 0.0725623, rtol=1e-5)


def test_known_answer_two_levels():
    """training_test.cc:122-191: f1 >= 2.5 [s:0.347222 n:6 np:4], then f2 >= 1.5 [s:0.0625 n:4 np:2] on its positive side."""
    f1 = np.array([1, 2, 3, 4, 3, 4], np.float32)
    f2 = np.array([1, 2, 1, 1, 2, 2], np.float32)
    y = np.array([0, 0, 1, 1, 1.5, 1.5], np.float32)
    ds = presorted_dataset([f1, f2], [float(f1.mean()), float(f2.mean())])
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(loss=1, max_depth=3, min_examples=1))
    gbt.set_labels(y)
    t = gbt.train_tree_on_gradients(y)
    root = t[0]
    assert (root["feature"], root["threshold_value"], root["num_examples"], root["num_pos_examples"]) == (0, 2.5, 6, 4)
    np.testing.assert_allclose(root["split_score"], 0.347222, rtol=1e-5)
    pos = t[root["pos_child"]]
    assert (pos["feature"], pos["threshold_value"], pos["num_examples"], pos["num_pos_examples"]) == (1, 1.5, 4, 2)
    np.testing.assert_allclose(pos["split_score"], 0.0625, rtol=1e-5)
    assert t[root["neg_child"]]["feature"] == -1


# ---- equal to the bucket paths on columns of at most 65535 values -----------------------------------------------------

def presorted_copy(cols, bins, raw):
    """The same table with every numerical column presorted (its lossless mean as NA replacement): -> (columns, float64
    matrix as encode_features makes it)."""
    pcols, rows, k = [], [], 0
    for f, c in enumerate(cols):
        if c.feature_type == _capi.FEATURE_CATEGORICAL:
            pcols.append(c)
            rows.append(bins[f].astype(np.float64))
            continue
        x = raw[k] if c.name != "twin" else raw[0]
        k += c.name != "twin"
        p = dataspec.infer_column_presorted(c.name, x)
        assert p.mean == c.mean
        pcols.append(p)
        rows.append(x.astype(np.float64))
    return pcols, np.stack(rows)


def assert_same_trees(a, b):
    """Every ygg_node field equal (threshold_value to the bit), but threshold_bin / condition_type of the presorted splits.
    -> the number of presorted splits."""
    assert len(a) == len(b)
    pre = (b["feature"] >= 0) & (b["condition_type"] == 2)
    assert ((a["condition_type"][pre] == 0) & (b["threshold_bin"][pre] == -1)).all()
    for name in a.dtype.names:
        x, y = a[name], b[name]
        if name in ("threshold_bin", "condition_type"):
            x, y = x[~pre], y[~pre]
        if x.dtype.kind == "f":   # floats to the bit (NaN included)
            u = np.uint32 if x.dtype.itemsize == 4 else np.uint64
            x, y = x.view(u), y.view(u)
        assert np.array_equal(x, y), name
    return int(pre.sum())


EQ_CASES = {
    "variance": dict(),
    "hessian": dict(use_hessian_gain=1),
    "regression": dict(loss=1),
    "depth2": dict(max_depth=2),
    "depth10": dict(max_depth=10, min_examples=5),
    "min_examples_400": dict(min_examples=400, max_depth=8),
    "subsample": dict(subsample=0.6),
    "goss": dict(goss_alpha=0.2, goss_beta=0.1),
    "no_sibling_subtraction": dict(sibling_subtraction=0),
    "tie_shuffle_twins": dict(candidate_shuffle=2, split_jobs_draw_seeds=1),
    "weighted": dict(weights=1, loss=1),
    "multinomial": dict(loss=2, num_classes=3, max_depth=5, num_trees=2),
    "best_first": dict(growing_strategy=1, max_num_nodes=20),
}


@pytest.mark.parametrize("case", sorted(EQ_CASES))
def test_presorted_trees_equal_the_bucket_paths(case):
    """The wide_table columns (3 byte and 2 wide lossless columns, one categorical) once through the byte / wide paths and
    once presorted: the same trees, losses and predictions, and the oracle's trees on the bucket codes."""
    kw = dict(max_depth=6, num_trees=4)
    kw.update(EQ_CASES[case])
    weighted = bool(kw.pop("weights", 0))
    task = {1: "regression", 2: "multi"}.get(kw.get("loss"), "binary")
    n = 200000 if case == "depth10" else 60000
    cols, bins, types, y, raw = WC.wide_table(n, seed=500 + sorted(EQ_CASES).index(case), task=task)
    if case.startswith("tie_shuffle"):   # a twin of the first column: equal scores on every node, the replay decides
        twin = dataspec.infer_column_lossless("twin", raw[0])
        cols, bins, types = cols + [twin], np.vstack([bins, bins[:1]]), np.append(types, 0).astype(np.int32)
    pcols, pbins = presorted_copy(cols, bins, raw)
    cfg = ydf_b200.default_config(**kw)
    w = np.random.default_rng(5).random(n).astype(np.float32) * 2 + 0.1 if weighted else None
    runs = []
    for ds in (WC.engine_dataset(cols, bins, types), dataspec.device_dataset(pbins, pcols)):
        gbt = ydf_b200.Gbt(ds, cfg)
        if w is not None:
            gbt.set_weights(w)
        gbt.set_labels(y)
        gbt.train(cfg.num_trees)
        runs.append((gbt, ds))
    (ga, _), (gb, dsb) = runs
    assert list(dsb.feature_types) == [2 if c.feature_type == 2 else c.feature_type for c in pcols]
    presorted = 0
    for i in range(ga.num_trees()):
        presorted += assert_same_trees(ga.get_tree(i), gb.get_tree(i))
    for i in range(cfg.num_trees):
        assert ga.train_loss(i) == gb.train_loss(i)
    assert np.array_equal(ga.get_predictions(), gb.get_predictions())
    assert presorted > 0
    if case.startswith("tie_shuffle"):
        assert gb.tie_stats()[0] > 0   # nodes renamed to a verified twin
    ref = WC.oracle_train(cols, bins, types, y, cfg, cfg.num_trees, weights=w,
                          best_first=kw.get("max_num_nodes") if kw.get("growing_strategy") else None)
    for i in range(gb.num_trees()):
        got, want = gb.get_tree(i).copy(), ref["trees"][i]
        # the oracle's codes are buckets: the presorted splits' bucket thresholds are the bucket path's (equal above)
        bucket = ga.get_tree(i)
        got["threshold_bin"], got["condition_type"] = bucket["threshold_bin"], bucket["condition_type"]
        if case == "depth10":
            got, want = prune_noise_splits(got, 1e-12), prune_noise_splits(want, 1e-12)
        errs = compare_trees(got, want)
        assert not errs, (case, i, errs[:5])


# ---- beyond 65535 values: every split against the numpy exact splitter ------------------------------------------------

def continuous_table(n, seed):
    """Two continuous columns (all values distinct, then 10 % of the rows on repeated values, 5 % missing), a byte
    column; -> (raw values, stored values, means, byte codes, margin)."""
    rng = np.random.default_rng(seed)
    a = rng.normal(size=n).astype(np.float32)
    b = (rng.random(n) * 1000).astype(np.float32)
    for x in (a, b):
        rep = rng.random(n) < 0.1
        x[rep] = np.round(x[rep], 1)
    c = rng.integers(0, 32, size=n).astype(np.uint8)
    margin = np.sin(3 * a) + (b > 400) * 0.8 + 0.01 * c + rng.normal(scale=0.3, size=n)
    for x in (a, b):
        x[rng.random(n) < 0.05] = np.nan
    raw = [a, b]
    means = [dataspec.infer_column_presorted(f"x{i}", x).mean for i, x in enumerate(raw)]
    stored = [np.where(np.isnan(x), np.float32(m), x).astype(np.float32) for x, m in zip(raw, means)]
    assert all(len(np.unique(x[~np.isnan(x)])) > 65535 for x in raw)
    return raw, stored, means, c, margin


def rows_of_nodes(tree, stored, byte):
    rows = [None] * len(tree)
    rows[0] = np.arange(len(stored[0]))
    for i in range(len(tree)):
        t = tree[i]
        if t["feature"] < 0:
            continue
        r = rows[i]
        if t["condition_type"] == 2:
            pos = stored[t["feature"]][r] >= t["threshold_value"]
        else:
            pos = byte[r].astype(np.int64) >= t["threshold_bin"]
        rows[t["pos_child"]], rows[t["neg_child"]] = r[pos], r[~pos]
    return rows


TREE_CASES = {
    "variance": dict(loss=1),
    "hessian": dict(loss=0, use_hessian_gain=1),
    "depth2": dict(loss=1, max_depth=2),
    "depth10": dict(loss=1, max_depth=10, min_examples=5),
    "min_examples_400": dict(loss=1, max_depth=8, min_examples=400),
    "no_sibling_subtraction": dict(loss=1, sibling_subtraction=0),
    "hessian_subtract_parent": dict(loss=0, use_hessian_gain=1, hessian_split_score_subtract_parent=1),
}


@pytest.mark.parametrize("case", sorted(TREE_CASES))
def test_every_split_beyond_65535_values_matches_the_numpy_exact_splitter(case):
    kw = dict(TREE_CASES[case])
    raw, stored, means, byte, margin = continuous_table(300000, seed=900 + sorted(TREE_CASES).index(case))
    ds = presorted_dataset(raw, means, byte[None], [32])
    cfg = ydf_b200.default_config(max_depth=kw.pop("max_depth", 6), **kw)
    gbt = ydf_b200.Gbt(ds, cfg)
    m = (margin - margin.mean()) / np.abs(margin - margin.mean()).max()
    rng = np.random.default_rng(7)
    if cfg.loss == 0:
        g, h = (0.98 * m).astype(np.float32), rng.uniform(0.01, 0.25, size=len(m)).astype(np.float32)
        gbt.set_labels((m > 0).astype(np.int32) + 1)
        P, V = 1.0, 0.25
    else:
        g, h = (3.0 * m).astype(np.float32), None
        gbt.set_labels(margin.astype(np.float32))
        P, V = float(pow2_cover(np.abs(g).max())), 1.0
    tree = gbt.train_tree_on_gradients(g, h)
    g_units = (quantize_q24(g, P) - 2 ** 23).astype(np.float64) * P / 2.0 ** 23
    h_units = None if h is None else quantize_second(h, V).astype(np.float64) * V / 2.0 ** 24
    use_hessian = bool(cfg.use_hessian_gain)
    rows = rows_of_nodes(tree, stored, byte)
    checked = 0
    for i in np.nonzero(tree["feature"] >= 0)[0]:
        t, r = tree[i], rows[i]
        assert len(r) == t["num_examples"]
        best = None
        for f in (0, 1):
            ref = PR.best_split(stored[f][r], g_units[r], None if h_units is None else h_units[r], use_hessian,
                                cfg.min_examples, subtract_parent=bool(cfg.hessian_split_score_subtract_parent))
            if t["feature"] == f:
                assert ref is not None and t["condition_type"] == 2 and t["threshold_bin"] == -1
                score, thr, n_pos = ref
                assert np.float32(t["threshold_value"]).view(np.uint32) == thr.view(np.uint32), (i, t["threshold_value"], thr)
                assert t["num_pos_examples"] == n_pos
                assert bool(t["na_value"]) == bool(np.float32(means[f]) >= thr)
                np.testing.assert_allclose(t["split_score"], score, rtol=1e-5)
                checked += 1
            elif ref is not None:
                best = max(best or 0.0, ref[0])
        if t["feature"] not in (0, 1) and best is not None:
            assert best <= t["split_score"] * (1 + 1e-5) + 1e-12, f"node {i}: a better presorted split was missed"
    assert checked > 0
    if case == "depth10":
        assert int(tree["depth"].max()) == 10


# ---- the learner end to end -------------------------------------------------------------------------------------------

def test_learner_reproduces_the_abalone_run_with_presorted_columns():
    """abalone_regression_gbdt_v2 at the reference's defaults, with presort_numerical_columns=True: the columns of more than
    255 distinct values are presorted instead of wide, and the run keeps the wide run's bars."""
    ref, data = R.load_run("abalone")
    model = ydf_b200.GradientBoostedTreesLearner(label="Rings", task="REGRESSION", presort_numerical_columns=True).train(
        {k: np.asarray(v) for k, v in data.items()})
    assert sum(c.feature_type == 2 for c in model.data_spec.columns) == 4
    logs = model.training_logs
    assert len(logs) == len(ref["log_training_loss"]) == 75 and model.num_trees() == 45
    got = np.array([e["loss"] for e in logs], np.float64)
    assert np.abs(got - ref["log_training_loss"].astype(np.float64)).max() <= 1e-5
    got = np.array([e["validation_loss"] for e in logs], np.float64)
    assert np.abs(got - ref["log_validation_loss"].astype(np.float64)).max() <= 1e-5
    assert abs(model.validation_loss - float(ref["validation_loss"])) <= 1e-5


def test_learner_on_adult_equals_the_wide_run():
    """Adult at the reference's defaults: fnlwgt presorted (presort_numerical_columns=True) gives the trees and logs of the
    max_exact_numerical_values=65535 run, where it is wide."""
    _, data = R.load_run("adult")
    L = ydf_b200.GradientBoostedTreesLearner
    a = L(label="income", max_exact_numerical_values=65535).train(data)
    b = L(label="income", presort_numerical_columns=True).train(data)
    assert [c.name for c in b.data_spec.columns if c.feature_type == 2] == ["fnlwgt"]
    assert a.training_logs == b.training_logs and a.num_trees() == b.num_trees()
    for ta, tb in zip(a.trees, b.trees):
        assert_same_trees(ta, tb)


def test_predictions_and_model_files_agree():
    """model.predict, ygg_gbt_predict and the saved model read back by predict_ydf_model, on held-out rows, values inside
    the gaps around every threshold and missing values: all three route by value >= threshold (NaN: na_value)."""
    raw, stored, means, byte, margin = continuous_table(120000, seed=77)
    y = (margin > np.median(margin)).astype(np.int32) + 1
    pcols = [dataspec.infer_column_presorted(f"x{i}", x) for i, x in enumerate(raw)]
    pcols.append(dataspec.infer_column_lossless("c", byte.astype(np.float32)))
    keep = np.random.default_rng(1).random(len(y)) < 0.8
    data = {"x0": raw[0], "x1": raw[1], "c": byte.astype(np.float32)}
    full = dataspec.device_dataset(dataspec.encode_features(data, pcols), pcols)
    tr, va = full.split_rows(keep)
    for f in (0, 1):
        np.testing.assert_array_equal(va.get_numerical_column(f), stored[f][~keep])
    gbt = ydf_b200.Gbt(tr, ydf_b200.default_config(max_depth=6, num_trees=8))
    gbt.set_labels(y[keep])
    gbt.set_validation(va, y[~keep])
    gbt.train(8)
    trees = [gbt.get_tree(i) for i in range(gbt.num_trees())]
    spec = dataspec.DataSpec(pcols, "y", "CLASSIFICATION", [1, 2], num_rows=len(y))
    model = ydf_b200.GradientBoostedTreesModel(spec, trees, gbt.initial_prediction(), "BINOMIAL_LOG_LIKELIHOOD")
    thr = np.concatenate([t["threshold_value"][(t["feature"] >= 0) & (t["condition_type"] == 2)] for t in trees])
    fs = np.concatenate([t["feature"][(t["feature"] >= 0) & (t["condition_type"] == 2)] for t in trees])
    assert len(thr) > 0
    held = {k: v[~keep] for k, v in data.items()}
    k = 3 * len(thr) + 1
    probe = {name: np.repeat(held[name][:1], k) for name in held}
    for j, (f, t) in enumerate(zip(fs, thr)):   # below, at and just above every threshold, on its own column
        for d, x in enumerate((np.nextafter(t, np.float32(-np.inf)), t, np.nextafter(t, np.float32(np.inf)))):
            probe[f"x{f}"] = probe[f"x{f}"].copy()
            probe[f"x{f}"][3 * j + d] = x
    probe["x0"][-1], probe["x1"][-1] = np.nan, np.nan
    for cols in (held, probe):
        bins = dataspec.encode_features(cols, pcols)
        host = model._raw(bins)
        pds = dataspec.device_dataset(bins, pcols)
        dev = gbt.predict(pds)
        pds.close()
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "m")
            model.save(path)
            io = model_io.predict_ydf_model(model_io.read_ydf_model(path), cols)
        # (a row routed differently would move by a whole leaf value; the sums themselves may differ in the last bit)
        np.testing.assert_allclose(dev, host, rtol=0, atol=2e-6)
        np.testing.assert_allclose(io, host, rtol=0, atol=2e-6)
    assert np.isfinite(gbt.validation_loss(7)[0])


# ---- refusals and memory ----------------------------------------------------------------------------------------------

def test_refusals_on_the_device():
    rng = np.random.default_rng(0)
    n = 5000
    ds = ydf_b200.Dataset(rng.integers(0, 8, size=(4, n)).astype(np.uint8), [8] * 4, [0] * 4, feature_types=[0, 0, 1, 0])
    v = rng.normal(size=n).astype(np.float32)
    ds.set_wide_column(3, rng.integers(0, 300, size=n).astype(np.uint16), 300, 0, np.arange(300, dtype=np.float32), 1.0)
    for feature, values in ((2, v), (3, v), (0, v[:-1]), (9, v)):   # categorical, wide, row count, out of range
        with pytest.raises(ydf_b200.YggError) as e:
            ds.set_numerical_column(feature, values, 0.0)
        assert e.value.code == 1, (feature, e.value)
    ds.set_numerical_column(0, v, 0.0)
    with pytest.raises(ydf_b200.YggError) as e:
        ds.set_numerical_column(0, v, 0.0)   # already numerical
    assert e.value.code == 1
    with pytest.raises(ydf_b200.YggError) as e:
        ds.set_feature_types([0, 0, 1, 0])   # a presorted feature stays FEATURE_NUMERICAL
    assert e.value.code == 1
    with pytest.raises(ydf_b200.YggError) as e:
        ds.partition_rows(np.arange(10, dtype=np.uint32), 0, 1)
    assert e.value.code == 4
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=4))
    with pytest.raises(ydf_b200.YggError) as e:
        ds.set_numerical_column(1, v, 0.0)   # after a handle
    assert e.value.code == 1
    for call in (lambda: gbt.set_feature_shard(0, 2, 0, 1),
                 lambda: gbt.set_row_shard(0, 1, n, 0.0, allreduce=lambda *a: 0)):
        with pytest.raises(ydf_b200.YggError) as e:
            call()
        assert e.value.code == 4
    gbt.set_labels(rng.integers(1, 3, size=n).astype(np.int32))
    other = ydf_b200.Dataset(rng.integers(0, 8, size=(4, n)).astype(np.uint8), [8] * 4, [0] * 4, feature_types=[0, 0, 1, 0])
    with pytest.raises(ydf_b200.YggError) as e:   # a validation dataset without the numerical column
        gbt.set_validation(other, rng.integers(1, 3, size=n).astype(np.int32))
    assert e.value.code == 1


def test_handles_do_not_leak_the_lists():
    """Create / destroy cycles: the master and level lists and the prefix sums (40 B per row and column) are freed with
    the handle (the pool keeps freed memory mapped and reuses it: the free figure must not fall)."""
    import torch
    n = 1 << 20
    rng = np.random.default_rng(2)
    ds = presorted_dataset([rng.normal(size=n).astype(np.float32) for _ in range(3)], [0.0] * 3)
    lists = 3 * n * 40

    def cycle():
        gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=6))
        gbt.close()
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info(0)[0]

    first = cycle()
    last = min(cycle() for _ in range(4))
    assert first - last < lists // 2, (first, last)
