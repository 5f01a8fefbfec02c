"""Presorted numerical columns (DESIGN.md §22) without a device: the learner option and its default, the column's mean
and NaN rule, the float64 matrix of encode_features, the model writer and reader on a Higher condition, the C ABI's
argument checks, and the numpy reference of the exact splitter against a brute-force loop over every cut."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

import ydf_b200
from ydf_b200 import _capi, dataspec, model_io
from ydf_b200.model import GradientBoostedTreesModel
from tests import presort_ref as PR


def test_learner_option_defaults_off_and_keeps_the_refusals():
    L = ydf_b200.GradientBoostedTreesLearner
    assert L(label="y").presort_numerical_columns is False
    assert L(label="y", presort_numerical_columns=True).presort_numerical_columns is True
    x = np.arange(1000, dtype=np.float32)
    with pytest.raises(NotImplementedError, match="more than 255 distinct values"):
        L(label="y").train({"x": x, "y": np.arange(1000) % 2})
    # a column without any present value is refused with the option on too, before anything touches the device
    with pytest.raises(NotImplementedError, match="distinct values"):
        L(label="y", presort_numerical_columns=True).train({"x": np.full(10, np.nan, np.float32), "y": np.arange(10) % 2})


def test_presorted_mean_and_nan_rule_follow_the_lossless_columns():
    rng = np.random.default_rng(3)
    x = rng.normal(size=5000).astype(np.float32)
    x[::17] = np.nan
    for max_rows in (None, 1000, 100000):
        c = dataspec.infer_column_presorted("x", x, max_rows)
        ref = dataspec.infer_column_lossless("x", np.round(x, 0), max_rows)   # (the same sample rule on a narrow copy)
        sample = x if max_rows is None else x[:max_rows]
        assert c.mean == float(sample[~np.isnan(sample)].astype(np.float64).mean())
        assert ref.mean == float(np.round(sample, 0)[~np.isnan(sample)].astype(np.float64).mean())
        assert c.num_missing == int(np.isnan(x).sum()) and c.num_values == len(x)
        assert c.num_distinct == len(np.unique(x[~np.isnan(x)]))
        assert (c.min_value, c.max_value) == (float(np.nanmin(x)), float(np.nanmax(x)))
    assert c.feature_type == _capi.FEATURE_NUMERICAL == 2
    # a sample without a present value: the mean of the distinct values, as infer_column_lossless
    y = np.concatenate([np.full(10, np.nan, np.float32), np.array([1, 2, 6], np.float32)])
    assert dataspec.infer_column_presorted("y", y, 5).mean == dataspec.infer_column_lossless("y", y, 5).mean == 3.0
    assert dataspec.infer_column_presorted("z", np.full(4, np.nan, np.float32)) is None


def test_encode_features_carries_the_raw_values():
    x = np.arange(1000, dtype=np.float32) / 7
    x[5] = np.nan
    narrow = dataspec.infer_column_lossless("a", np.arange(1000) % 10)
    wide = dataspec.infer_column_lossless("b", np.arange(1000, dtype=np.float32), max_distinct=65535)
    pre = dataspec.infer_column_presorted("c", x)
    cols = {"a": np.arange(1000) % 10, "b": np.arange(1000, dtype=np.float32), "c": x}
    out = dataspec.encode_features(cols, [narrow, wide, pre])
    assert out.dtype == np.float64 and out.shape == (3, 1000)
    assert (out[0] == narrow.encode(cols["a"])).all() and (out[1] == np.arange(1000)).all()
    np.testing.assert_array_equal(out[2], x.astype(np.float64))   # NaN kept


def _model_with_one_higher_split(thr, na_value):
    col = dataspec.PresortedColumn(name="x", mean=2.0, min_value=-3.0, max_value=9.0, num_missing=2, num_values=10,
                                   num_distinct=8)
    spec = dataspec.DataSpec(columns=[col], label="y", task="REGRESSION", num_rows=10, label_mean=1.0)
    t = np.zeros(3, dtype=_capi.NODE_DTYPE)
    t["feature"] = [0, -1, -1]
    t["neg_child"], t["pos_child"] = [1, -1, -1], [2, -1, -1]
    t["condition_type"][0] = _capi.FEATURE_NUMERICAL
    t["threshold_bin"][0] = -1
    t["threshold_value"] = [thr, np.nan, np.nan]
    t["na_value"][0] = na_value
    t["leaf_value"] = [0.0, -1.0, 1.0]
    t["num_examples"] = [10, 4, 6]
    t["num_pos_examples"][0] = 6
    t["split_score"][0] = 0.5
    return GradientBoostedTreesModel(spec, [t], 0.25, "SQUARED_ERROR", [{"loss": 1.0, "secondary": 1.0}])


@pytest.mark.parametrize("na_value", [0, 1])
def test_model_writer_and_reader_round_trip_a_higher_condition(na_value):
    thr = np.float32(1.5)
    model = _model_with_one_higher_split(thr, na_value)
    probe = np.array([1.4999999, 1.5, 1.5000001, -3, 9, np.nan, -0.0], np.float32)
    want = 0.25 + np.where(np.isnan(probe), 1.0 if na_value else -1.0, np.where(probe >= thr, 1.0, -1.0))
    np.testing.assert_array_equal(model.predict({"x": probe}), want.astype(np.float32))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "m")
        model.save(path)
        m = model_io.read_ydf_model(path)
    col = m["columns"][1]
    assert col["type"] == 1 and col["name"] == "x" and col["mean"] == 2.0 and "boundaries" not in col   # NUMERICAL
    root = m["nodes"][0]
    assert np.float32(root["higher_threshold"]) == thr and "discretized_threshold" not in root
    assert root["na_value"] == bool(na_value) and root["n_pos"] == 6
    np.testing.assert_array_equal(model_io.predict_ydf_model(m, {"x": probe}), want.astype(np.float32))


def test_abi_refuses_bad_numerical_arguments_without_a_device():
    """The checks that need no dataset come first, so they hold on a machine without a device too."""
    lib = ydf_b200.lib()

    def call(values, n=None, na_replacement=0.0):
        v = np.ascontiguousarray(values, np.float32)
        st = lib.ygg_dataset_set_numerical_column(None, 0, v.ctypes.data_as(C.POINTER(C.c_float)),
                                                  C.c_int64(len(v) if n is None else n), C.c_float(na_replacement))
        return st, lib.ygg_last_error().decode()

    ok = np.array([1.0, np.nan, -0.0, 3e38], np.float32)
    for args, msg in (((np.array([1.0, np.inf], np.float32),), "infinite"), ((np.array([-np.inf], np.float32),), "infinite"),
                      ((ok, None, np.nan), "na_replacement"), ((ok, None, np.inf), "na_replacement"),
                      ((ok, -1), "negative row count")):
        st, err = call(*args)
        assert st == 1 and msg in err, (args, st, err)
    st, err = call(ok)   # valid arguments: the missing dataset
    assert st == 1 and "null" in err
    assert lib.ygg_dataset_set_numerical_column(None, 0, None, C.c_int64(0), C.c_float(0)) == 1
    assert lib.ygg_dataset_get_numerical_column(None, 0, None) == 1


@pytest.mark.parametrize("seed,use_hessian,min_obs,repeats", [(0, False, 1, False), (1, False, 5, True),
                                                               (2, True, 1, True), (3, True, 20, False)])
def test_numpy_reference_equals_a_brute_force_loop_over_every_cut(seed, use_hessian, min_obs, repeats):
    rng = np.random.default_rng(seed)
    n = 400
    v = rng.normal(size=n).astype(np.float32)
    if repeats:
        v[rng.random(n) < 0.3] = np.float32(0.5)
        v[:10] = -0.0
        v[10:20] = 0.0
    g = rng.normal(size=n) + 0.8 * (v > 0.2)
    h = rng.uniform(0.05, 0.25, size=n) if use_hessian else None
    got = PR.best_split(v, g, h, use_hessian, min_obs)
    want = PR.brute_force(v, g, h, use_hessian, min_obs)
    assert got is not None and want is not None
    assert got[1] == want[1] and got[2] == want[2]
    np.testing.assert_allclose(got[0], want[0], rtol=1e-9)


def test_mid_threshold_is_the_reference_rule():
    assert PR.mid_threshold(1.0, 2.0) == np.float32(1.5)
    a = np.float32(1.0)
    b = np.nextafter(a, np.float32(2))
    assert PR.mid_threshold(a, b) == b   # adjacent floats: the middle rounds down to a, the rule takes b
