"""Discretized wide columns (DESIGN.md §25), host side: the 16-bit host rule (dataspec.infer_column16 over
csrc/ygg_dataspec.cc) against the numpy restatement of GenDiscretizedBoundaries in oracle/binning.py, the reference-made
Adult dataspec, the uint16 encoding, and the refusals that hold without a GPU."""
import ctypes as C
import os

import numpy as np
import pytest

import ydf_b200
from oracle import binning as B

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _columns(n, seed):
    """Distributions that exercise the rule: continuous, ties, NaN, -0 / +0, heavy values, constant, few distinct."""
    rng = np.random.default_rng(seed)
    out = {"normal": rng.normal(size=n).astype(np.float32),
           "ties": np.round(rng.normal(size=n) * 300).astype(np.float32)}
    x = rng.normal(size=n).astype(np.float32)
    x[rng.random(n) < 0.1] = np.nan
    out["nan"] = x
    x = rng.normal(size=n).astype(np.float32)
    x[rng.random(n) < 0.2] = -0.0
    x[rng.random(n) < 0.2] = 0.0
    out["signed_zero"] = x
    out["heavy"] = np.where(rng.random(n) < 0.3, np.float32(1.5),
                            np.where(rng.random(n) < 0.2, np.float32(-7.0), rng.exponential(size=n))).astype(np.float32)
    out["constant"] = np.full(n, 3.25, np.float32)
    out["few"] = rng.integers(0, 40, size=n).astype(np.float32)
    return out


@pytest.mark.parametrize("max_bins", [257, 1000, 4096, 65535])
def test_host_rule_matches_the_numpy_restatement(max_bins):
    for n in (3000, 200000):
        for name, x in _columns(n, seed=max_bins + n).items():
            col = ydf_b200.dataspec.infer_column16(name, x, max_bins)
            want, mean = B.discretize_boundaries(x, max_bins, 3)
            np.testing.assert_array_equal(col.boundaries, want, err_msg=f"{name} n={n}")
            assert col.boundaries.dtype == np.float32
            assert col.mean == mean
            assert col.num_bins == len(want) + 1 <= 65535
            assert col.na_bin == int(np.searchsorted(want, np.float32(mean), side="right"))
            assert col.num_missing == int(np.isnan(x).sum())


def test_many_bins_are_made_when_asked():
    """Continuous columns with more distinct values than the budget fill it: the uint16 range is used."""
    rng = np.random.default_rng(5)
    x = rng.normal(size=400000).astype(np.float32)
    for max_bins in (1000, 4096, 65535):
        col = ydf_b200.dataspec.infer_column16("x", x, max_bins)
        assert max_bins - 4 <= col.num_bins <= max_bins
        assert col.wide


def test_reference_made_dataspec_at_255_bins():
    """infer_column16 asked for 255 bins reproduces the boundaries GenDiscretizedBoundaries stored in the dataspec of the
    reference's golden model adult_binary_class_rf_discret_numerical, as infer_column does."""
    ref = np.load(os.path.join(GOLDEN, "ydf_adult_discretized_dataspec.npz"))
    data = np.load(os.path.join(GOLDEN, "adult_numerical.npz"))
    for name in ("age", "fnlwgt", "capital_gain", "capital_loss", "hours_per_week"):
        col = ydf_b200.dataspec.infer_column16(name, data[f"train_{name}"].astype(np.float32), 255)
        np.testing.assert_array_equal(col.boundaries, ref[f"boundaries_{name}"], err_msg=name)
        assert not col.wide


def test_encode16_is_upper_bound_with_nan_to_the_mean_bin():
    rng = np.random.default_rng(9)
    x = rng.normal(size=100000).astype(np.float32)
    x[::17] = np.nan
    col = ydf_b200.dataspec.infer_column16("x", x, 4096)
    codes = col.encode16(x)
    assert codes.dtype == np.uint16
    present = ~np.isnan(x)
    np.testing.assert_array_equal(codes[present], np.searchsorted(col.boundaries, x[present], side="right"))
    assert (codes[~present] == col.na_bin).all()
    assert codes.max() < col.num_bins


def test_refusals():
    x = np.arange(100, dtype=np.float32)
    for bad in (1, 65536):
        with pytest.raises(ydf_b200.YggError):
            ydf_b200.dataspec.infer_column16("x", x, bad)
    # the byte rule keeps its bounds and its uint8 refusal
    with pytest.raises(ydf_b200.YggError):
        ydf_b200.discretize_boundaries(x, 65535, 3)
    with pytest.raises(ValueError, match="uint8"):
        ydf_b200.dataspec.infer_column("x", np.arange(100000, dtype=np.float32), 1000)
    # the learner's bin budget
    L = ydf_b200.GradientBoostedTreesLearner
    for bad in (1, 65536, 100000):
        with pytest.raises(ValueError, match=r"\[2, 65535\]"):
            L(label="y", discretize_numerical_columns=True, num_discretized_numerical_bins=bad)
    for ok in (2, 256, 257, 1024, 65535):
        assert L(label="y", discretize_numerical_columns=True, num_discretized_numerical_bins=ok).num_discretized_numerical_bins == ok


def _call(codes, num_bins, na_bin, n=None):
    c = np.ascontiguousarray(codes, dtype=np.uint16)
    return ydf_b200.lib().ygg_dataset_set_wide_discretized_column(
        None, C.c_int32(0), c.ctypes.data_as(C.POINTER(C.c_uint16)), C.c_int64(len(c) if n is None else n),
        C.c_int32(num_bins), C.c_int32(na_bin))


def test_set_wide_discretized_column_argument_checks():
    """The checks that need no dataset run first, so they hold without a device."""
    INVALID = 1
    ok = np.arange(10, dtype=np.uint16)
    err = lambda: ydf_b200.lib().ygg_last_error().decode()   # noqa: E731
    assert _call(ok, 256, 0) == INVALID and "257, 65535" in err()
    assert _call(ok, 65536, 0) == INVALID
    assert _call(ok, 300, 300) == INVALID and "na_bin" in err()
    assert _call(ok, 300, -1) == INVALID
    assert _call(np.array([3, 300], np.uint16), 300, 0) == INVALID and "code 300" in err()
    assert _call(ok, 300, 0, n=-1) == INVALID
    assert _call(ok, 300, 0) == INVALID and "null" in err()
