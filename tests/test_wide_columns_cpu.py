"""Wide numerical columns (DESIGN.md §20) without a device: the learner option, the uint16 encoding, the dtype of
encode_features, the refusal above the limit before anything touches the device, and the C ABI's argument checks."""
import ctypes as C

import numpy as np
import pytest

import ydf_b200
from ydf_b200 import dataspec


def test_learner_option_range_and_messages():
    L = ydf_b200.GradientBoostedTreesLearner
    assert L(label="y").max_exact_numerical_values == 255
    for ok in (255, 256, 4096, 65535):
        assert L(label="y", max_exact_numerical_values=ok).max_exact_numerical_values == ok
    for bad in (0, 254, 65536, -1):
        with pytest.raises(ValueError, match="max_exact_numerical_values"):
            L(label="y", max_exact_numerical_values=bad)
    for bad in (300.0, "300", True):
        with pytest.raises(TypeError):
            L(label="y", max_exact_numerical_values=bad)


def test_refusal_above_the_limit_happens_before_the_device():
    L = ydf_b200.GradientBoostedTreesLearner
    x = np.arange(1000, dtype=np.float32)
    with pytest.raises(NotImplementedError, match="more than 255 distinct values"):
        L(label="y").train({"x": x, "y": np.arange(1000) % 2})
    with pytest.raises(NotImplementedError, match=r"more than 999 distinct values.*max_exact_numerical_values"):
        L(label="y", max_exact_numerical_values=999).train({"x": x, "y": np.arange(1000) % 2})
    # 65535 distinct values and a missing one: the mean would be bucket 65536
    v = np.empty(65536, dtype=np.float32)
    v[0] = np.nan
    v[1:] = np.arange(65535, dtype=np.float32) ** 2   # (the mean is none of the values)
    with pytest.raises(NotImplementedError, match="65535 buckets"):
        L(label="y", max_exact_numerical_values=65535).train({"x": v, "y": np.arange(len(v)) % 2})


def test_uint16_encoding_equals_the_byte_encoding():
    rng = np.random.default_rng(7)
    for k in (5, 100, 255):
        x = rng.integers(0, k, size=3000).astype(np.float32) * 0.37
        x[rng.random(3000) < 0.1] = np.nan
        c = dataspec.infer_column_lossless("x", x)
        assert c is not None and not c.wide
        probe = np.concatenate([x, np.array([-1e30, 1e30, np.inf, -np.inf, np.nan, 0.1], np.float32)])
        a, b = c.encode(probe), c.encode16(probe)
        assert b.dtype == np.uint16 and (a.astype(np.uint16) == b).all()
        assert (b[np.isnan(probe)] == c.na_bin).all()


def test_wide_column_inference_and_codes():
    rng = np.random.default_rng(8)
    x = rng.choice(np.arange(5000, dtype=np.float32) / 3, size=20000)
    x[::97] = np.nan
    assert dataspec.infer_column_lossless("x", x) is None
    c = dataspec.infer_column_lossless("x", x, max_distinct=65535)
    assert c.wide and c.num_bins == len(c.bucket_values) == len(np.unique(x[~np.isnan(x)])) + 1
    codes = c.encode16(x)
    assert (codes[np.isnan(x)] == c.na_bin).all()
    present = ~np.isnan(x)
    assert (c.bucket_values[codes[present]] == x[present]).all()   # one bucket per value
    assert c.bucket_values[c.na_bin] == np.float32(c.mean)


def test_encode_features_dtype():
    x = np.arange(1000, dtype=np.float32)
    narrow = dataspec.infer_column_lossless("a", x % 10)
    wide = dataspec.infer_column_lossless("b", x, max_distinct=65535)
    cols = {"a": x % 10, "b": x}
    assert dataspec.encode_features(cols, [narrow]).dtype == np.uint8
    out = dataspec.encode_features(cols, [narrow, wide])
    assert out.dtype == np.uint16 and out.shape == (2, 1000)
    assert (out[0] == narrow.encode(x % 10)).all() and (out[1] == np.arange(1000)).all()


def test_abi_entry_points_refuse_bad_arguments_without_a_device():
    lib = ydf_b200.lib()
    codes = np.zeros(10, np.uint16)
    vals = np.arange(300, dtype=np.float32)
    pc = codes.ctypes.data_as(C.POINTER(C.c_uint16))
    pv = vals.ctypes.data_as(C.POINTER(C.c_float))
    # null dataset / null arrays
    assert lib.ygg_dataset_set_wide_column(None, 0, pc, C.c_int64(10), 300, 0, pv, C.c_float(0)) == 1
    assert lib.ygg_dataset_get_wide_column(None, 0, pc, None, None) == 1
    assert lib.ygg_debug_wide_histogram(None, 1, None, None, None) == 1
    if ydf_b200.device_count() == 0:
        # every compute entry point needs the device; a dataset cannot exist without one
        b = np.zeros((1, 10), np.uint8)
        h = C.c_void_p()
        st = lib.ygg_dataset_create(C.byref(h), C.c_int64(10), 1, b.ctypes.data_as(C.POINTER(C.c_uint8)), C.c_int64(10),
                                    np.array([2], np.int32).ctypes.data_as(C.POINTER(C.c_int32)),
                                    np.array([0], np.int32).ctypes.data_as(C.POINTER(C.c_int32)), 0)
        assert st == 2


def test_abi_refuses_out_of_range_wide_arguments_without_a_device():
    """The argument checks that need no dataset come first, so they hold on a machine without a device too."""
    lib = ydf_b200.lib()

    def call(codes, num_bins, na_bin, values):
        c = np.ascontiguousarray(codes, np.uint16)
        v = np.ascontiguousarray(values, np.float32)
        st = lib.ygg_dataset_set_wide_column(None, 0, c.ctypes.data_as(C.POINTER(C.c_uint16)), C.c_int64(len(c)), num_bins,
                                             na_bin, v.ctypes.data_as(C.POINTER(C.c_float)), C.c_float(0))
        return st, lib.ygg_last_error().decode()

    ok_codes, ok_values = np.arange(10) % 300, np.arange(70000, dtype=np.float32)
    for args, msg in (((ok_codes, 256, 0, ok_values), "num_bins=256"), ((ok_codes, 65536, 0, ok_values), "num_bins=65536"),
                      ((ok_codes, 300, 300, ok_values), "na_bin=300"), ((ok_codes, 300, -1, ok_values), "na_bin=-1"),
                      ((np.full(10, 300), 300, 0, ok_values), "code 300"),
                      ((ok_codes, 300, 0, ok_values[::-1].copy()), "strictly ascending")):
        st, err = call(*args)
        assert st == 1 and msg in err, (args[1:3], st, err)
    st, err = call(ok_codes, 300, 0, ok_values)   # valid arguments: the missing dataset
    assert st == 1 and "null" in err
