"""Wide categorical columns (DESIGN.md §21) without a GPU: argument checks of the new ABI call, dictionary inference and
encode16 above 256 categories, the learner's categorical_arity_limit_for_random, the model writer's set encoding read
back by the generic reader, and the numpy CART reference the GPU tests compare against."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

import ydf_b200
from ydf_b200 import _capi, dataspec, model_io
from ydf_b200.model import GradientBoostedTreesModel
from tests import wide_cat_ref as W


def _call(codes, num_bins, na_bin, n=None):
    c = np.ascontiguousarray(codes, dtype=np.uint16)
    return _capi.lib().ygg_dataset_set_wide_categorical_column(
        None, C.c_int32(0), c.ctypes.data_as(C.POINTER(C.c_uint16)), C.c_int64(len(c) if n is None else n),
        C.c_int32(num_bins), C.c_int32(na_bin))


def test_abi_argument_checks_need_no_device():
    INVALID = 1
    ok = np.arange(10, dtype=np.uint16)
    assert _call(ok, 256, 0) == INVALID and "257, 65535" in _capi.lib().ygg_last_error().decode()
    assert _call(ok, 65536, 0) == INVALID
    assert _call(ok, 300, 300) == INVALID and "na_bin" in _capi.lib().ygg_last_error().decode()
    assert _call(ok, 300, -1) == INVALID
    assert _call(np.array([3, 300], np.uint16), 300, 0) == INVALID and "code 300" in _capi.lib().ygg_last_error().decode()
    assert _call(ok, 300, 0, n=-1) == INVALID
    # valid arguments reach the dataset checks: a null dataset
    assert _call(ok, 300, 0) == INVALID and "null" in _capi.lib().ygg_last_error().decode()


def _strings(k, reps=5):
    """k distinct keys, key i repeated reps + (k - i) times (distinct counts: one dictionary order)."""
    out = []
    for i in range(k):
        out += [f"v{i:05d}"] * (reps + (k - i) % 3)
    return np.array(out + ["", None], dtype=object)


@pytest.mark.parametrize("front_end", [dataspec.FRONT_END_CPP, dataspec.FRONT_END_PYDF])
@pytest.mark.parametrize("entries", [257, 299, 300, 2001])
def test_inference_and_encode16_above_256_categories(entries, front_end):
    v = _strings(entries - 1)
    c = dataspec.infer_categorical_column("c", v, min_vocab_frequency=1, max_vocab_count=-1 if front_end == "pydf" else 0,
                                          front_end=front_end)
    assert c.num_bins == entries and c.wide
    codes = c.encode16(v)
    assert codes.dtype == np.uint16
    index = {k: i for i, k in enumerate(c.vocabulary)}
    assert all(codes[i] == index[v[i]] for i in range(len(v) - 2))
    assert codes[-1] == codes[-2] == c.na_bin
    assert c.encode16(np.array(["never seen"], object))[0] == 0
    with pytest.raises(OverflowError):
        c.encode(v)   # uint8 codes cannot hold them


def test_inference_refuses_above_65535_categories():
    v = np.array([f"k{i}" for i in range(65535)], dtype=object)
    with pytest.raises(NotImplementedError, match="65535"):
        dataspec.infer_categorical_column("c", v, min_vocab_frequency=1, max_vocab_count=-1,
                                          front_end=dataspec.FRONT_END_PYDF)


def _table(entries):
    v = _strings(entries - 1)
    return {"c": v, "y": np.where(np.arange(len(v)) % 2 == 0, "a", "b")}


def test_learner_arity_limit():
    L = ydf_b200.GradientBoostedTreesLearner
    kw = dict(label="y", min_vocab_frequency=1, max_vocab_count=-1, num_trees=2)
    with pytest.raises(NotImplementedError, match=r"300 categories.*categorical_arity_limit_for_random.*random-mask"):
        L(**kw).train(_table(300))
    with pytest.raises(NotImplementedError, match="max_vocab_count"):
        L(**kw).train(_table(300))
    # accepted: 299 categories with the defaults, 300 with the limit raised; past the checks the next step needs a
    # device (here: none), not the option
    for entries, extra in ((299, {}), (300, dict(categorical_arity_limit_for_random=301))):
        try:
            L(**kw, **extra).train(_table(entries))
        except ydf_b200.YggError as e:
            assert "device" in str(e)
    with pytest.raises(NotImplementedError, match="65535"):
        v = np.array([f"k{i}" for i in range(65535)], dtype=object)
        L(**kw, categorical_arity_limit_for_random=10 ** 6).train({"c": v, "y": np.where(np.arange(65535) % 2, "a", "b")})
    with pytest.raises(ValueError):
        L(label="y", categorical_arity_limit_for_random=0)
    with pytest.raises(TypeError):
        L(label="y", categorical_arity_limit_for_random=2.5)


def _model_with_split(num_values, positive):
    """A one-split model on a categorical column of `num_values` entries whose positive set is `positive`."""
    col = dataspec.CategoricalColumn("c", ["<OOD>"] + [f"k{i}" for i in range(1, num_values)], [1] * num_values,
                                     num_values, 0)
    t = np.zeros(3, dtype=_capi.NODE_DTYPE)
    t["feature"] = [0, -1, -1]
    t["neg_child"] = [1, -1, -1]
    t["pos_child"] = [2, -1, -1]
    t["condition_type"] = [1, 0, 0]
    t["leaf_value"] = [0.0, -1.0, 1.0]
    t["num_examples"] = [10, 5, 5]
    t["num_pos_examples"] = [5, 0, 0]
    words = np.zeros((num_values + 31) // 32, np.uint32)
    for c in positive:
        words[c >> 5] |= np.uint32(1 << (c & 31))
    spec = dataspec.DataSpec(columns=[col], label="y", task="REGRESSION")
    return GradientBoostedTreesModel(spec, [t], 0.0, "SQUARED_ERROR", category_sets=[{0: words}]), col


@pytest.mark.parametrize("num_values,positive,field", [
    (300, [1, 7, 255, 256, 299], 4),                     # 5 x 4 B < 38 B of bitmap: ContainsVector
    (300, list(range(2, 300, 3)), 5),                    # 99 x 4 B > 38 B: ContainsBitmap
    (5000, [0, 4999, 3000, 257], 4),
    (5000, list(range(1, 5000, 2)), 5),
])
def test_model_writer_sizes_the_set_over_all_categories(num_values, positive, field):
    model, col = _model_with_split(num_values, positive)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "m")
        model.save(path)
        m = model_io.read_ydf_model(path)
        recs = model_io.read_blob_sequence(os.path.join(path, "nodes-00000-of-00001"))
    assert m["nodes"][0]["positive_categories"] == sorted(positive)
    cond = model_io.pb_decode(model_io._one(model_io.pb_decode(model_io._one(model_io.pb_decode(recs[0]), 3)), 3))
    assert [f for f, _, _ in cond] == [field]
    if field == 5:
        assert len(model_io._one(model_io.pb_decode(cond[0][2]), 1)) == (num_values + 7) // 8
    assert m["columns"][1]["number_of_unique_values"] == num_values
    assert len(m["columns"][1]["vocabulary"]) == num_values
    # the host model, the saved model and the raw set route every category alike
    keys = np.array(col.vocabulary[1:] + ["unknown"], dtype=object)
    raw_io = model_io.predict_ydf_model(m, {"c": keys})
    raw = model.predict({"c": keys})
    want = np.array([1.0 if i in set(positive) else -1.0 for i in list(range(1, num_values)) + [0]], np.float32)
    np.testing.assert_array_equal(raw, want)
    np.testing.assert_array_equal(raw_io, want)


@pytest.mark.parametrize("use_hessian", [False, True])
@pytest.mark.parametrize("B", [257, 1000, 5000])
def test_numpy_cart_against_brute_force(B, use_hessian):
    """The reference's vectorised scan against a plain loop over every sorted-prefix split of the node, with weights
    (the counts of a weighted node are weight sums) and keys tied by category index."""
    rng = np.random.default_rng(B)
    cnt = rng.integers(0, 30, size=B).astype(np.float64)
    cnt[::7] = 0
    w = cnt * rng.uniform(0.5, 2.0, size=B)                         # weight sums
    s = np.round(rng.normal(size=B) * 4) / 4 * (cnt > 0)           # quarter steps: many equal keys
    s[5::11] = 0.0
    h = w if not use_hessian else cnt * 0.25
    count = w if not use_hessian else cnt
    got = W.best_split(count, s, h, use_hessian, min_obs=1)
    k = W.keys(count, s, h, use_hessian)
    order = sorted(range(B), key=lambda i: (k[i], i))
    best, best_b = -1.0, None
    for b in range(B - 1):
        neg, pos = order[:b + 1], order[b + 1:]
        cn, cp = count[neg].sum(), count[pos].sum()
        if cn < 1 or cp < 1:
            continue
        sn, sp_ = s[neg].sum(), s[pos].sum()
        if not use_hessian:
            c0 = cn + cp
            d = sp_ * cn - sn * cp
            sc = (d / cp) * (d / cn) / (c0 * c0)
        else:
            hn, hp = max(h[neg].sum(), W.MIN_HESSIAN) + 1.0, max(h[pos].sum(), W.MIN_HESSIAN) + 1.0
            sc = sp_ ** 2 / hp + sn ** 2 / hn
            if sc <= (sn + sp_) ** 2 / (max(h.sum(), W.MIN_HESSIAN) + 1.0):   # not above the parent's term
                continue
        if sc > 0 and sc > best + 1e-12 * abs(best):
            best, best_b = sc, b
    assert got is not None and best_b is not None
    np.testing.assert_allclose(got[0], best, rtol=1e-9)
    assert np.array_equal(got[1], np.sort(order[best_b + 1:]))
