"""ctypes binding of libygg_b200.so (include/ygg_b200.h).  No torch types cross this boundary."""
import ctypes as C
import os

import numpy as np

from . import _build

_LIB = None


class YggError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"[ygg status {code}] {msg}")
        self.code = code


class GbtConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("loss", C.c_int32), ("num_trees", C.c_int32),
        ("shrinkage", C.c_float), ("max_depth", C.c_int32), ("min_examples", C.c_int32),
        ("in_split_min_examples_check", C.c_int32), ("use_hessian_gain", C.c_int32),
        ("l1_regularization", C.c_float), ("l2_regularization", C.c_float),
        ("l2_regularization_categorical", C.c_float), ("clamp_leaf_logit", C.c_float),
        ("hessian_split_score_subtract_parent", C.c_int32), ("random_seed", C.c_uint32),
        ("subsample", C.c_float), ("validation_ratio", C.c_float),
        ("sibling_subtraction", C.c_int32), ("early_stopping", C.c_int32),
        ("early_stopping_num_trees_look_ahead", C.c_int32), ("early_stopping_initial_iteration", C.c_int32),
        ("num_classes", C.c_int32), ("candidate_shuffle", C.c_int32), ("rng_words_consumed", C.c_uint32),
        ("split_jobs_draw_seeds", C.c_int32), ("growing_strategy", C.c_int32), ("max_num_nodes", C.c_int32),
        ("goss_alpha", C.c_float), ("goss_beta", C.c_float),
    ]


NODE_DTYPE = np.dtype([
    ("feature", "<i4"), ("threshold_bin", "<i4"), ("na_value", "<i4"), ("depth", "<i4"),
    ("neg_child", "<i4"), ("pos_child", "<i4"), ("split_score", "<f4"), ("leaf_value", "<f4"),
    ("num_examples", "<i8"), ("num_pos_examples", "<i8"), ("stat", "<f8", (3,)),
    ("condition_type", "<i4"), ("threshold_value", "<f4"), ("cat_mask", "<u4", (8,)),
])
assert NODE_DTYPE.itemsize == 112  # sizeof(ygg_node), include/ygg_b200.h

FEATURE_DISCRETIZED_NUMERICAL = 0
FEATURE_CATEGORICAL = 1
FEATURE_NUMERICAL = 2   # presorted numerical column (Dataset.set_numerical_column)

LEVEL_NODE_DTYPE = np.dtype([("node", "<i4"), ("candidate", "<i4"), ("derived", "<i4"), ("reserved", "<i4"),
                             ("num_examples", "<i8")])
assert LEVEL_NODE_DTYPE.itemsize == 24  # sizeof(ygg_level_node)
CANDIDATE_DTYPE = np.dtype([("found", "<i4"), ("score", "<f4"), ("threshold_bin", "<i4"), ("lo", "<i4"), ("hi", "<i4"),
                            ("num_pos_examples", "<i4"), ("threshold_value", "<f4"), ("cat_mask", "<u4", (8,))])
assert CANDIDATE_DTYPE.itemsize == 60  # sizeof(ygg_candidate)

HIST_ROOT_SUM, HIST_PACKED, HIST_SHARED, HIST2, HIST_SEGMENTED = 0, 1, 2, 3, 4   # enum ygg_hist_mode


class HistPlan(C.Structure):
    """One level's k_hist / k_hist2 / k_hist_seg / k_hist_root_rows launch (ygg_hist_plan)."""
    _fields_ = [("mode", C.c_int32), ("group", C.c_int32), ("hist2_tiles", C.c_int32), ("chunk_blocks", C.c_int32),
                ("slot_window", C.c_int32), ("grid", C.c_int32)]

    # the C union {hist2_tiles; root_lanes}: a ROOT_SUM plan's feature lanes (0: k_hist, 32: k_hist_root_rows)
    root_lanes = property(lambda self: self.hist2_tiles, lambda self, v: setattr(self, "hist2_tiles", v))

    def __repr__(self):
        return "HistPlan(%s)" % ", ".join("%s=%d" % (k, getattr(self, k)) for k, _ in self._fields_)

ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p)
ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p)
REDUCESCATTER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p)

EXPORTS = [
    "ygg_abi_version", "ygg_last_error", "ygg_device_count", "ygg_dataset_create",
    "ygg_dataset_set_feature_types", "ygg_dataset_destroy", "ygg_dataset_num_rows", "ygg_dataset_num_features",
    "ygg_gbt_config_init", "ygg_gbt_create", "ygg_gbt_destroy", "ygg_gbt_set_labels_i32",
    "ygg_gbt_set_labels_f32", "ygg_gbt_set_weights_f32", "ygg_gbt_set_validation_weights_f32", "ygg_gbt_set_feature_shard", "ygg_gbt_set_row_shard", "ygg_gbt_set_row_shard_scatter", "ygg_feature_shard",
    "ygg_merge_shard_best", "ygg_gbt_initial_prediction",
    "ygg_gbt_train", "ygg_gbt_train_timed", "ygg_gbt_step", "ygg_gbt_sync", "ygg_gbt_num_trees", "ygg_gbt_get_tree",
    "ygg_gbt_train_loss", "ygg_gbt_get_predictions", "ygg_gbt_set_predictions", "ygg_gbt_predict",
    "ygg_tree_train_on_gradients", "ygg_debug_hist_plan", "ygg_debug_level_histogram", "ygg_partition_rows",
    "ygg_gbt_set_profiling", "ygg_gbt_get_profile", "ygg_gbt_save_ydf",
    "ygg_discretize_boundaries", "ygg_discretize_encode", "ygg_model_write_ydf",
    "ygg_validation_split_mask", "ygg_dataset_split_rows", "ygg_gbt_set_validation_i32",
    "ygg_gbt_set_validation_f32", "ygg_gbt_validation_loss", "ygg_gbt_num_iterations", "ygg_gbt_final_validation",
    "ygg_gen_discretized_boundaries", "ygg_dataset_builder_create", "ygg_dataset_builder_add_numerical",
    "ygg_dataset_builder_add_numerical_async", "ygg_dataset_builder_get_numerical",
    "ygg_dataset_builder_add_bins", "ygg_dataset_builder_finish", "ygg_dataset_builder_destroy",
    "ygg_dataset_get_bins", "ygg_dataset_set_bucket_values", "ygg_gbt_tie_stats", "ygg_gbt_set_tie_rng_position",
    "ygg_gbt_best_split_window_bytes", "ygg_gbt_set_best_split_window", "ygg_comm_window_create",
    "ygg_comm_unique_id", "ygg_comm_create", "ygg_comm_destroy", "ygg_comm_allreduce", "ygg_comm_allgather", "ygg_comm_reducescatter",
    "ygg_dataset_set_wide_column", "ygg_dataset_get_wide_column", "ygg_debug_wide_histogram",
    "ygg_dataset_set_wide_categorical_column", "ygg_gbt_get_category_set",
    "ygg_dataset_set_numerical_column", "ygg_dataset_get_numerical_column",
    "ygg_debug_capture_candidates", "ygg_debug_level_candidates",
    "ygg_num_candidate_attributes", "ygg_candidate_key", "ygg_gbt_set_candidate_sampling", "ygg_debug_level_tried",
    "ygg_gbt_set_dart", "ygg_gbt_get_dart_weights", "ygg_gbt_get_dart_dropped",
    "ygg_dataset_set_wide_discretized_column", "ygg_dataset_builder_add_numerical16_async", "ygg_discretize_boundaries16",
]


def lib():
    """Loads (building if stale) the native library.  There is no fallback: if the library
    cannot be built or loaded this raises."""
    global _LIB
    if _LIB is None:
        path = _build.build()
        L = C.CDLL(path)
        L.ygg_last_error.restype = C.c_char_p
        L.ygg_dataset_num_rows.restype = C.c_int64
        L.ygg_gbt_config_init.restype = None
        L.ygg_candidate_key.restype = C.c_uint64
        L.ygg_candidate_key.argtypes = [C.c_uint32, C.c_int32, C.c_int32, C.c_int32]
        for name in EXPORTS:
            getattr(L, name)  # fail loudly on a missing symbol
        _LIB = L
    return _LIB


def check(status):
    if status != 0:
        raise YggError(status, lib().ygg_last_error().decode("utf-8", "replace"))


def ptr(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


def num_candidate_attributes(num_features, loss, num_candidate_attributes=-1, ratio=None):
    """k, the number of features a node tests under candidate feature sampling (ygg_num_candidate_attributes); ratio None
    (or negative): not set."""
    k = C.c_int32()
    check(lib().ygg_num_candidate_attributes(C.c_int32(int(num_features)), C.c_int32(int(loss)),
                                             C.c_int32(int(num_candidate_attributes)),
                                             C.c_float(-1.0 if ratio is None else float(ratio)), C.byref(k)))
    return k.value


def candidate_key(seed, tree, node, feature):
    """The key ordering `feature` among the candidates of node `node` of tree `tree` (ygg_candidate_key)."""
    return int(lib().ygg_candidate_key(int(seed) & 0xFFFFFFFF, int(tree), int(node), int(feature)))


def default_config(**kw):
    cfg = GbtConfig()
    lib().ygg_gbt_config_init(C.byref(cfg))
    for k, v in kw.items():
        if not hasattr(cfg, k):
            raise AttributeError(k)
        setattr(cfg, k, v)
    return cfg


class Dataset:
    """Device-resident bucketised dataset (ygg_dataset)."""

    def __init__(self, bins, num_bins, na_bin, device=0, feature_types=None):
        b = np.asarray(bins)
        # a row slice of a larger [F, N] matrix is taken in place (column_stride = the parent's N)
        if not (b.dtype == np.uint8 and b.ndim == 2 and b.strides[1] == 1 and b.strides[0] >= b.shape[1]):
            b = np.ascontiguousarray(bins, dtype=np.uint8)
        assert b.ndim == 2, "bins must be [n_features, n_rows] (column-major storage)"
        self.n_features, self.n_rows = b.shape
        self.num_bins = np.ascontiguousarray(num_bins, dtype=np.int32)
        self.na_bin = np.ascontiguousarray(na_bin, dtype=np.int32)
        assert len(self.num_bins) == self.n_features and len(self.na_bin) == self.n_features
        self.handle = C.c_void_p()
        self.h2d_bytes = self.n_features * self.n_rows
        # (the stride of a length-1 axis is arbitrary in numpy: a single-feature matrix has no second column to reach)
        col_stride = b.strides[0] if self.n_features > 1 else max(int(b.strides[0]), self.n_rows)
        check(lib().ygg_dataset_create(C.byref(self.handle), C.c_int64(self.n_rows),
                                       C.c_int32(self.n_features), C.cast(b.ctypes.data, C.POINTER(C.c_uint8)),
                                       C.c_int64(col_stride), ptr(self.num_bins, C.c_int32),
                                       ptr(self.na_bin, C.c_int32), C.c_int32(device)))
        self.feature_types = np.zeros(self.n_features, np.int32)
        if feature_types is not None:
            self.set_feature_types(feature_types)

    def set_bucket_values(self, feature, values, na_replacement):
        """Exact threshold rule for a numerical feature with one bucket per distinct value: values[b] = value of bucket b,
        na_replacement = the column mean."""
        v = np.ascontiguousarray(values, dtype=np.float32)
        check(lib().ygg_dataset_set_bucket_values(self.handle, C.c_int32(int(feature)), ptr(v, C.c_float), C.c_int32(len(v)),
                                                  C.c_float(float(np.float32(na_replacement)))))

    def set_wide_column(self, feature, codes, num_bins, na_bin, values, na_replacement):
        """Wide numerical column (257..65535 buckets, one per distinct value): codes[r] = the uint16 bucket of row r,
        values[b] = the value of bucket b, na_replacement = the column mean.  Always split with the exact threshold rule."""
        c = np.ascontiguousarray(codes, dtype=np.uint16)
        v = np.ascontiguousarray(values, dtype=np.float32)
        if len(v) != int(num_bins):
            raise ValueError(f"{len(v)} bucket values for {num_bins} buckets")
        check(lib().ygg_dataset_set_wide_column(self.handle, C.c_int32(int(feature)), ptr(c, C.c_uint16), C.c_int64(len(c)),
                                                C.c_int32(int(num_bins)), C.c_int32(int(na_bin)), ptr(v, C.c_float),
                                                C.c_float(float(np.float32(na_replacement)))))
        self.num_bins = self.num_bins.copy()
        self.na_bin = self.na_bin.copy()
        self.num_bins[feature], self.na_bin[feature] = 1, 0   # the byte column is a one-bucket filler
        self.wide = dict(getattr(self, "wide", {}))
        self.wide[int(feature)] = (int(num_bins), int(na_bin))

    def set_wide_categorical_column(self, feature, codes, num_bins, na_bin):
        """Wide categorical column (257..65535 categories): codes[r] = the uint16 category of row r, na_bin = the
        most_frequent_value missing values were folded into.  The feature must already be FEATURE_CATEGORICAL."""
        c = np.ascontiguousarray(codes, dtype=np.uint16)
        check(lib().ygg_dataset_set_wide_categorical_column(self.handle, C.c_int32(int(feature)), ptr(c, C.c_uint16),
                                                            C.c_int64(len(c)), C.c_int32(int(num_bins)), C.c_int32(int(na_bin))))
        self.num_bins = self.num_bins.copy()
        self.na_bin = self.na_bin.copy()
        self.num_bins[feature], self.na_bin[feature] = 1, 0   # the byte column is a one-bucket filler
        self.wide = dict(getattr(self, "wide", {}))
        self.wide[int(feature)] = (int(num_bins), int(na_bin))

    def set_wide_discretized_column(self, feature, codes, num_bins, na_bin):
        """Discretized wide column (257..65535 bins of GenDiscretizedBoundaries): codes[r] = the uint16 bin of row r,
        na_bin = the bin of the column mean missing values were folded into.  Split by the discretized threshold rule."""
        c = np.ascontiguousarray(codes, dtype=np.uint16)
        check(lib().ygg_dataset_set_wide_discretized_column(self.handle, C.c_int32(int(feature)), ptr(c, C.c_uint16),
                                                            C.c_int64(len(c)), C.c_int32(int(num_bins)), C.c_int32(int(na_bin))))
        self.num_bins = self.num_bins.copy()
        self.na_bin = self.na_bin.copy()
        self.num_bins[feature], self.na_bin[feature] = 1, 0   # the byte column is a one-bucket filler
        self.wide = dict(getattr(self, "wide", {}))
        self.wide[int(feature)] = (int(num_bins), int(na_bin))

    def get_wide_column(self, feature):
        """-> (uint16 codes, num_bins, na_bin) of a wide column."""
        out = np.empty(self.n_rows, np.uint16)
        nb, na = C.c_int32(), C.c_int32()
        check(lib().ygg_dataset_get_wide_column(self.handle, C.c_int32(int(feature)), ptr(out, C.c_uint16), C.byref(nb), C.byref(na)))
        return out, nb.value, na.value

    def set_numerical_column(self, feature, values, na_replacement):
        """Presorted numerical column: values[r] = the float value of row r (NaN = missing, stored as na_replacement, the
        column mean).  Split by the exact numerical splitter through sorted row lists, with no limit on distinct values;
        its splits route by value >= threshold_value."""
        v = np.ascontiguousarray(values, dtype=np.float32)
        check(lib().ygg_dataset_set_numerical_column(self.handle, C.c_int32(int(feature)), ptr(v, C.c_float), C.c_int64(len(v)),
                                                     C.c_float(float(np.float32(na_replacement)))))
        self.num_bins = self.num_bins.copy()
        self.na_bin = self.na_bin.copy()
        self.num_bins[feature], self.na_bin[feature] = 1, 0   # the byte column is a one-bucket filler
        self.feature_types = self.feature_types.copy()
        self.feature_types[feature] = FEATURE_NUMERICAL

    def get_numerical_column(self, feature):
        """-> float32 values of a presorted numerical column as stored (missing values replaced)."""
        out = np.empty(self.n_rows, np.float32)
        check(lib().ygg_dataset_get_numerical_column(self.handle, C.c_int32(int(feature)), ptr(out, C.c_float)))
        return out

    def set_feature_types(self, feature_types):
        """feature_types[f]: FEATURE_DISCRETIZED_NUMERICAL or FEATURE_CATEGORICAL (FEATURE_NUMERICAL, and only that, for
        the presorted numerical columns)."""
        ft = np.ascontiguousarray(feature_types, dtype=np.int32)
        check(lib().ygg_dataset_set_feature_types(self.handle, ptr(ft, C.c_int32), C.c_int32(len(ft))))
        self.feature_types = ft

    def close(self):
        if self.handle:
            lib().ygg_dataset_destroy(self.handle)
            self.handle = C.c_void_p()

    def split_rows(self, select):
        """-> (Dataset of the rows with select != 0, Dataset of the others), gathered on the device."""
        m = np.ascontiguousarray(select, dtype=np.uint8)
        assert m.shape == (self.n_rows,)
        a, b = C.c_void_p(), C.c_void_p()
        check(lib().ygg_dataset_split_rows(self.handle, ptr(m, C.c_uint8), C.byref(a), C.byref(b)))
        out = []
        for hnd, n in ((a, int(m.astype(bool).sum())), (b, int(len(m) - m.astype(bool).sum()))):
            d = Dataset.__new__(Dataset)
            d.handle, d.n_features, d.n_rows = hnd, self.n_features, n
            d.num_bins, d.na_bin, d.feature_types, d.h2d_bytes = self.num_bins, self.na_bin, self.feature_types, 0
            d.wide = dict(getattr(self, "wide", {}))
            out.append(d)
        return out[0], out[1]

    def get_bins(self, feature):
        out = np.empty(self.n_rows, np.uint8)
        check(lib().ygg_dataset_get_bins(self.handle, C.c_int32(feature), ptr(out, C.c_uint8)))
        return out

    def partition_rows(self, rows, feature, threshold_bin):
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        out = np.empty_like(rows)
        n_pos = C.c_int64()
        check(lib().ygg_partition_rows(self.handle, ptr(rows, C.c_uint32), C.c_int64(len(rows)),
                                       C.c_int32(feature), C.c_int32(threshold_bin),
                                       ptr(out, C.c_uint32), C.byref(n_pos)))
        return out[:n_pos.value], out[n_pos.value:]

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DatasetBuilder:
    """Column-by-column construction of a device-resident dataset with ON-GPU binning of the float32
    columns (include/ygg_b200_dataspec.h, csrc/ygg_binning.cu)."""

    def __init__(self, n_rows, n_features, device=0):
        self.handle = C.c_void_p()
        self.n_rows, self.n_features, self.device = int(n_rows), int(n_features), device
        self.num_bins = np.ones(n_features, np.int32)
        self.na_bin = np.zeros(n_features, np.int32)
        self.feature_types = np.zeros(n_features, np.int32)
        self.h2d_bytes = 0
        check(lib().ygg_dataset_builder_create(C.byref(self.handle), C.c_int64(n_rows), C.c_int32(n_features),
                                               C.c_int32(device)))

    def add_numerical(self, feature, values, maximum_num_bins=255, min_obs_in_bins=3, n_stats_rows=0):
        """-> (boundaries float32, mean, na_bin, num_missing); the column is binned on the GPU."""
        v = np.ascontiguousarray(values, dtype=np.float32)
        assert v.shape == (self.n_rows,)
        bounds = np.empty(256, np.float32)
        nb, mean, na, miss = C.c_int32(), C.c_double(), C.c_int32(), C.c_int64()
        check(lib().ygg_dataset_builder_add_numerical(
            self.handle, C.c_int32(feature), ptr(v, C.c_float), C.c_int64(n_stats_rows),
            C.c_int32(maximum_num_bins), C.c_int32(min_obs_in_bins), ptr(bounds, C.c_float), C.c_int32(256),
            C.byref(nb), C.byref(mean), C.byref(na), C.byref(miss)))
        self.num_bins[feature], self.na_bin[feature] = nb.value + 1, na.value
        self.h2d_bytes += v.nbytes
        return bounds[:nb.value].copy(), mean.value, na.value, miss.value

    def add_numerical_async(self, feature, values, maximum_num_bins=255, min_obs_in_bins=3, n_stats_rows=0):
        """Enqueues the column and returns; collect with get_numerical (or finish).  The array is kept
        alive by the builder until then."""
        v = np.ascontiguousarray(values, dtype=np.float32)
        assert v.shape == (self.n_rows,)
        self._pending = getattr(self, "_pending", {})
        self._pending[feature] = v
        check(lib().ygg_dataset_builder_add_numerical_async(
            self.handle, C.c_int32(feature), ptr(v, C.c_float), C.c_int64(n_stats_rows),
            C.c_int32(maximum_num_bins), C.c_int32(min_obs_in_bins)))
        self.h2d_bytes += v.nbytes

    def add_numerical16_async(self, feature, values, maximum_num_bins, min_obs_in_bins=3, n_stats_rows=0):
        """add_numerical_async for 257..65535 bins: a column that ends with more than 256 bins becomes a discretized
        wide column (uint16 codes) when the builder is finished, one with fewer a byte column."""
        v = np.ascontiguousarray(values, dtype=np.float32)
        assert v.shape == (self.n_rows,)
        self._pending = getattr(self, "_pending", {})
        check(lib().ygg_dataset_builder_add_numerical16_async(
            self.handle, C.c_int32(feature), ptr(v, C.c_float), C.c_int64(n_stats_rows),
            C.c_int32(maximum_num_bins), C.c_int32(min_obs_in_bins)))
        self._pending[feature] = v
        self._wide16 = getattr(self, "_wide16", set()) | {int(feature)}
        self.h2d_bytes += v.nbytes

    def get_numerical(self, feature):
        wide16 = int(feature) in getattr(self, "_wide16", ())
        capacity = 65535 if wide16 else 256
        bounds = np.empty(capacity, np.float32)
        nb, mean, na, miss = C.c_int32(), C.c_double(), C.c_int32(), C.c_int64()
        check(lib().ygg_dataset_builder_get_numerical(self.handle, C.c_int32(feature), ptr(bounds, C.c_float),
                                                      C.c_int32(capacity), C.byref(nb), C.byref(mean), C.byref(na),
                                                      C.byref(miss)))
        getattr(self, "_pending", {}).pop(feature, None)
        self.num_bins[feature], self.na_bin[feature] = nb.value + 1, na.value
        if wide16 and nb.value + 1 > 256:   # a discretized wide column at finish: its byte column is a one-bucket filler
            self.num_bins[feature], self.na_bin[feature] = 1, 0
            self.wide = dict(getattr(self, "wide", {}))
            self.wide[int(feature)] = (nb.value + 1, na.value)
        return bounds[:nb.value].copy(), mean.value, na.value, miss.value

    def add_bins(self, feature, bins, num_bins, na_bin, feature_type=0):
        b = np.ascontiguousarray(bins, dtype=np.uint8)
        assert b.shape == (self.n_rows,)
        check(lib().ygg_dataset_builder_add_bins(self.handle, C.c_int32(feature), ptr(b, C.c_uint8),
                                                 C.c_int32(num_bins), C.c_int32(na_bin), C.c_int32(feature_type)))
        self.num_bins[feature], self.na_bin[feature], self.feature_types[feature] = num_bins, na_bin, feature_type
        if int(feature) in getattr(self, "_wide16", ()):
            self._wide16.discard(int(feature))
            getattr(self, "wide", {}).pop(int(feature), None)
        self.h2d_bytes += b.nbytes

    def finish(self):
        """-> Dataset (the builder is consumed)."""
        for f in list(getattr(self, "_pending", {})):
            self.get_numerical(f)
        out = C.c_void_p()
        check(lib().ygg_dataset_builder_finish(self.handle, C.byref(out)))
        self.handle = C.c_void_p()
        ds = Dataset.__new__(Dataset)
        ds.handle = out
        ds.n_features, ds.n_rows = self.n_features, self.n_rows
        ds.num_bins, ds.na_bin, ds.feature_types = self.num_bins, self.na_bin, self.feature_types
        ds.h2d_bytes = self.h2d_bytes
        if getattr(self, "wide", None):
            ds.wide = dict(self.wide)
        return ds

    def close(self):
        if self.handle:
            lib().ygg_dataset_builder_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def validation_split_mask(random_seed, n_rows, validation_ratio):
    """ExtractValidationDataset's row draw: True = training row."""
    m = np.empty(n_rows, np.uint8)
    check(lib().ygg_validation_split_mask(C.c_uint32(random_seed), C.c_int64(n_rows), C.c_float(validation_ratio),
                                          ptr(m, C.c_uint8)))
    return m.astype(bool)


def gen_discretized_boundaries(values, counts, maximum_num_bins, min_obs_in_bins, special_values=()):
    """GenDiscretizedBoundaries on explicit (unique value, count) candidates (host)."""
    v = np.ascontiguousarray(values, dtype=np.float32)
    c = np.ascontiguousarray(counts, dtype=np.int64)
    sp = np.ascontiguousarray(special_values, dtype=np.float32)
    out = np.empty(len(v) + 2 * len(sp) + 4, np.float32)
    n = C.c_int32()
    st = lib().ygg_gen_discretized_boundaries(ptr(v, C.c_float), ptr(c, C.c_int64), C.c_int64(len(v)),
                                              C.c_int32(maximum_num_bins), C.c_int32(min_obs_in_bins),
                                              ptr(sp, C.c_float), C.c_int32(len(sp)), ptr(out, C.c_float),
                                              C.c_int32(len(out)), C.byref(n))
    if st != 0:
        raise YggError(st, "ygg_gen_discretized_boundaries: invalid argument")
    return out[:n.value].copy()


class Comm:
    """NCCL communicator owned by the native library (include/ygg_b200_comm.h): the collectives of the
    level loop are issued from C++ on the engine's stream.  `unique_id()` on rank 0, ship the 128 bytes
    to the other ranks (e.g. torch.distributed.broadcast), then Comm(id, rank, world, device)."""

    def __init__(self, unique_id: bytes, rank: int, world: int, device: int = 0):
        assert len(unique_id) == 128
        self.handle = C.c_void_p()
        self.rank, self.world = rank, world
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        check(lib().ygg_comm_create(C.byref(self.handle), buf, C.c_int32(rank), C.c_int32(world),
                                    C.c_int32(device)))

    @staticmethod
    def unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        check(lib().ygg_comm_unique_id(buf))
        return bytes(buf)

    @classmethod
    def from_torch_distributed(cls, device: int):
        """Bootstraps over an initialised torch.distributed process group (any backend)."""
        import torch
        import torch.distributed as dist
        rank, world = dist.get_rank(), dist.get_world_size()
        dev = torch.device(f"cuda:{device}") if dist.get_backend() == "nccl" else torch.device("cpu")
        t = torch.zeros(128, dtype=torch.uint8, device=dev)
        if rank == 0:
            t.copy_(torch.frombuffer(bytearray(cls.unique_id()), dtype=torch.uint8))
        dist.broadcast(t, src=0)
        return cls(bytes(t.cpu().numpy().tobytes()), rank, world, device)

    def close(self):
        if self.handle:
            lib().ygg_comm_destroy(self.handle)
            self.handle = C.c_void_p()


class Gbt:
    """Boosting state on one GPU (ygg_gbt)."""

    def __init__(self, dataset, cfg):
        self.dataset = dataset
        self.cfg = cfg
        self.handle = C.c_void_p()
        self._cb = None
        check(lib().ygg_gbt_create(C.byref(self.handle), dataset.handle, C.byref(cfg)))

    def close(self):
        if self.handle:
            lib().ygg_gbt_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_labels(self, labels):
        if self.cfg.loss in (0, 2):   # binomial {1, 2} / multinomial {1..K}
            l = np.ascontiguousarray(labels, dtype=np.int32)
            check(lib().ygg_gbt_set_labels_i32(self.handle, ptr(l, C.c_int32), C.c_int64(len(l))))
        else:
            l = np.ascontiguousarray(labels, dtype=np.float32)
            check(lib().ygg_gbt_set_labels_f32(self.handle, ptr(l, C.c_float), C.c_int64(len(l))))

    def set_weights(self, weights):
        """Example weights of the training rows (before set_labels): weighted histograms, leaves, losses, initial predictions."""
        w = np.ascontiguousarray(weights, dtype=np.float32)
        check(lib().ygg_gbt_set_weights_f32(self.handle, ptr(w, C.c_float), C.c_int64(len(w))))
        self._weighted = True

    def set_validation(self, dataset, labels, weights=None):
        """Held-out rows (same features / binning): validation loss per iteration + cfg.early_stopping."""
        self._set_validation(dataset, labels)
        if weights is not None:
            w = np.ascontiguousarray(weights, dtype=np.float32)
            check(lib().ygg_gbt_set_validation_weights_f32(self.handle, ptr(w, C.c_float), C.c_int64(len(w))))

    def _set_validation(self, dataset, labels):
        self._valid = dataset
        if self.cfg.loss in (0, 2):
            l = np.ascontiguousarray(labels, dtype=np.int32)
            check(lib().ygg_gbt_set_validation_i32(self.handle, dataset.handle, ptr(l, C.c_int32), C.c_int64(len(l))))
        else:
            l = np.ascontiguousarray(labels, dtype=np.float32)
            check(lib().ygg_gbt_set_validation_f32(self.handle, dataset.handle, ptr(l, C.c_float), C.c_int64(len(l))))

    def validation_loss(self, it):
        a, b = C.c_float(), C.c_float()
        check(lib().ygg_gbt_validation_loss(self.handle, C.c_int32(it), C.byref(a), C.byref(b)))
        return a.value, b.value

    def num_iterations(self):
        return int(lib().ygg_gbt_num_iterations(self.handle))

    def final_validation(self):
        """-> (Header.validation_loss, Header.early_stopping_triggered)."""
        a, t = C.c_float(), C.c_int32()
        check(lib().ygg_gbt_final_validation(self.handle, C.byref(a), C.byref(t)))
        return a.value, bool(t.value)

    def set_feature_shard(self, begin, end, rank, world, allgather=None):
        """allgather: a Comm (NCCL, called from C++ without touching Python), or a Python callable
        allgather(send_ptr, recv_ptr, nbytes, stream_ptr) -> int, called once per tree level."""
        self._hist_features = (int(begin), int(end))
        if isinstance(allgather, Comm):
            self._comm = allgather
            fn = C.cast(lib().ygg_comm_allgather, ALLGATHER_FN)
            check(lib().ygg_gbt_set_feature_shard(self.handle, C.c_int32(begin), C.c_int32(end),
                                                  C.c_int32(rank), C.c_int32(world), fn, allgather.handle))
            return
        if allgather is not None:
            def _cb(ctx, send, recv, nbytes, stream):
                try:
                    return int(allgather(send, recv, nbytes, stream) or 0)
                except Exception:  # never let an exception cross the C boundary
                    import traceback
                    traceback.print_exc()
                    return 1
            self._cb = ALLGATHER_FN(_cb)
            fn = self._cb
        else:
            fn = C.cast(None, ALLGATHER_FN)
        check(lib().ygg_gbt_set_feature_shard(self.handle, C.c_int32(begin), C.c_int32(end),
                                              C.c_int32(rank), C.c_int32(world), fn, None))

    def set_row_shard_scatter(self, rank, world, n_rows_global, initial_prediction, comm=None, allreduce=None,
                              reducescatter=None, allgather=None):
        """Row shards with one reduce-scatter (by feature chunk) + one all-gather of the best splits per level.
        Pass a Comm (NCCL from C++), or three Python callables (same conventions as set_row_shard /
        set_feature_shard; reducescatter(buf_ptr, count_per_rank, dtype, op, stream_ptr))."""
        if comm is not None:
            self._comm = comm
            fns = (C.cast(lib().ygg_comm_allreduce, ALLREDUCE_FN), C.cast(lib().ygg_comm_reducescatter, REDUCESCATTER_FN),
                   C.cast(lib().ygg_comm_allgather, ALLGATHER_FN))
            ctx = comm.handle
        elif allreduce is None:
            fns = (C.cast(None, ALLREDUCE_FN), C.cast(None, REDUCESCATTER_FN), C.cast(None, ALLGATHER_FN))
            ctx = None
        else:
            def wrap(fn, nargs):
                def _cb(ctx, *a):
                    try:
                        return int(fn(*a) or 0)
                    except Exception:
                        import traceback
                        traceback.print_exc()
                        return 1
                return _cb
            self._cbs = (ALLREDUCE_FN(wrap(allreduce, 5)), REDUCESCATTER_FN(wrap(reducescatter, 5)),
                         ALLGATHER_FN(wrap(allgather, 4)))
            fns, ctx = self._cbs, None
        check(lib().ygg_gbt_set_row_shard_scatter(self.handle, C.c_int32(rank), C.c_int32(world),
                                                  C.c_int64(n_rows_global), C.c_float(initial_prediction),
                                                  fns[0], fns[1], fns[2], ctx))

    def set_row_shard(self, rank, world, n_rows_global, initial_prediction, allreduce=None):
        """allreduce: a Comm (NCCL from C++), or a Python callable
        allreduce(buf_ptr, count, dtype, op, stream_ptr) -> int; dtype 0=u32 1=u64 2=f64, op 0=sum 1=max."""
        if isinstance(allreduce, Comm):
            self._comm = allreduce
            fn = C.cast(lib().ygg_comm_allreduce, ALLREDUCE_FN)
            check(lib().ygg_gbt_set_row_shard(self.handle, C.c_int32(rank), C.c_int32(world),
                                              C.c_int64(n_rows_global), C.c_float(initial_prediction), fn,
                                              allreduce.handle))
            return
        if allreduce is not None:
            def _cb(ctx, buf, count, dtype, op, stream):
                try:
                    return int(allreduce(buf, count, dtype, op, stream) or 0)
                except Exception:
                    import traceback
                    traceback.print_exc()
                    return 1
            self._cb = ALLREDUCE_FN(_cb)
            fn = self._cb
        else:
            fn = C.cast(None, ALLREDUCE_FN)
        check(lib().ygg_gbt_set_row_shard(self.handle, C.c_int32(rank), C.c_int32(world),
                                          C.c_int64(n_rows_global), C.c_float(initial_prediction), fn, None))

    def initial_prediction(self):
        v = C.c_float()
        check(lib().ygg_gbt_initial_prediction(self.handle, C.byref(v)))
        return v.value

    def train(self, num_iters, stop_flag=None):
        check(lib().ygg_gbt_train(self.handle, C.c_int32(num_iters), stop_flag))

    def train_timed(self, num_iters):
        """Returns (device milliseconds, kernel launches) for `num_iters` iterations."""
        ms, n = C.c_double(), C.c_int64()
        check(lib().ygg_gbt_train_timed(self.handle, C.c_int32(num_iters), C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def step(self):
        check(lib().ygg_gbt_step(self.handle))

    def sync(self):
        check(lib().ygg_gbt_sync(self.handle))

    def num_trees(self):
        return int(lib().ygg_gbt_num_trees(self.handle))

    def use_peer_windows(self, comm):
        """Best-split exchange over NVLink peer memory (ygg_gbt_set_best_split_window) instead of the all-gather."""
        L = lib()
        L.ygg_gbt_best_split_window_bytes.restype = C.c_int64
        nbytes = int(L.ygg_gbt_best_split_window_bytes(self.handle))
        peers = (C.c_void_p * comm.world)()
        check(L.ygg_comm_window_create(comm.handle, C.c_int64(nbytes), peers))
        check(L.ygg_gbt_set_best_split_window(self.handle, peers, C.c_int32(comm.world)))

    def set_tie_rng_position(self, words):
        check(lib().ygg_gbt_set_tie_rng_position(self.handle, C.c_uint64(int(words))))

    def tie_stats(self):
        """(renamed, unresolved) tied nodes of the trees trained so far (cfg.candidate_shuffle != 0)."""
        a, b = C.c_int64(), C.c_int64()
        check(lib().ygg_gbt_tie_stats(self.handle, C.byref(a), C.byref(b)))
        return a.value, b.value

    def get_tree(self, it):
        cap = (1 << (self.cfg.max_depth + (1 if self.cfg.growing_strategy == 1 else 0)))   # best-first: root depth 0
        out = np.zeros(cap, dtype=NODE_DTYPE)
        n = C.c_int32()
        check(lib().ygg_gbt_get_tree(self.handle, C.c_int32(it), out.ctypes.data_as(C.c_void_p),
                                     C.c_int32(cap), C.byref(n)))
        return out[:n.value].copy()

    def get_category_sets(self, it, tree=None):
        """{pre-order node index: uint32 words} of the splits of tree `it` on wide categorical columns (bit c of
        words[c // 32] set: category c is positive); `it` = -1: the tree of the last train_tree_on_gradients call.
        `tree`: that tree, if already fetched (required for -1)."""
        wide = getattr(self.dataset, "wide", {})
        if not wide:
            return {}
        t = self.get_tree(it) if tree is None else tree
        out = {}
        for i in np.flatnonzero((t["condition_type"] == FEATURE_CATEGORICAL) & (t["feature"] >= 0)):
            f = int(t["feature"][i])
            if f not in wide:
                continue
            words = np.zeros((wide[f][0] + 31) // 32, np.uint32)
            n = C.c_int32()
            check(lib().ygg_gbt_get_category_set(self.handle, C.c_int32(it), C.c_int32(int(i)), ptr(words, C.c_uint32),
                                                 C.c_int32(len(words)), C.byref(n)))
            out[int(i)] = words
        return out

    def train_loss(self, it):
        a, b = C.c_float(), C.c_float()
        check(lib().ygg_gbt_train_loss(self.handle, C.c_int32(it), C.byref(a), C.byref(b)))
        return a.value, b.value

    def get_predictions(self):
        """Training predictions: [n]; multinomial loss: [n, K] (the engine holds them as K planes)."""
        k = self.cfg.num_classes if self.cfg.loss == 2 else 1
        out = np.empty(self.dataset.n_rows * k, dtype=np.float32)
        check(lib().ygg_gbt_get_predictions(self.handle, ptr(out, C.c_float), C.c_int64(len(out))))
        return out if k == 1 else np.ascontiguousarray(out.reshape(k, self.dataset.n_rows).T)

    def predict(self, dataset):
        """Raw scores of the trained model on `dataset` (same features / binning): [n], or [n, K] for the multinomial loss
        (the layout of get_predictions)."""
        n = int(lib().ygg_dataset_num_rows(dataset.handle))
        K = int(self.cfg.num_classes) if self.cfg.loss == 2 else 1
        out = np.empty(n * K, dtype=np.float32)
        check(lib().ygg_gbt_predict(self.handle, dataset.handle, ptr(out, C.c_float), C.c_int64(n * K)))
        return out if K == 1 else np.ascontiguousarray(out.reshape(K, n).T)

    def set_predictions(self, pred):
        p = np.ascontiguousarray(pred, dtype=np.float32)
        check(lib().ygg_gbt_set_predictions(self.handle, ptr(p, C.c_float), C.c_int64(len(p))))

    def train_tree_on_gradients(self, g, h=None):
        g = np.ascontiguousarray(g, dtype=np.float32)
        h = None if h is None else np.ascontiguousarray(h, dtype=np.float32)
        cap = (1 << (self.cfg.max_depth + (1 if self.cfg.growing_strategy == 1 else 0)))
        out = np.zeros(cap, dtype=NODE_DTYPE)
        n = C.c_int32()
        check(lib().ygg_tree_train_on_gradients(self.handle, ptr(g, C.c_float), ptr(h, C.c_float),
                                                out.ctypes.data_as(C.c_void_p), C.c_int32(cap),
                                                C.byref(n)))
        return out[:n.value].copy()

    def hist_plan(self, level):
        """The k_hist / k_hist2 launch the handle runs at tree level `level` (HistPlan)."""
        p = HistPlan()
        check(lib().ygg_debug_hist_plan(self.handle, C.c_int32(level), C.byref(p)))
        return p

    def level_histogram(self, level, g, slot_of_row, n_slots, second=None, plan=None):
        """Raw integer histograms of one tree level run by the training code (ygg_debug_level_histogram): rows with
        slot_of_row[r] = s >= 0 go to slot s.  -> (sum u64, count u32, second-plane sum u64 or None) of shape
        [n_slots, features histogrammed by this handle, 256], and (P, V): the scales of g and of the second plane."""
        g = np.ascontiguousarray(g, dtype=np.float32)
        slots = np.ascontiguousarray(slot_of_row, dtype=np.int32)
        v = None if second is None else np.ascontiguousarray(second, dtype=np.float32)
        lo, hi = self.hist_features()
        shape = (int(n_slots), hi - lo, 256)
        s = np.zeros(shape, np.uint64)
        c = np.zeros(shape, np.uint32)
        s2 = None if v is None else np.zeros(shape, np.uint64)
        scales = np.zeros(2, np.float32)
        check(lib().ygg_debug_level_histogram(self.handle, C.c_int32(level), None if plan is None else C.byref(plan),
                                              ptr(g, C.c_float), ptr(v, C.c_float), ptr(slots, C.c_int32),
                                              C.c_int32(n_slots), ptr(s, C.c_uint64), ptr(c, C.c_uint32),
                                              ptr(s2, C.c_uint64), ptr(scales, C.c_float)))
        return s, c, s2, (float(scales[0]), float(scales[1]))

    def wide_histogram(self, n_slots):
        """Raw wide-column histograms of the last histogram phase (a training level or level_histogram):
        (sum u64, count u32, second-plane sum u64 or None), each [n_slots, sum of the wide features' buckets]."""
        total = sum(nb for nb, _ in getattr(self.dataset, "wide", {}).values())
        s = np.zeros((int(n_slots), total), np.uint64)
        c = np.zeros((int(n_slots), total), np.uint32)
        s2 = np.zeros((int(n_slots), total), np.uint64) if self.has_second_plane() else None
        check(lib().ygg_debug_wide_histogram(self.handle, C.c_int32(int(n_slots)), ptr(s, C.c_uint64), ptr(c, C.c_uint32),
                                             ptr(s2, C.c_uint64)))
        return s, c, s2

    def has_second_plane(self):
        """True when the handle accumulates a second histogram plane: hessians (hessian gain with a logit loss) or
        example weights (the caller's or GOSS's)."""
        weighted = getattr(self, "_weighted", False) or self.cfg.goss_alpha > 0 or self.cfg.goss_beta > 0
        logit = self.cfg.loss in (0, 2)   # binomial / multinomial log-likelihood
        return bool((self.cfg.use_hessian_gain and (logit or weighted)) or weighted)

    def debug_histogram(self, g, node_of_row, node, feature):
        """Histogram of feature `feature` over the rows with node_of_row == node, dequantised: (sum of the quantised
        gradients per bin as float64, row count per bin), num_bins[feature] entries each.  A view of level_histogram: one
        slot at the root level, accumulated by the shared layout (exact for any rows) at the root's chunk size and grid."""
        lo, hi = self.hist_features()
        if not lo <= feature < hi:
            raise ValueError(f"feature {feature} outside the histogrammed features [{lo}, {hi})")
        slots = np.where(np.asarray(node_of_row) == node, 0, -1).astype(np.int32)
        root = self.hist_plan(0)
        p = HistPlan(HIST_SHARED, 1, 0, root.chunk_blocks, 0, root.grid)
        second = np.zeros(len(slots), np.float32) if self.has_second_plane() else None
        s, c, _, (P, _) = self.level_histogram(0, g, slots, 1, second=second, plan=p)
        nb = int(self.dataset.num_bins[feature])
        cnt = c[0, feature - lo, :nb].astype(np.int64)
        raw = s[0, feature - lo, :nb].astype(np.int64) - cnt * 2 ** 23   # exact: |raw| <= rows * 2^23 < 2^63
        return raw.astype(np.float64) * (P / 2.0 ** 23), cnt

    def set_candidate_sampling(self, num_candidate_attributes=-1, ratio=None):
        """Candidate feature sampling (ygg_gbt_set_candidate_sampling): each node tests the first k valid features of its
        keyed order; ratio None: not set.  Before the first tree."""
        check(lib().ygg_gbt_set_candidate_sampling(self.handle, C.c_int32(int(num_candidate_attributes)),
                                                   C.c_float(-1.0 if ratio is None else float(ratio))))

    def set_dart(self, dropout_rate):
        """DART (ygg_gbt_set_dart): per-iteration dropout of earlier iterations at `dropout_rate`.  Before the first tree."""
        check(lib().ygg_gbt_set_dart(self.handle, C.c_float(float(dropout_rate))))

    def dart_weights(self):
        """The per-iteration DART weights (float32 [iterations]); after train(), the final model's."""
        n = C.c_int32()
        cap = int(self.cfg.num_trees)
        out = np.zeros(max(cap, 1), np.float32)
        check(lib().ygg_gbt_get_dart_weights(self.handle, ptr(out, C.c_float), C.c_int32(cap), C.byref(n)))
        return out[:n.value].copy()

    def dart_dropped(self, it):
        """The iterations dropped at iteration `it` (int32, ascending)."""
        n = C.c_int32()
        out = np.zeros(max(int(it), 1), np.int32)
        check(lib().ygg_gbt_get_dart_dropped(self.handle, C.c_int32(int(it)), ptr(out, C.c_int32), C.c_int32(len(out)),
                                             C.byref(n)))
        return out[:n.value].copy()

    def level_tried(self, level):
        """The validity flags of tree level `level` of the last captured tree (sampling set before capture_candidates):
        (tried uint8 [level nodes, features scanned by this handle], node-table index of the level's first node)."""
        cap = 1 << max(0, self.cfg.max_depth - 1)
        lo, hi = self.hist_features()
        out = np.zeros((cap, hi - lo), np.uint8)
        first, n = C.c_int32(), C.c_int32()
        check(lib().ygg_debug_level_tried(self.handle, C.c_int32(int(level)), C.c_int32(cap), ptr(out, C.c_uint8),
                                          C.byref(first), C.byref(n)))
        return out[:n.value].copy(), first.value

    def capture_candidates(self, on=True):
        """Candidate capture (ygg_debug_capture_candidates): while on, every tree grown copies each level's complete
        candidate table as the scan phase left it, before the selection."""
        check(lib().ygg_debug_capture_candidates(self.handle, C.c_int32(int(bool(on)))))

    def level_candidates(self, level):
        """The captured candidates of tree level `level` of the last tree grown with capture on, as a dict of numpy arrays:
        per level node `node` (pre-order index in the emitted tree), `candidate`, `derived`, `num_examples`; per (level node,
        feature scanned by this handle) `found`, `score`, `threshold_bin`, `lo` / `hi` (-1 unless packed by the exact
        rule), `num_pos_examples`, `threshold_value`, `cat_mask` [.., 8] and, with wide categorical columns, `sets`
        [nodes, wide features, words]; and the tree's scales `P`, `h_pow2`, `w_pow2`."""
        cap = 1 << max(0, self.cfg.max_depth - 1)
        lo, hi = self.hist_features()
        nodes = np.zeros(cap, LEVEL_NODE_DTYPE)
        cands = np.zeros((cap, hi - lo), CANDIDATE_DTYPE)
        wide = getattr(self.dataset, "wide", {})
        words = max([(nb + 31) // 32 for f, (nb, _) in wide.items()
                     if self.dataset.feature_types[f] == FEATURE_CATEGORICAL] or [0])
        sets = np.zeros((cap, len(wide), words), np.uint32) if words else None
        n, scales = C.c_int32(), np.zeros(3, np.float32)
        check(lib().ygg_debug_level_candidates(self.handle, C.c_int32(int(level)), C.c_int32(cap),
                                               nodes.ctypes.data_as(C.c_void_p), cands.ctypes.data_as(C.c_void_p),
                                               ptr(sets, C.c_uint32), C.c_int32(words), C.byref(n), ptr(scales, C.c_float)))
        k = n.value
        out = {name: nodes[name][:k].copy() for name in ("node", "candidate", "derived", "num_examples")}
        out.update({name: cands[name][:k].copy() for name in CANDIDATE_DTYPE.names})
        if sets is not None:
            out["sets"] = sets[:k].copy()
        out["P"], out["h_pow2"], out["w_pow2"] = (float(x) for x in scales)
        return out

    def hist_features(self):
        """[begin, end) of the features this handle histograms (its feature shard, or all features)."""
        return getattr(self, "_hist_features", (0, self.dataset.n_features))

    def set_profiling(self, enabled=True):
        check(lib().ygg_gbt_set_profiling(self.handle, C.c_int32(int(enabled))))

    def get_profile(self, name):
        ms, n = C.c_double(), C.c_int64()
        check(lib().ygg_gbt_get_profile(self.handle, name.encode(), C.byref(ms), C.byref(n)))
        return ms.value, n.value


SHARD_BEST_DTYPE = np.dtype([("score", "<f4"), ("feature", "<i4"), ("threshold_bin", "<i4"),
                             ("num_pos_examples", "<i4"), ("condition_type", "<i4"), ("na_value", "<i4"),
                             ("cat_mask", "<u4", (8,))])
assert SHARD_BEST_DTYPE.itemsize == 56  # sizeof(ygg_shard_best)


def feature_shard(n_features, rank, world):
    b, e = C.c_int32(), C.c_int32()
    check(lib().ygg_feature_shard(C.c_int32(n_features), C.c_int32(rank), C.c_int32(world),
                                  C.byref(b), C.byref(e)))
    return b.value, e.value


def merge_shard_best(records):
    """records: [world, nodes] array of SHARD_BEST_DTYPE -> [nodes]."""
    r = np.ascontiguousarray(records, dtype=SHARD_BEST_DTYPE)
    world, nodes = r.shape
    out = np.zeros(nodes, dtype=SHARD_BEST_DTYPE)
    check(lib().ygg_merge_shard_best(r.ctypes.data_as(C.c_void_p), C.c_int32(world), C.c_int32(nodes),
                                     out.ctypes.data_as(C.c_void_p)))
    return out


def device_count():
    return int(lib().ygg_device_count())


def discretize_boundaries(values, maximum_num_bins=255, min_obs_in_bins=3):
    v = np.ascontiguousarray(values, dtype=np.float32)
    out = np.zeros(max(2, maximum_num_bins + 4), dtype=np.float32)
    n = C.c_int32()
    mean = C.c_double()
    check(lib().ygg_discretize_boundaries(ptr(v, C.c_float), C.c_int64(len(v)),
                                          C.c_int32(maximum_num_bins), C.c_int32(min_obs_in_bins),
                                          ptr(out, C.c_float), C.c_int32(len(out)), C.byref(n),
                                          C.byref(mean)))
    return out[:n.value].copy(), mean.value


def discretize_boundaries16(values, maximum_num_bins, min_obs_in_bins=3):
    """discretize_boundaries for maximum_num_bins in [2, 65535] (up to 65535 bins, for uint16 codes)."""
    v = np.ascontiguousarray(values, dtype=np.float32)
    out = np.zeros(maximum_num_bins + 4, dtype=np.float32)
    n = C.c_int32()
    mean = C.c_double()
    check(lib().ygg_discretize_boundaries16(ptr(v, C.c_float), C.c_int64(len(v)),
                                            C.c_int32(maximum_num_bins), C.c_int32(min_obs_in_bins),
                                            ptr(out, C.c_float), C.c_int32(len(out)), C.byref(n),
                                            C.byref(mean)))
    return out[:n.value].copy(), mean.value


def discretize_encode(values, boundaries, na_bin):
    v = np.ascontiguousarray(values, dtype=np.float32)
    b = np.ascontiguousarray(boundaries, dtype=np.float32)
    out = np.empty(len(v), dtype=np.uint8)
    check(lib().ygg_discretize_encode(ptr(v, C.c_float), C.c_int64(len(v)), ptr(b, C.c_float),
                                      C.c_int32(len(b)), C.c_int32(na_bin), ptr(out, C.c_uint8)))
    return out
