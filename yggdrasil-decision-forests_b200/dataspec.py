"""Column semantics and binning of the engine's input (DISCRETIZED_NUMERICAL and CATEGORICAL columns).

Mirrors what PYDF does when `discretize_numerical_columns=True`
(port/python/ydf/dataset/dataset.cc:192-316 -> dataset/data_spec.cc:854-1018): per column a sorted
boundary vector, `bin = upper_bound(boundaries, x)`, NA replaced by the bin of the column mean.
String columns become CATEGORICAL with the reference's dictionary rule: items rarer than min_vocab_frequency are
folded into index 0 (<OOD>), the rest are ordered by count, NA is replaced by the column's most_frequent_value.  The
reference has TWO front ends that differ in the details (`front_end=`):
  * FRONT_END_CPP  — the C++ dataspec inference used by the CSV / CLI path (dataset/data_spec_inference.cc:277-441):
    equal counts ordered by key DESCENDING (std::greater on (count, key) pairs), most_frequent_value = the most
    frequent item, so missing strings train as that item;
  * FRONT_END_PYDF — PYDF's in-memory path builds the column spec itself (port/python/ydf/dataset/dataset.cc:402-455,
    :510-564): equal counts ordered by key ASCENDING, max_vocab_count = -1 means "no limit" and 0 "only <OOD>", and
    most_frequent_value is never set, so a PYDF-trained model carries 0 and missing strings train as <OOD>.
Both are pinned on reference artefacts: the C++ rule on the dataspec of the golden CLI model, the PYDF rule on the
dictionary and on every split of the golden PYDF model adult_binary_class_gbdt_v2 (tests/test_reference_replay.py).
"""
import dataclasses
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _capi


@dataclasses.dataclass
class DiscretizedColumn:
    name: str
    boundaries: np.ndarray  # float32, sorted
    mean: float
    num_bins: int
    na_bin: int
    num_missing: int = 0
    num_values: int = 0
    bucket_values: Optional[np.ndarray] = None   # lossless columns: the value of every bucket (exact threshold rule)
    maximum_num_bins: Optional[int] = None        # the bin budget asked for above 256 (DiscretizedNumericalSpec)
    feature_type = _capi.FEATURE_DISCRETIZED_NUMERICAL

    @property
    def wide(self) -> bool:
        """More buckets than a byte holds: a wide column (uint16 codes, _capi.Dataset.set_wide_column, or without bucket
        values _capi.Dataset.set_wide_discretized_column)."""
        return self.num_bins > 256

    def encode(self, values) -> np.ndarray:
        return _capi.discretize_encode(np.asarray(values, dtype=np.float32), self.boundaries, self.na_bin)

    def encode16(self, values) -> np.ndarray:
        """uint16 codes by encode's rule (bucket = upper_bound(boundaries, x), NaN -> na_bin), for up to 65535 buckets."""
        if self.num_bins > 65535:
            raise ValueError(f"column {self.name!r}: {self.num_bins} buckets do not fit uint16 codes below 65535")
        v = np.asarray(values, dtype=np.float32)
        out = np.searchsorted(np.asarray(self.boundaries, dtype=np.float32), v, side="right").astype(np.uint16)
        out[np.isnan(v)] = self.na_bin
        return out


@dataclasses.dataclass
class PresortedColumn:
    """A numerical column kept as its float values (_capi.Dataset.set_numerical_column): the exact numerical splitter
    through sorted row lists, with no limit on distinct values.  Saved as a NUMERICAL column; its splits are Higher
    conditions (value >= threshold, a missing value takes the node's na_value)."""
    name: str
    mean: float               # NA replacement, NumericalSpec.mean
    min_value: float
    max_value: float
    num_missing: int = 0
    num_values: int = 0
    num_distinct: int = 0
    feature_type = _capi.FEATURE_NUMERICAL
    wide = False

    def encode(self, values) -> np.ndarray:
        """The float32 values themselves, NaN = missing."""
        return np.asarray(values, dtype=np.float32)


@dataclasses.dataclass
class CategoricalColumn:
    name: str
    vocabulary: List[str]     # index -> key; vocabulary[0] == "<OOD>"
    counts: List[int]
    num_bins: int             # number_of_unique_values
    na_bin: int               # most_frequent_value
    num_missing: int = 0
    num_values: int = 0
    feature_type = _capi.FEATURE_CATEGORICAL

    @property
    def wide(self) -> bool:
        """More categories than a byte holds: a wide categorical column (_capi.Dataset.set_wide_categorical_column)."""
        return self.num_bins > 256

    def _codes(self, values, dtype) -> np.ndarray:
        index = {k: i for i, k in enumerate(self.vocabulary) if i > 0}
        keys, na = _categorical_keys(values)
        out = np.fromiter((index.get(k, 0) for k in keys), dtype=dtype, count=len(keys))
        out[na] = self.na_bin
        return out

    def encode(self, values) -> np.ndarray:
        return self._codes(values, np.uint8)

    def encode16(self, values) -> np.ndarray:
        """uint16 codes by encode's rule (dictionary index, 0 = out-of-dictionary, missing -> na_bin), up to 65535."""
        if self.num_bins > 65535:
            raise ValueError(f"column {self.name!r}: {self.num_bins} categories do not fit uint16 codes below 65535")
        return self._codes(values, np.uint16)


def _categorical_keys(values):
    """-> (list of str keys, NA mask).  Missing: None, NaN, or the empty string (data_spec_inference.cc:716)."""
    v = np.asarray(values, dtype=object)
    keys, na = [], np.zeros(len(v), dtype=bool)
    for i, x in enumerate(v):
        if x is None or (isinstance(x, float) and x != x):
            na[i] = True
            keys.append("")
            continue
        k = x.decode() if isinstance(x, bytes) else str(x)
        if k == "":
            na[i] = True
        keys.append(k)
    return keys, na


FRONT_END_CPP = "cpp"     # C++ dataspec inference (CSV / CLI front end)
FRONT_END_PYDF = "pydf"   # PYDF in-memory front end


def infer_categorical_column(name: str, values, min_vocab_frequency: int = 5, max_vocab_count: int = 2000,
                             max_rows: Optional[int] = None, front_end: str = FRONT_END_CPP) -> CategoricalColumn:
    if front_end not in (FRONT_END_CPP, FRONT_END_PYDF):
        raise ValueError(f"front_end: {front_end!r}")
    pydf = front_end == FRONT_END_PYDF
    keys, na = _categorical_keys(values if max_rows is None else values[:max_rows])
    raw: Dict[str, int] = {}
    for k, is_na in zip(keys, na):
        if not is_na:
            raw[k] = raw.get(k, 0) + 1
    ood = 0 if pydf else raw.pop("<OOD>", 0)
    if pydf:
        # dataset.cc:428-436: large counts first, then keys in ascending byte order
        items = sorted(((c, k.encode()) for k, c in raw.items()), key=lambda it: (-it[0], it[1]))
        limit = max_vocab_count if max_vocab_count >= 0 else None
    else:
        # std::greater<std::pair<int64, std::string>>: count, then key (byte order), both descending
        items = sorted(((c, k.encode()) for k, c in raw.items()), reverse=True)
        limit = max_vocab_count if max_vocab_count > 0 else None
    kept = [it for it in items if it[0] >= min_vocab_frequency]
    ood += sum(c for c, _ in items) - sum(c for c, _ in kept)
    items = kept
    if limit is not None and len(items) > limit:
        ood += sum(c for c, _ in items[limit:])
        items = items[:limit]
    vocabulary = ["<OOD>"] + [k.decode() for _, k in items]
    counts = [ood] + [c for c, _ in items]
    if len(vocabulary) > 65535:
        raise NotImplementedError(
            f"column {name!r}: {len(vocabulary)} categories do not fit the engine's uint16 codes (at most 65535; "
            "raise min_vocab_frequency or lower max_vocab_count)")
    if pydf:
        most_frequent = 0
    else:
        # the first non-OOD item with the highest count, unless <OOD> is strictly more frequent
        most_frequent = 1 if (len(counts) > 1 and counts[1] >= counts[0]) else 0
    return CategoricalColumn(name=name, vocabulary=vocabulary, counts=counts, num_bins=len(vocabulary),
                             na_bin=most_frequent, num_missing=int(na.sum()), num_values=len(keys))


@dataclasses.dataclass
class DataSpec:
    columns: List  # DiscretizedColumn | CategoricalColumn
    label: str
    task: str
    label_classes: Optional[List] = None   # classification: class 1, class 2 (index 0 is OOD)
    label_mean: float = 0.0
    label_sd: float = 0.0
    label_min: float = 0.0
    label_max: float = 0.0
    num_rows: int = 0

    @property
    def feature_names(self) -> List[str]:
        return [c.name for c in self.columns]


def as_columns(ds) -> Dict[str, np.ndarray]:
    """Accepts a dict of arrays or a pandas DataFrame (the two in-memory inputs PYDF takes)."""
    if isinstance(ds, dict):
        return {k: np.asarray(v) for k, v in ds.items()}
    try:
        import pandas as pd
        if isinstance(ds, pd.DataFrame):
            return {c: ds[c].to_numpy() for c in ds.columns}
    except ImportError:
        pass
    raise TypeError("dataset must be a dict of numpy arrays or a pandas DataFrame")


def infer_column(name: str, values, maximum_num_bins: int = 255, min_obs_in_bins: int = 3,
                 max_rows: Optional[int] = None) -> DiscretizedColumn:
    v = np.asarray(values, dtype=np.float32)
    sample = v if (max_rows is None or len(v) <= max_rows) else v[:max_rows]
    boundaries, mean = _capi.discretize_boundaries(sample, maximum_num_bins, min_obs_in_bins)
    if len(boundaries) + 1 > 256:
        raise ValueError(f"column {name!r}: {len(boundaries) + 1} bins do not fit the engine's uint8 bins")
    # NumericalToDiscretizedNumerical(mean): training.cc:917-922
    na_bin = int(np.searchsorted(boundaries, np.float32(mean), side="right"))
    return DiscretizedColumn(name=name, boundaries=boundaries, mean=float(mean),
                             num_bins=len(boundaries) + 1, na_bin=na_bin,
                             num_missing=int(np.isnan(v).sum()), num_values=len(v))


def infer_column16(name: str, values, maximum_num_bins: int, min_obs_in_bins: int = 3,
                   max_rows: Optional[int] = None) -> DiscretizedColumn:
    """infer_column for up to 65535 bins: the same rule (GenDiscretizedBoundaries with the special values {0, mean}).  A column that ends with more than 256 bins is a discretized wide column (encode16); one with fewer a
    byte column, exactly as infer_column would make it."""
    v = np.asarray(values, dtype=np.float32)
    sample = v if (max_rows is None or len(v) <= max_rows) else v[:max_rows]
    boundaries, mean = _capi.discretize_boundaries16(sample, maximum_num_bins, min_obs_in_bins)
    if len(boundaries) + 1 > 65535:
        raise ValueError(f"column {name!r}: {len(boundaries) + 1} bins do not fit the engine's uint16 codes")
    na_bin = int(np.searchsorted(boundaries, np.float32(mean), side="right"))
    return DiscretizedColumn(name=name, boundaries=boundaries, mean=float(mean),
                             num_bins=len(boundaries) + 1, na_bin=na_bin,
                             num_missing=int(np.isnan(v).sum()), num_values=len(v),
                             maximum_num_bins=int(maximum_num_bins) if maximum_num_bins > 256 else None)


def infer_column_lossless(name: str, values, max_rows: Optional[int] = None,
                          max_distinct: int = 255) -> Optional[DiscretizedColumn]:
    """One bin per distinct value, for a numerical column with at most 255 of them (None otherwise).

    The discretized splitter then sees exactly the candidate cuts of the reference's EXACT numerical splitter (a
    threshold between two consecutive distinct values, `splitter_scanner.h:1230-1430`), so on such columns its splits
    partition the training rows like the exact splitter's — checked on three complete runs of the reference in
    tests/test_reference_replay.py.  Boundaries are the mid-points of consecutive distinct values, which is also where
    the exact splitter puts a threshold when both neighbours are present in the node; when values are absent from the
    node the two differ in the stored threshold VALUE (middle of the empty bins vs middle of the two present values),
    not in the partition of the training rows."""
    v = np.asarray(values, dtype=np.float32)
    sample = v if (max_rows is None or len(v) <= max_rows) else v[:max_rows]
    # every row's value must have its own bucket: the distinct set comes from ALL rows, whatever `max_rows` says
    # about the statistics (a value outside the sample would otherwise be merged into a neighbour's bucket)
    distinct = np.unique(v[~np.isnan(v)])
    if len(distinct) == 0 or len(distinct) > max_distinct:   # byte buckets, or wide columns up to max_distinct values
        return None
    mean = _exact_mean(sample, distinct)
    num_missing = int(np.isnan(v).sum())
    if num_missing > 0:
        # The exact splitter imputes NA with the column mean (training.cc:2385-2392, splitter_scanner.h:1230-1430): the
        # missing rows sort as a value of their own BETWEEN two distinct values and the splitter may cut on either
        # side of them.  Give the mean its own bucket (= na_bin) so that both cuts exist here too.
        distinct = np.unique(np.append(distinct, np.float32(mean)))
        if len(distinct) > max(256, max_distinct + 1):
            return None
    lo, hi = distinct[:-1], distinct[1:]
    mid = (lo.astype(np.float64) + hi.astype(np.float64)) / 2
    boundaries = mid.astype(np.float32)
    boundaries = np.where(boundaries > lo, boundaries, hi).astype(np.float32)   # adjacent floats: the mid-point rounds down
    na_bin = int(np.searchsorted(boundaries, np.float32(mean), side="right"))
    return DiscretizedColumn(name=name, boundaries=boundaries, mean=mean, num_bins=len(boundaries) + 1, na_bin=na_bin,
                             num_missing=num_missing, num_values=len(v), bucket_values=distinct.astype(np.float32))


def _exact_mean(sample: np.ndarray, distinct: np.ndarray) -> float:
    """The exact splitter's NA replacement: the mean of the present values of the statistics sample (the first
    max_num_scanned_rows_to_compute_statistics rows), else of the distinct values of the whole column."""
    present = sample[~np.isnan(sample)]
    return float(present.astype(np.float64).mean()) if len(present) else float(distinct.astype(np.float64).mean())


def infer_column_presorted(name: str, values, max_rows: Optional[int] = None) -> Optional[PresortedColumn]:
    """A presorted numerical column (any number of distinct values; None for a column without a present value).  Its
    mean is infer_column_lossless's, from the same sample."""
    v = np.asarray(values, dtype=np.float32)
    sample = v if (max_rows is None or len(v) <= max_rows) else v[:max_rows]
    distinct = np.unique(v[~np.isnan(v)])
    if len(distinct) == 0:
        return None
    return PresortedColumn(name=name, mean=_exact_mean(sample, distinct), min_value=float(distinct[0]),
                           max_value=float(distinct[-1]), num_missing=int(np.isnan(v).sum()), num_values=len(v),
                           num_distinct=len(distinct))


def _presorted(c) -> bool:
    return c.feature_type == _capi.FEATURE_NUMERICAL


def encode_features(cols: Dict[str, np.ndarray], columns: Sequence[DiscretizedColumn]) -> np.ndarray:
    """[features, rows] bucket indices: uint8, or uint16 when a column has more than 256 buckets (wide columns).  With a
    presorted numerical column the matrix is float64: its rows hold the float32 values (NaN = missing), the others their
    bucket indices (exact in float64)."""
    n = len(next(iter(cols.values())))
    presorted = any(_presorted(c) for c in columns)
    wide = any(not _presorted(c) and c.num_bins > 256 for c in columns)
    out = np.empty((len(columns), n), dtype=np.float64 if presorted else (np.uint16 if wide else np.uint8))
    for i, c in enumerate(columns):
        out[i] = c.encode(cols[c.name]) if _presorted(c) or c.num_bins <= 256 else c.encode16(cols[c.name])
    return out


def device_dataset(bins: np.ndarray, columns: Sequence, device: int = 0) -> "_capi.Dataset":
    """The device dataset of encode_features' output: byte columns as they are, wide columns (more than 256 buckets)
    attached with their codes (and, exact numerical, their bucket values and mean), presorted numerical columns with
    their values and mean."""
    wide = [i for i, c in enumerate(columns) if _presorted(c) or c.num_bins > 256]
    byte_bins = np.zeros(bins.shape, np.uint8) if bins.dtype != np.uint8 else bins
    if bins.dtype != np.uint8:
        narrow = [i for i in range(len(columns)) if i not in set(wide)]
        byte_bins[narrow] = bins[narrow]
    num_bins = [1 if i in wide else c.num_bins for i, c in enumerate(columns)]
    na_bin = [0 if i in wide else c.na_bin for i, c in enumerate(columns)]
    # (a presorted column starts as a numerical one: set_numerical_column makes it FEATURE_NUMERICAL)
    types = [_capi.FEATURE_DISCRETIZED_NUMERICAL if _presorted(c) else c.feature_type for c in columns]
    ds = _capi.Dataset(byte_bins, num_bins, na_bin, device=device, feature_types=types)
    try:
        for i in wide:
            c = columns[i]
            if _presorted(c):
                ds.set_numerical_column(i, bins[i], c.mean)
            elif c.feature_type == _capi.FEATURE_CATEGORICAL:
                ds.set_wide_categorical_column(i, bins[i], c.num_bins, c.na_bin)
            elif c.bucket_values is None:   # discretized: no bucket values
                ds.set_wide_discretized_column(i, bins[i], c.num_bins, c.na_bin)
            else:
                ds.set_wide_column(i, bins[i], c.num_bins, c.na_bin, c.bucket_values, c.mean)
    except Exception:
        ds.close()
        raise
    return ds
