"""GradientBoostedTreesLearner — host-side mirror of the reference learner for the histogram path.

Same constructor names, meaning and error behaviour as PYDF's
`ydf.GradientBoostedTreesLearner` (port/python/ydf/learner/specialized_learners_pre_generated.py:
1847-1930, wrapping GradientBoostedTreesLearner::TrainWithStatusImpl,
learner/gradient_boosted_trees/gradient_boosted_trees.cc:1154) for the hyper-parameters the hot
path reads, DART's forest extraction included.  Options that select code outside the path (the
random categorical splitter, other losses ...) raise NotImplementedError instead of being ignored.
"""
import os
import warnings
from typing import List, Optional

import numpy as np

from . import _capi
from . import dataspec as ds_lib
from .model import GradientBoostedTreesModel


class Task:
    CLASSIFICATION = "CLASSIFICATION"
    REGRESSION = "REGRESSION"


_LOSS_ID = {"BINOMIAL_LOG_LIKELIHOOD": 0, "SQUARED_ERROR": 1, "MULTINOMIAL_LOG_LIKELIHOOD": 2}
_EARLY_STOPPING = {"NONE": 0, "MIN_LOSS_FINAL": 1, "LOSS_INCREASE": 2}
_TIE_BREAK = {"FEATURE_ORDER": 0, "LIBSTDCXX_SHUFFLE": 1, "LIBCXX_SHUFFLE": 2}


class GradientBoostedTreesLearner:
    def __init__(self,
                 label: str,
                 task: str = Task.CLASSIFICATION,
                 *,
                 features: Optional[List[str]] = None,
                 weights: Optional[str] = None,
                 discretize_numerical_columns: bool = False,
                 max_exact_numerical_values: int = 255,
                 presort_numerical_columns: bool = False,
                 num_discretized_numerical_bins: int = 255,
                 max_num_scanned_rows_to_compute_statistics: Optional[int] = None,
                 min_vocab_frequency: int = 5,
                 max_vocab_count: int = 2000,
                 categorical_algorithm: str = "CART",
                 categorical_arity_limit_for_random: int = 300,
                 num_trees: int = 300,
                 shrinkage: float = 0.1,
                 max_depth: int = 6,
                 min_examples: int = 5,
                 in_split_min_examples_check: bool = True,
                 use_hessian_gain: bool = False,
                 l1_regularization: float = 0.0,
                 l2_regularization: float = 0.0,
                 l2_categorical_regularization: float = 1.0,
                 clamp_leaf_logit: float = 5.0,
                 loss: str = "DEFAULT",
                 validation_ratio: float = 0.1,
                 early_stopping: str = "LOSS_INCREASE",
                 early_stopping_num_trees_look_ahead: int = 30,
                 early_stopping_initial_iteration: int = 10,
                 validation_interval_in_trees: int = 1,
                 subsample: float = 1.0,
                 sampling_method: Optional[str] = None,
                 goss_alpha: float = 0.2,
                 goss_beta: float = 0.1,
                 growing_strategy: str = "LOCAL",
                 max_num_nodes: int = 31,
                 num_candidate_attributes: int = -1,
                 num_candidate_attributes_ratio: Optional[float] = None,
                 forest_extraction: str = "MART",
                 dart_dropout: Optional[float] = None,
                 random_seed: int = 123456,
                 num_threads: Optional[int] = None,
                 sibling_subtraction: bool = True,
                 tie_break: str = "LIBCXX_SHUFFLE",
                 device: int = 0):
        self.label = label
        self.task = task
        self.features = features
        self.num_discretized_numerical_bins = int(num_discretized_numerical_bins)
        self.max_rows_stats = max_num_scanned_rows_to_compute_statistics
        self.device = device
        self.min_vocab_frequency = int(min_vocab_frequency)
        self.max_vocab_count = int(max_vocab_count)
        if categorical_algorithm != "CART":
            raise NotImplementedError("only categorical_algorithm=CART is implemented")
        # The reference's Categorical.arity_limit_for_random (decision_tree.proto:573-576, default 300): a column with at
        # least that many categories is split with the RANDOM algorithm whatever categorical_algorithm says
        # (training.cc:3214-3217, :3292-3295).  RANDOM is not built (DESIGN.md §21), so such columns are refused, not
        # approximated; raising the limit asks the reference for CART on them too, which is what the engine computes.
        if isinstance(categorical_arity_limit_for_random, bool) or \
                not isinstance(categorical_arity_limit_for_random, (int, np.integer)):
            raise TypeError("categorical_arity_limit_for_random must be an integer")
        if int(categorical_arity_limit_for_random) < 1:
            raise ValueError("categorical_arity_limit_for_random must be >= 1")
        self.categorical_arity_limit_for_random = int(categorical_arity_limit_for_random)
        # weights: name of a numerical column holding one non-negative weight per example (PYDF's `weights` argument ->
        # TrainingConfig.weight_definition); the column is not a feature.  Implemented for the variance gain, all three
        # losses (ygg_gbt_set_weights_f32).
        if weights is not None and use_hessian_gain:
            raise NotImplementedError("example weights are implemented for use_hessian_gain=False only (SURVEY.md §8f N3)")
        self.weights = weights
        # discretize_numerical_columns=False (the reference's default) asks for the EXACT numerical splitter.  This engine
        # is the bucketised split finder, but with one bucket per distinct value it examines exactly the exact splitter's
        # candidate cuts (dataspec.infer_column_lossless; default runs of the reference replayed that way in
        # tests/test_reference_replay.py), so the option is honoured for columns with at most 255 distinct values (byte
        # buckets), for wider ones up to max_exact_numerical_values (wide columns), and for the others refused — not
        # approximated — or, with presort_numerical_columns, split through sorted row lists (_build_dataset).
        self.discretize_numerical_columns = bool(discretize_numerical_columns)
        # The largest numerical column (distinct values) the exact splitter takes.  Columns of up to 255 values use byte
        # buckets; wider ones, up to this limit, become wide columns (uint16 buckets, DESIGN.md §20), whose histogram
        # memory grows with their buckets: a resource bound, like max_vocab_count.
        if isinstance(max_exact_numerical_values, bool) or not isinstance(max_exact_numerical_values, (int, np.integer)):
            raise TypeError("max_exact_numerical_values must be an integer")
        if not 255 <= int(max_exact_numerical_values) <= 65535:
            raise ValueError(f"max_exact_numerical_values={max_exact_numerical_values} outside [255, 65535] "
                             "(wide columns hold at most 65535 buckets)")
        self.max_exact_numerical_values = int(max_exact_numerical_values)
        # With the exact splitter, a numerical column with more distinct values than max_exact_numerical_values becomes a
        # presorted column (float values split through sorted row lists, DESIGN.md §22) instead of being refused.
        self.presort_numerical_columns = bool(presort_numerical_columns)
        if not 0.0 <= validation_ratio <= 1.0:
            raise ValueError("The validation set ratio should be in [0,1].")
        if early_stopping not in _EARLY_STOPPING:
            raise ValueError(f"unknown early_stopping {early_stopping!r}")
        if validation_interval_in_trees != 1:
            raise NotImplementedError("only validation_interval_in_trees=1 is implemented")
        self.validation_ratio = float(validation_ratio)
        # sampling_method: NONE / RANDOM (stochastic gradient boosting with `subsample`, gradient_boosted_trees.cc:2932-2956) /
        # GOSS (gradient-based one-side sampling, :2958-3007); the deprecated bare `subsample` means RANDOM, as in the
        # reference (:3222-3236).  SELGB (ranking) is not built.
        if sampling_method not in (None, "NONE", "RANDOM", "GOSS"):
            raise NotImplementedError(f"sampling_method {sampling_method} is outside the accelerated path (SURVEY.md §8f N3)")
        if not 0.0 < subsample <= 1.0:
            raise ValueError("subsample must be in (0, 1]")
        self.subsample = 1.0 if sampling_method in ("NONE", "GOSS") else float(subsample)
        self.goss = sampling_method == "GOSS"
        if self.goss:
            if not (0.0 <= goss_alpha <= 1.0 and 0.0 <= goss_beta <= 1.0) or goss_alpha + goss_beta == 0.0:
                raise ValueError("goss_alpha and goss_beta must be in [0, 1], not both 0")
            if use_hessian_gain or weights is not None:
                raise NotImplementedError("GOSS is implemented for use_hessian_gain=False without example weights")
        self.goss_alpha, self.goss_beta = (float(goss_alpha), float(goss_beta)) if self.goss else (0.0, 0.0)
        if growing_strategy not in ("LOCAL", "BEST_FIRST_GLOBAL"):
            raise ValueError(f"unknown growing_strategy {growing_strategy!r}")
        self.growing_strategy = growing_strategy
        # Candidate feature sampling (DecisionTreeTrainingConfig.num_candidate_attributes / _ratio): each node is split on
        # the best of k features taken in a per-node random order (ygg_gbt_set_candidate_sampling, DESIGN.md §23).
        # -1 / None: every feature; 0 or a ratio of 0: the task's default (sqrt(F) classification, F/3 regression).
        if isinstance(num_candidate_attributes, bool) or not isinstance(num_candidate_attributes, (int, np.integer)):
            raise TypeError("num_candidate_attributes must be an integer")
        if int(num_candidate_attributes) < -1:
            raise ValueError("num_candidate_attributes must be >= -1 (-1: every feature, 0: the task's default)")
        if num_candidate_attributes_ratio is not None:
            if isinstance(num_candidate_attributes_ratio, bool) or \
                    not isinstance(num_candidate_attributes_ratio, (int, float, np.integer, np.floating)):
                raise TypeError("num_candidate_attributes_ratio must be a number or None")
            if not 0.0 <= float(num_candidate_attributes_ratio) <= 1.0:
                raise ValueError("num_candidate_attributes_ratio must be in [0, 1]")
            if int(num_candidate_attributes) != -1:
                raise ValueError("Only one of the following hyperparameters can be set: num_candidate_attributes, "
                                 "num_candidate_attributes_ratio")
        self.num_candidate_attributes = int(num_candidate_attributes)
        self.num_candidate_attributes_ratio = (None if num_candidate_attributes_ratio is None
                                               else float(num_candidate_attributes_ratio))
        # forest_extraction: MART, or DART (per-iteration dropout of earlier trees, rescaled trees in the model;
        # ygg_gbt_set_dart, DESIGN.md §24).  dart_dropout None: the reference's default rate, 0.01.
        if forest_extraction not in ("MART", "DART"):
            raise NotImplementedError(f"forest_extraction {forest_extraction!r} is not implemented (MART and DART are)")
        self.forest_extraction = forest_extraction
        if dart_dropout is not None:
            if isinstance(dart_dropout, bool) or not isinstance(dart_dropout, (int, float, np.integer, np.floating)):
                raise TypeError("dart_dropout must be a number or None")
            if not 0.0 <= float(dart_dropout) <= 1.0:
                raise ValueError("dart_dropout must be in [0, 1]")
        self.dart_dropout = 0.01 if dart_dropout is None else float(dart_dropout)
        if task == Task.CLASSIFICATION:
            if loss not in ("DEFAULT", "BINOMIAL_LOG_LIKELIHOOD", "MULTINOMIAL_LOG_LIKELIHOOD"):
                raise NotImplementedError(f"loss {loss} is outside the accelerated path")
            # DEFAULT: binomial for two classes, multinomial for more (gradient_boosted_trees.cc:2636-2650);
            # resolved when the label column is seen
            self.loss = "BINOMIAL_LOG_LIKELIHOOD" if loss == "BINOMIAL_LOG_LIKELIHOOD" else loss
        elif task == Task.REGRESSION:
            if loss not in ("DEFAULT", "SQUARED_ERROR"):
                raise NotImplementedError(f"loss {loss} is outside the accelerated path")
            self.loss = "SQUARED_ERROR"
        else:
            raise NotImplementedError(f"task {task} is outside the accelerated path")
        # up to 256 bins: byte columns; above, columns with more than 256 bins become discretized wide columns (uint16 codes,
        # DESIGN.md §25), whose histogram memory grows with their bins
        if not (2 <= self.num_discretized_numerical_bins <= 65535):
            raise ValueError("num_discretized_numerical_bins must be in [2, 65535] (uint16 bins)")
        self.cfg = _capi.default_config(
            loss=_LOSS_ID.get(self.loss, 0), num_trees=int(num_trees), shrinkage=float(shrinkage),
            max_depth=int(max_depth), min_examples=int(min_examples),
            in_split_min_examples_check=int(bool(in_split_min_examples_check)),
            use_hessian_gain=int(bool(use_hessian_gain)),
            l1_regularization=float(l1_regularization), l2_regularization=float(l2_regularization),
            l2_regularization_categorical=float(l2_categorical_regularization),
            clamp_leaf_logit=float(clamp_leaf_logit), random_seed=int(random_seed), subsample=self.subsample,
            sibling_subtraction=int(bool(sibling_subtraction)),
            early_stopping=_EARLY_STOPPING[early_stopping],
            early_stopping_num_trees_look_ahead=int(early_stopping_num_trees_look_ahead),
            early_stopping_initial_iteration=int(early_stopping_initial_iteration))
        self.num_threads = num_threads or os.cpu_count()
        # Features whose best splits have EQUAL float scores (twin columns such as Adult's education / education_num):
        # the reference takes the first in its per-node shuffle of the candidates on the learner's random engine
        # (training.cc:4293-4306).  The engine replays that stream on the finished trees (cfg.candidate_shuffle); the
        # shuffle ALGORITHM is the standard library's: the reference's golden models follow libc++'s.
        if tie_break not in _TIE_BREAK:
            raise ValueError(f"unknown tie_break {tie_break!r}: one of {sorted(_TIE_BREAK)}")
        self.cfg.goss_alpha, self.cfg.goss_beta = self.goss_alpha, self.goss_beta
        self.cfg.growing_strategy = int(self.growing_strategy == "BEST_FIRST_GLOBAL")
        self.cfg.max_num_nodes = int(max_num_nodes)
        # (the shuffle replay follows the depth-first order of the local growth)
        self.cfg.candidate_shuffle = 0 if self.cfg.growing_strategy else _TIE_BREAK[tie_break]
        self._candidate_shuffle = self.cfg.candidate_shuffle
        self.cfg.split_jobs_draw_seeds = int(self.num_threads > 1)   # FindBestConditionConcurrentManager, training.cc:1658

    # -- dataspec + device dataset -----------------------------------------------------------------
    def _build_dataset(self, cols):
        """Infers the dataspec and fills the device-resident dataset column by column: numerical columns
        are uploaded as float32 and binned ON THE GPU (csrc/ygg_binning.cu), string columns are
        dictionary-encoded on the host (dataspec.infer_categorical_column)."""
        if self.label not in cols:
            raise ValueError(f'label column "{self.label}" not found')
        names = self.features or [c for c in cols if c != self.label and c != self.weights]
        if self.weights is not None and self.weights in names:
            raise ValueError(f'the weight column "{self.weights}" cannot be a feature')
        n = len(cols[self.label])
        lossless, categorical, presorted = {}, {}, {}
        for name in names:   # string columns -> CATEGORICAL (PYDF's semantic inference), checked before the device
            if cols[name].dtype.kind in "OUS":
                # this learner mirrors PYDF, whose string columns keep most_frequent_value = 0 (dataspec.py)
                c = ds_lib.infer_categorical_column(name, cols[name], self.min_vocab_frequency, self.max_vocab_count,
                                                    self.max_rows_stats, ds_lib.FRONT_END_PYDF)
                if c.num_bins >= self.categorical_arity_limit_for_random:
                    raise NotImplementedError(
                        f'column "{name}" has {c.num_bins} categories (with <OOD>), at least '
                        f"categorical_arity_limit_for_random (= {self.categorical_arity_limit_for_random}): the reference "
                        "splits such columns with its random-mask algorithm, which is not built.  Raise "
                        "categorical_arity_limit_for_random to split them with CART (the reference's result for that "
                        "setting), or lower max_vocab_count / raise min_vocab_frequency")
                categorical[name] = c
        if not self.discretize_numerical_columns:   # checked before anything is created on the device
            for name in names:
                if cols[name].dtype.kind in "fiub":
                    limit = self.max_exact_numerical_values
                    lossless[name] = ds_lib.infer_column_lossless(name, cols[name], self.max_rows_stats, max_distinct=limit)
                    if lossless[name] is not None and lossless[name].num_bins <= 65535:
                        continue
                    # the path follows the column's cardinality: byte buckets, wide columns up to the limit, presorted above
                    if self.presort_numerical_columns:
                        presorted[name] = ds_lib.infer_column_presorted(name, cols[name], self.max_rows_stats)
                    if presorted.get(name) is None:
                        raise NotImplementedError(
                            f'column "{name}" has more than {limit} distinct values: the exact numerical splitter is only '
                            "reproduced for columns that fit one bucket per value, up to max_exact_numerical_values "
                            f"(= {limit}; at most 65535 buckets with the mean of the missing values); raise it, or pass "
                            "discretize_numerical_columns=True for the reference's 255-bin discretisation")
        builder = _capi.DatasetBuilder(n, len(names), device=self.device)
        columns = [None] * len(names)
        pending = []
        try:
            for f, name in enumerate(names):
                v = cols[name]
                if v.dtype.kind in "OUS":
                    c = categorical[name]
                    if c.wide:   # attached after finish(); the byte column is a placeholder
                        builder.add_bins(f, np.zeros(n, np.uint8), 1, 0, _capi.FEATURE_CATEGORICAL)
                    else:
                        builder.add_bins(f, c.encode(v), c.num_bins, c.na_bin, _capi.FEATURE_CATEGORICAL)
                    columns[f] = c
                elif v.dtype.kind not in "fiub":
                    raise NotImplementedError(f'column "{name}" has unsupported dtype {v.dtype}')
                elif name in presorted:   # attached after finish(); the byte column is a placeholder
                    c = presorted[name]
                    builder.add_bins(f, np.zeros(n, np.uint8), 1, 0, _capi.FEATURE_DISCRETIZED_NUMERICAL)
                    columns[f] = c
                elif not self.discretize_numerical_columns:
                    c = lossless[name]
                    if c.wide:   # attached after finish(); the byte column is a placeholder
                        builder.add_bins(f, np.zeros(n, np.uint8), 1, 0, _capi.FEATURE_DISCRETIZED_NUMERICAL)
                    else:
                        builder.add_bins(f, c.encode(v), c.num_bins, c.na_bin, _capi.FEATURE_DISCRETIZED_NUMERICAL)
                    columns[f] = c
                elif self.num_discretized_numerical_bins < 4:
                    # the GPU rule needs >= 4 bins (two are reserved for the special values); host rule below
                    c = ds_lib.infer_column(name, v, self.num_discretized_numerical_bins, 3, self.max_rows_stats)
                    builder.add_bins(f, c.encode(v), c.num_bins, c.na_bin, _capi.FEATURE_DISCRETIZED_NUMERICAL)
                    columns[f] = c
                else:
                    stats = 0 if self.max_rows_stats is None else min(int(self.max_rows_stats), n)
                    # enqueued: the upload of this column overlaps the sort / boundary kernels of the previous ones
                    add = builder.add_numerical_async if self.num_discretized_numerical_bins <= 256 else \
                        builder.add_numerical16_async
                    add(f, np.asarray(v, dtype=np.float32), self.num_discretized_numerical_bins, 3, n_stats_rows=stats)
                    pending.append((f, name))
            for f, name in pending:
                bounds, mean, na_bin, missing = builder.get_numerical(f)
                columns[f] = ds_lib.DiscretizedColumn(
                    name=name, boundaries=bounds, mean=float(mean), num_bins=len(bounds) + 1, na_bin=na_bin,
                    num_missing=int(missing), num_values=n,
                    maximum_num_bins=self.num_discretized_numerical_bins if self.num_discretized_numerical_bins > 256 else None)
            dataset = builder.finish()
            for f, c in enumerate(columns):
                if c.feature_type == _capi.FEATURE_CATEGORICAL and c.wide:
                    dataset.set_wide_categorical_column(f, c.encode16(cols[c.name]), c.num_bins, c.na_bin)
                elif c.feature_type == _capi.FEATURE_NUMERICAL:
                    dataset.set_numerical_column(f, c.encode(cols[c.name]), c.mean)
            for f, c in enumerate(columns):   # exact numerical splitter: thresholds between the values present in a node
                if getattr(c, "bucket_values", None) is None:
                    continue
                if c.wide:
                    dataset.set_wide_column(f, c.encode16(cols[c.name]), c.num_bins, c.na_bin, c.bucket_values, c.mean)
                elif len(c.bucket_values) <= 255 or c.num_missing == 0:
                    # (256 buckets without a missing value: 256 distinct values, which max_exact_numerical_values >= 256
                    # lets through; the byte path carries them with the exact rule.  255 values + the mean keep the
                    # discretized rule, as before.)
                    dataset.set_bucket_values(f, c.bucket_values, c.mean)
        except Exception:
            builder.close()
            raise
        y = cols[self.label]
        spec = ds_lib.DataSpec(columns=columns, label=self.label, task=self.task, num_rows=len(y))
        if self.task == Task.CLASSIFICATION:
            classes = sorted(np.unique(y).tolist())
            if self.loss == "DEFAULT":
                self.loss = "BINOMIAL_LOG_LIKELIHOOD" if len(classes) == 2 else "MULTINOMIAL_LOG_LIKELIHOOD"
            if self.loss == "BINOMIAL_LOG_LIKELIHOOD" and len(classes) != 2:
                dataset.close()
                raise ValueError("Binomial log likelihood loss is only compatible with a BINARY "
                                 f"classification task (got {len(classes)} classes)")
            if self.loss == "MULTINOMIAL_LOG_LIKELIHOOD" and not 2 <= len(classes) <= 32:
                dataset.close()
                raise NotImplementedError(f"the multinomial loss supports 2..32 classes (got {len(classes)})")
            spec.label_classes = classes
            self.cfg.loss = _LOSS_ID[self.loss]
            self.cfg.num_classes = len(classes)
        else:
            yy = np.asarray(y, dtype=np.float64)
            spec.label_mean, spec.label_sd = float(yy.mean()), float(yy.std())
            spec.label_min, spec.label_max = float(yy.min()), float(yy.max())
        return spec, dataset

    def _weights(self, cols):
        """The example weights of `cols` (float32), or None.  Negative / non-finite weights are refused by the engine."""
        if self.weights is None:
            return None
        if self.weights not in cols:
            raise ValueError(f'weight column "{self.weights}" not found')
        w = cols[self.weights]
        if w.dtype.kind not in "fiub":
            raise ValueError(f'weight column "{self.weights}" must be numerical (got {w.dtype})')
        return np.asarray(w, dtype=np.float32)

    def _labels(self, cols, spec):
        y = cols[self.label]
        if self.task == Task.CLASSIFICATION:
            # integerised like the reference: index 0 = out-of-dictionary, 1.. = the classes
            lut = {c: i + 1 for i, c in enumerate(spec.label_classes)}
            values = np.asarray(y).tolist()
            unseen = sorted({str(v) for v in values if v not in lut})
            if unseen:
                raise ValueError(f"label column {self.label!r} holds values that are not classes of the training "
                                 f"dataset: {unseen[:5]} (classes: {list(spec.label_classes)})")
            return np.fromiter((lut[v] for v in values), dtype=np.int32, count=len(y))
        return np.asarray(y, dtype=np.float32)

    # -- training -------------------------------------------------------------------------------
    def train(self, ds, valid=None) -> GradientBoostedTreesModel:
        """Trains on `ds`.  Validation rows come from `valid` if given, else from a random hold-out of
        `validation_ratio` of the rows drawn like the reference does (ExtractValidationDataset,
        gradient_boosted_trees.cc:2718-2746); they drive the validation loss in the logs and early stopping."""
        cols = ds_lib.as_columns(ds)
        spec, full = self._build_dataset(cols)       # dataspec on every row, as the reference infers it
        labels = self._labels(cols, spec)
        weights, valid_weights = None, None
        train_ds, valid_ds, valid_labels = full, None, None
        try:
            weights = self._weights(cols)
            if valid is not None:
                vcols = ds_lib.as_columns(valid)
                vbins = ds_lib.encode_features(vcols, spec.columns)
                valid_ds = ds_lib.device_dataset(vbins, spec.columns, device=self.device)
                valid_labels = self._labels(vcols, spec)
                valid_weights = self._weights(vcols)
            elif self.validation_ratio > 0.0:
                in_training = _capi.validation_split_mask(self.cfg.random_seed, len(labels), self.validation_ratio)
                self.cfg.rng_words_consumed = len(labels)   # the hold-out draw took one engine word per row
                if not in_training.any():
                    raise ValueError("the validation hold-out left no training rows; lower validation_ratio")
                if in_training.all():
                    # the reference only warns and trains without validation (gradient_boosted_trees.cc:1215-1221)
                    warnings.warn("the validation hold-out is empty: training on every row without validation / early stopping")
                else:
                    train_ds, valid_ds = full.split_rows(in_training)
                    full.close()
                    full = None
                    valid_labels, labels = labels[~in_training], labels[in_training]
                    if weights is not None:
                        valid_weights, weights = weights[~in_training], weights[in_training]
            # with candidate sampling the per-node keys order the candidates: no tie-break replay (as best-first growth)
            k = _capi.num_candidate_attributes(train_ds.n_features, self.cfg.loss, self.num_candidate_attributes,
                                               self.num_candidate_attributes_ratio)
            self.cfg.candidate_shuffle = 0 if k < train_ds.n_features else self._candidate_shuffle
            gbt = _capi.Gbt(train_ds, self.cfg)
            try:
                if k < train_ds.n_features:
                    gbt.set_candidate_sampling(self.num_candidate_attributes, self.num_candidate_attributes_ratio)
                if self.forest_extraction == "DART":
                    gbt.set_dart(self.dart_dropout)
                if weights is not None:
                    gbt.set_weights(weights)     # before the labels: the initial predictions are weighted
                gbt.set_labels(labels)
                if valid_ds is not None:
                    gbt.set_validation(valid_ds, valid_labels, weights=valid_weights)
                gbt.train(self.cfg.num_trees)
                trees = [gbt.get_tree(i) for i in range(gbt.num_trees())]
                if self.forest_extraction == "DART":
                    # ScaleRegressorOutput: every leaf of iteration j times w_j, in float (the engine's saved model)
                    w = gbt.dart_weights()
                    K = self.cfg.num_classes if self.cfg.loss == _LOSS_ID["MULTINOMIAL_LOG_LIKELIHOOD"] else 1
                    for i, t in enumerate(trees):
                        leaf = t["feature"] < 0
                        t["leaf_value"][leaf] = (t["leaf_value"][leaf].astype(np.float32) * np.float32(w[i // K])).astype(np.float32)
                category_sets = [gbt.get_category_sets(i, t) for i, t in enumerate(trees)]
                logs = []
                for i in range(gbt.num_iterations()):
                    l, s = gbt.train_loss(i)
                    e = {"number_of_trees": i + 1, "loss": l, "secondary": s}
                    if valid_ds is not None:
                        e["validation_loss"], e["validation_secondary"] = gbt.validation_loss(i)
                    logs.append(e)
                init = gbt.initial_prediction()
                final = gbt.final_validation() if valid_ds is not None else (None, False)
            finally:
                gbt.close()
        finally:
            for d in (train_ds, valid_ds, full):
                if d is not None:
                    d.close()
        config = {k: getattr(self.cfg, k) for k, _ in self.cfg._fields_}
        config["num_candidate_attributes"] = self.num_candidate_attributes
        config["num_candidate_attributes_ratio"] = self.num_candidate_attributes_ratio
        config["forest_extraction"] = self.forest_extraction
        config["dart_dropout"] = self.dart_dropout if self.forest_extraction == "DART" else None
        model = GradientBoostedTreesModel(spec, trees, init, self.loss, logs, config=config, category_sets=category_sets)
        model.validation_loss, model.early_stopping_triggered = final
        return model
