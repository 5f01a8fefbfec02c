"""GradientBoostedTreesModel — the trained forest as returned by the learner.

Holds the trees in the engine's flat pre-order layout (ygg_node) plus the dataspec.  Inference
here is a plain numpy traversal for evaluation in tests; fast inference engines are out of scope
(SURVEY.md §2: serving/).
"""
import math
import os
from typing import List

import numpy as np

from . import dataspec as ds_lib


class GradientBoostedTreesModel:
    def __init__(self, spec: ds_lib.DataSpec, trees: List[np.ndarray], initial_prediction: float,
                 loss: str, training_logs=None, config=None, category_sets=None):
        self.data_spec = spec
        self.trees = trees
        # per tree {pre-order node index: uint32 words}: the positive sets of the splits on wide categorical columns
        # (more than 256 categories), whose cat_mask is empty
        self.category_sets = category_sets or [{} for _ in trees]
        self.initial_prediction = float(initial_prediction)
        self.loss = loss
        self.training_logs = training_logs or []
        self.config = config or {}
        self.validation_loss = None            # Header.validation_loss (validation rows only)
        self.early_stopping_triggered = False  # Header.early_stopping_triggered

    def num_trees(self) -> int:
        return len(self.trees)

    def num_trees_per_iter(self) -> int:
        return len(self.data_spec.label_classes) if self.loss == "MULTINOMIAL_LOG_LIKELIHOOD" else 1

    def num_nodes(self) -> int:
        return int(sum(len(t) for t in self.trees))

    def task(self) -> str:
        return self.data_spec.task

    def label_classes(self):
        """Class names in dictionary order, as strings (PYDF: model.label_classes())."""
        return [str(c) for c in (self.data_spec.label_classes or [])]

    def _raw(self, bins: np.ndarray) -> np.ndarray:
        """Sum of the leaves: [n], or [n, K] for the multinomial loss (tree i belongs to class i % K)."""
        n = bins.shape[1]
        k = self.num_trees_per_iter()
        acc = np.full((n, k), self.initial_prediction, dtype=np.float32)
        rows = np.arange(n)
        for ti, t in enumerate(self.trees):
            # the positive set of every node, words [nodes, width]: cat_mask, or the node's set from category_sets
            sets = self.category_sets[ti]
            width = max([8] + [len(w) for w in sets.values()])
            words = np.zeros((len(t), width), np.uint32)
            words[:, :8] = t["cat_mask"]
            for node_i, w in sets.items():
                words[node_i, :len(w)] = w
            node = np.zeros(n, dtype=np.int64)
            active = t["feature"][node] >= 0
            while active.any():
                idx = rows[active]
                nd = node[idx]
                f = t["feature"][nd]
                raw = bins[f, idx]
                # presorted numerical splits: value >= threshold_value on the raw float, a missing value -> na_value
                num = t["condition_type"][nd] == 2
                b = (np.nan_to_num(raw) if raw.dtype.kind == "f" else raw).astype(np.int64)
                cat = t["condition_type"][nd] == 1   # (a categorical code is below its column's num_bins <= 32 x width)
                go_pos = b >= t["threshold_bin"][nd]
                go_pos[cat] = ((words[nd[cat], b[cat] >> 5] >> (b[cat] & 31).astype(np.uint32)) & 1) != 0
                if num.any():
                    v = raw[num]
                    go_pos[num] = np.where(np.isnan(v), t["na_value"][nd[num]] != 0, v >= t["threshold_value"][nd[num]])
                node[idx] = np.where(go_pos, t["pos_child"][nd], t["neg_child"][nd])
                active = t["feature"][node] >= 0
            acc[:, ti % k] += t["leaf_value"][node]
        return acc[:, 0] if k == 1 else acc

    def predict(self, ds) -> np.ndarray:
        cols = ds_lib.as_columns(ds)
        bins = ds_lib.encode_features(cols, self.data_spec.columns)
        raw = self._raw(bins)
        if self.loss == "BINOMIAL_LOG_LIKELIHOOD":
            return (1.0 / (1.0 + np.exp(-raw.astype(np.float64)))).astype(np.float32)
        if self.loss == "MULTINOMIAL_LOG_LIKELIHOOD":   # softmax over the class scores: [n, K]
            e = np.exp(raw.astype(np.float64) - raw.max(axis=1, keepdims=True))
            return (e / e.sum(axis=1, keepdims=True)).astype(np.float32)
        return raw

    def evaluate(self, ds) -> dict:
        cols = ds_lib.as_columns(ds)
        y = cols[self.data_spec.label]
        p = self.predict(ds)
        if self.loss == "MULTINOMIAL_LOG_LIKELIHOOD":
            classes = list(self.data_spec.label_classes)
            yy = np.array([classes.index(v) for v in np.asarray(y).tolist()])
            ll = -np.mean(np.log(np.maximum(p[np.arange(len(yy)), yy], 1e-12)))
            return {"accuracy": float(np.mean(p.argmax(axis=1) == yy)), "loss": float(ll), "num_examples": int(len(yy))}
        if self.loss == "BINOMIAL_LOG_LIKELIHOOD":
            classes = self.data_spec.label_classes
            yy = (np.asarray(y) == classes[1]).astype(np.float64)
            eps = 1e-12
            ll = -np.mean(yy * np.log(np.maximum(p, eps)) + (1 - yy) * np.log(np.maximum(1 - p, eps)))
            return {"accuracy": float(np.mean((p > 0.5) == (yy > 0.5))), "loss": float(ll),
                    "num_examples": int(len(yy))}
        err = np.asarray(y, dtype=np.float64) - p
        return {"rmse": float(math.sqrt(np.mean(err * err))), "num_examples": int(len(err))}

    def save(self, path: str):
        from . import model_io
        model_io.save_ydf_model(self, path)

    def describe(self) -> str:
        lines = [f"GRADIENT_BOOSTED_TREES (ygg_b200) task={self.task()} loss={self.loss}",
                 f"trees={self.num_trees()} nodes={self.num_nodes()} "
                 f"initial_prediction={self.initial_prediction:.6g}"]
        if self.training_logs:
            last = self.training_logs[-1]
            lines.append(f"final train loss={last['loss']:.6g} secondary={last['secondary']:.6g}")
        return "\n".join(lines)
