"""Builds tests/golden/dart_cxx_test_folds.npz: the folds of the reference's two DART acceptance tests
(`GradientBoostedTreesOnIris.Dart` and `GradientBoostedTreesOnAdult.Dart`, learner/gradient_boosted_trees/
gradient_boosted_trees_test.cc:1774-1784 and :1458-1473), drawn like utils::TrainAndTestTester (utils/test_utils.cc:505-600):
`dataset_sampling_` (1.0 for both), then a 50 % split, each by DeterministicBinomial (:100-127).

Stored, per dataset and fold: numerical columns as raw float32 values (NaN = missing), categorical columns as C++ dictionary
codes (index into `<dataset>_vocabulary_<column>`, most frequent first; 0 = out of dictionary, missing = ""), labels as class
strings.  Run where the reference's test data are mounted at /root/reference."""
import csv
import os
from collections import Counter

import numpy as np

DATA = "/root/reference/yggdrasil_decision_forests/test_data/dataset"


class DeterministicBinomial:
    def __init__(self, rate):
        self.rate, self.pos, self.total = np.float32(rate), 0, 0

    def sample(self):
        if self.total == 0:
            self.total += 1
            if self.rate == 1:
                self.pos += 1
                return True
            return False
        if self.pos > float(self.rate * np.float32(self.total)):
            self.total += 1
            return False
        self.pos += 1
        self.total += 1
        return True


def tester_folds(n_rows, dataset_sampling):
    sampling, split = DeterministicBinomial(dataset_sampling), DeterministicBinomial(0.5)
    train, test = [], []
    for i in range(n_rows):
        if sampling.sample():
            (train if split.sample() else test).append(i)
    return np.array(train, np.int32), np.array(test, np.int32)


def cxx_vocabulary(values):
    """The C++ dictionary rule: <OOD> first, then by decreasing count, ties by value (descending, as the reference
    sorts (count, value) pairs)."""
    count = Counter(v for v in values if v != "")
    return ["<OOD>"] + sorted(count, key=lambda k: (count[k], k), reverse=True)


def build(name, csv_name, label, numerical, dataset_sampling, out):
    rows = list(csv.DictReader(open(os.path.join(DATA, csv_name))))
    names = list(rows[0].keys())
    train, test = tester_folds(len(rows), dataset_sampling)
    out[f"{name}_features"] = np.array([c for c in names if c != label])
    out[f"{name}_numerical"] = np.array([c for c in names if c in numerical])
    for c in names:
        raw = [r[c] for r in rows]
        if c == label:
            for fold, idx in (("train", train), ("test", test)):
                out[f"{name}_{fold}_{c}"] = np.array([raw[i] for i in idx])
        elif c in numerical:
            v = np.array([float(x) if x != "" else np.nan for x in raw], np.float32)
            for fold, idx in (("train", train), ("test", test)):
                out[f"{name}_{fold}_{c}"] = v[idx]
        else:
            voc = cxx_vocabulary(raw)
            index = {k: j for j, k in enumerate(voc)}
            codes = np.array([index.get(x, 0) if x != "" else 0xFFFF for x in raw], np.uint16)
            out[f"{name}_vocabulary_{c}"] = np.array(voc)
            for fold, idx in (("train", train), ("test", test)):
                out[f"{name}_{fold}_{c}"] = codes[idx]
    print(name, len(train), len(test))


out = {}
build("iris", "iris.csv", "class", ["Sepal.Length", "Sepal.Width", "Petal.Length", "Petal.Width"], 1.0, out)
build("adult", "adult.csv", "income", ["age", "fnlwgt", "education_num", "capital_gain", "capital_loss", "hours_per_week"],
      1.0, out)
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dart_cxx_test_folds.npz")
np.savez_compressed(OUT, **out)
print(OUT, os.path.getsize(OUT))
