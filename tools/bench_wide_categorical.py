"""Times the wide categorical path (DESIGN.md §21) at BASELINE config 5's shape: 10M rows x (100 numerical columns of 256
bins + 50 categorical columns with cardinalities log-uniform in [100, 2000], Zipf(1.2) frequencies, 5% missing),
regression, depth 8.  Columns above 256 categories are wide categorical columns (the learner's
categorical_arity_limit_for_random raised).  Prints one JSON line with the card, iterations/s and the per-level device
time of k_hist_wide and k_scan_wide_cat (CUDA events, ygg_gbt_set_profiling).
Usage: python tools/bench_wide_categorical.py [--rows N] [--steps K] [--warmup W]."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ydf_b200  # noqa: E402


def zipf(rng, n, k, missing=0.05):
    p = np.arange(1, k, dtype=np.float64) ** -1.2
    codes = (rng.choice(k - 1, size=n, p=p / p.sum()) + 1).astype(np.uint16)
    codes[rng.random(n) < missing] = 1   # missing values folded into the most frequent category
    return codes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--depth", type=int, default=8)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    n, n_num, n_cat = a.rows, 100, 50
    card = np.exp(rng.uniform(np.log(100), np.log(2000), size=n_cat)).astype(int)
    F = n_num + n_cat
    bins = np.zeros((F, n), np.uint8)
    bins[:n_num] = rng.integers(0, 256, size=(n_num, n), dtype=np.uint8)
    y = bins[:4].astype(np.float32).sum(0) / 256.0
    codes = []
    for j, k in enumerate(card):
        c = zipf(rng, n, int(k))
        y += rng.normal(size=int(k)).astype(np.float32)[c]
        codes.append(c)
        if k <= 256:
            bins[n_num + j] = c
    y = (y + rng.normal(size=n).astype(np.float32)).astype(np.float32)
    nb = [256] * n_num + [int(k) if k <= 256 else 1 for k in card]
    na = [0] * n_num + [1 if k <= 256 else 0 for k in card]
    ds = ydf_b200.Dataset(bins, nb, na, feature_types=[0] * n_num + [1] * n_cat)
    for j, k in enumerate(card):
        if k > 256:
            ds.set_wide_categorical_column(n_num + j, codes[j], int(k), 1)
    cfg = ydf_b200.default_config(loss=1, max_depth=a.depth, num_trees=a.warmup + a.steps + 1)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(y)
    gbt.train(a.warmup)
    gbt.set_profiling(True)
    ms, _ = gbt.train_timed(a.steps)
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, check=False).stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        gpu = "unknown"
    out = {"gpu": gpu, "rows": n, "wide_categorical_columns": int((card > 256).sum()),
           "iters_per_s": round(1000.0 * a.steps / ms, 3), "ms_per_iter": round(ms / a.steps, 3)}
    for name in ("hist", "scan", "hist_wide", "scan_wide_cat", "select", "partition"):
        try:
            t, launches = gbt.get_profile(name)
        except ydf_b200.YggError:
            continue
        if launches:
            out[f"{name}_ms_per_level"] = round(t / (a.steps * (a.depth - 1)), 4)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
