"""Times the discretized wide columns (DESIGN.md §25) on the C3 shape of bench.py: 10M rows x 200 float columns (20
informative), depth 8, variance gain, binomial loss.

1. GPU binning per column (ygg_dataset_builder_add_numerical16_async then _get_numerical, one column at a time, so the
   time is one column's upload + sort + boundary walk + encode) at 256 (the byte path), 1024 and 65535 bins.
2. Training iterations/s with every column binned on the GPU at 256 bins (byte columns, bench.py's setting) and at
   1024 bins (200 discretized wide columns), plus the per-level device time of hist / hist_wide / scan / scan_wide.

Prints one JSON line per measurement and the GPU's name, SM clock limit and power limit.
Usage: python tools/bench_discretized_wide.py [--rows N] [--features F] [--steps K] [--warmup W]."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ydf_b200  # noqa: E402


def column(seed, f, n):
    return np.random.default_rng([seed, f]).standard_normal(n, dtype=np.float32)


def labels(seed, n, informative):
    logit = np.zeros(n, np.float32)
    for f in range(informative):
        logit += np.sin(1.5 * column(seed, f, n)) * (1.0 if f % 2 else -0.7)
    rng = np.random.default_rng(seed + 1)
    return (rng.random(n, dtype=np.float32) < 1 / (1 + np.exp(-logit / 3))).astype(np.int32) + 1


def time_binning(n, bins, reps=7):
    b = ydf_b200.DatasetBuilder(n, 1)
    x = column(7, 0, n)
    add = b.add_numerical_async if bins <= 256 else b.add_numerical16_async
    for _ in range(3):           # warm-up: every lane's buffers (three lanes in turn), module load
        add(0, x, bins, 3)
        b.get_numerical(0)
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        add(0, x, bins, 3)
        bounds, _, _, _ = b.get_numerical(0)   # waits for the column's kernels
        ms.append((time.perf_counter() - t0) * 1e3)
    b.close()
    return {"bench": "binning", "rows": n, "max_bins": bins, "bins_made": len(bounds) + 1,
            "ms_per_column_median": round(float(np.median(ms)), 2), "ms_per_column_min": round(min(ms), 2),
            "ms_per_column_max": round(max(ms), 2), "ms_per_column": [round(m, 2) for m in ms]}


def train(n, F, bins, y, steps, warmup, seed):
    b = ydf_b200.DatasetBuilder(n, F)
    t0 = time.perf_counter()
    for f in range(F):
        add = b.add_numerical_async if bins <= 256 else b.add_numerical16_async
        add(f, column(seed, f, n), bins, 3)
        b.get_numerical(f)
    ds = b.finish()
    build_s = time.perf_counter() - t0
    cfg = ydf_b200.default_config(max_depth=8, num_trees=warmup + 2 * steps + 1)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(y)
    gbt.train(warmup)
    ms, _ = gbt.train_timed(steps)
    out = {"bench": "train", "max_bins": bins, "wide_columns": len(getattr(ds, "wide", {})),
           "iters_per_s": round(1000.0 * steps / ms, 3), "ms_per_iter": round(ms / steps, 3),
           "dataset_build_s": round(build_s, 2)}
    gbt.set_profiling(True)
    gbt.train_timed(steps)
    for name in ("hist", "scan", "hist_wide", "scan_wide"):
        try:
            t, launches = gbt.get_profile(name)
        except ydf_b200.YggError:
            continue
        if launches:
            out[f"{name}_ms_per_level"] = round(t / (steps * 7), 4)
    gbt.close()
    ds.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=200)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if ydf_b200.device_count() == 0:
        raise SystemExit("no CUDA device: nothing to measure")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    ydf_b200.lib()
    for bins in (256, 1024, 65535):
        print(json.dumps(time_binning(a.rows, bins)), flush=True)
    y = labels(11, a.rows, 20)
    for bins in (256, 1024):
        print(json.dumps(train(a.rows, a.features, bins, y, a.steps, a.warmup, 11)), flush=True)


if __name__ == "__main__":
    main()
