"""Times the wide-column path (DESIGN.md §20): 10M rows x (190 byte columns + 10 wide columns), depth 8, variance gain,
binomial loss, for wide columns of 65535 and 16611 buckets, against the same table with those 10 columns quantised to
256 bins.  Prints one JSON line per table: iterations/s and the per-level device time of k_hist_wide and k_scan_wide
(CUDA events, ygg_gbt_set_profiling).  Usage: python tools/bench_wide.py [--rows N] [--steps K] [--warmup W]."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ydf_b200  # noqa: E402


def run(bins, wide_codes, wide_bins, y, steps, warmup, depth):
    F = bins.shape[0]
    nb = np.full(F, 256, np.int32)
    ds = ydf_b200.Dataset(bins, nb, np.zeros(F, np.int32))
    for w, codes in enumerate(wide_codes):
        f = F - len(wide_codes) + w
        ds.set_wide_column(f, codes, wide_bins, wide_bins // 2, np.arange(wide_bins, dtype=np.float32), float(wide_bins // 2))
    cfg = ydf_b200.default_config(max_depth=depth, num_trees=warmup + steps + 1)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(y)
    gbt.train(warmup)
    gbt.set_profiling(True)
    ms, _ = gbt.train_timed(steps)
    out = {"iters_per_s": round(1000.0 * steps / ms, 3), "ms_per_iter": round(ms / steps, 3)}
    levels = depth - 1
    for name in ("hist", "scan", "hist_wide", "scan_wide"):
        try:
            t, launches = gbt.get_profile(name)
        except ydf_b200.YggError:
            continue
        if launches:
            out[f"{name}_ms_per_level"] = round(t / (steps * levels), 4)
    gbt.close()
    ds.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--depth", type=int, default=8)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    n, n_narrow, n_wide = a.rows, 190, 10
    narrow = rng.integers(0, 256, size=(n_narrow, n), dtype=np.uint8)
    u = rng.random((n_wide, n), dtype=np.float32)
    logit = (narrow[:4].astype(np.float32).sum(0) / 512.0 - 2.0) + 2 * (u[0] - 0.5) + np.sin(8 * u[1])
    y = (rng.random(n, dtype=np.float32) < 1 / (1 + np.exp(-logit))).astype(np.int32) + 1
    base = np.concatenate([narrow, (u * 256).astype(np.uint8)])
    ydf_b200.lib()   # (builds / loads the library before anything is timed)
    print(json.dumps({"table": "quantised_256", "wide_columns": 0, **run(base, [], 0, y, a.steps, a.warmup, a.depth)}), flush=True)
    for B in (65535, 16611):
        codes = [np.minimum((u[w] * B).astype(np.uint16), B - 1) for w in range(n_wide)]
        bins = np.concatenate([narrow, np.zeros((n_wide, n), np.uint8)])
        print(json.dumps({"table": f"wide_{B}", "wide_columns": n_wide, **run(bins, codes, B, y, a.steps, a.warmup, a.depth)}),
              flush=True)


if __name__ == "__main__":
    main()
