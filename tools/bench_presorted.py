"""Times the presorted numerical columns (DESIGN.md §22): 10M rows x (190 byte columns + 10 presorted columns of ~10M
distinct values), depth 8, variance gain, binomial loss; then the 10 columns of bench_wide.py's table at 16611 and 65535
values, once as wide columns and once presorted.  Prints one JSON line per table, with the card and its power limit:
iterations/s, and the per-level device time of the presort scan / partition and of the wide histogram / scan (CUDA
events, ygg_gbt_set_profiling).  Usage: python tools/bench_presorted.py [--rows N] [--steps K] [--warmup W]."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ydf_b200  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run(narrow, extra, kind, B, y, steps, warmup, depth):
    """kind: 'wide' (extra = uint16 codes of B buckets) or 'presorted' (extra = float values)."""
    F = narrow.shape[0] + len(extra)
    bins = np.concatenate([narrow, np.zeros((len(extra), narrow.shape[1]), np.uint8)])
    ds = ydf_b200.Dataset(bins, np.full(F, 256, np.int32), np.zeros(F, np.int32))
    for w, col in enumerate(extra):
        f = narrow.shape[0] + w
        if kind == "wide":
            ds.set_wide_column(f, col, B, B // 2, np.arange(B, dtype=np.float32), float(B // 2))
        else:
            ds.set_numerical_column(f, col, float(np.float32(col.mean(dtype=np.float64))))
    cfg = ydf_b200.default_config(max_depth=depth, num_trees=warmup + steps + 1)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(y)
    gbt.train(warmup)
    gbt.set_profiling(True)
    ms, _ = gbt.train_timed(steps)
    out = {"iters_per_s": round(1000.0 * steps / ms, 3), "ms_per_iter": round(ms / steps, 3)}
    levels = depth - 1
    for name in ("hist", "scan", "partition", "hist_wide", "scan_wide", "presort_scan", "presort_partition"):
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
    n, n_narrow, n_extra = a.rows, 190, 10
    narrow = rng.integers(0, 256, size=(n_narrow, n), dtype=np.uint8)
    u = rng.random((n_extra, n), dtype=np.float32)
    logit = (narrow[:4].astype(np.float32).sum(0) / 512.0 - 2.0) + 2 * (u[0] - 0.5) + np.sin(8 * u[1])
    y = (rng.random(n, dtype=np.float32) < 1 / (1 + np.exp(-logit))).astype(np.int32) + 1
    ydf_b200.lib()   # (builds / loads the library before anything is timed)
    gpu = card()
    cont = [u[w] * np.float32(1000.0) for w in range(n_extra)]
    distinct = len(np.unique(cont[0]))
    print(json.dumps({"gpu": gpu, "table": "presorted_continuous", "columns": n_extra, "distinct_values": distinct,
                      **run(narrow, cont, "presorted", 0, y, a.steps, a.warmup, a.depth)}), flush=True)
    for B in (16611, 65535):
        codes = [np.minimum((u[w] * B).astype(np.uint16), B - 1) for w in range(n_extra)]
        print(json.dumps({"gpu": gpu, "table": f"wide_{B}", "columns": n_extra,
                          **run(narrow, codes, "wide", B, y, a.steps, a.warmup, a.depth)}), flush=True)
        vals = [c.astype(np.float32) for c in codes]   # the same values, presorted
        print(json.dumps({"gpu": gpu, "table": f"presorted_{B}", "columns": n_extra,
                          **run(narrow, vals, "presorted", B, y, a.steps, a.warmup, a.depth)}), flush=True)


if __name__ == "__main__":
    main()
