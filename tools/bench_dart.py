"""DART's per-iteration cost at the C3 shape (10M rows x 200 byte features, depth 8, binomial): ms per iteration of MART and
of DART at dropout rates 0.01 and 0.1, timed around iteration `--at` (default 100).

All arms live in one process and are timed in alternating rounds (device events around `--steps` iterations of each);
the card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/bench_dart.py [--rows N] [--features F] [--at 100] [--steps 10] [--rounds 3]
"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=200)
    ap.add_argument("--depth", type=int, default=8)
    ap.add_argument("--at", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if ydf_b200.device_count() < 1:
        raise SystemExit("no GPU: this benchmark measures the device")
    rng = np.random.default_rng(0)
    n, F = args.rows, args.features
    bins = rng.integers(0, 256, size=(F, n), dtype=np.uint8)
    m = np.zeros(n, np.float32)
    for f in range(20):
        m += (bins[f].astype(np.float32) - 127.5) * np.float32(rng.normal())
    y = np.where(m + rng.normal(scale=float(m.std()), size=n).astype(np.float32) > 0, 2, 1).astype(np.int32)
    ds = ydf_b200.Dataset(bins, np.full(F, 256, np.int32), np.zeros(F, np.int32))
    del bins
    capacity = args.at + args.rounds * args.steps + 1
    arms = {}
    for name, rate in (("mart", None), ("dart_0.01", 0.01), ("dart_0.1", 0.1)):
        cfg = ydf_b200.default_config(loss=0, max_depth=args.depth, num_trees=capacity)
        g = ydf_b200.Gbt(ds, cfg)
        if rate is not None:
            g.set_dart(rate)
        g.set_labels(y)
        g.train_timed(args.at)          # up to the measured iteration (warms every shape)
        arms[name] = g
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name, g in arms.items():
            ms, _ = g.train_timed(args.steps)
            times[name].append(ms / args.steps)
    dropped = {k: float(np.mean([len(g.dart_dropped(i)) for i in range(args.at, args.at + args.rounds * args.steps)]))
               for k, g in arms.items() if k != "mart"}
    res = {"metric": "ms per boosting iteration", "rows": n, "features": F, "depth": args.depth, "at_iteration": args.at,
           "card": card(), "ms_per_iter": {k: float(np.median(v)) for k, v in times.items()},
           "ms_per_iter_rounds": times, "mean_dropped": dropped}
    print(json.dumps(res))
    for g in arms.values():
        g.close()
    ds.close()


if __name__ == "__main__":
    main()
