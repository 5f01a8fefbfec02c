"""Times candidate feature sampling (DESIGN.md §23) on bench.py's C3 workload (10M rows x 200 features, depth 8, binomial
loss): alternating rounds of the unsampled training, num_candidate_attributes_ratio = 0.5 and k = ceil(sqrt(F)).  Prints
one JSON line per run with the card and its power limit: iterations/s and the per-level device time of the "select" phase
(k_node_stats + k_select_local or k_select_sampled + k_select_global; CUDA events, ygg_gbt_set_profiling).
Usage: python tools/bench_candidate_sampling.py [--rows N] [--steps K] [--warmup W] [--rounds R]."""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import ydf_b200  # noqa: E402
from tools.bench_presorted import card  # noqa: E402


def run(dataset, w, sampling, steps, warmup):
    gbt = ydf_b200.Gbt(dataset, bench.gbt_config(w, warmup + steps + 1))
    gbt.set_labels(w["labels"])
    if sampling is not None:
        gbt.set_candidate_sampling(*sampling)
    gbt.train(warmup)
    gbt.set_profiling(True)
    ms, _ = gbt.train_timed(steps)
    t, _ = gbt.get_profile("select")
    trees = [gbt.get_tree(i).tobytes() for i in range(warmup, warmup + 2)]
    gbt.close()
    return {"iters_per_s": round(1000.0 * steps / ms, 3), "ms_per_iter": round(ms / steps, 3),
            "select_ms_per_level": round(t / (steps * (w["max_depth"] - 1)), 4)}, trees


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=None)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    w = dict(bench.WORKLOADS["c3"])
    if a.rows:
        w["rows"] = a.rows
    bins, nb, na, labels = bench.make_data(w, 0)
    w["labels"] = labels
    dataset = ydf_b200.Dataset(bins, nb, na, feature_types=w.get("feature_types"))
    F = w["features"]
    arms = {"unsampled": None, "ratio_0.5": (-1, 0.5), f"k_{math.ceil(math.sqrt(F))}": (math.ceil(math.sqrt(F)), None)}
    gpu = card()
    first_trees = {}
    for r in range(a.rounds):
        for name, sampling in arms.items():
            out, trees = run(dataset, w, sampling, a.steps, a.warmup)
            first_trees.setdefault(name, trees)
            assert first_trees[name] == trees, f"{name}: trees differ between rounds"
            print(json.dumps({"gpu": gpu, "workload": f"c3 {w['rows']}x{F} depth {w['max_depth']}", "arm": name,
                              "round": r, **out}), flush=True)
    dataset.close()


if __name__ == "__main__":
    main()
