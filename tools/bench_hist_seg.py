"""k_hist_seg's flush cost per work item at the C3 shape (10M rows x 200 byte features, depth 8, binomial).

Every variant is a build of the library whose only difference is kSegItemsPerCta (work items per CTA: the piece size P
follows from it).  More items per CTA cost more flushes and nothing else of the gather and atomic work, so per level the
slope of the time against the level's item count is what one item's flush costs, and slope x items is the flush's share
of the level.  Each variant runs in its own process (YGG_B200_LIB) on the same data:
  - `hist_L{l}` of the engine's own profile (device events around each level's histogram launches, ms per iteration);
  - in a separate torch.profiler run, per level, the kernel times of k_seg_count, cub's scan, k_seg_ranges,
    k_seg_scatter and k_hist_seg.
The item count of a level is the planned one, n_fg feature groups x ceil(items x grid / n_fg) pieces; the partial last
piece of each (slot, chunk) range adds about one piece per non-empty range, the same in every variant, so it does not
move the slope.  The card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/bench_hist_seg.py [--items 2,4,8] [--lib LABEL:ITEMS:PATH ...] [--build-dir DIR] [--build-only]

--items builds the tree's sources once per value into --build-dir (default: a temporary directory; a library already
there is reused); --lib adds prebuilt libraries (e.g. of another revision), labelled, with the items they were built
with.  Variants with the same label are fitted together.
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PKG = os.path.join(ROOT, "yggdrasil-decision-forests_b200")
SEG_KERNELS = ("k_seg_count", "scan", "k_seg_ranges", "k_seg_scatter", "k_hist_seg")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def build_variant(items, out_dir):
    """The tree's library with kSegItemsPerCta = items, built from a copy of its sources under out_dir."""
    sys.path.insert(0, PKG)
    import _build
    lib = os.path.join(out_dir, f"items{items}", "libygg_b200.so")
    if os.path.exists(lib):
        return lib
    src = os.path.join(out_dir, f"items{items}", "src")
    shutil.rmtree(src, ignore_errors=True)
    shutil.copytree(os.path.join(PKG, "csrc"), os.path.join(src, "pkg", "csrc"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(src, "include"))
    hdr = os.path.join(src, "pkg", "csrc", "ygg_hist_seg.cuh")
    text = open(hdr).read()
    text, n = re.subn(r"constexpr int kSegItemsPerCta = \d+;", f"constexpr int kSegItemsPerCta = {items};", text)
    if n != 1:
        raise SystemExit("kSegItemsPerCta not found in ygg_hist_seg.cuh")
    open(hdr, "w").write(text)
    srcs = [os.path.join(src, "pkg", "csrc", s) for s in _build.SOURCES]
    tmp = lib + ".tmp"
    subprocess.check_call([_build._nvcc()] + _build.NVCC_FLAGS + ["-o", tmp] + srcs)
    os.replace(tmp, lib)
    shutil.rmtree(src)
    return lib


def levels_of(gbt, depth):
    """Levels whose histograms k_hist_seg takes, with their planned item counts per kSegItemsPerCta."""
    from ydf_b200 import _capi
    F = gbt.hist_features()[1] - gbt.hist_features()[0]
    out = {}
    for l in range(depth - 1):
        p = gbt.hist_plan(l)
        if p.mode != _capi.HIST_SEGMENTED:
            continue
        fpl = 2 if p.group == 32 and F > 32 else 1
        n_fg = -(-F // (p.group * fpl))
        out[l] = {"grid": p.grid, "lanes": p.group, "feature_groups": n_fg}
    return out


def child(args):
    """One variant: the library is the one YGG_B200_LIB names."""
    import torch
    import bench
    import ydf_b200
    w = dict(bench.WORKLOADS["c3"])
    if args.rows:
        w["rows"] = args.rows
    if args.features:
        w["features"] = args.features
    bins, nb, na, labels = bench.make_data(w, 0)
    K, W = args.steps, args.warmup
    ds = ydf_b200.Dataset(bins, nb, na, device=0)
    gbt = ydf_b200.Gbt(ds, bench.gbt_config(w, W + 3 * K + 1))
    gbt.set_labels(labels)
    depth = w["max_depth"]
    gbt.train_timed(W)
    ms, _ = gbt.train_timed(K)
    gbt.set_profiling(True)
    gbt.train_timed(K)
    prof = {l: gbt.get_profile(f"hist_L{l}")[0] / K for l in range(depth - 1)}
    gbt.set_profiling(False)
    levels = levels_of(gbt, depth)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as pr:
        gbt.train_timed(K)
        torch.cuda.synchronize()
    # the level of a k_seg_count .. k_hist_seg run is its place among the iteration's k_hist_seg launches
    evs = sorted((e for e in pr.events() if e.device_type == torch.autograd.DeviceType.CUDA
                  and not e.name.startswith("Memcpy") and not e.name.startswith("Memset")),
                 key=lambda e: e.time_range.start)
    seg_levels = sorted(levels)
    per = {l: {k: 0.0 for k in SEG_KERNELS} for l in seg_levels}
    group, n_seg = None, 0
    for e in evs:
        name = e.name
        if "k_seg_count" in name:
            group = {k: 0.0 for k in SEG_KERNELS}
        if group is None:
            continue
        us = e.time_range.elapsed_us()
        for k in SEG_KERNELS:
            if (k in name) if k != "scan" else ("DeviceScan" in name):
                group[k] += us
        if "k_hist_seg" in name:
            l = seg_levels[n_seg % len(seg_levels)]
            for k in SEG_KERNELS:
                per[l][k] += group[k] / 1000.0 / K
            n_seg += 1
            group = None
    if n_seg != K * len(seg_levels):
        raise SystemExit(f"profile: {n_seg} k_hist_seg launches for {K} iterations x {len(seg_levels)} levels")
    for l in seg_levels:
        t = -(-args.items_per_cta * levels[l]["grid"] // levels[l]["feature_groups"])
        levels[l]["items"] = levels[l]["feature_groups"] * max(1, t)
        levels[l]["hist_ms"] = prof[l]
        levels[l]["kernel_ms"] = per[l]
    res = {"ms_per_iter": ms / K, "iters_per_s": K / (ms / 1000.0), "card": card(),
           "hist_ms": {f"L{l}": prof[l] for l in range(depth - 1)}, "seg_levels": {f"L{l}": v for l, v in levels.items()}}
    print("RESULT " + json.dumps(res))
    gbt.close()
    ds.close()


def fit(runs):
    """Per level, least squares of hist_L and k_hist_seg time against the item count over the runs of one label."""
    out = {}
    levels = sorted(runs[0]["seg_levels"], key=lambda s: int(s[1:]))
    for lv in levels:
        x = np.array([r["seg_levels"][lv]["items"] for r in runs], float)
        row = {"items": [int(v) for v in x]}
        for key, get in (("hist_ms", lambda r: r["seg_levels"][lv]["hist_ms"]),
                         ("k_hist_seg_ms", lambda r: r["seg_levels"][lv]["kernel_ms"]["k_hist_seg"])):
            y = np.array([get(r) for r in runs], float)
            row[key] = [round(v, 4) for v in y]
            if len(set(x)) > 1:
                slope, icpt = np.polyfit(x, y, 1)
                row[key + "_per_item_us"] = round(slope * 1000.0, 4)
        out[lv] = row
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", default="2,4,8", help="kSegItemsPerCta values to build from the tree ('' for none)")
    ap.add_argument("--lib", action="append", default=[], metavar="LABEL:ITEMS:PATH")
    ap.add_argument("--build-dir", default=None)
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--shipped", type=int, default=None, help="items per CTA of the shipped build (flush share)")
    ap.add_argument("--rows", type=int, default=None)
    ap.add_argument("--features", type=int, default=None)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--items-per-cta", type=int, default=4, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)

    build_dir = args.build_dir or tempfile.mkdtemp(prefix="ygg_hist_seg_")
    os.makedirs(build_dir, exist_ok=True)
    items = [int(v) for v in args.items.split(",") if v]
    with ThreadPoolExecutor(max_workers=max(1, len(items))) as ex:
        built = list(ex.map(lambda v: build_variant(v, build_dir), items))
    variants = [("tree", v, p) for v, p in zip(items, built)]
    for spec in args.lib:
        label, v, path = spec.split(":", 2)
        variants.append((label, int(v), os.path.abspath(path)))
    if args.build_only:
        print(json.dumps({"built": built}))
        return

    import ydf_b200
    if ydf_b200.device_count() < 1:
        raise SystemExit("no GPU: this benchmark measures the device")
    runs = {}
    for label, v, path in variants:
        env = dict(os.environ, YGG_B200_LIB=path)
        cmd = [sys.executable, os.path.abspath(__file__), "--child", "--items-per-cta", str(v), "--steps", str(args.steps),
               "--warmup", str(args.warmup)]
        if args.rows:
            cmd += ["--rows", str(args.rows)]
        if args.features:
            cmd += ["--features", str(args.features)]
        out = subprocess.run(cmd, env=env, capture_output=True, text=True)
        line = [s for s in out.stdout.splitlines() if s.startswith("RESULT ")]
        if out.returncode != 0 or not line:
            sys.stderr.write(out.stdout + out.stderr)
            raise SystemExit(f"variant {label}:{v} failed")
        r = json.loads(line[0][len("RESULT "):])
        r["items_per_cta"] = v
        runs.setdefault(label, []).append(r)
        print(f"{label} items/CTA {v}: {r['iters_per_s']:.2f} iters/s, hist " +
              " ".join(f"{k}={t:.3f}" for k, t in r["hist_ms"].items()), file=sys.stderr, flush=True)
    res = {"metric": "k_hist_seg flush cost per work item (ms per iteration, C3)", "card": card(), "fits": {}, "runs": runs}
    for label, rs in runs.items():
        f = fit(rs)
        shipped = args.shipped if args.shipped is not None else 4
        share = 0.0
        for lv, row in f.items():
            if "hist_ms_per_item_us" in row:
                items_shipped = [r["seg_levels"][lv]["items"] for r in rs if r["items_per_cta"] == shipped]
                if items_shipped:
                    row["flush_ms_at_shipped"] = round(row["hist_ms_per_item_us"] * items_shipped[0] / 1000.0, 4)
                    share += row["flush_ms_at_shipped"]
        res["fits"][label] = {"levels": f, "flush_ms_over_seg_levels": round(share, 4), "shipped_items_per_cta": shipped}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
