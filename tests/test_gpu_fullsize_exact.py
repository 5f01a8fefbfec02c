"""Full-size training checked exactly: every node and every split candidate of the benchmark's 10M-row workloads.

The planner takes some of its paths only at these sizes: 8-block sub-chunks above 4.2M rows (the packed-bound search and
the chunk sizes of k_hist and k_hist_seg), k_hist_seg at levels 1-7 fed by k_partition's active lists on 200 features
(paired features, three 64-feature groups and a tail), the shared layout wherever a heavy bin overflows the packed words,
and the second plane (hessians, example weights) over 4.5M-10M rows.  Each case trains with step() and candidate capture
on a table from bench.make_data and runs, on every tree:

- tests/test_gpu_boosting_exact.check_run: every node's counts and sums, leaves, predictions and losses, exactly;
- tests/test_gpu_scan_exact.check_scan on every level, with the one-pass histogram of tests/level_hist_ref.py: every
  (node, feature) candidate against the exact scan of the node's rows (the last class's tree of a multinomial iteration:
  the capture holds the last tree grown).  A tree whose gradient or hessian codes depend on a free exp rounding
  (boost_ref.exp_f32) is not scan-checked; such skips are counted and at least one tree per case must be checked.

Each case asserts the histogram plan it claims to cover (Gbt.hist_plan), so that a planner change moves no case off its
path silently, and prints what it checked with its time."""
import time

import numpy as np
import pytest

import ydf_b200
from tests import scan_ref as S
from tests.level_hist_ref import LevelHist
from tests.test_gpu_boosting_exact import check_run, labels_for
from tests.test_gpu_histogram import PACKED, ROOT_SUM, SHARED
from tests.test_gpu_histogram_segmented import SEG
from tests.test_gpu_scan_exact import LAYOUT, byte_cols, check_scan, mixed_bins
from tests.util import quantize_q24, quantize_second

pytestmark = pytest.mark.gpu

F32 = np.float32
MODE = {ROOT_SUM: "ROOT_SUM", PACKED: "PACKED", SHARED: "SHARED", SEG: "SEG"}


class BenchTable:
    """A bench.make_data table in the shape check_run reads (n, n_valid, ds, cols, vds, vcols), its labels `y` and the
    one-pass level histogram of its columns on the device."""

    def __init__(self, workload, **over):
        import bench
        self.w = dict(bench.WORKLOADS[workload], **over)
        self.bins, nb, na, self.y = bench.make_data(self.w, device=0)
        ft = self.w.get("feature_types")
        self.ds = ydf_b200.Dataset(self.bins, nb, na, feature_types=ft)
        self.n, self.n_valid = self.bins.shape[1], 0
        self.vds = self.vcols = None
        self.cols = [("cat" if ft is not None and ft[f] == 1 else "num", self.bins[f], int(nb[f]), None)
                     for f in range(len(nb))]
        self.hist = LevelHist(self.cols, device="cuda:0")

    def config(self, iters, **over):
        import bench
        cfg = bench.gbt_config(self.w, iters)
        for k, v in over.items():
            setattr(cfg, k, v)
        return cfg

    def close(self):
        self.hist.close()
        self.ds.close()


@pytest.fixture(scope="module")
def c3():
    t = BenchTable("c3")
    yield t
    t.close()


def free_codes(gbt, cfg, rows):
    """Trained rows whose gradient (hessian-gain: or hessian) codes at the tree's scales depend on exp's free rounding."""
    cap = gbt.level_candidates(0)
    free = quantize_q24(rows["g"], cap["P"]) != quantize_q24(rows["g_alt"], cap["P"])
    if cfg.use_hessian_gain and rows["h"] is not None and rows["w"] is None:
        free |= quantize_second(rows["h"], cap["h_pow2"]) != quantize_second(rows["h_alt"], cap["h_pow2"])
    if rows["sel"] is not None:
        free &= rows["sel"]
    return int(free.sum())


def run(name, table, cfg, iters, labels, weights=None):
    """check_run + check_scan on every tree (the last class's of a multinomial iteration); -> (plan, stats)."""
    t0 = time.time()
    K = int(cfg.num_classes) if cfg.loss == 2 else 1
    gbt = ydf_b200.Gbt(table.ds, cfg)
    if weights is not None:
        gbt.set_weights(weights)
    gbt.set_labels(labels)
    plan = [gbt.hist_plan(level) for level in range(cfg.max_depth - 1)]
    print(f"\n{name}: {table.n} rows x {len(table.cols)} features, plan "
          + " ".join(f"{MODE[p.mode]}(chunk {p.chunk_blocks}, group {p.group}, window {p.slot_window})" for p in plan))
    gbt.capture_candidates(True)
    hist = table.hist
    levels0, pairs0, derived0 = hist.levels, hist.pairs, hist.derived
    stats = dict(trees=0, nodes=0, scan_trees=0, skipped=0, candidates=0)

    def on_tree(t, rows):
        stats["trees"] += 1
        if t % K != K - 1:
            return
        free = free_codes(gbt, cfg, rows)
        if free:
            print(f"  tree {t}: {free} rows on a free exp rounding, not scan-checked")
            stats["skipped"] += 1
            return
        h = None if rows["w"] is not None or cfg.loss == 1 else rows["h"]
        stats["candidates"] += check_scan(gbt, cfg, rows["tree"], table.cols, rows["g"], h, w=rows["w"], tree_index=t,
                                          sel=rows["sel"], hist_of=hist)
        stats["scan_trees"] += 1

    try:
        stats["nodes"], _ = check_run(gbt, cfg, table, labels, weights=weights, iters=iters, step=True, on_tree=on_tree)
    finally:
        gbt.close()
    stats.update(levels=hist.levels - levels0, level_nodes=hist.pairs - pairs0, derived=hist.derived - derived0,
                 seconds=round(time.time() - t0, 1))
    # (level_nodes: (node, feature) sums the provider computed; candidates: those of candidate nodes that were checked)
    print(f"  {stats}")
    assert stats["trees"] == iters * K and stats["scan_trees"] >= 1, stats
    return plan, stats


def modes(plan):
    return [p.mode for p in plan]


def test_c3(c3):
    """C3 as benched: the root sum, then k_hist_seg on every level below it (32 lanes of paired features), with chunks of
    whole 8-block sub-chunks, fed by k_partition; derived nodes by sibling subtraction."""
    plan, stats = run("c3", c3, c3.config(3), 3, c3.y)
    assert modes(plan) == [ROOT_SUM] + [SEG] * 6
    for p in plan[1:]:
        assert p.group == 32 and p.chunk_blocks % 8 == 0 and p.slot_window == 0, p
    assert stats["derived"] > 0


def test_c3_subsample(c3):
    """Row sampling: the sampled root takes the packed layout (its counts are not the dataset's), with an 8-block chunk;
    the sampled rows reach k_hist_seg through k_partition."""
    plan, _ = run("c3_subsample", c3, c3.config(2, subsample=0.5), 2, c3.y)
    assert modes(plan) == [PACKED] + [SEG] * 6
    assert all(p.chunk_blocks % 8 == 0 for p in plan), plan


def test_c3_hessian(c3):
    """Hessian gain: the shared layout with the hessian plane at every level (k_hist_seg has no second plane)."""
    plan, _ = run("c3_hessian", c3, c3.config(2, use_hessian_gain=1), 2, c3.y)
    assert modes(plan) == [SHARED] * 7
    assert all(p.slot_window == 0 for p in plan), plan


def test_c5():
    """C5 as benched (100 numerical + 50 categorical columns, squared error): the first category of every categorical
    column holds about 30 % of the rows (its Zipf mass and the missing rows), far more than the 8191 updates the packed
    words take per 8-block sub-chunk, so every level below the root falls back to the shared layout.  Its root of 10M
    rows has a biased 31-bit gradient sum above 2^53 and odd gradient codes (squared error, P > 1): stat[0] is exact
    only if k_node_stats removes the bias before converting to double."""
    table = BenchTable("c5")
    try:
        cat = [f for f, c in enumerate(table.cols) if c[0] == "cat"]
        assert len(cat) == 50
        share = np.bincount(table.bins[cat[0]][:65536], minlength=256).max()
        assert share > 8191, share
        plan, stats = run("c5", table, table.config(2), 2, table.y)
        assert modes(plan) == [ROOT_SUM] + [SHARED] * 6
        assert stats["derived"] > 0
    finally:
        table.close()


def test_weighted_multinomial_4_5m():
    """4.5M rows x C2's 50 features, just above the 8-block sub-chunk threshold: the multinomial loss with K = 3 classes
    (quantiles of the margin), example weights in [0.1, 3] with 5 % zeros: the shared layout with the weight plane at
    every level.  The shared layout has no packed bound, so its chunks are whole blocks of any number (not 8-block
    sub-chunks); the 8-block table only decides the packed levels."""
    table = BenchTable("c2", rows=4_500_000, loss=1)
    try:
        assert table.n // 8192 >= 512
        y = labels_for(2, table.y.astype(np.float64), 3)
        rng = np.random.default_rng(45)
        w = rng.uniform(0.1, 3.0, size=table.n).astype(F32)
        w[rng.random(table.n) < 0.05] = 0.0
        plan, _ = run("wmc_4.5M", table, table.config(1, loss=2, num_classes=3), 1, y, weights=w)
        assert modes(plan) == [SHARED] * 5
    finally:
        table.close()


def test_provider_matches_bucket_sums():
    """The one-pass level histogram on the device against scan_ref.bucket_sums per (node, feature) at every level of a
    captured tree on a 50k-row mixed table; where they differ, the one-pass provider is the one that is wrong."""
    rng = np.random.default_rng(50)
    n = 50000
    bins, nb, ft = mixed_bins(rng, n, LAYOUT)
    ds = ydf_b200.Dataset(bins, nb, np.zeros(len(nb), np.int32), feature_types=ft)
    cfg = ydf_b200.default_config(loss=0, max_depth=6, use_hessian_gain=1)
    gbt = ydf_b200.Gbt(ds, cfg)
    effect = rng.normal(size=(len(nb), 256))
    m = sum(effect[f][bins[f]] for f in (0, 1, 4, 6)) + rng.normal(scale=0.5, size=n)
    g = (0.9 * m / np.abs(m).max()).astype(F32)
    h = rng.uniform(0.01, 0.25, size=n).astype(F32)
    gbt.set_labels((m > 0).astype(np.int32) + 1)
    gbt.capture_candidates(True)
    tree = gbt.train_tree_on_gradients(g, h)
    cols = byte_cols(bins, nb, ft)
    hist = LevelHist(cols, device="cuda:0")
    from tests.boost_ref import route
    rows_of = route(tree, cols)
    pairs = 0
    for level in range(cfg.max_depth - 1):
        cap = gbt.level_candidates(level)
        q, hq = quantize_q24(g, cap["P"]), quantize_second(h, cap["h_pow2"])
        sums = hist(level, cap, rows_of, q, hq)
        for j, node in enumerate(cap["node"]):
            for f, (_, codes, B, _) in enumerate(cols):
                want = S.bucket_sums(codes, rows_of[int(node)], q, hq, B)
                for got, w, what in zip(sums(j, f), want, ("count", "sum", "second sum")):
                    np.testing.assert_array_equal(got, w, err_msg=f"level {level} node {node} feature {f} {what}")
                pairs += 1
    assert pairs > 100
    assert check_scan(gbt, cfg, tree, cols, g, h, hist_of=hist) > 0
    hist.close()
    gbt.close()
    ds.close()
