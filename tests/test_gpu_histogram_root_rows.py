"""k_hist_root_rows: the root level's histogram with lanes = features over the row-major copy of the bins (32 lanes x 4
features, 16-bit carry counters).  The handle's plan on C3-sized data and the rule's precedence, the kernel's histograms
against the integer numpy reference, bit for bit, through the production launch path (ygg_debug_level_histogram), at
the geometries where it breaks (feature counts around the 128-feature groups, shards starting at odd features, partial
row blocks, reduce-scatter chunks, the largest chunk), the carry counters at their limit, and the plans it refuses."""
import numpy as np
import pytest

import ydf_b200
from ydf_b200 import _capi
from tests.test_gpu_histogram import BLOCK, HIST2, ROOT_SUM, check, gbt_of, make_bins, make_slots, num_sms, refused

pytestmark = pytest.mark.gpu

LANES, FPL, MAX_CHUNK = 32, 4, 2048


def rows_plan(chunk=1, grid=7, group=FPL, window=0):
    p = _capi.HistPlan(ROOT_SUM, group, 0, chunk, window, grid)
    p.root_lanes = LANES
    return p


@pytest.fixture(scope="module")
def c3():
    import bench
    bins, nb, na, _ = bench.make_data(dict(bench.WORKLOADS["c3"]), device=0)
    ds = ydf_b200.Dataset(bins, nb, na)
    g = np.random.default_rng(41).normal(size=bins.shape[1]).astype(np.float32)
    yield bins, ds, g
    ds.close()


def test_c3_root_plan_and_histogram(c3):
    """At C3 the root runs k_hist_root_rows (mode ROOT_SUM, 32 lanes of 4 features) and matches the reference."""
    bins, ds, g = c3
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=8, loss=1))
    p = gbt.hist_plan(0)
    assert p.mode == ROOT_SUM and p.root_lanes == LANES and p.group == FPL and p.grid == num_sms(), p
    check(gbt, bins, 0, g, np.zeros(bins.shape[1], np.int32), 1)
    gbt.close()


def test_hist2_takes_precedence(c3, monkeypatch):
    monkeypatch.setenv("YGG_HIST2", "1")
    _, ds, _ = c3
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=8, loss=1))
    p = gbt.hist_plan(0)
    assert p.mode == HIST2, p
    gbt.close()


@pytest.mark.parametrize("workload", ["c2", "tiny"])
def test_small_workloads_keep_k_hist(workload):
    import bench
    w = dict(bench.WORKLOADS[workload])
    bins, nb, na, _ = bench.make_data(w, device=0)
    gbt = gbt_of(bins, nb, na, loss=1, max_depth=w["max_depth"])
    p = gbt.hist_plan(0)
    assert p.mode == ROOT_SUM and p.root_lanes == 0, p
    gbt.close()


def test_heavy_bins_keep_k_hist():
    """Wide and large (as C5) but one dominant value: every level falls back to the shared layout, no level runs
    k_hist_seg, so the row-major copy is not built and the root stays on k_hist."""
    n, F = 8_000_000, 128
    bins = np.zeros((F, n), np.uint8)
    bins[:, ::3] = 1
    gbt = gbt_of(bins, np.full(F, 2, np.int32), np.zeros(F, np.int32), loss=1, max_depth=8)
    assert all(gbt.hist_plan(level).mode != 4 for level in range(7))
    p = gbt.hist_plan(0)
    assert p.mode == ROOT_SUM and p.root_lanes == 0, p
    gbt.close()


@pytest.mark.parametrize("F", [1, 8, 31, 33, 64, 65, 127, 129, 200])
def test_explicit_plans(F):
    """Every feature count around the 128-feature groups, whole and odd-start shards, partial last block, chunks of one
    block and the largest the carry counters allow, one CTA and many."""
    n = 3 * BLOCK + 77
    bins, nb, na = make_bins(n, F, seed=F)
    g = np.random.default_rng(F).normal(size=n).astype(np.float32)
    zero = np.zeros(n, np.int32)
    gbt = gbt_of(bins, nb, na, loss=1)
    for chunk, grid in ((1, 7), (2, 1), (MAX_CHUNK, num_sms())):
        check(gbt, bins, 0, g, zero, 1, p=rows_plan(chunk=chunk, grid=grid))
    gbt.close()
    for lo, hi in ((1, F), (3, F), (F // 2 | 1, F), (1, min(F, 130))):
        if lo >= hi:
            continue
        sh = gbt_of(bins, nb, na, loss=1)
        sh.set_feature_shard(lo, hi, 1, 2, lambda *a: 0)
        assert sh.hist_features() == (lo, hi)
        check(sh, bins, 0, g, zero, 1, p=rows_plan(chunk=1 + lo % 3, grid=5))
        sh.close()


def test_reduce_scatter_chunks():
    """Row shard with the level buffer cut into 3 feature chunks (150 features: 50 each)."""
    n = 2 * BLOCK + 100
    bins, nb, na = make_bins(n, 150, seed=8)
    gbt = gbt_of(bins, nb, na, loss=1)
    gbt.set_labels(np.zeros(n, np.float32))
    gbt.set_row_shard_scatter(0, 3, 3 * n, 0.0, allreduce=lambda *a: 0, reducescatter=lambda *a: 0,
                              allgather=lambda *a: 0)
    g = np.random.default_rng(9).normal(size=n).astype(np.float32)
    check(gbt, bins, 0, g, np.zeros(n, np.int32), 1, p=rows_plan(chunk=2, grid=4))
    gbt.close()


def test_carry_counters_at_their_limit():
    """Every gradient +P (code 2^24 - 1) and every row in bin 0 of 8 features, one chunk of 2048 blocks: 2^24 rows, 65535
    carries in each 16-bit counter, two counters per word."""
    n = MAX_CHUNK * BLOCK
    F = 8
    bins = np.zeros((F, n), np.uint8)
    bins[F - 1, ::5] = 1   # one column's carries split over two bins
    g = np.ones(n, np.float32)
    gbt = gbt_of(bins, np.full(F, 2, np.int32), np.zeros(F, np.int32), loss=1)
    s, c, _ = check(gbt, bins, 0, g, np.zeros(n, np.int32), 1, p=rows_plan(chunk=MAX_CHUNK, grid=1))
    assert c[0, 0, 0] == n and s[0, 0, 0] == n * (2 ** 24 - 1) and s[0, 0, 0] >> 32 == 65535
    gbt.close()


def test_refusals():
    n = BLOCK + 1
    bins, nb, na = make_bins(n, 40)
    g = np.random.default_rng(0).normal(size=n).astype(np.float32)
    zero, s5 = np.zeros(n, np.int32), make_slots(n, 5)
    gbt = gbt_of(bins, nb, na, loss=1)
    refused(gbt, 1, g, zero, 1, p=rows_plan(), match="root")                    # below the root
    refused(gbt, 0, g, s5, 5, p=rows_plan(), match="root")
    refused(gbt, 0, g, zero, 1, p=rows_plan(window=1), match="multi-pass")
    refused(gbt, 0, g, zero, 1, p=rows_plan(group=2), match="features per lane")
    refused(gbt, 0, g, zero, 1, p=rows_plan(chunk=MAX_CHUNK + 1), match="chunk_blocks")
    refused(gbt, 0, g, zero, 1, p=_capi.HistPlan(ROOT_SUM, 4, 16, 1, 0, 7), match="root_lanes")
    gbt.close()
    sampled = gbt_of(bins, nb, na, loss=1, subsample=0.5)
    refused(sampled, 0, g, zero, 1, p=rows_plan(), match="root")
    sampled.close()
    hg = gbt_of(bins, nb, na, loss=0, use_hessian_gain=1)
    refused(hg, 0, g, zero, 1, second=np.full(n, 0.1, np.float32), p=rows_plan(), match="second")
    hg.close()
