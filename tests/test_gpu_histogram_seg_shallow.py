"""k_hist_seg at tree levels 1 and 2 (one or two slots): the planner takes it there on shards of at least 128 features
and 1e9 rows x features (C3: 10M x 200).  The handle's plan per level on C3-sized data, its histograms against the
integer numpy reference, bit for bit, through the production launch path (ygg_debug_level_histogram with the handle's own
plan), and the one- and two-slot geometries through the seam on small data."""
import numpy as np
import pytest

import ydf_b200
from tests.test_gpu_histogram import BLOCK, PACKED, ROOT_SUM, SHARED, check, gbt_of, make_slots, num_sms, plan
from tests.test_gpu_histogram_segmented import SEG, uniform_bins
from tests.util import chunk_max_count

pytestmark = pytest.mark.gpu

C3 = dict(rows=10_000_000, features=200, max_depth=8, bins=256, informative=20)


def _modes(gbt, levels):
    return [gbt.hist_plan(level).mode for level in range(levels)]


def _one_empty(n, n_slots, empty, seed):
    """Random slots with some rows in none and slot `empty` holding no row."""
    s = np.random.default_rng(seed).integers(-1, n_slots, size=n).astype(np.int32)
    s[s == empty] = -1
    return s


@pytest.fixture(scope="module")
def c3():
    import bench
    bins, nb, na, _ = bench.make_data(dict(C3), device=0)
    ds = ydf_b200.Dataset(bins, nb, na)
    g = np.random.default_rng(40).normal(size=bins.shape[1]).astype(np.float32)
    yield bins, nb, na, ds, g
    ds.close()


def _gbt(ds, weights=None, **kw):
    h = ydf_b200.Gbt(ds, ydf_b200.default_config(**{"max_depth": 8, "loss": 1, **kw}))
    if weights is not None:
        h.set_weights(weights)
    return h


def test_plan_at_c3(c3):
    """Every level below the root runs k_hist_seg, with and without sibling subtraction; levels 1-2 keep the largest
    chunk the packed bound allows, as the deeper levels do."""
    _, _, _, ds, _ = c3
    for sub in (1, 0):
        gbt = _gbt(ds, sibling_subtraction=sub)
        assert _modes(gbt, 7) == [ROOT_SUM] + [SEG] * 6
        for level in (1, 2):
            p = gbt.hist_plan(level)
            assert p.group == 32 and p.slot_window == 0 and p.grid == num_sms()
            assert p.chunk_blocks == gbt.hist_plan(3).chunk_blocks and p.chunk_blocks % 8 == 0
        gbt.close()


def test_levels_1_and_2_match_the_reference(c3):
    """The handle's own plan at C3: level 1 with its one slot, level 2 with two of which one is empty, and level 1 with
    two slots without sibling subtraction."""
    bins, _, _, ds, g = c3
    n = bins.shape[1]
    gbt = _gbt(ds)
    check(gbt, bins, 1, g, make_slots(n, 1, seed=1), 1)
    check(gbt, bins, 2, g, _one_empty(n, 2, 0, seed=2), 2)
    gbt.close()
    nosub = _gbt(ds, sibling_subtraction=0)
    check(nosub, bins, 1, g, make_slots(n, 2, seed=3), 2)
    nosub.close()


def test_the_rule_follows_the_shard(c3):
    """A shard of features 1..200 (paired groups from byte 0, the first column dropped) takes k_hist_seg at levels 1 and 2
    and matches the reference there; a shard of 127 features, or 128 features over too few rows, keeps k_hist."""
    bins, nb, na, ds, g = c3
    n = bins.shape[1]
    odd = _gbt(ds)
    odd.set_feature_shard(1, 200, 1, 2, lambda *a: 0)
    assert odd.hist_features() == (1, 200)
    assert _modes(odd, 7) == [ROOT_SUM] + [SEG] * 6
    check(odd, bins, 2, g, make_slots(n, 2, seed=4), 2)
    odd.close()
    for lo, hi, want in ((0, 128, SEG), (5, 133, SEG), (0, 127, PACKED), (73, 200, PACKED)):
        h = _gbt(ds)
        h.set_feature_shard(lo, hi, 1, 2, lambda *a: 0)
        assert _modes(h, 7) == [ROOT_SUM, want, want] + [SEG] * 4, (lo, hi)
        h.close()
    small = gbt_of(bins[:200, : 20 * BLOCK], nb, na, loss=1, max_depth=8)   # 164k rows x 200 features
    assert _modes(small, 7) == [ROOT_SUM, PACKED, PACKED] + [SEG] * 4


def test_heavy_bins_fall_back_to_k_hist(c3):
    """C3 with one feature's first two blocks in one bin (the packed words overflow at one sub-chunk): levels 1 and 2
    take the shared layout with k_hist's own geometry (feature groups of at most 8, one CTA per SM), as every deeper
    level does."""
    bins, nb, na, _, g = c3
    n = bins.shape[1]
    saved = bins[0, : 2 * BLOCK].copy()
    bins[0, : 2 * BLOCK] = 3
    try:
        ds = ydf_b200.Dataset(bins, nb, na)
        hv = _gbt(ds)
        assert _modes(hv, 7) == [ROOT_SUM] + [SHARED] * 6
        for level in (1, 2):
            p = hv.hist_plan(level)
            assert 1 <= p.group <= 8 and p.grid == num_sms() and p.slot_window == 0
        check(hv, bins, 1, g, make_slots(n, 1, seed=5), 1)
        hv.close()
        ds.close()
    finally:
        bins[0, : 2 * BLOCK] = saved


def test_second_plane_and_sampled_root_stay_on_k_hist(c3):
    """Hessian gain and example weights (a second plane) never take k_hist_seg; a sampled root (packed words, not the
    root sum) stays on k_hist while the levels below it take k_hist_seg."""
    bins, _, _, ds, _ = c3
    hg = _gbt(ds, loss=0, use_hessian_gain=1)
    assert SEG not in _modes(hg, 7)
    hg.close()
    w = np.random.default_rng(41).uniform(0.5, 2.0, bins.shape[1]).astype(np.float32)
    wt = _gbt(ds, weights=w)
    assert SEG not in _modes(wt, 7)
    wt.close()
    sampled = _gbt(ds, subsample=0.5)
    assert _modes(sampled, 7) == [PACKED] + [SEG] * 6
    sampled.close()


# ---- the one- and two-slot geometries through the seam, on small data ------------------------------------------------

def test_one_and_two_slots_through_the_seam():
    """Level 1 with one slot (also empty), level 2 with two (one empty), level 1 with two; a shard starting at an odd
    feature; grids of one CTA, a few and more than one per SM; short last chunks."""
    n = 5 * BLOCK + 3
    bins, nb, na = uniform_bins(n, 150, seed=31)
    g = np.random.default_rng(32).normal(size=n).astype(np.float32)
    cases = [(1, make_slots(n, 1, seed=1), 1), (1, np.full(n, -1, np.int32), 1), (2, make_slots(n, 2, seed=2), 2),
             (2, _one_empty(n, 2, 0, seed=3), 2), (1, _one_empty(n, 2, 1, seed=4), 2)]
    for lo, hi in ((0, 150), (5, 150), (3, 140)):
        gbt = gbt_of(bins, nb, na, loss=1, max_depth=8)
        if (lo, hi) != (0, 150):
            gbt.set_feature_shard(lo, hi, 1, 2, lambda *a: 0)
        for i, (level, slots, n_slots) in enumerate(cases):
            chunk, grid = ((1, 1), (2, 7), (4, 3 * num_sms()), (127, 5))[(i + lo) % 4]
            check(gbt, bins, level, g, slots, n_slots, p=plan(SEG, group=32, chunk=chunk, grid=grid))


def test_one_slot_at_the_8191_limit():
    """Every row in the one slot of level 1, and bin 0 of feature f on 8191 rows of block f % 4 (one chunk of 4 blocks
    passes the packed bound).  With one CTA the pieces are two whole blocks (P = 16384), so the work item that holds
    block f % 4 takes all 8191 updates of a bin, in both halves of its lanes."""
    n, F_ = 4 * BLOCK, 136
    rng = np.random.default_rng(35)
    bins = rng.integers(1, 256, size=(F_, n), dtype=np.uint8)
    for f in range(F_):
        b = f % 4
        bins[f, b * BLOCK + rng.choice(BLOCK, 8191, replace=False)] = 0
    nb, na = np.full(F_, 256, np.int32), np.zeros(F_, np.int32)
    assert chunk_max_count(bins, 4) == 8191
    gbt = gbt_of(bins, nb, na, loss=1)
    g = rng.normal(size=n).astype(np.float32)
    slots = np.zeros(n, np.int32)
    s, c, _ = check(gbt, bins, 1, g, slots, 1, p=plan(SEG, group=32, chunk=4, grid=1))
    assert (c[0, :, 0] == 8191).all()
