"""k_hist_seg (one slot per work item, node-segmented rows gathered from the row-major copy of the bins) against the
integer numpy reference, bit for bit, through the production launch path (ygg_debug_level_histogram); the host's
choice of the kernel per level; its refusals; and a depth-8 training run against the oracle."""
import numpy as np
import pytest

from ydf_b200 import _capi
from tests.test_gpu_histogram import (BLOCK, PACKED, ROOT_SUM, SHARED, check, gbt_of, make_slots, num_sms, plan,
                                      refused)
from tests.util import chunk_max_count

pytestmark = pytest.mark.gpu

SEG = _capi.HIST_SEGMENTED


def uniform_bins(n, F, seed):
    """Every feature over all 256 bins, bin 255 also on every 97th row: no bin of a chunk of up to 127 blocks reaches the
    8191 bound at the sizes used here (<= 30 blocks)."""
    rng = np.random.default_rng(seed)
    bins = rng.integers(0, 256, size=(F, n), dtype=np.uint8)
    bins[:, ::97] = 255
    return bins, np.full(F, 256, np.int32), np.zeros(F, np.int32)


def lanes_for(F_):
    return (8, 16, 32) if F_ <= 33 else (32,)


def grids():
    return (1, 7, 3 * num_sms())


@pytest.mark.parametrize("F_", [1, 9, 33, 200])
@pytest.mark.parametrize("n_slots", [4, 32, 128])
def test_matches_reference(F_, n_slots):
    """Random slots (one of them empty, some rows in none), n not a multiple of 8192, chunks with a short last one."""
    n = 3 * BLOCK + 5
    bins, nb, na = uniform_bins(n, F_, seed=F_ + n_slots)
    gbt = gbt_of(bins, nb, na, loss=1)
    g = np.random.default_rng(n_slots).normal(size=n).astype(np.float32)
    slots = make_slots(n, n_slots, seed=F_)
    for i, fl in enumerate(lanes_for(F_)):
        for chunk in (1, 2, 127):
            assert chunk_max_count(bins, chunk) <= 8191
            check(gbt, bins, 1 + i % 3, g, slots, n_slots, p=plan(SEG, group=fl, chunk=chunk, grid=grids()[(i + chunk) % 3]))


def test_slots_empty_in_some_chunks():
    """Slot s holds rows of block s % 4 only, slot 5 none, and the last block (5 rows) one slot alone."""
    n = 4 * BLOCK + 5
    bins, nb, na = uniform_bins(n, 40, seed=2)
    gbt = gbt_of(bins, nb, na, loss=1)
    g = np.random.default_rng(3).normal(size=n).astype(np.float32)
    block = np.arange(n) // BLOCK
    rng = np.random.default_rng(4)
    slots = np.where(rng.random(n) < 0.6, block % 4 + 4 * rng.integers(0, 2, n), -1).astype(np.int32)
    slots[slots == 5] = -1
    slots[block == 4] = 7
    for chunk, grid in ((1, 1), (1, 5), (2, 3 * num_sms()), (3, 2)):
        check(gbt, bins, 2, g, slots, 8, p=plan(SEG, group=32, chunk=chunk, grid=grid))
    check(gbt, bins, 2, g, np.full(n, -1, np.int32), 8, p=plan(SEG, group=32, chunk=2))   # no active row at all


def test_feature_shard_starting_mid_group():
    """A shard of features 5..44 of 45: its groups of 32 lanes straddle the row's 32-byte sectors, the last group has 8."""
    n = 2 * BLOCK + 9
    bins, nb, na = uniform_bins(n, 45, seed=6)
    gbt = gbt_of(bins, nb, na, loss=1)
    gbt.set_feature_shard(5, 45, 1, 2, lambda *a: 0)
    assert gbt.hist_features() == (5, 45)
    g = np.random.default_rng(7).normal(size=n).astype(np.float32)
    for fl in (8, 16, 32):
        check(gbt, bins, 1, g, make_slots(n, 9, seed=fl), 9, p=plan(SEG, group=fl, chunk=1, grid=7))
    for level in (3, 4):   # the handle's own plan of the deep levels
        assert gbt.hist_plan(level).mode == SEG
        check(gbt, bins, level, g, make_slots(n, 1 << (level - 1), seed=level), 1 << (level - 1))


def test_reduce_scatter_feature_chunks():
    """Row shard whose level buffer is cut into 3 feature chunks (10 features: 4, 4 and 2)."""
    n = 2 * BLOCK + 100
    bins, nb, na = uniform_bins(n, 10, seed=8)
    gbt = gbt_of(bins, nb, na, loss=1)
    gbt.set_labels(np.zeros(n, np.float32))
    gbt.set_row_shard_scatter(0, 3, 3 * n, 0.0, allreduce=lambda *a: 0, reducescatter=lambda *a: 0,
                              allgather=lambda *a: 0)
    g = np.random.default_rng(9).normal(size=n).astype(np.float32)
    check(gbt, bins, 1, g, make_slots(n, 5), 5, p=plan(SEG, group=16, chunk=1, grid=3))
    check(gbt, bins, 2, g, make_slots(n, 40, seed=2), 40, p=plan(SEG, group=8, chunk=2, grid=1))
    for level in (3, 4):
        assert gbt.hist_plan(level).mode == SEG
        check(gbt, bins, level, g, make_slots(n, 1 << (level - 1), seed=level), 1 << (level - 1))


def test_packed_field_limit_8191_rows():
    """8191 rows of one bin in one block fill the packed count field; 8192 are refused (as for k_hist's packed words)."""
    g = np.ones(BLOCK, np.float32)
    slots = np.zeros(BLOCK, np.int32)
    slots[::3] = 1
    bins = np.zeros((1, BLOCK), np.uint8)
    bins[0, -1] = 1
    s, c, _ = check(gbt_of(bins, [2], [0], loss=1), bins, 1, g, slots, 4, p=plan(SEG, group=8, chunk=1, grid=1))
    assert c[0, 0, 0] + c[1, 0, 0] == 8191
    bins8192 = np.zeros((1, BLOCK), np.uint8)
    refused(gbt_of(bins8192, [2], [0], loss=1), 1, g, slots, 4, p=plan(SEG, group=8, chunk=1), match="8191")


def test_refusals():
    n = BLOCK + 1
    bins, nb, na = uniform_bins(n, 3, seed=1)
    gbt = gbt_of(bins, nb, na, loss=1)
    hg = gbt_of(bins, nb, na, loss=0, use_hessian_gain=1)
    g = np.random.default_rng(0).normal(size=n).astype(np.float32)
    h = np.full(n, 0.1, np.float32)
    zero, s5 = np.zeros(n, np.int32), make_slots(n, 5)
    refused(gbt, 0, g, zero, 1, p=plan(SEG, group=32), match="root")
    refused(hg, 1, g, s5, 5, second=h, p=plan(SEG, group=32), match="second")
    for fl in (0, 4, 12, 64):
        refused(gbt, 1, g, s5, 5, p=plan(SEG, group=fl), match="feature lanes")
    refused(gbt, 1, g, s5, 5, p=plan(SEG, group=32, window=2), match="multi-pass")
    refused(gbt, 1, g, s5, 5, p=plan(SEG, group=32, chunk=128))
    refused(gbt, 1, g, s5, 5, p=plan(SEG, group=32, grid=0))
    refused(gbt, 1, g, s5, 5, p=plan(5, group=32), match="unknown mode")


def _modes(gbt, levels):
    return [gbt.hist_plan(level).mode for level in range(levels)]


def test_handle_plan_at_depth_8():
    """The rule: packed layout, no second plane, slot bound >= 4.  Levels 3..6 with sibling subtraction, 2..6 without;
    none on a hessian-gain handle or on data whose bins overflow the packed words."""
    n = 20 * BLOCK + 3
    bins, nb, na = uniform_bins(n, 12, seed=21)
    g = np.random.default_rng(2).normal(size=n).astype(np.float32)
    gbt = gbt_of(bins, nb, na, loss=1, max_depth=8)
    assert _modes(gbt, 7) == [ROOT_SUM, PACKED, PACKED, SEG, SEG, SEG, SEG]
    for level in range(3, 7):
        p = gbt.hist_plan(level)
        assert p.group == 16 and p.slot_window == 0 and p.grid == num_sms()
        assert chunk_max_count(bins, p.chunk_blocks) <= 8191 and p.chunk_blocks == 21   # the largest chunk: every block
        ns = 1 << (level - 1)
        check(gbt, bins, level, g, make_slots(n, ns, seed=level), ns)
    nosub = gbt_of(bins, nb, na, loss=1, max_depth=8, sibling_subtraction=0)
    assert _modes(nosub, 7) == [ROOT_SUM, PACKED, SEG, SEG, SEG, SEG, SEG]
    check(nosub, bins, 2, g, make_slots(n, 4), 4)
    hg = gbt_of(bins, nb, na, loss=0, use_hessian_gain=1, max_depth=8)
    assert SEG not in _modes(hg, 7)
    heavy = bins.copy()
    heavy[0, : 2 * BLOCK] = 3    # 16384 rows of one bin in two blocks: packed words refused from one sub-chunk up
    hv = gbt_of(heavy, nb, na, loss=1, max_depth=8)
    assert _modes(hv, 7)[1:] == [SHARED] * 6
    check(hv, heavy, 4, g, make_slots(n, 8), 8)


def test_large_chunk_shrinks_to_the_packed_bound():
    """A bin that takes 3000 rows of every block: the seg levels keep the largest chunk the 8191 bound allows (2 blocks)."""
    n = 30 * BLOCK
    bins, nb, na = uniform_bins(n, 4, seed=5)
    bins[2].reshape(30, BLOCK)[:, :3000] = 9
    gbt = gbt_of(bins, nb, na, loss=1, max_depth=8)
    p = gbt.hist_plan(4)
    assert p.mode == SEG and p.chunk_blocks == 2
    assert chunk_max_count(bins, 2) <= 8191 < chunk_max_count(bins, 3)
    g = np.random.default_rng(6).normal(size=n).astype(np.float32)
    check(gbt, bins, 4, g, make_slots(n, 8), 8)


def test_depth_8_training_matches_the_oracle():
    """Three depth-8 trees on C3-shaped data (fewer rows and features): levels 3..6 run k_hist_seg."""
    from tests.test_gpu_baseline_parity import _assert_parity, _run
    par, got, _ = _run("c3", 3, rows=400_000, features=40, informative=10)
    _assert_parity(par, 3)
    assert len(got[0]) == 255
