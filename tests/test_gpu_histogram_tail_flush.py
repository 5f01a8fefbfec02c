"""k_hist's block tails and its flush against the integer numpy reference, bit for bit.

A warp takes kHistUnroll slots of 32 consecutive active-list entries per iteration; at the deep levels a block's list
ends inside the window, and the slots that still hold entries run unpredicated while the one holding the list's end adds
zero in its invalid lanes.  The flush tests cover many slots per work item in every layout and reduce-scatter feature
chunks that cut a group of features (the global runs of a slot end at a chunk boundary)."""
import numpy as np
import pytest

from tests.test_gpu_histogram import BLOCK, PACKED, ROOT_SUM, SHARED, check, gbt_of, plan

pytestmark = pytest.mark.gpu

# active rows per block: empty, single row, one short of / exactly / one past a slot (1024) and a window (4096), full,
# empty blocks between full ones, and the deep levels' typical count at 10M rows
BLOCK_COUNTS = [0, 1, 1023, 1024, 4095, 4096, 4097, 8192, 0, 0, 8192, 8191, 2270, 31, 33, 0]


def uniform_bins(n, F, seed):
    """256 bins of equal frequency in every feature: the packed layout takes chunks of up to 16 blocks."""
    bins = np.random.default_rng(seed).integers(0, 256, size=(F, n), dtype=np.uint8)
    return bins, np.full(F, 256, np.int32), np.zeros(F, np.int32)


def tail_slots(counts, n_slots, seed, n=None):
    """Slots of n rows (len(counts) blocks) with counts[b] active rows (random rows, random slots) in block b."""
    rng = np.random.default_rng(seed)
    n = len(counts) * BLOCK if n is None else n
    slots = np.full(n, -1, np.int32)
    for b, k in enumerate(counts):
        rows = rng.choice(min(BLOCK, n - b * BLOCK), size=k, replace=False) + b * BLOCK
        slots[rows] = rng.integers(0, n_slots, size=k)
    return slots


@pytest.fixture(scope="module")
def tail_data():
    n = len(BLOCK_COUNTS) * BLOCK
    bins, nb, na = uniform_bins(n, 9, seed=31)
    g = np.random.default_rng(32).normal(size=n).astype(np.float32)
    return bins, nb, na, g


@pytest.mark.parametrize("group,chunk", [(1, 1), (3, 5), (8, 3), (5, 16)])   # chunk 5 / 3: a short last chunk
@pytest.mark.parametrize("n_slots", [1, 6, 32])
def test_block_tails(tail_data, group, chunk, n_slots):
    bins, nb, na, g = tail_data
    gbt = gbt_of(bins, nb, na, loss=1)
    slots = tail_slots(BLOCK_COUNTS, n_slots, seed=group * 100 + n_slots)
    if 2 * group * n_slots * 256 * 4 + 3 * group * BLOCK + 64 > 226 * 1024:
        pytest.skip("the bins and tiles do not fit one CTA's shared memory")
    check(gbt, bins, 1, g, slots, n_slots, p=plan(PACKED, group=group, chunk=chunk, grid=5))
    check(gbt, bins, 1, g, slots, n_slots, p=plan(SHARED, group=group, chunk=chunk, grid=5))


def test_block_tails_handle_plan(tail_data):
    """The handle's own plan at every level of a depth-7 tree, with the tail counts."""
    bins, nb, na, g = tail_data
    gbt = gbt_of(bins, nb, na, loss=1, max_depth=7)
    for level, n_slots in [(1, 1), (2, 2), (3, 4), (4, 8), (5, 16)]:
        check(gbt, bins, level, g, tail_slots(BLOCK_COUNTS, n_slots, seed=level), n_slots)


@pytest.mark.parametrize("kind,p,n_slots,level", [
    ("plain", plan(PACKED, group=2, chunk=2), 32, 1),
    ("plain", plan(PACKED, group=7, chunk=1), 4, 1),
    ("plain", plan(SHARED, group=1, chunk=3), 32, 2),
    ("hess", plan(SHARED, group=2, chunk=2), 9, 1),
    ("plain", plan(PACKED, group=3, chunk=2, window=4), 11, 3),     # multi-pass windows
    ("hess", plan(SHARED, group=2, chunk=1, window=5), 11, 3),
    ("plain", plan(ROOT_SUM, group=8, chunk=2), 1, 0),
])
def test_flush_layouts(kind, p, n_slots, level):
    n = 5 * BLOCK + 77
    bins, nb, na = uniform_bins(n, 17, seed=41)
    rng = np.random.default_rng(42)
    g = rng.normal(size=n).astype(np.float32)
    if kind == "hess":
        gbt = gbt_of(bins, nb, na, loss=0, use_hessian_gain=1)
        second = (rng.random(n) * 0.25).astype(np.float32)
    else:
        gbt = gbt_of(bins, nb, na, loss=1)
        second = None
    slots = np.zeros(n, np.int32) if level == 0 else rng.integers(-1, n_slots, size=n).astype(np.int32)
    check(gbt, bins, level, g, slots, n_slots, second=second, p=p)


@pytest.mark.parametrize("world", [2, 3])
def test_flush_reduce_scatter_chunks(world):
    """Row shard whose level buffer is cut into `world` feature chunks of 7 features (13 features, 3 at most): groups of
    3 features start mid-chunk, so one item's features land in two chunks; the root layout's odd stats tail leaves odd
    chunks 8 bytes off a 16-byte boundary."""
    n = 3 * BLOCK + 500
    F = 13
    bins, nb, na = uniform_bins(n, F, seed=50 + world)
    gbt = gbt_of(bins, nb, na, loss=1)
    gbt.set_labels(np.zeros(n, np.float32))
    gbt.set_row_shard_scatter(0, world, world * n, 0.0, allreduce=lambda *a: 0, reducescatter=lambda *a: 0,
                              allgather=lambda *a: 0)
    rng = np.random.default_rng(world)
    g = rng.normal(size=n).astype(np.float32)
    zero = np.zeros(n, np.int32)
    check(gbt, bins, 0, g, zero, 1)
    check(gbt, bins, 0, g, zero, 1, p=plan(ROOT_SUM, group=3, chunk=1))
    for n_slots, p in [(1, plan(PACKED, group=3, chunk=1)), (9, plan(PACKED, group=3, chunk=2)),
                       (9, plan(SHARED, group=5, chunk=1)), (9, plan(PACKED, group=2, chunk=1, window=4))]:
        check(gbt, bins, 1, g, rng.integers(-1, n_slots, size=n).astype(np.int32), n_slots, p=p)
    for level in range(1, 5):
        check(gbt, bins, level, g, tail_slots([4097, 0, 1023, 31], 2 ** (level - 1), seed=level, n=n), 2 ** (level - 1))
