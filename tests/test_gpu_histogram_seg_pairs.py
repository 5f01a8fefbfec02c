"""k_hist_seg's paired form (32 lanes, two adjacent features per lane, groups of 64 features starting at an even byte of
the row) against the integer numpy reference, bit for bit, through the production launch path: feature counts around
the group and row sizes, shards starting at odd and even features and ending inside a pair, the last row of the
dataset, and the 8191-updates bound of the packed words."""
import numpy as np
import pytest

from tests.test_gpu_histogram import BLOCK, check, gbt_of, make_slots, num_sms, plan, refused
from tests.test_gpu_histogram_segmented import SEG, uniform_bins
from tests.util import chunk_max_count

pytestmark = pytest.mark.gpu


def row_bytes(F_):
    """Bytes per row of the row-major copy k_hist_seg gathers from (seg_row_bytes)."""
    b = 32
    while b < F_ and b < 256:
        b *= 2
    return b if b >= F_ else (F_ + 255) // 256 * 256


def shards(F_):
    """The whole row, odd and even first features, and a shard ending one byte before the row's end (its last pair
    holds a feature outside the shard)."""
    rb = row_bytes(F_)
    out = [(0, F_), (1, F_), (2, F_), (5, min(F_, rb - 1)), (4, min(F_, rb - 1))]
    return [s for i, s in enumerate(out) if s not in out[:i] and s[1] - s[0] > 32]


def sharded(bins, nb, na, lo, hi):
    gbt = gbt_of(bins, nb, na, loss=1)
    if (lo, hi) != (0, bins.shape[0]):
        gbt.set_feature_shard(lo, hi, 1, 2, lambda *a: 0)
    assert gbt.hist_features() == (lo, hi)
    return gbt


@pytest.mark.parametrize("F_", [34, 63, 64, 65, 127, 128, 129, 256])
def test_matches_reference(F_):
    """Random slots (one empty, some rows in none), n not a multiple of 8192, chunks with a short last one."""
    n = 3 * BLOCK + 5
    bins, nb, na = uniform_bins(n, F_, seed=F_)
    g = np.random.default_rng(F_).normal(size=n).astype(np.float32)
    grids = (1, 7, 3 * num_sms())
    for i, (lo, hi) in enumerate(shards(F_)):
        gbt = sharded(bins, nb, na, lo, hi)
        for j, chunk in enumerate((1, 2, 127)):
            assert chunk_max_count(bins, chunk, features=range(lo, hi)) <= 8191
            n_slots = (4, 32, 128)[(i + j) % 3]
            check(gbt, bins, 1 + (i + j) % 3, g, make_slots(n, n_slots, seed=i + j), n_slots,
                  p=plan(SEG, group=32, chunk=chunk, grid=grids[(i + 2 * j) % 3]))


@pytest.mark.parametrize("F_", [129, 256])
def test_last_row_of_the_dataset(F_):
    """n a multiple of 8192 (the last row is the last of the row-major copy): the last row alone in the highest slot, the
    last piece of the level, and a full last pair at the end of the row."""
    n = 2 * BLOCK
    bins, nb, na = uniform_bins(n, F_, seed=3)
    bins[:, -1] = np.arange(F_) % 256
    g = np.random.default_rng(4).normal(size=n).astype(np.float32)
    slots = make_slots(n, 7, seed=5)
    slots[slots == 7] = -1
    slots[-1] = 7
    for lo, hi in ((0, F_), (1, F_), (3, F_ - 1)):
        gbt = sharded(bins, nb, na, lo, hi)
        for chunk, grid in ((1, 1), (2, 7)):
            s, c, _ = check(gbt, bins, 3, g, slots, 8, p=plan(SEG, group=32, chunk=chunk, grid=grid))
            assert c[7].sum() == hi - lo


def test_packed_field_limit_8191_rows():
    """Pieces of one whole block (4 blocks, chunk 1, one CTA: P = 8192): 8191 rows of one bin per block fill the count
    field in both halves of a lane; the shard's neighbour in the first pair takes all 8192 rows of a bin in every item,
    and its column may not disturb the next item.  8192 rows of a shard feature are refused."""
    n = 4 * BLOCK
    F_ = 41
    bins = np.zeros((F_, n), np.uint8)
    bins[1:, BLOCK - 1::BLOCK] = 1
    nb, na = np.full(F_, 2, np.int32), np.zeros(F_, np.int32)
    g = np.ones(n, np.float32)
    slots = np.zeros(n, np.int32)
    for lo in (0, 1):
        gbt = sharded(bins, nb, na, 1, F_) if lo else gbt_of(bins[1:], nb[1:], na[1:], loss=1)
        ref_bins = bins if lo else bins[1:]
        s, c, _ = check(gbt, ref_bins, 1, g, slots, 4, p=plan(SEG, group=32, chunk=1, grid=1))
        assert (c[0, :, 0] == 4 * 8191).all()
    refused(gbt_of(bins, nb, na, loss=1), 1, g, slots, 4, p=plan(SEG, group=32, chunk=1), match="8191")
