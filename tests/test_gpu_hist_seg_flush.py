"""k_hist_seg's flush (tiles of consecutive bins of a few features per warp instruction) against the integer numpy
reference, bit for bit, through the production launch path: pieces that touch every bin and pieces that touch a few,
every instantiation (8, 16 and 32 lanes, one or two features per lane), shards whose feature count is not a multiple of
the group, shards starting on an odd feature, reduce-scatter feature chunks that cut a group's half, and the 8191-update
bound of the packed words in every column of a tile."""
import numpy as np
import pytest

from tests.test_gpu_histogram import BLOCK, check, gbt_of, make_slots, num_sms, plan
from tests.test_gpu_histogram_segmented import SEG, uniform_bins
from tests.util import chunk_max_count

pytestmark = pytest.mark.gpu


def sparse_bins(n, F, seed):
    """Every feature on a few bins of its own (2 to 5 of 256, bin 255 among them for every third feature): the flush
    finds most tiles empty and the non-empty bins scattered over the tiles."""
    rng = np.random.default_rng(seed)
    bins = np.empty((F, n), np.uint8)
    for f in range(F):
        vals = rng.choice(256, size=int(rng.integers(2, 6)), replace=False)
        if f % 3 == 0:
            vals[0] = 255
        bins[f] = vals[rng.integers(0, len(vals), size=n)]
    return bins, np.full(F, 256, np.int32), np.zeros(F, np.int32)


def lanes(F_):
    return (8, 16, 32) if F_ <= 32 else (32,)


@pytest.mark.parametrize("F_", [7, 24, 32, 45, 100, 200])
@pytest.mark.parametrize("kind", ["dense", "sparse"])
def test_dense_and_sparse_pieces(F_, kind):
    """Few large slots (pieces cover every bin of every feature) and many small ones (pieces of a few rows), over the
    whole row and, above 32 features, shards of an odd first feature and a count that is no multiple of 32 or 64."""
    n = 3 * BLOCK + 17
    bins, nb, na = (uniform_bins if kind == "dense" else sparse_bins)(n, F_, seed=F_)
    g = np.random.default_rng(F_ + 1).normal(size=n).astype(np.float32)
    shards = [(0, F_)] + ([(1, F_), (3, F_ - 2)] if F_ > 32 else [])
    for i, (lo, hi) in enumerate(shards):
        gbt = gbt_of(bins, nb, na, loss=1)
        if (lo, hi) != (0, F_):
            gbt.set_feature_shard(lo, hi, 1, 2, lambda *a: 0)
        assert gbt.hist_features() == (lo, hi)
        for j, fl in enumerate(lanes(F_)):
            for n_slots, chunk in ((2, 2 if kind == "dense" else 1), (200, 1)):
                assert chunk_max_count(bins, chunk, features=range(lo, hi)) <= 8191
                check(gbt, bins, 1 + (i + j) % 3, g, make_slots(n, n_slots, seed=i + j + n_slots), n_slots,
                      p=plan(SEG, group=fl, chunk=chunk, grid=(1, 5, 2 * num_sms())[(i + j) % 3]))


@pytest.mark.parametrize("F_,world", [(100, 3), (70, 5), (45, 2), (20, 3)])
def test_reduce_scatter_chunks_cut_the_halves(F_, world):
    """Row shard whose level buffer is cut into feature chunks of 34, 14, 23 and 7 features: the chunk boundaries fall
    inside the even and odd halves of a 64-feature group and inside the tiles of 8, 16 and 32 lanes."""
    n = 2 * BLOCK + 100
    bins, nb, na = uniform_bins(n, F_, seed=F_)
    gbt = gbt_of(bins, nb, na, loss=1)
    gbt.set_labels(np.zeros(n, np.float32))
    gbt.set_row_shard_scatter(0, world, world * n, 0.0, allreduce=lambda *a: 0, reducescatter=lambda *a: 0,
                              allgather=lambda *a: 0)
    g = np.random.default_rng(9).normal(size=n).astype(np.float32)
    for j, fl in enumerate(lanes(F_)):
        check(gbt, bins, 1 + j, g, make_slots(n, 6, seed=j), 6, p=plan(SEG, group=fl, chunk=1, grid=3))
        check(gbt, bins, 2, g, make_slots(n, 40, seed=j + 7), 40, p=plan(SEG, group=fl, chunk=2, grid=1))
    for level in (3, 4):
        assert gbt.hist_plan(level).mode == SEG
        check(gbt, bins, level, g, make_slots(n, 1 << (level - 1), seed=level), 1 << (level - 1))


@pytest.mark.parametrize("F_,shard", [(24, (0, 24)), (32, (0, 32)), (71, (0, 71)), (71, (1, 70))])
def test_packed_field_limit_8191_rows_in_every_column(F_, shard):
    """Pieces of one block (chunk 1, one CTA): 8191 rows of bin 0 and one of bin 1 in every block for every shard
    feature, so each column of each tile flushes a full count field next to a bin with one update; the pair's neighbour
    outside the shard (feature 0 of a shard starting at 1) takes all 8192 rows of bin 0 and is never flushed."""
    n = 4 * BLOCK
    lo, hi = shard
    bins = np.zeros((F_, n), np.uint8)
    bins[lo:hi, BLOCK - 1::BLOCK] = 1
    nb, na = np.full(F_, 2, np.int32), np.zeros(F_, np.int32)
    g = np.random.default_rng(F_).normal(size=n).astype(np.float32)
    slots = np.zeros(n, np.int32)
    gbt = gbt_of(bins, nb, na, loss=1)
    if shard != (0, F_):
        gbt.set_feature_shard(lo, hi, 1, 2, lambda *a: 0)
    for fl in lanes(hi - lo):
        s, c, _ = check(gbt, bins, 1, g, slots, 4, p=plan(SEG, group=fl, chunk=1, grid=1))
        assert (c[0, :, 0] == 4 * 8191).all() and (c[0, :, 1] == 4).all()
