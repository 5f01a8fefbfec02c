"""The level histograms of every k_hist / k_hist2 layout against an integer numpy reference, bit for bit.

The histograms are exact integer sums of 24-bit gradient codes (DESIGN.md §3); scores, sibling subtraction, the
row-shard all-reduce and run-to-run determinism rest on that.  Each layout keeps its sums exact only inside bounds
(packed words: <= 8191 updates of a bin per work item; shared words: < 2^20 rows and < 2^12 carries per chunk; the second
plane up to 2^24 inclusive per row), so the tests drive the production launch path (ygg_debug_level_histogram) at the
geometries and values where those bounds are reached, and check the host's choice of layout per level."""
import itertools

import numpy as np
import pytest

import ydf_b200
from ydf_b200 import _capi
from tests.util import chunk_max_count, level_histogram_ref, pow2_cover

pytestmark = pytest.mark.gpu

BLOCK = 8192
ROOT_SUM, PACKED, SHARED, HIST2 = _capi.HIST_ROOT_SUM, _capi.HIST_PACKED, _capi.HIST_SHARED, _capi.HIST2


def plan(mode, group=1, chunk=1, grid=7, window=0, tiles=0):
    return _capi.HistPlan(mode, group, tiles, chunk, window, grid)


def fits(G, S):
    """k_hist's dynamic shared memory (bins, 3 TMA stages, barriers) within the 224 KB budget (non-hessian layouts)."""
    return 2 * G * S * 256 * 4 + 3 * G * BLOCK + 64 <= 224 * 1024


def hist2_fits(FL, S, T, root):
    """k_hist2's dynamic shared memory (bins, 2 tile stages, entry staging, barriers) within its 216 KB budget."""
    stage = FL // 4 * (T * 1024 + 4) * 4 + (T * 1024 * 4 if root else 0)
    return 2 * S * 256 * FL * 4 + 2 * stage + 32 * 32 * 8 + 48 <= 216 * 1024


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def make_bins(n, F, seed=0, two_bin_every=3):
    """Features with 256 bins (bin 255 populated) and, every `two_bin_every`-th feature, 2 bins."""
    rng = np.random.default_rng(seed)
    bins = rng.integers(0, 256, size=(F, n), dtype=np.uint8)
    nb = np.full(F, 256, np.int32)
    for f in range(1, F, two_bin_every):
        bins[f] = rng.integers(0, 2, size=n, dtype=np.uint8)
        nb[f] = 2
    bins[::two_bin_every, :: 7] = 255
    return bins, nb, np.zeros(F, np.int32)


def make_slots(n, n_slots, seed=1):
    """Slots with some rows in none (-1) and, with more than 2 slots, some slots left empty."""
    rng = np.random.default_rng(seed)
    s = rng.integers(-1, n_slots, size=n).astype(np.int32)
    if n_slots > 2:
        s[s == n_slots // 2] = -1
    return s


def gbt_of(bins, nb, na, weights=None, **kw):
    ds = ydf_b200.Dataset(bins, nb, na)
    g = ydf_b200.Gbt(ds, ydf_b200.default_config(**{"max_depth": 6, **kw}))
    if weights is not None:
        g.set_weights(weights)
    return g


def check(gbt, bins, level, g, slots, n_slots, second=None, p=None):
    """Runs the seam and asserts every plane equal to the reference."""
    s, c, h2, (P, V) = gbt.level_histogram(level, g, slots, n_slots, second=second, plan=p)
    lo, hi = gbt.hist_features()
    ws, wc, wh, wP = level_histogram_ref(bins, slots, n_slots, g, second=second, V=V, features=range(lo, hi))
    assert P == wP
    np.testing.assert_array_equal(c.astype(np.int64), wc, err_msg=f"counts, plan {p}")
    np.testing.assert_array_equal(s.astype(np.int64), ws, err_msg=f"sums, plan {p}")
    if second is not None:
        np.testing.assert_array_equal(h2.astype(np.int64), wh, err_msg=f"second plane, plan {p}")
    return s, c, h2


def refused(gbt, level, g, slots, n_slots, second=None, p=None, match=None):
    with pytest.raises(ydf_b200.YggError) as e:
        gbt.level_histogram(level, g, slots, n_slots, second=second, plan=p)
    assert e.value.code == 1, str(e.value)
    if match:
        assert match in str(e.value), str(e.value)


# ---- every layout and variant --------------------------------------------------------------------------------------

N = 3 * BLOCK + 5
F = 9


@pytest.fixture(scope="module")
def data():
    bins, nb, na = make_bins(N, F, seed=11)
    rng = np.random.default_rng(5)
    g = rng.normal(size=N).astype(np.float32)
    h = (rng.random(N) * 0.25).astype(np.float32)
    h[:50] = 0.25          # quantises to 2^24 (inclusive)
    h[50:100] = 0.0
    w = rng.uniform(0.05, 3.0, N).astype(np.float32)
    w[:20] = 4.0           # the handle's power of two: the largest weight itself
    return bins, nb, na, g, h, w


@pytest.mark.parametrize("kind,p,n_slots,level", [
    ("plain", plan(ROOT_SUM, group=3, chunk=2), 1, 0),
    ("plain", plan(PACKED, group=4, chunk=1), 5, 1),
    ("plain", plan(SHARED, group=5, chunk=5), 5, 2),
    ("hess", plan(SHARED, group=2, chunk=3), 5, 1),
    ("weights", plan(SHARED, group=4, chunk=2), 5, 3),
    ("plain", plan(PACKED, group=3, chunk=1, window=2), 5, 4),    # MULTI: 3 windows, the last one half full
    ("plain", plan(SHARED, group=6, chunk=2, window=2), 5, 4),
    ("hess", plan(SHARED, group=3, chunk=2, window=3), 7, 4),
] + [("plain", plan(HIST2, group=fl, tiles=t, chunk=2), 1, 0) for fl in (8, 16, 32) for t in (1, 2)]
  + [("plain", plan(HIST2, group=fl, tiles=t, chunk=1), 2, 1) for fl in (8, 16, 32) for t in (1, 2)])
def test_layout_matches_reference(data, kind, p, n_slots, level):
    bins, nb, na, g, h, w = data
    if kind == "hess":
        gbt = gbt_of(bins, nb, na, loss=0, use_hessian_gain=1)
        second = h
    elif kind == "weights":
        gbt = gbt_of(bins, nb, na, loss=1, weights=w)
        second = w
    else:
        gbt = gbt_of(bins, nb, na, loss=1)
        second = None
    slots = np.zeros(N, np.int32) if n_slots == 1 and level == 0 else make_slots(N, n_slots)
    if p.mode == HIST2 and not hist2_fits(p.group, n_slots, p.hist2_tiles, level == 0):
        refused(gbt, level, g, slots, n_slots, p=p, match="shared memory")   # (configure_launches then takes T = 1)
        return
    check(gbt, bins, level, g, slots, n_slots, second=second, p=p)
    if second is not None:
        assert gbt.level_histogram(level, g, slots, n_slots, second=second, plan=p)[3][1] == pow2_cover(second.max())


def test_debug_histogram_is_the_dequantised_level_histogram(data):
    """Gbt.debug_histogram (one node, one feature, dequantised) on plain, hessian and weighted handles."""
    bins, nb, na, g, h, w = data
    node = np.random.default_rng(3).integers(0, 3, size=N)
    slots = np.where(node == 2, 0, -1)
    ws, wc, _, P = level_histogram_ref(bins, slots, 1, g)
    for gbt in (gbt_of(bins, nb, na, loss=1), gbt_of(bins, nb, na, loss=0, use_hessian_gain=1),
                gbt_of(bins, nb, na, loss=1, weights=w)):
        for f in (0, 1, 8):
            s, c = gbt.debug_histogram(g, node, 2, f)
            np.testing.assert_array_equal(c, wc[0, f, :nb[f]])
            np.testing.assert_array_equal(s, (ws[0, f, :nb[f]] - wc[0, f, :nb[f]] * 2 ** 23) * (float(P) / 2 ** 23))


# ---- geometry where kernels break -----------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 15, 17, 8191, 8192, 8193, 3 * BLOCK + 5])
@pytest.mark.parametrize("F_", [1, 3, 9, 33])
def test_geometry(n, F_):
    bins, nb, na = make_bins(n, F_, seed=n + F_)
    gbt = gbt_of(bins, nb, na, loss=1)
    g = np.random.default_rng(n).normal(size=n).astype(np.float32)
    sms = num_sms()
    groups = range(1, 9)
    chunks = (1, 2, 5, 127)
    grids = (1, 7, sms)
    n_slots_all = (1, 2, 5, 64)
    # a rotation through the parameters: every value of every axis is used for every (n, F)
    for i in range(8):
        G, chunk, grid, ns = groups[i], chunks[i % 4], grids[i % 3], n_slots_all[(i + n) % 4]
        slots = make_slots(n, ns, seed=i)
        mode = (SHARED, PACKED)[i % 2]
        window = 0
        if not fits(G, ns):      # more slots than one pass holds: the multi-pass form with the widest window that fits
            G = min(G, max(x for x in range(1, 9) if fits(x, 2)))
            window = max(w for w in (1, 2, 4, 8, 16, 32) if fits(G, w + 1))
        p = plan(mode, group=G, chunk=chunk, grid=grid, window=window)
        if mode == PACKED and chunk_max_count(bins, chunk) > 8191:
            refused(gbt, 1, g, slots, ns, p=p, match="packed")
        else:
            check(gbt, bins, 1, g, slots, ns, p=p)
    # the root layouts over every row, and k_hist2 on the same geometry
    zero = np.zeros(n, np.int32)
    check(gbt, bins, 0, g, zero, 1, p=plan(ROOT_SUM, group=min(8, F_), chunk=chunks[n % 4], grid=grids[n % 3]))
    check(gbt, bins, 0, g, zero, 1, p=plan(HIST2, group=32, tiles=1, chunk=chunks[F_ % 4], grid=grids[F_ % 3]))
    check(gbt, bins, 0, g, zero, 1, p=plan(HIST2, group=16, tiles=2, chunk=chunks[(F_ + 1) % 4], grid=grids[F_ % 3]))
    if chunk_max_count(bins, 1) <= 8191:
        check(gbt, bins, 1, g, make_slots(n, 2), 2, p=plan(HIST2, group=8, tiles=1, chunk=1, grid=grids[n % 3]))


def test_feature_shard_inside_an_interleave_group():
    """A feature shard starting at feature 5 (k_hist2 reads 4-feature groups: the shard starts inside group 1)."""
    n = 2 * BLOCK + 9
    bins, nb, na = make_bins(n, 11, seed=3)
    gbt = gbt_of(bins, nb, na, loss=1)
    gbt.set_feature_shard(5, 11, 1, 2, lambda *a: 0)
    assert gbt.hist_features() == (5, 11)
    g = np.random.default_rng(4).normal(size=n).astype(np.float32)
    zero = np.zeros(n, np.int32)
    for fl, t in itertools.product((8, 16, 32), (1, 2)):
        if hist2_fits(fl, 1, t, True):
            check(gbt, bins, 0, g, zero, 1, p=plan(HIST2, group=fl, tiles=t, chunk=1))
    check(gbt, bins, 1, g, make_slots(n, 2), 2, p=plan(HIST2, group=16, tiles=2, chunk=1))
    check(gbt, bins, 1, g, make_slots(n, 5), 5, p=plan(SHARED, group=4, chunk=2))
    check(gbt, bins, 0, g, zero, 1)


def test_reduce_scatter_handle():
    """Row shard with the level buffer cut into 3 feature chunks (10 features: chunks of 4, 4 and 2)."""
    n = 2 * BLOCK + 100
    bins, nb, na = make_bins(n, 10, seed=8)
    gbt = gbt_of(bins, nb, na, loss=1)
    gbt.set_labels(np.zeros(n, np.float32))
    gbt.set_row_shard_scatter(0, 3, 3 * n, 0.0, allreduce=lambda *a: 0, reducescatter=lambda *a: 0,
                              allgather=lambda *a: 0)
    g = np.random.default_rng(9).normal(size=n).astype(np.float32)
    zero = np.zeros(n, np.int32)
    check(gbt, bins, 0, g, zero, 1)
    check(gbt, bins, 0, g, zero, 1, p=plan(HIST2, group=8, tiles=2, chunk=1))
    check(gbt, bins, 1, g, make_slots(n, 5), 5, p=plan(SHARED, group=3, chunk=2))
    check(gbt, bins, 1, g, make_slots(n, 5), 5, p=plan(PACKED, group=3, chunk=1, window=2))
    for level in range(1, 5):
        check(gbt, bins, level, g, make_slots(n, 1, seed=level), 1)


# ---- value edges ----------------------------------------------------------------------------------------------------

def _edge_values(P):
    k = np.arange(0, 40, dtype=np.float64)
    ties = ((k + 0.5) * P / 2 ** 23).astype(np.float32)     # g * 2^23 / P exactly halfway: ties to even
    return np.concatenate([[P, -P, 0.0, P / 2, -P / 2, np.float32(P) * np.float32(0.999999)], ties, -ties]).astype(np.float32)


@pytest.mark.parametrize("P", [1.0, 4.0, 2.0 ** -10])
def test_value_edges(P):
    """One row per bin: every bin's sum is one gradient code, compared one by one."""
    v = _edge_values(P)
    n = len(v)
    bins = np.arange(n, dtype=np.uint8)[None, :]
    gbt = gbt_of(bins, [256], [0], loss=0, use_hessian_gain=1)
    h = np.linspace(0, 0.25, n).astype(np.float32)
    h[0], h[1] = 0.25, 0.0
    slots = np.zeros(n, np.int32)
    s, c, h2 = check(gbt, bins, 1, v, slots, 1, second=h, p=plan(SHARED, chunk=1))
    assert s[0, 0, 0] == 2 ** 24 - 1 and s[0, 0, 1] == 0       # g = +P clamps, g = -P is code 0
    assert h2[0, 0, 0] == 2 ** 24 and h2[0, 0, 1] == 0          # h = h_pow2 is 2^24, h = 0 is 0
    _, _, _, (Pd, V) = gbt.level_histogram(1, v, slots, 1, second=h, plan=plan(SHARED, chunk=1))
    assert Pd == P and V == 0.25                                 # max|g| exactly a power of two: P = max|g|


def test_all_zero_gradients():
    n = BLOCK + 3
    bins, nb, na = make_bins(n, 3)
    gbt = gbt_of(bins, nb, na, loss=1)
    g = np.zeros(n, np.float32)
    s, c, _ = check(gbt, bins, 1, g, make_slots(n, 2), 2, p=plan(PACKED, group=3, chunk=1))
    assert gbt.level_histogram(1, g, make_slots(n, 2), 2, plan=plan(SHARED))[3][0] == 1.0
    np.testing.assert_array_equal(s, c.astype(np.uint64) * 2 ** 23)


# ---- field limits: one bin at its maximum --------------------------------------------------------------------------

def test_field_limits_of_a_full_chunk():
    """A constant column, every gradient +P (code 2^24 - 1), one 127-block chunk: 1,040,384 rows in the 20-bit count
    field and 4063 carries in the 12-bit carry field (shared), the same sums through the root layout's carry plane, and
    the hessian plane at 2^24 per row."""
    n = 127 * BLOCK
    bins = np.zeros((1, n), np.uint8)
    g = np.ones(n, np.float32)
    zero = np.zeros(n, np.int32)
    gbt = gbt_of(bins, [1], [0], loss=1)
    for level, p in ((1, plan(SHARED, chunk=127, grid=1)), (0, plan(ROOT_SUM, chunk=127, grid=1)),
                     (0, plan(HIST2, group=8, tiles=1, chunk=127, grid=1)), (1, plan(SHARED, chunk=127, grid=3, window=1))):
        s, c, _ = check(gbt, bins, level, g, zero, 1, p=p)
        assert c[0, 0, 0] == n == 1040384 and s[0, 0, 0] == n * (2 ** 24 - 1) and s[0, 0, 0] >> 32 == 4063
    hg = gbt_of(bins, [1], [0], loss=0, use_hessian_gain=1)
    s, c, h2 = check(hg, bins, 1, g, zero, 1, second=np.full(n, 0.25, np.float32), p=plan(SHARED, chunk=127, grid=1))
    assert h2[0, 0, 0] == n * 2 ** 24


def test_packed_field_limit_8191_rows():
    """8191 rows of one bin in a one-block chunk fill the packed count field (coarse sum 516,033 of 2^19); 8192 are refused."""
    g = np.ones(BLOCK, np.float32)
    slots = np.zeros(BLOCK, np.int32)
    bins = np.zeros((1, BLOCK), np.uint8)
    bins[0, -1] = 1
    gbt = gbt_of(bins, [2], [0], loss=1)
    for p in (plan(PACKED, chunk=1, grid=1), plan(PACKED, chunk=1, grid=1, window=1), plan(HIST2, group=8, tiles=2, chunk=1)):
        s, c, _ = check(gbt, bins, 1, g, slots, 1, p=p)
        assert c[0, 0, 0] == 8191 and 8191 * ((2 ** 24 - 1) >> 18) == 516033
    bins8192 = np.zeros((1, BLOCK), np.uint8)
    gbt2 = gbt_of(bins8192, [2], [0], loss=1)
    for p in (plan(PACKED, chunk=1, grid=1), plan(HIST2, group=8, tiles=2, chunk=1)):
        refused(gbt2, 1, g, slots, 1, p=p, match="8191")
    check(gbt2, bins8192, 1, g, slots, 1, p=plan(SHARED, chunk=1, grid=1))


# ---- the host's plan -----------------------------------------------------------------------------------------------

def _dataset(kind):
    rng = np.random.default_rng(len(kind))
    if kind == "uniform":
        n = 600_000
        bins = rng.integers(0, 256, size=(3, n), dtype=np.uint8)
    elif kind == "dominant_some_blocks":
        n = 40 * BLOCK + 77
        bins = rng.integers(0, 256, size=(3, n), dtype=np.uint8)
        bins[1, 5 * BLOCK:9 * BLOCK] = 17            # one value fills 4 blocks of feature 1
    elif kind in ("bin_8191", "bin_8192"):
        n = 16 * BLOCK
        bins = rng.integers(1, 256, size=(2, n), dtype=np.uint8)
        k = 8191 if kind == "bin_8191" else 8192
        bins[0, 3 * BLOCK:3 * BLOCK + k] = 0         # bin 0 of feature 0: k rows of block 3, none elsewhere
    elif kind.startswith("over_4m"):                 # >= 512 blocks: the packed bound works in 8-block sub-chunks
        n = 513 * BLOCK + 11
        bins = rng.integers(0, 256, size=(2, n), dtype=np.uint8)
        if kind == "over_4m_heavy":                  # 20 % of the rows in one bin: 8 blocks overflow the packed count
            bins[0, rng.random(n) < 0.2] = 3
    else:                                            # "under_4m": 500 blocks, 8000 of every block's 8192 rows in one bin
        n = 500 * BLOCK
        bins = rng.integers(0, 256, size=(2, n), dtype=np.uint8)
        col = bins[0].reshape(500, BLOCK)
        col[:, :8000] = 42
    return bins


@pytest.mark.parametrize("kind", ["uniform", "dominant_some_blocks", "bin_8191", "bin_8192", "over_4m", "over_4m_heavy",
                                  "under_4m"])
def test_handle_plan(kind):
    bins = _dataset(kind)
    F_, n = bins.shape
    gbt = gbt_of(bins, np.full(F_, 256, np.int32), np.zeros(F_, np.int32), loss=1, max_depth=4)
    n_blocks = (n + BLOCK - 1) // BLOCK
    sub = 8 if n_blocks >= 512 else 1
    g = np.random.default_rng(1).normal(size=n).astype(np.float32)
    modes = []
    for level in range(3):
        p = gbt.hist_plan(level)
        modes.append(p.mode)
        packed = p.mode == PACKED or (p.mode == HIST2 and level > 0)
        if packed:
            assert p.chunk_blocks % sub == 0
            assert chunk_max_count(bins, p.chunk_blocks) <= 8191, p
        elif level > 0:
            assert p.mode == SHARED
            # fell back: even one sub-chunk would overflow the packed count field
            assert chunk_max_count(bins, sub) > 8191, p
        n_slots = 1 << max(0, level - 1)
        slots = np.zeros(n, np.int32) if level == 0 else make_slots(n, n_slots, seed=level)
        check(gbt, bins, level, g, slots, n_slots)
    if kind in ("bin_8191", "under_4m", "uniform", "over_4m"):
        assert modes[1:] == [PACKED, PACKED], modes       # a one-sub-chunk chunk keeps the packed layout
    if kind in ("bin_8192", "dominant_some_blocks", "over_4m_heavy"):
        assert modes[1:] == [SHARED, SHARED], modes


def test_handle_plan_with_hist2(monkeypatch):
    monkeypatch.setenv("YGG_HIST2", "1")
    n = 20 * BLOCK + 3
    bins, nb, na = make_bins(n, 9, seed=21)
    gbt = gbt_of(bins, nb, na, loss=1, max_depth=4)
    g = np.random.default_rng(2).normal(size=n).astype(np.float32)
    assert gbt.hist_plan(0).mode == HIST2 and gbt.hist_plan(1).mode == HIST2
    for level in range(3):
        n_slots = 1 << max(0, level - 1)
        check(gbt, bins, level, g, np.zeros(n, np.int32) if level == 0 else make_slots(n, n_slots), n_slots)


# ---- refusals -------------------------------------------------------------------------------------------------------

def test_unsafe_plans_are_refused():
    n = BLOCK + 1
    bins, nb, na = make_bins(n, 3)
    gbt = gbt_of(bins, nb, na, loss=1)
    hg = gbt_of(bins, nb, na, loss=0, use_hessian_gain=1)
    g = np.random.default_rng(0).normal(size=n).astype(np.float32)
    h = np.full(n, 0.1, np.float32)
    zero, s5 = np.zeros(n, np.int32), make_slots(n, 5)
    refused(gbt, 1, g, s5, 5, p=plan(SHARED, chunk=128))
    refused(gbt, 1, g, s5, 5, p=plan(SHARED, group=9))
    refused(gbt, 1, g, s5, 5, p=plan(SHARED, grid=0))
    refused(gbt, 1, g, s5, 64, p=plan(SHARED, group=8), match="shared memory")     # 64 slots need a window
    refused(gbt, 1, g, s5, 5, p=plan(HIST2, group=32, tiles=2, chunk=1), match="k_hist2")
    refused(gbt, 1, g, s5, 2, p=plan(HIST2, group=12, tiles=2, chunk=1))
    refused(gbt, 1, g, zero, 1, p=plan(ROOT_SUM), match="root")
    refused(gbt, 0, g, s5, 5, p=plan(ROOT_SUM), match="root")
    refused(gbt, 0, g, np.where(zero == 0, -1, 0).astype(np.int32), 1, p=plan(ROOT_SUM), match="root")
    refused(gbt, 0, g, zero, 1, p=plan(ROOT_SUM, window=1))
    refused(hg, 1, g, s5, 5, second=h, p=plan(PACKED), match="second")
    refused(hg, 0, g, zero, 1, second=h, p=plan(ROOT_SUM), match="second")
    refused(hg, 1, g, s5, 5, p=plan(SHARED))                                        # the plane's values are missing
    refused(hg, 1, g, s5, 5, second=np.full(n, 0.5, np.float32), p=plan(SHARED))    # above h_pow2 = 1/4
    refused(gbt, 1, g, s5, 5, second=h, p=plan(SHARED))
    bad = g.copy()
    bad[7] = np.nan
    refused(gbt, 1, bad, s5, 5)
    bad[7] = np.inf
    refused(gbt, 1, bad, s5, 5)
    refused(gbt, 1, g, s5, 4)                      # slot 4 of a 4-slot call
    refused(gbt, 1, g, s5 - 1, 5)                  # slot -2
    refused(gbt, 1, g, s5, 0)
    refused(gbt, 1, g, s5, 255)
    refused(gbt, 5, g, s5, 5)                      # max_depth 6: levels 0..4
    refused(gbt, 1, g, s5, 5)                      # the handle's plan of level 1 holds 1 slot
    with pytest.raises(ydf_b200.YggError):
        gbt.hist_plan(5)
    out = np.zeros((1, 3, 256), np.uint64)
    cnt = np.zeros((1, 3, 256), np.uint32)
    sc = np.zeros(2, np.float32)
    L = ydf_b200.lib()
    import ctypes as C
    P = _capi.ptr
    for args in ((None, P(zero, C.c_int32), P(out, C.c_uint64), P(cnt, C.c_uint32), P(sc, C.c_float)),
                 (P(g, C.c_float), None, P(out, C.c_uint64), P(cnt, C.c_uint32), P(sc, C.c_float)),
                 (P(g, C.c_float), P(zero, C.c_int32), None, P(cnt, C.c_uint32), P(sc, C.c_float)),
                 (P(g, C.c_float), P(zero, C.c_int32), P(out, C.c_uint64), None, P(sc, C.c_float)),
                 (P(g, C.c_float), P(zero, C.c_int32), P(out, C.c_uint64), P(cnt, C.c_uint32), None)):
        gr, sl, o, c, s = args
        assert L.ygg_debug_level_histogram(gbt.handle, 1, None, gr, None, sl, 1, o, c, None, s) == 1
    assert L.ygg_debug_hist_plan(gbt.handle, 0, None) == 1


# ---- training is left untouched -------------------------------------------------------------------------------------

@pytest.mark.parametrize("kw", [dict(loss=0), dict(loss=0, use_hessian_gain=1), dict(loss=1, subsample=0.7)])
def test_seam_leaves_training_untouched(kw):
    from tests.util import synth
    n = 3 * BLOCK + 123
    bins, nb, na, y = synth(n, 6, seed=4, task="binary" if kw["loss"] == 0 else "regression", bins=64)

    def run(interrupt):
        gbt = gbt_of(bins, nb, na, num_trees=4, **kw)
        gbt.set_labels(y)
        gbt.train(2)
        if interrupt:
            rng = np.random.default_rng(0)
            g = rng.normal(size=n).astype(np.float32)
            second = (rng.random(n) * 0.25).astype(np.float32) if kw.get("use_hessian_gain") else None
            for level in range(3):
                ns = 1 << max(0, level - 1)
                gbt.level_histogram(level, g, np.zeros(n, np.int32) if level == 0 else make_slots(n, ns), ns, second=second)
            if second is None:
                gbt.level_histogram(1, g, make_slots(n, 2), 2, plan=plan(HIST2, group=16, tiles=2, chunk=1))
            gbt.level_histogram(2, g, make_slots(n, 9), 9, second=second, plan=plan(SHARED, group=2, chunk=3, window=4))
        gbt.train(2)
        assert gbt.num_trees() == 4
        return ([gbt.get_tree(i).tobytes() for i in range(4)], [gbt.train_loss(i) for i in range(4)],
                gbt.get_predictions().tobytes())

    assert run(True) == run(False)
