"""The one-pass level histogram (tests/level_hist_ref.py) against scan_ref.bucket_sums per (node, feature), with torch on
the CPU: random slots with rows in none (-1), empty slots, empty buckets, extreme gradient codes and 16-bit columns."""
import numpy as np
import torch

from tests import level_hist_ref as L
from tests import scan_ref as S


def _codes(rng, n, B):
    c = rng.integers(0, B, size=n)
    if B > 4:   # runs of empty buckets, an empty last bucket
        c = np.where((c % 5 == 2) | (c == B - 1), c // 2, c)
    return c


def test_level_bucket_sums_match_bucket_sums():
    rng = np.random.default_rng(0)
    n, n_slots = 20000, 9
    slot = rng.integers(-1, n_slots, size=n)
    slot[slot == 4] = -1                      # an empty slot
    slot[slot == n_slots - 1] = -1            # ... and an empty last slot
    q = rng.integers(0, 2 ** 24, size=n)
    q[:50], q[50:100] = 0, 2 ** 24 - 1        # the code range's ends
    hq = rng.integers(0, 2 ** 24 + 1, size=n)
    hq[:30] = 2 ** 24
    for B in (1, 2, 3, 17, 256, 4096):
        codes = _codes(rng, n, B)
        dtype = np.uint8 if B <= 256 else np.uint16
        t = [torch.from_numpy(x) for x in (slot.astype(np.int64), codes.astype(dtype), q.astype(np.int64),
                                           hq.astype(np.int64))]
        cnt, s, hs = (x.numpy() for x in L.level_bucket_sums(*t, n_slots, B))
        assert cnt.shape == (n_slots, B)
        for j in range(n_slots):
            want = S.bucket_sums(codes, np.flatnonzero(slot == j), q, hq, B)
            for got, w, name in zip((cnt[j], s[j], hs[j]), want, ("count", "sum", "second sum")):
                np.testing.assert_array_equal(got, w, err_msg=f"B {B} slot {j} {name}")
        assert cnt[4].sum() == 0 and cnt[n_slots - 1].sum() == 0
        assert cnt.sum() == (slot >= 0).sum()


def test_level_hist_provider_matches_bucket_sums():
    """The provider as check_scan calls it: level nodes given by pre-order ids, rows_of from the routing (a node's rows
    in any order, some nodes empty, rows outside every level node), mixed byte, wide and presorted columns."""
    rng = np.random.default_rng(1)
    n = 30000
    cols = [("num", _codes(rng, n, 255).astype(np.uint8), 255, None),
            ("cat", _codes(rng, n, 40).astype(np.uint8), 40, None),
            ("pre", rng.normal(size=n).astype(np.float32), 0, None),
            ("wide_num", _codes(rng, n, 700).astype(np.uint16), 700, np.arange(700, dtype=np.float32)),
            ("num", np.zeros(n, np.uint8), 1, None)]
    node_of_row = rng.integers(0, 12, size=n)   # 10 and 11: rows in no level node (a sampled-out or leaf subtree)
    nodes = np.array([3, 8, 1, 20, 5, 6, 7, 9, 2, 4])   # pre-order ids, out of order; 20 holds no row
    rows_of = {int(v): rng.permutation(np.flatnonzero(node_of_row == i)) for i, v in enumerate(nodes)}
    rows_of[20] = np.zeros(0, np.int64)
    cap = {"node": nodes}
    q = rng.integers(0, 2 ** 24, size=n)
    hq = rng.integers(0, 2 ** 24 + 1, size=n)
    hist = L.LevelHist(cols)
    sums = hist(3, cap, rows_of, q, hq)
    for j, v in enumerate(nodes):
        for f, (kind, codes, B, _) in enumerate(cols):
            got = sums(j, f)
            if kind == "pre":
                assert got is None
                continue
            want = S.bucket_sums(codes, rows_of[int(v)], q, hq, B)
            for a, b in zip(got, want):
                np.testing.assert_array_equal(a, b, err_msg=f"node {v} feature {f}")
    assert hist.levels == 1 and hist.pairs == len(nodes) * 4
