"""The extended exact fuzz's drawer (tests/exact_fuzz_ext_draw.py) without a GPU: every suite draw is accepted, the exact
fuzz's own draws are unchanged, and the suite's seeds reach every new option a few times."""
import hashlib
import json

import numpy as np

from ydf_b200 import dataspec
from tests import exact_fuzz_draw as D
from tests import exact_fuzz_ext_draw as E

# sha256 over json.dumps(exact_fuzz_draw.draw(seed), sort_keys=True) for seeds 0..39, taken before the extended drawer
BASE_DIGEST = "8d4aad4440e4d5ab84258a554c0bb3c01e9cfa9c6fd8f65e1d0d93d69851e988"
AT_LEAST = 2


def _digest(seeds):
    h = hashlib.sha256()
    for s in seeds:
        h.update(json.dumps(D.draw(s), sort_keys=True).encode())
    return h.hexdigest()


def test_every_suite_draw_is_accepted():
    for seed in E.SUITE_SEEDS:
        d = E.draw(seed)
        assert E.refusal(d) is None, (seed, E.refusal(d))
        assert d == E.draw(seed)   # deterministic


def test_the_exact_fuzz_draws_are_unchanged():
    assert list(D.SUITE_SEEDS) == list(range(40))
    assert _digest(D.SUITE_SEEDS) == BASE_DIGEST
    for seed in E.SUITE_SEEDS:   # the extended draw leaves the base draw alone
        E.draw(seed)
    assert _digest(D.SUITE_SEEDS) == BASE_DIGEST


def test_refusal_restates_dart_limits():
    d = next(E.draw(s) for s in E.SUITE_SEEDS if E.draw(s)["dart"] is not None and E.draw(s)["drive"] == "step")
    assert E.refusal(dict(d, shards=2)) is not None
    assert E.refusal(dict(d, set_predictions=True)) is not None
    assert E.refusal(dict(d, dart=1.5)) is not None
    bad = dict(d, cfg=dict(d["cfg"], candidate_shuffle=1, max_depth=3), sampling="none", candidates=None)
    assert "max_depth 2" in E.refusal(bad)
    assert E.refusal(dict(d, drive="train", n_valid=0, vweights=False)) is not None


def _disc16_endings(seeds):
    """(wide, byte) counts of the suite's 16-bit columns, by the host rule on the training rows."""
    wide = byte = 0
    for s in seeds:
        d = E.draw(s)
        values = E.disc_values(d)
        for f, col in enumerate(d["columns"]):
            if col["kind"] != "disc16":
                continue
            x = values[f][:d["n"]]
            sample = x if col["n_stats"] <= 0 else x[:col["n_stats"]]
            if dataspec.infer_column16("x", sample, col["max_bins"], col["min_obs"]).wide:
                wide += 1
            else:
                byte += 1
    return wide, byte


def test_the_suite_covers_every_new_option():
    cov = E.coverage(E.SUITE_SEEDS)
    want = ["dart rate 0.0", "dart rate 0.1", "dart rate 0.5", "dart rate 1.0", "dart rate uniform",
            "dart validation weights", "dart weighted loss 0", "dart weighted loss 2", "dart goss", "dart candidates",
            "dart best first", "dart early stopping 0", "dart early stopping 1", "dart early stopping 2",
            "column disc8", "column disc16", "nan 0.5", "twin disc_copy", "n_stats"]
    want += [f"values {k}" for k in E.VALUE_KINDS]
    low = {k: cov.get(k, 0) for k in want if cov.get(k, 0) < AT_LEAST}
    assert not low, (low, cov)
    wide, byte = _disc16_endings(E.SUITE_SEEDS)
    assert wide >= AT_LEAST and byte >= AT_LEAST, (wide, byte)


def test_raw_values_keep_their_promises():
    """The generators do what the draws count on: NaN shares, -0 / +0, fewer than 257 distinct values, a constant, a
    huge finite range, and a mean of the present values that is itself present."""
    rng = np.random.default_rng(0)
    n = 20000
    for kind in E.VALUE_KINDS:
        col = dict(values=kind)
        v = E.raw_values(col, rng, n, 0.5)
        assert v.dtype == np.float32 and len(v) == n
        assert abs(np.isnan(v).mean() - 0.5) < 0.05, kind
        assert np.isfinite(v[~np.isnan(v)]).all(), kind
    v = E.raw_values(dict(values="zeros"), rng, n, 0.0)
    zero = v == 0
    assert np.signbit(v[zero]).any() and (~np.signbit(v[zero])).any()
    assert len(np.unique(E.raw_values(dict(values="few"), rng, n, 0.0))) < 257
    assert len(np.unique(E.raw_values(dict(values="const"), rng, n, 0.05)[:100])) <= 2
    h = np.abs(E.raw_values(dict(values="huge"), rng, n, 0.0).astype(np.float64))
    assert h.max() / h[h != 0].min() > 1e40
    for m in (1, 2, 7, 300, 2001):
        v = E.raw_values(dict(values="mean_hit"), rng, m, 0.3)
        present = v[~np.isnan(v)].astype(np.float64)
        assert present.mean() in set(present.tolist()), m
