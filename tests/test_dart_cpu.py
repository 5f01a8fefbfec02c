"""DART's accumulator and draws (tests/dart_ref.py) against hand-computed cases, and the learner's DART options."""
import numpy as np
import pytest

import ydf_b200
from tests import dart_ref as D

F32 = np.float32


def mt19937(seed):
    bg = np.random.MT19937(0)
    bg._legacy_seeding(seed)       # init_genrand(seed) = std::mt19937(seed)
    return lambda: int(bg.random_raw())


def test_accumulator_base_case():
    """DartPredictionAccumulator.Base (gradient_boosted_trees_test.cc:1982-): initial prediction 2.5, nothing dropped at
    the first iteration, one tree whose leaf of row 0 is 1.0 -> 3.5 sampled and full; the next draw drops one iteration."""
    acc = D.Accumulator([[2.5, 2.5, 2.5]])
    nxt = mt19937(12345)
    assert D.draw_dropped(nxt, 0, 0.5, libcxx=False) == []
    assert acc.sampled([])[0, 0] == F32(2.5)
    acc.update([[1.0, 2.0, 1.0]], [])
    assert acc.sampled([])[0, 0] == F32(3.5) and acc.acc[0, 0] == F32(3.5)
    assert acc.weights().tolist() == [1.0]
    assert len(D.draw_dropped(nxt, 1, 0.5, libcxx=False)) == 1
    # the second iteration (the same tree) with iteration 0 dropped: w_new = 1/2, the dropped tree scaled by 1/2
    acc.update([[1.0, 2.0, 1.0]], [0])
    assert acc.sampled([])[0, 0] == F32(2.5 + 1.0 * 1.0 * 1.0 / 2.0 + 1.0 * 1.0 / 2.0) == F32(3.5)
    assert acc.acc[0, 0] == F32(3.5)
    assert acc.sampled([0])[0, 0] == F32(3.0) and acc.sampled([1])[0, 0] == F32(3.0)
    assert acc.weights().tolist() == [0.5, 0.5]


def test_rate_one_drops_every_earlier_iteration():
    """p_0 = 1, p_1 = 2 (exact in binary): iteration 1 drops {0}: s = init, acc = init + 1 + 2/2 - 1/2, w = [1/2, 1/2];
    the scaled model init + 1/2 + 2/2 agrees."""
    nxt = mt19937(1)
    acc = D.Accumulator([[0.25]])
    acc.update([[1.0]], D.draw_dropped(nxt, 0, 1.0, libcxx=False))
    d1 = D.draw_dropped(nxt, 1, 1.0, libcxx=False)
    assert d1 == [0]
    assert acc.sampled(d1)[0, 0] == F32(0.25)
    acc.update([[2.0]], d1)
    assert acc.acc[0, 0] == F32(1.75)
    assert acc.weights().tolist() == [0.5, 0.5]
    assert D.scaled_sum(0.25, [[1.0], [2.0]], acc.weights())[0, 0] == F32(1.75)
    d2 = D.draw_dropped(nxt, 2, 1.0, libcxx=False)
    assert d2 == [0, 1]
    acc.update([[4.0]], d2)
    third = F32(F32(1) / F32(3))
    sf = F32(F32(2) / F32(3))
    assert acc.weights().tolist() == [F32(F32(0.5) * sf), F32(F32(0.5) * sf), third]
    assert np.array_equal(D.weights_after([[], [0], [0, 1]]), acc.weights())


def test_rate_zero_always_takes_the_uniform_fallback():
    """Rate 0: no draw is below it, so every iteration i > 0 drops exactly one iteration, drawn uniformly in [0, i)
    after the i unit draws."""
    for libcxx in (False, True):
        nxt = mt19937(42)
        words = mt19937(42)
        for i in range(1, 40):
            d = D.draw_dropped(nxt, i, 0.0, libcxx=libcxx)
            assert len(d) == 1 and 0 <= d[0] < i
            for _ in range(i):
                words()
            want = (D.uniform_int_libcxx if libcxx else D.uniform_int_libstdcxx)(words, i)
            assert d == [want]


def test_uniform_int_word_consumption():
    """libc++ draws nothing for a one-value range, libstdc++ one word; libc++ keeps the low bits of a word."""
    seen = []

    def counting():
        seen.append(1)
        return 0xFFFFFFF5
    assert D.uniform_int_libcxx(counting, 1) == 0 and not seen
    assert D.uniform_int_libstdcxx(counting, 1) == 0 and len(seen) == 1
    assert D.uniform_int_libcxx(lambda: 0xABCDEF06, 7) == 6   # low 3 bits
    assert D.uniform_int_libstdcxx(lambda: 3 << 30, 10) == 7  # (3 * 2^30 * 10) >> 32
    assert D.unit_float(0xFFFFFFFF) < F32(1)


def test_weights_sum_to_one_and_accumulator_matches_scaled_model():
    """Random runs: the weights always sum to about 1 per unit of output and the accumulator holds the scaled model up to
    float reassociation."""
    rng = np.random.default_rng(3)
    nxt = mt19937(7)
    n, iters = 50, 30
    acc = D.Accumulator(np.full((1, n), F32(0.1)))
    leaves = []
    for i in range(iters):
        d = D.draw_dropped(nxt, i, 0.2, libcxx=False)
        p = rng.normal(size=(1, n)).astype(F32)
        acc.update(p, d)
        leaves.append(p[0])
    want = D.scaled_sum(0.1, np.stack(leaves), acc.weights())
    assert np.allclose(acc.acc, want, rtol=1e-5, atol=1e-5)


def test_learner_dart_options():
    L = ydf_b200.GradientBoostedTreesLearner
    assert L("y", forest_extraction="DART").dart_dropout == pytest.approx(0.01)
    assert L("y", forest_extraction="DART", dart_dropout=0.3).dart_dropout == pytest.approx(0.3)
    for bad in (-0.1, 1.5):
        with pytest.raises(ValueError):
            L("y", forest_extraction="DART", dart_dropout=bad)
    with pytest.raises(NotImplementedError):
        L("y", forest_extraction="RANDOM_FOREST")


def _oracle_dart_run(rate, shuffle, K, seed):
    """A small oracle run (oracle_gbt_train_validated, no hold-out) with DART on; trees of depth 2, so exactly one
    candidate shuffle per tree, at its root."""
    from oracle import oracle as O
    from tests.util import synth_mixed
    n = 600
    bins, nb, na, ft, y = synth_mixed(n, 4, [6, 40], seed=seed, task="binary")
    if K > 1:
        y = ((bins[0].astype(np.int64) + bins[1]) % K + 1).astype(np.int32)
        y = np.where(np.random.default_rng(seed).random(n) < 0.3, (y % K) + 1, y).astype(np.int32)
    cfg = O.default_config(loss=O.LOSS_MULTINOMIAL if K > 1 else O.LOSS_BINOMIAL, num_classes=K if K > 1 else 0,
                           num_trees=30, max_depth=2, shrinkage=0.3, random_seed=seed)
    O.set_validated_shuffle_mode(shuffle)
    O.set_dart(rate)
    try:
        out = O.gbt_train_validated(bins, nb, na, y, cfg, 0.0, num_threads=1, feature_type=ft)
    finally:
        O.set_dart(None)
        O.set_validated_shuffle_mode(O.SHUFFLE_NONE)
    return out, bins.shape[0], int(cfg.random_seed)


@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.parametrize("shuffle", ["libstdcxx", "libcxx"])
@pytest.mark.parametrize("rate", [0.0, 0.1, 0.5, 1.0])
def test_oracle_dart_draws_match_the_restatement(rate, shuffle, K):
    """The oracle's DART loop (oracle.set_dart) and tests/dart_ref.py are two restatements of the reference's draws: on the
    same seed the oracle's dropped sets equal dart_ref.draw_dropped replayed on the learner's mt19937 (its words taken in
    the loop's order: the iteration's draws, then one candidate shuffle per tree), and its weights equal
    dart_ref.weights_after of those sets."""
    from oracle import oracle as O
    mode = O.SHUFFLE_LIBCXX if shuffle == "libcxx" else O.SHUFFLE_LIBSTDCXX
    out, F, seed = _oracle_dart_run(rate, mode, K, seed=17 + K)
    iters = out["num_entries"]
    assert iters == 30 and len(out["trees"]) == 30 * K and len(out["dart_dropped"]) == iters
    rng = O.Rng(seed)
    for i in range(iters):
        want = D.draw_dropped(rng.next, i, rate, libcxx=shuffle == "libcxx")
        assert out["dart_dropped"][i] == want, (i, out["dart_dropped"][i], want)
        for t in out["trees"][i * K:(i + 1) * K]:
            assert t["depth"].max() <= 2   # the root is the tree's only node that searches a split
            if shuffle == "libcxx":
                rng.shuffle_libcxx(F)
            else:
                rng.shuffle(F)
    assert np.array_equal(out["dart_weights"], D.weights_after(out["dart_dropped"]))
    if rate == 1.0:
        assert all(d == list(range(i)) for i, d in enumerate(out["dart_dropped"]))
    if rate == 0.0:
        assert all(len(d) == 1 for d in out["dart_dropped"][1:])


def test_oracle_without_dart_is_unchanged_by_an_earlier_dart_run():
    """set_dart(None) restores MART: the same run before and after a DART run gives the same trees and losses, and no
    DART state."""
    from oracle import oracle as O
    from tests.util import synth_mixed
    bins, nb, na, ft, y = synth_mixed(800, 4, [6, 40], seed=3, task="binary")
    cfg = O.default_config(loss=O.LOSS_BINOMIAL, num_trees=12, max_depth=4, shrinkage=0.3)
    before = O.gbt_train_validated(bins, nb, na, y, cfg, 0.2, num_threads=1, feature_type=ft)
    _oracle_dart_run(0.5, O.SHUFFLE_LIBCXX, 1, seed=5)
    after = O.gbt_train_validated(bins, nb, na, y, cfg, 0.2, num_threads=1, feature_type=ft)
    assert "dart_dropped" not in after and "dart_weights" not in after
    assert np.array_equal(before["train_loss"], after["train_loss"])
    assert np.array_equal(before["valid_loss"], after["valid_loss"])
    assert len(before["trees"]) == len(after["trees"])
    for a, b in zip(before["trees"], after["trees"]):
        assert np.array_equal(a, b)
