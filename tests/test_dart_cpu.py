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
