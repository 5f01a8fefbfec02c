"""Candidate feature sampling without a device: k, the keyed candidate order, and the learner's arguments."""
import numpy as np
import pytest
from scipy import stats

import ydf_b200
from ydf_b200 import _capi
from tests import candidate_sampling_ref as R

BINOMIAL, SQUARED_ERROR, MULTINOMIAL = 0, 1, 2


@pytest.mark.parametrize("F, loss, num, ratio, k", [
    (10, BINOMIAL, -1, None, 10),          # -1: every feature
    (10, BINOMIAL, 3, None, 3),
    (10, BINOMIAL, 50, None, 10),          # clamped to F
    (10, BINOMIAL, 0, None, 4),            # classification default: ceil(sqrt(10))
    (10, MULTINOMIAL, 0, None, 4),
    (10, SQUARED_ERROR, 0, None, 4),       # regression default: ceil(10 / 3)
    (200, SQUARED_ERROR, 0, None, 67),
    (200, BINOMIAL, 0, None, 15),
    (10, BINOMIAL, -1, 0.5, 5),
    (7, BINOMIAL, -1, 0.5, 4),             # ceil(3.5)
    (10, BINOMIAL, 3, 0.25, 3),            # the ratio takes precedence: ceil(2.5)
    (10, BINOMIAL, 7, 1.0, 10),
    (10, BINOMIAL, 7, 0.0, 4),             # a ratio of 0 gives the task's default
    (9, SQUARED_ERROR, -1, 0.0, 3),
    (1, BINOMIAL, 0, None, 1),
    (200, BINOMIAL, -1, 0.01, 2),
    # ratios whose product with F is not exact: float32(ratio) * F rounds to the integer in float arithmetic
    (10, BINOMIAL, -1, 0.1, 1),
    (5, BINOMIAL, -1, 0.2, 1),
    (10, BINOMIAL, -1, 0.3, 3),
    (200, BINOMIAL, -1, 0.1, 20),
    (10, BINOMIAL, -1, 0.7, 7),
    (3, SQUARED_ERROR, -1, 0.1, 1),
])
def test_number_of_candidate_attributes(F, loss, num, ratio, k):
    assert _capi.num_candidate_attributes(F, loss, num, ratio) == k
    assert R.num_candidate_attributes(F, loss, num, ratio) == k


@pytest.mark.parametrize("args", [(10, 0, -2, None), (10, 0, -1, 1.5), (10, 0, -1, float("nan")), (0, 0, -1, None),
                                  (10, 3, -1, None)])
def test_number_of_candidate_attributes_refusals(args):
    with pytest.raises(ydf_b200.YggError) as e:
        _capi.num_candidate_attributes(*args)
    assert e.value.code == 1


def test_key_matches_the_numpy_restatement():
    tuples = [(0, 0, 0, 0), (123456, 0, 0, 5), (123456, 7, 13, 199), (2 ** 32 - 1, 2 ** 31 - 1, 1023, 65534),
              (42, 599, 1, 2), (1, 2, 3, 4)]
    for t in tuples:
        assert _capi.candidate_key(*t) == int(R.keys(*t)), t
    rng = np.random.default_rng(0)
    seeds, trees, nodes, fs = (rng.integers(0, 2 ** 31, 200) for _ in range(4))
    got = [_capi.candidate_key(int(a), int(b), int(c), int(d)) for a, b, c, d in zip(seeds, trees, nodes, fs)]
    assert np.array_equal(np.array(got, np.uint64), R.keys(seeds, trees, nodes, fs))
    # fixed values: the formula itself (chained SplitMix64 finalizers) is part of the interface
    assert int(R.keys(0, 0, 0, 0)) == _capi.candidate_key(0, 0, 0, 0)
    assert R.mix(np.uint64(0)) == np.uint64(0xE220A8397B1DCDAF)   # SplitMix64's first output for seed 0


def test_order_is_uniform_over_nodes():
    """Each feature's position in the order, over 10^5 nodes of 8 trees, is uniform (chi-square); with k = 1 the first
    feature of the order varies across nodes and trees."""
    F, n_nodes = 12, 100000
    nodes = np.arange(n_nodes)
    tree = nodes % 8
    node = nodes // 8
    k = R.keys(123456, tree[:, None], node[:, None], np.arange(F)[None, :])   # [nodes, F]
    pos = np.argsort(np.argsort(k, axis=1, kind="stable"), axis=1, kind="stable")
    for f in range(F):
        counts = np.bincount(pos[:, f], minlength=F)
        assert stats.chisquare(counts).pvalue > 1e-4, (f, counts)
    first = np.argmin(k, axis=1)
    counts = np.bincount(first, minlength=F)
    assert stats.chisquare(counts).pvalue > 1e-4, counts
    for t in range(8):   # every tree's roots do not all start with the same feature
        assert len(np.unique(first[tree == t][:200])) == F


def test_select_takes_the_first_k_valid_features():
    F = 6
    o = R.order(7, 0, 3, F)
    tried = np.ones(F, np.uint8)
    found = np.ones(F, np.int32)
    score = np.zeros(F, np.float32)
    score[o] = [1.0, 2.0, 3.0, 4.0, 5.0, 6.0]
    assert R.select(7, 0, 3, tried, found, score, 1) == o[0]
    assert R.select(7, 0, 3, tried, found, score, 3) == o[2]
    tried[o[1]] = 0   # an invalid feature does not count towards k
    found[o[1]] = 0
    assert R.select(7, 0, 3, tried, found, score, 3) == o[3]
    assert R.select(7, 0, 3, tried, found, score, 99) == o[5]
    score[o] = [2.0, 0.0, 2.0, 2.0, 1.0, 1.0]   # equal scores: the first in the order
    assert R.select(7, 0, 3, tried, found, score, 99) == o[0]


def test_learner_arguments():
    L = ydf_b200.GradientBoostedTreesLearner
    assert L("y").num_candidate_attributes == -1 and L("y").num_candidate_attributes_ratio is None
    assert L("y", num_candidate_attributes=3).num_candidate_attributes == 3
    assert L("y", num_candidate_attributes_ratio=0.5).num_candidate_attributes_ratio == 0.5
    assert L("y", num_candidate_attributes_ratio=0).num_candidate_attributes_ratio == 0.0
    with pytest.raises(ValueError, match="Only one of"):
        L("y", num_candidate_attributes=3, num_candidate_attributes_ratio=0.5)
    with pytest.raises(ValueError):
        L("y", num_candidate_attributes=-2)
    with pytest.raises(ValueError):
        L("y", num_candidate_attributes_ratio=1.5)
    with pytest.raises(ValueError):
        L("y", num_candidate_attributes_ratio=-0.5)
    with pytest.raises(TypeError):
        L("y", num_candidate_attributes=2.5)
    with pytest.raises(TypeError):
        L("y", num_candidate_attributes=True)
    with pytest.raises(TypeError):
        L("y", num_candidate_attributes_ratio="half")
