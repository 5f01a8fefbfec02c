"""CPU tests: the oracle against complete training runs of the reference (tests/reference_replay.py).

These are the strongest pins of the oracle: not formulas on hand-made inputs but the reference's own default runs on
Adult (binomial, 163 trees), Iris (multinomial, 18 x 3 trees) and Abalone (squared error, 45 trees), replayed node by
node — 6034 splits, 6296 leaf values, 226 training-log entries and 229 tie-breaks in total."""
import os

import numpy as np
import pytest

from tests import reference_replay as R


def test_first_tree_of_the_adult_run():
    """All 27 splits and 28 leaves of the first tree of the reference's default run on Adult: on the reference's chosen
    feature the oracle finds the same partition of the rows, the same positive count, `na_value` and score (1e-6) — for
    numerical features too, because a bucket boundary of the 255-bin discretisation coincides with the exact threshold
    on every node of this tree — no other feature scores higher (three nodes tie exactly between `education` and
    `education_num`, one between `occupation` and `age`: equivalent partitions), and every leaf value (Newton step with
    shrinkage 0.1, loss_imp_binomial.cc) agrees.  This also pins how PYDF treats string columns: the model's dataspec
    has most_frequent_value = 0 for every categorical column and orders equal counts by key ascending, and the
    `occupation` / `native_country` splits only replay under those rules (dataspec.FRONT_END_PYDF)."""
    ref, data = R.load_run("adult")
    seen, logs = R.replay(ref, data, num_iterations=1)
    assert int(ref["tree_first"][1]) == 55
    assert (seen["splits"], seen["categorical"], seen["numerical"], seen["numerical_on_a_boundary"]) == (27, 7, 19, 19)
    assert (seen["leaves"], seen["noise"]) == (28, 1)
    # six of its nodes have several features with the same float score (education / education_num, occupation / age):
    # the reference took the one its per-node candidate shuffle had put first (R.candidate_orders)
    assert seen["ties"] == seen["ties_as_shuffled"] == 6
    assert max(R.max_log_error(ref, logs).values()) <= 2e-6


def test_whole_adult_run():
    """All 163 trees (8789 nodes): the 2266 categorical splits and the 1674 numerical splits that fall on a bucket
    boundary reproduce exactly (partition, count, score 1e-6), no feature ever beats the reference's choice, all 4476
    leaf values agree, and the reference's training log — training / validation loss and accuracy after every tree —
    is reproduced from the replayed predictions."""
    ref, data = R.load_run("adult")
    seen, logs = R.replay(ref, data)
    assert (seen["splits"], seen["leaves"]) == (4313, 4476) and seen["splits"] + seen["leaves"] == len(ref["n"]) == 8789
    assert (seen["categorical"], seen["numerical"], seen["numerical_on_a_boundary"], seen["noise"]) == (2266, 2042, 1674, 5)
    assert seen["argmax_checks"] == 4308 and seen["max_leaf_err"] <= 1e-7
    assert len(logs) == 163 and max(R.max_log_error(ref, logs).values()) <= 2e-6
    # tie-breaks: at 210 nodes several features reach the same float score.  The reference keeps the first one in the order
    # of its per-node std::shuffle of the candidate features; following its mt19937 through the whole run (hold-out draws,
    # then per split-search node one shuffle + one seed per feature, nodes depth-first positive child first) predicts the
    # chosen feature at ALL of them — with libc++'s shuffle algorithm (libstdc++'s gives chance level: the golden models
    # were built against libc++).  This pins what SURVEY.md §8c lists as "parity unpinned".
    assert seen["ties"] == seen["ties_as_shuffled"] == 210


def test_whole_iris_run_multinomial():
    """Multinomial log-likelihood, 3 trees per iteration (loss_imp_multinomial.cc, gradient_boosted_trees.cc:1490-1511):
    18 iterations, 54 trees.  432 of the 539 non-noise splits fall on a bucket boundary (min_obs_in_bins = 3 merges rare
    values) and reproduce; all 611 leaf values agree to 1e-8; the training log is reproduced float-exactly.  One split of
    score 1.2e-5 differs by 1.8e-6 relative (2e-11 absolute), hence the 1e-5 bound (the repo's stated bar)."""
    ref, data = R.load_run("iris")
    seen, logs = R.replay(ref, data, score_rtol=1e-5)
    assert (seen["splits"], seen["leaves"], seen["noise"]) == (557, 611, 18) and seen["splits"] + seen["leaves"] == 1168
    assert (seen["numerical"], seen["numerical_on_a_boundary"]) == (539, 432)
    assert seen["max_leaf_err"] <= 1e-7 and seen["max_score_rerr"] <= 2e-6
    assert len(logs) == 18 and max(R.max_log_error(ref, logs).values()) <= 1e-6
    assert seen["ties"] == seen["ties_as_shuffled"] == 10   # the random stream stays in step over 3 trees per iteration


def test_whole_abalone_run_squared_error():
    """Squared error (loss_imp_mean_square_error.cc): 45 trees, one categorical feature (Type) and seven numerical ones
    with up to 2429 distinct values.  All 68 categorical splits and the 647 numerical splits on a bucket boundary
    reproduce with float-identical scores, all 1209 leaf values are float-identical, the RMSE log is float-identical."""
    ref, data = R.load_run("abalone")
    seen, logs = R.replay(ref, data)
    assert (seen["splits"], seen["leaves"], seen["noise"]) == (1164, 1209, 0) and seen["splits"] + seen["leaves"] == 2373
    assert (seen["categorical"], seen["numerical"], seen["numerical_on_a_boundary"]) == (68, 1096, 647)
    assert seen["max_leaf_err"] <= 1e-7 and seen["max_score_rerr"] <= 1e-6
    assert len(logs) == 45 and max(R.max_log_error(ref, logs).values()) <= 1e-6
    assert seen["ties"] == seen["ties_as_shuffled"] == 9


# -- whole trees: the oracle's tree trainer on the reference's gradients, against the reference's trees ----------------

def test_oracle_trees_against_the_adult_run():
    """decision_tree::Train seam (R.replay_trees): from the gradients the reference had at each of its 163 iterations the
    oracle grows, on the 255-bin + dictionary encoding, trees that coincide with the reference's in lockstep — 2803
    splits with the same partition / count / score and 2791 leaves with the same value; 36 trees coincide completely.
    The rest lies below one of the 174 reference splits that cut inside a bucket (not expressible by this path) or below
    the one node where another partition has the same float score."""
    ref, data = R.load_run("adult")
    seen = R.replay_trees(ref, data, R.oracle_trainer)
    assert (seen["trees"], seen["identical_trees"], seen["splits"], seen["leaves"]) == (163, 36, 2803, 2791)
    assert (seen["skipped_subtrees"], seen["tied_subtrees"], seen["noise"]) == (174, 1, 5)
    assert seen["splits"] + seen["leaves"] + seen["skipped_nodes"] + 2 * seen["noise"] == len(ref["n"])
    assert seen["same_feature"] == 2718 and seen["mirrored"] == 26   # the others: equivalent cut through another feature
    assert seen["max_leaf_err"] <= 1e-7 and seen["max_score_rerr"] <= 1e-6


def test_oracle_trees_with_the_reference_shuffle_against_the_adult_run():
    """The same with the oracle drawing the per-node candidate shuffle (libc++ algorithm) from the learner's random engine,
    handed over in the state the reference had at the start of each tree: ties now break like in the reference, so the
    37 trees that are comparable down to the leaves come out IDENTICAL — same features, partitions, counts, scores, leaf
    values — and only 4 of 2805 lockstep splits use another feature (the stream loses step inside a tree once a subtree
    had to be skipped)."""
    ref, data = R.load_run("adult")
    seen = R.replay_trees(ref, data, R.oracle_trainer_shuffled)
    assert (seen["trees"], seen["identical_trees"], seen["identical_trees_same_features"]) == (163, 37, 37)
    assert (seen["splits"], seen["same_feature"], seen["mirrored"], seen["tied_subtrees"]) == (2805, 2801, 0, 0)
    assert (seen["leaves"], seen["skipped_subtrees"]) == (2794, 174)


def test_oracle_trees_against_the_iris_and_abalone_runs():
    ref, data = R.load_run("iris")
    seen = R.replay_trees(ref, data, R.oracle_trainer, score_rtol=1e-5)
    assert (seen["trees"], seen["identical_trees"], seen["splits"], seen["leaves"]) == (54, 7, 156, 157)
    assert (seen["skipped_subtrees"], seen["tied_subtrees"]) == (53, 0) and seen["same_feature"] == 156
    ref, data = R.load_run("abalone")
    seen = R.replay_trees(ref, data, R.oracle_trainer)
    assert (seen["trees"], seen["splits"], seen["leaves"]) == (45, 164, 131)
    assert (seen["skipped_subtrees"], seen["tied_subtrees"]) == (78, 0) and seen["same_feature"] == 163
    assert seen["max_leaf_err"] <= 1e-7 and seen["max_score_rerr"] <= 1e-6
    seen = R.replay_trees(ref, data, R.oracle_trainer_shuffled)
    assert (seen["splits"], seen["same_feature"]) == (164, 164)


# -- one bucket per distinct value: the discretized path on the exact splitter's candidate cuts ------------------------

def test_iris_run_reproduced_completely_with_lossless_buckets():
    """Iris has at most 43 distinct values per column, so with dataspec.infer_column_lossless every threshold of the
    reference's EXACT numerical splitter lies on a bucket boundary: all 539 non-noise splits of the run replay (50 of them
    tied between features — all 50 broken as the reference's shuffle dictates), and the oracle's tree trainer with that
    shuffle reproduces ALL 54 trees identically: feature, partition, count, score, leaf values."""
    ref, data = R.load_run("iris")
    seen, logs = R.replay(ref, data, score_rtol=1e-5, lossless=True)
    assert (seen["numerical"], seen["numerical_on_a_boundary"], seen["leaves"]) == (539, 539, 611)
    assert seen["ties"] == seen["ties_as_shuffled"] == 50
    seen = R.replay_trees(ref, data, R.oracle_trainer_shuffled, score_rtol=1e-5, lossless=True)
    assert (seen["trees"], seen["identical_trees"], seen["identical_trees_same_features"]) == (54, 54, 54)
    assert (seen["splits"], seen["same_feature"], seen["skipped_subtrees"], seen["tied_subtrees"]) == (539, 539, 0, 0)
    # without the shuffle (features in dataspec order, as the CUDA engine takes them): the same partitions in 53 trees
    seen = R.replay_trees(ref, data, R.oracle_trainer, score_rtol=1e-5, lossless=True)
    assert (seen["identical_trees"], seen["tied_subtrees"], seen["skipped_subtrees"]) == (53, 1, 0)


def test_oracle_training_loop_reproduces_the_iris_training_log():
    """No help from the reference's trees here: the oracle's own boosting loop (oracle_gbt_train_mc) on the 134 training
    rows, lossless buckets, features in dataspec order, reproduces the reference's training loss and accuracy after each
    of its 28 iterations to float precision (the one tied subtree of iteration 15 has the same leaf values)."""
    import ydf_b200
    from ydf_b200 import dataspec
    from oracle import oracle as O
    ref, data = R.load_run("iris")
    names = [str(s) for s in ref["column_names"]]
    keep = ydf_b200.validation_split_mask(123456, 150, 0.1)
    voc = [str(s) for s in ref["vocabulary_class"]]
    y = np.array([voc.index(s) for s in data["class"]], np.int32)
    cols = [dataspec.infer_column_lossless(n, data[n]) for n in names[1:]]
    bins = np.stack([c.encode(data[c.name]) for c in cols])[:, keep]
    cfg = O.default_config(loss=O.LOSS_MULTINOMIAL, num_classes=3, max_depth=6, min_examples=5, shrinkage=0.1)
    out = O.gbt_train_mc(bins, [c.num_bins for c in cols], [c.na_bin for c in cols], y[keep], cfg, 28, num_threads=4)
    assert np.abs(out["loss"] - ref["log_training_loss"]).max() <= 1e-7
    assert np.abs(out["secondary"] - ref["log_training_secondary"]).max() <= 1e-7


def test_adult_run_with_lossless_buckets():
    """Adult: five of the six numerical columns have at most 116 distinct values (fnlwgt has 16610 and keeps its 255
    quantile buckets).  1743 of the 2042 numerical splits are then on a boundary and 73 of the 163 trees come out
    identical from the oracle's tree trainer (37 with quantile buckets everywhere)."""
    ref, data = R.load_run("adult")
    seen = R.replay_trees(ref, data, R.oracle_trainer_shuffled, lossless=True)
    assert (seen["trees"], seen["identical_trees"], seen["identical_trees_same_features"]) == (163, 73, 73)
    assert (seen["splits"], seen["same_feature"], seen["skipped_subtrees"], seen["tied_subtrees"]) == (3458, 3455, 136, 0)


def test_all_three_runs_reproduced_completely_with_a_bucket_per_distinct_value():
    """The complete pin of the oracle.  Test-only setting: one bucket per distinct value for EVERY numerical column
    (uint16 codes — the oracle's storage type; `fnlwgt` alone has 16610), so that every threshold of the reference's exact
    splitter is a bucket boundary.  With the reference's candidate shuffle on the learner's random stream the oracle's tree
    trainer, handed the reference's gradients, reproduces EVERY tree of the three runs identically — 163 + 54 + 45 trees,
    6011 non-noise splits with the same feature, partition, count, `na_value` and score, 6296 leaf values.  Nothing of
    the reference's default GBT training on these datasets is left unexplained."""
    for name, rtol, trees in (("adult", 1e-6, 163), ("iris", 1e-5, 54), ("abalone", 1e-6, 45)):
        ref, data = R.load_run(name)
        seen = R.replay_trees(ref, data, R.oracle_trainer_shuffled, score_rtol=rtol, lossless="all")
        assert (seen["trees"], seen["identical_trees"], seen["identical_trees_same_features"]) == (trees, trees, trees), name
        assert seen["splits"] == seen["same_feature"] and seen["mirrored"] == seen["tied_subtrees"] == seen["skipped_subtrees"] == 0
        n_noise = int(((ref["feature"] >= 0) & (ref["split_score"] < 1e-12)).sum())
        n_splits = int((ref["feature"] >= 0).sum())
        assert seen["splits"] == n_splits - n_noise and seen["noise"] <= n_noise
        assert seen["max_leaf_err"] <= 1e-7 and seen["max_score_rerr"] <= 2e-6


# -- goldens of the reference's C++ tests: one thread, C++ dataspec inference, subsample, hessian gain -------------------

def test_cxx_golden_adult_subsampling_run():
    """test_data/golden/gbt_adult_subsampling = GradientBoostedTreesOnAdult.Subsampling{Deprecated,New}Param
    (gradient_boosted_trees_test.cc:592-636): adult.csv, the tester's 20 % sample and training fold (3257 rows), subsample
    0.9, depth 4, 99 trees kept of 100.  Pins, on a real run, what the PYDF goldens do not exercise: STOCHASTIC GRADIENT
    BOOSTING (the per-iteration row draw sits between the trees in the learner's random stream: every root's row count is
    the size of that draw, 99 times), the single-thread manager (running best re-rounded to float, no seed draws), the C++
    dataspec inference (most_frequent_value as the NA replacement) and the ORDER OF EQUAL CATEGORY BUCKETS after the
    reference's std::sort — implementation-defined: with libstdc++'s order two categorical splits cut differently, with
    a stable order one, with libc++'s algorithm (oracle CATEGORY_SORT_LIBCXX; the older libc++ algorithm too) none.  All 658 splits then pick the
    reference's feature and cut; all 757 leaf values and the 99-entry training log (training AND validation loss /
    accuracy) are float-exact."""
    from oracle import oracle as O
    ref, data = R.load_run("cxx_adult_subsampling")
    for mode, other in ((O.CATEGORY_SORT_LIBCXX, 0), (O.CATEGORY_SORT_LIBCXX_CLASSIC, 0), (O.CATEGORY_SORT_STABLE, 1),
                        (O.CATEGORY_SORT_LIBSTDCXX, 2)):
        O.set_stable_category_sort(mode)
        try:
            seen, logs = R.replay_cxx(ref, data)
        finally:
            O.set_stable_category_sort(O.CATEGORY_SORT_LIBSTDCXX)
        assert (seen["trees"], seen["splits"], seen["same_winner"], seen["other_winner"]) == (99, 658, 658, 0)
        assert (seen["same_partition"], seen["other_partition"], seen["leaves"]) == (658 - other, other, 757)
        assert seen["max_leaf_err"] <= 1e-7 and max(R.max_log_error(ref, logs).values()) <= 1e-6


def test_oracle_training_loop_reproduces_the_cxx_adult_subsampling_run_and_its_golden_metrics():
    """No help from the reference's trees: the oracle's whole learner loop (hold-out draw, per-iteration row draw, libc++
    candidate shuffle and bucket order, one-thread manager, early stopping, truncation; a bucket per distinct value with
    the exact splitter's threshold rule) reproduces all 100 entries of the golden's training log float-exactly — training
    and validation — keeps the same 99 trees, and evaluated on the tester's TEST fold gives the golden metric values of
    SubsamplingNewParam: accuracy 0.8658, log loss 0.294 (YDF_TEST_METRIC's kGoldenMargin = 1e-4)."""
    ref, data = R.load_run("cxx_adult_subsampling")
    out = R.oracle_loop_cxx(ref, data, stable_category_sort=3, num_trees=100)
    assert out["num_entries"] == len(ref["log_training_loss"]) == 100 and len(out["trees"]) == len(ref["tree_first"]) == 99
    assert np.abs(out["train_loss"] - ref["log_training_loss"]).max() <= 1e-6
    assert np.abs(out["valid_loss"] - ref["log_validation_loss"]).max() <= 1e-6
    assert abs(out["validation_loss"] - float(ref["validation_loss"])) <= 1e-6
    names = [str(s) for s in ref["column_names"]]
    test = {n: ref[f"test_{n}"] for n in names}
    voc = [str(s) for s in ref["vocabulary_income"]]
    yt = np.array([voc.index(s) for s in test["income"]])
    raw = out["predict"](test).astype(np.float64)
    p = 1 / (1 + np.exp(-raw))
    assert abs(float(np.mean((raw > 0).astype(np.int32) + 1 == yt)) - 0.8658) < 1e-4
    assert abs(float(-np.mean(np.where(yt == 2, np.log(p), np.log1p(-p)))) - 0.294) < 1e-4


def test_cxx_golden_iris_hessian_run():
    """test_data/golden/gbt_iris_hessian = GradientBoostedTreesOnIris.Hessian (:1752-1761): HESSIAN GAIN on a real run
    (multinomial loss, 27 iterations x 3 trees, one thread).  All 770 leaf values (Newton step on the hessian sums) agree
    to 4e-8 and the 27-entry training log is float-exact.  Scores agree to 3e-7 wherever the same cut is found (649 of
    689 splits); the reference's exact splitter sums its float buckets in sorted-value order and the bucket path in row
    order, so float-level ties between features / thresholds fall differently at 31 + 9 nodes — never with a score
    difference above 1e-5."""
    ref, data = R.load_run("cxx_iris_hessian")
    seen, logs = R.replay_cxx(ref, data, score_rtol=1e-5)
    assert (seen["trees"], seen["splits"], seen["leaves"]) == (81, 689, 770)
    assert seen["same_winner"] + seen["other_winner"] == 689 and seen["same_winner"] >= 650
    assert seen["same_partition"] >= 640 and seen["max_score_rerr"] <= 1e-6
    assert seen["max_leaf_err"] <= 1e-7 and max(R.max_log_error(ref, logs).values()) <= 1e-6


def test_cxx_golden_iris_and_abalone_runs():
    """gbt_iris (:1737-1743, 216 trees) and gbt_abalone (:1630-1635, 42 trees): variance gain with one thread.  Every split
    picks the reference's feature and cut — 1915 + 1016, the one exception a tie at score 7.6e-10 — every leaf value
    (2166 + 1058) and every log entry is reproduced."""
    ref, data = R.load_run("cxx_iris")
    seen, logs = R.replay_cxx(ref, data, score_rtol=1e-5)
    assert (seen["trees"], seen["splits"], seen["noise"], seen["leaves"]) == (216, 1950, 34, 2166)
    assert (seen["same_winner"], seen["other_winner"], seen["same_partition"], seen["other_partition"]) == (1915, 1, 1915, 0)
    assert max(R.max_log_error(ref, logs).values()) <= 1e-6
    ref, data = R.load_run("cxx_abalone")
    seen, logs = R.replay_cxx(ref, data)
    assert (seen["trees"], seen["splits"], seen["leaves"]) == (42, 1016, 1058)
    assert (seen["same_winner"], seen["same_partition"], seen["other_winner"], seen["other_partition"]) == (1016, 1016, 0, 0)
    assert seen["max_leaf_err"] <= 1e-7 and max(R.max_log_error(ref, logs).values()) <= 1e-6


def test_oracle_training_loop_reproduces_the_cxx_abalone_training_log():
    """The oracle's whole learner loop on its own state (oracle_gbt_train_validated: hold-out draw, one-thread manager,
    libc++ candidate shuffle, early stopping, truncation) on the C++ golden gbt_abalone, a bucket per distinct value: all
    72 training-loss entries are float-exact and the model keeps the same 42 trees.  The VALIDATION losses differ by up to
    0.009: a hold-out row whose value lies between two values present in a node is routed by the middle of the EMPTY
    BUCKETS here and by the middle of the two present VALUES in the exact splitter — DESIGN.md §14's caveat, measured."""
    from oracle import oracle as O
    ref, data = R.load_run("cxx_abalone")
    names = [str(s) for s in ref["column_names"]]
    label = names[int(ref["label_col_idx"])]
    bins, nb, na, ft = [], [], [], []
    for ci, name in enumerate(names):
        if name == label:
            continue
        if ref["column_types"][ci] == 4:
            voc = [str(s) for s in ref[f"vocabulary_{name}"]]
            index, mfv = {k: j for j, k in enumerate(voc)}, int(ref["most_frequent_value"][ci])
            bins.append(np.array([mfv if s == "" else index.get(s, 0) for s in data[name].tolist()], np.uint16))
            nb.append(len(voc)); na.append(mfv); ft.append(1)
        else:
            v = data[name].astype(np.float32)
            col = R.numerical_column(name, v, "all")
            bins.append(col.encode(v)); nb.append(col.num_bins); na.append(col.na_bin); ft.append(0)
    cfg = O.default_config(loss=1, num_trees=300, max_depth=6)
    O.set_validated_shuffle_mode(O.SHUFFLE_LIBCXX)
    try:
        out = O.gbt_train_validated(np.stack(bins), nb, na, data[label].astype(np.float32), cfg, 0.1, num_threads=1, feature_type=ft)
    finally:
        O.set_validated_shuffle_mode(O.SHUFFLE_NONE)
    assert out["num_entries"] == len(ref["log_training_loss"]) == 72 and len(out["trees"]) == len(ref["tree_first"]) == 42
    assert np.abs(out["train_loss"] - ref["log_training_loss"]).max() <= 1e-6
    assert 1e-4 < np.abs(out["valid_loss"] - ref["log_validation_loss"]).max() < 0.02
    # with the exact splitter's threshold rule (oracle.set_bucket_values) the validation log is float-exact too
    out = R.oracle_loop_cxx(ref, data)
    assert out["num_entries"] == 72 and len(out["trees"]) == 42
    assert np.abs(out["train_loss"] - ref["log_training_loss"]).max() <= 1e-6
    assert np.abs(out["valid_loss"] - ref["log_validation_loss"]).max() <= 1e-6
    assert abs(out["validation_loss"] - float(ref["validation_loss"])) <= 1e-6


@pytest.mark.parametrize("test_name,config,golden", [
    ("HessianAndSubsampling (:1475-1487)", dict(use_hessian_gain=1), (0.8612, 0.2924)),
    ("L2Regularization (:1296-1312)", dict(l2_regularization=0.1), (0.8621, 0.2952)),
    ("HessianL2Categorical (:1534-1547)", dict(use_hessian_gain=1, l2_regularization_categorical=10.0), (0.8627, 0.2901)),
    ("LeafWiseGrow (:1279-1293)", dict(best_first_global=True), (0.8646, 0.2958)),
    ("RandomCategorical (:1076-1097)", dict(categorical_random=True), (0.8676, 0.2941)),
    ("HessianRandomCategorical (:1504-1517)", dict(categorical_random=True, use_hessian_gain=1), (0.867, 0.2884)),
])
def test_golden_metric_values_of_more_cxx_tests(test_name, config, golden):
    """More of GradientBoostedTreesOnAdult (gradient_boosted_trees_test.cc), same tester folds, 100 trees, depth 4, subsample
    0.9: the oracle's whole loop (R.oracle_loop_cxx) lands within YDF_TEST_METRIC's golden margin 1e-4 of the reference's
    golden accuracy / log loss on the test fold — HESSIAN gain with the Newton leaves, `l2_regularization`,
    `l2_regularization_categorical` (the hessian-gain categorical score) and `growing_strategy = BEST_FIRST_GLOBAL`
    (GrowTreeBestFirstGlobal, training.cc:4499-4656: heap on score x n, children ingested positive first, 31 leaves, root
    depth 0) on real reference numbers, and `categorical_algorithm = RANDOM` (ScanSplitsRandomBuckets,
    splitter_scanner.h:1435-1569: 32 + active^2 random masks per node and feature, drawn from the learner's own engine
    with one thread; the algorithm the reference switches to by itself from 300 categories on — SURVEY.md §8 a12).  Best-
    first growth is a §8f N3 item, the random masks the unbuilt half of a12: their restatements are pinned before the
    engine gets them."""
    from oracle import oracle as O
    config = dict(config)
    bfg = config.pop("best_first_global", False)
    random_masks = config.pop("categorical_random", False)
    ref, data = R.load_run("cxx_adult_subsampling")
    O.set_growing_strategy(bfg, 31)
    O.set_categorical_random(random_masks)
    try:
        out = R.oracle_loop_cxx(ref, data, stable_category_sort=3, num_trees=100, **config)
    finally:
        O.set_growing_strategy(False, 31)
        O.set_categorical_random(False)
    names = [str(s) for s in ref["column_names"]]
    test = {n: ref[f"test_{n}"] for n in names}
    voc = [str(s) for s in ref["vocabulary_income"]]
    yt = np.array([voc.index(s) for s in test["income"]])
    raw = out["predict"](test).astype(np.float64)
    p = 1 / (1 + np.exp(-raw))
    assert abs(float(np.mean((raw > 0).astype(np.int32) + 1 == yt)) - golden[0]) < 1e-4, test_name
    assert abs(float(-np.mean(np.where(yt == 2, np.log(p), np.log1p(-p)))) - golden[1]) < 1e-4, test_name


def test_oracle_training_loop_reproduces_the_pydf_adult_and_abalone_runs():
    """From scratch, no help from the reference's trees: the oracle's whole learner loop (concurrent manager: one shuffle +
    one seed per feature job at every split-search node; PYDF dictionaries; a bucket per distinct value with the exact
    splitter's threshold rule; libc++ shuffle and bucket order) reproduces the reference's DEFAULT PYDF runs end to end —
    Adult: all 193 log entries (training loss to 3e-8, validation loss exactly) and the same 163 trees kept after early
    stopping; Abalone: all 75 entries exactly, 45 trees.  Two seconds of CPU."""
    for name, entries, trees in (("adult", 193, 163), ("abalone", 75, 45)):
        ref, data = R.load_run(name)
        out = R.oracle_loop_cxx(ref, data, stable_category_sort=3, num_threads=4)
        assert out["num_entries"] == len(ref["log_training_loss"]) == entries and len(out["trees"]) == trees, name
        assert np.abs(out["train_loss"] - ref["log_training_loss"]).max() <= 1e-6, name
        assert np.abs(out["valid_loss"] - ref["log_validation_loss"]).max() <= 1e-6, name
        assert abs(out["validation_loss"] - float(ref["validation_loss"])) <= 1e-6, name


def test_oracle_training_loop_reproduces_the_multinomial_runs():
    """The oracle's whole loop with K trees per iteration (oracle_gbt_train_validated; early stopping counts trees, its
    initial iteration iterations): the PYDF Iris golden (28 entries, 54 trees, validation loss 0.094591 — all exact), the
    C++ golden gbt_iris (82 entries, 216 trees) and gbt_iris_hessian (37 entries, 81 trees; hessian float ties move the
    losses by up to 2e-5 from iteration 8 on, the stopping point and the kept trees are the same)."""
    for name, threads, entries, trees, tol in (("iris", 4, 28, 54, 1e-6), ("cxx_iris", 1, 82, 216, 1e-6),
                                               ("cxx_iris_hessian", 1, 37, 81, 5e-5)):
        ref, data = R.load_run(name)
        out = R.oracle_loop_cxx(ref, data, stable_category_sort=3, num_threads=threads)
        assert out["num_entries"] == len(ref["log_training_loss"]) == entries and len(out["trees"]) == trees, name
        assert np.abs(out["train_loss"] - ref["log_training_loss"]).max() <= tol, name
        assert np.abs(out["valid_loss"] - ref["log_validation_loss"]).max() <= tol, name
        assert abs(out["validation_loss"] - float(ref["validation_loss"])) <= tol, name


def test_oracle_dart_loop_reproduces_the_golden_metrics_of_the_iris_dart_test():
    """GradientBoostedTreesOnIris.Dart (gradient_boosted_trees_test.cc:1774-1784): the gbt_iris configuration (the tester's
    training fold, one thread, libc++ shuffle, 10 % hold-out, early stopping) with forest_extraction DART at dropout 0.1,
    100 trees and the DART default shrinkage 1.0 (:3257-3262).  num_candidate_attributes 8 samples nothing on Iris's 4
    features.  The oracle's DART loop (oracle.set_dart) gives the golden accuracy 0.9733 and log loss 0.2019 on the test
    fold within YDF_TEST_METRIC's 1e-4: the draws, the sampled gradients, the early stopping and the scaled model follow
    the reference."""
    ref, data = R.load_run("cxx_iris")
    z = np.load(os.path.join(R.G, "dart_cxx_test_folds.npz"))
    names = [str(s) for s in ref["column_names"]]
    assert all(np.array_equal(z[f"iris_train_{n}"], data[n]) for n in names)   # the golden run's rows are the DART run's
    test = {n: z[f"iris_test_{n}"] for n in names}
    out = R.oracle_loop_cxx(ref, data, stable_category_sort=3, num_trees=100, shrinkage=1.0, dart=0.1)
    assert out["num_entries"] == len(out["dart_dropped"]) and len(out["dart_weights"]) == len(out["trees"]) // 3
    voc = [str(s) for s in ref["vocabulary_class"]]
    yt = np.array([voc.index(str(s)) for s in test["class"]])
    raw = out["predict"](test).astype(np.float64)
    e = np.exp(raw - raw.max(1, keepdims=True))
    p = e / e.sum(1, keepdims=True)
    assert abs(float(np.mean(p.argmax(1) + 1 == yt)) - 0.9733) < 1e-4
    assert abs(float(-np.mean(np.log(p[np.arange(len(yt)), yt - 1]))) - 0.2019) < 1e-4


@pytest.mark.parametrize("test_name,config,golden", [
    ("FakeMulticlass (:1315-1331)", dict(), (0.8646, 0.2966)),
    ("FakeMulticlassL2Regularization (:1335-1351)", dict(l2_regularization=0.1), (0.8725, 0.2953)),
])
def test_golden_metric_values_of_the_multinomial_cxx_tests(test_name, config, golden):
    """GradientBoostedTreesOnAdult.FakeMulticlass*: the MULTINOMIAL loss on Adult's two classes (two trees per iteration),
    subsample 0.9 — golden accuracy / log loss on the tester's test fold within 1e-4 from the oracle's own loop."""
    from oracle import oracle as O
    ref, data = R.load_run("cxx_adult_subsampling")
    out = R.oracle_loop_cxx(ref, data, stable_category_sort=3, num_trees=100, loss=O.LOSS_MULTINOMIAL, num_classes=2, **config)
    names = [str(s) for s in ref["column_names"]]
    test = {n: ref[f"test_{n}"] for n in names}
    voc = [str(s) for s in ref["vocabulary_income"]]
    yt = np.array([voc.index(s) for s in test["income"]])
    raw = out["predict"](test).astype(np.float64)
    e = np.exp(raw - raw.max(1, keepdims=True))
    p = e / e.sum(1, keepdims=True)
    assert abs(float(np.mean(p.argmax(1) + 1 == yt)) - golden[0]) < 1e-4, test_name
    assert abs(float(-np.mean(np.log(p[np.arange(len(yt)), yt - 1]))) - golden[1]) < 1e-4, test_name


def test_oracle_training_loop_reproduces_the_cxx_adult_base_run_and_its_golden_metrics():
    """GradientBoostedTreesOnAdult.Base (:571-590; golden model gbt_adult_base, whose header holds the training log): no
    row sampling, one thread.  The oracle's whole loop reproduces all 100 log entries (training loss exactly, validation
    loss to 6e-8), keeps all 100 trees, and gives the golden metrics 0.8664 / 0.2942 on the test fold — the values the
    reference also expects of its two GOSS tests.
    This run is what identifies the order of EQUAL category buckets in the reference's builds: libstdc++'s std::sort tracks
    it for 38 iterations, libc++'s algorithm up to LLVM 15 for 30, libc++'s introsort from LLVM 16 on for all 100 (and for
    all 658 splits of the subsampling golden): oracle CATEGORY_SORT_LIBCXX."""
    from oracle import oracle as O
    ref, data = R.load_run("cxx_adult_subsampling")          # same tester folds, same dataspec
    base = np.load(os.path.join(R.G, "ydf_run_cxx_adult_base_logs.npz"))
    diverge = {}
    for mode in (O.CATEGORY_SORT_LIBCXX, O.CATEGORY_SORT_LIBCXX_CLASSIC, O.CATEGORY_SORT_LIBSTDCXX):
        out = R.oracle_loop_cxx(ref, data, stable_category_sort=mode, num_trees=100, subsample=1.0)
        k = min(out["num_entries"], 100)
        bad = np.nonzero(np.abs(out["train_loss"][:k] - base["log_training_loss"][:k]) > 1e-6)[0]
        diverge[mode] = int(bad[0]) if len(bad) else None
        if mode == O.CATEGORY_SORT_LIBCXX:
            assert out["num_entries"] == 100 and len(out["trees"]) == int(base["num_trees"]) == 100
            assert np.abs(out["valid_loss"] - base["log_validation_loss"]).max() <= 1e-6
            assert abs(out["validation_loss"] - float(base["validation_loss"])) <= 1e-6
            names = [str(s) for s in ref["column_names"]]
            test = {n: ref[f"test_{n}"] for n in names}
            voc = [str(s) for s in ref["vocabulary_income"]]
            yt = np.array([voc.index(s) for s in test["income"]])
            raw = out["predict"](test).astype(np.float64)
            p = 1 / (1 + np.exp(-raw))
            assert abs(float(np.mean((raw > 0).astype(np.int32) + 1 == yt)) - 0.8664) < 1e-4
            assert abs(float(-np.mean(np.where(yt == 2, np.log(p), np.log1p(-p)))) - 0.2942) < 1e-4
    assert diverge == {O.CATEGORY_SORT_LIBCXX: None, O.CATEGORY_SORT_LIBCXX_CLASSIC: 31, O.CATEGORY_SORT_LIBSTDCXX: 39}, diverge
