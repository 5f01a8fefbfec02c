"""Candidate feature sampling on the device (ygg_gbt_set_candidate_sampling, DESIGN.md §23).

Every level of the checked trees is captured: each validity flag is compared with the "tried" predicate computed from the
node's rows (byte, wide and presorted columns), and each node's split with the numpy restatement of the keyed selection
(tests/candidate_sampling_ref.py) applied to the captured candidates."""
import numpy as np
import pytest

import ydf_b200
from tests import candidate_sampling_ref as R
from tests import scan_ref as S
from tests.test_gpu_scan_exact import mixed_bins, route
from tests.util import quantize_q24, quantize_second

pytestmark = pytest.mark.gpu

LAYOUT = [("num", 255), ("cat", 3), ("num", 2), ("num", 3), ("cat", 40), ("num", 64), ("cat", 17), ("num", 40),
          ("num", 16), ("num", 128), ("cat", 6), ("num", 8)]


def k_valid(cfg, F, num=-1, ratio=None):
    k = R.num_candidate_attributes(F, cfg.loss, num, ratio)
    return k if cfg.split_jobs_draw_seeds else k + 1


def check_levels(gbt, cfg, tree, tree_index, kv, cols=None, g=None, h=None, sel=None, w=None, trained_tree=False):
    """Selection of every captured level node against the restatement; with `cols` (route's column descriptions) also
    every validity flag against the tried predicate of the node's rows: all rows, or those of `sel` (subsample / GOSS),
    the gradients `g` (w*g with example weights `w`) and hessians `h` of the tree.  The tree is the last
    train_tree_on_gradients one, or with trained_tree=True tree `tree_index` of the training.
    -> (nodes checked, flags checked, invalid flags seen)."""
    wide_cat = cols and any(c[0] == "wide_cat" for c in cols)
    sets = gbt.get_category_sets(tree_index if trained_tree else -1, tree) if wide_cat else {}
    rows_of = route(tree, cols, sets) if cols else None
    if rows_of is not None and sel is not None:
        rows_of = {i: r[sel[r]] for i, r in rows_of.items()}
    min_obs = cfg.min_examples if cfg.in_split_min_examples_check else 1
    nodes = flags = invalid = 0
    for level in range(cfg.max_depth - 1):
        cap = gbt.level_candidates(level)
        tried, first = gbt.level_tried(level)
        for j in range(len(cap["node"])):
            if not cap["candidate"][j]:
                continue
            assert not (cap["found"][j] & ~tried[j].astype(bool)).any(), "a found candidate that was not tried"
            pre = int(cap["node"][j])
            want = R.select(cfg.random_seed, tree_index, first + j, tried[j], cap["found"][j], cap["score"][j], kv)
            nd = tree[pre]
            if want < 0:
                assert nd["feature"] == -1, (level, j)
            else:
                # (the stored split score is k_node_stats' recomputation from the children: not compared here)
                assert nd["feature"] == want, (level, j, int(nd["feature"]), want)
            nodes += 1
            if rows_of is None:
                continue
            rows = rows_of[pre]
            for f, (kind, codes, B, _) in enumerate(cols):
                if kind == "pre":
                    _, cnt = np.unique(codes[rows], return_counts=True)
                elif kind in ("cat", "wide_cat") and min_obs > 1:
                    P = cap["P"]
                    q = quantize_q24(g, P)
                    w_inv = None
                    if w is not None:
                        w_inv = cap["w_pow2"] / 2.0 ** 24
                        hq, hinv = quantize_second(w, cap["w_pow2"]), w_inv
                    elif h is not None:
                        hq, hinv = quantize_second(h, cap["h_pow2"]), cap["h_pow2"] / 2.0 ** 24
                    else:
                        hq, hinv = np.full(len(g), 2 ** 24, np.int64), cap["h_pow2"] / 2.0 ** 24
                    c, s, hs = S.bucket_sums(codes, rows, q, hq, B)
                    keys = S.category_keys(c, s, hs, bool(cfg.use_hessian_gain), P / 2.0 ** 23, hinv,
                                           cfg.l1_regularization, cfg.l2_regularization_categorical, w_inv=w_inv)
                    cnt = c[S.category_order(keys)]
                else:
                    cnt = np.bincount(codes[rows].astype(np.int64), minlength=B)
                ref = R.tried_from_counts(cnt, min_obs)
                assert bool(tried[j, f]) == ref, (level, pre, f, kind)
                flags += 1
                invalid += int(not ref)
    return nodes, flags, invalid


def dataset(rng, n, layout, constant=0):
    bins, nb, ft = mixed_bins(rng, n, layout)
    if constant:   # constant columns: never valid
        bins = np.concatenate([bins, np.zeros((constant, n), np.uint8)])
        nb = np.concatenate([nb, np.full(constant, 4, np.int32)])
        ft = np.concatenate([ft, np.zeros(constant, np.int32)])
    ds = ydf_b200.Dataset(bins, nb, np.zeros(len(nb), np.int32), feature_types=ft)
    cols = [("cat" if ft[f] == 1 else "num", bins[f], int(nb[f]), None) for f in range(len(nb))]
    return ds, bins, cols


def labels_for(rng, bins, cfg):
    m = (bins[0] / 64.0 + (bins[1] == 2) + 0.05 * bins[4] - 0.3 * (bins[6] % 3) + 0.02 * bins[9]
         + rng.normal(scale=0.7, size=bins.shape[1]))
    if cfg.loss == 0:
        return (m > np.median(m)).astype(np.int32) + 1
    if cfg.loss == 2:
        return np.digitize(m, np.quantile(m, [0.33, 0.66])).astype(np.int32) + 1
    return m.astype(np.float32)


# split_jobs_draw_seeds: 1 = the concurrent manager (exactly k valid features), 0 = the single-thread one (k + 1)
TRAIN_CASES = {
    "binomial_k3_concurrent": (dict(loss=0, split_jobs_draw_seeds=1), 3, None),
    "binomial_k3_single_thread": (dict(loss=0, split_jobs_draw_seeds=0), 3, None),
    "binomial_ratio_concurrent": (dict(loss=0, split_jobs_draw_seeds=1), -1, 0.5),
    "binomial_ratio_0.1_concurrent": (dict(loss=0, split_jobs_draw_seeds=1), -1, 0.1),
    "binomial_default_single_thread": (dict(loss=0, split_jobs_draw_seeds=0), 0, None),
    "binomial_hessian_concurrent": (dict(loss=0, use_hessian_gain=1, split_jobs_draw_seeds=1), 4, None),
    "binomial_hessian_single_thread": (dict(loss=0, use_hessian_gain=1, split_jobs_draw_seeds=0), 4, None),
    "squared_error_default_concurrent": (dict(loss=1, split_jobs_draw_seeds=1), 0, None),
    "squared_error_ratio0_hessian_single_thread": (dict(loss=1, use_hessian_gain=1, l2_regularization=1.0,
                                                        split_jobs_draw_seeds=0), -1, 0.0),
    "multinomial_k2_concurrent": (dict(loss=2, num_classes=3, split_jobs_draw_seeds=1), 2, None),
    "multinomial_single_thread": (dict(loss=2, num_classes=3, split_jobs_draw_seeds=0), -1, 0.3),
    "subsample_concurrent": (dict(loss=0, subsample=0.7, split_jobs_draw_seeds=1), 3, None),
    "goss_single_thread": (dict(loss=1, goss_alpha=0.2, goss_beta=0.3, split_jobs_draw_seeds=0), 2, None),
    "depth10_concurrent": (dict(loss=1, max_depth=10, min_examples=2, split_jobs_draw_seeds=1), -1, 0.25),
    "depth10_single_thread": (dict(loss=1, max_depth=10, min_examples=2, split_jobs_draw_seeds=0), 3, None),
    "k1_concurrent": (dict(loss=0, split_jobs_draw_seeds=1), 1, None),   # the radix select at rank 0
    "k1_single_thread": (dict(loss=0, split_jobs_draw_seeds=0), 1, None),
}


@pytest.mark.parametrize("case", sorted(TRAIN_CASES))
def test_trained_trees_follow_the_keyed_selection(case):
    kw, num, ratio = TRAIN_CASES[case]
    rng = np.random.default_rng(sorted(TRAIN_CASES).index(case) + 1)
    n = 40000
    ds, bins, _ = dataset(rng, n, LAYOUT)
    cfg = ydf_b200.default_config(**{"max_depth": 6, "num_trees": 4, "candidate_shuffle": 0, **kw})
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(labels_for(rng, bins, cfg))
    gbt.set_candidate_sampling(num, ratio)
    gbt.capture_candidates(True)
    gbt.train(3)
    last = gbt.num_trees() - 1
    nodes, _, _ = check_levels(gbt, cfg, gbt.get_tree(last), last, k_valid(cfg, ds.n_features, num, ratio))
    assert nodes >= 7


def test_validity_flags_byte_columns_with_constant_columns_and_large_min_examples():
    """Constant columns and min_examples = 300: many (node, feature) pairs are invalid and skipped by the cutoff."""
    rng = np.random.default_rng(17)
    n = 30000
    ds, bins, cols = dataset(rng, n, LAYOUT, constant=6)
    for in_split in (1, 0):
        cfg = ydf_b200.default_config(loss=1, max_depth=7, min_examples=300, in_split_min_examples_check=in_split,
                                      candidate_shuffle=0)
        gbt = ydf_b200.Gbt(ds, cfg)
        g = labels_for(rng, bins, cfg)
        gbt.set_labels(g)
        gbt.set_candidate_sampling(3, None)
        gbt.capture_candidates(True)
        tree = gbt.train_tree_on_gradients(g)
        nodes, flags, invalid = check_levels(gbt, cfg, tree, 0, k_valid(cfg, ds.n_features, 3), cols, g)
        assert nodes >= 7 and flags > 0 and invalid >= 6 * nodes


def test_validity_flags_hessian_gain_categorical_order():
    rng = np.random.default_rng(5)
    n = 30000
    ds, bins, cols = dataset(rng, n, LAYOUT)
    cfg = ydf_b200.default_config(loss=0, use_hessian_gain=1, max_depth=6, min_examples=50, candidate_shuffle=0)
    gbt = ydf_b200.Gbt(ds, cfg)
    y = labels_for(rng, bins, cfg)
    gbt.set_labels(y)
    gbt.set_candidate_sampling(-1, 0.5)
    gbt.capture_candidates(True)
    m = (bins[0] / 64.0 + 0.05 * bins[4] + rng.normal(size=n))
    g = (0.9 * m / np.abs(m).max()).astype(np.float32)
    h = rng.uniform(0.01, 0.25, size=n).astype(np.float32)
    tree = gbt.train_tree_on_gradients(g, h)
    nodes, flags, _ = check_levels(gbt, cfg, tree, 0, k_valid(cfg, ds.n_features, -1, 0.5), cols, g, h)
    assert nodes >= 7 and flags > 0


def test_validity_flags_wide_and_presorted_columns():
    rng = np.random.default_rng(9)
    n = 40000
    ds, bins, cols = dataset(rng, n, [("num", 64), ("cat", 9), ("num", 1), ("cat", 1), ("num", 1), ("num", 32)])
    # feature 2: a wide numerical column of 600 buckets, 3: a wide categorical one of 300, 4: a presorted float column
    wn = np.minimum(rng.geometric(0.01, size=n) - 1, 599).astype(np.uint16)
    ds.set_wide_column(2, wn, 600, 0, np.arange(600, dtype=np.float32), 0.0)
    wc = rng.integers(0, 300, size=n).astype(np.uint16)
    ds.set_wide_categorical_column(3, wc, 300, 0)
    pv = np.round(rng.normal(size=n), 2).astype(np.float32)
    ds.set_numerical_column(4, pv, float(pv.mean()))
    cols[2] = ("wide_num", wn, 600, None)
    cols[3] = ("wide_cat", wc, 300, None)
    cols[4] = ("pre", pv, 0, None)
    cfg = ydf_b200.default_config(loss=1, max_depth=6, min_examples=1, candidate_shuffle=0)
    gbt = ydf_b200.Gbt(ds, cfg)
    g = (bins[0] / 64.0 + (wn > 50) + 0.5 * (wc % 3 == 0) + pv + rng.normal(scale=0.5, size=n)).astype(np.float32)
    gbt.set_labels(g)
    gbt.set_candidate_sampling(2, None)
    gbt.capture_candidates(True)
    tree = gbt.train_tree_on_gradients(g)
    used = set(tree["feature"][tree["feature"] >= 0].tolist())
    assert used & {2, 3, 4}
    nodes, flags, _ = check_levels(gbt, cfg, tree, 0, k_valid(cfg, ds.n_features, 2), cols, g)
    assert nodes >= 7 and flags > 0


def _tree_hashes(gbt):
    return [gbt.get_tree(i).tobytes() for i in range(gbt.num_trees())]


@pytest.mark.parametrize("num, ratio", [(-1, None), (-1, 1.0), (13, None), (40, None)])
def test_every_feature_is_the_unsampled_training(num, ratio):
    """k >= F keeps the unsampled training, the tie-break replay included: feature 12 is a twin of feature 0, so the
    trees hold ties that the replay resolves."""
    rng = np.random.default_rng(3)
    bins, nb, ft = mixed_bins(rng, 20000, LAYOUT)
    bins, nb, ft = np.concatenate([bins, bins[:1]]), np.append(nb, nb[0]), np.append(ft, ft[0])
    ds = ydf_b200.Dataset(bins, nb, np.zeros(len(nb), np.int32), feature_types=ft)
    out, ties = [], []
    for sample in (False, True):
        cfg = ydf_b200.default_config(loss=0, max_depth=5, num_trees=5, candidate_shuffle=2)
        gbt = ydf_b200.Gbt(ds, cfg)
        gbt.set_labels(labels_for(np.random.default_rng(4), bins, cfg))
        if sample:
            gbt.set_candidate_sampling(num, ratio)
        gbt.train(5)
        out.append(_tree_hashes(gbt))
        ties.append(gbt.tie_stats())
    assert out[0] == out[1]
    assert ties[0] == ties[1] and sum(ties[0]) > 0, ties


def test_validity_flags_with_zero_example_weights():
    """Rows of weight 0: a boundary with rows but no weight on one side still counts as tried (the reference's
    IsValidSplit is always true for these accumulators), though it is never a split.  Feature 2 is binary and its bucket 0
    carries every zero weight."""
    rng = np.random.default_rng(23)
    n = 20000
    ds, bins, cols = dataset(rng, n, LAYOUT, constant=2)
    cfg = ydf_b200.default_config(loss=1, max_depth=6, min_examples=1, candidate_shuffle=0, split_jobs_draw_seeds=1)
    gbt = ydf_b200.Gbt(ds, cfg)
    w = np.where(bins[2] == 0, 0.0, rng.uniform(0.5, 2.0, size=n)).astype(np.float32)
    gbt.set_weights(w)
    gbt.set_labels(labels_for(rng, bins, cfg))
    gbt.set_candidate_sampling(3, None)
    gbt.capture_candidates(True)
    gbt.train(2)
    last = gbt.num_trees() - 1
    tree = gbt.get_tree(last)
    nodes, flags, _ = check_levels(gbt, cfg, tree, last, k_valid(cfg, ds.n_features, 3), cols)
    assert nodes >= 7 and flags > 0
    assert gbt.level_tried(0)[0][0, 2] == 1 and not gbt.level_candidates(0)["found"][0, 2]


def test_sampling_changes_the_trees_and_works_with_best_first_growth_and_validation():
    rng = np.random.default_rng(8)
    ds, bins, _ = dataset(rng, 30000, LAYOUT)
    vds, vbins, _ = dataset(np.random.default_rng(8), 5000, LAYOUT)
    hashes = []
    for strategy, num in ((0, -1), (0, 2), (1, -1), (1, 2)):
        cfg = ydf_b200.default_config(loss=0, max_depth=6, num_trees=30, growing_strategy=strategy, candidate_shuffle=0,
                                      early_stopping=2, early_stopping_num_trees_look_ahead=5,
                                      early_stopping_initial_iteration=2)
        gbt = ydf_b200.Gbt(ds, cfg)
        gbt.set_labels(labels_for(np.random.default_rng(4), bins, cfg))
        gbt.set_validation(vds, labels_for(np.random.default_rng(4), vbins, cfg))
        gbt.set_candidate_sampling(num, None)
        gbt.train(30)
        assert gbt.num_trees() >= 1
        hashes.append(_tree_hashes(gbt))
    assert hashes[0] != hashes[1] and hashes[2] != hashes[3]


def test_refusals():
    rng = np.random.default_rng(2)
    ds, bins, _ = dataset(rng, 5000, LAYOUT)
    F = ds.n_features

    def handle(**kw):
        cfg = ydf_b200.default_config(**{"loss": 1, "max_depth": 4, "num_trees": 2, "candidate_shuffle": 0, **kw})
        gbt = ydf_b200.Gbt(ds, cfg)
        gbt.set_labels(bins[0].astype(np.float32))
        return gbt

    def code(fn):
        with pytest.raises(ydf_b200.YggError) as e:
            fn()
        return e.value.code

    assert code(lambda: handle(candidate_shuffle=2).set_candidate_sampling(3)) == 1
    handle(candidate_shuffle=2).set_candidate_sampling(F)          # k >= F: nothing to refuse
    assert code(lambda: handle().set_candidate_sampling(-2)) == 1
    assert code(lambda: handle().set_candidate_sampling(-1, 1.5)) == 1
    g = handle()
    g.train(1)
    assert code(lambda: g.set_candidate_sampling(3)) == 1
    g = handle()
    g.set_candidate_sampling(3)
    assert code(lambda: g.set_feature_shard(0, F - 1, 0, 1)) == 4
    g = handle()
    g.set_feature_shard(0, F - 1, 0, 1)
    assert code(lambda: g.set_candidate_sampling(3)) == 4
    g = handle()
    with pytest.raises(ydf_b200.YggError) as e:
        g.level_tried(0)
    assert e.value.code == 1


def test_learner_passes_the_sampling_arguments():
    rng = np.random.default_rng(0)
    n = 4000
    cols = {f"x{i}": rng.normal(size=n).astype(np.float32) for i in range(8)}
    cols["y"] = (cols["x0"] + cols["x1"] > 0).astype(np.int64)
    kw = dict(num_trees=5, discretize_numerical_columns=True)
    m = ydf_b200.GradientBoostedTreesLearner("y", num_candidate_attributes_ratio=0.25, **kw).train(cols)
    assert m.config["num_candidate_attributes_ratio"] == 0.25 and m.config["num_candidate_attributes"] == -1
    assert m.config["candidate_shuffle"] == 0   # the keys order the candidates
    full = ydf_b200.GradientBoostedTreesLearner("y", **kw).train(cols)
    assert full.config["candidate_shuffle"] == 2 and full.config["num_candidate_attributes_ratio"] is None
    every = ydf_b200.GradientBoostedTreesLearner("y", num_candidate_attributes=8, **kw).train(cols)
    assert every.config["candidate_shuffle"] == 2   # k >= F: unsampled, with the tie-break replay
