"""DART on the device against the exact restatement of tests/dart_ref.py, driven by the device's own trees.

Per iteration: the dropped set equals the draws restated on the learner's mt19937; every node of the tree equals the integer
sums of the gradients taken at the sampled predictions (tests/boost_ref.py's node checks); the training accumulator
(get_predictions) and the weights equal the reference bit for bit; the training and held-out losses are those of the
reference's accumulators (accuracy exactly, losses within 1 ulp).  The model (predict) is the scaled sum, bit for bit.
"""
import numpy as np
import pytest

import ydf_b200
from oracle import oracle as O
from tests import boost_ref as R
from tests import dart_ref as D
from tests.test_gpu_boosting_exact import LAYOUT, Table, check_losses, labels_for

pytestmark = pytest.mark.gpu

F32 = np.float32


def gradients(loss, s, labels):
    """(g, h, g_alt, h_alt) [K, n] at the sampled predictions `s` [K, n]."""
    if loss == 2:
        cls = labels - 1
        g, h, amb = R.mc_gradients(s, cls)
        g_alt, h_alt, _ = R.mc_gradients(s, cls, flip=amb)
        return g, h, g_alt, h_alt
    if loss == 0:
        pos = labels == 2
        g, h, _ = R.binomial_gradients(s[0], pos)
        g_alt, h_alt, _ = R.binomial_gradients(s[0], pos, alt=True)
        return g[None], h[None], g_alt[None], h_alt[None]
    g, h, _ = R.squared_error_gradients(s[0], labels)
    return g[None], h[None], g[None], h[None]


def check_dart_run(gbt, cfg, table, labels, rate, iters, vlabels=None, weights=None, vweights=None, on_tree=None):
    """`cfg.candidate_shuffle` 1 / 2 takes trees of depth 2 (max_depth = 2): exactly one candidate shuffle per tree, at
    its root, which the restatement replays on the learner's stream after the iteration's DART and row draws.
    vweights: the held-out rows' weights.  on_tree(t, rows): called after each tree's checks, before the next step(),
    with the per-row quantities the tree was trained on (dict g, h, g_alt, h_alt, sel, w, tree, as check_run hands
    them out), taken at the sampled predictions."""
    n = table.n
    shuffle = int(cfg.candidate_shuffle)
    assert shuffle == 0 or int(cfg.max_depth) == 2
    loss = int(cfg.loss)
    K = int(cfg.num_classes) if loss == 2 else 1
    logit = loss in (0, 2)
    goss = cfg.goss_alpha > 0 or cfg.goss_beta > 0
    sub = cfg.subsample < 1.0
    weighted = weights is not None or goss
    labels = np.asarray(labels)
    init = F32(gbt.initial_prediction())
    acc = D.Accumulator(np.full((K, n), init, F32))
    vacc = D.Accumulator(np.full((K, table.n_valid), init, F32)) if vlabels is not None else None
    rng = O.Rng(int(cfg.random_seed))
    rng.discard(int(cfg.rng_words_consumed))
    if weights is not None:
        w_pow2 = R.pow2_cover(np.max(weights))
    elif goss:
        amp = float((F32(1) - F32(cfg.goss_alpha)) / F32(cfg.goss_beta)) if cfg.goss_beta > 0 else 1.0
        w_pow2 = 1.0
        while w_pow2 < amp:
            w_pow2 *= 2.0
    else:
        w_pow2 = None
    wide_cat = any(c[0] == "wide_cat" for c in table.cols)
    errs, dropped_sets, leaves = [], [], []
    for it in range(iters):
        gbt.step()
        got_acc = gbt.get_predictions()
        dropped = D.draw_dropped(rng.next, it, rate, libcxx=shuffle == 2)
        got_dropped = gbt.dart_dropped(it).tolist()
        if got_dropped != dropped:
            errs.append(f"iteration {it}: dropped {got_dropped} != {dropped}")
            dropped = got_dropped
        dropped_sets.append(dropped)
        s = acc.sampled(dropped)
        g, h, g_alt, h_alt = gradients(loss, s, labels)
        sel, w = None, weights
        if goss:
            sel, w = R.goss_selection(g[0], cfg.goss_alpha, cfg.goss_beta, rng)
        elif sub:
            sel = R.subsample_mask(rng, n, cfg.subsample)
        p_new = np.zeros((K, n), F32)
        vp_new = np.zeros((K, table.n_valid), F32) if vacc is not None else None
        for k in range(K):
            t = it * K + k
            tree = gbt.get_tree(t)
            sets = gbt.get_category_sets(t, tree) if wide_cat else {}
            if weighted:
                gk, hk, g2w = R.weigh(g[k], h[k], w, unit_hessian=not logit)
                gk_alt, hk_alt, g2w_alt = R.weigh(g_alt[k], h_alt[k], w, unit_hessian=not logit)
            else:
                gk, hk, gk_alt, hk_alt, g2w, g2w_alt = g[k], h[k], g_alt[k], h_alt[k], None, None
            P = 1.0 if (logit and not weighted) else R.pow2_cover(np.abs(gk).max())
            h_pow2 = (0.25 if logit else 1.0) * (w_pow2 if weighted else 1.0)
            has_h = logit or weighted
            rows = R.Rows(gk, hk if has_h else None, sel, P, h_pow2, g_alt=gk_alt, h_alt=hk_alt if has_h else None,
                          w=w if weighted else None, w_pow2=w_pow2, g2w=g2w, g2w_alt=g2w_alt)
            rows_of = R.route(tree, table.cols, sets)
            errs += R.check_tree(tree, rows_of, rows, cfg, logit, where=f"tree {t}")
            if on_tree is not None:
                on_tree(t, dict(g=gk, h=hk if has_h else None, g_alt=gk_alt, h_alt=hk_alt if has_h else None, sel=sel,
                                w=w if weighted else None, tree=tree))
            if shuffle == 1:
                rng.shuffle(len(table.cols))
            elif shuffle == 2:
                rng.shuffle_libcxx(len(table.cols))
            if shuffle and cfg.split_jobs_draw_seeds:
                rng.discard(len(table.cols))
            p_new[k] = tree["leaf_value"][R.leaf_of_rows(tree, rows_of, n)]
            leaves.append(p_new[k].copy())
            if vacc is not None:
                vrows = R.route(tree, table.vcols, sets)
                vp_new[k] = tree["leaf_value"][R.leaf_of_rows(tree, vrows, table.n_valid)]
        acc.update(p_new, dropped)
        if vacc is not None:
            vacc.update(vp_new, dropped)
        got = got_acc[None] if K == 1 else got_acc.T
        if not np.array_equal(got, acc.acc):
            errs.append(f"iteration {it}: accumulator differs in {int((got != acc.acc).sum())} values")
        got_w = gbt.dart_weights()
        if not np.array_equal(got_w, acc.weights()):
            errs.append(f"iteration {it}: weights {got_w.tolist()} != {acc.weights().tolist()}")
        errs += check_losses(gbt.train_loss(it), loss, acc.acc, labels, weights,
                             w_pow2 if weights is not None else None, f"train loss {it}")
        if vacc is not None:
            vw_pow2 = R.pow2_cover(np.max(vweights)) if vweights is not None else None
            errs += check_losses(gbt.validation_loss(it), loss, vacc.acc, np.asarray(vlabels), vweights, vw_pow2,
                                 f"validation loss {it}")
    # the model: every leaf of iteration j scaled by w_j, summed in tree order
    want = D.scaled_sum(init, np.stack(leaves), acc.weights(), K)
    p = gbt.predict(table.ds)
    p = p[None] if K == 1 else p.T
    if not np.array_equal(p, want):
        errs.append(f"predict differs from the scaled model in {int((p != want).sum())} values")
    assert not errs, f"{len(errs)} mismatches:\n" + "\n".join(errs[:30])
    assert np.allclose(acc.acc, want, rtol=1e-4, atol=1e-4)   # the same model, summed in another order
    return dropped_sets


CASES = {
    "binomial_r0.1": dict(n=20000, rate=0.1, cfg=dict(loss=0), valid=2000),
    "binomial_hessian_r0.5": dict(n=20000, rate=0.5, cfg=dict(loss=0, use_hessian_gain=1), valid=2000),
    "squared_error_r0": dict(n=15000, rate=0.0, cfg=dict(loss=1), scale=3.0, valid=1500),
    "squared_error_r1": dict(n=15000, rate=1.0, cfg=dict(loss=1, shrinkage=1.0), scale=3.0),
    "multinomial_k3_r0.5": dict(n=9000, rate=0.5, cfg=dict(loss=2, num_classes=3), K=3, valid=1000),
    "multinomial_k3_hessian_r0.1": dict(n=9000, rate=0.1, cfg=dict(loss=2, num_classes=3, use_hessian_gain=1), K=3),
    "weighted_squared_error_r0.5": dict(n=15000, rate=0.5, cfg=dict(loss=1), scale=3.0, weights=True),
    "subsample_binomial_r0.5": dict(n=20000, rate=0.5, cfg=dict(loss=0, subsample=0.5), valid=1000),
    "goss_binomial_r0.5": dict(n=20000, rate=0.5, cfg=dict(loss=0, goss_alpha=0.2, goss_beta=0.1)),
    "best_first_r0.5": dict(n=20000, rate=0.5, cfg=dict(loss=0, growing_strategy=1, max_num_nodes=6, max_depth=7), valid=1000),
    "candidate_sampling_r0.5": dict(n=20000, rate=0.5, cfg=dict(loss=1), scale=2.0, sample_k=2),
    # the tie-break replay's stream: libc++ mode (its uniform_int fallback at rate 0) and libstdc++ mode
    "binomial_shuffle_libcxx_r0": dict(n=12000, rate=0.0, cfg=dict(loss=0, max_depth=2, candidate_shuffle=2), valid=1000),
    "squared_error_shuffle_libcxx_r0.5": dict(n=12000, rate=0.5, cfg=dict(loss=1, max_depth=2, candidate_shuffle=2), scale=2.0),
    "multinomial_k3_shuffle_libstdcxx_r0.5": dict(n=9000, rate=0.5, cfg=dict(loss=2, num_classes=3, max_depth=2,
                                                                          candidate_shuffle=1), K=3, valid=1000),
    "wide_presorted_r0.5": dict(n=20000, rate=0.5, cfg=dict(loss=1, max_depth=5), scale=3.0, valid=2000,
                                extra={1: ("wide_cat", 700), 2: ("wide_num", 4096), 4: ("pre", 0)}),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_dart_iterations_match_the_reference(case):
    c = CASES[case]
    rng = np.random.default_rng(sorted(CASES).index(case) + 2024)
    K = c.get("K", 3)
    table = Table(rng, c["n"], c.get("valid", 0), LAYOUT, c.get("extra"))
    cfg = ydf_b200.default_config(**{"max_depth": 6, "num_trees": 10, **c["cfg"]})
    y = labels_for(cfg.loss, table.margin(rng, c.get("scale", 1.0)), K)
    ytr, yv = y[:table.n], (y[table.n:] if table.n_valid else None)
    gbt = ydf_b200.Gbt(table.ds, cfg)
    if c.get("sample_k"):
        gbt.set_candidate_sampling(c["sample_k"])
    gbt.set_dart(c["rate"])
    w = None
    if c.get("weights"):
        w = rng.uniform(0.1, 3.0, size=table.n).astype(F32)
        gbt.set_weights(w)
    gbt.set_labels(ytr)
    if yv is not None:
        gbt.set_validation(table.vds, yv)
    dropped = check_dart_run(gbt, cfg, table, ytr, c["rate"], iters=8, vlabels=yv, weights=w)
    if c["rate"] == 1.0:
        assert all(d == list(range(i)) for i, d in enumerate(dropped))
    if c["rate"] == 0.0:
        assert all(len(d) == 1 for d in dropped[1:])


@pytest.mark.parametrize("policy", [0, 1, 2])
def test_dart_early_stopping_keeps_the_weights_at_the_stop(policy):
    """NONE (held-out rows only logged) / MIN_LOSS_FINAL / LOSS_INCREASE: the model keeps every tree / the best prefix,
    scaled by the weights after the last iteration trained (the stop), replayed from the dropped sets; trees trained past
    the stop do not count."""
    rng = np.random.default_rng(77 + policy)
    table = Table(rng, 12000, 3000, LAYOUT)
    cfg = ydf_b200.default_config(max_depth=6, num_trees=60, loss=0, shrinkage=0.5, early_stopping=policy,
                                  early_stopping_num_trees_look_ahead=4, early_stopping_initial_iteration=2)
    y = labels_for(0, table.margin(rng, 0.3), 3)
    gbt = ydf_b200.Gbt(table.ds, cfg)
    gbt.set_dart(0.3)
    gbt.set_labels(y[:table.n])
    gbt.set_validation(table.vds, y[table.n:])
    gbt.train(60)
    trained, kept = gbt.num_iterations(), gbt.num_trees()
    assert kept <= trained <= 60
    if policy == 0:
        assert trained == kept == 60
    if policy == 2:
        assert trained < 60, "the held-out loss should rise on this noisy table"
    want_w = D.weights_after([gbt.dart_dropped(i).tolist() for i in range(trained)])[:kept]
    assert np.array_equal(gbt.dart_weights(), want_w)
    init = F32(gbt.initial_prediction())
    leaves = []
    for t in range(kept):
        tree = gbt.get_tree(t)
        leaves.append(tree["leaf_value"][R.leaf_of_rows(tree, R.route(tree, table.vcols), table.n_valid)])
    want = D.scaled_sum(init, np.stack(leaves) if leaves else np.zeros((0, table.n_valid), F32), want_w)[0]
    assert np.array_equal(gbt.predict(table.vds), want)


def test_dart_learner_end_to_end(tmp_path):
    rng = np.random.default_rng(5)
    n = 6000
    x = rng.normal(size=(4, n)).astype(F32)
    y = np.where(x[0] + 0.5 * x[1] * x[2] + rng.normal(scale=0.5, size=n) > 0, "a", "b")
    cols = {f"f{i}": x[i] for i in range(4)}
    cols["y"] = y
    learner = ydf_b200.GradientBoostedTreesLearner("y", forest_extraction="DART", dart_dropout=0.1, num_trees=40,
                                                   discretize_numerical_columns=True)
    model = learner.train(cols)
    assert model.config["forest_extraction"] == "DART" and model.config["dart_dropout"] == pytest.approx(0.1)
    ev = model.evaluate(cols)
    assert ev["accuracy"] > 0.75, ev
    # the saved model holds the scaled trees: read back, it predicts what the learner's model predicts
    model.save(str(tmp_path / "m"))
    back = ydf_b200.model_io.read_ydf_model(str(tmp_path / "m"))
    raw = ydf_b200.model_io.predict_ydf_model(back, {k: v for k, v in cols.items() if k != "y"})
    p = model.predict(cols)
    assert np.allclose(1.0 / (1.0 + np.exp(-np.asarray(raw, np.float64))), p, atol=1e-5)
    mart = ydf_b200.GradientBoostedTreesLearner("y", num_trees=40, discretize_numerical_columns=True).train(cols)
    assert mart.config["forest_extraction"] == "MART" and mart.config["dart_dropout"] is None


def test_dart_refusals():
    rng = np.random.default_rng(9)
    table = Table(rng, 3000, 0, LAYOUT)
    y = labels_for(0, table.margin(rng), 3)
    cfg = ydf_b200.default_config(max_depth=4, num_trees=5, loss=0)
    gbt = ydf_b200.Gbt(table.ds, cfg)
    for bad in (float("nan"), -0.1, 1.5):
        with pytest.raises(ydf_b200.YggError):
            gbt.set_dart(bad)
    gbt.set_dart(0.2)
    gbt.set_labels(y)
    with pytest.raises(ydf_b200.YggError, match="sharding"):
        gbt.set_feature_shard(0, 2, 0, 1)
    with pytest.raises(ydf_b200.YggError, match="sharding"):
        gbt.set_row_shard(0, 1, table.n, 0.0)
    with pytest.raises(ydf_b200.YggError, match="set_predictions"):
        gbt.set_predictions(np.zeros(table.n, F32))
    gbt.step()
    with pytest.raises(ydf_b200.YggError, match="before training"):
        gbt.set_dart(0.2)
    # a shard set first refuses DART
    other = ydf_b200.Gbt(table.ds, cfg)
    other.set_feature_shard(0, 2, 0, 1)
    with pytest.raises(ydf_b200.YggError, match="sharding"):
        other.set_dart(0.2)


def test_dart_save_ydf_writes_the_scaled_model(tmp_path):
    """ygg_gbt_save_ydf: every leaf of iteration j holds fl(leaf * w_j), internal nodes their unscaled values, and the
    directory equals the learner's model trained on the same rows (its scaled trees written by model_io)."""
    import ctypes as C
    from ydf_b200 import _capi, model_io
    rng = np.random.default_rng(11)
    n = 5000
    x = rng.normal(size=(3, n)).astype(F32)
    cols = {f"f{i}": x[i] for i in range(3)}
    cols["y"] = np.where(x[0] - x[1] * x[2] + rng.normal(scale=0.7, size=n) > 0, "p", "q")
    kw = dict(forest_extraction="DART", dart_dropout=0.3, num_trees=12, validation_ratio=0.0,
              discretize_numerical_columns=True, num_threads=1)
    learner = ydf_b200.GradientBoostedTreesLearner("y", **kw)
    spec, dataset = learner._build_dataset(cols)
    gbt = ydf_b200.Gbt(dataset, learner.cfg)
    try:
        gbt.set_dart(0.3)
        gbt.set_labels(learner._labels(cols, spec))
        gbt.train(12)
        trees = [gbt.get_tree(t) for t in range(gbt.num_trees())]
        w = gbt.dart_weights()
        pb, label_idx, feat_idx = model_io.encode_data_spec(spec)
        fidx = np.asarray(feat_idx, np.int32)
        _capi.check(_capi.lib().ygg_gbt_save_ydf(gbt.handle, str(tmp_path / "c").encode(), b"y", pb, C.c_int64(len(pb)),
                                                 C.c_int32(label_idx), _capi.ptr(fidx, C.c_int32)))
    finally:
        gbt.close()
        dataset.close()
    saved = model_io.read_ydf_model(str(tmp_path / "c"))
    assert saved["num_trees"] == len(trees) == 12 and len(w) == 12
    flat = np.concatenate(trees)
    scale = np.concatenate([np.full(len(t), w[i], F32) for i, t in enumerate(trees)])
    leaf = flat["feature"] < 0
    want = np.where(leaf, (flat["leaf_value"] * scale).astype(F32), flat["leaf_value"])
    got = np.array([nd["top_value"] for nd in saved["nodes"]], F32)
    assert np.array_equal(got, want)
    assert not np.array_equal(flat["leaf_value"][leaf], want[leaf])   # the scaling did something
    model = ydf_b200.GradientBoostedTreesLearner("y", **kw).train(cols)
    model.save(str(tmp_path / "m"))
    mine = model_io.read_ydf_model(str(tmp_path / "m"))
    assert np.array_equal(np.array([nd["top_value"] for nd in mine["nodes"]], F32), got)


def _cxx_fold(z, name, fold):
    """A fold of tests/golden/dart_cxx_test_folds.npz as raw columns: floats, category strings ("" = missing), labels."""
    cols = {}
    numerical = set(z[f"{name}_numerical"].tolist())
    label = {"iris": "class", "adult": "income"}[name]
    for c in z[f"{name}_features"].tolist() + [label]:
        v = z[f"{name}_{fold}_{c}"]
        if c in numerical or c == label:
            cols[c] = v
        else:
            voc = np.append(z[f"{name}_vocabulary_{c}"], "")
            cols[c] = voc[np.minimum(v.astype(np.int64), len(voc) - 1)]
    return cols, label


@pytest.mark.parametrize("name,window,golden", [
    ("iris", ((0.9467, 0.04), (0.1925, 0.1226)), (0.9733, 0.2019)),
    ("adult", ((0.8459, 0.0449), (0.3293, 0.0727)), None),
])
def test_dart_reference_acceptance_runs(name, window, golden):
    """GradientBoostedTreesOnIris.Dart (gradient_boosted_trees_test.cc:1774-1784) and GradientBoostedTreesOnAdult.Dart
    (:1458-1473) on the engine through the learner: the tester's folds at dataset_sampling 1.0, 100 trees, dropout 0.1,
    shrinkage 1.0 (the C++ learner's DART default), num_candidate_attributes 8 (every feature of Iris's 4; a sample of
    Adult's 14), the exact numerical splitter, one thread, libc++ tie-break, default hold-out and early stopping.
    Accuracy and log loss on the test fold must land in the reference's windows; the distance to Iris's golden values is
    printed.  The oracle's DART loop hits Iris's golden values within 1e-4 (tests/test_reference_replay.py) and the engine
    follows that loop tree for tree on noisy tables (test_dart_training_matches_the_oracle_loop); on Iris the engine
    stays in the window only, because the reference splits pure nodes on the rounding noise of its double sums (scores
    near 1e-17, DESIGN.md §6) and the engine's exact sums do not.  Those nodes draw candidate shuffles from the learner's
    engine, so DART's dropped sets, which come from the same stream, part from the reference's at iteration 3."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dart_cxx_test_folds.npz"))
    train, label = _cxx_fold(z, name, "train")
    test, _ = _cxx_fold(z, name, "test")
    learner = ydf_b200.GradientBoostedTreesLearner(
        label, forest_extraction="DART", dart_dropout=0.1, shrinkage=1.0, num_trees=100, num_candidate_attributes=8,
        num_threads=1, max_exact_numerical_values=65535, presort_numerical_columns=True, max_vocab_count=2000,
        categorical_arity_limit_for_random=1000)
    model = learner.train(train)
    ev = model.evaluate(test)
    acc, ll = ev["accuracy"], ev["loss"]
    print(f"{name} DART: accuracy {acc:.4f} log loss {ll:.4f} trees {model.num_trees()}"
          + (f"; golden distance {acc - golden[0]:+.4f} / {ll - golden[1]:+.4f}" if golden else ""))
    (a_mid, a_w), (l_mid, l_w) = window
    assert abs(acc - a_mid) <= a_w, (acc, window)
    assert abs(ll - l_mid) <= l_w, (ll, window)


def _leaf_nodes(tree, bins):
    """The leaf node id every column of `bins` ([F, n] bucket / dictionary codes) reaches in `tree`."""
    n = bins.shape[1]
    rows = np.arange(n)
    node = np.zeros(n, np.int64)
    while True:
        f = tree["feature"][node]
        act = np.nonzero(f >= 0)[0]
        if len(act) == 0:
            return node
        nd = node[act]
        v = bins[f[act], rows[act]].astype(np.int64)
        in_set = ((tree["cat_mask"][nd, v >> 5] >> (v & 31).astype(np.uint32)) & 1) != 0
        go = np.where(tree["condition_type"][nd] == 1, in_set, v >= tree["threshold_bin"][nd])
        node[act] = np.where(go, tree["pos_child"][nd], tree["neg_child"][nd])


# loss (0 binomial, 1 squared error, 2 multinomial K = 3), dropout rate, early_stopping (0 NONE, 1 MIN_LOSS_FINAL,
# 2 LOSS_INCREASE), candidate shuffle (0 none, 1 libstdc++, 2 libc++), rows, iterations, extra configuration
ORACLE_CASES = {
    "binomial_r0.1_none": (0, 0.1, 0, 0, 12000, 40, {}),
    "binomial_r0.5_min_loss_final": (0, 0.5, 1, 0, 12000, 40, {}),
    "binomial_r0_loss_increase_libcxx": (0, 0.0, 2, 2, 8000, 60, dict(max_depth=4)),
    # these two stop after 31 and 9 iterations: the engine reads the losses back 8 iterations at a time, past the stop
    "binomial_subsample_r0.5_loss_increase": (0, 0.5, 2, 0, 20000, 60, dict(subsample=0.5, stop_off_8=True)),
    "binomial_hessian_r0.1_min_loss_final": (0, 0.1, 1, 0, 12000, 40, dict(use_hessian_gain=1)),
    "squared_error_r0.1_loss_increase": (1, 0.1, 2, 0, 12000, 60, {}),
    "squared_error_r1_none": (1, 1.0, 0, 0, 10000, 30, {}),
    "squared_error_r0.5_min_loss_final_libstdcxx": (1, 0.5, 1, 1, 10000, 40, dict(max_depth=5)),
    "squared_error_r0_loss_increase_libstdcxx": (1, 0.0, 2, 1, 6000, 60, dict(max_depth=4)),
    "multinomial_k3_r0.1_loss_increase": (2, 0.1, 2, 0, 9000, 40, dict(min_examples=20, stop_off_8=True)),
    "multinomial_k3_r0.5_none_libcxx": (2, 0.5, 0, 2, 9000, 30, dict(max_depth=5, min_examples=20)),
    "multinomial_k3_r0_min_loss_final": (2, 0.0, 1, 0, 6000, 30, dict(min_examples=20)),
}


@pytest.mark.parametrize("case", sorted(ORACLE_CASES))
def test_dart_training_matches_the_oracle_loop(case):
    """The engine's whole DART run against the oracle's DART loop (oracle_gbt_train_validated with oracle.set_dart), which
    is pinned on the reference's Iris DART golden (tests/test_reference_replay.py): the same hold-out, every kept tree,
    every iteration's dropped set, the model's weights bit for bit, the number of iterations and trees, the training and
    validation losses, the final validation loss, and the scaled model's raw scores on the held-out rows bit for bit.
    This checks the engine's draws, sampled gradients, update, early stopping and scaling against a restatement that does
    not share the engine's code; the first iteration whose dropped set differs is named."""
    from tests.test_gpu_validation import _noisy, _oracle_cfg
    from tests.util import compare_trees, synth_mixed
    loss, rate, policy, shuffle, n, iters, extra = ORACLE_CASES[case]
    bins, nb, na, ft, y = _noisy(n, sorted(ORACLE_CASES).index(case) + 40, "regression" if loss == 1 else "binary")
    K = 3 if loss == 2 else 1
    if loss == 2:
        # numerical features only (the K planes' sums near-tie categorical bucket orders); a class that follows two
        # features, replaced by a uniform draw on half of the rows: no pure node of 20 rows
        bins, nb, na, ft, _ = synth_mixed(n, 6, [], seed=n + 1)
        y = ((bins[0].astype(np.int64) // 7 + bins[1]) % 3 + 1).astype(np.int32)
        r = np.random.default_rng(n)
        y = np.where(r.random(n) < 0.5, r.integers(1, 4, size=n), y).astype(np.int32)
    kw = dict(loss=loss, num_classes=K if loss == 2 else 0, num_trees=iters, max_depth=6, shrinkage=0.3, min_examples=2,
              early_stopping=policy, early_stopping_num_trees_look_ahead=12, early_stopping_initial_iteration=4,
              candidate_shuffle=shuffle, rng_words_consumed=n, split_jobs_draw_seeds=1)
    kw.update(extra)
    stop_off_8 = kw.pop("stop_off_8", False)
    cfg = ydf_b200.default_config(**kw)
    O.set_stable_category_sort(True)
    O.set_validated_shuffle_mode(shuffle)
    O.set_dart(rate)
    try:
        # the concurrent manager (equal float scores: the first candidate), one seed per feature job after each shuffle
        ref = O.gbt_train_validated(bins, nb, na, y, _oracle_cfg(cfg), 0.2, num_threads=4, feature_type=ft)
    finally:
        O.set_dart(None)
        O.set_validated_shuffle_mode(O.SHUFFLE_NONE)
        O.set_stable_category_sort(False)
    full = ydf_b200.Dataset(bins, nb, na, feature_types=ft)
    m = ydf_b200.validation_split_mask(cfg.random_seed, n, 0.2)
    np.testing.assert_array_equal(m, ref["in_training"])
    tr, va = full.split_rows(m)
    gbt = ydf_b200.Gbt(tr, cfg)
    gbt.set_dart(rate)
    gbt.set_labels(y[m])
    gbt.set_validation(va, y[~m])
    gbt.train(iters)
    trained, kept = gbt.num_iterations(), gbt.num_trees()
    print(f"{case}: {trained} iterations trained, {kept // K} kept; oracle {ref['num_entries']}, {len(ref['trees']) // K}")
    for i in range(min(trained, ref["num_entries"])):
        got = gbt.dart_dropped(i).tolist()
        assert got == ref["dart_dropped"][i], f"iteration {i}: dropped {got} != oracle {ref['dart_dropped'][i]}"
    for t in range(min(kept, len(ref["trees"]))):
        tree = gbt.get_tree(t)
        errs = compare_trees(tree, ref["trees"][t])
        if errs and len(tree) == len(ref["trees"][t]):
            bad = sorted({int(e.split(":")[0].split()[1]) for e in errs if e.startswith("node ")})
            errs += [f"node {b}: split scores {tree['split_score'][b]} / {ref['trees'][t]['split_score'][b]}" for b in bad[:3]]
        assert not errs, (f"tree {t} (iteration {t // K})", errs[:8])
    for i in range(min(trained, ref["num_entries"])):
        tl, _ = gbt.train_loss(i)
        vl, vs = gbt.validation_loss(i)
        assert abs(tl - ref["train_loss"][i]) <= 1e-5 * abs(ref["train_loss"][i]), (i, tl, ref["train_loss"][i])
        assert abs(vl - ref["valid_loss"][i]) <= 1e-5 * abs(ref["valid_loss"][i]), (i, vl, ref["valid_loss"][i])
        assert abs(vs - ref["valid_secondary"][i]) <= 1e-5 * max(1.0, abs(ref["valid_secondary"][i]))
    assert trained == ref["num_entries"] and kept == len(ref["trees"])
    if policy == 0:
        assert trained == iters and kept == iters * K
    if stop_off_8:
        assert trained < iters and trained % 8 != 0, trained
    w = gbt.dart_weights()
    assert np.array_equal(w, ref["dart_weights"]), (w, ref["dart_weights"])
    fv, trig = gbt.final_validation()
    assert trig == ref["early_stopping_triggered"]
    assert abs(fv - ref["validation_loss"]) <= 1e-5 * abs(ref["validation_loss"]), (fv, ref["validation_loss"])
    # the scaled model on the held-out rows: init + fl(leaf * w_{t // K}) in tree order, per class plane, with the
    # oracle's weights; bit for bit on the engine's leaf values (equal to the oracle's within compare_trees' 1e-5)
    vbins = bins[:, ~m]
    nodes = [_leaf_nodes(ref["trees"][t], vbins) for t in range(len(ref["trees"]))]
    init = F32(gbt.initial_prediction())
    want = D.scaled_sum(init, np.stack([gbt.get_tree(t)["leaf_value"][nd] for t, nd in enumerate(nodes)]), ref["dart_weights"], K)
    p = gbt.predict(va)
    p = p[None] if K == 1 else p.T
    assert np.array_equal(p, want), f"predict differs from the scaled model in {int((p != want).sum())} values"
    oracle_model = D.scaled_sum(init, np.stack([ref["trees"][t]["leaf_value"][nd] for t, nd in enumerate(nodes)]),
                                ref["dart_weights"], K)
    assert np.allclose(p, oracle_model, rtol=0, atol=1e-5 * len(nodes))
    gbt.close()
    tr.close()
    va.close()
    full.close()
