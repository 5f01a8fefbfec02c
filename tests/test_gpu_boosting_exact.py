"""Every boosting iteration's row pipeline against the exact reference of tests/boost_ref.py.

For each iteration the reference starts from the device's own output of the stage before: predictions are the float32
sums of the device trees' leaves in tree order (rows routed through the emitted trees), gradients, scales and the
iteration's row sample follow from them, and every node of the device tree is compared with the integer sums over its
rows.  Checked exactly: num_examples / num_pos_examples, stat[0..2] (inside [lo, hi] where an exp rounding is free),
leaf values (from the device's stat), training predictions (get_predictions and predict), held-out predictions, accuracy.
Within 1 float ulp: split scores (of the exact value) and losses (the double summation order is the only freedom).
"""
import numpy as np
import pytest

import ydf_b200
from oracle import oracle as O
from tests import boost_ref as R

pytestmark = pytest.mark.gpu

F32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------
# fixtures

def byte_table(rng, n, layout):
    """Byte columns: (kind, B) with kind 'num' / 'cat'; skewed codes with empty buckets."""
    bins, nb, ft = [], [], []
    for kind, B in layout:
        if kind == "num":
            c = np.clip(((rng.normal(size=n) + 3) / 6 * B).astype(np.int64), 0, B - 1)
        else:
            p = 1.0 / np.arange(1, B + 1) ** 1.1
            p /= p.sum()
            c = rng.choice(B, size=n, p=p)
        bins.append(c.astype(np.uint8))
        nb.append(B)
        ft.append(1 if kind == "cat" else 0)
    return np.stack(bins), np.array(nb, np.int32), np.array(ft, np.int32)


class Table:
    """A training table and a held-out table with the same columns, plus their reference column descriptions."""

    def __init__(self, rng, n, n_valid, layout, extra=None):
        self.n, self.n_valid = n, n_valid
        both, self.nb, self.ft = byte_table(rng, n + n_valid, layout)
        self.extra = extra or {}
        ext = {}
        for f, (kind, B) in self.extra.items():
            if kind == "wide_num":
                ext[f] = rng.integers(0, B, size=n + n_valid)
            elif kind == "wide_cat":
                p = 1.0 / np.arange(1, B + 1) ** 1.05
                ext[f] = rng.choice(B, size=n + n_valid, p=p / p.sum())
            else:   # presorted: ties, -0.0 / +0.0, NaN
                v = np.round(rng.normal(size=n + n_valid), 2).astype(F32)
                v[rng.random(n + n_valid) < 0.1] = F32(-0.0)
                v[rng.random(n + n_valid) < 0.1] = F32(0.0)
                v[rng.random(n + n_valid) < 0.05] = np.nan
                ext[f] = v
            both[f] = 0
            self.nb[f] = 1 if kind != "wide_cat" else self.nb[f]
            if kind == "wide_cat":
                self.ft[f] = 1
        self.ext = ext
        self.signal = both.astype(np.float64)   # for the labels
        for f, v in ext.items():
            self.signal[f] = np.nan_to_num(np.asarray(v, np.float64)) / max(1.0, float(np.nanmax(np.abs(v))))
        self.ds, self.cols = self._make(both[:, :n], slice(0, n))
        self.vds, self.vcols = self._make(both[:, n:], slice(n, n + n_valid)) if n_valid else (None, None)

    def _make(self, bins, part):
        ds = ydf_b200.Dataset(np.ascontiguousarray(bins), self.nb, np.zeros(len(self.nb), np.int32), feature_types=self.ft)
        cols = [("cat" if self.ft[f] == 1 else "num", bins[f], int(self.nb[f]), None) for f in range(len(self.nb))]
        for f, (kind, B) in self.extra.items():
            v = self.ext[f][part]
            if kind == "wide_num":
                values = np.arange(B, dtype=F32)
                ds.set_wide_column(f, v.astype(np.uint16), B, 0, values, 0.0)
                cols[f] = ("wide_num", v, B, values)
            elif kind == "wide_cat":
                ds.set_wide_categorical_column(f, v.astype(np.uint16), B, 0)
                cols[f] = ("wide_cat", v, B, None)
            else:
                ds.set_numerical_column(f, v, 0.0)
                cols[f] = ("pre", ds.get_numerical_column(f), 0, None)
        return ds, cols

    def margin(self, rng, scale=1.0):
        F = self.signal.shape[0]
        w = rng.normal(size=F)
        m = (w[:, None] * (self.signal - self.signal.mean(axis=1, keepdims=True))
             / (self.signal.std(axis=1, keepdims=True) + 1e-9)).sum(axis=0)
        return scale * m + rng.normal(scale=0.7, size=m.shape)


# ---------------------------------------------------------------------------------------------------------------------
# the driver

def check_run(gbt, cfg, table, labels, vlabels=None, weights=None, iters=3, step=False, vweights=None, on_tree=None,
              trained=False, logged=None, kept_trees=None):
    """Trains `iters` iterations (one train() call, or step() + get_predictions() per iteration) and checks every stage
    against the reference.  labels: binomial {1, 2}, multinomial 1..K, squared error floats.
    vweights: the held-out rows' weights.  on_tree(t, rows): called after each tree's checks with the per-row quantities
    it was trained on (dict g, h, g_alt, h_alt, sel, w); with step=True before the next step(), so that the tree's
    candidate capture is still the live one.  trained=True: the caller already trained `iters` iterations (train() with
    early stopping), of which `logged` have losses and whose model keeps the first `kept_trees` trees.
    -> (number of nodes checked, the reference's (P, g2w power of two or None) of every tree)."""
    n = table.n
    loss = int(cfg.loss)
    K = int(cfg.num_classes) if loss == 2 else 1
    logit = loss in (0, 2)
    goss = cfg.goss_alpha > 0 or cfg.goss_beta > 0
    sub = cfg.subsample < 1.0
    weighted = weights is not None or goss
    labels = np.asarray(labels)
    logged = iters if logged is None else logged
    kept_trees = iters * K if kept_trees is None else kept_trees
    stepped = []
    if not step and not trained:
        gbt.train(iters)
    init = F32(gbt.initial_prediction())
    wide_cat = any(c[0] == "wide_cat" for c in table.cols)
    pred = np.full((K, n), init, F32)
    vpred = np.full((K, table.n_valid), init, F32) if vlabels is not None else None
    kept = (pred.copy(), None if vpred is None else vpred.copy()) if kept_trees == 0 else None
    rng = O.Rng(int(cfg.random_seed))
    rng.discard(int(cfg.rng_words_consumed))   # the row draws share the learner's stream, after those words
    if weights is not None:
        w_pow2 = R.pow2_cover(np.max(weights))
    elif goss:
        amp = float((F32(1) - F32(cfg.goss_alpha)) / F32(cfg.goss_beta)) if cfg.goss_beta > 0 else 1.0
        w_pow2 = 1.0
        while w_pow2 < amp:
            w_pow2 *= 2.0
    else:
        w_pow2 = None
    errs, checked, scales = [], 0, []
    for it in range(iters):
        if step:
            gbt.step()
            stepped.append(gbt.get_predictions().copy())
        # per-row gradients from the predictions before the iteration
        if loss == 2:
            cls = labels - 1
            g, h, amb = R.mc_gradients(pred, cls)
            g_alt, h_alt, _ = R.mc_gradients(pred, cls, flip=amb)
        elif loss == 0:
            pos = labels == 2
            g, h, amb = R.binomial_gradients(pred[0], pos)
            g_alt, h_alt, _ = R.binomial_gradients(pred[0], pos, alt=True)
            g, h, g_alt, h_alt = g[None], h[None], g_alt[None], h_alt[None]
        else:
            g, h, amb = R.squared_error_gradients(pred[0], labels)
            g, h, g_alt, h_alt = g[None], h[None], g[None], h[None]
        sel, w = None, weights
        if goss:
            sel, w = R.goss_selection(g[0], cfg.goss_alpha, cfg.goss_beta, rng)
        elif sub:
            sel = R.subsample_mask(rng, n, cfg.subsample)
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
            scales.append((P, rows.g2pow2 if weighted else None))
            rows_of = R.route(tree, table.cols, sets)
            errs += R.check_tree(tree, rows_of, rows, cfg, logit, where=f"tree {t}")
            checked += len(tree)
            leaf = R.leaf_of_rows(tree, rows_of, n)
            pred[k] = (pred[k] + tree["leaf_value"][leaf]).astype(F32)
            if vpred is not None:
                vrows = R.route(tree, table.vcols, sets)
                vpred[k] = (vpred[k] + tree["leaf_value"][R.leaf_of_rows(tree, vrows, table.n_valid)]).astype(F32)
            if t + 1 == kept_trees:
                kept = (pred.copy(), None if vpred is None else vpred.copy())
            if on_tree is not None:
                on_tree(t, dict(g=gk, h=hk if has_h else None, g_alt=gk_alt, h_alt=hk_alt if has_h else None, sel=sel,
                                w=w if weighted else None, tree=tree))
        if step:
            got = stepped[it] if K == 1 else stepped[it].T
            if not np.array_equal(got.reshape(K, n), pred):
                errs.append(f"iteration {it}: get_predictions after step() differ in {int((got.reshape(K, n) != pred).sum())} rows")
        if it >= logged:
            continue
        errs += check_losses(gbt.train_loss(it), loss, pred, labels, weights, w_pow2 if weights is not None else None,
                             f"train loss {it}")
        if vpred is not None:
            vw_pow2 = R.pow2_cover(np.max(vweights)) if vweights is not None else None
            errs += check_losses(gbt.validation_loss(it), loss, vpred, np.asarray(vlabels), vweights, vw_pow2,
                                 f"validation loss {it}")
    got = gbt.get_predictions()
    got = got[None] if K == 1 else got.T
    if not np.array_equal(got, pred):
        errs.append(f"get_predictions differ in {int((got != pred).sum())} values")
    # predict() evaluates the model: the first kept_trees trees
    p = gbt.predict(table.ds)
    if not np.array_equal(p[None] if K == 1 else p.T, kept[0]):
        errs.append("predict(training table) differs from the leaf sums")
    if vpred is not None:
        p = gbt.predict(table.vds)
        if not np.array_equal(p[None] if K == 1 else p.T, kept[1]):
            errs.append("predict(held-out table) differs from the leaf sums")
    assert not errs, f"{len(errs)} mismatches:\n" + "\n".join(errs[:30])
    return checked, scales


def check_losses(got, loss, pred, labels, weights, w_pow2, where):
    """(loss, secondary) of one iteration against the per-row float terms."""
    errs = []
    n = pred.shape[1]
    denom = R.sequential_sum(weights) if weights is not None else float(n)
    if loss == 1:
        terms = R.squared_error_terms(pred[0], labels, weights)
        want = F32(np.sqrt(np.sum(terms.astype(np.float64)) / denom))
        want_sec = want
    else:
        if loss == 0:
            terms, hit = R.binomial_loss_terms(pred[0], labels == 2, weights)
        else:
            terms, hit = R.mc_loss_terms(pred, labels - 1, weights)
        want = F32(-np.sum(terms.astype(np.float64)) / denom)
        if weights is None:
            want_sec = F32(int(hit.sum()) / float(n))
        else:
            units = int(R.correct_units(weights, w_pow2)[hit].sum())
            want_sec = F32(units / float(F32(2.0 ** 31 / w_pow2)) / denom)
    if abs(float(got[0]) - float(want)) > R.ulp32(want):
        errs.append(f"{where}: loss {got[0]!r} vs {want!r}")
    if loss == 1:
        if abs(float(got[1]) - float(want_sec)) > R.ulp32(want_sec):
            errs.append(f"{where}: secondary {got[1]!r} vs {want_sec!r}")
    elif F32(got[1]) != want_sec:
        errs.append(f"{where}: accuracy {got[1]!r} vs {want_sec!r}")
    return errs


# ---------------------------------------------------------------------------------------------------------------------
# cases

LAYOUT = [("num", 255), ("cat", 7), ("num", 16), ("cat", 40), ("num", 64)]


def labels_for(loss, m, K=3):
    if loss == 0:
        return (m > np.median(m)).astype(np.int32) + 1
    if loss == 2:
        q = np.quantile(m, np.linspace(0, 1, K + 1)[1:-1])
        return (np.searchsorted(q, m) + 1).astype(np.int32)
    return m.astype(F32)


CASES = {
    # rows: one partial block, tails around the 8192-row block
    "squared_error_n1": dict(n=1, cfg=dict(loss=1, min_examples=1)),
    "binomial_n7": dict(n=7, cfg=dict(loss=0, min_examples=1)),
    "binomial_n8191": dict(n=8191, cfg=dict(loss=0), valid=3000),
    "binomial_n8193_step": dict(n=8193, cfg=dict(loss=0), step=True, valid=1000),
    "binomial_hessian_l1_l2_parent": dict(n=8192 * 3 + 5, cfg=dict(loss=0, use_hessian_gain=1, l1_regularization=0.5,
                                                                   l2_regularization=2.0, l2_regularization_categorical=3.0,
                                                                   hessian_split_score_subtract_parent=1)),
    "binomial_hessian_step": dict(n=8192 * 5 + 5, cfg=dict(loss=0, use_hessian_gain=1, min_examples=1), step=True),
    "binomial_clamp": dict(n=20000, cfg=dict(loss=0, shrinkage=1.0, clamp_leaf_logit=0.3, min_examples=1), clamp=True),
    "squared_error_1e3": dict(n=8192 * 2 + 5, cfg=dict(loss=1), scale=1e3, valid=2000),
    "squared_error_hessian_l2": dict(n=30000, cfg=dict(loss=1, use_hessian_gain=1, l2_regularization=1.0), scale=10.0),
    "squared_error_wide_presorted": dict(n=40000, cfg=dict(loss=1, max_depth=5), scale=3.0, valid=5000,
                                         extra={1: ("wide_cat", 1000), 2: ("wide_num", 4096), 4: ("pre", 0)}),
    "binomial_wide_presorted_step": dict(n=30000, cfg=dict(loss=0, max_depth=5), step=True, valid=3000,
                                         extra={1: ("wide_cat", 700), 4: ("pre", 0)}),
    "multinomial_k3_n7": dict(n=7, cfg=dict(loss=2, num_classes=3, min_examples=1), K=3),
    "multinomial_k3": dict(n=8192 + 5, cfg=dict(loss=2, num_classes=3), K=3, valid=2000),
    "multinomial_k7_step": dict(n=25000, cfg=dict(loss=2, num_classes=7), K=7, step=True, valid=2000),
    # shrinkage 1: max|g| (max|w*g|, max (w*g)*g) falls by a power of two after the first tree, so a tree quantised
    # with the previous iteration's scales would show in every node's stat[]
    "squared_error_scale_drop": dict(n=30000, cfg=dict(loss=1, shrinkage=1.0, min_examples=1), scale=8.0, scale_drop=True),
    "weighted_squared_error_scale_drop": dict(n=30000, cfg=dict(loss=1, shrinkage=1.0, min_examples=1), scale=8.0,
                                              weights=True, scale_drop=True),
    "weighted_squared_error": dict(n=30000, cfg=dict(loss=1, min_examples=3), scale=5.0, weights=True),
    "weighted_binomial": dict(n=30000, cfg=dict(loss=0), weights=True, valid=2000),
    "weighted_multinomial": dict(n=30000, cfg=dict(loss=2, num_classes=4), K=4, weights=True),
    "subsample_binomial": dict(n=30000, cfg=dict(loss=0, subsample=0.5), valid=2000),
    "subsample_squared_error_step": dict(n=20000, cfg=dict(loss=1, subsample=0.5), step=True, scale=2.0),
    "goss_binomial": dict(n=30000, cfg=dict(loss=0, goss_alpha=0.2, goss_beta=0.1)),
    "goss_squared_error": dict(n=30000, cfg=dict(loss=1, goss_alpha=0.3, goss_beta=0.15), scale=4.0),
    "pure_labels": dict(n=9000, cfg=dict(loss=1), pure=True),
    "best_first": dict(n=30000, cfg=dict(loss=0, growing_strategy=1, max_num_nodes=6, max_depth=7, min_examples=1),
                       valid=2000),
    "best_first_weighted": dict(n=30000, cfg=dict(loss=1, growing_strategy=1, max_num_nodes=9, max_depth=7), weights=True,
                                scale=3.0),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_boosting_iterations_match_the_reference(case):
    c = CASES[case]
    rng = np.random.default_rng(sorted(CASES).index(case) + 101)
    K = c.get("K", 3)
    table = Table(rng, c["n"], c.get("valid", 0), LAYOUT, c.get("extra"))
    cfg = ydf_b200.default_config(**{"max_depth": 6, **c["cfg"]})
    m = table.margin(rng, c.get("scale", 1.0))
    if c.get("scale", 1.0) >= 1e3:
        m = m + 1e3                     # labels around 1e3: P > 1 at every iteration
    if c.get("pure"):
        m = np.full_like(m, 2.5)
    y = labels_for(cfg.loss, m, K)
    ytr, yv = y[:table.n], (y[table.n:] if table.n_valid else None)
    gbt = ydf_b200.Gbt(table.ds, cfg)
    w = None
    if c.get("weights"):
        w = rng.uniform(0.1, 3.0, size=table.n).astype(F32)
        w[rng.random(table.n) < 0.05] = 0.0
        gbt.set_weights(w)
    gbt.set_labels(ytr)
    if yv is not None:
        gbt.set_validation(table.vds, yv)
    iters = 2 if cfg.loss == 2 and K > 3 else 3
    checked, scales = check_run(gbt, cfg, table, ytr, yv, weights=w, iters=iters, step=c.get("step", False))
    assert checked > 0
    if c.get("scale_drop"):
        assert scales[1][0] < scales[0][0], scales
        if w is not None:
            assert scales[1][1] < scales[0][1], scales
    if c.get("clamp"):
        leaves = np.concatenate([gbt.get_tree(t)["leaf_value"] for t in range(iters)])
        assert (np.abs(leaves) == F32(cfg.clamp_leaf_logit)).any()
    if c.get("pure"):
        assert all(len(gbt.get_tree(t)) == 1 for t in range(iters))
    if cfg.growing_strategy == 1:
        # pruned splits: rows below them keep deep node ids and must still get the leaf's value (checked above)
        assert all(int((gbt.get_tree(t)["feature"] < 0).sum()) <= cfg.max_num_nodes for t in range(iters))


def test_large_table_deepest_tree():
    """2.5M rows x 8 features at the deepest tree the engine grows, max_depth 10 (9 split levels), min_examples 1: more than
    2 x 132 blocks of 8192 rows per partition grid; the last k_partition, at level 8, with 256 split nodes (half of the
    kPartMaxLevelNodes shared node table) and 512 children on the single shared accumulator copy; earlier levels with 16
    and with 32 children on both sides of the lane-private bound.  A partition of 512 level nodes (1024 children) would
    need max_depth 11, whose level 9 needs 256 histogram slots: the active lists' 8-bit slots refuse it, checked below."""
    rng = np.random.default_rng(7)
    n = 2_500_000
    table = Table(rng, n, 0, [("num", 255), ("num", 255), ("cat", 30), ("num", 64), ("num", 200), ("cat", 9),
                              ("num", 255), ("num", 128)])
    cfg = ydf_b200.default_config(loss=0, max_depth=10, min_examples=1)
    gbt = ydf_b200.Gbt(table.ds, cfg)
    y = labels_for(0, table.margin(rng))
    gbt.set_labels(y)
    check_run(gbt, cfg, table, y, iters=2)
    for t in range(2):
        tree = gbt.get_tree(t)
        # every node of level 8 (depth 9) split: 256 nodes partitioned into 512 children
        assert ((tree["depth"] == 9) & (tree["feature"] >= 0)).sum() == 256
        assert (tree["depth"] == 10).sum() == 512
    with pytest.raises(ydf_b200.YggError) as e:
        ydf_b200.Gbt(table.ds, ydf_b200.default_config(loss=0, max_depth=11, min_examples=1))
    assert e.value.code == 4 and "8-bit slots" in str(e.value)


def test_gradient_sum_of_a_node_above_2_to_the_23_rows():
    """k_node_stats removes the 2^30 bias of every row's 31-bit gradient code in integers: over more than 2^23 rows the
    biased sum passes 2^53, where a double holds only even integers.  The root of 2^23 + 8192 rows with every gradient 0
    but one of 1.0 (P = 1, code 2^30) and one of 2^-30 (code 1): an odd biased sum, stat[0] = 1 + 2^-30 exactly; a
    rounded conversion gives 1 or 1 + 2^-29."""
    n = 2 ** 23 + 8192
    bins = np.zeros((1, n), np.uint8)
    bins[0, n // 2:] = 1
    ds = ydf_b200.Dataset(bins, np.array([2], np.int32), np.zeros(1, np.int32))
    cfg = ydf_b200.default_config(loss=1, max_depth=2, min_examples=1)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(np.zeros(n, F32))
    g = np.zeros(n, F32)
    g[0], g[n - 1] = 1.0, 2.0 ** -30
    tree = gbt.train_tree_on_gradients(g)
    assert tree[0]["num_examples"] == n
    assert tree[0]["stat"][0] == 1.0 + 2.0 ** -30, repr(tree[0]["stat"][0])
    assert tree[0]["leaf_value"] == R.leaf_value(1.0 + 2.0 ** -30, float(n), cfg, False)
    gbt.close()
    ds.close()


def test_weighted_near_pure_split_score():
    """Example weights, squared error, 300K rows: two regions of constant label, one of them split into halves whose
    labels differ by two units of the 24-bit gradient code (2 P / 2^23), about the least difference whose weighted score
    clears the scan's floor of half a unit per row (boundary_score).  That is where k_weight_sums_finish's contracted
    numerator `Sp*Wn - Sn*Wp` is least accurate relative to d (about 2^-31); it must still land within 1 float ulp of the
    exact score."""
    rng = np.random.default_rng(13)
    n = 300000
    table = Table(rng, n, 0, [("num", 255), ("num", 2), ("cat", 12)])
    b0, b1 = table.cols[0][1], table.cols[1][1]
    y = np.where(b1 == 1, F32(0.7), F32(0.3)).astype(F32)
    w = rng.uniform(0.5, 2.0, size=n).astype(F32)
    # the scale P of the first tree: max |w * (y - weighted mean)|, far from a power of two here
    mean = np.sum(w.astype(np.float64) * y) / np.sum(w.astype(np.float64))
    P = R.pow2_cover(np.abs(w * (y - F32(mean))).max())
    y = np.where((b1 == 0) & (b0 >= 128), y + F32(2 * P / 2 ** 23), y).astype(F32)
    cfg = ydf_b200.default_config(loss=1, max_depth=4, min_examples=1)
    gbt = ydf_b200.Gbt(table.ds, cfg)
    gbt.set_weights(w)
    gbt.set_labels(y)
    _, scales = check_run(gbt, cfg, table, y, weights=w, iters=1)
    assert scales[0][0] == P
    tree = gbt.get_tree(0)
    assert ((tree["feature"] == 0) & (tree["threshold_bin"] == 128)).any(), "the near-pure split was not found"
