"""Wide numerical columns (257..65535 buckets, uint16 codes; DESIGN.md §20) on the GPU: the raw integer histograms of
k_hist_wide against a numpy reference (`==`), trees against the oracle on the same uint16 codes with the exact threshold
rule, the learner end to end on the reference's Abalone run, prediction / model files, and the refusals."""
import os
import tempfile

import numpy as np
import pytest

import ydf_b200
from ydf_b200 import dataspec, model_io
from oracle import oracle as O
from tests import reference_replay as R
from tests.util import compare_trees, prune_noise_splits, quantize_q24, quantize_second

pytestmark = pytest.mark.gpu


def _oracle_cfg(cfg):
    o = O.default_config()
    for k, _ in cfg._fields_:
        if k != "reserved":
            setattr(o, k, getattr(cfg, k))
    return o


def wide_table(n, seed, n_narrow=3, wide_sizes=(300, 2000), n_cat=1, task="binary", na_frac=0.05):
    """Seeded table mixing narrow lossless, wide lossless (with missing values) and categorical columns.
    -> (columns, uint16 bins [F, n], feature types, labels)."""
    rng = np.random.default_rng(seed)
    raw, margin = [], np.zeros(n)
    for j in range(n_narrow):
        x = rng.integers(0, 40 + 30 * j, size=n).astype(np.float32) * 1.5
        raw.append(x)
        margin += rng.normal() * (x / x.max() - 0.5)
    for k in wide_sizes:
        grid = np.sort(rng.choice(100000, size=k, replace=False)).astype(np.float32) / 7.0
        x = grid[rng.integers(0, k, size=n)]
        x[rng.random(n) < na_frac] = np.nan
        raw.append(x)
        margin += 2.0 * np.sin(np.nan_to_num(x, nan=0.0) / grid.max() * 6.0)
    cols = [dataspec.infer_column_lossless(f"x{j}", x, max_distinct=65535) for j, x in enumerate(raw)]
    bins = [c.encode16(x) for c, x in zip(cols, raw)]
    types = [0] * len(cols)
    for j in range(n_cat):
        k = 12
        c = rng.integers(0, k, size=n).astype(np.uint8)
        margin += rng.normal(size=k)[c]
        cols.append(dataspec.CategoricalColumn(name=f"c{j}", vocabulary=["<OOD>"] + [str(i) for i in range(1, k)],
                                               counts=[0] * k, num_bins=k, na_bin=1))
        bins.append(c.astype(np.uint16))
        types.append(1)
    margin += rng.normal(scale=0.5, size=n)
    if task == "binary":
        y = (margin > np.median(margin)).astype(np.int32) + 1
    elif task == "multi":
        y = np.digitize(margin, np.quantile(margin, [1 / 3, 2 / 3])).astype(np.int32) + 1
    else:
        y = margin.astype(np.float32)
    return cols, np.stack(bins), np.array(types, np.int32), y, raw


def engine_dataset(cols, bins, types):
    """Byte columns as they are (bucket values for the narrow lossless ones), wide columns attached."""
    ds = dataspec.device_dataset(bins, cols)
    for f, c in enumerate(cols):
        if getattr(c, "bucket_values", None) is not None and not c.wide:
            ds.set_bucket_values(f, c.bucket_values, c.mean)
    assert list(ds.feature_types) == list(types)
    return ds


def oracle_train(cols, bins, types, y, cfg, iters, weights=None, best_first=None):
    vals = [getattr(c, "bucket_values", None) for c in cols]
    O.set_bucket_values(vals, [getattr(c, "mean", 0.0) for c in cols])
    if weights is not None:
        O.set_weights(weights)
    if best_first is not None:
        O.set_growing_strategy(True, best_first)
    O.set_hessian_buckets_double(bool(cfg.use_hessian_gain))   # the engine's hessian sums are exact integers
    O.set_goss_stable_sort(True)                               # equal |gradient|: row order, as the engine
    try:
        nb = [c.num_bins for c in cols]
        na = [c.na_bin for c in cols]
        if cfg.loss == 2:
            return O.gbt_train_mc(bins, nb, na, y, _oracle_cfg(cfg), iters, num_threads=4, feature_type=types)
        return O.gbt_train(bins, nb, na, y, _oracle_cfg(cfg), iters, num_threads=4, feature_type=types,
                           shuffle_candidates=cfg.candidate_shuffle)
    finally:
        O.set_bucket_values(None)
        O.set_weights(None)
        O.set_growing_strategy(False)
        O.set_hessian_buckets_double(False)
        O.set_goss_stable_sort(False)


# ---- histograms ------------------------------------------------------------------------------------------------------

def wide_hist_ref(codes, offs, total, slot_of_row, n_slots, q, second_q=None):
    s = np.zeros((n_slots, total), np.uint64)
    c = np.zeros((n_slots, total), np.uint32)
    s2 = None if second_q is None else np.zeros((n_slots, total), np.uint64)
    rows = np.nonzero(slot_of_row >= 0)[0]
    for w, code in enumerate(codes):
        idx = slot_of_row[rows].astype(np.int64) * total + offs[w] + code[rows]
        np.add.at(s.reshape(-1), idx, q[rows].astype(np.uint64))
        np.add.at(c.reshape(-1), idx, np.uint32(1))
        if s2 is not None:
            np.add.at(s2.reshape(-1), idx, second_q[rows].astype(np.uint64))
    return s, c, s2


@pytest.mark.parametrize("sizes,hessian,weighted,level,n_slots", [
    ((257, 4096), 0, False, 0, 1),
    ((16611, 65535), 0, False, 0, 1),
    ((257, 16611), 1, False, 2, 2),
    ((4096, 65535), 0, True, 3, 4),
])
def test_wide_histograms_are_exact(sizes, hessian, weighted, level, n_slots):
    """Raw u64 sums, u32 counts and the second plane (hessians with the hessian gain on the binomial loss, example weights on
    a weighted handle) of every wide bucket, `==` against numpy, through the seam that runs the training code: empty
    buckets, a bucket that takes every row of a column, rows outside every slot, several slots."""
    n = 70000
    rng = np.random.default_rng(sum(sizes) + level)
    codes = [rng.integers(0, B, size=n).astype(np.uint16) for B in sizes]
    codes[0][:] = sizes[0] - 1 if level else 5           # one bucket takes every row of the first wide column
    codes[1][codes[1] % 7 == 0] = 0                        # many empty buckets, a crowded bucket 0
    F = 2 + len(sizes)
    byte = rng.integers(0, 32, size=(F, n)).astype(np.uint8)
    ds = ydf_b200.Dataset(byte, [32] * F, [0] * F)
    for w, B in enumerate(sizes):
        ds.set_wide_column(2 + w, codes[w], B, B // 2, np.arange(B, dtype=np.float32), float(B // 2))
        got, nb, na = ds.get_wide_column(2 + w)
        assert (got == codes[w]).all() and nb == B and na == B // 2
    cfg = ydf_b200.default_config(max_depth=6, use_hessian_gain=hessian)
    gbt = ydf_b200.Gbt(ds, cfg)
    if weighted:
        gbt.set_weights(rng.random(n).astype(np.float32) * 3)
    g = (rng.normal(size=n) * 0.3).astype(np.float32)
    g[:100] = 0.0
    slots = rng.integers(-1 if n_slots > 1 else 0, n_slots, size=n).astype(np.int32)
    second = None
    if gbt.has_second_plane():
        second = (rng.random(n) * (3 if weighted else 0.25)).astype(np.float32)
    _, _, _, (P, V) = gbt.level_histogram(level, g, slots, n_slots, second=second)
    s, c, s2 = gbt.wide_histogram(n_slots)
    offs = np.concatenate([[0], np.cumsum(sizes)])
    rs, rc, rs2 = wide_hist_ref(codes, offs, int(offs[-1]), slots, n_slots, quantize_q24(g, P),
                                None if second is None else quantize_second(second, V))
    assert (c == rc).all() and (s == rs).all()
    if second is not None:
        assert (s2 == rs2).all()
    assert int(c.sum()) == int((slots >= 0).sum()) * len(sizes)


# ---- trees against the oracle ----------------------------------------------------------------------------------------

CASES = {
    "variance": dict(),
    "hessian": dict(use_hessian_gain=1),
    "regression": dict(loss=1),
    "depth2": dict(max_depth=2),
    "depth10": dict(max_depth=10, min_examples=5),
    "min_examples_edge": dict(min_examples=400, max_depth=8),
    "subsample": dict(subsample=0.6),
    "goss": dict(goss_alpha=0.2, goss_beta=0.1),
    "no_sibling_subtraction": dict(sibling_subtraction=0),
    "tie_shuffle": dict(candidate_shuffle=2, split_jobs_draw_seeds=1),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_trees_match_oracle(case):
    kw = dict(max_depth=6, num_trees=4)
    kw.update(CASES[case])
    task = "regression" if kw.get("loss") == 1 else "binary"
    n = 200000 if case == "depth10" else 60000
    cols, bins, types, y, _ = wide_table(n, seed=len(case), task=task)
    ds = engine_dataset(cols, bins, types)
    cfg = ydf_b200.default_config(**kw)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(y)
    gbt.train(cfg.num_trees)
    ref = oracle_train(cols, bins, types, y, cfg, cfg.num_trees)
    wide = {f for f, c in enumerate(cols) if getattr(c, "wide", False)}
    used = 0
    for i in range(cfg.num_trees):
        got, want = gbt.get_tree(i), ref["trees"][i]
        if case == "depth10":
            # deep nodes of a few rows with equal gradients: the oracle's doubles "split" them on 1e-16 of rounding noise
            # (score <= 1e-12), the exact integer sums give 0 and a leaf
            got, want = prune_noise_splits(got, 1e-12), prune_noise_splits(want, 1e-12)
            assert int(want["depth"].max()) == 10
        errs = compare_trees(got, want)
        assert not errs, (case, i, errs[:5])
        sp = (want["feature"] >= 0) & (want["condition_type"] == 0)   # numerical splits: all under the exact rule
        np.testing.assert_array_equal(got["threshold_value"][sp], want["threshold_value"][sp])
        used += sum(int(f in wide) for f in want["feature"][sp])
        assert abs(gbt.train_loss(i)[0] - ref["loss"][i]) <= 1e-5 * max(1.0, abs(ref["loss"][i]))
    assert used > 0, "no split on a wide column"
    # the same trees again on a new handle
    gbt2 = ydf_b200.Gbt(ds, cfg)
    gbt2.set_labels(y)
    gbt2.train(cfg.num_trees)
    for i in range(cfg.num_trees):
        assert gbt2.get_tree(i).tobytes() == gbt.get_tree(i).tobytes()


def test_weighted_trees_match_oracle():
    cols, bins, types, y, _ = wide_table(60000, seed=41)
    w = np.random.default_rng(5).random(len(y)).astype(np.float32) * 2 + 0.1
    ds = engine_dataset(cols, bins, types)
    cfg = ydf_b200.default_config(max_depth=6, num_trees=3)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_weights(w)
    gbt.set_labels(y)
    gbt.train(3)
    ref = oracle_train(cols, bins, types, y, cfg, 3, weights=w)
    for i in range(3):
        errs = compare_trees(gbt.get_tree(i), ref["trees"][i])
        assert not errs, (i, errs[:5])


def test_multinomial_trees_match_oracle():
    cols, bins, types, y, _ = wide_table(50000, seed=43, task="multi")
    ds = engine_dataset(cols, bins, types)
    cfg = ydf_b200.default_config(loss=2, num_classes=3, max_depth=5, num_trees=2)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(y)
    gbt.train(2)
    ref = oracle_train(cols, bins, types, y, cfg, 2)
    for i in range(6):
        errs = compare_trees(gbt.get_tree(i), ref["trees"][i])
        assert not errs, (i, errs[:5])


def test_best_first_trees_match_oracle():
    cols, bins, types, y, _ = wide_table(60000, seed=47)
    ds = engine_dataset(cols, bins, types)
    cfg = ydf_b200.default_config(max_depth=6, num_trees=3, growing_strategy=1, max_num_nodes=20)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(y)
    gbt.train(3)
    ref = oracle_train(cols, bins, types, y, cfg, 3, best_first=20)
    for i in range(3):
        errs = compare_trees(gbt.get_tree(i), ref["trees"][i])
        assert not errs, (i, errs[:5])


# ---- learner, prediction, model files ----------------------------------------------------------------------------

def test_learner_reproduces_the_abalone_run_with_wide_columns():
    """abalone_regression_gbdt_v2 with every setting at the reference's default and max_exact_numerical_values=65535:
    the 7 numerical columns (up to 2429 distinct values) are exact, 4 of them wide."""
    ref, data = R.load_run("abalone")
    label = "Rings"
    model = ydf_b200.GradientBoostedTreesLearner(label=label, task="REGRESSION", max_exact_numerical_values=65535).train(
        {k: np.asarray(v) for k, v in data.items()})
    assert any(getattr(c, "wide", False) for c in model.data_spec.columns)
    logs = model.training_logs
    assert len(logs) == len(ref["log_training_loss"]) == 75 and model.num_trees() == 45
    got = np.array([e["loss"] for e in logs], np.float64)
    assert np.abs(got - ref["log_training_loss"].astype(np.float64)).max() <= 1e-5
    got = np.array([e["validation_loss"] for e in logs], np.float64)
    assert np.abs(got - ref["log_validation_loss"].astype(np.float64)).max() <= 1e-5
    assert abs(model.validation_loss - float(ref["validation_loss"])) <= 1e-5


def test_predictions_and_model_files_agree():
    cols, bins, types, y, raw = wide_table(40000, seed=53, n_cat=0)
    names = [c.name for c in cols]
    data = {n: x for n, x in zip(names, raw)}
    data["y"] = np.where(y == 2, "a", "b")
    rng = np.random.default_rng(3)
    train = rng.random(len(y)) < 0.8
    tr = {k: v[train] for k, v in data.items()}
    te = {k: v[~train] for k, v in data.items()}
    L = ydf_b200.GradientBoostedTreesLearner
    # the explicit validation set takes the uint16 path of encode_features
    model = L(label="y", max_exact_numerical_values=65535, num_trees=15, validation_ratio=0.0).train(tr, valid=te)
    assert any(c.wide for c in model.data_spec.columns)
    assert all(len(e) > 3 for e in model.training_logs)   # validation losses logged
    vb = dataspec.encode_features(te, model.data_spec.columns)
    assert vb.dtype == np.uint16
    p_host = model.predict(te)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "m")
        model.save(path)
        m = model_io.read_ydf_model(path)
        raw_io = model_io.predict_ydf_model(m, {k: v for k, v in te.items() if k != "y"})
    p_io = 1 / (1 + np.exp(-raw_io.astype(np.float64)))
    np.testing.assert_allclose(p_io, p_host, rtol=0, atol=1e-6)
    # Routing of values the data spec has never seen, inside a gap of the column's values.  Every value present when the
    # data spec was built has its own bucket, so for those `code >= threshold_bin` IS `value >= threshold_value`.  A new
    # value inside a gap is routed by its bucket, i.e. by the column's boundary (the middle of its two neighbouring
    # values), in model.predict, in the saved model and on the device alike (DESIGN.md §20): pinned here on real rows.
    used = [t[t["feature"] >= 0] for t in model.trees]
    assert any(model.data_spec.columns[f].wide for t in used for f in t["feature"])
    gap_rows, differ = [], 0
    for t in used:
        for nd in t:
            c = model.data_spec.columns[nd["feature"]]
            if not c.wide:
                continue
            v, k, thr = c.bucket_values, int(nd["threshold_bin"]), np.float32(nd["threshold_value"])
            assert v[k - 1] < thr <= v[k]                         # values present: the bucket rule is the float rule
            for lo in (k - 2, k - 1, k):                          # new values in the gaps around the cut
                if 0 <= lo and lo + 1 < len(v):
                    for x in np.linspace(v[lo], v[lo + 1], 7, dtype=np.float32)[1:-1]:
                        code = int(c.encode16(np.array([x], np.float32))[0])
                        assert (code >= k) == (x >= c.boundaries[k - 1])   # the boundary decides
                        differ += int((code >= k) != (x >= thr))
                        gap_rows.append((c.name, x))
    assert differ > 0   # the two rules do part ways inside the gaps (the limit documented in DESIGN.md §20)
    probe = {k: np.repeat(te[k][:1], len(gap_rows)) for k in te}
    for i, (name, x) in enumerate(gap_rows):
        probe[name] = probe[name].copy()
        probe[name][i] = x
    p_host = model.predict(probe)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "m")
        model.save(path)
        raw_io = model_io.predict_ydf_model(model_io.read_ydf_model(path), {k: v for k, v in probe.items() if k != "y"})
    np.testing.assert_allclose(1 / (1 + np.exp(-raw_io.astype(np.float64))), p_host, rtol=0, atol=1e-6)


def test_engine_predict_on_a_held_out_split_agrees_with_the_host_model():
    cols, bins, types, y, _ = wide_table(50000, seed=59)
    ds = engine_dataset(cols, bins, types)
    keep = np.random.default_rng(1).random(len(y)) < 0.7
    tr, va = ds.split_rows(keep)
    for f, c in enumerate(cols):
        if getattr(c, "wide", False):
            assert (tr.get_wide_column(f)[0] == bins[f][keep]).all()
            assert (va.get_wide_column(f)[0] == bins[f][~keep]).all()
    cfg = ydf_b200.default_config(max_depth=6, num_trees=5)
    gbt = ydf_b200.Gbt(tr, cfg)
    gbt.set_labels(y[keep])
    gbt.set_validation(va, y[~keep])
    gbt.train(5)
    trees = [gbt.get_tree(i) for i in range(gbt.num_trees())]
    model = ydf_b200.GradientBoostedTreesModel(dataspec.DataSpec(cols, "y", "CLASSIFICATION", [1, 2]), trees,
                                               gbt.initial_prediction(), "BINOMIAL_LOG_LIKELIHOOD")
    np.testing.assert_allclose(gbt.predict(va), model._raw(bins[:, ~keep]), rtol=0, atol=2e-6)
    # the device's validation pass routes the held-out rows the same way
    assert np.isfinite(gbt.validation_loss(4)[0])
    # ygg_partition_rows on a wide feature: bucket >= threshold, stable
    f = next(f for f, c in enumerate(cols) if getattr(c, "wide", False))
    rows = np.arange(0, int(keep.sum()), 3, dtype=np.uint32)
    pos, neg = tr.partition_rows(rows, f, 150)
    col = bins[f][keep]
    assert (pos == rows[col[rows] >= 150]).all() and (neg == rows[col[rows] < 150]).all()


# ---- refusals --------------------------------------------------------------------------------------------------------

def test_refusals_on_the_device():
    rng = np.random.default_rng(0)
    n = 5000
    ds = ydf_b200.Dataset(rng.integers(0, 8, size=(3, n)).astype(np.uint8), [8, 8, 8], [0, 0, 0], feature_types=[0, 0, 1])
    codes = rng.integers(0, 300, size=n).astype(np.uint16)
    v = np.arange(300, dtype=np.float32)
    for bad in (dict(num_bins=256), dict(num_bins=65536), dict(na_bin=300), dict(codes=np.full(n, 300, np.uint16)),
                dict(values=v[::-1].copy()), dict(feature=2), dict(codes=codes[:-1])):
        a = dict(feature=0, codes=codes, num_bins=300, na_bin=0, values=v, na_replacement=1.0)
        a.update(bad)
        if "num_bins" in bad and "values" not in bad:
            a["values"] = np.arange(max(1, min(a["num_bins"], 70000)), dtype=np.float32)
        with pytest.raises(ydf_b200.YggError) as e:
            ds.set_wide_column(**a)
        assert e.value.code == 1, (bad, e.value)
    ds.set_wide_column(0, codes, 300, 7, v, 3.0)
    with pytest.raises(ydf_b200.YggError):
        ds.set_wide_column(0, codes, 300, 7, v, 3.0)   # already wide
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=4))
    for call in (lambda: gbt.set_feature_shard(0, 2, 0, 1),
                 lambda: gbt.set_row_shard(0, 1, n, 0.0, allreduce=lambda *a: 0)):
        with pytest.raises(ydf_b200.YggError) as e:
            call()
        assert e.value.code == 4


def test_weighted_handles_do_not_leak_the_wide_planes():
    """ygg_gbt_set_weights re-allocates the level buffers (a weighted handle gains a second plane): the wide planes are
    re-allocated with them, not leaked.  Device memory after several create / set_weights / destroy cycles stays where one
    cycle left it (the pool keeps freed memory mapped, so it is reused, not returned: the free figure must not fall)."""
    import torch
    n = 20000
    rng = np.random.default_rng(2)
    ds = ydf_b200.Dataset(rng.integers(0, 8, size=(3, n)).astype(np.uint8), [8, 8, 8], [0, 0, 0])
    for f in (1, 2):
        ds.set_wide_column(f, rng.integers(0, 65535, size=n).astype(np.uint16), 65535, 0,
                           np.arange(65535, dtype=np.float32), 0.0)
    planes = (32 + 2 * 64) * 2 * 65535 * 20   # depth 8, second plane: 0.42 GB per handle
    w = rng.random(n).astype(np.float32)

    def cycle():
        gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=8))
        gbt.set_weights(w)
        gbt.close()
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info(0)[0]

    first = cycle()
    last = min(cycle() for _ in range(4))
    assert first - last < planes // 2, (first, last)


def test_a_256_value_column_keeps_the_exact_rule():
    """max_exact_numerical_values >= 256 lets a column of 256 distinct values (no missing one) through: 256 buckets fit the
    byte path, which carries it with the exact threshold rule (a float threshold on every split)."""
    rng = np.random.default_rng(4)
    n = 20000
    x = (rng.integers(0, 256, size=n) * 3 + 1).astype(np.float32)
    y = np.where((x > 400) ^ (rng.random(n) < 0.1), "a", "b")
    model = ydf_b200.GradientBoostedTreesLearner(label="y", max_exact_numerical_values=256, num_trees=3,
                                                 validation_ratio=0.0).train({"x": x, "y": y})
    c = model.data_spec.columns[0]
    assert c.num_bins == 256 and not c.wide
    sp = np.concatenate([t[t["feature"] >= 0] for t in model.trees])
    assert len(sp) > 0 and np.isfinite(sp["threshold_value"]).all()


def test_sampled_root_histogram_is_exact():
    """A sampled root (subsample < 1): the root's lists hold the drawn rows only; rows outside the sample add nothing."""
    n = 50000
    rng = np.random.default_rng(9)
    codes = rng.integers(0, 4096, size=n).astype(np.uint16)
    ds = ydf_b200.Dataset(rng.integers(0, 16, size=(2, n)).astype(np.uint8), [16, 16], [0, 0])
    ds.set_wide_column(1, codes, 4096, 0, np.arange(4096, dtype=np.float32), 0.0)
    gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=4, subsample=0.5))
    g = (rng.normal(size=n) * 0.3).astype(np.float32)
    slots = np.where(rng.random(n) < 0.5, 0, -1).astype(np.int32)
    _, _, _, (P, _) = gbt.level_histogram(0, g, slots, 1)
    s, c, _ = gbt.wide_histogram(1)
    rs, rc, _ = wide_hist_ref([codes], [0], 4096, slots, 1, quantize_q24(g, P))
    assert (c == rc).all() and (s == rs).all() and int(c.sum()) == int((slots == 0).sum())


# ---- the reference's runs, tree by tree ------------------------------------------------------------------------------

def engine_trainer_wide(data, ref):
    """The engine's tree trainer (decision_tree::Train seam) on replay_trees' uint16 codes (lossless="all": one bucket per
    distinct value of every numerical column): columns of more than 256 buckets attached as wide columns, with their
    bucket values from dataspec.infer_column_lossless on the same data; the reference's candidate shuffle replayed."""
    names = [str(s) for s in ref["column_names"]]
    label = names[int(ref["label_col_idx"])]
    spec = []
    for ci, name in enumerate(names):
        if name == label:
            continue
        spec.append(None if ref["column_types"][ci] == 4 else
                    dataspec.infer_column_lossless(name, data[name].astype(np.float32), max_distinct=65000))

    def make(bins, num_bins, na_bin, feature_types, loss, num_classes):
        wide = [f for f, nb in enumerate(num_bins) if nb > 256]
        byte = np.where(np.asarray(num_bins)[:, None] > 256, 0, bins).astype(np.uint8)
        ds = ydf_b200.Dataset(byte, [1 if f in wide else nb for f, nb in enumerate(num_bins)],
                              [0 if f in wide else na for f, na in enumerate(na_bin)], feature_types=feature_types)
        for f in wide:
            c = spec[f]
            assert c.num_bins == num_bins[f] and c.na_bin == na_bin[f]
            ds.set_wide_column(f, bins[f], num_bins[f], na_bin[f], c.bucket_values, c.mean)
        cfg = ydf_b200.default_config(loss=loss, max_depth=6, min_examples=5, shrinkage=0.1, use_hessian_gain=0,
                                      candidate_shuffle=2, split_jobs_draw_seeds=1)
        if num_classes:
            cfg.num_classes = num_classes
        gbt = ydf_b200.Gbt(ds, cfg)

        def train(g, h, rng):
            gbt.set_tie_rng_position(rng.position)
            return gbt.train_tree_on_gradients(g, h)
        train.wants_rng = True
        train.keepalive = (ds, gbt)
        return train
    return make


def test_engine_trees_against_the_abalone_run_with_wide_columns():
    """All 45 trees of abalone_regression_gbdt_v2 with a bucket per distinct value of every numerical column (4 of the 7
    are wide): the engine grows every one of them identically, as the oracle does."""
    ref, data = R.load_run("abalone")
    seen = R.replay_trees(ref, data, engine_trainer_wide(data, ref), score_rtol=1e-5, leaf_atol=1e-5, lossless="all")
    assert (seen["trees"], seen["identical_trees"]) == (45, 45)
    assert seen["skipped_subtrees"] == 0 and seen["tied_subtrees"] == 0 and seen["max_leaf_err"] <= 1e-6


def test_engine_trees_against_the_adult_run_with_wide_columns():
    """All 163 trees of adult_binary_class_gbdt_v2 with a bucket per distinct value (fnlwgt wide, 16610 values), handed
    the reference's gradients.  Every one of the 4306 comparable splits has the reference's partition, count and score
    (34 through the education / education_num twin seen from the other side); 162 trees are identical.  The other one
    holds the single tied subtree: two DIFFERENT partitions with the same float score, ordered the other way by the 24-bit
    fixed-point sums (DESIGN.md §9) — the same one tie the byte path shows on this run."""
    ref, data = R.load_run("adult")
    seen = R.replay_trees(ref, data, engine_trainer_wide(data, ref), score_rtol=1e-5, leaf_atol=1e-5, lossless="all")
    assert (seen["trees"], seen["identical_trees"], seen["tied_subtrees"], seen["skipped_subtrees"]) == (163, 162, 1, 0), seen
    assert seen["splits"] == 4306 and seen["same_feature"] + seen["mirrored"] == 4306, seen
    assert seen["max_leaf_err"] <= 1e-6


def test_learner_on_the_adult_run_with_wide_columns():
    """The learner on Adult with max_exact_numerical_values=65535 (fnlwgt wide), every other setting at the reference's
    default: measured 192 log entries and 162 trees against the golden 193 and 163.  The tree trainer itself reproduces
    the reference's trees from the reference's gradients (test above); in the learner's own loop the device's gradients
    meet the run's float-level ties (DESIGN.md §20).  Pinned as measured."""
    ref, data = R.load_run("adult")
    m = ydf_b200.GradientBoostedTreesLearner(label="income", max_exact_numerical_values=65535).train(data)
    assert [c.name for c in m.data_spec.columns if getattr(c, "wide", False)] == ["fnlwgt"]
    assert (len(m.training_logs), m.num_trees()) == (192, 162)
    assert abs(m.training_logs[0]["loss"] - float(ref["log_training_loss"][0])) <= 1e-5
    assert abs(m.validation_loss - float(ref["validation_loss"])) <= 5e-4
