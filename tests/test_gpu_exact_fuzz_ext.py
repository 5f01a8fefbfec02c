"""Drawn DART and discretized-column configurations (tests/exact_fuzz_ext_draw.py), checked exactly at every stage.

Every draw builds its training table with ydf_b200.DatasetBuilder: its `disc8` / `disc16` columns binned on the GPU from
raw float32 values, the exact fuzz's other column kinds through add_bins and the dataset's setters.  Then:

- binning: every builder column against the host rule (dataspec.infer_column / infer_column16), bit for bit:
  boundaries, float32 mean, NA bin, missing count and every code, whether a 16-bit column ended wide or as bytes.  The
  held-out rows are encoded on the host with the training boundaries.
- training without DART: the exact fuzz's cases (tests/test_gpu_exact_fuzz: plain, early stopping, tie-break replay).
- DART stepped: tests/test_gpu_dart.check_dart_run (dropped sets, every node at the sampled predictions, accumulator,
  weights, weighted training and held-out losses, the scaled model), with every captured tree's candidates checked
  against the exact scan (and with candidate sampling, every validity flag), as the exact fuzz does.
- DART through train(): the stop restated on the reported losses (exact_fuzz_draw.early_stopping), the weights against
  dart_ref.weights_after of the device's dropped sets, every logged training and held-out loss against the replayed
  accumulators, and predict() on both tables against the scaled sum of the kept trees.
- the model: every split on a discretized column carries na_value = (its NA bin >= threshold_bin), the flag a model
  routes a missing value by; with a hold-out and a 16-bit column, the host model on the held-out raw floats (NaN
  included) and, for one output, the saved model read back give ygg_gbt_predict's scores bit for bit.

`python -m tests.test_gpu_exact_fuzz_ext N [offset]` runs seeds offset .. offset + N - 1 and prints every failing
configuration with its first mismatches."""
import os
import sys
import tempfile
import time

import numpy as np
import pytest

import ydf_b200
from ydf_b200 import dataspec, model_io
from tests import boost_ref as R
from tests import dart_ref as DR
from tests import exact_fuzz_draw as D
from tests import exact_fuzz_ext_draw as E
from tests import test_gpu_exact_fuzz as X
from tests.test_gpu_boosting_exact import check_losses
from tests.test_gpu_dart import check_dart_run

pytestmark = pytest.mark.gpu

F32 = np.float32
SUITE_SEEDS = E.SUITE_SEEDS
# A DART case holds its share of trees skipped for a free exp rounding (test_gpu_exact_fuzz.MAX_SKIPPED_SHARE) from
# this many scan-checkable trees on; the suite holds it over all its cases.  With every earlier tree dropped, the
# sampled predictions of many rows sit near the initial prediction, so one free rounding can skip one of 3 trees.
MIN_TREES_FOR_SHARE = 8
LOSS_NAMES = ("BINOMIAL_LOG_LIKELIHOOD", "SQUARED_ERROR", "MULTINOMIAL_LOG_LIKELIHOOD")


# ---------------------------------------------------------------------------------------------------------------------
# the tables

class ExtTable:
    """The training table of a draw built by the GPU binning step, and its held-out table encoded on the host with the
    training boundaries, in the shape check_run reads (n, n_valid, ds, cols, vds, vcols).  `spec[f]`: the host rule's
    DiscretizedColumn of discretized column f; `raw`: per feature the generated data (codes / values, or raw floats
    `x` for the training and held-out rows)."""

    def __init__(self, d, stats=None):
        rng = np.random.default_rng([d["seed"], 1])
        self.n, self.n_valid = n, nv = d["n"], d["n_valid"]
        base = [c for c in d["columns"] if c["kind"] not in E.DISC_KINDS]
        self.raw = D.make_columns(dict(columns=base), rng, n + nv)
        values = E.disc_values(d)   # (held-out rows with NaN: the model routes them by na_value)
        for f in range(len(base), len(d["columns"])):
            self.raw.append(dict(kind=d["columns"][f]["kind"], x=values[f], col=d["columns"][f]))
        self.spec = {}
        self.ds, self.cols = self._build(stats)
        self.vds, self.vcols = self._held_out() if nv else (None, None)
        sig = []
        for c in self.raw:
            v = np.nan_to_num(c["x"].astype(np.float64)) if "x" in c else None
            if v is not None:
                v = np.sign(v) * np.log1p(np.abs(v))   # (the huge-range generator)
                sig.append((v - v.mean()) / (v.std() + 1e-9))
            else:
                sig.append(D.signal(c))
        self.signal = np.stack(sig)

    def _build(self, stats):
        n, F = self.n, len(self.raw)
        b = ydf_b200.DatasetBuilder(n, F)
        for f, c in enumerate(self.raw):
            kind = c["kind"]
            if kind in ("num", "cat"):
                b.add_bins(f, c["codes"][:n], c["B"], 0, feature_type=int(kind == "cat"))
            elif kind in ("wide_num", "wide_cat", "pre"):   # a one-bucket filler; the setters attach the column
                b.add_bins(f, np.zeros(n, np.uint8), 1, 0, feature_type=int(kind == "wide_cat"))
            else:
                col = c["col"]
                add = b.add_numerical_async if kind == "disc8" else b.add_numerical16_async
                add(f, c["x"][:n], col["max_bins"], col["min_obs"], n_stats_rows=col["n_stats"])
        for f, c in enumerate(self.raw):
            if c["kind"] not in E.DISC_KINDS:
                continue
            col = c["col"]
            sample = c["x"][:n] if col["n_stats"] <= 0 else c["x"][:col["n_stats"]]
            infer = dataspec.infer_column if c["kind"] == "disc8" else dataspec.infer_column16
            want = infer(f"f{f}", sample, col["max_bins"], col["min_obs"])
            bounds, mean, na_bin, missing = b.get_numerical(f)
            assert np.array_equal(bounds.view(np.uint32), want.boundaries.view(np.uint32)), f"feature {f}: boundaries"
            assert F32(mean) == F32(want.mean) and mean == pytest.approx(want.mean, rel=1e-14, abs=1e-300), \
                f"feature {f}: mean {mean!r} != {want.mean!r}"
            assert na_bin == want.na_bin, f"feature {f}: NA bin {na_bin} != {want.na_bin}"
            assert missing == int(np.isnan(sample).sum()), f"feature {f}: missing {missing}"
            self.spec[f] = want
        ds = b.finish()
        cols = []
        for f, c in enumerate(self.raw):
            kind = c["kind"]
            if kind in ("num", "cat"):
                cols.append((kind, c["codes"][:n], c["B"], None))
            elif kind in E.DISC_KINDS:
                sp = self.spec[f]
                want = sp.encode16(c["x"][:n])
                if sp.wide:
                    got, nb, na = ds.get_wide_column(f)
                    assert (nb, na) == (sp.num_bins, sp.na_bin), (f, nb, na)
                    cols.append(("wide_num", got, sp.num_bins, None))
                else:
                    got = ds.get_bins(f)
                    cols.append(("num", got, sp.num_bins, None))
                assert np.array_equal(got.astype(np.uint16), want), \
                    f"feature {f}: {int((got != want).sum())} codes differ from the host rule"
                if stats is not None:
                    stats["binned"] += 1
                    stats["wide16" if sp.wide else "byte16" if kind == "disc16" else "byte8"] += 1
            else:
                cols.append(self._attach(ds, f, c, slice(0, n)))
        return ds, cols

    def _attach(self, ds, f, c, part):
        kind = c["kind"]
        if kind == "wide_num":
            v = np.ascontiguousarray(c["codes"][part])
            ds.set_wide_column(f, v, c["B"], 0, c["values"], float(c["values"][0]))
            return ("wide_num", v, c["B"], c["values"])
        if kind == "wide_cat":
            v = np.ascontiguousarray(c["codes"][part])
            ds.set_wide_categorical_column(f, v, c["B"], 0)
            return ("wide_cat", v, c["B"], None)
        ds.set_numerical_column(f, np.ascontiguousarray(c["values"][part]), 0.0)
        return ("pre", ds.get_numerical_column(f), 0, None)

    def _held_out(self):
        n, nv, F = self.n, self.n_valid, len(self.raw)
        part = slice(n, n + nv)
        bins = np.zeros((F, nv), np.uint8)
        nb, na, ft = np.ones(F, np.int32), np.zeros(F, np.int32), np.zeros(F, np.int32)
        codes = {}
        for f, c in enumerate(self.raw):
            kind = c["kind"]
            ft[f] = int(kind in ("cat", "wide_cat"))
            if kind in ("num", "cat"):
                bins[f], nb[f] = c["codes"][part], c["B"]
            elif kind in E.DISC_KINDS:
                sp = self.spec[f]
                codes[f] = sp.encode16(c["x"][part])
                if not sp.wide:
                    bins[f], nb[f], na[f] = codes[f], sp.num_bins, sp.na_bin
        ds = ydf_b200.Dataset(bins, nb, na, feature_types=ft)
        cols = []
        for f, c in enumerate(self.raw):
            kind = c["kind"]
            if kind in ("num", "cat"):
                cols.append((kind, bins[f], c["B"], None))
            elif kind in E.DISC_KINDS:
                sp = self.spec[f]
                if sp.wide:
                    ds.set_wide_discretized_column(f, codes[f], sp.num_bins, sp.na_bin)
                    cols.append(("wide_num", codes[f], sp.num_bins, None))
                else:
                    cols.append(("num", bins[f], sp.num_bins, None))
            else:
                cols.append(self._attach(ds, f, c, part))
        return ds, cols

    def margin(self, rng, scale):
        w = rng.normal(size=self.signal.shape[0])
        return scale * (w[:, None] * self.signal).sum(axis=0) + rng.normal(scale=0.7, size=self.signal.shape[1])

    def model_spec(self, vcols):
        """Per feature (DataSpec column, held-out raw values): the discretized columns with their boundaries and raw
        floats, byte and wide codes as DiscretizedColumns of one bin per code, categories as strings, presorted columns
        with their stored values."""
        out = []
        for f, c in enumerate(self.raw):
            kind, name = c["kind"], f"f{f}"
            if kind in E.DISC_KINDS:
                out.append((self.spec[f], c["x"][self.n:]))
            elif kind in ("num", "wide_num"):
                B = c["B"]
                col = dataspec.DiscretizedColumn(name=name, boundaries=(np.arange(1, B) - 0.5).astype(F32), mean=0.0,
                                                 num_bins=B, na_bin=0)
                out.append((col, vcols[f][1].astype(F32)))
            elif kind in ("cat", "wide_cat"):
                B = c["B"]
                col = dataspec.CategoricalColumn(name=name, vocabulary=["<OOD>"] + [str(i) for i in range(1, B)],
                                                 counts=[0] * B, num_bins=B, na_bin=0)
                out.append((col, np.array([str(int(v)) if v else "<OOD>" for v in vcols[f][1]], dtype=object)))
            else:
                v = vcols[f][1]
                col = dataspec.PresortedColumn(name=name, mean=0.0, min_value=float(v.min()) if len(v) else 0.0,
                                               max_value=float(v.max()) if len(v) else 0.0)
                out.append((col, v))
        return out


class ExtCase(X.Case):
    """A draw's builder tables, labels and weights, and its handles (with DART when drawn)."""

    def __init__(self, d, stats=None):
        super().__init__(d, ExtTable(d, stats))

    def handle(self, **override):
        gbt, cfg = super().handle(**override)
        if self.d["dart"] is not None:
            gbt.set_dart(self.d["dart"])
        return gbt, cfg


# ---------------------------------------------------------------------------------------------------------------------
# one case

def new_stats():
    return dict(trees=0, nodes=0, candidates=0, scan_trees=0, dart_scan_trees=0, skipped=0, flags=0, renamed=0,
                unresolved=0, binned=0, byte8=0, byte16=0, wide16=0, disc_splits=0, model_checks=0)


def run_case(seed):
    """Checks one draw; raises AssertionError on the first mismatch.  -> counts of what was checked."""
    d = E.draw(seed)
    stats = new_stats()
    case = ExtCase(d, stats)
    if d["dart"] is not None:
        gbt = _dart_early_stopping_case(case, stats) if d["drive"] == "train" else _dart_case(case, stats)
    elif d["cfg"]["early_stopping"]:
        gbt = X._early_stopping_case(case, stats)
    elif d["replay"]:
        gbt = X._replay_case(case, stats)
    else:
        gbt = X._plain_case(case, stats)
    _check_model(case, gbt, stats)
    return stats


def _tables(table):
    out = [(table.ds, table.cols, table.n)]
    if table.n_valid:
        out.append((table.vds, table.vcols, table.n_valid))
    return out


def _leaves(gbt, trees, cols, m, wide_cat):
    """[trees, m] leaf value of every row of a table in each of `trees` (tree index, tree)."""
    out = np.zeros((len(trees), m), F32)
    for i, (t, tree) in enumerate(trees):
        sets = gbt.get_category_sets(t, tree) if wide_cat else {}
        out[i] = tree["leaf_value"][R.leaf_of_rows(tree, R.route(tree, cols, sets), m)]
    return out


def _dart_case(case, stats):
    d, table = case.d, case.table
    gbt, cfg = case.handle()
    on_tree = X.scan_checker(gbt, cfg, d, table, stats)
    scan_before = stats["scan_trees"]
    check_dart_run(gbt, cfg, table, case.y, d["dart"], d["iters"], vlabels=case.vy, weights=case.w, vweights=case.vw,
                   on_tree=on_tree)
    stats["dart_scan_trees"] += stats["scan_trees"] - scan_before
    if stats["scan_trees"] + stats["skipped"] >= MIN_TREES_FOR_SHARE:
        X.check_skipped_share(stats)
    K = d["K"]
    trees = [(t, gbt.get_tree(t)) for t in range(d["iters"] * K)]
    stats["nodes"] += sum(len(tr) for _, tr in trees)
    if table.n_valid:   # the scaled model on the held-out rows
        wide_cat = any(c[0] == "wide_cat" for c in table.cols)
        want = DR.scaled_sum(F32(gbt.initial_prediction()), _leaves(gbt, trees, table.vcols, table.n_valid, wide_cat),
                             gbt.dart_weights(), K)
        p = gbt.predict(table.vds)
        p = p[None] if K == 1 else p.T
        assert np.array_equal(p, want), f"predict(held-out) differs from the scaled model in {int((p != want).sum())} values"
    return gbt


def _dart_early_stopping_case(case, stats):
    d, table = case.d, case.table
    c = d["cfg"]
    gbt, cfg = case.handle()
    K, iters, loss = d["K"], d["iters"], c["loss"]
    gbt.train(iters)
    logged = gbt.num_iterations()
    losses = [gbt.validation_loss(i)[0] for i in range(logged)]
    want = D.early_stopping(losses, c["early_stopping"], c["early_stopping_num_trees_look_ahead"],
                            c["early_stopping_initial_iteration"], K, iters)
    assert logged == want["logged"], (logged, want)
    kept = gbt.num_trees()
    assert kept == want["kept_trees"], (kept, want)
    fl, trig = gbt.final_validation()   # (NaN on a one-row table of one class: its initial prediction is infinite)
    assert trig == want["triggered"] and np.array_equal(F32(fl), F32(want["final_loss"]), equal_nan=True), \
        ((fl, trig), want)
    dropped = [gbt.dart_dropped(i).tolist() for i in range(logged)]
    want_w = DR.weights_after(dropped)[:kept // K]
    assert np.array_equal(gbt.dart_weights(), want_w), (gbt.dart_weights(), want_w)
    # every logged loss from the accumulators replayed with the device's trees and dropped sets
    init = F32(gbt.initial_prediction())
    wide_cat = any(col[0] == "wide_cat" for col in table.cols)
    trees = [(t, gbt.get_tree(t)) for t in range(logged * K)]
    stats["trees"] += len(trees)
    stats["nodes"] += sum(len(tr) for _, tr in trees)
    w_pow2 = R.pow2_cover(np.max(case.w)) if case.w is not None else None
    vw_pow2 = R.pow2_cover(np.max(case.vw)) if case.vw is not None else None
    errs = []
    for (ds, cols, m), labels, w, wp, read in zip(_tables(table), (case.y, case.vy), (case.w, case.vw), (w_pow2, vw_pow2),
                                                  (gbt.train_loss, gbt.validation_loss)):
        leaves = _leaves(gbt, trees, cols, m, wide_cat)
        acc = DR.Accumulator(np.full((K, m), init, F32))
        for it in range(logged):
            acc.update(leaves[it * K:(it + 1) * K], dropped[it])
            errs += check_losses(read(it), loss, acc.acc, np.asarray(labels), w, wp, f"{read.__name__} {it}")
        # the model: the kept trees, scaled by the weights after the stop
        p = gbt.predict(ds)
        p = p[None] if K == 1 else p.T
        scaled = DR.scaled_sum(init, leaves[:kept], want_w, K)
        if not np.array_equal(p, scaled):
            errs.append(f"predict({m} rows) differs from the scaled model in {int((p != scaled).sum())} values")
    assert not errs, f"{len(errs)} mismatches:\n" + "\n".join(errs[:30])
    return gbt


def _check_model(case, gbt, stats):
    """na_value of every split on a discretized column; with a hold-out and a 16-bit column, the host model on the raw
    held-out floats and (one output) the saved model read back against ygg_gbt_predict."""
    d, table = case.d, case.table
    K = d["K"]
    trees = [gbt.get_tree(t) for t in range(gbt.num_trees())]
    for t, tree in enumerate(trees):
        for i, nd in enumerate(tree):
            f = int(nd["feature"])
            if f in table.spec:
                want = int(table.spec[f].na_bin >= int(nd["threshold_bin"]))
                assert int(nd["na_value"]) == want, \
                    f"tree {t} node {i}: na_value {nd['na_value']} on feature {f} (NA bin {table.spec[f].na_bin}, " \
                    f"threshold {nd['threshold_bin']})"
                stats["disc_splits"] += 1
    if not table.n_valid or not any(c["kind"] == "disc16" for c in table.raw):
        return
    model_trees = trees
    if d["dart"] is not None:   # the model holds the scaled leaves
        w = gbt.dart_weights()
        model_trees = []
        for t, tree in enumerate(trees):
            s = tree.copy()
            leaf = s["feature"] < 0
            s["leaf_value"][leaf] = (s["leaf_value"][leaf] * w[t // K]).astype(F32)
            model_trees.append(s)
    wide_cat = any(c[0] == "wide_cat" for c in table.cols)
    sets = [gbt.get_category_sets(t, tree) if wide_cat else {} for t, tree in enumerate(trees)]
    cols_raw = table.model_spec(table.vcols)
    loss = d["cfg"]["loss"]
    spec = dataspec.DataSpec(columns=[c for c, _ in cols_raw], label="y",
                             task="REGRESSION" if loss == 1 else "CLASSIFICATION",
                             label_classes=None if loss == 1 else [str(k) for k in range(1, K + 2 if loss == 0 else K + 1)])
    model = ydf_b200.GradientBoostedTreesModel(spec, model_trees, gbt.initial_prediction(), LOSS_NAMES[loss],
                                               category_sets=sets)
    raw = {c.name: v for c, v in cols_raw}
    got = gbt.predict(table.vds)
    host = model._raw(dataspec.encode_features(raw, spec.columns))
    assert np.array_equal(host, got), f"the host model on the raw held-out values differs in {int((host != got).sum())}"
    if K == 1:
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "m")
            model.save(path)
            saved = model_io.predict_ydf_model(model_io.read_ydf_model(path), raw)
        assert np.array_equal(saved, got), \
            f"the saved model on the raw held-out values differs in {int((saved != got).sum())} rows"
    stats["model_checks"] += 1


# ---------------------------------------------------------------------------------------------------------------------
# the suite

TOTALS = {}


@pytest.mark.parametrize("seed", list(SUITE_SEEDS))
def test_drawn_configuration_is_exact(seed):
    stats = run_case(seed)
    assert stats["trees"] > 0
    for k, v in stats.items():
        TOTALS[k] = TOTALS.get(k, 0) + v


def test_totals():
    """What the suite's cases checked (printed with -s; meaningful after the parametrized cases ran), and the share of
    scan-checkable trees skipped over the suite."""
    print("extended exact fuzz totals:", TOTALS)
    X.check_skipped_share(dict(scan_trees=TOTALS.get("scan_trees", 0), skipped=TOTALS.get("skipped", 0)))


def main(argv):
    n = int(argv[0]) if argv else 50
    offset = int(argv[1]) if len(argv) > 1 else SUITE_SEEDS.stop
    failures, totals = [], {}
    t0 = time.time()
    for seed in range(offset, offset + n):
        try:
            stats = run_case(seed)
        except Exception as e:   # a mismatch, or a refusal the drawer should have restated
            failures.append(seed)
            d = E.draw(seed)
            print(f"seed {seed} FAILED: {type(e).__name__}")
            print(f"  config: n={d['n']} n_valid={d['n_valid']} K={d['K']} dart={d['dart']} sampling={d['sampling']} "
                  f"weights={d['weights']} vweights={d['vweights']} candidates={d['candidates']} replay={d['replay']} "
                  f"drive={d['drive']} iters={d['iters']}")
            print(f"  cfg: {d['cfg']}")
            print(f"  columns: {[(c['kind'], c.get('B', c.get('max_bins')), c.get('values'), c.get('twin')) for c in d['columns']]}")
            print("  " + "\n  ".join(str(e).splitlines()[:12]))
            continue
        for k, v in stats.items():
            totals[k] = totals.get(k, 0) + v
        print(f"seed {seed} ok", flush=True)
    print(f"seeds {offset}..{offset + n - 1}: {n - len(failures)} passed, {len(failures)} failed {failures}; "
          f"{time.time() - t0:.0f} s; totals {totals}")
    try:
        X.check_skipped_share(dict(scan_trees=totals.get("scan_trees", 0), skipped=totals.get("skipped", 0)))
    except AssertionError:
        print("the share of skipped trees over the sweep is above", X.MAX_SKIPPED_SHARE)
        return 1
    return 1 if failures else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
