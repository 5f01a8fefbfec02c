"""Randomly drawn training configurations (tests/exact_fuzz_draw.py), checked exactly at every tree.

Every case runs the boosting reference (tests/test_gpu_boosting_exact.check_run) on every tree: gradients, row sample,
node statistics, leaves, training and held-out predictions, training and (weighted) validation losses.  On top of it:

- step()-driven level-wise cases without the tie-break replay capture every tree's candidates and check them against the
  exact scan (tests/test_gpu_scan_exact.check_scan) on the tree's trained rows and weights: every tree for K = 1, the
  last class of each iteration for K > 1 (the capture holds the last tree grown).  With candidate sampling the selection
  is the keyed one and every validity flag is checked against the node's trained rows (check_levels).  A tree whose
  gradients depend on a free exp rounding (boost_ref.exp_f32) is not scan-checked; such skips are counted.
- early stopping: EarlyStoppingState and ygg_gbt_train's finalisation are restated on the reported validation losses;
  num_trees(), num_iterations(), final_validation(), the refusal of unlogged iterations, and predict() on both tables
  (the kept trees only) follow it, while every trained tree (whole batches of 8 iterations) is still checked.
- tie-break replay: the same data trained without the replay (capturing the candidates) and with it must give the same
  trees except at renamed nodes, where only the condition may change, and the same training losses and predictions.
  For K = 1 the renamed nodes and tie_stats() must equal the restated replay (exact_fuzz_draw.tie_expectation).  The
  multinomial replay cases get the comparison without the restatement: the capture only holds the last class's tree.

`python -m tests.test_gpu_exact_fuzz N [offset]` runs seeds offset .. offset + N - 1 and prints every failing
configuration with its first mismatches."""
import sys
import time

import numpy as np
import pytest

import ydf_b200
from oracle import oracle as O
from tests import candidate_sampling_ref as CS
from tests import exact_fuzz_draw as D
from tests.test_gpu_boosting_exact import check_run, labels_for
from tests.test_gpu_candidate_sampling import check_levels, k_valid
from tests.test_gpu_scan_exact import check_scan

pytestmark = pytest.mark.gpu

F32 = np.float32
SUITE_SEEDS = D.SUITE_SEEDS
MAX_SKIPPED_SHARE = 0.25   # of the scan-checked trees of a case (a first run of the suite skipped none in 40 seeds)


class FuzzTable:
    """The training and held-out tables of a draw, in the shape check_run reads (n, n_valid, ds, cols, vds, vcols)."""

    def __init__(self, d):
        rng = np.random.default_rng([d["seed"], 1])
        self.n, self.n_valid = d["n"], d["n_valid"]
        self.raw = D.make_columns(d, rng, self.n + self.n_valid)
        self.ds, self.cols = self._make(slice(0, self.n))
        self.vds, self.vcols = self._make(slice(self.n, self.n + self.n_valid)) if self.n_valid else (None, None)
        self.signal = np.stack([D.signal(c) for c in self.raw])

    def _make(self, part):
        F, m = len(self.raw), part.stop - part.start
        bins = np.zeros((F, m), np.uint8)
        nb, ft = np.ones(F, np.int32), np.zeros(F, np.int32)
        for f, c in enumerate(self.raw):
            if c["kind"] in ("num", "cat"):
                bins[f], nb[f] = c["codes"][part], c["B"]
            ft[f] = 1 if c["kind"] in ("cat", "wide_cat") else 0
        ds = ydf_b200.Dataset(bins, nb, np.zeros(F, np.int32), feature_types=ft)
        cols = []
        for f, c in enumerate(self.raw):
            if c["kind"] in ("num", "cat"):
                cols.append((c["kind"], bins[f], c["B"], None))
            elif c["kind"] == "wide_num":
                v = np.ascontiguousarray(c["codes"][part])
                ds.set_wide_column(f, v, c["B"], 0, c["values"], float(c["values"][0]))
                cols.append(("wide_num", v, c["B"], c["values"]))
            elif c["kind"] == "wide_cat":
                v = np.ascontiguousarray(c["codes"][part])
                ds.set_wide_categorical_column(f, v, c["B"], 0)
                cols.append(("wide_cat", v, c["B"], None))
            else:
                ds.set_numerical_column(f, np.ascontiguousarray(c["values"][part]), 0.0)
                cols.append(("pre", ds.get_numerical_column(f), 0, None))
        return ds, cols

    def margin(self, rng, scale):
        w = rng.normal(size=self.signal.shape[0])
        return scale * (w[:, None] * self.signal).sum(axis=0) + rng.normal(scale=0.7, size=self.signal.shape[1])


def _weights(rng, m):
    w = rng.uniform(0.1, 3.0, size=m).astype(F32)
    w[rng.random(m) < 0.05] = 0.0
    if not w.any():
        w[0] = 1.0
    return w


class Case:
    """A draw's data, labels and weights, and the handles trained on them."""

    def __init__(self, d, table=None):
        self.d = d
        self.table = FuzzTable(d) if table is None else table
        rng = np.random.default_rng([d["seed"], 2])
        m = self.table.margin(rng, d["scale"])
        if d["scale"] >= 1e3:
            m = m + 1e3
        y = labels_for(d["cfg"]["loss"], m, d["K"])
        n = d["n"]
        self.y, self.vy = y[:n], (y[n:] if d["n_valid"] else None)
        self.w = _weights(rng, n) if d["weights"] else None
        self.vw = _weights(rng, d["n_valid"]) if d["vweights"] else None

    def handle(self, **override):
        d = self.d
        cfg = ydf_b200.default_config(**{**d["cfg"], **override})
        gbt = ydf_b200.Gbt(self.table.ds, cfg)
        if self.w is not None:
            gbt.set_weights(self.w)
        gbt.set_labels(self.y)
        if self.vy is not None:
            gbt.set_validation(self.table.vds, self.vy, self.vw)
        if d["candidates"] is not None:
            gbt.set_candidate_sampling(*d["candidates"])
        return gbt, cfg


# ---------------------------------------------------------------------------------------------------------------------
# one case

def run_case(seed):
    """Checks one draw; raises AssertionError on the first mismatch.  -> counts of what was checked."""
    d = D.draw(seed)
    case = Case(d)
    stats = dict(trees=0, nodes=0, candidates=0, scan_trees=0, skipped=0, flags=0, renamed=0, unresolved=0)
    if d["cfg"]["early_stopping"]:
        _early_stopping_case(case, stats)
    elif d["replay"]:
        _replay_case(case, stats)
    else:
        _plain_case(case, stats)
    return stats


def _plain_case(case, stats):
    d, table = case.d, case.table
    gbt, cfg = case.handle()
    checked, _ = check_run(gbt, cfg, table, case.y, case.vy, weights=case.w, iters=d["iters"],
                           step=d["drive"] == "step", vweights=case.vw, on_tree=scan_checker(gbt, cfg, d, table, stats))
    stats["nodes"] += checked
    check_skipped_share(stats)
    if d["n_valid"]:
        # without early stopping the model is whole: the last iteration's loss, not triggered
        got = gbt.final_validation()
        assert got == (gbt.validation_loss(d["iters"] - 1)[0], False), got
    return gbt


def scan_checker(gbt, cfg, d, table, stats):
    """The on_tree callback of check_run (and tests/test_gpu_dart.check_dart_run) that checks the captured candidates
    of the draw's trees against the exact scan, where the draw allows the capture (which it turns on)."""
    capture = D.capture_allowed(d)
    K = d["K"]
    kv = k_valid(cfg, d["F"], *d["candidates"]) if d["candidates"] is not None else None
    sampled = kv is not None and CS.num_candidate_attributes(d["F"], cfg.loss, *d["candidates"]) < d["F"]
    if capture:
        gbt.capture_candidates(True)

    def on_tree(t, rows):
        stats["trees"] += 1
        if not capture or t % K != K - 1:
            return
        sel = rows["sel"]
        on = np.ones(table.n, bool) if sel is None else sel
        free = (rows["g"] != rows["g_alt"])
        if rows["h"] is not None:
            free |= rows["h"] != rows["h_alt"]
        if (free & on).any():
            stats["skipped"] += 1
            return
        select = None
        if sampled:
            def select(level, j, cap):
                tried, first = gbt.level_tried(level)
                return CS.select(cfg.random_seed, t, first + j, tried[j], cap["found"][j], cap["score"][j], kv)
        h = None if rows["w"] is not None or cfg.loss == 1 else rows["h"]
        stats["candidates"] += check_scan(gbt, cfg, rows["tree"], table.cols, rows["g"], h, w=rows["w"], tree_index=t,
                                          sel=sel, select=select)
        stats["scan_trees"] += 1
        if sampled:
            _, flags, _ = check_levels(gbt, cfg, rows["tree"], t, kv, cols=table.cols, g=rows["g"], h=h, sel=sel,
                                       w=rows["w"], trained_tree=True)
            stats["flags"] += flags

    return on_tree


def check_skipped_share(stats):
    if stats["scan_trees"] + stats["skipped"]:
        assert stats["skipped"] <= MAX_SKIPPED_SHARE * (stats["scan_trees"] + stats["skipped"]), stats


def _early_stopping_case(case, stats):
    d, table = case.d, case.table
    c = d["cfg"]
    gbt, cfg = case.handle()
    K, iters = d["K"], d["iters"]
    gbt.train(iters)
    logged = gbt.num_iterations()
    losses = [gbt.validation_loss(i)[0] for i in range(logged)]
    want = D.early_stopping(losses, c["early_stopping"], c["early_stopping_num_trees_look_ahead"],
                            c["early_stopping_initial_iteration"], K, iters)
    assert logged == want["logged"], (logged, want)
    assert gbt.num_trees() == want["kept_trees"], (gbt.num_trees(), want)
    fl, trig = gbt.final_validation()
    assert (F32(fl), trig) == (F32(want["final_loss"]), want["triggered"]), ((fl, trig), want)
    for bad in (logged, want["trained"]):
        for read in (gbt.validation_loss, gbt.train_loss):
            with pytest.raises(ydf_b200.YggError) as e:
                read(bad)
            assert e.value.code == 1
    # every trained tree exists (whole batches), none past them
    gbt.get_tree(want["trained"] * K - 1)
    with pytest.raises(ydf_b200.YggError):
        gbt.get_tree(want["trained"] * K)
    checked, _ = check_run(gbt, cfg, table, case.y, case.vy, weights=case.w, iters=want["trained"], vweights=case.vw,
                           trained=True, logged=logged, kept_trees=want["kept_trees"],
                           on_tree=lambda t, rows: stats.__setitem__("trees", stats["trees"] + 1))
    stats["nodes"] += checked
    return gbt


# what a rename may change: the whole condition, its kind included (on a small node a numerical column can send the
# rows exactly like a categorical one)
CONDITION = ("feature", "condition_type", "threshold_bin", "na_value", "cat_mask", "threshold_value")


def _replay_case(case, stats):
    d, table = case.d, case.table
    K, iters, F = d["K"], d["iters"], d["F"]
    # mode 0, stepped, with the candidates of every tree (K = 1)
    base, cfg0 = case.handle(candidate_shuffle=0)
    base.capture_candidates(True)
    cands, base_trees = [], []
    for _ in range(iters):
        base.step()
        for k in range(K):
            t = len(base_trees)
            base_trees.append(base.get_tree(t))
        if K == 1:
            cands.append(_tie_candidates(base, cfg0, base_trees[-1], len(base_trees) - 1, table))
    gbt, cfg = case.handle()
    checked, _ = check_run(gbt, cfg, table, case.y, case.vy, weights=case.w, iters=iters, step=d["drive"] == "step",
                           vweights=case.vw, on_tree=lambda t, rows: stats.__setitem__("trees", stats["trees"] + 1))
    stats["nodes"] += checked
    renamed = {}
    for t in range(iters * K):
        a, b = base_trees[t], gbt.get_tree(t)
        assert len(a) == len(b), t
        diff = np.flatnonzero(np.array([a[i].tobytes() != b[i].tobytes() for i in range(len(a))], bool))
        for i in diff:
            other = [k for k in a.dtype.names if k not in CONDITION and not np.array_equal(a[i][k], b[i][k])]
            assert not other, f"tree {t} node {i}: more than the condition: {[(k, a[i][k], b[i][k]) for k in other]}"
            assert a[i]["feature"] != b[i]["feature"], f"tree {t} node {i}: same feature, other condition"
            renamed[(t, int(i))] = int(b[i]["feature"])
    for it in range(iters):
        assert base.train_loss(it) == gbt.train_loss(it), it
    assert np.array_equal(base.get_predictions(), gbt.get_predictions())
    ties = gbt.tie_stats()
    assert ties[0] == len(renamed), (ties, renamed)
    if K == 1:
        rng = O.Rng(int(cfg.random_seed))
        rng.discard(int(cfg.rng_words_consumed))
        want, n_renamed, n_unresolved = D.tie_expectation(base_trees, cands, rng, d["replay"],
                                                          int(cfg.split_jobs_draw_seeds), F)
        assert renamed == want, (renamed, want)
        assert ties == (n_renamed, n_unresolved), (ties, n_renamed, n_unresolved)
    stats["renamed"] += ties[0]
    stats["unresolved"] += ties[1]
    return gbt


def _tie_candidates(gbt, cfg, tree, t, table):
    """{pre-order node: (found, score, went_pos)} of the captured candidate nodes of tree t, the last one grown."""
    from tests.boost_ref import route
    rows_of = route(tree, table.cols, gbt.get_category_sets(t, tree))
    out = {}
    for level in range(cfg.max_depth - 1):
        cap = gbt.level_candidates(level)
        for j in range(len(cap["node"])):
            if not cap["candidate"][j]:
                continue
            pre = int(cap["node"][j])
            rows = rows_of[pre]

            def went_pos(f, j=j, rows=rows, cap=cap):
                kind, codes, _, _ = table.cols[f]
                if kind == "wide_cat":
                    return None
                if kind == "pre":
                    return codes[rows] >= cap["threshold_value"][j, f]
                if kind == "cat":
                    b = codes[rows].astype(np.int64)
                    return ((cap["cat_mask"][j, f][b >> 5] >> (b & 31).astype(np.uint32)) & 1) != 0
                return codes[rows].astype(np.int64) >= cap["threshold_bin"][j, f]
            out[pre] = (cap["found"][j].copy(), cap["score"][j].copy(), went_pos)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the suite

TOTALS = {}


@pytest.mark.parametrize("seed", list(SUITE_SEEDS))
def test_drawn_configuration_is_exact(seed):
    stats = run_case(seed)
    assert stats["trees"] > 0
    for k, v in stats.items():
        TOTALS[k] = TOTALS.get(k, 0) + v


def test_every_draw_of_the_suite_is_accepted():
    """Every draw of the suite's seed range builds its tables and a handle with all its settings."""
    for seed in SUITE_SEEDS:
        d = D.draw(seed)
        case = Case(d)
        gbt, _ = case.handle()
        if D.capture_allowed(d):
            gbt.capture_candidates(True)
        gbt.close()


def test_presorted_column_against_a_byte_column_is_refused():
    """A model trained with feature 1 presorted refuses a table whose feature 1 is a one-bucket byte column, in predict()
    and as validation rows: the two kinds route rows by different data (feature types 2 and 0)."""
    rng = np.random.default_rng(3)
    n = 2000
    bins = rng.integers(0, 8, size=(2, n)).astype(np.uint8)
    nb = np.array([8, 1], np.int32)
    ds = ydf_b200.Dataset(bins * np.array([[1], [0]], np.uint8), nb, np.zeros(2, np.int32))
    ds.set_numerical_column(1, rng.normal(size=n).astype(F32), 0.0)
    other = ydf_b200.Dataset(bins * np.array([[1], [0]], np.uint8), nb, np.zeros(2, np.int32))
    y = (bins[0] > 3).astype(np.int32) + 1
    cfg = ydf_b200.default_config(loss=0, max_depth=3, num_trees=2)
    gbt = ydf_b200.Gbt(ds, cfg)
    gbt.set_labels(y)
    with pytest.raises(ydf_b200.YggError) as e:
        gbt.set_validation(other, y)
    assert e.value.code == 1
    gbt.train(1)
    with pytest.raises(ydf_b200.YggError) as e:
        gbt.predict(other)
    assert e.value.code == 1


def test_totals():
    """What the suite's cases checked (printed with -s; meaningful after the parametrized cases ran)."""
    print("exact fuzz totals:", TOTALS)


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
            d = D.draw(seed)
            print(f"seed {seed} FAILED: {type(e).__name__}")
            print(f"  config: n={d['n']} n_valid={d['n_valid']} K={d['K']} sampling={d['sampling']} "
                  f"weights={d['weights']} vweights={d['vweights']} candidates={d['candidates']} replay={d['replay']} "
                  f"drive={d['drive']} iters={d['iters']}")
            print(f"  cfg: {d['cfg']}")
            print(f"  columns: {[(c['kind'], c.get('B'), c.get('twin')) for c in d['columns']]}")
            print("  " + "\n  ".join(str(e).splitlines()[:12]))
            continue
        for k, v in stats.items():
            totals[k] = totals.get(k, 0) + v
        print(f"seed {seed} ok", flush=True)
    print(f"seeds {offset}..{offset + n - 1}: {n - len(failures)} passed, {len(failures)} failed {failures}; "
          f"{time.time() - t0:.0f} s; totals {totals}")
    return 1 if failures else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
