"""Sharded training checked exactly, on one GPU through the in-process fake communicator of tests/test_gpu_sharding.py.

Every case first trains the single-rank run and checks it against the exact boosting reference
(tests/test_gpu_boosting_exact.check_run: every node's counts and statistics, leaves, predictions and losses), then
trains the same table in a shard mode:
  * rows         : integer level histograms all-reduced;
  * rows_scatter : reduce-scattered by feature chunk (the fake poisons the chunks a rank does not own), bests all-gathered;
  * features     : every rank holds every row and scans its features, bests all-gathered.
Each rank must give the single-rank run's tree bytes and categorical sets, its slice of the training predictions (all
of them for feature shards), the single-rank predict() on the whole table, accuracies equal and losses within 1 float
ulp (the order of the double sums is the only freedom).

The row splits are adversarial: rows ordered by the bins of the informative column or by label before the cut, ranks of
1, 8191, 8192 and 8193 rows, the largest |label| or weight on one rank, a heavy bin on one rank only (a different
histogram layout per rank).  A rank decision that reads a local quantity where the job's is needed (which child is
histogrammed, min_examples, the root candidate, purity, the gradient and weight scales, a node empty on one rank) shows
up as a tree that differs.  Then drawn configurations (tests/shard_draw.py) and the setters' call orders, whose refusals
must come before any collective."""
import ctypes as C

import numpy as np
import pytest

import ydf_b200
from tests import boost_ref as R
from tests import shard_draw as SD
from tests.test_gpu_boosting_exact import check_run, labels_for
from tests.test_gpu_sharding import FakeComm, _run_ranks

pytestmark = pytest.mark.gpu

F32 = np.float32
INVALID, UNIMPLEMENTED = 1, 4


class CountingComm(FakeComm):
    """The fake communicator, counting every collective call per rank and kind."""

    def __init__(self, world):
        super().__init__(world)
        self.calls = [dict(allreduce=0, reducescatter=0, allgather=0) for _ in range(world)]

    def _counted(self, kind, rank, fn):
        def call(*a):
            self.calls[rank][kind] += 1
            return fn(*a)
        return call

    def allreduce(self, rank):
        return self._counted("allreduce", rank, super().allreduce(rank))

    def reducescatter(self, rank):
        return self._counted("reducescatter", rank, super().reducescatter(rank))

    def allgather(self, rank):
        return self._counted("allgather", rank, super().allgather(rank))

    def total(self, rank=None):
        ranks = range(self.world) if rank is None else [rank]
        return sum(sum(self.calls[r].values()) for r in ranks)


class LoneComm(CountingComm):
    """For call orders that must be refused: a collective is counted and fails at once instead of waiting for the
    other ranks, so a refusal that comes too late shows as a count, never as a wait."""

    def _counted(self, kind, rank, fn):
        def call(*a):
            self.calls[rank][kind] += 1
            return 1
        return call


# ---------------------------------------------------------------------------------------------------------------------
# tables

class ShardTable:
    """Byte columns in the shape check_run reads (n, n_valid, ds, cols, vds, vcols), cut into per-rank datasets.
    columns: dicts kind 'num' / 'cat', B, and for 'num' optional exact (bucket values: the exact threshold rule) and
    const (one bucket value for every row)."""

    def __init__(self, rng, n, columns):
        self.n, self.n_valid, self.vds, self.vcols = n, 0, None, None
        F = len(columns)
        self.bins = np.zeros((F, n), np.uint8)
        self.nb = np.array([c["B"] for c in columns], np.int32)
        self.ft = np.array([1 if c["kind"] == "cat" else 0 for c in columns], np.int32)
        self.values = {}
        for f, c in enumerate(columns):
            B = c["B"]
            if c["kind"] == "cat":
                p = 1.0 / np.arange(1, B + 1) ** 1.1
                self.bins[f] = rng.choice(B, size=n, p=p / p.sum())
            elif c.get("const"):
                self.bins[f] = int(rng.integers(0, B))
            else:
                self.bins[f] = np.clip(((rng.normal(size=n) + 3) / 6 * B).astype(np.int64), 0, B - 1)
            if c["kind"] == "num" and c.get("exact"):
                self.values[f] = np.cumsum(rng.uniform(0.1, 1.0, size=B)).astype(F32)
        self.signal = (self.bins - self.bins.mean(axis=1, keepdims=True)) / (self.bins.std(axis=1, keepdims=True) + 1e-9)
        self.finish()

    def reorder(self, order):
        """The table's rows in `order` (the adversarial cuts are contiguous slices of the reordered table)."""
        self.bins = np.ascontiguousarray(self.bins[:, order])
        self.signal = self.signal[:, order]
        self.finish()

    def finish(self):
        self.ds = self.dataset(0, self.n)
        self.cols = [("cat" if self.ft[f] else "num", self.bins[f], int(self.nb[f]), self.values.get(f))
                     for f in range(len(self.nb))]

    def dataset(self, r0, r1):
        ds = ydf_b200.Dataset(self.bins[:, r0:r1], self.nb, np.zeros(len(self.nb), np.int32), feature_types=self.ft)
        for f, v in self.values.items():
            ds.set_bucket_values(f, v, v[0])
        return ds

    def margin(self, rng, scale=1.0, lead=None):
        w = rng.normal(size=self.signal.shape[0])
        if lead is not None:   # one column carries most of the signal
            w[lead] = 4.0
        return scale * (w[:, None] * self.signal).sum(axis=0) + rng.normal(scale=0.7, size=self.n)


def category_words(gbt, t, tree):
    """{pre-order node: ygg_gbt_get_category_set words} of tree t's categorical splits."""
    out = {}
    for i in np.flatnonzero((tree["condition_type"] == 1) & (tree["feature"] >= 0)):
        words = np.zeros(8, np.uint32)
        n = C.c_int32()
        status = ydf_b200.lib().ygg_gbt_get_category_set(gbt.handle, C.c_int32(t), C.c_int32(int(i)),
                                                         words.ctypes.data_as(C.POINTER(C.c_uint32)), C.c_int32(8),
                                                         C.byref(n))
        assert status == 0, ydf_b200.lib().ygg_last_error()
        out[int(i)] = words[:n.value].tobytes()
    return out


def _train(gbt, iters, drive):
    if drive == "train":
        gbt.train(iters)
    else:
        for _ in range(iters):
            gbt.step()
        gbt.sync()


def _result(gbt, iters, full_ds):
    trees = [gbt.get_tree(t) for t in range(iters)]
    return dict(trees=[t.tobytes() for t in trees], sets=[category_words(gbt, i, t) for i, t in enumerate(trees)],
                losses=[gbt.train_loss(i) for i in range(iters)], pred=gbt.get_predictions(),
                predict=gbt.predict(full_ds), nodes=sum(len(t) for t in trees))


STATS = dict(cases=0, single_nodes=0, shard_rank_runs=0, shard_nodes=0)


def run_case(table, cfg_kw, y, w=None, mode="rows", world=2, cuts=None, iters=3, drive="train", on_ranks=None):
    """The single-rank run checked against the reference, then `mode` over `world` ranks holding `cuts` (row ranges of
    the table; default: equal slices) compared with it.  on_ranks(handles): called in each rank's thread after training.
    -> (single-rank result, per-rank results, the communicator)."""
    cfg = ydf_b200.default_config(**cfg_kw)
    one = ydf_b200.Gbt(table.ds, cfg)
    if w is not None:
        one.set_weights(w)
    one.set_labels(y)
    nodes, _ = check_run(one, cfg, table, y, weights=w, iters=iters, step=drive == "step")
    want = _result(one, iters, table.ds)
    init = one.initial_prediction()
    n = table.n
    if cuts is None:
        cuts = [((n * r) // world, (n * (r + 1)) // world) for r in range(world)] if mode != "features" else [(0, n)] * world
    comm = CountingComm(world)
    handles = [None] * world

    def rank_main(r):
        r0, r1 = cuts[r]
        ds = table.dataset(r0, r1)
        gbt = ydf_b200.Gbt(ds, cfg)
        handles[r] = gbt
        if w is not None:
            gbt.set_weights(w[r0:r1])
        gbt.set_labels(y[r0:r1])
        if mode == "rows":
            gbt.set_row_shard(r, world, n, init, comm.allreduce(r))
        elif mode == "rows_scatter":
            gbt.set_row_shard_scatter(r, world, n, init, allreduce=comm.allreduce(r), reducescatter=comm.reducescatter(r),
                                      allgather=comm.allgather(r))
        else:
            b, e = ydf_b200.feature_shard(len(table.nb), r, world)
            gbt.set_feature_shard(b, e, r, world, comm.allgather(r))
        _train(gbt, iters, drive)
        out = _result(gbt, iters, table.ds)
        if on_ranks is not None:
            out["extra"] = on_ranks(gbt)
        return out

    res = _run_ranks(world, rank_main, comm)
    loss = int(cfg.loss)
    for r, got in enumerate(res):
        where = f"{mode} rank {r} of {world} ({cuts[r][1] - cuts[r][0]} rows)"
        for t in range(iters):
            assert got["trees"][t] == want["trees"][t], f"{where}: tree {t} differs from the single-rank run"
            assert got["sets"][t] == want["sets"][t], f"{where}: categorical sets of tree {t} differ"
        r0, r1 = cuts[r]
        assert np.array_equal(got["pred"], want["pred"][r0:r1]), f"{where}: training predictions differ"
        assert np.array_equal(got["predict"], want["predict"]), f"{where}: predict() on the whole table differs"
        for i, ((l, s), (wl, ws)) in enumerate(zip(got["losses"], want["losses"])):
            assert abs(float(l) - float(wl)) <= R.ulp32(F32(wl)), f"{where}: loss {i}: {l!r} vs {wl!r}"
            if loss == 1:
                assert abs(float(s) - float(ws)) <= R.ulp32(F32(ws)), f"{where}: secondary {i}: {s!r} vs {ws!r}"
            else:
                assert s == ws, f"{where}: accuracy {i}: {s!r} vs {ws!r}"
    STATS["cases"] += 1
    STATS["single_nodes"] += nodes
    STATS["shard_rank_runs"] += world
    STATS["shard_nodes"] += sum(g["nodes"] for g in res)
    return want, res, comm


# ---------------------------------------------------------------------------------------------------------------------
# adversarial row splits

LAYOUT = [dict(kind="num", B=255), dict(kind="cat", B=40), dict(kind="num", B=64, exact=True), dict(kind="cat", B=256),
          dict(kind="num", B=16), dict(kind="num", B=200), dict(kind="cat", B=7)]   # 7 features: 4 scatter chunks
ROW_MODES = ["rows", "rows_scatter"]


def _table(seed, n, layout=LAYOUT):
    rng = np.random.default_rng(seed)
    return rng, ShardTable(rng, n, layout)


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("mode", ROW_MODES)
def test_rows_ordered_by_the_informative_column(mode, world):
    """Each rank holds a narrow range of column 0's bins: many nodes have no local rows on some ranks (empty segments of
    k_hist_seg, no rows in k_partition, empty level lists), and each rank's row counts of a split differ from the job's."""
    rng, table = _table(11 + world, 40000)
    m = table.margin(rng, lead=0)
    order = np.argsort(table.bins[0], kind="stable")
    table.reorder(order)
    y = labels_for(1, m[order] * 3.0).astype(F32)
    run_case(table, dict(loss=1, max_depth=9, min_examples=2), y, mode=mode, world=world)


def _sorted_table(seed, n, key_fn):
    rng = np.random.default_rng(seed)
    table = ShardTable(rng, n, LAYOUT)
    m = table.margin(rng, lead=0)
    order = key_fn(table, m)
    table.reorder(order)
    return rng, table, m[order]


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("mode", ROW_MODES)
def test_rows_ordered_by_bin_binomial_hessian(mode, world):
    """The same cut with the binomial loss and the hessian gain, depth 10 with sibling subtraction (multi-pass slot
    windows on the deep levels, all-reduced or reduce-scattered after the passes)."""
    rng, table, m = _sorted_table(21 + world, 40000, lambda t, m: np.argsort(t.bins[0], kind="stable"))
    y = labels_for(0, m)
    run_case(table, dict(loss=0, use_hessian_gain=1, max_depth=10, min_examples=1, l2_regularization=1.0), y, mode=mode,
             world=world, iters=2)


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("mode", ROW_MODES)
def test_binomial_rows_ordered_by_label(mode, world):
    """Rank 0 holds only negatives: its nodes are pure locally but not in the job."""
    rng, table, m = _sorted_table(31 + world, 30000, lambda t, m: np.argsort(m, kind="stable"))
    y = labels_for(0, m)
    assert (y[:30000 // world] == 1).all() and (y[-(30000 // world):] == 2).all()
    run_case(table, dict(loss=0, max_depth=7, min_examples=5), y, mode=mode, world=world)


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("mode", ROW_MODES)
def test_tiny_and_uneven_ranks(mode, world):
    """Ranks of 1, 8191 and 8192 rows in turn around the 8192-row block, the rest (8193 and more) on the last rank;
    min_examples 40 with the in-split check off (the checks read the job's counts, never a rank's)."""
    n = 8192 * 3 + 9000
    rng, table = _table(41 + world, n)
    y = labels_for(1, table.margin(rng, 2.0)).astype(F32)
    d = dict(n=n, world=world, mode=mode, split="tiny")
    cuts = SD.cuts(d)
    assert [e - b for b, e in cuts][:world - 1] == list(SD.TINY[:world - 1])
    run_case(table, dict(loss=1, max_depth=6, min_examples=40, in_split_min_examples_check=0), y, mode=mode, world=world,
             cuts=cuts, drive="step")


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("mode", ROW_MODES)
def test_largest_label_on_the_last_rank(mode, world):
    """Squared error whose largest |label| (and so max|g|, the gradient scale P of every tree) lives on the last rank
    only: P must be the job's (the gmax_bits all-reduce)."""
    rng, table = _table(51 + world, 30000)
    y = labels_for(1, table.margin(rng, 3.0)).astype(F32)
    y[np.argmax(np.abs(y))] = F32(400.0)
    order = np.argsort(np.abs(y), kind="stable")   # ascending: the outlier is the last row
    table.reorder(order)
    y = y[order]
    run_case(table, dict(loss=1, max_depth=6, min_examples=1, shrinkage=1.0), y, mode=mode, world=world)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("mode", ROW_MODES)
@pytest.mark.parametrize("loss", [0, 1])
def test_weights_skewed_over_the_ranks(mode, world, loss):
    """The largest weight on rank 0 only, and most of the zero weights on the last rank: the weight scale, the weight
    sums and the scale of max|w*g| are the job's."""
    n = 30000
    rng, table = _table(61 + world + 10 * loss, n)
    m = table.margin(rng, 2.0)
    w = rng.uniform(0.1, 2.0, size=n).astype(F32)
    w[rng.random(n) < 0.2] = 0.0
    w[np.argmax(w)] = F32(9.0)
    order = np.lexsort((-w, w == 0))   # non-zero weights first, largest weight first; zeros at the end
    table.reorder(order)
    w, m = w[order], m[order]
    assert w[0] == 9.0 and (w[-(n // world):] == 0).sum() > 0.5 * (w == 0).sum()
    y = labels_for(loss, m).astype(F32 if loss == 1 else np.int32)
    run_case(table, dict(loss=loss, max_depth=6, min_examples=3), y, w=w, mode=mode, world=world)


@pytest.mark.parametrize("mode", ROW_MODES)
def test_heavy_bin_on_one_rank_changes_its_histogram_layout(mode):
    """Column 1 holds one category on rank 0's first 12000 rows: a whole 8192-row block in one bin exceeds the packed
    words' bound on rank 0 only, whose deeper levels fall back to the carry-detecting layout while rank 1's stay packed.
    The ranks run different histogram kernels on the same tree and must still reduce to the single-rank trees."""
    n = 30000
    rng, table = _table(71, n)
    table.bins[1, :12000] = 0
    table.signal = (table.bins - table.bins.mean(axis=1, keepdims=True)) / (table.bins.std(axis=1, keepdims=True) + 1e-9)
    table.finish()
    y = labels_for(0, table.margin(rng))
    cfg = dict(loss=0, max_depth=6, min_examples=1)

    def plans(gbt):
        return [(p.mode, p.chunk_blocks) for p in (gbt.hist_plan(l) for l in range(cfg["max_depth"] - 1))]

    _, res, _ = run_case(table, cfg, y, mode=mode, world=2, on_ranks=plans)
    p0, p1 = res[0]["extra"], res[1]["extra"]
    assert p0 != p1, (p0, p1)
    assert any(a[0] == 2 and b[0] != 2 for a, b in zip(p0, p1)), (p0, p1)   # YGG_HIST_SHARED on rank 0 only


def test_a_rank_without_rows_is_refused_before_any_collective():
    """A rank cannot hold zero rows: ygg_dataset_create refuses the empty dataset (INVALID_ARGUMENT) before the rank has a
    handle, so it never reaches a shard setter or a collective."""
    rng, table = _table(81, 5000)
    with pytest.raises(ydf_b200.YggError) as e:
        table.dataset(2500, 2500)
    assert e.value.code == INVALID and "empty dataset" in str(e.value)


# ---------------------------------------------------------------------------------------------------------------------
# uneven feature splits

def test_one_feature_per_rank():
    rng, table = _table(91, 20000, [dict(kind="num", B=255), dict(kind="cat", B=30), dict(kind="num", B=64)])
    y = labels_for(0, table.margin(rng))
    run_case(table, dict(loss=0, max_depth=6), y, mode="features", world=3)


@pytest.mark.parametrize("mode", ["features", "rows_scatter"])
def test_a_rank_owning_only_categorical_features(mode):
    rng, table = _table(92, 20000, [dict(kind="cat", B=256), dict(kind="cat", B=7), dict(kind="num", B=128),
                                    dict(kind="num", B=32, exact=True)])
    y = labels_for(1, table.margin(rng, 2.0)).astype(F32)
    run_case(table, dict(loss=1, max_depth=7, l2_regularization_categorical=3.0), y, mode=mode, world=2)


@pytest.mark.parametrize("mode", ["features", "rows_scatter"])
def test_a_rank_owning_only_constant_features(mode):
    """Rank 1 owns single-bucket and constant columns: its shard best is never found."""
    layout = [dict(kind="num", B=255), dict(kind="cat", B=12), dict(kind="num", B=1), dict(kind="num", B=64, const=True)]
    rng, table = _table(93, 20000, layout)
    y = labels_for(0, table.margin(rng))
    want, _, _ = run_case(table, dict(loss=0, max_depth=6), y, mode=mode, world=2)
    feats = np.concatenate([np.frombuffer(t, dtype=ydf_b200.NODE_DTYPE)["feature"] for t in want["trees"]])
    assert not np.isin(feats, [2, 3]).any() and (feats >= 0).any()


def test_scatter_at_the_largest_world_with_a_last_chunk_of_one_feature():
    """9 features over 5 ranks: chunks of 2, 2, 2, 2 and 1 feature."""
    layout = [dict(kind="num", B=64), dict(kind="cat", B=9)] * 4 + [dict(kind="num", B=255)]
    rng, table = _table(94, 30000, layout)
    y = labels_for(0, table.margin(rng))
    w = rng.uniform(0.2, 2.0, size=30000).astype(F32)
    run_case(table, dict(loss=0, max_depth=6), y, w=w, mode="rows_scatter", world=5)


def test_scatter_chunks_refused_before_any_collective():
    """9 features do not cut into 6 non-empty chunks of 2: refused before the weight scales are all-reduced (the refusal
    once came after that collective)."""
    layout = [dict(kind="num", B=64)] * 9
    rng, table = _table(95, 6000, layout)
    y = labels_for(0, table.margin(rng))
    w = rng.uniform(0.2, 2.0, size=6000).astype(F32)
    world = 6
    comm = CountingComm(world)

    def rank_main(r):
        r0, r1 = (6000 * r) // world, (6000 * (r + 1)) // world
        gbt = ydf_b200.Gbt(table.dataset(r0, r1), ydf_b200.default_config(loss=0))
        gbt.set_weights(w[r0:r1])
        gbt.set_labels(y[r0:r1])
        with pytest.raises(ydf_b200.YggError) as e:
            gbt.set_row_shard_scatter(r, world, 6000, 0.0, allreduce=comm.allreduce(r),
                                      reducescatter=comm.reducescatter(r), allgather=comm.allgather(r))
        return e.value.code, str(e.value)

    for code, msg in _run_ranks(world, rank_main, comm):
        assert code == INVALID and "non-empty chunks" in msg, msg
    assert comm.total() == 0, comm.calls


# ---------------------------------------------------------------------------------------------------------------------
# drawn configurations

def drawn_case(seed):
    d = SD.draw_sharded(seed)
    rng = np.random.default_rng([seed, 3])
    table = ShardTable(rng, d["n"], d["columns"])
    loss = d["cfg"]["loss"]
    lead = int(np.argmax([c["B"] for c in d["columns"]]))
    m = table.margin(rng, d["scale"], lead=lead)
    if d["scale"] >= 1e3:
        m = m + 1e3
    w = None
    if d["weights"]:
        w = rng.uniform(0.1, 3.0, size=d["n"]).astype(F32)
        w[rng.random(d["n"]) < 0.1] = 0.0
        w[0] = 1.0
    order = None
    if d["split"] == "by_bin":
        order = np.argsort(table.bins[lead], kind="stable")
    elif d["split"] == "by_label":
        order = np.argsort(m, kind="stable")
    elif d["split"] == "label_last":
        order = np.argsort(np.abs(m), kind="stable")
    elif d["split"] == "weight_skew":
        w[np.argmax(w)] = F32(7.0)
        order = np.lexsort((-w, w == 0))
    if order is not None:
        table.reorder(order)
        m = m[order]
        w = None if w is None else w[order]
    y = labels_for(loss, m)
    y = y.astype(F32) if loss == 1 else y
    run_case(table, d["cfg"], y, w=w, mode=d["mode"], world=d["world"], cuts=SD.cuts(d), iters=d["iters"],
             drive=d["drive"])


@pytest.mark.parametrize("seed", list(SD.SUITE_SEEDS))
def test_drawn_sharded_configuration_is_exact(seed):
    drawn_case(seed)


def test_every_sharded_draw_of_the_suite_is_accepted():
    """Every draw builds its rank datasets and handles and is accepted by its shard setter (no training)."""
    for seed in SD.SUITE_SEEDS:
        d = SD.draw_sharded(seed)
        table = ShardTable(np.random.default_rng([seed, 3]), d["n"], d["columns"])
        comm = LoneComm(d["world"])
        for r, (r0, r1) in enumerate(SD.cuts(d)):
            gbt = ydf_b200.Gbt(table.dataset(r0, r1), ydf_b200.default_config(**d["cfg"]))
            if d["mode"] == "features":
                b, e = ydf_b200.feature_shard(d["F"], r, d["world"])
                gbt.set_feature_shard(b, e, r, d["world"], comm.allgather(r))
            else:
                gbt.set_labels(np.ones(r1 - r0, F32 if d["cfg"]["loss"] == 1 else np.int32))
                setter = gbt.set_row_shard if d["mode"] == "rows" else None
                if setter is not None:
                    setter(r, d["world"], d["n"], 0.0, comm.allreduce(r))
                else:
                    gbt.set_row_shard_scatter(r, d["world"], d["n"], 0.0, allreduce=comm.allreduce(r),
                                              reducescatter=comm.reducescatter(r), allgather=comm.allgather(r))
            gbt.close()
        assert comm.total() == 0


# ---------------------------------------------------------------------------------------------------------------------
# call orders

MODES = ["rows", "rows_scatter", "features"]


def _handle(mode, loss=0, n=3000, F=4, labels=True, **cfg):
    """Rank 0 of 2: (handle, table, shard(gbt) -> None, the lone communicator)."""
    rng, table = _table(101, n, [dict(kind="num", B=32), dict(kind="cat", B=5)] * (F // 2))
    y = labels_for(loss, table.margin(rng), K=3)
    gbt = ydf_b200.Gbt(table.dataset(0, n // 2), ydf_b200.default_config(loss=loss, **cfg))
    comm = LoneComm(2)
    if labels:
        gbt.set_labels(y[:n // 2])

    def shard():
        if mode == "rows":
            gbt.set_row_shard(0, 2, n, 0.0, comm.allreduce(0))
        elif mode == "rows_scatter":
            gbt.set_row_shard_scatter(0, 2, n, 0.0, allreduce=comm.allreduce(0), reducescatter=comm.reducescatter(0),
                                      allgather=comm.allgather(0))
        else:
            gbt.set_feature_shard(0, F // 2, 0, 2, comm.allgather(0))
    return gbt, table, shard, comm, y[:n // 2]


def _refused(fn, code):
    with pytest.raises(ydf_b200.YggError) as e:
        fn()
    assert e.value.code == code, (e.value.code, str(e.value))
    return str(e.value)


@pytest.mark.parametrize("mode", MODES)
def test_validation_with_a_shard_is_refused(mode):
    """Held-out rows are evaluated per rank, unreduced: refused in either order (the setters once accepted validation
    rows attached before the shard)."""
    gbt, table, shard, comm, y = _handle(mode)
    vds = table.dataset(0, 500)
    gbt.set_validation(vds, labels_for(0, table.margin(np.random.default_rng(1)))[:500])
    _refused(shard, UNIMPLEMENTED)
    gbt, table, shard, comm2, y = _handle(mode)
    shard()
    _refused(lambda: gbt.set_validation(vds, np.ones(500, np.int32)), UNIMPLEMENTED)
    assert comm.total() == 0 and comm2.total() == 0


@pytest.mark.parametrize("mode", ["rows", "rows_scatter"])
@pytest.mark.parametrize("loss", [0, 1])
def test_labels_after_a_row_shard_are_refused(mode, loss):
    """Labels before the row shard are required; labels after it would replace the job's initial prediction by this
    rank's (they were once accepted)."""
    gbt, table, shard, comm, y = _handle(mode, loss=loss, labels=False)
    _refused(shard, INVALID)
    gbt.set_labels(y)
    shard()
    msg = _refused(lambda: gbt.set_labels(y), INVALID)
    assert "after the row shard" in msg
    assert gbt.initial_prediction() == 0.0   # the job's value passed to the setter
    assert comm.total() == 0


@pytest.mark.parametrize("mode", MODES)
def test_candidate_sampling_and_dart_are_refused_in_either_order(mode):
    for option in (lambda g: g.set_candidate_sampling(1), lambda g: g.set_dart(0.3)):
        gbt, _, shard, comm, _ = _handle(mode)
        option(gbt)
        _refused(shard, UNIMPLEMENTED)
        gbt, _, shard, comm2, _ = _handle(mode)
        shard()
        _refused(lambda: option(gbt), UNIMPLEMENTED)
        assert comm.total() == 0 and comm2.total() == 0


@pytest.mark.parametrize("mode", MODES)
def test_candidate_shuffle_wide_and_presorted_columns_are_refused(mode):
    gbt, _, shard, comm, _ = _handle(mode, candidate_shuffle=1)
    _refused(shard, UNIMPLEMENTED)
    for kind in ("wide", "presorted"):
        rng = np.random.default_rng(5)
        n = 1500
        ds = ydf_b200.Dataset(rng.integers(0, 8, size=(4, n)).astype(np.uint8), [8, 8, 8, 8], [0, 0, 0, 0])
        if kind == "wide":
            ds.set_wide_column(3, rng.integers(0, 300, size=n).astype(np.uint16), 300, 0, np.arange(300, dtype=F32), 0.0)
        else:
            ds.set_numerical_column(3, rng.normal(size=n).astype(F32), 0.0)
        gbt = ydf_b200.Gbt(ds, ydf_b200.default_config(loss=0))
        gbt.set_labels(rng.integers(1, 3, size=n).astype(np.int32))
        if mode == "rows":
            _refused(lambda: gbt.set_row_shard(0, 2, 2 * n, 0.0, comm.allreduce(0)), UNIMPLEMENTED)
        elif mode == "rows_scatter":
            _refused(lambda: gbt.set_row_shard_scatter(0, 2, 2 * n, 0.0, allreduce=comm.allreduce(0),
                                                       reducescatter=comm.reducescatter(0), allgather=comm.allgather(0)),
                     UNIMPLEMENTED)
        else:
            _refused(lambda: gbt.set_feature_shard(0, 2, 0, 2, comm.allgather(0)), UNIMPLEMENTED)
    assert comm.total() == 0


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("what", ["multinomial", "subsample", "goss"])
def test_multinomial_subsample_and_goss_are_refused_before_the_first_collective(mode, what):
    """Accepted by the setters, refused by the first step() (and train()) before that iteration's first collective, so
    that no rank waits on another."""
    cfg = dict(multinomial=dict(loss=2, num_classes=3), subsample=dict(loss=0, subsample=0.5),
               goss=dict(loss=1, goss_alpha=0.2, goss_beta=0.1))[what]
    loss = cfg.pop("loss")
    gbt, _, shard, comm, _ = _handle(mode, loss=loss, **cfg)
    shard()
    _refused(gbt.step, UNIMPLEMENTED)
    _refused(lambda: gbt.train(2), UNIMPLEMENTED)
    assert comm.total() == 0, comm.calls


def test_totals():
    """What the suite's cases checked (printed with -s; meaningful after the cases above ran)."""
    print("sharded exact totals:", STATS)
