"""Node-by-node replay of a REAL training run of the reference against the oracle (test infrastructure).

The reference's golden models adult_binary_class_gbdt_v2 / iris_multi_class_gbdt_v2 / abalone_regression_gbdt_v2 are
default PYDF GBT runs whose training sets ship with the reference, so every quantity the learner computed can be
recomputed: the hold-out draw, the dictionaries, gradients and hessians of every iteration, the best split of every
node, every leaf value and the training log (fixtures: tests/golden/make_ydf_run_fixtures.py).

Boosting state (predictions -> gradients / hessians) follows the REFERENCE's trees and, inside a tree, rows are routed by
the REFERENCE's conditions.  Nothing can drift: every node is an independent check of the oracle's split search and
leaf rule on exactly the statistics the reference had at that node.

Those runs used the reference's EXACT numerical splitter, this repo's path is the DISCRETIZED one (255 bins).  A
numerical split of the reference is comparable when a bucket boundary separates the node's rows exactly like its
threshold does ("on a boundary"); then the discretized scan must find the same partition, count and score — only the
stored threshold value differs (mid-point of neighbouring values vs bucket boundary).  Categorical splits are always
comparable.  For every split, comparable or not, no feature may score higher than the reference's choice."""
import os

import numpy as np

import ydf_b200
from ydf_b200 import dataspec
from oracle import oracle as O

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LOSS_OF_MODEL = {1: O.LOSS_BINOMIAL, 2: 1, 3: O.LOSS_MULTINOMIAL}  # model proto Loss enum -> oracle / ABI loss id


def load_run(name):
    """-> (fixture, {column name: raw values}) ; Adult's CSV columns live in their own fixtures.  `cxx_*`: goldens of the
    reference's C++ tests (training fold of the tester only)."""
    if name.startswith("cxx_"):
        ref = np.load(os.path.join(G, f"ydf_run_{name}.npz"))
        return ref, {str(c): ref[f"data_{c}"] for c in ref["column_names"]}
    ref = np.load(os.path.join(G, f"ydf_run_{name}_v2.npz"))
    names = [str(s) for s in ref["column_names"]]
    if name == "adult":
        cat, num = np.load(os.path.join(G, "adult_categorical.npz")), np.load(os.path.join(G, "adult_numerical.npz"))
        data = {}
        for c, t in zip(names, ref["column_types"]):
            if c == "income":
                data[c] = np.array(["<=50K", ">50K"])[num["train_income"]]
            elif t == 4:
                data[c] = cat[f"strings_{c}"][cat[f"train_{c}"]]
            else:
                data[c] = num[f"train_{c}"].astype(np.float32)
    else:
        data = {c: ref[f"data_{c}"] for c in names}
    return ref, data


def candidate_orders(ref, n_rows_all, num_features, num_trees, seed=123456, max_depth=6, min_examples=5):
    """The order in which the reference evaluated the features at every split-search node of its first `num_trees` trees,
    recovered by following the learner's random engine through the run:
      * utils::RandomEngine = std::mt19937(random_seed) (gradient_boosted_trees.cc:1198);
      * ExtractValidationDataset draws one word per row of the full dataset (:1214, :2718-2807);
      * every node that reaches FindBestCondition — n >= min_examples and depth < max_depth (training.cc:4909-4914) —
        shuffles the candidate features with std::shuffle (GetCandidateAttributes, training.cc:4293-4306) and then
        draws one seed per feature job (FindBestConditionConcurrentManager, training.cc:1658, :1781);
      * nodes are visited depth-first, positive child first (NodeTrain pushes negative then positive, :5031-5046), trees
        in training order (K per iteration).
    std::shuffle is implementation-defined: the golden models follow LIBC++'s algorithm (oracle.Rng.shuffle_libcxx),
    not libstdc++'s — established by the tie-breaks themselves (tests/test_reference_replay.py).
    -> {node index: [position of candidate 0.., i.e. a permutation of range(num_features)]}."""
    rng = O.Rng(seed)
    rng.discard(n_rows_all)
    orders = {}
    for t in range(num_trees):
        advance_rng_through_tree(rng, ref, t, num_features, max_depth, min_examples, orders)
    return orders


def advance_rng_through_tree(rng, ref, t, num_features, max_depth=6, min_examples=5, orders=None):
    """Moves `rng` over the draws the reference made while growing its tree `t` (see candidate_orders)."""
    def end(i):
        return i + 1 if ref["feature"][i] < 0 else end(end(i + 1))
    stack = [(int(ref["tree_first"][t]), 1)]
    while stack:
        i, depth = stack.pop()
        if int(ref["n"][i]) < min_examples or depth >= max_depth:
            assert ref["feature"][i] < 0
            continue
        order = rng.shuffle_libcxx(num_features)
        if orders is not None:
            orders[i] = order
        rng.discard(num_features)
        if ref["feature"][i] >= 0:
            stack.append((i + 1, depth + 1))
            stack.append((end(i + 1), depth + 1))


def numerical_column(name, v, lossless):
    """255 quantile bins (GenDiscretizedBoundaries), or — `lossless` — one bin per distinct value where a column has at
    most 255 of them (dataspec.infer_column_lossless: the exact splitter's candidate cuts)."""
    if lossless == "all":
        # test-only: one bucket per distinct value whatever their number (uint16 codes: the oracle's storage type, not
        # the engine's) — the discretized algorithm on ALL of the exact splitter's candidate cuts
        col = dataspec.infer_column_lossless(name, v, max_distinct=65000)
        col.encode = lambda x, b=col.boundaries: np.searchsorted(b, np.asarray(x, np.float32), side="right").astype(np.uint16)
        return col
    col = dataspec.infer_column_lossless(name, v) if lossless else None
    return col if col is not None else dataspec.infer_column(name, v)   # over all rows: PYDF infers before the hold-out


def replay(ref, data, num_iterations=None, score_rtol=1e-6, leaf_atol=1e-6, lossless=False):
    names = [str(s) for s in ref["column_names"]]
    label_name = names[int(ref["label_col_idx"])]
    loss = LOSS_OF_MODEL[int(ref["loss"])]
    K = int(ref["num_trees_per_iter"])
    n_all = len(data[label_name])
    keep = ydf_b200.validation_split_mask(123456, n_all, 0.1)   # ExtractValidationDataset, gradient_boosted_trees.cc
    if loss == 1:
        y = data[label_name].astype(np.float32)
    else:
        # PYDF label dictionary: np.unique order (port/python/ydf/dataset/dataset.py:366-380)
        voc = [str(s) for s in ref[f"vocabulary_{label_name}"]]
        assert voc == ["<OOD>"] + sorted(set(data[label_name].tolist()))
        y = np.array([voc.index(s) for s in data[label_name]], np.int32)
    assert all(int(v) == 0 for v, t in zip(ref["most_frequent_value"], ref["column_types"]) if t == 4)
    feats = {}
    for ci, name in enumerate(names):  # dataspec order = candidate order
        if name == label_name:
            continue
        if ref["column_types"][ci] == 4:
            col = dataspec.infer_categorical_column(name, data[name], front_end=dataspec.FRONT_END_PYDF)
            assert col.vocabulary == list(ref[f"vocabulary_{name}"]), name   # ties: key ascending
            feats[ci] = (True, col, col.encode(data[name]).astype(np.uint16), None)
        else:
            v = data[name].astype(np.float32)
            col = numerical_column(name, v, lossless)
            feats[ci] = (False, col, col.encode(v).astype(np.uint16), v)
    anyf = min(feats)
    cfg = O.default_config(max_depth=1, min_examples=5, shrinkage=0.1, use_hessian_gain=0, loss=loss, num_classes=K if K > 1 else 0)
    init = ref["initial_predictions"].astype(np.float32)
    if K == 1:
        assert abs(O.initial_prediction(loss, y[keep]) - float(init[0])) <= 1e-6 * max(1.0, abs(float(init[0])))
    else:
        assert not init.any()   # multinomial: zeros (loss_imp_multinomial.cc)
    pred = np.tile(init, (n_all, 1))   # [rows, K], training AND hold-out rows
    train_rows, valid_rows = np.nonzero(keep)[0], np.nonzero(~keep)[0]
    seen = dict(splits=0, categorical=0, numerical=0, numerical_on_a_boundary=0, leaves=0, ties=0, ties_as_shuffled=0,
                noise=0, argmax_checks=0, max_leaf_err=0.0, max_score_rerr=0.0)
    logs = []
    total_iters = len(ref["tree_first"]) // K
    cand = sorted(feats)   # config_link.features(): column indices, ascending
    orders = candidate_orders(ref, n_all, len(cand), (total_iters if num_iterations is None else num_iterations) * K)
    for it in range(total_iters if num_iterations is None else num_iterations):
        if K == 1:
            gk, hk = O.update_gradients(loss, y[keep], pred[keep, 0])
            gk, hk = gk[None, :], hk[None, :]
        else:
            gk, hk = O.mc_update_gradients(y[keep], K, pred[keep])
        nxt = pred.copy()
        for k in range(K):
            g = np.zeros(n_all, np.float32)
            h = np.zeros(n_all, np.float32)
            g[keep], h[keep] = gk[k], hk[k]
            t = it * K + k

            def walk(i, rows, other):
                """rows: training rows in the node (checked); other: hold-out rows (routed only)."""
                assert len(rows) == int(ref["n"][i]), (t, i)
                f = int(ref["feature"][i])
                if f < 0:
                    leaf = O.train_tree(feats[anyf][2][rows][None, :], [feats[anyf][1].num_bins], [feats[anyf][1].na_bin],
                                        g[rows], h[rows], cfg)
                    err = abs(float(leaf[0]["leaf_value"]) - float(ref["value"][i]))
                    assert len(leaf) == 1 and err <= leaf_atol, (t, i, err)
                    seen["max_leaf_err"] = max(seen["max_leaf_err"], err)
                    seen["leaves"] += 1
                    nxt[rows, k] += ref["value"][i]
                    nxt[other, k] += ref["value"][i]
                    return i + 1
                is_cat, col, codes, raw = feats[f]

                def route(rr):
                    if is_cat:
                        return (int(ref["positive_mask"][i]) >> codes[rr].astype(np.uint64)) & 1 == 1
                    return raw[rr] >= ref["threshold"][i]
                go, go_other = route(rows), route(other)
                assert int(go.sum()) == int(ref["n_pos"][i]), (t, i)
                want = float(ref["split_score"][i])
                seen["splits"] += 1
                if want < 1e-12:
                    seen["noise"] += 1   # a pure node: +-1e-16 rounding noise of the variance arithmetic (util.prune_noise_splits)
                else:
                    res = {c: O.find_split(cd, cl.num_bins, cl.na_bin, rows, g, min_num_obs=5, categorical=kind)
                           for c, (kind, cl, cd, _) in feats.items()}
                    r = res[f]
                    top = max([v["split_score"] for v in res.values() if v["result"] == 0] + [0.0])
                    assert top <= want * (1 + score_rtol), (t, i, top, want)   # nothing beats the reference's choice
                    seen["argmax_checks"] += 1
                    c = codes[rows]
                    if is_cat:
                        seen["categorical"] += 1
                        mine = np.isin(c, r["positive_categories"])
                        assert r["na_value"] == bool(ref["na_value"][i]), (t, i)
                        comparable = True
                    else:
                        seen["numerical"] += 1
                        comparable = c[go].min() > c[~go].max()
                        seen["numerical_on_a_boundary"] += int(comparable)
                        mine = c >= r["threshold"]
                    if comparable:
                        assert r["result"] == 0 and r["num_pos"] == int(ref["n_pos"][i]) and np.array_equal(mine, go), (t, i)
                        rerr = abs(r["split_score"] - want) / want
                        assert rerr <= score_rtol, (t, i, r["split_score"], want)
                        seen["max_score_rerr"] = max(seen["max_score_rerr"], rerr)
                        # strict '>' over float scores in candidate order: the winner is the FIRST of the tied features in the
                        # order the node's shuffle produced
                        tied = [cc for cc, v in res.items() if v["result"] == 0 and np.float32(v["split_score"]) == np.float32(want)]
                        if f in tied and len(tied) > 1:
                            seen["ties"] += 1
                            winner = next(cand[o] for o in orders[i] if cand[o] in tied)
                            seen["ties_as_shuffled"] += int(winner == f)
                j = walk(i + 1, rows[~go], other[~go_other])
                return walk(j, rows[go], other[go_other])

            end = walk(int(ref["tree_first"][t]), train_rows, valid_rows)
            assert end == (int(ref["tree_first"][t + 1]) if t + 1 < len(ref["tree_first"]) else len(ref["n"]))
        pred = nxt
        if K == 1:
            tl, ts = O.loss_value(loss, y[keep], pred[keep, 0])
            vl, vs = O.loss_value(loss, y[~keep], pred[~keep, 0])
        else:
            tl, ts = O.mc_loss(y[keep], K, pred[keep])
            vl, vs = O.mc_loss(y[~keep], K, pred[~keep])
        logs.append((tl, ts, vl, vs))
    return seen, np.array(logs)


def replay_cxx(ref, data, num_iterations=None, score_rtol=1e-6, leaf_atol=1e-6):
    """The node-by-node replay for the goldens of the reference's C++ tests (`ExpectEqualGoldenModel`,
    gradient_boosted_trees_test.cc), which differ from the PYDF runs in everything around the splitter:
      * rows: the training fold of utils::TrainAndTestTester (fixture), then the learner's 10 % hold-out;
      * dataspec: the C++ inference over the whole CSV — dictionaries and most_frequent_value (the NA replacement) are
        taken from the model's dataspec;
      * one thread: FindBestConditionSingleThreadManager (training.cc:1364-1488) — features evaluated one after the other
        in the shuffled order, each against the RUNNING best score re-rounded to float, and no seed draws;
      * optionally stochastic gradient boosting: one word per training row and iteration, drawn before the trees
        (SampleTrainingExamples, gradient_boosted_trees.cc:2932-2956) — the tree sees the kept rows, predictions and losses
        all rows;
      * optionally hessian gain (float bucket sums, l2_categorical = 1 on categorical features).
    Numerical columns get one bucket per distinct value (the exact splitter's candidate cuts).  The walk is depth-first,
    positive child first, consuming the learner's mt19937 as it goes, so a single wrong assumption about the stream shows
    up at the next root (its row count is the size of that iteration's row draw).
    With hessian gain the reference's exact splitter sums floats in sorted-value order, the bucket path in row order per
    bucket: scores agree to ~1e-6 but float-level ties between features may break differently ("other_winner")."""
    names = [str(s) for s in ref["column_names"]]
    label_name = names[int(ref["label_col_idx"])]
    loss = LOSS_OF_MODEL[int(ref["loss"])]
    K = int(ref["num_trees_per_iter"])
    hessian, subsample = bool(ref["run_use_hessian_gain"]), np.float32(ref["run_subsample"])
    max_depth, min_examples = int(ref["run_max_depth"]), 5
    assert str(ref["run_front_end"]) == "cpp" and int(ref["run_single_thread"]) == 1
    n_all = len(data[label_name])
    keep = ydf_b200.validation_split_mask(123456, n_all, 0.1)
    if loss == 1:
        y = data[label_name].astype(np.float32)
    else:
        voc = [str(s) for s in ref[f"vocabulary_{label_name}"]]
        y = np.array([voc.index(s) for s in data[label_name]], np.int32)
    feats = {}
    for ci, name in enumerate(names):
        if name == label_name:
            continue
        if ref["column_types"][ci] == 4:
            voc = [str(s) for s in ref[f"vocabulary_{name}"]]
            index, mfv = {k: j for j, k in enumerate(voc)}, int(ref["most_frequent_value"][ci])
            codes = np.array([mfv if s == "" else index.get(s, 0) for s in data[name].tolist()], np.uint16)
            feats[ci] = (True, dataspec.CategoricalColumn(name, voc, [0] * len(voc), len(voc), mfv), codes[keep], None)
        else:
            v = data[name].astype(np.float32)
            col = numerical_column(name, v, "all")
            feats[ci] = (False, col, col.encode(v)[keep], v[keep])
    cand = sorted(feats)
    F = len(cand)
    yk, n = y[keep], int(keep.sum())
    init = ref["initial_predictions"].astype(np.float32)
    if K == 1:
        assert abs(O.initial_prediction(loss, yk) - float(init[0])) <= 1e-6 * max(1.0, abs(float(init[0])))
    pred = np.tile(init, (n_all, 1))
    valid_rows = np.arange(n, n_all)   # hold-out rows are routed only: index them after the kept ones
    vfeats = None
    if n_all > n:
        vfeats = {}
        for ci, name in enumerate(names):
            if ci in feats:
                is_cat, col, _codes, _raw = feats[ci]
                if is_cat:
                    index = {k: j for j, k in enumerate(col.vocabulary)}
                    allc = np.array([col.na_bin if s == "" else index.get(s, 0) for s in data[name].tolist()], np.uint16)
                    vfeats[ci] = (allc[~keep], None)
                else:
                    vfeats[ci] = (None, data[name].astype(np.float32)[~keep])
    cfg = O.default_config(max_depth=1, min_examples=min_examples, shrinkage=0.1, use_hessian_gain=int(hessian), loss=loss,
                           num_classes=K if K > 1 else 0)
    rng = O.Rng(123456)
    rng.discard(n_all)
    seen = dict(splits=0, same_winner=0, other_winner=0, same_partition=0, other_partition=0, leaves=0, noise=0, trees=0,
                max_leaf_err=0.0, max_score_rerr=0.0)
    pk = np.tile(init, (n, 1))          # predictions of the kept rows
    pv = np.tile(init, (n_all - n, 1))  # and of the hold-out rows
    yv = y[~keep]
    logs = []

    def end(i):
        return i + 1 if ref["feature"][i] < 0 else end(end(i + 1))
    total_iters = len(ref["tree_first"]) // K
    for it in range(total_iters if num_iterations is None else num_iterations):
        if K == 1:
            gk, hk = O.update_gradients(loss, yk, pk[:, 0])
            gk, hk = gk[None, :], hk[None, :]
        else:
            gk, hk = O.mc_update_gradients(yk, K, pk)
        if subsample < 1:
            sel = np.array([r for r in range(n) if np.float32(rng.next()) / np.float32(4294967296.0) < subsample])
        else:
            sel = np.arange(n)
        unsel = np.setdiff1d(np.arange(n), sel)
        nk, nv = pk.copy(), pv.copy()
        for k in range(K):
            t = it * K + k
            g, h = gk[k], hk[k]
            stack = [(int(ref["tree_first"][t]), sel, unsel, np.arange(n_all - n), 1)]
            while stack:
                i, rows, other, vrows, depth = stack.pop()
                assert len(rows) == int(ref["n"][i]), (t, i, len(rows), int(ref["n"][i]))
                f = int(ref["feature"][i])

                def set_leaf():
                    anyf = cand[0]
                    leaf = O.train_tree(feats[anyf][2][rows][None, :], [feats[anyf][1].num_bins], [feats[anyf][1].na_bin],
                                        g[rows], h[rows], cfg)
                    err = abs(float(leaf[0]["leaf_value"]) - float(ref["value"][i]))
                    assert len(leaf) == 1 and err <= leaf_atol, (t, i, err)
                    seen["max_leaf_err"] = max(seen["max_leaf_err"], err)
                    seen["leaves"] += 1
                    nk[rows, k] += ref["value"][i]
                    nk[other, k] += ref["value"][i]
                    nv[vrows, k] += ref["value"][i]
                if len(rows) < min_examples or depth >= max_depth:
                    assert f < 0
                    set_leaf()
                    continue
                order = rng.shuffle_libcxx(F)      # GetCandidateAttributes; no seed draws with one thread
                if f < 0:
                    set_leaf()
                    continue
                is_cat, col, codes, raw = feats[f]

                def route(cc, rr):
                    if is_cat:
                        return (int(ref["positive_mask"][i]) >> cc.astype(np.uint64)) & 1 == 1
                    return rr >= ref["threshold"][i]
                go = route(codes[rows], None if is_cat else raw[rows])
                go_other = route(codes[other], None if is_cat else raw[other])
                go_v = route(vfeats[f][0][vrows], None) if is_cat else route(None, vfeats[f][1][vrows])
                assert int(go.sum()) == int(ref["n_pos"][i]), (t, i)
                want = float(ref["split_score"][i])
                seen["splits"] += 1
                if want < 1e-12:
                    seen["noise"] += 1
                else:
                    best, winner, rwin = np.float32(0.0), None, None
                    for o in order:
                        c = cand[o]
                        kind, cl, cd, _ = feats[c]
                        r = O.find_split(cd, cl.num_bins, cl.na_bin, rows, g, hessians=h, use_hessian_gain=hessian,
                                         min_num_obs=min_examples, l2=1.0 if (kind and hessian) else 0.0, categorical=kind,
                                         initial_split_score=float(best))
                        if r["result"] == 0:
                            best, winner, rwin = np.float32(r["split_score"]), c, r
                    assert winner is not None and float(best) <= want * (1 + max(score_rtol, 2e-6 if hessian else 0)), (t, i)
                    if winner == f:
                        seen["same_winner"] += 1
                        mine = np.isin(codes[rows], rwin["positive_categories"]) if is_cat else codes[rows] >= rwin["threshold"]
                        if np.array_equal(mine, go):
                            rerr = abs(float(best) - want) / want
                            assert rerr <= score_rtol or abs(float(best) - want) <= 1e-14, (t, i, float(best), want)
                            if want > 1e-9:
                                seen["max_score_rerr"] = max(seen["max_score_rerr"], rerr)
                            seen["same_partition"] += 1
                        else:
                            # category buckets with EQUAL label means: their order after the reference's std::sort is
                            # implementation-defined, and with it which prefixes the scan can reach
                            assert is_cat or hessian or want < 1e-8, (t, i)
                            seen["other_partition"] += 1
                    else:
                        # another feature with the same score to float precision: hessian gain (float sums in another
                        # order), or variance scores of ~1e-9 and below late in training (rounding noise of the doubles)
                        assert hessian or want < 1e-8, (t, i, names[f], names[winner], want)
                        assert abs(float(best) - want) <= 1e-5 * want, (t, i, float(best), want)
                        seen["other_winner"] += 1
                j = i + 1
                stack.append((j, rows[~go], other[~go_other], vrows[~go_v], depth + 1))
                stack.append((end(j), rows[go], other[go_other], vrows[go_v], depth + 1))
            seen["trees"] += 1
        pk, pv = nk, nv
        if K == 1:
            tl, ts = O.loss_value(loss, yk, pk[:, 0])
            vl, vs = O.loss_value(loss, yv, pv[:, 0])
        else:
            tl, ts = O.mc_loss(yk, K, pk)
            vl, vs = O.mc_loss(yv, K, pv)
        logs.append((tl, ts, vl, vs))
    return seen, np.array(logs)


def oracle_loop_cxx(ref, data, stable_category_sort=True, num_threads=1, dart=None, **config):
    """The oracle's WHOLE learner loop on its own state, set up like utils::TrainAndTestTester sets up the reference for a
    C++ test: training fold, C++ dataspec (dictionaries of the model), one thread, libc++ candidate shuffle, default 10 %
    hold-out + early stopping, and — to stand in for the exact numerical splitter — one bucket per distinct value with the
    exact threshold rule (oracle.set_bucket_values).  `config` overrides GBT hyper-parameters; num_threads > 1 selects the
    concurrent manager (PYDF runs: the model's dictionaries are PYDF's then); `dart` a dropout rate selects DART
    (oracle.set_dart).  Returns the oracle's result dict plus `predict(columns) -> raw scores` that routes RAW rows by
    the float thresholds / dictionaries; under DART it sums fl(leaf * w) in tree order, the model's scaled leaves."""
    names = [str(s) for s in ref["column_names"]]
    label = names[int(ref["label_col_idx"])]
    loss = LOSS_OF_MODEL[int(ref["loss"])]
    feat_names, bins, nb, na, ft, vals, means, dicts = [], [], [], [], [], [], [], {}
    for ci, name in enumerate(names):
        if name == label:
            continue
        feat_names.append(name)
        if ref["column_types"][ci] == 4:
            voc = [str(s) for s in ref[f"vocabulary_{name}"]]
            index, mfv = {k: j for j, k in enumerate(voc)}, int(ref["most_frequent_value"][ci])
            dicts[name] = (index, mfv)
            bins.append(np.array([mfv if s == "" else index.get(s, 0) for s in data[name].tolist()], np.uint16))
            nb.append(len(voc)); na.append(mfv); ft.append(1); vals.append(None); means.append(0.0)
        else:
            v = data[name].astype(np.float32)
            col = numerical_column(name, v, "all")
            bins.append(col.encode(v)); nb.append(col.num_bins); na.append(col.na_bin); ft.append(0)
            vals.append(np.unique(v[~np.isnan(v)])); means.append(col.mean)
    if loss == 1:
        y = data[label].astype(np.float32)
    else:
        voc = [str(s) for s in ref[f"vocabulary_{label}"]]
        y = np.array([voc.index(s) for s in data[label]], np.int32)
    kw = dict(loss=loss, num_trees=300, max_depth=int(ref["run_max_depth"]), subsample=float(ref["run_subsample"]),
              use_hessian_gain=int(ref["run_use_hessian_gain"]))
    if int(ref["num_trees_per_iter"]) > 1:
        kw["num_classes"] = int(ref["num_trees_per_iter"])
    kw.update(config)
    cfg = O.default_config(**kw)
    O.set_validated_shuffle_mode(O.SHUFFLE_LIBCXX)
    O.set_stable_category_sort(stable_category_sort)   # libc++ orders up to 30 equal buckets stably (insertion sort)
    O.set_bucket_values(vals, means)
    O.set_dart(dart)
    try:
        out = O.gbt_train_validated(np.stack(bins), nb, na, y, cfg, 0.1, num_threads=num_threads, feature_type=ft)
    finally:
        O.set_dart(None)
        O.set_validated_shuffle_mode(O.SHUFFLE_NONE)
        O.set_stable_category_sort(False)
        O.set_bucket_values(None)
    loss = kw["loss"]   # a test may run another loss than the golden's (FakeMulticlass: multinomial on two classes)
    init = 0.0 if loss == O.LOSS_MULTINOMIAL else O.initial_prediction(loss, y[out["in_training"]])

    K_out = int(kw.get("num_classes", 0)) if loss == O.LOSS_MULTINOMIAL else 1

    def predict(columns):
        """-> raw scores [n] (one output) or [n, K] (multinomial: tree i belongs to class i mod K)."""
        n = len(columns[feat_names[0]])
        raw = np.full((n, K_out), init, np.float32)
        enc = {}
        for name in feat_names:
            if name in dicts:
                index, mfv = dicts[name]
                enc[name] = np.array([mfv if s == "" else index.get(s, 0) for s in columns[name].tolist()], np.int64)
        for ti, t in enumerate(out["trees"]):
            node = np.zeros(n, np.int64)
            thr = t["threshold_value"]
            while True:
                f = t["feature"][node]
                act = np.nonzero(f >= 0)[0]
                if len(act) == 0:
                    break
                go = np.zeros(len(act), bool)
                for fi in np.unique(f[act]):
                    m = f[act] == fi
                    rows, nd = act[m], node[act[m]]
                    name = feat_names[fi]
                    if name in dicts:
                        c = enc[name][rows]
                        go[m] = ((t["cat_mask"][nd, c >> 5] >> (c & 31).astype(np.uint32)) & 1) != 0
                    else:
                        x = columns[name][rows].astype(np.float32)
                        go[m] = np.where(np.isnan(x), t["na_value"][nd] != 0, x >= thr[nd])
                node[act] = np.where(go, t["pos_child"][node[act]], t["neg_child"][node[act]])
            leaf = t["leaf_value"][node]
            if dart is not None:
                leaf = (leaf * out["dart_weights"][ti // K_out]).astype(np.float32)
            raw[:, ti % K_out] += leaf
        return raw[:, 0] if K_out == 1 else raw
    out["predict"] = predict
    out["labels"] = y
    return out


LOG_KEYS = ["log_training_loss", "log_training_secondary", "log_validation_loss", "log_validation_secondary"]


def max_log_error(ref, logs):
    """Largest |replayed - logged| over the replayed iterations, per log column."""
    n = len(logs)
    assert list(ref["log_num_trees"][:n]) == list(range(1, n + 1))
    return {key: float(np.abs(logs[:, k] - ref[key][:n].astype(np.float64)).max()) for k, key in enumerate(LOG_KEYS)}


# ------------------------------------------------------------------------------------------------------------------
# Whole trees of a trainer (the oracle on CPU, the CUDA engine on the GPU) against the reference's trees


def replay_trees(ref, data, make_trainer, num_iterations=None, score_rtol=1e-6, leaf_atol=1e-6, lossless=False):
    """For every tree of the reference run: hand the gradients / hessians the REFERENCE had at that iteration to a tree
    trainer (decision_tree::Train seam) working on this repo's 255-bin + dictionary encoding of the training rows, and
    compare the returned tree with the reference's tree in lockstep from the root:
      * a reference leaf must be a leaf with the same value;
      * a comparable reference split (categorical, or numerical on a bucket boundary) must be a split with the same
        partition of the node's rows, the same positive count and score — the FEATURE may differ when two features
        give the same partition, possibly seen from the other side (exact float ties are resolved by the reference's
        per-node candidate shuffle: candidate_orders);
      * below a reference split that cuts inside a bucket ("skipped_subtrees"), or where the trainer found a
        DIFFERENT partition with the same float score ("tied_subtrees": the arg-max is not unique), the two trees
        legitimately differ: the subtree is skipped and counted.
    make_trainer(bins [F, n] uint8, num_bins, na_bin, feature_types, loss, num_classes) -> fn(g, h) -> node array
    (ydf_b200.NODE_DTYPE).  A trainer with the attribute `wants_rng` is called as fn(g, h, rng) with the learner's random
    engine in the state it had when the reference started that tree (candidate_orders): it can then break ties between
    equal-score features exactly like the reference did.  Returns the counters."""
    from tests.util import prune_noise_splits
    names = [str(s) for s in ref["column_names"]]
    label_name = names[int(ref["label_col_idx"])]
    loss = LOSS_OF_MODEL[int(ref["loss"])]
    K = int(ref["num_trees_per_iter"])
    n_all = len(data[label_name])
    keep = ydf_b200.validation_split_mask(123456, n_all, 0.1)
    if loss == 1:
        y = data[label_name].astype(np.float32)
    else:
        voc = [str(s) for s in ref[f"vocabulary_{label_name}"]]
        y = np.array([voc.index(s) for s in data[label_name]], np.int32)
    feats = []   # our feature order = dataspec order without the label
    for ci, name in enumerate(names):
        if name == label_name:
            continue
        if ref["column_types"][ci] == 4:
            col = dataspec.infer_categorical_column(name, data[name], front_end=dataspec.FRONT_END_PYDF)
            feats.append((ci, True, col, col.encode(data[name])[keep], None))
        else:
            v = data[name].astype(np.float32)
            col = numerical_column(name, v, lossless)
            feats.append((ci, False, col, col.encode(v)[keep], v[keep]))
    of_ref = {ci: j for j, (ci, *_rest) in enumerate(feats)}
    bins = np.stack([f[3] for f in feats]).astype(np.uint16 if lossless == "all" else np.uint8)
    trainer = make_trainer(bins, [f[2].num_bins for f in feats], [f[2].na_bin for f in feats],
                           [int(f[1]) for f in feats], loss, K if K > 1 else 0)
    n = int(keep.sum())
    yk = y[keep]
    pred = np.tile(ref["initial_predictions"].astype(np.float32), (n, 1))
    shadow = O.Rng(123456)
    shadow.discard(n_all)
    seen = dict(trees=0, identical_trees=0, identical_trees_same_features=0, splits=0, same_feature=0, mirrored=0, leaves=0,
                noise=0, skipped_subtrees=0, tied_subtrees=0, skipped_nodes=0, max_leaf_err=0.0, max_score_rerr=0.0)

    def subtree_end(i):
        return i + 1 if ref["feature"][i] < 0 else subtree_end(subtree_end(i + 1))

    total_iters = len(ref["tree_first"]) // K
    for it in range(total_iters if num_iterations is None else num_iterations):
        if K == 1:
            gk, hk = O.update_gradients(loss, yk, pred[:, 0])
            gk, hk = gk[None, :], hk[None, :]
        else:
            gk, hk = O.mc_update_gradients(yk, K, pred)
        nxt = pred.copy()
        for k in range(K):
            t = it * K + k
            if getattr(trainer, "wants_rng", False):
                ours = trainer(gk[k], hk[k], shadow.clone())
            else:
                ours = trainer(gk[k], hk[k])
            advance_rng_through_tree(shadow, ref, t, len(feats))
            ours = prune_noise_splits(ours, 1e-12)
            skipped_before = seen["skipped_subtrees"] + seen["tied_subtrees"]
            other_feature_before = seen["splits"] - seen["same_feature"]

            def walk(i, j, rows):
                assert len(rows) == int(ref["n"][i]) == int(ours[j]["num_examples"]), (t, i, j)
                f = int(ref["feature"][i])
                mine = ours[j]
                if f < 0 or float(ref["split_score"][i]) < 1e-12:
                    # leaf — or a "split" of a pure node on 1e-16 rounding noise, whose children repeat the node's value
                    seen["noise"] += int(f >= 0)
                    assert mine["feature"] < 0, (t, i, j, "reference leaf, trainer split")
                    err = abs(float(mine["leaf_value"]) - float(ref["value"][i]))
                    assert err <= leaf_atol, (t, i, j, err)
                    seen["max_leaf_err"] = max(seen["max_leaf_err"], err)
                    seen["leaves"] += 1
                    end = subtree_end(i)
                    for q in range(i, end):   # routing below a noise split does not matter: equal values
                        if ref["feature"][q] < 0:
                            assert abs(float(ref["value"][q]) - float(ref["value"][i])) <= 1e-6
                    nxt[rows, k] += ref["value"][i] if f < 0 else ref["value"][i + 1]
                    return end
                _, is_cat, col, codes, raw = feats[of_ref[f]]
                c = codes[rows]
                if is_cat:
                    go = (int(ref["positive_mask"][i]) >> c.astype(np.uint64)) & 1 == 1
                    comparable = True
                else:
                    go = raw[rows] >= ref["threshold"][i]
                    comparable = c[go].min() > c[~go].max()
                assert int(go.sum()) == int(ref["n_pos"][i])
                def skip_subtree(counter):
                    """The two trees legitimately differ below this node; predictions follow the reference's tree."""
                    seen[counter] += 1
                    end = subtree_end(i)
                    seen["skipped_nodes"] += end - i

                    def apply(q, rr):
                        fq = int(ref["feature"][q])
                        if fq < 0:
                            nxt[rr, k] += ref["value"][q]
                            return q + 1
                        _, qc, _, qcodes, qraw = feats[of_ref[fq]]
                        g2 = ((int(ref["positive_mask"][q]) >> qcodes[rr].astype(np.uint64)) & 1 == 1) if qc else (qraw[rr] >= ref["threshold"][q])
                        return apply(apply(q + 1, rr[~g2]), rr[g2])
                    assert apply(i, rows) == end
                    return end
                if not comparable:
                    return skip_subtree("skipped_subtrees")
                assert mine["feature"] >= 0, (t, i, j, "reference split, trainer leaf")
                b = bins[int(mine["feature"]), rows].astype(np.int64)
                if mine["condition_type"] == 1:
                    my_go = ((mine["cat_mask"][b >> 5] >> (b & 31).astype(np.uint32)) & 1) != 0
                else:
                    my_go = b >= mine["threshold_bin"]
                assert int(mine["num_pos_examples"]) == int(my_go.sum())
                want = float(ref["split_score"][i])
                rerr = abs(float(mine["split_score"]) - want) / want
                # scores of ~1e-12 sit on the rounding noise of the variance arithmetic (1e-16 absolute)
                assert rerr <= score_rtol or abs(float(mine["split_score"]) - want) <= 1e-14, (t, i, j, float(mine["split_score"]), want)
                mirrored = False
                if not np.array_equal(my_go, go):
                    # an equally good split (score equal to float precision) that cuts the rows differently: the arg-max
                    # is not unique — e.g. Adult tree 0, 434 rows: `occupation in {...}` sets 5 rows apart,
                    # `age >= 79.5` another 5 with the same gradient sums (first gradients take two values only)
                    assert int(mine["feature"]) != of_ref[f], (t, i, j)
                    if np.array_equal(my_go, ~go):
                        mirrored = True
                        seen["mirrored"] += 1
                    else:
                        return skip_subtree("tied_subtrees")
                if want > 1e-9:
                    seen["max_score_rerr"] = max(seen["max_score_rerr"], rerr)
                seen["splits"] += 1
                seen["same_feature"] += int(int(mine["feature"]) == of_ref[f])
                nxt_i = walk(i + 1, int(mine["pos_child" if mirrored else "neg_child"]), rows[~go])
                return walk(nxt_i, int(mine["neg_child" if mirrored else "pos_child"]), rows[go])

            end = walk(int(ref["tree_first"][t]), 0, np.arange(n))
            assert end == (int(ref["tree_first"][t + 1]) if t + 1 < len(ref["tree_first"]) else len(ref["n"]))
            seen["trees"] += 1
            identical = seen["skipped_subtrees"] + seen["tied_subtrees"] == skipped_before
            seen["identical_trees"] += int(identical)
            seen["identical_trees_same_features"] += int(identical and seen["splits"] - seen["same_feature"] == other_feature_before)
        pred = nxt
    return seen


def oracle_trainer_shuffled(bins, num_bins, na_bin, feature_types, loss, num_classes):
    """The oracle with the reference's per-node candidate shuffle (libc++ std::shuffle) on the learner's random stream."""
    cfg = O.default_config(max_depth=6, min_examples=5, shrinkage=0.1, use_hessian_gain=0, loss=loss, num_classes=num_classes)

    def train(g, h, rng):
        return O.train_tree_rng(bins, num_bins, na_bin, g, h, cfg, rng, shuffle=O.SHUFFLE_LIBCXX, feature_type=feature_types)
    train.wants_rng = True
    return train


def oracle_trainer(bins, num_bins, na_bin, feature_types, loss, num_classes):
    cfg = O.default_config(max_depth=6, min_examples=5, shrinkage=0.1, use_hessian_gain=0, loss=loss, num_classes=num_classes)
    return lambda g, h: O.train_tree(bins, num_bins, na_bin, g, h, cfg, num_threads=4, feature_type=feature_types)
