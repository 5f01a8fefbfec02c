"""CPU tests of the exact fuzz's host side (tests/exact_fuzz_draw.py): the drawer, the early-stopping restatement, the
selection-aware bucket sums and the tie-break replay's expectation."""
import numpy as np

from oracle import oracle as O
from tests import exact_fuzz_draw as D
from tests import scan_ref as S
from tests.util import quantize_q24, quantize_second

REQUIRED = (
    [f"rows {n}" for n in D.ROWS] + [f"loss {l}" for l in range(3)] + [f"classes {k}" for k in range(2, 6)]
    + [f"column {k}" for k in D.KINDS] + ["column num runs", "column num const", "column cat absent"]
    + [f"twin {t}" for t in D.TWIN_KINDS]
    + ["gain variance", "gain hessian", "l1_regularization", "l2_regularization", "l2_regularization_categorical",
       "hessian_split_score_subtract_parent", "in_split 0", "in_split 1", "sibling 0", "sibling 1"]
    + [f"depth {k}" for k in (2, 3, 4, 5, 6, 7, 10)]
    + ["shrinkage 1", "clamp", "sampling none", "sampling subsample", "sampling goss", "weights", "candidates ratio",
       "candidates num", "draw seeds 0", "draw seeds 1", "best first", "replay 0", "replay 1", "replay 2", "validation",
       "validation weights", "early stopping 0", "early stopping 1", "early stopping 2", "drive step", "drive train"])


def test_draws_are_deterministic_and_accepted():
    for seed in list(D.SUITE_SEEDS) + [1000, 4321]:
        a, b = D.draw(seed), D.draw(seed)
        assert repr(a) == repr(b)
        assert D.refusal(a) is None
        ca = D.make_columns(a, np.random.default_rng([seed, 1]), min(a["n"], 500))
        cb = D.make_columns(a, np.random.default_rng([seed, 1]), min(a["n"], 500))
        for x, y in zip(ca, cb):
            assert x["kind"] == y["kind"] and repr(x) == repr(y)


def test_the_suite_covers_every_option():
    cov = D.coverage(D.SUITE_SEEDS)
    missing = [k for k in REQUIRED if k not in cov]
    assert not missing, f"not drawn by the suite's seeds: {missing}"


def test_the_refusals_are_restated():
    d = D.draw(0)
    for change, reason in ((dict(goss_alpha=0.2, subsample=0.5), "GOSS with subsample"),
                           (dict(growing_strategy=1, candidate_shuffle=2), "the replay with best-first growth"),
                           (dict(max_depth=10, sibling_subtraction=0), "more than 254 histogram slots")):
        bad = dict(d, cfg=dict(d["cfg"], **change))
        assert D.refusal(bad) == reason
    assert D.refusal(dict(d, weights=True, cfg=dict(d["cfg"], use_hessian_gain=1))) is not None


def test_twins_route_like_their_source():
    d = None
    for seed in range(200):
        d = D.draw(seed)
        if any("twin" in c for c in d["columns"]):
            break
    cols = D.make_columns(d, np.random.default_rng(1), 3000)
    for c, spec in zip(cols, d["columns"]):
        if "twin" not in spec:
            continue
        src = cols[spec["of"]]
        if spec["twin"] == "pre_scaled":
            np.testing.assert_array_equal(np.isnan(c["values"]), np.isnan(src["values"]))
        elif spec["twin"] == "cat_permuted":
            # one category of the twin per category of the source
            pairs = set(zip(src["codes"].tolist(), c["codes"].tolist()))
            assert len(pairs) == len(set(src["codes"].tolist()))
        else:
            np.testing.assert_array_equal(c["codes"], src["codes"])


def test_early_stopping_restatement_matches_the_oracle():
    """EarlyStoppingState + ygg_gbt_train's finalisation on the oracle's validation losses give the oracle's log length,
    kept trees, final loss and trigger."""
    rng = np.random.default_rng(0)
    n = 2500
    bins = rng.integers(0, 32, size=(5, n)).astype(np.uint8)
    y = ((bins[0] > 15) ^ (rng.random(n) < 0.35)).astype(np.int32) + 1
    for policy, look_ahead, initial, trees in ((2, 3, 1, 40), (2, 1, 0, 40), (1, 5, 3, 25), (2, 5, 30, 12), (0, 5, 0, 6)):
        cfg = O.default_config(num_trees=trees, max_depth=5, shrinkage=0.3, min_examples=2, early_stopping=policy,
                               early_stopping_num_trees_look_ahead=look_ahead, early_stopping_initial_iteration=initial)
        r = O.gbt_train_validated(bins, [32] * 5, [0] * 5, y, cfg, 0.2)
        want = D.early_stopping(list(r["valid_loss"]), policy, look_ahead, initial, 1, trees)
        assert want["logged"] == r["num_entries"], (policy, want, r["num_entries"])
        assert want["kept_trees"] == len(r["trees"]), (policy, want, len(r["trees"]))
        assert np.float32(want["final_loss"]) == np.float32(r["validation_loss"])
        assert want["triggered"] == r["early_stopping_triggered"]
        assert want["trained"] >= want["logged"] and (want["trained"] % D.TRAIN_BATCH == 0 or want["trained"] == trees)


def test_early_stopping_trains_whole_batches():
    losses = [5.0, 4.0, 3.0, 3.5, 3.6, 3.7, 3.8, 3.9, 4.0, 4.1, 4.2]
    r = D.early_stopping(losses, 2, 2, 0, 1, 20)
    assert r["logged"] == 5 and r["trained"] == 8 and r["kept_trees"] == 3 and r["triggered"]
    r = D.early_stopping(losses, 2, 2, 0, 3, 20)   # K = 3: trees, not iterations, are counted
    assert r["logged"] == 4 and r["kept_trees"] == 9
    r = D.early_stopping(losses[:3], 2, 2, 5, 1, 3)   # too few iterations: whole model, last loss
    assert r == dict(trained=3, logged=3, kept_trees=3, final_loss=np.float32(3.0), triggered=False)


def test_selection_aware_bucket_sums_match_brute_force():
    """The sums of a node's SELECTED rows (subsample / GOSS): bucket_sums on the filtered rows, for byte codes and for a
    presorted column's distinct values, against per-row loops."""
    rng = np.random.default_rng(5)
    n, B = 3000, 37
    codes = rng.integers(0, B, size=n)
    g = rng.normal(size=n).astype(np.float32)
    w = rng.uniform(0, 3, size=n).astype(np.float32)
    sel = rng.random(n) < 0.4
    node = np.sort(rng.choice(n, size=1200, replace=False))
    q, hq = quantize_q24(g, 4.0), quantize_second(w, 4.0)
    rows = node[sel[node]]
    cnt, s, h = S.bucket_sums(codes, rows, q, hq, B)
    for b in range(B):
        members = [i for i in node if sel[i] and codes[i] == b]
        assert cnt[b] == len(members)
        assert s[b] == sum(int(q[i]) - 2 ** 23 for i in members)
        assert h[b] == sum(int(hq[i]) for i in members)
    vals = np.round(rng.normal(size=n), 1).astype(np.float32)
    distinct, inv = np.unique(vals[rows], return_inverse=True)
    cnt, s, _ = S.bucket_sums(inv, np.arange(len(rows)), q[rows], hq[rows], len(distinct))
    for k, v in enumerate(distinct):
        members = [i for i in node if sel[i] and vals[i] == v]
        assert cnt[k] == len(members) and s[k] == sum(int(q[i]) - 2 ** 23 for i in members)


def _tree(features):
    """A pre-order tree of root + two leaves per split in `features` (one split: nodes 0, 1 (neg), 2 (pos))."""
    dt = np.dtype([("feature", "<i4"), ("neg_child", "<i4"), ("pos_child", "<i4")])
    t = np.zeros(3, dt)
    t[0] = (features, 1, 2)
    t[1] = (-1, -1, -1)
    t[2] = (-1, -1, -1)
    return t


def test_tie_expectation_follows_a_known_stream():
    """Three one-split trees over F = 6 features, mode 2 (libc++ shuffle) with draw seeds: each root draws one shuffle
    plus 6 words.  Tree 0: feature 0 chosen, feature 4 tied and a twin -> renamed iff 4 precedes 0 in its shuffle.
    Tree 1: feature 1 chosen, 3 tied but cutting the rows differently -> unresolved iff 3 precedes 1.  Tree 2: four
    tied alternatives -> unresolved whatever the order."""
    F, seed = 6, 77
    rows = np.arange(10)
    side = rows >= 4
    found = np.ones(F, np.int32)

    def cand(tied, twin):
        score = np.where(np.isin(np.arange(F), tied), 2.0, 1.0).astype(np.float32)
        return {0: (found, score, lambda f: side if f in twin else ~side)}

    trees = [_tree(0), _tree(1), _tree(0)]
    cands = [cand([0, 4], {0, 4}), cand([1, 3], {1}), cand([0, 1, 2, 3, 5], {0, 1, 2, 3, 5})]
    ref = O.Rng(seed)
    ref.discard(5)
    perms = []
    for _ in trees:
        perms.append(ref.shuffle_libcxx(F))
        ref.discard(F)
    rng = O.Rng(seed)
    rng.discard(5)
    renames, n_renamed, n_unresolved = D.tie_expectation(trees, cands, rng, 2, 1, F)
    want_renames = {(0, 0): 4} if perms[0].index(4) < perms[0].index(0) else {}
    want_unresolved = (1 if perms[1].index(3) < perms[1].index(1) else 0) + 1
    assert renames == want_renames and n_renamed == len(want_renames) and n_unresolved == want_unresolved
    # the stream continues across trees: the same walk from one position later differs in its shuffles
    assert rng.position == ref.position
