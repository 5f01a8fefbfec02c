"""Seeded training configurations for the exact fuzz (tests/test_gpu_exact_fuzz.py), and the host rules it checks them by.

`draw(seed)` returns one configuration a single-GPU handle accepts: rows, columns (byte, wide and presorted, with twins
when the tie-break replay is drawn), loss, gain, tree limits, leaf settings, row and candidate sampling, growth, hold-out,
early stopping and the driving call.  The engine's refusals are restated in `refusal()`, read from ygg_gbt_create,
ygg_gbt_set_weights_f32, ygg_gbt_set_candidate_sampling, ygg_debug_capture_candidates, ygg_gbt_train and the level slot
bound of configure_launches; every draw passes it.

`early_stopping()` restates EarlyStoppingState and the finalisation of ygg_gbt_train, `tie_expectation()` the tie-break
replay (k_select_local's tie record, k_verify_ties, resolve_tree_on_host).  Plain numpy; no device."""
import numpy as np

F32 = np.float32

SUITE_SEEDS = range(0, 40)   # the seeds tests/test_gpu_exact_fuzz.py runs
ROWS =(1, 7, 300, 8191, 8193, 30000, 100000)
BIG_ROWS = 2 ** 18 + 5
KINDS = ("num", "cat", "wide_num", "wide_cat", "pre")
TWIN_KINDS = ("copy", "wide_values", "pre_scaled", "cat_permuted")
TRAIN_BATCH = 8          # ygg_gbt_train's kBatch: iterations stepped between two reads of the validation losses
MAX_TIE_ALTS = 3         # kMaxTieAlts


# ---------------------------------------------------------------------------------------------------------------------
# the draw

def _column(rng, kind, wide_ok):
    if kind == "num":
        return dict(kind="num", B=int(rng.choice([2, 3, 16, 64, 255, 256, int(rng.integers(2, 257))])),
                    runs=bool(rng.random() < 0.5), const=bool(rng.random() < 0.1))
    if kind == "cat":
        return dict(kind="cat", B=int(rng.choice([2, 3, 7, 40, 256, int(rng.integers(2, 257))])),
                    absent=bool(rng.random() < 0.6))
    if kind == "wide_num":
        return dict(kind="wide_num", B=int(rng.choice([257, 300, 4096, 65535, int(rng.integers(257, 65536))])))
    if kind == "wide_cat":
        return dict(kind="wide_cat", B=int(rng.choice([257, 700, 5000, int(rng.integers(257, 5001))])))
    return dict(kind="pre")


def draw(seed):
    """One configuration: a dict of plain values (see the module docstring)."""
    rng = np.random.default_rng([seed, 0x5EED])
    d = dict(seed=seed)
    d["n"] = BIG_ROWS if rng.random() < 0.03 else int(rng.choice(ROWS))
    loss = int(rng.choice([0, 1, 2], p=[0.4, 0.35, 0.25]))
    K = 2 + seed % 4 if loss == 2 else 1
    d["K"] = K
    # growth and ties first: they decide which other options are allowed
    best_first = bool(rng.random() < 0.15)
    replay = 0 if best_first or rng.random() < 0.7 else int(rng.integers(1, 3))
    d["replay"] = replay
    F = int(rng.integers(1, 13))
    wide_ok = d["n"] <= 100000
    kinds = rng.choice(KINDS, size=F, p=[0.35, 0.25, 0.12, 0.08, 0.2] if wide_ok else [0.55, 0.35, 0, 0, 0.1])
    cols = [_column(rng, str(k), wide_ok) for k in kinds]
    if replay:
        for _ in range(int(rng.integers(1, 3))):
            src = int(rng.integers(0, len(cols)))
            kind = cols[src]["kind"]
            twin = {"num": "copy", "cat": str(rng.choice(["copy", "cat_permuted"])), "wide_num": "wide_values",
                    "wide_cat": "cat_permuted", "pre": "pre_scaled"}[kind]
            cols.append(dict(cols[src], twin=twin, of=src))
    d["columns"] = cols
    F = len(cols)
    d["F"] = F
    cfg = dict(loss=loss, random_seed=int(rng.integers(0, 2 ** 32)), num_trees=64)
    if loss == 2:
        cfg["num_classes"] = K
    cfg["use_hessian_gain"] = int(rng.random() < 0.35)
    cfg["l1_regularization"] = float(rng.choice([0.0, 0.0, 0.5]))
    cfg["l2_regularization"] = float(rng.choice([0.0, 1.0, 2.0]))
    cfg["l2_regularization_categorical"] = float(rng.choice([1.0, 3.0]))
    cfg["hessian_split_score_subtract_parent"] = int(rng.random() < 0.3)
    cfg["min_examples"] = int(rng.choice([1, 2, 5, 40]))
    cfg["in_split_min_examples_check"] = int(rng.random() < 0.8)
    cfg["sibling_subtraction"] = int(rng.random() < 0.8)
    depth = int(rng.choice([2, 3, 4, 5, 6, 7, 10], p=[0.15, 0.15, 0.2, 0.2, 0.15, 0.1, 0.05]))
    if depth == 10 and (not cfg["sibling_subtraction"] or F > 6 or best_first):
        depth = 6
    cfg["max_depth"] = depth
    cfg["shrinkage"] = float(rng.choice([0.1, 0.3, 1.0]))
    cfg["clamp_leaf_logit"] = float(rng.choice([5.0, 0.3])) if loss != 1 else 5.0
    if best_first:
        cfg["growing_strategy"] = 1
        cfg["max_num_nodes"] = int(rng.choice([-1, 3, 6, 13]))
    cfg["candidate_shuffle"] = replay
    cfg["rng_words_consumed"] = int(rng.choice([0, 0, 17]))
    cfg["split_jobs_draw_seeds"] = int(rng.random() < 0.5)
    d["scale"] = float(rng.choice([1.0, 10.0, 1e3])) if loss == 1 else 1.0
    # row sampling, weights: not with the replay (its check trains twice on one row stream)
    sampling = "none"
    if not replay and d["n"] >= 300:
        sampling = str(rng.choice(["none", "subsample", "goss"], p=[0.5, 0.25, 0.25]))
    if sampling == "goss" and (loss == 2 or cfg["use_hessian_gain"]):
        sampling = "subsample"
    if sampling == "subsample":
        cfg["subsample"] = float(rng.choice([0.3, 0.5, 0.9]))
    elif sampling == "goss":
        cfg["goss_alpha"] = float(rng.choice([0.1, 0.2, 0.3]))
        cfg["goss_beta"] = float(rng.choice([0.0, 0.1, 0.3]))
    d["sampling"] = sampling
    d["weights"] = bool(sampling != "goss" and not cfg["use_hessian_gain"] and rng.random() < 0.35)
    # candidate sampling (below F: not with the replay)
    d["candidates"] = None
    if not replay and F > 1 and rng.random() < 0.35:
        d["candidates"] = (-1, float(rng.choice([0.1, 0.3, 0.5]))) if rng.random() < 0.5 else \
            (int(rng.integers(0, F)), None)
    # hold-out and early stopping
    d["n_valid"] = int(rng.choice([0, 0, 7, 2000]))
    d["vweights"] = bool(d["n_valid"] and rng.random() < 0.5)
    es = 0
    if d["n_valid"] and rng.random() < 0.4:
        es = 1 + seed % 2
        cfg["early_stopping_num_trees_look_ahead"] = int(rng.choice([1, 2, 3, 5]))
        cfg["early_stopping_initial_iteration"] = int(rng.choice([0, 1, 3]))
    cfg["early_stopping"] = es
    d["drive"] = "train" if es or rng.random() < 0.3 else "step"
    d["iters"] = int(rng.integers(9, 14)) if es else (2 if K > 3 else 3)
    d["cfg"] = cfg
    assert refusal(d) is None, (seed, refusal(d))
    return d


def capture_allowed(d):
    """ygg_debug_capture_candidates: level-wise trees without the replay; and the scan check reads one tree per step."""
    return d["drive"] == "step" and d["replay"] == 0 and d["cfg"].get("growing_strategy", 0) == 0


def refusal(d):
    """The reason the engine would refuse the configuration, None when it accepts it."""
    c = d["cfg"]
    goss = c.get("goss_alpha", 0) > 0 or c.get("goss_beta", 0) > 0
    best_first = c.get("growing_strategy", 0) == 1
    F = len(d["columns"])
    if c["loss"] == 2 and not 2 <= c["num_classes"] <= 32:
        return "num_classes outside [2, 32]"
    if best_first and c["candidate_shuffle"]:
        return "the replay with best-first growth"
    if goss and c.get("subsample", 1.0) < 1:
        return "GOSS with subsample"
    if goss and (c["use_hessian_gain"] or c["loss"] == 2):
        return "GOSS with the hessian gain or the multinomial loss"
    if goss and c.get("goss_alpha", 0) == 0:
        return "GOSS may select no row"
    if d["weights"] and (goss or c["use_hessian_gain"]):
        return "weights with GOSS or the hessian gain"
    if d["candidates"] is not None:
        num, ratio = d["candidates"]
        if c["candidate_shuffle"] and _k(F, c["loss"], num, ratio) < F:
            return "candidate sampling below F with the replay"
    if c["candidate_shuffle"] and d["sampling"] != "none":
        return "row sampling with the replay check"
    # level slot bound: level l of the histogram holds 2^(l-1) slots with sibling subtraction, 2^l without, at most 254
    levels = c["max_depth"] + (1 if best_first else 0) - 1
    if levels > 1 and (1 << (levels - 1 - (1 if c["sibling_subtraction"] else 0))) > 254:
        return "more than 254 histogram slots"
    if c["max_depth"] < 2:
        return "max_depth < 2"
    if c["early_stopping"] and (not d["n_valid"] or d["drive"] != "train"):
        return "early stopping without a hold-out or outside train()"
    if d["vweights"] and not d["n_valid"]:
        return "validation weights without a hold-out"
    if d["sampling"] == "subsample" and d["n"] < 300:
        return "a subsample of a few rows may be empty"
    return None


def _k(F, loss, num, ratio):
    """NumAttributesToTest (tests/candidate_sampling_ref.num_candidate_attributes)."""
    from tests.candidate_sampling_ref import num_candidate_attributes
    return num_candidate_attributes(F, loss, num, ratio)


def coverage(seeds):
    """{option: number of draws of `seeds` that have it}."""
    out = {}

    def hit(key):
        out[key] = out.get(key, 0) + 1

    for s in seeds:
        d = draw(s)
        c = d["cfg"]
        hit(f"rows {d['n']}")
        hit(f"loss {c['loss']}")
        if c["loss"] == 2:
            hit(f"classes {c['num_classes']}")
        for col in d["columns"]:
            hit(f"column {col['kind']}")
            if col.get("runs"):
                hit("column num runs")
            if col.get("const"):
                hit("column num const")
            if col.get("absent"):
                hit("column cat absent")
            if "twin" in col:
                hit(f"twin {col['twin']}")
        hit(f"gain {'hessian' if c['use_hessian_gain'] else 'variance'}")
        for key in ("l1_regularization", "l2_regularization", "hessian_split_score_subtract_parent"):
            if c[key]:
                hit(key)
        if c["l2_regularization_categorical"] != 1.0:
            hit("l2_regularization_categorical")
        hit(f"in_split {c['in_split_min_examples_check']}")
        hit(f"sibling {c['sibling_subtraction']}")
        hit(f"depth {c['max_depth']}")
        if c["shrinkage"] == 1.0:
            hit("shrinkage 1")
        if c["clamp_leaf_logit"] < 5:
            hit("clamp")
        hit(f"sampling {d['sampling']}")
        if d["weights"]:
            hit("weights")
        if d["candidates"] is not None:
            hit("candidates ratio" if d["candidates"][1] is not None else "candidates num")
            hit(f"draw seeds {c['split_jobs_draw_seeds']}")
        if c.get("growing_strategy", 0):
            hit("best first")
        hit(f"replay {d['replay']}")
        if d["n_valid"]:
            hit("validation")
        if d["vweights"]:
            hit("validation weights")
        hit(f"early stopping {c['early_stopping']}")
        hit(f"drive {d['drive']}")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# data

def make_columns(d, rng, n):
    """Per column of the draw: dict(kind, codes (uint8 / uint16) or values (float32), B, values (wide bucket values)), for
    `n` rows."""
    out = []
    for col in d["columns"]:
        kind, B = col["kind"], col.get("B", 0)
        if "twin" in col:
            src = out[col["of"]]
            t = dict(src)
            if col["twin"] == "wide_values":
                t["values"] = np.cumsum(rng.uniform(0.5, 1.5, size=B)).astype(F32)
            elif col["twin"] == "pre_scaled":
                t["values"] = (src["values"] * F32(2)).astype(F32)
            elif col["twin"] == "cat_permuted":
                perm = rng.permutation(B)
                t["codes"] = perm[src["codes"]].astype(src["codes"].dtype)
            out.append(t)
            continue
        if kind == "num":
            c = np.clip(((rng.normal(size=n) + 3) / 6 * B).astype(np.int64), 0, B - 1)
            if col["runs"] and B > 8:   # runs of empty buckets, and empty trailing buckets
                c = np.where((c % 7 == 3) | (c >= B - 3), np.maximum(c - 1, 0), c)
            if col["const"]:
                c = np.full(n, int(rng.integers(0, B)))
            out.append(dict(kind=kind, codes=c.astype(np.uint8), B=B, values=None))
        elif kind == "cat":
            p = 1.0 / np.arange(1, B + 1) ** 1.1
            if col["absent"] and B > 2:
                p[rng.choice(B, size=max(1, B // 5), replace=False)] = 0.0
            p /= p.sum()
            out.append(dict(kind=kind, codes=rng.choice(B, size=n, p=p).astype(np.uint8), B=B, values=None))
        elif kind == "wide_num":
            c = np.where(rng.random(n) < 0.5, rng.integers(0, min(B, 256), size=n), rng.integers(B - B // 3 - 1, B, size=n))
            out.append(dict(kind=kind, codes=c.astype(np.uint16), B=B,
                            values=np.cumsum(rng.uniform(0.1, 1.0, size=B)).astype(F32)))
        elif kind == "wide_cat":
            p = 1.0 / np.arange(1, B + 1) ** 1.05
            out.append(dict(kind=kind, codes=rng.choice(B, size=n, p=p / p.sum()).astype(np.uint16), B=B, values=None))
        else:   # presorted: ties, -0.0 / +0.0, NaN
            v = np.round(rng.normal(size=n), 2).astype(F32)
            v[rng.random(n) < 0.1] = F32(-0.0)
            v[rng.random(n) < 0.1] = F32(0.0)
            v[rng.random(n) < 0.05] = np.nan
            out.append(dict(kind=kind, values=v, B=0))
    return out


def signal(col):
    """A standardised float view of a column, for the labels."""
    v = np.nan_to_num(np.asarray(col["values"] if col["kind"] == "pre" else col["codes"], np.float64))
    return (v - v.mean()) / (v.std() + 1e-9)


# ---------------------------------------------------------------------------------------------------------------------
# early stopping (EarlyStoppingState, ygg_gbt_train)

def early_stopping(losses, policy, look_ahead, initial_iteration, K, num_iters):
    """The device's validation losses of the iterations, as ygg_gbt_validation_loss returns them (at least those up to
    the stop) -> dict(trained: iterations stepped (whole batches), logged: iterations kept in the logs, kept_trees,
    final_loss, triggered).  policy 0 (none) leaves the model whole."""
    if policy == 0:
        return dict(trained=num_iters, logged=num_iters, kept_trees=num_iters * K, final_loss=losses[num_iters - 1],
                    triggered=False)
    best_loss, best_trees, last_loss, last_trees = 0.0, -1, 0.0, 0
    stop = -1
    for it in range(min(num_iters, len(losses))):
        v = F32(losses[it])
        if it >= initial_iteration and (best_trees == -1 or v < best_loss):
            best_loss, best_trees = v, (it + 1) * K
        last_loss, last_trees = v, (it + 1) * K
        if policy == 2 and it >= initial_iteration and last_trees - best_trees >= look_ahead:
            stop = it
            break
    logged = stop + 1 if stop >= 0 else num_iters
    trained = min(num_iters, -(-logged // TRAIN_BATCH) * TRAIN_BATCH)
    if logged < initial_iteration + 1:
        return dict(trained=trained, logged=logged, kept_trees=logged * K, final_loss=last_loss, triggered=False)
    return dict(trained=trained, logged=logged, kept_trees=best_trees, final_loss=best_loss, triggered=True)


# ---------------------------------------------------------------------------------------------------------------------
# the tie-break replay

def tie_expectation(trees, candidates, rng, mode, draw_seeds, F):
    """The replay's outcome on the trees of a run without it (mode 0).

    trees: the mode-0 trees in training order; candidates[t]: {pre-order node: (found [F], score [F], went_pos)} for the
    nodes of tree t that reached the scan (`candidate`), went_pos(f) the side (bool per row of the node) feature f's
    candidate sends the node's rows to, None for a wide categorical column; rng: an oracle Rng positioned at
    rng_words_consumed.  Nodes are visited depth-first, positive child first; each one
    draws a shuffle of the F features (mode 1: libstdc++'s std::shuffle, 2: libc++'s), then F discarded words with
    split_jobs_draw_seeds.  The tied set of a split is the other features with `found` and a float score equal to the
    best; more than MAX_TIE_ALTS of them: unresolved; else the first of the tied set in shuffle order, if it precedes
    the chosen feature, renames the node when its candidate sends every row of the node to the chosen side (and is not
    a wide categorical column), else the node is unresolved.
    -> ({(tree, node): new feature}, renamed count, unresolved count)."""
    renames, unresolved = {}, 0
    for t, tree in enumerate(trees):
        cand = candidates[t]
        stack = [0]
        while stack:
            i = stack.pop()
            if i not in cand:
                continue
            perm = rng.shuffle_libcxx(F) if mode == 2 else rng.shuffle(F)
            if draw_seeds:
                rng.discard(F)
            nd = tree[i]
            f0 = int(nd["feature"])
            if f0 < 0:
                continue
            found, score, went_pos = cand[i]
            sc = np.where(found != 0, score, 0).astype(F32)
            best = sc[f0]
            tied = [f for f in range(F) if f != f0 and found[f] and F32(score[f]) == best]
            if tied:
                rank = {f: r for r, f in enumerate(perm)}
                first = min(tied[:MAX_TIE_ALTS], key=lambda f: rank[f])
                if len(tied) > MAX_TIE_ALTS:
                    unresolved += 1
                elif rank[first] < rank[f0]:
                    pos = went_pos(first)
                    if pos is not None and np.array_equal(pos, went_pos(f0)):
                        renames[(t, i)] = first
                    else:
                        unresolved += 1
            stack.append(int(nd["neg_child"]))
            stack.append(int(nd["pos_child"]))
    return renames, len(renames), unresolved
