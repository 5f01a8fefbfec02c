"""Seeded sharded training configurations for tests/test_gpu_shard_exact.py, and the rule they are checked by.

`draw_sharded(seed)` returns one configuration the shard setters accept: byte numerical (some under the exact threshold
rule) and categorical columns, binomial or squared error, gain, weights, leaf settings, growth, the driving call, the
shard mode, the world size and how the rows are cut between the ranks.  The setters' refusals are restated in
`refusal()`, read from ygg_gbt_create, ygg_gbt_set_weights_f32, ygg_dataset_create, ygg_feature_shard,
ygg_gbt_set_row_shard*, ygg_gbt_set_feature_shard and the level slot bound of configure_launches; every draw passes it.

`cuts()` restates the row splits: contiguous slices of the table after an optional reordering.  Plain numpy; no
device."""
import numpy as np

SUITE_SEEDS = range(0, 24)   # the seeds tests/test_gpu_shard_exact.py runs
ROWS = (40, 1000, 8193, 20000, 40000)
MODES = ("rows", "rows_scatter", "features")
# how the rows are cut: i.i.d. slices; ordered by the bins of the most informative column; binomial rows ordered by
# label; tiny first ranks around the 8192-row block; the largest |label| on the last rank; the largest weight on
# rank 0 and most zero weights on the last rank
SPLITS = ("random", "by_bin", "by_label", "tiny", "label_last", "weight_skew")
TINY = (1, 8191, 8192, 8193)


def draw_sharded(seed):
    """One configuration: a dict of plain values (see the module docstring)."""
    rng = np.random.default_rng([seed, 0x5A59])
    d = dict(seed=seed)
    loss = int(rng.choice([0, 1]))
    best_first = bool(rng.random() < 0.2)
    F = int(rng.integers(2, 11))
    cols = []
    for _ in range(F):
        if rng.random() < 0.35:
            cols.append(dict(kind="cat", B=int(rng.choice([2, 5, 40, 256, int(rng.integers(2, 257))]))))
        else:
            B = int(rng.choice([2, 16, 64, 255, 256, int(rng.integers(2, 257))]))
            cols.append(dict(kind="num", B=B, exact=bool(rng.random() < 0.3), const=bool(rng.random() < 0.08)))
    d["columns"] = cols
    d["F"] = F
    cfg = dict(loss=loss, random_seed=int(rng.integers(0, 2 ** 32)), num_trees=8)
    cfg["use_hessian_gain"] = int(rng.random() < 0.35)
    cfg["l1_regularization"] = float(rng.choice([0.0, 0.0, 0.5]))
    cfg["l2_regularization"] = float(rng.choice([0.0, 1.0, 2.0]))
    cfg["l2_regularization_categorical"] = float(rng.choice([1.0, 3.0]))
    cfg["hessian_split_score_subtract_parent"] = int(rng.random() < 0.3)
    cfg["min_examples"] = int(rng.choice([1, 2, 5, 40]))
    cfg["in_split_min_examples_check"] = int(rng.random() < 0.7)
    cfg["sibling_subtraction"] = int(rng.random() < 0.75)
    depth = int(rng.choice([2, 3, 4, 5, 6, 7, 9, 10], p=[0.08, 0.1, 0.12, 0.12, 0.12, 0.1, 0.16, 0.2]))
    if depth >= 9 and (not cfg["sibling_subtraction"] or best_first):
        depth = 7 if not best_first else 6
    cfg["max_depth"] = depth
    cfg["shrinkage"] = float(rng.choice([0.1, 0.3, 1.0]))
    cfg["clamp_leaf_logit"] = float(rng.choice([5.0, 0.3])) if loss == 0 else 5.0
    if best_first:
        cfg["growing_strategy"] = 1
        cfg["max_num_nodes"] = int(rng.choice([-1, 3, 6, 13]))
    cfg["rng_words_consumed"] = int(rng.choice([0, 0, 17]))
    d["cfg"] = cfg
    d["scale"] = float(rng.choice([1.0, 10.0, 1e3])) if loss == 1 else 1.0
    d["weights"] = bool(not cfg["use_hessian_gain"] and rng.random() < 0.35)
    d["drive"] = str(rng.choice(["step", "train"]))
    d["iters"] = 3
    # the decomposition
    mode = str(rng.choice(MODES))
    world = int(rng.integers(2, 5))
    if mode == "features":
        world = min(world, F)
    elif mode == "rows_scatter":
        while world > 2 and (world > F or (world - 1) * -(-F // world) >= F):
            world -= 1
        if (world - 1) * -(-F // world) >= F:
            mode = "rows"
    d["mode"], d["world"] = mode, world
    kinds = ["by_bin", "tiny", "by_label" if loss == 0 else "label_last"] + (["weight_skew"] if d["weights"] else [])
    d["split"] = "random" if mode == "features" or rng.random() < 0.2 else str(rng.choice(kinds))
    n = int(rng.choice(ROWS))
    if d["split"] == "tiny":
        n = max(n, sum(TINY[:world - 1]) + 1000)
    d["n"] = n
    assert refusal(d) is None, (seed, refusal(d))
    return d


def cuts(d, n_rows=None):
    """[(begin, end)] of every rank in the reordered table: contiguous, the tiny split's first ranks 1, 8191, 8192,
    8193 rows in turn and the rest on the last rank."""
    n, world = d["n"] if n_rows is None else n_rows, d["world"]
    if d["mode"] == "features":
        return [(0, n)] * world
    if d["split"] == "tiny":
        sizes = list(TINY[:world - 1])
        sizes.append(n - sum(sizes))
    else:
        sizes = [(n * (r + 1)) // world - (n * r) // world for r in range(world)]
    ends = np.cumsum(sizes)
    return [(int(e - s), int(e)) for s, e in zip(sizes, ends)]


def refusal(d):
    """The reason the engine would refuse the configuration, None when it accepts it."""
    c = d["cfg"]
    best_first = c.get("growing_strategy", 0) == 1
    F, world, mode = len(d["columns"]), d["world"], d["mode"]
    if c["loss"] not in (0, 1):
        return "the multinomial loss is not combined with sharding"
    if d["weights"] and c["use_hessian_gain"]:
        return "weights with the hessian gain"
    if c["max_depth"] < 2:
        return "max_depth < 2"
    levels = c["max_depth"] + (1 if best_first else 0) - 1
    if levels > 1 and (1 << (levels - 1 - (1 if c["sibling_subtraction"] else 0))) > 254:
        return "more than 254 histogram slots"
    if world < 2:
        return "not sharded"
    if mode == "features" and F < world:
        return "fewer features than ranks"
    if mode == "rows_scatter" and (world > F or (world - 1) * -(-F // world) >= F):
        return "the features do not cut into world non-empty chunks"
    if mode != "features" and any(e - b < 1 for b, e in cuts(d)):
        return "a rank without rows"
    if d["split"] == "by_label" and c["loss"] != 0:
        return "label order is drawn for binomial rows"
    if d["split"] == "weight_skew" and not d["weights"]:
        return "the weight split needs weights"
    return None


def coverage(seeds):
    """{option: number of draws of `seeds` that have it}."""
    out = {}

    def hit(key):
        out[key] = out.get(key, 0) + 1

    for s in seeds:
        d = draw_sharded(s)
        c = d["cfg"]
        hit(f"loss {c['loss']}")
        hit(f"mode {d['mode']}")
        hit(f"world {d['world']}")
        hit(f"split {d['split']}")
        for col in d["columns"]:
            hit(f"column {col['kind']}")
            if col.get("exact"):
                hit("exact rule")
            if col["B"] == 256:
                hit(f"{col['kind']} 256")
        hit(f"gain {'hessian' if c['use_hessian_gain'] else 'variance'}")
        for key in ("l1_regularization", "l2_regularization", "hessian_split_score_subtract_parent",
                    "rng_words_consumed"):
            if c[key]:
                hit(key)
        if c["clamp_leaf_logit"] < 5:
            hit("clamp")
        hit(f"min_examples {c['min_examples']}")
        hit(f"in_split {c['in_split_min_examples_check']}")
        hit(f"sibling {c['sibling_subtraction']}")
        hit(f"depth {c['max_depth']}")
        if d["weights"]:
            hit("weights")
        if c.get("growing_strategy", 0):
            hit("best first")
        hit(f"drive {d['drive']}")
    return out
