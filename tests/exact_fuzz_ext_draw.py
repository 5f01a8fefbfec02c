"""Seeded configurations for the extended exact fuzz (tests/test_gpu_exact_fuzz_ext.py): DART and columns binned from raw
float32 values on the GPU, on top of the configurations of tests/exact_fuzz_draw.py.

`draw(seed)` starts from `exact_fuzz_draw.draw(seed)`, unchanged, and draws the new options from its own stream
(`default_rng([seed, 0xDA27])`), so the exact fuzz's draws stay what they are:

- DART (about half of the draws): the dropout rate, and with it training weights, held-out weights and early stopping
  (each of the three policies through train(); none through step()) drawn more often than the base draw does;
- `disc8` / `disc16` columns: raw float32 values binned by `ydf_b200.DatasetBuilder` (`add_numerical_async`, at most
  256 bins / `add_numerical16_async`, 257..65535 bins: a wide column, or a byte column when the values leave at most
  256 bins), from value generators with NaN, ties, few distinct values, -0 / +0, constants, a huge range and a mean
  that lands on a present value;
- `disc_copy`: with the tie-break replay, the raw values of a discretized column binned again, whose splits tie.

`refusal()` is exact_fuzz_draw.refusal with DART's refusals and the DART harness's limit added.  Plain numpy; no
device."""
import numpy as np

from tests import exact_fuzz_draw as D

F32 = np.float32

SUITE_SEEDS = range(0, 40)   # the seeds tests/test_gpu_exact_fuzz_ext.py runs
DISC_KINDS = ("disc8", "disc16")
VALUE_KINDS = ("normal", "ties", "few", "zeros", "const", "huge", "mean_hit")
RATES = (0.0, 0.1, 0.5, 1.0)   # and "uniform": a rate drawn in (0, 1)


def _disc_column(rng, kind, n):
    col = dict(kind=kind, values=str(rng.choice(VALUE_KINDS)), nan=float(rng.choice([0.0, 0.05, 0.5])),
               min_obs=int(rng.choice([1, 3, 50])))
    if kind == "disc8":
        col["max_bins"] = int(rng.choice([4, 5, 16, 255, 256]))   # (the byte binning path takes 4..256)
    else:
        col["max_bins"] = int(rng.choice([257, 1024, 4096, 65535, int(rng.integers(257, 65536))]))
    # statistics on a prefix of the training rows (not with "mean_hit": its mean is set by the whole column)
    col["n_stats"] = int(rng.integers(1, n)) if n > 1 and col["values"] != "mean_hit" and rng.random() < 0.25 else 0
    return col


def draw(seed):
    """One configuration: exact_fuzz_draw.draw(seed) with the options of the module docstring added."""
    d = D.draw(seed)
    rng = np.random.default_rng([seed, 0xDA27])
    cfg = d["cfg"]
    n = d["n"]
    cols = d["columns"]
    # discretized columns, binned from raw values; 16-bit ones on the tables that take wide columns
    if rng.random() < 0.85:
        for _ in range(int(rng.integers(1, 4))):
            kind = "disc16" if n <= 100000 and rng.random() < 0.55 else "disc8"
            cols.append(_disc_column(rng, kind, n))
    if d["replay"]:
        disc = [i for i, c in enumerate(cols) if c["kind"] in DISC_KINDS]
        if disc and rng.random() < 0.8:
            src = int(rng.choice(disc))
            cols.append(dict(cols[src], twin="disc_copy", of=src))
    d["F"] = len(cols)
    if cfg["max_depth"] == 10 and d["F"] > 6:
        cfg["max_depth"] = 6
    # DART
    d["dart"] = None
    if rng.random() < 0.6:
        r = seed % (len(RATES) + 1)   # every rate class in every few seeds
        d["dart"] = float(RATES[r]) if r < len(RATES) else float(F32(rng.uniform(0.02, 0.98)))
        if (d["sampling"] == "none" and n >= 300 and not d["replay"] and cfg["loss"] != 2
                and not cfg["use_hessian_gain"] and not d["weights"] and rng.random() < 0.5):
            d["sampling"] = "goss"
            cfg["goss_alpha"] = float(rng.choice([0.1, 0.2, 0.3]))
            cfg["goss_beta"] = float(rng.choice([0.0, 0.1, 0.3]))
        goss = cfg.get("goss_alpha", 0) > 0
        if not d["weights"] and not goss and not cfg["use_hessian_gain"] and rng.random() < 0.6:
            d["weights"] = True
        if not d["n_valid"] and rng.random() < 0.5:
            d["n_valid"] = int(rng.choice([7, 2000]))
        if d["n_valid"] and not d["vweights"] and rng.random() < 0.7:
            d["vweights"] = True
        if d["replay"]:   # check_dart_run replays one candidate shuffle per tree, at its root
            cfg["max_depth"] = 2
            if n < 300:
                cfg["candidate_shuffle"] = d["replay"] = 0
                cols[:] = [col for col in cols if "twin" not in col]
                d["F"] = len(cols)
        if d["n_valid"] and rng.random() < 0.6:
            policy = int(rng.integers(0, 3))
            cfg["early_stopping"] = policy
            cfg["early_stopping_num_trees_look_ahead"] = int(rng.choice([1, 2, 3, 5]))
            cfg["early_stopping_initial_iteration"] = int(rng.choice([0, 1, 3]))
            d["drive"] = "train"
            d["iters"] = int(rng.integers(9, 14))
        else:
            cfg["early_stopping"] = 0
            d["drive"] = "step"
            d["iters"] = int(rng.integers(4, 7)) if d["K"] <= 3 else 3
    assert refusal(d) is None, (seed, refusal(d))
    return d


def refusal(d):
    """The reason the engine (or the DART harness) would refuse the configuration, None when both accept it."""
    why = D.refusal(d)
    if why is not None:
        return why
    for col in d["columns"]:
        lo, hi = (4, 256) if col["kind"] == "disc8" else (257, 65535)
        if col["kind"] in DISC_KINDS and not lo <= col["max_bins"] <= hi:
            return f"maximum_num_bins {col['max_bins']} outside [{lo}, {hi}] on the {col['kind']} binning path"
    if d.get("dart") is None:
        return None
    c = d["cfg"]
    if not 0.0 <= d["dart"] <= 1.0:
        return "a dropout rate outside [0, 1]"
    if d.get("shards") or d.get("set_predictions"):
        return "DART with sharding or set_predictions"
    if c["candidate_shuffle"] and (c["max_depth"] != 2 or d["n"] < 300):
        # check_dart_run replays one shuffle per tree, drawn at its root: the root must reach the scan
        return "DART with the replay above max_depth 2 or on fewer than 300 rows"
    if not c["early_stopping"] and d["drive"] == "train" and d["n_valid"]:
        return None   # policy NONE through train(): the early-stopping path
    if d["drive"] == "train" and not d["n_valid"]:
        return "DART through train() without a hold-out (check_dart_run steps)"
    return None


def coverage(seeds):
    """{option: number of draws of `seeds` that have it}, for the options this module adds."""
    out = {}

    def hit(key):
        out[key] = out.get(key, 0) + 1

    for s in seeds:
        d = draw(s)
        c = d["cfg"]
        for col in d["columns"]:
            if col["kind"] in DISC_KINDS:
                hit(f"column {col['kind']}")
                hit(f"values {col['values']}")
                hit(f"nan {col['nan']}")
                if col["n_stats"]:
                    hit("n_stats")
                if col.get("twin") == "disc_copy":
                    hit("twin disc_copy")
        if d["dart"] is None:
            continue
        hit("dart")
        rate = d["dart"]
        hit(f"dart rate {rate}" if rate in RATES else "dart rate uniform")
        hit(f"dart loss {c['loss']}")
        if d["vweights"]:
            hit("dart validation weights")
        if d["weights"]:
            hit(f"dart weighted loss {c['loss']}")
        if c.get("goss_alpha", 0) > 0:
            hit("dart goss")
        if c.get("subsample", 1.0) < 1:
            hit("dart subsample")
        if d["candidates"] is not None:
            hit("dart candidates")
        if c.get("growing_strategy", 0):
            hit("dart best first")
        if c["clamp_leaf_logit"] < 5:
            hit("dart clamp")
        if d["replay"]:
            hit("dart replay")
        if d["drive"] == "train":
            hit(f"dart early stopping {c['early_stopping']}")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# raw values

def disc_values(d):
    """{feature: float32 raw values of the training rows, then of the held-out rows} of the draw's discretized columns;
    a `disc_copy` twin holds its source's values.  The held-out rows always hold some NaN."""
    rng = np.random.default_rng([d["seed"], 0xDA27, 1])
    n, nv = d["n"], d["n_valid"]
    out = {}
    for f, col in enumerate(d["columns"]):
        if col["kind"] not in DISC_KINDS:
            continue
        if col.get("twin") == "disc_copy":
            out[f] = out[col["of"]]
            continue
        out[f] = np.concatenate([raw_values(col, rng, n, col["nan"]),
                                 raw_values(col, rng, nv, max(col["nan"], 0.05))]).astype(F32)
    return out


def raw_values(col, rng, n, nan_share):
    """float32 values of a discretized column for `n` rows, by its generator, with a share `nan_share` of NaN."""
    kind = col["values"]
    if kind == "normal":
        v = rng.normal(size=n) * float(rng.choice([1.0, 1e-3, 50.0]))
    elif kind == "ties":   # heavy ties on a few hundred values
        v = np.round(rng.exponential(size=n) * float(rng.choice([3.0, 40.0, 300.0])))
    elif kind == "few":    # fewer distinct values than 257: a 16-bit column ends as a byte column
        pool = np.sort(rng.normal(size=int(rng.integers(1, 200)))) * 10
        v = pool[rng.integers(0, len(pool), size=n)]
    elif kind == "zeros":  # -0.0 / +0.0 and a few other values
        v = np.where(rng.random(n) < 0.5, -0.0, 0.0)
        other = rng.random(n) < 0.2
        v[other] = np.round(rng.normal(size=int(other.sum())), 1)
    elif kind == "const":
        v = np.full(n, float(rng.choice([0.0, -2.5, 7.0])))
    elif kind == "huge":   # finite values over a huge range
        v = rng.normal(size=n) * np.exp(rng.uniform(-60, 60, size=n))
    else:                  # mean_hit: pairs c +- d (NaN by pairs), so that the mean of the present values is c itself
        c = float(rng.integers(-3, 4))
        m = n // 2
        dd = rng.integers(0, 40, size=m) * 0.25
        gone = rng.random(m) < nan_share
        if m:
            dd[0], gone[0] = 0.0, False   # c is present
        dd = np.where(gone, np.nan, dd)
        v = np.concatenate([c + dd, c - dd, np.full(n - 2 * m, c)])
        return v.astype(F32)[rng.permutation(n)]
    v = np.asarray(v, F32)
    if nan_share:
        v[rng.random(n) < nan_share] = np.nan
    return v
