"""Shared helpers for the parity tests: synthetic data (SURVEY.md §8d generator), tree comparison."""
import numpy as np


def synth(n, f, seed=1234, informative=None, task="binary", bins=255, sample=100000):
    """X ~ N(0,1) [f, n]; y = 1[sum_j w_j x_j + 0.5 x0 x1 + 0.3 sin(3 x2) + eps > 0] (binary) or the
    margin itself (regression).  Returns (bins uint8 [f, n], num_bins, na_bin, labels)."""
    import ydf_b200
    rng = np.random.default_rng(seed)
    informative = informative or min(10, f)
    w = rng.normal(size=informative)
    margin = np.zeros(n, dtype=np.float64)
    out = np.empty((f, n), dtype=np.uint8)
    nb, na = [], []
    cols = {}
    for j in range(f):
        x = rng.normal(size=n).astype(np.float32)
        if j < informative:
            margin += w[j] * x
        if j < 3:
            cols[j] = x
        b, mean = ydf_b200.discretize_boundaries(x[:sample], bins, 3)
        nbin = len(b) + 1
        nab = int(np.searchsorted(b, np.float32(mean), side="right"))
        out[j] = ydf_b200.discretize_encode(x, b, nab)
        nb.append(nbin)
        na.append(nab)
    if f >= 3:
        margin += 0.5 * cols[0] * cols[1] + 0.3 * np.sin(3 * cols[2])
    margin += rng.normal(scale=0.5, size=n)
    if task == "binary":
        y = (margin > 0).astype(np.int32) + 1
    else:
        y = margin.astype(np.float32)
    return out, np.array(nb, np.int32), np.array(na, np.int32), y


def synth_mixed(n, f_num, cat_sizes, seed=77, task="binary", bins=64):
    """Numerical features as in synth() plus one categorical feature per entry of `cat_sizes`
    (number_of_unique_values incl. index 0 = <OOD>; skewed frequencies, some categories empty, a
    per-category effect on the margin).  Returns (bins, num_bins, na_bin, feature_type, labels)."""
    b, nb, na, _ = synth(n, f_num, seed=seed, task="regression", bins=bins)
    rng = np.random.default_rng(seed + 1)
    margin = np.zeros(n)
    for j in range(min(f_num, 4)):
        margin += rng.normal() * (b[j].astype(np.float64) / nb[j] - 0.5) * 3
    cols, cnb, cna = [], [], []
    for k in cat_sizes:
        p = 1.0 / np.arange(1, k + 1) ** 1.1
        p[0] = p[-1] * 0.5                      # <OOD> is rare
        if k > 8:
            p[rng.choice(np.arange(1, k), size=max(1, k // 10), replace=False)] = 0.0  # unseen categories
        p /= p.sum()
        c = rng.choice(k, size=n, p=p).astype(np.uint8)
        effect = rng.normal(size=k)
        effect[rng.random(k) < 0.3] = 0.0
        margin += effect[c]
        cols.append(c)
        cnb.append(k)
        cna.append(int(np.bincount(c, minlength=k)[1:].argmax()) + 1 if k > 1 else 0)
    margin += rng.normal(scale=0.7, size=n)
    allb = np.concatenate([b, np.stack(cols)]) if cols else b
    ft = np.array([0] * f_num + [1] * len(cat_sizes), np.int32)
    # interleave so that shards / candidate order mix both kinds
    order = rng.permutation(len(ft))
    y = (margin > np.median(margin)).astype(np.int32) + 1 if task == "binary" else margin.astype(np.float32)
    return (np.ascontiguousarray(allb[order]), np.concatenate([nb, cnb]).astype(np.int32)[order],
            np.concatenate([na, cna]).astype(np.int32)[order], ft[order], y)


def compare_trees(a, b, score_rtol=1e-5, leaf_atol=1e-5, stat_rtol=1e-6, stat_atol_per_row=2e-8):
    """a, b: node arrays (pre-order).  Returns a list of mismatch strings (empty = parity)."""
    errs = []
    if len(a) != len(b):
        return [f"node count {len(a)} != {len(b)}"]
    for i, (x, y) in enumerate(zip(a, b)):
        for k in ("feature", "threshold_bin", "na_value", "depth", "neg_child", "pos_child",
                  "num_examples", "num_pos_examples", "condition_type"):
            if x[k] != y[k]:
                errs.append(f"node {i}: {k} {x[k]} != {y[k]}")
        if not np.array_equal(x["cat_mask"], y["cat_mask"]):
            errs.append(f"node {i}: cat_mask {x['cat_mask']} != {y['cat_mask']}")
        if abs(float(x["split_score"]) - float(y["split_score"])) > score_rtol * max(1e-30, abs(float(y["split_score"]))):
            errs.append(f"node {i}: split_score {x['split_score']} vs {y['split_score']}")
        if abs(float(x["leaf_value"]) - float(y["leaf_value"])) > leaf_atol:
            errs.append(f"node {i}: leaf_value {x['leaf_value']} vs {y['leaf_value']}")
        for s in range(3):
            d = abs(float(x["stat"][s]) - float(y["stat"][s]))
            # sums over n rows: 1e-6 relative, or 2e-8 per row (fixed-point resolution / 1-ulp
            # differences of the per-row gradients between devices)
            if d > max(stat_rtol * abs(float(y["stat"][s])), stat_atol_per_row * float(y["num_examples"]), 1e-9):
                errs.append(f"node {i}: stat[{s}] {x['stat'][s]} vs {y['stat'][s]}")
    return errs


def prune_noise_splits(tree, eps):
    """Collapses every split with split_score <= eps into a leaf (pre-order array in, pre-order array
    out).  On a pure node (constant gradients) the reference's double-precision variance arithmetic
    leaves +-1e-16 of rounding noise, so whether it still "splits" such a node into children with
    identical leaf values depends on the accumulation order; the GPU's integer sums give exactly 0
    (DESIGN.md §6).  Predictions are unaffected either way."""
    out = []

    def walk(i):
        nd = tree[i].copy()
        me = len(out)
        out.append(nd)
        if nd["feature"] >= 0 and nd["split_score"] <= eps:
            for k, v in (("feature", -1), ("threshold_bin", 0), ("na_value", 0), ("split_score", 0.0),
                         ("num_pos_examples", 0), ("condition_type", 0), ("neg_child", -1), ("pos_child", -1)):
                nd[k] = v
            nd["cat_mask"] = 0
        elif nd["feature"] >= 0:
            nd["neg_child"] = len(out)
            walk(int(tree[i]["neg_child"]))
            nd["pos_child"] = len(out)
            walk(int(tree[i]["pos_child"]))
        out[me] = nd

    walk(0)
    return np.array(out, dtype=tree.dtype)


def drop_absent_categories(tree, bins):
    """Clears, in every categorical split, the mask bits of categories that no row of the node carries.
    Such categories have empty buckets (sort key 0); they can only change sides when a NON-empty bucket's key
    is exactly 0 as well (gradient sums that cancel exactly, e.g. iteration 0 of the multinomial loss with
    p = 1/K), which the 24-bit quantised sums do not reproduce bit for bit (DESIGN.md §6).  Training rows are
    unaffected by where absent categories go."""
    out = tree.copy()

    def walk(i, rows):
        nd = out[i]
        if nd["feature"] < 0:
            return
        b = bins[nd["feature"], rows].astype(np.int64)
        if nd["condition_type"] == 1:
            present = np.zeros(8, np.uint32)
            for c in np.unique(b):
                present[c >> 5] |= np.uint32(1) << np.uint32(c & 31)
            out[i]["cat_mask"] = nd["cat_mask"] & present
            go = ((nd["cat_mask"][b >> 5] >> (b & 31).astype(np.uint32)) & 1) != 0
        else:
            go = b >= nd["threshold_bin"]
        walk(int(nd["neg_child"]), rows[~go])
        walk(int(nd["pos_child"]), rows[go])

    walk(0, np.arange(bins.shape[1]))
    return out


def first_divergence(trees_a, trees_b, prune_noise=None, present_in=None, **kw):
    for t, (a, b) in enumerate(zip(trees_a, trees_b)):
        if prune_noise is not None:
            a, b = prune_noise_splits(a, prune_noise), prune_noise_splits(b, prune_noise)
        if present_in is not None:
            a, b = drop_absent_categories(a, present_in), drop_absent_categories(b, present_in)
        e = compare_trees(a, b, **kw)
        if e:
            return t, e
    return None, []


def pow2_cover(m):
    """Smallest power of two >= m (a normal float32 >= 0); 1 for m == 0: the histogram scale P of max|g| = m."""
    m = np.float32(m)
    if m == 0:
        return np.float32(1.0)
    f, e = np.frexp(m)          # m = f * 2^e, f in [0.5, 1)
    return np.float32(np.ldexp(np.float32(1.0), int(e) - 1 if f == 0.5 else int(e)))


def quantize_q24(g, P):
    """Biased 24-bit gradient code: clip(rint(g * 2^23 / P) + 2^23, 0, 2^24 - 1).  Exact in float32: the scale is a power
    of two, so g * 2^23 / P is the exact product, and integers up to 2^24 are float32 values."""
    g = np.asarray(g, np.float32)
    t = np.rint(g * np.float32(2.0 ** 23 / float(P))) + np.float32(2.0 ** 23)
    return np.clip(t, 0, 2 ** 24 - 1).astype(np.int64)


def quantize_second(v, V):
    """Hessian / weight code: min(rint(v * 2^24 / V), 2^24), 2^24 inclusive (v == V stays exact)."""
    v = np.asarray(v, np.float32)
    return np.minimum(np.rint(v * np.float32(2.0 ** 24 / float(V))), np.float32(2.0 ** 24)).astype(np.int64)


def level_histogram_ref(bins, slot_of_row, n_slots, g, second=None, V=None, features=None):
    """Integer reference of one level's slot histograms: per (slot, feature, bin) the sum of the biased gradient codes,
    the row count and (with `second`, quantised against the power of two V) the sum of the second-plane codes.
    -> (sum, count, second sum or None, P), int64 arrays of shape [n_slots, len(features), 256]."""
    features = range(bins.shape[0]) if features is None else features
    slot_of_row = np.asarray(slot_of_row)
    P = pow2_cover(np.abs(np.asarray(g, np.float32)).max() if len(g) else 0)
    q = quantize_q24(g, P)
    hq = quantize_second(second, V) if second is not None else None
    act = slot_of_row >= 0
    assert (int(act.sum()) + 1) * 2 ** 24 < 2 ** 53
    s = slot_of_row[act].astype(np.int64) * 256
    qa = q[act]
    ha = hq[act] if hq is not None else None
    shape = (n_slots, len(features), 256)
    out_s, out_c = np.zeros(shape, np.int64), np.zeros(shape, np.int64)
    out_h = np.zeros(shape, np.int64) if hq is not None else None
    for i, f in enumerate(features):
        key = s + bins[f][act]
        out_c[:, i, :] = np.bincount(key, minlength=n_slots * 256).reshape(n_slots, 256)
        # float64 accumulation of integers < 2^24 is exact while every partial sum stays below 2^53 (asserted above)
        out_s[:, i, :] = np.bincount(key, weights=qa, minlength=n_slots * 256).astype(np.int64).reshape(n_slots, 256)
        if hq is not None:
            out_h[:, i, :] = np.bincount(key, weights=ha, minlength=n_slots * 256).astype(np.int64).reshape(n_slots, 256)
    return out_s, out_c, out_h, P


def chunk_max_count(bins, chunk_blocks, features=None, block_rows=8192):
    """Largest number of rows of one aligned chunk of `chunk_blocks` row blocks that share a bin of one feature."""
    features = range(bins.shape[0]) if features is None else features
    n = bins.shape[1]
    n_blocks = (n + block_rows - 1) // block_rows
    n_chunks = (n_blocks + chunk_blocks - 1) // chunk_blocks
    chunk_of_row = np.arange(n) // (block_rows * chunk_blocks)
    best = 0
    for f in features:
        c = np.bincount(chunk_of_row * 256 + bins[f], minlength=n_chunks * 256)
        best = max(best, int(c.max()))
    return best


def predict_raw(trees, initial_prediction, bins):
    """Sum of the leaves reached by every column of `bins` ([F, n] bucket / dictionary codes) — numpy walk of
    ydf_b200.NODE_DTYPE trees (DiscretizedHigher and Contains conditions)."""
    n = bins.shape[1]
    rows = np.arange(n)
    raw = np.full(n, initial_prediction, np.float32)
    for t in trees:
        node = np.zeros(n, np.int64)
        while True:
            f = t["feature"][node]
            act = np.nonzero(f >= 0)[0]
            if len(act) == 0:
                break
            nd = node[act]
            v = bins[f[act], rows[act]].astype(np.int64)
            in_set = ((t["cat_mask"][nd, v >> 5] >> (v & 31).astype(np.uint32)) & 1) != 0
            go = np.where(t["condition_type"][nd] == 1, in_set, v >= t["threshold_bin"][nd])
            node[act] = np.where(go, t["pos_child"][nd], t["neg_child"][nd])
        raw += t["leaf_value"][node]
    return raw
