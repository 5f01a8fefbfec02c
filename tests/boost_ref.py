"""Exact reference of one boosting iteration's row pipeline: predictions, gradients, fixed-point scales, node sums, node
fields, leaf values, split scores and losses, driven by the trees the device emitted (tests/test_gpu_boosting_exact.py).

Plain numpy, Python ints and Fractions.  Every formula names the kernel it restates (ygg_kernels.cuh / ygg_engine.cu).

FMA contraction (nvcc contracts a*b + c unless -fmad=false; read from `cuobjdump -sass` of libygg_b200.so for sm_90a):
- k_mc_grad: `(label == k) - e[k] * normalization` compiles to FFMA R, e, -norm, ind: ONE rounding of the exact value.
  `mc_gradients` restates it as the exact double product (float x float fits 48 bits) and the exact difference rounded once
  to float (TwoSum, see `sub_round_f32`).
- k_weight_sums_finish: `d = Sp*Wn - Sn*Wp` compiles to DMUL + DFMA, so d keeps the rounding error of one product
  (about 2^-53 of it).  What bounds that error relative to d is the weighted scan's floor (boundary_score): a boundary
  is only scored when |d| on the 24-bit histogram sums exceeds half a code unit per row, so the weighted means of the
  two sides differ by at least about one 24-bit unit, 2^-23 P.  k_weight_sums_finish recomputes d from the 31-bit node
  sums of the same rows, which agree with the 24-bit ones to within their rounding, so |Sn*Wp| / |d| stays below about
  2^24 and d's relative error near 2^-29: below a float ulp of the stored score.  `split_score_weighted` is the exact
  value, and the stored score is held to 1 float ulp of it (tests/test_gpu_boosting_exact.py probes a split at that
  floor).
- k_pred_grad's `label * pred - log(...)` may contract too, but label is 0 or 1: the product is exact either way.

Rounding that cannot be pinned: the device evaluates exp in double (exp_rn) and rounds once to float.  Where the double
value lies within a few double ulps of a float rounding midpoint, both float neighbours are legitimate.  `exp_f32` reports
those inputs; the gradients then come in two variants and the node sums in [lo, hi] intervals.
"""
from fractions import Fraction

import numpy as np

F32 = np.float32
S_BIAS = 1 << 30          # kSBias (ygg_device.cuh)
S_ONE = 1 << 31           # 2^kSBits
MIN_HESSIAN = 0.001       # kMinHessianForNewtonStep
AMBIGUOUS_ULPS = 4        # double ulps around a float midpoint within which exp's float rounding is free


# ---------------------------------------------------------------------------------------------------------------------
# routing

def route(tree, cols, sets=None):
    """{pre-order node: row indices} of every node: byte and wide codes against threshold_bin or the category mask /
    wide positive set (`sets`, Gbt.get_category_sets), presorted values ('pre': the stored values) >= threshold_value.
    `cols`: per feature (kind, codes or stored values, buckets, bucket values), kind 'num' / 'cat' / 'wide_num' /
    'wide_cat' / 'pre'."""
    out = {}
    sets = sets or {}

    def walk(i, rows):
        out[i] = rows
        nd = tree[i]
        if nd["feature"] < 0:
            return
        kind, codes, _, _ = cols[nd["feature"]]
        if kind == "pre":
            go = codes[rows] >= nd["threshold_value"]
        elif nd["condition_type"] == 1:
            b = codes[rows].astype(np.int64)
            words = sets[i] if kind == "wide_cat" else nd["cat_mask"]
            go = ((words[b >> 5] >> (b & 31).astype(np.uint32)) & 1) != 0
        else:
            go = codes[rows].astype(np.int64) >= nd["threshold_bin"]
        walk(int(nd["neg_child"]), rows[~go])
        walk(int(nd["pos_child"]), rows[go])

    walk(0, np.arange(len(cols[0][1])))
    return out


def leaf_of_rows(tree, rows_of, n):
    """Pre-order leaf index of every row."""
    leaf = np.full(n, -1, np.int64)
    for i, rows in rows_of.items():
        if tree[i]["feature"] < 0:
            leaf[rows] = i
    assert (leaf >= 0).all()
    return leaf


# ---------------------------------------------------------------------------------------------------------------------
# float helpers

def pow2_cover(m):
    """ygg_kernels.cuh pow2_cover: smallest power of two >= m (m a float >= 0), 1 for m == 0."""
    m = F32(m)
    if m == 0:
        return 1.0
    f, e = np.frexp(m)
    return float(np.ldexp(1.0, int(e) - 1 if f == 0.5 else int(e)))


def ulp32(x):
    x = F32(abs(x))
    return float(np.nextafter(x, F32(np.inf)) - x)


def exp_f32(x):
    """exp_rn (ygg_kernels.cuh): float(exp(double(x))).  -> (value, alternative, ambiguous): `alternative` is the float
    on the other side of the nearest rounding midpoint, used where the double lies within AMBIGUOUS_ULPS of it."""
    return f32_candidates(np.exp(np.asarray(x, F32).astype(np.float64)))


def f32_candidates(e):
    """The float rounding of the doubles `e`, the float across the nearest rounding midpoint, and whether `e` lies
    within AMBIGUOUS_ULPS double ulps of that midpoint."""
    e = np.asarray(e, np.float64)
    f = e.astype(F32)
    up = np.nextafter(f, F32(np.inf))
    dn = np.nextafter(f, F32(-np.inf))
    mid_up = (f.astype(np.float64) + up.astype(np.float64)) / 2
    mid_dn = (f.astype(np.float64) + dn.astype(np.float64)) / 2
    tol = AMBIGUOUS_ULPS * np.spacing(e)
    near_up = np.abs(e - mid_up) <= tol
    near_dn = np.abs(e - mid_dn) <= tol
    amb = (near_up | near_dn) & np.isfinite(e) & (e > 0)
    alt = np.where(near_up, up, np.where(near_dn, dn, f)).astype(F32)
    return f, alt, amb


def log_f32(x):
    """log_rn: float(log(double(x)))."""
    return np.log(np.asarray(x, F32).astype(np.float64)).astype(F32)


def sub_round_f32(a, b):
    """float(a - b) rounded ONCE from the exact difference of two doubles (an FFMA's result when b is an exact float x
    float product): TwoSum gives the exact s + err; only a double s that is a float midpoint needs err's sign."""
    a = np.asarray(a, np.float64)
    b = -np.asarray(b, np.float64)
    s = a + b
    bb = s - a
    err = (a - (s - bb)) + (b - bb)
    f = s.astype(F32)
    fd = f.astype(np.float64)
    other = np.where(s > fd, np.nextafter(f, F32(np.inf)), np.nextafter(f, F32(-np.inf)))
    tie = (s != fd) & (np.abs(s - fd) == np.abs(other.astype(np.float64) - s)) & (err != 0)
    # at a tie the exact value lies on err's side of s
    toward = np.where(err > 0, np.maximum(f, other), np.minimum(f, other))
    return np.where(tie, toward, f).astype(F32)


# ---------------------------------------------------------------------------------------------------------------------
# gradients (k_pred_grad, k_mc_grad, k_apply_weights)

def binomial_gradients(pred, positive, alt=False):
    """k_pred_grad<0>: proba = 1 / (1 + exp_rn(-pred)) in float, g = label - proba, h = proba (1 - proba).
    -> (g, h, ambiguous rows); alt=True takes the other rounding of exp on the ambiguous rows."""
    pred = np.asarray(pred, F32)
    e, e_alt, amb = exp_f32(-pred)
    if alt:
        e = np.where(amb, e_alt, e)
    proba = F32(1) / (F32(1) + e)
    label = np.asarray(positive, F32)
    g = (label - proba).astype(F32)
    h = (proba * (F32(1) - proba)).astype(F32)
    return g, h, amb


def squared_error_gradients(pred, y):
    """k_pred_grad<1>: g = label - pred, h = 1."""
    g = (np.asarray(y, F32) - np.asarray(pred, F32)).astype(F32)
    return g, np.ones_like(g), np.zeros(len(g), bool)


def mc_gradients(pred, label, flip=None):
    """k_mc_grad: pred [K, n], label class 0..K-1.  e_k = exp_rn(pred_k), summed in float in class order,
    norm = 1 / sum, g_k = fma(-e_k, norm, [label == k]) (contracted, one rounding), a = |g_k|, h_k = a (1 - a).
    `flip` [K, n] bool: take exp's other rounding there.  -> (g [K, n], h [K, n], ambiguous [K, n])."""
    pred = np.asarray(pred, F32)
    K, n = pred.shape
    e, e_alt, amb = exp_f32(pred)
    if flip is not None:
        e = np.where(flip, e_alt, e)
    s = np.zeros(n, F32)
    for k in range(K):
        s = (s + e[k]).astype(F32)
    norm = (F32(1) / s).astype(F32)
    g = np.empty((K, n), F32)
    h = np.empty((K, n), F32)
    for k in range(K):
        ind = (np.asarray(label) == k).astype(np.float64)
        g[k] = sub_round_f32(ind, e[k].astype(np.float64) * norm.astype(np.float64))
        a = np.abs(g[k])
        h[k] = (a * (F32(1) - a)).astype(F32)
    return g, h, amb


def weigh(g, h, w, unit_hessian):
    """k_pred_grad<., WEIGHTED> / k_apply_weights / k_mc_grad<true>: wg = g * w, h -> w * h (w with unit hessians),
    g2w = wg * g.  All float products."""
    g = np.asarray(g, F32)
    w = np.asarray(w, F32)
    wg = (g * w).astype(F32)
    wh = w.copy() if unit_hessian else (w * np.asarray(h, F32)).astype(F32)
    return wg, wh, (wg * g).astype(F32)


# ---------------------------------------------------------------------------------------------------------------------
# row sampling (draw_sample / draw_goss, k_goss_apply)

def unit_draws(rng, m):
    """std::uniform_real_distribution<float> on the learner's mt19937: float(word) / 2^32, below 1."""
    words = np.array([rng.next() for _ in range(m)], np.uint64)
    u = (words.astype(F32) / F32(4294967296.0)).astype(F32)
    return np.minimum(u, np.nextafter(F32(1), F32(0)))


def subsample_mask(rng, n, ratio):
    """draw_sample: one engine word per row; the row is in iff its draw < subsample (an empty sample takes one row, not
    restated: the tests use samples far from empty)."""
    sel = unit_draws(rng, n) < F32(ratio)
    assert sel.any()
    return sel


def goss_selection(g, alpha, beta, rng):
    """draw_goss + k_goss_keys / sort / k_goss_apply: rows by decreasing |g| (stable: ties by row index); the first
    ceil(alpha * n) are kept with weight 1, each later row iff its draw (one per row of the tail, in that order) < beta,
    with weight (1 - alpha) / beta in float; rows outside the sample keep weight 1.  -> (selected bool [n], weight)."""
    g = np.asarray(g, F32)
    n = len(g)
    order = np.argsort(-np.abs(g).astype(np.float64), kind="stable")
    cutoff = min(int(np.ceil(F32(alpha) * F32(n))), n)
    sel = np.zeros(n, bool)
    w = np.ones(n, F32)
    sel[order[:cutoff]] = True
    if beta > 0:
        u = unit_draws(rng, n - cutoff)
        tail = order[cutoff:][u < F32(beta)]
        sel[tail] = True
        amp = (F32(1) - F32(alpha)) / F32(beta)
        w[tail] = F32(1) * amp
    return sel, w


# ---------------------------------------------------------------------------------------------------------------------
# quantisers (ygg_kernels.cuh quant_stat_signed / quant_stat_unsigned)

def quant_signed(v, P):
    """quant_stat_signed(v, 2^30 / P) WITHOUT the bias: clamp(rint(v * 2^30 / P), -2^30, 2^30) (exact float product)."""
    t = np.rint(np.asarray(v, F32) * F32(2.0 ** 30 / P))
    return np.clip(t, -S_BIAS, S_BIAS).astype(np.int64)


def quant_unsigned(v, V):
    """quant_stat_unsigned(v, 2^31 / V): min(rint(v * 2^31 / V), 2^31), v >= 0."""
    t = np.rint(np.asarray(v, F32) * F32(2.0 ** 31 / V))
    return np.minimum(t, S_ONE).astype(np.int64)


def g2_codes(g, P):
    """The sum-of-squares code of k_quantize / partition_impl: quant_stat_unsigned(g * g, 2^31 / P^2), float product."""
    g = np.asarray(g, F32)
    return quant_unsigned((g * g).astype(F32), P * P)


# ---------------------------------------------------------------------------------------------------------------------
# one tree

class Rows:
    """Per-row quantities one tree is trained on, in two variants (lo / hi codes: equal except on ambiguous rows)."""

    def __init__(self, g, h, sel, P, h_pow2, g_alt=None, h_alt=None, w=None, w_pow2=None, g2w=None, g2w_alt=None):
        g_alt = g if g_alt is None else g_alt
        h_alt = h if h_alt is None else h_alt
        self.P, self.h_pow2, self.w_pow2 = P, h_pow2, w_pow2
        self.sel = np.ones(len(g), bool) if sel is None else np.asarray(sel, bool)

        def pair(a, b):
            return np.minimum(a, b), np.maximum(a, b)

        self.sg = pair(quant_signed(g, P), quant_signed(g_alt, P))
        self.sg2 = pair(g2_codes(g, P), g2_codes(g_alt, P))
        self.sh = None if h is None else pair(quant_unsigned(h, h_pow2), quant_unsigned(h_alt, h_pow2))
        self.weighted = w is not None
        if self.weighted:
            g2w_alt = g2w if g2w_alt is None else g2w_alt
            self.g2pow2 = max(pow2_cover(np.max(g2w) if len(g2w) else 0), pow2_cover(np.max(g2w_alt) if len(g2w) else 0))
            self.ws = quant_unsigned(w, w_pow2)
            self.gws = pair(quant_unsigned(g2w, self.g2pow2), quant_unsigned(g2w_alt, self.g2pow2))

    def sums(self, rows):
        """Integer sums over the node's SELECTED rows: {name: (lo, hi)}, plus the row count.  The gradient sum is
        unbiased: the kernels' sum of biased codes minus n * 2^30, which k_node_stats subtracts exactly."""
        r = rows[self.sel[rows]]
        out = {"n": len(r)}

        def s(pair):
            return int(pair[0][r].sum()), int(pair[1][r].sum())

        out["sg"] = s(self.sg)
        out["sg2"] = s(self.sg2)
        if self.sh is not None:
            out["sh"] = s(self.sh)
        if self.weighted:
            out["w"] = (int(self.ws[r].sum()),) * 2
            out["g2w"] = s(self.gws)
        return out


def l1_threshold(v, l1):
    if l1 == 0.0:
        return v
    t = max(0.0, abs(v) - l1)
    return t if v > 0 else -t


def leaf_value(sum_g, sum_h, cfg, logit):
    """k_node_stats: float(shrinkage * l1(sum_g) / (max(sum_h, kMin) + l2)) in doubles, then the logit clamp."""
    num = l1_threshold(sum_g, float(F32(cfg.l1_regularization)))
    den = max(sum_h, MIN_HESSIAN) + float(F32(cfg.l2_regularization))
    v = F32(float(F32(cfg.shrinkage)) * num / den)
    if logit:
        c = F32(cfg.clamp_leaf_logit)
        v = min(max(v, -c), c)
    return F32(v)


def expected_stats(s, rows, cfg, logit):
    """Expected stat[0..2] of a node as intervals [(lo, hi)] x 3 (k_node_stats, k_weight_sums_finish), and the
    node's sum_h interval (None where stat carries it)."""
    P, n = rows.P, s["n"]
    ginv = P / 2.0 ** 30
    stat0 = tuple(float(v) * ginv for v in s["sg"])
    has_h = rows.sh is not None
    sum_h = tuple(float(v) * (rows.h_pow2 / 2.0 ** 31) for v in s["sh"]) if has_h else (float(n),) * 2
    if rows.weighted:
        stat1 = tuple(float(v) * (rows.g2pow2 / 2.0 ** 31) for v in s["g2w"])
        stat2 = tuple(float(v) * (rows.w_pow2 / 2.0 ** 31) for v in s["w"])
    elif cfg.use_hessian_gain:
        stat1 = tuple(max(v, MIN_HESSIAN) for v in sum_h)
        stat2 = (float(n),) * 2
    else:
        stat1 = tuple(float(v) * (P * P / 2.0 ** 31) for v in s["sg2"])
        stat2 = (float(n),) * 2
    return (stat0, stat1, stat2), sum_h


def split_score_variance(sp, sn, np_, nn, P):
    """Exact variance-gain score from the children's unbiased 31-bit gradient sums (k_node_stats, boundary_score):
    d = (sp nn - sn np) P / 2^30, score = d^2 / (np nn (np + nn)^2)."""
    d = Fraction(sp * nn - sn * np_) * Fraction(P) / 2 ** 30
    return d * d / (np_ * nn * (np_ + nn) ** 2)


def split_score_weighted(sp, sn, wp, wn, P, w_pow2):
    """Exact weighted variance-gain score (k_weight_sums_finish): weight sums wp / wn (codes, units of w_pow2 / 2^31) in
    place of the counts.  None when a side has no weight (the kernel keeps the scan's score)."""
    if wp == 0 or wn == 0:
        return None
    Wp, Wn = Fraction(wp) * Fraction(w_pow2) / 2 ** 31, Fraction(wn) * Fraction(w_pow2) / 2 ** 31
    d = (Fraction(sp) * Wn - Fraction(sn) * Wp) * Fraction(P) / 2 ** 30
    return d * d / (Wp * Wn * (Wp + Wn) ** 2)


def split_score_hessian(par_stat, pos, neg, rows, cfg, l2):
    """k_node_stats' double sequence: gp^2 / (max(Hp, kMin) + l2) + gn^2 / (max(Hn, kMin) + l2) - [parent term].
    pos / neg: the children's sums (single values)."""
    ginv = rows.P / 2.0 ** 30
    hinv = rows.h_pow2 / 2.0 ** 31
    l1 = float(F32(cfg.l1_regularization))
    terms = []
    for s in (pos, neg):
        S = float(s["sg"]) * ginv
        H = float(s["sh"]) * hinv if rows.sh is not None else float(s["n"])
        g = l1_threshold(S, l1)
        terms.append(g * g / (max(H, MIN_HESSIAN) + l2))
    score = terms[0] + terms[1]
    if cfg.hessian_split_score_subtract_parent:
        g0 = l1_threshold(par_stat[0], l1)
        score = score - g0 * g0 / (par_stat[1] + l2)
    return score


def check_tree(tree, rows_of, rows, cfg, logit, where=""):
    """Compares every node of a device tree with the reference sums over its rows.  -> list of mismatch strings."""
    errs = []
    sums = {}
    for i in range(len(tree)):
        sums[i] = rows.sums(rows_of[i])
    for i, nd in enumerate(tree):
        s = sums[i]
        at = f"{where} node {i}"
        if int(nd["num_examples"]) != s["n"]:
            errs.append(f"{at}: num_examples {nd['num_examples']} != {s['n']}")
            continue
        if nd["feature"] >= 0:
            npos = sums[int(nd["pos_child"])]["n"]
            if int(nd["num_pos_examples"]) != npos:
                errs.append(f"{at}: num_pos_examples {nd['num_pos_examples']} != {npos}")
        want, sum_h = expected_stats(s, rows, cfg, logit)
        for k in range(3):
            got = float(nd["stat"][k])
            lo, hi = want[k]
            if not lo <= got <= hi:
                errs.append(f"{at}: stat[{k}] {got!r} not in [{lo!r}, {hi!r}]")
        # leaf value from the device's own stat[0] (and stat[1] where it is the hessian sum).  With example weights
        # k_weight_sums_finish overwrites stat[1] with the (w*g)*g sum; the engine refuses weights with the hessian gain,
        # and this reference does not restate that combination either.
        assert not (rows.weighted and cfg.use_hessian_gain), "weights with the hessian gain are not restated"
        if cfg.use_hessian_gain:
            sh = (float(nd["stat"][1]),) * 2
        else:
            sh = sum_h
        if sh[0] == sh[1]:
            lv = leaf_value(float(nd["stat"][0]), sh[0], cfg, logit)
            if F32(nd["leaf_value"]) != lv:
                errs.append(f"{at}: leaf_value {nd['leaf_value']!r} != {lv!r}")
        if nd["feature"] < 0:
            continue
        p, q = sums[int(nd["pos_child"])], sums[int(nd["neg_child"])]
        if p["sg"][0] != p["sg"][1] or q["sg"][0] != q["sg"][1]:
            continue   # an ambiguous row in a child: the score is not pinned
        sp, sn = p["sg"][0], q["sg"][0]
        if rows.weighted:
            exact = split_score_weighted(sp, sn, p["w"][0], q["w"][0], rows.P, rows.w_pow2)
        elif cfg.use_hessian_gain:
            if rows.sh is not None and (p["sh"][0] != p["sh"][1] or q["sh"][0] != q["sh"][1]):
                continue
            l2 = float(F32(cfg.l2_regularization_categorical if nd["condition_type"] == 1 else cfg.l2_regularization))
            one = lambda d: {"sg": d["sg"][0], "n": d["n"], "sh": d["sh"][0] if "sh" in d else None}
            exact = split_score_hessian(nd["stat"], one(p), one(q), rows, cfg, l2)
        else:
            exact = split_score_variance(sp, sn, p["n"], q["n"], rows.P)
        if exact is None or exact <= 0:
            continue   # the kernels keep the scan's positive score
        w = F32(float(exact))
        if abs(float(nd["split_score"]) - float(w)) > ulp32(w):
            errs.append(f"{at}: split_score {nd['split_score']!r} vs exact {float(exact)!r}")
    return errs


# ---------------------------------------------------------------------------------------------------------------------
# losses (k_pred_grad / k_valid_update / k_mc_grad), per-row float terms

def binomial_loss_terms(pred, positive, w=None):
    """-> (loss terms in float, to be SUBTRACTED; correct counts).  inner = label * pred - log_rn(1 + exp_rn(pred)),
    term = 2 * inner (2 * w * inner); a row is correct when (pred > 0) == label."""
    pred = np.asarray(pred, F32)
    label = np.asarray(positive, F32)
    e, _, _ = exp_f32(pred)
    inner = (label * pred - log_f32(F32(1) + e)).astype(F32)
    term = (F32(2) * inner) if w is None else ((F32(2) * np.asarray(w, F32)).astype(F32) * inner)
    hit = (pred > 0) == (np.asarray(positive) != 0)
    return term.astype(F32), hit


def squared_error_terms(pred, y, w=None):
    d = (np.asarray(y, F32) - np.asarray(pred, F32)).astype(F32)
    if w is None:
        return (d * d).astype(F32)
    return ((np.asarray(w, F32) * d).astype(F32) * d).astype(F32)


def mc_loss_terms(pred, label, w=None):
    """k_mc_grad's loss part: log_rn(e[label] / sum_exp) (subtracted, times w), and the predicted class = the first
    strict maximum of the e_k."""
    pred = np.asarray(pred, F32)
    K, n = pred.shape
    e, _, _ = exp_f32(pred)
    s = np.zeros(n, F32)
    for k in range(K):
        s = (s + e[k]).astype(F32)
    el = e[np.asarray(label), np.arange(n)]
    term = log_f32((el / s).astype(F32))
    if w is not None:
        term = (np.asarray(w, F32) * term).astype(F32)
    predicted = np.argmax(e, axis=0)   # the first maximum
    return term, predicted == np.asarray(label)


def correct_units(w, w_pow2):
    """Weighted accuracy units: rint(w * 2^31 / w_pow2) per correct row (exact float product)."""
    return np.rint(np.asarray(w, F32) * F32(2.0 ** 31 / w_pow2)).astype(np.int64)


def sequential_sum(v):
    """A double sum in row order (the host's sum of the weights)."""
    return float(np.cumsum(np.asarray(v, np.float64))[-1]) if len(v) else 0.0
