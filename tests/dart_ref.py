"""Exact reference of DART's prediction accumulator and dropout draws (ygg_engine.cu draw_dart, ygg_kernels.cuh dart_update /
dart_sample), in numpy float32: one rounding per operation, no fused multiply-add, left to right.

State: `acc` [K, n], the full predictions, starting at the initial predictions; per past iteration j its trees' per-row
leaf values p_j [K, n] and its weight w_j.  Iteration i with dropped set D (ascending):
  sampled:  s = acc, then s = s - p_j * w_j for j in D                      (the gradients are taken at s)
  update:   w_new = 1 / (|D| + 1), sf = |D| / (|D| + 1)
            acc = acc + p_i * w_new, then acc = acc + (p_j * w_j) * (sf - 1) for j in D
            w_j = w_j * sf for j in D, w_i = w_new
The model keeps every leaf of iteration j scaled to leaf * w_j.
"""
import numpy as np

F32 = np.float32
TWO32 = 4294967296


def unit_float(word):
    """std::uniform_real_distribution<float> (libstdc++) on one mt19937 word: float(word) / 2^32, kept below 1."""
    u = F32(F32(int(word)) / F32(TWO32))
    return min(u, np.nextafter(F32(1), F32(0)))


def unit_float_libcxx(word):
    """libc++'s std::uniform_real_distribution<float> on one mt19937 word: float(word) / 2^32 as rounded, so the words
    from 2^32 - 128 on give 1.0."""
    return F32(F32(int(word)) / F32(TWO32))


def uniform_int_libstdcxx(next_word, n):
    """libstdc++'s std::uniform_int_distribution<int>(0, n - 1) on a 32-bit engine: Lemire's multiply-shift with rejection
    (one word per try, one word even for n == 1)."""
    product = next_word() * n
    low = product & 0xFFFFFFFF
    if low < n:
        threshold = (TWO32 - n) % n
        while low < threshold:
            product = next_word() * n
            low = product & 0xFFFFFFFF
    return product >> 32


def uniform_int_libcxx(next_word, n):
    """libc++'s std::uniform_int_distribution(0, n - 1): nothing drawn for n == 1, else the low w bits of one word
    (2^w >= n), redrawn while >= n."""
    if n == 1:
        return 0
    w = (n - 1).bit_length()
    while True:
        u = next_word() & ((1 << w) - 1)
        if u < n:
            return u


def draw_dropped(next_word, i, rate, libcxx):
    """The dropped set of iteration i: one unit draw per earlier iteration, dropped iff < rate; an empty set takes one
    iteration drawn uniformly.  `next_word`: the learner's mt19937, one 32-bit word per call; `libcxx` selects libc++'s
    unit draw and uniform integer, else libstdc++'s."""
    if i == 0:
        return []
    rate = F32(rate)
    unit = unit_float_libcxx if libcxx else unit_float
    dropped = [j for j in range(i) if unit(next_word()) < rate]
    if not dropped:
        dropped = [(uniform_int_libcxx if libcxx else uniform_int_libstdcxx)(next_word, i)]
    return dropped


class Accumulator:
    """DartPredictionAccumulator restated.  `init`: [K, n] (or [n]) initial predictions."""

    def __init__(self, init):
        self.acc = np.array(init, F32, ndmin=2)
        self.p = []   # per iteration: [K, n] leaf values
        self.w = []   # per iteration: weight (float32)

    def sampled(self, dropped):
        s = self.acc.copy()
        for j in dropped:
            s = (s - (self.p[j] * self.w[j]).astype(F32)).astype(F32)
        return s

    def update(self, p_new, dropped):
        """Adds iteration len(self.p) with per-row leaf values `p_new` ([K, n]) and dropped set `dropped`."""
        p_new = np.array(p_new, F32, ndmin=2)
        d = F32(len(dropped))
        w_new = F32(F32(1) / (d + F32(1)))
        sf = F32(d / (d + F32(1)))
        sf_m1 = F32(sf - F32(1))
        acc = (self.acc + (p_new * w_new).astype(F32)).astype(F32)
        for j in dropped:
            acc = (acc + ((self.p[j] * self.w[j]).astype(F32) * sf_m1).astype(F32)).astype(F32)
        self.acc = acc
        for j in dropped:
            self.w[j] = F32(self.w[j] * sf)
        self.p.append(p_new)
        self.w.append(w_new)

    def weights(self):
        return np.array(self.w, F32)


def weights_after(dropped_sets):
    """The weights after the given per-iteration dropped sets, replayed (ygg_engine.cu dart_weights_after)."""
    w = []
    for dropped in dropped_sets:
        d = F32(len(dropped))
        sf = F32(d / (d + F32(1)))
        for j in dropped:
            w[j] = F32(w[j] * sf)
        w.append(F32(F32(1) / (d + F32(1))))
    return np.array(w, F32)


def scaled_sum(init, leaves, weights, K=1):
    """The scaled model's raw score (k_predict<true>): init + leaf_t * w_{t // K} summed in tree order per class plane.
    `leaves`: [trees, n] leaf value of every row in every tree."""
    leaves = np.asarray(leaves, F32)
    n = leaves.shape[1]
    out = np.full((K, n), F32(init), F32)
    for t in range(leaves.shape[0]):
        out[t % K] = (out[t % K] + (leaves[t] * F32(weights[t // K])).astype(F32)).astype(F32)
    return out
