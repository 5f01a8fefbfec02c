"""Numpy restatement of candidate feature sampling (include/ygg_b200.h, DESIGN.md §23): k, the keyed candidate order and
the selection of a node's split from its candidates.  Shares no code with the engine."""
import math

import numpy as np


def mix(z):
    """SplitMix64's finalizer on uint64 numpy values (wrapping arithmetic)."""
    with np.errstate(over="ignore"):
        z = np.asarray(z, np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def keys(seed, tree, node, features):
    """key(seed, tree, node, f) for every f of `features` (arrays broadcast)."""
    def u32(v):   # an int32 argument's bits, as the C ABI takes it
        return (np.asarray(v, np.int64) & 0xFFFFFFFF).astype(np.uint64)
    z = mix(u32(seed))
    z = mix(z ^ u32(tree))
    z = mix(z ^ u32(node))
    return mix(z ^ u32(features))


def order(seed, tree, node, num_features):
    """The node's candidate order: features by ascending (key, f)."""
    k = keys(seed, tree, node, np.arange(num_features))
    return np.lexsort((np.arange(num_features), k))


def num_candidate_attributes(F, loss, num=-1, ratio=None):
    """NumAttributesToTest (training.cc:4244-4289); loss 1 = squared error (regression), else classification."""
    # the float ratio times the count in float32, as the reference's float proto field times an int
    k = int(math.ceil(np.float32(ratio) * np.float32(F))) if ratio is not None and ratio >= 0 else int(num)
    if k == 0:
        k = int(math.ceil(F / 3)) if loss == 1 else int(math.ceil(math.sqrt(F)))
    if k == -1:
        k = F
    return min(k, F)


def select(seed, tree, node, tried, found, score, k_valid):
    """The feature a node splits on (-1: none): the first maximum float score > 0 among the features taken in the node's
    order until k_valid of them were tried (all when fewer)."""
    best, best_score = -1, np.float32(0)
    seen = 0
    for f in order(seed, tree, node, len(tried)):
        if seen >= k_valid:
            break
        seen += int(tried[f])
        if found[f] and np.float32(score[f]) > best_score:
            best, best_score = int(f), np.float32(score[f])
    return best


def tried_from_counts(cnt, min_obs):
    """Whether a scan over buckets with row counts `cnt` (in scan order) scores at least one boundary."""
    cs = np.cumsum(np.asarray(cnt, np.int64))[:-1]
    n = int(np.sum(cnt))
    return bool(((cs >= min_obs) & (n - cs >= min_obs)).any())
