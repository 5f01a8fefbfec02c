"""Exact bucket sums of every node of one tree level, one pass per feature: a histogram provider for
tests/test_gpu_scan_exact.check_scan that scales to 10M rows x 200 features.

Every row of the level is keyed by `slot * B + code` (slot: the node's index in the level, -1: in no node) and its count,
unbiased gradient code (q - 2^23) and second-plane code are added into int64 planes with torch's index_add_.  Integer
addition is exact and does not depend on the order of the adds, so the result is the same on the CPU and on a device, and
the same as scan_ref.bucket_sums per node.  Presorted columns have no fixed buckets: the provider leaves them to
check_scan's per-node path."""
import numpy as np
import torch

Q_BIAS = 2 ** 23


def level_bucket_sums(slot, codes, q, hq, n_slots, num_bins):
    """(count, unbiased gradient-code sum, second-plane sum) per (slot, bucket), int64 tensors [n_slots, num_bins].
    slot: int64 [n], -1 for a row in no slot; codes: integer [n] in [0, num_bins); q: biased 24-bit gradient codes;
    hq: second-plane codes (int64 [n] each, on the device of `slot`)."""
    act = torch.nonzero(slot >= 0).squeeze(1)
    return _sums(slot[act], codes[act], q[act] - Q_BIAS, hq[act], n_slots, num_bins)


def _sums(slot_a, codes_a, sq_a, hq_a, n_slots, num_bins):
    key = slot_a * num_bins + codes_a.to(torch.int64)
    size = n_slots * num_bins
    z = lambda: torch.zeros(size, dtype=torch.int64, device=key.device)   # noqa: E731
    cnt = z().index_add_(0, key, torch.ones_like(key))
    s = z().index_add_(0, key, sq_a)
    hs = z().index_add_(0, key, hq_a)
    return cnt.view(n_slots, num_bins), s.view(n_slots, num_bins), hs.view(n_slots, num_bins)


class LevelHist:
    """check_scan's `hist_of`: hist(level, cap, rows_of, q, hq) -> sums(j, f) -> (cnt, s, hs) int64 numpy arrays of
    feature f's buckets over the rows of level node j (cap["node"][j]), or None for a presorted column.  `cols` as
    check_scan's; the codes are copied to `device` once.  Counts the levels, the (node, feature) sums it computed and the
    derived (sibling-subtracted) level nodes it saw in `self.levels`, `self.pairs` and `self.derived`."""

    def __init__(self, cols, device="cpu"):
        self.device = torch.device(device)
        self.B = [int(c[2]) for c in cols]
        self.n = len(cols[0][1])
        self.codes = {f: torch.from_numpy(np.ascontiguousarray(c[1])).to(self.device)
                      for f, c in enumerate(cols) if c[0] != "pre"}
        self.levels, self.pairs, self.derived = 0, 0, 0

    def __call__(self, level, cap, rows_of, q, hq):
        J = len(cap["node"])
        slot = torch.full((self.n,), -1, dtype=torch.int64)
        for j, node in enumerate(cap["node"]):
            r = torch.from_numpy(np.asarray(rows_of[int(node)], np.int64))
            assert bool((slot[r] == -1).all()), f"level {level}: a row in two nodes"
            slot[r] = j
        slot = slot.to(self.device)
        act = torch.nonzero(slot >= 0).squeeze(1)
        slot_a = slot[act]
        sq_a = torch.from_numpy(np.asarray(q, np.int64)).to(self.device)[act] - Q_BIAS
        hq_a = torch.from_numpy(np.asarray(hq, np.int64)).to(self.device)[act]
        out = {}
        for f, codes in self.codes.items():
            c, s, h = _sums(slot_a, codes[act], sq_a, hq_a, J, self.B[f])
            out[f] = (c.cpu().numpy(), s.cpu().numpy(), h.cpu().numpy())
        self.levels += 1
        self.pairs += J * len(out)
        self.derived += int(np.count_nonzero(cap.get("derived", ())))

        def sums(j, f):
            if f not in out:
                return None
            c, s, h = out[f]
            return c[j], s[j], h[j]
        return sums

    def close(self):
        self.codes = {}
