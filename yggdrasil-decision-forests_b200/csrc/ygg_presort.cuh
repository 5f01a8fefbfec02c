// ygg_presort.cuh — the presorted numerical columns' level lists, scan and partition (DESIGN.md §22).
//
// A presorted column is a numerical feature stored as float values (ygg_dataset.d_num).  Each training handle sorts every
// such column once into a master list of (value, row) pairs, ties in row order.  Each level keeps, per column, a list of
// the rows of the level's candidate nodes: one segment per candidate node, in level node order, each segment in (value,
// row) order.  A segment starts at seg_off[node] (an exclusive scan of the candidate nodes' n) inside the column's
// stride of n entries.  The scan takes u64 prefix sums of the same quantised gradients the histograms use (exact and
// order independent, DESIGN.md §3) and scores every boundary between two different values with boundary_score; the
// partition stable-partitions every segment into its children's segments.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "ygg_kernels.cuh"

namespace ygg {

struct PresortParams {
  ScanParams s;                     // the level's scan parameters (nodes, scales, gain options, candidates)
  int level;
  int P;                            // presorted columns
  int64_t n;                        // stride of a column's list (the dataset's rows)
  const int32_t* num_feature;       // [P] dataset feature
  const float* val;                 // this level's lists [P][n]
  const uint32_t* row;
  const uint16_t* node_of_row;
  const int64_t* seg_off;           // [max_nodes] segment start of a candidate node in its level's lists
  const int64_t* seg_total;         // [levels] entries of a level's lists (per column)
  const uint32_t* q24;              // [n_pad] per-row quantised gradients (k_quantize)
  const uint32_t* hq24;             // second plane, null without one
  unsigned long long* ps;           // [P][n] inclusive prefix sums of q24 over the lists
  unsigned long long* ph;           // [P][n] of hq24 (used with hq24 only)
  unsigned long long* best;         // [level nodes][P] double bits of the best score (0: none)
  unsigned long long* best_idx;     // [level nodes][P] list index of the best boundary's lower entry
  float* thr_value;                 // [level nodes][f_count] (SelectParams.wide_thr_value)
};

// Segment starts of level `level`'s candidate nodes and the level's list length; one CTA of 1024 threads.
__global__ void __launch_bounds__(1024) k_presort_segments(const LevelDesc* __restrict__ levels, const NodeRec* __restrict__ nodes,
                                                           int level, int64_t* __restrict__ seg_off, int64_t* __restrict__ seg_total) {
  __shared__ int s_warp[32];
  __shared__ long long s_run;
  const LevelDesc lv = levels[level];
  if (threadIdx.x == 0) s_run = 0;
  __syncthreads();
  for (int j0 = 0; j0 < lv.num_nodes; j0 += blockDim.x) {
    const int j = j0 + threadIdx.x;
    const NodeRec* nd = j < lv.num_nodes ? &nodes[lv.first_node + j] : nullptr;
    const int len = (nd != nullptr && nd->candidate) ? static_cast<int>(nd->n) : 0;
    int tot;
    const int excl = block_exclusive_scan(len, s_warp, &tot);
    const long long run = s_run;
    if (nd != nullptr) seg_off[lv.first_node + j] = run + excl;
    __syncthreads();
    if (threadIdx.x == 0) s_run = run + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) seg_total[level] = s_run;
}

// The sampled root: flags = the master entries whose row is in the iteration's sample.
__global__ void __launch_bounds__(256) k_presort_sample_flags(const uint32_t* __restrict__ master_row, int64_t total,
                                                              const uint8_t* __restrict__ selected, uint32_t* __restrict__ flags) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride)
    flags[i] = selected[master_row[i]] ? 1u : 0u;
}
// Stable compaction of every column's master list by the flags' exclusive scan `excl`.
__global__ void __launch_bounds__(256) k_presort_sample_scatter(const float* __restrict__ master_val, const uint32_t* __restrict__ master_row,
                                                                int64_t n, int64_t total, const uint8_t* __restrict__ selected,
                                                                const uint32_t* __restrict__ excl, float* __restrict__ out_val,
                                                                uint32_t* __restrict__ out_row) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const uint32_t r = master_row[i];
    if (!selected[r]) continue;
    const int64_t col = (i / n) * n;
    const int64_t dst = col + static_cast<uint32_t>(excl[i] - excl[col]);   // (u32 differences are exact)
    out_val[dst] = master_val[i];
    out_row[dst] = r;
  }
}

// The quantised gradients of every list entry, in list order (zero past the level's entries), for the prefix sums.
__global__ void __launch_bounds__(256) k_presort_gather(PresortParams p) {
  const int64_t m = p.seg_total[p.level];
  const int64_t total = static_cast<int64_t>(p.P) * p.n;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const bool in = i % p.n < m;
    const uint32_t r = in ? p.row[i] : 0u;
    p.ps[i] = in ? p.q24[r] : 0ull;
    if (p.hq24 != nullptr) p.ph[i] = in ? p.hq24[r] : 0ull;
  }
}

// Sums (count, unbiased q, second plane) of list entries [lo, i] from the inclusive prefix sums.
template <bool HESS>
__device__ __forceinline__ Scan3 presort_range(const PresortParams& p, int64_t lo, int64_t i) {
  const long long c = i - lo + 1;
  const unsigned long long s = p.ps[i] - (lo > 0 ? p.ps[lo - 1] : 0ull);
  unsigned long long h = 0ull;
  if (HESS) h = p.hq24 != nullptr ? p.ph[i] - (lo > 0 ? p.ph[lo - 1] : 0ull) : static_cast<unsigned long long>(c) << kQBits;
  return Scan3{c, static_cast<long long>(s) - c * static_cast<long long>(kQBias), static_cast<long long>(h)};
}

// Score of the boundary after list entry i (false: no valid boundary there).  *slot = the (level node, column) pair;
// *tried = boundary_tried there (false: no boundary between two different values).
template <bool HESS>
__device__ __forceinline__ bool presort_boundary(const PresortParams& p, int64_t i, int64_t m, double* score, int64_t* slot,
                                                 bool* tried) {
  const int64_t col = (i / p.n) * p.n;
  if (i - col >= m) return false;
  const int node = p.node_of_row[p.row[i]];
  const int64_t lo = col + p.seg_off[node];
  const int64_t hi = lo + p.s.nodes[node].n - 1;
  if (i >= hi || !(p.val[i] < p.val[i + 1])) return false;
  const Scan3 tot = presort_range<HESS>(p, lo, hi), inc = presort_range<HESS>(p, lo, i);
  const double ginv = static_cast<double>(p.s.st->g_pow2) / static_cast<double>(1u << (kQBits - 1));
  const double hinv = static_cast<double>(p.s.st->h_pow2) / static_cast<double>(1u << kQBits);
  *slot = static_cast<int64_t>(node - p.s.levels[p.level].first_node) * p.P + i / p.n;
  *tried = boundary_tried(p.s, tot, inc, true);
  return boundary_score(p.s, tot, inc, true, ginv, hinv, score);
}

// Two passes over every boundary: MAX_PASS keeps each (node, column)'s best score (positive doubles order like their
// bits), the other pass the lowest list index that reaches it — the first maximum in ascending value order, as
// k_scan_wide keeps over buckets.  A warp whose valid boundaries all belong to one (node, column) combines them first.
template <bool HESS, bool MAX_PASS>
__global__ void __launch_bounds__(256) k_presort_scan(PresortParams p) {
  const int64_t m = p.seg_total[p.level];
  const int64_t total = static_cast<int64_t>(p.P) * p.n;
  const int lane = threadIdx.x & 31;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t w0 = static_cast<int64_t>(blockIdx.x) * blockDim.x + (threadIdx.x & ~31); w0 < total; w0 += stride) {
    const int64_t i = w0 + lane;
    double score = 0.0;
    int64_t slot = -1;
    bool tried = false;
    const bool valid = i < total && presort_boundary<HESS>(p, i, m, &score, &slot, &tried);
    // (k_scan left 0 for the pair: its filler column has one bucket)
    if (MAX_PASS && tried && p.s.tried != nullptr)
      p.s.tried[static_cast<size_t>(slot / p.P) * p.s.f_count + (p.num_feature[slot % p.P] - p.s.f_begin)] = 1;
    if (!valid) slot = -1;
    unsigned long long key = 0ull;   // MAX_PASS: the score's bits; else the candidate index (or ~0)
    if (MAX_PASS) key = valid ? static_cast<unsigned long long>(__double_as_longlong(score)) : 0ull;
    else key = (valid && static_cast<unsigned long long>(__double_as_longlong(score)) == p.best[slot]) ? static_cast<unsigned long long>(i) : ~0ull;
    const unsigned mask = __ballot_sync(0xffffffffu, valid);
    if (mask == 0u) continue;
    const int64_t slot0 = __shfl_sync(0xffffffffu, slot, __ffs(mask) - 1);
    if (__all_sync(0xffffffffu, !valid || slot == slot0)) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
        key = MAX_PASS ? max(key, other) : min(key, other);
      }
      if (lane == 0) {
        if (MAX_PASS) atomicMax(&p.best[slot0], key);
        else if (key != ~0ull) atomicMin(&p.best_idx[slot0], key);
      }
    } else if (valid) {
      if (MAX_PASS) atomicMax(&p.best[slot], key);
      else if (key != ~0ull) atomicMin(&p.best_idx[slot], key);
    }
  }
}

// One thread per (level node, column): the candidate of a candidate node, written where k_scan keeps it (its candidate
// of the filler column: never found), and the float threshold to the side array.  thr = 1: the engine's "bin" of a row
// for a numerical split is value >= thr_value (0 or 1), so every bin-threshold consumer routes it unchanged.
__global__ void __launch_bounds__(256) k_presort_candidates(PresortParams p) {
  const LevelDesc lv = p.s.levels[p.level];
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= lv.num_nodes * p.P) return;
  const int j = t / p.P, c = t % p.P;
  const NodeRec& nd = p.s.nodes[lv.first_node + j];
  if (!nd.candidate) return;
  const size_t ci = static_cast<size_t>(j) * p.s.f_count + (p.num_feature[c] - p.s.f_begin);
  const unsigned long long bits = p.best[t];
  Candidate cand{0.f, 0, 0, 0};
  float threshold = __builtin_nanf("");
  if (bits != 0ull) {
    const int64_t i = static_cast<int64_t>(p.best_idx[t]);
    const int64_t lo = static_cast<int64_t>(c) * p.n + p.seg_off[lv.first_node + j];
    threshold = mid_threshold(p.val[i], p.val[i + 1]);
    cand.found = 1;
    cand.score = static_cast<float>(__longlong_as_double(static_cast<long long>(bits)));
    cand.thr = 1;
    cand.n_pos = static_cast<int32_t>(nd.n - (i - lo + 1));
  }
  p.s.cand[ci] = cand;
  p.thr_value[ci] = threshold;
}

// After k_partition (node_of_row holds the children): flag 1 for the entries that go to a positive child.  The children
// of a split are created as (pos, neg) pairs from the next level's first node, so a positive child sits at an even offset.
__global__ void __launch_bounds__(256) k_presort_flags(PresortParams p, uint32_t* __restrict__ flags) {
  const int64_t m = p.seg_total[p.level];
  const int first_next = p.s.levels[p.level + 1].first_node;
  const int64_t total = static_cast<int64_t>(p.P) * p.n;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    uint32_t f = 0u;
    if (i % p.n < m) {
      const int child = p.node_of_row[p.row[i]];
      f = (child >= first_next && ((child - first_next) & 1) == 0) ? 1u : 0u;
    }
    flags[i] = f;
  }
}

// Stable partition of every segment into its children's segments of the next level's lists (`excl`: exclusive scan of
// the flags).  An entry's rank among its parent segment's entries that go to the same side is its offset in the child's
// segment; rows of nodes that did not split, or whose child is not a candidate, are dropped.
__global__ void __launch_bounds__(256) k_presort_scatter(PresortParams p, const uint32_t* __restrict__ excl, float* __restrict__ out_val,
                                                         uint32_t* __restrict__ out_row) {
  const int64_t m = p.seg_total[p.level];
  const int first_next = p.s.levels[p.level + 1].first_node;
  const int64_t total = static_cast<int64_t>(p.P) * p.n;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t col = (i / p.n) * p.n;
    if (i - col >= m) continue;
    const uint32_t r = p.row[i];
    const int child = p.node_of_row[r];
    if (child < first_next || !p.s.nodes[child].candidate) continue;
    const int64_t lo = col + p.seg_off[p.s.nodes[child].parent];
    const int64_t pos_rank = static_cast<uint32_t>(excl[i] - excl[lo]);
    const int64_t rank = ((child - first_next) & 1) == 0 ? pos_rank : (i - lo) - pos_rank;
    // (the children's n come from the scan's counts and the rows were routed by value >= threshold: equal unless the
    // threshold overflowed to +inf between two values near the float range's end; never write past a segment)
    if (rank >= p.s.nodes[child].n) continue;
    const int64_t dst = col + p.seg_off[child] + rank;
    out_val[dst] = p.val[i];
    out_row[dst] = r;
  }
}

}  // namespace ygg
