// ygg_wide.cuh — histogram and scan kernels of the wide numerical columns (DESIGN.md §20).
//
// A wide column is a numerical feature with 257..65535 buckets, one per distinct value (or, discretized, one per bin of
// the GPU binning step, DESIGN.md §25), stored as uint16 codes in its own matrix (ygg_dataset.d_wide).  Its histograms do not fit k_hist's shared-memory tiles: they live in global memory
// as [slot][sum over the wide features of B_f] planes, accumulated with 64-bit / 32-bit integer atomics from the same
// active lists and 24-bit quantised gradients as k_hist's (exact and order independent, DESIGN.md §3), and scanned by
// one CTA per (family, wide feature) in tiles of 256 buckets with a running carry, scored by boundary_score.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "ygg_kernels.cuh"

namespace ygg {

struct WideHistParams {
  const uint16_t* wide;       // [wide features][n_pad] codes
  int64_t n_pad;
  const int64_t* off;         // [wide features] first bucket of the feature in a slot's plane
  const uint2* act;           // the level's active lists (k_quantize / k_compact_root / k_partition): (q24 | slot << 24, row)
  const uint32_t* act_h;      // second plane (hessians or weights), null without one
  const int32_t* act_count;
  int n_blocks;
  int64_t total;              // buckets of one slot's plane (sum over the wide features)
  unsigned long long* sum;    // [slots][total] sums of q24
  uint32_t* cnt;              // [slots][total] row counts
  unsigned long long* hsum;   // [slots][total] second plane (null without one)
};

// Grid: x strides over the 8192-row blocks, y = wide feature.  One thread per active-list entry; the slot is the
// entry's own 8-bit tag, so multi-pass levels of k_hist (slot windows) need nothing here.
__global__ void __launch_bounds__(256) k_hist_wide(WideHistParams p) {
  const int w = blockIdx.y;
  const uint16_t* __restrict__ col = p.wide + static_cast<int64_t>(w) * p.n_pad;
  const int64_t off = p.off[w];
  for (int blk = blockIdx.x; blk < p.n_blocks; blk += gridDim.x) {
    const int64_t base = static_cast<int64_t>(blk) * kBlockRows;
    const int count = p.act_count[blk];
    for (int i = threadIdx.x; i < count; i += blockDim.x) {
      const uint2 e = p.act[base + i];
      const uint32_t slot = e.x >> 24;
      if (slot == kNoSlot) continue;
      const size_t at = static_cast<size_t>(slot) * p.total + off + col[base + e.y];
      atomicAdd(&p.sum[at], static_cast<unsigned long long>(e.x & kQMax));
      atomicAdd(&p.cnt[at], 1u);
      if (p.hsum != nullptr) atomicAdd(&p.hsum[at], static_cast<unsigned long long>(p.act_h[base + i]));
    }
  }
}

struct WideScanParams {
  ScanParams s;                  // the level's scan parameters (families, nodes, scales, gain options, candidates)
  const int32_t* wide_feature;   // [wide features] dataset feature
  const int32_t* wide_bins;      // [wide features] B_f
  const int64_t* off;            // [wide features]
  const float* values;           // bucket values, feature w at off[w]
  int64_t total;
  // this level's slot planes [slot][total]; per-node copies [level nodes][total] of this level and of the parent level
  const unsigned long long* slot_sum;
  const uint32_t* slot_cnt;
  const unsigned long long* slot_hsum;
  unsigned long long* node_sum;
  uint32_t* node_cnt;
  unsigned long long* node_hsum;
  const unsigned long long* pnode_sum;
  const uint32_t* pnode_cnt;
  const unsigned long long* pnode_hsum;
  float* thr_value;              // [level nodes][f_count] float threshold of the wide candidates (SelectParams.wide_thr_value)
  const int32_t* wide_disc;      // [wide features] 1: discretized threshold rule (DESIGN.md §25); null without such columns
  // wide categorical columns (k_scan_wide_cat; null / 0 without them)
  const int32_t* wide_cat;       // [wide features] 1: categorical
  int n_wide, set_words;
  uint32_t* set_out;             // [level nodes][n_wide][set_words] positive sets (SelectParams.wide_set)
  double* sort_key;              // [grid.x][sort_total] per-CTA sort scratch: feature w's block of sort_pad(B_w) entries
  int32_t* sort_idx;             // starts at sort_off[w]
  const int64_t* sort_off;       // [wide features]
  int64_t sort_total;
};

// Bucket b of a node: the direct histogram (slot plane at `d`), or parent (node plane at `x`) - direct.  Sums unbiased.
template <bool HESS>
__device__ __forceinline__ Scan3 wide_bucket(const WideScanParams& p, size_t d, size_t x, bool derived, int b) {
  long long c = p.slot_cnt[d + b];
  unsigned long long s = p.slot_sum[d + b];
  unsigned long long h = HESS && p.s.has_h ? p.slot_hsum[d + b] : 0ull;
  if (derived) {
    c = static_cast<long long>(p.pnode_cnt[x + b]) - c;
    s = p.pnode_sum[x + b] - s;
    if (HESS && p.s.has_h) h = p.pnode_hsum[x + b] - h;
  }
  if (HESS && !p.s.has_h) h = static_cast<unsigned long long>(c) << kQBits;   // h == 1: a row contributes 2^24
  return Scan3{c, static_cast<long long>(s) - c * static_cast<long long>(kQBias), static_cast<long long>(h)};
}

// Scans one node of one wide feature (all 256 threads); thread 0 writes the Candidate and the float threshold.
// `copy_to` (or null): the node's plane at the level, kept when it is a parent at the next level.  `disc`: the column
// takes the discretized threshold rule (bucket interpolation, no float threshold) instead of §14's exact one.
template <bool HESS>
__device__ void scan_wide_node(const WideScanParams& p, int node, int fl, int B, const float* values, size_t d, size_t x,
                               bool derived, size_t copy_to, bool copy, bool disc) {
  __shared__ Scan3 s_warp[8];
  __shared__ double s_best_score[8];
  __shared__ int s_best_b[8];
  __shared__ long long s_npos;
  __shared__ int s_hi;
  const LevelDesc lv = p.s.levels[p.s.level];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  // pass 1: the node's totals (and its copy for the next level)
  Scan3 mine{0, 0, 0};
  for (int b = tid; b < B; b += blockDim.x) {
    const Scan3 v = wide_bucket<HESS>(p, d, x, derived, b);
    mine.c += v.c; mine.s += v.s; mine.h += v.h;
    if (copy) {
      p.node_cnt[copy_to + b] = static_cast<uint32_t>(v.c);
      p.node_sum[copy_to + b] = static_cast<unsigned long long>(v.s + v.c * static_cast<long long>(kQBias));
      if (HESS && p.s.has_h) p.node_hsum[copy_to + b] = static_cast<unsigned long long>(v.h);
    }
  }
  Scan3 tot;
  block_inclusive_scan(mine, s_warp, &tot);
  const double ginv = static_cast<double>(p.s.st->g_pow2) / static_cast<double>(1u << (kQBits - 1));
  const double hinv = static_cast<double>(p.s.st->h_pow2) / static_cast<double>(1u << kQBits);
  // pass 2: every boundary, tile by tile with a running carry; the first maximum of each thread, then of the block
  double bs = -1.0;
  int bb = 0x7fffffff;
  long long bnpos = 0;
  Scan3 carry{0, 0, 0};
  bool tried = false;
  for (int t0 = 0; t0 < B; t0 += blockDim.x) {
    const int b = t0 + tid;
    const Scan3 v = b < B ? wide_bucket<HESS>(p, d, x, derived, b) : Scan3{0, 0, 0};
    Scan3 tile;
    Scan3 inc = block_inclusive_scan(v, s_warp, &tile);
    inc.c += carry.c; inc.s += carry.s; inc.h += carry.h;
    carry.c += tile.c; carry.s += tile.s; carry.h += tile.h;
    double score;
    if (boundary_score(p.s, tot, inc, b <= B - 2, ginv, hinv, &score) && score > bs) { bs = score; bb = b; bnpos = tot.c - inc.c; }
    if (p.s.tried != nullptr) tried = tried || boundary_tried(p.s, tot, inc, b <= B - 2);
  }
  if (p.s.tried != nullptr) {
    const int any = __syncthreads_or(tried);
    if (tid == 0) p.s.tried[static_cast<size_t>(node - lv.first_node) * p.s.f_count + fl] = any ? 1 : 0;
  }
  const int my_b = bb;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double os = __shfl_xor_sync(0xffffffffu, bs, o);
    const int ob = __shfl_xor_sync(0xffffffffu, bb, o);
    if (os > bs || (os == bs && ob < bb)) { bs = os; bb = ob; }
  }
  if (lane == 0) { s_best_score[w] = bs; s_best_b[w] = bb; }
  __syncthreads();
  bs = s_best_score[0]; bb = s_best_b[0];
  for (int i = 1; i < 8; i++)
    if (s_best_score[i] > bs || (s_best_score[i] == bs && s_best_b[i] < bb)) { bs = s_best_score[i]; bb = s_best_b[i]; }
  const bool found = bb != 0x7fffffff;
  if (found && my_b == bb) s_npos = bnpos;
  if (tid == 0) s_hi = 0x7fffffff;
  __syncthreads();
  // pass 3: hi = the first non-empty bucket after the best boundary (it exists: the positive side has rows)
  if (found) {
    for (int t0 = (bb + 1) & ~(static_cast<int>(blockDim.x) - 1); t0 < B; t0 += blockDim.x) {
      const int b = t0 + tid;
      if (b > bb && b < B && wide_bucket<HESS>(p, d, x, derived, b).c > 0) atomicMin(&s_hi, b);
      __syncthreads();
      const int hi = s_hi;
      __syncthreads();   // every thread has read s_hi before the next tile may lower it
      if (hi != 0x7fffffff) break;
    }
  }
  if (tid == 0) {
    const size_t ci = static_cast<size_t>(node - lv.first_node) * p.s.f_count + fl;
    Candidate c{0.f, 0, 0, 0};
    float threshold = __builtin_nanf("");
    if (found && disc) {
      // scan_node's bucket interpolation (splitter_scanner.h:993-1000, :1076-1086): hi is the first non-empty bucket
      // after the best boundary; the scan visits it only below B - 1
      int idx = bb;
      if (s_hi <= B - 2 && s_hi != bb + 1) idx = (bb + s_hi) / 2;
      c.found = 1;
      c.score = static_cast<float>(bs);
      c.thr = idx + 1;
      c.n_pos = static_cast<int32_t>(s_npos);
    } else if (found) {
      const int hi = s_hi != 0x7fffffff ? s_hi : bb + 1;
      // §14's exact rule: the middle of the two values present in the node around the cut; the bin threshold is the
      // first bucket whose value reaches it (every bucket in between is empty in this node)
      threshold = mid_threshold(values[bb], values[hi]);
      int lo = bb + 1, up = hi;   // lower_bound in [bb + 1, hi)
      while (lo < up) {
        const int mid = (lo + up) >> 1;
        if (values[mid] < threshold) lo = mid + 1; else up = mid;
      }
      c.found = 1;
      c.score = static_cast<float>(bs);
      c.thr = lo;
      c.n_pos = static_cast<int32_t>(s_npos);
    }
    p.s.cand[ci] = c;
    p.thr_value[ci] = threshold;
  }
  __syncthreads();
}

// One CTA of 256 threads per (family, wide feature); runs after k_scan, whose candidates of the wide features (their
// one-bucket filler columns: never found) it overwrites.  The direct node is read from its slot plane, the derived one
// is parent - direct on the exact integers, and both are kept as the next level's parent planes (ping-pong buffers,
// the counterpart of k_scan's d_hist_* copies).
template <bool HESS>
__global__ void __launch_bounds__(256) k_scan_wide(WideScanParams p) {
  const LevelDesc lv = p.s.levels[p.s.level];
  if (static_cast<int>(blockIdx.x) >= lv.num_families) return;
  const Family fam = p.s.families[blockIdx.x];
  const int w = blockIdx.y;
  if (p.wide_cat != nullptr && p.wide_cat[w]) return;   // k_scan_wide_cat's
  const int f = p.wide_feature[w];
  const int fl = f - p.s.f_begin;
  const int B = p.wide_bins[w];
  const int64_t off = p.off[w];
  const float* values = p.values + off;
  const bool disc = p.wide_disc != nullptr && p.wide_disc[w];
  const NodeRec direct = p.s.nodes[fam.direct];
  const size_t d = static_cast<size_t>(direct.slot) * p.total + off;
  const size_t dn = static_cast<size_t>(fam.direct - lv.first_node) * p.total + off;
  // a node's plane is needed at the next level only if it can be split there
  if (direct.candidate) scan_wide_node<HESS>(p, fam.direct, fl, B, values, d, 0, false, dn, p.s.write_derived != 0, disc);
  if (fam.derived >= 0) {
    const NodeRec derived = p.s.nodes[fam.derived];
    if (derived.candidate) {
      const LevelDesc plv = p.s.levels[p.s.level - 1];
      const size_t x = static_cast<size_t>(fam.parent - plv.first_node) * p.total + off;
      const size_t xn = static_cast<size_t>(fam.derived - lv.first_node) * p.total + off;
      scan_wide_node<HESS>(p, fam.derived, fl, B, values, d, x, true, xn, p.s.write_derived != 0, disc);
    }
  }
}

// Wide categorical columns (DESIGN.md §21): scan_node_categorical for B = 257..65535 buckets.  The keys (category_key),
// sorted ascending by (key, category index) with a bitonic sort over the CTA's global scratch (`key` / `idx`,
// sort_pad(B) entries, +inf past B), then the sorted buckets scanned in tiles of 256 with a running carry and scored by
// boundary_score with l2_categorical; the first maximum wins.  The categories after the best boundary form the positive
// set, written to p.set_out.
// Entries of the sort scratch of a categorical column of B categories: the power of two >= B.
__host__ __device__ inline int sort_pad(int B) {
  int P = 1;
  while (P < B) P <<= 1;
  return P;
}

template <bool HESS>
__device__ void scan_wide_cat_node(const WideScanParams& p, int node, int fl, int w, int B, size_t d, size_t x, bool derived,
                                   size_t copy_to, bool copy, double* key, int32_t* idx) {
  __shared__ Scan3 s_warp[8];
  __shared__ double s_best_score[8];
  __shared__ int s_best_b[8];
  __shared__ long long s_npos;
  const LevelDesc lv = p.s.levels[p.s.level];
  const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
  const int P = sort_pad(B);
  const double ginv = static_cast<double>(p.s.st->g_pow2) / static_cast<double>(1u << (kQBits - 1));
  const double hinv = static_cast<double>(p.s.st->h_pow2) / static_cast<double>(1u << kQBits);
  // pass 1: the node's totals (and its copy for the next level), the keys
  Scan3 mine{0, 0, 0};
  for (int b = tid; b < P; b += blockDim.x) {
    double k = __longlong_as_double(0x7FF0000000000000ll);   // +inf: past the feature's categories
    if (b < B) {
      const Scan3 v = wide_bucket<HESS>(p, d, x, derived, b);
      mine.c += v.c; mine.s += v.s; mine.h += v.h;
      if (copy) {
        p.node_cnt[copy_to + b] = static_cast<uint32_t>(v.c);
        p.node_sum[copy_to + b] = static_cast<unsigned long long>(v.s + v.c * static_cast<long long>(kQBias));
        if (HESS && p.s.has_h) p.node_hsum[copy_to + b] = static_cast<unsigned long long>(v.h);
      }
      k = category_key(p.s, v.c, v.s, v.h, ginv, hinv);
    }
    key[b] = k;
    idx[b] = b;
  }
  Scan3 tot;
  block_inclusive_scan(mine, s_warp, &tot);
  __syncthreads();
  // bitonic sort of (key, index) pairs, ascending; -0.0 == +0.0, equal keys in index order
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += blockDim.x) {
        const int partner = i ^ j;
        if (partner > i) {
          const double ka = key[i], kb = key[partner];
          const int ia = idx[i], ib = idx[partner];
          const bool a_gt_b = ka > kb || (ka == kb && ia > ib);
          if (a_gt_b == ((i & k) == 0)) { key[i] = kb; key[partner] = ka; idx[i] = ib; idx[partner] = ia; }
        }
      }
      __syncthreads();
    }
  }
  // pass 2: every boundary between sorted positions, tile by tile with a running carry
  ScanParams sp = p.s;
  sp.l2 = p.s.l2_categorical;
  double bs = -1.0;
  int bb = 0x7fffffff;
  long long bnpos = 0;
  Scan3 carry{0, 0, 0};
  bool tried = false;
  for (int t0 = 0; t0 < B; t0 += blockDim.x) {
    const int pos = t0 + tid;
    const Scan3 v = pos < B ? wide_bucket<HESS>(p, d, x, derived, idx[pos]) : Scan3{0, 0, 0};
    Scan3 tile;
    Scan3 inc = block_inclusive_scan(v, s_warp, &tile);
    inc.c += carry.c; inc.s += carry.s; inc.h += carry.h;
    carry.c += tile.c; carry.s += tile.s; carry.h += tile.h;
    double score;
    if (boundary_score(sp, tot, inc, pos <= B - 2, ginv, hinv, &score) && score > bs) { bs = score; bb = pos; bnpos = tot.c - inc.c; }
    if (p.s.tried != nullptr) tried = tried || boundary_tried(sp, tot, inc, pos <= B - 2);
  }
  if (p.s.tried != nullptr) {
    const int any = __syncthreads_or(tried);
    if (tid == 0) p.s.tried[static_cast<size_t>(node - lv.first_node) * p.s.f_count + fl] = any ? 1 : 0;
  }
  const int my_b = bb;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double os = __shfl_xor_sync(0xffffffffu, bs, o);
    const int ob = __shfl_xor_sync(0xffffffffu, bb, o);
    if (os > bs || (os == bs && ob < bb)) { bs = os; bb = ob; }
  }
  if (lane == 0) { s_best_score[wp] = bs; s_best_b[wp] = bb; }
  __syncthreads();
  bs = s_best_score[0]; bb = s_best_b[0];
  for (int i = 1; i < 8; i++)
    if (s_best_score[i] > bs || (s_best_score[i] == bs && s_best_b[i] < bb)) { bs = s_best_score[i]; bb = s_best_b[i]; }
  const bool found = bb != 0x7fffffff;
  if (found && my_b == bb) s_npos = bnpos;
  // pass 3: the positive set = the categories at sorted positions after the best boundary
  const size_t j = static_cast<size_t>(node - lv.first_node);
  uint32_t* set = p.set_out + (j * p.n_wide + w) * p.set_words;
  for (int i = tid; i < p.set_words; i += blockDim.x) set[i] = 0u;
  __syncthreads();
  if (found)
    for (int pos = bb + 1 + tid; pos < B; pos += blockDim.x) {
      const int c = idx[pos];
      atomicOr(&set[c >> 5], 1u << (c & 31));
    }
  if (tid == 0) {
    const size_t ci = j * p.s.f_count + fl;
    Candidate c{0.f, 0, 0, 0};
    if (found) {
      c.found = 1;
      c.score = static_cast<float>(bs);
      c.n_pos = static_cast<int32_t>(s_npos);
    }
    p.s.cand[ci] = c;
    p.thr_value[ci] = __builtin_nanf("");
  }
  __syncthreads();   // the scratch is reused by the CTA's next node
}

// One CTA of 256 threads per (family, wide categorical feature), launched next to k_scan_wide (which skips these
// features); same planes, same ping-pong copies.
template <bool HESS>
__global__ void __launch_bounds__(256) k_scan_wide_cat(WideScanParams p) {
  const LevelDesc lv = p.s.levels[p.s.level];
  if (static_cast<int>(blockIdx.x) >= lv.num_families) return;
  const int w = blockIdx.y;
  if (!p.wide_cat[w]) return;
  const Family fam = p.s.families[blockIdx.x];
  const int fl = p.wide_feature[w] - p.s.f_begin;
  const int B = p.wide_bins[w];
  const int64_t off = p.off[w];
  double* key = p.sort_key + static_cast<size_t>(blockIdx.x) * p.sort_total + p.sort_off[w];
  int32_t* idx = p.sort_idx + static_cast<size_t>(blockIdx.x) * p.sort_total + p.sort_off[w];
  const NodeRec direct = p.s.nodes[fam.direct];
  const size_t d = static_cast<size_t>(direct.slot) * p.total + off;
  const size_t dn = static_cast<size_t>(fam.direct - lv.first_node) * p.total + off;
  if (direct.candidate) scan_wide_cat_node<HESS>(p, fam.direct, fl, w, B, d, 0, false, dn, p.s.write_derived != 0, key, idx);
  if (fam.derived >= 0) {
    const NodeRec derived = p.s.nodes[fam.derived];
    if (derived.candidate) {
      const LevelDesc plv = p.s.levels[p.s.level - 1];
      const size_t x = static_cast<size_t>(fam.parent - plv.first_node) * p.total + off;
      const size_t xn = static_cast<size_t>(fam.derived - lv.first_node) * p.total + off;
      scan_wide_cat_node<HESS>(p, fam.derived, fl, w, B, d, x, true, xn, p.s.write_derived != 0, key, idx);
    }
  }
}

// After k_select_global: a node of the level split on a wide categorical feature gets its positive set copied from the
// level's side array into the tree's pool [max_nodes][set_words] (one CTA per level node).
__global__ void __launch_bounds__(256) k_store_sets(const NodeRec* __restrict__ nodes, const LevelDesc* __restrict__ levels,
                                                    int level, const int32_t* __restrict__ wide_of,
                                                    const uint32_t* __restrict__ wide_set, int n_wide, int set_words,
                                                    uint32_t* __restrict__ pool) {
  const LevelDesc lv = levels[level];
  const int j = blockIdx.x;
  if (j >= lv.num_nodes) return;
  const NodeRec& nd = nodes[lv.first_node + j];
  if (nd.feature < 0 || nd.cond_type != 1) return;
  const int wi = wide_of[nd.feature];
  if (wi < 0) return;
  const uint32_t* src = wide_set + (static_cast<size_t>(j) * n_wide + wi) * set_words;
  uint32_t* dst = pool + static_cast<size_t>(lv.first_node + j) * set_words;
  for (int i = threadIdx.x; i < set_words; i += blockDim.x) dst[i] = src[i];
}

// Whether row code `b` of split node `nd` goes to the positive child: the pooled set of a wide categorical split
// (`set`: the node's pool entry; wide = the split feature is a wide column), else the byte mask or the threshold.
__device__ __forceinline__ bool split_goes_pos(const NodeRec& nd, uint32_t b, bool wide, const uint32_t* set) {
  if (nd.cond_type != 1) return static_cast<int>(b) >= nd.thr;
  const uint32_t word = wide ? set[b >> 5] : nd.mask[b >> 5];
  return ((word >> (b & 31)) & 1u) != 0;
}

}  // namespace ygg
