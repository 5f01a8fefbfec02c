// ygg_device.cuh — device-side data contracts of the GBT split-finding engine.
//
// Fixed-point design (DESIGN.md §3): every floating-point accumulation on the hot path is done in
// integers so that results are exact, order-independent and identical for any CTA count, stream
// order or GPU count:
//   * histogram sums   : per row a 24-bit biased quantised gradient q24 = rint(g * 2^23 / P) + 2^23
//                        (P = power of two >= max|g|), accumulated with native 32-bit shared-memory
//                        atomics (ATOMS.ADD) + carry word, flushed to 64-bit global sums;
//   * node statistics  : 31-bit biased quantisation, 64-bit sums (resolution 2^-30 * P).
// The reference accumulates the same quantities in double (variance gain) or float (hessian
// gain): learner/decision_tree/splitter_accumulator.h:1473-1566, :1662-1824.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace ygg {

constexpr int kMaxBins = 256;
constexpr int kQBits = 24;                       // histogram quantisation bits (biased)
constexpr uint32_t kQBias = 1u << (kQBits - 1);  // 2^23
constexpr uint32_t kQMax = (1u << kQBits) - 1;
constexpr int kSBits = 31;                       // node-statistics quantisation bits
constexpr uint32_t kSBias = 1u << (kSBits - 1);  // 2^30
constexpr uint32_t kNoSlot = 0xFFu;              // rowinfo slot byte of a row that is not histogrammed
constexpr int kMaxSlotsPerPass = 64;             // shared-memory bound: 64 slots * 256 bins * 8 B = 128 KB
constexpr double kMinHessianForNewtonStep = 0.001;  // loss_utils.cc:101, splitter_accumulator.h:753

// A candidate split whose float score EQUALS the chosen one's (another feature): the reference decides between them
// by its per-node candidate shuffle (training.cc:4293-4306), which the host replays on the finished tree.
constexpr int kMaxTieAlts = 3;
struct TieAlt {
  int32_t feature, thr, n_pos, cond_type, na_value;
  float thr_value;   // see NodeRec
  uint32_t mask[8];
};
// Per node of a level, written by k_select_local: the ties of the level's best split.
struct TieRec {
  int32_t count;              // candidates with the best score besides the chosen one (may exceed kMaxTieAlts)
  TieAlt alt[kMaxTieAlts];    // the first of them in feature order
};

// One node of the tree being grown (device table; one table per tree).
struct NodeRec {
  int32_t parent;       // node id of the parent, -1 for the root
  int32_t depth;        // root = 1
  int32_t feature;      // -1 while a leaf
  int32_t thr;          // DiscretizedHigher threshold (bin >= thr -> positive)
  int32_t na_value;
  int32_t pos_child, neg_child;
  int32_t slot;         // histogram slot at its level, -1 if derived by subtraction / not needed
  int32_t candidate;    // 1 if the node may still be split (n >= min_examples && depth < max_depth)
  int32_t sibling;      // the other child of the parent, -1 for the root
  float score;
  float leaf_value;
  int32_t cond_type;    // 0: bin >= thr ; 1: category in mask (Contains condition)
  uint32_t mask[8];     // positive categories of a categorical split
  int64_t n;            // number of rows
  int64_t n_pos;        // rows going to the positive child
  unsigned long long sg, sh, sg2;  // biased fixed-point sums of g, h, (float)(g*g) over the rows
  double stat[3];       // what the reference stores in the node proto (loss_utils.cc:109-117)
  int32_t tie_count;    // split nodes: other features with the same float score (see TieAlt)
  float thr_value;      // exact numerical splitter's float threshold (features with bucket values), NaN otherwise
  TieAlt tie[kMaxTieAlts];
};

struct LevelDesc {
  int32_t first_node;   // id of the first node of this level
  int32_t num_nodes;
  int32_t num_slots;    // nodes of this level whose histogram is accumulated from rows
  int32_t num_families; // scan work items: the root, or the child pair of one split parent
};

// Scan work item: children of one split (or the root alone).
struct Family {
  int32_t parent;  // node id of the parent whose histogram is subtracted from; -1: no subtraction
  int32_t direct;  // node whose histogram was accumulated from rows (slot holder)
  int32_t derived; // node = parent - direct; -1 if none
};

// Best split of one (node, feature) pair — the result of ScanSplits
// (learner/decision_tree/splitter_scanner.h:931-1101).
struct Candidate {
  float score;      // split_score as float (NodeCondition.split_score); valid iff found
  int32_t thr;      // threshold (after bucket interpolation)
  int32_t n_pos;    // positive rows at the best boundary (fits int32: N < 2^31)
  int32_t found;    // 1 = kBetterSplitFound
};

// Exact threshold rule (features with bucket values, ygg_dataset_set_bucket_values): k_scan packs, next to the threshold
// bin k, the best boundary's bucket `lo` and the next NON-EMPTY bucket `hi` into Candidate.thr / ShardBest.thr, so that
// whoever consumes the winning candidate (k_select_*) can form the reference's float threshold
// MidThreshold(value[lo], value[hi]) (splitter_accumulator.h:213-232, utils.h:103-109) without another exchange.
constexpr int32_t kThrExactFlag = 1 << 26;
__host__ __device__ inline int32_t pack_exact_thr(int k, int lo, int hi) { return k | (lo << 9) | (hi << 17) | kThrExactFlag; }
__host__ __device__ inline int32_t thr_bin_of(int32_t thr) { return (thr & kThrExactFlag) ? (thr & 0x1FF) : thr; }
__host__ __device__ inline float mid_threshold(float a, float b) {   // learner/decision_tree/utils.h:103-109
  float t = a + (b - a) / 2.f;
  if (t <= a) t = b;
  return t;
}
// The float threshold of a packed candidate (NaN for a plain discretized one); `values` = the feature's bucket values.
__host__ __device__ inline float thr_value_of(int32_t thr, const float* values) {
  if (!(thr & kThrExactFlag)) return __builtin_nanf("");
  return mid_threshold(values[(thr >> 9) & 0xFF], values[(thr >> 17) & 0x1FF]);
}

// Best split of one node over a feature shard, exchanged between GPUs once per level.
struct ShardBest {
  float score;
  int32_t feature;  // global feature index, -1 if none
  int32_t thr;
  int32_t n_pos;
  int32_t cond_type;
  int32_t na_value;  // only meaningful for categorical splits (numerical: derived from thr)
  uint32_t mask[8];
};

// Ordered arg-max over feature shards (FindBestConditionConcurrentManager, training.cc:1728-1746):
// shards are contiguous, ascending feature ranges, so taking the FIRST strictly greater float score
// in rank order equals the reference's fold over all features in candidate order.  Shared by
// k_select_global (device) and ygg_merge_shard_best (host; exercised by the gloo tests).
#ifdef __CUDACC__
__host__ __device__
#endif
inline ShardBest merge_shard_bests(const ShardBest* records, int world, int stride, int node) {
  ShardBest best{};
  best.feature = -1;
  float best_score = 0.f;  // NodeCondition.split_score default
  for (int r = 0; r < world; r++) {
    const ShardBest sb = records[static_cast<long long>(r) * stride + node];
    if (sb.feature >= 0 && sb.score > best_score) {
      best_score = sb.score;
      best = sb;
    }
  }
  return best;
}

// Candidate feature sampling (DESIGN.md §23): the key that orders feature f among the candidates of node `node` (its place
// in the tree's node table) of tree `tree` (iteration * K + class).  Chained SplitMix64 finalizers; the candidate order of a
// node is ascending (key, f).  Restated in include/ygg_b200.h (ygg_candidate_key).
#ifdef __CUDACC__
__host__ __device__
#endif
inline uint64_t splitmix64_mix(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
#ifdef __CUDACC__
__host__ __device__
#endif
inline uint64_t candidate_key(uint32_t seed, int32_t tree, int32_t node, int32_t f) {
  uint64_t z = splitmix64_mix(seed);
  z = splitmix64_mix(z ^ static_cast<uint32_t>(tree));
  z = splitmix64_mix(z ^ static_cast<uint32_t>(node));
  return splitmix64_mix(z ^ static_cast<uint32_t>(f));
}

// Scalars living in device memory so the level loop never syncs with the host.
struct DeviceState {
  float g_pow2;        // P: power of two > max|g| (histogram + statistics scale of g)
  float h_pow2;        // power of two >= max h
  unsigned int gmax_bits;  // float bits of max|g| of the current iteration (atomicMax)
  int32_t num_nodes;   // nodes allocated in the current tree
  unsigned long long loss_sum_fix;  // scratch
  double loss_sum;     // sum of per-row loss terms of the pending tree
  unsigned long long correct;       // correctly classified rows (binomial secondary metric)
  unsigned long long root_sg, root_sh, root_sg2;
  int32_t error_flag;  // non-zero: an invariant was violated on device
  unsigned int g2w_max_bits;  // example weights: float bits of max (w*g)*g of the current iteration
};

}  // namespace ygg
