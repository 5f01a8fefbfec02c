// ygg_oracle.cc — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// CPU restatement ("port") of the reference's GBT histogram split-finding path, used only as the
// checker in tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
// Nothing under yggdrasil-decision-forests_b200/ may include, link or call this file.
//
// Parity status: the reference itself cannot be built in this image (bazel + abseil + protobuf +
// highway absent, SURVEY.md §8c), so this restatement is pinned by the reference's own
// known-answer tests, restated in tests/test_oracle_kat.py:
//   learner/decision_tree/decision_tree_test.cc:2593-2626, :3052-3084
//   learner/decision_tree/training_test.cc:193-267, :826-860
//   learner/gradient_boosted_trees/loss/loss_imp_binomial_test.cc:92-170
//   learner/gradient_boosted_trees/loss/loss_imp_mean_square_error_test.cc:74-175
//   learner/gradient_boosted_trees/loss/loss_imp_multinomial_test.cc:92-197 (multinomial gradients / loss)
//   learner/decision_tree/decision_tree_test.cc:1208-1297 (categorical CART split)
// by node-by-node replays of three complete training runs of the reference (its golden PYDF models of Adult: binomial,
// 163 trees; Iris: multinomial, 54 trees; Abalone: squared error, 45 trees): hold-out rows, initial predictions, every
// categorical split, every numerical split that falls on a bucket boundary, all 6296 leaf values and the whole training
// logs are reproduced (partitions and counts exactly, scores 1e-6, losses 2e-6; tests/test_reference_replay.py); with
// one bucket per distinct value and the candidate shuffle below, all 262 trees of those runs come out identical,
// by four goldens of the reference's C++ tests replayed the same way (gbt_adult_subsampling: stochastic gradient boosting
// in the random stream; gbt_iris_hessian: hessian gain; gbt_iris, gbt_abalone: the single-thread manager), by the GOLDEN
// METRIC VALUES of the reference's C++ tests of the discretized path (BaseDiscretizedNumerical, HessianDiscretizedNumerical:
// all four within YDF_TEST_METRIC's 1e-4) and of eleven more of its GBT tests (Base, Subsampling*, HessianAndSubsampling,
// L2Regularization, HessianL2Categorical, LeafWiseGrow, RandomCategorical, HessianRandomCategorical, FakeMulticlass*)
// reproduced by oracle_gbt_train_validated on its own state (tests/test_adult.py, tests/test_reference_replay.py),
// and by artefacts the reference itself produced: the node statistics of its golden model
// test_data/model/8bits_numerical_binary_class_gbdt (a GBT trained on DISCRETIZED_NUMERICAL features: split-score,
// leaf and na_value formulas, tests/test_oracle_kat.py) and, for the model format, its golden Adult GBT model with
// the golden predictions of its `predict` tool (tests/test_model_io.py).
// Tie-break order between equal-score features = the per-node std::shuffle of the candidates on the learner's
// mt19937.  No reference test pins it, the replays do: all 229 tied nodes of the three runs follow the stream with
// libc++'s shuffle algorithm (shuffle_candidates = 2; 1 = libstdc++'s, which the golden models do NOT follow).
// Order of EQUAL category buckets = the reference's std::sort; the goldens follow libc++'s LLVM >= 16 introsort, restated
// below (libcxx_sort), which is what lets whole runs with categorical ties be reproduced.
// As test switches pinned on those goldens the file also restates stochastic gradient boosting, growing_strategy
// BEST_FIRST_GLOBAL, categorical_algorithm RANDOM (the one the engine does not have) and the exact numerical splitter's
// threshold rule on buckets that hold one distinct value each.
// Example weights (oracle_set_weights: weighted bucket filler, leaves, losses, initial predictions; variance gain) are
// pinned on the reference's weighted KATs (loss_imp_binomial_test.cc:92-188, loss_imp_mean_square_error_test.cc:74-177,
// loss_utils_test.cc:58-79); no reference test holds a TREE trained with weights, so beyond those the weighted path is
// held to two properties (unit weights == the pinned unweighted run bit for bit, integer weights == repeated rows).
// GOSS (SampleTrainingExamplesWithGoss) is pinned on the sampler KAT gradient_boosted_trees_test.cc:472-506; the two
// golden metric values of the reference's GOSS tests equal its UNSAMPLED Base run's and do not pin the path (DESIGN.md §19).
// DART (oracle_set_dart: DartPredictionAccumulator's draws, sampled gradients, updates and model scaling in
// oracle_gbt_train_validated) is pinned on the golden metric values of GradientBoostedTreesOnIris.Dart
// (gradient_boosted_trees_test.cc:1774-1784: accuracy and log loss within YDF_TEST_METRIC's 1e-4,
// tests/test_reference_replay.py), on the gbt_iris configuration whose golden run the loop reproduces in full.
//
// Every function cites the reference file:line it follows; paths are relative to
// /root/reference/yggdrasil_decision_forests/.  Storage types are the reference's:
// bins uint16 (65535 = missing, dataset/data_spec.h:45-48), example ids uint32, gradients f32,
// variance buckets f64, hessian buckets f32 accumulated sequentially in row order.

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <queue>
#include <numeric>
#include <random>
#include <vector>

#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>

#include "../include/ygg_b200.h"

namespace {

constexpr uint16_t kMissing = 65535;            // dataset/data_spec.h:45-48
constexpr double kMinHessianForNewtonStep = 0.001;  // splitter_accumulator.h:753, loss_utils.cc

// learner/decision_tree/utils.h:83-95
template <typename T1, typename T2>
T1 l1_threshold(const T1 value, const T2 l1) {
  if (l1 == static_cast<T2>(0)) return value;
  const T1 length = std::max(static_cast<T1>(0), std::abs(value) - static_cast<T1>(l1));
  return value > 0 ? length : -length;
}

// Feature-parallel / row-block-parallel helper standing in for the reference's
// StreamProcessor / ConcurrentForLoop thread pools (utils/concurrency_streamprocessor.h:31-92).
// fn(thread_index, item) for item in [0, n), dynamically scheduled on a PERSISTENT pool of workers (the
// reference keeps its splitter threads alive for the whole training too, training.cc:1490-1530): a parallel
// region costs two condition-variable hand-offs instead of `num_threads` thread creations per tree node.
// Only one region runs at a time (regions are never nested on this path).
class WorkerPool {
 public:
  static WorkerPool& Get() {
    static WorkerPool* pool = new WorkerPool();  // leaked on purpose: workers may outlive static destructors
    return *pool;
  }
  // Runs job(worker_index) on `workers` threads (worker 0 = the caller) and returns when all are done.
  void Run(int workers, const std::function<void(int)>& job) {
    std::unique_lock<std::mutex> region(region_mu_);  // one region at a time
    Grow(workers - 1);
    {
      std::lock_guard<std::mutex> lk(mu_);
      job_ = &job;
      active_ = workers - 1;
      pending_ = workers - 1;
      generation_++;
    }
    cv_start_.notify_all();
    job(0);
    std::unique_lock<std::mutex> lk(mu_);
    cv_done_.wait(lk, [&] { return pending_ == 0; });
    job_ = nullptr;
  }

 private:
  void Grow(int n) {
    while (static_cast<int>(threads_.size()) < n) {
      const int idx = static_cast<int>(threads_.size());
      uint64_t seen;
      {
        std::lock_guard<std::mutex> lk(mu_);
        seen = generation_;
      }
      threads_.emplace_back([this, idx, seen]() mutable {
        while (true) {
          const std::function<void(int)>* job = nullptr;
          {
            std::unique_lock<std::mutex> lk(mu_);
            cv_start_.wait(lk, [&] { return generation_ != seen; });
            seen = generation_;
            if (idx < active_) job = job_;
          }
          if (job == nullptr) continue;
          (*job)(idx + 1);
          std::lock_guard<std::mutex> lk(mu_);
          if (--pending_ == 0) cv_done_.notify_one();
        }
      });
      threads_.back().detach();
    }
  }
  std::mutex region_mu_, mu_;
  std::condition_variable cv_start_, cv_done_;
  std::vector<std::thread> threads_;
  const std::function<void(int)>* job_ = nullptr;
  int active_ = 0, pending_ = 0;
  uint64_t generation_ = 0;
};

template <typename Fn>
void ParallelFor(int num_threads, int64_t n, int64_t chunk, Fn fn) {
  if (num_threads <= 1 || n <= chunk) {
    for (int64_t i = 0; i < n; i++) fn(0, i);
    return;
  }
  std::atomic<int64_t> next(0);
  const int workers = static_cast<int>(std::min<int64_t>(num_threads, (n + chunk - 1) / chunk));
  const std::function<void(int)> job = [&](int t) {
    while (true) {
      const int64_t begin = next.fetch_add(chunk);
      if (begin >= n) break;
      const int64_t end = std::min(n, begin + chunk);
      for (int64_t i = begin; i < end; i++) fn(t, i);
    }
  };
  WorkerPool::Get().Run(workers, job);
}

struct Dataset {
  int64_t n_rows;
  int32_t n_features;
  const uint16_t* bins;  // [F][N]
  const int32_t* num_bins;
  const int32_t* na_bin;
  const int32_t* feature_type = nullptr;  // null: all DISCRETIZED_NUMERICAL; 1 = CATEGORICAL
  const uint16_t* col(int f) const { return bins + static_cast<int64_t>(f) * n_rows; }
  bool categorical(int f) const { return feature_type != nullptr && feature_type[f] == 1; }
};

// Test switch: break ties between equal bucket keys by bucket index (std::stable_sort) instead of
// the reference's std::sort, whose tie order is an implementation detail of libstdc++'s introsort.
// The GPU sorts (key, index) pairs, i.e. the stable order; comparisons against it use this mode.
int g_stable_category_sort = 0;  // 0: libstdc++'s std::sort; 1: stable; 2: libc++'s std::sort (LLVM <= 15); 3: libc++ >= 16

// libc++'s std::sort as shipped up to LLVM 15 (libcxx/include/__algorithm/sort.h: __sort3/4/5, __insertion_sort_3 for up to
// 30 trivially copyable elements, otherwise median-of-3 (of 5 from 1000 elements) quicksort with
// __insertion_sort_incomplete shortcuts).  std::sort is not stable and its order of EQUAL elements is an implementation
// detail; the reference sorts the category buckets by label mean with it (splitter_scanner.h:904-908), so which categories
// end up on which side of a tie depends on the standard library of the build.  Mode 2 of the category sort.
namespace libcxx_sort {
template <class C> unsigned sort3(int* x, int* y, int* z, C c) {
  unsigned r = 0;
  if (!c(*y, *x)) {
    if (!c(*z, *y)) return r;
    std::swap(*y, *z); r = 1;
    if (c(*y, *x)) { std::swap(*x, *y); r = 2; }
    return r;
  }
  if (c(*z, *y)) { std::swap(*x, *z); return 1; }
  std::swap(*x, *y); r = 1;
  if (c(*z, *y)) { std::swap(*y, *z); r = 2; }
  return r;
}
template <class C> unsigned sort4(int* x1, int* x2, int* x3, int* x4, C c) {
  unsigned r = sort3(x1, x2, x3, c);
  if (c(*x4, *x3)) { std::swap(*x3, *x4); ++r;
    if (c(*x3, *x2)) { std::swap(*x2, *x3); ++r;
      if (c(*x2, *x1)) { std::swap(*x1, *x2); ++r; } } }
  return r;
}
template <class C> unsigned sort5(int* x1, int* x2, int* x3, int* x4, int* x5, C c) {
  unsigned r = sort4(x1, x2, x3, x4, c);
  if (c(*x5, *x4)) { std::swap(*x4, *x5); ++r;
    if (c(*x4, *x3)) { std::swap(*x3, *x4); ++r;
      if (c(*x3, *x2)) { std::swap(*x2, *x3); ++r;
        if (c(*x2, *x1)) { std::swap(*x1, *x2); ++r; } } } }
  return r;
}
template <class C> void insertion_sort_3(int* first, int* last, C c) {
  int* j = first + 2;
  sort3(first, first + 1, j, c);
  for (int* i = j + 1; i != last; ++i) {
    if (c(*i, *j)) {
      int t = *i; int* k = j; j = i;
      do { *j = *k; j = k; } while (j != first && c(t, *--k));
      *j = t;
    }
    j = i;
  }
}
template <class C> bool insertion_sort_incomplete(int* first, int* last, C c) {
  switch (last - first) {
    case 0: case 1: return true;
    case 2: if (c(*--last, *first)) std::swap(*first, *last); return true;
    case 3: sort3(first, first + 1, --last, c); return true;
    case 4: sort4(first, first + 1, first + 2, --last, c); return true;
    case 5: sort5(first, first + 1, first + 2, first + 3, --last, c); return true;
  }
  int* j = first + 2;
  sort3(first, first + 1, j, c);
  const unsigned limit = 8;
  unsigned count = 0;
  for (int* i = j + 1; i != last; ++i) {
    if (c(*i, *j)) {
      int t = *i; int* k = j; j = i;
      do { *j = *k; j = k; } while (j != first && c(t, *--k));
      *j = t;
      if (++count == limit) return ++i == last;
    }
    j = i;
  }
  return true;
}
template <class C> void sort(int* first, int* last, C c) {
  const std::ptrdiff_t limit = 30;
  while (true) {
  restart:
    std::ptrdiff_t len = last - first;
    switch (len) {
      case 0: case 1: return;
      case 2: if (c(*--last, *first)) std::swap(*first, *last); return;
      case 3: sort3(first, first + 1, --last, c); return;
      case 4: sort4(first, first + 1, first + 2, --last, c); return;
      case 5: sort5(first, first + 1, first + 2, first + 3, --last, c); return;
    }
    if (len <= limit) { insertion_sort_3(first, last, c); return; }
    int* m = first;
    int* lm1 = last; --lm1;
    unsigned n_swaps;
    {
      std::ptrdiff_t delta;
      if (len >= 1000) { delta = len / 2; m += delta; delta /= 2; n_swaps = sort5(first, first + delta, m, m + delta, lm1, c); }
      else { delta = len / 2; m += delta; n_swaps = sort3(first, m, lm1, c); }
    }
    int* i = first;
    int* j = lm1;
    if (!c(*i, *m)) {
      while (true) {
        if (i == --j) {
          ++i; j = last;
          if (!c(*first, *--j)) {
            while (true) {
              if (i == j) return;
              if (c(*first, *i)) { std::swap(*i, *j); ++n_swaps; ++i; break; }
              ++i;
            }
          }
          if (i == j) return;
          while (true) {
            while (!c(*first, *i)) ++i;
            while (c(*first, *--j)) {}
            if (i >= j) break;
            std::swap(*i, *j); ++n_swaps; ++i;
          }
          first = i;
          goto restart;
        }
        if (c(*j, *m)) { std::swap(*i, *j); ++n_swaps; break; }
      }
    }
    ++i;
    if (i < j) {
      while (true) {
        while (c(*i, *m)) ++i;
        while (!c(*--j, *m)) {}
        if (i > j) break;
        std::swap(*i, *j); ++n_swaps;
        if (m == i) m = j;
        ++i;
      }
    }
    if (i != m && c(*m, *i)) { std::swap(*i, *m); ++n_swaps; }
    if (n_swaps == 0) {
      const bool fs = insertion_sort_incomplete(first, i, c);
      if (insertion_sort_incomplete(i + 1, last, c)) { if (fs) return; last = i; continue; }
      else if (fs) { first = ++i; continue; }
    }
    if (i - first < last - i) { sort(first, i, c); first = ++i; }
    else { sort(i + 1, last, c); last = i; }
  }
}

// libc++'s std::sort from LLVM 16 on (__introsort in sort.h, the pdqsort-style rewrite) for element types that are not
// arithmetic (category buckets are structs, so no bitset partition): insertion sort below 24 elements, median of 3 moved
// to the FRONT as pivot (ninther above 128), __partition_with_equals_on_right / _on_left, __insertion_sort_incomplete
// shortcuts when a partition needed no swap.  Mode 3 of the category sort.
template <class C> void insertion_sort_plain(int* first, int* last, C c) {
  if (first == last) return;
  for (int* i = first + 1; i != last; ++i) {
    int* j = i - 1;
    if (c(*i, *j)) {
      int t = *i; int* k = j; j = i;
      do { *j = *k; j = k; } while (j != first && c(t, *--k));
      *j = t;
    }
  }
}
template <class C> void insertion_sort_unguarded(int* first, int* last, C c) {
  if (first == last) return;
  for (int* i = first + 1; i != last; ++i) {
    int* j = i - 1;
    if (c(*i, *j)) {
      int t = *i; int* k = j; j = i;
      do { *j = *k; j = k; } while (c(t, *--k));  // an element <= t exists to the left of `first`
      *j = t;
    }
  }
}
template <class C> std::pair<int*, bool> partition_equals_on_right(int* first, int* last, C c) {
  int* begin = first;
  const int pivot = *first;
  do { ++first; } while (c(*first, pivot));
  if (begin == first - 1) { while (first < last && !c(*--last, pivot)) {} }
  else { while (!c(*--last, pivot)) {} }
  const bool already_partitioned = first >= last;
  while (first < last) {
    std::swap(*first, *last);
    while (c(*++first, pivot)) {}
    while (!c(*--last, pivot)) {}
  }
  int* pivot_pos = first - 1;
  if (begin != pivot_pos) *begin = *pivot_pos;
  *pivot_pos = pivot;
  return {pivot_pos, already_partitioned};
}
template <class C> int* partition_equals_on_left(int* first, int* last, C c) {
  int* begin = first;
  const int pivot = *first;
  if (c(pivot, *(last - 1))) { while (!c(pivot, *++first)) {} }
  else { while (++first < last && !c(pivot, *first)) {} }
  if (first < last) { while (c(pivot, *--last)) {} }
  while (first < last) {
    std::swap(*first, *last);
    while (!c(pivot, *++first)) {}
    while (c(pivot, *--last)) {}
  }
  int* pivot_pos = first - 1;
  if (begin != pivot_pos) *begin = *pivot_pos;
  *pivot_pos = pivot;
  return first;
}
template <class C> void introsort(int* first, int* last, C c, int depth, bool leftmost = true) {
  const std::ptrdiff_t limit = 24, ninther_threshold = 128;
  while (true) {
    std::ptrdiff_t len = last - first;
    switch (len) {
      case 0: case 1: return;
      case 2: if (c(*--last, *first)) std::swap(*first, *last); return;
      case 3: sort3(first, first + 1, --last, c); return;
      case 4: sort4(first, first + 1, first + 2, --last, c); return;
      case 5: sort5(first, first + 1, first + 2, first + 3, --last, c); return;
    }
    if (len < limit) {
      if (leftmost) insertion_sort_plain(first, last, c); else insertion_sort_unguarded(first, last, c);
      return;
    }
    if (depth == 0) { std::make_heap(first, last, c); std::sort_heap(first, last, c); return; }
    --depth;
    const std::ptrdiff_t half = len / 2;
    if (len > ninther_threshold) {
      sort3(first, first + half, last - 1, c);
      sort3(first + 1, first + (half - 1), last - 2, c);
      sort3(first + 2, first + (half + 1), last - 3, c);
      sort3(first + (half - 1), first + half, first + (half + 1), c);
      std::swap(*first, *(first + half));
    } else {
      sort3(first + half, first, last - 1, c);
    }
    if (!leftmost && !c(*(first - 1), *first)) {
      first = partition_equals_on_left(first, last, c);
      continue;
    }
    auto ret = partition_equals_on_right(first, last, c);
    int* i = ret.first;
    if (ret.second) {
      const bool fs = insertion_sort_incomplete(first, i, c);
      if (insertion_sort_incomplete(i + 1, last, c)) { if (fs) return; last = i; continue; }
      else if (fs) { first = ++i; continue; }
    }
    introsort(first, i, c, depth, leftmost);
    leftmost = false;
    first = ++i;
  }
}
template <class C> void sort_llvm16(int* first, int* last, C c) {
  const std::ptrdiff_t n = last - first;
  int depth = 0;
  for (std::ptrdiff_t k = n; k > 1; k >>= 1) depth++;   // 2 * floor(log2(n))
  introsort(first, last, c, 2 * depth);
}
}  // namespace libcxx_sort

// Test switch: the EXACT numerical splitter's threshold rule on buckets that hold one distinct value each
// (oracle_set_bucket_values).  FeatureNumericalBucket::Filler::SetConditionFinal (splitter_accumulator.h:213-232) puts
// the threshold at MidThreshold(v_lo, v_hi) (utils.h:103-109) of the two neighbouring values PRESENT in the node and sets
// na_value = (na_replacement >= threshold); the discretized path interpolates over the empty BUCKETS instead
// (:304-328).  Both cut the training rows identically; they differ for an unseen value inside the gap.
std::vector<std::vector<float>> g_bucket_values;  // [feature][bucket] -> the value of the bucket; empty: discretized rule
std::vector<float> g_na_replacement;              // [feature] NumericalSpec.mean

inline float MidThreshold(float a, float b) {
  float threshold = a + (b - a) / 2.f;
  if (threshold <= a) threshold = b;
  return threshold;
}

// proto::NodeCondition fields the path writes.
struct Condition {
  int32_t attribute = -1;
  float threshold_value = std::numeric_limits<float>::quiet_NaN();  // Higher.threshold (exact rule only)
  int32_t threshold = 0;  // DiscretizedHigher.threshold
  bool na_value = false;
  float split_score = 0.f;  // proto default 0
  int64_t num_examples = 0;
  int64_t num_pos_examples = 0;
  double num_pos_weighted = 0;
  bool is_categorical = false;
  uint32_t mask[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // positive categories (Contains condition)
};

enum SplitSearchResult { kBetterSplitFound, kNoBetterSplitFound, kInvalidAttribute };

// categorical_algorithm = RANDOM (proto::Categorical::Random; ScanSplitsRandomBuckets, splitter_scanner.h:1435-1569) — what
// the reference also switches to on its own from arity_limit_for_random (300) categories on.  Test switch
// (oracle_set_categorical_random).  Trials = min(max_num_trials, 32 + active^num_trial_exponent)
// (NumTrialsForRandomCategoricalSplit, training.cc:98-108).  Each trial draws its mask from the random engine it is given:
// `random_bits = (*random)()` into a uint64 consumed 64 buckets at a time — mt19937 yields 32 bits, so within every
// group of 64 ACTIVE buckets the last 32 always go to the positive side (bit == 0 selects positive).
int g_categorical_random = 0;
float g_random_num_trial_exponent = 2.f;
int g_random_max_num_trials = 5000;

inline int NumRandomCategoricalTrials(int active_dictionary_size) {
  const int num_trials = 32 + std::pow(active_dictionary_size, g_random_num_trial_exponent);
  return std::min(num_trials, g_random_max_num_trials);
}

// Exact rule (see g_bucket_values): lo = the best boundary's bucket, hi = the next non-empty one.
template <typename Items>
bool ApplyExactThresholdRule(int f, const Items& items, int best_bucket_idx, int num_bins, Condition* condition) {
  if (f >= static_cast<int>(g_bucket_values.size()) || g_bucket_values[f].empty()) return false;
  const std::vector<float>& values = g_bucket_values[f];
  int hi = best_bucket_idx + 1;
  while (hi < num_bins && items[hi].count == 0) hi++;
  if (hi >= num_bins) return false;
  const float threshold = MidThreshold(values[best_bucket_idx], values[hi]);
  int k = best_bucket_idx + 1;
  while (k < hi && values[k] < threshold) k++;   // first bucket whose value is >= threshold
  condition->threshold = k;
  condition->threshold_value = threshold;
  condition->na_value = g_na_replacement[f] >= threshold;
  return true;
}

// ---------------------------------------------------------------------------------------------
// Variance gain: LabelNumericalBucket / LabelNumericalScoreAccumulator
// (splitter_accumulator.h:1473-1566, :611-631; utils/distribution.h:42-131).
struct NormalDist {  // utils::NormalDistributionDouble
  double sum = 0, sum_squares = 0, count = 0;
  void AddF(float v) {  // distribution.h:66-71, Value = float: v*v is a float product
    sum += v;
    sum_squares += v * v;
    count += 1.f;
  }
  void AddW(float v, float w) {  // distribution.h:58-64, Value = float: v*w and (v*w)*v are float products
    const float value_weight = v * w;
    sum += value_weight;
    sum_squares += value_weight * v;
    count += w;
  }
  void Add(const NormalDist& o) { sum += o.sum; sum_squares += o.sum_squares; count += o.count; }
  void Sub(const NormalDist& o) { sum -= o.sum; sum_squares -= o.sum_squares; count -= o.count; }
  double VarTimesSumWeights() const { return sum_squares - (sum * sum) / count; }  // :118-120
};
struct VarBucket { NormalDist value; int64_t count = 0; };
// Example weights of the rows the current tree is trained on (LabelNumericalBucket<weighted=true>,
// splitter_accumulator.h:1552-1560; SetLeafValueWithNewtonRaphsonStep<true>, loss_utils.cc:81-89), or null.
const float* g_weights = nullptr;
std::vector<float> g_all_weights;  // oracle_set_weights: one weight per row of the dataset handed to oracle_gbt_train*

// Hessian gain: LabelHessianNumericalBucket (splitter_accumulator.h:1662-1824) and
// LabelHessianNumericalScoreAccumulator (:749-830).
struct HessBucket { float sum_gradient = 0, sum_hessian = 0; int64_t count = 0; double dg = 0, dh = 0; };
// Test switch: accumulate the hessian-gain buckets in double instead of the reference's float.
// The reference's f32 sequential sums are order-dependent at the 1e-6..1e-5 level; comparing the
// GPU's exact fixed-point sums against BOTH modes separates "reference rounding" from real bugs
// (SURVEY.md §7 hard part 2).
bool g_hessian_buckets_double = false;
struct HessAcc {
  double sum_gradient = 0, sum_hessian = 0, sum_weights = 0, l1 = 0, l2 = 0;
  double Score() const {  // :755-773 (no min/max constraint on this path)
    const double numerator = l1_threshold(sum_gradient, l1);
    const double denominator = std::max(sum_hessian, kMinHessianForNewtonStep) + l2;
    return numerator * numerator / denominator;
  }
};

struct TreeConfig {
  int max_depth, min_examples;
  bool in_split_min_examples_check, use_hessian_gain, subtract_parent;
  double l1, l2, l2_categorical;
  float shrinkage, clamp_leaf_logit;
  bool logit_loss;
  int leaf_mode;  // 0 = Newton step (GBT), 1 = label mean (plain regression tree KAT)
  int num_threads;
  int shuffle_candidates;  // 0: dataspec order; 1: libstdc++'s std::shuffle; 2: libc++'s std::shuffle (golden models)
};

// FillExampleBucketSet + ScanSplits<bucket_interpolation=true> for one (node, feature),
// variance gain.  splitter_scanner.h:859-909 (fill), :931-1101 (scan), :911-926 (Score);
// dispatch training.cc:904-940 and :2806-2835.
SplitSearchResult FindSplitVariance(const Dataset& ds, const uint32_t* rows, int64_t n,
                                    const float* labels, int f, const NormalDist& parent,
                                    int min_num_obs, Condition* condition,
                                    std::vector<VarBucket>* cache, std::mt19937* random = nullptr) {
  const int num_bins = ds.num_bins[f];
  const int na_bin = ds.na_bin[f];
  const uint16_t* col = ds.col(f);
  auto& items = *cache;
  items.assign(num_bins, VarBucket());
  for (int64_t i = 0; i < n; i++) {  // splitter_scanner.h:877-886
    const uint32_t r = rows[i];
    uint16_t b = col[r];
    if (b == kMissing) b = static_cast<uint16_t>(na_bin);  // splitter_accumulator.h:288-299
    if (g_weights) items[b].value.AddW(labels[r], g_weights[r]);  // :1552-1560
    else items[b].value.AddF(labels[r]);
    items[b].count++;
  }
  if (items.size() <= 1) return kInvalidAttribute;  // splitter_scanner.h:944-946
  const bool categorical = ds.categorical(f);
  if (categorical && g_categorical_random) {
    // ScanSplitsRandomBuckets (splitter_scanner.h:1435-1569), variance gain
    std::vector<int> active;
    for (int b = 0; b < num_bins; b++) if (items[b].count > 0) active.push_back(b);
    if (active.size() <= 1) return kInvalidAttribute;
    const double initial_variance_time_weight = parent.VarTimesSumWeights();
    const double sum_weights = parent.count;
    double best_score = std::max<double>(condition->split_score, 0.0);
    std::vector<int> best_pos, pos_buckets;
    int64_t best_num_pos = 0;
    double best_num_pos_w = 0;
    bool tried_one_split = false;
    const int num_trials = NumRandomCategoricalTrials(static_cast<int>(active.size()));
    for (int trial = 0; trial < num_trials; trial++) {
      pos_buckets.clear();
      int64_t num_pos_examples = 0;
      NormalDist neg = parent, pos;  // InitFull(&neg), InitEmpty(&pos)
      uint64_t random_bits = 0;
      int bits_left = 0;
      for (const int b : active) {
        if (bits_left == 0) { random_bits = (*random)(); bits_left = 64; }
        if ((random_bits & 1) == 0) {
          num_pos_examples += items[b].count;
          neg.Sub(items[b].value);
          pos.Add(items[b].value);
          pos_buckets.push_back(b);
        }
        random_bits >>= 1;
        bits_left--;
      }
      const int64_t num_neg_examples = n - num_pos_examples;
      if (num_pos_examples < min_num_obs || num_neg_examples < min_num_obs) continue;
      const double score = (initial_variance_time_weight - (pos.VarTimesSumWeights() + neg.VarTimesSumWeights())) / sum_weights;
      tried_one_split = true;
      if (score > best_score) {
        best_pos = pos_buckets;
        best_score = score;
        best_num_pos = num_pos_examples;
        best_num_pos_w = pos.count;
      }
    }
    if (best_pos.empty()) return tried_one_split ? kNoBetterSplitFound : kInvalidAttribute;
    condition->is_categorical = true;
    for (auto& m : condition->mask) m = 0u;
    bool na_in_pos = false;
    for (const int v : best_pos) {  // SetConditionFinalWithBuckets (splitter_accumulator.h:447-454)
      condition->mask[v >> 5] |= 1u << (v & 31);
      if (v == na_bin) na_in_pos = true;
    }
    condition->threshold = 0;
    condition->na_value = na_in_pos;
    condition->attribute = f;
    condition->num_examples = n;
    condition->num_pos_examples = best_num_pos;
    condition->num_pos_weighted = best_num_pos_w;
    condition->split_score = static_cast<float>(best_score);
    return kBetterSplitFound;
  }
  // FindBestSplit<..., require_label_sorting=true> (splitter_scanner.h:1823-1826): the buckets are
  // sorted by label mean (LabelNumericalBucket::operator<, splitter_accumulator.h:1492-1494)
  // before the scan (:904-908).  order[k] = category of the k-th bucket.
  std::vector<int> order(num_bins);
  std::iota(order.begin(), order.end(), 0);
  if (categorical) {
    auto mean = [&](int b) { return items[b].value.count == 0 ? 0.0 : items[b].value.sum / items[b].value.count; };
    auto less = [&](int a, int b) { return mean(a) < mean(b); };
    if (g_stable_category_sort == 3) libcxx_sort::sort_llvm16(order.data(), order.data() + order.size(), less);
    else if (g_stable_category_sort == 2) libcxx_sort::sort(order.data(), order.data() + order.size(), less);
    else if (g_stable_category_sort) std::stable_sort(order.begin(), order.end(), less);
    else std::sort(order.begin(), order.end(), less);
  }

  // Initializer (splitter_accumulator.h:1495-1532).
  const double initial_variance_time_weight = parent.VarTimesSumWeights();
  const double sum_weights = parent.count;
  NormalDist neg, pos = parent;  // InitEmpty / InitFull
  int64_t num_pos_examples = n, num_neg_examples = 0;
  bool tried_one_split = false;
  const double weighted_num_examples = pos.count;
  const int end_bucket_idx = num_bins - 1;
  double best_score = std::max<double>(condition->split_score, 0.0);  // MinimumScore() = 0
  int best_bucket_idx = -1, best_bucket_interpolation_idx = -1;
  bool no_new_examples_since_last_new_best_split = false;
  int64_t best_num_pos = 0;
  double best_num_pos_w = 0;

  for (int bucket_idx = 0; bucket_idx < end_bucket_idx; bucket_idx++) {
    const VarBucket& item = items[order[bucket_idx]];
    if (!categorical && no_new_examples_since_last_new_best_split && item.count > 0) {  // :993-1000 (interpolation: discretized only)
      best_bucket_interpolation_idx = bucket_idx;
      no_new_examples_since_last_new_best_split = false;
    }
    neg.Add(item.value);  // :1004-1005
    pos.Sub(item.value);
    num_pos_examples -= item.count;
    num_neg_examples += item.count;
    if (num_pos_examples < min_num_obs) break;     // :1019-1024
    if (num_neg_examples < min_num_obs) continue;  // :1026-1031
    // Score<> with kNormalizeByWeight=false (:911-926) and NormalizeScore (:1517-1519).
    const double score_neg = neg.VarTimesSumWeights();
    const double score_pos = pos.VarTimesSumWeights();
    const double score = (initial_variance_time_weight - (score_pos + score_neg)) / sum_weights;
    tried_one_split = true;
    if (score > best_score) {  // :1047
      best_bucket_idx = bucket_idx;
      best_score = score;
      best_num_pos = num_pos_examples;
      best_num_pos_w = pos.count;
      no_new_examples_since_last_new_best_split = true;
      best_bucket_interpolation_idx = -1;
    }
  }
  if (best_bucket_idx == -1) return tried_one_split ? kNoBetterSplitFound : kInvalidAttribute;
  int final_idx = best_bucket_idx;
  if (best_bucket_interpolation_idx != -1 &&
      best_bucket_interpolation_idx != best_bucket_idx + 1) {  // :1076-1086
    final_idx = (best_bucket_idx + best_bucket_interpolation_idx) / 2;  // accumulator.h:314-328
  }
  condition->is_categorical = categorical;
  for (auto& m : condition->mask) m = 0u;
  if (categorical) {
    // FeatureCategoricalBucket::Filler::SetConditionFinal (splitter_accumulator.h:391-411): the
    // buckets after the best one form the positive set; na_value = NA replacement in that set.
    bool na_in_pos = false;
    for (int k = best_bucket_idx + 1; k < num_bins; k++) {
      const int v = order[k];
      condition->mask[v >> 5] |= 1u << (v & 31);
      if (v == na_bin) na_in_pos = true;
    }
    condition->threshold = 0;
    condition->na_value = na_in_pos;
  } else if (!ApplyExactThresholdRule(f, items, best_bucket_idx, num_bins, condition)) {
    condition->threshold = final_idx + 1;  // splitter_accumulator.h:304-312
    condition->na_value = na_bin > final_idx;
  }
  condition->attribute = f;
  condition->num_examples = n;
  condition->num_pos_examples = best_num_pos;
  condition->num_pos_weighted = best_num_pos_w;
  condition->split_score = static_cast<float>(best_score);  // :1095, float proto field
  (void)weighted_num_examples;
  return kBetterSplitFound;
}

// Same for hessian gain.  Dispatch training.cc:662-703, :2665-2700; f32 sequential bucket sums
// (splitter_accumulator.h:1806-1814); initializer :1698-1768.
SplitSearchResult FindSplitHessian(const Dataset& ds, const uint32_t* rows, int64_t n,
                                   const float* gradients, const float* hessians, int f,
                                   double sum_gradient, double sum_hessian, double sum_weights,
                                   const TreeConfig& cfg, int min_num_obs, Condition* condition,
                                   std::vector<HessBucket>* cache, std::mt19937* random = nullptr) {
  const int num_bins = ds.num_bins[f];
  const int na_bin = ds.na_bin[f];
  const uint16_t* col = ds.col(f);
  auto& items = *cache;
  items.assign(num_bins, HessBucket());
  for (int64_t i = 0; i < n; i++) {
    const uint32_t r = rows[i];
    uint16_t b = col[r];
    if (b == kMissing) b = static_cast<uint16_t>(na_bin);
    items[b].sum_gradient += gradients[r];  // float += float, row order
    items[b].sum_hessian += hessians[r];
    items[b].dg += gradients[r];
    items[b].dh += hessians[r];
    items[b].count++;
  }
  if (g_hessian_buckets_double) {
    // not the reference's arithmetic: exact-sum variant for cross-checking
    for (auto& it : items) { it.sum_gradient = 0; it.sum_hessian = 0; }
  }
  if (items.size() <= 1) return kInvalidAttribute;
  const bool categorical = ds.categorical(f);
  // Categorical features use hessian_l2_categorical for the bucket priority, the parent score and
  // the split scores (training.cc:3203-3213).
  const double l2 = categorical ? cfg.l2_categorical : cfg.l2;
  if (categorical && g_categorical_random) {
    // ScanSplitsRandomBuckets, hessian gain (initializer as below: splitter_accumulator.h:1706-1747)
    std::vector<int> active;
    for (int b = 0; b < num_bins; b++) if (items[b].count > 0) active.push_back(b);
    if (active.size() <= 1) return kInvalidAttribute;
    const double sg_l1 = l1_threshold(sum_gradient, cfg.l1);
    const double parent_full = (sg_l1 * sg_l1) / (sum_hessian + l2);
    const double parent_sub = cfg.subtract_parent ? parent_full : 0.0;
    double best_score = std::max<double>(condition->split_score, cfg.subtract_parent ? 0.0 : parent_full);
    std::vector<int> best_pos, pos_buckets;
    int64_t best_num_pos = 0;
    double best_num_pos_w = 0;
    bool tried_one_split = false;
    const int num_trials = NumRandomCategoricalTrials(static_cast<int>(active.size()));
    for (int trial = 0; trial < num_trials; trial++) {
      pos_buckets.clear();
      int64_t num_pos_examples = 0;
      HessAcc neg, pos;
      neg.l1 = pos.l1 = cfg.l1;
      neg.l2 = pos.l2 = l2;
      neg.sum_gradient = sum_gradient;  // InitFull(&neg)
      neg.sum_hessian = sum_hessian;
      neg.sum_weights = sum_weights;
      uint64_t random_bits = 0;
      int bits_left = 0;
      for (const int b : active) {
        if (bits_left == 0) { random_bits = (*random)(); bits_left = 64; }
        if ((random_bits & 1) == 0) {
          const HessBucket& item = items[b];
          const float cnt_f = static_cast<float>(item.count);
          const double bg = g_hessian_buckets_double ? item.dg : static_cast<double>(item.sum_gradient);
          const double bh = g_hessian_buckets_double ? item.dh : static_cast<double>(item.sum_hessian);
          num_pos_examples += item.count;
          neg.sum_gradient -= bg; neg.sum_hessian -= bh; neg.sum_weights -= cnt_f;
          pos.sum_gradient += bg; pos.sum_hessian += bh; pos.sum_weights += cnt_f;
          pos_buckets.push_back(b);
        }
        random_bits >>= 1;
        bits_left--;
      }
      const int64_t num_neg_examples = n - num_pos_examples;
      if (num_pos_examples < min_num_obs || num_neg_examples < min_num_obs) continue;
      const double score = (pos.Score() + neg.Score()) - parent_sub;
      tried_one_split = true;
      if (score > best_score) {
        best_pos = pos_buckets;
        best_score = score;
        best_num_pos = num_pos_examples;
        best_num_pos_w = pos.sum_weights;
      }
    }
    if (best_pos.empty()) return tried_one_split ? kNoBetterSplitFound : kInvalidAttribute;
    condition->is_categorical = true;
    for (auto& m : condition->mask) m = 0u;
    bool na_in_pos = false;
    for (const int v : best_pos) {
      condition->mask[v >> 5] |= 1u << (v & 31);
      if (v == na_bin) na_in_pos = true;
    }
    condition->threshold = 0;
    condition->na_value = na_in_pos;
    condition->attribute = f;
    condition->num_examples = n;
    condition->num_pos_examples = best_num_pos;
    condition->num_pos_weighted = best_num_pos_w;
    condition->split_score = static_cast<float>(best_score);
    return kBetterSplitFound;
  }
  std::vector<int> order(num_bins);
  std::iota(order.begin(), order.end(), 0);
  if (categorical) {
    // LabelHessianNumericalBucket::Filler::Finalize (splitter_accumulator.h:1797-1804) computes a
    // float priority per bucket; SortLabel orders by it (:1699-1701).
    std::vector<float> priority(num_bins);
    for (int b = 0; b < num_bins; b++) {
      const double sg = g_hessian_buckets_double ? items[b].dg : static_cast<double>(items[b].sum_gradient);
      const double sh = g_hessian_buckets_double ? items[b].dh : static_cast<double>(items[b].sum_hessian);
      priority[b] = sh > 0 ? static_cast<float>(l1_threshold(sg, cfg.l1) / (sh + l2)) : 0.f;
    }
    auto less = [&](int a, int b) { return priority[a] < priority[b]; };
    if (g_stable_category_sort == 3) libcxx_sort::sort_llvm16(order.data(), order.data() + order.size(), less);
    else if (g_stable_category_sort == 2) libcxx_sort::sort(order.data(), order.data() + order.size(), less);
    else if (g_stable_category_sort) std::stable_sort(order.begin(), order.end(), less);
    else std::sort(order.begin(), order.end(), less);
  }

  // Initializer constructor (splitter_accumulator.h:1706-1727).
  const double sum_gradient_l1 = l1_threshold(sum_gradient, cfg.l1);
  const double parent_score_full = (sum_gradient_l1 * sum_gradient_l1) / (sum_hessian + l2);
  const double parent_score = cfg.subtract_parent ? parent_score_full : 0.0;
  const double min_score = cfg.subtract_parent ? 0.0 : parent_score_full;

  HessAcc neg, pos;
  neg.l1 = pos.l1 = cfg.l1;
  neg.l2 = pos.l2 = l2;
  pos.sum_gradient = sum_gradient;  // InitFull
  pos.sum_hessian = sum_hessian;
  pos.sum_weights = sum_weights;
  int64_t num_pos_examples = n, num_neg_examples = 0;
  bool tried_one_split = false;
  const int end_bucket_idx = num_bins - 1;
  double best_score = std::max<double>(condition->split_score, min_score);
  int best_bucket_idx = -1, best_bucket_interpolation_idx = -1;
  bool no_new = false;
  int64_t best_num_pos = 0;
  double best_num_pos_w = 0;
  for (int bucket_idx = 0; bucket_idx < end_bucket_idx; bucket_idx++) {
    const HessBucket& item = items[order[bucket_idx]];
    if (!categorical && no_new && item.count > 0) {
      best_bucket_interpolation_idx = bucket_idx;
      no_new = false;
    }
    // AddToScoreAcc / SubToScoreAcc, unweighted: weight = static_cast<float>(count) (:1677-1697)
    const float cnt_f = static_cast<float>(item.count);
    const double bg = g_hessian_buckets_double ? item.dg : static_cast<double>(item.sum_gradient);
    const double bh = g_hessian_buckets_double ? item.dh : static_cast<double>(item.sum_hessian);
    neg.sum_gradient += bg;
    neg.sum_hessian += bh;
    neg.sum_weights += cnt_f;
    pos.sum_gradient -= bg;
    pos.sum_hessian -= bh;
    pos.sum_weights -= cnt_f;
    num_pos_examples -= item.count;
    num_neg_examples += item.count;
    if (num_pos_examples < min_num_obs) break;
    if (num_neg_examples < min_num_obs) continue;
    const double score = (pos.Score() + neg.Score()) - parent_score;  // NormalizeScore :1745-1747
    tried_one_split = true;
    if (score > best_score) {
      best_bucket_idx = bucket_idx;
      best_score = score;
      best_num_pos = num_pos_examples;
      best_num_pos_w = pos.sum_weights;
      no_new = true;
      best_bucket_interpolation_idx = -1;
    }
  }
  if (best_bucket_idx == -1) return tried_one_split ? kNoBetterSplitFound : kInvalidAttribute;
  int final_idx = best_bucket_idx;
  if (best_bucket_interpolation_idx != -1 && best_bucket_interpolation_idx != best_bucket_idx + 1)
    final_idx = (best_bucket_idx + best_bucket_interpolation_idx) / 2;
  condition->is_categorical = categorical;
  for (auto& m : condition->mask) m = 0u;
  if (categorical) {
    bool na_in_pos = false;
    for (int k = best_bucket_idx + 1; k < num_bins; k++) {
      const int v = order[k];
      condition->mask[v >> 5] |= 1u << (v & 31);
      if (v == na_bin) na_in_pos = true;
    }
    condition->threshold = 0;
    condition->na_value = na_in_pos;
  } else if (!ApplyExactThresholdRule(f, items, best_bucket_idx, num_bins, condition)) {
    condition->threshold = final_idx + 1;
    condition->na_value = na_bin > final_idx;
  }
  condition->attribute = f;
  condition->num_examples = n;
  condition->num_pos_examples = best_num_pos;
  condition->num_pos_weighted = best_num_pos_w;
  condition->split_score = static_cast<float>(best_score);
  return kBetterSplitFound;
}

// ---------------------------------------------------------------------------------------------
struct Node {
  Condition cond;
  bool is_leaf = true;
  int depth = 1;
  int neg = -1, pos = -1;
  float top_value = 0;
  double stat[3] = {0, 0, 0};
  int64_t n = 0;
};

// SetLeafValueWithNewtonRaphsonStep<weighted=false> (loss/loss_utils.cc:49-132), or the plain
// regression leaf (label mean) for the decision-tree KAT.
void SetLeaf(const TreeConfig& cfg, const uint32_t* rows, int64_t n, const float* gradient,
             const float* hessian, Node* node) {
  double sum_g = 0, sum_g2 = 0, sum_h = 0;
  double sum_weights = static_cast<double>(n);
  if (g_weights) {  // :81-89: float products weight * unit, in this order
    sum_weights = 0;
    for (int64_t i = 0; i < n; i++) {
      const float g = gradient[rows[i]];
      const float h = hessian ? hessian[rows[i]] : 1.f;
      const float weight = g_weights[rows[i]];
      sum_g += weight * g;
      sum_h += weight * h;
      if (!cfg.use_hessian_gain) sum_g2 += weight * g * g;
      sum_weights += weight;
    }
  } else
  for (int64_t i = 0; i < n; i++) {
    const float g = gradient[rows[i]];
    const float h = hessian ? hessian[rows[i]] : 1.f;
    sum_g += g;
    sum_h += h;
    if (!cfg.use_hessian_gain) sum_g2 += g * g;  // float product, :94
  }
  if (cfg.leaf_mode == 1) {
    node->stat[0] = sum_g; node->stat[1] = sum_g2; node->stat[2] = sum_weights;
    node->top_value = static_cast<float>(sum_g / sum_weights);
    return;
  }
  if (sum_h <= kMinHessianForNewtonStep) sum_h = kMinHessianForNewtonStep;  // :101-103
  if (cfg.use_hessian_gain) {
    node->stat[0] = sum_g; node->stat[1] = sum_h; node->stat[2] = sum_weights;
  } else {
    node->stat[0] = sum_g; node->stat[1] = sum_g2; node->stat[2] = sum_weights;
  }
  const double numerator = l1_threshold(sum_g, cfg.l1);
  const double denominator = sum_h + cfg.l2;
  float value = cfg.shrinkage * numerator / denominator;  // :121-123
  if (cfg.logit_loss) value = std::clamp(value, -cfg.clamp_leaf_logit, cfg.clamp_leaf_logit);
  node->top_value = value;
}

struct SplitCaches {
  std::vector<VarBucket> var;
  std::vector<HessBucket> hess;
};

SplitSearchResult EvalFeature(const Dataset& ds, const TreeConfig& cfg, const uint32_t* rows,
                              int64_t n, const float* g, const float* h, const Node& node, int f,
                              Condition* cond, SplitCaches* caches, std::mt19937* random = nullptr) {
  const int min_num_obs = cfg.in_split_min_examples_check ? cfg.min_examples : 1;  // :840-841
  if (cfg.use_hessian_gain) {
    return FindSplitHessian(ds, rows, n, g, h, f, node.stat[0], node.stat[1], node.stat[2], cfg,
                            min_num_obs, cond, &caches->hess, random);
  }
  NormalDist parent;  // label_distribution.Load(parent.regressor().distribution()) :1908
  parent.sum = node.stat[0];
  parent.sum_squares = node.stat[1];
  parent.count = node.stat[2];
  return FindSplitVariance(ds, rows, n, g, f, parent, min_num_obs, cond, &caches->var, random);
}

// FindBestCondition -> FindBestConditionManager (training.cc:1795-1818):
//  num_threads <= 1 : FindBestConditionSingleThreadManager (:1364-1488) — the running best
//                     condition (float split_score) is the floor of every later feature's scan;
//  num_threads  > 1 : FindBestConditionConcurrentManager (:1490-1793) — each feature is scanned
//                     against the node's initial score; results are consumed in candidate order
//                     and compared as floats with strict '>' (:1740-1744).
// std::shuffle is implementation-defined.  libc++ (llvm libcxx/include/__algorithm/shuffle.h + uniform_int_distribution
// over __independent_bits_engine): for every position but the last draw i in [0, d] as the low w bits of one engine
// word, redrawn while >= d + 1 (w = bits of d + 1), and swap.  The reference's golden PYDF models were built against
// libc++: their tie-breaks between equal-score features follow this order on all 229 ties of three complete runs
// (tests/test_reference_replay.py).
// libc++'s uniform_int_distribution over [0, rp) on mt19937: nothing drawn for rp == 1, else the low w bits of one word
// (2^w >= rp), redrawn while >= rp.
uint32_t UniformIntLibcxx(uint64_t rp, std::mt19937* g) {
  if (rp == 1) return 0;
  int w = 63 - __builtin_clzll(rp);
  if (rp & ((1ull << w) - 1)) ++w;
  uint32_t u;
  do { u = (*g)() & static_cast<uint32_t>((1ull << w) - 1); } while (u >= rp);
  return u;
}

void ShuffleLibcxx(std::vector<int32_t>* v, std::mt19937* g) {
  const int64_t n = static_cast<int64_t>(v->size());
  int64_t d = n - 1;
  for (int64_t first = 0; first < n - 1; ++first, --d) {
    const uint32_t u = UniformIntLibcxx(static_cast<uint64_t>(d) + 1, g);
    if (u != 0) std::swap((*v)[first], (*v)[first + u]);
  }
}

bool FindBestCondition(const Dataset& ds, const TreeConfig& cfg, const uint32_t* rows, int64_t n,
                       const float* g, const float* h, const Node& node, std::mt19937* random,
                       Condition* best, std::vector<SplitCaches>* caches) {
  const int F = ds.n_features;
  std::vector<int32_t> candidates(F);
  std::iota(candidates.begin(), candidates.end(), 0);
  if (cfg.shuffle_candidates == 2) {
    ShuffleLibcxx(&candidates, random);
  } else if (cfg.shuffle_candidates) {
    std::shuffle(candidates.begin(), candidates.end(), *random);  // training.cc:4293-4306
  }
  bool found = false;
  if (cfg.num_threads <= 1) {
    for (int i = 0; i < F; i++) {
      if (EvalFeature(ds, cfg, rows, n, g, h, node, candidates[i], best, &(*caches)[0], random) ==
          kBetterSplitFound)  // one thread: the splitters draw from the learner's engine itself
        found = true;
    }
    return found;
  }
  // Concurrent manager: one RNG draw per job for the request seed (:1658) + discard (:1781).
  // (every job gets its own engine seeded with that word: SplitterWorkRequest.seed)
  std::vector<uint32_t> seeds(F, 0u);
  if (cfg.shuffle_candidates) for (int i = 0; i < F; i++) seeds[i] = (*random)();
  std::vector<Condition> results(F);
  std::vector<int> status(F);
  const float initial_score = best->split_score;
  ParallelFor(cfg.num_threads, F, 1, [&](int tid, int64_t i) {
    Condition c;
    c.split_score = initial_score;
    if (g_categorical_random && ds.categorical(candidates[i])) {  // the only consumer of the job's engine on this path
      std::mt19937 job_random(seeds[i]);
      status[i] = EvalFeature(ds, cfg, rows, n, g, h, node, candidates[i], &c, &(*caches)[tid], &job_random);
    } else {
      status[i] = EvalFeature(ds, cfg, rows, n, g, h, node, candidates[i], &c, &(*caches)[tid]);
    }
    results[i] = c;
  });
  float best_split_score = best->split_score;
  for (int i = 0; i < F; i++) {
    if (status[i] == kBetterSplitFound && results[i].split_score > best_split_score) {
      *best = results[i];
      best_split_score = results[i].split_score;
      found = true;
    }
  }
  return found;
}

// SplitExamplesInPlace -> EvalConditionTemplate (model/decision_tree/decision_tree.cc:957-1012)
// with EvalConditionDiscretizedHigher (:724-743): positives forward, negatives backward, then
// the negatives are reversed => both children keep the parent's (ascending) order.
// Categorical conditions: EvalConditionContainsCategorical / ContainsBitmap (decision_tree.cc:766-812).
int64_t PartitionRows(const uint16_t* col, int threshold, bool na_value, const uint32_t* active,
                      uint32_t* inactive, int64_t n, const uint32_t* mask = nullptr) {
  int64_t next_pos = 0, next_neg = n - 1;
  for (int64_t i = 0; i < n; i++) {
    const uint32_t r = active[i];
    const uint16_t v = col[r];
    const bool eval = (v == kMissing) ? na_value
                                      : (mask ? ((mask[v >> 5] >> (v & 31)) & 1u) != 0 : (v >= threshold));
    if (eval) inactive[next_pos++] = r; else inactive[next_neg--] = r;
  }
  std::reverse(inactive + next_pos, inactive + n);
  return next_pos;
}

// DecisionTreeTrain -> GrowTreeLocal -> NodeTrain (training.cc:4658, :5051-5082, :4865-5049):
// explicit stack, positive child processed first, root depth 1.
extern int g_best_first_global;
void TrainTreeBestFirstGlobal(const Dataset& ds, const TreeConfig& cfg, const float* g, const float* h,
                              std::mt19937* random, std::vector<Node>* nodes, std::vector<uint32_t>* buf_a,
                              std::vector<uint32_t>* buf_b, const std::vector<uint32_t>* selected);

// `selected` = the rows the tree is trained on (ascending; nullptr: all rows) — the selected_examples of
// decision_tree::Train (gradient_boosted_trees.cc:1507-1511).
void TrainTree(const Dataset& ds, const TreeConfig& cfg, const float* g, const float* h,
               std::mt19937* random, std::vector<Node>* nodes, std::vector<uint32_t>* buf_a,
               std::vector<uint32_t>* buf_b, const std::vector<uint32_t>* selected = nullptr) {
  if (g_best_first_global) {
    TrainTreeBestFirstGlobal(ds, cfg, g, h, random, nodes, buf_a, buf_b, selected);
    return;
  }
  const int64_t N = selected ? static_cast<int64_t>(selected->size()) : ds.n_rows;
  buf_a->resize(N);
  buf_b->resize(N);
  if (selected) std::copy(selected->begin(), selected->end(), buf_a->begin());
  else std::iota(buf_a->begin(), buf_a->end(), 0u);
  nodes->clear();
  nodes->reserve(1024);
  nodes->emplace_back();
  std::vector<SplitCaches> caches(std::max(1, cfg.num_threads));
  struct Work { int node; uint32_t* active; uint32_t* inactive; int64_t n; int depth; bool leaf_set; };
  std::vector<Work> stack;
  stack.push_back({0, buf_a->data(), buf_b->data(), N, 1, false});
  while (!stack.empty()) {
    Work w = stack.back();
    stack.pop_back();
    Node* node = &(*nodes)[w.node];
    node->n = w.n;
    node->depth = w.depth;
    if (!w.leaf_set) SetLeaf(cfg, w.active, w.n, g, h, node);  // :4888-4894
    if (w.n < cfg.min_examples || (cfg.max_depth >= 0 && w.depth >= cfg.max_depth)) continue;  // :4909
    Condition cond;
    if (!FindBestCondition(ds, cfg, w.active, w.n, g, h, *node, random, &cond, &caches)) continue;
    const int64_t n_pos = PartitionRows(ds.col(cond.attribute), cond.threshold, cond.na_value,
                                        w.active, w.inactive, w.n, cond.is_categorical ? cond.mask : nullptr);
    if (n_pos == 0 || n_pos == w.n) continue;  // :4981-4987 (children cleared, stays a leaf)
    const int pos_idx = static_cast<int>(nodes->size());
    nodes->emplace_back();
    const int neg_idx = static_cast<int>(nodes->size());
    nodes->emplace_back();
    node = &(*nodes)[w.node];
    node->cond = cond;
    node->is_leaf = false;
    node->pos = pos_idx;
    node->neg = neg_idx;
    // Children: active <- inactive span, inactive <- active span (:988-993 of decision_tree.cc).
    SetLeaf(cfg, w.inactive, n_pos, g, h, &(*nodes)[pos_idx]);                     // :5007-5012
    SetLeaf(cfg, w.inactive + n_pos, w.n - n_pos, g, h, &(*nodes)[neg_idx]);
    stack.push_back({neg_idx, w.inactive + n_pos, w.active + n_pos, w.n - n_pos, w.depth + 1, true});
    stack.push_back({pos_idx, w.inactive, w.active, n_pos, w.depth + 1, true});      // :5031-5046
  }
  // Depth of never-visited children is set when popped; all pushed nodes are popped.
}

// growing_strategy = BEST_FIRST_GLOBAL (GrowTreeBestFirstGlobal, training.cc:4499-4656): a max-heap of candidate
// splits keyed by split_score * n (float); the best one is applied, its children are ingested POSITIVE FIRST (each
// ingest sets the leaf value and runs FindBestCondition, i.e. consumes the candidate shuffle), until max_num_nodes
// leaves exist (default 31, -1 = unlimited).  Root depth is 0 here (1 in the local growth): with the same max_depth
// the tree may be one level deeper.  Test switch: oracle_set_growing_strategy.
int g_best_first_global = 0;
int g_max_num_nodes = 31;

void TrainTreeBestFirstGlobal(const Dataset& ds, const TreeConfig& cfg, const float* g, const float* h,
                              std::mt19937* random, std::vector<Node>* nodes, std::vector<uint32_t>* buf_a,
                              std::vector<uint32_t>* buf_b, const std::vector<uint32_t>* selected) {
  const int64_t N = selected ? static_cast<int64_t>(selected->size()) : ds.n_rows;
  buf_a->resize(N);
  buf_b->resize(N);
  if (selected) std::copy(selected->begin(), selected->end(), buf_a->begin());
  else std::iota(buf_a->begin(), buf_a->end(), 0u);
  nodes->clear();
  nodes->reserve(4096);
  nodes->emplace_back();
  std::vector<SplitCaches> caches(std::max(1, cfg.num_threads));
  struct Candidate {
    Condition cond; uint32_t* active; uint32_t* inactive; int64_t n; float score; int node; int depth;
    bool operator<(const Candidate& o) const { return score < o.score; }
  };
  std::priority_queue<Candidate> candidates;
  auto ingest = [&](uint32_t* active, uint32_t* inactive, int64_t n, int node_idx, int depth) {
    Node* node = &(*nodes)[node_idx];
    node->n = n;
    node->depth = depth + 1;  // reported like the local growth (root = 1)
    SetLeaf(cfg, active, n, g, h, node);
    if (n < cfg.min_examples || (cfg.max_depth >= 0 && depth >= cfg.max_depth)) return;
    Condition cond;
    if (!FindBestCondition(ds, cfg, active, n, g, h, *node, random, &cond, &caches)) return;
    candidates.push({cond, active, inactive, n, cond.split_score * static_cast<float>(n), node_idx, depth});
  };
  ingest(buf_a->data(), buf_b->data(), N, 0, 0);
  int num_nodes = 1;
  while (!candidates.empty() && (g_max_num_nodes < 0 || num_nodes < g_max_num_nodes)) {
    while (g_max_num_nodes >= 0 && static_cast<int>(candidates.size()) > g_max_num_nodes) candidates.pop();
    Candidate split = candidates.top();
    candidates.pop();
    const int64_t n_pos = PartitionRows(ds.col(split.cond.attribute), split.cond.threshold, split.cond.na_value,
                                        split.active, split.inactive, split.n,
                                        split.cond.is_categorical ? split.cond.mask : nullptr);
    const int pos_idx = static_cast<int>(nodes->size());
    nodes->emplace_back();
    const int neg_idx = static_cast<int>(nodes->size());
    nodes->emplace_back();
    Node* node = &(*nodes)[split.node];
    node->cond = split.cond;
    node->is_leaf = false;
    node->pos = pos_idx;
    node->neg = neg_idx;
    ingest(split.inactive, split.active, n_pos, pos_idx, split.depth + 1);
    ingest(split.inactive + n_pos, split.active + n_pos, split.n - n_pos, neg_idx, split.depth + 1);
    num_nodes++;
  }
}

// Pre-order emission: node, negative subtree, positive subtree (decision_tree.cc:624-632).
void EmitPreOrder(const std::vector<Node>& nodes, int idx, std::vector<ygg_node>* out) {
  const Node& n = nodes[idx];
  const int my = static_cast<int>(out->size());
  out->emplace_back();
  ygg_node o;
  std::memset(&o, 0, sizeof(o));
  o.feature = n.is_leaf ? -1 : n.cond.attribute;
  o.threshold_bin = n.is_leaf ? 0 : n.cond.threshold;
  o.na_value = n.is_leaf ? 0 : (n.cond.na_value ? 1 : 0);
  o.depth = n.depth;
  o.neg_child = o.pos_child = -1;
  o.split_score = n.is_leaf ? 0.f : n.cond.split_score;
  o.leaf_value = n.top_value;
  o.num_examples = n.n;
  o.num_pos_examples = n.is_leaf ? 0 : n.cond.num_pos_examples;
  o.stat[0] = n.stat[0]; o.stat[1] = n.stat[1]; o.stat[2] = n.stat[2];
  o.condition_type = (!n.is_leaf && n.cond.is_categorical) ? YGG_FEATURE_CATEGORICAL : YGG_FEATURE_DISCRETIZED_NUMERICAL;
  if (!n.is_leaf && !n.cond.is_categorical && !std::isnan(n.cond.threshold_value)) {
    o.threshold_value = n.cond.threshold_value;  // exact rule: the float threshold
  }
  if (!n.is_leaf && n.cond.is_categorical) std::memcpy(o.cat_mask, n.cond.mask, sizeof(o.cat_mask));
  if (!n.is_leaf) {
    o.neg_child = static_cast<int>(out->size());
    (*out)[my] = o;
    EmitPreOrder(nodes, n.neg, out);
    o.pos_child = static_cast<int>(out->size());
    (*out)[my] = o;
    EmitPreOrder(nodes, n.pos, out);
  }
  (*out)[my] = o;
}

TreeConfig MakeTreeConfig(const ygg_gbt_config& c, int num_threads, int shuffle, int leaf_mode) {
  TreeConfig t;
  t.max_depth = c.max_depth;
  t.min_examples = c.min_examples;
  t.in_split_min_examples_check = c.in_split_min_examples_check != 0;
  t.use_hessian_gain = c.use_hessian_gain != 0;
  t.subtract_parent = c.hessian_split_score_subtract_parent != 0;
  t.l1 = c.l1_regularization;
  t.l2 = c.l2_regularization;
  t.l2_categorical = c.l2_regularization_categorical;
  t.shrinkage = c.shrinkage;
  t.clamp_leaf_logit = c.clamp_leaf_logit;
  t.logit_loss = c.loss == YGG_LOSS_BINOMIAL_LOG_LIKELIHOOD ||
                 c.loss == YGG_LOSS_MULTINOMIAL_LOG_LIKELIHOOD;  // IsLogitLoss, loss_utils.cc:41-45
  t.leaf_mode = leaf_mode;
  t.num_threads = num_threads;
  t.shuffle_candidates = shuffle;
  return t;
}

// DecisionTree::GetLeaf with EvalConditionDiscretizedHigher (decision_tree.cc:1572, :724-743).
inline float LeafOf(const Dataset& ds, const std::vector<ygg_node>& tree, int64_t r) {
  int i = 0;
  while (tree[i].feature >= 0) {
    const uint16_t v = ds.col(tree[i].feature)[r];
    const bool eval = (v == kMissing) ? (tree[i].na_value != 0)
                      : (tree[i].condition_type == YGG_FEATURE_CATEGORICAL
                             ? ((tree[i].cat_mask[v >> 5] >> (v & 31)) & 1u) != 0
                             : (v >= tree[i].threshold_bin));
    i = eval ? tree[i].pos_child : tree[i].neg_child;
  }
  return tree[i].leaf_value;
}

}  // namespace

extern "C" {

// Single (node, feature) fill + scan, for the KATs.  hessians may be null (variance gain).
// parent_stat: variance (sum, sum_squares, count) / hessian (sum_g, sum_h, sum_w).
// Returns 0 = better split found, 1 = no better split, 2 = invalid attribute.
int oracle_find_split(const uint16_t* column, int64_t n_rows, int32_t num_bins, int32_t na_bin,
                      const uint32_t* rows, int64_t n, const float* gradients,
                      const float* hessians, const double* parent_stat, int32_t use_hessian_gain,
                      int32_t min_num_obs, double l1, double l2, int32_t subtract_parent,
                      float initial_split_score, int32_t* threshold, int32_t* na_value,
                      float* split_score, int64_t* num_pos, int32_t categorical, uint32_t* mask_out) {
  const int32_t ftype = categorical ? 1 : 0;
  Dataset ds{n_rows, 1, column, &num_bins, &na_bin, &ftype};
  Condition c;
  c.split_score = initial_split_score;
  SplitSearchResult r;
  if (use_hessian_gain) {
    TreeConfig cfg{};
    cfg.l1 = l1; cfg.l2 = l2; cfg.l2_categorical = l2; cfg.subtract_parent = subtract_parent != 0;
    std::vector<HessBucket> cache;
    r = FindSplitHessian(ds, rows, n, gradients, hessians, 0, parent_stat[0], parent_stat[1],
                         parent_stat[2], cfg, min_num_obs, &c, &cache);
  } else {
    NormalDist p; p.sum = parent_stat[0]; p.sum_squares = parent_stat[1]; p.count = parent_stat[2];
    std::vector<VarBucket> cache;
    r = FindSplitVariance(ds, rows, n, gradients, 0, p, min_num_obs, &c, &cache);
  }
  *threshold = c.threshold; *na_value = c.na_value; *split_score = c.split_score;
  *num_pos = c.num_pos_examples;
  if (mask_out) std::memcpy(mask_out, c.mask, sizeof(c.mask));
  return static_cast<int>(r);
}

// SplitExamplesInPlace KAT.  Returns n_pos; out = [positives..., negatives...].
int64_t oracle_partition(const uint16_t* column, int32_t threshold, int32_t na_value,
                         const uint32_t* rows, int64_t n, uint32_t* out) {
  return PartitionRows(column, threshold, na_value != 0, rows, out, n);
}

// decision_tree::Train on caller gradients.  leaf_mode 0 = Newton, 1 = label mean.
// Returns the node count (pre-order), or -1 if capacity is too small.
int32_t oracle_train_tree(const uint16_t* bins, int64_t n_rows, int32_t n_features,
                          const int32_t* num_bins, const int32_t* na_bin, const float* gradients,
                          const float* hessians, const ygg_gbt_config* cfg, int32_t num_threads,
                          int32_t shuffle_candidates, int32_t leaf_mode, ygg_node* out,
                          int32_t capacity, const int32_t* feature_type) {
  Dataset ds{n_rows, n_features, bins, num_bins, na_bin, feature_type};
  TreeConfig t = MakeTreeConfig(*cfg, num_threads, shuffle_candidates, leaf_mode);
  std::mt19937 random(cfg->random_seed);
  std::vector<Node> nodes;
  std::vector<uint32_t> a, b;
  const float* weights = static_cast<int64_t>(g_all_weights.size()) == n_rows ? g_all_weights.data() : nullptr;
  if (weights && cfg->use_hessian_gain) return -2;  // weighted hessian gain is not restated
  struct WeightScope { WeightScope(const float* w) { g_weights = w; } ~WeightScope() { g_weights = nullptr; } } weight_scope(weights);
  TrainTree(ds, t, gradients, hessians, &random, &nodes, &a, &b);
  std::vector<ygg_node> flat;
  EmitPreOrder(nodes, 0, &flat);
  if (static_cast<int32_t>(flat.size()) > capacity) return -1;
  std::memcpy(out, flat.data(), flat.size() * sizeof(ygg_node));
  return static_cast<int32_t>(flat.size());
}

// The same with the learner's random engine supplied by the caller (oracle_rng_*), so that the per-node candidate
// shuffles continue the stream of a whole training run.
int32_t oracle_train_tree_rng(const uint16_t* bins, int64_t n_rows, int32_t n_features,
                              const int32_t* num_bins, const int32_t* na_bin, const float* gradients,
                              const float* hessians, const ygg_gbt_config* cfg, int32_t num_threads,
                              int32_t shuffle_candidates, void* rng, ygg_node* out, int32_t capacity,
                              const int32_t* feature_type) {
  Dataset ds{n_rows, n_features, bins, num_bins, na_bin, feature_type};
  TreeConfig t = MakeTreeConfig(*cfg, num_threads, shuffle_candidates, 0);
  std::vector<Node> nodes;
  std::vector<uint32_t> a, b;
  TrainTree(ds, t, gradients, hessians, static_cast<std::mt19937*>(rng), &nodes, &a, &b);
  std::vector<ygg_node> flat;
  EmitPreOrder(nodes, 0, &flat);
  if (static_cast<int32_t>(flat.size()) > capacity) return -1;
  std::memcpy(out, flat.data(), flat.size() * sizeof(ygg_node));
  return static_cast<int32_t>(flat.size());
}

// loss->InitialPredictions (loss_imp_binomial.cc:65-99; loss_imp_mean_square_error.cc:56-88).
float oracle_initial_prediction_w(int32_t loss, const int32_t* labels_i32, const float* labels_f32,
                                  const float* weights, int64_t n) {
  if (loss == YGG_LOSS_BINOMIAL_LOG_LIKELIHOOD) {
    double sum_weights = static_cast<double>(n);
    double pos = 0;
    if (weights) {  // loss_imp_binomial.cc:83-88
      sum_weights = 0;
      for (int64_t i = 0; i < n; i++) {
        sum_weights += weights[i];
        pos += weights[i] * (labels_i32[i] == 2);
      }
    } else {
      pos = static_cast<double>(std::count(labels_i32, labels_i32 + n, 2));
    }
    const double ratio = pos / sum_weights;
    if (ratio == 0.0) return -std::numeric_limits<float>::max();
    if (ratio == 1.0) return std::numeric_limits<float>::max();
    return static_cast<float>(std::log(ratio / (1. - ratio)));
  }
  double s = 0, sum_weights = static_cast<double>(n);
  if (weights) {  // loss_imp_mean_square_error.cc:72-77
    sum_weights = 0;
    for (int64_t i = 0; i < n; i++) {
      sum_weights += weights[i];
      s += weights[i] * labels_f32[i];
    }
  } else {
    for (int64_t i = 0; i < n; i++) s += labels_f32[i];
  }
  return static_cast<float>(s / sum_weights);
}
float oracle_initial_prediction(int32_t loss, const int32_t* labels_i32, const float* labels_f32,
                                int64_t n) {
  return oracle_initial_prediction_w(loss, labels_i32, labels_f32, nullptr, n);
}

// loss->UpdateGradients (loss_imp_binomial.cc:124-144; loss_imp_mean_square_error.cc:96-120).
void oracle_update_gradients(int32_t loss, const int32_t* labels_i32, const float* labels_f32,
                             const float* predictions, int64_t n, float* gradient, float* hessian) {
  if (loss == YGG_LOSS_BINOMIAL_LOG_LIKELIHOOD) {
    for (int64_t i = 0; i < n; i++) {
      const float label = (labels_i32[i] == 2) ? 1.f : 0.f;
      const float prediction = predictions[i];
      const float proba = 1.f / (1.f + std::exp(-prediction));
      gradient[i] = label - proba;
      hessian[i] = proba * (1 - proba);
    }
  } else {
    for (int64_t i = 0; i < n; i++) {
      gradient[i] = labels_f32[i] - predictions[i];
      hessian[i] = 1.f;
    }
  }
}

// loss->Loss (loss_imp_binomial.cc:204-300; metric/metric.cc:2120-2170 for RMSE).
void oracle_loss_w(int32_t loss, const int32_t* labels_i32, const float* labels_f32,
                   const float* predictions, const float* weights, int64_t n, float* out_loss, float* out_secondary) {
  if (loss == YGG_LOSS_BINOMIAL_LOG_LIKELIHOOD) {
    double sum_loss = 0;
    double correct = 0, total = 0;  // IntegersConfusionMatrixDouble: trace and sum
    for (int64_t i = 0; i < n; i++) {
      const bool pos_label = labels_i32[i] == 2;
      const float label_for_loss = pos_label ? 1.f : 0.f;
      const float prediction = predictions[i];
      const int predicted_label = prediction > 0.f ? 2 : 1;
      if (weights) {  // loss_imp_binomial.cc:218-224
        const float weight = weights[i];
        total += weight;
        if (predicted_label == labels_i32[i]) correct += weight;
        sum_loss -= 2 * weight * (label_for_loss * prediction - std::log(1.f + std::exp(prediction)));
      } else {
        total += 1.f;
        if (predicted_label == labels_i32[i]) correct += 1.f;
        sum_loss -= 2 * (label_for_loss * prediction - std::log(1.f + std::exp(prediction)));
      }
    }
    *out_loss = static_cast<float>(sum_loss / total);
    *out_secondary = static_cast<float>(correct / total);
  } else {
    double sum_sq = 0, sum_weights = static_cast<double>(n);
    if (weights) {  // metric/metric.cc:2097-2111
      sum_weights = 0;
      for (int64_t i = 0; i < n; i++) {
        const float label = labels_f32[i];
        const float prediction = predictions[i];
        const float weight = weights[i];
        sum_weights += weight;
        sum_sq += weight * (label - prediction) * (label - prediction);
      }
    } else {
      for (int64_t i = 0; i < n; i++) {
        const float label = labels_f32[i];
        const float prediction = predictions[i];
        sum_sq += (label - prediction) * (label - prediction);
      }
    }
    *out_loss = static_cast<float>(std::sqrt(sum_sq / sum_weights));
    *out_secondary = *out_loss;
  }
}
void oracle_loss(int32_t loss, const int32_t* labels_i32, const float* labels_f32,
                 const float* predictions, int64_t n, float* out_loss, float* out_secondary) {
  oracle_loss_w(loss, labels_i32, labels_f32, predictions, nullptr, n, out_loss, out_secondary);
}

// SampleTrainingExamples (gradient_boosted_trees.cc:2932-2956): stochastic gradient boosting.  One word of the
// learner's mt19937 per row and iteration (uniform_real_distribution<float>), drawn BEFORE the iteration's trees;
// nothing is drawn for sample >= 1.  Returns false when every row is selected.
bool SampleTrainingExamples(int64_t num_rows, float sample, std::mt19937* random, std::vector<uint32_t>* selected) {
  if (sample >= 1.f - std::numeric_limits<float>::epsilon()) return false;
  selected->clear();
  std::uniform_real_distribution<float> unif_dist_unit;
  for (int64_t r = 0; r < num_rows; r++) {
    if (unif_dist_unit(*random) < sample) selected->push_back(static_cast<uint32_t>(r));
  }
  if (selected->empty()) {  // at least one example
    selected->push_back(std::uniform_int_distribution<uint32_t>(static_cast<uint32_t>(num_rows - 1))(*random));
  }
  return true;
}

// SampleTrainingExamplesWithGoss (gradient_boosted_trees.cc:2958-3007): rows sorted by decreasing |gradient| (L1 norm over
// the gradient dimensions; one here), the first ceil(alpha * rows) kept, each of the others kept with probability beta —
// one engine word per row, in sorted order — and its weight multiplied by (1 - alpha) / beta.  `weights` holds the dataset's
// weights on entry (all 1: use_optimized_unit_weights is off with GOSS, :1236-1242).  The sort is the reference's
// std::sort (equal keys in the standard library's order) or, with g_goss_stable_sort, a stable sort: equal keys by row
// index, which is what the engine's device radix sort gives.
int g_goss_stable_sort = 0;
void SampleTrainingExamplesWithGoss(const float* gradient, int64_t num_rows, float alpha, float beta, std::mt19937* random,
                                    std::vector<uint32_t>* selected, std::vector<float>* weights) {
  std::vector<std::pair<uint32_t, float>> l1_norm;
  l1_norm.reserve(num_rows);
  for (int64_t r = 0; r < num_rows; r++) {
    float example_l1_norm = 0.f;
    example_l1_norm += std::fabs(gradient[r]);
    l1_norm.push_back(std::make_pair(static_cast<uint32_t>(r), example_l1_norm));
  }
  auto greater = [](const std::pair<uint32_t, float>& a, const std::pair<uint32_t, float>& b) { return a.second > b.second; };
  if (g_goss_stable_sort) std::stable_sort(l1_norm.begin(), l1_norm.end(), greater);
  else std::sort(l1_norm.begin(), l1_norm.end(), greater);
  selected->clear();
  const int cutoff = std::ceil(alpha * static_cast<uint32_t>(num_rows));   // float * UnsignedExampleIdx, :2983
  for (int64_t idx = 0; idx < cutoff && idx < num_rows; idx++) selected->push_back(l1_norm[idx].first);
  if (beta > 0) {
    const float amplification_factor = (1.f - alpha) / beta;
    std::uniform_real_distribution<float> unif_dist_unit;
    for (int64_t idx = cutoff; idx < num_rows; idx++) {
      if (unif_dist_unit(*random) < beta) {
        const uint32_t example_idx = l1_norm[idx].first;
        selected->push_back(example_idx);
        (*weights)[example_idx] *= amplification_factor;
      }
    }
  }
  if (selected->empty()) {
    selected->push_back(std::uniform_int_distribution<uint32_t>(static_cast<uint32_t>(num_rows - 1))(*random));
  }
}
inline bool UsesGoss(const ygg_gbt_config& c) { return c.goss_alpha > 0.f || c.goss_beta > 0.f; }

// The boosting loop, GradientBoostedTreesLearner::TrainWithStatusImpl
// (gradient_boosted_trees.cc:1428-1571) with validation_ratio = 0, cfg->subsample (stochastic gradient boosting,
// :1484-1488), no early stopping, one tree per iteration.  Trees are written back-to-back into `out_nodes`
// (tree t occupies [tree_offsets[t], tree_offsets[t+1])).  predictions (N floats) is in/out:
// if init_predictions != 0 it is first filled with the initial prediction.
// Returns the number of trees trained, or -1 if out_nodes is too small.
int32_t oracle_gbt_train(const uint16_t* bins, int64_t n_rows, int32_t n_features,
                         const int32_t* num_bins, const int32_t* na_bin, const int32_t* labels_i32,
                         const float* labels_f32, const ygg_gbt_config* cfg, int32_t num_iters,
                         int32_t num_threads, int32_t shuffle_candidates, int32_t init_predictions,
                         float* predictions, ygg_node* out_nodes, int64_t node_capacity,
                         int64_t* tree_offsets, float* out_loss, float* out_secondary,
                         float* out_gradients, float* out_hessians, const int32_t* feature_type) {
  Dataset ds{n_rows, n_features, bins, num_bins, na_bin, feature_type};
  TreeConfig t = MakeTreeConfig(*cfg, num_threads, shuffle_candidates, 0);
  std::mt19937 random(cfg->random_seed);  // gradient_boosted_trees.cc:1198
  const int64_t N = n_rows;
  const float* weights = static_cast<int64_t>(g_all_weights.size()) == N ? g_all_weights.data() : nullptr;
  if (weights && cfg->use_hessian_gain) return -2;  // not restated
  struct WeightScope { WeightScope(const float* w) { g_weights = w; } ~WeightScope() { g_weights = nullptr; } } weight_scope(weights);
  if (init_predictions) {
    const float init = oracle_initial_prediction_w(cfg->loss, labels_i32, labels_f32, weights, N);
    std::fill(predictions, predictions + N, init);
  }
  std::vector<float> g(N), h(N), goss_weights;
  std::vector<Node> nodes;
  std::vector<uint32_t> a, b, selected;
  int64_t offset = 0;
  tree_offsets[0] = 0;
  for (int iter = 0; iter < num_iters; iter++) {
    oracle_update_gradients(cfg->loss, labels_i32, labels_f32, predictions, N, g.data(), h.data());
    if (iter == num_iters - 1 && out_gradients) {
      std::memcpy(out_gradients, g.data(), N * sizeof(float));
      std::memcpy(out_hessians, h.data(), N * sizeof(float));
    }
    bool sampled;
    if (UsesGoss(*cfg)) {   // :1455-1468: the tree sees the GOSS weights, the losses the dataset's (all 1)
      if (weights || cfg->use_hessian_gain) return -2;   // not restated
      goss_weights.assign(N, 1.f);
      SampleTrainingExamplesWithGoss(g.data(), N, cfg->goss_alpha, cfg->goss_beta, &random, &selected, &goss_weights);
      g_weights = goss_weights.data();
      sampled = true;
    } else {
      sampled = SampleTrainingExamples(N, cfg->subsample, &random, &selected);
    }
    TrainTree(ds, t, g.data(), h.data(), &random, &nodes, &a, &b, sampled ? &selected : nullptr);
    if (UsesGoss(*cfg)) g_weights = nullptr;
    std::vector<ygg_node> flat;
    EmitPreOrder(nodes, 0, &flat);
    if (offset + static_cast<int64_t>(flat.size()) > node_capacity) return -1;
    std::memcpy(out_nodes + offset, flat.data(), flat.size() * sizeof(ygg_node));
    offset += flat.size();
    tree_offsets[iter + 1] = offset;
    // UpdatePredictionWithSingleUnivariateTree (loss_utils.cc:214-229): all rows, by traversal.
    // (the reference runs this single-threaded; row blocks here only shorten the baseline run,
    // the result is identical)
    ParallelFor(num_threads, N, 1 << 16, [&](int, int64_t r) { predictions[r] += LeafOf(ds, flat, r); });
    if (out_loss) {
      oracle_loss_w(cfg->loss, labels_i32, labels_f32, predictions, weights, N, &out_loss[iter],
                    &out_secondary[iter]);
    }
  }
  return num_iters;
}

// The learner's outer loop WITH the validation hold-out and early stopping
// (GradientBoostedTreesLearner::TrainWithStatusImpl, gradient_boosted_trees.cc:1154-1740):
//   ExtractValidationDataset            :2718-2746  (row r trains iff unif_dist_01(random) > ratio; the
//                                                    first consumer of the mt19937 seeded with random_seed)
//   initial predictions on the TRAINING rows        :1288-1296, applied to the validation rows :1330-1336
//   per iteration: train tree on the training rows, UpdatePredictions on both sets :1544-1566,
//                  training / validation Loss :1573-1626, EarlyStopping::Update / ShouldStop :1628-1647
//                  (early_stopping/early_stopping.cc:30-62)
//   FinalizeModelWithValidationDataset  :212-272    (truncate to best_num_trees unless fewer than
//                                                    initial_iteration + 1 trees were trained)
// Inputs are the FULL dataset; out_in_training receives the split.  Returns the number of trees of the final
// model; *out_num_entries = iterations with log entries, out_* arrays are per iteration.
void oracle_mc_update_gradients(const int32_t* labels, int32_t K, const float* predictions, int64_t n, float* gradient,
                                float* hessian);
void oracle_mc_loss(const int32_t* labels, int32_t K, const float* predictions, int64_t n, float* out_loss,
                    float* out_secondary);
void oracle_mc_loss_w(const int32_t* labels, int32_t K, const float* predictions, const float* weights, int64_t n,
                      float* out_loss, float* out_secondary);

// Candidate-shuffle mode of oracle_gbt_train_validated (0 = dataspec order, 1 = libstdc++, 2 = libc++; FindBestCondition).
static int g_validated_shuffle_mode = 0;

// forest_extraction = DART in oracle_gbt_train_validated (oracle_set_dart; a negative rate: MART).  The draws and the
// accumulator restate DartPredictionAccumulator (gradient_boosted_trees.cc:3102-3223) with the standard library that
// g_validated_shuffle_mode selects (2: libc++, otherwise libstdc++).  The run leaves its dropped sets and the model's
// per-iteration leaf scales here (oracle_get_dart_*).
static float g_dart_rate = -1.f;
static std::vector<std::vector<int32_t>> g_dart_dropped;
static std::vector<float> g_dart_scales;

// std::uniform_real_distribution<float> on one mt19937 word.  libstdc++'s generate_canonical keeps a result that rounds to
// 1 just below it; libc++'s returns float(word) / 2^32 as it rounds, 1.0 for the words from 2^32 - 128 on.
static float DartUnitDraw(std::mt19937* random) {
  if (g_validated_shuffle_mode == 2) return static_cast<float>((*random)()) / 4294967296.f;
  return std::uniform_real_distribution<float>()(*random);
}

// SampleIterIndices (gradient_boosted_trees.cc:3108-3130): nothing drawn before the first iteration; then one unit draw
// per earlier iteration, dropped iff < rate; an empty set takes one iteration by uniform_int_distribution<int>(0, i - 1).
static std::vector<int32_t> DartSampleIterIndices(int num_iters, float rate, std::mt19937* random) {
  std::vector<int32_t> dropped;
  if (num_iters == 0) return dropped;
  for (int j = 0; j < num_iters; j++)
    if (DartUnitDraw(random) < rate) dropped.push_back(j);
  if (dropped.empty()) {
    dropped.push_back(g_validated_shuffle_mode == 2 ? static_cast<int32_t>(UniformIntLibcxx(num_iters, random))
                                                    : std::uniform_int_distribution<int>(0, num_iters - 1)(*random));
  }
  return dropped;
}

// One DartPredictionAccumulator: `acc` the full predictions, per past iteration its trees' leaf of every element
// (0 + leaf, UpdatePredictions on a zero vector, :3172-3177).  Elements are the loop's predictions, [row][K].
struct DartAccumulator {
  std::vector<float>* acc;
  std::vector<std::vector<float>> per_iter;
  // GetSampledPredictions (:3141-3163): acc -= p_j * w_j over the dropped iterations in ascending order.
  void Sampled(const std::vector<int32_t>& dropped, const std::vector<float>& w, int num_threads, std::vector<float>* out) const {
    *out = *acc;
    if (dropped.empty()) return;   // GetAllPredictions
    ParallelFor(num_threads, static_cast<int64_t>(out->size()), 1 << 16, [&](int, int64_t e) {
      float v = (*out)[e];
      for (const int32_t j : dropped) v -= per_iter[j][e] * w[j];
      (*out)[e] = v;
    });
  }
  // UpdateWithNewIteration (:3165-3214) before the weights change: acc += p_new * w_new, then
  // acc += p_j * w_j * (sf - 1) for each dropped j.
  void Update(std::vector<float>&& p_new, const std::vector<int32_t>& dropped, const std::vector<float>& w, int num_threads) {
    const float w_new = 1.0f / (dropped.size() + 1);
    const float sampled_factor = static_cast<float>(dropped.size()) / (dropped.size() + 1);
    ParallelFor(num_threads, static_cast<int64_t>(acc->size()), 1 << 16, [&](int, int64_t e) {
      float v = (*acc)[e];
      v += p_new[e] * w_new;
      for (const int32_t j : dropped) v += per_iter[j][e] * w[j] * (sampled_factor - 1.f);
      (*acc)[e] = v;
    });
    per_iter.push_back(std::move(p_new));
  }
};

int32_t oracle_gbt_train_validated(const uint16_t* bins, int64_t n_rows, int32_t n_features, const int32_t* num_bins,
                                   const int32_t* na_bin, const int32_t* labels_i32, const float* labels_f32,
                                   const ygg_gbt_config* cfg, float validation_ratio, int32_t num_threads,
                                   const int32_t* feature_type, uint8_t* out_in_training, ygg_node* out_nodes,
                                   int64_t node_capacity, int64_t* tree_offsets, float* out_train_loss,
                                   float* out_valid_loss, float* out_valid_secondary, int32_t* out_num_entries,
                                   float* out_final_validation_loss, int32_t* out_early_stopping_triggered) {
  std::mt19937 random(cfg->random_seed);
  std::uniform_real_distribution<float> unif_dist_01;
  std::vector<uint32_t> train_rows, valid_rows;
  for (int64_t r = 0; r < n_rows; r++) {
    const bool in_training = validation_ratio == 0.f ? true : unif_dist_01(random) > validation_ratio;
    out_in_training[r] = in_training ? 1 : 0;
    (in_training ? train_rows : valid_rows).push_back(static_cast<uint32_t>(r));
  }
  auto extract = [&](const std::vector<uint32_t>& rows, std::vector<uint16_t>* b, std::vector<int32_t>* li,
                     std::vector<float>* lf) {
    const int64_t n = static_cast<int64_t>(rows.size());
    b->resize(static_cast<size_t>(n) * n_features);
    for (int f = 0; f < n_features; f++)
      for (int64_t i = 0; i < n; i++) (*b)[static_cast<size_t>(f) * n + i] = bins[static_cast<size_t>(f) * n_rows + rows[i]];
    if (labels_i32) { li->resize(n); for (int64_t i = 0; i < n; i++) (*li)[i] = labels_i32[rows[i]]; }
    if (labels_f32) { lf->resize(n); for (int64_t i = 0; i < n; i++) (*lf)[i] = labels_f32[rows[i]]; }
  };
  std::vector<uint16_t> tb, vb;
  std::vector<int32_t> tli, vli;
  std::vector<float> tlf, vlf;
  extract(train_rows, &tb, &tli, &tlf);
  extract(valid_rows, &vb, &vli, &vlf);
  // example weights follow their rows into the two datasets (the hold-out is extracted from the weighted dataset,
  // gradient_boosted_trees.cc:1262-1280)
  std::vector<float> tw, vw;
  const bool weighted = static_cast<int64_t>(g_all_weights.size()) == n_rows;
  if (weighted) {
    if (cfg->use_hessian_gain) return -2;  // not restated
    for (const uint32_t r : train_rows) tw.push_back(g_all_weights[r]);
    for (const uint32_t r : valid_rows) vw.push_back(g_all_weights[r]);
  }
  const float* train_w = weighted ? tw.data() : nullptr;
  const float* valid_w = weighted ? vw.data() : nullptr;
  struct WeightScope { WeightScope(const float* w) { g_weights = w; } ~WeightScope() { g_weights = nullptr; } } weight_scope(train_w);
  const int64_t NT = static_cast<int64_t>(train_rows.size()), NV = static_cast<int64_t>(valid_rows.size());
  const bool has_valid = NV > 0;
  Dataset ds{NT, n_features, tb.data(), num_bins, na_bin, feature_type};
  Dataset vds{NV, n_features, vb.data(), num_bins, na_bin, feature_type};
  TreeConfig t = MakeTreeConfig(*cfg, num_threads, g_validated_shuffle_mode, 0);
  const int32_t* tl_i = labels_i32 ? tli.data() : nullptr;
  const float* tl_f = labels_f32 ? tlf.data() : nullptr;
  // K trees per iteration for the multinomial loss (gradient_boosted_trees.cc:1490-1511): predictions [row][K],
  // gradient planes [K][row]; early stopping counts TREES (num_trees = (iter + 1) * K), its initial iteration ITERATIONS.
  const bool multinomial = cfg->loss == YGG_LOSS_MULTINOMIAL_LOG_LIKELIHOOD;
  const int K = multinomial ? cfg->num_classes : 1;
  const float init = multinomial ? 0.f : oracle_initial_prediction_w(cfg->loss, tl_i, tl_f, train_w, NT);
  std::vector<float> pred(static_cast<size_t>(NT) * K, init), vpred(static_cast<size_t>(NV) * K, init);
  std::vector<float> g(static_cast<size_t>(NT) * K), h(static_cast<size_t>(NT) * K), goss_weights;
  std::vector<Node> nodes;
  std::vector<uint32_t> a, b, selected;
  struct { float best_loss = 0, last_loss = 0; int best_num_trees = -1, last_num_trees = 0; } es;
  const int look_ahead = cfg->early_stopping_num_trees_look_ahead, initial_iteration = cfg->early_stopping_initial_iteration;
  int64_t offset = 0;
  tree_offsets[0] = 0;
  int trained = 0;
  const int32_t* vl_i = labels_i32 ? vli.data() : nullptr;
  const float* vl_f = labels_f32 ? vlf.data() : nullptr;
  // DART (:1311-1324): one accumulator per dataset over pred / vpred, which then hold the full predictions; the two share
  // the dropped sets and therefore the weights.
  const bool dart = g_dart_rate >= 0.f;
  g_dart_dropped.clear();
  g_dart_scales.clear();
  DartAccumulator dart_train{&pred, {}}, dart_valid{&vpred, {}};
  std::vector<float> dart_w, sampled_pred;
  for (int iter = 0; iter < cfg->num_trees; iter++) {
    // :1436-1442: the draws come first in the iteration, the gradients are taken at the sampled predictions
    std::vector<int32_t> dropped;
    if (dart) {
      dropped = DartSampleIterIndices(iter, g_dart_rate, &random);
      dart_train.Sampled(dropped, dart_w, num_threads, &sampled_pred);
    }
    const float* grad_pred = dart ? sampled_pred.data() : pred.data();
    if (multinomial) oracle_mc_update_gradients(tl_i, K, grad_pred, NT, g.data(), h.data());
    else oracle_update_gradients(cfg->loss, tl_i, tl_f, grad_pred, NT, g.data(), h.data());
    bool sampled;
    if (UsesGoss(*cfg)) {
      if (weighted || multinomial || cfg->use_hessian_gain) return -2;   // not restated
      goss_weights.assign(NT, 1.f);
      SampleTrainingExamplesWithGoss(g.data(), NT, cfg->goss_alpha, cfg->goss_beta, &random, &selected, &goss_weights);
      g_weights = goss_weights.data();
      sampled = true;
    } else {
      sampled = SampleTrainingExamples(NT, cfg->subsample, &random, &selected);  // :1484-1488
    }
    std::vector<std::vector<ygg_node>> new_trees(K);
    for (int k = 0; k < K; k++) {
      TrainTree(ds, t, g.data() + static_cast<size_t>(k) * NT, h.data() + static_cast<size_t>(k) * NT, &random, &nodes,
                &a, &b, sampled ? &selected : nullptr);
      EmitPreOrder(nodes, 0, &new_trees[k]);
      if (offset + static_cast<int64_t>(new_trees[k].size()) > node_capacity) return -1;
      std::memcpy(out_nodes + offset, new_trees[k].data(), new_trees[k].size() * sizeof(ygg_node));
      offset += new_trees[k].size();
      tree_offsets[iter * K + k + 1] = offset;
    }
    trained = iter + 1;
    if (UsesGoss(*cfg)) g_weights = nullptr;
    if (dart) {
      // :1526-1541: both accumulators take the iteration with the same dropped set, then the dropped weights shrink
      std::vector<float> p_new(static_cast<size_t>(NT) * K), vp_new(static_cast<size_t>(NV) * K);
      ParallelFor(num_threads, NT, 1 << 16, [&](int, int64_t r) {
        for (int k = 0; k < K; k++) p_new[r * K + k] = LeafOf(ds, new_trees[k], r);
      });
      ParallelFor(num_threads, NV, 1 << 16, [&](int, int64_t r) {
        for (int k = 0; k < K; k++) vp_new[r * K + k] = LeafOf(vds, new_trees[k], r);
      });
      dart_train.Update(std::move(p_new), dropped, dart_w, num_threads);
      dart_valid.Update(std::move(vp_new), dropped, dart_w, num_threads);
      const float sampled_factor = static_cast<float>(dropped.size()) / (dropped.size() + 1);   // :3207-3212
      for (const int32_t j : dropped) dart_w[j] *= sampled_factor;
      dart_w.push_back(1.0f / (dropped.size() + 1));
      g_dart_dropped.push_back(std::move(dropped));
    } else {
      ParallelFor(num_threads, NT, 1 << 16, [&](int, int64_t r) {
        for (int k = 0; k < K; k++) pred[r * K + k] += LeafOf(ds, new_trees[k], r);
      });
      ParallelFor(num_threads, NV, 1 << 16, [&](int, int64_t r) {
        for (int k = 0; k < K; k++) vpred[r * K + k] += LeafOf(vds, new_trees[k], r);
      });
    }
    float sec;
    if (multinomial) oracle_mc_loss_w(tl_i, K, pred.data(), train_w, NT, &out_train_loss[iter], &sec);
    else oracle_loss_w(cfg->loss, tl_i, tl_f, pred.data(), train_w, NT, &out_train_loss[iter], &sec);
    if (has_valid) {
      if (multinomial) oracle_mc_loss_w(vl_i, K, vpred.data(), valid_w, NV, &out_valid_loss[iter], &out_valid_secondary[iter]);
      else oracle_loss_w(cfg->loss, vl_i, vl_f, vpred.data(), valid_w, NV, &out_valid_loss[iter], &out_valid_secondary[iter]);
      const float vl = out_valid_loss[iter];
      const int num_trees = (iter + 1) * K;
      if (iter >= initial_iteration && (es.best_num_trees == -1 || vl < es.best_loss)) {
        es.best_loss = vl;
        es.best_num_trees = num_trees;
      }
      es.last_loss = vl;
      es.last_num_trees = num_trees;
      if (cfg->early_stopping == YGG_EARLY_STOPPING_LOSS_INCREASE && iter >= initial_iteration &&
          es.last_num_trees - es.best_num_trees >= look_ahead)
        break;
    }
  }
  *out_num_entries = trained;
  *out_early_stopping_triggered = 0;
  *out_final_validation_loss = 0.f;
  int final_trees = trained * K;
  if (has_valid) {
    if (cfg->early_stopping == YGG_EARLY_STOPPING_NONE) {
      *out_final_validation_loss = es.last_loss;
    } else if (trained * K < (initial_iteration + 1) * K) {  // :224-228, in trees
      *out_final_validation_loss = es.last_loss;
    } else {
      *out_final_validation_loss = es.best_loss;
      final_trees = es.best_num_trees;
      *out_early_stopping_triggered = 1;
    }
  }
  if (dart) {
    // :1706-1722, after the truncation: iteration j of the kept ones scales its trees' leaves (ScaleRegressorOutput,
    // decision_tree.cc:1980-1988) by its weight as the loop ended.  The trees are returned as grown.
    g_dart_scales.assign(dart_w.begin(), dart_w.begin() + final_trees / K);
  }
  return final_trees;
}

// ---- multinomial log-likelihood (K classes, K trees per iteration) ---------------------------------
// MultinomialLogLikelihoodLoss::TemplatedUpdateGradients (loss_imp_multinomial.cc:150-193): predictions are
// interleaved [example][class]; gradients / hessians are written per class plane [class][example].
void oracle_mc_update_gradients(const int32_t* labels, int32_t K, const float* predictions, int64_t n, float* gradient,
                                float* hessian) {
  std::vector<float> accumulator(K);
  for (int64_t i = 0; i < n; i++) {
    float sum_exp = 0;
    for (int k = 0; k < K; k++) {
      const float exp_val = std::exp(predictions[k + i * K]);
      accumulator[k] = exp_val;
      sum_exp += exp_val;
    }
    const float normalization = 1.f / sum_exp;
    const int label_cat = labels[i];
    for (int k = 0; k < K; k++) {
      const float label = (label_cat == (k + 1)) ? 1.f : 0.f;
      const float prediction = accumulator[k] * normalization;
      const float grad = label - prediction;
      const float abs_grad = std::abs(grad);
      gradient[static_cast<size_t>(k) * n + i] = grad;
      hessian[static_cast<size_t>(k) * n + i] = abs_grad * (1 - abs_grad);
    }
  }
}

// TemplatedLossImp / TemplatedLoss (loss_imp_multinomial.cc:225-349), unweighted.
void oracle_mc_loss_w(const int32_t* labels, int32_t K, const float* predictions, const float* weights, int64_t n,
                      float* out_loss, float* out_secondary) {
  double loss = 0;
  double correct = 0, total = 0;   // confusion matrix: trace and sum (weights when weighted, :238-246)
  for (int64_t i = 0; i < n; i++) {
    const int label = labels[i];
    int predicted_class = -1;
    float predicted_class_exp_value = 0;
    float sum_exp = 0;
    for (int k = 0; k < K; k++) {
      const float exp_val = std::exp(predictions[k + i * K]);
      sum_exp += exp_val;
      if (exp_val > predicted_class_exp_value) {
        predicted_class_exp_value = exp_val;
        predicted_class = k + 1;
      }
    }
    const float tree_label_exp_value = std::exp(predictions[(label - 1) + i * K]);
    if (weights) {
      const float weight = weights[i];
      total += weight;
      if (predicted_class == label) correct += weight;
      loss -= weight * std::log(tree_label_exp_value / sum_exp);
    } else {
      total += 1;
      if (predicted_class == label) correct += 1;
      loss -= std::log(tree_label_exp_value / sum_exp);
    }
  }
  *out_loss = static_cast<float>(loss / total);
  *out_secondary = static_cast<float>(correct / total);
}
void oracle_mc_loss(const int32_t* labels, int32_t K, const float* predictions, int64_t n, float* out_loss,
                    float* out_secondary) {
  oracle_mc_loss_w(labels, K, predictions, nullptr, n, out_loss, out_secondary);
}

// The boosting loop with num_trees_per_iter = K (gradient_boosted_trees.cc:1428-1571; the K trees of an
// iteration are trained on the gradients taken at its start, :1490-1511, then all added to the predictions,
// :1544).  Initial predictions are 0 (initialize_with_class_priors = false, loss_imp_multinomial.cc:64-66).
// predictions: [n][K] out.  Trees are emitted iteration-major, class-minor.  Returns the number of trees.
int32_t oracle_gbt_train_mc(const uint16_t* bins, int64_t n_rows, int32_t n_features, const int32_t* num_bins,
                            const int32_t* na_bin, const int32_t* labels, const ygg_gbt_config* cfg, int32_t num_iters,
                            int32_t num_threads, const int32_t* feature_type, float* predictions, ygg_node* out_nodes,
                            int64_t node_capacity, int64_t* tree_offsets, float* out_loss, float* out_secondary) {
  const int K = cfg->num_classes;
  Dataset ds{n_rows, n_features, bins, num_bins, na_bin, feature_type};
  TreeConfig t = MakeTreeConfig(*cfg, num_threads, 0, 0);
  std::mt19937 random(cfg->random_seed);
  const int64_t N = n_rows;
  const float* weights = static_cast<int64_t>(g_all_weights.size()) == N ? g_all_weights.data() : nullptr;
  if (weights && cfg->use_hessian_gain) return -2;   // not restated
  struct WeightScope { WeightScope(const float* w) { g_weights = w; } ~WeightScope() { g_weights = nullptr; } } weight_scope(weights);
  std::fill(predictions, predictions + N * K, 0.f);
  std::vector<float> g(static_cast<size_t>(N) * K), h(static_cast<size_t>(N) * K);
  std::vector<Node> nodes;
  std::vector<uint32_t> a, b;
  int64_t offset = 0;
  int n_trees = 0;
  tree_offsets[0] = 0;
  for (int iter = 0; iter < num_iters; iter++) {
    oracle_mc_update_gradients(labels, K, predictions, N, g.data(), h.data());
    std::vector<std::vector<ygg_node>> new_trees(K);
    for (int k = 0; k < K; k++) {
      TrainTree(ds, t, g.data() + static_cast<size_t>(k) * N, h.data() + static_cast<size_t>(k) * N, &random, &nodes, &a, &b);
      EmitPreOrder(nodes, 0, &new_trees[k]);
      if (offset + static_cast<int64_t>(new_trees[k].size()) > node_capacity) return -1;
      std::memcpy(out_nodes + offset, new_trees[k].data(), new_trees[k].size() * sizeof(ygg_node));
      offset += new_trees[k].size();
      tree_offsets[++n_trees] = offset;
    }
    ParallelFor(num_threads, N, 1 << 15, [&](int, int64_t r) {
      for (int k = 0; k < K; k++) predictions[k + r * K] += LeafOf(ds, new_trees[k], r);
    });
    if (out_loss) oracle_mc_loss_w(labels, K, predictions, weights, N, &out_loss[iter], &out_secondary[iter]);
  }
  return n_trees;
}

// Installs (n_features > 0) or removes (0) the exact threshold rule: values[offsets[f] .. offsets[f + 1]) are the bucket
// values of feature f (none for a categorical feature), na_replacement[f] its NumericalSpec.mean.
void oracle_set_bucket_values(int32_t n_features, const float* values, const int64_t* offsets, const float* na_replacement) {
  g_bucket_values.clear();
  g_na_replacement.clear();
  for (int f = 0; f < n_features; f++) {
    g_bucket_values.emplace_back(values + offsets[f], values + offsets[f + 1]);
    g_na_replacement.push_back(na_replacement[f]);
  }
}
void oracle_set_categorical_random(int32_t enabled, float num_trial_exponent, int32_t max_num_trials) {
  g_categorical_random = enabled;
  g_random_num_trial_exponent = num_trial_exponent;
  g_random_max_num_trials = max_num_trials;
}
void oracle_set_growing_strategy(int32_t best_first_global, int32_t max_num_nodes) {
  g_best_first_global = best_first_global;
  g_max_num_nodes = max_num_nodes;
}
// Example weights for oracle_gbt_train / oracle_gbt_train_validated / oracle_train_tree (n = 0: unweighted).  Variance gain only.
void oracle_set_weights(const float* weights, int64_t n) {
  g_all_weights.assign(weights, weights + (weights ? n : 0));
}
void oracle_set_goss_stable_sort(int32_t enabled) { g_goss_stable_sort = enabled != 0; }
// The GOSS sampler alone (KAT gradient_boosted_trees_test.cc:472-506).  weights: in/out, n floats; returns the selected count.
int32_t oracle_goss_sample(const float* gradient, int64_t n, float alpha, float beta, void* rng, uint32_t* out_selected,
                           float* weights) {
  std::vector<uint32_t> selected;
  std::vector<float> w(weights, weights + n);
  SampleTrainingExamplesWithGoss(gradient, n, alpha, beta, static_cast<std::mt19937*>(rng), &selected, &w);
  std::copy(selected.begin(), selected.end(), out_selected);
  std::copy(w.begin(), w.end(), weights);
  return static_cast<int32_t>(selected.size());
}
void oracle_set_validated_shuffle_mode(int32_t mode) { g_validated_shuffle_mode = mode; }
// DART in oracle_gbt_train_validated at this dropout rate; negative: off (MART).
void oracle_set_dart(float rate) { g_dart_rate = rate; }
// The last DART run: its trained iterations, the dropped set of iteration `iter` (returns its size; -1: capacity too
// small or no such iteration) and the model's per-iteration leaf scales (returns their number).
int32_t oracle_get_dart_num_iterations(void) { return static_cast<int32_t>(g_dart_dropped.size()); }
int32_t oracle_get_dart_dropped(int32_t iter, int32_t* out, int32_t capacity) {
  if (iter < 0 || iter >= static_cast<int32_t>(g_dart_dropped.size())) return -1;
  const std::vector<int32_t>& d = g_dart_dropped[iter];
  if (static_cast<int32_t>(d.size()) > capacity) return -1;
  std::copy(d.begin(), d.end(), out);
  return static_cast<int32_t>(d.size());
}
int32_t oracle_get_dart_scales(float* out, int32_t capacity) {
  if (static_cast<int32_t>(g_dart_scales.size()) > capacity) return -1;
  std::copy(g_dart_scales.begin(), g_dart_scales.end(), out);
  return static_cast<int32_t>(g_dart_scales.size());
}
void oracle_set_hessian_buckets_double(int32_t enabled) { g_hessian_buckets_double = enabled != 0; }
void oracle_set_stable_category_sort(int32_t mode) { g_stable_category_sort = mode; }

// The learner's random engine, exposed so that tests can follow its stream through a training run:
// utils::RandomEngine = std::mt19937 (utils/random.h:25) seeded with TrainingConfig.random_seed; consumed by
// ExtractValidationDataset (one word per row), per split node by GetCandidateAttributes' std::shuffle
// (training.cc:4293-4306) and by one seed per split-search job (training.cc:1658, :1781).
void* oracle_rng_create(uint32_t seed) { return new std::mt19937(seed); }
void* oracle_rng_clone(void* rng) { return new std::mt19937(*static_cast<std::mt19937*>(rng)); }
void oracle_rng_destroy(void* rng) { delete static_cast<std::mt19937*>(rng); }
void oracle_rng_discard(void* rng, uint64_t n) { static_cast<std::mt19937*>(rng)->discard(n); }
uint32_t oracle_rng_next(void* rng) { return (*static_cast<std::mt19937*>(rng))(); }
void oracle_rng_shuffle(void* rng, int32_t* values, int32_t n) {
  std::shuffle(values, values + n, *static_cast<std::mt19937*>(rng));
}

int32_t oracle_max_threads(void) {
  const unsigned n = std::thread::hardware_concurrency();
  return n == 0 ? 1 : static_cast<int32_t>(n);
}

}  // extern "C"
