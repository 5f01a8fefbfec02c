/*
 * ygg_b200.h — C ABI of libygg_b200.so, the GBT split-finding engine for the H100 (sm_90a).
 *
 * Scope: the bucketised-feature (histogram) split finder of YDF's gradient-boosted-trees
 * learner, and nothing else (SURVEY.md §8).  The reference has no C ABI for this path; its
 * seam is C++ virtuals + protobuf messages.  Each entry point below names the reference
 * interface it stands in for (paths relative to the reference's yggdrasil_decision_forests/).
 *
 * Conventions (mirroring the reference's ownership / error rules, SURVEY.md §8b):
 *  - every function returns an int status: 0 = OK, non-zero = error (absl::Status analogue);
 *    the message of the last error on the calling thread is ygg_last_error();
 *    no C++ exception ever crosses this boundary;
 *  - inputs are borrowed for the duration of the call only (the engine copies to HBM);
 *  - a handle is not thread-safe; distinct handles are independent;
 *  - there is NO CPU fallback: without a CUDA device every compute entry point fails with
 *    YGG_ERR_NO_DEVICE.
 */
#ifndef YGG_B200_H_
#define YGG_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YGG_ABI_VERSION 3

enum ygg_status {
  YGG_OK = 0,
  YGG_ERR_INVALID_ARGUMENT = 1, /* absl::InvalidArgumentError */
  YGG_ERR_NO_DEVICE = 2,        /* no CUDA device / extension built without one */
  YGG_ERR_CUDA = 3,             /* a CUDA runtime call failed (absl::InternalError) */
  YGG_ERR_UNIMPLEMENTED = 4,    /* absl::UnimplementedError: option outside the hot path */
  YGG_ERR_CANCELLED = 5,        /* stop flag raised (stop_training_trigger) */
  YGG_ERR_IO = 6
};

/* proto::Loss values the hot path covers
 * (learner/gradient_boosted_trees/gradient_boosted_trees.proto; loss/loss_imp_binomial.cc,
 * loss/loss_imp_mean_square_error.cc). */
enum ygg_loss {
  YGG_LOSS_BINOMIAL_LOG_LIKELIHOOD = 0,
  YGG_LOSS_SQUARED_ERROR = 1,
  /* K >= 2 classes, labels in 1..K, K trees per iteration, one per class
   * (loss_imp_multinomial.cc; gradient_boosted_trees.cc:1490-1511); cfg.num_classes = K */
  YGG_LOSS_MULTINOMIAL_LOG_LIKELIHOOD = 2
};

/* The proto fields the path reads, as a POD.  Defaults (ygg_gbt_config_init) are the proto
 * defaults: gradient_boosted_trees.proto:35-278, decision_tree.proto:32-108,
 * gradient_boosted_trees.cc:3238-3262 (max_depth 6, all attributes tested). */
typedef struct ygg_gbt_config {
  int32_t abi_version;          /* YGG_ABI_VERSION */
  int32_t loss;                 /* enum ygg_loss */
  int32_t num_trees;            /* 300 */
  float shrinkage;              /* 0.1 */
  int32_t max_depth;            /* 6; root has depth 1, depth >= max_depth => leaf */
  int32_t min_examples;         /* 5 */
  int32_t in_split_min_examples_check; /* 1 */
  int32_t use_hessian_gain;     /* 0 => variance-reduction gain (reference default) */
  float l1_regularization;      /* 0 */
  float l2_regularization;      /* 0 */
  float l2_regularization_categorical; /* 1 (reserved for categorical features) */
  float clamp_leaf_logit;       /* 5 */
  int32_t hessian_split_score_subtract_parent; /* 0 */
  uint32_t random_seed;         /* 123456; consumed by the hold-out draw (ygg_validation_split_mask) and the tie-break replay */
  float subsample;              /* must be 1.0 (row sampling is SURVEY §8f N3) */
  float validation_ratio;       /* 0: the engine trains on the rows it is given; validation rows are attached
                                   with ygg_gbt_set_validation_* (split helpers below).  Kept for hosts that
                                   forward GradientBoostedTreesTrainingConfig.validation_set_ratio */
  int32_t sibling_subtraction;  /* 1: build the smaller child's histogram, derive the other
                                   by exact integer subtraction (bit-identical results) */
  int32_t early_stopping;       /* enum ygg_early_stopping, 2 (LOSS_INCREASE); inert without validation rows */
  int32_t early_stopping_num_trees_look_ahead; /* 30 */
  int32_t early_stopping_initial_iteration;    /* 10 */
  int32_t num_classes;          /* multinomial loss: K (2..32); ignored otherwise */
  /* Tie-break between features whose best splits have EQUAL float scores: the reference takes the first one in the
   * order of its per-node std::shuffle of the candidate features on the learner's std::mt19937
   * (GetCandidateAttributes, learner/decision_tree/training.cc:4293-4306), visiting the nodes depth-first, positive
   * child first.  0 (default): lowest feature index.  1 / 2: replay that stream with libstdc++'s / libc++'s
   * std::shuffle algorithm (the reference's golden models follow libc++'s) and give tied nodes the feature the reference
   * picks; done on the finished trees, see DESIGN.md §9.  Single GPU only. */
  int32_t candidate_shuffle;
  uint32_t rng_words_consumed;     /* words of the learner's engine drawn before the first tree (the hold-out draw:
                                      one per row when validation_ratio > 0, gradient_boosted_trees.cc:2731-2738) */
  int32_t split_jobs_draw_seeds;   /* 1: FindBestConditionConcurrentManager (num_threads > 1) — one engine word per
                                      feature job after every shuffle (training.cc:1658, :1781); 0: single-thread manager */
  /* DecisionTreeTrainingConfig.growing_strategy (decision_tree.proto:205-232).  0: growing_strategy_local (default).
   * 1: growing_strategy_best_first_global (GrowTreeBestFirstGlobal, training.cc:4499-4656): the node with the largest
   * split_score * num_examples is split next until max_num_nodes leaves exist; the root has depth 0 there, so a tree may be
   * one level deeper than with the local growth and the same max_depth.  The engine grows the full tree level-wise and
   * replays the priority queue on it (DESIGN.md §17): the scores of a node do not depend on the order of growth. */
  int32_t growing_strategy;
  int32_t max_num_nodes;           /* best-first growth: 31; -1 = unlimited */
  /* GradientOneSideSampling (gradient_boosted_trees.proto:317-335; SampleTrainingExamplesWithGoss,
   * gradient_boosted_trees.cc:2958-3007), on when alpha > 0 or beta > 0 (both 0 = off; the reference's defaults are 0.2 / 0.1):
   * every iteration the ceil(alpha * rows) rows with the largest |gradient| are kept, every other row with probability beta
   * (one word of the learner's engine each, in decreasing-|gradient| order) and weight (1 - alpha) / beta.  Rows with EQUAL
   * |gradient| are ordered by row index (the reference: whatever its std::sort does; DESIGN.md §19).  Variance gain,
   * binomial / squared error, single GPU, not with subsample < 1 or example weights.  (These 8 bytes were `reserved`, zero.) */
  float goss_alpha;
  float goss_beta;
} ygg_gbt_config;

/* GradientBoostedTreesTrainingConfig.EarlyStopping (gradient_boosted_trees.proto:150-169). */
enum ygg_early_stopping {
  YGG_EARLY_STOPPING_NONE = 0,
  YGG_EARLY_STOPPING_MIN_LOSS_FINAL = 1, /* MIN_VALIDATION_LOSS_ON_FULL_MODEL: train every tree, keep the best prefix */
  YGG_EARLY_STOPPING_LOSS_INCREASE = 2   /* VALIDATION_LOSS_INCREASE: stop when the best loss is look_ahead trees old */
};

/* One tree node, flat.  Trees are emitted in the reference's serialization order
 * (model/decision_tree/decision_tree.cc:609-646): node, negative subtree, positive subtree.
 * Mirrors proto::Node + proto::NodeCondition (model/decision_tree/decision_tree.proto). */
enum ygg_feature_type {
  YGG_FEATURE_DISCRETIZED_NUMERICAL = 0, /* condition: bin >= threshold_bin */
  YGG_FEATURE_CATEGORICAL = 1,           /* condition: category in cat_mask (CART); a wide categorical column's set
                                            is read with ygg_gbt_get_category_set */
  YGG_FEATURE_NUMERICAL = 2              /* presorted numerical column (ygg_dataset_set_numerical_column): condition
                                            value >= threshold_value (threshold_bin = -1), a missing value -> na_value */
};

typedef struct ygg_node {
  int32_t feature;          /* NodeCondition.attribute (dataset feature index); -1 for a leaf */
  int32_t threshold_bin;    /* Condition.DiscretizedHigher.threshold: bin >= threshold => positive
                               (0 for a categorical condition) */
  int32_t na_value;         /* NodeCondition.na_value */
  int32_t depth;            /* root = 1 */
  int32_t neg_child;        /* index in the emitted array, -1 for a leaf */
  int32_t pos_child;
  float split_score;        /* NodeCondition.split_score */
  float leaf_value;         /* NodeRegressorOutput.top_value (set on every node, as the reference does) */
  int64_t num_examples;     /* num_training_examples_without_weight of the node */
  int64_t num_pos_examples; /* num_pos_training_examples_without_weight of the split */
  /* Label statistics saved in the node (loss_utils.cc:109-117):
   *   variance gain: stat[0]=sum, stat[1]=sum_squares, stat[2]=count
   *   hessian gain : stat[0]=sum_gradients, stat[1]=sum_hessians (floored at 1e-3), stat[2]=sum_weights */
  double stat[3];
  /* Categorical condition (Condition.ContainsVector / ContainsBitmap,
   * learner/decision_tree/utils.cc:31-63): bit c set => category c goes to the positive child. */
  int32_t condition_type;   /* enum ygg_feature_type of the split feature; 0 for a leaf */
  float threshold_value;    /* Condition.Higher.threshold of the EXACT numerical splitter for features with bucket values
                               (ygg_dataset_set_bucket_values); NaN otherwise (discretized rule: threshold_bin only) */
  uint32_t cat_mask[8];
} ygg_node;

typedef struct ygg_dataset ygg_dataset;
typedef struct ygg_gbt ygg_gbt;

/* ---- library ------------------------------------------------------------------------- */
int ygg_abi_version(void);
const char* ygg_last_error(void);
/* Number of visible CUDA devices (0 if none; never fails). */
int ygg_device_count(void);

/* ---- dataset: the engine's input contract ----------------------------------------------
 * Replaces dataset::VerticalDataset with DISCRETIZED_NUMERICAL columns
 * (dataset/vertical_dataset.h:377-378) as consumed by
 * FeatureDiscretizedNumericalBucket::Filler (learner/decision_tree/splitter_accumulator.h:253-338).
 *  bins        : column-major, bins[f * column_stride + r], one byte per value, value < num_bins[f].
 *                The reference stores uint16 with 65535 = missing; here missing values are
 *                already folded into na_bin[f], which is what GetBucketIndex
 *                (splitter_accumulator.h:288-299) and EvalConditionDiscretizedHigher
 *                (model/decision_tree/decision_tree.cc:724-743, with na_value = na_bin >= threshold)
 *                do with them.
 *  num_bins[f] : boundaries_size()+1, 2..256.
 *  na_bin[f]   : NumericalToDiscretizedNumerical(column mean) (training.cc:917-922).
 * Categorical columns (dataset/vertical_dataset.h:416; ygg_dataset_set_feature_types) use the same
 * byte layout: value = integerised category (0 = out-of-dictionary), num_bins[f] =
 * number_of_unique_values <= 256, na_bin[f] = most_frequent_value (the NA replacement,
 * training.cc:3262-3314); they are split with the CART rule (buckets sorted by label mean /
 * hessian priority, then scanned).  Columns with 257..65535 categories are wide categorical columns
 * (ygg_dataset_set_wide_categorical_column), also split with CART: the engine has no random-mask algorithm
 * (decision_tree.proto:573-576), which is the learner's business (categorical_arity_limit_for_random).
 *  device      : CUDA ordinal this handle lives on (one process per GPU).
 */
int ygg_dataset_create(ygg_dataset** out, int64_t n_rows, int32_t n_features,
                       const uint8_t* bins, int64_t column_stride,
                       const int32_t* num_bins, const int32_t* na_bin, int32_t device);
/* feature_types[f]: enum ygg_feature_type (default: all DISCRETIZED_NUMERICAL). */
int ygg_dataset_set_feature_types(ygg_dataset* ds, const int32_t* feature_types, int32_t n_features);
/* Exact numerical splits through lossless buckets (one bucket per distinct value, DESIGN.md §14): `values[b]` = the value
 * of bucket b of `feature` (ascending, n = its number of bins).  For such a feature the engine places thresholds like the
 * reference's exact splitter: the middle of the two values PRESENT in the node around the cut
 * (FeatureNumericalBucket::Filler::SetConditionFinal, splitter_accumulator.h:213-232; MidThreshold, utils.h:103-109)
 * instead of the middle of the empty buckets (bucket interpolation) — the same partition of the training rows, the
 * reference's side for a held-out value inside the gap — and reports the float threshold in ygg_node.threshold_value.
 * `na_replacement` = the column mean the exact splitter imputes missing values with: na_value = na_replacement >= threshold
 * (splitter_accumulator.h:218). */
int ygg_dataset_set_bucket_values(ygg_dataset* ds, int32_t feature, const float* values, int32_t n, float na_replacement);
/* Wide numerical column (DESIGN.md §20): a numerical feature with num_bins = 257..65535 buckets, one per distinct value
 * (the column mean is one more when it has missing values), that the byte columns cannot hold.  codes[r] < num_bins is the
 * bucket of row r (missing values already folded into na_bin); values[b] = the value of bucket b (finite, strictly
 * ascending); na_replacement = the column mean.  Such a feature is always split with the exact threshold rule of
 * ygg_dataset_set_bucket_values: ygg_node.threshold_bin is a bucket index (compare it with the code), threshold_value the
 * float threshold.  The feature's byte column becomes a one-bucket filler that the byte kernels never split on.  Call
 * before ygg_gbt_create; single GPU only (the shard setters return YGG_ERR_UNIMPLEMENTED on such a dataset).  Training
 * and validation / prediction datasets must have the same wide features and buckets. */
int ygg_dataset_set_wide_column(ygg_dataset* ds, int32_t feature, const uint16_t* codes, int64_t n, int32_t num_bins, int32_t na_bin,
                                const float* values, float na_replacement);
/* Wide categorical column (DESIGN.md §21): a feature already set to YGG_FEATURE_CATEGORICAL with num_bins = 257..65535
 * categories (number_of_unique_values), codes[r] < num_bins the category of row r (missing values already folded into
 * na_bin = most_frequent_value).  Split with CART like a byte categorical column; the positive set of such a split is
 * read with ygg_gbt_get_category_set (its ygg_node.cat_mask is zero).  Same rules as ygg_dataset_set_wide_column: before
 * ygg_gbt_create, single GPU, validation / prediction datasets with the same wide columns. */
int ygg_dataset_set_wide_categorical_column(ygg_dataset* ds, int32_t feature, const uint16_t* codes, int64_t n, int32_t num_bins,
                                            int32_t na_bin);
/* Read-back of a wide column: codes[n_rows], and (may be NULL) its num_bins / na_bin. */
int ygg_dataset_get_wide_column(const ygg_dataset* ds, int32_t feature, uint16_t* codes, int32_t* num_bins, int32_t* na_bin);
/* Presorted numerical column (DESIGN.md §22): a numerical feature stored as its float values, with no limit on its
 * distinct values.  It is split by the reference's exact numerical splitter (ScanSplitsPresortedSparse,
 * splitter_scanner.h:1232-1430) through per-level lists of its rows sorted by value, never histogrammed.  values[r] is
 * row r's value, NaN = missing; the engine stores a missing value as `na_replacement` (the column mean the exact
 * splitter imputes, training.cc:2385-2392) and -0.0 as +0.0.  A split on it has condition_type YGG_FEATURE_NUMERICAL,
 * threshold_bin = -1 and threshold_value = the float threshold: value >= threshold_value goes to the positive child,
 * na_value = na_replacement >= threshold_value.  The feature becomes YGG_FEATURE_NUMERICAL and its byte column a
 * one-bucket filler.  INVALID_ARGUMENT for +-inf values, a non-finite na_replacement, a wrong row count, a categorical,
 * wide or already numerical feature, or a call after ygg_gbt_create on the dataset.  Single GPU only (the shard setters
 * return YGG_ERR_UNIMPLEMENTED); validation / prediction datasets must have the same numerical features. */
int ygg_dataset_set_numerical_column(ygg_dataset* ds, int32_t feature, const float* values, int64_t n, float na_replacement);
/* Read-back of a presorted numerical column as stored: values[n_rows] (missing values replaced). */
int ygg_dataset_get_numerical_column(const ygg_dataset* ds, int32_t feature, float* values);
/* Releases the dataset; while ygg_gbt handles still use it, the release waits for the last of them to be destroyed. */
int ygg_dataset_destroy(ygg_dataset* ds);
int64_t ygg_dataset_num_rows(const ygg_dataset* ds);
int32_t ygg_dataset_num_features(const ygg_dataset* ds);

/* ---- learner -----------------------------------------------------------------------------
 * Replaces GradientBoostedTreesLearner::TrainWithStatusImpl
 * (learner/gradient_boosted_trees/gradient_boosted_trees.cc:1154-1732) for configurations
 * whose features are all DISCRETIZED_NUMERICAL. */
void ygg_gbt_config_init(ygg_gbt_config* cfg);
int ygg_gbt_create(ygg_gbt** out, ygg_dataset* ds, const ygg_gbt_config* cfg);
int ygg_gbt_destroy(ygg_gbt* h);

/* Labels.  i32: integerised categorical label as the reference stores it (1 = negative,
 * 2 = positive; loss_imp_binomial.cc:133).  f32: regression target.  INVALID_ARGUMENT after ygg_gbt_set_row_shard*: a
 * row shard holds the job's initial prediction, which this rank's labels would replace. */
int ygg_gbt_set_labels_i32(ygg_gbt* h, const int32_t* labels, int64_t n);
int ygg_gbt_set_labels_f32(ygg_gbt* h, const float* labels, int64_t n);

/* Example weights (TrainingConfig.weight_definition -> dataset::GetWeights, learner/abstract_learner.cc; consumed as the
 * `weights` spans of InitialPredictions / Loss (loss_imp_binomial.cc:65-99, :204-234; loss_imp_mean_square_error.cc:56-88;
 * metric/metric.cc:2097-2115), of the bucket filler (LabelNumericalBucket<weighted=true>, splitter_accumulator.h:1552-1560)
 * and of SetLeafValueWithNewtonRaphsonStep<true> (loss_utils.cc:81-89)).  One non-negative float per training row, host
 * memory; call BEFORE ygg_gbt_set_labels_* (the initial predictions are weighted).  min_examples keeps counting rows.
 * Row shards: every rank passes its rows' weights (before ygg_gbt_set_row_shard*, which reduces the scales and the weight sum).
 * YGG_ERR_UNIMPLEMENTED with use_hessian_gain (the reference's weighted hessian filler sums UNWEIGHTED gradients into the buckets
 * it compares with a WEIGHTED parent, splitter_accumulator.h:1806-1814: neither reproduced nor silently corrected). */
int ygg_gbt_set_weights_f32(ygg_gbt* h, const float* weights, int64_t n);

/* ---- validation rows and early stopping (SURVEY.md §8f N2) ------------------------------------
 * The reference holds out validation rows before training (ExtractValidationDataset,
 * gradient_boosted_trees.cc:2718-2746: row r trains iff uniform_real_distribution<float>(mt19937(seed)) >
 * ratio, the first use of the learner's random engine), evaluates the loss on them after every
 * iteration (:1610-1626), feeds EarlyStopping (early_stopping/early_stopping.cc:30-62) and finally
 * truncates the model to the best number of trees (FinalizeModelWithValidationDataset, :212-272).
 * Here: ygg_validation_split_mask reproduces the row draw (libstdc++ semantics), ygg_dataset_split_rows
 * gathers the two row sets on the device, ygg_gbt_set_validation_* attaches the held-out rows (same
 * features and binning as the training dataset).  ygg_gbt_train then applies cfg.early_stopping;
 * afterwards ygg_gbt_num_trees is the truncated model size and ygg_gbt_num_iterations the number of
 * iterations that have log entries (training stopped there).  Not combined with sharding: YGG_ERR_UNIMPLEMENTED in
 * either call order (ygg_gbt_set_validation_* on a sharded handle, or a shard setter with world > 1 on a handle with
 * validation rows), since every rank would evaluate and stop on its own. */
int ygg_validation_split_mask(uint32_t random_seed, int64_t n_rows, float validation_ratio,
                              uint8_t* out_in_training /* [n_rows] 1 = training row */);
int ygg_dataset_split_rows(const ygg_dataset* ds, const uint8_t* select, ygg_dataset** selected,
                           ygg_dataset** rest);
int ygg_gbt_set_validation_i32(ygg_gbt* h, const ygg_dataset* valid, const int32_t* labels, int64_t n);
int ygg_gbt_set_validation_f32(ygg_gbt* h, const ygg_dataset* valid, const float* labels, int64_t n);
/* Weights of the validation rows (the hold-out is cut from the weighted dataset, gradient_boosted_trees.cc:1262-1280):
 * validation loss and accuracy become weighted.  After ygg_gbt_set_validation_*, before training. */
int ygg_gbt_set_validation_weights_f32(ygg_gbt* h, const float* weights, int64_t n);
/* Validation loss / secondary metric after iteration `iter` (TrainingLogs.Entry.validation_loss); `iter` below
 * ygg_gbt_num_iterations (early stopping trains whole batches: the iterations past the stop have no entry). */
int ygg_gbt_validation_loss(ygg_gbt* h, int32_t iter, float* loss, float* secondary);
/* Iterations with log entries; > ygg_gbt_num_trees when the model was truncated. */
int32_t ygg_gbt_num_iterations(const ygg_gbt* h);
/* Header.validation_loss and Header.early_stopping_triggered of the final model. */
int ygg_gbt_final_validation(ygg_gbt* h, float* validation_loss, int32_t* early_stopping_triggered);

/* Feature sharding across the GPUs of one box (SURVEY.md §8e; the reference's model is
 * distributed_decision_tree: workers own feature subsets).  This rank histograms and scans
 * features [feature_begin, feature_end) only; all ranks hold all columns so the row partition
 * is local.  `exchange` is called once per tree level with this rank's packed best-split
 * records (device pointer, `bytes` bytes) and must all-gather them into `recv` (device pointer,
 * world*bytes) on `stream` (a cudaStream_t) — NCCL in production, see INTEGRATION.md.
 * Refused up front: wide and presorted columns, candidate feature sampling, DART, candidate_shuffle and (world > 1)
 * validation rows; the multinomial loss, subsample < 1 and GOSS by the first ygg_gbt_step, before any collective. */
typedef int (*ygg_allgather_fn)(void* ctx, const void* send, void* recv, int64_t bytes,
                                void* stream);
int ygg_gbt_set_feature_shard(ygg_gbt* h, int32_t feature_begin, int32_t feature_end,
                              int32_t rank, int32_t world, ygg_allgather_fn exchange, void* ctx);

/* Row sharding (data parallel): this rank holds n_rows of n_rows_global rows of ALL features.  Per
 * tree level the engine fills its local integer histograms and calls `allreduce` ONCE on the level
 * buffer (sum, u64) — the "NCCL all-reduce of per-node histograms"; integer sums make the result
 * exact and independent of the reduction order, so trees are identical for any world size.  Child
 * statistics ride in the same buffer.  `allreduce(ctx, buf, count, dtype, op, stream)` must reduce
 * `count` elements in place on `stream`: dtype 0 = u32, 1 = u64, 2 = f64; op 0 = sum, 1 = max.
 * Call after ygg_gbt_set_labels_* (labels set afterwards are refused); `initial_prediction` is the job-wide value (the
 * harness owns the global label statistics, loss_imp_binomial.cc:65-99).  Every rank holds at least one row:
 * ygg_dataset_create refuses an empty dataset with INVALID_ARGUMENT, so a rank without rows is refused before it has a
 * handle or calls a collective; give each rank at least one row, or use fewer ranks.  Ranks may hold any other
 * uneven share, down to one row.  Refused up front, before any collective, like the feature shard: wide and presorted
 * columns, candidate feature sampling, DART, candidate_shuffle and validation rows.  The multinomial loss, subsample < 1
 * and GOSS are refused (YGG_ERR_UNIMPLEMENTED) by the first ygg_gbt_step, before that iteration's first collective. */
typedef int (*ygg_allreduce_fn)(void* ctx, void* buf, int64_t count, int32_t dtype, int32_t op, void* stream);
int ygg_gbt_set_row_shard(ygg_gbt* h, int32_t rank, int32_t world, int64_t n_rows_global,
                          float initial_prediction, ygg_allreduce_fn allreduce, void* ctx);

/* Row sharding with a reduce-scatter: the level buffer is cut into `world` chunks by feature
 * (chunk r = features [r*c, (r+1)*c), c = ceil(F / world), plus a copy of the node statistics), ONE
 * reduce-scatter per level gives rank r the summed histograms of its features only, every rank scans its
 * chunk and the best splits are all-gathered like in feature sharding (<= 3.5 KB): half the collective
 * bytes of the all-reduce and no replicated scan.  `reducescatter(ctx, buf, count_per_rank, dtype, op,
 * stream)` reduces world*count_per_rank elements in place, rank r's result at buf + r*count_per_rank;
 * `allreduce` is still used for a few scalars per iteration.  INVALID_ARGUMENT, before any collective, when
 * world > num_features or the features do not cut into `world` non-empty chunks ((world - 1) * c >= F). */
typedef int (*ygg_reducescatter_fn)(void* ctx, void* buf, int64_t count_per_rank, int32_t dtype, int32_t op,
                                    void* stream);
int ygg_gbt_set_row_shard_scatter(ygg_gbt* h, int32_t rank, int32_t world, int64_t n_rows_global,
                                  float initial_prediction, ygg_allreduce_fn allreduce,
                                  ygg_reducescatter_fn reducescatter, ygg_allgather_fn allgather, void* ctx);

/* Contiguous feature range of `rank` (the shard layout every rank must agree on). */
int ygg_feature_shard(int32_t n_features, int32_t rank, int32_t world, int32_t* begin, int32_t* end);

/* The record exchanged per (level, node): this rank's best split over its features. */
typedef struct ygg_shard_best {
  float score;      /* split_score as float; only meaningful if feature >= 0 */
  int32_t feature;  /* global feature index, -1 = no valid split in this shard */
  int32_t threshold_bin;
  int32_t num_pos_examples;
  int32_t condition_type; /* ygg_feature_type of `feature` */
  int32_t na_value;       /* categorical splits: 1 if the NA replacement category is positive */
  uint32_t cat_mask[8];   /* categorical splits: positive categories */
} ygg_shard_best;
/* Host restatement of the on-device merge (records: [world][nodes], out: [nodes]): the first strictly
 * greater float score in rank order, i.e. the ordered consumption of
 * FindBestConditionConcurrentManager (learner/decision_tree/training.cc:1728-1746). */
int ygg_merge_shard_best(const ygg_shard_best* records, int32_t world, int32_t nodes, ygg_shard_best* out);

/* loss->InitialPredictions (loss_imp_binomial.cc:65-99, loss_imp_mean_square_error.cc:56-88). */
int ygg_gbt_initial_prediction(ygg_gbt* h, float* out);

/* Runs `num_iters` boosting iterations (gradient_boosted_trees.cc:1428-1571).  `stop_flag`
 * (may be NULL) is polled between iterations like stop_training_trigger
 * (gradient_boosted_trees.cc:1430-1433). */
int ygg_gbt_train(ygg_gbt* h, int32_t num_iters, const volatile int32_t* stop_flag);
/* One iteration, asynchronous on the handle's stream; ygg_gbt_sync waits for it. */
int ygg_gbt_step(ygg_gbt* h);
int ygg_gbt_sync(ygg_gbt* h);

/* `num_iters` iterations (including the final prediction update) bracketed by CUDA events on the
 * handle's stream; *device_ms receives the elapsed device time, *kernel_launches (may be NULL)
 * the number of kernels this library launched in between.  Used by bench.py. */
int ygg_gbt_train_timed(ygg_gbt* h, int32_t num_iters, double* device_ms, int64_t* kernel_launches);

int32_t ygg_gbt_num_trees(const ygg_gbt* h);
/* Best-split exchange over peer memory instead of the all-gather callback (feature shards and row shards with the
 * reduce-scatter layout): `peer_windows[r]` = this process's mapping of rank r's window of
 * ygg_gbt_best_split_window_bytes(h) zeroed bytes (ygg_comm_window_create of ygg_b200_comm.h).  k_select_global then
 * stores this rank's ShardBest records of a level straight into every rank's window over NVLink, publishes an epoch
 * flag and waits for the other ranks' flags in its own window: no collective call, no extra kernel per level. */
int64_t ygg_gbt_best_split_window_bytes(const ygg_gbt* h);
int ygg_gbt_set_best_split_window(ygg_gbt* h, void* const* peer_windows, int32_t world);

/* Tie-break replay (cfg.candidate_shuffle != 0; GetCandidateAttributes, training.cc:4293-4306): resolves the ties of
 * every tree trained so far and reports how many tied nodes were given the reference's feature (`renamed`) and how many
 * could not be (`unresolved`: the tied candidates cut the node's rows differently, or more than 3 features tied). */
int ygg_gbt_tie_stats(ygg_gbt* h, int64_t* renamed, int64_t* unresolved);
/* Positions the tie-break stream `words` engine words after the seed: for callers of ygg_tree_train_on_gradients (the
 * decision_tree::Train seam), whose trees are not grown in the handle's own boosting loop. */
int ygg_gbt_set_tie_rng_position(ygg_gbt* h, uint64_t words);

/* Candidate feature sampling (DecisionTreeTrainingConfig.num_candidate_attributes / num_candidate_attributes_ratio,
 * decision_tree.proto; DESIGN.md §23): each node is split on the best of a random subset of the features.
 *
 * k, the number of features to test (NumAttributesToTest, training.cc:4244-4289), for F features:
 *   k = ceil(ratio * F) if ratio >= 0 (the product in float arithmetic), else num_candidate_attributes;  k == 0 -> ceil(sqrt(F)) for the binomial and
 *   multinomial losses, ceil(F / 3) for squared error;  k == -1 -> F;  then k = min(k, F).
 * ygg_num_candidate_attributes computes it; INVALID_ARGUMENT for num_candidate_attributes < -1, a ratio above 1 or NaN
 * (a negative ratio means "not set"), F < 1 or an unknown loss.
 *
 * Candidate order: the features of node `node` (its index in the handle's node table of the tree) of tree `tree` (the
 * index ygg_gbt_get_tree takes: iteration * K + class) are ordered by ascending (key, feature) with
 *   mix(z)  = SplitMix64's finalizer: z += 0x9E3779B97F4A7C15; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;
 *             z = (z ^ (z >> 27)) * 0x94D049BB133111EB; return z ^ (z >> 31)      (all modulo 2^64)
 *   key     = mix(mix(mix(mix(random_seed) ^ (uint32)tree) ^ (uint32)node) ^ (uint32)feature)
 * (ygg_candidate_key).  The order depends on the node alone, not on the order in which nodes are searched, so it draws
 * nothing from the learner's random stream (row sampling and GOSS are unaffected) and works with every growth strategy.
 *
 * Selection: features are taken in that order until k of them (k + 1 with split_jobs_draw_seeds = 0, the reference's
 * single-thread manager, training.cc:1407) are valid — the scan scored at least one of their boundaries: two non-empty
 * sides of at least min_examples rows (with in_split_min_examples_check), with or without example weight — or every
 * feature is taken; the node's split is
 * the first maximum, by float score, of the taken features in that order.
 *
 * ygg_gbt_set_candidate_sampling: after ygg_gbt_create, before the first tree; k >= F keeps the unsampled selection (and
 * the tie-break replay).  With k < F: YGG_ERR_UNIMPLEMENTED on a feature or row shard (either call order: the shard
 * setters refuse a sampling handle), INVALID_ARGUMENT with candidate_shuffle != 0 (the keys define the order). */
int ygg_num_candidate_attributes(int32_t num_features, int32_t loss, int32_t num_candidate_attributes,
                                 float num_candidate_attributes_ratio, int32_t* k);
uint64_t ygg_candidate_key(uint32_t random_seed, int32_t tree, int32_t node, int32_t feature);
int ygg_gbt_set_candidate_sampling(ygg_gbt* h, int32_t num_candidate_attributes, float num_candidate_attributes_ratio);

/* DART (GradientBoostedTreesTrainingConfig.dart, DESIGN.md §24): at the start of iteration i > 0 every earlier iteration
 * is dropped with probability dropout_rate (one draw each from the learner's random stream; none dropped: one drawn
 * uniformly), the iteration's gradients are taken at the predictions without the dropped trees, and after its trees the
 * new iteration gets weight 1 / (|D| + 1) while the dropped ones are scaled by |D| / (|D| + 1).  Under DART the reference
 * defaults shrinkage to 1.0 when it is not set; this ABI takes cfg.shrinkage as given.
 *
 * ygg_gbt_set_dart: after ygg_gbt_create, before the first tree.  INVALID_ARGUMENT for a NaN rate, one outside [0, 1], or
 * after the first tree; YGG_ERR_UNIMPLEMENTED on a feature or row shard (either call order: the shard setters refuse a
 * DART handle), and from ygg_gbt_set_predictions.  A ygg_gbt_step that fails after its DART draws leaves the handle unable
 * to train further (the next step returns INVALID_ARGUMENT); its trees and model so far stay readable.  Allocates the leaf-id history of every tree: tree capacity x rows x 2
 * bytes for the training rows (10M rows, 300 trees: 6 GB) and the same for the held-out rows; a failed allocation returns
 * YGG_ERR_CUDA with the byte count.
 *
 * ygg_gbt_get_tree returns the trees as grown (unscaled leaves).  ygg_gbt_predict and ygg_gbt_save_ydf use the SCALED
 * model: each leaf of iteration j becomes leaf * w_j (internal nodes unchanged), summed in tree order.
 * ygg_gbt_get_predictions returns the training accumulator: the same model, but built by the per-iteration updates, so
 * it is not bitwise equal to the scaled model's sum (the operations are in another order).
 *
 * ygg_gbt_get_dart_weights: the per-iteration weights w_j, one per iteration; after ygg_gbt_train they are the final
 * model's (early stopping: the weights at the stop, for the iterations the model keeps).  ygg_gbt_get_dart_dropped: the
 * dropped iterations of iteration `iter`, ascending. */
int ygg_gbt_set_dart(ygg_gbt* h, float dropout_rate);
int ygg_gbt_get_dart_weights(ygg_gbt* h, float* out, int32_t capacity, int32_t* n);
int ygg_gbt_get_dart_dropped(ygg_gbt* h, int32_t iter, int32_t* out, int32_t capacity, int32_t* n);

/* Copies tree `iter` (pre-order: node, neg subtree, pos subtree).  *n_nodes receives the node
 * count; fails with INVALID_ARGUMENT if capacity is too small. */
int ygg_gbt_get_tree(ygg_gbt* h, int32_t iter, ygg_node* out, int32_t capacity, int32_t* n_nodes);
/* The positive set of categorical split `node` (pre-order index, as in ygg_gbt_get_tree) of tree `iter` (-1: the tree
 * the last ygg_tree_train_on_gradients call returned): bit c of
 * words[c / 32] set => category c goes to the positive child.  *n_words = ceil(num_bins / 32) for a wide categorical
 * column, 8 (cat_mask) for a byte one; fails with INVALID_ARGUMENT if capacity is smaller or the node is not a
 * categorical split. */
int ygg_gbt_get_category_set(ygg_gbt* h, int32_t iter, int32_t node, uint32_t* words, int32_t capacity, int32_t* n_words);
/* Training loss / secondary metric after iteration `iter` (loss->Loss,
 * gradient_boosted_trees.cc:1575-1580): binomial => (2x mean log-loss, accuracy);
 * squared error => (rmse, rmse).  `iter` below ygg_gbt_num_iterations. */
int ygg_gbt_train_loss(ygg_gbt* h, int32_t iter, float* loss, float* secondary);
/* Current raw predictions (logits / regression values), N floats to host. */
int ygg_gbt_get_predictions(ygg_gbt* h, float* out, int64_t n);
/* Raw scores (before the loss' activation) of the trained model — the trees kept after early stopping — on ANY dataset that
 * has the training dataset's features and binning: out[k * n_rows + r], k < classes (1 unless multinomial).  The device
 * counterpart of ComputePredictions (gradient_boosted_trees.cc:2872-2930), e.g. to resume training from a model
 * (ygg_gbt_set_predictions) or to evaluate a test fold without leaving the GPU. */
int ygg_gbt_predict(ygg_gbt* h, const ygg_dataset* ds, float* out, int64_t n);

/* Overwrites the current predictions (warm start from another model; also the teacher-forcing hook of the parity tests). */
int ygg_gbt_set_predictions(ygg_gbt* h, const float* pred, int64_t n);

/* decision_tree::Train seam (learner/decision_tree/training.h:1012-1021): grows ONE regression
 * tree on caller-provided per-example gradients / hessians (host pointers) with the handle's
 * tree hyper-parameters; does not touch the boosting state.  The positive sets of its splits on wide categorical
 * columns are read with ygg_gbt_get_category_set(h, -1, ...). */
int ygg_tree_train_on_gradients(ygg_gbt* h, const float* gradients, const float* hessians,
                                ygg_node* out, int32_t capacity, int32_t* n_nodes);

/* Level-histogram seam (FillExampleBucketSet, learner/decision_tree/splitter_scanner.h:859-909): the histogram phase of
 * one tree level, run by the same code as training, on caller-chosen gradients and slots. */
enum ygg_hist_mode {
  YGG_HIST_ROOT_SUM = 0,  /* k_hist, root layout: no count atomics, counts from the precomputed root count histogram */
  YGG_HIST_PACKED = 1,    /* k_hist, packed count | coarse-sum words (no bin may take more than 8191 rows per work item) */
  YGG_HIST_SHARED = 2,    /* k_hist, count | carries words (any data; the only layout with a second plane) */
  YGG_HIST_HIST2 = 3,     /* k_hist2: its root variant at level 0, its packed variant below */
  YGG_HIST_SEGMENTED = 4, /* k_hist_seg: packed words, one slot per work item, rows gathered from a row-major copy (level >= 1) */
};
typedef struct ygg_hist_plan {  /* one level's k_hist / k_hist2 / k_hist_seg launch */
  int32_t mode;            /* enum ygg_hist_mode */
  int32_t group;           /* features per work item G (k_hist, 1..8), or feature lanes FL (k_hist2, k_hist_seg: 8, 16, 32;
                              k_hist_seg at 32 lanes over more than 32 features takes two adjacent features per lane) */
  int32_t hist2_tiles;     /* sub-tiles of 1024 rows per tile T (k_hist2 only: 1, 2) */
  int32_t chunk_blocks;    /* 8192-row blocks per work item, 1..127 */
  int32_t slot_window;     /* 0: one pass over every slot; else slots per pass (multi-pass k_hist + one dummy slot) */
  int32_t grid;            /* CTAs */
} ygg_hist_plan;
/* The launch the handle runs at tree level `level` (0 <= level < max_depth - 1). */
int ygg_debug_hist_plan(const ygg_gbt* h, int32_t level, ygg_hist_plan* out);
/* Accumulates the histograms of `n_slots` slots (1..254) at tree level `level`: row r goes to slot slot_of_row[r] (-1: none).
 * `gradients` (and `second`: the hessians, or the example weights on a weighted handle; exactly when the handle keeps a
 * second histogram plane, else NULL) are host arrays of one float per row, quantised as the training loop does: g to
 * q = clamp(rint(g * 2^23 / P) + 2^23, 0, 2^24 - 1) with P the smallest power of two >= max|g| (1 if all are zero), the
 * second plane to min(rint(v * 2^24 / V), 2^24) with V the handle's power of two of that plane.  `plan` NULL: the
 * handle's own plan of the level; an explicit plan uses n_slots shared-memory slots (slot_window + 1 with a window).
 * Outputs, [n_slots][features histogrammed by this handle][256]: out_sum the raw sums of q, out_cnt the row counts,
 * out_second the raw sums of the second plane (NULL without one); out_scales = {P, V} (V = 0 without a second plane).
 * Refuses (INVALID_ARGUMENT, before any launch) a plan the kernels cannot run exactly: shared memory over budget, too
 * many slots for one pass, the root layouts anywhere but at an unsampled level 0 with every row in slot 0, k_hist2 with
 * more than 2 slots, k_hist_seg at level 0 or with a slot window, a layout other than the shared one with a second plane, or a packed layout (k_hist_seg's included) whose chunk lets a bin
 * of some feature receive more than 8191 rows (or is not a whole number of the 8-block sub-chunks above 4M rows).  Only scratch that every training iteration rewrites is overwritten. */
int ygg_debug_level_histogram(ygg_gbt* h, int32_t level, const ygg_hist_plan* plan, const float* gradients,
                              const float* second, const int32_t* slot_of_row, int32_t n_slots, uint64_t* out_sum,
                              uint32_t* out_cnt, uint64_t* out_second, float* out_scales);

/* The wide columns' histograms of the last histogram phase run on the handle (a training level, or
 * ygg_debug_level_histogram, which accumulates them too): [n_slots][sum over the wide features of num_bins] raw sums of q,
 * row counts and (exactly when the handle keeps one, else NULL) second-plane sums; the buckets of the wide features
 * follow each other in the order they were set. */
int ygg_debug_wide_histogram(ygg_gbt* h, int32_t n_slots, uint64_t* out_sum, uint32_t* out_cnt, uint64_t* out_second);

/* Split-candidate capture of the level loop.  enabled != 0: every tree the handle grows afterwards copies, at each level,
 * the complete candidate table left by the scan phase (every node of the level x every feature the handle scans, with the
 * wide and presorted columns' float thresholds and wide categorical positive sets) into buffers allocated here, before the
 * selection; the copies are asynchronous.  enabled == 0 frees them: the level loop is then exactly as without capture. */
int ygg_debug_capture_candidates(ygg_gbt* h, int32_t enabled);
typedef struct ygg_level_node {
  int32_t node;            /* pre-order index in the emitted tree */
  int32_t candidate;       /* 1: the node was scanned (it may be split) */
  int32_t derived;         /* 1: its histogram was parent - sibling; 0: accumulated from its rows */
  int32_t reserved;
  int64_t num_examples;
} ygg_level_node;
typedef struct ygg_candidate {
  int32_t found;
  float score;
  int32_t threshold_bin;   /* thr_bin_of: bin >= threshold_bin is positive (1 for a presorted column) */
  int32_t lo, hi;          /* the exact threshold rule's buckets around the cut (byte columns with bucket values), else -1 */
  int32_t num_pos_examples;
  float threshold_value;   /* float threshold of an exact-rule, wide numerical or presorted candidate, else NaN */
  uint32_t cat_mask[8];    /* positive categories of a byte categorical candidate */
} ygg_candidate;
/* The capture of tree level `level` of the last tree grown with capture enabled (a ygg_tree_train_on_gradients tree,
 * level-wise growth, candidate_shuffle = 0).  nodes[capacity], cands[capacity][features scanned by this handle], sets
 * (or NULL) [capacity][wide features][set_words] of the wide categorical candidates; *n_nodes = the level's nodes;
 * scales = {P, the hessian plane's power of two, the weight plane's power of two}.  INVALID_ARGUMENT on a null handle or
 * output, a level outside the captured tree, a capacity below the level's nodes or no capture. */
int ygg_debug_level_candidates(ygg_gbt* h, int32_t level, int32_t capacity, ygg_level_node* nodes, ygg_candidate* cands,
                               uint32_t* sets, int32_t set_words, int32_t* n_nodes, float* scales);
/* The candidate feature sampling validity flags of the same capture (sampling set before the capture was enabled):
 * tried[capacity][features] = 1 when the scan scored at least one boundary of the (level node, feature) pair, 0 otherwise
 * and on nodes that were not scanned; *first_node = the node-table index of the level's first node (level node j is
 * node first_node + j of ygg_candidate_key).  INVALID_ARGUMENT as ygg_debug_level_candidates, or without sampling. */
int ygg_debug_level_tried(ygg_gbt* h, int32_t level, int32_t capacity, uint8_t* tried, int32_t* first_node, int32_t* n_nodes);

/* SplitExamplesInPlace seam (learner/decision_tree/training.cc:5243-5305 ->
 * model/decision_tree/decision_tree.cc:957-1012): stable two-way partition of a row-id list by
 * `bin(feature,row) >= threshold_bin`; positives then negatives, both ascending-stable.  YGG_ERR_UNIMPLEMENTED on a
 * presorted numerical feature (it has no bins).
 * rows_in/rows_out are host pointers of n entries; *n_pos receives the positive count. */
int ygg_partition_rows(ygg_dataset* ds, const uint32_t* rows_in, int64_t n, int32_t feature,
                       int32_t threshold_bin, uint32_t* rows_out, int64_t* n_pos);

/* Per-kernel device time of the last ygg_gbt_step/train call, in milliseconds, summed over
 * launches, measured with CUDA events on the handle's stream when profiling is enabled.
 * names: "grad", "hist", "scan", "select", "partition", "total"; with presorted numerical columns also "presort_scan"
 * (their scan, included in "scan") and "presort_partition" (their list partition, after "partition"). */
int ygg_gbt_set_profiling(ygg_gbt* h, int32_t enabled);
int ygg_gbt_get_profile(ygg_gbt* h, const char* name, double* ms, int64_t* launches);

/* model::SaveModel analogue (model/gradient_boosted_trees/gradient_boosted_trees.cc:111-139):
 * writes header.pb, data_spec.pb, gradient_boosted_trees_header.pb, nodes-00000-of-00001, done.
 * data_spec_pb / n: an already-serialised dataset::proto::DataSpecification (built by the host
 * harness, which owns column names and boundaries). */
int ygg_gbt_save_ydf(ygg_gbt* h, const char* directory, const char* label_name,
                     const uint8_t* data_spec_pb, int64_t data_spec_len, int32_t label_col_idx,
                     const int32_t* feature_col_idx);

#ifdef __cplusplus
}
#endif
#endif /* YGG_B200_H_ */
