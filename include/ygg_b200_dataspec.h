/*
 * ygg_b200_dataspec.h — host-side binning helpers of libygg_b200.so (no GPU needed).
 * They implement the rule that produces the engine's input contract (uint8 bins); the reference
 * does this inside dataspec inference and VerticalDataset population.
 */
#ifndef YGG_B200_DATASPEC_H_
#define YGG_B200_DATASPEC_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* GenDiscretizedBoundaries itself (dataset/data_spec.cc:854-986): candidates = strictly increasing
 * unique values with their counts; special values get a one-value bin (AddBucket, :77-107).
 * Pinned by the reference's known-answer tests dataset/data_spec_test.cc:567-684. */
int ygg_gen_discretized_boundaries(const float* values, const int64_t* counts, int64_t n_candidates,
                                   int32_t maximum_num_bins, int32_t min_obs_in_bins,
                                   const float* special_values, int32_t n_special, float* out_boundaries,
                                   int32_t capacity, int32_t* out_num_boundaries);

/* GenDiscretizedBoundaries (dataset/data_spec.cc:854-986) with the special values {0, mean}
 * (FinalizeComputeSpecDiscretizedNumerical, dataset/data_spec_inference.cc:226-250).
 * values: n floats, NaN = missing.  Writes the sorted boundaries (at most maximum_num_bins - 1)
 * and the column mean of the non-missing values.  Returns 0 or YGG_ERR_INVALID_ARGUMENT. */
int ygg_discretize_boundaries(const float* values, int64_t n, int32_t maximum_num_bins,
                              int32_t min_obs_in_bins, float* out_boundaries, int32_t capacity,
                              int32_t* out_num_boundaries, double* out_mean);

/* ygg_discretize_boundaries for maximum_num_bins in [2, 65535]: up to 65535 bins, for uint16 codes. */
int ygg_discretize_boundaries16(const float* values, int64_t n, int32_t maximum_num_bins,
                                int32_t min_obs_in_bins, float* out_boundaries, int32_t capacity,
                                int32_t* out_num_boundaries, double* out_mean);

/* NumericalToDiscretizedNumerical (dataset/data_spec.cc:1006-1018): bin = upper_bound(boundaries, x);
 * missing values are folded into na_bin (see ygg_dataset_create). */
int ygg_discretize_encode(const float* values, int64_t n, const float* boundaries,
                          int32_t num_boundaries, int32_t na_bin, uint8_t* out);

/* ---- on-GPU dataspec step (SURVEY.md §8f N1) --------------------------------------------------
 * Builds the device-resident dataset of ygg_b200.h column by column without materialising the uint8
 * matrix on the host.  A float32 column is uploaded, its boundaries are computed ON THE GPU with the
 * same rule as ygg_discretize_boundaries (radix sort -> distinct values and counts -> the greedy
 * quantile rule of GenDiscretizedBoundaries, dataset/data_spec.cc:854-986, special values {0, mean},
 * dataset/data_spec_inference.cc:226-250) and it is encoded in place
 * (NumericalToDiscretizedNumerical, dataset/data_spec.cc:1006-1018; NaN -> the bin of the mean,
 * learner/decision_tree/training.cc:917-922).  What PYDF does on the host in
 * port/python/ydf/dataset/dataset.cc:192-316.  Results are bit-identical to the host functions above.
 *   n_stats_rows : rows used for the boundaries and the mean (max_num_scanned_rows_to_compute_statistics;
 *                  <= 0 = all rows); every row is encoded.
 *   maximum_num_bins in [4, 256].  Outputs (each may be NULL): the boundaries, their number, the mean,
 *   the NA-replacement bin and the number of missing values among the statistics rows. */
typedef struct ygg_dataset_builder ygg_dataset_builder;
struct ygg_dataset;
int ygg_dataset_builder_create(ygg_dataset_builder** out, int64_t n_rows, int32_t n_features, int32_t device);
int ygg_dataset_builder_add_numerical(ygg_dataset_builder* b, int32_t feature, const float* values,
                                      int64_t n_stats_rows, int32_t maximum_num_bins, int32_t min_obs_in_bins,
                                      float* out_boundaries, int32_t capacity, int32_t* out_num_boundaries,
                                      double* out_mean, int32_t* out_na_bin, int64_t* out_num_missing);
/* The same in two steps, so that the upload of the next column overlaps the kernels of the previous
 * ones (three columns in flight): _async enqueues and returns at once — `values` must stay valid and
 * unchanged until the column is collected with _get_numerical or the builder is finished. */
int ygg_dataset_builder_add_numerical_async(ygg_dataset_builder* b, int32_t feature, const float* values,
                                            int64_t n_stats_rows, int32_t maximum_num_bins,
                                            int32_t min_obs_in_bins);
int ygg_dataset_builder_get_numerical(ygg_dataset_builder* b, int32_t feature, float* out_boundaries,
                                      int32_t capacity, int32_t* out_num_boundaries, double* out_mean,
                                      int32_t* out_na_bin, int64_t* out_num_missing);
/* The same rule for maximum_num_bins in [257, 65535] (DESIGN.md §25): the column becomes a discretized wide column
 * (ygg_dataset_set_wide_discretized_column) of uint16 codes when the builder is finished, or a byte column when its
 * boundaries leave at most 256 bins.  Collected with ygg_dataset_builder_get_numerical like the byte columns. */
int ygg_dataset_builder_add_numerical16_async(ygg_dataset_builder* b, int32_t feature, const float* values,
                                              int64_t n_stats_rows, int32_t maximum_num_bins,
                                              int32_t min_obs_in_bins);
/* A column that is already bucketised on the host (categorical dictionary indices, or bins made by
 * ygg_discretize_encode): n_rows bytes. */
int ygg_dataset_builder_add_bins(ygg_dataset_builder* b, int32_t feature, const uint8_t* bins, int32_t num_bins,
                                 int32_t na_bin, int32_t feature_type);
/* Every feature must have been added.  On success the builder is consumed and *out owns the dataset. */
int ygg_dataset_builder_finish(ygg_dataset_builder* b, struct ygg_dataset** out);
int ygg_dataset_builder_destroy(ygg_dataset_builder* b);
/* Copies the n_rows bins of one feature back to the host (tests, debugging). */
int ygg_dataset_get_bins(const struct ygg_dataset* ds, int32_t feature, uint8_t* out);

#ifdef __cplusplus
}
#endif
#endif /* YGG_B200_DATASPEC_H_ */
