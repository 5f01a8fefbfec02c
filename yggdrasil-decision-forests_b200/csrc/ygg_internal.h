// ygg_internal.h — declarations shared by the translation units of libygg_b200.so (not part of the ABI).
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

// Records `msg` as this thread's ygg_last_error() and returns `code`.
__attribute__((visibility("hidden"))) int ygg_set_error_msg(int code, const char* msg);

// Device-resident bucketised dataset (include/ygg_b200.h): bins[f][n_pad] uint8, column-major.
struct ygg_dataset {
  int device = 0;
  int64_t n = 0, n_pad = 0;
  int F = 0;
  uint8_t* d_bins = nullptr;
  uint32_t* d_bins4 = nullptr;   // interleaved copy [ceil(F/4)][n_pad] for k_hist2 (built on first use, ygg_hist2.cuh)
  uint8_t* d_bins_rows = nullptr;   // row-major copy [n_pad][F rounded up to 32] for k_hist_seg (built on first use, ygg_hist_seg.cuh)
  int32_t* d_num_bins = nullptr;
  int32_t* d_na_bin = nullptr;
  int32_t* d_feature_type = nullptr;
  float* d_bucket_values = nullptr;   // [F][256] exact threshold rule (ygg_dataset_set_bucket_values), allocated on first use
  int32_t* d_exact_rule = nullptr;    // [F]
  float* d_na_replacement = nullptr;  // [F] NumericalSpec.mean of the features under the exact rule
  std::vector<int32_t> num_bins, na_bin, feature_type;
  int num_sms = 0;
  // Wide numerical columns (ygg_dataset_set_wide_column, DESIGN.md §20): 257..65535 buckets, uint16 codes.  The feature's
  // byte column in d_bins holds a filler with num_bins[f] = 1, so the byte kernels never split on it.
  uint16_t* d_wide = nullptr;          // [wide features][n_pad] codes, in wide-index order
  int wide_cap = 0;                    // planes allocated in d_wide (>= wide features)
  int32_t* d_wide_of = nullptr;        // [F] wide index of a feature, -1 for a byte column
  int64_t* d_wide_off = nullptr;       // [wide features] offset of the feature's buckets in d_wide_values / the wide planes
  float* d_wide_values = nullptr;      // [sum of the wide features' buckets] bucket values (ascending per feature)
  // Wide categorical columns (ygg_dataset_set_wide_categorical_column, DESIGN.md §21) share these tables: wide_cat[w] = 1,
  // and their bucket values are zeros that nothing reads.  Discretized wide columns (ygg_dataset_set_wide_discretized_column,
  // DESIGN.md §25) too: wide_disc[w] = 1, split by the discretized threshold rule (NA rows: wide_na_bin[w] >= threshold).
  std::vector<int32_t> wide_of, wide_feature, wide_bins, wide_na_bin, wide_cat, wide_disc;
  std::vector<int64_t> wide_off;       // host copy of d_wide_off, plus the total at the end
  std::vector<float> wide_values, wide_na_replacement;
  int n_wide() const { return static_cast<int>(wide_feature.size()); }
  // 32-bit words of the widest categorical wide column's positive set (0 without one)
  int set_words() const {
    int m = 0;
    for (int w = 0; w < n_wide(); w++)
      if (wide_cat[w]) m = std::max(m, (wide_bins[w] + 31) / 32);
    return m;
  }
  // Presorted numerical columns (ygg_dataset_set_numerical_column, DESIGN.md §22): float values, NaN already replaced by
  // the column mean and -0.0 stored as +0.0.  feature_type[f] = YGG_FEATURE_NUMERICAL and the byte column is the same
  // one-bucket filler as a wide column's.
  float* d_num = nullptr;              // [numerical features][n_pad] values, in numerical-index order
  int32_t* d_num_of = nullptr;         // [F] numerical index of a feature, -1 otherwise
  std::vector<int32_t> num_of, num_feature;
  std::vector<float> num_na_replacement;
  int n_num() const { return static_cast<int>(num_feature.size()); }
  int handles = 0;                     // live ygg_gbt handles on this dataset (wide columns are set before the first)
  bool destroy_pending = false;        // ygg_dataset_destroy ran while handles were live: the last handle's destroy frees it
};

__attribute__((visibility("hidden"))) int ygg_internal_dataset_alloc(ygg_dataset** out, int64_t n_rows,
                                                                     int32_t n_features, int32_t device);
__attribute__((visibility("hidden"))) int ygg_internal_dataset_finalize(ygg_dataset* ds);
// Grows d_wide to hold at least `planes` code planes (one allocation for the columns that will be attached).
__attribute__((visibility("hidden"))) int ygg_internal_reserve_wide(ygg_dataset* ds, int planes);
// ygg_dataset_set_wide_discretized_column with the codes already on the device (the GPU binning step's output).
__attribute__((visibility("hidden"))) int ygg_internal_attach_wide_discretized(ygg_dataset* ds, int32_t feature,
                                                                              const uint16_t* d_codes, int32_t num_bins,
                                                                              int32_t na_bin);
