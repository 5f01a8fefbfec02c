// ygg_dataspec.cc — host-side binning rule of DISCRETIZED_NUMERICAL columns (the engine's input
// contract).  Follows the reference's rule so that thresholds mean the same thing:
//   GenDiscretizedBoundaries        dataset/data_spec.cc:854-986
//   AddBucket (special values)      dataset/data_spec.cc:77-107
//   FinalizeComputeSpecDiscretizedNumerical  dataset/data_spec_inference.cc:226-250
//   NumericalToDiscretizedNumerical dataset/data_spec.cc:1006-1018
// Written from the algorithm's description; storage and control flow are this repo's own.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <utility>
#include <vector>

#include "../../include/ygg_b200.h"
#include "../../include/ygg_b200_dataspec.h"

namespace {

// Inserts the one-value bin [v - ulp, v + ulp] for a special value.
void add_special_bucket(float v, std::vector<float>* bounds) {
  const float lo = std::nextafter(v, v - 1.f);
  const float hi = std::nextafter(v, v + 1.f);
  if (bounds->empty()) {
    bounds->push_back(lo);
    bounds->push_back(hi);
    return;
  }
  bounds->erase(std::remove_if(bounds->begin(), bounds->end(),
                               [lo, hi](float b) { return b >= lo && b <= hi; }),
                bounds->end());
  if (bounds->empty()) {  // every boundary was inside the special bucket (the reference reads min_element of an
                          // empty vector here, data_spec.cc:95-98: undefined; keep the one special bucket)
    bounds->push_back(lo);
    bounds->push_back(hi);
    return;
  }
  const float mn = *std::min_element(bounds->begin(), bounds->end());
  const float mx = *std::max_element(bounds->begin(), bounds->end());
  if (mn < hi) bounds->push_back(lo);
  if (mx > lo) bounds->push_back(hi);
}

// GenDiscretizedBoundaries proper: candidates = sorted unique values with counts.
int gen_boundaries(const std::vector<std::pair<float, int64_t>>& cand, int32_t maximum_num_bins, int32_t min_obs_in_bins,
                   const float* special, int n_special, std::vector<float>* out) {
  int in_bounds = 0;
  if (!cand.empty())
    for (int k = 0; k < n_special; k++)
      if (special[k] > cand.front().first && special[k] < cand.back().first) in_bounds++;
  // The reference evaluates max(1, maximum_num_bins - #special - in_bounds) in size_t: a negative value
  // wraps, the later "more candidates than bins" test is then false and every candidate gets its own
  // boundary (data_spec.cc:889-896; KAT data_spec_test.cc:640-645).
  const int64_t reserved = static_cast<int64_t>(maximum_num_bins) - n_special - in_bounds;
  const bool unlimited = reserved < 0;
  int64_t max_bins = std::max<int64_t>(1, reserved);
  const int64_t max_boundaries = max_bins - 1;
  std::vector<float>& bounds = *out;
  bounds.clear();
  const int64_t nc = static_cast<int64_t>(cand.size());
  if (!unlimited && nc > max_bins) {
    int64_t total = 0;
    for (auto& c : cand) total += c.second;
    max_bins = std::min<int64_t>(max_bins, total / min_obs_in_bins);
    if (max_bins < 1) max_bins = 1;  // fewer rows than min_obs_in_bins: the reference divides by zero (:900-903)
    const int64_t large = total / max_bins;
    int64_t remaining_bins = max_bins, remaining = total;
    std::vector<char> is_large(nc, 0);
    for (int64_t i = 0; i < nc; i++) {
      if (cand[i].second >= large) {
        is_large[i] = 1;
        remaining_bins--;
        remaining -= cand[i].second;
      }
    }
    if (remaining_bins < 1) remaining_bins = 1;
    int64_t cur_large = remaining / remaining_bins;
    int64_t running = 0, made = 0;
    for (int64_t i = 0; i + 1 < nc; i++) {
      if (!is_large[i]) remaining -= cand[i].second;
      running += cand[i].second;
      const bool cut = is_large[i] || running >= cur_large ||
                       (is_large[i + 1] && running >= std::max<int64_t>(1, cur_large / 2));
      if (!cut) continue;
      bounds.push_back((cand[i].first + cand[i + 1].first) / 2);
      if (++made >= max_boundaries) break;
      running = 0;
      if (!is_large[i]) {
        remaining_bins = std::max<int64_t>(1, remaining_bins - 1);
        cur_large = remaining / remaining_bins;
      }
    }
  } else {
    int64_t running = 0;
    for (int64_t i = 0; i + 1 < nc; i++) {
      running += cand[i].second;
      if (running >= min_obs_in_bins) {
        bounds.push_back((cand[i].first + cand[i + 1].first) / 2);
        running = 0;
      }
    }
  }
  for (int k = 0; k < n_special; k++) add_special_bucket(special[k], &bounds);
  std::sort(bounds.begin(), bounds.end());
  return YGG_OK;
}

// ygg_discretize_boundaries(16) once maximum_num_bins is checked: sort + unique + gen_boundaries with {0, mean}.
int discretize_column(const float* values, int64_t n, int32_t maximum_num_bins, int32_t min_obs_in_bins,
                      float* out_boundaries, int32_t capacity, int32_t* out_num_boundaries, double* out_mean) {
  if (!values || !out_boundaries || !out_num_boundaries || !out_mean) return YGG_ERR_INVALID_ARGUMENT;
  if (min_obs_in_bins < 1) return YGG_ERR_INVALID_ARGUMENT;
  // Non-missing values, their mean (numerical().mean(), data_spec_inference.cc:255-262).
  std::vector<float> v;
  v.reserve(n);
  long double sum = 0;
  for (int64_t i = 0; i < n; i++) {
    if (!std::isnan(values[i])) {
      v.push_back(values[i]);
      sum += values[i];
    }
  }
  const double mean = v.empty() ? 0.0 : static_cast<double>(sum / static_cast<long double>(v.size()));
  *out_mean = mean;
  std::sort(v.begin(), v.end());
  // Unique values with counts = the "candidates".
  std::vector<std::pair<float, int64_t>> cand;
  for (size_t i = 0; i < v.size();) {
    size_t j = i;
    while (j < v.size() && v[j] == v[i]) j++;
    cand.emplace_back(v[i], static_cast<int64_t>(j - i));
    i = j;
  }
  const float special[2] = {0.f, static_cast<float>(mean)};
  std::vector<float> bounds;
  gen_boundaries(cand, maximum_num_bins, min_obs_in_bins, special, 2, &bounds);
  *out_num_boundaries = static_cast<int32_t>(bounds.size());
  if (static_cast<int32_t>(bounds.size()) > capacity) return YGG_ERR_INVALID_ARGUMENT;
  std::memcpy(out_boundaries, bounds.data(), bounds.size() * sizeof(float));
  return YGG_OK;
}

}  // namespace

extern "C" {

int ygg_gen_discretized_boundaries(const float* values, const int64_t* counts, int64_t n_candidates,
                                   int32_t maximum_num_bins, int32_t min_obs_in_bins, const float* special_values,
                                   int32_t n_special, float* out_boundaries, int32_t capacity,
                                   int32_t* out_num_boundaries) {
  if ((n_candidates > 0 && (!values || !counts)) || !out_num_boundaries || (n_special > 0 && !special_values))
    return YGG_ERR_INVALID_ARGUMENT;
  if (maximum_num_bins < 1 || maximum_num_bins > 65534 || min_obs_in_bins < 1 || n_candidates < 0 || n_special < 0)
    return YGG_ERR_INVALID_ARGUMENT;
  std::vector<std::pair<float, int64_t>> cand(n_candidates);
  for (int64_t i = 0; i < n_candidates; i++) {
    if (counts[i] < 1 || (i > 0 && !(values[i] > values[i - 1]))) return YGG_ERR_INVALID_ARGUMENT;
    cand[i] = {values[i], counts[i]};
  }
  std::vector<float> bounds;
  gen_boundaries(cand, maximum_num_bins, min_obs_in_bins, special_values, n_special, &bounds);
  *out_num_boundaries = static_cast<int32_t>(bounds.size());
  if (static_cast<int32_t>(bounds.size()) > capacity || (!out_boundaries && !bounds.empty())) return YGG_ERR_INVALID_ARGUMENT;
  if (!bounds.empty()) std::memcpy(out_boundaries, bounds.data(), bounds.size() * sizeof(float));
  return YGG_OK;
}

int ygg_discretize_boundaries(const float* values, int64_t n, int32_t maximum_num_bins,
                              int32_t min_obs_in_bins, float* out_boundaries, int32_t capacity,
                              int32_t* out_num_boundaries, double* out_mean) {
  if (maximum_num_bins < 2 || maximum_num_bins > 65534) return YGG_ERR_INVALID_ARGUMENT;
  return discretize_column(values, n, maximum_num_bins, min_obs_in_bins, out_boundaries, capacity, out_num_boundaries,
                           out_mean);
}

int ygg_discretize_boundaries16(const float* values, int64_t n, int32_t maximum_num_bins,
                                int32_t min_obs_in_bins, float* out_boundaries, int32_t capacity,
                                int32_t* out_num_boundaries, double* out_mean) {
  if (maximum_num_bins < 2 || maximum_num_bins > 65535) return YGG_ERR_INVALID_ARGUMENT;
  return discretize_column(values, n, maximum_num_bins, min_obs_in_bins, out_boundaries, capacity, out_num_boundaries,
                           out_mean);
}

int ygg_discretize_encode(const float* values, int64_t n, const float* boundaries, int32_t num_boundaries,
                          int32_t na_bin, uint8_t* out) {
  if (!values || !out || (!boundaries && num_boundaries > 0)) return YGG_ERR_INVALID_ARGUMENT;
  if (num_boundaries + 1 > 256 || na_bin < 0 || na_bin > num_boundaries) return YGG_ERR_INVALID_ARGUMENT;
  for (int64_t i = 0; i < n; i++) {
    const float x = values[i];
    if (std::isnan(x)) {
      out[i] = static_cast<uint8_t>(na_bin);  // missing folded into the NA-replacement bin
    } else {
      out[i] = static_cast<uint8_t>(std::upper_bound(boundaries, boundaries + num_boundaries, x) - boundaries);
    }
  }
  return YGG_OK;
}

}  // extern "C"
