// ygg_binning.cu — on-GPU dataspec step in front of the split finder (SURVEY.md §8f N1): float32 columns
// -> discretization boundaries -> uint8 bins written straight into the device-resident dataset (or, above 256
// bins, uint16 codes that become a discretized wide column, DESIGN.md §25).
//
// Same rule as the host path (ygg_dataspec.cc), i.e. the reference's
//   GenDiscretizedBoundaries                 dataset/data_spec.cc:854-986
//   AddBucket (special values {0, mean})     dataset/data_spec.cc:77-107
//   FinalizeComputeSpecDiscretizedNumerical  dataset/data_spec_inference.cc:226-250
//   NumericalToDiscretizedNumerical          dataset/data_spec.cc:1006-1018
// but restructured for the GPU, one column at a time (all HBM-bound integer work, DESIGN.md §9):
//   k_bin_keys      float -> order-preserving u32 key (-0 -> +0, NaN -> 0xFFFFFFFF), sum + count of the
//                   non-missing values (fixed-order reduction: the result does not depend on the grid);
//   k_radix_*       stable LSD radix sort of the keys, 4 passes of 8 bits: per-tile digit histogram,
//                   one-block exclusive scan of the [digit][tile] table, stable scatter (warp match_any
//                   ranking, per-warp digit counters in shared memory);
//   k_heads_*       positions of the first occurrence of every distinct value = the reference's sorted
//                   "unique value, count" candidates: count_i = pos[i+1] - pos[i];
//   k_bin_prep / k_bin_find_large / k_bin_boundaries
//                   the greedy boundary rule.  The reference walks all candidates; here every cut is
//                   found by a warp-cooperative search over the prefix counts (pos[]), so a column costs
//                   <= 255 searches instead of 10^7 sequential steps — identical cuts, proven against
//                   the host rule bit for bit in tests/test_gpu_binning.py;
//   k_bin_encode    bin = upper_bound(boundaries, x), NaN -> the bin of the mean.
// Up to 65535 bins (ygg_dataset_builder_add_numerical16_async, DESIGN.md §25) the sort, distinct-value and mean kernels
// are the same; the large candidates are listed in order by a compaction (k_bin_large_count / _write), the cuts are walked
// by k_bin_boundaries16 with its lists in global memory, k_bin_specials16 inserts the special values' bins, and
// k_bin_encode16 writes uint16 codes through a two-level search.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/ygg_b200.h"
#include "../../include/ygg_b200_dataspec.h"
#include "ygg_internal.h"

namespace {

constexpr int kSortThreads = 512;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kSortRounds = 16;                                 // keys per thread
constexpr int kSortTile = kSortThreads * kSortRounds;           // 8192 keys per CTA
constexpr int kMaxBoundaries = 255;
constexpr int kMaxLarge = 1024;                                 // >= 2 * maximum_num_bins (see k_bin_find_large)
constexpr uint32_t kNanKey = 0xFFFFFFFFu;
constexpr int kMaxBoundaries16 = 65534;                         // uint16 codes 0..65534
constexpr int kBoundaries16Cap = kMaxBoundaries16 + 8;          // room for the special values' bins before the check
constexpr int kMaxLarge16 = 2 * 65536;                          // >= 2 * maximum_num_bins
constexpr int kCoarseStep = 64;                                 // k_bin_encode16: boundaries per coarse entry
constexpr int kCoarse = 1024;                                   // coarse entries (kCoarse * kCoarseStep > kMaxBoundaries16)

struct BinState {
  unsigned long long n_valid;   // non-missing values
  double sum;                   // their sum (compensated, fixed order)
  double mean;
  uint32_t nc;                  // number of distinct values
  int32_t mode;                 // 0: one boundary per candidate group (few candidates), 1: greedy quantiles
  int32_t max_bins;             // after reserving the special bins (before the min_obs clamp)
  int32_t max_bins_eff;         // min(max_bins, total / min_obs)
  long long large;              // candidates with count >= large own a bin
  uint32_t n_large;
  int32_t num_boundaries;
  int32_t na_bin;
  int32_t error;                // 1: more than kMaxLarge large candidates / too many boundaries
};

__device__ __forceinline__ uint32_t float_to_key(float x) {
  if (x != x) return kNanKey;
  x += 0.0f;  // -0 -> +0: the reference's candidates compare equal (float ==), so they must share a key
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_to_float(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// ---- keys + sum ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSortThreads) k_bin_keys(const float* __restrict__ values, int64_t n, int64_t n_stats,
                                                           uint32_t* __restrict__ keys, double* __restrict__ partial,
                                                           BinState* st) {
  __shared__ double s_sum[kSortWarps];
  __shared__ unsigned int s_cnt[kSortWarps];
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kSortTile;
  double sum = 0;
  unsigned int cnt = 0;
#pragma unroll
  for (int r = 0; r < kSortRounds; r++) {
    const int64_t i = base + r * kSortThreads + threadIdx.x;
    uint32_t key = kNanKey;  // padding and rows beyond the statistics sample sort behind every value
    if (i < n_stats) {
      const float x = values[i];
      key = float_to_key(x);
      if (key != kNanKey) { sum += static_cast<double>(x); cnt++; }
    }
    keys[i] = key;  // keys[] is padded to a whole number of tiles
  }
  // fixed-order tree reduction (lane, then warp): deterministic for a given n
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_down_sync(0xffffffffu, sum, o);
    cnt += __shfl_down_sync(0xffffffffu, cnt, o);
  }
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { s_sum[w] = sum; s_cnt[w] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    unsigned int c = 0;
    for (int i = 0; i < kSortWarps; i++) { t += s_sum[i]; c += s_cnt[i]; }
    partial[blockIdx.x] = t;
    atomicAdd(&st->n_valid, static_cast<unsigned long long>(c));
  }
  (void)n;
}

// ---- radix sort ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSortThreads) k_radix_hist(const uint32_t* __restrict__ keys, int shift, int n_tiles,
                                                             uint32_t* __restrict__ table /*[256][n_tiles]*/) {
  __shared__ unsigned int s_hist[256];
  if (threadIdx.x < 256) s_hist[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kSortTile;
#pragma unroll
  for (int r = 0; r < kSortRounds; r++) {
    const uint32_t key = keys[base + r * kSortThreads + threadIdx.x];
    atomicAdd(&s_hist[(key >> shift) & 255u], 1u);
  }
  __syncthreads();
  if (threadIdx.x < 256) table[static_cast<size_t>(threadIdx.x) * n_tiles + blockIdx.x] = s_hist[threadIdx.x];
}

// Exclusive scan of `count` u32 entries in place, three phases: k_scan_local scans chunks of 4096 entries
// and records their totals, k_scan_tops scans the totals (one CTA), k_scan_add adds them back.
constexpr int kScanChunk = 4096;

__device__ __forceinline__ uint32_t block_exclusive_scan_1024(uint32_t t, uint32_t* s_warp /*[32]*/, uint32_t* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t inc = t;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t x = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += x;
  }
  if (lane == 31) s_warp[w] = inc;
  __syncthreads();
  if (w == 0) {
    uint32_t x = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    s_warp[lane] = x;  // inclusive over warps
  }
  __syncthreads();
  const uint32_t excl = (w > 0 ? s_warp[w - 1] : 0u) + (inc - t);
  *total = s_warp[31];
  __syncthreads();
  return excl;
}

__global__ void __launch_bounds__(1024) k_scan_local(uint32_t* data, int64_t count, uint32_t* chunk_total) {
  __shared__ uint32_t s_warp[32];
  const int64_t i0 = static_cast<int64_t>(blockIdx.x) * kScanChunk + static_cast<int64_t>(threadIdx.x) * 4;
  uint32_t v[4], t = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) { v[k] = (i0 + k < count) ? data[i0 + k] : 0u; t += v[k]; }
  uint32_t total;
  uint32_t excl = block_exclusive_scan_1024(t, s_warp, &total);
#pragma unroll
  for (int k = 0; k < 4; k++) {
    if (i0 + k < count) data[i0 + k] = excl;
    excl += v[k];
  }
  if (threadIdx.x == 0) chunk_total[blockIdx.x] = total;
}

// Scans up to 1024 * 4 chunk totals in place (count <= 16.7M entries overall) and reports the grand total.
__global__ void __launch_bounds__(1024) k_scan_tops(uint32_t* chunk_total, int n_chunks, uint32_t* total_out) {
  __shared__ uint32_t s_warp[32];
  const int i0 = threadIdx.x * 4;
  uint32_t v[4], t = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) { v[k] = (i0 + k < n_chunks) ? chunk_total[i0 + k] : 0u; t += v[k]; }
  uint32_t total;
  uint32_t excl = block_exclusive_scan_1024(t, s_warp, &total);
#pragma unroll
  for (int k = 0; k < 4; k++) {
    if (i0 + k < n_chunks) chunk_total[i0 + k] = excl;
    excl += v[k];
  }
  if (threadIdx.x == 0 && total_out != nullptr) *total_out = total;
}

__global__ void __launch_bounds__(1024) k_scan_add(uint32_t* data, int64_t count, const uint32_t* chunk_total) {
  const uint32_t add = chunk_total[blockIdx.x];
  const int64_t i0 = static_cast<int64_t>(blockIdx.x) * kScanChunk + static_cast<int64_t>(threadIdx.x) * 4;
#pragma unroll
  for (int k = 0; k < 4; k++)
    if (i0 + k < count) data[i0 + k] += add;
}

// Stable scatter of one tile.  The keys are first placed in tile-local sorted order in shared memory
// (warp match_any ranking + per-warp digit offsets), then written out by consecutive threads: keys of the
// same digit are contiguous, so the global stores are coalesced runs instead of 32 scattered 4-byte
// writes per warp instruction.
__global__ void __launch_bounds__(kSortThreads) k_radix_scatter(const uint32_t* __restrict__ in, uint32_t* __restrict__ out,
                                                                int shift, int n_tiles,
                                                                const uint32_t* __restrict__ table /*scanned*/) {
  __shared__ uint16_t s_cnt[kSortWarps][256];   // per-warp digit counts, then tile-local offsets (<= 8192)
  __shared__ uint32_t s_keys[kSortTile];
  __shared__ uint32_t s_gbase[256];             // global offset of the digit minus its tile-local offset
  __shared__ uint32_t s_wsum[8];
  for (int i = threadIdx.x; i < kSortWarps * 256; i += kSortThreads) (&s_cnt[0][0])[i] = 0;
  __syncthreads();
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // warp w owns the 512 consecutive keys [w*512, (w+1)*512) of the tile, 32 at a time, in order
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kSortTile + w * (kSortRounds * 32);
  uint32_t key[kSortRounds];
  uint16_t wrank[kSortRounds];                  // rank of the key among the keys of its digit in this warp
#pragma unroll
  for (int r = 0; r < kSortRounds; r++) key[r] = in[base + r * 32 + lane];
#pragma unroll
  for (int r = 0; r < kSortRounds; r++) {
    const uint32_t d = (key[r] >> shift) & 255u;
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    const int leader = __ffs(peers) - 1;
    uint32_t before = 0;                         // keys of this digit in the earlier rounds of the warp
    if (lane == leader) {                        // one writer per digit
      before = s_cnt[w][d];
      s_cnt[w][d] = static_cast<uint16_t>(before + __popc(peers));
    }
    before = __shfl_sync(0xffffffffu, before, leader);
    wrank[r] = static_cast<uint16_t>(before + __popc(peers & ((1u << lane) - 1u)));
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x < 256) {
    const int d = threadIdx.x;
    uint32_t c = 0;
#pragma unroll
    for (int i = 0; i < kSortWarps; i++) c += s_cnt[i][d];
    // exclusive scan of the tile's digit counts over the 256 digits (8 warps)
    uint32_t inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t x = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += x;
    }
    if (lane == 31) s_wsum[w] = inc;
    // (only the first 8 warps are here; a named barrier keeps the other warps out of it)
    asm volatile("bar.sync 1, 256;");
    uint32_t local_base = inc - c;
    for (int i = 0; i < w; i++) local_base += s_wsum[i];
    s_gbase[d] = table[static_cast<size_t>(d) * n_tiles + blockIdx.x] - local_base;
    uint32_t running = local_base;
#pragma unroll
    for (int i = 0; i < kSortWarps; i++) {
      const uint32_t t = s_cnt[i][d];
      s_cnt[i][d] = static_cast<uint16_t>(running);
      running += t;
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < kSortRounds; r++) s_keys[s_cnt[w][(key[r] >> shift) & 255u] + wrank[r]] = key[r];
  __syncthreads();
#pragma unroll
  for (int r = 0; r < kSortRounds; r++) {
    const int i = r * kSortThreads + threadIdx.x;
    const uint32_t k = s_keys[i];
    out[s_gbase[(k >> shift) & 255u] + i] = k;
  }
}

// ---- distinct values ----------------------------------------------------------------------------
__device__ __forceinline__ bool is_head(const uint32_t* keys, int64_t i, unsigned long long n_valid) {
  return i < static_cast<int64_t>(n_valid) && (i == 0 || keys[i] != keys[i - 1]);
}

__global__ void __launch_bounds__(kSortThreads) k_heads_count(const uint32_t* __restrict__ keys, const BinState* st,
                                                              uint32_t* __restrict__ tile_count) {
  __shared__ unsigned int s_total;
  if (threadIdx.x == 0) s_total = 0;
  __syncthreads();
  const unsigned long long nv = st->n_valid;
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kSortTile + static_cast<int64_t>(threadIdx.x) * kSortRounds;
  unsigned int c = 0;
#pragma unroll
  for (int r = 0; r < kSortRounds; r++) c += is_head(keys, base + r, nv) ? 1u : 0u;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_total, c);
  __syncthreads();
  if (threadIdx.x == 0) tile_count[blockIdx.x] = s_total;
}

__global__ void __launch_bounds__(kSortThreads) k_heads_write(const uint32_t* __restrict__ keys, BinState* st,
                                                              const uint32_t* __restrict__ tile_offset /*scanned*/,
                                                              const uint32_t* __restrict__ total, uint32_t* __restrict__ pos) {
  __shared__ uint32_t s_warp[kSortWarps];
  const unsigned long long nv = st->n_valid;
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kSortTile + static_cast<int64_t>(threadIdx.x) * kSortRounds;
  uint32_t flags = 0, c = 0;
#pragma unroll
  for (int r = 0; r < kSortRounds; r++)
    if (is_head(keys, base + r, nv)) { flags |= 1u << r; c++; }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t inc = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t x = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += x;
  }
  if (lane == 31) s_warp[w] = inc;
  __syncthreads();
  uint32_t off = tile_offset[blockIdx.x] + (inc - c);
  for (int i = 0; i < w; i++) off += s_warp[i];
#pragma unroll
  for (int r = 0; r < kSortRounds; r++)
    if (flags & (1u << r)) pos[off++] = static_cast<uint32_t>(base + r);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    st->nc = *total;
    pos[*total] = static_cast<uint32_t>(nv);  // sentinel: count_i = pos[i+1] - pos[i]
  }
}

// ---- boundary rule ------------------------------------------------------------------------------
__device__ __forceinline__ void neumaier_add(double& s, double& comp, double x) {
  const double t = s + x;
  if (isfinite(t)) comp += (fabs(s) >= fabs(x)) ? (s - t) + x : (x - t) + s;
  s = t;
}

// One warp: the per-tile sums are added with Neumaier compensation (lane-strided, then the 32 lane sums
// in lane order) — a fixed order, so the mean is reproducible.
__global__ void __launch_bounds__(32) k_bin_prep(const uint32_t* __restrict__ keys, const double* __restrict__ partial,
                                                 int n_tiles, int maximum_num_bins, int min_obs, BinState* st) {
  double s = 0, comp = 0;
  for (int i = threadIdx.x; i < n_tiles; i += 32) neumaier_add(s, comp, partial[i]);
  __shared__ double s_s[32], s_c[32];
  s_s[threadIdx.x] = s; s_c[threadIdx.x] = comp;
  __syncwarp();
  if (threadIdx.x != 0) return;
  s = 0; comp = 0;
  for (int i = 0; i < 32; i++) { neumaier_add(s, comp, s_s[i]); comp += s_c[i]; }
  const unsigned long long nv = st->n_valid;
  st->sum = s + comp;
  const double mean = nv ? (s + comp) / static_cast<double>(nv) : 0.0;
  st->mean = mean;
  const uint32_t nc = st->nc;
  int in_bounds = 0;
  if (nc > 0) {
    const float lo = key_to_float(keys[0]), hi = key_to_float(keys[nv - 1]);
    const float special[2] = {0.f, static_cast<float>(mean)};
    for (int k = 0; k < 2; k++)
      if (special[k] > lo && special[k] < hi) in_bounds++;
  }
  const int reserved = maximum_num_bins - 2 - in_bounds;  // >= 0: the host validates maximum_num_bins >= 4
  int max_bins = reserved < 1 ? 1 : reserved;
  st->max_bins = max_bins;
  st->mode = 0;
  st->n_large = 0;
  st->large = 0;
  st->max_bins_eff = max_bins;
  if (static_cast<long long>(nc) > max_bins) {
    long long eff = static_cast<long long>(nv) / min_obs;
    if (eff > max_bins) eff = max_bins;
    if (eff < 1) eff = 1;
    st->max_bins_eff = static_cast<int>(eff);
    st->large = static_cast<long long>(nv) / eff;
    st->mode = 1;
  }
}

__global__ void __launch_bounds__(256) k_bin_find_large(const uint32_t* __restrict__ pos, BinState* st,
                                                        uint32_t* __restrict__ large_idx) {
  if (st->mode != 1) return;
  const uint32_t nc = st->nc;
  const long long large = st->large;
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < nc; u += gridDim.x * blockDim.x) {
    if (static_cast<long long>(pos[u + 1] - pos[u]) >= large) {
      // at most total / floor(total / bins) < 2 * bins candidates can be this large
      const uint32_t k = atomicAdd(&st->n_large, 1u);
      if (k < kMaxLarge) large_idx[k] = u; else st->error = 1;
    }
  }
}

// First j in [lo, hi) with pos[j] >= target (hi if none); the 32 lanes probe 32 pivots per step.
__device__ uint32_t warp_lower_bound(const uint32_t* __restrict__ pos, uint32_t lo, uint32_t hi, unsigned long long target) {
  const int lane = threadIdx.x & 31;
  while (hi - lo > 32) {
    const uint32_t step = (hi - lo + 31) / 32;   // pivots lo + step*(lane+1) - 1
    const unsigned long long p = static_cast<unsigned long long>(lo) + static_cast<unsigned long long>(step) * (lane + 1) - 1;
    const bool ge = p >= hi ? true : (pos[p] >= target);
    const uint32_t mask = __ballot_sync(0xffffffffu, ge);
    if (mask == 0u) return hi;                   // even pos[hi - 1] < target
    const int first = __ffs(mask) - 1;
    const uint32_t new_lo = lo + step * first;
    unsigned long long new_hi = static_cast<unsigned long long>(lo) + static_cast<unsigned long long>(step) * (first + 1) - 1;
    if (new_hi > hi) new_hi = hi;
    lo = new_lo;
    hi = static_cast<uint32_t>(new_hi);
    // invariant: the answer lies in [lo, hi] where pos[hi] >= target (or hi is the original end)
  }
  const uint32_t j = lo + lane;
  const bool ge = j >= hi ? true : (pos[j] >= target);
  const uint32_t mask = __ballot_sync(0xffffffffu, ge);
  if (mask == 0u) return hi;
  const uint32_t r = lo + (__ffs(mask) - 1);
  return r < hi ? r : hi;
}

__device__ void add_special_bucket(float v, float* b, int* n) {
  const float lo = nextafterf(v, v - 1.f), hi = nextafterf(v, v + 1.f);
  if (*n == 0) { b[0] = lo; b[1] = hi; *n = 2; return; }
  int m = 0;
  for (int i = 0; i < *n; i++)
    if (!(b[i] >= lo && b[i] <= hi)) b[m++] = b[i];
  *n = m;
  if (m == 0) { b[0] = lo; b[1] = hi; *n = 2; return; }
  float mn = b[0], mx = b[0];
  for (int i = 1; i < m; i++) { mn = fminf(mn, b[i]); mx = fmaxf(mx, b[i]); }
  if (mn < hi) b[(*n)++] = lo;
  if (mx > lo) b[(*n)++] = hi;
}

// One warp.  Lane 0 carries the state of the reference's loop; the searches are warp-wide.
__global__ void __launch_bounds__(32) k_bin_boundaries(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ pos,
                                                       uint32_t* __restrict__ large_idx, int min_obs, BinState* st,
                                                       float* __restrict__ out_boundaries /*[kMaxBoundaries + 5]*/) {
  __shared__ float s_b[kMaxBoundaries + 8];
  __shared__ uint32_t s_cut[kMaxBoundaries + 1];   // candidate index before each cut; the values are read afterwards
  __shared__ uint32_t s_large[kMaxLarge];
  __shared__ uint32_t s_sorted[kMaxLarge];
  const int lane = threadIdx.x;
  const uint32_t nc = st->nc;
  const unsigned long long total = st->n_valid;
  int nb = 0;
  bool overflow = st->error != 0;
  auto value = [&](uint32_t u) { return key_to_float(keys[pos[u]]); };
  if (st->mode == 0) {
    if (lane == 0) {
      long long running = 0;
      for (uint32_t i = 0; i + 1 < nc; i++) {  // nc <= max_bins <= 254 here
        running += pos[i + 1] - pos[i];
        if (running >= min_obs) {
          if (nb < kMaxBoundaries) s_cut[nb++] = i; else overflow = true;
          running = 0;
        }
      }
    }
    nb = __shfl_sync(0xffffffffu, nb, 0);
  } else if (!overflow) {
    // sort the indices of the large candidates (rank sort, <= kMaxLarge entries)
    const uint32_t nL = min(st->n_large, static_cast<uint32_t>(kMaxLarge));
    for (uint32_t i = lane; i < nL; i += 32) s_large[i] = large_idx[i];
    __syncwarp();
    for (uint32_t i = lane; i < nL; i += 32) {
      const uint32_t v = s_large[i];
      uint32_t r = 0;
      for (uint32_t j = 0; j < nL; j++) r += s_large[j] < v ? 1u : 0u;
      s_sorted[r] = v;
    }
    __syncwarp();
    const int max_boundaries = st->max_bins - 1;
    long long total_nonlarge = static_cast<long long>(total);
    for (uint32_t i = 0; i < nL; i++) total_nonlarge -= pos[s_sorted[i] + 1] - pos[s_sorted[i]];
    long long remaining_bins = static_cast<long long>(st->max_bins_eff) - nL;
    if (remaining_bins < 1) remaining_bins = 1;
    long long cur_large = total_nonlarge / remaining_bins;
    uint32_t s = 0, li = 0;
    long long lsum = 0;  // counts of the large candidates with index < s
    int made = 0;
    while (static_cast<unsigned long long>(s) + 2 <= nc) {
      const uint32_t next_large = li < nL ? s_sorted[li] : 0xFFFFFFFFu;   // first large index >= s
      const unsigned long long ps = pos[s];
      // (a) running >= cur_large: first i >= s with pos[i+1] - pos[s] >= cur_large
      uint32_t i_a;
      if (cur_large <= 0) {
        i_a = s;
      } else {
        const uint32_t j = warp_lower_bound(pos, s + 1, nc + 1, ps + static_cast<unsigned long long>(cur_large));
        i_a = j <= nc ? j - 1 : 0xFFFFFFFFu;
      }
      // (b) the next large candidate cuts at its own index; (c) the candidate before it cuts early
      uint32_t i_star = min(i_a, next_large);
      if (next_large != 0xFFFFFFFFu && next_large >= s + 1) {
        const long long half = cur_large / 2 > 1 ? cur_large / 2 : 1;
        if (static_cast<long long>(pos[next_large] - ps) >= half) i_star = min(i_star, next_large - 1);
      }
      if (static_cast<unsigned long long>(i_star) + 2 > nc) break;     // the loop stops at nc - 2
      if (lane == 0) {
        if (nb < kMaxBoundaries) s_cut[nb] = i_star; else overflow = true;
      }
      nb++;
      if (++made >= max_boundaries) break;   // checked after the push, as the reference does
      const bool large_cut = i_star == next_large;
      if (large_cut) { lsum += pos[next_large + 1] - pos[next_large]; li++; }
      const long long remaining = total_nonlarge - (static_cast<long long>(pos[i_star + 1]) - lsum);
      if (!large_cut) {
        remaining_bins = remaining_bins - 1 < 1 ? 1 : remaining_bins - 1;
        cur_large = remaining / remaining_bins;
      }
      s = i_star + 1;
    }
    if (nb > kMaxBoundaries) { nb = kMaxBoundaries; overflow = true; }
  }
  __syncwarp();
  // boundary = midpoint of the candidates around each cut (float arithmetic, as the reference)
  for (int k = lane; k < nb; k += 32) s_b[k] = (value(s_cut[k]) + value(s_cut[k] + 1)) / 2;
  __syncwarp();
  if (lane == 0) {
    const float special[2] = {0.f, static_cast<float>(st->mean)};
    for (int k = 0; k < 2; k++) add_special_bucket(special[k], s_b, &nb);
    // insertion sort (<= 259 entries, nearly sorted)
    for (int i = 1; i < nb; i++) {
      const float x = s_b[i];
      int j = i - 1;
      while (j >= 0 && s_b[j] > x) { s_b[j + 1] = s_b[j]; j--; }
      s_b[j + 1] = x;
    }
    if (nb > kMaxBoundaries) overflow = true;
    int na = 0;  // upper_bound(boundaries, (float)mean)
    const float m = static_cast<float>(st->mean);
    const int lim = nb < kMaxBoundaries ? nb : kMaxBoundaries;
    for (int i = 0; i < lim; i++) {
      out_boundaries[i] = s_b[i];
      if (s_b[i] <= m) na = i + 1;
    }
    st->num_boundaries = nb;
    st->na_bin = na;
    if (overflow) st->error = 1;
  }
}

// ---- encode -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_bin_encode(const float* __restrict__ values, int64_t n, const BinState* st,
                                                    const float* __restrict__ boundaries, uint8_t* __restrict__ out) {
  __shared__ float s_b[256];
  const int nb = min(st->num_boundaries, kMaxBoundaries);
  const int na = st->na_bin;
  s_b[threadIdx.x] = threadIdx.x < nb ? boundaries[threadIdx.x] : __int_as_float(0x7f800000);  // +inf padding
  __syncthreads();
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float x = values[i];
    int bin = na;
    if (x == x) {
      // upper_bound over 256 padded entries: number of boundaries <= x
      int lo = 0;
#pragma unroll
      for (int step = 128; step > 0; step >>= 1)
        if (s_b[lo + step - 1] <= x) lo += step;
      bin = lo < nb ? lo : nb;  // x = +inf passes the padding too
    }
    out[i] = static_cast<uint8_t>(bin);
  }
}

// ---- up to 65535 bins ---------------------------------------------------------------------------
// The large candidates (count >= st->large) in increasing order: per tile of kSortTile candidates a count, scanned, then
// written at their offsets.  st->n_large = their number; more than kMaxLarge16 sets st->error.
__device__ __forceinline__ bool is_large(const uint32_t* pos, int64_t u, uint32_t nc, long long large) {
  return u < static_cast<int64_t>(nc) && static_cast<long long>(pos[u + 1] - pos[u]) >= large;
}

__global__ void __launch_bounds__(kSortThreads) k_bin_large_count(const uint32_t* __restrict__ pos, const BinState* st,
                                                                  uint32_t* __restrict__ tile_count) {
  __shared__ unsigned int s_total;
  if (threadIdx.x == 0) s_total = 0;
  __syncthreads();
  unsigned int c = 0;
  if (st->mode == 1) {
    const uint32_t nc = st->nc;
    const long long large = st->large;
    const int64_t base = static_cast<int64_t>(blockIdx.x) * kSortTile + static_cast<int64_t>(threadIdx.x) * kSortRounds;
#pragma unroll
    for (int r = 0; r < kSortRounds; r++) c += is_large(pos, base + r, nc, large) ? 1u : 0u;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_total, c);
  __syncthreads();
  if (threadIdx.x == 0) tile_count[blockIdx.x] = s_total;
}

__global__ void __launch_bounds__(kSortThreads) k_bin_large_write(const uint32_t* __restrict__ pos, BinState* st,
                                                                  const uint32_t* __restrict__ tile_offset /*scanned*/,
                                                                  const uint32_t* __restrict__ total,
                                                                  uint32_t* __restrict__ large_idx) {
  __shared__ uint32_t s_warp[kSortWarps];
  if (st->mode != 1) return;
  const uint32_t nc = st->nc;
  const long long large = st->large;
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kSortTile + static_cast<int64_t>(threadIdx.x) * kSortRounds;
  uint32_t flags = 0, c = 0;
#pragma unroll
  for (int r = 0; r < kSortRounds; r++)
    if (is_large(pos, base + r, nc, large)) { flags |= 1u << r; c++; }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t inc = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t x = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += x;
  }
  if (lane == 31) s_warp[w] = inc;
  __syncthreads();
  uint32_t off = tile_offset[blockIdx.x] + (inc - c);
  for (int i = 0; i < w; i++) off += s_warp[i];
#pragma unroll
  for (int r = 0; r < kSortRounds; r++)
    if (flags & (1u << r)) {
      if (off < static_cast<uint32_t>(kMaxLarge16)) large_idx[off] = static_cast<uint32_t>(base + r);
      off++;
    }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    st->n_large = *total;
    if (*total > static_cast<uint32_t>(kMaxLarge16)) st->error = 1;
  }
}

// k_bin_boundaries' walk with its lists in global memory: `large_idx` sorted (k_bin_large_write), the cuts in `cut`
// [kMaxBoundaries16], their midpoints in `mids` and their number in st->num_boundaries (before the special values).
__global__ void __launch_bounds__(32) k_bin_boundaries16(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ pos,
                                                         const uint32_t* __restrict__ large_idx, int min_obs, BinState* st,
                                                         uint32_t* __restrict__ cut, float* __restrict__ mids) {
  const int lane = threadIdx.x;
  const uint32_t nc = st->nc;
  const unsigned long long total = st->n_valid;
  int nb = 0;
  bool overflow = st->error != 0;
  auto value = [&](uint32_t u) { return key_to_float(keys[pos[u]]); };
  if (st->mode == 0) {
    if (lane == 0) {
      long long running = 0;
      for (uint32_t i = 0; i + 1 < nc; i++) {  // nc <= max_bins <= 65533 here
        running += pos[i + 1] - pos[i];
        if (running >= min_obs) {
          if (nb < kMaxBoundaries16) cut[nb++] = i; else overflow = true;
          running = 0;
        }
      }
    }
    nb = __shfl_sync(0xffffffffu, nb, 0);
  } else if (!overflow) {
    const uint32_t nL = st->n_large;
    const int max_boundaries = st->max_bins - 1;
    long long lsum_all = 0;
    for (uint32_t i = lane; i < nL; i += 32) lsum_all += pos[large_idx[i] + 1] - pos[large_idx[i]];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lsum_all += __shfl_xor_sync(0xffffffffu, lsum_all, o);
    const long long total_nonlarge = static_cast<long long>(total) - lsum_all;
    long long remaining_bins = static_cast<long long>(st->max_bins_eff) - nL;
    if (remaining_bins < 1) remaining_bins = 1;
    long long cur_large = total_nonlarge / remaining_bins;
    uint32_t s = 0, li = 0;
    long long lsum = 0;  // counts of the large candidates with index < s
    int made = 0;
    while (static_cast<unsigned long long>(s) + 2 <= nc) {
      const uint32_t next_large = li < nL ? large_idx[li] : 0xFFFFFFFFu;   // first large index >= s
      const unsigned long long ps = pos[s];
      // (a) running >= cur_large: first i >= s with pos[i+1] - pos[s] >= cur_large
      uint32_t i_a;
      if (cur_large <= 0) {
        i_a = s;
      } else {
        const uint32_t j = warp_lower_bound(pos, s + 1, nc + 1, ps + static_cast<unsigned long long>(cur_large));
        i_a = j <= nc ? j - 1 : 0xFFFFFFFFu;
      }
      // (b) the next large candidate cuts at its own index; (c) the candidate before it cuts early
      uint32_t i_star = min(i_a, next_large);
      if (next_large != 0xFFFFFFFFu && next_large >= s + 1) {
        const long long half = cur_large / 2 > 1 ? cur_large / 2 : 1;
        if (static_cast<long long>(pos[next_large] - ps) >= half) i_star = min(i_star, next_large - 1);
      }
      if (static_cast<unsigned long long>(i_star) + 2 > nc) break;     // the loop stops at nc - 2
      if (lane == 0) {
        if (nb < kMaxBoundaries16) cut[nb] = i_star; else overflow = true;
      }
      nb++;
      if (++made >= max_boundaries) break;   // checked after the push, as the reference does
      const bool large_cut = i_star == next_large;
      if (large_cut) { lsum += pos[next_large + 1] - pos[next_large]; li++; }
      const long long remaining = total_nonlarge - (static_cast<long long>(pos[i_star + 1]) - lsum);
      if (!large_cut) {
        remaining_bins = remaining_bins - 1 < 1 ? 1 : remaining_bins - 1;
        cur_large = remaining / remaining_bins;
      }
      s = i_star + 1;
    }
    if (nb > kMaxBoundaries16) { nb = kMaxBoundaries16; overflow = true; }
  }
  __syncwarp();
  // boundary = midpoint of the candidates around each cut (float arithmetic, as the reference); non-decreasing
  for (int k = lane; k < nb; k += 32) mids[k] = (value(cut[k]) + value(cut[k] + 1)) / 2;
  if (lane == 0) {
    st->num_boundaries = nb;
    if (overflow) st->error = 1;
  }
}

// add_special_bucket on a SORTED boundary list `in` [n], written sorted to `out` (all threads of the CTA): the entries
// inside [v - ulp, v + ulp] go, v - ulp comes in when an entry stays below it, v + ulp when one stays above it, both
// when none stays.  The host rule appends and sorts at the end; the sorted list is the same.
__device__ int special_pass16(const float* __restrict__ in, int n, float v, float* __restrict__ out, int* s_i) {
  const float lo = nextafterf(v, v - 1.f), hi = nextafterf(v, v + 1.f);
  if (threadIdx.x == 0) {
    int a = 0, b = n;   // first entry >= lo
    while (a < b) { const int m = (a + b) >> 1; if (in[m] < lo) a = m + 1; else b = m; }
    s_i[0] = a;
    b = n;              // first entry > hi
    while (a < b) { const int m = (a + b) >> 1; if (in[m] <= hi) a = m + 1; else b = m; }
    s_i[1] = a;
  }
  __syncthreads();
  const int i0 = s_i[0], i1 = s_i[1];
  __syncthreads();
  const bool none_left = i0 == 0 && i1 == n;
  const int extra = none_left ? 2 : (i0 > 0 ? 1 : 0) + (i1 < n ? 1 : 0);
  const int n_out = i0 + extra + (n - i1);
  for (int k = threadIdx.x; k < n_out; k += blockDim.x) {
    float x;
    if (k < i0) x = in[k];
    else if (k - i0 < extra) x = (k == i0 && (none_left || i0 > 0)) ? lo : hi;
    else x = in[i1 + (k - i0 - extra)];
    out[k] = x;
  }
  __syncthreads();
  return n_out;
}

// One CTA: the special values {0, mean} (as k_bin_boundaries), the count check and na_bin = upper_bound(boundaries, mean).
__global__ void __launch_bounds__(1024) k_bin_specials16(BinState* st, const float* __restrict__ mids, float* __restrict__ tmp,
                                                         float* __restrict__ out) {
  __shared__ int s_i[2];
  const int nb0 = st->num_boundaries;
  const float m = static_cast<float>(st->mean);
  const int nb1 = special_pass16(mids, nb0, 0.f, tmp, s_i);
  const int nb = special_pass16(tmp, nb1, m, out, s_i);
  if (threadIdx.x == 0) {
    int a = 0, b = nb;   // upper_bound(boundaries, (float)mean)
    while (a < b) { const int k = (a + b) >> 1; if (out[k] <= m) a = k + 1; else b = k; }
    st->num_boundaries = nb;
    st->na_bin = a;
    if (nb > kMaxBoundaries16) st->error = 1;
  }
}

// bin = upper_bound(boundaries, x) over up to 65534 boundaries, NaN -> the bin of the mean: the coarse table (every
// kCoarseStep-th boundary) in shared memory picks a run of kCoarseStep - 1 boundaries, searched in global memory (L2).
__global__ void __launch_bounds__(256) k_bin_encode16(const float* __restrict__ values, int64_t n, const BinState* st,
                                                      const float* __restrict__ boundaries, uint16_t* __restrict__ out) {
  __shared__ float s_c[kCoarse];
  const int nb = min(st->num_boundaries, kMaxBoundaries16);
  const int na = st->na_bin;
  const float inf = __int_as_float(0x7f800000);
  for (int k = threadIdx.x; k < kCoarse; k += blockDim.x) {
    const int i = (k + 1) * kCoarseStep - 1;
    s_c[k] = i < nb ? boundaries[i] : inf;   // +inf padding
  }
  __syncthreads();
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < n;
       r += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float x = values[r];
    int bin = na;
    if (x == x) {
      int c = 0;   // coarse entries <= x
#pragma unroll
      for (int step = kCoarse / 2; step > 0; step >>= 1)
        if (s_c[c + step - 1] <= x) c += step;
      const int base = c * kCoarseStep;
      if (base >= nb) {
        bin = nb;
      } else {
        // boundaries [base, base + kCoarseStep - 1) hold the answer; the entry after them is the coarse one, > x
        int p = 0;
#pragma unroll
        for (int step = kCoarseStep / 2; step > 0; step >>= 1) {
          const int i = p + step - 1;
          const float b = (i < kCoarseStep - 1 && base + i < nb) ? __ldg(boundaries + base + i) : inf;
          if (b <= x) p += step;
        }
        bin = min(base + p, nb);   // x = +inf passes the padding too
      }
    }
    out[r] = static_cast<uint16_t>(bin);
  }
}

// A column binned by the 16-bit path that ended with at most 256 bins: its codes as a byte column.
__global__ void __launch_bounds__(256) k_bin_narrow16(const uint16_t* __restrict__ in, int64_t n, uint8_t* __restrict__ out) {
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < n;
       r += static_cast<int64_t>(gridDim.x) * blockDim.x)
    out[r] = static_cast<uint8_t>(in[r]);
}

#define YGG_BIN_CUDA(expr)                                                                   \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      char _m[256];                                                                          \
      std::snprintf(_m, sizeof(_m), "%s failed: %s", #expr, cudaGetErrorString(_e));         \
      return ygg_set_error_msg(YGG_ERR_CUDA, _m);                                            \
    }                                                                                        \
  } while (0)

}  // namespace

constexpr int kRing = 3;  // columns in flight: upload of column k+1 overlaps the kernels of column k

struct HostResult {   // pinned
  BinState st;
  float bounds[256];
};

struct ColumnResult {
  int status = -1;    // -1: not a GPU-binned column, 0: done, 1: in flight
  int lane = -1;
  int64_t n_stats = 0;
  BinState st{};
  float bounds[256];
  bool wide16 = false;           // binned by the 16-bit path: its boundaries are in bounds16
  std::vector<float> bounds16;
};

struct BinLane {
  cudaStream_t stream = nullptr;
  int feature = -1;                 // column in flight on this lane
  float* d_values = nullptr;        // one column
  uint32_t* d_keys[2] = {nullptr, nullptr};
  uint32_t* d_pos = nullptr;        // first index of every distinct value (+ sentinel)
  uint32_t* d_table = nullptr;      // [256][n_tiles] digit counts / [n_tiles] head counts
  uint32_t* d_chunk = nullptr;      // scan chunk totals
  uint32_t* d_total = nullptr;
  uint32_t* d_large = nullptr;
  double* d_partial = nullptr;
  float* d_boundaries = nullptr;
  BinState* d_state = nullptr;
  HostResult* h_result = nullptr;
  // the 16-bit path's lists (allocated on its first column)
  uint32_t* d_large16 = nullptr;    // [kMaxLarge16]
  uint32_t* d_cut = nullptr;        // [kBoundaries16Cap]
  float* d_mids = nullptr;          // [kBoundaries16Cap] each
  float* d_tmp16 = nullptr;
  float* d_bounds16 = nullptr;
  float* h_bounds16 = nullptr;      // pinned
};

struct ygg_dataset_builder {
  ygg_dataset* ds = nullptr;
  std::vector<char> filled;
  std::vector<ColumnResult> results;
  std::vector<uint16_t*> codes16;   // [F] device codes of the 16-bit columns with more than 256 bins (attached at finish)
  int64_t n_tiles = 0;
  int next_lane = 0;
  BinLane lane[kRing];
};

namespace {

void free_builder(ygg_dataset_builder* b) {
  if (b == nullptr) return;
  if (b->ds != nullptr) cudaSetDevice(b->ds->device);
  for (BinLane& l : b->lane) {
    if (l.stream) cudaStreamSynchronize(l.stream);
    cudaFree(l.d_values); cudaFree(l.d_keys[0]); cudaFree(l.d_keys[1]); cudaFree(l.d_pos); cudaFree(l.d_table);
    cudaFree(l.d_chunk); cudaFree(l.d_total); cudaFree(l.d_large); cudaFree(l.d_partial); cudaFree(l.d_boundaries);
    cudaFree(l.d_state);
    cudaFree(l.d_large16); cudaFree(l.d_cut); cudaFree(l.d_mids); cudaFree(l.d_tmp16); cudaFree(l.d_bounds16);
    if (l.h_bounds16) cudaFreeHost(l.h_bounds16);
    if (l.h_result) cudaFreeHost(l.h_result);
    if (l.stream) cudaStreamDestroy(l.stream);
  }
  for (uint16_t* c : b->codes16) cudaFree(c);
  if (b->ds != nullptr) ygg_dataset_destroy(b->ds);
  delete b;
}

int ensure_lane(ygg_dataset_builder* b, BinLane* l) {
  if (l->d_values != nullptr) return YGG_OK;
  const int64_t n_sort = b->n_tiles * kSortTile;
  YGG_BIN_CUDA(cudaStreamCreateWithFlags(&l->stream, cudaStreamNonBlocking));
  YGG_BIN_CUDA(cudaMalloc(&l->d_values, sizeof(float) * b->ds->n));
  YGG_BIN_CUDA(cudaMalloc(&l->d_keys[0], sizeof(uint32_t) * n_sort));
  YGG_BIN_CUDA(cudaMalloc(&l->d_keys[1], sizeof(uint32_t) * n_sort));
  YGG_BIN_CUDA(cudaMalloc(&l->d_pos, sizeof(uint32_t) * (n_sort + 1)));
  YGG_BIN_CUDA(cudaMalloc(&l->d_table, sizeof(uint32_t) * 256 * b->n_tiles));
  YGG_BIN_CUDA(cudaMalloc(&l->d_chunk, sizeof(uint32_t) * kScanChunk));
  YGG_BIN_CUDA(cudaMalloc(&l->d_total, sizeof(uint32_t)));
  YGG_BIN_CUDA(cudaMalloc(&l->d_large, sizeof(uint32_t) * kMaxLarge));
  YGG_BIN_CUDA(cudaMalloc(&l->d_partial, sizeof(double) * b->n_tiles));
  YGG_BIN_CUDA(cudaMalloc(&l->d_boundaries, sizeof(float) * 256));
  YGG_BIN_CUDA(cudaMalloc(&l->d_state, sizeof(BinState)));
  YGG_BIN_CUDA(cudaMallocHost(&l->h_result, sizeof(HostResult)));
  return YGG_OK;
}

int ensure_lane16(BinLane* l) {
  if (l->d_large16 != nullptr) return YGG_OK;
  YGG_BIN_CUDA(cudaMalloc(&l->d_large16, sizeof(uint32_t) * kMaxLarge16));
  YGG_BIN_CUDA(cudaMalloc(&l->d_cut, sizeof(uint32_t) * kBoundaries16Cap));
  YGG_BIN_CUDA(cudaMalloc(&l->d_mids, sizeof(float) * kBoundaries16Cap));
  YGG_BIN_CUDA(cudaMalloc(&l->d_tmp16, sizeof(float) * kBoundaries16Cap));
  YGG_BIN_CUDA(cudaMalloc(&l->d_bounds16, sizeof(float) * kBoundaries16Cap));
  YGG_BIN_CUDA(cudaMallocHost(&l->h_bounds16, sizeof(float) * kBoundaries16Cap));
  return YGG_OK;
}

// Frees the 16-bit codes of a feature that is binned again or replaced.
void drop_codes16(ygg_dataset_builder* b, int f) {
  cudaFree(b->codes16[f]);
  b->codes16[f] = nullptr;
}

int launch_scan(BinLane* l, uint32_t* data, int64_t count, uint32_t* total_out) {
  const int64_t n_chunks = (count + kScanChunk - 1) / kScanChunk;
  if (n_chunks > kScanChunk) return ygg_set_error_msg(YGG_ERR_UNIMPLEMENTED, "too many rows for the GPU binning path");
  k_scan_local<<<static_cast<int>(n_chunks), 1024, 0, l->stream>>>(data, count, l->d_chunk);
  k_scan_tops<<<1, 1024, 0, l->stream>>>(l->d_chunk, static_cast<int>(n_chunks), total_out);
  k_scan_add<<<static_cast<int>(n_chunks), 1024, 0, l->stream>>>(data, count, l->d_chunk);
  return YGG_OK;
}

// retire_lane for a column of the 16-bit path (its stream is idle): a column with at most 256 bins becomes a byte
// column, a wider one keeps its codes for ygg_dataset_builder_finish.
int retire_column16(ygg_dataset_builder* b, BinLane* l, int f, ColumnResult* r) {
  ygg_dataset* ds = b->ds;
  if (r->st.error != 0 || r->st.num_boundaries > kMaxBoundaries16) {
    r->status = -1;
    drop_codes16(b, f);
    char m[160];
    std::snprintf(m, sizeof(m), "feature %d needs more than 65535 bins (or has too many heavy values)", f);
    return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, m);
  }
  r->bounds16.assign(l->h_bounds16, l->h_bounds16 + r->st.num_boundaries);
  const int num_bins = r->st.num_boundaries + 1;
  ds->feature_type[f] = YGG_FEATURE_DISCRETIZED_NUMERICAL;
  if (num_bins <= 256) {
    k_bin_narrow16<<<ds->num_sms * 8, 256, 0, l->stream>>>(b->codes16[f], ds->n, ds->d_bins + static_cast<size_t>(f) * ds->n_pad);
    YGG_BIN_CUDA(cudaGetLastError());
    YGG_BIN_CUDA(cudaStreamSynchronize(l->stream));
    drop_codes16(b, f);
    ds->num_bins[f] = num_bins;
    ds->na_bin[f] = r->st.na_bin;
  } else {   // the byte column becomes the wide column's filler at finish
    ds->num_bins[f] = 1;
    ds->na_bin[f] = 0;
  }
  b->filled[f] = 1;
  return YGG_OK;
}

// Waits for the column in flight on `l` (if any) and files its result.
int retire_lane(ygg_dataset_builder* b, BinLane* l) {
  if (l->feature < 0) return YGG_OK;
  const int f = l->feature;
  l->feature = -1;
  ColumnResult& r = b->results[f];
  YGG_BIN_CUDA(cudaStreamSynchronize(l->stream));
  r.st = l->h_result->st;
  std::memcpy(r.bounds, l->h_result->bounds, sizeof(r.bounds));
  r.status = 0;
  r.lane = -1;
  if (r.wide16) return retire_column16(b, l, f, &r);
  if (r.st.error != 0 || r.st.num_boundaries > kMaxBoundaries) {
    r.status = -1;
    char m[160];
    std::snprintf(m, sizeof(m), "feature %d needs more than 256 bins (or has too many heavy values)", f);
    return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, m);
  }
  ygg_dataset* ds = b->ds;
  ds->num_bins[f] = r.st.num_boundaries + 1;
  ds->na_bin[f] = r.st.na_bin;
  ds->feature_type[f] = YGG_FEATURE_DISCRETIZED_NUMERICAL;
  b->filled[f] = 1;
  return YGG_OK;
}

// The two add_numerical entries once their bin budget is checked: uploads the column and enqueues its kernels on the
// next lane.  `wide16`: the 16-bit path (up to 65535 bins, uint16 codes kept for finish), else the byte path.
int enqueue_column(ygg_dataset_builder* b, int32_t feature, const float* values, int64_t n_stats_rows,
                   int32_t maximum_num_bins, int32_t min_obs_in_bins, bool wide16) {
  ygg_dataset* ds = b->ds;
  if (min_obs_in_bins < 1) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "min_obs_in_bins < 1");
  if (b->results[feature].status == 1) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "the feature is already in flight");
  const int64_t n = ds->n;
  if (n_stats_rows <= 0 || n_stats_rows > n) n_stats_rows = n;
  YGG_BIN_CUDA(cudaSetDevice(ds->device));
  // a non-sticky error left behind by somebody else's earlier runtime call in this thread (e.g. a framework probing
  // a device ordinal that does not exist) must not be reported as the result of the launches below
  (void)cudaGetLastError();
  BinLane* l = &b->lane[b->next_lane];
  const int lane_id = b->next_lane;
  b->next_lane = (b->next_lane + 1) % kRing;
  if (int st = ensure_lane(b, l)) return st;
  if (wide16)
    if (int st = ensure_lane16(l)) return st;
  if (int st = retire_lane(b, l)) return st;
  drop_codes16(b, feature);
  if (wide16) YGG_BIN_CUDA(cudaMalloc(&b->codes16[feature], sizeof(uint16_t) * (n > 0 ? n : 1)));
  cudaStream_t s = l->stream;
  const int n_tiles = static_cast<int>(b->n_tiles);
  YGG_BIN_CUDA(cudaMemcpyAsync(l->d_values, values, sizeof(float) * n, cudaMemcpyHostToDevice, s));
  YGG_BIN_CUDA(cudaMemsetAsync(l->d_state, 0, sizeof(BinState), s));
  k_bin_keys<<<n_tiles, kSortThreads, 0, s>>>(l->d_values, n, n_stats_rows, l->d_keys[0], l->d_partial, l->d_state);
  int cur = 0;
  for (int pass = 0; pass < 4; pass++) {
    const int shift = 8 * pass;
    k_radix_hist<<<n_tiles, kSortThreads, 0, s>>>(l->d_keys[cur], shift, n_tiles, l->d_table);
    if (int st = launch_scan(l, l->d_table, static_cast<int64_t>(256) * n_tiles, nullptr)) return st;
    k_radix_scatter<<<n_tiles, kSortThreads, 0, s>>>(l->d_keys[cur], l->d_keys[cur ^ 1], shift, n_tiles, l->d_table);
    cur ^= 1;
  }
  const uint32_t* sorted = l->d_keys[cur];
  k_heads_count<<<n_tiles, kSortThreads, 0, s>>>(sorted, l->d_state, l->d_table);
  if (int st = launch_scan(l, l->d_table, n_tiles, l->d_total)) return st;
  k_heads_write<<<n_tiles, kSortThreads, 0, s>>>(sorted, l->d_state, l->d_table, l->d_total, l->d_pos);
  k_bin_prep<<<1, 32, 0, s>>>(sorted, l->d_partial, n_tiles, maximum_num_bins, min_obs_in_bins, l->d_state);
  if (wide16) {
    k_bin_large_count<<<n_tiles, kSortThreads, 0, s>>>(l->d_pos, l->d_state, l->d_table);
    if (int st = launch_scan(l, l->d_table, n_tiles, l->d_total)) return st;
    k_bin_large_write<<<n_tiles, kSortThreads, 0, s>>>(l->d_pos, l->d_state, l->d_table, l->d_total, l->d_large16);
    k_bin_boundaries16<<<1, 32, 0, s>>>(sorted, l->d_pos, l->d_large16, min_obs_in_bins, l->d_state, l->d_cut, l->d_mids);
    k_bin_specials16<<<1, 1024, 0, s>>>(l->d_state, l->d_mids, l->d_tmp16, l->d_bounds16);
    k_bin_encode16<<<ds->num_sms * 8, 256, 0, s>>>(l->d_values, n, l->d_state, l->d_bounds16, b->codes16[feature]);
    YGG_BIN_CUDA(cudaMemcpyAsync(l->h_bounds16, l->d_bounds16, sizeof(float) * kBoundaries16Cap, cudaMemcpyDeviceToHost, s));
  } else {
    k_bin_find_large<<<ds->num_sms * 4, 256, 0, s>>>(l->d_pos, l->d_state, l->d_large);
    k_bin_boundaries<<<1, 32, 0, s>>>(sorted, l->d_pos, l->d_large, min_obs_in_bins, l->d_state, l->d_boundaries);
    k_bin_encode<<<ds->num_sms * 8, 256, 0, s>>>(l->d_values, n, l->d_state, l->d_boundaries,
                                                  ds->d_bins + static_cast<size_t>(feature) * ds->n_pad);
  }
  YGG_BIN_CUDA(cudaGetLastError());
  YGG_BIN_CUDA(cudaMemcpyAsync(&l->h_result->st, l->d_state, sizeof(BinState), cudaMemcpyDeviceToHost, s));
  YGG_BIN_CUDA(cudaMemcpyAsync(l->h_result->bounds, l->d_boundaries, sizeof(float) * 256, cudaMemcpyDeviceToHost, s));
  l->feature = feature;
  ColumnResult& r = b->results[feature];
  r.status = 1;
  r.lane = lane_id;
  r.n_stats = n_stats_rows;
  r.wide16 = wide16;
  b->filled[feature] = 0;
  return YGG_OK;
}

}  // namespace

extern "C" {

int ygg_dataset_builder_create(ygg_dataset_builder** out, int64_t n_rows, int32_t n_features, int32_t device) {
  if (out == nullptr) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "null argument");
  ygg_dataset* ds = nullptr;
  if (int st = ygg_internal_dataset_alloc(&ds, n_rows, n_features, device)) return st;
  auto* b = new ygg_dataset_builder();
  b->ds = ds;
  b->filled.assign(n_features, 0);
  b->results.resize(n_features);
  b->codes16.assign(n_features, nullptr);
  b->n_tiles = (n_rows + kSortTile - 1) / kSortTile;
  *out = b;
  return YGG_OK;
}

int ygg_dataset_builder_add_numerical_async(ygg_dataset_builder* b, int32_t feature, const float* values,
                                            int64_t n_stats_rows, int32_t maximum_num_bins, int32_t min_obs_in_bins) {
  if (!b || !b->ds || !values) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "null argument");
  ygg_dataset* ds = b->ds;
  if (feature < 0 || feature >= ds->F) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "feature index out of range");
  if (maximum_num_bins < 4 || maximum_num_bins > 256)
    return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "maximum_num_bins must be in [4, 256] on the GPU binning path");
  return enqueue_column(b, feature, values, n_stats_rows, maximum_num_bins, min_obs_in_bins, false);
}

int ygg_dataset_builder_add_numerical16_async(ygg_dataset_builder* b, int32_t feature, const float* values,
                                              int64_t n_stats_rows, int32_t maximum_num_bins, int32_t min_obs_in_bins) {
  if (!b || !b->ds || !values) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "null argument");
  ygg_dataset* ds = b->ds;
  if (feature < 0 || feature >= ds->F) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "feature index out of range");
  if (maximum_num_bins < 257 || maximum_num_bins > 65535)
    return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "maximum_num_bins must be in [257, 65535] on the 16-bit GPU binning path");
  return enqueue_column(b, feature, values, n_stats_rows, maximum_num_bins, min_obs_in_bins, true);
}

int ygg_dataset_builder_get_numerical(ygg_dataset_builder* b, int32_t feature, float* out_boundaries, int32_t capacity,
                                      int32_t* out_num_boundaries, double* out_mean, int32_t* out_na_bin,
                                      int64_t* out_num_missing) {
  if (!b || !b->ds) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "null argument");
  if (feature < 0 || feature >= b->ds->F) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "feature index out of range");
  ColumnResult& r = b->results[feature];
  if (r.status == 1) {
    YGG_BIN_CUDA(cudaSetDevice(b->ds->device));
    if (int st = retire_lane(b, &b->lane[r.lane])) return st;
  }
  if (r.status != 0) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "the feature was not binned on the GPU");
  if (out_num_boundaries) *out_num_boundaries = r.st.num_boundaries;
  if (out_boundaries) {
    if (capacity < r.st.num_boundaries) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "boundary buffer too small");
    std::memcpy(out_boundaries, r.wide16 ? r.bounds16.data() : r.bounds, sizeof(float) * r.st.num_boundaries);
  }
  if (out_mean) *out_mean = r.st.mean;
  if (out_na_bin) *out_na_bin = r.st.na_bin;
  if (out_num_missing) *out_num_missing = r.n_stats - static_cast<int64_t>(r.st.n_valid);
  return YGG_OK;
}

int ygg_dataset_builder_add_numerical(ygg_dataset_builder* b, int32_t feature, const float* values,
                                      int64_t n_stats_rows, int32_t maximum_num_bins, int32_t min_obs_in_bins,
                                      float* out_boundaries, int32_t capacity, int32_t* out_num_boundaries,
                                      double* out_mean, int32_t* out_na_bin, int64_t* out_num_missing) {
  if (int st = ygg_dataset_builder_add_numerical_async(b, feature, values, n_stats_rows, maximum_num_bins, min_obs_in_bins))
    return st;
  return ygg_dataset_builder_get_numerical(b, feature, out_boundaries, capacity, out_num_boundaries, out_mean,
                                           out_na_bin, out_num_missing);
}

int ygg_dataset_builder_add_bins(ygg_dataset_builder* b, int32_t feature, const uint8_t* bins, int32_t num_bins,
                                 int32_t na_bin, int32_t feature_type) {
  if (!b || !b->ds || !bins) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "null argument");
  ygg_dataset* ds = b->ds;
  if (feature < 0 || feature >= ds->F) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "feature index out of range");
  if (num_bins < 1 || num_bins > 256 || na_bin < 0 || na_bin >= num_bins)
    return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "num_bins outside [1, 256] or na_bin outside [0, num_bins)");
  if (feature_type != YGG_FEATURE_DISCRETIZED_NUMERICAL && feature_type != YGG_FEATURE_CATEGORICAL)
    return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "unknown feature type");
  if (b->results[feature].status == 1) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "the feature is in flight");
  YGG_BIN_CUDA(cudaSetDevice(ds->device));
  YGG_BIN_CUDA(cudaMemcpy(ds->d_bins + static_cast<size_t>(feature) * ds->n_pad, bins, ds->n, cudaMemcpyHostToDevice));
  drop_codes16(b, feature);
  ds->num_bins[feature] = num_bins;
  ds->na_bin[feature] = na_bin;
  ds->feature_type[feature] = feature_type;
  b->results[feature].status = -1;
  b->filled[feature] = 1;
  return YGG_OK;
}

int ygg_dataset_builder_finish(ygg_dataset_builder* b, ygg_dataset** out) {
  if (!b || !b->ds || !out) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "null argument");
  YGG_BIN_CUDA(cudaSetDevice(b->ds->device));
  for (BinLane& l : b->lane)
    if (int st = retire_lane(b, &l)) return st;
  for (size_t f = 0; f < b->filled.size(); f++)
    if (!b->filled[f]) {
      char m[96];
      std::snprintf(m, sizeof(m), "feature %zu was never added to the builder", f);
      return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, m);
    }
  if (int st = ygg_internal_dataset_finalize(b->ds)) return st;
  int n16 = 0;
  for (const uint16_t* c : b->codes16) n16 += c != nullptr ? 1 : 0;
  if (n16 > 0)   // one allocation for all of them, then each attach copies one plane
    if (int st = ygg_internal_reserve_wide(b->ds, b->ds->n_wide() + n16)) return st;
  for (int f = 0; f < b->ds->F; f++) {   // the 16-bit columns with more than 256 bins
    if (b->codes16[f] == nullptr) continue;
    const ColumnResult& r = b->results[f];
    if (int st = ygg_internal_attach_wide_discretized(b->ds, f, b->codes16[f], r.st.num_boundaries + 1, r.st.na_bin)) return st;
    drop_codes16(b, f);
  }
  *out = b->ds;
  b->ds = nullptr;  // ownership moves to the caller
  free_builder(b);
  return YGG_OK;
}

int ygg_dataset_builder_destroy(ygg_dataset_builder* b) {
  free_builder(b);
  return YGG_OK;
}

int ygg_dataset_get_bins(const ygg_dataset* ds, int32_t feature, uint8_t* out) {
  if (!ds || !out || feature < 0 || feature >= ds->F) return ygg_set_error_msg(YGG_ERR_INVALID_ARGUMENT, "bad argument");
  YGG_BIN_CUDA(cudaSetDevice(ds->device));
  YGG_BIN_CUDA(cudaMemcpy(out, ds->d_bins + static_cast<size_t>(feature) * ds->n_pad, ds->n, cudaMemcpyDeviceToHost));
  return YGG_OK;
}

}  // extern "C"
