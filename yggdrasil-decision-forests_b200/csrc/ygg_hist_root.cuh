// ygg_hist_root.cuh — k_hist_root_rows: the root level's histogram from the row-major copy of the bins, lanes = features.
//
// k_hist<false, kHistRootSum> streams the column-major matrix with lanes = rows: the 32 atomics of a warp instruction add
// into random bins of one feature, and every returning ATOMS replays as several wavefronts (DESIGN.md §5).  Here a warp
// reads one row at a time from the row-major copy (k_bins_to_rows, ygg_hist_seg.cuh): lane l loads the 4 adjacent bytes
// 4l..4l+3 of the row's 128-byte segment of the group (one coalesced request of 4 sectors per row and group), and the
// histogram is [bin][feature in lane][lane], so every atomic of a warp instruction hits bank = lane.
// Work item = (chunk of consecutive row blocks) x (group of 32 lanes x kRootFpl = 128 features; groups start at the
// multiple of 4 at or below the shard's first feature: seg_feature_groups).  Columns outside the shard (the group's
// leading bytes, the row's zero padding, lanes past the shard that re-read its last word) are accumulated and dropped.
// The root layout: sums only (the counts are the dataset's, precomputed: d_root_cnt), one returning atomic per element on
// the low word of the sum; a carry seen in the returned value goes to a 16-bit carry counter (two per 32-bit word) with
// a rare RED.  A chunk of at most kRootRowsMaxChunkBlocks blocks has at most 2^24 rows, so a column's carries stay
// below 2^24 * (2^24 - 1) / 2^32 < 2^16: the flush rebuilds the exact sum as carries << 32 | low.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "ygg_device.cuh"
#include "ygg_hist.cuh"
#include "ygg_hist_seg.cuh"

namespace ygg {

constexpr int kRootThreads = 1024;
constexpr int kRootLanes = 32;
constexpr int kRootFpl = 4;                                  // features per lane
constexpr int kRootFeatures = kRootLanes * kRootFpl;         // features per work item
constexpr int kRootRowsPerWarp = 8;                          // rows per warp iteration (loaded one iteration ahead)
constexpr int kRootRowsMaxChunkBlocks = 2048;                // 2^24 rows: < 2^16 carries per column
static_assert(static_cast<unsigned long long>(kRootRowsMaxChunkBlocks) * kBlockRows * kQMax >> 32 < (1ull << 16),
              "the 16-bit carry counters of a chunk");
// Shared memory: 32-bit low words [256][FPL][32] and 16-bit carries [256][FPL][32] (192 KB).
constexpr size_t kRootSmemBytes = static_cast<size_t>(kMaxBins) * kRootFeatures * (4 + 2);

struct RootRowsParams {
  const uint8_t* rows;          // [n_pad][row_bytes]
  uint32_t row_bytes;
  const uint32_t* q24;          // [n_pad] quantised gradient of every row
  const int32_t* act_count;     // [n_blocks] rows of each block accumulated at the root (a prefix of the block)
  int n_blocks, chunk_blocks;
  int f_begin, f_count;         // this shard's features
  unsigned long long* hist_sum; // as HistParams (slot 0)
  int f_chunk;
  long long chunk_stride;
};

__device__ __forceinline__ uint32_t ldg_row_word(const uint8_t* p) {
  return __ldg(reinterpret_cast<const uint32_t*>(p));
}

__global__ void __launch_bounds__(kRootThreads, 1) k_hist_root_rows(RootRowsParams p) {
  constexpr int kWarps = kRootThreads / 32;
  constexpr int U = kRootRowsPerWarp;
  constexpr uint32_t kSumWords = kMaxBins * kRootFeatures;
  extern __shared__ __align__(16) uint32_t s_sum[];   // word (bin*FPL + k)*32 + lane; then the carry words
  uint32_t* s_carry = s_sum + kSumWords;              // word ((bin*FPL + k)*32 + lane) / 2, lane parity = half
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t s_base = static_cast<uint32_t>(__cvta_generic_to_shared(s_sum));
  asm volatile("mov.u32 %0, %0;" : "+r"(s_base));   // (see k_hist)
  const uint32_t a_lane = s_base + static_cast<uint32_t>(lane) * 4u;
  const uint32_t c_lane = s_base + kSumWords * 4u + static_cast<uint32_t>(lane >> 1) * 4u;
  const uint32_t c_inc = 1u << (16 * (lane & 1));
  const int off = p.f_begin & (kRootFpl - 1);
  const int n_fg = seg_feature_groups(kRootLanes, kRootFpl, p.f_begin, p.f_count);
  const int n_chunks = (p.n_blocks + p.chunk_blocks - 1) / p.chunk_blocks;
  const int n_items = n_chunks * n_fg;
  for (int i = tid; i < static_cast<int>(kRootSmemBytes / 4); i += kRootThreads) s_sum[i] = 0u;
  __syncthreads();

  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int chunk = item / n_fg, fg = item - chunk * n_fg;
    const int f0 = fg * kRootFeatures - off;            // shard feature of the group's column 0
    const int last = min(kRootFeatures, p.f_count - f0) - 1;
    // lanes past the group's last column re-read its word: no load leaves the row
    const uint8_t* col = p.rows + p.f_begin + f0 + min(lane * kRootFpl, last & ~(kRootFpl - 1));
    const int64_t r0 = static_cast<int64_t>(chunk) * p.chunk_blocks * kBlockRows;
    const int64_t r1 = min(static_cast<int64_t>(p.n_blocks), static_cast<int64_t>(chunk + 1) * p.chunk_blocks) * kBlockRows;

    // A warp takes U consecutive rows per iteration (never across a block: U divides kBlockRows), their words and gradients
    // loaded one iteration ahead; the gradients are one broadcast load per 4 rows.  Rows past the block's count add 0.
    uint32_t w[U];
    uint4 qv[U / 4];
    int cnt = 0;
    auto load = [&](int64_t r) {
      if (r < r1) {
#pragma unroll
        for (int u = 0; u < U; u++) w[u] = ldg_row_word(col + static_cast<size_t>(r + u) * p.row_bytes);
#pragma unroll
        for (int v = 0; v < U / 4; v++) qv[v] = __ldg(reinterpret_cast<const uint4*>(p.q24 + r) + v);
        cnt = __ldg(p.act_count + (r / kBlockRows));
      }
    };
    int64_t r = r0 + static_cast<int64_t>(warp) * U;
    load(r);
    for (; r < r1; r += static_cast<int64_t>(kWarps) * U) {
      uint32_t wc[U], q[U];
#pragma unroll
      for (int u = 0; u < U; u++) wc[u] = w[u];
#pragma unroll
      for (int v = 0; v < U / 4; v++) {
        q[4 * v] = qv[v].x; q[4 * v + 1] = qv[v].y; q[4 * v + 2] = qv[v].z; q[4 * v + 3] = qv[v].w;
      }
      const int in_block = static_cast<int>(r & (kBlockRows - 1));
#pragma unroll
      for (int u = 0; u < U; u++) q[u] = in_block + u < cnt ? q[u] : 0u;
      load(r + static_cast<int64_t>(kWarps) * U);
#pragma unroll
      for (int u = 0; u < U; u += 2) {
        uint32_t a[2 * kRootFpl], old[2 * kRootFpl];
#pragma unroll
        for (int j = 0; j < 2; j++)
#pragma unroll
          for (int k = 0; k < kRootFpl; k++)
            a[j * kRootFpl + k] = a_lane + static_cast<uint32_t>(k) * 128u + (((wc[u + j] >> (8 * k)) & 0xFFu) << 9);
#pragma unroll
        for (int j = 0; j < 2; j++)
#pragma unroll
          for (int k = 0; k < kRootFpl; k++) old[j * kRootFpl + k] = smem_add(a[j * kRootFpl + k], q[u + j]);
        bool carry = false;
#pragma unroll
        for (int j = 0; j < 2; j++)
#pragma unroll
          for (int k = 0; k < kRootFpl; k++) carry |= old[j * kRootFpl + k] + q[u + j] < old[j * kRootFpl + k];
        if (carry) {
#pragma unroll
          for (int j = 0; j < 2; j++)
#pragma unroll
            for (int k = 0; k < kRootFpl; k++)
              if (old[j * kRootFpl + k] + q[u + j] < old[j * kRootFpl + k])
                smem_red(c_lane + ((a[j * kRootFpl + k] - a_lane) >> 1), c_inc);
        }
      }
    }
    __syncthreads();

    // Flush the non-empty bins of the group's shard columns and zero every word for the next item, tiled as k_hist_seg's
    // flush: lane (tr, tq) takes bin tr of a tile of 8 bins and the 4 adjacent words of lanes 4tq'..4tq'+3 of one feature
    // in lane, so that the 8 lanes holding one column cover 8 consecutive bins of the global [feature][bin] plane.
    constexpr int TB = 8, QL = 4;
    constexpr int kQuadGroups = kRootLanes / (4 * QL);                 // 2
    constexpr int kTiles = kMaxBins / TB * kRootFpl * kQuadGroups;     // 256
    const int tr = lane / QL, tq = lane % QL;
    for (int t = warp; t < kTiles; t += kWarps) {
      const int bin = t / (kRootFpl * kQuadGroups) * TB + tr;
      const int k = t / kQuadGroups % kRootFpl;
      const int l0 = (t % kQuadGroups * QL + tq) * 4;                  // first of the 4 lanes
      const int wi = (bin * kRootFpl + k) * kRootLanes + l0;
      uint4* sw = reinterpret_cast<uint4*>(s_sum + wi);
      uint2* cw = reinterpret_cast<uint2*>(s_carry + wi / 2);
      const uint4 lo4 = *sw;
      const uint2 c2 = *cw;
      *sw = make_uint4(0u, 0u, 0u, 0u);
      *cw = make_uint2(0u, 0u);
      const uint32_t los[4] = {lo4.x, lo4.y, lo4.z, lo4.w};
      const uint32_t cs[4] = {c2.x & 0xFFFFu, c2.x >> 16, c2.y & 0xFFFFu, c2.y >> 16};
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int f = f0 + (l0 + j) * kRootFpl + k;    // its shard feature
        const unsigned long long sum = static_cast<unsigned long long>(cs[j]) << 32 | los[j];
        if (sum == 0ull || f < 0 || f >= p.f_count) continue;
        size_t oc;
        atomicAdd(&p.hist_sum[slot_hist_offset(0, f, bin, p.f_chunk, p.chunk_stride, &oc)], sum);
      }
    }
    __syncthreads();
  }
}

}  // namespace ygg
