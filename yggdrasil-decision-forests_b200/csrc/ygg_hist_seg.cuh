// ygg_hist_seg.cuh — k_hist_seg: the level histograms of the deep tree levels (and of levels 1-2 on wide, large shards),
// one node's rows per work item.
//
// k_hist streams the whole column-major matrix at every level and keeps all S slots of a level in one CTA's shared
// memory; below level 2 a level accumulates ~30 % of the rows, and S pushes its feature group G down to 2-5.  Here:
//   rows[r][f]     a row-major copy of the bins, u8 [n_pad][row_bytes] (seg_row_bytes: F rounded up to a power of two
//                  from 32 to 256, zero padding), so that 32 consecutive features of a row are one 32-byte sector and a
//                  row one aligned region of at most 256 bytes (k_bins_to_rows, built on first use);
//   seg[k]         the level's active-list entries (q24 | slot << 24, global row), grouped by slot and, inside a slot, in
//                  (row block, row) order (k_seg_count, cub's inclusive scan, k_seg_ranges, k_seg_scatter, from the
//                  per-block lists d_act);
//   seg_off[r]     start of range r = slot * n_chunks + chunk (chunk = `chunk_blocks` consecutive row blocks), [R + 1].
// Work item = (piece of one range of at most P entries) x (group of FL x FPL features: FPL features per lane, 1 or 2).
// A CTA holds ONE slot of the group in shared memory, [bin][plane][half][lane] packed words as kHistPacked
// (ygg_hist.cuh), so that at 32 lanes every atomic of a warp instruction hits bank = lane.  A warp gathers, per row, FPL
// adjacent bytes per lane: FPL = 1 is one 32-byte sector per row and group, FPL = 2 (FL = 32, shards of more than 32
// features) two sectors in ONE load request, the requests per row halved.  A paired group starts at an even byte of the
// row (the shard's first feature rounded down) so that every 2-byte load is aligned; its columns outside the shard are
// accumulated and dropped.
// A piece is a subset of one (slot, chunk) range, and a chunk's rows give every bin at most as many updates as the
// chunk_max_count bound checks: the packed words stay exact.  Pieces are taken from a work counter (slot sizes
// differ a lot); the feature groups of a piece are consecutive items, so their CTAs read the same rows at about the same
// time and a row's other sectors come from L2 (ldg_row).
#pragma once
#include <cstdint>
#include <type_traits>
#include <cub/block/block_scan.cuh>
#include <cuda_runtime.h>

#include "ygg_device.cuh"
#include "ygg_hist.cuh"

namespace ygg {

constexpr int kSegThreads = 1024;
constexpr int kSegMinBlocks = 1;       // CTAs per SM (<= 64 registers: 32 gathers in flight per lane)
constexpr int kSegMinSlots = 4;        // level slot bound from which the planner takes k_hist_seg (DESIGN.md §5)
// Levels 1 and 2 (one or two slots) take k_hist_seg on shards of at least this many features and rows x features
// (measured on C3-shaped data, DESIGN.md §5): per added row it costs as much as k_hist at 100 features and less from 128
// on, and the whole-matrix stream it saves pays for its grouping pass from ~0.8e9 elements on (200 features: 4M rows
// break even).
constexpr int kSegShallowMinFeatures = 128;
constexpr long long kSegShallowMinElements = 1000000000LL;
constexpr int kSegItemsPerCta = 4;     // target work items per CTA: sets the piece size P
constexpr int kSegMinPiece = 4096;     // smallest P: the flush of FL x FPL x 256 bins stays small against the piece
constexpr int kSegMaxSlots = 256;      // slots the pass handles (the entries carry 8-bit slots)
constexpr int kSegScanThreads = 512;

// Features per lane of a launch with FL lanes over a shard of f_count features: two at 32 lanes above 32 features.
inline int seg_lane_features(int FL, int f_count) { return FL == 32 && f_count > 32 ? 2 : 1; }
// Level slot bound from which the planner takes k_hist_seg for a shard of f_count features over `rows` rows: every
// level below the root on wide, large shards (paired form), kSegMinSlots otherwise.
inline int seg_min_slots(int f_count, long long rows) {
  return f_count >= kSegShallowMinFeatures && rows * f_count >= kSegShallowMinElements ? 1 : kSegMinSlots;
}
// Shared memory of a work item of FI = FL x FPL features.
__host__ __device__ inline size_t seg_smem_bytes(int FI) { return static_cast<size_t>(kMaxBins) * 2 * FI * 4; }
// Feature groups of a shard: FPL = 2 (4) starts its groups at the byte at or below the shard's first feature that is a
// multiple of 2 (4), so that every lane's FPL-byte load is aligned.
__host__ __device__ inline int seg_feature_groups(int FL, int FPL, int f_begin, int f_count) {
  const int off = f_begin & (FPL - 1);
  return (f_count + off + FL * FPL - 1) / (FL * FPL);
}
// Bytes per row of the row-major copy: the power of two >= F from 32 to 256 (a row is one aligned region of at most
// 256 bytes: ldg_row), above 256 features a multiple of 256.
inline int seg_row_bytes(int F) {
  int b = 32;
  while (b < F && b < 256) b *= 2;
  return b >= F ? b : (F + 255) / 256 * 256;
}

// rows[r][f] = bins[f][r]; bytes of features >= F are zero.  CTA = 256 rows x 32 features; a thread writes one row's
// 32-byte sector.
__global__ void __launch_bounds__(256) k_bins_to_rows(const uint8_t* bins, int64_t n_pad, int F, int row_bytes, uint8_t* rows) {
  const int64_t r = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x;
  const int f0 = blockIdx.y * 32;
  if (r >= n_pad) return;
  uint32_t w[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
#pragma unroll
  for (int k = 0; k < 32; k++) {
    const int f = f0 + k;
    const uint32_t v = f < F ? bins[static_cast<int64_t>(f) * n_pad + r] : 0u;
    w[k >> 2] |= v << (8 * (k & 3));
  }
  uint4* dst = reinterpret_cast<uint4*>(rows + r * row_bytes + f0);
  dst[0] = make_uint4(w[0], w[1], w[2], w[3]);
  dst[1] = make_uint4(w[4], w[5], w[6], w[7]);
}

// Entries of slots >= the level's num_slots are skipped by the pass (k_hist accumulates them into bins it never flushes).
__device__ __forceinline__ uint32_t seg_slot_of(uint2 e, bool valid, uint32_t ns) {
  const uint32_t slot = e.x >> 24;
  return (valid && slot < ns) ? slot : 0xFFFFFFFFu;
}

// Per (slot, row block): active rows of the level, blk[slot * n_blocks + block] for slots [0, S).  One CTA per block;
// a warp adds the lanes of one slot with one shared-memory add (match.any: a level has few slots, plain atomics would
// serialise on them).
__global__ void __launch_bounds__(256) k_seg_count(const uint2* act, const int32_t* act_count, int n_blocks, int S,
                                                   const LevelDesc* levels, int level, long long* blk) {
  __shared__ int c[kSegMaxSlots];
  const uint32_t ns = static_cast<uint32_t>(min(S, levels[level].num_slots));
  const int lane = threadIdx.x & 31;
  for (int b = blockIdx.x; b < n_blocks; b += gridDim.x) {
    for (int i = threadIdx.x; i < S; i += blockDim.x) c[i] = 0;
    __syncthreads();
    const int n = act_count[b];
    const uint2* a = act + static_cast<int64_t>(b) * kBlockRows;
    for (int i0 = threadIdx.x & ~31; i0 < n; i0 += blockDim.x) {
      const int i = i0 + lane;
      const uint32_t slot = seg_slot_of(i < n ? __ldg(a + i) : make_uint2(0u, 0u), i < n, ns);
      const uint32_t mask = __match_any_sync(0xFFFFFFFFu, slot);
      if (slot != 0xFFFFFFFFu && (mask & ((1u << lane) - 1u)) == 0u) atomicAdd(&c[slot], __popc(mask));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < S; i += blockDim.x) blk[static_cast<size_t>(i) * n_blocks + b] = c[i];
    __syncthreads();
  }
}

// After the inclusive scan of blk in slot-major order (cub, in place): one CTA computes the ranges' starts
// seg_off[S * n_chunks + 1], the piece size P = max(kSegMinPiece, ceil(total / target_pieces)), each range's first piece
// piece_start[R + 1], and meta = {P, pieces, work counter = 0}.
__global__ void __launch_bounds__(kSegScanThreads) k_seg_ranges(const long long* incl, int S, int n_blocks, int chunk_blocks,
                                                                int n_chunks, int target_pieces, long long* seg_off,
                                                                int32_t* piece_start, int32_t* meta) {
  using Scan = cub::BlockScan<long long, kSegScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const int tid = threadIdx.x;
  const int R = S * n_chunks;
  const long long total = incl[static_cast<size_t>(S) * n_blocks - 1];
  for (int r = tid; r < R; r += kSegScanThreads) {
    const int s = r / n_chunks, c = r - s * n_chunks;
    const size_t i = static_cast<size_t>(s) * n_blocks + static_cast<size_t>(c) * chunk_blocks;
    seg_off[r] = i == 0 ? 0 : incl[i - 1];
  }
  if (tid == 0) seg_off[R] = total;
  const long long P = max(static_cast<long long>(kSegMinPiece), (total + target_pieces - 1) / target_pieces);
  __syncthreads();
  const int per = (R + kSegScanThreads - 1) / kSegScanThreads;
  const int r0 = min(R, tid * per), r1 = min(R, r0 + per);
  long long pieces = 0;
  for (int r = r0; r < r1; r++) pieces += (seg_off[r + 1] - seg_off[r] + P - 1) / P;
  long long first = 0, n_pieces = 0;
  Scan(tmp).ExclusiveSum(pieces, first, n_pieces);
  for (int r = r0; r < r1; r++) {
    piece_start[r] = static_cast<int32_t>(first);
    first += (seg_off[r + 1] - seg_off[r] + P - 1) / P;
  }
  if (tid == 0) {
    piece_start[R] = static_cast<int32_t>(n_pieces);
    meta[0] = static_cast<int32_t>(P);
    meta[1] = static_cast<int32_t>(n_pieces);
    meta[2] = 0;
  }
}

// One CTA per row block: its entries, in list order, to their slots' places in seg.  The 8 warps take consecutive parts
// of the block's list: each counts its part's slots, the parts' cursors follow from those counts, then each warp
// scatters its part, 32 entries at a time, the lanes of one slot at consecutive places in lane order (match.any).
__global__ void __launch_bounds__(256) k_seg_scatter(const uint2* act, const int32_t* act_count, int n_blocks, int S,
                                                     const LevelDesc* levels, int level, const long long* incl, uint2* seg) {
  __shared__ int cnt[8][kSegMaxSlots];
  __shared__ long long cur[8][kSegMaxSlots];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t ns = static_cast<uint32_t>(min(S, levels[level].num_slots));
  const uint32_t lt = (1u << lane) - 1u;
  for (int b = blockIdx.x; b < n_blocks; b += gridDim.x) {
    for (int s = lane; s < static_cast<int>(ns); s += 32) cnt[warp][s] = 0;
    __syncwarp();
    const int n = act_count[b];
    const int part = (n + 8 * 32 - 1) / (8 * 32) * 32;
    const int e0 = min(n, warp * part), e1 = min(n, e0 + part);
    const uint2* a = act + static_cast<int64_t>(b) * kBlockRows;
    for (int i0 = e0; i0 < e1; i0 += 32) {
      const int i = i0 + lane;
      const uint32_t slot = seg_slot_of(i < e1 ? __ldg(a + i) : make_uint2(0u, 0u), i < e1, ns);
      const uint32_t mask = __match_any_sync(0xFFFFFFFFu, slot);
      if (slot != 0xFFFFFFFFu && (mask & lt) == 0u) cnt[warp][slot] += __popc(mask);
      __syncwarp();
    }
    __syncthreads();
    for (int s = threadIdx.x; s < static_cast<int>(ns); s += blockDim.x) {
      const size_t gi = static_cast<size_t>(s) * n_blocks + b;
      long long o = gi == 0 ? 0 : incl[gi - 1];
#pragma unroll
      for (int w = 0; w < 8; w++) {
        cur[w][s] = o;
        o += cnt[w][s];
      }
    }
    __syncthreads();
    const uint32_t row0 = static_cast<uint32_t>(b) * kBlockRows;
    for (int i0 = e0; i0 < e1; i0 += 32) {
      const int i = i0 + lane;
      const uint2 e = i < e1 ? __ldg(a + i) : make_uint2(0u, 0u);
      const uint32_t slot = seg_slot_of(e, i < e1, ns);
      const uint32_t mask = __match_any_sync(0xFFFFFFFFu, slot);
      const int rank = __popc(mask & lt);
      long long o = 0;
      if (slot != 0xFFFFFFFFu) o = cur[warp][slot];
      __syncwarp();
      if (slot != 0xFFFFFFFFu && rank == 0) cur[warp][slot] = o + __popc(mask);
      __syncwarp();
      if (slot != 0xFFFFFFFFu) seg[o + rank] = make_uint2(e.x, row0 + e.y);
    }
    __syncthreads();
  }
}

// One byte (FPL = 1) or two aligned bytes (FPL = 2, the first in bits 0-7) of a row, with a hint to fetch the row's whole
// aligned 256-byte region into L2: the other feature groups of the row are read by the CTAs of the piece's other items at
// about the same time, so a row costs one 256-byte DRAM access instead of one sector access per feature group.
template <int FPL>
__device__ __forceinline__ uint32_t ldg_row(const uint8_t* p) {
  uint32_t v;
  if constexpr (FPL == 2) asm("ld.global.nc.L2::256B.u16 %0, [%1];" : "=r"(v) : "l"(p));
  else asm("ld.global.nc.L2::256B.u8 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}

struct SegParams {
  const uint8_t* rows;          // [n_pad][row_bytes]
  uint32_t row_bytes;
  const uint2* seg;
  const long long* seg_off;     // [n_ranges + 1]
  const int32_t* piece_start;   // [n_ranges + 1]
  int32_t* meta;                // P, pieces, work counter (k_seg_ranges)
  int n_ranges, n_chunks;
  int f_begin, f_count;         // this shard's features
  unsigned long long* hist_sum; // as HistParams
  uint32_t* hist_cnt;
  int f_chunk;
  long long chunk_stride;
};

template <int FL, int FPL>
__global__ void __launch_bounds__(kSegThreads, kSegMinBlocks) k_hist_seg(SegParams p) {
  static_assert(FL == 8 || FL == 16 || FL == 32, "feature lanes");
  static_assert(FPL == 1 || (FPL == 2 && FL == 32), "two features per lane at 32 lanes only");
  constexpr int FI = FL * FPL;             // features per work item
  constexpr int R = 32 / FL;               // rows per warp step (FL < 32: few features)
  constexpr int kSteps = 32 / R;           // rows per lane per warp iteration of 32 entries
  constexpr int kInFlight = FL == 32 ? 32 : 8;   // gathers issued before their atomics (within 64 registers)
  constexpr int kWarps = kSegThreads / 32;
  constexpr int kWords = kMaxBins * 2 * FI;
  constexpr uint32_t kBinBytes = 2u * FI * 4u, kPlaneBytes = FI * 4u, kHalfBytes = FL * 4u;
  extern __shared__ __align__(16) uint32_t s_bins[];   // word ((bin*2 + plane)*FPL + half)*FL + lane
  __shared__ int s_item;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int fl = lane % FL, sub = lane / FL;
  uint32_t s_base = static_cast<uint32_t>(__cvta_generic_to_shared(s_bins));
  asm volatile("mov.u32 %0, %0;" : "+r"(s_base));   // (see k_hist)
  // FPL = 2: the groups start at the even byte f_begin - off of the row, column 0 of the first group is feature -off
  const int off = FPL == 2 ? (p.f_begin & 1) : 0;
  const int n_fg = seg_feature_groups(FL, FPL, p.f_begin, p.f_count);
  const int P = p.meta[0];
  const int n_items = p.meta[1] * n_fg;
  for (int i = tid; i < kWords; i += kSegThreads) s_bins[i] = 0u;
  const uint32_t a_lane = s_base + static_cast<uint32_t>(fl) * 4u;
  for (;;) {
    if (tid == 0) s_item = atomicAdd(&p.meta[2], 1);
    __syncthreads();
    const int item = s_item;
    if (item >= n_items) break;
    const int piece = item / n_fg, fg = item - piece * n_fg;
    int lo = 0, hi = p.n_ranges;   // piece_start[lo] <= piece < piece_start[hi]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (__ldg(p.piece_start + mid) <= piece) lo = mid;
      else hi = mid;
    }
    const long long beg = __ldg(p.seg_off + lo) + static_cast<long long>(piece - __ldg(p.piece_start + lo)) * P;
    const int len = static_cast<int>(min(static_cast<long long>(P), __ldg(p.seg_off + lo + 1) - beg));
    const int slot = lo / p.n_chunks;
    const int f0 = fg * FI - off;                     // shard feature of the group's column 0
    const int last = min(FI, p.f_count - f0) - 1;     // the group's last column inside the shard
    // lanes past it re-read its last feature (pair): no load leaves the row (a pair ending at an odd byte < row_bytes)
    const uint8_t* col = p.rows + p.f_begin + f0 + min(fl * FPL, last & ~(FPL - 1));
    const uint2* sp = p.seg + beg;

    // A warp takes 32 entries at a time, one per lane (coalesced, loaded one iteration ahead), and issues the gathers of
    // their rows before their atomics (32 in flight per lane at FL = 32).  x = q | 1 << 31 for a row of the piece, 0
    // past its end (row 0, adding nothing): w0 += coarse << 13 | valid, w1 += q, in the word of each gathered byte.
    int e = warp * 32;
    uint2 cur = e + lane < len ? __ldg(sp + e + lane) : make_uint2(0u, 0u);
    for (; e < len; e += kWarps * 32) {
      const int en = e + kWarps * 32 + lane;
      const uint2 nxt = en < len ? __ldg(sp + en) : make_uint2(0u, 0u);
      const uint32_t xq = e + lane < len ? ((cur.x & kQMax) | 0x80000000u) : 0u;
#pragma unroll
      for (int j0 = 0; j0 < kSteps; j0 += kInFlight) {
        uint32_t b[kInFlight];
#pragma unroll
        for (int j = 0; j < kInFlight; j++) {
          const uint32_t row = __shfl_sync(0xFFFFFFFFu, cur.y, (j0 + j) * R + sub);
          b[j] = ldg_row<FPL>(col + static_cast<size_t>(row) * p.row_bytes);
        }
#pragma unroll
        for (int j = 0; j < kInFlight; j++) {
          const uint32_t x = __shfl_sync(0xFFFFFFFFu, xq, (j0 + j) * R + sub);
          const uint32_t inc = (((x >> kPackedCoarseShift) & 0x3Fu) << kPackedCntBits) | (x >> 31), q = x & kQMax;
          const uint32_t a = a_lane + (FPL == 2 ? b[j] & 0xFFu : b[j]) * kBinBytes;
          smem_red(a, inc);
          smem_red(a + kPlaneBytes, q);
          if constexpr (FPL == 2) {
            const uint32_t a1 = a_lane + kHalfBytes + (b[j] >> 8) * kBinBytes;
            smem_red(a1, inc);
            smem_red(a1 + kPlaneBytes, q);
          }
        }
      }
      cur = nxt;
    }
    __syncthreads();

    // flush the non-empty bins of the group's features and zero every word for the next item.  A column of the shard
    // receives <= 8191 updates, so its count is 0 only when both its words are; the others (re-read features, FPL = 2:
    // the shard's neighbours and the row's zero padding) may receive any number and are cleared, never flushed.
    // The global planes are [slot][feature][bin]: a warp instruction whose lanes hold TB consecutive bins of each of QL
    // features reduces into QL x 2 sectors of sums and QL x 1 of counts (TB = 8), where one lane per feature (the
    // shared layout's order) touched 32 sectors of each.  Lane (r, q) takes bin r of a tile of TB bins and the 4 adjacent
    // columns 4q..4q+3 (one half of a lane pair, FL % 4 == 0) of both planes with two 16-byte loads: the 8 lanes of a
    // quarter-warp (one 16-byte access phase) cover 8 / QL bins x 4 QL columns, a 2-way bank conflict.
    constexpr int QL = FI >= 16 ? 4 : 2;                // column quads per tile
    constexpr int TB = 32 / QL;                         // bins per tile
    constexpr int kQuadGroups = FI / (4 * QL);
    constexpr int kTiles = kMaxBins / TB * kQuadGroups;
    const int tr = lane / QL, tq = lane % QL;
    for (int t = warp; t < kTiles; t += kWarps) {
      const int bin = t / kQuadGroups * TB + tr;
      const int k0 = (t % kQuadGroups * QL + tq) * 4;  // k = half * FL + lane
      uint4* w = reinterpret_cast<uint4*>(s_bins + bin * 2 * FI + k0);
      const uint4 c4 = w[0], l4 = w[FI / 4];
      w[0] = make_uint4(0u, 0u, 0u, 0u);
      w[FI / 4] = make_uint4(0u, 0u, 0u, 0u);
      const uint32_t cs[4] = {c4.x, c4.y, c4.z, c4.w}, ls[4] = {l4.x, l4.y, l4.z, l4.w};
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int k = k0 + j;
        const int f = f0 + (k % FL) * FPL + k / FL;   // its shard feature
        const uint32_t c = cs[j];
        if (c == 0u || f < 0 || f >= p.f_count) continue;
        size_t oc;
        const size_t o = slot_hist_offset(slot, f, bin, p.f_chunk, p.chunk_stride, &oc);
        const unsigned long long base = static_cast<unsigned long long>(c >> kPackedCntBits) << kPackedCoarseShift;
        atomicAdd(&p.hist_sum[o], base + static_cast<uint32_t>(ls[j] - static_cast<uint32_t>(base)));
        atomicAdd(&p.hist_cnt[oc], c & kPackedMaxUpdates);
      }
    }
  }
}

}  // namespace ygg
