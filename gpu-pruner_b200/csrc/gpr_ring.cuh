// gpr_ring.cuh — the resident ring of daemon mode: a tick's columns scattered into the time ring, buckets opened
// without data, and the optional block-maxima index (GPR_F_BLOCK_INDEX) kept in step with both.
//
// The kernels here are plain CUDA C++ without inline PTX, and the host-side arithmetic of gpr_append /
// gpr_resident_advance (which source columns survive, where they land, what each plane gets, the grid, the index
// row length) is plain functions.  gpr_api.cu launches what these return; tests/cpp/ring_emul.cpp runs the same
// source on the CPU against a numpy model of the ring.  gpr_resident_remap's row gather and map check are here too
// (tests/cpp/remap_emul.cpp), gpr_resident_live_rows' row test (tests/cpp/live_rows_emul.cpp) and gpr_resident_cols'
// band gather (tests/cpp/ring_cols_emul.cpp), and gpr_resident_retime's regrouping of the newest buckets
// (tests/cpp/retime_emul.cpp).
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "gpr_kernels.cuh"

namespace gpr {

constexpr uint32_t kIdxBlock = 64;               // ring samples per index block
constexpr uint32_t kRingThreads = 128;           // block size of k_append / k_open / k_reindex
constexpr uint32_t kNoSampleBits = 0xFFFFFFFFu;  // a NaN: what gpr_resident_init and k_fill_columns store

// n_new columns appended at ring position `head` of a ring of T.  Only the newest T of them can survive: source
// columns [src_col, src_col + n) land at ring positions (start + j) % T, and the head moves on to next_head.
struct RingSpan {
  uint32_t src_col, n, start, next_head;
};

inline RingSpan ring_span(uint32_t head, uint32_t n_new, uint32_t T) {
  RingSpan s;
  s.src_col = n_new > T ? n_new - T : 0u;
  s.n = n_new - s.src_col;
  s.start = (uint32_t)(((uint64_t)head + s.src_col) % T);
  s.next_head = (uint32_t)(((uint64_t)head + n_new) % T);
  return s;
}

// What one resident plane gets from gpr_append / gpr_resident_advance.
enum RingLaunch {
  kRingNone = 0,     // the ring has no such plane
  kRingScatter = 1,  // k_append: the caller's columns
  kRingOpen = 2,     // k_open: "no sample", and the index blocks recomputed
  kRingFill = 3,     // "no sample" without an index to keep (k_fill_columns, or a memset of the whole plane)
};

// gpr_append: a plane whose columns the caller did not pass (power_cols NULL) has no sample in the new buckets
inline RingLaunch append_launch(bool plane, bool cols) { return !plane ? kRingNone : cols ? kRingScatter : kRingOpen; }

// gpr_resident_advance: on an index ring the opened buckets' blocks must be recomputed (their old maxima are gone)
inline RingLaunch advance_launch(bool plane, bool index) { return !plane ? kRingNone : index ? kRingOpen : kRingFill; }

// CTAs of k_append / k_open / k_reindex: one row per CTA and round, at most 16 CTAs per SM
inline uint32_t ring_grid(size_t rows, int sm_count) {
  return (uint32_t)std::min<size_t>(rows, (size_t)sm_count * 16u);
}

// index row length: ceil(T / 64) blocks, padded to a multiple of 4 so that index rows are TMA-able (padding stays NaN)
inline uint32_t index_ld(uint32_t T) { return (((T + kIdxBlock - 1) / kIdxBlock) + 3u) & ~3u; }

// NaN-skipping max of block b (samples [64 b, min(T, 64 b + 64)) of one ring row), one warp; NaN = no sample in it
__device__ __forceinline__ float block_max_warp(const float* row, uint32_t T, uint32_t b, int lane) {
  const uint32_t t0 = b * kIdxBlock;
  float m = nan_f();
  for (uint32_t t = t0 + lane; t < min(T, t0 + kIdxBlock); t += 32) m = fmaxf(m, row[t]);
  return warp_max(m);
}

// The index blocks of one row that hold ring positions [start, start + n) modulo T (start < T, n <= T), recomputed by
// the warps of one CTA after its stores to the row (__syncthreads).  They are at most two runs: from start's block to
// the end of the span or of the ring, and, if the span wraps, from block 0 — which stops short of the first run, so
// no block is written by two warps.
__device__ __forceinline__ void recompute_blocks(const float* row, uint32_t T, uint32_t start, uint32_t n,
                                                 float* idx_row, int warp, int n_warps, int lane) {
  const uint32_t first = start / kIdxBlock;
  const uint32_t span_end = start + n;  // exclusive, may exceed T (wraps)
  const uint32_t last = (min(span_end, T) - 1) / kIdxBlock;
  for (uint32_t b = first + warp; b <= last; b += n_warps) {
    const float m = block_max_warp(row, T, b, lane);
    if (lane == 0) idx_row[b] = m;
  }
  if (span_end > T) {  // wrapped part [0, span_end - T)
    const uint32_t wend = min((span_end - T - 1) / kIdxBlock + 1, first);
    for (uint32_t b = warp; b < wend; b += n_warps) {
      const float m = block_max_warp(row, T, b, lane);
      if (lane == 0) idx_row[b] = m;
    }
  }
}

// Scatter n columns of every row into the ring at positions (start + j) % T; with an index, recompute the blocks
// they landed in (the overwritten samples may have been the old maximum).
__global__ void __launch_bounds__(kRingThreads) k_append(float* __restrict__ dst, const float* __restrict__ src,
                                                         uint32_t n_rows, uint32_t T, uint32_t start, uint32_t n,
                                                         uint64_t ld_src, float* __restrict__ idx, uint32_t idx_ld) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  for (uint32_t r = blockIdx.x; r < n_rows; r += gridDim.x) {
    float* out = dst + (size_t)r * T;
    const float* in = src + (size_t)r * ld_src;
    for (uint32_t j = threadIdx.x; j < n; j += blockDim.x) {
      uint32_t t = start + j;
      if (t >= T) t -= T;
      out[t] = in[j];
    }
    if (idx) {
      __syncthreads();  // this CTA's column stores are visible to its own warps
      recompute_blocks(out, T, start, n, idx + (size_t)r * idx_ld, warp, n_warps, lane);
      __syncthreads();
    }
  }
}

// Open n buckets at ring positions (start + j) % T of every row: no sample there; with an index, recompute the blocks
// they are in with the same code as k_append.
__global__ void __launch_bounds__(kRingThreads) k_open(float* __restrict__ plane, uint32_t n_rows, uint32_t T,
                                                       uint32_t start, uint32_t n, float* __restrict__ idx,
                                                       uint32_t idx_ld) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  for (uint32_t r = blockIdx.x; r < n_rows; r += gridDim.x) {
    float* out = plane + (size_t)r * T;
    for (uint32_t j = threadIdx.x; j < n; j += blockDim.x) {
      uint32_t t = start + j;
      if (t >= T) t -= T;
      reinterpret_cast<uint32_t*>(out)[t] = kNoSampleBits;
    }
    if (idx) {
      __syncthreads();
      recompute_blocks(out, T, start, n, idx + (size_t)r * idx_ld, warp, n_warps, lane);
      __syncthreads();
    }
  }
}

// full rebuild of the index (after the caller wrote the resident planes directly)
__global__ void __launch_bounds__(kRingThreads) k_reindex(const float* __restrict__ plane, uint32_t n_rows,
                                                          uint32_t T, float* __restrict__ idx, uint32_t idx_ld) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const uint32_t n_blocks = (T + kIdxBlock - 1) / kIdxBlock;
  for (uint32_t r = blockIdx.x; r < n_rows; r += gridDim.x)
    for (uint32_t b = warp; b < n_blocks; b += n_warps) {
      const float m = block_max_warp(plane + (size_t)r * T, T, b, lane);
      if (lane == 0) idx[(size_t)r * idx_ld + b] = m;
    }
}

// ---- gpr_resident_remap: the ring's rows moved to a new [P][G] shape, out of place
constexpr uint32_t kRowNone = 0xFFFFFFFFu;  // GPR_ROW_NONE: a new row without a source (no sample)

// The first new row of a remap whose source is bad: an old row >= n_old that is not kRowNone, or an old row that is
// also the source of another new row (every new row that shares it counts, the first of them included); n_new if the
// map is good.  What k_remap_check computes on the GPU, for a host map.
inline size_t remap_first_bad(const uint32_t* src_rows, size_t n_new, size_t n_old) {
  std::vector<uint8_t> uses(n_old, 0);  // 0, 1, 2 = more than one
  for (size_t i = 0; i < n_new; ++i)
    if (src_rows[i] < n_old) uses[src_rows[i]] = (uint8_t)std::min(2, uses[src_rows[i]] + 1);
  for (size_t i = 0; i < n_new; ++i) {
    const uint32_t s = src_rows[i];
    if (s == kRowNone) continue;
    if (s >= n_old || uses[s] > 1) return i;
  }
  return n_new;
}

// k_remap_check's two passes over a device map (a grid-wide barrier between them: two launches).  `seen` and `dup`
// are bitmaps of the n_old old rows, zeroed by the caller.  Pass 0 checks the range and marks every old row in `seen`,
// and in `dup` if it was marked already; pass 1 names the new rows whose old row is in `dup`.  `first` (the caller
// sets it to n_new) ends as remap_first_bad's answer.  Its minimum is an atomicMin written as a CAS loop, because
// tests/cpp/cuda_shim.hpp, under which the CPU emulators compile this whole namespace, has atomicCAS and no atomicMin.
__global__ void __launch_bounds__(256) k_remap_check(const uint32_t* __restrict__ src_rows, uint32_t n_new,
                                                     uint32_t n_old, unsigned int* seen, unsigned int* dup,
                                                     unsigned int* first, int pass) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_new; i += gridDim.x * blockDim.x) {
    const uint32_t s = src_rows[i];
    if (s == kRowNone) continue;
    const unsigned int bit = 1u << (s % 32);
    bool bad;
    if (pass == 0) {
      bad = s >= n_old;
      if (!bad && (atomicOr(seen + s / 32, bit) & bit)) atomicOr(dup + s / 32, bit);
    } else {
      bad = s < n_old && (dup[s / 32] & bit);
    }
    if (!bad) continue;
    unsigned int old = atomicOr(first, 0u);  // an atomic read
    while (i < old) {
      const unsigned int seen_first = atomicCAS(first, old, i);
      if (seen_first == old) break;
      old = seen_first;
    }
  }
}

// One new row of length `len` per CTA and round (grid: ring_grid): new row r is old row src_rows[r], or "no sample"
// for kRowNone.  The same gather moves the planes (len = T) and their index (len = idx_ld, padding included, so it
// stays NaN).  16-byte accesses when every row starts on a 16-byte boundary (len % 4 == 0), 4-byte ones otherwise.
__global__ void __launch_bounds__(kRingThreads) k_remap_rows(uint32_t* __restrict__ dst,
                                                             const uint32_t* __restrict__ src,
                                                             const uint32_t* __restrict__ src_rows, uint32_t n_rows,
                                                             uint32_t len) {
  for (uint32_t r = blockIdx.x; r < n_rows; r += gridDim.x) {
    const uint32_t s = src_rows[r];
    uint32_t* out = dst + (size_t)r * len;
    const uint32_t* in = s == kRowNone ? nullptr : src + (size_t)s * len;
    if (len % 4u == 0) {
      uint4* out4 = reinterpret_cast<uint4*>(out);
      const uint4* in4 = reinterpret_cast<const uint4*>(in);
      const uint4 none = make_uint4(kNoSampleBits, kNoSampleBits, kNoSampleBits, kNoSampleBits);
      for (uint32_t j = threadIdx.x; j < len / 4u; j += blockDim.x) out4[j] = in ? in4[j] : none;
    } else {
      for (uint32_t j = threadIdx.x; j < len; j += blockDim.x) out[j] = in ? in[j] : kNoSampleBits;
    }
  }
}

// ---- gpr_resident_live_rows: which rows hold at least one sample
constexpr uint32_t kLiveWarps = kRingThreads / 32;  // warps of a k_live_rows CTA, 32 rows (one bitmap word) each

// CTAs of k_live_rows: one bitmap word per warp and round, as many CTAs as ring_grid gives for that many CTA rounds
inline uint32_t live_rows_grid(size_t rows, int sm_count) {
  const size_t words = (rows + 31) / 32;
  return ring_grid(std::max<size_t>(1, (words + kLiveWarps - 1) / kLiveWarps), sm_count);
}

// what gpr_resident_live_rows reads: a current block index (1/64 of the bytes) if the ring has one, else the planes
inline bool live_rows_from_index(bool has_index, bool index_stale) { return has_index && !index_stale; }

// every NaN is "no sample" (gpr_resident_planes writers and gpr_append columns may store other NaNs than the fill)
__device__ __forceinline__ bool has_sample_bits(uint32_t b) { return (b & 0x7FFFFFFFu) <= 0x7F800000u; }

// One warp: does the row of `len` cells hold a cell that is not NaN?  The answer is the same on every lane.  The reads
// stop at the first step that finds one: the first step is one coalesced load per lane (a live row usually ends
// there), later steps issue four independent loads per lane so that a row without a sample is read at full rate.
// 16-byte loads when rows start on a 16-byte boundary (len % 4 == 0), 4-byte ones otherwise.
__device__ __forceinline__ bool row_has_sample(const uint32_t* __restrict__ row, uint32_t len, int lane) {
  if (len % 4u == 0) {
    const uint4* r4 = reinterpret_cast<const uint4*>(row);
    const uint32_t n4 = len / 4u;
    uint32_t per = 1;
    for (uint32_t base = 0; base < n4; base += 32u * per, per = 4) {
      bool hit = false;
#pragma unroll
      for (uint32_t u = 0; u < 4; ++u) {
        const uint32_t k = base + u * 32u + (uint32_t)lane;
        if (u < per && k < n4) {
          const uint4 v = r4[k];
          hit |= has_sample_bits(v.x) || has_sample_bits(v.y) || has_sample_bits(v.z) || has_sample_bits(v.w);
        }
      }
      if (__ballot_sync(0xFFFFFFFFu, hit)) return true;
    }
    return false;
  }
  uint32_t per = 1;
  for (uint32_t base = 0; base < len; base += 32u * per, per = 4) {
    bool hit = false;
#pragma unroll
    for (uint32_t u = 0; u < 4; ++u) {
      const uint32_t k = base + u * 32u + (uint32_t)lane;
      if (u < per && k < len) hit |= has_sample_bits(row[k]);
    }
    if (__ballot_sync(0xFFFFFFFFu, hit)) return true;
  }
  return false;
}

// Bit r of bits[r / 32] = row r holds a cell that is not NaN in p0 or, if given, p1 (rows of `len` cells: the planes
// with len = T, or their block index with len = idx_ld, whose padding is NaN).  A warp owns a word: it reads its 32
// rows one after the other, lane i keeps row i's answer, and one ballot makes the word.  Padding bits are zero, every
// word is written once, no atomics.  Grid: live_rows_grid.
__global__ void __launch_bounds__(kRingThreads) k_live_rows(const uint32_t* __restrict__ p0,
                                                            const uint32_t* __restrict__ p1, uint32_t n_rows,
                                                            uint32_t len, uint32_t* __restrict__ bits) {
  const int lane = threadIdx.x & 31;
  const uint32_t n_words = (n_rows + 31u) / 32u, n_warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < n_words; w += n_warps) {
    const uint32_t r0 = w * 32u, n = min(32u, n_rows - r0);
    bool mine = false;
    for (uint32_t i = 0; i < n; ++i) {
      const size_t r = (size_t)r0 + i;
      bool live = row_has_sample(p0 + r * len, len, lane);
      if (!live && p1) live = row_has_sample(p1 + r * len, len, lane);
      if ((uint32_t)lane == i) mine = live;
    }
    const uint32_t word = __ballot_sync(0xFFFFFFFFu, mine);
    if (lane == 0) bits[w] = word;
  }
}

// ---- gpr_resident_cols: a band of the ring's newest buckets, read out oldest first
// Ring position of the band's oldest bucket: the n_cols buckets that end `newer` buckets before the newest, which is at
// (head + T - 1) % T.  Needs newer + n_cols <= T.
inline uint32_t ring_cols_start(uint32_t head, uint32_t T, uint32_t newer, uint32_t n_cols) {
  return (uint32_t)(((uint64_t)head + T - newer - n_cols) % T);
}

// out[r * n_cols + j] = ring row r at position (start + j) % T: one row per CTA and round (grid: ring_grid), the band
// gathered across the ring's wrap point.  Words are moved as bits, so every NaN payload comes out as it is stored.
__global__ void __launch_bounds__(kRingThreads) k_ring_cols(uint32_t* __restrict__ out,
                                                            const uint32_t* __restrict__ plane, uint32_t n_rows,
                                                            uint32_t T, uint32_t start, uint32_t n_cols) {
  for (uint32_t r = blockIdx.x; r < n_rows; r += gridDim.x) {
    const uint32_t* in = plane + (size_t)r * T;
    uint32_t* o = out + (size_t)r * n_cols;
    for (uint32_t j = threadIdx.x; j < n_cols; j += blockDim.x) {
      uint32_t t = start + j;
      if (t >= T) t -= T;
      o[j] = in[t];
    }
  }
}

// ---- gpr_resident_retime: the ring's newest n_keep buckets regrouped `factor` to a bucket, out of place.  Whether a
// change of step and window is exact, and what n_keep and factor it takes, is gpr::retime_plan (gpr_retime.h).
// Row length after the retime: ceil(n_keep / factor).
inline uint32_t retime_len(uint32_t n_keep, uint32_t factor) { return (n_keep + factor - 1) / factor; }

// A cell's bits as an int whose order is the float order, with -0 below +0: keys of non-negative floats are their bits,
// keys of negative ones have the magnitude bits flipped.  The map is its own inverse.  Comparing keys instead of floats
// keeps denormals exact whatever the float compare flushes.
__device__ __forceinline__ int32_t retime_key(uint32_t b) {
  return (int32_t)(b ^ ((uint32_t)((int32_t)b >> 31) >> 1));
}

// New cell of one group: the maximum of the n old cells at ring positions t, t + 1, ... (mod T), as text::atomic_merge
// leaves a fill cell that took them in any order — every NaN is no sample, a group without one is kNoSampleBits, and
// +0 beats -0.  Every finite or infinite key is above INT32_MIN.
__device__ __forceinline__ uint32_t retime_group(const uint32_t* __restrict__ row, uint32_t T, uint32_t t, uint32_t n) {
  int32_t best = INT32_MIN;
  for (uint32_t j = 0; j < n; ++j) {
    const uint32_t b = row[t];
    if (has_sample_bits(b)) best = max(best, retime_key(b));
    if (++t == T) t = 0;
  }
  return best == INT32_MIN ? kNoSampleBits : (uint32_t)retime_key((uint32_t)best);
}

// New position p (0 = oldest) of a retimed row: new bucket T' - 1 - p is old buckets [k b', min(k b' + k, n_keep))
// counted from the newest, which sits at ring position head + T - 1; the group is read oldest first.
__device__ __forceinline__ uint32_t retime_cell(const uint32_t* __restrict__ row, uint32_t T, uint32_t head,
                                                uint32_t n_keep, uint32_t factor, uint32_t T_new, uint32_t p) {
  const uint32_t lo = (T_new - 1 - p) * factor, hi = min(lo + factor, n_keep);  // old buckets [lo, hi)
  return retime_group(row, T, (uint32_t)(((uint64_t)head + T - hi) % T), hi - lo);
}

// One new row per CTA and round (grid: ring_grid): old row r of length T with its head at `head` becomes new row r of
// length T_new = retime_len(n_keep, factor), oldest first (its head is 0).  Lane i of a warp takes new cell i, so a warp's
// loads of one group step cover 32 groups `factor` words apart and the later steps find those lines in L1.  16-byte stores
// when new rows start on a 16-byte boundary (T_new % 4 == 0), 4-byte ones otherwise.  With an index (idx, of rows
// idx_ld long), the CTA then rebuilds the row's blocks from the row it wrote and sets the padding to no sample.
__global__ void __launch_bounds__(kRingThreads) k_retime_rows(uint32_t* __restrict__ dst, const uint32_t* __restrict__ src,
                                                              uint32_t n_rows, uint32_t T, uint32_t head, uint32_t n_keep,
                                                              uint32_t factor, float* __restrict__ idx, uint32_t idx_ld) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const uint32_t T_new = (n_keep + factor - 1) / factor;  // retime_len
  for (uint32_t r = blockIdx.x; r < n_rows; r += gridDim.x) {
    const uint32_t* in = src + (size_t)r * T;
    uint32_t* out = dst + (size_t)r * T_new;
    if (T_new % 4u == 0) {
      uint4* out4 = reinterpret_cast<uint4*>(out);
      for (uint32_t j = threadIdx.x; j < T_new / 4u; j += blockDim.x) {
        const uint32_t p = 4u * j;
        out4[j] = make_uint4(retime_cell(in, T, head, n_keep, factor, T_new, p),
                             retime_cell(in, T, head, n_keep, factor, T_new, p + 1),
                             retime_cell(in, T, head, n_keep, factor, T_new, p + 2),
                             retime_cell(in, T, head, n_keep, factor, T_new, p + 3));
      }
    } else {
      for (uint32_t p = threadIdx.x; p < T_new; p += blockDim.x) out[p] = retime_cell(in, T, head, n_keep, factor, T_new, p);
    }
    if (idx) {
      float* idx_row = idx + (size_t)r * idx_ld;
      __syncthreads();  // this CTA's stores to the row are visible to its own warps
      recompute_blocks(reinterpret_cast<const float*>(out), T_new, 0, T_new, idx_row, warp, n_warps, lane);
      for (uint32_t b = (T_new + kIdxBlock - 1) / kIdxBlock + threadIdx.x; b < idx_ld; b += blockDim.x)
        reinterpret_cast<uint32_t*>(idx_row)[b] = kNoSampleBits;
      __syncthreads();
    }
  }
}

}  // namespace gpr
