// gpr_ring.cuh — the resident ring of daemon mode: a tick's columns scattered into the time ring, buckets opened
// without data, and the optional block-maxima index (GPR_F_BLOCK_INDEX) kept in step with both.
//
// The kernels here are plain CUDA C++ without inline PTX, and the host-side arithmetic of gpr_append /
// gpr_resident_advance (which source columns survive, where they land, what each plane gets, the grid, the index
// row length) is plain functions.  gpr_api.cu launches what these return; tests/cpp/ring_emul.cpp runs the same
// source on the CPU against a numpy model of the ring.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <algorithm>

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

}  // namespace gpr
