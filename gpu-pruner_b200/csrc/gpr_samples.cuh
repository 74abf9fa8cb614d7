// gpr_samples.cuh — decoded range-vector samples merged into a plane on the GPU (gpr_samples_scatter).
//
// A caller whose Prometheus client has already decoded the matrix (a label map and [(timestamp, value)] per series)
// hands the samples over in CSR form: series s owns samples [offsets[s], offsets[s+1]), which go to row rows[s];
// sample i is (ts[i] in milliseconds, values[i] as f64).  Every sample is treated exactly as the text parser treats
// the same sample written as text (gpr_text.cuh): column_of() on milliseconds, to_f32() and, on the power plane,
// snap_power(); NaN is dropped and cells merge with the text kernel's atomic NaN-aware max (atomic_merge,
// gpr_text_kernels.cuh).  So a window built from samples is bit for bit the window built from the response text.
//
// The work is balanced by sample count, not by series (daemon slices have ~180 samples per series, full windows
// ~1800, and a series may be empty): the samples are cut into chunks of kChunk, CTAs take chunks grid-stride, and in
// a chunk thread t handles the sample pairs t, t + kThreads, ... — one 16-byte ld.global.nc of two timestamps and one
// of two values per pair, coalesced across the warp.  Lane 0 of each warp binary-searches `offsets` once per chunk
// for the series of the warp's first sample; each lane then walks forward from there (series_from).
//
// Host batches are uploaded in pieces of at most kHostPiece samples (for_each_piece); the scatter of piece k runs
// while piece k + 1 crosses PCIe, so a batch needs staging memory, not a device copy of itself.
//
// Everything here except the kernels is plain C++ as well: tests/cpp/samples_emul.cpp runs this source on the CPU.
#pragma once
#include <stdint.h>

#include "gpr_text.cuh"
#include "gpr_text_kernels.cuh"  // atomic_merge, and ldg_stream_u4 of gpr_kernels.cuh

namespace gpr {
namespace samples {

constexpr uint32_t kThreads = 256;                                  // per CTA
constexpr uint32_t kPairs = 4;                                      // sample pairs per thread and chunk
constexpr uint64_t kChunk = (uint64_t)kThreads * kPairs * 2;        // samples per CTA step
constexpr uint64_t kHostPiece = 2ull << 20;                         // samples per upload piece (32 MB of ts + values)

constexpr uint32_t kBadRow = 1u, kBadOrder = 2u, kBadStart = 4u;    // series_faults() bits

// What is wrong with series s of a batch of n_series (0 = nothing).  s = 0 also checks offsets[0]; a batch without
// series is checked with s = 0 alone.
GPR_HD uint32_t series_faults(const uint64_t* offsets, const uint32_t* rows, uint32_t n_series, uint32_t s,
                              uint32_t n_rows) {
  uint32_t f = (s == 0 && offsets[0] != 0) ? kBadStart : 0u;
  if (s < n_series) {
    if (rows[s] >= n_rows) f |= kBadRow;
    if (offsets[s + 1] < offsets[s]) f |= kBadOrder;
  }
  return f;
}

// the series that owns sample i, searched in [lo, hi): needs offsets[lo] <= i < offsets[hi].  The owner is the last
// series that starts at or before i (an empty series starts where the next one does).
GPR_HD uint32_t series_in(const uint64_t* offsets, uint32_t lo, uint32_t hi, uint64_t i) {
  while (hi - lo > 1) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (offsets[mid] <= i) lo = mid;
    else hi = mid;
  }
  return lo;
}

// the owner of sample i, given the owner s of an earlier sample (or any series that starts at or before i): one
// load while i stays in s, a galloping search past s otherwise
GPR_HD uint32_t series_from(const uint64_t* offsets, uint32_t n_series, uint32_t s, uint64_t i) {
  if (offsets[s + 1] > i) return s;
  uint32_t lo = s + 1, step = 1;  // offsets[lo] <= i
  while (lo + step < n_series && offsets[lo + step] <= i) lo += step, step *= 2;
  return series_in(offsets, lo, lo + step < n_series ? lo + step : n_series, i);
}

// A piece of a host batch: samples [begin, end) and the series sample `begin` belongs to.
struct Piece {
  uint64_t begin, end;
  uint32_t series;
};

// Cuts the elements [0, total) of a CSR batch (samples here, chunks in gpr_chunks.cuh) into pieces, in order: the
// piece that begins at b ends at cut(b), which must lie in (b, total].  fn(const Piece&) returns 0 to go on; the first
// other value stops the walk and is returned.
template <typename Cut, typename Fn>
inline int for_each_cut(const uint64_t* offsets, uint32_t n_series, uint64_t total, Cut&& cut, Fn&& fn) {
  uint32_t s = 0;
  for (uint64_t b = 0; b < total;) {
    s = series_from(offsets, n_series, s, b);
    const Piece p{b, cut(b), s};
    const int rc = fn(p);
    if (rc != 0) return rc;
    b = p.end;
  }
  return 0;
}

// Cuts the samples [0, total) of a batch into pieces of at most `piece` samples, wherever the cut falls: between
// series or inside one.
template <typename Fn>
inline int for_each_piece(const uint64_t* offsets, uint32_t n_series, uint64_t total, uint64_t piece, Fn&& fn) {
  return for_each_cut(offsets, n_series, total, [&](uint64_t b) { return total - b < piece ? total : b + piece; }, fn);
}

struct ScatterArgs {
  const uint64_t* offsets;   // n_series + 1, device
  const uint32_t* rows;      // n_series, device
  const int64_t* ts;         // sample i at ts[i - base]
  const double* values;      // sample i at values[i - base]
  uint64_t base, end;        // the samples [base, end) of the batch this launch merges
  uint32_t n_series;
  uint32_t s_base;           // the series sample `base` belongs to
  float* plane;
  unsigned long long* stats; // [2]: samples outside the window, in-window values kept non-zero by to_f32
  text::Grid g;
};

// One sample: the cell and the value gpr_text_parse gives the same sample written as text.
__device__ __forceinline__ void scatter_sample(const text::Grid& g, float* plane, uint32_t row, int64_t ts, double v,
                                               uint32_t& n_oow, uint32_t& n_tiny) {
  const int64_t col = text::column_of(g, ts);
  if (col < 0) {
    ++n_oow;
    return;
  }
  const float f = text::snap_power(v, text::to_f32(v, &n_tiny), g.power);
  text::atomic_merge(plane + (uint64_t)row * g.ld + (uint64_t)col, f);
}

// kVec: ts and values are 16-byte aligned, so a pair (i - base even) is one 128-bit load of each
template <bool kVec>
__global__ void __launch_bounds__(kThreads) k_samples_scatter(const ScatterArgs a) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint64_t n = a.end - a.base;
  const uint64_t n_chunks = (n + kChunk - 1) / kChunk;
  uint32_t n_oow = 0, n_tiny = 0;
  for (uint64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const uint64_t c0 = a.base + c * kChunk;  // first sample of the chunk
    // the warp's first sample is its first pair in round 0; lane 0 finds its series, the lanes walk on from there
    const uint64_t w0 = c0 + 2ull * warp * 32u;
    uint32_t s = 0;
    if (lane == 0 && w0 < a.end) s = series_in(a.offsets, a.s_base, a.n_series, w0);
    s = __shfl_sync(0xffffffffu, s, 0);
    if (w0 >= a.end) continue;  // (the whole warp: w0 is uniform)
    uint64_t i0[kPairs];
    int64_t t[kPairs][2];
    double v[kPairs][2];
#pragma unroll
    for (uint32_t k = 0; k < kPairs; ++k) {  // all loads first: 2 x kPairs 16-byte loads in flight per thread
      i0[k] = c0 + 2ull * (k * kThreads + threadIdx.x);
      const uint64_t j = i0[k] - a.base;
      if (kVec && i0[k] + 1 < a.end) {
        const uint4 x = ldg_stream_u4(reinterpret_cast<const uint4*>(a.ts + j));
        const uint4 y = ldg_stream_u4(reinterpret_cast<const uint4*>(a.values + j));
        t[k][0] = (int64_t)(((uint64_t)x.y << 32) | x.x);
        t[k][1] = (int64_t)(((uint64_t)x.w << 32) | x.z);
        v[k][0] = text::bits_to_double(((uint64_t)y.y << 32) | y.x);
        v[k][1] = text::bits_to_double(((uint64_t)y.w << 32) | y.z);
      } else {
        t[k][0] = t[k][1] = 0;
        v[k][0] = v[k][1] = 0.0;
        if (i0[k] < a.end) t[k][0] = __ldg(a.ts + j), v[k][0] = __ldg(a.values + j);
        if (i0[k] + 1 < a.end) t[k][1] = __ldg(a.ts + j + 1), v[k][1] = __ldg(a.values + j + 1);
      }
    }
#pragma unroll
    for (uint32_t k = 0; k < kPairs; ++k) {
#pragma unroll
      for (uint32_t h = 0; h < 2; ++h) {
        const uint64_t i = i0[k] + h;
        if (i >= a.end) break;
        s = series_from(a.offsets, a.n_series, s, i);
        scatter_sample(a.g, a.plane, __ldg(a.rows + s), t[k][h], v[k][h], n_oow, n_tiny);
      }
    }
  }
  const uint32_t w_oow = __reduce_add_sync(0xffffffffu, n_oow), w_tiny = __reduce_add_sync(0xffffffffu, n_tiny);
  if (lane == 0) {
    if (w_oow) atomicAdd(a.stats + 0, (unsigned long long)w_oow);
    if (w_tiny) atomicAdd(a.stats + 1, (unsigned long long)w_tiny);
  }
}

// Checks a device batch before anything is written: the series_faults() bits of every series are OR-ed into *bad.
__global__ void __launch_bounds__(256) k_samples_check(const uint64_t* offsets, const uint32_t* rows, uint32_t n_series,
                                                       uint32_t n_rows, unsigned int* bad) {
  const uint32_t n = n_series ? n_series : 1u;
  uint32_t f = 0;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x)
    f |= series_faults(offsets, rows, n_series, s, n_rows);
  if (f) atomicOr(bad, f);
}

}  // namespace samples
}  // namespace gpr
