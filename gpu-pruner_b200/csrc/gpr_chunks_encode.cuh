// gpr_chunks_encode.cuh — the resident ring exported as Prometheus XOR chunks, encoded on the GPU
// (gpr_resident_export).
//
// The encoder is Prometheus' XOR appender (tsdb/chunkenc/xor.go) written from the format gpr_chunks.cuh states:
//   bytes 0-1   the sample count, big-endian u16
//   sample 0    timestamp as a zigzag varint, then the 64 bits of the float64
//   sample 1    timestamp delta as an unsigned varint, then the value in XOR form
//   sample n>=2 delta-of-delta: 0 -> '0'; in [-(2^13 - 1), 2^13] -> '10' + 14 bits; [-(2^16 - 1), 2^16] -> '110' + 17;
//               [-(2^19 - 1), 2^19] -> '1110' + 20; otherwise '1111' + 64 (two's complement, low bits)
//   XOR form    x = value ^ previous value.  x = 0 -> '0'.  Otherwise the leading zeros of x (at most 31, Go's clamp)
//               and its trailing zeros: if a window is set and x fits it (leading >= the window's, trailing >= its
//               trailing) -> '10' + the window's bits of x; else the window becomes x's -> '11' + 5 bits leading
//               + 6 bits significant (64 written as 0) + the significant bits
// so the bytes are those the reference appender writes for the same samples (tests/chunks_ref.py encode()).
//
// Row r of the ring is one series.  Its sample j (oldest first) is the cell at ring position (head + j) % T, with
//   ts_ms = t_end_ms - (T - 1 - j) * step_ms,   value = (double)cell
// and NaN cells (any NaN) are skipped.  A row's present cells are cut into chunks of at most per_chunk samples.
//
// Three launches and a read-back:
//   k_export_size   a warp per row finds where each chunk starts (ballots over 32 cells at a time and popcounts), then
//                   one lane per chunk encodes it without storing (bit-serial, as the decoder reads): the chunk's byte
//                   count, the row's chunks, bytes and samples
//   k_export_scan   one CTA: exclusive scans over the rows of chunks, bytes and "has a chunk" -> each row's first
//                   chunk, first byte and series index, and the totals
//   k_export_write  a warp per row: its chunks' offsets (a warp scan of their sizes), then one lane per chunk encodes
//                   it again, storing its bytes
// The ring is only read.
//
// Everything here except the kernels is plain C++ as well; tests/cpp/chunks_export_emul.cpp runs the kernels' source
// on the CPU.
#pragma once
#include <stdint.h>

#include "gpr_text.cuh"  // GPR_HD, clz64, f32_from_bits

namespace gpr {
namespace chunks {

constexpr uint32_t kEncThreads = 128;               // k_export_size / k_export_write: a warp per row
constexpr uint32_t kEncWarps = kEncThreads / 32;
constexpr uint32_t kScanThreads = 1024;             // k_export_scan: one CTA
constexpr uint32_t kScanSmem = 32 * (8 + 8 + 4);    // its shared memory: the warps' totals

// ---- the bit stream, written -----------------------------------------------------------------------------------
struct BitW {
  uint8_t* p;     // the next byte to store; nullptr = count the bits only
  uint64_t acc;   // the bits not yet stored are its low n bits
  uint32_t n;
  uint64_t bits;  // bits put so far
};

GPR_HD BitW bitw_at(uint8_t* p) { return BitW{p, 0ull, 0u, 0ull}; }

// the low k bits of v, MSB first; 1 <= k <= 32
GPR_HD void put(BitW& w, uint64_t v, uint32_t k) {
  w.bits += k;
  if (!w.p) return;
  w.acc = (w.acc << k) | (v & ((1ull << k) - 1ull));
  w.n += k;
  while (w.n >= 8u) w.n -= 8u, *w.p++ = (uint8_t)(w.acc >> w.n);
}

// the low k bits of v, 1 <= k <= 64
GPR_HD void put_wide(BitW& w, uint64_t v, uint32_t k) {
  if (k > 32u) put(w, v >> 32, k - 32u), k = 32u;
  put(w, v, k);
}

// the last byte, its unused low bits 0
GPR_HD void flush(BitW& w) {
  if (w.p && w.n) *w.p++ = (uint8_t)(w.acc << (8u - w.n)), w.n = 0;
}

// an unsigned varint (Go's binary.PutUvarint) written byte by byte into the bit stream
GPR_HD void put_uvarint(BitW& w, uint64_t x) {
  while (x >= 0x80u) put(w, (x & 0x7fu) | 0x80u, 8u), x >>= 7;
  put(w, x, 8u);
}

GPR_HD uint64_t double_bits(double d) {
#if defined(__CUDA_ARCH__)
  return (uint64_t)__double_as_longlong(d);
#else
  uint64_t b;
  memcpy(&b, &d, sizeof b);
  return b;
#endif
}

GPR_HD uint32_t ctz64(uint64_t x) {  // x != 0
#if defined(__CUDA_ARCH__)
  return (uint32_t)__ffsll((long long)x) - 1u;
#else
  return (uint32_t)__builtin_ctzll(x);
#endif
}

// -(2^(n-1) - 1) <= dod <= 2^(n-1): the range of an n-bit delta-of-delta bucket
GPR_HD bool in_bucket(int64_t dod, uint32_t n) {
  return dod >= -((1ll << (n - 1u)) - 1) && dod <= (1ll << (n - 1u));
}

// ---- the appender -------------------------------------------------------------------------------------------------
struct Enc {
  BitW w;
  uint32_t n;            // samples appended
  uint64_t t, delta, v;  // the previous timestamp, delta and value bits (wrapping arithmetic, as Go's)
  uint32_t lead, trail;  // the XOR window; lead 0xff = none yet
};

GPR_HD Enc enc_at(uint8_t* body) { return Enc{bitw_at(body), 0u, 0ull, 0ull, 0ull, 0xffu, 0u}; }

GPR_HD void append(Enc& e, int64_t ts, uint64_t v) {
  const uint64_t t = (uint64_t)ts;
  if (e.n == 0) {
    put_uvarint(e.w, (t << 1) ^ (uint64_t)(ts >> 63));  // zigzag
    put_wide(e.w, v, 64u);
  } else {
    const uint64_t delta = t - e.t;
    if (e.n == 1) {
      put_uvarint(e.w, delta);
    } else {
      const int64_t dod = (int64_t)(delta - e.delta);
      if (dod == 0) put(e.w, 0u, 1u);
      else if (in_bucket(dod, 14u)) put(e.w, 0x2u, 2u), put(e.w, (uint64_t)dod, 14u);
      else if (in_bucket(dod, 17u)) put(e.w, 0x6u, 3u), put(e.w, (uint64_t)dod, 17u);
      else if (in_bucket(dod, 20u)) put(e.w, 0xeu, 4u), put(e.w, (uint64_t)dod, 20u);
      else put(e.w, 0xfu, 4u), put_wide(e.w, (uint64_t)dod, 64u);
    }
    e.delta = delta;
    const uint64_t x = v ^ e.v;
    if (x == 0) {
      put(e.w, 0u, 1u);
    } else {
      uint32_t lead = (uint32_t)text::clz64(x);
      if (lead > 31u) lead = 31u;  // the 5-bit field
      const uint32_t trail = ctz64(x);
      if (e.lead != 0xffu && lead >= e.lead && trail >= e.trail) {
        put(e.w, 0x2u, 2u);
        put_wide(e.w, x >> e.trail, 64u - e.lead - e.trail);
      } else {
        e.lead = lead, e.trail = trail;
        const uint32_t sig = 64u - lead - trail;
        put(e.w, 0x3u, 2u);
        put(e.w, lead, 5u);
        put(e.w, sig & 63u, 6u);
        put_wide(e.w, x >> trail, sig);
      }
    }
  }
  e.t = t, e.v = v;
  ++e.n;
}

// ---- the ring as series ---------------------------------------------------------------------------------------
struct ExportArgs {
  const uint32_t* plane;      // the ring plane [rows][T], f32 bits
  uint32_t rows, T, head;
  uint32_t per_chunk;         // 1..65535
  int64_t t_end_ms, step_ms;  // sample j: t_end_ms - (T - 1 - j) * step_ms
  uint32_t max_chunks;        // ceil(T / per_chunk): the row stride of sizes
  uint32_t* sizes;            // [rows][max_chunks]: the bytes of each chunk (size pass out, write pass in)
  uint64_t* row_chunks;       // [rows + 1]: chunks per row, then (scan) the row's first chunk; [rows] the total
  uint64_t* row_bytes;        // [rows + 1]: bytes per row, then (scan) the row's first byte; [rows] the total
  uint32_t* row_series;       // [rows + 1]: (scan) the row's series index; [rows] the number of series
  unsigned long long* totals; // [4]: chunks, bytes, series (scan), samples (size pass, atomicAdd)
  // outputs (write pass)
  uint64_t* series_chunks;    // n_series + 1
  uint32_t* out_rows;         // n_series
  uint64_t* chunk_bytes;      // n_chunks + 1
  uint8_t* data;              // n_bytes
};

GPR_HD bool cell_present(uint32_t b) { return (b & 0x7fffffffu) <= 0x7f800000u; }  // not a NaN

GPR_HD int64_t sample_ts(const ExportArgs& a, uint32_t j) {
  return a.t_end_ms - (int64_t)(a.T - 1u - j) * a.step_ms;
}

// Encodes the chunk whose first sample is row cell j0 (present): the next per_chunk present cells, or up to the row's
// end.  body = where the bytes after the 2-byte header go (nullptr = count only).  Returns the chunk's bytes; *count
// = its samples.
GPR_HD uint64_t encode_chunk(const ExportArgs& a, const uint32_t* cells, uint32_t j0, uint8_t* body, uint32_t* count) {
  Enc e = enc_at(body);
  uint32_t pos = a.head + j0;
  if (pos >= a.T) pos -= a.T;
  for (uint32_t j = j0; j < a.T && e.n < a.per_chunk; ++j) {
    const uint32_t b = cells[pos];
    if (++pos == a.T) pos = 0;
    if (!cell_present(b)) continue;
    append(e, sample_ts(a, j), double_bits((double)text::f32_from_bits(b)));
  }
  flush(e.w);
  if (body) body[-2] = (uint8_t)(e.n >> 8), body[-1] = (uint8_t)e.n;
  *count = e.n;
  return 2u + (e.w.bits + 7u) / 8u;
}

// the position of the n-th (from 0) set bit of b
__device__ __forceinline__ uint32_t nth_bit(uint32_t b, uint32_t n) {
  for (uint32_t k = 0; k < n; ++k) b &= b - 1u;
  return (uint32_t)__ffs((int)b) - 1u;
}

// Finds where each chunk of a row starts and calls fn(k, j0) on the lane that owns chunk k (k % 32 == lane), 32 chunks
// per round; returns the row's chunks.  Called by the whole warp (row-uniform); fn must not synchronise the warp.
// A round scans the row 32 cells at a time from where the last one stopped: a ballot marks the present cells, and
// the lane whose chunk's first sample (present cell number k * per_chunk) falls in this window takes its position.
// The round ends at the window where the next round's first chunk starts, which that round scans again.
template <typename Fn>
__device__ __forceinline__ uint32_t for_each_chunk(const ExportArgs& a, const uint32_t* cells, Fn&& fn) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t M = a.per_chunk;
  uint32_t j = 0;  // the window's first cell
  uint64_t q = 0;  // present cells before it
  for (uint32_t k0 = 0;; k0 += 32u) {
    const uint64_t want = (uint64_t)(k0 + lane) * M, next = (uint64_t)(k0 + 32u) * M;
    uint32_t start = ~0u;
    bool more = false;
    while (j < a.T) {
      bool present = false;
      if (j + lane < a.T) {
        uint32_t pos = a.head + j + lane;
        if (pos >= a.T) pos -= a.T;
        present = cell_present(__ldg(cells + pos));
      }
      const uint32_t b = __ballot_sync(0xffffffffu, present);
      const uint32_t pc = (uint32_t)__popc(b);
      if (want >= q && want < q + pc) start = j + nth_bit(b, (uint32_t)(want - q));
      if (next < q + pc) {
        more = true;
        break;
      }
      q += pc, j += 32u;
    }
    const uint32_t n = (uint32_t)__popc(__ballot_sync(0xffffffffu, start != ~0u));
    if (start != ~0u) fn(k0 + lane, start);
    if (!more) return k0 + n;
  }
}

__device__ __forceinline__ uint64_t warp_sum64(uint64_t v) {
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t lo = __shfl_xor_sync(0xffffffffu, (uint32_t)v, o);
    const uint32_t hi = __shfl_xor_sync(0xffffffffu, (uint32_t)(v >> 32), o);
    v += ((uint64_t)hi << 32) | lo;
  }
  return v;
}

__device__ __forceinline__ uint64_t shfl_up64(uint64_t v, int d) {
  const uint32_t lo = __shfl_up_sync(0xffffffffu, (uint32_t)v, d);
  const uint32_t hi = __shfl_up_sync(0xffffffffu, (uint32_t)(v >> 32), d);
  return ((uint64_t)hi << 32) | lo;
}

// Pass 1: per row its chunks and bytes, per chunk its bytes, and the samples in all (a.totals[3]).
__global__ void __launch_bounds__(kEncThreads) k_export_size(const ExportArgs a) {
  const uint32_t lane = threadIdx.x & 31u;
  uint64_t samples = 0;
  for (uint32_t r = blockIdx.x * kEncWarps + (threadIdx.x >> 5); r < a.rows; r += gridDim.x * kEncWarps) {
    const uint32_t* cells = a.plane + (uint64_t)r * a.T;
    uint32_t* sizes = a.sizes + (uint64_t)r * a.max_chunks;
    uint64_t bytes = 0;
    const uint32_t n = for_each_chunk(a, cells, [&](uint32_t k, uint32_t j0) {
      uint32_t count = 0;
      const uint64_t sz = encode_chunk(a, cells, j0, nullptr, &count);
      sizes[k] = (uint32_t)sz;
      bytes += sz, samples += count;
    });
    bytes = warp_sum64(bytes);
    if (lane == 0) a.row_chunks[r] = n, a.row_bytes[r] = bytes;
  }
  if (samples) atomicAdd(a.totals + 3, (unsigned long long)samples);
}

// Pass 2, one CTA of kScanThreads: row_chunks, row_bytes -> their exclusive prefix sums over the rows, and row_series
// = the rows with a chunk before each; entry [rows] and totals[0..2] get the totals.  Thread t takes a run of
// consecutive rows: the run's sums, a scan of those across the CTA (warp shuffles, then the warps' totals), then the
// run again.
__global__ void __launch_bounds__(kScanThreads) k_export_scan(const ExportArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t* s_c = reinterpret_cast<uint64_t*>(smem);
  uint64_t* s_b = s_c + 32;
  uint32_t* s_s = reinterpret_cast<uint32_t*>(s_b + 32);
  const uint32_t t = threadIdx.x, lane = t & 31u, warp = t >> 5;
  const uint64_t per = ((uint64_t)a.rows + kScanThreads - 1) / kScanThreads;
  const uint64_t lo = t * per < a.rows ? t * per : a.rows, hi = lo + per < a.rows ? lo + per : a.rows;
  uint64_t c = 0, b = 0;
  uint32_t s = 0;
  for (uint64_t r = lo; r < hi; ++r) c += a.row_chunks[r], b += a.row_bytes[r], s += a.row_chunks[r] != 0;
  uint64_t ic = c, ib = b;  // inclusive over the warp
  uint32_t is = s;
  for (int d = 1; d < 32; d <<= 1) {
    const uint64_t xc = shfl_up64(ic, d), xb = shfl_up64(ib, d);
    const uint32_t xs = __shfl_up_sync(0xffffffffu, is, d);
    if ((int)lane >= d) ic += xc, ib += xb, is += xs;
  }
  if (lane == 31u) s_c[warp] = ic, s_b[warp] = ib, s_s[warp] = is;
  __syncthreads();
  if (warp == 0) {  // the warps' totals -> exclusive
    const uint64_t wc = s_c[lane], wb = s_b[lane];
    const uint32_t ws = s_s[lane];
    uint64_t jc = wc, jb = wb;
    uint32_t js = ws;
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t xc = shfl_up64(jc, d), xb = shfl_up64(jb, d);
      const uint32_t xs = __shfl_up_sync(0xffffffffu, js, d);
      if ((int)lane >= d) jc += xc, jb += xb, js += xs;
    }
    s_c[lane] = jc - wc, s_b[lane] = jb - wb, s_s[lane] = js - ws;
  }
  __syncthreads();
  c = s_c[warp] + ic - c, b = s_b[warp] + ib - b, s = s_s[warp] + is - s;  // before this thread's run
  for (uint64_t r = lo; r < hi; ++r) {
    const uint64_t rc = a.row_chunks[r], rb = a.row_bytes[r];
    a.row_chunks[r] = c, a.row_bytes[r] = b, a.row_series[r] = s;
    c += rc, b += rb, s += rc != 0;
  }
  if (t == kScanThreads - 1u) {
    a.row_chunks[a.rows] = c, a.row_bytes[a.rows] = b, a.row_series[a.rows] = s;
    a.totals[0] = c, a.totals[1] = b, a.totals[2] = s;
  }
}

// Pass 3: the outputs.  Row r's series (if it has a chunk) is row_series[r]; its chunks start at row_chunks[r] and
// their bytes at row_bytes[r].
__global__ void __launch_bounds__(kEncThreads) k_export_write(const ExportArgs a) {
  const uint32_t lane = threadIdx.x & 31u;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.series_chunks[a.row_series[a.rows]] = a.row_chunks[a.rows];
    a.chunk_bytes[a.row_chunks[a.rows]] = a.row_bytes[a.rows];
  }
  for (uint32_t r = blockIdx.x * kEncWarps + (threadIdx.x >> 5); r < a.rows; r += gridDim.x * kEncWarps) {
    const uint64_t c0 = a.row_chunks[r], nc = a.row_chunks[r + 1] - c0;
    if (nc == 0) continue;  // (row-uniform)
    if (lane == 0) a.series_chunks[a.row_series[r]] = c0, a.out_rows[a.row_series[r]] = r;
    const uint32_t* cells = a.plane + (uint64_t)r * a.T;
    const uint32_t* sizes = a.sizes + (uint64_t)r * a.max_chunks;
    uint64_t base = a.row_bytes[r];
    for (uint64_t k0 = 0; k0 < nc; k0 += 32u) {  // the chunks' offsets: a warp scan of their sizes, 32 at a time
      const uint64_t k = k0 + lane;
      const uint64_t sz = k < nc ? sizes[k] : 0u;
      uint64_t in = sz;
      for (int d = 1; d < 32; d <<= 1) {
        const uint64_t x = shfl_up64(in, d);
        if ((int)lane >= d) in += x;
      }
      if (k < nc) a.chunk_bytes[c0 + k] = base + in - sz;
      base += ((uint64_t)__shfl_sync(0xffffffffu, (uint32_t)(in >> 32), 31) << 32) |
              __shfl_sync(0xffffffffu, (uint32_t)in, 31);
    }
    for_each_chunk(a, cells, [&](uint32_t k, uint32_t j0) {
      uint8_t* out = a.data + a.chunk_bytes[c0 + k];  // this lane's own store above
      uint32_t count = 0;
      encode_chunk(a, cells, j0, out + 2, &count);
    });
  }
}

}  // namespace chunks
}  // namespace gpr
