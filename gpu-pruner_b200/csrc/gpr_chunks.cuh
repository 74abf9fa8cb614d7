// gpr_chunks.cuh — Prometheus XOR chunks decoded and merged into a plane on the GPU (gpr_chunks_scatter).
//
// Prometheus stores a series as XOR chunks (tsdb/chunkenc/xor.go, Gorilla compression), and remote read
// (STREAMED_XOR_CHUNKS) and the Thanos StoreAPI hand those bytes out as they are stored.  A caller puts the `data`
// field of every chunk into one buffer, back to back, and says which row each series feeds; in CSR form series s owns
// chunks [series_chunks[s], series_chunks[s+1]) and chunk c is data[chunk_bytes[c], chunk_bytes[c+1]).
//
// The format, MSB first after a 2-byte header:
//   bytes 0-1   the sample count, big-endian u16
//   sample 0    timestamp as a zigzag varint (bytes written into the bit stream), then 64 raw bits of float64
//   sample 1    timestamp delta as an unsigned varint, then the value in XOR form
//   sample n>=2 delta-of-delta: '0' = 0, '10' + 14 bits, '110' + 17, '1110' + 20, '1111' + 64; a payload of sz bits
//               above 2^(sz-1) is negative (subtract 2^sz); then the value in XOR form
//   XOR form    '0' = the previous value; '10' = xor bits in the previous window (leading / significant bits);
//               '11' + 5 bits leading + 6 bits significant (0 means 64) + the significant bits
// Bytes after the last sample are not read.  A sample goes through the text kernel's own rules, exactly as
// gpr_samples_scatter takes the same (ts_ms, value): samples::scatter_sample (column_of, to_f32, snap_power,
// atomic_merge).  So a window built from chunks is bit for bit the window built from the samples, or from the text.
//
// One lane decodes one chunk (the decode is bit-serial inside a chunk; a C2 window is some 600,000 chunks), reading its
// bytes eight at a time into a 64-bit buffer.  A warp takes 32 consecutive chunks; CTAs grid-stride over groups of
// 32.  (Staging each warp's chunks in shared memory with coalesced 16-byte loads first was 7 % slower on the C2
// window: DESIGN.md §8g.)
//
// The reader never loads a byte outside its chunk, so a malformed chunk cannot make a kernel read out of bounds; the
// check (chunk_faults, k_chunks_check) still rejects such a batch before anything is written.
//
// Everything here except the kernels is plain C++ as well: tests/cpp/chunks_emul.cpp runs this source on the CPU.
#pragma once
#include <stdint.h>

#include "gpr_samples.cuh"  // series_faults, series_in / series_from, for_each_cut, scatter_sample

namespace gpr {
namespace chunks {

constexpr uint32_t kThreads = 128;                  // per CTA
constexpr uint32_t kWarps = kThreads / 32;
constexpr uint64_t kHostPiece = 32ull << 20;        // bytes of chunk data per upload piece

// fault bits: the series bits of samples::series_faults, then the chunk bits of chunk_faults
constexpr uint32_t kBadRow = samples::kBadRow, kBadOrder = samples::kBadOrder, kBadStart = samples::kBadStart;
constexpr uint32_t kBadChunkStart = 8u;   // chunk_bytes[0] != 0
constexpr uint32_t kBadChunkOrder = 16u;  // chunk_bytes decrease
constexpr uint32_t kShort = 32u;          // a chunk shorter than its 2-byte header
constexpr uint32_t kOverrun = 64u;        // the decode would read past the chunk's bytes
constexpr uint32_t kNoWindow = 128u;      // a value reuses the XOR window before any was set
constexpr uint32_t kBadVarint = 256u;     // a varint longer than 64 bits

// ---- the bit stream --------------------------------------------------------------------------------------------
struct Bits {
  const uint8_t* p;    // the next byte to load
  const uint8_t* end;  // one past the chunk's last byte
  uint64_t buf;        // the next n bits, from the top; the bits below them are 0 or the stream's own next bits
  uint32_t n;
  bool over;           // a read wanted bits past `end`
};

GPR_HD Bits bits_at(const uint8_t* p, const uint8_t* end) { return Bits{p, end, 0ull, 0u, false}; }

// at least 57 bits in buf, or every byte of the chunk; called with n < 32
GPR_HD void refill(Bits& r) {
  if (r.end - r.p >= 8) {
    uint64_t w = 0;
    for (int k = 0; k < 8; ++k) w = (w << 8) | r.p[k];
    r.buf |= w >> r.n;  // the next 64 - n bits; the whole bytes among them are counted
    const uint32_t take = (64u - r.n) >> 3;
    r.p += take, r.n += take * 8u;
  } else {
    while (r.n <= 56u && r.p < r.end) r.buf |= (uint64_t)*r.p++ << (56u - r.n), r.n += 8u;
  }
}

// the next k bits, 1 <= k <= 32; 0 and `over` set if the chunk has fewer
GPR_HD uint64_t take(Bits& r, uint32_t k) {
  if (r.n < k) {
    refill(r);
    if (r.n < k) {
      r.over = true;
      r.n = 0;
      return 0;
    }
  }
  const uint64_t v = r.buf >> (64u - k);
  r.buf <<= k, r.n -= k;
  return v;
}

// the next k bits, 1 <= k <= 64
GPR_HD uint64_t take_wide(Bits& r, uint32_t k) {
  if (k <= 32u) return take(r, k);
  const uint64_t hi = take(r, k - 32u);
  return (hi << 32) | take(r, 32u);
}

// an unsigned varint (Go's binary.ReadUvarint) read byte by byte from the bit stream
GPR_HD uint64_t uvarint(Bits& r, bool* bad) {
  uint64_t x = 0;
  for (uint32_t i = 0, s = 0; i < 10u; ++i, s += 7u) {
    const uint64_t b = take(r, 8u);
    if (r.over) return 0;
    if (b < 0x80u) {
      if (i == 9u && b > 1u) *bad = true;
      return x | (b << s);
    }
    x |= (b & 0x7fu) << s;
  }
  *bad = true;
  return x;
}

// ---- one chunk ---------------------------------------------------------------------------------------------------
// Decodes the chunk [p, end) and calls emit(ts_ms, value) for each sample, in order; stops at the first fault.
// Returns that fault's bit, as Prometheus' iterator reports its first error (0 = the chunk is well formed).  A bad
// varint is found at its last byte, before the rest of its sample is read; a read past the end leaves every later
// bit 0, so no window can be missing after it.
template <typename Emit>
GPR_HD uint32_t decode_chunk(const uint8_t* p, const uint8_t* end, Emit&& emit) {
  if (end - p < 2) return kShort;
  const uint32_t count = ((uint32_t)p[0] << 8) | p[1];
  Bits r = bits_at(p + 2, end);
  bool bad_varint = false, no_window = false;
  uint64_t t = 0, delta = 0, v = 0;  // wrapping arithmetic, as Go's
  uint32_t sig = 0, trail = 0;       // the XOR window: significant bits (0 = none yet) and their shift
  for (uint32_t i = 0; i < count; ++i) {
    if (i == 0) {
      const uint64_t u = uvarint(r, &bad_varint);
      t = (u >> 1) ^ (0ull - (u & 1u));  // zigzag
      v = take_wide(r, 64u);
    } else {
      if (i == 1) {
        delta = uvarint(r, &bad_varint);
      } else {
        uint32_t sz = 0;
        if (take(r, 1u)) sz = !take(r, 1u) ? 14u : !take(r, 1u) ? 17u : !take(r, 1u) ? 20u : 64u;
        if (sz) {
          uint64_t dod = take_wide(r, sz);
          if (sz < 64u && dod > (1ull << (sz - 1u))) dod -= 1ull << sz;
          delta += dod;
        }
      }
      t += delta;
      if (take(r, 1u)) {
        if (take(r, 1u)) {
          const uint32_t lead = (uint32_t)take(r, 5u);
          const uint32_t m = (uint32_t)take(r, 6u);
          sig = m ? m : 64u;
          // as Prometheus' uint8 arithmetic: a window wider than 64 bits reads its bits and changes nothing
          trail = (64u - lead - sig) & 0xffu;
        } else if (sig == 0) {
          no_window = true;
          break;
        }
        const uint64_t x = take_wide(r, sig);
        if (trail < 64u) v ^= x << trail;
      }
    }
    if (r.over || bad_varint) break;
    emit((int64_t)t, text::bits_to_double(v));
  }
  return bad_varint ? kBadVarint : r.over ? kOverrun : no_window ? kNoWindow : 0u;
}

// What is wrong with chunk c's bounds: chunk_bytes[0] must be 0, and each chunk at least its 2-byte header.
GPR_HD uint32_t bound_faults(const uint64_t* chunk_bytes, uint64_t c) {
  uint32_t f = (c == 0 && chunk_bytes[0] != 0) ? kBadChunkStart : 0u;
  if (chunk_bytes[c + 1] < chunk_bytes[c]) f |= kBadChunkOrder;
  else if (chunk_bytes[c + 1] - chunk_bytes[c] < 2u) f |= kShort;
  return f;
}

// The sample count in a chunk's header (its bounds are good).
GPR_HD uint32_t chunk_count(const uint8_t* p) { return ((uint32_t)p[0] << 8) | p[1]; }

// What is wrong with chunk c: its bounds, then its decode.  data[b - data_base] is byte b of the batch.
GPR_HD uint32_t chunk_faults(const uint64_t* chunk_bytes, const uint8_t* data, uint64_t data_base, uint64_t c) {
  const uint32_t f = bound_faults(chunk_bytes, c);
  if (f) return f;
  const uint8_t* p = data + (chunk_bytes[c] - data_base);
  return decode_chunk(p, data + (chunk_bytes[c + 1] - data_base), [](int64_t, double) {});
}

struct ScatterArgs {
  const uint64_t* series_chunks;  // n_series + 1, device
  const uint32_t* rows;           // n_series, device
  const uint64_t* chunk_bytes;    // n_chunks + 1, device
  const uint8_t* data;            // byte b of the batch at data[b - data_base]
  uint64_t data_base;
  uint64_t base, end;             // the chunks [base, end) of the batch this launch merges
  uint32_t n_series;
  uint32_t s_base;                // the series chunk `base` belongs to
  float* plane;
  unsigned long long* stats;      // [2]: samples outside the window, in-window values kept non-zero by to_f32
  text::Grid g;
};

__global__ void __launch_bounds__(kThreads) k_chunks_scatter(const ScatterArgs a) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint64_t n_groups = (a.end - a.base + 31u) / 32u;
  uint32_t n_oow = 0, n_tiny = 0;
  for (uint64_t grp = (uint64_t)blockIdx.x * kWarps + warp; grp < n_groups; grp += (uint64_t)gridDim.x * kWarps) {
    const uint64_t c0 = a.base + grp * 32u;
    const uint64_t c = c0 + lane;
    uint32_t s = 0;
    if (lane == 0) s = samples::series_in(a.series_chunks, a.s_base, a.n_series, c0);
    s = __shfl_sync(0xffffffffu, s, 0);
    if (c < a.end) {
      s = samples::series_from(a.series_chunks, a.n_series, s, c);
      const uint32_t row = __ldg(a.rows + s);
      const uint8_t* p = a.data + (__ldg(a.chunk_bytes + c) - a.data_base);
      const uint8_t* e = a.data + (__ldg(a.chunk_bytes + c + 1) - a.data_base);
      decode_chunk(p, e, [&](int64_t ts, double v) { samples::scatter_sample(a.g, a.plane, row, ts, v, n_oow, n_tiny); });
    }
  }
  const uint32_t w_oow = __reduce_add_sync(0xffffffffu, n_oow), w_tiny = __reduce_add_sync(0xffffffffu, n_tiny);
  if (lane == 0) {
    if (w_oow) atomicAdd(a.stats + 0, (unsigned long long)w_oow);
    if (w_tiny) atomicAdd(a.stats + 1, (unsigned long long)w_tiny);
  }
}

struct CheckArgs {
  const uint64_t* chunk_bytes;  // n_chunks + 1, device
  const uint8_t* data;          // byte b of the batch at data[b - data_base]
  uint64_t data_base;
  uint64_t base, end;           // the chunks [base, end) to check
  unsigned int* bad;            // the chunk_faults() bits of every chunk, OR-ed
  unsigned long long* first;    // the first faulty chunk (atomicMin; starts at ~0)
  unsigned long long* n_in;     // += the sample counts of the good chunks
};

// Checks chunks before anything is written: decodes each one without writing and reports its fault bits.
__global__ void __launch_bounds__(256) k_chunks_check(const CheckArgs a) {
  uint32_t f_all = 0, n = 0;
  if (a.base == 0 && blockIdx.x == 0 && threadIdx.x == 0 && a.chunk_bytes[0] != 0) {  // also without chunks
    f_all = kBadChunkStart;
    atomicMin(a.first, 0ull);
  }
  for (uint64_t c = a.base + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c < a.end;
       c += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t f = chunk_faults(a.chunk_bytes, a.data, a.data_base, c);
    if (f) {
      f_all |= f;
      atomicMin(a.first, (unsigned long long)c);
    } else {
      n += chunk_count(a.data + (__ldg(a.chunk_bytes + c) - a.data_base));
    }
  }
  if (f_all) atomicOr(a.bad, f_all);
  if (n) atomicAdd(a.n_in, (unsigned long long)n);
}

}  // namespace chunks
}  // namespace gpr
