// gpr_text.cuh — device-side parse of a Prometheus range-query response (matrix JSON) straight into
// the dense (pod x gpu x t) f32 tensor in HBM.
//
// Wire shape: the one gpu-pruner/src/bin/querytest.rs:41-53 walks — per series a label
// map and a list of [<unix time>, "<value>"] pairs:
//     {"metric":{...},"values":[[1700000000,"0"],[1700000001,"37"],...]}
// More than 99 % of the bytes are the sample lists; the label maps (hashing, string work, ~1 % of the
// bytes) stay on the host (gpu-pruner_b200/host/ingest_device.cpp), which turns them into one
// `Span` per series: where its sample list sits in the text and which tensor row it feeds.
//
// Two passes over the text, both flat over bytes (the work is balanced whatever the series lengths are):
//   scan  : report the offsets of `},"values":[` and `"]]` — the two byte patterns that delimit a
//           sample list.  Neither can occur inside a JSON string (a raw '"' ends the string), so in the
//           compact encoding Prometheus emits they are exact; the host cross-checks every series and
//           falls back to the CPU parser for anything else (pretty-printed JSON, histograms, ...).
//   parse : every '[' inside a span starts a sample.  A warp takes a 4 KB tile of text, lists its '['
//           offsets, and hands ONE SAMPLE TO EVERY LANE per round (parse_candidate below), so the 32
//           lanes execute the same digit loops on similar input at the same time.
//
// What a sample becomes: the value, rounded exactly like strtod + (float) (Clinger's fast path, else
// Eisel-Lemire with the 128-bit table of gpr_pow10_table.h), merged into cell (row, column(ts)) with a
// NaN-aware max.  `max` is what the consumer computes over the row (max_over_time,
// gpu-pruner/src/query.promql.j2:10,16), so two samples of a series that fall into one
// column, samples arriving in any order and several threads hitting one cell all give the same tensor —
// no ordering or collision bookkeeping.  Cells start as 0xFFFFFFFF (a NaN whose bit pattern is -1 as an
// int): for the non-negative values DCGM exports the merge is one integer atomicMax without a return
// value (RED.MAX.S32 at L2).
//
// Strictness instead of generality: a sample that is not exactly `[digits[.digits],"number|NaN|±Inf"]`,
// a number with more than 19 significant digits, or one of the rare inputs Eisel-Lemire declines marks
// the whole SPAN `hard`; the host re-parses the rows of hard spans with the CPU text parser (strtod) and
// overwrites them.  So the tensor equals the CPU ingest (gpu-pruner_b200/host/ingest.cpp) for every
// input, and malformed input raises the same errors.
//
// Everything that decides a byte's meaning is in GPR_HD functions that also compile as plain C++:
// tests/cpp/text_emul.cpp runs the very same code candidate by candidate on the CPU against the CPU ingest.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define GPR_HD __host__ __device__ __forceinline__
#else
#define GPR_HD inline
#endif

#include "gpr_pow10_table.h"

namespace gpr {
namespace text {

constexpr uint32_t kSpanShared = 1u;  // in : several series feed this row (informational: every merge is atomic)
constexpr uint32_t kSpanHard = 2u;    // out: the host must re-parse this span's row
constexpr uint32_t kScanBytes = 16;   // bytes per thread, scan pass
constexpr uint32_t kTileBytes = 4096; // bytes per warp and step, parse pass
constexpr uint32_t kTileHalo = 96;    // a sample may run this far past the tile that owns its '['
constexpr uint32_t kMaxSample = 80;   // longest sample the device parser accepts (longer: hard)
constexpr uint32_t kTextPad = 256;    // zero bytes the caller guarantees after the text

struct Span {        // mirrors gpr_text_span (include/gpr.h)
  uint64_t begin;    // offset of the first byte after `"values":[`
  uint64_t end;      // offset of the ']' that closes the list
  uint32_t row;      // destination row = pod * G + slot
  uint32_t flags;    // kSpan*
  uint32_t n_in;     // out: samples parsed
  uint32_t n_oow;    // out: samples outside the window
  uint32_t n_tiny;   // out: values below the f32 denormal range, clamped to +-denorm_min
  uint32_t reserved;
};

// Time axis of the destination (gpu-pruner_b200/host/ingest_internal.hpp column_of is the same rule), in
// MILLISECONDS — the resolution of Prometheus timestamps, so membership and bucketing are exact.
// A sample is inside the window iff t_lo < ts <= t_end  (PromQL's [Nm] selector evaluated at t_end,
// left-open as in Prometheus 3.x).  Buckets are `step` wide and end at t_end:
//     back = (t_end - ts) / step            0 = newest bucket
//     col  = (col_end - back) mod T
// A dense window has col_end = T - 1 (column c = bucket T-1-c); the resident ring of daemon mode passes
// the ring position of its newest bucket.
struct PowerSnap {   // how power samples are stored against the veto threshold: power_snap() / snap_power() below
  double thr;        // NaN = no snapping
  float up, down;    // smallest f32 >= thr, and the f32 just below it
};

struct Grid {
  int64_t t_end;     // newest millisecond (inclusive)
  int64_t t_lo;      // t_end - window (exclusive)
  uint32_t step;     // milliseconds per column, > 0
  uint32_t T;        // columns of the plane
  uint32_t col_end;  // column of the newest bucket
  uint32_t pad;
  uint64_t ld;       // elements between rows of the plane
  PowerSnap power;   // power_snap(threshold) for the power plane, power_snap(0) for the util plane
};

constexpr int64_t kBadTs = INT64_MIN / 4;  // timestamp that is no sane epoch time: outside any window

GPR_HD int64_t column_of(const Grid& g, int64_t ts) {
  if (ts > g.t_end || ts <= g.t_lo) return -1;
  const uint64_t d = (uint64_t)(g.t_end - ts);
  const uint64_t back = d <= 0xffffffffull ? (uint64_t)((uint32_t)d / g.step) : d / g.step;
  if (back >= g.T) return -1;
  return back <= g.col_end ? (int64_t)(g.col_end - back) : (int64_t)(g.col_end + g.T - back);
}

// ---- numbers -------------------------------------------------------------------------------------------
// exact powers of ten: 10^0 .. 10^22 are representable in binary64
GPR_HD double pow10_exact(int e) {
  // a switch (not a table) keeps this usable from host and device without a __constant__ copy
  switch (e) {
    case 0: return 1e0;   case 1: return 1e1;   case 2: return 1e2;   case 3: return 1e3;
    case 4: return 1e4;   case 5: return 1e5;   case 6: return 1e6;   case 7: return 1e7;
    case 8: return 1e8;   case 9: return 1e9;   case 10: return 1e10; case 11: return 1e11;
    case 12: return 1e12; case 13: return 1e13; case 14: return 1e14; case 15: return 1e15;
    case 16: return 1e16; case 17: return 1e17; case 18: return 1e18; case 19: return 1e19;
    case 20: return 1e20; case 21: return 1e21; default: return 1e22;
  }
}

GPR_HD void mul64(uint64_t a, uint64_t b, uint64_t* hi, uint64_t* lo) {
#if defined(__CUDA_ARCH__)
  *lo = a * b;
  *hi = __umul64hi(a, b);
#else
  const unsigned __int128 p = (unsigned __int128)a * b;
  *lo = (uint64_t)p, *hi = (uint64_t)(p >> 64);
#endif
}

GPR_HD int clz64(uint64_t x) {
#if defined(__CUDA_ARCH__)
  return __clzll((long long)x);
#else
  return __builtin_clzll(x);
#endif
}

GPR_HD double bits_to_double(uint64_t b) {
#if defined(__CUDA_ARCH__)
  return __longlong_as_double((long long)b);
#else
  double d;
  memcpy(&d, &b, sizeof d);
  return d;
#endif
}

// Eisel-Lemire: man * 10^e10 (man != 0, at most 19 decimal digits) -> the correctly rounded binary64,
// or false when this method cannot decide (caller marks the span hard; the CPU's strtod decides).
// The formulation with truncated 128-bit powers of ten and the two carry checks of the Wuffs / Go
// strconv implementations; subnormal and overflowing results are declined too.
GPR_HD bool eisel_lemire(uint64_t man, int e10, double* out) {
  if (e10 < kPow10Min || e10 > kPow10Max) return false;
#if defined(__CUDA_ARCH__)
  const uint64_t p_hi = kPow10MantDev[e10 - kPow10Min][0], p_lo = kPow10MantDev[e10 - kPow10Min][1];
#else
  const uint64_t p_hi = kPow10MantHost[e10 - kPow10Min][0], p_lo = kPow10MantHost[e10 - kPow10Min][1];
#endif
  const int clz = clz64(man);
  man <<= clz;
  // floor(log2(10^e10)) = (217706 * e10) >> 16 for the table's range
  uint64_t exp2 = (uint64_t)(((217706ll * e10) >> 16) + 64 + 1023) - (uint64_t)clz;
  uint64_t x_hi, x_lo;
  mul64(man, p_hi, &x_hi, &x_lo);
  if ((x_hi & 0x1FF) == 0x1FF && x_lo + man < man) {  // the truncated low half could carry into the result
    uint64_t y_hi, y_lo;
    mul64(man, p_lo, &y_hi, &y_lo);
    uint64_t m_hi = x_hi;
    const uint64_t m_lo = x_lo + y_hi;
    if (m_lo < x_lo) ++m_hi;
    if ((m_hi & 0x1FF) == 0x1FF && m_lo + 1 == 0 && y_lo + man < man) return false;
    x_hi = m_hi, x_lo = m_lo;
  }
  const uint64_t msb = x_hi >> 63;
  uint64_t mant = x_hi >> (msb + 9);
  exp2 -= 1 ^ msb;
  if (x_lo == 0 && (x_hi & 0x1FF) == 0 && (mant & 3) == 1) return false;  // exactly half way: undecidable here
  mant += mant & 1;
  mant >>= 1;
  if (mant >> 53) {
    mant >>= 1;
    ++exp2;
  }
  if (exp2 - 1 >= 0x7FF - 1) return false;  // subnormal or overflow: leave it to strtod
  *out = bits_to_double((exp2 << 52) | (mant & 0x000FFFFFFFFFFFFFull));
  return true;
}

// what gph::to_f32 does (ingest.cpp): a non-zero value that rounds to 0 in f32 stays non-zero
GPR_HD float to_f32(double x, uint32_t* tiny) {
  float f = (float)x;
  if (x != 0.0 && f == 0.0f && x == x) {
#if defined(__CUDA_ARCH__)
    f = __int_as_float(x < 0 ? 0x80000001 : 0x00000001);
#else
    union { uint32_t u; float f; } c;
    c.u = x < 0 ? 0x80000001u : 0x00000001u;
    f = c.f;
#endif
    ++*tiny;
  }
  return f;
}

GPR_HD float f32_from_bits(uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __uint_as_float(b);
#else
  float f;
  memcpy(&f, &b, sizeof f);
  return f;
#endif
}
GPR_HD uint32_t f32_bits(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(f);
#else
  uint32_t b;
  memcpy(&b, &f, sizeof b);
  return b;
#endif
}
GPR_HD float quiet_nan_f32() { return f32_from_bits(0x7fc00000u); }
constexpr uint32_t kFillBits = 0xFFFFFFFFu;  // "no sample": a NaN that is -1 as an int (below every non-negative value)

// ---- power samples against the veto threshold ------------------------------------------------------------
// The veto compares the f32 row max with up = the smallest f32 >= thr (gpr_decide), which equals Prometheus'
// float64 `x >= thr` only for samples that are f32 already: a reading within half an f32 ulp below thr
// (149.999999 for 150) rounds UP to `up` and would veto.  So power samples are stored snapped:
//     x >= thr  ->  at least up          x < thr  ->  at most down, the f32 just below up
// after which `max >= up` holds exactly when some x >= thr, for every float64 threshold.  NaN and
// +-Inf are left alone (they compare the same either way); thr = NaN turns the snap off (util plane, or no
// power clause: a threshold of 0 or NaN, the truthiness rule of the template).  PowerSnap is defined above Grid.
GPR_HD float f32_next_up(float f) {  // toward +Inf; f is neither NaN nor +Inf
  const uint32_t b = f32_bits(f);
  if ((b & 0x7fffffffu) == 0u) return f32_from_bits(1u);
  return f32_from_bits((b >> 31) ? b - 1u : b + 1u);
}
GPR_HD float f32_next_down(float f) {  // toward -Inf; f is neither NaN nor -Inf
  const uint32_t b = f32_bits(f);
  if ((b & 0x7fffffffu) == 0u) return f32_from_bits(0x80000001u);
  return f32_from_bits((b >> 31) ? b + 1u : b - 1u);
}

// smallest f32 >= thr: (m >= threshold_up(thr)) in f32 equals ((double)m >= thr) for every f32 m
GPR_HD float threshold_up(double thr) {
  float t = (float)thr;
  if ((double)t < thr) t = f32_next_up(t);
  return t;
}

GPR_HD PowerSnap power_snap(double thr) {
  PowerSnap s;
  if (thr != thr || thr == 0.0) {
    s.thr = bits_to_double(0x7ff8000000000000ull);
    s.up = s.down = 0.0f;
    return s;
  }
  s.thr = thr;
  s.up = threshold_up(thr);
  s.down = f32_bits(s.up) == 0xff800000u ? s.up : f32_next_down(s.up);  // thr = -Inf: nothing is below it
  return s;
}

// x: the sample in float64, f: its f32 (to_f32)
GPR_HD float snap_power(double x, float f, const PowerSnap& s) {
  if (x >= s.thr) return f < s.up ? s.up : f;
  if (x < s.thr && f >= s.up) return s.down;
  return f;
}

// ---- one sample ------------------------------------------------------------------------------------------
// `Src` is anything with `uint8_t operator[](uint32_t) const` (shared-memory tile on the device, a plain
// buffer in the emulation).  Offsets are relative to the tile; nothing at or beyond p + kMaxSample is read.
//
// [-+]digits[.digits][(e|E)[-+]digits] at t[p...] -> *v.  Prometheus prints sample values with strconv 'f' and
// switches to 'e' below 1e-6 and from 1e21 on (util/jsonutil MarshalFloat), so both forms occur.
// Returns the offset after the number, 0 = not convertible here.  `snap`: power_snap() of the plane (see above).
template <typename Src>
GPR_HD uint32_t parse_value(const Src& t, uint32_t p, uint32_t limit, float* val, uint32_t* tiny, const PowerSnap& snap) {
  bool neg = false;
  uint32_t c = t[p];
  if (c == '-' || c == '+') neg = c == '-', c = t[++p];
  uint64_t m = 0;
  int sig = 0, frac = 0;
  bool any = false, dot = false;
  for (; p < limit; c = t[++p]) {
    const uint32_t d = c - '0';
    if (d < 10u) {
      any = true;
      if (sig == 19) {
        if (d != 0 || !dot) return 0;  // a 20th significant digit (trailing fractional zeros are harmless)
        continue;
      }
      m = m * 10 + d;
      sig += (m != 0);
      frac += dot;
    } else if (c == '.' && !dot && any) {
      dot = true;
      any = false;  // at least one digit must follow the point
    } else {
      break;
    }
  }
  if (!any || p >= limit) return 0;
  int e10 = -frac;
  bool has_exp = false;
  if (c == 'e' || c == 'E') {
    has_exp = true;
    c = t[++p];
    bool eneg = false;
    if (c == '-' || c == '+') eneg = c == '-', c = t[++p];
    int ex = 0, nd = 0;
    for (; c - '0' < 10u && nd < 4; c = t[++p], ++nd) ex = ex * 10 + (int)(c - '0');
    if (nd == 0 || nd > 3) return 0;
    e10 += eneg ? -ex : ex;
  }
  float f;
  if (m == 0) {
    f = 0.0f;
  } else if (!dot && !has_exp && m < (1ull << 24)) {
    f = (float)(uint32_t)m;  // every DCGM_FI_DEV_GPU_UTIL / POWER_USAGE integer: exact
  } else {
    double d;
    if (m > (1ull << 53))  // "13098385200945040.0": trailing zeros carry no information, and without them
      while (m % 10 == 0) m /= 10, ++e10;  // the exact path below applies (rare; 64-bit division is slow)
    if (m <= (1ull << 53) && e10 >= -22 && e10 <= 22) {
      d = (double)m;  // exact; one IEEE multiplication or division by an exact power of ten: correctly rounded (Clinger)
      if (e10 < 0) d = d / pow10_exact(-e10);
      else if (e10 > 0) d = d * pow10_exact(e10);
    } else if (!eisel_lemire(m, e10, &d)) {
      return 0;
    }
    // (the exact integer and zero paths above need no snap: a sample that is an f32 compares the same either way)
    f = to_f32(d, tiny);
    *val = snap_power(neg ? -d : d, neg ? -f : f, snap);
    return p;
  }
  *val = neg ? -f : f;
  return p;
}

// the same for a plane without a power clause (utilisation, PROF ratios): plain rounding
template <typename Src>
GPR_HD uint32_t parse_value(const Src& t, uint32_t p, uint32_t limit, float* val, uint32_t* tiny) {
  return parse_value(t, p, limit, val, tiny, power_snap(0.0));
}

// t[p] == '['.  `[digits[.digits],` -> milliseconds.  At most 13 integer and 3 fractional digits (Prometheus
// prints timestamps with millisecond resolution; anything finer is declined and goes to the CPU parser, whose
// llround(strtod() * 1000) this reproduces exactly for such input).  Returns the offset of the ','.
template <typename Src>
GPR_HD uint32_t parse_timestamp(const Src& t, uint32_t p, int64_t* ts) {
  uint64_t ip = 0;
  uint32_t q = p + 1, c = t[q];
  const uint32_t q0 = q;
  for (; c - '0' < 10u && q - q0 < 14; c = t[++q]) ip = ip * 10 + (c - '0');
  if (q == q0 || q - q0 > 13) return 0;
  uint32_t ms = 0;
  if (c == '.') {
    c = t[++q];
    const uint32_t f0 = q;
    uint32_t scale = 100;
    for (; c - '0' < 10u && q - f0 < 4; c = t[++q]) ms += (c - '0') * scale, scale /= 10;
    if (q == f0 || q - f0 > 3) return 0;
  }
  if (c != ',') return 0;
  *ts = ip < 4000000000000ull ? (int64_t)(ip * 1000 + ms) : kBadTs;
  return q;
}

// Returns the offset after the sample's ']' or 0 (hard).
template <typename Src>
GPR_HD uint32_t parse_sample(const Src& t, uint32_t p, int64_t* ts, float* val, uint32_t* tiny, const PowerSnap& snap) {
  const uint32_t limit = p + kMaxSample - 2;
  uint32_t q = parse_timestamp(t, p, ts);
  if (q == 0 || t[q + 1] != '"') return 0;
  q += 2;  // past ,"
  const uint32_t c = t[q];
  if (c == 'N') {
    if (t[q + 1] != 'a' || t[q + 2] != 'N') return 0;
    *val = quiet_nan_f32();
    q += 3;
  } else if (c == 'I' || ((c == '+' || c == '-') && t[q + 1] == 'I')) {
    const bool neg = c == '-';
    if (c != 'I') ++q;
    if (t[q + 1] != 'n' || t[q + 2] != 'f') return 0;
    *val = f32_from_bits(neg ? 0xff800000u : 0x7f800000u);
    q += 3;
  } else {
    q = parse_value(t, q, limit, val, tiny, snap);
    if (q == 0) return 0;
  }
  if (t[q] != '"' || t[q + 1] != ']') return 0;
  return q + 2;
}

// ---- spans -------------------------------------------------------------------------------------------------
// index of the first span whose end lies beyond `pos` (spans sorted by begin, non-overlapping)
GPR_HD uint32_t find_span(const Span* __restrict__ spans, uint32_t n, uint64_t pos) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (spans[mid].end > pos) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

// ---- the scan pass: one slice of kScanBytes ----------------------------------------------------------------
// Sink: void values_open(uint64_t pos_of_closing_brace), void values_close(uint64_t pos_of_quote)
template <typename Sink>
GPR_HD void scan_slice(const uint8_t* __restrict__ t, uint64_t n, uint64_t slice, Sink& sink) {
  const uint64_t b = slice * kScanBytes;
  if (b >= n) return;
  // the slice's 16 bytes plus 4 of look-ahead live in registers (the text is padded, so reading
  // past n is safe; `t` is 16-byte aligned and slices are 16 bytes, so the vector load is aligned)
  uint32_t w[5];
#if defined(__CUDA_ARCH__)
  const uint4 x = *reinterpret_cast<const uint4*>(t + b);
  w[0] = x.x, w[1] = x.y, w[2] = x.z, w[3] = x.w;
  w[4] = *reinterpret_cast<const uint32_t*>(t + b + 16);
#else
  memcpy(w, t + b, sizeof w);
#endif
#define GPR_TEXT_BYTE(k) ((w[(k) >> 2] >> (((k)&3) * 8)) & 0xffu)
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int k = 0; k < (int)kScanBytes; ++k) {
    const uint64_t p = b + (uint64_t)k;
    if (p >= n) break;
    const uint32_t c = GPR_TEXT_BYTE(k);
    if (c == '"') {
      if (GPR_TEXT_BYTE(k + 1) == ']' && GPR_TEXT_BYTE(k + 2) == ']') sink.values_close(p);
    } else if (c == '}') {
      // },"values":[   (rare: once per series, plus the '}' that end label maps)
      if (t[p + 1] == ',' && t[p + 2] == '"' && t[p + 3] == 'v' && t[p + 4] == 'a' && t[p + 5] == 'l' &&
          t[p + 6] == 'u' && t[p + 7] == 'e' && t[p + 8] == 's' && t[p + 9] == '"' && t[p + 10] == ':' &&
          t[p + 11] == '[')
        sink.values_open(p);
    }
  }
#undef GPR_TEXT_BYTE
}

// ---- the parse pass: one candidate ('[' at tile offset o) ------------------------------------------------------
// Sink: void put(uint64_t cell, float v)       merge v into plane[cell] (NaN-aware max; NaN never replaces)
//       void hard(uint32_t span)
//       void count(uint32_t span, uint32_t n_in, uint32_t n_oow, uint32_t n_tiny)   (the sink aggregates)
// `tile` holds the text bytes [tile_off, tile_off + kTileBytes + kTileHalo).  `s` is a cursor: on entry any
// index <= the candidate's span (the kernel starts it at find_span(tile_off) and keeps it per lane, candidates
// of a lane come in increasing offset order); on return the candidate's span.
template <typename Src, typename Sink>
GPR_HD void parse_candidate(const Src& tile, uint64_t tile_off, uint32_t o, const Span* __restrict__ spans,
                            uint32_t n_spans, uint32_t& s, const Grid& g, Sink& sink) {
  const uint64_t pos = tile_off + o;
  while (s < n_spans && spans[s].end <= pos) ++s;
  if (s >= n_spans || spans[s].begin > pos) return;  // a '[' outside every sample list (label text)
  const uint64_t se = spans[s].end;
  int64_t ts;
  float v;
  uint32_t tiny = 0;
  const uint32_t q = parse_sample(tile, o, &ts, &v, &tiny, g.power);
  // between samples exactly one ',' ; after the last one the list closes at `se`
  if (q == 0 || tile_off + q > se || !(tile_off + q == se || (tile[q] == ',' && tile[q + 1] == '['))) {
    sink.hard(s);
    return;
  }
  const int64_t col = column_of(g, ts);
  sink.count(s, 1u, col < 0 ? 1u : 0u, col < 0 ? 0u : tiny);  // clamped values are counted where they are stored
  if (col >= 0) sink.put((uint64_t)spans[s].row * g.ld + (uint64_t)col, v);
}

// reference merge for host-side sinks (the device sink is atomic, gpr_text_kernels.cuh)
GPR_HD void merge_cell_bits(uint32_t* cell, float v) {
  if (v != v) return;
  const float c = f32_from_bits(*cell);
  if (c != c || c < v) *cell = f32_bits(v);
}

}  // namespace text
}  // namespace gpr
