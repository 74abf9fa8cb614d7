// Host emulation of gpr_chunks_scatter: k_chunks_check and k_chunks_scatter compiled from the SOURCE TEXT of
// gpu-pruner_b200/csrc/gpr_chunks.cuh (with gpr_samples.cuh, whose series search, check and scatter_sample it uses)
// under tests/cpp/cuda_shim.hpp, with the text kernel's atomic_merge cut out of gpr_text_kernels.cuh, launched the
// way gpr_api.cu launches them.
//
// tests/test_chunks_emul.py writes the extracts, a directory of batch files and runs
//     chunks_emul SM_COUNT DIR
// DIR/params.txt: n_series n_rows T t_end_ms t_lo_ms step_ms col_end power_threshold piece shift
//   piece 0    = a device batch: the series check kernel, then one check launch and one scatter launch over all
//                chunks, read in place
//   piece > 0  = a host batch: the index arrays checked on the host, then the pieces of at most `piece` bytes of whole
//                chunks, at least one, (gpr::samples::for_each_cut, as gpr_api.cu cuts them), each copied into a buffer of exactly
//                its size (a read past a piece is an AddressSanitizer error), checked piece by piece, then scattered
//                piece by piece
//   shift      = the data sits `shift` bytes past a 16-byte boundary
// DIR/series.u64 rows.u32 cbytes.u64 data.u8 plane.u32 (the plane before the call, n_rows x T)
// DIR/out.bin: u32 fault bits (0 = accepted), u32 0, u64 first bad chunk (~0 if none), u64 n_in, u64 n_oow,
// u64 n_tiny, then the plane after the call.  A rejected batch leaves the plane as it was.  The host walk of
// chunk_faults and the check kernel must agree (exit 3).  A host batch whose chunk_bytes rises from 0 but has a chunk
// with bad bounds is rejected by the host walk alone, which then decodes the other chunks as gpr_api.cu does.
#include "cuda_shim.hpp"

static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) {
  unsigned long long old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (v < old && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_SEQ_CST, __ATOMIC_RELAXED)) {
  }
  return old;
}

#include "../../gpu-pruner_b200/csrc/gpr_text.cuh"
namespace gpr {
namespace text {
#include "text_kernel_extract.inc"
}
}  // namespace gpr
namespace gpr {
namespace samples {
#include "samples_extract.inc"
}
}  // namespace gpr
namespace gpr {
namespace chunks {
#include "chunks_extract.inc"
}
}  // namespace gpr

namespace gc = gpr::chunks;
namespace gs = gpr::samples;

template <class T>
static std::vector<T> read_all(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  if (!f) {
    fprintf(stderr, "cannot read %s\n", path.c_str());
    exit(2);
  }
  f.seekg(0, std::ios::end);
  std::vector<T> v((size_t)f.tellg() / sizeof(T));
  f.seekg(0);
  f.read(reinterpret_cast<char*>(v.data()), (std::streamsize)(v.size() * sizeof(T)));
  return v;
}

// an exact-size copy of n bytes, `shift` bytes past a 16-byte boundary
struct Bytes {
  std::vector<unsigned char> store;
  uint8_t* p = nullptr;
  Bytes(const uint8_t* src, size_t n, unsigned shift) {
    store.resize(n + 32);
    uintptr_t a = reinterpret_cast<uintptr_t>(store.data());
    a = ((a + 15) & ~(uintptr_t)15) + shift;
    p = reinterpret_cast<uint8_t*>(a);
    if (n) memcpy(p, src, n);
  }
};

static unsigned g_sm = 1;

static void check(const gc::CheckArgs& a) {
  if (a.end <= a.base) return;
  const unsigned blocks = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((a.end - a.base + 255) / 256, g_sm * 8));
  launch(blocks, 256, 0, [&] { gc::k_chunks_check(a); });
}

static void scatter(const gc::ScatterArgs& a) {
  if (a.end <= a.base) return;
  const uint64_t groups = (a.end - a.base + 31) / 32;
  const unsigned blocks =
      (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((groups + gc::kWarps - 1) / gc::kWarps, g_sm * 8));
  launch(blocks, gc::kThreads, 0, [&] { gc::k_chunks_scatter(a); });
}

int main(int argc, char** argv) {
  if (argc != 3) {
    fprintf(stderr, "usage: chunks_emul SM_COUNT DIR\n");
    return 2;
  }
  g_sm = (unsigned)atoi(argv[1]);
  g_max_resident_ctas = 4;  // CTAs of the check and the scatter never wait for one another
  const std::string dir = argv[2];
  std::ifstream pf(dir + "/params.txt");
  uint32_t n_series, n_rows, T, col_end;
  long long t_end, t_lo, step;
  double thr;
  unsigned long long piece;
  unsigned shift;
  if (!(pf >> n_series >> n_rows >> T >> t_end >> t_lo >> step >> col_end >> thr >> piece >> shift)) return 2;
  const std::vector<uint64_t> series = read_all<uint64_t>(dir + "/series.u64");
  const std::vector<uint32_t> rows_v = read_all<uint32_t>(dir + "/rows.u32");
  const std::vector<uint64_t> cbytes = read_all<uint64_t>(dir + "/cbytes.u64");
  const std::vector<uint8_t> data = read_all<uint8_t>(dir + "/data.u8");
  std::vector<uint32_t> plane = read_all<uint32_t>(dir + "/plane.u32");
  if (series.size() != (size_t)n_series + 1 || rows_v.size() != n_series || plane.size() != (size_t)n_rows * T) return 2;
  std::vector<uint64_t> d_series(series), d_cbytes(cbytes);  // the "device" index arrays: exact size
  std::vector<uint32_t> d_rows(rows_v);

  // ---- the check: series, then the chunks' bounds and data; the host walk and the kernels agree
  uint32_t bad = 0;
  for (uint32_t s = 0; s < std::max(n_series, 1u); ++s)
    bad |= gs::series_faults(series.data(), rows_v.data(), n_series, s, n_rows);
  unsigned int dev_bad = 0;
  const unsigned sblocks = std::max(1u, std::min((std::max(n_series, 1u) + 255u) / 256u, g_sm * 8u));
  launch(sblocks, 256, 0, [&] { gs::k_samples_check(d_series.data(), d_rows.data(), n_series, n_rows, &dev_bad); });
  if (bad != dev_bad) {
    fprintf(stderr, "series: host check %u != device check %u\n", bad, dev_bad);
    return 3;
  }
  unsigned long long first = ~0ull, n_in = 0;
  unsigned long long stats[2] = {0, 0};
  const uint64_t n_chunks = bad ? 0 : series[n_series];
  if (!bad) {
    if (cbytes.size() != n_chunks + 1) return 2;
    uint32_t host_bad = cbytes[0] != 0 ? gc::kBadChunkStart : 0u;
    unsigned long long host_first = host_bad ? 0 : ~0ull, host_in = 0;
    for (uint64_t c = 0; c < n_chunks; ++c) {  // the bounds first: the host batch's check, and the data walk needs them
      const uint32_t f = gc::bound_faults(cbytes.data(), c);
      if (f && host_first == ~0ull) host_first = c;
      host_bad |= f;
    }
    const bool bounds_ok = host_bad == 0;
    // chunk_bytes rises from 0 (every chunk inside the data): gpr_api.cu's host walk decodes the chunks whose own
    // bounds are good, so a host batch then reports what a device batch does
    const bool rising = !(host_bad & (gc::kBadChunkStart | gc::kBadChunkOrder));
    if (rising) {
      if (data.size() != cbytes[n_chunks]) return 2;
      for (uint64_t c = 0; c < n_chunks; ++c) {
        if (gc::bound_faults(cbytes.data(), c)) continue;
        const uint32_t f = gc::chunk_faults(cbytes.data(), data.data(), 0, c);
        if (f && c < host_first) host_first = c;
        host_bad |= f;
        if (!f) host_in += gc::chunk_count(data.data() + cbytes[c]);
      }
    }
    // the kernel: on a device batch whatever its bounds, whole; on a host batch whose bounds passed, piece by piece
    if (piece == 0 || bounds_ok) {
      unsigned int k_bad = 0;
      gc::CheckArgs ck;
      ck.chunk_bytes = d_cbytes.data(), ck.bad = &k_bad, ck.first = &first, ck.n_in = &n_in;
      if (piece == 0) {
        Bytes bd(data.data(), data.size(), shift);
        ck.data = bd.p, ck.data_base = 0, ck.base = 0, ck.end = n_chunks;
        launch(std::max<unsigned>(1, std::min<uint64_t>((n_chunks + 255) / 256, g_sm * 8)), 256, 0,
               [&] { gc::k_chunks_check(ck); });
      } else {
        const auto cut = [&](uint64_t b) {
          const uint64_t* e = std::upper_bound(cbytes.data() + b + 1, cbytes.data() + n_chunks + 1, cbytes[b] + piece);
          return std::max<uint64_t>(b + 1, (uint64_t)(e - cbytes.data()) - 1);
        };
        gs::for_each_cut(series.data(), n_series, n_chunks, cut, [&](const gs::Piece& p) -> int {
          Bytes bd(data.data() + cbytes[p.begin], cbytes[p.end] - cbytes[p.begin], shift);
          gc::CheckArgs c = ck;
          c.data = bd.p, c.data_base = cbytes[p.begin], c.base = p.begin, c.end = p.end;
          check(c);
          return 0;
        });
      }
      // chunk_bytes not rising: the kernel also decodes the chunks whose own bounds are good, and may find more
      const bool agree = rising ? k_bad == host_bad && (!host_bad || first == host_first)
                                : (k_bad & host_bad) == host_bad && first <= host_first;
      if (!agree) {
        fprintf(stderr, "chunks: host check %u (chunk %llu) != kernel %u (chunk %llu)\n", host_bad, host_first, k_bad,
                first);
        return 3;
      }
      if (!host_bad && n_in != host_in) return 3;
      if (!bounds_ok) host_bad = k_bad, host_first = first;  // what a device batch reports
    }
    bad = host_bad, first = host_first;
  }
  if (!bad) {
    gc::ScatterArgs a;
    memset(&a, 0, sizeof a);
    a.g.t_end = t_end, a.g.t_lo = t_lo, a.g.step = (uint32_t)step, a.g.T = T, a.g.col_end = col_end, a.g.ld = T;
    a.g.power = gpr::text::power_snap(thr);
    a.series_chunks = d_series.data(), a.rows = d_rows.data(), a.chunk_bytes = d_cbytes.data();
    a.n_series = n_series, a.plane = reinterpret_cast<float*>(plane.data()), a.stats = stats;
    if (piece == 0) {
      Bytes bd(data.data(), data.size(), shift);
      a.data = bd.p, a.data_base = 0, a.base = 0, a.end = n_chunks, a.s_base = 0;
      scatter(a);
    } else {
      uint64_t covered = 0;  // the pieces are contiguous, cover the batch and respect the byte limit
      const auto cut = [&](uint64_t b) {
        const uint64_t* e = std::upper_bound(cbytes.data() + b + 1, cbytes.data() + n_chunks + 1, cbytes[b] + piece);
        return std::max<uint64_t>(b + 1, (uint64_t)(e - cbytes.data()) - 1);
      };
      const int rc = gs::for_each_cut(series.data(), n_series, n_chunks, cut, [&](const gs::Piece& p) -> int {
        if (p.begin != covered || p.end <= p.begin) return 1;
        if (p.end - p.begin > 1 && cbytes[p.end] - cbytes[p.begin] > piece) return 2;
        if (series[p.series] > p.begin || series[p.series + 1] <= p.begin) return 3;  // p.series owns p.begin
        covered = p.end;
        Bytes bd(data.data() + cbytes[p.begin], cbytes[p.end] - cbytes[p.begin], shift);
        gc::ScatterArgs b = a;
        b.data = bd.p, b.data_base = cbytes[p.begin], b.base = p.begin, b.end = p.end, b.s_base = p.series;
        scatter(b);
        return 0;
      });
      if (rc != 0 || covered != n_chunks) {
        fprintf(stderr, "bad piece walk (rc %d, %llu of %llu chunks)\n", rc, (unsigned long long)covered,
                (unsigned long long)n_chunks);
        return 4;
      }
    }
  }
  FILE* out = fopen((dir + "/out.bin").c_str(), "wb");
  if (!out) return 2;
  const uint32_t head[2] = {bad, 0};
  fwrite(head, 4, 2, out);
  const unsigned long long tail[4] = {bad ? first : ~0ull, bad ? 0 : n_in, stats[0], stats[1]};
  fwrite(tail, 8, 4, out);
  fwrite(plane.data(), 4, plane.size(), out);
  fclose(out);
  return 0;
}
