// Host emulation of gpr_samples_scatter: k_samples_check and k_samples_scatter compiled from the SOURCE TEXT of
// gpu-pruner_b200/csrc/gpr_samples.cuh under tests/cpp/cuda_shim.hpp (CTAs of real threads, warps with emulated
// shuffles and reductions, atomics into the plane), with the text kernel's atomic_merge cut out of
// gpr_text_kernels.cuh, launched the way gpr_api.cu launches them.
//
// tests/test_samples_emul.py writes samples_extract.inc / text_kernel_extract.inc, a directory of batch files and
// runs
//     samples_emul SM_COUNT DIR
// DIR/params.txt: n_series n_rows T t_end_ms t_lo_ms step_ms col_end power_threshold piece unaligned
//   piece 0    = a device batch: one launch over all samples, read in place
//   piece > 0  = a host batch: the pieces of gpr::samples::for_each_piece of that size, each copied into buffers of
//                exactly its size (a read past a piece is an AddressSanitizer error), one launch per piece
//   unaligned  = the timestamps and values sit 8 bytes off a 16-byte boundary (the scalar-load instantiation)
// DIR/offsets.u64 rows.u32 ts.i64 values.f64 plane.u32 (the plane before the call, n_rows x T)
// DIR/out.bin: u32 fault bits (0 = the batch was accepted), u32 0, u64 n_oow, u64 n_tiny, then the plane after the
// call.  A rejected batch leaves the plane as it was.  The host check and the check kernel must agree (exit 3).
#include "cuda_shim.hpp"

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

// an exact-size copy of src[b, e), at a 16-byte boundary or 8 bytes off one
template <class T>
struct Buf {
  std::vector<unsigned char> store;
  T* p = nullptr;
  Buf(const T* src, size_t n, bool unaligned) {
    store.resize(n * sizeof(T) + 16);
    uintptr_t a = reinterpret_cast<uintptr_t>(store.data());
    a = (a + 15) & ~(uintptr_t)15;
    if (unaligned) a += 8;
    p = reinterpret_cast<T*>(a);
    if (n) memcpy(p, src, n * sizeof(T));
  }
};

static unsigned g_sm = 1;

static void scatter(const gs::ScatterArgs& a) {
  const uint64_t chunks = (a.end - a.base + gs::kChunk - 1) / gs::kChunk;
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(chunks, (uint64_t)g_sm * 8));
  const bool vec = reinterpret_cast<uintptr_t>(a.ts) % 16 == 0 && reinterpret_cast<uintptr_t>(a.values) % 16 == 0;
  if (vec) launch(grid, gs::kThreads, 0, [&] { gs::k_samples_scatter<true>(a); });
  else launch(grid, gs::kThreads, 0, [&] { gs::k_samples_scatter<false>(a); });
}

int main(int argc, char** argv) {
  if (argc != 3) {
    fprintf(stderr, "usage: samples_emul SM_COUNT DIR\n");
    return 2;
  }
  g_sm = (unsigned)atoi(argv[1]);
  g_max_resident_ctas = 4;  // CTAs of the scatter never wait for one another
  const std::string dir = argv[2];
  std::ifstream pf(dir + "/params.txt");
  uint32_t n_series, n_rows, T, col_end;
  long long t_end, t_lo, step;
  double thr;
  unsigned long long piece;
  int unaligned;
  if (!(pf >> n_series >> n_rows >> T >> t_end >> t_lo >> step >> col_end >> thr >> piece >> unaligned)) return 2;
  const std::vector<uint64_t> offsets = read_all<uint64_t>(dir + "/offsets.u64");
  const std::vector<uint32_t> rows_v = read_all<uint32_t>(dir + "/rows.u32");
  const std::vector<int64_t> ts = read_all<int64_t>(dir + "/ts.i64");
  const std::vector<double> values = read_all<double>(dir + "/values.f64");
  std::vector<uint32_t> plane = read_all<uint32_t>(dir + "/plane.u32");
  if (offsets.size() != (size_t)n_series + 1 || rows_v.size() != n_series || plane.size() != (size_t)n_rows * T) return 2;
  // exact-size device-side copies of the series arrays
  Buf<uint64_t> d_off(offsets.data(), offsets.size(), false);
  Buf<uint32_t> d_rows(rows_v.data(), rows_v.size(), false);

  // ---- the check: on the host for a host batch, by the check kernel for a device batch; both here, and they agree
  uint32_t host_bad = 0;
  for (uint32_t s = 0; s < std::max(n_series, 1u); ++s)
    host_bad |= gs::series_faults(offsets.data(), rows_v.data(), n_series, s, n_rows);
  unsigned int dev_bad = 0;
  const unsigned blocks = std::max(1u, std::min((std::max(n_series, 1u) + 255u) / 256u, g_sm * 8u));
  launch(blocks, 256, 0, [&] { gs::k_samples_check(d_off.p, d_rows.p, n_series, n_rows, &dev_bad); });
  if (host_bad != dev_bad) {
    fprintf(stderr, "host check %u != device check %u\n", host_bad, dev_bad);
    return 3;
  }
  unsigned long long stats[2] = {0, 0};
  if (host_bad == 0) {
    const uint64_t total = offsets[n_series];
    if (ts.size() != total || values.size() != total) return 2;
    gs::ScatterArgs a;
    memset(&a, 0, sizeof a);
    a.g.t_end = t_end, a.g.t_lo = t_lo, a.g.step = (uint32_t)step, a.g.T = T, a.g.col_end = col_end, a.g.ld = T;
    a.g.power = gpr::text::power_snap(thr);
    a.offsets = d_off.p, a.rows = d_rows.p, a.n_series = n_series;
    a.plane = reinterpret_cast<float*>(plane.data());
    a.stats = stats;
    if (piece == 0) {
      if (total) {
        Buf<int64_t> bt(ts.data(), total, unaligned);
        Buf<double> bv(values.data(), total, unaligned);
        a.ts = bt.p, a.values = bv.p, a.base = 0, a.end = total, a.s_base = 0;
        scatter(a);
      }
    } else {
      uint64_t covered = 0;  // the pieces are contiguous and cover the batch
      const int rc = gs::for_each_piece(offsets.data(), n_series, total, piece, [&](const gs::Piece& p) -> int {
        if (p.begin != covered || p.end <= p.begin || p.end - p.begin > piece) return 1;
        if (offsets[p.series] > p.begin || offsets[p.series + 1] <= p.begin) return 2;  // p.series owns p.begin
        covered = p.end;
        Buf<int64_t> bt(ts.data() + p.begin, p.end - p.begin, unaligned);
        Buf<double> bv(values.data() + p.begin, p.end - p.begin, unaligned);
        gs::ScatterArgs b = a;
        b.ts = bt.p, b.values = bv.p, b.base = p.begin, b.end = p.end, b.s_base = p.series;
        scatter(b);
        return 0;
      });
      if (rc != 0 || covered != total) {
        fprintf(stderr, "bad piece walk (rc %d, %llu of %llu samples)\n", rc, (unsigned long long)covered,
                (unsigned long long)total);
        return 4;
      }
    }
  }
  FILE* out = fopen((dir + "/out.bin").c_str(), "wb");
  if (!out) return 2;
  const uint32_t head[2] = {host_bad, 0};
  fwrite(head, 4, 2, out);
  fwrite(stats, 8, 2, out);
  fwrite(plane.data(), 4, plane.size(), out);
  fclose(out);
  return 0;
}
