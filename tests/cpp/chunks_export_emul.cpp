// Host emulation of gpr_resident_export: k_export_size, k_export_scan and k_export_write compiled from the SOURCE TEXT
// of gpu-pruner_b200/csrc/gpr_chunks_encode.cuh under tests/cpp/cuda_shim.hpp (the scan's dynamic shared memory is the
// emulated CTA's), launched the way gpr_api.cu launches them, with its capacity rule in between.
//
// tests/test_chunks_export_emul.py writes DIR/params.txt and DIR/plane.u32 and runs
//     chunks_export_emul SM_COUNT DIR
// DIR/params.txt: rows T head per_chunk t_end_ms step_ms cap_series cap_chunks cap_bytes
// DIR/plane.u32:  the ring plane [rows][T] as f32 bits
// DIR/out.bin:    u64 status (0 = written, 1 = a capacity too small: nothing written), u64 n_series, n_chunks,
//                 n_bytes, n_samples, then (status 0) series_chunks (n_series + 1), chunk_bytes (n_chunks + 1), rows
//                 (n_series, u32) and data (n_bytes).
// The outputs are vectors of exactly their size, so a store past one is an AddressSanitizer error.  The ring must be
// unchanged (exit 3 otherwise).
#include "cuda_shim.hpp"

#include "../../gpu-pruner_b200/csrc/gpr_text.cuh"
namespace gpr {
namespace chunks {
#include "chunks_export_extract.inc"
}
}  // namespace gpr

namespace gc = gpr::chunks;

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

int main(int argc, char** argv) {
  if (argc != 3) {
    fprintf(stderr, "usage: chunks_export_emul SM_COUNT DIR\n");
    return 2;
  }
  const unsigned sm = (unsigned)atoi(argv[1]);
  g_max_resident_ctas = 4;  // CTAs of the size and write passes never wait for one another
  const std::string dir = argv[2];
  std::ifstream pf(dir + "/params.txt");
  uint32_t rows, T, head, per_chunk;
  long long t_end_ms, step_ms;
  unsigned long long cap_series, cap_chunks, cap_bytes;
  if (!(pf >> rows >> T >> head >> per_chunk >> t_end_ms >> step_ms >> cap_series >> cap_chunks >> cap_bytes)) return 2;
  const std::vector<uint32_t> plane = read_all<uint32_t>(dir + "/plane.u32");
  if (plane.size() != (size_t)rows * T) return 2;
  const std::vector<uint32_t> before(plane);

  gc::ExportArgs a;
  memset(&a, 0, sizeof a);
  a.plane = plane.data(), a.rows = rows, a.T = T, a.head = head, a.per_chunk = per_chunk;
  a.t_end_ms = t_end_ms, a.step_ms = step_ms;
  a.max_chunks = (T + per_chunk - 1) / per_chunk;
  std::vector<uint32_t> sizes((size_t)rows * a.max_chunks), series((size_t)rows + 1);
  std::vector<uint64_t> row_chunks((size_t)rows + 1), row_bytes((size_t)rows + 1);
  unsigned long long totals[4] = {0, 0, 0, 0};
  a.sizes = sizes.data(), a.row_chunks = row_chunks.data(), a.row_bytes = row_bytes.data();
  a.row_series = series.data(), a.totals = totals;
  const unsigned blocks =
      (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(((uint64_t)rows + gc::kEncWarps - 1) / gc::kEncWarps, sm * 16));
  launch(blocks, gc::kEncThreads, 0, [&] { gc::k_export_size(a); });
  launch(1, gc::kScanThreads, gc::kScanSmem, [&] { gc::k_export_scan(a); });

  const unsigned long long n_chunks = totals[0], n_bytes = totals[1], n_series = totals[2], n_samples = totals[3];
  const bool fits = n_series <= cap_series && n_chunks <= cap_chunks && n_bytes <= cap_bytes;
  std::vector<uint64_t> o_series, o_cbytes;
  std::vector<uint32_t> o_rows;
  std::vector<uint8_t> o_data;
  if (fits) {
    o_series.assign(n_series + 1, ~0ull), o_cbytes.assign(n_chunks + 1, ~0ull);
    o_rows.assign(n_series, ~0u), o_data.assign(n_bytes, 0xA5);
    a.series_chunks = o_series.data(), a.chunk_bytes = o_cbytes.data(), a.out_rows = o_rows.data();
    a.data = o_data.data();
    launch(blocks, gc::kEncThreads, 0, [&] { gc::k_export_write(a); });
  }
  if (plane != before) {
    fprintf(stderr, "the export wrote the ring\n");
    return 3;
  }
  FILE* out = fopen((dir + "/out.bin").c_str(), "wb");
  if (!out) return 2;
  const unsigned long long head_words[5] = {fits ? 0ull : 1ull, n_series, n_chunks, n_bytes, n_samples};
  fwrite(head_words, 8, 5, out);
  if (fits) {
    fwrite(o_series.data(), 8, o_series.size(), out);
    fwrite(o_cbytes.data(), 8, o_cbytes.size(), out);
    if (!o_rows.empty()) fwrite(o_rows.data(), 4, o_rows.size(), out);
    if (!o_data.empty()) fwrite(o_data.data(), 1, o_data.size(), out);
  }
  fclose(out);
  return 0;
}
