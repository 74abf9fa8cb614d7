// Host emulation of gpr_resident_live_rows: k_live_rows compiled from the SOURCE TEXT of
// gpu-pruner_b200/csrc/gpr_ring.cuh under tests/cpp/cuda_shim.hpp (CTAs of real threads), launched with the grid
// gpr_api.cu uses (live_rows_grid) on the buffers it picks (live_rows_from_index: a current index, else the planes).
//
// tests/test_live_rows_emul.py writes the cut-out namespace bodies of gpr_kernels.cuh and gpr_ring.cuh
// -> hotpath_extract.inc / ring_extract.inc, a case list and a data file of uint32 words, and runs
//     live_rows_emul SM_COUNT CASES DATA OUT
// CASES: one line per call, "N_ROWS T FLAGS" (FLAGS: 1 = power plane, 2 = block index, 4 = the index is stale).  DATA
// holds, per case, the util ring [N_ROWS][T], [the power ring], [the util index [N_ROWS][idx_ld], [the power index]].
// OUT gets, per case, the ceil(N_ROWS / 32) words of the bitmap.  Every buffer is its own exact-size allocation, so a
// read past the last row or a store past the last word is an AddressSanitizer error; the bitmap starts as 0xA5A5A5A5,
// so a word the kernel does not write shows.
#include "cuda_shim.hpp"

#define __host__
namespace gpr {
#include "hotpath_extract.inc"
#include "ring_extract.inc"
}

static std::vector<uint32_t> g_data;
static size_t g_off = 0;

static std::vector<uint32_t> take(size_t n) {   // an exact-size copy of the next n words of DATA
  if (g_off + n > g_data.size()) {
    fprintf(stderr, "data file too short (%zu + %zu > %zu)\n", g_off, n, g_data.size());
    exit(2);
  }
  std::vector<uint32_t> v(g_data.begin() + (ptrdiff_t)g_off, g_data.begin() + (ptrdiff_t)(g_off + n));
  g_off += n;
  return v;
}

int main(int argc, char** argv) {
  if (argc != 5) {
    fprintf(stderr, "usage: live_rows_emul SM_COUNT CASES DATA OUT\n");
    return 2;
  }
  const int sm_count = atoi(argv[1]);
  {
    std::ifstream f(argv[3], std::ios::binary);
    f.seekg(0, std::ios::end);
    g_data.resize((size_t)f.tellg() / 4);
    f.seekg(0);
    f.read(reinterpret_cast<char*>(g_data.data()), (std::streamsize)(g_data.size() * 4));
  }
  std::ifstream cases(argv[2]);
  FILE* out = fopen(argv[4], "wb");
  if (!cases || !out) return 2;
  g_max_resident_ctas = 8;   // no CTA of this kernel waits for another
  uint32_t n_rows, T, flags;
  while (cases >> n_rows >> T >> flags) {
    const uint32_t idx_ld = gpr::index_ld(T);
    const bool power = flags & 1, index = flags & 2, stale = flags & 4;
    std::vector<uint32_t> util = take((size_t)n_rows * T), pow, iu, ip;
    if (power) pow = take((size_t)n_rows * T);
    if (index) {
      iu = take((size_t)n_rows * idx_ld);
      if (power) ip = take((size_t)n_rows * idx_ld);
    }
    const bool from_index = gpr::live_rows_from_index(index, stale);
    const uint32_t* p0 = from_index ? iu.data() : util.data();
    const uint32_t* p1 = !power ? nullptr : from_index ? ip.data() : pow.data();
    const uint32_t len = from_index ? idx_ld : T;
    std::vector<uint32_t> bits((n_rows + 31) / 32, 0xA5A5A5A5u);
    uint32_t* dst = bits.data();
    launch(gpr::live_rows_grid(n_rows, sm_count), gpr::kRingThreads, 0,
           [&] { gpr::k_live_rows(p0, p1, n_rows, len, dst); });
    fwrite(bits.data(), 4, bits.size(), out);
  }
  fclose(out);
  return 0;
}
