// Host emulation of gpr_resident_remap: k_remap_check, k_remap_rows and remap_first_bad compiled from the SOURCE TEXT
// of gpu-pruner_b200/csrc/gpr_ring.cuh under tests/cpp/cuda_shim.hpp (CTAs of real threads), launched with the grids
// and in the order gpr_api.cu uses: the map is checked (both check passes over it as a device map, and the host walk
// as for a host map, which must agree: exit 3 otherwise), and only a good map builds the new ring.
//
// tests/test_remap_emul.py writes the cut-out namespace bodies of gpr_kernels.cuh and gpr_ring.cuh
// -> hotpath_extract.inc / ring_extract.inc, a case list and a data file of uint32 words, and runs
//     remap_emul SM_COUNT CASES DATA OUT
// CASES: one line per remap, "N_OLD T FLAGS N_NEW" (FLAGS: 1 = power plane, 2 = block index).  DATA holds, per case,
// the old util ring [N_OLD][T], [the old power ring], [the util index [N_OLD][idx_ld], [the power index]], then the
// map [N_NEW].  OUT gets, per case: the first bad new row (N_NEW if none), then for a good map the new buffers in the
// same order.  Every buffer, the map included, is its own exact-size allocation, so a read or write past the last
// row is an AddressSanitizer error.
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
    fprintf(stderr, "usage: remap_emul SM_COUNT CASES DATA OUT\n");
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
  g_max_resident_ctas = 8;   // no CTA of these kernels waits for another
  uint32_t n_old, T, flags, n_new;
  while (cases >> n_old >> T >> flags >> n_new) {
    const uint32_t idx_ld = gpr::index_ld(T);
    std::vector<std::vector<uint32_t>> old;   // the present buffers, in ABI order
    std::vector<uint32_t> len;
    for (int k = 0; k < 4; ++k) {
      const bool power = k % 2 == 1, index = k >= 2;
      if ((power && !(flags & 1)) || (index && !(flags & 2))) continue;
      len.push_back(index ? idx_ld : T);
      old.push_back(take((size_t)n_old * len.back()));
    }
    const std::vector<uint32_t> map = take(n_new);
    // the check: host walk and device passes
    const uint32_t host_first = (uint32_t)gpr::remap_first_bad(map.data(), n_new, n_old);
    const size_t words = ((size_t)n_old + 31) / 32;
    std::vector<unsigned int> seen(words, 0), dup(words, 0);
    unsigned int first = n_new;
    const uint32_t blocks = std::max(1u, std::min((n_new + 255u) / 256u, (uint32_t)sm_count * 8u));
    for (int pass = 0; pass < 2; ++pass)
      launch(blocks, 256, 0, [&] {
        gpr::k_remap_check(map.data(), n_new, n_old, seen.data(), dup.data(), &first, pass);
      });
    if (first != host_first) {
      fprintf(stderr, "the check kernel names new row %u, the host walk %u\n", first, host_first);
      return 3;
    }
    fwrite(&first, 4, 1, out);
    if (first < n_new) continue;   // nothing is allocated or written
    const uint32_t grid = gpr::ring_grid(n_new, sm_count);
    for (size_t k = 0; k < old.size(); ++k) {
      std::vector<uint32_t> next((size_t)n_new * len[k]);
      uint32_t* dst = next.data();
      const uint32_t* src = old[k].data();
      const uint32_t L = len[k];
      launch(grid, gpr::kRingThreads, 0, [&] { gpr::k_remap_rows(dst, src, map.data(), n_new, L); });
      fwrite(next.data(), 4, next.size(), out);
    }
  }
  fclose(out);
  return 0;
}
