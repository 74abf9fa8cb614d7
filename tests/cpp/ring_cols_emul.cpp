// Host emulation of gpr_resident_cols: k_ring_cols compiled from the SOURCE TEXT of gpu-pruner_b200/csrc/gpr_ring.cuh
// under tests/cpp/cuda_shim.hpp (CTAs of real threads), launched with the grid and the start position gpr_api.cu uses
// (ring_grid, ring_cols_start).
//
// tests/test_ring_cols_emul.py writes the cut-out namespace bodies of gpr_kernels.cuh and gpr_ring.cuh
// -> hotpath_extract.inc / ring_extract.inc, a case list and a data file of uint32 words, and runs
//     ring_cols_emul SM_COUNT CASES DATA OUT
// CASES: one line per call, "N_ROWS T HEAD NEWER N_COLS".  DATA holds, per case, the plane [N_ROWS][T].  OUT gets, per
// case, the band [N_ROWS][N_COLS].  Every buffer is its own exact-size allocation, so a read past the plane or a store
// past the band is an AddressSanitizer error; the band starts as 0xA5A5A5A5, so a cell the kernel does not write shows.
#include "cuda_shim.hpp"

#define __host__
namespace gpr {
#include "hotpath_extract.inc"
#include "ring_extract.inc"
}

int main(int argc, char** argv) {
  if (argc != 5) {
    fprintf(stderr, "usage: ring_cols_emul SM_COUNT CASES DATA OUT\n");
    return 2;
  }
  const int sm_count = atoi(argv[1]);
  std::vector<uint32_t> data;
  {
    std::ifstream f(argv[3], std::ios::binary);
    f.seekg(0, std::ios::end);
    data.resize((size_t)f.tellg() / 4);
    f.seekg(0);
    f.read(reinterpret_cast<char*>(data.data()), (std::streamsize)(data.size() * 4));
  }
  std::ifstream cases(argv[2]);
  FILE* out = fopen(argv[4], "wb");
  if (!cases || !out) return 2;
  g_max_resident_ctas = 8;  // no CTA of this kernel waits for another
  size_t off = 0;
  uint32_t n_rows, T, head, newer, n_cols;
  while (cases >> n_rows >> T >> head >> newer >> n_cols) {
    const size_t n = (size_t)n_rows * T;
    if (off + n > data.size()) {
      fprintf(stderr, "data file too short\n");
      return 2;
    }
    std::vector<uint32_t> plane(data.begin() + (ptrdiff_t)off, data.begin() + (ptrdiff_t)(off + n));
    off += n;
    std::vector<uint32_t> band((size_t)n_rows * n_cols, 0xA5A5A5A5u);
    uint32_t* dst = band.data();
    const uint32_t* src = plane.data();
    const uint32_t start = gpr::ring_cols_start(head, T, newer, n_cols);
    launch(gpr::ring_grid(n_rows, sm_count), gpr::kRingThreads, 0,
           [&] { gpr::k_ring_cols(dst, src, n_rows, T, start, n_cols); });
    fwrite(band.data(), 4, band.size(), out);
  }
  fclose(out);
  return 0;
}
