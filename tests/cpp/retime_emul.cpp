// Host emulation of gpr_resident_retime: k_retime_rows compiled from the SOURCE TEXT of gpu-pruner_b200/csrc/gpr_ring.cuh
// under tests/cpp/cuda_shim.hpp (CTAs of real threads), launched with the grid gpr_api.cu uses (ring_grid) on one plane
// and, optionally, its new index; and gpr::retime_plan (gpu-pruner_b200/csrc/gpr_retime.h) as the session calls it.
//
// tests/test_retime_emul.py writes the cut-out namespace bodies of gpr_kernels.cuh and gpr_ring.cuh
// -> hotpath_extract.inc / ring_extract.inc, and runs either
//     retime_emul rows SM_COUNT CASES DATA OUT
// CASES: one line per call, "N_ROWS T HEAD N_KEEP FACTOR INDEX" (INDEX 1: rebuild the block index).  DATA holds, per
// case, the old plane [N_ROWS][T] as uint32 words.  OUT gets, per case, the new plane [N_ROWS][T'] and, with INDEX, the
// new index [N_ROWS][index_ld(T')].  Every buffer is its own exact-size allocation, so a read past the old plane or a
// store past the new one is an AddressSanitizer error; outputs start as 0xA5A5A5A5, so a word the kernel does not write
// shows.  Or
//     retime_emul plan PLANS
// PLANS: one line per call, "N S T N2 S2"; prints "keep N_KEEP FACTOR" or "refused <reason>" per line.
#include "cuda_shim.hpp"

#include "gpr_retime.h"

#define __host__
namespace gpr {
#include "hotpath_extract.inc"
#include "ring_extract.inc"
}

static int run_plans(const char* path) {
  std::ifstream in(path);
  if (!in) return 2;
  long long N, s, N2, s2;
  unsigned T;
  while (in >> N >> s >> T >> N2 >> s2) {
    const gpr::RetimePlan p = gpr::retime_plan(N, s, T, N2, s2);
    if (p.refusal) printf("refused %s\n", p.refusal);
    else printf("keep %u %u\n", p.n_keep, p.factor);
  }
  return 0;
}

int main(int argc, char** argv) {
  if (argc == 3 && std::string(argv[1]) == "plan") return run_plans(argv[2]);
  if (argc != 6 || std::string(argv[1]) != "rows") {
    fprintf(stderr, "usage: retime_emul rows SM_COUNT CASES DATA OUT | retime_emul plan PLANS\n");
    return 2;
  }
  const int sm_count = atoi(argv[2]);
  std::vector<uint32_t> data;
  {
    std::ifstream f(argv[4], std::ios::binary);
    f.seekg(0, std::ios::end);
    data.resize((size_t)f.tellg() / 4);
    f.seekg(0);
    f.read(reinterpret_cast<char*>(data.data()), (std::streamsize)(data.size() * 4));
  }
  std::ifstream cases(argv[3]);
  FILE* out = fopen(argv[5], "wb");
  if (!cases || !out) return 2;
  g_max_resident_ctas = 8;  // no CTA of this kernel waits for another
  size_t off = 0;
  uint32_t n_rows, T, head, n_keep, factor, index;
  while (cases >> n_rows >> T >> head >> n_keep >> factor >> index) {
    const size_t n_old = (size_t)n_rows * T;
    if (off + n_old > data.size()) {
      fprintf(stderr, "data file too short\n");
      return 2;
    }
    const std::vector<uint32_t> old(data.begin() + (ptrdiff_t)off, data.begin() + (ptrdiff_t)(off + n_old));
    off += n_old;
    const uint32_t T_new = gpr::retime_len(n_keep, factor), ld = index ? gpr::index_ld(T_new) : 0;
    std::vector<uint32_t> plane((size_t)n_rows * T_new, 0xA5A5A5A5u), idx((size_t)n_rows * ld, 0xA5A5A5A5u);
    uint32_t* dst = plane.data();
    float* di = index ? reinterpret_cast<float*>(idx.data()) : nullptr;
    const uint32_t* src = old.data();
    launch(gpr::ring_grid(n_rows, sm_count), gpr::kRingThreads, 0,
           [&] { gpr::k_retime_rows(dst, src, n_rows, T, head, n_keep, factor, di, ld); });
    fwrite(plane.data(), 4, plane.size(), out);
    if (index) fwrite(idx.data(), 4, idx.size(), out);
  }
  fclose(out);
  return 0;
}
