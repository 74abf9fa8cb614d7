// Host emulation of the resident ring of daemon mode: k_append, k_open, k_reindex and block_max_warp, compiled from
// the SOURCE TEXT of gpu-pruner_b200/csrc/gpr_ring.cuh under tests/cpp/cuda_shim.hpp (CTAs of real threads, warps
// with emulated shuffles), launched with the grid, spans and per-plane choices gpr_api.cu takes from the same header.
//
// tests/test_ring_emul.py writes the cut-out namespace bodies of gpr_kernels.cuh (nan_f, warp_max) and gpr_ring.cuh
// -> hotpath_extract.inc / ring_extract.inc, a script and a data file of uint32 cell bits, and runs
//     ring_emul SM_COUNT SCRIPT DATA OUT
// Script lines (one operation each, like the C ABI calls of the same names):
//     init P G T FLAGS                 FLAGS: 1 = power plane, 2 = block index
//     append N_NEW LD OFF power|nopower  device columns at DATA[OFF], util rows then (power) power rows, row stride LD
//     advance N
//     write PLANE OFF                  direct write of a whole plane (as through gpr_resident_planes) from DATA[OFF]
//     reindex
// After every operation OUT gets: head (u32), the util ring, [the power ring], [the util index, [the power index]]
// as uint32 bits.  Every buffer is its own exact-size allocation, so a read or write past a row of the last row is
// an AddressSanitizer error.
#include "cuda_shim.hpp"

#define __host__
namespace gpr {
#include "hotpath_extract.inc"
#include "ring_extract.inc"
}

struct Ring {
  uint32_t P = 0, G = 0, T = 0, flags = 0, head = 0, idx_ld = 0;
  size_t rows = 0;
  std::vector<float> plane[2], idx[2];
  bool has(int pl) const { return !plane[pl].empty(); }
  float* idx_of(int pl) { return idx[pl].empty() ? nullptr : idx[pl].data(); }
};

static std::vector<uint32_t> g_data;

static std::vector<float> take(size_t off, size_t n) {   // an exact-size copy of DATA[off, off + n)
  if (off + n > g_data.size()) {
    fprintf(stderr, "data file too short (%zu + %zu > %zu)\n", off, n, g_data.size());
    exit(2);
  }
  std::vector<float> v(n);
  memcpy(v.data(), g_data.data() + off, n * 4);
  return v;
}

static void dump(FILE* out, Ring& r) {
  fwrite(&r.head, 4, 1, out);
  for (int pl = 0; pl < 2; ++pl)
    if (r.has(pl)) fwrite(r.plane[pl].data(), 4, r.plane[pl].size(), out);
  for (int pl = 0; pl < 2; ++pl)
    if (!r.idx[pl].empty()) fwrite(r.idx[pl].data(), 4, r.idx[pl].size(), out);
}

int main(int argc, char** argv) {
  if (argc != 5) {
    fprintf(stderr, "usage: ring_emul SM_COUNT SCRIPT DATA OUT\n");
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
  std::ifstream script(argv[2]);
  FILE* out = fopen(argv[4], "wb");
  if (!script || !out) return 2;
  g_max_resident_ctas = 8;   // none of these kernels waits for another CTA of its grid
  Ring r;
  std::string op;
  while (script >> op) {
    if (op == "init") {
      r = Ring();
      script >> r.P >> r.G >> r.T >> r.flags;
      r.rows = (size_t)r.P * r.G;
      r.plane[0].assign(r.rows * r.T, u2f(gpr::kNoSampleBits));
      if (r.flags & 1) r.plane[1].assign(r.rows * r.T, u2f(gpr::kNoSampleBits));
      if (r.flags & 2) {
        r.idx_ld = gpr::index_ld(r.T);
        for (int pl = 0; pl < 2; ++pl)
          if (r.has(pl)) r.idx[pl].assign(r.rows * r.idx_ld, u2f(gpr::kNoSampleBits));
      }
    } else if (op == "append") {
      uint32_t n_new;
      unsigned long long ld, off;
      std::string pw;
      script >> n_new >> ld >> off >> pw;
      const gpr::RingSpan sp = gpr::ring_span(r.head, n_new, r.T);
      const uint32_t grid = gpr::ring_grid(r.rows, sm_count);
      for (int pl = 0; pl < 2; ++pl) {
        const bool cols = pl == 0 || pw == "power";
        const gpr::RingLaunch what = gpr::append_launch(r.has(pl), cols);
        if (what == gpr::kRingNone) continue;
        float* dst = r.plane[pl].data();
        float* idx = r.idx_of(pl);
        if (what == gpr::kRingOpen) {
          launch(grid, gpr::kRingThreads, 0, [&] { gpr::k_open(dst, (uint32_t)r.rows, r.T, sp.start, sp.n, idx, r.idx_ld); });
          continue;
        }
        const std::vector<float> src = take(off + (size_t)pl * r.rows * ld, r.rows * ld);
        const float* in = src.data() + sp.src_col;
        launch(grid, gpr::kRingThreads, 0,
               [&] { gpr::k_append(dst, in, (uint32_t)r.rows, r.T, sp.start, sp.n, ld, idx, r.idx_ld); });
      }
      r.head = sp.next_head;
    } else if (op == "advance") {
      uint32_t n;
      script >> n;
      const gpr::RingSpan sp = gpr::ring_span(r.head, n, r.T);
      for (int pl = 0; pl < 2; ++pl) {
        const gpr::RingLaunch what = gpr::advance_launch(r.has(pl), r.idx_of(pl) != nullptr);
        if (what == gpr::kRingNone) continue;
        float* dst = r.plane[pl].data();
        float* idx = r.idx_of(pl);
        if (what == gpr::kRingOpen) {
          launch(gpr::ring_grid(r.rows, sm_count), gpr::kRingThreads, 0,
                 [&] { gpr::k_open(dst, (uint32_t)r.rows, r.T, sp.start, sp.n, idx, r.idx_ld); });
        } else {   // no index: k_fill_columns or a memset (text_emul.cpp runs k_fill_columns' source)
          for (size_t row = 0; row < r.rows; ++row)
            for (uint32_t j = 0; j < std::min(n, r.T); ++j)
              r.plane[pl][row * r.T + ((uint64_t)r.head + j) % r.T] = u2f(gpr::kNoSampleBits);
        }
      }
      r.head = sp.next_head;
    } else if (op == "write") {
      int pl;
      unsigned long long off;
      script >> pl >> off;
      r.plane[pl] = take(off, r.rows * r.T);
    } else if (op == "reindex") {
      for (int pl = 0; pl < 2; ++pl)
        if (!r.idx[pl].empty()) {
          float* src = r.plane[pl].data();
          float* idx = r.idx[pl].data();
          launch(gpr::ring_grid(r.rows, sm_count), gpr::kRingThreads, 0,
                 [&] { gpr::k_reindex(src, (uint32_t)r.rows, r.T, idx, r.idx_ld); });
        }
    } else {
      fprintf(stderr, "unknown operation %s\n", op.c_str());
      return 2;
    }
    dump(out, r);
  }
  fclose(out);
  return 0;
}
