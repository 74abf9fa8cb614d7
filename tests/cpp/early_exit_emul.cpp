// Bytes each reduce kernel reads, row by row: k_reduce_ldg and k_reduce_tma compiled from the SOURCE TEXT of
// gpu-pruner_b200/csrc/gpr_kernels.cuh (see hotpath_emul.cpp for the shim), with the loads and bulk copies renamed by
// tests/test_early_exit_emul.py to the counting versions below.  Every load and copy is attributed to the row of the
// plane it reads, so the test can compare the bytes of every row with a model of the early-exit rule.
//
// usage: early_exit_emul DIR...   DIR/params.txt: P G T ld use_power thr_bits want_smax shift sm_count tma_warps
//        tma_chunk tma_depth ldg_ctas variant(ldg|tma); DIR/util.f32 [DIR/power.f32]
// prints  <dir> <kernel> <dbits hex> <cbits hex> <vbits hex> <n_series> <n_cand> <n_dec> <smax hex|->
// and writes DIR/bytes.u64: bytes read per util row, then per power row.
#include "cuda_shim.hpp"
#include "../../gpu-pruner_b200/csrc/gpr_launch.h"

struct Plane {
  const char* lo = nullptr;
  const char* hi = nullptr;
  uint64_t row_bytes = 1;
  std::vector<uint64_t>* bytes = nullptr;
};
static Plane g_planes[2];

static void count(const void* p, uint64_t n) {
  const char* c = static_cast<const char*>(p);
  for (Plane& pl : g_planes) {
    if (pl.bytes && c >= pl.lo && c < pl.hi) {
      const uint64_t r = (uint64_t)(c - pl.lo) / pl.row_bytes;
      if ((uint64_t)(c + n - pl.lo - 1) / pl.row_bytes != r) {
        fprintf(stderr, "a load crosses a row boundary\n");
        abort();
      }
      __atomic_fetch_add(&(*pl.bytes)[r], n, __ATOMIC_RELAXED);
      return;
    }
  }
  fprintf(stderr, "a load outside the window\n");
  abort();
}
template <class T> static inline T cnt_ldg(const T* p) { count(p, sizeof(T)); return __ldg(p); }
static inline float4 cnt_ldg_stream(const float4* p) { count(p, 16); return ldg_stream(p); }
static inline void cnt_tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  count(src, bytes);
  tma_load_1d(dst, src, bytes, bar, pol);
}

#define __host__
namespace gpr {
#include "early_exit_extract.inc"
}

template <class T>
static void slurp(const std::string& path, std::vector<T>* out) {
  std::ifstream f(path, std::ios::binary);
  f.seekg(0, std::ios::end);
  const size_t n = (size_t)f.tellg();
  f.seekg(0);
  out->resize(n / sizeof(T));
  f.read(reinterpret_cast<char*>(out->data()), (std::streamsize)(out->size() * sizeof(T)));
}

static void print_words(const std::vector<uint32_t>& w) {
  for (uint32_t x : w) printf("%08x", x);
  if (w.empty()) printf("-");
}

int main(int argc, char** argv) {
  g_max_resident_ctas = 4;
  for (int a = 1; a < argc; ++a) {
    const std::string dir = argv[a];
    uint32_t P, G, T, thr_bits;
    unsigned long long ld;
    int use_power, want_smax, shift;
    std::string variant;
    gpr::LaunchKnobs k;
    {
      std::ifstream f(dir + "/params.txt");
      f >> P >> G >> T >> ld >> use_power >> thr_bits >> want_smax >> shift >> k.sm_count >> k.tma_warps >>
          k.tma_chunk_bytes >> k.tma_depth_max >> k.ldg_ctas_per_sm >> variant;
    }
    k.fold_threads = 64;
    k.variant = variant == "tma" ? GPR_KERNEL_TMA : GPR_KERNEL_LDG;
    const uint32_t S = P * G, MW = (G + 31) / 32, W = (P + 31) / 32;
    std::vector<float> u, w;
    slurp(dir + "/util.f32", &u);
    if (use_power) slurp(dir + "/power.f32", &w);
    std::vector<float> ubuf(u.size() + 16 + shift), pbuf(w.size() + 16 + shift);
    auto aligned = [&](std::vector<float>& b) {
      float* p = b.data();
      while (reinterpret_cast<uintptr_t>(p) % 16u) ++p;
      return p + shift;
    };
    float* util = aligned(ubuf);
    memcpy(util, u.data(), u.size() * 4);
    float* power = use_power ? aligned(pbuf) : nullptr;
    if (use_power) memcpy(power, w.data(), w.size() * 4);
    std::vector<uint64_t> bytes(2 * (size_t)S, 0);
    std::vector<uint64_t> ub(S, 0), pb(S, 0);
    g_planes[0] = Plane{reinterpret_cast<const char*>(util), reinterpret_cast<const char*>(util + u.size()), ld * 4, &ub};
    g_planes[1] = Plane{};
    if (use_power)
      g_planes[1] = Plane{reinterpret_cast<const char*>(power), reinterpret_cast<const char*>(power + w.size()), ld * 4, &pb};

    std::vector<uint32_t> masks((size_t)2 * P * MW + 16, 0u), dbits(W), cbits(W), vbits(W);
    std::vector<float> smax(S, -12345.f);
    unsigned long long acc[3] = {0, 0, 0}, done = 0, other_done = 0, counts[3] = {0, 0, 0};
    unsigned int ticket = 0, err = 0;
    gpr::ReduceParams rp;
    memset(&rp, 0, sizeof rp);
    rp.seg[0] = gpr::Segment{util, masks.data(), want_smax ? smax.data() : nullptr, S, 0u};
    rp.seg[1] = gpr::Segment{power, masks.data() + (size_t)P * MW, nullptr, use_power ? S : 0u, 1u};
    rp.ld = ld, rp.T = T, rp.G = G, rp.mw = MW;
    rp.total_rows = S + (use_power ? S : 0u);
    memcpy(&rp.thr, &thr_bits, 4);
    rp.done = &done, rp.need = 0;
    auto a16 = [](const void* p) { return reinterpret_cast<uintptr_t>(p) % 16u == 0; };
    const bool tma_ok = T % 4u == 0 && ld % 4u == 0 && a16(util) && (!use_power || a16(power));
    const gpr::ReducePlan plan = gpr::plan_reduce(k, T, rp.total_rows, tma_ok, false);
    if (plan.kernel == gpr::kReduceLdg) {
      launch(plan.grid, plan.block, 0, [&] { gpr::k_reduce_ldg<gpr::kLdgWarps, gpr::kLdgUnroll>(rp); });
    } else if (k.tma_warps == 4) {
      launch(plan.grid, plan.block, plan.smem, [&] { gpr::k_reduce_tma<4>(rp, plan.L); });
    } else if (k.tma_warps == 8) {
      launch(plan.grid, plan.block, plan.smem, [&] { gpr::k_reduce_tma<8>(rp, plan.L); });
    } else if (k.tma_warps == 16) {
      launch(plan.grid, plan.block, plan.smem, [&] { gpr::k_reduce_tma<16>(rp, plan.L); });
    } else {
      launch(plan.grid, plan.block, plan.smem, [&] { gpr::k_reduce_tma<32>(rp, plan.L); });
    }
    gpr::FoldParams fp;
    memset(&fp, 0, sizeof fp);
    fp.idle_mask = masks.data();
    fp.veto_mask = use_power ? masks.data() + (size_t)P * MW : nullptr;
    fp.dbits = dbits.data(), fp.cbits = cbits.data(), fp.vbits = vbits.data();
    fp.counts = counts, fp.acc = acc, fp.ticket = &ticket;
    fp.done = &done, fp.need = 0;
    fp.prev_done = &other_done, fp.prev_need = 0;
    fp.P = P, fp.G = G, fp.mw = MW;
    fp.world = 1, fp.rank = 0;
    fp.err = &err;
    launch(gpr::fold_grid(k, P), 64, 0, [&] { gpr::k_fold<false>(fp); });
    printf("%s %s%s ", dir.c_str(), plan.kernel == gpr::kReduceTma ? "tma" : "ldg", shift ? "+1" : "");
    print_words(dbits), printf(" "), print_words(cbits), printf(" "), print_words(vbits);
    printf(" %llu %llu %llu ", counts[0], counts[1], counts[2]);
    if (want_smax)
      for (float v : smax) printf("%08x", f2u(v));
    else
      printf("-");
    printf(" head=%u chunk=%u depth=%u\n", plan.L.head_elems, plan.L.chunk_elems, plan.L.depth);
    memcpy(bytes.data(), ub.data(), S * 8);
    memcpy(bytes.data() + S, pb.data(), S * 8);
    std::ofstream(dir + "/bytes.u64", std::ios::binary)
        .write(reinterpret_cast<const char*>(bytes.data()), (std::streamsize)(bytes.size() * 8));
    fflush(stdout);
  }
  return 0;
}
