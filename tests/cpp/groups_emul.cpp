// A whole decision with a `sum by` group table, on the CPU: k_group_rows and k_group_sum (the SOURCE TEXT of
// gpu-pruner_b200/csrc/gpr_groups.cuh) around k_reduce_ldg / k_reduce_tma / k_reduce_u8 and k_fold (gpr_kernels.cuh,
// cut out as in hotpath_emul.cpp), launched in decide_impl's order with the geometry of gpr_launch.h.  Loads and bulk
// copies of the window are renamed by tests/test_groups_emul.py to the counting versions below, as in
// early_exit_emul.cpp, so the test sees the bytes of every row.
//
// usage: groups_emul DIR...   DIR/params.txt: P G T ld use_power thr_bits want_smax shift sm_count tma_warps tma_chunk
//        tma_depth ldg_ctas variant(ldg|tma|u8) has_table; DIR/util.f32 (u8: util.u8) [DIR/power.f32] [DIR/groups.u32]
// prints  <dir> <kernel> <dbits hex> <cbits hex> <vbits hex> <n_series> <n_cand> <n_dec> <idle_slots hex> <bad> <smax|->
// and writes DIR/bytes.u64: bytes read per util row, then per power row.
#include <cmath>
#include <limits>
using std::fabs;
using std::isinf;
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
static inline uint4 cnt_ldg_stream_u4(const uint4* p) { count(p, 16); return ldg_stream_u4(p); }
static inline void cnt_tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  count(src, bytes);
  tma_load_1d(dst, src, bytes, bar, pol);
}

// test_groups_emul.py appends a call of this to k_group_sum's `idle = ...` line: the float64 value of every group it
// sums ([P][G] at the leader's slot, NaN for a group without a present member)
static std::vector<double> g_values;
static uint32_t g_values_G = 0;
static void record_group_value(uint32_t p, uint32_t g, bool any, double v) {
  g_values[(size_t)p * g_values_G + g] = any ? v : std::numeric_limits<double>::quiet_NaN();
}

#define __host__
namespace gpr {
#include "groups_kernels_extract.inc"
#include "groups_extract.inc"
}

template <class T>
static bool slurp(const std::string& path, std::vector<T>* out) {
  std::ifstream f(path, std::ios::binary);
  if (!f) return false;
  f.seekg(0, std::ios::end);
  const size_t n = (size_t)f.tellg();
  f.seekg(0);
  out->resize(n / sizeof(T));
  f.read(reinterpret_cast<char*>(out->data()), (std::streamsize)(out->size() * sizeof(T)));
  return true;
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
    int use_power, want_smax, shift, has_table;
    std::string variant;
    gpr::LaunchKnobs k;
    {
      std::ifstream f(dir + "/params.txt");
      f >> P >> G >> T >> ld >> use_power >> thr_bits >> want_smax >> shift >> k.sm_count >> k.tma_warps >>
          k.tma_chunk_bytes >> k.tma_depth_max >> k.ldg_ctas_per_sm >> variant >> has_table;
    }
    k.fold_threads = 64;
    k.variant = variant == "tma" ? GPR_KERNEL_TMA : GPR_KERNEL_LDG;
    const bool u8 = variant == "u8";
    const uint32_t S = P * G, MW = (G + 31) / 32, W = (P + 31) / 32;
    const size_t esize = u8 ? 1 : 4;
    std::vector<unsigned char> u;
    std::vector<float> w;
    std::vector<uint32_t> table;
    slurp(dir + (u8 ? "/util.u8" : "/util.f32"), &u);
    if (use_power) slurp(dir + "/power.f32", &w);
    if (has_table) slurp(dir + "/groups.u32", &table);
    std::vector<unsigned char> ubuf(u.size() + 64 + shift * esize);
    std::vector<float> pbuf(w.size() + 16 + shift);
    unsigned char* ub0 = ubuf.data();
    while (reinterpret_cast<uintptr_t>(ub0) % 16u) ++ub0;
    unsigned char* util = ub0 + shift * esize;
    memcpy(util, u.data(), u.size());
    float* power = nullptr;
    if (use_power) {
      power = pbuf.data();
      while (reinterpret_cast<uintptr_t>(power) % 16u) ++power;
      power += shift;
      memcpy(power, w.data(), w.size() * 4);
    }
    std::vector<uint64_t> ubytes(S, 0), pbytes(S, 0);
    g_planes[0] = Plane{reinterpret_cast<const char*>(util), reinterpret_cast<const char*>(util + u.size()), ld * esize,
                        &ubytes};
    g_planes[1] = Plane{};
    if (use_power)
      g_planes[1] = Plane{reinterpret_cast<const char*>(power), reinterpret_cast<const char*>(power + w.size()), ld * 4,
                          &pbytes};

    std::vector<uint32_t> masks((size_t)2 * P * MW + 16, 0u), dbits(W), cbits(W), vbits(W), islots((size_t)P * MW, 0xdeadu);
    std::vector<float> smax(S, -12345.f), gmax(S, -777.f);
    std::vector<uint32_t> grouped((size_t)P * MW + 4, 0xffffffffu), gpods(P + 4, 0xffffffffu);
    unsigned long long acc[3] = {0, 0, 0}, done = 0, other_done = 0, counts[3] = {0, 0, 0};
    unsigned int ticket = 0, err = 0, bad = 0;

    gpr::GroupParams gq;
    memset(&gq, 0, sizeof gq);
    gq.table = table.data();
    gq.need = grouped.data();
    gq.n_pods = gpods.data();
    gq.pods = gpods.data() + 1;
    gq.gmax = want_smax ? smax.data() : gmax.data();
    gq.idle_mask = masks.data();
    gq.bad = &bad;
    gq.P = P, gq.G = G, gq.mw = MW;
    const uint32_t group_grid = gpr::group_grid(k, P);
    const uint64_t sentinel = 0x7FF8DEADBEEF0000ull;
    double sentinel_d;
    memcpy(&sentinel_d, &sentinel, 8);
    g_values.assign(S, sentinel_d);
    g_values_G = G;
    if (has_table) {
      gpods[0] = 0;
      launch(group_grid, gpr::kGroupBlock, 0, [&] { gpr::k_group_rows(gq); });
    }

    gpr::ReduceParams rp;
    memset(&rp, 0, sizeof rp);
    rp.seg[0] = gpr::Segment{reinterpret_cast<const float*>(util), masks.data(), want_smax ? smax.data() : nullptr, S, 0u};
    rp.seg[1] = gpr::Segment{power, masks.data() + (size_t)P * MW, nullptr, use_power ? S : 0u, 1u};
    rp.ld = ld, rp.T = T, rp.G = G, rp.mw = MW;
    rp.total_rows = S + (use_power ? S : 0u);
    memcpy(&rp.thr, &thr_bits, 4);
    rp.done = &done, rp.need = 0;
    rp.util_u8 = u8 ? 1u : 0u;
    if (has_table) rp.grouped = grouped.data(), rp.gmax = gmax.data();
    auto a16 = [](const void* p) { return reinterpret_cast<uintptr_t>(p) % 16u == 0; };
    const bool tma_ok = T % 4u == 0 && ld % 4u == 0 && a16(util) && (!use_power || a16(power));
    const gpr::ReducePlan plan = gpr::plan_reduce(k, T, rp.total_rows, tma_ok, u8);
    // the instantiation gpr_api.cu's launch_reduce picks: with a table, the one that tests every row
    if (plan.kernel == gpr::kReduceU8) {
      launch(plan.grid, plan.block, 0, [&] {
        has_table ? gpr::k_reduce_u8<gpr::kLdgWarps, gpr::kU8Unroll, true>(rp)
                  : gpr::k_reduce_u8<gpr::kLdgWarps, gpr::kU8Unroll, false>(rp);
      });
    } else if (plan.kernel == gpr::kReduceLdg) {
      launch(plan.grid, plan.block, 0, [&] {
        has_table ? gpr::k_reduce_ldg<gpr::kLdgWarps, gpr::kLdgUnroll, true>(rp)
                  : gpr::k_reduce_ldg<gpr::kLdgWarps, gpr::kLdgUnroll, false>(rp);
      });
    } else if (k.tma_warps == 4) {
      launch(plan.grid, plan.block, plan.smem, [&] { has_table ? gpr::k_reduce_tma<4, true>(rp, plan.L) : gpr::k_reduce_tma<4, false>(rp, plan.L); });
    } else if (k.tma_warps == 8) {
      launch(plan.grid, plan.block, plan.smem, [&] { has_table ? gpr::k_reduce_tma<8, true>(rp, plan.L) : gpr::k_reduce_tma<8, false>(rp, plan.L); });
    } else {
      launch(plan.grid, plan.block, plan.smem, [&] { has_table ? gpr::k_reduce_tma<16, true>(rp, plan.L) : gpr::k_reduce_tma<16, false>(rp, plan.L); });
    }
    if (has_table) launch(group_grid, gpr::kGroupBlock, 0, [&] { gpr::k_group_sum(gq); });

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
    fp.islots = islots.data();
    launch(gpr::fold_grid(k, P), 64, 0, [&] { gpr::k_fold<false, true>(fp); });
    for (size_t i = 0; i < (size_t)2 * P * MW; ++i)
      if (masks[i]) {
        fprintf(stderr, "flag word %zu left set after the fold\n", i);
        return 3;
      }
    const char* kname = plan.kernel == gpr::kReduceU8 ? "u8" : plan.kernel == gpr::kReduceTma ? "tma" : "ldg";
    printf("%s %s ", dir.c_str(), kname);
    print_words(dbits), printf(" "), print_words(cbits), printf(" "), print_words(vbits);
    printf(" %llu %llu %llu ", counts[0], counts[1], counts[2]);
    print_words(islots);
    printf(" %u ", bad);
    if (want_smax)
      for (float v : smax) printf("%08x", f2u(v));
    else
      printf("-");
    printf("\n");
    std::vector<uint64_t> bytes(ubytes);
    bytes.insert(bytes.end(), pbytes.begin(), pbytes.end());
    std::ofstream(dir + "/values.f64", std::ios::binary)
        .write(reinterpret_cast<const char*>(g_values.data()), (std::streamsize)(g_values.size() * 8));
    std::ofstream(dir + "/bytes.u64", std::ios::binary)
        .write(reinterpret_cast<const char*>(bytes.data()), (std::streamsize)(bytes.size() * 8));
    fflush(stdout);
  }
  return 0;
}
