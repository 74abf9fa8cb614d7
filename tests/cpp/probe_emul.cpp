// k_reduce_probe compiled from the SOURCE TEXT of gpu-pruner_b200/csrc/gpr_probe.cuh (and of gpr_kernels.cuh, whose
// helpers it uses) under the host shim, launched with the geometry gpr_launch.h's plan_reduce picks for an AUTO call
// whose rows may stop.  tests/test_probe_emul.py renames the loads and bulk copies to the counting versions below.
//
// The bulk copies of this shim do not complete when they are issued: each one waits on its stage until a poll of that
// stage's barrier (mbar_test_wait) completes it, with probability 1/4 per poll from a seeded generator.  So the copies
// of a warp land in an order unrelated to the order they were issued in, and the kernel has to serve them as they come.
//
// usage: probe_emul DIR...   DIR/params.txt: P G T ld use_power thr_bits shift sm_count tma_warps seed
//        (tma_warps must not change the probe plan);
//        DIR/util.f32 [DIR/power.f32]
// prints  <dir> <kernel> <dbits hex> <cbits hex> <vbits hex> <n_series> <n_cand> <n_dec> - head=H chunk=C depth=D
// and writes DIR/bytes.u64: bytes read per util row, then per power row.
#include <mutex>
#include <random>
#include <unordered_map>

#include "cuda_shim.hpp"
#include "../../gpu-pruner_b200/csrc/gpr_launch.h"

#undef __launch_bounds__
#define __launch_bounds__(...)

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

// ---- bulk copies that land out of order -------------------------------------------------------------------------
struct Pending {
  void* dst = nullptr;
  const void* src = nullptr;
  uint32_t bytes = 0;
  bool live = false;
};
constexpr int kStripes = 64;
static std::mutex g_mu[kStripes];
static std::unordered_map<const uint64_t*, Pending> g_pending[kStripes];
static uint64_t g_seed = 1;
static thread_local std::mt19937_64 tl_rng;
static thread_local bool tl_seeded = false;
static unsigned long long g_copies = 0, g_held = 0;   // copies issued; polls that held a pending copy back

static int stripe(const uint64_t* bar) { return (int)((reinterpret_cast<uintptr_t>(bar) >> 3) % kStripes); }

static inline void cnt_tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t) {
  if (bytes % 16u != 0 || reinterpret_cast<uintptr_t>(src) % 16u != 0 || reinterpret_cast<uintptr_t>(dst) % 16u != 0) {
    fprintf(stderr, "bulk copy with unaligned address or size (%u bytes)\n", bytes);   // what the hardware rejects
    abort();
  }
  count(src, bytes);
  std::lock_guard<std::mutex> g(g_mu[stripe(bar)]);
  Pending& p = g_pending[stripe(bar)][bar];
  if (p.live) {
    fprintf(stderr, "a second copy on a stage whose copy has not landed\n");
    abort();
  }
  p = Pending{dst, src, bytes, true};
  __atomic_fetch_add(&g_copies, 1ull, __ATOMIC_RELAXED);
}

// poll: maybe land the stage's pending copy, then report whether the phase of `parity` has completed
static inline bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  if (!tl_seeded) {
    tl_rng.seed(g_seed * 0x9E3779B97F4A7C15ull + blockIdx.x * 4096ull + threadIdx.x);
    tl_seeded = true;
  }
  {
    std::lock_guard<std::mutex> g(g_mu[stripe(bar)]);
    auto it = g_pending[stripe(bar)].find(bar);
    if (it != g_pending[stripe(bar)].end() && it->second.live) {
      if (tl_rng() % 4u == 0u) {
        memcpy(it->second.dst, it->second.src, it->second.bytes);
        it->second.live = false;
        __atomic_fetch_add(bar, (uint64_t)1, __ATOMIC_RELEASE);
      } else {
        __atomic_fetch_add(&g_held, 1ull, __ATOMIC_RELAXED);
      }
    }
  }
  return (__atomic_load_n(bar, __ATOMIC_ACQUIRE) & 1u) != parity;
}

#define __host__
namespace gpr {
#include "probe_extract.inc"
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
    int use_power, shift;
    gpr::LaunchKnobs k;
    {
      std::ifstream f(dir + "/params.txt");
      f >> P >> G >> T >> ld >> use_power >> thr_bits >> shift >> k.sm_count >> k.tma_warps >> g_seed;
    }
    k.fold_threads = 64;
    k.variant = GPR_KERNEL_AUTO;
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
    unsigned long long acc[3] = {0, 0, 0}, done = 0, other_done = 0, counts[3] = {0, 0, 0};
    unsigned int ticket = 0, err = 0;
    gpr::ReduceParams rp;
    memset(&rp, 0, sizeof rp);
    rp.seg[0] = gpr::Segment{util, masks.data(), nullptr, S, 0u};
    rp.seg[1] = gpr::Segment{power, masks.data() + (size_t)P * MW, nullptr, use_power ? S : 0u, 1u};
    rp.ld = ld, rp.T = T, rp.G = G, rp.mw = MW;
    rp.total_rows = S + (use_power ? S : 0u);
    memcpy(&rp.thr, &thr_bits, 4);
    rp.done = &done, rp.need = 0;
    auto a16 = [](const void* p) { return reinterpret_cast<uintptr_t>(p) % 16u == 0; };
    const bool tma_ok = T % 4u == 0 && ld % 4u == 0 && a16(util) && (!use_power || a16(power));
    const gpr::ReducePlan plan = gpr::plan_reduce(k, T, rp.total_rows, tma_ok, false, true);
    if (plan.kernel != gpr::kReduceProbe) {
      fprintf(stderr, "%s: AUTO with rows that may stop did not plan the probe kernel\n", dir.c_str());
      return 2;
    }
    g_copies = g_held = 0;
    if (plan.block != 32u * gpr::kProbeWarps) {
      fprintf(stderr, "%s: the probe plan's block is not kProbeWarps warps\n", dir.c_str());
      return 2;
    }
    launch(plan.grid, plan.block, plan.smem, [&] { gpr::k_reduce_probe<gpr::kProbeWarps>(rp, plan.L); });
    for (auto& m : g_pending)
      for (auto& kv : m)
        if (kv.second.live) {
          fprintf(stderr, "%s: a copy was issued and never consumed\n", dir.c_str());
          return 2;
        }
    for (auto& m : g_pending) m.clear();
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
    printf("%s probe ", dir.c_str());
    print_words(dbits), printf(" "), print_words(cbits), printf(" "), print_words(vbits);
    printf(" %llu %llu %llu - head=%u chunk=%u depth=%u grid=%u copies=%llu held=%llu\n", counts[0], counts[1],
           counts[2], plan.L.head_elems, plan.L.chunk_elems, plan.L.depth, plan.grid, g_copies, g_held);
    memcpy(bytes.data(), ub.data(), S * 8);
    memcpy(bytes.data() + S, pb.data(), S * 8);
    std::ofstream(dir + "/bytes.u64", std::ios::binary)
        .write(reinterpret_cast<const char*>(bytes.data()), (std::streamsize)(bytes.size() * 8));
    fflush(stdout);
  }
  return 0;
}
