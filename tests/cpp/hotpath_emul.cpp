// Host emulation of the whole decision path: the three reduce kernels (k_reduce_ldg, k_reduce_tma, k_reduce_u8) and
// the fold kernel, compiled from the SOURCE TEXT of gpu-pruner_b200/csrc/gpr_kernels.cuh.
//
// tests/test_hotpath_emul.py cuts the body of `namespace gpr` out of the kernel header, removes the small helper
// functions that are nothing but inline PTX (loads with cache hints, mbarrier / bulk-copy instructions, scoped
// atomics, %globaltimer) and rewrites the three inline-PTX statements and the __shared__ declarations inside the
// kernels to shim calls -> hotpath_extract.inc.  This file supplies those helpers and the CUDA built-ins on top of
// std::thread: a CTA is a group of threads with a barrier, a warp 32 of them with emulated shuffles / ballots /
// reductions, a bulk copy is a memcpy that completes an emulated mbarrier phase.
//
// For every case directory given on the command line (files written by the test: util.f32, [power.f32], [elig.u8],
// [created.i64], [util.u8], params.txt, [knobs.txt]) it runs each requested reduce variant + the fold, twice on the
// same scratch set, with exactly the launch geometry gpr_api.cu would pick (gpr_launch.h) for the emulated SM count
// and knobs, and prints one line per variant:   <dir> <variant> <clean> <dbits hex> <cbits hex> <vbits hex> <n_series>
// <n_cand> <n_dec> <smax hex...> plan=<what ran>.  The tests compare them with the known answers and the oracle.
// It validates the SOURCE logic of the kernels (row tails, NaN rules, ANY-GPU fold, veto, gates, counters, scratch
// reuse) — not the generated machine code; tests/test_gpu_parity.py does that on an H100.
#include "cuda_shim.hpp"
#include "../../gpu-pruner_b200/csrc/gpr_launch.h"   // the launch geometry gpr_api.cu uses (not extracted: host code)

#define __host__
namespace gpr {
#include "hotpath_extract.inc"
#include "synth_extract.inc"   // gpr_synth.cuh: the device generator of the synthetic windows (no PTX in it)
}

// ---- driver --------------------------------------------------------------------------------------------------------
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

struct Case {
  uint32_t P = 0, G = 0, T = 0;
  uint64_t ld = 0;
  int use_power = 0;
  uint32_t thr_bits = 0;
  int64_t cutoff = 0;
  std::vector<float> util, power;
  std::vector<uint8_t> elig, util_u8;
  std::vector<int64_t> created;
  // emulated device and tuning knobs (knobs.txt: sm_count tma_warps tma_chunk_bytes tma_depth ldg_ctas fold_threads
  // labels), and the runs to make: ldg / ldg+1 request the LDG kernel, tma / tma+1 the TMA kernel (+1: rows start
  // 4 bytes off 16-byte alignment), u8 the byte kernel.  Without knobs.txt: a 3-SM device with small tilings.
  gpr::LaunchKnobs knobs;
  std::vector<std::string> labels;
};

static void default_knobs(gpr::LaunchKnobs* k) {
  k->sm_count = 3, k->tma_warps = 4, k->tma_chunk_bytes = 512, k->tma_depth_max = 2, k->ldg_ctas_per_sm = 1;
  k->fold_threads = 64;
}

static const char* kernel_name(int k) { return k == gpr::kReduceTma ? "tma" : k == gpr::kReduceU8 ? "u8" : "ldg"; }

static void print_words(const std::vector<uint32_t>& w) {
  for (uint32_t x : w) printf("%08x", x);
  if (w.empty()) printf("-");
}

static void run_variant(const std::string& dir, const char* name, const Case& c, int variant, size_t shift_floats) {
  const uint32_t P = c.P, G = c.G, T = c.T, S = P * G, MW = (G + 31) / 32, W = (P + 31) / 32;
  // the planes, 16-byte aligned plus an optional shift (the vectorised kernels peel to alignment themselves)
  std::vector<float> ubuf((size_t)S * c.ld + 16 + shift_floats), pbuf(c.use_power ? (size_t)S * c.ld + 16 + shift_floats : 0);
  auto aligned = [&](std::vector<float>& b) {
    float* p = b.data();
    while (reinterpret_cast<uintptr_t>(p) % 16u) ++p;
    return p + shift_floats;
  };
  float* util = aligned(ubuf);
  memcpy(util, c.util.data(), c.util.size() * 4);
  float* power = nullptr;
  if (c.use_power) power = aligned(pbuf), memcpy(power, c.power.data(), c.power.size() * 4);
  std::vector<uint32_t> masks((size_t)2 * P * MW + 16, 0u);
  unsigned long long acc[3] = {0, 0, 0}, done = 0, other_done = 0;
  unsigned int ticket = 0, err = 0;
  gpr::ReducePlan plan;
  for (int rep = 0; rep < 2; ++rep) {   // the second decision reuses the scratch set the first one must have zeroed
    std::vector<uint32_t> dbits(W, 0xdeadbeefu), cbits(W, 0xdeadbeefu), vbits(W, 0xdeadbeefu);
    std::vector<float> smax(S, -12345.f);
    unsigned long long counts[3] = {~0ull, ~0ull, ~0ull};
    gpr::ReduceParams rp;
    memset(&rp, 0, sizeof rp);
    rp.seg[0] = gpr::Segment{variant == 2 ? reinterpret_cast<const float*>(c.util_u8.data()) : util, masks.data(),
                             smax.data(), S, 0u};
    rp.seg[1] = gpr::Segment{power, masks.data() + (size_t)P * MW, nullptr, c.use_power ? S : 0u, 1u};
    rp.ld = c.ld, rp.T = T, rp.G = G, rp.mw = MW;
    rp.total_rows = S + (c.use_power ? S : 0u);
    memcpy(&rp.thr, &c.thr_bits, 4);
    rp.done = &done, rp.need = (unsigned long long)rep;
    rp.util_u8 = variant == 2 ? 1u : 0u;
    // exactly the launch gpr_api.cu would make for this window on this device with these knobs
    gpr::LaunchKnobs k = c.knobs;
    k.variant = variant == 1 ? GPR_KERNEL_TMA : GPR_KERNEL_LDG;
    auto a16 = [](const void* p) { return reinterpret_cast<uintptr_t>(p) % 16u == 0; };
    const bool tma_ok = T % 4u == 0 && c.ld % 4u == 0 && a16(util) && (!c.use_power || a16(power));
    plan = gpr::plan_reduce(k, T, rp.total_rows, tma_ok, rp.util_u8 != 0);
    if (plan.kernel == gpr::kReduceLdg) {
      launch(plan.grid, plan.block, 0, [&] { gpr::k_reduce_ldg<gpr::kLdgWarps, gpr::kLdgUnroll>(rp); });
    } else if (plan.kernel == gpr::kReduceU8) {
      launch(plan.grid, plan.block, 0, [&] { gpr::k_reduce_u8<gpr::kLdgWarps, gpr::kU8Unroll>(rp); });
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
    fp.veto_mask = c.use_power ? masks.data() + (size_t)P * MW : nullptr;
    fp.eligible = c.elig.empty() ? nullptr : c.elig.data();
    fp.created = c.created.empty() ? nullptr : c.created.data();
    fp.cutoff = c.cutoff;
    fp.dbits = dbits.data(), fp.cbits = cbits.data(), fp.vbits = vbits.data();
    fp.counts = counts, fp.acc = acc, fp.ticket = &ticket;
    fp.done = &done, fp.need = (unsigned long long)rep;
    fp.prev_done = &other_done, fp.prev_need = 0;
    fp.P = P, fp.G = G, fp.mw = MW;
    fp.world = 1, fp.rank = 0;
    fp.err = &err;
    const uint32_t fold_grid = gpr::fold_grid(c.knobs, P);
    launch(fold_grid, (unsigned)c.knobs.fold_threads, 0, [&] { gpr::k_fold<false>(fp); });
    bool clean = done == (unsigned long long)rep + 1 && ticket == 0 && !acc[0] && !acc[1] && !acc[2];
    for (uint32_t m : masks) clean = clean && m == 0;
    printf("%s %s%s %s ", dir.c_str(), name, rep ? "#2" : "", clean ? "clean" : "DIRTY");
    print_words(dbits), printf(" "), print_words(cbits), printf(" "), print_words(vbits);
    printf(" %llu %llu %llu ", counts[0], counts[1], counts[2]);
    for (float v : smax) printf("%08x", f2u(v));
    // what ran: kernel fallback grid block smem depth stage_bytes chunk_elems n_chunks fold_grid fold_threads rounds
    printf(" plan=%s,%d,%u,%u,%zu,%u,%u,%u,%u,%u,%d,%u\n", kernel_name(plan.kernel), plan.fallback, plan.grid,
           plan.block, plan.smem, plan.L.depth, plan.L.stage_bytes, plan.L.chunk_elems, plan.L.n_chunks, fold_grid,
           c.knobs.fold_threads, gpr::fold_rounds(c.knobs, P));
  }
}

int main(int argc, char** argv) {
  // --synth SEED P G T OUT_PREFIX : run the device generator's source, write <prefix>.util.f32 / .power.f32 / .elig.u8
  if (argc == 7 && std::string(argv[1]) == "--synth") {
    const uint64_t seed = strtoull(argv[2], nullptr, 0);
    const uint32_t P = (uint32_t)atoi(argv[3]), G = (uint32_t)atoi(argv[4]), T = (uint32_t)atoi(argv[5]);
    const std::string prefix = argv[6];
    std::vector<float> buf((size_t)P * G * T);
    for (int plane = 0; plane < 2; ++plane) {
      launch(5, 64, 0, [&] { gpr::k_synth_fill(buf.data(), seed, plane, 0, P * G, T, T); });
      std::ofstream(prefix + (plane ? ".power.f32" : ".util.f32"), std::ios::binary)
          .write(reinterpret_cast<const char*>(buf.data()), (std::streamsize)(buf.size() * 4));
    }
    std::vector<uint8_t> e(P);
    launch(2, 64, 0, [&] { gpr::k_synth_eligible(e.data(), seed, 0, P); });
    std::ofstream(prefix + ".elig.u8", std::ios::binary).write(reinterpret_cast<const char*>(e.data()), (std::streamsize)e.size());
    return 0;
  }
  // --rowsplit GRID TOTAL... : the rows k_reduce_* give each CTA (cta_row_count); prints grid total sum min max
  if (argc >= 4 && std::string(argv[1]) == "--rowsplit") {
    const unsigned grid = (unsigned)strtoul(argv[2], nullptr, 0);
    for (int a = 3; a < argc; ++a) {
      const uint32_t total = (uint32_t)strtoull(argv[a], nullptr, 0);
      uint64_t sum = 0, lo = ~0ull, hi = 0;
      gridDim.x = grid;
      for (unsigned b = 0; b < grid; ++b) {
        blockIdx.x = b;
        const uint64_t n = gpr::cta_row_count(total);
        sum += n, lo = std::min(lo, n), hi = std::max(hi, n);
      }
      printf("%u %u %llu %llu %llu\n", grid, total, (unsigned long long)sum, (unsigned long long)lo, (unsigned long long)hi);
    }
    return 0;
  }
  g_max_resident_ctas = 4;   // the kernels run here never wait for another CTA of their grid
  for (int a = 1; a < argc; ++a) {
    const std::string dir = argv[a];
    Case c;
    {
      std::ifstream f(dir + "/params.txt");
      unsigned long long ld;
      f >> c.P >> c.G >> c.T >> ld >> c.use_power >> c.thr_bits >> c.cutoff;
      c.ld = ld;
    }
    default_knobs(&c.knobs);
    if (std::ifstream f(dir + "/knobs.txt"); f) {
      gpr::LaunchKnobs& k = c.knobs;
      std::string labels;
      f >> k.sm_count >> k.tma_warps >> k.tma_chunk_bytes >> k.tma_depth_max >> k.ldg_ctas_per_sm >> k.fold_threads >> labels;
      for (size_t i = 0; i < labels.size();) {
        const size_t j = std::min(labels.find(',', i), labels.size());
        c.labels.push_back(labels.substr(i, j - i));
        i = j + 1;
      }
    }
    slurp(dir + "/util.f32", &c.util);
    if (c.use_power) slurp(dir + "/power.f32", &c.power);
    slurp(dir + "/elig.u8", &c.elig);
    slurp(dir + "/created.i64", &c.created);
    const bool has_u8 = slurp(dir + "/util.u8", &c.util_u8);
    if (c.P == 0) continue;
    if (c.labels.empty()) {
      run_variant(dir, "ldg", c, 0, 0);
      run_variant(dir, "ldg+1", c, 0, 1);   // rows start 4 bytes off 16-byte alignment
      if (c.T % 4 == 0 && c.ld % 4 == 0) run_variant(dir, "tma", c, 1, 0);
      if (has_u8) run_variant(dir, "u8", c, 2, 0);
    }
    for (const std::string& l : c.labels) {
      if (l == "u8" && !has_u8) continue;
      run_variant(dir, l.c_str(), c, l == "u8" ? 2 : l.rfind("tma", 0) == 0 ? 1 : 0, l.back() == '1' ? 1 : 0);
    }
    fflush(stdout);
  }
  return 0;
}
