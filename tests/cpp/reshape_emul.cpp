// TEST INFRASTRUCTURE.  Daemon mode with --reshape-ring (IngestOptions::reshape, DESIGN.md §8e) on the EMULATED device
// of tests/cpp/text_emul.cpp (its kernel flavour: k_text_parse's source under tests/cpp/cuda_shim.hpp), extended by the
// two methods reshaping needs.  They run the SOURCE of k_live_rows and k_remap_rows (gpu-pruner_b200/csrc/gpr_ring.cuh,
// cut out with gpr_kernels.cuh into ring_extract.inc / hotpath_extract.inc by tests/test_resident_reshape.py), launched
// as gpr_resident_live_rows and gpr_resident_remap launch them.  The emulator's ring is reached through its own
// interface (ring_row, patch_row, resident_init): both kernels work on the unrolled ring (a row's cells in any fixed
// order are all they read), and a remapped ring is written back row by row into a fresh ring of the new shape.
//
//   reshape_emul [--reshape] <duration_min> <dir>        dir/tick-0000/{full,delta}/..., as text_emul --ticks reads it
// After every tick the resident ring must hold exactly the window a fresh full-range ingest of that tick yields: the
// same samples for every series of every pod (by identity: a reshape orders rows differently), nothing but "no sample"
// anywhere else.  Prints per tick  OK tick=<k> mode=<full|delta|failed> [why]  |  MISMATCH tick=<k> <what>,  where a
// reshaping delta tick's why is the session's log line, then the tick's MAXIMA lines (see maxima_lines).
// EMUL_FAIL_REMAP=1: every remap fails as a GPR_E_NOMEM would.
#define main text_emul_main
#include "text_emul.cpp"
#undef main

#define __host__
namespace gpr {
#include "hotpath_extract.inc"
#include "ring_extract.inc"
}

#include <limits>

namespace {

class ReshapeDevice : public EmulDevice {
 public:
  void resident_init(uint32_t pods, uint32_t G, uint32_t T, bool with_power) override {
    EmulDevice::resident_init(pods, G, T, with_power);
    rows_ = pods * G, T_ = T;
  }
  uint32_t ring_rows() const { return rows_; }

  // as gpr_resident_live_rows launches k_live_rows on a ring without an index (the binary's), on a one-SM grid
  void resident_live_rows(std::vector<uint32_t>* bits) override {
    const std::vector<uint32_t> p0 = unrolled(0), p1 = has_ring_power() ? unrolled(1) : std::vector<uint32_t>();
    std::vector<uint32_t> out((rows_ + 31) / 32, 0xA5A5A5A5u);  // every word must be written
    const uint32_t rows = rows_, T = T_;
    const uint32_t* q1 = p1.empty() ? nullptr : p1.data();
    launch(gpr::live_rows_grid(rows, 1), gpr::kRingThreads, 0, [&] { gpr::k_live_rows(p0.data(), q1, rows, T, out.data()); });
    bits->swap(out);
  }

  // as gpr_resident_remap: the host map checked first, then k_remap_rows per plane into a new buffer
  void resident_remap(uint32_t pods, uint32_t G, const std::vector<uint32_t>& src_rows) override {
    if (getenv("EMUL_FAIL_REMAP")) throw std::runtime_error("gpr_resident_remap (4): emulated: out of device memory");
    const uint32_t n_new = pods * G, T = T_;
    if (src_rows.size() != n_new) throw std::logic_error("emul: remap map has the wrong size");
    if (gpr::remap_first_bad(src_rows.data(), n_new, rows_) < n_new) throw std::logic_error("emul: bad remap map");
    const bool power = has_ring_power();
    std::vector<std::vector<uint32_t>> next;
    for (int k = 0; k < (power ? 2 : 1); ++k) {
      const std::vector<uint32_t> old = unrolled(k);
      next.emplace_back((size_t)n_new * T, 0xA5A5A5A5u);
      uint32_t* dst = next.back().data();
      launch(gpr::ring_grid(n_new, 1), gpr::kRingThreads, 0,
             [&] { gpr::k_remap_rows(dst, old.data(), src_rows.data(), n_new, T); });
    }
    resident_init(pods, G, T, power);
    for (int k = 0; k < (int)next.size(); ++k)
      for (uint32_t r = 0; r < n_new; ++r)
        patch_row(k, r, T, reinterpret_cast<const float*>(next[k].data() + (size_t)r * T), T, true);
  }

 private:
  std::vector<uint32_t> unrolled(int plane) const {  // oldest bucket first
    std::vector<uint32_t> cells((size_t)rows_ * T_);
    for (uint32_t r = 0; r < rows_; ++r) {
      const std::vector<float> row = ring_row(plane, r);
      memcpy(cells.data() + (size_t)r * T_, row.data(), (size_t)T_ * 4);
    }
    return cells;
  }
  uint32_t rows_ = 0, T_ = 0;
};

// "" = the resident ring holds exactly the window a fresh full-range ingest of the tick yields
std::string fresh_mismatch(const ReshapeDevice& dev, const Window& wr, const Window& wf) {
  if (!wr.resident) return "session did not keep the window resident";
  if (wr.T != wf.T || wr.step != wf.step || wr.t_end != wf.t_end || wr.span != wf.span) return "grid";
  if ((size_t)wr.resident_pods * wr.G != dev.ring_rows()) return "the session's shape is not the ring's";
  std::vector<uint8_t> row_used((size_t)wr.resident_pods * wr.G, 0);
  for (uint32_t pf = 0; pf < wf.P; ++pf) {
    const PodEntry& a = wf.pods[pf];
    uint32_t pr = 0;
    while (pr < wr.P && !(wr.pods[pr].name == a.name && wr.pods[pr].ns == a.ns)) ++pr;
    if (pr == wr.P) return "pod " + a.name + " missing from the resident window";
    const PodEntry& b = wr.pods[pr];
    for (uint32_t sf = 0; sf < a.slots.size(); ++sf) {  // duplicates of one series key: any order
      bool found = false;
      for (uint32_t sr = 0; !found && sr < b.slots.size(); ++sr) {
        const size_t row = (size_t)pr * wr.G + sr;
        if (row_used[row] || slot_key(b.slots[sr]) != slot_key(a.slots[sf])) continue;
        if (rows_equal(dev.ring_row(0, (uint32_t)row), wf.util.data() + ((size_t)pf * wf.G + sf) * wf.T)) row_used[row] = 1, found = true;
      }
      if (!found) return "util row of " + a.name + " gpu " + a.slots[sf].gpu + " differs from a fresh ingest";
    }
    if (a.power_slots) {
      if (!dev.has_ring_power()) return "no resident power plane";
      std::vector<uint8_t> used(b.power_slots, 0);  // power rows carry no identity beyond the pod: a multiset
      for (uint32_t sf = 0; sf < a.power_slots; ++sf) {
        bool found = false;
        for (uint32_t sr = 0; !found && sr < b.power_slots; ++sr)
          if (!used[sr] && rows_equal(dev.ring_row(1, pr * wr.G + sr), wf.power.data() + ((size_t)pf * wf.G + sf) * wf.T)) used[sr] = 1, found = true;
        if (!found) return "power row of " + a.name + " differs from a fresh ingest";
      }
      for (uint32_t sr = 0; sr < b.power_slots; ++sr)
        if (!used[sr] && !row_is_empty(dev.ring_row(1, pr * wr.G + sr))) return "stale power row in " + a.name;
    }
  }
  for (size_t row = 0; row < row_used.size(); ++row)
    if (!row_used[row] && !row_is_empty(dev.ring_row(0, (uint32_t)row))) return "stale samples in resident row " + std::to_string(row);
  return "";
}

// What the verdict of a tick is made of, independent of where the rows sit in the ring: per pod (by name), its series
// (by key) with the NaN-aware maximum and the sample count of their rows, its power rows as a sorted list.  Two runs of
// one timeline that decide alike print the same lines.
std::string maxima_lines(int k, const ReshapeDevice& dev, const Window& wr) {
  auto stat = [&](int plane, uint32_t row) {
    float m = std::numeric_limits<float>::quiet_NaN();
    int n = 0;
    for (float v : dev.ring_row(plane, row))
      if (!std::isnan(v)) m = std::isnan(m) ? v : std::max(m, v), ++n;
    char b[64];
    snprintf(b, sizeof b, "%.9g/%d", m, n);
    return std::string(b);
  };
  std::vector<std::string> pods;
  for (uint32_t p = 0; p < wr.P; ++p) {
    const PodEntry& pe = wr.pods[p];
    std::vector<std::string> util, power;
    for (uint32_t s = 0; s < pe.slots.size(); ++s)
      if (!row_is_empty(dev.ring_row(0, p * wr.G + s))) util.push_back(slot_key(pe.slots[s]) + "=" + stat(0, p * wr.G + s));
    for (uint32_t s = 0; s < pe.power_slots && dev.has_ring_power(); ++s)
      if (!row_is_empty(dev.ring_row(1, p * wr.G + s))) power.push_back(stat(1, p * wr.G + s));
    if (util.empty() && power.empty()) continue;  // a pod without a sample in the window is not in a fresh ingest
    std::sort(util.begin(), util.end()), std::sort(power.begin(), power.end());
    std::string line = pe.ns + "/" + pe.name + ":";
    for (const std::string& u : util) line += " " + u;
    line += " |";
    for (const std::string& x : power) line += " " + x;
    pods.push_back(line);
  }
  std::sort(pods.begin(), pods.end());
  std::string out;
  for (const std::string& l : pods) out += "MAXIMA tick=" + std::to_string(k) + " " + l + "\n";
  return out;
}

int run(bool reshape, int64_t duration_min, const std::string& dir) {
  ReshapeDevice dev;
  DeviceIngestSession session(dev);
  int bad = 0;
  for (int k = 0;; ++k) {
    char name[32];
    snprintf(name, sizeof name, "/tick-%04d", k);
    const std::string base = dir + name;
    if (!file_there(base + "/full/util.json")) break;
    auto load = [&](const std::string& d, std::string* util, std::string* prof, std::string* power, bool* hp, bool* hw,
                    IngestOptions* o) {
      slurp(d + "/util.json", util);
      *hp = slurp(d + "/prof.json", prof), *hw = slurp(d + "/power.json", power);
      const Json meta = Json::parse_file(d + "/query.json");
      o->duration_min = duration_min;
      o->t_end = (int64_t)meta["end"].as_number(0), o->step = (int64_t)meta["step"].as_number(0);
      o->reshape = reshape;
      return (int64_t)meta["start"].as_number(0);
    };
    std::string util, prof, power, mode = "full", why;
    bool hp = false, hw = false, done = false;
    IngestOptions o;
    Window wr;
    try {
      const int64_t since = session.resident_t_end();
      if (since > 0 && file_there(base + "/delta/util.json")) {
        const int64_t start = load(base + "/delta", &util, &prof, &power, &hp, &hw, &o);
        if (start == since) {
          o.slice_seconds = o.t_end - start, o.resident = true;
          try {
            wr = session.ingest(util, hp ? &prof : nullptr, hw ? &power : nullptr, o);
            mode = "delta", done = true, why = wr.stats.ring_reshape;
          } catch (const NeedFullWindow& e) {
            why = e.what();
          } catch (const std::runtime_error& e) {
            printf("OK tick=%d mode=failed %s\n", k, e.what());  // the controller logs "Failed to run query!"
            continue;
          }
        } else {
          why = "delta does not continue the resident window";
        }
      }
      load(base + "/full", &util, &prof, &power, &hp, &hw, &o);
      o.slice_seconds = 0, o.resident = true;
      if (!done) wr = session.ingest(util, hp ? &prof : nullptr, hw ? &power : nullptr, o);
      IngestOptions of = o;
      of.resident = false;
      const Window wf = ingest_matrix_text(util, hp ? &prof : nullptr, hw ? &power : nullptr, of, 2);
      const std::string what = fresh_mismatch(dev, wr, wf);
      if (what.empty()) printf("OK tick=%d mode=%s %s\n%s", k, mode.c_str(), why.c_str(), maxima_lines(k, dev, wr).c_str());
      else printf("MISMATCH tick=%d %s\n", k, what.c_str()), ++bad;
    } catch (const std::exception& e) {
      printf("MISMATCH tick=%d exception %s\n", k, e.what());
      ++bad;
    }
  }
  return bad ? 1 : 0;
}

}  // namespace

int main(int argc, char** argv) {
  const bool reshape = argc == 4 && std::string(argv[1]) == "--reshape";
  if (argc != 3 + (int)reshape) return 2;
  return run(reshape, atoll(argv[1 + reshape]), argv[2 + reshape]);
}
