// TEST INFRASTRUCTURE.  `gpu-pruner -d --retime-ring` (DESIGN.md §8e) on the EMULATED device of tests/cpp/text_emul.cpp
// (its kernel flavour: k_text_parse's source under tests/cpp/cuda_shim.hpp), extended by what a retiming tick needs: the
// SOURCE of k_retime_rows (gpu-pruner_b200/csrc/gpr_ring.cuh), launched as gpr_resident_retime launches it, the sources
// of k_live_rows and k_remap_rows for the PROF-row check, ring growth and reshapes, k_ring_cols for --late-seconds, and a
// row patch at any column range.  The ticks go through the binary's own FileSource (controller.cpp), so the delta
// ranges, the slicing, the logging and the full-range fallback are the binary's.
//
//   retime_ticks_emul [--retime] <L> <S> <duration_min> <power_threshold> <dir>     dir/tick-%04d/{full,delta}/...
// dir/tick-%04d/duration (optional) holds the --duration in minutes from that tick on.  After every tick the resident
// ring must hold exactly the window a fresh full-range ingest of full/ at that tick's step and duration yields: every
// series' row by identity, nothing but "no sample" anywhere else.  Prints per tick
//   OK tick=<k> mode=<full|delta|failed> T=<T>  |  MISMATCH tick=<k> <what>
// then the tick's MAXIMA lines: per pod, its series with the NaN-aware maximum of their rows (what the verdict is made
// of; the sample count depends on the step).  The binary's log goes to stderr.
// EMUL_RESTORE_BEFORE=k: before tick k the session is saved, the ring kept aside, and both restored into a new session,
// as a restart with --snapshot-file does.  EMUL_FAIL_RETIME=1: every retime fails as a GPR_E_NOMEM would.
// EMUL_RESHAPE=1: the run also has --reshape-ring.
#define main text_emul_main
#include "text_emul.cpp"
#undef main

#define __host__
namespace gpr {
#include "hotpath_extract.inc"
#include "ring_extract.inc"
}

#include <limits>

#include "controller.hpp"

namespace {

class RetimeDevice : public EmulDevice {
 public:
  void resident_init(uint32_t pods, uint32_t G, uint32_t T, bool with_power) override {
    EmulDevice::resident_init(pods, G, T, with_power);
    rows_ = pods * G, T_ = T;
  }
  uint32_t ring_rows() const { return rows_; }
  uint32_t ring_T() const { return T_; }

  // as gpr_resident_retime: k_retime_rows per plane into a new buffer.  ring_row() unrolls a row oldest first, so the
  // unrolled plane is a ring with head 0; the new ring is written back row by row into a fresh ring of the new length
  void resident_retime(uint32_t n_keep, uint32_t factor) override {
    if (getenv("EMUL_FAIL_RETIME")) throw std::runtime_error("gpr_resident_retime (4): emulated: out of device memory");
    if (factor == 0 || n_keep == 0 || n_keep > T_) throw std::logic_error("emul: bad retime");
    const uint32_t T_new = gpr::retime_len(n_keep, factor), rows = rows_, T = T_;
    const bool power = has_ring_power();
    std::vector<std::vector<uint32_t>> next;
    for (int k = 0; k < (power ? 2 : 1); ++k) {
      const std::vector<uint32_t> old = unrolled(k);
      next.emplace_back((size_t)rows * T_new, 0xA5A5A5A5u);
      uint32_t* dst = next.back().data();
      launch(gpr::ring_grid(rows, 2), gpr::kRingThreads, 0,
             [&] { gpr::k_retime_rows(dst, old.data(), rows, T, 0, n_keep, factor, nullptr, 0); });
    }
    resident_init(rows, 1, T_new, power);  // only the row count matters to the emulated ring
    for (int k = 0; k < (int)next.size(); ++k)
      for (uint32_t r = 0; r < rows; ++r)
        patch_row(k, r, T_new, reinterpret_cast<const float*>(next[k].data() + (size_t)r * T_new), T_new, true);
    ++retimes;
  }
  int retimes = 0;

  void resident_cols(int plane, uint32_t newer, uint32_t n_cols, std::vector<float>* out) override {
    if (plane == 1 && !has_ring_power()) throw std::logic_error("emul: no power plane");
    if (n_cols == 0 || (uint64_t)newer + n_cols > T_) throw std::logic_error("emul: band outside the ring");
    const std::vector<uint32_t> cells = unrolled(plane);
    std::vector<uint32_t> band((size_t)rows_ * n_cols, 0xA5A5A5A5u);
    uint32_t* dst = band.data();
    const uint32_t rows = rows_, T = T_, start = gpr::ring_cols_start(0, T_, newer, n_cols);
    launch(gpr::ring_grid(rows, 2), gpr::kRingThreads, 0,
           [&] { gpr::k_ring_cols(dst, cells.data(), rows, T, start, n_cols); });
    out->resize(band.size());
    memcpy(out->data(), band.data(), band.size() * 4);
  }

  void resident_live_rows(std::vector<uint32_t>* bits) override {
    const std::vector<uint32_t> p0 = unrolled(0), p1 = has_ring_power() ? unrolled(1) : std::vector<uint32_t>();
    bits->assign(((size_t)rows_ + 31) / 32, 0xA5A5A5A5u);
    uint32_t* dst = bits->data();
    const uint32_t rows = rows_, T = T_;
    launch(gpr::live_rows_grid(rows, 1), gpr::kRingThreads, 0,
           [&] { gpr::k_live_rows(p0.data(), p1.empty() ? nullptr : p1.data(), rows, T, dst); });
  }

  void resident_remap(uint32_t pods, uint32_t G, const std::vector<uint32_t>& src_rows) override {
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

  void patch_cols(int plane, uint32_t row, uint32_t T, const float* data, uint32_t n, uint32_t newer,
                  bool resident) override {
    if (!resident || n + newer > T) throw std::logic_error("emul: column patch outside the ring");
    std::vector<float> r = ring_row(plane, row);
    memcpy(r.data() + (T - newer - n), data, (size_t)n * 4);
    patch_row(plane, row, T, r.data(), T, true);
  }

  void keep_for_restore() {
    kept_.assign(has_ring_power() ? 2 : 1, {});
    for (size_t k = 0; k < kept_.size(); ++k)
      for (uint32_t r = 0; r < rows_; ++r) kept_[k].push_back(ring_row((int)k, r));
  }
  void resident_restore(uint32_t pods, uint32_t G, uint32_t T, bool with_power, const ChunkPlaneView*,
                        const TextGrid&) override {
    resident_init(pods, G, T, with_power);
    if (kept_.size() != (with_power ? 2u : 1u)) throw std::logic_error("emul: restore without a kept ring");
    for (size_t k = 0; k < kept_.size(); ++k)
      for (uint32_t r = 0; r < rows_ && r < kept_[k].size(); ++r) patch_row((int)k, r, T, kept_[k][r].data(), T, true);
    kept_.clear();
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
  std::vector<std::vector<std::vector<float>>> kept_;
};

class EmulIngestor : public TextIngestor {
 public:
  explicit EmulIngestor(RetimeDevice& dev) : dev_(dev), session_(new DeviceIngestSession(dev)) {}
  Window ingest(const Cli&, const std::string& util, const std::string* prof, const std::string* power,
                const IngestOptions& opt, std::string*) override {
    last_delta = opt.slice_seconds > 0;
    return session_->ingest(util, prof, power, opt);
  }
  Window ingest_slices(const Cli&, const SlicedFetch& f, const IngestOptions& opt, std::string*) override {
    last_delta = opt.slice_seconds > 0;
    return session_->ingest_slices(f, opt);
  }
  int64_t resident_t_end() const override { return session_->resident_t_end(); }
  bool restart() {
    SnapshotState s;
    if (!session_->save_state(&s)) return false;
    dev_.keep_for_restore();
    session_.reset(new DeviceIngestSession(dev_));
    ChunkPlaneView planes[2];
    session_->restore_state(s, planes);
    return true;
  }
  bool last_delta = false;

 private:
  RetimeDevice& dev_;
  std::unique_ptr<DeviceIngestSession> session_;
};

std::string fresh_mismatch(const RetimeDevice& dev, const Window& wr, const Window& wf) {
  if (!wr.resident) return "session did not keep the window resident";
  if (wr.T != wf.T || wr.step != wf.step || wr.t_end != wf.t_end || wr.span != wf.span) return "grid";
  if ((size_t)wr.resident_pods * wr.G != dev.ring_rows() || wr.T != dev.ring_T()) return "the session's shape is not the ring's";
  std::vector<uint8_t> row_used((size_t)wr.resident_pods * wr.G, 0), power_used(row_used.size(), 0);
  for (uint32_t pf = 0; pf < wf.P; ++pf) {
    const PodEntry& a = wf.pods[pf];
    uint32_t pr = 0;
    while (pr < wr.P && !(wr.pods[pr].name == a.name && wr.pods[pr].ns == a.ns)) ++pr;
    if (pr == wr.P) return "pod " + a.name + " missing from the resident window";
    const PodEntry& b = wr.pods[pr];
    for (uint32_t sf = 0; sf < a.slots.size(); ++sf) {
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
      for (uint32_t sf = 0; sf < a.power_slots; ++sf) {
        bool found = false;
        for (uint32_t sr = 0; !found && sr < b.power_slots; ++sr) {
          const size_t row = (size_t)pr * wr.G + sr;
          if (!power_used[row] && rows_equal(dev.ring_row(1, (uint32_t)row), wf.power.data() + ((size_t)pf * wf.G + sf) * wf.T))
            power_used[row] = 1, found = true;
        }
        if (!found) return "power row of " + a.name + " differs from a fresh ingest";
      }
    }
  }
  for (size_t row = 0; row < row_used.size(); ++row) {
    if (!row_used[row] && !row_is_empty(dev.ring_row(0, (uint32_t)row))) return "stale samples in util row " + std::to_string(row);
    if (dev.has_ring_power() && !power_used[row] && !row_is_empty(dev.ring_row(1, (uint32_t)row)))
      return "stale samples in power row " + std::to_string(row);
  }
  return "";
}

// per pod (by name): its series (by key) with the NaN-aware maximum of their rows, its power rows' maxima sorted
std::string maxima_lines(int k, const RetimeDevice& dev, const Window& wr) {
  auto stat = [&](int plane, uint32_t row) {
    float m = std::numeric_limits<float>::quiet_NaN();
    for (float v : dev.ring_row(plane, row))
      if (!std::isnan(v)) m = std::isnan(m) ? v : std::max(m, v);
    char b[64];
    snprintf(b, sizeof b, "%.9g", m);
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
    if (util.empty() && power.empty()) continue;
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

int run(bool retime, int64_t L, int64_t S, int64_t duration_min, double thr, const std::string& dir) {
  RetimeDevice dev;
  EmulIngestor ing(dev);
  Logger log(LogFormat::Default, stderr);
  std::unique_ptr<WindowSource> src = make_window_source("file://" + dir, &ing, &log);
  Cli args;
  args.daemon_mode = true, args.duration = duration_min, args.query_slice = S, args.retime_ring = retime;
  args.late_seconds = L;
  args.reshape_ring = getenv("EMUL_RESHAPE") != nullptr;
  if (thr != 0.0) args.power_threshold = thr;
  int bad = 0;
  const int restore_before = getenv("EMUL_RESTORE_BEFORE") ? atoi(getenv("EMUL_RESTORE_BEFORE")) : -1;
  for (int k = 0;; ++k) {
    if (k == restore_before) ing.restart();
    char name[32];
    snprintf(name, sizeof name, "/tick-%04d", k);
    const std::string base = dir + name;
    if (!file_there(base + "/full/query.json")) break;
    std::string dur;
    if (slurp(base + "/duration", &dur)) args.duration = atoll(dur.c_str());
    Window wr;
    try {
      wr = src->fetch(args);
    } catch (const std::exception& e) {
      printf("OK tick=%d mode=failed T=0 %s\n", k, e.what());
      continue;
    }
    try {
      std::string util, prof, power;
      const std::string fd = base + "/full";
      slurp(fd + "/util.json", &util);
      const bool hp = slurp(fd + "/prof.json", &prof);
      const bool hw = thr != 0.0 && slurp(fd + "/power.json", &power);
      const Json meta = Json::parse_file(fd + "/query.json");
      IngestOptions of;
      of.duration_min = args.duration, of.power_threshold = thr;
      of.t_end = (int64_t)meta["end"].as_number(0), of.step = (int64_t)meta["step"].as_number(0);
      const Window wf = ingest_matrix_text(util, hp ? &prof : nullptr, hw ? &power : nullptr, of, 2);
      const std::string what = fresh_mismatch(dev, wr, wf);
      if (what.empty())
        printf("OK tick=%d mode=%s T=%u\n%s", k, ing.last_delta ? "delta" : "full", wr.T, maxima_lines(k, dev, wr).c_str());
      else
        printf("MISMATCH tick=%d %s\n", k, what.c_str()), ++bad;
    } catch (const std::exception& e) {
      printf("MISMATCH tick=%d exception %s\n", k, e.what());
      ++bad;
    }
  }
  fflush(stdout);
  return bad ? 1 : 0;
}

}  // namespace

int main(int argc, char** argv) {
  const bool retime = argc == 7 && std::string(argv[1]) == "--retime";
  if (argc != 6 + (int)retime) return 2;
  const int a = 1 + retime;
  return run(retime, atoll(argv[a]), atoll(argv[a + 1]), atoll(argv[a + 2]), strtod(argv[a + 3], nullptr), argv[a + 4]);
}
