// TEST INFRASTRUCTURE.  `gpu-pruner -d --query-slice S` (DESIGN.md §8e) on the EMULATED device of tests/cpp/text_emul.cpp
// (its kernel flavour: k_text_parse's source under tests/cpp/cuda_shim.hpp), extended by what a sliced fetch needs: the
// SOURCE of k_remap_rows (gpu-pruner_b200/csrc/gpr_ring.cuh) for ring growth, launched as gpr_resident_remap launches
// it, and a row patch at any column range.  The ticks go through the binary's own FileSource (controller.cpp), so the
// slicing rule, the slice checks and the full-range fallback are the binary's.
//
//   slice_emul [--reshape] <S> <duration_min> <power_threshold> <dir>     dir/tick-%04d/{full,delta}/[slice-%04d/]...
// After every tick the resident ring must hold exactly the window a fresh full-range ingest of the tick's whole-range
// responses yields: every series' row by identity, nothing but "no sample" anywhere else.  Prints per tick
//   OK tick=<k> mode=<full|delta|failed> slices=<n> [why]  |  MISMATCH tick=<k> <what>
// then the tick's MAXIMA lines: per pod, its series' maxima and sample counts, independent of where the rows sit.
// EMUL_RESTORE_BEFORE=k: before tick k the session is saved (save_state), the ring kept aside, and both restored into a
// new session (restore_state), as a restart with --snapshot-file does.
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

class SliceDevice : public EmulDevice {
 public:
  void resident_init(uint32_t pods, uint32_t G, uint32_t T, bool with_power) override {
    EmulDevice::resident_init(pods, G, T, with_power);
    rows_ = pods * G, T_ = T;
  }
  uint32_t ring_rows() const { return rows_; }

  // as gpr_resident_remap: the host map checked first, then k_remap_rows per plane into a new buffer
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

  // the n buckets ending `newer` before the newest; every other bucket of the row keeps its bits
  void patch_cols(int plane, uint32_t row, uint32_t T, const float* data, uint32_t n, uint32_t newer,
                  bool resident) override {
    if (!resident || n + newer > T) throw std::logic_error("emul: column patch outside the ring");
    std::vector<float> r = ring_row(plane, row);
    memcpy(r.data() + (T - newer - n), data, (size_t)n * 4);
    ++patched_cols_calls;
    if (newer) ++patched_older_calls;
    patch_row(plane, row, T, r.data(), T, true);
  }
  int patched_cols_calls = 0, patched_older_calls = 0;

  // a process restart (EMUL_RESTORE_BEFORE): the ring's rows are kept aside as the snapshot's planes would carry them,
  // and a fresh ring of the snapshot's shape gets them back, as gpr_chunks_scatter merges the exported chunks
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

// the binary's GprVerdictEngine as a TextIngestor, over the emulated device
class EmulIngestor : public TextIngestor {
 public:
  explicit EmulIngestor(SliceDevice& dev) : dev_(dev), session_(new DeviceIngestSession(dev)) {}
  Window ingest(const Cli&, const std::string& util, const std::string* prof, const std::string* power,
                const IngestOptions& opt, std::string*) override {
    last_delta = opt.slice_seconds > 0, last_slices = 1;
    return session_->ingest(util, prof, power, opt);
  }
  Window ingest_slices(const Cli&, const SlicedFetch& f, const IngestOptions& opt, std::string*) override {
    last_delta = opt.slice_seconds > 0, last_slices = f.ranges.size();
    DeviceIngestReport rep;
    Window w = session_->ingest_slices(f, opt, &rep);
    growths += rep.ring_growths;
    return w;
  }
  int64_t resident_t_end() const override { return session_->resident_t_end(); }
  // the session saved between ticks and restored into a new one, as --snapshot-file does across a restart
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
  size_t last_slices = 0;
  uint64_t growths = 0;

 private:
  SliceDevice& dev_;
  std::unique_ptr<DeviceIngestSession> session_;
};

std::string fresh_mismatch(const SliceDevice& dev, const Window& wr, const Window& wf) {
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
      std::vector<uint8_t> used(b.power_slots, 0);
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

std::string maxima_lines(int k, const SliceDevice& dev, const Window& wr) {
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

int run(bool reshape, int64_t S, int64_t duration_min, double thr, const std::string& dir) {
  SliceDevice dev;
  EmulIngestor ing(dev);
  Logger log(LogFormat::Default, stderr);
  std::unique_ptr<WindowSource> src = make_window_source("file://" + dir, &ing, &log);
  Cli args;
  args.daemon_mode = true, args.duration = duration_min, args.query_slice = S, args.reshape_ring = reshape;
  if (thr != 0.0) args.power_threshold = thr;
  int bad = 0, restores = 0;
  const int restore_before = getenv("EMUL_RESTORE_BEFORE") ? atoi(getenv("EMUL_RESTORE_BEFORE")) : -1;
  for (int k = 0;; ++k) {
    if (k == restore_before) restores += ing.restart();
    char name[32];
    snprintf(name, sizeof name, "/tick-%04d", k);
    const std::string base = dir + name;
    if (!file_there(base + "/full/query.json")) break;
    Window wr;
    try {
      wr = src->fetch(args);
    } catch (const std::exception& e) {
      printf("OK tick=%d mode=failed slices=0 %s\n", k, e.what());
      continue;
    }
    try {
      std::string util, prof, power;
      slurp(base + "/full/util.json", &util);
      const bool hp = slurp(base + "/full/prof.json", &prof);
      const bool hw = thr != 0.0 && slurp(base + "/full/power.json", &power);
      const Json meta = Json::parse_file(base + "/full/query.json");
      IngestOptions of;
      of.duration_min = duration_min, of.power_threshold = thr;
      of.t_end = (int64_t)meta["end"].as_number(0), of.step = (int64_t)meta["step"].as_number(0);
      const Window wf = ingest_matrix_text(util, hp ? &prof : nullptr, hw ? &power : nullptr, of, 2);
      std::string what = fresh_mismatch(dev, wr, wf);
      // the shape a one-query ingest gives the ring, after every full fetch
      if (what.empty() && !ing.last_delta && (wr.resident_pods != wr.P + wr.P / 4 + 64 || wr.G != wf.G))
        what = "the ring's shape after a full fetch is not the one-query shape";
      if (what.empty())
        printf("OK tick=%d mode=%s slices=%zu\n%s", k, ing.last_delta ? "delta" : "full", ing.last_slices,
               maxima_lines(k, dev, wr).c_str());
      else
        printf("MISMATCH tick=%d %s\n", k, what.c_str()), ++bad;
    } catch (const std::exception& e) {
      printf("MISMATCH tick=%d exception %s\n", k, e.what());
      ++bad;
    }
  }
  printf("TOTAL growths=%llu older_patches=%d restores=%d\n", (unsigned long long)ing.growths, dev.patched_older_calls,
         restores);
  return bad ? 1 : 0;
}

}  // namespace

int main(int argc, char** argv) {
  const bool reshape = argc == 6 && std::string(argv[1]) == "--reshape";
  if (argc != 5 + (int)reshape) return 2;
  return run(reshape, atoll(argv[1 + reshape]), atoll(argv[2 + reshape]), strtod(argv[3 + reshape], nullptr),
             argv[4 + reshape]);
}
