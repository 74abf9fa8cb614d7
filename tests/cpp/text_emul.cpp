// TEST INFRASTRUCTURE.  Runs the device ingest (gpu-pruner_b200/host/ingest_device.cpp) on an EMULATED
// device: the very functions the CUDA kernels call (gpu-pruner_b200/csrc/gpr_text.cuh, GPR_HD) executed
// tile by tile, candidate by candidate on the CPU, seeing exactly the bytes a warp's shared-memory stage
// holds (tile + halo).  Each case directory (util.json [prof.json]
// [power.json]) is ingested by the CPU text path and by the emulated device path; shape, pods,
// statistics and every tensor cell must agree, or both must reject the input.
//
//   text_emul <t_end> <step> <duration_min> <case_dir>...       (case_dir/power_threshold: optional, one number)
// prints per case:  OK device=<0|1> spans=.. hard=.. patched=.. [reason]  |  REJECT  |  MISMATCH <what>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <stdexcept>
#include <string>

#ifdef EMUL_PARSE_KERNEL
// The parse pass runs the SOURCE of k_text_parse (gpu-pruner_b200/csrc/gpr_text_kernels.cuh, cut out verbatim into
// text_kernel_extract.inc by the test) as real threads — warps compacting '[' offsets with shuffles, the two-stage
// bulk-copy ring, one candidate per lane — instead of the tile-by-tile loop below.
#include "cuda_shim.hpp"
#endif
#include "../../gpu-pruner_b200/csrc/gpr_text.cuh"
#include "ingest_device.hpp"
#ifdef EMUL_PARSE_KERNEL
namespace gpr {
namespace text {
#include "text_kernel_extract.inc"
}
}
#endif

using namespace gph;
namespace tx = gpr::text;

static_assert(sizeof(gpr_text_span) == sizeof(tx::Span), "gpr_text_span mirrors gpr::text::Span");

namespace {

class EmulDevice : public TextDevice {
 public:
  // the pipelined scan, in chunks far smaller than the device's 4 MB so that series and marker patterns straddle
  // chunk borders all the time
  void scan_begin(int slot, const char* text, size_t n) override {
    std::vector<uint8_t>& t = text_[slot];
    t.assign(n + tx::kTextPad, 0);
    memcpy(t.data(), text, n);
    n_[slot] = n;
    scan_slot_ = slot, scan_pos_ = 0;
  }
  bool scan_next(std::vector<uint64_t>* opens, std::vector<uint64_t>* closes, uint64_t* bytes_done) override {
    if (getenv("EMUL_DECLINE_SCAN") && scan_pos_ > 0) throw DeviceDeclined("emulated: too many markers in one chunk");
    opens->clear(), closes->clear();
    const std::vector<uint8_t>& t = text_[scan_slot_];
    const uint64_t n = n_[scan_slot_];
    struct Sink {
      std::vector<uint64_t>*o, *c;
      void values_open(uint64_t p) { o->push_back(p); }
      void values_close(uint64_t p) { c->push_back(p); }
    } sink{opens, closes};
    const uint64_t end = std::min<uint64_t>(n, scan_pos_ + kEmulChunk);
    const uint64_t s0 = scan_pos_ / tx::kScanBytes, s1 = (end + tx::kScanBytes - 1) / tx::kScanBytes;
    // reversed slice order: nothing may depend on the order threads run in
    for (uint64_t s = s1; s-- > s0;) tx::scan_slice(t.data(), n, s, sink);
    std::sort(opens->begin(), opens->end());
    std::sort(closes->begin(), closes->end());
    scan_pos_ = end;
    *bytes_done = end;
    return end < n;
  }

  // fault injection for the tick tests: the first parse of tick `fail_at_tick` dies like a CUDA error would
  int fail_at_tick = -1, current_tick = 0;
  void parse(int slot, std::vector<gpr_text_span>& spans, const TextGrid& grid, int plane) override {
    if (current_tick == fail_at_tick) {
      fail_at_tick = -1;
      throw std::runtime_error("injected device failure");
    }
    std::vector<uint32_t>& pl = grid.resident ? ring_[plane] : plane_[plane];
    const uint32_t T = grid.T;
    if (grid.resident) {
      if (T != ring_T_ || (size_t)grid.n_rows * T > pl.size()) throw std::logic_error("emul: grid does not match the ring");
    } else {
      if (grid.fill) pl.assign((size_t)grid.n_rows * T, tx::kFillBits);
      if (pl.size() != (size_t)grid.n_rows * T) throw std::logic_error("emul: plane shape changed without fill");
    }
    struct Sink {
      std::vector<uint32_t>& pl;
      tx::Span* sp;
      void put(uint64_t cell, float v) { tx::merge_cell_bits(&pl[cell], v); }
      void hard(uint32_t s) { sp[s].flags |= tx::kSpanHard; }
      void count(uint32_t s, uint32_t a, uint32_t b, uint32_t c) {
        sp[s].n_in += a, sp[s].n_oow += b, sp[s].n_tiny += c;
      }
    } sink{pl, reinterpret_cast<tx::Span*>(spans.data())};
    tx::Grid g;
    memset(&g, 0, sizeof g);
    g.t_end = grid.t_end * 1000, g.t_lo = (grid.t_end - grid.span) * 1000, g.step = (uint32_t)(grid.step * 1000), g.T = T;
    g.col_end = grid.resident ? (ring_head_ + T - 1) % T : T - 1, g.ld = T;
    g.power = tx::power_snap(plane == 1 ? grid.power_threshold : 0.0);  // as gpr_text_parse sets it (gpr_api.cu)
    const std::vector<uint8_t>& text = text_[slot];
    const uint64_t n = n_[slot];
    const tx::Span* sp = reinterpret_cast<const tx::Span*>(spans.data());
    const uint64_t tiles = (n + tx::kTileBytes - 1) / tx::kTileBytes;
#ifdef EMUL_PARSE_KERNEL
    if (!spans.empty() && n) {
      // as gpr_text_parse launches it (gpr_api.cu), on a small grid so that warps own several tiles each
      constexpr int kWarps = 4;
      const unsigned blocks = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((tiles + kWarps - 1) / kWarps, 2));
      tx::Span* dsp = reinterpret_cast<tx::Span*>(spans.data());
      float* dpl = reinterpret_cast<float*>(pl.data());
      const uint32_t n_spans = (uint32_t)spans.size();
      launch(blocks, kWarps * 32, tx::text_parse_smem<kWarps>(), [&] {
        tx::k_text_parse<kWarps>(text.data(), n, n + tx::kTextPad, dsp, n_spans, g, dpl);
      });
    }
    (void)sp, (void)sink;
    return;
#endif
    // what a warp sees: one tile plus the halo, nothing else (bytes beyond are poisoned); tiles in reverse
    // order and candidates from the back: nothing may depend on the order things run in
    struct Tile {
      const uint8_t* p;
      uint32_t operator[](uint32_t i) const { return p[i]; }
    };
    std::vector<uint8_t> stage(tx::kTileBytes + tx::kTileHalo + 64);
    for (uint64_t k = tiles; k-- > 0;) {
      const uint64_t off = k * tx::kTileBytes;
      const uint64_t have = std::min<uint64_t>(tx::kTileBytes + tx::kTileHalo, (n + tx::kTextPad - off) & ~15ull);
      memset(stage.data(), 0xEE, stage.size());
      memcpy(stage.data(), text.data() + off, have);
      const uint32_t tile_n = (uint32_t)std::min<uint64_t>(tx::kTileBytes, n - off);
      const uint32_t s0 = tx::find_span(sp, (uint32_t)spans.size(), off);
      const Tile tile{stage.data()};
      for (uint32_t o = tile_n; o-- > 0;) {
        if (stage[o] != '[') continue;
        uint32_t s = s0;
        tx::parse_candidate(tile, off, o, sp, (uint32_t)spans.size(), s, g, sink);
      }
    }
  }

  void patch_row(int plane, uint32_t row, uint32_t T, const float* data, uint32_t n_newest, bool resident) override {
    uint32_t* base = (resident ? ring_[plane] : plane_[plane]).data() + (size_t)row * T;
    const uint32_t head = resident ? ring_head_ : 0;
    for (uint32_t i = 0; i < n_newest; ++i) memcpy(base + (head + T - n_newest + i) % T, data + i, 4);
  }
  const float* plane(int plane) override { return reinterpret_cast<const float*>(plane_[plane].data()); }
  void resident_init(uint32_t pods, uint32_t G, uint32_t T, bool with_power) override {
    ring_T_ = T, ring_head_ = 0, ring_rows_ = pods * G;
    ring_[0].assign((size_t)ring_rows_ * T, tx::kFillBits);
    ring_[1].clear();
    if (with_power) ring_[1].assign((size_t)ring_rows_ * T, tx::kFillBits);
  }
  void resident_advance(uint32_t n_new) override {
#ifdef EMUL_PARSE_KERNEL
    for (auto& pl : ring_) {   // the source of k_fill_columns, as gpr_resident_advance launches it
      if (pl.empty()) continue;
      float* p = reinterpret_cast<float*>(pl.data());
      const uint32_t rows = ring_rows_, T = ring_T_, head = ring_head_;
      launch(2, 256, 0, [&] { tx::k_fill_columns(p, rows, T, (uint64_t)T, head, n_new); });
    }
    ring_head_ = (ring_head_ + n_new) % ring_T_;
    return;
#endif
    for (auto& pl : ring_)
      for (size_t r = 0; r * ring_T_ < pl.size(); ++r)
        for (uint32_t i = 0; i < n_new; ++i) pl[r * ring_T_ + (ring_head_ + i) % ring_T_] = tx::kFillBits;
    ring_head_ = (ring_head_ + n_new) % ring_T_;
  }
  // row of the ring in chronological order (oldest bucket first)
  std::vector<float> ring_row(int plane, uint32_t row) const {
    std::vector<float> out(ring_T_);
    for (uint32_t c = 0; c < ring_T_; ++c) memcpy(&out[c], &ring_[plane][(size_t)row * ring_T_ + (ring_head_ + c) % ring_T_], 4);
    return out;
  }
  bool has_ring_power() const { return !ring_[1].empty(); }

 private:
  static constexpr uint64_t kEmulChunk = 1024;   // a multiple of the scan slice
  std::vector<uint8_t> text_[3];
  uint64_t n_[3] = {0, 0, 0};
  int scan_slot_ = 0;
  uint64_t scan_pos_ = 0;
  std::vector<uint32_t> plane_[2];   // f32 bit patterns (cells start as 0xFFFFFFFF, like the device planes)
  std::vector<uint32_t> ring_[2];    // the resident window of daemon mode: [rows][T], a ring over the time axis
  uint32_t ring_T_ = 0, ring_head_ = 0, ring_rows_ = 0;
};

bool slurp(const std::string& path, std::string* out) {
  std::ifstream f(path, std::ios::binary);
  if (!f) return false;
  out->assign((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  return true;
}

// value equality: NaN matches NaN (any payload), otherwise ==; `bits` additionally compares bit patterns
bool same_plane(const float* a, const float* b, size_t n, bool bits, size_t* where) {
  for (size_t i = 0; i < n; ++i) {
    const bool na = std::isnan(a[i]), nb = std::isnan(b[i]);
    bool ok = na == nb && (na || a[i] == b[i]);
    if (ok && bits && !na && a[i] != 0.0f) ok = memcmp(a + i, b + i, 4) == 0;  // the sign of a zero may differ after a merge
    if (!ok) {
      *where = i;
      return false;
    }
  }
  return true;
}

}  // namespace

// ---- daemon mode: a sequence of ticks through one DeviceIngestSession on the emulated ring -------------------------
//   text_emul --ticks <duration_min> <dir>      dir/tick-0000/{full,delta}/{util.json,[prof.json],[power.json],query.json}
// After every tick the resident ring must hold exactly the window a fresh full-range ingest of that tick yields:
// same samples for every series of every pod, nothing but "no sample" anywhere else.
// prints per tick:  OK tick=<k> mode=<full|delta> [why]   |   MISMATCH tick=<k> <what>
namespace {
std::string slot_key(const GpuSlot& s) {
  return s.hostname + "\x1f" + s.container + "\x1f" + s.gpu + "\x1f" + s.model + "\x1f" + (s.from_prof ? "P" : "U");
}
bool file_there(const std::string& p) {
  std::ifstream f(p);
  return (bool)f;
}
bool row_is_empty(const std::vector<float>& r) {
  for (float v : r)
    if (!std::isnan(v)) return false;
  return true;
}
bool rows_equal(const std::vector<float>& a, const float* b) {
  for (size_t i = 0; i < a.size(); ++i) {
    const bool na = std::isnan(a[i]), nb = std::isnan(b[i]);
    if (na != nb || (!na && a[i] != b[i])) return false;
  }
  return true;
}

int run_ticks(int64_t duration_min, const std::string& dir) {
  EmulDevice dev;
  if (const char* f = getenv("EMUL_FAIL_PARSE_TICK")) dev.fail_at_tick = atoi(f);
  DeviceIngestSession session(dev);
  int bad = 0;
  for (int k = 0;; ++k) {
    dev.current_tick = k;
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
      return (int64_t)meta["start"].as_number(0);
    };
    std::string util, prof, power, mode = "full", why;
    bool hp = false, hw = false;
    IngestOptions o;
    Window wr;
    bool done = false;
    const int64_t since = session.resident_t_end();
    try {
      if (since > 0 && file_there(base + "/delta/util.json")) {
        const int64_t start = load(base + "/delta", &util, &prof, &power, &hp, &hw, &o);
        if (start == since) {
          o.slice_seconds = o.t_end - start, o.resident = true;
          try {
            wr = session.ingest(util, hp ? &prof : nullptr, hw ? &power : nullptr, o);
            mode = "delta", done = true;
          } catch (const NeedFullWindow& e) {
            why = e.what();
          } catch (const std::runtime_error& e) {
            // the tick fails (the controller logs "Failed to run query!" and waits for the next one)
            printf("OK tick=%d mode=failed %s\n", k, e.what());
            continue;
          }
        } else {
          why = "delta does not continue the resident window";
        }
      }
      load(base + "/full", &util, &prof, &power, &hp, &hw, &o);
      o.slice_seconds = 0, o.resident = true;
      if (!done) wr = session.ingest(util, hp ? &prof : nullptr, hw ? &power : nullptr, o);
      // the reference for this tick: a fresh full-range ingest on the CPU
      IngestOptions of = o;
      of.resident = false;
      const Window wf = ingest_matrix_text(util, hp ? &prof : nullptr, hw ? &power : nullptr, of, 2);
      std::string what;
      if (!wr.resident) what = "session did not keep the window resident";
      if (what.empty() && (wr.T != wf.T || wr.step != wf.step || wr.t_end != wf.t_end || wr.span != wf.span)) what = "grid";
      std::vector<uint8_t> row_used((size_t)wr.resident_pods * wr.G, 0);
      for (uint32_t pf = 0; what.empty() && pf < wf.P; ++pf) {
        const PodEntry& a = wf.pods[pf];
        uint32_t pr = 0;
        while (pr < wr.P && !(wr.pods[pr].name == a.name && wr.pods[pr].ns == a.ns)) ++pr;
        if (pr == wr.P) {
          what = "pod " + a.name + " missing from the resident window";
          break;
        }
        const PodEntry& b = wr.pods[pr];
        // every fresh row must be found among the resident rows of the same series key (duplicates: any order)
        for (uint32_t sf = 0; what.empty() && sf < a.slots.size(); ++sf) {
          bool found = false;
          for (uint32_t sr = 0; !found && sr < b.slots.size(); ++sr) {
            const size_t row = (size_t)pr * wr.G + sr;
            if (row_used[row] || slot_key(b.slots[sr]) != slot_key(a.slots[sf])) continue;
            if (rows_equal(dev.ring_row(0, (uint32_t)row), wf.util.data() + ((size_t)pf * wf.G + sf) * wf.T)) row_used[row] = 1, found = true;
          }
          if (!found) what = "util row of " + a.name + " gpu " + a.slots[sf].gpu + " differs from a fresh ingest";
        }
        if (what.empty() && a.power_slots) {
          if (!dev.has_ring_power()) what = "no resident power plane";
          // power rows carry no identity beyond the pod: compare as a multiset
          std::vector<uint8_t> used(b.power_slots, 0);
          for (uint32_t sf = 0; what.empty() && sf < a.power_slots; ++sf) {
            bool found = false;
            for (uint32_t sr = 0; !found && sr < b.power_slots; ++sr)
              if (!used[sr] && rows_equal(dev.ring_row(1, pr * wr.G + sr), wf.power.data() + ((size_t)pf * wf.G + sf) * wf.T)) used[sr] = 1, found = true;
            if (!found) what = "power row of " + a.name + " differs from a fresh ingest";
          }
          for (uint32_t sr = 0; what.empty() && sr < b.power_slots; ++sr)
            if (!used[sr] && !row_is_empty(dev.ring_row(1, pr * wr.G + sr))) what = "stale power row in " + a.name;
        }
      }
      // everything else in the ring — aged-out series, pods that left, unused rows — must hold no sample
      for (size_t row = 0; what.empty() && row < row_used.size(); ++row)
        if (!row_used[row] && !row_is_empty(dev.ring_row(0, (uint32_t)row))) what = "stale samples in resident row " + std::to_string(row);
      if (what.empty()) printf("OK tick=%d mode=%s %s\n", k, mode.c_str(), why.c_str());
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
  if (argc == 4 && std::string(argv[1]) == "--ticks") return run_ticks(atoll(argv[2]), argv[3]);
  if (argc < 5) return 2;
  IngestOptions o;
  o.t_end = atoll(argv[1]), o.step = atoll(argv[2]), o.duration_min = atoll(argv[3]);
  int bad = 0;
  for (int i = 4; i < argc; ++i) {
    const std::string dir = argv[i];
    std::string util, prof, power;
    if (!slurp(dir + "/util.json", &util)) {
      printf("MISMATCH %s no util.json\n", dir.c_str());
      ++bad;
      continue;
    }
    const bool has_prof = slurp(dir + "/prof.json", &prof), has_power = slurp(dir + "/power.json", &power);
    // optional: the --power-threshold the power plane is ingested for (its samples are snapped to it)
    std::string thr_text;
    IngestOptions oc = o;
    if (slurp(dir + "/power_threshold", &thr_text)) oc.power_threshold = strtod(thr_text.c_str(), nullptr);
    Window wc, wd;
    bool ok_c = true, ok_d = true;
    std::string err_c, err_d;
    DeviceIngestReport rep;
    EmulDevice dev;
    try {
      wc = ingest_matrix_text(util, has_prof ? &prof : nullptr, has_power ? &power : nullptr, oc, 2);
    } catch (const std::exception& e) {
      ok_c = false, err_c = e.what();
    }
    try {
      wd = ingest_matrix_device(dev, util, has_prof ? &prof : nullptr, has_power ? &power : nullptr, oc, &rep);
    } catch (const std::logic_error& e) {
      printf("MISMATCH %s %s\n", dir.c_str(), e.what());
      ++bad;
      continue;
    } catch (const std::exception& e) {
      ok_d = false, err_d = e.what();
    }
    if (!ok_c || !ok_d) {
      if (ok_c == ok_d) {
        printf("REJECT %s device=%d\n", dir.c_str(), (int)rep.on_device);
      } else {
        printf("MISMATCH %s cpu %s / device %s\n", dir.c_str(), ok_c ? "ok" : err_c.c_str(),
               ok_d ? "ok" : err_d.c_str());
        ++bad;
      }
      continue;
    }
    std::string what;
    if (wc.P != wd.P || wc.G != wd.G || wc.T != wd.T || wc.t_end != wd.t_end || wc.step != wd.step) what = "shape";
    if (what.empty() && wc.pods.size() != wd.pods.size()) what = "pods";
    for (size_t p = 0; what.empty() && p < wc.pods.size(); ++p) {
      const PodEntry &a = wc.pods[p], &b = wd.pods[p];
      if (a.name != b.name || a.ns != b.ns || a.slots.size() != b.slots.size() || a.power_slots != b.power_slots)
        what = "pod " + a.name;
      for (size_t s = 0; what.empty() && s < a.slots.size(); ++s)
        if (a.slots[s].hostname != b.slots[s].hostname || a.slots[s].gpu != b.slots[s].gpu ||
            a.slots[s].container != b.slots[s].container || a.slots[s].model != b.slots[s].model ||
            a.slots[s].node_type != b.slots[s].node_type || a.slots[s].from_prof != b.slots[s].from_prof)
          what = "slot of " + a.name;
    }
    const IngestStats &sa = wc.stats, &sb = wd.stats;
    if (what.empty() && (sa.series_in != sb.series_in || sa.series_skipped != sb.series_skipped ||
                         sa.samples_in != sb.samples_in || sa.samples_out_of_window != sb.samples_out_of_window ||
                         sa.duplicates_merged != sb.duplicates_merged ||
                         sa.tiny_values_clamped != sb.tiny_values_clamped)) {
      char buf[256];
      snprintf(buf, sizeof buf, "stats in %llu/%llu oow %llu/%llu tiny %llu/%llu series %llu/%llu",
               (unsigned long long)sa.samples_in, (unsigned long long)sb.samples_in,
               (unsigned long long)sa.samples_out_of_window, (unsigned long long)sb.samples_out_of_window,
               (unsigned long long)sa.tiny_values_clamped, (unsigned long long)sb.tiny_values_clamped,
               (unsigned long long)sa.series_in, (unsigned long long)sb.series_in);
      what = buf;
    }
    if (what.empty()) {
      const size_t cells = (size_t)wc.P * wc.G * wc.T;
      const float* du = rep.on_device ? wd.d_util : wd.util.data();
      const float* dp = rep.on_device ? wd.d_power : (wd.power.empty() ? nullptr : wd.power.data());
      size_t at = 0;
      const bool bits = true;
      if (cells && !same_plane(wc.util.data(), du, cells, bits, &at)) what = "util cell " + std::to_string(at);
      if (what.empty() && !wc.power.empty() && (!dp || !same_plane(wc.power.data(), dp, cells, bits, &at)))
        what = "power cell " + std::to_string(at);
      if (what.empty() && wc.power.empty() && rep.on_device && wd.d_power) what = "unexpected power plane";
    }
    if (!what.empty()) {
      printf("MISMATCH %s %s\n", dir.c_str(), what.c_str());
      ++bad;
    } else {
      printf("OK %s device=%d spans=%llu hard=%llu patched=%llu %s\n", dir.c_str(), (int)rep.on_device,
             (unsigned long long)rep.spans, (unsigned long long)rep.hard_spans,
             (unsigned long long)rep.rows_patched, rep.reason.c_str());
    }
  }
  return bad ? 1 : 0;
}
