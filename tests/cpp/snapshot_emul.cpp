// TEST INFRASTRUCTURE.  Daemon mode across a restart (--snapshot-file, DESIGN.md §8i) on the EMULATED device of
// tests/cpp/text_emul.cpp (its kernel flavour: k_text_parse's source under tests/cpp/cuda_shim.hpp), extended by the two
// snapshot methods of TextDevice.  These run the SOURCE of the export kernels (gpr_chunks_encode.cuh) and of the chunk
// check and scatter kernels (gpr_chunks.cuh with gpr_samples.cuh), cut out by tests/test_snapshot.py, launched as
// gpr_resident_export and gpr_chunks_scatter launch them.  The emulator's ring is reached through its own interface
// (ring_row, patch_row, resident_init): export encodes the unrolled ring (head 0, which is what the kernels read at any
// head), restore scatters into an unrolled plane and writes it back row by row.
#define main text_emul_main
#include "text_emul.cpp"
#undef main

#include <tuple>

static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) {
  unsigned long long old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (v < old && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_SEQ_CST, __ATOMIC_RELAXED)) {
  }
  return old;
}
namespace gpr {
namespace samples {
#include "samples_extract.inc"
}
namespace chunks {
#include "chunks_extract.inc"
}
namespace chunks_enc {
#include "chunks_export_extract.inc"
}
}  // namespace gpr

#include "snapshot.hpp"

namespace {

class SnapDevice : public EmulDevice {
 public:
  void resident_init(uint32_t pods, uint32_t G, uint32_t T, bool with_power) override {
    EmulDevice::resident_init(pods, G, T, with_power);
    rows_ = pods * G, T_ = T;
  }
  uint32_t ring_rows() const { return rows_; }

  void resident_export(int plane, const TextGrid& grid, ChunkPlaneView* out, double* export_ms, double* copy_ms) override {
    namespace gx = gpr::chunks_enc;
    if (grid.T != T_ || (plane == 1 && !has_ring_power())) throw std::logic_error("emul: export grid does not match the ring");
    std::vector<uint32_t> cells((size_t)rows_ * T_);  // the ring unrolled: oldest bucket first
    for (uint32_t r = 0; r < rows_; ++r) {
      const std::vector<float> row = ring_row(plane, r);
      memcpy(cells.data() + (size_t)r * T_, row.data(), (size_t)T_ * 4);
    }
    gx::ExportArgs a;
    memset(&a, 0, sizeof a);
    a.plane = cells.data(), a.rows = rows_, a.T = T_, a.head = 0, a.per_chunk = 120;
    a.t_end_ms = grid.t_end * 1000, a.step_ms = grid.step * 1000;
    a.max_chunks = (a.T + a.per_chunk - 1) / a.per_chunk;
    std::vector<uint32_t> sizes((size_t)a.rows * a.max_chunks), series((size_t)a.rows + 1);
    std::vector<uint64_t> row_chunks((size_t)a.rows + 1), row_bytes((size_t)a.rows + 1);
    unsigned long long totals[4] = {0, 0, 0, 0};
    a.sizes = sizes.data(), a.row_chunks = row_chunks.data(), a.row_bytes = row_bytes.data();
    a.row_series = series.data(), a.totals = totals;
    const unsigned blocks = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((a.rows + gx::kEncWarps - 1) / gx::kEncWarps, 2));
    launch(blocks, gx::kEncThreads, 0, [&] { gx::k_export_size(a); });
    launch(1, gx::kScanThreads, gx::kScanSmem, [&] { gx::k_export_scan(a); });
    ExportOut& o = xout_[plane];  // exact sizes: a store past one is an AddressSanitizer error
    o.series.assign(totals[2] + 1, ~0ull), o.cbytes.assign(totals[0] + 1, ~0ull);
    o.rows.assign(totals[2], ~0u), o.data.assign(totals[1], 0xA5);
    a.series_chunks = o.series.data(), a.chunk_bytes = o.cbytes.data(), a.out_rows = o.rows.data(), a.data = o.data.data();
    launch(blocks, gx::kEncThreads, 0, [&] { gx::k_export_write(a); });
    out->n_series = totals[2], out->n_chunks = totals[0], out->n_bytes = totals[1];
    out->series_chunks = o.series.data(), out->chunk_bytes = o.cbytes.data(), out->rows = o.rows.data();
    out->data = o.data.data();
    *export_ms = *copy_ms = 0;
  }

  void resident_restore(uint32_t pods, uint32_t G, uint32_t T, bool with_power, const ChunkPlaneView planes[2],
                        const TextGrid& grid) override {
    namespace gc = gpr::chunks;
    namespace gs = gpr::samples;
    resident_init(pods, G, T, with_power);
    if (grid.T != T || grid.n_rows > rows_) throw std::logic_error("emul: restore grid does not match the ring");
    for (int k = 0; k < (with_power ? 2 : 1); ++k) {
      const ChunkPlaneView& v = planes[k];
      const uint32_t S = (uint32_t)v.n_series;
      // as gpr_chunks_scatter: the index arrays, then every chunk, checked before anything is written
      uint32_t bad = 0;
      for (uint32_t s = 0; s < std::max(S, 1u); ++s) bad |= gs::series_faults(v.series_chunks, v.rows, S, s, grid.n_rows);
      if (bad) throw std::runtime_error("gpr_chunks_scatter: emulated: bad series index (" + std::to_string(bad) + ")");
      const uint64_t n_chunks = v.series_chunks[S];
      unsigned int k_bad = 0;
      unsigned long long first = ~0ull, n_in = 0;
      gc::CheckArgs ck;
      ck.chunk_bytes = v.chunk_bytes, ck.data = v.data, ck.data_base = 0, ck.base = 0, ck.end = n_chunks;
      ck.bad = &k_bad, ck.first = &first, ck.n_in = &n_in;
      launch(std::max<unsigned>(1, (unsigned)std::min<uint64_t>((n_chunks + 255) / 256, 2)), 256, 0, [&] { gc::k_chunks_check(ck); });
      if (k_bad)
        throw std::runtime_error("gpr_chunks_scatter: emulated: chunk " + std::to_string(first) + " refused (" +
                                 std::to_string(k_bad) + ")");
      // the scatter into an unrolled plane (newest bucket in column T - 1), then into the ring row by row
      std::vector<uint32_t> cells((size_t)rows_ * T, tx::kFillBits);
      unsigned long long stats[2] = {0, 0};
      gc::ScatterArgs a;
      memset(&a, 0, sizeof a);
      a.g.t_end = grid.t_end * 1000, a.g.t_lo = (grid.t_end - grid.span) * 1000, a.g.step = (uint32_t)(grid.step * 1000);
      a.g.T = T, a.g.ld = T, a.g.col_end = T - 1;
      a.g.power = tx::power_snap(k == 1 ? grid.power_threshold : 0.0);
      a.series_chunks = v.series_chunks, a.rows = v.rows, a.chunk_bytes = v.chunk_bytes, a.data = v.data;
      a.data_base = 0, a.base = 0, a.end = n_chunks, a.s_base = 0, a.n_series = S;
      a.plane = reinterpret_cast<float*>(cells.data()), a.stats = stats;
      if (n_chunks) {
        const uint64_t groups = (n_chunks + 31) / 32;
        launch((unsigned)std::max<uint64_t>(1, std::min<uint64_t>((groups + gc::kWarps - 1) / gc::kWarps, 2)), gc::kThreads, 0,
               [&] { gc::k_chunks_scatter(a); });
      }
      for (uint32_t r = 0; r < rows_; ++r)
        patch_row(k, r, T, reinterpret_cast<const float*>(cells.data() + (size_t)r * T), T, true);
    }
  }

 private:
  uint32_t rows_ = 0, T_ = 0;
  struct ExportOut {
    std::vector<uint64_t> series, cbytes;
    std::vector<uint32_t> rows;
    std::vector<uint8_t> data;
  } xout_[2];
};

// what a tick fetched and ingested: mode "full" / "delta" / "failed" (why: the reason), wr the session's window, wf a
// fresh full-range ingest of the same tick on the CPU (the reference)
struct TickOut {
  std::string mode = "full", why;
  Window wr, wf;
};
// false = no such tick.  Throws what the ingest throws on a full range.
bool ingest_tick(DeviceIngestSession& session, int64_t duration_min, const std::string& dir, int k, TickOut* out) {
  char name[32];
  snprintf(name, sizeof name, "/tick-%04d", k);
  const std::string base = dir + name;
  if (!file_there(base + "/full/util.json")) return false;
  auto load = [&](const std::string& d, std::string* util, std::string* prof, std::string* power, bool* hp, bool* hw,
                  IngestOptions* o) {
    slurp(d + "/util.json", util);
    *hp = slurp(d + "/prof.json", prof), *hw = slurp(d + "/power.json", power);
    const Json meta = Json::parse_file(d + "/query.json");
    o->duration_min = duration_min;
    o->t_end = (int64_t)meta["end"].as_number(0), o->step = (int64_t)meta["step"].as_number(0);
    return (int64_t)meta["start"].as_number(0);
  };
  std::string util, prof, power;
  bool hp = false, hw = false;
  IngestOptions o;
  bool done = false;
  TickOut& t = *out;
  t = TickOut();
  const int64_t since = session.resident_t_end();
  if (since > 0 && file_there(base + "/delta/util.json")) {
    const int64_t start = load(base + "/delta", &util, &prof, &power, &hp, &hw, &o);
    if (start == since) {
      o.slice_seconds = o.t_end - start, o.resident = true;
      try {
        t.wr = session.ingest(util, hp ? &prof : nullptr, hw ? &power : nullptr, o);
        t.mode = "delta", done = true;
      } catch (const NeedFullWindow& e) {
        t.why = e.what();
      } catch (const std::runtime_error& e) {
        // the tick fails (the controller logs "Failed to run query!" and waits for the next one)
        t.mode = "failed", t.why = e.what();
        return true;
      }
    } else {
      t.why = "delta does not continue the resident window";
    }
  }
  load(base + "/full", &util, &prof, &power, &hp, &hw, &o);
  o.slice_seconds = 0, o.resident = true;
  if (!done) t.wr = session.ingest(util, hp ? &prof : nullptr, hw ? &power : nullptr, o);
  IngestOptions of = o;
  of.resident = false;
  t.wf = ingest_matrix_text(util, hp ? &prof : nullptr, hw ? &power : nullptr, of, 2);
  return true;
}

// "" = the resident ring holds exactly the window a fresh full-range ingest of the tick yields: same samples for every
// series of every pod, nothing but "no sample" anywhere else
std::string fresh_mismatch(const SnapDevice& dev, const Window& wr, const Window& wf) {
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
  return what;
}

// ---- daemon mode across a restart: snapshots -------------------------------------------------------------------------
//   snapshot_emul --save   <duration_min> <dir> <k> <snapshot> <key.json>   ticks 0..k-1, then the snapshot
//   snapshot_emul --resume <duration_min> <dir> <k> <snapshot> <key.json>   an uninterrupted session U over every tick, and a
//                                                                        fresh device + session B restored from the
//                                                                        snapshot over ticks k..
// key.json: {"span": s, "power_threshold": x, "selectors": [util, prof, power]} — the key of the run (SnapshotKey).
// --save prints the ticks as --ticks does, then  SAVED bytes=<n>  |  NOSAVE <why>.
// --resume prints  RESTORE ok  |  RESTORE refused <why>,  then per tick  OK tick=<k> mode=<B's> umode=<U's> [why]  |
// MISMATCH tick=<k> <what>.  Every tick of B must hold the window of a fresh full-range ingest; after a restore B must
// also take the same path as U, hold U's ring (unrolled, bit for bit; every NaN is "no sample") and U's session (pods,
// slots, known series with their (pod, slot, result), power keys, PROF signatures and rows).
SnapshotKey read_key(const std::string& path) {
  const Json j = Json::parse_file(path);
  SnapshotKey key;
  key.span = (int64_t)j["span"].as_number(0);
  key.power_threshold = j["power_threshold"].as_number(0);
  for (int i = 0; i < 3; ++i) key.selectors[i] = j["selectors"][i].as_string();
  return key;
}

std::string ring_mismatch(const SnapDevice& a, const SnapDevice& b) {
  if (a.ring_rows() != b.ring_rows() || a.has_ring_power() != b.has_ring_power()) return "ring shape";
  for (int plane = 0; plane < (a.has_ring_power() ? 2 : 1); ++plane)
    for (uint32_t r = 0; r < a.ring_rows(); ++r) {
      const std::vector<float> x = a.ring_row(plane, r), y = b.ring_row(plane, r);
      for (size_t c = 0; c < x.size(); ++c)
        if (!(std::isnan(x[c]) && std::isnan(y[c])) && memcmp(&x[c], &y[c], 4) != 0)
          return "ring plane " + std::to_string(plane) + " row " + std::to_string(r) + " differs from the uninterrupted one";
    }
  return "";
}

std::string state_mismatch(const DeviceIngestSession& u, const DeviceIngestSession& b) {
  SnapshotState x, y;
  const bool hx = u.save_state(&x), hy = b.save_state(&y);
  if (hx != hy) return "one session holds a window, the other not";
  if (!hx) return "";
  if (x.span != y.span || x.step != y.step || x.t_end != y.t_end || x.T != y.T || x.pods_cap != y.pods_cap || x.G != y.G ||
      x.with_power != y.with_power || memcmp(&x.power_threshold, &y.power_threshold, 8) != 0)
    return "session shape";
  if (x.pods.size() != y.pods.size()) return "pods";
  for (size_t p = 0; p < x.pods.size(); ++p) {
    const PodEntry &a = x.pods[p], &c = y.pods[p];
    if (a.name != c.name || a.ns != c.ns || a.power_slots != c.power_slots || a.has_groups != c.has_groups ||
        a.slots.size() != c.slots.size())
      return "pod " + a.name;
    for (size_t g = 0; g < a.slots.size(); ++g)
      if (slot_key(a.slots[g]) != slot_key(c.slots[g]) || a.slots[g].group != c.slots[g].group ||
          a.slots[g].node_type != c.slots[g].node_type)
        return "slot of " + a.name;
  }
  auto key = [](const SnapshotState::Known& k) { return std::make_tuple(k.h1, k.h2, k.result, k.pod, k.slot); };
  auto sorted = [&](std::vector<SnapshotState::Known> v) {
    std::sort(v.begin(), v.end(), [&](const SnapshotState::Known& l, const SnapshotState::Known& r) { return key(l) < key(r); });
    std::vector<decltype(key(v[0]))> out;
    for (const auto& k : v) out.push_back(key(k));
    return out;
  };
  if (x.known.size() != y.known.size() || sorted(x.known) != sorted(y.known)) return "known series";
  if (x.power_keys != y.power_keys) return "power keys";
  if (x.prof_sigs != y.prof_sigs) return "PROF signatures";
  if (x.prof_rows != y.prof_rows) return "PROF rows";
  return "";
}

int run_save(int64_t duration_min, const std::string& dir, int k_cut, const std::string& snap, const SnapshotKey& key) {
  SnapDevice dev;
  DeviceIngestSession session(dev);
  int bad = 0;
  for (int k = 0; k < k_cut; ++k) {
    TickOut t;
    try {
      if (!ingest_tick(session, duration_min, dir, k, &t)) break;
      const std::string what = t.mode == "failed" ? "" : fresh_mismatch(dev, t.wr, t.wf);
      if (what.empty()) printf("OK tick=%d mode=%s %s\n", k, t.mode.c_str(), t.why.c_str());
      else printf("MISMATCH tick=%d %s\n", k, what.c_str()), ++bad;
    } catch (const std::exception& e) {
      printf("MISMATCH tick=%d exception %s\n", k, e.what());
      ++bad;
    }
  }
  SnapshotTimes st;
  std::string err;
  if (save_snapshot(session, key, snap, &st, &err)) printf("SAVED bytes=%llu\n", (unsigned long long)st.bytes);
  else printf("NOSAVE %s\n", err.empty() ? "nothing resident" : err.c_str()), ++bad;
  return bad ? 1 : 0;
}

int run_resume(int64_t duration_min, const std::string& dir, int k_cut, const std::string& snap, const SnapshotKey& key) {
  SnapDevice du, db;
  DeviceIngestSession u(du), b(db);
  int bad = 0;
  SnapshotTimes st;
  std::string why;
  const bool restored = restore_snapshot(b, key, snap, &st, &why);
  if (restored) printf("RESTORE ok\n");
  else printf("RESTORE refused %s\n", why.c_str());
  if (!restored && b.resident_t_end() != 0) printf("MISMATCH tick=%d a refused restore left a resident window\n", k_cut), ++bad;
  for (int k = 0;; ++k) {
    TickOut tu, tb;
    try {
      if (!ingest_tick(u, duration_min, dir, k, &tu)) break;
      if (k < k_cut) continue;
      if (!ingest_tick(b, duration_min, dir, k, &tb)) break;
      std::string what = tb.mode == "failed" ? "B's tick failed: " + tb.why : fresh_mismatch(db, tb.wr, tb.wf);
      if (what.empty() && restored) {
        if (tb.mode != tu.mode) what = "B took the " + tb.mode + " path, U the " + tu.mode + " path";
        if (what.empty()) what = ring_mismatch(du, db);
        if (what.empty()) what = state_mismatch(u, b);
      }
      if (what.empty()) printf("OK tick=%d mode=%s umode=%s %s\n", k, tb.mode.c_str(), tu.mode.c_str(), tb.why.c_str());
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
  if (argc == 7 && std::string(argv[1]) == "--save") return run_save(atoll(argv[2]), argv[3], atoi(argv[4]), argv[5], read_key(argv[6]));
  if (argc == 7 && std::string(argv[1]) == "--resume")
    return run_resume(atoll(argv[2]), argv[3], atoi(argv[4]), argv[5], read_key(argv[6]));
  return 2;
}
