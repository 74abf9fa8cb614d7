// ingest_device.cpp — host half of the device-side ingest (see ingest_device.hpp and
// gpu-pruner_b200/csrc/gpr_text.cuh).  The wire shape is the matrix result that
// gpu-pruner/src/bin/querytest.rs:41-53 walks; label precedence and defaults follow
// PodMetricData::try_from (gpu-pruner/src/lib.rs:153-187) through the Assigner shared with ingest.cpp.
// The device reports where sample lists open and close; this file walks the series with those offsets,
// turns every label map into a tensor row, lets the device parse the samples, and re-parses on the CPU
// the few rows the strict device parser declined.
#include "ingest_device.hpp"

#include <algorithm>
#include <chrono>
#include <cstring>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>

#include "../csrc/gpr_retime.h"
#include "ingest_internal.hpp"

namespace gph {

using namespace detail;

namespace {

struct NotCompact {  // the response is not in the one encoding the device scan understands
  std::string why;
};

struct DevSeries {
  uint32_t pod, slot;
  uint64_t begin, end;  // gpr_text_span.begin / .end
};

struct TextPlan {
  int slot = 0;                    // resident text slot on the device
  const std::string* text = nullptr;
  std::vector<DevSeries> series;   // placed series, in text order
};

const char kHead[] = "{\"status\":\"success\",\"data\":{\"resultType\":\"matrix\",\"result\":[";
const char kMetric[] = "{\"metric\":";

bool starts_with(const std::string& s, size_t at, const char* lit) {
  const size_t n = strlen(lit);
  return at + n <= s.size() && memcmp(s.data() + at, lit, n) == 0;
}

size_t skip_trailing_ws(const std::string& s, size_t at) {
  while (at < s.size() && (s[at] == ' ' || s[at] == '\n' || s[at] == '\r' || s[at] == '\t')) ++at;
  return at;
}

double ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

struct SeriesLoc {
  size_t mb, close_brace, vb, list_close;  // label map [mb, close_brace], list [vb, list_close]
};

// A few worker threads for the per-series label work (parse the label map, hash it, probe the table of known
// series): independent per series, and on the critical path of a tick while the text is crossing PCIe.
class Workers {
 public:
  explicit Workers(int n) : n_(std::max(1, n)) {
    for (int i = 1; i < n_; ++i) th_.emplace_back([this, i] { loop(i); });
  }
  ~Workers() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      quit_ = true;
    }
    cv_.notify_all();
    for (std::thread& t : th_) t.join();
  }
  // fn(begin, end) over [0, n) in contiguous shares; returns when all shares are done.  Exceptions are carried over.
  void run(size_t n, const std::function<void(size_t, size_t)>& fn) {
    if (n_ == 1 || n < 256) {
      fn(0, n);
      return;
    }
    {
      std::lock_guard<std::mutex> lk(mu_);
      fn_ = &fn, total_ = n, pending_ = n_ - 1, ++gen_, error_.clear();
    }
    cv_.notify_all();
    share(0);
    std::unique_lock<std::mutex> lk(mu_);
    done_.wait(lk, [this] { return pending_ == 0; });
    fn_ = nullptr;
    if (!error_.empty()) throw std::runtime_error(error_);
  }

 private:
  void share(int i) {
    const size_t b = total_ * (size_t)i / (size_t)n_, e = total_ * (size_t)(i + 1) / (size_t)n_;
    try {
      if (b < e) (*fn_)(b, e);
    } catch (const std::exception& ex) {
      std::lock_guard<std::mutex> lk(mu_);
      error_ = ex.what();
    }
  }
  void loop(int i) {
    unsigned long seen = 0;
    std::unique_lock<std::mutex> lk(mu_);
    while (true) {
      cv_.wait(lk, [&] { return quit_ || gen_ != seen; });
      if (quit_) return;
      seen = gen_;
      lk.unlock();
      share(i);
      lk.lock();
      if (--pending_ == 0) done_.notify_one();
    }
  }
  int n_;
  std::vector<std::thread> th_;
  std::mutex mu_;
  std::condition_variable cv_, done_;
  const std::function<void(size_t, size_t)>* fn_ = nullptr;
  size_t total_ = 0;
  int pending_ = 0;
  unsigned long gen_ = 0;
  bool quit_ = false;
  std::string error_;
};

Workers& label_workers() {
  static Workers w([] {
    const char* v = getenv("GPR_LABEL_THREADS");
    const int n = v && *v ? atoi(v) : (int)std::min(16u, std::max(1u, std::thread::hardware_concurrency() / 2));
    return std::max(1, std::min(64, n));
  }());
  return w;
}

// [[ts,"v"],[ts,"v"],...] exactly as Prometheus prints it: digits with an optional fraction, a quoted number
// (strict_sample_value), no white space.  (Anything else is for the CPU parser to judge.)
bool samples_are_compact(const char* p, const char* e) {
  if (p >= e || *p++ != '[') return false;
  if (p < e && *p == ']') return p + 1 == e;
  while (true) {
    if (p >= e || *p++ != '[') return false;
    const char* d = p;
    while (p < e && *p >= '0' && *p <= '9') ++p;
    if (p == d) return false;
    if (p < e && *p == '.') {
      d = ++p;
      while (p < e && *p >= '0' && *p <= '9') ++p;
      if (p == d) return false;
    }
    if (e - p < 2 || p[0] != ',' || p[1] != '"') return false;
    p += 2;
    d = p;
    while (p < e && *p != '"') ++p;
    double v;
    if (e - p < 2 || p[1] != ']' || !detail::strict_sample_value(d, p, &v)) return false;
    p += 2;
    if (p >= e) return false;
    if (*p == ']') return p + 1 == e;
    if (*p++ != ',') return false;
  }
}

// Walk the series of one response with the device's marker lists, as they arrive: the upload + scan runs as a
// pipeline (TextDevice::scan_begin / scan_next).  Every batch of series whose markers are in goes through three steps
// while later chunks of the text are still on their way to the GPU:
//   walk    (this thread, markers only)   series i <-> i-th `},"values":[`; its list ends at the first `"]]` behind
//                                         it, or is empty when that lies beyond the next series' marker
//   labels  (worker threads, per series)  check the framing bytes around the markers, then either recognise the
//                                         series by the hash of its label bytes (daemon mode) or parse the label
//                                         map in place and pull out the six labels the assignment needs
//   assign  (this thread, in text order)  label set -> (pod, slot) through `asg`
void plan_text(TextDevice& dev, TextPlan& plan, Assigner& asg, Window& w, bool is_power, bool is_prof,
               DeviceIngestReport& rep, bool remember) {
  const std::string& t = *plan.text;
  size_t at0;
  bool bare;
  if (starts_with(t, 0, kHead)) at0 = sizeof kHead - 1, bare = false;
  else if (starts_with(t, 0, "[")) at0 = 1, bare = true;
  else throw NotCompact{"response does not start with the compact success/matrix header"};

  struct Loc {
    size_t at, close_brace, list_close;  // series object starts at `at`; '}' of the label map; ']' closing the list
    bool empty;                          // "values":[]
  };
  struct Rec {
    const char* err = nullptr;  // framing violation (a string literal)
    bool known = false, flat = false;
    Assigner::Result r = Assigner::Skipped;
    uint32_t pod = 0, slot = 0;
    uint64_t h1 = 0, h2 = 0;
    LabelFields f;
  };
  std::vector<uint64_t> opens, closes, co, cc;  // all markers so far (sorted: chunks come in text order)
  std::vector<Loc> locs;
  std::vector<Rec> recs;
  size_t oi = 0, ci = 0;     // next series' open marker; cursor into closes
  size_t at = at0;           // where the next series object starts
  const size_t kM = sizeof kMetric - 1;

  // consume every series that is completely covered by the markers delivered so far
  auto drain = [&](bool final) {
    // ---- walk: markers only ----------------------------------------------------------------------------------------
    const auto tw = std::chrono::steady_clock::now();
    locs.clear();
    while (oi < opens.size()) {
      if (!final && oi + 1 >= opens.size()) break;  // emptiness of list i is decided by where series i + 1 begins
      const size_t close_brace = (size_t)opens[oi], vb = close_brace + 12;
      if (close_brace < at + kM) throw NotCompact{"values marker inside the framing of a series"};
      while (ci < closes.size() && closes[ci] < vb) ++ci;
      const uint64_t next_open = oi + 1 < opens.size() ? opens[oi + 1] : (uint64_t)t.size();
      Loc l;
      l.at = at, l.close_brace = close_brace;
      l.empty = ci == closes.size() || closes[ci] > next_open;
      l.list_close = l.empty ? vb : (size_t)closes[ci] + 2;
      if (l.list_close + 3 > t.size()) throw NotCompact{"truncated values list"};
      locs.push_back(l);
      at = l.list_close + 3;  // past `]},`
      ++oi;
    }
    // ---- labels: per series, in parallel --------------------------------------------------------------------------
    recs.resize(locs.size());  // (every worker resets the records of its share)
    label_workers().run(locs.size(), [&](size_t b, size_t e) {
      FlatLabels flat;
      for (size_t i = b; i < e; ++i) {
        const Loc& l = locs[i];
        Rec& r = recs[i];
        r = Rec();
        const size_t mb = l.at + kM, vb = l.close_brace + 12;
        if (!starts_with(t, l.at, kMetric) || t[mb] != '{') r.err = "series does not start with {\"metric\":{";
        else if (t[vb] != (l.empty ? ']' : '[')) r.err = l.empty ? "unterminated values list" : "values list does not start with a sample";
        else if (t[l.list_close + 1] != '}') r.err = "series object has members after \"values\"";
        if (r.err) continue;
        const char* lb = t.data() + mb;
        const char* le = t.data() + l.close_brace + 1;
        if (remember && !l.empty) {
          Assigner::series_identity(std::string_view(lb, (size_t)(le - lb)), is_power, is_prof, &r.h1, &r.h2);
          r.known = asg.find_known(r.h1, r.h2, &r.r, &r.pod, &r.slot);
          if (r.known) continue;  // same bytes as in an earlier tick: validated then, same row now
        }
        // The label map is parsed for EVERY series (also the ones whose list is empty): a complete JSON object ending
        // exactly at the marker's '}' proves that [mb, close_brace] is the whole map and that no series without a
        // "values" member was jumped over.  (A `},"values":[` inside a label value is impossible: a raw '"' ends a
        // JSON string.)  Prometheus' own shape — string values, no escapes — is read in place without allocating.
        r.flat = flat.parse(lb, le);
        if (r.flat && !l.empty) r.f = extract_fields(flat);
      }
    });
    rep.labels_ms += ms_since(tw);  // walk + parallel label phase
    // ---- assign: in text order ----------------------------------------------------------------------------------------
    const auto ta = std::chrono::steady_clock::now();
    FlatLabels flat;
    for (size_t i = 0; i < locs.size(); ++i) {
      const Loc& l = locs[i];
      Rec& r = recs[i];
      if (r.err) throw NotCompact{r.err};
      // between series exactly one ',' ; the last one is followed by the ']' of the result array
      const char sep = t[l.list_close + 2];
      const bool last = final && oi == opens.size() && i + 1 == locs.size();
      if (sep != (last ? ']' : ',')) throw NotCompact{"expected ',' or ']' after a series"};
      ++w.stats.series_in;
      if (l.empty) {
        if (!r.flat) {  // still has to be a label map
          try {
            if (!Json::parse(std::string(t.data() + l.at + kM, t.data() + l.close_brace + 1)).is_object())
              throw NotCompact{"label map is not an object"};
          } catch (const std::exception& ex) {
            throw NotCompact{std::string("label map: ") + ex.what()};
          }
        }
        continue;  // an empty list is no element (as in the CPU paths)
      }
      const char* lb = t.data() + l.at + kM;
      const char* le = t.data() + l.close_brace + 1;
      if (r.known) {
        if (r.r == Assigner::Skipped) asg.count_skipped();
      } else if (r.flat) {
        r.r = asg.assign_fields(r.f, is_power, is_prof, [&]() {
          flat.parse(lb, le);
          return label_signature(flat);
        }, &r.pod, &r.slot);
        if (remember) asg.insert_known(r.h1, r.h2, r.r, r.pod, r.slot);
      } else {
        Json metric;
        try {
          metric = Json::parse(std::string(lb, le));
        } catch (const std::exception& ex) {
          throw NotCompact{std::string("label map: ") + ex.what()};
        }
        if (!metric.is_object()) throw NotCompact{"label map is not an object"};
        r.r = asg.assign(metric, is_power, is_prof, &r.pod, &r.slot);
        if (remember) asg.insert_known(r.h1, r.h2, r.r, r.pod, r.slot);
      }
      if (r.r == Assigner::Placed)
        plan.series.push_back(DevSeries{r.pod, r.slot, (uint64_t)l.close_brace + 12, (uint64_t)l.list_close});
      // A series that gets no row (no workload-pod label, lib.rs:161-175) is never seen by the device parser, so its
      // samples are checked here: a response that is malformed there is malformed, and the CPU parser — which reads
      // every sample — has to be the one to say so.  Such series are rare by construction (the selector asks for a
      // non-empty pod label).  Series shadowed by a PROF series of the same label set are NOT walked: there can be as
      // many of them as there are series, and nothing in them can reach the verdict.
      else if (r.r == Assigner::Skipped && !samples_are_compact(t.data() + l.close_brace + 11, t.data() + l.list_close + 1))
        throw NotCompact{"values list of a skipped series is not in the compact encoding"};
    }
    rep.assign_ms += ms_since(ta);
  };

  auto t0 = std::chrono::steady_clock::now();
  dev.scan_begin(plan.slot, t.data(), t.size());
  bool more = true;
  try {
    while (more) {
      uint64_t ready = 0;
      more = dev.scan_next(&co, &cc, &ready);
      rep.scan_ms += ms_since(t0);  // time spent waiting for the upload / scan
      t0 = std::chrono::steady_clock::now();
      opens.insert(opens.end(), co.begin(), co.end());
      closes.insert(closes.end(), cc.begin(), cc.end());
      // batches of a few thousand series keep the workers' hand-over cost negligible
      if (!more || opens.size() - oi >= 4096) drain(!more);  // (timed inside: labels_ms / assign_ms)
      t0 = std::chrono::steady_clock::now();
    }
  } catch (...) {
    while (more) {  // let the pipeline run to its end: the device slot must not be left half written
      uint64_t ready = 0;
      try {
        more = dev.scan_next(&co, &cc, &ready);
      } catch (...) {
        break;
      }
    }
    throw;
  }
  // the result array closes right behind the last series (or at once when there is none)
  if (opens.empty()) {
    if (at0 >= t.size() || t[at0] != ']') throw NotCompact{"label map without a following \"values\" list"};
    at = at0 + 1;
  }
  if (!bare) {
    if (!starts_with(t, at, "}}")) throw NotCompact{"response has members after \"result\""};
    at += 2;
  }
  if (skip_trailing_ws(t, at) != t.size()) throw NotCompact{"trailing bytes after the response"};
}

// IngestOptions::reshape: a delta tick whose pods outgrew the ring's rows (`pods_cap`) or whose pod gained a slot
// beyond w.G.  The tick's buckets are open already (resident_advance), so a pod whose last sample aged out with this
// tick has no live row.  Kept: every pod with a live row in either plane, or with a series in this tick's slice; the
// others are dropped.  The new shape applies the full rebuild's head-room rule to the kept pods, and G never shrinks:
// [kept + kept / 4 + 64][max(G, slots needed)].  Kept pod `slot` moves to `slot'` with its rows
// (src_rows[slot' * G' + g] = slot * G + g), a pod that joined this tick starts without a sample.  Then everything
// that names a pod or a row is renumbered: the pods, the Assigner (pod table, known series, power keys, PROF
// signatures), the session's PROF rows and this tick's series.  Returns the log line.
std::string reshape_ring(TextDevice& dev, Window& w, Assigner& asg, uint32_t* pods_cap,
                         std::vector<std::pair<uint32_t, uint32_t>>* prof_rows, TextPlan* plans, int n_plans) {
  const uint32_t P_old = *pods_cap, G_old = w.G, n_pods = (uint32_t)w.pods.size();
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<uint32_t> bits;
  dev.resident_live_rows(&bits);
  const double live_ms = ms_since(t0);
  if (bits.size() < ((size_t)P_old * G_old + 31) / 32) throw std::logic_error("live-row bitmap shorter than the ring");
  std::vector<uint8_t> keep(n_pods, 0);
  for (uint32_t p = 0; p < std::min(n_pods, P_old); ++p)
    for (uint32_t g = 0; g < G_old && !keep[p]; ++g) {
      const size_t r = (size_t)p * G_old + g;
      keep[p] = (uint8_t)((bits[r >> 5] >> (r & 31)) & 1u);
    }
  for (int k = 0; k < n_plans; ++k)
    for (const DevSeries& s : plans[k].series) keep[s.pod] = 1;
  std::vector<uint32_t> to(n_pods, Assigner::kDropped);
  uint32_t kept = 0, G_new = G_old;
  const PodList& pods = w.pods;
  for (uint32_t p = 0; p < n_pods; ++p) {
    if (!keep[p]) continue;
    to[p] = kept++;
    G_new = std::max<uint32_t>(G_new, std::max<uint32_t>((uint32_t)pods[p].slots.size(), pods[p].power_slots));
  }
  const uint32_t P_new = kept + kept / 4 + 64;
  std::vector<uint32_t> src((size_t)P_new * G_new, GPR_ROW_NONE);
  for (uint32_t p = 0; p < std::min(n_pods, P_old); ++p)
    if (keep[p])
      for (uint32_t g = 0; g < G_old; ++g) src[(size_t)to[p] * G_new + g] = p * G_old + g;
  const auto t1 = std::chrono::steady_clock::now();
  dev.resident_remap(P_new, G_new, src);
  const double remap_ms = ms_since(t1);
  asg.renumber_pods(to);
  w.G = G_new, *pods_cap = P_new;
  // the session's PROF rows equal this tick's (the delta check), so they belong to kept pods
  for (auto& r : *prof_rows) r.first = to[r.first];
  std::sort(prof_rows->begin(), prof_rows->end());
  for (int k = 0; k < n_plans; ++k)
    for (DevSeries& s : plans[k].series) s.pod = to[s.pod];
  char line[200];
  snprintf(line, sizeof line,
           "Resident window reshaped on the GPU: %u -> %u, %u -> %u, %u pods dropped (live rows %.2f ms, remap %.2f ms)",
           P_old, P_new, G_old, G_new, n_pods - kept, live_ms, remap_ms);
  return line;
}

// IngestOptions::reask_seconds: the ring's re-asked buckets as they were before the tick's merge — the n_re buckets that
// end n_new (the buckets this tick opens) before the newest — per resident plane, read once the ring's shape for the
// tick is known.  A row is found by (pod, slot): a ring that grows on the way keeps every pod's number, and a row it
// did not have when the band was read holds no sample.
struct ReaskBand {
  uint32_t n_new = 0, n_re = 0, G = 0, rows = 0;
  std::vector<float> before[2];

  // cell of ring row r (of a ring with G_now slots per pod) `back` buckets before the newest, before the merge
  float cell(int plane, uint32_t r, uint32_t G_now, uint32_t back) const {
    const uint32_t pod = r / G_now, slot = r % G_now;
    const size_t row = (size_t)pod * G + slot;
    if (slot >= G || row >= rows) return std::numeric_limits<float>::quiet_NaN();
    return before[plane][row * n_re + (n_new + n_re - 1 - back)];
  }
  bool covers(uint32_t back) const { return back >= n_new && back < n_new + n_re; }
};

void read_band(TextDevice& dev, ReaskBand* band, uint32_t G, int n_planes, IngestStats& st) {
  const auto t0 = std::chrono::steady_clock::now();
  band->G = G;
  for (int k = 0; k < n_planes; ++k) dev.resident_cols(k, band->n_new, band->n_re, &band->before[k]);
  band->rows = (uint32_t)(band->before[0].size() / band->n_re);
  st.band_ms += ms_since(t0);
}

// After the tick's last merge: the cells of the re-asked buckets whose bits changed, per plane — what late samples
// raised.  (A max never lowers a cell, so every change is a raise.)  Only the rows of the window's pods are compared:
// the ring's head-room rows have no series.  A row the band did not have when it was read (the ring grew) had no
// sample there.
void count_late(TextDevice& dev, const ReaskBand& band, uint32_t n_pods, uint32_t G_now, int n_planes, IngestStats& st) {
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<float> after;
  const uint32_t n_re = band.n_re;
  for (int k = 0; k < n_planes; ++k) {
    dev.resident_cols(k, band.n_new, n_re, &after);
    uint64_t n = 0;
    const size_t rows = std::min<size_t>(after.size() / n_re, (size_t)n_pods * G_now);
    for (size_t r = 0; r < rows; ++r) {
      const uint32_t pod = (uint32_t)(r / G_now), slot = (uint32_t)(r % G_now);
      const size_t old = (size_t)pod * band.G + slot;
      const bool had = slot < band.G && old < band.rows;
      const float* now = after.data() + r * n_re;
      const float* was = had ? band.before[k].data() + old * n_re : nullptr;
      for (uint32_t j = 0; j < n_re; ++j) {
        const bool now_nan = std::isnan(now[j]), was_nan = !was || std::isnan(was[j]);
        n += !(now_nan && was_nan) && (now_nan != was_nan || memcmp(&was[j], &now[j], sizeof(float)) != 0);
      }
    }
    (k == 0 ? st.late_util_cells : st.late_power_cells) += n;
  }
  st.band_ms += ms_since(t0);
}

// Parses the series of `texts` into plane `plane` (0 util, 1 power) on `grid` (its fill applies to the first text only),
// then re-parses on the CPU every series feeding a row the device gave up on and writes back that row's buckets of
// `patch`: a run of patch.T buckets ending at patch.t_end, `newer` buckets before the grid's newest one.  Buckets that
// `band` covers were asked again (IngestOptions::reask_seconds): there the re-parse is merged with what the ring held
// before the tick (NaN-aware max) instead of overwriting it, so re-asking never lowers a cell.
void parse_plane(TextDevice& dev, Window& w, const std::vector<TextPlan*>& texts, int plane, TextDevice::TextGrid grid,
                 const Window& patch, uint32_t newer, double power_threshold, DeviceIngestReport& rep,
                 const ReaskBand* band = nullptr) {
  const uint32_t n_rows = grid.n_rows;
  grid.power_threshold = plane == 1 ? power_threshold : 0.0;
  std::vector<uint32_t> writers(n_rows, 0);
  for (TextPlan* tp : texts)
    for (const DevSeries& s : tp->series) ++writers[(size_t)s.pod * w.G + s.slot];
  std::vector<std::vector<gpr_text_span>> spans(texts.size());
  for (size_t k = 0; k < texts.size(); ++k) {
    for (const DevSeries& s : texts[k]->series) {
      gpr_text_span sp;
      memset(&sp, 0, sizeof sp);
      sp.begin = s.begin, sp.end = s.end, sp.row = s.pod * w.G + s.slot;
      sp.flags = writers[sp.row] > 1 ? GPR_SPAN_SHARED : 0u;
      spans[k].push_back(sp);
    }
    const auto tp = std::chrono::steady_clock::now();
    dev.parse(texts[k]->slot, spans[k], grid, plane);
    rep.parse_ms += ms_since(tp);
    grid.fill = false;
    rep.spans += spans[k].size();
  }
  // rows the device gave up on: re-parse every series feeding them with the CPU walker
  std::vector<uint8_t> dirty(n_rows, 0);
  bool any_dirty = false;
  for (const auto& list : spans)
    for (const gpr_text_span& sp : list)
      if (sp.flags & GPR_SPAN_HARD) dirty[sp.row] = 1, any_dirty = true, ++rep.hard_spans;
  std::vector<std::vector<float>> rows;
  std::vector<uint32_t> row_ids;
  std::vector<int64_t> row_slot(any_dirty ? n_rows : 0, -1);
  const gpr::text::PowerSnap snap = gpr::text::power_snap(plane == 1 ? power_threshold : 0.0);
  // a bucket without a sample is written back as the fill, the one NaN the device merge raises: a re-asked bucket
  // (IngestOptions::reask_seconds) may be merged into again by a later tick, and any other NaN would hold off its
  // samples for good (atomic_merge is an integer max for non-negative values)
  float no_sample;
  memcpy(&no_sample, &gpr::text::kFillBits, sizeof no_sample);
  for (size_t k = 0; k < texts.size(); ++k) {
    const std::string& t = *texts[k]->text;
    for (const gpr_text_span& sp : spans[k]) {
      if (!dirty[sp.row]) {
        w.stats.samples_in += sp.n_in;
        w.stats.samples_out_of_window += sp.n_oow;
        w.stats.tiny_values_clamped += sp.n_tiny;
        continue;
      }
      if (row_slot[sp.row] < 0) {
        row_slot[sp.row] = (int64_t)rows.size();
        rows.emplace_back(patch.T, no_sample);
        row_ids.push_back(sp.row);
      }
      float* row = rows[(size_t)row_slot[sp.row]].data();
      for_each_sample(t.data() + sp.begin - 1, t.data() + sp.end + 1, [&](double ts, double v) {
        ++w.stats.samples_in;
        const int64_t col = column_of(patch, ts_millis(ts));
        if (col < 0) {
          ++w.stats.samples_out_of_window;
          return;
        }
        merge_cell(row[col], to_cell(v, snap, &w.stats.tiny_values_clamped));
      });
    }
  }
  if (band)
    for (size_t i = 0; i < rows.size(); ++i)
      for (uint32_t c = 0; c < patch.T; ++c) {
        const uint32_t back = newer + patch.T - 1 - c;
        if (band->covers(back)) merge_cell(rows[i][c], band->cell(plane, row_ids[i], w.G, back));
      }
  for (size_t i = 0; i < rows.size(); ++i)
    dev.patch_cols(plane, row_ids[i], w.T, rows[i].data(), patch.T, newer, grid.resident);
  rep.rows_patched += rows.size();
}

constexpr const char* kGridChanged = "step / window length changed";

// The first failing check of a delta tick against the resident window (nullptr: the ring can take the tick): same
// grid (unless `grid` is false: the checks after a retime), contiguous with what is resident, the same power plane
template <typename State>
const char* delta_blocker(const State& st, const IngestOptions& opt, bool with_power, bool grid = true) {
  if (!st.valid) return "nothing resident";
  if (grid && (opt.step != st.w.step || opt.duration_min * 60 != st.w.span)) return kGridChanged;
  if (opt.t_end - opt.slice_seconds != st.w.t_end) return "the slice does not start where the resident window ends";
  if (opt.slice_seconds % opt.step != 0) return "the slice is not a whole number of steps";
  if (opt.slice_seconds / opt.step >= (int64_t)st.w.T) return "the slice is as long as the window";
  if (opt.reask_seconds > 0 && (opt.slice_seconds + opt.reask_seconds + opt.step - 1) / opt.step >= (int64_t)st.w.T)
    return "the slice and the re-asked seconds are as long as the window";
  if (with_power != st.with_power) return "power plane appeared / disappeared";
  if (with_power && !(opt.power_threshold == st.power_threshold ||
                      (std::isnan(opt.power_threshold) && std::isnan(st.power_threshold))))
    return "the power threshold changed";
  return nullptr;
}

// IngestOptions::retime: a delta tick whose only failing check is the grid's.  When gpr::retime_plan finds the change
// exact (a step that grew by a whole factor, a window that got shorter on an old bucket edge), the session takes the new
// grid, the other checks are evaluated against it, and the ring is retimed on the GPU (gpr_resident_retime).  Every
// PROF-fed row must still hold a sample: a fresh query of the new window would stop shadowing the UTIL twin of one
// that does not, and those UTIL samples were never parsed.  Returns the log line; anything else throws NeedFullWindow
// with the session invalid, and the tick takes the full range.
template <typename State>
std::string retime_ring(TextDevice& dev, State& st, const IngestOptions& opt, bool with_power) {
  Window& w = st.w;
  auto refuse = [&st](const std::string& why) {
    st.valid = false;
    throw NeedFullWindow(why);
  };
  const int64_t N_old = w.span, s_old = w.step, N_new = std::max<int64_t>(1, opt.duration_min * 60);
  const uint32_t T_old = w.T;
  const gpr::RetimePlan plan = gpr::retime_plan(N_old, s_old, T_old, N_new, opt.step);
  if (plan.refusal) refuse(std::string(kGridChanged) + " (" + plan.refusal + ")");
  w.step = opt.step, w.span = N_new, w.T = (plan.n_keep + plan.factor - 1) / plan.factor;
  if (const char* why = delta_blocker(st, opt, with_power, /*grid=*/false)) refuse(why);
  const auto t0 = std::chrono::steady_clock::now();
  try {
    dev.resident_retime(plan.n_keep, plan.factor);
  } catch (const std::exception& e) {  // GPR_E_NOMEM included (the peak is the old ring plus the new one)
    refuse(std::string("the resident window could not be retimed: ") + e.what());
  }
  const double retime_ms = ms_since(t0);
  if (!st.prof_rows.empty()) {
    std::vector<uint32_t> bits;
    try {
      dev.resident_live_rows(&bits);
    } catch (const std::exception& e) {
      refuse(std::string("the live rows of the retimed window could not be read: ") + e.what());
    }
    for (const auto& pr : st.prof_rows) {
      const size_t r = (size_t)pr.first * w.G + pr.second;
      if (r / 32 >= bits.size() || !((bits[r / 32] >> (r % 32)) & 1u))
        refuse("a DCGM_FI_PROF_GR_ENGINE_ACTIVE series has no sample left in the retimed window");
    }
  }
  char line[200];
  snprintf(line, sizeof line,
           "Resident window retimed on the GPU: %u -> %u (step %lld -> %lld s, window %lld -> %lld s, retime %.2f ms)",
           T_old, w.T, (long long)s_old, (long long)w.step, (long long)N_old, (long long)w.span, retime_ms);
  return line;
}

uint32_t slots_needed(const Window& w) {
  uint32_t g = 1;
  for (const PodEntry& pe : w.pods) g = std::max<uint32_t>(g, std::max<uint32_t>((uint32_t)pe.slots.size(), pe.power_slots));
  return g;
}

}  // namespace

struct DeviceIngestSession::State {
  Window w;                        // skeleton: pods / slots / shape, no planes
  std::unique_ptr<Assigner> asg;   // bound to `w`; lives as long as the rows do
  bool valid = false;              // the resident ring holds the window ending at w.t_end
  uint32_t pods_cap = 0;           // pods the ring has rows for
  bool with_power = false;
  double power_threshold = 0.0;    // what the resident power samples are snapped to
  std::vector<std::pair<uint32_t, uint32_t>> prof_rows;  // (pod, slot) fed by PROF series, sorted
};

DeviceIngestSession::DeviceIngestSession(TextDevice& dev) : dev_(dev), st_(new State()) {}
DeviceIngestSession::~DeviceIngestSession() { delete st_; }
int64_t DeviceIngestSession::resident_t_end() const { return st_->valid ? st_->w.t_end : 0; }
void DeviceIngestSession::invalidate() { st_->valid = false; }

Window DeviceIngestSession::ingest(const std::string& util, const std::string* prof, const std::string* power,
                                   const IngestOptions& opt, DeviceIngestReport* report) {
  DeviceIngestReport local;
  DeviceIngestReport& rep = report ? *report : local;
  rep = DeviceIngestReport{};
  State& st = *st_;
  const bool delta = opt.slice_seconds > 0;
  auto cpu = [&](const std::string& why) {
    st.valid = false;
    if (delta) throw NeedFullWindow("device ingest not possible for the tick's slice: " + why);
    rep.on_device = false, rep.reason = why;
    Window w = ingest_matrix_text(util, prof, power, opt);
    w.stats.warnings.push_back("device ingest not used: " + why);
    return w;
  };
  if (opt.t_end <= 0 || opt.step <= 0) return cpu("window end / step not given (query.json)");

  std::string retimed;  // IngestOptions::retime: the log line of this tick's retime ("" = none)
  if (delta) {
    // what must hold for the ring to take this tick: same grid, contiguous with what is resident
    if (const char* why = delta_blocker(st, opt, power != nullptr)) {
      if (!(opt.retime && why == kGridChanged)) {
        st.valid = false;
        throw NeedFullWindow(why);
      }
      retimed = retime_ring(dev_, st, opt, power != nullptr);
    }
    // From here on the session's rows and the ring are being changed: whatever interrupts this tick (a device error
    // in the parse, a malformed slice) must not leave a ring that claims to hold the window ending at this tick —
    // a slice that never arrived reads as "no samples", and a busy GPU would look idle.  result() sets it again.
    st.valid = false;
  } else {
    st.w = Window();
    st.asg.reset(new Assigner(st.w));
    st.valid = false;
    st.prof_rows.clear();
  }
  Window& w = st.w;
  w.stats = IngestStats();
  w.stats.ring_retime = retimed;
  Assigner& asg = *st.asg;

  TextPlan plans[3];  // prof, util, power — the order the CPU paths assign rows in
  int n_plans = 0;
  auto add = [&](const std::string* text, int slot) -> TextPlan* {
    if (!text) return nullptr;
    plans[n_plans].slot = slot, plans[n_plans].text = text;
    return &plans[n_plans++];
  };
  TextPlan* pl_prof = add(prof, 0);
  TextPlan* pl_util = add(&util, 1);
  TextPlan* pl_power = add(power, 2);
  try {
    const bool remember = delta || opt.resident;
    if (pl_prof) plan_text(dev_, *pl_prof, asg, w, false, true, rep, remember);
    plan_text(dev_, *pl_util, asg, w, false, false, rep, remember);
    if (pl_power) plan_text(dev_, *pl_power, asg, w, true, false, rep, remember);
  } catch (const NotCompact& e) {
    return cpu(e.why);
  } catch (const DeviceDeclined& e) {
    return cpu(e.what());
  }
  std::vector<std::pair<uint32_t, uint32_t>> prof_rows;
  if (pl_prof)
    for (const DevSeries& s : pl_prof->series) prof_rows.emplace_back(s.pod, s.slot);
  std::sort(prof_rows.begin(), prof_rows.end());

  uint32_t n_new = 0;  // buckets this call opens (delta) — 0: the whole window
  ReaskBand band;      // IngestOptions::reask_seconds: the re-asked buckets before the merge (n_re == 0: none)
  if (!delta) {
    finish_shape(w, opt, 0, 1, power != nullptr, /*allocate=*/false);  // t_end / step given: nothing to infer
    st.with_power = power != nullptr;
    st.power_threshold = opt.power_threshold;
    st.prof_rows = prof_rows;
    if (opt.resident) {
      st.pods_cap = w.P + w.P / 4 + 64;   // head-room: new pods get rows without a rebuild
      dev_.resident_init(st.pods_cap, w.G, w.T, st.with_power);
    }
  } else {
    // the shape is the ring's: anything that does not fit needs the full window again
    uint32_t g_now = 1;
    for (const PodEntry& pe : w.pods) g_now = std::max<uint32_t>(g_now, std::max<uint32_t>((uint32_t)pe.slots.size(), pe.power_slots));
    const char* why = nullptr;
    const bool shape = w.pods.size() > st.pods_cap || g_now > w.G;  // what reshaping the ring can absorb
    if (w.pods.size() > st.pods_cap && !opt.reshape) why = "more pods than the resident window has rows for";
    else if (g_now > w.G && !opt.reshape) why = "a pod gained a GPU slot beyond the resident window's shape";
    // `A or B` (query.promql.j2:10-20) is resolved per tick at assignment time; if the set of PROF-fed rows
    // changes, UTIL samples that were (not) shadowed earlier in the window no longer match a fresh query
    else if (prof_rows != st.prof_rows) why = "the set of DCGM_FI_PROF_GR_ENGINE_ACTIVE series changed";
    if (why) {
      st.valid = false;
      throw NeedFullWindow(why);
    }
    w.t_end = opt.t_end;
    n_new = (uint32_t)(opt.slice_seconds / opt.step);
    dev_.resident_advance(n_new);
    if (shape) {
      try {
        w.stats.ring_reshape = reshape_ring(dev_, w, asg, &st.pods_cap, &st.prof_rows, plans, n_plans);
      } catch (const std::exception& e) {  // GPR_E_NOMEM included (the peak is the old ring plus the new one)
        st.valid = false;
        throw NeedFullWindow(std::string("the resident window could not be reshaped: ") + e.what());
      }
    }
    w.P = (uint32_t)w.pods.size();
    if (opt.reask_seconds > 0 && w.P > 0) {
      band.n_new = n_new, band.n_re = (uint32_t)((opt.reask_seconds + opt.step - 1) / opt.step);
      try {
        read_band(dev_, &band, w.G, st.with_power ? 2 : 1, w.stats);
      } catch (const std::exception& e) {
        st.valid = false;
        throw NeedFullWindow(std::string("the re-asked buckets could not be read: ") + e.what());
      }
    }
  }
  const bool resident = delta || opt.resident;
  const uint32_t n_rows = (resident ? st.pods_cap : w.P) * w.G;
  auto result = [&]() {
    Window out = w;  // pods / shape / stats
    out.resident = resident;
    if (resident) out.resident_pods = st.pods_cap, out.resident_power = st.with_power, st.valid = true;
    return out;
  };
  if (w.P == 0) {
    rep.on_device = true;
    return result();
  }

  // window the parse accepts: the whole range, or only the tick's slice; the CPU re-parse patches the same buckets
  TextDevice::TextGrid grid;
  grid.t_end = w.t_end, grid.span = delta ? opt.slice_seconds + opt.reask_seconds : w.span, grid.step = w.step;
  grid.T = w.T, grid.n_rows = n_rows, grid.fill = !resident, grid.resident = resident;
  Window patch;
  patch.t_end = w.t_end, patch.step = w.step, patch.span = grid.span, patch.T = delta ? n_new + band.n_re : w.T;
  const ReaskBand* re = band.n_re ? &band : nullptr;
  std::vector<TextPlan*> util_texts;
  if (pl_prof) util_texts.push_back(pl_prof);
  util_texts.push_back(pl_util);
  parse_plane(dev_, w, util_texts, 0, grid, patch, 0, opt.power_threshold, rep, re);
  if (pl_power) parse_plane(dev_, w, {pl_power}, 1, grid, patch, 0, opt.power_threshold, rep, re);
  if (re) count_late(dev_, band, (uint32_t)w.pods.size(), w.G, st.with_power ? 2 : 1, w.stats);
  rep.on_device = true;
  Window out = result();
  if (!resident) {
    out.d_util = dev_.plane(0);
    if (pl_power) out.d_power = dev_.plane(1);
  }
  return out;
}

// A range asked as several queries (--query-slice, DESIGN.md §8e).  Every slice is planned and parsed before the next
// one is read: PROF slices first, then UTIL, then POWER, each oldest first — so every PROF series of the range is known
// before a UTIL series is assigned, and `A or B` shadows exactly as in one query.  Each slice is parsed against the
// grid of the whole fetch; slices meet on the bucket grid, so a row the device declines is patched in its slice's
// buckets only.  The session is valid again only after the last slice.
Window DeviceIngestSession::ingest_slices(const SlicedFetch& f, const IngestOptions& opt, DeviceIngestReport* report) {
  DeviceIngestReport local;
  DeviceIngestReport& rep = report ? *report : local;
  rep = DeviceIngestReport{};
  State& st = *st_;
  const bool delta = opt.slice_seconds > 0;
  std::string retimed;  // IngestOptions::retime: the log line of this tick's retime ("" = none)
  if (delta) {
    if (const char* why = delta_blocker(st, opt, f.has_power)) {
      if (!(opt.retime && why == kGridChanged)) {
        st.valid = false;
        throw NeedFullWindow(why);
      }
      retimed = retime_ring(dev_, st, opt, f.has_power);
    }
  }
  st.valid = false;
  if (opt.t_end <= 0 || opt.step <= 0) throw std::runtime_error("a sliced query needs the window end and step (query.json)");
  const int64_t span = delta ? opt.slice_seconds + opt.reask_seconds : std::max<int64_t>(1, opt.duration_min * 60);
  // the slices must tile (t_end - span, t_end] and meet on the bucket grid
  if (f.ranges.empty() || f.ranges.front().first != opt.t_end - span || f.ranges.back().second != opt.t_end)
    throw std::runtime_error("the query slices do not cover the queried range");
  for (size_t j = 0; j < f.ranges.size(); ++j)
    if (f.ranges[j].first >= f.ranges[j].second || (j && f.ranges[j].first != f.ranges[j - 1].second) ||
        (opt.t_end - f.ranges[j].second) % opt.step != 0)
      throw std::runtime_error("query slice " + std::to_string(j) + " does not meet its neighbours on the bucket grid");
  if (!delta) {
    st.w = Window();
    st.asg.reset(new Assigner(st.w));
    st.prof_rows.clear();
    st.pods_cap = 0;
    st.with_power = f.has_power;
    st.power_threshold = opt.power_threshold;
    finish_shape(st.w, opt, 0, 1, f.has_power, /*allocate=*/false);  // the grid; the shape follows the slices
  }
  Window& w = st.w;
  w.stats = IngestStats();
  w.stats.ring_retime = retimed;
  Assigner& asg = *st.asg;
  ReaskBand band;  // IngestOptions::reask_seconds: the re-asked buckets before the merge (n_re == 0: none)
  if (delta) {
    w.t_end = opt.t_end;
    dev_.resident_advance((uint32_t)(opt.slice_seconds / opt.step));
    if (opt.reask_seconds > 0) {
      band.n_new = (uint32_t)(opt.slice_seconds / opt.step);
      band.n_re = (uint32_t)((opt.reask_seconds + opt.step - 1) / opt.step);
      try {
        read_band(dev_, &band, w.G, st.with_power ? 2 : 1, w.stats);
      } catch (const std::exception& e) {
        throw NeedFullWindow(std::string("the re-asked buckets could not be read: ") + e.what());
      }
    }
  }
  const ReaskBand* re = band.n_re ? &band : nullptr;
  // the ring keeps every row it has; new pods and slots get rows of their own
  auto grow = [&](uint32_t pods, uint32_t G) {
    std::vector<uint32_t> src((size_t)pods * G, GPR_ROW_NONE);
    for (uint32_t p = 0; p < std::min(pods, st.pods_cap); ++p)
      for (uint32_t g = 0; g < w.G; ++g) src[(size_t)p * G + g] = p * w.G + g;
    try {
      dev_.resident_remap(pods, G, src);
    } catch (const std::exception& e) {
      if (delta) throw NeedFullWindow(std::string("the resident window could not be grown: ") + e.what());
      throw;
    }
    st.pods_cap = pods, w.G = G;
  };
  TextDevice::TextGrid grid;
  grid.t_end = w.t_end, grid.span = span, grid.step = w.step, grid.T = w.T;
  grid.fill = false, grid.resident = true;
  std::vector<std::pair<uint32_t, uint32_t>> prof_rows;
  for (int kind = 0; kind < 3; ++kind) {  // 0 PROF, 1 UTIL, 2 POWER: the order the one-query paths assign rows in
    if (kind == 1) {
      std::sort(prof_rows.begin(), prof_rows.end());  // the union: a series in several slices feeds one row
      prof_rows.erase(std::unique(prof_rows.begin(), prof_rows.end()), prof_rows.end());
      // `A or B` over the whole window: the PROF-fed rows of every slice against those of the resident window
      if (delta && prof_rows != st.prof_rows) throw NeedFullWindow("the set of DCGM_FI_PROF_GR_ENGINE_ACTIVE series changed");
    }
    if ((kind == 0 && !f.has_prof) || (kind == 2 && !f.has_power)) continue;
    for (size_t j = 0; j < f.ranges.size(); ++j) {
      std::string text;
      f.load(kind, j, &text);
      TextPlan plan;
      plan.slot = kind, plan.text = &text;
      try {
        plan_text(dev_, plan, asg, w, kind == 2, kind == 0, rep, /*remember=*/true);
      } catch (const NotCompact& e) {
        const std::string why = "device ingest not possible for query slice " + std::to_string(j) + ": " + e.why;
        if (delta) throw NeedFullWindow(why);
        throw std::runtime_error(why);
      } catch (const DeviceDeclined& e) {
        const std::string why = "device ingest not possible for query slice " + std::to_string(j) + ": " + e.what();
        if (delta) throw NeedFullWindow(why);
        throw std::runtime_error(why);
      }
      if (kind == 0)
        for (const DevSeries& s : plan.series) prof_rows.emplace_back(s.pod, s.slot);
      const uint32_t n_pods = (uint32_t)w.pods.size(), g_now = slots_needed(w);
      if (st.pods_cap == 0) {  // the first slice of a full fetch: the ring, with the usual head-room
        st.pods_cap = n_pods + n_pods / 4 + 64, w.G = g_now;
        dev_.resident_init(st.pods_cap, w.G, w.T, st.with_power);
      } else if (n_pods > st.pods_cap || g_now > w.G) {
        if (delta && !opt.reshape)
          throw NeedFullWindow(n_pods > st.pods_cap ? "more pods than the resident window has rows for"
                                                    : "a pod gained a GPU slot beyond the resident window's shape");
        grow(std::max(st.pods_cap, n_pods + n_pods / 4 + 64), std::max(w.G, g_now));
        ++rep.ring_growths;
      }
      // this slice's buckets: (ranges[j].first, ranges[j].second], `newer` buckets before the newest of the grid
      Window patch;
      patch.t_end = f.ranges[j].second, patch.step = w.step, patch.span = f.ranges[j].second - f.ranges[j].first;
      const uint32_t newer = (uint32_t)((w.t_end - patch.t_end) / w.step);
      patch.T = (uint32_t)std::min<int64_t>(w.T - newer, (patch.span + w.step - 1) / w.step);
      grid.n_rows = st.pods_cap * w.G;
      parse_plane(dev_, w, {&plan}, kind == 2 ? 1 : 0, grid, patch, newer, opt.power_threshold, rep, re);
    }
  }
  if (re) count_late(dev_, band, (uint32_t)w.pods.size(), w.G, st.with_power ? 2 : 1, w.stats);
  if (!delta) {
    st.prof_rows = prof_rows;
    // the shape a one-query ingest of the range gives the ring, so that later ticks take the same path
    const uint32_t n_pods = (uint32_t)w.pods.size(), want = n_pods + n_pods / 4 + 64, g_now = slots_needed(w);
    if (want != st.pods_cap || g_now != w.G) grow(want, g_now), ++rep.ring_growths;
  }
  w.P = (uint32_t)w.pods.size();
  rep.on_device = true;
  rep.slices = f.ranges.size();
  Window out = w;
  out.resident = true;
  out.resident_pods = st.pods_cap, out.resident_power = st.with_power;
  st.valid = true;
  return out;
}

bool DeviceIngestSession::save_state(SnapshotState* out) const {
  const State& st = *st_;
  if (!st.valid || !st.asg) return false;
  const Window& w = st.w;
  SnapshotState& s = *out;
  s = SnapshotState();
  s.span = w.span, s.step = w.step, s.t_end = w.t_end;
  s.T = w.T, s.pods_cap = st.pods_cap, s.G = w.G;
  s.with_power = st.with_power, s.power_threshold = st.power_threshold;
  s.pods.assign(w.pods.begin(), w.pods.end());
  st.asg->each_known([&](uint64_t h1, uint64_t h2, Assigner::Result r, uint32_t pod, uint32_t slot) {
    s.known.push_back(SnapshotState::Known{h1, h2, (uint32_t)r, pod, slot});
  });
  s.power_keys = st.asg->power_keys();
  s.power_keys.resize(s.pods.size());
  s.prof_sigs.assign(st.asg->prof_sigs().begin(), st.asg->prof_sigs().end());
  s.prof_rows = st.prof_rows;
  return true;
}

void DeviceIngestSession::export_planes(ChunkPlaneView planes[2], double* export_ms, double* copy_ms) {
  const State& st = *st_;
  if (!st.valid) throw std::logic_error("nothing resident to export");
  TextDevice::TextGrid grid;
  grid.t_end = st.w.t_end, grid.span = st.w.span, grid.step = st.w.step, grid.T = st.w.T;
  grid.n_rows = st.pods_cap * st.w.G, grid.fill = false, grid.resident = true;
  *export_ms = *copy_ms = 0;
  planes[0] = planes[1] = ChunkPlaneView();
  for (int k = 0; k < (st.with_power ? 2 : 1); ++k) {
    grid.power_threshold = k == 1 ? st.power_threshold : 0.0;
    double e = 0, c = 0;
    dev_.resident_export(k, grid, &planes[k], &e, &c);
    *export_ms += e, *copy_ms += c;
  }
}

void DeviceIngestSession::restore_state(const SnapshotState& s, const ChunkPlaneView planes[2]) {
  State& st = *st_;
  st.valid = false;
  st.w = Window();
  st.asg.reset(new Assigner(st.w));
  st.prof_rows.clear();
  TextDevice::TextGrid grid;
  grid.t_end = s.t_end, grid.span = s.span, grid.step = s.step, grid.T = s.T;
  grid.n_rows = s.pods_cap * s.G, grid.fill = false, grid.resident = true;
  grid.power_threshold = s.power_threshold;
  dev_.resident_restore(s.pods_cap, s.G, s.T, s.with_power, planes, grid);  // throws: the session stays cold
  Window& w = st.w;
  for (const PodEntry& pe : s.pods) w.pods.push_back(pe);
  w.P = (uint32_t)s.pods.size(), w.G = s.G, w.T = s.T;
  w.t_end = s.t_end, w.step = s.step, w.span = s.span;
  std::map<std::pair<uint32_t, uint32_t>, std::vector<std::string>> sigs(s.prof_sigs.begin(), s.prof_sigs.end());
  st.asg->adopt_pods(s.power_keys, std::move(sigs));
  for (const SnapshotState::Known& k : s.known)
    st.asg->insert_known(k.h1, k.h2, (Assigner::Result)k.result, k.pod, k.slot);
  st.pods_cap = s.pods_cap;
  st.with_power = s.with_power;
  st.power_threshold = s.power_threshold;
  st.prof_rows = s.prof_rows;
  st.valid = true;
}

Window ingest_matrix_device(TextDevice& dev, const std::string& util, const std::string* prof,
                            const std::string* power, const IngestOptions& opt, DeviceIngestReport* report) {
  DeviceIngestSession once(dev);
  IngestOptions o = opt;
  o.slice_seconds = 0, o.resident = false;
  return once.ingest(util, prof, power, o, report);
}

}  // namespace gph
