#include "controller.hpp"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <limits>
#include <stdexcept>
#include <sys/stat.h>
#include <thread>
#include <unordered_map>

#include "ingest_device.hpp"

namespace gph {

// ---- logging (main.rs:157-243: default | json | pretty) --------------------------------------------
void Logger::log(const char* level, const std::string& msg,
                 const std::vector<std::pair<std::string, std::string>>& fields) const {
  const auto now = std::chrono::system_clock::now();
  const int64_t ns = std::chrono::duration_cast<std::chrono::nanoseconds>(now.time_since_epoch()).count();
  const std::string ts = rfc3339(ns / 1000 * 1000);
  if (fmt_ == LogFormat::Json) {
    Json f = Json::object();
    f.set("message", msg);
    for (auto& kv : fields) f.set(kv.first, kv.second);
    Json j = Json::object();
    j.set("timestamp", ts);
    j.set("level", level);
    j.set("fields", f);
    j.set("target", "gpu_pruner");
    fprintf(out_, "%s\n", j.dump().c_str());
  } else if (fmt_ == LogFormat::Pretty) {
    fprintf(out_, "  %s %s gpu_pruner: %s\n", ts.c_str(), level, msg.c_str());
    for (auto& kv : fields) fprintf(out_, "    %s: %s\n", kv.first.c_str(), kv.second.c_str());
  } else {
    std::string extra;
    for (auto& kv : fields) extra += " " + kv.first + "=" + kv.second;
    fprintf(out_, "%s %5s gpu_pruner: %s%s\n", ts.c_str(), level, msg.c_str(), extra.c_str());
  }
  fflush(out_);
}
void Logger::counter(const char* level, const std::string& name, uint64_t v, const std::string& msg) const {
  log(level, msg, {{name, std::to_string(v)}});
}

// ---- window sources ----------------------------------------------------------------------------------
namespace {

bool file_exists(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0;
}

// a recorded response can be more than a gigabyte: one sized read, not a character iterator
std::string read_file(const std::string& path, uint64_t* read_bytes) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) throw std::runtime_error("cannot open " + path);
  std::string s;
  struct stat st;
  if (fstat(fileno(f), &st) == 0 && st.st_size > 0) s.resize((size_t)st.st_size);
  size_t got = 0;
  while (got < s.size()) {
    const size_t k = fread(&s[got], 1, s.size() - got, f);
    if (k == 0) break;
    got += k;
  }
  s.resize(got);
  char tail[4096];  // a file that grew after fstat (or has no size): read on
  for (size_t k; (k = fread(tail, 1, sizeof tail, f)) > 0;) s.append(tail, k);
  fclose(f);
  *read_bytes += s.size();
  return s;
}

// file://DIR — recorded range-query responses instead of a Prometheus server:
//   DIR/util.json [prof.json] [power.json] [dmi.json] [query.json = {"end": ts, "step": s}]     every tick the same
//   DIR/tick-0000/..., DIR/tick-0001/...                                                       one directory per tick,
//     each either with the files above, or with full/ (the whole [Nm] range) and delta/ (only what was scraped
//     since the previous tick: query.json = {"end", "step", "start"}, samples in (start, end]) — the two answers a
//     server would give to the two questions daemon mode can ask.
class FileSource : public WindowSource {
 public:
  FileSource(std::string dir, TextIngestor* ingestor, const Logger* log)
      : dir_(std::move(dir)), ingestor_(ingestor), log_(log) {}
  Window fetch(const Cli& args) override {
    std::string base = dir_;
    if (file_exists(dir_ + "/tick-0000")) {
      char name[32];
      snprintf(name, sizeof name, "/tick-%04d", tick_++);
      base = dir_ + name;
      if (!file_exists(base)) throw std::runtime_error("Failed to run query! " + base + " not found (no more recorded ticks)");
    }
    const bool can_reside = args.daemon_mode && ingestor_ != nullptr;
    // --query-slice: a range longer than S seconds is asked as consecutive queries of at most S seconds
    const int64_t S = ingestor_ ? args.query_slice : 0;
    // daemon mode with a resident window: ask only for what was scraped since the previous tick
    const int64_t since = can_reside ? ingestor_->resident_t_end() : 0;
    // --late-seconds: the delta also asks again for the newest L seconds the resident window holds
    const int64_t L = can_reside ? args.late_seconds : 0;
    const bool delta_there = file_exists(base + "/delta/util.json") || (S > 0 && file_exists(base + "/delta/slice-0000"));
    if (since > 0 && delta_there && file_exists(base + "/delta/query.json")) {
      const Json meta = Json::parse_file(base + "/delta/query.json");
      const int64_t start = (int64_t)meta["start"].as_number(0), end = (int64_t)meta["end"].as_number(0);
      if (start == since - L && end > since) {
        try {
          if (S > 0 && end - start > S) return load_slices(args, base + "/delta", start, end, S, true, L);
          return load(args, base + "/delta", end - since, true, L);
        } catch (const NeedFullWindow& e) {
          if (log_) log_->info(std::string("Resident window rebuilt from the full range: ") + e.what());
        }
      } else if (log_) {
        log_->info("Recorded delta does not continue the resident window (starts at " + std::to_string(start) +
                   ", resident up to " + std::to_string(since) + "): using the full range");
      }
    }
    if (S > 0 && args.duration * 60 > S) {
      const std::string full = file_exists(base + "/full/query.json") ? base + "/full" : base;
      const int64_t end = file_exists(full + "/query.json")
                              ? (int64_t)Json::parse_file(full + "/query.json")["end"].as_number(0) : 0;
      return load_slices(args, full, end - args.duration * 60, end, S, false);
    }
    return load(args, file_exists(base + "/full/util.json") ? base + "/full" : base, 0, can_reside);
  }

 private:
  // --retime-ring: one line per retime, with its counter
  void log_retime(const Window& w) const {
    if (log_ && !w.stats.ring_retime.empty()) log_->counter("INFO", "monotonic_counter.ring_retimes", 1, w.stats.ring_retime);
  }

  // --late-seconds: what the re-ask of a delta tick changed, one line and a counter per tick that raised a cell
  void log_late(const Window& w, int64_t reask) const {
    const uint64_t u = w.stats.late_util_cells, p = w.stats.late_power_cells;
    if (!log_ || u + p == 0) return;
    char line[200];
    snprintf(line, sizeof line, "Late samples raised %llu util cells and %llu power cells in the re-asked %lld s",
             (unsigned long long)u, (unsigned long long)p, (long long)reask);
    log_->counter("INFO", "monotonic_counter.late_cells", u + p, line);
  }

  Window load(const Cli& args, const std::string& d, int64_t slice_seconds, bool resident, int64_t reask = 0) {
    const std::string up = d + "/util.json";
    if (!file_exists(up)) throw std::runtime_error("Failed to run query! " + up + " not found");
    const auto read_t0 = std::chrono::steady_clock::now();
    uint64_t read_bytes = 0;
    auto slurp = [&read_bytes](const std::string& path) { return read_file(path, &read_bytes); };
    const std::string util = slurp(up);
    std::string prof, power;
    const std::string *pprof = nullptr, *ppower = nullptr;
    if (file_exists(d + "/prof.json")) prof = slurp(d + "/prof.json"), pprof = &prof;
    const bool want_power = args.power_threshold && *args.power_threshold != 0.0;
    if (want_power && file_exists(d + "/power.json")) power = slurp(d + "/power.json"), ppower = &power;
    IngestOptions opt;
    opt.duration_min = args.duration;
    opt.power_threshold = want_power ? *args.power_threshold : 0.0;
    if (file_exists(d + "/query.json")) {
      const Json meta = Json::parse_file(d + "/query.json");
      opt.t_end = (int64_t)meta["end"].as_number(0);
      opt.step = (int64_t)meta["step"].as_number(0);
    }
    opt.slice_seconds = slice_seconds;
    opt.reask_seconds = reask;
    opt.resident = resident;
    opt.reshape = args.reshape_ring;
    opt.retime = args.retime_ring;
    if (log_) {
      char rbuf[160];
      snprintf(rbuf, sizeof rbuf, "Recorded responses read from %s: %.1f MB in %.1f ms", d.c_str(), read_bytes / 1e6,
               std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - read_t0).count());
      log_->info(rbuf);
    }
    Window w;
    if (!ingestor_) {
      w = ingest_matrix_text(util, pprof, ppower, opt);
    } else {
      std::string note;
      w = ingestor_->ingest(args, util, pprof, ppower, opt, &note);
      log_retime(w);
      if (log_ && !w.stats.ring_reshape.empty())  // --reshape-ring: one line per reshape, with its counter
        log_->counter("INFO", "monotonic_counter.ring_reshapes", 1, w.stats.ring_reshape);
      if (log_ && !note.empty()) log_->info(note);
      log_late(w, reask);
    }
    // node_type for the rows of PodMetricData: the node_dmi_info join of query.promql.j2:23-34
    if (file_exists(d + "/dmi.json")) apply_node_types(w, Json::parse_file(d + "/dmi.json"));
    return w;
  }

  // (start, end] asked as consecutive queries of at most S seconds, the newest ending at `end`: d/slice-0000/ (oldest)
  // ... each with util.json [prof.json] [power.json] and query.json = {"start", "end", "step"} of that query.  A slice
  // that is missing or answers another range fails the query; the session is cold then (ingest_slices reads the
  // slices one by one, after it has given up the resident window).
  Window load_slices(const Cli& args, const std::string& d, int64_t start, int64_t end, int64_t S, bool delta,
                     int64_t reask = 0) {
    if (!file_exists(d + "/query.json")) throw std::runtime_error("Failed to run query! " + d + "/query.json not found");
    const int64_t step = (int64_t)Json::parse_file(d + "/query.json")["step"].as_number(0);
    if (step <= 0 || S % step != 0)
      throw std::runtime_error("Failed to run query! --query-slice " + std::to_string(S) +
                               " s is not a whole number of the query step (" + std::to_string(step) +
                               " s): slices would share buckets");
    SlicedFetch f;
    const int64_t n = (end - start + S - 1) / S;
    for (int64_t j = 0; j < n; ++j) f.ranges.emplace_back(std::max(start, end - (n - j) * S), end - (n - 1 - j) * S);
    auto dir = [&d](size_t j) {
      char name[32];
      snprintf(name, sizeof name, "/slice-%04zu", j);
      return d + name;
    };
    const bool want_power = args.power_threshold && *args.power_threshold != 0.0;
    f.has_prof = file_exists(dir(0) + "/prof.json");
    f.has_power = want_power && file_exists(dir(0) + "/power.json");
    uint64_t read_bytes = 0;
    double read_ms = 0;
    f.load = [&](int kind, size_t j, std::string* text) {
      const auto t0 = std::chrono::steady_clock::now();
      const std::string sd = dir(j);
      if (!file_exists(sd + "/query.json")) throw std::runtime_error("Failed to run query! " + sd + "/query.json not found");
      const Json q = Json::parse_file(sd + "/query.json");
      const int64_t qs = (int64_t)q["start"].as_number(0), qe = (int64_t)q["end"].as_number(0);
      if (qs != f.ranges[j].first || qe != f.ranges[j].second || (int64_t)q["step"].as_number(0) != step)
        throw std::runtime_error("Failed to run query! recorded slice " + sd + " answers (" + std::to_string(qs) + ", " +
                                 std::to_string(qe) + "], the query asks for (" + std::to_string(f.ranges[j].first) +
                                 ", " + std::to_string(f.ranges[j].second) + "]");
      static const char* const kFile[3] = {"/prof.json", "/util.json", "/power.json"};
      const std::string path = sd + kFile[kind];
      if (!file_exists(path)) throw std::runtime_error("Failed to run query! " + path + " not found");
      *text = read_file(path, &read_bytes);
      read_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    };
    IngestOptions opt;
    opt.duration_min = args.duration;
    opt.power_threshold = want_power ? *args.power_threshold : 0.0;
    opt.t_end = end, opt.step = step;
    opt.slice_seconds = delta ? end - start - reask : 0;
    opt.reask_seconds = delta ? reask : 0;
    opt.resident = true;
    opt.reshape = args.reshape_ring;
    opt.retime = args.retime_ring;
    std::string note;
    Window w = ingestor_->ingest_slices(args, f, opt, &note);
    log_retime(w);
    if (log_) {
      char rbuf[200];
      snprintf(rbuf, sizeof rbuf, "Recorded responses read from %s: %zu query slices of at most %lld s, %.1f MB in %.1f ms",
               d.c_str(), f.ranges.size(), (long long)S, read_bytes / 1e6, read_ms);
      log_->info(rbuf);
      if (!note.empty()) log_->info(note);
    }
    log_late(w, opt.reask_seconds);
    if (file_exists(d + "/dmi.json")) apply_node_types(w, Json::parse_file(d + "/dmi.json"));
    return w;
  }

  std::string dir_;
  TextIngestor* ingestor_;
  const Logger* log_;
  int tick_ = 0;
};

class CpuTextIngestor : public TextIngestor {
 public:
  Window ingest(const Cli&, const std::string& util, const std::string* prof, const std::string* power,
                const IngestOptions& opt, std::string* note) override {
    const auto t0 = std::chrono::steady_clock::now();
    Window w = ingest_matrix_text(util, prof, power, opt);
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (note) {
      char buf[160];
      snprintf(buf, sizeof buf, "Device ingest not used (GPR_INGEST=cpu): CPU text parser, %.1f ms", ms);
      *note = buf;
    }
    return w;
  }
  DeviceIngestSession* resident_session(const Cli&, std::string* error) override {
    *error = "GPR_INGEST=cpu keeps no resident window";
    return nullptr;
  }
};

class UnsupportedSource : public WindowSource {
 public:
  explicit UnsupportedSource(std::string url) : url_(std::move(url)) {}
  Window fetch(const Cli&) override {
    throw std::runtime_error("Failed to run query! HTTP transport to " + url_ +
                             " is not part of this build (no network); use file://DIR");
  }

 private:
  std::string url_;
};

}  // namespace

std::unique_ptr<TextIngestor> make_cpu_text_ingestor() { return std::make_unique<CpuTextIngestor>(); }

std::unique_ptr<WindowSource> make_window_source(const std::string& url, TextIngestor* ingestor, const Logger* log) {
  if (url.rfind("file://", 0) == 0) return std::make_unique<FileSource>(url.substr(7), ingestor, log);
  return std::make_unique<UnsupportedSource>(url);
}

// ---- controller -----------------------------------------------------------------------------------------
Controller::Controller(const Cli& args, KubeApi* kube, VerdictEngine* engine, Logger log, Clock clock)
    : args_(args), kube_(kube), engine_(engine), log_(log), clock_(std::move(clock)),
      enabled_(get_enabled_resources(args.enabled_resources)) {}

TickResult Controller::run_query_and_scale(const Window& w) {
  TickResult out;
  const uint32_t P = w.P, G = w.G;
  const uint32_t W = (P + 31) / 32;
  std::vector<uint32_t> dbits(std::max<uint32_t>(W, 1), 0), cbits(std::max<uint32_t>(W, 1), 0);
  std::vector<float> smax((size_t)P * G + 1, 0.f);
  std::vector<uint32_t> idle_slots;   // the engine's, when it resolved the `sum by` groups itself

  // lookback = duration + grace (main.rs:413-414); `now` once per tick
  const int64_t now_ns = args_.now_override ? args_.now_override * 1000000000ll : clock_.now_ns();
  const int64_t lookback_ns = (args_.duration * 60 + args_.grace_period) * 1000000000ll;
  const int64_t cutoff = now_ns - lookback_ns;

  // Pod metadata for the fused gate.  With a pod cache (fixtures / informer) every pod's phase and
  // creation time are known up front and ride along into the kernel; pods that cannot be
  // fetched are skipped exactly as main.rs:452-471 does.
  std::vector<uint8_t> eligible(std::max<uint32_t>(P, 1), 1);
  std::vector<int64_t> created(std::max<uint32_t>(P, 1), std::numeric_limits<int64_t>::max());
  std::vector<Json> pod_objs(P);
  std::vector<std::string> skip_reason(P);
  for (uint32_t p = 0; p < P && kube_; ++p) {
    const PodEntry& pe = w.pods[p];
    std::optional<Json> pod;
    try {
      pod = kube_->get_pod(pe.ns, pe.name);
    } catch (const std::exception& e) {
      eligible[p] = 0;
      skip_reason[p] = std::string("retrieval error: ") + e.what();
      continue;
    }
    if (!pod) {
      eligible[p] = 0;
      skip_reason[p] = "pod no longer exists";
      continue;
    }
    if ((*pod)["status"]["phase"].as_string() == "Pending") {   // main.rs:473-483
      eligible[p] = 0;
      skip_reason[p] = "it's still pending";
    }
    const Json& ct = (*pod)["metadata"]["creationTimestamp"];
    if (ct.is_string()) {
      try {
        created[p] = parse_rfc3339(ct.as_string());
      } catch (const std::exception&) {
        skip_reason[p] = "unparseable creation timestamp";
      }
    } else if (skip_reason[p].empty()) {
      skip_reason[p] = "has no creation timestamp";            // main.rs:485-492
    }
    pod_objs[p] = std::move(*pod);
  }

  if (P > 0) {
    VerdictRequest rq;
    rq.window = &w;
    rq.power_on = (!w.power.empty() || w.d_power || (w.resident && w.resident_power)) && args_.power_threshold &&
                  *args_.power_threshold != 0.0;
    rq.power_threshold = rq.power_on ? *args_.power_threshold : 0.0;
    rq.eligible = kube_ ? eligible.data() : nullptr;
    rq.created_ts = kube_ ? created.data() : nullptr;
    rq.cutoff_ts = cutoff;
    rq.gpu_device = args_.gpu_device;
    Verdict v;
    std::string err;
    if (!engine_ || !engine_->decide(rq, &v, &err)) {
      out.error = "Failed to run query! " + (engine_ ? err : std::string("no idle engine"));
      return out;
    }
    const size_t MW = (G + 31) / 32;
    if (v.decision_bits.size() < W || v.candidate_bits.size() < W ||
        (v.groups_resolved ? v.idle_slots.size() < (size_t)P * MW : v.series_max.size() < (size_t)P * G)) {
      out.error = "Failed to run query! idle engine returned a short result";
      return out;
    }
    // pods with several series in one `sum by` group: the element is the SUM of the members' maxima
    // (query.promql.j2:9,21); the engine does that itself given the group table, otherwise it is re-derived here
    // from the per-series maxima
    if (v.groups_resolved) {
      idle_slots = std::move(v.idle_slots);
    } else if (v.veto_bits.size() >= W || !rq.power_on) {
      const GroupFixup fx = resolve_sum_by_groups(w, v.series_max.data(), v.veto_bits.size() >= W ? v.veto_bits.data() : nullptr,
                                                  rq.eligible, rq.created_ts, rq.cutoff_ts, v.candidate_bits.data(),
                                                  v.decision_bits.data(), &v.n_series, &v.n_candidates, &v.n_decisions);
      if (fx.pods_changed)
        log_.info("sum by: " + std::to_string(fx.pods_examined) + " pod(s) with duplicate series re-evaluated, " +
                  std::to_string(fx.pods_changed) + " verdict(s) changed");
    } else {
      for (const PodEntry& pe : w.pods)
        if (pe.has_groups) {
          out.error = "Failed to run query! idle engine returned no veto bitmap for a window with duplicate series";
          return out;
        }
    }
    std::copy(v.decision_bits.begin(), v.decision_bits.begin() + W, dbits.begin());
    std::copy(v.candidate_bits.begin(), v.candidate_bits.begin() + W, cbits.begin());
    if (!v.groups_resolved) std::copy(v.series_max.begin(), v.series_max.begin() + (size_t)P * G, smax.begin());
    out.qr.num_pods = (size_t)v.n_series;
    out.kernel_ms = v.kernel_ms;
    out.n_candidates = v.n_candidates;
    out.n_decisions = v.n_decisions;
  }

  // candidates -> PodMetricData rows (first idle series of the pod wins, main.rs:430-435)
  for (uint32_t p = 0; p < P; ++p) {
    if (!(cbits[p >> 5] >> (p & 31) & 1u)) continue;
    const PodEntry& pe = w.pods[p];
    PodMetricData pmd;
    pmd.name = pe.name, pmd.ns = pe.ns;
    if (!idle_slots.empty()) {
      // the first slot that starts an idle element; its value is 0 (a cancelling round-to-nearest sum is +0.0)
      const size_t MW = (G + 31) / 32;
      for (uint32_t g = 0; g < pe.slots.size(); ++g) {
        if (!(idle_slots[(size_t)p * MW + (g >> 5)] >> (g & 31) & 1u)) continue;
        const GpuSlot& s = pe.slots[g];
        pmd.container = s.container, pmd.node_type = s.node_type, pmd.gpu_model = s.model;
        pmd.value = 0.0;
        break;
      }
      out.unique_pods.push_back(pmd);
      continue;
    }
    for (uint32_t g = 0; g < pe.slots.size(); ++g) {
      if (pe.slots[g].group != g) continue;              // elements are `sum by` groups (j2:9)
      const double value = group_value(w, smax.data(), p, g);
      if (value == 0.0) {
        const GpuSlot& s = pe.slots[g];
        pmd.container = s.container, pmd.node_type = s.node_type, pmd.gpu_model = s.model;
        pmd.value = value;                               // what lib.rs:184 reads: 0 for every survivor of `== 0`
        break;
      }
    }
    out.unique_pods.push_back(pmd);
  }
  log_.info("Query returned " + std::to_string(out.qr.num_pods) + " series across " +
            std::to_string(out.unique_pods.size()) + " unique pods");

  // gates (already folded into decision_bits) + owner walk (main.rs:444-532)
  std::unordered_set<ScaleKind, ScaleKindHash> seen;
  for (uint32_t p = 0; p < P; ++p) {
    if (!(cbits[p >> 5] >> (p & 31) & 1u)) continue;
    const PodEntry& pe = w.pods[p];
    const bool decided = (dbits[p >> 5] >> (p & 31)) & 1u;
    if (!kube_) continue;
    if (!decided) {
      const std::string why = !skip_reason[p].empty() ? skip_reason[p]
                              : "created after the lookback window (" + rfc3339(created[p]) + " >= " + rfc3339(cutoff) + ")";
      log_.info("Skipping " + pe.ns + ":" + pe.name + ", " + why);
      continue;
    }
    log_.info("Pod " + pe.ns + ":" + pe.name + " is idle and eligible for scaledown");
    RootResult rr;
    try {
      rr = find_root_object(*kube_, pod_objs[p]["metadata"]);
    } catch (const std::exception& e) {
      rr.error = e.what();
    }
    if (!rr.root) {
      log_.warn("Skipping " + pe.ns + ":" + pe.name + ", no scalable root object: " + rr.error);
      continue;
    }
    if (seen.insert(*rr.root).second) out.shutdown.push_back(*rr.root);
  }
  out.qr.shutdown_events = out.shutdown.size();

  const char* pod_name_env = getenv("POD_NAME");
  for (const ScaleKind& sk : out.shutdown) {
    const std::string id = "[" + sk.kind_name() + "] " + sk.ns().value_or("") + ":" + sk.name();
    if (args_.run_mode == Mode::DryRun) {               // main.rs:540-551
      log_.info("Dry-run: Would have sent " + id + " for scaledown");
      continue;
    }
    log_.info("Sending " + id + " for scaledown");
    if (!(enabled_ & sk.resource_kind())) {             // main.rs:337-345
      log_.info("Skipping resource type \"" + sk.kind_name() + "\" because it is not enabled");
      continue;
    }
    for (Request& rq : scale_requests(sk, clock_, pod_name_env ? pod_name_env : "")) out.requests.push_back(std::move(rq));
    ++scale_successes;
    log_.counter("INFO", "monotonic_counter.scale_successes", 1,
                 "Scaled Resource: [" + sk.kind_name() + "] - " + sk.ns().value_or("default") + ":" + sk.name());
  }
  out.ok = true;
  return out;
}

int Controller::run(WindowSource& src) {
  size_t consecutive_failures = 0;   // QUERY_FAILURES, main.rs:136
  int ticks = 0;
  std::ofstream patch_out;
  if (args_.patch_out) patch_out.open(*args_.patch_out, std::ios::app);
  if (snapshots_ && args_.daemon_mode) {
    std::string line;
    const bool ok = snapshots_->restore(&line);
    log_.log(ok ? "INFO" : "WARN", line);
  }
  auto next_tick = std::chrono::steady_clock::now();
  while (true) {
    if (args_.daemon_mode) {          // first tick fires immediately (tokio interval), main.rs:292-294
      std::this_thread::sleep_until(next_tick);
      next_tick += std::chrono::seconds(args_.check_interval);
    }
    TickResult tr;
    const auto tick_t0 = std::chrono::steady_clock::now();
    double fetch_ms = 0;
    bool resident = false;
    try {
      Window w = src.fetch(args_);
      fetch_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tick_t0).count();
      resident = w.resident;
      tr = run_query_and_scale(w);
    } catch (const std::exception& e) {
      tr.ok = false;
      tr.error = e.what();
    }
    if (tr.ok) {
      const double tick_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tick_t0).count();
      char tbuf[200];
      snprintf(tbuf, sizeof tbuf, "Tick %d: window ready in %.2f ms, verdict and gates in %.2f ms (decision kernels %.3f ms)", ticks,
               fetch_ms, tick_ms - fetch_ms, tr.kernel_ms);
      log_.info(tbuf);
      consecutive_failures = 0;
      ++query_successes;
      log_.counter("INFO", "monotonic_counter.query_successes", 1, "Query succeeded");
      log_.counter("INFO", "counter.query_returned_candidates", tr.qr.num_pods, "Returned candidates");
      log_.counter("INFO", "counter.query_returned_shutdown_events", tr.qr.shutdown_events,
                   "Returned shutdown events");
      for (const Request& rq : tr.requests) {
        Json j = Json::object();
        j.set("method", rq.method), j.set("path", rq.path), j.set("contentType", rq.content_type);
        j.set("body", rq.body);
        if (patch_out.is_open()) patch_out << j.dump() << "\n" << std::flush;
        else fprintf(stdout, "%s\n", j.dump().c_str());
      }
      // the verdict is out: now the window it was decided on may go to disk.  A failed write costs the next start
      // the full range, nothing else — not the tick's result, not query_failures.
      if (snapshots_ && resident) {
        std::string line;
        const int rc = snapshots_->save(&line);
        if (rc > 0) {
          log_.info(line);
        } else if (rc < 0) {
          ++snapshot_failures;
          log_.counter("ERROR", "monotonic_counter.snapshot_failures", 1, "Snapshot not written: " + line);
        }
      }
    } else {
      const size_t failures = consecutive_failures++;   // fetch_add returns the previous value
      ++query_failures;
      log_.counter("ERROR", "monotonic_counter.query_failures", 1,
                   "Failed to run query and scale down: " + tr.error);
      if (failures > 5) {                               // main.rs:317-320
        log_.error("Too many consecutive failures, exiting");
        break;   // the reference leaves the loop and main() still returns Ok(()) -> exit code 0
      }
    }
    ++ticks;
    if (!args_.daemon_mode) break;
    if (args_.max_ticks && ticks >= args_.max_ticks) break;
  }
  return 0;  // like the reference: failures are logged and counted, never turned into an exit code
}

}  // namespace gph
