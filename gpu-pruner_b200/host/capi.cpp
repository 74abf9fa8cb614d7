// capi.cpp — a small extern "C" surface over the host library so the test-suite (pytest + ctypes)
// can exercise the pure host logic — CLI parsing, PromQL rendering, matrix ingest, owner walk,
// scale requests — without a GPU.  Strings are returned in a caller-provided buffer as JSON.
#include <chrono>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

#include "cli.hpp"
#include "controller.hpp"
#include "ingest.hpp"
#include "json.hpp"
#include "kube.hpp"
#include "promql.hpp"
#include "snapshot.hpp"

#define GPH_API extern "C" __attribute__((visibility("default")))

namespace {
int put(const std::string& s, char* out, int cap) {
  if ((int)s.size() + 1 > cap) return -(int)(s.size() + 1);
  memcpy(out, s.c_str(), s.size() + 1);
  return (int)s.size();
}
std::vector<std::string> split_args(const char* nul_separated, int n) {
  std::vector<std::string> v;
  const char* p = nul_separated;
  for (int i = 0; i < n; ++i) {
    v.emplace_back(p);
    p += v.back().size() + 1;
  }
  return v;
}
gph::Json cli_json(const gph::Cli& c) {
  using gph::Json;
  Json j = Json::object();
  j.set("duration", (int64_t)c.duration);
  j.set("daemon_mode", c.daemon_mode);
  j.set("enabled_resources", c.enabled_resources);
  j.set("check_interval", (int64_t)c.check_interval);
  j.set("namespace", c.ns ? Json(*c.ns) : Json());
  j.set("grace_period", (int64_t)c.grace_period);
  j.set("model_name", c.model_name ? Json(*c.model_name) : Json());
  j.set("power_threshold", c.power_threshold ? Json(*c.power_threshold) : Json());
  j.set("honor_labels", c.honor_labels);
  j.set("run_mode", gph::to_string(c.run_mode));
  j.set("prometheus_url", c.prometheus_url);
  j.set("prometheus_token", c.prometheus_token ? Json(*c.prometheus_token) : Json());
  j.set("prometheus_tls_mode", gph::to_string(c.prometheus_tls_mode));
  j.set("prometheus_tls_cert", c.prometheus_tls_cert ? Json(*c.prometheus_tls_cert) : Json());
  j.set("log_format", gph::to_string(c.log_format));
  return j;
}
}  // namespace

// args: n NUL-terminated strings back to back.  JSON out: {"ok":bool,"exit_code":n,"message":s,"cli":{...}}
GPH_API int gph_parse_cli(const char* args, int n, char* out, int cap) {
  gph::ParseOutcome po = gph::parse_cli(split_args(args, n));
  gph::Json j = gph::Json::object();
  j.set("ok", po.ok);
  j.set("exit_code", po.exit_code);
  j.set("message", po.message);
  j.set("cli", cli_json(po.cli));
  return put(j.dump(), out, cap);
}

GPH_API int gph_render_query(const char* args, int n, char* out, int cap) {
  gph::ParseOutcome po = gph::parse_cli(split_args(args, n));
  if (!po.ok) return put(po.message, out, cap) >= 0 ? -1 : -2;
  return put(gph::render_query(po.cli), out, cap);
}

GPH_API int gph_render_selectors(const char* args, int n, char* out, int cap) {
  gph::ParseOutcome po = gph::parse_cli(split_args(args, n));
  if (!po.ok) return -1;
  gph::Selectors s = gph::render_selectors(po.cli);
  gph::Json j = gph::Json::object();
  j.set("prof", s.prof), j.set("util", s.util), j.set("power", s.power);
  return put(j.dump(), out, cap);
}

// CRC32C of the snapshot file (snapshot.hpp): portable = 1 forces the slice-by-8 tables, 0 takes the SSE4.2
// instruction when the CPU has it
GPH_API unsigned gph_crc32c(const void* data, unsigned long long n, unsigned crc, int portable) {
  return portable ? gph::crc32c_portable(data, (size_t)n, crc) : gph::crc32c(data, (size_t)n, crc);
}

GPH_API int gph_enabled_resources(const char* letters) { return gph::get_enabled_resources(letters); }

GPH_API int gph_format_float(double v, char* out, int cap) { return put(gph::format_float(v), out, cap); }

// ingest: JSON texts in, tensor out.  Returns 0 or negative; dims written to dims[3] = P,G,T.
// util_out/power_out may be NULL to query dimensions + the pod table (JSON) first.
// gph_ingest_for_threshold: the same, with the threshold the power plane will be decided with
// (IngestOptions::power_threshold: power samples are snapped to it; 0 = none, which is what gph_ingest does).
static int g_ingest_threads = -1;  // -1: DOM path; >= 0: text path with that many threads (0 = all)
GPH_API void gph_ingest_mode(int threads) { g_ingest_threads = threads; }
// response of the `node_dmi_info` query applied by the following gph_ingest calls (NULL / "" = none)
static std::string g_dmi_json;
GPH_API void gph_ingest_dmi(const char* dmi_json) { g_dmi_json = dmi_json ? dmi_json : ""; }
static gph::Window g_last_window;  // the window of the most recent successful gph_ingest (tensor dropped)

GPH_API int gph_ingest_for_threshold(const char* util_json, const char* prof_json, const char* power_json,
                                     long long duration_min, long long step, long long t_end, double power_threshold,
                                     unsigned* dims, float* util_out, float* power_out, char* pods_json, int cap) {
  try {
    gph::IngestOptions o;
    o.duration_min = duration_min, o.step = step, o.t_end = t_end, o.power_threshold = power_threshold;
    gph::Window w;
    const auto t0 = std::chrono::steady_clock::now();
    if (g_ingest_threads >= 0) {
      std::string us(util_json), ps, ws;
      if (prof_json) ps = prof_json;
      if (power_json) ws = power_json;
      w = gph::ingest_matrix_text(us, prof_json ? &ps : nullptr, power_json ? &ws : nullptr, o,
                                  g_ingest_threads);
    } else {
      gph::Json u = gph::Json::parse(util_json, 2), pf, pw;   // (2: the response envelope is a struct)
      const gph::Json *ppf = nullptr, *ppw = nullptr;
      if (prof_json) pf = gph::Json::parse(prof_json, 2), ppf = &pf;
      if (power_json) pw = gph::Json::parse(power_json, 2), ppw = &pw;
      w = gph::ingest_matrix(u, ppf, ppw, o);
    }
    if (!g_dmi_json.empty()) gph::apply_node_types(w, gph::Json::parse(g_dmi_json));
    const double ingest_ms =
        std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    dims[0] = w.P, dims[1] = w.G, dims[2] = w.T;
    if (util_out) memcpy(util_out, w.util.data(), w.util.size() * sizeof(float));
    if (power_out && !w.power.empty()) memcpy(power_out, w.power.data(), w.power.size() * sizeof(float));
    gph::Json pods = gph::Json::array();
    for (const gph::PodEntry& pe : w.pods) {
      gph::Json p = gph::Json::object();
      p.set("name", pe.name), p.set("namespace", pe.ns);
      gph::Json slots = gph::Json::array();
      for (const gph::GpuSlot& s : pe.slots) {
        gph::Json sj = gph::Json::object();
        sj.set("Hostname", s.hostname), sj.set("container", s.container), sj.set("gpu", s.gpu);
        sj.set("modelName", s.model), sj.set("node_type", s.node_type), sj.set("from_prof", s.from_prof);
        sj.set("group", (int64_t)s.group);
        slots.push(sj);
      }
      p.set("slots", slots);
      p.set("has_groups", pe.has_groups);
      p.set("power_slots", (int64_t)pe.power_slots);
      pods.push(p);
    }
    gph::Json meta = gph::Json::object();
    meta.set("pods", pods);
    meta.set("t_end", (int64_t)w.t_end), meta.set("step", (int64_t)w.step);
    meta.set("ingest_ms", ingest_ms);
    meta.set("series_in", (int64_t)w.stats.series_in), meta.set("series_skipped", (int64_t)w.stats.series_skipped);
    meta.set("samples_out_of_window", (int64_t)w.stats.samples_out_of_window);
    meta.set("duplicates_merged", (int64_t)w.stats.duplicates_merged);
    meta.set("tiny_values_clamped", (int64_t)w.stats.tiny_values_clamped);
    meta.set("span", (int64_t)w.span);
    g_last_window = std::move(w);
    g_last_window.util.clear(), g_last_window.power.clear();
    return pods_json ? (put(meta.dump(), pods_json, cap) >= 0 ? 0 : -3) : 0;
  } catch (const std::exception& e) {
    if (pods_json) put(std::string("{\"error\":\"") + gph::json_escape(e.what()) + "\"}", pods_json, cap);
    return -1;
  }
}

GPH_API int gph_ingest(const char* util_json, const char* prof_json, const char* power_json,
                       long long duration_min, long long step, long long t_end, unsigned* dims,
                       float* util_out, float* power_out, char* pods_json, int cap) {
  return gph_ingest_for_threshold(util_json, prof_json, power_json, duration_min, step, t_end, 0.0, dims, util_out,
                                  power_out, pods_json, cap);
}

// Exact `sum by` for the window of the last gph_ingest: corrects the engine's / oracle's raw verdict arrays in
// place (gph::resolve_sum_by_groups).  veto_bits / eligible / created_ts may be NULL.  counts = n_series,
// n_candidates, n_decisions.  Returns the number of pods whose verdict changed, or negative.
GPH_API int gph_resolve_groups(const float* series_max, const unsigned* veto_bits, const unsigned char* eligible,
                               const long long* created_ts, long long cutoff, unsigned* candidate_bits,
                               unsigned* decision_bits, unsigned long long* counts) {
  try {
    uint64_t c[3] = {counts[0], counts[1], counts[2]};
    const gph::GroupFixup fx = gph::resolve_sum_by_groups(
        g_last_window, series_max, veto_bits, eligible, reinterpret_cast<const int64_t*>(created_ts), cutoff,
        candidate_bits, decision_bits, &c[0], &c[1], &c[2]);
    counts[0] = c[0], counts[1] = c[1], counts[2] = c[2];
    return (int)fx.pods_changed;
  } catch (const std::exception&) {
    return -1;
  }
}
// value Prometheus reports for every `sum by` group of the last window (NaN for rows that do not start a group
// or groups without an element), [P][G] like series_max
GPH_API int gph_group_values(const float* series_max, double* out) {
  const gph::Window& w = g_last_window;
  for (uint32_t p = 0; p < w.P; ++p)
    for (uint32_t g = 0; g < w.G; ++g)
      out[(size_t)p * w.G + g] = g < w.pods[p].slots.size() && w.pods[p].slots[g].group == g
                                     ? gph::group_value(w, series_max, p, g)
                                     : std::numeric_limits<double>::quiet_NaN();
  return 0;
}

// the engine's group table (gpr_window.groups) of the last window, for `pods` pods (>= P: head-room rows lead
// themselves): pods * G entries
GPH_API int gph_group_table(unsigned pods, unsigned* out) {
  const std::vector<uint32_t> t = gph::group_table(g_last_window, pods);
  std::copy(t.begin(), t.end(), out);
  return 0;
}

// owner walk over a fixture directory: pod_meta_json = the pod's .metadata.  JSON out:
// {"kind":..,"name":..,"namespace":..,"uid":..,"apiVersion":..,"calls":n} or {"error":..}
GPH_API int gph_find_root(const char* fixture_dir, const char* pod_meta_json, char* out, int cap) {
  try {
    gph::FixtureKubeApi api(fixture_dir);
    gph::RootResult r = gph::find_root_object(api, gph::Json::parse(pod_meta_json));
    gph::Json j = gph::Json::object();
    if (r.root) {
      j.set("kind", r.root->kind_name()), j.set("name", r.root->name());
      j.set("namespace", r.root->ns() ? gph::Json(*r.root->ns()) : gph::Json());
      j.set("uid", r.root->uid() ? gph::Json(*r.root->uid()) : gph::Json());
      j.set("apiVersion", r.root->api_version());
      j.set("resourceVersion", r.root->resource_version() ? gph::Json(*r.root->resource_version()) : gph::Json());
      j.set("resource_kind", (int64_t)r.root->resource_kind());
    } else {
      j.set("error", r.error);
    }
    j.set("calls", (int64_t)api.calls);
    return put(j.dump(), out, cap);
  } catch (const std::exception& e) {
    return put(std::string("{\"error\":\"") + gph::json_escape(e.what()) + "\"}", out, cap);
  }
}

static bool kind_from(const std::string& k, gph::Kind* out) {
  if (k == "Deployment") *out = gph::Kind::Deployment;
  else if (k == "ReplicaSet") *out = gph::Kind::ReplicaSet;
  else if (k == "StatefulSet") *out = gph::Kind::StatefulSet;
  else if (k == "InferenceService") *out = gph::Kind::InferenceService;
  else if (k == "Notebook") *out = gph::Kind::Notebook;
  else return false;
  return true;
}

// requests that ScaleKind::scale would send, with a fixed clock / uuid for reproducible tests
GPH_API int gph_scale_requests(const char* kind, const char* object_json, long long now_ns,
                               const char* uuid, const char* pod_name_env, char* out, int cap) {
  try {
    gph::Kind k;
    if (!kind_from(kind, &k)) return -1;
    gph::ScaleKind sk{k, gph::Json::parse(object_json)};
    gph::Clock c;
    c.now_ns = [now_ns] { return (int64_t)now_ns; };
    std::string u = uuid;
    c.uuid_simple = [u] { return u; };
    gph::Json arr = gph::Json::array();
    for (const gph::Request& rq : gph::scale_requests(sk, c, pod_name_env ? pod_name_env : "")) {
      gph::Json j = gph::Json::object();
      j.set("method", rq.method), j.set("path", rq.path), j.set("contentType", rq.content_type);
      j.set("body", rq.body);
      arr.push(j);
    }
    return put(arr.dump(), out, cap);
  } catch (const std::exception&) {
    return -2;
  }
}

// ScaleKind Eq / Hash (lib.rs:45-82): 1 if equal, 0 if not; hashes written to h[2]
GPH_API int gph_scalekind_eq(const char* kind_a, const char* obj_a, const char* kind_b, const char* obj_b,
                             unsigned long long* h) {
  try {
    gph::Kind ka, kb;
    if (!kind_from(kind_a, &ka) || !kind_from(kind_b, &kb)) return -1;
    gph::ScaleKind a{ka, gph::Json::parse(obj_a)}, b{kb, gph::Json::parse(obj_b)};
    if (h) h[0] = a.hash(), h[1] = b.hash();
    return a == b ? 1 : 0;
  } catch (const std::exception&) {
    return -2;
  }
}

GPH_API int gph_rfc3339(long long ns, char* out, int cap) { return put(gph::rfc3339(ns), out, cap); }
GPH_API long long gph_parse_rfc3339(const char* s) {
  try {
    return gph::parse_rfc3339(s);
  } catch (const std::exception&) {
    return -1;
  }
}

// Event that generate_scale_event builds (lib.rs:388-427)
GPH_API int gph_generate_event(const char* kind, const char* object_json, long long now_ns,
                               const char* uuid, const char* pod_name_env, char* out, int cap) {
  try {
    gph::Kind k;
    if (!kind_from(kind, &k)) return -1;
    gph::ScaleKind sk{k, gph::Json::parse(object_json)};
    gph::Clock c = gph::system_clock();
    if (now_ns) c.now_ns = [now_ns] { return (int64_t)now_ns; };
    if (uuid && *uuid) {
      std::string u = uuid;
      c.uuid_simple = [u] { return u; };
    }
    return put(gph::generate_scale_event(sk, c, pod_name_env ? pod_name_env : "").dump(), out, cap);
  } catch (const std::exception&) {
    return -2;
  }
}

// ---- controller under test: one tick with RECORDED verdicts -----------------------------------------
// The product engine is libgpr (gpr_engine.cpp) and is not linked into this test library.  Here the
// test supplies the verdict arrays (computed by the CPU oracle on the ingested window) so that the
// gates / owner walk / dedup / request emission of Controller::run_query_and_scale can run on CPU.
namespace {
class ScriptedEngine : public gph::VerdictEngine {
 public:
  gph::Verdict verdict;
  bool fail = false;
  gph::VerdictRequest last;
  std::vector<uint8_t> eligible_seen;
  std::vector<int64_t> created_seen;
  bool decide(const gph::VerdictRequest& rq, gph::Verdict* out, std::string* error) override {
    last = rq;
    const uint32_t P = rq.window->P;
    if (rq.eligible) eligible_seen.assign(rq.eligible, rq.eligible + P);
    if (rq.created_ts) created_seen.assign(rq.created_ts, rq.created_ts + P);
    if (fail) {
      *error = "scripted failure";
      return false;
    }
    *out = verdict;
    // the fused gate (main.rs:473-510) is part of the verdict: apply it to the recorded candidates
    const uint32_t W = (P + 31) / 32;
    out->decision_bits.assign(W, 0);
    out->n_decisions = 0;
    for (uint32_t p = 0; p < P; ++p) {
      const bool cand = (verdict.candidate_bits[p >> 5] >> (p & 31)) & 1u;
      const bool elig = (!rq.eligible || rq.eligible[p]) && !(rq.created_ts && rq.created_ts[p] >= rq.cutoff_ts);
      if (cand && elig) out->decision_bits[p >> 5] |= 1u << (p & 31), ++out->n_decisions;
    }
    return true;
  }
};
}  // namespace

// args: CLI argv (NUL separated).  candidate_bits / series_max / n_series are the recorded verdict for
// the window the controller will ingest from --prometheus-url file://...  Output JSON:
// {"ok":..,"error":..,"num_pods":..,"shutdown_events":..,"unique_pods":[..],"requests":[..],
//  "eligible":[..],"cutoff":..,"power_on":..}
GPH_API int gph_run_tick(const char* args, int n, const unsigned* candidate_bits, const float* series_max,
                         unsigned long long n_series, int fail, const char* log_path, char* out, int cap) {
  try {
    gph::ParseOutcome po = gph::parse_cli(split_args(args, n));
    if (!po.ok) return put(po.message, out, cap) >= 0 ? -1 : -2;
    const gph::Cli& cli = po.cli;
    std::unique_ptr<gph::FixtureKubeApi> kube;
    if (cli.kube_fixture) kube = std::make_unique<gph::FixtureKubeApi>(*cli.kube_fixture);
    FILE* lf = log_path && *log_path ? fopen(log_path, "w") : nullptr;
    gph::Logger log(cli.log_format, lf ? lf : stderr);
    ScriptedEngine eng;
    eng.fail = fail != 0;
    gph::Json j = gph::Json::object();
    std::unique_ptr<gph::WindowSource> src = gph::make_window_source(cli.prometheus_url);
    gph::Window w;
    try {
      w = src->fetch(cli);
    } catch (const std::exception& e) {
      j.set("ok", false), j.set("error", std::string(e.what()));
      if (lf) fclose(lf);
      return put(j.dump(), out, cap);
    }
    const uint32_t W = (w.P + 31) / 32;
    eng.verdict.candidate_bits.assign(candidate_bits, candidate_bits + W);
    eng.verdict.decision_bits.assign(W, 0);
    eng.verdict.series_max.assign(series_max, series_max + (size_t)w.P * w.G);
    eng.verdict.n_series = n_series;
    for (uint32_t k = 0; k < W; ++k) eng.verdict.n_candidates += (uint64_t)__builtin_popcount(candidate_bits[k]);
    gph::Clock clock = gph::system_clock();
    clock.uuid_simple = [] { return std::string("00000000000040008000000000000000"); };
    gph::Controller ctl(cli, kube.get(), &eng, log, clock);
    gph::TickResult tr = ctl.run_query_and_scale(w);
    if (lf) fclose(lf);
    j.set("ok", tr.ok), j.set("error", tr.error);
    j.set("num_pods", (int64_t)tr.qr.num_pods), j.set("shutdown_events", (int64_t)tr.qr.shutdown_events);
    gph::Json ups = gph::Json::array();
    for (const gph::PodMetricData& p : tr.unique_pods) {
      gph::Json o = gph::Json::object();
      o.set("name", p.name), o.set("namespace", p.ns), o.set("container", p.container);
      o.set("node_type", p.node_type), o.set("gpu_model", p.gpu_model), o.set("value", p.value);
      ups.push(o);
    }
    j.set("unique_pods", ups);
    gph::Json roots = gph::Json::array();
    for (const gph::ScaleKind& sk : tr.shutdown) {
      gph::Json o = gph::Json::object();
      o.set("kind", sk.kind_name()), o.set("name", sk.name());
      roots.push(o);
    }
    j.set("roots", roots);
    gph::Json reqs = gph::Json::array();
    for (const gph::Request& rq : tr.requests) {
      gph::Json o = gph::Json::object();
      o.set("method", rq.method), o.set("path", rq.path), o.set("contentType", rq.content_type);
      o.set("body", rq.body);
      reqs.push(o);
    }
    j.set("requests", reqs);
    gph::Json el = gph::Json::array();
    for (uint8_t e : eng.eligible_seen) el.push((int)e);
    j.set("eligible", el);
    j.set("cutoff", (int64_t)eng.last.cutoff_ts), j.set("power_on", eng.last.power_on);
    j.set("power_threshold", eng.last.power_threshold);
    gph::Json pods = gph::Json::array();
    for (const gph::PodEntry& pe : w.pods) pods.push(pe.name);
    j.set("pods", pods);
    j.set("shape", gph::Json::array());
    return put(j.dump(), out, cap);
  } catch (const std::exception& e) {
    return put(std::string("{\"ok\":false,\"error\":\"") + gph::json_escape(e.what()) + "\"}", out, cap);
  }
}

// Synthetic range-query response in Prometheus' compact encoding, written at memory speed (for the
// ingest benchmarks: P pods x G GPUs, n samples each ending at t_end, DCGM-like integer percentages with
// ~60 % idle series).  Returns the number of bytes written, or -needed if `cap` is too small.
GPH_API long long gph_synth_response(unsigned P, unsigned G, unsigned n, long long t_end, unsigned long long seed,
                                     char* out, long long cap) {
  auto mix = [](unsigned long long x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
  };
  const long long need = 64 + (long long)P * G * (260 + (long long)n * 19);
  if (!out || cap < need) return -need;
  char* p = out;
  auto lit = [&](const char* s) {
    const size_t k = strlen(s);
    memcpy(p, s, k), p += k;
  };
  auto num = [&](unsigned long long v) {
    char tmp[24];
    int k = 0;
    do tmp[k++] = (char)('0' + v % 10), v /= 10; while (v);
    while (k) *p++ = tmp[--k];
  };
  lit("{\"status\":\"success\",\"data\":{\"resultType\":\"matrix\",\"result\":[");
  for (unsigned pod = 0; pod < P; ++pod)
    for (unsigned g = 0; g < G; ++g) {
      if (pod || g) *p++ = ',';
      lit("{\"metric\":{\"__name__\":\"DCGM_FI_DEV_GPU_UTIL\",\"Hostname\":\"node-"), num(pod % 512);
      lit("\",\"UUID\":\"GPU-"), num(pod), *p++ = '-', num(g);
      lit("\",\"device\":\"nvidia"), num(g), lit("\",\"exported_container\":\"main\",\"exported_namespace\":\"ns-");
      num(pod % 64), lit("\",\"exported_pod\":\"pod-"), num(pod), lit("\",\"gpu\":\""), num(g);
      lit("\",\"instance\":\"10.0.0.1:9400\",\"job\":\"dcgm\",\"modelName\":\"NVIDIA B200\"},\"values\":[");
      const unsigned long long hs = mix(seed ^ ((unsigned long long)pod * G + g));
      const bool idle = hs % 100 < 60;
      for (unsigned i = 0; i < n; ++i) {
        if (i) *p++ = ',';
        const unsigned long long t_abs = (unsigned long long)(t_end - (long long)n + 1 + i);
        *p++ = '[', num(t_abs), lit(",\"");
        const unsigned long long hc = mix(hs ^ t_abs);  // a function of absolute time: slices of one timeline agree
        num(idle ? 0 : ((hc >> 10) & 1 ? 1 + (hc >> 11) % 100 : 0));
        lit("\"]");
      }
      lit("]}");
    }
  lit("]}}");
  return (long long)(p - out);
}
