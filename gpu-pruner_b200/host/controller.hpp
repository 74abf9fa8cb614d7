// controller.hpp — the tick: window -> GPU decision -> gates -> owner walk -> scale requests.
//
// C++ mirror of run_query_and_scale and the two tasks around it
// (gpu-pruner/src/main.rs:286-367, 390-570).  The aggregation that the reference
// delegates to Prometheus is done by libgpr (include/gpr.h); everything after it follows the
// reference step by step, with the Kubernetes API behind the KubeApi interface.
#pragma once
#include <cstdint>
#include <functional>
#include <memory>
#include <string>
#include <unordered_set>
#include <vector>

#include "cli.hpp"
#include "ingest.hpp"
#include "kube.hpp"

namespace gph {

class DeviceIngestSession;
struct SlicedFetch;

// lib.rs:136-145
struct PodMetricData {
  std::string name, ns, container, node_type, gpu_model;
  double value = 0;
};
// lib.rs:131-134
struct QueryResponse {
  size_t num_pods = 0;         // series returned by the query, pre-dedup (main.rs:418)
  size_t shutdown_events = 0;  // distinct root objects (main.rs:536)
};

class Logger {
 public:
  Logger(LogFormat f, FILE* out) : fmt_(f), out_(out) {}
  void log(const char* level, const std::string& msg,
           const std::vector<std::pair<std::string, std::string>>& fields = {}) const;
  void info(const std::string& m) const { log("INFO", m); }
  void warn(const std::string& m) const { log("WARN", m); }
  void error(const std::string& m) const { log("ERROR", m); }
  void counter(const char* level, const std::string& name, uint64_t v, const std::string& msg) const;

 private:
  LogFormat fmt_;
  FILE* out_;
};

struct TickResult {
  bool ok = false;
  std::string error;
  QueryResponse qr;
  std::vector<PodMetricData> unique_pods;     // after the ANY-GPU dedup (main.rs:416-437)
  std::vector<ScaleKind> shutdown;            // distinct roots, insertion order
  std::vector<Request> requests;              // what scale-down mode would send
  double kernel_ms = 0;
  uint64_t n_candidates = 0, n_decisions = 0;
};

// The idle decision itself, behind an interface so that the controller logic does not depend on how
// it is produced.  The product implementation is GprVerdictEngine (gpr_engine.cpp: libgpr.so, CUDA,
// no CPU fallback); the test-suite injects recorded verdicts through the C test API to exercise the
// gates / owner walk / dedup / request emission without a GPU.
struct VerdictRequest {
  const Window* window = nullptr;
  const uint8_t* eligible = nullptr;     // [P] or null
  const int64_t* created_ts = nullptr;   // [P] or null
  int64_t cutoff_ts = 0;
  bool power_on = false;
  double power_threshold = 0.0;
  int gpu_device = 0;
};
struct Verdict {
  std::vector<uint32_t> decision_bits, candidate_bits;   // ceil(P/32) words
  std::vector<uint32_t> veto_bits;                       // ceil(P/32) words or empty: pods vetoed by the power clause
  std::vector<float> series_max;                         // [P*G], or empty when groups_resolved
  // groups_resolved: the engine decided on `sum by` groups itself (gpr_window.groups), so the bits and counts are
  // PromQL's already; idle_slots [P][ceil(G/32)] then says which slots start an idle element (gpr_result.idle_slots)
  bool groups_resolved = false;
  std::vector<uint32_t> idle_slots;
  uint64_t n_series = 0, n_candidates = 0, n_decisions = 0;
  double kernel_ms = 0;
};
// Turns the raw range-query responses into a Window.  Default: the threaded CPU text parser
// (ingest_matrix_text).  The product engine also offers one that parses the text on the GPU straight
// into HBM (ingest_device.hpp); selected with GPR_INGEST=gpu.
class TextIngestor {
 public:
  virtual ~TextIngestor() = default;
  virtual Window ingest(const Cli& args, const std::string& util, const std::string* prof, const std::string* power,
                        const IngestOptions& opt, std::string* note) = 0;
  // daemon mode: newest second of the window this ingestor keeps resident between ticks (0 = none: the next
  // tick must bring the full range).  An ingest with opt.slice_seconds > 0 may throw NeedFullWindow.
  virtual int64_t resident_t_end() const { return 0; }
  // --query-slice: the same range asked as several queries, merged into the resident window (ingest_device.hpp
  // DeviceIngestSession::ingest_slices).  An ingestor without a resident window cannot take slices and throws.
  virtual Window ingest_slices(const Cli& args, const SlicedFetch& f, const IngestOptions& opt, std::string* note) {
    (void)args, (void)f, (void)opt, (void)note;
    throw std::runtime_error("this ingestor cannot merge query slices");
  }
  // daemon mode: the session that keeps the window resident, for snapshots (snapshot.hpp); created if need be.
  // nullptr (*error says why): this ingestor keeps no resident window, so there is nothing to snapshot.
  virtual DeviceIngestSession* resident_session(const Cli&, std::string* error) {
    *error = "this ingestor keeps no resident window";
    return nullptr;
  }
};
// --snapshot-file: the resident window saved after every tick and restored at start (snapshot.hpp make_file_snapshots).
class WindowSnapshots {
 public:
  virtual ~WindowSnapshots() = default;
  // before the first fetch: true = the window is resident again; *line says what was restored or why not
  virtual bool restore(std::string* line) = 0;
  // after a successful tick whose window is resident: 1 = written (*line describes it), 0 = nothing resident,
  // -1 = the write failed (*line says why; the previous file is intact)
  virtual int save(std::string* line) = 0;
};
class VerdictEngine {
 public:
  virtual ~VerdictEngine() = default;
  virtual bool decide(const VerdictRequest& rq, Verdict* out, std::string* error) = 0;
  virtual TextIngestor* text_ingestor() { return nullptr; }   // device-side ingest, if the engine has one
};
std::unique_ptr<VerdictEngine> make_gpr_engine();   // gpr_engine.cpp (links libgpr.so)

// Where the window comes from, selected by the scheme of --prometheus-url.
class WindowSource {
 public:
  virtual ~WindowSource() = default;
  virtual Window fetch(const Cli& args) = 0;   // throws std::runtime_error on failure
};
// The default CPU text parser behind the TextIngestor interface, reporting its time the way the device
// ingestor does (GPR_INGEST=cpu; used to compare the two on the same fixtures).
std::unique_ptr<TextIngestor> make_cpu_text_ingestor();
std::unique_ptr<WindowSource> make_window_source(const std::string& url, TextIngestor* ingestor = nullptr,
                                                 const Logger* log = nullptr);

class Controller {
 public:
  Controller(const Cli& args, KubeApi* kube, VerdictEngine* engine, Logger log, Clock clock);
  Controller(const Controller&) = delete;

  // one pass of main.rs:390-570 on an already-fetched window
  TickResult run_query_and_scale(const Window& w);
  // main.rs:286-330: one-shot or daemon loop with the consecutive-failure budget; returns exit code
  int run(WindowSource& src);
  // --snapshot-file: restore before the first fetch, save after every successful tick with a resident window
  void use_snapshots(WindowSnapshots* snapshots) { snapshots_ = snapshots; }

  uint64_t query_successes = 0, query_failures = 0, scale_successes = 0, scale_failures = 0;
  uint64_t snapshot_failures = 0;

 private:
  Cli args_;
  KubeApi* kube_;
  VerdictEngine* engine_;
  Logger log_;
  Clock clock_;
  uint8_t enabled_;
  WindowSnapshots* snapshots_ = nullptr;
};

}  // namespace gph
