// cli.cpp — hand-written parser with clap's observable behaviour for the flags of
// gpu-pruner/src/main.rs:46-119: `-t 30`, `-t30`, `--duration 30`,
// `--duration=30`, boolean switches, kebab-case enum values, a required --prometheus-url,
// exit code 2 with an "error: ..." message on misuse, exit code 0 for -h/--help.
#include "cli.hpp"

#include <cerrno>
#include <climits>
#include <cstdlib>
#include <functional>
#include <map>

namespace gph {

const char* to_string(Mode m) { return m == Mode::ScaleDown ? "scale-down" : "dry-run"; }
const char* to_string(LogFormat f) {
  return f == LogFormat::Json ? "json" : f == LogFormat::Pretty ? "pretty" : "default";
}
const char* to_string(TlsMode t) { return t == TlsMode::Skip ? "skip" : "verify"; }

std::string usage() {
  return
      "`gpu-pruner` is a tool to prune idle pods based on GPU utilization. It uses Prometheus to query\n"
      "GPU utilization metrics and scales down pods that have been idle for a certain duration.\n\n"
      "Usage: gpu-pruner [OPTIONS] --prometheus-url <PROMETHEUS_URL>\n\n"
      "Options:\n"
      "  -t, --duration <DURATION>                  time in minutes of no gpu activity to use for pruning [default: 30]\n"
      "  -d, --daemon-mode                          daemon mode to run in, if true, will run indefinitely\n"
      "  -e, --enabled-resources <ENABLED_RESOURCES>  d Deployment, r ReplicaSet, s StatefulSet, i InferenceService, n Notebook [default: drsin]\n"
      "  -c, --check-interval <CHECK_INTERVAL>      interval in seconds to check for idle pods, only used in daemon mode [default: 180]\n"
      "  -n, --namespace <NAMESPACE>                namespace to use for search filter (pattern match)\n"
      "  -g, --grace-period <GRACE_PERIOD>          Seconds of grace period to allow for metrics to be published [default: 300]\n"
      "  -m, --model-name <MODEL_NAME>              model name of GPU to use for filter, eg. \"NVIDIA A10G\" (pattern match)\n"
      "      --power-threshold <POWER_THRESHOLD>    Power draw threshold in watts (veto for idle candidates)\n"
      "      --honor-labels                         ServiceMonitor uses honorLabels: true (pod/namespace/container labels)\n"
      "  -r, --run-mode <RUN_MODE>                  [default: dry-run] [possible values: scale-down, dry-run]\n"
      "      --prometheus-url <PROMETHEUS_URL>      Prometheus URL; this build reads recorded range-query responses from file://DIR\n"
      "      --prometheus-token <PROMETHEUS_TOKEN>  Prometheus token (accepted for compatibility)\n"
      "      --prometheus-tls-mode <MODE>           [default: verify] [possible values: skip, verify]\n"
      "      --prometheus-tls-cert <CERT>           Custom .crt file to use for TLS verification\n"
      "  -l, --log-format <LOG_FORMAT>              [default: default] [possible values: json, default, pretty]\n"
      "      --kube-fixture <DIR>                   (extension) Kubernetes objects as JSON files instead of an API server\n"
      "      --patch-out <FILE>                     (extension) write scale-down requests here as JSON lines\n"
      "      --print-query                          (extension) print the rendered PromQL and exit\n"
      "      --gpu-device <N>                       (extension) CUDA device ordinal [default: 0]\n"
      "      --snapshot-file <PATH>                 (extension) with -d: save the resident window after every tick, resume from it at start\n"
      "      --reshape-ring                         (extension) with -d: reshape the resident window on the GPU when pods or GPU slots outgrow it\n"
      "      --retime-ring                          (extension) with -d: retime the resident window on the GPU when the query step grows by a whole factor or --duration shrinks\n"
      "      --query-slice <SECONDS>                (extension) ask ranges longer than this as consecutive queries of at most this length, merged on the GPU; no CPU-parser fallback for slices [default: 0 = one query]\n"
      "      --late-seconds <SECONDS>               (extension) with -d: ask every tick again for the newest SECONDS of the resident window, so samples that reach Prometheus late still count [default: 0 = off]\n"
      "  -h, --help                                 Print help\n";
}

namespace {

struct Spec {
  char short_name;            // 0 = none
  bool takes_value;
  std::function<std::string(const std::string&)> set;  // returns error text or ""
};

std::string parse_i64(const std::string& v, int64_t* out) {
  errno = 0;
  char* end = nullptr;
  long long x = strtoll(v.c_str(), &end, 10);
  if (v.empty() || *end || errno) return "invalid digit found in string";
  *out = x;
  return "";
}
std::string parse_u64(const std::string& v, uint64_t* out) {
  if (!v.empty() && v[0] == '-') return "invalid digit found in string";
  errno = 0;
  char* end = nullptr;
  unsigned long long x = strtoull(v.c_str(), &end, 10);
  if (v.empty() || *end || errno) return "invalid digit found in string";
  *out = x;
  return "";
}
std::string parse_f64(const std::string& v, double* out) {
  errno = 0;
  char* end = nullptr;
  double x = strtod(v.c_str(), &end);
  if (v.empty() || *end) return "invalid float literal";
  *out = x;
  return "";
}

}  // namespace

ParseOutcome parse_cli(const std::vector<std::string>& args) {
  ParseOutcome out;
  Cli& c = out.cli;
  bool have_url = false;

  std::map<std::string, Spec> specs;
  auto enum_err = [](const std::string& v, const char* choices) {
    return "invalid value '" + v + "' [possible values: " + choices + "]";
  };
  specs["duration"] = {'t', true, [&](const std::string& v) { return parse_i64(v, &c.duration); }};
  specs["daemon-mode"] = {'d', false, [&](const std::string&) { c.daemon_mode = true; return std::string(); }};
  specs["enabled-resources"] = {'e', true, [&](const std::string& v) { c.enabled_resources = v; return std::string(); }};
  specs["check-interval"] = {'c', true, [&](const std::string& v) { return parse_u64(v, &c.check_interval); }};
  specs["namespace"] = {'n', true, [&](const std::string& v) { c.ns = v; return std::string(); }};
  specs["grace-period"] = {'g', true, [&](const std::string& v) { return parse_i64(v, &c.grace_period); }};
  specs["model-name"] = {'m', true, [&](const std::string& v) { c.model_name = v; return std::string(); }};
  specs["power-threshold"] = {0, true, [&](const std::string& v) {
    double d = 0.0;
    std::string e = parse_f64(v, &d);
    if (e.empty()) c.power_threshold = d;
    return e;
  }};
  specs["honor-labels"] = {0, false, [&](const std::string&) { c.honor_labels = true; return std::string(); }};
  specs["run-mode"] = {'r', true, [&](const std::string& v) {
    if (v == "scale-down") c.run_mode = Mode::ScaleDown;
    else if (v == "dry-run") c.run_mode = Mode::DryRun;
    else return enum_err(v, "scale-down, dry-run");
    return std::string();
  }};
  specs["prometheus-url"] = {0, true, [&](const std::string& v) { c.prometheus_url = v; have_url = true; return std::string(); }};
  specs["prometheus-token"] = {0, true, [&](const std::string& v) { c.prometheus_token = v; return std::string(); }};
  specs["prometheus-tls-mode"] = {0, true, [&](const std::string& v) {
    if (v == "skip") c.prometheus_tls_mode = TlsMode::Skip;
    else if (v == "verify") c.prometheus_tls_mode = TlsMode::Verify;
    else return enum_err(v, "skip, verify");
    return std::string();
  }};
  specs["prometheus-tls-cert"] = {0, true, [&](const std::string& v) { c.prometheus_tls_cert = v; return std::string(); }};
  specs["log-format"] = {'l', true, [&](const std::string& v) {
    if (v == "json") c.log_format = LogFormat::Json;
    else if (v == "default") c.log_format = LogFormat::Default;
    else if (v == "pretty") c.log_format = LogFormat::Pretty;
    else return enum_err(v, "json, default, pretty");
    return std::string();
  }};
  // extensions
  specs["kube-fixture"] = {0, true, [&](const std::string& v) { c.kube_fixture = v; return std::string(); }};
  specs["patch-out"] = {0, true, [&](const std::string& v) { c.patch_out = v; return std::string(); }};
  specs["print-query"] = {0, false, [&](const std::string&) { c.print_query = true; return std::string(); }};
  specs["gpu-device"] = {0, true, [&](const std::string& v) {
    int64_t x;
    std::string e = parse_i64(v, &x);
    if (e.empty()) c.gpu_device = (int)x;
    return e;
  }};
  specs["snapshot-file"] = {0, true, [&](const std::string& v) { c.snapshot_file = v; return std::string(); }};
  specs["reshape-ring"] = {0, false, [&](const std::string&) { c.reshape_ring = true; return std::string(); }};
  specs["retime-ring"] = {0, false, [&](const std::string&) { c.retime_ring = true; return std::string(); }};
  specs["query-slice"] = {0, true, [&](const std::string& v) {
    uint64_t x = 0;
    std::string e = parse_u64(v, &x);
    if (e.empty() && x > (uint64_t)INT32_MAX) e = "number too large to fit in target type";
    if (e.empty()) c.query_slice = (int64_t)x;
    return e;
  }};
  bool late_given = false;
  specs["late-seconds"] = {0, true, [&](const std::string& v) {
    uint64_t x = 0;
    std::string e = parse_u64(v, &x);
    if (e.empty() && x > (uint64_t)INT32_MAX) e = "number too large to fit in target type";
    if (e.empty()) c.late_seconds = (int64_t)x, late_given = true;
    return e;
  }};
  specs["now"] = {0, true, [&](const std::string& v) { return parse_i64(v, &c.now_override); }};
  specs["max-ticks"] = {0, true, [&](const std::string& v) {
    int64_t x;
    std::string e = parse_i64(v, &x);
    if (e.empty()) c.max_ticks = (int)x;
    return e;
  }};

  std::map<char, std::string> shorts;
  for (auto& kv : specs)
    if (kv.second.short_name) shorts[kv.second.short_name] = kv.first;

  auto fail = [&](const std::string& msg) {
    out.ok = false;
    out.exit_code = 2;
    out.message = "error: " + msg + "\n\nFor more information, try '--help'.\n";
    return out;
  };

  for (size_t i = 0; i < args.size(); ++i) {
    const std::string& a = args[i];
    std::string name, value;
    bool has_inline = false;
    if (a == "-h" || a == "--help") {
      out.ok = false;
      out.exit_code = 0;
      out.message = usage();
      return out;
    }
    if (a.rfind("--", 0) == 0 && a.size() > 2) {
      const size_t eq = a.find('=');
      name = a.substr(2, eq == std::string::npos ? std::string::npos : eq - 2);
      if (eq != std::string::npos) value = a.substr(eq + 1), has_inline = true;
    } else if (a.size() >= 2 && a[0] == '-' && a[1] != '-') {
      auto it = shorts.find(a[1]);
      if (it == shorts.end()) return fail("unexpected argument '-" + std::string(1, a[1]) + "' found");
      name = it->second;
      if (a.size() > 2) {
        if (!specs[name].takes_value) {
          // clustered switches such as -d are the only boolean short; anything after is an error
          return fail("unexpected argument '" + a + "' found");
        }
        value = a.substr(a[2] == '=' ? 3 : 2), has_inline = true;
      }
    } else {
      return fail("unexpected argument '" + a + "' found");
    }
    auto it = specs.find(name);
    if (it == specs.end()) return fail("unexpected argument '--" + name + "' found");
    const Spec& sp = it->second;
    if (sp.takes_value) {
      if (!has_inline) {
        if (i + 1 >= args.size())
          return fail("a value is required for '--" + name + "' but none was supplied");
        value = args[++i];
      }
    } else if (has_inline) {
      return fail("unexpected value '" + value + "' for '--" + name + "' found; no more were expected");
    }
    const std::string err = sp.set(value);
    if (!err.empty()) return fail("invalid value '" + value + "' for '--" + name + "': " + err);
  }
  if (c.snapshot_file && !c.daemon_mode)
    return fail("the argument '--snapshot-file <PATH>' can only be used with '--daemon-mode'");
  if (c.reshape_ring && !c.daemon_mode)
    return fail("the argument '--reshape-ring' can only be used with '--daemon-mode'");
  if (c.retime_ring && !c.daemon_mode)
    return fail("the argument '--retime-ring' can only be used with '--daemon-mode'");
  if (late_given && !c.daemon_mode)
    return fail("the argument '--late-seconds <SECONDS>' can only be used with '--daemon-mode'");
  if (c.late_seconds > 0 && c.late_seconds >= c.duration * 60)
    return fail("invalid value '" + std::to_string(c.late_seconds) + "' for '--late-seconds <SECONDS>': must be less " +
                "than the window (--duration " + std::to_string(c.duration) + " = " + std::to_string(c.duration * 60) +
                " s)");
  if (!have_url && !c.print_query)
    return fail("the following required arguments were not provided:\n  --prometheus-url <PROMETHEUS_URL>");
  out.ok = true;
  return out;
}

}  // namespace gph
