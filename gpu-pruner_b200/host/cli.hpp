// cli.hpp — the controller's command line, flag for flag as the reference declares it
// (gpu-pruner/src/main.rs:46-134, clap derive).  Names, short forms, defaults
// and enum spellings are the surface a user of the reference relies on.
#pragma once
#include <cstdint>
#include <optional>
#include <string>
#include <vector>

namespace gph {

enum class Mode { ScaleDown, DryRun };            // main.rs:121-126, kebab-case on the wire
enum class LogFormat { Json, Default, Pretty };   // main.rs:128-134
enum class TlsMode { Skip, Verify };              // lib.rs:233-238

struct Cli {
  int64_t duration = 30;                      // -t, --duration            minutes   (main.rs:48-50)
  bool daemon_mode = false;                   // -d, --daemon-mode                    (main.rs:52-54)
  std::string enabled_resources = "drsin";    // -e, --enabled-resources             (main.rs:56-64)
  uint64_t check_interval = 180;              // -c, --check-interval      seconds   (main.rs:66-68)
  std::optional<std::string> ns;              // -n, --namespace           regex     (main.rs:70-72)
  int64_t grace_period = 300;                 // -g, --grace-period        seconds   (main.rs:74-76)
  std::optional<std::string> model_name;      // -m, --model-name          regex     (main.rs:78-80)
  std::optional<double> power_threshold;      //     --power-threshold     watts     (main.rs:82-86)
  bool honor_labels = false;                  //     --honor-labels                   (main.rs:88-92)
  Mode run_mode = Mode::DryRun;               // -r, --run-mode                       (main.rs:94-96)
  std::string prometheus_url;                 //     --prometheus-url      required  (main.rs:98-101)
  std::optional<std::string> prometheus_token;//     --prometheus-token (parsed, unused: main.rs:103-107)
  TlsMode prometheus_tls_mode = TlsMode::Verify;  // --prometheus-tls-mode           (main.rs:109-110)
  std::optional<std::string> prometheus_tls_cert; // --prometheus-tls-cert           (main.rs:112-114)
  LogFormat log_format = LogFormat::Default;  // -l, --log-format                     (main.rs:116-118)

  // ---- extensions of this build (no counterpart in the reference) -------------------------
  std::optional<std::string> kube_fixture;    // --kube-fixture DIR: JSON objects instead of an API server
  std::optional<std::string> patch_out;       // --patch-out FILE: where scale-down requests are written
  bool print_query = false;                   // --print-query: render the legacy PromQL and exit
  int gpu_device = 0;                         // --gpu-device N
  int64_t now_override = 0;                   // --now UNIX_SECONDS (tests): 0 = wall clock
  int max_ticks = 0;                          // --max-ticks N (tests): stop the daemon loop after N ticks
  std::optional<std::string> snapshot_file;   // --snapshot-file PATH (-d only): save the resident window after every
                                              // tick, resume from it at start (DESIGN.md §8i)
  bool reshape_ring = false;                  // --reshape-ring (-d only): a tick whose cluster outgrew the resident
                                              // window's shape reshapes it on the GPU instead of querying the full
                                              // range (DESIGN.md §8e)
  bool retime_ring = false;                   // --retime-ring (-d only): a tick whose query step grew by a whole factor,
                                              // or whose --duration got shorter, retimes the resident window on the GPU
                                              // instead of querying the full range (DESIGN.md §8e)
  int64_t query_slice = 0;                    // --query-slice SECONDS: a range longer than this is asked as consecutive
                                              // queries of at most this length, merged into the resident window on the
                                              // GPU (DESIGN.md §8e); 0 = one query per range
  int64_t late_seconds = 0;                   // --late-seconds L (-d only): every delta tick asks again for the newest L
                                              // seconds of the resident window, so samples that reach the server up to
                                              // L s late still count (DESIGN.md §8e); 0 = off
};

struct ParseOutcome {
  bool ok = false;
  int exit_code = 0;        // 0 for --help, 2 for usage errors (clap's convention)
  std::string message;      // help text or error
  Cli cli;
};

ParseOutcome parse_cli(const std::vector<std::string>& args);  // args exclude argv[0]
std::string usage();
const char* to_string(Mode m);
const char* to_string(LogFormat f);
const char* to_string(TlsMode t);

}  // namespace gph
