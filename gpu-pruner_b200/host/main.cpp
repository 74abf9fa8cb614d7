// gpu-pruner — C++ host of the H100 idle-decision engine, with the reference controller's
// command-line surface (gpu-pruner/src/main.rs:46-134, 273-375).
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

#include "cli.hpp"
#include "controller.hpp"
#include "kube.hpp"
#include "promql.hpp"
#include "snapshot.hpp"

int main(int argc, char** argv) {
  std::vector<std::string> args(argv + 1, argv + argc);
  gph::ParseOutcome po = gph::parse_cli(args);
  if (!po.ok) {
    fputs(po.message.c_str(), po.exit_code == 0 ? stdout : stderr);
    return po.exit_code;
  }
  const gph::Cli& cli = po.cli;
  if (cli.print_query) {  // the text the reference logs as "Running w/ Query: ..." (main.rs:282)
    fputs(gph::render_query(cli).c_str(), stdout);
    return 0;
  }
  gph::Logger log(cli.log_format, stderr);
  log.info("Enabled resources: " + std::to_string((int)gph::get_enabled_resources(cli.enabled_resources)));
  log.info("Running w/ Query: " + gph::render_query(cli));
  const gph::Selectors sel = gph::render_selectors(cli);
  log.info("Engine selectors: " + sel.util + (sel.power.empty() ? "" : " ; " + sel.power));

  std::unique_ptr<gph::FixtureKubeApi> kube;
  if (cli.kube_fixture) kube = std::make_unique<gph::FixtureKubeApi>(*cli.kube_fixture);
  std::unique_ptr<gph::VerdictEngine> engine = gph::make_gpr_engine();   // libgpr.so; no CPU fallback
  // The response text is parsed on the GPU straight into HBM (ingest_device.hpp); responses that are not
  // in Prometheus' compact encoding fall back to the CPU text parser by themselves.  GPR_INGEST=cpu forces
  // the threaded CPU text parser (window uploaded by gpr_decide) for comparison.
  const char* ing = getenv("GPR_INGEST");
  std::unique_ptr<gph::TextIngestor> cpu_ingestor;
  gph::TextIngestor* ingestor = engine->text_ingestor();
  if (ing && std::string(ing) == "cpu") cpu_ingestor = gph::make_cpu_text_ingestor(), ingestor = cpu_ingestor.get();
  // --query-slice merges the slices into the resident window on the GPU; the CPU ingest asks for whole ranges
  gph::Cli run = cli;
  if (cpu_ingestor && run.query_slice > 0) {
    log.warn("--query-slice ignored: slicing needs the device ingest (GPR_INGEST=cpu asks for whole ranges)");
    run.query_slice = 0;
  }
  if (cpu_ingestor && run.late_seconds > 0) {
    log.warn("--late-seconds ignored: GPR_INGEST=cpu keeps no resident window and asks for the full range every tick");
    run.late_seconds = 0;
  }
  if (cpu_ingestor && run.retime_ring) {
    log.warn("--retime-ring ignored: GPR_INGEST=cpu keeps no resident window and asks for the full range every tick");
    run.retime_ring = false;
  }
  std::unique_ptr<gph::WindowSource> src = gph::make_window_source(cli.prometheus_url, ingestor, &log);
  gph::Controller ctl(run, kube.get(), engine.get(), log, gph::system_clock());
  // --snapshot-file: the resident window survives a restart (snapshot.hpp).  The CPU ingest keeps no resident window,
  // so there is nothing to save: said once, and the run is the one without the flag.
  std::unique_ptr<gph::WindowSnapshots> snapshots;
  if (cli.snapshot_file) {
    std::string why;
    if (!ingestor->resident_session(cli, &why)) {
      log.warn("--snapshot-file ignored: snapshots need the device ingest (" + why + ")");
    } else {
      gph::SnapshotKey key;
      key.span = cli.duration * 60;
      const bool want_power = cli.power_threshold && *cli.power_threshold != 0.0;
      key.power_threshold = want_power ? *cli.power_threshold : 0.0;   // as FileSource ingests the power plane
      key.selectors[0] = sel.util, key.selectors[1] = sel.prof, key.selectors[2] = sel.power;
      snapshots = gph::make_file_snapshots(*cli.snapshot_file, key, [ingestor, &cli](std::string* error) {
        return ingestor->resident_session(cli, error);
      }, run.retime_ring);
      ctl.use_snapshots(snapshots.get());
    }
  }
  return ctl.run(*src);
}
