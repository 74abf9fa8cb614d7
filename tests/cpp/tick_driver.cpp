// TEST INFRASTRUCTURE.  One tick of the gpu-pruner binary — the same objects main.cpp builds (CLI, fixture kube,
// libgpr engine with its device ingest, file:// window source, Controller) — that prints what the tick decided,
// including the PodMetricData rows the binary keeps to itself (main.rs:419-437 never logs them):
//   {"ok":..,"error":..,"num_pods":..,"unique_pods":[{"name","namespace","container","node_type","gpu_model","value"}],
//    "shutdown":[..]}
// usage: tick_driver <gpu-pruner arguments>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "cli.hpp"
#include "controller.hpp"
#include "json.hpp"
#include "kube.hpp"

int main(int argc, char** argv) {
  std::vector<std::string> args(argv + 1, argv + argc);
  gph::ParseOutcome po = gph::parse_cli(args);
  if (!po.ok) {
    fputs(po.message.c_str(), stderr);
    return 2;
  }
  const gph::Cli& cli = po.cli;
  gph::Logger log(cli.log_format, stderr);
  std::unique_ptr<gph::FixtureKubeApi> kube;
  if (cli.kube_fixture) kube = std::make_unique<gph::FixtureKubeApi>(*cli.kube_fixture);
  std::unique_ptr<gph::VerdictEngine> engine = gph::make_gpr_engine();
  std::unique_ptr<gph::WindowSource> src = gph::make_window_source(cli.prometheus_url, engine->text_ingestor(), &log);
  gph::Controller ctl(cli, kube.get(), engine.get(), log, gph::system_clock());
  gph::Json out = gph::Json::object();
  try {
    const gph::Window w = src->fetch(cli);
    const gph::TickResult tr = ctl.run_query_and_scale(w);
    out.set("ok", tr.error.empty());
    out.set("error", tr.error);
    out.set("num_pods", (int64_t)tr.qr.num_pods);
    gph::Json ups = gph::Json::array();
    for (const gph::PodMetricData& p : tr.unique_pods) {
      gph::Json o = gph::Json::object();
      o.set("name", p.name), o.set("namespace", p.ns), o.set("container", p.container);
      o.set("node_type", p.node_type), o.set("gpu_model", p.gpu_model), o.set("value", p.value);
      ups.push(o);
    }
    out.set("unique_pods", ups);
    gph::Json sd = gph::Json::array();
    for (const gph::ScaleKind& sk : tr.shutdown) sd.push(gph::Json(sk.name()));
    out.set("shutdown", sd);
  } catch (const std::exception& e) {
    out.set("ok", false);
    out.set("error", std::string(e.what()));
  }
  printf("%s\n", out.dump().c_str());
  return 0;
}
