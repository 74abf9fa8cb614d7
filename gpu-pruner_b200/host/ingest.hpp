// ingest.hpp — Prometheus range-vector (matrix) wire format -> dense (pod x gpu x t) f32 tensor.
//
// The reference never receives raw samples: it asks Prometheus for the already-aggregated instant
// vector (gpu-pruner/src/main.rs:397-409).  The only reference code that walks a
// matrix result is the debug tool gpu-pruner/src/bin/querytest.rs:41-53
// (series = label map + [(timestamp f64, value)]); that is the shape ingested here.  Label
// precedence follows PodMetricData::try_from (gpu-pruner/src/lib.rs:153-187): exported_* first,
// then the bare name; node_type defaults to "unknown"; modelName is mandatory.
#pragma once
#include <cstdint>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <string>
#include <vector>

#include "json.hpp"

namespace gph {

struct GpuSlot {            // one SERIES of a (Hostname, container, pod, namespace, gpu, modelName) group
  std::string hostname, container, gpu, model, node_type;
  bool from_prof = false;   // row holds DCGM_FI_PROF_GR_ENGINE_ACTIVE (0..1) rather than GPU_UTIL (0..100)
  uint32_t group = 0;       // slot index of the first series of its `sum by` group (== own index: first / only one)
};

struct PodEntry {
  std::string name, ns;
  std::vector<GpuSlot> slots;        // util / prof series, in order of first appearance
  uint32_t power_slots = 0;          // power series (each its own row: `unless` needs no grouping)
  bool has_groups = false;           // some `sum by` group of this pod has more than one series
};

// The pod table of a window.  Copy-on-write: daemon mode hands the controller a Window every tick while the
// ingest session keeps the table for the next one — copying a Window shares the table (10,000 pods x a dozen
// strings would otherwise be duplicated and freed every tick), and whoever writes to a shared table gets its own.
class PodList {
 public:
  size_t size() const { return v_ ? v_->size() : 0; }
  bool empty() const { return size() == 0; }
  const PodEntry& operator[](size_t i) const { return (*v_)[i]; }
  PodEntry& operator[](size_t i) { return mut()[i]; }
  const PodEntry* begin() const { return v_ ? v_->data() : nullptr; }
  const PodEntry* end() const { return v_ ? v_->data() + v_->size() : nullptr; }
  PodEntry* begin() { return mut().data(); }
  PodEntry* end() {
    std::vector<PodEntry>& v = mut();
    return v.data() + v.size();
  }
  PodEntry& emplace_back() {
    mut().emplace_back();
    return v_->back();
  }
  void push_back(PodEntry e) { mut().push_back(std::move(e)); }
  PodEntry& back() { return mut().back(); }
  const PodEntry& back() const { return v_->back(); }

 private:
  std::vector<PodEntry>& mut() {
    if (!v_) v_ = std::make_shared<std::vector<PodEntry>>();
    else if (v_.use_count() > 1) v_ = std::make_shared<std::vector<PodEntry>>(*v_);
    return *v_;
  }
  std::shared_ptr<std::vector<PodEntry>> v_;
};

struct IngestStats {
  uint64_t series_in = 0, series_skipped = 0, samples_in = 0, samples_out_of_window = 0,
           duplicates_merged = 0, tiny_values_clamped = 0;
  std::vector<std::string> warnings;
  // daemon mode with IngestOptions::reshape: what reshaping the resident ring did this tick ("" = it was not reshaped)
  std::string ring_reshape;
  // daemon mode with IngestOptions::retime: what retiming the resident ring did this tick ("" = it was not retimed)
  std::string ring_retime;
  // daemon mode with IngestOptions::reask_seconds: cells of the re-asked buckets whose bits the tick changed, per plane
  // (late samples), and the time spent reading the band before and after the merge
  uint64_t late_util_cells = 0, late_power_cells = 0;
  double band_ms = 0;
};

struct Window {
  uint32_t P = 0, G = 0, T = 0;
  // seconds.  A sample is inside iff t_end - span < ts <= t_end (the [Nm] selector evaluated at t_end,
  // left-open); column c holds the bucket (t_end - (T-c)*step, t_end - (T-1-c)*step], T = ceil(span/step)
  int64_t t_end = 0, step = 1, span = 0;
  PodList pods;
  std::vector<float> util;            // [P][G][T], NaN = no sample
  std::vector<float> power;           // empty, or [P][G][T]
  // device-resident planes (ingest_matrix_device): util / power above are empty then
  const float* d_util = nullptr;
  const float* d_power = nullptr;
  // daemon mode: the window lives in the engine's resident ring (gpr_resident_*); P counts the pods known so
  // far, the ring has room for resident_rows / G of them
  bool resident = false;
  bool resident_power = false;
  uint32_t resident_pods = 0;
  IngestStats stats;
};

struct IngestOptions {
  int64_t duration_min = 30;          // window length, --duration
  int64_t step = 0;                   // seconds; 0 = infer (the most frequent positive timestamp delta)
  int64_t t_end = 0;                  // 0 = newest timestamp in the response
  // daemon mode (main.rs:286-330, --check-interval): > 0 = the responses only cover (t_end - slice_seconds, t_end],
  // what was scraped since the previous tick; the rest of the window is resident in HBM
  int64_t slice_seconds = 0;
  bool resident = false;              // keep the window resident for the following ticks
  // --power-threshold the power plane will be decided with: its samples are stored snapped to it so that the f32
  // veto agrees with Prometheus' float64 `x >= threshold` (include/gpr.h, gpr_window.power_threshold).
  // 0 / NaN = no power clause: plain rounding
  double power_threshold = 0.0;
  // daemon mode (--reshape-ring): a delta tick whose pods outgrow the ring's rows, or whose pod gains a series slot
  // beyond its G, reshapes the ring on the GPU (gpr_resident_live_rows + gpr_resident_remap) instead of throwing
  // NeedFullWindow; pods without a sample left in the window are dropped then
  bool reshape = false;
  // daemon mode (--retime-ring): a delta tick whose step grew by a whole factor, or whose window got shorter on an edge
  // of the old step's buckets, retimes the ring on the GPU (gpr::retime_plan, gpr_resident_retime) instead of throwing
  // NeedFullWindow; every other change of step or window still throws
  bool retime = false;
  // daemon mode (--late-seconds): a delta's responses cover (t_end - slice_seconds - reask_seconds, t_end]: the newest
  // reask_seconds the ring already holds are asked again, so samples that reached the server late are merged in (a
  // NaN-aware max, so a sample seen twice leaves its cell as it was).  Only slice_seconds / step buckets are opened.
  int64_t reask_seconds = 0;
};

// thrown by a delta ingest when the resident state cannot absorb the tick (new GPU slot beyond the ring's shape,
// more pods than it has rows for, a PROF series that stopped reporting, a changed step / window): the caller
// fetches the full window again
struct NeedFullWindow : std::runtime_error {
  using std::runtime_error::runtime_error;
};

// `util` is required; `prof` and `power` may be null pointers.  Each is a full Prometheus HTTP API
// response ({"status":"success","data":{"resultType":"matrix","result":[...]}}) or just the
// "result" array.  Throws std::runtime_error on malformed input / non-matrix result types.
Window ingest_matrix(const Json& util, const Json* prof, const Json* power, const IngestOptions& opt);

// Same result from the raw response TEXT, without building a DOM for the samples: series boundaries
// are found with one memmem per series, label sets go through the small DOM parser, and the sample
// arrays — >99 % of the bytes — are parsed by n_threads workers (0 = hardware concurrency) straight
// into the tensor rows.  This is the path the controller uses; ingest_matrix() is the reference
// implementation it is tested against (tests/test_host.py).
Window ingest_matrix_text(const std::string& util, const std::string* prof, const std::string* power,
                          const IngestOptions& opt, int n_threads = 0);

// `node_dmi_info` enrichment (query.promql.j2:23-34): `dmi` is the response of the instant (or range) query
// `node_dmi_info`; every slot whose Hostname has a DMI series gets that series' product_name as node_type,
// the others keep "unknown" (lib.rs:176-179).  Two DMI series for one Hostname make the reference's query
// fail (many-to-one matching with a duplicate on the "one" side): throws std::runtime_error.
void apply_node_types(Window& w, const Json& dmi);

// Exact `sum by` (query.promql.j2:9,21) for pods with duplicate series.  The tensor keeps every series
// in its own row; the engine's verdict treats every row as an element.  For pods with has_groups this
// re-derives the verdict from the per-series window maxima: element value = compensated float64 sum of
// the members' maxima (UTIL members / 100), element idle iff value == 0, pod candidate iff any element is
// idle and the pod is not vetoed.  Arrays are the engine's outputs, corrected in place; `eligible` /
// `created_ts` / `cutoff` re-apply the gates (main.rs:473-510) for the pods that change.
struct GroupFixup {
  uint64_t pods_examined = 0, pods_changed = 0;
};
GroupFixup resolve_sum_by_groups(const Window& w, const float* series_max, const uint32_t* veto_bits,
                                 const uint8_t* eligible, const int64_t* created_ts, int64_t cutoff,
                                 uint32_t* candidate_bits, uint32_t* decision_bits, uint64_t* n_series,
                                 uint64_t* n_candidates, uint64_t* n_decisions);
// value of the element (group) that slot `slot` of pod `p` starts, from the per-series maxima: what
// Prometheus reports for it (NaN = no element)
double group_value(const Window& w, const float* series_max, uint32_t p, uint32_t slot);
// The same groups as the engine's table (gpr_window.groups, include/gpr.h): [pods][G] entries, bits 0-7 the slot of the
// group's first member, GPR_GROUP_UTIL for a GPU_UTIL member.  Slots beyond a pod's series and pods beyond w.P (the
// head-room rows of a resident ring) lead themselves.  The one place on the host that knows the encoding.
std::vector<uint32_t> group_table(const Window& w, uint32_t pods);

}  // namespace gph
