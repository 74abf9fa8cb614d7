#include "ingest.hpp"

#include <thread>
#include <unordered_map>

#include "ingest_internal.hpp"
#include "../../include/gpr.h"

namespace gph {

using namespace detail;

namespace {

// =====================================================================================================
// DOM path
// =====================================================================================================
const Json& result_array(const Json& resp) {
  if (resp.is_array()) return resp;
  if (resp.is_object()) {
    const Json& st = resp["status"];
    if (st.is_string() && st.as_string() != "success")
      throw std::runtime_error("prometheus response status: " + st.as_string() + " " +
                               resp["error"].as_string());
    const Json& data = resp["data"];
    const Json& rt = data["resultType"];
    if (rt.is_string() && rt.as_string() != "matrix")
      throw std::runtime_error("expected matrix response from prometheus, got " + rt.as_string());
    if (data["result"].is_array()) return data["result"];
  }
  throw std::runtime_error("not a Prometheus matrix response");
}

double sample_value(const Json& v) {
  if (v.is_string()) {  // "NaN", "+Inf", "0.37" — and nothing that is not a number (see strict_sample_value)
    const std::string& t = v.as_string();
    double d;
    if (!detail::strict_sample_value(t.data(), t.data() + t.size(), &d)) detail::bad("sample value is not a number");
    return d;
  }
  return v.as_number(std::numeric_limits<double>::quiet_NaN());
}

struct RawSeries {
  uint32_t pod, slot;
  const Json* values;
};

}  // namespace


Window ingest_matrix(const Json& util, const Json* prof, const Json* power, const IngestOptions& opt) {
  Window w;
  Assigner asg(w);
  std::vector<RawSeries> useries, pseries;
  int64_t newest = kNoTs;
  StepVote vote;

  auto scan = [&](const Json& resp, bool is_power, bool is_prof) {
    for (const Json& s : result_array(resp).items()) {
      ++w.stats.series_in;
      const Json& vals = s["values"];
      uint32_t p, slot;
      if (!vals.is_array() || vals.size() == 0) {  // no sample in range: no element
        // still counts as skipped if it could not have been converted
        continue;
      }
      // Whose samples are read: every series that is placed or skipped (a sample that is not [time, "number"] fails
      // the query as it fails the reference's decode, wherever it sits — in the window or not); a UTIL series shadowed
      // by a PROF series of the same label set is not opened by any of the three ingest paths.
      const Assigner::Result placed = asg.assign(s["metric"], is_power, is_prof, &p, &slot);
      if (placed == Assigner::Shadowed) continue;
      if (placed == Assigner::Placed) (is_power ? pseries : useries).push_back(RawSeries{p, slot, &vals});
      int64_t prev = kNoTs;
      for (const Json& tv : vals.items()) {
        // a sample is exactly [ <unix time>, "<value>" ]; anything else is a malformed response
        // (all paths reject it, the tick then counts as a query failure, main.rs:310-321)
        if (!tv.is_array() || tv.size() != 2 || !tv[0].is_number())
          throw std::runtime_error("matrix response: sample is not [time, value]");
        (void)sample_value(tv[1]);
        if (placed != Assigner::Placed) continue;
        const int64_t ts = ts_seconds(tv[0].as_number());
        if (ts == kBadTs) continue;
        newest = std::max(newest, ts);
        if (prev != kNoTs) vote.add(ts - prev);
        prev = ts;
      }
    }
  };
  if (prof) scan(*prof, false, true);  // PROF first so it wins the `or`
  scan(util, false, false);
  if (power) scan(*power, true, false);
  finish_shape(w, opt, newest, vote.result(), power != nullptr);

  auto place = [&](const std::vector<RawSeries>& list, std::vector<float>& plane, const gpr::text::PowerSnap& snap) {
    for (const RawSeries& rs : list) {
      float* row = plane.data() + ((size_t)rs.pod * w.G + rs.slot) * w.T;
      for (const Json& tv : rs.values->items()) {
        ++w.stats.samples_in;
        const int64_t col = column_of(w, ts_millis(tv[0].as_number()));
        if (col < 0) {
          ++w.stats.samples_out_of_window;
          continue;
        }
        merge_cell(row[col], to_cell(sample_value(tv[1]), snap, &w.stats.tiny_values_clamped));
      }
    }
  };
  place(useries, w.util, gpr::text::power_snap(0.0));
  if (power) place(pseries, w.power, gpr::text::power_snap(opt.power_threshold));
  return w;
}

// =====================================================================================================
// text path: no DOM for the samples.  The response is scanned once for series boundaries (the
// `values` array of a series contains no nested brackets beyond its [ts,"v"] pairs and no escapes,
// so its end is the first "]]"), label sets are parsed with the small DOM parser, and the sample
// arrays — the bulk of the bytes — are parsed by worker threads straight into the tensor rows.

Window ingest_matrix_text(const std::string& util, const std::string* prof, const std::string* power,
                          const IngestOptions& opt, int n_threads) {
  Window w;
  Assigner asg(w);
  std::vector<TextSeries> useries, pseries;
  if (n_threads <= 0) n_threads = (int)std::max(1u, std::thread::hardware_concurrency());

  FlatLabels flat;
  auto scan = [&](const std::string& text, bool is_power, bool is_prof) {
    for (const Span& s : series_spans(text)) {
      ++w.stats.series_in;
      if (!s.values_b || !s.metric_b) continue;
      const char* v = skip_ws(s.values_b + 1, s.values_e);
      if (v < s.values_e && *v == ']') continue;  // no sample in range: no element
      uint32_t p, slot;
      Assigner::Result placed;
      if (flat.parse(s.metric_b, s.metric_e)) {  // Prometheus' own shape: read in place
        placed = asg.assign(flat, is_power, is_prof, &p, &slot);
      } else {
        const Json metric = Json::parse(std::string(s.metric_b, s.metric_e));
        placed = asg.assign(metric, is_power, is_prof, &p, &slot);
      }
      if (placed == Assigner::Placed) {
        (is_power ? pseries : useries).push_back(TextSeries{p, slot, s.values_b, s.values_e, true});
      } else if (placed == Assigner::Skipped) {
        for_each_sample(s.values_b, s.values_e, [](double, double) {});  // no row, but its samples are still vetted
      }
    }
  };
  if (prof) scan(*prof, false, true);
  scan(util, false, false);
  if (power) scan(*power, true, false);

  // pre-pass only when the caller did not say where the window ends / what the step is
  int64_t newest = kNoTs;
  StepVote vote;
  if (opt.t_end <= 0 || opt.step <= 0) {
    auto pre = [&](const std::vector<TextSeries>& list) {
      for (const TextSeries& ts : list) {
        int64_t prev = kNoTs;
        for_each_sample(ts.vb, ts.ve, [&](double t, double) {
          const int64_t ti = ts_seconds(t);
          if (ti == kBadTs) return;
          newest = std::max(newest, ti);
          if (prev != kNoTs) vote.add(ti - prev);
          prev = ti;
        });
      }
    };
    pre(useries);
    pre(pseries);
  }
  finish_shape(w, opt, newest, vote.result(), power != nullptr);

  auto place = [&](std::vector<TextSeries>& list, std::vector<float>& plane, const gpr::text::PowerSnap& snap) {
    // rows written by exactly one series can be filled concurrently; shared rows are merged afterwards
    std::vector<uint32_t> writers((size_t)w.P * w.G, 0);
    for (const TextSeries& ts : list) ++writers[(size_t)ts.pod * w.G + ts.slot];
    for (TextSeries& ts : list) ts.sole = writers[(size_t)ts.pod * w.G + ts.slot] == 1;
    std::vector<IngestStats> st((size_t)n_threads);
    auto work = [&](int tid, bool sole_pass) {
      // thread-local counters (adjacent IngestStats would false-share a cache line per sample)
      uint64_t n_in = 0, n_out = 0, n_tiny = 0;
      for (size_t i = (size_t)tid; i < list.size(); i += (size_t)(sole_pass ? n_threads : 1)) {
        const TextSeries& ts = list[i];
        if (ts.sole != sole_pass) continue;
        float* row = plane.data() + ((size_t)ts.pod * w.G + ts.slot) * w.T;
        for_each_sample(ts.vb, ts.ve, [&](double t, double v) {
          ++n_in;
          const int64_t col = column_of(w, ts_millis(t));
          if (col < 0) {
            ++n_out;
            return;
          }
          merge_cell(row[col], to_cell(v, snap, &n_tiny));
        });
      }
      IngestStats& s = st[(size_t)tid];
      s.samples_in += n_in, s.samples_out_of_window += n_out, s.tiny_values_clamped += n_tiny;
    };
    // a malformed sample array must surface as an exception on the caller's thread, not terminate()
    std::vector<std::string> errors((size_t)n_threads);
    auto guarded = [&](int tid, bool sole_pass) {
      try {
        work(tid, sole_pass);
      } catch (const std::exception& e) {
        errors[(size_t)tid] = e.what();
      }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_threads; ++t) th.emplace_back(guarded, t, true);
    guarded(0, true);
    for (std::thread& t : th) t.join();
    for (const std::string& e : errors)
      if (!e.empty()) throw std::runtime_error(e);
    work(0, false);  // duplicates of one group: sequential, order-independent merge
    for (const IngestStats& s : st) {
      w.stats.samples_in += s.samples_in;
      w.stats.samples_out_of_window += s.samples_out_of_window;
      w.stats.tiny_values_clamped += s.tiny_values_clamped;
    }
  };
  place(useries, w.util, gpr::text::power_snap(0.0));
  if (power) place(pseries, w.power, gpr::text::power_snap(opt.power_threshold));
  return w;
}

// =====================================================================================================
// node_dmi_info join (query.promql.j2:23-34)
//   label_replace(label_replace(node_dmi_info, "Hostname", "$1", "instance", "(.+)"), "node_type", "$1",
//                 "product_name", "(.+)")
//   idle_gpus * on (Hostname) group_left(node_type) (...)  or on (...) idle_gpus
// node_dmi_info has the value 1, so only the label travels.  label_replace leaves the destination label
// untouched when the (fully anchored) regex does not match, i.e. when the source label is empty or absent.
void apply_node_types(Window& w, const Json& dmi) {
  const Json* result = &dmi;
  if (dmi.is_object()) {
    const Json& st = dmi["status"];
    if (st.is_string() && st.as_string() != "success")
      throw std::runtime_error("prometheus response status: " + st.as_string());
    result = &dmi["data"]["result"];
  }
  if (!result->is_array()) throw std::runtime_error("node_dmi_info: not a Prometheus vector / matrix response");
  std::unordered_map<std::string, std::string> by_host;  // Hostname -> node_type ("" = label absent)
  for (const Json& s : result->items()) {
    const Json& m = s["metric"];
    if (!m.is_object()) throw std::runtime_error("node_dmi_info: series without a label map");
    auto str = [&](const char* k) {
      const Json* v = m.find(k);
      return v && v->is_string() ? v->as_string() : std::string();
    };
    const std::string instance = str("instance"), product = str("product_name");
    const std::string host = !instance.empty() ? instance : str("Hostname");
    const std::string node_type = !product.empty() ? product : str("node_type");
    // many-to-one matching: two series with the same `on` signature on the "one" side fail the whole query
    if (!by_host.emplace(host, node_type).second)
      throw std::runtime_error("Failed to run query! found duplicate series for the match group {Hostname=\"" + host +
                               "\"} on the right hand-side of the operation (node_dmi_info)");
  }
  // no DMI series for the host: `or on (...)` restores the element without the label; a DMI series
  // without product_name: group_left copies an absent label.  Both read back as "unknown" (lib.rs:176-179)
  auto type_of = [&](const GpuSlot& g) -> const std::string& {
    static const std::string unknown = "unknown";
    auto it = by_host.find(g.hostname);
    return it != by_host.end() && !it->second.empty() ? it->second : unknown;
  };
  // the pod table may be shared with the ingest session of daemon mode (copy-on-write): write only what changes
  const PodList& current = w.pods;
  for (size_t p = 0; p < current.size(); ++p)
    for (size_t g = 0; g < current[p].slots.size(); ++g)
      if (current[p].slots[g].node_type != type_of(current[p].slots[g])) {
        GpuSlot& slot = w.pods[p].slots[g];
        slot.node_type = type_of(slot);
      }
}

// =====================================================================================================
// exact `sum by` for duplicate series (query.promql.j2:9,21)
namespace {
// Prometheus' `sum` (promql/engine.go, kahanSumInc): Neumaier-compensated float64 sum
struct KahanSum {
  double sum = 0.0, c = 0.0;
  bool any = false;
  void add(double x) {
    any = true;
    const double t = sum + x;
    if (std::isinf(t)) c = 0.0;
    else if (std::fabs(sum) >= std::fabs(x)) c += (sum - t) + x;
    else c += (x - t) + sum;
    sum = t;
  }
  double value() const { return std::isinf(sum) ? sum : sum + c; }
};
}  // namespace

double group_value(const Window& w, const float* series_max, uint32_t p, uint32_t slot) {
  const PodEntry& pe = w.pods[p];
  KahanSum k;
  for (uint32_t g = slot; g < pe.slots.size(); ++g) {
    if (pe.slots[g].group != slot) continue;
    const float m = series_max[(size_t)p * w.G + g];
    if (std::isnan(m)) continue;  // no sample in the window: the series is no element of the instant vector
    // `/ 100` on the UTIL branch happens before the sum (query.promql.j2:20)
    k.add(pe.slots[g].from_prof ? (double)m : (double)m / 100.0);
  }
  return k.any ? k.value() : std::numeric_limits<double>::quiet_NaN();
}

std::vector<uint32_t> group_table(const Window& w, uint32_t pods) {
  std::vector<uint32_t> t((size_t)pods * w.G);
  for (uint32_t p = 0; p < pods; ++p)
    for (uint32_t g = 0; g < w.G; ++g) {
      uint32_t e = g;
      if (p < w.P && g < w.pods[p].slots.size()) {
        const GpuSlot& s = w.pods[p].slots[g];
        e = s.group | (s.from_prof ? 0u : (uint32_t)GPR_GROUP_UTIL);
      }
      t[(size_t)p * w.G + g] = e;
    }
  return t;
}

GroupFixup resolve_sum_by_groups(const Window& w, const float* series_max, const uint32_t* veto_bits,
                                 const uint8_t* eligible, const int64_t* created_ts, int64_t cutoff,
                                 uint32_t* candidate_bits, uint32_t* decision_bits, uint64_t* n_series,
                                 uint64_t* n_candidates, uint64_t* n_decisions) {
  GroupFixup fx;
  for (uint32_t p = 0; p < w.P; ++p) {
    const PodEntry& pe = w.pods[p];
    if (!pe.has_groups) continue;
    ++fx.pods_examined;
    const uint32_t word = p >> 5, bit = 1u << (p & 31);
    const bool veto = veto_bits && (veto_bits[word] & bit);
    // what the engine counted: every idle ROW of a candidate pod
    const bool was_cand = (candidate_bits[word] & bit) != 0, was_dec = (decision_bits[word] & bit) != 0;
    uint64_t rows_idle = 0, groups_idle = 0;
    for (uint32_t g = 0; g < pe.slots.size(); ++g) {
      if (series_max[(size_t)p * w.G + g] == 0.0f) ++rows_idle;
      if (pe.slots[g].group == g && group_value(w, series_max, p, g) == 0.0) ++groups_idle;
    }
    const bool cand = groups_idle > 0 && !veto;
    const bool dec = cand && (!eligible || eligible[p]) && !(created_ts && created_ts[p] >= cutoff);
    if (n_series) *n_series = *n_series - (was_cand ? rows_idle : 0) + (cand ? groups_idle : 0);
    if (n_candidates) *n_candidates = *n_candidates - (was_cand ? 1 : 0) + (cand ? 1 : 0);
    if (n_decisions) *n_decisions = *n_decisions - (was_dec ? 1 : 0) + (dec ? 1 : 0);
    if (cand != was_cand || dec != was_dec) ++fx.pods_changed;
    candidate_bits[word] = cand ? candidate_bits[word] | bit : candidate_bits[word] & ~bit;
    decision_bits[word] = dec ? decision_bits[word] | bit : decision_bits[word] & ~bit;
  }
  return fx;
}

}  // namespace gph
