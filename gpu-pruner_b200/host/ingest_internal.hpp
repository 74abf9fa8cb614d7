// ingest_internal.hpp — pieces shared by the three ingest front ends (DOM reference path and threaded
// text path in ingest.cpp, device path in ingest_device.cpp): label set -> (pod, slot) assignment,
// window shape, time bucketing, and the CPU text walker for sample lists.  Not a public interface.
#pragma once
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <stdexcept>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "../csrc/gpr_text.cuh"  // power_snap / snap_power: one rule for the CPU and the device parser
#include "ingest.hpp"

namespace gph {
namespace detail {


const int64_t kNoTs = std::numeric_limits<int64_t>::min();

// ---- what the row assignment needs from a label map ------------------------------------------------------
// Two interchangeable views: a parsed DOM object (any JSON), or FlatLabels — string_views straight into
// the response text for the only shape Prometheus emits ({"k":"v",...}: string values, no escapes, no
// whitespace, unique keys), built without a single allocation.  `str(key, &v)`: member present AND a
// string; `each(f)`: f(key, value-or-"" ) over the members in text order.
struct JsonMetric {
  const Json& j;
  bool str(std::string_view key, std::string_view* out) const {
    const Json* m = j.find(std::string(key));
    if (!m || !m->is_string()) return false;
    *out = m->as_string();
    return true;
  }
  template <typename F>
  void each(F&& f) const {
    for (const Json::Member& kv : j.members()) f(std::string_view(kv.first), std::string_view(kv.second.as_string()));
  }
};

struct FlatLabels {
  std::vector<std::pair<std::string_view, std::string_view>> kv;
  bool str(std::string_view key, std::string_view* out) const {
    for (const auto& m : kv)
      if (m.first == key) {
        *out = m.second;
        return true;
      }
    return false;
  }
  template <typename F>
  void each(F&& f) const {
    for (const auto& m : kv) f(m.first, m.second);
  }
  // [b, e) must be exactly {"k":"v","k":"v",...}; false = use the DOM parser (escapes, non-string values,
  // whitespace, control characters, duplicate keys, or not a label map at all)
  bool parse(const char* b, const char* e) {
    kv.clear();
    const char* p = b;
    if (p >= e || *p != '{') return false;
    ++p;
    if (p < e && *p == '}') return p + 1 == e;
    while (true) {
      std::string_view k, v;
      if (!quoted(p, e, &k) || p >= e || *p != ':') return false;
      ++p;
      if (!quoted(p, e, &v)) return false;
      for (const auto& m : kv)
        if (m.first == k) return false;
      kv.emplace_back(k, v);
      if (p < e && *p == ',') {
        ++p;
        continue;
      }
      return p + 1 == e && *p == '}';
    }
  }

 private:
  static bool quoted(const char*& p, const char* e, std::string_view* out) {
    if (p >= e || *p != '"') return false;
    const char* s = ++p;
    while (p < e && *p != '"') {
      if (*p == '\\' || (unsigned char)*p < 0x20) return false;
      ++p;
    }
    if (p >= e) return false;
    *out = std::string_view(s, (size_t)(p - s));
    ++p;
    return true;
  }
};

// exported_<x> first, then <x> (lib.rs:158-175)
template <typename M>
inline bool label(const M& metric, std::string_view exported, std::string_view bare, std::string_view* out) {
  return metric.str(exported, out) || metric.str(bare, out);
}

inline float to_f32(double x, uint64_t* clamped) {
  float f = (float)x;
  if (x != 0.0 && f == 0.0f && !std::isnan(x)) {  // below the f32 denormal range: keep it non-zero
    f = std::copysign(std::numeric_limits<float>::denorm_min(), (float)(x < 0 ? -1.0 : 1.0));
    ++*clamped;
  }
  return f;
}

// what a cell of a plane holds for sample x: util plane (snap = power_snap(0)) rounded, power plane also snapped to
// the veto threshold (gpr_text.cuh)
inline float to_cell(double x, const gpr::text::PowerSnap& snap, uint64_t* clamped) {
  return gpr::text::snap_power(x, to_f32(x, clamped), snap);
}

// several samples of one series in one bucket: NaN-aware max — what max_over_time over the row computes anyway
inline void merge_cell(float& cell, float v) {
  cell = std::isnan(cell) ? v : (std::isnan(v) ? cell : std::max(cell, v));
}

// ---- label set -> (pod, slot): shared by the DOM and the text path -----------------------------------
// Hot on the ingest path (40,000 series per C2 tick, while the response is still crossing PCIe), so no
// per-series allocation and no tree lookups: pods are found through an open-addressing table on a 64-bit
// hash of (pod, namespace) verified against the stored strings, and a pod's handful of slots by comparing
// the four group labels directly.
inline uint64_t hash_bytes(uint64_t h, std::string_view s) {
  for (unsigned char c : s) h = (h ^ c) * 0x100000001B3ull;  // FNV-1a
  return (h ^ 0xff) * 0x100000001B3ull;                      // field separator
}

// the labels the row assignment looks at, as views into the label map (text or DOM)
struct LabelFields {
  std::string_view pod, ns, ctr, model, host, gpu;
  bool has_pod = false, has_ns = false, has_ctr = false, has_model = false;
  uint64_t pod_hash = 0;
};
template <typename M>
inline LabelFields extract_fields(const M& m) {
  LabelFields f;
  f.has_pod = label(m, "exported_pod", "pod", &f.pod);
  f.has_ns = label(m, "exported_namespace", "namespace", &f.ns);
  f.has_ctr = label(m, "exported_container", "container", &f.ctr);
  f.has_model = m.str("modelName", &f.model);
  m.str("Hostname", &f.host), m.str("gpu", &f.gpu);   // absent / non-string: ""
  f.pod_hash = hash_bytes(hash_bytes(0xcbf29ce484222325ull, f.pod), f.ns);
  return f;
}
// full label set of a series without the metric name, canonical: what `A or B` compares (query.promql.j2:10-20)
template <typename M>
inline std::string label_signature(const M& m) {
  std::vector<std::string> parts;
  m.each([&](std::string_view k, std::string_view v) {
    if (k != "__name__") parts.push_back(std::string(k) + "\x1f" + std::string(v));
  });
  std::sort(parts.begin(), parts.end());
  std::string sig;
  for (const std::string& x : parts) sig += x + "\x1e";
  return sig;
}

class Assigner {
 public:
  explicit Assigner(Window& w) : w_(w) { table_.assign(1024, 0); }
  enum Result { Skipped, Shadowed, Placed };

  // identity of a series across ticks: see lookup_known.  The two-step form below lets worker threads hash and
  // probe (find_known is read-only) while the single assigning thread inserts afterwards.
  static void series_identity(std::string_view raw_labels, bool is_power, bool is_prof, uint64_t* h1, uint64_t* h2) {
    hash128(raw_labels, is_power ? 0x57 : (is_prof ? 0x50 : 0x55), h1, h2);
  }
  bool find_known(uint64_t h1, uint64_t h2, Result* result, uint32_t* pod_out, uint32_t* slot_out) const {
    if (known_.empty()) return false;
    const size_t mask = known_.size() - 1;
    for (size_t i = (size_t)h1 & mask;; i = (i + 1) & mask) {
      const Known& k = known_[i];
      if (k.h1 == 0 && k.h2 == 0) return false;
      if (k.h1 == h1 && k.h2 == h2) {
        *pod_out = k.pod, *slot_out = k.slot, *result = k.result;
        return true;
      }
    }
  }
  void insert_known(uint64_t h1, uint64_t h2, Result r, uint32_t pod, uint32_t slot) {
    if (known_.empty()) known_.assign(4096, Known{0, 0, Skipped, 0, 0});
    size_t mask = known_.size() - 1, i = (size_t)h1 & mask;
    while (known_[i].h1 || known_[i].h2) {
      if (known_[i].h1 == h1 && known_[i].h2 == h2) return;
      i = (i + 1) & mask;
    }
    probe_at_ = i, probe_h1_ = h1, probe_h2_ = h2;
    remember(r, pod, slot);
  }
  void count_skipped() { ++w_.stats.series_skipped; }

  // Daemon-mode snapshots (snapshot.hpp): what lives beyond one tick, and its restore into a fresh Assigner whose
  // window already holds the pods.  The pod table is rebuilt from the pods, not stored.  The identities stay valid
  // across processes because hash128 depends on the label bytes alone (a change to it changes kSnapshotVersion).
  template <typename F>
  void each_known(F&& f) const {
    for (const Known& k : known_)
      if (k.h1 || k.h2) f(k.h1, k.h2, k.result, k.pod, k.slot);
  }
  const std::vector<std::vector<uint64_t>>& power_keys() const { return power_keys_; }
  const std::map<std::pair<uint32_t, uint32_t>, std::vector<std::string>>& prof_sigs() const { return prof_sigs_; }
  void adopt_pods(std::vector<std::vector<uint64_t>> power_keys,
                  std::map<std::pair<uint32_t, uint32_t>, std::vector<std::string>> prof_sigs) {
    const size_t P = w_.pods.size();
    size_t cap = 1024;
    while (P * 2 > cap) cap *= 4;  // the load factor find_or_add_pod keeps
    table_.assign(cap, 0);
    pod_hash_.clear();
    const size_t mask = cap - 1;
    for (size_t q = 0; q < P; ++q) {
      const PodEntry& pe = static_cast<const PodList&>(w_.pods)[q];
      const uint64_t h = hash_bytes(hash_bytes(0xcbf29ce484222325ull, pe.name), pe.ns);  // as extract_fields
      pod_hash_.push_back(h);
      size_t j = (size_t)(h ^ (h >> 32)) & mask;
      while (table_[j]) j = (j + 1) & mask;
      table_[j] = (uint32_t)q + 1;
    }
    power_keys_ = std::move(power_keys);
    power_keys_.resize(P);
    prof_sigs_ = std::move(prof_sigs);
  }
  // Daemon mode, the resident ring reshaped (IngestOptions::reshape): pod p becomes pod to[p], in the same order, or
  // leaves when to[p] == kDropped — with its power keys, its PROF signatures and the placed series that name it, so
  // that a name that comes back is a new pod, as in a fresh ingest.  Skipped and Shadowed entries name no pod (their
  // pod / slot are never read) and stay.
  static constexpr uint32_t kDropped = 0xFFFFFFFFu;
  void renumber_pods(const std::vector<uint32_t>& to) {
    const PodList& old = w_.pods;
    PodList kept;
    std::vector<std::vector<uint64_t>> keys;
    for (size_t p = 0; p < to.size(); ++p)
      if (to[p] != kDropped) kept.push_back(old[p]), keys.push_back(power_keys_[p]);  // (one entry per pod)
    std::map<std::pair<uint32_t, uint32_t>, std::vector<std::string>> sigs;
    for (const auto& kv : prof_sigs_)
      if (to[kv.first.first] != kDropped) sigs[std::make_pair(to[kv.first.first], kv.first.second)] = kv.second;
    std::vector<Known> entries;
    for (const Known& k : known_)
      if ((k.h1 || k.h2) && (k.result != Placed || to[k.pod] != kDropped))
        entries.push_back(Known{k.h1, k.h2, k.result, k.result == Placed ? to[k.pod] : k.pod, k.slot});
    known_.clear(), n_known_ = 0;
    for (const Known& k : entries) insert_known(k.h1, k.h2, k.result, k.pod, k.slot);
    w_.pods = std::move(kept);
    adopt_pods(std::move(keys), std::move(sigs));
  }

  // Daemon mode: the same series comes back every tick and must keep its row.  A series is identified by the
  // bytes of its label map as the server prints them (sorted keys, so the text is canonical) plus the plane it
  // feeds; known series skip the label work altogether.
  // (identity = two independent 64-bit hashes of those bytes: 128 bits, no copy of the label text is kept)
  // lookup_known: true = the series has been seen, *result / *pod_out / *slot_out are what assign() returned then
  // (its label map need not even be parsed again: identical bytes were validated when it was first seen).
  bool lookup_known(std::string_view raw_labels, bool is_power, bool is_prof, Result* result, uint32_t* pod_out,
                    uint32_t* slot_out) {
    hash128(raw_labels, is_power ? 0x57 : (is_prof ? 0x50 : 0x55), &probe_h1_, &probe_h2_);
    if (known_.empty()) known_.assign(4096, Known{0, 0, Skipped, 0, 0});
    const size_t mask = known_.size() - 1;
    for (probe_at_ = (size_t)probe_h1_ & mask;; probe_at_ = (probe_at_ + 1) & mask) {
      const Known& k = known_[probe_at_];
      if (k.h1 == 0 && k.h2 == 0) return false;
      if (k.h1 == probe_h1_ && k.h2 == probe_h2_) {
        *pod_out = k.pod, *slot_out = k.slot, *result = k.result;
        if (k.result == Skipped) ++w_.stats.series_skipped;
        return true;
      }
    }
  }
  // records the outcome for the series of the lookup_known() call that just returned false
  void remember(Result r, uint32_t pod, uint32_t slot) {
    known_[probe_at_] = Known{probe_h1_, probe_h2_, r, pod, slot};
    if (++n_known_ * 2 > known_.size()) {
      std::vector<Known> bigger(known_.size() * 4, Known{0, 0, Skipped, 0, 0});
      const size_t mask = bigger.size() - 1;
      for (const Known& k : known_) {
        if (k.h1 == 0 && k.h2 == 0) continue;
        size_t j = (size_t)k.h1 & mask;
        while (bigger[j].h1 || bigger[j].h2) j = (j + 1) & mask;
        bigger[j] = k;
      }
      known_.swap(bigger);
    }
  }

  Result assign(const Json& m, bool is_power, bool is_prof, uint32_t* pod_out, uint32_t* slot_out) {
    return assign(JsonMetric{m}, is_power, is_prof, pod_out, slot_out);
  }

  template <typename M>
  Result assign(const M& m, bool is_power, bool is_prof, uint32_t* pod_out, uint32_t* slot_out) {
    return assign_fields(extract_fields(m), is_power, is_prof, [&]() { return label_signature(m); }, pod_out, slot_out);
  }

  // `signature` is only called when a PROF series is involved (never for the usual UTIL-only tick)
  template <typename Sig>
  Result assign_fields(const LabelFields& f, bool is_power, bool is_prof, Sig&& signature, uint32_t* pod_out,
                       uint32_t* slot_out) {
    // the selector demands pod != "" (query.promql.j2:11,17,40); a series that cannot be turned into
    // PodMetricData is skipped with a log line (main.rs:423-428)
    if (!f.has_pod || f.pod.empty() || !f.has_ns || (!is_power && (!f.has_ctr || !f.has_model))) {
      ++w_.stats.series_skipped;
      return Skipped;
    }
    const uint32_t p = find_or_add_pod(f.pod, f.ns, f.pod_hash);
    PodEntry& pe = w_.pods[p];
    // `sum by (Hostname, container, pod, namespace, gpu, modelName)` groups (query.promql.j2:9)
    uint32_t slot;
    if (is_power) {
      // every power series is its own row: `unless on (pod, namespace)` looks at each series' max
      // (query.promql.j2:36-44), there is no `sum by` on that side; the group key only feeds the statistic
      const uint64_t gk = hash_bytes(hash_bytes(hash_bytes(hash_bytes(0xcbf29ce484222325ull, f.host), f.ctr), f.gpu), f.model);
      std::vector<uint64_t>& seen = power_keys_[p];
      if (std::find(seen.begin(), seen.end(), gk) != seen.end()) ++w_.stats.duplicates_merged;
      else seen.push_back(gk);
      slot = pe.power_slots++;
    } else {
      std::vector<GpuSlot>& slots = pe.slots;
      uint32_t group = (uint32_t)slots.size();
      for (uint32_t i = 0; i < slots.size(); ++i) {
        const GpuSlot& g = slots[i];
        if (g.group == i && g.gpu == f.gpu && g.hostname == f.host && g.container == f.ctr && g.model == f.model) {
          group = i;
          break;
        }
      }
      const bool fresh = group == slots.size();
      // `A or B` (query.promql.j2:10-20) matches on the FULL label set: a UTIL element is dropped only
      // if a PROF element with identical labels exists; series that differ in any other label both
      // survive the `or` and are then added up by `sum by`
      if (is_prof) {
        prof_sigs_[std::make_pair(p, group)].push_back(signature());
      } else if (!prof_sigs_.empty()) {
        auto ps = prof_sigs_.find(std::make_pair(p, group));
        if (ps != prof_sigs_.end()) {
          const std::string sig = signature();
          for (const std::string& x : ps->second)
            if (x == sig) return Shadowed;
        }
      }
      // every series keeps its own row; members of one `sum by` group are tied together by `group`
      slot = (uint32_t)slots.size();
      slots.emplace_back();
      GpuSlot& g = slots.back();
      g.hostname.assign(f.host), g.container.assign(f.ctr), g.gpu.assign(f.gpu), g.model.assign(f.model);
      g.node_type = "unknown";  // lib.rs:176-179; the node_dmi_info join fills it in (apply_node_types)
      g.from_prof = is_prof;
      g.group = group;
      if (!fresh) pe.has_groups = true, ++w_.stats.duplicates_merged;
    }
    *pod_out = p, *slot_out = slot;
    return Placed;
  }

 private:
  uint32_t find_or_add_pod(std::string_view pod, std::string_view ns, uint64_t h) {
    size_t mask = table_.size() - 1, i = (size_t)(h ^ (h >> 32)) & mask;
    const PodList& known = w_.pods;  // read-only view: no copy-on-write check per probe
    for (;; i = (i + 1) & mask) {
      const uint32_t e = table_[i];
      if (e == 0) break;
      if (pod_hash_[e - 1] == h && known[e - 1].name == pod && known[e - 1].ns == ns) return e - 1;
    }
    const uint32_t p = (uint32_t)w_.pods.size();
    w_.pods.emplace_back();
    w_.pods.back().name.assign(pod), w_.pods.back().ns.assign(ns);
    w_.pods.back().slots.reserve(8);  // a pod rarely has more GPUs: no regrowth while its series arrive
    pod_hash_.push_back(h);
    power_keys_.emplace_back();
    table_[i] = p + 1;
    if ((size_t)(p + 1) * 2 > table_.size()) {  // keep the load factor below 1/2
      std::vector<uint32_t> bigger(table_.size() * 4, 0);
      mask = bigger.size() - 1;
      for (uint32_t q = 0; q <= p; ++q) {
        size_t j = (size_t)(pod_hash_[q] ^ (pod_hash_[q] >> 32)) & mask;
        while (bigger[j]) j = (j + 1) & mask;
        bigger[j] = q + 1;
      }
      table_.swap(bigger);
    }
    return p;
  }

  struct Known {
    uint64_t h1, h2;  // both zero = empty (hash128 never returns that pair)
    Result result;
    uint32_t pod, slot;
  };
  // two multiply-mix hashes over 8-byte words with different seeds and multipliers
  static void hash128(std::string_view s, uint64_t tag, uint64_t* h1, uint64_t* h2) {
    uint64_t a = 0x9E3779B97F4A7C15ull ^ tag, b = 0xC2B2AE3D27D4EB4Full + tag;
    const char* p = s.data();
    size_t n = s.size();
    auto mix = [](uint64_t x, uint64_t m) {
      x *= m;
      return x ^ (x >> 29);
    };
    for (; n >= 8; p += 8, n -= 8) {
      uint64_t w;
      memcpy(&w, p, 8);
      a = mix(a ^ w, 0xD6E8FEB86659FD93ull);
      b = mix(b + w, 0xA0761D6478BD642Full) ^ (b << 7);
    }
    uint64_t w = 0;
    memcpy(&w, p, n);
    w |= (uint64_t)s.size() << 56;
    a = mix(a ^ w, 0xD6E8FEB86659FD93ull);
    b = mix(b + w, 0xA0761D6478BD642Full) ^ (b << 7);
    a = mix(a, 0xFF51AFD7ED558CCDull), b = mix(b, 0xC4CEB9FE1A85EC53ull);
    if (a == 0 && b == 0) b = 1;
    *h1 = a, *h2 = b;
  }
  std::vector<Known> known_;  // open addressing
  size_t n_known_ = 0, probe_at_ = 0;
  uint64_t probe_h1_ = 0, probe_h2_ = 0;
  Window& w_;
  std::vector<uint32_t> table_;                    // open addressing: pod index + 1, 0 = empty
  std::vector<uint64_t> pod_hash_;                 // per pod
  std::vector<std::vector<uint64_t>> power_keys_;  // per pod: group-key hashes of its power series (statistic only)
  std::map<std::pair<uint32_t, uint32_t>, std::vector<std::string>> prof_sigs_;
};

// the scrape interval when the caller does not give one: the most frequent positive gap between
// consecutive samples (the smallest gap would let one exporter restart or 29/30/31 s jitter decide)
struct StepVote {
  std::unordered_map<int64_t, uint64_t> votes;
  void add(int64_t delta) {
    if (delta > 0) ++votes[delta];
  }
  int64_t result() const {
    int64_t best = 1;
    uint64_t n = 0;
    for (const auto& kv : votes)
      if (kv.second > n || (kv.second == n && kv.first < best)) best = kv.first, n = kv.second;
    return best;
  }
};

inline void finish_shape(Window& w, const IngestOptions& opt, int64_t newest, int64_t inferred_step, bool with_power,
                         bool allocate = true) {
  w.P = (uint32_t)w.pods.size();
  uint32_t G = 1;
  for (const PodEntry& pe : w.pods)
    G = std::max<uint32_t>(G, std::max<uint32_t>((uint32_t)pe.slots.size(), pe.power_slots));
  w.G = G;
  w.step = opt.step > 0 ? opt.step : std::max<int64_t>(1, inferred_step);
  w.t_end = opt.t_end > 0 ? opt.t_end : (newest == kNoTs ? 0 : newest);
  w.span = std::max<int64_t>(1, opt.duration_min * 60);
  w.T = (uint32_t)((w.span + w.step - 1) / w.step);  // every second of (t_end - N, t_end] has a bucket
  if (!allocate) return;  // device ingest: the planes live in HBM
  const size_t cells = (size_t)w.P * w.G * w.T;
  const float nan = std::numeric_limits<float>::quiet_NaN();
  w.util.assign(cells, nan);
  if (with_power) w.power.assign(cells, nan);
}

// timestamp in whole seconds; anything that is not a sane epoch time maps to "far outside any window"
constexpr int64_t kBadTs = std::numeric_limits<int64_t>::min() / 4;
inline int64_t ts_seconds(double t) {
  if (!(t > -4e12 && t < 4e12)) return kBadTs;
  return (int64_t)std::llround(t);
}

// Prometheus timestamps are milliseconds; window membership and bucketing are exact in that unit (rounding
// to whole seconds first would move samples across the window's edges — and across the ticks of daemon mode)
inline int64_t ts_millis(double t) {
  if (!(t > -4e12 && t < 4e12)) return kBadTs;
  return (int64_t)std::llround(t * 1000.0);
}

// column of a timestamp (milliseconds), or -1 when it lies outside (t_end - N, t_end].  Buckets are `step`
// wide and end at t_end (the device parser uses the same rule, csrc/gpr_text.cuh column_of)
inline int64_t column_of(const Window& w, int64_t ts_ms) {
  const int64_t end = w.t_end * 1000;
  if (ts_ms > end || ts_ms <= end - w.span * 1000) return -1;
  const int64_t back = (end - ts_ms) / (w.step * 1000);  // 0 = newest column
  if (back >= (int64_t)w.T) return -1;
  return (int64_t)w.T - 1 - back;
}

// =====================================================================================================
// text walker
// =====================================================================================================

struct Span {
  const char *metric_b, *metric_e, *values_b, *values_e;  // values_b at '[', values_e one past the final ']'
};

[[noreturn]] inline void bad(const char* what) { throw std::runtime_error(std::string("matrix response: ") + what); }

inline const char* skip_ws(const char* p, const char* e) {
  while (p < e && (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r')) ++p;
  return p;
}

// p at '"': returns one past the closing quote
inline const char* skip_string(const char* p, const char* e) {
  for (++p; p < e; ++p) {
    if (*p == '\\') ++p;
    else if (*p == '"') return p + 1;
  }
  bad("unterminated string");
}

// balanced skip of any JSON value
inline const char* skip_value(const char* p, const char* e) {
  p = skip_ws(p, e);
  if (p >= e) bad("unexpected end");
  if (*p == '"') return skip_string(p, e);
  if (*p == '{' || *p == '[') {
    int depth = 0;
    for (; p < e; ++p) {
      if (*p == '"') p = skip_string(p, e) - 1;
      else if (*p == '{' || *p == '[') ++depth;
      else if (*p == '}' || *p == ']') {
        if (--depth == 0) return p + 1;
      }
    }
    bad("unbalanced brackets");
  }
  while (p < e && *p != ',' && *p != '}' && *p != ']') ++p;
  return p;
}

// first occurrence of "]]" in [p, e): eight bytes per step (a values array has a ']' every ~17 bytes,
// which defeats memchr, and glibc's memmem manages ~1 GB/s on a 2-byte needle)
inline const char* find_close2(const char* p, const char* e) {
  const uint64_t pat = 0x5D5D5D5D5D5D5D5Dull;  // ']' x 8
  const uint64_t lo = 0x0101010101010101ull, hi = 0x8080808080808080ull;
  while (e - p >= 9) {
    uint64_t a, b;
    memcpy(&a, p, 8);
    memcpy(&b, p + 1, 8);
    const uint64_t xa = a ^ pat, xb = b ^ pat;
    // zero bytes of x mark ']' — exact zero-byte detection (no false positives across bytes)
    const uint64_t za = ~(((xa & ~hi) + ~hi) | xa) & hi, zb = ~(((xb & ~hi) + ~hi) | xb) & hi;
    const uint64_t both = za & zb;
    if (both) return p + (__builtin_ctzll(both) >> 3);
    p += 8;
    (void)lo;
  }
  for (; p + 1 < e; ++p)
    if (p[0] == ']' && p[1] == ']') return p;
  return nullptr;
}

// Walks the members of the object at p ('{').  `on_member(key_begin, key_len, value_ptr)` may consume
// the value itself and return the position after it; returning nullptr means "skip it for me".
// Returns the position after the closing '}'.
template <typename F>
const char* walk_object(const char* p, const char* e, F&& on_member) {
  p = skip_ws(p, e);
  if (p >= e || *p != '{') bad("expected object");
  ++p;
  while (true) {
    p = skip_ws(p, e);
    if (p < e && *p == '}') return p + 1;
    if (p >= e || *p != '"') bad("expected member name");
    const char* ks = p + 1;
    const char* ke = skip_string(p, e) - 1;
    p = skip_ws(ke + 1, e);
    if (p >= e || *p != ':') bad("expected ':'");
    p = skip_ws(p + 1, e);
    const char* after = on_member(ks, (size_t)(ke - ks), p);
    p = skip_ws(after ? after : skip_value(p, e), e);
    if (p < e && *p == ',') { ++p; continue; }
    if (p < e && *p == '}') return p + 1;
    bad("expected ',' or '}'");
  }
}

inline bool key_is(const char* ks, size_t kl, const char* name) {
  return kl == strlen(name) && memcmp(ks, name, kl) == 0;
}

// the series of a result array starting at arr ('['); returns the position after its ']'
inline const char* result_spans(const char* arr, const char* e, std::vector<Span>& out) {
  const char* p = skip_ws(arr + 1, e);
  while (true) {
    if (p >= e) bad("unterminated result array");
    if (*p == ']') return p + 1;
    Span s{nullptr, nullptr, nullptr, nullptr};
    p = walk_object(p, e, [&](const char* ks, size_t kl, const char* v) -> const char* {
      if (key_is(ks, kl, "values") && v < e && *v == '[') {
        // a values array holds nothing but [ts,"v"] pairs: it ends at the first "]]" (or is "[]"),
        // so the bulk of the response is skipped with memmem instead of being walked
        const char* in = skip_ws(v + 1, e);
        const char* end;
        if (in < e && *in == ']') {
          end = in + 1;
        } else if (in != v + 1) {
          // whitespace right after the '[': an indented (pretty-printed) response, whose list does not
          // end in a literal "]]" — walk it bracket by bracket instead (no server emits this; a proxy or a
          // hand-made fixture may)
          end = skip_value(v, e);
        } else {
          const char* hit = find_close2(v, e);
          if (!hit) bad("unterminated values array");
          end = hit + 2;
        }
        s.values_b = v, s.values_e = end;
        return end;
      }
      if (key_is(ks, kl, "metric")) {
        const char* ve = skip_value(v, e);
        s.metric_b = v, s.metric_e = ve;
        return ve;
      }
      return nullptr;
    });
    out.push_back(s);
    p = skip_ws(p, e);
    if (p < e && *p == ',') p = skip_ws(p + 1, e);
  }
}

inline std::vector<Span> series_spans(const std::string& text) {
  const char* b = text.data();
  const char* e = b + text.size();
  const char* p = skip_ws(b, e);
  std::vector<Span> out;
  if (p < e && *p == '[') {  // bare result array
    result_spans(p, e, out);
    return out;
  }
  bool saw_result = false;
  auto quoted = [&](const char* v) { return std::string(v + 1, skip_string(v, e) - 1); };
  walk_object(p, e, [&](const char* ks, size_t kl, const char* v) -> const char* {
    if (key_is(ks, kl, "status") && *v == '"' && quoted(v) != "success")
      throw std::runtime_error("prometheus response status: " + quoted(v));
    if (!key_is(ks, kl, "data")) return nullptr;
    return walk_object(v, e, [&](const char* ks2, size_t kl2, const char* v2) -> const char* {
      if (key_is(ks2, kl2, "resultType") && *v2 == '"' && quoted(v2) != "matrix")
        throw std::runtime_error("expected matrix response from prometheus, got " + quoted(v2));
      if (key_is(ks2, kl2, "result") && *v2 == '[') {
        saw_result = true;
        return result_spans(v2, e, out);
      }
      return nullptr;
    });
  });
  if (!saw_result) bad("not a Prometheus matrix response");
  return out;
}

// fast decimal: [-+]digits[.digits]; anything else (exponent, NaN, Inf) goes through strtod
inline double parse_number(const char* p, const char* e, const char** end) {
  const char* s = p;
  bool neg = false;
  if (p < e && (*p == '-' || *p == '+')) neg = *p == '-', ++p;
  const char* d0 = p;
  uint64_t ip = 0;
  while (p < e && *p >= '0' && *p <= '9' && p - d0 < 18) ip = ip * 10 + (uint64_t)(*p - '0'), ++p;
  if (p == d0 || (p < e && *p >= '0' && *p <= '9')) goto slow;
  {
    double v = (double)ip;
    if (p < e && *p == '.') {
      ++p;
      const char* f0 = p;
      uint64_t fp = 0;
      while (p < e && *p >= '0' && *p <= '9' && p - f0 < 18) fp = fp * 10 + (uint64_t)(*p - '0'), ++p;
      if (p < e && *p >= '0' && *p <= '9') goto slow;
      static const double pow10[19] = {1,    1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,
                                       1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18};
      // exact only when both parts fit 53 bits; otherwise let strtod round correctly
      if (ip > (1ull << 53) || fp > (1ull << 53) || (p - f0) > 15) goto slow;
      v += (double)fp / pow10[p - f0];
      if (ip != 0 && fp != 0) goto slow;  // sum of two roundings is not always correctly rounded
    }
    if (p < e && (*p == 'e' || *p == 'E')) goto slow;
    *end = p;
    return neg ? -v : v;
  }
slow : {
  char buf[64];
  size_t n = 0;
  const char* q = s;
  while (q < e && n + 1 < sizeof buf && *q != '"' && *q != ',' && *q != ']') buf[n++] = *q++;
  buf[n] = 0;
  char* ep = nullptr;
  const double v = strtod(buf, &ep);
  *end = s + (ep - buf);
  return v;
}
}

// A sample value is what Rust's f64::from_str accepts (the reference decodes it that way: prometheus-http-query 0.8.3
// behind main.rs:405-409, so a value that is not a number fails the whole query) — decimal digits with optional sign,
// fraction and exponent, "NaN", "Inf" / "Infinity" with optional sign, nothing around it.  strtod is more generous
// (hex floats, leading white space, "nan(...)", a valid prefix followed by garbage): those are refused here, because
// garbage read as 0.0 is an idle GPU.
inline bool strict_sample_value(const char* b, const char* e, double* out) {
  const size_t n = (size_t)(e - b);
  char buf[64];
  if (n == 0 || n + 1 > sizeof buf) return false;
  for (size_t i = 0; i < n; ++i) {
    const char c = b[i];
    const bool ok = (c >= '0' && c <= '9') || c == '+' || c == '-' || c == '.' || c == 'e' || c == 'E' ||
                    c == 'N' || c == 'n' || c == 'a' || c == 'A' || c == 'I' || c == 'i' || c == 'f' || c == 'F' ||
                    c == 't' || c == 'T' || c == 'y' || c == 'Y';
    if (!ok) return false;
    buf[i] = c;
  }
  buf[n] = 0;
  char* ep = nullptr;
  const double v = strtod(buf, &ep);
  if (ep != buf + n) return false;
  *out = v;
  return true;
}

// walks [[ts,"v"],[ts,"v"],...] calling f(ts, value)
template <typename F>
void for_each_sample(const char* p, const char* e, F&& f) {
  ++p;  // outer '['
  while (true) {
    p = skip_ws(p, e);
    if (p >= e || *p == ']') return;
    if (*p != '[') bad("expected [ts, value]");
    p = skip_ws(p + 1, e);
    const char* q;
    const double ts = parse_number(p, e, &q);
    if (q == p) bad("bad timestamp");
    p = skip_ws(q, e);
    if (p >= e || *p != ',') bad("expected ','");
    p = skip_ws(p + 1, e);
    double v;
    if (p < e && *p == '"') {
      const char* r = p + 1;
      bool plain = true;  // sign, digits, point: the exact fast path; everything else ("NaN", "+Inf", "5e-07") is vetted
      for (; r < e && *r != '"'; ++r) plain = plain && ((*r >= '0' && *r <= '9') || *r == '.' || *r == '-' || *r == '+');
      if (r >= e) bad("unterminated sample value");
      if (plain) {
        v = parse_number(p + 1, r, &q);
        if (q != r || r == p + 1) bad("sample value is not a number");
      } else if (!strict_sample_value(p + 1, r, &v)) {
        bad("sample value is not a number");
      }
      p = r + 1;
    } else {
      v = parse_number(p, e, &q);
      if (q == p) bad("sample value is not a number");
      p = q;
    }
    p = skip_ws(p, e);
    if (p >= e || *p != ']') bad("expected ']'");
    ++p;
    f(ts, v);
    p = skip_ws(p, e);
    if (p < e && *p == ',') ++p;
  }
}

struct TextSeries {
  uint32_t pod, slot;
  const char *vb, *ve;
  bool sole;  // the only series writing its tensor row
};


}  // namespace detail
}  // namespace gph
