// ingest_device.hpp — the matrix wire format parsed ON THE GPU: the host keeps only what needs hashing
// and strings (label maps -> tensor rows, ~1 % of the bytes); the sample lists go to the device as
// text and land in the dense tensor in HBM (include/gpr.h, gpr_text_scan / gpr_text_parse).  The f32
// window never exists on the host.  Result: the same Window as ingest_matrix_text() — shape, pods,
// statistics — with `d_util` / `d_power` device planes instead of the host vectors, bit-identical
// cell for cell (tests/test_text_device_cpu.py on an emulated device, tests/test_gpu_text.py on the GPU).
#pragma once
#include <cstdint>
#include <functional>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/gpr.h"
#include "ingest.hpp"
#include "snapshot.hpp"

namespace gph {

// What the orchestration needs from the device; implemented over libgpr.so in gpr_engine.cpp.
// Thrown by a TextDevice that cannot take a response although nothing is wrong with the response (more series
// markers in one upload chunk than the scan has room for — label sets a tenth of DCGM's size): the session hands the
// response to the CPU parser instead of failing the tick.
struct DeviceDeclined : std::runtime_error {
  using std::runtime_error::runtime_error;
};

class TextDevice {
 public:
  virtual ~TextDevice() = default;
  // Upload `text` into resident slot `slot` (0..2) and scan it for `},"values":[` ('}' position) and `"]]`
  // ('"' position), as a pipeline: scan_begin starts the upload, every scan_next blocks until the next chunk of
  // the text has been scanned on the device and returns that chunk's markers (sorted, absolute offsets) and how
  // much of the text is covered; false with the last chunk.  The host works on the series it already has
  // markers for while later chunks are still crossing PCIe.
  virtual void scan_begin(int slot, const char* text, size_t n) = 0;
  virtual bool scan_next(std::vector<uint64_t>* opens, std::vector<uint64_t>* closes, uint64_t* bytes_done) = 0;
  // parse the samples of `spans` (sorted by begin) of the text in `slot` into plane 0 (util) / 1 (power):
  // samples with grid.t_end - grid.span < ts <= grid.t_end, bucket (t_end - ts) / step, NaN-aware max merge
  struct TextGrid {
    int64_t t_end = 0, span = 0, step = 1;
    uint32_t T = 0, n_rows = 0;
    bool fill = true;        // start from an all-"no sample" plane
    bool resident = false;   // destination = the resident ring of daemon mode instead of the context plane
    double power_threshold = 0.0;  // plane 1: samples are snapped to it (IngestOptions::power_threshold)
  };
  virtual void parse(int slot, std::vector<gpr_text_span>& spans, const TextGrid& grid, int plane) = 0;
  // overwrite the newest `n_newest` buckets of `row` (chronological order in `data`; n_newest == T: the whole
  // row) — rows the strict device parser declined, re-parsed on the CPU
  virtual void patch_row(int plane, uint32_t row, uint32_t T, const float* data, uint32_t n_newest, bool resident) = 0;
  // patch_row for any run of buckets: the `n` buckets that end `newer` buckets before the newest (a slice of a range
  // asked as several queries).  A device that patches only the newest buckets throws for newer > 0.
  virtual void patch_cols(int plane, uint32_t row, uint32_t T, const float* data, uint32_t n, uint32_t newer,
                          bool resident) {
    if (newer) throw std::logic_error("this device patches only the newest buckets of a row");
    patch_row(plane, row, T, data, n, resident);
  }
  virtual const float* plane(int plane) = 0;
  // daemon mode: (re)create the resident ring [rows][T] (all "no sample"), and open the next n_new buckets
  virtual void resident_init(uint32_t pods, uint32_t G, uint32_t T, bool with_power) = 0;
  virtual void resident_advance(uint32_t n_new) = 0;
  // daemon-mode snapshots (snapshot.hpp): plane `plane` of the resident ring as Prometheus XOR chunks of at most 120
  // samples (gpr_resident_export), in host memory the device keeps until its next export of that plane; the time spent
  // encoding and copying out goes to *export_ms / *copy_ms.  A device that cannot snapshot throws (save_snapshot then
  // reports a failed write; restore_snapshot a refused snapshot).
  virtual void resident_export(int plane, const TextGrid& grid, ChunkPlaneView* out, double* export_ms,
                               double* copy_ms) {
    (void)plane, (void)grid, (void)out, (void)export_ms, (void)copy_ms;
    throw std::logic_error("this device keeps no snapshots");
  }
  // a fresh ring of the given shape (resident_init) holding the exported planes (planes[1] only with_power), merged in
  // by gpr_chunks_scatter(GPR_TEXT_RESIDENT) on `grid`; throws if a plane is refused
  virtual void resident_restore(uint32_t pods, uint32_t G, uint32_t T, bool with_power, const ChunkPlaneView planes[2],
                                const TextGrid& grid) {
    (void)pods, (void)G, (void)T, (void)with_power, (void)planes, (void)grid;
    throw std::logic_error("this device keeps no snapshots");
  }
  // IngestOptions::reshape: the ring's rows moved to the shape [pods][G] (gpr_resident_remap: new row i holds old row
  // src_rows[i], or no sample for GPR_ROW_NONE), and which rows hold a sample in either plane (gpr_resident_live_rows:
  // bit r of (*bits)[r / 32]).  A device that cannot reshape throws; the session then takes the full range.
  virtual void resident_remap(uint32_t pods, uint32_t G, const std::vector<uint32_t>& src_rows) {
    (void)pods, (void)G, (void)src_rows;
    throw std::logic_error("this device cannot reshape its ring");
  }
  virtual void resident_live_rows(std::vector<uint32_t>* bits) {
    (void)bits;
    throw std::logic_error("this device cannot reshape its ring");
  }
  // IngestOptions::retime: the ring's newest n_keep buckets merged `factor` to a bucket (gpr_resident_retime, with the
  // arguments gpr::retime_plan gives); the rows and the power plane stay, the head becomes 0.  A device that cannot
  // retime throws; the session then takes the full range.
  virtual void resident_retime(uint32_t n_keep, uint32_t factor) {
    (void)n_keep, (void)factor;
    throw std::logic_error("this device cannot retime its ring");
  }
  // IngestOptions::reask_seconds: plane `plane` of the ring's n_cols buckets that end `newer` buckets before the newest,
  // oldest first, for every row (gpr_resident_cols: (*out)[r * n_cols + j]).  A device that cannot read a band throws;
  // the session then takes the full range.
  virtual void resident_cols(int plane, uint32_t newer, uint32_t n_cols, std::vector<float>* out) {
    (void)plane, (void)newer, (void)n_cols, (void)out;
    throw std::logic_error("this device cannot read a band of its ring");
  }
};

struct DeviceIngestReport {
  bool on_device = false;        // false: the CPU text path produced the window (reason says why)
  std::string reason;
  uint64_t spans = 0, hard_spans = 0, rows_patched = 0;
  uint64_t slices = 0, ring_growths = 0;  // ingest_slices: queries per metric, and how often the ring grew on the way
  // where the time went: device scan (text upload + marker scan), series walk over the markers,
  // label maps -> rows, device parse (NaN fill + sample parse)
  double scan_ms = 0, labels_ms = 0, assign_ms = 0, parse_ms = 0;
};

// One-shot: needs opt.t_end > 0 and opt.step > 0 (the caller issued the range query, so it knows both);
// otherwise, and for any response that is not in Prometheus' compact encoding, the CPU text path
// runs instead and the returned Window carries host vectors as usual.
Window ingest_matrix_device(TextDevice& dev, const std::string& util, const std::string* prof,
                            const std::string* power, const IngestOptions& opt,
                            DeviceIngestReport* report = nullptr);

// A range asked as consecutive queries (--query-slice): slice j covers (ranges[j].first, ranges[j].second], oldest
// first, each starting where the previous one ends.  load(kind, j, &text) reads the response of metric `kind` (0 PROF,
// 1 UTIL, 2 POWER) for slice j, or throws; it is called only for the metrics the fetch has.
struct SlicedFetch {
  std::vector<std::pair<int64_t, int64_t>> ranges;
  bool has_prof = false, has_power = false;
  std::function<void(int kind, size_t j, std::string* text)> load;
};

// Daemon mode (main.rs:286-330): the row assignment and the window survive between ticks.  The first tick (and
// any tick after NeedFullWindow) ingests the full range query into the engine's resident ring; later ticks ingest
// only what was scraped since (opt.slice_seconds), appended to the ring.  Pods and slots keep their rows for the
// life of the session, so a pod whose series stop reporting simply ages out of the window.
class DeviceIngestSession {
 public:
  explicit DeviceIngestSession(TextDevice& dev);
  ~DeviceIngestSession();
  // opt.slice_seconds == 0: full window (re)build; > 0: delta — throws NeedFullWindow if it cannot be absorbed
  Window ingest(const std::string& util, const std::string* prof, const std::string* power, const IngestOptions& opt,
                DeviceIngestReport* report = nullptr);
  // The same fetch asked as several queries (--query-slice, DESIGN.md §8e): full (opt.slice_seconds == 0) or delta, into
  // the resident ring, with the result a one-query ingest of the range gives.  The ring starts from the first slice and
  // grows (gpr_resident_remap, nothing dropped) when a later slice brings more pods or slots; a full fetch ends with the
  // one-query shape [P + P/4 + 64][G].  A delta that outgrows the ring throws NeedFullWindow as ingest() does, unless
  // opt.reshape.  Throws std::runtime_error for a slice that fails or a response the device cannot take (no CPU
  // fallback here); the session then stays cold.
  Window ingest_slices(const SlicedFetch& f, const IngestOptions& opt, DeviceIngestReport* report = nullptr);
  // newest second the resident window holds (0 = nothing resident): the next delta must start right after it
  int64_t resident_t_end() const;
  void invalidate();
  // Snapshots of the session between ticks (snapshot.hpp).  save_state: false = nothing resident.  export_planes: the
  // ring's planes through the device (planes[1] only with a power plane).  restore_state: the ring first, through the
  // device, then the session; the session is valid only once both are in place — if the device refuses a plane (it
  // throws) the session stays cold and the next tick takes the full range.  The existing delta checks then decide
  // whether the first slice can be absorbed.
  bool save_state(SnapshotState* out) const;
  void export_planes(ChunkPlaneView planes[2], double* export_ms, double* copy_ms);
  void restore_state(const SnapshotState& s, const ChunkPlaneView planes[2]);

 private:
  struct State;
  TextDevice& dev_;
  State* st_;
};

}  // namespace gph
