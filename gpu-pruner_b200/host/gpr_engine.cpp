// gpr_engine.cpp — the product VerdictEngine: libgpr.so (include/gpr.h), CUDA on sm_90a.
// There is no other implementation in the product; without a CUDA device every tick fails and is
// counted like a failed Prometheus query in the reference (main.rs:310-321).
//
// The same object is the product's TextDevice / TextIngestor (GPR_INGEST=gpu): the response text is
// parsed on the GPU straight into HBM and the decision runs on those device planes — the f32 window
// never crosses PCIe, only the text does (once).
#include <chrono>
#include <algorithm>
#include <cstring>
#include <limits>
#include <memory>
#include <vector>
#include <stdexcept>

#include "../../include/gpr.h"
#include "controller.hpp"
#include "ingest_device.hpp"

namespace gph {
namespace {

class GprVerdictEngine : public VerdictEngine, public TextIngestor, private TextDevice {
 public:
  ~GprVerdictEngine() override {
    if (ctx_) {
      free_exports();
      if (d_elig_) gpr_device_free(ctx_, d_elig_);
      if (d_created_) gpr_device_free(ctx_, d_created_);
      if (d_table_) gpr_device_free(ctx_, d_table_);
      gpr_destroy(ctx_);
    }
  }

  TextIngestor* text_ingestor() override { return this; }

  // ---- VerdictEngine --------------------------------------------------------------------------------
  bool decide(const VerdictRequest& rq, Verdict* out, std::string* error) override {
    const Window& w = *rq.window;
    if (w.resident) return decide_resident(rq, out, error);
    const bool on_device = w.d_util != nullptr;
    if (on_device ? !ensure_ctx(rq.gpu_device, error) : !ensure(w, rq.power_on, rq.gpu_device, error)) return false;
    const uint32_t W = (w.P + 31) / 32;
    out->decision_bits.assign(W, 0), out->candidate_bits.assign(W, 0);
    // the engine resolves `sum by` groups itself and says which slots start idle elements: no per-series maxima
    // (the reduce stops reading a row once its flag is settled), no veto bitmap
    out->idle_slots.assign((size_t)w.P * ((w.G + 31) / 32), 0u);
    out->groups_resolved = true;
    const std::vector<uint32_t> table = has_groups(w) ? group_table(w, w.P) : std::vector<uint32_t>();
    gpr_window win;
    memset(&win, 0, sizeof win);
    win.struct_size = sizeof win;
    win.power_threshold = rq.power_on ? rq.power_threshold : 0.0;
    win.cutoff_ts = rq.cutoff_ts;
    win.n_pods = w.P, win.n_gpus = w.G, win.n_samples = w.T;
    if (on_device) {
      // planes are in HBM already (device ingest); mem_kind covers the gates too, so they follow
      win.mem_kind = GPR_MEM_DEVICE;
      win.util = w.d_util;
      win.power = rq.power_on ? w.d_power : nullptr;
      if (!upload_gates(rq, w.P, &win, error) || !upload_table(table, &win, error)) return false;
    } else {
      win.mem_kind = GPR_MEM_HOST;
      win.util = w.util.data();
      win.power = rq.power_on ? w.power.data() : nullptr;
      win.eligible = rq.eligible;
      win.created_ts = rq.created_ts;
      win.groups = table.empty() ? nullptr : table.data();
    }
    gpr_result res;
    memset(&res, 0, sizeof res);
    res.struct_size = sizeof res;
    res.out_mem_kind = GPR_MEM_HOST;
    res.decision_bits = out->decision_bits.data();
    res.candidate_bits = out->candidate_bits.data();
    res.idle_slots = out->idle_slots.data();
    const int rc = gpr_decide(ctx_, &win, &res);
    if (rc != GPR_OK) {
      *error = "idle engine (" + std::to_string(rc) + "): " + gpr_last_error(ctx_);
      return false;
    }
    out->n_series = res.n_series, out->n_candidates = res.n_candidates, out->n_decisions = res.n_decisions;
    out->kernel_ms = res.kernel_ms;
    return true;
  }

  // the resident window of daemon mode: same kernels on the ring, gates from the host
  bool decide_resident(const VerdictRequest& rq, Verdict* out, std::string* error) {
    const Window& w = *rq.window;
    if (!ctx_) {
      *error = "idle engine: no resident window";
      return false;
    }
    // the ring has rows for resident_pods pods; the ones beyond the pods known so far hold no sample
    const uint32_t Pr = w.resident_pods, W = (Pr + 31) / 32, MW = (w.G + 31) / 32;
    std::vector<uint32_t> dbits(W, 0), cbits(W, 0), islots((size_t)Pr * MW, 0u);
    const std::vector<uint32_t> table = has_groups(w) ? group_table(w, Pr) : std::vector<uint32_t>();
    std::vector<uint8_t> elig(Pr, 0);
    std::vector<int64_t> created(Pr, std::numeric_limits<int64_t>::max());
    for (uint32_t p = 0; p < w.P; ++p) {
      elig[p] = rq.eligible ? rq.eligible[p] : 1;
      if (rq.created_ts) created[p] = rq.created_ts[p];
    }
    gpr_window win;
    memset(&win, 0, sizeof win);
    win.struct_size = sizeof win;
    win.mem_kind = GPR_MEM_HOST;  // the gates; the planes are the ring's
    win.power_threshold = rq.power_on && w.resident_power ? rq.power_threshold : 0.0;
    win.cutoff_ts = rq.cutoff_ts;
    win.eligible = elig.data();
    win.created_ts = rq.created_ts ? created.data() : nullptr;
    win.groups = table.empty() ? nullptr : table.data();
    gpr_result res;
    memset(&res, 0, sizeof res);
    res.struct_size = sizeof res;
    res.out_mem_kind = GPR_MEM_HOST;
    res.decision_bits = dbits.data(), res.candidate_bits = cbits.data(), res.idle_slots = islots.data();
    const int rc = gpr_decide_resident(ctx_, &win, &res);
    if (rc != GPR_OK) {
      *error = "idle engine (" + std::to_string(rc) + "): " + gpr_last_error(ctx_);
      return false;
    }
    const uint32_t Wp = (w.P + 31) / 32;
    out->decision_bits.assign(dbits.begin(), dbits.begin() + Wp);
    out->candidate_bits.assign(cbits.begin(), cbits.begin() + Wp);
    out->idle_slots.assign(islots.begin(), islots.begin() + (size_t)w.P * MW);
    out->groups_resolved = true;
    out->n_series = res.n_series, out->n_candidates = res.n_candidates, out->n_decisions = res.n_decisions;
    out->kernel_ms = res.kernel_ms;
    return true;
  }

  // ---- TextIngestor ---------------------------------------------------------------------------------
  int64_t resident_t_end() const override { return session_ ? session_->resident_t_end() : 0; }
  DeviceIngestSession* resident_session(const Cli& args, std::string* error) override {
    if (!ensure_ctx(args.gpu_device, error)) return nullptr;
    if (!session_) session_.reset(new DeviceIngestSession(*this));
    return session_.get();
  }

  Window ingest(const Cli& args, const std::string& util, const std::string* prof, const std::string* power,
                const IngestOptions& opt, std::string* note) override {
    std::string error;
    if (!ensure_ctx(args.gpu_device, &error)) throw std::runtime_error("Failed to run query! " + error);
    const auto t0 = std::chrono::steady_clock::now();
    DeviceIngestReport rep;
    if (!session_) session_.reset(new DeviceIngestSession(*this));
    Window w = session_->ingest(util, prof, power, opt, &rep);
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (note) {
      char buf[600];
      if (rep.on_device && opt.slice_seconds > 0)
        snprintf(buf, sizeof buf,
                 "Device ingest: %llu series lists of the last %lld s appended to the resident %ux%ux%u window in %.1f ms "
                 "(%llu re-parsed on the CPU, %llu rows patched; waiting for upload+scan %.1f, label maps (parallel) %.1f, rows (sequential) %.1f, "
                 "parse %.1f ms)",
                 (unsigned long long)rep.spans, (long long)opt.slice_seconds, w.P, w.G, w.T, ms,
                 (unsigned long long)rep.hard_spans, (unsigned long long)rep.rows_patched, rep.scan_ms, rep.labels_ms,
                 rep.assign_ms, rep.parse_ms);
      else if (rep.on_device)
        snprintf(buf, sizeof buf,
                 "Device ingest: %llu series lists parsed on the GPU into a %s%ux%ux%u window in %.1f ms "
                 "(%llu re-parsed on the CPU, %llu rows patched; waiting for upload+scan %.1f, label maps (parallel) %.1f, rows (sequential) %.1f, "
                 "parse %.1f ms)",
                 (unsigned long long)rep.spans, w.resident ? "resident " : "", w.P, w.G, w.T, ms,
                 (unsigned long long)rep.hard_spans,
                 (unsigned long long)rep.rows_patched, rep.scan_ms, rep.labels_ms, rep.assign_ms, rep.parse_ms);
      else
        snprintf(buf, sizeof buf, "Device ingest not used (%s): CPU text parser, %.1f ms", rep.reason.c_str(), ms);
      *note = buf;
      if (rep.on_device && opt.slice_seconds > 0 && opt.reask_seconds > 0) *note += reask_note(opt, w);
    }
    return w;
  }

  Window ingest_slices(const Cli& args, const SlicedFetch& f, const IngestOptions& opt, std::string* note) override {
    std::string error;
    if (!ensure_ctx(args.gpu_device, &error)) throw std::runtime_error("Failed to run query! " + error);
    const auto t0 = std::chrono::steady_clock::now();
    DeviceIngestReport rep;
    if (!session_) session_.reset(new DeviceIngestSession(*this));
    Window w = session_->ingest_slices(f, opt, &rep);
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (note) {
      char buf[600];
      snprintf(buf, sizeof buf,
               "Device ingest: %llu series lists of %llu query slices over the last %lld s parsed on the GPU into the "
               "resident %ux%ux%u window in %.1f ms (ring grown %llu times, %llu re-parsed on the CPU, %llu rows patched; "
               "waiting for upload+scan %.1f, label maps (parallel) %.1f, rows (sequential) %.1f, parse %.1f ms)",
               (unsigned long long)rep.spans, (unsigned long long)rep.slices,
               (long long)(opt.slice_seconds > 0 ? opt.slice_seconds : w.span), w.P, w.G, w.T, ms,
               (unsigned long long)rep.ring_growths, (unsigned long long)rep.hard_spans,
               (unsigned long long)rep.rows_patched, rep.scan_ms, rep.labels_ms, rep.assign_ms, rep.parse_ms);
      *note = buf;
      if (opt.slice_seconds > 0 && opt.reask_seconds > 0) *note += reask_note(opt, w);
    }
    return w;
  }

  // --late-seconds: what the re-ask cost on top of the tick's own slice
  static std::string reask_note(const IngestOptions& opt, const Window& w) {
    char buf[160];
    snprintf(buf, sizeof buf, "; re-asked the newest %lld s, band read and compare %.2f ms", (long long)opt.reask_seconds,
             w.stats.band_ms);
    return buf;
  }

 private:
  // ---- TextDevice over libgpr -------------------------------------------------------------------------
  void check(int rc, const char* what) {
    if (rc != GPR_OK) throw std::runtime_error(std::string(what) + " (" + std::to_string(rc) + "): " + gpr_last_error(ctx_));
  }
  // The response sits in ordinary (pageable) memory: the library stages it through its pinned ring with a few
  // producer threads and scans every chunk as it lands (gpr_text_scan_begin / _next); this thread meanwhile turns
  // the label maps of the series it already has markers for into tensor rows.
  // (A caller that receives the response straight into gpr_host_alloc memory skips the staging copy.)
  void scan_begin(int slot, const char* text, size_t n) override {
    check(gpr_text_scan_begin(ctx_, slot, text, n, GPR_MEM_HOST), "gpr_text_scan_begin");
  }
  bool scan_next(std::vector<uint64_t>* opens, std::vector<uint64_t>* closes, uint64_t* bytes_done) override {
    const uint64_t cap = 1u << 14;  // markers of one kind per chunk the library can report
    opens->resize(cap), closes->resize(cap);
    uint64_t no = 0, nc = 0;
    int32_t more = 0;
    const int rc = gpr_text_scan_next(ctx_, opens->data(), closes->data(), cap, &no, &nc, bytes_done, &more);
    // more series markers in one chunk than the scan holds: not an error of the response — the CPU parser takes it
    if (rc == GPR_E_CAPACITY) throw DeviceDeclined(std::string("device scan: ") + gpr_last_error(ctx_));
    check(rc, "gpr_text_scan_next");
    opens->resize(no), closes->resize(nc);
    return more != 0;
  }
  void parse(int slot, std::vector<gpr_text_span>& spans, const TextGrid& grid, int plane) override {
    const gpr_text_grid g = text_grid(grid);
    check(gpr_text_parse(ctx_, slot, spans.data(), (uint32_t)spans.size(), &g, plane), "gpr_text_parse");
  }
  void patch_row(int plane, uint32_t row, uint32_t T, const float* data, uint32_t n_newest, bool resident) override {
    patch_cols(plane, row, T, data, n_newest, 0, resident);
  }
  void patch_cols(int plane, uint32_t row, uint32_t T, const float* data, uint32_t n, uint32_t newer,
                  bool resident) override {
    float *u = nullptr, *p = nullptr;
    uint32_t head = 0;  // dense planes: the newest bucket is column T - 1, as if the head were at 0
    if (resident) {
      uint64_t ld = 0;
      check(gpr_resident_planes(ctx_, &u, &p, &ld), "gpr_resident_planes");
      check(gpr_resident_head(ctx_, &head), "gpr_resident_head");
    } else {
      check(gpr_text_planes(ctx_, &u, &p), "gpr_text_planes");
    }
    float* base = (plane == 0 ? u : p) + (size_t)row * T;
    // the n buckets ending `newer` before the newest sit at ring positions head - newer - n .. head - newer - 1
    // (mod T): at most two runs
    const uint32_t first = (head + 2 * T - newer % T - n % T) % T;
    const uint32_t run1 = std::min(n, T - first);
    check(gpr_memcpy(ctx_, base + first, data, (size_t)run1 * sizeof(float), GPR_MEM_DEVICE, GPR_MEM_HOST), "row patch");
    if (run1 < n)
      check(gpr_memcpy(ctx_, base, data + run1, (size_t)(n - run1) * sizeof(float), GPR_MEM_DEVICE, GPR_MEM_HOST),
            "row patch");
  }
  void resident_init(uint32_t pods, uint32_t G, uint32_t T, bool with_power) override {
    check(gpr_resident_init(ctx_, pods, G, T, with_power ? GPR_F_POWER_PLANE : 0u), "gpr_resident_init");
    resident_rows_ = pods * G;
  }
  void resident_advance(uint32_t n_new) override { check(gpr_resident_advance(ctx_, n_new), "gpr_resident_advance"); }
  // --reshape-ring: the map goes up from the host (gpr_resident_remap checks it there), the bitmap comes back to it
  void resident_remap(uint32_t pods, uint32_t G, const std::vector<uint32_t>& src_rows) override {
    check(gpr_resident_remap(ctx_, pods, G, src_rows.data(), GPR_MEM_HOST), "gpr_resident_remap");
    resident_rows_ = pods * G;
  }
  void resident_live_rows(std::vector<uint32_t>* bits) override {
    bits->assign(((size_t)resident_rows_ + 31) / 32, 0u);
    check(gpr_resident_live_rows(ctx_, bits->data(), GPR_MEM_HOST), "gpr_resident_live_rows");
  }
  // --retime-ring: the rows stay, only their length and the head change
  void resident_retime(uint32_t n_keep, uint32_t factor) override {
    check(gpr_resident_retime(ctx_, n_keep, factor), "gpr_resident_retime");
  }
  // --late-seconds: the re-asked band comes back to the host, before and after the tick's merge
  void resident_cols(int plane, uint32_t newer, uint32_t n_cols, std::vector<float>* out) override {
    out->resize((size_t)resident_rows_ * n_cols);
    check(gpr_resident_cols(ctx_, plane, newer, n_cols, out->data(), GPR_MEM_HOST), "gpr_resident_cols");
  }
  // Snapshots: the encoder writes into device buffers kept across ticks, then one copy per array lands in pinned host
  // memory (the two are timed apart).  Capacities carry a quarter of head-room, so a steady tick encodes once; a
  // grown ring is sized by the first call (GPR_E_CAPACITY returns the true counts) and encoded again.
  struct ExportBufs {
    void* d = nullptr;  // series_chunks | chunk_bytes | rows | data, on the device
    void* h = nullptr;  // the same, pinned host memory
    uint64_t cap_series = 0, cap_chunks = 0, cap_bytes = 0;
    size_t bytes() const { return (cap_series + 1) * 8 + (cap_chunks + 1) * 8 + cap_series * 4 + cap_bytes; }
  };
  void free_exports() {
    for (ExportBufs& b : xb_) {
      if (b.d) gpr_device_free(ctx_, b.d);
      if (b.h) gpr_host_free(ctx_, b.h);
      b = ExportBufs();
    }
  }
  void grow_export(ExportBufs& b, uint64_t series, uint64_t chunks, uint64_t bytes) {
    if (b.d) gpr_device_free(ctx_, b.d), b.d = nullptr;
    if (b.h) gpr_host_free(ctx_, b.h), b.h = nullptr;
    b.cap_series = series + series / 4 + 64, b.cap_chunks = chunks + chunks / 4 + 64, b.cap_bytes = bytes + bytes / 4 + 4096;
    check(gpr_device_alloc(ctx_, b.bytes(), &b.d), "snapshot buffer");
    check(gpr_host_alloc(ctx_, b.bytes(), &b.h), "snapshot buffer");
  }
  static gpr_text_grid text_grid(const TextGrid& grid) {
    gpr_text_grid g;
    memset(&g, 0, sizeof g);
    g.struct_size = sizeof g;
    g.flags = (grid.fill ? GPR_TEXT_FILL : 0u) | (grid.resident ? GPR_TEXT_RESIDENT : 0u);
    g.t_end = grid.t_end, g.window_seconds = grid.span, g.step = grid.step;
    g.n_samples = grid.T, g.n_rows = grid.n_rows;
    g.power_threshold = grid.power_threshold;
    return g;
  }
  void resident_export(int plane, const TextGrid& grid, ChunkPlaneView* out, double* export_ms, double* copy_ms) override {
    ExportBufs& b = xb_[plane];
    const gpr_text_grid g = text_grid(grid);
    const auto t0 = std::chrono::steady_clock::now();
    if (!b.d) grow_export(b, 0, 0, 0);
    gpr_chunk_export x;
    for (int attempt = 0;; ++attempt) {
      unsigned char* d = static_cast<unsigned char*>(b.d);
      memset(&x, 0, sizeof x);
      x.struct_size = sizeof x;
      x.mem_kind = GPR_MEM_DEVICE;
      x.series_chunks = reinterpret_cast<uint64_t*>(d);
      x.chunk_bytes = reinterpret_cast<uint64_t*>(d + (b.cap_series + 1) * 8);
      x.rows = reinterpret_cast<uint32_t*>(d + (b.cap_series + 1) * 8 + (b.cap_chunks + 1) * 8);
      x.data = d + (b.cap_series + 1) * 8 + (b.cap_chunks + 1) * 8 + b.cap_series * 4;
      x.cap_series = b.cap_series, x.cap_chunks = b.cap_chunks, x.cap_bytes = b.cap_bytes;
      const int rc = gpr_resident_export(ctx_, &g, plane, 120, &x);
      if (rc == GPR_E_CAPACITY && attempt == 0) {
        grow_export(b, x.n_series, x.n_chunks, x.n_bytes);
        continue;
      }
      check(rc, "gpr_resident_export");
      break;
    }
    const auto t1 = std::chrono::steady_clock::now();
    unsigned char* d = static_cast<unsigned char*>(b.d);
    unsigned char* h = static_cast<unsigned char*>(b.h);
    const size_t o_cb = (b.cap_series + 1) * 8, o_rows = o_cb + (b.cap_chunks + 1) * 8, o_data = o_rows + b.cap_series * 4;
    check(gpr_memcpy(ctx_, h, d, (x.n_series + 1) * 8, GPR_MEM_HOST, GPR_MEM_DEVICE), "snapshot copy");
    check(gpr_memcpy(ctx_, h + o_cb, d + o_cb, (x.n_chunks + 1) * 8, GPR_MEM_HOST, GPR_MEM_DEVICE), "snapshot copy");
    if (x.n_series) check(gpr_memcpy(ctx_, h + o_rows, d + o_rows, x.n_series * 4, GPR_MEM_HOST, GPR_MEM_DEVICE), "snapshot copy");
    if (x.n_bytes) check(gpr_memcpy(ctx_, h + o_data, d + o_data, x.n_bytes, GPR_MEM_HOST, GPR_MEM_DEVICE), "snapshot copy");
    const auto t2 = std::chrono::steady_clock::now();
    out->n_series = x.n_series, out->n_chunks = x.n_chunks, out->n_bytes = x.n_bytes;
    out->series_chunks = reinterpret_cast<const uint64_t*>(h);
    out->chunk_bytes = reinterpret_cast<const uint64_t*>(h + o_cb);
    out->rows = reinterpret_cast<const uint32_t*>(h + o_rows);
    out->data = h + o_data;
    *export_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    *copy_ms = std::chrono::duration<double, std::milli>(t2 - t1).count();
  }
  // The planes go up as host batches: gpr_chunks_scatter checks and merges them in pieces through its own staging,
  // so the file's buffer needs no device copy of itself.  The binary's ring has no block index (no GPR_F_BLOCK_INDEX),
  // so there is nothing to reindex.
  void resident_restore(uint32_t pods, uint32_t G, uint32_t T, bool with_power, const ChunkPlaneView planes[2],
                        const TextGrid& grid) override {
    resident_init(pods, G, T, with_power);
    for (int k = 0; k < (with_power ? 2 : 1); ++k) {
      const ChunkPlaneView& v = planes[k];
      gpr_chunk_batch cb;
      memset(&cb, 0, sizeof cb);
      cb.struct_size = sizeof cb;
      cb.mem_kind = GPR_MEM_HOST;
      cb.series_chunks = v.series_chunks, cb.rows = v.rows, cb.chunk_bytes = v.chunk_bytes, cb.data = v.data;
      cb.n_series = (uint32_t)v.n_series;
      TextGrid pg = grid;
      pg.power_threshold = k == 1 ? grid.power_threshold : 0.0;
      const gpr_text_grid g = text_grid(pg);
      check(gpr_chunks_scatter(ctx_, &cb, &g, k, nullptr), k == 0 ? "gpr_chunks_scatter (util plane)" : "gpr_chunks_scatter (power plane)");
    }
  }
  const float* plane(int plane) override {
    float *u = nullptr, *p = nullptr;
    check(gpr_text_planes(ctx_, &u, &p), "gpr_text_planes");
    return plane == 0 ? u : p;
  }

  // ---- context ------------------------------------------------------------------------------------------
  static bool has_groups(const Window& w) {
    for (const PodEntry& pe : w.pods)
      if (pe.has_groups) return true;
    return false;
  }
  // the group table of a device window lives on the device too (gpr_window.groups follows mem_kind)
  bool upload_table(const std::vector<uint32_t>& table, gpr_window* win, std::string* error) {
    if (table.empty()) return true;
    const size_t bytes = table.size() * sizeof(uint32_t);
    if (bytes > table_cap_) {
      if (d_table_) gpr_device_free(ctx_, d_table_), d_table_ = nullptr;
      table_cap_ = 0;
      if (gpr_device_alloc(ctx_, bytes + bytes / 4 + 256, &d_table_) != GPR_OK) {
        *error = std::string("idle engine: group table buffer: ") + gpr_last_error(ctx_);
        return false;
      }
      table_cap_ = bytes + bytes / 4 + 256;
    }
    if (gpr_memcpy(ctx_, d_table_, table.data(), bytes, GPR_MEM_DEVICE, GPR_MEM_HOST) != GPR_OK) {
      *error = std::string("idle engine: group table upload: ") + gpr_last_error(ctx_);
      return false;
    }
    win->groups = static_cast<const uint32_t*>(d_table_);
    return true;
  }

  bool upload_gates(const VerdictRequest& rq, uint32_t P, gpr_window* win, std::string* error) {
    if (P > gate_cap_) {
      if (d_elig_) gpr_device_free(ctx_, d_elig_), d_elig_ = nullptr;
      if (d_created_) gpr_device_free(ctx_, d_created_), d_created_ = nullptr;
      const size_t cap = (size_t)P + P / 4 + 64;
      if (gpr_device_alloc(ctx_, cap, &d_elig_) != GPR_OK ||
          gpr_device_alloc(ctx_, cap * sizeof(int64_t), &d_created_) != GPR_OK) {
        *error = std::string("idle engine: gate buffers: ") + gpr_last_error(ctx_);
        return false;
      }
      gate_cap_ = cap;
    }
    int rc = GPR_OK;
    if (rq.eligible && P) {
      rc = gpr_memcpy(ctx_, d_elig_, rq.eligible, P, GPR_MEM_DEVICE, GPR_MEM_HOST);
      win->eligible = static_cast<const uint8_t*>(d_elig_);
    }
    if (rc == GPR_OK && rq.created_ts && P) {
      rc = gpr_memcpy(ctx_, d_created_, rq.created_ts, (size_t)P * sizeof(int64_t), GPR_MEM_DEVICE, GPR_MEM_HOST);
      win->created_ts = static_cast<const int64_t*>(d_created_);
    }
    if (rc != GPR_OK) {
      *error = std::string("idle engine: gate upload: ") + gpr_last_error(ctx_);
      return false;
    }
    return true;
  }

  // a context without host-window staging is enough for device-resident windows
  bool ensure_ctx(int device, std::string* error) {
    if (ctx_) return true;
    return create(0, 1, 1, false, device, error);
  }
  bool ensure(const Window& w, bool need_power, int device, std::string* error) {
    const uint64_t cells = (uint64_t)w.P * w.G * w.T;
    if (ctx_ && cells <= cap_cells_ && (!need_power || cap_power_)) return true;
    drop();
    // head-room so that a growing cluster does not re-create the context every tick
    return create(w.P + w.P / 4 > 64 ? w.P + w.P / 4 : 64, w.G ? w.G : 1, w.T ? w.T : 1, need_power, device, error);
  }
  void drop() {
    if (!ctx_) return;
    session_.reset();  // its resident window dies with the context
    free_exports();
    if (d_elig_) gpr_device_free(ctx_, d_elig_), d_elig_ = nullptr;
    if (d_created_) gpr_device_free(ctx_, d_created_), d_created_ = nullptr;
    if (d_table_) gpr_device_free(ctx_, d_table_), d_table_ = nullptr;
    gate_cap_ = 0, table_cap_ = 0;
    gpr_destroy(ctx_), ctx_ = nullptr;
  }
  bool create(uint32_t max_pods, uint32_t max_gpus, uint32_t max_samples, bool need_power, int device,
              std::string* error) {
    gpr_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.struct_size = sizeof cfg;
    cfg.device = device;
    cfg.max_pods = max_pods, cfg.max_gpus = max_gpus, cfg.max_samples = max_samples;
    cfg.flags = need_power ? GPR_F_POWER_PLANE : 0;
    const int rc = gpr_create(&cfg, &ctx_);
    if (rc != GPR_OK) {
      *error = std::string("idle engine unavailable (") + std::to_string(rc) + "): " + gpr_last_error(nullptr);
      ctx_ = nullptr;
      return false;
    }
    cap_cells_ = (uint64_t)cfg.max_pods * cfg.max_gpus * cfg.max_samples;
    cap_power_ = need_power;
    return true;
  }

  gpr_ctx* ctx_ = nullptr;
  std::unique_ptr<DeviceIngestSession> session_;
  ExportBufs xb_[2];
  uint32_t resident_rows_ = 0;  // rows of the resident ring (pods x G)
  uint64_t cap_cells_ = 0;
  bool cap_power_ = false;
  void* d_elig_ = nullptr;
  void* d_created_ = nullptr;
  size_t gate_cap_ = 0;
  void* d_table_ = nullptr;
  size_t table_cap_ = 0;
};

}  // namespace

std::unique_ptr<VerdictEngine> make_gpr_engine() { return std::make_unique<GprVerdictEngine>(); }

}  // namespace gph
