// snapshot.cpp — the snapshot file of daemon mode (snapshot.hpp; layout in DESIGN.md §8i).
#include "snapshot.hpp"

#include <cerrno>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include "controller.hpp"
#include "ingest_device.hpp"

#if !defined(__BYTE_ORDER__) || __BYTE_ORDER__ != __ORDER_LITTLE_ENDIAN__
#error "the snapshot layout is little-endian and written as the host lays out its integers"
#endif

namespace gph {

// ---- CRC32C ---------------------------------------------------------------------------------------------------------
namespace {

struct Crc32cTables {
  uint32_t t[8][256];
  Crc32cTables() {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
      t[0][i] = c;
    }
    for (uint32_t i = 0; i < 256; ++i)
      for (int s = 1; s < 8; ++s) t[s][i] = (t[s - 1][i] >> 8) ^ t[0][t[s - 1][i] & 0xffu];
  }
};
const Crc32cTables& tables() {
  static const Crc32cTables t;
  return t;
}

#if defined(__x86_64__)
__attribute__((target("sse4.2"))) uint32_t crc32c_sse42(const uint8_t* p, size_t n, uint32_t c) {
  while (n && (reinterpret_cast<uintptr_t>(p) & 7u)) c = __builtin_ia32_crc32qi(c, *p++), --n;
  for (; n >= 8; p += 8, n -= 8) {
    uint64_t w;
    memcpy(&w, p, 8);
    c = (uint32_t)__builtin_ia32_crc32di(c, w);
  }
  while (n--) c = __builtin_ia32_crc32qi(c, *p++);
  return c;
}
bool have_sse42() {
  static const bool yes = __builtin_cpu_supports("sse4.2");
  return yes;
}
#endif

double ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace

uint32_t crc32c_portable(const void* data, size_t n, uint32_t crc) {
  const Crc32cTables& T = tables();
  const uint8_t* p = static_cast<const uint8_t*>(data);
  uint32_t c = ~crc;
  while (n && (reinterpret_cast<uintptr_t>(p) & 7u)) c = T.t[0][(c ^ *p++) & 0xffu] ^ (c >> 8), --n;
  for (; n >= 8; p += 8, n -= 8) {
    uint32_t a, b;
    memcpy(&a, p, 4);
    memcpy(&b, p + 4, 4);
    a ^= c;
    c = T.t[7][a & 0xffu] ^ T.t[6][(a >> 8) & 0xffu] ^ T.t[5][(a >> 16) & 0xffu] ^ T.t[4][a >> 24] ^
        T.t[3][b & 0xffu] ^ T.t[2][(b >> 8) & 0xffu] ^ T.t[1][(b >> 16) & 0xffu] ^ T.t[0][b >> 24];
  }
  while (n--) c = T.t[0][(c ^ *p++) & 0xffu] ^ (c >> 8);
  return ~c;
}

uint32_t crc32c(const void* data, size_t n, uint32_t crc) {
#if defined(__x86_64__)
  if (have_sse42()) return ~crc32c_sse42(static_cast<const uint8_t*>(data), n, ~crc);
#endif
  return crc32c_portable(data, n, crc);
}

// ---- layout ---------------------------------------------------------------------------------------------------------
namespace {

const char kMagic[8] = {'G', 'P', 'R', 'S', 'N', 'A', 'P', '\0'};
const uint8_t kZeros[8] = {0, 0, 0, 0, 0, 0, 0, 0};

struct Out {
  std::string b;
  void raw(const void* p, size_t n) { b.append(static_cast<const char*>(p), n); }
  void u8(uint8_t v) { raw(&v, 1); }
  void u32(uint32_t v) { raw(&v, 4); }
  void u64(uint64_t v) { raw(&v, 8); }
  void i64(int64_t v) { raw(&v, 8); }
  void f64(double v) { raw(&v, 8); }
  void str(const std::string& s) {
    u32((uint32_t)s.size());
    raw(s.data(), s.size());
  }
  void pad8() { b.append((8 - b.size() % 8) % 8, '\0'); }
};

// Bounded reader: every take checks the room first, so no input can make it read past the buffer.
struct In {
  const uint8_t* p;
  size_t n, at = 0;
  bool ok = true;
  const char* section = "header";
  bool take(size_t k, const uint8_t** out) {
    if (!ok || k > n - at) return ok = false;
    *out = p + at, at += k;
    return true;
  }
  template <typename V>
  V get() {
    V v{};
    const uint8_t* q;
    if (take(sizeof v, &q)) memcpy(&v, q, sizeof v);
    return v;
  }
  std::string str() {
    const uint32_t k = get<uint32_t>();
    const uint8_t* q;
    if (!take(k, &q)) return std::string();
    return std::string(reinterpret_cast<const char*>(q), k);
  }
  void pad8() {
    const uint8_t* q;
    take((8 - at % 8) % 8, &q);
  }
  // an array of `count` elements of V at an offset the layout keeps aligned for V: refused before the multiplication
  // can overflow
  template <typename V>
  const V* array(uint64_t count) {
    const uint8_t* q = nullptr;
    if (!ok || count > (n - at) / sizeof(V)) {
      ok = false;
      return nullptr;
    }
    take((size_t)count * sizeof(V), &q);
    return reinterpret_cast<const V*>(q);
  }
};

uint64_t f64_bits(double d) {
  uint64_t b;
  memcpy(&b, &d, 8);
  return b;
}

// magic .. session, padded to 8 bytes
std::string head_bytes(const SnapshotKey& key, const SnapshotState& st) {
  Out o;
  o.raw(kMagic, 8);
  o.u32(kSnapshotVersion);
  o.u32(st.with_power ? kSnapshotPower : 0u);
  // fingerprint
  o.i64(st.span), o.i64(st.step);
  o.u32(st.T), o.u32(st.pods_cap), o.u32(st.G), o.u32(0);
  o.f64(st.power_threshold);
  for (const std::string& s : key.selectors) o.str(s);
  o.i64(st.t_end);
  // session
  o.u32((uint32_t)st.pods.size());
  for (const PodEntry& pe : st.pods) {
    o.str(pe.name), o.str(pe.ns);
    o.u32(pe.power_slots), o.u8(pe.has_groups ? 1 : 0);
    o.u32((uint32_t)pe.slots.size());
    for (const GpuSlot& g : pe.slots) {
      o.str(g.hostname), o.str(g.container), o.str(g.gpu), o.str(g.model), o.str(g.node_type);
      o.u8(g.from_prof ? 1 : 0), o.u32(g.group);
    }
  }
  o.u64(st.known.size());
  for (const SnapshotState::Known& k : st.known) o.u64(k.h1), o.u64(k.h2), o.u32(k.result), o.u32(k.pod), o.u32(k.slot);
  for (const std::vector<uint64_t>& keys : st.power_keys) {
    o.u32((uint32_t)keys.size());
    for (uint64_t k : keys) o.u64(k);
  }
  o.u32((uint32_t)st.prof_sigs.size());
  for (const auto& ps : st.prof_sigs) {
    o.u32(ps.first.first), o.u32(ps.first.second), o.u32((uint32_t)ps.second.size());
    for (const std::string& s : ps.second) o.str(s);
  }
  o.u32((uint32_t)st.prof_rows.size());
  for (const auto& r : st.prof_rows) o.u32(r.first), o.u32(r.second);
  o.pad8();
  return o.b;
}

const char* check_state(const SnapshotState& st) {
  if (st.step <= 0 || st.span <= 0 || st.T == 0 || st.G == 0) return "empty grid";
  if ((int64_t)st.T != (st.span + st.step - 1) / st.step) return "window length, step and columns disagree";
  if (st.pods.size() > st.pods_cap || (uint64_t)st.pods_cap * st.G > 0x7fffffffull) return "more pods than rows";
  if (st.power_keys.size() != st.pods.size()) return "power keys do not match the pods";
  const uint32_t P = (uint32_t)st.pods.size();
  for (const PodEntry& pe : st.pods) {
    if (pe.slots.size() > st.G || pe.power_slots > st.G) return "a pod has more slots than the window";
    for (const GpuSlot& g : pe.slots)
      if (g.group >= pe.slots.size()) return "a slot's group is not a slot of its pod";
  }
  for (const SnapshotState::Known& k : st.known) {
    if ((k.h1 == 0 && k.h2 == 0) || k.result > 2) return "bad known-series entry";
    if (k.result == 2 && (k.pod >= P || k.slot >= st.G)) return "a known series is placed outside the window";
  }
  for (const auto& ps : st.prof_sigs)
    if (ps.first.first >= P) return "PROF signature of an unknown pod";
  for (const auto& r : st.prof_rows)
    if (r.first >= P || r.second >= st.G) return "PROF row outside the window";
  return nullptr;
}

}  // namespace

bool parse_snapshot(const uint8_t* buf, size_t n, SnapshotKey* key, SnapshotState* st, ChunkPlaneView planes[2],
                    std::string* why, double* crc_ms) {
  auto refuse = [&](const std::string& w) {
    *why = w;
    return false;
  };
  if (n < 16 || memcmp(buf, kMagic, 8) != 0) return refuse("bad magic (not a gpu-pruner snapshot)");
  uint32_t version;
  memcpy(&version, buf + 8, 4);
  if (version != kSnapshotVersion)
    return refuse("format version " + std::to_string(version) + ", this build reads " + std::to_string(kSnapshotVersion));
  if (n < 16 + 12) return refuse("truncated (no trailer)");
  uint64_t total;
  uint32_t want;
  memcpy(&total, buf + n - 12, 8);
  memcpy(&want, buf + n - 4, 4);
  if (total != n) return refuse("truncated: the trailer says " + std::to_string(total) + " bytes, the file has " + std::to_string(n));
  const auto t0 = std::chrono::steady_clock::now();
  const uint32_t got = crc32c(buf, n - 4);
  if (crc_ms) *crc_ms = ms_since(t0);
  if (got != want) {
    char b[96];
    snprintf(b, sizeof b, "checksum mismatch (CRC32C %08x, trailer %08x)", got, want);
    return refuse(b);
  }
  In in{buf, n - 12};
  in.at = 12;
  const uint32_t flags = in.get<uint32_t>();
  in.section = "fingerprint";
  st->span = in.get<int64_t>(), st->step = in.get<int64_t>();
  st->T = in.get<uint32_t>(), st->pods_cap = in.get<uint32_t>(), st->G = in.get<uint32_t>();
  (void)in.get<uint32_t>();
  st->power_threshold = in.get<double>();
  for (std::string& s : key->selectors) s = in.str();
  key->span = st->span, key->power_threshold = st->power_threshold;
  st->t_end = in.get<int64_t>();
  st->with_power = (flags & kSnapshotPower) != 0;
  in.section = "session";
  const uint32_t P = in.get<uint32_t>();
  st->pods.clear();
  for (uint32_t p = 0; in.ok && p < P; ++p) {
    PodEntry pe;
    pe.name = in.str(), pe.ns = in.str();
    pe.power_slots = in.get<uint32_t>(), pe.has_groups = in.get<uint8_t>() != 0;
    const uint32_t S = in.get<uint32_t>();
    for (uint32_t s = 0; in.ok && s < S && s <= st->G; ++s) {
      GpuSlot g;
      g.hostname = in.str(), g.container = in.str(), g.gpu = in.str(), g.model = in.str(), g.node_type = in.str();
      g.from_prof = in.get<uint8_t>() != 0, g.group = in.get<uint32_t>();
      pe.slots.push_back(std::move(g));
    }
    if (S > st->G) return refuse("session: a pod has more slots than the window");
    st->pods.push_back(std::move(pe));
  }
  const uint64_t n_known = in.get<uint64_t>();
  if (n_known > (in.n - in.at) / 28) return refuse("truncated or malformed session (known series)");
  st->known.resize(in.ok ? (size_t)n_known : 0);
  for (SnapshotState::Known& k : st->known)
    k.h1 = in.get<uint64_t>(), k.h2 = in.get<uint64_t>(), k.result = in.get<uint32_t>(), k.pod = in.get<uint32_t>(),
    k.slot = in.get<uint32_t>();
  st->power_keys.assign(in.ok ? P : 0, {});
  for (std::vector<uint64_t>& keys : st->power_keys) {  // (not 8-byte aligned: read value by value)
    const uint32_t m = in.get<uint32_t>();
    if (m > (in.n - in.at) / 8) in.ok = false;
    for (uint32_t j = 0; in.ok && j < m; ++j) keys.push_back(in.get<uint64_t>());
  }
  const uint32_t n_sigs = in.get<uint32_t>();
  st->prof_sigs.clear();
  for (uint32_t i = 0; in.ok && i < n_sigs; ++i) {
    std::pair<std::pair<uint32_t, uint32_t>, std::vector<std::string>> ps;
    ps.first.first = in.get<uint32_t>(), ps.first.second = in.get<uint32_t>();
    const uint32_t m = in.get<uint32_t>();
    for (uint32_t j = 0; in.ok && j < m; ++j) ps.second.push_back(in.str());
    st->prof_sigs.push_back(std::move(ps));
  }
  const uint32_t n_prof = in.get<uint32_t>();
  if (n_prof > (in.n - in.at) / 8) in.ok = false;
  st->prof_rows.clear();
  for (uint32_t i = 0; in.ok && i < n_prof; ++i) {
    const uint32_t pod = in.get<uint32_t>();
    st->prof_rows.emplace_back(pod, in.get<uint32_t>());
  }
  in.pad8();
  if (!in.ok) return refuse(std::string("truncated or malformed ") + in.section);
  if (const char* bad = check_state(*st)) return refuse(std::string("session: ") + bad);
  for (int k = 0; k < 2; ++k) {
    planes[k] = ChunkPlaneView();
    if (k == 1 && !st->with_power) break;
    in.section = k == 0 ? "plane 0" : "plane 1";
    ChunkPlaneView& v = planes[k];
    v.n_series = in.get<uint64_t>(), v.n_chunks = in.get<uint64_t>(), v.n_bytes = in.get<uint64_t>();
    if (v.n_series > 0xffffffffull) return refuse(std::string(in.section) + ": too many series");
    v.series_chunks = in.array<uint64_t>(v.n_series + (in.ok ? 1 : 0));
    v.rows = in.array<uint32_t>(v.n_series);
    in.pad8();
    v.chunk_bytes = in.array<uint64_t>(v.n_chunks + (in.ok ? 1 : 0));
    v.data = in.array<uint8_t>(v.n_bytes);
    in.pad8();
    if (!in.ok) return refuse(std::string("truncated or malformed ") + in.section);
    if (v.series_chunks[v.n_series] != v.n_chunks || v.chunk_bytes[v.n_chunks] != v.n_bytes)
      return refuse(std::string(in.section) + ": the chunk index does not match its counts");
  }
  if (in.at != in.n) return refuse("bytes after the last plane");
  return true;
}

// ---- save / restore -------------------------------------------------------------------------------------------------
namespace {

bool write_all(int fd, const void* p, size_t n) {
  const char* c = static_cast<const char*>(p);
  while (n) {
    const ssize_t k = ::write(fd, c, n > (1u << 30) ? (1u << 30) : n);
    if (k < 0 && errno == EINTR) continue;
    if (k <= 0) return false;
    c += k, n -= (size_t)k;
  }
  return true;
}

std::string sys_error(const char* what, const std::string& path) {
  return std::string(what) + " " + path + ": " + strerror(errno);
}

}  // namespace

bool save_snapshot(DeviceIngestSession& session, const SnapshotKey& key, const std::string& path, SnapshotTimes* t,
                   std::string* error) {
  const auto t0 = std::chrono::steady_clock::now();
  error->clear();
  *t = SnapshotTimes();
  SnapshotState st;
  if (!session.save_state(&st)) return false;
  ChunkPlaneView planes[2];
  try {
    session.export_planes(planes, &t->export_ms, &t->copy_ms);
  } catch (const std::exception& e) {
    *error = std::string("export: ") + e.what();
    return false;
  }
  // the file as pieces written back to back: no copy of the plane arrays
  const std::string head = head_bytes(key, st);
  std::vector<std::pair<const void*, size_t>> pieces{{head.data(), head.size()}};
  std::string counts[2];
  uint64_t total = head.size();
  auto add = [&](const void* p, size_t n) {
    if (n) pieces.emplace_back(p, n);
    total += n;
  };
  for (int k = 0; k < (st.with_power ? 2 : 1); ++k) {
    const ChunkPlaneView& v = planes[k];
    Out o;
    o.u64(v.n_series), o.u64(v.n_chunks), o.u64(v.n_bytes);
    counts[k] = o.b;
    add(counts[k].data(), counts[k].size());
    add(v.series_chunks, (v.n_series + 1) * 8);
    add(v.rows, v.n_series * 4);
    add(kZeros, (8 - total % 8) % 8);
    add(v.chunk_bytes, (v.n_chunks + 1) * 8);
    add(v.data, v.n_bytes);
    add(kZeros, (8 - total % 8) % 8);
  }
  total += 12;
  const auto tc = std::chrono::steady_clock::now();
  uint32_t crc = 0;
  for (const auto& pc : pieces) crc = crc32c(pc.first, pc.second, crc);
  crc = crc32c(&total, 8, crc);
  t->crc_ms = ms_since(tc);
  uint8_t trailer[12];
  memcpy(trailer, &total, 8), memcpy(trailer + 8, &crc, 4);
  pieces.emplace_back(trailer, 12);
  // PATH.tmp, fsync, rename over PATH: a crash mid-write leaves the previous snapshot as it was
  const auto tw = std::chrono::steady_clock::now();
  const std::string tmp = path + ".tmp";
  const int fd = ::open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
  if (fd < 0) {
    *error = sys_error("cannot create", tmp);
    return false;
  }
  bool ok = true;
  for (const auto& pc : pieces)
    if (!(ok = write_all(fd, pc.first, pc.second))) break;
  if (!ok) *error = sys_error("cannot write", tmp);
  else if (::fsync(fd) != 0) ok = false, *error = sys_error("cannot fsync", tmp);
  if (::close(fd) != 0 && ok) ok = false, *error = sys_error("cannot close", tmp);
  if (ok && ::rename(tmp.c_str(), path.c_str()) != 0) ok = false, *error = sys_error("cannot rename over", path);
  if (!ok) {
    ::unlink(tmp.c_str());
    return false;
  }
  // the rename itself is durable once the directory is
  const size_t slash = path.rfind('/');
  const std::string dir = slash == std::string::npos ? "." : (slash == 0 ? "/" : path.substr(0, slash));
  const int dfd = ::open(dir.c_str(), O_RDONLY | O_DIRECTORY | O_CLOEXEC);
  if (dfd >= 0) ::fsync(dfd), ::close(dfd);
  t->write_ms = ms_since(tw);
  t->bytes = total;
  t->total_ms = ms_since(t0);
  return true;
}

bool restore_snapshot(DeviceIngestSession& session, const SnapshotKey& key, const std::string& path, SnapshotTimes* t,
                      std::string* why, bool retime) {
  const auto t0 = std::chrono::steady_clock::now();
  *t = SnapshotTimes();
  session.invalidate();
  const int fd = ::open(path.c_str(), O_RDONLY | O_CLOEXEC);
  if (fd < 0) {
    *why = errno == ENOENT ? "no snapshot file at " + path : sys_error("cannot open", path);
    return false;
  }
  struct stat sb;
  std::vector<uint64_t> buf;  // 8-byte aligned: the plane arrays are read in place
  bool ok = ::fstat(fd, &sb) == 0;
  const size_t n = ok ? (size_t)sb.st_size : 0;
  if (ok) {
    buf.resize((n + 7) / 8);
    char* p = reinterpret_cast<char*>(buf.data());
    for (size_t got = 0; ok && got < n;) {
      const ssize_t k = ::read(fd, p + got, n - got);
      if (k < 0 && errno == EINTR) continue;
      if (k <= 0) ok = false;
      else got += (size_t)k;
    }
  }
  if (!ok) *why = sys_error("cannot read", path);
  ::close(fd);
  if (!ok) return false;
  t->read_ms = ms_since(t0);
  t->bytes = n;
  SnapshotKey have;
  SnapshotState st;
  ChunkPlaneView planes[2];
  if (!parse_snapshot(reinterpret_cast<const uint8_t*>(buf.data()), n, &have, &st, planes, why, &t->crc_ms)) return false;
  // taken for another window: the CLI or the window length changed since (a shorter window is retimed from a longer
  // one by the first delta tick when `retime`)
  if (have.span != key.span && !(retime && have.span > key.span)) {
    *why = "fingerprint mismatch: window of " + std::to_string(have.span) + " s, now " + std::to_string(key.span) + " s";
    return false;
  }
  if (f64_bits(have.power_threshold) != f64_bits(key.power_threshold)) {
    char b[128];
    snprintf(b, sizeof b, "fingerprint mismatch: power threshold %.17g, now %.17g", have.power_threshold, key.power_threshold);
    *why = b;
    return false;
  }
  // The selectors end with the window as their range ("[<minutes>m]", promql.cpp render_selectors): a retimed
  // snapshot's selectors are compared with this run's rendered at the snapshot's window, so every other part must match.
  const std::string now_range = "[" + std::to_string(key.span / 60) + "m]";
  const std::string then_range = "[" + std::to_string(have.span / 60) + "m]";
  auto at_snapshot_window = [&](std::string sel) {
    if (have.span != key.span && sel.size() >= now_range.size() &&
        sel.compare(sel.size() - now_range.size(), now_range.size(), now_range) == 0)
      sel.replace(sel.size() - now_range.size(), now_range.size(), then_range);
    return sel;
  };
  static const char* kNames[3] = {"util", "prof", "power"};
  for (int i = 0; i < 3; ++i)
    if (have.selectors[i] != at_snapshot_window(key.selectors[i])) {
      *why = std::string("fingerprint mismatch: the ") + kNames[i] + " selector changed";
      return false;
    }
  const auto tr = std::chrono::steady_clock::now();
  try {
    session.restore_state(st, planes);
  } catch (const std::exception& e) {
    *why = std::string("ring not restored: ") + e.what();
    return false;
  }
  t->restore_ms = ms_since(tr);
  t->total_ms = ms_since(t0);
  return true;
}

// ---- the controller's view ----------------------------------------------------------------------------------------
namespace {

class FileSnapshots : public WindowSnapshots {
 public:
  FileSnapshots(std::string path, SnapshotKey key, std::function<DeviceIngestSession*(std::string*)> session, bool retime)
      : path_(std::move(path)), key_(std::move(key)), session_(std::move(session)), retime_(retime) {}

  bool restore(std::string* line) override {
    std::string err;
    DeviceIngestSession* s = session_(&err);
    if (!s) {
      *line = "Snapshot not restored (" + err + "): starting from the full range";
      return false;
    }
    SnapshotTimes t;
    std::string why;
    if (!restore_snapshot(*s, key_, path_, &t, &why, retime_)) {
      *line = "Snapshot not restored (" + why + "): starting from the full range";
      return false;
    }
    char b[400];
    snprintf(b, sizeof b,
             "Snapshot restored from %s: %llu bytes in %.1f ms (read %.1f, checksum %.1f, restore %.1f ms), resident "
             "window up to %lld",
             path_.c_str(), (unsigned long long)t.bytes, t.total_ms, t.read_ms, t.crc_ms, t.restore_ms,
             (long long)s->resident_t_end());
    *line = b;
    return true;
  }

  int save(std::string* line) override {
    std::string err;
    DeviceIngestSession* s = session_(&err);
    if (!s) {
      *line = err;
      return -1;
    }
    SnapshotTimes t;
    if (!save_snapshot(*s, key_, path_, &t, &err)) {
      *line = err;
      return err.empty() ? 0 : -1;
    }
    char b[400];
    snprintf(b, sizeof b,
             "Snapshot written to %s: %llu bytes in %.1f ms (export %.1f, copy %.1f, checksum %.1f, write %.1f ms)",
             path_.c_str(), (unsigned long long)t.bytes, t.total_ms, t.export_ms, t.copy_ms, t.crc_ms, t.write_ms);
    *line = b;
    return 1;
  }

 private:
  std::string path_;
  SnapshotKey key_;
  std::function<DeviceIngestSession*(std::string*)> session_;
  bool retime_;
};

}  // namespace

std::unique_ptr<WindowSnapshots> make_file_snapshots(std::string path, SnapshotKey key,
                                                     std::function<DeviceIngestSession*(std::string*)> session,
                                                     bool retime) {
  return std::make_unique<FileSnapshots>(std::move(path), std::move(key), std::move(session), retime);
}

}  // namespace gph
