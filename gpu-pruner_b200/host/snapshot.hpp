// snapshot.hpp — daemon mode's resident window as a file, so a restarted `gpu-pruner -d` resumes where it stopped
// instead of asking Prometheus for the whole [Nm] range again (--snapshot-file, DESIGN.md §8i).
//
// A snapshot holds what DeviceIngestSession carries between ticks (the pod / slot skeleton, the table of known series,
// the power keys, the PROF rows) and the ring itself as Prometheus XOR chunks, encoded on the GPU by
// gpr_resident_export and restored by gpr_chunks_scatter(GPR_TEXT_RESIDENT), which checks every chunk before it
// writes.  The file ends in its length and a CRC32C of everything before it; the reader checks magic, version, length
// and CRC before it parses anything, and never reads past the buffer, whatever the bytes are.
#pragma once
#include <cstdint>
#include <functional>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "ingest.hpp"

namespace gph {

class DeviceIngestSession;
class WindowSnapshots;

// CRC32C (Castagnoli, reflected, init and xor-out 0xFFFFFFFF).  `crc` is the CRC of the bytes before `data` (0 to
// start), so a file can be checked piece by piece.  Uses the SSE4.2 crc32 instruction when the CPU has it.
uint32_t crc32c(const void* data, size_t n, uint32_t crc = 0);
uint32_t crc32c_portable(const void* data, size_t n, uint32_t crc = 0);  // slice-by-8 tables, any CPU

constexpr uint32_t kSnapshotVersion = 1;  // bump when the layout, or Assigner's hash128, changes
constexpr uint32_t kSnapshotPower = 1u;   // flags bit 0: the power plane is present

// One plane of the ring as gpr_chunk_export's CSR, in host memory (views: the owner keeps the arrays alive).
struct ChunkPlaneView {
  uint64_t n_series = 0, n_chunks = 0, n_bytes = 0;
  const uint64_t* series_chunks = nullptr;  // n_series + 1
  const uint32_t* rows = nullptr;           // n_series
  const uint64_t* chunk_bytes = nullptr;    // n_chunks + 1
  const uint8_t* data = nullptr;            // n_bytes
};

// What a snapshot is keyed on besides the ring's own shape: a snapshot whose key differs was taken for another window.
struct SnapshotKey {
  int64_t span = 0;               // --duration * 60
  double power_threshold = 0.0;   // what the power plane is snapped to (0 = no power clause); compared bit for bit
  std::string selectors[3];       // util, prof, power as rendered from the CLI: --namespace, --model-name and
                                  // --honor-labels live there
};

// The session between two ticks (DeviceIngestSession::save_state / restore_state).  Everything Assigner can rebuild
// from these (its pod hash table) is rebuilt, not stored.
struct SnapshotState {
  int64_t span = 0, step = 0, t_end = 0;  // t_end: newest second of the resident window
  uint32_t T = 0, pods_cap = 0, G = 0;
  bool with_power = false;
  double power_threshold = 0.0;
  std::vector<PodEntry> pods;
  struct Known {
    uint64_t h1, h2;
    uint32_t result, pod, slot;  // Assigner::Result, and where the series went
  };
  std::vector<Known> known;
  std::vector<std::vector<uint64_t>> power_keys;  // per pod
  std::vector<std::pair<std::pair<uint32_t, uint32_t>, std::vector<std::string>>> prof_sigs;  // (pod, group) -> sigs
  std::vector<std::pair<uint32_t, uint32_t>> prof_rows;
};

struct SnapshotTimes {
  uint64_t bytes = 0;
  double export_ms = 0, copy_ms = 0;  // save: encode on the device, copy to the host
  double read_ms = 0;                 // restore: the file into memory
  double crc_ms = 0;                  // checksum
  double write_ms = 0;                // save: write + fsync + rename
  double restore_ms = 0;              // restore: ring init + chunk scatter + session
  double total_ms = 0;
};

// Parses and checks a whole file held in `buf` (8-byte aligned).  The plane views point into buf.  false: *why says
// what is wrong.
bool parse_snapshot(const uint8_t* buf, size_t n, SnapshotKey* key, SnapshotState* st, ChunkPlaneView planes[2],
                    std::string* why, double* crc_ms = nullptr);

// Session-level save and restore, shared by the binary and the emulated device's tests.
// save: false with an empty *error = nothing resident to save; false with *error = the write failed (the previous
// file, if any, is intact: the new one goes to PATH.tmp, is fsync'ed and renamed over PATH).
bool save_snapshot(DeviceIngestSession& session, const SnapshotKey& key, const std::string& path, SnapshotTimes* t,
                   std::string* error);
// restore: false = refused, *why says why, and the session is cold (nothing resident).  A snapshot whose key differs
// from `key` is refused — except, with `retime` (--retime-ring), a longer window than key.span: the session is restored
// at the snapshot's shape and its first delta tick retimes the ring to the shorter window.
bool restore_snapshot(DeviceIngestSession& session, const SnapshotKey& key, const std::string& path, SnapshotTimes* t,
                      std::string* why, bool retime = false);

// The controller's view (controller.hpp WindowSnapshots) of a snapshot file.  `session` returns the ingestor's
// resident session (nullptr + error: none can be had); it is asked every time, since the engine may replace it.
std::unique_ptr<WindowSnapshots> make_file_snapshots(std::string path, SnapshotKey key,
                                                     std::function<DeviceIngestSession*(std::string*)> session,
                                                     bool retime = false);

}  // namespace gph
