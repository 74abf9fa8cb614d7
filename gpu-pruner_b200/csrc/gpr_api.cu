// gpr_api.cu — the C ABI of include/gpr.h over the sm_90a kernels.
//
// Seam replaced in the reference (paths relative to the reference repository):
//   gpu-pruner/src/main.rs:397-437   send PromQL, decode instant vector, dedup by (pod, ns)
//   gpu-pruner/src/main.rs:494,508   age gate
// The library never falls back to a CPU path: every entry point that computes needs a CUDA
// device and reports GPR_E_CUDA otherwise.
#include "../../include/gpr.h"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>
#include <nvtx3/nvToolsExt.h>  // header-only; ranges show up in nsys / ncu --nvtx timelines

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <thread>
#include <utility>
#include <vector>

#include "gpr_kernels.cuh"
#include "gpr_groups.cuh"
#include "gpr_probe.cuh"
#include "gpr_ring.cuh"
#include "gpr_synth.cuh"
#include "gpr_text_kernels.cuh"
#include "gpr_samples.cuh"
#include "gpr_chunks.cuh"
#include "gpr_chunks_encode.cuh"

namespace {

using gpr::kLdgUnroll;
using gpr::kLdgWarps;
using gpr::kTmaSmemBudget;
using gpr::kProbeSmemBudget;
constexpr int kSlots = 256;      // outstanding async results
constexpr int kMaxChunkEvents = 64;
constexpr int kExchangeDepth = 4;  // exchange buffer sets of the fused multi-GPU path = 2 x scratch sets

std::mutex g_err_mu;
char g_create_err[512] = "";

// ---- NCCL, loaded on demand so the library itself has no hard dependency on it ----------
struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t,
                            cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
NcclApi g_nccl;
std::mutex g_nccl_mu;

bool load_nccl(char* err, size_t n) {
  std::lock_guard<std::mutex> lk(g_nccl_mu);
  if (g_nccl.ok) return true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* nm : names) {
    g_nccl.handle = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
    if (g_nccl.handle) break;
  }
  if (!g_nccl.handle) {
    snprintf(err, n, "NCCL not loadable: %s", dlerror());
    return false;
  }
#define GPR_SYM(field, name)                                              \
  g_nccl.field = reinterpret_cast<decltype(g_nccl.field)>(dlsym(g_nccl.handle, name)); \
  if (!g_nccl.field) {                                                    \
    snprintf(err, n, "NCCL symbol %s missing", name);                     \
    return false;                                                         \
  }
  GPR_SYM(GetUniqueId, "ncclGetUniqueId")
  GPR_SYM(CommInitRank, "ncclCommInitRank")
  GPR_SYM(CommDestroy, "ncclCommDestroy")
  GPR_SYM(AllGather, "ncclAllGather")
  GPR_SYM(GetErrorString, "ncclGetErrorString")
#undef GPR_SYM
  g_nccl.ok = true;
  return true;
}

struct Pending {
  gpr_result* res;
  int slot;
};

// ---- what a context owns: every buffer, event and stream of a gpr_ctx is one of these and releases itself when the
// context is deleted, so gpr_destroy lists none of them.  A buffer counts in elements of T and lives in device memory,
// or (kPinned) in pinned host memory from cudaHostAlloc with the given flags.
template <typename T, bool kPinned = false>
struct Buf {
  T* p = nullptr;
  size_t cap = 0;
  Buf() = default;
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
  ~Buf() { release(); }
  operator T*() const { return p; }
  cudaError_t release() {
    const cudaError_t e = !p ? cudaSuccess : kPinned ? cudaFreeHost(p) : cudaFree(p);
    p = nullptr, cap = 0;
    return e;
  }
  // exactly n elements in place of what is held (nothing may still use it)
  cudaError_t alloc(size_t n, unsigned flags = cudaHostAllocDefault) {
    cudaError_t e = release();
    void* q = nullptr;
    if (e == cudaSuccess) e = kPinned ? cudaHostAlloc(&q, n * sizeof(T), flags) : cudaMalloc(&q, n * sizeof(T));
    if (e == cudaSuccess) p = static_cast<T*>(q), cap = n;
    return e;
  }
  // n elements on first use; later calls keep what is held
  cudaError_t alloc_once(size_t n, unsigned flags = cudaHostAllocDefault) { return p ? cudaSuccess : alloc(n, flags); }
  // The growth rule of the context's scratch: nothing happens while cap >= need.  Otherwise the work on `st` that may
  // still read the buffer is waited for and need + need / 4 + 64 elements replace it (a caller that must know
  // whether it grew compares cap).
  cudaError_t grow(cudaStream_t st, size_t need) {
    if (need <= cap) return cudaSuccess;
    if (p) {
      const cudaError_t e = cudaStreamSynchronize(st);
      if (e != cudaSuccess) return e;
    }
    return alloc(need + need / 4 + 64);
  }
  // trade what is held with o (a buffer built beside this one takes its place)
  void swap(Buf& o) {
    std::swap(p, o.p);
    std::swap(cap, o.cap);
  }
};
template <typename T>
using PinnedBuf = Buf<T, true>;

// an event or a stream; create() makes it on first use and keeps it after
template <typename H, cudaError_t (*Create)(H*, unsigned), cudaError_t (*Destroy)(H)>
struct Handle {
  H h = nullptr;
  Handle() = default;
  Handle(const Handle&) = delete;
  Handle& operator=(const Handle&) = delete;
  ~Handle() {
    if (h) Destroy(h);
  }
  operator H() const { return h; }
  cudaError_t create(unsigned flags) { return h ? cudaSuccess : Create(&h, flags); }
};
using Event = Handle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;
using Stream = Handle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;

}  // namespace

struct gpr_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;  // the caller's (never destroyed here) unless own_stream
  bool own_stream = false;
  Stream copy_stream;
  Event ev_k0, ev_k1, ev_t0, ev_t1, ev_join;
  Event ev_chunk[kMaxChunkEvents];
  int sm_count = 0;
  size_t l2_bytes = 0, hbm_bytes = 0;
  int cc_major = 0, cc_minor = 0;
  char name[64] = "";
  int variant = GPR_KERNEL_AUTO;
  int ldg_ctas_per_sm = 2;
  int tma_depth_max = 3;
  int tma_warps = 16;
  int tma_chunk_bytes = 8192;
  size_t chunk_bytes = 32u << 20;
  int parse_ctas_per_sm = 6;   // k_text_parse: 4 warps and 37 KB of shared memory per CTA (GPR_PARSE_CTAS)

  // capacity for host windows
  uint32_t max_pods = 0, max_gpus = 0, max_samples = 0;
  bool cap_power = false;
  Buf<float> d_util_stage;
  Buf<float> d_power_stage;
  Buf<uint8_t> d_elig_stage;
  Buf<int64_t> d_created_stage;

  // scratch (grown on demand)
  // Two scratch sets used alternately by successive single-launch decisions so that a launch may
  // start (programmatic dependent launch) while its predecessor is still folding.
  Buf<uint32_t> d_masks[2];     // each [idle P | veto P], all-zero between uses
  bool masks_dirty = false;     // a failed call may have left bits behind
  Buf<unsigned int> d_tickets;          // [2] fold-grid tickets
  Buf<unsigned long long> d_acc;        // [2][3] fold-grid count accumulators
  Buf<unsigned long long> d_done;       // [2] completed folds per scratch set
  unsigned long long uses[2] = {0, 0};        // folds issued per scratch set
  unsigned parity = 0;
  bool pdl_enabled = true;      // GPR_PDL=0 disables programmatic dependent launch
  bool last_was_reduce = false; // the newest op on the stream is one of our fold kernels
  Buf<uint32_t> d_bits;    // [dbits W | cbits W]
  Buf<uint32_t> d_gather;  // [world][2W]
  Buf<float> d_smax;
  // `sum by` groups (gpr_window.groups, gpr_groups.cuh): single-buffered, so a decision with a table runs without PDL
  Buf<uint32_t> d_grouped;   // [P][MW] rows of groups of two or more
  Buf<uint32_t> d_gpods;     // [1 + P]: count, then the pods with such groups
  Buf<float> d_gmax;         // [P*G] max of the grouped rows when the caller did not ask for series_max
  Buf<uint32_t> d_gtable;    // [P*G] a host table, uploaded
  Buf<uint32_t> d_islots;    // [P][MW] idle_slots for host outputs
  unsigned int* h_gerr = nullptr;  // host-mapped: 1 + a pod whose device group table is malformed
  PinnedBuf<unsigned long long> h_counts;  // [kSlots][4]: n_series, n_candidates, n_decisions,
                                           // %globaltimer at completion; then [mark, error word]
  unsigned long long* h_mark = nullptr;    // %globaltimer written by the last gpr_timer_begin
  unsigned int* h_err = nullptr;           // raised by a kernel whose peer wait timed out (h_gerr is the next word)
  std::vector<Pending> pending;
  std::vector<uint64_t> stamps;            // completion stamps of the decisions retired by the last gpr_sync
  std::vector<uint64_t> phase_stamps;      // 4 per decision: fold start, folded, flags raised, peers arrived
  unsigned long long rdv_seq = 0;          // rendezvous sequence number (same on all ranks)

  Buf<unsigned char> d_flush;

  // resident window (daemon mode)
  Buf<float> d_res_util;
  Buf<float> d_res_power;
  uint32_t res_P = 0, res_G = 0, res_T = 0, res_head = 0;
  // optional index (GPR_F_BLOCK_INDEX): max of every 64-sample block of every resident row, kept up to
  // date by gpr_append.  max-of-block-maxima == max-of-samples (NaN = block without a sample), so the
  // index is itself a window tensor with ceil(T/64) "samples" per series and the same kernels decide on it
  Buf<float> d_idx_util;
  Buf<float> d_idx_power;
  uint32_t idx_ld = 0;      // padded to a multiple of 4 (TMA-able rows), padding stays NaN
  // gpr_text_parse(GPR_TEXT_RESIDENT) merged samples into the ring behind the index's back: deciding on the index
  // is refused until gpr_resident_reindex has rebuilt it
  bool idx_stale = false;
  Buf<float> d_cols;
  // gpr_resident_remap builds the new ring here, beside the old one, and the two change places once it is complete:
  // [util, power, util index, power index]
  Buf<float> d_res_next[4];
  Buf<uint32_t> d_remap_map;            // a host map, uploaded
  Buf<unsigned int> d_remap_check;      // a device map's check: [first bad new row | seen bitmap | dup bitmap]
  Buf<uint32_t> d_live;                 // gpr_resident_live_rows' bitmap for a host destination
  Buf<uint32_t> d_band;                 // gpr_resident_cols' band for a host destination

  // device-side ingest of response text (gpr_text_scan / gpr_text_parse)
  Buf<uint8_t> d_text[3];
  uint64_t text_n[3] = {0, 0, 0};
  Buf<gpr::text::Span> d_spans;
  Buf<float> d_tplane[2];
  // The text goes up in chunks through a few producer threads (pageable text is staged through a small pinned
  // ring) and every chunk is scanned as soon as it has landed; the markers of a chunk are written by the scan
  // kernel straight into a block of mapped pinned memory (ScanPipe, gpr_text_scan_begin / _next).
  static constexpr int kUpThreads = 16, kUpSlots = 2;
  // chunk size.  Pageable text: GPR_TEXT_CHUNK_MB (1..16), default 2 — the pinned staging ring is
  // up_threads x 2 x chunk, and page-locking it is paid by the first scan of a process, so a small chunk keeps
  // that set-up cheap.  Pinned / device text needs no staging and goes in 16 MB pieces.
  // Whatever the chunk, its markers are collected per scan unit of at most kScanUnit bytes, one marker block
  // each: the room per byte of text is the same for every source and chunk size.
  static constexpr size_t kPinnedChunk = 16u << 20;
  static constexpr size_t kScanUnit = 2u << 20;
  static constexpr int kMarkBlocks = 64;                   // ring of marker blocks (units in flight ahead of the consumer)
  static constexpr uint32_t kMarkCap = 16384;              // markers of one kind per unit (2 MB: one per 128 B)
  size_t up_chunk = 2u << 20;
  size_t up_slot_bytes = 0;            // up_chunk + a page (the 16 bytes of overlap, page aligned)
  PinnedBuf<unsigned char> h_up_ring;  // [up_threads][kUpSlots][up_slot_bytes]
  PinnedBuf<uint32_t> h_mark_blocks;   // [kMarkBlocks][2 + 2 * kMarkCap], device-mapped (8 MB)
  Buf<uint32_t> d_mark_blocks;         // the same in device memory: the scan appends here (atomics), then publishes
  Stream up_stream[kUpThreads];
  Event up_event[kUpThreads][kUpSlots];
  Event mark_event[kMarkBlocks];
  int up_threads = 8;                  // GPR_TEXT_UPLOAD_THREADS (1..16)
  struct ScanPipe* pipe = nullptr;     // the scan in progress (gpr_text_scan_begin .. last gpr_text_scan_next)

  // decoded samples (gpr_samples_scatter).  A host batch goes up in pieces of gpr::samples::kHostPiece samples through
  // two device buffers (and, for pageable memory, two pinned ones): piece k + 1 is copied while piece k is scattered.
  Buf<uint64_t> d_soffsets;            // a host batch's offsets and rows, uploaded whole (12 B per series)
  Buf<uint32_t> d_srows;
  Buf<unsigned long long> d_sstats;    // [n_oow, n_tiny, check word, n_in, first bad chunk]
  Buf<unsigned char> d_sstage;         // [2][ts kHostPiece | values kHostPiece]
  PinnedBuf<unsigned char> h_sstage;   // the same, pinned
  Event ev_sup[2];                     // piece in buffer b uploaded
  Event ev_sdone[2];                   // piece in buffer b scattered
  // XOR chunks (gpr_chunks_scatter) share that staging, and d_soffsets / d_srows for a host batch's series_chunks
  // and rows
  Buf<uint64_t> d_cbytes;              // a host batch's chunk_bytes, uploaded whole (8 B per chunk)
  // the resident ring exported as XOR chunks (gpr_resident_export, gpr_chunks_encode.cuh)
  Buf<uint32_t> d_xsizes;              // [rows][ceil(T / per_chunk)]: the bytes of each chunk
  Buf<uint64_t> d_xrows;               // [2][rows + 1]: chunks and bytes per row, then their exclusive scans
  Buf<uint32_t> d_xseries;             // [rows + 1]: the series index of each row
  Buf<unsigned long long> d_xtotals;   // [4]: chunks, bytes, series, samples
  Buf<unsigned char> d_xout;           // host outputs, encoded here first: [series_chunks | chunk_bytes | rows | data]

  // multi-GPU
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1;
  // fused exchange over peer memory (gpr_p2p_init / gpr_p2p_attach)
  Buf<unsigned char> p2p_block;                  // [flags u64 x kMaxPeers | rendezvous flags | gather[4][world][stride] | slots[4][world][stride]]
  unsigned char* p2p_peer[gpr::kMaxPeers] = {};  // peer-mapped base of every rank's block (self = local)
  // Exchange buffers are kExchangeDepth deep (step % depth), twice the number of scratch sets: with the late
  // output ordering a rank may push step n + 4 only after every peer has consumed step n (see k_fold)
  size_t p2p_gather_off[kExchangeDepth] = {};
  size_t p2p_ll_off[kExchangeDepth] = {};        // tagged 64-bit slot arrays [world][stride], one per step % depth
  bool exchange_ll = true;                       // tagged 64-bit slots (default); GPR_EXCHANGE=flags: data + fence + flag
  bool exchange_late = false;                    // GPR_EXCHANGE=pipelined: tagged slots, and a fold waits for its
                                                 // predecessor only before it writes the caller's outputs
  int fold_threads = 256;                        // GPR_FOLD_THREADS: 64 / 128 / 256 threads per fold CTA
  uint32_t p2p_stride = 0;                       // words per rank slot = 2 * W_max
  bool p2p_ready = false;
  int exchange_debug = 0;                        // GPR_DEBUG_EXCHANGE (developer timing switch)
  unsigned int poll_ns = 4000;                   // GPR_POLL_NS: longest pause between polls of the peers' flags
  unsigned long long p2p_step = 0;

  uint64_t launches = 0;
  char err[512] = "";
};

void scan_pipe_abort(gpr_ctx* ctx);   // defined with the text ingest below

namespace {

int fail(gpr_ctx* c, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (c) {
    snprintf(c->err, sizeof c->err, "%s", buf);
  } else {
    std::lock_guard<std::mutex> lk(g_err_mu);
    snprintf(g_create_err, sizeof g_create_err, "%s", buf);
  }
  return code;
}

#define CU(call)                                                                          \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess)                                                                \
      return fail(ctx, e_ == cudaErrorMemoryAllocation ? GPR_E_NOMEM : GPR_E_CUDA,        \
                  "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__);   \
  } while (0)

#define NC(call)                                                                          \
  do {                                                                                    \
    ncclResult_t r_ = (call);                                                             \
    if (r_ != ncclSuccess)                                                                \
      return fail(ctx, GPR_E_NCCL, "%s: %s", #call, g_nccl.GetErrorString(r_));           \
  } while (0)

int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return (v && *v) ? atoi(v) : dflt;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Whether both host arrays are pinned (registered with CUDA); pageable ones go up through pinned staging.
bool host_pinned(const void* a, const void* b) {
  bool pinned = true;
  for (const void* p : {a, b}) {
    if (!p) continue;
    cudaPointerAttributes at;
    pinned = pinned && cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeHost;
    (void)cudaGetLastError();  // an unregistered pointer may leave an error code behind
  }
  return pinned;
}

// smallest f32 >= thr, so that (m >= thr_f) in f32 equals ((double)m >= thr) for every f32 m
float threshold_f32(double thr) { return gpr::text::threshold_up(thr); }

bool power_truthy(double thr) { return thr != 0.0 && !std::isnan(thr); }

// the context's tuning knobs as the launch geometry (gpr_launch.h) takes them
gpr::LaunchKnobs launch_knobs(const gpr_ctx* ctx) {
  gpr::LaunchKnobs k;
  k.sm_count = ctx->sm_count;
  k.variant = ctx->variant;
  k.ldg_ctas_per_sm = ctx->ldg_ctas_per_sm;
  k.tma_warps = ctx->tma_warps;
  k.tma_chunk_bytes = ctx->tma_chunk_bytes;
  k.tma_depth_max = ctx->tma_depth_max;
  k.fold_threads = ctx->fold_threads;
  return k;
}

// The prologue of every entry point that enqueues work on the context's stream or waits for it.  Whatever the call
// enqueues is not one of our folds, so the next decision's reduce must not start early behind it (programmatic
// dependent launch is requested only while last_was_reduce holds, DESIGN.md §4).
int enter(gpr_ctx* ctx) {
  ctx->last_was_reduce = false;
  CU(cudaSetDevice(ctx->device));
  return GPR_OK;
}

// Every kernel on the context's stream is launched here, and counted (gpr_launch_count).  `pdl` adds the
// programmatic-stream-serialization attribute so the kernel may begin while the previous reduce kernel on the stream
// drains.
template <typename Kernel, typename... Args>
int launch(gpr_ctx* ctx, Kernel k, uint32_t grid, uint32_t block, size_t smem, bool pdl, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid), cfg.blockDim = dim3(block), cfg.dynamicSmemBytes = smem, cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  ctx->launches++;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, k, std::forward<Args>(args)...);
  CU(cudaGetLastError());  // (a failed launch leaves its error here too: this clears it)
  CU(e);
  return GPR_OK;
}

// ceil(n / per_cta) CTAs, at most per_sm per SM and at least one
uint32_t capped_grid(const gpr_ctx* ctx, uint64_t n, uint64_t per_cta, uint32_t per_sm) {
  return (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((n + per_cta - 1) / per_cta, (uint64_t)ctx->sm_count * per_sm));
}

// launch one reduce pass over the rows described by rp (kGroups: the instantiation for a group table)
template <bool kGroups>
int launch_reduce_as(gpr_ctx* ctx, gpr::ReduceParams& rp, bool tma_ok, bool pdl) {
  if (rp.total_rows == 0) return GPR_OK;
  // AUTO = the probe kernel when every row may stop early, else the TMA pipeline (DESIGN.md §4.3); rows
  // that are not 16-byte aligned or have T % 4 != 0 cannot be bulk-copied and take the LDG kernel.
  // Rows may stop unless the call asks for series_max (the host-side form of rows_may_stop) or has a group table.
  const bool may_stop = !kGroups && rp.seg[0].smax == nullptr && rp.seg[1].smax == nullptr;
  const gpr::ReducePlan plan =
      gpr::plan_reduce(launch_knobs(ctx), rp.T, rp.total_rows, tma_ok, rp.util_u8 != 0, may_stop);
  if (plan.kernel == gpr::kReduceProbe)
    return launch(ctx, gpr::k_reduce_probe<gpr::kProbeWarps>, plan.grid, plan.block, plan.smem, pdl, rp, plan.L);
  if (plan.kernel == gpr::kReduceU8)
    return launch(ctx, gpr::k_reduce_u8<kLdgWarps, gpr::kU8Unroll, kGroups>, plan.grid, plan.block, 0, pdl, rp);
  if (plan.kernel == gpr::kReduceTma) {
    const int nw = ctx->tma_warps;
    const auto k = nw == 4    ? gpr::k_reduce_tma<4, kGroups>
                   : nw == 16 ? gpr::k_reduce_tma<16, kGroups>
                   : nw == 32 ? gpr::k_reduce_tma<32, kGroups>
                              : gpr::k_reduce_tma<8, kGroups>;
    return launch(ctx, k, plan.grid, plan.block, plan.smem, pdl, rp, plan.L);
  }
  return launch(ctx, gpr::k_reduce_ldg<kLdgWarps, kLdgUnroll, kGroups>, plan.grid, plan.block, 0, pdl, rp);
}
int launch_reduce(gpr_ctx* ctx, gpr::ReduceParams& rp, bool tma_ok, bool pdl) {
  return rp.grouped ? launch_reduce_as<true>(ctx, rp, tma_ok, pdl) : launch_reduce_as<false>(ctx, rp, tma_ok, pdl);
}

// n_rows rows of T elements, `ld` elements apart in src, to dense rows at dst: one plain copy when src is dense too
int copy_rows(gpr_ctx* ctx, void* dst, const void* src, size_t n_rows, uint64_t T, uint64_t ld, size_t esize,
              cudaMemcpyKind kind, cudaStream_t s) {
  if (n_rows == 0) return GPR_OK;
  if (ld == T) {
    CU(cudaMemcpyAsync(dst, src, n_rows * (size_t)T * esize, kind, s));
  } else {
    CU(cudaMemcpy2DAsync(dst, (size_t)T * esize, src, (size_t)ld * esize, (size_t)T * esize, n_rows, kind, s));
  }
  return GPR_OK;
}

struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

// What a decision reads (the caller's window, or the resident ring or its block index) and its shape, as read_window
// resolved and checked it
struct Window {
  uint32_t P, G, T;
  uint32_t MW, W, S;        // mask words per pod, bitmap words, series
  uint64_t ld;              // elements between rows
  const float* util;        // biased bytes when u8
  const float* power;
  const uint32_t* groups;   // nullptr for a caller built before gpr_window.groups existed
  uint32_t* idle_slots;     // nullptr for a caller built before gpr_result.idle_slots existed
  bool u8, use_power;
  bool host_in;             // util and power are in host memory and go up in pieces through the staging planes
  bool host_arrays;         // the gates and the group table are in host memory (mem_kind, for the ring too)
  bool grouped;             // a group table over one pod or more
  bool fused, comm;         // the bitmaps are exchanged between ranks (fused: over peer memory, else by NCCL)
};

// Every check of a decision, before anything is enqueued: the structs, the window, the result, the exchange, the host
// group table and the staging capacity.
int read_window(gpr_ctx* ctx, const gpr_window* win, const gpr_result* res, bool resident, Window* w) {
  if (!win || !res) return fail(ctx, GPR_E_INVALID, "window/result is NULL");
  // a caller built before gpr_window.groups / gpr_result.idle_slots existed passes the older sizes: no such fields
  const size_t win_v1 = offsetof(gpr_window, groups), res_v1 = offsetof(gpr_result, idle_slots);
  if ((win->struct_size != sizeof(gpr_window) && win->struct_size != win_v1) ||
      (res->struct_size != sizeof(gpr_result) && res->struct_size != res_v1))
    return fail(ctx, GPR_E_INVALID, "struct_size mismatch (window %u/%zu or %zu, result %u/%zu or %zu)",
                win->struct_size, sizeof(gpr_window), win_v1, res->struct_size, sizeof(gpr_result), res_v1);
  const uint32_t* const groups = win->struct_size == sizeof(gpr_window) ? win->groups : nullptr;
  uint32_t* const idle_slots = res->struct_size == sizeof(gpr_result) ? res->idle_slots : nullptr;
  CU(cudaSetDevice(ctx->device));

  uint32_t P = win->n_pods, G = win->n_gpus, T = win->n_samples;
  uint64_t ld = win->row_stride ? win->row_stride : T;
  const float* util = win->util;
  const float* power = win->power;
  int in_kind = win->mem_kind;
  const bool u8 = !resident && win->util_format == GPR_FMT_U8B;
  if (!resident && win->util_format != GPR_FMT_F32 && win->util_format != GPR_FMT_U8B)
    return fail(ctx, GPR_E_INVALID, "bad util_format %u", win->util_format);
  if (resident) {
    if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window (gpr_resident_init)");
    P = ctx->res_P, G = ctx->res_G, T = ctx->res_T, ld = T;
    util = ctx->d_res_util;
    power = ctx->d_res_power;
    if (ctx->d_idx_util) {  // decide on the block-maxima index: same verdict, T/64 of the bytes
      if (ctx->idx_stale)
        return fail(ctx, GPR_E_STATE, "the block index is stale: gpr_text_parse(GPR_TEXT_RESIDENT) merged samples "
                    "into the ring; call gpr_resident_reindex before gpr_decide_resident");
      T = ctx->idx_ld, ld = ctx->idx_ld;
      util = ctx->d_idx_util;
      power = ctx->d_idx_power;
    }
  }
  if (in_kind != GPR_MEM_HOST && in_kind != GPR_MEM_DEVICE)
    return fail(ctx, GPR_E_INVALID, "bad mem_kind %d", in_kind);
  if (res->out_mem_kind != GPR_MEM_HOST && res->out_mem_kind != GPR_MEM_DEVICE)
    return fail(ctx, GPR_E_INVALID, "bad out_mem_kind %d", res->out_mem_kind);
  if (G == 0 || T == 0) return fail(ctx, GPR_E_INVALID, "n_gpus and n_samples must be > 0");
  if (G > 256) return fail(ctx, GPR_E_UNSUPPORTED, "n_gpus %u > 256 series slots per pod is not supported", G);
  const uint32_t MW = (G + 31u) / 32u;  // mask words per pod
  if (ld < T) return fail(ctx, GPR_E_INVALID, "row_stride %llu < n_samples %u",
                          (unsigned long long)ld, T);
  if (P > 0 && !util) return fail(ctx, GPR_E_INVALID, "util is NULL");
  if (!res->decision_bits && P > 0) return fail(ctx, GPR_E_INVALID, "decision_bits is NULL");
  const uint64_t S64 = (uint64_t)P * G;
  if (S64 > 0x7fffffffull) return fail(ctx, GPR_E_INVALID, "too many series (%llu)",
                                       (unsigned long long)S64);
  const uint32_t S = (uint32_t)S64;
  const uint32_t W = (P + 31u) / 32u;
  const bool use_power = power != nullptr && power_truthy(win->power_threshold);
  const bool host_in = !resident && in_kind == GPR_MEM_HOST;
  const bool fused = ctx->p2p_ready && ctx->world > 1;
  const bool comm = (ctx->comm != nullptr || fused) && ctx->world > 1;
  if (fused && 2u * W > ctx->p2p_stride)
    return fail(ctx, GPR_E_CAPACITY, "n_pods %u exceeds the p2p exchange capacity (%u pods per rank)", P,
                ctx->p2p_stride * 16u);
  if (comm && (P % 32u) != 0)
    return fail(ctx, GPR_E_INVALID, "with a communicator n_pods must be a multiple of 32 (got %u)", P);
  if ((int)ctx->pending.size() >= kSlots)
    return fail(ctx, GPR_E_STATE, "too many outstanding async results; call gpr_sync");
  // a host group table is checked here, before anything is enqueued (a device table by k_group_rows)
  const bool grouped = groups != nullptr && P > 0;
  if (grouped && in_kind == GPR_MEM_HOST) {
    for (uint32_t p = 0; p < P; ++p) {
      const uint32_t* e = groups + (size_t)p * G;
      for (uint32_t g = 0; g < G; ++g) {
        const uint32_t x = e[g], l = x & gpr::kGroupLeader;
        if ((x & ~(gpr::kGroupLeader | gpr::kGroupUtil)) != 0u || l > g || (e[l] & gpr::kGroupLeader) != l)
          return fail(ctx, GPR_E_INVALID, "gpr_window.groups: malformed entry 0x%x at pod %u slot %u (leader above its "
                      "slot, a leader that does not lead itself, or bits other than 0-7 and GPR_GROUP_UTIL)", x, p, g);
      }
    }
  }

  if (host_in) {
    // staging is dense, so only the number of cells matters: a window with one more GPU slot or a few more
    // samples than the shape given at gpr_create still fits as long as the product does
    if ((uint64_t)P * G * T > (uint64_t)ctx->max_pods * ctx->max_gpus * ctx->max_samples)
      return fail(ctx, GPR_E_CAPACITY, "host window %ux%ux%u exceeds the staging capacity of %ux%ux%u cells", P, G, T,
                  ctx->max_pods, ctx->max_gpus, ctx->max_samples);
    if (use_power && !ctx->cap_power)
      return fail(ctx, GPR_E_CAPACITY, "power plane not reserved (GPR_F_POWER_PLANE)");
  }
  w->P = P, w->G = G, w->T = T, w->MW = MW, w->W = W, w->S = S, w->ld = ld;
  w->util = util, w->power = power, w->groups = groups, w->idle_slots = idle_slots;
  w->u8 = u8, w->use_power = use_power, w->host_in = host_in, w->host_arrays = in_kind == GPR_MEM_HOST;
  w->grouped = grouped, w->fused = fused, w->comm = comm;
  return GPR_OK;
}

int decide_impl(gpr_ctx* ctx, const gpr_window* win, gpr_result* res, bool resident, bool async) {
  NvtxRange nvtx_range(resident ? "gpr_decide_resident" : "gpr_decide");
  Window w{};
  int rc = read_window(ctx, win, res, resident, &w);
  if (rc != GPR_OK) return rc;
  const uint32_t P = w.P, G = w.G, T = w.T, MW = w.MW, W = w.W, S = w.S;
  const bool use_power = w.use_power, host_in = w.host_in, grouped = w.grouped, fused = w.fused;
  const bool nccl = w.comm && !w.fused;  // the bitmaps are gathered by ncclAllGather after the fold
  const bool host_out = res->out_mem_kind == GPR_MEM_HOST;

  // ---- scratch ---------------------------------------------------------------------------
  const unsigned sset = ctx->parity;  // scratch set of this call; successive calls alternate
  ctx->parity ^= 1u;
  if (ctx->masks_dirty) {  // a failed launch may also have left ticket / accumulators behind
    CU(cudaMemsetAsync(ctx->d_tickets, 0, 2 * sizeof(unsigned int), ctx->stream));
    CU(cudaMemsetAsync(ctx->d_acc, 0, 6 * sizeof(unsigned long long), ctx->stream));
    ctx->last_was_reduce = false;
  }
  for (int k = 0; k < 2; ++k) {
    const size_t cap_before = ctx->d_masks[k].cap;
    CU(ctx->d_masks[k].grow(ctx->stream, (size_t)2 * P * MW + 16));
    if (ctx->d_masks[k].cap != cap_before || ctx->masks_dirty) {
      CU(cudaMemsetAsync(ctx->d_masks[k], 0, ctx->d_masks[k].cap * sizeof(uint32_t), ctx->stream));
      ctx->last_was_reduce = false;
    }
  }
  ctx->masks_dirty = false;
  uint32_t* const masks = ctx->d_masks[sset];
  CU(ctx->d_bits.grow(ctx->stream, (size_t)3 * W + 2));
  if (nccl) CU(ctx->d_gather.grow(ctx->stream, (size_t)ctx->world * 2 * W + 2));
  const bool want_smax = res->series_max != nullptr;
  if (want_smax && host_out) CU(ctx->d_smax.grow(ctx->stream, (size_t)S + 4));
  if (w.idle_slots && host_out) CU(ctx->d_islots.grow(ctx->stream, (size_t)P * MW + 4));
  if (grouped) {
    CU(ctx->d_grouped.grow(ctx->stream, (size_t)P * MW + 4));
    CU(ctx->d_gpods.grow(ctx->stream, (size_t)P + 4));
    if (!want_smax) CU(ctx->d_gmax.grow(ctx->stream, (size_t)S + 4));
    if (w.host_arrays) CU(ctx->d_gtable.grow(ctx->stream, (size_t)S + 4));
  }

  // ---- gates -----------------------------------------------------------------------------
  const uint8_t* d_elig = win->eligible;
  const int64_t* d_created = win->created_ts;
  if (w.host_arrays && (win->eligible || win->created_ts)) {
    CU(ctx->d_elig_stage.grow(ctx->stream, P));
    CU(ctx->d_created_stage.grow(ctx->stream, P));
    ctx->last_was_reduce = false;
    if (win->eligible) {
      CU(cudaMemcpyAsync(ctx->d_elig_stage, win->eligible, P, cudaMemcpyHostToDevice, ctx->stream));
      d_elig = ctx->d_elig_stage;
    }
    if (win->created_ts) {
      CU(cudaMemcpyAsync(ctx->d_created_stage, win->created_ts, (size_t)P * sizeof(int64_t),
                         cudaMemcpyHostToDevice, ctx->stream));
      d_created = ctx->d_created_stage;
    }
  }

  // ---- output targets --------------------------------------------------------------------
  const bool direct_bits = !host_out && !w.comm;
  uint32_t* dbits_dev = direct_bits ? res->decision_bits : ctx->d_bits;
  uint32_t* cbits_dev = direct_bits ? res->candidate_bits
                                    : ((res->candidate_bits || w.comm) ? ctx->d_bits + W : nullptr);
  // pods vetoed by the power clause: never exchanged (this rank's pods only)
  uint32_t* vbits_dev = res->veto_bits ? (host_out ? ctx->d_bits + 2 * (size_t)W : res->veto_bits) : nullptr;
  uint32_t* my_gather = nullptr;  // local gather buffer of this call (fused exchange)
  const unsigned xset = (unsigned)((ctx->p2p_step + 1ull) % kExchangeDepth);  // exchange buffers of this step
  if (fused) {
    my_gather = reinterpret_cast<uint32_t*>(ctx->p2p_block + ctx->p2p_gather_off[xset]);
    dbits_dev = my_gather + (size_t)ctx->rank * ctx->p2p_stride;   // this rank's slot: [decision | candidate]
    cbits_dev = dbits_dev + W;
  }
  // (a series_max target also tells the reduce kernels to read every row whole: the true max is an output; without
  // one they stop reading a row at the first sample that settles its flag, gpr_kernels.cuh "early exit")
  float* smax_dev = want_smax ? (host_out ? ctx->d_smax : res->series_max) : nullptr;
  uint32_t* islots_dev = w.idle_slots ? (host_out ? ctx->d_islots : w.idle_slots) : nullptr;

  gpr::FoldParams fp{};
  fp.idle_mask = masks;
  fp.veto_mask = use_power ? masks + (size_t)P * MW : nullptr;
  fp.eligible = d_elig;
  fp.created = d_created;
  fp.cutoff = win->cutoff_ts;
  fp.dbits = dbits_dev;
  fp.cbits = cbits_dev;
  fp.vbits = vbits_dev;
  // single-launch path: the last CTA stores the three counters straight into this call's
  // pinned (device-mapped, UVA) host slot, so no copy operation separates back-to-back steps
  const int slot = (int)ctx->pending.size();
  unsigned long long* h_slot = ctx->h_counts + (size_t)slot * 8;
  fp.counts = h_slot;
  fp.stamp = h_slot + 3;
  fp.err = ctx->h_err;
  fp.acc = ctx->d_acc + 3 * sset;
  fp.ticket = ctx->d_tickets + sset;
  fp.done = ctx->d_done + sset;
  fp.need = ctx->uses[sset];
  fp.prev_done = ctx->d_done + (sset ^ 1u);
  fp.prev_need = ctx->uses[sset ^ 1u];
  fp.P = P;
  fp.G = G;
  fp.mw = MW;
  fp.world = 1;
  fp.poll_ns = ctx->poll_ns;
  fp.islots = islots_dev;
  if (fused) {
    fp.exchange_debug = ctx->exchange_debug;
    fp.world = ctx->world, fp.rank = ctx->rank;
    fp.rank_stride = ctx->p2p_stride;
    for (int r = 0; r < ctx->world; ++r) {
      fp.peer_gather[r] = reinterpret_cast<uint32_t*>(ctx->p2p_peer[r] + ctx->p2p_gather_off[xset]);
      fp.peer_flag[r] = reinterpret_cast<unsigned long long*>(ctx->p2p_peer[r]) + ctx->rank;
    }
    fp.my_flags = reinterpret_cast<const unsigned long long*>(ctx->p2p_block.p);
    if (ctx->exchange_ll) {
      for (int r = 0; r < ctx->world; ++r)
        fp.peer_ll[r] = reinterpret_cast<unsigned long long*>(ctx->p2p_peer[r] + ctx->p2p_ll_off[xset]);
      fp.my_ll = reinterpret_cast<unsigned long long*>(ctx->p2p_block + ctx->p2p_ll_off[xset]);
      // (veto bits and idle_slots go straight to the caller's buffers from every fold CTA, so such a call keeps the
      // early wait)
      fp.late_order = ctx->exchange_late && vbits_dev == nullptr && islots_dev == nullptr ? 1 : 0;
    }
    fp.step = ++ctx->p2p_step;
    fp.out_dbits = host_out ? nullptr : res->decision_bits;
    fp.out_cbits = host_out ? nullptr : res->candidate_bits;
  }

  gpr::ReduceParams rp{};
  rp.ld = host_in ? T : w.ld;  // staging is dense
  rp.T = T;
  rp.G = G;
  rp.mw = MW;
  rp.thr = threshold_f32(win->power_threshold);
  rp.done = fp.done;
  rp.need = fp.need;
  rp.util_u8 = w.u8 ? 1u : 0u;
  const bool can_pdl = ctx->pdl_enabled && ctx->own_stream;
  // the fold grid: 32 bitmap words per CTA and round; a handful of CTAs even at millions of pods
  // one bitmap word per warp and round, 4 words per warp in flight (fold_words<4>): small CTAs spread the fold's
  // loads over many SMs — each SM's path to L2 is busy with the next decision's reduce CTA
  const uint32_t fold_threads = (uint32_t)ctx->fold_threads;
  const uint32_t fold_grid = gpr::fold_grid(launch_knobs(ctx), P);

  // ---- `sum by` groups: the table's kernels around the reduce (gpr_groups.cuh) -----------------
  gpr::GroupParams gq{};
  if (grouped) {
    gq.table = w.groups;
    if (w.host_arrays) {
      CU(cudaMemcpyAsync(ctx->d_gtable, w.groups, (size_t)S * 4u, cudaMemcpyHostToDevice, ctx->stream));
      gq.table = ctx->d_gtable;
    }
    gq.need = ctx->d_grouped;
    gq.n_pods = ctx->d_gpods;
    gq.pods = ctx->d_gpods + 1;
    gq.gmax = want_smax ? smax_dev : ctx->d_gmax;
    gq.idle_mask = masks;
    gq.bad = ctx->h_gerr;
    gq.P = P, gq.G = G, gq.mw = MW;
    ctx->last_was_reduce = false;   // the group scratch is single-buffered: no PDL into or out of this decision
  }
  const uint32_t group_grid = gpr::group_grid(launch_knobs(ctx), P);

  if (!async) {
    CU(cudaEventRecord(ctx->ev_k0, ctx->stream));
    ctx->last_was_reduce = false;
  }

  // ---- the reduce over the window's pieces of whole pods, then the fold --------------------------
  // A device window is one piece, read in place.  A host window is cut into pieces of chunk_bytes: each is copied
  // into the dense staging planes on the copy stream, and its reduce waits for that copy only, so the next piece's
  // copy overlaps it.
  if (host_in) {
    ctx->last_was_reduce = false;
    CU(cudaEventRecord(ctx->ev_join, ctx->stream));
    CU(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_join, 0));
  }
  if (P > 0) {
    // The reduce grid may start while the previous decision's fold is still running, but only
    // when that is provably safe: our own stream (no foreign producer kernels between), the
    // newest op on it is one of our fold kernels, and this launch writes nothing but its own
    // scratch set (series_max would go straight to the caller's buffer).
    // (nor with a group table: k_group_rows writes the table's single-buffered scratch; nor behind a staging copy)
    const bool chain = can_pdl && !host_in;
    const bool reduce_pdl = chain && ctx->last_was_reduce && !want_smax && !grouped;
    const size_t usize = w.u8 ? 1u : 4u;  // bytes per util sample on the wire and in the staging plane
    const size_t pod_bytes = (size_t)G * T * (usize + (use_power ? 4u : 0u));
    const uint32_t piece_pods =
        host_in ? (uint32_t)std::max<size_t>(1, ctx->chunk_bytes / std::max<size_t>(pod_bytes, 1)) : P;
    const uint32_t n_pieces = (P + piece_pods - 1) / piece_pods;
    // bulk copies need rows of a multiple of 4 samples at 16-byte aligned addresses (the staging planes are dense)
    const bool tma_ok = (T % 4u) == 0 &&
                        (host_in || ((w.ld % 4u) == 0 && aligned16(w.util) && (!use_power || aligned16(w.power))));
    if (grouped) {
      CU(cudaMemsetAsync(ctx->d_gpods, 0, sizeof(uint32_t), ctx->stream));
      if ((rc = launch(ctx, gpr::k_group_rows, group_grid, gpr::kGroupBlock, 0, false, gq)) != GPR_OK) return rc;
    }
    for (uint32_t c = 0; c < n_pieces; ++c) {
      const uint32_t p0 = c * piece_pods, p1 = std::min(P, p0 + piece_pods);
      const size_t row0 = (size_t)p0 * G, n_rows = (size_t)(p1 - p0) * G;
      const float* pu = w.util;  // a device window's one piece (row0 = 0)
      const float* pp = w.power;
      if (host_in) {
        float* du = reinterpret_cast<float*>(reinterpret_cast<char*>(ctx->d_util_stage.p) + row0 * T * usize);
        float* dp = use_power ? ctx->d_power_stage + row0 * T : nullptr;
        if ((rc = copy_rows(ctx, du, reinterpret_cast<const char*>(w.util) + row0 * w.ld * usize, n_rows, T, w.ld,
                            usize, cudaMemcpyHostToDevice, ctx->copy_stream)) != GPR_OK)
          return rc;
        if (use_power && (rc = copy_rows(ctx, dp, w.power + row0 * w.ld, n_rows, T, w.ld, 4u, cudaMemcpyHostToDevice,
                                         ctx->copy_stream)) != GPR_OK)
          return rc;
        cudaEvent_t ev = ctx->ev_chunk[c % kMaxChunkEvents];
        CU(cudaEventRecord(ev, ctx->copy_stream));
        CU(cudaStreamWaitEvent(ctx->stream, ev, 0));
        pu = du, pp = dp;
      }
      rp.seg[0] = gpr::Segment{pu, masks + (size_t)p0 * MW, smax_dev ? smax_dev + row0 : nullptr,
                               (uint32_t)n_rows, 0u};
      rp.seg[1] = gpr::Segment{pp, masks + ((size_t)P + p0) * MW, nullptr,
                               use_power ? (uint32_t)n_rows : 0u, 1u};
      rp.total_rows = (uint32_t)n_rows * (use_power ? 2u : 1u);
      if (grouped) rp.grouped = ctx->d_grouped + (size_t)p0 * MW, rp.gmax = ctx->d_gmax ? ctx->d_gmax + row0 : nullptr;
      if ((rc = launch_reduce(ctx, rp, tma_ok, reduce_pdl)) != GPR_OK) return rc;
    }
    if (grouped && (rc = launch(ctx, gpr::k_group_sum, group_grid, gpr::kGroupBlock, 0, false, gq)) != GPR_OK)
      return rc;
    const auto fold = fused ? (islots_dev ? gpr::k_fold<true, true> : gpr::k_fold<true, false>)
                            : (islots_dev ? gpr::k_fold<false, true> : gpr::k_fold<false, false>);
    if ((rc = launch(ctx, fold, fold_grid, fold_threads, 0, chain && !grouped, fp)) != GPR_OK) return rc;
    ctx->uses[sset]++;
    ctx->last_was_reduce = !host_in && !grouped;
  }
  if (P == 0) memset(h_slot, 0, 8 * sizeof(unsigned long long));  // slot is not in flight

  // ---- the one collective: allgather of the packed bitmap over NVLink ----------------------
  if (nccl || host_out || !async) ctx->last_was_reduce = false;  // something follows
  if (nccl && W > 0) {
    NC(g_nccl.AllGather(ctx->d_bits, ctx->d_gather, (size_t)2 * W, ncclUint32, ctx->comm,
                        ctx->stream));
  }
  if (!async) CU(cudaEventRecord(ctx->ev_k1, ctx->stream));

  // ---- deliver -----------------------------------------------------------------------------
  // The decision and candidate bitmaps are `rows` rows of W words, `pitch` words apart: this rank's one row in d_bits,
  // or a row per rank in the fused exchange's gather block or in the NCCL gather buffer.  They are copied for host
  // outputs, and for device outputs only out of the NCCL buffer (otherwise the fold wrote them in place).  Veto
  // bits, series_max and idle_slots (this rank's pods) are copied out of their staging for host outputs only.
  const uint32_t* bits = fused ? my_gather : nccl ? ctx->d_gather : ctx->d_bits;
  const size_t pitch = fused ? ctx->p2p_stride : nccl ? 2 * (size_t)W : W;
  const size_t rows = w.comm ? (size_t)ctx->world : 1;
  const struct {
    void* dst;
    const void* src;
    size_t rows, words, pitch;
    bool copy;
  } outs[] = {
      {res->decision_bits, bits, rows, W, pitch, host_out || nccl},
      {res->candidate_bits, bits + W, rows, W, pitch, host_out || nccl},
      {res->veto_bits, ctx->d_bits + 2 * (size_t)W, 1, W, W, host_out},
      {res->series_max, ctx->d_smax, 1, S, S, host_out},
      {w.idle_slots, ctx->d_islots, 1, (size_t)P * MW, (size_t)P * MW, host_out},
  };
  const cudaMemcpyKind out_kind = host_out ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  for (const auto& o : outs)
    if (o.copy && o.dst && o.words > 0 &&
        (rc = copy_rows(ctx, o.dst, o.src, o.rows, o.words, o.pitch, 4u, out_kind, ctx->stream)) != GPR_OK)
      return rc;
  ctx->pending.push_back(Pending{res, slot});
  res->kernel_ms = 0.0;
  return GPR_OK;
}

// The one failure rule of a decision: whether a check refused it or a launch or copy failed after part of it was
// enqueued, the scratch may hold bits, tickets or counts of its own, so the next decision re-zeroes it first.
int decide(gpr_ctx* ctx, const gpr_window* win, gpr_result* res, bool resident, bool async) {
  if (!ctx) return GPR_E_INVALID;
  const int rc = decide_impl(ctx, win, res, resident, async);
  if (rc != GPR_OK) ctx->masks_dirty = true;
  return rc;
}

int sync_impl(gpr_ctx* ctx) {
  CU(cudaSetDevice(ctx->device));
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) {
    ctx->pending.clear();
    ctx->masks_dirty = true;
    return fail(ctx, GPR_E_CUDA, "cudaStreamSynchronize: %s", cudaGetErrorString(e));
  }
  ctx->stamps.clear();
  ctx->phase_stamps.clear();
  for (const Pending& p : ctx->pending) {
    const unsigned long long* c = ctx->h_counts + (size_t)p.slot * 8;
    p.res->n_series = c[0];
    p.res->n_candidates = c[1];
    p.res->n_decisions = c[2];
    ctx->stamps.push_back(c[3]);
    for (int k = 4; k < 8; ++k) ctx->phase_stamps.push_back(c[k]);
  }
  ctx->pending.clear();
  const unsigned int gerr = *ctx->h_gerr;
  *ctx->h_gerr = 0;
  if (*ctx->h_err) {
    *ctx->h_err = 0;
    ctx->masks_dirty = true;
    return fail(ctx, GPR_E_STATE, "a peer rank never arrived at the bitmap exchange / rendezvous (waited %llu s); "
                "the results of this batch are not global", gpr::kPeerTimeoutNs / 1000000000ull);
  }
  if (gerr) {
    ctx->masks_dirty = true;
    return fail(ctx, GPR_E_INVALID, "gpr_window.groups: malformed device group table at pod %u (leader above its slot, "
                "a leader that does not lead itself, or bits other than 0-7 and GPR_GROUP_UTIL)", gerr - 1u);
  }
  return GPR_OK;
}

}  // namespace

// ---- upload + scan pipeline ------------------------------------------------------------------------------------
// The text is cut into chunks.  A few producer threads each take every nt-th chunk: copy it into their pinned
// double buffer (pageable sources; a plain cudaMemcpy would go through the driver's single bounce buffer at
// ~10 GB/s), enqueue the H2D copy on their own stream, and right behind it the scan kernel for that chunk, which
// appends the chunk's markers to a block of mapped pinned memory.  A chunk is copied with 16 bytes of overlap
// into the next one (identical bytes written twice), so its scan never needs another stream's data.  A chunk
// is cut into scan units of at most kScanUnit bytes (unit j of chunk c is [c * chunk + j * unit, ...), global
// index c * units_per_chunk + j), and each unit's markers go to a block of their own.  The consumer
// (gpr_text_scan_next) takes the units in text order while later chunks are still in flight.
struct ScanPipe {
  int slot = 0;
  const char* src = nullptr;
  uint8_t* dst = nullptr;
  uint64_t n = 0, n_chunks = 0, chunk = 0;
  uint64_t unit = 0, units_per_chunk = 1, n_units = 0;
  int nt = 1;
  int src_kind = GPR_MEM_HOST;
  bool staged = false;  // source is pageable host memory: goes through the pinned ring
  std::vector<std::thread> th;
  std::atomic<uint64_t> consumed{0};                      // units handed to the caller
  std::atomic<uint64_t> recorded[gpr_ctx::kMarkBlocks];   // unit + 1 whose event has been recorded in this block
  std::atomic<int> error{0};                              // first cudaError_t of a producer
  std::atomic<bool> stop{false};
  uint64_t next = 0;                                      // next unit the consumer returns
};

namespace {

constexpr uint32_t kBlockWords = 2 + 2 * gpr_ctx::kMarkCap;

// markers of one chunk, each in the block of its unit, as 32-bit offsets relative to the unit:
// [n_open, n_close, opens[cap], closes[cap]] per block; the chunk's first unit has global index u0
struct ChunkSink {
  uint32_t* blocks;  // the device ring, kMarkBlocks blocks
  uint64_t base, unit, u0;
  __device__ __forceinline__ void put(uint64_t p, uint32_t which) {
    const uint64_t j = (p - base) / unit;
    uint32_t* block = blocks + (size_t)((u0 + j) % gpr_ctx::kMarkBlocks) * kBlockWords;
    const uint32_t i = atomicAdd(block + which, 1u);
    if (i < gpr_ctx::kMarkCap) block[2 + which * gpr_ctx::kMarkCap + i] = (uint32_t)(p - base - j * unit);
  }
  __device__ __forceinline__ void values_open(uint64_t p) { put(p, 0); }
  __device__ __forceinline__ void values_close(uint64_t p) { put(p, 1); }
};

// copies the markers of units u0 .. u0 + gridDim.x - 1 from their device blocks to the host-mapped ones with plain
// coalesced stores (the scan's atomic appends must not go to host memory: an atomic across PCIe costs microseconds)
__global__ void __launch_bounds__(256) k_publish_marks(const uint32_t* __restrict__ d_blocks, uint32_t* __restrict__ h_blocks,
                                                       uint64_t u0) {
  const size_t at = (size_t)((u0 + blockIdx.x) % gpr_ctx::kMarkBlocks) * kBlockWords;
  const uint32_t* d_block = d_blocks + at;
  uint32_t* h_block = h_blocks + at;
  const uint32_t no = min(d_block[0], gpr_ctx::kMarkCap), nc = min(d_block[1], gpr_ctx::kMarkCap);
  for (uint32_t i = threadIdx.x; i < no; i += blockDim.x) h_block[2 + i] = d_block[2 + i];
  for (uint32_t i = threadIdx.x; i < nc; i += blockDim.x)
    h_block[2 + gpr_ctx::kMarkCap + i] = d_block[2 + gpr_ctx::kMarkCap + i];
  if (threadIdx.x == 0) h_block[0] = d_block[0], h_block[1] = d_block[1];
}

__global__ void __launch_bounds__(256) k_text_scan_chunk(const uint8_t* __restrict__ t, uint64_t n, uint64_t slice_begin,
                                                         uint64_t slice_end, uint32_t* blocks, uint64_t unit, uint64_t u0) {
  ChunkSink sink{blocks, slice_begin * gpr::text::kScanBytes, unit, u0};
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t slice = slice_begin + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; slice < slice_end; slice += stride)
    gpr::text::scan_slice(t, n, slice, sink);
}

void scan_producer(gpr_ctx* ctx, ScanPipe* sp, int k) {
  constexpr int NS = gpr_ctx::kUpSlots, NB = gpr_ctx::kMarkBlocks;
  const size_t SLOT = ctx->up_slot_bytes;
  cudaError_t e = cudaSetDevice(ctx->device);
  bool used[NS] = {};
  int slot = 0;
  cudaStream_t st = ctx->up_stream[k];
  for (uint64_t c = (uint64_t)k; c < sp->n_chunks && e == cudaSuccess && !sp->stop.load(); c += (uint64_t)sp->nt) {
    const uint64_t off = c * sp->chunk;
    const uint64_t len = std::min<uint64_t>(sp->chunk, sp->n - off);
    const uint64_t len_ov = std::min<uint64_t>(len + 16, sp->n - off);  // overlap into the next chunk
    const uint64_t u0 = c * sp->units_per_chunk, nu = (len + sp->unit - 1) / sp->unit;
    // the marker block of unit u is free once the consumer has taken unit u - NB (NB >= units_per_chunk)
    for (int spins = 0; u0 + nu > sp->consumed.load(std::memory_order_acquire) + NB && !sp->stop.load(); ++spins) {
      if (spins < 64) std::this_thread::yield();
      else std::this_thread::sleep_for(std::chrono::microseconds(50));  // a slow consumer: do not burn the core
    }
    if (sp->stop.load()) break;
    const void* from = sp->src + off;
    if (sp->staged) {
      unsigned char* buf = ctx->h_up_ring + ((size_t)k * NS + slot) * SLOT;
      if (used[slot]) e = cudaEventSynchronize(ctx->up_event[k][slot]);  // its previous DMA has drained
      if (e != cudaSuccess) break;
      memcpy(buf, from, len_ov);
      from = buf;
    }
    e = cudaMemcpyAsync(sp->dst + off, from, len_ov,
                        sp->src_kind == GPR_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && sp->staged) e = cudaEventRecord(ctx->up_event[k][slot], st), used[slot] = true;
    slot = (slot + 1) % NS;
    if (e != cudaSuccess) break;
    // (the kernels that last used the blocks of units u0 .. u0 + nu - 1 have completed: their units were consumed)
    for (uint64_t u = u0; u < u0 + nu && e == cudaSuccess; ++u)
      e = cudaMemsetAsync(ctx->d_mark_blocks + (size_t)(u % NB) * kBlockWords, 0, 2 * sizeof(uint32_t), st);
    if (e != cudaSuccess) break;
    const uint64_t s0 = off / gpr::text::kScanBytes;
    const uint64_t s1 = (off + len + gpr::text::kScanBytes - 1) / gpr::text::kScanBytes;
    const uint32_t grid = capped_grid(ctx, s1 - s0, 256, 8);
    k_text_scan_chunk<<<grid, 256, 0, st>>>(sp->dst, sp->n, s0, s1, ctx->d_mark_blocks, sp->unit, u0);
    k_publish_marks<<<(uint32_t)nu, 256, 0, st>>>(ctx->d_mark_blocks, ctx->h_mark_blocks, u0);
    e = cudaGetLastError();
    for (uint64_t u = u0; u < u0 + nu && e == cudaSuccess; ++u) {
      e = cudaEventRecord(ctx->mark_event[u % NB], st);
      if (e == cudaSuccess) sp->recorded[u % NB].store(u + 1, std::memory_order_release);
    }
  }
  if (e != cudaSuccess) {
    int zero = 0;
    sp->error.compare_exchange_strong(zero, (int)e);
    sp->stop.store(true);
  }
}

int scan_pipe_finish(gpr_ctx* ctx, bool ok) {
  ScanPipe* sp = ctx->pipe;
  if (!sp) return GPR_OK;
  if (!ok) sp->stop.store(true);
  for (std::thread& t : sp->th) t.join();
  cudaError_t e = (cudaError_t)sp->error.load();
  // work queued on the context's stream afterwards (the parse kernels) must see the whole text
  for (int k = 0; k < sp->nt && e == cudaSuccess; ++k) {
    e = cudaEventRecord(ctx->up_event[k][0], ctx->up_stream[k]);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, ctx->up_event[k][0], 0);
  }
  if (!ok)
    for (int k = 0; k < sp->nt; ++k) cudaStreamSynchronize(ctx->up_stream[k]);
  delete sp;
  ctx->pipe = nullptr;
  if (e != cudaSuccess) return fail(ctx, GPR_E_CUDA, "text upload / scan: %s", cudaGetErrorString(e));
  return GPR_OK;
}

// the time axis of a gpr_text_grid, as gpr_text_parse and gpr_samples_scatter check it
int check_grid(gpr_ctx* ctx, const gpr_text_grid* grid) {
  if (grid->step <= 0 || grid->step > 4000000ll || grid->n_samples == 0 || grid->window_seconds <= 0 ||
      grid->window_seconds > 4000000000ll)
    return fail(ctx, GPR_E_INVALID, "step (<= 4e6 s), window_seconds and n_samples must be > 0");
  if ((grid->window_seconds + grid->step - 1) / grid->step > (int64_t)grid->n_samples)
    return fail(ctx, GPR_E_INVALID, "window of %lld s needs more than %u columns of %lld s", (long long)grid->window_seconds,
                grid->n_samples, (long long)grid->step);
  return GPR_OK;
}

// Where gpr_text_parse, gpr_samples_scatter and gpr_chunks_scatter merge samples, and its time axis in milliseconds
// (the resolution of Prometheus timestamps): the resident ring (GPR_TEXT_RESIDENT) or the context plane `plane`, grown
// to the grid (a plane that has to grow must be filled).  The caller has checked everything else, so the merge is
// certain once this succeeds: it fills the plane (GPR_TEXT_FILL) or marks the ring's index stale.
int open_destination(gpr_ctx* ctx, const gpr_text_grid* grid, int32_t plane, gpr::text::Grid* g, float** pl) {
  const uint32_t n_samples = grid->n_samples, n_rows = grid->n_rows;
  memset(g, 0, sizeof *g);
  g->t_end = grid->t_end * 1000, g->t_lo = (grid->t_end - grid->window_seconds) * 1000;
  g->step = (uint32_t)(grid->step * 1000), g->T = n_samples;
  g->power = gpr::text::power_snap(plane == 1 ? grid->power_threshold : 0.0);
  if (grid->flags & GPR_TEXT_RESIDENT) {
    if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window (gpr_resident_init)");
    if (n_samples != ctx->res_T || (uint64_t)n_rows > (uint64_t)ctx->res_P * ctx->res_G)
      return fail(ctx, GPR_E_INVALID, "grid %u rows x %u does not match the resident window (%u x %u)", n_rows, n_samples,
                  ctx->res_P * ctx->res_G, ctx->res_T);
    *pl = plane == 0 ? ctx->d_res_util : ctx->d_res_power;
    if (!*pl) return fail(ctx, GPR_E_STATE, "the resident window has no power plane");
    g->ld = ctx->res_T;
    g->col_end = (ctx->res_head + ctx->res_T - 1) % ctx->res_T;  // the newest bucket sits just before the head
    if (ctx->d_idx_util) ctx->idx_stale = true;  // the merge does not touch the index (gpr_resident_reindex)
  } else {
    const size_t cells = (size_t)n_rows * n_samples;
    const size_t cap_before = ctx->d_tplane[plane].cap;
    CU(ctx->d_tplane[plane].grow(ctx->stream, cells + 4));
    if (ctx->d_tplane[plane].cap != cap_before && !(grid->flags & GPR_TEXT_FILL))
      return fail(ctx, GPR_E_STATE, "plane %d had to grow: the first parse of a window must pass GPR_TEXT_FILL", plane);
    *pl = ctx->d_tplane[plane];
    g->ld = n_samples, g->col_end = n_samples - 1;
    // 0xFFFFFFFF: a NaN, and -1 as an int — below every non-negative sample for the integer atomicMax merge
    if ((grid->flags & GPR_TEXT_FILL) && cells) CU(cudaMemsetAsync(*pl, 0xFF, cells * sizeof(float), ctx->stream));
  }
  return GPR_OK;
}

}  // namespace

void scan_pipe_abort(gpr_ctx* ctx) {
  if (ctx && ctx->pipe) (void)scan_pipe_finish(ctx, false);
}


// ===========================================================================================
// extern "C"
// ===========================================================================================
#define GPR_TRY try {
#define GPR_CATCH(ctxp)                                                     \
  }                                                                         \
  catch (const std::bad_alloc&) {                                           \
    return fail(ctxp, GPR_E_NOMEM, "host allocation failed");               \
  }                                                                         \
  catch (...) {                                                             \
    return fail(ctxp, GPR_E_INVALID, "unexpected C++ exception");           \
  }

extern "C" {

int gpr_version(void) {
  return GPR_VERSION_MAJOR * 10000 + GPR_VERSION_MINOR * 100 + GPR_VERSION_PATCH;
}

const char* gpr_last_error(const gpr_ctx* ctx) { return ctx ? ctx->err : g_create_err; }

// The members release every buffer, event and stream when ctx is deleted; this stops what could still use them first:
// an unfinished scan's producer threads (joined, their streams drained), then the work on the context's stream.
void gpr_destroy(gpr_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  scan_pipe_abort(ctx);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  if (ctx->comm && g_nccl.ok) g_nccl.CommDestroy(ctx->comm);
  for (int r = 0; r < gpr::kMaxPeers; ++r)
    if (ctx->p2p_peer[r] && ctx->p2p_peer[r] != ctx->p2p_block) cudaIpcCloseMemHandle(ctx->p2p_peer[r]);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

int gpr_create(const gpr_config* cfg, gpr_ctx** out) {
  gpr_ctx* ctx = nullptr;  // errors before allocation go to the global slot
  GPR_TRY
  if (!cfg || !out) return fail(nullptr, GPR_E_INVALID, "config/out is NULL");
  *out = nullptr;
  if (cfg->struct_size != sizeof(gpr_config))
    return fail(nullptr, GPR_E_INVALID, "gpr_config.struct_size %u != %zu", cfg->struct_size,
                sizeof(gpr_config));
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0)
    return fail(nullptr, GPR_E_CUDA, "no CUDA device (%s); this engine has no CPU fallback",
                e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
  if (cfg->device < 0 || cfg->device >= n_dev)
    return fail(nullptr, GPR_E_INVALID, "device %d out of range [0,%d)", cfg->device, n_dev);
  gpr_ctx* c = new gpr_ctx();
  c->device = cfg->device;
  // from here on failures are reported through the global slot too, then the ctx is freed
  auto bail = [&](int code) {
    {
      std::lock_guard<std::mutex> lk(g_err_mu);
      snprintf(g_create_err, sizeof g_create_err, "%s", c->err);
    }
    gpr_destroy(c);
    return code;
  };
  ctx = c;
  auto body = [&]() -> int {
    CU(cudaSetDevice(c->device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, c->device));
    c->sm_count = prop.multiProcessorCount;
    c->l2_bytes = (size_t)prop.l2CacheSize;
    c->hbm_bytes = prop.totalGlobalMem;
    c->cc_major = prop.major, c->cc_minor = prop.minor;
    memcpy(c->name, prop.name, sizeof c->name - 1);
    // arch-specific sm_90a code loads only on compute capability 9.0 (H100 / H200)
    if (prop.major != 9 || prop.minor != 0)
      return fail(c, GPR_E_UNSUPPORTED, "device %s is sm_%d%d; this library is built for sm_90a",
                  prop.name, prop.major, prop.minor);
    if (cfg->stream) {
      c->stream = static_cast<cudaStream_t>(cfg->stream);
    } else {
      CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
      c->own_stream = true;
    }
    CU(c->copy_stream.create(cudaStreamNonBlocking));
    for (Event* ev : {&c->ev_k0, &c->ev_k1, &c->ev_t0, &c->ev_t1}) CU(ev->create(cudaEventDefault));
    CU(c->ev_join.create(cudaEventDisableTiming));
    for (Event& ev : c->ev_chunk) CU(ev.create(cudaEventDisableTiming));
    CU(c->d_acc.alloc(6));
    CU(c->d_tickets.alloc(2));
    CU(c->d_done.alloc(2));
    CU(cudaMemset(c->d_acc, 0, 6 * sizeof(unsigned long long)));
    CU(cudaMemset(c->d_tickets, 0, 2 * sizeof(unsigned int)));
    CU(cudaMemset(c->d_done, 0, 2 * sizeof(unsigned long long)));
    c->pdl_enabled = env_int("GPR_PDL", 1) != 0;
    c->up_threads = std::max(1, std::min((int)gpr_ctx::kUpThreads, env_int("GPR_TEXT_UPLOAD_THREADS", 8)));
    c->up_chunk = (size_t)std::max(1, std::min(16, env_int("GPR_TEXT_CHUNK_MB", 2))) << 20;
    c->up_slot_bytes = c->up_chunk + 4096;
    c->exchange_debug = env_int("GPR_DEBUG_EXCHANGE", 0);
    c->poll_ns = (unsigned int)std::max(100, std::min(100000, env_int("GPR_POLL_NS", 4000)));
    if (const char* x = getenv("GPR_EXCHANGE")) {
      c->exchange_ll = strcmp(x, "flags") != 0;
      c->exchange_late = strcmp(x, "pipelined") == 0;
    }
    c->fold_threads = env_int("GPR_FOLD_THREADS", 256);
    if (c->fold_threads != 64 && c->fold_threads != 128 && c->fold_threads != 256) c->fold_threads = 256;
    CU(c->h_counts.alloc((size_t)kSlots * 8 + 2));
    memset(c->h_counts, 0, c->h_counts.cap * sizeof(unsigned long long));
    c->h_mark = c->h_counts + (size_t)kSlots * 8;
    c->h_err = reinterpret_cast<unsigned int*>(c->h_mark + 1);
    c->h_gerr = c->h_err + 1;
    c->pending.reserve(kSlots);
    c->stamps.reserve(kSlots);

    c->variant = cfg->kernel_variant;
    if (const char* k = getenv("GPR_KERNEL")) {
      if (!strcmp(k, "ldg")) c->variant = GPR_KERNEL_LDG;
      else if (!strcmp(k, "tma")) c->variant = GPR_KERNEL_TMA;
    }
    if (c->variant < GPR_KERNEL_AUTO || c->variant > GPR_KERNEL_TMA)
      return fail(c, GPR_E_INVALID, "bad kernel_variant %d", c->variant);
    c->ldg_ctas_per_sm = std::max(1, env_int("GPR_LDG_CTAS", 2));
    c->tma_depth_max = std::max(1, env_int("GPR_TMA_DEPTH", 3));
    c->tma_warps = env_int("GPR_TMA_WARPS", 16);
    if (c->tma_warps != 4 && c->tma_warps != 8 && c->tma_warps != 16 && c->tma_warps != 32)
      c->tma_warps = 16;
    c->tma_chunk_bytes = std::min(65536, std::max(512, env_int("GPR_TMA_CHUNK", 8192))) & ~15;
    c->chunk_bytes = (size_t)std::max(1, env_int("GPR_CHUNK_MB", 32)) << 20;
    c->parse_ctas_per_sm = std::max(1, std::min(8, env_int("GPR_PARSE_CTAS", 6)));
    CU(cudaFuncSetAttribute(gpr::k_reduce_tma<4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)kTmaSmemBudget));
    CU(cudaFuncSetAttribute(gpr::k_reduce_tma<8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)kTmaSmemBudget));
    CU(cudaFuncSetAttribute(gpr::k_reduce_tma<16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)kTmaSmemBudget));
    CU(cudaFuncSetAttribute(gpr::k_reduce_tma<32>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)kTmaSmemBudget));
    CU(cudaFuncSetAttribute(gpr::k_reduce_probe<gpr::kProbeWarps>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)kProbeSmemBudget));
    // (the instantiations for calls with a `sum by` group table)
    CU(cudaFuncSetAttribute(gpr::k_reduce_tma<4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)kTmaSmemBudget));
    CU(cudaFuncSetAttribute(gpr::k_reduce_tma<8, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)kTmaSmemBudget));
    CU(cudaFuncSetAttribute(gpr::k_reduce_tma<16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)kTmaSmemBudget));
    CU(cudaFuncSetAttribute(gpr::k_reduce_tma<32, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            (int)kTmaSmemBudget));

    c->max_pods = cfg->max_pods, c->max_gpus = cfg->max_gpus, c->max_samples = cfg->max_samples;
    c->cap_power = (cfg->flags & GPR_F_POWER_PLANE) != 0;
    const size_t cells = (size_t)cfg->max_pods * cfg->max_gpus * cfg->max_samples;
    if (cells) {
      CU(c->d_util_stage.alloc(cells + 64));
      if (c->cap_power) CU(c->d_power_stage.alloc(cells + 64));
    }
    return GPR_OK;
  };
  int rc = body();
  if (rc != GPR_OK) return bail(rc);
  *out = c;
  return GPR_OK;
  GPR_CATCH(nullptr)
}

int gpr_decide_async(gpr_ctx* ctx, const gpr_window* win, gpr_result* res) {
  GPR_TRY
  return decide(ctx, win, res, false, true);
  GPR_CATCH(ctx)
}

int gpr_decide_batch_async(gpr_ctx* ctx, const gpr_window* wins, gpr_result* results, uint32_t n) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  if (n && (!wins || !results)) return fail(ctx, GPR_E_INVALID, "windows/results is NULL");
  for (uint32_t i = 0; i < n; ++i)
    if (const int rc = decide(ctx, &wins[i], &results[i], false, true)) return rc;
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_sync(gpr_ctx* ctx) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  return sync_impl(ctx);
  GPR_CATCH(ctx)
}

static int decide_blocking(gpr_ctx* ctx, const gpr_window* win, gpr_result* res, bool resident) {
  // like the async paths, a failed call leaves the decisions enqueued before it pending (the next gpr_sync or
  // successful blocking call fills their counters) and enqueues no result of its own
  int rc = decide(ctx, win, res, resident, false);
  if (rc != GPR_OK) return rc;
  rc = sync_impl(ctx);
  if (rc != GPR_OK) return rc;
  float ms = 0.f;
  CU(cudaEventElapsedTime(&ms, ctx->ev_k0, ctx->ev_k1));
  res->kernel_ms = ms;
  return GPR_OK;
}

int gpr_decide(gpr_ctx* ctx, const gpr_window* win, gpr_result* res) {
  GPR_TRY
  return decide_blocking(ctx, win, res, false);
  GPR_CATCH(ctx)
}

int gpr_decide_resident(gpr_ctx* ctx, const gpr_window* win, gpr_result* res) {
  GPR_TRY
  return decide_blocking(ctx, win, res, true);
  GPR_CATCH(ctx)
}

// ---- resident window -----------------------------------------------------------------------
int gpr_resident_init(gpr_ctx* ctx, uint32_t P, uint32_t G, uint32_t T, uint32_t flags) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  if (const int rc = enter(ctx)) return rc;
  if (P == 0 || G == 0 || T == 0) return fail(ctx, GPR_E_INVALID, "empty resident window");
  if ((uint64_t)P * G > 0x7fffffffull) return fail(ctx, GPR_E_INVALID, "too many series");
  CU(cudaStreamSynchronize(ctx->stream));
  for (Buf<float>* b : {&ctx->d_res_util, &ctx->d_res_power, &ctx->d_idx_util, &ctx->d_idx_power}) CU(b->release());
  ctx->idx_ld = 0;
  const size_t cells = (size_t)P * G * T;
  CU(ctx->d_res_util.alloc(cells));
  // 0xFFFFFFFF is a NaN: every step starts out "no sample"
  CU(cudaMemsetAsync(ctx->d_res_util, 0xFF, cells * sizeof(float), ctx->stream));
  if (flags & GPR_F_POWER_PLANE) {
    CU(ctx->d_res_power.alloc(cells));
    CU(cudaMemsetAsync(ctx->d_res_power, 0xFF, cells * sizeof(float), ctx->stream));
  }
  if (flags & GPR_F_BLOCK_INDEX) {
    ctx->idx_ld = gpr::index_ld(T);
    const size_t ic = (size_t)P * G * ctx->idx_ld;
    CU(ctx->d_idx_util.alloc(ic));
    CU(cudaMemsetAsync(ctx->d_idx_util, 0xFF, ic * sizeof(float), ctx->stream));
    if (flags & GPR_F_POWER_PLANE) {
      CU(ctx->d_idx_power.alloc(ic));
      CU(cudaMemsetAsync(ctx->d_idx_power, 0xFF, ic * sizeof(float), ctx->stream));
    }
  }
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->res_P = P, ctx->res_G = G, ctx->res_T = T, ctx->res_head = 0;
  ctx->idx_stale = false;
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_resident_reindex(gpr_ctx* ctx) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  if (const int rc = enter(ctx)) return rc;
  if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window (gpr_resident_init)");
  if (!ctx->d_idx_util) return GPR_OK;  // no index to maintain
  const size_t rows = (size_t)ctx->res_P * ctx->res_G;
  const uint32_t grid = gpr::ring_grid(rows, ctx->sm_count);
  int rc = launch(ctx, gpr::k_reindex, grid, gpr::kRingThreads, 0, false, ctx->d_res_util, (uint32_t)rows, ctx->res_T,
                  ctx->d_idx_util, ctx->idx_ld);
  if (rc == GPR_OK && ctx->d_res_power)
    rc = launch(ctx, gpr::k_reindex, grid, gpr::kRingThreads, 0, false, ctx->d_res_power, (uint32_t)rows, ctx->res_T,
                ctx->d_idx_power, ctx->idx_ld);
  if (rc != GPR_OK) return rc;
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->idx_stale = false;
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_append(gpr_ctx* ctx, const float* util_cols, const float* power_cols, uint32_t n_new,
               uint64_t row_stride, int32_t mem_kind) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  if (const int rc = enter(ctx)) return rc;
  if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window (gpr_resident_init)");
  if (n_new == 0) return GPR_OK;
  if (!util_cols) return fail(ctx, GPR_E_INVALID, "util_cols is NULL");
  if (mem_kind != GPR_MEM_HOST && mem_kind != GPR_MEM_DEVICE)
    return fail(ctx, GPR_E_INVALID, "bad mem_kind %d", mem_kind);
  const uint32_t T = ctx->res_T;
  const size_t rows = (size_t)ctx->res_P * ctx->res_G;
  uint64_t ld = row_stride ? row_stride : n_new;
  if (ld < n_new) return fail(ctx, GPR_E_INVALID, "row_stride < n_new");
  // only the newest T columns can survive in a ring of T
  const gpr::RingSpan sp = gpr::ring_span(ctx->res_head, n_new, T);
  const uint32_t n_eff = sp.n;
  const uint32_t grid = gpr::ring_grid(rows, ctx->sm_count);
  const float* planes_in[2] = {util_cols, power_cols};
  float* planes_out[2] = {ctx->d_res_util, ctx->d_res_power};
  float* planes_idx[2] = {ctx->d_idx_util, ctx->d_idx_power};
  for (int pl = 0; pl < 2; ++pl) {
    const gpr::RingLaunch what = gpr::append_launch(planes_out[pl] != nullptr, planes_in[pl] != nullptr);
    if (what == gpr::kRingNone) continue;
    int rc;
    if (what == gpr::kRingOpen) {  // no columns for this plane: its new buckets hold no sample
      if ((rc = launch(ctx, gpr::k_open, grid, gpr::kRingThreads, 0, false, planes_out[pl], (uint32_t)rows, T, sp.start,
                       sp.n, planes_idx[pl], ctx->idx_ld)) != GPR_OK)
        return rc;
      continue;
    }
    const float* src = planes_in[pl] + sp.src_col;
    uint64_t ld_dev = ld;
    if (mem_kind == GPR_MEM_HOST) {
      CU(ctx->d_cols.grow(ctx->stream, rows * n_eff + 4));
      if (ld == n_eff)  // dense block: one linear copy (a 2-D copy of 720-byte rows runs at ~6 GB/s)
        CU(cudaMemcpyAsync(ctx->d_cols, src, rows * (size_t)n_eff * 4u, cudaMemcpyHostToDevice,
                           ctx->stream));
      else
        CU(cudaMemcpy2DAsync(ctx->d_cols, (size_t)n_eff * 4u, src, (size_t)ld * 4u,
                             (size_t)n_eff * 4u, rows, cudaMemcpyHostToDevice, ctx->stream));
      src = ctx->d_cols;
      ld_dev = n_eff;
    }
    if ((rc = launch(ctx, gpr::k_append, grid, gpr::kRingThreads, 0, false, planes_out[pl], src, (uint32_t)rows, T,
                     sp.start, sp.n, ld_dev, planes_idx[pl], ctx->idx_ld)) != GPR_OK)
      return rc;
  }
  ctx->res_head = sp.next_head;
  CU(cudaStreamSynchronize(ctx->stream));
  return GPR_OK;
  GPR_CATCH(ctx)
}

// The first new row of a device map that gpr::remap_first_bad would name (n_new if none), by k_remap_check's two
// passes; the old row it names goes to *src.
static int remap_check_device(gpr_ctx* ctx, const uint32_t* src_rows, uint32_t n_new, uint32_t n_old, uint32_t* first,
                              uint32_t* src) {
  const size_t words = ((size_t)n_old + 31) / 32;
  CU(ctx->d_remap_check.grow(ctx->stream, 1 + 2 * words));
  unsigned int* d = ctx->d_remap_check;
  CU(cudaMemsetAsync(d + 1, 0, 2 * words * sizeof(unsigned int), ctx->stream));
  CU(cudaMemcpyAsync(d, &n_new, sizeof n_new, cudaMemcpyHostToDevice, ctx->stream));
  const uint32_t blocks = capped_grid(ctx, n_new, 256, 8);
  for (int pass = 0; pass < 2; ++pass) {
    const int rc = launch(ctx, gpr::k_remap_check, blocks, 256, 0, false, src_rows, n_new, n_old, d + 1, d + 1 + words,
                          d, pass);
    if (rc != GPR_OK) return rc;
  }
  CU(cudaMemcpyAsync(first, d, sizeof *first, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (*first < n_new) {
    CU(cudaMemcpyAsync(src, src_rows + *first, sizeof *src, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  return GPR_OK;
}

// The new ring in d_res_next, gathered from the old one on the context's stream after whatever is enqueued there (the
// decisions still pending read the old ring), and waited for.
static int remap_build(gpr_ctx* ctx, const uint32_t* map, uint32_t n_rows) {
  Buf<float>* cur[4] = {&ctx->d_res_util, &ctx->d_res_power, &ctx->d_idx_util, &ctx->d_idx_power};
  const uint32_t len[4] = {ctx->res_T, ctx->res_T, ctx->idx_ld, ctx->idx_ld};
  const uint32_t grid = gpr::ring_grid(n_rows, ctx->sm_count);
  for (int k = 0; k < 4; ++k) {
    if (!*cur[k]) continue;
    CU(ctx->d_res_next[k].alloc((size_t)n_rows * len[k]));
    const int rc = launch(ctx, gpr::k_remap_rows, grid, gpr::kRingThreads, 0, false,
                          reinterpret_cast<uint32_t*>(ctx->d_res_next[k].p), reinterpret_cast<const uint32_t*>(cur[k]->p),
                          map, n_rows, len[k]);
    if (rc != GPR_OK) return rc;
  }
  CU(cudaStreamSynchronize(ctx->stream));
  return GPR_OK;
}

int gpr_resident_remap(gpr_ctx* ctx, uint32_t n_pods, uint32_t n_gpus, const uint32_t* src_rows, int32_t mem_kind) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  NvtxRange nvtx_range("gpr_resident_remap");
  if (const int rc = enter(ctx)) return rc;
  if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window (gpr_resident_init)");
  if (n_pods == 0 || n_gpus == 0) return fail(ctx, GPR_E_INVALID, "empty resident window");
  if ((uint64_t)n_pods * n_gpus > 0x7fffffffull) return fail(ctx, GPR_E_INVALID, "too many series");
  if (!src_rows) return fail(ctx, GPR_E_INVALID, "src_rows is NULL");
  if (mem_kind != GPR_MEM_HOST && mem_kind != GPR_MEM_DEVICE) return fail(ctx, GPR_E_INVALID, "bad mem_kind %d", mem_kind);
  const uint32_t n_new = n_pods * n_gpus, n_old = ctx->res_P * ctx->res_G;
  // ---- the map is checked before the new ring is allocated or anything of the ring is written
  uint32_t first = n_new, src = 0;
  if (mem_kind == GPR_MEM_HOST) {
    first = (uint32_t)gpr::remap_first_bad(src_rows, n_new, n_old);
    if (first < n_new) src = src_rows[first];
  } else {
    const int rc = remap_check_device(ctx, src_rows, n_new, n_old, &first, &src);
    if (rc != GPR_OK) return rc;
  }
  if (first < n_new && src >= n_old)
    return fail(ctx, GPR_E_INVALID, "src_rows[%u] = %u: the resident window has %u rows (%u x %u)", first, src, n_old,
                ctx->res_P, ctx->res_G);
  if (first < n_new)
    return fail(ctx, GPR_E_INVALID, "src_rows[%u] = %u: old row %u is the source of more than one new row", first, src,
                src);
  // ---- the new ring beside the old one; they change places only once it is complete
  const uint32_t* map = src_rows;
  if (mem_kind == GPR_MEM_HOST) {
    CU(ctx->d_remap_map.grow(ctx->stream, n_new));
    CU(cudaMemcpyAsync(ctx->d_remap_map, src_rows, (size_t)n_new * sizeof(uint32_t), cudaMemcpyHostToDevice,
                       ctx->stream));
    map = ctx->d_remap_map;
  }
  const int rc = remap_build(ctx, map, n_new);
  if (rc != GPR_OK) {
    (void)cudaStreamSynchronize(ctx->stream);  // a gather may still be writing a new buffer
    for (Buf<float>& b : ctx->d_res_next) (void)b.release();
    return rc;
  }
  Buf<float>* cur[4] = {&ctx->d_res_util, &ctx->d_res_power, &ctx->d_idx_util, &ctx->d_idx_power};
  for (int k = 0; k < 4; ++k) cur[k]->swap(ctx->d_res_next[k]);
  ctx->res_P = n_pods, ctx->res_G = n_gpus;
  for (Buf<float>& b : ctx->d_res_next) CU(b.release());  // the old ring
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_resident_live_rows(gpr_ctx* ctx, uint32_t* bits, int32_t mem_kind) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  NvtxRange nvtx_range("gpr_resident_live_rows");
  if (const int rc = enter(ctx)) return rc;
  if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window (gpr_resident_init)");
  if (!bits) return fail(ctx, GPR_E_INVALID, "bits is NULL");
  if (mem_kind != GPR_MEM_HOST && mem_kind != GPR_MEM_DEVICE) return fail(ctx, GPR_E_INVALID, "bad mem_kind %d", mem_kind);
  const uint32_t rows = ctx->res_P * ctx->res_G, words = (rows + 31) / 32;
  // a current index answers from 1/64 of the bytes (its block maxima are NaN exactly where a block has no sample); a
  // stale one is not read, and not refused either: this call only reads
  const bool index = gpr::live_rows_from_index(ctx->d_idx_util != nullptr, ctx->idx_stale);
  const float* p0 = index ? ctx->d_idx_util : ctx->d_res_util;
  const float* p1 = index ? ctx->d_idx_power : ctx->d_res_power;
  const uint32_t len = index ? ctx->idx_ld : ctx->res_T;
  uint32_t* out = bits;
  if (mem_kind == GPR_MEM_HOST) {
    CU(ctx->d_live.grow(ctx->stream, words));
    out = ctx->d_live;
  }
  const int rc = launch(ctx, gpr::k_live_rows, gpr::live_rows_grid(rows, ctx->sm_count), gpr::kRingThreads, 0, false,
                        reinterpret_cast<const uint32_t*>(p0), reinterpret_cast<const uint32_t*>(p1), rows, len, out);
  if (rc != GPR_OK) return rc;
  if (mem_kind == GPR_MEM_HOST)
    CU(cudaMemcpyAsync(bits, out, (size_t)words * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_resident_cols(gpr_ctx* ctx, int32_t plane, uint32_t newer, uint32_t n_cols, float* out, int32_t mem_kind) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  NvtxRange nvtx_range("gpr_resident_cols");
  if (const int rc = enter(ctx)) return rc;
  if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window (gpr_resident_init)");
  if (plane != 0 && plane != 1) return fail(ctx, GPR_E_INVALID, "bad plane %d", plane);
  if (plane == 1 && !ctx->d_res_power) return fail(ctx, GPR_E_STATE, "the resident window has no power plane");
  if (n_cols == 0) return fail(ctx, GPR_E_INVALID, "n_cols is 0");
  if ((uint64_t)newer + n_cols > ctx->res_T)
    return fail(ctx, GPR_E_INVALID, "newer + n_cols = %llu > n_samples = %u", (unsigned long long)newer + n_cols,
                ctx->res_T);
  if (!out) return fail(ctx, GPR_E_INVALID, "out is NULL");
  if (mem_kind != GPR_MEM_HOST && mem_kind != GPR_MEM_DEVICE) return fail(ctx, GPR_E_INVALID, "bad mem_kind %d", mem_kind);
  const size_t rows = (size_t)ctx->res_P * ctx->res_G, cells = rows * n_cols;
  uint32_t* dst = reinterpret_cast<uint32_t*>(out);
  if (mem_kind == GPR_MEM_HOST) {
    CU(ctx->d_band.grow(ctx->stream, cells));
    dst = ctx->d_band;
  }
  const float* src = plane == 0 ? ctx->d_res_util : ctx->d_res_power;
  const int rc = launch(ctx, gpr::k_ring_cols, gpr::ring_grid(rows, ctx->sm_count), gpr::kRingThreads, 0, false, dst,
                        reinterpret_cast<const uint32_t*>(src), (uint32_t)rows, ctx->res_T,
                        gpr::ring_cols_start(ctx->res_head, ctx->res_T, newer, n_cols), n_cols);
  if (rc != GPR_OK) return rc;
  if (mem_kind == GPR_MEM_HOST)
    CU(cudaMemcpyAsync(out, dst, cells * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_resident_retime(gpr_ctx* ctx, uint32_t n_keep, uint32_t factor) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  NvtxRange nvtx_range("gpr_resident_retime");
  if (const int rc = enter(ctx)) return rc;
  if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window (gpr_resident_init)");
  if (factor == 0) return fail(ctx, GPR_E_INVALID, "factor is 0");
  if (n_keep == 0 || n_keep > ctx->res_T)
    return fail(ctx, GPR_E_INVALID, "n_keep = %u: the resident window has %u samples", n_keep, ctx->res_T);
  // ---- the new ring beside the old one, gathered on the stream after whatever is enqueued there (the decisions still
  // pending read the old ring); they change places only once it is complete
  const uint32_t T_new = gpr::retime_len(n_keep, factor);
  const uint32_t rows = ctx->res_P * ctx->res_G;
  const bool index = ctx->d_idx_util != nullptr;
  const uint32_t ld_new = index ? gpr::index_ld(T_new) : 0;
  Buf<float>* cur[2] = {&ctx->d_res_util, &ctx->d_res_power};
  int rc = GPR_OK;
  for (int k = 0; k < 2 && rc == GPR_OK; ++k) {
    if (!*cur[k]) continue;
    Buf<float>& plane = ctx->d_res_next[k];
    Buf<float>& idx = ctx->d_res_next[2 + k];
    cudaError_t e = plane.alloc((size_t)rows * T_new);
    if (e == cudaSuccess && index) e = idx.alloc((size_t)rows * ld_new);
    if (e != cudaSuccess) {
      rc = fail(ctx, e == cudaErrorMemoryAllocation ? GPR_E_NOMEM : GPR_E_CUDA, "gpr_resident_retime: %s",
                cudaGetErrorString(e));
      break;
    }
    rc = launch(ctx, gpr::k_retime_rows, gpr::ring_grid(rows, ctx->sm_count), gpr::kRingThreads, 0, false,
                reinterpret_cast<uint32_t*>(plane.p), reinterpret_cast<const uint32_t*>(cur[k]->p), rows, ctx->res_T,
                ctx->res_head, n_keep, factor, index ? idx.p : nullptr, ld_new);
  }
  if (rc == GPR_OK) {
    const cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) rc = fail(ctx, GPR_E_CUDA, "gpr_resident_retime: %s", cudaGetErrorString(e));
  }
  if (rc != GPR_OK) {
    (void)cudaStreamSynchronize(ctx->stream);  // a gather may still be writing a new buffer
    for (Buf<float>& b : ctx->d_res_next) (void)b.release();
    return rc;
  }
  Buf<float>* all[4] = {&ctx->d_res_util, &ctx->d_res_power, &ctx->d_idx_util, &ctx->d_idx_power};
  for (int k = 0; k < 4; ++k) all[k]->swap(ctx->d_res_next[k]);
  ctx->res_T = T_new, ctx->res_head = 0;
  if (index) ctx->idx_ld = ld_new, ctx->idx_stale = false;  // rebuilt from the new planes
  for (Buf<float>& b : ctx->d_res_next) CU(b.release());    // the old ring
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_resident_planes(gpr_ctx* ctx, float** util, float** power, uint64_t* row_stride) {
  if (!ctx) return GPR_E_INVALID;
  if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window");
  if (util) *util = ctx->d_res_util;
  if (power) *power = ctx->d_res_power;
  if (row_stride) *row_stride = ctx->res_T;
  return GPR_OK;
}

int gpr_resident_head(gpr_ctx* ctx, uint32_t* head) {
  if (!ctx || !head) return GPR_E_INVALID;
  if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window");
  *head = ctx->res_head;
  return GPR_OK;
}

int gpr_resident_advance(gpr_ctx* ctx, uint32_t n_new) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  if (const int rc = enter(ctx)) return rc;
  if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window (gpr_resident_init)");
  if (n_new == 0) return GPR_OK;
  const uint32_t T = ctx->res_T;
  const size_t rows = (size_t)ctx->res_P * ctx->res_G;
  const gpr::RingSpan sp = gpr::ring_span(ctx->res_head, n_new, T);
  float* planes[2] = {ctx->d_res_util, ctx->d_res_power};
  float* planes_idx[2] = {ctx->d_idx_util, ctx->d_idx_power};
  for (int k = 0; k < 2; ++k) {
    float* pl = planes[k];
    const gpr::RingLaunch what = gpr::advance_launch(pl != nullptr, planes_idx[k] != nullptr);
    if (what == gpr::kRingNone) continue;
    int rc = GPR_OK;
    if (what == gpr::kRingOpen) {  // the opened buckets' old samples leave the index too
      rc = launch(ctx, gpr::k_open, gpr::ring_grid(rows, ctx->sm_count), gpr::kRingThreads, 0, false, pl, (uint32_t)rows,
                  T, sp.start, sp.n, planes_idx[k], ctx->idx_ld);
    } else if (n_new >= T) {
      CU(cudaMemsetAsync(pl, 0xFF, rows * (size_t)T * sizeof(float), ctx->stream));
    } else {
      rc = launch(ctx, gpr::text::k_fill_columns, capped_grid(ctx, (uint64_t)rows * n_new, 256, 16), 256, 0, false, pl,
                  (uint32_t)rows, T, T, ctx->res_head, n_new);
    }
    if (rc != GPR_OK) return rc;
  }
  ctx->res_head = sp.next_head;
  CU(cudaStreamSynchronize(ctx->stream));
  return GPR_OK;
  GPR_CATCH(ctx)
}

// ---- multi-GPU -------------------------------------------------------------------------------
int gpr_comm_unique_id(void* id128) {
  gpr_ctx* ctx = nullptr;
  GPR_TRY
  if (!id128) return fail(nullptr, GPR_E_INVALID, "id buffer is NULL");
  char err[256];
  if (!load_nccl(err, sizeof err)) return fail(nullptr, GPR_E_NCCL, "%s", err);
  static_assert(sizeof(ncclUniqueId) == GPR_UNIQUE_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId id;
  NC(g_nccl.GetUniqueId(&id));
  memcpy(id128, &id, sizeof id);
  return GPR_OK;
  GPR_CATCH(nullptr)
}

int gpr_comm_init(gpr_ctx* ctx, const void* id128, int rank, int world) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  if (const int rc = enter(ctx)) return rc;
  if (!id128 || world < 1 || rank < 0 || rank >= world)
    return fail(ctx, GPR_E_INVALID, "bad communicator arguments (rank %d world %d)", rank, world);
  if (ctx->comm) return fail(ctx, GPR_E_STATE, "communicator already attached");
  char err[256];
  if (!load_nccl(err, sizeof err)) return fail(ctx, GPR_E_NCCL, "%s", err);
  ncclUniqueId id;
  memcpy(&id, id128, sizeof id);
  NC(g_nccl.CommInitRank(&ctx->comm, world, id, rank));
  ctx->rank = rank, ctx->world = world;
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_comm_destroy(gpr_ctx* ctx) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  if (const int rc = enter(ctx)) return rc;
  if (ctx->comm) {
    CU(cudaStreamSynchronize(ctx->stream));
    NC(g_nccl.CommDestroy(ctx->comm));
    ctx->comm = nullptr;
  }
  ctx->rank = 0, ctx->world = 1;
  return GPR_OK;
  GPR_CATCH(ctx)
}

// Fused exchange over NVLink peer memory: every rank allocates one exchange block, publishes its
// CUDA IPC handle, and maps everybody else's.  From then on gpr_decide needs no collective launch.
int gpr_p2p_init(gpr_ctx* ctx, int rank, int world, uint32_t max_pods_per_rank, void* handle64) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  if (const int rc = enter(ctx)) return rc;
  if (!handle64 || world < 2 || world > gpr::kMaxPeers || rank < 0 || rank >= world)
    return fail(ctx, GPR_E_INVALID, "bad p2p arguments (rank %d world %d, at most %d ranks)", rank, world,
                gpr::kMaxPeers);
  if (ctx->p2p_block) return fail(ctx, GPR_E_STATE, "p2p exchange already initialised");
  if (ctx->comm && (ctx->rank != rank || ctx->world != world))
    return fail(ctx, GPR_E_INVALID, "rank/world differ from the NCCL communicator's");
  static_assert(sizeof(cudaIpcMemHandle_t) == GPR_P2P_HANDLE_BYTES, "cudaIpcMemHandle_t size");
  const uint32_t w_max = (max_pods_per_rank + 31u) / 32u;
  ctx->p2p_stride = 2u * std::max<uint32_t>(w_max, 1u);
  const size_t gather_bytes = ((size_t)world * ctx->p2p_stride * 4u + 255u) & ~(size_t)255u;
  const size_t ll_bytes = ((size_t)world * ctx->p2p_stride * 8u + 255u) & ~(size_t)255u;
  for (int k = 0; k < kExchangeDepth; ++k) {
    ctx->p2p_gather_off[k] = 256 + (size_t)k * gather_bytes;
    ctx->p2p_ll_off[k] = 256 + (size_t)kExchangeDepth * gather_bytes + (size_t)k * ll_bytes;
  }
  const size_t total = 256 + (size_t)kExchangeDepth * (gather_bytes + ll_bytes);
  CU(ctx->p2p_block.alloc(total));
  CU(cudaMemset(ctx->p2p_block, 0, total));
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, ctx->p2p_block));
  memcpy(handle64, &h, sizeof h);
  ctx->rank = rank, ctx->world = world;
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_p2p_attach(gpr_ctx* ctx, const void* handles) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  if (const int rc = enter(ctx)) return rc;
  if (!handles) return fail(ctx, GPR_E_INVALID, "handles is NULL");
  if (!ctx->p2p_block) return fail(ctx, GPR_E_STATE, "call gpr_p2p_init first");
  if (ctx->p2p_ready) return fail(ctx, GPR_E_STATE, "p2p exchange already attached");
  for (int r = 0; r < ctx->world; ++r) {
    if (r == ctx->rank) {
      ctx->p2p_peer[r] = ctx->p2p_block;
      continue;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, static_cast<const unsigned char*>(handles) + (size_t)r * GPR_P2P_HANDLE_BYTES, sizeof h);
    void* p = nullptr;
    CU(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    ctx->p2p_peer[r] = static_cast<unsigned char*>(p);
  }
  ctx->p2p_ready = true;
  return GPR_OK;
  GPR_CATCH(ctx)
}

// ---- memory helpers -----------------------------------------------------------------------------
int gpr_host_alloc(gpr_ctx* ctx, size_t bytes, void** out) {
  if (!ctx || !out) return GPR_E_INVALID;
  if (const int rc = enter(ctx)) return rc;
  CU(cudaMallocHost(out, bytes ? bytes : 1));
  return GPR_OK;
}
int gpr_host_free(gpr_ctx* ctx, void* p) {
  if (!ctx) return GPR_E_INVALID;
  if (p) CU(cudaFreeHost(p));
  return GPR_OK;
}
int gpr_device_alloc(gpr_ctx* ctx, size_t bytes, void** out) {
  if (!ctx || !out) return GPR_E_INVALID;
  if (const int rc = enter(ctx)) return rc;
  CU(cudaMalloc(out, bytes ? bytes : 1));
  return GPR_OK;
}
int gpr_device_free(gpr_ctx* ctx, void* p) {
  if (!ctx) return GPR_E_INVALID;
  if (const int rc = enter(ctx)) return rc;
  if (p) CU(cudaFree(p));
  return GPR_OK;
}
int gpr_memcpy(gpr_ctx* ctx, void* dst, const void* src, size_t bytes, int32_t dst_kind,
               int32_t src_kind) {
  if (!ctx) return GPR_E_INVALID;
  if (const int rc = enter(ctx)) return rc;
  if (bytes == 0) return GPR_OK;
  if (!dst || !src) return fail(ctx, GPR_E_INVALID, "NULL pointer in gpr_memcpy");
  cudaMemcpyKind k = dst_kind == GPR_MEM_DEVICE
                         ? (src_kind == GPR_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice)
                         : (src_kind == GPR_MEM_DEVICE ? cudaMemcpyDeviceToHost : cudaMemcpyHostToHost);
  CU(cudaMemcpyAsync(dst, src, bytes, k, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return GPR_OK;
}

// ---- measurement support --------------------------------------------------------------------------
int gpr_timer_begin(gpr_ctx* ctx) {
  if (!ctx) return GPR_E_INVALID;
  if (const int rc = enter(ctx)) return rc;
  // rendezvous first, then the start event: with an exchange attached the timed regions of all ranks
  // begin within an NVLink round trip of each other, whatever the skew between their host threads
  gpr::RendezvousParams q;
  memset(&q, 0, sizeof q);
  q.world = 1, q.rank = 0;
  q.stamp = ctx->h_mark;
  q.err = ctx->h_err;
  if (ctx->p2p_ready && ctx->world > 1) {
    q.world = ctx->world, q.rank = ctx->rank;
    q.seq = ++ctx->rdv_seq;
    for (int r = 0; r < ctx->world; ++r)
      q.peer_flag[r] = reinterpret_cast<unsigned long long*>(ctx->p2p_peer[r]) + gpr::kMaxPeers + ctx->rank;
    q.my_flags = reinterpret_cast<const unsigned long long*>(ctx->p2p_block.p) + gpr::kMaxPeers;
  } else if (ctx->comm && ctx->world > 1) {
    // NCCL only: a one-word allgather is the rendezvous
    CU(ctx->d_gather.grow(ctx->stream, (size_t)ctx->world + 2));
    CU(ctx->d_bits.grow(ctx->stream, 4));
    NC(g_nccl.AllGather(ctx->d_bits, ctx->d_gather, 1, ncclUint32, ctx->comm, ctx->stream));
  }
  if (const int rc = launch(ctx, gpr::k_rendezvous, 1, 32, 0, false, q)) return rc;
  CU(cudaEventRecord(ctx->ev_t0, ctx->stream));
  return GPR_OK;
}
int gpr_step_stamps(gpr_ctx* ctx, uint64_t* ns, uint32_t cap, uint32_t* n, uint64_t* begin_ns) {
  if (!ctx || !n) return GPR_E_INVALID;
  *n = (uint32_t)ctx->stamps.size();
  if (begin_ns) *begin_ns = *ctx->h_mark;
  if (ns)
    for (uint32_t i = 0; i < cap && i < *n; ++i) ns[i] = ctx->stamps[i];
  return GPR_OK;
}
int gpr_phase_stamps(gpr_ctx* ctx, uint64_t* ns, uint32_t cap, uint32_t* n) {
  if (!ctx || !n) return GPR_E_INVALID;
  *n = (uint32_t)ctx->phase_stamps.size();
  if (ns)
    for (uint32_t i = 0; i < cap && i < *n; ++i) ns[i] = ctx->phase_stamps[i];
  return GPR_OK;
}
int gpr_p2p_debug(gpr_ctx* ctx, int32_t mode) {
  if (!ctx) return GPR_E_INVALID;
  if (mode < 0 || mode > 2) return fail(ctx, GPR_E_INVALID, "exchange debug mode %d (0..2)", mode);
  ctx->exchange_debug = mode;
  return GPR_OK;
}
int gpr_timer_end(gpr_ctx* ctx, double* ms) {
  if (!ctx || !ms) return GPR_E_INVALID;
  if (const int rc = enter(ctx)) return rc;
  CU(cudaEventRecord(ctx->ev_t1, ctx->stream));
  CU(cudaEventSynchronize(ctx->ev_t1));
  float f = 0.f;
  CU(cudaEventElapsedTime(&f, ctx->ev_t0, ctx->ev_t1));
  *ms = f;
  return GPR_OK;
}
int gpr_flush_l2(gpr_ctx* ctx) {
  if (!ctx) return GPR_E_INVALID;
  if (const int rc = enter(ctx)) return rc;
  CU(ctx->d_flush.alloc_once(std::max<size_t>(ctx->l2_bytes * 2, (size_t)256 << 20)));
  CU(cudaMemsetAsync(ctx->d_flush, 0x5a, ctx->d_flush.cap, ctx->stream));
  return GPR_OK;
}
int gpr_launch_count(const gpr_ctx* ctx, uint64_t* n) {
  if (!ctx || !n) return GPR_E_INVALID;
  *n = ctx->launches;
  return GPR_OK;
}
int gpr_get_device_info(gpr_ctx* ctx, gpr_device_info* info) {
  if (!ctx || !info) return GPR_E_INVALID;
  if (info->struct_size != sizeof(gpr_device_info))
    return fail(ctx, GPR_E_INVALID, "gpr_device_info.struct_size mismatch");
  info->sm_count = ctx->sm_count;
  info->cc_major = ctx->cc_major, info->cc_minor = ctx->cc_minor;
  info->l2_bytes = ctx->l2_bytes, info->hbm_bytes = ctx->hbm_bytes;
  memcpy(info->name, ctx->name, sizeof info->name);
  return GPR_OK;
}

// ---- synthetic windows -----------------------------------------------------------------------------
// ---- device-side ingest of the response text -------------------------------------------------------
static_assert(sizeof(gpr_text_span) == sizeof(gpr::text::Span) && offsetof(gpr_text_span, row) == offsetof(gpr::text::Span, row) &&
                  offsetof(gpr_text_span, n_tiny) == offsetof(gpr::text::Span, n_tiny),
              "gpr_text_span mirrors gpr::text::Span");
static_assert(GPR_SPAN_SHARED == gpr::text::kSpanShared && GPR_SPAN_HARD == gpr::text::kSpanHard, "span flags");

int gpr_text_scan_begin(gpr_ctx* ctx, int32_t slot, const char* text, uint64_t n_bytes, int32_t mem_kind) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  NvtxRange nvtx_range("gpr_text_scan_begin");
  if (const int rc = enter(ctx)) return rc;
  if (slot < 0 || slot > 2) return fail(ctx, GPR_E_INVALID, "text slot %d (0..2)", slot);
  if (!text && n_bytes) return fail(ctx, GPR_E_INVALID, "text is NULL");
  if (mem_kind != GPR_MEM_HOST && mem_kind != GPR_MEM_DEVICE) return fail(ctx, GPR_E_INVALID, "bad mem_kind %d", mem_kind);
  scan_pipe_abort(ctx);  // an unfinished scan is dropped
  CU(ctx->d_text[slot].grow(ctx->stream, (size_t)n_bytes + gpr::text::kTextPad));
  constexpr int NT = gpr_ctx::kUpThreads, NS = gpr_ctx::kUpSlots, NB = gpr_ctx::kMarkBlocks;
  CU(ctx->h_mark_blocks.alloc_once((size_t)NB * kBlockWords, cudaHostAllocMapped));
  CU(ctx->d_mark_blocks.alloc_once((size_t)NB * kBlockWords));
  for (Event& ev : ctx->mark_event) CU(ev.create(cudaEventDisableTiming));
  for (int k = 0; k < NT; ++k) {
    CU(ctx->up_stream[k].create(cudaStreamNonBlocking));
    for (Event& ev : ctx->up_event[k]) CU(ev.create(cudaEventDisableTiming));
  }
  uint8_t* d = ctx->d_text[slot];
  ctx->text_n[slot] = n_bytes;
  // the zero pad behind the text, and everything earlier on the context's stream that may still read the buffer
  CU(cudaMemsetAsync(d + n_bytes, 0, gpr::text::kTextPad, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  ScanPipe* sp = new ScanPipe();
  sp->slot = slot, sp->src = text, sp->dst = d, sp->n = n_bytes, sp->src_kind = mem_kind;
  for (auto& r : sp->recorded) r.store(0);
  sp->staged = mem_kind == GPR_MEM_HOST && n_bytes && !host_pinned(text, nullptr);
  sp->chunk = sp->staged ? ctx->up_chunk : gpr_ctx::kPinnedChunk;
  sp->n_chunks = (n_bytes + sp->chunk - 1) / sp->chunk;
  sp->unit = std::min<uint64_t>(sp->chunk, gpr_ctx::kScanUnit);
  sp->units_per_chunk = (sp->chunk + sp->unit - 1) / sp->unit;
  sp->n_units = sp->n_chunks ? (sp->n_chunks - 1) * sp->units_per_chunk +
                                   (n_bytes - (sp->n_chunks - 1) * sp->chunk + sp->unit - 1) / sp->unit
                             : 0;
  static_assert(gpr_ctx::kPinnedChunk / gpr_ctx::kScanUnit <= (size_t)gpr_ctx::kMarkBlocks, "a chunk's units fit the ring");
  // pinned and device sources need no staging copy: one producer keeps the DMA engine busy
  sp->nt = sp->staged ? (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)ctx->up_threads, sp->n_chunks)) : 1;
  if (sp->staged) CU(ctx->h_up_ring.alloc_once((size_t)ctx->up_threads * NS * ctx->up_slot_bytes));
  ctx->pipe = sp;
  ctx->launches += 2 * sp->n_chunks;
  try {
    for (int k = 0; k < sp->nt; ++k) sp->th.emplace_back(scan_producer, ctx, sp, k);
  } catch (...) {
    if (sp->th.empty()) {  // no thread to be had at all: produce on this thread (blocks run ahead by at most NB chunks)
      (void)scan_pipe_finish(ctx, false);
      return fail(ctx, GPR_E_NOMEM, "could not start an upload thread");
    }
    sp->nt = (int)sp->th.size();  // fewer producers than planned would skip chunks: restart with what we have
    (void)scan_pipe_finish(ctx, false);
    return fail(ctx, GPR_E_NOMEM, "could not start the upload threads");
  }
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_text_scan_next(gpr_ctx* ctx, uint64_t* opens, uint64_t* closes, uint64_t cap, uint64_t* n_opens, uint64_t* n_closes,
                       uint64_t* bytes_done, int32_t* more) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  if (const int rc = enter(ctx)) return rc;
  if (!n_opens || !n_closes || !bytes_done || !more || (cap && (!opens || !closes)))
    return fail(ctx, GPR_E_INVALID, "output pointers are NULL");
  ScanPipe* sp = ctx->pipe;
  if (!sp) return fail(ctx, GPR_E_STATE, "no scan in progress (gpr_text_scan_begin)");
  *n_opens = *n_closes = 0;
  if (sp->next >= sp->n_units) {  // everything delivered (also: empty text)
    *bytes_done = sp->n, *more = 0;
    return scan_pipe_finish(ctx, true);
  }
  constexpr int NB = gpr_ctx::kMarkBlocks;
  const uint64_t u = sp->next;
  while (sp->recorded[u % NB].load(std::memory_order_acquire) != u + 1) {
    if (sp->error.load() || sp->stop.load()) return scan_pipe_finish(ctx, false) != GPR_OK ? GPR_E_CUDA : fail(ctx, GPR_E_CUDA, "text upload stopped");
    std::this_thread::yield();
  }
  cudaError_t e = cudaEventSynchronize(ctx->mark_event[u % NB]);
  if (e != cudaSuccess) {
    (void)scan_pipe_finish(ctx, false);
    return fail(ctx, GPR_E_CUDA, "text scan: %s", cudaGetErrorString(e));
  }
  const uint32_t* block = ctx->h_mark_blocks + (size_t)(u % NB) * kBlockWords;
  const uint64_t c = u / sp->units_per_chunk;
  const uint64_t base = c * sp->chunk + (u % sp->units_per_chunk) * sp->unit;
  const uint64_t end = std::min<uint64_t>({sp->n, (c + 1) * sp->chunk, base + sp->unit});
  const uint64_t no = block[0], nc = block[1];
  if (no > gpr_ctx::kMarkCap || nc > gpr_ctx::kMarkCap || no > cap || nc > cap) {
    const bool caller = no <= gpr_ctx::kMarkCap && nc <= gpr_ctx::kMarkCap;
    *n_opens = no, *n_closes = nc;
    if (!caller) (void)scan_pipe_finish(ctx, false);  // (a too small `cap` may be retried with a larger one)
    return fail(ctx, GPR_E_CAPACITY, "%llu / %llu markers in the %llu bytes of text at offset %llu, room for %llu",
                (unsigned long long)no, (unsigned long long)nc, (unsigned long long)(end - base), (unsigned long long)base,
                (unsigned long long)(caller ? cap : gpr_ctx::kMarkCap));
  }
  for (uint64_t i = 0; i < no; ++i) opens[i] = base + block[2 + i];
  for (uint64_t i = 0; i < nc; ++i) closes[i] = base + block[2 + gpr_ctx::kMarkCap + i];
  std::sort(opens, opens + no);
  std::sort(closes, closes + nc);
  *n_opens = no, *n_closes = nc;
  sp->next = u + 1;
  sp->consumed.store(u + 1, std::memory_order_release);
  *bytes_done = end;
  *more = 1;
  if (sp->next >= sp->n_units) {
    *more = 0;
    return scan_pipe_finish(ctx, true);
  }
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_text_scan(gpr_ctx* ctx, int32_t slot, const char* text, uint64_t n_bytes, int32_t mem_kind,
                  uint64_t* opens, uint64_t* closes, uint64_t cap, uint64_t* n_opens, uint64_t* n_closes) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  NvtxRange nvtx_range("gpr_text_scan");
  if (const int rc = enter(ctx)) return rc;
  if (!n_opens || !n_closes || (cap && (!opens || !closes))) return fail(ctx, GPR_E_INVALID, "output arrays are NULL");
  int rc = gpr_text_scan_begin(ctx, slot, text, n_bytes, mem_kind);
  if (rc != GPR_OK) return rc;
  std::vector<uint64_t> co(gpr_ctx::kMarkCap), cc(gpr_ctx::kMarkCap);
  uint64_t no = 0, nc = 0;
  int32_t more = 1;
  while (more) {
    uint64_t a = 0, b = 0, done = 0;
    rc = gpr_text_scan_next(ctx, co.data(), cc.data(), gpr_ctx::kMarkCap, &a, &b, &done, &more);
    if (rc != GPR_OK) {
      scan_pipe_abort(ctx);
      return rc;
    }
    for (uint64_t i = 0; i < a; ++i, ++no)
      if (no < cap) opens[no] = co[i];
    for (uint64_t i = 0; i < b; ++i, ++nc)
      if (nc < cap) closes[nc] = cc[i];
  }
  CU(cudaStreamSynchronize(ctx->stream));
  *n_opens = no, *n_closes = nc;
  if (no > cap || nc > cap)
    return fail(ctx, GPR_E_CAPACITY, "%llu / %llu markers, room for %llu: call again with a larger cap", (unsigned long long)no,
                (unsigned long long)nc, (unsigned long long)cap);
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_text_parse(gpr_ctx* ctx, int32_t slot, gpr_text_span* spans, uint32_t n_spans, const gpr_text_grid* grid,
                   int32_t plane) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  NvtxRange nvtx_range("gpr_text_parse");
  if (const int rc = enter(ctx)) return rc;
  if (!grid || grid->struct_size != sizeof(gpr_text_grid)) return fail(ctx, GPR_E_INVALID, "grid is NULL / struct_size mismatch");
  if (slot < 0 || slot > 2 || plane < 0 || plane > 1) return fail(ctx, GPR_E_INVALID, "bad slot %d / plane %d", slot, plane);
  if (!ctx->d_text[slot]) return fail(ctx, GPR_E_STATE, "no text in slot %d (gpr_text_scan)", slot);
  if (n_spans && !spans) return fail(ctx, GPR_E_INVALID, "spans is NULL");
  const uint32_t n_rows = grid->n_rows;
  int rc;
  if ((rc = check_grid(ctx, grid)) != GPR_OK) return rc;
  const uint64_t n = ctx->text_n[slot];
  for (uint32_t i = 0; i < n_spans; ++i) {
    if (spans[i].begin > spans[i].end || spans[i].end > n || spans[i].row >= n_rows ||
        (i && spans[i].begin < spans[i - 1].end))
      return fail(ctx, GPR_E_INVALID, "span %u is out of order, out of the text or out of the plane", i);
    spans[i].flags &= GPR_SPAN_SHARED;
    spans[i].n_in = spans[i].n_oow = spans[i].n_tiny = 0;
  }
  float* pl = nullptr;
  gpr::text::Grid g;
  if ((rc = open_destination(ctx, grid, plane, &g, &pl)) != GPR_OK) return rc;
  CU(ctx->d_spans.grow(ctx->stream, (size_t)n_spans + 1));
  if (n_spans && n) {
    CU(cudaMemcpyAsync(ctx->d_spans, spans, (size_t)n_spans * sizeof(gpr_text_span), cudaMemcpyHostToDevice,
                       ctx->stream));
    constexpr int kWarps = 4;
    const uint64_t tiles = (n + gpr::text::kTileBytes - 1) / gpr::text::kTileBytes;
    if ((rc = launch(ctx, gpr::text::k_text_parse<kWarps>, capped_grid(ctx, tiles, kWarps, ctx->parse_ctas_per_sm),
                     kWarps * 32, gpr::text::text_parse_smem<kWarps>(), false, ctx->d_text[slot], n,
                     n + gpr::text::kTextPad, ctx->d_spans, n_spans, g, pl)) != GPR_OK)
      return rc;
    CU(cudaMemcpyAsync(spans, ctx->d_spans, (size_t)n_spans * sizeof(gpr_text_span), cudaMemcpyDeviceToHost,
                       ctx->stream));
  }
  CU(cudaStreamSynchronize(ctx->stream));
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_text_planes(gpr_ctx* ctx, float** util, float** power) {
  if (!ctx) return GPR_E_INVALID;
  if (util) *util = ctx->d_tplane[0];
  if (power) *power = ctx->d_tplane[1];
  return GPR_OK;
}

// ---- decoded samples (gpr_samples.cuh) and Prometheus XOR chunks (gpr_chunks.cuh) --------------------------------
// Both merges check a batch the same way before anything is written, then merge into gpr_text_parse's destination.
static_assert(sizeof(gpr_sample_stats) == 24, "gpr_sample_stats");

// The arguments of a batch (gpr_sample_batch or gpr_chunk_batch) and of its grid
extern "C++" {  // (templates)
template <typename Batch>
static int check_batch_args(gpr_ctx* ctx, const Batch* batch, const gpr_text_grid* grid, int32_t plane) {
  if (!batch || batch->struct_size != sizeof(Batch)) return fail(ctx, GPR_E_INVALID, "batch is NULL / struct_size mismatch");
  if (!grid || grid->struct_size != sizeof(gpr_text_grid)) return fail(ctx, GPR_E_INVALID, "grid is NULL / struct_size mismatch");
  if (plane < 0 || plane > 1) return fail(ctx, GPR_E_INVALID, "bad plane %d", plane);
  if (batch->mem_kind != GPR_MEM_HOST && batch->mem_kind != GPR_MEM_DEVICE)
    return fail(ctx, GPR_E_INVALID, "bad mem_kind %d", batch->mem_kind);
  return check_grid(ctx, grid);
}
}  // extern "C++"

// A batch's series index, offsets[n_series + 1] (into its samples, or its chunks) and rows[n_series], checked where it
// is: on the host, or on the device by k_samples_check.  *bad gets the series_faults() bits of every series and *total
// offsets[n_series].  (The first use of a batch's scratch d_sstats, which is allocated here.)
static int check_series_index(gpr_ctx* ctx, const uint64_t* offsets, const uint32_t* rows, uint32_t S, bool host,
                              uint32_t n_rows, uint32_t* bad, uint64_t* total) {
  namespace gs = gpr::samples;
  CU(ctx->d_sstats.alloc_once(5));
  if (host) {
    *bad = 0;
    for (uint32_t s = 0; s < std::max(S, 1u); ++s) *bad |= gs::series_faults(offsets, rows, S, s, n_rows);
    *total = offsets[S];
    return GPR_OK;
  }
  unsigned long long back[2] = {0, 0};  // the check word, offsets[n_series]
  unsigned int* d_bad = reinterpret_cast<unsigned int*>(ctx->d_sstats + 2);
  CU(cudaMemsetAsync(d_bad, 0, sizeof(unsigned long long), ctx->stream));
  const int rc = launch(ctx, gs::k_samples_check, capped_grid(ctx, std::max(S, 1u), 256, 8), 256, 0, false, offsets, rows,
                        S, n_rows, d_bad);
  if (rc != GPR_OK) return rc;
  CU(cudaMemcpyAsync(&back[0], d_bad, sizeof back[0], cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(&back[1], offsets + S, sizeof back[1], cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  *bad = (uint32_t)back[0], *total = back[1];
  return GPR_OK;
}

// a host batch's series index, uploaded whole (12 B per series)
static int upload_series_index(gpr_ctx* ctx, const uint64_t* offsets, const uint32_t* rows, uint32_t S) {
  CU(ctx->d_soffsets.grow(ctx->stream, (size_t)S + 1));
  CU(ctx->d_srows.grow(ctx->stream, (size_t)S + 1));
  CU(cudaMemcpyAsync(ctx->d_soffsets, offsets, ((size_t)S + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(ctx->d_srows, rows, (size_t)S * 4, cudaMemcpyHostToDevice, ctx->stream));
  return GPR_OK;
}

// rc, after the stream has drained if it is an error: the staging buffers of a failed step may still be read
static int drain_on_error(gpr_ctx* ctx, int rc) {
  if (rc != GPR_OK) (void)cudaStreamSynchronize(ctx->stream);
  return rc;
}

// The end of a merge whose work is enqueued with status rc: n_in and the merge's counts go to *stats.
static int finish_merge(gpr_ctx* ctx, int rc, uint64_t n_in, gpr_sample_stats* stats) {
  if (drain_on_error(ctx, rc) != GPR_OK) return rc;
  unsigned long long counts[2] = {0, 0};
  CU(cudaMemcpyAsync(counts, ctx->d_sstats, sizeof counts, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (stats) stats->n_in = n_in, stats->n_oow = counts[0], stats->n_tiny = counts[1];
  return GPR_OK;
}

static int launch_scatter(gpr_ctx* ctx, const gpr::samples::ScatterArgs& a, bool vec) {
  namespace gs = gpr::samples;
  return launch(ctx, vec ? gs::k_samples_scatter<true> : gs::k_samples_scatter<false>,
                capped_grid(ctx, a.end - a.base, gs::kChunk, 8), gs::kThreads, 0, false, a);
}

// The staging of a host batch (gpr_samples_scatter, gpr_chunks_scatter): two device buffers of 2 x kStageHalf bytes
// and, for pageable batches, two pinned ones.  Piece k goes into buffer k % 2.
constexpr size_t kStageHalf = gpr::samples::kHostPiece * 8;  // bytes of one piece's timestamps, or of its values
static_assert(gpr::chunks::kHostPiece == 2 * kStageHalf, "a piece of chunk data fills one staging buffer");

static int open_staging(gpr_ctx* ctx, bool pinned) {
  CU(ctx->d_sstage.alloc_once(4 * kStageHalf));
  if (!pinned) CU(ctx->h_sstage.alloc_once(4 * kStageHalf));
  for (int b = 0; b < 2; ++b) {
    CU(ctx->ev_sup[b].create(cudaEventDisableTiming));
    CU(ctx->ev_sdone[b].create(cudaEventDisableTiming));
  }
  return GPR_OK;
}

// Piece k of a host batch: the host ranges src[i] (bytes[i] each, at most kStageHalf when there are two, or
// 2 x kStageHalf for one) are copied, through pinned staging unless `pinned`, into device buffer k % 2 on the copy
// stream; the context's stream waits for them and consume(device buffer) enqueues the work on the piece, after which
// the buffer is marked free.  So piece k + 1 crosses PCIe while piece k is consumed.
extern "C++" {  // (templates)
template <typename Consume>
static int stage_piece(gpr_ctx* ctx, uint64_t k, bool pinned, const void* const (&src)[2], const size_t (&bytes)[2],
                       Consume&& consume) {
  const int b = (int)(k & 1);
  unsigned char* dst = ctx->d_sstage + (size_t)b * 2 * kStageHalf;
  if (k >= 2) CU(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_sdone[b], 0));  // piece k - 2 has left buffer b
  if (!pinned && k >= 2) CU(cudaEventSynchronize(ctx->ev_sup[b]));  // piece k - 2's upload has drained pinned buffer b
  size_t at = 0;
  for (int i = 0; i < 2; ++i) {
    if (!bytes[i]) continue;
    const void* from = src[i];
    if (!pinned) {
      unsigned char* stage = ctx->h_sstage + (size_t)b * 2 * kStageHalf + at;
      memcpy(stage, src[i], bytes[i]);
      from = stage;
    }
    CU(cudaMemcpyAsync(dst + at, from, bytes[i], cudaMemcpyHostToDevice, ctx->copy_stream));
    at += kStageHalf;
  }
  CU(cudaEventRecord(ctx->ev_sup[b], ctx->copy_stream));
  CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_sup[b], 0));
  const int r = consume(dst);
  if (r != GPR_OK) return r;
  CU(cudaEventRecord(ctx->ev_sdone[b], ctx->stream));
  return GPR_OK;
}
}  // extern "C++"

// A host batch, piece by piece: piece k is copied into device buffer k % 2 on the copy stream and scattered on the
// context's stream, so piece k + 1 crosses PCIe while piece k merges.
static int scatter_host_pieces(gpr_ctx* ctx, const gpr_sample_batch* batch, uint64_t total, gpr::samples::ScatterArgs a) {
  namespace gs = gpr::samples;
  const uint32_t S = batch->n_series;
  int rc;
  if ((rc = upload_series_index(ctx, batch->offsets, batch->rows, S)) != GPR_OK) return rc;
  a.offsets = ctx->d_soffsets, a.rows = ctx->d_srows;
  const bool pinned = host_pinned(batch->ts_ms, batch->values);
  if ((rc = open_staging(ctx, pinned)) != GPR_OK) return rc;
  uint64_t k = 0;
  return gs::for_each_piece(batch->offsets, S, total, gs::kHostPiece, [&](const gs::Piece& p) -> int {
    const uint64_t n = p.end - p.begin;
    const void* const src[2] = {batch->ts_ms + p.begin, batch->values + p.begin};
    const size_t bytes[2] = {n * 8, n * 8};
    return stage_piece(ctx, k++, pinned, src, bytes, [&](unsigned char* dst) {
      a.ts = reinterpret_cast<const int64_t*>(dst);
      a.values = reinterpret_cast<const double*>(dst + kStageHalf);
      a.base = p.begin, a.end = p.end, a.s_base = p.series;
      return launch_scatter(ctx, a, true);
    });
  });
}

int gpr_samples_scatter(gpr_ctx* ctx, const gpr_sample_batch* batch, const gpr_text_grid* grid, int32_t plane,
                        gpr_sample_stats* stats) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  NvtxRange nvtx_range("gpr_samples_scatter");
  namespace gs = gpr::samples;
  int rc;
  if ((rc = enter(ctx)) != GPR_OK || (rc = check_batch_args(ctx, batch, grid, plane)) != GPR_OK) return rc;
  const uint32_t S = batch->n_series;
  const bool host = batch->mem_kind == GPR_MEM_HOST;
  if (!batch->offsets || (S && !batch->rows)) return fail(ctx, GPR_E_INVALID, "offsets / rows is NULL");
  // ---- the batch is checked before anything is written
  uint32_t bad = 0;
  uint64_t total = 0;
  if ((rc = check_series_index(ctx, batch->offsets, batch->rows, S, host, grid->n_rows, &bad, &total)) != GPR_OK)
    return rc;
  if (bad & gs::kBadStart) return fail(ctx, GPR_E_INVALID, "gpr_sample_batch: offsets[0] != 0");
  if (bad & gs::kBadOrder) return fail(ctx, GPR_E_INVALID, "gpr_sample_batch: offsets decrease");
  if (bad & gs::kBadRow) return fail(ctx, GPR_E_INVALID, "gpr_sample_batch: a row >= grid.n_rows (%u)", grid->n_rows);
  if (total && (!batch->ts_ms || !batch->values)) return fail(ctx, GPR_E_INVALID, "ts_ms / values is NULL");
  // ---- the destination, then the merge
  gs::ScatterArgs a;
  memset(&a, 0, sizeof a);
  if ((rc = open_destination(ctx, grid, plane, &a.g, &a.plane)) != GPR_OK) return rc;
  CU(cudaMemsetAsync(ctx->d_sstats, 0, 2 * sizeof(unsigned long long), ctx->stream));
  a.n_series = S, a.stats = ctx->d_sstats;
  if (total && !host) {  // read in place
    a.offsets = batch->offsets, a.rows = batch->rows, a.ts = batch->ts_ms, a.values = batch->values;
    a.base = 0, a.end = total, a.s_base = 0;
    rc = launch_scatter(ctx, a, aligned16(batch->ts_ms) && aligned16(batch->values));
  } else if (total) {
    rc = scatter_host_pieces(ctx, batch, total, a);
  }
  return finish_merge(ctx, rc, total, stats);
  GPR_CATCH(ctx)
}

// ---- Prometheus XOR chunks (gpr_chunks.cuh) -----------------------------------------------------------------
constexpr uint32_t kChunkTooLarge = 1u << 31;  // a host batch's chunk that does not fit one upload piece
// The fault bits of a chunk batch as GPR_E_INVALID; `first` is the first chunk at fault (the bits are those of all
// faulty chunks: the message gives the first kind found).
static int chunk_batch_fault(gpr_ctx* ctx, uint32_t bad, uint64_t first, uint32_t n_rows) {
  namespace gc = gpr::chunks;
  const unsigned long long c = first;
  if (bad & gc::kBadStart) return fail(ctx, GPR_E_INVALID, "gpr_chunk_batch: series_chunks[0] != 0");
  if (bad & gc::kBadOrder) return fail(ctx, GPR_E_INVALID, "gpr_chunk_batch: series_chunks decrease");
  if (bad & gc::kBadRow) return fail(ctx, GPR_E_INVALID, "gpr_chunk_batch: a row >= grid.n_rows (%u)", n_rows);
  if (bad & gc::kBadChunkStart) return fail(ctx, GPR_E_INVALID, "gpr_chunk_batch: chunk_bytes[0] != 0");
  const char* what = (bad & gc::kBadChunkOrder) ? "chunk_bytes decrease"
                     : (bad & gc::kShort)       ? "shorter than its 2-byte header"
                     : (bad & gc::kOverrun)     ? "its samples run past its bytes"
                     : (bad & gc::kNoWindow)    ? "a value reuses the XOR window before one was set"
                     : (bad & gc::kBadVarint)   ? "a varint overflows 64 bits"
                                                : "a host chunk larger than an upload piece (32 MB)";
  return fail(ctx, GPR_E_INVALID, "gpr_chunk_batch: chunk %llu is the first malformed one (%s)", c, what);
}

static int launch_chunks_check(gpr_ctx* ctx, const gpr::chunks::CheckArgs& a) {
  return launch(ctx, gpr::chunks::k_chunks_check, capped_grid(ctx, a.end - a.base, 256, 8), 256, 0, false, a);
}

static int launch_chunks_scatter(gpr_ctx* ctx, const gpr::chunks::ScatterArgs& a) {
  namespace gc = gpr::chunks;
  if (a.end <= a.base) return GPR_OK;
  const uint64_t groups = (a.end - a.base + 31) / 32;
  return launch(ctx, gc::k_chunks_scatter, capped_grid(ctx, groups, gc::kWarps, 8), gc::kThreads, 0, false, a);
}

// A host batch's chunk data, piece by piece: each piece is the most whole chunks that fit kHostPiece bytes, and at
// least one (none is larger: the host check saw to it); consume(piece, device bytes of the piece) enqueues the work
// on each.
extern "C++" {  // (templates)
template <typename Consume>
static int chunk_pieces(gpr_ctx* ctx, const gpr_chunk_batch* batch, uint64_t n_chunks, bool pinned, Consume&& consume) {
  namespace gc = gpr::chunks;
  namespace gs = gpr::samples;
  const uint64_t* cb = batch->chunk_bytes;
  const auto cut = [&](uint64_t b) {
    const uint64_t* e = std::upper_bound(cb + b + 1, cb + n_chunks + 1, cb[b] + gc::kHostPiece);
    return std::max<uint64_t>(b + 1, (uint64_t)(e - cb) - 1);
  };
  uint64_t k = 0;
  return gs::for_each_cut(batch->series_chunks, batch->n_series, n_chunks, cut, [&](const gs::Piece& p) -> int {
    const void* const src[2] = {batch->data + cb[p.begin], nullptr};
    const size_t bytes[2] = {(size_t)(cb[p.end] - cb[p.begin]), 0};
    return stage_piece(ctx, k++, pinned, src, bytes, [&](unsigned char* dst) { return consume(p, dst); });
  });
}
}  // extern "C++"

int gpr_chunks_scatter(gpr_ctx* ctx, const gpr_chunk_batch* batch, const gpr_text_grid* grid, int32_t plane,
                       gpr_sample_stats* stats) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  NvtxRange nvtx_range("gpr_chunks_scatter");
  namespace gc = gpr::chunks;
  namespace gs = gpr::samples;
  int rc;
  if ((rc = enter(ctx)) != GPR_OK || (rc = check_batch_args(ctx, batch, grid, plane)) != GPR_OK) return rc;
  const uint32_t S = batch->n_series;
  const bool host = batch->mem_kind == GPR_MEM_HOST;
  if (!batch->series_chunks || !batch->chunk_bytes || (S && !batch->rows))
    return fail(ctx, GPR_E_INVALID, "series_chunks / chunk_bytes / rows is NULL");
  // ---- the batch is checked before anything is written: the index arrays, then the chunks' data
  uint32_t bad = 0;
  uint64_t n_chunks = 0, first = ~0ull;
  if ((rc = check_series_index(ctx, batch->series_chunks, batch->rows, S, host, grid->n_rows, &bad, &n_chunks)) != GPR_OK)
    return rc;
  if (bad) return chunk_batch_fault(ctx, bad, 0, grid->n_rows);
  if (host) {
    constexpr uint32_t kBadIndex = gc::kBadChunkStart | gc::kBadChunkOrder;
    if (batch->chunk_bytes[0] != 0) bad |= gc::kBadChunkStart;
    for (uint64_t c = 0; c < n_chunks && !(bad & kBadIndex); ++c) {
      uint32_t f = gc::bound_faults(batch->chunk_bytes, c);
      if (!f && batch->chunk_bytes[c + 1] - batch->chunk_bytes[c] > gc::kHostPiece) f = kChunkTooLarge;
      if (f && !bad) first = c;
      bad |= f;
    }
    if (bad) {
      // Such a batch never goes up.  While chunk_bytes rises from 0 every chunk lies inside the data, so the chunks
      // with good bounds are decoded here, as k_chunks_check decodes a device batch's: the first bad chunk and the
      // faults are then those a device batch reports.
      for (uint64_t c = 0; !(bad & kBadIndex) && batch->data && c < n_chunks; ++c) {
        if (gc::bound_faults(batch->chunk_bytes, c)) continue;
        const uint32_t f = gc::chunk_faults(batch->chunk_bytes, batch->data, 0, c);
        bad |= f;
        if (f && c < first) first = c;
      }
      return chunk_batch_fault(ctx, bad, first, grid->n_rows);
    }
  }
  if (n_chunks && !batch->data) return fail(ctx, GPR_E_INVALID, "data is NULL");
  // the chunks' data, by the check kernel: in place for a device batch, piece by piece as it lands for a host one
  CU(cudaMemsetAsync(ctx->d_sstats + 2, 0, 2 * sizeof(unsigned long long), ctx->stream));
  CU(cudaMemsetAsync(ctx->d_sstats + 4, 0xFF, sizeof(unsigned long long), ctx->stream));
  gc::CheckArgs ck;
  ck.bad = reinterpret_cast<unsigned int*>(ctx->d_sstats + 2), ck.n_in = ctx->d_sstats + 3, ck.first = ctx->d_sstats + 4;
  const bool pinned = host && host_pinned(batch->data, nullptr);
  std::vector<gs::Piece> checked;  // a host batch's pieces, in the order they went up
  if (host) {
    if ((rc = upload_series_index(ctx, batch->series_chunks, batch->rows, S)) != GPR_OK) return rc;
    CU(ctx->d_cbytes.grow(ctx->stream, (size_t)n_chunks + 1));
    CU(cudaMemcpyAsync(ctx->d_cbytes, batch->chunk_bytes, ((size_t)n_chunks + 1) * 8, cudaMemcpyHostToDevice,
                       ctx->stream));
    if ((rc = open_staging(ctx, pinned)) != GPR_OK) return rc;
    rc = chunk_pieces(ctx, batch, n_chunks, pinned, [&](const gs::Piece& p, const unsigned char* d) {
      checked.push_back(p);
      ck.chunk_bytes = ctx->d_cbytes, ck.data = d, ck.data_base = batch->chunk_bytes[p.begin];
      ck.base = p.begin, ck.end = p.end;
      return launch_chunks_check(ctx, ck);
    });
  } else {
    ck.chunk_bytes = batch->chunk_bytes, ck.data = batch->data, ck.data_base = 0, ck.base = 0, ck.end = n_chunks;
    rc = launch_chunks_check(ctx, ck);
  }
  if ((rc = drain_on_error(ctx, rc)) != GPR_OK) return rc;
  unsigned long long back[3] = {0, 0, 0};  // the check word, n_in, the first bad chunk
  CU(cudaMemcpyAsync(back, ctx->d_sstats + 2, sizeof back, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (back[0]) return chunk_batch_fault(ctx, (uint32_t)back[0], back[2], grid->n_rows);
  // ---- the destination, then the merge
  gc::ScatterArgs a;
  memset(&a, 0, sizeof a);
  if ((rc = open_destination(ctx, grid, plane, &a.g, &a.plane)) != GPR_OK) return rc;
  CU(cudaMemsetAsync(ctx->d_sstats, 0, 2 * sizeof(unsigned long long), ctx->stream));
  a.n_series = S, a.stats = ctx->d_sstats;
  if (!host) {  // read in place
    a.series_chunks = batch->series_chunks, a.rows = batch->rows, a.chunk_bytes = batch->chunk_bytes;
    a.data = batch->data, a.data_base = 0, a.base = 0, a.end = n_chunks, a.s_base = 0;
    rc = launch_chunks_scatter(ctx, a);
  } else {
    a.series_chunks = ctx->d_soffsets, a.rows = ctx->d_srows, a.chunk_bytes = ctx->d_cbytes;
    const auto scatter = [&](const gs::Piece& p, const unsigned char* d) {
      a.data = d, a.data_base = batch->chunk_bytes[p.begin], a.base = p.begin, a.end = p.end, a.s_base = p.series;
      return launch_chunks_scatter(ctx, a);
    };
    if (checked.size() <= 2) {  // the checked pieces are still in the two staging buffers
      for (size_t k = 0; k < checked.size() && rc == GPR_OK; ++k)
        rc = scatter(checked[k], ctx->d_sstage + k * 2 * kStageHalf);
    } else {
      rc = chunk_pieces(ctx, batch, n_chunks, pinned, scatter);
    }
  }
  return finish_merge(ctx, rc, back[1], stats);
  GPR_CATCH(ctx)
}

// ---- the resident ring as XOR chunks (gpr_chunks_encode.cuh) --------------------------------------------------
static_assert(sizeof(gpr_chunk_export) == 96, "gpr_chunk_export");

int gpr_resident_export(gpr_ctx* ctx, const gpr_text_grid* grid, int32_t plane, uint32_t max_per_chunk,
                        gpr_chunk_export* out) {
  if (!ctx) return GPR_E_INVALID;
  GPR_TRY
  NvtxRange nvtx_range("gpr_resident_export");
  namespace gc = gpr::chunks;
  if (const int rc = enter(ctx)) return rc;
  if (!out || out->struct_size != sizeof(gpr_chunk_export))
    return fail(ctx, GPR_E_INVALID, "out is NULL / struct_size mismatch");
  out->n_series = out->n_chunks = out->n_bytes = out->n_samples = 0;
  if (!grid || grid->struct_size != sizeof(gpr_text_grid)) return fail(ctx, GPR_E_INVALID, "grid is NULL / struct_size mismatch");
  if (plane < 0 || plane > 1) return fail(ctx, GPR_E_INVALID, "bad plane %d", plane);
  if (out->mem_kind != GPR_MEM_HOST && out->mem_kind != GPR_MEM_DEVICE)
    return fail(ctx, GPR_E_INVALID, "bad mem_kind %d", out->mem_kind);
  if (max_per_chunk < 1 || max_per_chunk > 65535)
    return fail(ctx, GPR_E_INVALID, "max_per_chunk %u is outside 1..65535 (a chunk counts its samples in a u16)",
                max_per_chunk);
  if (!out->series_chunks || (out->cap_series && !out->rows) || !out->chunk_bytes || (out->cap_bytes && !out->data))
    return fail(ctx, GPR_E_INVALID, "series_chunks / rows / chunk_bytes / data is NULL");
  if (!ctx->d_res_util) return fail(ctx, GPR_E_STATE, "no resident window (gpr_resident_init)");
  if (plane == 1 && !ctx->d_res_power) return fail(ctx, GPR_E_STATE, "the resident window has no power plane");
  int rc;
  if ((rc = check_grid(ctx, grid)) != GPR_OK) return rc;
  if (grid->n_samples != ctx->res_T)
    return fail(ctx, GPR_E_INVALID, "grid.n_samples %u is not the resident window's %u", grid->n_samples, ctx->res_T);
  const uint32_t rows = ctx->res_P * ctx->res_G, T = ctx->res_T;
  gc::ExportArgs a;
  memset(&a, 0, sizeof a);
  a.plane = reinterpret_cast<const uint32_t*>(plane == 0 ? ctx->d_res_util.p : ctx->d_res_power.p);
  a.rows = rows, a.T = T, a.head = ctx->res_head, a.per_chunk = max_per_chunk;
  a.t_end_ms = grid->t_end * 1000, a.step_ms = grid->step * 1000;
  a.max_chunks = (T + max_per_chunk - 1) / max_per_chunk;
  // ---- sizes, and their scan
  CU(ctx->d_xsizes.grow(ctx->stream, (size_t)rows * a.max_chunks));
  CU(ctx->d_xrows.grow(ctx->stream, 2 * ((size_t)rows + 1)));
  CU(ctx->d_xseries.grow(ctx->stream, (size_t)rows + 1));
  CU(ctx->d_xtotals.alloc_once(4));
  a.sizes = ctx->d_xsizes, a.row_chunks = ctx->d_xrows, a.row_bytes = ctx->d_xrows + rows + 1;
  a.row_series = ctx->d_xseries, a.totals = ctx->d_xtotals;
  CU(cudaMemsetAsync(a.totals, 0, 4 * sizeof(unsigned long long), ctx->stream));
  const uint32_t blocks = capped_grid(ctx, rows, gc::kEncWarps, 16);
  if ((rc = launch(ctx, gc::k_export_size, blocks, gc::kEncThreads, 0, false, a)) != GPR_OK ||
      (rc = launch(ctx, gc::k_export_scan, 1, gc::kScanThreads, gc::kScanSmem, false, a)) != GPR_OK)
    return rc;
  unsigned long long tot[4];
  CU(cudaMemcpyAsync(tot, a.totals, sizeof tot, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  out->n_chunks = tot[0], out->n_bytes = tot[1], out->n_series = tot[2], out->n_samples = tot[3];
  if (out->n_series > out->cap_series || out->n_chunks > out->cap_chunks || out->n_bytes > out->cap_bytes)
    return fail(ctx, GPR_E_CAPACITY, "%llu series, %llu chunks, %llu bytes; room for %llu, %llu, %llu: call again with "
                "larger capacities", tot[2], tot[0], tot[1], (unsigned long long)out->cap_series,
                (unsigned long long)out->cap_chunks, (unsigned long long)out->cap_bytes);
  // ---- the outputs: in place on the device, or in context scratch copied out once per array
  const size_t b_sc = (tot[2] + 1) * 8, b_cb = (tot[0] + 1) * 8, b_rows = tot[2] * 4, b_data = tot[1];
  const bool host = out->mem_kind == GPR_MEM_HOST;
  if (host) {
    CU(ctx->d_xout.grow(ctx->stream, b_sc + b_cb + b_rows + b_data));
    unsigned char* o = ctx->d_xout;
    a.series_chunks = reinterpret_cast<uint64_t*>(o), a.chunk_bytes = reinterpret_cast<uint64_t*>(o + b_sc);
    a.out_rows = reinterpret_cast<uint32_t*>(o + b_sc + b_cb), a.data = o + b_sc + b_cb + b_rows;
  } else {
    a.series_chunks = out->series_chunks, a.out_rows = out->rows, a.chunk_bytes = out->chunk_bytes, a.data = out->data;
  }
  if ((rc = launch(ctx, gc::k_export_write, blocks, gc::kEncThreads, 0, false, a)) != GPR_OK) return rc;
  if (host) {
    CU(cudaMemcpyAsync(out->series_chunks, a.series_chunks, b_sc, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(out->chunk_bytes, a.chunk_bytes, b_cb, cudaMemcpyDeviceToHost, ctx->stream));
    if (b_rows) CU(cudaMemcpyAsync(out->rows, a.out_rows, b_rows, cudaMemcpyDeviceToHost, ctx->stream));
    if (b_data) CU(cudaMemcpyAsync(out->data, a.data, b_data, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CU(cudaStreamSynchronize(ctx->stream));
  return GPR_OK;
  GPR_CATCH(ctx)
}

int gpr_synth_fill(gpr_ctx* ctx, uint64_t seed, int32_t plane, float* dst, uint64_t pod_offset,
                   uint32_t n_pods, uint32_t n_gpus, uint32_t n_samples, uint64_t row_stride) {
  if (!ctx) return GPR_E_INVALID;
  if (const int rc = enter(ctx)) return rc;
  if (!dst || n_gpus == 0 || n_samples == 0 || (plane != 0 && plane != 1))
    return fail(ctx, GPR_E_INVALID, "bad gpr_synth_fill arguments");
  const uint64_t rows = (uint64_t)n_pods * n_gpus;
  if (rows == 0) return GPR_OK;
  if (rows > 0x7fffffffull) return fail(ctx, GPR_E_INVALID, "too many series");
  const uint64_t ld = row_stride ? row_stride : n_samples;
  if (const int rc = launch(ctx, gpr::k_synth_fill, capped_grid(ctx, rows, 1, 32), 256, 0, false, dst, seed, plane,
                            pod_offset * n_gpus, (uint32_t)rows, n_samples, ld))
    return rc;
  CU(cudaStreamSynchronize(ctx->stream));
  return GPR_OK;
}

int gpr_synth_eligible(gpr_ctx* ctx, uint64_t seed, uint8_t* dst, uint64_t pod_offset,
                       uint32_t n_pods) {
  if (!ctx) return GPR_E_INVALID;
  if (const int rc = enter(ctx)) return rc;
  if (!dst) return fail(ctx, GPR_E_INVALID, "dst is NULL");
  if (n_pods == 0) return GPR_OK;
  if (const int rc = launch(ctx, gpr::k_synth_eligible, capped_grid(ctx, n_pods, 256, 8), 256, 0, false, dst, seed,
                            pod_offset, n_pods))
    return rc;
  CU(cudaStreamSynchronize(ctx->stream));
  return GPR_OK;
}

}  // extern "C"

#ifdef GPR_TIMELINE
extern "C" GPR_API int gpr_debug_timeline(gpr_ctx* ctx, unsigned long long* out, int n_ctas) {
  if (!ctx || !out) return GPR_E_INVALID;
  if (const int rc = enter(ctx)) return rc;
  CU(cudaStreamSynchronize(ctx->stream));
  CU(cudaMemcpyFromSymbol(out, gpr::g_timeline, sizeof(unsigned long long) * 4 * (size_t)n_ctas));
  return GPR_OK;
}
#endif
