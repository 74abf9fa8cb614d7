/*
 * gpr.h — C ABI of the H100 idle-decision engine (libgpr.so).
 *
 * This is the drop-in boundary for gpu-pruner's one data-parallel path: the per-pod
 * windowed aggregation of DCGM GPU-utilisation samples into an idle/active verdict.
 * In the reference that arithmetic is a PromQL expression evaluated by a remote
 * Prometheus server; the seam this ABI replaces is, in the reference tree,
 *
 *     gpu-pruner/src/main.rs:397      client.query(query).get().await        (send PromQL)
 *     gpu-pruner/src/main.rs:405-409  response.data().into_vector()          (decode result)
 *     gpu-pruner/src/main.rs:416-437  HashSet<(pod, namespace)> dedup        (ANY-GPU fold)
 *     gpu-pruner/src/main.rs:494,508  create_time >= now - lookback => skip  (age gate)
 *
 * i.e. "obtain window matrix -> gpr_decide() -> expand set bits to PodMetricData".
 * Everything after main.rs:444 (Kubernetes lookups, owner walk, scale patches) is
 * unchanged host logic.
 *
 * Conventions (SURVEY.md §8(b)):
 *   - every entry point returns int: 0 = GPR_OK, negative = GPR_E_*; the message for the
 *     last failure on a context is gpr_last_error(ctx) (gpr_last_error(NULL) for a failed
 *     gpr_create).  Nothing aborts, exits or throws across this boundary, so the caller's
 *     failure accounting (main.rs:310-321, QUERY_FAILURES) keeps working.
 *   - the caller owns every in/out buffer; the library owns only what is behind gpr_ctx*.
 *   - a context is NOT re-entrant (one call at a time, matching the single caller at
 *     main.rs:297) but it is thread-agnostic: every entry point selects its device itself
 *     and keeps no thread-local state, because tokio may migrate the caller between ticks.
 *   - plain pointers and sizes only; no torch / C++ types.
 *
 *   - device buffers handed to the library must be complete when the call is made: the context's
 *     own stream is not ordered with the caller's streams.  Either synchronise first or give the
 *     context the caller's stream (gpr_config.stream), in which case stream order is enough.
 *
 * There is no CPU fallback: without a CUDA device gpr_create fails with GPR_E_CUDA.
 */
#ifndef GPR_H_
#define GPR_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define GPR_API __attribute__((visibility("default")))
#else
#define GPR_API
#endif

#define GPR_VERSION_MAJOR 0
#define GPR_VERSION_MINOR 2
#define GPR_VERSION_PATCH 0

/* ---- status codes ------------------------------------------------------------------- */
enum {
  GPR_OK = 0,
  GPR_E_INVALID = -1,   /* bad argument / shape / struct_size                           */
  GPR_E_CUDA = -2,      /* CUDA runtime or driver error (message has the CUDA string)    */
  GPR_E_NOMEM = -3,     /* allocation failed (host or device)                            */
  GPR_E_CAPACITY = -4,  /* window larger than the capacity given at gpr_create           */
  GPR_E_STATE = -5,     /* call not valid in this state (e.g. resident window not set)   */
  GPR_E_NCCL = -6,      /* NCCL error or NCCL library not loadable                       */
  GPR_E_UNSUPPORTED = -7
};

/* ---- where a buffer lives ------------------------------------------------------------ */
enum {
  GPR_MEM_HOST = 0,   /* host memory (pinned via gpr_host_alloc for full PCIe speed)     */
  GPR_MEM_DEVICE = 1  /* device memory on the context's GPU                              */
};

/* ---- kernel selection (both variants are always built; see DESIGN.md §kernels) ------- */
enum {
  GPR_KERNEL_AUTO = 0,
  GPR_KERNEL_LDG = 1,  /* 128-bit ld.global.nc streaming loads, warp per series          */
  GPR_KERNEL_TMA = 2   /* cp.async.bulk (TMA) rows into an mbarrier-guarded smem ring     */
};

/* ---- sample format of gpr_window.util (gpr_window.util_format) ----------------------------
 * DCGM_FI_DEV_GPU_UTIL is an integer percentage, so a caller that parses the range query itself
 * can hand the window over at one byte per sample: a quarter of the PCIe / HBM bytes of the f32
 * layout and the same verdict.  The power plane and the resident ring stay f32.               */
enum {
  GPR_FMT_F32 = 0,  /* f32, NaN = no sample                                               */
  GPR_FMT_U8B = 1   /* biased u8: 0 = no sample, b in 1..255 = sample value b - 1 (0..254);
                       a zero-filled buffer is an all-absent window, like a NaN-filled f32 one;
                       `util` then points at bytes and row_stride counts bytes               */
};

/* ---- gpr_config.flags ---------------------------------------------------------------- */
#define GPR_F_POWER_PLANE 0x1u /* reserve staging for the power plane (host windows)      */
#define GPR_F_BLOCK_INDEX 0x2u /* gpr_resident_init: keep the max of every 64-sample block of the
                                  resident rows up to date in gpr_append / gpr_resident_advance and
                                  decide on that index — identical verdict and series_max, 1/64 of
                                  the bytes per tick.  After gpr_text_parse(GPR_TEXT_RESIDENT) or
                                  direct writes call gpr_resident_reindex (see there)              */

typedef struct gpr_ctx gpr_ctx;

/* Creation-time configuration.  Set struct_size = sizeof(gpr_config).                    */
typedef struct gpr_config {
  uint32_t struct_size;
  int32_t device;          /* CUDA device ordinal                                        */
  uint32_t max_pods;       /* capacity for HOST windows (staging in HBM); 0 = none        */
  uint32_t max_gpus;
  uint32_t max_samples;
  uint32_t flags;          /* GPR_F_*                                                    */
  int32_t kernel_variant;  /* GPR_KERNEL_*                                               */
  int32_t reserved0;
  void *stream;            /* optional caller-owned cudaStream_t all work is ordered on;
                              NULL = the context creates its own non-blocking stream      */
} gpr_config;

/*
 * One window = the range-vector result laid out densely.
 *
 *   n_gpus          series slots per pod, 1..256 (GPR_E_UNSUPPORTED above).
 *   capacity        for HOST windows only the number of cells counts: n_pods * n_gpus * n_samples must not
 *                   exceed max_pods * max_gpus * max_samples of gpr_create (staging is dense).
 *   util[p][g][t]   f32, t fastest; NaN = "no sample" (stale / absent / scrape gap); or biased
 *                   bytes when util_format = GPR_FMT_U8B (cast the pointer).
 *                   Restates DCGM_FI_DEV_GPU_UTIL{pod != ""}[Nm]   (query.promql.j2:16-20)
 *   power[p][g][t]  f32 or NULL.  Restates DCGM_FI_DEV_POWER_USAGE{...}[Nm]
 *                   (query.promql.j2:39-42).  Used only if power_threshold is "truthy".
 *   row_stride      elements between consecutive (p,g) rows; 0 means n_samples.
 *   power_threshold watts; the veto clause exists iff power != NULL and the threshold is
 *                   neither 0.0 nor NaN (Jinja truthiness of `args.power_threshold`,
 *                   query.promql.j2:36).  veto(p) = any g: max_t power[p][g][:] >= up, with
 *                   up = the smallest f32 >= threshold — exactly `(double)cell >= threshold`.
 *                   That equals Prometheus' float64 `x >= threshold` on the samples x only if
 *                   each cell was stored from its sample x by the POWER RULE:
 *                       f = x rounded to nearest f32;
 *                       if (x >= threshold && f <  up) f = up;
 *                       if (x <  threshold && f >= up) f = the f32 just below up;
 *                   (NaN and +-Inf unchanged).  Plain rounding alone vetoes a reading within
 *                   half an f32 ulp below the threshold (149.999999 W rounds to 150.0f).
 *                   gpr_text_parse applies the rule (gpr_text_grid.power_threshold); a caller
 *                   that fills power planes itself (gpr_decide, gpr_append) must apply it too.
 *   eligible[p]     u8 or NULL: 0 = pod fails the Pending / missing-timestamp gates
 *                   (main.rs:473-492).  NULL = all eligible.
 *   created_ts[p]   i64 or NULL: pod creation time in caller-chosen ticks; the pod is skipped
 *                   iff created_ts[p] >= cutoff_ts   (main.rs:494,508-510, cutoff = now -
 *                   (duration*60 + grace_period)).  INT64_MAX = "no creationTimestamp".
 *   groups[p][g]    u32 or NULL (follows mem_kind like the gates): the `sum by (Hostname, container,
 *                   pod, namespace, gpu, modelName)` groups of the query (query.promql.j2:9,21), for
 *                   callers whose window keeps several series of one group in separate rows.
 *                   Bits 0-7: slot of the group's first member (its leader), <= g; a leader's own
 *                   entry leads itself.  GPR_GROUP_UTIL: the row is a DCGM_FI_DEV_GPU_UTIL series,
 *                   divided by 100 before the sum (j2:20); without it the row is summed as it is
 *                   (DCGM_FI_PROF_GR_ENGINE_ACTIVE).  Any other bit, a leader > g or a leader whose
 *                   entry is not its own is GPR_E_INVALID (a host table before anything is enqueued,
 *                   a device table at gpr_sync / the blocking call's return).
 *                   With a table an element is a group, not a row: its value is Prometheus' sum
 *                   (Neumaier-compensated float64, in slot order) of the window maxima of its
 *                   members that have a sample, NaN if none has; the element is idle iff value == 0.
 *                   candidate = some idle element && !veto; n_series counts idle elements.  A row of
 *                   a group of two or more is read whole (no early exit).  series_max and veto_bits
 *                   keep their per-row meaning; the power plane is never grouped (`unless on` needs
 *                   no grouping).  NULL: every row is its own element, as before.
 *   struct_size     sizeof(gpr_window), or offsetof(gpr_window, groups) for a caller built before
 *                   `groups` existed (no table).
 */
typedef struct gpr_window {
  uint32_t struct_size;
  int32_t mem_kind;        /* GPR_MEM_*: applies to util, power, eligible, created_ts     */
  const float *util;
  const float *power;
  const uint8_t *eligible;
  const int64_t *created_ts;
  int64_t cutoff_ts;
  uint32_t n_pods;
  uint32_t n_gpus;
  uint32_t n_samples;
  uint32_t util_format;    /* GPR_FMT_*; ignored by gpr_decide_resident (the ring is f32)   */
  uint64_t row_stride;
  double power_threshold;
  const uint32_t *groups;
} gpr_window;

#define GPR_GROUP_UTIL 0x100u /* gpr_window.groups: a GPU_UTIL member, summed as max / 100 (bits 0-7: leader) */

/*
 * Result.  Bitmaps are packed little-endian within a word: pod p is bit (p & 31) of word
 * (p >> 5); padding bits above n_pods are zero.  With a communicator attached
 * (gpr_comm_init) the bitmaps cover all ranks: world * ceil(n_pods/32) words, rank-major,
 * and n_pods must be a multiple of 32 and identical on every rank.
 *
 *   decision_bits   required.  candidate(p) && eligible(p)         (after main.rs:473-510)
 *   candidate_bits  optional.  (any g: max_t util == 0) && !veto(p) (what Prometheus + the
 *                   dedup at main.rs:416-437 return)
 *   series_max      optional, n_pods * n_gpus f32: window max per series, NaN if no sample
 *                   (the reference's reported `value` is this / 100; lib.rs:184,
 *                   query.promql.j2:20).
 *   veto_bits       optional, ceil(n_pods/32) words, THIS rank's pods only (never exchanged): pods with a
 *                   power series at or above the threshold (the `unless on (pod, namespace)` clause,
 *                   query.promql.j2:36-44).  With series_max it lets a caller re-derive a pod's verdict
 *                   (exact `sum by` of duplicate series, gpu-pruner_b200/host/ingest.cpp).
 *   idle_slots      optional, n_pods * ceil(n_gpus/32) words, THIS rank's pods only: bit g of pod p's
 *                   words is set iff slot g starts an element whose value is == 0 — without a group
 *                   table iff row g's window max == 0; with one iff g leads a group whose sum is == 0
 *                   (members are never set).  Veto and gates do not touch it.  The first set bit of a
 *                   candidate pod is the element the reference reports (main.rs:430-435, value 0).
 *   out_mem_kind    where the buffers above live.
 *   n_series        number of idle elements (series, or groups with gpr_window.groups) in non-vetoed
 *                   pods = QueryResponse.num_pods (main.rs:418; a series count despite the name).
 *   struct_size     sizeof(gpr_result), or offsetof(gpr_result, idle_slots) (no idle_slots).
 *   n_candidates / n_decisions   popcounts of the two bitmaps (this rank's pods).
 *   kernel_ms       device time of the decision kernel(s) for this call (CUDA events);
 *                   0 from the _async entry point.
 */
typedef struct gpr_result {
  uint32_t struct_size;
  int32_t out_mem_kind;
  uint32_t *decision_bits;
  uint32_t *candidate_bits;
  float *series_max;
  uint32_t *veto_bits;
  uint64_t n_series;
  uint64_t n_candidates;
  uint64_t n_decisions;
  double kernel_ms;
  uint32_t *idle_slots;
} gpr_result;

/* ---- lifecycle ----------------------------------------------------------------------- */
GPR_API int gpr_version(void); /* major*10000 + minor*100 + patch */
GPR_API int gpr_create(const gpr_config *cfg, gpr_ctx **out);
/* Releases everything the context owns.  An unfinished gpr_text_scan_begin is stopped (its upload threads joined,
 * their copies and scans drained) and the context's stream synchronised before anything is released. */
GPR_API void gpr_destroy(gpr_ctx *ctx);
GPR_API const char *gpr_last_error(const gpr_ctx *ctx);

/* ---- the hot path -------------------------------------------------------------------- */
/* Blocking: on return the result buffers and counters are complete, and so are those of every
 * decision enqueued before it (the call retires them like gpr_sync).  A failing call never drops
 * or changes decisions enqueued before it: they stay pending for the next gpr_sync.       */
GPR_API int gpr_decide(gpr_ctx *ctx, const gpr_window *win, gpr_result *res);
/* Enqueue only (device or pinned-host buffers); counters are filled by gpr_sync().       */
GPR_API int gpr_decide_async(gpr_ctx *ctx, const gpr_window *win, gpr_result *res);
/* Waits for everything enqueued and fills the counters of every pending result, whatever failed in
 * between (a failed gpr_decide / gpr_decide_resident / _async call leaves earlier results pending). */
GPR_API int gpr_sync(gpr_ctx *ctx);
/* Enqueue n independent decisions (windows[i] -> results[i]) in one call: the same as n calls of
 * gpr_decide_async, without n trips through the caller's FFI.  At most 256 results may be
 * outstanding between two gpr_sync calls.  Stops at the first failing window and returns its code. */
GPR_API int gpr_decide_batch_async(gpr_ctx *ctx, const gpr_window *windows, gpr_result *results,
                                   uint32_t n);

/* ---- resident window for daemon mode (--daemon-mode / --check-interval, main.rs:286-330)
 * The window lives in HBM as a ring over the time axis; each tick appends the columns that
 * arrived since the previous tick and rescans.  max is order-independent so ring order is
 * irrelevant to the verdict.                                                              */
GPR_API int gpr_resident_init(gpr_ctx *ctx, uint32_t n_pods, uint32_t n_gpus, uint32_t n_samples,
                      uint32_t flags /* GPR_F_POWER_PLANE | GPR_F_BLOCK_INDEX */);
/* new columns laid out [p][g][n_new] (row_stride 0 = n_new); power cells stored by the power
 * rule of gpr_window.power_threshold.  power_cols may be NULL: the power plane (if any) then
 * has no sample in the new buckets, as after gpr_resident_advance.  Only the newest n_samples
 * of the columns are kept.  With GPR_F_BLOCK_INDEX the index blocks of the new buckets are
 * recomputed.                                                                             */
GPR_API int gpr_append(gpr_ctx *ctx, const float *util_cols, const float *power_cols, uint32_t n_new,
               uint64_t row_stride, int32_t mem_kind);
/* Open the next n_new buckets of the ring without data: their columns become "no sample" in every row of
 * every resident plane and the ring head moves on; with GPR_F_BLOCK_INDEX their index blocks are recomputed.
 * The tick's samples are then merged in by gpr_text_parse(GPR_TEXT_RESIDENT) (device-side ingest of the
 * tick's range-query slice), which leaves the index stale: call gpr_resident_reindex after the parse,
 * before gpr_decide_resident (which returns GPR_E_STATE on a stale index).                          */
GPR_API int gpr_resident_advance(gpr_ctx *ctx, uint32_t n_new);
/* rebuild the GPR_F_BLOCK_INDEX index from the resident planes; a no-op without an index.  Required
 * after gpr_text_parse(GPR_TEXT_RESIDENT) (the library marks the index stale and refuses to decide on
 * it) and after writing the planes directly through gpr_resident_planes (which the library cannot
 * see: deciding before the rebuild gives the verdict of the old index, without an error).          */
GPR_API int gpr_resident_reindex(gpr_ctx *ctx);
/* win->util / win->power are ignored (resident planes are used); gates come from win.     */
GPR_API int gpr_decide_resident(gpr_ctx *ctx, const gpr_window *win, gpr_result *res);
/* device pointers of the resident planes (for generators / inspection); power may be NULL */
GPR_API int gpr_resident_planes(gpr_ctx *ctx, float **util, float **power, uint64_t *row_stride);
/* ring position the next appended bucket goes to; the newest bucket is at (head + n_samples - 1) % n_samples  */
GPR_API int gpr_resident_head(gpr_ctx *ctx, uint32_t *head);
/* Give the ring a new shape [n_pods][n_gpus][n_samples] without losing its history: new row i
 * (= pod * n_gpus + slot) holds old row src_rows[i] with every sample at its ring position, or no
 * sample for GPR_ROW_NONE.  So pods can join beyond the head-room, a pod can gain series slots, and
 * departed pods can be dropped without a query of the full window: the ring equals the one a rebuild
 * from the full range would give if new row i were fed by the series that fed old row src_rows[i].
 * n_samples, the head, the power plane and the GPR_F_BLOCK_INDEX index stay; index rows move with
 * their rows (a stale index stays stale).  src_rows holds n_pods * n_gpus entries in host or device
 * memory (mem_kind); it is checked before the new ring is allocated or the old one written (a
 * device map's check uses context scratch of 2 bits per old row): an entry >= the old
 * n_pods * n_gpus that is not GPR_ROW_NONE, or an old row named twice, is GPR_E_INVALID, and the
 * message names the first new row whose entry is out of range or shared with another new row; no
 * resident window is GPR_E_STATE.  On any error (GPR_E_NOMEM included) the ring, its index and its
 * head are as they were.  Out of place: the new ring is built beside the old
 * one, so the peak is the old ring plus the new one in HBM.  Decisions enqueued before the call read
 * the old ring and retire at the next gpr_sync; pointers from gpr_resident_planes are stale after it.  */
#define GPR_ROW_NONE 0xFFFFFFFFu
GPR_API int gpr_resident_remap(gpr_ctx *ctx, uint32_t n_pods, uint32_t n_gpus, const uint32_t *src_rows,
                               int32_t mem_kind);
/* bit r of bits[r >> 5] (bit r & 31) = ring row r holds at least one sample in plane 0 or, if the ring has
 * one, plane 1; ceil(n_rows / 32) words, padding bits zero.  host or device output (mem_kind).
 * Every NaN cell counts as "no sample", not only the fill.  With GPR_F_BLOCK_INDEX and a current
 * index the index rows are read instead of the planes (1/64 of the bytes); a stale index is not read
 * and not refused.  Blocking, reads the ring only; decisions enqueued before it stay pending.  No
 * resident window is GPR_E_STATE, a NULL bits or a bad mem_kind GPR_E_INVALID; on any error bits is
 * untouched.
 * The remap recipe of a daemon caller whose cluster outgrew the ring: open the tick's buckets
 * (gpr_resident_advance), read the live rows, keep every pod with a live row or a series in the tick's
 * slice, and gpr_resident_remap the kept pods' rows (and GPR_ROW_NONE for the new ones) into
 * [kept + head-room][max(G, slots needed)]; then append the slice as on any tick.                    */
GPR_API int gpr_resident_live_rows(gpr_ctx *ctx, uint32_t *bits, int32_t mem_kind);
/* out[r * n_cols + j] = plane `plane` of ring row r at the bucket (n_cols - 1 - j + newer) back from the newest:
 * the n_cols buckets that end `newer` buckets before the newest, oldest first, for every ring row (n_pods * n_gpus).
 * Cells are copied as bits (a NaN is "no sample").  Host or device output (mem_kind); a host one goes through
 * context scratch and is copied out once.  Blocking, reads the ring only; decisions enqueued before it stay
 * pending.  No resident window, or plane 1 on a ring without a power plane, is GPR_E_STATE; a plane other than
 * 0 or 1, n_cols == 0, newer + n_cols > n_samples, a NULL out or a bad mem_kind GPR_E_INVALID; on any error out
 * is untouched.
 * A daemon caller that re-asks the newest L seconds it already holds (samples that reached the server late)
 * reads the re-asked band before and after the tick's merge to see what the late samples changed.           */
GPR_API int gpr_resident_cols(gpr_ctx *ctx, int32_t plane, uint32_t newer, uint32_t n_cols, float *out,
                              int32_t mem_kind);
/* Put the ring on a coarser or shorter time grid without a query: keep its newest n_keep buckets and merge them
 * `factor` to a bucket, newest first, so new bucket b (0 = newest) is the maximum of old buckets
 * [factor * b, min(factor * b + factor, n_keep)) and n_samples becomes ceil(n_keep / factor).  The merge gives the
 * bits a fresh gpr_samples_scatter of the same samples gives: every NaN is "no sample", a group without a sample is
 * the fill 0xFFFFFFFF, +0 beats -0.  A window of N s at step s ending at t_end becomes exactly the window of N' s
 * at step s' = factor * s ending at t_end when N' <= N and N' % s == 0 (n_keep = N' / s) or N' == N
 * (n_keep = n_samples); other grids need samples the ring does not hold.  n_pods, n_gpus, the rows and the power
 * plane stay (power cells are snapped already: a maximum of snapped values is snapped); afterwards
 * gpr_resident_head reports 0.  With GPR_F_BLOCK_INDEX the index is reallocated for the new n_samples and rebuilt
 * from the new planes, so it is current after the call even if it was stale before.  Out of place like
 * gpr_resident_remap: the gathers run on the context's stream after whatever is enqueued there, the call waits for
 * them, and the peak is the old ring plus the new one in HBM.  Decisions enqueued before the call read the old ring
 * and retire at the next gpr_sync; pointers from gpr_resident_planes are stale after it.  No resident window is
 * GPR_E_STATE; factor == 0, n_keep == 0 or n_keep > n_samples GPR_E_INVALID.  On any error (GPR_E_NOMEM included)
 * the ring, its index and its head are as they were.                                                          */
GPR_API int gpr_resident_retime(gpr_ctx *ctx, uint32_t n_keep, uint32_t factor);

/* ---- multi-GPU: one process per GPU, pods sharded by rank, one allgather of the bitmap - */
#define GPR_UNIQUE_ID_BYTES 128
GPR_API int gpr_comm_unique_id(void *id128);                       /* rank 0; ship to the others */
GPR_API int gpr_comm_init(gpr_ctx *ctx, const void *id128, int rank, int world);
GPR_API int gpr_comm_destroy(gpr_ctx *ctx);

/* ---- multi-GPU, fused: the decision kernel itself exchanges the bitmap over NVLink peer memory.
 * Each rank: gpr_p2p_init -> ship the 64-byte handle to every rank (any side channel) ->
 * gpr_p2p_attach(all handles, rank-major).  Afterwards gpr_decide behaves as with a communicator
 * (global rank-major bitmaps, n_pods a multiple of 32 and <= max_pods_per_rank, all ranks calling
 * in lock-step) but launches no collective: the fold kernel's CTAs store this rank's words into every peer's
 * buffer as 64-bit {step tag, word} slots the moment they exist (no fence, no flag), and its last CTA reads the
 * peers' slots until their tags match and assembles the result.  (GPR_EXCHANGE=flags selects the older protocol:
 * words, one system-scope fence, one flag per peer; GPR_EXCHANGE=pipelined lets a decision's exchange overlap
 * with its predecessor's — only the write of the caller's outputs stays ordered.)  At most 8 ranks.  A peer that never arrives does not hang the
 * GPU: the wait gives up after 20 s and the next gpr_sync / blocking call returns GPR_E_STATE.                  */
#define GPR_P2P_HANDLE_BYTES 64
GPR_API int gpr_p2p_init(gpr_ctx *ctx, int rank, int world, uint32_t max_pods_per_rank,
                         void *handle64);
GPR_API int gpr_p2p_attach(gpr_ctx *ctx, const void *handles /* world * 64 bytes */);
/* Timing switch for attributing the cost of the fused exchange (bench.py's breakdown); all ranks must
 * switch together.  0 = normal; 1 = push the words and flags but do not wait for the peers; 2 = no push
 * at all.  In modes 1 and 2 the returned bitmaps are NOT global.                                    */
GPR_API int gpr_p2p_debug(gpr_ctx *ctx, int32_t mode);

/* ---- memory helpers ------------------------------------------------------------------ */
GPR_API int gpr_host_alloc(gpr_ctx *ctx, size_t bytes, void **out); /* pinned host memory         */
GPR_API int gpr_host_free(gpr_ctx *ctx, void *p);
GPR_API int gpr_device_alloc(gpr_ctx *ctx, size_t bytes, void **out);
GPR_API int gpr_device_free(gpr_ctx *ctx, void *p);
GPR_API int gpr_memcpy(gpr_ctx *ctx, void *dst, const void *src, size_t bytes,
               int32_t dst_kind, int32_t src_kind);          /* blocking                   */

/* ---- measurement support ------------------------------------------------------------- */
/* CUDA events on the context's stream: begin; ...enqueue...; end -> elapsed ms.
 * gpr_timer_begin first enqueues a device-side rendezvous: with a fused exchange attached
 * (gpr_p2p_attach) every rank's stream waits, on the GPU, until all ranks have reached their
 * gpr_timer_begin, so the timed regions of all ranks start within an NVLink round trip of each other
 * whatever the skew between the host threads (with gpr_comm_init only, a one-word ncclAllGather plays
 * that role).  It is therefore COLLECTIVE when world > 1: all ranks must call it in lock-step.     */
GPR_API int gpr_timer_begin(gpr_ctx *ctx);
GPR_API int gpr_timer_end(gpr_ctx *ctx, double *ms);
/* Per-decision completion times: ns[i] = the device's %globaltimer (nanoseconds) at which the i-th of
 * the decisions retired by the most recent gpr_sync / blocking call finished (bitmap complete, exchange
 * included); *begin_ns = the same clock at the release of the last gpr_timer_begin.  *n = number of
 * decisions retired (may exceed cap).  Differences of consecutive stamps are the per-step device times
 * SURVEY.md §8(d) asks the median of.                                                              */
GPR_API int gpr_step_stamps(gpr_ctx *ctx, uint64_t *ns, uint32_t cap, uint32_t *n, uint64_t *begin_ns);
/* Four more stamps per retired decision, for attributing the time of the fold / exchange kernel: the fold kernel's
 * start (the reduce has completed and the previous fold is done), fold finished, peer flags raised (stores and
 * system-scope fence done; 0 without an exchange), all peers' words arrived (0 without an exchange).           */
GPR_API int gpr_phase_stamps(gpr_ctx *ctx, uint64_t *ns, uint32_t cap, uint32_t *n);
/* writes > L2-size bytes so the next launch starts with a cold L2                          */
GPR_API int gpr_flush_l2(gpr_ctx *ctx);
/* number of kernels this context has launched since creation                               */
GPR_API int gpr_launch_count(const gpr_ctx *ctx, uint64_t *n);
/* device facts: sm_count, l2 bytes, total HBM bytes, cc major/minor                        */
typedef struct gpr_device_info {
  uint32_t struct_size;
  int32_t sm_count;
  int32_t cc_major, cc_minor;
  uint64_t l2_bytes;
  uint64_t hbm_bytes;
  char name[64];
} gpr_device_info;
GPR_API int gpr_get_device_info(gpr_ctx *ctx, gpr_device_info *info);

/* ---- synthetic DCGM windows (SURVEY.md §8(d)); counter-based so any implementation can
 * regenerate any cell.  plane: 0 = util, 1 = power.  Fills rows for pods
 * [pod_offset, pod_offset + n_pods) of a seeded (.., n_gpus, n_samples) universe into dst
 * (device memory, row_stride 0 = n_samples).  elig/created are optional device outputs.    */
GPR_API int gpr_synth_fill(gpr_ctx *ctx, uint64_t seed, int32_t plane, float *dst, uint64_t pod_offset,
                   uint32_t n_pods, uint32_t n_gpus, uint32_t n_samples, uint64_t row_stride);
GPR_API int gpr_synth_eligible(gpr_ctx *ctx, uint64_t seed, uint8_t *dst, uint64_t pod_offset,
                       uint32_t n_pods);

/* ---- device-side ingest of the range-query response TEXT ---------------------------------------
 * The step before the hot path: Prometheus' matrix JSON (the shape gpu-pruner/src/bin/querytest.rs:41-53
 * walks; series = label map + [[<unix time>, "<value>"], ...]) is parsed on the GPU straight into the
 * dense tensor in HBM, so the f32 window never exists on the host.  Division of labour:
 *   gpr_text_scan    uploads the text and reports where every sample list opens (`},"values":[`)
 *                    and closes (`"]]`);
 *   the caller       parses the label maps (~1 % of the bytes) and assigns every series its tensor
 *                    row — label precedence of lib.rs:153-187, `sum by` groups of query.promql.j2:9
 *                    (gpu-pruner_b200/host/ingest_device.cpp does this);
 *   gpr_text_parse   parses all samples of the given spans into a plane [n_rows][n_samples] f32
 *                    (0xFFFFFFFF, a NaN = no sample) — a context-owned plane, or the resident ring of
 *                    daemon mode.
 * Where a sample goes (the same rule as the CPU ingest, gpu-pruner_b200/host/ingest_internal.hpp):
 *   inside the window iff  t_end - window_seconds < ts <= t_end      (PromQL [Nm] at t_end, left-open)
 *   bucket back = (t_end - ts) / step  (0 = newest), column n_samples - 1 - back; several samples of a
 *   row in one bucket are merged with a NaN-aware max — which is what max_over_time over the row
 *   (query.promql.j2:10,16) computes anyway, so collisions, sample order and duplicate series need no
 *   special handling.
 * Numbers are converted exactly like strtod + (float): Clinger's fast path or Eisel-Lemire (17-digit
 * DCGM_FI_PROF_GR_ENGINE_ACTIVE ratios included).  The device parser is strict: anything but
 * `[digits[.digits],"<decimal, at most 19 significant digits>|NaN|+Inf|-Inf"]` sets GPR_SPAN_HARD on the span;
 * the caller re-parses the rows of hard spans on the CPU and overwrites them with gpr_memcpy, so the
 * tensor equals a CPU ingest for every input.
 */
typedef struct gpr_text_span {
  uint64_t begin;    /* offset of the first byte after `"values":[` (a '[')                    */
  uint64_t end;      /* offset of the ']' that closes the sample list                          */
  uint32_t row;      /* destination row = pod * n_gpus + slot                                  */
  uint32_t flags;    /* GPR_SPAN_SHARED in; GPR_SPAN_HARD out                                  */
  uint32_t n_in;     /* out: samples parsed                                                    */
  uint32_t n_oow;    /* out: samples outside the window                                        */
  uint32_t n_tiny;   /* out: non-zero values below the f32 denormal range, kept non-zero       */
  uint32_t reserved;
} gpr_text_span;
#define GPR_SPAN_SHARED 1u /* several series feed this row (informational; every merge is atomic)   */
#define GPR_SPAN_HARD 2u   /* the device parser gave up on this span: re-parse its row on the CPU */

typedef struct gpr_text_grid {
  uint32_t struct_size;
  uint32_t flags;          /* GPR_TEXT_*                                                            */
  int64_t t_end;           /* newest second of the window (inclusive)                               */
  int64_t window_seconds;  /* samples with t_end - window_seconds < ts <= t_end are inside          */
  int64_t step;            /* seconds per column, > 0                                               */
  uint32_t n_samples;      /* columns; >= ceil(window_seconds / step)                               */
  uint32_t n_rows;
  double power_threshold;  /* plane 1: the gpr_window.power_threshold the plane will be decided with;
                              its samples are stored by the power rule of gpr_window (0.0 / NaN: no
                              power clause, plain rounding).  Ignored for plane 0.                  */
} gpr_text_grid;
#define GPR_TEXT_FILL 1u     /* fill the destination plane with "no sample" first (context planes)    */
#define GPR_TEXT_RESIDENT 2u /* destination = the resident ring (gpr_resident_init): n_samples must be its
                                n_samples, n_rows <= its rows; the newest bucket is the ring's newest
                                column (call gpr_resident_advance first to open the tick's buckets)  */

/* Copy `n_bytes` of response text to the device (pinned host memory from gpr_host_alloc moves at
 * full PCIe speed; ordinary memory is staged through a pinned ring by a few host threads, and every
 * chunk is scanned as it lands) and scan it.  Up to `cap` offsets are written to each of opens[]
 * (position of the '}' of `},"values":[`) and closes[] (position of the '"' of `"]]`), UNSORTED; the
 * true counts are returned in *n_opens / *n_closes (GPR_E_CAPACITY if either exceeds cap; call again
 * with a larger one).  The scan itself has room for 16,384 markers of each kind in every piece of the
 * text (gpr_text_scan_next): one per 128 bytes, for every source memory and GPR_TEXT_CHUNK_MB.  A text
 * whose `},"values":[` and whose `"]]` are each at least 128 bytes apart always fits; a denser piece
 * fails the scan with GPR_E_CAPACITY naming the piece (the text is not malformed: parse it on the CPU).
 * The text stays resident in the context's slot `slot` (0..2: a tick has up to three responses — PROF,
 * UTIL, POWER) for gpr_text_parse until the next gpr_text_scan of that slot.  Blocking.              */
GPR_API int gpr_text_scan(gpr_ctx *ctx, int32_t slot, const char *text, uint64_t n_bytes,
                          int32_t mem_kind, uint64_t *opens, uint64_t *closes, uint64_t cap,
                          uint64_t *n_opens, uint64_t *n_closes);
/* The same, as a pipeline the caller can work alongside: gpr_text_scan_begin starts the upload (producer threads
 * owned by the library) and returns; every gpr_text_scan_next blocks until the next piece of the text (2 MB; 1 MB
 * for pageable text at GPR_TEXT_CHUNK_MB=1) has landed and been scanned and returns that piece's markers (sorted;
 * room for `cap` of each kind — 16,384 always suffices) together with *bytes_done = how much of the text is covered
 * so far.  A piece with more than `cap` markers of a kind returns GPR_E_CAPACITY with its true counts and may be
 * asked for again with a larger cap; a piece with more than 16,384 (markers less than 128 bytes apart on average)
 * returns GPR_E_CAPACITY and ends the scan.  *more = 0 with the last piece
 * (or at once for an empty text); the scan is then complete and the text ready for gpr_text_parse.  Between the
 * calls the caller can already walk the series whose markers it has (gpu-pruner_b200/host/ingest_device.cpp turns
 * label maps into tensor rows while later chunks are still crossing PCIe).  Dropped by the next
 * gpr_text_scan_begin / gpr_text_scan / gpr_destroy if not run to the end.  `text` must stay valid until then. */
GPR_API int gpr_text_scan_begin(gpr_ctx *ctx, int32_t slot, const char *text, uint64_t n_bytes, int32_t mem_kind);
GPR_API int gpr_text_scan_next(gpr_ctx *ctx, uint64_t *opens, uint64_t *closes, uint64_t cap, uint64_t *n_opens,
                               uint64_t *n_closes, uint64_t *bytes_done, int32_t *more);
/* Parse the samples of spans[0..n_spans) (host array, sorted by begin, non-overlapping) of the text in
 * `slot` into plane `plane` (0 = util, 1 = power).  Out-fields of the spans are filled.  Blocking.  */
GPR_API int gpr_text_parse(gpr_ctx *ctx, int32_t slot, gpr_text_span *spans, uint32_t n_spans,
                           const gpr_text_grid *grid, int32_t plane);
/* Device pointers of the context planes (NULL if never parsed); valid until the next gpr_text_parse
 * or gpr_samples_scatter that has to grow them, or gpr_destroy.  Hand them to gpr_decide with
 * mem_kind = GPR_MEM_DEVICE.                                                                         */
GPR_API int gpr_text_planes(gpr_ctx *ctx, float **util, float **power);

/* ---- decoded samples into the same planes -----------------------------------------------------------
 * For a caller whose Prometheus client has already decoded the range query (prometheus-http-query's
 * RangeVector: a label map and samples() = [(timestamp f64 s, value f64)] per series): the samples go
 * straight into a context plane or the resident ring, with every rule of the text path applied on the GPU.
 *
 * Samples in CSR form: series s owns samples [offsets[s], offsets[s+1]) and they go to row rows[s] of the
 * destination (several series may feed one row; samples may come in any order).  Timestamps are Unix
 * MILLISECONDS.  A Rust caller converts Sample::timestamp() with (ts * 1000.0).round() as i64, which is
 * exact: Prometheus timestamps are whole milliseconds.  Values are passed as decoded (f64).           */
struct gpr_sample_batch {
  uint32_t struct_size;     /* sizeof(gpr_sample_batch)                                                */
  int32_t mem_kind;         /* GPR_MEM_*: applies to every array below                                 */
  const uint64_t *offsets;  /* n_series + 1, non-decreasing, offsets[0] = 0                            */
  const uint32_t *rows;     /* n_series, each < grid.n_rows                                            */
  const int64_t *ts_ms;     /* offsets[n_series] timestamps, Unix milliseconds (any order)             */
  const double *values;     /* offsets[n_series] values as decoded (f64)                               */
  uint32_t n_series;
  uint32_t reserved;
};
typedef struct gpr_sample_batch gpr_sample_batch;

/* n_in: samples in the batch; n_oow: of those, outside the window; n_tiny: in-window non-zero values
 * below the f32 denormal range, kept non-zero — the sums of gpr_text_span's counters for the same
 * samples written as text.                                                                          */
struct gpr_sample_stats {
  uint64_t n_in;
  uint64_t n_oow;
  uint64_t n_tiny;
};
typedef struct gpr_sample_stats gpr_sample_stats;

/* Same destination, grid and flags as gpr_text_parse (GPR_TEXT_FILL: a context plane; GPR_TEXT_RESIDENT:
 * the ring, after gpr_resident_advance; like a text parse it leaves the block index stale, so call
 * gpr_resident_reindex before gpr_decide_resident).  The cell a sample lands in, and the value it leaves
 * there, are those gpr_text_parse produces for the same sample written as text ([ts_ms / 1000 as a
 * decimal, "<value printed round-trip>"]):
 *   value  to_f32 (rounded to nearest, a non-zero value stays non-zero), and on plane 1 the POWER RULE of
 *          gpr_window against grid.power_threshold; NaN samples are dropped;
 *   cell   t_end - window_seconds < ts <= t_end (in ms), bucket (t_end - ts) / step counted back from the
 *          newest column;
 *   merge  NaN-aware max, as in the text path.
 * The batch is checked before anything is written — host arrays on the host, device arrays by a kernel
 * whose verdict is read back first: a bad struct_size, offsets[0] != 0, decreasing offsets or a row
 * >= grid.n_rows returns GPR_E_INVALID and leaves the destination untouched.  GPR_TEXT_RESIDENT without a
 * resident window is GPR_E_STATE.  Device arrays are read in place; host arrays (pinned from
 * gpr_host_alloc, or pageable) are uploaded in pieces that overlap with the scatter, so a batch needs no
 * device copy of itself.  stats may be NULL.  Blocking; results enqueued before the call stay pending.   */
GPR_API int gpr_samples_scatter(gpr_ctx *ctx, const gpr_sample_batch *batch, const gpr_text_grid *grid,
                                int32_t plane, gpr_sample_stats *stats);

/* ---- Prometheus XOR chunks into the same planes ------------------------------------------------------
 * For a caller that reads series as stored chunks (Prometheus remote read with the STREAMED_XOR_CHUNKS
 * response type, or a Thanos StoreAPI Series call): the `data` field of every XOR chunk, back to back in
 * one buffer, decoded and merged on the GPU.  Framing, CRCs and label maps stay with the caller.
 *
 * CSR over chunks: series s owns chunks [series_chunks[s], series_chunks[s+1]) and feeds row rows[s];
 * chunk c is data[chunk_bytes[c], chunk_bytes[c+1]), in Prometheus' XOR encoding (tsdb/chunkenc/xor.go:
 * a big-endian u16 sample count, then the bit stream).  Chunks may overlap in time and come in any
 * order.  Histogram chunks are not accepted.                                                         */
struct gpr_chunk_batch {
  uint32_t struct_size;           /* sizeof(gpr_chunk_batch)                                             */
  int32_t mem_kind;               /* GPR_MEM_*: applies to every array below                             */
  const uint64_t *series_chunks;  /* n_series + 1: series s owns chunks [series_chunks[s], series_chunks[s+1]) */
  const uint32_t *rows;           /* n_series, each < grid.n_rows                                        */
  const uint64_t *chunk_bytes;    /* n_chunks + 1: chunk c is data[chunk_bytes[c], chunk_bytes[c+1])     */
  const uint8_t *data;            /* the XOR chunks' `data` fields, back to back, any alignment          */
  uint32_t n_series;
  uint32_t reserved;
};
typedef struct gpr_chunk_batch gpr_chunk_batch;

/* Same destination, grid, flags and stats as gpr_samples_scatter: every decoded sample lands in the cell,
 * with the f32 bits, that gpr_samples_scatter gives the same (ts_ms, value), and so gpr_text_parse.  NaN
 * samples are dropped, Prometheus' staleness marker (0x7ff0000000000002) among them.  stats->n_in counts
 * the decoded samples; a chunk's samples outside the window are counted in n_oow (chunks come whole, so a
 * daemon slice has many).  The batch is checked before anything is written: a bad struct_size, offsets
 * that do not start at 0 or decrease (series_chunks or chunk_bytes), a row >= grid.n_rows, a chunk
 * shorter than its 2-byte header, a chunk whose decode would read past its own bytes (or whose varint
 * overflows 64 bits), a value that reuses the XOR window before one was set, or (host batches) a chunk
 * over 32 MB returns GPR_E_INVALID, naming the first bad chunk, with the destination untouched.  The
 * index arrays of a host batch are checked on the host; chunk data, and every array of a device batch,
 * by a check kernel whose verdict is read back before the merge.  Device arrays are read in place; host chunk data goes up in pieces cut at chunk
 * boundaries through the staging of gpr_samples_scatter (a batch larger than two pieces, 64 MB, crosses
 * PCIe twice: once to be checked, once to be merged).  stats may be NULL.  Blocking; results enqueued
 * before the call stay pending.                                                                       */
GPR_API int gpr_chunks_scatter(gpr_ctx *ctx, const gpr_chunk_batch *batch, const gpr_text_grid *grid,
                               int32_t plane, gpr_sample_stats *stats);

/* ---- the resident ring as XOR chunks: a snapshot a restarted caller restores ---------------------------
 * gpr_resident_export encodes one plane of the ring (0 = util, 1 = power) on the GPU as Prometheus XOR
 * chunks, in the CSR form gpr_chunks_scatter takes.  Every ring row with a sample is one series; its
 * samples are its cells oldest first, sample j (ring position (head + j) % n_samples) at
 *   ts_ms = grid.t_end * 1000 - (n_samples - 1 - j) * grid.step * 1000,   value = (double)cell,
 * NaN cells skipped, cut into chunks of at most max_per_chunk samples (Prometheus cuts at 120).  The bytes
 * are those Prometheus' appender writes for the same samples.
 *
 * Sizes follow the two calls of gpr_text_scan: with a capacity too small (n_series > cap_series,
 * n_chunks > cap_chunks or n_bytes > cap_bytes) the call returns GPR_E_CAPACITY with the true counts and
 * writes none of the five arrays; call again with room.  The counts are filled whenever the ring was
 * encoded.  Errors: a bad struct_size, grid (as gpr_chunks_scatter checks it), grid.n_samples other than
 * the ring's, mem_kind, a NULL series_chunks or chunk_bytes (or rows / data with room), or max_per_chunk
 * outside 1..65535 is GPR_E_INVALID; no
 * resident window, or plane 1 on a ring without a power plane, is GPR_E_STATE.  grid.n_rows and
 * grid.flags are ignored; grid.window_seconds is for the restore.  Device outputs are written in
 * place; host outputs (pinned or pageable) are encoded into context scratch and copied out, each array
 * once.  Context scratch: 4 B per chunk the ring could hold (n_samples / max_per_chunk rounded up, per row)
 * and 20 B per row, plus the outputs for host ones.  The ring, its head and its index are only read.
 * Blocking; results enqueued before the call stay pending.
 *
 * Restore: gpr_resident_init with the same n_samples, then gpr_chunks_scatter(GPR_TEXT_RESIDENT) with the
 * same grid and power_threshold (and `rows` mapped through the caller's pod table if the shape changed),
 * then gpr_resident_reindex.  This gives a ring whose unrolled window equals the exported one bit for bit
 * (every NaN reads back as the fill 0xFFFFFFFF) when every column is inside the grid's window:
 * (n_samples - 1) * step < window_seconds, as with n_samples = ceil(window_seconds / step).  DESIGN.md §8h
 * gives the argument.                                                                                   */
struct gpr_chunk_export {
  uint32_t struct_size;    /* sizeof(gpr_chunk_export)                                                  */
  int32_t mem_kind;        /* GPR_MEM_*: where the four arrays below live                               */
  uint64_t *series_chunks; /* cap_series + 1: series s owns chunks [series_chunks[s], series_chunks[s+1]) */
  uint32_t *rows;          /* cap_series: the ring row of each exported series, ascending               */
  uint64_t *chunk_bytes;   /* cap_chunks + 1: chunk c is data[chunk_bytes[c], chunk_bytes[c+1])          */
  uint8_t *data;           /* cap_bytes: the chunks, back to back                                       */
  uint64_t cap_series;
  uint64_t cap_chunks;
  uint64_t cap_bytes;
  uint64_t n_series;       /* out: rows with at least one sample                                        */
  uint64_t n_chunks;       /* out                                                                        */
  uint64_t n_bytes;        /* out                                                                        */
  uint64_t n_samples;      /* out: present cells                                                        */
};
typedef struct gpr_chunk_export gpr_chunk_export;

GPR_API int gpr_resident_export(gpr_ctx *ctx, const gpr_text_grid *grid, int32_t plane,
                                uint32_t max_per_chunk, gpr_chunk_export *out);

#ifdef __cplusplus
}
#endif
#endif /* GPR_H_ */
