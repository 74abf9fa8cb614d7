// gpr_kernels.cuh — sm_90a kernels of the idle-decision engine.
//
// The arithmetic replaced here is the PromQL expression of the reference,
// gpu-pruner/src/query.promql.j2:1-44, plus the Rust-side ANY-GPU dedup
// (gpu-pruner/src/main.rs:416-437) and age gate (main.rs:473-510):
//
//   smax(p,g)   = max_over_time(util[p,g,:])         NaN = missing step, NaN iff none present
//   idle_s(p,g) = smax(p,g) == 0                     (query.promql.j2:35)
//   veto(p)     = any g: max_over_time(power[p,g,:]) >= T       (query.promql.j2:36-44)
//   candidate   = (any g: idle_s) && !veto           (main.rs:416-437)
//   decision    = candidate && eligible && !(created >= cutoff)  (main.rs:473-510)
//
// Two phases:
//   reduce : one pass over the f32 tensor(s) — 100 % of the algorithmic bytes — producing one
//            flag byte per series row.  Two interchangeable implementations:
//              k_reduce_ldg  128-bit ld.global.nc streaming loads, warp per row
//              k_reduce_tma  cp.async.bulk (TMA, SASS UBLKCP) row chunks into warp-private,
//                            mbarrier-guarded shared-memory rings
//   fold   : per-pod masks -> verdict -> packed uint32 bitmaps + counts (touches 4 B per pod, <0.1 %),
//            plus, on more than one GPU, the exchange of the packed words over NVLink peer memory.
//            A small second kernel (k_fold) chained to the reduce kernel by programmatic dependent
//            launch: it is resident before the reduce ends, folds the moment the reduce grid has
//            completed, and never occupies a streaming CTA's SM slot, so the next decision's reduce
//            kernel takes over the SMs while this one is still folding / exchanging.
//
// HBM-bound streaming max: ~1 FMNMX per 4 bytes, no tensor cores, no reuse.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "gpr_launch.h"

namespace gpr {

// ------------------------------------------------------------------------------------------
// parameters
// ------------------------------------------------------------------------------------------
constexpr int kMaxPeers = 8;  // one NVSwitch box

struct Segment {
  const float* base;   // first row of this segment (device)
  uint32_t* mask;      // per-pod bitmask (MW = ceil(G / 32) words per pod), bit g set when series (pod, g) is
                       // flagged: util plane -> idle_s = (max == 0), power plane -> veto_s = (max >= thr);
                       // word (first_pod + local_row / G) * MW + g / 32; zero between calls (the fold
                       // clears every word it reads)
  float* smax;         // optional per-row window max (util segment only)
  uint32_t n_rows;
  uint32_t is_power;
};

struct FoldParams {
  uint32_t* idle_mask;        // [P]   read, then cleared
  uint32_t* veto_mask;        // [P] or nullptr
  const uint8_t* eligible;    // [P] or nullptr
  const int64_t* created;     // [P] or nullptr
  int64_t cutoff;
  uint32_t* dbits;            // [ceil(P/32)]
  uint32_t* cbits;            // [ceil(P/32)] or nullptr
  uint32_t* vbits;            // [ceil(P/32)] or nullptr: pods vetoed by the power clause (this rank's pods)
  unsigned long long* counts; // [3] n_series, n_candidates, n_decisions of this call (host-mapped slot
                              //     or device memory); written once by the last fold CTA
  unsigned long long* acc;    // [3] device accumulator of the fold grid, zero between calls
  unsigned int* ticket;       // self-resetting arrival counter of the fold grid
  unsigned long long* done;   // folds completed on this scratch set (monotonic)
  unsigned long long need;    // value of *done required before this decision may touch the set
  const unsigned long long* prev_done;  // the other scratch set's counter ...
  unsigned long long prev_need;         // ... and the value it must have reached (previous decision
                                        // folded) before this fold may write the caller's outputs
  uint32_t P, G;
  uint32_t mw;                // mask words per pod = ceil(G / 32)
  // ---- fused bitmap exchange over NVLink peer memory (world > 1, gpr_p2p_*) -------------------
  // Instead of a separate collective launch, the folding CTA stores this rank's packed words
  // straight into every peer's gather buffer, raises a per-source step flag on each peer with
  // release.sys semantics, waits for the peers' flags, and copies the assembled global bitmap to
  // the caller's buffers.  peer_gather[r] / peer_flag[r] are peer-mapped (CUDA IPC) addresses.
  int world, rank;                       // world <= 1: no exchange
  uint32_t rank_stride;                  // words per rank slot in a gather buffer (2 * W_max)
  uint32_t* peer_gather[kMaxPeers];      // gather buffer (this call's parity) on rank r
  unsigned long long* peer_flag[kMaxPeers];  // &flags[my_rank] on rank r
  const unsigned long long* my_flags;    // local flags[world], written by the peers
  unsigned long long step;               // exchange sequence number of this call (same on all ranks)
  uint32_t* out_dbits;                   // caller's global bitmaps on this device (may be null)
  uint32_t* out_cbits;
  int exchange_debug;                    // 0 normal; timing switches (gpr_p2p_debug): 1 = do not wait for the
                                         // peers, 2 = no push at all (results are then NOT global)
  unsigned long long* stamp;             // host-mapped [5]: %globaltimer (ns) when this decision completed, then
                                         // fold start / folded / flags raised / peers arrived (exchange phases)
  unsigned int* err;                     // host-mapped: set to 1 when a peer never showed up (see spin_until)
  unsigned int poll_ns;                  // longest pause between two polls of the peers' flags
  // tagged-slot form of the exchange (GPR_EXCHANGE=ll): every word travels as one 64-bit store {step tag, word} into
  // the receiver's slot array, so there is no fence and no flag — a slot is valid when its tag says so
  unsigned long long* peer_ll[kMaxPeers];  // slot array (this call's parity) on rank r; null = flag protocol
  unsigned long long* my_ll;               // local slot array (this call's parity)
  // 1 (tagged slots only): this fold's words are produced, sent and collected without waiting for the previous
  // decision's fold; only the CTA that assembles the caller's outputs waits for it.  The peers' wait — the long part
  // of an exchange — then overlaps with the predecessor's instead of queueing behind it.  Safe because the exchange
  // buffers are 2 x (scratch sets) deep: my push of step n + 4 follows my fold n + 2 (its scratch set is reused by
  // reduce n + 4), which saw every peer's step n + 2 words, which a peer sends only after its reduce n + 2 ran, which
  // waited for that peer's fold n — so nobody still polls for step n when its slots are overwritten.
  int late_order;
  uint32_t* islots;                      // [P][mw] or nullptr: gpr_result.idle_slots, each pod's idle words before
                                         // the fold clears them (this rank's pods)
};

// One rank's view of the exchange block header, for the stand-alone rendezvous (gpr_timer_begin)
struct RendezvousParams {
  int world, rank;
  unsigned long long* peer_flag[kMaxPeers];  // &rdv_flags[my_rank] on rank r
  const unsigned long long* my_flags;        // local rdv_flags[world]
  unsigned long long seq;
  unsigned long long* stamp;                 // host-mapped, %globaltimer at release
  unsigned int* err;
};

struct ReduceParams {
  Segment seg[2];
  uint64_t ld;        // elements between rows
  uint32_t T;
  uint32_t G;         // rows per pod
  uint32_t mw;        // mask words per pod = ceil(G / 32)
  uint32_t total_rows;
  float thr;          // smallest f32 >= (double) power threshold
  const unsigned long long* done;  // scratch-set guard, see wait_scratch_free
  unsigned long long need;
  uint32_t util_u8;   // seg[0] rows are biased bytes (GPR_FMT_U8B), k_reduce_u8 only
  // group table (gpr_groups.cuh), or nullptr: bit g of word (local / G) * mw + g / 32 marks a util row of a `sum by`
  // group of two or more.  Such a row is read whole and its max goes to gmax[local] (seg[0].smax when that is set).
  const uint32_t* grouped;
  float* gmax;
};

__device__ __forceinline__ unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
#ifdef GPR_TIMELINE
// developer-only: per-CTA (smid, t_start, t_stream_end, t_exit) in ns, see tools/timeline.py
__device__ unsigned long long g_timeline[4 * 4096];
__device__ __forceinline__ void tl_mark(int slot) {
  if (threadIdx.x == 0 && blockIdx.x < 4096) {
    if (slot == 0) {
      unsigned int smid;
      asm volatile("mov.u32 %0, %smid;" : "=r"(smid));
      g_timeline[4 * blockIdx.x] = smid;
    }
    g_timeline[4 * blockIdx.x + 1 + slot] = gtime();
  }
}
#define TL_MARK(slot) tl_mark(slot)
#else
#define TL_MARK(slot)
#endif

// ---- programmatic dependent launch (back-to-back decisions on the context's own stream) -------
// Stream order of successive decisions: R0 F0 R1 F1 R2 ...  (R = reduce grid, F = fold grid).
// Every kernel executes launch_dependents at entry, so its successor may become resident as soon
// as SM resources allow: F_n sits in griddepcontrol.wait until R_n has completed; R_{n+1} streams
// its input while F_n folds / exchanges.  Decisions alternate between two scratch sets (masks,
// ticket, accumulator); R_{n+2} checks the set's `done` counter (F_n finished) before its first
// mask update, and F_{n+1} checks the other set's counter (F_n finished) before it writes the
// caller's outputs.
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait_prior_grids() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// poll with relaxed loads, order with one fence at the end (an acquire per poll costs an L1 invalidate each time)
__device__ __forceinline__ void spin_until_gpu(const unsigned long long* p, unsigned long long want) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  while (v < want) {
    __nanosleep(64);
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  }
  asm volatile("fence.acq_rel.gpu;" ::: "memory");
}
__device__ __forceinline__ void st_release_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Wait for a peer-written sequence number.  A peer that never arrives (crashed rank, a rank that
// skipped a collective call) must not hang this GPU: after kPeerTimeoutNs the wait gives up, raises
// the host-visible error word (gpr_sync then fails with GPR_E_STATE) and the kernel runs to completion.
constexpr unsigned long long kPeerTimeoutNs = 20ull * 1000 * 1000 * 1000;
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// Polls with RELAXED loads, fences once when the value has arrived, and polls RARELY: the CTA that waits shares
// the chip with the next decision's reduce kernel, and every system-scope poll of a peer-written line costs that
// kernel bandwidth, and the more often it polls the more it costs.  The
// exchange has a whole step of slack before anything depends on it, so a late wake-up is free.
__device__ __forceinline__ void spin_until_sys(const unsigned long long* p, unsigned long long want,
                                               unsigned int* err, unsigned int poll_ns) {
  if (ld_relaxed_sys_u64(p) < want) {
    const unsigned long long t0 = gtime();
    unsigned int polls = 0, sleep_ns = 200;
    while (true) {
      __nanosleep(sleep_ns);
      if (ld_relaxed_sys_u64(p) >= want) break;
      if (sleep_ns < poll_ns) sleep_ns = min(poll_ns, sleep_ns * 2);
      if ((++polls & 255u) == 0 && gtime() - t0 > kPeerTimeoutNs) {
        if (err) *err = 1u;
        return;
      }
    }
  }
  asm volatile("fence.acq_rel.sys;" ::: "memory");  // the peer's words are ordered before its flag
}

__device__ __forceinline__ float nan_f() { return __int_as_float(0x7fffffff); }

// PTX max.f32: if exactly one operand is NaN the other is returned; NaN only if both are.
// Folding from NaN therefore reproduces Prometheus' max_over_time on the present samples.
// Built without -use_fast_math / -ftz so denormals are compared, not flushed (K7).
__device__ __forceinline__ float fold4(float m, const float4& v) {
  return fmaxf(fmaxf(fmaxf(m, v.x), fmaxf(v.y, v.z)), v.w);
}

__device__ __forceinline__ float warp_max(float m) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  return m;
}

// streaming 128-bit load: read-only path, do not allocate in L1 (every byte is used once)
__device__ __forceinline__ float4 ldg_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

// ------------------------------------------------------------------------------------------
// fold: flags -> verdict bits.  One lane per pod, one warp per bitmap word.
// ------------------------------------------------------------------------------------------
// Loads of a batch are unconditional (addresses clamped) and nothing consumes them until the
// whole batch is in flight: the fold is a pure latency chain, so a dependent use inside the load
// loop would serialise BATCH round trips to L2.
template <int BATCH>
__device__ __forceinline__ void fold_words(const FoldParams& f, uint32_t w_begin, uint32_t w_end,
                                           uint32_t w_step, int lane, unsigned long long& n_series,
                                           unsigned long long& n_cand, unsigned long long& n_dec) {
  const uint32_t last_pod = f.P - 1u;  // callers guarantee P > 0
  bool waited = false;  // (the CTA-wide barrier below: every warp passes it exactly once, see the end)
  for (uint32_t w0 = w_begin; w0 < w_end; w0 += w_step * BATCH) {
    uint32_t idle[BATCH], veto[BATCH];
    uint8_t elig[BATCH];
    long long created[BATCH];
#pragma unroll
    uint32_t n_idle[BATCH];
    for (int b = 0; b < BATCH; ++b) {
      const uint32_t pod = min((w0 + b * w_step) * 32u + lane, last_pod);
      idle[b] = __ldcg(f.idle_mask + (size_t)pod * f.mw);
      veto[b] = f.veto_mask ? __ldcg(f.veto_mask + (size_t)pod * f.mw) : 0u;
      n_idle[b] = __popc(idle[b]);
      for (uint32_t k = 1; k < f.mw; ++k) {  // pods with more than 32 series slots: further mask words
        const uint32_t x = __ldcg(f.idle_mask + (size_t)pod * f.mw + k);
        idle[b] |= x, n_idle[b] += __popc(x);
        if (f.veto_mask) veto[b] |= __ldcg(f.veto_mask + (size_t)pod * f.mw + k);
      }
      elig[b] = f.eligible ? f.eligible[pod] : (uint8_t)1;
      created[b] = f.created ? f.created[pod] : (long long)0x8000000000000000ll;
    }
    if (!waited) {
      // The caller's output buffers may still be written by the previous decision's fold.  That wait comes AFTER
      // the loads above are in flight: while the next reduce kernel streams, every trip to L2 costs microseconds.
      // (late_order: nothing written here is the caller's — the assembling CTA waits instead, see k_fold)
      if (threadIdx.x == 0 && !f.late_order) spin_until_gpu(f.prev_done, f.prev_need);
      __syncthreads();
      waited = true;
    }
#pragma unroll
    for (int b = 0; b < BATCH; ++b) {
      const uint32_t w = w0 + b * w_step;
      if (w >= w_end) break;  // warp-uniform
      const uint32_t pod = w * 32u + lane;
      const bool valid = pod < f.P;
      const bool cand = valid && idle[b] != 0u && veto[b] == 0u;
      const bool dec = cand && elig[b] != 0 && !(f.created && created[b] >= f.cutoff);
      const uint32_t cw = __ballot_sync(0xffffffffu, cand);
      const uint32_t dw = __ballot_sync(0xffffffffu, dec);
      const uint32_t vw = __ballot_sync(0xffffffffu, valid && veto[b] != 0u);
      uint32_t ns = cand ? n_idle[b] : 0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ns += __shfl_xor_sync(0xffffffffu, ns, o);
      if (valid) {  // leave the scratch zeroed for the next call
        for (uint32_t k = 0; k < f.mw; ++k) {
          if (idle[b]) f.idle_mask[(size_t)pod * f.mw + k] = 0u;
          if (veto[b]) f.veto_mask[(size_t)pod * f.mw + k] = 0u;
        }
      }
      if (f.my_ll && f.exchange_debug != 2) {
        // tagged-slot exchange: the word leaves for every peer the moment it exists — lane 2 i sends the decision
        // word to the i-th peer, lane 2 i + 1 the candidate word (one 64-bit NVLink store each, no fence, no flag)
        const int peer = lane >> 1, r = peer + (peer >= f.rank ? 1 : 0);
        if (peer < f.world - 1) {
          const unsigned long long v = ((f.step & 0xffffffffull) << 32) | (unsigned long long)((lane & 1) ? cw : dw);
          unsigned long long* dst = f.peer_ll[r] + (size_t)f.rank * f.rank_stride + ((lane & 1) ? (f.P + 31u) / 32u : 0u) + w;
          asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(dst), "l"(v) : "memory");
        }
      }
      if (lane == 0) {
        f.dbits[w] = dw;
        if (f.cbits) f.cbits[w] = cw;
        if (f.vbits) f.vbits[w] = vw;
        n_series += ns;
        n_cand += __popc(cw);
        n_dec += __popc(dw);
      }
    }
  }
  if (!waited) {  // a warp without a word of its own still takes part in the barrier
    if (threadIdx.x == 0 && !f.late_order) spin_until_gpu(f.prev_done, f.prev_need);
    __syncthreads();
  }
}

// block-level sum of the three counters into fold.counts (call from all threads)
__device__ __forceinline__ void block_counts(unsigned long long* sh3, unsigned long long a,
                                             unsigned long long b, unsigned long long c, int lane) {
  if (lane == 0 && (a | b | c)) {
    atomicAdd(&sh3[0], a);
    atomicAdd(&sh3[1], b);
    atomicAdd(&sh3[2], c);
  }
}

// The one exchange of the multi-GPU path, fused into the folding CTA.  f.dbits / f.cbits point at
// this rank's slot of the LOCAL gather buffer; the same 2*W words are pushed to every peer.
// `mine` = this rank's 2 * n_words words [decision | candidate]: its slot of the local gather buffer, or the
// copy the single-CTA fold keeps in shared memory (no second trip to L2 before the push)
__device__ __forceinline__ void exchange_bitmaps(const FoldParams& f, uint32_t n_words, const uint32_t* mine) {
  __syncthreads();  // the fold's word stores are visible to the whole CTA
  const uint32_t span = 2u * n_words;  // [decision | candidate], candidate slot always present
  // each word is read once and fanned out to every peer (a per-peer reload would put world-1
  // dependent L2 round trips per word on this CTA's critical path)
  for (uint32_t w0 = threadIdx.x; w0 < span && f.exchange_debug != 2; w0 += 4u * blockDim.x) {
    uint32_t v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t w = w0 + k * blockDim.x;
      v[k] = w < span ? mine[w] : 0u;
    }
    for (int r = 0; r < f.world; ++r) {
      if (r == f.rank) continue;
      uint32_t* dst = f.peer_gather[r] + (size_t)f.rank * f.rank_stride;   // NVLink peer stores
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t w = w0 + k * blockDim.x;
        if (w < span) dst[w] = v[k];
      }
    }
  }
  // bar.sync orders every thread's peer stores before the flag threads' release (the release is
  // cumulative at system scope), so one fence per peer instead of one per thread
  __syncthreads();
  if ((int)threadIdx.x < f.world && (int)threadIdx.x != f.rank && f.exchange_debug != 2) {
    st_release_sys_u64(f.peer_flag[threadIdx.x], f.step);             // "rank's words of step k are there"
    if (f.stamp && threadIdx.x == (f.rank == 0 ? 1u : 0u)) f.stamp[3] = gtime();   // flags raised (fence included)
    if (f.exchange_debug == 0) spin_until_sys(f.my_flags + threadIdx.x, f.step, f.err, f.poll_ns);
  }
  __syncthreads();
  if (threadIdx.x == 0 && f.stamp) f.stamp[4] = gtime();             // every peer's words have arrived
  // assemble the caller's rank-major global bitmaps from the local gather buffer
  if (f.out_dbits) {
    const uint32_t* g = f.peer_gather[f.rank];
    for (uint32_t i = threadIdx.x; i < n_words * (uint32_t)f.world; i += blockDim.x) {
      const uint32_t r = i / n_words, w = i - r * n_words;
      f.out_dbits[i] = __ldcg(g + (size_t)r * f.rank_stride + w);
      if (f.out_cbits) f.out_cbits[i] = __ldcg(g + (size_t)r * f.rank_stride + n_words + w);
    }
  }
}

// Tagged-slot form of the same exchange: no system-scope fence on the sender (under load the fence has to wait for
// the acknowledgements of stores into seven busy GPUs), no flags, and no funnel through the last CTA on the sending
// side: every fold CTA sends its words as it produces them (fold_words); here the last CTA only reads every peer's
// slots until their tags match and assembles the result.
constexpr int kCollectBatch = 16;   // slots per thread and polling round (8 ranks x 10,000 pods: 20 per thread, two rounds)
constexpr int kAssembleBatch = 8;   // output words per thread and round (same case: 10 per thread)
__device__ __forceinline__ void exchange_bitmaps_ll(const FoldParams& f, uint32_t n_words, const uint32_t* mine) {
  __syncthreads();  // the fold's word stores are visible to the whole CTA
  uint32_t* g = f.peer_gather[f.rank];  // local gather buffer: [rank][decision | candidate]
  const uint32_t span = 2u * n_words;
  const unsigned long long tag = (f.step & 0xffffffffull) << 32;
  (void)mine;  // every fold CTA has already sent its own words (fold_words)
  if (threadIdx.x == 0 && f.stamp) f.stamp[3] = gtime();
  if (f.exchange_debug == 0) {
    // Every slot of every peer.  All loads of a round are in flight before the first one is looked at: while the
    // next reduce kernel streams, a dependent trip to L2 is slow, and a load-compare-store chain per slot (20
    // slots per thread at 8 ranks and 10,000 pods) would serialise those trips.
    const uint32_t total = (uint32_t)f.world * span;
    const unsigned long long t0 = gtime();
    for (uint32_t i0 = threadIdx.x; i0 < total; i0 += (uint32_t)kCollectBatch * blockDim.x) {
      unsigned int pending = 0;
      uint32_t off[kCollectBatch];  // r * rank_stride + w (< 2^32: at most 8 ranks x 2^28 words)
#pragma unroll
      for (int k = 0; k < kCollectBatch; ++k) {
        const uint32_t i = i0 + (uint32_t)k * blockDim.x;
        const uint32_t r = i / span, w = i - r * span;
        off[k] = r * f.rank_stride + w;
        if (i < total && (int)r != f.rank) pending |= 1u << k;
      }
      unsigned int polls = 0;
      while (pending) {
        unsigned long long v[kCollectBatch];
#pragma unroll
        for (int k = 0; k < kCollectBatch; ++k)
          v[k] = (pending >> k & 1u) ? ld_relaxed_sys_u64(f.my_ll + off[k]) : 0ull;
#pragma unroll
        for (int k = 0; k < kCollectBatch; ++k) {
          if ((pending >> k & 1u) && (v[k] >> 32) == (tag >> 32)) {
            g[off[k]] = (uint32_t)v[k];   // the local gather buffer holds every rank's words again
            pending &= ~(1u << k);
          }
        }
        if (pending) {
          __nanosleep(100);
          if ((++polls & 1023u) == 0 && gtime() - t0 > kPeerTimeoutNs) {
            if (f.err) *f.err = 1u;
            break;
          }
        }
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (f.stamp) f.stamp[4] = gtime();
    // the caller's buffers belong to the previous decision until its fold has finished
    if (f.late_order) spin_until_gpu(f.prev_done, f.prev_need);
  }
  __syncthreads();
  if (f.out_dbits) {
    // same rule for the copy into the caller's rank-major bitmaps: loads first, then stores
    const uint32_t n_out = n_words * (uint32_t)f.world;
    for (uint32_t i0 = threadIdx.x; i0 < n_out; i0 += (uint32_t)kAssembleBatch * blockDim.x) {
      uint32_t d[kAssembleBatch], c[kAssembleBatch];
#pragma unroll
      for (int k = 0; k < kAssembleBatch; ++k) {
        const uint32_t i = i0 + (uint32_t)k * blockDim.x;
        d[k] = c[k] = 0u;
        if (i < n_out) {
          const uint32_t r = i / n_words, w = i - r * n_words;
          d[k] = g[(size_t)r * f.rank_stride + w];
          if (f.out_cbits) c[k] = g[(size_t)r * f.rank_stride + n_words + w];
        }
      }
#pragma unroll
      for (int k = 0; k < kAssembleBatch; ++k) {
        const uint32_t i = i0 + (uint32_t)k * blockDim.x;
        if (i < n_out) {
          f.out_dbits[i] = d[k];
          if (f.out_cbits) f.out_cbits[i] = c[k];
        }
      }
    }
  }
}

// The fold kernel.  Launched right behind the reduce kernel with the programmatic-stream-
// serialization attribute: its CTAs become resident while the reduce grid is still streaming, park
// in griddepcontrol.wait (no polling) and run the moment the reduce grid has completed and its
// mask updates are visible.  Grid = a handful of CTAs (32 words each); the last one to finish
// (ticket) performs the multi-GPU exchange, publishes the counters and releases the scratch set.
// kExchange = false is the single-GPU instantiation: the exchange (and the registers its batched loads need) is
// compiled out, so that path is the same code as before the exchange existed.  kSlots: the call asked for
// gpr_result.idle_slots (f.islots); without it that copy is compiled out too.
template <bool kExchange, bool kSlots = false>
__global__ void __launch_bounds__(256) k_fold(FoldParams f) {
  __shared__ unsigned long long s_cnt[3];
  __shared__ unsigned int s_last;
  pdl_launch_dependents();   // the next decision's reduce kernel may start streaming right away
  if (threadIdx.x == 0) s_cnt[0] = s_cnt[1] = s_cnt[2] = 0;
  pdl_wait_prior_grids();    // reduce grid of THIS decision complete, masks visible
  const unsigned long long t_start = gtime();
  const int lane = threadIdx.x & 31;
  const uint32_t warps_per_cta = blockDim.x >> 5;
  const uint32_t gw = blockIdx.x * warps_per_cta + (threadIdx.x >> 5);
  const uint32_t n_words = (f.P + 31u) / 32u;
  unsigned long long a = 0, b = 0, c = 0;
  if (kSlots) {
    // each pod's idle words as they are (idle elements, before veto and gates), read by the warp that clears them
    // in fold_words below: the same words in the same order.  idle_slots is the caller's buffer, like the bitmaps:
    // the previous decision's fold may still be writing it, so the copy waits for that fold first (a call with
    // idle_slots never takes the late output ordering).
    if (threadIdx.x == 0) spin_until_gpu(f.prev_done, f.prev_need);
    __syncthreads();
    for (uint32_t w = gw; w < n_words; w += gridDim.x * warps_per_cta) {
      const uint32_t pod = w * 32u + (uint32_t)lane;
      if (pod < f.P)
        for (uint32_t k = 0; k < f.mw; ++k)
          f.islots[(size_t)pod * f.mw + k] = __ldcg(f.idle_mask + (size_t)pod * f.mw + k);
    }
  }
  fold_words<4>(f, gw, n_words, gridDim.x * warps_per_cta, lane, a, b, c);
  block_counts(s_cnt, a, b, c, lane);
  __syncthreads();  // (thread 0's fence below is cumulative over what the CTA stored before this barrier)
  if (threadIdx.x == 0) {
    if (s_cnt[0] | s_cnt[1] | s_cnt[2]) {
      atomicAdd(&f.acc[0], s_cnt[0]);
      atomicAdd(&f.acc[1], s_cnt[1]);
      atomicAdd(&f.acc[2], s_cnt[2]);
    }
    __threadfence();
    s_last = (atomicAdd(f.ticket, 1u) == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (threadIdx.x == 0 && f.stamp) f.stamp[1] = t_start, f.stamp[2] = gtime(), f.stamp[3] = f.stamp[4] = 0;
  if (kExchange && f.world > 1) {
    // (other CTAs wrote most of the words: read them at L2)
    const uint32_t* mine = f.peer_gather[f.rank] + (size_t)f.rank * f.rank_stride;
    if (f.my_ll) exchange_bitmaps_ll(f, n_words, mine);
    else exchange_bitmaps(f, n_words, mine);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    f.counts[0] = __ldcg(&f.acc[0]);
    f.counts[1] = __ldcg(&f.acc[1]);
    f.counts[2] = __ldcg(&f.acc[2]);
    f.acc[0] = f.acc[1] = f.acc[2] = 0ull;
    *f.ticket = 0u;
    if (f.stamp) *f.stamp = gtime();
    __threadfence();
    st_release_u64(f.done, f.need + 1ull);
  }
}

// Device-side rendezvous + time mark (gpr_timer_begin).  With an exchange attached every rank raises
// its sequence number on every peer and waits for theirs, so the kernels that follow on each rank's
// stream start within an NVLink round trip of each other instead of a host-launch skew apart.
__global__ void __launch_bounds__(32) k_rendezvous(RendezvousParams q) {
  const int t = threadIdx.x;
  if (t < q.world && t != q.rank) {
    st_release_sys_u64(q.peer_flag[t], q.seq);
    spin_until_sys(q.my_flags + t, q.seq, q.err, 200u);  // the rendezvous wants a prompt release
  }
  __syncwarp();
  if (t == 0 && q.stamp) *q.stamp = gtime();
}

// ------------------------------------------------------------------------------------------
// shared row bookkeeping
// ------------------------------------------------------------------------------------------
// (kernel parameters live in constant memory: select fields with ?: — a runtime index into
// p.seg[] would force a stack copy of the whole struct)
__device__ __forceinline__ const float* row_ptr(const ReduceParams& p, uint32_t r, uint32_t& seg,
                                                uint32_t& local) {
  const uint32_t n0 = p.seg[0].n_rows;
  seg = r >= n0 ? 1u : 0u;
  local = r - (seg ? n0 : 0u);
  const float* base = seg ? p.seg[1].base : p.seg[0].base;
  return base + (size_t)local * p.ld;
}

// rows owned by this CTA under the strided assignment row = blockIdx.x + j * gridDim.x.  In 64 bits: with a power
// plane total_rows reaches 2^32 - 2, and adding gridDim.x - 1 to it would wrap.
__device__ __forceinline__ uint32_t cta_row_count(uint32_t total_rows) {
  return total_rows > blockIdx.x
             ? (uint32_t)(((uint64_t)total_rows - blockIdx.x + gridDim.x - 1) / gridDim.x)
             : 0u;
}

// before a warp's first publish: the decision that last used this scratch set must have folded
__device__ __forceinline__ void wait_scratch_free(const ReduceParams& p) { spin_until_gpu(p.done, p.need); }

// a util row of a `sum by` group of two or more (ReduceParams.grouped); without a table a uniform false
__device__ __forceinline__ bool row_grouped(const ReduceParams& p, uint32_t seg, uint32_t local) {
  if (p.grouped == nullptr || seg != 0u) return false;
  const uint32_t g = local % p.G;
  return (p.grouped[(size_t)(local / p.G) * p.mw + (g >> 5)] >> (g & 31u)) & 1u;
}

__device__ __forceinline__ void publish_row(const ReduceParams& p, uint32_t seg, uint32_t local,
                                            float m, bool grouped) {
  const bool is_power = seg ? p.seg[1].is_power != 0 : p.seg[0].is_power != 0;
  uint32_t* mask = seg ? p.seg[1].mask : p.seg[0].mask;
  float* smax = seg ? p.seg[1].smax : p.seg[0].smax;
  // util: `== 0` (NaN fails, -0.0 passes); power: `>= T` (NaN fails)
  const bool flag = is_power ? (m >= p.thr) : (m == 0.0f);
  // fire-and-forget RED at L2; unflagged rows write nothing at all
  if (flag) {
    const uint32_t g = local % p.G;
    atomicOr(mask + (size_t)(local / p.G) * p.mw + (g >> 5), 1u << (g & 31u));
  }
  if (smax) smax[local] = m;
  else if (grouped) p.gmax[local] = m;   // the group sum (k_group_sum) reads it
}

// ------------------------------------------------------------------------------------------
// early exit
// ------------------------------------------------------------------------------------------
// The verdict needs two yes/no answers, not the max: util `max == 0`, power `max >= thr`.  A max
// over part of a row settles its flag once it is > 0 (util: not idle, whatever follows) or >= thr
// (power: vetoed); NaN, zeros and negatives settle nothing, a denormal positive does (no ftz, K7).
// A row may stop being read at the first read sample that settles it, unless the call asks for
// series_max: the true max is an output then, and every row is read in full.  An idle row — the
// only kind n_series counts — is always read to its end, so every output is what a full read gives.
// A row of a `sum by` group of two or more (row_grouped) is read in full too: its max is summed.
__device__ __forceinline__ bool settles(float m, bool is_power, float thr) {
  return is_power ? m >= thr : m > 0.0f;
}
__device__ __forceinline__ bool rows_may_stop(const ReduceParams& p) {
  return p.seg[0].smax == nullptr && p.seg[1].smax == nullptr;
}

// ------------------------------------------------------------------------------------------
// reduce, variant 1: vectorised streaming loads
// ------------------------------------------------------------------------------------------
// One warp per series row; rows of a CTA's contiguous range are handed out through a
// shared-memory counter so the SM stays busy until its range is exhausted.  Any base
// alignment / T / stride is accepted: a scalar peel to 16-byte alignment, a float4 body, a
// scalar tail.  With `stop`, the peel plus the body's first 16-byte load per lane is the row's
// head; after it and after every batch of U loads the warp leaves once a lane has seen a
// sample that settles the row (nothing is loaded ahead of that test).
template <int U>
__device__ __forceinline__ float row_max_ldg(const float* __restrict__ row, uint32_t T, int lane, bool stop,
                                             bool is_power, float thr) {
  float m = nan_f();
  const uintptr_t a = reinterpret_cast<uintptr_t>(row);
  uint32_t head = (uint32_t)(((16u - (a & 15u)) & 15u) >> 2);
  if (head > T) head = T;
  if ((uint32_t)lane < head) m = __ldg(row + lane);
  const float4* __restrict__ v = reinterpret_cast<const float4*>(row + head);
  const uint32_t nv = (T - head) >> 2;
  uint32_t b = 0;  // first float4 of the warp's next batch (warp-uniform: the tests below are warp-wide)
  if (stop) {
    if ((uint32_t)lane < nv) m = fold4(m, ldg_stream(v + lane));
    b = 32u;
    if (__ballot_sync(0xffffffffu, settles(m, is_power, thr))) return warp_max(m);
  }
  // full batches: U independent 16-byte loads per lane in flight
  for (; b + 32u * U <= nv; b += 32u * U) {
    float4 x[U];
#pragma unroll
    for (int j = 0; j < U; ++j) x[j] = ldg_stream(v + b + lane + 32u * j);
#pragma unroll
    for (int j = 0; j < U; ++j) m = fold4(m, x[j]);
    if (stop && __ballot_sync(0xffffffffu, settles(m, is_power, thr))) return warp_max(m);
  }
  // one predicated batch for the remainder
  if (b < nv) {
    float4 x[U];
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint32_t k = b + lane + 32u * j;
      x[j] = make_float4(nan_f(), nan_f(), nan_f(), nan_f());
      if (k < nv) x[j] = ldg_stream(v + k);
    }
#pragma unroll
    for (int j = 0; j < U; ++j) m = fold4(m, x[j]);
    if (stop && __ballot_sync(0xffffffffu, settles(m, is_power, thr))) return warp_max(m);
  }
  const uint32_t done = head + nv * 4u;
  if (done + lane < T) m = fmaxf(m, __ldg(row + done + lane));
  return warp_max(m);
}

// kGroups: the instantiation for calls with a group table (ReduceParams.grouped); without one the kernel is compiled
// without the per-row test, so the ungrouped path is the same code as before tables existed.
template <int WARPS, int U, bool kGroups = false>
__global__ void __launch_bounds__(WARPS * 32) k_reduce_ldg(ReduceParams p) {
  __shared__ unsigned int s_next;
  const int lane = threadIdx.x & 31;
  const uint32_t warp = threadIdx.x >> 5;
  // CTA b owns rows b, b + grid, b + 2*grid, ...: at any instant the whole chip streams one
  // narrow, advancing band of the tensor (sequential DRAM pages, few live TLB entries) and every
  // CTA's share differs by at most one row.
  TL_MARK(0);
  pdl_launch_dependents();
  const uint32_t n_mine = cta_row_count(p.total_rows);
  const bool stop = rows_may_stop(p);
  if (threadIdx.x == 0) s_next = WARPS;
  __syncthreads();
  uint32_t j = warp;
  bool scratch_ok = false;
  while (j < n_mine) {
    uint32_t seg, local;
    const float* row = row_ptr(p, blockIdx.x + j * gridDim.x, seg, local);
    const bool is_power = seg ? p.seg[1].is_power != 0 : p.seg[0].is_power != 0;
    const bool grouped = kGroups && row_grouped(p, seg, local);
    const float m = row_max_ldg<U>(row, p.T, lane, stop && !grouped, is_power, p.thr);
    if (lane == 0) {
      if (!scratch_ok) wait_scratch_free(p), scratch_ok = true;
      publish_row(p, seg, local, m, grouped);
      j = atomicAdd(&s_next, 1u);
    }
    j = __shfl_sync(0xffffffffu, j, 0);
  }
  TL_MARK(1);
  TL_MARK(2);
}

// ------------------------------------------------------------------------------------------
// reduce over biased bytes (GPR_FMT_U8B): 0 = no sample, b = value b - 1
// ------------------------------------------------------------------------------------------
// Same question, one byte per sample.  With the bias the whole row folds with OR: the window max
// is 0 exactly when the OR of every byte of the row is 0x01 (some sample present, none above 0),
// and no sample is present when it is 0x00 - one LOP3 per 8 bytes, so the kernel stays bound by
// memory, not by emulated byte-SIMD max.  The true maximum (series_max) is only folded when the
// caller asked for it.  Rows may start at any byte: byte head to 16-byte alignment, 128-bit
// body, byte tail; absent (0) is the identity of both OR and max, so predicated-off loads are 0.
__device__ __forceinline__ uint4 ldg_stream_u4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// returns the window max as the f32 the other kernels would have produced (NaN = no sample);
// without want_max any positive maximum is reported as 1.0f (only `== 0` is consumed)
template <int U>
__device__ __forceinline__ float row_max_u8(const uint8_t* __restrict__ row, uint32_t T, int lane,
                                            bool want_max) {
  uint32_t acc = 0, m4 = 0;
  const uintptr_t a = reinterpret_cast<uintptr_t>(row);
  uint32_t head = (uint32_t)((16u - (a & 15u)) & 15u);
  if (head > T) head = T;
  uint32_t hb = 0, tb = 0;  // one head byte and one tail byte per lane (at most 15 of each)
  if ((uint32_t)lane < head) hb = __ldg(row + lane);
  const uint4* __restrict__ v = reinterpret_cast<const uint4*>(row + head);
  const uint32_t nv = (T - head) >> 4;
  for (uint32_t i = lane; i < nv; i += 32u * U) {
    uint4 x[U];
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint32_t k = i + 32u * j;
      x[j] = make_uint4(0u, 0u, 0u, 0u);
      if (k < nv) x[j] = ldg_stream_u4(v + k);
    }
#pragma unroll
    for (int j = 0; j < U; ++j) {
      acc |= (x[j].x | x[j].y) | (x[j].z | x[j].w);
      if (want_max) m4 = __vmaxu4(__vmaxu4(m4, x[j].x), __vmaxu4(__vmaxu4(x[j].y, x[j].z), x[j].w));
    }
  }
  const uint32_t done = head + nv * 16u;
  if (done + lane < T) tb = __ldg(row + done + lane);
  acc |= hb | tb;
  acc |= acc >> 16;
  acc |= acc >> 8;
  acc = __reduce_or_sync(0xffffffffu, acc & 0xffu);
  if (acc == 0u) return nan_f();   // no sample in the window
  if (acc == 1u) return 0.0f;      // samples present, none above 0
  if (!want_max) return 1.0f;
  m4 = __vmaxu4(m4, max(hb, tb));  // head / tail bytes are plain values: byte lane 0
  uint32_t m = max(max(m4 & 0xffu, (m4 >> 8) & 0xffu), max((m4 >> 16) & 0xffu, m4 >> 24));
  m = __reduce_max_sync(0xffffffffu, m);
  return (float)(m - 1u);
}

template <int WARPS, int U, bool kGroups = false>
__global__ void __launch_bounds__(WARPS * 32) k_reduce_u8(ReduceParams p) {
  __shared__ unsigned int s_next;
  const int lane = threadIdx.x & 31;
  const uint32_t warp = threadIdx.x >> 5;
  pdl_launch_dependents();
  const uint32_t n_mine = cta_row_count(p.total_rows);
  if (threadIdx.x == 0) s_next = WARPS;
  __syncthreads();
  uint32_t j = warp;
  bool scratch_ok = false;
  while (j < n_mine) {
    uint32_t seg, local;
    const float* frow = row_ptr(p, blockIdx.x + j * gridDim.x, seg, local);
    float m;
    const bool grouped = kGroups && row_grouped(p, seg, local);
    if (seg == 0u && p.util_u8) {
      const uint8_t* row = reinterpret_cast<const uint8_t*>(p.seg[0].base) + (size_t)local * p.ld;
      m = row_max_u8<U>(row, p.T, lane, p.seg[0].smax != nullptr || grouped);
    } else {
      m = row_max_ldg<U>(frow, p.T, lane, false, false, 0.0f);   // (byte-window calls read every row whole)
    }
    if (lane == 0) {
      if (!scratch_ok) wait_scratch_free(p), scratch_ok = true;
      publish_row(p, seg, local, m, grouped);
      j = atomicAdd(&s_next, 1u);
    }
    j = __shfl_sync(0xffffffffu, j, 0);
  }
}

// ------------------------------------------------------------------------------------------
// reduce, variant 2: TMA bulk copies into a shared-memory ring
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D bulk async copy global -> shared, completion counted in bytes on an mbarrier.
// The data is read exactly once: L2 evict_first keeps it from displacing anything useful.
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                            uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

// The ring layout, chosen on the host by gpr_launch.h's tma_layout.  The same definition is in gpr_launch.h; the guard
// keeps whichever comes first, so that this header's namespace body also stands alone (the CPU emulation of the
// kernels compiles it without the host header).
#ifndef GPR_TMA_LAYOUT_DEFINED
#define GPR_TMA_LAYOUT_DEFINED
struct TmaLayout {
  uint32_t depth;         // stages per warp = rows in flight per warp
  uint32_t stage_bytes;   // capacity of one stage (multiple of 128)
  uint32_t chunk_elems;   // elements copied per chunk (multiple of 4); a row read whole = n_chunks chunks
  uint32_t n_chunks;
  uint32_t head_elems;    // elements of a row's first copy when the row may stop early (multiple of 4, <= chunk_elems)
};
#endif

// Requirements (checked on the host): every row base 16-byte aligned, T % 4 == 0.
//
// Every warp runs its own TMA pipeline: a private ring of `depth` stages, each with one
// mbarrier, and each carrying one row with exactly one bulk copy in flight.  A row's copies are
// its head (elements [0, h)) and then chunks of chunk_elems: copy c >= 1 covers
// [h + (c - 1) chunk_elems, ...).  h = head_elems when rows may stop early, else chunk_elems (the
// row is then cut exactly as n_chunks chunks).  Lane 0 issues a 1-D bulk copy with the byte count
// expected on the stage's barrier; the warp visits the stages in ring order, waits for the bytes,
// folds them out of shared memory with conflict-free 128-bit LDS into the row's running max and,
// once every lane has finished reading, lane 0 re-arms the same stage: with the row's next chunk
// if the row is neither finished nor settled, else — after publishing the row — with the head of
// the next row the CTA hands out.  A copy is requested only after the row's previous copy has
// been examined, so the bytes a row costs depend on nothing but its data and the layout, and no
// copy is ever issued that would not be consumed.  No producer warp, no empty barriers: a stage
// is only ever touched by its owner warp, so the mbarrier phase parity cannot alias.
// The CTA owns rows b, b + grid, ... (see k_reduce_ldg); its first NW * depth rows start the
// stages, the rest are handed out through a counter behind the barriers in shared memory, since
// rows now cost anything from a head to a full read.
template <int NW, bool kGroups = false>
__global__ void __launch_bounds__(NW * 32) k_reduce_tma(ReduceParams p, TmaLayout L) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int lane = threadIdx.x & 31;
  const uint32_t w = threadIdx.x >> 5;
  const uint32_t D = L.depth;  // <= 32: lane s keeps the row state of stage s
  unsigned char* stage0 = smem + (size_t)w * D * L.stage_bytes;
  uint64_t* const bars = reinterpret_cast<uint64_t*>(smem + (size_t)NW * D * L.stage_bytes);
  uint64_t* full = bars + w * D;
  unsigned int* next_row = reinterpret_cast<unsigned int*>(bars + NW * D);

  pdl_launch_dependents();
  const uint32_t n_rows = cta_row_count(p.total_rows);
  const bool stop = rows_may_stop(p);
  const uint32_t h = stop ? L.head_elems : L.chunk_elems;
  bool scratch_ok = false;

  if (lane == 0) {
    for (uint32_t s = 0; s < D; ++s) mbar_init(&full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x == 0) *next_row = NW * D;
  __syncthreads();
  const uint64_t pol = l2_evict_first_policy();

  // copy c of the CTA's j-th row into stage s (called by every lane, acted on by lane 0)
  auto issue = [&](uint32_t s, uint32_t j, uint32_t c) {
    uint32_t seg, local;
    const float* row = row_ptr(p, blockIdx.x + j * gridDim.x, seg, local);
    const uint32_t e0 = c ? h + (c - 1u) * L.chunk_elems : 0u;
    const uint32_t bytes = min(c ? L.chunk_elems : h, p.T - e0) * 4u;
    if (lane == 0) {
      mbar_expect_tx(&full[s], bytes);
      tma_load_1d(stage0 + (size_t)s * L.stage_bytes, row + e0, bytes, &full[s], pol);
    }
  };
  // stage s's row (CTA-local index, >= n_rows: the stage is drained), its next copy and running max, kept by lane s
  uint32_t my_j = min(w + NW * (uint32_t)lane, n_rows), my_c = 0;
  float my_m = nan_f();
  uint32_t live = 0;
  for (uint32_t s = 0; s < D; ++s) {
    const uint32_t j = w + NW * s;
    if (j < n_rows) issue(s, j, 0u), ++live;
  }

  uint32_t phase = 0;  // bit s: parity of stage s's next completion
  for (uint32_t s = 0; live; s = s + 1u == D ? 0u : s + 1u) {
    uint32_t j = __shfl_sync(0xffffffffu, my_j, (int)s);
    if (j >= n_rows) continue;
    uint32_t c = __shfl_sync(0xffffffffu, my_c, (int)s);
    float m = __uint_as_float(__shfl_sync(0xffffffffu, __float_as_uint(my_m), (int)s));
    mbar_wait(&full[s], (phase >> s) & 1u);
    phase ^= 1u << s;
    const uint32_t e0 = c ? h + (c - 1u) * L.chunk_elems : 0u;
    const uint32_t n = min(c ? L.chunk_elems : h, p.T - e0);
    const float4* v = reinterpret_cast<const float4*>(stage0 + (size_t)s * L.stage_bytes);
    const uint32_t nv = n >> 2;
    float m0 = nan_f(), m1 = nan_f();
    uint32_t k = lane;
#pragma unroll 4
    for (; k + 32u < nv; k += 64u) {
      const float4 a = v[k], b = v[k + 32u];
      m0 = fold4(m0, a);
      m1 = fold4(m1, b);
    }
    if (k < nv) m0 = fold4(m0, v[k]);
    m = fmaxf(m, warp_max(fmaxf(m0, m1)));
    __syncwarp();  // every lane has its data in registers: the stage may be overwritten
    uint32_t seg, local;
    (void)row_ptr(p, blockIdx.x + j * gridDim.x, seg, local);
    const bool is_power = seg ? p.seg[1].is_power != 0 : p.seg[0].is_power != 0;
    if (e0 + n < p.T && !(stop && settles(m, is_power, p.thr) && !(kGroups && row_grouped(p, seg, local)))) {
      issue(s, j, ++c);
    } else {
      uint32_t next = 0;
      if (lane == 0) {
        if (!scratch_ok) wait_scratch_free(p), scratch_ok = true;
        publish_row(p, seg, local, m, kGroups && row_grouped(p, seg, local));
        next = atomicAdd(next_row, 1u);
      }
      j = min(__shfl_sync(0xffffffffu, next, 0), n_rows), c = 0, m = nan_f();
      if (j < n_rows) issue(s, j, 0u);
      else --live;
    }
    if ((uint32_t)lane == s) my_j = j, my_c = c, my_m = m;
  }
}

}  // namespace gpr
