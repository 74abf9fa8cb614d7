// gpr_launch.h — launch geometry of the decision kernels (host only, no CUDA).
//
// Which reduce kernel runs, with which grid, block, shared memory and TMA ring layout, and how large the fold grid
// is, as plain functions of the device's SM count, the tuning knobs gpr_create reads from the environment, the
// window's shape and its alignment.  gpr_api.cu launches exactly what these functions return; the CPU emulation of
// the kernels (tests/cpp/hotpath_emul.cpp) and the GPU tests use the same functions, so every geometry the library
// can pick is one the tests can reproduce.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <algorithm>

#include "../../include/gpr.h"

namespace gpr {

constexpr int kLdgWarps = 16;     // k_reduce_ldg / k_reduce_u8: warps per CTA
constexpr int kLdgUnroll = 8;     // k_reduce_ldg: 16-byte loads per lane in flight
constexpr int kU8Unroll = 4;      // k_reduce_u8: 16-byte loads per lane in flight
constexpr size_t kTmaSmemBudget = 208 * 1024;
// k_reduce_tma: samples in the first copy of a row (multiple of 4).  Most busy rows are settled by their first
// sample, so the head is all that is read of them; a row the head does not settle is read on in chunk_elems chunks.
constexpr uint32_t kTmaHeadElems = 128;
constexpr uint32_t kTmaMaxDepth = 32;   // k_reduce_tma keeps the row of stage s in lane s
// k_reduce_probe (gpr_probe.cuh), the AUTO kernel of calls whose rows may stop: a 32-sample head, then 512-sample
// chunks (DESIGN.md §4.1).  Most busy rows settle in their first samples and pay 128 B; a row that settles late pays
// at most one 2 KB chunk past its first settling sample.  One CTA of kProbeWarps warps per SM on the full budget:
// 3 stages per warp at T >= 512, 96 rows in flight.  A warp serves its landed stages one after another, so the rows
// are spread over as many warps as a CTA holds; 16 warps of 6 stages were 8 % slower at C2 (DESIGN.md §4.3).
constexpr uint32_t kProbeHeadElems = 32;
constexpr uint32_t kProbeChunkElems = 512;
constexpr int kProbeCtasPerSm = 1;
constexpr int kProbeWarps = 32;
constexpr size_t kProbeSmemBudget = kTmaSmemBudget;

// (the same definition, under the same guard, is in gpr_kernels.cuh's namespace body, which must also compile alone)
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

// The tuning knobs (GPR_KERNEL, GPR_LDG_CTAS, GPR_TMA_WARPS, GPR_TMA_CHUNK, GPR_TMA_DEPTH, GPR_FOLD_THREADS), as
// gpr_create has validated them, and the device's SM count.
struct LaunchKnobs {
  int sm_count = 1;
  int variant = GPR_KERNEL_AUTO;
  int ldg_ctas_per_sm = 2;
  int tma_warps = 16;         // 4, 8, 16 or 32
  int tma_chunk_bytes = 8192; // 512 .. 65536, multiple of 16
  int tma_depth_max = 3;
  int fold_threads = 256;     // 64, 128 or 256
};

enum ReduceKernel { kReduceLdg = 1, kReduceTma = 2, kReduceU8 = 3, kReduceProbe = 4 };
// why a TMA request runs the LDG kernel instead
enum TmaFallback { kNoFallback = 0, kFallbackAlignment = 1, kFallbackSmem = 2 };

struct ReducePlan {
  int kernel;        // ReduceKernel
  int fallback;      // TmaFallback
  uint32_t grid, block;
  size_t smem;       // dynamic shared memory (TMA only)
  TmaLayout L;       // TMA and probe only
};

// Rows are cut into n_chunks nearly equal chunks of at most tma_chunk_bytes, each a multiple of 4 elements
// (the bulk copy moves multiples of 16 bytes); as many stages per warp as fit the budget, at most tma_depth_max.
inline TmaLayout tma_layout(const LaunchKnobs& k, uint32_t T, int nw) {
  TmaLayout L;
  const uint64_t row_bytes = (uint64_t)T * 4u;
  const uint32_t max_chunk = (uint32_t)k.tma_chunk_bytes;
  L.n_chunks = (uint32_t)((row_bytes + max_chunk - 1) / max_chunk);
  uint32_t ce = (T + L.n_chunks - 1) / L.n_chunks;
  ce = (ce + 3u) & ~3u;
  L.chunk_elems = ce;
  L.n_chunks = (T + ce - 1) / ce;
  L.stage_bytes = (ce * 4u + 127u) & ~127u;
  uint32_t d = (uint32_t)((kTmaSmemBudget - 1024) / ((size_t)L.stage_bytes * nw));
  d = std::min<uint32_t>(d, std::min<uint32_t>((uint32_t)k.tma_depth_max, kTmaMaxDepth));
  L.depth = std::max<uint32_t>(d, 1u);
  L.head_elems = std::min<uint32_t>(kTmaHeadElems, ce);
  return L;
}

// stages, one mbarrier per stage, and the CTA's row counter
inline size_t tma_smem_bytes(const TmaLayout& L, int nw) {
  return (size_t)nw * L.depth * L.stage_bytes + (size_t)nw * L.depth * sizeof(uint64_t) + sizeof(uint64_t);
}

// k_reduce_probe's ring: stages of one chunk (a window shorter than a chunk gets stages of its own length), as many
// per warp as kProbeSmemBudget holds, at most kTmaMaxDepth.  The tma knobs do not apply.
// n_chunks = copies of a row read to its end.
inline TmaLayout probe_layout(uint32_t T, int nw) {
  TmaLayout L;
  L.chunk_elems = std::min<uint32_t>(kProbeChunkElems, std::max<uint32_t>((T + 3u) & ~3u, 4u));
  L.head_elems = std::min<uint32_t>(kProbeHeadElems, L.chunk_elems);
  L.n_chunks = 1u + (T > L.head_elems ? (T - L.head_elems + L.chunk_elems - 1u) / L.chunk_elems : 0u);
  L.stage_bytes = (L.chunk_elems * 4u + 127u) & ~127u;
  // (each stage also has its 8-byte barrier, and the CTA one row counter: short stages make the barriers count)
  const uint32_t d = (uint32_t)((kProbeSmemBudget - 8) / (((size_t)L.stage_bytes + 8) * nw));
  L.depth = std::max<uint32_t>(std::min<uint32_t>(d, kTmaMaxDepth), 1u);
  return L;
}

// The reduce launch for `total_rows` rows of T samples.  tma_ok: every row base is 16-byte aligned and T % 4 == 0
// (what a bulk copy needs); util_u8: the util plane is in GPR_FMT_U8B; may_stop: every row may stop at its first
// settling sample (no series_max target and no group table, so no row is read whole for its max).  AUTO means the
// probe kernel when rows may stop and the bulk copies and the f32 util plane allow it, else TMA (DESIGN.md §4.3).
inline ReducePlan plan_reduce(const LaunchKnobs& k, uint32_t T, uint32_t total_rows, bool tma_ok, bool util_u8,
                              bool may_stop = false) {
  ReducePlan r = {};
  if (k.variant == GPR_KERNEL_AUTO && may_stop && tma_ok && !util_u8) {
    const int nw = kProbeWarps;
    r.kernel = kReduceProbe;
    r.grid = (uint32_t)std::max<uint64_t>(
        1, std::min<uint64_t>((uint64_t)k.sm_count * kProbeCtasPerSm, ((uint64_t)total_rows + nw - 1) / nw));
    r.block = (uint32_t)nw * 32u;
    r.L = probe_layout(T, nw);
    r.smem = tma_smem_bytes(r.L, nw);
    return r;
  }
  int variant = k.variant == GPR_KERNEL_AUTO ? GPR_KERNEL_TMA : k.variant;
  if (variant == GPR_KERNEL_TMA && !tma_ok) variant = GPR_KERNEL_LDG, r.fallback = kFallbackAlignment;
  if (variant == GPR_KERNEL_TMA && tma_smem_bytes(tma_layout(k, T, k.tma_warps), k.tma_warps) > kTmaSmemBudget)
    variant = GPR_KERNEL_LDG, r.fallback = kFallbackSmem;  // a GPR_TMA_WARPS / GPR_TMA_CHUNK that does not fit
  // (64-bit: total_rows reaches 2^32 - 2 with a power plane)
  const uint64_t ldg_need = ((uint64_t)total_rows + kLdgWarps - 1) / kLdgWarps;
  const uint64_t ldg_grid = std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)k.sm_count * k.ldg_ctas_per_sm, ldg_need));
  if (util_u8) {  // biased-byte util plane: one kernel, any alignment (the power plane stays f32)
    r.kernel = kReduceU8, r.fallback = kNoFallback;
    r.grid = (uint32_t)ldg_grid, r.block = kLdgWarps * 32;
  } else if (variant == GPR_KERNEL_TMA) {
    const int nw = k.tma_warps;
    r.kernel = kReduceTma;
    r.grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)k.sm_count, ((uint64_t)total_rows + nw - 1) / nw));
    r.block = (uint32_t)nw * 32u;
    r.L = tma_layout(k, T, nw);
    r.smem = tma_smem_bytes(r.L, nw);
  } else {
    r.kernel = kReduceLdg;
    r.grid = (uint32_t)ldg_grid, r.block = kLdgWarps * 32;
  }
  return r;
}

// The fold grid for P pods: one bitmap word per warp and round, 4 words per warp in flight (fold_words<4>), at
// most one CTA per SM.  The fold loops when ceil(P / 32) > 4 * (fold_threads / 32) * sm_count.
inline uint32_t fold_grid(const LaunchKnobs& k, uint32_t P) {
  const uint32_t W = (uint32_t)(((uint64_t)P + 31u) / 32u), warps = (uint32_t)k.fold_threads / 32u;
  return std::max<uint32_t>(1u, std::min<uint32_t>((W + 4u * warps - 1u) / (4u * warps), (uint32_t)k.sm_count));
}

// k_group_rows / k_group_sum (gpr_groups.cuh, only with a group table): CTAs of kGroupBlock threads, one warp per pod
// and round, at most 8 CTAs per SM; both kernels loop over the pods (k_group_sum over the listed ones).
constexpr uint32_t kGroupBlock = 256;
inline uint32_t group_grid(const LaunchKnobs& k, uint32_t P) {
  const uint64_t ctas = ((uint64_t)P + kGroupBlock / 32u - 1u) / (kGroupBlock / 32u);
  return (uint32_t)std::max<uint64_t>(1u, std::min<uint64_t>(ctas, (uint64_t)k.sm_count * 8u));
}

// rounds of fold_words' outer loop for the first warp of the fold grid
inline uint32_t fold_rounds(const LaunchKnobs& k, uint32_t P) {
  const uint32_t W = (uint32_t)(((uint64_t)P + 31u) / 32u);
  const uint32_t per_round = 4u * fold_grid(k, P) * ((uint32_t)k.fold_threads / 32u);
  return (W + per_round - 1u) / per_round;
}

}  // namespace gpr
