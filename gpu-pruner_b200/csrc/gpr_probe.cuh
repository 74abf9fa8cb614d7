// gpr_probe.cuh — k_reduce_probe, the reduce kernel AUTO runs for calls whose rows may stop (DESIGN.md §4.1).
//
// Early exit leaves most rows after a few samples, so the time of such a call goes to round trips, not to bytes: a
// kernel with few rows in flight per SM waits for one copy after another.  This kernel keeps many short copies in
// flight and serves them in the order they land.
#pragma once

#include "gpr_kernels.cuh"

namespace gpr {

// non-blocking test of a stage's mbarrier: true once the phase of the given parity has completed
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "mbarrier.test_wait.parity.shared::cta.b64 P1, [%1], %2;\n"
      "selp.u32 %0, 1, 0, P1;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0u;
}

// Requirements (checked on the host): every row base 16-byte aligned, T % 4 == 0, no series_max target and no group
// table (every row may stop at its first settling sample).
//
// A row is read as its head [0, head_elems), then chunks of chunk_elems (layout: gpr_launch.h probe_layout), one copy
// in flight per row, each requested after the row's previous copy was examined; the row stops at the first copy that
// holds a settling sample, an idle row is read to its end.  So the bytes a row costs depend on nothing but its data
// and the two constants, as in k_reduce_tma.
//
// Each warp owns a ring of `depth` stages (one mbarrier, one row, one copy in flight each; lane s keeps stage s's row,
// copy index and running max).  Unlike k_reduce_tma the warp does not visit its stages in ring order: every lane
// polls its own stage's barrier without blocking, and the warp serves every stage whose copy has landed, so a 128 B
// head that has arrived is never held up behind a 2 KB chunk still in flight.  Serving a stage folds its bytes into
// the row's max, then re-arms the stage with the row's next chunk, or publishes the row and re-arms the stage with
// the head of the next row the CTA hands out.  A stage is only ever touched by its owner warp, so its phase parity
// cannot alias.  Rows are split between CTAs as in the other reduce kernels (cta_row_count).  A warp serves its
// landed stages one at a time, so the service rate grows with the warp count: the library launches NW = kProbeWarps
// (32) with 3 stages each.  (Capped at 48 registers, which would leave room for a fold CTA beside it, the kernel
// was 11 % slower on windows read whole.)
template <int NW>
__global__ void __launch_bounds__(NW * 32, kProbeCtasPerSm) k_reduce_probe(ReduceParams p, TmaLayout L) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int lane = threadIdx.x & 31;
  const uint32_t w = threadIdx.x >> 5;
  const uint32_t D = L.depth;  // <= 32
  unsigned char* stage0 = smem + (size_t)w * D * L.stage_bytes;
  uint64_t* const bars = reinterpret_cast<uint64_t*>(smem + (size_t)NW * D * L.stage_bytes);
  uint64_t* full = bars + w * D;
  unsigned int* next_row = reinterpret_cast<unsigned int*>(bars + NW * D);

  pdl_launch_dependents();
  const uint32_t n_rows = cta_row_count(p.total_rows);
  const uint32_t h = L.head_elems, ce = L.chunk_elems;
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
    const uint32_t e0 = c ? h + (c - 1u) * ce : 0u;
    const uint32_t bytes = min(c ? ce : h, p.T - e0) * 4u;
    if (lane == 0) {
      mbar_expect_tx(&full[s], bytes);
      tma_load_1d(stage0 + (size_t)s * L.stage_bytes, row + e0, bytes, &full[s], pol);
    }
  };
  uint32_t my_j = min(w + NW * (uint32_t)lane, n_rows), my_c = 0;
  float my_m = nan_f();
  uint32_t live = 0;   // bit s: stage s has a copy in flight
  for (uint32_t s = 0; s < D; ++s) {
    const uint32_t j = w + NW * s;
    if (j < n_rows) issue(s, j, 0u), live |= 1u << s;
  }

  uint32_t phase = 0;  // bit s: parity of stage s's next completion
  while (live) {
    const bool landed = ((live >> lane) & 1u) && mbar_test_wait(&full[lane], (phase >> lane) & 1u);
    uint32_t ready = __ballot_sync(0xffffffffu, landed);
    while (ready) {
      const uint32_t s = (uint32_t)__ffs(ready) - 1u;
      ready &= ready - 1u;
      uint32_t j = __shfl_sync(0xffffffffu, my_j, (int)s);
      uint32_t c = __shfl_sync(0xffffffffu, my_c, (int)s);
      float m = __uint_as_float(__shfl_sync(0xffffffffu, __float_as_uint(my_m), (int)s));
      mbar_wait(&full[s], (phase >> s) & 1u);  // returns at once; orders every lane's reads after the copy
      phase ^= 1u << s;
      const uint32_t e0 = c ? h + (c - 1u) * ce : 0u;
      const uint32_t n = min(c ? ce : h, p.T - e0);
      const float4* v = reinterpret_cast<const float4*>(stage0 + (size_t)s * L.stage_bytes);
      const uint32_t nv = n >> 2;
      float m0 = nan_f(), m1 = nan_f();
      uint32_t k = lane;
#pragma unroll 2
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
      if (e0 + n < p.T && !settles(m, is_power, p.thr)) {
        issue(s, j, ++c);
      } else {
        uint32_t next = 0;
        if (lane == 0) {
          if (!scratch_ok) wait_scratch_free(p), scratch_ok = true;
          publish_row(p, seg, local, m, false);
          next = atomicAdd(next_row, 1u);
        }
        j = min(__shfl_sync(0xffffffffu, next, 0), n_rows), c = 0, m = nan_f();
        if (j < n_rows) issue(s, j, 0u);
        else live &= ~(1u << s);
      }
      if ((uint32_t)lane == s) my_j = j, my_c = c, my_m = m;
    }
  }
}

}  // namespace gpr
