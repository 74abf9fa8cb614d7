// TEST INFRASTRUCTURE.  The launch geometry of gpu-pruner_b200/csrc/gpr_launch.h as a filter, so that the tests can
// choose shapes that reach a given regime and check which kernel the library ran for a window.
// One query per input line:
//   sm_count variant tma_warps tma_chunk_bytes tma_depth ldg_ctas fold_threads T total_rows tma_ok util_u8 P may_stop
// one answer per output line:
//   kernel fallback grid block smem depth stage_bytes chunk_elems n_chunks fold_grid fold_rounds head_elems
// (kernel: 1 LDG, 2 TMA, 3 U8, 4 probe; fallback: 0 none, 1 alignment / T % 4, 2 shared memory over budget;
// may_stop: the call has no series_max target and no group table, so every row may stop at its first settling sample)
#include <cstdio>
#include <iostream>

#include "../../gpu-pruner_b200/csrc/gpr_launch.h"

int main() {
  gpr::LaunchKnobs k;
  unsigned long long T, rows, P;
  int tma_ok, u8, may_stop;
  while (std::cin >> k.sm_count >> k.variant >> k.tma_warps >> k.tma_chunk_bytes >> k.tma_depth_max >>
         k.ldg_ctas_per_sm >> k.fold_threads >> T >> rows >> tma_ok >> u8 >> P >> may_stop) {
    const gpr::ReducePlan r =
        gpr::plan_reduce(k, (uint32_t)T, (uint32_t)rows, tma_ok != 0, u8 != 0, may_stop != 0);
    printf("%d %d %u %u %zu %u %u %u %u %u %u %u\n", r.kernel, r.fallback, r.grid, r.block, r.smem, r.L.depth,
           r.L.stage_bytes, r.L.chunk_elems, r.L.n_chunks, gpr::fold_grid(k, (uint32_t)P),
           gpr::fold_rounds(k, (uint32_t)P), r.L.head_elems);
  }
  return 0;
}
