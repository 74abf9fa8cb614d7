// TEST INFRASTRUCTURE.  gpu-pruner_b200/csrc/gpr_launch.h's plan_reduce with its may_stop argument, as a filter.
// One query per input line:
//   sm_count variant tma_warps tma_chunk_bytes tma_depth T total_rows tma_ok util_u8 may_stop
// one answer per output line:
//   kernel fallback grid block smem depth stage_bytes chunk_elems n_chunks head_elems
// (kernel: 1 LDG, 2 TMA, 3 U8, 4 probe)
#include <cstdio>
#include <iostream>

#include "../../gpu-pruner_b200/csrc/gpr_launch.h"

int main() {
  gpr::LaunchKnobs k;
  unsigned long long T, rows;
  int tma_ok, u8, may_stop;
  while (std::cin >> k.sm_count >> k.variant >> k.tma_warps >> k.tma_chunk_bytes >> k.tma_depth_max >> T >> rows >>
         tma_ok >> u8 >> may_stop) {
    const gpr::ReducePlan r =
        gpr::plan_reduce(k, (uint32_t)T, (uint32_t)rows, tma_ok != 0, u8 != 0, may_stop != 0);
    printf("%d %d %u %u %zu %u %u %u %u %u\n", r.kernel, r.fallback, r.grid, r.block, r.smem, r.L.depth,
           r.L.stage_bytes, r.L.chunk_elems, r.L.n_chunks, r.L.head_elems);
  }
  return 0;
}
