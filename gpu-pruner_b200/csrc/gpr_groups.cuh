// gpr_groups.cuh — exact `sum by` groups on the device (gpr_window.groups).
//
// In the reference query an element is a `sum by (Hostname, container, pod, namespace, gpu, modelName)` group
// (query.promql.j2:9,21), not a series: a pod can carry several series of one group (a PROF series with an extra
// label next to the UTIL one, a second exporter), and the element's value is Prometheus' float64 sum of their window
// maxima, UTIL members divided by 100 first (j2:20).  The tensor keeps every series in its own row; a group table says
// which rows belong together, and two kernels turn the per-row flags into per-element flags:
//
//   k_group_rows  (before the reduce) one warp per pod: checks the pod's table entries, marks every row of a group of
//                 two or more in a per-pod bitmap laid out like the flag words (the reduce reads such rows whole and
//                 keeps their max), and lists the pods that have such a group.
//   k_group_sum   (between the reduce and the fold) one warp per listed pod: for every group of two or more, in
//                 ascending slot order, the Neumaier sum of its members' maxima; the pod's flag words lose their
//                 member bits and get the leader's bit iff the sum is == 0.  k_fold then runs unchanged and its
//                 popcounts count elements.
//
// A lone row (a group of one) keeps the bit the reduce gave it: its group value is its max (/ 100), which is == 0
// exactly when the max is (a -0.0 max sums to +0.0, a denormal / 100 stays non-zero in float64).
//
// Plain CUDA C++ without inline PTX or shared memory: tests/cpp/groups_emul.cpp runs this source on the CPU.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include "gpr_launch.h"

namespace gpr {

constexpr uint32_t kGroupLeader = 0xffu;     // gpr_window.groups bits 0-7: slot of the group's first member
constexpr uint32_t kGroupUtil = 0x100u;      // GPR_GROUP_UTIL: a GPU_UTIL member (max / 100)

struct GroupParams {
  const uint32_t* table;   // [P][G] gpr_window.groups, device
  uint32_t* need;          // [P][mw] out of k_group_rows: bit g set iff row (p, g) is in a group of two or more
  uint32_t* pods;          // [P] out of k_group_rows: the pods with such a group, in no particular order
  unsigned int* n_pods;    // length of `pods`; zero before k_group_rows
  const float* gmax;       // [P * G] window max of every row marked in `need` (the reduce's output)
  uint32_t* idle_mask;     // [P][mw] the util flag words of this decision, rewritten by k_group_sum
  unsigned int* bad;       // host-mapped: 1 + a pod whose table is malformed; 0 = none
  uint32_t P, G, mw;
};

// Prometheus' `sum` (promql/engine.go kahanSumInc), operation for operation as host/ingest.cpp's KahanSum: the
// build has no fast-math and no FMA contraction, so every step rounds as the host's does.
struct NeumaierSum {
  double sum = 0.0, c = 0.0;
  bool any = false;
  __device__ __forceinline__ void add(double x) {
    any = true;
    const double t = sum + x;
    if (isinf(t)) c = 0.0;
    else if (fabs(sum) >= fabs(x)) c += (sum - t) + x;
    else c += (x - t) + sum;
    sum = t;
  }
  __device__ __forceinline__ double value() const { return isinf(sum) ? sum : sum + c; }
};

// Is entry x of slot g malformed?  (e = the pod's entries)
__device__ __forceinline__ bool group_entry_bad(const uint32_t* e, uint32_t g, uint32_t x) {
  const uint32_t l = x & kGroupLeader;
  return (x & ~(kGroupLeader | kGroupUtil)) != 0u || l > g || (e[l] & kGroupLeader) != l;
}

__global__ void __launch_bounds__(kGroupBlock) k_group_rows(GroupParams q) {
  const uint32_t lane = threadIdx.x & 31u, warps = blockDim.x >> 5;
  for (uint32_t p = blockIdx.x * warps + (threadIdx.x >> 5); p < q.P; p += gridDim.x * warps) {
    const uint32_t* e = q.table + (size_t)p * q.G;
    bool bad = false;
    for (uint32_t g = lane; g < q.G; g += 32u) bad = bad || group_entry_bad(e, g, e[g]);
    bad = __ballot_sync(0xffffffffu, bad) != 0u;
    uint32_t any = 0;
    for (uint32_t k = 0; k < q.mw; ++k) {
      // word k: its members, and the leaders (in word k) of members anywhere at or after it
      uint32_t w = 0;
      for (uint32_t j = k; j < q.mw && !bad; ++j) {
        const uint32_t g = j * 32u + lane;
        const uint32_t l = g < q.G ? (e[g] & kGroupLeader) : g;
        const bool member = l != g;
        if (j == k) w |= __ballot_sync(0xffffffffu, member);
        w |= __reduce_or_sync(0xffffffffu, member && (l >> 5) == k ? 1u << (l & 31u) : 0u);
      }
      if (lane == 0) q.need[(size_t)p * q.mw + k] = w;
      any |= w;
    }
    if (lane == 0) {
      if (bad) *q.bad = p + 1u;   // any malformed pod will do: the call fails and names it
      else if (any) q.pods[atomicAdd(q.n_pods, 1u)] = p;
    }
  }
}

__global__ void __launch_bounds__(kGroupBlock) k_group_sum(GroupParams q) {
  const uint32_t lane = threadIdx.x & 31u, warps = blockDim.x >> 5;
  const uint32_t n = *q.n_pods;
  for (uint32_t i = blockIdx.x * warps + (threadIdx.x >> 5); i < n; i += gridDim.x * warps) {
    const uint32_t p = q.pods[i];
    const uint32_t* e = q.table + (size_t)p * q.G;
    const float* m = q.gmax + (size_t)p * q.G;
    for (uint32_t k = 0; k < q.mw; ++k) {
      const uint32_t g = k * 32u + lane;
      const uint32_t nb = q.need[(size_t)p * q.mw + k];
      bool idle = false;
      if (g < q.G && (nb >> lane & 1u) && (e[g] & kGroupLeader) == g) {   // leads a group of two or more
        NeumaierSum s;
        for (uint32_t h = g; h < q.G; ++h) {   // members follow their leader, in slot order
          const uint32_t x = e[h];
          if ((x & kGroupLeader) != g) continue;
          const float v = m[h];
          if (v != v) continue;   // no sample in the window: the series is no element of the instant vector
          s.add((x & kGroupUtil) ? (double)v / 100.0 : (double)v);
        }
        idle = s.any && s.value() == 0.0;   // no present member: NaN, not idle
      }
      const uint32_t lead = __ballot_sync(0xffffffffu, idle);
      if (lane == 0) {
        uint32_t* word = q.idle_mask + (size_t)p * q.mw + k;
        *word = (*word & ~nb) | lead;
      }
    }
  }
}

}  // namespace gpr
