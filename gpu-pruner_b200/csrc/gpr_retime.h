// gpr_retime.h — when the resident ring can be retimed exactly (gpr_resident_retime, gpr_ring.cuh k_retime_rows), in
// plain C++: the daemon session asks it before a retime, and the tests take it as the rule.
//
// The ring holds a window of N seconds at step s: T = ceil(N / s) buckets ending at t_end.  A window of N' seconds at
// step s' ending at the same t_end is the retimed ring, bit for bit, iff s' = k s (k >= 1), N' <= N, and N' % s == 0
// or N' == N.  Then it keeps the newest n_keep = ceil(N' / s) old buckets and new bucket b' (0 = newest) is the maximum
// of old buckets [k b', min(k b' + k, n_keep)): for an integer d = t_end - ts >= 0, floor(d / s') = floor(floor(d / s)
// / k), and old bucket n_keep - 1 lies inside (t_end - N', t_end] when N' % s == 0, or is cut where the old window cut
// it when N' == N.  Everything else (a finer step, a step that is not a multiple, a longer window, a shorter window
// that cuts an old bucket) would need samples the ring does not hold.
#pragma once

#include <stdint.h>

namespace gpr {

struct RetimePlan {
  uint32_t n_keep = 0, factor = 0;  // the arguments of gpr_resident_retime
  const char* refusal = nullptr;    // nullptr: the retime is exact
};

// N, s: the ring's window and step in seconds, T its buckets; N2, s2: the new window and step.  The same grid (s2 == s,
// N2 == N) is refused too: there is nothing to retime.
inline RetimePlan retime_plan(int64_t N, int64_t s, uint32_t T, int64_t N2, int64_t s2) {
  RetimePlan p;
  if (N <= 0 || s <= 0 || N2 <= 0 || s2 <= 0 || (int64_t)T != (N + s - 1) / s) p.refusal = "the grid is not a ring's grid";
  else if (s2 == s && N2 == N) p.refusal = "the grid did not change";
  else if (s2 < s) p.refusal = "the step got finer";
  else if (s2 % s != 0) p.refusal = "the new step is not a whole multiple of the old one";
  else if (N2 > N) p.refusal = "the window got longer";
  else if (N2 < N && N2 % s != 0) p.refusal = "the shorter window cuts a bucket of the old step";
  if (p.refusal) return p;
  p.n_keep = N2 == N ? T : (uint32_t)(N2 / s);
  p.factor = (uint32_t)(s2 / s);
  return p;
}

}  // namespace gpr
