// balm_rule.h — the damping rule of BALM2::damping_iter (reference include/BALM/bavoxel.hpp:662-767): the accept / reject
// decision of one LM pass, its update of u and v and the stop test, for the single and the window-batched LiDAR LM.
// Plain C++ (no CUDA): tests/emu/balm_rule_emu.cpp compiles it on the host.
#pragma once
#include <cmath>
#include <cstdio>

#include "../../include/lvba_b200.h"

namespace lvba {

// the LM state of one solve (bavoxel.hpp:664-671)
struct BalmState {
  double u = 0.01, v = 2.0, residual1 = 0.0;
  double cost_first = 0.0, cost_last = 0.0;
  bool have_first = false, converged = false;
  int iters = 0, accepted = 0, term = LVBA_TERM_MAX_ITER;
  // a new solve with the options' damping; cost_first and cost_last keep their values until its first pass sets them
  void reset(const lvba_lidar_opts& o) {
    u = o.u0; v = o.v0; residual1 = 0.0;
    have_first = converged = false;
    iters = accepted = 0; term = LVBA_TERM_MAX_ITER;
  }
};

// One pass (bavoxel.hpp:733-762).  sc = [r1 sum, q1, non-finite flag, r2 sum] of the pass, V the AVG_THR divisor (:635);
// rebuilt: H was built this pass and sc[0] is the residual at the current poses.  A non-finite step, model or trial residual
// is rejected.  Returns whether the trial poses are accepted.  `label` starts the verbose line.
inline bool balm_step(BalmState& s, const double sc[4], double V, bool rebuilt, const lvba_lidar_opts& o, const char* label) {
  if (rebuilt) s.residual1 = sc[0] / V;
  if (!s.have_first) { s.cost_first = s.residual1; s.cost_last = s.residual1; s.have_first = true; }
  const double q1 = sc[1] / V;                                 // :732
  double residual2 = sc[3] / V;
  const bool bad = sc[2] != 0.0 || !std::isfinite(residual2) || !std::isfinite(q1);
  if (bad) residual2 = NAN;
  double q = s.residual1 - residual2;
  ++s.iters;
  if (o.verbose)
    fprintf(stderr, "[%s] iter %d: (%.9g %.9g) u: %g v: %g q: %g q1: %g\n", label, s.iters - 1, s.residual1, residual2, s.u, s.v, q, q1);
  const bool accept = q > 0;
  if (accept) {                                                // :744-752
    q = q / q1;
    s.v = 2;
    q = 1 - std::pow(2 * q - 1, 3);
    s.u *= (q < (1.0 / 3.0) ? (1.0 / 3.0) : q);
    ++s.accepted;
    s.cost_last = residual2;
  } else {                                                     // :753-758
    s.u = s.u * s.v;
    s.v = 2 * s.v;
  }
  if (o.rel_tol >= 0 && std::fabs(s.residual1 - residual2) / s.residual1 < o.rel_tol) {   // :760
    s.converged = true;
    s.term = LVBA_TERM_FUNCTION_TOL;
  }
  return accept;
}

}  // namespace lvba
