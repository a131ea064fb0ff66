// The damping rule of the LiDAR LM (global-lvba_b200/csrc/balm_rule.h) on the host, driven by tests/test_lm_rules_emu.py the
// way lvba_lidar_iterate drives it (residual1 refreshed only after an accepted pass rebuilt H) or the way lvba_lidar_lm_batch
// drives every window (H rebuilt every pass).
#include "../../global-lvba_b200/csrc/balm_rule.h"

// n passes with the results sc[4k..4k+3] = [r1 sum, q1, non-finite flag, r2 sum] and divisor V, until the stop test;
// after pass k: u[k], v[k], accepted[k], term[k].  Returns the passes run.
extern "C" int balm_rule_run(double u0, double v0, double rel_tol, int batched, int verbose, int n, const double* sc, double V,
                             double* u, double* v, int* accepted, int* term) {
  lvba_lidar_opts o{};
  o.u0 = u0; o.v0 = v0; o.rel_tol = rel_tol; o.max_iter = n; o.verbose = verbose;
  lvba::BalmState s;
  s.reset(o);
  bool rebuilt = true;
  int k = 0;
  for (; k < n && !s.converged; ++k) {
    const bool acc = lvba::balm_step(s, sc + 4 * k, V, rebuilt, o, "emu");
    rebuilt = batched || acc;
    u[k] = s.u; v[k] = s.v; accepted[k] = acc; term[k] = s.term;
  }
  return k;
}
