// visual_dogleg_emu.cpp — TEST INFRASTRUCTURE: the passes of the DOGLEG trust-region strategy
// (global-lvba_b200/csrc/visual_dogleg.h) run through the host policy over every landmark of a problem, so that
// tests/test_visual_dogleg_emu.py can compare D, g, GN, alpha, the chosen step and its model cost change with
// tests/visual_dogleg_oracle.py without a GPU.  Never part of the product.
#include <cmath>
#include <vector>

#include "../../global-lvba_b200/csrc/visual_dogleg.h"
#include "host_exec.h"

using namespace lvba;

// At the state (q, t, X) with the Jacobi scale s_cam [n_rows*6] / s_pt [Tv*3], from the camera rows' column norms and gradient
// (cam_colsq, cam_grad [n_rows*6]), the solve's camera step y [n_rows*6] and the back-substitution's pt_step [T*3] (caller
// landmarks): vdog::linearised, then vdog::step at each of the n_radius radii (the first fresh, the others reusing).
// Outputs: D, g, GN [n] (n = 6 n_rows + 3 Tv); per radius j: sc [j][kNScal], v [j][n], Xc [j][T*3], scal [j][3] (model, step^2,
// x^2 of the landmarks)
extern "C" void emu_dogleg_run(int n_rows, int64_t Tv, const int* trk_ptr, const int* trk_id, const int* obs_cam, const int* obs_row,
                               const float* obs_uv, const double* plane, const double* intr, double sigma_px, double sigma_pl,
                               int loss_px, double a_px, int loss_pl, double a_pl, const double* q, const double* t, const double* X,
                               int64_t T, const double* s_cam, const double* s_pt, const double* cam_colsq, const double* cam_grad,
                               const double* y, const double* pt_step, int n_radius, const double* radius, double* D, double* g,
                               double* gn, double* sc, double* v, double* Xc, double* scal) {
  VisualView vv{};
  vv.trk_ptr = trk_ptr; vv.trk_id = trk_id; vv.obs_cam = obs_cam; vv.obs_row = obs_row;
  vv.obs_uv = reinterpret_cast<const float2*>(obs_uv); vv.plane = plane;
  for (int i = 0; i < 8; ++i) vv.intr[i] = intr[i];
  vv.inv_sigma_px = 1.0 / sigma_px;
  vv.inv_sigma_pl = 1.0 / std::max(1e-9, sigma_pl);
  vv.loss_px = loss_px; vv.loss_a_px = a_px; vv.loss_pl = loss_pl; vv.loss_a_pl = a_pl;
  const bool loss = loss_px != kLossNone || loss_pl != kLossNone;
  const VisualState st{q, t, X};
  const VisualLM lm{1e8, 1e-6, 1e32, s_cam, s_pt};
  const int64_t n = 6 * (int64_t)n_rows + 3 * Tv;
  HostExec ex;
  HostExec::Buf<double> buf;
  const int64_t ps = vdog::prod_size(n, Tv), pp = vdog::part_size(n, Tv);
  buf.alloc((size_t)(4 * n + ps + pp + vdog::kNScal));
  double* b = buf.p;
  const vdog::Bufs B{b, b + n, b + 2 * n, b + 3 * n, b + 4 * n, b + 4 * n + ps, b + 4 * n + ps + pp};
  std::vector<double> xc((size_t)T * 3), sl(16, 0.0);
  if (loss) vdog::linearised<true>(ex, vv, st, lm, n_rows, Tv, cam_colsq, cam_grad, y, pt_step, B);
  else vdog::linearised<false>(ex, vv, st, lm, n_rows, Tv, cam_colsq, cam_grad, y, pt_step, B);
  for (int64_t i = 0; i < n; ++i) { D[i] = B.D[i]; g[i] = B.g[i]; gn[i] = B.gn[i]; }
  for (int j = 0; j < n_radius; ++j) {
    for (int64_t i = 0; i < T * 3; ++i) xc[(size_t)i] = X[i];
    if (loss) vdog::step<true>(ex, vv, st, lm, n_rows, Tv, radius[j], j == 0, xc.data(), B, sl.data());
    else vdog::step<false>(ex, vv, st, lm, n_rows, Tv, radius[j], j == 0, xc.data(), B, sl.data());
    for (int i = 0; i < vdog::kNScal; ++i) sc[(int64_t)j * vdog::kNScal + i] = B.sc[i];
    for (int64_t i = 0; i < n; ++i) v[(int64_t)j * n + i] = B.v[i];
    for (int64_t i = 0; i < T * 3; ++i) Xc[(int64_t)j * T * 3 + i] = xc[(size_t)i];
    for (int i = 0; i < 3; ++i) scal[3 * j + i] = sl[2 + i];
  }
}
