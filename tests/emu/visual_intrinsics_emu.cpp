// visual_intrinsics_emu.cpp — TEST INFRASTRUCTURE: the passes of the intrinsics block of the visual LM
// (global-lvba_b200/csrc/visual_intr.h) run through the host policy, so that tests/test_visual_intrinsics_emu.py can compare the
// border, the corner, rhs_k, the column norms and the back-substitution with tests/visual_intr_oracle.py without a GPU.  The
// row CSR of the border gather is built as visual_intr_setup builds it.  Never part of the product.
#include <cmath>
#include <vector>

#include "../../global-lvba_b200/csrc/visual_intr.h"
#include "host_exec.h"

using namespace lvba;

// Jacobi scales from the caller: s_cam [n_rows*6], s_pt [Tv*3], sk [8] (0 in the held entries).  Outputs: colsq0 [8] (unscaled
// column norms, ColF), sys [kSys] (C upper, rhs_k, scaled column norms, gradient), B [8][n_rows*6]; with y_cam / yk: X_cand,
// pt_step [T*3] and out[0..2] = model-cost change, step^2, x^2 of the landmarks.
extern "C" void emu_vintr_step(int n_rows, int64_t Tv, const int* trk_ptr, const int* trk_id, const int* obs_cam, const int* obs_row,
                               const float* obs_uv, const double* plane, const double* intr, double sigma_px, double sigma_pl,
                               int loss_px, double loss_a_px, int loss_pl, double loss_a_pl, const double* q, const double* t,
                               const double* X, const double* s_cam, const double* s_pt, const double* sk, double radius,
                               double min_diag, double max_diag, const double* y_cam, const double* yk, double* colsq0, double* sys,
                               double* B, double* X_cand, double* pt_step, double* out) {
  VisualView vv{};
  vv.trk_ptr = trk_ptr; vv.trk_id = trk_id; vv.obs_cam = obs_cam; vv.obs_row = obs_row;
  vv.obs_uv = reinterpret_cast<const float2*>(obs_uv); vv.plane = plane;
  for (int i = 0; i < 8; ++i) vv.intr[i] = intr[i];
  vv.inv_sigma_px = 1.0 / sigma_px;
  vv.inv_sigma_pl = 1.0 / std::max(1e-9, sigma_pl);
  vv.loss_px = loss_px; vv.loss_a_px = loss_a_px; vv.loss_pl = loss_pl; vv.loss_a_pl = loss_a_pl;
  const bool robust = loss_px != kLossNone || loss_pl != kLossNone;
  const VisualState st{q, t, X};
  const VisualLM lm{radius, min_diag, max_diag, s_cam, s_pt};
  const int64_t nnz = trk_ptr[Tv], n6 = (int64_t)n_rows * 6, nch = std::max<int64_t>((Tv + 255) / 256, 1);
  HostExec ex;
  HostExec::Buf<double> slot, part, rec;
  slot.alloc((size_t)std::max<int64_t>(Tv, 1) * vintr::kSys);
  part.alloc((size_t)nch * vintr::kSys);
  rec.alloc((size_t)std::max<int64_t>(nnz, 1) * vintr::kRec);
  auto reduce = [&](int W, double* dst) {
    ex.for_each(nch * W, vintr::ReduceF{slot.p, Tv, 256, W, part.p});
    ex.for_each(W, vintr::ReduceF{part.p, nch, nch, W, dst});
  };
  if (robust) ex.for_each(Tv, vintr::ColF<true>{vv, st, slot.p});
  else ex.for_each(Tv, vintr::ColF<false>{vv, st, slot.p});
  reduce(8, colsq0);
  if (robust) ex.for_each(Tv, vintr::TrackF<true>{vv, st, lm, sk, slot.p, rec.p});
  else ex.for_each(Tv, vintr::TrackF<false>{vv, st, lm, sk, slot.p, rec.p});
  reduce(vintr::kSys, sys);
  std::vector<int64_t> ptr((size_t)n_rows + 1, 0), obs;
  for (int64_t w = 0; w < nnz; ++w)
    if (obs_row[w] >= 0) ++ptr[(size_t)obs_row[w] + 1];
  for (int r = 0; r < n_rows; ++r) ptr[(size_t)r + 1] += ptr[(size_t)r];
  obs.resize((size_t)ptr[(size_t)n_rows]);
  std::vector<int64_t> at(ptr.begin(), ptr.end() - 1);
  for (int64_t w = 0; w < nnz; ++w)
    if (obs_row[w] >= 0) obs[(size_t)at[(size_t)obs_row[w]]++] = w;
  ex.for_each(n6 / 6 * vintr::kRec, vintr::RowGatherF{ptr.data(), obs.data(), rec.p, n6, B});
  if (!y_cam) return;
  if (robust) {
    vintr::BacksubF<true> f{vv, st, lm, sk, y_cam, {}, X_cand, pt_step, slot.p};
    for (int i = 0; i < 8; ++i) f.yk[i] = yk[i];
    ex.for_each(Tv, f);
  } else {
    vintr::BacksubF<false> f{vv, st, lm, sk, y_cam, {}, X_cand, pt_step, slot.p};
    for (int i = 0; i < 8; ++i) f.yk[i] = yk[i];
    ex.for_each(Tv, f);
  }
  reduce(3, out);
}

// the corner solve of visual_intr_corner_kernel: S [k*k] row-major, r [k]; returns 1 and the solution in r, or 0
extern "C" int emu_vintr_corner_solve(int k, double* S, double* r) { return vintr::corner_solve(k, S, r) ? 1 : 0; }
