// visual_loss_emu.cpp — TEST INFRASTRUCTURE: the kLoss instantiations of the big-landmark passes of
// global-lvba_b200/csrc/visual_big.h run through the host policy over ALL landmarks of a problem, with robust losses on the
// reprojection and plane blocks, so that tests/test_visual_loss_emu.py can compare cost, column norms, the reduced camera
// system, rhs and the back-substitution with tests/visual_loss_oracle.py without a GPU.  Never part of the product.
#include <cmath>
#include <vector>

#include "../../global-lvba_b200/csrc/visual_big.h"
#include "host_exec.h"

namespace {

using namespace lvba;

struct Problem {
  VisualView vv{};
  vbig::View bv{};
  std::vector<int64_t> pair_ptr;
  Problem(int64_t Tv, const int* trk_ptr, const int* trk_id, const int* obs_cam, const int* obs_row, const float* obs_uv,
          const double* plane, const double* intr, double sigma_px, double sigma_pl, const int* loss_kind, const double* loss_a,
          const int* first, const long long* row_start) {
    vv.trk_ptr = trk_ptr; vv.trk_id = trk_id; vv.obs_cam = obs_cam; vv.obs_row = obs_row;
    vv.obs_uv = reinterpret_cast<const float2*>(obs_uv); vv.plane = plane;
    for (int i = 0; i < 8; ++i) vv.intr[i] = intr[i];
    vv.inv_sigma_px = 1.0 / sigma_px;
    vv.inv_sigma_pl = 1.0 / std::max(1e-9, sigma_pl);
    vv.loss_px = loss_kind[0]; vv.loss_pl = loss_kind[1]; vv.loss_a_px = loss_a[0]; vv.loss_a_pl = loss_a[1];
    pair_ptr.assign((size_t)Tv + 1, 0);
    for (int64_t k = 0; k < Tv; ++k) { const int64_t K = trk_ptr[k + 1] - trk_ptr[k]; pair_ptr[k + 1] = pair_ptr[k] + K * (K - 1); }
    bv = vbig::View{Tv, 0, pair_ptr.data(), first, row_start};   // every landmark is "big"
  }
};

}  // namespace

// cost (1/2 sum rho) at the state (q, t, X); loss_kind / loss_a [2]: reprojection, plane
extern "C" double emu_vloss_cost(int64_t Tv, const int* trk_ptr, const int* trk_id, const int* obs_cam, const int* obs_row, const float* obs_uv,
                                 const double* plane, const double* intr, double sigma_px, double sigma_pl, const int* loss_kind,
                                 const double* loss_a, const double* q, const double* t, const double* X) {
  Problem P(Tv, trk_ptr, trk_id, obs_cam, obs_row, obs_uv, plane, intr, sigma_px, sigma_pl, loss_kind, loss_a, nullptr, nullptr);
  std::vector<double> part((size_t)Tv);
  HostExec ex;
  ex.for_each(Tv, vbig::CostPass<true>{P.vv, P.bv, VisualState{q, t, X}, part.data()});
  double c = 0.0;
  for (double v : part) c += v;
  return c;
}

// As emu_vbig_step (tests/emu/visual_big_emu.cpp), through the kLoss passes
extern "C" void emu_vloss_step(int n_rows, int64_t Tv, const int* trk_ptr, const int* trk_id, const int* obs_cam, const int* obs_row,
                               const float* obs_uv, const double* plane, const double* intr, double sigma_px, double sigma_pl,
                               const int* loss_kind, const double* loss_a, const int* first, const long long* row_start,
                               const double* q, const double* t, const double* X, int jacobi_scaling, double radius, double min_diag,
                               double max_diag, const double* y_cam, double* cam_colsq0, double* pt_colsq0, double* S, double* rhs,
                               double* cam_colsq, double* cam_grad, double* X_cand, double* pt_step, double* out) {
  Problem P(Tv, trk_ptr, trk_id, obs_cam, obs_row, obs_uv, plane, intr, sigma_px, sigma_pl, loss_kind, loss_a, first, row_start);
  const VisualState st{q, t, X};
  const int64_t nnz = trk_ptr[Tv];
  HostExec ex;
  HostExec::Buf<double> obs, params, cost, gmax, bout;
  obs.alloc((size_t)nnz * vbig::kObs); params.alloc((size_t)Tv * kTrkParams);
  cost.alloc((size_t)Tv); gmax.alloc((size_t)Tv); bout.alloc((size_t)Tv * 4);
  ex.fill_zero(cam_colsq0, (size_t)n_rows * 6);
  ex.for_each(nnz, vbig::ColObsPass<false, true>{P.vv, P.bv, st, obs.p, cam_colsq0});
  ex.for_each(Tv, vbig::ColTrackPass<true>{P.vv, P.bv, st, obs.p, pt_colsq0});
  std::vector<double> s_cam((size_t)n_rows * 6), s_pt((size_t)Tv * 3);
  for (size_t i = 0; i < s_cam.size(); ++i) s_cam[i] = jacobi_scaling ? 1.0 / (1.0 + std::sqrt(cam_colsq0[i])) : 1.0;
  for (size_t i = 0; i < s_pt.size(); ++i) s_pt[i] = jacobi_scaling ? 1.0 / (1.0 + std::sqrt(pt_colsq0[i])) : 1.0;
  const VisualLM lm{radius, min_diag, max_diag, s_cam.data(), s_pt.data()};
  ex.for_each(nnz, vbig::ObsPass<true>{P.vv, P.bv, st, lm, obs.p});
  ex.for_each(Tv, vbig::TrackPass<true>{P.vv, P.bv, st, lm, obs.p, params.p, cost.p, gmax.p});
  ex.for_each(nnz, vbig::SlotsF{P.vv, P.bv, params.p, obs.p, S, rhs, cam_colsq, cam_grad});
  ex.for_each(P.pair_ptr[Tv], vbig::PairsF{P.vv, P.bv, obs.p, S});
  out[0] = 0.0; out[1] = 0.0;
  for (int64_t b = 0; b < Tv; ++b) { out[0] += cost.p[b]; out[1] = std::fmax(out[1], gmax.p[b]); }
  if (!y_cam) return;
  ex.for_each(Tv, vbig::BacksubPass<true>{P.vv, P.bv, st, lm, obs.p, params.p, y_cam, X_cand, pt_step, bout.p});
  out[2] = out[3] = out[4] = 0.0;
  for (int64_t b = 0; b < Tv; ++b) for (int j = 0; j < 3; ++j) out[2 + j] += bout.p[4 * b + j];
}
