// visual_implicit_emu.cpp — TEST INFRASTRUCTURE: the matrix-free reduced camera system of ITERATIVE_SCHUR
// (global-lvba_b200/csrc/visual_implicit.h) run through the host policy over ALL landmarks of a problem, beside the explicit
// passes of visual_big.h on the same problem, so that tests/test_visual_implicit_emu.py can compare the two builds, the product
// and the whole conjugate-gradients solve with tests/visual_pcg_oracle.py without a GPU.  Never part of the product.
#include <cmath>
#include <vector>

#include "../../global-lvba_b200/csrc/visual_implicit.h"
#include "host_exec.h"

using namespace lvba;

// vimp::visual_matrix_free of the plan's counts
extern "C" int emu_imp_choose(int64_t free_obs, int64_t n_pairs, int64_t n_blocks_env, int n_rows) {
  return vimp::visual_matrix_free(free_obs, n_pairs, n_blocks_env, n_rows) ? 1 : 0;
}

// At the state (q, t, X), Jacobi scale as emu_vbig_step computes it:
//   explicit (visual_big.h, every landmark big) -> S [nblocks*36], rhs_x / colsq_x / grad_x [n_rows*6], out_x[0..1] cost, gmax
//   matrix-free (visual_implicit.h), with its own scale pass -> rhs / colsq / grad [n_rows*6], D [n_rows*36] (undamped), out[0..1]
// then, with the damping dadd [n_rows*6]: y = (S + diag(dadd)) x by the matrix-free product; and the solve of
// (S + diag(dadd)) x_sol = rhs by vpcg::solve_with on that product and the PrecDF preconditioner, info = iterations, termination
extern "C" void emu_imp_run(int n_rows, int64_t Tv, const int* trk_ptr, const int* trk_id, const int* obs_cam, const int* obs_row,
                            const float* obs_uv, const double* plane, const double* intr, double sigma_px, double sigma_pl,
                            int loss_px, double a_px, int loss_pl, double a_pl, const int* first, const long long* row_start,
                            const double* q, const double* t, const double* X, int jacobi_scaling, double radius,
                            double* S, double* rhs_x, double* colsq_x, double* grad_x, double* out_x,
                            double* rhs, double* colsq, double* grad, double* D, double* out,
                            const double* dadd, const double* x, double* y, double eta, int min_iter, int max_iter, double* x_sol,
                            int* info) {
  VisualView vv{};
  vv.trk_ptr = trk_ptr; vv.trk_id = trk_id; vv.obs_cam = obs_cam; vv.obs_row = obs_row;
  vv.obs_uv = reinterpret_cast<const float2*>(obs_uv); vv.plane = plane;
  for (int i = 0; i < 8; ++i) vv.intr[i] = intr[i];
  vv.inv_sigma_px = 1.0 / sigma_px;
  vv.inv_sigma_pl = 1.0 / std::max(1e-9, sigma_pl);
  vv.loss_px = loss_px; vv.loss_a_px = a_px; vv.loss_pl = loss_pl; vv.loss_a_pl = a_pl;
  const bool loss = loss_px != kLossNone || loss_pl != kLossNone;
  std::vector<int64_t> pair_ptr((size_t)Tv + 1, 0);
  for (int64_t k = 0; k < Tv; ++k) { const int64_t K = trk_ptr[k + 1] - trk_ptr[k]; pair_ptr[k + 1] = pair_ptr[k] + K * (K - 1); }
  const vbig::View bv{Tv, 0, pair_ptr.data(), first, row_start};
  const VisualState st{q, t, X};
  const int64_t nnz = trk_ptr[Tv], n6 = (int64_t)n_rows * 6;
  HostExec ex;
  HostExec::Buf<double> obs, params, cost, gmax, c0, p0;
  obs.alloc((size_t)nnz * vbig::kObs); params.alloc((size_t)Tv * kTrkParams);
  cost.alloc((size_t)Tv); gmax.alloc((size_t)Tv); c0.alloc((size_t)std::max<int64_t>(n6, 1)); p0.alloc((size_t)Tv * 3);
  // Jacobi scale
  ex.fill_zero(c0.p, (size_t)n6);
  if (loss) {
    ex.for_each(nnz, vbig::ColObsPass<false, true>{vv, bv, st, obs.p, c0.p});
    ex.for_each(Tv, vbig::ColTrackPass<true>{vv, bv, st, obs.p, p0.p});
  } else {
    ex.for_each(nnz, vbig::ColObsF{vv, bv, st, obs.p, c0.p});
    ex.for_each(Tv, vbig::ColTrackF{vv, bv, st, obs.p, p0.p});
  }
  std::vector<double> s_cam((size_t)std::max<int64_t>(n6, 1)), s_pt((size_t)Tv * 3);
  for (int64_t i = 0; i < n6; ++i) s_cam[i] = jacobi_scaling ? 1.0 / (1.0 + std::sqrt(c0.p[i])) : 1.0;
  for (size_t i = 0; i < s_pt.size(); ++i) s_pt[i] = jacobi_scaling ? 1.0 / (1.0 + std::sqrt(p0.p[i])) : 1.0;
  const VisualLM lm{radius, 1e-6, 1e32, s_cam.data(), s_pt.data()};
  auto reduce = [&](double* o) {
    o[0] = 0.0; o[1] = 0.0;
    for (int64_t b = 0; b < Tv; ++b) { o[0] += cost.p[b]; o[1] = std::fmax(o[1], gmax.p[b]); }
  };
  // explicit
  ex.fill_zero(S, (size_t)row_start[n_rows] * 36);
  ex.fill_zero(rhs_x, (size_t)n6); ex.fill_zero(colsq_x, (size_t)n6); ex.fill_zero(grad_x, (size_t)n6);
  if (loss) {
    ex.for_each(nnz, vbig::ObsPass<true>{vv, bv, st, lm, obs.p});
    ex.for_each(Tv, vbig::TrackPass<true>{vv, bv, st, lm, obs.p, params.p, cost.p, gmax.p});
  } else {
    ex.for_each(nnz, vbig::ObsF{vv, bv, st, lm, obs.p});
    ex.for_each(Tv, vbig::TrackF{vv, bv, st, lm, obs.p, params.p, cost.p, gmax.p});
  }
  ex.for_each(nnz, vbig::SlotsF{vv, bv, params.p, obs.p, S, rhs_x, colsq_x, grad_x});
  ex.for_each(pair_ptr[Tv], vbig::PairsF{vv, bv, obs.p, S});
  reduce(out_x);
  // matrix-free
  std::vector<int64_t> row_ptr, row_obs;
  vimp::row_csr(n_rows, nnz, obs_row, row_ptr, row_obs);
  const int64_t n_free = row_ptr[(size_t)n_rows];
  HostExec::Buf<int> row_trk;
  HostExec::Buf<double> rec, iparams, part, u;
  row_trk.alloc((size_t)std::max<int64_t>(n_free, 1)); rec.alloc((size_t)nnz * vimp::kRec); iparams.alloc((size_t)Tv * kTrkParams);
  part.alloc((size_t)std::max(n_rows, 1) * vimp::kLanes * vimp::kRowOut); u.alloc((size_t)Tv * 6);
  ex.for_each(n_free, vimp::RowTrkF{trk_ptr, Tv, row_obs.data(), row_trk.p});
  const vimp::View iv{Tv, n_rows, row_ptr.data(), row_obs.data(), row_trk.p, rec.p, iparams.p};
  if (loss) {                                                    // the matrix-free plan's own Jacobi scale
    ex.for_each(nnz, vimp::ColObsF<true>{vv, iv, st});
    ex.for_each(Tv, vimp::ColTrkF<true>{vv, iv, st, p0.p});
  } else {
    ex.for_each(nnz, vimp::ColObsF<false>{vv, iv, st});
    ex.for_each(Tv, vimp::ColTrkF<false>{vv, iv, st, p0.p});
  }
  ex.for_each(n6, vimp::ColRowF{iv, c0.p});
  for (int64_t i = 0; i < n6; ++i) s_cam[i] = jacobi_scaling ? 1.0 / (1.0 + std::sqrt(c0.p[i])) : 1.0;
  for (size_t i = 0; i < s_pt.size(); ++i) s_pt[i] = jacobi_scaling ? 1.0 / (1.0 + std::sqrt(p0.p[i])) : 1.0;
  if (loss) {
    ex.for_each(nnz, vimp::ObsF<true>{vv, iv, st, lm});
    ex.for_each(Tv, vimp::TrackF<true>{vv, iv, st, lm, cost.p, gmax.p});
  } else {
    ex.for_each(nnz, vimp::ObsF<false>{vv, iv, st, lm});
    ex.for_each(Tv, vimp::TrackF<false>{vv, iv, st, lm, cost.p, gmax.p});
  }
  ex.for_each((int64_t)n_rows * vimp::kLanes, vimp::RowPartF{iv, part.p});
  ex.for_each((int64_t)n_rows * vimp::kRowOut, vimp::RowSumF{part.p, rhs, colsq, grad, D});
  reduce(out);
  // the product and the solve
  HostExec::Buf<double> vec, minv, cpart, sd;
  HostExec::Buf<int> si;
  vec.alloc((size_t)(4 * n6)); minv.alloc((size_t)(6 * n6)); cpart.alloc((size_t)vpcg::chunks(n6) + 1);
  sd.alloc(vpcg::kNDouble); si.alloc(vpcg::kNInt);
  const vpcg::Bufs B{vec.p, vec.p + n6, vec.p + 2 * n6, vec.p + 3 * n6, minv.p, vpcg::Ctl{si.p, sd.p, cpart.p}};
  auto prod = [&](const double* in, double* o) {
    ex.for_each(Tv, vimp::ProdTrackF{B.c, iv, trk_ptr, obs_row, in, u.p});
    return ex.for_each(n_rows, vimp::ProdRowF{B.c, iv, dadd, in, u.p, o});
  };
  si.p[vpcg::kDone] = 0;
  prod(x, y);
  int h[vpcg::kNInt];
  int64_t d2h = 0;
  vpcg::solve_with(ex, n_rows, vpcg::PrecDF{D, dadd, B.minv, B.c}, rhs, x_sol, B, vpcg::Params{eta, min_iter, max_iter}, prod, h, &d2h);
  info[0] = h[vpcg::kIter];
  info[1] = h[vpcg::kTerm];
}
