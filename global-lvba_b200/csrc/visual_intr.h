// visual_intr.h — the shared camera intrinsics (fx fy cx cy k1 k2 p1 p2) as one variable parameter block of the visual LM
// (lvba_visual_opts::refine_intrinsics): ceres::Problem with the intrinsics a parameter block of size 8 of every
// ReprojErrorWhitenedDistorted (reference include/utils.hpp:51-111), a SubsetManifold holding the entries whose bit is clear.
//
// The camera system of visual.cuh / visual_big.h is built as it is without the block.  The block borders it: with J_k the
// 2x8 intrinsics Jacobian of an observation (intr_jac, Jacobi-scaled, zero in the held entries), V_t, W_o = J_c^T J_X and
// E_t = sum_{o in t} J_k^T J_X,
//   B_c  = sum_{o in c} (J_c^T J_k - W_o V_t^-1 E_t^T)                          6x8 per camera row
//   C    = sum_o J_k^T J_k - sum_t E_t V_t^-1 E_t^T                             8x8
//   rhs_k = -(g_k - sum_t E_t V_t^-1 g_X,t)
// and the back-substitution becomes dX_t = V_t^-1 (-g_X,t - sum_o W_o^T dc - E_t^T dk).
//
//   TrackF     (one item per local landmark)  V_t^-1, E_t; the landmark's terms of C, rhs_k, the intrinsics column norms and
//                                             gradient into its slot [kSys]; each observation's B contribution into its own
//                                             record [kRec] (camera rows only)
//   ReduceF    (one item per chunk column)    the slots summed in landmark order, a chunk at a time
//   RowGatherF (one item per row element)     each row's records summed in observation order into the border, column-major
//   ColF, ScaleF                              the unscaled column norms and the Jacobi scale of the block
//   BacksubF   (one item per local landmark)  dX_t, the candidate landmark and the model cost change of its residuals
// Every sum runs in a fixed order, so the block's terms have the same bits on every run.  The passes recompute each landmark's
// residuals observation by observation inside one item, tile and big landmarks alike.  Functors over index ranges, launched by
// visual_api.cuh.
#pragma once
#include "lidar_big.h"     // LVBA_BHD
#include "visual_math.h"

namespace lvba {
namespace vintr {

// per-landmark slot: C (upper triangle of 8x8, row by row), rhs_k, squared column norms, gradient J_k^T r (all Jacobi-scaled)
constexpr int kC = 0, kRhs = 36, kCol = 44, kGrad = 52, kSys = 60;
constexpr int kRec = 48;           // per observation: its 6x8 contribution to B_c, row-major

LVBA_BHD int ut(int i, int j) { return i * 8 - i * (i - 1) / 2 + (j - i); }   // (i, j), i <= j, in the upper triangle

// r, J_c, J_X of obs_eval and J_k of intr_jac for observation s of local landmark k, corrected by the reprojection loss (kLoss).
// kScaled: J_X times s_pt, J_c times s_cam (zero for a constant camera), J_k times sk (zero in the held entries).
template <bool kLoss, bool kScaled>
LVBA_BHD void obs_full(const VisualView& vv, const VisualState& st, const VisualLM& lm, const double* sk, int64_t k, int64_t s,
                       ObsEval& o, double Jk[16], int& row) {
  const int64_t tr = vv.trk_id[k], cam = vv.obs_cam[s];
  row = vv.obs_row[s];
  const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
  obs_eval<true>(vv, st.q + 4 * cam, st.t + 3 * cam, X, vv.obs_uv[s], o);
  intr_jac(vv, st.q + 4 * cam, st.t + 3 * cam, X, Jk);
  if constexpr (kLoss) {
    double rho, rho1;
    loss_eval(vv.loss_px, vv.loss_a_px, o.r[0] * o.r[0] + o.r[1] * o.r[1], rho, rho1);
    const double w = sqrt(rho1);
    obs_loss<true>(vv, o);
    for (int i = 0; i < 16; ++i) Jk[i] *= w;
  }
  if constexpr (kScaled) {
    const double* sp = lm.s_pt + 3 * k;
    for (int rho = 0; rho < 2; ++rho)
      for (int m = 0; m < 3; ++m) o.JX[3 * rho + m] *= sp[m];
    if (row >= 0) {
      const double* sc = lm.s_cam + 6 * (int64_t)row;
      for (int rho = 0; rho < 2; ++rho)
        for (int a = 0; a < 6; ++a) o.Jc[6 * rho + a] *= sc[a];
    } else {
      for (int a = 0; a < 12; ++a) o.Jc[a] = 0.0;
    }
    for (int i = 0; i < 8; ++i) { Jk[i] *= sk[i]; Jk[8 + i] *= sk[i]; }
  }
}

// the landmark block of visual_front: Vi = (sum J_X^T J_X + plane term + LM diagonal)^-1 (sym3_inverse layout), g = J_X^T r
template <bool kLoss>
LVBA_BHD void point_block(const VisualView& vv, const VisualState& st, const VisualLM& lm, const double* sk, int64_t k,
                          double Vi[6], double g[3]) {
  double acc[9];
  for (int q = 0; q < 9; ++q) acc[q] = 0.0;
  ObsEval o;
  double Jk[16];
  int row;
  for (int64_t s = vv.trk_ptr[k]; s < vv.trk_ptr[k + 1]; ++s) {
    obs_full<kLoss, true>(vv, st, lm, sk, k, s, o, Jk, row);
    acc[0] += o.JX[0] * o.JX[0] + o.JX[3] * o.JX[3];
    acc[1] += o.JX[0] * o.JX[1] + o.JX[3] * o.JX[4];
    acc[2] += o.JX[0] * o.JX[2] + o.JX[3] * o.JX[5];
    acc[3] += o.JX[1] * o.JX[1] + o.JX[4] * o.JX[4];
    acc[4] += o.JX[1] * o.JX[2] + o.JX[4] * o.JX[5];
    acc[5] += o.JX[2] * o.JX[2] + o.JX[5] * o.JX[5];
    acc[6] += o.JX[0] * o.r[0] + o.JX[3] * o.r[1];
    acc[7] += o.JX[1] * o.r[0] + o.JX[4] * o.r[1];
    acc[8] += o.JX[2] * o.r[0] + o.JX[5] * o.r[1];
  }
  const int64_t tr = vv.trk_id[k];
  const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
  double rp, Jpl[3];
  plane_eval(vv, vv.plane + 4 * k, X, rp, Jpl);
  if constexpr (kLoss) plane_loss(vv, rp, Jpl);
  const double* sp = lm.s_pt + 3 * k;
  Jpl[0] *= sp[0]; Jpl[1] *= sp[1]; Jpl[2] *= sp[2];
  acc[0] += Jpl[0] * Jpl[0]; acc[1] += Jpl[0] * Jpl[1]; acc[2] += Jpl[0] * Jpl[2];
  acc[3] += Jpl[1] * Jpl[1]; acc[4] += Jpl[1] * Jpl[2]; acc[5] += Jpl[2] * Jpl[2];
  acc[6] += Jpl[0] * rp; acc[7] += Jpl[1] * rp; acc[8] += Jpl[2] * rp;
  const double ir = 1.0 / lm.radius;
  acc[0] += fmin(fmax(acc[0], lm.min_diag), lm.max_diag) * ir;
  acc[3] += fmin(fmax(acc[3], lm.min_diag), lm.max_diag) * ir;
  acc[5] += fmin(fmax(acc[5], lm.min_diag), lm.max_diag) * ir;
  sym3_inverse(acc, Vi);
  g[0] = acc[6]; g[1] = acc[7]; g[2] = acc[8];
}

template <bool kLoss>
struct TrackF {
  VisualView vv; VisualState st; VisualLM lm; const double* sk;
  double* sys;   // [Tv][kSys]
  double* rec;   // [nnz][kRec]
  LVBA_BHD void operator()(int64_t k) const {
    double Vi[6], g[3];
    point_block<kLoss>(vv, st, lm, sk, k, Vi, g);
    double E[24], out[kSys];
    for (int i = 0; i < 24; ++i) E[i] = 0.0;
    for (int i = 0; i < kSys; ++i) out[i] = 0.0;
    ObsEval o;
    double Jk[16];
    int row;
    for (int64_t s = vv.trk_ptr[k]; s < vv.trk_ptr[k + 1]; ++s) {
      obs_full<kLoss, true>(vv, st, lm, sk, k, s, o, Jk, row);
      for (int i = 0; i < 8; ++i) {
        for (int m = 0; m < 3; ++m) E[3 * i + m] += Jk[i] * o.JX[m] + Jk[8 + i] * o.JX[3 + m];
        for (int j = i; j < 8; ++j) out[kC + ut(i, j)] += Jk[i] * Jk[j] + Jk[8 + i] * Jk[8 + j];
        out[kGrad + i] += Jk[i] * o.r[0] + Jk[8 + i] * o.r[1];
        out[kCol + i] += Jk[i] * Jk[i] + Jk[8 + i] * Jk[8 + i];
      }
    }
    const double Ci[9] = {Vi[0], Vi[1], Vi[2], Vi[1], Vi[3], Vi[4], Vi[2], Vi[4], Vi[5]};
    double F[24];                                           // V^-1 E^T (3x8)
    for (int m = 0; m < 3; ++m)
      for (int i = 0; i < 8; ++i) F[8 * m + i] = Ci[3 * m] * E[3 * i] + Ci[3 * m + 1] * E[3 * i + 1] + Ci[3 * m + 2] * E[3 * i + 2];
    const double w[3] = {Ci[0] * g[0] + Ci[1] * g[1] + Ci[2] * g[2], Ci[3] * g[0] + Ci[4] * g[1] + Ci[5] * g[2],
                         Ci[6] * g[0] + Ci[7] * g[1] + Ci[8] * g[2]};
    for (int i = 0; i < 8; ++i) {
      for (int j = i; j < 8; ++j) out[kC + ut(i, j)] -= E[3 * i] * F[j] + E[3 * i + 1] * F[8 + j] + E[3 * i + 2] * F[16 + j];
      out[kRhs + i] = -(out[kGrad + i] - (E[3 * i] * w[0] + E[3 * i + 1] * w[1] + E[3 * i + 2] * w[2]));
    }
    for (int i = 0; i < kSys; ++i) sys[kSys * k + i] = out[i];
    for (int64_t s = vv.trk_ptr[k]; s < vv.trk_ptr[k + 1]; ++s) {
      obs_full<kLoss, true>(vv, st, lm, sk, k, s, o, Jk, row);
      if (row < 0) continue;
      double* rc = rec + kRec * s;
      for (int a = 0; a < 6; ++a) {
        const double W[3] = {o.Jc[a] * o.JX[0] + o.Jc[6 + a] * o.JX[3], o.Jc[a] * o.JX[1] + o.Jc[6 + a] * o.JX[4],
                             o.Jc[a] * o.JX[2] + o.Jc[6 + a] * o.JX[5]};
        for (int i = 0; i < 8; ++i)
          rc[8 * a + i] = o.Jc[a] * Jk[i] + o.Jc[6 + a] * Jk[8 + i] - (W[0] * F[i] + W[1] * F[8 + i] + W[2] * F[16 + i]);
      }
    }
  }
};

// out[c][j] = sum of in[r][j] over the rows r of chunk c ([c chunk, (c + 1) chunk) within n), in row order.  Item c * W + j.
struct ReduceF {
  const double* in; int64_t n, chunk; int W; double* out;
  LVBA_BHD void operator()(int64_t i) const {
    const int64_t c = i / W, j = i - c * W;
    const int64_t r1 = (c + 1) * chunk < n ? (c + 1) * chunk : n;
    double v = 0.0;
    for (int64_t r = c * chunk; r < r1; ++r) v += in[r * W + j];
    out[i] = v;
  }
};

// B (column-major, [8][n6]): item r * kRec + e sums element e of the records of row r's observations (row_obs[row_ptr[r] ..
// row_ptr[r + 1]), ascending) into B[i][6 r + a], e = 8 a + i
struct RowGatherF {
  const int64_t* row_ptr; const int64_t* row_obs; const double* rec; int64_t n6; double* B;
  LVBA_BHD void operator()(int64_t it) const {
    const int64_t r = it / kRec, e = it - r * kRec, a = e / 8, i = e - a * 8;
    double v = 0.0;
    for (int64_t q = row_ptr[r]; q < row_ptr[r + 1]; ++q) v += rec[kRec * row_obs[q] + e];
    B[i * n6 + 6 * r + a] = v;
  }
};

// unscaled squared column norms of J_k, per landmark: out[8 k + i]
template <bool kLoss>
struct ColF {
  VisualView vv; VisualState st; double* out;
  LVBA_BHD void operator()(int64_t k) const {
    double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    ObsEval o;
    double Jk[16];
    int row;
    const VisualLM lm{1.0, 0.0, 0.0, nullptr, nullptr};
    for (int64_t s = vv.trk_ptr[k]; s < vv.trk_ptr[k + 1]; ++s) {
      obs_full<kLoss, false>(vv, st, lm, nullptr, k, s, o, Jk, row);
      for (int i = 0; i < 8; ++i) acc[i] += Jk[i] * Jk[i] + Jk[8 + i] * Jk[8 + i];
    }
    for (int i = 0; i < 8; ++i) out[8 * k + i] = acc[i];
  }
};

// sk[i] = 1 / (1 + sqrt(colsq[i])) (1 when Jacobi scaling is off) for a free entry, 0 for a held one
struct ScaleF {
  const double* colsq; unsigned mask; int enabled; double* sk;
  LVBA_BHD void operator()(int64_t i) const {
    sk[i] = ((mask >> i) & 1u) ? (enabled ? 1.0 / (1.0 + sqrt(colsq[i])) : 1.0) : 0.0;
  }
};

// dX_t = -V^-1 (g_X + sum_o J_X^T (J_c y_c + J_k y_k)), the candidate landmark, its step and the model cost change
// -(J~ y)^T (r + 1/2 J~ y) of its residuals: out[3 k] = model, step^2, x^2.  y_cam, yk: the scaled steps.
template <bool kLoss>
struct BacksubF {
  VisualView vv; VisualState st; VisualLM lm; const double* sk; const double* y_cam; double yk[8];
  double* X_cand; double* pt_step; double* out;
  LVBA_BHD void jy_cam(const ObsEval& o, const double Jk[16], int row, double& j0, double& j1) const {
    j0 = 0.0; j1 = 0.0;
    if (row >= 0)
      for (int a = 0; a < 6; ++a) { const double y = y_cam[6 * (int64_t)row + a]; j0 += o.Jc[a] * y; j1 += o.Jc[6 + a] * y; }
    for (int i = 0; i < 8; ++i) { j0 += Jk[i] * yk[i]; j1 += Jk[8 + i] * yk[i]; }
  }
  LVBA_BHD void operator()(int64_t k) const {
    double Vi[6], g[3];
    point_block<kLoss>(vv, st, lm, sk, k, Vi, g);
    ObsEval o;
    double Jk[16];
    int row;
    double a[3] = {0.0, 0.0, 0.0};
    for (int64_t s = vv.trk_ptr[k]; s < vv.trk_ptr[k + 1]; ++s) {
      obs_full<kLoss, true>(vv, st, lm, sk, k, s, o, Jk, row);
      double j0, j1;
      jy_cam(o, Jk, row, j0, j1);
      for (int m = 0; m < 3; ++m) a[m] += o.JX[m] * j0 + o.JX[3 + m] * j1;
    }
    const double b[3] = {g[0] + a[0], g[1] + a[1], g[2] + a[2]};
    const double yp[3] = {-(Vi[0] * b[0] + Vi[1] * b[1] + Vi[2] * b[2]), -(Vi[1] * b[0] + Vi[3] * b[1] + Vi[4] * b[2]),
                          -(Vi[2] * b[0] + Vi[4] * b[1] + Vi[5] * b[2])};
    const int64_t tr = vv.trk_id[k];
    const double* sp = lm.s_pt + 3 * k;
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    const double d[3] = {sp[0] * yp[0], sp[1] * yp[1], sp[2] * yp[2]};
    for (int m = 0; m < 3; ++m) {
      X_cand[3 * tr + m] = X[m] + d[m];
      if (pt_step) pt_step[3 * tr + m] = d[m];
    }
    double model = 0.0;
    double rp, Jpl[3];
    plane_eval(vv, vv.plane + 4 * k, X, rp, Jpl);
    if constexpr (kLoss) plane_loss(vv, rp, Jpl);
    const double jp = Jpl[0] * d[0] + Jpl[1] * d[1] + Jpl[2] * d[2];
    model -= jp * (rp + 0.5 * jp);
    for (int64_t s = vv.trk_ptr[k]; s < vv.trk_ptr[k + 1]; ++s) {
      obs_full<kLoss, true>(vv, st, lm, sk, k, s, o, Jk, row);
      double j0, j1;
      jy_cam(o, Jk, row, j0, j1);
      j0 += o.JX[0] * yp[0] + o.JX[1] * yp[1] + o.JX[2] * yp[2];
      j1 += o.JX[3] * yp[0] + o.JX[4] * yp[1] + o.JX[5] * yp[2];
      model -= j0 * (o.r[0] + 0.5 * j0) + j1 * (o.r[1] + 0.5 * j1);
    }
    out[3 * k] = model;
    out[3 * k + 1] = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
    out[3 * k + 2] = X[0] * X[0] + X[1] * X[1] + X[2] * X[2];
  }
};

// Cholesky solve of the k x k corner S (row-major, overwritten) for r (overwritten by the solution).  false on a pivot that is
// not finite and > 0.
LVBA_BHD bool corner_solve(int k, double* S, double* r) {
  for (int j = 0; j < k; ++j) {
    double d = S[j * k + j];
    for (int m = 0; m < j; ++m) d -= S[j * k + m] * S[j * k + m];
    if (!(d > 0.0 && d <= DBL_MAX)) return false;
    const double l = sqrt(d);
    S[j * k + j] = l;
    for (int i = j + 1; i < k; ++i) {
      double v = S[i * k + j];
      for (int m = 0; m < j; ++m) v -= S[i * k + m] * S[j * k + m];
      S[i * k + j] = v / l;
    }
  }
  for (int i = 0; i < k; ++i) {
    double v = r[i];
    for (int m = 0; m < i; ++m) v -= S[i * k + m] * r[m];
    r[i] = v / S[i * k + i];
  }
  for (int i = k - 1; i >= 0; --i) {
    double v = r[i];
    for (int m = i + 1; m < k; ++m) v -= S[m * k + i] * r[m];
    r[i] = v / S[i * k + i];
  }
  return true;
}

}  // namespace vintr
}  // namespace lvba
