// visual_implicit.h — the matrix-free reduced camera system of ITERATIVE_SCHUR (visual_pcg.h): the product y = (S + diag(dadd)) x
// through the Jacobian blocks, without forming S, as Ceres' ImplicitSchurComplement does for ITERATIVE_SCHUR with
// use_explicit_schur_complement = false.  With E_o = J_c^T J_X of observation o and C_l the damped point block of landmark l,
//
//   S = sum_o J_c^T J_c - sum_l (sum_{o in l} E_o) C_l^-1 (sum_{o in l} E_o)^T
//   u_l = C_l^-1 sum_{o in l} J_X^T (J_c x_row(o))                          (ProdTrackF; double-double, see DD below)
//   y_r = sum_{o in r} J_c^T (J_c x_r - J_X u_l(o)) + dadd_r o x_r           (ProdRowF)
//
// so a product costs O(observations), where the explicit S costs O(sum K^2) to build.  visual_matrix_free (below) chooses
// between the two from the plan's counts.  The linearisation of a matrix-free pass produces what the rest of the pass reads:
//
//   ObsF       (one item per observation)   r, J_c (zero for a constant camera) and J_X, scaled and loss-corrected, and the
//                                           observation's cost term -> rec [nnz][kRec]
//   TrackF     (one item per landmark)      C, C^-1, g_p, w = C^-1 g_p (kTrkParams layout, vbig::landmark_step), the landmark's
//                                           cost and max |g_p| into its partial slots
//   RowPartF   (kLanes items per row)       lane j of camera row r: the observations at positions j, j + kLanes, ... of the
//                                           row's list that start a landmark's run in it, each with the whole run: rhs, the
//                                           column norms, the gradient and the diagonal block
//                                           D_r = sum_o J_c^T J_c - sum_runs E_run C^-1 E_run^T, E_run = sum_{o in run} E_o
//   RowSumF    (kRowOut items per row)      the lanes' partials in lane order -> rhs, cam_colsq, cam_grad, D [n_rows][36]
//
// and the Jacobi scale's column norms without atomics (ColObsF, ColRowF, ColTrkF).
// The row CSR lists the observations of every row in ascending order.  The local CSR is landmark-major, so the observations
// of one landmark in one row (a camera it sees more than once) are contiguous there: a run.  Every sum runs in a fixed order
// and nothing uses atomics, so the matrix-free pass has the same bits on every run.  Functors over index ranges, launched by
// visual_api.cuh and, for the CPU checks, by tests/emu/visual_implicit_emu.cpp.  The device's product runs the kernels of
// visual_api.cuh (a lane group per landmark, a warp per row) on the per-observation terms below; ProdTrackF / ProdRowF give the
// same terms in observation order.
#pragma once
#include <vector>

#include "visual_big.h"
#include "visual_pcg.h"

namespace lvba {
namespace vimp {

// per observation: r (2), J_c (12), J_X (6) where vbig's records hold them (so vbig::BacksubPass reads these records), the
// cost term (r^2 or rho), pad
constexpr int kRec = 24, kRecCost = 20;
static_assert(vbig::kObR == 0 && vbig::kObJc == 2 && vbig::kObJX == 14, "the records share vbig's offsets");
constexpr int kLanes = 32;                           // lanes of one camera row in RowPartF
constexpr int kRowOut = 39;                          // per lane: rhs (6) | column norms (6) | gradient (6) | D's lower triangle (21)

// index of (a, b), a >= b, in a lower triangle stored row by row
LVBA_BHD int tri(int a, int b) { return a * (a + 1) / 2 + b; }

struct View {
  int64_t Tv;                // local landmarks
  int n_rows;
  const int64_t* row_ptr;    // [n_rows + 1] the row CSR: the observations of row r are row_obs[row_ptr[r] .. row_ptr[r + 1])
  const int64_t* row_obs;    //   in ascending order
  const int* row_trk;        //   and their local landmarks
  double* rec;               // [nnz][kRec]
  double* params;            // [Tv][kTrkParams]
};

// The row CSR of a plan from the camera row of every local observation (-1: constant): ptr [n_rows + 1], and obs, the
// observations of every row in ascending order (host; the library's visual_row_csr and the CPU tests)
inline void row_csr(int n_rows, int64_t nnz, const int* obs_row, std::vector<int64_t>& ptr, std::vector<int64_t>& obs) {
  ptr.assign((size_t)n_rows + 1, 0);
  for (int64_t w = 0; w < nnz; ++w)
    if (obs_row[w] >= 0) ++ptr[(size_t)obs_row[w] + 1];
  for (int r = 0; r < n_rows; ++r) ptr[(size_t)r + 1] += ptr[(size_t)r];
  obs.resize((size_t)ptr[(size_t)n_rows]);
  std::vector<int64_t> at(ptr.begin(), ptr.end() - 1);
  for (int64_t w = 0; w < nnz; ++w)
    if (obs_row[w] >= 0) obs[(size_t)at[(size_t)obs_row[w]]++] = w;
}

// The choice of the product for a plan of ITERATIVE_SCHUR: true for the matrix-free one.  Per LM pass the explicit product
// costs its build, a sum over every camera-pair contribution to S (n_pairs), plus the envelope it zeroes and reads once per
// CG iteration (n_blocks_env blocks); the matrix-free one costs a pass over the free observations (free_obs) plus two reads
// of their Jacobian records per CG iteration.  The rule compares n_pairs + kBlockWeight n_blocks_env with kObsRatio free_obs.
// Measured on an NVIDIA H100 80GB HBM3 at 700 W, tools/bench_visual_implicit.py with both products, LM passes/s at Ceres'
// defaults (the ratio is (n_pairs + 8 n_blocks_env) / free_obs):
//   config C                          ratio  3.1   explicit 477   matrix-free 255   -> explicit
//   config C + 200 long tracks        ratio   87   explicit  22   matrix-free 184   -> matrix-free
//   loop-closed, 400 cameras          ratio  662   explicit 341   matrix-free 654   -> matrix-free
//   street, 400 cameras, long tracks  ratio  128   explicit 126   matrix-free 226   -> matrix-free
// kObsRatio = 16 sits between the two sides (DESIGN.md §5.9).  n_rows = 0: nothing to solve, explicit.
inline bool visual_matrix_free(int64_t free_obs, int64_t n_pairs, int64_t n_blocks_env, int n_rows) {
  constexpr double kBlockWeight = 8.0, kObsRatio = 16.0;
  if (n_rows <= 0 || free_obs <= 0) return false;
  return (double)n_pairs + kBlockWeight * (double)n_blocks_env > kObsRatio * (double)free_obs;
}

// One observation s of local landmark k at the state st: r, J_c and J_X (kLoss: corrected; returns rho(|r|^2), else 0), J_X
// times s_pt, J_c times s_cam, zero for a constant / unused camera (no columns).  vbig::ObsPass, step for step.
template <bool kLoss>
LVBA_BHD double obs_scaled(const VisualView& vv, const VisualState& st, const VisualLM& lm, int64_t s, int64_t k, ObsEval& o) {
  const int64_t tr = vv.trk_id[k];
  const int cam = vv.obs_cam[s], row = vv.obs_row[s];
  const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
  obs_eval<true>(vv, st.q + 4 * (int64_t)cam, st.t + 3 * (int64_t)cam, X, vv.obs_uv[s], o);
  double rho = 0.0;
  if constexpr (kLoss) rho = obs_loss<true>(vv, o);
  const double* sp = lm.s_pt + 3 * k;
  for (int r = 0; r < 2; ++r)
    for (int m = 0; m < 3; ++m) o.JX[3 * r + m] *= sp[m];
  if (row >= 0) {
    const double* sc = lm.s_cam + 6 * (int64_t)row;
    for (int r = 0; r < 2; ++r)
      for (int a = 0; a < 6; ++a) o.Jc[6 * r + a] *= sc[a];
  } else {
    for (int a = 0; a < 12; ++a) o.Jc[a] = 0.0;          // constant / unused camera: no columns
  }
  return rho;
}

template <bool kLoss>
struct ObsF {                  // one item per observation s of the local CSR
  VisualView vv; View iv; VisualState st; VisualLM lm;
  LVBA_BHD void operator()(int64_t s) const {
    const vbig::View all{iv.Tv, 0, nullptr, nullptr, nullptr};
    ObsEval o;
    const double rho = obs_scaled<kLoss>(vv, st, lm, s, vbig::track_of(vv, all, s), o);
    double* f = iv.rec + kRec * s;
    f[vbig::kObR] = o.r[0]; f[vbig::kObR + 1] = o.r[1];
    for (int a = 0; a < 12; ++a) f[vbig::kObJc + a] = o.Jc[a];
    for (int a = 0; a < 6; ++a) f[vbig::kObJX + a] = o.JX[a];
    f[kRecCost] = kLoss ? rho : o.r[0] * o.r[0] + o.r[1] * o.r[1];
  }
};

template <bool kLoss>
struct TrackF {                // one item per local landmark k; cost[k] = 1/2 sum r^2 (kLoss: 1/2 sum rho), gmax[k] = max |g_p|
  VisualView vv; View iv; VisualState st; VisualLM lm; double* cost; double* gmax;
  LVBA_BHD void operator()(int64_t k) const {
    const int64_t tr = vv.trk_id[k];
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    double acc[9], c = 0.0;
    for (int q = 0; q < 9; ++q) acc[q] = 0.0;
    for (int64_t s = vv.trk_ptr[k]; s < vv.trk_ptr[k + 1]; ++s) {
      const double* f = iv.rec + kRec * s;
      const double* JX = f + vbig::kObJX; const double* r = f + vbig::kObR;
      c += f[kRecCost];
      acc[0] += JX[0] * JX[0] + JX[3] * JX[3]; acc[1] += JX[0] * JX[1] + JX[3] * JX[4]; acc[2] += JX[0] * JX[2] + JX[3] * JX[5];
      acc[3] += JX[1] * JX[1] + JX[4] * JX[4]; acc[4] += JX[1] * JX[2] + JX[4] * JX[5]; acc[5] += JX[2] * JX[2] + JX[5] * JX[5];
      acc[6] += JX[0] * r[0] + JX[3] * r[1]; acc[7] += JX[1] * r[0] + JX[4] * r[1]; acc[8] += JX[2] * r[0] + JX[5] * r[1];
    }
    vbig::landmark_step<kLoss>(vv, lm, k, X, acc, c, iv.params, cost, gmax, k);
  }
};

struct RowPartF {              // one item per (row, lane): part[kRowOut (kLanes r + lane) ..]
  View iv; double* part;
  LVBA_BHD void operator()(int64_t i) const {
    const int64_t r = i / kLanes, lane = i - r * kLanes;
    const int64_t lo = iv.row_ptr[r], hi = iv.row_ptr[r + 1];
    double acc[kRowOut];
    for (int m = 0; m < kRowOut; ++m) acc[m] = 0.0;
    for (int64_t p = lo + lane; p < hi; p += kLanes) {
      const int l = iv.row_trk[p];
      if (p > lo && iv.row_trk[p - 1] == l) continue;          // not the start of the run of landmark l in this row
      double E[18];
      for (int m = 0; m < 18; ++m) E[m] = 0.0;
      for (int64_t q = p; q < hi && iv.row_trk[q] == l; ++q) {
        const double* f = iv.rec + kRec * iv.row_obs[q];
        const double* Jc = f + vbig::kObJc; const double* JX = f + vbig::kObJX; const double* rr = f + vbig::kObR;
        for (int a = 0; a < 6; ++a) {
          const double gc = Jc[a] * rr[0] + Jc[6 + a] * rr[1];
          acc[a] -= gc;
          acc[6 + a] += Jc[a] * Jc[a] + Jc[6 + a] * Jc[6 + a];
          acc[12 + a] += gc;
          for (int b = 0; b <= a; ++b) acc[18 + tri(a, b)] += Jc[a] * Jc[b] + Jc[6 + a] * Jc[6 + b];
          for (int m = 0; m < 3; ++m) E[3 * a + m] += Jc[a] * JX[m] + Jc[6 + a] * JX[3 + m];
        }
      }
      const double* pp = iv.params + kTrkParams * (int64_t)l;
      const double Ci[9] = {pp[0], pp[1], pp[2], pp[1], pp[3], pp[4], pp[2], pp[4], pp[5]};
      for (int a = 0; a < 6; ++a) {
        acc[a] += E[3 * a] * pp[9] + E[3 * a + 1] * pp[10] + E[3 * a + 2] * pp[11];
        double Y[3];
        for (int m = 0; m < 3; ++m) Y[m] = E[3 * a] * Ci[m] + E[3 * a + 1] * Ci[3 + m] + E[3 * a + 2] * Ci[6 + m];
        for (int b = 0; b <= a; ++b) acc[18 + tri(a, b)] -= Y[0] * E[3 * b] + Y[1] * E[3 * b + 1] + Y[2] * E[3 * b + 2];
      }
    }
    double* o = part + kRowOut * i;
    for (int m = 0; m < kRowOut; ++m) o[m] = acc[m];
  }
};

struct RowSumF {               // one item per (row, output): the lanes' partials in lane order
  const double* part; double* rhs; double* cam_colsq; double* cam_grad; double* D;
  LVBA_BHD void operator()(int64_t j) const {
    const int64_t r = j / kRowOut;
    const int m = (int)(j - r * kRowOut);
    const double* p = part + kRowOut * kLanes * r + m;
    double v = 0.0;
    for (int lane = 0; lane < kLanes; ++lane) v += p[kRowOut * lane];
    if (m < 6) rhs[6 * r + m] = v;
    else if (m < 12) cam_colsq[6 * r + m - 6] = v;
    else if (m < 18) cam_grad[6 * r + m - 12] = v;
    else {
      int a = 0;
      while (tri(a + 1, 0) <= m - 18) ++a;
      const int b = m - 18 - tri(a, 0);
      D[36 * r + 6 * a + b] = v;
      D[36 * r + 6 * b + a] = v;
    }
  }
};

// The column norms of the Jacobi scale (Ceres: once, at iteration 0) on a matrix-free plan, every sum in a fixed order, as the
// unscaled squared column norms of vbig::ColObsPass / ColTrackPass: ColObsF writes each observation's (J_c: 6, J_X: 3) into
// its record, ColRowF sums a row's in the row CSR's order, ColTrkF a landmark's after its plane term in observation order
template <bool kLoss>
struct ColObsF {               // one item per observation s of the local CSR
  VisualView vv; View iv; VisualState st;
  LVBA_BHD void operator()(int64_t s) const {
    const vbig::View all{iv.Tv, 0, nullptr, nullptr, nullptr};
    const int64_t tr = vv.trk_id[vbig::track_of(vv, all, s)];
    const int cam = vv.obs_cam[s];
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    ObsEval o;
    obs_eval<true>(vv, st.q + 4 * (int64_t)cam, st.t + 3 * (int64_t)cam, X, vv.obs_uv[s], o);
    if constexpr (kLoss) obs_loss<true>(vv, o);
    double* f = iv.rec + kRec * s;
    for (int a = 0; a < 6; ++a) f[a] = o.Jc[a] * o.Jc[a] + o.Jc[6 + a] * o.Jc[6 + a];
    for (int m = 0; m < 3; ++m) f[6 + m] = o.JX[m] * o.JX[m] + o.JX[3 + m] * o.JX[3 + m];
  }
};
struct ColRowF {               // one item per (row, column)
  View iv; double* cam_colsq;
  LVBA_BHD void operator()(int64_t j) const {
    const int64_t r = j / 6;
    const int a = (int)(j - 6 * r);
    double v = 0.0;
    for (int64_t p = iv.row_ptr[r]; p < iv.row_ptr[r + 1]; ++p) v += iv.rec[kRec * iv.row_obs[p] + a];
    cam_colsq[j] = v;
  }
};
template <bool kLoss>
struct ColTrkF {               // one item per local landmark
  VisualView vv; View iv; VisualState st; double* pt_colsq;
  LVBA_BHD void operator()(int64_t k) const {
    const int64_t tr = vv.trk_id[k];
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    double rp, J[3];
    plane_eval(vv, vv.plane + 4 * k, X, rp, J);
    if constexpr (kLoss) plane_loss(vv, rp, J);
    double a[3] = {J[0] * J[0], J[1] * J[1], J[2] * J[2]};
    for (int64_t s = vv.trk_ptr[k]; s < vv.trk_ptr[k + 1]; ++s)
      for (int m = 0; m < 3; ++m) a[m] += iv.rec[kRec * s + 6 + m];
    for (int m = 0; m < 3; ++m) pt_colsq[3 * k + m] = a[m];
  }
};

// the landmark of every entry of the row CSR (the last landmark whose observations start at or before it)
struct RowTrkF {
  const int* trk_ptr; int64_t Tv; const int64_t* row_obs; int* row_trk;
  LVBA_BHD void operator()(int64_t p) const {
    const int64_t s = row_obs[p];
    int64_t lo = 0, hi = Tv;
    while (hi - lo > 1) { const int64_t m = (lo + hi) >> 1; if (trk_ptr[m] <= s) lo = m; else hi = m; }
    row_trk[p] = (int)lo;
  }
};

// ---- the product's terms, per observation record f, in double-double arithmetic (hi + lo, Dekker / Knuth error-free
// transformations, as in Hida, Li and Bailey's QD library).  The explicit S is one symmetric matrix, rounded once; a product
// through the Jacobian blocks rounds inside every application, and on a long track the terms J_c x and J_X u nearly cancel
// along the system's small eigenvectors.  Rounded in double, that makes the operator slightly non-symmetric and non-linear, and
// a CG run on long past convergence (a forced iteration count at a tiny eta) then drifts away from the solution.  In
// double-double every product is the exact operator of the rounded records (symmetric and linear) rounded once at the end.
struct DD { double hi, lo; };
LVBA_BHD DD dd_quick(double a, double b) { const double s = a + b; return DD{s, b - (s - a)}; }      // |a| >= |b|
LVBA_BHD DD dd_two_sum(double a, double b) {
  const double s = a + b, bb = s - a;
  return DD{s, (a - (s - bb)) + (b - bb)};
}
LVBA_BHD DD dd_add(DD a, DD b) {
  const DD s = dd_two_sum(a.hi, b.hi);
  return dd_quick(s.hi, s.lo + (a.lo + b.lo));
}
// acc + x c
LVBA_BHD DD dd_fma(DD acc, DD x, double c) {
  const double p = x.hi * c;
  const double pe = fma(x.hi, c, -p) + x.lo * c;
  const DD s = dd_two_sum(acc.hi, p);
  return dd_quick(s.hi, s.lo + (pe + acc.lo));
}
LVBA_BHD DD dd_fma(DD acc, double x, double c) { return dd_fma(acc, DD{x, 0.0}, c); }

// J_c x_r (2) of one record
LVBA_BHD void jc_x(const double* Jc, const double* xr, DD j[2]) {
  j[0] = DD{0.0, 0.0}; j[1] = DD{0.0, 0.0};
  for (int a = 0; a < 6; ++a) { j[0] = dd_fma(j[0], Jc[a], xr[a]); j[1] = dd_fma(j[1], Jc[6 + a], xr[a]); }
}
// a += J_X^T (J_c x_r)
LVBA_BHD void track_term(const double* f, const double* xr, DD a[3]) {
  const double* JX = f + vbig::kObJX;
  DD j[2];
  jc_x(f + vbig::kObJc, xr, j);
  for (int m = 0; m < 3; ++m) a[m] = dd_fma(dd_fma(a[m], j[0], JX[m]), j[1], JX[3 + m]);
}
// u = C^-1 a (C^-1 of the landmark's params), u [6]: hi, lo of each component
LVBA_BHD void track_finish(const double* p, const DD a[3], double* u) {
  const double Ci[9] = {p[0], p[1], p[2], p[1], p[3], p[4], p[2], p[4], p[5]};
  for (int m = 0; m < 3; ++m) {
    DD v{0.0, 0.0};
    for (int k = 0; k < 3; ++k) v = dd_fma(v, a[k], Ci[3 * m + k]);
    u[2 * m] = v.hi; u[2 * m + 1] = v.lo;
  }
}
// acc += J_c^T (J_c x_r - J_X u), u [6] as track_finish writes it
LVBA_BHD void row_term(const double* f, const double* xr, const double* u, DD acc[6]) {
  const double* Jc = f + vbig::kObJc; const double* JX = f + vbig::kObJX;
  DD j[2];
  jc_x(Jc, xr, j);
  for (int m = 0; m < 3; ++m) {
    const DD um{u[2 * m], u[2 * m + 1]};
    j[0] = dd_fma(j[0], um, -JX[m]);
    j[1] = dd_fma(j[1], um, -JX[3 + m]);
  }
  for (int a = 0; a < 6; ++a) acc[a] = dd_fma(dd_fma(acc[a], j[0], Jc[a]), j[1], Jc[6 + a]);
}
// y_r = acc + dadd_r o x_r, rounded once
LVBA_BHD double row_finish(DD acc, double dadd, double x) { const DD v = dd_fma(acc, dadd, x); return v.hi + v.lo; }

struct ProdTrackF {            // one item per landmark: u [Tv][6]
  vpcg::Ctl c; View iv; const int* trk_ptr; const int* obs_row; const double* x; double* u;
  LVBA_BHD void operator()(int64_t k) const {
    if (c.done()) return;
    DD a[3] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
    for (int64_t s = trk_ptr[k]; s < trk_ptr[k + 1]; ++s) {
      const int row = obs_row[s];
      if (row >= 0) track_term(iv.rec + kRec * s, x + 6 * (int64_t)row, a);
    }
    track_finish(iv.params + kTrkParams * k, a, u + 6 * k);
  }
};

struct ProdRowF {              // one item per camera row: y_r
  vpcg::Ctl c; View iv; const double* dadd; const double* x; const double* u; double* y;
  LVBA_BHD void operator()(int64_t r) const {
    if (c.done()) return;
    DD acc[6] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
    const double* xr = x + 6 * r;
    for (int64_t p = iv.row_ptr[r]; p < iv.row_ptr[r + 1]; ++p)
      row_term(iv.rec + kRec * iv.row_obs[p], xr, u + 6 * (int64_t)iv.row_trk[p], acc);
    for (int a = 0; a < 6; ++a) y[6 * r + a] = row_finish(acc[a], dadd[6 * r + a], xr[a]);
  }
};

}  // namespace vimp
}  // namespace lvba
