// visual_dogleg.h — Ceres' DOGLEG trust-region strategy for the visual LM (lvba_visual_opts::trust_region_strategy =
// LVBA_TR_DOGLEG), TRADITIONAL_DOGLEG.  Ceres is not part of this repository; the rule below is restated from the
// ceres-solver 2.1.0 sources (DoglegStrategy, TrustRegionMinimizer), as visual_pcg.h restates ITERATIVE_SCHUR and SURVEY.md
// §8 Q9 / Q10 the rest of the LM.  tests/visual_dogleg_oracle.py is the same rule in numpy.
//
// Every quantity lives in the Jacobi-scaled space of the LM: J~ the scaled, loss-corrected Jacobian, f the corrected residuals,
// one entry per free parameter (the camera rows' 6 columns, then every local landmark's 3).
//
//   D     = sqrt(clamp(diag(J~^T J~), min_lm_diagonal, max_lm_diagonal))
//   g     = (J~^T f) / D                                              (ComputeGradient)
//   alpha = |g|^2 / |J~ (g / D)|^2                                    (ComputeCauchyPoint; -alpha g is the Cauchy point)
//   GN    = D o y, y the DENSE_SCHUR step of the LM at radius 1 / mu  (ComputeGaussNewtonStep: the LM diagonal D sqrt(mu);
//           Ceres solves for -y and negates)
//   mu starts at kMinMu.  A solve that fails (a non-zero factorisation status) or a y that is not finite multiplies mu by
//   kMuIncrease and solves again while mu < kMaxMu; when mu reaches kMaxMu without a good solve the step is invalid.  Here a
//   retry is a whole linearisation at the same state (the build runs with the solve): the handle's hessian_builds counts it.
//
// The step, in the D-scaled space, with Delta the radius (ComputeTraditionalDoglegStep):
//   case 1  |GN| <= Delta                 s = GN,                        |s| = |GN|
//   case 2  alpha |g| >= Delta            s = -(Delta / |g|) g,          |s| = Delta
//   case 3  otherwise, with a = -alpha g, b = GN:
//           b.a = -alpha g.GN,  |a|^2 = (alpha |g|)^2,  |b - a|^2 = |a|^2 - 2 b.a + |GN|^2,  c = b.a - |a|^2,
//           d = sqrt(c^2 + |b - a|^2 (Delta^2 - |a|^2)),
//           beta = (d - c) / |b - a|^2 if c <= 0, else (Delta^2 - |a|^2) / (d + c)
//           s = -alpha (1 - beta) g + beta GN,   |s|^2 = (alpha (1 - beta))^2 |g|^2 - 2 alpha (1 - beta) beta g.GN + beta^2 |GN|^2
//           (Ceres takes |s| from the vector; the three terms here are all >= 0, so the two agree to rounding)
// and the trust-region step is s / D, the candidate x [+] (s / D) o jacobi_scale as for the LM.
//
// After the step (TrustRegionMinimizer, then DoglegStrategy::StepAccepted / StepRejected / StepIsInvalid):
//   model  = -(J~ s')^T (f + J~ s' / 2), s' = s / D; the step is invalid unless model > 0 (and, as for the LM here, model and
//            the ambient step norm are finite)
//   invalid   mu *= kMuIncrease, relinearise on the next pass; Delta unchanged.  Five in a row end the solve
//             (LVBA_TERM_INVALID_STEPS), as for the LM.
//   accepted  (rho > min_relative_decrease, finite candidate cost): rho < kDecrease: Delta *= 0.5; rho > kIncrease:
//             Delta = max(Delta, 3 |s|); mu = max(kMinMu, 2 mu / kMuIncrease); relinearise on the next pass.  Delta is NOT
//             clamped to max_radius: Ceres' DoglegStrategy keeps max_radius but never reads it.
//   rejected  Delta *= 0.5 and reuse: the next pass keeps D, g, alpha and GN and only moves the dogleg point (no build, no
//             solve; one J~ v pass and a candidate cost).
//   Delta < min_radius after an accepted or a rejected step ends the solve (LVBA_TERM_RADIUS; Ceres tests the radius after every
//   iteration, and the dogleg's radius also shrinks on an accepted step).  The function, gradient and parameter tolerances, the
//   acceptance test and the cost are the LM's.  The gradient tolerance is tested on a new linearisation only: a rejected step
//   leaves the state, and so the gradient, unchanged.
//
// Passes (functors over index ranges, run by CudaExec on the device and by the host policy in tests/emu/visual_dogleg_emu.cpp).
// Vectors of n = 6 n_rows + 3 Tv entries, the camera rows first:
//   CamF   (one item per camera column)  D, g, GN of the camera rows from the build's column norms and gradient and the solve's y
//   TrkF   (one item per local landmark) the landmark's column norms and J~_X^T f (its observations in order, then its plane),
//                                        D, g, and GN from the back-substitution's pt_step (= s_pt o y_X)
//   DotF   (one item per entry)          g.g, GN.GN, g.GN per entry -> summed by vintr::ReduceF in chunks of 256, then the chunks
//   JvF    (one item per local landmark) |J~ v|^2 and -(J~ v)^T (f + J~ v / 2) over the landmark's observations and plane; with
//                                        Xc, the candidate landmark X + s_pt o v and its step^2, x^2 -> per-landmark records,
//                                        summed as above
//   CaseF  (one item)                    alpha (on a new linearisation), the case, beta, the coefficients of g and GN, |s|
//   StepF  (one item per entry)          v = (c_g g + c_n GN) / D
// The candidate's cameras and its cost are the LM's kernels.  Every sum runs in a fixed order and nothing uses atomics, so in
// deterministic mode a dogleg solve has the same bits on every run.  Recomputing J~ per observation (rather than keeping the
// 24-double records of the matrix-free product) keeps no per-observation memory; DESIGN.md §5.10 has the measured cost.
#pragma once
#include "visual_implicit.h"
#include "visual_intr.h"
#if defined(__CUDACC__)
#include "exec.cuh"
#include "runtime.cuh"
#endif

namespace lvba {
namespace vdog {

constexpr double kMinMu = 1e-8, kMaxMu = 1.0, kMuIncrease = 10.0;   // DoglegStrategy: min_mu_, max_mu_, mu_increase_factor_
constexpr double kDecrease = 0.25, kIncrease = 0.75;               // decrease_threshold_, increase_threshold_
constexpr int kChunk = 256;                                        // rows per partial of the two-level sums

// the step cases (lvba_visual_dogleg_state)
enum Case { kNone = 0, kGaussNewton = 1, kCauchy = 2, kDogleg = 3 };
// device scalars: the sums (g.g, GN.GN, g.GN), alpha, the case, beta, the coefficients of g and GN, |s|, then the four sums of
// the last J~ v pass
enum { kGG = 0, kNN, kGN, kAlpha, kCase, kBeta, kCoefG, kCoefN, kStepNorm, kJv, kNScal = kJv + 4 };
// per-landmark record of JvF: model, step^2, x^2 (the LM's scal[2..4] order), |J~ v|^2
constexpr int kJvRec = 4, kJvModel = 0, kJvStep2 = 1, kJvX2 = 2, kJvSq = 3;

// The per-landmark passes (TrkF, JvF: a loop over the landmark's observations, each recomputing J~): the device runs them at
// 128 threads per CTA (wide_pass), where their registers fit without a spill, the host policy item by item
template <class Exec, class F>
int landmark_pass(Exec& ex, int64_t n, const F& f) { return ex.for_each(n, f); }
#if defined(__CUDACC__)
template <class F>
int landmark_pass(CudaExec& ex, int64_t n, const F& f) {
  wide_pass(ex.stream, n, f, &ex.launches);
  LVBA_CUDA(cudaGetLastError());
  return LVBA_OK;
}
#endif

LVBA_BHD double clamp_sqrt(double v, double lo, double hi) { return sqrt(fmin(fmax(v, lo), hi)); }

struct CamF {                  // one item per camera column i < 6 n_rows
  const double* colsq; const double* grad; const double* y; double min_d, max_d; double* D; double* g; double* gn;
  LVBA_BHD void operator()(int64_t i) const {
    const double d = clamp_sqrt(colsq[i], min_d, max_d);
    D[i] = d; g[i] = grad[i] / d; gn[i] = d * y[i];
  }
};

template <bool kLoss>
struct TrkF {                  // one item per local landmark k: entries n6 + 3 k ..
  VisualView vv; VisualState st; VisualLM lm; int64_t n6; const double* pt_step; double* D; double* g; double* gn;
  LVBA_BHD void operator()(int64_t k) const {
    const int64_t tr = vv.trk_id[k];
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    const double* sp = lm.s_pt + 3 * k;
    double col[3] = {0.0, 0.0, 0.0}, gr[3] = {0.0, 0.0, 0.0};
    for (int64_t s = vv.trk_ptr[k]; s < vv.trk_ptr[k + 1]; ++s) {
      ObsEval o;
      vimp::obs_scaled<kLoss>(vv, st, lm, s, k, o);
      for (int m = 0; m < 3; ++m) {
        col[m] += o.JX[m] * o.JX[m] + o.JX[3 + m] * o.JX[3 + m];
        gr[m] += o.JX[m] * o.r[0] + o.JX[3 + m] * o.r[1];
      }
    }
    double rp, J[3];
    plane_eval(vv, vv.plane + 4 * k, X, rp, J);
    if constexpr (kLoss) plane_loss(vv, rp, J);
    for (int m = 0; m < 3; ++m) {
      const double j = J[m] * sp[m];
      col[m] += j * j;
      gr[m] += j * rp;
      const int64_t i = n6 + 3 * k + m;
      const double d = clamp_sqrt(col[m], lm.min_diag, lm.max_diag);
      D[i] = d; g[i] = gr[m] / d; gn[i] = d * (pt_step[3 * tr + m] / sp[m]);
    }
  }
};

struct DotF {                  // one item per entry: prod[3 i ..] = g_i^2, GN_i^2, g_i GN_i
  const double* g; const double* gn; double* prod;
  LVBA_BHD void operator()(int64_t i) const { prod[3 * i] = g[i] * g[i]; prod[3 * i + 1] = gn[i] * gn[i]; prod[3 * i + 2] = g[i] * gn[i]; }
};

// J~ v per landmark k (v: n6 camera entries, then 3 per landmark): out[kJvRec k ..].  Xc non-null: also the candidate landmark
// X + s_pt o v_k, its step^2 and x^2
template <bool kLoss>
struct JvF {
  VisualView vv; VisualState st; VisualLM lm; int64_t n6; const double* v; double* Xc; double* out;
  LVBA_BHD void operator()(int64_t k) const {
    const int64_t tr = vv.trk_id[k];
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    const double* sp = lm.s_pt + 3 * k;
    const double* vp = v + n6 + 3 * k;
    const double d[3] = {sp[0] * vp[0], sp[1] * vp[1], sp[2] * vp[2]};   // J~ v = J (s o v)
    double sq = 0.0, model = 0.0;
    for (int64_t s = vv.trk_ptr[k]; s < vv.trk_ptr[k + 1]; ++s) {
      const int cam = vv.obs_cam[s], row = vv.obs_row[s];
      ObsEval o;
      obs_eval<true>(vv, st.q + 4 * (int64_t)cam, st.t + 3 * (int64_t)cam, X, vv.obs_uv[s], o);
      if constexpr (kLoss) obs_loss<true>(vv, o);
      double dc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};   // a constant camera: no columns
      if (row >= 0)
        for (int a = 0; a < 6; ++a) dc[a] = lm.s_cam[6 * (int64_t)row + a] * v[6 * (int64_t)row + a];
      for (int r = 0; r < 2; ++r) {
        double j = o.JX[3 * r] * d[0] + o.JX[3 * r + 1] * d[1] + o.JX[3 * r + 2] * d[2];
        for (int a = 0; a < 6; ++a) j += o.Jc[6 * r + a] * dc[a];
        sq += j * j;
        model -= j * (o.r[r] + 0.5 * j);
      }
    }
    double rp, J[3];
    plane_eval(vv, vv.plane + 4 * k, X, rp, J);
    if constexpr (kLoss) plane_loss(vv, rp, J);
    const double j = J[0] * d[0] + J[1] * d[1] + J[2] * d[2];
    sq += j * j;
    model -= j * (rp + 0.5 * j);
    double* o = out + kJvRec * k;
    o[kJvModel] = model; o[kJvSq] = sq;
    o[kJvStep2] = 0.0; o[kJvX2] = 0.0;
    if (Xc) {
      for (int m = 0; m < 3; ++m) Xc[3 * tr + m] = X[m] + d[m];
      o[kJvStep2] = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
      o[kJvX2] = X[0] * X[0] + X[1] * X[1] + X[2] * X[2];
    }
  }
};

// The choice of the step at radius `radius`.  fresh: a new linearisation, alpha from the sums in sc[kGG] and sc[kJv + kJvSq];
// otherwise alpha and the sums of the last one
struct CaseF {
  double* sc; double radius; bool fresh;
  LVBA_BHD void operator()(int64_t) const {
    if (fresh) sc[kAlpha] = sc[kGG] / sc[kJv + kJvSq];
    const double alpha = sc[kAlpha];
    const double gnorm = sqrt(sc[kGG]), gn_norm = sqrt(sc[kNN]);
    double cg, cn, norm, beta = 0.0;
    int c;
    if (gn_norm <= radius) {
      c = kGaussNewton; cg = 0.0; cn = 1.0; norm = gn_norm;
    } else if (gnorm * alpha >= radius) {
      c = kCauchy; cg = -(radius / gnorm); cn = 0.0; norm = radius;
    } else {
      const double b_dot_a = -alpha * sc[kGN];
      const double a2 = (alpha * gnorm) * (alpha * gnorm);
      const double bma2 = a2 - 2.0 * b_dot_a + gn_norm * gn_norm;
      const double cc = b_dot_a - a2;
      const double d = sqrt(cc * cc + bma2 * (radius * radius - a2));
      beta = (cc <= 0.0) ? (d - cc) / bma2 : (radius * radius - a2) / (d + cc);
      c = kDogleg; cg = -alpha * (1.0 - beta); cn = beta;
      norm = sqrt(cg * cg * sc[kGG] + 2.0 * cg * cn * sc[kGN] + cn * cn * sc[kNN]);
    }
    sc[kCase] = c; sc[kBeta] = beta; sc[kCoefG] = cg; sc[kCoefN] = cn; sc[kStepNorm] = norm;
  }
};

struct StepF {                 // one item per entry: v = (c_g g + c_n GN) / D
  const double* sc; const double* D; const double* g; const double* gn; double* v;
  LVBA_BHD void operator()(int64_t i) const { v[i] = (sc[kCoefG] * g[i] + sc[kCoefN] * gn[i]) / D[i]; }
};

struct ScaleF {                // one item per entry: v = g / D (the Cauchy direction in the trust-region step's space)
  const double* D; const double* g; double* v;
  LVBA_BHD void operator()(int64_t i) const { v[i] = g[i] / D[i]; }
};

struct CopyF {                 // one item per j < n: dst[j] = src[j]
  const double* src; double* dst;
  LVBA_BHD void operator()(int64_t j) const { dst[j] = src[j]; }
};

// out[j] = sum_r in[r][j] (j < W, r < n) in a fixed order: chunks of kChunk rows in order, then the chunks; part [chunks][W]
template <class Exec>
int reduce(Exec& ex, const double* in, int64_t n, int W, double* part, double* out) {
  const int64_t nch = n > 0 ? (n + kChunk - 1) / kChunk : 1;
  int rc;
  if ((rc = ex.for_each(nch * W, vintr::ReduceF{in, n, kChunk, W, part}))) return rc;
  return ex.for_each(W, vintr::ReduceF{part, nch, nch, W, out});
}

// Buffers of one dogleg solve over n entries (n6 camera columns first) and Tv landmarks
struct Bufs {
  double *D, *g, *gn, *v, *prod, *part, *sc;
};
LVBA_BHD int64_t prod_size(int64_t n, int64_t Tv) { return 3 * n > kJvRec * Tv ? 3 * n : kJvRec * Tv; }
LVBA_BHD int64_t part_size(int64_t n, int64_t Tv) { return 4 * ((prod_size(n, Tv) + kChunk - 1) / kChunk + 1); }

// D, g, GN, their sums and alpha on a new linearisation: the build's camera column norms and gradient, the solve's y and the
// back-substitution's pt_step
template <bool kLoss, class Exec>
int linearised(Exec& ex, const VisualView& vv, const VisualState& st, const VisualLM& lm, int n_rows, int64_t Tv,
               const double* cam_colsq, const double* cam_grad, const double* y, const double* pt_step, const Bufs& B) {
  const int64_t n6 = 6 * (int64_t)n_rows, n = n6 + 3 * Tv;
  int rc;
  if ((rc = ex.for_each(n6, CamF{cam_colsq, cam_grad, y, lm.min_diag, lm.max_diag, B.D, B.g, B.gn}))) return rc;
  if ((rc = landmark_pass(ex, Tv, TrkF<kLoss>{vv, st, lm, n6, pt_step, B.D, B.g, B.gn}))) return rc;
  if ((rc = ex.for_each(n, DotF{B.g, B.gn, B.prod}))) return rc;
  if ((rc = reduce(ex, B.prod, n, 3, B.part, B.sc + kGG))) return rc;
  if ((rc = ex.for_each(n, ScaleF{B.D, B.g, B.v}))) return rc;
  if ((rc = landmark_pass(ex, Tv, JvF<kLoss>{vv, st, lm, n6, B.v, nullptr, B.prod}))) return rc;
  return reduce(ex, B.prod, Tv, kJvRec, B.part, B.sc + kJv);
}

// The dogleg step at `radius` (fresh: the first since linearised()): the case, v, the candidate landmarks into Xc and the
// model, step^2 and x^2 of the landmarks into scal[2..4] (the LM's layout); the cameras' candidate is the caller's
template <bool kLoss, class Exec>
int step(Exec& ex, const VisualView& vv, const VisualState& st, const VisualLM& lm, int n_rows, int64_t Tv, double radius, bool fresh,
         double* Xc, const Bufs& B, double* scal) {
  const int64_t n6 = 6 * (int64_t)n_rows, n = n6 + 3 * Tv;
  int rc;
  if ((rc = ex.for_each(1, CaseF{B.sc, radius, fresh}))) return rc;
  if ((rc = ex.for_each(n, StepF{B.sc, B.D, B.g, B.gn, B.v}))) return rc;
  if ((rc = landmark_pass(ex, Tv, JvF<kLoss>{vv, st, lm, n6, B.v, Xc, B.prod}))) return rc;
  if ((rc = reduce(ex, B.prod, Tv, kJvRec, B.part, B.sc + kJv))) return rc;
  return ex.for_each(3, CopyF{B.sc + kJv, scal + 2});
}

}  // namespace vdog
}  // namespace lvba
