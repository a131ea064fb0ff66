// visual_big.h — path B for landmarks with MORE observations than one batch CTA holds (K > kSlots = 128).
//
// The tiles and batches of visual.cuh keep a whole landmark in one CTA, a thread per observation.  A distant facade seen through
// hundreds of images, or a revisit that the matcher joins to an earlier pass, gives longer tracks; the reference adds one
// residual block per inlier whatever the track's length (src/lvba_system.cpp:1614-1632).  Set-up puts those landmarks after all
// small ones in the local order (local landmarks t0 .. t0 + n_big - 1, their observations at the end of the CSR) and they take
// the passes below, which restate the phases of visual_front / visual_build_kernel / visual_colnorm_kernel /
// visual_backsub_kernel / visual_cost_kernel observation by observation, with the camera-side sums added by atomics:
//
//   ObsF       (one item per observation)   r, J_c, J_X scaled by s_cam / s_pt; J_X^T J_X, J_X^T r       -> obs buffer
//   TrackF     (one item per landmark)      C = sum J_X^T J_X + plane term + LM diagonal, C^-1, g_p, w = C^-1 g_p (kTrkParams
//                                           layout), 1/2 (sum r^2 + r_p^2) and max |g_p| into the landmark's partial slots
//   SlotsF     (one item per observation)   E, Y = E C^-1, diagonal block J_c^T J_c - Y E^T, rhs, column norms, gradient
//                                           (atomics into S, rhs, cam_colsq, cam_grad); keeps Y and E in the obs buffer
//   PairsF     (one item per ordered pair)  S(row_x, row_y) -= Y_x E_y^T when row_x >= row_y >= 0 (both orders for a camera seen
//                                           twice, as VisPairKeyF)
//   ColObsF, ColTrackF                      the unscaled squared column norms of visual_colnorm_kernel
//   BacksubF   (one item per landmark)      y_p = -C^-1 (g_p + sum E^T y_c), the candidate landmark, its step, step^2, x^2 and
//                                           the model-cost change of its residuals
//   CostF      (one item per landmark)      1/2 (sum r^2 + r_p^2) at a given state
//
// The sums over a landmark's observations run sequentially inside one item; the pair pass is O(K^2) per landmark.  Functors over
// index ranges, launched by visual_api.cuh and, for the CPU check against oracle/visual_oracle.py, by tests/emu/.
#pragma once
#include "lidar_big.h"     // big::atomic_add_f64, LVBA_BHD
#include "visual_math.h"

namespace lvba {
namespace vbig {

// per observation: r (2), J_c (12), J_X (6) scaled, J_X^T J_X (6) J_X^T r (3) (the point column norms in ColObsF), Y (18), E (18).
// With a robust loss (kLoss) r, J_c and J_X are the corrected ones, and the slot kObRho holds rho(|r|^2) of the observation
// from ObsPass until SlotsPass overwrites it with Y (TrackPass reads it in between).
constexpr int kObR = 0, kObJc = 2, kObJX = 14, kObStage = 20, kObY = 29, kObE = 47, kObs = 65;
constexpr int kObRho = kObY;
static_assert(kObRho >= kObY && kObRho < kObY + 18, "rho must sit in the Y slot, which SlotsPass rewrites before any read of Y");

struct View {
  int64_t n_big;                // landmarks with more than kSlots observations
  int64_t t0;                   // local index of the first one (= the number of small landmarks)
  const int64_t* pair_ptr;      // [n_big + 1] prefix sums of K (K - 1): the ordered observation pairs of every big landmark
  const int* first;             // envelope of the reduced camera system
  const long long* row_start;
};

// big landmark of the observation `s` (an index into the local CSR, s >= trk_ptr[t0]): the last one starting at or before s
LVBA_BHD int64_t track_of(const VisualView& vv, const View& bv, int64_t s) {
  int64_t lo = bv.t0, hi = bv.t0 + bv.n_big;
  while (hi - lo > 1) { const int64_t m = (lo + hi) >> 1; if (vv.trk_ptr[m] <= s) lo = m; else hi = m; }
  return lo;
}

// kLoss (here and below): the robust losses of vv, the corrected residuals and Jacobians, cost terms rho
template <bool kLoss>
struct ObsPass {               // one item per observation of the big landmarks
  VisualView vv; View bv; VisualState st; VisualLM lm; double* obs;
  LVBA_BHD void operator()(int64_t i) const {
    const int64_t s = vv.trk_ptr[bv.t0] + i, k = track_of(vv, bv, s);
    const int64_t tr = vv.trk_id[k];
    const int cam = vv.obs_cam[s], row = vv.obs_row[s];
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    ObsEval o;
    obs_eval<true>(vv, st.q + 4 * (int64_t)cam, st.t + 3 * (int64_t)cam, X, vv.obs_uv[s], o);
    if constexpr (kLoss) obs[kObs * i + kObRho] = obs_loss<true>(vv, o);
    const double* sp = lm.s_pt + 3 * k;
    for (int rho = 0; rho < 2; ++rho)
      for (int m = 0; m < 3; ++m) o.JX[3 * rho + m] *= sp[m];
    if (row >= 0) {
      const double* sc = lm.s_cam + 6 * (int64_t)row;
      for (int rho = 0; rho < 2; ++rho)
        for (int a = 0; a < 6; ++a) o.Jc[6 * rho + a] *= sc[a];
    } else {
      for (int a = 0; a < 12; ++a) o.Jc[a] = 0.0;          // constant / unused camera: no columns
    }
    double* f = obs + kObs * i;
    f[kObR] = o.r[0]; f[kObR + 1] = o.r[1];
    for (int a = 0; a < 12; ++a) f[kObJc + a] = o.Jc[a];
    for (int a = 0; a < 6; ++a) f[kObJX + a] = o.JX[a];
    double* sg = f + kObStage;
    sg[0] = o.JX[0] * o.JX[0] + o.JX[3] * o.JX[3];
    sg[1] = o.JX[0] * o.JX[1] + o.JX[3] * o.JX[4];
    sg[2] = o.JX[0] * o.JX[2] + o.JX[3] * o.JX[5];
    sg[3] = o.JX[1] * o.JX[1] + o.JX[4] * o.JX[4];
    sg[4] = o.JX[1] * o.JX[2] + o.JX[4] * o.JX[5];
    sg[5] = o.JX[2] * o.JX[2] + o.JX[5] * o.JX[5];
    sg[6] = o.JX[0] * o.r[0] + o.JX[3] * o.r[1];
    sg[7] = o.JX[1] * o.r[0] + o.JX[4] * o.r[1];
    sg[8] = o.JX[2] * o.r[0] + o.JX[5] * o.r[1];
  }
};

// The landmark step of local landmark k at X, from acc = sum J_X^T J_X (xx xy xz yy yz zz) | sum J_X^T r and c = sum r^2 (kLoss:
// sum rho) over its observations: the plane term, the LM diagonal of the point columns, C^-1, g_p and w = C^-1 g_p into
// params + kTrkParams b (kTrkParams layout), 1/2 (c + the plane's term) into cost[b] and max |g_p| (unscaled) into gmax[b].
// TrackPass and the matrix-free linearisation (visual_implicit.h) share it.
template <bool kLoss>
LVBA_BHD void landmark_step(const VisualView& vv, const VisualLM& lm, int64_t k, const double* X, double* acc, double c, double* params,
                            double* cost, double* gmax, int64_t b) {
  double rp, Jpl[3];
  plane_eval(vv, vv.plane + 4 * k, X, rp, Jpl);
  if constexpr (kLoss) c += plane_loss(vv, rp, Jpl);
  else c += rp * rp;
  const double* sp = lm.s_pt + 3 * k;
  Jpl[0] *= sp[0]; Jpl[1] *= sp[1]; Jpl[2] *= sp[2];
  acc[0] += Jpl[0] * Jpl[0]; acc[1] += Jpl[0] * Jpl[1]; acc[2] += Jpl[0] * Jpl[2];
  acc[3] += Jpl[1] * Jpl[1]; acc[4] += Jpl[1] * Jpl[2]; acc[5] += Jpl[2] * Jpl[2];
  acc[6] += Jpl[0] * rp; acc[7] += Jpl[1] * rp; acc[8] += Jpl[2] * rp;
  // LM diagonal of the point columns: clamp(||J~[:,j]||^2)/radius   (Ceres LevenbergMarquardtStrategy)
  const double ir = 1.0 / lm.radius;
  acc[0] += fmin(fmax(acc[0], lm.min_diag), lm.max_diag) * ir;
  acc[3] += fmin(fmax(acc[3], lm.min_diag), lm.max_diag) * ir;
  acc[5] += fmin(fmax(acc[5], lm.min_diag), lm.max_diag) * ir;
  double* p = params + kTrkParams * b;
  sym3_inverse(acc, p);
  p[6] = acc[6]; p[7] = acc[7]; p[8] = acc[8];
  p[9] = p[0] * acc[6] + p[1] * acc[7] + p[2] * acc[8];
  p[10] = p[1] * acc[6] + p[3] * acc[7] + p[4] * acc[8];
  p[11] = p[2] * acc[6] + p[4] * acc[7] + p[5] * acc[8];
  cost[b] = 0.5 * c;
  gmax[b] = fmax(fabs(p[6] / sp[0]), fmax(fabs(p[7] / sp[1]), fabs(p[8] / sp[2])));
}

template <bool kLoss>
struct TrackPass {             // one item per big landmark; cost[b] = 1/2 sum r^2 (kLoss: 1/2 sum rho), gmax[b] = max |g_p| (unscaled)
  VisualView vv; View bv; VisualState st; VisualLM lm; const double* obs; double* params; double* cost; double* gmax;
  LVBA_BHD void operator()(int64_t b) const {
    const int64_t k = bv.t0 + b, base = vv.trk_ptr[bv.t0];
    const int64_t lo = vv.trk_ptr[k] - base, hi = vv.trk_ptr[k + 1] - base;
    const int64_t tr = vv.trk_id[k];
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    double acc[9], c = 0.0;
    for (int q = 0; q < 9; ++q) acc[q] = 0.0;
    for (int64_t i = lo; i < hi; ++i) {
      const double* f = obs + kObs * i;
      if constexpr (kLoss) c += f[kObRho];
      else c += f[kObR] * f[kObR] + f[kObR + 1] * f[kObR + 1];
      for (int q = 0; q < 9; ++q) acc[q] += f[kObStage + q];
    }
    landmark_step<kLoss>(vv, lm, k, X, acc, c, params, cost, gmax, b);
  }
};

// kDet = false: the camera-side sums go into S, rhs, cam_colsq and cam_grad by atomics.  true (deterministic mode): S = the
// observations' records [n_obs][36] and rhs = [n_obs][18] (rhs | column norms | gradient), one record per observation, summed per
// destination by tiles::GatherF (lidar_tiles.h) in observation order; cam_colsq and cam_grad are not used.
// With a loss, kObRho (inside Y) still holds rho from ObsPass when this pass runs, after TrackPass; this pass writes Y and E of
// every observation of a non-constant camera, the only ones PairsPass reads.  Keep that order: ObsPass, TrackPass, SlotsPass,
// PairsPass.
template <bool kDet>
struct SlotsPass {             // one item per observation of the big landmarks
  VisualView vv; View bv; const double* params; double* obs; double* S; double* rhs; double* cam_colsq; double* cam_grad;
  LVBA_BHD void operator()(int64_t i) const {
    const int64_t s = vv.trk_ptr[bv.t0] + i;
    const int row = vv.obs_row[s];
    if (row < 0) return;
    const int64_t b = track_of(vv, bv, s) - bv.t0;
    double* f = obs + kObs * i;
    const double* Jc = f + kObJc; const double* JX = f + kObJX; const double* r = f + kObR;
    const double* p = params + kTrkParams * b;
    const double Ci[9] = {p[0], p[1], p[2], p[1], p[3], p[4], p[2], p[4], p[5]};
    double* E = f + kObE; double* Y = f + kObY;
    for (int a = 0; a < 6; ++a)
      for (int m = 0; m < 3; ++m) E[3 * a + m] = Jc[a] * JX[m] + Jc[6 + a] * JX[3 + m];
    for (int a = 0; a < 6; ++a)
      for (int m = 0; m < 3; ++m) Y[3 * a + m] = E[3 * a] * Ci[m] + E[3 * a + 1] * Ci[3 + m] + E[3 * a + 2] * Ci[6 + m];
    for (int a = 0; a < 6; ++a) {
      const double gc = Jc[a] * r[0] + Jc[6 + a] * r[1];
      const double ra = -(gc - (E[3 * a] * p[9] + E[3 * a + 1] * p[10] + E[3 * a + 2] * p[11]));
      const double ca = Jc[a] * Jc[a] + Jc[6 + a] * Jc[6 + a];
      if constexpr (kDet) {
        double* G = rhs + 18 * i;
        G[a] = ra; G[6 + a] = ca; G[12 + a] = gc;
      } else {
        big::atomic_add_f64(rhs + 6 * (int64_t)row + a, ra);
        big::atomic_add_f64(cam_colsq + 6 * (int64_t)row + a, ca);
        big::atomic_add_f64(cam_grad + 6 * (int64_t)row + a, gc);
      }
      for (int c = 0; c < 6; ++c) {
        const double d = Jc[a] * Jc[c] + Jc[6 + a] * Jc[6 + c]
                       - (Y[3 * a] * E[3 * c] + Y[3 * a + 1] * E[3 * c + 1] + Y[3 * a + 2] * E[3 * c + 2]);
        if constexpr (kDet) S[36 * i + 6 * a + c] = d;
        else big::atomic_add_f64(S + (bv.row_start[row] + (row - bv.first[row])) * 36 + 6 * a + c, d);
      }
    }
  }
};

// ordered observation pair p (x != y) of the big landmarks: its two observations in the local CSR
LVBA_BHD void pair_obs(const VisualView& vv, const View& bv, int64_t p, int64_t& sx, int64_t& sy) {
  int64_t b = 0, hi = bv.n_big;
  while (hi - b > 1) { const int64_t m = (b + hi) >> 1; if (bv.pair_ptr[m] <= p) b = m; else hi = m; }
  const int64_t k = bv.t0 + b;
  const int64_t r = p - bv.pair_ptr[b], K1 = vv.trk_ptr[k + 1] - vv.trk_ptr[k] - 1;
  const int64_t x = r / K1, y0 = r - x * K1, y = y0 + (y0 >= x);
  sx = vv.trk_ptr[k] + x; sy = vv.trk_ptr[k] + y;
}

// kDet = false: the block goes into S by atomics; true: S = the pairs' records [n_pairs][36] (see SlotsPass)
template <bool kDet>
struct PairsPass {             // one item per ordered observation pair (x, y), x != y, of a big landmark
  VisualView vv; View bv; const double* obs; double* S;
  LVBA_BHD void operator()(int64_t p) const {
    const int64_t base = vv.trk_ptr[bv.t0];
    int64_t sx, sy;
    pair_obs(vv, bv, p, sx, sy);
    const int rx = vv.obs_row[sx], ry = vv.obs_row[sy];
    if (!(ry >= 0 && rx >= ry)) return;                  // both rows >= 0: SlotsPass wrote Y_x over ObsPass' rho (kObRho)
    const double* Yx = obs + kObs * (sx - base) + kObY;
    const double* Ey = obs + kObs * (sy - base) + kObE;
    double* B = kDet ? S + 36 * p : S + (bv.row_start[rx] + (ry - bv.first[rx])) * 36;
    for (int a = 0; a < 6; ++a)
      for (int c = 0; c < 6; ++c) {
        const double d = -(Yx[3 * a] * Ey[3 * c] + Yx[3 * a + 1] * Ey[3 * c + 1] + Yx[3 * a + 2] * Ey[3 * c + 2]);
        if constexpr (kDet) B[6 * a + c] = d;
        else big::atomic_add_f64(B + 6 * a + c, d);
      }
  }
};

// kDet = false: camera columns into cam_colsq by atomics; true: cam_colsq = the observations' records [n_obs][6]
template <bool kDet, bool kLoss = false>
struct ColObsPass {            // unscaled column norms, one item per observation: camera columns by atomics, point columns kept
  VisualView vv; View bv; VisualState st; double* obs; double* cam_colsq;
  LVBA_BHD void operator()(int64_t i) const {
    const int64_t s = vv.trk_ptr[bv.t0] + i, k = track_of(vv, bv, s);
    const int64_t tr = vv.trk_id[k];
    const int cam = vv.obs_cam[s], row = vv.obs_row[s];
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    ObsEval o;
    obs_eval<true>(vv, st.q + 4 * (int64_t)cam, st.t + 3 * (int64_t)cam, X, vv.obs_uv[s], o);
    if constexpr (kLoss) obs_loss<true>(vv, o);
    double* sg = obs + kObs * i + kObStage;
    sg[0] = o.JX[0] * o.JX[0] + o.JX[3] * o.JX[3];
    sg[1] = o.JX[1] * o.JX[1] + o.JX[4] * o.JX[4];
    sg[2] = o.JX[2] * o.JX[2] + o.JX[5] * o.JX[5];
    if (row >= 0)
      for (int a = 0; a < 6; ++a) {
        const double c = o.Jc[a] * o.Jc[a] + o.Jc[6 + a] * o.Jc[6 + a];
        if constexpr (kDet) cam_colsq[6 * i + a] = c;
        else big::atomic_add_f64(cam_colsq + 6 * (int64_t)row + a, c);
      }
  }
};

using ObsF = ObsPass<false>;
using TrackF = TrackPass<false>;
using SlotsF = SlotsPass<false>;
using PairsF = PairsPass<false>;
using ColObsF = ColObsPass<false>;
using SlotsDetF = SlotsPass<true>;
using PairsDetF = PairsPass<true>;
using ColObsDetF = ColObsPass<true>;

// Destinations of the deterministic records of SlotsDetF / ColObsDetF (the observation's diagonal S block and its row) and of
// PairsDetF (the lower S block of the pair), in the units of tiles::FixedSum; n_blocks / n_rows mark a record without one
// (a constant camera, or a pair that is not in the lower envelope)
struct ObsDstF {
  VisualView vv; View bv; long long n_blocks; int n_rows; int64_t* dst_S; int64_t* dst_row;
  LVBA_BHD void operator()(int64_t i) const {
    const int row = vv.obs_row[vv.trk_ptr[bv.t0] + i];
    dst_S[i] = row >= 0 ? bv.row_start[row] + (row - bv.first[row]) : n_blocks;
    dst_row[i] = row >= 0 ? row : n_rows;
  }
};
struct PairDstF {
  VisualView vv; View bv; long long n_blocks; int64_t* dst_S;
  LVBA_BHD void operator()(int64_t p) const {
    int64_t sx, sy;
    pair_obs(vv, bv, p, sx, sy);
    const int rx = vv.obs_row[sx], ry = vv.obs_row[sy];
    dst_S[p] = (ry >= 0 && rx >= ry) ? bv.row_start[rx] + (ry - bv.first[rx]) : n_blocks;
  }
};

template <bool kLoss>
struct ColTrackPass {          // one item per big landmark: its three point columns
  VisualView vv; View bv; VisualState st; const double* obs; double* pt_colsq;
  LVBA_BHD void operator()(int64_t b) const {
    const int64_t k = bv.t0 + b, base = vv.trk_ptr[bv.t0];
    const int64_t tr = vv.trk_id[k];
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    double rp, J[3];
    plane_eval(vv, vv.plane + 4 * k, X, rp, J);
    if constexpr (kLoss) plane_loss(vv, rp, J);
    double a0 = J[0] * J[0], a1 = J[1] * J[1], a2 = J[2] * J[2];
    for (int64_t i = vv.trk_ptr[k] - base; i < vv.trk_ptr[k + 1] - base; ++i) {
      const double* sg = obs + kObs * i + kObStage;
      a0 += sg[0]; a1 += sg[1]; a2 += sg[2];
    }
    double* o = pt_colsq + 3 * k;
    o[0] = a0; o[1] = a1; o[2] = a2;
  }
};

// one item per big landmark, after ObsPass / TrackPass at the same state and scale: out[4 b ..] = model-cost change, step^2,
// x^2, 0
// kStride: the doubles per observation record of obs (r, J_c and J_X at kObR, kObJc and kObJX): kObs for ObsPass' records
// (BacksubPass), vimp::kRec for those of the matrix-free linearisation (visual_implicit.h)
template <bool kLoss, int kStride>
struct BacksubStridePass {
  VisualView vv; View bv; VisualState st; VisualLM lm; const double* obs; double* params; const double* y_cam;
  double* X_cand; double* pt_step; double* out;
  LVBA_BHD void operator()(int64_t b) const {
    const int64_t k = bv.t0 + b, base = vv.trk_ptr[bv.t0];
    const int64_t lo = vv.trk_ptr[k] - base, hi = vv.trk_ptr[k + 1] - base;
    double a0 = 0, a1 = 0, a2 = 0;
    for (int64_t i = lo; i < hi; ++i) {                 // E^T y_c = J_X^T (J_c y_c)
      const double* f = obs + kStride * i;
      double j0, j1;
      camera_part(f, vv.obs_row[base + i], j0, j1);
      const double* JX = f + kObJX;
      a0 += JX[0] * j0 + JX[3] * j1; a1 += JX[1] * j0 + JX[4] * j1; a2 += JX[2] * j0 + JX[5] * j1;
    }
    double* p = params + kTrkParams * b;
    const double y0 = -(p[9] + p[0] * a0 + p[1] * a1 + p[2] * a2);
    const double y1 = -(p[10] + p[1] * a0 + p[3] * a1 + p[4] * a2);
    const double y2 = -(p[11] + p[2] * a0 + p[4] * a1 + p[5] * a2);
    p[12] = y0; p[13] = y1; p[14] = y2;
    const int64_t tr = vv.trk_id[k];
    const double* sp = lm.s_pt + 3 * k;
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    const double d[3] = {sp[0] * y0, sp[1] * y1, sp[2] * y2};
    X_cand[3 * tr] = X[0] + d[0]; X_cand[3 * tr + 1] = X[1] + d[1]; X_cand[3 * tr + 2] = X[2] + d[2];
    if (pt_step) { pt_step[3 * tr] = d[0]; pt_step[3 * tr + 1] = d[1]; pt_step[3 * tr + 2] = d[2]; }
    double rp, Jpl[3];
    plane_eval(vv, vv.plane + 4 * k, X, rp, Jpl);
    if constexpr (kLoss) plane_loss(vv, rp, Jpl);
    const double jy = Jpl[0] * d[0] + Jpl[1] * d[1] + Jpl[2] * d[2];   // J~ y = J (s o y)
    double model = -jy * (rp + 0.5 * jy);
    for (int64_t i = lo; i < hi; ++i) {
      const double* f = obs + kStride * i;
      double j0, j1;
      camera_part(f, vv.obs_row[base + i], j0, j1);
      const double* JX = f + kObJX;
      const double jy0 = j0 + JX[0] * y0 + JX[1] * y1 + JX[2] * y2;
      const double jy1 = j1 + JX[3] * y0 + JX[4] * y1 + JX[5] * y2;
      model -= jy0 * (f[kObR] + 0.5 * jy0) + jy1 * (f[kObR + 1] + 0.5 * jy1);
    }
    double* o = out + 4 * b;
    o[0] = model; o[1] = d[0] * d[0] + d[1] * d[1] + d[2] * d[2]; o[2] = X[0] * X[0] + X[1] * X[1] + X[2] * X[2]; o[3] = 0.0;
  }
  // J_c y_c of one observation (zero for a constant camera)
  LVBA_BHD void camera_part(const double* f, int row, double& j0, double& j1) const {
    j0 = 0.0; j1 = 0.0;
    if (row < 0) return;
    const double* yc = y_cam + 6 * (int64_t)row;
    const double* Jc = f + kObJc;
    j0 = Jc[0] * yc[0] + Jc[1] * yc[1] + Jc[2] * yc[2] + Jc[3] * yc[3] + Jc[4] * yc[4] + Jc[5] * yc[5];
    j1 = Jc[6] * yc[0] + Jc[7] * yc[1] + Jc[8] * yc[2] + Jc[9] * yc[3] + Jc[10] * yc[4] + Jc[11] * yc[5];
  }
};

template <bool kLoss>
struct CostPass {              // one item per big landmark: cost[b] = 1/2 (sum r^2 + r_p^2) (kLoss: 1/2 sum rho) at the state `st`
  VisualView vv; View bv; VisualState st; double* cost;
  LVBA_BHD void operator()(int64_t b) const {
    const int64_t k = bv.t0 + b;
    const int64_t tr = vv.trk_id[k];
    const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
    double c = 0.0;
    for (int64_t s = vv.trk_ptr[k]; s < vv.trk_ptr[k + 1]; ++s) {
      const int cam = vv.obs_cam[s];
      ObsEval o;
      obs_eval<false>(vv, st.q + 4 * (int64_t)cam, st.t + 3 * (int64_t)cam, X, vv.obs_uv[s], o);
      if constexpr (kLoss) c += obs_loss<false>(vv, o);
      else c += o.r[0] * o.r[0] + o.r[1] * o.r[1];
    }
    double rp, J[3];
    plane_eval(vv, vv.plane + 4 * k, X, rp, J);
    if constexpr (kLoss) cost[b] = 0.5 * (c + plane_loss(vv, rp, J));
    else cost[b] = 0.5 * (c + rp * rp);
  }
};

template <bool kLoss>
struct BacksubPass : BacksubStridePass<kLoss, kObs> {};

using ColTrackF = ColTrackPass<false>;
using BacksubF = BacksubPass<false>;
using CostF = CostPass<false>;

}  // namespace vbig
}  // namespace lvba
