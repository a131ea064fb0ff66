// visual_math.h — path B arithmetic shared by the kernels of visual.cuh and the passes of visual_big.h: the reprojection and
// point-to-plane residuals with their analytic Jacobians, the robust losses and the 3x3 landmark block inverse.  Compiled for the device and, for
// the CPU tests of tests/emu/, for the host.
//
// Restates (analytic Jacobians instead of ceres::Jet auto-diff):
//   ReprojErrorWhitenedDistorted::operator()   reference include/utils.hpp:61-111
//   PointPlaneErrorWhitened::operator()        reference include/utils.hpp:133-139
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>

#include "vec3.h"

#if defined(__CUDACC__)
#include <vector_types.h>
#else
struct alignas(8) float2 { float x, y; };   // CUDA's float2, for host compilers without the CUDA headers
#endif

namespace lvba {

constexpr int kTrkParams = 16;     // per landmark: Cinv(6) g_p(3) w(3) y_p(3) pad

struct VisualView {
  int n_batches;             // back-substitution and cost: batches of <= kSlots observations
  const int* batch_trk;      // [n_batches+1] landmark range per batch
  int n_tiles;               // build and column norms: tiles of <= kVisTileSlots observations (visual_tiles.h)
  const int* tile_trk;       // [n_tiles+1] landmark range per tile
  const int64_t* tile_prun;  // [n_tiles+1] pair runs of every tile
  const int64_t* prun_ptr;   // run r = pairs[prun_ptr[r] .. prun_ptr[r+1]): the camera-pair contributions of one S block
  const unsigned* pairs;     // hi | lo << 16, observations local to the tile (contribution -Y_hi E_lo^T)
  const int64_t* tile_drun;  // [n_tiles+1] row runs of every tile
  const int64_t* drun_ptr;   // run r = dslot[drun_ptr[r] .. drun_ptr[r+1]): the observations of one system row
  const unsigned* dslot;     // observations local to the tile
  const int* trk_ptr;        // [Tv+1] obs offsets (valid landmarks only, compact)
  const int* trk_id;         // [Tv]   original landmark index
  const int* obs_cam;        // [nnz] original camera index
  const int* obs_row;        // [nnz] reduced-system row of that camera, -1 when constant / unused
  const float2* obs_uv;      // [nnz]
  const double* plane;       // [Tv*4]
  double intr[8];
  double inv_sigma_px, inv_sigma_pl;
  int loss_px, loss_pl;      // robust loss (kLoss*) of the reprojection / plane blocks; read by the kLoss instantiations only
  double loss_a_px, loss_a_pl;   // their scales
};

// lvba_loss_kind (include/lvba_b200.h)
constexpr int kLossNone = 0, kLossHuber = 1, kLossCauchy = 2;

struct VisualState {
  const double* q;   // [M*4]
  const double* t;   // [M*3]
  const double* X;   // [T*3]
};

struct VisualLM {
  double radius, min_diag, max_diag;
  const double* s_cam;   // [n_rows*6] Jacobi scale of the camera tangent columns
  const double* s_pt;    // [Tv*3]
};

struct ObsEval {
  double r[2];
  double Jc[12];     // 2x6  [rho][0..2 rotation tangent | 3..5 translation]
  double JX[6];      // 2x3
};

// utils.hpp:61-111 forward model + analytic Jacobians (SURVEY.md A.2, Q9 tangent basis)
template <bool kJac>
LVBA_HD void obs_eval(const VisualView& vv, const double* __restrict__ qp, const double* __restrict__ tp,
                      const double* X, float2 uv, ObsEval& o) {
  double q0 = qp[0], q1 = qp[1], q2 = qp[2], q3 = qp[3];
  const double inv = 1.0 / sqrt(q0 * q0 + q1 * q1 + q2 * q2 + q3 * q3);   // QuaternionRotatePoint normalises
  q0 *= inv; q1 *= inv; q2 *= inv; q3 *= inv;
  const double v[3] = {q1, q2, q3};
  double vxX[3], t2[3];
  cross3(v, X, vxX);
  const double uvv[3] = {2.0 * vxX[0], 2.0 * vxX[1], 2.0 * vxX[2]};
  cross3(v, uvv, t2);
  const double Xc[3] = {X[0] + q0 * uvv[0] + t2[0] + tp[0], X[1] + q0 * uvv[1] + t2[1] + tp[1],
                        X[2] + q0 * uvv[2] + t2[2] + tp[2]};
  const double z = Xc[2];
  if (!(z > 1e-8)) {                                   // utils.hpp:78
    o.r[0] = 0.0; o.r[1] = 0.0;
    if (kJac) {
LVBA_UNROLL
      for (int i = 0; i < 12; ++i) o.Jc[i] = 0.0;
LVBA_UNROLL
      for (int i = 0; i < 6; ++i) o.JX[i] = 0.0;
    }
    return;
  }
  const double fx = vv.intr[0], fy = vv.intr[1], cx = vv.intr[2], cy = vv.intr[3];
  const double k1 = vv.intr[4], k2 = vv.intr[5], p1 = vv.intr[6], p2 = vv.intr[7];
  const double iz = 1.0 / z;
  const double xn = Xc[0] * iz, yn = Xc[1] * iz;
  const double r2 = xn * xn + yn * yn;
  const double rad = 1.0 + k1 * r2 + k2 * r2 * r2;
  const double xd = xn * rad + 2.0 * p1 * xn * yn + p2 * (r2 + 2.0 * xn * xn);
  const double yd = yn * rad + p1 * (r2 + 2.0 * yn * yn) + 2.0 * p2 * xn * yn;
  const double is = vv.inv_sigma_px;
  o.r[0] = (fx * xd + cx - (double)uv.x) * is;
  o.r[1] = (fy * yd + cy - (double)uv.y) * is;
  if (!kJac) return;
  const double g = 2.0 * (k1 + 2.0 * k2 * r2);
  const double d00 = rad + xn * xn * g + 2.0 * p1 * yn + 6.0 * p2 * xn;
  const double d01 = xn * yn * g + 2.0 * p1 * xn + 2.0 * p2 * yn;
  const double d11 = rad + yn * yn * g + 6.0 * p1 * yn + 2.0 * p2 * xn;
  // Jpix = diag(fx,fy)/sigma * Dd * [1/z 0 -xn/z ; 0 1/z -yn/z]
  double Jp[6];
  const double sx = fx * is, sy = fy * is;
  Jp[0] = sx * d00 * iz; Jp[1] = sx * d01 * iz; Jp[2] = -sx * (d00 * xn + d01 * yn) * iz;
  Jp[3] = sy * d01 * iz; Jp[4] = sy * d11 * iz; Jp[5] = -sy * (d01 * xn + d11 * yn) * iz;
  // rotation matrix of the unit quaternion
  double R[9];
  R[0] = 1 - 2 * (q2 * q2 + q3 * q3); R[1] = 2 * (q1 * q2 - q0 * q3); R[2] = 2 * (q1 * q3 + q0 * q2);
  R[3] = 2 * (q1 * q2 + q0 * q3); R[4] = 1 - 2 * (q1 * q1 + q3 * q3); R[5] = 2 * (q2 * q3 - q0 * q1);
  R[6] = 2 * (q1 * q3 - q0 * q2); R[7] = 2 * (q2 * q3 + q0 * q1); R[8] = 1 - 2 * (q1 * q1 + q2 * q2);
LVBA_UNROLL
  for (int rho = 0; rho < 2; ++rho)
LVBA_UNROLL
    for (int m = 0; m < 3; ++m)
      o.JX[3 * rho + m] = Jp[3 * rho] * R[m] + Jp[3 * rho + 1] * R[3 + m] + Jp[3 * rho + 2] * R[6 + m];
  // ambient d(RX)/dq (3x4): col0 = 2 v x X ; cols1..3 = -2w hat(X) - 2 hat(v x X) - 2 X v^T + 2 (v.X) I
  double Ja[12];
  const double vX = dot3(v, X);
  double hX[9], hC[9];
  hat3(X, hX);
  hat3(vxX, hC);
LVBA_UNROLL
  for (int i = 0; i < 3; ++i) {
    Ja[4 * i] = 2.0 * vxX[i];
LVBA_UNROLL
    for (int j = 0; j < 3; ++j)
      Ja[4 * i + 1 + j] = -2.0 * q0 * hX[3 * i + j] - 2.0 * hC[3 * i + j] - 2.0 * X[i] * v[j] + ((i == j) ? 2.0 * vX : 0.0);
  }
  // EigenQuaternionManifold::PlusJacobian on memory (m0..m3) = (w,x,y,z)  (Q9)
  const double m0 = q0, m1 = q1, m2 = q2, m3 = q3;
  const double PJ[12] = {m3, m2, -m1,   -m2, m3, m0,   m1, -m0, m3,   -m0, -m1, -m2};
  double Jt3[9];   // 3x3 = Ja (3x4) * PJ (4x3)
LVBA_UNROLL
  for (int i = 0; i < 3; ++i)
LVBA_UNROLL
    for (int j = 0; j < 3; ++j)
      Jt3[3 * i + j] = Ja[4 * i] * PJ[j] + Ja[4 * i + 1] * PJ[3 + j] + Ja[4 * i + 2] * PJ[6 + j] + Ja[4 * i + 3] * PJ[9 + j];
LVBA_UNROLL
  for (int rho = 0; rho < 2; ++rho)
LVBA_UNROLL
    for (int j = 0; j < 3; ++j) {
      o.Jc[6 * rho + j] = Jp[3 * rho] * Jt3[j] + Jp[3 * rho + 1] * Jt3[3 + j] + Jp[3 * rho + 2] * Jt3[6 + j];
      o.Jc[6 * rho + 3 + j] = Jp[3 * rho + j];
    }
}

// d r / d (fx fy cx cy k1 k2 p1 p2) of the whitened residual of obs_eval (2x8, row-major: Jk[8 rho + i]), with obs_eval's
// projection step for step; zero where the depth test z > 1e-8 fails (utils.hpp:78).  A function of its own, as obs_depth, so
// that the kernels that call obs_eval keep their code.
LVBA_HD void intr_jac(const VisualView& vv, const double* __restrict__ qp, const double* __restrict__ tp, const double* X,
                      double Jk[16]) {
  double q0 = qp[0], q1 = qp[1], q2 = qp[2], q3 = qp[3];
  const double inv = 1.0 / sqrt(q0 * q0 + q1 * q1 + q2 * q2 + q3 * q3);
  q0 *= inv; q1 *= inv; q2 *= inv; q3 *= inv;
  const double v[3] = {q1, q2, q3};
  double vxX[3], t2[3];
  cross3(v, X, vxX);
  const double uvv[3] = {2.0 * vxX[0], 2.0 * vxX[1], 2.0 * vxX[2]};
  cross3(v, uvv, t2);
  const double Xc[3] = {X[0] + q0 * uvv[0] + t2[0] + tp[0], X[1] + q0 * uvv[1] + t2[1] + tp[1],
                        X[2] + q0 * uvv[2] + t2[2] + tp[2]};
  const double z = Xc[2];
  for (int i = 0; i < 16; ++i) Jk[i] = 0.0;
  if (!(z > 1e-8)) return;
  const double fx = vv.intr[0], fy = vv.intr[1], k1 = vv.intr[4], k2 = vv.intr[5], p1 = vv.intr[6], p2 = vv.intr[7];
  const double iz = 1.0 / z;
  const double xn = Xc[0] * iz, yn = Xc[1] * iz;
  const double r2 = xn * xn + yn * yn;
  const double rad = 1.0 + k1 * r2 + k2 * r2 * r2;
  const double xd = xn * rad + 2.0 * p1 * xn * yn + p2 * (r2 + 2.0 * xn * xn);
  const double yd = yn * rad + p1 * (r2 + 2.0 * yn * yn) + 2.0 * p2 * xn * yn;
  const double is = vv.inv_sigma_px, sx = fx * is, sy = fy * is;
  Jk[0] = xd * is; Jk[2] = is;
  Jk[4] = sx * xn * r2; Jk[5] = sx * xn * r2 * r2; Jk[6] = sx * 2.0 * xn * yn; Jk[7] = sx * (r2 + 2.0 * xn * xn);
  Jk[9] = yd * is; Jk[11] = is;
  Jk[12] = sy * yn * r2; Jk[13] = sy * yn * r2 * r2; Jk[14] = sy * (r2 + 2.0 * yn * yn); Jk[15] = sy * 2.0 * xn * yn;
}

// The camera-frame depth obs_eval tests (utils.hpp:78), with obs_eval's arithmetic step for step, so that the two agree on
// every bit.  A function of its own rather than a part factored out of obs_eval: that keeps the code of the kernels that call
// obs_eval as it was.
LVBA_HD double obs_depth(const double* __restrict__ qp, const double* __restrict__ tp, const double* X) {
  double q0 = qp[0], q1 = qp[1], q2 = qp[2], q3 = qp[3];
  const double inv = 1.0 / sqrt(q0 * q0 + q1 * q1 + q2 * q2 + q3 * q3);
  q0 *= inv; q1 *= inv; q2 *= inv; q3 *= inv;
  const double v[3] = {q1, q2, q3};
  double vxX[3], t2[3];
  cross3(v, X, vxX);
  const double uvv[3] = {2.0 * vxX[0], 2.0 * vxX[1], 2.0 * vxX[2]};
  cross3(v, uvv, t2);
  return X[2] + q0 * uvv[2] + t2[2] + tp[2];
}

// utils.hpp:133-139
LVBA_HD void plane_eval(const VisualView& vv, const double* pl, const double* X, double& r, double J[3]) {
  const double e = -(pl[0] * X[0] + pl[1] * X[1] + pl[2] * X[2] + pl[3]);
  const double root = sqrt(e * e + 1e-12);
  r = root * vv.inv_sigma_pl;
  const double k = (e / root) * vv.inv_sigma_pl;
  J[0] = -k * pl[0]; J[1] = -k * pl[1]; J[2] = -k * pl[2];
}

// rho(s) and rho'(s) of a robust loss with scale a at the squared norm s of a residual block: ceres-solver 2.1.0 HuberLoss and
// CauchyLoss (loss_function.cc), b = a^2.  Both have rho'' <= 0 everywhere, so Ceres' Corrector (corrector.cc) reduces to
// scaling the residual and the Jacobian by sqrt(rho'); rho'' is never needed.  kLossNone: rho = s, rho' = 1.
LVBA_HD void loss_eval(int kind, double a, double s, double& rho, double& rho1) {
  const double b = a * a;
  if (kind == kLossHuber && s > b) {
    const double r = sqrt(s);
    rho = 2.0 * a * r - b;
    rho1 = fmax(DBL_MIN, a / r);
  } else if (kind == kLossCauchy) {
    const double c = 1.0 / b, u = 1.0 + s * c;
    rho = b * log(u);
    rho1 = fmax(DBL_MIN, 1.0 / u);
  } else {
    rho = s;
    rho1 = 1.0;
  }
}

// Corrector of one reprojection block: returns its cost term rho(|r|^2); with kCorrect, r, J_c and J_X times sqrt(rho')
template <bool kCorrect>
LVBA_HD double obs_loss(const VisualView& vv, ObsEval& o) {
  double rho, rho1;
  loss_eval(vv.loss_px, vv.loss_a_px, o.r[0] * o.r[0] + o.r[1] * o.r[1], rho, rho1);
  if (kCorrect) {
    const double w = sqrt(rho1);
    o.r[0] *= w; o.r[1] *= w;
LVBA_UNROLL
    for (int i = 0; i < 12; ++i) o.Jc[i] *= w;
LVBA_UNROLL
    for (int i = 0; i < 6; ++i) o.JX[i] *= w;
  }
  return rho;
}

// Corrector of one plane block (r, J of plane_eval): returns rho(r^2); r and J times sqrt(rho')
LVBA_HD double plane_loss(const VisualView& vv, double& r, double J[3]) {
  double rho, rho1;
  loss_eval(vv.loss_pl, vv.loss_a_pl, r * r, rho, rho1);
  const double w = sqrt(rho1);
  r *= w; J[0] *= w; J[1] *= w; J[2] *= w;
  return rho;
}

LVBA_HD void sym3_inverse(const double* c /*xx xy xz yy yz zz*/, double* o) {
  const double a = c[0], b = c[1], cc = c[2], d = c[3], e = c[4], f = c[5];
  const double A = d * f - e * e, B = cc * e - b * f, Cc = b * e - cc * d;
  const double det = a * A + b * B + cc * Cc;
  const double id = 1.0 / det;
  o[0] = A * id; o[1] = B * id; o[2] = Cc * id;
  o[3] = (a * f - cc * cc) * id; o[4] = (b * cc - a * e) * id; o[5] = (a * d - b * b) * id;
}

}  // namespace lvba
