// common.cuh — device-side small FP64 linear algebra shared by the LVBA kernels (sm_90a).
// All 3x3 / 6x6 products are register-resident scalar FP64 (DFMA); no tensor cores (north star).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "vec3.h"

#define LVBA_DEV __device__ __forceinline__

namespace lvba {

// SMs of the target GPU (H100 SXM): caps the grids of the grid-stride passes at a few CTAs per SM
constexpr int kNumSMs = 132;

// ---------------------------------------------------------------- vectorised global loads
LVBA_DEV double2 ldg2(const double2* p) { return __ldg(p); }

// ---------------------------------------------------------------- 3x3 helpers (row-major double[9])
LVBA_DEV void mat3_mul(const double* A, const double* B, double* C) {   // C = A B
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
LVBA_DEV void mat3_mul_bt(const double* A, const double* B, double* C) {  // C = A B^T
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      C[3 * i + j] = A[3 * i] * B[3 * j] + A[3 * i + 1] * B[3 * j + 1] + A[3 * i + 2] * B[3 * j + 2];
}
LVBA_DEV void mat3_vec(const double* A, const double* x, double* y) {    // y = A x
#pragma unroll
  for (int i = 0; i < 3; ++i) y[i] = A[3 * i] * x[0] + A[3 * i + 1] * x[1] + A[3 * i + 2] * x[2];
}
LVBA_DEV void mat3t_vec(const double* A, const double* x, double* y) {   // y = A^T x
#pragma unroll
  for (int i = 0; i < 3; ++i) y[i] = A[i] * x[0] + A[3 + i] * x[1] + A[6 + i] * x[2];
}
// cross3, dot3, hat3: vec3.h
// A * hat(w) without forming hat:  (A hat(w))_{:,0} = A_{:,1} w2 - A_{:,2} w1, ...
LVBA_DEV void mat3_mul_hat(const double* A, const double* w, double* C) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double a0 = A[3 * i], a1 = A[3 * i + 1], a2 = A[3 * i + 2];
    C[3 * i + 0] = a1 * w[2] - a2 * w[1];
    C[3 * i + 1] = a2 * w[0] - a0 * w[2];
    C[3 * i + 2] = a0 * w[1] - a1 * w[0];
  }
}
// hat(w) * A : row i of result = w x (columns)  ->  (hat(w) A)_{0,:} = -w2 A_{1,:} + w1 A_{2,:}
LVBA_DEV void hat_mul_mat3(const double* w, const double* A, double* C) {
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const double a0 = A[j], a1 = A[3 + j], a2 = A[6 + j];
    C[j] = -w[2] * a1 + w[1] * a2;
    C[3 + j] = w[2] * a0 - w[0] * a2;
    C[6 + j] = -w[1] * a0 + w[0] * a1;
  }
}

// ---------------------------------------------------------------- symmetric 3x3 eigen solver
// Cyclic Jacobi in FP64; replaces Eigen::SelfAdjointEigenSolver<Matrix3d> (bavoxel.hpp:98,198):
// eigenvalues ascending, eigenvectors as columns U[:,k] stored as u[k][0..2]. Eigenvector sign
// is irrelevant for the path (every use is even in u — SURVEY.md Q6).
template <bool kVectors>
LVBA_DEV void eig3_sym(double a00, double a01, double a02, double a11, double a12, double a22,
                       double lam[3], double u[3][3]) {
  double v[3][3];
  if (kVectors) {
    v[0][0] = 1; v[0][1] = 0; v[0][2] = 0;
    v[1][0] = 0; v[1][1] = 1; v[1][2] = 0;
    v[2][0] = 0; v[2][1] = 0; v[2][2] = 1;
  }
#define LVBA_JROT(app, aqq, apq, apr, aqr, P, Q)                                        \
  if (fabs(apq) > 1e-22 * (fabs(app) + fabs(aqq)) && apq != 0.0) {                      \
    const double theta = (aqq - app) / (2.0 * apq);                                     \
    const double tt = copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0)); \
    const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;                             \
    app -= tt * apq; aqq += tt * apq; apq = 0.0;                                        \
    const double t1 = c * apr - s * aqr, t2 = s * apr + c * aqr;                        \
    apr = t1; aqr = t2;                                                                 \
    if (kVectors) {                                                                     \
      _Pragma("unroll") for (int k = 0; k < 3; ++k) {                                   \
        const double vp = v[k][P], vq = v[k][Q];                                        \
        v[k][P] = c * vp - s * vq; v[k][Q] = s * vp + c * vq;                           \
      }                                                                                 \
    }                                                                                   \
    ++rot;                                                                              \
  }
  for (int sweep = 0; sweep < 12; ++sweep) {
    int rot = 0;
    LVBA_JROT(a00, a11, a01, a02, a12, 0, 1)
    LVBA_JROT(a00, a22, a02, a01, a12, 0, 2)
    LVBA_JROT(a11, a22, a12, a01, a02, 1, 2)
    if (rot == 0) break;
  }
#undef LVBA_JROT
  // sort ascending (3-element network)
  double l0 = a00, l1 = a11, l2 = a22;
  int i0 = 0, i1 = 1, i2 = 2;
  if (l0 > l1) { double t = l0; l0 = l1; l1 = t; int k = i0; i0 = i1; i1 = k; }
  if (l1 > l2) { double t = l1; l1 = l2; l2 = t; int k = i1; i1 = i2; i2 = k; }
  if (l0 > l1) { double t = l0; l0 = l1; l1 = t; int k = i0; i0 = i1; i1 = k; }
  lam[0] = l0; lam[1] = l1; lam[2] = l2;
  if (kVectors) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      // dynamic column select without local-memory indexing
      u[0][k] = (i0 == 0) ? v[k][0] : (i0 == 1) ? v[k][1] : v[k][2];
      u[1][k] = (i1 == 0) ? v[k][0] : (i1 == 1) ? v[k][1] : v[k][2];
      u[2][k] = (i2 == 0) ? v[k][0] : (i2 == 1) ? v[k][1] : v[k][2];
    }
  }
}

// Smallest eigenvalue only (the residual-only pass: lambda_0 of every voxel, bavoxel.hpp:176-203 keeps nothing else).
// Newton on the characteristic polynomial from 0: for a positive semi-definite matrix 0 <= lambda_0 lies left of every root,
// where the iteration increases monotonically to lambda_0 and converges quadratically — 4 to 6 steps of one division and
// six FMAs for a plane voxel (lambda_0 << lambda_1), against ~15 Jacobi rotations with a division and two square roots each.
// The root's error is eps |A|^3 / ((lambda_1 - lambda_0)(lambda_2 - lambda_0)) = eps |A|^3 / |p'(lambda_0)|: when the two
// smallest eigenvalues are close (|p'| < 1e-2 tr^2), or the iteration has not settled, the Jacobi solver decides.
LVBA_DEV double sym3_smallest_eigenvalue(double a00, double a01, double a02, double a11, double a12, double a22) {
  const double m00 = a11 * a22 - a12 * a12, m01 = a01 * a22 - a12 * a02, m02 = a01 * a12 - a11 * a02;
  const double c2 = a00 + a11 + a22;
  const double c1 = m00 + (a00 * a22 - a02 * a02) + (a00 * a11 - a01 * a01);
  const double c0 = a00 * m00 - a01 * m01 + a02 * m02;
  double lam = 0.0, fp = -c1;
  bool settled = false;
#pragma unroll 1
  for (int it = 0; it < 10; ++it) {
    const double f = fma(fma(c2 - lam, lam, -c1), lam, c0);
    fp = fma(fma(-3.0, lam, 2.0 * c2), lam, -c1);
    const double d = f / fp;
    lam -= d;
    if (fabs(d) <= 1e-16 * fabs(c2)) { settled = true; break; }
  }
  if (settled && fabs(fp) >= 1e-2 * c2 * c2) return lam;
  double l[3], u[3][3];
  eig3_sym<false>(a00, a01, a02, a11, a12, a22, l, u);
  return l[0];
}

// Full eigen-decomposition of a plane voxel's covariance without the Jacobi sweeps (one warp of a batch CTA solves ~18 of them
// while the other three wait: a third of the CTA's life in lidar_build_kernel): lambda_0 by the Newton iteration above, its
// eigenvector as the largest cross product of two rows of A - lambda_0 I (rank 2), the other two pairs from the 2 x 2 problem in
// the plane orthogonal to it (one Jacobi rotation).  Residuals |A u - lambda u| and orthogonality ~1e-15 |A| whenever
// |p'(lambda_0)| = (lambda_1 - lambda_0)(lambda_2 - lambda_0) >= 1e-2 tr^2; otherwise eig3_sym decides.  Eigenvalues ascending,
// u[k] = eigenvector k; signs undefined, as with every other solver (every use is even in u, SURVEY.md Q6).
LVBA_DEV void eig3_sym_plane(double a00, double a01, double a02, double a11, double a12, double a22, double lam[3], double u[3][3]) {
  const double m00 = a11 * a22 - a12 * a12, m01 = a01 * a22 - a12 * a02, m02 = a01 * a12 - a11 * a02;
  const double c2 = a00 + a11 + a22;
  const double c1 = m00 + (a00 * a22 - a02 * a02) + (a00 * a11 - a01 * a01);
  const double c0 = a00 * m00 - a01 * m01 + a02 * m02;
  double l0 = 0.0, fp = -c1;
  bool settled = false;
#pragma unroll 1
  for (int it = 0; it < 10; ++it) {
    const double f = fma(fma(c2 - l0, l0, -c1), l0, c0);
    fp = fma(fma(-3.0, l0, 2.0 * c2), l0, -c1);
    const double d = f / fp;
    l0 -= d;
    if (fabs(d) <= 1e-16 * fabs(c2)) { settled = true; break; }
  }
  if (!(settled && fabs(fp) >= 1e-2 * c2 * c2)) { eig3_sym<true>(a00, a01, a02, a11, a12, a22, lam, u); return; }
  // null vector of M = A - l0 I
  const double r0[3] = {a00 - l0, a01, a02}, r1[3] = {a01, a11 - l0, a12}, r2[3] = {a02, a12, a22 - l0};
  double x01[3], x02[3], x12[3];
  cross3(r0, r1, x01); cross3(r0, r2, x02); cross3(r1, r2, x12);
  const double n01 = dot3(x01, x01), n02 = dot3(x02, x02), n12 = dot3(x12, x12);
  double e0[3], nn = n01;
  e0[0] = x01[0]; e0[1] = x01[1]; e0[2] = x01[2];
  if (n02 > nn) { nn = n02; e0[0] = x02[0]; e0[1] = x02[1]; e0[2] = x02[2]; }
  if (n12 > nn) { nn = n12; e0[0] = x12[0]; e0[1] = x12[1]; e0[2] = x12[2]; }
  const double in0 = rsqrt(nn);
  // rsqrt is not correctly rounded: one normalisation step more keeps |u0| = 1 to the last bits
  e0[0] *= in0; e0[1] *= in0; e0[2] *= in0;
  { const double fix = 1.0 / sqrt(dot3(e0, e0)); e0[0] *= fix; e0[1] *= fix; e0[2] *= fix; }
  // orthonormal basis of the plane: v1 = u0 x e_axis (axis of the smallest |u0| component), v2 = u0 x v1
  const double ax = fabs(e0[0]), ay = fabs(e0[1]), az = fabs(e0[2]);
  double v1[3];
  if (ax <= ay && ax <= az) { v1[0] = 0.0; v1[1] = e0[2]; v1[2] = -e0[1]; }
  else if (ay <= az) { v1[0] = -e0[2]; v1[1] = 0.0; v1[2] = e0[0]; }
  else { v1[0] = e0[1]; v1[1] = -e0[0]; v1[2] = 0.0; }
  { const double fix = 1.0 / sqrt(dot3(v1, v1)); v1[0] *= fix; v1[1] *= fix; v1[2] *= fix; }
  double v2[3];
  cross3(e0, v1, v2);
  const double Av1[3] = {a00 * v1[0] + a01 * v1[1] + a02 * v1[2], a01 * v1[0] + a11 * v1[1] + a12 * v1[2], a02 * v1[0] + a12 * v1[1] + a22 * v1[2]};
  const double Av2[3] = {a00 * v2[0] + a01 * v2[1] + a02 * v2[2], a01 * v2[0] + a11 * v2[1] + a12 * v2[2], a02 * v2[0] + a12 * v2[1] + a22 * v2[2]};
  const double b11 = dot3(v1, Av1), b12 = dot3(v1, Av2), b22 = dot3(v2, Av2);
  double l1 = b11, l2 = b22, c = 1.0, sn = 0.0;
  if (b12 != 0.0) {
    const double theta = (b22 - b11) / (2.0 * b12);
    const double t = copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
    c = 1.0 / sqrt(t * t + 1.0); sn = t * c;
    l1 = b11 - t * b12; l2 = b22 + t * b12;
  }
  double w1[3], w2[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) { w1[k] = c * v1[k] - sn * v2[k]; w2[k] = sn * v1[k] + c * v2[k]; }
  const bool swap = l1 > l2;
  lam[0] = l0; lam[1] = swap ? l2 : l1; lam[2] = swap ? l1 : l2;
#pragma unroll
  for (int k = 0; k < 3; ++k) { u[0][k] = e0[k]; u[1][k] = swap ? w2[k] : w1[k]; u[2][k] = swap ? w1[k] : w2[k]; }
}

// ---------------------------------------------------------------- Rodrigues, reference tools.hpp:62-77
LVBA_DEV void so3_exp(const double* w, double* R) {
  const double th = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (th >= 1e-11) {
    const double a[3] = {w[0] / th, w[1] / th, w[2] / th};
    double s, c;
    sincos(th, &s, &c);
    double K[9], KK[9];
    hat3(a, K);
    mat3_mul(K, K, KK);
    const double oc = 1.0 - c;
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = s * K[i] + oc * KK[i];
    R[0] += 1.0; R[4] += 1.0; R[8] += 1.0;
  } else {
    R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
  }
}

// ---------------------------------------------------------------- block reductions
LVBA_DEV double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// deterministic block sum; `red` is >= 32 doubles of shared memory; result valid in thread 0
template <int kThreads>
LVBA_DEV double block_sum(double v, double* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) red[w] = v;
  __syncthreads();
  double r = 0.0;
  if (w == 0) {
    r = (lane < kThreads / 32) ? red[lane] : 0.0;
    r = warp_sum(r);
  }
  __syncthreads();
  return r;
}

}  // namespace lvba
