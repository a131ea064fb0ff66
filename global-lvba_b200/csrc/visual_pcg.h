// visual_pcg.h — ITERATIVE_SCHUR for the visual LM (lvba_visual_opts::linear_solver = LVBA_LINEAR_ITERATIVE_SCHUR):
// preconditioned conjugate gradients on the explicit reduced camera system, the solver Ceres runs for ITERATIVE_SCHUR with
// use_explicit_schur_complement = true and the SCHUR_JACOBI preconditioner.  Ceres is not part of this repository; the rule
// below is restated from the ceres-solver 2.1.0 sources (ConjugateGradientsSolver::Solve,
// BlockRandomAccessDiagonalMatrix::Invert, LevenbergMarquardtStrategy), as SURVEY.md §8 Q9 / Q10 restate the rest of the LM.
//
//   A = S + diag(dadd)  (S in envelope storage, Jacobi-scaled, its diagonal blocks read through their lower triangle as the
//                        LDL^T reads them), b = rhs, x = 0, r = b
//   M^-1 = blockdiag(A_rr)^-1, each damped 6x6 block inverted through its Cholesky factor; a pivot that is not finite and > 0
//   is FAILURE before the first iteration.  ||b|| = 0: x = 0, SUCCESS after 0 iterations.  Q0 = 0.  For i = 1, 2, ...:
//     z = M^-1 r;  rho = r.z                       rho 0 or not finite: FAILURE
//     p = z (i = 1) | z + beta p, beta = rho/rho_prev    beta 0 or not finite: FAILURE
//     q = A p;  pq = p.q                           pq <= 0 or +-inf: NO_CONVERGENCE (x kept); NaN: FAILURE
//     alpha = rho/pq                               alpha not finite: FAILURE
//     x += alpha p;  r = b - A x when i % 10 == 0 (residual_reset_period), else r -= alpha q
//     Q1 = -x.(b + r);  zeta = i (Q1 - Q0)/Q1      zeta < eta and i >= min_iter: SUCCESS
//     Q0 = Q1;  i >= max_iter: NO_CONVERGENCE
// (r_tolerance = -1: LevenbergMarquardtStrategy turns the residual test off.  Ceres lets a NaN run on to the iteration limit;
// here every non-finite rho, beta, pq or alpha stops at once with FAILURE, which the LM treats as an invalid step either way.)
//
// The passes are functors over index ranges, run by CudaExec on the device and by the host policy in the CPU tests.  Every one
// of them is a no-op once the device status word says the solve is done, so the host enqueues the iterations in groups and
// reads the word once per group; the iteration count and the bits do not depend on the group size.  Every dot product is a
// fixed-order two-level sum (chunks of kChunk elements in index order, then the chunks in order), so, given S, the solve has the
// same bits on every run.  The product q = A p is ProdF here; the device runs the warp-per-row visual_pcg_product_kernel
// instead (visual_api.cuh), which agrees with it to rounding.  On a plan that chose the matrix-free product (visual_implicit.h)
// solve_with takes that product and PrecDF, which reads the diagonal blocks that product's build makes instead of S.
#pragma once
#include "env_types.h"
#include "lidar_big.h"     // LVBA_BHD

namespace lvba {
namespace vpcg {

constexpr int kChunk = 256;        // elements per partial of a dot product
constexpr int kResetPeriod = 10;   // Ceres' residual_reset_period
constexpr int kGroup = 10;         // iterations enqueued between two reads of the status word

enum Term { kSuccess = 0, kNoConvergence = 1, kFailure = 2 };
// int status words: done flag, iterations run, termination, a bad preconditioner pivot, 1 for FAILURE (the LM's invalid step)
enum { kDone = 0, kIter, kTerm, kBadPrec, kFail, kNInt };
// double scalars: rho, rho_prev, beta, alpha, Q0
enum { kRho = 0, kRhoPrev, kBeta, kAlpha, kQ0, kNDouble };

struct Ctl {
  int* si;        // [kNInt]
  double* sd;     // [kNDouble]
  double* part;   // [chunks(n6)]
  LVBA_BHD bool done() const { return si[kDone] != 0; }
  LVBA_BHD void stop(int term) const { si[kDone] = 1; si[kTerm] = term; si[kFail] = term == kFailure; }
};
LVBA_BHD int64_t chunks(int64_t n6) { return (n6 + kChunk - 1) / kChunk; }
LVBA_BHD bool zero_or_not_finite(double v) { return v == 0.0 || !(v - v == 0.0); }

// element (a, b) of the symmetric diagonal block at d (its lower triangle)
LVBA_BHD double sym(const double* d, int a, int b) { return a >= b ? d[a * 6 + b] : d[b * 6 + a]; }

// the status words of a new solve
struct StartF {
  Ctl c;
  LVBA_BHD void operator()(int64_t) const {
    for (int i = 0; i < kNInt; ++i) c.si[i] = 0;
    for (int i = 0; i < kNDouble; ++i) c.sd[i] = 0.0;
  }
};

// out = (d + diag(dadd_r))^-1 of the symmetric 6x6 block d (read through its lower triangle) through its Cholesky factor;
// false for a pivot that is not finite and > 0
LVBA_BHD bool prec_block(const double* d, const double* dadd_r, double* out) {
  double L[36], Li[36];
  for (int i = 0; i < 36; ++i) { L[i] = 0.0; Li[i] = 0.0; }
  bool ok = true;
  for (int j = 0; j < 6; ++j) {
    double v = sym(d, j, j) + dadd_r[j];
    for (int m = 0; m < j; ++m) v -= L[j * 6 + m] * L[j * 6 + m];
    if (!(v > 0.0 && v <= 1.7976931348623157e308)) { ok = false; v = 1.0; }
    const double l = sqrt(v);
    L[j * 6 + j] = l;
    for (int i = j + 1; i < 6; ++i) {
      double w = sym(d, i, j);
      for (int m = 0; m < j; ++m) w -= L[i * 6 + m] * L[j * 6 + m];
      L[i * 6 + j] = w / l;
    }
  }
  for (int j = 0; j < 6; ++j)                          // Li = L^-1, column by column
    for (int i = j; i < 6; ++i) {
      double w = i == j ? 1.0 : 0.0;
      for (int m = j; m < i; ++m) w -= L[i * 6 + m] * Li[m * 6 + j];
      Li[i * 6 + j] = w / L[i * 6 + i];
    }
  for (int a = 0; a < 6; ++a)                          // L^-T L^-1
    for (int b = 0; b < 6; ++b) {
      double w = 0.0;
      for (int m = a > b ? a : b; m < 6; ++m) w += Li[m * 6 + a] * Li[m * 6 + b];
      out[a * 6 + b] = w;
    }
  return ok;
}

// minv[36 r] = (S_rr + diag(dadd_r))^-1 through its Cholesky factor; a pivot that is not finite and > 0 sets kBadPrec
struct PrecF {
  EnvView e; const double* S; const double* dadd; double* minv; Ctl c;
  LVBA_BHD void operator()(int64_t r) const {
    if (!prec_block(S + 36 * (e.row_start[r] + (r - e.first[r])), dadd + 6 * r, minv + 36 * r)) c.si[kBadPrec] = 1;
  }
};

// the same from the diagonal blocks D [n][36] of the matrix-free product (visual_implicit.h)
struct PrecDF {
  const double* D; const double* dadd; double* minv; Ctl c;
  LVBA_BHD void operator()(int64_t r) const {
    if (!prec_block(D + 36 * r, dadd + 6 * r, minv + 36 * r)) c.si[kBadPrec] = 1;
  }
};

// x = 0, r = b
struct InitF {
  const double* b; double* x; double* r;
  LVBA_BHD void operator()(int64_t i) const { x[i] = 0.0; r[i] = b[i]; }
};

// part[k] = sum over the elements i of chunk k, in order, of u[i] (v[i] + w[i]) (w may be null)
struct DotF {
  Ctl c; int64_t n6; const double* u; const double* v; const double* w; bool always;
  LVBA_BHD void operator()(int64_t k) const {
    if (!always && c.done()) return;
    const int64_t i1 = (k + 1) * kChunk < n6 ? (k + 1) * kChunk : n6;
    double s = 0.0;
    for (int64_t i = k * kChunk; i < i1; ++i) s += u[i] * (w ? v[i] + w[i] : v[i]);
    c.part[k] = s;
  }
};
LVBA_BHD double sum_parts(const Ctl& c, int64_t nch) {
  double s = 0.0;
  for (int64_t k = 0; k < nch; ++k) s += c.part[k];
  return s;
}

// before the first iteration: ||b|| = 0 is SUCCESS after 0 iterations, a bad preconditioner pivot FAILURE
struct CheckF {
  Ctl c; int64_t nch;
  LVBA_BHD void operator()(int64_t) const {
    if (sum_parts(c, nch) == 0.0) c.stop(kSuccess);
    else if (c.si[kBadPrec]) c.stop(kFailure);
  }
};

// z = M^-1 r, one item per block row
struct ZF {
  Ctl c; const double* minv; const double* r; double* z;
  LVBA_BHD void operator()(int64_t row) const {
    if (c.done()) return;
    const double* m = minv + 36 * row;
    const double* rr = r + 6 * row;
    for (int a = 0; a < 6; ++a) {
      double w = 0.0;
      for (int b = 0; b < 6; ++b) w += m[a * 6 + b] * rr[b];
      z[6 * row + a] = w;
    }
  }
};

// iteration i begins: rho = r.z and beta
struct RhoF {
  Ctl c; int64_t nch; int i;
  LVBA_BHD void operator()(int64_t) const {
    if (c.done()) return;
    c.si[kIter] = i;
    c.sd[kRhoPrev] = c.sd[kRho];
    const double rho = sum_parts(c, nch);
    c.sd[kRho] = rho;
    if (zero_or_not_finite(rho)) { c.stop(kFailure); return; }
    if (i > 1) {
      const double beta = rho / c.sd[kRhoPrev];
      if (zero_or_not_finite(beta)) { c.stop(kFailure); return; }
      c.sd[kBeta] = beta;
    }
  }
};

// p = z (first iteration) or z + beta p
struct PF {
  Ctl c; const double* z; double* p; bool first;
  LVBA_BHD void operator()(int64_t i) const {
    if (c.done()) return;
    p[i] = first ? z[i] : z[i] + c.sd[kBeta] * p[i];
  }
};

// pq = p.q and alpha
struct AlphaF {
  Ctl c; int64_t nch;
  LVBA_BHD void operator()(int64_t) const {
    if (c.done()) return;
    const double pq = sum_parts(c, nch);
    if (pq != pq) { c.stop(kFailure); return; }
    if (pq <= 0.0 || !(pq - pq == 0.0)) { c.stop(kNoConvergence); return; }
    const double alpha = c.sd[kRho] / pq;
    if (!(alpha - alpha == 0.0)) { c.stop(kFailure); return; }
    c.sd[kAlpha] = alpha;
  }
};

// x += alpha p; r -= alpha q unless this iteration resets r (ResetF)
struct XF {
  Ctl c; const double* p; const double* q; double* x; double* r; bool reset;
  LVBA_BHD void operator()(int64_t i) const {
    if (c.done()) return;
    const double a = c.sd[kAlpha];
    x[i] += a * p[i];
    if (!reset) r[i] -= a * q[i];
  }
};

// r = b - A x (ax: the product of x)
struct ResetF {
  Ctl c; const double* b; const double* ax; double* r;
  LVBA_BHD void operator()(int64_t i) const {
    if (c.done()) return;
    r[i] = b[i] - ax[i];
  }
};

// Q1 = -x.(b + r), zeta, and the end of iteration i
struct ZetaF {
  Ctl c; int64_t nch; int i; double eta; int min_iter, max_iter;
  LVBA_BHD void operator()(int64_t) const {
    if (c.done()) return;
    const double Q1 = -sum_parts(c, nch);
    const double zeta = i * (Q1 - c.sd[kQ0]) / Q1;
    if (zeta < eta && i >= min_iter) { c.stop(kSuccess); return; }
    c.sd[kQ0] = Q1;
    if (i >= max_iter) c.stop(kNoConvergence);
  }
};

// y = A x, one item per block row in a fixed order: the row's blocks left to right (the diagonal block through its lower
// triangle), then the transposes of the blocks below it top to bottom, then the damping
struct ProdF {
  Ctl c; EnvView e; const double* S; const double* dadd; const double* x; double* y;
  LVBA_BHD void operator()(int64_t r) const {
    if (c.done()) return;
    double acc[6] = {0, 0, 0, 0, 0, 0};
    const double* row = S + 36 * e.row_start[r];
    for (int col = e.first[r]; col < r; ++col) {
      const double* blk = row + 36 * (col - e.first[r]);
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) acc[a] += blk[a * 6 + b] * x[6 * col + b];
    }
    const double* d = row + 36 * (r - e.first[r]);
    for (int a = 0; a < 6; ++a)
      for (int b = 0; b < 6; ++b) acc[a] += sym(d, a, b) * x[6 * r + b];
    for (int r2 = (int)r + 1; r2 <= e.last[r]; ++r2) {
      const double* blk = S + 36 * (e.row_start[r2] + (r - e.first[r2]));
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) acc[b] += blk[a * 6 + b] * x[6 * r2 + a];
    }
    for (int a = 0; a < 6; ++a) y[6 * r + a] = acc[a] + dadd[6 * r + a] * x[6 * r + a];
  }
};

struct Bufs {
  double *r, *z, *p, *q, *minv;
  Ctl c;
};
struct Params { double eta; int min_iter, max_iter; };

// The whole solve of A x = b over n block rows.  prec is the preconditioner's pass (PrecF or PrecDF, one item per row),
// prod(in, out) enqueues out = A in (a no-op once the solve is done).  The status words come to the host once before the first
// iteration and once per kGroup iterations; si_host [kNInt] holds the last copy, so after the return si_host[kIter] / [kTerm] /
// [kFail] describe the solve.
template <class Exec, class Prec, class Prod>
int solve_with(Exec& ex, int64_t n, const Prec& prec, const double* b, double* x, const Bufs& B, const Params& o, const Prod& prod,
               int* si_host, int64_t* d2h) {
  const int64_t n6 = 6 * n, nch = chunks(n6);
  const Ctl& c = B.c;
  int rc;
  if ((rc = ex.for_each(1, StartF{c}))) return rc;
  if ((rc = ex.for_each(n, prec))) return rc;
  if ((rc = ex.for_each(n6, InitF{b, x, B.r}))) return rc;
  if ((rc = ex.for_each(nch, DotF{c, n6, b, b, nullptr, true}))) return rc;
  if ((rc = ex.for_each(1, CheckF{c, nch}))) return rc;
  if ((rc = ex.fetch(si_host, c.si, kNInt))) return rc;
  *d2h += sizeof(int) * kNInt;
  for (int i = 1; !si_host[kDone] && i <= o.max_iter; ++i) {
    if ((rc = ex.for_each(n, ZF{c, B.minv, B.r, B.z}))) return rc;
    if ((rc = ex.for_each(nch, DotF{c, n6, B.r, B.z, nullptr, false}))) return rc;
    if ((rc = ex.for_each(1, RhoF{c, nch, i}))) return rc;
    if ((rc = ex.for_each(n6, PF{c, B.z, B.p, i == 1}))) return rc;
    if ((rc = prod(B.p, B.q))) return rc;
    if ((rc = ex.for_each(nch, DotF{c, n6, B.p, B.q, nullptr, false}))) return rc;
    if ((rc = ex.for_each(1, AlphaF{c, nch}))) return rc;
    const bool reset = i % kResetPeriod == 0;
    if ((rc = ex.for_each(n6, XF{c, B.p, B.q, x, B.r, reset}))) return rc;
    if (reset) {
      if ((rc = prod(x, B.q))) return rc;
      if ((rc = ex.for_each(n6, ResetF{c, b, B.q, B.r}))) return rc;
    }
    if ((rc = ex.for_each(nch, DotF{c, n6, x, b, B.r, false}))) return rc;
    if ((rc = ex.for_each(1, ZetaF{c, nch, i, o.eta, o.min_iter, o.max_iter}))) return rc;
    if (i % kGroup == 0 || i == o.max_iter) {
      if ((rc = ex.fetch(si_host, c.si, kNInt))) return rc;
      *d2h += sizeof(int) * kNInt;
    }
  }
  return 0;
}

// the solve on the explicit S in envelope storage
template <class Exec, class Prod>
int solve(Exec& ex, const EnvView& e, const double* S, const double* dadd, const double* b, double* x, const Bufs& B,
          const Params& o, const Prod& prod, int* si_host, int64_t* d2h) {
  return solve_with(ex, e.n, PrecF{e, S, dadd, B.minv, B.c}, b, x, B, o, prod, si_host, d2h);
}

}  // namespace vpcg
}  // namespace lvba
