// lidar_big.h — path A for voxels seen from MORE poses than one batch CTA holds (K > kSlots = 128).
//
// The batch kernels of lidar.cuh keep a whole voxel in one 128-thread CTA.  A room scanned for minutes gives floor and
// wall voxels that hundreds of anchor poses see; the reference's VOX_HESS::acc_evaluate2 (include/BALM/bavoxel.hpp:68-174)
// simply loops over them.  Those voxels are taken out of the batches and go through the three passes below, which restate
// the same arithmetic slot by slot and pair by pair with the contributions added into H and g by atomics:
//
//   params  (one item per big voxel)   merged world-frame cluster (tools.hpp:450-456), covariance, ascending eigen system,
//                                      u_k = u_0, umumT = sum_{m=1,2} 2/(l0 - lm) um um^T (:98-110), lambda_0 -> residual
//   slots   (one item per slot)        A_i = d(cov u_k)/d(pose i) (:112-140), g_i = A_i^T u_k, the diagonal block H_ii (:141-149)
//   pairs   (one item per slot pair)   the off-diagonal block H_ij (:151-167), stored as its transpose in the LOWER envelope
//
// The residual-only pass (evaluate_only_residual, :176-203) is `params` alone.  Functors over index ranges, compiled for the
// device by lidar_api.cuh and, for the CPU check of the arithmetic against oracle/lidar_oracle.py, by tests/emu/.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define LVBA_BHD __host__ __device__ __forceinline__
#else
#define LVBA_BHD inline
#endif

namespace lvba {
namespace big {

LVBA_BHD void atomic_add_f64(double* p, double v) {
#if defined(__CUDA_ARCH__)
  atomicAdd(p, v);
#else
  *p += v;
#endif
}

constexpr int kFeat = 22;       // per slot: A (3x6 row-major), w = v x R^T u_k (3), n
constexpr int kParams = 20;     // per voxel: u_k (3), umumT (9), vbar (3), NN, lambda0..2, valid

struct View {
  int64_t n_vox;                // big voxels
  const int64_t* vox_ptr;       // [n_vox + 1] slot offsets into the arrays below
  const int32_t* pose_idx;      // [n_slots]
  const double* clusters;       // [n_slots * 10] body-frame AoS records
  const int64_t* pair_ptr;      // [n_vox + 1] prefix sums of K (K - 1) / 2
  // envelope of the pose system
  const int* first;
  const long long* row_start;
  // constant poses (lvba_lidar_opts::pose_fixed): row_of[pose] = its row, -1 for a constant pose; null: every pose is its own
  // row.  A slot or pair of a constant pose adds nothing to H and g; its deterministic record gets no destination (nblocks
  // for H, W for g: the destination counts of tiles::FixedSum in lidar_det_index).
  const int* row_of = nullptr;
  int64_t nblocks = 0;
  int W = 0;
};

LVBA_BHD int row_of_pose(const View& bv, int pose) { return bv.row_of ? bv.row_of[pose] : pose; }

LVBA_BHD void mat3_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
LVBA_BHD void hat3(const double* v, double* H) {                      // tools.hpp:105-112
  H[0] = 0.0; H[1] = -v[2]; H[2] = v[1];
  H[3] = v[2]; H[4] = 0.0; H[5] = -v[0];
  H[6] = -v[1]; H[7] = v[0]; H[8] = 0.0;
}

// cyclic Jacobi, eigenvalues ascending with their vectors (columns U[:, m] returned as u[m][0..2])
LVBA_BHD void eig3_full(const double C[9], double lam[3], double u[3][3]) {
  double a[3][3] = {{C[0], C[1], C[2]}, {C[1], C[4], C[5]}, {C[2], C[5], C[8]}};
  double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int sweep = 0; sweep < 16; ++sweep) {
    int rot = 0;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        const double apq = a[p][q];
        if (apq == 0.0 || !(fabs(apq) > 1e-22 * (fabs(a[p][p]) + fabs(a[q][q])))) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
        const double t = copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) { const double akp = a[k][p], akq = a[k][q]; a[k][p] = c * akp - s * akq; a[k][q] = s * akp + c * akq; }
        for (int k = 0; k < 3; ++k) { const double apk = a[p][k], aqk = a[q][k]; a[p][k] = c * apk - s * aqk; a[q][k] = s * apk + c * aqk; }
        for (int k = 0; k < 3; ++k) { const double vkp = v[k][p], vkq = v[k][q]; v[k][p] = c * vkp - s * vkq; v[k][q] = s * vkp + c * vkq; }
        ++rot;
      }
    if (!rot) break;
  }
  int o[3] = {0, 1, 2};
  const double l[3] = {a[0][0], a[1][1], a[2][2]};
  if (l[o[0]] > l[o[1]]) { const int k = o[0]; o[0] = o[1]; o[1] = k; }
  if (l[o[1]] > l[o[2]]) { const int k = o[1]; o[1] = o[2]; o[2] = k; }
  if (l[o[0]] > l[o[1]]) { const int k = o[0]; o[0] = o[1]; o[1] = k; }
  for (int m = 0; m < 3; ++m) { lam[m] = l[o[m]]; for (int k = 0; k < 3; ++k) u[m][k] = v[k][o[m]]; }
}

struct ParamsF {               // one item per big voxel
  View bv; const double* poses; double* params; double* residual;   // residual[b] = lambda_0 of voxel b
  LVBA_BHD void operator()(int64_t b) const {
    double Pm[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, vm[3] = {0, 0, 0}, Nm = 0.0;
    for (int64_t s = bv.vox_ptr[b]; s < bv.vox_ptr[b + 1]; ++s) {      // PointCluster::transform + operator+=  (tools.hpp:434-456)
      const double* c = bv.clusters + 10 * s;
      const double* R = poses + 12 * (int64_t)bv.pose_idx[s];
      const double* t = R + 9;
      const double P[9] = {c[0], c[1], c[2], c[1], c[3], c[4], c[2], c[4], c[5]};
      double RP[9], Rv[3];
      mat3_mul(R, P, RP);
      for (int i = 0; i < 3; ++i) Rv[i] = R[3 * i] * c[6] + R[3 * i + 1] * c[7] + R[3 * i + 2] * c[8];
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
          Pm[3 * i + j] += (RP[3 * i] * R[3 * j] + RP[3 * i + 1] * R[3 * j + 1] + RP[3 * i + 2] * R[3 * j + 2]) + Rv[i] * t[j] + Rv[j] * t[i] + c[9] * t[i] * t[j];
      for (int i = 0; i < 3; ++i) vm[i] += Rv[i] + c[9] * t[i];
      Nm += c[9];
    }
    double vbar[3], C[9], lam[3], u[3][3];
    for (int i = 0; i < 3; ++i) vbar[i] = vm[i] / Nm;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) C[3 * i + j] = Pm[3 * i + j] / Nm - vbar[i] * vbar[j];
    eig3_full(C, lam, u);
    double* q = params + kParams * b;
    for (int i = 0; i < 3; ++i) q[i] = u[0][i];                                   // u_k = u_0  (:100)
    for (int i = 0; i < 9; ++i) q[3 + i] = 0.0;
    for (int m = 1; m < 3; ++m) {                                                 // :107-110
      const double w = 2.0 / (lam[0] - lam[m]);
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) q[3 + 3 * i + j] += w * u[m][i] * u[m][j];
    }
    for (int i = 0; i < 3; ++i) q[12 + i] = vbar[i];
    q[15] = trunc(Nm);                                                            // int NN = sig.N  (:101)
    q[16] = lam[0]; q[17] = lam[1]; q[18] = lam[2]; q[19] = 1.0;
    residual[b] = lam[0];
  }
};

// kDet = false: the contributions go into H and g by atomics; true (deterministic mode): H = the slots' records [n_slots][36]
// and g = [n_slots][6], one record per slot, summed per destination by tiles::GatherF (lidar_tiles.h) in slot order.
template <bool kDet>
struct SlotsPass {             // one item per slot of the big voxels
  View bv; const double* poses; const double* params; double* feat; double* H; double* g;
  LVBA_BHD void operator()(int64_t s) const {
    int64_t lo = 0, hi = bv.n_vox;                                                // voxel of the slot
    while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if (bv.vox_ptr[mid] <= s) lo = mid; else hi = mid; }
    const double* q = params + kParams * lo;
    const double* uk = q; const double* um = q + 3; const double* vbar = q + 12;
    const double NN = q[15];
    const double* c = bv.clusters + 10 * s;
    const int pose = bv.pose_idx[s];
    const double* R = poses + 12 * (int64_t)pose;
    const double* t = R + 9;
    const double P[9] = {c[0], c[1], c[2], c[1], c[3], c[4], c[2], c[4], c[5]};
    const double* v = c + 6;
    const double n = c[9];
    double RiTuk[3], PiRiTuk[3], w[3], ti_v[3], Rv[3], combo2[3];
    for (int i = 0; i < 3; ++i) RiTuk[i] = R[i] * uk[0] + R[3 + i] * uk[1] + R[6 + i] * uk[2];
    for (int i = 0; i < 3; ++i) PiRiTuk[i] = P[3 * i] * RiTuk[0] + P[3 * i + 1] * RiTuk[1] + P[3 * i + 2] * RiTuk[2];
    w[0] = v[1] * RiTuk[2] - v[2] * RiTuk[1]; w[1] = v[2] * RiTuk[0] - v[0] * RiTuk[2]; w[2] = v[0] * RiTuk[1] - v[1] * RiTuk[0];   // hat(v) R^T u_k
    for (int i = 0; i < 3; ++i) ti_v[i] = t[i] - vbar[i];
    const double ukTti_v = uk[0] * ti_v[0] + uk[1] * ti_v[1] + uk[2] * ti_v[2];
    double combo1[9], vhat[9], RiTukhat[9];
    hat3(PiRiTuk, combo1); hat3(v, vhat); hat3(RiTuk, RiTukhat);
    for (int i = 0; i < 9; ++i) combo1[i] += vhat[i] * ukTti_v;
    for (int i = 0; i < 3; ++i) Rv[i] = R[3 * i] * v[0] + R[3 * i + 1] * v[1] + R[3 * i + 2] * v[2];
    for (int i = 0; i < 3; ++i) combo2[i] = Rv[i] + n * ti_v[i];
    // A = [ (R P + ti_v v^T) hat(R^T u_k) - R combo1 | combo2 u_k^T + (combo2 . u_k) I ] / NN        (3 x 6)
    double M[9], MR[9], Rc1[9], A[18];
    mat3_mul(R, P, M);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) M[3 * i + j] += ti_v[i] * v[j];
    mat3_mul(M, RiTukhat, MR);
    mat3_mul(R, combo1, Rc1);
    const double c2uk = combo2[0] * uk[0] + combo2[1] * uk[1] + combo2[2] * uk[2];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        A[6 * i + j] = (MR[3 * i + j] - Rc1[3 * i + j]) / NN;
        A[6 * i + 3 + j] = (combo2[i] * uk[j] + (i == j ? c2uk : 0.0)) / NN;
      }
    double jjt[6];
    for (int j = 0; j < 6; ++j) jjt[j] = A[j] * uk[0] + A[6 + j] * uk[1] + A[12 + j] * uk[2];      // A^T u_k
    double* f = feat + kFeat * s;
    for (int i = 0; i < 18; ++i) f[i] = A[i];
    f[18] = w[0]; f[19] = w[1]; f[20] = w[2]; f[21] = n;
    // ---- diagonal block (:141-149)
    double UA[18], Hd[36];
    for (int a = 0; a < 3; ++a)
      for (int j = 0; j < 6; ++j) UA[6 * a + j] = um[3 * a] * A[j] + um[3 * a + 1] * A[6 + j] + um[3 * a + 2] * A[12 + j];
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) Hd[6 * i + j] = A[i] * UA[j] + A[6 + i] * UA[6 + j] + A[12 + i] * UA[12 + j];
    double T1[9], T2[9], jh[9];
    mat3_mul(RiTukhat, P, T1);
    for (int i = 0; i < 9; ++i) T1[i] = combo1[i] - T1[i];
    mat3_mul(T1, RiTukhat, T2);
    hat3(jjt, jh);
    const double c1 = 2.0 / NN, c2 = 2.0 / NN / NN;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        Hd[6 * i + j] += c1 * T2[3 * i + j] - c2 * w[i] * w[j] - 0.5 * jh[3 * i + j];
        const double hrt = c1 * (1.0 - n / NN) * w[i] * uk[j];
        Hd[6 * i + 3 + j] += hrt;
        Hd[6 * (3 + j) + i] += hrt;
        Hd[6 * (3 + i) + 3 + j] += c1 * (n - n * n / NN) * uk[i] * uk[j];
      }
    if constexpr (kDet) {
      for (int i = 0; i < 36; ++i) H[36 * s + i] = Hd[i];
      for (int j = 0; j < 6; ++j) g[6 * s + j] = jjt[j];
    } else {
      const int row = row_of_pose(bv, pose);
      if (row < 0) return;
      double* Hb = H + (bv.row_start[row] + (row - bv.first[row])) * 36;
      for (int i = 0; i < 36; ++i) atomic_add_f64(Hb + i, Hd[i]);
      for (int j = 0; j < 6; ++j) atomic_add_f64(g + 6 * (int64_t)row + j, jjt[j]);
    }
  }
};

// slot pair p (i < j) of the big voxels: its voxel lo and its two slots si < sj
LVBA_BHD void pair_slots(const View& bv, int64_t p, int64_t& lo, int64_t& si, int64_t& sj) {
  lo = 0;
  int64_t hi = bv.n_vox;
  while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if (bv.pair_ptr[mid] <= p) lo = mid; else hi = mid; }
  const int64_t t = p - bv.pair_ptr[lo];                          // strict lower-triangular index: j > i, t = j (j - 1) / 2 + i
  int64_t j = (int64_t)((sqrt(8.0 * (double)t + 1.0) + 1.0) * 0.5);
  while (j * (j - 1) / 2 > t) --j;
  while ((j + 1) * j / 2 <= t) ++j;
  const int64_t i = t - j * (j - 1) / 2;
  si = bv.vox_ptr[lo] + i; sj = bv.vox_ptr[lo] + j;
}

// kDet = false: the block goes into H by atomics; true: H = the pairs' records [n_pairs][36] (see SlotsF)
template <bool kDet>
struct PairsPass {             // one item per slot pair (i < j) of the big voxels
  View bv; const double* params; const double* feat; double* H;
  LVBA_BHD void operator()(int64_t p) const {
    int64_t lo, si, sj;
    pair_slots(bv, p, lo, si, sj);
    const double* q = params + kParams * lo;
    const double* uk = q; const double* um = q + 3;
    const double NN = q[15];
    const double* fi = feat + kFeat * si;
    const double* fj = feat + kFeat * sj;
    double UA[18], Hb[36];
    for (int a = 0; a < 3; ++a)
      for (int c = 0; c < 6; ++c) UA[6 * a + c] = um[3 * a] * fj[c] + um[3 * a + 1] * fj[6 + c] + um[3 * a + 2] * fj[12 + c];
    for (int r = 0; r < 6; ++r)
      for (int c = 0; c < 6; ++c) Hb[6 * r + c] = fi[r] * UA[c] + fi[6 + r] * UA[6 + c] + fi[12 + r] * UA[12 + c];
    const double k = -2.0 / NN / NN, ni = fi[21], nj = fj[21];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {                                                                   // :159-163
        Hb[6 * r + c] += k * fi[18 + r] * fj[18 + c];
        Hb[6 * r + 3 + c] += k * nj * fi[18 + r] * uk[c];
        Hb[6 * (3 + r) + c] += k * ni * uk[r] * fj[18 + c];
        Hb[6 * (3 + r) + 3 + c] += k * ni * nj * uk[r] * uk[c];
      }
    if constexpr (kDet) {
      for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) H[36 * p + 6 * c + r] = Hb[6 * r + c];
    } else {
      const int pi = row_of_pose(bv, bv.pose_idx[si]), pj = row_of_pose(bv, bv.pose_idx[sj]);   // ascending inside a voxel: pi < pj
      if (pi < 0 || pj < 0) return;
      double* B = H + (bv.row_start[pj] + (pi - bv.first[pj])) * 36;  // lower block (pj, pi) = Hb^T   (:171-173)
      for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) atomic_add_f64(B + 6 * c + r, Hb[6 * r + c]);
    }
  }
};

using SlotsF = SlotsPass<false>;
using PairsF = PairsPass<false>;
using SlotsDetF = SlotsPass<true>;
using PairsDetF = PairsPass<true>;

// Destinations of the deterministic records of SlotsDetF (the slot's diagonal H block and gradient row) and PairsDetF
// (the lower H block of the pair), in the units of tiles::FixedSum
struct SlotDstF {
  View bv; int64_t* dst_H; int64_t* dst_g;
  LVBA_BHD void operator()(int64_t s) const {
    const int row = row_of_pose(bv, bv.pose_idx[s]);
    dst_H[s] = row < 0 ? bv.nblocks : bv.row_start[row] + (row - bv.first[row]);
    dst_g[s] = row < 0 ? bv.W : row;
  }
};
struct PairDstF {
  View bv; int64_t* dst_H;
  LVBA_BHD void operator()(int64_t p) const {
    int64_t lo, si, sj;
    pair_slots(bv, p, lo, si, sj);
    const int pi = row_of_pose(bv, bv.pose_idx[si]), pj = row_of_pose(bv, bv.pose_idx[sj]);
    dst_H[p] = (pi < 0 || pj < 0) ? bv.nblocks : bv.row_start[pj] + (pi - bv.first[pj]);
  }
};

}  // namespace big
}  // namespace lvba
