// lidar.cuh — hot path A kernels: BALM2 voxel plane-factor gradient / Hessian accumulation and the
// residual-only pass.  Restates (in a different, batch-flattened schedule) the arithmetic of
//   VOX_HESS::acc_evaluate2            reference include/BALM/bavoxel.hpp:68-174
//   VOX_HESS::evaluate_only_residual   reference include/BALM/bavoxel.hpp:176-203
//   PointCluster::transform            reference include/BALM/tools.hpp:450-456
//
// Work decomposition (GPU-first, not the reference's 16 std::threads over dense W-slot vectors):
//   * the non-empty (voxel, pose) slots are stored CSR, the voxels in the order of their lowest pose (lidar_tiles.h);
//   * the Hessian build cuts them into *tiles* of consecutive voxels holding <= kTileSlots slots, one CTA of kTileSlots
//     threads per tile; the residual pass cuts the same order into batches of <= kSlots slots, one 128-thread CTA each;
//   * phase 1: one thread per slot — coalesced double2 loads of the SoA cluster record, gathered pose,
//              rigid transform of the cluster, staged in shared memory;
//   * phase 2: one thread per voxel — merge the staged clusters, 3x3 Jacobi eigen-solve;
//   * phase 3: one thread per slot — A_i (3x6), g_i, H_ii and the three 6-vectors
//              f1 = A_i^T u1, f2 = A_i^T u2, b = [v_i x R_i^T u0 ; n_i u0]; the off-diagonal block of any
//              pose pair is the rank-3 product  c1 f1_i f1_j^T + c2 f2_i f2_j^T - 2/N^2 b_i b_j^T
//              (algebraically identical to bavoxel.hpp:159-163, re-associated);
//   * phase 4: every distinct H block and gradient row of the tile is summed on chip and written with one RED.ADD.F64 per
//              element.  A destination table built once per structure (lidar_tiles.h) lists the tile's pose pairs grouped
//              by H block and its slots grouped by pose.  Off-diagonal blocks: four lanes per block, each summing 9 elements
//              (3-FMA products of the factors) over the pairs of the block in registers, one aligned 32-byte sector per RED
//              instruction.  Diagonal blocks and g_i: staged in shared memory and summed per pose.
//              Sorted voxels share pose pairs: at config C a 256-slot tile holds 2.5 pairs per distinct block and 8 slots
//              per pose, and the element REDs per build fall from 246 M (one per pair and slot) to 83 M.  512-slot tiles
//              (4.2 pairs per block, 48 M REDs) measured slower on the H100: one CTA per SM, and 128 registers at 512 threads.
// FP64 throughout: lambda0 ~ 1e-4 m^2 is a difference of O(1e4) m^2 terms (P/N - vbar vbar^T).
#pragma once
#include "common.cuh"
#include "envelope.cuh"
#include "lidar_tiles.h"

namespace lvba {

using tiles::kTileSlots;
using tiles::kMaxVoxPerTile;
using tiles::kSlots;
constexpr int kStageStride = 37;       // visual build: doubles per slot in the staging buffer (36 + 1 pad: odd => no LDS.64 bank conflicts)
constexpr int kLStage = 19;            // LiDAR build: 10 cluster values, then HALF a diagonal block (18 + 1 pad)
constexpr int kFStride = 19;           // 18 factor doubles + 1 pad
constexpr int kVoxParams = 16;

struct LidarView {
  int W;
  const double2* cl;        // [5][nnz_pad] SoA pairs: (Pxx,Pxy) (Pxz,Pyy) (Pyz,Pzz) (vx,vy) (vz,N)
  long long nnz_pad;
  const int* pidx;          // [nnz] pose index per slot
  const int* vox_ptr;       // [V_local+1] slot offsets
  int n_batches;            // residual pass: batches of <= kSlots slots
  const int* batch_vox;     // [n_batches+1] voxel range per batch
  int n_tiles;              // Hessian build: tiles of <= kTileSlots slots (lidar_tiles.h)
  const int* tile_vox;      // [n_tiles+1] voxel range per tile
  const int64_t* tile_prun; // [n_tiles+1] pair runs of every tile
  const int64_t* prun_ptr;  // run r = pairs[prun_ptr[r] .. prun_ptr[r+1]): the pose pairs of one H block
  const unsigned* pairs;    // li | lj << 16, li < lj slots local to the tile
  const int64_t* tile_drun; // [n_tiles+1] pose runs of every tile
  const int64_t* drun_ptr;  // run r = dslot[drun_ptr[r] .. drun_ptr[r+1]): the slots of one pose
  const unsigned* dslot;    // slots local to the tile; a tile's items are dslot[s0 .. s0 + ns) (constant poses: see row_of)
  // constant poses (lvba_lidar_opts::pose_fixed, read by lidar_build_kernel<*, true>): row_of[pose] = its row of the pose
  // system, -1 for a constant pose.  Slots of constant poses have no pose run, so a tile's slot items are then
  // dslot[drun_ptr[tile_drun[b]] .. drun_ptr[tile_drun[b + 1]]).
  const int* row_of;
};

struct SlotData {
  double R[9], t[3], P[6], v[3], n;
};

LVBA_DEV void load_slot(const LidarView& lv, const double* __restrict__ poses, long long slot, int pose, SlotData& s) {
  const double2 c0 = ldg2(lv.cl + 0 * lv.nnz_pad + slot);
  const double2 c1 = ldg2(lv.cl + 1 * lv.nnz_pad + slot);
  const double2 c2 = ldg2(lv.cl + 2 * lv.nnz_pad + slot);
  const double2 c3 = ldg2(lv.cl + 3 * lv.nnz_pad + slot);
  const double2 c4 = ldg2(lv.cl + 4 * lv.nnz_pad + slot);
  const double2* pp = reinterpret_cast<const double2*>(poses + 12 * (long long)pose);
  const double2 p0 = pp[0], p1 = pp[1], p2 = pp[2], p3 = pp[3], p4 = pp[4], p5 = pp[5];
  s.P[0] = c0.x; s.P[1] = c0.y; s.P[2] = c1.x; s.P[3] = c1.y; s.P[4] = c2.x; s.P[5] = c2.y;
  s.v[0] = c3.x; s.v[1] = c3.y; s.v[2] = c4.x; s.n = c4.y;
  s.R[0] = p0.x; s.R[1] = p0.y; s.R[2] = p1.x; s.R[3] = p1.y; s.R[4] = p2.x; s.R[5] = p2.y;
  s.R[6] = p3.x; s.R[7] = p3.y; s.R[8] = p4.x; s.t[0] = p4.y; s.t[1] = p5.x; s.t[2] = p5.y;
}

// PointCluster::transform (tools.hpp:450-456): out[0..5] = P' (xx xy xz yy yz zz), out[6..8] = v', out[9] = N
LVBA_DEV void transform_cluster(const SlotData& s, double* out) {
  const double Pf[9] = {s.P[0], s.P[1], s.P[2], s.P[1], s.P[3], s.P[4], s.P[2], s.P[4], s.P[5]};
  double RP[9], RPRt[9], Rv[3];
  mat3_mul(s.R, Pf, RP);
  mat3_mul_bt(RP, s.R, RPRt);
  mat3_vec(s.R, s.v, Rv);
  const double* t = s.t;
  out[0] = RPRt[0] + 2.0 * Rv[0] * t[0] + s.n * t[0] * t[0];
  out[1] = RPRt[1] + Rv[0] * t[1] + Rv[1] * t[0] + s.n * t[0] * t[1];
  out[2] = RPRt[2] + Rv[0] * t[2] + Rv[2] * t[0] + s.n * t[0] * t[2];
  out[3] = RPRt[4] + 2.0 * Rv[1] * t[1] + s.n * t[1] * t[1];
  out[4] = RPRt[5] + Rv[1] * t[2] + Rv[2] * t[1] + s.n * t[1] * t[2];
  out[5] = RPRt[8] + 2.0 * Rv[2] * t[2] + s.n * t[2] * t[2];
  out[6] = Rv[0] + s.n * t[0];
  out[7] = Rv[1] + s.n * t[1];
  out[8] = Rv[2] + s.n * t[2];
  out[9] = s.n;
}

// merged covariance of one voxel from the staged clusters (bavoxel.hpp:87-98)
LVBA_DEV void voxel_cov(const double* stage, int s_lo, int s_hi, double cov[6], double vbar[3], double& Nsum) {
  double acc[10];
#pragma unroll
  for (int q = 0; q < 10; ++q) acc[q] = 0.0;
  for (int s = s_lo; s < s_hi; ++s) {
    const double* p = stage + s * kLStage;
#pragma unroll
    for (int q = 0; q < 10; ++q) acc[q] += p[q];
  }
  Nsum = acc[9];
  const double inv = 1.0 / Nsum;
  vbar[0] = acc[6] * inv; vbar[1] = acc[7] * inv; vbar[2] = acc[8] * inv;
  cov[0] = acc[0] * inv - vbar[0] * vbar[0];
  cov[1] = acc[1] * inv - vbar[0] * vbar[1];
  cov[2] = acc[2] * inv - vbar[0] * vbar[2];
  cov[3] = acc[3] * inv - vbar[1] * vbar[1];
  cov[4] = acc[4] * inv - vbar[1] * vbar[2];
  cov[5] = acc[5] * inv - vbar[2] * vbar[2];
}

// ------------------------------------------------------------------------------------------------
// residual-only pass: sum_v lambda0 (per-batch partial written to batch_res[blockIdx.x]).
// kPerVoxel = true (lvba_lidar_voxel_residuals): every voxel's lambda0 is stored instead, at out[vox_id[v]] for local voxel v
// (out[v] when vox_id is null: the local order is the handle's), and nothing is summed.
// The four warps of a batch CTA work on their own quarter of the batch's voxels — whose slots are contiguous — without a
// block barrier in between: lane = slot (load, transform, stage), then lane = voxel (merge, smallest eigenvalue).  With one barrier
// between "all slots" and "all voxels" three warps of four would wait for the one that holds the ~18 voxels; this way a warp
// only ever waits for its own loads.
template <bool kPerVoxel>
__global__ void __launch_bounds__(kSlots)
lidar_residual_kernel(LidarView lv, const double* __restrict__ poses, double* __restrict__ batch_res, const int* __restrict__ vox_id) {
  constexpr int kS = 11;                      // 10 doubles per slot + 1 pad (odd stride)
  constexpr int kWarps = kSlots / 32;
  __shared__ double stage[kSlots * kS];
  __shared__ double red[kWarps];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int v0 = lv.batch_vox[b], v1 = lv.batch_vox[b + 1], nv = v1 - v0;
  const int s0 = lv.vox_ptr[v0];
  const int wv0 = v0 + (nv * warp) / kWarps, wv1 = v0 + (nv * (warp + 1)) / kWarps;
  const int lo = lv.vox_ptr[wv0] - s0, hi = lv.vox_ptr[wv1] - s0;
  for (int sl = lo + lane; sl < hi; sl += 32) {
    SlotData s;
    load_slot(lv, poses, s0 + sl, lv.pidx[s0 + sl], s);
    double out[10];
    transform_cluster(s, out);
#pragma unroll
    for (int q = 0; q < 10; ++q) stage[sl * kS + q] = out[q];
  }
  __syncwarp();
  double lam0 = 0.0;
  for (int v = wv0 + lane; v < wv1; v += 32) {
    const int a = lv.vox_ptr[v] - s0, e = lv.vox_ptr[v + 1] - s0;
    double acc[10];
#pragma unroll
    for (int q = 0; q < 10; ++q) acc[q] = 0.0;
    for (int sl = a; sl < e; ++sl)
#pragma unroll
      for (int q = 0; q < 10; ++q) acc[q] += stage[sl * kS + q];
    const double inv = 1.0 / acc[9];
    const double m0 = acc[6] * inv, m1 = acc[7] * inv, m2 = acc[8] * inv;
    const double lam = sym3_smallest_eigenvalue(acc[0] * inv - m0 * m0, acc[1] * inv - m0 * m1, acc[2] * inv - m0 * m2,
                                                acc[3] * inv - m1 * m1, acc[4] * inv - m1 * m2, acc[5] * inv - m2 * m2);
    if constexpr (kPerVoxel) batch_res[vox_id ? vox_id[v] : v] = lam;
    else lam0 += lam;
  }
  if constexpr (kPerVoxel) return;
  lam0 = warp_sum(lam0);
  if (lane == 0) red[warp] = lam0;
  __syncthreads();
  if (tid == 0) {
    double tot = 0.0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) tot += red[w];
    batch_res[b] = tot;
  }
}

// ------------------------------------------------------------------------------------------------
// Hessian + gradient + residual build: one CTA of kTileSlots threads per tile.
// kDet = false: every run's sum goes into H and g by RED.  kDet = true (deterministic mode): H and g are the records of
// tiles::FixedSum (lidar_tiles.h) and every run's sum is stored into its own: the pair runs' blocks at H[r], the pose runs'
// diagonal blocks at H[n_pair_runs + r] and their gradient rows at g[r]; tiles::GatherF adds them up in a fixed order.
// kFixed = true (constant poses): phase 1 addresses the envelope and g through lv.row_of.  A slot of a constant pose still
// enters its voxel's plane and lambda_0; the destination table gives it no pose run and its pairs no pair run, so phases 3-4
// write nothing for it.  sPose then holds the slot's row (-1: constant).
template <bool kDet, bool kFixed>
__global__ void __launch_bounds__(kTileSlots, 512 / kTileSlots)
lidar_build_kernel(LidarView lv, EnvView env, const double* __restrict__ poses, double* __restrict__ H,
                   double* __restrict__ g, double* __restrict__ batch_res) {
  constexpr int S = kTileSlots;
  extern __shared__ double sm[];
  double* stage = sm;                                   // [S][kLStage]
  double* sF = stage + S * kLStage;                     // [S][kFStride]
  double* sG = sF + S * kFStride;                       // [S][6]
  double* sV = sG + S * 6;                              // [kMaxVoxPerTile][kVoxParams]
  double* red = sV + kMaxVoxPerTile * kVoxParams;       // [32]
  long long* sDiag = reinterpret_cast<long long*>(red + 32);   // [S] element offset of the slot's diagonal block
  long long* sRowRS = sDiag + S;                        // [S] envelope row_start of the slot's pose row
  int* sPose = reinterpret_cast<int*>(sRowRS + S);      // [S]
  int* sRowFirst = sPose + S;                           // [S] envelope first[] of the slot's pose row
  unsigned short* sVoxOf = reinterpret_cast<unsigned short*>(sRowFirst + S);   // [S] tile-local voxel of the slot
  unsigned short* sDSlot = sVoxOf + S;                  // [S] the tile's slots grouped by pose
  unsigned short* sDRun = sDSlot + S;                   // [S + 1] pose run r = sDSlot[sDRun[r] .. sDRun[r + 1])

  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int v0 = lv.tile_vox[b], v1 = lv.tile_vox[b + 1], nv = v1 - v0;
  const int s0 = lv.vox_ptr[v0], ns = lv.vox_ptr[v1] - s0;
  const int64_t d0 = lv.tile_drun[b];
  const int nd = (int)(lv.tile_drun[b + 1] - d0);
  const int dbase = kFixed ? (int)lv.drun_ptr[d0] : s0;    // the tile's slot items: dslot[dbase ..)

  // ---- phase 1: load + transform
  SlotData s;
  int pose = 0;
  if (tid < ns) {
    pose = lv.pidx[s0 + tid];
    load_slot(lv, poses, s0 + tid, pose, s);
    double out[10];
    transform_cluster(s, out);
#pragma unroll
    for (int q = 0; q < 10; ++q) stage[tid * kLStage + q] = out[q];
    if constexpr (kFixed) {
      const int row = lv.row_of[pose];
      sPose[tid] = row;
      if (row >= 0) {
        const long long rs = env.row_start[row];
        const int fr = env.first[row];
        sRowRS[tid] = rs; sRowFirst[tid] = fr;
        sDiag[tid] = (rs + (row - fr)) * 36;
      }
    } else {
      sPose[tid] = pose;
      const long long rs = env.row_start[pose];
      const int fr = env.first[pose];
      sRowRS[tid] = rs; sRowFirst[tid] = fr;
      sDiag[tid] = (rs + (pose - fr)) * 36;
      sDSlot[tid] = (unsigned short)lv.dslot[s0 + tid];   // the tile's slot items are dslot[s0 .. s0 + ns), grouped by pose
    }
  }
  if constexpr (kFixed) {                               // the slots with a row, grouped by row
    const int nds = (int)(lv.drun_ptr[d0 + nd] - dbase);
    if (tid < nds) sDSlot[tid] = (unsigned short)lv.dslot[dbase + tid];
  }
  for (int r = tid; r <= nd; r += S) sDRun[r] = (unsigned short)(lv.drun_ptr[d0 + r] - dbase);
  __syncthreads();

  // ---- phase 2: per voxel merge + eigen solve (bavoxel.hpp:97-110)
  double lam0 = 0.0;
  if (tid < nv) {
    const int lo = lv.vox_ptr[v0 + tid] - s0, hi = lv.vox_ptr[v0 + tid + 1] - s0;
    double cov[6], vbar[3], Nsum;
    voxel_cov(stage, lo, hi, cov, vbar, Nsum);
    double lam[3], u[3][3];
    eig3_sym_plane(cov[0], cov[1], cov[2], cov[3], cov[4], cov[5], lam, u);
    lam0 = lam[0];
    double* p = sV + tid * kVoxParams;
#pragma unroll
    for (int k = 0; k < 3; ++k) { p[k] = u[0][k]; p[3 + k] = u[1][k]; p[6 + k] = u[2][k]; p[12 + k] = vbar[k]; }
    p[9] = 2.0 / (lam[0] - lam[1]);       // umumT weights, bavoxel.hpp:110
    p[10] = 2.0 / (lam[0] - lam[2]);
    p[11] = (double)(int)Nsum;            // int NN = sig.N, bavoxel.hpp:101
    for (int q = lo; q < hi; ++q) sVoxOf[q] = (unsigned short)tid;
  }
  const double tot = block_sum<S>(lam0, red);   // contains __syncthreads
  if (tid == 0) batch_res[b] = tot;
  __syncthreads();

  // ---- phase 3: per slot A_i, g_i, H_ii, factors (bavoxel.hpp:112-149)
  double Hb[36];
  if (tid < ns) {
    const double* vp = sV + sVoxOf[tid] * kVoxParams;
    const double uk[3] = {vp[0], vp[1], vp[2]}, u1[3] = {vp[3], vp[4], vp[5]}, u2[3] = {vp[6], vp[7], vp[8]};
    const double c1 = vp[9], c2 = vp[10], NN = vp[11];
    const double iN = 1.0 / NN;
    const double Pf[9] = {s.P[0], s.P[1], s.P[2], s.P[1], s.P[3], s.P[4], s.P[2], s.P[4], s.P[5]};
    double a[3], Pa[3], w[3], tiv[3], Rv[3];
    mat3t_vec(s.R, uk, a);                 // RiTuk
    mat3_vec(Pf, a, Pa);                   // PiRiTuk
    cross3(s.v, a, w);                     // viRiTuk = hat(vi) RiTuk
    tiv[0] = s.t[0] - vp[12]; tiv[1] = s.t[1] - vp[13]; tiv[2] = s.t[2] - vp[14];
    const double sc = dot3(uk, tiv);       // ukTti_v
    const double x[3] = {Pa[0] + sc * s.v[0], Pa[1] + sc * s.v[1], Pa[2] + sc * s.v[2]};   // combo1 = hat(x)
    mat3_vec(s.R, s.v, Rv);
    const double c2v[3] = {Rv[0] + s.n * tiv[0], Rv[1] + s.n * tiv[1], Rv[2] + s.n * tiv[2]};   // combo2
    // Auk (3x6), rows r, cols 0..5
    double M1[9], A0[9], Rc1[9];
    mat3_mul(s.R, Pf, M1);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) M1[3 * i + j] += tiv[i] * s.v[j];
    mat3_mul_hat(M1, a, A0);               // (Ri Pi + ti_v vi^T) hat(RiTuk)
    mat3_mul_hat(s.R, x, Rc1);             // Ri * combo1
    double Auk[18];
    const double c2u = dot3(c2v, uk);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        Auk[6 * i + j] = (A0[3 * i + j] - Rc1[3 * i + j]) * iN;
        Auk[6 * i + 3 + j] = (c2v[i] * uk[j] + ((i == j) ? c2u : 0.0)) * iN;
      }
    }
    double jjt[6], f1[6], f2[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      jjt[j] = Auk[j] * uk[0] + Auk[6 + j] * uk[1] + Auk[12 + j] * uk[2];
      f1[j] = Auk[j] * u1[0] + Auk[6 + j] * u1[1] + Auk[12 + j] * u1[2];
      f2[j] = Auk[j] * u2[0] + Auk[6 + j] * u2[1] + Auk[12 + j] * u2[2];
    }
    // diagonal block
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int j = 0; j < 6; ++j) Hb[6 * i + j] = c1 * f1[i] * f1[j] + c2 * f2[i] * f2[j];
    {
      // (0,0) += 2/NN (combo1 - hat(a) Pi) hat(a) - 2/NN^2 w w^T - 0.5 hat(jjt[0:3])
      double haP[9], D0[9], hx[9], E[9];
      hat_mul_mat3(a, Pf, haP);
      hat3(x, hx);
#pragma unroll
      for (int q = 0; q < 9; ++q) D0[q] = hx[q] - haP[q];
      mat3_mul_hat(D0, a, E);
      double hj[9];
      hat3(jjt, hj);
      const double k2 = 2.0 * iN, k22 = 2.0 * iN * iN;
      const double hrt = 2.0 * iN * (1.0 - s.n * iN);
      const double k33 = 2.0 * iN * (s.n - s.n * s.n * iN);
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          Hb[6 * i + j] += k2 * E[3 * i + j] - k22 * w[i] * w[j] - 0.5 * hj[3 * i + j];
          const double h = hrt * w[i] * uk[j];
          Hb[6 * i + 3 + j] += h;
          Hb[6 * (3 + j) + i] += h;
          Hb[6 * (3 + i) + 3 + j] += k33 * uk[i] * uk[j];
        }
    }
    // stage: gradient, factors (the diagonal block follows in two halves, below)
    double* sg = sG + tid * 6;
    double* sf = sF + tid * kFStride;
    // off-diagonal blocks are  c1 f1 f1^T + c2 f2 f2^T - 2/N^2 b b^T  with c1, c2 < 0 (lambda0 is the smallest
    // eigenvalue): store the factors pre-scaled by sqrt(|c|) so that phase 4 is a plain 3-term dot product
    const double s1 = sqrt(-c1), s2 = sqrt(-c2), s3 = 1.4142135623730951 * iN;
#pragma unroll
    for (int j = 0; j < 6; ++j) { sg[j] = jjt[j]; sf[j] = s1 * f1[j]; sf[6 + j] = s2 * f2[j]; }
    sf[12] = s3 * w[0]; sf[13] = s3 * w[1]; sf[14] = s3 * w[2];
    const double s3n = s3 * s.n;
    sf[15] = s3n * uk[0]; sf[16] = s3n * uk[1]; sf[17] = s3n * uk[2];
  }

  // ---- phase 4a: diagonal blocks and gradient rows, summed per pose of the tile (nd runs) and written with one RED per
  //      element.  The blocks go through the staging buffer in two halves of 18 doubles per slot.
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    __syncthreads();                                      // half 0: phase 2 is done with the clusters; half 1: flush 0 is done
    if (tid < ns) {
      double* st = stage + tid * kLStage;
#pragma unroll
      for (int q = 0; q < 18; ++q) st[q] = Hb[18 * half + q];
    }
    __syncthreads();
    for (int e = tid; e < nd * 18; e += S) {
      const int r = e / 18, el = e - r * 18;
      const int qa = sDRun[r], qb = sDRun[r + 1];
      double v = 0.0;
      for (int q = qa; q < qb; ++q) v += stage[sDSlot[q] * kLStage + el];
      if constexpr (kDet) H[(lv.tile_prun[lv.n_tiles] + d0 + r) * 36 + 18 * half + el] = v;
      else atomicAdd(H + sDiag[sDSlot[qa]] + 18 * half + el, v);
    }
  }
  for (int e = tid; e < nd * 6; e += S) {
    const int r = e / 6, el = e - r * 6;
    const int qa = sDRun[r], qb = sDRun[r + 1];
    double v = 0.0;
    for (int q = qa; q < qb; ++q) v += sG[sDSlot[q] * 6 + el];
    if constexpr (kDet) g[(d0 + r) * 6 + el] = v;
    else atomicAdd(g + 6 * (long long)sPose[sDSlot[qa]] + el, v);
  }

  // ---- phase 4b: off-diagonal blocks.  The tile's pose pairs come grouped by destination block (runs); every warp takes 8
  // runs at a time, sums each block in registers over the pairs of its run and writes it with 9 REDs per lane.
  // Lane (pq, k) = (lane >> 2, lane & 3) owns the elements 4 m + k, m = 0..8, of run pq: every RED instruction of the warp
  // writes one aligned 32-byte sector per run (8 full sectors, as a linear mapping would), and a lane reads the 27 factor values
  // of its 9 elements of a pair from shared memory once.  With el = 4 m + k, row = el / 6 and column = el % 6 depend on the
  // lane only through k:
  //   m % 3 == 0: row 2j,                 column k
  //   m % 3 == 1: row 2j + (k >= 2),      column k < 2 ? 4 + k : k - 2
  //   m % 3 == 2: row 2j + 1,             column 2 + k                      (j = m / 3)
  // so the three columns sit in registers indexed by m % 3 (compile time) and the row of the middle case is a select.
  const int64_t r0 = lv.tile_prun[b], nr = lv.tile_prun[b + 1] - r0;
  const int pq = lane >> 2, k = lane & 3;
  const bool hi = k >= 2;
  const int col0 = k, col1 = hi ? k - 2 : 4 + k, col2 = 2 + k;
  for (int64_t c = (int64_t)warp * 8; c < nr; c += (S / 32) * 8) {
    if (c + pq >= nr) continue;
    const int64_t qa = lv.prun_ptr[r0 + c + pq], qb = lv.prun_ptr[r0 + c + pq + 1];
    unsigned code = lv.pairs[qa];
    // lower-triangle block: row = larger pose (slot lj, ascending order inside a voxel), col = slot li
    double* dst;
    if constexpr (kDet) dst = H + (r0 + c + pq) * 36 + k;
    else dst = H + (sRowRS[code >> 16] + (sPose[code & 0xffff] - sRowFirst[code >> 16])) * 36 + k;
    double acc[9];
#pragma unroll
    for (int m = 0; m < 9; ++m) acc[m] = 0.0;
    for (int64_t q = qa; q < qb; ++q) {
      const unsigned code_next = q + 1 < qb ? lv.pairs[q + 1] : 0u;
      const double* fi = sF + (code & 0xffff) * kFStride;   // column factors
      const double* fj = sF + (code >> 16) * kFStride;      // row factors
      double ci[3][3], rj[6][3];
#pragma unroll
      for (int t = 0; t < 3; ++t) { ci[0][t] = fi[6 * t + col0]; ci[1][t] = fi[6 * t + col1]; ci[2][t] = fi[6 * t + col2]; }
#pragma unroll
      for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int t = 0; t < 3; ++t) rj[a][t] = fj[6 * t + a];
#pragma unroll
      for (int m = 0; m < 9; ++m) {
        const int j2 = 2 * (m / 3), ph = m % 3;
        double x0, x1, x2;
        if (ph == 0) { x0 = rj[j2][0]; x1 = rj[j2][1]; x2 = rj[j2][2]; }
        else if (ph == 2) { x0 = rj[j2 + 1][0]; x1 = rj[j2 + 1][1]; x2 = rj[j2 + 1][2]; }
        else { x0 = hi ? rj[j2 + 1][0] : rj[j2][0]; x1 = hi ? rj[j2 + 1][1] : rj[j2][1]; x2 = hi ? rj[j2 + 1][2] : rj[j2][2]; }
        acc[m] -= ci[ph][0] * x0 + ci[ph][1] * x1 + ci[ph][2] * x2;
      }
      code = code_next;
    }
#pragma unroll
    for (int m = 0; m < 9; ++m) {
      if constexpr (kDet) dst[4 * m] = acc[m];
      else atomicAdd(dst + 4 * m, acc[m]);
    }
  }
}

constexpr size_t lidar_build_smem_bytes() {
  return sizeof(double) * (kTileSlots * (kLStage + kFStride + 6) + kMaxVoxPerTile * kVoxParams + 32)
       + sizeof(long long) * 2 * kTileSlots + sizeof(int) * 2 * kTileSlots + sizeof(unsigned short) * (3 * kTileSlots + 1) + 64;
}
static_assert(lidar_build_smem_bytes() <= 227 * 1024, "lidar_build_kernel: shared memory above the 227 kB an H100 CTA may hold");

// ------------------------------------------------------------------------------------------------
// small LM helpers
// deterministic sum of n partials by one block
__global__ void reduce_partials_kernel(const double* __restrict__ part, int n, double* __restrict__ out) {
  __shared__ double red[32];
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) s += part[i];
  const double tot = block_sum<256>(s, red);
  if (threadIdx.x == 0) out[0] = tot;
}

// trial = poses (+) dx : R <- R Exp(dphi), p <- p + dp   (bavoxel.hpp:722-727)
__global__ void lidar_retract_kernel(int W, const double* __restrict__ poses, const double* __restrict__ dx,
                                     double* __restrict__ trial) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= W) return;
  const double* p = poses + 12 * j;
  const double* d = dx + 6 * j;
  double E[9], R[9], Rn[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) R[q] = p[q];
  so3_exp(d, E);
  mat3_mul(R, E, Rn);
  double* o = trial + 12 * j;
#pragma unroll
  for (int q = 0; q < 9; ++q) o[q] = Rn[q];
  o[9] = p[9] + d[3]; o[10] = p[10] + d[4]; o[11] = p[11] + d[5];
}

// the same with constant poses: dx holds the rows of the free poses (row_of[j] = row of pose j, -1: constant), and a constant
// pose is copied as it is, so that it comes back bit-identical
__global__ void lidar_retract_rows_kernel(int W, const double* __restrict__ poses, const double* __restrict__ dx,
                                          const int* __restrict__ row_of, double* __restrict__ trial) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= W) return;
  const double* p = poses + 12 * j;
  double* o = trial + 12 * j;
  const int r = row_of[j];
  if (r < 0) {
#pragma unroll
    for (int q = 0; q < 12; ++q) o[q] = p[q];
    return;
  }
  const double* d = dx + 6 * r;
  double E[9], R[9], Rn[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) R[q] = p[q];
  so3_exp(d, E);
  mat3_mul(R, E, Rn);
#pragma unroll
  for (int q = 0; q < 9; ++q) o[q] = Rn[q];
  o[9] = p[9] + d[3]; o[10] = p[10] + d[4]; o[11] = p[11] + d[5];
}

// q1 = 0.5 * dx . (u * D * dx - g), D = diag(H)   (bavoxel.hpp:729); also flags non-finite dx
__global__ void lidar_q1_kernel(int n6, const double* __restrict__ dx, const double* __restrict__ diag,
                                const double* __restrict__ g, double u, double* __restrict__ out /* [2]: q1, nonfinite */) {
  __shared__ double red[32];
  double s = 0.0, bad = 0.0;
  for (int i = threadIdx.x; i < n6; i += 256) {
    const double d = dx[i];
    s += d * (u * diag[i] * d - g[i]);
    if (!isfinite(d)) bad = 1.0;
  }
  const double tot = block_sum<256>(s, red);
  const double tb = block_sum<256>(bad, red);
  if (threadIdx.x == 0) { out[0] = 0.5 * tot; out[1] = tb; }
}

// z = -g ; dadd = u * diag
__global__ void lidar_rhs_kernel(int n6, const double* __restrict__ g, const double* __restrict__ diag, double u,
                                 double* __restrict__ z, double* __restrict__ dadd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n6) { z[i] = -g[i]; dadd[i] = u * diag[i]; }
}

}  // namespace lvba
