// visual.cuh — hot path B kernels: per-track reprojection / point-to-plane residuals and analytic
// Jacobians, Schur elimination of the 3x3 landmark blocks straight into the block-envelope reduced
// camera system, back-substitution and the model-cost evaluation.
//
// Restates (analytic Jacobians instead of ceres::Jet auto-diff; block-sparse instead of DENSE_SCHUR):
//   ReprojErrorWhitenedDistorted::operator()   reference include/utils.hpp:61-111
//   PointPlaneErrorWhitened::operator()        reference include/utils.hpp:133-139
//   problem structure of optimizeCameraPoses   reference src/lvba_system.cpp:1578-1640
//   ceres-solver 2.1.0 (not vendored): Jacobi column scaling, LM diagonal, Schur complement,
//   EigenQuaternionManifold on {w,x,y,z} memory (SURVEY.md Q9-Q11, Appendix A.2/A.3).
//
// Schedule: the observations of the landmarks that have a valid plane are stored CSR, the landmarks in the order of the
// lowest system row of their clique (visual_tiles.h).  The build and the column norms cut them into tiles of consecutive
// landmarks with <= kVisTileSlots observations, one CTA of kVisTileSlots threads each; back-substitution and the cost cut the
// same order into batches of <= kSlots observations, one CTA of kSlots threads each.
//   phase 1  thread = observation: r (2), J_cam (2x6, tangent), J_X (2x3); J_X^T J_X, J_X^T r staged
//   phase 2  thread = landmark   : C = sum J_X^T J_X + plane term + D_p^2, C^-1, g_p, w = C^-1 g_p
//   phase 3  thread = observation: E = J_c^T J_X, Y = E C^-1, diagonal block J_c^T J_c - Y E^T,
//                                  reduced rhs -(g_c - E w), column norms; factors [Y|E] to shared memory
//   phase 4  every distinct S block, diagonal block and camera row of the tile is summed on chip and written with one
//            RED.ADD.F64 per element.  A destination table built once per structure lists the tile's camera-pair
//            contributions grouped by S block and its observations grouped by row.  Off-diagonal blocks: four lanes per
//            block sum S(hi,lo)[a][b] -= sum_m Y_hi[a][m] E_lo[b][m] over the block's pairs in registers.  Diagonal blocks,
//            rhs, column norms and gradient: staged in shared memory and summed per row.
//            Sorted landmarks share cameras: at config C a 256-slot tile holds 3.9 pair contributions per distinct block
//            and 12 observations per row, and the element REDs per build fall from 79 M (one per pair and observation) to
//            15 M.
// The Jacobian is never materialised in HBM; back-substitution recomputes it.
#pragma once
#include "common.cuh"
#include "envelope.cuh"
#include "lidar.cuh"   // kSlots, kStageStride, reduce kernels
#include "visual_intr.h"
#include "visual_math.h"   // VisualView, obs_eval, plane_eval, sym3_inverse
#include "visual_tiles.h"

namespace lvba {

using tiles::kVisTileSlots;
using tiles::kMaxTrkPerTile;
using tiles::kMaxTrkPerBatch;
constexpr int kVFStride = 37;      // Y(18) E(18) + pad

// ------------------------------------------------------------------------------------------------
// phase 1+2 shared by build and back-substitution.  Leaves per-landmark params in sT:
//   [0..5] Cinv  [6..8] g_p  [9..11] w = Cinv g_p ; returns this thread's observation in `o` (scaled)
// The CTA (kThreads threads) takes the landmarks t0 .. t1 (<= kThreads observations, <= 256 landmarks).  With `env`, the
// envelope row_start / first of the observation's row are loaded beside its camera state (rs, fr; untouched when row < 0).
// kLoss: the robust losses of vv; cost_part is then sum rho and the residuals (and, with kNeedJac, the Jacobians) are the
// corrected ones, before the Jacobi scaling.  The plain instantiations (kLoss = false) never read the loss fields.
template <int kThreads, bool kNeedJac, bool kLoss = false>
LVBA_DEV void visual_front(const VisualView& vv, const VisualState& st, const VisualLM& lm, int t0, int t1,
                           double* stage, double* sT, ObsEval& o, int& row, int& ltrk, double* Xown,
                           double& cost_part, const EnvView* env = nullptr, long long* rs = nullptr, int* fr = nullptr) {
  const int tid = threadIdx.x;
  const int nt = t1 - t0;
  const int s0 = vv.trk_ptr[t0], ns = vv.trk_ptr[t1] - s0;
  __shared__ unsigned char sTrkOf[kThreads];
  if (tid < nt) {
    const int lo = vv.trk_ptr[t0 + tid] - s0, hi = vv.trk_ptr[t0 + tid + 1] - s0;
    for (int q = lo; q < hi; ++q) sTrkOf[q] = (unsigned char)tid;
  }
  __syncthreads();
  cost_part = 0.0;
  row = -1; ltrk = 0;
  if (tid < ns) {
    ltrk = sTrkOf[tid];
    const int tr = vv.trk_id[t0 + ltrk];
    const int cam = vv.obs_cam[s0 + tid];
    row = vv.obs_row[s0 + tid];
    if (env && row >= 0) { *rs = env->row_start[row]; *fr = env->first[row]; }
    Xown[0] = st.X[3 * (long long)tr]; Xown[1] = st.X[3 * (long long)tr + 1]; Xown[2] = st.X[3 * (long long)tr + 2];
    obs_eval<kNeedJac>(vv, st.q + 4 * (long long)cam, st.t + 3 * (long long)cam, Xown, vv.obs_uv[s0 + tid], o);
    if constexpr (kLoss) cost_part = obs_loss<kNeedJac>(vv, o);
    else cost_part = o.r[0] * o.r[0] + o.r[1] * o.r[1];
    if (kNeedJac) {
      const double* sp = lm.s_pt + 3 * (long long)(t0 + ltrk);
#pragma unroll
      for (int rho = 0; rho < 2; ++rho)
#pragma unroll
        for (int m = 0; m < 3; ++m) o.JX[3 * rho + m] *= sp[m];
      if (row >= 0) {
        const double* sc = lm.s_cam + 6 * (long long)row;
#pragma unroll
        for (int rho = 0; rho < 2; ++rho)
#pragma unroll
          for (int a = 0; a < 6; ++a) o.Jc[6 * rho + a] *= sc[a];
      } else {
#pragma unroll
        for (int a = 0; a < 12; ++a) o.Jc[a] = 0.0;     // constant / unused camera: no columns
      }
      double* sg = stage + tid * kStageStride;
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
  }
  __syncthreads();
  if (tid < nt) {
    const int lo = vv.trk_ptr[t0 + tid] - s0, hi = vv.trk_ptr[t0 + tid + 1] - s0;
    const int tr = vv.trk_id[t0 + tid];
    const double Xp[3] = {st.X[3 * (long long)tr], st.X[3 * (long long)tr + 1], st.X[3 * (long long)tr + 2]};
    double rp, Jpl[3];
    plane_eval(vv, vv.plane + 4 * (long long)(t0 + tid), Xp, rp, Jpl);
    if constexpr (kLoss) cost_part += plane_loss(vv, rp, Jpl);
    else cost_part += rp * rp;
    if (kNeedJac) {
      const double* sp = lm.s_pt + 3 * (long long)(t0 + tid);
      Jpl[0] *= sp[0]; Jpl[1] *= sp[1]; Jpl[2] *= sp[2];
      double acc[9];
#pragma unroll
      for (int q = 0; q < 9; ++q) acc[q] = 0.0;
      for (int s = lo; s < hi; ++s)
#pragma unroll
        for (int q = 0; q < 9; ++q) acc[q] += stage[s * kStageStride + q];
      acc[0] += Jpl[0] * Jpl[0]; acc[1] += Jpl[0] * Jpl[1]; acc[2] += Jpl[0] * Jpl[2];
      acc[3] += Jpl[1] * Jpl[1]; acc[4] += Jpl[1] * Jpl[2]; acc[5] += Jpl[2] * Jpl[2];
      acc[6] += Jpl[0] * rp; acc[7] += Jpl[1] * rp; acc[8] += Jpl[2] * rp;
      // LM diagonal of the point columns: clamp(||J~[:,j]||^2)/radius   (Ceres LevenbergMarquardtStrategy)
      const double ir = 1.0 / lm.radius;
      acc[0] += fmin(fmax(acc[0], lm.min_diag), lm.max_diag) * ir;
      acc[3] += fmin(fmax(acc[3], lm.min_diag), lm.max_diag) * ir;
      acc[5] += fmin(fmax(acc[5], lm.min_diag), lm.max_diag) * ir;
      double* p = sT + tid * kTrkParams;
      sym3_inverse(acc, p);
      p[6] = acc[6]; p[7] = acc[7]; p[8] = acc[8];
      p[9] = p[0] * acc[6] + p[1] * acc[7] + p[2] * acc[8];
      p[10] = p[1] * acc[6] + p[3] * acc[7] + p[4] * acc[8];
      p[11] = p[2] * acc[6] + p[4] * acc[7] + p[5] * acc[8];
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// 1/2 sum r^2 partial per batch (candidate evaluation)
__global__ void __launch_bounds__(kSlots)
visual_cost_kernel(VisualView vv, VisualState st, double* __restrict__ batch_cost) {
  __shared__ double red[32];
  __shared__ double dummyT[1];
  ObsEval o;
  int row, ltrk;
  double Xown[3], cp;
  VisualLM lm{1.0, 0.0, 0.0, nullptr, nullptr};
  visual_front<kSlots, false>(vv, st, lm, vv.batch_trk[blockIdx.x], vv.batch_trk[blockIdx.x + 1], nullptr, dummyT, o, row, ltrk, Xown, cp);
  const double tot = block_sum<kSlots>(cp, red);
  if (threadIdx.x == 0) batch_cost[blockIdx.x] = 0.5 * tot;
}
// 1/2 sum rho partial per batch with the robust losses of vv.  A kernel of its own rather than an instantiation of the one above:
// that keeps the plain kernel's static shared memory, and with it its code, as it was.
__global__ void __launch_bounds__(kSlots)
visual_cost_loss_kernel(VisualView vv, VisualState st, double* __restrict__ batch_cost) {
  __shared__ double red[32];
  __shared__ double dummyT[1];
  ObsEval o;
  int row, ltrk;
  double Xown[3], cp;
  VisualLM lm{1.0, 0.0, 0.0, nullptr, nullptr};
  visual_front<kSlots, false, true>(vv, st, lm, vv.batch_trk[blockIdx.x], vv.batch_trk[blockIdx.x + 1], nullptr, dummyT, o, row, ltrk, Xown, cp);
  const double tot = block_sum<kSlots>(cp, red);
  if (threadIdx.x == 0) batch_cost[blockIdx.x] = 0.5 * tot;
}

// ------------------------------------------------------------------------------------------------
// unscaled squared column norms (Jacobi scaling, computed when the scale is reset).  One CTA per build tile: the camera
// columns are summed per row of the tile (row runs of the destination table) before one RED per element.  kDet = true
// (deterministic mode): cam_colsq holds records of 6 doubles, and row run r of the tiles stores its sum into record r with a
// plain store (summed per row by tiles::GatherF in record order).  kLoss: the norms of the corrected Jacobian.
template <bool kDet, bool kLoss = false>
__global__ void __launch_bounds__(kVisTileSlots)
visual_colnorm_kernel(VisualView vv, VisualState st, double* __restrict__ cam_colsq, double* __restrict__ pt_colsq) {
  constexpr int NS = kVisTileSlots, kC = 9;              // per observation: 3 point columns, 6 camera columns
  const int b = blockIdx.x, tid = threadIdx.x;
  const int t0 = vv.tile_trk[b], t1 = vv.tile_trk[b + 1], nt = t1 - t0;
  const int s0 = vv.trk_ptr[t0], ns = vv.trk_ptr[t1] - s0;
  const int64_t d0 = vv.tile_drun[b];
  const int nd = (int)(vv.tile_drun[b + 1] - d0);
  const int64_t q0 = vv.drun_ptr[d0];
  const int nq = (int)(vv.drun_ptr[d0 + nd] - q0);
  __shared__ double stage[NS * kC];
  __shared__ unsigned short sDSlot[NS], sDRun[NS + 1];
  if (tid < ns) {
    // locate landmark by scanning is avoided: recompute from trk_ptr with a small search
    int lo = 0, hi = nt;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (vv.trk_ptr[t0 + mid] - s0 <= tid) lo = mid; else hi = mid; }
    const int tr = vv.trk_id[t0 + lo];
    const int cam = vv.obs_cam[s0 + tid];
    const double X[3] = {st.X[3 * (long long)tr], st.X[3 * (long long)tr + 1], st.X[3 * (long long)tr + 2]};
    ObsEval o;
    obs_eval<true>(vv, st.q + 4 * (long long)cam, st.t + 3 * (long long)cam, X, vv.obs_uv[s0 + tid], o);
    if constexpr (kLoss) obs_loss<true>(vv, o);
    double* sg = stage + tid * kC;
    sg[0] = o.JX[0] * o.JX[0] + o.JX[3] * o.JX[3];
    sg[1] = o.JX[1] * o.JX[1] + o.JX[4] * o.JX[4];
    sg[2] = o.JX[2] * o.JX[2] + o.JX[5] * o.JX[5];
#pragma unroll
    for (int a = 0; a < 6; ++a) sg[3 + a] = o.Jc[a] * o.Jc[a] + o.Jc[6 + a] * o.Jc[6 + a];
  }
  if (tid < nq) sDSlot[tid] = (unsigned short)vv.dslot[q0 + tid];
  for (int r = tid; r <= nd; r += NS) sDRun[r] = (unsigned short)(vv.drun_ptr[d0 + r] - q0);
  __syncthreads();
  if (tid < nt) {
    const int lo = vv.trk_ptr[t0 + tid] - s0, hi = vv.trk_ptr[t0 + tid + 1] - s0;
    const int tr = vv.trk_id[t0 + tid];
    const double X[3] = {st.X[3 * (long long)tr], st.X[3 * (long long)tr + 1], st.X[3 * (long long)tr + 2]};
    double rp, J[3];
    plane_eval(vv, vv.plane + 4 * (long long)(t0 + tid), X, rp, J);
    if constexpr (kLoss) plane_loss(vv, rp, J);
    double a0 = J[0] * J[0], a1 = J[1] * J[1], a2 = J[2] * J[2];
    for (int s = lo; s < hi; ++s) { a0 += stage[s * kC]; a1 += stage[s * kC + 1]; a2 += stage[s * kC + 2]; }
    double* o = pt_colsq + 3 * (long long)(t0 + tid);
    o[0] = a0; o[1] = a1; o[2] = a2;
  }
  for (int e = tid; e < nd * 6; e += NS) {
    const int r = e / 6, a = e - r * 6;
    const int qa = sDRun[r], qb = sDRun[r + 1];
    double v = 0.0;
    for (int q = qa; q < qb; ++q) v += stage[sDSlot[q] * kC + 3 + a];
    if constexpr (kDet) cam_colsq[(d0 + r) * 6 + a] = v;
    else atomicAdd(cam_colsq + 6 * (long long)vv.obs_row[s0 + sDSlot[qa]] + a, v);
  }
}

// scale = 1 / (1 + sqrt(colsq))  (Ceres jacobi_scaling) ; or 1 when disabled
__global__ void visual_scale_kernel(long long n, const double* __restrict__ colsq, int enabled, double* __restrict__ scale) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) scale[i] = enabled ? 1.0 / (1.0 + sqrt(colsq[i])) : 1.0;
}

// ------------------------------------------------------------------------------------------------
// linearise + Schur-eliminate: S (envelope, lower), rhs, camera column norms, camera gradient.  One CTA per tile.
// kDet = false: every run's sum goes into S, rhs, cam_colsq and cam_grad by RED.  kDet = true (deterministic mode): S and rhs
// are the records of tiles::FixedSum and every run stores its sum into its own record: the pair runs' blocks at S[r], the row
// runs' diagonal blocks at S[n_pair_runs + r] and their rhs | column-norm | gradient rows at rhs[18 r]; cam_colsq and cam_grad
// are not used.  tiles::GatherF adds the records up in a fixed order.  kLoss: from the corrected residuals and Jacobians
// (visual_front), through the same sums.
template <bool kDet, bool kLoss = false>
__global__ void __launch_bounds__(kVisTileSlots, 1)
visual_build_kernel(VisualView vv, EnvView env, VisualState st, VisualLM lm, double* __restrict__ S,
                    double* __restrict__ rhs, double* __restrict__ cam_colsq, double* __restrict__ cam_grad,
                    double* __restrict__ batch_cost, double* __restrict__ batch_gmax) {
  constexpr int NS = kVisTileSlots;
  extern __shared__ double sm[];
  double* stage = sm;                                    // [NS][kStageStride]
  double* sF = stage + NS * kStageStride;                // [NS][kVFStride]   Y | E
  double* sG = sF + NS * kVFStride;                      // [NS][18]  rhs | colsq | grad
  double* sT = sG + NS * 18;                             // [kMaxTrkPerTile][kTrkParams]
  double* red = sT + kMaxTrkPerTile * kTrkParams;        // [32]
  long long* sDiag = reinterpret_cast<long long*>(red + 32);     // [NS]
  long long* sRowRS = sDiag + NS;                                // [NS] envelope row_start of the camera row
  int* sRow = reinterpret_cast<int*>(sRowRS + NS);               // [NS]
  int* sRowFirst = sRow + NS;                                    // [NS]
  unsigned short* sDSlot = reinterpret_cast<unsigned short*>(sRowFirst + NS);   // [NS] the tile's observations grouped by row
  unsigned short* sDRun = sDSlot + NS;                           // [NS + 1] row run r = sDSlot[sDRun[r] .. sDRun[r + 1])

  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int t0 = vv.tile_trk[b], t1 = vv.tile_trk[b + 1], nt = t1 - t0;
  const int ns = vv.trk_ptr[t1] - vv.trk_ptr[t0];
  // With one CTA per SM no other CTA hides a dependent global load, so every load that does not depend on phases 1-3 is issued
  // here, into registers, where it overlaps the loads of phase 1: the tile's row runs and the first pair run of every lane of
  // phase 4b.  The envelope rows of the observations come with the camera state in visual_front.
  const int64_t d0 = vv.tile_drun[b];
  const int nd = (int)(vv.tile_drun[b + 1] - d0);
  const int64_t q0 = vv.drun_ptr[d0];
  const bool has_dslot = tid < vv.drun_ptr[d0 + nd] - q0;
  const unsigned dslot = has_dslot ? vv.dslot[q0 + tid] : 0u;
  const int64_t drun = tid <= nd ? vv.drun_ptr[d0 + tid] : 0;
  const int64_t r0 = vv.tile_prun[b], nr = vv.tile_prun[b + 1] - r0;
  const int pq = lane >> 2, k = lane & 3;
  int64_t qa = 0, qb = 0;                                // pair run of this lane in the current round of phase 4b
  unsigned code = 0;
  if ((int64_t)warp * 8 + pq < nr) { qa = vv.prun_ptr[r0 + warp * 8 + pq]; qb = vv.prun_ptr[r0 + warp * 8 + pq + 1]; code = vv.pairs[qa]; }
  ObsEval o;
  int row, ltrk;
  long long rs = 0;
  int fr = 0;
  double Xown[3], cp;
  visual_front<NS, true, kLoss>(vv, st, lm, t0, t1, stage, sT, o, row, ltrk, Xown, cp, &env, &rs, &fr);
  // gradient max-norm (unscaled) of the point blocks
  double gm = 0.0;
  if (tid < nt) {
    const double* p = sT + tid * kTrkParams;
    const double* sp = lm.s_pt + 3 * (long long)(t0 + tid);
    gm = fmax(fabs(p[6] / sp[0]), fmax(fabs(p[7] / sp[1]), fabs(p[8] / sp[2])));
  }
  {
    const double tot = block_sum<NS>(cp, red);
    if (tid == 0) batch_cost[b] = 0.5 * tot;
    // max via the same scratch
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) gm = fmax(gm, __shfl_xor_sync(0xffffffffu, gm, off));
    if (lane == 0) red[warp] = gm;
    __syncthreads();
    if (tid == 0) {
      double m = 0.0;
      for (int w = 0; w < NS / 32; ++w) m = fmax(m, red[w]);
      batch_gmax[b] = m;
    }
    __syncthreads();
  }

  // ---- phase 3
  if (tid < ns) {
    sRow[tid] = row;
    double* sf = sF + tid * kVFStride;
    double* sg = sG + tid * 18;
    double* sd = stage + tid * kStageStride;
    if (row >= 0) {
      const double* p = sT + ltrk * kTrkParams;
      const double Ci[9] = {p[0], p[1], p[2], p[1], p[3], p[4], p[2], p[4], p[5]};
      double E[18], Y[18];
#pragma unroll
      for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int m = 0; m < 3; ++m) E[3 * a + m] = o.Jc[a] * o.JX[m] + o.Jc[6 + a] * o.JX[3 + m];
#pragma unroll
      for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int m = 0; m < 3; ++m) Y[3 * a + m] = E[3 * a] * Ci[m] + E[3 * a + 1] * Ci[3 + m] + E[3 * a + 2] * Ci[6 + m];
#pragma unroll
      for (int a = 0; a < 6; ++a) {
        const double gc = o.Jc[a] * o.r[0] + o.Jc[6 + a] * o.r[1];
        sg[a] = -(gc - (E[3 * a] * p[9] + E[3 * a + 1] * p[10] + E[3 * a + 2] * p[11]));
        sg[6 + a] = o.Jc[a] * o.Jc[a] + o.Jc[6 + a] * o.Jc[6 + a];
        sg[12 + a] = gc;
#pragma unroll
        for (int c = 0; c < 6; ++c)
          sd[6 * a + c] = o.Jc[a] * o.Jc[c] + o.Jc[6 + a] * o.Jc[6 + c]
                        - (Y[3 * a] * E[3 * c] + Y[3 * a + 1] * E[3 * c + 1] + Y[3 * a + 2] * E[3 * c + 2]);
      }
#pragma unroll
      for (int q = 0; q < 18; ++q) { sf[q] = Y[q]; sf[18 + q] = E[q]; }
      sRowRS[tid] = rs; sRowFirst[tid] = fr;
      sDiag[tid] = (rs + (row - fr)) * 36;
    }
  }
  if (has_dslot) sDSlot[tid] = (unsigned short)dslot;
  if (tid <= nd) sDRun[tid] = (unsigned short)(drun - q0);
  if (tid == 0 && nd == NS) sDRun[NS] = (unsigned short)(vv.drun_ptr[d0 + NS] - q0);
  __syncthreads();
  // ---- phase 4a: diagonal blocks, rhs, column norms and gradient, summed per row of the tile (nd runs) and written with one
  //      RED per element
  for (int e = tid; e < nd * 36; e += NS) {
    const int r = e / 36, el = e - r * 36;
    const int qa = sDRun[r], qb = sDRun[r + 1];
    double v = 0.0;
    for (int q = qa; q < qb; ++q) v += stage[sDSlot[q] * kStageStride + el];
    if constexpr (kDet) S[(vv.tile_prun[vv.n_tiles] + d0 + r) * 36 + el] = v;
    else atomicAdd(S + sDiag[sDSlot[qa]] + el, v);
  }
  for (int e = tid; e < nd * 18; e += NS) {
    const int r = e / 18, el = e - r * 18;
    const int qa = sDRun[r], qb = sDRun[r + 1];
    double v = 0.0;
    for (int q = qa; q < qb; ++q) v += sG[sDSlot[q] * 18 + el];
    if constexpr (kDet) {
      rhs[(d0 + r) * 18 + el] = v;
    } else {
      const int which = el / 6, a = el - which * 6;
      double* dst = (which == 0) ? rhs : (which == 1) ? cam_colsq : cam_grad;
      atomicAdd(dst + 6 * (long long)sRow[sDSlot[qa]] + a, v);
    }
  }
  // ---- phase 4b: off-diagonal blocks.  The tile's camera-pair contributions come grouped by destination block (runs); every
  //      warp takes 8 runs at a time, sums each block in registers over the pairs of its run and writes it with 9 REDs per lane.
  //      Lane (pq, k) = (lane >> 2, lane & 3) owns the elements 4 m + k, m = 0..8, of run pq (the mapping of
  //      lidar_build_kernel's phase 4b): one aligned 32-byte sector per run and RED instruction.  The next round's run bounds are
  //      loaded at the start of a round, its first code after the round's sums.
  const bool upper = k >= 2;
  const int col0 = k, col1 = upper ? k - 2 : 4 + k, col2 = 2 + k;
  for (int64_t c = (int64_t)warp * 8; c < nr; c += (NS / 32) * 8) {
    const int64_t cn = c + (NS / 32) * 8;
    int64_t qa_next = 0, qb_next = 0;
    if (cn + pq < nr) { qa_next = vv.prun_ptr[r0 + cn + pq]; qb_next = vv.prun_ptr[r0 + cn + pq + 1]; }
    if (c + pq < nr) {
    double* dst;
    if constexpr (kDet) dst = S + (r0 + c + pq) * 36 + k;
    else dst = S + (sRowRS[code & 0xffff] + (sRow[code >> 16] - sRowFirst[code & 0xffff])) * 36 + k;
    double acc[9];
#pragma unroll
    for (int m = 0; m < 9; ++m) acc[m] = 0.0;
    for (int64_t q = qa; q < qb; ++q) {
      const unsigned code_next = q + 1 < qb ? vv.pairs[q + 1] : 0u;
      const double* y = sF + (code & 0xffff) * kVFStride;       // Y_hi, row a at 3 a
      const double* ee = sF + (code >> 16) * kVFStride + 18;    // E_lo, row bq at 3 bq
      double ce[3][3], ry[6][3];
#pragma unroll
      for (int t = 0; t < 3; ++t) { ce[0][t] = ee[3 * col0 + t]; ce[1][t] = ee[3 * col1 + t]; ce[2][t] = ee[3 * col2 + t]; }
#pragma unroll
      for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int t = 0; t < 3; ++t) ry[a][t] = y[3 * a + t];
#pragma unroll
      for (int m = 0; m < 9; ++m) {
        const int j2 = 2 * (m / 3), ph = m % 3;
        double r0_, r1_, r2_;
        if (ph == 0) { r0_ = ry[j2][0]; r1_ = ry[j2][1]; r2_ = ry[j2][2]; }
        else if (ph == 2) { r0_ = ry[j2 + 1][0]; r1_ = ry[j2 + 1][1]; r2_ = ry[j2 + 1][2]; }
        else { r0_ = upper ? ry[j2 + 1][0] : ry[j2][0]; r1_ = upper ? ry[j2 + 1][1] : ry[j2][1]; r2_ = upper ? ry[j2 + 1][2] : ry[j2][2]; }
        acc[m] -= r0_ * ce[ph][0] + r1_ * ce[ph][1] + r2_ * ce[ph][2];
      }
      code = code_next;
    }
#pragma unroll
    for (int m = 0; m < 9; ++m) {
      if constexpr (kDet) dst[4 * m] = acc[m];
      else atomicAdd(dst + 4 * m, acc[m]);
    }
    }
    qa = qa_next; qb = qb_next;
    code = cn + pq < nr ? vv.pairs[qa] : 0u;
  }
}

constexpr size_t visual_build_smem_bytes() {
  return sizeof(double) * (kVisTileSlots * (kStageStride + kVFStride + 18) + kMaxTrkPerTile * kTrkParams + 32)
       + sizeof(long long) * 2 * kVisTileSlots + sizeof(int) * 2 * kVisTileSlots + sizeof(unsigned short) * (2 * kVisTileSlots + 1) + 64;
}
// the static sTrkOf of visual_front comes on top
static_assert(visual_build_smem_bytes() + kVisTileSlots <= 227 * 1024, "visual_build_kernel: shared memory above the 227 kB an H100 CTA may hold");

// ------------------------------------------------------------------------------------------------
// back-substitution y_p = -C^-1 (g_p + sum E^T y_c), model cost change, candidate landmarks.  kLoss: the model cost change
// -(J~ y)^T (r~ + 1/2 J~ y) of the corrected residuals and Jacobians.
template <bool kLoss>
__global__ void __launch_bounds__(kSlots)
visual_backsub_kernel(VisualView vv, VisualState st, VisualLM lm, const double* __restrict__ y_cam,
                      double* __restrict__ X_cand, double* __restrict__ pt_step,
                      double* __restrict__ batch_out /* [n_batches][4]: model, step^2, x^2, - */) {
  extern __shared__ double sm[];
  double* stage = sm;                                    // [kSlots][kStageStride]
  double* sT = stage + kSlots * kStageStride;            // [kMaxTrkPerBatch][kTrkParams]
  double* red = sT + kMaxTrkPerBatch * kTrkParams;       // [32]
  const int b = blockIdx.x, tid = threadIdx.x;
  const int t0 = vv.batch_trk[b], t1 = vv.batch_trk[b + 1], nt = t1 - t0;
  const int s0 = vv.trk_ptr[t0], ns = vv.trk_ptr[t1] - s0;
  ObsEval o;
  int row, ltrk;
  double Xown[3], cp;
  visual_front<kSlots, true, kLoss>(vv, st, lm, t0, t1, stage, sT, o, row, ltrk, Xown, cp);
  double yc[6] = {0, 0, 0, 0, 0, 0};
  if (tid < ns) {
    if (row >= 0)
#pragma unroll
      for (int a = 0; a < 6; ++a) yc[a] = y_cam[6 * (long long)row + a];
    // E^T y_c = J_X^T (J_c y_c)
    const double j0 = o.Jc[0] * yc[0] + o.Jc[1] * yc[1] + o.Jc[2] * yc[2] + o.Jc[3] * yc[3] + o.Jc[4] * yc[4] + o.Jc[5] * yc[5];
    const double j1 = o.Jc[6] * yc[0] + o.Jc[7] * yc[1] + o.Jc[8] * yc[2] + o.Jc[9] * yc[3] + o.Jc[10] * yc[4] + o.Jc[11] * yc[5];
    double* sg = stage + tid * kStageStride;
    sg[0] = o.JX[0] * j0 + o.JX[3] * j1;
    sg[1] = o.JX[1] * j0 + o.JX[4] * j1;
    sg[2] = o.JX[2] * j0 + o.JX[5] * j1;
    sg[3] = j0; sg[4] = j1;
  }
  __syncthreads();
  double model = 0.0, step2 = 0.0, x2 = 0.0;
  if (tid < nt) {
    const int lo = vv.trk_ptr[t0 + tid] - s0, hi = vv.trk_ptr[t0 + tid + 1] - s0;
    double a0 = 0, a1 = 0, a2 = 0;
    for (int s = lo; s < hi; ++s) { a0 += stage[s * kStageStride]; a1 += stage[s * kStageStride + 1]; a2 += stage[s * kStageStride + 2]; }
    double* p = sT + tid * kTrkParams;
    const double y0 = -(p[9] + p[0] * a0 + p[1] * a1 + p[2] * a2);
    const double y1 = -(p[10] + p[1] * a0 + p[3] * a1 + p[4] * a2);
    const double y2 = -(p[11] + p[2] * a0 + p[4] * a1 + p[5] * a2);
    p[12] = y0; p[13] = y1; p[14] = y2;
    const int tr = vv.trk_id[t0 + tid];
    const double* sp = lm.s_pt + 3 * (long long)(t0 + tid);
    const double X[3] = {st.X[3 * (long long)tr], st.X[3 * (long long)tr + 1], st.X[3 * (long long)tr + 2]};
    const double d[3] = {sp[0] * y0, sp[1] * y1, sp[2] * y2};
    X_cand[3 * (long long)tr] = X[0] + d[0]; X_cand[3 * (long long)tr + 1] = X[1] + d[1]; X_cand[3 * (long long)tr + 2] = X[2] + d[2];
    if (pt_step) { pt_step[3 * (long long)tr] = d[0]; pt_step[3 * (long long)tr + 1] = d[1]; pt_step[3 * (long long)tr + 2] = d[2]; }
    step2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
    x2 = X[0] * X[0] + X[1] * X[1] + X[2] * X[2];
    // plane residual contribution to the model cost change
    double rp, Jpl[3];
    plane_eval(vv, vv.plane + 4 * (long long)(t0 + tid), X, rp, Jpl);
    if constexpr (kLoss) plane_loss(vv, rp, Jpl);
    const double jy = Jpl[0] * d[0] + Jpl[1] * d[1] + Jpl[2] * d[2];   // J~ y = J (s o y)
    model -= jy * (rp + 0.5 * jy);
  }
  __syncthreads();
  if (tid < ns) {
    const double* p = sT + ltrk * kTrkParams;
    const double* sg = stage + tid * kStageStride;
    const double jy0 = sg[3] + o.JX[0] * p[12] + o.JX[1] * p[13] + o.JX[2] * p[14];
    const double jy1 = sg[4] + o.JX[3] * p[12] + o.JX[4] * p[13] + o.JX[5] * p[14];
    model -= jy0 * (o.r[0] + 0.5 * jy0) + jy1 * (o.r[1] + 0.5 * jy1);
  }
  const double tm = block_sum<kSlots>(model, red);
  const double ts = block_sum<kSlots>(step2, red);
  const double tx = block_sum<kSlots>(x2, red);
  if (tid == 0) { batch_out[4 * b] = tm; batch_out[4 * b + 1] = ts; batch_out[4 * b + 2] = tx; batch_out[4 * b + 3] = 0.0; }
}

constexpr size_t visual_backsub_smem_bytes() {
  return sizeof(double) * (kSlots * kStageStride + kMaxTrkPerBatch * kTrkParams + 32) + 64;
}

// camera candidates: q <- Plus(q, s o y[0:3]) with the Q9 manifold, t <- t + s o y[3:6].
// out[2 rows] partial sums: step^2 and x^2 in the ambient space (Ceres ParameterToleranceReached).
__global__ void visual_cam_update_kernel(int n_rows, const int* __restrict__ cam_of_row, const double* __restrict__ q,
                                         const double* __restrict__ t, const double* __restrict__ y,
                                         const double* __restrict__ s_cam, double* __restrict__ q_cand,
                                         double* __restrict__ t_cand, double* __restrict__ cam_step,
                                         double* __restrict__ out /* [gridDim][2] */) {
  __shared__ double red[32];
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  double step2 = 0.0, x2 = 0.0;
  if (r < n_rows) {
    const int c = cam_of_row[r];
    const double* yy = y + 6 * (long long)r;
    const double* sc = s_cam + 6 * (long long)r;
    const double d[6] = {sc[0] * yy[0], sc[1] * yy[1], sc[2] * yy[2], sc[3] * yy[3], sc[4] * yy[4], sc[5] * yy[5]};
    const double m0 = q[4 * c], m1 = q[4 * c + 1], m2 = q[4 * c + 2], m3 = q[4 * c + 3];
    const double nd = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    double n0 = m0, n1 = m1, n2 = m2, n3 = m3;
    if (nd > 0.0) {
      double sn, cs;
      sincos(nd, &sn, &cs);
      const double k = sn / nd;
      const double s0 = k * d[0], s1 = k * d[1], s2 = k * d[2];
      // (cs; s) (x) (m3; m0,m1,m2)  — Hamilton product, Eigen memory order (Q9)
      n3 = cs * m3 - (s0 * m0 + s1 * m1 + s2 * m2);
      n0 = cs * m0 + m3 * s0 + (s1 * m2 - s2 * m1);
      n1 = cs * m1 + m3 * s1 + (s2 * m0 - s0 * m2);
      n2 = cs * m2 + m3 * s2 + (s0 * m1 - s1 * m0);
    }
    q_cand[4 * c] = n0; q_cand[4 * c + 1] = n1; q_cand[4 * c + 2] = n2; q_cand[4 * c + 3] = n3;
    const double t0 = t[3 * c], t1 = t[3 * c + 1], t2 = t[3 * c + 2];
    t_cand[3 * c] = t0 + d[3]; t_cand[3 * c + 1] = t1 + d[4]; t_cand[3 * c + 2] = t2 + d[5];
    if (cam_step)
#pragma unroll
      for (int a = 0; a < 6; ++a) cam_step[6 * (long long)c + a] = d[a];
    step2 = (n0 - m0) * (n0 - m0) + (n1 - m1) * (n1 - m1) + (n2 - m2) * (n2 - m2) + (n3 - m3) * (n3 - m3)
          + d[3] * d[3] + d[4] * d[4] + d[5] * d[5];
    x2 = m0 * m0 + m1 * m1 + m2 * m2 + m3 * m3 + t0 * t0 + t1 * t1 + t2 * t2;
  }
  const double ts = block_sum<128>(step2, red);
  const double tx = block_sum<128>(x2, red);
  if (threadIdx.x == 0) { out[2 * blockIdx.x] = ts; out[2 * blockIdx.x + 1] = tx; }
}

// The corner of the bordered system of the intrinsics block (visual_intr.h), one CTA.  Bk, Yk: [8][n6], column i the border
// B[:, i] and Yk[:, i] = A^-1 B[:, i], A the damped camera system; y = A^-1 r_c.  For the free entries f (bits of mask):
//   Sigma = C + D_k - B_f^T Y_f,  D_k = clamp(colsq, min_d, max_d) / radius,  r = rhs_k - B_f^T y,
// Cholesky, y_k = Sigma^-1 r, then y <- y - Y_f y_k (the camera step).  dev[0..7] = y_k, dev[8..15] = sk o y_k (zeros in the held
// entries); scal[9] = the unscaled intrinsics gradient max-norm, scal[10] = 1 on a pivot that is not finite and > 0 (y_k = 0),
// else 0.  Every sum runs in a fixed order.
__global__ void __launch_bounds__(256) visual_intr_corner_kernel(int64_t n6, const double* __restrict__ Bk, const double* __restrict__ Yk,
                                                                 double* __restrict__ y, const double* __restrict__ sys,
                                                                 const double* __restrict__ sk, unsigned mask, double min_d,
                                                                 double max_d, double radius, double* __restrict__ dev,
                                                                 double* __restrict__ scal) {
  __shared__ double red[32];
  __shared__ double sBY[36 + 8];        // B_f^T Y_f (upper triangle over the free entries), then B_f^T y
  __shared__ double syk[8];
  int fi[8], k = 0;
  for (int i = 0; i < 8; ++i)
    if ((mask >> i) & 1u) fi[k++] = i;
  const int np = k * (k + 1) / 2;
  for (int p = 0, a = 0, b = 0; p < np + k; ++p) {
    const double* u;
    const double* v;
    if (p < np) { u = Bk + fi[a] * n6; v = Yk + fi[b] * n6; if (++b == k) { ++a; b = a; } }
    else { u = Bk + fi[p - np] * n6; v = y; }
    double s = 0.0;
    for (int64_t m = threadIdx.x; m < n6; m += 256) s += u[m] * v[m];
    const double tot = block_sum<256>(s, red);
    if (threadIdx.x == 0) sBY[p] = tot;
  }
  if (threadIdx.x == 0) {
    double S[64], r[8];
    for (int a = 0; a < k; ++a) {
      for (int b = 0; b < k; ++b) {
        const int lo = a < b ? a : b, hi = a < b ? b : a;
        S[a * k + b] = sys[vintr::kC + vintr::ut(fi[lo], fi[hi])] - sBY[lo * k - lo * (lo - 1) / 2 + (hi - lo)];
      }
      S[a * k + a] += fmin(fmax(sys[vintr::kCol + fi[a]], min_d), max_d) / radius;
      r[a] = sys[vintr::kRhs + fi[a]] - sBY[np + a];
    }
    const bool ok = vintr::corner_solve(k, S, r);
    double gm = 0.0;
    for (int i = 0; i < 8; ++i) syk[i] = 0.0;
    for (int a = 0; a < k; ++a) {
      if (ok) syk[fi[a]] = r[a];
      gm = fmax(gm, fabs(sys[vintr::kGrad + fi[a]] / sk[fi[a]]));
    }
    for (int i = 0; i < 8; ++i) { dev[i] = syk[i]; dev[8 + i] = sk[i] * syk[i]; }
    scal[9] = gm;
    scal[10] = ok ? 0.0 : 1.0;
  }
  __syncthreads();
  for (int64_t m = threadIdx.x; m < n6; m += 256) {
    double v = y[m];
    for (int a = 0; a < k; ++a) v -= Yk[fi[a] * n6 + m] * syk[fi[a]];
    y[m] = v;
  }
}

// dadd = clamp(colsq, min, max) / radius  (camera LM diagonal) ; also camera gradient max-norm (unscaled)
__global__ void visual_cam_diag_kernel(int n6, const double* __restrict__ colsq, const double* __restrict__ grad,
                                       const double* __restrict__ s_cam, double min_d, double max_d, double radius,
                                       double* __restrict__ dadd, double* __restrict__ gmax_out) {
  __shared__ double red[32];
  double gm = 0.0;
  for (int i = threadIdx.x; i < n6; i += blockDim.x) {
    dadd[i] = fmin(fmax(colsq[i], min_d), max_d) / radius;
    gm = fmax(gm, fabs(grad[i] / s_cam[i]));
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) gm = fmax(gm, __shfl_xor_sync(0xffffffffu, gm, off));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = gm;
  __syncthreads();
  if (threadIdx.x == 0) {
    double m = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = fmax(m, red[w]);
    gmax_out[0] = m;
  }
}

// generic strided partial reductions: out[j] = sum_i part[i*stride + j] (j < ncol) ; max variant
__global__ void reduce_cols_kernel(const double* __restrict__ part, int n, int stride, int ncol, double* __restrict__ out) {
  __shared__ double red[32];
  for (int j = 0; j < ncol; ++j) {
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) s += part[(long long)i * stride + j];
    const double tot = block_sum<256>(s, red);
    if (threadIdx.x == 0) out[j] = tot;
  }
}
__global__ void reduce_max_kernel(const double* __restrict__ part, int n, double* __restrict__ out) {
  __shared__ double red[32];
  double m = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) m = fmax(m, part[i]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    double r = 0.0;
    for (int w = 0; w < 8; ++w) r = fmax(r, red[w]);
    out[0] = fmax(out[0], r);
  }
}

// multi-GPU gather of the landmark updates: every rank owns a disjoint set of landmarks
__global__ void visual_delta_kernel(long long Tv, const int* __restrict__ trk_id, const double* __restrict__ X,
                                    const double* __restrict__ X0, double* __restrict__ delta) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= Tv * 3) return;
  const long long k = i / 3, q = i - 3 * k;
  const long long tr = trk_id[k];
  delta[3 * tr + q] = X[3 * tr + q] - X0[3 * tr + q];
}
__global__ void visual_add_kernel(long long n, const double* __restrict__ X0, const double* __restrict__ delta, double* __restrict__ out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) out[i] = X0[i] + delta[i];
}

// ------------------------------------------------------------------------------------------------
// Per-observation reprojection errors (lvba_visual_obs_residuals): one thread per local observation w, tile and big landmarks
// alike.  sq[obs_src[w]] = r0^2 + r1^2 of obs_eval<false>, the term the cost pass sums before any loss, or +inf where the
// camera-frame depth fails z > 1e-8 (obs_eval's residual, and the cost, are 0 there).  The landmark of w: the last k with
// trk_ptr[k] <= w.
__global__ void visual_obs_sq_kernel(VisualView vv, VisualState st, long long nnz, int Tv, const int64_t* __restrict__ obs_src,
                                     double* __restrict__ sq) {
  const long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (w >= nnz) return;
  int lo = 0, hi = Tv;
  while (hi - lo > 1) { const int m = (lo + hi) >> 1; if (vv.trk_ptr[m] <= w) lo = m; else hi = m; }
  const long long tr = vv.trk_id[lo];
  const long long cam = vv.obs_cam[w];
  const double X[3] = {st.X[3 * tr], st.X[3 * tr + 1], st.X[3 * tr + 2]};
  ObsEval o;
  obs_eval<false>(vv, st.q + 4 * cam, st.t + 3 * cam, X, vv.obs_uv[w], o);
  sq[obs_src[w]] = (obs_depth(st.q + 4 * cam, st.t + 3 * cam, X) > 1e-8) ? o.r[0] * o.r[0] + o.r[1] * o.r[1] : (double)INFINITY;
}

}  // namespace lvba
