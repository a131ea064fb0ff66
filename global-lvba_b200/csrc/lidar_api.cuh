// lidar_api.cuh — host side of boundary B1 (include/lvba_b200.h): symbolic set-up, device-resident
// problem handle and the damping_iter LM loop of reference include/BALM/bavoxel.hpp:662-767.
#pragma once
#include <cmath>
#include <unordered_set>

#include "runtime.cuh"   // (pulls comm.cuh in)
#include "balm_rule.h"
#include "exec.cuh"
#include "lidar.cuh"
#include "lidar_outliers.h"
#include "lidar_plan.h"

namespace lvba {

__global__ void lidar_aos_to_soa_kernel(long long nnz, long long nnz_pad, const double* __restrict__ aos,
                                        double2* __restrict__ soa) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= nnz) return;
  const double2* r = reinterpret_cast<const double2*>(aos + 10 * i);   // 80-byte records: 16-byte aligned
#pragma unroll
  for (int q = 0; q < 5; ++q) soa[q * nnz_pad + i] = r[q];
}

// ---- batched window BA (LvbaSystem::runWindowBA, reference src/lvba_system.cpp:232-302): per-window reductions.
// One CTA per window; ranges are contiguous because tiles, batches and poses are ordered by window.
__global__ void lidar_group_sum_kernel(const double* __restrict__ part, const int* __restrict__ rng /*[G+1]*/, double* __restrict__ out, int slot) {
  __shared__ double red[32];
  const int g = blockIdx.x;
  double s = 0.0;
  for (int i = rng[g] + threadIdx.x; i < rng[g + 1]; i += 128) s += part[i];
  const double tot = block_sum<128>(s, red);
  if (threadIdx.x == 0) out[4 * g + slot] = tot;
}
// z = -g ; dadd = u_w * diag with the window's own damping (bavoxel.hpp:692-693 per window)
__global__ void lidar_rhs_grouped_kernel(int n6, const double* __restrict__ g, const double* __restrict__ diag, const double* __restrict__ u_grp,
                                         const int* __restrict__ pose_grp, double* __restrict__ z, double* __restrict__ dadd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n6) { z[i] = -g[i]; dadd[i] = u_grp[pose_grp[i / 6]] * diag[i]; }
}
// q1_w = 0.5 dx_w . (u_w D dx_w - g_w) (bavoxel.hpp:729) -> out[4w+1]; non-finite dx or singular pivot -> out[4w+2]
__global__ void lidar_q1_grouped_kernel(const int* __restrict__ grp_ptr, const double* __restrict__ dx, const double* __restrict__ diag,
                                        const double* __restrict__ g, const double* __restrict__ u_grp, const int* __restrict__ status,
                                        double* __restrict__ out) {
  __shared__ double red[32];
  const int w = blockIdx.x;
  const double u = u_grp[w];
  double s = 0.0, bad = 0.0;
  for (int i = 6 * grp_ptr[w] + threadIdx.x; i < 6 * grp_ptr[w + 1]; i += 128) {
    const double d = dx[i];
    s += d * (u * diag[i] * d - g[i]);
    if (!isfinite(d)) bad = 1.0;
  }
  const double tot = block_sum<128>(s, red);
  const double tb = block_sum<128>(bad, red);
  if (threadIdx.x == 0) { out[4 * w + 1] = 0.5 * tot; out[4 * w + 2] = tb + (status[w] ? 1.0 : 0.0); }
}
// poses <- trial for the windows whose step was accepted (bavoxel.hpp:744-746 per window)
__global__ void lidar_select_poses_kernel(int W, const int* __restrict__ pose_grp, const int* __restrict__ accept,
                                          const double* __restrict__ trial, double* __restrict__ poses) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 12 * W && accept[pose_grp[i / 12]]) poses[i] = trial[i];
}

// the local voxel order is not the caller's (voxels ordered by lowest pose, or a shard's share): the caller's records and pose
// indices are on the device as they are, and every local slot w picks its own.  Local voxel i of w by binary search in the
// local CSR; slot0[i] = its first slot in the caller's arrays.
__global__ void lidar_gather_slots_kernel(long long nnz, long long nnz_pad, int n_vox, const int* __restrict__ l_vox_ptr,
                                          const int* __restrict__ slot0, const int* __restrict__ caller_pidx,
                                          const double* __restrict__ aos, int* __restrict__ pidx, double2* __restrict__ soa) {
  const long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (w >= nnz) return;
  int lo = 0, hi = n_vox;
  while (hi - lo > 1) { const int m = (lo + hi) >> 1; if (l_vox_ptr[m] <= w) lo = m; else hi = m; }
  const long long q = slot0[lo] + (w - l_vox_ptr[lo]);
  pidx[w] = caller_pidx[q];
  const double2* r = reinterpret_cast<const double2*>(aos + 10 * q);
#pragma unroll
  for (int k = 0; k < 5; ++k) soa[k * nnz_pad + w] = r[k];
}

// out[i] = aos[src[i]]   (10-double cluster records)
__global__ void lidar_gather_aos_kernel(long long n, const int* __restrict__ src, const double* __restrict__ aos, double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* a = aos + 10 * (long long)src[i];
#pragma unroll
  for (int k = 0; k < 10; ++k) out[10 * i + k] = a[k];
}

}  // namespace lvba

struct lvba_lidar_problem {
  int W = 0;
  long long V_total = 0;          // voxels of the whole problem (the AVG_THR divisor, bavoxel.hpp:635)
  long long V_local = 0, nnz_local = 0, n_pairs = 0;
  int n_batches = 0, n_tiles = 0;
  int device = 0;
  // host copies kept for counters / structure queries
  std::vector<long long> h_vox_ptr_all;
  std::vector<int> h_pose_idx_all;
  bool have_structure = false;
  cudaStream_t stream = nullptr;
  lvba::DevBuf<double2> cl;
  lvba::DevBuf<int> pidx, vox_ptr, batch_vox, tile_vox;
  lvba::tiles::Runs<lvba::CudaExec> prun, drun;   // the build's destination table: pose pairs by H block, slots by pose
  lvba::DevBuf<double> poses, poses0, trial, H, g, diag, dadd, dx, batch_res, scal;
  lvba::Envelope env;
  lvba::EnvSolver solver;
  lvba::PhaseTimers timers;
  double* h_scal = nullptr;       // pinned: [0] r1 sum, [1] q1, [2] dx non-finite flag, [3] r2 sum, [4] factor status
  int64_t launches = 0, h2d = 0, d2h = 0;
  double ms_setup = 0.0;
  // LM state
  lvba_lidar_opts opts;
  lvba::BalmState lm;
  bool is_calc_hess = true;
  int builds = 0;
  // ---- batched window BA: n_groups independent windows in one block-diagonal system
  int n_groups = 0;
  std::vector<int> grp_ptr;            // [G+1] pose offsets
  std::vector<long long> grp_V;        // voxels per window (AVG_THR divisor of each window)
  lvba::DevBuf<int> d_grp_ptr, d_pose_grp, d_grp_batch, d_grp_tile, d_accept;   // d_grp_batch / d_grp_tile: batch / tile range per window
  lvba::DevBuf<double> d_u_grp, d_grp_scal;
  double* h_grp_scal = nullptr;        // pinned [4G]: r1 sum, q1, bad flag, r2 sum per window
  size_t h_grp_scal_bytes = 0;
  // ---- voxels seen from more than kSlots poses: outside the batches, through the passes of lidar_big.h
  long long n_big = 0, n_big_slots = 0, n_big_pairs = 0;
  lvba::DevBuf<int64_t> big_vox_ptr, big_pair_ptr;
  lvba::DevBuf<int32_t> big_pose;
  lvba::DevBuf<double> big_cl, big_params, big_feat;
  // ---- deterministic mode (lvba_lidar_opts::deterministic): the records of every contribution to H and g and the order in
  // which they are summed, set up when a reset first asks for the mode (lidar_det_setup)
  bool det = false, det_ready = false;
  lvba::tiles::FixedSum<lvba::CudaExec> det_H, det_g;
  // ---- the rows of the pose system (lvba_lidar_opts::pose_fixed): the free poses in ascending order.  Without a mask every
  // pose is its own row (n_rows = W; row_of, pose_of_row and d_row_of empty)
  int n_rows = 0;
  std::vector<uint8_t> pose_fixed;                 // the handle's constant poses (empty: none)
  std::vector<int> row_of, pose_of_row;
  lvba::DevBuf<int> d_row_of;
  std::vector<int> grp_row_ptr;                    // batched window BA: [G+1] row offsets of the windows
  lvba::DevBuf<int> d_grp_row_ptr, d_row_grp;      // the same on the device, and the window of every row
  bool unusable = false;                           // a re-plan failed and so did restoring the previous one (lidar_replan)
  // ---- voxel outlier removal (lidar_outliers.h; one GPU, a handle with its host structure): where every voxel's records are,
  // and on the device, uploaded at the first per-voxel residual of a plan, the handle voxel of every local voxel (none when the
  // layout is the identity) and of every big voxel
  bool have_home = false, vox_id_ready = false;
  lvba::outliers::VoxelHome home;
  lvba::DevBuf<int> d_vox_id, d_big_id;
  lvba::DevBuf<double> d_vox_res;                  // [V_total] lambda_0 of every voxel, handle order
  lvba::big::View big_view() const {
    return lvba::big::View{(int64_t)n_big, big_vox_ptr.p, big_pose.p, big_cl.p, big_pair_ptr.p, env.d_first.p, env.d_row_start.p,
                           d_row_of.p, (int64_t)env.nblocks, W};
  }

  // the tiles' CSR for the passes of lidar_tiles.h (vox_pair: set by lidar_tables)
  lvba::tiles::TableIn table_in() const {
    return lvba::tiles::TableIn{n_tiles, W, env.nblocks, tile_vox.p, vox_ptr.p, pidx.p, nullptr, env.d_first.p, env.d_row_start.p, d_row_of.p};
  }
  lvba::LidarView view() const {
    lvba::LidarView v_;
    v_.W = W; v_.cl = cl.p; v_.nnz_pad = (long long)(cl.n / 5);
    v_.pidx = pidx.p; v_.vox_ptr = vox_ptr.p;
    v_.n_batches = n_batches; v_.batch_vox = batch_vox.p;
    v_.n_tiles = n_tiles; v_.tile_vox = tile_vox.p;
    v_.tile_prun = prun.tile_run.p; v_.prun_ptr = prun.run_ptr.p; v_.pairs = prun.code.p;
    v_.tile_drun = drun.tile_run.p; v_.drun_ptr = drun.run_ptr.p; v_.dslot = drun.code.p;
    v_.row_of = d_row_of.p;
    return v_;
  }
  ~lvba_lidar_problem() {
    if (stream) { cudaStreamSynchronize(stream); cudaStreamDestroy(stream); }     // buffers (members, destroyed after this body) must be idle when parked
    lvba::pinned_pool().give(h_scal, 8 * sizeof(double));                          // after the drain: no read-back may still be writing them
    lvba::pinned_pool().give(h_grp_scal, h_grp_scal_bytes);
  }
};

namespace lvba {

inline int lidar_validate(int32_t W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx,
                          const double* clusters, const double* poses) {
  if (W <= 0 || V < 0) return fail(LVBA_ERR_INVALID_ARG, "W=%d V=%lld must be positive", W, (long long)V);
  if (!vox_ptr || !poses || (V > 0 && (!pose_idx || !clusters))) return fail(LVBA_ERR_INVALID_ARG, "null input pointer");
  if (vox_ptr[0] != 0) return fail(LVBA_ERR_INVALID_ARG, "vox_ptr[0] must be 0");
  // the CSR is checked in parallel chunks; the first offending voxel (lowest index) is reported
  int64_t bad_at[kMaxSetupThreads]; int bad_kind[kMaxSetupThreads]; int64_t bad_aux[kMaxSetupThreads];
  for (int w = 0; w < kMaxSetupThreads; ++w) { bad_at[w] = -1; bad_kind[w] = 0; bad_aux[w] = 0; }
  parallel_chunks(V, 1 << 14, [&](int64_t a0, int64_t a1, int w) {
    for (int64_t a = a0; a < a1; ++a) {
      const int64_t lo = vox_ptr[a], hi = vox_ptr[a + 1];
      int kind = 0; int64_t aux = 0;
      if (hi <= lo) kind = 1;
      else
        for (int64_t s = lo; s < hi; ++s) {
          const int p = pose_idx[s];
          if (p < 0 || p >= W) { kind = 3; aux = s; break; }
          if (s > lo && pose_idx[s - 1] >= p) { kind = 4; break; }
        }
      if (kind) { bad_at[w] = a; bad_kind[w] = kind; bad_aux[w] = aux; return; }
    }
  });
  for (int w = 0; w < kMaxSetupThreads; ++w) {
    if (bad_at[w] < 0) continue;
    const long long a = (long long)bad_at[w];
    switch (bad_kind[w]) {
      case 1: return fail(LVBA_ERR_INVALID_ARG, "voxel %lld has no slots (vox_ptr not increasing)", a);
      case 3: return fail(LVBA_ERR_INVALID_ARG, "pose_idx[%lld]=%d out of [0,%d)", (long long)bad_aux[w], pose_idx[bad_aux[w]], W);
      default: return fail(LVBA_ERR_INVALID_ARG, "pose_idx must be strictly ascending inside voxel %lld", a);
    }
  }
  if (vox_ptr[V] >= (1LL << 31)) return fail(LVBA_ERR_UNSUPPORTED, "more than 2^31 slots");
  return LVBA_OK;
}

// lvba_lidar_opts::pose_fixed as the handle keeps it: W bytes with a nonzero entry, or empty (NULL and all-zero masks)
inline std::vector<uint8_t> lidar_mask(int W, const uint8_t* pose_fixed) {
  if (!pose_fixed || std::none_of(pose_fixed, pose_fixed + W, [](uint8_t b) { return b != 0; })) return {};
  std::vector<uint8_t> m(pose_fixed, pose_fixed + W);
  for (uint8_t& b : m) b = b != 0;
  return m;
}

// constant poses run on one GPU (a voxel's shard follows its lowest pose, whatever is constant; a sharded handle is not re-planned)
inline int lidar_check_mask(bool has_mask) {
  if (has_mask && comm().active())
    return fail(LVBA_ERR_UNSUPPORTED, "pose_fixed runs on one GPU: constant poses are not supported with an active communicator");
  return LVBA_OK;
}

// a handle whose failed re-plan could not be undone (lidar_replan) takes no further calls but destroy and the pose copies
inline int lidar_check_usable(const lvba_lidar_problem* P) {
  if (P->unusable) return fail(LVBA_ERR_INVALID_ARG, "this handle lost its plan in a failed lvba_lidar_reset_lm: destroy it");
  return LVBA_OK;
}

// The rows of the pose system for the constant poses `mask` (empty: none), their envelope over the caller's CSR and, for the
// single solve, the solver path.  A voxel without a free slot couples no rows; one row system per handle.
inline int lidar_plan_rows(lvba_lidar_problem* P, const std::vector<uint8_t>& mask, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx) {
  cudaStream_t s = P->stream;
  if (mask.empty()) {
    P->n_rows = P->W;
    P->row_of.clear(); P->pose_of_row.clear();
    P->d_row_of.release();
  } else {
    P->n_rows = lidar_row_map(P->W, mask.data(), P->row_of, P->pose_of_row);
    LVBA_TRY(P->d_row_of.upload(P->row_of, s, &P->h2d));
  }
  if (P->n_rows > 0) {
    LVBA_TRY(P->env.build(lidar_first_rows(P->W, V, vox_ptr, pose_idx, mask.empty() ? nullptr : P->row_of.data(), P->n_rows), s, &P->h2d));
    if (P->n_groups == 0) LVBA_TRY(P->solver.prepare(P->env, s));
  } else {                                   // every pose constant: no pose system
    Envelope& e = P->env;
    e.n = 0; e.nblocks = 0; e.max_col = 0;
    e.first.clear(); e.last.clear(); e.row_start.clear();
    e.d_first.release(); e.d_last.release(); e.d_row_start.release();
  }
  return LVBA_OK;
}

// The rest of the plan that follows the rows, once the voxel layout is on the device: the windows' rows and the block-diagonal
// solver of a batch (a window without a free pose is an empty group), the build's destination table and the row-sized buffers.
inline int lidar_plan_tables(lvba_lidar_problem* P) {
  cudaStream_t s = P->stream;
  if (P->n_groups > 0) {
    const int G = P->n_groups;
    for (int g = 0; g < G; ++g)                                // counted in poses, constant ones included
      if (P->grp_ptr[g + 1] - P->grp_ptr[g] > 31)
        return fail(LVBA_ERR_UNSUPPORTED, "window %d has %d poses; the batched solve handles <= 31 per window", g, P->grp_ptr[g + 1] - P->grp_ptr[g]);
    P->grp_row_ptr.assign((size_t)G + 1, 0);
    std::vector<int> row_grp;
    row_grp.reserve((size_t)P->n_rows);
    for (int g = 0; g < G; ++g) {
      for (int p = P->grp_ptr[g]; p < P->grp_ptr[g + 1]; ++p)
        if (P->row_of.empty() || P->row_of[p] >= 0) row_grp.push_back(g);
      P->grp_row_ptr[g + 1] = (int)row_grp.size();
    }
    if (P->n_rows > 0) LVBA_TRY(P->solver.prepare(P->env, s, LVBA_SOLVE_AUTO, 0, P->grp_row_ptr));
    LVBA_TRY(P->d_grp_row_ptr.upload(P->grp_row_ptr, s, &P->h2d));
    LVBA_TRY(P->d_row_grp.upload(row_grp, s, &P->h2d));
    LVBA_CUDA(cudaStreamSynchronize(s));                       // row_grp is uploaded
  }
  if (P->n_tiles <= 0) {                                       // no tiles (a removal left only big voxels): no runs from a previous plan
    for (tiles::Runs<CudaExec>* r : {&P->prun, &P->drun}) { r->code.release(); r->run_ptr.release(); r->tile_run.release(); r->n_runs = 0; }
  }
  {                                                            // destination table of the build, on the device from the local CSR
    CudaExec ex;
    ex.stream = s;
    LVBA_TRY(lidar_tables(ex, P->table_in(), P->V_local, P->n_pairs, P->nnz_local, P->prun, P->drun));
    P->launches += ex.launches;
  }
  LVBA_TRY(P->H.alloc((size_t)P->env.nblocks * 36));
  LVBA_TRY(P->g.alloc((size_t)P->n_rows * 6));
  LVBA_TRY(P->diag.alloc((size_t)P->n_rows * 6));
  LVBA_TRY(P->dadd.alloc((size_t)P->n_rows * 6));
  LVBA_TRY(P->dx.alloc((size_t)P->n_rows * 6));
  return LVBA_OK;
}

// pose_fixed: the constant poses to plan with (null: none; lidar_mask'ed by the caller's opts); the one-shot calls plan once
// with their mask, a handle starts with none.
inline int lidar_create_impl(int32_t W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx,
                             const double* clusters, const double* poses, int32_t device,
                             lvba_lidar_problem** out, int32_t n_groups = 0, const int32_t* grp_ptr = nullptr,
                             const double* d_clusters = nullptr, bool keep_structure = true, const uint8_t* pose_fixed = nullptr) {
  // keep_structure: copy the caller's CSR for lvba_lidar_counts (a handle may outlive the caller's arrays); the one-shot calls,
  // whose handle dies before they return, skip the 7 MB of copies
  // d_clusters: the same AoS records already resident on the selected device (a voxel map's export buffer); when set,
  // `clusters` may be null and no cluster bytes cross PCIe.
  if (!out) return fail(LVBA_ERR_INVALID_ARG, "out is null");
  *out = nullptr;
  const double t_val0 = wall_ms();
  LVBA_TRY(lidar_validate(W, V, vox_ptr, pose_idx, d_clusters ? d_clusters : clusters, poses));
  std::vector<uint8_t> mask = lidar_mask(W, pose_fixed);
  LVBA_TRY(lidar_check_mask(!mask.empty()));
  LVBA_TRY(select_device(device));
  const double t0 = wall_ms();
  SetupLaps lap("lidar setup", 22, nullptr, t_val0);
  lap.host("validate");
  std::unique_ptr<lvba_lidar_problem> P(new lvba_lidar_problem());
  P->W = W; P->V_total = V;
  LVBA_CUDA(cudaGetDevice(&P->device));
  LVBA_CUDA(cudaStreamCreateWithFlags(&P->stream, cudaStreamNonBlocking));
  P->timers.stream = P->stream;
  LVBA_TRY(pinned_pool().take(8 * sizeof(double), (void**)&P->h_scal));
  cudaStream_t s = P->stream;

  lap("ctx/stream/pinned");
  // the caller's cluster records (the bulk of the upload: 80 B per slot) start crossing PCIe now, in ONE copy, while the
  // host derives the structure below; every path further down reads them from `aos_dev`
  // (on a stream of its own: the set-up below synchronises `s` several times for its small uploads)
  DevBuf<double> aos;
  const double* aos_dev = d_clusters;
  struct CopyLane {
    cudaStream_t st = nullptr; cudaEvent_t done = nullptr;
    ~CopyLane() { if (st) { cudaStreamSynchronize(st); cudaStreamDestroy(st); } if (done) cudaEventDestroy(done); }
  } lane;
  if (!aos_dev && vox_ptr[V] > 0) {
    LVBA_TRY(aos.alloc((size_t)vox_ptr[V] * 10));
    LVBA_CUDA(cudaStreamCreateWithFlags(&lane.st, cudaStreamNonBlocking));
    LVBA_CUDA(cudaEventCreateWithFlags(&lane.done, cudaEventDisableTiming));
    LVBA_CUDA(cudaMemcpyAsync(aos.p, clusters, (size_t)vox_ptr[V] * 10 * sizeof(double), cudaMemcpyHostToDevice, lane.st));
    LVBA_CUDA(cudaEventRecord(lane.done, lane.st));
    P->h2d += vox_ptr[V] * 80;
    aos_dev = aos.p;
  }
  if (keep_structure) {
    P->h_vox_ptr_all.assign(vox_ptr, vox_ptr + V + 1);
    P->h_pose_idx_all.assign(pose_idx, pose_idx + vox_ptr[V]);
  }
  P->have_structure = keep_structure;
  lap("host copies");

  Comm& cm = comm();
  const bool sharded = cm.active();
  if (n_groups > 0) {
    if (sharded) return fail(LVBA_ERR_UNSUPPORTED, "the batched window BA runs on one GPU per call (windows are independent: shard them across ranks)");
    P->n_groups = n_groups;
    P->grp_ptr.assign(grp_ptr, grp_ptr + n_groups + 1);
  }
  // ---- rows and their envelope over ALL voxels (identical on every rank).  A rank holds the voxels of its poses, cut by the
  // solver's row split: the solver is prepared first.  The batched solve (one GPU) is prepared after the layout, which checks
  // that no voxel spans two windows (lidar_plan_tables).
  P->pose_fixed = std::move(mask);
  LVBA_TRY(lidar_plan_rows(P.get(), P->pose_fixed, V, vox_ptr, pose_idx));
  lap("envelope+solver alloc");

  // ---- shard: voxel -> owner of its lowest pose index (SURVEY.md §8e)
  std::vector<int64_t> owned;
  if (sharded) {
    owned.reserve((size_t)V);
    for (int64_t a = 0; a < V; ++a)
      if ((P->solver.dist() ? P->solver.dist_owner(pose_idx[vox_ptr[a]]) : shard_owner(pose_idx[vox_ptr[a]], W, cm.n_ranks)) == cm.rank)
        owned.push_back(a);
  }
  LidarLayout L;
  switch (lidar_layout(W, V, vox_ptr, pose_idx, sharded ? &owned : nullptr, n_groups, grp_ptr, L)) {
    case kLayoutSpansWindows: return fail(LVBA_ERR_INVALID_ARG, "voxel %lld spans two windows", (long long)L.err_vox);
    case kLayoutBigInBatch:
      return fail(LVBA_ERR_UNSUPPORTED, "batched window BA: voxel %lld is seen from %lld poses (more than %d)", (long long)L.err_vox,
                  (long long)(vox_ptr[L.err_vox + 1] - vox_ptr[L.err_vox]), kSlots);
  }
  if (keep_structure && !sharded && n_groups == 0) {
    outliers::voxel_home(V, vox_ptr, L, P->home);
    P->have_home = true;
  }
  const int64_t Vl = (int64_t)L.slot0.size();
  const long long nnz = L.nnz;
  P->V_local = Vl; P->nnz_local = nnz; P->n_pairs = L.n_pairs;
  P->n_batches = (int)L.batch_vox.size() - 1;
  P->n_tiles = (int)L.tile_vox.size() - 1;
  if (n_groups > 0) {
    P->grp_V = L.grp_V;
    LVBA_TRY(P->d_grp_batch.upload(L.grp_batch, s, &P->h2d));
    LVBA_TRY(P->d_grp_tile.upload(L.grp_tile, s, &P->h2d));
    LVBA_TRY(P->d_grp_ptr.upload(P->grp_ptr, s, &P->h2d));
    LVBA_TRY(P->d_pose_grp.upload(L.pose_grp, s, &P->h2d));
    LVBA_TRY(P->d_accept.alloc((size_t)n_groups));
    LVBA_TRY(P->d_u_grp.alloc((size_t)n_groups));
    LVBA_TRY(P->d_grp_scal.alloc((size_t)4 * n_groups));
    LVBA_TRY(P->d_grp_scal.zero(s));
    P->h_grp_scal_bytes = (size_t)4 * n_groups * sizeof(double);
    LVBA_TRY(pinned_pool().take(P->h_grp_scal_bytes, (void**)&P->h_grp_scal));
    LVBA_CUDA(cudaStreamSynchronize(s));                       // L's vectors are uploaded
  }

  lap("order+batches+tiles");
  // ---- upload.  Clusters: the caller's AoS records go up in ONE copy and are transposed to the SoA double2 layout
  //      by a kernel (which also picks the slots in the local voxel order unless that is the caller's).
  const long long nnz_pad = ((nnz + 31) / 32) * 32 + 32;
  LVBA_TRY(P->cl.alloc((size_t)5 * nnz_pad));
  LVBA_TRY(P->cl.zero(s));
  LVBA_TRY(P->vox_ptr.upload(L.l_vox_ptr, s, &P->h2d));
  if (lane.done) LVBA_CUDA(cudaStreamWaitEvent(s, lane.done, 0));            // the kernels below read the records
  {
    if (L.identity) {
      if (nnz > 0) {
        lidar_aos_to_soa_kernel<<<(unsigned)((nnz + 255) / 256), 256, 0, s>>>(nnz, nnz_pad, aos_dev, P->cl.p);
        ++P->launches;
      }
    } else {
      // reordered (or a shard's scattered) voxels: the ONE copy of the caller's records and pose indices + a device-side gather
      DevBuf<int> d_slot0, d_caller_pidx;
      if (nnz > 0) {
        LVBA_TRY(d_slot0.upload(L.slot0, s, &P->h2d));
        LVBA_TRY(d_caller_pidx.upload(reinterpret_cast<const int*>(pose_idx), (size_t)vox_ptr[V], s, &P->h2d));
        LVBA_TRY(P->pidx.alloc((size_t)nnz));
        lidar_gather_slots_kernel<<<(unsigned)((nnz + 255) / 256), 256, 0, s>>>(nnz, nnz_pad, (int)Vl, P->vox_ptr.p, d_slot0.p, d_caller_pidx.p,
                                                                                aos_dev, P->pidx.p, P->cl.p);
        ++P->launches;
      }
      if (!L.big_vox.empty()) {              // the big voxels' records stay AoS (lidar_big.h reads them slot by slot)
        P->n_big = (long long)L.big_vox.size(); P->n_big_slots = (long long)L.big_src.size(); P->n_big_pairs = L.big_pair_ptr.back();
        DevBuf<int> d_bsrc;
        LVBA_TRY(d_bsrc.upload(L.big_src, s, &P->h2d));
        LVBA_TRY(P->big_vox_ptr.upload(L.big_vox_ptr, s, &P->h2d));
        LVBA_TRY(P->big_pair_ptr.upload(L.big_pair_ptr, s, &P->h2d));
        LVBA_TRY(P->big_pose.upload(L.big_pose, s, &P->h2d));
        LVBA_TRY(P->big_cl.alloc((size_t)P->n_big_slots * 10));
        LVBA_TRY(P->big_params.alloc((size_t)P->n_big * big::kParams));
        LVBA_TRY(P->big_feat.alloc((size_t)P->n_big_slots * big::kFeat));
        lidar_gather_aos_kernel<<<(unsigned)((P->n_big_slots + 255) / 256), 256, 0, s>>>(P->n_big_slots, d_bsrc.p, aos_dev, P->big_cl.p);
        ++P->launches;
        LVBA_CUDA(cudaStreamSynchronize(s)); // d_bsrc goes out of scope
      }
      LVBA_CUDA(cudaStreamSynchronize(s));   // d_slot0 and d_caller_pidx are freed on scope exit
    }
  }
  lap("cluster upload+SoA", s);
  static_assert(sizeof(int) == sizeof(int32_t), "pose_idx is uploaded as it is");
  if (L.identity) LVBA_TRY(P->pidx.upload(reinterpret_cast<const int*>(pose_idx), (size_t)nnz, s, &P->h2d));
  LVBA_TRY(P->batch_vox.upload(L.batch_vox, s, &P->h2d));
  LVBA_TRY(P->tile_vox.upload(L.tile_vox, s, &P->h2d));
  LVBA_TRY(lidar_plan_tables(P.get()));                       // destination table from the CSR just uploaded, row buffers
  lap("destination table");
  LVBA_TRY(P->poses.upload(poses, (size_t)W * 12, s, &P->h2d));
  LVBA_TRY(P->poses0.upload(poses, (size_t)W * 12, s));
  LVBA_TRY(P->trial.alloc((size_t)W * 12));
  LVBA_TRY(P->batch_res.alloc((size_t)std::max<long long>(std::max(P->n_batches, P->n_tiles) + P->n_big, 1)));
  LVBA_TRY(P->scal.alloc(8));
  LVBA_TRY(P->scal.zero(s));
  LVBA_CUDA(cudaFuncSetAttribute(lidar_build_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lidar_build_smem_bytes()));
  LVBA_CUDA(cudaFuncSetAttribute(lidar_build_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lidar_build_smem_bytes()));
  LVBA_CUDA(cudaStreamSynchronize(s));
  aos.release();                                               // the caller's records were consumed by the kernels above
  lap("index upload+allocs");
  lvba_lidar_default_opts(&P->opts);
  P->ms_setup = wall_ms() - t0;
  *out = P.release();
  return LVBA_OK;
}

// Deterministic mode: the records of the build and their destinations (lidar_det_index)
inline int lidar_det_setup(lvba_lidar_problem* P) {
  if (P->det_ready) return LVBA_OK;
  const int64_t nH = P->prun.n_runs + P->drun.n_runs + P->n_big_slots + P->n_big_pairs;
  if (nH >= (int64_t)1 << 32) return fail(LVBA_ERR_UNSUPPORTED, "deterministic mode: %lld contributions to H (at most 2^32)", (long long)nH);
  CudaExec ex;
  ex.stream = P->stream;
  LVBA_TRY(lidar_det_index(ex, P->table_in(), P->prun, P->drun, P->big_view(), P->n_big_slots, P->n_big_pairs, P->det_H, P->det_g));
  LVBA_CUDA(cudaFuncSetAttribute(lidar_build_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lidar_build_smem_bytes()));
  LVBA_CUDA(cudaFuncSetAttribute(lidar_build_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lidar_build_smem_bytes()));
  P->launches += ex.launches;
  P->det_ready = true;
  return LVBA_OK;
}

// A new set of constant poses on a handle (lvba_lidar_reset_lm): the rows, the envelope, the solver, the build's tables and the
// row-sized buffers again, from the handle's host copy of the caller's CSR.  The voxel layout does not depend on the rows
// (voxels stay in the order of their lowest pose), so the clusters, batches and tiles stay as they are on the device.  The
// result equals a fresh one-shot call with that mask, bit for bit in deterministic mode.  One GPU only (lidar_check_mask).
// A failure leaves the handle as it was (the previous plan is made again) with deterministic mode off; only if that fails too
// is the handle marked unusable, and then every call but destroy and the pose copies refuses it.
inline int lidar_replan(lvba_lidar_problem* P, std::vector<uint8_t> mask) {
  if (!P->have_structure) return fail(LVBA_ERR_UNSUPPORTED, "this problem was created without its host-side structure copy: it cannot be re-planned");
  cudaStream_t s = P->stream;
  LVBA_CUDA(cudaStreamSynchronize(s));                         // nothing in flight reads the buffers re-planned below
  // the records of deterministic mode follow the table: set up again when the mode is next asked for (lidar_set_mode)
  tiles::fixed_sum_release(P->det_H); tiles::fixed_sum_release(P->det_g);
  P->det_ready = false;
  P->det = false;
  P->solver.set_deterministic(false);
  static_assert(sizeof(long long) == sizeof(int64_t), "the host copy of vox_ptr is read as it is");
  auto plan_with = [&](const std::vector<uint8_t>& m) -> int {
    LVBA_TRY(lidar_plan_rows(P, m, P->V_total, reinterpret_cast<const int64_t*>(P->h_vox_ptr_all.data()), P->h_pose_idx_all.data()));
    LVBA_TRY(lidar_plan_tables(P));
    LVBA_CUDA(cudaStreamSynchronize(s));
    return LVBA_OK;
  };
  int rc;
  try { rc = plan_with(mask); } catch (const std::bad_alloc&) { rc = fail(LVBA_ERR_NOMEM, "host allocation failed"); }
  if (rc != LVBA_OK) {
    const std::string why = last_error_ref();
    cudaStreamSynchronize(s);
    cudaGetLastError();
    int rc_back;
    try { rc_back = plan_with(P->pose_fixed); } catch (const std::bad_alloc&) { rc_back = LVBA_ERR_NOMEM; }
    if (rc_back != LVBA_OK) {
      P->unusable = true;
      return fail(rc, "re-plan for the new pose_fixed failed (%s), and so did restoring the previous plan: destroy the handle", why.c_str());
    }
    return fail(rc, "re-plan for the new pose_fixed failed (%s); the handle keeps its previous constant poses", why.c_str());
  }
  P->pose_fixed = std::move(mask);
  return LVBA_OK;
}

// the LM mode of the handle (lvba_lidar_reset_lm and the one-shot calls): the constant poses and deterministic mode
inline int lidar_set_mode(lvba_lidar_problem* P, const lvba_lidar_opts& o) {
  if (o.deterministic && comm().active())
    return fail(LVBA_ERR_UNSUPPORTED, "deterministic mode runs on one GPU: the multi-GPU sums of NCCL have no fixed order");
  std::vector<uint8_t> mask = lidar_mask(P->W, o.pose_fixed);
  LVBA_TRY(lidar_check_mask(!mask.empty() || !P->pose_fixed.empty()));
  if (mask != P->pose_fixed) {
    LVBA_CUDA(cudaSetDevice(P->device));
    LVBA_TRY(lidar_replan(P, std::move(mask)));
  }
  if (o.deterministic) {
    LVBA_CUDA(cudaSetDevice(P->device));
    const int rc = lidar_det_setup(P);
    if (rc != LVBA_OK) {                                      // nothing half set up stays on the handle
      tiles::fixed_sum_release(P->det_H); tiles::fixed_sum_release(P->det_g);
      return rc;
    }
  }
  P->det = o.deterministic != 0;
  P->solver.set_deterministic(P->det);
  return LVBA_OK;
}

// voxels seen from more than kSlots poses (lidar_big.h): lambda_0 of voxel b -> batch_res[n_before + b] (after the partials of
// the tiles or batches); with the Hessian, their gradient / diagonal-block / pair-block contributions are added to g and H by
// atomics, or in deterministic mode stored into their records
inline int lidar_big_passes(lvba_lidar_problem* P, const double* d_poses, bool residual_only, int n_before) {
  cudaStream_t s = P->stream;
  const big::View bv = P->big_view();
  auto launch = [&](int64_t items, const auto& f) { wide_pass(s, items, f, &P->launches); };
  launch((int64_t)P->n_big, big::ParamsF{bv, d_poses, P->big_params.p, P->batch_res.p + n_before});
  if (!residual_only && P->det) {
    const int64_t h0 = P->prun.n_runs + P->drun.n_runs, g0 = P->drun.n_runs;
    launch((int64_t)P->n_big_slots, big::SlotsDetF{bv, d_poses, P->big_params.p, P->big_feat.p, P->det_H.rec.p + 36 * h0, P->det_g.rec.p + 6 * g0});
    launch((int64_t)P->n_big_pairs, big::PairsDetF{bv, P->big_params.p, P->big_feat.p, P->det_H.rec.p + 36 * (h0 + P->n_big_slots)});
  } else if (!residual_only) {
    launch((int64_t)P->n_big_slots, big::SlotsF{bv, d_poses, P->big_params.p, P->big_feat.p, P->H.p, P->g.p});
    launch((int64_t)P->n_big_pairs, big::PairsF{bv, P->big_params.p, P->big_feat.p, P->H.p});
  }
  LVBA_CUDA(cudaGetLastError());
  return LVBA_OK;
}

// H and g at the poses in `d_poses`; the partial residual sums of the tiles and big voxels in batch_res
inline int lidar_build_hg(lvba_lidar_problem* P, const double* d_poses) {
  cudaStream_t s = P->stream;
  LVBA_TRY(P->H.zero(s));
  LVBA_TRY(P->g.zero(s));
  if (P->n_tiles > 0) {
    const bool fixed = !P->pose_fixed.empty();
    double* H = P->det ? P->det_H.rec.p : P->H.p;
    double* g = P->det ? P->det_g.rec.p : P->g.p;
    const unsigned smem = (unsigned)lidar_build_smem_bytes();
    if (P->det && fixed) lidar_build_kernel<true, true><<<P->n_tiles, kTileSlots, smem, s>>>(P->view(), P->env.view(), d_poses, H, g, P->batch_res.p);
    else if (P->det) lidar_build_kernel<true, false><<<P->n_tiles, kTileSlots, smem, s>>>(P->view(), P->env.view(), d_poses, H, g, P->batch_res.p);
    else if (fixed) lidar_build_kernel<false, true><<<P->n_tiles, kTileSlots, smem, s>>>(P->view(), P->env.view(), d_poses, H, g, P->batch_res.p);
    else lidar_build_kernel<false, false><<<P->n_tiles, kTileSlots, smem, s>>>(P->view(), P->env.view(), d_poses, H, g, P->batch_res.p);
    ++P->launches;
  }
  if (P->n_big > 0) LVBA_TRY(lidar_big_passes(P, d_poses, /*residual_only=*/false, P->n_tiles));
  if (P->det) {
    CudaExec ex;
    ex.stream = s;
    LVBA_TRY(ex.for_each(P->det_H.by_dst.n_runs * 36, tiles::gather_of(P->det_H, P->H.p)));
    LVBA_TRY(ex.for_each(P->det_g.by_dst.n_runs * 6, tiles::gather_of(P->det_g, P->g.p)));
    P->launches += ex.launches;
  }
  LVBA_CUDA(cudaGetLastError());
  return LVBA_OK;
}

// H, g, sum(lambda0) at the poses in `d_poses`; result scalar lands in scal[slot]
inline int lidar_build_dev(lvba_lidar_problem* P, const double* d_poses, int slot) {
  cudaStream_t s = P->stream;
  LVBA_TRY(lidar_build_hg(P, d_poses));
  reduce_partials_kernel<<<1, 256, 0, s>>>(P->batch_res.p, (int)(P->n_tiles + P->n_big), P->scal.p + slot);
  ++P->launches;
  LVBA_CUDA(cudaGetLastError());
  Comm& cm = comm();
  if (cm.active()) {
    // row-owned H (SURVEY.md 8(e)): only the <= max_col block rows a rank's voxels reach into its right neighbour's range travel
    // (one ncclSend / ncclRecv pair); the full-matrix all-reduce remains for structures the chunked solver cannot cut per rank
    if (P->solver.dist()) LVBA_TRY(P->solver.exchange_rows(P->env, P->H.p, s, &P->launches));
    else LVBA_TRY(cm.allreduce_sum(P->H.p, (size_t)P->env.nblocks * 36, s));
    LVBA_TRY(cm.allreduce_sum(P->g.p, (size_t)P->W * 6, s));
    LVBA_TRY(cm.allreduce_sum(P->scal.p + slot, 1, s));
  }
  return LVBA_OK;
}

inline int lidar_residual_dev(lvba_lidar_problem* P, const double* d_poses, int slot) {
  cudaStream_t s = P->stream;
  if (P->n_batches > 0) {
    lidar_residual_kernel<false><<<P->n_batches, kSlots, 0, s>>>(P->view(), d_poses, P->batch_res.p, nullptr);
    ++P->launches;
  }
  if (P->n_big > 0) LVBA_TRY(lidar_big_passes(P, d_poses, /*residual_only=*/true, P->n_batches));
  reduce_partials_kernel<<<1, 256, 0, s>>>(P->batch_res.p, (int)(P->n_batches + P->n_big), P->scal.p + slot);
  ++P->launches;
  LVBA_CUDA(cudaGetLastError());
  Comm& cm = comm();
  if (cm.active()) LVBA_TRY(cm.allreduce_sum(P->scal.p + slot, 1, s));
  return LVBA_OK;
}

// (H + u diag(H)) dx = -g over the rows ; q1 ; leaves dx on the device.  scal[1] = q1, scal[2] = non-finite flag
inline int lidar_solve_dev(lvba_lidar_problem* P, double u) {
  cudaStream_t s = P->stream;
  if (P->n_rows == 0) {                                      // every pose constant: nothing to solve, q1 = 0
    LVBA_CUDA(cudaMemsetAsync(P->scal.p + 1, 0, 2 * sizeof(double), s));
    return LVBA_OK;
  }
  const int n6 = 6 * P->n_rows;
  const EnvView ev = P->env.view();
  env_get_diag_kernel<<<(n6 + 255) / 256, 256, 0, s>>>(ev, P->H.p, P->diag.p);
  if (P->solver.dist()) {                                    // a rank holds the rows it owns: the diagonal of the others arrives by all-reduce
    nd_pass_kernel<<<(n6 + 255) / 256, 256, 0, s>>>((long long)n6, nd::ZeroForeignF{P->diag.p, P->solver.dist_begin(), P->solver.dist_end()});
    ++P->launches;
    LVBA_TRY(comm().allreduce_sum(P->diag.p, (size_t)n6, s));
  }
  lidar_rhs_kernel<<<(n6 + 255) / 256, 256, 0, s>>>(n6, P->g.p, P->diag.p, u, P->solver.z.p, P->dadd.p);
  P->launches += 2;
  LVBA_TRY(P->solver.solve(P->env, P->H.p, P->dadd.p, P->dx.p, s, &P->launches));
  lidar_q1_kernel<<<1, 256, 0, s>>>(n6, P->dx.p, P->diag.p, P->g.p, u, P->scal.p + 1);
  ++P->launches;
  LVBA_CUDA(cudaGetLastError());
  return LVBA_OK;
}

inline int lidar_fetch_scal(lvba_lidar_problem* P) {
  LVBA_CUDA(cudaMemcpyAsync(P->h_scal, P->scal.p, 8 * sizeof(double), cudaMemcpyDeviceToHost, P->stream));
  if (P->n_rows > 0) LVBA_CUDA(cudaMemcpyAsync(P->h_scal + 7, P->solver.status.p, sizeof(int), cudaMemcpyDeviceToHost, P->stream));
  else memset(P->h_scal + 7, 0, sizeof(int));                // no solver ran: a status of 0
  LVBA_CUDA(cudaStreamSynchronize(P->stream));
  P->d2h += 8 * sizeof(double) + sizeof(int);
  return LVBA_OK;
}

// trial = poses (+) dx, constant poses copied as they are
inline void lidar_retract(lvba_lidar_problem* P) {
  if (P->pose_fixed.empty())
    lidar_retract_kernel<<<(P->W + 127) / 128, 128, 0, P->stream>>>(P->W, P->poses.p, P->dx.p, P->trial.p);
  else
    lidar_retract_rows_kernel<<<(P->W + 127) / 128, 128, 0, P->stream>>>(P->W, P->poses.p, P->dx.p, P->d_row_of.p, P->trial.p);
  ++P->launches;
}

// n passes of the damping_iter loop body (bavoxel.hpp:686-766)
inline int lidar_iterate_impl(lvba_lidar_problem* P, int n_iter, lvba_summary* sum) {
  const double t0 = wall_ms();
  const int64_t l0 = P->launches, h0 = P->h2d, d0 = P->d2h;
  const double V = (double)P->V_total;
  BalmState& lm = P->lm;
  const int iters0 = lm.iters, acc0 = lm.accepted, builds0 = P->builds;
  if (P->n_rows == 0 && n_iter > 0 && !lm.converged) {       // every pose constant: the residual once, nothing to solve (Ceres:
    P->timers.begin(PH_RESID);                               // no free parameter block, function tolerance)
    LVBA_TRY(lidar_residual_dev(P, P->poses.p, 3));
    P->timers.end();
    LVBA_TRY(lidar_fetch_scal(P));
    lm.cost_first = lm.cost_last = lm.residual1 = P->h_scal[3] / V;
    lm.have_first = lm.converged = true;
    lm.term = LVBA_TERM_FUNCTION_TOL;
  }
  for (int it = 0; it < n_iter && !lm.converged; ++it) {
    if (P->is_calc_hess) {                                   // divide_thread, :688-689
      P->timers.begin(PH_BUILD);
      LVBA_TRY(lidar_build_dev(P, P->poses.p, 0));
      P->timers.end();
      ++P->builds;
    }
    P->timers.begin(PH_SOLVE);
    LVBA_TRY(lidar_solve_dev(P, lm.u));                      // :692-710, :729
    P->timers.end();
    P->timers.begin(PH_RESID);
    lidar_retract(P);                                        // :722-727
    LVBA_TRY(lidar_residual_dev(P, P->trial.p, 3));          // only_residual, :731
    P->timers.end();
    LVBA_TRY(lidar_fetch_scal(P));
    // residual1 is refreshed after a build only; an accepted step rebuilds H at the new poses (:744-758)
    P->is_calc_hess = balm_step(lm, P->h_scal, V, P->is_calc_hess, P->opts, "lvba lidar");
    if (P->is_calc_hess) std::swap(P->poses.p, P->trial.p);
  }
  if (sum) {
    LVBA_CUDA(cudaStreamSynchronize(P->stream));
    double ms[PH_COUNT] = {0, 0, 0};
    P->timers.collect(ms);
    write_summary(sum, lm.iters - iters0, lm.accepted - acc0, P->builds - builds0, lm.term, lm.cost_first, lm.cost_last, lm.u, ms,
                  wall_ms() - t0, P->launches - l0, P->h2d - h0, P->d2h - d0);
  }
  return LVBA_OK;
}

// ---------------------------------------------------------------- voxel outlier removal (lidar_outliers.h)
// the calls that read or change the handle's voxel set: one GPU, the handle's host structure and the voxel homes
inline int lidar_check_voxel_set(const lvba_lidar_problem* P) {
  LVBA_TRY(lidar_check_usable(P));
  if (comm().active()) return fail(LVBA_ERR_UNSUPPORTED, "per-voxel residuals and voxel removal run on one GPU: not with an active communicator");
  if (!P->have_structure || !P->have_home)
    return fail(LVBA_ERR_UNSUPPORTED, "this problem was created without its host-side structure copy: its voxels cannot be listed or removed");
  return LVBA_OK;
}

// lambda_0 of every voxel at `d_poses` into d_vox_res, handle order: the residual pass with kPerVoxel for the batches, and the
// big voxels' lambda_0 that lidar_big_passes leaves after them in batch_res scattered to their handle positions
inline int lidar_voxel_residuals_dev(lvba_lidar_problem* P, const double* d_poses) {
  cudaStream_t s = P->stream;
  if (!P->vox_id_ready) {
    if (!P->home.local_vox.empty()) LVBA_TRY(P->d_vox_id.upload(P->home.local_vox, s, &P->h2d)); else P->d_vox_id.release();
    if (!P->home.big_vox.empty()) LVBA_TRY(P->d_big_id.upload(P->home.big_vox, s, &P->h2d)); else P->d_big_id.release();
    P->vox_id_ready = true;
  }
  if (P->d_vox_res.n < (size_t)P->V_total) LVBA_TRY(P->d_vox_res.alloc((size_t)P->V_total));
  if (P->n_batches > 0) {
    lidar_residual_kernel<true><<<P->n_batches, kSlots, 0, s>>>(P->view(), d_poses, P->d_vox_res.p, P->d_vox_id.p);
    ++P->launches;
  }
  if (P->n_big > 0) {
    LVBA_TRY(lidar_big_passes(P, d_poses, /*residual_only=*/true, P->n_batches));
    CudaExec ex;
    ex.stream = s;
    LVBA_TRY(ex.for_each(P->n_big, outliers::ScatterF{P->batch_res.p + P->n_batches, P->d_big_id.p, P->d_vox_res.p}));
    P->launches += ex.launches;
  }
  LVBA_CUDA(cudaGetLastError());
  return LVBA_OK;
}

// The handle's plan after removing the voxels with remove[a] != 0 (host, [V_total], at least one voxel kept): the same plan as
// lvba_lidar_create on the kept voxels' CSR and records with the handle's constant poses.  The records move device to device:
// a gather fills new SoA and big-voxel buffers, built beside the old ones, from where each kept voxel lives (P->home); only
// index arrays cross PCIe.  Then the rows, envelope, solver and tables of the kept CSR (as lidar_replan).  On failure the old
// buffers and plan come back (or else the handle is marked unusable).  Poses stay; the LM state is reset as lvba_lidar_reset_lm
// with the handle's opts would, and deterministic mode's records are set up again.
inline int lidar_remove_impl(lvba_lidar_problem* P, const uint8_t* remove) {
  cudaStream_t s = P->stream;
  LVBA_CUDA(cudaStreamSynchronize(s));                         // nothing in flight reads the buffers replaced below
  outliers::KeptPlan K;
  static_assert(sizeof(long long) == sizeof(int64_t), "the host copy of vox_ptr is read as it is");
  if (outliers::plan_kept(P->W, P->V_total, reinterpret_cast<const int64_t*>(P->h_vox_ptr_all.data()), P->h_pose_idx_all.data(), P->home,
                          remove, K) != kLayoutOk)
    return fail(LVBA_ERR_INVALID_ARG, "the kept voxels have no single-GPU layout");
  const LidarLayout& L = K.L;
  // ---- the new records beside the old ones
  struct Set {
    long long V_total = 0, V_local = 0, nnz_local = 0, n_pairs = 0, n_big = 0, n_big_slots = 0, n_big_pairs = 0;
    int n_batches = 0, n_tiles = 0;
    DevBuf<double2> cl;
    DevBuf<int> pidx, vox_ptr, batch_vox, tile_vox;
    DevBuf<int64_t> big_vox_ptr, big_pair_ptr;
    DevBuf<int32_t> big_pose;
    DevBuf<double> big_cl, big_params, big_feat, batch_res;
  } N;
  N.V_total = K.V; N.V_local = (long long)L.slot0.size(); N.nnz_local = L.nnz; N.n_pairs = L.n_pairs;
  N.n_batches = (int)L.batch_vox.size() - 1; N.n_tiles = (int)L.tile_vox.size() - 1;
  N.n_big = (long long)L.big_vox.size(); N.n_big_slots = (long long)L.big_src.size(); N.n_big_pairs = L.big_pair_ptr.back();
  {
    CudaExec ex;
    ex.stream = s;
    const long long nnz_pad = ((N.nnz_local + 31) / 32) * 32 + 32;  // as lidar_create_impl
    LVBA_TRY(N.cl.alloc((size_t)5 * nnz_pad));
    LVBA_TRY(N.cl.zero(s));
    LVBA_TRY(N.vox_ptr.upload(L.l_vox_ptr, s, &P->h2d));
    LVBA_TRY(N.pidx.alloc((size_t)N.nnz_local));
    DevBuf<int> d_src0, d_bsrc;
    if (N.nnz_local > 0) {
      LVBA_TRY(d_src0.upload(K.src0, s, &P->h2d));
      LVBA_TRY(ex.for_each(N.nnz_local, outliers::GatherSoaF{(int32_t)N.V_local, N.vox_ptr.p, d_src0.p, reinterpret_cast<const double*>(P->cl.p),
                                                             (int64_t)(P->cl.n / 5), P->pidx.p, reinterpret_cast<double*>(N.cl.p), nnz_pad, N.pidx.p}));
    }
    if (N.n_big > 0) {
      LVBA_TRY(d_bsrc.upload(K.big_src, s, &P->h2d));
      LVBA_TRY(N.big_vox_ptr.upload(L.big_vox_ptr, s, &P->h2d));
      LVBA_TRY(N.big_pair_ptr.upload(L.big_pair_ptr, s, &P->h2d));
      LVBA_TRY(N.big_pose.upload(L.big_pose, s, &P->h2d));
      LVBA_TRY(N.big_cl.alloc((size_t)N.n_big_slots * 10));
      LVBA_TRY(N.big_params.alloc((size_t)N.n_big * big::kParams));
      LVBA_TRY(N.big_feat.alloc((size_t)N.n_big_slots * big::kFeat));
      LVBA_TRY(ex.for_each(N.n_big_slots, outliers::GatherAosF{d_bsrc.p, P->big_cl.p, N.big_cl.p}));
    }
    LVBA_TRY(N.batch_vox.upload(L.batch_vox, s, &P->h2d));
    LVBA_TRY(N.tile_vox.upload(L.tile_vox, s, &P->h2d));
    LVBA_TRY(N.batch_res.alloc((size_t)std::max<long long>(std::max(N.n_batches, N.n_tiles) + N.n_big, 1)));
    LVBA_CUDA(cudaStreamSynchronize(s));                       // the gathers are done; d_src0 and d_bsrc are freed on scope exit
    P->launches += ex.launches;
  }
  // ---- swap them in (swapping again restores the old set)
  auto swap_set = [&](Set& o) {
    std::swap(P->V_total, o.V_total); std::swap(P->V_local, o.V_local); std::swap(P->nnz_local, o.nnz_local); std::swap(P->n_pairs, o.n_pairs);
    std::swap(P->n_big, o.n_big); std::swap(P->n_big_slots, o.n_big_slots); std::swap(P->n_big_pairs, o.n_big_pairs);
    std::swap(P->n_batches, o.n_batches); std::swap(P->n_tiles, o.n_tiles);
    P->cl.swap(o.cl); P->pidx.swap(o.pidx); P->vox_ptr.swap(o.vox_ptr); P->batch_vox.swap(o.batch_vox); P->tile_vox.swap(o.tile_vox);
    P->big_vox_ptr.swap(o.big_vox_ptr); P->big_pair_ptr.swap(o.big_pair_ptr); P->big_pose.swap(o.big_pose);
    P->big_cl.swap(o.big_cl); P->big_params.swap(o.big_params); P->big_feat.swap(o.big_feat); P->batch_res.swap(o.batch_res);
  };
  tiles::fixed_sum_release(P->det_H); tiles::fixed_sum_release(P->det_g);     // they follow the table: set up again below
  P->det_ready = false;
  swap_set(N);
  // the new plan, with deterministic mode's records when the handle is in that mode: a failure anywhere here restores the old one
  auto plan_with = [&](int64_t V, const int64_t* vp, const int32_t* pi, bool det) -> int {
    LVBA_TRY(lidar_plan_rows(P, P->pose_fixed, V, vp, pi));
    LVBA_TRY(lidar_plan_tables(P));
    if (det) LVBA_TRY(lidar_det_setup(P));
    LVBA_CUDA(cudaStreamSynchronize(s));
    return LVBA_OK;
  };
  int rc;
  try { rc = plan_with(K.V, K.vox_ptr.data(), K.pose_idx.data(), P->det); } catch (const std::bad_alloc&) { rc = fail(LVBA_ERR_NOMEM, "host allocation failed"); }
  if (rc != LVBA_OK) {
    const std::string why = last_error_ref();
    cudaStreamSynchronize(s);
    cudaGetLastError();
    tiles::fixed_sum_release(P->det_H); tiles::fixed_sum_release(P->det_g);
    P->det_ready = false;
    swap_set(N);
    int rc_back;
    try { rc_back = plan_with(P->V_total, reinterpret_cast<const int64_t*>(P->h_vox_ptr_all.data()), P->h_pose_idx_all.data(), false); }
    catch (const std::bad_alloc&) { rc_back = LVBA_ERR_NOMEM; }
    P->det = false;
    P->solver.set_deterministic(false);
    if (rc_back != LVBA_OK) {
      P->unusable = true;
      return fail(rc, "re-plan after the voxel removal failed (%s), and so did restoring the previous plan: destroy the handle", why.c_str());
    }
    return fail(rc, "re-plan after the voxel removal failed (%s); the handle keeps its voxels, deterministic mode is off", why.c_str());
  }
  P->h_vox_ptr_all.assign(K.vox_ptr.begin(), K.vox_ptr.end());
  P->h_pose_idx_all.swap(K.pose_idx);
  P->home = std::move(K.home);
  P->vox_id_ready = false;
  // the LM state of lvba_lidar_reset_lm with the handle's opts
  P->lm.reset(P->opts);
  P->is_calc_hess = true;
  P->builds = 0;
  P->solver.set_deterministic(P->det);
  return LVBA_OK;
}

// ---------------------------------------------------------------- batched window BA
// damping_iter (bavoxel.hpp:662-767) for every window at once: the windows share the kernels (one block-diagonal
// system, one CTA per window in the factorisation) but keep their own u, v, accept/reject decision and stop test,
// exactly as n_windows separate calls would.  A rejected window keeps its poses, so rebuilding H for everybody
// reproduces its previous H (":753-758 H not rebuilt" costs nothing in parity).
inline int lidar_batch_lm_impl(lvba_lidar_problem* P, int min_voxels_per_pose, lvba_summary* sums, lvba_summary* total) {
  const double t0 = wall_ms();
  const int G = P->n_groups;
  cudaStream_t s = P->stream;
  struct WinState : BalmState { bool active = false, skipped = false; };
  std::vector<WinState> ws((size_t)G);
  std::vector<double> u_host((size_t)G);
  std::vector<int> acc_host((size_t)G);
  int n_active = 0;
  bool any_constant = false;
  for (int g = 0; g < G; ++g) {
    const int Wg = P->grp_ptr[g + 1] - P->grp_ptr[g];       // the skip rule counts every pose of the window, constant ones included
    WinState& w = ws[g];
    w.reset(P->opts);
    w.skipped = Wg <= 0 || P->grp_V[g] == 0 || P->grp_V[g] < (long long)min_voxels_per_pose * Wg;   // src/lvba_system.cpp:262-266
    w.active = !w.skipped && P->grp_row_ptr[g + 1] > P->grp_row_ptr[g];
    if (w.skipped) w.term = LVBA_TERM_SKIPPED;
    any_constant = any_constant || (!w.skipped && !w.active);
    n_active += w.active;
  }
  if (any_constant) {                                          // windows whose poses are all constant: their residual once
    P->timers.begin(PH_RESID);
    if (P->n_batches > 0) {
      lidar_residual_kernel<false><<<P->n_batches, kSlots, 0, s>>>(P->view(), P->poses.p, P->batch_res.p, nullptr);
      ++P->launches;
    }
    lidar_group_sum_kernel<<<G, 128, 0, s>>>(P->batch_res.p, P->d_grp_batch.p, P->d_grp_scal.p, 3);
    ++P->launches;
    P->timers.end();
    LVBA_CUDA(cudaMemcpyAsync(P->h_grp_scal, P->d_grp_scal.p, (size_t)4 * G * sizeof(double), cudaMemcpyDeviceToHost, s));
    LVBA_CUDA(cudaStreamSynchronize(s));
    P->d2h += (int64_t)G * 32;
    for (int g = 0; g < G; ++g) {
      WinState& w = ws[g];
      if (w.skipped || w.active) continue;
      w.cost_first = w.cost_last = w.residual1 = P->h_grp_scal[4 * g + 3] / (double)P->grp_V[g];
      w.have_first = w.converged = true;
      w.term = LVBA_TERM_FUNCTION_TOL;
    }
  }
  const int n6 = 6 * P->n_rows;
  const EnvView ev = P->env.view();
  int passes = 0;
  for (int it = 0; it < P->opts.max_iter && n_active > 0; ++it, ++passes) {
    for (int g = 0; g < G; ++g) u_host[g] = ws[g].u;
    LVBA_CUDA(cudaMemcpyAsync(P->d_u_grp.p, u_host.data(), (size_t)G * sizeof(double), cudaMemcpyHostToDevice, s));
    P->h2d += (int64_t)G * 8;
    // ---- H, g, sum(lambda0) per window
    P->timers.begin(PH_BUILD);
    LVBA_TRY(lidar_build_hg(P, P->poses.p));
    lidar_group_sum_kernel<<<G, 128, 0, s>>>(P->batch_res.p, P->d_grp_tile.p, P->d_grp_scal.p, 0);
    ++P->launches;
    P->timers.end();
    ++P->builds;
    // ---- (H + u_w diag(H)) dx = -g, q1 per window
    P->timers.begin(PH_SOLVE);
    env_get_diag_kernel<<<(n6 + 255) / 256, 256, 0, s>>>(ev, P->H.p, P->diag.p);
    lidar_rhs_grouped_kernel<<<(n6 + 255) / 256, 256, 0, s>>>(n6, P->g.p, P->diag.p, P->d_u_grp.p, P->d_row_grp.p, P->solver.z.p, P->dadd.p);
    P->launches += 2;
    LVBA_TRY(P->solver.solve(P->env, P->H.p, P->dadd.p, P->dx.p, s, &P->launches));
    lidar_q1_grouped_kernel<<<G, 128, 0, s>>>(P->d_grp_row_ptr.p, P->dx.p, P->diag.p, P->g.p, P->d_u_grp.p, P->solver.status.p, P->d_grp_scal.p);
    ++P->launches;
    P->timers.end();
    // ---- trial state and its residual per window
    P->timers.begin(PH_RESID);
    lidar_retract(P);
    if (P->n_batches > 0) {
      lidar_residual_kernel<false><<<P->n_batches, kSlots, 0, s>>>(P->view(), P->trial.p, P->batch_res.p, nullptr);
      ++P->launches;
    }
    lidar_group_sum_kernel<<<G, 128, 0, s>>>(P->batch_res.p, P->d_grp_batch.p, P->d_grp_scal.p, 3);
    ++P->launches;
    P->timers.end();
    LVBA_CUDA(cudaMemcpyAsync(P->h_grp_scal, P->d_grp_scal.p, (size_t)4 * G * sizeof(double), cudaMemcpyDeviceToHost, s));
    LVBA_CUDA(cudaStreamSynchronize(s));
    P->d2h += (int64_t)G * 32;
    LVBA_CUDA(cudaGetLastError());
    // ---- per-window decision (bavoxel.hpp:733-762)
    for (int g = 0; g < G; ++g) {
      WinState& w = ws[g];
      acc_host[g] = 0;
      if (!w.active) continue;
      char label[32] = "";
      if (P->opts.verbose) snprintf(label, sizeof label, "lvba window %d", g);
      acc_host[g] = balm_step(w, P->h_grp_scal + 4 * g, (double)P->grp_V[g], /*rebuilt=*/true, P->opts, label);
      if (w.converged) { w.active = false; --n_active; }
    }
    LVBA_CUDA(cudaMemcpyAsync(P->d_accept.p, acc_host.data(), (size_t)G * sizeof(int), cudaMemcpyHostToDevice, s));
    P->h2d += (int64_t)G * 4;
    lidar_select_poses_kernel<<<(12 * P->W + 255) / 256, 256, 0, s>>>(P->W, P->d_pose_grp.p, P->d_accept.p, P->trial.p, P->poses.p);
    ++P->launches;
    LVBA_CUDA(cudaStreamSynchronize(s));                       // acc_host is reused next pass
  }
  double ms[PH_COUNT] = {0, 0, 0};
  P->timers.collect(ms);
  int accepted = 0;
  for (int g = 0; g < G; ++g) {
    const WinState& w = ws[g];
    if (sums) write_summary(&sums[g], w.iters, w.accepted, w.iters, w.term, w.cost_first, w.cost_last, w.u);
    accepted += w.accepted;
  }
  if (total) write_summary(total, passes, accepted, passes, /*term=*/0, 0.0, 0.0, 0.0, ms, wall_ms() - t0);
  return LVBA_OK;
}

// The rest of lvba_lidar_lm_batch and lvba_voxel_map_lidar_lm_batch once the call has created its batched handle p (`name`
// in the error message): every window's LM, the poses written back and the totals in *total on success; p destroyed.
inline int lidar_batch_one_shot(lvba_lidar_problem* p, const lvba_lidar_opts& o, int min_voxels_per_pose, double* poses,
                                lvba_summary* summaries, lvba_summary* total, double t0, const char* name) {
  p->opts = o;
  lvba_summary tot;
  memset(&tot, 0, sizeof tot);
  int rc = lidar_set_mode(p, o);
  if (rc == LVBA_OK) {
    try { rc = lidar_batch_lm_impl(p, min_voxels_per_pose, summaries, &tot); }
    catch (...) { rc = fail(LVBA_ERR_NOMEM, "host allocation failed in %s", name); }
  }
  if (rc == LVBA_OK) rc = lvba_lidar_get_poses(p, poses);     // written back only on success; skipped windows are unchanged on the device
  if (rc == LVBA_OK && total) {
    *total = tot;
    one_shot_totals(total, p, t0);
  }
  lvba_lidar_destroy(p);
  return rc;
}

}  // namespace lvba

// ================================================================ C ABI
extern "C" {

void lvba_lidar_default_opts(lvba_lidar_opts* o) {
  if (!o) return;
  o->u0 = 0.01; o->v0 = 2.0; o->max_iter = 10; o->rel_tol = 1e-6; o->device = -1; o->verbose = 0; o->deterministic = 0;
  o->pose_fixed = nullptr;
}

int lvba_lidar_create(int32_t W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx,
                      const double* clusters, const double* poses, int32_t device, lvba_lidar_problem** out) LVBA_ABI_BEGIN {
  return lvba::lidar_create_impl(W, V, vox_ptr, pose_idx, clusters, poses, device, out);
} LVBA_ABI_END("lvba_lidar_create")

int lvba_lidar_destroy(lvba_lidar_problem* p) LVBA_ABI_BEGIN {
  if (!p) return LVBA_OK;
  cudaSetDevice(p->device);
  delete p;
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_destroy")

int lvba_lidar_set_poses(lvba_lidar_problem* p, const double* poses) LVBA_ABI_BEGIN {
  if (!p || !poses) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_CUDA(cudaSetDevice(p->device));
  LVBA_TRY(p->poses.upload(poses, (size_t)p->W * 12, p->stream, &p->h2d));
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_set_poses")

int lvba_lidar_get_poses(lvba_lidar_problem* p, double* poses) LVBA_ABI_BEGIN {
  if (!p || !poses) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_CUDA(cudaSetDevice(p->device));
  LVBA_CUDA(cudaMemcpyAsync(poses, p->poses.p, (size_t)p->W * 12 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  p->d2h += (int64_t)p->W * 96;
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_get_poses")

int lvba_lidar_build(lvba_lidar_problem* p, double* residual_sum) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::lidar_check_usable(p));
  LVBA_CUDA(cudaSetDevice(p->device));
  LVBA_TRY(lvba::lidar_build_dev(p, p->poses.p, 0));
  LVBA_TRY(lvba::lidar_fetch_scal(p));
  if (residual_sum) *residual_sum = p->h_scal[0];
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_build")

int lvba_lidar_residual(lvba_lidar_problem* p, const double* poses, double* residual_sum) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::lidar_check_usable(p));
  LVBA_CUDA(cudaSetDevice(p->device));
  const double* dp = p->poses.p;
  if (poses) {
    LVBA_TRY(p->trial.upload(poses, (size_t)p->W * 12, p->stream, &p->h2d));
    dp = p->trial.p;
  }
  LVBA_TRY(lvba::lidar_residual_dev(p, dp, 3));
  LVBA_TRY(lvba::lidar_fetch_scal(p));
  if (residual_sum) *residual_sum = p->h_scal[3];
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_residual")

int lvba_lidar_solve(lvba_lidar_problem* p, double u, double* dx) LVBA_ABI_BEGIN {
  if (!p || !dx) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::lidar_check_usable(p));
  LVBA_CUDA(cudaSetDevice(p->device));
  LVBA_TRY(lvba::lidar_solve_dev(p, u));
  if (p->pose_fixed.empty()) {
    LVBA_CUDA(cudaMemcpyAsync(dx, p->dx.p, (size_t)p->W * 6 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    LVBA_TRY(lvba::lidar_fetch_scal(p));
  } else {                                                    // the rows' steps, zeros for the constant poses
    std::vector<double> dr((size_t)p->n_rows * 6);
    if (p->n_rows > 0) LVBA_CUDA(cudaMemcpyAsync(dr.data(), p->dx.p, dr.size() * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    LVBA_TRY(lvba::lidar_fetch_scal(p));
    std::fill(dx, dx + (size_t)p->W * 6, 0.0);
    for (int r = 0; r < p->n_rows; ++r) std::copy(dr.begin() + 6 * r, dr.begin() + 6 * r + 6, dx + 6 * (size_t)p->pose_of_row[r]);
  }
  p->d2h += (int64_t)p->n_rows * 48;
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_solve")

int lvba_lidar_rows(lvba_lidar_problem* p, int32_t* n_rows, int32_t* pose_of_row) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::lidar_check_usable(p));
  if (n_rows) *n_rows = p->n_rows;
  if (pose_of_row)
    for (int r = 0; r < p->n_rows; ++r) pose_of_row[r] = p->pose_fixed.empty() ? r : p->pose_of_row[r];
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_rows")

int lvba_lidar_structure(lvba_lidar_problem* p, int64_t* nblocks, int32_t* brow, int32_t* bcol) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::lidar_check_usable(p));
  if (nblocks) *nblocks = p->env.nblocks;
  if (brow && bcol) {
    for (int r = 0; r < p->env.n; ++r)
      for (int c = p->env.first[r]; c <= r; ++c) {
        const long long b = p->env.row_start[r] + (c - p->env.first[r]);
        brow[b] = r; bcol[b] = c;
      }
  }
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_structure")

int lvba_lidar_get_system(lvba_lidar_problem* p, double* g, double* blocks) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::lidar_check_usable(p));
  LVBA_CUDA(cudaSetDevice(p->device));
  if (g && p->n_rows > 0) LVBA_CUDA(cudaMemcpyAsync(g, p->g.p, (size_t)p->n_rows * 6 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  if (blocks && p->env.nblocks > 0) LVBA_CUDA(cudaMemcpyAsync(blocks, p->H.p, (size_t)p->env.nblocks * 36 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_get_system")

int lvba_lidar_reset_lm(lvba_lidar_problem* p, const lvba_lidar_opts* opts) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::lidar_check_usable(p));
  lvba_lidar_opts o;
  if (opts) o = *opts; else lvba_lidar_default_opts(&o);
  LVBA_TRY(lvba::lidar_set_mode(p, o));
  p->opts = o;
  p->lm.reset(o);
  p->is_calc_hess = true;
  p->builds = 0;
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_reset_lm")

int lvba_lidar_reset_state(lvba_lidar_problem* p) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_CUDA(cudaSetDevice(p->device));
  LVBA_CUDA(cudaMemcpyAsync(p->poses.p, p->poses0.p, (size_t)p->W * 12 * sizeof(double), cudaMemcpyDeviceToDevice, p->stream));
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_reset_state")

int lvba_lidar_iterate(lvba_lidar_problem* p, int32_t n_iter, lvba_summary* summary) LVBA_ABI_BEGIN {
  if (!p || n_iter < 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "bad argument");
  LVBA_TRY(lvba::lidar_check_usable(p));
  LVBA_CUDA(cudaSetDevice(p->device));
  return lvba::lidar_iterate_impl(p, n_iter, summary);
} LVBA_ABI_END("lvba_lidar_iterate")

int lvba_lidar_counts(lvba_lidar_problem* p, int64_t* nnz, int64_t* n_blocks_env, int64_t* n_blocks_nonzero, int64_t* n_pairs) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::lidar_check_usable(p));
  if (!p->have_structure) return lvba::fail(LVBA_ERR_UNSUPPORTED, "this problem was created without its host-side structure copy");
  if (nnz) *nnz = (int64_t)p->h_pose_idx_all.size();
  if (n_blocks_env) *n_blocks_env = p->env.nblocks;
  int64_t np = 0;
  std::unordered_set<uint64_t> seen;
  const bool want_nz = n_blocks_nonzero != nullptr;
  if (p->pose_fixed.empty()) {
    for (int64_t a = 0; a < p->V_total; ++a) {
      const int64_t lo = p->h_vox_ptr_all[a], hi = p->h_vox_ptr_all[a + 1];
      np += (hi - lo) * (hi - lo - 1) / 2;
      if (want_nz)
        for (int64_t x = lo; x < hi; ++x)
          for (int64_t y = x; y < hi; ++y)
            seen.insert(((uint64_t)p->h_pose_idx_all[x] << 32) | (uint32_t)p->h_pose_idx_all[y]);
    }
  } else {                                                    // the row system: pairs and blocks of free poses only
    std::vector<int> rows;
    for (int64_t a = 0; a < p->V_total; ++a) {
      rows.clear();
      for (int64_t x = p->h_vox_ptr_all[a]; x < p->h_vox_ptr_all[a + 1]; ++x)
        if (p->row_of[p->h_pose_idx_all[x]] >= 0) rows.push_back(p->row_of[p->h_pose_idx_all[x]]);
      const int64_t k = (int64_t)rows.size();
      np += k * (k - 1) / 2;
      if (want_nz)
        for (int64_t x = 0; x < k; ++x)
          for (int64_t y = x; y < k; ++y) seen.insert(((uint64_t)rows[x] << 32) | (uint32_t)rows[y]);
    }
  }
  if (n_pairs) *n_pairs = np;
  if (want_nz) *n_blocks_nonzero = (int64_t)seen.size();
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_counts")

int lvba_lidar_voxel_residuals(lvba_lidar_problem* p, const double* poses, double* lambda0) LVBA_ABI_BEGIN {
  if (!p || !lambda0) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::lidar_check_voxel_set(p));
  LVBA_CUDA(cudaSetDevice(p->device));
  const double* dp = p->poses.p;
  if (poses) {
    LVBA_TRY(p->trial.upload(poses, (size_t)p->W * 12, p->stream, &p->h2d));
    dp = p->trial.p;
  }
  LVBA_TRY(lvba::lidar_voxel_residuals_dev(p, dp));
  LVBA_CUDA(cudaMemcpyAsync(lambda0, p->d_vox_res.p, (size_t)p->V_total * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  p->d2h += p->V_total * 8;
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_voxel_residuals")

int lvba_lidar_remove_voxels(lvba_lidar_problem* p, const uint8_t* remove, int64_t* n_left) LVBA_ABI_BEGIN {
  if (!p || !remove) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::lidar_check_voxel_set(p));
  const int64_t V = p->V_total;
  const int64_t n_rm = std::count_if(remove, remove + V, [](uint8_t b) { return b != 0; });
  if (n_rm == V) return lvba::fail(LVBA_ERR_INVALID_ARG, "the removal would leave no voxel");
  LVBA_CUDA(cudaSetDevice(p->device));
  LVBA_TRY(lvba::lidar_remove_impl(p, remove));
  if (n_left) *n_left = p->V_total;
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_remove_voxels")

int lvba_lidar_remove_outliers(lvba_lidar_problem* p, double ratio, uint8_t* removed, int64_t* n_removed) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::lidar_check_voxel_set(p));
  const int64_t V = p->V_total;
  int64_t k_thr = 0, reject_num = 0;
  if (!lvba::outliers::rule_params(ratio, V, &k_thr, &reject_num))
    return lvba::fail(LVBA_ERR_INVALID_ARG, "ratio=%g: it must be finite, in [0, 1), with floor((1 - ratio) * %lld) >= 1", ratio, (long long)V);
  LVBA_CUDA(cudaSetDevice(p->device));
  LVBA_TRY(lvba::lidar_voxel_residuals_dev(p, p->poses.p));
  std::vector<uint8_t> mask((size_t)V);
  {
    lvba::CudaExec ex;
    ex.stream = p->stream;
    lvba::DevBuf<uint8_t> d_mask;
    LVBA_TRY(d_mask.alloc((size_t)V));
    lvba::outliers::RuleOut r;
    LVBA_TRY(lvba::outliers::remove_rule(ex, p->d_vox_res.p, V, ratio, d_mask.p, r));
    p->launches += ex.launches;
    if (r.non_finite) return lvba::fail(LVBA_ERR_INVALID_ARG, "a voxel's lambda_0 is not finite at the current poses: no outlier threshold");
    LVBA_TRY(ex.fetch(mask.data(), d_mask.p, (size_t)V));
    p->d2h += V + 24;
  }
  const int64_t n_rm = std::count_if(mask.begin(), mask.end(), [](uint8_t b) { return b != 0; });
  if (n_rm == V) return lvba::fail(LVBA_ERR_INVALID_ARG, "ratio=%g would remove every voxel (all lambda_0 at the threshold)", ratio);
  if (n_rm > 0) LVBA_TRY(lvba::lidar_remove_impl(p, mask.data()));
  else {                                                      // nothing to erase: the plan stays, the LM state is reset all the same
    p->lm.reset(p->opts);
    p->is_calc_hess = true;
    p->builds = 0;
  }
  if (removed) std::copy(mask.begin(), mask.end(), removed);
  if (n_removed) *n_removed = n_rm;
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_remove_outliers")

int lvba_lidar_lm(int32_t W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx, const double* clusters,
                  double* poses, const lvba_lidar_opts* opts, lvba_summary* summary) LVBA_ABI_BEGIN {
  const double t0 = lvba::wall_ms();
  lvba_lidar_opts o;
  if (opts) o = *opts; else lvba_lidar_default_opts(&o);
  lvba_lidar_problem* p = nullptr;
  LVBA_TRY(lvba::lidar_create_impl(W, V, vox_ptr, pose_idx, clusters, poses, o.device, &p, 0, nullptr, nullptr, /*keep_structure=*/false,
                                    o.pose_fixed));
  return lvba::lm_one_shot(p, o, V > 0, lvba_lidar_reset_lm, lvba_lidar_iterate, lvba_lidar_destroy,
                           [&] { return lvba_lidar_get_poses(p, poses); }, t0, summary);     // x_stats written back only on success
} LVBA_ABI_END("lvba_lidar_lm")

int lvba_lidar_lm_batch(int32_t n_windows, const int32_t* win_ptr, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx,
                        const double* clusters, double* poses, int32_t min_voxels_per_pose, const lvba_lidar_opts* opts,
                        lvba_summary* summaries, lvba_summary* total) LVBA_ABI_BEGIN {
  const double t0 = lvba::wall_ms();
  if (n_windows <= 0 || !win_ptr) return lvba::fail(LVBA_ERR_INVALID_ARG, "n_windows=%d must be positive and win_ptr non-null", n_windows);
  if (win_ptr[0] != 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "win_ptr[0] must be 0");
  for (int w = 0; w < n_windows; ++w)
    if (win_ptr[w + 1] < win_ptr[w]) return lvba::fail(LVBA_ERR_INVALID_ARG, "win_ptr must be non-decreasing");
  if (min_voxels_per_pose < 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "min_voxels_per_pose must be >= 0");
  lvba_lidar_opts o;
  if (opts) o = *opts; else lvba_lidar_default_opts(&o);
  lvba_lidar_problem* p = nullptr;
  LVBA_TRY(lvba::lidar_create_impl(win_ptr[n_windows], V, vox_ptr, pose_idx, clusters, poses, o.device, &p, n_windows, win_ptr, nullptr, true,
                                    o.pose_fixed));
  return lvba::lidar_batch_one_shot(p, o, min_voxels_per_pose, poses, summaries, total, t0, "lvba_lidar_lm_batch");
} LVBA_ABI_END("lvba_lidar_lm_batch")

}  // extern "C"
