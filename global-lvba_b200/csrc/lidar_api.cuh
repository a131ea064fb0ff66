// lidar_api.cuh — host side of boundary B1 (include/lvba_b200.h): symbolic set-up, device-resident
// problem handle and the damping_iter LM loop of reference include/BALM/bavoxel.hpp:662-767.
#pragma once
#include <cmath>
#include <unordered_set>

#include "runtime.cuh"   // (pulls comm.cuh in)
#include "balm_rule.h"
#include "exec.cuh"
#include "lidar.cuh"
#include "lidar_big.h"
#include "lidar_tiles.h"

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
  lvba::big::View big_view() const {
    return lvba::big::View{(int64_t)n_big, big_vox_ptr.p, big_pose.p, big_cl.p, big_pair_ptr.p, env.d_first.p, env.d_row_start.p};
  }

  lvba::LidarView view() const {
    lvba::LidarView v_;
    v_.W = W; v_.cl = cl.p; v_.nnz_pad = (long long)(cl.n / 5);
    v_.pidx = pidx.p; v_.vox_ptr = vox_ptr.p;
    v_.n_batches = n_batches; v_.batch_vox = batch_vox.p;
    v_.n_tiles = n_tiles; v_.tile_vox = tile_vox.p;
    v_.tile_prun = prun.tile_run.p; v_.prun_ptr = prun.run_ptr.p; v_.pairs = prun.code.p;
    v_.tile_drun = drun.tile_run.p; v_.drun_ptr = drun.run_ptr.p; v_.dslot = drun.code.p;
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

inline int lidar_create_impl(int32_t W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx,
                             const double* clusters, const double* poses, int32_t device,
                             lvba_lidar_problem** out, int32_t n_groups = 0, const int32_t* grp_ptr = nullptr,
                             const double* d_clusters = nullptr, bool keep_structure = true) {
  // keep_structure: copy the caller's CSR for lvba_lidar_counts (a handle may outlive the caller's arrays); the one-shot calls,
  // whose handle dies before they return, skip the 7 MB of copies
  // d_clusters: the same AoS records already resident on the selected device (a voxel map's export buffer); when set,
  // `clusters` may be null and no cluster bytes cross PCIe.
  if (!out) return fail(LVBA_ERR_INVALID_ARG, "out is null");
  *out = nullptr;
  const double t_val0 = wall_ms();
  LVBA_TRY(lidar_validate(W, V, vox_ptr, pose_idx, d_clusters ? d_clusters : clusters, poses));
  LVBA_TRY(select_device(device));
  const double t0 = wall_ms();
  const bool tlog = getenv("LVBA_SETUP_TIMING") != nullptr;
  double tprev = t0;
  auto lap = [&](const char* what) { if (tlog) { cudaStreamSynchronize(nullptr); const double t = wall_ms(); fprintf(stderr, "[lidar setup] %-22s %8.2f ms\n", what, t - tprev); tprev = t; } };
  if (tlog) fprintf(stderr, "[lidar setup] %-22s %8.2f ms\n", "validate", t0 - t_val0);
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

  // ---- envelope structure over ALL voxels (identical on every rank)
  std::vector<int> first_raw(W);
  for (int r = 0; r < W; ++r) first_raw[r] = r;
  {
    std::vector<int> first_w((size_t)kMaxSetupThreads * (size_t)W);
    for (int w = 0; w < kMaxSetupThreads; ++w) std::copy(first_raw.begin(), first_raw.end(), first_w.begin() + (size_t)w * (size_t)W);
    parallel_chunks(V, 1 << 14, [&](int64_t a0, int64_t a1, int w) {
      int* fr = first_w.data() + (size_t)w * (size_t)W;
      for (int64_t a = a0; a < a1; ++a) {
        const int m = pose_idx[vox_ptr[a]];
        for (int64_t q = vox_ptr[a]; q < vox_ptr[a + 1]; ++q) fr[pose_idx[q]] = std::min(fr[pose_idx[q]], m);
      }
    });
    for (int w = 0; w < kMaxSetupThreads; ++w)
      for (int r = 0; r < W; ++r) first_raw[r] = std::min(first_raw[r], first_w[(size_t)w * (size_t)W + r]);
  }
  LVBA_TRY(P->env.build(first_raw, s, &P->h2d));
  // ---- batched window BA: window of every pose, every voxel inside one window
  std::vector<int> pose_grp;
  if (n_groups > 0) {
    if (comm().active()) return fail(LVBA_ERR_UNSUPPORTED, "the batched window BA runs on one GPU per call (windows are independent: shard them across ranks)");
    P->n_groups = n_groups;
    P->grp_ptr.assign(grp_ptr, grp_ptr + n_groups + 1);
    pose_grp.resize((size_t)W);
    for (int g = 0; g < n_groups; ++g)
      for (int r = grp_ptr[g]; r < grp_ptr[g + 1]; ++r) pose_grp[r] = g;
    P->grp_V.assign((size_t)n_groups, 0);
    for (int64_t a = 0; a < V; ++a) {
      const int g = pose_grp[pose_idx[vox_ptr[a]]];
      if (pose_grp[pose_idx[vox_ptr[a + 1] - 1]] != g)
        return fail(LVBA_ERR_INVALID_ARG, "voxel %lld spans two windows", (long long)a);
      ++P->grp_V[g];
    }
  }
  LVBA_TRY(P->solver.prepare(P->env, s, LVBA_SOLVE_AUTO, 0, P->grp_ptr));     // grp_ptr empty: not batched
  lap("envelope+solver alloc");

  // ---- shard: voxel -> owner of its lowest pose index (SURVEY.md §8e)
  Comm& cm = comm();
  // the voxels this rank holds (all of them on one rank: `owned` stays empty and stands for 0..V-1)
  std::vector<int64_t> owned;
  const bool sharded = cm.active();
  if (sharded) {
    owned.reserve((size_t)V);
    for (int64_t a = 0; a < V; ++a)
      if ((P->solver.dist() ? P->solver.dist_owner(pose_idx[vox_ptr[a]]) : shard_owner(pose_idx[vox_ptr[a]], W, cm.n_ranks)) == cm.rank)
        owned.push_back(a);
  }
  // voxels seen from more than kSlots poses do not fit a batch CTA: they leave `owned` and take the passes of lidar_big.h
  std::vector<int64_t> bigv;
  {
    const int64_t n_own = sharded ? (int64_t)owned.size() : V;
    bool has_big = false;
    for (int64_t j = 0; j < n_own && !has_big; ++j) { const int64_t a = sharded ? owned[j] : j; has_big = vox_ptr[a + 1] - vox_ptr[a] > kSlots; }
    if (has_big) {
      std::vector<int64_t> small;
      for (int64_t j = 0; j < n_own; ++j) {
        const int64_t a = sharded ? owned[j] : j;
        (vox_ptr[a + 1] - vox_ptr[a] > kSlots ? bigv : small).push_back(a);
      }
      owned.swap(small);
    }
    // the batched window LM (lidar_batch_lm_impl) has no big-voxel passes: such a voxel would silently drop out of H, g and the
    // residual sums while still counting in the AVG_THR divisor.  A window holds <= 31 poses (EnvSolver::prepare), so this cannot
    // happen today; refuse loudly if that ever changes (ADVICE r1).
    if (n_groups > 0 && !bigv.empty())
      return fail(LVBA_ERR_UNSUPPORTED, "batched window BA: voxel %lld is seen from %lld poses (more than %d)", (long long)bigv[0],
                  (long long)(vox_ptr[bigv[0] + 1] - vox_ptr[bigv[0]]), kSlots);
  }
  const bool all = !sharded && bigv.empty();
  // voxels in the order of their lowest pose: the voxels of a build tile then share pose pairs, whose H blocks the tile sums on
  // chip (lidar_tiles.h); the windows of the batched window BA, consecutive pose ranges, come out contiguous and in order
  std::vector<int> slot0, l_vox_ptr;                           // first caller slot / first local slot of every local voxel
  const int64_t Vl = all ? V : (int64_t)owned.size();
  const long long nnz = tiles::order_by_lowest_pose(W, all ? nullptr : owned.data(), Vl, vox_ptr, pose_idx, slot0, l_vox_ptr);
  bool identity = all;                                         // the caller's voxels, in the caller's order
  long long np = 0;                                            // pose pairs
  for (int64_t i = 0; i < Vl; ++i) {
    const long long K = l_vox_ptr[i + 1] - l_vox_ptr[i];
    np += K * (K - 1) / 2;
    identity = identity && slot0[i] == l_vox_ptr[i];
  }
  P->V_local = Vl; P->nnz_local = nnz; P->n_pairs = np;

  // ---- residual batches (<= kSlots slots) and build tiles (<= kTileSlots slots): consecutive voxels, never across a window
  std::vector<int> vox_grp(n_groups > 0 ? (size_t)Vl : (size_t)0);
  for (int64_t i = 0; i < (int64_t)vox_grp.size(); ++i) vox_grp[i] = pose_grp[pose_idx[slot0[i]]];
  const int* grp = n_groups > 0 ? vox_grp.data() : nullptr;
  const std::vector<int> batch_vox = tiles::cut_ranges(Vl, l_vox_ptr.data(), grp, kSlots, kSlots);
  const std::vector<int> tile_vox = tiles::cut_ranges(Vl, l_vox_ptr.data(), grp, kTileSlots, kMaxVoxPerTile);
  P->n_batches = (int)batch_vox.size() - 1;
  P->n_tiles = (int)tile_vox.size() - 1;
  if (n_groups > 0) {
    auto per_window = [&](const std::vector<int>& cut) {      // range of batches / tiles of every window
      std::vector<int> r((size_t)n_groups + 1, 0);
      for (size_t k = 0; k + 1 < cut.size(); ++k) ++r[(size_t)vox_grp[cut[k]] + 1];
      for (int g = 0; g < n_groups; ++g) r[g + 1] += r[g];
      return r;
    };
    LVBA_TRY(P->d_grp_batch.upload(per_window(batch_vox), s, &P->h2d));
    LVBA_TRY(P->d_grp_tile.upload(per_window(tile_vox), s, &P->h2d));
    LVBA_TRY(P->d_grp_ptr.upload(P->grp_ptr, s, &P->h2d));
    LVBA_TRY(P->d_pose_grp.upload(pose_grp, s, &P->h2d));
    LVBA_TRY(P->d_accept.alloc((size_t)n_groups));
    LVBA_TRY(P->d_u_grp.alloc((size_t)n_groups));
    LVBA_TRY(P->d_grp_scal.alloc((size_t)4 * n_groups));
    LVBA_TRY(P->d_grp_scal.zero(s));
    P->h_grp_scal_bytes = (size_t)4 * n_groups * sizeof(double);
    LVBA_TRY(pinned_pool().take(P->h_grp_scal_bytes, (void**)&P->h_grp_scal));
    LVBA_CUDA(cudaStreamSynchronize(s));                       // local vectors
  }

  lap("order+batches+tiles");
  // ---- upload.  Clusters: the caller's AoS records go up in ONE copy and are transposed to the SoA double2 layout
  //      by a kernel (which also picks the slots in the local voxel order unless that is the caller's).
  const long long nnz_pad = ((nnz + 31) / 32) * 32 + 32;
  LVBA_TRY(P->cl.alloc((size_t)5 * nnz_pad));
  LVBA_TRY(P->cl.zero(s));
  LVBA_TRY(P->vox_ptr.upload(l_vox_ptr, s, &P->h2d));
  if (lane.done) LVBA_CUDA(cudaStreamWaitEvent(s, lane.done, 0));            // the kernels below read the records
  {
    if (identity) {
      if (nnz > 0) {
        lidar_aos_to_soa_kernel<<<(unsigned)((nnz + 255) / 256), 256, 0, s>>>(nnz, nnz_pad, aos_dev, P->cl.p);
        ++P->launches;
      }
    } else {
      // reordered (or a shard's scattered) voxels: the ONE copy of the caller's records and pose indices + a device-side gather
      DevBuf<int> d_slot0, d_caller_pidx;
      if (nnz > 0) {
        LVBA_TRY(d_slot0.upload(slot0, s, &P->h2d));
        LVBA_TRY(d_caller_pidx.upload(reinterpret_cast<const int*>(pose_idx), (size_t)vox_ptr[V], s, &P->h2d));
        LVBA_TRY(P->pidx.alloc((size_t)nnz));
        lidar_gather_slots_kernel<<<(unsigned)((nnz + 255) / 256), 256, 0, s>>>(nnz, nnz_pad, (int)Vl, P->vox_ptr.p, d_slot0.p, d_caller_pidx.p,
                                                                                aos_dev, P->pidx.p, P->cl.p);
        ++P->launches;
      }
      if (!bigv.empty()) {                   // the big voxels' records stay AoS (lidar_big.h reads them slot by slot)
        std::vector<int64_t> bvp{0}, bpp{0};
        std::vector<int32_t> bpose;
        std::vector<int> bsrc;
        for (int64_t a : bigv) {
          for (int64_t q = vox_ptr[a]; q < vox_ptr[a + 1]; ++q) { bsrc.push_back((int)q); bpose.push_back(pose_idx[q]); }
          const int64_t K = vox_ptr[a + 1] - vox_ptr[a];
          bvp.push_back((int64_t)bsrc.size());
          bpp.push_back(bpp.back() + K * (K - 1) / 2);
        }
        P->n_big = (long long)bigv.size(); P->n_big_slots = (long long)bsrc.size(); P->n_big_pairs = bpp.back();
        DevBuf<int> d_bsrc;
        LVBA_TRY(d_bsrc.upload(bsrc, s, &P->h2d));
        LVBA_TRY(P->big_vox_ptr.upload(bvp, s, &P->h2d));
        LVBA_TRY(P->big_pair_ptr.upload(bpp, s, &P->h2d));
        LVBA_TRY(P->big_pose.upload(bpose, s, &P->h2d));
        LVBA_TRY(P->big_cl.alloc((size_t)P->n_big_slots * 10));
        LVBA_TRY(P->big_params.alloc((size_t)P->n_big * big::kParams));
        LVBA_TRY(P->big_feat.alloc((size_t)P->n_big_slots * big::kFeat));
        lidar_gather_aos_kernel<<<(unsigned)((P->n_big_slots + 255) / 256), 256, 0, s>>>(P->n_big_slots, d_bsrc.p, aos_dev, P->big_cl.p);
        ++P->launches;
        LVBA_CUDA(cudaStreamSynchronize(s)); // the host vectors and d_bsrc go out of scope
      }
      LVBA_CUDA(cudaStreamSynchronize(s));   // d_slot0 and d_caller_pidx are freed on scope exit
    }
  }
  if (tlog) { cudaStreamSynchronize(s); } lap("cluster upload+SoA");
  static_assert(sizeof(int) == sizeof(int32_t), "pose_idx is uploaded as it is");
  if (identity) LVBA_TRY(P->pidx.upload(reinterpret_cast<const int*>(pose_idx), (size_t)nnz, s, &P->h2d));
  LVBA_TRY(P->batch_vox.upload(batch_vox, s, &P->h2d));
  LVBA_TRY(P->tile_vox.upload(tile_vox, s, &P->h2d));
  if (P->n_tiles > 0) {                                        // destination table of the build, on the device from the CSR just uploaded
    CudaExec ex;
    ex.stream = s;
    DevBuf<long long> d_pair_cnt, d_vox_pair;                  // pose pairs before every local voxel
    LVBA_TRY(d_pair_cnt.alloc((size_t)Vl + 1));
    LVBA_TRY(d_vox_pair.alloc((size_t)Vl + 1));
    LVBA_TRY(ex.for_each(Vl + 1, tiles::PairCountF{P->vox_ptr.p, Vl, d_pair_cnt.p}));
    LVBA_TRY(ex.exclusive_scan(d_pair_cnt.p, d_vox_pair.p, Vl + 1));
    const tiles::TableIn tin{P->n_tiles, W, P->env.nblocks, P->tile_vox.p, P->vox_ptr.p, P->pidx.p, d_vox_pair.p,
                             P->env.d_first.p, P->env.d_row_start.p};
    LVBA_TRY(tiles::build_runs(ex, tin, /*by_slot=*/false, np, P->prun));
    LVBA_TRY(tiles::build_runs(ex, tin, /*by_slot=*/true, nnz, P->drun));
    P->launches += ex.launches;
  }
  lap("destination table");
  LVBA_TRY(P->poses.upload(poses, (size_t)W * 12, s, &P->h2d));
  LVBA_TRY(P->poses0.upload(poses, (size_t)W * 12, s));
  LVBA_TRY(P->trial.alloc((size_t)W * 12));
  LVBA_TRY(P->H.alloc((size_t)P->env.nblocks * 36));
  LVBA_TRY(P->g.alloc((size_t)W * 6));
  LVBA_TRY(P->diag.alloc((size_t)W * 6));
  LVBA_TRY(P->dadd.alloc((size_t)W * 6));
  LVBA_TRY(P->dx.alloc((size_t)W * 6));
  LVBA_TRY(P->batch_res.alloc((size_t)std::max<long long>(std::max(P->n_batches, P->n_tiles) + P->n_big, 1)));
  LVBA_TRY(P->scal.alloc(8));
  LVBA_TRY(P->scal.zero(s));
  LVBA_CUDA(cudaFuncSetAttribute(lidar_build_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lidar_build_smem_bytes()));
  LVBA_CUDA(cudaStreamSynchronize(s));
  aos.release();                                               // the caller's records were consumed by the kernels above
  lap("index upload+allocs");
  lvba_lidar_default_opts(&P->opts);
  P->ms_setup = wall_ms() - t0;
  *out = P.release();
  return LVBA_OK;
}

// Deterministic mode: the records of the build and their destinations.  Records of H: the tiles' pair runs, the tiles' pose
// runs, the big voxels' slots, the big voxels' pairs; records of g: the tiles' pose runs, the big voxels' slots.  Each set in
// its enumeration order, so that every destination's records come in ascending (tile, run) order, then in item order.
inline int lidar_det_setup(lvba_lidar_problem* P) {
  if (P->det_ready) return LVBA_OK;
  const int64_t npr = P->prun.n_runs, ndr = P->drun.n_runs;
  const int64_t nH = npr + ndr + P->n_big_slots + P->n_big_pairs, ng = ndr + P->n_big_slots;
  if (nH >= (int64_t)1 << 32) return fail(LVBA_ERR_UNSUPPORTED, "deterministic mode: %lld contributions to H (at most 2^32)", (long long)nH);
  CudaExec ex;
  ex.stream = P->stream;
  LVBA_TRY(tiles::fixed_sum_alloc(P->det_H, nH, 36));
  LVBA_TRY(tiles::fixed_sum_alloc(P->det_g, ng, 6));
  if (P->n_tiles > 0) {
    const tiles::TableIn tin{P->n_tiles, P->W, P->env.nblocks, P->tile_vox.p, P->vox_ptr.p, P->pidx.p, nullptr,
                             P->env.d_first.p, P->env.d_row_start.p};
    LVBA_TRY(ex.for_each(npr, tiles::PairRunDstF{tin, P->prun.tile_run.p, P->prun.run_ptr.p, P->prun.code.p, P->det_H.dst.p}));
    LVBA_TRY(ex.for_each(ndr, tiles::SlotRunDstF{tin, P->drun.tile_run.p, P->drun.run_ptr.p, P->drun.code.p, P->det_H.dst.p + npr,
                                                 P->det_g.dst.p}));
  }
  if (P->n_big > 0) {
    const big::View bv = P->big_view();
    LVBA_TRY(ex.for_each(P->n_big_slots, big::SlotDstF{bv, P->det_H.dst.p + npr + ndr, P->det_g.dst.p + ndr}));
    LVBA_TRY(ex.for_each(P->n_big_pairs, big::PairDstF{bv, P->det_H.dst.p + npr + ndr + P->n_big_slots}));
  }
  LVBA_TRY(tiles::fixed_sum_index(ex, P->det_H, P->env.nblocks));
  LVBA_TRY(tiles::fixed_sum_index(ex, P->det_g, P->W));
  LVBA_CUDA(cudaFuncSetAttribute(lidar_build_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lidar_build_smem_bytes()));
  P->launches += ex.launches;
  P->det_ready = true;
  return LVBA_OK;
}

// the LM mode of the handle (lvba_lidar_reset_lm and the one-shot calls)
inline int lidar_set_mode(lvba_lidar_problem* P, const lvba_lidar_opts& o) {
  if (o.deterministic && comm().active())
    return fail(LVBA_ERR_UNSUPPORTED, "deterministic mode runs on one GPU: the multi-GPU sums of NCCL have no fixed order");
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
    if (P->det)
      lidar_build_kernel<true><<<P->n_tiles, kTileSlots, lidar_build_smem_bytes(), s>>>(P->view(), P->env.view(), d_poses, P->det_H.rec.p,
                                                                                         P->det_g.rec.p, P->batch_res.p);
    else
      lidar_build_kernel<false><<<P->n_tiles, kTileSlots, lidar_build_smem_bytes(), s>>>(P->view(), P->env.view(), d_poses, P->H.p, P->g.p,
                                                                                          P->batch_res.p);
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
    lidar_residual_kernel<<<P->n_batches, kSlots, 0, s>>>(P->view(), d_poses, P->batch_res.p);
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

// (H + u diag(H)) dx = -g ; q1 ; leaves dx on the device.  scal[1] = q1, scal[2] = non-finite flag
inline int lidar_solve_dev(lvba_lidar_problem* P, double u) {
  cudaStream_t s = P->stream;
  const int n6 = 6 * P->W;
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
  LVBA_CUDA(cudaMemcpyAsync(P->h_scal + 7, P->solver.status.p, sizeof(int), cudaMemcpyDeviceToHost, P->stream));
  LVBA_CUDA(cudaStreamSynchronize(P->stream));
  P->d2h += 8 * sizeof(double) + sizeof(int);
  return LVBA_OK;
}

// n passes of the damping_iter loop body (bavoxel.hpp:686-766)
inline int lidar_iterate_impl(lvba_lidar_problem* P, int n_iter, lvba_summary* sum) {
  const double t0 = wall_ms();
  const int64_t l0 = P->launches, h0 = P->h2d, d0 = P->d2h;
  const double V = (double)P->V_total;
  BalmState& lm = P->lm;
  const int iters0 = lm.iters, acc0 = lm.accepted, builds0 = P->builds;
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
    lidar_retract_kernel<<<(P->W + 127) / 128, 128, 0, P->stream>>>(P->W, P->poses.p, P->dx.p, P->trial.p);   // :722-727
    ++P->launches;
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
  for (int g = 0; g < G; ++g) {
    const int Wg = P->grp_ptr[g + 1] - P->grp_ptr[g];
    WinState& w = ws[g];
    w.reset(P->opts);
    w.skipped = Wg <= 0 || P->grp_V[g] == 0 || P->grp_V[g] < (long long)min_voxels_per_pose * Wg;   // src/lvba_system.cpp:262-266
    w.active = !w.skipped;
    if (w.skipped) w.term = LVBA_TERM_SKIPPED;
    n_active += w.active;
  }
  const int n6 = 6 * P->W;
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
    lidar_rhs_grouped_kernel<<<(n6 + 255) / 256, 256, 0, s>>>(n6, P->g.p, P->diag.p, P->d_u_grp.p, P->d_pose_grp.p, P->solver.z.p, P->dadd.p);
    P->launches += 2;
    LVBA_TRY(P->solver.solve(P->env, P->H.p, P->dadd.p, P->dx.p, s, &P->launches));
    lidar_q1_grouped_kernel<<<G, 128, 0, s>>>(P->d_grp_ptr.p, P->dx.p, P->diag.p, P->g.p, P->d_u_grp.p, P->solver.status.p, P->d_grp_scal.p);
    ++P->launches;
    P->timers.end();
    // ---- trial state and its residual per window
    P->timers.begin(PH_RESID);
    lidar_retract_kernel<<<(P->W + 127) / 128, 128, 0, s>>>(P->W, P->poses.p, P->dx.p, P->trial.p);
    ++P->launches;
    if (P->n_batches > 0) {
      lidar_residual_kernel<<<P->n_batches, kSlots, 0, s>>>(P->view(), P->trial.p, P->batch_res.p);
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
}

int lvba_lidar_create(int32_t W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx,
                      const double* clusters, const double* poses, int32_t device, lvba_lidar_problem** out) {
  try { return lvba::lidar_create_impl(W, V, vox_ptr, pose_idx, clusters, poses, device, out); }
  catch (const std::bad_alloc&) { return lvba::fail(LVBA_ERR_NOMEM, "host allocation failed"); }
  catch (...) { return lvba::fail(LVBA_ERR_INVALID_ARG, "unexpected exception in lvba_lidar_create"); }
}

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
  LVBA_CUDA(cudaSetDevice(p->device));
  LVBA_TRY(lvba::lidar_build_dev(p, p->poses.p, 0));
  LVBA_TRY(lvba::lidar_fetch_scal(p));
  if (residual_sum) *residual_sum = p->h_scal[0];
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_build")

int lvba_lidar_residual(lvba_lidar_problem* p, const double* poses, double* residual_sum) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
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
  LVBA_CUDA(cudaSetDevice(p->device));
  LVBA_TRY(lvba::lidar_solve_dev(p, u));
  LVBA_CUDA(cudaMemcpyAsync(dx, p->dx.p, (size_t)p->W * 6 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  LVBA_TRY(lvba::lidar_fetch_scal(p));
  p->d2h += (int64_t)p->W * 48;
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_solve")

int lvba_lidar_structure(lvba_lidar_problem* p, int64_t* nblocks, int32_t* brow, int32_t* bcol) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
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
  LVBA_CUDA(cudaSetDevice(p->device));
  if (g) LVBA_CUDA(cudaMemcpyAsync(g, p->g.p, (size_t)p->W * 6 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  if (blocks) LVBA_CUDA(cudaMemcpyAsync(blocks, p->H.p, (size_t)p->env.nblocks * 36 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_get_system")

int lvba_lidar_reset_lm(lvba_lidar_problem* p, const lvba_lidar_opts* opts) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
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
  LVBA_CUDA(cudaSetDevice(p->device));
  return lvba::lidar_iterate_impl(p, n_iter, summary);
} LVBA_ABI_END("lvba_lidar_iterate")

int lvba_lidar_counts(lvba_lidar_problem* p, int64_t* nnz, int64_t* n_blocks_env, int64_t* n_blocks_nonzero, int64_t* n_pairs) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  if (!p->have_structure) return lvba::fail(LVBA_ERR_UNSUPPORTED, "this problem was created without its host-side structure copy");
  if (nnz) *nnz = (int64_t)p->h_pose_idx_all.size();
  if (n_blocks_env) *n_blocks_env = p->env.nblocks;
  int64_t np = 0;
  std::unordered_set<uint64_t> seen;
  const bool want_nz = n_blocks_nonzero != nullptr;
  for (int64_t a = 0; a < p->V_total; ++a) {
    const int64_t lo = p->h_vox_ptr_all[a], hi = p->h_vox_ptr_all[a + 1];
    np += (hi - lo) * (hi - lo - 1) / 2;
    if (want_nz)
      for (int64_t x = lo; x < hi; ++x)
        for (int64_t y = x; y < hi; ++y)
          seen.insert(((uint64_t)p->h_pose_idx_all[x] << 32) | (uint32_t)p->h_pose_idx_all[y]);
  }
  if (n_pairs) *n_pairs = np;
  if (want_nz) *n_blocks_nonzero = (int64_t)seen.size();
  return LVBA_OK;
} LVBA_ABI_END("lvba_lidar_counts")

int lvba_lidar_lm(int32_t W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx, const double* clusters,
                  double* poses, const lvba_lidar_opts* opts, lvba_summary* summary) {
  const double t0 = lvba::wall_ms();
  lvba_lidar_opts o;
  if (opts) o = *opts; else lvba_lidar_default_opts(&o);
  lvba_lidar_problem* p = nullptr;
  int rc;
  try { rc = lvba::lidar_create_impl(W, V, vox_ptr, pose_idx, clusters, poses, o.device, &p, 0, nullptr, nullptr, /*keep_structure=*/false); }
  catch (const std::bad_alloc&) { return lvba::fail(LVBA_ERR_NOMEM, "host allocation failed"); }
  catch (...) { return lvba::fail(LVBA_ERR_INVALID_ARG, "unexpected exception in lvba_lidar_lm"); }
  if (rc != LVBA_OK) return rc;
  return lvba::lm_one_shot(p, o, V > 0, lvba_lidar_reset_lm, lvba_lidar_iterate, lvba_lidar_destroy,
                           [&] { return lvba_lidar_get_poses(p, poses); }, t0, summary);     // x_stats written back only on success
}

int lvba_lidar_lm_batch(int32_t n_windows, const int32_t* win_ptr, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx,
                        const double* clusters, double* poses, int32_t min_voxels_per_pose, const lvba_lidar_opts* opts,
                        lvba_summary* summaries, lvba_summary* total) {
  const double t0 = lvba::wall_ms();
  if (n_windows <= 0 || !win_ptr) return lvba::fail(LVBA_ERR_INVALID_ARG, "n_windows=%d must be positive and win_ptr non-null", n_windows);
  if (win_ptr[0] != 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "win_ptr[0] must be 0");
  for (int w = 0; w < n_windows; ++w)
    if (win_ptr[w + 1] < win_ptr[w]) return lvba::fail(LVBA_ERR_INVALID_ARG, "win_ptr must be non-decreasing");
  if (min_voxels_per_pose < 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "min_voxels_per_pose must be >= 0");
  lvba_lidar_opts o;
  if (opts) o = *opts; else lvba_lidar_default_opts(&o);
  lvba_lidar_problem* p = nullptr;
  int rc;
  try { rc = lvba::lidar_create_impl(win_ptr[n_windows], V, vox_ptr, pose_idx, clusters, poses, o.device, &p, n_windows, win_ptr); }
  catch (const std::bad_alloc&) { return lvba::fail(LVBA_ERR_NOMEM, "host allocation failed"); }
  catch (...) { return lvba::fail(LVBA_ERR_INVALID_ARG, "unexpected exception in lvba_lidar_lm_batch"); }
  if (rc != LVBA_OK) return rc;
  return lvba::lidar_batch_one_shot(p, o, min_voxels_per_pose, poses, summaries, total, t0, "lvba_lidar_lm_batch");
}

}  // extern "C"
