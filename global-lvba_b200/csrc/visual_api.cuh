// visual_api.cuh — host side of boundary B2 (include/lvba_b200.h): problem set-up mirroring the Ceres
// problem built at reference src/lvba_system.cpp:1578-1640 and the trust-region LM loop of
// ceres-solver 2.1.0 (TrustRegionMinimizer + LevenbergMarquardtStrategy, SURVEY.md Q10/A.3).
#pragma once
#include <cmath>
#include <memory>

#include "exec.cuh"
#include "runtime.cuh"   // (pulls comm.cuh in)
#include "visual.cuh"
#include "visual_outliers.h"
#include "visual_plan.h"

namespace lvba {
// the trust-region state of one solve (Ceres TrustRegionMinimizer + LevenbergMarquardtStrategy)
struct TrustRegionState {
  double radius = 1e4, nu = 2.0, cost = 0.0, cost_first = 0.0;
  bool have_scale = false, have_first = false, converged = false;
  int iters = 0, accepted = 0, builds = 0, invalid = 0, termination = LVBA_TERM_MAX_ITER;
  // a new solve from the options; cost and cost_first keep their values until its first pass sets them
  void reset(const lvba_visual_opts& o) {
    radius = o.initial_radius; nu = 2.0;
    have_scale = have_first = converged = false;
    iters = accepted = builds = invalid = 0; termination = LVBA_TERM_MAX_ITER;
  }
};
}  // namespace lvba

struct lvba_visual_problem {
  int M = 0;
  long long T = 0, Tv = 0, nnz = 0, n_pairs = 0;
  int n_rows = 0, n_batches = 0, n_tiles = 0, device = 0, fixed_cam = 0;
  std::vector<int> cam_of_row;
  std::vector<uint8_t> cam_fixed;                   // constant cameras of the plan besides fixed_cam (lvba_visual_opts::cam_fixed,
                                                    // one 0 / 1 per camera); empty: none
  bool unusable = false;                            // a re-plan failed and so did restoring the previous one (visual_replan)
  cudaStream_t stream = nullptr;
  double intr[8];
  double sigma_px = 1, sigma_pl = 1;
  lvba::DevBuf<int> trk_ptr, trk_id, batch_trk, tile_trk, obs_cam, obs_row, d_cam_of_row;
  lvba::tiles::Runs<lvba::CudaExec> prun, drun;   // the build's destination table: pair contributions by S block, observations by row
  lvba::DevBuf<float2> obs_uv;
  lvba::DevBuf<double> plane;
  lvba::DevBuf<double> q, t, X, qc, tc, Xc;         // state and candidate
  lvba::DevBuf<double> q0, t0, X0;                  // state given at create (lvba_visual_reset_state)
  lvba::DevBuf<double> S, rhs, y, dadd, cam_colsq, cam_grad, s_cam, s_pt, pt_colsq;
  lvba::DevBuf<double> batch_cost, batch_gmax, batch_out, cam_out, scal, cam_step, pt_step;
  lvba::Envelope env;
  lvba::EnvSolver solver;
  // landmarks with more than kSlots observations: local landmarks [Tv_small, Tv), outside the tiles and batches, through the
  // passes of visual_big.h
  long long Tv_small = 0, n_big = 0, n_big_obs = 0, n_big_pairs = 0;
  lvba::DevBuf<int64_t> big_pair_ptr;
  lvba::DevBuf<double> big_obs, big_params;
  // ---- deterministic mode (lvba_visual_opts::deterministic): the records of every contribution to S and to the camera rows
  // (rhs | column norms | gradient, and the column norms of the scale pass, which share the rows' records and order), set up
  // when a reset first asks for the mode (visual_det_setup)
  bool det = false, det_ready = false;
  lvba::tiles::FixedSum<lvba::CudaExec> det_S, det_G;
  lvba::DevBuf<double> det_C;                       // [det_G.n_rec][6] records of the column-norm pass
  // ---- robust losses (lvba_visual_opts::reproj_loss / plane_loss), set by lvba_visual_reset_lm; with either one the passes
  // run their kLoss instantiations
  int loss_px = LVBA_LOSS_NONE, loss_pl = LVBA_LOSS_NONE;
  double loss_a_px = 1.0, loss_a_pl = 0.1;
  bool robust() const { return loss_px != LVBA_LOSS_NONE || loss_pl != LVBA_LOSS_NONE; }
  // ---- the intrinsics block (lvba_visual_opts::refine_intrinsics, set by lvba_visual_reset_lm; visual_intr.h).  The kernels take
  // the intrinsics by value in VisualView, so the handle keeps them on the host: intr above is the current value, intr_c the
  // candidate of the last pass (intr + intr_step), intr0 the value given at create.  The row CSR of the border gather
  // (intr_row_ptr / intr_row_obs, the observations of every camera row in ascending order) follows the plan: visual_plan clears
  // intr_ready and the next pass with the block builds it again.
  uint32_t intr_mask = 0;
  double intr0[8], intr_c[8], intr_step[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  bool intr_ready = false;
  bool intr_have_sys = false;                       // intr_B / intr_sys / intr_step hold the block of the last pass since the last reset
  lvba::DevBuf<int64_t> intr_row_ptr, intr_row_obs;
  lvba::DevBuf<double> intr_slot, intr_rec, intr_part, intr_sys, intr_B, intr_Y, intr_dev;   // intr_dev: sk | colsq | y_k | dk
  lvba::PhaseTimers timers;
  double* h_scal = nullptr;
  int64_t launches = 0, h2d = 0, d2h = 0;
  double ms_setup = 0.0;
  // ---- per-observation calls (visual_outliers.h): the caller's observation CSR as given at create (T + 1 offsets), the caller
  // index of every local observation (obs_src, derived when a call first needs it; once it exists every re-plan carries it
  // along, since after a removal it can no longer be derived), and the caller-indexed s_q of lvba_visual_obs_residuals
  std::vector<int64_t> h_obs_ptr;
  lvba::DevBuf<int64_t> obs_src;
  bool obs_src_ready = false;
  lvba::DevBuf<double> obs_sq;
  // LM state
  lvba_visual_opts opts;
  lvba::TrustRegionState lm;

  lvba::VisualView view() const {
    lvba::VisualView v;
    v.n_batches = n_batches; v.batch_trk = batch_trk.p; v.n_tiles = n_tiles; v.tile_trk = tile_trk.p;
    v.tile_prun = prun.tile_run.p; v.prun_ptr = prun.run_ptr.p; v.pairs = prun.code.p;
    v.tile_drun = drun.tile_run.p; v.drun_ptr = drun.run_ptr.p; v.dslot = drun.code.p;
    v.trk_ptr = trk_ptr.p; v.trk_id = trk_id.p; v.obs_cam = obs_cam.p; v.obs_row = obs_row.p;
    v.obs_uv = obs_uv.p; v.plane = plane.p;
    for (int i = 0; i < 8; ++i) v.intr[i] = intr[i];
    v.inv_sigma_px = 1.0 / sigma_px;
    v.inv_sigma_pl = 1.0 / std::max(1e-9, sigma_pl);        // utils.hpp:131
    v.loss_px = loss_px; v.loss_pl = loss_pl; v.loss_a_px = loss_a_px; v.loss_a_pl = loss_a_pl;
    return v;
  }
  // the tiles' CSR for the passes of visual_tiles.h (trk_pair: set by visual_tables)
  lvba::tiles::VisTableIn table_in() const {
    return lvba::tiles::VisTableIn{n_tiles, n_rows, env.nblocks, tile_trk.p, trk_ptr.p, obs_row.p, nullptr, env.d_first.p, env.d_row_start.p};
  }
  lvba::vbig::View big_view() const { return lvba::vbig::View{(int64_t)n_big, (int64_t)Tv_small, big_pair_ptr.p, env.d_first.p, env.d_row_start.p}; }
  lvba::VisualState state() const { return lvba::VisualState{q.p, t.p, X.p}; }
  lvba::VisualState cand() const { return lvba::VisualState{qc.p, tc.p, Xc.p}; }
  ~lvba_visual_problem() {
    if (stream) { cudaStreamSynchronize(stream); cudaStreamDestroy(stream); }     // buffers (members) must be idle when parked
    lvba::pinned_pool().give(h_scal, 16 * sizeof(double));                         // after the drain
  }
};

namespace lvba {

// ---- set-up kernel: the per-observation arrays are derived on the device from the caller's arrays (uploaded as they are: one
// DMA each from the caller's — ideally pinned — memory) instead of being gathered on the host and pushed through pageable
// staging copies (config C: 16 MB of observations).
// One thread per local landmark k (source landmark trk_id[k]): its observations, camera rows and plane.
__global__ void visual_gather_kernel(long long Tv, const int* __restrict__ trk_id, const int* __restrict__ trk_ptr,
                                     const long long* __restrict__ obs_ptr, const int* __restrict__ raw_cam,
                                     const float2* __restrict__ raw_uv, const double* __restrict__ raw_plane,
                                     const int* __restrict__ row_of_cam, int* __restrict__ l_cam, int* __restrict__ l_row,
                                     float2* __restrict__ l_uv, double* __restrict__ l_plane) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= Tv) return;
  const long long i = trk_id[k];
#pragma unroll
  for (int j = 0; j < 4; ++j) l_plane[4 * k + j] = raw_plane[4 * i + j];
  long long w = trk_ptr[k];
  for (long long q = obs_ptr[i]; q < obs_ptr[i + 1]; ++q, ++w) {
    const int c = raw_cam[q];
    l_cam[w] = c; l_row[w] = row_of_cam[c]; l_uv[w] = raw_uv[q];
  }
}

// The constant cameras of lvba_visual_opts::cam_fixed as the handle keeps them: one 0 / 1 per camera, empty when no entry is
// nonzero (an all-zero mask is no mask)
inline std::vector<uint8_t> visual_mask(int M, const uint8_t* cam_fixed) {
  std::vector<uint8_t> m;
  if (!cam_fixed) return m;
  bool any = false;
  for (int c = 0; c < M && !any; ++c) any = cam_fixed[c] != 0;
  if (!any) return m;
  m.resize((size_t)M);
  for (int c = 0; c < M; ++c) m[c] = cam_fixed[c] ? 1 : 0;
  return m;
}

// The device arrays visual_plan gathers the per-observation arrays from, indexed by source landmark
struct VisualSrc {
  const long long* obs_ptr = nullptr;
  const int* cam = nullptr;
  const float2* uv = nullptr;
  const double* plane = nullptr;
  const int64_t* obs_src = nullptr;    // the caller index of every source observation, gathered into P->obs_src; null: none yet
};

// Everything the handle derives from its system rows (row_of_cam and P->cam_of_row): the envelope and the solver path, the
// shard, the landmark layout with its batches and tiles, the per-observation arrays, the destination table, the buffers of the
// big landmarks and the row-sized buffers.  valid: the source landmarks with a usable plane, in ascending order of the caller's
// landmark; obs_ptr / obs_cam: the host CSR of the source landmarks; src_id: the caller's landmark of every source landmark
// (null: the source landmarks are the caller's).  get_src(VisualSrc&) provides the device arrays once there are landmarks to
// gather.  visual_create_impl plans from the caller's arrays, visual_replan from the handle's own.
template <class GetSrc>
inline int visual_plan(lvba_visual_problem* P, const std::vector<int64_t>& valid, const int64_t* obs_ptr, const int32_t* obs_cam,
                       const std::vector<int>& row_of_cam, const int* src_id, const GetSrc& get_src, SetupLaps& lap) {
  cudaStream_t s = P->stream;
  P->n_rows = (int)P->cam_of_row.size();
  P->intr_ready = false;
  P->intr_have_sys = false;
  const int64_t Tv_all = (int64_t)valid.size();
  DevBuf<int> d_row_of_cam, d_src_trk;

  // ---- envelope of the reduced camera system over ALL valid landmarks
  std::vector<int> min_row, min_sys_row;     // shard key: lowest camera; row-owned reduced system: lowest row of the clique
  std::vector<int> first_raw = visual_first_rows(P->n_rows, valid.data(), Tv_all, obs_ptr, obs_cam, row_of_cam.data(), min_row, min_sys_row);
  if (P->n_rows > 0) {
    first_raw.resize(P->n_rows);
    LVBA_TRY(P->env.build(first_raw, s, &P->h2d));
    LVBA_TRY(P->solver.prepare(P->env, s));
  } else {                                   // every camera constant (or unseen): no reduced system
    Envelope& e = P->env;
    e.n = 0; e.nblocks = 0; e.max_col = 0;
    e.first.clear(); e.last.clear(); e.row_start.clear();
    e.d_first.release(); e.d_last.release(); e.d_row_start.release();
  }

  lap("envelope + solver prepare");
  // ---- shard (SURVEY.md §8e): landmark -> owner of its lowest camera index
  Comm& cm = comm();
  std::vector<int64_t> own;                                    // indices into valid
  if (cm.active())
    for (int64_t k = 0; k < Tv_all; ++k)
      if ((P->solver.dist() ? P->solver.dist_owner(min_sys_row[k]) : shard_owner(min_row[k], P->M, cm.n_ranks)) == cm.rank) own.push_back(k);
  VisualLayout L;                                              // landmark order and list, batches and tiles
  visual_layout(P->n_rows, valid.data(), Tv_all, cm.active() ? &own : nullptr, min_sys_row.data(), obs_ptr, obs_cam, row_of_cam.data(), L);
  const int64_t Tv = L.Tv, Tv_small = L.Tv_small;
  P->Tv = Tv;
  P->Tv_small = Tv_small;
  P->n_big = Tv - Tv_small;
  P->nnz = L.nnz;
  lap("landmark list");
  P->n_batches = (int)L.batch_trk.size() - 1;
  P->n_tiles = (int)L.tile_trk.size() - 1;
  lap("batches + tiles");

  // ---- gather the per-observation arrays and build the destination table on the device
  LVBA_TRY(P->trk_ptr.upload(L.trk_ptr, s, &P->h2d));
  LVBA_TRY(P->batch_trk.upload(L.batch_trk, s, &P->h2d));
  LVBA_TRY(P->tile_trk.upload(L.tile_trk, s, &P->h2d));
  P->n_pairs = 0;
  P->obs_src.release();
  P->obs_src_ready = false;
  if (Tv > 0) {
    VisualSrc src;
    LVBA_TRY(get_src(src));
    LVBA_TRY(d_row_of_cam.upload(row_of_cam, s, &P->h2d));
    if (src_id) {                                              // the kernels index the state by the caller's landmark
      std::vector<int> id(L.trk_id.size());
      for (size_t k = 0; k < id.size(); ++k) id[k] = src_id[L.trk_id[k]];
      LVBA_TRY(d_src_trk.upload(L.trk_id, s, &P->h2d));
      LVBA_TRY(P->trk_id.upload(id, s, &P->h2d));
    } else {
      LVBA_TRY(P->trk_id.upload(L.trk_id, s, &P->h2d));
    }
    LVBA_TRY(P->obs_cam.alloc((size_t)P->nnz)); LVBA_TRY(P->obs_row.alloc((size_t)P->nnz)); LVBA_TRY(P->obs_uv.alloc((size_t)P->nnz));
    LVBA_TRY(P->plane.alloc((size_t)Tv * 4));
    visual_gather_kernel<<<(unsigned)((Tv + 127) / 128), 128, 0, s>>>(Tv, src_id ? d_src_trk.p : P->trk_id.p, P->trk_ptr.p, src.obs_ptr, src.cam,
                                                                     src.uv, src.plane, d_row_of_cam.p, P->obs_cam.p, P->obs_row.p, P->obs_uv.p,
                                                                     P->plane.p);
    LVBA_CUDA(cudaGetLastError());
    ++P->launches;
    CudaExec ex;                                               // the destination table covers the small landmarks only
    ex.stream = s;
    if (src.obs_src) {
      LVBA_TRY(P->obs_src.alloc((size_t)P->nnz));
      LVBA_TRY(ex.for_each(Tv, voutliers::GatherSrcF{src_id ? d_src_trk.p : P->trk_id.p, P->trk_ptr.p, src.obs_ptr, src.obs_src, P->obs_src.p}));
      P->obs_src_ready = true;
    }
    int64_t np = 0;
    LVBA_TRY(visual_tables(ex, P->table_in(), Tv_small, L.n_ordered, L.trk_ptr[Tv_small], P->prun, P->drun, &np));
    P->launches += ex.launches;
    P->n_pairs = np + L.big_pairs;
    if (P->n_big > 0) {
      P->n_big_obs = P->nnz - L.trk_ptr[Tv_small];
      P->n_big_pairs = L.big_pair_ptr.back();
      LVBA_TRY(P->big_pair_ptr.upload(L.big_pair_ptr, s, &P->h2d));
      LVBA_TRY(P->big_obs.alloc((size_t)P->n_big_obs * vbig::kObs));
      LVBA_TRY(P->big_params.alloc((size_t)P->n_big * kTrkParams));
    }
  }
  lap("device gather + destination table");
  if (P->n_rows > 0) LVBA_TRY(P->d_cam_of_row.upload(P->cam_of_row, s, &P->h2d));
  const size_t n6 = (size_t)std::max(P->n_rows, 1) * 6;
  LVBA_TRY(P->S.alloc((size_t)std::max<long long>(P->env.nblocks, 1) * 36));
  LVBA_TRY(P->rhs.alloc(n6)); LVBA_TRY(P->y.alloc(n6)); LVBA_TRY(P->dadd.alloc(n6));
  LVBA_TRY(P->cam_colsq.alloc(n6)); LVBA_TRY(P->cam_grad.alloc(n6)); LVBA_TRY(P->s_cam.alloc(n6));
  LVBA_TRY(P->s_pt.alloc((size_t)std::max<int64_t>(Tv, 1) * 3));
  LVBA_TRY(P->pt_colsq.alloc((size_t)std::max<int64_t>(Tv, 1) * 3));
  const size_t nb = (size_t)std::max<long long>(std::max(P->n_batches, P->n_tiles) + P->n_big, 1);   // partial slots, big landmarks last
  LVBA_TRY(P->batch_cost.alloc(nb)); LVBA_TRY(P->batch_gmax.alloc(nb)); LVBA_TRY(P->batch_out.alloc(nb * 4));
  LVBA_TRY(P->cam_out.alloc((size_t)((P->n_rows + 127) / 128 + 1) * 2));
  LVBA_CUDA(cudaStreamSynchronize(s));                         // the temporaries above are idle before they are parked
  return LVBA_OK;
}

inline int visual_create_impl(int32_t M, int64_t T, const double* q, const double* t, const double* X,
                              const double* plane_nd, const int64_t* obs_ptr, const int32_t* obs_cam,
                              const float* obs_uv, const double intr[8], double sigma_px, double sigma_plane,
                              int32_t fixed_cam, const uint8_t* cam_fixed, int32_t device, lvba_visual_problem** out) {
  if (!out) return fail(LVBA_ERR_INVALID_ARG, "out is null");
  *out = nullptr;
  if (M <= 0 || T < 0) return fail(LVBA_ERR_INVALID_ARG, "M=%d T=%lld", M, (long long)T);
  if (!q || !t || !intr || !obs_ptr || (T > 0 && (!X || !plane_nd || !obs_cam || !obs_uv))) return fail(LVBA_ERR_INVALID_ARG, "null input pointer");
  if (!(sigma_px > 0)) return fail(LVBA_ERR_INVALID_ARG, "sigma_px must be positive");
  if (obs_ptr[0] != 0) return fail(LVBA_ERR_INVALID_ARG, "obs_ptr[0] must be 0");
  {
    int64_t bad_i[kMaxSetupThreads], bad_s[kMaxSetupThreads];
    for (int w = 0; w < kMaxSetupThreads; ++w) { bad_i[w] = -1; bad_s[w] = -1; }
    parallel_chunks(T, 1 << 14, [&](int64_t i0, int64_t i1, int w) {
      for (int64_t i = i0; i < i1; ++i) {
        if (obs_ptr[i + 1] < obs_ptr[i]) { bad_i[w] = i; return; }
        for (int64_t s = obs_ptr[i]; s < obs_ptr[i + 1]; ++s)
          if (obs_cam[s] < 0 || obs_cam[s] >= M) { bad_i[w] = i; bad_s[w] = s; return; }
      }
    });
    for (int w = 0; w < kMaxSetupThreads; ++w) {
      if (bad_i[w] < 0) continue;
      if (bad_s[w] < 0) return fail(LVBA_ERR_INVALID_ARG, "obs_ptr not monotone at %lld", (long long)bad_i[w]);
      return fail(LVBA_ERR_INVALID_ARG, "obs_cam[%lld]=%d out of [0,%d)", (long long)bad_s[w], obs_cam[bad_s[w]], M);
    }
  }
  LVBA_TRY(select_device(device));
  const double t_begin = wall_ms();
  SetupLaps lap("visual setup", 26, nullptr, t_begin);
  std::unique_ptr<lvba_visual_problem> P(new lvba_visual_problem());
  P->M = M; P->T = T; P->fixed_cam = fixed_cam;
  P->cam_fixed = visual_mask(M, cam_fixed);
  for (int i = 0; i < 8; ++i) P->intr[i] = P->intr0[i] = P->intr_c[i] = intr[i];
  P->sigma_px = sigma_px; P->sigma_pl = sigma_plane;
  P->h_obs_ptr.assign(obs_ptr, obs_ptr + T + 1);
  LVBA_CUDA(cudaGetDevice(&P->device));
  LVBA_CUDA(cudaStreamCreateWithFlags(&P->stream, cudaStreamNonBlocking));
  P->timers.stream = P->stream;
  LVBA_TRY(pinned_pool().take(16 * sizeof(double), (void**)&P->h_scal));
  cudaStream_t s = P->stream;

  // ---- valid landmarks, active cameras (src/lvba_system.cpp:1582-1583, 1598-1603; SURVEY.md Q11)
  std::vector<int64_t> valid;
  std::vector<int> row_of_cam;
  visual_rows(M, T, plane_nd, obs_ptr, obs_cam, fixed_cam, P->cam_fixed.empty() ? nullptr : P->cam_fixed.data(), valid, row_of_cam,
              P->cam_of_row);
  lap("valid landmarks / rows");

  // ---- the caller's arrays go up as they are (one DMA each from the caller's, ideally pinned, memory); the plan gathers the
  // per-observation arrays from them on the device
  DevBuf<long long> d_obs_ptr;
  DevBuf<int> d_raw_cam;
  DevBuf<float2> d_raw_uv;
  DevBuf<double> d_raw_plane;
  auto upload_raw = [&](VisualSrc& src) -> int {
    const int64_t nnz_all = obs_ptr[T];
    static_assert(sizeof(long long) == sizeof(int64_t), "obs_ptr is uploaded as it is");
    LVBA_TRY(d_obs_ptr.upload(reinterpret_cast<const long long*>(obs_ptr), (size_t)T + 1, s, &P->h2d));
    LVBA_TRY(d_raw_cam.upload(obs_cam, (size_t)nnz_all, s, &P->h2d));
    LVBA_TRY(d_raw_uv.upload(reinterpret_cast<const float2*>(obs_uv), (size_t)nnz_all, s, &P->h2d));
    LVBA_TRY(d_raw_plane.upload(plane_nd, (size_t)T * 4, s, &P->h2d));
    src = VisualSrc{d_obs_ptr.p, d_raw_cam.p, d_raw_uv.p, d_raw_plane.p};
    return LVBA_OK;
  };
  LVBA_TRY(visual_plan(P.get(), valid, obs_ptr, obs_cam, row_of_cam, nullptr, upload_raw, lap));
  LVBA_TRY(P->q.upload(q, (size_t)M * 4, s, &P->h2d));
  LVBA_TRY(P->t.upload(t, (size_t)M * 3, s, &P->h2d));
  LVBA_TRY(P->X.upload(X, (size_t)T * 3, s, &P->h2d));
  {   // restore point and candidate start as device-side copies of what just went up (no second and third trip over PCIe)
    auto dup = [&](DevBuf<double>& dst, const DevBuf<double>& src, size_t count) -> int {
      LVBA_TRY(dst.alloc(count));
      if (count) LVBA_CUDA(cudaMemcpyAsync(dst.p, src.p, count * sizeof(double), cudaMemcpyDeviceToDevice, s));
      return LVBA_OK;
    };
    LVBA_TRY(dup(P->q0, P->q, (size_t)M * 4)); LVBA_TRY(dup(P->t0, P->t, (size_t)M * 3)); LVBA_TRY(dup(P->X0, P->X, (size_t)T * 3));
    LVBA_TRY(dup(P->qc, P->q, (size_t)M * 4)); LVBA_TRY(dup(P->tc, P->t, (size_t)M * 3)); LVBA_TRY(dup(P->Xc, P->X, (size_t)T * 3));
  }
  LVBA_TRY(P->scal.alloc(16)); LVBA_TRY(P->scal.zero(s));
  LVBA_TRY(P->cam_step.alloc((size_t)M * 6)); LVBA_TRY(P->pt_step.alloc((size_t)std::max<int64_t>(T, 1) * 3));
  LVBA_CUDA(cudaFuncSetAttribute(visual_build_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)visual_build_smem_bytes()));
  LVBA_CUDA(cudaFuncSetAttribute(visual_build_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)visual_build_smem_bytes()));
  LVBA_CUDA(cudaFuncSetAttribute(visual_backsub_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)visual_backsub_smem_bytes()));
  LVBA_CUDA(cudaFuncSetAttribute(visual_backsub_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)visual_backsub_smem_bytes()));
  LVBA_CUDA(cudaStreamSynchronize(s));
  lap("uploads + allocations");
  lvba_visual_default_opts(&P->opts);
  P->ms_setup = wall_ms() - t_begin;
  *out = P.release();
  return LVBA_OK;
}

inline int visual_det_setup(lvba_visual_problem* P);

// A removal of observations (lvba_visual_remove_observations / _remove_outliers) for visual_replan: host copies of the rule's
// keep flags [nnz] and kept counts [Tv] over the current local CSR, and the kept observations' camera, pixel and caller index,
// compacted on the device in the local order (voutliers::CompactF).
struct VisualKept {
  const uint8_t* keep = nullptr;
  const int32_t* kcnt = nullptr;
  const int* cam = nullptr;
  const float2* uv = nullptr;
  const int64_t* src = nullptr;
};

// A new set of constant cameras on a handle (lvba_visual_reset_lm), or a removal (kept != null): visual_plan again, from the
// handle's own arrays.  The source landmarks are the local landmarks of the current plan, taken in the caller's order, so that
// the new plan is the one lvba_visual_create would make with this mask (and, after a removal, from the kept observations with
// the dropped landmarks' planes left out); observations, planes and the state stay on the device.  One GPU only: the local
// landmarks are then all valid ones (visual_set_mode and the removal calls refuse an active communicator).
// Deterministic mode is off afterwards unless `det` asks for its records as part of the new plan.
// A failure leaves the handle as it was (the previous plan is made again from the same source arrays) with deterministic mode
// off; only if that fails too is the handle marked unusable, and then every call but destroy, get_state, set_state and
// reset_state refuses it.
inline int visual_replan(lvba_visual_problem* P, std::vector<uint8_t> mask, const VisualKept* kept = nullptr, bool det = false) {
  SetupLaps lap("visual re-plan", 26, P->stream, wall_ms());
  cudaStream_t s = P->stream;
  const int64_t Tv = P->Tv;
  std::vector<int> trk_ptr((size_t)Tv + 1, 0), trk_id((size_t)Tv), cam((size_t)P->nnz);
  if (Tv > 0) {
    LVBA_CUDA(cudaMemcpyAsync(trk_ptr.data(), P->trk_ptr.p, trk_ptr.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    LVBA_CUDA(cudaMemcpyAsync(trk_id.data(), P->trk_id.p, trk_id.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (!cam.empty()) LVBA_CUDA(cudaMemcpyAsync(cam.data(), P->obs_cam.p, cam.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    LVBA_CUDA(cudaStreamSynchronize(s));
    P->d2h += (int64_t)(trk_ptr.size() + trk_id.size() + cam.size()) * (int64_t)sizeof(int);
  }
  voutliers::ReplanSource all, cut;
  voutliers::replan_source(Tv, trk_id.data(), trk_ptr.data(), cam.data(), nullptr, nullptr, all);
  if (kept) voutliers::replan_source(Tv, trk_id.data(), trk_ptr.data(), cam.data(), kept->keep, kept->kcnt, cut);
  lap("rows");
  // the records of deterministic mode follow the table: set up again when the mode is next asked for (visual_set_mode)
  auto det_release = [&] {
    tiles::fixed_sum_release(P->det_S); tiles::fixed_sum_release(P->det_G); P->det_C.release();
    P->det_ready = false;
    P->det = false;
    P->solver.set_deterministic(false);
  };
  det_release();
  DevBuf<long long> d_src_ptr;
  DevBuf<int> old_cam;
  DevBuf<float2> old_uv;
  DevBuf<double> old_plane;
  DevBuf<int64_t> old_src;
  const bool had_src = P->obs_src_ready;
  old_cam.swap(P->obs_cam); old_uv.swap(P->obs_uv); old_plane.swap(P->plane); old_src.swap(P->obs_src);
  auto plan_with = [&](const std::vector<uint8_t>& m, const voutliers::ReplanSource& S, const VisualSrc& arrays, bool with_det) -> int {
    std::vector<char> used((size_t)P->M, 0);
    for (int c : S.cam) used[c] = 1;
    std::vector<int> row_of_cam;
    visual_row_map(P->M, used, P->fixed_cam, m.empty() ? nullptr : m.data(), row_of_cam, P->cam_of_row);
    auto get = [&](VisualSrc& src) -> int {
      LVBA_TRY(d_src_ptr.upload(reinterpret_cast<const long long*>(S.src_ptr.data()), S.src_ptr.size(), s, &P->h2d));
      src = arrays;
      src.obs_ptr = d_src_ptr.p;
      return LVBA_OK;
    };
    LVBA_TRY(visual_plan(P, S.valid, S.src_ptr.data(), S.cam.data(), row_of_cam, trk_id.data(), get, lap));
    if (with_det) {
      LVBA_TRY(visual_det_setup(P));
      P->det = true;
      P->solver.set_deterministic(true);
    }
    return P->scal.zero(s);                                    // no stale camera gradient when the new plan has no rows
  };
  const VisualSrc old_arrays{nullptr, old_cam.p, old_uv.p, old_plane.p, had_src ? old_src.p : nullptr};
  const char* what = kept ? "re-plan after the removal" : "re-plan for the new cam_fixed";
  const char* keeps = kept ? "nothing was removed" : "the handle keeps its previous constant cameras";
  int rc;
  try {
    rc = kept ? plan_with(mask, cut, VisualSrc{nullptr, kept->cam, kept->uv, old_plane.p, kept->src}, det) : plan_with(mask, all, old_arrays, false);
  } catch (const std::bad_alloc&) { rc = fail(LVBA_ERR_NOMEM, "host allocation failed"); }
  if (rc != LVBA_OK) {
    const std::string why = last_error_ref();
    cudaStreamSynchronize(s);
    cudaGetLastError();
    det_release();
    int rc_back;
    try { rc_back = plan_with(P->cam_fixed, all, old_arrays, false); } catch (const std::bad_alloc&) { rc_back = LVBA_ERR_NOMEM; }
    if (rc_back != LVBA_OK) {
      P->unusable = true;
      return fail(rc, "%s failed (%s), and so did restoring the previous plan: destroy the handle", what, why.c_str());
    }
    return fail(rc, "%s failed (%s); %s", what, why.c_str(), keeps);
  }
  P->cam_fixed = std::move(mask);
  return LVBA_OK;
}

// Deterministic mode: the records of the build and their destinations (visual_det_index), and the records of the column-norm pass
inline int visual_det_setup(lvba_visual_problem* P) {
  if (P->det_ready) return LVBA_OK;
  const int64_t nS = P->prun.n_runs + P->drun.n_runs + P->n_big_obs + P->n_big_pairs;
  if (nS >= (int64_t)1 << 32) return fail(LVBA_ERR_UNSUPPORTED, "deterministic mode: %lld contributions to S (at most 2^32)", (long long)nS);
  CudaExec ex;
  ex.stream = P->stream;
  LVBA_TRY(visual_det_index(ex, P->table_in(), P->prun, P->drun, P->view(), P->big_view(), P->n_big_obs, P->n_big_pairs, P->det_S, P->det_G));
  LVBA_TRY(P->det_C.alloc((size_t)std::max<int64_t>(P->det_G.n_rec, 1) * 6));
  LVBA_CUDA(cudaFuncSetAttribute(visual_build_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)visual_build_smem_bytes()));
  LVBA_CUDA(cudaFuncSetAttribute(visual_build_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)visual_build_smem_bytes()));
  P->launches += ex.launches;
  P->det_ready = true;
  return LVBA_OK;
}

// the robust losses of lvba_visual_opts: a known kind, and for a loss a finite scale > 0 (checked before any device work)
inline int visual_check_loss(const lvba_visual_opts& o) {
  const int32_t kinds[2] = {o.reproj_loss, o.plane_loss};
  const double scales[2] = {o.reproj_loss_scale, o.plane_loss_scale};
  const char* names[2] = {"reproj_loss", "plane_loss"};
  for (int i = 0; i < 2; ++i) {
    if (kinds[i] != LVBA_LOSS_NONE && kinds[i] != LVBA_LOSS_HUBER && kinds[i] != LVBA_LOSS_CAUCHY)
      return fail(LVBA_ERR_INVALID_ARG, "%s = %d is not an lvba_loss_kind", names[i], (int)kinds[i]);
    if (kinds[i] != LVBA_LOSS_NONE && !(std::isfinite(scales[i]) && scales[i] > 0.0))
      return fail(LVBA_ERR_INVALID_ARG, "%s_scale = %g: a loss needs a finite scale > 0", names[i], scales[i]);
  }
  return LVBA_OK;
}

// a handle whose failed re-plan could not be undone (visual_replan) takes no further calls but destroy and the state copies
inline int visual_check_usable(const lvba_visual_problem* P) {
  if (P->unusable) return fail(LVBA_ERR_INVALID_ARG, "this handle lost its plan in a failed lvba_visual_reset_lm: destroy it");
  return LVBA_OK;
}

// constant cameras beyond fixed_cam run on one GPU (the shard of a landmark follows its lowest camera, whatever is constant)
inline int visual_check_mask(bool has_mask) {
  if (has_mask && comm().active())
    return fail(LVBA_ERR_UNSUPPORTED, "cam_fixed runs on one GPU: constant cameras are not supported with an active communicator");
  return LVBA_OK;
}

// no intrinsics system or step until the next pass (a reset or a new mask): lvba_visual_get_intrinsics_system returns nothing older
inline void visual_intr_forget(lvba_visual_problem* P) {
  P->intr_have_sys = false;
  for (int i = 0; i < 8; ++i) P->intr_step[i] = 0.0;
}

// the LM mode of the handle (lvba_visual_reset_lm and the one-shot call): the constant cameras, deterministic mode and the
// robust losses
inline int visual_set_mode(lvba_visual_problem* P, const lvba_visual_opts& o) {
  LVBA_TRY(visual_check_loss(o));
  if (o.refine_intrinsics >> 8)
    return fail(LVBA_ERR_INVALID_ARG, "refine_intrinsics = 0x%x: only bits 0..7 name intrinsics", (unsigned)o.refine_intrinsics);
  if (o.refine_intrinsics && comm().active())
    return fail(LVBA_ERR_UNSUPPORTED, "refine_intrinsics runs on one GPU: not with an active communicator");
  if (o.deterministic && comm().active())
    return fail(LVBA_ERR_UNSUPPORTED, "deterministic mode runs on one GPU: the multi-GPU sums of NCCL have no fixed order");
  std::vector<uint8_t> mask = visual_mask(P->M, o.cam_fixed);
  LVBA_TRY(visual_check_mask(!mask.empty() || !P->cam_fixed.empty()));
  if (mask != P->cam_fixed) {
    LVBA_CUDA(cudaSetDevice(P->device));
    LVBA_TRY(visual_replan(P, std::move(mask)));
  }
  if (o.deterministic) {
    LVBA_CUDA(cudaSetDevice(P->device));
    const int rc = visual_det_setup(P);
    if (rc != LVBA_OK) {                                      // nothing half set up stays on the handle
      tiles::fixed_sum_release(P->det_S); tiles::fixed_sum_release(P->det_G); P->det_C.release();
      return rc;
    }
  }
  P->det = o.deterministic != 0;
  P->solver.set_deterministic(P->det);
  P->loss_px = o.reproj_loss; P->loss_a_px = o.reproj_loss_scale;
  P->loss_pl = o.plane_loss; P->loss_a_pl = o.plane_loss_scale;
  P->intr_mask = o.refine_intrinsics;
  visual_intr_forget(P);
  return LVBA_OK;
}

// ---------------------------------------------------------------- the intrinsics block (visual_intr.h)
// The row CSR of the border gather and the block's buffers, for the current plan
inline int visual_intr_setup(lvba_visual_problem* P) {
  if (P->intr_ready) return LVBA_OK;
  cudaStream_t s = P->stream;
  std::vector<int> row((size_t)P->nnz);
  if (P->nnz > 0) {
    LVBA_CUDA(cudaMemcpyAsync(row.data(), P->obs_row.p, row.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    LVBA_CUDA(cudaStreamSynchronize(s));
    P->d2h += P->nnz * (int64_t)sizeof(int);
  }
  std::vector<int64_t> ptr((size_t)P->n_rows + 1, 0), obs;
  for (int r : row)
    if (r >= 0) ++ptr[(size_t)r + 1];
  for (int r = 0; r < P->n_rows; ++r) ptr[(size_t)r + 1] += ptr[(size_t)r];
  obs.resize((size_t)ptr[(size_t)P->n_rows]);
  {
    std::vector<int64_t> at(ptr.begin(), ptr.end() - 1);
    for (int64_t w = 0; w < P->nnz; ++w)
      if (row[(size_t)w] >= 0) obs[(size_t)at[(size_t)row[(size_t)w]]++] = w;
  }
  LVBA_TRY(P->intr_row_ptr.upload(ptr, s, &P->h2d));
  LVBA_TRY(P->intr_row_obs.alloc(std::max<size_t>(obs.size(), 1)));
  if (!obs.empty()) LVBA_TRY(P->intr_row_obs.upload(obs, s, &P->h2d));
  const size_t Tv = (size_t)std::max<int64_t>(P->Tv, 1), n6 = (size_t)std::max(P->n_rows, 1) * 6;
  LVBA_TRY(P->intr_slot.alloc(Tv * vintr::kSys));
  LVBA_TRY(P->intr_rec.alloc((size_t)std::max<int64_t>(P->nnz, 1) * vintr::kRec));
  LVBA_TRY(P->intr_part.alloc(((Tv + 255) / 256) * vintr::kSys));
  LVBA_TRY(P->intr_sys.alloc(vintr::kSys));
  LVBA_TRY(P->intr_B.alloc(8 * n6)); LVBA_TRY(P->intr_Y.alloc(8 * n6));
  if (P->intr_dev.n == 0) { LVBA_TRY(P->intr_dev.alloc(32)); LVBA_TRY(P->intr_dev.zero(s)); }
  LVBA_CUDA(cudaStreamSynchronize(s));                         // the host vectors are idle before they go out of scope
  P->intr_ready = true;
  return LVBA_OK;
}

// out[j] = sum_r in[r][j] (j < W, r < n), in row order: chunks of 256 rows, then the chunks
inline int visual_intr_reduce(lvba_visual_problem* P, CudaExec& ex, const double* in, int64_t n, int W, double* out) {
  const int64_t nch = std::max<int64_t>((n + 255) / 256, 1);
  LVBA_TRY(ex.for_each(nch * W, vintr::ReduceF{in, n, 256, W, P->intr_part.p}));
  return ex.for_each(W, vintr::ReduceF{P->intr_part.p, nch, nch, W, out});
}

// Jacobi scaling vectors from the Jacobian at the current state (Ceres: once, at iteration 0)
template <bool kLoss>
inline int visual_compute_scale_t(lvba_visual_problem* P, int enabled) {
  cudaStream_t s = P->stream;
  LVBA_TRY(P->cam_colsq.zero(s));
  if (P->n_tiles > 0) {
    if (P->det) visual_colnorm_kernel<true, kLoss><<<P->n_tiles, kVisTileSlots, 0, s>>>(P->view(), P->state(), P->det_C.p, P->pt_colsq.p);
    else visual_colnorm_kernel<false, kLoss><<<P->n_tiles, kVisTileSlots, 0, s>>>(P->view(), P->state(), P->cam_colsq.p, P->pt_colsq.p);
    ++P->launches;
  }
  if (P->n_big > 0) {
    if (P->det)
      wide_pass(s, P->n_big_obs, vbig::ColObsPass<true, kLoss>{P->view(), P->big_view(), P->state(), P->big_obs.p,
                                                               P->det_C.p + 6 * P->drun.n_runs}, &P->launches);
    else
      wide_pass(s, P->n_big_obs, vbig::ColObsPass<false, kLoss>{P->view(), P->big_view(), P->state(), P->big_obs.p, P->cam_colsq.p}, &P->launches);
    wide_pass(s, P->n_big, vbig::ColTrackPass<kLoss>{P->view(), P->big_view(), P->state(), P->big_obs.p, P->pt_colsq.p}, &P->launches);
  }
  if (P->det) {
    CudaExec ex;
    ex.stream = s;
    LVBA_TRY(ex.for_each(P->det_G.by_dst.n_runs * 6, tiles::gather_part(P->det_G, P->det_C.p, 6, 0, 6, P->cam_colsq.p)));
    P->launches += ex.launches;
  }
  Comm& cm = comm();
  if (cm.active()) LVBA_TRY(cm.allreduce_sum(P->cam_colsq.p, (size_t)P->n_rows * 6, s));
  const long long nc = (long long)P->n_rows * 6, np = (long long)P->Tv * 3;
  if (nc > 0) { visual_scale_kernel<<<(unsigned)((nc + 255) / 256), 256, 0, s>>>(nc, P->cam_colsq.p, enabled, P->s_cam.p); ++P->launches; }
  if (np > 0) { visual_scale_kernel<<<(unsigned)((np + 255) / 256), 256, 0, s>>>(np, P->pt_colsq.p, enabled, P->s_pt.p); ++P->launches; }
  if (P->intr_mask) {                                          // the block's scale: sk in intr_dev[0..7], its column norms in [8..15]
    LVBA_TRY(visual_intr_setup(P));
    CudaExec ex;
    ex.stream = s;
    LVBA_TRY(ex.for_each(P->Tv, vintr::ColF<kLoss>{P->view(), P->state(), P->intr_slot.p}));
    LVBA_TRY(visual_intr_reduce(P, ex, P->intr_slot.p, P->Tv, 8, P->intr_dev.p + 8));
    LVBA_TRY(ex.for_each(8, vintr::ScaleF{P->intr_dev.p + 8, P->intr_mask, enabled, P->intr_dev.p}));
    P->launches += ex.launches;
  }
  LVBA_CUDA(cudaGetLastError());
  P->lm.have_scale = true;
  return LVBA_OK;
}
inline int visual_compute_scale(lvba_visual_problem* P, int enabled) {
  return P->robust() ? visual_compute_scale_t<true>(P, enabled) : visual_compute_scale_t<false>(P, enabled);
}

// 1/2 sum r^2 (with a loss: 1/2 sum rho) at the state `st` into *out (device): batches, big landmarks, reduction.  intr: the
// intrinsics to evaluate with (null: the handle's current ones)
template <bool kLoss>
inline void visual_cost_t(lvba_visual_problem* P, const VisualState& st, double* out, const double* intr = nullptr) {
  cudaStream_t s = P->stream;
  VisualView vv = P->view();
  if (intr) for (int i = 0; i < 8; ++i) vv.intr[i] = intr[i];
  if (P->n_batches > 0) {
    if constexpr (kLoss) visual_cost_loss_kernel<<<P->n_batches, kSlots, 0, s>>>(vv, st, P->batch_cost.p);
    else visual_cost_kernel<<<P->n_batches, kSlots, 0, s>>>(vv, st, P->batch_cost.p);
    ++P->launches;
  }
  if (P->n_big > 0) wide_pass(s, P->n_big, vbig::CostPass<kLoss>{vv, P->big_view(), st, P->batch_cost.p + P->n_batches}, &P->launches);
  reduce_partials_kernel<<<1, 256, 0, s>>>(P->batch_cost.p, (int)(P->n_batches + P->n_big), out);
  ++P->launches;
}

inline VisualLM visual_lm_params(const lvba_visual_problem* P, double radius) {
  return VisualLM{radius, P->opts.min_lm_diagonal, P->opts.max_lm_diagonal, P->s_cam.p, P->s_pt.p};
}

// scal layout: [0] cost  [1] gmax  [2] model  [3] step^2 (pts)  [4] x^2 (pts)  [5] -  [6] step^2 (cams) [7] x^2 (cams)
//              [8] candidate cost
template <bool kLoss>
inline int visual_linearize_solve_t(lvba_visual_problem* P, double radius, bool want_steps) {
  cudaStream_t s = P->stream;
  const VisualLM lm = visual_lm_params(P, radius);
  const EnvView ev = P->env.view();
  Comm& cm = comm();
  P->timers.begin(PH_BUILD);
  LVBA_TRY(P->S.zero(s)); LVBA_TRY(P->rhs.zero(s)); LVBA_TRY(P->cam_colsq.zero(s)); LVBA_TRY(P->cam_grad.zero(s));
  LVBA_CUDA(cudaMemsetAsync(P->scal.p + 1, 0, sizeof(double), s));
  if (P->n_tiles > 0) {
    if (P->det)
      visual_build_kernel<true, kLoss><<<P->n_tiles, kVisTileSlots, visual_build_smem_bytes(), s>>>(
          P->view(), ev, P->state(), lm, P->det_S.rec.p, P->det_G.rec.p, nullptr, nullptr, P->batch_cost.p, P->batch_gmax.p);
    else
      visual_build_kernel<false, kLoss><<<P->n_tiles, kVisTileSlots, visual_build_smem_bytes(), s>>>(
          P->view(), ev, P->state(), lm, P->S.p, P->rhs.p, P->cam_colsq.p, P->cam_grad.p, P->batch_cost.p, P->batch_gmax.p);
    ++P->launches;
  }
  if (P->n_big > 0) {        // cost and gradient max of landmark b in the partial slots n_tiles + b
    const VisualView vv = P->view();
    const vbig::View bv = P->big_view();
    wide_pass(s, P->n_big_obs, vbig::ObsPass<kLoss>{vv, bv, P->state(), lm, P->big_obs.p}, &P->launches);
    wide_pass(s, P->n_big, vbig::TrackPass<kLoss>{vv, bv, P->state(), lm, P->big_obs.p, P->big_params.p,
                                                  P->batch_cost.p + P->n_tiles, P->batch_gmax.p + P->n_tiles}, &P->launches);
    if (P->det) {
      const int64_t s0 = P->prun.n_runs + P->drun.n_runs, g0 = P->drun.n_runs;
      wide_pass(s, P->n_big_obs, vbig::SlotsDetF{vv, bv, P->big_params.p, P->big_obs.p, P->det_S.rec.p + 36 * s0,
                                                 P->det_G.rec.p + 18 * g0, nullptr, nullptr}, &P->launches);
      wide_pass(s, P->n_big_pairs, vbig::PairsDetF{vv, bv, P->big_obs.p, P->det_S.rec.p + 36 * (s0 + P->n_big_obs)}, &P->launches);
    } else {
      wide_pass(s, P->n_big_obs, vbig::SlotsF{vv, bv, P->big_params.p, P->big_obs.p, P->S.p, P->rhs.p, P->cam_colsq.p, P->cam_grad.p}, &P->launches);
      wide_pass(s, P->n_big_pairs, vbig::PairsF{vv, bv, P->big_obs.p, P->S.p}, &P->launches);
    }
  }
  if (P->det) {
    CudaExec ex;
    ex.stream = s;
    const int64_t nr = P->det_G.by_dst.n_runs;
    LVBA_TRY(ex.for_each(P->det_S.by_dst.n_runs * 36, tiles::gather_of(P->det_S, P->S.p)));
    LVBA_TRY(ex.for_each(nr * 6, tiles::gather_part(P->det_G, P->det_G.rec.p, 18, 0, 6, P->rhs.p)));
    LVBA_TRY(ex.for_each(nr * 6, tiles::gather_part(P->det_G, P->det_G.rec.p, 18, 6, 6, P->cam_colsq.p)));
    LVBA_TRY(ex.for_each(nr * 6, tiles::gather_part(P->det_G, P->det_G.rec.p, 18, 12, 6, P->cam_grad.p)));
    P->launches += ex.launches;
  }
  reduce_partials_kernel<<<1, 256, 0, s>>>(P->batch_cost.p, (int)(P->n_tiles + P->n_big), P->scal.p + 0);
  reduce_max_kernel<<<1, 256, 0, s>>>(P->batch_gmax.p, (int)(P->n_tiles + P->n_big), P->scal.p + 1);
  P->launches += 2;
  if (cm.active()) {
    // row-owned reduced camera system (SURVEY.md 8(e)): see lidar_build_dev
    if (P->solver.dist()) LVBA_TRY(P->solver.exchange_rows(P->env, P->S.p, s, &P->launches));
    else LVBA_TRY(cm.allreduce_sum(P->S.p, (size_t)P->env.nblocks * 36, s));
    LVBA_TRY(cm.allreduce_sum(P->rhs.p, (size_t)P->n_rows * 6, s));
    LVBA_TRY(cm.allreduce_sum(P->cam_colsq.p, (size_t)P->n_rows * 6, s));
    LVBA_TRY(cm.allreduce_sum(P->cam_grad.p, (size_t)P->n_rows * 6, s));
    LVBA_TRY(cm.allreduce_sum(P->scal.p + 0, 1, s));
  }
  const bool intr = P->intr_mask != 0;
  const int64_t n6 = (int64_t)P->n_rows * 6;
  if (intr) {                                                  // the border, the corner and rhs_k of the intrinsics block
    LVBA_TRY(visual_intr_setup(P));
    CudaExec ex;
    ex.stream = s;
    LVBA_TRY(ex.for_each(P->Tv, vintr::TrackF<kLoss>{P->view(), P->state(), lm, P->intr_dev.p, P->intr_slot.p, P->intr_rec.p}));
    LVBA_TRY(visual_intr_reduce(P, ex, P->intr_slot.p, P->Tv, vintr::kSys, P->intr_sys.p));
    LVBA_TRY(ex.for_each(P->n_rows * (int64_t)vintr::kRec, vintr::RowGatherF{P->intr_row_ptr.p, P->intr_row_obs.p, P->intr_rec.p, n6, P->intr_B.p}));
    P->launches += ex.launches;
  }
  P->timers.end();
  ++P->lm.builds;
  P->timers.begin(PH_SOLVE);
  if (P->n_rows > 0) {
    visual_cam_diag_kernel<<<1, 256, 0, s>>>(6 * P->n_rows, P->cam_colsq.p, P->cam_grad.p, P->s_cam.p, P->opts.min_lm_diagonal,
                                             P->opts.max_lm_diagonal, radius, P->dadd.p, P->scal.p + 5);
    ++P->launches;
    if (intr)                                                  // Y[:, i] = A^-1 B[:, i] for every free entry, through solver.z and y
      for (int i = 0; i < 8; ++i) {
        if (!((P->intr_mask >> i) & 1u)) continue;
        LVBA_CUDA(cudaMemcpyAsync(P->solver.z.p, P->intr_B.p + i * n6, (size_t)n6 * sizeof(double), cudaMemcpyDeviceToDevice, s));
        LVBA_TRY(P->solver.solve(P->env, P->S.p, P->dadd.p, P->y.p, s, &P->launches));
        LVBA_CUDA(cudaMemcpyAsync(P->intr_Y.p + i * n6, P->y.p, (size_t)n6 * sizeof(double), cudaMemcpyDeviceToDevice, s));
      }
    LVBA_CUDA(cudaMemcpyAsync(P->solver.z.p, P->rhs.p, (size_t)P->n_rows * 6 * sizeof(double), cudaMemcpyDeviceToDevice, s));
    LVBA_TRY(P->solver.solve(P->env, P->S.p, P->dadd.p, P->y.p, s, &P->launches));
  }
  double yk[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (intr) {                                                  // the corner, y_k and the camera step y - Y y_k
    visual_intr_corner_kernel<<<1, 256, 0, s>>>(n6, P->intr_B.p, P->intr_Y.p, P->y.p, P->intr_sys.p, P->intr_dev.p, P->intr_mask,
                                                P->opts.min_lm_diagonal, P->opts.max_lm_diagonal, radius, P->intr_dev.p + 16, P->scal.p);
    ++P->launches;
    // the candidate intrinsics go into the cost kernels' VisualView by value: the step comes to the host here
    double h[16];
    LVBA_CUDA(cudaMemcpyAsync(h, P->intr_dev.p + 16, sizeof(h), cudaMemcpyDeviceToHost, s));
    LVBA_CUDA(cudaStreamSynchronize(s));
    P->d2h += sizeof(h);
    for (int i = 0; i < 8; ++i) { yk[i] = h[i]; P->intr_step[i] = h[8 + i]; P->intr_c[i] = P->intr[i] + h[8 + i]; }
    P->intr_have_sys = true;
  }
  P->timers.end();
  P->timers.begin(PH_RESID);
  if (intr) {
    CudaExec ex;
    ex.stream = s;
    vintr::BacksubF<kLoss> f{P->view(), P->state(), lm, P->intr_dev.p, P->y.p, {}, P->Xc.p, want_steps ? P->pt_step.p : nullptr, P->intr_slot.p};
    for (int i = 0; i < 8; ++i) f.yk[i] = yk[i];
    LVBA_TRY(ex.for_each(P->Tv, f));
    LVBA_TRY(visual_intr_reduce(P, ex, P->intr_slot.p, P->Tv, 3, P->scal.p + 2));
    P->launches += ex.launches;
  } else if (P->n_batches > 0) {
    visual_backsub_kernel<kLoss><<<P->n_batches, kSlots, visual_backsub_smem_bytes(), s>>>(
        P->view(), P->state(), lm, P->y.p, P->Xc.p, want_steps ? P->pt_step.p : nullptr, P->batch_out.p);
    ++P->launches;
  }
  if (!intr) {
    if (P->n_big > 0)
      wide_pass(s, P->n_big, vbig::BacksubPass<kLoss>{P->view(), P->big_view(), P->state(), lm, P->big_obs.p, P->big_params.p, P->y.p,
                                                      P->Xc.p, want_steps ? P->pt_step.p : nullptr,
                                                      P->batch_out.p + 4 * (int64_t)P->n_batches}, &P->launches);
    reduce_cols_kernel<<<1, 256, 0, s>>>(P->batch_out.p, (int)(P->n_batches + P->n_big), 4, 3, P->scal.p + 2);
    ++P->launches;
  }
  const int ncb = (P->n_rows + 127) / 128;
  if (ncb > 0) {
    visual_cam_update_kernel<<<ncb, 128, 0, s>>>(P->n_rows, P->d_cam_of_row.p, P->q.p, P->t.p, P->y.p, P->s_cam.p, P->qc.p, P->tc.p,
                                                 want_steps ? P->cam_step.p : nullptr, P->cam_out.p);
    ++P->launches;
  }
  reduce_cols_kernel<<<1, 256, 0, s>>>(P->cam_out.p, ncb, 2, 2, P->scal.p + 6);
  ++P->launches;
  if (cm.active()) LVBA_TRY(cm.allreduce_sum(P->scal.p + 2, 3, s));   // model, step^2, x^2 of the landmark shard
  visual_cost_t<kLoss>(P, P->cand(), P->scal.p + 8, intr ? P->intr_c : nullptr);   // candidate cost
  if (cm.active()) LVBA_TRY(cm.allreduce_sum(P->scal.p + 8, 1, s));
  P->timers.end();
  LVBA_CUDA(cudaGetLastError());
  LVBA_CUDA(cudaMemcpyAsync(P->h_scal, P->scal.p, 16 * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (P->n_rows > 0) LVBA_CUDA(cudaMemcpyAsync(P->h_scal + 15, P->solver.status.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  LVBA_CUDA(cudaStreamSynchronize(s));
  if (P->n_rows == 0) *reinterpret_cast<int*>(P->h_scal + 15) = 0;   // every camera constant: nothing was factorised
  P->d2h += 16 * sizeof(double);
  if (intr) {        // the block in the gradient max-norm, the status and the norms (Ceres: ||x|| over all 8 entries of the block)
    double* h = P->h_scal;
    h[1] = std::max(h[1], h[9]);
    if (h[10] != 0.0) *reinterpret_cast<int*>(h + 15) |= 1;
    for (int i = 0; i < 8; ++i) { h[3] += P->intr_step[i] * P->intr_step[i]; h[4] += P->intr[i] * P->intr[i]; }
  }
  return LVBA_OK;
}
inline int visual_linearize_solve(lvba_visual_problem* P, double radius, bool want_steps) {
  return P->robust() ? visual_linearize_solve_t<true>(P, radius, want_steps) : visual_linearize_solve_t<false>(P, radius, want_steps);
}

inline int visual_iterate_impl(lvba_visual_problem* P, int n_iter, lvba_summary* sum) {
  const double t0 = wall_ms();
  const int64_t l0 = P->launches, h0 = P->h2d, d0 = P->d2h;
  TrustRegionState& lm = P->lm;
  const int iters0 = lm.iters, acc0 = lm.accepted, builds0 = lm.builds;
  const lvba_visual_opts& o = P->opts;
  if (!lm.have_scale) LVBA_TRY(visual_compute_scale(P, o.jacobi_scaling));
  for (int it = 0; it < n_iter && !lm.converged; ++it) {
    LVBA_TRY(visual_linearize_solve(P, lm.radius, false));
    const double* h = P->h_scal;
    lm.cost = h[0];
    if (!lm.have_first) { lm.cost_first = lm.cost; lm.have_first = true; }
    const double gmax = std::max(h[1], h[5]);
    if (o.gradient_tolerance >= 0 && gmax <= o.gradient_tolerance) { lm.converged = true; lm.termination = LVBA_TERM_GRADIENT_TOL; break; }
    ++lm.iters;
    const double model = h[2];
    const double cand = h[8];
    const int fstat = *reinterpret_cast<const int*>(h + 15);
    const double step_norm = std::sqrt(h[3] + h[6]), x_norm = std::sqrt(h[4] + h[7]);
    const bool valid = fstat == 0 && std::isfinite(model) && std::isfinite(step_norm) && model > 0.0;
    if (o.verbose)
      fprintf(stderr, "[lvba visual] iter %d: cost %.9g cand %.9g model %.6g radius %.3g step %.3g valid %d\n", lm.iters, lm.cost, cand, model, lm.radius, step_norm, (int)valid);
    if (!valid) {                                    // LevenbergMarquardtStrategy::StepIsInvalid
      ++lm.invalid;
      lm.radius *= 0.5;
      if (lm.invalid >= 5) { lm.converged = true; lm.termination = LVBA_TERM_INVALID_STEPS; }
      continue;
    }
    lm.invalid = 0;
    const double rho = (lm.cost - cand) / model;
    if (o.parameter_tolerance >= 0 && step_norm <= o.parameter_tolerance * (x_norm + o.parameter_tolerance)) {
      lm.converged = true; lm.termination = LVBA_TERM_PARAMETER_TOL; break;
    }
    if (o.function_tolerance >= 0 && std::fabs(lm.cost - cand) <= o.function_tolerance * lm.cost) {
      lm.converged = true; lm.termination = LVBA_TERM_FUNCTION_TOL; break;     // Ceres returns x, not the candidate
    }
    if (std::isfinite(cand) && rho > o.min_relative_decrease) {             // StepAccepted
      std::swap(P->q.p, P->qc.p); std::swap(P->t.p, P->tc.p); std::swap(P->X.p, P->Xc.p);
      if (P->intr_mask) std::copy(P->intr_c, P->intr_c + 8, P->intr);
      // keep untouched entries (constant cameras, skipped landmarks) identical in both buffers: they never change
      lm.cost = cand;
      ++lm.accepted;
      lm.radius = std::min(o.max_radius, lm.radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * rho - 1.0, 3)));
      lm.nu = 2.0;
    } else {                                                                  // StepRejected
      lm.radius /= lm.nu;
      lm.nu *= 2.0;
      if (lm.radius < o.min_radius) { lm.converged = true; lm.termination = LVBA_TERM_RADIUS; }
    }
  }
  if (sum) {
    LVBA_CUDA(cudaStreamSynchronize(P->stream));
    double ms[PH_COUNT] = {0, 0, 0};
    P->timers.collect(ms);
    write_summary(sum, lm.iters - iters0, lm.accepted - acc0, lm.builds - builds0, lm.termination, lm.cost_first, lm.cost, lm.radius, ms,
                  wall_ms() - t0, P->launches - l0, P->h2d - h0, P->d2h - d0);
  }
  return LVBA_OK;
}


// ---------------------------------------------------------------- per-observation residuals and removal (visual_outliers.h)
// the calls that read or change the handle's observation set: one GPU (a rank holds only its own landmarks)
inline int visual_check_obs_calls(const lvba_visual_problem* P) {
  LVBA_TRY(visual_check_usable(P));
  if (comm().active()) return fail(LVBA_ERR_UNSUPPORTED, "per-observation residuals and removal run on one GPU: not with an active communicator");
  return LVBA_OK;
}

// obs_src: derived from trk_id, trk_ptr and the caller's obs_ptr while nothing has been removed (afterwards it always exists)
inline int visual_obs_src(lvba_visual_problem* P) {
  if (P->obs_src_ready) return LVBA_OK;
  cudaStream_t s = P->stream;
  LVBA_TRY(P->obs_src.alloc((size_t)P->nnz));
  if (P->Tv > 0) {
    DevBuf<int64_t> d_ptr;
    LVBA_TRY(d_ptr.upload(P->h_obs_ptr, s, &P->h2d));
    CudaExec ex;
    ex.stream = s;
    LVBA_TRY(ex.for_each(P->Tv, voutliers::DeriveSrcF{P->trk_id.p, P->trk_ptr.p, d_ptr.p, P->obs_src.p}));
    P->launches += ex.launches;
    LVBA_CUDA(cudaStreamSynchronize(s));                       // d_ptr is idle before it is parked
  }
  P->obs_src_ready = true;
  return LVBA_OK;
}

// s_q of every caller observation at the current state into P->obs_sq [N_obs]: NaN everywhere, then the observations in the
// problem (visual_obs_sq_kernel)
inline int visual_obs_sq_dev(lvba_visual_problem* P) {
  cudaStream_t s = P->stream;
  const int64_t n_obs = P->h_obs_ptr[(size_t)P->T];
  LVBA_TRY(visual_obs_src(P));
  if (P->obs_sq.n < (size_t)n_obs) LVBA_TRY(P->obs_sq.alloc((size_t)n_obs));
  CudaExec ex;
  ex.stream = s;
  LVBA_TRY(ex.for_each(n_obs, voutliers::NanFillF{P->obs_sq.p}));
  P->launches += ex.launches;
  if (P->nnz > 0) {
    visual_obs_sq_kernel<<<(unsigned)((P->nnz + 255) / 256), 256, 0, s>>>(P->view(), P->state(), P->nnz, (int)P->Tv, P->obs_src.p, P->obs_sq.p);
    LVBA_CUDA(cudaGetLastError());
    ++P->launches;
  }
  return LVBA_OK;
}

// The removal: keep flags by the caller's device mask d_remove [N_obs] (or, when null, s_q in P->obs_sq <= tau), the dropped
// landmarks, then the re-plan from the kept observations compacted on the device (visual_replan).  Only the keep flags and the
// kept counts come to the host.  Refused with nothing changed when no observation would be left.  The LM state is reset as
// lvba_visual_reset_lm with the handle's options would reset it; deterministic mode's records are set up again with the plan.
// Outputs are written on success only.
inline int visual_remove_impl(lvba_visual_problem* P, const uint8_t* d_remove, double tau, int32_t min_len, uint8_t* removed,
                              int64_t* n_obs_left, int64_t* n_trk_left, int64_t* n_rm_obs, int64_t* n_rm_trk) {
  cudaStream_t s = P->stream;
  const int64_t n_obs = P->h_obs_ptr[(size_t)P->T], nnz = P->nnz, Tv = P->Tv;
  LVBA_TRY(visual_obs_src(P));
  CudaExec ex;
  ex.stream = s;
  voutliers::RuleBufs<CudaExec> B;
  int64_t kept_obs = 0, kept_trk = 0;
  LVBA_TRY(voutliers::keep_rule(ex, nnz, Tv, P->trk_ptr.p, P->obs_src.p, d_remove, P->obs_sq.p, tau, min_len, B, &kept_obs, &kept_trk));
  P->d2h += 8;
  if (kept_obs == 0) return fail(LVBA_ERR_INVALID_ARG, "the removal would leave no observation in the problem");
  std::vector<uint8_t> h_removed;
  if (removed) {
    DevBuf<uint8_t> d_rm;
    LVBA_TRY(d_rm.alloc((size_t)n_obs));
    LVBA_TRY(ex.fill_zero(d_rm.p, (size_t)n_obs));
    LVBA_TRY(ex.for_each(nnz, voutliers::RemovedF{B.keep.p, P->obs_src.p, d_rm.p}));
    h_removed.resize((size_t)n_obs);
    LVBA_TRY(ex.fetch(h_removed.data(), d_rm.p, (size_t)n_obs));
    P->d2h += n_obs;
  }
  if (kept_obs < nnz || kept_trk < Tv) {
    std::vector<uint8_t> keep((size_t)nnz);
    std::vector<int32_t> kcnt((size_t)Tv);
    DevBuf<uint8_t> d_keep;
    LVBA_TRY(d_keep.alloc((size_t)nnz));
    LVBA_TRY(ex.for_each(nnz, voutliers::KeepBytesF{B.keep.p, d_keep.p}));
    LVBA_TRY(ex.fetch(keep.data(), d_keep.p, (size_t)nnz));
    LVBA_TRY(ex.fetch(kcnt.data(), B.kcnt.p, (size_t)Tv));
    P->d2h += nnz + Tv * 4;
    DevBuf<int> ccam;
    DevBuf<float2> cuv;
    DevBuf<int64_t> csrc;
    LVBA_TRY(ccam.alloc((size_t)kept_obs)); LVBA_TRY(cuv.alloc((size_t)kept_obs)); LVBA_TRY(csrc.alloc((size_t)kept_obs));
    LVBA_TRY(ex.for_each(nnz, voutliers::CompactF{B.keep.p, B.pos.p, P->obs_cam.p, P->obs_uv.p, P->obs_src.p, ccam.p, cuv.p, csrc.p}));
    LVBA_CUDA(cudaStreamSynchronize(s));
    const VisualKept K{keep.data(), kcnt.data(), ccam.p, cuv.p, csrc.p};
    LVBA_TRY(visual_replan(P, P->cam_fixed, &K, P->det));
    // the candidate starts as the state: a dropped landmark or a camera without observations is no longer written by a step,
    // and an accepted step swaps the buffers, so its candidate entry must hold its state
    const size_t nq = (size_t)P->M * 4 * sizeof(double), nt = (size_t)P->M * 3 * sizeof(double), nx = (size_t)P->T * 3 * sizeof(double);
    LVBA_CUDA(cudaMemcpyAsync(P->qc.p, P->q.p, nq, cudaMemcpyDeviceToDevice, s));
    LVBA_CUDA(cudaMemcpyAsync(P->tc.p, P->t.p, nt, cudaMemcpyDeviceToDevice, s));
    if (nx) LVBA_CUDA(cudaMemcpyAsync(P->Xc.p, P->X.p, nx, cudaMemcpyDeviceToDevice, s));
    LVBA_CUDA(cudaStreamSynchronize(s));                       // the compacted arrays are idle before they are parked
  }
  P->launches += ex.launches;
  P->lm.reset(P->opts);
  if (removed) std::copy(h_removed.begin(), h_removed.end(), removed);
  if (n_obs_left) *n_obs_left = kept_obs;
  if (n_trk_left) *n_trk_left = kept_trk;
  if (n_rm_obs) *n_rm_obs = nnz - kept_obs;
  if (n_rm_trk) *n_rm_trk = Tv - kept_trk;
  return LVBA_OK;
}

}  // namespace lvba

extern "C" {

void lvba_visual_default_opts(lvba_visual_opts* o) {
  if (!o) return;
  o->max_iter = 50; o->initial_radius = 1e4; o->max_radius = 1e16; o->min_radius = 1e-32;
  o->min_lm_diagonal = 1e-6; o->max_lm_diagonal = 1e32; o->min_relative_decrease = 1e-3;
  o->function_tolerance = 1e-6; o->gradient_tolerance = 1e-10; o->parameter_tolerance = 1e-8;
  o->jacobi_scaling = 1; o->device = -1; o->verbose = 0; o->deterministic = 0;
  // no loss (src/lvba_system.cpp:1630, :1639); the scales of the reference's HuberLoss objects (:1585-1586)
  o->reproj_loss = LVBA_LOSS_NONE; o->reproj_loss_scale = 1.0;
  o->plane_loss = LVBA_LOSS_NONE; o->plane_loss_scale = 0.1;
  o->cam_fixed = nullptr;
  o->refine_intrinsics = 0;
}

int lvba_visual_create(int32_t M, int64_t T, const double* q, const double* t, const double* X, const double* plane_nd,
                       const int64_t* obs_ptr, const int32_t* obs_cam, const float* obs_uv, const double intr[8],
                       double sigma_px, double sigma_plane, int32_t fixed_cam, int32_t device, lvba_visual_problem** out) LVBA_ABI_BEGIN {
  return lvba::visual_create_impl(M, T, q, t, X, plane_nd, obs_ptr, obs_cam, obs_uv, intr, sigma_px, sigma_plane, fixed_cam, nullptr, device, out);
} LVBA_ABI_END("lvba_visual_create")

int lvba_visual_destroy(lvba_visual_problem* p) LVBA_ABI_BEGIN {
  if (!p) return LVBA_OK;
  cudaSetDevice(p->device);
  delete p;
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_destroy")

int lvba_visual_set_state(lvba_visual_problem* p, const double* q, const double* t, const double* X) LVBA_ABI_BEGIN {
  if (!p || !q || !t || (p->T > 0 && !X)) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_CUDA(cudaSetDevice(p->device));
  LVBA_TRY(p->q.upload(q, (size_t)p->M * 4, p->stream, &p->h2d)); LVBA_TRY(p->qc.upload(q, (size_t)p->M * 4, p->stream));
  LVBA_TRY(p->t.upload(t, (size_t)p->M * 3, p->stream, &p->h2d)); LVBA_TRY(p->tc.upload(t, (size_t)p->M * 3, p->stream));
  LVBA_TRY(p->X.upload(X, (size_t)p->T * 3, p->stream, &p->h2d)); LVBA_TRY(p->Xc.upload(X, (size_t)p->T * 3, p->stream));
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_set_state")

int lvba_visual_get_state(lvba_visual_problem* p, double* q, double* t, double* X) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_CUDA(cudaSetDevice(p->device));
  if (q) LVBA_CUDA(cudaMemcpyAsync(q, p->q.p, (size_t)p->M * 4 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  if (t) LVBA_CUDA(cudaMemcpyAsync(t, p->t.p, (size_t)p->M * 3 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  if (X && p->T > 0) {
    if (lvba::comm().active()) {
      // landmarks are sharded: gather every rank's updates (disjoint) with one all-reduce of the deltas
      lvba::DevBuf<double> delta, merged;
      const long long n3 = (long long)p->T * 3;
      LVBA_TRY(delta.alloc((size_t)n3)); LVBA_TRY(merged.alloc((size_t)n3));
      LVBA_TRY(delta.zero(p->stream));
      if (p->Tv > 0) { lvba::visual_delta_kernel<<<(unsigned)((p->Tv * 3 + 255) / 256), 256, 0, p->stream>>>(p->Tv, p->trk_id.p, p->X.p, p->X0.p, delta.p); ++p->launches; }
      LVBA_TRY(lvba::comm().allreduce_sum(delta.p, (size_t)n3, p->stream));
      lvba::visual_add_kernel<<<(unsigned)((n3 + 255) / 256), 256, 0, p->stream>>>(n3, p->X0.p, delta.p, merged.p); ++p->launches;
      LVBA_CUDA(cudaMemcpyAsync(X, merged.p, (size_t)n3 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
      LVBA_CUDA(cudaStreamSynchronize(p->stream));
    } else {
      LVBA_CUDA(cudaMemcpyAsync(X, p->X.p, (size_t)p->T * 3 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    }
  }
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  p->d2h += (int64_t)p->M * 56 + p->T * 24;
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_get_state")

int lvba_visual_cost(lvba_visual_problem* p, double* cost) LVBA_ABI_BEGIN {
  if (!p || !cost) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::visual_check_usable(p));
  LVBA_CUDA(cudaSetDevice(p->device));
  cudaStream_t s = p->stream;
  if (p->robust()) lvba::visual_cost_t<true>(p, p->state(), p->scal.p + 8);
  else lvba::visual_cost_t<false>(p, p->state(), p->scal.p + 8);
  if (lvba::comm().active()) LVBA_TRY(lvba::comm().allreduce_sum(p->scal.p + 8, 1, s));
  LVBA_CUDA(cudaMemcpyAsync(p->h_scal, p->scal.p + 8, sizeof(double), cudaMemcpyDeviceToHost, s));
  LVBA_CUDA(cudaStreamSynchronize(s));
  *cost = p->h_scal[0];
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_cost")

int lvba_visual_step(lvba_visual_problem* p, double radius, int32_t jacobi_scaling, int32_t recompute_scale,
                     double* cam_step, double* pt_step, double* model_cost_change, double* cost) LVBA_ABI_BEGIN {
  if (!p || !(radius > 0)) return lvba::fail(LVBA_ERR_INVALID_ARG, "bad argument");
  LVBA_TRY(lvba::visual_check_usable(p));
  LVBA_CUDA(cudaSetDevice(p->device));
  if (recompute_scale || !p->lm.have_scale) LVBA_TRY(lvba::visual_compute_scale(p, jacobi_scaling));
  LVBA_CUDA(cudaMemsetAsync(p->cam_step.p, 0, (size_t)p->M * 6 * sizeof(double), p->stream));
  if (p->T > 0) LVBA_CUDA(cudaMemsetAsync(p->pt_step.p, 0, (size_t)p->T * 3 * sizeof(double), p->stream));
  LVBA_TRY(lvba::visual_linearize_solve(p, radius, true));
  if (cam_step) LVBA_CUDA(cudaMemcpyAsync(cam_step, p->cam_step.p, (size_t)p->M * 6 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  if (pt_step && p->T > 0) LVBA_CUDA(cudaMemcpyAsync(pt_step, p->pt_step.p, (size_t)p->T * 3 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  if (model_cost_change) *model_cost_change = p->h_scal[2];
  if (cost) *cost = p->h_scal[0];
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_step")

int lvba_visual_structure(lvba_visual_problem* p, int32_t* n_active, int32_t* cam_of_row, int64_t* nblocks, int32_t* brow, int32_t* bcol) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::visual_check_usable(p));
  if (n_active) *n_active = p->n_rows;
  if (cam_of_row) for (int r = 0; r < p->n_rows; ++r) cam_of_row[r] = p->cam_of_row[r];
  if (nblocks) *nblocks = p->env.nblocks;
  if (brow && bcol)
    for (int r = 0; r < p->env.n; ++r)
      for (int c = p->env.first[r]; c <= r; ++c) {
        const long long b = p->env.row_start[r] + (c - p->env.first[r]);
        brow[b] = r; bcol[b] = c;
      }
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_structure")

int lvba_visual_get_system(lvba_visual_problem* p, double* rhs, double* blocks) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::visual_check_usable(p));
  LVBA_CUDA(cudaSetDevice(p->device));
  if (rhs && p->n_rows > 0) LVBA_CUDA(cudaMemcpyAsync(rhs, p->rhs.p, (size_t)p->n_rows * 6 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  if (blocks && p->env.nblocks > 0) LVBA_CUDA(cudaMemcpyAsync(blocks, p->S.p, (size_t)p->env.nblocks * 36 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_get_system")

int lvba_visual_reset_lm(lvba_visual_problem* p, const lvba_visual_opts* opts) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::visual_check_usable(p));
  lvba_visual_opts o;
  if (opts) o = *opts; else lvba_visual_default_opts(&o);
  LVBA_TRY(lvba::visual_set_mode(p, o));
  p->opts = o;
  p->lm.reset(o);
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_reset_lm")

int lvba_visual_reset_state(lvba_visual_problem* p) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_CUDA(cudaSetDevice(p->device));
  cudaStream_t s = p->stream;
  const size_t nq = (size_t)p->M * 4 * sizeof(double), nt = (size_t)p->M * 3 * sizeof(double), nx = (size_t)p->T * 3 * sizeof(double);
  LVBA_CUDA(cudaMemcpyAsync(p->q.p, p->q0.p, nq, cudaMemcpyDeviceToDevice, s)); LVBA_CUDA(cudaMemcpyAsync(p->qc.p, p->q0.p, nq, cudaMemcpyDeviceToDevice, s));
  LVBA_CUDA(cudaMemcpyAsync(p->t.p, p->t0.p, nt, cudaMemcpyDeviceToDevice, s)); LVBA_CUDA(cudaMemcpyAsync(p->tc.p, p->t0.p, nt, cudaMemcpyDeviceToDevice, s));
  if (nx) { LVBA_CUDA(cudaMemcpyAsync(p->X.p, p->X0.p, nx, cudaMemcpyDeviceToDevice, s)); LVBA_CUDA(cudaMemcpyAsync(p->Xc.p, p->X0.p, nx, cudaMemcpyDeviceToDevice, s)); }
  std::copy(p->intr0, p->intr0 + 8, p->intr);
  std::copy(p->intr0, p->intr0 + 8, p->intr_c);
  lvba::visual_intr_forget(p);
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_reset_state")

int lvba_visual_iterate(lvba_visual_problem* p, int32_t n_iter, lvba_summary* summary) LVBA_ABI_BEGIN {
  if (!p || n_iter < 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "bad argument");
  LVBA_TRY(lvba::visual_check_usable(p));
  LVBA_CUDA(cudaSetDevice(p->device));
  return lvba::visual_iterate_impl(p, n_iter, summary);
} LVBA_ABI_END("lvba_visual_iterate")

int lvba_visual_counts(lvba_visual_problem* p, int64_t* nnz_valid, int64_t* n_valid_tracks, int64_t* n_blocks_env, int64_t* n_pairs) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::visual_check_usable(p));
  if (nnz_valid) *nnz_valid = p->nnz;
  if (n_valid_tracks) *n_valid_tracks = p->Tv;
  if (n_blocks_env) *n_blocks_env = p->env.nblocks;
  if (n_pairs) *n_pairs = p->n_pairs;
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_counts")

int lvba_visual_big_counts(lvba_visual_problem* p, int64_t* n_big, int64_t* n_big_obs, int64_t* n_big_pairs) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::visual_check_usable(p));
  if (n_big) *n_big = p->n_big;
  if (n_big_obs) *n_big_obs = p->n_big_obs;
  if (n_big_pairs) *n_big_pairs = p->n_big_pairs;
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_big_counts")

int lvba_visual_lm(int32_t M, int64_t T, double* q, double* t, double* X, const double* plane_nd, const int64_t* obs_ptr,
                   const int32_t* obs_cam, const float* obs_uv, const double intr[8], double sigma_px, double sigma_plane,
                   int32_t fixed_cam, const lvba_visual_opts* opts, lvba_summary* summary) LVBA_ABI_BEGIN {
  const double t0 = lvba::wall_ms();
  lvba_visual_opts o;
  if (opts) o = *opts; else lvba_visual_default_opts(&o);
  LVBA_TRY(lvba::visual_check_loss(o));                       // before any device work: the buffers stay untouched
  if (o.refine_intrinsics)
    return lvba::fail(LVBA_ERR_INVALID_ARG, "refine_intrinsics needs a handle (lvba_visual_reset_lm): the one-shot call's intr is const");
  LVBA_TRY(lvba::visual_check_mask(M > 0 && !lvba::visual_mask(M, o.cam_fixed).empty()));
  lvba_visual_problem* p = nullptr;
  // planned once, with the constant cameras: the reset below finds the handle's mask equal to the options'
  int rc = lvba::visual_create_impl(M, T, q, t, X, plane_nd, obs_ptr, obs_cam, obs_uv, intr, sigma_px, sigma_plane, fixed_cam, o.cam_fixed,
                                    o.device, &p);
  if (rc != LVBA_OK) return rc;
  return lvba::lm_one_shot(p, o, p->Tv > 0, lvba_visual_reset_lm, lvba_visual_iterate, lvba_visual_destroy,
                           [&] { return lvba_visual_get_state(p, q, t, X); }, t0, summary);   // write-back, src/lvba_system.cpp:1651-1665
} LVBA_ABI_END("lvba_visual_lm")


int lvba_visual_obs_residuals(lvba_visual_problem* p, double* sq_res) LVBA_ABI_BEGIN {
  if (!p || !sq_res) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::visual_check_obs_calls(p));
  LVBA_CUDA(cudaSetDevice(p->device));
  LVBA_TRY(lvba::visual_obs_sq_dev(p));
  const int64_t n_obs = p->h_obs_ptr[(size_t)p->T];
  LVBA_CUDA(cudaMemcpyAsync(sq_res, p->obs_sq.p, (size_t)n_obs * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  p->d2h += n_obs * 8;
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_obs_residuals")

int lvba_visual_remove_observations(lvba_visual_problem* p, const uint8_t* remove, int32_t min_track_len, int64_t* n_obs_left,
                                    int64_t* n_tracks_left) LVBA_ABI_BEGIN {
  if (!p || !remove) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::visual_check_obs_calls(p));
  if (min_track_len < 1) return lvba::fail(LVBA_ERR_INVALID_ARG, "min_track_len=%d: it must be >= 1", (int)min_track_len);
  LVBA_CUDA(cudaSetDevice(p->device));
  const int64_t n_obs = p->h_obs_ptr[(size_t)p->T];
  lvba::DevBuf<uint8_t> d_mask;
  LVBA_TRY(d_mask.upload(remove, (size_t)n_obs, p->stream, &p->h2d));
  const int rc = lvba::visual_remove_impl(p, d_mask.p, 0.0, min_track_len, nullptr, n_obs_left, n_tracks_left, nullptr, nullptr);
  cudaStreamSynchronize(p->stream);                            // d_mask is idle before it is parked
  return rc;
} LVBA_ABI_END("lvba_visual_remove_observations")

int lvba_visual_remove_outliers(lvba_visual_problem* p, double max_err_px, int32_t min_track_len, uint8_t* removed,
                                int64_t* n_removed_obs, int64_t* n_removed_tracks) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::visual_check_obs_calls(p));
  if (!(std::isfinite(max_err_px) && max_err_px > 0.0))
    return lvba::fail(LVBA_ERR_INVALID_ARG, "max_err_px=%g: it must be finite and > 0", max_err_px);
  if (min_track_len < 1) return lvba::fail(LVBA_ERR_INVALID_ARG, "min_track_len=%d: it must be >= 1", (int)min_track_len);
  LVBA_CUDA(cudaSetDevice(p->device));
  const double e = max_err_px / p->sigma_px;
  // an overflowing threshold stays finite, so that +inf (the depth test failed) is still above it
  const double tau = std::min(e * e, DBL_MAX);
  LVBA_TRY(lvba::visual_obs_sq_dev(p));
  return lvba::visual_remove_impl(p, nullptr, tau, min_track_len, removed, nullptr, nullptr, n_removed_obs, n_removed_tracks);
} LVBA_ABI_END("lvba_visual_remove_outliers")

int lvba_visual_get_intrinsics(lvba_visual_problem* p, double intr[8]) LVBA_ABI_BEGIN {
  if (!p || !intr) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  std::copy(p->intr, p->intr + 8, intr);
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_get_intrinsics")

int lvba_visual_set_intrinsics(lvba_visual_problem* p, const double intr[8]) LVBA_ABI_BEGIN {
  if (!p || !intr) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  for (int i = 0; i < 8; ++i)
    if (!std::isfinite(intr[i])) return lvba::fail(LVBA_ERR_INVALID_ARG, "intr[%d] = %g is not finite", i, intr[i]);
  std::copy(intr, intr + 8, p->intr);
  std::copy(intr, intr + 8, p->intr_c);
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_set_intrinsics")

int lvba_visual_get_intrinsics_system(lvba_visual_problem* p, int32_t* k, double* border, double* corner, double* rhs,
                                      double* step) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  LVBA_TRY(lvba::visual_check_usable(p));
  int fi[8], nk = 0;
  for (int i = 0; i < 8; ++i)
    if ((p->intr_mask >> i) & 1u) fi[nk++] = i;
  if (k) *k = nk;
  if (step) std::copy(p->intr_step, p->intr_step + 8, step);
  if (nk == 0 || !p->intr_have_sys || !(border || corner || rhs)) return LVBA_OK;
  LVBA_CUDA(cudaSetDevice(p->device));
  const size_t n6 = (size_t)p->n_rows * 6;
  std::vector<double> B(8 * n6), sys(lvba::vintr::kSys);
  if (n6) LVBA_CUDA(cudaMemcpyAsync(B.data(), p->intr_B.p, B.size() * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  LVBA_CUDA(cudaMemcpyAsync(sys.data(), p->intr_sys.p, sys.size() * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  if (border)
    for (size_t m = 0; m < n6; ++m)
      for (int a = 0; a < nk; ++a) border[m * nk + a] = B[fi[a] * n6 + m];
  for (int a = 0; a < nk; ++a) {
    if (rhs) rhs[a] = sys[lvba::vintr::kRhs + fi[a]];
    if (corner)
      for (int b = 0; b < nk; ++b) corner[a * nk + b] = sys[lvba::vintr::kC + lvba::vintr::ut(std::min(fi[a], fi[b]), std::max(fi[a], fi[b]))];
  }
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_get_intrinsics_system")

}  // extern "C"
