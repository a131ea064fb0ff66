// visual_api.cuh — host side of boundary B2 (include/lvba_b200.h): problem set-up mirroring the Ceres
// problem built at reference src/lvba_system.cpp:1578-1640 and the trust-region LM loop of
// ceres-solver 2.1.0 (TrustRegionMinimizer + LevenbergMarquardtStrategy, SURVEY.md Q10/A.3).
#pragma once
#include <cmath>
#include <memory>

#include "exec.cuh"
#include "runtime.cuh"   // (pulls comm.cuh in)
#include "visual.cuh"
#include "visual_big.h"

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
  lvba::PhaseTimers timers;
  double* h_scal = nullptr;
  int64_t launches = 0, h2d = 0, d2h = 0;
  double ms_setup = 0.0;
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

inline bool plane_valid(const double* p) {   // has_valid_plane, src/lvba_system.cpp:1598
  for (int i = 0; i < 4; ++i) if (!std::isfinite(p[i])) return false;
  return std::fabs(p[0]) > 1e-6 || std::fabs(p[1]) > 1e-6 || std::fabs(p[2]) > 1e-6;
}

inline int visual_create_impl(int32_t M, int64_t T, const double* q, const double* t, const double* X,
                              const double* plane_nd, const int64_t* obs_ptr, const int32_t* obs_cam,
                              const float* obs_uv, const double intr[8], double sigma_px, double sigma_plane,
                              int32_t fixed_cam, int32_t device, lvba_visual_problem** out) {
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
  const bool tlog = getenv("LVBA_SETUP_TIMING") != nullptr;
  double tprev = t_begin;
  auto lap = [&](const char* what) { if (tlog) { cudaStreamSynchronize(nullptr); const double tn = wall_ms(); fprintf(stderr, "[visual setup] %-26s %8.2f ms\n", what, tn - tprev); tprev = tn; } };
  std::unique_ptr<lvba_visual_problem> P(new lvba_visual_problem());
  P->M = M; P->T = T; P->fixed_cam = fixed_cam;
  for (int i = 0; i < 8; ++i) P->intr[i] = intr[i];
  P->sigma_px = sigma_px; P->sigma_pl = sigma_plane;
  LVBA_CUDA(cudaGetDevice(&P->device));
  LVBA_CUDA(cudaStreamCreateWithFlags(&P->stream, cudaStreamNonBlocking));
  P->timers.stream = P->stream;
  LVBA_TRY(pinned_pool().take(16 * sizeof(double), (void**)&P->h_scal));
  cudaStream_t s = P->stream;

  // ---- valid landmarks, active cameras (src/lvba_system.cpp:1582-1583, 1598-1603; SURVEY.md Q11)
  std::vector<int64_t> valid;
  std::vector<char> cam_used(M, 0);
  {
    std::vector<char> is_valid((size_t)T, 0), used_w((size_t)kMaxSetupThreads * (size_t)M, 0);
    parallel_chunks(T, 1 << 13, [&](int64_t i0, int64_t i1, int w) {
      char* used = used_w.data() + (size_t)w * (size_t)M;
      for (int64_t i = i0; i < i1; ++i) {
        if (!plane_valid(plane_nd + 4 * i)) continue;
        is_valid[(size_t)i] = 1;
        for (int64_t q_ = obs_ptr[i]; q_ < obs_ptr[i + 1]; ++q_) used[obs_cam[q_]] = 1;
      }
    });
    for (int w = 0; w < kMaxSetupThreads; ++w)
      for (int c = 0; c < M; ++c) cam_used[c] |= used_w[(size_t)w * (size_t)M + c];
    for (int64_t i = 0; i < T; ++i) if (is_valid[(size_t)i]) valid.push_back(i);
  }
  if (fixed_cam >= 0 && fixed_cam < M) cam_used[fixed_cam] = 0;
  std::vector<int> row_of_cam(M, -1);
  for (int c = 0; c < M; ++c) if (cam_used[c]) { row_of_cam[c] = (int)P->cam_of_row.size(); P->cam_of_row.push_back(c); }
  P->n_rows = (int)P->cam_of_row.size();
  const int64_t Tv_all = (int64_t)valid.size();

  lap("valid landmarks / rows");
  // ---- envelope of the reduced camera system over ALL valid landmarks
  std::vector<int> first_raw(std::max(P->n_rows, 1));
  for (int r = 0; r < P->n_rows; ++r) first_raw[r] = r;
  std::vector<int> min_row(Tv_all, 0), min_sys_row(Tv_all, 0);
  {
    const size_t nr = first_raw.size();
    std::vector<int> first_w((size_t)kMaxSetupThreads * nr);
    for (int w = 0; w < kMaxSetupThreads; ++w) std::copy(first_raw.begin(), first_raw.end(), first_w.begin() + (size_t)w * nr);
    parallel_chunks(Tv_all, 1 << 13, [&](int64_t k0, int64_t k1, int w) {
      int* fr = first_w.data() + (size_t)w * nr;
      for (int64_t k = k0; k < k1; ++k) {
        const int64_t i = valid[k];
        int m = INT32_MAX, mcam = INT32_MAX;
        for (int64_t q_ = obs_ptr[i]; q_ < obs_ptr[i + 1]; ++q_) {
          const int r = row_of_cam[obs_cam[q_]];
          if (r >= 0) m = std::min(m, r);
          mcam = std::min(mcam, (int)obs_cam[q_]);
        }
        min_row[k] = (mcam == INT32_MAX) ? 0 : mcam;      // shard key: lowest camera index
        min_sys_row[k] = (m == INT32_MAX) ? 0 : m;        // row-owned reduced system: lowest row of the landmark's clique
        if (m == INT32_MAX) continue;
        for (int64_t q_ = obs_ptr[i]; q_ < obs_ptr[i + 1]; ++q_) {
          const int r = row_of_cam[obs_cam[q_]];
          if (r >= 0) fr[r] = std::min(fr[r], m);
        }
      }
    });
    for (int w = 0; w < kMaxSetupThreads; ++w)
      for (size_t r = 0; r < nr; ++r) first_raw[r] = std::min(first_raw[r], first_w[(size_t)w * nr + r]);
  }
  if (P->n_rows > 0) {
    first_raw.resize(P->n_rows);
    LVBA_TRY(P->env.build(first_raw, s, &P->h2d));
    LVBA_TRY(P->solver.prepare(P->env, s));
  }

  lap("envelope + solver prepare");
  // ---- shard (SURVEY.md §8e): landmark -> owner of its lowest camera index
  Comm& cm = comm();
  std::vector<int64_t> own;                                    // indices into valid
  for (int64_t k = 0; k < Tv_all; ++k)
    if (!cm.active() || (P->solver.dist() ? P->solver.dist_owner(min_sys_row[k]) : shard_owner(min_row[k], M, cm.n_ranks)) == cm.rank)
      own.push_back(k);
  const int64_t Tv = (int64_t)own.size();
  // the landmarks in the order of the lowest system row of their clique: the landmarks of a build tile then share cameras,
  // whose S blocks and rows the tile sums on chip (visual_tiles.h).  Landmarks with more than kSlots observations go after all
  // small ones, in the same order: they take the passes of visual_big.h.
  std::vector<int64_t> mine((size_t)Tv);
  int64_t Tv_small = 0;
  {
    std::vector<int> key((size_t)Tv);
    for (int64_t j = 0; j < Tv; ++j) key[j] = min_sys_row[own[j]];
    const std::vector<int64_t> order = tiles::order_by_key(std::max(P->n_rows, 1), key.data(), Tv);
    auto is_big = [&](int64_t i) { return obs_ptr[i + 1] - obs_ptr[i] > kSlots; };
    for (int64_t j = 0; j < Tv; ++j) if (!is_big(valid[own[order[j]]])) mine[Tv_small++] = valid[own[order[j]]];
    int64_t w = Tv_small;
    for (int64_t j = 0; j < Tv; ++j) if (is_big(valid[own[order[j]]])) mine[w++] = valid[own[order[j]]];
  }
  P->Tv = Tv;
  P->Tv_small = Tv_small;
  P->n_big = Tv - Tv_small;
  std::vector<int> trk_ptr(Tv + 1, 0), trk_id(Tv);
  for (int64_t k = 0; k < Tv; ++k) {
    trk_id[k] = (int)mine[k];
    trk_ptr[k + 1] = trk_ptr[k] + (int)(obs_ptr[mine[k] + 1] - obs_ptr[mine[k]]);
  }
  const long long nnz = trk_ptr[Tv];
  P->nnz = nnz;
  lap("landmark list");
  // ---- back-substitution / cost batches (<= kSlots observations) and build tiles (<= kVisTileSlots observations)
  const std::vector<int> batch_trk = tiles::cut_ranges(Tv_small, trk_ptr.data(), nullptr, kSlots, kMaxTrkPerBatch);
  const std::vector<int> tile_trk = tiles::cut_ranges(Tv_small, trk_ptr.data(), nullptr, kVisTileSlots, kMaxTrkPerTile);
  P->n_batches = (int)batch_trk.size() - 1;
  P->n_tiles = (int)tile_trk.size() - 1;
  lap("batches + tiles");

  // ---- upload the caller's arrays as they are; gather the per-observation arrays and build the destination table on the device
  LVBA_TRY(P->trk_ptr.upload(trk_ptr, s, &P->h2d));
  LVBA_TRY(P->batch_trk.upload(batch_trk, s, &P->h2d));
  LVBA_TRY(P->tile_trk.upload(tile_trk, s, &P->h2d));
  if (Tv > 0) {
    const int64_t nnz_all = obs_ptr[T];
    DevBuf<long long> d_obs_ptr;
    DevBuf<int> d_raw_cam, d_row_of_cam;
    DevBuf<float2> d_raw_uv;
    DevBuf<double> d_raw_plane;
    static_assert(sizeof(long long) == sizeof(int64_t), "obs_ptr is uploaded as it is");
    LVBA_TRY(d_obs_ptr.upload(reinterpret_cast<const long long*>(obs_ptr), (size_t)T + 1, s, &P->h2d));
    LVBA_TRY(d_raw_cam.upload(obs_cam, (size_t)nnz_all, s, &P->h2d));
    LVBA_TRY(d_raw_uv.upload(reinterpret_cast<const float2*>(obs_uv), (size_t)nnz_all, s, &P->h2d));
    LVBA_TRY(d_raw_plane.upload(plane_nd, (size_t)T * 4, s, &P->h2d));
    LVBA_TRY(d_row_of_cam.upload(row_of_cam, s, &P->h2d));
    LVBA_TRY(P->trk_id.upload(trk_id, s, &P->h2d));
    LVBA_TRY(P->obs_cam.alloc((size_t)nnz)); LVBA_TRY(P->obs_row.alloc((size_t)nnz)); LVBA_TRY(P->obs_uv.alloc((size_t)nnz));
    LVBA_TRY(P->plane.alloc((size_t)Tv * 4));
    visual_gather_kernel<<<(unsigned)((Tv + 127) / 128), 128, 0, s>>>(Tv, P->trk_id.p, P->trk_ptr.p, d_obs_ptr.p, d_raw_cam.p, d_raw_uv.p,
                                                                     d_raw_plane.p, d_row_of_cam.p, P->obs_cam.p, P->obs_row.p, P->obs_uv.p, P->plane.p);
    LVBA_CUDA(cudaGetLastError());
    ++P->launches;
    if (Tv_small > 0) {                                        // the destination table covers the small landmarks only
      CudaExec ex;
      ex.stream = s;
      DevBuf<long long> d_pair_cnt, d_trk_pair;                // ordered observation pairs before every local landmark
      LVBA_TRY(d_pair_cnt.alloc((size_t)Tv_small + 1));
      LVBA_TRY(d_trk_pair.alloc((size_t)Tv_small + 1));
      LVBA_TRY(ex.for_each(Tv_small + 1, tiles::VisPairCountF{P->trk_ptr.p, Tv_small, d_pair_cnt.p}));
      LVBA_TRY(ex.exclusive_scan(d_pair_cnt.p, d_trk_pair.p, Tv_small + 1));
      long long n_ordered = 0;
      for (int64_t k = 0; k < Tv_small; ++k) n_ordered += (long long)(trk_ptr[k + 1] - trk_ptr[k]) * (trk_ptr[k + 1] - trk_ptr[k] - 1);
      const tiles::VisTableIn tin{P->n_tiles, P->n_rows, P->env.nblocks, P->tile_trk.p, P->trk_ptr.p, P->obs_row.p, d_trk_pair.p,
                                  P->env.d_first.p, P->env.d_row_start.p};
      LVBA_TRY(tiles::sort_runs(ex, n_ordered, P->n_tiles, (uint64_t)P->env.nblocks, tiles::VisPairKeyF{tin}, P->prun));
      LVBA_TRY(tiles::sort_runs(ex, (int64_t)trk_ptr[Tv_small], P->n_tiles, (uint64_t)P->n_rows, tiles::ObsKeyF{tin}, P->drun));
      int64_t np = 0;
      LVBA_TRY(ex.fetch(&np, P->prun.run_ptr.p + P->prun.n_runs, 1));
      P->n_pairs = np;
      P->launches += ex.launches;
    }
    if (P->n_big > 0) {
      // pair items of the big landmarks (K (K - 1) each) and their camera-pair contributions: an unordered pair of observations
      // of two distinct rows once, of one row in both orders, i.e. C(n, 2) + sum_row C(n_row, 2) over the n observations of
      // non-constant cameras
      std::vector<int64_t> bpp((size_t)P->n_big + 1, 0);
      std::vector<int> rows;
      for (int64_t b = 0; b < P->n_big; ++b) {
        const int64_t i = mine[Tv_small + b], K = obs_ptr[i + 1] - obs_ptr[i];
        bpp[b + 1] = bpp[b] + K * (K - 1);
        rows.clear();
        for (int64_t q_ = obs_ptr[i]; q_ < obs_ptr[i + 1]; ++q_) if (row_of_cam[obs_cam[q_]] >= 0) rows.push_back(row_of_cam[obs_cam[q_]]);
        std::sort(rows.begin(), rows.end());
        const long long n = (long long)rows.size();
        long long contrib = n * (n - 1) / 2;
        for (size_t a = 0; a < rows.size();) {
          size_t e = a;
          while (e < rows.size() && rows[e] == rows[a]) ++e;
          contrib += (long long)(e - a) * (long long)(e - a - 1) / 2;
          a = e;
        }
        P->n_pairs += contrib;
      }
      P->n_big_obs = nnz - trk_ptr[Tv_small];
      P->n_big_pairs = bpp.back();
      LVBA_TRY(P->big_pair_ptr.upload(bpp, s, &P->h2d));
      LVBA_TRY(P->big_obs.alloc((size_t)P->n_big_obs * vbig::kObs));
      LVBA_TRY(P->big_params.alloc((size_t)P->n_big * kTrkParams));
    }
  } else {
    P->n_pairs = 0;
  }
  lap("device gather + destination table");
  if (P->n_rows > 0) LVBA_TRY(P->d_cam_of_row.upload(P->cam_of_row, s, &P->h2d));
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
  const size_t n6 = (size_t)std::max(P->n_rows, 1) * 6;
  LVBA_TRY(P->S.alloc((size_t)std::max<long long>(P->env.nblocks, 1) * 36));
  LVBA_TRY(P->rhs.alloc(n6)); LVBA_TRY(P->y.alloc(n6)); LVBA_TRY(P->dadd.alloc(n6));
  LVBA_TRY(P->cam_colsq.alloc(n6)); LVBA_TRY(P->cam_grad.alloc(n6)); LVBA_TRY(P->s_cam.alloc(n6));
  LVBA_TRY(P->s_pt.alloc((size_t)std::max<int64_t>(Tv, 1) * 3));
  LVBA_TRY(P->pt_colsq.alloc((size_t)std::max<int64_t>(Tv, 1) * 3));
  const size_t nb = (size_t)std::max<long long>(std::max(P->n_batches, P->n_tiles) + P->n_big, 1);   // partial slots, big landmarks last
  LVBA_TRY(P->batch_cost.alloc(nb)); LVBA_TRY(P->batch_gmax.alloc(nb)); LVBA_TRY(P->batch_out.alloc(nb * 4));
  LVBA_TRY(P->cam_out.alloc((size_t)((P->n_rows + 127) / 128 + 1) * 2));
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

// Deterministic mode: the records of the build and their destinations.  Records of S: the tiles' pair runs, the tiles' row runs,
// the big landmarks' observations, the big landmarks' ordered pairs; records of the camera rows: the tiles' row runs, the big
// landmarks' observations.  Each set in its enumeration order, so that every destination's records come in ascending (tile, run)
// order, then in item order.  Observations of constant cameras and pairs outside the lower envelope get a record without a
// destination.
inline int visual_det_setup(lvba_visual_problem* P) {
  if (P->det_ready) return LVBA_OK;
  const int64_t npr = P->prun.n_runs, ndr = P->drun.n_runs;
  const int64_t nS = npr + ndr + P->n_big_obs + P->n_big_pairs, nG = ndr + P->n_big_obs;
  if (nS >= (int64_t)1 << 32) return fail(LVBA_ERR_UNSUPPORTED, "deterministic mode: %lld contributions to S (at most 2^32)", (long long)nS);
  CudaExec ex;
  ex.stream = P->stream;
  LVBA_TRY(tiles::fixed_sum_alloc(P->det_S, nS, 36));
  LVBA_TRY(tiles::fixed_sum_alloc(P->det_G, nG, 18));
  LVBA_TRY(P->det_C.alloc((size_t)std::max<int64_t>(nG, 1) * 6));
  if (P->n_tiles > 0) {
    const tiles::VisTableIn tin{P->n_tiles, P->n_rows, P->env.nblocks, P->tile_trk.p, P->trk_ptr.p, P->obs_row.p, nullptr,
                                P->env.d_first.p, P->env.d_row_start.p};
    LVBA_TRY(ex.for_each(npr, tiles::VisPairRunDstF{tin, P->prun.tile_run.p, P->prun.run_ptr.p, P->prun.code.p, P->det_S.dst.p}));
    LVBA_TRY(ex.for_each(ndr, tiles::ObsRunDstF{tin, P->drun.tile_run.p, P->drun.run_ptr.p, P->drun.code.p, P->det_S.dst.p + npr,
                                                P->det_G.dst.p}));
  }
  if (P->n_big > 0) {
    const VisualView vv = P->view();
    const vbig::View bv = P->big_view();
    LVBA_TRY(ex.for_each(P->n_big_obs, vbig::ObsDstF{vv, bv, P->env.nblocks, P->n_rows, P->det_S.dst.p + npr + ndr, P->det_G.dst.p + ndr}));
    LVBA_TRY(ex.for_each(P->n_big_pairs, vbig::PairDstF{vv, bv, P->env.nblocks, P->det_S.dst.p + npr + ndr + P->n_big_obs}));
  }
  LVBA_TRY(tiles::fixed_sum_index(ex, P->det_S, P->env.nblocks));
  LVBA_TRY(tiles::fixed_sum_index(ex, P->det_G, P->n_rows));
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

// the LM mode of the handle (lvba_visual_reset_lm and the one-shot call): deterministic mode and the robust losses
inline int visual_set_mode(lvba_visual_problem* P, const lvba_visual_opts& o) {
  LVBA_TRY(visual_check_loss(o));
  if (o.deterministic && comm().active())
    return fail(LVBA_ERR_UNSUPPORTED, "deterministic mode runs on one GPU: the multi-GPU sums of NCCL have no fixed order");
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
  return LVBA_OK;
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
  LVBA_CUDA(cudaGetLastError());
  P->lm.have_scale = true;
  return LVBA_OK;
}
inline int visual_compute_scale(lvba_visual_problem* P, int enabled) {
  return P->robust() ? visual_compute_scale_t<true>(P, enabled) : visual_compute_scale_t<false>(P, enabled);
}

// 1/2 sum r^2 (with a loss: 1/2 sum rho) at the state `st` into *out (device): batches, big landmarks, reduction
template <bool kLoss>
inline void visual_cost_t(lvba_visual_problem* P, const VisualState& st, double* out) {
  cudaStream_t s = P->stream;
  if (P->n_batches > 0) {
    if constexpr (kLoss) visual_cost_loss_kernel<<<P->n_batches, kSlots, 0, s>>>(P->view(), st, P->batch_cost.p);
    else visual_cost_kernel<<<P->n_batches, kSlots, 0, s>>>(P->view(), st, P->batch_cost.p);
    ++P->launches;
  }
  if (P->n_big > 0) wide_pass(s, P->n_big, vbig::CostPass<kLoss>{P->view(), P->big_view(), st, P->batch_cost.p + P->n_batches}, &P->launches);
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
  P->timers.end();
  ++P->lm.builds;
  P->timers.begin(PH_SOLVE);
  if (P->n_rows > 0) {
    visual_cam_diag_kernel<<<1, 256, 0, s>>>(6 * P->n_rows, P->cam_colsq.p, P->cam_grad.p, P->s_cam.p, P->opts.min_lm_diagonal,
                                             P->opts.max_lm_diagonal, radius, P->dadd.p, P->scal.p + 5);
    ++P->launches;
    LVBA_CUDA(cudaMemcpyAsync(P->solver.z.p, P->rhs.p, (size_t)P->n_rows * 6 * sizeof(double), cudaMemcpyDeviceToDevice, s));
    LVBA_TRY(P->solver.solve(P->env, P->S.p, P->dadd.p, P->y.p, s, &P->launches));
  }
  P->timers.end();
  P->timers.begin(PH_RESID);
  if (P->n_batches > 0) {
    visual_backsub_kernel<kLoss><<<P->n_batches, kSlots, visual_backsub_smem_bytes(), s>>>(
        P->view(), P->state(), lm, P->y.p, P->Xc.p, want_steps ? P->pt_step.p : nullptr, P->batch_out.p);
    ++P->launches;
  }
  if (P->n_big > 0)
    wide_pass(s, P->n_big, vbig::BacksubPass<kLoss>{P->view(), P->big_view(), P->state(), lm, P->big_obs.p, P->big_params.p, P->y.p,
                                                    P->Xc.p, want_steps ? P->pt_step.p : nullptr,
                                                    P->batch_out.p + 4 * (int64_t)P->n_batches}, &P->launches);
  reduce_cols_kernel<<<1, 256, 0, s>>>(P->batch_out.p, (int)(P->n_batches + P->n_big), 4, 3, P->scal.p + 2);
  ++P->launches;
  const int ncb = (P->n_rows + 127) / 128;
  if (ncb > 0) {
    visual_cam_update_kernel<<<ncb, 128, 0, s>>>(P->n_rows, P->d_cam_of_row.p, P->q.p, P->t.p, P->y.p, P->s_cam.p, P->qc.p, P->tc.p,
                                                 want_steps ? P->cam_step.p : nullptr, P->cam_out.p);
    ++P->launches;
  }
  reduce_cols_kernel<<<1, 256, 0, s>>>(P->cam_out.p, ncb, 2, 2, P->scal.p + 6);
  ++P->launches;
  if (cm.active()) LVBA_TRY(cm.allreduce_sum(P->scal.p + 2, 3, s));   // model, step^2, x^2 of the landmark shard
  visual_cost_t<kLoss>(P, P->cand(), P->scal.p + 8);                      // candidate cost
  if (cm.active()) LVBA_TRY(cm.allreduce_sum(P->scal.p + 8, 1, s));
  P->timers.end();
  LVBA_CUDA(cudaGetLastError());
  LVBA_CUDA(cudaMemcpyAsync(P->h_scal, P->scal.p, 16 * sizeof(double), cudaMemcpyDeviceToHost, s));
  LVBA_CUDA(cudaMemcpyAsync(P->h_scal + 15, P->solver.status.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  LVBA_CUDA(cudaStreamSynchronize(s));
  P->d2h += 16 * sizeof(double);
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
}

int lvba_visual_create(int32_t M, int64_t T, const double* q, const double* t, const double* X, const double* plane_nd,
                       const int64_t* obs_ptr, const int32_t* obs_cam, const float* obs_uv, const double intr[8],
                       double sigma_px, double sigma_plane, int32_t fixed_cam, int32_t device, lvba_visual_problem** out) {
  try { return lvba::visual_create_impl(M, T, q, t, X, plane_nd, obs_ptr, obs_cam, obs_uv, intr, sigma_px, sigma_plane, fixed_cam, device, out); }
  catch (const std::bad_alloc&) { return lvba::fail(LVBA_ERR_NOMEM, "host allocation failed"); }
  catch (...) { return lvba::fail(LVBA_ERR_INVALID_ARG, "unexpected exception in lvba_visual_create"); }
}

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
  LVBA_CUDA(cudaSetDevice(p->device));
  if (rhs && p->n_rows > 0) LVBA_CUDA(cudaMemcpyAsync(rhs, p->rhs.p, (size_t)p->n_rows * 6 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  if (blocks && p->env.nblocks > 0) LVBA_CUDA(cudaMemcpyAsync(blocks, p->S.p, (size_t)p->env.nblocks * 36 * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  LVBA_CUDA(cudaStreamSynchronize(p->stream));
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_get_system")

int lvba_visual_reset_lm(lvba_visual_problem* p, const lvba_visual_opts* opts) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
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
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_reset_state")

int lvba_visual_iterate(lvba_visual_problem* p, int32_t n_iter, lvba_summary* summary) LVBA_ABI_BEGIN {
  if (!p || n_iter < 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "bad argument");
  LVBA_CUDA(cudaSetDevice(p->device));
  return lvba::visual_iterate_impl(p, n_iter, summary);
} LVBA_ABI_END("lvba_visual_iterate")

int lvba_visual_counts(lvba_visual_problem* p, int64_t* nnz_valid, int64_t* n_valid_tracks, int64_t* n_blocks_env, int64_t* n_pairs) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  if (nnz_valid) *nnz_valid = p->nnz;
  if (n_valid_tracks) *n_valid_tracks = p->Tv;
  if (n_blocks_env) *n_blocks_env = p->env.nblocks;
  if (n_pairs) *n_pairs = p->n_pairs;
  return LVBA_OK;
} LVBA_ABI_END("lvba_visual_counts")

int lvba_visual_big_counts(lvba_visual_problem* p, int64_t* n_big, int64_t* n_big_obs, int64_t* n_big_pairs) LVBA_ABI_BEGIN {
  if (!p) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
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
  lvba_visual_problem* p = nullptr;
  int rc = lvba_visual_create(M, T, q, t, X, plane_nd, obs_ptr, obs_cam, obs_uv, intr, sigma_px, sigma_plane, fixed_cam, o.device, &p);
  if (rc != LVBA_OK) return rc;
  return lvba::lm_one_shot(p, o, p->Tv > 0, lvba_visual_reset_lm, lvba_visual_iterate, lvba_visual_destroy,
                           [&] { return lvba_visual_get_state(p, q, t, X); }, t0, summary);   // write-back, src/lvba_system.cpp:1651-1665
} LVBA_ABI_END("lvba_visual_lm")

}  // extern "C"
