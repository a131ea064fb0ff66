// visual_plan.h — the symbolic set-up of the visual problem handle (visual_create_impl and visual_det_setup, visual_api.cuh),
// plain C++ with no CUDA: the valid landmarks and system rows, the envelope rows, the landmark layout (order, big landmarks,
// batches, tiles), the build's destination table and the record index of deterministic mode.  The table and the index are item
// passes run by an execution policy: CudaExec (exec.cuh) in the library, the host policy of tests/emu in the CPU tests, which
// call these same functions.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <utility>
#include <vector>

#include "setup_pool.h"
#include "visual_big.h"
#include "visual_tiles.h"

#ifndef LVBA_PLAN_TRY
#define LVBA_PLAN_TRY(call) do { const int rc__ = (call); if (rc__ != 0) return rc__; } while (0)
#endif

namespace lvba {

inline bool plane_valid(const double* p) {   // has_valid_plane, src/lvba_system.cpp:1598
  for (int i = 0; i < 4; ++i) if (!std::isfinite(p[i])) return false;
  return std::fabs(p[0]) > 1e-6 || std::fabs(p[1]) > 1e-6 || std::fabs(p[2]) > 1e-6;
}

// The system rows from the cameras seen by a valid landmark (cam_used [M]): one row per such camera that is not constant, in
// ascending camera order.  Constant: fixed_cam and every c with cam_fixed[c] != 0 (cam_fixed may be null).
// row_of_cam[c] = system row of camera c (-1: constant or unseen), cam_of_row its inverse.
inline void visual_row_map(int M, std::vector<char> cam_used, int fixed_cam, const uint8_t* cam_fixed, std::vector<int>& row_of_cam,
                           std::vector<int>& cam_of_row) {
  if (fixed_cam >= 0 && fixed_cam < M) cam_used[fixed_cam] = 0;
  if (cam_fixed)
    for (int c = 0; c < M; ++c) if (cam_fixed[c]) cam_used[c] = 0;
  row_of_cam.assign(M, -1);
  cam_of_row.clear();
  for (int c = 0; c < M; ++c) if (cam_used[c]) { row_of_cam[c] = (int)cam_of_row.size(); cam_of_row.push_back(c); }
}

// Valid landmarks (a usable plane) and active cameras (seen by one, not constant), src/lvba_system.cpp:1582-1583, 1598-1603:
// valid in ascending order, the rows as visual_row_map.
inline void visual_rows(int M, int64_t T, const double* plane_nd, const int64_t* obs_ptr, const int32_t* obs_cam, int fixed_cam,
                        const uint8_t* cam_fixed, std::vector<int64_t>& valid, std::vector<int>& row_of_cam, std::vector<int>& cam_of_row) {
  std::vector<char> cam_used(M, 0);
  {
    std::vector<char> is_valid((size_t)T, 0), used_w((size_t)kMaxSetupThreads * (size_t)M, 0);
    parallel_chunks(T, 1 << 13, [&](int64_t i0, int64_t i1, int w) {
      char* used = used_w.data() + (size_t)w * (size_t)M;
      for (int64_t i = i0; i < i1; ++i) {
        if (!plane_valid(plane_nd + 4 * i)) continue;
        is_valid[(size_t)i] = 1;
        for (int64_t q = obs_ptr[i]; q < obs_ptr[i + 1]; ++q) used[obs_cam[q]] = 1;
      }
    });
    for (int w = 0; w < kMaxSetupThreads; ++w)
      for (int c = 0; c < M; ++c) cam_used[c] |= used_w[(size_t)w * (size_t)M + c];
    for (int64_t i = 0; i < T; ++i) if (is_valid[(size_t)i]) valid.push_back(i);
  }
  visual_row_map(M, std::move(cam_used), fixed_cam, cam_fixed, row_of_cam, cam_of_row);
}

// The raw envelope of the reduced camera system over the landmarks valid[0..n): first[r] = the lowest row that shares a landmark
// with row r (r when there is none; max(n_rows, 1) entries).  Per landmark k the two keys a rank's share and the layout's order
// are cut by: min_cam[k] = its lowest camera, min_row[k] = the lowest row of its clique (0 when it has none).
inline std::vector<int> visual_first_rows(int n_rows, const int64_t* valid, int64_t n, const int64_t* obs_ptr, const int32_t* obs_cam,
                                          const int* row_of_cam, std::vector<int>& min_cam, std::vector<int>& min_row) {
  std::vector<int> first(std::max(n_rows, 1));
  for (int r = 0; r < n_rows; ++r) first[r] = r;
  min_cam.assign((size_t)n, 0); min_row.assign((size_t)n, 0);
  const size_t nr = first.size();
  std::vector<int> first_w((size_t)kMaxSetupThreads * nr);
  for (int w = 0; w < kMaxSetupThreads; ++w) std::copy(first.begin(), first.end(), first_w.begin() + (size_t)w * nr);
  parallel_chunks(n, 1 << 13, [&](int64_t k0, int64_t k1, int w) {
    int* fr = first_w.data() + (size_t)w * nr;
    for (int64_t k = k0; k < k1; ++k) {
      const int64_t i = valid[k];
      int m = INT_MAX, mcam = INT_MAX;
      for (int64_t q = obs_ptr[i]; q < obs_ptr[i + 1]; ++q) {
        const int r = row_of_cam[obs_cam[q]];
        if (r >= 0) m = std::min(m, r);
        mcam = std::min(mcam, (int)obs_cam[q]);
      }
      min_cam[k] = (mcam == INT_MAX) ? 0 : mcam;
      min_row[k] = (m == INT_MAX) ? 0 : m;
      if (m == INT_MAX) continue;
      for (int64_t q = obs_ptr[i]; q < obs_ptr[i + 1]; ++q) {
        const int r = row_of_cam[obs_cam[q]];
        if (r >= 0) fr[r] = std::min(fr[r], m);
      }
    }
  });
  for (int w = 0; w < kMaxSetupThreads; ++w)
    for (size_t r = 0; r < nr; ++r) first[r] = std::min(first[r], first_w[(size_t)w * nr + r]);
  return first;
}

struct VisualLayout {
  int64_t Tv = 0, Tv_small = 0;               // local landmarks; the small ones come first
  std::vector<int> trk_ptr, trk_id;           // local CSR of the observations; trk_id = the caller's landmark
  std::vector<int> batch_trk, tile_trk;       // back-substitution / cost batches and build tiles over the small landmarks
  long long nnz = 0, n_ordered = 0;           // observations; ordered observation pairs of the small landmarks
  std::vector<int64_t> big_pair_ptr;          // [n_big + 1] prefix sums of K (K - 1) over the big landmarks
  long long big_pairs = 0;                    // camera-pair contributions of the big landmarks (their share of n_pairs)
};

// The layout of the landmarks valid[own[j]] a rank holds (own null: all n_valid).  The landmarks in the order of the lowest
// system row of their clique (min_row of visual_first_rows): the landmarks of a build tile then share cameras, whose S blocks and
// rows the tile sums on chip (visual_tiles.h).  Landmarks with more than batch_slots observations go after all small ones, in the
// same order: they take the passes of visual_big.h.
inline void visual_layout(int n_rows, const int64_t* valid, int64_t n_valid, const std::vector<int64_t>* own, const int* min_row,
                          const int64_t* obs_ptr, const int32_t* obs_cam, const int* row_of_cam, VisualLayout& L, int tile_slots = tiles::kVisTileSlots,
                          int tile_trk = tiles::kMaxTrkPerTile, int batch_slots = tiles::kSlots, int batch_trk = tiles::kMaxTrkPerBatch) {
  const int64_t n = own ? (int64_t)own->size() : n_valid;
  std::vector<int> key;
  if (own) {
    key.resize((size_t)n);
    for (int64_t j = 0; j < n; ++j) key[j] = min_row[(*own)[j]];
  }
  const std::vector<int64_t> order = tiles::order_by_key(std::max(n_rows, 1), own ? key.data() : min_row, n);
  auto src = [&](int64_t j) { const int64_t k = order[j]; return valid[own ? (*own)[k] : k]; };
  auto is_big = [&](int64_t i) { return obs_ptr[i + 1] - obs_ptr[i] > batch_slots; };
  L.Tv = n;
  L.trk_id.resize((size_t)n);
  for (int64_t j = 0; j < n; ++j) if (!is_big(src(j))) L.trk_id[L.Tv_small++] = (int)src(j);
  int64_t w = L.Tv_small;
  for (int64_t j = 0; j < n; ++j) if (is_big(src(j))) L.trk_id[w++] = (int)src(j);
  L.trk_ptr.assign((size_t)n + 1, 0);
  for (int64_t k = 0; k < n; ++k) L.trk_ptr[k + 1] = L.trk_ptr[k] + (int)(obs_ptr[L.trk_id[k] + 1] - obs_ptr[L.trk_id[k]]);
  L.nnz = L.trk_ptr[n];
  for (int64_t k = 0; k < L.Tv_small; ++k) L.n_ordered += (long long)(L.trk_ptr[k + 1] - L.trk_ptr[k]) * (L.trk_ptr[k + 1] - L.trk_ptr[k] - 1);
  L.batch_trk = tiles::cut_ranges(L.Tv_small, L.trk_ptr.data(), nullptr, batch_slots, batch_trk);
  L.tile_trk = tiles::cut_ranges(L.Tv_small, L.trk_ptr.data(), nullptr, tile_slots, tile_trk);
  // pair items of the big landmarks (K (K - 1) each) and their camera-pair contributions: an unordered pair of observations of
  // two distinct rows once, of one row in both orders, i.e. C(n, 2) + sum_row C(n_row, 2) over the n observations of
  // non-constant cameras
  L.big_pair_ptr.assign((size_t)(n - L.Tv_small) + 1, 0);
  std::vector<int> rows;
  for (int64_t b = 0; b < n - L.Tv_small; ++b) {
    const int64_t i = L.trk_id[L.Tv_small + b], K = obs_ptr[i + 1] - obs_ptr[i];
    L.big_pair_ptr[b + 1] = L.big_pair_ptr[b] + K * (K - 1);
    rows.clear();
    for (int64_t q = obs_ptr[i]; q < obs_ptr[i + 1]; ++q) if (row_of_cam[obs_cam[q]] >= 0) rows.push_back(row_of_cam[obs_cam[q]]);
    std::sort(rows.begin(), rows.end());
    const long long nr = (long long)rows.size();
    long long contrib = nr * (nr - 1) / 2;
    for (size_t a = 0; a < rows.size();) {
      size_t e = a;
      while (e < rows.size() && rows[e] == rows[a]) ++e;
      contrib += (long long)(e - a) * (long long)(e - a - 1) / 2;
      a = e;
    }
    L.big_pairs += contrib;
  }
}

// The build's destination table (visual_tiles.h) from the local CSR in the policy's memory (in.trk_pair is set here): the
// camera-pair contributions of the tiles grouped by S block (prun), their observations grouped by row (drun).  n_small, n_ordered,
// n_obs: small landmarks, their ordered observation pairs and observations.  *n_pairs = the contributions with a destination.
template <class Ex>
int visual_tables(Ex& ex, tiles::VisTableIn in, int64_t n_small, int64_t n_ordered, int64_t n_obs, tiles::Runs<Ex>& prun,
                  tiles::Runs<Ex>& drun, int64_t* n_pairs) {
  *n_pairs = 0;
  if (in.n_tiles <= 0) return 0;
  typename Ex::template Buf<long long> cnt, trk_pair;           // ordered observation pairs before every local landmark
  LVBA_PLAN_TRY(cnt.alloc((size_t)n_small + 1));
  LVBA_PLAN_TRY(trk_pair.alloc((size_t)n_small + 1));
  LVBA_PLAN_TRY(ex.for_each(n_small + 1, tiles::VisPairCountF{in.trk_ptr, n_small, cnt.p}));
  LVBA_PLAN_TRY(ex.exclusive_scan(cnt.p, trk_pair.p, n_small + 1));
  in.trk_pair = trk_pair.p;
  LVBA_PLAN_TRY(tiles::sort_runs(ex, n_ordered, in.n_tiles, (uint64_t)in.nblocks, tiles::VisPairKeyF{in}, prun));
  LVBA_PLAN_TRY(tiles::sort_runs(ex, n_obs, in.n_tiles, (uint64_t)in.n_rows, tiles::ObsKeyF{in}, drun));
  return ex.fetch(n_pairs, prun.run_ptr.p + prun.n_runs, 1);
}

// Deterministic mode: the records of the build and their destinations.  Records of S: the tiles' pair runs, the tiles' row runs,
// the big landmarks' observations, the big landmarks' ordered pairs; records of the camera rows: the tiles' row runs, the big
// landmarks' observations.  Each set in its enumeration order, so that every destination's records come in ascending (tile, run)
// order, then in item order.  Observations of constant cameras and pairs outside the lower envelope get a record without a
// destination.
template <class Ex>
int visual_det_index(Ex& ex, const tiles::VisTableIn& in, const tiles::Runs<Ex>& prun, const tiles::Runs<Ex>& drun, const VisualView& vv,
                     const vbig::View& bv, int64_t n_big_obs, int64_t n_big_pairs, tiles::FixedSum<Ex>& S, tiles::FixedSum<Ex>& G) {
  const int64_t npr = prun.n_runs, ndr = drun.n_runs;
  LVBA_PLAN_TRY(tiles::fixed_sum_alloc(S, npr + ndr + n_big_obs + n_big_pairs, 36));
  LVBA_PLAN_TRY(tiles::fixed_sum_alloc(G, ndr + n_big_obs, 18));
  LVBA_PLAN_TRY(ex.for_each(npr, tiles::VisPairRunDstF{in, prun.tile_run.p, prun.run_ptr.p, prun.code.p, S.dst.p}));
  LVBA_PLAN_TRY(ex.for_each(ndr, tiles::ObsRunDstF{in, drun.tile_run.p, drun.run_ptr.p, drun.code.p, S.dst.p + npr, G.dst.p}));
  LVBA_PLAN_TRY(ex.for_each(n_big_obs, vbig::ObsDstF{vv, bv, in.nblocks, in.n_rows, S.dst.p + npr + ndr, G.dst.p + ndr}));
  LVBA_PLAN_TRY(ex.for_each(n_big_pairs, vbig::PairDstF{vv, bv, in.nblocks, S.dst.p + npr + ndr + n_big_obs}));
  LVBA_PLAN_TRY(tiles::fixed_sum_index(ex, S, in.nblocks));
  return tiles::fixed_sum_index(ex, G, in.n_rows);
}

}  // namespace lvba
