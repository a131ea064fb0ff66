// lidar_plan.h — the symbolic set-up of the LiDAR problem handle (lidar_create_impl and lidar_det_setup, lidar_api.cuh), plain
// C++ with no CUDA: the envelope rows, the voxel layout (big voxels, voxel order, batches, tiles, windows), the build's
// destination table and the record index of deterministic mode.  The table and the index are item passes run by an execution
// policy: CudaExec (exec.cuh) in the library, the host policy of tests/emu in the CPU tests, which call these same functions.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "lidar_big.h"
#include "lidar_tiles.h"
#include "setup_pool.h"

#ifndef LVBA_PLAN_TRY
#define LVBA_PLAN_TRY(call) do { const int rc__ = (call); if (rc__ != 0) return rc__; } while (0)
#endif

namespace lvba {

// The rows of the pose system under constant poses (lvba_lidar_opts::pose_fixed, mask: W bytes or null): the free poses in
// ascending order.  row_of[pose] = its row, -1 for a constant pose; pose_of_row its inverse.  Returns the number of rows.
inline int lidar_row_map(int W, const uint8_t* mask, std::vector<int>& row_of, std::vector<int>& pose_of_row) {
  row_of.assign((size_t)W, -1);
  pose_of_row.clear();
  for (int p = 0; p < W; ++p)
    if (!mask || !mask[p]) { row_of[p] = (int)pose_of_row.size(); pose_of_row.push_back(p); }
  return (int)pose_of_row.size();
}

// The raw envelope of the pose system: first[r] = the lowest row that shares a voxel with row r (r when there is none).
// Clique minima over the caller's CSR in parallel chunks, one row array per worker.  row_of (lidar_row_map, n_rows rows): the
// rows of the free poses, a voxel's constant slots couple nothing; null: every pose is its own row (n_rows = W).
inline std::vector<int> lidar_first_rows(int W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx, const int* row_of = nullptr,
                                         int n_rows = -1) {
  const int n = row_of ? n_rows : W;
  auto row = [&](int64_t q) { return row_of ? row_of[pose_idx[q]] : pose_idx[q]; };
  std::vector<int> first(n);
  for (int r = 0; r < n; ++r) first[r] = r;
  std::vector<int> first_w((size_t)kMaxSetupThreads * (size_t)n);
  for (int w = 0; w < kMaxSetupThreads; ++w) std::copy(first.begin(), first.end(), first_w.begin() + (size_t)w * (size_t)n);
  parallel_chunks(V, 1 << 14, [&](int64_t a0, int64_t a1, int w) {
    int* fr = first_w.data() + (size_t)w * (size_t)n;
    for (int64_t a = a0; a < a1; ++a) {
      int64_t q0 = vox_ptr[a];                                 // the voxel's lowest free row (ascending poses: ascending rows)
      while (q0 < vox_ptr[a + 1] && row(q0) < 0) ++q0;
      if (q0 == vox_ptr[a + 1]) continue;
      const int m = row(q0);
      for (int64_t q = q0; q < vox_ptr[a + 1]; ++q)
        if (row(q) >= 0) fr[row(q)] = std::min(fr[row(q)], m);
    }
  });
  for (int w = 0; w < kMaxSetupThreads; ++w)
    for (int r = 0; r < n; ++r) first[r] = std::min(first[r], first_w[(size_t)w * (size_t)n + r]);
  return first;
}

enum LidarLayoutError { kLayoutOk = 0, kLayoutSpansWindows, kLayoutBigInBatch };

struct LidarLayout {
  int err = kLayoutOk;
  int64_t err_vox = -1;                       // the caller's voxel that caused err
  // voxels seen from more than batch_slots poses, in the caller's order, as lidar_big.h reads them; big_src = caller slot
  std::vector<int64_t> big_vox, big_vox_ptr{0}, big_pair_ptr{0};
  std::vector<int32_t> big_pose;
  std::vector<int> big_src;
  // the other voxels in the order of their lowest pose: slot0[i] = first caller slot of local voxel i, l_vox_ptr[i] = its
  // first local slot
  std::vector<int> slot0, l_vox_ptr;
  bool identity = false;                      // the local voxels are the caller's, in the caller's order
  std::vector<int> batch_vox, tile_vox;       // residual batches and build tiles: voxel ranges
  // batched window BA: window of every pose, batch / tile range and voxel count of every window
  std::vector<int> pose_grp, grp_batch, grp_tile;
  std::vector<long long> grp_V;
  long long nnz = 0, n_pairs = 0;             // slots and pose pairs of the local voxels
};

// The layout of the caller's CSR on one rank.  owned: the caller's voxels this rank holds, ascending (null: all V).  n_groups > 0: the poses
// fall into windows grp_ptr[0..n_groups], and every voxel must lie inside one.  Voxels with more than batch_slots slots leave the
// batches and tiles for the passes of lidar_big.h (refused in a batched solve).  Residual batches hold <= batch_slots slots, build
// tiles <= tile_slots slots and <= tile_vox voxels; neither crosses a window.  Returns L.err.
inline int lidar_layout(int W, int64_t V, const int64_t* vox_ptr, const int32_t* pose_idx, const std::vector<int64_t>* owned, int n_groups, const int32_t* grp_ptr, LidarLayout& L, int tile_slots = tiles::kTileSlots,
                        int tile_vox = tiles::kMaxVoxPerTile, int batch_slots = tiles::kSlots) {
  if (n_groups > 0) {
    L.pose_grp.resize((size_t)W);
    for (int g = 0; g < n_groups; ++g)
      for (int r = grp_ptr[g]; r < grp_ptr[g + 1]; ++r) L.pose_grp[r] = g;
    L.grp_V.assign((size_t)n_groups, 0);
    for (int64_t a = 0; a < V; ++a) {
      const int g = L.pose_grp[pose_idx[vox_ptr[a]]];
      if (L.pose_grp[pose_idx[vox_ptr[a + 1] - 1]] != g) { L.err_vox = a; return L.err = kLayoutSpansWindows; }
      ++L.grp_V[g];
    }
  }
  // voxels seen from more than batch_slots poses do not fit a batch CTA: they leave the rank's list for lidar_big.h
  const int64_t n_in = owned ? (int64_t)owned->size() : V;
  auto caller = [&](int64_t j) { return owned ? (*owned)[j] : j; };
  auto is_big = [&](int64_t a) { return vox_ptr[a + 1] - vox_ptr[a] > batch_slots; };
  std::vector<int64_t> small;
  bool has_big = false;
  for (int64_t j = 0; j < n_in && !has_big; ++j) has_big = is_big(caller(j));
  if (has_big) {
    for (int64_t j = 0; j < n_in; ++j) (is_big(caller(j)) ? L.big_vox : small).push_back(caller(j));
    // the batched window LM (lidar_batch_lm_impl) has no big-voxel passes: such a voxel would drop out of H, g and the
    // residual sums while still counting in the AVG_THR divisor.  A window holds <= 31 poses (EnvSolver::prepare), so this
    // cannot happen today; refuse loudly if that ever changes.
    if (n_groups > 0) { L.err_vox = L.big_vox[0]; return L.err = kLayoutBigInBatch; }
    for (int64_t a : L.big_vox) {
      for (int64_t q = vox_ptr[a]; q < vox_ptr[a + 1]; ++q) { L.big_src.push_back((int)q); L.big_pose.push_back(pose_idx[q]); }
      const int64_t K = vox_ptr[a + 1] - vox_ptr[a];
      L.big_vox_ptr.push_back((int64_t)L.big_src.size());
      L.big_pair_ptr.push_back(L.big_pair_ptr.back() + K * (K - 1) / 2);
    }
  }
  const int64_t* in = has_big ? small.data() : owned ? owned->data() : nullptr;
  const int64_t Vl = has_big ? (int64_t)small.size() : n_in;
  // voxels in the order of their lowest pose: the voxels of a build tile then share pose pairs, whose H blocks the tile sums on
  // chip (lidar_tiles.h); the windows, consecutive pose ranges, come out contiguous and in order
  L.nnz = tiles::order_by_lowest_pose(W, in, Vl, vox_ptr, pose_idx, L.slot0, L.l_vox_ptr);
  L.identity = !owned && !has_big;
  for (int64_t i = 0; i < Vl; ++i) {
    const long long K = L.l_vox_ptr[i + 1] - L.l_vox_ptr[i];
    L.n_pairs += K * (K - 1) / 2;
    L.identity = L.identity && L.slot0[i] == L.l_vox_ptr[i];
  }
  std::vector<int> vox_grp(n_groups > 0 ? (size_t)Vl : (size_t)0);
  for (int64_t i = 0; i < (int64_t)vox_grp.size(); ++i) vox_grp[i] = L.pose_grp[pose_idx[L.slot0[i]]];
  const int* grp = n_groups > 0 ? vox_grp.data() : nullptr;
  L.batch_vox = tiles::cut_ranges(Vl, L.l_vox_ptr.data(), grp, batch_slots, batch_slots);
  L.tile_vox = tiles::cut_ranges(Vl, L.l_vox_ptr.data(), grp, tile_slots, tile_vox);
  if (n_groups > 0) {
    auto per_window = [&](const std::vector<int>& cut) {      // range of batches / tiles of every window
      std::vector<int> r((size_t)n_groups + 1, 0);
      for (size_t k = 0; k + 1 < cut.size(); ++k) ++r[(size_t)vox_grp[cut[k]] + 1];
      for (int g = 0; g < n_groups; ++g) r[g + 1] += r[g];
      return r;
    };
    L.grp_batch = per_window(L.batch_vox);
    L.grp_tile = per_window(L.tile_vox);
  }
  return kLayoutOk;
}

// The build's destination table (lidar_tiles.h) from the local CSR in the policy's memory (in.vox_pair is set here): the pose
// pairs of the tiles grouped by H block (prun), their slots grouped by pose (drun).  n_vox, n_pairs, nnz: of the local voxels.
template <class Ex>
int lidar_tables(Ex& ex, tiles::TableIn in, int64_t n_vox, int64_t n_pairs, int64_t nnz, tiles::Runs<Ex>& prun, tiles::Runs<Ex>& drun) {
  if (in.n_tiles <= 0) return 0;
  typename Ex::template Buf<long long> cnt, vox_pair;          // pose pairs before every local voxel
  LVBA_PLAN_TRY(cnt.alloc((size_t)n_vox + 1));
  LVBA_PLAN_TRY(vox_pair.alloc((size_t)n_vox + 1));
  LVBA_PLAN_TRY(ex.for_each(n_vox + 1, tiles::PairCountF{in.vox_ptr, n_vox, cnt.p}));
  LVBA_PLAN_TRY(ex.exclusive_scan(cnt.p, vox_pair.p, n_vox + 1));
  in.vox_pair = vox_pair.p;
  LVBA_PLAN_TRY(tiles::build_runs(ex, in, /*by_slot=*/false, n_pairs, prun));
  return tiles::build_runs(ex, in, /*by_slot=*/true, nnz, drun);
}

// Deterministic mode: the records of the build and their destinations.  Records of H: the tiles' pair runs, the tiles' pose runs,
// the big voxels' slots, the big voxels' pairs; records of g: the tiles' pose runs, the big voxels' slots.  Each set in its
// enumeration order, so that every destination's records come in ascending (tile, run) order, then in item order.
template <class Ex>
int lidar_det_index(Ex& ex, const tiles::TableIn& in, const tiles::Runs<Ex>& prun, const tiles::Runs<Ex>& drun, const big::View& bv,
                    int64_t n_big_slots, int64_t n_big_pairs, tiles::FixedSum<Ex>& H, tiles::FixedSum<Ex>& g) {
  const int64_t npr = prun.n_runs, ndr = drun.n_runs;
  LVBA_PLAN_TRY(tiles::fixed_sum_alloc(H, npr + ndr + n_big_slots + n_big_pairs, 36));
  LVBA_PLAN_TRY(tiles::fixed_sum_alloc(g, ndr + n_big_slots, 6));
  LVBA_PLAN_TRY(ex.for_each(npr, tiles::PairRunDstF{in, prun.tile_run.p, prun.run_ptr.p, prun.code.p, H.dst.p}));
  LVBA_PLAN_TRY(ex.for_each(ndr, tiles::SlotRunDstF{in, drun.tile_run.p, drun.run_ptr.p, drun.code.p, H.dst.p + npr, g.dst.p}));
  LVBA_PLAN_TRY(ex.for_each(n_big_slots, big::SlotDstF{bv, H.dst.p + npr + ndr, g.dst.p + ndr}));
  LVBA_PLAN_TRY(ex.for_each(n_big_pairs, big::PairDstF{bv, H.dst.p + npr + ndr + n_big_slots}));
  LVBA_PLAN_TRY(tiles::fixed_sum_index(ex, H, in.nblocks));
  return tiles::fixed_sum_index(ex, g, in.W);
}

}  // namespace lvba
