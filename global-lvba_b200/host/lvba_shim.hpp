// lvba_shim.hpp — host-side C++ mirror of the two reference call sites, written against the C ABI of
// include/lvba_b200.h.  Header only, C++17, no Eigen / Ceres / PCL / ROS includes of its own: the functions
// are templates over the reference's own types (IMUST, PointCluster, VOX_HESS, Eigen matrices are only
// touched through operator()(i,j) / operator()(i) / public members), so the same header compiles inside
// src/lvba_system.cpp of the reference and inside tests/shim/test_shim.cpp with plain mock structs.
//
//   lvba_b200::damping_iter(x_stats, voxhess)        replaces BALM2::damping_iter   include/BALM/bavoxel.hpp:662-767
//   lvba_b200::evaluate_residual(x_stats, voxhess)   VOX_HESS::evaluate_residual (commented out in the reference, :205-234)
//   lvba_b200::remove_outlier(x_stats, voxhess, r)   BALM2::remove_outlier (commented out in the reference, :650-660)
//   lvba_b200::solve_visual(...)                     replaces the Ceres block       src/lvba_system.cpp:1571-1656
//   lvba_b200::solve_visual_remove_outliers(...)     the same, then a reprojection filter and a second solve on one handle
//   lvba_b200::solve_visual_refine_intrinsics(...)   solve_visual with the intrinsics a parameter block, refined and written back
//   lvba_b200::WindowBatch                           collects the windows of runWindowBA (src/lvba_system.cpp:232-302) and
//                                                    solves them in one lvba_lidar_lm_batch call
//   lvba_b200::SurfMap                               replaces the surf_map built by cut_voxel + recut (+ tras_opt) in front of
//                                                    every solve (src/lvba_system.cpp:247-258, 361-378, 1498-1506) and the
//                                                    plane lookup of recompute_local_planes (:1529-1566)
//   lvba_b200::run_window_stage                      the whole window loop of runWindowBA (src/lvba_system.cpp:232-266): one voxel
//                                                    map per window built together + every window solved in one batched LM
//   lvba_b200::run_window_ba                         all of runWindowBA (:205-316): the window stage, then the anchors — aligned window
//                                                    poses, rel_poses_to_anchor_, anchor_index_per_frame_, anchor poses and the
//                                                    merged + down-sampled anchor clouds (boundary B6)
//   lvba_b200::DepthRenderer                         replaces buildGridMapFromOptimized + generateDepthWithVoxel
//                                                    (src/lvba_system.cpp:1266-1338, 835-919)
//   lvba_b200::build_tracks_and_fuse_3d              replaces BuildTracksAndFuse3D (src/lvba_system.cpp:921-1263): matches +
//                                                    keypoints + depth candidates -> tracks_ (boundary B7)
//
// Same names, argument meaning and error behaviour as the reference: void-like use (the reference ignores
// solver failure), state written back only on success, size mismatches throw std::runtime_error like
// src/lvba_system.cpp:1427-1432.  See INTEGRATION.md for the three-line patches.
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "lvba_b200.h"

namespace lvba_b200 {

// opts with the constant poses pose_fixed (null: opts as they are; else one entry per pose, nonzero = constant, which
// overrides opts->pose_fixed); `o` holds the copy when one is needed
inline const lvba_lidar_opts* with_pose_fixed(const lvba_lidar_opts* opts, const std::vector<uint8_t>* pose_fixed, int W,
                                              lvba_lidar_opts& o, const char* who) {
  if (!pose_fixed) return opts;
  if ((int)pose_fixed->size() != W) throw std::runtime_error(std::string("lvba_b200::") + who + ": pose_fixed needs one entry per pose");
  if (opts) o = *opts; else lvba_lidar_default_opts(&o);
  o.pose_fixed = pose_fixed->data();
  return &o;
}

// ---- B1: x_stats[i].R (3x3), x_stats[i].p (3) ; voxhess.plvec_voxels[a] -> const vector<PointCluster>* with
//      (*ptr)[i].P (3x3), .v (3), .N ; voxhess.win_size.  The problem in the CSR of lvba_lidar_lm: the slots with N != 0
//      (bavoxel.hpp:91, :113) of every voxel in plvec_voxels order, and the first win_size poses.
struct LidarCsr {
  int W = 0;
  std::vector<int64_t> vox_ptr;
  std::vector<int32_t> pose_idx;
  std::vector<double> clusters, poses;
  int64_t V() const { return (int64_t)vox_ptr.size() - 1; }
};

template <class PoseVec, class VoxHess>
inline LidarCsr pack_lidar(const PoseVec& x_stats, const VoxHess& voxhess, const char* who) {
  LidarCsr c;
  const int W = c.W = voxhess.win_size;
  if ((int)x_stats.size() < W) throw std::runtime_error(std::string("lvba_b200::") + who + ": x_stats smaller than win_size");
  const int64_t V = (int64_t)voxhess.plvec_voxels.size();
  c.vox_ptr.assign((size_t)V + 1, 0);
  for (int64_t a = 0; a < V; ++a) {
    const auto& sig = *voxhess.plvec_voxels[a];
    for (int i = 0; i < W; ++i) {
      if (sig[i].N == 0) continue;
      c.pose_idx.push_back(i);
      const auto& P = sig[i].P; const auto& v = sig[i].v;
      const double rec[10] = {P(0, 0), P(0, 1), P(0, 2), P(1, 1), P(1, 2), P(2, 2), v(0), v(1), v(2), (double)sig[i].N};
      c.clusters.insert(c.clusters.end(), rec, rec + 10);
    }
    c.vox_ptr[a + 1] = (int64_t)c.pose_idx.size();
  }
  c.poses.resize((size_t)W * 12);
  for (int i = 0; i < W; ++i) {
    for (int r = 0; r < 3; ++r) for (int k = 0; k < 3; ++k) c.poses[12 * i + 3 * r + k] = x_stats[i].R(r, k);
    for (int r = 0; r < 3; ++r) c.poses[12 * i + 9 + r] = x_stats[i].p(r);
  }
  return c;
}

// pose_fixed (null: none) holds poses constant (lvba_lidar_opts::pose_fixed).
template <class PoseVec, class VoxHess>
inline int damping_iter(PoseVec& x_stats, VoxHess& voxhess, const lvba_lidar_opts* opts = nullptr,
                        lvba_summary* summary = nullptr, const std::vector<uint8_t>* pose_fixed = nullptr) {
  LidarCsr c = pack_lidar(x_stats, voxhess, "damping_iter");
  const int W = c.W;
  lvba_lidar_opts o;
  opts = with_pose_fixed(opts, pose_fixed, W, o, "damping_iter");
  const int rc = lvba_lidar_lm(W, c.V(), c.vox_ptr.data(), c.pose_idx.data(), c.clusters.data(), c.poses.data(), opts, summary);
  if (rc != LVBA_OK) return rc;                        // reference: silent on failure, state untouched
  for (int i = 0; i < W; ++i) {                        // x_stats = x_stats_temp (bavoxel.hpp:746)
    for (int r = 0; r < 3; ++r) for (int k = 0; k < 3; ++k) x_stats[i].R(r, k) = c.poses[12 * i + 3 * r + k];
    for (int r = 0; r < 3; ++r) x_stats[i].p(r) = c.poses[12 * i + 9 + r];
  }
  return LVBA_OK;
}

// VOX_HESS::evaluate_residual (bavoxel.hpp:205-234, commented out in the reference): lambda_0 of every voxel of plvec_voxels at
// x_stats, through lvba_lidar_voxel_residuals on a handle of its own.  Throws std::runtime_error with the library's message.
template <class PoseVec, class VoxHess>
inline std::vector<double> evaluate_residual(const PoseVec& x_stats, const VoxHess& voxhess, int32_t device = -1) {
  LidarCsr c = pack_lidar(x_stats, voxhess, "evaluate_residual");
  std::vector<double> lam((size_t)c.V());
  lvba_lidar_problem* p = nullptr;
  int rc = lvba_lidar_create(c.W, c.V(), c.vox_ptr.data(), c.pose_idx.data(), c.clusters.data(), c.poses.data(), device, &p);
  if (rc == LVBA_OK) rc = lvba_lidar_voxel_residuals(p, nullptr, lam.data());
  const std::string why = rc == LVBA_OK ? "" : lvba_last_error();
  lvba_lidar_destroy(p);
  if (rc != LVBA_OK) throw std::runtime_error("lvba_b200::evaluate_residual: " + why);
  return lam;
}

// BALM2::remove_outlier(x_stats, voxhess, ratio) (bavoxel.hpp:650-660 with VOX_HESS::remove_residual :236-268, commented out in
// the reference): erases from voxhess.plvec_voxels exactly the voxels the reference's walk would (lvba_lidar_remove_outliers;
// the rule and its quirks are in include/lvba_b200.h), keeping the others in order.  Returns the library's status; on an error
// (a ratio outside [0, 1), floor((1 - ratio) V) < 1, a non-finite lambda_0, a removal of every voxel) plvec_voxels is untouched.
template <class PoseVec, class VoxHess>
inline int remove_outlier(const PoseVec& x_stats, VoxHess& voxhess, double ratio, int64_t* n_removed = nullptr, int32_t device = -1) {
  LidarCsr c = pack_lidar(x_stats, voxhess, "remove_outlier");
  std::vector<uint8_t> removed((size_t)c.V(), 0);
  lvba_lidar_problem* p = nullptr;
  int rc = lvba_lidar_create(c.W, c.V(), c.vox_ptr.data(), c.pose_idx.data(), c.clusters.data(), c.poses.data(), device, &p);
  if (rc == LVBA_OK) rc = lvba_lidar_remove_outliers(p, ratio, removed.data(), n_removed);
  lvba_lidar_destroy(p);
  if (rc != LVBA_OK) return rc;
  size_t w = 0;                                        // plvec_voxels.erase for every removed voxel, survivors in order
  for (size_t a = 0; a < removed.size(); ++a)
    if (!removed[a]) voxhess.plvec_voxels[w++] = voxhess.plvec_voxels[a];
  voxhess.plvec_voxels.resize(w);
  return LVBA_OK;
}

// ---- B1 batched: runWindowBA builds one (x_win, voxhess) pair per window and calls damping_iter on each
//      (src/lvba_system.cpp:239-264).  WindowBatch::add() packs a window instead of solving it; solve() runs every
//      packed window in one call and writes the poses back into the x_win vectors it was given (which must outlive
//      solve()).  Windows below the reference's `plvec_voxels.size() < 3 * x_win.size()` rule (:262-266) are packed too
//      and come back untouched with LVBA_TERM_SKIPPED, so the caller's bookkeeping (win_skipped) can read the summary.
template <class PoseVec>
class WindowBatch {
 public:
  template <class VoxHess>
  void add(PoseVec& x_win, const VoxHess& voxhess) {
    const int W = voxhess.win_size;
    if ((int)x_win.size() < W) throw std::runtime_error("lvba_b200::WindowBatch::add: x_win smaller than win_size");
    const int32_t base = win_ptr_.back();
    for (const auto* sigp : voxhess.plvec_voxels) {
      const auto& sig = *sigp;
      for (int i = 0; i < W; ++i) {
        if (sig[i].N == 0) continue;
        pose_idx_.push_back(base + i);
        const auto& P = sig[i].P; const auto& v = sig[i].v;
        const double rec[10] = {P(0, 0), P(0, 1), P(0, 2), P(1, 1), P(1, 2), P(2, 2), v(0), v(1), v(2), (double)sig[i].N};
        clusters_.insert(clusters_.end(), rec, rec + 10);
      }
      vox_ptr_.push_back((int64_t)pose_idx_.size());
    }
    for (int i = 0; i < W; ++i) {
      double rec[12];
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) rec[3 * r + c] = x_win[i].R(r, c);
      for (int r = 0; r < 3; ++r) rec[9 + r] = x_win[i].p(r);
      poses_.insert(poses_.end(), rec, rec + 12);
    }
    win_ptr_.push_back(base + W);
    targets_.push_back(&x_win);
  }
  int size() const { return (int)targets_.size(); }
  // returns LVBA_OK or a negative lvba_status; on failure no window is modified (reference: silent, state untouched)
  int solve(int min_voxels_per_pose = 3, const lvba_lidar_opts* opts = nullptr, std::vector<lvba_summary>* summaries = nullptr,
            lvba_summary* total = nullptr) {
    if (targets_.empty()) return LVBA_OK;
    std::vector<lvba_summary> local((size_t)size());
    const int rc = lvba_lidar_lm_batch(size(), win_ptr_.data(), (int64_t)vox_ptr_.size() - 1, vox_ptr_.data(), pose_idx_.data(),
                                       clusters_.data(), poses_.data(), min_voxels_per_pose, opts, local.data(), total);
    if (rc != LVBA_OK) return rc;
    for (int w = 0; w < size(); ++w) {
      PoseVec& x = *targets_[w];
      for (int i = 0; i < win_ptr_[w + 1] - win_ptr_[w]; ++i) {
        const double* rec = poses_.data() + 12 * (size_t)(win_ptr_[w] + i);
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) x[i].R(r, c) = rec[3 * r + c];
        for (int r = 0; r < 3; ++r) x[i].p(r) = rec[9 + r];
      }
    }
    if (summaries) *summaries = local;
    return LVBA_OK;
  }

 private:
  std::vector<int32_t> win_ptr_{0};
  std::vector<int64_t> vox_ptr_{0};
  std::vector<int32_t> pose_idx_;
  std::vector<double> clusters_, poses_;
  std::vector<PoseVec*> targets_;
};

// ---- B3: the adaptive voxel map.  The reference fills an unordered_map<VOXEL_LOC, OCTO_TREE_ROOT*> with one
//      cut_voxel call per scan, then recut()s every root and walks it with tras_opt (BA voxels) or
//      findCorrespondPoint (plane of a landmark).  SurfMap takes the same inputs — the scans as
//      pcl::PointCloud<PointType>::Ptr-like handles (anything with ->points[k].x/.y/.z and ->points.size()), the poses,
//      the root voxel size and the eigen-ratio array — builds the map on the device and keeps it there.
template <class PoseVec>
class SurfMap {
 public:
  SurfMap() = default;
  SurfMap(const SurfMap&) = delete;
  SurfMap& operator=(const SurfMap&) = delete;
  ~SurfMap() { clear(); }
  void clear() { if (map_) lvba_voxel_map_destroy(map_); map_ = nullptr; }

  // cut_voxel(surf_map, *clouds[j], x_buf[j], j, win_size, voxel_size, eigen_ratio) for every j, then recut(x_buf).
  // eigen_ratio_array: the four per-layer thresholds in force (set_eigen_ratio_array, src/lvba_system.cpp:360).
  template <class CloudPtrVec>
  int build(const CloudPtrVec& clouds, const PoseVec& x_buf, double voxel_size, const float eigen_ratio_array[4],
            lvba_voxel_summary* summary = nullptr) {
    clear();
    const int W = (int)clouds.size();
    if ((int)x_buf.size() < W) throw std::runtime_error("lvba_b200::SurfMap::build: fewer poses than scans");
    std::vector<int64_t> scan_ptr((size_t)W + 1, 0);
    for (int j = 0; j < W; ++j) scan_ptr[j + 1] = scan_ptr[j] + (int64_t)clouds[j]->points.size();
    std::vector<float> xyz((size_t)scan_ptr[W] * 3);
    for (int j = 0; j < W; ++j) {
      float* dst = xyz.data() + 3 * (size_t)scan_ptr[j];
      for (const auto& pt : clouds[j]->points) { *dst++ = pt.x; *dst++ = pt.y; *dst++ = pt.z; }
    }
    std::vector<double> poses((size_t)W * 12);
    for (int i = 0; i < W; ++i) {
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) poses[12 * i + 3 * r + c] = x_buf[i].R(r, c);
      for (int r = 0; r < 3; ++r) poses[12 * i + 9 + r] = x_buf[i].p(r);
    }
    lvba_voxel_opts o;
    lvba_voxel_default_opts(&o);
    o.voxel_size = voxel_size;
    for (int k = 0; k < 4; ++k) o.eigen_ratio[k] = eigen_ratio_array[k];
    win_size_ = W;
    return lvba_voxel_map_create(W, scan_ptr.data(), xyz.data(), 3, poses.data(), &o, &map_, summary);
  }

  // tras_opt(voxhess) + BALM2::damping_iter(x_stats, voxhess) on the map's plane voxels.  min_voxels_per_pose mirrors the
  // caller's `plvec_voxels.size() < 3 * x_win.size()` skip (src/lvba_system.cpp:262-266): returns LVBA_OK with
  // summary->termination = LVBA_TERM_SKIPPED and x_stats untouched when there are too few voxels.  pose_fixed: as damping_iter.
  int damping_iter(PoseVec& x_stats, int min_voxels_per_pose = 0, const lvba_lidar_opts* opts = nullptr, lvba_summary* summary = nullptr,
                   const std::vector<uint8_t>* pose_fixed = nullptr) {
    if (!map_) throw std::runtime_error("lvba_b200::SurfMap::damping_iter: map not built");
    if ((int)x_stats.size() < win_size_) throw std::runtime_error("lvba_b200::SurfMap::damping_iter: x_stats smaller than win_size");
    lvba_lidar_opts o;
    opts = with_pose_fixed(opts, pose_fixed, win_size_, o, "SurfMap::damping_iter");
    std::vector<double> poses((size_t)win_size_ * 12);
    for (int i = 0; i < win_size_; ++i) {
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) poses[12 * i + 3 * r + c] = x_stats[i].R(r, c);
      for (int r = 0; r < 3; ++r) poses[12 * i + 9 + r] = x_stats[i].p(r);
    }
    lvba_summary local{};
    const int rc = lvba_voxel_map_lidar_lm(map_, poses.data(), min_voxels_per_pose, opts, &local);   // clusters stay on the device
    if (rc != LVBA_OK) return rc;
    if (summary) *summary = local;
    if (local.termination == LVBA_TERM_SKIPPED) return LVBA_OK;
    for (int i = 0; i < win_size_; ++i) {
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) x_stats[i].R(r, c) = poses[12 * i + 3 * r + c];
      for (int r = 0; r < 3; ++r) x_stats[i].p(r) = poses[12 * i + 9 + r];
    }
    return LVBA_OK;
  }

  // damping_iter, remove_outlier(ratio) and damping_iter again on ONE device handle of the map's plane voxels (the sequence the
  // reference's commented-out BALM2::remove_outlier, bavoxel.hpp:650-660, was written for): the second solve runs on the kept
  // voxels from the poses of the first, with a fresh LM state.  pose_fixed: as damping_iter.  n_removed (may be null): the voxels
  // erased.  x_stats is written back only on success.
  int damping_iter_remove_outlier(PoseVec& x_stats, double ratio, const lvba_lidar_opts* opts = nullptr, int64_t* n_removed = nullptr,
                                  lvba_summary* first = nullptr, lvba_summary* second = nullptr, const std::vector<uint8_t>* pose_fixed = nullptr) {
    if (!map_) throw std::runtime_error("lvba_b200::SurfMap::damping_iter_remove_outlier: map not built");
    if ((int)x_stats.size() < win_size_) throw std::runtime_error("lvba_b200::SurfMap::damping_iter_remove_outlier: x_stats smaller than win_size");
    lvba_lidar_opts o;
    opts = with_pose_fixed(opts, pose_fixed, win_size_, o, "SurfMap::damping_iter_remove_outlier");
    lvba_lidar_opts d;
    if (opts) d = *opts; else lvba_lidar_default_opts(&d);
    std::vector<double> poses((size_t)win_size_ * 12);
    for (int i = 0; i < win_size_; ++i) {
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) poses[12 * i + 3 * r + c] = x_stats[i].R(r, c);
      for (int r = 0; r < 3; ++r) poses[12 * i + 9 + r] = x_stats[i].p(r);
    }
    lvba_lidar_problem* p = nullptr;
    lvba_summary s1{}, s2{};
    int rc = lvba_voxel_map_lidar_create(map_, poses.data(), &p);
    if (rc == LVBA_OK) rc = lvba_lidar_reset_lm(p, &d);
    if (rc == LVBA_OK) rc = lvba_lidar_iterate(p, d.max_iter, &s1);
    if (rc == LVBA_OK) rc = lvba_lidar_remove_outliers(p, ratio, nullptr, n_removed);
    if (rc == LVBA_OK) rc = lvba_lidar_iterate(p, d.max_iter, &s2);
    if (rc == LVBA_OK) rc = lvba_lidar_get_poses(p, poses.data());
    lvba_lidar_destroy(p);
    if (rc != LVBA_OK) return rc;
    if (first) *first = s1;
    if (second) *second = s2;
    for (int i = 0; i < win_size_; ++i) {
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) x_stats[i].R(r, c) = poses[12 * i + 3 * r + c];
      for (int r = 0; r < 3; ++r) x_stats[i].p(r) = poses[12 * i + 9 + r];
    }
    return LVBA_OK;
  }

  // recompute_local_planes (src/lvba_system.cpp:1529-1566): plane_n[pi], plane_d[pi] of the PLANE node Xs[pi] falls in,
  // zeros when there is none.
  int recompute_local_planes(const std::vector<std::array<double, 3>>& Xs, std::vector<std::array<double, 3>>& plane_n,
                             std::vector<double>& plane_d) {
    if (!map_) throw std::runtime_error("lvba_b200::SurfMap::recompute_local_planes: map not built");
    const int64_t n = (int64_t)Xs.size();
    std::vector<double> nd((size_t)n * 4);
    const int rc = lvba_voxel_map_lookup(map_, n, n ? Xs[0].data() : nullptr, nd.data());
    if (rc != LVBA_OK) return rc;
    plane_n.resize((size_t)n); plane_d.resize((size_t)n);
    for (int64_t i = 0; i < n; ++i) { plane_n[i] = {nd[4 * i], nd[4 * i + 1], nd[4 * i + 2]}; plane_d[i] = nd[4 * i + 3]; }
    return LVBA_OK;
  }

  int64_t voxels() const { lvba_voxel_summary vs{}; return map_ && lvba_voxel_map_summary(map_, &vs) == LVBA_OK ? vs.n_voxels : 0; }
  lvba_voxel_map* handle() const { return map_; }

 private:
  lvba_voxel_map* map_ = nullptr;
  int win_size_ = 0;
};

// ---- B3 + B1 batched: the window loop of runWindowBA (src/lvba_system.cpp:232-266) in two library calls.  pl_fulls / x_buf_full
//      are dataset_io_->pl_fulls_ / x_buf_; windows are the consecutive `window_size` slices of the loop at :232-233.  On return
//      x_wins[w] holds the optimised x_win of window w (the odometry poses when the window was skipped by the
//      `plvec_voxels.size() < 3 * x_win.size()` rule, :259-263, which summaries[w].termination == LVBA_TERM_SKIPPED reports).
//      pose_fixed (null: none): one entry per frame of the concatenated windows, nonzero = held constant (a window whose frames
//      are all constant reports LVBA_TERM_FUNCTION_TOL with no iteration).
template <class CloudPtrVec, class PoseVec>
inline int run_window_stage(const CloudPtrVec& pl_fulls, const PoseVec& x_buf_full, int window_size, double root_voxel_size,
                            const float eigen_ratio_array[4], std::vector<PoseVec>& x_wins, std::vector<lvba_summary>* summaries = nullptr,
                            lvba_summary* total = nullptr, const lvba_lidar_opts* opts = nullptr,
                            const std::vector<uint8_t>* pose_fixed = nullptr) {
  if (window_size <= 0) throw std::runtime_error("lvba_b200::run_window_stage: window_size must be positive");
  const int total_size = (int)std::min(pl_fulls.size(), x_buf_full.size());
  lvba_lidar_opts lo;
  opts = with_pose_fixed(opts, pose_fixed, total_size, lo, "run_window_stage");
  std::vector<int32_t> win_ptr{0};
  for (int start = 0; start < total_size; start += window_size) win_ptr.push_back(std::min(start + window_size, total_size));
  const int n_windows = (int)win_ptr.size() - 1;
  x_wins.clear();
  if (n_windows == 0) return LVBA_OK;
  std::vector<int64_t> scan_ptr((size_t)total_size + 1, 0);
  for (int j = 0; j < total_size; ++j) scan_ptr[j + 1] = scan_ptr[j] + (int64_t)pl_fulls[j]->points.size();
  std::vector<float> xyz((size_t)scan_ptr[total_size] * 3);
  for (int j = 0; j < total_size; ++j) {
    float* dst = xyz.data() + 3 * (size_t)scan_ptr[j];
    for (const auto& pt : pl_fulls[j]->points) { *dst++ = pt.x; *dst++ = pt.y; *dst++ = pt.z; }
  }
  std::vector<double> poses((size_t)total_size * 12);
  for (int i = 0; i < total_size; ++i) {
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) poses[12 * i + 3 * r + c] = x_buf_full[i].R(r, c);
    for (int r = 0; r < 3; ++r) poses[12 * i + 9 + r] = x_buf_full[i].p(r);
  }
  lvba_voxel_opts o;
  lvba_voxel_default_opts(&o);
  o.voxel_size = root_voxel_size;
  for (int k = 0; k < 4; ++k) o.eigen_ratio[k] = eigen_ratio_array[k];
  lvba_voxel_map* map = nullptr;
  int rc = lvba_voxel_map_create_windows(n_windows, win_ptr.data(), scan_ptr.data(), xyz.data(), 3, poses.data(), &o, &map, nullptr);
  if (rc != LVBA_OK) return rc;
  std::vector<lvba_summary> local((size_t)n_windows);
  rc = lvba_voxel_map_lidar_lm_batch(map, poses.data(), /*min_voxels_per_pose=*/3, opts, local.data(), total);
  lvba_voxel_map_destroy(map);
  if (rc != LVBA_OK) return rc;
  for (int w = 0; w < n_windows; ++w) {
    PoseVec x_win(x_buf_full.begin() + win_ptr[w], x_buf_full.begin() + win_ptr[w + 1]);      // :239 (keeps .t and any other member)
    for (int i = 0; i < win_ptr[w + 1] - win_ptr[w]; ++i) {
      const double* rec = poses.data() + 12 * (size_t)(win_ptr[w] + i);
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) x_win[i].R(r, c) = rec[3 * r + c];
      for (int r = 0; r < 3; ++r) x_win[i].p(r) = rec[9 + r];
    }
    x_wins.push_back(std::move(x_win));
  }
  if (summaries) *summaries = local;
  return LVBA_OK;
}

// ---- all of runWindowBA (src/lvba_system.cpp:205-316).  After the window stage (run_window_stage) every window that was
//      solved becomes an anchor: its poses are re-aligned to the odometry start when use_window_ba_rel is set (:268-278), every
//      scan is expressed relative to the window's first odometry pose (:284-296) and the scans are merged and down-sampled into the
//      anchor cloud (:288-298, boundary B6).  Skipped windows produce no anchor, exactly as the `continue` at :265.
struct AnchorCloud { struct P3 { float x, y, z; }; std::vector<P3> points; };
template <class PoseVec>
struct WindowBAResult {
  PoseVec anchor_poses;                          // one per solved window: x_win_odom[0]
  std::vector<AnchorCloud> anchor_clouds;        // the merged, down-sampled cloud of each anchor (anchor frame)
  PoseVec rel_poses_to_anchor;                   // per frame (identity where the frame has no anchor)
  std::vector<int> anchor_index_per_frame;       // -1 where the frame's window was skipped
  std::vector<lvba_summary> summaries;           // per window
  int win_total = 0, win_skipped = 0;
};

template <class CloudPtrVec, class PoseVec>
inline int run_window_ba(const CloudPtrVec& pl_fulls, const PoseVec& x_buf_full, int window_size, double root_voxel_size,
                         const float eigen_ratio_array[4], double anchor_leaf, bool use_window_ba_rel, WindowBAResult<PoseVec>& res,
                         const lvba_lidar_opts* opts = nullptr, const std::vector<uint8_t>* pose_fixed = nullptr) {
  std::vector<PoseVec> x_wins;
  int rc = run_window_stage(pl_fulls, x_buf_full, window_size, root_voxel_size, eigen_ratio_array, x_wins, &res.summaries, nullptr, opts,
                            pose_fixed);
  if (rc != LVBA_OK) return rc;
  const int total_size = (int)std::min(pl_fulls.size(), x_buf_full.size());
  res.anchor_poses.clear(); res.anchor_clouds.clear();
  res.rel_poses_to_anchor.assign(x_buf_full.begin(), x_buf_full.begin() + total_size);
  res.anchor_index_per_frame.assign((size_t)total_size, -1);
  for (int i = 0; i < total_size; ++i) {                       // rel_poses_to_anchor_[i].setZero() = identity (:223)
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) res.rel_poses_to_anchor[i].R(r, c) = r == c ? 1.0 : 0.0; res.rel_poses_to_anchor[i].p(r) = 0.0; }
  }
  res.win_total = (int)x_wins.size(); res.win_skipped = 0;
  auto mul3 = [](const double* A, const double* B, double* C) { for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j]; };
  auto get = [](const auto& x, double* R, double* p) { for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) R[3 * r + c] = x.R(r, c); p[r] = x.p(r); } };
  std::vector<int32_t> win_ptr{0};
  std::vector<int64_t> scan_ptr{0};
  std::vector<float> xyz;
  std::vector<double> rel_all;
  int start = 0;
  for (size_t w = 0; w < x_wins.size(); ++w) {
    const int curr = (int)x_wins[w].size();
    if (res.summaries[w].termination == LVBA_TERM_SKIPPED) { ++res.win_skipped; start += curr; continue; }
    double Ro[9], po[3], Rq[9], pq[3], Ralign[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, palign[3] = {0, 0, 0};
    get(x_buf_full[start], Ro, po);                            // anchor_pose = x_win_odom[0]
    if (use_window_ba_rel) {                                   // R_align = odom0.R * opt0.R^T ; p_align = odom0.p - R_align * opt0.p
      get(x_wins[w][0], Rq, pq);
      const double Rqt[9] = {Rq[0], Rq[3], Rq[6], Rq[1], Rq[4], Rq[7], Rq[2], Rq[5], Rq[8]};
      mul3(Ro, Rqt, Ralign);
      for (int i = 0; i < 3; ++i) palign[i] = po[i] - (Ralign[3 * i] * pq[0] + Ralign[3 * i + 1] * pq[1] + Ralign[3 * i + 2] * pq[2]);
    }
    const double Rot[9] = {Ro[0], Ro[3], Ro[6], Ro[1], Ro[4], Ro[7], Ro[2], Ro[5], Ro[8]};
    const int anchor_idx = (int)res.anchor_poses.size();
    for (int j = 0; j < curr; ++j) {
      double Ra[9], pa[3];
      if (use_window_ba_rel) {                                 // x_win_aligned[j] = (R_align x.R, R_align x.p + p_align)
        double Rx[9], px[3];
        get(x_wins[w][j], Rx, px);
        mul3(Ralign, Rx, Ra);
        for (int i = 0; i < 3; ++i) pa[i] = (Ralign[3 * i] * px[0] + Ralign[3 * i + 1] * px[1] + Ralign[3 * i + 2] * px[2]) + palign[i];
      } else {
        get(x_buf_full[start + j], Ra, pa);                    // x_win_aligned = x_win_odom (:277)
      }
      double Rr[9], d[3] = {pa[0] - po[0], pa[1] - po[1], pa[2] - po[2]}, pr[3];
      mul3(Rot, Ra, Rr);                                       // rel.R = anchor.R^T * aligned.R ; rel.p = anchor.R^T (aligned.p - anchor.p)
      for (int i = 0; i < 3; ++i) pr[i] = Rot[3 * i] * d[0] + Rot[3 * i + 1] * d[1] + Rot[3 * i + 2] * d[2];
      auto& rel = res.rel_poses_to_anchor[start + j];
      for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) rel.R(r, c) = Rr[3 * r + c]; rel.p(r) = pr[r]; }
      res.anchor_index_per_frame[start + j] = anchor_idx;
      rel_all.insert(rel_all.end(), Rr, Rr + 9); rel_all.insert(rel_all.end(), pr, pr + 3);
      for (const auto& pt : pl_fulls[start + j]->points) { xyz.push_back(pt.x); xyz.push_back(pt.y); xyz.push_back(pt.z); }
      scan_ptr.push_back((int64_t)xyz.size() / 3);
    }
    win_ptr.push_back((int32_t)scan_ptr.size() - 1);
    res.anchor_poses.push_back(x_buf_full[start]);
    start += curr;
  }
  const int n_anchor = (int)win_ptr.size() - 1;
  res.anchor_clouds.assign((size_t)n_anchor, AnchorCloud());
  if (n_anchor == 0) return LVBA_OK;
  lvba_anchor_clouds* ac = nullptr;
  int64_t n_pts = 0;
  rc = lvba_anchor_clouds_create(n_anchor, win_ptr.data(), scan_ptr.data(), xyz.data(), 3, rel_all.data(), anchor_leaf, -1, &ac, &n_pts);
  if (rc != LVBA_OK) return rc;
  std::vector<int64_t> cloud_ptr((size_t)n_anchor + 1);
  std::vector<float> out((size_t)n_pts * 3);
  rc = lvba_anchor_clouds_export(ac, cloud_ptr.data(), out.data(), nullptr);
  lvba_anchor_clouds_destroy(ac);
  if (rc != LVBA_OK) return rc;
  for (int a = 0; a < n_anchor; ++a)
    for (int64_t q = cloud_ptr[a]; q < cloud_ptr[a + 1]; ++q) res.anchor_clouds[a].points.push_back({out[3 * q], out[3 * q + 1], out[3 * q + 2]});
  return LVBA_OK;
}

// ---- B4: depth rendering.  buildGridMapFromOptimized() buckets the world points of every LiDAR frame
//      (dataset_io_->pl_fulls_, x_buf_ with .R .p and the timestamp .t) into 0.5 m voxels and lists, per image, the voxels
//      of the frames within +-0.5 s; generateDepthWithVoxel() z-buffers them into one CV_32FC1 image per camera pose.
//      DepthRenderer does both on the device.  Depth images come back in one contiguous float array, image k at
//      depth.data() + k * width * height (wrap as cv::Mat(height, width, CV_32FC1, ptr) — see INTEGRATION.md).
class DepthRenderer {
 public:
  DepthRenderer() = default;
  DepthRenderer(const DepthRenderer&) = delete;
  DepthRenderer& operator=(const DepthRenderer&) = delete;
  ~DepthRenderer() { clear(); }
  void clear() { if (grid_) lvba_depth_grid_destroy(grid_); grid_ = nullptr; }

  // buildGridMapFromOptimized: clouds[i]->points[k].x/.y/.z, x_buf[i].R / .p / .t (ascending), vox = 0.5
  template <class CloudPtrVec, class PoseVec>
  int buildGridMapFromOptimized(const CloudPtrVec& pl_fulls, const PoseVec& x_buf, double vox = 0.5, lvba_depth_summary* summary = nullptr) {
    clear();
    const int F = (int)std::min(pl_fulls.size(), x_buf.size());                       // :1271
    std::vector<int64_t> scan_ptr((size_t)F + 1, 0);
    for (int j = 0; j < F; ++j) scan_ptr[j + 1] = scan_ptr[j] + (int64_t)pl_fulls[j]->points.size();
    std::vector<float> xyz((size_t)scan_ptr[F] * 3);
    for (int j = 0; j < F; ++j) {
      float* dst = xyz.data() + 3 * (size_t)scan_ptr[j];
      for (const auto& pt : pl_fulls[j]->points) { *dst++ = pt.x; *dst++ = pt.y; *dst++ = pt.z; }
    }
    std::vector<double> poses((size_t)F * 12), ts((size_t)F);
    for (int i = 0; i < F; ++i) {
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) poses[12 * i + 3 * r + c] = x_buf[i].R(r, c);
      for (int r = 0; r < 3; ++r) poses[12 * i + 9 + r] = x_buf[i].p(r);
      ts[i] = x_buf[i].t;
    }
    return lvba_depth_grid_create(F, scan_ptr.data(), xyz.data(), 3, poses.data(), ts.data(), vox, -1, &grid_, summary);
  }

  // generateDepthWithVoxel: Rcw_all[k](r,c), tcw_all[k](r) as computed at :861-864; image_ts[k] = the parsed image id
  // (NaN when parseTimestampFromName fails, :1309-1314).  depth: n_images * height * width floats, 0 = no point.
  template <class Mat3Vec, class Vec3Vec>
  int generateDepthWithVoxel(const Mat3Vec& Rcw_all, const Vec3Vec& tcw_all, const std::vector<double>& image_ts,
                             double fx, double fy, double cx, double cy, double k1, double k2, double p1, double p2,
                             int image_width, int image_height, std::vector<float>& depth, double half_w = 0.5,
                             lvba_depth_summary* summary = nullptr) {
    if (!grid_) throw std::runtime_error("lvba_b200::DepthRenderer: grid not built");
    const int M = (int)image_ts.size();
    if ((int)Rcw_all.size() != M || (int)tcw_all.size() != M) throw std::runtime_error("lvba_b200::DepthRenderer: pose / image count mismatch");   // cf. :839-846
    std::vector<double> cams((size_t)M * 12);
    for (int k = 0; k < M; ++k) {
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) cams[12 * k + 3 * r + c] = Rcw_all[k](r, c);
      for (int r = 0; r < 3; ++r) cams[12 * k + 9 + r] = tcw_all[k](r);
    }
    const double intr[8] = {fx, fy, cx, cy, k1, k2, p1, p2};
    depth.assign((size_t)M * image_width * image_height, 0.0f);
    return lvba_depth_render(grid_, M, cams.data(), image_ts.data(), half_w, intr, image_width, image_height, depth.data(), summary);
  }

  // The depth candidates of BuildTracksAndFuse3D (:1020-1038) for every keypoint: all_keypoints[i][k].x / .y, result in
  // (image, keypoint) order: kp_Xw [n_kp * 3] (zeros where invalid), kp_valid [n_kp].  The depth images stay on the device.
  template <class Mat3Vec, class Vec3Vec, class KeypointImages>
  int backproject(const Mat3Vec& Rcw_all, const Vec3Vec& tcw_all, const std::vector<double>& image_ts, const KeypointImages& all_keypoints,
                  double fx, double fy, double cx, double cy, double k1, double k2, double p1, double p2, int image_width, int image_height,
                  std::vector<double>& kp_Xw, std::vector<uint8_t>& kp_valid, double half_w = 0.5, lvba_depth_summary* summary = nullptr) {
    if (!grid_) throw std::runtime_error("lvba_b200::DepthRenderer: grid not built");
    const int M = (int)image_ts.size();
    if ((int)Rcw_all.size() != M || (int)tcw_all.size() != M || (int)all_keypoints.size() != M)
      throw std::runtime_error("lvba_b200::DepthRenderer: pose / image / keypoint count mismatch");
    std::vector<double> cams((size_t)M * 12);
    std::vector<int64_t> kp_ptr((size_t)M + 1, 0);
    for (int k = 0; k < M; ++k) {
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) cams[12 * k + 3 * r + c] = Rcw_all[k](r, c);
      for (int r = 0; r < 3; ++r) cams[12 * k + 9 + r] = tcw_all[k](r);
      kp_ptr[k + 1] = kp_ptr[k] + (int64_t)all_keypoints[k].size();
    }
    std::vector<float> uv((size_t)kp_ptr[M] * 2);
    for (int k = 0; k < M; ++k)
      for (size_t j = 0; j < all_keypoints[k].size(); ++j) { uv[2 * (kp_ptr[k] + j)] = all_keypoints[k][j].x; uv[2 * (kp_ptr[k] + j) + 1] = all_keypoints[k][j].y; }
    const double intr[8] = {fx, fy, cx, cy, k1, k2, p1, p2};
    kp_Xw.assign((size_t)kp_ptr[M] * 3, 0.0);
    kp_valid.assign((size_t)kp_ptr[M], 0);
    return lvba_depth_backproject(grid_, M, cams.data(), image_ts.data(), half_w, intr, image_width, image_height, kp_ptr.data(), uv.data(),
                                  kp_Xw.data(), kp_valid.data(), summary);
  }

 private:
  lvba_depth_grid* grid_ = nullptr;
};

// ---- B2: the flat arrays optimizeCameraPoses already builds (qs, ts, Xs, plane_n, plane_d) plus the
//      observation list it walks at :1614-1631.  obs_of_point[pi] = list of (cam_id, u, v).
struct Observation { int cam; float u, v; };

// The ABI's CSR of the per-point observation lists and the (n, d) planes; throws on size mismatches (who: the caller's name)
struct VisualCsr {
  std::vector<int64_t> obs_ptr;
  std::vector<int32_t> obs_cam;
  std::vector<float> obs_uv;
  std::vector<double> plane_nd;
};
inline VisualCsr pack_visual(int M, const std::vector<std::array<double, 3>>& ts, const std::vector<std::array<double, 3>>& Xs,
                             const std::vector<std::array<double, 3>>& plane_n, const std::vector<double>& plane_d,
                             const std::vector<std::vector<Observation>>& obs_of_point, const std::vector<uint8_t>* cam_fixed, const char* who) {
  const int64_t T = (int64_t)Xs.size();
  if ((int)ts.size() != M) throw std::runtime_error(std::string("lvba_b200::") + who + ": qs/ts size mismatch");      // cf. :1427
  if ((int64_t)plane_n.size() != T || (int64_t)plane_d.size() != T || (int64_t)obs_of_point.size() != T)
    throw std::runtime_error(std::string("lvba_b200::") + who + ": per-point array size mismatch");
  if (cam_fixed && (int)cam_fixed->size() != M) throw std::runtime_error(std::string("lvba_b200::") + who + ": cam_fixed needs one entry per camera");
  VisualCsr c;
  c.obs_ptr.assign((size_t)T + 1, 0);
  c.plane_nd.resize((size_t)T * 4);
  for (int64_t i = 0; i < T; ++i) {
    for (const auto& o : obs_of_point[i]) { c.obs_cam.push_back(o.cam); c.obs_uv.push_back(o.u); c.obs_uv.push_back(o.v); }
    c.obs_ptr[i + 1] = (int64_t)c.obs_cam.size();
    c.plane_nd[4 * i] = plane_n[i][0]; c.plane_nd[4 * i + 1] = plane_n[i][1]; c.plane_nd[4 * i + 2] = plane_n[i][2]; c.plane_nd[4 * i + 3] = plane_d[i];
  }
  return c;
}

// opts (null: the defaults) with cam_fixed (null: opts' own) in o; returns the options to pass
inline const lvba_visual_opts* with_cam_fixed(const lvba_visual_opts* opts, const std::vector<uint8_t>* cam_fixed, lvba_visual_opts& o) {
  if (!cam_fixed) return opts;
  if (opts) o = *opts; else lvba_visual_default_opts(&o);
  o.cam_fixed = cam_fixed->data();
  return &o;
}

// opts: null = lvba_visual_default_opts, plain least squares as the reference's nullptr losses (:1630, :1639).  Its
// loss_function_reproj / loss_function_plane (HuberLoss(1.0) / HuberLoss(0.1), :1585-1586) map to reproj_loss = plane_loss =
// LVBA_LOSS_HUBER with the default scales 1.0 / 0.1 (INTEGRATION.md, B2).  Camera 0 is constant, as in the reference
// (:1582-1583); cam_fixed (null: none, else one entry per camera, nonzero = constant) holds further cameras constant and
// overrides opts->cam_fixed.
inline int solve_visual(std::vector<std::array<double, 4>>& qs, std::vector<std::array<double, 3>>& ts,
                        std::vector<std::array<double, 3>>& Xs, const std::vector<std::array<double, 3>>& plane_n,
                        const std::vector<double>& plane_d, const std::vector<std::vector<Observation>>& obs_of_point,
                        double fx, double fy, double cx, double cy, double k1, double k2, double p1, double p2,
                        double sigma_px = 0.5, double sigma_plane = 0.01, const lvba_visual_opts* opts = nullptr,
                        lvba_summary* summary = nullptr, const std::vector<uint8_t>* cam_fixed = nullptr) {
  const int M = (int)qs.size();
  const int64_t T = (int64_t)Xs.size();
  const VisualCsr c = pack_visual(M, ts, Xs, plane_n, plane_d, obs_of_point, cam_fixed, "solve_visual");
  lvba_visual_opts o;
  opts = with_cam_fixed(opts, cam_fixed, o);
  const double intr[8] = {fx, fy, cx, cy, k1, k2, p1, p2};
  // qs/ts/Xs are contiguous arrays of std::array<double,N>: exactly the M*4 / M*3 / T*3 layout of the ABI
  return lvba_visual_lm(M, T, qs.empty() ? nullptr : qs[0].data(), ts.empty() ? nullptr : ts[0].data(),
                        Xs.empty() ? nullptr : Xs[0].data(), c.plane_nd.data(), c.obs_ptr.data(), c.obs_cam.data(), c.obs_uv.data(), intr,
                        sigma_px, sigma_plane, /*fixed_cam=*/0, opts, summary);
}

// solve_visual_refine_intrinsics: solve_visual on a device handle with the intrinsics a parameter block of every
// ReprojErrorWhitenedDistorted, as a Ceres user gets by passing fx_ .. d3_ to the cost functor as a parameter block instead of
// constants: the entries whose bit is set in `refine` (lvba_visual_opts::refine_intrinsics, LVBA_INTR_*) are refined, the others
// held by a SubsetManifold.  qs, ts, Xs and fx .. p2 are written back after the solve (refine = 0: the intrinsics come back
// unchanged, and the solve is solve_visual's).  opts->refine_intrinsics is ignored; a bad mask is LVBA_ERR_INVALID_ARG.
inline int solve_visual_refine_intrinsics(std::vector<std::array<double, 4>>& qs, std::vector<std::array<double, 3>>& ts,
                                          std::vector<std::array<double, 3>>& Xs, const std::vector<std::array<double, 3>>& plane_n,
                                          const std::vector<double>& plane_d, const std::vector<std::vector<Observation>>& obs_of_point,
                                          double& fx, double& fy, double& cx, double& cy, double& k1, double& k2, double& p1, double& p2,
                                          uint32_t refine, double sigma_px = 0.5, double sigma_plane = 0.01,
                                          const lvba_visual_opts* opts = nullptr, lvba_summary* summary = nullptr,
                                          const std::vector<uint8_t>* cam_fixed = nullptr) {
  const int M = (int)qs.size();
  const int64_t T = (int64_t)Xs.size();
  const VisualCsr c = pack_visual(M, ts, Xs, plane_n, plane_d, obs_of_point, cam_fixed, "solve_visual_refine_intrinsics");
  lvba_visual_opts o;
  opts = with_cam_fixed(opts, cam_fixed, o);
  lvba_visual_opts use;
  if (opts) use = *opts; else lvba_visual_default_opts(&use);
  use.refine_intrinsics = refine;
  double intr[8] = {fx, fy, cx, cy, k1, k2, p1, p2};
  lvba_visual_problem* p = nullptr;
  int rc = lvba_visual_create(M, T, qs.empty() ? nullptr : qs[0].data(), ts.empty() ? nullptr : ts[0].data(), Xs.empty() ? nullptr : Xs[0].data(),
                              c.plane_nd.data(), c.obs_ptr.data(), c.obs_cam.data(), c.obs_uv.data(), intr, sigma_px, sigma_plane,
                              /*fixed_cam=*/0, use.device, &p);
  if (rc != LVBA_OK) return rc;
  rc = lvba_visual_reset_lm(p, &use);
  if (rc == LVBA_OK) rc = lvba_visual_iterate(p, use.max_iter, summary);
  if (rc == LVBA_OK)
    rc = lvba_visual_get_state(p, qs.empty() ? nullptr : qs[0].data(), ts.empty() ? nullptr : ts[0].data(), Xs.empty() ? nullptr : Xs[0].data());
  if (rc == LVBA_OK) rc = lvba_visual_get_intrinsics(p, intr);
  lvba_visual_destroy(p);
  if (rc != LVBA_OK) return rc;
  fx = intr[0]; fy = intr[1]; cx = intr[2]; cy = intr[3]; k1 = intr[4]; k2 = intr[5]; p1 = intr[6]; p2 = intr[7];
  return LVBA_OK;
}

// solve_visual, then lvba_visual_remove_outliers(max_err_px, min_track_len), then a second solve, on one device handle: the
// solve, filter, solve-again loop of a Ceres bundle adjustment (include/lvba_b200.h, B2, states the rule).  Each solve is
// lvba_visual_reset_lm with opts (and cam_fixed) and up to opts->max_iter iterations; summary_first / summary_second (may be
// null) are their summaries.  removed (may be null) gets one entry per observation of obs_of_point, in its order: 1 for every
// observation the filter took out, those of dropped landmarks included, so that a caller can erase the same entries from its
// tr.inlier_indices.  A landmark whose observations are all removed is dropped: its Xs entry comes back as the first solve left
// it, and the caller treats it as a landmark without a plane.  qs, ts, Xs are written back after the second solve, and, when
// intr_out is not null, the handle's intrinsics (refined by both solves when opts->refine_intrinsics is set).
inline int solve_visual_remove_outliers(std::vector<std::array<double, 4>>& qs, std::vector<std::array<double, 3>>& ts,
                                        std::vector<std::array<double, 3>>& Xs, const std::vector<std::array<double, 3>>& plane_n,
                                        const std::vector<double>& plane_d, const std::vector<std::vector<Observation>>& obs_of_point,
                                        double fx, double fy, double cx, double cy, double k1, double k2, double p1, double p2,
                                        double sigma_px, double sigma_plane, const lvba_visual_opts* opts, double max_err_px,
                                        int32_t min_track_len, std::vector<std::vector<uint8_t>>* removed = nullptr,
                                        lvba_summary* summary_first = nullptr, lvba_summary* summary_second = nullptr,
                                        const std::vector<uint8_t>* cam_fixed = nullptr, double* intr_out = nullptr) {
  const int M = (int)qs.size();
  const int64_t T = (int64_t)Xs.size();
  const VisualCsr c = pack_visual(M, ts, Xs, plane_n, plane_d, obs_of_point, cam_fixed, "solve_visual_remove_outliers");
  lvba_visual_opts o;
  opts = with_cam_fixed(opts, cam_fixed, o);
  lvba_visual_opts d;
  lvba_visual_default_opts(&d);
  const lvba_visual_opts& use = opts ? *opts : d;
  const double intr[8] = {fx, fy, cx, cy, k1, k2, p1, p2};
  lvba_visual_problem* p = nullptr;
  int rc = lvba_visual_create(M, T, qs.empty() ? nullptr : qs[0].data(), ts.empty() ? nullptr : ts[0].data(), Xs.empty() ? nullptr : Xs[0].data(),
                              c.plane_nd.data(), c.obs_ptr.data(), c.obs_cam.data(), c.obs_uv.data(), intr, sigma_px, sigma_plane,
                              /*fixed_cam=*/0, use.device, &p);
  if (rc != LVBA_OK) return rc;
  std::vector<uint8_t> mask((size_t)c.obs_ptr[(size_t)T]);
  if (rc == LVBA_OK) rc = lvba_visual_reset_lm(p, &use);
  if (rc == LVBA_OK) rc = lvba_visual_iterate(p, use.max_iter, summary_first);
  if (rc == LVBA_OK) rc = lvba_visual_remove_outliers(p, max_err_px, min_track_len, mask.data(), nullptr, nullptr);
  if (rc == LVBA_OK) rc = lvba_visual_iterate(p, use.max_iter, summary_second);
  if (rc == LVBA_OK)
    rc = lvba_visual_get_state(p, qs.empty() ? nullptr : qs[0].data(), ts.empty() ? nullptr : ts[0].data(), Xs.empty() ? nullptr : Xs[0].data());
  if (rc == LVBA_OK && intr_out) rc = lvba_visual_get_intrinsics(p, intr_out);
  lvba_visual_destroy(p);
  if (rc != LVBA_OK) return rc;
  if (removed) {
    removed->assign((size_t)T, {});
    for (int64_t i = 0; i < T; ++i)
      (*removed)[(size_t)i].assign(mask.begin() + c.obs_ptr[(size_t)i], mask.begin() + c.obs_ptr[(size_t)i + 1]);
  }
  return LVBA_OK;
}

// ---- B7: BuildTracksAndFuse3D (src/lvba_system.cpp:921-1263).  all_keypoints[i][k].x/.y, all_matches[pairIndex(i,j,N)] =
//      vector<pair<int,int>> in the reference's upper-triangular pair layout (utils.hpp pairIndex), Rcw / tcw per image,
//      kp_Xw / kp_valid = the depth candidate of every keypoint in (image, keypoint) order (DepthRenderer::backproject ==
//      the loop at :1020-1038).  Fills tracks with the reference's Track fields: observations (image, keypoint) of the whole
//      component, inlier_indices, Xw_fused.  Track order, observation order and inlier sets are those of the reference up to
//      the iteration order of its unordered_maps (include/lvba_b200.h).
struct FusedTrack {
  std::vector<std::pair<int, int>> observations;
  std::vector<int> inlier_indices;
  std::array<double, 3> Xw_fused;
  int source;                    // 1 depth candidate, 2 triangulation
  double mean_reproj;
};
template <class KeypointImages, class MatchTable, class RotVec, class VecVec>
inline int build_tracks_and_fuse_3d(const KeypointImages& all_keypoints, const MatchTable& all_matches, const RotVec& Rcw_all, const VecVec& tcw_all,
                                    double fx, double fy, double cx, double cy, double d0, double d1, double d2, double d3,
                                    const std::vector<double>& kp_Xw, const std::vector<uint8_t>& kp_valid, std::vector<FusedTrack>& tracks,
                                    const lvba_fuse_opts* opts = nullptr, lvba_fuse_summary* summary = nullptr) {
  const int N = (int)all_keypoints.size();
  if ((int)Rcw_all.size() != N || (int)tcw_all.size() != N) throw std::runtime_error("lvba_b200::build_tracks_and_fuse_3d: pose / image count mismatch");
  std::vector<int64_t> kp_ptr((size_t)N + 1, 0);
  for (int i = 0; i < N; ++i) kp_ptr[i + 1] = kp_ptr[i] + (int64_t)all_keypoints[i].size();
  const int64_t n_kp = kp_ptr[N];
  if ((int64_t)kp_valid.size() != n_kp || (int64_t)kp_Xw.size() != 3 * n_kp) throw std::runtime_error("lvba_b200::build_tracks_and_fuse_3d: depth candidate size mismatch");
  std::vector<float> uv((size_t)n_kp * 2);
  for (int i = 0; i < N; ++i)
    for (size_t k = 0; k < all_keypoints[i].size(); ++k) { uv[2 * (kp_ptr[i] + k)] = all_keypoints[i][k].x; uv[2 * (kp_ptr[i] + k) + 1] = all_keypoints[i][k].y; }
  std::vector<int32_t> ma, ka, mb, kb;
  for (int i = 0; i < N - 1; ++i)                                   // the visiting order of :937-953
    for (int j = i + 1; j < N; ++j) {
      const size_t idx = (size_t)i * (size_t)N - (size_t)i * ((size_t)i + 1) / 2 + (size_t)(j - i - 1);      // pairIndex(i, j, N)
      if (idx >= all_matches.size()) continue;
      for (const auto& m : all_matches[idx]) { ma.push_back(i); ka.push_back(m.first); mb.push_back(j); kb.push_back(m.second); }
    }
  std::vector<double> cams((size_t)N * 12);
  for (int i = 0; i < N; ++i) {
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) cams[12 * i + 3 * r + c] = Rcw_all[i](r, c);
    for (int r = 0; r < 3; ++r) cams[12 * i + 9 + r] = tcw_all[i](r);
  }
  const double intr[8] = {fx, fy, cx, cy, d0, d1, d2, d3};
  lvba_track_set* h = nullptr;
  lvba_fuse_summary s;
  const int rc = lvba_tracks_fuse_create(N, kp_ptr.data(), uv.data(), (int64_t)ma.size(), ma.data(), ka.data(), mb.data(), kb.data(), cams.data(),
                                         intr, kp_Xw.data(), kp_valid.data(), opts, &h, &s);
  if (rc != LVBA_OK) return rc;
  std::vector<int64_t> obs_ptr((size_t)s.n_tracks + 1);
  std::vector<int32_t> img((size_t)s.n_obs), kp((size_t)s.n_obs);
  std::vector<uint8_t> inl((size_t)s.n_obs), src((size_t)s.n_tracks);
  std::vector<double> Xw((size_t)s.n_tracks * 3), mean((size_t)s.n_tracks);
  const int rc2 = lvba_tracks_fuse_export(h, obs_ptr.data(), img.data(), kp.data(), inl.data(), Xw.data(), src.data(), mean.data());
  lvba_tracks_fuse_destroy(h);
  if (rc2 != LVBA_OK) return rc2;
  tracks.clear();
  tracks.resize((size_t)s.n_tracks);
  for (int64_t t = 0; t < s.n_tracks; ++t) {
    FusedTrack& tr = tracks[(size_t)t];
    for (int64_t o = obs_ptr[t]; o < obs_ptr[t + 1]; ++o) {
      tr.observations.emplace_back(img[(size_t)o], kp[(size_t)o]);
      if (inl[(size_t)o]) tr.inlier_indices.push_back((int)(o - obs_ptr[t]));
    }
    tr.Xw_fused = {Xw[3 * t], Xw[3 * t + 1], Xw[3 * t + 2]};
    tr.source = src[(size_t)t]; tr.mean_reproj = mean[(size_t)t];
  }
  if (summary) *summary = s;
  return LVBA_OK;
}

}  // namespace lvba_b200
